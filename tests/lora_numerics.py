"""The float64 restatement of tests/numerics.py with LoRA adapters (include/rwkv_b200.h, "adapters").

An adapted projection of a bound token gets delta = s * B (A f) in f64 added before its f32 rounding, where f is the
f32 activation the projection quantises (prefill.cuh pf_combine, k_ad_shrink, k_ad_expand). Everything else is
numerics.py's arithmetic, reused through its helpers: the dataflow of numerics.forward with a delta on each projection.

An adapter here is a dict of "scale" and "A" / "B", which map a key of numerics.Model.proj ("k", "v", "r", "out",
"ffn_k", "ffn_v", "ffn_r") to arrays [L][r][in] and [L][out][r]."""
import numpy as np

import numerics as nm


def adapter_delta(adapter, name, l, f):
    """The adapter's correction of projection `name` of layer l for f32 inputs f [T][N]: s * B[l] (A[l] f) in f64,
    [T][M]; None where there is no adapter or it lacks the projection."""
    if adapter is None or name not in adapter["A"]:
        return None
    A, B = (np.asarray(adapter[k][name][l], np.float64) for k in ("A", "B"))
    return adapter["scale"] * ((f.astype(np.float64) @ A.T) @ B.T)


def project(f, w, r, o, mode, delta=0.0):
    """numerics.project (no mutation) with delta [T][M] added before the f32 rounding."""
    f64 = f.astype(np.float64)
    r64, o64 = np.asarray(r, np.float64), np.asarray(o, np.float64)
    if mode == "exact":
        return (nm._product(f64 * r64, w, False) + (f64 @ o64)[:, None] + delta).astype(np.float32)
    xs = nm.round22((f64 * r64).astype(np.float32))
    m = np.abs(xs).max(axis=1)
    inv = nm.quant_inv(m)
    q = np.rint(xs.astype(np.float64) * inv.astype(np.float64)[:, None])
    S = m.astype(np.float64) * (1.0 / nm.KQMAX)
    oc = (128.0 * r64 + o64).astype(np.float32).astype(np.float64)
    return (S[:, None] * nm._product(q, w, True) + (f64 @ oc)[:, None] + delta).astype(np.float32)


def forward(model, streams, adapters, states=None, mode="engine"):
    """numerics.forward with adapters[i] (an adapter or None) applied to every token of stream i. Returns (logits
    [T_s][V] f32 per stream, the state after each stream's last token)."""
    L, E = model.L, model.E
    sts = [{k: np.array(s[k], np.float64).reshape(L, E) for k in ("xy", "aa", "bb", "pp", "dd")}
           for s in (states or [nm.zero_state(L, E) for _ in streams])]
    toks = np.concatenate([np.asarray(s, np.int64) for s in streams])
    sid = np.concatenate([np.full(len(s), i) for i, s in enumerate(streams)])
    first = np.concatenate([np.arange(len(s)) == 0 for s in streams])
    last = np.concatenate([np.arange(len(s)) == len(s) - 1 for s in streams])

    def proj(f, name, l):
        delta = np.zeros((len(f), model.proj[name][0].shape[2]))
        for i, ad in enumerate(adapters):
            d = adapter_delta(ad, name, l, f[sid == i])
            if d is not None:
                delta[sid == i] = d
        return project(f, *(a[l] for a in model.proj[name]), mode=mode, delta=delta)

    def shifted(cur, key, l):
        prev = np.roll(cur, 1, axis=0)
        for t in np.flatnonzero(first):
            prev[t] = sts[sid[t]][key][l]
        for t in np.flatnonzero(last):
            sts[sid[t]][key][l] = cur[t]
        return prev

    def mix(m, cur, prev):
        return (m * cur + (1.0 - m) * prev).astype(np.float32)

    ln = model.ln
    x = nm.layernorm(np.asarray(model.embed[toks], np.float64), ln[0], ln[1])
    for l in range(L):
        a = nm.layernorm(x, ln[4 * l + 2], ln[4 * l + 3])
        prev = shifted(a, "xy", l)
        k = proj(mix(model.mix_k[l], a, prev), "k", l)
        v = proj(mix(model.mix_v[l], a, prev), "v", l)
        r = proj(mix(model.mix_r[l], a, prev), "r", l)
        rw = np.empty_like(k)
        u, wd = model.bonus[l], model.decay[l]
        ew = np.exp(wd)
        for t in range(len(toks)):
            st = sts[sid[t]]
            if first[t]:
                aa, bb = st["aa"][l].copy(), st["bb"][l].copy()
            kf, vv = k[t].astype(np.float64), v[t].astype(np.float64)
            e1 = np.exp(u + wd + kf)
            y = (aa + e1 * vv) / (bb + e1)
            y = (1.0 / (1.0 + nm.expf(-r[t]).astype(np.float64))) * y
            ek = np.exp(kf)
            aa, bb = (aa + ek * vv) * ew, (bb + ek) * ew
            if last[t]:
                st["aa"][l], st["bb"][l] = aa, bb
            rw[t] = y.astype(np.float32)
        x = (x.astype(np.float32) + proj(rw, "out", l)).astype(np.float64)
        b = nm.layernorm(x, ln[4 * (l + 1)], ln[4 * (l + 1) + 1])
        prev = shifted(b, "dd", l)
        sr = (1.0 / (1.0 + np.exp(-proj(mix(model.ffn_mix_v[l], b, prev), "ffn_r", l).astype(np.float64)))).astype(np.float32)
        kk = np.maximum(proj(mix(model.ffn_mix_k[l], b, prev), "ffn_k", l), np.float32(0))
        x = x + (proj(kk * kk, "ffn_v", l) * sr).astype(np.float64)
    h = nm.layernorm(x, ln[4 * L + 2], ln[4 * L + 3]).astype(np.float32)
    logits = nm.project(h, *model.head, mode=mode)
    ends = np.cumsum([len(s) for s in streams])
    return np.split(logits, ends[:-1]), [{k: s[k].reshape(-1) for k in s} for s in sts]
