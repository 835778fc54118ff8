"""A float64 restatement of the engine's forward, for tests that hold the kernels to their true error rather than to the
1e-3 contract tolerance.

Two modes over the same dataflow (csrc/token_kernel.cuh for one token, csrc/prefill.cuh for a pass):
- "exact": f64 activations, no quantisation. It keeps the reference's f32 cast points: the inputs of every projection
  and its outputs, the residual's f32 round trip through the output projection, sigma(r) via expf, layernorm mean and
  standard deviation rounded to f32 with E - 1 and no epsilon.
- "engine": the engine's activation pipeline on top. xs = f32(f32(f) * r) rounded to 22 mantissa bits ((bits + 2) & ~3),
  m = max|xs|, inv = f32(kQMax / m) stepped down until m * inv - kQMax < 0.5 (common.cuh quant_scale), q = rint(xs * inv),
  y = f32(m / kQMax * (q . (w - 128)) + sum_j f_j * oc_j) with oc_j = f32(128 r_j + o_j) (prefill.cuh pf_combine).
  The integer dot products are exact: |q . w'| <= 20480 * 2^22 * 128 < 2^53, so a float64 product of q against w - 128
  has no rounding in any summation order.

MUTATIONS are the kernel bugs the forward tests must catch, applied to the quantiser of every projection: a dropped
or misread limb plane, a coarser quantiser, a dequantisation scale off by one part in 65536.

Streams are independent token sequences, each on its own state (a dict of the engine's arrays, L * E doubles each),
run layer by layer over all tokens at once like the tensor-core pass: the GEMMs see every token, the token shift and
the WKV scan follow each stream."""
import os

import numpy as np

V = 50277
KQMAX = 4194303        # 2^22 - 1, csrc/common.cuh
KEYS = ("xy", "aa", "bb", "dd")
MUTATIONS = ("drop_plane0", "plane0_signed", "plane1_signed", "bits15", "scale_2^-16")

# The .bin layout, include/rwkv/rwkv/format.h: (name, dtype, element count) in file order. Counts are named by shape.
_COUNT = {"E": lambda L, E: E, "VE": lambda L, E: V * E, "LN": lambda L, E: 4 * (L + 1) * E, "L": lambda L, E: L * E,
          "V": lambda L, E: V, "4E": lambda L, E: 4 * E, "LEE": lambda L, E: L * E * E, "4LEE": lambda L, E: 4 * L * E * E,
          "4L": lambda L, E: 4 * L * E}
_LAYOUT = [
    ("xbuf", "f8", "E"), ("embed", "f4", "VE"), ("layernorms", "f8", "LN"), ("state_xy", "f8", "L"),
    ("state_aa", "f8", "L"), ("state_bb", "f8", "L"), ("state_pp", "f8", "L"), ("state_dd", "f8", "L"),
    ("buffer1", "f8", "E"), ("buffer2", "f4", "V"), ("buffer3", "f4", "E"), ("buffer4", "f4", "E"),
    ("mix_k", "f8", "L"), ("mix_v", "f8", "L"), ("mix_r", "f8", "L"), ("km", "u1", "LEE"),
    ("vm", "u1", "LEE"), ("rm", "u1", "LEE"), ("kr", "f4", "L"), ("vr", "f4", "L"), ("rr", "f4", "L"),
    ("o1", "f4", "L"), ("o2", "f4", "L"), ("o3", "f4", "L"), ("att_out", "u1", "LEE"),
    ("att_out_r", "f4", "L"), ("att_out_o", "f4", "L"), ("ffn_mix_k", "f8", "L"), ("ffn_mix_v", "f8", "L"),
    ("ffn_k", "u1", "4LEE"), ("ffn_v", "u1", "4LEE"), ("ffn_r", "u1", "LEE"), ("ffn_kr", "f4", "L"),
    ("ffn_vr", "f4", "4L"), ("ffn_rr", "f4", "L"), ("ffn_ko", "f4", "L"), ("ffn_vo", "f4", "4L"),
    ("ffn_ro", "f4", "L"), ("ffn_k_buffer", "f8", "E"), ("ffn_v_buffer", "f8", "E"), ("ffn_r_buffer", "f4", "4E"),
    ("decay", "f8", "L"), ("bonus", "f8", "L"), ("head", "u1", "VE"), ("head_r", "f4", "E"), ("head_o", "f4", "E"),
]


def tensors(path, mode="r"):
    """(L, E, {name: flat memmap of the tensor}) of a reference-format .bin."""
    L, E = (int(x) for x in np.fromfile(path, np.int64, 2))
    off, t = 16, {}
    for name, dt, count in _LAYOUT:
        n = _COUNT[count](L, E)
        t[name] = np.memmap(path, dtype=dt, mode=mode, offset=off, shape=(n,))
        off += n * np.dtype(dt).itemsize
    return L, E, t


class Model:
    """Read-only views of the tensors of a reference-format .bin. Projections are u8 [in][out] with a scale and an
    offset per input row."""

    def __init__(self, path):
        L, E, t = tensors(path)
        self.L, self.E = L, E
        self.embed = t["embed"].reshape(V, E)
        self.ln = t["layernorms"].reshape(4 * (L + 1), E)
        for k in ("mix_k", "mix_v", "mix_r", "ffn_mix_k", "ffn_mix_v", "decay", "bonus"):
            setattr(self, k, t[k].reshape(L, E))
        sq = lambda name, n_in, n_out: t[name].reshape(L, n_in, n_out)
        vec = lambda name, n: t[name].reshape(L, n)
        self.proj = {  # name -> (weights [L][in][out], scale [L][in], offset [L][in])
            "k": (sq("km", E, E), vec("kr", E), vec("o1", E)),
            "v": (sq("vm", E, E), vec("vr", E), vec("o2", E)),
            "r": (sq("rm", E, E), vec("rr", E), vec("o3", E)),
            "out": (sq("att_out", E, E), vec("att_out_r", E), vec("att_out_o", E)),
            "ffn_k": (sq("ffn_k", E, 4 * E), vec("ffn_kr", E), vec("ffn_ko", E)),
            "ffn_v": (sq("ffn_v", 4 * E, E), vec("ffn_vr", 4 * E), vec("ffn_vo", 4 * E)),
            "ffn_r": (sq("ffn_r", E, E), vec("ffn_rr", E), vec("ffn_ro", E)),
        }
        self.head = (t["head"].reshape(E, V), t["head_r"], t["head_o"])


_POOL = []


def _widen(w, centre):
    """The u8 block w as float64 (minus 128 if centre), converted by row blocks on every host core: at 7B and 14B the
    single-threaded conversion, not the product, is most of a forward's time."""
    threads = os.cpu_count() or 1
    if not _POOL:
        from concurrent.futures import ThreadPoolExecutor
        _POOL.append(ThreadPoolExecutor(threads))
    out = np.empty(w.shape)
    rows = -(-w.shape[0] // threads)

    def part(i):
        if centre:
            np.subtract(w[i:i + rows], 128.0, out=out[i:i + rows])
        else:
            out[i:i + rows] = w[i:i + rows]
    list(_POOL[0].map(part, range(0, w.shape[0], rows)))
    return out


def _product(a, w, centre):
    """a [T][N] float64 times the u8 matrix w [N][M] (minus 128 if centre), in column chunks of <= 256 MB."""
    n, m = w.shape
    out = np.empty((a.shape[0], m))
    step = max(1, (1 << 25) // n)
    for c in range(0, m, step):
        out[:, c:c + step] = a @ _widen(w[:, c:c + step], centre)
    return out


def round22(x):
    """f32 -> f32 rounded to 22 mantissa bits, as the engine rounds every activation it quantises (exchange.cuh)."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((b + np.uint32(2)) & np.uint32(0xFFFFFFFC)).view(np.float32)


def quant_inv(m, qmax=KQMAX):
    """Per element of m (f32 >= 0) the quantiser's scale as common.cuh quant_scale computes it, 0 where m == 0:
    inv = f32(qmax * f32(1 / m)) (the reciprocal after its Newton step is the rounded 1 / m), then one ulp down while
    f32(m * inv - qmax) >= 0.5, so |q| <= qmax. Where the outliers of a model make max|xs| 300 times the typical
    element, a scale one ulp away from the engine's moves the state by 1e-4, so this follows the kernel's steps."""
    m = np.asarray(m, np.float32)
    pos = m > 0
    r = np.float32(1) / np.where(pos, m, np.float32(1))
    inv = np.where(pos, np.float32(qmax) * r, np.float32(0)).astype(np.float32)
    m64 = m.astype(np.float64)
    for _ in range(3):  # m * inv - qmax is exact in float64 (two 24-bit significands), then rounded like the fma
        over = pos & ((m64 * inv.astype(np.float64) - qmax).astype(np.float32) >= 0.5)
        inv = np.where(over, np.nextafter(inv, np.float32(0)), inv)
    return inv


def project(f, w, r, o, mode, mutation=None):
    """y[t][k] = sum_j f[t][j] * (w[j][k] * r[j] + o[j]) for f32 activations f [T][N]; f32 [T][M]."""
    f64 = f.astype(np.float64)
    r64, o64 = np.asarray(r, np.float64), np.asarray(o, np.float64)
    if mode == "exact":
        return (_product(f64 * r64, w, False) + (f64 @ o64)[:, None]).astype(np.float32)
    qmax = 2 ** 14 - 1 if mutation == "bits15" else KQMAX
    xs = round22((f64 * r64).astype(np.float32))
    m = np.abs(xs).max(axis=1)
    inv = quant_inv(m, qmax)
    q = np.rint(xs.astype(np.float64) * inv.astype(np.float64)[:, None])
    if mutation in ("drop_plane0", "plane0_signed", "plane1_signed"):
        qi = q.astype(np.int64)
        if mutation == "drop_plane0":
            qi &= ~0xFF
        elif mutation == "plane0_signed":
            qi -= 256 * ((qi & 0xFF) >= 128)
        else:
            qi -= 65536 * (((qi >> 8) & 0xFF) >= 128)
        q = qi.astype(np.float64)
    S = m.astype(np.float64) * (1.0 / qmax)
    if mutation == "scale_2^-16":
        S = S * (1.0 + 2.0 ** -16)
    oc = (128.0 * r64 + o64).astype(np.float32).astype(np.float64)   # aux_kernels.cuh k_centre_offsets
    return (S[:, None] * _product(q, w, True) + (f64 @ oc)[:, None]).astype(np.float32)


def layernorm(x, w, b):
    """Rows of x [T][E] (f64): the sum rounded to f32, the mean f32(sum) / f32(E), the unbiased variance around that
    mean rounded to f32, sqrtf, no epsilon (rwkv.cu:412-465, 40-57; prefill.cuh pf_row_stats)."""
    E = x.shape[1]
    acc = x.sum(axis=1).astype(np.float32)
    mean_f = (acc / np.float32(E)).astype(np.float64)
    q = ((x - mean_f[:, None]) ** 2).sum(axis=1)
    sd = np.sqrt(q.astype(np.float32) / np.float32(E - 1)).astype(np.float32)
    mean = acc.astype(np.float64) / E
    return w * ((x - mean[:, None]) * (1.0 / sd.astype(np.float64))[:, None]) + b


def zero_state(L, E):
    return {k: np.zeros(L * E) for k in ("xy", "aa", "bb", "pp", "dd")}


def expf(x, nudge=None):
    """f32 exp of f32 x, correctly rounded (CUDA's expf is within 2 ulp; numpy's float32 exp is not correctly rounded
    on 4 of 10 arguments). nudge: a generator that moves a random half of the results one ulp up."""
    with np.errstate(over="ignore"):
        e = np.exp(np.asarray(x, np.float64)).astype(np.float32)
    if nudge is not None:
        e = np.where(nudge.random(e.shape) < 0.5, np.nextafter(e, np.float32(np.inf)), e)
    return e


def forward(model, streams, states=None, mode="engine", mutation=None, nudge=None, mutation_layers=None, inputs=None):
    """Run every stream (a list of token ids) from its state (None: zeros). Returns (logits [T_s][V] f32 per stream,
    the state after each stream's last token). nudge: a seed; a random half of the expf results of sigma(r) in the WKV
    then come out one ulp higher (see sensitivity).

    mutation_layers: the layers whose projections `mutation` applies to (None: every layer and the head), a bug that
    hits one layer of many. inputs: a dict that a run without mutation fills with the residual stream entering each
    layer ("x", [L] of [T][E]) and its states ("states"); a run of the same streams and states with mutation_layers
    given that dict starts at the first mutated layer, since every layer before it computes what the plain run did."""
    nudge = None if nudge is None else np.random.default_rng(nudge)
    L, E = model.L, model.E
    sts = [{k: np.array(s[k], np.float64).reshape(L, E) for k in ("xy", "aa", "bb", "pp", "dd")}
           for s in (states or [zero_state(L, E) for _ in streams])]
    toks = np.concatenate([np.asarray(s, np.int64) for s in streams])
    sid = np.concatenate([np.full(len(s), i) for i, s in enumerate(streams)])
    first = np.concatenate([np.arange(len(s)) == 0 for s in streams])
    last = np.concatenate([np.arange(len(s)) == len(s) - 1 for s in streams])
    hit = lambda l: mutation_layers is None or l in mutation_layers
    proj = lambda f, name, l: project(f, *(a[l] for a in model.proj[name]), mode=mode,
                                      mutation=mutation if hit(l) else None)
    l0 = 0
    if inputs is not None and mutation is None:
        inputs["x"] = []
    elif inputs is not None:
        assert mutation_layers and nudge is None and "states" in inputs, "inputs: a plain run fills it, a mutated one reads it"
        l0 = min(mutation_layers)
        for st, done in zip(sts, inputs["states"]):
            for k in st:
                st[k][:l0] = done[k].reshape(L, E)[:l0]

    def shifted(cur, key, l):
        """Token-shift input of every row: the previous row of its stream, or the stream's state at its first row."""
        prev = np.roll(cur, 1, axis=0)
        for t in np.flatnonzero(first):
            prev[t] = sts[sid[t]][key][l]
        for t in np.flatnonzero(last):
            sts[sid[t]][key][l] = cur[t]
        return prev

    def mix(m, cur, prev):
        return (m * cur + (1.0 - m) * prev).astype(np.float32)

    ln = model.ln
    x = layernorm(np.asarray(model.embed[toks], np.float64), ln[0], ln[1]) if l0 == 0 else inputs["x"][l0]
    for l in range(l0, L):
        if inputs is not None and mutation is None:
            inputs["x"].append(x)
        a = layernorm(x, ln[4 * l + 2], ln[4 * l + 3])
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
            y = (1.0 / (1.0 + expf(-r[t], nudge).astype(np.float64))) * y
            ek = np.exp(kf)
            aa, bb = (aa + ek * vv) * ew, (bb + ek) * ew
            if last[t]:
                st["aa"][l], st["bb"][l] = aa, bb
            rw[t] = y.astype(np.float32)
        x = (x.astype(np.float32) + proj(rw, "out", l)).astype(np.float64)
        b = layernorm(x, ln[4 * (l + 1)], ln[4 * (l + 1) + 1])
        prev = shifted(b, "dd", l)
        sr = (1.0 / (1.0 + np.exp(-proj(mix(model.ffn_mix_v[l], b, prev), "ffn_r", l).astype(np.float64)))).astype(np.float32)
        kk = np.maximum(proj(mix(model.ffn_mix_k[l], b, prev), "ffn_k", l), np.float32(0))
        x = x + (proj(kk * kk, "ffn_v", l) * sr).astype(np.float64)
    h = layernorm(x, ln[4 * L + 2], ln[4 * L + 3]).astype(np.float32)
    logits = project(h, *model.head, mode=mode, mutation=mutation if mutation_layers is None else None)
    ends = np.cumsum([len(s) for s in streams])
    out = np.split(logits, ends[:-1])
    final = [{k: s[k].reshape(-1) for k in s} for s in sts]
    if inputs is not None and mutation is None:
        inputs["states"] = final
    return out, final


def sensitivity(model, streams, states=None, seeds=(1, 2)):
    """How far the engine restatement moves when a random half of the expf results of sigma(r) come out one ulp higher:
    (logits, state) as in worst(), the larger over `seeds`. A restatement that is not bit-exact cannot be held closer
    to the kernel than this. It is ~1e-7 on the plain models; on the outlier-channel model, where one K quantiser step
    is 300 times coarser for every other channel, a single q that rounds the other way is visible and it is ~3e-5."""
    base_l, base_s = forward(model, streams, states)
    le = se = 0.0
    for seed in seeds:
        l, s = forward(model, streams, states, nudge=seed)
        a, b, _ = worst(l, base_l, s, base_s, model.L, model.E)
        le, se = max(le, a), max(se, b)
    return le, se


def case_tol(model, streams, states=None):
    """The tolerance of a case against the engine restatement: TOL, or 4 times the restatement's sensitivity where that
    is larger (logits and state separately)."""
    le, se = sensitivity(model, streams, states)
    return max(TOL, 4 * le), max(TOL, 4 * se)


# -- how far apart two forwards are -------------------------------------------------------------------------------

def logits_err(got, ref):
    """Worst over tokens of max|got - ref| relative to max|ref| of the token."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float((np.abs(got - ref).max(axis=-1) / np.maximum(np.abs(ref).max(axis=-1), 1e-30)).max())


def state_errs(got, ref, L, E):
    """Per array, the worst over layers of max|got - ref| relative to max|ref| of that layer; bb (> 0, with channels
    10^-9 of its maximum) element by element relative to itself."""
    out = {}
    for k in KEYS:
        g = np.asarray(got[k], np.float64)[:L * E].reshape(L, E)
        r = np.asarray(ref[k], np.float64)[:L * E].reshape(L, E)
        if k == "bb":
            out[k] = float((np.abs(g - r) / np.maximum(np.abs(r), 1e-300)).max())
        else:
            out[k] = float((np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-30)).max())
    return out


def worst(logits_got, logits_ref, states_got, states_ref, L, E):
    """(worst logits error, worst state error, name of the worst state array) over every stream."""
    le = max(logits_err(g, r) for g, r in zip(logits_got, logits_ref))
    se, sk = 0.0, "-"
    for g, r in zip(states_got, states_ref):
        for k, e in state_errs(g, r, L, E).items():
            if not e <= se:
                se, sk = e, k
    return le, se, sk


# -- the forward cases of tests/test_numerics_gpu.py ----------------------------------------------------------------
# The stress and edge cases run the same 8 tokens on both paths, so the two kernels are compared on the same input.
# path: "decode" = the decode kernel token by token (prefill 0), "tc" = one GPT chunk on the tensor cores, "parralel"
# = MODE::PARRALEL (token i alone on slot i), "ragged" = one forward_streams pass on slots that hold state.
TOL = 1e-5              # the engine against the "engine" restatement, logits and every state array
DECODE_WIDTHS = [144, 256, 272, 768, 784, 1024, 1040, 2048, 2560, 3072, 3600, 4096, 5104, 5120]  # one per (CPL, FULL)
CHUNKS = {144: 20, 272: 40, 784: 72, 1024: 128, 1040: 200}  # Tp = 32, 64, 96, 128; 1040 x 200 = two passes, K tail
STRESS = ("outliers", "tiny_residual", "offset_residual", "negative_keys", "one_positive_key")
RAGGED_LENS = (1, 7, 33, 20)
OUTLIER = {"xy": 1e2, "dd": 1e4}  # the K input goes through exp(k): 10^4 there overflows f64, in the reference too


def _case(cid, L, E, path, T, kind=None, edge=None):
    return {"id": cid, "L": L, "E": E, "path": path, "T": T, "kind": kind, "edge": edge}


def cases():
    out = [_case("decode-%d" % E, 1 if E >= 4096 else 2, E, "decode", 8) for E in DECODE_WIDTHS]
    out += [_case("tc-%dx%d" % (E, T), 2, E, "tc", T) for E, T in CHUNKS.items()]
    out += [_case("parralel-768", 2, 768, "parralel", 16), _case("ragged-784", 2, 784, "ragged", sum(RAGGED_LENS))]
    for kind in STRESS:
        out += [_case("%s-%s" % (p, kind), 2, 768, p, T, kind=kind) for p, T in (("decode", 8), ("tc", 8))]
    for key in OUTLIER:
        out += [_case("%s-%s-outlier" % (p, key), 2, 768, p, T, edge=key) for p, T in (("decode", 8), ("tc", 8))]
    return out


def inputs(case, model):
    """(streams, initial states or None) of a case."""
    from util import token_stream
    E, T = case["E"], case["T"]
    if case["path"] == "parralel":
        return [[t] for t in token_stream(T, seed=E + 1)], None
    if case["path"] == "ragged":
        streams = [token_stream(n, seed=E + i) for i, n in enumerate(RAGGED_LENS)]
        return streams, [forward(model, [token_stream(3, seed=100 + i)])[1][0] for i in range(len(streams))]
    if case["edge"] is None:
        return [token_stream(T, seed=E)], None
    # one element of the token-shift state (the K/V/R input for xy, the ffn input for dd) far above the rest, negative
    st = forward(model, [token_stream(2, seed=7)])[1][0]
    a = st[case["edge"]].reshape(model.L, E)
    for l in range(model.L):
        a[l, E // 3 + l] = -OUTLIER[case["edge"]] * np.abs(a[l]).max()
    return [token_stream(T, seed=E)], [st]


def case_model(case, make_model, tmp_dir):
    """Path of the case's model: the synthetic L x E model, or a stress_model copy of it."""
    import os

    from util import stress_model
    src = make_model(case["L"], case["E"])
    if case["kind"] is None:
        return src
    dst = os.path.join(tmp_dir, "%s_L%d_E%d.bin" % (case["kind"], case["L"], case["E"]))
    if not os.path.exists(dst):
        stress_model(src, dst, case["kind"], L=case["L"], E=case["E"])
    return dst


# -- the cases of tests/test_depth_numerics_gpu.py ------------------------------------------------------------------
# Production depth and width. Each model's cases are restated together, as independent streams of one pass, since the
# restatement's cost is one conversion of every weight per pass; each stream comes out as it would alone.
DEPTH_L = 3
WIDE = {4096: {"decode": 8, "tc": 128}, 5104: {"decode": 8, "tc": 140}, 5120: {"decode": 8}}  # tc at 5104: two passes
# The ragged calls at 3 x 4096: 24 one-token rows (generate_streams' decode step) and three streams, 128 tokens a call,
# on 27 slots that hold state; the second call runs on the state the first wrote.
RAGGED_CALLS = ((1,) * 10 + (40,) + (1,) * 7 + (33,) + (1,) * 7 + (31,),
                (1,) * 5 + (37,) + (1,) * 12 + (45,) + (1,) * 7 + (22,))
RAGGED_SLOTS = tuple((5 * i + 3) % 27 for i in range(27))
BENCH_CASES = {"7b": {"decode": 16, "tc": 64, "greedy": 32}, "14b": {"decode": 8, "tc": 64},
               "1b5": {"long": 1024, "switch": 264}}
SWITCH = (200, 24, 40)   # 1b5: tensor cores, then the decode kernel, then tensor cores again, on one state


def wide_streams(E):
    """(case ids, streams) of the single-stream cases of width E of WIDE, each from the zero state."""
    from util import token_stream
    ids = ["%s-%dx%d" % (p, DEPTH_L, E) for p in WIDE[E]]
    return ids, [token_stream(T, seed=E + i) for i, T in enumerate(WIDE[E].values())]


def depth_passes(group, model, greedy=None):
    """The restatement passes of a group (a width of WIDE or a workload of BENCH_CASES), in order: a list of
    (case ids, streams, initial states or None). A "ragged-2" pass starts from the state a "ragged-1" pass ends in,
    so passes() resolves its states (None here) from the previous pass. greedy: the tokens the 7B greedy chain fed the
    device (the reference's greedy tokens where no device ran, on the host)."""
    from util import reference_golden, token_stream
    if group in WIDE:
        ids, streams = wide_streams(group)
        if group != 4096:
            return [(ids, streams, None)]
        pre = forward(model, [token_stream(3, seed=100 + i) for i in range(len(RAGGED_SLOTS))])[1]
        rag = [[[int(t) for t in np.random.default_rng(1000 * c + i).integers(0, V, size=n)] for i, n in enumerate(lens)]
               for c, lens in enumerate(RAGGED_CALLS)]
        first = (ids + ["ragged-1"] * len(rag[0]), streams + rag[0], [zero_state(model.L, model.E)] * len(streams) + pre)
        return [first, (["ragged-2"] * len(rag[1]), rag[1], None)]
    g = [int(t) for t in reference_golden(group)["tokens"]]
    ids, streams = [], []
    for what, T in BENCH_CASES[group].items():
        ids.append("%s-%s" % (what, group))
        streams.append(token_stream(T, seed=2048) if what == "switch" else
                       list(greedy) if what == "greedy" and greedy is not None else g[:T])
    return [(ids, streams, None)]


def stream_tols(model, streams, states, base, seeds=(1, 2)):
    """case_tol of every stream of one pass, from the pass restated plainly (base) and nudged with each of `seeds`."""
    tol = [[TOL, TOL] for _ in streams]
    for seed in seeds:
        l, s = forward(model, streams, states, nudge=seed)
        for i in range(len(streams)):
            le, se, _ = worst([l[i]], [base[0][i]], [s[i]], [base[1][i]], model.L, model.E)
            tol[i] = [max(tol[i][0], 4 * le), max(tol[i][1], 4 * se)]
    return [tuple(t) for t in tol]


def passes(group, model, greedy=None, inputs=False):
    """depth_passes with each pass restated: a list of dicts of ids, streams, states (initial), logits, final (states),
    tols and, with inputs, the per-layer inputs of forward(inputs=) for layer-restricted mutations."""
    out = []
    for ids, streams, states in depth_passes(group, model, greedy):
        if states is None and out:
            states = [out[-1]["final"][i] for i, c in enumerate(out[-1]["ids"]) if c == "ragged-1"]
        rec = {} if inputs else None
        logits, final = forward(model, streams, states, inputs=rec)
        out.append({"ids": ids, "streams": streams, "states": states, "logits": logits, "final": final, "inputs": rec,
                    "tols": stream_tols(model, streams, states, (logits, final))})
    return out
