"""Phase-level timing of the persistent token kernel from %globaltimer stamps (thread 0 of every CTA).
usage: python trace_token.py [workload=7b] [tokens=4]"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
workload = sys.argv[1] if len(sys.argv) > 1 else "7b"
ntok = int(sys.argv[2]) if len(sys.argv) > 2 else 4
L, E = bench.SHAPES[workload]
eng = pkg.Engine(bench.model_path(workload, pkg))
eng.set_option("trace", 1)
for kv in sys.argv[3:]:
    k, v = kv.split("=")
    eng.set_option(k, v)
tok = bench.SEED_TOKEN
for _ in range(ntok):
    tok = eng.forward_greedy(tok)
tr = eng.read_trace().astype(np.int64)
n = int((tr[0] > 0).sum())
tr = tr[:, :n]
t0 = tr[:, 0].min()
tr = tr - t0
out_dir = os.path.join(ROOT, "gpurun_out")
if os.path.isdir(out_dir):
    np.save(os.path.join(out_dir, "trace_raw_%s.npy" % workload), tr.astype(np.int32))
print("stamps per CTA", n, "token time us", (tr[:, -1].max()) / 1e3)
# stamp layout (token_kernel.cuh): start | ln0+stats, publish | per layer 21 | head 4 | end
ST = ["st.sync", "st.pub", "st.first", "st.all", "st.calc", "st.ret"]  # slice_stats
GA = ["g.meet", "g.words", "g.max", "g.sync", "g.quant"]                    # gather
names = ["ln0." + x for x in ST] + ["ln0.pub"]
layer = ["kvr." + x for x in GA] + ["kvr.gemv", "kvr.epi"] + \
        ["out." + x for x in GA] + ["out.gemv", "out.resid"] + ["out." + x for x in ST] + ["out.ln2pub"] + \
        ["rk." + x for x in GA] + ["rk.gemv", "rk.epi"] + ["fr.gemv", "fr.epi"] + \
        ["v." + x for x in GA] + ["v.gemv", "v.resid"] + ["v." + x for x in ST] + ["v.ln1pub", "v.end"]
for _ in range(L):
    names += layer
names += ["head." + x for x in GA] + ["head.gemv", "head.epi", "done"]
d = np.diff(tr, axis=1)  # [cta, n-1]
if d.shape[1] != len(names):
    print("WARNING: %d segments recorded, %d expected" % (d.shape[1], len(names)))
agg = {}
for i, nm in enumerate(names[:d.shape[1]]):
    agg.setdefault(nm, []).append(d[:, i])
print("%-12s %8s %8s %8s %8s   (us; mean over CTAs and layers, median, min/max of per-CTA means)" % ("segment", "mean", "median", "min", "max"))
tot = 0
groups = {}
for nm, lst in agg.items():
    a = np.stack(lst, 1) / 1e3  # [cta, layers]
    tot += a.mean(0).sum()
    print("%-12s %8.2f %8.2f %8.2f %8.2f   x%d" % (nm, a.mean(), np.median(a), a.mean(1).min(), a.mean(1).max(), a.shape[1]))
    kind = ".".join(nm.split(".")[1:])
    if nm.split(".")[0] in ("kvr", "out", "rk", "fr", "v"):
        groups[kind] = groups.get(kind, 0.0) + a.mean()
print("sum of means (us):", round(tot, 1))
print("per layer (us):", {k: round(v, 2) for k, v in groups.items()}, "total", round(sum(groups.values()), 2))

# ---- tile-level: how far ahead of the consumers does the producer run? -------------------------
tt = eng.read_tile_trace().astype(np.int64)
if os.path.isdir(out_dir):
    np.save(os.path.join(out_dir, "tile_raw_%s%s.npy" % (workload, os.environ.get("TRACE_TAG", ""))), (tt[:, :8] - t0).astype(np.int32))
    np.save(os.path.join(out_dir, "trace_raw_%s%s.npy" % (workload, os.environ.get("TRACE_TAG", ""))), tr[:8].astype(np.int32))
for cta in (0, 77):
    issue, ready = tt[0, cta], tt[1, cta]
    n_t = int((issue > 0).sum())
    issue, ready = (issue[:n_t] - t0) / 1e3, (ready[:n_t] - t0) / 1e3
    d_t = np.diff(ready)
    inside = d_t[d_t < 1.2]  # consecutive tiles of one streaming phase (gaps are phase boundaries)
    print("CTA %d: tiles %d; tile period inside a phase (us): median %.3f mean %.3f p90 %.3f" % (
        cta, n_t, np.median(inside), inside.mean(), np.percentile(inside, 90)))
    lead = ready - issue
    print("CTA %d: lead of the producer (issue -> consumed), us: median %.2f p10 %.2f p90 %.2f" % (
        cta, np.median(lead), np.percentile(lead, 10), np.percentile(lead, 90)))
print("stamps per layer:", len(layer))
eng.close()
