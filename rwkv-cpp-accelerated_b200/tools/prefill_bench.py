"""Batched path (wgmma integer GEMMs) against the token-by-token decode kernel for T tokens in one call:
wall time of `forward` (host timed, synchronous call, logits of the last token only in GPT mode).
usage: python prefill_bench.py [workload=7b] [T ...]"""
import importlib
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
workload = sys.argv[1] if len(sys.argv) > 1 else "7b"
Ts = [int(a) for a in sys.argv[2:]] or [2, 4, 8, 16, 32, 64, 128]
eng = pkg.Engine(bench.model_path(workload, pkg), max_gpt=max(Ts))
eng.set_option("prefill_min", 2)
rng = np.random.default_rng(1)


def run(T, batched, mode, graph=1):
    eng.set_option("prefill", 1 if batched else 0)
    eng.set_option("prefill_graph", graph)
    toks = rng.integers(0, 50000, T)
    best = 1e9
    for _ in range(4):  # (the first batched call of a shape records its CUDA graph)
        eng.state_zero()
        t0 = time.perf_counter()
        eng.forward(toks, mode=mode, want_logits=False)
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


print("%-6s %-9s %12s %12s %12s %9s %14s" % ("T", "mode", "batched ms", "no-graph ms", "by-token ms", "ratio", "batched tok/s"))
for mode, name in ((1, "GPT"), (0, "PARRALEL")):
    for T in Ts:
        if mode == 0 and T > eng.max_gpt:
            continue
        a, a0, b = run(T, True, mode), run(T, True, mode, graph=0), run(T, False, mode)
        print("%-6d %-9s %12.3f %12.3f %12.3f %9.2f %14.0f" % (T, name, a, a0, b, b / a, T / a * 1e3), flush=True)
eng.close()
