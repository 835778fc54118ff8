"""LoRA adapters bound to state slots: what they cost on the tensor-core pass.

For R = 8, 32 and 128 one-token rows (each on its own slot), in these configurations, alternating in one run:
  none      no slot bound
  r8 / r16 / r64   every row bound to one adapter of that rank (all seven projections)
  4x16 / 16x16     row i bound to adapter i mod 4 (or 16), each of rank 16
it reports the time of one pass (forward_streams with the device arg-max, synchronised) and the ms per step of
generate_streams (arg-max, --new tokens per row). Host timer around calls that return synchronised; every shape is
warmed first (its first call records the pass's CUDA graph); each entry is the best of --rounds rounds. The card's name
and power limit are read in the same run.

--profile runs one pass of each configuration at 128 rows under torch.profiler instead, and prints the CUDA time per
kernel name (k_ad_shrink and k_ad_expand are the adapter kernels) and the pass total.
usage: python adapter_bench.py [workload=7b] [--new N] [--rounds R] [--profile]"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

ROWS = (8, 32, 128)
CONFIGS = (("none", 0, 0), ("r8", 8, 1), ("r16", 16, 1), ("r64", 64, 1), ("4x16", 16, 4), ("16x16", 16, 16))


def adapter_dict(pkg, L, E, rank, seed):
    """A random adapter of `rank` over all seven projections, in Engine.add_adapter's key naming."""
    rng = np.random.default_rng(seed)
    w = {}
    for name in pkg.engine.ADAPTER_MATRICES:
        n_in, n_out = pkg.engine.adapter_dims(name, E)
        A = (rng.standard_normal((rank, n_in), np.float32) * n_in ** -0.5)
        B = (rng.standard_normal((n_out, rank), np.float32) * 0.01)
        for l in range(L):   # the same values in every layer; each layer is still its own copy on the device
            w["blocks.%d.%s.lora_A" % (l, name)] = A
            w["blocks.%d.%s.lora_B" % (l, name)] = B
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--new", type=int, default=32, help="tokens generated per row")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    L, E = bench.SHAPES[args.workload]
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(ROWS))
    ids = {}
    for rank in (8, 64):
        ids[(rank, 0)] = eng.add_adapter(adapter_dict(pkg, L, E, rank, rank), float(rank))
    for i in range(16):
        ids[(16, i)] = eng.add_adapter(adapter_dict(pkg, L, E, 16, 100 + i), 16.0)
    print("workload %s (L=%d, E=%d); an adapter holds %.1f MB per unit of rank" % (args.workload, L, E, 20 * E * L * 4 / 1e6),
          flush=True)

    def bind(cfg):
        _, rank, k = cfg
        for s in range(max(ROWS)):
            eng.bind_adapter(s, ids[(rank, s % k)] if k else None)

    rng = np.random.default_rng(1)
    first = {R: [int(t) for t in rng.integers(0, 50000, R)] for R in ROWS}

    def one_pass(R):
        eng.forward_streams([(s, [t]) for s, t in enumerate(first[R])], want_logits=False, want_next=True)

    def generate(R):
        out = eng.generate_streams([(s, t) for s, t in enumerate(first[R])], args.new)
        assert all(len(o) == args.new for o in out)

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for cfg in CONFIGS:
            bind(cfg)
            one_pass(128)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                one_pass(128)
            per = {}
            for ev in prof.events():
                if ev.device_type.name == "CUDA":
                    key = ev.name.split("<")[0].split("(")[0]
                    per[key] = per.get(key, 0.0) + ev.device_time / 1e3
            total = sum(per.values())
            ad = sum(v for k, v in per.items() if "k_ad_" in k)
            print("\n%s, 128 rows: kernels %.3f ms, adapter kernels %.3f ms (%.1f %%)" % (cfg[0], total, ad, 100 * ad / total))
            for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:8]:
                print("  %-40s %9.3f ms" % (k[:40], v))
        eng.close()
        return

    best = {}
    for cfg in CONFIGS:   # warm-up: records the graphs of every shape with and without adapters
        bind(cfg)
        for R in ROWS:
            one_pass(R)
            generate(R)
    for _ in range(args.rounds):
        for cfg in CONFIGS:
            bind(cfg)
            for R in ROWS:
                for name, fn in (("pass", one_pass), ("gen", generate)):
                    t0 = time.perf_counter()
                    fn(R)
                    dt = time.perf_counter() - t0
                    key = (cfg[0], R, name)
                    best[key] = min(best.get(key, 1e9), dt)
    print("\n%-7s %5s %12s %10s %14s %10s" % ("config", "rows", "pass ms", "vs none", "gen ms/step", "vs none"))
    for R in ROWS:
        for cfg in CONFIGS:
            p, g = best[(cfg[0], R, "pass")] * 1e3, best[(cfg[0], R, "gen")] * 1e3 / args.new
            p0, g0 = best[("none", R, "pass")] * 1e3, best[("none", R, "gen")] * 1e3 / args.new
            print("%-7s %5d %12.3f %9.3fx %14.3f %9.3fx" % (cfg[0], R, p, p / p0, g, g / g0), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
