"""Classifier-free guidance: what the guidance rows cost per emitted token.

For S = 1, 8 and 32 streams, ms per emitted token of generate_streams(sampling=...) (rwkv_b200_generate_streams_ex)
against the same call with every stream guided at gamma 1.5 (rwkv_b200_generate_streams_guided, S + S rows per step),
both nucleus-sampled at temperature 1 with the same uniforms and max_new tokens per stream with no stop, so every
stream emits max_new tokens. Each shape runs on the default path (the tensor cores from prefill_min rows, else the
decode kernel) and on the tensor cores with prefill_min = 2. The two calls alternate in each of --rounds rounds after a
warm-up of each, host timer around calls that return synchronised; the best round is reported. The card's name and
power limit are read in the same run.
usage: python guidance_bench.py [workload ...] [--max-new N] [--rounds R]   (default workloads: 169m 7b)"""
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

STREAMS = (1, 8, 32)
SCALE = 1.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["169m", "7b"])
    ap.add_argument("--max-new", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    N = args.max_new
    print("| workload | path | S | guided call rows | unguided ms/step | guided ms/step | guided / unguided |")
    print("|---|---|---|---|---|---|---|")
    for wl in args.workloads:
        eng = pkg.Engine(bench.model_path(wl, pkg), max_gpt=2 * max(STREAMS))
        for path in ("default", "prefill_min 2"):
            if path != "default":
                eng.set_option("prefill_min", 2)
            for S in STREAMS:
                rng = np.random.default_rng(S)
                first = [int(x) for x in rng.integers(0, 50000, S)]
                streams = [(s, first[s]) for s in range(S)]
                guidance = [(S + s, int(rng.integers(0, 50000)), SCALE) for s in range(S)]
                samp = [pkg.Sampler(1.0, 0.9)] * S
                u = rng.random((N, S))
                calls = {
                    "plain": lambda: eng.generate_streams(streams, N, sampling=samp, u=u),
                    "guided": lambda: eng.generate_streams(streams, N, sampling=samp, u=u, guidance=guidance),
                }
                best = {k: float("inf") for k in calls}
                for k, fn in calls.items():  # warm-up: recorded graphs, buffers
                    fn()
                for _ in range(args.rounds):
                    for k, fn in calls.items():
                        t = time.perf_counter()
                        out = fn()
                        dt = time.perf_counter() - t
                        assert sum(len(x) for x in out) == S * N
                        best[k] = min(best[k], dt)
                ms = {k: 1e3 * v / N for k, v in best.items()}  # per step: one token of every stream
                print("| %s | %s | %d | %d | %.3f | %.3f | %.2f |" % (wl, path, S, 2 * S, ms["plain"], ms["guided"],
                                                                      ms["guided"] / ms["plain"]), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
