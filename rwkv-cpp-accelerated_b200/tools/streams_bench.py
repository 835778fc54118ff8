"""Multi-stream serving on one GPU: what a decode step of S conversations costs through forward_streams, and what a
step that also prefills a new conversation's prompt chunk costs against the same work as separate calls.

(a) S streams x 1 token with the device arg-max (next_out), S in 1, 8, 16, 32, 64, 128: step time and aggregate
    tokens/s, beside forward_greedy single-stream tokens/s.
(b) S - 1 decoding streams + one 64-token prompt chunk in one call, against one call for the S - 1 streams and one
    for the chunk.

Host timer around calls that return synchronised; every shape is warmed first (its first call records the CUDA
graph of the pass). The card's name and power limit are read in the same run.
usage: python streams_bench.py [workload=7b] [--steps N]"""
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

DECODE_S = (1, 8, 16, 32, 64, 128)
MIXED_S = (8, 16, 32, 64)
CHUNK = 64


def timed(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    return (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(DECODE_S))
    rng = np.random.default_rng(1)
    L, E = bench.SHAPES[args.workload]
    print("workload %s (L=%d, E=%d), %d timed steps per row" % (args.workload, L, E, args.steps), flush=True)

    tok = [4118]

    def greedy():
        tok[0] = int(eng.forward_greedy(tok[0]))
    single = timed(greedy, args.steps)
    print("\nforward_greedy, one stream: %.3f ms/token, %.1f tokens/s" % (single * 1e3, 1.0 / single), flush=True)

    print("\n(a) decode step, S streams x 1 token, next_out")
    print("%5s %12s %14s %16s" % ("S", "step ms", "tokens/s", "vs single stream"))
    for S in DECODE_S:
        streams = [(s, [int(t)]) for s, t in enumerate(rng.integers(0, 50000, S))]
        dt = timed(lambda: eng.forward_streams(streams, want_logits=False, want_next=True), args.steps)
        print("%5d %12.3f %14.1f %15.2fx" % (S, dt * 1e3, S / dt, S / dt * single), flush=True)

    print("\n(b) mixed step: S-1 decoding streams + one %d-token prompt chunk" % CHUNK)
    print("%5s %12s %16s %9s" % ("S", "one call ms", "separate ms", "ratio"))
    for S in MIXED_S:
        dec = [(s, [int(t)]) for s, t in enumerate(rng.integers(0, 50000, S - 1))]
        chunk = (S - 1, [int(t) for t in rng.integers(0, 50000, CHUNK)])
        mixed = timed(lambda: eng.forward_streams(dec + [chunk], want_logits=False, want_next=True), args.steps)

        def separate():
            eng.forward_streams(dec, want_logits=False, want_next=True)
            eng.forward_streams([chunk], want_logits=False, want_next=True)
        sep = timed(separate, args.steps)
        print("%5d %12.3f %16.3f %8.2fx" % (S, mixed * 1e3, sep * 1e3, sep / mixed), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
