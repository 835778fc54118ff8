"""The cost of stop strings on the device: steps per second of generate_streams_ex against generate_streams_stop with
stop sets that never match, so that every emitted token's bytes are walked through the automaton every step.

  S = 1, 16, 64 streams, --new tokens each, arg-max; best of --rounds alternating rounds. Each stream of the stop call
  has a set of --strings strings of 8 bytes (bytes 0x01..0x08, which no token of the vocabulary emits in that order).

The card's name and power limit are read in the same run.
usage: python stop_bench.py [workload=7b] [--new N] [--rounds R] [--strings K]"""
import argparse
import importlib
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

import numpy as np  # noqa: E402

STREAMS = (1, 16, 64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--new", type=int, default=64, help="tokens generated per stream")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--strings", type=int, default=4, help="strings per stop set")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(STREAMS))
    L, E = bench.SHAPES[args.workload]
    print("workload %s (L=%d, E=%d), %d new tokens per stream, arg-max" % (args.workload, L, E, args.new), flush=True)
    never = [bytes([1 + (i + j) % 8 for j in range(8)]) for i in range(args.strings)]
    sid = eng.add_stop_set(never)
    rng = np.random.default_rng(1)
    print("%5s %14s %14s %10s" % ("S", "ex steps/s", "stop steps/s", "overhead"))
    for S in STREAMS:
        streams = [(s, int(t)) for s, t in enumerate(rng.integers(0, 50000, S))]

        def ex():
            out = eng.generate_streams(streams, args.new, sampling=pkg.Sampler(temperature=0.0))
            assert all(len(o) == args.new for o in out)

        def stop():
            out = eng.generate_streams(streams, args.new, sampling=pkg.Sampler(temperature=0.0), stop_strings=sid)
            assert all(len(o["tokens"]) == args.new and o["stop_hit"] is None for o in out)

        fns = {"ex": ex, "stop": stop}
        best = {n: 1e9 for n in fns}
        for f in fns.values():  # warm-up: every buffer grown
            f()
        for _ in range(args.rounds):
            for n, f in fns.items():
                t0 = time.perf_counter()
                f()
                best[n] = min(best[n], time.perf_counter() - t0)
        rate = {n: args.new / best[n] for n in fns}
        print("%5d %14.1f %14.1f %9.2f%%" % (S, rate["ex"], rate["stop"], 100.0 * (best["stop"] / best["ex"] - 1.0)),
              flush=True)
    eng.close()


if __name__ == "__main__":
    main()
