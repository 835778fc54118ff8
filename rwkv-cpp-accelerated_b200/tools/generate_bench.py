"""Device-resident generation against the host loop it replaces: 64 new tokens per stream, both in the same run,
alternating.

  greedy   S = 1          loop: forward_greedy per token
           S = 8 .. 128   loop: forward_streams(want_next) per step
  typical  S = 1          loop: forward(token) + sample_typical per token
           S = 16         loop: forward_streams(want_next) + sample_typical_streams per step
  generate                one generate_streams call for the 64 tokens of every stream

Host timer around calls that return synchronised. Every shape is warmed first (its first tensor-core call records
the CUDA graph of the pass); each row reports the best of --rounds alternating rounds. The card's name and power
limit are read in the same run.
usage: python generate_bench.py [workload=7b] [--new N] [--rounds R]"""
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

GREEDY_S = (1, 8, 16, 64, 128)
TYPICAL_S = (1, 16)
TEMP = 0.9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--new", type=int, default=64, help="tokens generated per stream")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(GREEDY_S))
    L, E = bench.SHAPES[args.workload]
    N = args.new
    rng = np.random.default_rng(1)
    print("workload %s (L=%d, E=%d), %d new tokens per stream, best of %d alternating rounds"
          % (args.workload, L, E, N, args.rounds), flush=True)

    def host_loop(S, first, u):
        cur = list(first)
        if S == 1 and u is None:
            for _ in range(N):
                cur[0] = int(eng.forward_greedy(cur[0]))
        elif S == 1:
            for k in range(N):
                eng.forward([cur[0]], want_logits=False)
                cur[0] = eng.sample_typical(TEMP, float(u[k][0]))[0]
        else:
            for k in range(N):
                _, nxt = eng.forward_streams([(s, [t]) for s, t in enumerate(cur)], want_logits=False, want_next=True)
                cur = [int(x) for x in nxt] if u is None else [int(x) for x in eng.sample_typical_streams(TEMP, u[k])[0]]

    def generate(S, first, u):
        out = eng.generate_streams([(s, t) for s, t in enumerate(first)], N, temp=TEMP, u=u)
        assert all(len(o) == N for o in out)

    rows = [("greedy", S) for S in GREEDY_S] + [("typical", S) for S in TYPICAL_S]
    print("\n%-8s %5s %14s %14s %16s %16s %9s" % ("pick", "S", "loop ms/step", "gen ms/step", "loop tokens/s", "gen tokens/s",
                                                 "speed-up"))
    for pick, S in rows:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        u = rng.random((N, S)) if pick == "typical" else None
        best = {"loop": 1e9, "gen": 1e9}
        fns = {"loop": host_loop, "gen": generate}
        for name in fns:  # warm-up: records the graphs of the shape, touches every buffer
            fns[name](S, first, u)
        for _ in range(args.rounds):
            for name in ("loop", "gen"):
                t0 = time.perf_counter()
                fns[name](S, first, u)
                best[name] = min(best[name], time.perf_counter() - t0)
        lp, gn = best["loop"] / N, best["gen"] / N
        print("%-8s %5d %14.3f %14.3f %16.1f %16.1f %8.3fx" % (pick, S, lp * 1e3, gn * 1e3, S / lp, S / gn, lp / gn), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
