"""Scoring on the device (rwkv_b200_score_streams) against what it replaces.

  call      score_streams with every position scored (each token's target is the next token), top_n = 0 and 20, on
            1 x 128 tokens, 1 x 1024 tokens (one call: eight 128-token passes) and 16 x 64 tokens: ms per call and
            scored tokens/s, best of --rounds alternating rounds
  host      the path a caller had before: forward (GPT mode, one stream per call) with the logits of every token, then
            a numpy float64 log-softmax and the rank of the target, alternating with the device path
  forward   forward_streams state-only on the same tokens: what scoring costs over the forward itself
  kernel    device time of one k_logprob_rows launch at 1, 16 and 128 scored rows, top_n = 0 and 20, from the CUDA
            kernel records of torch.profiler, averaged over --reps calls

The card's name and power limit are read in the same run.
usage: python score_bench.py [workload=7b] [--rounds R] [--reps K]"""
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

V = 50277
SHAPES = ((1, 128), (1, 1024), (16, 64))  # streams x tokens
ROWS = (1, 16, 128)


def kernel_us(fn, name, reps):
    """Mean device time (us) per launch of the kernels whose name contains `name`, over `reps` calls of fn."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    t, c = 0.0, 0
    for ev in prof.events():
        if name in ev.name and ev.device_type.name == "CUDA":
            t += ev.device_time
            c += 1
    return t / c if c else None


def host_score(logits, targets):
    """What the device computes, on the host: float64 log-softmax and the rank of each target (ties: lower index)."""
    l = logits.astype(np.float64)
    m = l.max(axis=1, keepdims=True)
    lse = np.log(np.exp(l - m).sum(axis=1))
    r = np.arange(len(targets))
    ly = l[r, targets]
    lp = (ly - m[:, 0]) - lse
    idx = np.arange(V)
    rank = ((l > ly[:, None]) | ((l == ly[:, None]) & (idx[None, :] < targets[:, None]))).sum(axis=1)
    return lp, rank


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    max_tokens = max(s * n for s, n in SHAPES)
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max_tokens)
    L, E = bench.SHAPES[args.workload]
    rng = np.random.default_rng(1)
    print("workload %s (L=%d, E=%d)" % (args.workload, L, E), flush=True)

    print("\nms per call (scored tokens/s), best of %d alternating rounds; every position scored" % args.rounds)
    print("%10s %20s %20s %20s %20s" % ("shape", "score top_n=0", "score top_n=20", "host path", "forward state-only"))
    for S, n in SHAPES:
        seqs = [[int(x) for x in rng.integers(0, 50000, n + 1)] for _ in range(S)]
        streams = [(s, q[:n]) for s, q in enumerate(seqs)]
        targets = [q[1:] for q in seqs]
        scored = S * n

        def score0():
            eng.score_streams(streams, targets, top_n=0)

        def score20():
            eng.score_streams(streams, targets, top_n=20)

        def host():
            for s, q in enumerate(seqs):  # forward's GPT mode is one stream on slot 0
                lg = eng.forward(q[:n])
                host_score(lg, np.asarray(q[1:], np.int64))

        def fwd():
            eng.forward_streams(streams, want_logits=False)

        fns = {"s0": score0, "s20": score20, "host": host, "fwd": fwd}
        best = dict.fromkeys(fns, 1e9)
        for fn in fns.values():  # warm-up: the graphs of every pass shape, every buffer touched
            fn()
        for _ in range(args.rounds):
            for k, fn in fns.items():
                t0 = time.perf_counter()
                fn()
                best[k] = min(best[k], time.perf_counter() - t0)
        cell = lambda t: "%.2f (%.0f)" % (t * 1e3, scored / t)
        print("%10s %20s %20s %20s %20s" % ("%dx%d" % (S, n), cell(best["s0"]), cell(best["s20"]), cell(best["host"]),
                                             cell(best["fwd"])), flush=True)

    print("\nk_logprob_rows device time per launch (us), one CTA per scored row")
    print("%6s %12s %12s" % ("rows", "top_n=0", "top_n=20"))
    seq = [int(x) for x in rng.integers(0, 50000, 129)]
    for R in ROWS:
        tg = [None] * (128 - R) + seq[129 - R:]
        row = {}
        for top_n in (0, 20):
            fn = lambda: eng.score_streams([(0, seq[:128])], [tg], top_n=top_n)
            fn()
            row[top_n] = kernel_us(fn, "k_logprob_rows", args.reps)
        fmt = lambda x: "%.1f" % x if x is not None else "not measured"
        print("%6d %12s %12s" % (R, fmt(row[0]), fmt(row[20])), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
