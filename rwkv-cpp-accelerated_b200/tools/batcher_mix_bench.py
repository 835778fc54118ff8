"""What the per-request features of continuous batching cost: the offline trace of batcher_bench.py replayed through
Engine.batcher with four request mixes.

  plain        every request as in batcher_bench.py (arg-max, no penalties, no stops)
  logprobs     every request also scores its tokens, top_n 5, raw and processed alternating
  constrained  every other request has a token automaton (regex [a-z ,.]+, which never completes) and logit overrides
  all          both: every request scored, every other one constrained with overrides

Reported per (rows, mix): generated tokens/s, the batcher steps run, and the mean time per step. Every shape is warmed
first; each row is the best of --rounds alternating rounds. --kernels also profiles one round of "all" with
torch.profiler and prints the mean device time per launch of the kernels the features add or change. The card's name
and power limit are read in the same run.
usage: python batcher_mix_bench.py [workload=169m] [--rows 32 128] [--prefill 512] [--rounds 3]
       [--mixes plain logprobs constrained all] [--kernels]"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import batcher_bench  # noqa: E402

bench = batcher_bench.bench
MIXES = ("plain", "logprobs", "constrained", "all")
OVERRIDES = {11: 3.0, 187: -99.0, 50: -np.inf}
KERNELS = ("k_gen_logprob", "k_gen_override", "k_gen_mask", "k_gen_feedback", "k_sample_nucleus")


def options(mix, i, cid):
    """The submit keywords of request i under a mix."""
    kw = {}
    if mix in ("logprobs", "all"):
        kw.update(logprobs="raw" if i % 2 == 0 else "processed", top_n=5)
    if mix in ("constrained", "all") and i % 2 == 1:
        kw.update(constraint=cid, overrides=OVERRIDES)
    return kw


def run(eng, reqs, rows, prefill, mix, cid):
    """One replay: (tokens emitted, steps run, wall seconds)."""
    t0 = time.perf_counter()
    steps = toks = 0
    with eng.batcher(rows, prefill) as bat:
        nxt, live, free = 0, {}, list(range(rows))
        while nxt < len(reqs) or live:
            while nxt < len(reqs) and free:
                s = free.pop()
                live[bat.submit(s, reqs[nxt]["prompt"], reqs[nxt]["max_new"], **options(mix, nxt, cid))] = s
                nxt += 1
            steps += bat.run(16)
            for rid, s in list(live.items()):
                t, st = bat.read(rid)
                if st == "done":
                    toks += len(t)
                    bat.release(rid)
                    free.append(s)
                    del live[rid]
    return toks, steps, time.perf_counter() - t0


def profile_kernels(eng, reqs, rows, prefill, cid):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(eng, reqs, rows, prefill, "all", cid)
    agg = {}
    for ev in prof.events():
        name = ev.name
        for k in KERNELS:
            if k in name:
                n, us = agg.get(k, (0, 0.0))
                agg[k] = (n + 1, us + ev.device_time)
    return agg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="169m")
    ap.add_argument("--rows", type=int, nargs="+", default=[32, 128])
    ap.add_argument("--prefill", type=int, default=512)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--mixes", nargs="+", default=list(MIXES), choices=MIXES)
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    max_gpt = max(128, max(args.rows))
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max_gpt)
    L, E = bench.SHAPES[args.workload]
    cid = None
    if any(m in ("constrained", "all") for m in args.mixes) or args.kernels:
        C = pkg.constrain
        cid = eng.add_constraint(C.token_automaton(C.compile_regex(r"[a-z ,.]+"), C.token_bytes(), eos=0))
    reqs = batcher_bench.trace(args.requests, 5, 1.0, "offline")
    print("workload %s (L=%d, E=%d), %d requests, prefill %d, best of %d alternating rounds" % (
        args.workload, L, E, args.requests, args.prefill, args.rounds), flush=True)
    print("\n%5s %-12s %10s %7s %12s" % ("rows", "mix", "tokens/s", "steps", "ms per step"))
    for rows in args.rows:
        warm = batcher_bench.trace(2 * rows, 6, 1.0, "offline")
        for mix in args.mixes:
            run(eng, warm, rows, args.prefill, mix, cid)
        best = {}
        for _ in range(args.rounds):
            for mix in args.mixes:
                toks, steps, wall = run(eng, reqs, rows, args.prefill, mix, cid)
                if mix not in best or toks / wall > best[mix][0] / best[mix][2]:
                    best[mix] = (toks, steps, wall)
        for mix in args.mixes:
            toks, steps, wall = best[mix]
            print("%5d %-12s %10.0f %7d %12.3f" % (rows, mix, toks / wall, steps, 1e3 * wall / steps), flush=True)
        if args.kernels:
            agg = profile_kernels(eng, reqs, rows, args.prefill, cid)
            for k in KERNELS:
                if k in agg:
                    n, us = agg[k]
                    print("      rows %d, mix all: %-18s %7d launches %9.2f us per launch" % (rows, k, n, us / n), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
