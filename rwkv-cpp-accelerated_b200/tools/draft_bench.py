"""Speculative generation with a draft model against prompt lookup and one-token-per-step generation, in the same run.

  drafted  generate_speculative(drafter=...): a synthetic 7B-shape target (32 x 4096) with a synthetic 169M-shape
           drafter (12 x 768), S streams, k drafts, greedy, max_new = --new
  lookup   generate_speculative with prompt-lookup drafts (no context) at the same S and k
  ex-tc    generate_streams_ex (arg-max) on the tensor cores (prefill_min = 2; a lone stream gets a pad stream)

Synthetic weights make an unrelated drafter's drafts almost never right, so the measured tokens per step are near 1.
Each row reports ms per step of each call (host timer around calls that return synchronised, best of --rounds
alternating rounds, every shape warmed first), the drafted call's tokens per step, and two derived numbers, labelled so:
the draft work's share of a drafted step (drafted minus lookup step time, over the drafted step time; prompt lookup's
own draft kernel is a few microseconds) and the break-even per-token acceptance a at which the drafted call's expected
tokens per step, (1 - a^(k+1)) / (1 - a), pay for its step time against ex-tc. The card's name and power limit are
read in the same run.
usage: python draft_bench.py [--new N] [--rounds R]"""
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

STREAMS = (1, 8, 16, 32)
DRAFTS = (2, 4)


def break_even(ratio, k):
    """The acceptance a in [0, 1) with (1 - a^(k+1)) / (1 - a) = ratio (bisection), or None when ratio > k + 1."""
    if ratio > k + 1:
        return None
    lo, hi = 0.0, 1.0
    for _ in range(60):
        a = (lo + hi) / 2
        if sum(a ** i for i in range(k + 1)) < ratio:
            lo = a
        else:
            hi = a
    return lo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=32, help="max_new of each stream")
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    kmax, smax, N = max(DRAFTS), max(STREAMS), args.new
    tgt = pkg.Engine(bench.model_path("7b", pkg), max_gpt=smax * (kmax + 1))
    drf = pkg.Engine(bench.model_path("169m", pkg), max_gpt=2 * smax)
    pad = smax * (kmax + 1) - 1  # never a first slot: first slots are s * (kmax + 1)
    greedy = pkg.Sampler(temperature=0.0)
    print("target 7b (32 x 4096), drafter 169m (12 x 768), max_new = %d, greedy, best of %d alternating rounds"
          % (N, args.rounds), flush=True)

    def zero(S):
        for s in range(S):
            tgt.slot_zero(s * (kmax + 1))
            drf.slot_zero(2 * s)

    def spec_streams(S, k, first):
        return [([s * (kmax + 1) + i for i in range(k + 1)], first[s]) for s in range(S)]

    def drafted(S, k, first):
        zero(S)
        return tgt.generate_speculative(spec_streams(S, k, first), N, k, sampling=greedy,
                                        drafter=(drf, [(2 * s, 2 * s + 1) for s in range(S)]))

    def lookup(S, k, first):
        zero(S)
        return tgt.generate_speculative(spec_streams(S, k, first), N, k, sampling=greedy)

    def ex_tc(S, k, first):
        zero(S)
        tgt.set_option("prefill_min", 2)
        streams = [(s * (kmax + 1), first[s]) for s in range(S)] + ([(pad, first[0])] if S < 2 else [])
        out = tgt.generate_streams(streams, N, sampling=greedy)
        tgt.set_option("prefill_min", 8)
        return [{"tokens": t, "steps": len(t)} for t in out[:S]]

    calls = {"drafted": drafted, "lookup": lookup, "ex-tc": ex_tc}
    rng = np.random.default_rng(1)
    print("%3s %2s | %10s %10s %10s | %9s | %14s %20s" % ("S", "k", "drafted", "lookup", "ex-tc", "tok/step",
                                                         "draft share*", "break-even accept.*"))
    for S in STREAMS:
        for k in DRAFTS:
            first = [int(x) for x in rng.integers(0, 50277, size=S)]
            best, res = {}, {}
            for name, fn in calls.items():  # warm every shape (the first tensor-core call records its graphs)
                res[name] = fn(S, k, first)
            ref = [[int(x) for x in r["tokens"]] for r in res["ex-tc"]]
            for name in ("drafted", "lookup"):
                assert [[int(x) for x in r["tokens"]] for r in res[name]] == ref, name + ": tokens differ from ex-tc"
            for _ in range(args.rounds):
                for name, fn in calls.items():
                    t0 = time.perf_counter()
                    out = fn(S, k, first)
                    dt = time.perf_counter() - t0
                    steps = max(r["steps"] for r in out)
                    best[name] = min(best.get(name, 1e9), dt * 1e3 / steps)
                    res[name] = out
            tps = sum(len(r["tokens"]) for r in res["drafted"]) / sum(r["steps"] for r in res["drafted"])
            share = (best["drafted"] - best["lookup"]) / best["drafted"]
            be = break_even(best["drafted"] / best["ex-tc"], k)
            print("%3d %2d | %7.2f ms %7.2f ms %7.2f ms | %9.3f | %13.0f%% %20s"
                  % (S, k, best["drafted"], best["lookup"], best["ex-tc"], tps, 100 * share,
                     "%.2f" % be if be is not None else "never"), flush=True)
    print("* derived from the measured step times, not measured directly")
    tgt.close()
    drf.close()


if __name__ == "__main__":
    main()
