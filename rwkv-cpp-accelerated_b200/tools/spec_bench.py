"""Speculative generation with prompt-lookup drafts against one-token-per-step generation, in the same run, alternating.

  spec     generate_speculative: S streams, k drafts, max_new = 64, greedy, with one of three lookup contexts:
             ceiling  the stream's own greedy output (its first token and what follows): nearly every draft is right;
             floor    256 random tokens: lookup rarely finds anything that fits;
             none     self-lookup only (the stream's own emitted tokens)
  ex-tc    generate_streams_ex (arg-max) on the tensor cores (prefill_min = 2; a lone stream gets a pad stream): the
           call whose tokens spec reproduces
  default  generate_streams (arg-max) with the default path: the decode kernel below 8 streams

Every call starts from zeroed first slots, so the ceiling context is exactly the run's own output. Host timer around
calls that return synchronised; every shape is warmed first (its first tensor-core call records the CUDA graph of the
pass); each row reports the best of --rounds alternating rounds, in ms per emitted token, and spec's tokens per step
(emitted tokens / steps). --profile takes, in a run of its own, the kernel time of k_spec_draft and k_spec_accept from
torch.profiler. The card's name and power limit are read in the same run.
usage: python spec_bench.py [workload=7b] [--new N] [--rounds R] [--profile]"""
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
DRAFTS = (2, 4, 8)
CONTEXTS = ("ceiling", "floor", "none")


def kernel_us(fn, names):
    """Mean device time (us) per launch of each kernel whose name contains one of `names`, over one call of fn."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for n in names:
        ts = [ev.device_time for ev in prof.events() if n in ev.name and ev.device_type.name == "CUDA"]
        out[n] = (sum(ts) / len(ts), len(ts)) if ts else (None, 0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--new", type=int, default=64, help="max_new of each stream")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="kernel times of the new kernels instead of the table")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    kmax = max(DRAFTS)
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(STREAMS) * (kmax + 1))
    L, E = bench.SHAPES[args.workload]
    N = args.new
    rng = np.random.default_rng(1)
    print("workload %s (L=%d, E=%d), max_new = %d, greedy, ngram = 3, best of %d alternating rounds"
          % (args.workload, L, E, N, args.rounds), flush=True)
    pad = max(STREAMS) * (kmax + 1) - 1  # never a first slot: first slots are s * (kmax + 1)

    def zero(S):
        for s in range(S):
            eng.slot_zero(s * (kmax + 1))

    def ex_tc(S, first):
        zero(S)
        eng.set_option("prefill_min", 2)
        streams = [(s * (kmax + 1), first[s]) for s in range(S)] + ([(pad, first[0])] if S < 2 else [])
        out = eng.generate_streams(streams, N, sampling=pkg.Sampler(temperature=0.0))
        eng.set_option("prefill_min", 8)
        return out[:S], None

    def default(S, first):
        zero(S)
        return eng.generate_streams([(s * (kmax + 1), first[s]) for s in range(S)], N), None

    def spec(S, first, k, context):
        zero(S)
        res = eng.generate_speculative([([s * (kmax + 1) + i for i in range(k + 1)], first[s]) for s in range(S)], N, k,
                                       context=context)
        return [r["tokens"] for r in res], sum(r["steps"] for r in res)

    if args.profile:
        print("\nkernel time, one call, ceiling context (us per launch, launches)", flush=True)
        names = ("k_spec_draft", "k_spec_accept")
        for S in STREAMS:
            first = [int(t) for t in rng.integers(0, 50000, S)]
            ref, _ = ex_tc(S, first)
            ctx = [[first[s]] + [int(x) for x in ref[s]] for s in range(S)]
            for k in DRAFTS:
                spec(S, first, k, ctx)
                r = kernel_us(lambda: spec(S, first, k, ctx), names)
                print("S = %2d, k = %d: " % (S, k) + ", ".join(
                    "%s %s (%d)" % (n, "%.1f" % r[n][0] if r[n][0] is not None else "-", r[n][1]) for n in names), flush=True)
        eng.close()
        return

    print("\n%4s %3s %8s %12s %12s %12s %12s %11s %10s" % ("S", "k", "context", "spec ms/tok", "tok/step", "ex-tc ms/tok",
                                                           "default", "vs ex-tc", "vs default"), flush=True)
    for S in STREAMS:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        ref, _ = ex_tc(S, first)
        contexts = {"ceiling": [[first[s]] + [int(x) for x in ref[s]] for s in range(S)],
                    "floor": [[int(x) for x in rng.integers(0, 50000, 256)] for _ in range(S)], "none": None}
        fns = {"ex-tc": lambda: ex_tc(S, first), "default": lambda: default(S, first)}
        for k in DRAFTS:
            for c in CONTEXTS:
                fns[(k, c)] = (lambda k=k, c=c: spec(S, first, k, contexts[c]))
        best, tps = {}, {}
        for name, fn in fns.items():  # warm-up: records the graphs of the shapes, grows every buffer; checks the tokens
            toks, steps = fn()
            if name != "default":
                assert all(np.array_equal(a, b) for a, b in zip(toks, ref)), "%s: tokens differ from ex-tc" % (name,)
            n_tok = sum(len(t) for t in toks)
            tps[name] = (n_tok / steps) if steps else None
            best[name] = (1e9, n_tok)
        for _ in range(args.rounds):
            for name, fn in fns.items():
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[name] = (min(best[name][0], dt), best[name][1])
        per_tok = {n: best[n][0] / best[n][1] * 1e3 for n in best}
        for k in DRAFTS:
            for c in CONTEXTS:
                x = per_tok[(k, c)]
                print("%4d %3d %8s %12.3f %12.2f %12.3f %12.3f %10.2fx %9.2fx" % (
                    S, k, c, x, tps[(k, c)], per_tok["ex-tc"], per_tok["default"], per_tok["ex-tc"] / x,
                    per_tok["default"] / x), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
