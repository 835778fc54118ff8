"""Prefix state cache: what restoring a cached prefix saves, and what the cache itself costs.

Tables, each alternating the configurations in one run, best of --rounds rounds, host timer around calls that return
synchronised, every shape warmed first:
  serve     the batcher with N rows and N requests sharing a system prompt of P = 512 and 2,048 tokens, each with a
            32-token unique suffix and max_new 64. "plain": every request on a zeroed slot; "cache": every request
            submitted with a cache opened for the round, into which one state-only prefix_forward puts the system prompt
            first (a server's cache already holds it). Wall time to finish, prompt tokens run and hit tokens.
  eval      Q questions behind one 1,024-token few-shot context, each scoring a 4-token answer: prefix_forward of context
            + question followed by score_streams of the answer, against score_streams of the whole text.
  restore   k_prefix_copy in a state-only prefix_forward of n fully cached streams (one copy kernel, no pass): the
            kernel's time from torch.profiler in a run of its own, as GB/s of the bytes it must move (4 arrays read, 5
            written, per stream) against the data sheet's 3.35 TB/s, and the whole call's time.
  snapshot  prefix_forward of one 128-token stream with its arg-max and 0 snapshots (block 2048, its only position
            already cached), 2 (block 64) and 8 (block 16) snapshots (the cache cleared before each call).
The card's name and power limit are read in the same run.
usage: python prefix_bench.py [workload=7b] [--requests N] [--questions Q] [--rounds R]"""
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

HBM = 3.35e12
SUFFIX, MAX_NEW, CONTEXT, QUESTION, ANSWER = 32, 64, 1024, 24, 4


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--questions", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    L, E = bench.SHAPES[args.workload]
    N, Q = args.requests, args.questions
    max_gpt = max(2048 + SUFFIX, CONTEXT + QUESTION + ANSWER, N, Q, 128)
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max_gpt)
    eng.set_option("prefill_min", 2)  # short score_streams calls on the tensor cores too, so both modes score the same bits
    LE = L * E
    print("workload %s (L=%d, E=%d): one cached state is %.2f MiB" % (args.workload, L, E, 4 * LE * 8 / 2 ** 20), flush=True)
    rng = np.random.default_rng(3)
    rand = lambda n: [int(x) for x in rng.integers(0, 50000, n)]

    # ---- serve ----
    print("\nserve: batcher, %d requests (rows %d), shared system prompt + %d unique tokens, max_new %d"
          % (N, N, SUFFIX, MAX_NEW))
    print("%6s %6s %10s %12s %12s" % ("P", "mode", "seconds", "prefilled", "hit tokens"))
    for P in (512, 2048):
        system = rand(P)
        prompts = [system + rand(SUFFIX) for _ in range(N)]

        def serve(use_cache):
            cache = eng.prefix_cache(4 * N, block=64) if use_cache else None
            if cache:  # a server's cache already holds its system prompt: one state-only call puts it there
                cache.forward([(0, system)], want_logits=False)
            else:
                for s in range(N):
                    eng.slot_zero(s)
            with eng.batcher(N, 2048) as bat:
                ids = [bat.submit(s, p, MAX_NEW, prefix_cache=cache) for s, p in enumerate(prompts)]
                while bat.run(256):
                    pass
                toks = [bat.result(i)["tokens"].tolist() for i in ids]
            if cache:
                st = cache.stats()
                cache.close()
                return st["prefilled_tokens"], st["hit_tokens"], toks
            return sum(len(p) - 1 for p in prompts), 0, toks

        serve(False)
        serve(True)
        best = {}
        for _ in range(args.rounds):
            for mode in ("plain", "cache"):
                dt, (pre, hit, toks) = timed(lambda: serve(mode == "cache"))
                best.setdefault(mode, [dt, pre, hit, toks])
                best[mode][0] = min(best[mode][0], dt)
        assert best["plain"][3] == best["cache"][3], "the cache changed the generated tokens"
        for mode in ("plain", "cache"):
            dt, pre, hit, _ = best[mode]
            print("%6d %6s %10.3f %12d %12d" % (P, mode, dt, pre, hit), flush=True)

    # ---- eval ----
    print("\neval: %d questions of %d tokens behind a %d-token context, %d-token answers" % (Q, QUESTION, CONTEXT, ANSWER))
    ctx = rand(CONTEXT)
    qs = [(rand(QUESTION), rand(ANSWER)) for _ in range(Q)]

    def evaluate(use_cache):
        scores = []
        cache = eng.prefix_cache(8, block=CONTEXT) if use_cache else None
        for q, a in qs:
            if cache:
                cache.forward([(0, ctx + q[:-1])], want_logits=False)
                r = eng.score_streams([(0, q[-1:] + a[:-1])], targets=[a])
            else:
                eng.slot_zero(0)
                text = ctx + q + a[:-1]
                r = eng.score_streams([(0, text)], targets=[[None] * (len(ctx) + len(q) - 1) + a])
            scores.append(r[0]["logprobs"][-ANSWER:].tolist())
        if cache:
            cache.close()
        return scores

    evaluate(False)
    evaluate(True)
    best = {}
    for _ in range(args.rounds):
        for mode in ("plain", "cache"):
            dt, sc = timed(lambda: evaluate(mode == "cache"))
            best.setdefault(mode, [dt, sc])
            best[mode][0] = min(best[mode][0], dt)
    assert best["plain"][1] == best["cache"][1], "the cache changed the scores"
    for mode in ("plain", "cache"):
        print("%6s %10.3f s  %8.2f ms per question" % (mode, best[mode][0], 1e3 * best[mode][0] / Q), flush=True)

    # ---- restore ----
    print("\nrestore: k_prefix_copy of n fully cached streams, kernel time from torch.profiler (CUDA activity)")
    print("%6s %10s %10s %10s %12s" % ("n", "kernel ms", "GB/s", "of 3.35TB/s", "call ms"))
    from torch.profiler import ProfilerActivity, profile
    with eng.prefix_cache(128, block=2048) as cache:
        keys = [rand(8) for _ in range(128)]
        cache.forward([(s, k) for s, k in enumerate(keys)], want_logits=False)
        for n in (1, 8, 32, 128):
            streams = [(s, keys[s]) for s in range(n)]
            cache.forward(streams, want_logits=False)
            reps = max(4, 256 // n)
            dt, _ = timed(lambda: [cache.forward(streams, want_logits=False) for _ in range(reps)])
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    cache.forward(streams, want_logits=False)
            ev = [e for e in prof.key_averages() if "k_prefix_copy" in e.key]
            assert ev, "torch.profiler saw no k_prefix_copy"
            us = getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total
            t = us * 1e-6 / ev[0].count
            gbs = n * 9 * LE * 8 / t
            print("%6d %10.3f %10.1f %9.1f%% %12.3f" % (n, 1e3 * t, gbs / 1e9, 100 * gbs / HBM, 1e3 * dt / reps), flush=True)

    # ---- snapshot ----
    print("\nsnapshot: prefix_forward of one 128-token stream with its arg-max, nothing restored")
    toks = rand(128)
    configs = (("0", 2048), ("2", 64), ("8", 16))
    caches = {name: eng.prefix_cache(16, block=b) for name, b in configs}
    caches["0"].forward([(0, toks)], want_logits=False)  # its one snapshot position (128) exists from now on

    def one(name):
        if name != "0":
            caches[name].clear()
        _, _, cached = caches[name].forward([(0, toks)], want_logits=False, want_next=True)
        assert cached[0] == 0

    for name, _ in configs:
        one(name)
    best = {}
    for _ in range(args.rounds * 5):
        for name, _ in configs:
            dt, _ = timed(lambda: [one(name) for _ in range(8)])
            best[name] = min(best.get(name, 1e9), dt / 8)
    print("%10s %10s" % ("snapshots", "ms"))
    for name, _ in configs:
        print("%10s %10.3f" % (name, 1e3 * best[name]), flush=True)
    before = {name: caches[name].stats()["snapshots"] for name, _ in configs}
    one("0")
    one("8")
    assert caches["0"].stats()["snapshots"] == before["0"] and caches["8"].stats()["snapshots"] == before["8"] + 8
    for c in caches.values():
        c.close()


if __name__ == "__main__":
    main()
