"""Continuous batching against the two ways the multi-stream API served a request stream before it.

A seeded trace of --requests requests (prompts of 16-512 tokens, max_new of 16-256, arg-max, no penalties, no stop
tokens, so every system generates exactly the same tokens) is replayed in two modes:

  offline    every request arrives at t = 0
  arrivals   a seeded Poisson trace in wall-clock time (--rate requests per second); a driver submits the requests
             that have arrived before each step of work

by three systems, each with at most `rows` requests in flight:

  batcher    Engine.batcher(rows, prefill_tokens): arrived requests are submitted between run(16) calls
  static     (a) up to `rows` arrived requests at a time: forward_streams of their prompts, then one
             generate_streams_ex call until all of them finish
  short      (b) 16-step generate_streams_ex calls over the running requests, new prompts forwarded between calls

Reported per system: generated tokens/s over the whole trace, time to first token p50 / p90 (arrival to the first
moment the host holds a token of the request) and request latency p50 / p90 (arrival to the last token on the host).
Every shape is warmed first; each row is the best round (by tokens/s) of --rounds alternating rounds. The card's name
and power limit are read in the same run, and so is the number of tensor-core pass graphs each system recorded.
usage: python batcher_bench.py [workload=7b] [--rows 32 64 128] [--prefill 128 512] [--rounds 3] [--rate R]
       [--modes offline arrivals]"""
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
GREEDY = dict(temperature=0.0)  # arg-max, no penalties: every system emits the same tokens


def trace(n, seed, rate, mode):
    rng = np.random.default_rng(seed)
    reqs = []
    for i in range(n):
        L = int(rng.integers(16, 513))
        reqs.append(dict(prompt=[int(x) for x in rng.integers(0, V, size=L)], max_new=int(rng.integers(16, 257))))
    gaps = rng.exponential(1.0 / rate, size=n)
    at = np.cumsum(gaps) - gaps[0] if mode == "arrivals" else np.zeros(n)
    for r, t in zip(reqs, at):
        r["at"] = float(t)
    return reqs


def forward_prompts(eng, items, max_gpt):
    """State-only forward of every (slot, tokens) pair, cut into forward_streams calls of at most max_gpt tokens."""
    call, n = [], 0
    for slot, toks in items:
        off = 0
        while off < len(toks):
            take = min(len(toks) - off, max_gpt - n)
            call.append((slot, toks[off:off + take]))
            n += take
            off += take
            if n == max_gpt:
                eng.forward_streams(call, want_logits=False)
                call, n = [], 0
    if call:
        eng.forward_streams(call, want_logits=False)


def run_batcher(eng, reqs, rows, prefill):
    t0 = time.perf_counter()
    first, last = {}, {}
    with eng.batcher(rows, prefill) as bat:
        nxt, ids, free = 0, {}, list(range(rows))
        slot_of = {}
        while len(last) < len(reqs):
            now = time.perf_counter() - t0
            while nxt < len(reqs) and reqs[nxt]["at"] <= now and free:
                s = free.pop()
                rid = bat.submit(s, reqs[nxt]["prompt"], reqs[nxt]["max_new"])
                ids[rid], slot_of[rid] = nxt, s
                nxt += 1
            if not bat.run(16):
                if nxt < len(reqs):
                    time.sleep(max(0.0, reqs[nxt]["at"] - (time.perf_counter() - t0)))
                continue
            now = time.perf_counter() - t0
            for rid, i in list(ids.items()):
                toks, st = bat.read(rid)
                if len(toks) and i not in first:
                    first[i] = now
                if st == "done":
                    last[i] = now
                    bat.release(rid)
                    free.append(slot_of[rid])
                    del ids[rid]
    return first, last, time.perf_counter() - t0


def run_static(eng, reqs, rows, max_gpt):
    t0 = time.perf_counter()
    first, last = {}, {}
    nxt = 0
    while nxt < len(reqs):
        now = time.perf_counter() - t0
        if reqs[nxt]["at"] > now:
            time.sleep(reqs[nxt]["at"] - now)
            now = time.perf_counter() - t0
        batch = []
        while nxt < len(reqs) and reqs[nxt]["at"] <= now and len(batch) < rows:
            batch.append(nxt)
            nxt += 1
        forward_prompts(eng, [(j, reqs[i]["prompt"][:-1]) for j, i in enumerate(batch)], max_gpt)
        mx = max(reqs[i]["max_new"] for i in batch)
        eng.generate_streams([(j, reqs[i]["prompt"][-1]) for j, i in enumerate(batch)], mx,
                             budgets=[reqs[i]["max_new"] for i in batch], sampling=GREEDY)
        now = time.perf_counter() - t0
        for i in batch:
            first[i] = last[i] = now
    return first, last, time.perf_counter() - t0


def run_short(eng, reqs, rows, max_gpt):
    t0 = time.perf_counter()
    first, last = {}, {}
    nxt, active, free = 0, {}, list(range(rows))  # active: request -> [slot, current token, emitted]
    while len(last) < len(reqs):
        now = time.perf_counter() - t0
        new = []
        while nxt < len(reqs) and reqs[nxt]["at"] <= now and free:
            s = free.pop()
            active[nxt] = [s, reqs[nxt]["prompt"][-1], 0]
            new.append((s, reqs[nxt]["prompt"][:-1]))
            nxt += 1
        if new:
            forward_prompts(eng, new, max_gpt)
        if not active:
            time.sleep(max(0.0, reqs[nxt]["at"] - now))
            continue
        order = list(active)
        left = [reqs[i]["max_new"] - active[i][2] for i in order]
        out = eng.generate_streams([(active[i][0], active[i][1]) for i in order], 16, budgets=[min(16, x) for x in left],
                                   sampling=GREEDY)
        now = time.perf_counter() - t0
        for i, toks in zip(order, out):
            first.setdefault(i, now)
            active[i][1], active[i][2] = int(toks[-1]), active[i][2] + len(toks)
            if active[i][2] == reqs[i]["max_new"]:
                last[i] = now
                free.append(active[i][0])
                del active[i]
    return first, last, time.perf_counter() - t0


def stats(reqs, first, last, wall):
    at = np.array([r["at"] for r in reqs])
    ttft = np.array([first[i] for i in range(len(reqs))]) - at
    lat = np.array([last[i] for i in range(len(reqs))]) - at
    toks = sum(r["max_new"] for r in reqs)
    return dict(tps=toks / wall, ttft50=np.percentile(ttft, 50), ttft90=np.percentile(ttft, 90),
                lat50=np.percentile(lat, 50), lat90=np.percentile(lat, 90))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--rows", type=int, nargs="+", default=[32, 64, 128])
    ap.add_argument("--prefill", type=int, nargs="+", default=[128, 512])
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--rate", type=float, default=8.0, help="arrivals per second in the arrivals mode")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--modes", nargs="+", default=["offline", "arrivals"], choices=["offline", "arrivals"])
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    max_gpt = max(128, max(args.rows))
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max_gpt)
    L, E = bench.SHAPES[args.workload]
    print("workload %s (L=%d, E=%d), %d requests, best of %d alternating rounds" % (args.workload, L, E, args.requests,
                                                                                   args.rounds), flush=True)

    def graphs():
        a = np.zeros(1, np.uint64)
        eng.lib.rwkv_b200_debug_read(eng.h, b"graph_records", a.ctypes.data, 8)
        return int(a[0])

    print("\n%-9s %5s %8s %-9s %10s %9s %9s %9s %9s %7s" % ("mode", "rows", "prefill", "system", "tokens/s", "ttft p50",
                                                           "ttft p90", "lat p50", "lat p90", "graphs"))
    for mode in args.modes:
        reqs = trace(args.requests, 5, args.rate, mode)
        for rows in args.rows:
            systems = [("batcher", p) for p in args.prefill] + [("static", None), ("short", None)]
            # warm every shape: one small trace per system
            warm = trace(2 * rows, 6, 1e9, "offline")
            for name, p in systems:
                run_one(eng, name, warm, rows, p, max_gpt)
            best = {}
            for _ in range(args.rounds):
                for name, p in systems:
                    g0 = graphs()
                    s = stats(reqs, *run_one(eng, name, reqs, rows, p, max_gpt))
                    s["graphs"] = graphs() - g0
                    if (name, p) not in best or s["tps"] > best[(name, p)]["tps"]:
                        best[(name, p)] = s
            for name, p in systems:
                s = best[(name, p)]
                print("%-9s %5d %8s %-9s %10.0f %8.2fs %8.2fs %8.2fs %8.2fs %7d" % (
                    mode, rows, p if p else "-", name, s["tps"], s["ttft50"], s["ttft90"], s["lat50"], s["lat90"], s["graphs"]),
                    flush=True)
    eng.close()


def run_one(eng, name, reqs, rows, p, max_gpt):
    if name == "batcher":
        return run_batcher(eng, reqs, rows, p)
    if name == "static":
        return run_static(eng, reqs, rows, max_gpt)
    return run_short(eng, reqs, rows, max_gpt)


if __name__ == "__main__":
    main()
