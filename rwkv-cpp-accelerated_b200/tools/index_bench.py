"""State indexes (rwkv_b200_index_*, Engine.embed, StateIndex.search) against the examples/vectordb way.

  embed     Engine.embed of --docs documents of --doc-len tokens (ragged forward_streams passes of up to --max-gpt
            tokens, state only, --slots slots) in docs/s and tokens/s; against it, the example's way on the first
            --host-docs documents: one document at a time on slot 0 (forward in GPT mode), then slot_download
  search    per index size (entries of D = n_layers * n_embed doubles, filled from embedded slots): the call time of one
            search of Q = 8 query slots (k = 10, l2), the device time of its scan kernel and of all its kernels from the
            CUDA kernel records of torch.profiler (--reps calls), the scan's achieved bytes/s (live rows x D x 8 over
            the scan time) and its share of the data sheet's 3.35 TB/s; against it, for indexes up to 1 GiB, the host way:
            slot_download of each query, then numpy l1 and l2 over the index's vectors held on the host, and a top k

The card's name, power limit and maximum SM clock are read in the same run.
usage: python index_bench.py [workload=7b] [--docs N] [--doc-len T] [--sizes a,b,..] [--reps K]"""
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

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
Q, K = 8, 10


def kernel_us(fn, names, reps):
    """Mean device time (us) per call of fn of the kernels whose name contains one of `names`, over `reps` calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    t = 0.0
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and any(n in ev.name for n in names):
            t += ev.device_time
    return t / reps if t else None


def best_of(fn, reps):
    best = 1e9
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--docs", type=int, default=1024)
    ap.add_argument("--doc-len", type=int, default=64)
    ap.add_argument("--host-docs", type=int, default=64)
    ap.add_argument("--max-gpt", type=int, default=1024)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--sizes", default="8,64,512,2048,8192")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    L, E = bench.SHAPES[args.workload]
    D = L * E
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=args.max_gpt)
    print("workload %s (L=%d, E=%d): D = %d doubles, %.2f MiB per entry" % (args.workload, L, E, D, D * 8 / 2 ** 20), flush=True)
    rng = np.random.default_rng(1)
    docs = [[int(x) for x in rng.integers(0, 50000, args.doc_len)] for _ in range(args.docs)]
    slots = list(range(args.slots))

    # -- embedding --------------------------------------------------------------------------------------------------
    with eng.create_index(args.docs + 64, None) as idx:
        eng.embed(docs[:64], slots, idx)  # warm-up: every pass shape of the timed run
        t0 = time.perf_counter()
        eng.embed(docs, slots, idx)
        t_embed = time.perf_counter() - t0

    def host_way():
        for d in docs[:args.host_docs]:
            eng.slot_zero(0)
            eng.forward(d, mode=pkg.engine.MODE_GPT, want_logits=False)
            eng.slot_download(0)

    eng.forward(docs[0], mode=pkg.engine.MODE_GPT, want_logits=False)
    t0 = time.perf_counter()
    host_way()
    t_host = time.perf_counter() - t0
    n_tok = args.docs * args.doc_len
    print("\nembedding %d documents of %d tokens" % (args.docs, args.doc_len))
    print("  Engine.embed (max_gpt %d, %d slots): %.3f s, %.1f docs/s, %.0f tokens/s" %
          (args.max_gpt, args.slots, t_embed, args.docs / t_embed, n_tok / t_embed))
    print("  one document at a time on slot 0 + slot_download (%d documents): %.1f docs/s, %.0f tokens/s -> %.1fx" %
          (args.host_docs, args.host_docs / t_host, args.host_docs * args.doc_len / t_host,
           (args.docs / t_embed) / (args.host_docs / t_host)), flush=True)

    # -- search -----------------------------------------------------------------------------------------------------
    # states to fill the indexes from: one document per slot
    src = list(range(min(args.max_gpt, 64)))
    eng.forward_streams([(s, docs[s % len(docs)][:8]) for s in src], want_logits=False)
    queries = list(range(Q))
    print("\nsearch of %d query slots, k = %d, l2; call = best of %d; device times from torch.profiler over %d calls" %
          (Q, K, args.reps, args.reps))
    print("%8s %10s %10s %10s %10s %12s %8s %14s" % ("entries", "index MiB", "call ms", "scan us", "all us", "scan GB/s",
                                                    "of peak", "host ms"))
    for n in [int(x) for x in args.sizes.split(",")]:
        try:
            idx = eng.create_index(n, None)
        except pkg.EngineError as e:
            print("%8d  not measured: %s" % (n, e), flush=True)
            continue
        with idx:
            for i in range(0, n, len(src)):
                idx.add(src[:min(len(src), n - i)])
            fn = lambda: idx.search(queries, K, "l2")
            fn()
            t_call = best_of(fn, args.reps)
            scan = kernel_us(fn, ("k_index_scan",), args.reps)
            total = kernel_us(fn, ("k_index_",), args.reps)
            gbs = n * D * 8 / (scan * 1e-6) if scan else None
            host = "not measured"
            if n * D * 8 <= 2 ** 30:
                vecs = idx.vectors(np.arange(n))

                def host_search():
                    for q in queries:
                        a = eng.slot_download(q)["dd"]
                        d = vecs - a
                        l1 = np.abs(d).sum(axis=1) / E
                        l2 = np.sqrt((d * d).sum(axis=1) / E)
                        np.lexsort((np.arange(n), l2))[:K], l1
                host = "%.2f" % (best_of(host_search, max(2, args.reps // 3)) * 1e3)
                del vecs
            fmt = lambda x, f: f % x if x is not None else "not measured"
            print("%8d %10.0f %10.3f %10s %10s %12s %8s %14s" % (n, n * D * 8 / 2 ** 20, t_call * 1e3, fmt(scan, "%.1f"),
                                                                fmt(total, "%.1f"), fmt(gbs and gbs / 1e9, "%.0f"),
                                                                fmt(gbs and gbs / HBM_PEAK * 100, "%.0f%%"), host), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
