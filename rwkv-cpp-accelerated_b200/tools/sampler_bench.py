"""The per-stream sampler (rwkv_b200_sample_streams, rwkv_b200_generate_streams_ex) against what it replaces.

  kernel    S = 1, 16, 128 rows of the last forward_streams: device time of one k_sample_nucleus launch
            (T = 1, top_p = 0.85, and T = 1, top_p = 0.85, top_k = 40) next to k_sample_typical and k_argmax_rows,
            from the CUDA kernel records of torch.profiler, averaged over --reps launches
  generate  64 new tokens per stream: generate_streams_ex (T = 1, top_p = 0.85, presence = frequency = 0.2,
            decay = 0.996) against generate_streams with the typical sampler, best of --rounds alternating rounds
  host      the loop a caller needs for the same penalised top-p sampling without generate_streams_ex:
            forward_streams with logits, numpy penalties and top-p (a sort per row), the pick fed back;
            --loop-steps steps, best of --rounds

The card's name and power limit are read in the same run.
usage: python sampler_bench.py [workload=7b] [--new N] [--rounds R] [--reps K] [--loop-steps N]"""
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

STREAMS = (1, 16, 128)
V = 50277
TOP_P, PEN, DECAY = 0.85, 0.2, 0.996


def kernel_us(fn, names, reps):
    """Mean device time (us) per launch of each kernel whose name contains one of `names`, over `reps` calls of fn."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        for n in names:
            if n in ev.name and ev.device_type.name == "CUDA":
                t, c = out.get(n, (0.0, 0))
                out[n] = (t + ev.device_time, c + 1)
    return {n: (t / c if c else None) for n, (t, c) in out.items()}


def host_pick(logits, cnt, seen, u):
    """Penalties and top-p on the host, then the draw: what generate_streams_ex does on the device."""
    S = logits.shape[0]
    l = logits.copy()
    l[seen] -= np.float32(PEN) + np.float32(PEN) * cnt[seen]
    l64 = l.astype(np.float64)
    p = np.exp(l64 - l64.max(axis=1, keepdims=True))
    order = np.argsort(-l64, axis=1, kind="stable")
    ps = np.take_along_axis(p, order, axis=1)
    cs = np.cumsum(ps, axis=1)
    n_keep = (cs < TOP_P * cs[:, -1:]).sum(axis=1) + 1
    picks = np.empty(S, np.int64)
    for s in range(S):
        k = n_keep[s]
        c = np.cumsum(ps[s, :k]) / cs[s, k - 1]
        picks[s] = order[s, min(int(np.searchsorted(c, u[s])), k - 1)]
    cnt *= np.float32(DECAY)
    cnt[np.arange(S), picks] += np.float32(1.0)
    seen[np.arange(S), picks] = True
    return picks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--new", type=int, default=64, help="tokens generated per stream")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--loop-steps", type=int, default=16)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    Sm = pkg.Sampler
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(STREAMS))
    L, E = bench.SHAPES[args.workload]
    N = args.new
    rng = np.random.default_rng(1)
    print("workload %s (L=%d, E=%d)" % (args.workload, L, E), flush=True)

    print("\nkernel time per launch (us, device), one CTA per row")
    print("%5s %16s %22s %16s %14s" % ("S", "nucleus top-p", "nucleus top-p+top-k", "typical", "arg-max"))
    for S in STREAMS:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        u = rng.random(S)
        eng.forward_streams([(s, [t]) for s, t in enumerate(first)], want_logits=False, want_next=True)
        row = {}
        for key, fn in (("p", lambda: eng.sample_streams(Sm(1.0, TOP_P), u)),
                        ("pk", lambda: eng.sample_streams(Sm(1.0, TOP_P, 40), u)),
                        ("typ", lambda: eng.sample_typical_streams(1.0, u))):
            fn()
            row[key] = kernel_us(fn, ["k_sample_nucleus", "k_sample_typical"], args.reps)
        am = kernel_us(lambda: eng.forward_streams([(s, [t]) for s, t in enumerate(first)], want_logits=False, want_next=True),
                       ["k_argmax_rows"], 3)
        fmt = lambda x: "%.1f" % x if x is not None else "not measured"
        print("%5d %16s %22s %16s %14s" % (S, fmt(row["p"].get("k_sample_nucleus")), fmt(row["pk"].get("k_sample_nucleus")),
                                           fmt(row["typ"].get("k_sample_typical")), fmt(am.get("k_argmax_rows"))), flush=True)

    sampler = Sm(1.0, TOP_P, 0, PEN, PEN, DECAY)
    print("\n%d new tokens per stream; ms per step (tokens/s), best of %d alternating rounds; host loop over %d steps"
          % (N, args.rounds, args.loop_steps))
    print("%5s %22s %22s %22s" % ("S", "generate_streams_ex", "generate_streams typ.", "host loop"))
    for S in STREAMS:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        streams = [(s, t) for s, t in enumerate(first)]
        u = rng.random((N, S))

        def ex():
            assert all(len(o) == N for o in eng.generate_streams(streams, N, u=u, sampling=sampler))

        def typ():
            assert all(len(o) == N for o in eng.generate_streams(streams, N, temp=1.0, u=u))

        def loop():
            cur = list(first)
            cnt = np.zeros((S, V), np.float32)
            seen = np.zeros((S, V), bool)
            for k in range(args.loop_steps):
                logits, _ = eng.forward_streams([(s, [t]) for s, t in enumerate(cur)])
                cur = [int(x) for x in host_pick(logits, cnt, seen, u[k])]

        best = {"ex": 1e9, "typ": 1e9, "loop": 1e9}
        fns = {"ex": ex, "typ": typ, "loop": loop}
        steps = {"ex": N, "typ": N, "loop": args.loop_steps}
        for name in fns:  # warm-up: graphs of the shape, every buffer touched
            fns[name]()
        for _ in range(args.rounds):
            for name in fns:
                t0 = time.perf_counter()
                fns[name]()
                best[name] = min(best[name], (time.perf_counter() - t0) / steps[name])
        cell = lambda t: "%.3f (%.0f)" % (t * 1e3, S / t)
        print("%5d %22s %22s %22s" % (S, cell(best["ex"]), cell(best["typ"]), cell(best["loop"])), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
