"""Log-probabilities of generated tokens on the device (rwkv_b200_generate_streams_logprobs) against generation without
them and against the host loop it replaces.

  generate  --new tokens per stream at S = 1, 16, 128; ms per step, best of --rounds alternating rounds, of
            generate_streams_ex (T = 1, top_p = 0.85) without log-probabilities, then with them in raw mode at
            top_n = 0 and 20 and in processed mode at top_n = 0; and the same sampler with presence = frequency = 0.2,
            decay = 0.996, without log-probabilities and in raw mode (which copies the step's rows before the penalties)
  kernel    device time of one k_gen_logprob launch at top_n = 0 and 20, from the CUDA kernel records of
            torch.profiler over one call of 16 steps
  host      what a caller does without the entry point: forward_streams with logits, numpy top-p and the pick, a
            float64 log-softmax for the picked token's log-probability and its top 20, the pick fed back;
            --loop-steps steps, best of --rounds

The card's name and power limit are read in the same run.
usage: python gen_logprobs_bench.py [workload=7b] [--new N] [--rounds R] [--loop-steps N]"""
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


def kernel_us(fn, name):
    """Mean device time (us) per launch of the kernels whose name contains `name`, over one call of fn."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ts = [ev.device_time for ev in prof.events() if name in ev.name and ev.device_type.name == "CUDA"]
    return sum(ts) / len(ts) if ts else None


def host_pick(logits, u):
    """Top-p and the draw on the host, then the picked token's log-probability and the top 20 of the row."""
    l64 = logits.astype(np.float64)
    z = l64 - l64.max(axis=1, keepdims=True)
    p = np.exp(z)
    order = np.argsort(-l64, axis=1, kind="stable")
    ps = np.take_along_axis(p, order, axis=1)
    cs = np.cumsum(ps, axis=1)
    n_keep = (cs < TOP_P * cs[:, -1:]).sum(axis=1) + 1
    S = logits.shape[0]
    picks = np.empty(S, np.int64)
    for s in range(S):
        k = n_keep[s]
        c = np.cumsum(ps[s, :k]) / cs[s, k - 1]
        picks[s] = order[s, min(int(np.searchsorted(c, u[s])), k - 1)]
    log_s = np.log(cs[:, -1])
    lp = z[np.arange(S), picks] - log_s
    top_lp = np.take_along_axis(z, order[:, :20], axis=1) - log_s[:, None]
    return picks, lp, top_lp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="7b")
    ap.add_argument("--new", type=int, default=64, help="tokens generated per stream")
    ap.add_argument("--rounds", type=int, default=3)
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

    plain, pen = Sm(1.0, TOP_P), Sm(1.0, TOP_P, 0, PEN, PEN, DECAY)
    cols = [("ex", plain, None, 0), ("raw", plain, "raw", 0), ("raw top20", plain, "raw", 20),
            ("processed", plain, "processed", 0), ("ex pen.", pen, None, 0), ("raw pen.", pen, "raw", 0)]
    print("\n%d new tokens per stream; ms per step, best of %d alternating rounds; host loop over %d steps"
          % (N, args.rounds, args.loop_steps))
    print("%5s" % "S" + "".join("%12s" % c[0] for c in cols) + "%12s" % "host loop" + "%14s %14s" % ("k top_n 0 us",
                                                                                                     "k top_n 20 us"))
    for S in STREAMS:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        streams = [(s, t) for s, t in enumerate(first)]
        u = rng.random((N, S))

        def gen(sampler, mode, top_n, n=N):
            if mode is None:
                out = eng.generate_streams(streams, n, u=u[:n], sampling=sampler)
            else:
                out = [r["tokens"] for r in eng.generate_streams(streams, n, u=u[:n], sampling=sampler, logprobs=mode,
                                                                 top_n=top_n)]
            assert all(len(o) == n for o in out)

        def loop():
            cur = list(first)
            for k in range(args.loop_steps):
                logits, _ = eng.forward_streams([(s, [t]) for s, t in enumerate(cur)])
                cur = [int(x) for x in host_pick(logits, u[k])[0]]

        fns = {c[0]: (lambda c=c: gen(*c[1:])) for c in cols}
        fns["host loop"] = loop
        steps = {name: N for name in fns}
        steps["host loop"] = args.loop_steps
        best = {name: 1e9 for name in fns}
        for name in fns:  # warm-up: graphs of the shape, every buffer touched
            fns[name]()
        for _ in range(args.rounds):
            for name in fns:
                t0 = time.perf_counter()
                fns[name]()
                best[name] = min(best[name], (time.perf_counter() - t0) / steps[name])
        k0 = kernel_us(lambda: gen(plain, "raw", 0, 16), "k_gen_logprob")
        k20 = kernel_us(lambda: gen(plain, "raw", 20, 16), "k_gen_logprob")
        fmt = lambda x: "%.1f" % x if x is not None else "not measured"
        print("%5d" % S + "".join("%12.3f" % (best[n] * 1e3) for n in fns) + "%14s %14s" % (fmt(k0), fmt(k20)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
