"""Device-resident beam search against the host loop a caller needs without it, in the same run, alternating.

  device  one beam_search call: G groups of B = 4 beams, max_new = 64, no stop tokens (every group runs every step),
          length penalty 1
  loop    per step forward_streams with the logits of every live beam (201 KB per beam over PCIe), a numpy float64
          log-softmax and top-B per row, the selection of the group's B best, and slot_copy for each fork
          (--loop-steps steps timed)

Host timer around calls that return synchronised; every shape is warmed first (its first tensor-core call records the
CUDA graph of the pass); each row reports the best of --rounds alternating rounds, in ms per step. A separate run takes
the kernel time of k_beam_expand, k_beam_select and k_beam_fork from torch.profiler over one call. The card's name and
power limit are read in the same run.
usage: python beam_bench.py [workload=7b] [--new N] [--rounds R] [--loop-steps S]"""
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

GROUPS = (1, 4, 16, 32)
B = 4
ALPHA = 1.0


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
    ap.add_argument("--new", type=int, default=64, help="max_new of each group")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-steps", type=int, default=16)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(GROUPS) * B)
    L, E = bench.SHAPES[args.workload]
    N = args.new
    rng = np.random.default_rng(1)
    print("workload %s (L=%d, E=%d), B = %d, max_new = %d, alpha = %g, best of %d alternating rounds"
          % (args.workload, L, E, B, N, ALPHA, args.rounds), flush=True)

    def device(G, first):
        eng.beam_search([(list(range(g * B, (g + 1) * B)), first[g]) for g in range(G)], N, B, length_penalty=ALPHA)

    def loop(G, first):
        beams = [[(g * B, first[g], 0.0)] for g in range(G)]  # per group: (slot, input token, cum)
        for step in range(args.loop_steps):
            call = [(s, [t]) for bs in beams for s, t, _ in bs]
            logits, _ = eng.forward_streams(call)
            l64 = logits.astype(np.float64)
            m = l64.max(axis=1, keepdims=True)
            lp = (l64 - m) - np.log(np.exp(l64 - m).sum(axis=1, keepdims=True))
            top = np.argpartition(-l64, B - 1, axis=1)[:, :B]
            r = 0
            for g, bs in enumerate(beams):
                cands = []
                for j, (s, _, cum) in enumerate(bs):
                    for v in top[r]:
                        cands.append((cum + lp[r, v], j, int(v)))
                    r += 1
                cands.sort(key=lambda x: (-x[0], x[1]))
                new = cands[:B]
                prev = [s for s, _, _ in bs] if step else list(range(g * B, (g + 1) * B))
                child = {j for _, j, _ in new}
                free = [p for p in range(B) if p not in child]
                taken, nb = set(), []
                for c, j, v in new:
                    if j not in taken:
                        taken.add(j)
                        nb.append((prev[j], v, c))
                    else:
                        dst = prev[free.pop(0)]
                        eng.slot_copy(prev[j], dst)
                        nb.append((dst, v, c))
                beams[g] = nb

    print("\n%5s %7s %16s %16s %9s" % ("G", "rows", "loop ms/step", "device ms/step", "speed-up"), flush=True)
    for G in GROUPS:
        first = [int(t) for t in rng.integers(0, 50000, G)]
        best = {"loop": 1e9, "device": 1e9}
        steps = {"loop": args.loop_steps, "device": N}
        fns = {"loop": loop, "device": device}
        for name in fns:  # warm-up: records the graphs of the shapes, grows every buffer
            fns[name](G, first)
        for _ in range(args.rounds):
            for name in ("loop", "device"):
                t0 = time.perf_counter()
                fns[name](G, first)
                best[name] = min(best[name], (time.perf_counter() - t0) / steps[name])
        print("%5d %7d %16.3f %16.3f %8.2fx" % (G, G * B, best["loop"] * 1e3, best["device"] * 1e3, best["loop"] / best["device"]),
              flush=True)

    print("\nkernel time, one call (us per launch, launches)", flush=True)
    names = ("k_beam_expand", "k_beam_select", "k_beam_fork")
    for G in GROUPS:
        first = [int(t) for t in rng.integers(0, 50000, G)]
        k = kernel_us(lambda: device(G, first), names)
        print("G = %2d: " % G + ", ".join("%s %s (%d)" % (n, "%.1f" % k[n][0] if k[n][0] is not None else "-", k[n][1])
                                            for n in names), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
