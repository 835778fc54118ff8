"""Constrained generation on the device (rwkv_b200_generate_streams_constrained) against unconstrained generation and
against the host loop it replaces.

  generate  --new tokens per stream at S = 1, 16, 128; ms per step, best of --rounds alternating rounds, of
            generate_streams_ex (T = 1, top_p = 0.85), the same call constrained by the fixed-key JSON regex, and
            constrained by a one-state automaton that allows every token (the cost of the mask and the automaton advance
            alone). The JSON streams end on completion; the call still runs whole groups of 16 steps, so its time is
            divided by the steps it ran (the longest stream rounded up to 16), and the longest stream is reported
  kernel    device time of one k_gen_mask launch, from the CUDA kernel records of torch.profiler over one call of 16 steps
  host      what a caller does without the entry point: forward_streams with logits, the numpy mask of each stream's
            automaton state, sample_streams(logits=...), the automaton advanced on the host; --loop-steps steps, best of
            --rounds

The card's name and power limit are read in the same run.
usage: python constrain_bench.py [workload=7b] [--new N] [--rounds R] [--loop-steps N]"""
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
TOP_P = 0.85
JSON = r'\{"name": "[a-z]{1,12}", "age": \d{1,3}\}'


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
    C = pkg.constrain
    t0 = time.perf_counter()
    json_ta = C.token_automaton(C.compile_regex(JSON), C.token_bytes(), eos=0)
    print("JSON automaton: %d states, %d edges, built in %.2f s" % (json_ta.n_states, len(json_ta.edge_tokens),
                                                                    time.perf_counter() - t0), flush=True)
    allowed = np.zeros((json_ta.n_states, V), bool)
    for q in range(json_ta.n_states):
        allowed[q, json_ta.edges(q)[0].astype(np.int64)] = True
    eng = pkg.Engine(bench.model_path(args.workload, pkg), max_gpt=max(STREAMS))
    json_id, all_id = eng.add_constraint(json_ta), eng.add_constraint(C.allow_all())
    L, E = bench.SHAPES[args.workload]
    N = args.new
    rng = np.random.default_rng(1)
    print("workload %s (L=%d, E=%d)" % (args.workload, L, E), flush=True)
    sp = pkg.Sampler(1.0, TOP_P)
    cols = ("ex", "json", "allow-all", "host loop")
    print("\n%d new tokens per stream; ms per step, best of %d alternating rounds; host loop over %d steps"
          % (N, args.rounds, args.loop_steps))
    print("%5s" % "S" + "".join("%12s" % c for c in cols) + "%12s %14s" % ("json len/ran", "k_gen_mask us"))
    for S in STREAMS:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        streams = [(s, t) for s, t in enumerate(first)]
        u = rng.random((N, S))
        ran, longest = {}, [0]

        def gen(cid, n=N):
            if cid is None:
                out = eng.generate_streams(streams, n, u=u[:n], sampling=sp)
                assert all(len(o) == n for o in out)
                return n
            out = eng.generate_streams(streams, n, u=u[:n], sampling=sp, constraints=cid)
            m = max(len(r["tokens"]) for r in out)
            if cid == json_id:
                longest[0] = m
            return min(n, -(-m // 16) * 16)

        def loop():
            cur, state = list(first), [0] * S
            for k in range(args.loop_steps):
                logits, _ = eng.forward_streams([(s, [t]) for s, t in enumerate(cur)])
                for s in range(S):
                    logits[s][~allowed[state[s]]] = -np.inf
                toks, _ = eng.sample_streams(sp, u[k], logits=logits)
                cur = [int(x) for x in toks]
                for s in range(S):
                    q = json_ta.walk([cur[s]], state[s])
                    state[s] = 0 if json_ta.complete(q) else q  # a completed stream starts a new object
            return args.loop_steps

        fns = {"ex": lambda: gen(None), "json": lambda: gen(json_id), "allow-all": lambda: gen(all_id), "host loop": loop}
        best = {name: 1e9 for name in fns}
        for name in fns:  # warm-up: graphs of the shape, every buffer touched
            fns[name]()
        for _ in range(args.rounds):
            for name in fns:
                t0 = time.perf_counter()
                ran[name] = fns[name]()
                best[name] = min(best[name], (time.perf_counter() - t0) / ran[name])
        km = kernel_us(lambda: gen(all_id, 16), "k_gen_mask")
        fmt = lambda x: "%.1f" % x if x is not None else "not measured"
        print("%5d" % S + "".join("%12.3f" % (best[n] * 1e3) for n in cols) + "%12s %14s" % (
            "%d / %d" % (longest[0], ran["json"]), fmt(km)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
