"""What log-probabilities and token automata cost speculative generation, against generate_streams with the same
features, in the same run, alternating.

Four feature sets, each run by every call below:
  plain     arg-max, nothing else
  logprobs  processed log-probabilities with top_n 5
  automaton a token automaton on every stream (regex [a-z ,.]+, eos 0, as batcher_mix_bench.py uses)
  both      the two together
Calls:
  spec k=K ctx   generate_speculative with K drafts and one of two lookup contexts: ceiling (the stream's own output under
                 the same features: nearly every draft is right) or floor (256 random tokens: drafts rarely fit, and under
                 the automaton most rows die at their first draft)
  gen-tc         generate_streams on the tensor cores (prefill_min = 2; a lone stream gets a pad stream): the call whose
                 tokens and log-probabilities spec reproduces, checked in the warm-up
  gen-default    generate_streams with the default path (the decode kernel below 8 streams)

Every call starts from zeroed first slots. Host timer around calls that return synchronised; every shape is warmed first;
each row is the best of --rounds alternating rounds, in ms per emitted token, with spec's tokens per step. --profile
takes, in a run of its own, the mean device time per launch of the speculative step's kernels from torch.profiler, for
the "both" set. The card's name and power limit are read in the same run.
usage: python spec_constrained_bench.py [workloads=7b 169m] [--new N] [--rounds R] [--profile]"""
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
CONTEXTS = ("ceiling", "floor")
SETS = ("plain", "logprobs", "automaton", "both")
KERNELS = ("k_spec_draft", "k_gen_mask", "k_argmax_rows", "k_spec_accept", "k_spec_logprob")


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


def same(a, b):
    """Tokens, and the log-probability fields by bits."""
    if not isinstance(b, dict):
        return np.array_equal(a["tokens"] if isinstance(a, dict) else a, b)
    return all(np.asarray(a[f]).tobytes() == np.asarray(b[f]).tobytes() for f in b if f != "steps")


def run_workload(pkg, workload, args):
    kmax = max(DRAFTS)
    eng = pkg.Engine(bench.model_path(workload, pkg), max_gpt=max(STREAMS) * (kmax + 1))
    L, E = bench.SHAPES[workload]
    C = pkg.constrain
    cid = eng.add_constraint(C.token_automaton(C.compile_regex(r"[a-z ,.]+"), C.token_bytes(), eos=0))
    N = args.new
    rng = np.random.default_rng(1)
    pad = max(STREAMS) * (kmax + 1) - 1  # never a first slot: first slots are s * (kmax + 1)
    print("\nworkload %s (L=%d, E=%d), max_new = %d, arg-max, ngram = 3, best of %d alternating rounds"
          % (workload, L, E, N, args.rounds), flush=True)

    def feats(fs, S):
        kw = {}
        if fs in ("logprobs", "both"):
            kw.update(logprobs="processed", top_n=5)
        if fs in ("automaton", "both"):
            kw["constraints"] = [cid] * S
        return kw

    def zero(S):
        for s in range(S):
            eng.slot_zero(s * (kmax + 1))

    def strip(res, S):
        return [{f: v for f, v in r.items() if f != "state"} if isinstance(r, dict) else r for r in res[:S]]

    def gen(S, first, fs, tc):
        zero(S)
        kw = feats(fs, S)
        streams = [(s * (kmax + 1), first[s]) for s in range(S)]
        if tc:
            eng.set_option("prefill_min", 2)
            if S < 2:
                streams.append((pad, first[0]))
                if "constraints" in kw:
                    kw["constraints"] = kw["constraints"] + [None]
        out = eng.generate_streams(streams, N, sampling=pkg.Sampler(temperature=0.0), **kw)
        eng.set_option("prefill_min", 8)
        return strip(out, S), None

    def spec(S, first, fs, k, context):
        zero(S)
        res = eng.generate_speculative([([s * (kmax + 1) + i for i in range(k + 1)], first[s]) for s in range(S)], N, k,
                                       context=context, **feats(fs, S))
        return strip(res, S), sum(r["steps"] for r in res)

    def tokens_of(res):
        return [[int(x) for x in (r["tokens"] if isinstance(r, dict) else r)] for r in res]

    if args.profile:
        print("kernel time, one call, feature set 'both' (us per launch, launches)", flush=True)
        for S in STREAMS:
            first = [int(t) for t in rng.integers(0, 50000, S)]
            ref, _ = gen(S, first, "both", True)
            for c in CONTEXTS:
                ctx = ([[first[s]] + tokens_of(ref)[s] for s in range(S)] if c == "ceiling" else
                       [[int(x) for x in rng.integers(0, 50000, 256)] for _ in range(S)])
                for k in DRAFTS:
                    spec(S, first, "both", k, ctx)
                    r = kernel_us(lambda: spec(S, first, "both", k, ctx), KERNELS)
                    print("S = %2d, k = %d, %-7s: " % (S, k, c) + ", ".join(
                        "%s %s (%d)" % (n, "%.1f" % r[n][0] if r[n][0] is not None else "-", r[n][1]) for n in KERNELS),
                        flush=True)
        eng.close()
        return

    print("%4s %-9s %3s %8s %12s %9s %12s %12s %9s" % ("S", "features", "k", "context", "spec ms/tok", "tok/step",
                                                       "gen-tc", "gen-default", "vs gen-tc"), flush=True)
    for S in STREAMS:
        first = [int(t) for t in rng.integers(0, 50000, S)]
        floor = [[int(x) for x in rng.integers(0, 50000, 256)] for _ in range(S)]
        fns, refs = {}, {}
        for fs in SETS:
            refs[fs], _ = gen(S, first, fs, True)
            ceiling = [[first[s]] + tokens_of(refs[fs])[s] for s in range(S)]
            fns[(fs, "gen-tc")] = lambda fs=fs: gen(S, first, fs, True)
            fns[(fs, "gen-default")] = lambda fs=fs: gen(S, first, fs, False)
            for k in DRAFTS:
                for c, ctx in (("ceiling", ceiling), ("floor", floor)):
                    fns[(fs, k, c)] = lambda fs=fs, k=k, ctx=ctx: spec(S, first, fs, k, ctx)
        best, tps = {}, {}
        for key, fn in fns.items():  # warm-up: grows every buffer, records the graphs; checks against gen-tc
            res, steps = fn()
            if key[1] != "gen-default":
                assert all(same(a, b) for a, b in zip(res, refs[key[0]])), "%s: differs from gen-tc" % (key,)
            n_tok = sum(len(t) for t in tokens_of(res))
            tps[key] = n_tok / steps if steps else None
            best[key] = (1e9, n_tok)
        for _ in range(args.rounds):
            for key, fn in fns.items():
                t0 = time.perf_counter()
                fn()
                best[key] = (min(best[key][0], time.perf_counter() - t0), best[key][1])
        ms = {key: best[key][0] / best[key][1] * 1e3 for key in best}
        for fs in SETS:
            for k in DRAFTS:
                for c in CONTEXTS:
                    x = ms[(fs, k, c)]
                    print("%4d %-9s %3d %8s %12.3f %9.2f %12.3f %12.3f %8.2fx" % (
                        S, fs, k, c, x, tps[(fs, k, c)], ms[(fs, "gen-tc")], ms[(fs, "gen-default")],
                        ms[(fs, "gen-tc")] / x), flush=True)
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["7b", "169m"])
    ap.add_argument("--new", type=int, default=48, help="max_new of each stream")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="kernel times instead of the table")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    for w in args.workloads:
        run_workload(pkg, w, args)


if __name__ == "__main__":
    main()
