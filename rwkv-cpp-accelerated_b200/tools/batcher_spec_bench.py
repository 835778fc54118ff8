"""Speculation in the batcher (rwkv_b200_batcher_submit_spec) against the same requests without it.

Per workload, rows R and draft k: R arg-max requests, each with a 128-token prompt and max_new = --max-new, all submitted
at once to Engine.batcher(R, 512) and run in 16-step groups until every one is done. The prompts are fed into the
slots beforehand (untimed), so a timed run is the decode phase: each request's prompt in the batcher is its last
token, and the rest of the prompt is the front of its lookup context, so the lookup history is the same as with the
whole prompt submitted. Three contexts:

  ceiling   the request's own arg-max output before the prompt: every draft is right wherever the lookup locks on
  floor     128 random tokens before the prompt
  none      the prompt only

Reported: ms per emitted token (wall time of the whole run over the tokens emitted) for the plain batcher and with
speculation, their ratio, and tokens per step of the speculative requests. Each number is the best of --rounds rounds
that alternate the two systems; every round checks that both emit the same tokens. The card's name and power limit are
read in the same run.
usage: python batcher_spec_bench.py [--workloads 7b 169m] [--rows 1 8 16 32] [--drafts 2 4] [--max-new 128]
       [--rounds 3]"""
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
PROMPT = 128
PREFILL = 512


def feed(eng, prompts):
    """Slot i holds prompt i but its last token, from a zero state (forward_streams calls of at most max_gpt tokens,
    state only)."""
    call, n = [], 0
    for i, p in enumerate(prompts):
        eng.slot_zero(i)
        call.append((i, p[:-1]))
        n += len(p) - 1
        if n + PROMPT > eng.max_gpt:
            eng.forward_streams(call, want_logits=False)
            call, n = [], 0
    if call:
        eng.forward_streams(call, want_logits=False)


def run(eng, prompts, max_new, k=0, contexts=None):
    """One timed batcher run: (seconds, tokens per request, steps per request)."""
    feed(eng, prompts)
    R = len(prompts)
    t0 = time.perf_counter()
    with eng.batcher(R, PREFILL) as bat:
        ids = []
        for i, p in enumerate(prompts):
            if k:
                spares = [R + i * k + j for j in range(k)]
                ids.append(bat.submit(i, p[-1:], max_new, draft=k, spare_slots=spares, ngram=3,
                                      context=list(contexts[i]) + list(p[:-1])))
            else:
                ids.append(bat.submit(i, p[-1:], max_new))
        while bat.run(16):
            pass
        dt = time.perf_counter() - t0
        res = [bat.result(i) for i in ids]
    return dt, [[int(x) for x in r["tokens"]] for r in res], [r.get("steps", 0) for r in res]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["7b", "169m"])
    ap.add_argument("--rows", type=int, nargs="+", default=[1, 8, 16, 32])
    ap.add_argument("--drafts", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--max-new", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[0] if card else "unknown (nvidia-smi gave nothing)"), flush=True)
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    rng = np.random.default_rng(7)
    for wl in args.workloads:
        R_max = max(args.rows)
        eng = pkg.Engine(bench.model_path(wl, pkg), max_gpt=max(R_max * (max(args.drafts) + 1), PROMPT * 2))
        L, E = bench.SHAPES[wl]
        print("\nworkload %s (L=%d, E=%d), prompts of %d tokens, max_new %d, arg-max, best of %d alternating rounds"
              % (wl, L, E, PROMPT, args.max_new, args.rounds), flush=True)
        print("%5s %3s %-8s %12s %12s %7s %11s" % ("rows", "k", "context", "plain ms/t", "spec ms/t", "ratio", "tokens/step"))
        for R in args.rows:
            prompts = [[int(x) for x in rng.integers(0, V, size=PROMPT)] for _ in range(R)]
            _, own, _ = run(eng, prompts, args.max_new)  # the ceiling contexts; also warms the plain shapes
            ctxs = {"ceiling": own, "floor": [[int(x) for x in rng.integers(0, V, size=PROMPT)] for _ in range(R)],
                    "none": [[] for _ in range(R)]}
            for k in args.drafts:
                for name in ("ceiling", "floor", "none"):
                    run(eng, prompts, args.max_new, k, ctxs[name])  # warm
                    best_p = best_s = 1e9
                    for _ in range(args.rounds):
                        tp, toks_p, _ = run(eng, prompts, args.max_new)
                        ts, toks_s, steps = run(eng, prompts, args.max_new, k, ctxs[name])
                        assert toks_s == toks_p, "speculation changed the tokens (rows %d, k %d, %s)" % (R, k, name)
                        best_p, best_s = min(best_p, tp), min(best_s, ts)
                    n = sum(len(t) for t in toks_p)
                    print("%5d %3d %-8s %12.3f %12.3f %7.2f %11.2f" % (R, k, name, 1e3 * best_p / n, 1e3 * best_s / n,
                                                                      best_p / best_s, n / sum(steps)), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
