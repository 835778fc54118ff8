"""Regenerates tests/golden/ref_*.npz: what the unmodified reference CUDA build computes on the synthetic models
the GPU parity tests use, so that those tests compare against the reference without needing it at test time.

The reference (rwkv.cu + rwkv.h) is compiled into oracle/_ref/ref_harness by `make -C oracle ref`, which needs
the reference sources at build time; this script then needs a GPU. Each case is one ref_harness run:

  oracle_3x768          8 tokens teacher-forced on the oracle's greedy stream (tests/test_parity_gpu.py)
  169m, 1b5, 7b, 14b    greedy decode from token 4118 by the reference itself at the BASELINE sizes
  stress_<kind>         8 tokens teacher-forced on the oracle's greedy stream of an edited 3 x 768 model
                        (tests/test_long_parity_gpu.py)

A full logits vector is 201 KB, so each dumped step keeps the logits at a fixed seeded sample of 256 vocabulary
rows, the 8 largest logits, the arg-max, max|logits| and the top-1/top-2 margin; the final state keeps a seeded
sample of 4096 entries of each array and its max-abs.

Run:  python tests/golden/make_reference_golden.py [OUT_DIR]     (default: tests/golden)
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

SEED = 20240924
SEED_TOKEN = 4118
VOCAB = 50277
N_IDX, N_TOP, N_STATE = 256, 8, 4096

# name -> (workload or (L, E), tokens, dump_every, token source)
CASES = {
    "oracle_3x768": ((3, 768), 8, 1, "oracle"),
    "169m": ("169m", 256, 1, "greedy"),
    "1b5": ("1b5", 1024, 4, "greedy"),
    "7b": ("7b", 64, 1, "greedy"),
    "14b": ("14b", 64, 1, "greedy"),
    "stress_outliers": ((3, 768), 8, 1, "oracle"),
    "stress_tiny_residual": ((3, 768), 8, 1, "oracle"),
    "stress_offset_residual": ((3, 768), 8, 1, "oracle"),
}


def oracle_stream(path, n):
    from oracle.oracle import Oracle
    orc = Oracle(path)
    toks, tok = [], SEED_TOKEN
    for _ in range(n):
        toks.append(tok)
        tok = int(orc.forward(tok).argmax())
    orc.close()
    return toks


def summarise(d, toks):
    rng = np.random.default_rng(SEED)
    idx = np.sort(rng.choice(VOCAB, size=N_IDX, replace=False))
    lg = np.stack(d["logits"])
    top_idx = np.argsort(-lg, axis=1, kind="stable")[:, :N_TOP]
    out = {"tokens": np.array(toks, np.int64), "steps": np.array(d["steps"], np.int64), "idx": idx.astype(np.int64),
           "logits": lg[:, idx].astype(np.float32), "top_idx": top_idx.astype(np.int64),
           "top_val": np.take_along_axis(lg, top_idx, axis=1).astype(np.float32),
           "argmax": lg.argmax(axis=1).astype(np.int64), "maxabs": np.abs(lg).max(axis=1).astype(np.float64)}
    top2 = np.sort(lg, axis=1)[:, -2:].astype(np.float64)
    out["margin"] = (top2[:, 1] - top2[:, 0]) / np.maximum(out["maxabs"], 1e-6)
    for k in ("xy", "aa", "bb", "dd"):
        s = d["state"][k]
        si = np.sort(rng.choice(s.size, size=min(N_STATE, s.size), replace=False))
        out["state_%s_idx" % k] = si.astype(np.int64)
        out["state_%s" % k] = s[si]
        out["state_%s_maxabs" % k] = np.float64(np.abs(s).max())
    return out


def main():
    import importlib
    import bench
    from oracle.oracle import REF_HARNESS, read_ref_dump
    from util import stress_model
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    if not os.path.exists(REF_HARNESS):
        sys.exit("oracle/_ref/ref_harness is not built (make -C oracle ref, with the reference sources present)")
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    with tempfile.TemporaryDirectory() as td:
        small = os.path.join(td, "syn_L3_E768.bin")
        pkg.build.genmodel(3, 768, SEED, small)
        for name, (shape, n, every, src) in CASES.items():
            if isinstance(shape, str):
                path = bench.model_path(shape, pkg)
            elif name.startswith("stress_"):
                path = stress_model(small, os.path.join(td, name + ".bin"), name[len("stress_"):])
            else:
                path = small
            tf = os.path.join(td, "tokens.txt")
            dump = os.path.join(td, "dump.bin")
            cmd = [REF_HARNESS, path, tf, dump, "--dump-every", str(every)]
            if src == "greedy":
                with open(tf, "w") as f:
                    f.write("%d\n" % SEED_TOKEN)
                cmd += ["--greedy", str(n)]
            else:
                with open(tf, "w") as f:
                    f.write("\n".join(map(str, oracle_stream(path, n))))
            r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
            if r.returncode != 0:
                sys.exit("%s: ref_harness failed:\n%s%s" % (name, r.stdout[-2000:], r.stderr[-2000:]))
            toks = [int(x) for x in open(dump + ".tokens").read().split()]
            d = read_ref_dump(dump)
            np.savez_compressed(os.path.join(out_dir, "ref_%s.npz" % name), **summarise(d, toks))
            print("%s: %d tokens, %d dumped steps" % (name, len(toks), len(d["steps"])), flush=True)


if __name__ == "__main__":
    main()
