import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
PKG_DIR = os.path.join(ROOT, "rwkv-cpp-accelerated_b200")
VOCAB_DIR = os.path.join(INCLUDE, "rwkv", "tokenizer", "vocab")


def compile_cpp(src, out, link_engine=False, extra=()):
    cmd = ["g++", "-O1", "-std=c++17", "-I" + INCLUDE, src, "-o", out] + list(extra)
    if link_engine:
        cmd += ["-L" + PKG_DIR, "-lrwkv_b200", "-Wl,-rpath," + PKG_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, "g++ failed:\n" + r.stderr[-4000:]
    return out


VOCAB = 50277
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def stress_model(src, dst, kind, L=3, E=768):
    """A copy of the L x E synthetic model `src` at `dst` with its layernorm parameters edited in place.
    LAYERNORMS = f64 [4(L+1)][E] after xbuf (f64 [E]) and embed (f32 [V][E]): rows 0,1 = ln0 w,b;
    4i+2, 4i+3 = ln1 of layer i; 4(i+1), 4(i+1)+1 = ln2 of layer i (convert_model.py:30-46)."""
    import shutil

    import numpy as np
    shutil.copyfile(src, dst)
    ln = np.memmap(dst, dtype=np.float64, mode="r+", offset=16 + 8 * E + 4 * VOCAB * E, shape=(4 * (L + 1), E))
    if kind == "outliers":
        rng = np.random.default_rng(7)
        for i in range(L):
            ch = rng.choice(E, size=3, replace=False)
            ln[4 * i + 2, ch] *= 300.0      # ln1 weight: three channels 300x the rest
            ln[4 * (i + 1), ch] *= 300.0    # ln2 weight
    elif kind == "tiny_residual":
        ln[0] *= 1e-3                       # ln0 weight and bias: residual stream of magnitude 1e-3
        ln[1] *= 1e-3
    elif kind == "offset_residual":
        ln[1] += 50.0                       # ln0 bias: |mean| >> std in every later layernorm
    else:
        raise ValueError(kind)
    ln.flush()
    del ln
    return dst


def reference_golden(name):
    """What the reference CUDA build computed for case `name` (tests/golden/make_reference_golden.py)."""
    import numpy as np
    with np.load(os.path.join(GOLDEN_DIR, "ref_%s.npz" % name)) as z:
        return {k: z[k] for k in z.files}


def golden_logits_err(got, g, i):
    """Relative error of a full logits vector against dumped step i of golden `g`, over the stored entries
    (a seeded sample of the vocabulary and the reference's 8 largest logits), relative to max|logits|."""
    import numpy as np
    got = np.asarray(got, np.float64)
    e = max(np.abs(got[g["idx"]] - g["logits"][i]).max(), np.abs(got[g["top_idx"][i]] - g["top_val"][i]).max())
    return float(e / max(float(g["maxabs"][i]), 1e-6))


def golden_state_err(state, g, k):
    """Relative error of a full state array against the golden sample of array `k`."""
    import numpy as np
    got = np.asarray(state, np.float64).reshape(-1)[g["state_%s_idx" % k]]
    return float(np.abs(got - g["state_%s" % k]).max() / max(float(g["state_%s_maxabs" % k]), 1e-6))
