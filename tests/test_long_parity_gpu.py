"""Parity at the sizes and lengths BASELINE.json names, against the REFERENCE ITSELF: what the unmodified
rwkv.cu + rwkv.h computed on the same seeded models (tests/golden/ref_*.npz, written by
tests/golden/make_reference_golden.py from a greedy decode by the reference). The engine replays the same tokens
teacher-forced, token by token through the decode kernel and as one GPT chunk on the tensor cores; logits are compared
at every dumped step and the recurrent state at the end. Plus stress models
for the fixed-point activation quantiser and the layernorm statistics: outlier channels, a tiny residual stream
and a residual stream with a large mean.

Tolerance (north_star): logits within 1e-3 of max|logits|; arg-max identical wherever the reference's own
top-1 / top-2 margin exceeds 1e-3 of max|logits|."""
import sys

import numpy as np
import pytest

from util import REL_TOL, ROOT, SEED_TOKEN, golden_logits_err, golden_state_err, reference_golden, rel_err, stress_model

pytestmark = pytest.mark.gpu


def compare_with_reference(pkg, path, name, n_tokens):
    """Teacher-force the engine on the tokens of golden case `name` and compare with the reference's outputs."""
    g = reference_golden(name)
    toks = [int(t) for t in g["tokens"]]
    assert len(toks) >= n_tokens
    want = {int(s): i for i, s in enumerate(g["steps"])}
    eng = pkg.Engine(path)
    worst, checked = 0.0, 0
    for step in range(n_tokens):
        if step in want:
            i = want[step]
            got = eng.forward([toks[step]])[0]
            e = golden_logits_err(got, g, i)
            worst = max(worst, e)
            assert e < REL_TOL, "step %d: logits rel err %.3g" % (step, e)
            if g["margin"][i] > 1e-3:
                assert int(got.argmax()) == int(g["argmax"][i]), "step %d argmax" % step
                checked += 1
        else:
            eng.forward([toks[step]], want_logits=False)
    st = eng.state_download()
    for k in ("xy", "aa", "bb", "dd"):
        assert golden_state_err(st[k], g, k) < REL_TOL, "state %s" % k
    eng.close()
    return worst, checked, len(want), toks


def bench_model(pkg, workload):
    sys.path.insert(0, ROOT)
    import bench
    return bench.model_path(workload, pkg)


@pytest.mark.parametrize("workload,n_tokens,dump_every", [
    ("169m", 256, 1),    # BASELINE config 2: 169M storygen, 256 tokens
    ("1b5", 1024, 4),    # BASELINE config 3: 1.5B, 1k tokens
    ("7b", 64, 1),       # BASELINE config 4 (headline): the bench model itself
    ("14b", 64, 1),      # BASELINE config 5 at full depth (40 x 5120) on one GPU
])
def test_decode_matches_the_reference_at_baseline_sizes(pkg, workload, n_tokens, dump_every):
    assert set(range(0, n_tokens, dump_every)) <= {int(s) for s in reference_golden(workload)["steps"]}
    worst, checked, compared, _ = compare_with_reference(pkg, bench_model(pkg, workload), workload, n_tokens)
    print("%s x %d tokens vs the reference CUDA build: worst logits rel err %.3g over %d compared steps, argmax checked on %d"
          % (workload, n_tokens, worst, compared, checked))


@pytest.mark.parametrize("workload,n_tokens", [
    ("169m", 256),   # two passes of 128
    ("1b5", 1024),   # eight passes of 128
    ("7b", 64),      # one pass of 64
    ("14b", 64),     # one pass of 64 at 40 x 5120
])
def test_tensor_core_chunk_matches_the_reference_at_baseline_sizes(pkg, workload, n_tokens):
    """The same token lists as one GPT-mode forward on the tensor cores (csrc/prefill.cuh), compared at every dumped
    step and in the final state."""
    g = reference_golden(workload)
    toks = [int(t) for t in g["tokens"]][:n_tokens]
    assert len(toks) == n_tokens
    eng = pkg.Engine(bench_model(pkg, workload), max_gpt=n_tokens)
    got = eng.forward(toks, mode=1)
    worst, checked, compared = 0.0, 0, 0
    for i, step in enumerate(int(s) for s in g["steps"]):
        if step >= n_tokens:
            continue
        e = golden_logits_err(got[step], g, i)
        worst = max(worst, e)
        compared += 1
        assert e < REL_TOL, "step %d: logits rel err %.3g" % (step, e)
        if g["margin"][i] > 1e-3:
            assert int(got[step].argmax()) == int(g["argmax"][i]), "step %d argmax" % step
            checked += 1
    st = eng.state_download()
    eng.close()
    serr = max(golden_state_err(st[k], g, k) for k in ("xy", "aa", "bb", "dd"))
    print("%s x %d tokens in one tensor-core chunk vs the reference CUDA build: worst logits rel err %.3g over %d compared "
          "steps, argmax checked on %d, state %.3g" % (workload, n_tokens, worst, compared, checked, serr))
    assert serr < REL_TOL


@pytest.mark.parametrize("kind", ["outliers", "tiny_residual", "offset_residual"])
def test_stress_models_match_oracle_and_reference(pkg, make_model, tmp_path, kind):
    """Activation vectors with outlier channels 10^2-10^3 x the median (real RWKV-4 checkpoints have them) leave
    the typical element few quantisation levels of the per-vector scale; a residual stream of magnitude 1e-3 or
    with |mean| >> std probes the layernorm statistics."""
    from oracle.oracle import Oracle
    path = stress_model(make_model(3, 768), str(tmp_path / ("stress_%s.bin" % kind)), kind)
    orc = Oracle(path)
    eng = pkg.Engine(path)
    toks, tok, worst = [], SEED_TOKEN, 0.0
    for step in range(8):
        toks.append(tok)
        got = eng.forward([tok])[0]
        ref = orc.forward(tok)
        assert np.all(np.isfinite(ref))
        e = rel_err(got, ref)
        worst = max(worst, e)
        assert e < REL_TOL, "%s step %d: logits rel err %.3g" % (kind, step, e)
        tok = int(ref.argmax())
    eng.close()
    orc.close()
    w2, _, _, ref_toks = compare_with_reference(pkg, path, "stress_" + kind, 8)
    assert ref_toks == toks, "the oracle's greedy stream differs from the one the reference ran"
    print("%s: worst logits rel err vs oracle %.3g, vs the reference CUDA build %.3g" % (kind, worst, w2))
