"""The float64 restatement of the engine's forward (tests/numerics.py) on the CPU: the unquantised restatement against
the CPU oracle, the engine restatement against the unquantised one, and the proof that tests/test_numerics_gpu.py can
see the bugs it is there for: every mutation of the quantiser moves logits or state by at least 4 times the case's
tolerance on every case of that file up to width 1040. The wider cases (decode kernel at 2048 and up) are left out to
bound the time and the size of the models; the mutations move the restatement by the same amounts there (1.8e-4 for a
dropped limb plane, 7.5e-5 for a 15-bit quantiser at 1 x 5120)."""
import numpy as np
import pytest

import numerics as nm

EXACT_VS_ORACLE = 2e-6   # f64 against the reference's f32 accumulation: measured <= 1.7e-6 (bb at 1 x 5120)
ENGINE_VS_EXACT = 2e-6   # the quantiser's rounding on the plain synthetic models: measured <= 1.3e-6
POWER_CASES = [c for c in nm.cases() if c["E"] <= 1040]
# On the stress models and at the quantiser edges the quantiser's resolution is what the case stresses (the outlier
# channels alone move the engine restatement 3.6e-4 from the unquantised one in bb), so there only the power check runs.
NEAR_EXACT = [c for c in POWER_CASES if c["edge"] is None and c["kind"] is None]


def _model(case, make_model, tmp_path_factory):
    path = nm.case_model(case, make_model, str(tmp_path_factory.getbasetemp()))
    return path, nm.Model(path)


@pytest.mark.parametrize("L,E,T", [(2, 768, 8), (2, 144, 6), (1, 1040, 6)])
def test_exact_restatement_matches_oracle(make_model, L, E, T):
    """Pins the restatement: the oracle restates the reference's CUDA build, which tests/test_parity_gpu.py pins."""
    from oracle.oracle import Oracle
    from util import token_stream
    path = make_model(L, E)
    model = nm.Model(path)
    toks = token_stream(T, seed=E)
    lg, st = nm.forward(model, [toks], mode="exact")
    orc = Oracle(path)
    ref = np.stack([orc.forward(t) for t in toks])
    le, se, sk = nm.worst(lg, [ref], st, [orc.state], L, E)
    orc.close()
    print("%d x %d: exact restatement vs oracle: logits %.3g, state %.3g (%s)" % (L, E, le, se, sk))
    assert le <= EXACT_VS_ORACLE and se <= EXACT_VS_ORACLE


@pytest.mark.parametrize("case", NEAR_EXACT, ids=[c["id"] for c in NEAR_EXACT])
def test_engine_restatement_near_exact(make_model, tmp_path_factory, case):
    path, model = _model(case, make_model, tmp_path_factory)
    streams, states = nm.inputs(case, model)
    en_l, en_s = nm.forward(model, streams, states, "engine")
    ex_l, ex_s = nm.forward(model, streams, states, "exact")
    le, se, sk = nm.worst(en_l, ex_l, en_s, ex_s, case["L"], case["E"])
    print("%s: engine restatement vs exact: logits %.3g, state %.3g (%s)" % (case["id"], le, se, sk))
    assert le <= ENGINE_VS_EXACT and se <= ENGINE_VS_EXACT


@pytest.mark.parametrize("case", POWER_CASES, ids=[c["id"] for c in POWER_CASES])
def test_mutations_exceed_the_gpu_tolerance(make_model, tmp_path_factory, case):
    """Each mutation moves logits or state by >= 4 x the case's tolerance in tests/test_numerics_gpu.py (numerics.TOL,
    or 4 x the restatement's sensitivity on the outlier-channel model), so the GPU test fails on each of those bugs."""
    path, model = _model(case, make_model, tmp_path_factory)
    streams, states = nm.inputs(case, model)
    base_l, base_s = nm.forward(model, streams, states, "engine")
    for g in base_l:
        assert np.isfinite(g).all()
    ex_l, ex_s = nm.forward(model, streams, states, "exact")
    floor = max(nm.worst(base_l, ex_l, base_s, ex_s, case["L"], case["E"])[:2])
    moved = {}
    for mu in nm.MUTATIONS:
        ml, ms = nm.forward(model, streams, states, "engine", mutation=mu)
        moved[mu] = nm.worst(ml, base_l, ms, base_s, case["L"], case["E"])[:2]
    tol_l, tol_s = nm.case_tol(model, streams, states)
    print("%s: engine vs exact %.3g, tolerance logits %.3g state %.3g; mutants move (logits, state) %s"
          % (case["id"], floor, tol_l, tol_s, ", ".join("%s %.3g %.3g" % (k, *v) for k, v in moved.items())))
    for mu, (le, se) in moved.items():
        assert le >= 4 * tol_l or se >= 4 * tol_s, (mu, le, se)
