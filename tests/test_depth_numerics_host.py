"""The float64 restatement of tests/numerics.py at production depth, on the CPU.

- The unquantised restatement against what the reference CUDA build computed on the bench models
  (tests/golden/ref_*.npz): 7B and 14B over their 64 tokens and 1.5B over its 1024, at the stored indices. This pins
  the restatement at 24 to 40 layers without the engine.
- The proof that tests/test_depth_numerics_gpu.py can see the bugs it is there for: on every case of that file, a
  mutated quantiser moves logits or state by at least 4 times the case's tolerance. The 3-layer wide cases run every
  mutation of numerics.MUTATIONS on every layer; the full-depth cases run a dropped limb plane in one middle layer only
  and in the last layer only, a bug that hits one layer of many (a ring-phase or exchange-tag slip at a layer
  boundary). Ragged passes are measured at the rows the GPU test compares.

What depth costs: the restatement's own sensitivity (one ulp of expf in sigma(r)) grows with the layers, to 1.1e-5 -
1.7e-5 of the state at 24 to 40 layers, so the state tolerance there is 4.4e-5 - 6.7e-5. A dequantisation scale off by
2^-16 in ONE layer of many moves the state by only 3.8e-5 - 6.0e-5 and the logits by 0.7e-5 - 1.4e-5: below 4 times
the tolerance on every full-depth case, at a middle layer and at the last. The GPU tests cannot tell that bug from the
restatement's own error at full depth; it is printed here, not asserted. Over 3 layers, or in every layer, they can.

Each case prints the wall time of its restatement. Measured on 8 host cores: 1.5B x 1024 exact 29 s, 7B x 64 26 s,
14B x 64 33 s; the whole file about 11 minutes."""
import time

import numpy as np
import pytest

import numerics as nm
from util import ROOT, golden_logits_err, golden_state_err, reference_golden

# Unquantised restatement against the reference's f32 CUDA build at full depth: measured 1.3e-6 (14B logits), 1.0e-6
# (7B logits), 8.9e-7 (14B dd), 8.3e-7 (1.5B logits): the small-width bound of tests/test_numerics_host.py holds.
EXACT_VS_GOLDEN = 2e-6
FULL_DEPTH_MUTATIONS = ("drop_plane0", "scale_2^-16")
BELOW_TOLERANCE_AT_DEPTH = ("scale_2^-16",)   # measured, see above: printed at full depth, not asserted


def bench_model(pkg, workload):
    import sys
    sys.path.insert(0, ROOT)
    import bench
    return nm.Model(bench.model_path(workload, pkg))


@pytest.mark.parametrize("workload,n", [("1b5", 1024), ("7b", 64), ("14b", 64)])
def test_exact_restatement_matches_reference_golden(pkg, workload, n):
    model = bench_model(pkg, workload)
    g = reference_golden(workload)
    toks = [int(t) for t in g["tokens"]]
    assert len(toks) == n
    t0 = time.time()
    lg, st = nm.forward(model, [toks], mode="exact")
    wall = time.time() - t0
    le = max(golden_logits_err(lg[0][s], g, i) for i, s in enumerate(int(s) for s in g["steps"]))
    se = {k: golden_state_err(st[0][k], g, k) for k in nm.KEYS}
    print("%s x %d tokens (%d x %d): exact restatement vs the reference CUDA build: logits %.3g, state %s; bound %.3g; "
          "restated in %.1f s" % (workload, n, model.L, model.E, le, " ".join("%s %.3g" % kv for kv in se.items()),
                                  EXACT_VS_GOLDEN, wall))
    assert le <= EXACT_VS_GOLDEN and max(se.values()) <= EXACT_VS_GOLDEN


def rows_compared(case_id):
    """The ragged GPU case compares each stream's last row (forward_streams returns no other); the others every row."""
    return (lambda x: x[-1:]) if case_id.startswith("ragged") else (lambda x: x)


def moved(model, p, lg, st):
    """Per case of pass p: (logits, state) distance of a mutated run (lg, st) from the plain one, at the GPU's rows."""
    out = {}
    for i, cid in enumerate(p["ids"]):
        rows = rows_compared(cid)
        le, se, _ = nm.worst([rows(lg[i])], [rows(p["logits"][i])], [st[i]], [p["final"][i]], model.L, model.E)
        a, b = out.get(cid, (0.0, 0.0))
        out[cid] = (max(a, le), max(b, se))
    return out


def case_tols(p):
    out = {}
    for cid, (tl, ts) in zip(p["ids"], p["tols"]):
        a, b = out.get(cid, (0.0, 0.0))
        out[cid] = (max(a, tl), max(b, ts))
    return out


@pytest.mark.parametrize("group", sorted(nm.WIDE) + sorted(nm.BENCH_CASES))
def test_mutations_exceed_the_gpu_tolerance_at_depth(pkg, make_model, group):
    """Each mutation moves logits or state of every case by >= 4 x its tolerance in tests/test_depth_numerics_gpu.py,
    numerics.case_tol of the case as restated in its group's pass (numerics.stream_tols)."""
    wide = group in nm.WIDE
    model = nm.Model(make_model(nm.DEPTH_L, group)) if wide else bench_model(pkg, group)
    t0 = time.time()
    ps = nm.passes(group, model, inputs=not wide)
    wall = time.time() - t0
    if wide:
        runs = [(mu, None) for mu in nm.MUTATIONS]
    else:
        runs = [(mu, [l]) for l in (model.L // 2, model.L - 1) for mu in FULL_DEPTH_MUTATIONS]
    t1 = time.time()
    failed = []
    for p in ps:
        for g in p["logits"]:
            assert np.isfinite(g).all()
        tols = case_tols(p)
        results = {cid: [] for cid in tols}
        for mu, layers in runs:
            lg, st = nm.forward(model, p["streams"], p["states"], mutation=mu, mutation_layers=layers,
                                inputs=p["inputs"] if layers else None)
            for cid, (le, se) in moved(model, p, lg, st).items():
                results[cid].append((mu, layers, le, se))
        for cid, rs in results.items():
            tl, ts = tols[cid]
            print("%s (%d x %d): tolerance logits %.3g state %.3g; 4 x tolerance %.3g %.3g; mutants move (logits, state) %s"
                  % (cid, model.L, model.E, tl, ts, 4 * tl, 4 * ts,
                     ", ".join("%s%s %.3g %.3g" % (mu, "" if ls is None else "@%d" % ls[0], le, se)
                               for mu, ls, le, se in rs)))
            failed += [(cid, mu, ls, le, se) for mu, ls, le, se in rs if not (le >= 4 * tl or se >= 4 * ts)
                       and (wide or mu not in BELOW_TOLERANCE_AT_DEPTH)]
    print("%s: restated with tolerances in %.1f s, mutants in %.1f s" % (group, wall, time.time() - t1))
    assert not failed, failed
