"""The engine against the float64 restatement of its own arithmetic (tests/numerics.py, "engine" mode), within 1e-5:
logits at every token (relative to max|logits| of the token) and the state after the last token, per layer and per
array (bb element by element, relative to itself). Where the restatement itself moves by more than a quarter of that
when sigma(r)'s expf rounds differently by one ulp (numerics.sensitivity: the outlier-channel model, ~3e-5), the case
is held to 4 times that movement instead, since no restatement short of the kernel's own bits predicts it.

The engine's only rounding is the activation quantiser, so it reproduces the restatement to ~5e-7; a limb, quantiser or
dequantisation-scale bug moves logits or state by 4e-5 or more (tests/test_numerics_host.py proves that for these cases
on the CPU), well above this tolerance and far below the 1e-3 contract tolerance of the other parity tests.

Cases (numerics.cases()): the decode kernel at one width per (CPL, FULL) variant, a tensor-core chunk at every padded
pass size and one of two passes with a K tail, MODE::PARRALEL, a ragged forward_streams pass on slots holding state,
the stress models, and quantiser edges: a token-shift state with one element 10^2 (K/V/R input) or 10^4 (ffn input)
times the rest and negative, every ffn key negative (the ffn-V input is all zeros), exactly one ffn key positive. Every
case prints its worst error against the restatement, the unquantised restatement and the CPU oracle."""
import numpy as np
import pytest

import numerics as nm

pytestmark = pytest.mark.gpu

CASES = [pytest.param(c, id=c["id"]) for c in nm.cases()]
RAGGED_SLOTS = (5, 0, 3, 6)


def run_engine(pkg, path, case, streams, states):
    """(logits per stream, state per stream) from the engine: every token's logits, except on the ragged path, which
    returns each stream's last row."""
    L, E = case["L"], case["E"]
    n = L * E
    if case["path"] in ("decode", "tc"):
        toks = streams[0]
        eng = pkg.Engine(path, max_gpt=len(toks))
        # both paths named explicitly: the decode kernel for every token, or the tensor cores from 2 tokens on
        eng.set_option("prefill", 0) if case["path"] == "decode" else eng.set_option("prefill_min", 2)
        if states:
            eng.state_upload(states[0])
        logits = [eng.forward(toks, mode=1)]
        st = [eng.state_download()]
    elif case["path"] == "parralel":
        eng = pkg.Engine(path, max_gpt=len(streams))
        eng.set_option("prefill_min", 2)
        logits = list(eng.forward([s[0] for s in streams], mode=0)[:, None, :])
        sd = eng.state_download(len(streams))
        st = [{k: sd[k][i * n:(i + 1) * n] for k in sd} for i in range(len(streams))]
    else:
        slots = max(RAGGED_SLOTS) + 1
        eng = pkg.Engine(path, max_gpt=64)
        eng.set_option("prefill_min", 2)
        up = {k: np.zeros(slots * n) for k in nm.KEYS}
        for slot, s in zip(RAGGED_SLOTS, states):
            for k in nm.KEYS:
                up[k][slot * n:(slot + 1) * n] = s[k]
        eng.state_upload(up, slots)
        lg, _ = eng.forward_streams(list(zip(RAGGED_SLOTS, streams)))
        logits = [row[None, :] for row in lg]
        sd = eng.state_download(slots)
        st = [{k: sd[k][s * n:(s + 1) * n] for k in sd} for s in RAGGED_SLOTS]
    eng.close()
    return logits, st


def oracle_run(path, streams, states, L, E):
    from oracle.oracle import Oracle
    orc = Oracle(path)
    logits, st = [], []
    for i, toks in enumerate(streams):
        orc.reset()
        if states:
            for k in nm.KEYS:
                orc.state[k][:] = states[i][k]
        logits.append(np.stack([orc.forward(t) for t in toks]))
        st.append({k: orc.state[k].copy() for k in nm.KEYS})
    orc.close()
    return logits, st


@pytest.mark.parametrize("case", CASES)
def test_engine_matches_restatement(pkg, make_model, tmp_path_factory, case):
    L, E = case["L"], case["E"]
    path = nm.case_model(case, make_model, str(tmp_path_factory.getbasetemp()))
    model = nm.Model(path)
    streams, states = nm.inputs(case, model)
    got_l, got_s = run_engine(pkg, path, case, streams, states)
    for g in got_l:
        assert np.isfinite(g).all(), "%s: non-finite logits" % case["id"]
    for s in got_s:
        for k in nm.KEYS:
            assert np.isfinite(s[k][:L * E]).all(), "%s: non-finite state %s" % (case["id"], k)
    ragged = case["path"] == "ragged"
    rows = (lambda ls: [x[-1:] for x in ls]) if ragged else (lambda ls: ls)
    tol_l, tol_s = nm.case_tol(model, streams, states)
    report = []
    for what, mode in (("restatement", "engine"), ("exact", "exact"), ("oracle", None)):
        ref_l, ref_s = oracle_run(path, streams, states, L, E) if mode is None else nm.forward(model, streams, states, mode)
        le, se, sk = nm.worst(got_l, rows(ref_l), got_s, ref_s, L, E)
        report.append("%s logits %.3g state %.3g (%s)" % (what, le, se, sk))
        if mode == "engine":
            errs = (le, se, sk)
    report.append("tolerance logits %.3g state %.3g" % (tol_l, tol_s))
    print("%s: vs %s" % (case["id"], "; vs ".join(report)))
    le, se, sk = errs
    assert le <= tol_l, "%s: logits %.3g from the restatement" % (case["id"], le)
    assert se <= tol_s, "%s: state %s %.3g from the restatement" % (case["id"], sk, se)


def test_quant_scale_and_expf_as_restated(tmp_path):
    """The two device functions the restatement reproduces on the host: quant_scale (rcp.approx.ftz plus one Newton
    step, then the steps down) equals numerics.quant_inv for every f32 mantissa, so the reciprocal after the Newton step
    is the rounded 1 / m wherever it matters; and expf, which numerics.expf takes as correctly rounded, is within its
    documented 2 ulp (on an H100: 30 % of the arguments off the rounded value). Those differences are why the outlier
    model is held to numerics.case_tol rather than TOL."""
    import os
    import subprocess

    from util import PKG_DIR, ROOT
    pkg_build = __import__("importlib").import_module("rwkv-cpp-accelerated_b200.build")
    exe, out = str(tmp_path / "probe"), str(tmp_path / "probe.bin")
    r = subprocess.run([pkg_build.nvcc(), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I" + os.path.join(PKG_DIR, "csrc"), os.path.join(ROOT, "tests", "helpers", "quant_scale_probe.cu"),
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    r = subprocess.run([exe, out], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = np.fromfile(out, np.uint32)
    nm_, ne = 1 << 23, 1 << 20
    m = (np.uint32(0x3F800000) | np.arange(nm_, dtype=np.uint32)).view(np.float32)
    host = nm.quant_inv(m).view(np.uint32)
    bad = int(np.count_nonzero(raw[:nm_] != host))
    x, e = raw[nm_:nm_ + ne].view(np.float32), raw[nm_ + ne:].view(np.float32)
    ref = nm.expf(-x)
    ulps = np.abs(e.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    print("quant_scale: %d of %d mantissas differ from the restatement; expf: %.4f of arguments off the rounded value, "
          "at most %d ulp" % (bad, nm_, float(np.mean(ulps > 0)), int(ulps.max())))
    assert bad == 0
    assert ulps.max() <= 2
