"""Device sampler (SURVEY §8f N4): rwkv_b200_sample_typical / RWKV::sample against the host sampler, which is
itself pinned to the reference binary's sequences (tests/test_sampler.py)."""
import os
import subprocess

import numpy as np
import pytest

from decoding import host_pick
from util import ROOT, compile_cpp

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("temp", [0.9, 0.5, 1.0, 0.3, 2.0])
def test_device_sampler_matches_host_distribution(pkg, make_model, temp):
    eng = pkg.Engine(make_model(2, 768))
    rng = np.random.default_rng(7)
    tok, unsure = 4118, 0
    for step in range(6):
        logits = eng.forward([tok])[0]
        us = list(rng.random(40)) + [1e-12, 0.5, 1.0 - 1e-12]
        ref0, cp = host_pick(logits, temp, us[0])
        for u in us:
            got, margin = eng.sample_typical(temp, float(u))
            want = int(np.searchsorted(cp, u, side="left"))
            if margin >= 1e-9:
                assert got == want, "temp %g step %d u %.17g: device %d host %d (margin %g)" % (temp, step, u, got, want, margin)
            else:
                unsure += 1      # the C++ wrapper lets the host decide these
                assert abs(got - want) <= 1
        tok = int(logits.argmax())
    assert unsure <= 12          # only the two probes per step placed next to 0 and 1 may be ambiguous
    eng.close()


def test_rwkv_sample_equals_typical_sequence(pkg, make_model, tmp_path):
    """C++ surface: RWKV::sample() draws the token typical(out, ...) draws from the same generator state."""
    exe = compile_cpp(os.path.join(ROOT, "tests", "helpers", "sample_gpu_test.cpp"), str(tmp_path / "sample_gpu_test"),
                      link_engine=True)
    r = subprocess.run([exe, make_model(2, 768)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALL OK 200 draws" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
