"""Every decode-kernel variant the engine instantiates is launched by some width of the GPU parity suite.

csrc/engine.cu instantiates k_token<CPL, FULL> for each CPL of RK_CPLS and both values of FULL, and picks one from
n_embed with chunks_per_lane (FULL = n_embed == CPL * 512). The widths of tests/test_widths_gpu.py together with those
of test_parity_gpu.test_engine_matches_oracle must reach every pair: adding a variant without a width that launches it
fails here, without a GPU."""
import os
import re

import test_parity_gpu
import test_widths_gpu
from util import PKG_DIR

ENGINE_CU = os.path.join(PKG_DIR, "csrc", "engine.cu")


def engine_source():
    with open(ENGINE_CU) as f:
        return f.read()


def rk_cpls():
    m = re.search(r"#define\s+RK_CPLS\(X\)((?:\s*X\(\d+\))+)", engine_source())
    assert m, "RK_CPLS not found in csrc/engine.cu"
    return [int(x) for x in re.findall(r"X\((\d+)\)", m.group(1))]


def chunks_per_lane(seg_bytes):
    """csrc/engine.cu, chunks_per_lane: 16-byte chunks per lane of a row (32 lanes), rounded up to an even count >= 2."""
    c = max((seg_bytes + 511) // 512, 2)
    return (c + 1) & ~1


def variant(E):
    cpl = chunks_per_lane(E)
    return cpl, E == cpl * 512


def parity_widths():
    marks = [m for m in test_parity_gpu.test_engine_matches_oracle.pytestmark if m.name == "parametrize"]
    names = [s.strip() for s in marks[0].args[0].split(",")]
    return {int(p[names.index("E")]) for p in marks[0].args[1]}


def test_restated_chunks_per_lane_is_the_engines():
    src = re.sub(r"\s+", " ", engine_source())
    body = "int chunks_per_lane(unsigned long long seg_bytes) { int c = (int)((seg_bytes + 511) / 512); if (c < 2) c = 2; return (c + 1) & ~1; }"
    assert body in src, "chunks_per_lane changed in csrc/engine.cu: restate it here"


def test_every_decode_variant_has_a_width():
    cpls = rk_cpls()
    assert cpls, "RK_CPLS is empty"
    widths = set(test_widths_gpu.WIDTHS) | parity_widths()
    for E in widths:  # every width is one the loader accepts (do_load)
        assert E % 16 == 0 and 132 <= E <= 5120, E
        assert variant(E)[0] in cpls, "E=%d needs CPL=%d, which RK_CPLS does not instantiate" % (E, variant(E)[0])
    reached = {variant(E) for E in widths}
    missing = [(c, f) for c in cpls for f in (False, True) if (c, f) not in reached]
    assert not missing, "decode-kernel variants <CPL, FULL> no GPU parity test launches: %s" % missing


def test_tensor_core_chunks_cover_every_pass_shape():
    """The single-stream chunks of test_widths_gpu reach every padded pass size, and a width with a K tail (E % 128 != 0)
    runs a chunk of more than one pass."""
    pads = set()
    for T in test_widths_gpu.WIDTHS.values():
        pads |= {(min(128, T - t0) + 31) // 32 * 32 for t0 in range(0, T, 128)}
    assert pads == {32, 64, 96, 128}, sorted(pads)
    assert any(E % 128 and T > 128 for E, T in test_widths_gpu.WIDTHS.items())
    assert any(E % 128 for E in test_widths_gpu.FEATURE_WIDTHS)
