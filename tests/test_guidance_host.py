"""Classifier-free guidance without a GPU: the declaration and export of rwkv_b200_generate_streams_guided, the NULL
handle, the header's constant and struct against the binding's, and engine.guide_rows (rule 2 of include/rwkv_b200.h)
against an f64 evaluation of the formula."""
import ctypes
import os
import re

import numpy as np

from util import ROOT

HEADER = os.path.join(ROOT, "include", "rwkv_b200.h")


def test_symbol_declared_and_exported(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_generate_streams_guided" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2
    text = open(HEADER).read()
    assert re.search(r"int rwkv_b200_generate_streams_guided\(", text)


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    args = [None] * 26
    args[3], args[4], args[7], args[10] = 1, 4, 0, 0  # n_streams, max_new, n_stop, n_override
    args[15], args[16] = 0, 0  # logprob_mode, top_n
    assert lib.rwkv_b200_generate_streams_guided(*args) != 0
    assert b"null model handle" in lib.rwkv_b200_last_error()


def test_constant_and_struct_match_the_header(pkg):
    E = pkg.engine
    text = open(HEADER).read()
    m = re.search(r"#define RWKV_B200_NO_GUIDANCE (0x[0-9A-Fa-f]+)ULL", text)
    assert m and int(m.group(1), 16) == E.NO_GUIDANCE
    body = re.search(r"typedef struct rwkv_b200_guidance \{(.*?)\} rwkv_b200_guidance;", text, re.S).group(1)
    names = ["slots", "first_tokens", "scales"]
    assert re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S)) == names
    assert [f for f, _ in E.Guidance._fields_] == names
    assert [getattr(E.Guidance, f).offset for f in names] == [0, 8, 16] and ctypes.sizeof(E.Guidance) == 24


def test_guide_rows_scale_one_is_the_identity(pkg):
    rng = np.random.default_rng(1)
    for _ in range(4):
        c = (rng.standard_normal(50277) * 8).astype(np.float32)
        q = (rng.standard_normal(50277) * 8).astype(np.float32)
        got = pkg.engine.guide_rows(c, q, 1.0)
        assert got.dtype == np.float32 and got.tobytes() == c.tobytes()


def test_guide_rows_matches_the_formula(pkg):
    """Within the rounding of three f32 operations of an f64 evaluation; bit for bit the numpy float32 expression."""
    rng = np.random.default_rng(2)
    for scale in (0.0, 0.5, 1.5, 3.0, 100.0):
        c = (rng.standard_normal((3, 50277)) * 8).astype(np.float32)
        q = (rng.standard_normal((3, 50277)) * 8).astype(np.float32)
        got = pkg.engine.guide_rows(c, q, scale)
        w = np.float32(np.float32(scale) - np.float32(1))
        assert got.tobytes() == (c + w * (c - q)).tobytes()
        c64, q64 = c.astype(np.float64), q.astype(np.float64)
        ref = c64 + float(w) * (c64 - q64)
        bound = 3 * np.finfo(np.float32).eps * (np.abs(c64) + abs(float(w)) * (np.abs(c64) + np.abs(q64)))
        assert np.all(np.abs(got.astype(np.float64) - ref) <= bound + 1e-30), scale
    # gamma 0 is the guidance row itself up to rounding: c + (-1) * (c - q)
    got = pkg.engine.guide_rows(c, q, 0.0)
    assert np.all(np.abs(got.astype(np.float64) - q64) <= 2 * np.finfo(np.float32).eps * (np.abs(c64) + np.abs(q64)))


def test_python_arguments(pkg):
    E = pkg.engine
    g = E._guidance([None, (5, 11, 1.5)], 2, "generate_streams")
    assert list(g._keep[0]) == [E.NO_GUIDANCE, 5] and list(g._keep[1]) == [0, 11]
    assert g._keep[2].dtype == np.float32 and list(g._keep[2]) == [1.0, 1.5]
