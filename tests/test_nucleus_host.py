"""rwkv_b200_sample_streams / rwkv_b200_generate_streams_ex without a GPU: declared by the Python binding, added without
an ABI version change, the Python Sampler laid out as the C struct, and safe to call with a NULL handle."""
import ctypes
import os
import subprocess

import numpy as np

from util import compile_cpp

SIZEOF_SRC = r"""
#include <cstddef>
#include <cstdio>
#include "rwkv_b200.h"
int main() {
    std::printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(rwkv_b200_sampler), offsetof(rwkv_b200_sampler, temperature),
                offsetof(rwkv_b200_sampler, top_p), offsetof(rwkv_b200_sampler, top_k),
                offsetof(rwkv_b200_sampler, presence_penalty), offsetof(rwkv_b200_sampler, frequency_penalty),
                offsetof(rwkv_b200_sampler, penalty_decay));
    return 0;
}
"""


def test_binding_declares_the_sampler_entry_points(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_sample_streams" in lib._declared
    assert "rwkv_b200_generate_streams_ex" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_python_struct_matches_the_header(pkg, tmp_path):
    src = tmp_path / "sizeof.cpp"
    src.write_text(SIZEOF_SRC)
    exe = compile_cpp(str(src), str(tmp_path / "sizeof"))
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    S = pkg.Sampler
    want = [ctypes.sizeof(S)] + [getattr(S, f).offset for f, _ in S._fields_]
    assert got == want


def test_sampler_defaults(pkg):
    s = pkg.Sampler()
    assert (s.temperature, s.top_p, s.top_k, s.presence_penalty, s.frequency_penalty, s.penalty_decay) == (1.0, 1.0, 0, 0.0, 0.0, 1.0)


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    sp = (pkg.Sampler * 1)(pkg.Sampler())
    u = np.array([0.5], np.float64)
    toks, margins = np.zeros(1, np.uint64), np.zeros(1, np.float64)
    rc = lib.rwkv_b200_sample_streams(None, 1, sp, u.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), None,
                                      toks.ctypes.data_as(P), margins.ctypes.data_as(ctypes.POINTER(ctypes.c_double)))
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
    slots, first = np.array([0], np.uint64), np.array([4118], np.uint64)
    out, lens = np.zeros(4, np.uint64), np.zeros(1, np.uint64)
    rc = lib.rwkv_b200_generate_streams_ex(None, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 4, None, None, 0, None,
                                           None, 0, sp, None, out.ctypes.data_as(P), lens.ctypes.data_as(P))
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
