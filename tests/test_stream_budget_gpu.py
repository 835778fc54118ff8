"""The token kernel's weight-stream schedule (set_option "sub_bytes", "budget", "qbudget": bulk-copy size and bytes in
flight per SM, csrc/token_kernel.cuh produce_token) only decides when weight bytes arrive, never what is computed with
them: every setting must give the logits and the five state arrays of the defaults bit for bit.

Covered: the exact consume_sub path (n_embed = 4096, the 7B rows, on three layers) and the bounded one (784, a width of
tests/test_widths_gpu.py), copies from 1 KB to a whole stage, the smallest and largest budgets, and greedy decode_timed
over 40 tokens."""
import os

import numpy as np
import pytest

from util import token_stream

pytestmark = pytest.mark.gpu

KEYS = ("xy", "aa", "bb", "pp", "dd")
SHAPES = {"exact": (3, 4096), "bounded": (2, 784)}


@pytest.fixture(scope="module")
def stream_models(pkg, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("stream_budget"))
    out = {}
    for kind, (L, E) in SHAPES.items():
        out[kind] = os.path.join(d, "L%d_E%d.bin" % (L, E))
        pkg.build.genmodel(L, E, 4242 + E, out[kind])
    return out


def settings(E):
    tile, top = 8 * E, 12 * 8 * E  # a stage holds 8 rows; budgets go up to 12 stages

    def sub(n):  # a copy is at most one stage (6272 bytes at n_embed = 784)
        return min(n, tile)
    return [
        {"sub_bytes": 1024}, {"sub_bytes": sub(4096)}, {"sub_bytes": sub(8192)}, {"sub_bytes": tile},
        {"sub_bytes": sub(4096), "qbudget": 0}, {"sub_bytes": sub(8192), "qbudget": 16384},
        {"sub_bytes": 1024, "budget": tile, "qbudget": 0},          # smallest budgets
        {"sub_bytes": sub(4096), "budget": top, "qbudget": top},    # largest budgets
        {"budget": tile, "qbudget": top},
    ]


def teacher_forced(pkg, path, opts, toks):
    eng = pkg.Engine(path)
    eng.set_option("prefill", 0)  # every token through the decode kernel
    for k, v in opts.items():
        eng.set_option(k, v)
    logits = np.stack([eng.forward([t])[0] for t in toks])
    state = eng.state_download()
    eng.close()
    return logits, state


def assert_same(got, want, what):
    (gl, gs), (wl, ws) = got, want
    assert np.array_equal(gl, wl), "%s: logits differ from the default schedule" % what
    for k in KEYS:
        assert np.array_equal(gs[k], ws[k]), "%s: state %s differs from the default schedule" % (what, k)


@pytest.mark.parametrize("kind", sorted(SHAPES))
def test_schedules_are_bit_identical(pkg, stream_models, kind):
    L, E = SHAPES[kind]
    toks = token_stream(6, seed=E)
    want = teacher_forced(pkg, stream_models[kind], {}, toks)
    for opts in settings(E):
        assert_same(teacher_forced(pkg, stream_models[kind], opts, toks), want, "E=%d %s" % (E, opts))


@pytest.mark.parametrize("kind", sorted(SHAPES))
def test_greedy_decode_timed_is_bit_identical(pkg, stream_models, kind):
    L, E = SHAPES[kind]

    def run(opts):
        eng = pkg.Engine(stream_models[kind])
        for k, v in opts.items():
            eng.set_option(k, v)
        eng.state_zero()
        eng.decode_timed([4118] * 40, teacher_forced=False)
        out = eng.debug_read("logits").copy(), eng.state_download()
        eng.close()
        return out

    want = run({})
    for opts in ({"sub_bytes": 4096, "qbudget": 4096}, {"sub_bytes": 2048, "budget": 12 * 8 * E, "qbudget": 0}):
        assert_same(run(opts), want, "E=%d decode_timed %s" % (E, opts))


def test_option_ranges(pkg, stream_models):
    E = SHAPES["bounded"][1]
    tile = 8 * E
    eng = pkg.Engine(stream_models["bounded"])
    for k, v in (("sub_bytes", 8), ("sub_bytes", 1000), ("sub_bytes", tile + 16), ("budget", tile - 16),
                 ("budget", 12 * tile + 16), ("qbudget", -1), ("qbudget", 12 * tile + 16), ("window", 2)):
        with pytest.raises(Exception):
            eng.set_option(k, v)
    for k, v in (("sub_bytes", 16), ("sub_bytes", tile), ("budget", tile), ("qbudget", 0), ("qbudget", 12 * tile)):
        eng.set_option(k, v)
    eng.close()
