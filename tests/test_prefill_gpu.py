"""Batched forward over T tokens (SURVEY 8f N1 / N3): the int8 tensor-core GEMM path (csrc/prefill.cuh) against
the token-by-token decode kernel of the same engine, and a short chunk against the CPU oracle. The two paths
quantise the same numbers and accumulate exactly; they differ only in the order of a few double-precision sums
(layernorm statistics, offset sums), so they agree to ~1e-6 of max|logits| - far inside the 1e-3 contract."""
import numpy as np
import pytest

from util import rel_err, token_stream

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("L,E,T", [(3, 768, 16), (2, 2048, 40), (2, 4096, 16), (2, 4096, 64), (2, 4096, 128), (1, 5120, 32)])
def test_gpt_chunk_on_tensor_cores_matches_decode_kernel(pkg, make_model, L, E, T):
    path = make_model(L, E)
    toks = token_stream(T, seed=3)
    a = pkg.Engine(path, max_gpt=T)
    chunk = a.forward(toks, mode=1)          # >= 16 tokens: the batched path
    sa = a.state_download()
    b = pkg.Engine(path, max_gpt=T)
    b.set_option("prefill", 0)               # the same call, token by token through the decode kernel
    single = b.forward(toks, mode=1)
    sb = b.state_download()
    worst = max(rel_err(chunk[t], single[t]) for t in range(T))
    print("L=%d E=%d T=%d: batched vs token-by-token worst logits rel err %.3g" % (L, E, T, worst))
    assert worst < 2e-5
    n = a.n_layers * a.n_embed
    for k in ("xy", "aa", "bb", "dd"):
        ref = sb[k][:n]
        assert np.abs(sa[k][:n] - ref).max() / max(np.abs(ref).max(), 1e-6) < 2e-5, k
    # and the next single token continues from the chunk's state
    nxt = int(single[-1].argmax())
    assert rel_err(a.forward([nxt])[0], b.forward([nxt])[0]) < 2e-5
    a.close()
    b.close()


def test_gpt_chunk_matches_oracle(pkg, make_model):
    from oracle.oracle import Oracle
    path = make_model(3, 768)
    toks = token_stream(24, seed=5)
    eng = pkg.Engine(path, max_gpt=24)
    got = eng.forward(toks, mode=1)
    orc = Oracle(path)
    worst = 0.0
    for t, tok in enumerate(toks):
        worst = max(worst, rel_err(got[t], orc.forward(tok)))
    print("batched chunk vs oracle: worst logits rel err %.3g" % worst)
    assert worst < 1e-3
    st = eng.state_download()
    for k in ("xy", "aa", "bb", "dd"):
        ref = orc.state[k]
        assert np.abs(st[k][:ref.size] - ref).max() / max(np.abs(ref).max(), 1e-6) < 1e-3, k
    eng.close()
    orc.close()


def test_parralel_streams_on_tensor_cores(pkg, make_model):
    """MODE::PARRALEL: token t on state slot t (rwkv.cu:238-240); 16 streams, two steps each."""
    path = make_model(2, 2048)
    T = 16
    toks1, toks2 = token_stream(T, seed=7), token_stream(T, seed=8)
    a = pkg.Engine(path, max_gpt=T)
    first = a.forward(toks1, mode=0)
    second = a.forward(toks2, mode=0)
    b = pkg.Engine(path)
    for i in range(T):
        b.state_zero()
        assert rel_err(first[i], b.forward([toks1[i]])[0]) < 2e-5
        assert rel_err(second[i], b.forward([toks2[i]])[0]) < 2e-5
    a.close()
    b.close()


def test_prefill_throughput_reported(pkg, make_model):
    """Prompt tokens/s of the batched path vs T x the single-token time (E = 4096, two layers + head)."""
    import time
    path = make_model(2, 4096)
    T = 128
    toks = token_stream(T, seed=3)
    a = pkg.Engine(path, max_gpt=T)
    a.forward(toks, mode=1, want_logits=False)
    t0 = time.perf_counter()
    for _ in range(3):
        a.forward(toks, mode=1, want_logits=False)
    batched = (time.perf_counter() - t0) / 3
    a.set_option("prefill", 0)
    a.forward(toks, mode=1, want_logits=False)
    t0 = time.perf_counter()
    a.forward(toks, mode=1, want_logits=False)
    single = time.perf_counter() - t0
    print("T=%d: batched %.2f ms (%.0f prompt tokens/s), token by token %.2f ms (%.0f tokens/s): %.1fx"
          % (T, batched * 1e3, T / batched, single * 1e3, T / single, single / batched))
    assert batched < single
    a.close()
