"""Both forward paths at every kind of model width the loader accepts (n_embed % 16 == 0, <= 5120), against the CPU
oracle.

The decode kernel has one template variant per (CPL, FULL) pair (csrc/engine.cu, RK_CPLS and chunks_per_lane): CPL =
16-byte chunks per lane of an n_embed-byte row, FULL = n_embed == CPL * 512. WIDTHS holds one width per variant that
tests/test_parity_gpu.py does not launch, including the RWKV-4 430M (1024) and 3B (2560) widths, plus widths that are
not a multiple of 128: there every tensor-core GEMM ends in a partial 128-byte K tile (csrc/prefill.cuh, k_gemm_i8).
tests/test_widths_host.py checks that these widths and the ones of test_parity_gpu.py reach every variant.

Tolerances are those of the other parity tests: logits within 1e-3 of max|logits| and the arg-max identical wherever
the oracle's top-1 / top-2 margin exceeds 1e-3 of max|logits|; the tensor-core path within 2e-5 of the decode kernel
(tests/test_prefill_gpu.py) and bit-exact between a ragged pass and each stream alone (tests/test_streams_gpu.py)."""
import numpy as np
import pytest

from decoding import KEYS4, V, check_generated, host_loop, run_pair, run_ragged_vs_solo
from util import REL_TOL, margin, rel_err, token_stream

pytestmark = pytest.mark.gpu

PATH_TOL = 2e-5
L = 2

# n_embed -> tokens of the single-stream GPT chunk on the tensor cores. Every padded pass size (Tp = 32, 64, 96, 128)
# gets one, and two chunks at widths with a K tail take two passes.
WIDTHS = {
    144: 20,    # <2,F>, E % 128 = 16: the narrowest width a 132-CTA grid takes, some CTAs own one row; Tp = 32
    272: 40,    # <2,F>, E % 128 = 16; Tp = 64
    784: 72,    # <2,F>, E % 128 = 16; Tp = 96
    1024: 128,  # <2,T>, RWKV-4 430M; Tp = 128
    1040: 200,  # <4,F>, E % 128 = 16; passes of 128 and 72 tokens (Tp = 128, 96)
    2560: 33,   # <6,F>, RWKV-4 3B; Tp = 64
    3072: 96,   # <6,T>; Tp = 96
    3600: 112,  # <8,F>, E % 128 = 16; Tp = 128
    5104: 140,  # <10,F>, E % 128 = 112; passes of 128 and 12 tokens (Tp = 128, 32)
}
FEATURE_WIDTHS = [784, 2560]  # one width with a K tail, one real model width


def oracle_run(path, toks):
    """The oracle's logits after every token of `toks` from the zero state, and its state after the last."""
    from oracle.oracle import Oracle
    orc = Oracle(path)
    logits = np.stack([orc.forward(t) for t in toks])
    state = {k: orc.state[k].copy() for k in KEYS4}
    orc.close()
    return logits, state


def check_rows(got, ref, what):
    """Every row of `got` against the oracle's: (worst logits error, rows whose arg-max was checked)."""
    worst, checked = 0.0, 0
    for t in range(len(ref)):
        e = rel_err(got[t], ref[t])
        worst = max(worst, e)
        assert e < REL_TOL, "%s, token %d: logits rel err %.3g" % (what, t, e)
        if margin(ref[t]) > 1e-3:
            assert int(got[t].argmax()) == int(ref[t].argmax()), "%s, token %d: argmax" % (what, t)
            checked += 1
    return worst, checked


def state_err(got, ref):
    n = ref["xy"].size
    return max(rel_err(got[k][:n], ref[k]) for k in KEYS4)


@pytest.mark.parametrize("E", sorted(WIDTHS))
def test_decode_kernel_matches_oracle(pkg, make_model, E):
    """Eight teacher-forced tokens through the decode kernel variant of the width; logits and final state."""
    worst, n = run_pair(pkg, make_model(L, E), 8)
    print("E=%d decode kernel vs oracle: worst logits rel err %.3g (argmax checked on %d/8 steps)" % (E, worst, n))


@pytest.mark.parametrize("E", sorted(WIDTHS))
def test_gpt_chunk_on_tensor_cores_matches_oracle(pkg, make_model, E):
    """One GPT chunk on the tensor cores against the oracle token by token, against the same call through the decode
    kernel, and the next single token from the chunk's state."""
    T = WIDTHS[E]
    path = make_model(L, E)
    toks = token_stream(T, seed=E)
    a = pkg.Engine(path, max_gpt=T)
    chunk = a.forward(toks, mode=1)
    sa = a.state_download()
    ref, ref_state = oracle_run(path, toks)
    worst, checked = check_rows(chunk, ref, "E=%d T=%d chunk" % (E, T))
    se = state_err(sa, ref_state)
    assert se < REL_TOL, "E=%d chunk state vs oracle: %.3g" % (E, se)
    b = pkg.Engine(path, max_gpt=T)
    b.set_option("prefill", 0)
    single = b.forward(toks, mode=1)
    sb = b.state_download()
    path_worst = max(rel_err(chunk[t], single[t]) for t in range(T))
    print("E=%d T=%d: tensor cores vs oracle worst logits rel err %.3g (argmax checked on %d/%d), state %.3g; "
          "vs decode kernel %.3g" % (E, T, worst, checked, T, se, path_worst))
    assert path_worst < PATH_TOL
    n = a.n_layers * a.n_embed
    for k in KEYS4:
        assert rel_err(sa[k][:n], sb[k][:n]) < PATH_TOL, k
    nxt = int(single[-1].argmax())
    assert rel_err(a.forward([nxt])[0], b.forward([nxt])[0]) < PATH_TOL
    a.close()
    b.close()


@pytest.mark.parametrize("E", sorted(WIDTHS))
def test_parralel_on_tensor_cores(pkg, make_model, E):
    """MODE::PARRALEL, 16 tokens on slots 0..15: every slot as the decode kernel on a zeroed slot."""
    path = make_model(L, E)
    T = 16
    toks = token_stream(T, seed=E + 1)
    a = pkg.Engine(path, max_gpt=T)
    got = a.forward(toks, mode=0)
    b = pkg.Engine(path)
    worst = 0.0
    for i in range(T):
        b.state_zero()
        worst = max(worst, rel_err(got[i], b.forward([toks[i]])[0]))
    print("E=%d PARRALEL x %d vs decode kernel: worst logits rel err %.3g" % (E, T, worst))
    assert worst < PATH_TOL
    a.close()
    b.close()


@pytest.mark.parametrize("E", FEATURE_WIDTHS)
def test_ragged_pass_matches_each_stream_alone(pkg, make_model, E):
    """forward_streams: a ragged pass on slots that hold state, one stream crossing the 128-token cut."""
    lens, slots = [1, 7, 33, 150, 20], [9, 0, 3, 200, 5]
    streams = [(s, token_stream(n, seed=E + i)) for i, (s, n) in enumerate(zip(slots, lens))]
    run_ragged_vs_solo(pkg, make_model(L, E), 256, streams)


@pytest.mark.parametrize("E", FEATURE_WIDTHS)
def test_score_streams_match_oracle(pkg, make_model, E):
    """score_streams over two streams of 40 tokens against a float64 log-softmax of the oracle's logits.

    The engine's logits are within REL_TOL * max|l| of the oracle's, so a log-probability l_y - logsumexp(l) is within
    2 * REL_TOL * max|l| (l_y and the log-sum-exp each move by at most the largest logit error). The rank (tokens
    ranked before the target) must lie between the count of tokens whose oracle logit beats the target's by more than
    two logit errors and the count that come within two errors of it, hence equal the oracle's rank wherever no logit
    is that close to the target's. A random next token sits among many near-equal logits, so a third of the targets are
    the oracle's top-1 and a third its third-ranked token, where the gaps are wide enough to pin the rank."""
    path = make_model(L, E)
    seqs = [token_stream(40, seed=E + 10), token_stream(40, seed=E + 11)]
    refs = [oracle_run(path, seq)[0] for seq in seqs]
    targets = []
    for seq, ref in zip(seqs, refs):
        order = [np.lexsort((np.arange(V), -row)) for row in ref]
        targets.append([seq[t + 1] if t % 3 == 0 else int(order[t][0 if t % 3 == 1 else 2]) for t in range(len(seq) - 1)] + [None])
    eng = pkg.Engine(path, max_gpt=128)
    res = eng.score_streams([(0, seqs[0]), (1, seqs[1])], targets)
    eng.close()
    worst, exact = 0.0, 0
    for ref, tg, r in zip(refs, targets, res):
        for t, y in enumerate(tg[:-1]):
            l = ref[t].astype(np.float64)
            scale = np.abs(l).max()
            tol = 2 * REL_TOL * scale
            lp = (l[y] - l.max()) - np.log(np.exp(l - l.max()).sum())
            got = float(r["logprobs"][t])
            worst = max(worst, abs(got - lp) / scale)
            assert abs(got - lp) <= tol, (t, got, lp)
            lo = int(np.count_nonzero(l > l[y] + tol))       # ahead of the target whatever the errors
            hi = int(np.count_nonzero(l >= l[y] - tol)) - 1  # possibly ahead (the target itself not counted)
            rank = int(r["ranks"][t])
            assert lo <= rank <= hi, (t, rank, lo, hi)
            exact += lo == hi
        assert np.isnan(r["logprobs"][-1])
    print("E=%d score_streams vs oracle: worst log-probability error %.3g of max|logits|, rank pinned on %d of 78"
          % (E, worst, exact))
    assert exact >= 26  # at least half of the 52 top-1 and third-ranked targets


@pytest.mark.parametrize("E", FEATURE_WIDTHS)
def test_generate_greedy_on_tensor_cores(pkg, make_model, E):
    """generate_streams, arg-max, 12 streams (every step on the tensor cores): token for token the host loop of
    forward_streams + arg-max, and the oracle's greedy continuation wherever its margin exceeds 1e-3."""
    from oracle.oracle import Oracle
    path = make_model(L, E)
    max_gpt, max_new = 16, 12
    a = pkg.Engine(path, max_gpt=max_gpt)
    b = pkg.Engine(path, max_gpt=max_gpt)
    slots = [9, 0, 3, 12, 5, 1, 14, 7, 2, 11, 6, 10]
    streams = list(zip(slots, token_stream(12, seed=E + 20)))
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new)
    want = host_loop(b, streams, max_new)
    check_generated(a, b, before, streams, got, want, max_gpt, "E=%d" % E)
    a.close()
    b.close()
    orc = Oracle(path)
    checked = 0
    for (_, first), seq in zip(streams, got):
        orc.reset()
        for i, tok in enumerate([first] + [int(x) for x in seq[:-1]]):
            ref = orc.forward(tok)
            if margin(ref) > 1e-3:
                assert int(seq[i]) == int(ref.argmax()), "E=%d stream from %d, token %d" % (E, first, i)
                checked += 1
    orc.close()
    print("E=%d generate_streams x 12: oracle's greedy pick checked on %d of %d tokens" % (E, checked, 12 * max_new))
    assert checked > 0


@pytest.mark.parametrize("layers,E,n_decode", [(24, 1024, 16), (32, 2560, 4)])
def test_full_depth_real_widths(pkg, make_model, layers, E, n_decode):
    """RWKV-4 430M (24 x 1024) and 3B (32 x 2560) at full depth: decode tokens and a 16-token tensor-core chunk."""
    path = make_model(layers, E)
    toks = token_stream(16, seed=layers)
    ref, ref_state = oracle_run(path, toks)
    eng = pkg.Engine(path)
    got = np.stack([eng.forward([t])[0] for t in toks[:n_decode]])
    eng.close()
    dw, dn = check_rows(got, ref[:n_decode], "%d x %d decode" % (layers, E))
    eng = pkg.Engine(path, max_gpt=len(toks))
    chunk = eng.forward(toks, mode=1)
    se = state_err(eng.state_download(), ref_state)
    eng.close()
    cw, cn = check_rows(chunk, ref, "%d x %d chunk" % (layers, E))
    print("%d x %d vs oracle: decode worst logits rel err %.3g (%d tokens, argmax checked on %d), tensor-core chunk %.3g "
          "(%d tokens, argmax checked on %d), chunk state %.3g" % (layers, E, dw, n_decode, dn, cw, len(toks), cn, se))
    assert se < REL_TOL
