"""The tensor-core pass's launch geometry, restated on the host: how csrc/prefill.cuh cuts a ragged call into passes
(pass_layout), pads a pass (pf_padded) and launches each GEMM of it (pf_gemm: the split-K factor, the token-block
template NB = Tp / 32 and the dynamic shared memory), and whether every such launch fits what the kernels hold.

Every width the loader accepts, every pass size 1..128 and every head row count produce one (ks, NB, K tail, M tail)
per GEMM. A geometry that broke a kernel limit would read past shared memory or drop part of K with no error at the
launch; a geometry the GPU tests never run could hide a bug below every tolerance of the tests that compare the tensor
cores with the decode kernel or with themselves. So this file also fails if tests/test_pass_geometry_gpu.py misses a
reachable (GEMM, ks, NB) cell, a K or M tail at some NB, a head smaller than its pass, or a multi-pass layout shape."""
import os
import re

import pytest

import numerics as nm
import test_pass_geometry_gpu as gpu
from util import PKG_DIR

CSRC = os.path.join(PKG_DIR, "csrc")
WIDTHS = range(16, 5121, 16)  # every n_embed the loader accepts (engine.cu do_load)
SMS = 132                     # pf_gemm splits K until a launch has at least this many CTAs (an H100 SXM's SMs)


def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def flat(text):
    return re.sub(r"\s+", " ", text)


def constant(name, file):
    m = re.search(r"constexpr int (?:\w+ = \d+, )*%s = (\d+)[;,]" % name, source(file))
    assert m, "%s not found in csrc/%s" % (name, file)
    return int(m.group(1))


K = {n: constant(n, "prefill.cuh") for n in ("kPrefillMinTokens", "kPfMaxTokens", "kPfBM", "kPfBK", "kPfStages",
                                             "kPfConsumerWGs")}
K.update({n: constant(n, "common.cuh") for n in ("kSmemLimit", "kVocab")})
BM, BK, STAGES, TMAX = K["kPfBM"], K["kPfBK"], K["kPfStages"], K["kPfMaxTokens"]
ALIGN = 16 * K["kPfConsumerWGs"]          # kPfTokenAlign
THREADS = 128 * K["kPfConsumerWGs"] + 32  # kPfThreads
V = K["kVocab"]
NB_ALL = tuple(range(1, TMAX // ALIGN + 1))
# The GEMMs of a pass (prefill_chunk_body): kind -> (M, K) as functions of n_embed. The att K, V, R and out-proj and the
# ffn R GEMM share one shape; the head's M is the vocabulary.
GEMMS = {"ExE": lambda E: (E, E), "ffn_k": lambda E: (4 * E, E), "ffn_v": lambda E: (E, 4 * E), "head": lambda E: (V, E)}


# -- the restatements -----------------------------------------------------------------------------------------------

def padded(n):
    """pf_padded."""
    return -(-n // ALIGN) * ALIGN


def split_k(M, Kb):
    """pf_gemm's split-K factor of an M x K GEMM."""
    mt, ks = -(-M // BM), 1
    while mt * ks < SMS and ks < 8 and (Kb // (ks * 2)) % BK == 0 and Kb // (ks * 2) >= 4 * BK:
        ks *= 2
    return ks


def smem(Tp):
    """pf_gemm's dynamic shared memory: the stages of one A tile and three B planes, alignment slack, barriers."""
    return STAGES * (BM * BK + 3 * Tp * BK) + 1024 + 128


def launch(kind, E, T):
    """(ks, NB, K tail, M tail) of GEMM `kind` in a pass of T tokens at width E (T = the head rows for the head)."""
    M, Kb = GEMMS[kind](E)
    return split_k(M, Kb), padded(T) // ALIGN, Kb % BK != 0, M % BM != 0


def pass_layout(lens, head, need=None, stream_head=None):
    """pass_layout: per pass a dict of T, desc (slot index = stream, first, last per token), rows (head rows), out_row0
    and H (heads[i]). Tokens are stream-major; stream i owns lens[i] tokens."""
    n = sum(lens)
    passes = []
    stream = pos = ended = 0
    for i in range(-(-n // TMAX)):
        t0 = i * TMAX
        T = min(TMAX, n - t0)
        p = {"T": T, "desc": [], "rows": [], "out_row0": t0 if head == 1 else ended}
        needed = need is None
        for t in range(T):
            if need is not None and need[t0 + t]:
                needed = True
            while pos == lens[stream]:
                stream += 1
                pos = 0
            fin = pos + 1 == lens[stream]
            headed = fin and (stream_head is None or stream_head[stream])
            p["desc"].append((stream, pos == 0 or t == 0, fin or t == T - 1))
            if head == 1 or (head == 2 and headed):
                p["rows"].append(t)
            if headed:
                ended += 1
            pos += 1
        p["H"] = len(p["rows"]) if needed else 0
        passes.append(p)
    return passes


# -- the restatements are the engine's ----------------------------------------------------------------------------------

def test_restated_geometry_is_the_engines():
    pf = flat(source("prefill.cuh"))
    bodies = {
        "pf_gemm split": "const int mt = (M + kPfBM - 1) / kPfBM; int ks = 1; while (mt * ks < 132 && ks < 8 && (K / (ks * 2)) "
                         "% kPfBK == 0 && K / (ks * 2) >= 4 * kPfBK) ks *= 2; g.ksplit = ks;",
        "pf_gemm smem": "const size_t smem = (size_t)kPfStages * (kPfBM * kPfBK + 3 * (size_t)Tp * kPfBK) + 1024 + 128;",
        "pf_gemm NB": "switch (Tp / kPfTokenAlign) { case 1: k_gemm_i8<1><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); break; "
                      "case 2: k_gemm_i8<2><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); break; case 3: k_gemm_i8<3><<<dim3(mt, "
                      "ks), kPfThreads, smem, st>>>(g); break; default: k_gemm_i8<4><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); "
                      "break; }",
        "kPfThreads": "constexpr int kPfThreads = 128 * kPfConsumerWGs + 32;",
        "kPfTokenAlign": "constexpr int kPfTokenAlign = 16 * kPfConsumerWGs;",
        "pf_padded": "inline int pf_padded(int n) { return (n + kPfTokenAlign - 1) / kPfTokenAlign * kPfTokenAlign; }",
        "k_gemm_i8 K range": "const int kper = g.K / g.ksplit, k0 = blockIdx.y * kper, nkt = (kper + kPfBK - 1) / kPfBK;",
        "k_gemm_i8 stage": "b_bytes = 3u * (uint32_t)Tp * kPfBK, stage_bytes = a_bytes + b_bytes; const uint32_t bars = base + "
                           "kPfStages * stage_bytes;",
        "k_gemm_i8 M tail": "if (row < g.M) {",
        "k_pf_embed row": "__shared__ double row[5120];",
        "k_pf_wkv descriptors": "__shared__ uint32_t desc[kPfMaxTokens], snap[kPfMaxTokens];",
        "GEMMs of a pass": "pf_gemm(s, st, p.wk + mo, E, E, s.limbs, (size_t)9 * Tp, 0 * Tp, Tp, Ca))) "
                           "return rc; if ((rc = pf_gemm(s, st, p.wv + mo, E, E, s.limbs, (size_t)9 * Tp, 3 * Tp, Tp, Cb))) "
                           "return rc; if ((rc = pf_gemm(s, st, p.wr + mo, E, E, s.limbs, (size_t)9 * Tp, 6 * Tp, Tp, Cc)))",
        "GEMM out-proj": "pf_gemm(s, st, p.wo + mo, E, E, s.limbs, (size_t)3 * Tp, 0, Tp, Ca)",
        "GEMMs ffn R, K": "pf_gemm(s, st, p.wfr + mo, E, E, s.limbs, (size_t)6 * Tp, 0 * Tp, Tp, Ca))) return rc; if ((rc = "
                          "pf_gemm(s, st, p.wfk + 4 * mo, 4 * E, E, s.limbs, (size_t)6 * Tp, 3 * Tp, Tp, Ck4)))",
        "GEMM ffn V": "pf_gemm(s, st, p.wfv + 4 * mo, E, 4 * E, s.limbs, (size_t)3 * Tp, 0, Tp, Ca)",
        "GEMM head": "const int Hp = pf_padded(H); const unsigned gH = (unsigned)H;",
        "GEMM head launch": "pf_gemm(s, st, p.whead, p.Vr, E, s.limbs, (size_t)3 * Hp, 0, Hp, s.C)",
        "pass_layout": "passes.assign((size_t)(n + kPfMaxTokens - 1) / kPfMaxTokens, PassDesc{}); heads.assign(passes.size(), "
                       "0); int stream = 0, pos = 0; // current stream, index of the next token inside it int ended = 0; // "
                       "streams whose final token lies in an earlier pass for (size_t i = 0; i < passes.size(); ++i) { "
                       "PassDesc &h = passes[i]; const int t0 = (int)i * kPfMaxTokens, T = std::min(kPfMaxTokens, n - t0); "
                       "int H = 0; bool needed = need == nullptr; h.out_row0 = head == 1 ? t0 : ended; for (int t = 0; t < "
                       "T; ++t) { if (need && need[t0 + t]) needed = true; while (pos == (int)lens[stream]) { ++stream; pos = "
                       "0; } const bool fin = pos + 1 == (int)lens[stream]; const bool headed = fin && (!stream_head || "
                       "stream_head[stream]); h.tokens[t] = tokens[t0 + t]; h.desc[t] = (uint32_t)slots[stream] | (pos == 0 "
                       "|| t == 0 ? kDescFirst : 0u) | (fin || t == T - 1 ? kDescLast : 0u); if (head == 1 || (head == 2 && "
                       "headed)) h.rows[H++] = t; if (headed) ++ended; ++pos; } heads[i] = needed ? H : 0; }",
    }
    stale = [what for what, body in bodies.items() if body not in pf]
    assert not stale, "changed in csrc/prefill.cuh: restate them in tests/test_pass_geometry_host.py: %s" % stale
    # the decode-kernel floor of the boundary cases is the engine's default
    assert gpu.PREFILL_MIN == K["kPrefillMinTokens"]


def test_restated_splits():
    """The split-K factors of the issue's table: E x E 2 at 1024 and 5120, 4 from 2048 to 4096; ffn-K 2 from 1024 to
    2048; ffn-V 4 at 768 and 4096, 8 at 1024 and 2048; the head never splits."""
    want = {768: (1, 1, 4), 1024: (2, 2, 8), 2048: (4, 2, 8), 3072: (4, 1, 4), 4096: (4, 1, 4), 5120: (2, 1, 2),
            784: (1, 1, 1), 1040: (1, 1, 1), 5104: (1, 1, 1)}
    for E, (exe, fk, fv) in want.items():
        assert (launch("ExE", E, 1)[0], launch("ffn_k", E, 1)[0], launch("ffn_v", E, 1)[0]) == (exe, fk, fv), E
        assert launch("head", E, 1)[0] == 1
    seen = {kind: sorted({launch(kind, E, 1)[0] for E in WIDTHS}) for kind in GEMMS}
    assert seen == {"ExE": [1, 2, 4], "ffn_k": [1, 2], "ffn_v": [1, 2, 4, 8], "head": [1]}, seen


# -- every launch fits the kernels ----------------------------------------------------------------------------------

def test_every_launch_fits_the_kernels():
    """Every width, every pass size 1..128 and every GEMM of the pass, the head at every head row count."""
    bad, checked = [], 0
    assert THREADS == 32 * (4 * K["kPfConsumerWGs"] + 1), "two consumer warpgroups and one producer warp"
    for T in range(1, TMAX + 1):
        Tp = padded(T)
        nb = Tp // ALIGN
        need = [("Tp a whole number of 16-token blocks per warpgroup", Tp % ALIGN, 0),
                ("Tp <= kPfMaxTokens", max(Tp - TMAX, 0), 0),
                ("NB has an instantiation", 0 if nb in NB_ALL else 1, 0),
                ("B box rows (TMA: at most 256)", max(Tp - 256, 0), 0),
                ("shared memory <= kSmemLimit", max(smem(Tp) - K["kSmemLimit"], 0), 0),
                ("accumulators: 3 planes x NB x 8 registers <= 96", max(3 * nb * 8 - 96, 0), 0)]
        bad += ["T=%d: %s" % (T, what) for what, got, want in need if got != want]
    for E in WIDTHS:
        if E > 5120:
            bad.append("E=%d: k_pf_embed's row holds 5120 doubles" % E)
        for kind, shape in GEMMS.items():
            M, Kb = shape(E)
            ks = split_k(M, Kb)
            mt, kper = -(-M // BM), Kb // ks
            nkt = -(-kper // BK)
            checked += 1
            if ks > 1 and kper % BK:
                bad.append("E=%d %s: ks %d leaves %d bytes, not a whole number of %d-byte tiles" % (E, kind, ks, kper, BK))
            if ks > 1 and kper * ks != Kb:
                bad.append("E=%d %s: ks %d drops %d bytes of K" % (E, kind, ks, Kb - kper * ks))
            if nkt * BK * ks < Kb or (ks > 1 and nkt * BK != kper):
                bad.append("E=%d %s: the K tiles do not cover K exactly once" % (E, kind))
            if mt * BM < M:
                bad.append("E=%d %s: the row tiles miss rows" % (E, kind))
            if Kb % 16:
                bad.append("E=%d %s: K is not a multiple of 16 bytes (a TMA row stride)" % (E, kind))
    # k_pf_wkv reads the descriptors of T <= kPfMaxTokens tokens into its shared arrays
    assert all(p["T"] <= TMAX for lens in gpu.RAGGED.values() for p in pass_layout(lens, 2))
    assert checked == len(WIDTHS) * len(GEMMS)
    assert not bad, "pf_gemm launches a geometry the kernels cannot hold:\n" + "\n".join(bad[:20])


# -- the GPU file covers every reachable cell ---------------------------------------------------------------------------

def reachable():
    """(GEMM kind, ks, NB) of every launch of every width and pass size (the head: every head row count)."""
    return {(kind, launch(kind, E, T)[0], launch(kind, E, T)[1]) for E in WIDTHS for kind in GEMMS for T in range(1, TMAX + 1)}


def gpu_passes():
    """(E, T, H) of every tensor-core pass tests/test_pass_geometry_gpu.py runs."""
    out = []
    for E in gpu.STEP_WIDTHS:
        for c in gpu.cases(E):
            lens = [len(s) for s in c["streams"]]
            if c["kind"] == "boundary" and sum(lens) < gpu.PREFILL_MIN:
                continue
            heads = (2, 1) if c["kind"] == "ragged" else (2,)
            out += [(E, p["T"], p["H"]) for h in heads for p in pass_layout(lens, h)]
    return out


def visited():
    """(cells, (K tail, NB), (M tail, NB), passes whose head is padded to another size) of the GPU file's passes."""
    cells, ktail, mtail, small_head = set(), set(), set(), []
    for E, T, H in gpu_passes():
        for kind in GEMMS:
            if kind == "head" and H == 0:
                continue
            ks, nb, kt, mt = launch(kind, E, H if kind == "head" else T)
            cells.add((kind, ks, nb))
            if kind != "head":
                if kt:
                    ktail.add(nb)
                if mt:
                    mtail.add(nb)
        if H and padded(H) != padded(T):
            small_head.append((E, T, H))
    return cells, ktail, mtail, small_head


def test_gpu_cases_visit_every_reachable_cell():
    want = reachable()
    cells, ktail, mtail, small_head = visited()
    table = {}
    for kind, ks, nb in sorted(want):
        table.setdefault((kind, ks), []).append(nb)
    print("reachable (GEMM, ks): NB = " + "; ".join("%s ks %d: %s" % (k, s, v) for (k, s), v in sorted(table.items())))
    missing = sorted(want - cells)
    assert not missing, "tests/test_pass_geometry_gpu.py runs no pass of (GEMM, ks, NB) %s" % missing
    assert sorted(cells - want) == [], "the GPU file visits cells the restatement calls unreachable"
    assert len(want) == 4 * (3 + 2 + 4 + 1), "every split of the table at every NB"
    assert set(NB_ALL) <= ktail, "a K tail (n_embed % 128 != 0) at NB %s only" % sorted(ktail)
    assert set(NB_ALL) <= mtail, "an M tail (rows % 64 != 0) below the head at NB %s only" % sorted(mtail)
    assert small_head, "no pass whose head is padded to fewer tokens than the pass"
    assert {padded(T) // ALIGN for _, T, _ in small_head} >= {4}, small_head


def test_gpu_decode_steps_and_boundary():
    """Every width runs every S of the step list as one pass of S rows (S = 1 with its pad row), and the replayed
    shapes are shapes the same engine recorded just before (among its last 8 graphs)."""
    for E in gpu.STEP_WIDTHS:
        cs = gpu.cases(E)
        steps = [c for c in cs if c["kind"] == "step"]
        assert [len(c["streams"]) for c in steps] == [max(S, 2) for S in gpu.STEP_ROWS]
        assert {padded(len(c["streams"])) // ALIGN for c in steps} == set(NB_ALL)
        shapes = [len(c["streams"]) for c in steps]
        recorded = list(dict.fromkeys(shapes))[-8:]
        for c in cs:
            assert len(set(c["slots"])) == len(c["slots"]) and max(c["slots"]) < gpu.NSLOTS, c["id"]
            assert all(len(s) == 1 for s in c["streams"]) or c["kind"] in ("ragged", "boundary"), c["id"]
            if c["kind"] == "replay":
                assert len(c["streams"]) in recorded, c["id"]
                twin = [s for s in steps if len(s["streams"]) == len(c["streams"])][0]
                assert c["slots"] != twin["slots"] and c["streams"] != twin["streams"], c["id"]
    b = [sum(len(s) for s in c["streams"]) for c in gpu.cases(gpu.BOUNDARY_E) if c["kind"] == "boundary"]
    assert b == [gpu.PREFILL_MIN - 1, gpu.PREFILL_MIN]


# -- the multi-pass layouts ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("E", sorted(gpu.RAGGED))
def test_ragged_layouts(E):
    """pass_layout on the GPU file's multi-pass calls: a stream that crosses a cut is last in one pass and first in the
    next; every other token is first only at its stream's start and last only at its end; the head rows of head 2 land
    on their stream's logits row, those of head 1 on their token's."""
    lens = gpu.RAGGED[E]
    n = sum(lens)
    owner = [i for i, m in enumerate(lens) for _ in range(m)]
    start = [sum(lens[:i]) for i in range(len(lens))]
    for head in (1, 2):
        ps = pass_layout(lens, head)
        assert len(ps) == -(-n // TMAX) and sum(p["T"] for p in ps) == n
        for i, p in enumerate(ps):
            t0 = i * TMAX
            for t, (s, first, last) in enumerate(p["desc"]):
                g = t0 + t
                assert s == owner[g]
                assert first == (g == start[s] or t == 0), (head, g)
                assert last == (g == start[s] + lens[s] - 1 or t == p["T"] - 1), (head, g)
            for j, t in enumerate(p["rows"]):
                row = p["out_row0"] + j
                if head == 1:
                    assert row == t0 + t
                else:
                    s = p["desc"][t][0]
                    assert t0 + t == start[s] + lens[s] - 1 and row == s, (i, j)
            assert p["H"] == len(p["rows"])
        if head == 2:
            assert sorted(p["out_row0"] + j for p in ps for j in range(p["H"])) == list(range(len(lens)))
    # the shapes the GPU file's comment promises
    cuts = range(TMAX, n, TMAX)
    spans = [{(start[s] + k) // TMAX for k in range(lens[s])} for s in range(len(lens))]
    crossing = [s for s in range(len(lens)) if len(spans[s]) > 1]
    assert len(crossing) >= 3, crossing
    assert any(len(sp) >= 3 for sp in spans), "a stream spans three passes"
    assert any(lens[s] == 2 and start[s] + 1 in cuts for s in range(len(lens))), "one token on each side of a cut"
    assert any(p["H"] == 0 for p in pass_layout(lens, 2)), "a pass that ends no stream"
    assert len(lens) <= gpu.NSLOTS and n <= gpu.MAX_GPT


def test_layout_with_need_and_stream_heads():
    """The head-row rules the GPU file reaches through score_streams (need) and the batcher (stream_head)."""
    lens = (3, 200, 5)
    need = [0] * 208
    need[1] = 1
    ps = pass_layout(lens, 1, need=need)
    assert [p["H"] for p in ps] == [128, 0]
    ps = pass_layout(lens, 2, stream_head=[1, 0, 1])
    assert [(p["out_row0"], p["rows"]) for p in ps] == [(0, [2]), (1, [207 - 128])]
    # the head's rows are the vocabulary the restatement of the GPU file uses
    assert nm.V == V
