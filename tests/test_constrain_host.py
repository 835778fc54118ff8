"""Constrained generation without a GPU: the regex compiler against Python's re, token_bytes against this repository's
tokenizer, the token automaton against the tokenizer and re, and the binding of the three new C entry points."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from util import INCLUDE, ROOT, VOCAB_DIR, compile_cpp

PATTERNS = [
    r"-?\d+(\.\d+)?",                                   # a number with an optional fraction
    r"\d{4}-\d{2}-\d{2}",                               # a date
    r"positive|negative|neutral",                       # one of a few labels
    r'\{"name": "[a-z]{1,12}", "age": \d{1,3}\}',       # JSON with fixed keys
    r"(a(b|c)*d){2,3}",                                 # nested quantifiers
    r'"[^"\\\n]*"',                                     # a negated class
    r"(?:[A-Z][a-z]+ ?){1,3}",
    r"[\w.-]+@[\w-]+\.(com|org)",
    r"(ab|a)*b?|x{2,}",
    r"\x41[\x00-\x1f]?.\s\S\W\D[]a-]+[^]x]",
    r"(x|y){0,2}z*\?\*\+\(\)\[\]\{\}\|\.\\",
]
TOKEN_PATTERNS = PATTERNS[:6]


@pytest.fixture(scope="module")
def C(pkg):
    return pkg.constrain


@pytest.fixture(scope="module")
def tbytes(C):
    return C.token_bytes()


def random_strings(dfa, pattern, rng, n):
    """Strings biased towards near-matches: random walks of the DFA stopped in accepting states, then each mutated by
    an inserted, deleted or replaced byte; plus short random strings over the pattern's own bytes."""
    alphabet = sorted(set(pattern.encode())) + [0, 10, 32, 48, 97, 200]
    dist = np.where(dfa.accept, 0, 10 ** 6)  # bytes to the nearest accepting state
    for _ in range(dfa.n_states):
        nxt = np.where(dfa.trans >= 0, dist[np.maximum(dfa.trans, 0)] + 1, 10 ** 6).min(axis=1)
        dist = np.minimum(dist, nxt)
    out = []
    for _ in range(n):
        q, s, free = 0, bytearray(), int(rng.integers(0, 30))
        while True:  # free steps, then the shortest way to an accepting state
            nxt = np.nonzero(dfa.trans[q] >= 0)[0]
            if dfa.accept[q] and (len(s) >= free or rng.random() < 0.1 or not len(nxt)):
                break
            if len(s) >= free:
                nxt = [b for b in nxt if dist[dfa.trans[q, b]] < dist[q]]
            b = int(rng.choice(nxt))
            s.append(b)
            q = int(dfa.trans[q, b])
        out.append(bytes(s))
        m = bytearray(s)
        k = int(rng.integers(0, 3))
        at = int(rng.integers(0, len(m) + 1))
        b = int(rng.choice(alphabet))
        if k == 0:
            m.insert(at, b)
        elif k == 1 and m:
            del m[min(at, len(m) - 1)]
        elif m:
            m[min(at, len(m) - 1)] = b
        out.append(bytes(m))
        out.append(bytes(int(x) for x in rng.choice(alphabet, int(rng.integers(0, 8)))))
    return out


@pytest.mark.parametrize("pattern", PATTERNS)
def test_compile_regex_equals_fullmatch(C, pattern):
    dfa = C.compile_regex(pattern)
    rx = re.compile(pattern.encode())
    rng = np.random.default_rng(len(pattern))
    strings = random_strings(dfa, pattern, rng, 1500)
    hits = 0
    for s in strings:
        want = rx.fullmatch(s) is not None
        assert dfa.match(s) == want, (pattern, s)
        hits += want
    assert 0.15 * len(strings) < hits < 0.9 * len(strings)  # both sides are exercised


def test_compile_regex_is_minimal_and_live(C):
    dfa = C.compile_regex(r"(a|b)*abb")
    assert dfa.n_states == 4  # the textbook minimal DFA
    dfa = C.compile_regex(r"ab|ac|ad")
    assert dfa.n_states == 3
    assert all((dfa.trans[q] >= 0).any() or dfa.accept[q] for q in range(dfa.n_states))


@pytest.mark.parametrize("pattern", [r"^a", r"a$", r"\bfoo", r"(a)\1", r"(?=a)b", r"(?!a)b", r"(?<=a)b", r"(?P<n>a)",
                                     r"a*?", r"a+?", r"a??", r"a{2", r"a{x}", r"a{3,2}", r"\Aa", r"a\Z", r"a**",
                                     r"(a", r"a)", r"[a", r"[z-a]", r"[\d-z]", r"\q", r"\x4", "café", r"*a",
                                     r"a{1001}", r"\1", r"[^\x00-\xff]"])
def test_unsupported_syntax_raises(C, pattern):
    with pytest.raises(C.RegexError):
        C.compile_regex(pattern)


# -- token bytes and the token automaton -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tok_tools(tmp_path_factory):
    d = tmp_path_factory.mktemp("tokc")
    dec = compile_cpp(os.path.join(ROOT, "tests", "helpers", "tok_decode.cpp"), str(d / "tok_decode"))
    cli = compile_cpp(os.path.join(ROOT, "tests", "helpers", "tok_cli.cpp"), str(d / "tok_cli"))
    return dec, cli


def run_tool(exe, lines):
    r = subprocess.run([exe, VOCAB_DIR + "/vocab.json", VOCAB_DIR + "/merges.txt"], input="\n".join(lines) + "\n",
                       capture_output=True, text=True, check=True)
    return r.stdout.split("\n")[:len(lines)]


def encode(cli, strings):
    rows = run_tool(cli, [s.hex() for s in strings])
    return [[int(x) for x in row.split(" | ")[0].split()] if row.split(" | ")[0].strip() else [] for row in rows]


def test_token_bytes_equal_the_tokenizer_decode(tbytes, tok_tools):
    assert len(tbytes) == 50277
    got = run_tool(tok_tools[0], [str(i) for i in range(50277)])
    bad = [i for i in range(50277) if bytes.fromhex(got[i]) != tbytes[i]]
    assert not bad, bad[:10]
    assert tbytes[0] == b"<|endoftext|>" and tbytes[1] == b"<|padding|>"
    assert all(set(tbytes[i]) == {0} for i in range(50254, 50277))  # quirk Q3: raw spaces decode to NUL bytes


@pytest.mark.parametrize("pattern", TOKEN_PATTERNS)
def test_token_automaton_against_tokenizer_and_re(C, tbytes, tok_tools, pattern):
    dfa = C.compile_regex(pattern)
    ta = C.token_automaton(dfa, tbytes, eos=0)
    rx = re.compile(pattern.encode())
    rng = np.random.default_rng(7 + len(pattern))
    # the CSR form: tokens ascending inside each state, targets in range; "no edges" is exactly the sink
    st = ta.edge_start.astype(np.int64)
    assert st[0] == 0 and np.all(np.diff(st) >= 0) and st[-1] == len(ta.edge_tokens)
    for q in range(ta.n_states):
        t, x = ta.edges(q)
        assert np.all(np.diff(t.astype(np.int64)) > 0) and np.all(x < ta.n_states)
        assert ta.complete(q) == (q == ta.sink)
    # every tokenisation the tokenizer gives a matching string walks to the sink with eos appended
    # (a string the tokenizer cannot spell, e.g. bytes that are not UTF-8, gets id 0 for its unknown symbols: skipped)
    matching = [s for s in random_strings(dfa, pattern, rng, 150) if rx.fullmatch(s)][:120]
    spelled = [(s, ids) for s, ids in zip(matching, encode(tok_tools[1], matching)) if 0 not in ids]
    assert len(spelled) >= 30
    for s, ids in spelled:
        assert b"".join(tbytes[i] for i in ids) == s
        assert ta.walk(ids + [0]) == ta.sink, (s, ids)
    # random token sequences: accepted exactly when re.fullmatch holds on their bytes
    pool = [t for t in range(2, 50277) if 0 < len(tbytes[t]) <= 3 and set(tbytes[t]) <= set(pattern.encode()) | set(b"0123456789abcdez")]
    accepted = 0
    for i in range(600):
        if i % 2:  # a random walk of the automaton, sometimes cut short or perturbed
            seq, q = [], 0
            while not ta.complete(q) and len(seq) < 30:
                t, x = ta.edges(q)
                k = int(rng.integers(0, len(t)))
                if int(t[k]) == 0:
                    break
                seq.append(int(t[k]))
                q = int(x[k])
            if seq and rng.random() < 0.3:
                seq[int(rng.integers(0, len(seq)))] = int(rng.choice(pool))
        else:
            seq = [int(x) for x in rng.choice(pool, int(rng.integers(1, 8)))]
        want = rx.fullmatch(b"".join(tbytes[t] for t in seq)) is not None
        assert (ta.walk(seq + [0]) == ta.sink) == want, (seq, want)
        accepted += want
    assert 20 < accepted < 580


def test_token_automaton_without_eos_and_pruning(C, tbytes):
    ta = C.token_automaton(C.compile_regex(r"yes|no"), tbytes, eos=None)
    yes = [i for i in range(2, 50277) if tbytes[i] == b"yes"][0]
    q = ta.walk([yes])
    assert q is not None and ta.complete(q)
    assert ta.sink is None and 0 not in ta.edge_tokens
    # a state from which no token path completes is pruned with the edges into it: in this small vocabulary no token
    # holds a "d", so after "a" nothing completes "ad"
    small = [b"<|endoftext|>", b"<|padding|>", b"a", b"c", b"ab", b""]
    ta = C.token_automaton(C.compile_regex(r"ad|c|ab"), small, eos=0)
    assert ta.walk([2]) is None and ta.walk([3, 0]) == ta.sink and ta.walk([4, 0]) == ta.sink
    assert [int(t) for t in ta.edges(0)[0]] == [3, 4]
    for q in range(ta.n_states):
        assert not ta.complete(q) or q == ta.sink
    with pytest.raises(ValueError):
        C.token_automaton(C.compile_regex(r"ad"), small, eos=0)
    allow = C.allow_all()
    assert allow.n_states == 1 and allow.walk(range(50277)) == 0


# -- binding ------------------------------------------------------------------------------------------------------------

def test_binding_declares_the_constrained_entry_points(pkg):
    lib = pkg.load_library()
    for name in ("rwkv_b200_constraint_add", "rwkv_b200_constraint_remove", "rwkv_b200_generate_streams_constrained"):
        assert name in lib._declared
    assert lib.rwkv_b200_abi_version() == 2
    with open(os.path.join(INCLUDE, "rwkv_b200.h")) as f:
        hdr = f.read()
    assert int(re.search(r"#define RWKV_B200_NO_CONSTRAINT\s+(0x[0-9A-F]+)ULL", hdr).group(1), 16) == pkg.engine.NO_CONSTRAINT
    assert int(re.search(r"#define RWKV_B200_MAX_CONSTRAINT_STATES\s+(\d+)", hdr).group(1)) == pkg.engine.MAX_CONSTRAINT_STATES


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    start, toks, nxt = np.array([0, 1], np.uint64), np.array([5], np.uint64), np.array([0], np.uint64)
    cid = ctypes.c_ulonglong()
    rc = lib.rwkv_b200_constraint_add(None, 1, start.ctypes.data_as(P), toks.ctypes.data_as(P), nxt.ctypes.data_as(P),
                                      ctypes.byref(cid))
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
    assert lib.rwkv_b200_constraint_remove(None, 1) != 0 and b"null model handle" in lib.rwkv_b200_last_error()
    slots, first = np.array([0], np.uint64), np.array([4118], np.uint64)
    out, lens, ids = np.zeros(4, np.uint64), np.zeros(1, np.uint64), np.array([1], np.uint64)
    rc = lib.rwkv_b200_generate_streams_constrained(None, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 4, None, None,
                                                    0, None, None, 0, None, None, out.ctypes.data_as(P),
                                                    lens.ctypes.data_as(P), 0, 0, None, None, None, None,
                                                    ids.ctypes.data_as(P), None, None)
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
