"""Stop strings without a GPU: the byte automaton of csrc/stopmatch.h (compiled with g++) against a naive host search
that follows the rule of include/rwkv_b200.h, the binding's declarations and struct layout, and the Python argument
handling of stop sets."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from util import ROOT, compile_cpp


@pytest.fixture(scope="module")
def walker(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("stopm") / "stopmatch_test")
    return compile_cpp(os.path.join(ROOT, "tests", "helpers", "stopmatch_test.cpp"), out)


def run(exe, strings, chunks, start=0, table=False):
    """(states, table rows [(hit, next[256])] or None, [(hit, state, tail)] per chunk) from the helper."""
    hx = lambda b: b.hex() if b else "-"
    text = " ".join([str(len(strings))] + [hx(s) for s in strings] + [str(int(table)), str(start), str(len(chunks))] +
                    [hx(c) for c in chunks])
    r = subprocess.run([exe], input=text, capture_output=True, text=True, check=True)
    lines = r.stdout.split("\n")
    states = int(lines[0])
    rows = None
    k = 1
    if table:
        rows = []
        for line in lines[1:1 + states]:
            v = [int(x) for x in line.split()]
            rows.append((v[0], v[1:]))
        k = 1 + states
    walks = [tuple(int(x) for x in line.split()) for line in lines[k:k + len(chunks)]]
    return states, rows, walks


def naive_table(strings, pre):
    """Per state its hit (1 + the lowest index of a string that is a suffix of it) and the state of each byte."""
    index = {p: q for q, p in enumerate(pre)}
    out = []
    for p in pre:
        ends = [k for k, s in enumerate(strings) if p.endswith(s)]
        nxt = []
        for c in range(256):
            t = p + bytes([c])
            nxt.append(next(index[t[k:]] for k in range(len(t) + 1) if t[k:] in index))
        out.append((ends[0] + 1 if ends else 0, nxt))
    return out


def check(pkg, exe, strings, chunks, start=0, table=True):
    E = pkg.engine
    pre = E.stop_prefixes(strings)
    states, rows, walks = run(exe, strings, chunks, start, table)
    assert states == len(pre)
    if table:
        assert rows == naive_table(strings, pre)
    q = start
    for c, (hit, state, tail) in zip(chunks, walks):
        j, h, t, q = E.stop_match(strings, [c], q)
        assert (hit, state, tail) == ((h + 1, q, t) if j is not None else (0, q, 0)), (strings, c)


FIXED = [
    [b"aaa", b"aa"],
    [b"abab", b"bab"],
    [b"ab", b"abc"],          # one a prefix of the other
    [b"abc", b"bc", b"c"],    # suffixes
    [b"xy", b"xy", b"y"],     # duplicates: the lowest index wins
    [b"\x00\xff", b"\xff\x00", b"\x00"],
    [b"\n\nUser:", b"</answer>", b"###"],
]


@pytest.mark.parametrize("strings", FIXED, ids=lambda s: "_".join(x.hex() for x in s))
def test_fixed_sets(pkg, walker, strings):
    rng = np.random.default_rng(7)
    alphabet = sorted(set(b"".join(strings)))
    data = bytes(rng.choice(alphabet, size=400).astype(np.uint8))
    cuts = sorted(rng.choice(np.arange(1, len(data)), size=120, replace=False))
    chunks = [data[a:b] for a, b in zip([0] + cuts, cuts + [len(data)])] + [b""]
    check(pkg, walker, strings, chunks)
    check(pkg, walker, strings, [bytes([x]) for x in data[:200]])  # every byte its own step


def test_overlap_rules(pkg, walker):
    """The earliest end byte wins, then the lowest index; tail counts the bytes after it."""
    _, _, w = run(walker, [b"aaa", b"aa"], [b"aaaa"])
    assert w[0][0] == 2 and w[0][2] == 2  # "aa" ends at byte 1
    _, _, w = run(walker, [b"bab", b"abab"], [b"xabab"])
    assert w[0][0] == 1 and w[0][2] == 0  # both end at the last byte: the lower index
    _, _, w = run(walker, [b"User:"], [b"\n\nUs", b"er:\n"])
    assert w[0][0] == 0 and w[1][0] == 1 and w[1][2] == 1


@pytest.mark.parametrize("seed", range(12))
def test_random_sets(pkg, walker, seed):
    rng = np.random.default_rng(100 + seed)
    alphabet = [0, 0xFF, 97, 98] if seed % 2 else list(range(256))
    n = int(rng.integers(1, 7))
    strings = [bytes(rng.choice(alphabet, size=int(rng.integers(1, 6))).astype(np.uint8)) for _ in range(n)]
    if seed % 3 == 0:
        strings.append(strings[0])  # a duplicate
    pick = alphabet if len(alphabet) < 256 else sorted(set(b"".join(strings)) | {0, 255})
    chunks = [bytes(rng.choice(pick, size=int(rng.integers(0, 5))).astype(np.uint8)) for _ in range(150)]
    start = int(rng.integers(0, len(pkg.engine.stop_prefixes(strings))))
    check(pkg, walker, strings, chunks, start)


def test_largest_set(pkg, walker):
    """RWKV_B200_MAX_STOP_BYTES bytes in total: 4097 states at most, and matches deep in a long string."""
    rng = np.random.default_rng(5)
    long = bytes(rng.integers(0, 256, size=4000).astype(np.uint8))
    strings = [long] + [bytes(rng.integers(0, 256, size=8).astype(np.uint8)) for _ in range(12)]
    assert sum(len(s) for s in strings) == pkg.engine.MAX_STOP_BYTES
    states, _, walks = run(walker, strings, [long[:1000], long[1000:3999], long[3999:] + b"zz"])
    assert states == len(pkg.engine.stop_prefixes(strings)) and states <= 4097
    assert walks[0][0] == 0 and walks[1][0] == 0 and walks[2] == (1, 4000, 2)
    distinct = [bytes([i]) * 16 for i in range(256)]
    assert run(walker, distinct, [])[0] == 4097


def test_binding_declares_stop_calls(pkg):
    lib = pkg.load_library()
    for n in ("token_bytes_set", "stop_set_add", "stop_set_remove", "generate_streams_stop",
              "generate_streams_speculative_stop", "batcher_submit_stop", "batcher_read_stop"):
        assert "rwkv_b200_" + n in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_handles_are_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.c_ulonglong
    start, data = pkg.engine.stop_set_bytes(["ab"])
    sid = P()
    assert lib.rwkv_b200_stop_set_add(None, 1, start.ctypes.data_as(ctypes.POINTER(P)),
                                      data.ctypes.data_as(ctypes.POINTER(ctypes.c_ubyte)), ctypes.byref(sid)) != 0
    assert b"null model handle" in lib.rwkv_b200_last_error()
    assert lib.rwkv_b200_stop_set_remove(None, 1) != 0
    assert lib.rwkv_b200_batcher_read_stop(None, 1, None, None, None) != 0
    assert b"null batcher handle" in lib.rwkv_b200_last_error()


def test_stop_request_layout(pkg):
    R = pkg.engine.StopRequest
    names = ["set_ids", "start_states", "states_out", "hit_out", "tail_out"]
    assert [f for f, _ in R._fields_] == names
    assert [getattr(R, f).offset for f in names] == [0, 8, 16, 24, 32] and ctypes.sizeof(R) == 40
    text = open(os.path.join(ROOT, "include", "rwkv_b200.h")).read()
    body = re.search(r"typedef struct rwkv_b200_stop_request \{(.*?)\} rwkv_b200_stop_request;", text, re.S).group(1)
    assert re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S)) == names


def test_python_arguments(pkg):
    E = pkg.engine
    start, data = E.stop_set_bytes(["é", b"\x00\xff", "ab"])
    assert list(start) == [0, 2, 4, 6] and bytes(data) == "é".encode() + b"\x00\xffab"
    start, data = E.stop_set_bytes("###")
    assert list(start) == [0, 3] and bytes(data) == b"###"
    with pytest.raises(E.EngineError):
        E.stop_set_bytes([3])
    ids, starts = E.stop_spec(5, 3, "generate_streams")
    assert list(ids) == [5, 5, 5] and list(starts) == [0, 0, 0]
    ids, starts = E.stop_spec([4, (6, 2), None], 3, "generate_streams")
    assert list(ids) == [4, 6, E.NO_STOP_SET] and list(starts) == [0, 2, 0]
    with pytest.raises(E.EngineError, match="2 stop_strings entries for 3 streams"):
        E.stop_spec([1, 2], 3, "generate_streams")
    assert E.stop_prefixes(["ab", "b", "ac"]) == [b"", b"a", b"ab", b"b", b"ac"]
    # a match that starts in the carried text of a start state
    assert E.stop_match(["abc"], [b"c"], state=2) == (0, 0, 0, 3)
