"""Prefix state cache without a GPU: the index of csrc/prefix_index.h (compiled with g++) against a Python restatement of
the policy in include/rwkv_b200.h, the binding's declarations and struct layout, and the Python-side argument errors."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from util import ROOT, compile_cpp


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("prefix") / "prefix_index_test")
    return compile_cpp(os.path.join(ROOT, "tests", "helpers", "prefix_index_test.cpp"), out)


def toks(t):
    return "%d %s" % (len(t), " ".join(str(x) for x in t))


def run(exe, cmds):
    """The output lines of the helper for a list of command lines."""
    r = subprocess.run([exe], input="\n".join(cmds) + "\n", capture_output=True, text=True, check=True)
    return [[int(x) for x in line.split()] for line in r.stdout.strip().split("\n") if line]


class Model:
    """The policy of include/rwkv_b200.h, restated naively: every scan is over all entries."""

    def __init__(self, capacity):
        self.e = [None] * capacity  # None, or [binding, key tuple, used, pinned]
        self.clock = 0
        self.st = dict(live=0, lookups=0, hit_tokens=0, prefilled_tokens=0, snapshots=0, skipped=0, evictions=0)

    def find(self, b, key):
        key = tuple(key)
        for i, x in enumerate(self.e):
            if x and x[0] == b and x[1] == key:
                return i
        return -1

    def touch(self, i):
        self.clock += 1
        self.e[i][2] = self.clock

    def lookup(self, b, limit, t):
        self.st["lookups"] += 1
        for n in range(limit, 0, -1):
            i = self.find(b, t[:n])
            if i >= 0:
                self.touch(i)
                self.st["hit_tokens"] += n
                return [n, i]
        return [0, -1]

    def extended(self, i):
        b, key = self.e[i][0], self.e[i][1]
        return any(y and j != i and y[0] == b and len(y[1]) > len(key) and y[1][:len(key)] == key
                   for j, y in enumerate(self.e))

    def take(self, b, t):
        i = self.find(b, t)
        if i >= 0:
            self.touch(i)
            self.e[i][3] = True
            return [i, 0]
        free = [j for j, x in enumerate(self.e) if x is None]
        if free:
            i = free[0]
        else:
            cands = [j for j, x in enumerate(self.e) if not x[3] and not self.extended(j)]
            if not cands:
                self.st["skipped"] += 1
                return [-1, 0]
            i = min(cands, key=lambda j: self.e[j][2])
            self.e[i] = None
            self.st["live"] -= 1
            self.st["evictions"] += 1
        self.e[i] = [b, tuple(t), 0, True]
        self.st["live"] += 1
        self.st["snapshots"] += 1
        self.touch(i)
        return [i, 1]

    def unpin(self):
        for x in self.e:
            if x:
                x[3] = False

    def clear(self):
        self.e = [None] * len(self.e)
        self.st["live"] = 0

    def stats(self):
        return [self.st[k] for k in ("live", "lookups", "hit_tokens", "prefilled_tokens", "snapshots", "skipped",
                                     "evictions")]


def test_longest_prefix(driver):
    out = run(driver, ["new 8 18446744073709551615",
                       "take 7 %s" % toks([1, 2]), "take 7 %s" % toks([1, 2, 3, 4]), "unpin",
                       "lookup 7 6 %s" % toks([1, 2, 3, 4, 5, 6]),   # longest: 4 tokens
                       "lookup 7 3 %s" % toks([1, 2, 3, 4, 5, 6]),   # limit 3: the 2-token entry
                       "lookup 7 3 %s" % toks([1, 2, 3]),
                       "lookup 7 1 %s" % toks([1, 2, 3]),
                       "lookup 7 5 %s" % toks([1, 3, 2, 4, 5]),
                       "stats"])
    assert out[0] == [0, 1] and out[1] == [1, 1]
    assert out[2] == [4, 1] and out[3] == [2, 0]
    assert out[4] == [2, 0] and out[5] == [0, -1] and out[6] == [0, -1]
    assert out[7] == [2, 5, 8, 0, 2, 0, 0]


def test_forced_collisions_match_exactly(driver):
    """With a hash mask of 0 every key shares one bucket: matches are decided by the tokens alone."""
    rng = np.random.default_rng(3)
    keys = [list(rng.integers(0, 4, size=int(rng.integers(1, 6)))) for _ in range(30)]
    cmds = ["new 64 0"] + ["take 0 %s" % toks(k) for k in keys] + ["unpin"]
    probes = [list(rng.integers(0, 4, size=8)) for _ in range(40)]
    cmds += ["lookup 0 8 %s" % toks(p) for p in probes] + ["find 0 %s" % toks(k) for k in keys]
    out = run(driver, cmds)
    m = Model(64)
    want = [m.take(0, [int(x) for x in k]) for k in keys]
    m.unpin()
    want += [m.lookup(0, 8, [int(x) for x in p]) for p in probes]
    want += [[m.find(0, [int(x) for x in k])] for k in keys]
    assert out == want


def test_leaves_first_lru(driver):
    """The least recently used leaf goes first; an entry extended by a live entry stays until its extension is gone."""
    a, ab, abc, x = [5], [5, 6], [5, 6, 7], [9]
    out = run(driver, ["new 3 18446744073709551615",
                       "take 0 %s" % toks(a), "take 0 %s" % toks(ab), "take 0 %s" % toks(x), "unpin",
                       "lookup 0 1 %s" % toks(x),   # x is now the most recent
                       "take 0 %s" % toks(abc),     # a is oldest but extended by ab: ab (a leaf) is evicted
                       "unpin",
                       "find 0 %s" % toks(ab), "find 0 %s" % toks(a),
                       "take 0 %s" % toks([1]),      # a is extended by abc; x is the LRU leaf
                       "unpin", "find 0 %s" % toks(x), "stats"])
    assert out[:3] == [[0, 1], [1, 1], [2, 1]]
    assert out[3] == [1, 2]
    assert out[4] == [1, 1]                          # abc took ab's entry
    assert out[5] == [-1] and out[6] == [0]
    assert out[7] == [2, 1] and out[8] == [-1]
    assert out[9] == [3, 1, 1, 0, 5, 0, 2]


def test_pinning_and_skipped_snapshots(driver):
    """Entries taken for the layout being built are never evicted by it; with none left a snapshot is skipped."""
    out = run(driver, ["new 2 18446744073709551615",
                       "take 0 %s" % toks([1]), "take 0 %s" % toks([2]),
                       "take 0 %s" % toks([3]),      # both pinned: skipped
                       "take 0 %s" % toks([1]),      # an existing key: a use, not a snapshot
                       "unpin",
                       "take 0 %s" % toks([3]),      # [2] is the LRU now
                       "stats"])
    assert out[0] == [0, 1] and out[1] == [1, 1]
    assert out[2] == [-1, 0] and out[3] == [0, 0]
    assert out[4] == [1, 1]
    assert out[5] == [2, 0, 0, 0, 3, 1, 1]


def test_bindings_separate_keys_and_clear(driver):
    out = run(driver, ["new 4 18446744073709551615",
                       "take 18446744073709551615 %s" % toks([1, 2]), "take 3 %s" % toks([1, 2]), "unpin",
                       "lookup 3 2 %s" % toks([1, 2]), "lookup 18446744073709551615 2 %s" % toks([1, 2]),
                       "lookup 4 2 %s" % toks([1, 2]),
                       "clear", "lookup 3 2 %s" % toks([1, 2]), "find 3 %s" % toks([1, 2]),
                       "take 3 %s" % toks([1]), "stats"])
    assert out[0] == [0, 1] and out[1] == [1, 1]
    assert out[2] == [2, 1] and out[3] == [2, 0] and out[4] == [0, -1]
    assert out[5] == [0, -1] and out[6] == [-1]
    assert out[7] == [0, 1]
    assert out[8] == [1, 4, 4, 0, 3, 0, 0]


@pytest.mark.parametrize("seed", range(6))
def test_random_policy(driver, seed):
    """Random lookups, snapshot layouts and clears against the restatement, with and without forced collisions."""
    rng = np.random.default_rng(50 + seed)
    cap = int(rng.integers(1, 7))
    mask = 0 if seed % 2 else (1 << 64) - 1
    m = Model(cap)
    cmds, want = ["new %d %d" % (cap, mask)], []
    base = [int(x) for x in rng.integers(0, 3, size=12)]
    for _ in range(120):
        b = int(rng.integers(0, 2))
        t = base[:int(rng.integers(0, 6))] + [int(x) for x in rng.integers(0, 3, size=int(rng.integers(1, 6)))]
        op = rng.random()
        if op < 0.35:
            limit = int(rng.integers(0, len(t) + 1))
            cmds.append("lookup %d %d %s" % (b, limit, toks(t)))
            want.append(m.lookup(b, limit, t))
        elif op < 0.9:
            for _ in range(int(rng.integers(1, 4))):  # one layout's snapshots, then unpin
                n = int(rng.integers(1, len(t) + 1))
                cmds.append("take %d %s" % (b, toks(t[:n])))
                want.append(m.take(b, t[:n]))
            cmds.append("unpin")
            m.unpin()
        elif op < 0.95:
            cmds.append("clear")
            m.clear()
        else:
            cmds.append("find %d %s" % (b, toks(t)))
            want.append([m.find(b, t)])
    cmds.append("stats")
    want.append(m.stats())
    assert run(driver, cmds) == want


def test_binding_declares_prefix_calls(pkg):
    lib = pkg.load_library()
    for n in ("prefix_cache_open", "prefix_cache_close", "prefix_forward", "prefix_insert", "prefix_download",
              "prefix_clear", "prefix_stats", "batcher_submit_prefix", "batcher_read_prefix"):
        assert "rwkv_b200_" + n in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_prefix_stats_layout(pkg):
    S = pkg.engine.PrefixStats
    names = ["live", "lookups", "hit_tokens", "prefilled_tokens", "snapshots", "skipped", "evictions"]
    assert [f for f, _ in S._fields_] == names and ctypes.sizeof(S) == 56
    text = open(os.path.join(ROOT, "include", "rwkv_b200.h")).read()
    body = re.search(r"struct rwkv_b200_prefix_stats \{.*?\*/(.*?)\};", text, re.S).group(1)
    assert re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S)) == names
    assert "#define RWKV_B200_PREFIX_NOT_CACHED %d" % pkg.engine.PREFIX_NOT_CACHED in text


def test_null_handles_are_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.c_ulonglong
    h = ctypes.c_void_p()
    assert lib.rwkv_b200_prefix_cache_open(None, 4, 64, ctypes.byref(h)) != 0
    assert b"null model handle" in lib.rwkv_b200_last_error()
    t = (P * 2)(1, 2)
    for rc in (lib.rwkv_b200_prefix_insert(None, 0, t, 2), lib.rwkv_b200_prefix_download(None, t, 2, None, None, None, None),
               lib.rwkv_b200_prefix_clear(None), lib.rwkv_b200_prefix_stats(None, None),
               lib.rwkv_b200_prefix_forward(None, t, 2, t, t, 1, None, None, t)):
        assert rc != 0
        assert b"null prefix cache handle" in lib.rwkv_b200_last_error()
    assert lib.rwkv_b200_prefix_cache_close(None) == 0
    assert lib.rwkv_b200_batcher_submit_prefix(None, None, None, 0, 0, None, None, None) != 0
    assert lib.rwkv_b200_batcher_read_prefix(None, 1, None) != 0
    assert b"null batcher handle" in lib.rwkv_b200_last_error()


def test_python_arguments(pkg):
    """A closed cache refuses every call in Python, before the library sees it."""
    E = pkg.engine
    c = E.PrefixCache.__new__(E.PrefixCache)
    c.engine, c.lib, c.h = None, pkg.load_library(), None
    for call in (lambda: c.forward([(0, [1, 2])]), lambda: c.insert(0, [1]), lambda: c.download([1]), c.stats, c.clear):
        with pytest.raises(E.EngineError, match="prefix cache is closed"):
            call()
    c.close()
    with c as same:
        assert same is c
