"""Host-side builders for constrained generation (include/rwkv_b200.h, rwkv_b200_generate_streams_constrained).

  token_bytes()                          the bytes of every token id, as GPT2Tokenizer::decode({id}) gives them
  compile_regex(pattern) -> ByteDFA      a minimal DFA over bytes for a small regular-expression subset
  token_automaton(dfa, token_bytes, eos=0) -> TokenAutomaton
                                         the automaton over token ids that Engine.add_constraint uploads

compile_regex matches the whole byte string (re.fullmatch semantics) and supports:
  ASCII literals, and \\xHH for any byte;
  .            any byte except \\n;
  [...]        sets with ranges and a leading ^ for the complement (a leading ] or a - at either end is literal);
  \\d \\w \\s \\D \\W \\S   with Python's bytes-pattern meanings ([0-9], [a-zA-Z0-9_], [ \\t\\n\\r\\f\\v] and complements);
  \\n \\t \\r \\f \\v \\a, and a backslash before any other ASCII punctuation or space for that character;
  ( ), (?: ), |, and the greedy quantifiers * + ? {m} {m,} {m,n} (counts up to 1000).
Anything else raises RegexError: anchors (^ $ \\b \\A \\Z), back-references, lookaround and other (? groups, lazy or
possessive quantifiers, a { that does not start a quantifier, and non-ASCII characters in a str pattern. The NFA is
Thompson's construction, made deterministic by subset construction over byte classes, then minimised (Moore's
partition refinement); states from which no match is reachable are dropped, so every DFA state is live.
"""
import json
import os
import re

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
VOCAB_JSON = os.path.join(os.path.dirname(_PKG), "include", "rwkv", "tokenizer", "vocab", "vocab.json")
VOCAB = 50277
SPECIAL = (0, 1)  # <|endoftext|> and <|padding|>: never reached through bytes
_ALL = (1 << 256) - 1
_MAX_REPEAT = 1000


class RegexError(ValueError):
    pass


# -- token bytes --------------------------------------------------------------------------------------------------------

def _byte_decoder():
    """GPT-2 bytes_to_unicode, inverted: code point -> byte."""
    dec, nxt = {}, 256
    for b in range(256):
        keep = 33 <= b <= 126 or 161 <= b <= 172 or 174 <= b <= 255
        dec[chr(b if keep else nxt)] = b
        nxt += 0 if keep else 1
    return dec


def token_bytes(vocab_json=VOCAB_JSON):
    """The bytes of every token id 0..50276, equal to GPT2Tokenizer::decode({id}) of include/rwkv/tokenizer/tokenizer.h:
    each code point of the token's vocabulary string maps back through bytes_to_unicode, and a code point outside that
    table decodes to a NUL byte (its quirk Q3; the 23 raw-space tokens 50254..50276 are such runs of NUL bytes). An id
    that the vocabulary lacks has no bytes; for an id listed twice the first entry counts."""
    with open(vocab_json, encoding="utf-8") as f:
        pairs = json.load(f, object_pairs_hook=list)
    dec = _byte_decoder()
    out = [None] * VOCAB
    for sym, i in pairs:
        if 0 <= i < VOCAB and out[i] is None:
            out[i] = bytes(dec.get(ch, 0) for ch in sym)
    return [b if b is not None else b"" for b in out]


# -- regular expression -> byte DFA -------------------------------------------------------------------------------------

_CLASSES = {
    "d": sum(1 << b for b in range(48, 58)),
    "w": sum(1 << b for b in list(range(48, 58)) + list(range(65, 91)) + list(range(97, 123)) + [95]),
    "s": sum(1 << b for b in b" \t\n\r\f\v"),
}
_CONTROL = {"n": 10, "t": 9, "r": 13, "f": 12, "v": 11, "a": 7}


class _Parser:
    """Recursive descent into nodes ('set', mask), ('cat', [nodes]), ('alt', [nodes]), ('rep', node, m, n | None)."""

    def __init__(self, p):
        self.p, self.i = p, 0

    def peek(self):
        return self.p[self.i] if self.i < len(self.p) else None

    def err(self, msg):
        return RegexError("%s at position %d of %r" % (msg, self.i, self.p))

    def parse(self):
        node = self.alt()
        if self.i != len(self.p):
            raise self.err("unbalanced ')'")
        return node

    def alt(self):
        items = [self.cat()]
        while self.peek() == ord("|"):
            self.i += 1
            items.append(self.cat())
        return ("alt", items) if len(items) > 1 else items[0]

    def cat(self):
        items = []
        while self.peek() is not None and self.peek() not in b"|)":
            items.append(self.repeat())
        return ("cat", items)

    def repeat(self):
        atom = self.atom()
        if self.peek() is None or self.peek() not in b"*+?{":
            return atom
        m, n = self.quantifier()
        if self.peek() is not None and self.peek() in b"*+?{":
            raise self.err("lazy, possessive or repeated quantifiers are not supported")
        return ("rep", atom, m, n)

    def quantifier(self):
        c = chr(self.p[self.i])
        self.i += 1
        if c in "*+?":
            return {"*": (0, None), "+": (1, None), "?": (0, 1)}[c]
        j = self.p.find(b"}", self.i)
        q = re.fullmatch(rb"(\d+)(,(\d*))?", self.p[self.i:j]) if j >= 0 else None
        if not q:
            raise self.err("'{' must start a quantifier {m}, {m,} or {m,n}")
        m = int(q.group(1))
        n = m if q.group(2) is None else (int(q.group(3)) if q.group(3) else None)
        if (n is not None and n < m) or max(m, n or 0) > _MAX_REPEAT:
            raise self.err("repeat counts must satisfy m <= n <= %d" % _MAX_REPEAT)
        self.i = j + 1
        return m, n

    def atom(self):
        c = self.p[self.i]
        if c == ord("("):
            self.i += 1
            if self.p.startswith(b"?:", self.i):
                self.i += 2
            elif self.peek() == ord("?"):
                raise self.err("only (?:...) group extensions are supported")
            node = self.alt()
            if self.peek() != ord(")"):
                raise self.err("missing ')'")
            self.i += 1
            return node
        if c == ord("["):
            return ("set", self.set())
        if c == ord("."):
            self.i += 1
            return ("set", _ALL & ~(1 << 10))
        if c == ord("\\"):
            return ("set", self.escape()[0])
        if c in b"^$":
            raise self.err("anchors are not supported")
        if c in b"*+?{":
            raise self.err("nothing to repeat")
        self.i += 1
        return ("set", 1 << c)

    def escape(self):
        """(mask, byte or None) of the escape at self.i."""
        self.i += 1
        if self.i >= len(self.p):
            raise self.err("trailing backslash")
        ch = chr(self.p[self.i])
        self.i += 1
        if ch == "x":
            h = self.p[self.i:self.i + 2]
            if not re.fullmatch(rb"[0-9a-fA-F]{2}", h):
                raise self.err("\\x needs two hex digits")
            self.i += 2
            return 1 << int(h, 16), int(h, 16)
        if ch.lower() in _CLASSES:
            m = _CLASSES[ch.lower()]
            return (m if ch.islower() else _ALL & ~m), None
        if ch in _CONTROL:
            return 1 << _CONTROL[ch], _CONTROL[ch]
        if ord(ch) < 128 and not ch.isalnum():
            return 1 << ord(ch), ord(ch)
        raise self.err("unsupported escape \\%s" % ch)

    def set(self):
        self.i += 1
        neg = self.peek() == ord("^")
        self.i += neg
        mask, first = 0, True
        while True:
            if self.i >= len(self.p):
                raise self.err("unterminated '['")
            if self.p[self.i] == ord("]") and not first:
                self.i += 1
                break
            first = False
            lo_mask, lo = self.set_item()
            if self.peek() == ord("-") and self.i + 1 < len(self.p) and self.p[self.i + 1] != ord("]"):
                self.i += 1
                _, hi = self.set_item()
                if lo is None or hi is None or hi < lo:
                    raise self.err("bad character range")
                mask |= ((1 << (hi + 1)) - 1) & ~((1 << lo) - 1)
            else:
                mask |= lo_mask
        return _ALL & ~mask if neg else mask

    def set_item(self):
        if self.p[self.i] == ord("\\"):
            return self.escape()
        c = self.p[self.i]
        self.i += 1
        return 1 << c, c


class _NFA:
    """Thompson's construction: per state its epsilon targets and its (byte mask, target) edges."""

    def __init__(self):
        self.eps, self.edges = [], []

    def new(self):
        self.eps.append([])
        self.edges.append([])
        return len(self.eps) - 1

    def build(self, node):
        kind = node[0]
        if kind == "set":
            s, e = self.new(), self.new()
            self.edges[s].append((node[1], e))
            return s, e
        if kind == "cat":
            s = cur = self.new()
            for x in node[1]:
                a, b = self.build(x)
                self.eps[cur].append(a)
                cur = b
            return s, cur
        if kind == "alt":
            s, e = self.new(), self.new()
            for x in node[1]:
                a, b = self.build(x)
                self.eps[s].append(a)
                self.eps[b].append(e)
            return s, e
        _, x, m, n = node
        s = cur = self.new()
        for _ in range(m):
            a, b = self.build(x)
            self.eps[cur].append(a)
            cur = b
        if n is None:
            loop = self.new()
            self.eps[cur].append(loop)
            a, b = self.build(x)
            self.eps[loop].append(a)
            self.eps[b].append(loop)
            return s, loop
        end = self.new()
        for _ in range(n - m):
            self.eps[cur].append(end)
            a, b = self.build(x)
            self.eps[cur].append(a)
            cur = b
        self.eps[cur].append(end)
        return s, end

    def closure(self, states):
        seen, stack = set(states), list(states)
        while stack:
            for t in self.eps[stack.pop()]:
                if t not in seen:
                    seen.add(t)
                    stack.append(t)
        return frozenset(seen)


class ByteDFA:
    """A minimal DFA over bytes: trans[q][b] is the next state or -1 (no match possible any more), accept[q] marks the
    states where the bytes read so far match. The start state is 0; every state can still reach a match."""

    def __init__(self, trans, accept):
        self.trans = np.asarray(trans, np.int32)
        self.accept = np.asarray(accept, bool)

    @property
    def n_states(self):
        return len(self.accept)

    def run(self, data, state=0):
        """The state after `data` from `state`, or -1."""
        for b in data:
            state = int(self.trans[state, b])
            if state < 0:
                return -1
        return state

    def match(self, data):
        q = self.run(data)
        return q >= 0 and bool(self.accept[q])


def compile_regex(pattern):
    """A ByteDFA that accepts exactly the byte strings `pattern` fully matches (re.fullmatch(pattern, s) for a bytes
    pattern). pattern: bytes, or an ASCII str. See the module docstring for the supported subset."""
    if isinstance(pattern, str):
        try:
            pattern = pattern.encode("ascii")
        except UnicodeEncodeError:
            raise RegexError("a str pattern must be ASCII; give bytes or \\xHH escapes for other bytes") from None
    nfa = _NFA()
    start, final = nfa.build(_Parser(bytes(pattern)).parse())
    # byte classes: bytes that every edge mask treats alike
    masks = sorted({m for es in nfa.edges for m, _ in es})
    sig = [tuple((m >> b) & 1 for m in masks) for b in range(256)]
    reps = sorted(set(sig), key=sig.index)
    byte_class = np.array([reps.index(s) for s in sig], np.int64)
    rep_byte = [sig.index(s) for s in reps]
    # subset construction; -1 is the empty set
    d0 = nfa.closure([start])
    index, states, trans = {d0: 0}, [d0], []
    while len(trans) < len(states):
        d = states[len(trans)]
        row = []
        for b in rep_byte:
            tgt = {t for n in d for m, t in nfa.edges[n] if (m >> b) & 1}
            if not tgt:
                row.append(-1)
                continue
            c = nfa.closure(tgt)
            if c not in index:
                index[c] = len(states)
                states.append(c)
            row.append(index[c])
        trans.append(row)
    n, C = len(states), len(rep_byte)
    # Moore minimisation with an explicit dead state n
    T = np.array(trans, np.int64).reshape(n, C)
    T[T < 0] = n
    T = np.vstack([T, np.full((1, C), n, np.int64)])
    acc = np.array([final in d for d in states] + [False])
    block = acc.astype(np.int64)
    nb = len(np.unique(block))
    while True:
        _, block2 = np.unique(np.concatenate([block[:, None], block[T]], axis=1), axis=0, return_inverse=True)
        block2 = block2.reshape(-1)
        nb2 = int(block2.max()) + 1
        block = block2
        if nb2 == nb:
            break
        nb = nb2
    # quotient automaton; drop the states that cannot reach an accepting one (the dead block among them)
    QT = np.zeros((nb, C), np.int64)
    QT[block] = block[T]
    qacc = np.zeros(nb, bool)
    qacc[block[acc]] = True
    live = qacc.copy()
    while True:
        grown = live | live[QT].any(axis=1)
        if (grown == live).all():
            break
        live = grown
    q0 = int(block[0])
    if not live[q0]:
        raise RegexError("the pattern %r matches nothing" % (pattern,))
    # renumber the live states in breadth-first order from the start
    order, pos = [q0], {q0: 0}
    for q in order:
        for t in QT[q]:
            t = int(t)
            if live[t] and t not in pos:
                pos[t] = len(order)
                order.append(t)
    out = np.full((len(order), C), -1, np.int32)
    for i, q in enumerate(order):
        for c in range(C):
            t = int(QT[q, c])
            if live[t]:
                out[i, c] = pos[t]
    return ByteDFA(out[:, byte_class], qacc[order])


# -- byte DFA -> token automaton ----------------------------------------------------------------------------------------

class TokenAutomaton:
    """An automaton over token ids in the CSR form of rwkv_b200_constraint_add: state q's edges are
    (edge_tokens[e], edge_next[e]) for e in [edge_start[q], edge_start[q + 1]), tokens ascending. The start state is 0;
    a state without edges is complete. `sink` is the state the eos edges lead to (None without eos)."""

    def __init__(self, edge_start, edge_tokens, edge_next, sink=None, eos=None):
        self.edge_start = np.ascontiguousarray(edge_start, np.uint64)
        self.edge_tokens = np.ascontiguousarray(edge_tokens, np.uint64)
        self.edge_next = np.ascontiguousarray(edge_next, np.uint64)
        self.sink, self.eos = sink, eos

    @property
    def n_states(self):
        return len(self.edge_start) - 1

    def edges(self, state):
        a, b = int(self.edge_start[state]), int(self.edge_start[state + 1])
        return self.edge_tokens[a:b], self.edge_next[a:b]

    def complete(self, state):
        return self.edge_start[state] == self.edge_start[state + 1]

    def walk(self, tokens, state=0):
        """The state after `tokens` from `state`, or None when some token has no edge."""
        for t in tokens:
            toks, nxt = self.edges(state)
            i = int(np.searchsorted(toks, np.uint64(int(t))))
            if i == len(toks) or int(toks[i]) != int(t):
                return None
            state = int(nxt[i])
        return state


def _token_runs(dfa, tbytes, ids):
    """ends[q][i]: the DFA state after the bytes of token ids[i] from DFA state q, or dfa.n_states (dead)."""
    n = dfa.n_states
    T = np.vstack([np.where(dfa.trans < 0, n, dfa.trans), np.full((1, 256), n)]).astype(np.int32)
    lens = np.array([len(tbytes[t]) for t in ids], np.int64)
    width = int(lens.max()) if len(ids) else 0
    B = np.zeros((len(ids), width), np.uint8)
    for i, t in enumerate(ids):
        B[i, :lens[i]] = np.frombuffer(tbytes[t], np.uint8)
    first = np.searchsorted(lens, np.arange(width), side="right")  # ids are sorted by length
    ends = np.empty((n, len(ids)), np.int32)
    for q0 in range(0, n, 64):  # a batch of start states at a time bounds the memory
        cur = np.full((min(64, n - q0), len(ids)), 0, np.int32) + np.arange(q0, min(q0 + 64, n), dtype=np.int32)[:, None]
        for j in range(width):
            a = first[j]
            cur[:, a:] = T[cur[:, a:], B[a:, j]]
        ends[q0:q0 + len(cur)] = cur
    return ends


def token_automaton(dfa, tbytes, eos=0):
    """The token automaton of `dfa` over tokens with bytes `tbytes` (token_bytes()).

    Its states are the DFA states reachable at token boundaries, the start renumbered to 0. Token t has an edge from q to
    q' when its bytes lead from q to the live state q'; ids 0 and 1, the eos id and tokens without bytes have no byte
    edges. With eos given, every accepting state gets an edge eos -> sink, and the sink has no edges. Then, until
    nothing changes, every state without edges other than the sink (and, with eos=None, other than an accepting state)
    is removed with the edges into it. So "no edges" always means "complete": with eos, generation ends by emitting eos
    in an accepting state; with eos=None, by reaching an accepting state that cannot be extended (an accepting state with
    edges lets the stream go on). Raises ValueError when no token sequence completes the automaton."""
    ids = [t for t in range(len(tbytes)) if t not in SPECIAL and t != eos and len(tbytes[t]) > 0]
    ids.sort(key=lambda t: len(tbytes[t]))
    ids_arr = np.array(ids, np.int64)
    n = dfa.n_states
    ends = _token_runs(dfa, tbytes, ids)
    # breadth-first over token boundaries from the DFA start
    order, pos = [0], {0: 0}
    for q in order:
        for t in np.unique(ends[q][ends[q] < n]):
            if int(t) not in pos:
                pos[int(t)] = len(order)
                order.append(int(t))
    sink = len(order) if eos is not None else None
    edges = []  # per state: (tokens ascending, next states)
    for q in order:
        ok = ends[q] < n
        toks, nxt = ids_arr[ok], np.array([pos[int(x)] for x in ends[q][ok]], np.int64)
        if eos is not None and dfa.accept[q]:
            toks, nxt = np.append(toks, eos), np.append(nxt, sink)
        srt = np.argsort(toks, kind="stable")
        edges.append((toks[srt], nxt[srt]))
    if sink is not None:
        edges.append((np.zeros(0, np.int64), np.zeros(0, np.int64)))
    terminal = np.zeros(len(edges), bool)  # states allowed to have no edges
    if sink is not None:
        terminal[sink] = True
    else:
        terminal[:len(order)] = dfa.accept[order]
    kept = np.ones(len(edges), bool)
    while True:
        edges = [(t[kept[x]], x[kept[x]]) for t, x in edges]
        drop = kept & ~terminal & np.array([len(t) == 0 for t, _ in edges])
        if not drop.any():
            break
        kept &= ~drop
    if not kept[0]:
        raise ValueError("no token sequence completes this automaton")
    # renumber the kept states reachable from the start, breadth-first
    order2, pos2 = [0], {0: 0}
    for q in order2:
        for x in edges[q][1]:
            if int(x) not in pos2:
                pos2[int(x)] = len(order2)
                order2.append(int(x))
    start, toks, nxt = [0], [], []
    for q in order2:
        t, x = edges[q]
        toks.append(t)
        nxt.append(np.array([pos2[int(v)] for v in x], np.int64))
        start.append(start[-1] + len(t))
    cat = lambda a: np.concatenate(a) if a else np.zeros(0, np.int64)
    return TokenAutomaton(start, cat(toks), cat(nxt), sink=pos2.get(sink) if sink is not None else None, eos=eos)


def allow_all(eos=None):
    """A one-state automaton whose every token leads back to it: masks nothing and never completes."""
    return TokenAutomaton([0, VOCAB], np.arange(VOCAB), np.zeros(VOCAB, np.int64), eos=eos)
