"""ctypes binding of the C ABI in include/rwkv_b200.h (tests + bench.py only).

Fails loudly: if the CUDA library has not been built, or no CUDA device is visible,
constructing an Engine raises EngineError. There is no CPU fallback.
"""
import ctypes
import os

import numpy as np

VOCAB = 50277
MODE_PARRALEL, MODE_GPT = 0, 1
NO_TARGET = 0xFFFFFFFFFFFFFFFF  # RWKV_B200_NO_TARGET: a position score_streams does not score
MAX_TOP_N = 20                  # RWKV_B200_MAX_TOP_N
LOGPROBS_RAW, LOGPROBS_PROCESSED = 0, 1  # RWKV_B200_LOGPROBS_*: the row generate_streams(logprobs=...) scores on
NO_CONSTRAINT = 0xFFFFFFFFFFFFFFFF       # RWKV_B200_NO_CONSTRAINT: a stream of a constrained call without an automaton
MAX_CONSTRAINT_STATES = 65536            # RWKV_B200_MAX_CONSTRAINT_STATES

_PKG = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class EngineError(RuntimeError):
    pass


class Sampler(ctypes.Structure):
    """rwkv_b200_sampler: temperature (0 = arg-max), top_p in (0, 1], top_k (0 = no limit), and the presence /
    frequency penalties with their decay, which only generate_streams(sampling=...) applies."""
    _fields_ = [("temperature", ctypes.c_float), ("top_p", ctypes.c_float), ("top_k", ctypes.c_uint),
                ("presence_penalty", ctypes.c_float), ("frequency_penalty", ctypes.c_float),
                ("penalty_decay", ctypes.c_float)]

    def __init__(self, temperature=1.0, top_p=1.0, top_k=0, presence_penalty=0.0, frequency_penalty=0.0,
                 penalty_decay=1.0):
        super().__init__(temperature, top_p, top_k, presence_penalty, frequency_penalty, penalty_decay)


def _samplers(spec, n):
    """One Sampler (or dict of its fields) for all n streams, or a sequence of n of them, as a ctypes array."""
    one = lambda x: x if isinstance(x, Sampler) else Sampler(**x)
    if isinstance(spec, (Sampler, dict)):
        items = [one(spec)] * n
    else:
        items = [one(x) for x in spec]
        if len(items) != n:
            raise EngineError("%d samplers for %d streams" % (len(items), n))
    return (Sampler * n)(*items)


def _gen_args(streams, max_new, budgets, stop, overrides, u):
    """The arrays of a generate_streams call: S, slots, first tokens, budgets, stops, override tokens and values,
    uniforms, and the emitted tokens and lengths to fill."""
    S = len(streams)
    slots = np.ascontiguousarray([int(s) for s, _ in streams], dtype=np.uint64)
    first = np.ascontiguousarray([int(t) for _, t in streams], dtype=np.uint64)
    bud = np.ascontiguousarray(budgets, dtype=np.uint64) if budgets is not None else None
    stops = np.ascontiguousarray(list(stop), dtype=np.uint64)
    ovr = dict(overrides or {})
    otok = np.ascontiguousarray(list(ovr.keys()), dtype=np.uint64)
    oval = np.ascontiguousarray(list(ovr.values()), dtype=np.float32)
    us = np.ascontiguousarray(u, dtype=np.float64) if u is not None else None
    if bud is not None and bud.shape != (S,):
        raise EngineError("generate_streams: %d budgets for %d streams" % (bud.size, S))
    if us is not None and us.shape != (max_new, S):
        raise EngineError("generate_streams: u has shape %s, expected (%d, %d)" % (us.shape, max_new, S))
    return S, slots, first, bud, stops, otok, oval, us, np.zeros((S, max_new), np.uint64), np.zeros(S, np.uint64)


def lib_path():
    # RWKV_B200_LIB: A/B-test another build of the same ABI (tools/sweep.py); default is the in-tree library
    return os.environ.get("RWKV_B200_LIB") or os.path.join(_PKG, "librwkv_b200.so")


def load_library():
    """dlopen librwkv_b200.so and declare every symbol of include/rwkv_b200.h."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise EngineError("CUDA extension not built: %s (run python __graft_entry__.py build)" % path)
    lib = ctypes.CDLL(path)
    c = ctypes
    ull, vp, cp, i32 = c.c_ulonglong, c.c_void_p, c.c_char_p, c.c_int
    pull, pdbl, pflt = c.POINTER(ull), c.POINTER(c.c_double), c.POINTER(c.c_float)
    sig = {
        "rwkv_b200_last_error": (cp, []),
        "rwkv_b200_abi_version": (i32, []),
        "rwkv_b200_device_count": (i32, []),
        "rwkv_b200_load": (i32, [cp, ull, i32, i32, c.POINTER(vp), pull, pull]),
        "rwkv_b200_load_tp": (i32, [cp, ull, i32, i32, i32, i32, c.POINTER(vp), pull, pull]),
        "rwkv_b200_free": (None, [vp]),
        "rwkv_b200_tensor": (vp, [vp, i32]),
        "rwkv_b200_n_layers": (ull, [vp]),
        "rwkv_b200_n_embed": (ull, [vp]),
        "rwkv_b200_max_gpt": (ull, [vp]),
        "rwkv_b200_host_alloc": (vp, [c.c_size_t]),
        "rwkv_b200_host_free": (None, [vp]),
        "rwkv_b200_state_upload": (i32, [vp, pdbl, pdbl, pdbl, pdbl, pdbl, ull]),
        "rwkv_b200_state_download": (i32, [vp, pdbl, pdbl, pdbl, pdbl, pdbl, ull]),
        "rwkv_b200_state_zero": (i32, [vp]),
        "rwkv_b200_forward": (i32, [vp, pull, ull, i32, pflt]),
        "rwkv_b200_forward_greedy": (i32, [vp, ull, pull, pflt]),
        "rwkv_b200_logits_host": (pflt, [vp]),
        "rwkv_b200_sample_typical": (i32, [vp, c.c_float, c.c_double, pull, pdbl]),
        "rwkv_b200_debug_read": (c.c_longlong, [vp, cp, vp, c.c_size_t]),
        "rwkv_b200_decode_timed": (i32, [vp, pull, ull, i32, pflt]),
        "rwkv_b200_kernel_count": (i32, []),
        "rwkv_b200_kernel_name": (cp, [i32]),
        "rwkv_b200_profile": (i32, [vp, pull, ull, pflt, pull, pdbl]),
        "rwkv_b200_launch_count": (ull, [vp]),
        "rwkv_b200_set_option": (i32, [vp, cp, cp]),
        "rwkv_b200_tp_buffer_bytes": (c.c_size_t, [vp]),
        "rwkv_b200_tp_export": (i32, [vp, vp]),
        "rwkv_b200_tp_import": (i32, [vp, vp]),
        "rwkv_b200_forward_streams": (i32, [vp, pull, ull, pull, pull, ull, pflt, pull]),
        "rwkv_b200_sample_typical_streams": (i32, [vp, ull, c.c_float, pdbl, pull, pdbl]),
        "rwkv_b200_generate_streams": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull, c.c_float, pdbl,
                                             pull, pull]),
        "rwkv_b200_sample_streams": (i32, [vp, ull, c.POINTER(Sampler), pdbl, pflt, pull, pdbl]),
        "rwkv_b200_generate_streams_ex": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull, c.POINTER(Sampler),
                                                pdbl, pull, pull]),
        "rwkv_b200_score_streams": (i32, [vp, pull, ull, pull, pull, ull, pull, c.c_uint, pdbl, pull, pull, pdbl]),
        "rwkv_b200_generate_streams_logprobs": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                      c.POINTER(Sampler), pdbl, pull, pull, i32, c.c_uint, pdbl, pull, pull,
                                                      pdbl]),
        "rwkv_b200_constraint_add": (i32, [vp, ull, pull, pull, pull, pull]),
        "rwkv_b200_constraint_remove": (i32, [vp, ull]),
        "rwkv_b200_generate_streams_constrained": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                         c.POINTER(Sampler), pdbl, pull, pull, i32, c.c_uint, pdbl, pull,
                                                         pull, pdbl, pull, pull, pull]),
        "rwkv_b200_beam_search": (i32, [vp, pull, pull, ull, c.c_uint, ull, pull, ull, c.c_double, c.c_uint, pull, pull, pdbl,
                                        pdbl, c.POINTER(c.c_ubyte), pdbl]),
        "rwkv_b200_slot_zero": (i32, [vp, ull]),
        "rwkv_b200_slot_copy": (i32, [vp, ull, ull]),
        "rwkv_b200_slot_upload": (i32, [vp, ull, pdbl, pdbl, pdbl, pdbl, pdbl]),
        "rwkv_b200_slot_download": (i32, [vp, ull, pdbl, pdbl, pdbl, pdbl, pdbl]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
    lib._declared = sorted(sig)
    _LIB = lib
    return lib


def _ptr(a, ctype):
    return a.ctypes.data_as(ctypes.POINTER(ctype)) if a is not None else None


class Engine:
    """One loaded model on one GPU. Mirrors the reference's RWKV host class at the
    granularity the tests need: load, forward(tokens, mode), host<->device state."""

    def __init__(self, path, max_gpt=1, device=0, quiet=True, tp_rank=0, tp_size=1):
        """tp_size > 1: this process is rank `tp_rank` of a tensor-parallel group (one GPU per rank); wire the
        ranks with tp.connect(engine) before the first forward (include/rwkv_b200.h, "tensor-parallel wiring")."""
        self.lib = load_library()
        if self.lib.rwkv_b200_device_count() <= 0:
            raise EngineError("no CUDA device visible; the H100 engine has no CPU fallback")
        h = ctypes.c_void_p()
        L, E = ctypes.c_ulonglong(), ctypes.c_ulonglong()
        rc = self.lib.rwkv_b200_load_tp(path.encode(), max_gpt, device, 1 if quiet else 0, tp_rank, tp_size,
                                        ctypes.byref(h), ctypes.byref(L), ctypes.byref(E))
        if rc != 0:
            raise EngineError("rwkv_b200_load(%s) failed [%d]: %s" % (path, rc, self._err()))
        self.h = h
        self.n_layers, self.n_embed, self.max_gpt = L.value, E.value, max_gpt
        self.tp_rank, self.tp_size = tp_rank, tp_size

    # -- tensor-parallel wiring ------------------------------------------------------------
    def tp_export(self):
        """CUDA IPC handle (64 bytes) of this rank's exchange block."""
        buf = (ctypes.c_ubyte * 64)()
        self._ck(self.lib.rwkv_b200_tp_export(self.h, ctypes.cast(buf, ctypes.c_void_p)), "tp_export")
        return bytes(buf)

    def tp_import(self, handles):
        """handles: one 64-byte handle per rank, in rank order (the own entry is ignored)."""
        if len(handles) != self.tp_size or any(len(x) != 64 for x in handles):
            raise EngineError("tp_import needs %d handles of 64 bytes" % self.tp_size)
        blob = b"".join(handles)
        buf = (ctypes.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._ck(self.lib.rwkv_b200_tp_import(self.h, ctypes.cast(buf, ctypes.c_void_p)), "tp_import")

    def _err(self):
        return self.lib.rwkv_b200_last_error().decode(errors="replace")

    def _ck(self, rc, what):
        if rc != 0:
            raise EngineError("%s failed [%d]: %s" % (what, rc, self._err()))

    def close(self):
        if getattr(self, "h", None):
            self.lib.rwkv_b200_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- compute ---------------------------------------------------------------------------
    def forward(self, tokens, mode=MODE_GPT, want_logits=True):
        toks = np.ascontiguousarray(np.atleast_1d(np.asarray(tokens, dtype=np.uint64)))
        out = np.empty((len(toks), VOCAB), np.float32) if want_logits else None
        self._ck(self.lib.rwkv_b200_forward(self.h, _ptr(toks, ctypes.c_ulonglong), len(toks), mode,
                                            _ptr(out, ctypes.c_float)), "forward")
        return out

    def sample_typical(self, temp, u):
        """Device sampler on the logits of the last forward: (token, margin) for the uniform `u`."""
        tok, margin = ctypes.c_ulonglong(), ctypes.c_double()
        self._ck(self.lib.rwkv_b200_sample_typical(self.h, temp, u, ctypes.byref(tok), ctypes.byref(margin)), "sample_typical")
        return int(tok.value), float(margin.value)

    def forward_greedy(self, token, want_logits=False):
        nxt = ctypes.c_ulonglong()
        out = np.empty(VOCAB, np.float32) if want_logits else None
        self._ck(self.lib.rwkv_b200_forward_greedy(self.h, int(token), ctypes.byref(nxt),
                                                   _ptr(out, ctypes.c_float)), "forward_greedy")
        return (nxt.value, out) if want_logits else nxt.value

    # -- multi-stream serving --------------------------------------------------------------
    def forward_streams(self, streams, want_logits=True, want_next=False):
        """One ragged forward: streams = [(slot, tokens), ...], each advancing its own state slot.
        Returns (logits [S][V] after each stream's last token | None, device arg-max [S] | None)."""
        slots = np.ascontiguousarray([int(s) for s, _ in streams], dtype=np.uint64)
        seqs = [np.atleast_1d(np.asarray(t, dtype=np.uint64)) for _, t in streams]
        lens = np.ascontiguousarray([len(t) for t in seqs], dtype=np.uint64)
        toks = np.ascontiguousarray(np.concatenate(seqs) if seqs else np.zeros(0, np.uint64))
        logits = np.empty((len(seqs), VOCAB), np.float32) if want_logits else None
        nxt = np.empty(len(seqs), np.uint64) if want_next else None
        self._ck(self.lib.rwkv_b200_forward_streams(self.h, _ptr(toks, ctypes.c_ulonglong), len(toks),
                                                    _ptr(slots, ctypes.c_ulonglong), _ptr(lens, ctypes.c_ulonglong),
                                                    len(seqs), _ptr(logits, ctypes.c_float),
                                                    _ptr(nxt, ctypes.c_ulonglong)), "forward_streams")
        return logits, nxt

    def sample_typical_streams(self, temp, us):
        """Device sampler on every row of the last forward_streams call: (tokens [S], margins [S])."""
        u = np.ascontiguousarray(us, dtype=np.float64)
        toks = np.empty(len(u), np.uint64)
        margins = np.empty(len(u), np.float64)
        self._ck(self.lib.rwkv_b200_sample_typical_streams(self.h, len(u), temp, _ptr(u, ctypes.c_double),
                                                           _ptr(toks, ctypes.c_ulonglong), _ptr(margins, ctypes.c_double)),
                 "sample_typical_streams")
        return toks, margins

    def sample_streams(self, params, us, logits=None):
        """Per-row sampler (include/rwkv_b200.h, rwkv_b200_sampler) on the rows of the last forward_streams call, or on
        the host rows `logits` [S][V] when given: (tokens [S], margins [S]). params: one Sampler (or dict) for every
        row, or one per row; us: S uniforms in [0, 1), or None when every row has temperature 0."""
        u = np.ascontiguousarray(us, dtype=np.float64) if us is not None else None
        lg = np.ascontiguousarray(logits, dtype=np.float32) if logits is not None else None
        if lg is not None:
            if lg.ndim != 2 or lg.shape[1] != VOCAB:
                raise EngineError("sample_streams: logits have shape %s, expected (S, %d)" % (lg.shape, VOCAB))
            n = lg.shape[0]
        elif u is not None:
            n = len(u)
        elif not isinstance(params, (Sampler, dict)):
            n = len(params)
        else:
            raise EngineError("sample_streams: the row count is unknown (give us, logits or one sampler per row)")
        if u is not None and u.shape != (n,):
            raise EngineError("sample_streams: %d uniforms for %d rows" % (u.size, n))
        sp = _samplers(params, n)
        toks = np.empty(n, np.uint64)
        margins = np.empty(n, np.float64)
        self._ck(self.lib.rwkv_b200_sample_streams(self.h, n, sp, _ptr(u, ctypes.c_double), _ptr(lg, ctypes.c_float),
                                                   _ptr(toks, ctypes.c_ulonglong), _ptr(margins, ctypes.c_double)),
                 "sample_streams")
        return toks, margins

    def generate_streams(self, streams, max_new, budgets=None, stop=(), overrides=None, temp=None, u=None, sampling=None,
                         logprobs=None, top_n=0, constraints=None):
        """Generate up to max_new tokens per stream on the device: streams = [(slot, first_token), ...].
        Arg-max when u is None, else the typical sampler with u[step][stream] and temp (default 1.0). budgets: tokens
        per stream (None = max_new each); stop: token ids that end a stream (emitted, not fed); overrides = {token:
        logit value} applied before every pick. sampling: one Sampler (or dict) for every stream, or one per stream;
        then the call is rwkv_b200_generate_streams_ex (penalties, temperature, top-p, top-k; u as above, None only if
        every temperature is 0) and temp is not used. Returns one numpy uint64 array of emitted tokens per stream.
        logprobs = "raw" or "processed": the same generation (sampling=None is the arg-max; the typical sampler is not
        available) also scores each emitted token on the device (rwkv_b200_generate_streams_logprobs): "raw" on the
        model's logits, "processed" on the row the sampler read divided by the stream's temperature. Then it returns
        one dict per stream: "tokens", "logprobs" (float64), "ranks" (uint64, tokens ranked before the emitted one),
        and with top_n > 0 "top_tokens" [len][top_n] and "top_logprobs" [len][top_n], each as long as the stream.
        constraints: one id of add_constraint for every stream, or one entry per stream: an id, (id, start_state) or
        None (rwkv_b200_generate_streams_constrained: each step masks every token without an edge out of the stream's
        automaton state, and a stream ends when its state has no edges). Then it returns one dict per stream with
        "tokens" and "state" (the final automaton state, None without a constraint), plus the logprob fields when
        logprobs is given. Like logprobs, constraints need sampling=... or the arg-max (not the typical sampler)."""
        if logprobs is not None or constraints is not None:
            return self._generate_scored(streams, max_new, budgets, stop, overrides, temp, u, sampling, logprobs, top_n,
                                         constraints)
        temp = 1.0 if temp is None else temp
        S, slots, first, bud, stops, otok, oval, us, out, lens = _gen_args(streams, max_new, budgets, stop, overrides, u)
        P = ctypes.c_ulonglong
        if sampling is not None:
            self._ck(self.lib.rwkv_b200_generate_streams_ex(self.h, _ptr(slots, P), _ptr(first, P), S, max_new, _ptr(bud, P),
                                                            _ptr(stops, P), len(stops), _ptr(otok, P),
                                                            _ptr(oval, ctypes.c_float), len(otok), _samplers(sampling, S),
                                                            _ptr(us, ctypes.c_double), _ptr(out, P), _ptr(lens, P)),
                     "generate_streams_ex")
            return [out[s, :int(lens[s])].copy() for s in range(S)]
        self._ck(self.lib.rwkv_b200_generate_streams(self.h, _ptr(slots, P), _ptr(first, P), S, max_new, _ptr(bud, P),
                                                     _ptr(stops, P), len(stops), _ptr(otok, P), _ptr(oval, ctypes.c_float),
                                                     len(otok), temp, _ptr(us, ctypes.c_double), _ptr(out, P),
                                                     _ptr(lens, P)), "generate_streams")
        return [out[s, :int(lens[s])].copy() for s in range(S)]

    def _generate_scored(self, streams, max_new, budgets, stop, overrides, temp, u, sampling, logprobs, top_n, constraints):
        """generate_streams with logprobs or constraints: rwkv_b200_generate_streams_constrained when constraints are
        given, else rwkv_b200_generate_streams_logprobs. One dict per stream."""
        modes = {None: LOGPROBS_RAW, "raw": LOGPROBS_RAW, "processed": LOGPROBS_PROCESSED}
        if logprobs not in modes:
            raise EngineError("generate_streams: logprobs must be 'raw' or 'processed', not %r" % (logprobs,))
        if sampling is None and (u is not None or temp is not None):
            if constraints is not None:
                raise EngineError("generate_streams: constraints need sampling=... (or neither u nor temp, for the "
                                  "arg-max); the typical sampler does not take them")
            raise EngineError("generate_streams: logprobs need sampling=... (or neither u nor temp, for the arg-max); "
                              "the typical sampler reports no log-probabilities")
        S, slots, first, bud, stops, otok, oval, us, out, lens = _gen_args(streams, max_new, budgets, stop, overrides, u)
        lp = ranks = top_tok = top_lp = None
        if logprobs is not None:
            lp = np.empty((S, max_new), np.float64)
            ranks = np.empty((S, max_new), np.uint64)
            if top_n > 0:
                top_tok = np.empty((S, max_new, top_n), np.uint64)
                top_lp = np.empty((S, max_new, top_n), np.float64)
        P = ctypes.c_ulonglong
        sp = _samplers(sampling, S) if sampling is not None else None
        args = (self.h, _ptr(slots, P), _ptr(first, P), S, max_new, _ptr(bud, P), _ptr(stops, P), len(stops), _ptr(otok, P),
                _ptr(oval, ctypes.c_float), len(otok), sp, _ptr(us, ctypes.c_double), _ptr(out, P), _ptr(lens, P),
                modes[logprobs], int(top_n), _ptr(lp, ctypes.c_double), _ptr(ranks, P), _ptr(top_tok, P),
                _ptr(top_lp, ctypes.c_double))
        if constraints is None:
            self._ck(self.lib.rwkv_b200_generate_streams_logprobs(*args), "generate_streams_logprobs")
        else:
            spec = [constraints] * S if isinstance(constraints, (int, np.integer)) else list(constraints)
            if len(spec) != S:
                raise EngineError("generate_streams: %d constraints for %d streams" % (len(spec), S))
            pairs = [(NO_CONSTRAINT, 0) if c is None else (int(c[0]), int(c[1])) if isinstance(c, (tuple, list))
                     else (int(c), 0) for c in spec]
            ids = np.ascontiguousarray([c for c, _ in pairs], np.uint64)
            starts = np.ascontiguousarray([q for _, q in pairs], np.uint64)
            states = np.zeros(S, np.uint64)
            self._ck(self.lib.rwkv_b200_generate_streams_constrained(*args, _ptr(ids, P), _ptr(starts, P), _ptr(states, P)),
                     "generate_streams_constrained")
        res = []
        for s in range(S):
            n = int(lens[s])
            d = {"tokens": out[s, :n].copy()}
            if constraints is not None:
                d["state"] = int(states[s]) if ids[s] != np.uint64(NO_CONSTRAINT) else None
            if lp is not None:
                d["logprobs"], d["ranks"] = lp[s, :n].copy(), ranks[s, :n].copy()
                if top_n > 0:
                    d["top_tokens"], d["top_logprobs"] = top_tok[s, :n].copy(), top_lp[s, :n].copy()
            res.append(d)
        return res

    def add_constraint(self, automaton):
        """Upload a token automaton (constrain.TokenAutomaton, or anything with its edge_start, edge_tokens and
        edge_next arrays) for generate_streams(constraints=...); returns its id."""
        start = np.ascontiguousarray(automaton.edge_start, np.uint64)
        toks = np.ascontiguousarray(automaton.edge_tokens, np.uint64)
        nxt = np.ascontiguousarray(automaton.edge_next, np.uint64)
        cid = ctypes.c_ulonglong()
        P = ctypes.c_ulonglong
        self._ck(self.lib.rwkv_b200_constraint_add(self.h, len(start) - 1, _ptr(start, P), _ptr(toks, P), _ptr(nxt, P),
                                                   ctypes.byref(cid)), "constraint_add")
        return int(cid.value)

    def remove_constraint(self, cid):
        self._ck(self.lib.rwkv_b200_constraint_remove(self.h, int(cid)), "constraint_remove")

    def score_streams(self, streams, targets=None, top_n=0):
        """Score target tokens in one ragged forward: streams = [(slot, tokens), ...], each advancing its own state slot
        as forward_streams does. targets: None scores each stream's own next tokens (tokens[1:]; its last position is
        not scored); otherwise one list per stream, as long as its tokens, of the token expected after each position or
        None for a position that is not scored. Returns per stream a dict of "logprobs" (float64, NaN where not scored)
        and "ranks" (uint64, tokens ranked before the target; NO_TARGET where not scored), and with top_n > 0
        "top_tokens" [len][top_n] and "top_logprobs" [len][top_n], the first top_n tokens by logit (ties: lower index)."""
        slots = np.ascontiguousarray([int(s) for s, _ in streams], dtype=np.uint64)
        seqs = [np.atleast_1d(np.asarray(t, dtype=np.uint64)) for _, t in streams]
        lens = np.ascontiguousarray([len(t) for t in seqs], dtype=np.uint64)
        toks = np.ascontiguousarray(np.concatenate(seqs) if seqs else np.zeros(0, np.uint64))
        if targets is None:
            tg = [list(t[1:]) + [None] for t in seqs]
        else:
            tg = list(targets)
            if len(tg) != len(seqs) or any(len(a) != len(b) for a, b in zip(tg, seqs)):
                raise EngineError("score_streams: targets need one list per stream, as long as its tokens")
        tgt = np.ascontiguousarray([NO_TARGET if x is None else int(x) for row in tg for x in row], dtype=np.uint64)
        n = len(toks)
        lp = np.empty(n, np.float64)
        ranks = np.empty(n, np.uint64)
        top_tok = np.empty((n, top_n), np.uint64) if top_n > 0 else None
        top_lp = np.empty((n, top_n), np.float64) if top_n > 0 else None
        P = ctypes.c_ulonglong
        self._ck(self.lib.rwkv_b200_score_streams(self.h, _ptr(toks, P), n, _ptr(slots, P), _ptr(lens, P), len(seqs),
                                                  _ptr(tgt, P), int(top_n), _ptr(lp, ctypes.c_double), _ptr(ranks, P),
                                                  _ptr(top_tok, P), _ptr(top_lp, ctypes.c_double)), "score_streams")
        out, t0 = [], 0
        for t in seqs:
            sl = slice(t0, t0 + len(t))
            d = {"logprobs": lp[sl].copy(), "ranks": ranks[sl].copy()}
            if top_n > 0:
                d["top_tokens"] = top_tok[sl].copy()
                d["top_logprobs"] = top_lp[sl].copy()
            out.append(d)
            t0 += len(t)
        return out

    def beam_search(self, groups, max_new, beams, stop=(), length_penalty=1.0, n_best=1, token_logprobs=False):
        """Beam search on the device (rwkv_b200_beam_search): groups = [(slots, first_token), ...], each with `beams`
        distinct slots, the first holding the prompt state (the others are overwritten). stop: token ids that finish a
        hypothesis; length_penalty: alpha of score = logprob / len ** alpha. Returns per group its n_best hypotheses,
        best first, each a dict of "tokens" (uint64), "logprob" (the sum of the token logprobs), "score", "finished"
        (ended by a stop token), and with token_logprobs=True "token_logprobs" (float64, one per token)."""
        G = len(groups)
        flat = [int(s) for slots, _ in groups for s in slots]
        if any(len(slots) != beams for slots, _ in groups):
            raise EngineError("beam_search: every group needs %d slots" % beams)
        slots = np.ascontiguousarray(flat, dtype=np.uint64)
        first = np.ascontiguousarray([int(t) for _, t in groups], dtype=np.uint64)
        stops = np.ascontiguousarray(list(stop), dtype=np.uint64)
        K = max(int(n_best), 1)
        toks = np.zeros((G, K, max_new), np.uint64)
        lens = np.zeros((G, K), np.uint64)
        lp = np.zeros((G, K), np.float64)
        scores = np.zeros((G, K), np.float64)
        fin = np.zeros((G, K), np.uint8)
        tlp = np.zeros((G, K, max_new), np.float64) if token_logprobs else None
        P = ctypes.c_ulonglong
        self._ck(self.lib.rwkv_b200_beam_search(self.h, _ptr(slots, P), _ptr(first, P), G, int(beams), int(max_new),
                                                _ptr(stops, P), len(stops), float(length_penalty), int(n_best),
                                                _ptr(toks, P), _ptr(lens, P), _ptr(lp, ctypes.c_double),
                                                _ptr(scores, ctypes.c_double), _ptr(fin, ctypes.c_ubyte),
                                                _ptr(tlp, ctypes.c_double)), "beam_search")
        res = []
        for g in range(G):
            hyps = []
            for i in range(K):
                n = int(lens[g, i])
                d = {"tokens": toks[g, i, :n].copy(), "logprob": float(lp[g, i]), "score": float(scores[g, i]),
                     "finished": bool(fin[g, i])}
                if token_logprobs:
                    d["token_logprobs"] = tlp[g, i, :n].copy()
                hyps.append(d)
            res.append(hyps)
        return res

    def slot_zero(self, slot):
        self._ck(self.lib.rwkv_b200_slot_zero(self.h, slot), "slot_zero")

    def slot_copy(self, src, dst):
        self._ck(self.lib.rwkv_b200_slot_copy(self.h, src, dst), "slot_copy")

    def slot_download(self, slot):
        n = self.n_layers * self.n_embed
        arrs = [np.empty(n, np.float64) for _ in range(5)]
        self._ck(self.lib.rwkv_b200_slot_download(self.h, slot, *[_ptr(a, ctypes.c_double) for a in arrs]), "slot_download")
        return dict(zip(("xy", "aa", "bb", "pp", "dd"), arrs))

    def slot_upload(self, slot, st):
        arrs = [np.ascontiguousarray(st[k], np.float64) if st.get(k) is not None else None
                for k in ("xy", "aa", "bb", "pp", "dd")]
        self._ck(self.lib.rwkv_b200_slot_upload(self.h, slot, *[_ptr(a, ctypes.c_double) for a in arrs]), "slot_upload")

    # -- state -----------------------------------------------------------------------------
    def state_zero(self):
        self._ck(self.lib.rwkv_b200_state_zero(self.h), "state_zero")

    def state_download(self, slots=1):
        n = self.n_layers * self.n_embed * slots
        arrs = [np.empty(n, np.float64) for _ in range(5)]
        self._ck(self.lib.rwkv_b200_state_download(self.h, *[_ptr(a, ctypes.c_double) for a in arrs], slots),
                 "state_download")
        return dict(zip(("xy", "aa", "bb", "pp", "dd"), arrs))

    def state_upload(self, st, slots=1):
        arrs = [np.ascontiguousarray(st[k], np.float64) if st.get(k) is not None else None
                for k in ("xy", "aa", "bb", "pp", "dd")]
        self._ck(self.lib.rwkv_b200_state_upload(self.h, *[_ptr(a, ctypes.c_double) for a in arrs], slots),
                 "state_upload")

    # -- knobs / measurement ---------------------------------------------------------------
    def set_option(self, key, value):
        self._ck(self.lib.rwkv_b200_set_option(self.h, key.encode(), str(value).encode()), "set_option(%s)" % key)

    def debug_read(self, name):
        E = self.n_embed
        dt, n = {"x": (np.float64, E), "logits": (np.float32, VOCAB)}[name]
        a = np.empty(n, dt)
        got = self.lib.rwkv_b200_debug_read(self.h, name.encode(), a.ctypes.data_as(ctypes.c_void_p), a.nbytes)
        if got != n:
            raise EngineError("debug_read(%s) failed" % name)
        return a

    def read_trace(self, grid=132, per_cta=2048):
        """Per-CTA globaltimer stamps of the last token kernel (set_option('trace', 1) first)."""
        a = np.zeros(grid * per_cta, np.uint64)
        got = self.lib.rwkv_b200_debug_read(self.h, b"trace", a.ctypes.data_as(ctypes.c_void_p), a.nbytes)
        if got != a.size:
            raise EngineError("read_trace failed (trace option not enabled?)")
        return a.reshape(grid, per_cta)

    def read_tile_trace(self, grid=132, per_cta=4096):
        """[2][grid][per_cta] globaltimer: tile copy issued by the producer / tile seen ready by consumer thread 0."""
        a = np.zeros(2 * grid * per_cta, np.uint64)
        got = self.lib.rwkv_b200_debug_read(self.h, b"ptrace", a.ctypes.data_as(ctypes.c_void_p), a.nbytes)
        if got != a.size:
            raise EngineError("read_tile_trace failed")
        return a.reshape(2, grid, per_cta)

    def decode_timed(self, tokens, teacher_forced=True):
        toks = np.ascontiguousarray(np.asarray(tokens, dtype=np.uint64))
        ms = ctypes.c_float()
        self._ck(self.lib.rwkv_b200_decode_timed(self.h, _ptr(toks, ctypes.c_ulonglong), len(toks),
                                                 1 if teacher_forced else 0, ctypes.byref(ms)), "decode_timed")
        return ms.value

    def profile(self, tokens):
        k = self.lib.rwkv_b200_kernel_count()
        toks = np.ascontiguousarray(np.asarray(tokens, dtype=np.uint64))
        ms = np.zeros(k, np.float32)
        cnt = np.zeros(k, np.uint64)
        by = np.zeros(k, np.float64)
        self._ck(self.lib.rwkv_b200_profile(self.h, _ptr(toks, ctypes.c_ulonglong), len(toks),
                                            _ptr(ms, ctypes.c_float), _ptr(cnt, ctypes.c_ulonglong),
                                            _ptr(by, ctypes.c_double)), "profile")
        names = [self.lib.rwkv_b200_kernel_name(i).decode() for i in range(k)]
        return {n: {"ms_sum": float(ms[i]), "launches": int(cnt[i]), "bytes_per_launch": float(by[i])}
                for i, n in enumerate(names)}

    @property
    def launch_count(self):
        return int(self.lib.rwkv_b200_launch_count(self.h))
