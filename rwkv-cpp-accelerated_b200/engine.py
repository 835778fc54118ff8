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
NO_STOP_SET = 0xFFFFFFFFFFFFFFFF         # RWKV_B200_NO_STOP_SET: a stream of a stop-string call without a set
MAX_STOP_BYTES = 4096                    # RWKV_B200_MAX_STOP_BYTES
INDEX_L1, INDEX_L2 = 0, 1                # RWKV_B200_INDEX_*: the metric a StateIndex search ranks by
MAX_NEIGHBOURS = 256                     # RWKV_B200_MAX_NEIGHBOURS
NO_ENTRY = 0xFFFFFFFFFFFFFFFF            # RWKV_B200_NO_ENTRY: a search position past the entries found
NO_ADAPTER = 0xFFFFFFFFFFFFFFFF          # RWKV_B200_NO_ADAPTER: Engine.bind_adapter(slot, None)
NO_GUIDANCE = 0xFFFFFFFFFFFFFFFF         # RWKV_B200_NO_GUIDANCE: an unguided stream of generate_streams(guidance=...)
MAX_ADAPTER_RANK = 64                    # RWKV_B200_MAX_ADAPTER_RANK
# RWKV_B200_AD_* in order: the checkpoint's Linear name inside a block of each projection an adapter may adapt
ADAPTER_MATRICES = ("att.key", "att.value", "att.receptance", "att.output", "ffn.key", "ffn.value", "ffn.receptance")

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


class Request(ctypes.Structure):
    """rwkv_b200_request: one request of a Batcher."""
    P = ctypes.POINTER(ctypes.c_ulonglong)
    _fields_ = [("slot", ctypes.c_ulonglong), ("prompt", P), ("n_prompt", ctypes.c_ulonglong),
                ("max_new", ctypes.c_ulonglong), ("sampler", Sampler), ("u", ctypes.POINTER(ctypes.c_double)),
                ("stop", P), ("n_stop", ctypes.c_ulonglong)]


class RequestEx(ctypes.Structure):
    """rwkv_b200_request_ex: what Batcher.submit adds to a request (overrides, an automaton, log-probabilities)."""
    _fields_ = [("override_tokens", ctypes.POINTER(ctypes.c_ulonglong)), ("override_values", ctypes.POINTER(ctypes.c_float)),
                ("n_override", ctypes.c_ulonglong), ("constraint_id", ctypes.c_ulonglong),
                ("start_state", ctypes.c_ulonglong), ("logprobs", ctypes.c_int), ("logprob_mode", ctypes.c_int),
                ("top_n", ctypes.c_uint)]


class RequestSpec(ctypes.Structure):
    """rwkv_b200_request_spec: prompt-lookup speculation for one batcher request."""
    _fields_ = [("spare_slots", ctypes.POINTER(ctypes.c_ulonglong)), ("draft", ctypes.c_uint), ("ngram", ctypes.c_uint),
                ("context", ctypes.POINTER(ctypes.c_ulonglong)), ("n_context", ctypes.c_ulonglong)]


class StopRequest(ctypes.Structure):
    """rwkv_b200_stop_request: per stream its stop set id and start state, and where the results go."""
    P = ctypes.POINTER(ctypes.c_ulonglong)
    _fields_ = [("set_ids", P), ("start_states", P), ("states_out", P), ("hit_out", P), ("tail_out", P)]


class Guidance(ctypes.Structure):
    """rwkv_b200_guidance: per stream its guidance slot (or NO_GUIDANCE), guidance first token and scale gamma."""
    _fields_ = [("slots", ctypes.POINTER(ctypes.c_ulonglong)), ("first_tokens", ctypes.POINTER(ctypes.c_ulonglong)),
                ("scales", ctypes.POINTER(ctypes.c_float))]


class Drafter(ctypes.Structure):
    """rwkv_b200_drafter: the draft model of rwkv_b200_generate_streams_drafted and its slots [n_streams][2] (D0, D1)."""
    _fields_ = [("model", ctypes.c_void_p), ("slots", ctypes.POINTER(ctypes.c_ulonglong))]


def guide_rows(c, q, scale):
    """Rule 2 of classifier-free guidance (include/rwkv_b200.h) in numpy: c + (scale - 1) * (c - q) in float32, each
    operation rounded once, with w = scale - 1 itself rounded to float32. c, q: the conditional and guidance logits."""
    c = np.asarray(c, np.float32)
    q = np.asarray(q, np.float32)
    w = np.float32(np.float32(scale) - np.float32(1.0))
    return c + w * (c - q)


def _guidance(guidance, S, what):
    """The Guidance struct of one entry per stream: None, or (slot, first_token, scale)."""
    spec = list(guidance)
    if len(spec) != S:
        raise EngineError("%s: %d guidance entries for %d streams" % (what, len(spec), S))
    slots = np.ascontiguousarray([NO_GUIDANCE if g is None else int(g[0]) for g in spec], np.uint64)
    first = np.ascontiguousarray([0 if g is None else int(g[1]) for g in spec], np.uint64)
    scales = np.ascontiguousarray([1.0 if g is None else float(g[2]) for g in spec], np.float32)
    gd = Guidance(_ptr(slots, ctypes.c_ulonglong), _ptr(first, ctypes.c_ulonglong), _ptr(scales, ctypes.c_float))
    gd._keep = (slots, first, scales)
    return gd


class PrefixStats(ctypes.Structure):
    """struct rwkv_b200_prefix_stats (include/rwkv_b200.h)."""
    _fields_ = [(f, ctypes.c_ulonglong) for f in ("live", "lookups", "hit_tokens", "prefilled_tokens", "snapshots", "skipped",
                                                  "evictions")]


class Adapter(ctypes.Structure):
    """rwkv_b200_adapter: the rank, the scale and per projection the A and B arrays (NULL: not adapted)."""
    PF = ctypes.POINTER(ctypes.c_float)
    _fields_ = [("rank", ctypes.c_uint), ("scale", ctypes.c_double), ("A", PF * 7), ("B", PF * 7)]


REQ_STATUS = ("queued", "prefilling", "generating", "done", "cancelled")  # RWKV_B200_REQ_* in order


def adapter_dims(name, E):
    """(in, out) of the projection `name` (an entry of ADAPTER_MATRICES) at width E."""
    return (4 * E if name == "ffn.value" else E), (4 * E if name == "ffn.key" else E)


def parse_adapter(weights, L, E):
    """(rank, {name: (A [L][r][in], B [L][out][r]) float32}) of a LoRA state dict whose keys are the checkpoint's Linear
    names with ".lora_A" ([r][in]) or ".lora_B" ([out][r]), e.g. "blocks.3.att.key.lora_A". Layers a projection lacks
    get zeros. Raises ValueError, naming the key, for an unknown key, a key without its partner, a rank that differs
    from the others or is outside 1..64, a wrong shape, and an empty dict."""
    per = {}  # (layer, name) -> {"A": array, "B": array}
    for key, val in weights.items():
        parts = key.split(".")
        ok = (len(parts) == 5 and parts[0] == "blocks" and parts[1].isdigit() and ".".join(parts[2:4]) in ADAPTER_MATRICES
              and parts[4] in ("lora_A", "lora_B"))
        if not ok:
            hint = ""
            if any(p.startswith("time_") or p.startswith("ln") for p in parts):
                hint = (" (full-parameter tensors such as time_* and ln are not adapters; merge them into the model with "
                        "tools/convert_model.py --lora)")
            raise ValueError("adapter key %r is not <blocks.N.{att,ffn}.<projection>.lora_A|lora_B>%s" % (key, hint))
        l, name = int(parts[1]), ".".join(parts[2:4])
        if l >= L:
            raise ValueError("adapter key %r: layer %d >= n_layers %d" % (key, l, L))
        a = np.asarray(val.detach().cpu().numpy() if hasattr(val, "detach") else val, np.float32)
        per.setdefault((l, name), {})[parts[4][-1]] = (key, a)
    if not per:
        raise ValueError("the adapter has no lora_A / lora_B tensors")
    rank = None
    mats = {}
    for (l, name), ab in sorted(per.items()):
        for half in "AB":
            if half not in ab:
                other = ab["B" if half == "A" else "A"][0]
                raise ValueError("adapter key %r has no lora_%s partner" % (other, half))
        n_in, n_out = adapter_dims(name, E)
        (ka, A), (kb, B) = ab["A"], ab["B"]
        r = A.shape[0] if A.ndim == 2 else -1
        if rank is None:
            rank = r
        if not 1 <= r <= MAX_ADAPTER_RANK:
            raise ValueError("adapter key %r: rank %d is outside 1..%d" % (ka, r, MAX_ADAPTER_RANK))
        if r != rank:
            raise ValueError("adapter key %r has rank %d, other projections have rank %d" % (ka, r, rank))
        if A.shape != (rank, n_in):
            raise ValueError("adapter key %r has shape %s, expected %s" % (ka, A.shape, (rank, n_in)))
        if B.shape != (n_out, rank):
            raise ValueError("adapter key %r has shape %s, expected %s" % (kb, B.shape, (n_out, rank)))
        if name not in mats:
            mats[name] = (np.zeros((L, rank, n_in), np.float32), np.zeros((L, n_out, rank), np.float32))
        mats[name][0][l], mats[name][1][l] = A, B
    return rank, mats


def _stop_strings(strings):
    """One str (UTF-8) or bytes, or a sequence of them, as a list of bytes."""
    items = [strings] if isinstance(strings, (str, bytes, bytearray)) else list(strings)
    enc = []
    for s in items:
        if isinstance(s, str):
            enc.append(s.encode("utf-8"))
        elif isinstance(s, (bytes, bytearray)):
            enc.append(bytes(s))
        else:
            raise EngineError("stop strings are str or bytes, not %r" % type(s).__name__)
    return enc


def stop_set_bytes(strings):
    """A stop set as rwkv_b200_stop_set_add takes it: (string_start [n + 1] uint64, bytes uint8). strings: one str
    (UTF-8) or bytes, or a sequence of them."""
    enc = _stop_strings(strings)
    start = np.ascontiguousarray(np.cumsum([0] + [len(s) for s in enc]), dtype=np.uint64)
    return start, np.frombuffer(b"".join(enc) or b"\0", np.uint8).copy()


def stop_spec(spec, S, what):
    """stop_strings of a generate call as (set ids [S], start states [S]): one set id for every stream, or one entry per
    stream: an id, (id, start_state) or None."""
    items = [spec] * S if isinstance(spec, (int, np.integer)) else list(spec)
    if len(items) != S:
        raise EngineError("%s: %d stop_strings entries for %d streams" % (what, len(items), S))
    pairs = [(NO_STOP_SET, 0) if c is None else (int(c[0]), int(c[1])) if isinstance(c, (tuple, list)) else (int(c), 0)
             for c in items]
    return (np.ascontiguousarray([c for c, _ in pairs], np.uint64), np.ascontiguousarray([q for _, q in pairs], np.uint64))


def stop_prefixes(strings):
    """The match states of a stop set (include/rwkv_b200.h, "Stop strings"): state q stands for prefixes[q], the q-th
    distinct prefix of the strings in order of first appearance (the empty prefix first)."""
    out, seen = [b""], {b""}
    for s in _stop_strings(strings):
        for k in range(1, len(s) + 1):
            if s[:k] not in seen:
                seen.add(s[:k])
                out.append(s[:k])
    return out


def stop_match(strings, chunks, state=0):
    """The stop-string rule restated on the host: walk chunks (the bytes of each emitted token, in order) from match
    state `state`. Returns (j, hit, tail, state): j the index of the first chunk in which a string ends (None if none
    does), hit the index of that string (the lowest among those ending at the same byte), tail the bytes of chunk j
    after it, and the match state after the last byte walked."""
    enc = _stop_strings(strings)
    pre = stop_prefixes(enc)
    index = {p: q for q, p in enumerate(pre)}
    keep = max(len(s) for s in enc)
    text = pre[state]
    for j, chunk in enumerate(chunks):
        chunk = bytes(chunk)
        for i in range(len(chunk)):
            text = (text + chunk[i:i + 1])[-keep:]
            ends = [k for k, s in enumerate(enc) if text.endswith(s)]
            if ends:
                return j, ends[0], len(chunk) - i - 1, index[_longest_prefix(text, index)]
    return None, None, 0, index[_longest_prefix(text, index)]


def _longest_prefix(text, index):
    for k in range(len(text) + 1):
        if text[k:] in index:
            return text[k:]


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


def _gen_args(streams, max_new, budgets, stop, overrides, u, slots=None):
    """The arguments the generate_streams calls share: S; the ten after the model handle (slots, first tokens, S,
    max_new, budgets, stops, n_stop, override tokens, values, n_override); the three after the sampler or temperature
    (uniforms, emitted tokens, lengths); and the emitted tokens and lengths arrays they fill. slots: every stream's slots
    flattened, when a stream names several (generate_speculative); None: each stream's one slot."""
    S = len(streams)
    if slots is None:
        slots = [int(s) for s, _ in streams]
    slots = np.ascontiguousarray(slots, dtype=np.uint64)
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
    out, lens = np.zeros((S, max_new), np.uint64), np.zeros(S, np.uint64)
    P = ctypes.c_ulonglong
    lead = (_ptr(slots, P), _ptr(first, P), S, max_new, _ptr(bud, P), _ptr(stops, P), len(stops), _ptr(otok, P),
            _ptr(oval, ctypes.c_float), len(otok))
    return S, lead, (_ptr(us, ctypes.c_double), _ptr(out, P), _ptr(lens, P)), out, lens


_LOGPROB_MODES = {None: LOGPROBS_RAW, "raw": LOGPROBS_RAW, "processed": LOGPROBS_PROCESSED}


def _logprob_mode(logprobs, what):
    if logprobs not in _LOGPROB_MODES:
        raise EngineError("%s: logprobs must be 'raw' or 'processed', not %r" % (what, logprobs))
    return _LOGPROB_MODES[logprobs]


def _scored_args(S, max_new, logprobs, top_n, constraints, what):
    """The log-probability and automaton arguments of a call of S streams (logprobs None: no scoring; constraints None:
    no automata): the six from logprob_mode to top_logprobs_out, the three from constraint_ids to states_out, and
    result(s, n) -> the dict of "state" and the logprob fields of stream s with n emitted tokens."""
    P = ctypes.c_ulonglong
    lp = ranks = top_tok = top_lp = None
    if logprobs is not None:
        lp = np.empty((S, max_new), np.float64)
        ranks = np.empty((S, max_new), np.uint64)
        if top_n > 0:
            top_tok = np.empty((S, max_new, top_n), np.uint64)
            top_lp = np.empty((S, max_new, top_n), np.float64)
    ids = starts = states = None
    if constraints is not None:
        spec = [constraints] * S if isinstance(constraints, (int, np.integer)) else list(constraints)
        if len(spec) != S:
            raise EngineError("%s: %d constraints for %d streams" % (what, len(spec), S))
        pairs = [(NO_CONSTRAINT, 0) if c is None else (int(c[0]), int(c[1])) if isinstance(c, (tuple, list))
                 else (int(c), 0) for c in spec]
        ids = np.ascontiguousarray([c for c, _ in pairs], np.uint64)
        starts = np.ascontiguousarray([q for _, q in pairs], np.uint64)
        states = np.zeros(S, np.uint64)
    lp_args = (_LOGPROB_MODES[logprobs], int(top_n), _ptr(lp, ctypes.c_double), _ptr(ranks, P), _ptr(top_tok, P),
               _ptr(top_lp, ctypes.c_double))
    c_args = (_ptr(ids, P), _ptr(starts, P), _ptr(states, P))

    def result(s, n):
        d = {}
        if constraints is not None:
            d["state"] = int(states[s]) if ids[s] != np.uint64(NO_CONSTRAINT) else None
        if lp is not None:
            d["logprobs"], d["ranks"] = lp[s, :n].copy(), ranks[s, :n].copy()
            if top_n > 0:
                d["top_tokens"], d["top_logprobs"] = top_tok[s, :n].copy(), top_lp[s, :n].copy()
        return d
    return lp_args, c_args, result


def lookup_drafts(history, draft, ngram):
    """The k = draft prompt-lookup drafts of rwkv_b200_generate_streams_speculative for a history h (context, first token,
    tokens emitted so far): for n = ngram down to 1 with n < len(h), the largest j <= len(h) - n - 1 with
    h[j:j+n] == h[-n:]; the first such n proposes h[j+n : j+n+draft], padded with its last token; no match: h[-1]."""
    h = [int(x) for x in history]
    L = len(h)
    for n in range(ngram, 0, -1):
        if n >= L:
            continue
        tail = h[L - n:]
        for j in range(L - n - 1, -1, -1):
            if h[j:j + n] == tail:
                prop = h[j + n:min(j + n + draft, L)]
                return prop + [prop[-1]] * (draft - len(prop))
    return [h[-1]] * draft


def speculative_steps(context, first, tokens, draft, ngram):
    """The steps_out a speculative call reports for a stream that emitted `tokens`: each step emits p_0 and then p_i
    while draft i equals p_(i-1), so the emitted tokens and the draft rule decide where every step ends."""
    h = [int(x) for x in context] + [int(first)]
    t = [int(x) for x in tokens]
    pos = steps = 0
    while pos < len(t):
        d = lookup_drafts(h, draft, ngram)
        c = 1
        while c <= draft and pos + c < len(t) and d[c - 1] == t[pos + c - 1]:
            c += 1
        h += t[pos:pos + c]
        pos += c
        steps += 1
    return steps


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
        "rwkv_b200_generate_streams_speculative": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                         c.POINTER(Sampler), pdbl, pull, pull, c.c_uint, c.c_uint, pull,
                                                         pull, pull]),
        "rwkv_b200_batcher_open": (i32, [vp, ull, ull, c.POINTER(vp)]),
        "rwkv_b200_batcher_submit": (i32, [vp, c.POINTER(Request), pull]),
        "rwkv_b200_batcher_submit_ex": (i32, [vp, c.POINTER(Request), c.POINTER(RequestEx), pull]),
        "rwkv_b200_batcher_run": (i32, [vp, ull, pull]),
        "rwkv_b200_batcher_read": (i32, [vp, ull, pull, ull, pull, c.POINTER(i32)]),
        "rwkv_b200_batcher_read_ex": (i32, [vp, ull, ull, pull, pdbl, pull, pull, pdbl, pull, pull, c.POINTER(i32)]),
        "rwkv_b200_token_bytes_set": (i32, [vp, pull, c.POINTER(c.c_ubyte)]),
        "rwkv_b200_stop_set_add": (i32, [vp, ull, pull, c.POINTER(c.c_ubyte), pull]),
        "rwkv_b200_stop_set_remove": (i32, [vp, ull]),
        "rwkv_b200_generate_streams_stop": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                  c.POINTER(Sampler), pdbl, pull, pull, i32, c.c_uint, pdbl, pull, pull,
                                                  pdbl, pull, pull, pull, c.POINTER(StopRequest)]),
        "rwkv_b200_generate_streams_guided": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                    c.POINTER(Sampler), pdbl, pull, pull, i32, c.c_uint, pdbl, pull, pull,
                                                    pdbl, pull, pull, pull, c.POINTER(StopRequest), c.POINTER(Guidance)]),
        "rwkv_b200_generate_streams_speculative_stop": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                              c.POINTER(Sampler), pdbl, pull, pull, c.c_uint, c.c_uint,
                                                              pull, pull, pull, c.POINTER(StopRequest)]),
        "rwkv_b200_generate_streams_speculative_constrained": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt,
                                                                     ull, c.POINTER(Sampler), pdbl, pull, pull, c.c_uint,
                                                                     c.c_uint, pull, pull, pull, i32, c.c_uint, pdbl, pull,
                                                                     pull, pdbl, pull, pull, pull, c.POINTER(StopRequest)]),
        "rwkv_b200_generate_streams_drafted": (i32, [vp, pull, pull, ull, ull, pull, pull, ull, pull, pflt, ull,
                                                     c.POINTER(Sampler), pdbl, pull, pull, c.c_uint, c.POINTER(Drafter),
                                                     pull, i32, c.c_uint, pdbl, pull, pull, pdbl, pull, pull, pull,
                                                     c.POINTER(StopRequest)]),
        "rwkv_b200_batcher_submit_stop": (i32, [vp, c.POINTER(Request), c.POINTER(RequestEx), ull, ull, pull]),
        "rwkv_b200_batcher_read_stop": (i32, [vp, ull, pull, pull, pull]),
        "rwkv_b200_batcher_submit_spec": (i32, [vp, c.POINTER(Request), c.POINTER(RequestEx), ull, ull,
                                                c.POINTER(RequestSpec), pull]),
        "rwkv_b200_batcher_read_spec": (i32, [vp, ull, pull]),
        "rwkv_b200_batcher_cancel": (i32, [vp, ull]),
        "rwkv_b200_batcher_release": (i32, [vp, ull]),
        "rwkv_b200_batcher_close": (None, [vp]),
        "rwkv_b200_slot_zero": (i32, [vp, ull]),
        "rwkv_b200_slot_copy": (i32, [vp, ull, ull]),
        "rwkv_b200_slot_upload": (i32, [vp, ull, pdbl, pdbl, pdbl, pdbl, pdbl]),
        "rwkv_b200_slot_download": (i32, [vp, ull, pdbl, pdbl, pdbl, pdbl, pdbl]),
        "rwkv_b200_index_create": (i32, [vp, ull, ull, ull, pull]),
        "rwkv_b200_index_free": (i32, [vp, ull]),
        "rwkv_b200_index_add_slots": (i32, [vp, ull, pull, ull, pull]),
        "rwkv_b200_index_upload": (i32, [vp, ull, pdbl, ull, pull]),
        "rwkv_b200_index_download": (i32, [vp, ull, pull, ull, pdbl]),
        "rwkv_b200_index_remove": (i32, [vp, ull, pull, ull]),
        "rwkv_b200_index_search": (i32, [vp, ull, pull, ull, i32, c.c_uint, pull, pdbl, pdbl, pull]),
        "rwkv_b200_adapter_add": (i32, [vp, c.POINTER(Adapter), pull]),
        "rwkv_b200_adapter_remove": (i32, [vp, ull]),
        "rwkv_b200_slot_adapter": (i32, [vp, ull, ull]),
        "rwkv_b200_prefix_cache_open": (i32, [vp, ull, ull, c.POINTER(vp)]),
        "rwkv_b200_prefix_cache_close": (i32, [vp]),
        "rwkv_b200_prefix_forward": (i32, [vp, pull, ull, pull, pull, ull, pflt, pull, pull]),
        "rwkv_b200_prefix_insert": (i32, [vp, ull, pull, ull]),
        "rwkv_b200_prefix_download": (i32, [vp, pull, ull, pdbl, pdbl, pdbl, pdbl]),
        "rwkv_b200_prefix_clear": (i32, [vp]),
        "rwkv_b200_batcher_submit_prefix": (i32, [vp, c.POINTER(Request), c.POINTER(RequestEx), ull, ull,
                                                  c.POINTER(RequestSpec), vp, pull]),
        "rwkv_b200_batcher_read_prefix": (i32, [vp, ull, pull]),
        "rwkv_b200_prefix_stats": (i32, [vp, c.POINTER(PrefixStats)]),
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
                         logprobs=None, top_n=0, constraints=None, stop_strings=None, guidance=None):
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
        logprobs is given. Like logprobs, constraints need sampling=... or the arg-max (not the typical sampler).
        stop_strings: one id of add_stop_set for every stream, or one entry per stream: an id, (id, start_state) or None
        (rwkv_b200_generate_streams_stop: a stream ends after the token whose bytes complete one of its set's strings).
        Then it returns one dict per stream with "tokens", "stop_hit" (the index of the matched string, or None),
        "stop_tail" (bytes of the last token after the match) and "stop_state" (the final match state, None without a
        set), plus the logprob and constraint fields when those are given. It needs sampling=... or the arg-max too.
        guidance: classifier-free guidance, one entry per stream: None, or (slot, first_token, scale)
        (rwkv_b200_generate_streams_guided). Each step also runs the guidance slot on first_token, then on the token the
        stream emitted last, and the stream picks from c + (scale - 1) * (c - q) (guide_rows) of its own row c and the
        guidance row q. The return shapes stay as above; it needs sampling=... or the arg-max too. Three uses:

            # a negative prompt: its state on slot 9, its last token fed by the call
            eng.slot_zero(9); eng.forward_streams([(9, neg[:-1])], want_logits=False)
            eng.generate_streams([(0, tok)], 64, guidance=[(9, neg[-1], 1.5)])
            # unconditional guidance: an empty context on a zeroed slot, token 0
            eng.slot_zero(9); eng.generate_streams([(0, tok)], 64, guidance=[(9, 0, 1.5)])
            # adapter contrast: slot 0 bound to a fine-tune, its copy on slot 9 to the base model
            eng.slot_copy(0, 9); eng.bind_adapter(0, ft); eng.bind_adapter(9, None)
            eng.generate_streams([(0, tok)], 64, guidance=[(9, tok, 2.0)])"""
        if logprobs is not None or constraints is not None or stop_strings is not None or guidance is not None:
            return self._generate_scored(streams, max_new, budgets, stop, overrides, temp, u, sampling, logprobs, top_n,
                                         constraints, stop_strings, guidance)
        temp = 1.0 if temp is None else temp
        S, lead, tail, out, lens = _gen_args(streams, max_new, budgets, stop, overrides, u)
        if sampling is not None:
            self._ck(self.lib.rwkv_b200_generate_streams_ex(self.h, *lead, _samplers(sampling, S), *tail),
                     "generate_streams_ex")
        else:
            self._ck(self.lib.rwkv_b200_generate_streams(self.h, *lead, temp, *tail), "generate_streams")
        return [out[s, :int(lens[s])].copy() for s in range(S)]

    def _generate_scored(self, streams, max_new, budgets, stop, overrides, temp, u, sampling, logprobs, top_n, constraints,
                         stop_strings=None, guidance=None):
        """generate_streams with logprobs, constraints, stop strings or guidance: rwkv_b200_generate_streams_guided with
        guidance, rwkv_b200_generate_streams_stop with stop strings, rwkv_b200_generate_streams_constrained with
        constraints, else rwkv_b200_generate_streams_logprobs. One dict per stream, or with guidance alone one array."""
        _logprob_mode(logprobs, "generate_streams")
        if sampling is None and (u is not None or temp is not None):
            if guidance is not None:
                raise EngineError("generate_streams: guidance needs sampling=... (or neither u nor temp, for the arg-max); "
                                  "the typical sampler does not take it")
            if stop_strings is not None:
                raise EngineError("generate_streams: stop_strings need sampling=... (or neither u nor temp, for the "
                                  "arg-max); the typical sampler does not take them")
            if constraints is not None:
                raise EngineError("generate_streams: constraints need sampling=... (or neither u nor temp, for the "
                                  "arg-max); the typical sampler does not take them")
            raise EngineError("generate_streams: logprobs need sampling=... (or neither u nor temp, for the arg-max); "
                              "the typical sampler reports no log-probabilities")
        S, lead, tail, out, lens = _gen_args(streams, max_new, budgets, stop, overrides, u)
        lp_args, cargs, scored = _scored_args(S, max_new, logprobs, top_n, constraints, "generate_streams")
        sp = _samplers(sampling, S) if sampling is not None else None
        args = (self.h, *lead, sp, *tail, *lp_args)
        if stop_strings is not None:
            sreq, sres = self._stop_request(stop_strings, S, "generate_streams")
        if guidance is not None:
            gd = _guidance(guidance, S, "generate_streams")
            self._ck(self.lib.rwkv_b200_generate_streams_guided(*args, *cargs, ctypes.byref(sreq) if stop_strings is not None
                                                                else None, ctypes.byref(gd)), "generate_streams_guided")
            if logprobs is None and constraints is None and stop_strings is None:
                return [out[s, :int(lens[s])].copy() for s in range(S)]
        elif stop_strings is not None:
            self._ck(self.lib.rwkv_b200_generate_streams_stop(*args, *cargs, ctypes.byref(sreq)), "generate_streams_stop")
        elif constraints is not None:
            self._ck(self.lib.rwkv_b200_generate_streams_constrained(*args, *cargs), "generate_streams_constrained")
        else:
            self._ck(self.lib.rwkv_b200_generate_streams_logprobs(*args), "generate_streams_logprobs")
        res = []
        for s in range(S):
            n = int(lens[s])
            d = {"tokens": out[s, :n].copy()}
            if stop_strings is not None:
                d.update(sres(s))
            d.update(scored(s, n))
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

    def add_adapter(self, weights, alpha):
        """Register a LoRA adapter and return its id; bind it to slots with bind_adapter. `weights` is a state dict or
        the path of a .pth file loaded with torch. Keys follow the RWKV-4 LoRA trainers' convention: the checkpoint's
        Linear name plus ".lora_A" [r][in] or ".lora_B" [out][r] (e.g. "blocks.3.att.key.lora_A"), for att key, value,
        receptance and output and ffn key, value and receptance. The scale is alpha / r. Only synthetic checkpoints in
        this naming have been tested. Unknown keys, mismatched ranks and wrong shapes raise ValueError; full-parameter
        tensors (time_*, ln) cannot be applied at run time: merge them with tools/convert_model.py --lora."""
        if isinstance(weights, (str, os.PathLike)):
            import torch
            weights = torch.load(weights, map_location="cpu", weights_only=True)
        rank, mats = parse_adapter(weights, self.n_layers, self.n_embed)
        d = Adapter()
        d.rank, d.scale = rank, float(alpha) / rank
        keep = []
        for k, name in enumerate(ADAPTER_MATRICES):
            if name in mats:
                A, B = (np.ascontiguousarray(x) for x in mats[name])
                keep += [A, B]
                d.A[k], d.B[k] = _ptr(A, ctypes.c_float), _ptr(B, ctypes.c_float)
        aid = ctypes.c_ulonglong()
        self._ck(self.lib.rwkv_b200_adapter_add(self.h, ctypes.byref(d), ctypes.byref(aid)), "adapter_add")
        return aid.value

    def remove_adapter(self, aid):
        self._ck(self.lib.rwkv_b200_adapter_remove(self.h, int(aid)), "adapter_remove")

    def bind_adapter(self, slot, aid):
        """Bind state slot `slot` to adapter `aid`, or unbind it with None. Every multi-stream call on the slot then
        applies the adapter (on the tensor cores); the binding stays with the slot, not with the state."""
        self._ck(self.lib.rwkv_b200_slot_adapter(self.h, int(slot), NO_ADAPTER if aid is None else int(aid)),
                 "slot_adapter")

    def remove_constraint(self, cid):
        self._ck(self.lib.rwkv_b200_constraint_remove(self.h, int(cid)), "constraint_remove")

    def add_stop_set(self, strings):
        """Upload a stop set (one str (UTF-8) or bytes, or a sequence of them) for generate_streams(stop_strings=...),
        generate_speculative and Batcher.submit; returns its id. The first set also uploads the token bytes
        (constrain.token_bytes()) that the device walks."""
        if not getattr(self, "_token_bytes", False):
            from . import constrain
            tb = constrain.token_bytes()
            start = np.ascontiguousarray(np.cumsum([0] + [len(b) for b in tb]), dtype=np.uint64)
            data = np.frombuffer(b"".join(tb), np.uint8).copy()
            self._ck(self.lib.rwkv_b200_token_bytes_set(self.h, _ptr(start, ctypes.c_ulonglong), _ptr(data, ctypes.c_ubyte)),
                     "token_bytes_set")
            self._token_bytes = True
        start, data = stop_set_bytes(strings)
        sid = ctypes.c_ulonglong()
        self._ck(self.lib.rwkv_b200_stop_set_add(self.h, len(start) - 1, _ptr(start, ctypes.c_ulonglong),
                                                 _ptr(data, ctypes.c_ubyte), ctypes.byref(sid)), "stop_set_add")
        return int(sid.value)

    def remove_stop_set(self, sid):
        self._ck(self.lib.rwkv_b200_stop_set_remove(self.h, int(sid)), "stop_set_remove")

    @staticmethod
    def _stop_request(stop_strings, S, what):
        """(StopRequest, result(s) -> dict of "stop_hit", "stop_tail", "stop_state") of stop_strings for S streams."""
        ids, starts = stop_spec(stop_strings, S, what)
        out = [np.zeros(S, np.uint64) for _ in range(3)]
        P = ctypes.c_ulonglong
        req = StopRequest(_ptr(ids, P), _ptr(starts, P), *[_ptr(a, P) for a in out])
        req._keep = (ids, starts, out)
        state, hit, tail = out

        def result(s):
            on = ids[s] != np.uint64(NO_STOP_SET)
            return {"stop_hit": int(hit[s]) - 1 if hit[s] else None, "stop_tail": int(tail[s]),
                    "stop_state": int(state[s]) if on else None}
        return req, result

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

    def generate_speculative(self, streams, max_new, draft, ngram=3, context=None, budgets=None, stop=(), overrides=None,
                             sampling=None, u=None, stop_strings=None, logprobs=None, top_n=0, constraints=None,
                             drafter=None):
        """generate_streams(sampling=...) with prompt-lookup drafts (rwkv_b200_generate_streams_speculative): the same
        tokens and first-slot states, several tokens per step where the drafts are right. streams = [(slots, first_token),
        ...], each with draft + 1 distinct slots, the first holding the conversation (the others are scratch). context:
        None, or one token list (or None) per stream of extra lookup tokens. sampling None is the arg-max. Returns one
        dict per stream: "tokens" (uint64) and "steps" (the steps that emitted a token). stop_strings as in
        generate_streams (rwkv_b200_generate_streams_speculative_stop) adds "stop_hit", "stop_tail" and "stop_state".
        logprobs, top_n and constraints as in generate_streams (rwkv_b200_generate_streams_speculative_constrained) add
        "logprobs", "ranks", "top_tokens", "top_logprobs" and "state", bit for bit generate_streams' values.
        drafter = (draft_engine, draft_slots): the drafts come from a second, smaller model of the same vocabulary
        (rwkv_b200_generate_streams_drafted) instead of prompt lookup; draft_slots holds one (D0, D1) pair of
        draft_engine's slots per stream, D0 primed with the same tokens as the stream's first slot, D1 scratch. D0 ends
        holding the tokens the first slot absorbed. It takes neither context nor ngram; the results are as above."""
        if drafter is not None:
            deng, dslots = drafter
            if context is not None or ngram != 3:
                raise EngineError("generate_speculative: a drafter takes neither context nor ngram")
            if deng is self:
                raise EngineError("generate_speculative: the draft engine is the target engine")
            if len(dslots) != len(streams) or any(len(pair) != 2 for pair in dslots):
                raise EngineError("generate_speculative: the drafter needs one (D0, D1) slot pair per stream (%d)"
                                  % len(streams))
        extended = logprobs is not None or constraints is not None
        if extended:
            _logprob_mode(logprobs, "generate_speculative")
        if any(len(slots) != draft + 1 for slots, _ in streams):
            raise EngineError("generate_speculative: every stream needs draft + 1 = %d slots" % (draft + 1))
        S, lead, tail, out, lens = _gen_args(streams, max_new, budgets, stop, overrides, u,
                                             slots=[int(s) for sl, _ in streams for s in sl])
        steps = np.zeros(S, np.uint64)
        cstart = ctx = None
        if context is not None:
            if len(context) != S:
                raise EngineError("generate_speculative: %d contexts for %d streams" % (len(context), S))
            seqs = [[int(x) for x in (c if c is not None else ())] for c in context]
            cstart = np.ascontiguousarray(np.cumsum([0] + [len(c) for c in seqs]), dtype=np.uint64)
            ctx = np.ascontiguousarray([x for c in seqs for x in c], dtype=np.uint64)
        if extended or drafter is not None:
            lp_args, cargs, scored = _scored_args(S, max_new, logprobs, top_n, constraints, "generate_speculative")
        sp = _samplers(sampling, S) if sampling is not None else None
        P = ctypes.c_ulonglong
        args = (self.h, *lead, sp, *tail, int(draft), int(ngram), _ptr(cstart, P), _ptr(ctx, P), _ptr(steps, P))
        sreq, sres = self._stop_request(stop_strings, S, "generate_speculative") if stop_strings is not None else (None, None)
        sq = ctypes.byref(sreq) if sreq is not None else None
        if drafter is not None:
            dsl = np.ascontiguousarray([int(x) for pair in dslots for x in pair], dtype=np.uint64)
            dr = Drafter(deng.h.value if deng.h is not None else None, _ptr(dsl, P))
            self._ck(self.lib.rwkv_b200_generate_streams_drafted(self.h, *lead, sp, *tail, int(draft), ctypes.byref(dr),
                                                                 _ptr(steps, P), *lp_args, *cargs, sq),
                     "generate_streams_drafted")
        # the narrowest entry point that has the features asked for
        elif extended:
            name, more = "generate_streams_speculative_constrained", (*lp_args, *cargs, sq)
        elif sq is not None:
            name, more = "generate_streams_speculative_stop", (sq,)
        else:
            name, more = "generate_streams_speculative", ()
        if drafter is None:
            self._ck(getattr(self.lib, "rwkv_b200_" + name)(*args, *more), name)
        res = []
        for s in range(S):
            n = int(lens[s])
            d = {"tokens": out[s, :n].copy(), "steps": int(steps[s])}
            if sres is not None:
                d.update(sres(s))
            if extended:
                d.update(scored(s, n))
            res.append(d)
        return res

    def batcher(self, rows, prefill_tokens):
        """Continuous batching (include/rwkv_b200.h, rwkv_b200_batcher_open): a Batcher with at most `rows` admitted
        requests and `prefill_tokens` prompt tokens per step."""
        return Batcher(self, rows, prefill_tokens)

    def prefix_cache(self, capacity, block=64):
        """A PrefixCache of `capacity` entries that snapshots every `block` tokens (include/rwkv_b200.h, "Prefix state
        cache")."""
        return PrefixCache(self, capacity, block)

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

    # -- state indexes ---------------------------------------------------------------------
    def create_index(self, capacity, layers=None):
        """A StateIndex of `capacity` entries (include/rwkv_b200.h, "State indexes") over `layers`: None for every
        layer, else a range of consecutive layers."""
        return StateIndex(self, capacity, layers)

    def embed(self, docs, slots, index):
        """The vectordb loop in ragged passes: run each document (a list of >= 1 token ids) from a zeroed slot of `slots`
        and add its final state to `index`. The documents share forward_streams calls of at most max_gpt tokens (state
        only; a document may span calls), a slot is reused once its document has been added, and the ids of the
        documents are returned in document order."""
        seqs = [np.atleast_1d(np.asarray(d, dtype=np.uint64)) for d in docs]
        free = [int(s) for s in slots]
        if not free:
            raise EngineError("embed: no slots")
        if len(set(free)) != len(free):
            raise EngineError("embed: a slot appears twice")
        for i, t in enumerate(seqs):
            if t.ndim != 1 or len(t) == 0:
                raise EngineError("embed: document %d has no tokens" % i)
        ids = [None] * len(seqs)
        pending = list(range(len(seqs)))[::-1]
        active = []  # [slot, document, tokens already run], in the order the documents started
        while pending or active:
            while free and pending:
                slot, d = free.pop(0), pending.pop()
                self.slot_zero(slot)
                active.append([slot, d, 0])
            call, room = [], self.max_gpt
            for a in active:
                take = min(len(seqs[a[1]]) - a[2], room)
                if take == 0:
                    break
                call.append((a[0], seqs[a[1]][a[2]:a[2] + take]))
                a[2] += take
                room -= take
            self.forward_streams(call, want_logits=False)
            done = [a for a in active if a[2] == len(seqs[a[1]])]
            if done:
                got = index.add([a[0] for a in done])
                for a, e in zip(done, got):
                    ids[a[1]] = int(e)
                    free.append(a[0])
                active = [a for a in active if a[2] < len(seqs[a[1]])]
        return ids

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


class Batcher:
    """Continuous batching on one Engine (include/rwkv_b200.h, "Continuous batching"): submit requests at any time
    between runs, run them in groups of 16 steps, read each request's tokens as they grow. A context manager; close()
    frees it (the engine keeps at most one open batcher)."""

    def __init__(self, engine, rows, prefill_tokens):
        self.engine, self.lib = engine, engine.lib
        h = ctypes.c_void_p()
        engine._ck(self.lib.rwkv_b200_batcher_open(engine.h, int(rows), int(prefill_tokens), ctypes.byref(h)),
                   "batcher_open")
        self.h = h
        self._ext = {}  # id -> (top_n or None without log-probabilities, constrained) of requests sent through submit_ex
        self._stop = set()  # ids of requests with a stop set
        self._spec = set()  # ids of requests with speculation
        self._prefix = set()  # ids of requests with a prefix cache

    def submit(self, slot, prompt, max_new, sampling=None, u=None, stop=(), overrides=None, constraint=None, logprobs=None,
               top_n=0, stop_strings=None, draft=0, spare_slots=(), ngram=3, context=None, prefix_cache=None):
        """Queue a request on state slot `slot`: prompt (>= 1 token ids), up to max_new new tokens, a Sampler or dict
        (None: arg-max), u: max_new uniforms in [0, 1) (None only at temperature 0), stop: this request's stop tokens.
        overrides = {token: logit value} as in generate_streams; constraint: an id of Engine.add_constraint, or (id,
        start_state); logprobs = "raw" or "processed" scores every emitted token, with top_n top entries (read them with
        result); stop_strings: an id of Engine.add_stop_set, or (id, start_state). draft > 0 speculates with
        prompt-lookup drafts (rwkv_b200_batcher_submit_spec): spare_slots are its draft scratch slots, ngram the longest
        n-gram looked up and context extra lookup tokens before the prompt; the tokens are those without speculation and
        result adds "steps". prefix_cache: a PrefixCache of the engine (rwkv_b200_batcher_submit_prefix): the request
        starts from the zero state, restores its longest cached prompt prefix at admission and snapshots its prefill;
        result adds "cached". Returns its id. Every array is copied."""
        if int(draft) < 0:
            raise EngineError("batcher.submit: draft %d < 0" % int(draft))
        spares = np.ascontiguousarray([int(z) for z in spare_slots], dtype=np.uint64)
        if len(spares) != int(draft):
            raise EngineError("batcher.submit: draft = %d needs %d spare slots, got %d" % (int(draft), int(draft),
                                                                                         len(spares)))
        ctx = np.ascontiguousarray([int(t) for t in (context if context is not None else ())], dtype=np.uint64)
        if len(ctx) and not draft:
            raise EngineError("batcher.submit: a lookup context needs draft > 0")
        sp = _samplers(sampling if sampling is not None else Sampler(temperature=0.0), 1)[0]
        pr = np.ascontiguousarray(np.atleast_1d(np.asarray(prompt, dtype=np.uint64)))
        st = np.ascontiguousarray(list(stop), dtype=np.uint64)
        us = np.ascontiguousarray(u, dtype=np.float64) if u is not None else None
        if us is not None and us.shape != (int(max_new),):
            raise EngineError("batcher.submit: u has shape %s, expected (%d,)" % (us.shape, int(max_new)))
        P = ctypes.c_ulonglong
        req = Request(int(slot), _ptr(pr, P), len(pr), int(max_new), sp, _ptr(us, ctypes.c_double), _ptr(st, P), len(st))
        extended = overrides is not None or constraint is not None or logprobs is not None
        x = None
        if extended:
            mode = _logprob_mode(logprobs, "batcher.submit")
            ovr = dict(overrides or {})
            otok = np.ascontiguousarray(list(ovr.keys()), dtype=np.uint64)
            oval = np.ascontiguousarray(list(ovr.values()), dtype=np.float32)
            cid, q0 = NO_CONSTRAINT, 0
            if constraint is not None:
                cid, q0 = ((int(constraint[0]), int(constraint[1])) if isinstance(constraint, (tuple, list))
                           else (int(constraint), 0))
            x = RequestEx(_ptr(otok, P), _ptr(oval, ctypes.c_float), len(otok), cid, q0, 1 if logprobs is not None else 0,
                          mode, int(top_n))
        sid, s0 = NO_STOP_SET, 0
        if stop_strings is not None:
            ids, starts = stop_spec([stop_strings], 1, "batcher.submit")
            sid, s0 = int(ids[0]), int(starts[0])
        rid = ctypes.c_ulonglong()
        xr = ctypes.byref(x) if x is not None else None
        # the entry point of what the request uses: each one is exactly the next one's call with its extension NULL
        spec = RequestSpec(_ptr(spares, P), int(draft), int(ngram), _ptr(ctx, P) if len(ctx) else None, len(ctx))
        if prefix_cache is not None:
            rc = self.lib.rwkv_b200_batcher_submit_prefix(self.h, ctypes.byref(req), xr, sid, s0,
                                                          ctypes.byref(spec) if draft else None,
                                                          prefix_cache._handle("batcher.submit"), ctypes.byref(rid))
        elif draft:
            rc = self.lib.rwkv_b200_batcher_submit_spec(self.h, ctypes.byref(req), xr, sid, s0, ctypes.byref(spec),
                                                        ctypes.byref(rid))
        elif stop_strings is not None:
            rc = self.lib.rwkv_b200_batcher_submit_stop(self.h, ctypes.byref(req), xr, sid, s0, ctypes.byref(rid))
        elif extended:
            rc = self.lib.rwkv_b200_batcher_submit_ex(self.h, ctypes.byref(req), xr, ctypes.byref(rid))
        else:
            rc = self.lib.rwkv_b200_batcher_submit(self.h, ctypes.byref(req), ctypes.byref(rid))
        self.engine._ck(rc, "batcher_submit")
        rid = int(rid.value)
        if stop_strings is not None:
            self._stop.add(rid)
        if extended:
            self._ext[rid] = (int(top_n) if logprobs is not None else None, constraint is not None)
        if draft:
            self._spec.add(rid)
        if prefix_cache is not None:
            self._prefix.add(rid)
        return rid

    def run(self, max_steps):
        """Run up to max_steps steps (groups of 16); returns the steps run (fewer when everything has finished)."""
        n = ctypes.c_ulonglong()
        self.engine._ck(self.lib.rwkv_b200_batcher_run(self.h, int(max_steps), ctypes.byref(n)), "batcher_run")
        return int(n.value)

    def read(self, rid):
        """(tokens emitted so far as np.uint64, status): status is one of REQ_STATUS."""
        n, status = ctypes.c_ulonglong(), ctypes.c_int()
        self.engine._ck(self.lib.rwkv_b200_batcher_read(self.h, int(rid), None, 0, ctypes.byref(n), ctypes.byref(status)),
                        "batcher_read")
        out = np.zeros(int(n.value), np.uint64)
        self.engine._ck(self.lib.rwkv_b200_batcher_read(self.h, int(rid), _ptr(out, ctypes.c_ulonglong), len(out), None, None),
                        "batcher_read")
        return out, REQ_STATUS[status.value]

    def result(self, rid):
        """Everything a request has produced so far, as a dict: "tokens" (np.uint64) and "status" (one of REQ_STATUS);
        with logprobs "logprobs" (float64) and "ranks" (uint64), and with top_n > 0 "top_tokens" / "top_logprobs"
        [len][top_n], as generate_streams(logprobs=...) returns them; with a constraint "state" (the automaton's
        current state); with a stop set "stop_hit", "stop_tail" and "stop_state" as generate_streams(stop_strings=...)
        returns them; with speculation "steps" (the steps that emitted a token)."""
        top_n, constrained = self._ext.get(int(rid), (None, False))
        n, status = ctypes.c_ulonglong(), ctypes.c_int()
        self.engine._ck(self.lib.rwkv_b200_batcher_read(self.h, int(rid), None, 0, ctypes.byref(n), ctypes.byref(status)),
                        "batcher_read")
        L = int(n.value)
        toks = np.zeros(L, np.uint64)
        lp = np.zeros(L, np.float64) if top_n is not None else None
        ranks = np.zeros(L, np.uint64) if top_n is not None else None
        top_tok = np.zeros((L, top_n), np.uint64) if top_n else None
        top_lp = np.zeros((L, top_n), np.float64) if top_n else None
        state = ctypes.c_ulonglong()
        P, D = ctypes.c_ulonglong, ctypes.c_double
        self.engine._ck(self.lib.rwkv_b200_batcher_read_ex(self.h, int(rid), L, _ptr(toks, P), _ptr(lp, D), _ptr(ranks, P),
                                                           _ptr(top_tok, P), _ptr(top_lp, D), ctypes.byref(state), None,
                                                           None), "batcher_read_ex")
        d = {"tokens": toks, "status": REQ_STATUS[status.value]}
        if top_n is not None:
            d["logprobs"], d["ranks"] = lp, ranks
            if top_n:
                d["top_tokens"], d["top_logprobs"] = top_tok, top_lp
        if constrained:
            d["state"] = int(state.value)
        if int(rid) in self._stop:
            hit, tail, mstate = ctypes.c_ulonglong(), ctypes.c_ulonglong(), ctypes.c_ulonglong()
            self.engine._ck(self.lib.rwkv_b200_batcher_read_stop(self.h, int(rid), ctypes.byref(hit), ctypes.byref(tail),
                                                                 ctypes.byref(mstate)), "batcher_read_stop")
            d.update(stop_hit=int(hit.value) - 1 if hit.value else None, stop_tail=int(tail.value),
                     stop_state=int(mstate.value))
        if int(rid) in self._spec:
            steps = ctypes.c_ulonglong()
            self.engine._ck(self.lib.rwkv_b200_batcher_read_spec(self.h, int(rid), ctypes.byref(steps)), "batcher_read_spec")
            d["steps"] = int(steps.value)
        if int(rid) in self._prefix:
            cached = ctypes.c_ulonglong()
            self.engine._ck(self.lib.rwkv_b200_batcher_read_prefix(self.h, int(rid), ctypes.byref(cached)),
                            "batcher_read_prefix")
            d["cached"] = int(cached.value)
        return d

    def cancel(self, rid):
        self.engine._ck(self.lib.rwkv_b200_batcher_cancel(self.h, int(rid)), "batcher_cancel")

    def release(self, rid):
        self.engine._ck(self.lib.rwkv_b200_batcher_release(self.h, int(rid)), "batcher_release")
        self._ext.pop(int(rid), None)
        self._stop.discard(int(rid))
        self._spec.discard(int(rid))

    def close(self):
        if getattr(self, "h", None) and getattr(self.engine, "h", None):
            self.lib.rwkv_b200_batcher_close(self.h)
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class StateIndex:
    """An index of state vectors in HBM (include/rwkv_b200.h, "State indexes"): each entry is a slot's dd array over
    the index's layers, D = n_layers * n_embed float64 elements. Entries get ids 0, 1, 2, ... in the order they are
    added; removed entries are never returned again. A context manager; close() frees it."""

    def __init__(self, engine, capacity, layers=None):
        self.engine, self.lib = engine, engine.lib
        if layers is None:
            layers = range(engine.n_layers)
        layers = list(layers)
        if not layers or layers != list(range(layers[0], layers[0] + len(layers))):
            raise EngineError("create_index: layers must be a non-empty range of consecutive layers")
        self.layer_begin, self.n_layers = int(layers[0]), len(layers)
        self.D = self.n_layers * engine.n_embed
        self.h = None
        iid = ctypes.c_ulonglong()
        engine._ck(self.lib.rwkv_b200_index_create(engine.h, self.layer_begin, self.n_layers, int(capacity),
                                                   ctypes.byref(iid)), "index_create")
        self.h = int(iid.value)

    @staticmethod
    def _ids(ids):
        return np.ascontiguousarray(np.atleast_1d(np.asarray(ids, dtype=np.uint64)))

    def add(self, slots):
        """Append the vectors of state slots (a device-to-device copy); returns their ids."""
        s = self._ids(slots)
        out = np.zeros(len(s), np.uint64)
        self.engine._ck(self.lib.rwkv_b200_index_add_slots(self.engine.h, self.h, _ptr(s, ctypes.c_ulonglong), len(s),
                                                           _ptr(out, ctypes.c_ulonglong)), "index_add_slots")
        return out

    def upload(self, vectors):
        """Append vectors [n][D] (float64, finite); returns their ids."""
        v = np.ascontiguousarray(vectors, dtype=np.float64)
        if v.ndim == 1:
            v = v[None, :]
        if v.ndim != 2 or v.shape[1] != self.D:
            raise EngineError("index upload: vectors have shape %s, expected (n, %d)" % (v.shape, self.D))
        out = np.zeros(v.shape[0], np.uint64)
        self.engine._ck(self.lib.rwkv_b200_index_upload(self.engine.h, self.h, _ptr(v, ctypes.c_double), v.shape[0],
                                                        _ptr(out, ctypes.c_ulonglong)), "index_upload")
        return out

    def vectors(self, ids):
        """The vectors of live entries, [n][D] float64."""
        e = self._ids(ids)
        out = np.empty((len(e), self.D), np.float64)
        self.engine._ck(self.lib.rwkv_b200_index_download(self.engine.h, self.h, _ptr(e, ctypes.c_ulonglong), len(e),
                                                          _ptr(out, ctypes.c_double)), "index_download")
        return out

    def remove(self, ids):
        e = self._ids(ids)
        self.engine._ck(self.lib.rwkv_b200_index_remove(self.engine.h, self.h, _ptr(e, ctypes.c_ulonglong), len(e)),
                        "index_remove")

    def search(self, query_slots, k, metric="l2"):
        """Rank the live entries for each query slot by metric "l1" or "l2": (entries [Q][k] uint64, l1 [Q][k], l2
        [Q][k], found [Q]); positions past found hold NO_ENTRY and NaN."""
        metrics = {"l1": INDEX_L1, "l2": INDEX_L2}
        if metric not in metrics:
            raise EngineError("index search: metric must be 'l1' or 'l2', not %r" % (metric,))
        q = self._ids(query_slots)
        k = int(k)
        ent = np.zeros((len(q), max(k, 0)), np.uint64)
        l1, l2 = np.zeros(ent.shape), np.zeros(ent.shape)
        found = np.zeros(len(q), np.uint64)
        P, D = ctypes.c_ulonglong, ctypes.c_double
        self.engine._ck(self.lib.rwkv_b200_index_search(self.engine.h, self.h, _ptr(q, P), len(q), metrics[metric], max(k, 0),
                                                        _ptr(ent, P), _ptr(l1, D), _ptr(l2, D), _ptr(found, P)),
                        "index_search")
        return ent, l1, l2, found

    def close(self):
        if self.h is not None and getattr(self.engine, "h", None):
            self.lib.rwkv_b200_index_free(self.engine.h, self.h)
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


PREFIX_NOT_CACHED = 2  # RWKV_B200_PREFIX_NOT_CACHED


class PrefixCache:
    """Recurrent states after token prefixes, kept on the device (include/rwkv_b200.h, "Prefix state cache"): a stream
    run through forward() starts from the zero state, restores its longest cached prefix and stores snapshots of the
    rest. A context manager; close() frees the cache."""

    def __init__(self, engine, capacity, block=64):
        self.engine, self.lib = engine, engine.lib
        self.h = None
        h = ctypes.c_void_p()
        engine._ck(self.lib.rwkv_b200_prefix_cache_open(engine.h, int(capacity), int(block), ctypes.byref(h)),
                   "prefix_cache_open")
        self.h = h

    @staticmethod
    def _tokens(tokens):
        return np.ascontiguousarray(np.atleast_1d(np.asarray(tokens, dtype=np.uint64)))

    def _handle(self, what):
        if self.h is None or not getattr(self.engine, "h", None):
            raise EngineError("%s: the prefix cache is closed" % what)
        return self.h

    def forward(self, streams, want_logits=True, want_next=False):
        """forward_streams from the zero state with cached prefixes: streams = [(slot, tokens), ...]. Returns (logits
        [S][V] | None, arg-max [S] | None, cached [S]: the tokens each stream restored)."""
        h = self._handle("prefix_forward")
        slots = np.ascontiguousarray([int(s) for s, _ in streams], dtype=np.uint64)
        seqs = [self._tokens(t) for _, t in streams]
        lens = np.ascontiguousarray([len(t) for t in seqs], dtype=np.uint64)
        toks = np.ascontiguousarray(np.concatenate(seqs) if seqs else np.zeros(0, np.uint64))
        logits = np.empty((len(seqs), VOCAB), np.float32) if want_logits else None
        nxt = np.empty(len(seqs), np.uint64) if want_next else None
        cached = np.zeros(len(seqs), np.uint64)
        P = ctypes.c_ulonglong
        self.engine._ck(self.lib.rwkv_b200_prefix_forward(h, _ptr(toks, P), len(toks), _ptr(slots, P), _ptr(lens, P),
                                                          len(seqs), _ptr(logits, ctypes.c_float), _ptr(nxt, P),
                                                          _ptr(cached, P)), "prefix_forward")
        return logits, nxt, cached

    def insert(self, slot, tokens):
        """Store slot's state as the state after `tokens` (a zeroed slot fed exactly those tokens)."""
        h = self._handle("prefix_insert")
        t = self._tokens(tokens)
        self.engine._ck(self.lib.rwkv_b200_prefix_insert(h, int(slot), _ptr(t, ctypes.c_ulonglong), len(t)),
                        "prefix_insert")

    def download(self, tokens):
        """The state of the unbound entry keyed exactly by `tokens`: a dict of xy, aa, bb, dd, or None."""
        h = self._handle("prefix_download")
        t = self._tokens(tokens)
        n = self.engine.n_layers * self.engine.n_embed
        arrs = [np.empty(n, np.float64) for _ in range(4)]
        rc = self.lib.rwkv_b200_prefix_download(h, _ptr(t, ctypes.c_ulonglong), len(t),
                                                *[_ptr(a, ctypes.c_double) for a in arrs])
        if rc == PREFIX_NOT_CACHED:
            return None
        self.engine._ck(rc, "prefix_download")
        return dict(zip(("xy", "aa", "bb", "dd"), arrs))

    def stats(self):
        h, st = self._handle("prefix_stats"), PrefixStats()
        self.engine._ck(self.lib.rwkv_b200_prefix_stats(h, ctypes.byref(st)), "prefix_stats")
        return {f: int(getattr(st, f)) for f, _ in PrefixStats._fields_}

    def clear(self):
        h = self._handle("prefix_clear")
        self.engine._ck(self.lib.rwkv_b200_prefix_clear(h), "prefix_clear")

    def close(self):
        if self.h is not None and getattr(self.engine, "h", None):
            self.engine._ck(self.lib.rwkv_b200_prefix_cache_close(self.h), "prefix_cache_close")
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
