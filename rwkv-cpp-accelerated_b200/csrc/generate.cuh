// generate.cuh — device side of rwkv_b200_generate_streams: the per-step feedback that lets many decode steps of
// many streams run without returning to the host.
//
// A call keeps one record per stream on the device (GenStream). Each step of a group is enqueued by the host with no
// synchronisation inside the group: forward (tensor-core passes or the decode kernel, row r = a live stream), then
// k_gen_override on the logits rows, the existing pick (k_argmax_rows or k_sample_typical), and k_gen_feedback, which
// appends the picked token, decides whether the stream is done and writes the next step's input. A stream that
// finishes inside a group keeps its row until the group ends but is frozen: its slot is not written again.
// generate_streams_logprobs adds k_gen_logprob (score.cuh) between the pick and k_gen_feedback.
// generate_streams_constrained adds k_gen_mask after the overrides, and k_gen_feedback advances each constrained
// stream's token automaton (GenConstraint) after appending its token. generate_streams_stop has k_gen_feedback walk each
// emitted token's bytes through the stream's stop-string automaton (GenStop) as well. The rule that appends a token and
// decides whether it ends its stream is gen_emit, over the arguments in GenEmit; k_spec_accept (speculate.cuh) emits its
// accepted tokens by the same function. generate_streams_guided adds a guidance row per guided stream after the
// streams' rows: k_gen_guide combines each pair of rows before the pick chain, and k_gen_guide_feedback feeds the
// stream's emitted token to its guidance row after k_gen_feedback.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/rwkv_b200.h"
#include "common.cuh"
#include "prefill.cuh"
#include "stopmatch.h"

namespace rk {

struct GenStream {
    unsigned long long slot;   // the stream's state slot
    unsigned long long budget; // tokens it may emit
    unsigned long long tok;    // its next input: the first token, then the last token emitted
    unsigned long long len;    // tokens emitted so far
    unsigned long long done;   // 1 after a stop token or the budget
};

// Decode-kernel step of row r: its input token and slot into the control block. A finished stream runs on the
// scratch slot, because the decode kernel always stores the state of the slot it ran on.
__global__ void k_gen_gate(const GenStream *gs, const int *row_stream, int r, unsigned long long scratch, Ctrl *ctrl) {
    const GenStream &g = gs[row_stream[r]];
    ctrl->token = g.tok;
    ctrl->slot = g.done ? scratch : g.slot;
}

// logits[r][tok[i]] = val[i] for every row, in the order given (a repeated token keeps its last value). The batcher
// gives each row its own list: with `start` set, row r applies i in [start[s], start[s + 1]) of its stream s =
// row_stream[r] (n is not read); start == nullptr: i in [0, n) for every row.
__global__ void k_gen_override(float *logits, int V, int rows, const unsigned long long *tok, const float *val, int n,
                               const int *row_stream = nullptr, const unsigned long long *start = nullptr) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    unsigned long long i0 = 0, i1 = (unsigned long long)n;
    if (start) {
        const int s = row_stream[r];
        i0 = start[s];
        i1 = start[s + 1];
    }
    for (unsigned long long i = i0; i < i1; ++i) logits[(size_t)r * V + tok[i]] = val[i];
}

// A stream's token automaton (include/rwkv_b200.h, rwkv_b200_constraint_add) and its current state. State q's edges are
// tok[start[q] .. start[q + 1]) (ascending) with targets next[..]; mask[q] has bit v set when token v has an edge out of
// q. mask == nullptr: the stream has no constraint.
constexpr int kMaskWords = (int)((RWKV_B200_VOCAB + 31) / 32); // u32 words of one state's allow mask
struct GenConstraint {
    const unsigned long long *start; // [n_states + 1]
    const uint32_t *tok, *next;      // [n_edges]
    const uint32_t *mask;            // [n_states][kMaskWords]
    unsigned long long state;
};

// No state: a missing edge, and the per-row state of a row that is not masked (k_gen_mask's row_state).
constexpr unsigned long long kNoState = ~0ull;
// The row_state of a batcher row that is not speculative: masked by its stream's record, as without row_state.
constexpr unsigned long long kStreamState = ~0ull - 1;

// The target of token tok's edge out of state q, or kNoState when q has no edge for tok: a binary search over q's
// ascending edge tokens.
__device__ __forceinline__ unsigned long long gen_edge(const GenConstraint &c, unsigned long long q, unsigned long long tok) {
    const unsigned long long end = c.start[q + 1];
    unsigned long long lo = c.start[q], hi = end;
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) / 2;
        if (c.tok[mid] < tok) lo = mid + 1;
        else hi = mid;
    }
    return lo < end && c.tok[lo] == tok ? (unsigned long long)c.next[lo] : kNoState;
}

// Advance a constrained stream's automaton by its emitted token tok; true when that ends the stream: the new state has
// no edges (complete), or tok has no edge. The mask makes a missing edge impossible unless the pick broke its contract:
// the first one is recorded in fault {s + 1, token, state} for the host.
__device__ __forceinline__ bool gen_constraint_step(GenConstraint &c, unsigned long long tok, int s, unsigned long long *fault) {
    const unsigned long long q = c.state, q2 = gen_edge(c, q, tok);
    if (q2 != kNoState) {
        c.state = q2;
        return c.start[q2] == c.start[q2 + 1];
    }
    if (atomicCAS(fault, 0ull, (unsigned long long)s + 1) == 0ull) {
        fault[1] = tok;
        fault[2] = q;
    }
    return true;
}

// logits[r][v] = -inf for every token v without an edge out of the current state of row r's stream. Grid
// (ceil(V / kMaskThreads), rows), one thread per token. Unconstrained and finished streams are left alone: a finished
// stream may sit in a state without edges, and masking its row would leave the pick no finite value. With row_state
// (speculative generation), row r is masked by state row_state[r] of its stream's automaton instead, and left alone
// where that is kNoState; where it is kStreamState (a batcher's one-token lane) the row follows the rule without it.
constexpr int kMaskThreads = 256;
__global__ void __launch_bounds__(kMaskThreads) k_gen_mask(float *logits, int V, const GenStream *gs, const int *row_stream,
                                                           const GenConstraint *gc,
                                                           const unsigned long long *row_state = nullptr) {
    const int r = blockIdx.y, s = row_stream[r];
    const GenConstraint &c = gc[s];
    unsigned long long q = row_state ? row_state[r] : kStreamState;
    if (q == kNoState) return;
    if (q == kStreamState) {
        if (!c.mask || gs[s].done) return;
        q = c.state;
    }
    const int v = blockIdx.x * kMaskThreads + threadIdx.x;
    if (v >= V) return;
    if (!((c.mask[q * kMaskWords + (v >> 5)] >> (v & 31)) & 1u)) logits[(size_t)r * V + v] = -INFINITY;
}

// A stream's stop set (include/rwkv_b200.h, rwkv_b200_stop_set_add): the set's byte automaton (stopmatch.h), the model's
// token bytes (token v is bytes[tb_start[v] .. tb_start[v + 1])), the current state, and once a string matched, its hit
// (1 + the string's index) and the bytes of the last token after the match. next == nullptr: the stream has no set.
struct GenStop {
    const uint32_t *next, *hit;       // [states][256], [states]
    const unsigned long long *tb_start; // [V + 1]
    const unsigned char *tb_bytes;
    unsigned long long state, match, tail;
};

// Walk the bytes of emitted token tok through the stream's stop automaton; true when a stop string ends in them.
__device__ __forceinline__ bool gen_stop_walk(GenStop &m, unsigned long long tok) {
    const unsigned long long b0 = m.tb_start[tok];
    uint32_t q = (uint32_t)m.state;
    unsigned long long tail = 0;
    const uint32_t h = stopmatch::walk(m.next, m.hit, q, m.tb_bytes + b0, m.tb_start[tok + 1] - b0, tail);
    m.state = q;
    if (!h) return false;
    m.match = h;
    m.tail = tail;
    return true;
}

// Where emitted tokens go and what ends a stream: k_gen_feedback's and k_spec_accept's shared arguments (gen_emit).
struct GenEmit {
    unsigned long long *out;         // [n_streams][max_new]: token k of stream s at [s][k % max_new]
    unsigned long long max_new;
    const unsigned long long *stop;  // [n_stop], or the tokens stop_start indexes
    int n_stop;
    // the batcher: stream s's own stop tokens are stop[stop_start[s] .. stop_start[s + 1]) (n_stop is not read);
    // nullptr: stop[0 .. n_stop) for every stream
    const unsigned long long *stop_start;
    GenConstraint *gc;               // [n_streams] token automata (generate_streams_constrained), else nullptr
    unsigned long long *fault;       // {stream + 1, token, state} of the first emitted token without an edge (gc only)
    GenStop *gst;                    // [n_streams] stop sets (generate_streams_stop, batcher lanes with sets), else nullptr
};

// Append token tok of stream s as its entry number len (0-based) and say whether the stream ends with it. The checks
// run in this order: the stream's budget, the stop tokens, its automaton (advanced by tok) and its stop strings (tok's
// bytes walked through its stop set). A generate_streams call emits at most max_new tokens per stream, so `% max_new`
// leaves its index alone; a batcher lane keeps one group's tokens in a ring.
__device__ __forceinline__ bool gen_emit(const GenEmit &e, int s, unsigned long long len, unsigned long long budget,
                                         unsigned long long tok) {
    e.out[(size_t)s * e.max_new + len % e.max_new] = tok;
    bool stop = len + 1 == budget;
    if (e.stop_start) {
        for (unsigned long long i = e.stop_start[s]; i < e.stop_start[s + 1]; ++i) stop |= e.stop[i] == tok;
    } else {
        for (int i = 0; i < e.n_stop; ++i) stop |= e.stop[i] == tok;
    }
    if (e.gc && e.gc[s].mask) stop |= gen_constraint_step(e.gc[s], tok, s, e.fault);
    if (e.gst && e.gst[s].next) stop |= gen_stop_walk(e.gst[s], tok);
    return stop;
}

struct GenFeedbackArgs {
    GenStream *gs;
    const int *row_stream;           // [rows] stream of each row
    int rows;
    const unsigned long long *next;  // arg-max per row, or nullptr when sampling
    const double *sample;            // {token, margin} per row when sampling
    PassDesc *passes;                // tensor-core path: the descriptors of the next step, else nullptr
    GenEmit emit;
};

// One thread per row: emit the picked token of a live stream (gen_emit), then write the next step's input. On the
// tensor-core path that is the row's token and descriptor in its pass; a finished stream loses kDescLast, so no pass
// stores its slot again. `passes` is the next step's layout, whose row r is token r (the rows lead every pass set); the
// batcher passes each step the layout of the step after it, since their prefill tokens differ.
__global__ void k_gen_feedback(const GenFeedbackArgs a) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.rows) return;
    const int s = a.row_stream[r];
    GenStream g = a.gs[s];
    if (!g.done) {
        const unsigned long long tok = a.next ? a.next[r] : (unsigned long long)a.sample[2 * r];
        g.done = gen_emit(a.emit, s, g.len, g.budget, tok) ? 1ull : 0ull;
        g.len += 1;
        g.tok = tok;
        a.gs[s] = g;
    }
    if (a.passes) {
        PassDesc &pd = a.passes[r / kPfMaxTokens];
        const int t = r % kPfMaxTokens;
        pd.tokens[t] = g.tok;
        pd.desc[t] = (uint32_t)g.slot | kDescFirst | (g.done ? 0u : kDescLast);
    }
}

// Classifier-free guidance (rwkv_b200_generate_streams_guided). A guided stream has a second stream record, its
// guidance record: the guidance slot, and as tok the guidance first token, then the token the stream emitted last.
// A step's rows are the `rows` conditional rows (the pick chain's), then one guidance row per live guided stream, in
// the order of their conditional rows. Guided row j has its conditional row and scale gamma in GenGuide j, and its
// guidance row is rows + j. Gate and passes read the guidance rows' records like any other row's.
struct GenGuide {
    int row;     // the stream's conditional row
    float scale; // gamma
};

// Rule 2 of include/rwkv_b200.h on guided row j, in place on its conditional row c with guidance row q:
// c[v] + (gamma - 1) * (c[v] - q[v]), each operation rounded to nearest f32 and none fused. Grid
// (ceil(V / kGuideThreads), guided rows), one thread per token.
constexpr int kGuideThreads = 256;
__global__ void __launch_bounds__(kGuideThreads) k_gen_guide(float *logits, int V, int rows, const GenGuide *guide) {
    const int j = blockIdx.y, v = blockIdx.x * kGuideThreads + threadIdx.x;
    if (v >= V) return;
    const GenGuide g = guide[j];
    float *c = logits + (size_t)g.row * V + v;
    const float q = logits[(size_t)(rows + j) * V + v];
    const float w = __fsub_rn(g.scale, 1.0f);
    *c = __fadd_rn(*c, __fmul_rn(w, __fsub_rn(*c, q)));
}

// After k_gen_feedback, one thread per guided row j: the guidance record takes the stream's emitted token and done
// flag, so the guidance slot is fed what the stream emitted and is frozen with it. On the tensor-core path the
// guidance row's token and descriptor go into the next step's passes (a finished stream's loses kDescLast). A separate
// launch, so that k_gen_feedback has written every stream record before it is read here.
__global__ void k_gen_guide_feedback(GenStream *gs, const int *row_stream, int rows, int n_guide, const GenGuide *guide,
                                     PassDesc *passes) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_guide) return;
    const int r = rows + j;
    const GenStream c = gs[row_stream[guide[j].row]];
    GenStream &g = gs[row_stream[r]];
    g.tok = c.tok;
    g.done = c.done;
    if (passes) {
        PassDesc &pd = passes[r / kPfMaxTokens];
        const int t = r % kPfMaxTokens;
        pd.tokens[t] = c.tok;
        pd.desc[t] = (uint32_t)g.slot | kDescFirst | (c.done ? 0u : kDescLast);
    }
}

} // namespace rk
