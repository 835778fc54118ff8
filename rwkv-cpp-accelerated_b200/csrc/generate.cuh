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
// stream's token automaton (GenConstraint) after appending its token.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/rwkv_b200.h"
#include "common.cuh"
#include "prefill.cuh"

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

// logits[r][tok[i]] = val[i] for every row, in the order given (a repeated token keeps its last value).
__global__ void k_gen_override(float *logits, int V, int rows, const unsigned long long *tok, const float *val, int n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    for (int i = 0; i < n; ++i) logits[(size_t)r * V + tok[i]] = val[i];
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

// logits[r][v] = -inf for every token v without an edge out of the current state of row r's stream. Grid
// (ceil(V / kMaskThreads), rows), one thread per token. Unconstrained and finished streams are left alone: a finished
// stream may sit in a state without edges, and masking its row would leave the pick no finite value.
constexpr int kMaskThreads = 256;
__global__ void __launch_bounds__(kMaskThreads) k_gen_mask(float *logits, int V, const GenStream *gs, const int *row_stream,
                                                           const GenConstraint *gc) {
    const int r = blockIdx.y, s = row_stream[r];
    const GenConstraint &c = gc[s];
    if (!c.mask || gs[s].done) return;
    const int v = blockIdx.x * kMaskThreads + threadIdx.x;
    if (v >= V) return;
    if (!((c.mask[c.state * kMaskWords + (v >> 5)] >> (v & 31)) & 1u)) logits[(size_t)r * V + v] = -INFINITY;
}

struct GenFeedbackArgs {
    GenStream *gs;
    const int *row_stream;           // [rows] stream of each row
    int rows;
    const unsigned long long *next;  // arg-max per row, or nullptr when sampling
    const double *sample;            // {token, margin} per row when sampling
    const unsigned long long *stop;  // [n_stop]
    int n_stop;
    unsigned long long *out;         // [n_streams][max_new]
    unsigned long long max_new;
    PassDesc *passes;                // tensor-core path: the descriptors of the next step, else nullptr
    GenConstraint *gc;               // [n_streams] generate_streams_constrained, else nullptr
    unsigned long long *fault;       // {stream + 1, token, state} of the first emitted token without an edge (gc only)
};

// One thread per row: emit the picked token of a live stream, then write the next step's input. On the tensor-core
// path that is the row's token and descriptor in its pass; a finished stream loses kDescLast, so no pass stores its
// slot again.
__global__ void k_gen_feedback(const GenFeedbackArgs a) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.rows) return;
    const int s = a.row_stream[r];
    GenStream g = a.gs[s];
    if (!g.done) {
        const unsigned long long tok = a.next ? a.next[r] : (unsigned long long)a.sample[2 * r];
        a.out[(size_t)s * a.max_new + g.len] = tok;
        g.len += 1;
        g.tok = tok;
        bool stop = g.len == g.budget;
        for (int i = 0; i < a.n_stop; ++i) stop |= a.stop[i] == tok;
        if (a.gc && a.gc[s].mask) {
            // advance the automaton; a state without edges completes it. The mask makes a missing edge impossible
            // unless the pick broke its contract: record it for the host and end the stream
            GenConstraint &c = a.gc[s];
            const unsigned long long q = c.state, end = c.start[q + 1];
            unsigned long long lo = c.start[q], hi = end;
            while (lo < hi) {
                const unsigned long long mid = (lo + hi) / 2;
                if (c.tok[mid] < tok) lo = mid + 1;
                else hi = mid;
            }
            if (lo < end && c.tok[lo] == tok) {
                const unsigned long long q2 = c.next[lo];
                c.state = q2;
                stop |= c.start[q2] == c.start[q2 + 1];
            } else {
                if (atomicCAS(a.fault, 0ull, (unsigned long long)s + 1) == 0ull) {
                    a.fault[1] = tok;
                    a.fault[2] = q;
                }
                stop = true;
            }
        }
        g.done = stop ? 1ull : 0ull;
        a.gs[s] = g;
    }
    if (a.passes) {
        PassDesc &pd = a.passes[r / kPfMaxTokens];
        const int t = r % kPfMaxTokens;
        pd.tokens[t] = g.tok;
        pd.desc[t] = (uint32_t)g.slot | kDescFirst | (g.done ? 0u : kDescLast);
    }
}

} // namespace rk
