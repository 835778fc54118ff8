// generate.cuh — device side of rwkv_b200_generate_streams: the per-step feedback that lets many decode steps of
// many streams run without returning to the host.
//
// A call keeps one record per stream on the device (GenStream). Each step of a group is enqueued by the host with no
// synchronisation inside the group: forward (tensor-core passes or the decode kernel, row r = a live stream), then
// k_gen_override on the logits rows, the existing pick (k_argmax_rows or k_sample_typical), and k_gen_feedback, which
// appends the picked token, decides whether the stream is done and writes the next step's input. A stream that
// finishes inside a group keeps its row until the group ends but is frozen: its slot is not written again.
// generate_streams_logprobs adds k_gen_logprob (score.cuh) between the pick and k_gen_feedback.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

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
