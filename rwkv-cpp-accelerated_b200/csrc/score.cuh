// score.cuh — scoring: the log-probability, the rank and the top alternatives of a target token, per row of logits.
//
// The rule (DESIGN §4.3), per scored row of f32 logits l with target y:
//   m        = (double) max_v l[v];
//   S        = sum_v exp((double)l[v] - m), each thread summing its contiguous run of the vocabulary in index order,
//              then block_sum_scan's fixed-order reduction (no floating-point atomics);
//   logprob  = ((double)l[y] - m) - log(S);
//   rank     = #{v : l[v] ranks before y}, ranking by l descending, ties by lower index, -0 with +0 (order_key): an exact
//              integer count, 0 exactly when y is k_argmax_rows' pick;
//   top_n    the first top_n (<= kMaxTopN) tokens of that ranking, in ranking order, each with the logprob of the same
//              formula (bit for bit what the row reports when that token is the target).
// Generation's processed mode divides by a temperature tau: z[v] = ((double)l[v] - m) / tau, S = sum_v exp(z[v]),
// logprob = z[y] - log(S); the rank and the top entries keep the ranking by l. tau = 1 (scoring, raw mode) divides
// exactly, so it is the rule above bit for bit.
// Every output depends only on the row's bits, y, tau and top_n. The top entries come from radix_select (sampling.cuh) by
// count: the tokens with a key above the cut, then the first `take` tokens with the cut's key in index order; one warp
// orders the at most kMaxTopN of them.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/rwkv_b200.h"
#include "aux_kernels.cuh"
#include "sampling.cuh"

namespace rk {

constexpr int kMaxTopN = RWKV_B200_MAX_TOP_N;

// The float whose order_key is k (+0 for the key shared by -0 and +0).
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// One formula for the target and for the top entries, so that both give the same bits. tau = 1 divides exactly.
__device__ __forceinline__ double row_logprob(float l, double m, double tau, double log_s) { return (((double)l - m) / tau) - log_s; }

// Scores one row of f32 logits with target y and divisor tau (z = (l - m) / tau; tau = 1 is the rule above):
// *logprob, *rank, and the first top_n entries of the ranking into top_tokens[0..top_n), top_logprobs[0..top_n).
// Called by a whole CTA of kNucThreads.
__device__ __forceinline__ void logprob_row(const float *row, int V, int y, double tau, int top_n, double *logprob,
                                            unsigned long long *rank, unsigned long long *top_tokens, double *top_logprobs) {
    __shared__ NucShared sh;
    __shared__ uint32_t s_kmax, top_key[kMaxTopN];
    __shared__ unsigned s_rank, s_above;
    __shared__ int top_idx[kMaxTopN];
    const int tid = threadIdx.x, lane = tid & 31;
    const float ly = row[y];
    const uint32_t ky = order_key(ly);
    if (tid == 0) {
        s_kmax = 0;
        s_rank = 0;
        s_above = 0;
    }
    __syncthreads();

    // pass 1: the largest key and the tokens ranked before y (integer reductions, independent of the order)
    uint32_t kmax = 0;
    unsigned before = 0;
    for (int i = tid; i < V; i += kNucThreads) {
        const uint32_t k = order_key(row[i]);
        kmax = max(kmax, k);
        before += k > ky || (k == ky && i < y);
    }
    kmax = __reduce_max_sync(0xffffffffu, kmax);
    before = __reduce_add_sync(0xffffffffu, before);
    if (lane == 0) {
        atomicMax(&s_kmax, kmax);
        atomicAdd(&s_rank, before);
    }
    __syncthreads();
    const double m = (double)key_value(s_kmax);

    // pass 2: the sum of the exponentials, each thread over its contiguous run, then the fixed-order block reduction
    const int per = (V + kNucThreads - 1) / kNucThreads;
    const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
    double part = 0.0;
    for (int i = i0; i < i1; ++i) part += exp(((double)row[i] - m) / tau);
    double dummy;
    const double log_s = log(block_sum_scan(part, sh.scan, dummy));
    if (tid == 0) {
        *logprob = row_logprob(ly, m, tau, log_s);
        *rank = s_rank;
    }
    if (top_n == 0) return;

    // the first top_n tokens of the ranking: key above the cut (any order), then the first `take` with the cut's key
    const Cut c = radix_select(row, V, false, (unsigned long long)top_n, 0.0, 1.0, sh);
    unsigned eq = 0;
    for (int i = i0; i < i1; ++i) {
        const uint32_t k = order_key(row[i]);
        if (k > c.key) {
            const unsigned at = atomicAdd(&s_above, 1u);
            top_key[at] = k;
            top_idx[at] = i;
        }
        eq += k == c.key;
    }
    double eq_before;
    block_sum_scan((double)eq, sh.scan, eq_before); // exact: integers far below 2^53
    unsigned r = (unsigned)eq_before;
    for (int i = i0; i < i1 && r < c.take; ++i)
        if (order_key(row[i]) == c.key) {
            top_key[c.above + r] = c.key;
            top_idx[c.above + r] = i;
            ++r;
        }
    __syncthreads();
    // one warp places each entry by counting the entries ranked before it
    if (tid < 32 && lane < top_n) {
        const uint32_t k = top_key[lane];
        const int idx = top_idx[lane];
        int pos = 0;
        for (int e = 0; e < top_n; ++e) pos += top_key[e] > k || (top_key[e] == k && top_idx[e] < idx);
        top_tokens[pos] = (unsigned long long)idx;
        top_logprobs[pos] = row_logprob(row[idx], m, tau, log_s);
    }
}

struct ScoreArgs {
    const float *logits;                 // [rows][V]
    int V;
    const int *rows;                     // [n] row of `logits` scored by CTA j
    const unsigned long long *targets;   // [n] target token of CTA j (< V)
    int top_n;                           // 0..kMaxTopN
    double *logprob;                     // [n]
    unsigned long long *rank;            // [n]
    unsigned long long *top_tokens;      // [n][top_n]
    double *top_logprobs;                // [n][top_n]
};

// One CTA of kNucThreads per scored row j.
__global__ void __launch_bounds__(kNucThreads) k_logprob_rows(ScoreArgs a) {
    const int j = blockIdx.x;
    logprob_row(a.logits + (size_t)a.rows[j] * a.V, a.V, (int)a.targets[j], 1.0, a.top_n, a.logprob + j, a.rank + j,
                a.top_tokens + (size_t)j * a.top_n, a.top_logprobs + (size_t)j * a.top_n);
}

// What the batcher asks of one lane: mode < 0: no scoring, else RWKV_B200_LOGPROBS_*; top_n <= the call's top_n.
struct LogprobLane {
    int mode;
    int top_n;
};

struct GenLogprobArgs {
    const float *logits;                 // [rows][V] the rows of the current step
    int V;
    const GenStream *gs;
    const int *row_stream;               // [rows] stream of each row
    const unsigned long long *next;      // arg-max per row, or nullptr when sampling
    const double *sample;                // {token, margin} per row when sampling
    const rwkv_b200_sampler *samp;       // processed mode with samplers: tau = temperature (> 0), else nullptr: tau = 1
    int top_n;                           // top entries per token, and the stride of the top arrays
    unsigned long long max_new;
    double *logprob;                     // [n_streams][max_new]: token k of stream s at [s][k % max_new]
    unsigned long long *rank;            // [n_streams][max_new]
    unsigned long long *top_tokens;      // [n_streams][max_new][top_n]
    double *top_logprobs;                // [n_streams][max_new][top_n]
    // the batcher: each stream's own mode and top_n (samp then holds every stream's sampler); raw-mode streams read
    // `raw` ([rows][V], nullptr: `logits`). lane == nullptr: every stream has the call's mode (samp) and top_n
    const LogprobLane *lane;
    const float *raw;
};

// Score pick y of row r of the step, stream s, into entry o of the result arrays: on a.logits divided by the stream's
// temperature with a.samp (processed mode), else on a.logits; a batcher lane by its own mode and top_n, raw lanes on
// a.raw when set. A lane without scoring returns at once (the whole CTA, before any barrier).
__device__ __forceinline__ void gen_logprob_at(const GenLogprobArgs &a, int s, int r, int y, size_t o) {
    const float *logits = a.logits;
    const rwkv_b200_sampler *samp = a.samp;
    int top_n = a.top_n;
    if (a.lane) {
        const LogprobLane ln = a.lane[s];
        if (ln.mode < 0) return;
        top_n = ln.top_n;
        if (ln.mode == RWKV_B200_LOGPROBS_RAW) {
            samp = nullptr;
            if (a.raw) logits = a.raw;
        }
    }
    const float T = samp ? samp[s].temperature : 0.0f;
    logprob_row(logits + (size_t)r * a.V, a.V, y, T > 0.0f ? (double)T : 1.0, top_n, a.logprob + o, a.rank + o,
                a.top_tokens + o * a.top_n, a.top_logprobs + o * a.top_n);
}

// generate_streams_logprobs: one CTA of kNucThreads per row of the step, between the pick and k_gen_feedback. It scores
// the picked token of a live stream at entry [s][len]; with `lane` (the batcher) at [s][len % max_new], a ring of
// entries per lane, as k_gen_feedback keeps its tokens. A stream that finished earlier in the group still has a row, and
// its len may equal max_new, so writing for it would land on stream s + 1; it returns at once (the whole CTA, before any
// barrier).
__global__ void __launch_bounds__(kNucThreads) k_gen_logprob(const GenLogprobArgs a) {
    const int r = blockIdx.x, s = a.row_stream[r];
    const GenStream &g = a.gs[s];
    if (g.done) return;
    const int y = a.next ? (int)a.next[r] : (int)a.sample[2 * r];
    // the division only where it can matter: a 64-bit `%` on every path costs k_gen_logprob spills at 64 registers
    gen_logprob_at(a, s, r, y, (size_t)s * a.max_new + (a.lane ? g.len % a.max_new : g.len));
}

} // namespace rk
