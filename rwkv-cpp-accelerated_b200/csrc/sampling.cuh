// sampling.cuh — the tunable per-stream sampler: temperature, top-p (nucleus), top-k, and presence / frequency
// penalties over the tokens a stream has emitted during a generate_streams_ex call.
//
// The rule (DESIGN §4.3), per row of f32 logits l' (penalties and overrides already applied):
//   order   tokens by l' descending, ties by lower index (-0 ranks with +0);
//   T = 0   the first token of the order: exactly k_argmax_rows' pick, u ignored, margin reported as 1;
//   T > 0   p[v] = exp(((double)l'[v] - (double)max l') / (double)T); the kept set is the first min(n_p, top_k) tokens
//           of the order (top_k = 0: no limit), n_p the smallest n whose first-n mass reaches top_p * sum(p)
//           (top_p = 1: every token); the draw walks the kept tokens in vocabulary order with
//           c_v = sum_{kept w <= v} p_w / sum_kept and takes the first kept v with p_v > 0 and c_v >= u; a rounding
//           remainder (c < u at the end) goes to the last kept token with p > 0.
//
// No sort: the cut is found by radix selection on an order-preserving uint32 key of l', four rounds of 8-bit digits.
// Each round histograms the tokens still matching the decided high digits (counts, and for the top-p cut their
// probability mass) and keeps the bin holding the boundary. The mass is summed in 2^-47 fixed point with integer
// atomics, so the histogram does not depend on the order the threads arrive in; its rounding (< 4e-10 of the total)
// only moves a top-p cut that lies that close to a token boundary. The draw itself is in double with block scans in a
// fixed order. Every output is a function of the row's bits and the parameters only.
#pragma once
#include <cooperative_groups.h>
#include <cooperative_groups/reduce.h>
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/rwkv_b200.h"
#include "aux_kernels.cuh"
#include "generate.cuh"

namespace rk {

constexpr int kNucThreads = 1024;
constexpr double kMassScale = 140737488355328.0; // 2^47: 50277 tokens of mass <= 1 stay below 2^63

// Order-preserving key: a > b as floats <=> key(a) > key(b); -0 and +0 share the key of +0.
__device__ __forceinline__ uint32_t order_key(float f) {
    uint32_t b = __float_as_uint(f);
    if ((b << 1) == 0) b = 0;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ double nucleus_prob(float l, double m, double T) { return exp(((double)l - m) / T); }

struct NucShared {
    unsigned cnt[256];
    unsigned long long mass[256];
    double scan[64];
    float wv[kNucThreads / 32];
    int wi[kNucThreads / 32];
    unsigned long long sel_mass_above, sel_mass_bin; // the chosen bin: mass of the bins above it, its own mass
    unsigned sel_cnt_above, sel_cnt_bin;             // the same in tokens
    int sel_digit, claim, last;
};

// The boundary of the first tokens of the order: every token with key > `key`, then the first `take` tokens with key
// == `key` in index order. by_mass: the smallest such prefix whose fixed-point mass reaches `target`; else the first
// `target` tokens. `above` is the count of tokens with key > `key`. Called by the whole block.
struct Cut {
    uint32_t key;
    unsigned above, take;
};
__device__ __noinline__ Cut radix_select(const float *row, int V, bool by_mass, unsigned long long target, double m, double T,
                                         NucShared &sh) {
    namespace cg = cooperative_groups;
    const int tid = threadIdx.x, lane = tid & 31;
    uint32_t prefix = 0;
    unsigned above_n = 0;
    unsigned long long above_m = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += kNucThreads) {
            sh.cnt[i] = 0;
            sh.mass[i] = 0;
        }
        __syncthreads();
        const uint32_t hi_mask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
        for (int i = tid; i < V; i += kNucThreads) {
            const float l = row[i];
            const uint32_t k = order_key(l);
            if ((k & hi_mask) != prefix) continue;
            // the lanes of a warp that hit the same bin add up first (exact integer sums): one atomic per bin and warp
            const unsigned d = (k >> shift) & 255u;
            const auto peers = cg::labeled_partition(cg::coalesced_threads(), d);
            unsigned long long q = 0;
            if (by_mass) q = cg::reduce(peers, __double2ull_rn(nucleus_prob(l, m, T) * kMassScale), cg::plus<unsigned long long>());
            if (peers.thread_rank() == 0) {
                atomicAdd(&sh.cnt[d], peers.size());
                if (q) atomicAdd(&sh.mass[d], q);
            }
        }
        __syncthreads();
        if (tid < 32) {
            // lane j holds bins 255 - 8j down to 248 - 8j; find the first bin from the top where the prefix reaches target
            unsigned long long sm = 0;
            unsigned sc = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int d = 255 - (lane * 8 + j);
                sm += sh.mass[d];
                sc += sh.cnt[d];
            }
            unsigned long long im = sm;
            unsigned ic = sc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long ym = __shfl_up_sync(0xffffffffu, im, o);
                const unsigned yc = __shfl_up_sync(0xffffffffu, ic, o);
                if (lane >= o) {
                    im += ym;
                    ic += yc;
                }
            }
            const bool hit = by_mass ? above_m + im >= target : (unsigned long long)(above_n + ic) >= target;
            const unsigned hits = __ballot_sync(0xffffffffu, hit);
            if (lane == __ffs(hits) - 1) {
                unsigned long long rm = im - sm;
                unsigned rc = ic - sc;
                for (int j = 0; j < 8; ++j) {
                    const int d = 255 - (lane * 8 + j);
                    const bool last = by_mass ? above_m + rm + sh.mass[d] >= target
                                              : (unsigned long long)(above_n + rc + sh.cnt[d]) >= target;
                    if (last) {
                        sh.sel_digit = d;
                        sh.sel_mass_above = rm;
                        sh.sel_cnt_above = rc;
                        sh.sel_mass_bin = sh.mass[d];
                        sh.sel_cnt_bin = sh.cnt[d];
                        break;
                    }
                    rm += sh.mass[d];
                    rc += sh.cnt[d];
                }
            }
        }
        __syncthreads();
        prefix |= (uint32_t)sh.sel_digit << shift;
        above_n += sh.sel_cnt_above;
        above_m += sh.sel_mass_above;
        __syncthreads(); // everyone has read the selection before the next round clears the bins
    }
    // every token of the last bin has the key `prefix`, hence the same probability
    unsigned take;
    if (by_mass) {
        const unsigned long long q = sh.sel_mass_bin / sh.sel_cnt_bin;
        take = (unsigned)((target - above_m + q - 1) / q);
    } else {
        take = (unsigned)(target - above_n);
    }
    return Cut{prefix, above_n, take};
}

// One CTA per row r of logits (row stride V): parameters params[row_stream ? row_stream[r] : r], uniform us[r]
// (us may be NULL when every row is greedy). out[2r] = token, out[2r + 1] = margin: the distance of u to the edges of
// the drawn token's cumulative interval (1 for a greedy row).
__global__ void __launch_bounds__(kNucThreads) k_sample_nucleus(const float *logits, int V, const rwkv_b200_sampler *params,
                                                               const int *row_stream, const double *us, double *out) {
    __shared__ NucShared sh;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const float *row = logits + (size_t)blockIdx.x * V;
    const rwkv_b200_sampler sp = params[row_stream ? row_stream[blockIdx.x] : (int)blockIdx.x];
    out += 2 * (size_t)blockIdx.x;

    // the maximum, first index on ties (k_argmax_rows' comparisons)
    float best = -INFINITY;
    int bidx = 0x7fffffff;
    for (int i = tid; i < V; i += kNucThreads) {
        const float y = row[i];
        if (y > best) {
            best = y;
            bidx = i;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
        if (ov > best || (ov == best && oi < bidx)) {
            best = ov;
            bidx = oi;
        }
    }
    if (lane == 0) {
        sh.wv[w] = best;
        sh.wi[w] = bidx;
    }
    if (tid == 0) {
        sh.claim = kNucThreads;
        sh.last = -1;
    }
    __syncthreads();
    if (sp.temperature == 0.0f) {
        if (tid == 0) {
            for (int j = 1; j < kNucThreads / 32; ++j)
                if (sh.wv[j] > best || (sh.wv[j] == best && sh.wi[j] < bidx)) {
                    best = sh.wv[j];
                    bidx = sh.wi[j];
                }
            out[0] = (double)bidx;
            out[1] = 1.0;
        }
        return;
    }
    for (int j = 0; j < kNucThreads / 32; ++j) best = fmaxf(best, sh.wv[j]);
    const double m = best, T = sp.temperature;

    // the kept set: key > kc, or key == kc and among the first rc such tokens by index (kc = 0: every token)
    uint32_t kc = 0;
    unsigned rc = 0;
    unsigned n_keep = (unsigned)V;
    if (sp.top_p < 1.0f) {
        unsigned long long total = 0; // fixed-point mass of the row: each thread's part, then one integer reduction
        for (int i = tid; i < V; i += kNucThreads) total += __double2ull_rn(nucleus_prob(row[i], m, T) * kMassScale);
        for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
        if (lane == 0) sh.mass[w] = total;
        __syncthreads();
        total = 0;
        for (int j = 0; j < kNucThreads / 32; ++j) total += sh.mass[j];
        __syncthreads();
        const unsigned long long target = (unsigned long long)ceil((double)sp.top_p * (double)total);
        const Cut c = radix_select(row, V, true, target, m, T, sh);
        kc = c.key;
        rc = c.take;
        n_keep = c.above + c.take;
    }
    if (sp.top_k != 0 && sp.top_k < n_keep) {
        const Cut c = radix_select(row, V, false, sp.top_k, m, T, sh);
        kc = c.key;
        rc = c.take;
    }

    // the draw, in vocabulary order: every thread owns a contiguous run
    const int per = (V + kNucThreads - 1) / kNucThreads;
    const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
    unsigned rank = 0; // tokens with key kc before this run (exact: integers below 2^53)
    if (kc != 0) {
        unsigned eq = 0;
        for (int i = i0; i < i1; ++i) eq += order_key(row[i]) == kc;
        double before_eq;
        block_sum_scan((double)eq, sh.scan, before_eq);
        rank = (unsigned)before_eq;
    }
    double own = 0.0;
    {
        unsigned r = rank;
        for (int i = i0; i < i1; ++i) {
            const uint32_t k = order_key(row[i]);
            if (k > kc || (k == kc && r++ < rc)) own += nucleus_prob(row[i], m, T);
        }
    }
    double before;
    const double S = block_sum_scan(own, sh.scan, before);
    const double u = us ? us[blockIdx.x] : 0.0;
    // the drawing thread: the first with mass whose run ends at or above u; if rounding leaves every run below u, the
    // last thread with mass takes the remainder
    if (own > 0.0) {
        if ((before + own) / S >= u) atomicMin(&sh.claim, tid);
        atomicMax(&sh.last, tid);
    }
    __syncthreads();
    const int drawer = sh.claim < kNucThreads ? sh.claim : sh.last;
    if (tid != drawer) return;
    unsigned r = rank;
    double run = 0.0, prev = before / S;
    int tok = -1;
    double margin = 0.0;
    for (int i = i0; i < i1; ++i) {
        const uint32_t k = order_key(row[i]);
        if (!(k > kc || (k == kc && r++ < rc))) continue;
        const double p = nucleus_prob(row[i], m, T);
        if (p == 0.0) continue;
        run += p;
        const double c = (before + run) / S;
        tok = i;
        if (c >= u) {
            margin = fmin(u - prev, c - u);
            break;
        }
        margin = u - prev; // remainder: u lies above c of the last token with mass
        prev = c;
    }
    out[0] = (double)tok;
    out[1] = fmax(margin, 0.0);
}

// Presence and frequency penalties of generate_streams_ex, before the overrides and the pick of a step. Grid
// (ceil(V / 256), rows). cnt / seen are [n_streams][V], indexed by stream. A live stream that has emitted a token
// folds that token in first (every count times decay, then +1 and seen for the token), then every seen token's logit
// becomes l - (presence + frequency * cnt). Finished streams and streams without penalties are left alone.
constexpr int kPenaltyThreads = 256;
__global__ void __launch_bounds__(kPenaltyThreads) k_gen_penalty(float *logits, int V, const GenStream *gs, const int *row_stream,
                                                                 const rwkv_b200_sampler *params, float *cnt, unsigned char *seen) {
    const int r = blockIdx.y, s = row_stream[r];
    const rwkv_b200_sampler sp = params[s];
    if (sp.presence_penalty == 0.0f && sp.frequency_penalty == 0.0f) return;
    const GenStream &g = gs[s];
    if (g.done) return;
    const int v = blockIdx.x * kPenaltyThreads + threadIdx.x;
    if (v >= V) return;
    const size_t o = (size_t)s * V + v;
    float c = cnt[o];
    unsigned char sn = seen[o];
    if (g.len > 0) {
        c = __fmul_rn(c, sp.penalty_decay);
        if ((unsigned long long)v == g.tok) {
            c = __fadd_rn(c, 1.0f);
            sn = 1;
            seen[o] = 1;
        }
        cnt[o] = c;
    }
    if (sn) {
        float &l = logits[(size_t)r * V + v];
        l = __fsub_rn(l, __fadd_rn(sp.presence_penalty, __fmul_rn(sp.frequency_penalty, c)));
    }
}

} // namespace rk
