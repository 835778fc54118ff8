// aux_kernels.cuh — load-time repack kernels and the device sampler (not on the per-token hot path).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace rk {

// =======================================================================================
// Load-time repack: u8 [R][C] (leading dim ldin) -> s8 out[c][r0 + r] (leading dim ldout),
// value ^ 0x80. 64x64-byte tiles through shared memory, 32-bit accesses on both sides.
// =======================================================================================
__global__ void __launch_bounds__(256) k_transpose_xor(const uint8_t *__restrict__ in, size_t ldin, int R, int C,
                                                       int8_t *__restrict__ out, size_t ldout, size_t r0) {
    __shared__ uint8_t t[64][68];
    const int bx = blockIdx.x * 64, by = blockIdx.y * 64; // bx: column block, by: row block
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4; // 16 x 16
    for (int rr = ty; rr < 64; rr += 16) {
        const int r = by + rr;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int c = bx + tx * 4 + e;
            t[rr][tx * 4 + e] = (r < R && c < C) ? in[(size_t)r * ldin + c] : 0;
        }
    }
    __syncthreads();
    for (int cc = ty; cc < 64; cc += 16) {
        const int c = bx + cc;
        if (c >= C) continue;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int r = by + tx * 4 + e;
            if (r < R) out[(size_t)c * ldout + r0 + r] = (int8_t)(t[tx * 4 + e][cc] ^ 0x80);
        }
    }
}

__global__ void k_exp_table(const double *__restrict__ in, double *__restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = exp(in[i]);
}

// oc[j] = 128*r[j] + o[j]
__global__ void k_centre_offsets(const float *__restrict__ r, const float *__restrict__ o, float *__restrict__ oc, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) oc[i] = (float)(128.0 * (double)r[i] + (double)o[i]);
}

// ---------------------------------------------------------------------------------------
// Device-side restatement of the reference sampler (include/rwkv/sampler/typical.h = what the
// reference's typical.h:20-58 actually computes): probs = exp(l)/sum, probs^e with e = uint8(1/temp),
// renormalise, cumulative sums, first index whose cumulative probability reaches the uniform `u`
// drawn on the host. One CTA per row of logits, every thread owns a contiguous run of the vocabulary. Sums are block
// reductions, so cumulative values can differ from the host's sequential ones by ~1e-13; the kernel
// therefore also returns how far `u` is from the nearest interval boundary, and the caller falls
// back to the host path when that margin is below 1e-9 (probability ~1e-9 per draw): identical
// tokens by construction. Row r: out[2r] = token, out[2r + 1] = margin.
// ---------------------------------------------------------------------------------------
constexpr int kSampleThreads = 1024;
__device__ __forceinline__ double sample_prob(float logit, double total, int exponent) {
    if (exponent == 0) return 1.0;
    const double q = exp((double)logit) / total;
    double v = q;
    for (int e = 1; e < exponent; ++e) v *= q;
    return v;
}
__device__ __forceinline__ double block_sum_scan(double v, double *sh, double &prefix_excl) {
    // inclusive scan over the 1024 threads; returns the block total, prefix_excl = sum of lower threads
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[w] = x;
    __syncthreads();
    if (w == 0) {
        double t = sh[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        sh[32 + lane] = t; // inclusive totals of the warps
    }
    __syncthreads();
    const double warp_off = w ? sh[32 + w - 1] : 0.0;
    const double total = sh[63];
    prefix_excl = warp_off + x - v;
    __syncthreads();
    return total;
}
// One CTA per row: row r samples logits + r * row_stride with u[r] into out[2r], out[2r + 1].
__global__ void __launch_bounds__(kSampleThreads) k_sample_typical(const float *logits, size_t row_stride, int len, int exponent,
                                                                  const double *us, double *out) {
    __shared__ double sh[64];
    __shared__ double starts[kSampleThreads + 1];
    logits += (size_t)blockIdx.x * row_stride;
    out += 2 * (size_t)blockIdx.x;
    const double u = us[blockIdx.x];
    const int per = (len + kSampleThreads - 1) / kSampleThreads;
    const int i0 = min(len, (int)threadIdx.x * per), i1 = min(len, i0 + per);
    double dummy;
    double part = 0.0;
    for (int i = i0; i < i1; ++i) part += exp((double)logits[i]);
    const double total = block_sum_scan(part, sh, dummy);
    part = 0.0;
    for (int i = i0; i < i1; ++i) part += sample_prob(logits[i], total, exponent);
    double before;
    const double s = block_sum_scan(part, sh, before);
    // thread t's run covers cumulative probability (starts[t], starts[t+1]]: the runs tile [0, inf) exactly
    starts[threadIdx.x] = before / s;
    if (threadIdx.x == 0) {
        starts[kSampleThreads] = 2.0; // cp_last is forced to 1.0: everything above goes to the end
        out[0] = 0.0;                 // u <= 0 (probability 2^-53): nobody claims it; margin 0 sends the caller
        out[1] = 0.0;                 // to the host path
    }
    __syncthreads();
    const double lo = starts[threadIdx.x], hi = starts[threadIdx.x + 1];
    if (i0 < i1 && lo < u && !(hi < u)) {
        double c = lo, margin = 0.0;
        int tok = i1 - 1; // rounding left u just above this run's own running sum: margin 0 -> host path decides
        for (int i = i0; i < i1; ++i) {
            const double prev = c;
            c += sample_prob(logits[i], total, exponent) / s;
            if (i == len - 1 || !(c < u)) {
                tok = i;
                margin = i == len - 1 ? u - prev : fmin(u - prev, c - u);
                break;
            }
        }
        out[0] = (double)tok;
        out[1] = margin;
    }
}

// One CTA per row of logits[rows][V]: arg-max, the first index wins ties (as the decode kernel's greedy arg-max).
constexpr int kArgmaxThreads = 256;
__global__ void __launch_bounds__(kArgmaxThreads) k_argmax_rows(const float *logits, int V, unsigned long long *out) {
    __shared__ float bv[kArgmaxThreads / 32];
    __shared__ int bi[kArgmaxThreads / 32];
    const float *row = logits + (size_t)blockIdx.x * V;
    float best = -INFINITY;
    int bidx = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += kArgmaxThreads) {
        const float y = row[i];
        if (y > best) { // i ascending per thread: first maximum kept
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
    if ((threadIdx.x & 31) == 0) {
        bv[threadIdx.x >> 5] = best;
        bi[threadIdx.x >> 5] = bidx;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kArgmaxThreads / 32; ++w)
            if (bv[w] > best || (bv[w] == best && bi[w] < bidx)) {
                best = bv[w];
                bidx = bi[w];
            }
        out[blockIdx.x] = (unsigned long long)bidx;
    }
}

} // namespace rk
