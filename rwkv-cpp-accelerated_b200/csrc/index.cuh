// index.cuh — state-vector search: the distances between query slots and the rows of a state index, and a
// deterministic top-k by (distance, id) (include/rwkv_b200.h, "State indexes"; DESIGN §4.3).
//
// The rule, per query vector a and entry vector b of D = n_layers * E doubles:
//   l1 = (sum_j |a_j - b_j|) / E,   l2 = sqrt((sum_j (a_j - b_j)^2) / E)
// summed in one fixed order that depends only on D:
//   * D is cut into segments of kIdxSeg elements (the last one shorter); a segment is summed by one warp, lane t adding
//     the elements t, t + 32, t + 64, ... of the segment in that order (|d| into one sum, fma(d, d, .) into the other),
//     then the 32 lane sums are combined by a fixed xor butterfly (offsets 16, 8, 4, 2, 1);
//   * the segment sums are added in segment order, from 0.0.
// Which CTA or warp sums a segment, how many rows a CTA owns, which slot of the query batch a query takes, and which
// entries are live change nothing: each distance is a function of the two vectors' bits alone.
//
// k_index_scan: one CTA per (segment, run of rows) of an entry block. It keeps the segment of each query of the batch
// (up to kIdxQB) in shared memory and streams each row's segment from HBM once, 32 independent 256-byte loads per warp
// in flight, each element feeding the queries' two sums from one difference. Per (query, row, segment) it writes the
// two sums to `partial`; k_index_combine adds them in segment order and writes l1 and l2. Entry blocks bound `partial`.
//
// k_index_select: the first min(k, live) entries by (key, id), key the metric's distance as an order-preserving integer
// (NaN above +inf). Each CTA sorts up to kIdxSelN (key, id) pairs with a bitonic network in shared memory and keeps its
// first k; passes repeat over the survivors until one CTA holds them all. (key, id) is a total order on distinct ids,
// so the chosen entries and their order do not depend on how the entries are cut into CTAs. radix_select
// (sampling.cuh) is not used: it ranks f32 logits by a 32-bit key inside one row of at most V tokens with 32-bit
// counts, while this ranks 64-bit keys with an id tie-break across CTAs.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace rk {

constexpr int kIdxQB = 8;             // queries per scan of the index
constexpr int kIdxSeg = 1024;         // elements per segment: one warp, 32 per lane
constexpr int kIdxWarps = 8;          // warps per scan CTA
constexpr int kIdxSelN = 4096;        // (key, id) pairs one selection CTA sorts
constexpr int kIdxSelThreads = 1024;
constexpr unsigned long long kIdxNone = ~0ULL;  // the sentinel key and id: a dead entry or an empty position

struct IndexScanArgs {
    const double *rows;                 // [capacity][D]
    const unsigned char *alive;         // [capacity]
    const double *q[kIdxQB];            // the batch's query vectors (the first nq)
    int nq;
    unsigned long long D;
    unsigned long long e0, n;           // the entry block: rows e0 .. e0 + n
    unsigned long long rows_per_cta;
    unsigned G;                         // segments
    double *partial;                    // [nq][n][G][2]
};

// Grid (G, ceil(n / rows_per_cta)), kIdxWarps * 32 threads, kIdxQB * kIdxSeg doubles of dynamic shared memory.
__global__ void __launch_bounds__(kIdxWarps * 32) k_index_scan(const IndexScanArgs a) {
    extern __shared__ double qs[]; // [nq][kIdxSeg], zero past the segment's end
    const unsigned g = blockIdx.x;
    const unsigned long long j0 = (unsigned long long)g * kIdxSeg;
    const int len = (int)(a.D - j0 < (unsigned long long)kIdxSeg ? a.D - j0 : kIdxSeg);
    for (int i = threadIdx.x; i < a.nq * kIdxSeg; i += blockDim.x) {
        const int q = i / kIdxSeg, j = i % kIdxSeg;
        qs[i] = j < len ? a.q[q][j0 + j] : 0.0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned long long r0 = (unsigned long long)blockIdx.y * a.rows_per_cta;
    const unsigned long long r1 = r0 + a.rows_per_cta < a.n ? r0 + a.rows_per_cta : a.n;
    for (unsigned long long r = r0 + w; r < r1; r += kIdxWarps) {
        const unsigned long long e = a.e0 + r;
        if (!a.alive[e]) continue; // warp-uniform
        const double *row = a.rows + e * a.D + j0;
        double v[32];
        // the padding past the segment's end is 0 on both sides: |0 - 0| and 0 * 0 add +0 and change no sum
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = lane + 32 * i < len ? __ldcs(row + lane + 32 * i) : 0.0;
        for (int q = 0; q < a.nq; ++q) {
            const double *qq = qs + q * kIdxSeg + lane;
            double s1 = 0.0, s2 = 0.0;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const double d = v[i] - qq[32 * i];
                s1 += fabs(d);
                s2 = fma(d, d, s2);
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            }
            if (lane == 0) {
                double *p = a.partial + (((unsigned long long)q * a.n + r) * a.G + g) * 2;
                p[0] = s1;
                p[1] = s2;
            }
        }
    }
}

// One thread per (query, row) of the block: the segment sums in segment order, then l1 and l2 into [q][stride].
__global__ void k_index_combine(const double *partial, const unsigned char *alive, int nq, unsigned long long e0,
                                unsigned long long n, unsigned G, double E, double *l1, double *l2, unsigned long long stride) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (unsigned long long)nq * n) return;
    const unsigned long long q = t / n, r = t % n;
    if (!alive[e0 + r]) return;
    const double *p = partial + t * G * 2;
    double s1 = 0.0, s2 = 0.0;
    for (unsigned g = 0; g < G; ++g) {
        s1 += p[2 * g];
        s2 += p[2 * g + 1];
    }
    l1[q * stride + e0 + r] = s1 / E;
    l2[q * stride + e0 + r] = sqrt(s2 / E);
}

// A distance as an order-preserving key: a distance is +0, positive, +inf or NaN; NaN ranks after +inf.
__device__ __forceinline__ unsigned long long dist_key(double d) {
    if (d != d) return 0x7ff8000000000000ULL;
    const unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b << 1) == 0 ? 0 : b;
}

struct IndexSelArgs {
    // the first pass (in_key == nullptr): the entries 0 .. n, each query's key from dist[q * stride + e], dead rows
    // skipped; later passes: the survivors in_key / in_id [q][n]
    const double *dist;
    const unsigned char *alive;
    unsigned long long stride;
    const unsigned long long *in_key, *in_id;
    unsigned long long n;
    int k;
    int sort_n;                         // a power of two, at most kIdxSelN: the pairs one CTA sorts
    unsigned long long *out_key, *out_id; // [q][gridDim.x][k]
};

// Grid (ceil(n / sort_n), nq), kIdxSelThreads threads, 2 * kIdxSelN u64 of dynamic shared memory.
__global__ void __launch_bounds__(kIdxSelThreads) k_index_select(const IndexSelArgs a) {
    extern __shared__ unsigned long long sel[]; // keys [sort_n], then ids [sort_n]
    unsigned long long *sk = sel, *si = sel + a.sort_n;
    const unsigned long long q = blockIdx.y, base = (unsigned long long)blockIdx.x * a.sort_n;
    const int N = a.sort_n;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const unsigned long long j = base + i;
        unsigned long long key = kIdxNone, id = kIdxNone;
        if (j < a.n) {
            if (!a.in_key) {
                if (a.alive[j]) key = dist_key(a.dist[q * a.stride + j]), id = j;
            } else {
                key = a.in_key[q * a.n + j];
                id = a.in_id[q * a.n + j];
            }
        }
        sk[i] = key;
        si[i] = id;
    }
    for (int size = 2; size <= N; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < N / 2; t += blockDim.x) {
                const int i = 2 * t - (t & (stride - 1)), j = i + stride;
                const bool up = (i & size) == 0;
                const unsigned long long ki = sk[i], kj = sk[j], ii = si[i], ij = si[j];
                const bool j_first = kj < ki || (kj == ki && ij < ii);
                if (j_first == up) {
                    sk[i] = kj, sk[j] = ki;
                    si[i] = ij, si[j] = ii;
                }
            }
        }
    __syncthreads();
    const unsigned long long o = (q * gridDim.x + blockIdx.x) * a.k;
    for (int i = threadIdx.x; i < a.k; i += blockDim.x) {
        a.out_key[o + i] = i < N ? sk[i] : kIdxNone;
        a.out_id[o + i] = i < N ? si[i] : kIdxNone;
    }
}

// One thread per (query, position): the chosen entry's id and both distances, or NO_ENTRY and NaN.
__global__ void k_index_finish(const unsigned long long *id, const double *l1, const double *l2, unsigned long long stride,
                               int nq, int k, unsigned long long *entries, double *l1_out, double *l2_out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq * k) return;
    const unsigned long long q = t / k, e = id[t];
    const bool none = e == kIdxNone;
    entries[t] = e;
    l1_out[t] = none ? __longlong_as_double(0x7ff8000000000000LL) : l1[q * stride + e];
    l2_out[t] = none ? __longlong_as_double(0x7ff8000000000000LL) : l2[q * stride + e];
}

} // namespace rk
