// prefill.cuh — batched forward over T tokens with the weights read ONCE for all of them
// (SURVEY 8f N1: forward(vector, GPT) with maxGPT > 1, rwkv.h:339-376, 395-413; N3: MODE::PARRALEL,
// rwkv.cu:238-240, 336, 378-380).
//
// With T tokens every projection is a GEMM  Y[out][t] = sum_j W'[out][j] * q[t][j]  between the int8 weight
// matrix and the tokens' activation limbs - the same exact-integer formulation as the decode kernel (common.cuh):
// each token's vector is quantised to a 23-bit integer and its three byte limbs are three columns of the B
// operand (two unsigned planes, one signed plane), so the tensor cores compute bit for bit what the IDP.4A
// loop computes: wgmma.mma_async m64nNk32, s8 x u8 / s8 x s8 -> s32 in registers, planes recombined in the epilogue.
// No dequantisation, no fp error, and the weights go straight from HBM to shared memory by TMA in the
// K-major, 128-byte-swizzled layout the MMA wants (they are stored [out][in] = K-major already).
//
// One GEMM launch: grid = (ceil(M / 64), ksplit); CTA = two consumer warpgroups + one TMA producer warp. Tile
// 64 rows x (3 Tp) x 128 bytes of K per stage; each consumer warpgroup owns NB = Tp / 32 blocks of 16 tokens in
// all three planes (at most 3 x 4 x 8 accumulator registers per thread). NB is a template parameter so that every
// wgmma sits on a uniform path (a data-dependent branch around them makes the compiler serialise them). Split-K
// partial sums are added with integer atomics (exact, order-free). Any K that is a multiple of 16 (every n_embed the
// loader accepts) works: K tiles round up and the out-of-bounds tail of the last one is zero-filled by TMA in both
// operands; split-K is used only when every split is a whole number of 128-byte tiles.
// Everything around the GEMMs (layernorm, token shift, WKV scan over t, activations, quantisation) is plain
// CUDA, one small kernel per step, with the reference's rounding points (rwkv.cu:40-57, 221-259, 313-465).
//
// A pass is ragged: its tokens belong to independent streams, each on its own state slot. A per-token
// descriptor (slot, "first in pass", "last in pass"), uploaded with the tokens, tells the step kernels where a
// token's predecessor lives (the previous row, or the slot's state) and where the state goes after it. GPT mode is
// one stream on slot 0, MODE::PARRALEL is T streams of one token on slots 0..T-1. The head runs on the rows of a
// row map (every token, or the last token of each stream) into a compact logits buffer.
#pragma once
#include <cuda.h>

#include <string>
#include <vector>

#include "common.cuh"

namespace rk {

constexpr int kPrefillMinTokens = 8;   // shorter calls run token by token through the decode kernel
constexpr int kPfMaxTokens = 128;      // tokens per pass
constexpr int kPfBM = 64, kPfBK = 128, kPfStages = 3;
constexpr int kPfConsumerWGs = 2;
constexpr int kPfThreads = 128 * kPfConsumerWGs + 32;
constexpr int kPfTokenAlign = 16 * kPfConsumerWGs; // padded token count: the same number of blocks per warpgroup

// Stream descriptor of one token of a pass: its state slot and two flags. A "last" token stores its state into its own
// slot, which need not be the slot its segment's "first" token loaded: a speculative step (speculate.cuh) continues one
// segment through draft rows on other slots. Every other producer of descriptors (pass_layout, k_gen_feedback,
// k_beam_select, the batcher) names one slot per segment, for which the two are the same.
constexpr uint32_t kDescFirst = 1u << 31; // token shift and WKV start from the slot's state, not from token t - 1
constexpr uint32_t kDescLast = 1u << 30;  // the token's slot receives the state after this token
constexpr uint32_t kDescSlot = kDescLast - 1u;
__host__ __device__ __forceinline__ size_t desc_slot(uint32_t d) { return (size_t)(d & kDescSlot); }

// Everything a pass reads that changes from pass to pass; one host-to-device copy per pass. The kernels of a
// recorded graph read it through fixed pointers, so the layout is data and never part of the graph.
// Snapshots (prefix caches, prefix.cuh): snap[t] = e + 1 writes the state after token t into entry e of the pool whose
// xy, aa, bb and dd arrays start at pool[0..3] (entry stride L * E, like the slots); 0 takes none. A zero-initialised
// descriptor takes no snapshot, so every producer that fills only tokens and desc stays correct, and a graph recorded
// for one pass serves passes with and without a cache.
struct PassDesc {
    unsigned long long tokens[kPfMaxTokens];
    uint32_t desc[kPfMaxTokens];
    int rows[kPfMaxTokens]; // head row i = token rows[i] of the pass
    int out_row0;           // head row i goes to logits row out_row0 + i
    uint32_t snap[kPfMaxTokens];
    double *pool[4];
};
enum : int { kPoolXY = 0, kPoolAA, kPoolBB, kPoolDD };

// ---- LoRA adapters (include/rwkv_b200.h, "adapters") ----------------------------------------------------------
// A slot's adapter record lives in a per-slot device table, so a token finds its adapter through its descriptor's slot
// and no layout code knows about adapters. Matrix m of the record: A [L][rank][in] and B [L][out][rank] in f32, or both
// NULL (not adapted). rank 0: the slot is unbound.
constexpr int kAdMats = 7, kAdMaxRank = 64;
enum : int { kAdAttK = 0, kAdAttV, kAdAttR, kAdAttO, kAdFfnK, kAdFfnV, kAdFfnR };
struct AdapterRec {
    int rank;
    double scale;
    const float *A[kAdMats], *B[kAdMats];
};

// ---- wgmma / TMA helpers ---------------------------------------------------------------------------------
__device__ __forceinline__ void pf_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(bar), "r"(parity)
                     : "memory");
    }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(map), "r"(c0), "r"(c1), "r"(bar)
                 : "memory");
}
// Shared-memory matrix descriptor of a K-major operand tile in the 128-byte swizzle (the layout TMA writes):
// rows of 128 bytes, 8-row groups 1024 bytes apart (SBO); LBO is unused for swizzled K-major layouts. A step of
// 32 bytes along K inside the swizzle atom advances the start address only.
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// d[64 x 16] += A[64 x 32] (s8) * B[16 x 32]^T (u8 or s8), both from shared memory, K-major.
template <bool BSigned>
__device__ __forceinline__ void wgmma_i8_n16(int (&d)[8], uint64_t da, uint64_t db) {
    if constexpr (BSigned) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}"
                     : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                     : "l"(da), "l"(db), "r"(1)
                     : "memory");
    } else {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.u8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}"
                     : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                     : "l"(da), "l"(db), "r"(1)
                     : "memory");
    }
}

struct GemmArgs {
    CUtensorMap map_a; // weights  [M][K]  int8, box 64 x 128
    CUtensorMap map_b; // limbs    [rows][K] u8, box Tp x 128 (three loads per stage: planes 0, 1, 2)
    int M, K;          // rows of the weight matrix (this launch), bytes per row
    int Tp;            // padded token count (multiple of kPfTokenAlign, <= 128)
    int b_row0;        // first limb row of this GEMM's vector: planes at b_row0, +Tp, +2Tp
    int ksplit;        // gridDim.y
    int *C;            // [M][3 Tp] int32, zeroed; columns [0, 2Tp) unsigned planes, [2Tp, 3Tp) signed plane
};

// C[m][n] += sum_k A[m][k] * B[n][k] over this CTA's K range; NB = Tp / kPfTokenAlign.
template <int NB>
__global__ void __launch_bounds__(kPfThreads, 1) k_gemm_i8(const __grid_constant__ GemmArgs g) {
    extern __shared__ __align__(1024) uint8_t pf_smem[];
    const uint32_t base = (smem_u32(pf_smem) + 1023u) & ~1023u;
    const int Tp = g.Tp;
    const uint32_t a_bytes = kPfBM * kPfBK, b_bytes = 3u * (uint32_t)Tp * kPfBK, stage_bytes = a_bytes + b_bytes;
    const uint32_t bars = base + kPfStages * stage_bytes; // full[stages], empty[stages]
    auto full = [&](int s) { return bars + 8u * (uint32_t)s; };
    auto empty = [&](int s) { return bars + 8u * (uint32_t)(kPfStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * kPfBM;
    // K tiles round up: the last tile of a K that is not a multiple of 128 (ksplit = 1 only) reaches past the end of
    // both operands, and TMA fills that part of the box with zeros (and still counts the whole box's bytes).
    const int kper = g.K / g.ksplit, k0 = blockIdx.y * kper, nkt = (kper + kPfBK - 1) / kPfBK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kPfStages; ++s) {
            mbar_init(full(s), 1);
            mbar_init(empty(s), 4 * kPfConsumerWGs); // one arrival per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 4 * kPfConsumerWGs) {
        if (lane == 0) { // ---- TMA producer ----
            for (int kt = 0; kt < nkt; ++kt) {
                const int s = kt % kPfStages;
                if (kt >= kPfStages) pf_mbar_wait(empty(s), (uint32_t)((kt / kPfStages - 1) & 1));
                mbar_expect_tx(full(s), stage_bytes);
                const uint32_t sa = base + (uint32_t)s * stage_bytes, sb = sa + a_bytes;
                const int kc = k0 + kt * kPfBK;
                tma_load_2d(sa, &g.map_a, kc, m0, full(s));
                for (int pl = 0; pl < 3; ++pl) tma_load_2d(sb + (uint32_t)(pl * Tp) * kPfBK, &g.map_b, kc, g.b_row0 + pl * Tp, full(s));
            }
        }
        return;
    }

    // ---- consumers: warpgroup wg owns token blocks wg * NB .. wg * NB + NB - 1 ----
    const int wg = warp >> 2, wl = warp & 3;
    int acc[3][NB][8];
#pragma unroll
    for (int pl = 0; pl < 3; ++pl)
#pragma unroll
        for (int i = 0; i < NB; ++i)
#pragma unroll
            for (int r = 0; r < 8; ++r) acc[pl][i][r] = 0;
    for (int kt = 0; kt < nkt; ++kt) {
        const int s = kt % kPfStages;
        pf_mbar_wait(full(s), (uint32_t)((kt / kPfStages) & 1));
        const uint32_t sa = base + (uint32_t)s * stage_bytes, sb = sa + a_bytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kPfBK / 32; ++k) { // K = 32 bytes of int8 per instruction
            const uint64_t da = wgmma_desc_k128(sa + 32u * k);
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                const uint32_t bj = sb + (uint32_t)(16 * (wg * NB + i)) * kPfBK + 32u * k;
                wgmma_i8_n16<false>(acc[0][i], da, wgmma_desc_k128(bj));                                // plane 0 (unsigned)
                wgmma_i8_n16<false>(acc[1][i], da, wgmma_desc_k128(bj + (uint32_t)Tp * kPfBK));         // plane 1 (unsigned)
                wgmma_i8_n16<true>(acc[2][i], da, wgmma_desc_k128(bj + 2u * (uint32_t)Tp * kPfBK));     // plane 2 (signed)
            }
        }
        wgmma_commit();
        wgmma_wait_all();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s)); // this warp's MMAs have read the stage
    }

    // ---- epilogue: accumulator fragment of m64nNk32 - rows 16 * wl + lane / 4 (+8), columns 2 * (lane % 4) (+1, +8)
    const int r0 = m0 + 16 * wl + (lane >> 2);
#pragma unroll
    for (int pl = 0; pl < 3; ++pl)
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            const int j = wg * NB + i;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int col = pl * Tp + 16 * j + 8 * h + 2 * (lane & 3);
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int row = r0 + 8 * half;
                    if (row < g.M) {
                        int *c = g.C + (size_t)row * 3 * Tp + col;
                        atomicAdd(c, acc[pl][i][4 * h + 2 * half]);
                        atomicAdd(c + 1, acc[pl][i][4 * h + 2 * half + 1]);
                    }
                }
            }
        }
}

// ---- element-wise kernels ----------------------------------------------------------------------------------
// Block-wide sum over 256 threads in double, fixed tree (deterministic); everybody gets the result.
__device__ __forceinline__ double pf_block_sum(double v, double *sh) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
    return t;
}
__device__ __forceinline__ uint32_t pf_block_max(uint32_t v, uint32_t *sh) {
    __syncwarp();
    v = __reduce_max_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = max(t, sh[w]);
    return t;
}
// mean and 1/std of a row of E doubles with the reference's f32 rounding (rwkv.cu:412-465, 43-44)
__device__ __forceinline__ void pf_row_stats(const double *x, int E, double *sh, double &mean, double &rstd) {
    double s = 0.0;
    for (int j = threadIdx.x; j < E; j += blockDim.x) s += x[j];
    s = pf_block_sum(s, sh);
    const float mean_acc = (float)s;
    const double mean_f = (double)(mean_acc / (float)E);
    double q = 0.0;
    for (int j = threadIdx.x; j < E; j += blockDim.x) {
        const double d = x[j] - mean_f;
        q += d * d;
    }
    q = pf_block_sum(q, sh);
    mean = (double)mean_acc / (double)E;
    rstd = 1.0 / (double)sqrtf((float)q / (float)(E - 1));
}

// x[t] = LN0(emb[token_t])  (rwkv.cu:513-524)
__global__ void __launch_bounds__(256) k_pf_embed(const float *emb, const double *ln, const unsigned long long *tokens, int E, double *x) {
    __shared__ double sh[8];
    __shared__ double row[5120];
    const int t = blockIdx.x;
    const float *e = emb + (size_t)tokens[t] * E;
    for (int j = threadIdx.x; j < E; j += blockDim.x) row[j] = (double)e[j];
    __syncthreads();
    double mean, rstd;
    pf_row_stats(row, E, sh, mean, rstd);
    for (int j = threadIdx.x; j < E; j += blockDim.x) x[(size_t)t * E + j] = ln[j] * ((row[j] - mean) * rstd) + ln[E + j];
}

// Layernorm of row rows[t] of x with parameters lw, lb -> lnout[t] (block = output row)
__global__ void __launch_bounds__(256) k_pf_ln(const double *x, const double *lw, const double *lb, int E, const int *rows, double *lnout) {
    __shared__ double sh[8];
    const int t = blockIdx.x;
    const double *xr = x + (size_t)rows[t] * E;
    double mean, rstd;
    pf_row_stats(xr, E, sh, mean, rstd);
    for (int j = threadIdx.x; j < E; j += blockDim.x) lnout[(size_t)t * E + j] = lw[j] * ((xr[j] - mean) * rstd) + lb[j];
}

// Token shift + scale + quantisation of one token (block = token): NV vectors
//   f_v = float(m_v * ln_t + (1 - m_v) * prev),  xs_v = float(f_v * r_v)   (rwkv.cu:313-392)
// prev = the state of the token's slot for the first token of a stream in the pass, else ln of token t - 1.
// Limbs of vector v, plane p, token t at row (v*3 + p) * Tp + t of `limbs` (K = E bytes per row);
// scale[v*Tp + t] = S, offs[v*Tp + t] = sum_j f * oc. The activations are rounded to 22 mantissa bits first,
// exactly like the decode kernel's exchange words (exchange.cuh), so both paths quantise the same numbers.
struct MixArgs {
    const double *ln;      // [T][E]
    const double *state;   // [slots][L][E] + layer offset applied by the host: pointer to [E] of slot 0
    size_t slot_stride;    // doubles between slots
    const uint32_t *desc;  // [T] stream descriptors
    const double *mix[3];
    const float *r[3], *oc[3];
    int nv, E, Tp;
    uint8_t *limbs;
    double *scale, *offs;
    float *fout; // NULL, or [nv][Tp][E]: the mixed activation f (before the r-scaling and the 22-bit rounding), for adapters
};
__global__ void __launch_bounds__(256) k_pf_mix_quant(const __grid_constant__ MixArgs a) {
    __shared__ double sh[8];
    __shared__ uint32_t shm[8];
    const int t = blockIdx.x, E = a.E;
    const uint32_t d = a.desc[t];
    const double *cur = a.ln + (size_t)t * E;
    const double *prev = (d & kDescFirst) ? a.state + desc_slot(d) * a.slot_stride : a.ln + (size_t)(t - 1) * E;
    for (int v = 0; v < a.nv; ++v) {
        uint32_t mx = 0;
        double of = 0.0;
        for (int j = threadIdx.x; j < E; j += blockDim.x) {
            const double m = a.mix[v][j];
            const float f = (float)(m * cur[j] + (1.0 - m) * prev[j]);
            if (a.fout) a.fout[((size_t)v * a.Tp + t) * E + j] = f;
            const float xs = (float)((double)f * (double)a.r[v][j]);
            mx = max(mx, ((__float_as_uint(xs) + 2u) & ~3u) & 0x7fffffffu);
            of += (double)f * (double)a.oc[v][j];
        }
        mx = pf_block_max(mx, shm);
        of = pf_block_sum(of, sh);
        const float mf = __uint_as_float(mx);
        const float inv = quant_scale(mf);
        if (threadIdx.x == 0) {
            a.scale[v * a.Tp + t] = (double)mf * (1.0 / (double)kQMax);
            a.offs[v * a.Tp + t] = of;
        }
        uint8_t *p0 = a.limbs + ((size_t)(v * 3 + 0) * a.Tp + t) * E, *p1 = a.limbs + ((size_t)(v * 3 + 1) * a.Tp + t) * E,
                *p2 = a.limbs + ((size_t)(v * 3 + 2) * a.Tp + t) * E;
        for (int j = threadIdx.x; j < E; j += blockDim.x) {
            const double m = a.mix[v][j];
            const float f = (float)(m * cur[j] + (1.0 - m) * prev[j]);
            const float xs = __uint_as_float((__float_as_uint((float)((double)f * (double)a.r[v][j])) + 2u) & ~3u);
            const uint32_t q = __float_as_uint(fmaf(xs, inv, 12582912.0f)) - 0x4B400000u;
            p0[j] = (uint8_t)q;
            p1[j] = (uint8_t)(q >> 8);
            p2[j] = (uint8_t)(q >> 16);
        }
    }
}

// Quantise rows of pre-scaled f32 activations xs[t][N] (already rounded to 22 bits) -> limbs of one vector;
// offs[t] = sum_j a[t][j] * oc[j] where a = the unscaled activation.
__global__ void __launch_bounds__(256) k_pf_quant_rows(const float *xs, const float *a, const float *oc, int N, int Tp, uint8_t *limbs, double *scale,
                                                       double *offs) {
    __shared__ double sh[8];
    __shared__ uint32_t shm[8];
    const int t = blockIdx.x;
    const float *x = xs + (size_t)t * N, *ar = a + (size_t)t * N;
    uint32_t mx = 0;
    double of = 0.0;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
        mx = max(mx, __float_as_uint(x[j]) & 0x7fffffffu);
        of += (double)ar[j] * (double)oc[j];
    }
    mx = pf_block_max(mx, shm);
    of = pf_block_sum(of, sh);
    const float mf = __uint_as_float(mx);
    const float inv = quant_scale(mf);
    if (threadIdx.x == 0) {
        scale[t] = (double)mf * (1.0 / (double)kQMax);
        offs[t] = of;
    }
    uint8_t *p0 = limbs + ((size_t)0 * Tp + t) * N, *p1 = limbs + ((size_t)1 * Tp + t) * N, *p2 = limbs + ((size_t)2 * Tp + t) * N;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
        const uint32_t q = __float_as_uint(fmaf(x[j], inv, 12582912.0f)) - 0x4B400000u;
        p0[j] = (uint8_t)q;
        p1[j] = (uint8_t)(q >> 8);
        p2[j] = (uint8_t)(q >> 16);
    }
}

// value of output row m for token t from the three plane sums: S * ((t2*256 + t1)*256 + t0) + off, plus an adapter's
// delta. A token without one adds -0.0, which leaves every double (signed zeros included) exactly as it was.
__device__ __forceinline__ float pf_combine(const int *C, int Tp, size_t m, int t, double S, double off, double delta = -0.0) {
    const int *c = C + m * 3 * Tp;
    const long long tot = (((long long)c[2 * Tp + t] << 8) + (long long)c[Tp + t]) * 256 + (long long)c[t];
    return (float)(S * (double)tot + off + delta);
}

// WKV over the pass (rwkv.cu:221-259): thread = channel, sequential over t. The state is loaded from the slot at
// a stream's first token and stored into the slot of each token marked last. Writes the unscaled rwkv (f32) and xs = rwkv * r_out
// rounded to 22 bits.
struct WkvArgs {
    const int *Ck, *Cv, *Cr;          // [E][3 Tp]
    const double *scale, *offs;       // [3][Tp] (k, v, r)
    const double *decay, *bonus, *expdecay; // [E] of this layer
    const float *ro;                  // [E]
    double *aa, *bb;                  // state of slot 0 for this layer
    size_t slot_stride;
    const uint32_t *desc;             // [T] stream descriptors
    int E, T, Tp;
    float *rw, *xs;                   // [T][E]
    const double *dk, *dv, *dr;       // NULL, or the adapters' deltas [T][E]
    const PassDesc *pass;             // its snap and pool (snapshots of aa, bb)
    size_t lo;                        // this layer's offset inside an entry
};
__global__ void __launch_bounds__(256) k_pf_wkv(const __grid_constant__ WkvArgs a) {
    __shared__ uint32_t desc[kPfMaxTokens], snap[kPfMaxTokens]; // read once per t by every thread of the sequential scan
    for (int t = threadIdx.x; t < a.T; t += blockDim.x) {
        desc[t] = a.desc[t];
        snap[t] = a.pass->snap[t];
    }
    __syncthreads();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.E) return;
    const double wd = a.decay[c], ub = a.bonus[c], ew = a.expdecay[c];
    const float ro = a.ro[c];
    double aa = 0.0, bb = 0.0;
    size_t so = 0;
    for (int t = 0; t < a.T; ++t) {
        const uint32_t d = desc[t];
        if (d & kDescFirst) {
            so = desc_slot(d) * a.slot_stride + c;
            aa = a.aa[so];
            bb = a.bb[so];
        }
        const size_t tc = (size_t)t * a.E + c;
        const float kf = pf_combine(a.Ck, a.Tp, (size_t)c, t, a.scale[0 * a.Tp + t], a.offs[0 * a.Tp + t], a.dk ? a.dk[tc] : -0.0);
        const float vf = pf_combine(a.Cv, a.Tp, (size_t)c, t, a.scale[1 * a.Tp + t], a.offs[1 * a.Tp + t], a.dv ? a.dv[tc] : -0.0);
        const float rf = pf_combine(a.Cr, a.Tp, (size_t)c, t, a.scale[2 * a.Tp + t], a.offs[2 * a.Tp + t], a.dr ? a.dr[tc] : -0.0);
        const double vv = (double)vf;
        const double e1 = exp(ub + wd + (double)kf);
        double y = (aa + e1 * vv) / (bb + e1);
        y = (1.0 / (1.0 + (double)expf(-rf))) * y;
        const double ek = exp((double)kf);
        aa = (aa + ek * vv) * ew;
        bb = (bb + ek) * ew;
        if (d & kDescLast) { // into the token's own slot, like k_pf_store_state (speculate.cuh: a row per draft)
            const size_t o = desc_slot(d) * a.slot_stride + c;
            a.aa[o] = aa;
            a.bb[o] = bb;
        }
        if (const uint32_t e = snap[t]) { // the state after this token into a prefix cache entry
            const size_t o = (size_t)(e - 1) * a.slot_stride + a.lo + c;
            a.pass->pool[kPoolAA][o] = aa;
            a.pass->pool[kPoolBB][o] = bb;
        }
        const float rw = (float)y;
        a.rw[(size_t)t * a.E + c] = rw;
        a.xs[(size_t)t * a.E + c] = __uint_as_float((__float_as_uint((float)((double)rw * (double)ro)) + 2u) & ~3u);
    }
}

// x[t][j] = f32(x) + y  (out-proj, rwkv.cu:548-553)   /   x[t][j] += kv * sr  (ffn, rwkv.cu:574-577)
// delta: NULL, or the adapters' deltas [T][E].
__global__ void __launch_bounds__(256) k_pf_residual(const int *C, const double *scale, const double *offs, const float *sr, int E, int T, int Tp, double *x,
                                                     const double *delta) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)T * E) return;
    const int t = (int)(i / E), j = (int)(i % E);
    const float y = pf_combine(C, Tp, (size_t)j, t, scale[t], offs[t], delta ? delta[i] : -0.0);
    if (sr == nullptr) x[i] = (double)((float)x[i] + y);
    else x[i] = x[i] + (double)(y * sr[i]);
}

// sigmoid(ffn r) [T][E]; a = relu(k)^2 [T][4E] and xs = a * r_ffnv rounded to 22 bits (rwkv.cu:566-573).
// dr, dk: NULL, or the adapters' deltas of ffn r [T][E] and ffn k [T][4E].
__global__ void __launch_bounds__(256) k_pf_ffn_act(const int *Cr, const int *Ck, const double *scale, const double *offs, const float *rfv, int E, int T,
                                                    int Tp, float *sr, float *act, float *xs, const double *dr, const double *dk) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)T * 5 * E) return;
    const int t = (int)(i / (5 * (size_t)E)), j = (int)(i % (5 * (size_t)E));
    if (j < E) {
        const float y = pf_combine(Cr, Tp, (size_t)j, t, scale[0 * Tp + t], offs[0 * Tp + t], dr ? dr[(size_t)t * E + j] : -0.0);
        sr[(size_t)t * E + j] = (float)(1.0 / (1.0 + exp(-(double)y)));
    } else {
        const int k = j - E;
        float a = pf_combine(Ck, Tp, (size_t)k, t, scale[1 * Tp + t], offs[1 * Tp + t], dk ? dk[(size_t)t * 4 * E + k] : -0.0);
        a = a > 0.0f ? a : 0.0f;
        a = a * a;
        act[(size_t)t * 4 * E + k] = a;
        xs[(size_t)t * 4 * E + k] = __uint_as_float((__float_as_uint((float)((double)a * (double)rfv[k])) + 2u) & ~3u);
    }
}

// logits[*row0 + h][v] of head row h from the head GEMM (rwkv.cu:589)
__global__ void __launch_bounds__(256) k_pf_logits(const int *C, const double *scale, const double *offs, int V, int H, int Tp, const int *row0,
                                                   float *logits) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)H * V) return;
    const int h = (int)(i / V), v = (int)(i % V);
    logits[(size_t)*row0 * V + i] = pf_combine(C, Tp, (size_t)v, h, scale[h], offs[h]);
}

// token-shift state after the pass: state[slot] = ln[t] for the last token t of each stream in the pass, and array
// `which` of entry snap[t] - 1 at layer offset lo for a snapshot token (block = token; the blocks of the other tokens
// leave at once)
__global__ void __launch_bounds__(256) k_pf_store_state(const double *ln, int E, const PassDesc *pass, size_t slot_stride, double *state,
                                                        int which, size_t lo) {
    const int t = blockIdx.x;
    const uint32_t d = pass->desc[t], e = pass->snap[t];
    if (d & kDescLast) {
        double *dst = state + desc_slot(d) * slot_stride;
        for (int j = threadIdx.x; j < E; j += blockDim.x) dst[j] = ln[(size_t)t * E + j];
    }
    if (e) {
        double *dst = pass->pool[which] + (size_t)(e - 1) * slot_stride + lo;
        for (int j = threadIdx.x; j < E; j += blockDim.x) dst[j] = ln[(size_t)t * E + j];
    }
}

// ---- adapter deltas: delta[t][m] = s * sum_i B[m][i] * h[t][i],  h[t][i] = sum_j A[i][j] * f[t][j], both in f64 ----
// One adaptation point adapts nv <= 3 matrices of layer l whose inputs are rows of f. Each token's sums run in an order
// fixed by the shapes alone (lane-strided products and a butterfly for h, i ascending for delta), so a token's delta
// depends only on its own f and its slot's adapter, never on the other tokens of the pass.
struct AdArgs {
    const AdapterRec *table; // [slots]
    const uint32_t *desc;    // [T] stream descriptors
    int T, l;
    int nv, mat[3], K, M[3]; // matrix, input width and output width of each vector
    const float *f;          // vector v, token t at f + v * f_vstride + t * K
    size_t f_vstride;
    double *h;               // [3][T][kAdMaxRank]
    double *delta;           // vector v, token t at delta + v * d_vstride + t * M[v]
    size_t d_vstride;
};
constexpr int kAdThreads = 256;
constexpr int kAdShrinkTokens = kAdThreads / 32; // tokens of a k_ad_shrink block: one per warp
constexpr int kAdExpandTokens = 4;               // tokens of a k_ad_expand block, in turn

// h: block (i, v, g) = rank row i of matrix v for the tokens of group g, one per warp. A row of A is read from HBM once
// per pass and from L2 by the other groups of tokens with the same adapter.
__global__ void __launch_bounds__(kAdThreads) k_ad_shrink(const __grid_constant__ AdArgs a) {
    const int i = blockIdx.x, v = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.z * kAdShrinkTokens + warp;
    if (t < a.T) {
        const AdapterRec &r = a.table[desc_slot(a.desc[t])];
        const float *A = r.A[a.mat[v]];
        if (A == nullptr || i >= r.rank) return;
        const float *row = A + ((size_t)a.l * r.rank + i) * a.K, *f = a.f + v * a.f_vstride + (size_t)t * a.K;
        double s = 0.0;
        for (int j = lane; j < a.K; j += 32) s += (double)row[j] * (double)f[j];
        s = warp_sum(s);
        if (lane == 0) a.h[((size_t)v * a.T + t) * kAdMaxRank + i] = s;
    }
}

// delta: block (x, v, g) = output rows of vector v for the tokens of group g, thread = output row m, sequential over
// the group's tokens (a row of B stays in L1 across them). Tokens without the matrix get -0.0, which pf_combine adds
// without changing a bit.
__global__ void __launch_bounds__(kAdThreads) k_ad_expand(const __grid_constant__ AdArgs a) {
    const int v = blockIdx.y, M = a.M[v];
    const int m = blockIdx.x * kAdThreads + threadIdx.x;
    if (m >= M) return;
    double *out = a.delta + v * a.d_vstride + m;
    const int t1 = min(a.T, (int)(blockIdx.z + 1) * kAdExpandTokens);
    for (int t = blockIdx.z * kAdExpandTokens; t < t1; ++t) {
        const AdapterRec &r = a.table[desc_slot(a.desc[t])];
        const float *B = r.B[a.mat[v]];
        if (B == nullptr || r.rank == 0) {
            out[(size_t)t * M] = -0.0;
            continue;
        }
        const float *b = B + ((size_t)a.l * M + m) * r.rank;
        const double *h = a.h + ((size_t)v * a.T + t) * kAdMaxRank;
        double s = 0.0;
        for (int i = 0; i < r.rank; ++i) s += (double)b[i] * h[i];
        out[(size_t)t * M] = r.scale * s;
    }
}

// ---- host side -------------------------------------------------------------------------------------------------
typedef CUresult (*PfnEncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                   const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct PrefillState {
    bool disabled = false;
    int min_tokens = kPrefillMinTokens; // shorter calls run token by token through the decode kernel
    bool ready = false;
    PfnEncodeTiled encode = nullptr;
    PassDesc *pass = nullptr;   // device copy of the current pass's tokens, descriptors and head row map
    int *iota = nullptr;        // [kPfMaxTokens] 0, 1, 2, ...: the row map of the per-layer layernorms
    uint32_t *head_desc = nullptr; // [kPfMaxTokens] "first" on slot 0: the head's quantisation has no token shift
    double *x = nullptr, *ln = nullptr, *scale = nullptr, *offs = nullptr;
    uint8_t *limbs = nullptr;   // [3 vectors][3 planes][Tp][4E] worst case
    int *C = nullptr;           // the largest accumulator set of a step
    float *rw = nullptr, *xs = nullptr, *sr = nullptr, *act = nullptr;
    // adapters: `adapt` is set by the caller for the passes of a call that names a bound slot, which then add the
    // deltas of the slots' records in `ad_table`. Allocated at the first such pass.
    bool adapt = false;
    const AdapterRec *ad_table = nullptr;
    float *ad_f = nullptr;                    // [3][T][E] the mixed activations of k_pf_mix_quant
    double *ad_h = nullptr, *ad_d = nullptr;  // [3][T][kAdMaxRank], [5][T][E]
    unsigned long long launches = 0;
    std::string err;
    // One pass is ~21 small launches per layer: replayed as a CUDA graph per (tokens, head rows) shape, so that a
    // caller stepping S streams or prefilling in equal chunks pays the host side once. Slots and stream boundaries
    // are data in `pass`, never part of the key: a decode loop whose set of slots changes replays the same graph.
    struct Graph {
        int T, H;
        bool adapt;
        cudaGraphExec_t exec;
        unsigned long long launches;
    };
    std::vector<Graph> graphs;
    bool use_graph = true;
    unsigned long long records = 0; // graphs recorded since load (a shape that left the cache is recorded again)
};
inline std::string &prefill_err_slot() {
    static thread_local std::string e;
    return e;
}
inline const char *prefill_error() { return prefill_err_slot().c_str(); }
inline bool prefill_enabled(const PrefillState &s) { return !s.disabled; }
inline unsigned long long prefill_launches(PrefillState &s) {
    const unsigned long long n = s.launches;
    s.launches = 0;
    return n;
}
inline void prefill_free(PrefillState &s) {
    for (auto &g : s.graphs) cudaGraphExecDestroy(g.exec);
    s.graphs.clear();
    for (void *p : {(void *)s.pass, (void *)s.iota, (void *)s.head_desc, (void *)s.x, (void *)s.ln, (void *)s.scale, (void *)s.offs, (void *)s.limbs,
                    (void *)s.C, (void *)s.rw, (void *)s.xs, (void *)s.sr, (void *)s.act, (void *)s.ad_f, (void *)s.ad_h, (void *)s.ad_d})
        if (p) cudaFree(p);
    s = PrefillState{};
}
inline int pf_fail(const char *what, cudaError_t e) {
    prefill_err_slot() = std::string("batched prefill: ") + what + ": " + cudaGetErrorString(e);
    return 100 + (int)e;
}
#define PF_CK(call)                                   \
    do {                                              \
        cudaError_t e__ = (call);                     \
        if (e__ != cudaSuccess) return pf_fail(#call, e__); \
    } while (0)

inline int prefill_init(PrefillState &s, const Params &p) {
    if (s.ready) return 0;
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    PF_CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (!fn || q != cudaDriverEntryPointSuccess) {
        prefill_err_slot() = "batched prefill: the driver does not export cuTensorMapEncodeTiled";
        return 3;
    }
    s.encode = (PfnEncodeTiled)fn;
    const size_t E = (size_t)p.E, V = kVocab, T = kPfMaxTokens;
    PF_CK(cudaMalloc((void **)&s.pass, sizeof(PassDesc)));
    PF_CK(cudaMalloc((void **)&s.iota, T * sizeof(int)));
    PF_CK(cudaMalloc((void **)&s.head_desc, T * sizeof(uint32_t)));
    {
        std::vector<int> iota(T);
        std::vector<uint32_t> first(T, kDescFirst);
        for (size_t t = 0; t < T; ++t) iota[t] = (int)t;
        PF_CK(cudaMemcpy(s.iota, iota.data(), T * sizeof(int), cudaMemcpyHostToDevice));
        PF_CK(cudaMemcpy(s.head_desc, first.data(), T * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    PF_CK(cudaMalloc((void **)&s.x, T * E * 8));
    PF_CK(cudaMalloc((void **)&s.ln, T * E * 8));
    PF_CK(cudaMalloc((void **)&s.scale, 3 * T * 8));
    PF_CK(cudaMalloc((void **)&s.offs, 3 * T * 8));
    PF_CK(cudaMalloc((void **)&s.limbs, 9 * T * 4 * E));
    PF_CK(cudaMalloc((void **)&s.C, std::max((size_t)5 * E, V) * 3 * T * 4 + 3 * E * 3 * T * 4));
    PF_CK(cudaMalloc((void **)&s.rw, T * E * 4));
    PF_CK(cudaMalloc((void **)&s.xs, T * 4 * E * 4));
    PF_CK(cudaMalloc((void **)&s.sr, T * E * 4));
    PF_CK(cudaMalloc((void **)&s.act, T * 4 * E * 4));
    PF_CK(cudaFuncSetAttribute(k_gemm_i8<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    PF_CK(cudaFuncSetAttribute(k_gemm_i8<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    PF_CK(cudaFuncSetAttribute(k_gemm_i8<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    PF_CK(cudaFuncSetAttribute(k_gemm_i8<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    s.ready = true;
    return 0;
}

inline int pf_make_map(PrefillState &s, CUtensorMap *m, const void *base, size_t rows, size_t K, uint32_t box_rows) {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)K};
    cuuint32_t box[2] = {(cuuint32_t)kPfBK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = s.encode(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        prefill_err_slot() = "batched prefill: cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")";
        return 3;
    }
    return 0;
}

// C = W[M][K] x limbs(vector at b_row0)^T ; C is zeroed here.
inline int pf_gemm(PrefillState &s, cudaStream_t st, const int8_t *W, int M, int K, const uint8_t *limbs, size_t limb_rows, int b_row0, int Tp, int *C) {
    GemmArgs g;
    int rc;
    if ((rc = pf_make_map(s, &g.map_a, W, (size_t)M, (size_t)K, kPfBM))) return rc;
    if ((rc = pf_make_map(s, &g.map_b, limbs, limb_rows, (size_t)K, (uint32_t)Tp))) return rc;
    g.M = M;
    g.K = K;
    g.Tp = Tp;
    g.b_row0 = b_row0;
    const int mt = (M + kPfBM - 1) / kPfBM;
    int ks = 1;
    while (mt * ks < 132 && ks < 8 && (K / (ks * 2)) % kPfBK == 0 && K / (ks * 2) >= 4 * kPfBK) ks *= 2;
    g.ksplit = ks;
    g.C = C;
    PF_CK(cudaMemsetAsync(C, 0, (size_t)M * 3 * Tp * 4, st));
    const size_t smem = (size_t)kPfStages * (kPfBM * kPfBK + 3 * (size_t)Tp * kPfBK) + 1024 + 128;
    static_assert(kPfMaxTokens == 4 * kPfTokenAlign, "one instantiation per block count");
    switch (Tp / kPfTokenAlign) {
    case 1: k_gemm_i8<1><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); break;
    case 2: k_gemm_i8<2><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); break;
    case 3: k_gemm_i8<3><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); break;
    default: k_gemm_i8<4><<<dim3(mt, ks), kPfThreads, smem, st>>>(g); break;
    }
    PF_CK(cudaGetLastError());
    s.launches += 1;
    return 0;
}

inline int pf_padded(int n) { return (n + kPfTokenAlign - 1) / kPfTokenAlign * kPfTokenAlign; }

// One pass of T <= 128 tokens on a single GPU, laid out by s.pass. H > 0: the head runs on the H rows of the row
// map and writes logits rows pass->out_row0 .. + H - 1 of `logits` ([rows][V], device).
// The deltas of one adaptation point: nv matrices of layer l whose inputs are at f (vector stride f_vstride, row K),
// into s.ad_d (vector stride T * E, row M[v]).
inline void pf_adapt(PrefillState &s, const Params &p, cudaStream_t st, int T, int l, int nv, const int (&mat)[3], int K,
                     const int (&M)[3], const float *f, size_t f_vstride) {
    AdArgs a{};
    a.table = s.ad_table;
    a.desc = s.pass->desc;
    a.T = T;
    a.l = l;
    a.nv = nv;
    a.K = K;
    int maxM = 0;
    for (int v = 0; v < 3; ++v) {
        a.mat[v] = mat[v];
        a.M[v] = M[v];
        maxM = std::max(maxM, M[v]);
    }
    a.f = f;
    a.f_vstride = f_vstride;
    a.h = s.ad_h;
    a.delta = s.ad_d;
    a.d_vstride = (size_t)T * p.E;
    k_ad_shrink<<<dim3(kAdMaxRank, nv, (T + kAdShrinkTokens - 1) / kAdShrinkTokens), kAdThreads, 0, st>>>(a);
    k_ad_expand<<<dim3((maxM + kAdThreads - 1) / kAdThreads, nv, (T + kAdExpandTokens - 1) / kAdExpandTokens), kAdThreads, 0, st>>>(a);
}

inline int prefill_chunk_body(PrefillState &s, const Params &p, cudaStream_t st, int T, int H, float *logits, bool ad) {
    const int E = p.E, L = p.L, Tp = pf_padded(T);
    const size_t LE = (size_t)L * E;
    double *saa = reinterpret_cast<double *>(p.xch[p.rank] + p.off_saa), *sbb = reinterpret_cast<double *>(p.xch[p.rank] + p.off_sbb);
    const unsigned gT = (unsigned)T;
    auto blocks = [](size_t n) { return (unsigned)((n + 255) / 256); };
    int rc;
    PF_CK(cudaMemsetAsync(s.limbs, 0, (size_t)9 * Tp * 4 * E, st)); // padded token rows stay zero
    k_pf_embed<<<gT, 256, 0, st>>>(p.emb, p.ln, s.pass->tokens, E, s.x);
    int *Ca = s.C, *Cb = s.C + (size_t)E * 3 * Tp, *Cc = s.C + (size_t)2 * E * 3 * Tp; // three accumulator sets; the big ones reuse [0]
    for (int l = 0; l < L; ++l) {
        const size_t lo = (size_t)l * E;
        // ---- att: LN1, token shift, K/V/R, WKV, out-proj ------------------------------------------------------
        k_pf_ln<<<gT, 256, 0, st>>>(s.x, p.ln + (size_t)(4 * l + 2) * E, p.ln + (size_t)(4 * l + 3) * E, E, s.iota, s.ln);
        MixArgs m{};
        m.ln = s.ln;
        m.state = p.sxy + lo;
        m.slot_stride = LE;
        m.desc = s.pass->desc;
        m.mix[0] = p.mixk + lo; m.mix[1] = p.mixv + lo; m.mix[2] = p.mixr + lo;
        m.r[0] = p.rk + lo; m.r[1] = p.rv + lo; m.r[2] = p.rr + lo;
        m.oc[0] = p.ock + lo; m.oc[1] = p.ocv + lo; m.oc[2] = p.ocr + lo;
        m.nv = 3; m.E = E; m.Tp = Tp;
        m.limbs = s.limbs; m.scale = s.scale; m.offs = s.offs;
        m.fout = ad ? s.ad_f : nullptr;
        k_pf_mix_quant<<<gT, 256, 0, st>>>(m);
        k_pf_store_state<<<gT, 256, 0, st>>>(s.ln, E, s.pass, LE, p.sxy + lo, kPoolXY, lo);
        const size_t mo = (size_t)l * E * E;
        if ((rc = pf_gemm(s, st, p.wk + mo, E, E, s.limbs, (size_t)9 * Tp, 0 * Tp, Tp, Ca))) return rc;
        if ((rc = pf_gemm(s, st, p.wv + mo, E, E, s.limbs, (size_t)9 * Tp, 3 * Tp, Tp, Cb))) return rc;
        if ((rc = pf_gemm(s, st, p.wr + mo, E, E, s.limbs, (size_t)9 * Tp, 6 * Tp, Tp, Cc))) return rc;
        WkvArgs w{};
        w.Ck = Ca; w.Cv = Cb; w.Cr = Cc;
        w.scale = s.scale; w.offs = s.offs;
        w.decay = p.decay + lo; w.bonus = p.bonus + lo; w.expdecay = p.expdecay + lo;
        w.ro = p.ro + lo;
        w.aa = saa + lo; w.bb = sbb + lo;
        w.slot_stride = LE;
        w.desc = s.pass->desc;
        w.E = E; w.T = T; w.Tp = Tp;
        w.rw = s.rw; w.xs = s.xs;
        w.pass = s.pass; w.lo = lo;
        const size_t TE = (size_t)T * E;
        if (ad) {
            pf_adapt(s, p, st, T, l, 3, {kAdAttK, kAdAttV, kAdAttR}, E, {E, E, E}, s.ad_f, (size_t)Tp * E);
            w.dk = s.ad_d; w.dv = s.ad_d + TE; w.dr = s.ad_d + 2 * TE;
        }
        k_pf_wkv<<<blocks(E), 256, 0, st>>>(w);
        k_pf_quant_rows<<<gT, 256, 0, st>>>(s.xs, s.rw, p.oco + lo, E, Tp, s.limbs, s.scale, s.offs);
        if ((rc = pf_gemm(s, st, p.wo + mo, E, E, s.limbs, (size_t)3 * Tp, 0, Tp, Ca))) return rc;
        if (ad) pf_adapt(s, p, st, T, l, 1, {kAdAttO, 0, 0}, E, {E, 0, 0}, s.rw, 0);
        k_pf_residual<<<blocks((size_t)T * E), 256, 0, st>>>(Ca, s.scale, s.offs, nullptr, E, T, Tp, s.x, ad ? s.ad_d : nullptr);
        // ---- ffn: LN2, token shift, R/K, activations, V -------------------------------------------------------
        k_pf_ln<<<gT, 256, 0, st>>>(s.x, p.ln + (size_t)(4 * (l + 1)) * E, p.ln + (size_t)(4 * (l + 1) + 1) * E, E, s.iota, s.ln);
        MixArgs f{};
        f.ln = s.ln;
        f.state = p.sdd + lo;
        f.slot_stride = LE;
        f.desc = s.pass->desc;
        f.mix[0] = p.fmixr + lo; f.mix[1] = p.fmixk + lo;
        f.r[0] = p.rfr + lo; f.r[1] = p.rfk + lo;
        f.oc[0] = p.ocfr + lo; f.oc[1] = p.ocfk + lo;
        f.nv = 2; f.E = E; f.Tp = Tp;
        f.limbs = s.limbs; f.scale = s.scale; f.offs = s.offs;
        f.fout = ad ? s.ad_f : nullptr;
        k_pf_mix_quant<<<gT, 256, 0, st>>>(f);
        k_pf_store_state<<<gT, 256, 0, st>>>(s.ln, E, s.pass, LE, p.sdd + lo, kPoolDD, lo);
        int *Ck4 = s.C + (size_t)E * 3 * Tp; // [4E][3Tp] behind the ffn-R accumulators
        if ((rc = pf_gemm(s, st, p.wfr + mo, E, E, s.limbs, (size_t)6 * Tp, 0 * Tp, Tp, Ca))) return rc;
        if ((rc = pf_gemm(s, st, p.wfk + 4 * mo, 4 * E, E, s.limbs, (size_t)6 * Tp, 3 * Tp, Tp, Ck4))) return rc;
        if (ad) pf_adapt(s, p, st, T, l, 2, {kAdFfnR, kAdFfnK, 0}, E, {E, 4 * E, 0}, s.ad_f, (size_t)Tp * E);
        k_pf_ffn_act<<<blocks((size_t)T * 5 * E), 256, 0, st>>>(Ca, Ck4, s.scale, s.offs, p.rfv + (size_t)l * 4 * E, E, T, Tp, s.sr, s.act, s.xs,
                                                                ad ? s.ad_d : nullptr, ad ? s.ad_d + TE : nullptr);
        k_pf_quant_rows<<<gT, 256, 0, st>>>(s.xs, s.act, p.ocfv + (size_t)l * 4 * E, 4 * E, Tp, s.limbs, s.scale, s.offs);
        if ((rc = pf_gemm(s, st, p.wfv + 4 * mo, E, 4 * E, s.limbs, (size_t)3 * Tp, 0, Tp, Ca))) return rc;
        if (ad) pf_adapt(s, p, st, T, l, 1, {kAdFfnV, 0, 0}, 4 * E, {E, 0, 0}, s.act, 0);
        k_pf_residual<<<blocks((size_t)T * E), 256, 0, st>>>(Ca, s.scale, s.offs, s.sr, E, T, Tp, s.x, ad ? s.ad_d : nullptr);
        s.launches += ad ? 18 : 10;
    }
    // ---- head: the rows of the row map only -----------------------------------------------------------------------
    if (H > 0) {
        const int Hp = pf_padded(H);
        const unsigned gH = (unsigned)H;
        k_pf_ln<<<gH, 256, 0, st>>>(s.x, p.ln + (size_t)(4 * L + 2) * E, p.ln + (size_t)(4 * L + 3) * E, E, s.pass->rows, s.ln);
        MixArgs h{}; // scale + quantise without a token shift: a mix vector of ones selects the current token only
        h.ln = s.ln;
        h.state = s.ln; // read, but multiplied by 1 - 1 = 0
        h.slot_stride = 0;
        h.desc = s.head_desc;
        h.mix[0] = p.ones;
        h.r[0] = p.rhead;
        h.oc[0] = p.ochead;
        h.nv = 1; h.E = E; h.Tp = Hp;
        h.limbs = s.limbs; h.scale = s.scale; h.offs = s.offs;
        k_pf_mix_quant<<<gH, 256, 0, st>>>(h);
        if ((rc = pf_gemm(s, st, p.whead, p.Vr, E, s.limbs, (size_t)3 * Hp, 0, Hp, s.C))) return rc;
        k_pf_logits<<<blocks((size_t)H * kVocab), 256, 0, st>>>(s.C, s.scale, s.offs, kVocab, H, Hp, &s.pass->out_row0, logits);
        s.launches += 4;
    }
    PF_CK(cudaGetLastError());
    return 0;
}

// One pass of the layout already in s.pass: replay (or record) the graph of its shape.
inline int prefill_run(PrefillState &s, const Params &p, cudaStream_t st, int T, int H, float *logits) {
    int rc;
    const bool ad = s.adapt;
    if (ad && !s.ad_f) {
        if (!s.ad_table) {
            prefill_err_slot() = "batched prefill: a pass with adapters but no adapter table";
            return 3;
        }
        const size_t E = (size_t)p.E, Tm = kPfMaxTokens;
        PF_CK(cudaMalloc((void **)&s.ad_f, 3 * Tm * E * 4));
        PF_CK(cudaMalloc((void **)&s.ad_h, 3 * Tm * kAdMaxRank * 8));
        PF_CK(cudaMalloc((void **)&s.ad_d, 5 * Tm * E * 8));
    }
    PrefillState::Graph *g = nullptr;
    for (auto &e : s.graphs)
        if (e.T == T && e.H == H && e.adapt == ad) g = &e;
    if (!g && s.use_graph) {
        // record the pass once (nothing runs during the capture), then replay it
        const unsigned long long before = s.launches;
        PF_CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        rc = prefill_chunk_body(s, p, st, T, H, logits, ad);
        cudaGraph_t graph = nullptr;
        const cudaError_t ee = cudaStreamEndCapture(st, &graph);
        const unsigned long long n = s.launches - before;
        s.launches = before;
        if (rc) {
            if (graph) cudaGraphDestroy(graph);
            return rc;
        }
        if (ee != cudaSuccess) return pf_fail("cudaStreamEndCapture", ee);
        cudaGraphExec_t exec = nullptr;
        const cudaError_t ei = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ei != cudaSuccess) return pf_fail("cudaGraphInstantiate", ei);
        if (s.graphs.size() >= 8) {
            cudaGraphExecDestroy(s.graphs.front().exec);
            s.graphs.erase(s.graphs.begin());
        }
        s.graphs.push_back(PrefillState::Graph{T, H, ad, exec, n});
        s.records += 1;
        g = &s.graphs.back();
    }
    if (g) {
        PF_CK(cudaGraphLaunch(g->exec, st));
        s.launches += g->launches;
    } else if ((rc = prefill_chunk_body(s, p, st, T, H, logits, ad))) {
        return rc;
    }
    return 0;
}

// The passes of a ragged forward: `tokens` are stream-major, stream i owns lens[i] consecutive tokens and advances
// state slot slots[i]. The list is cut into passes of at most 128 tokens (pass i starts at token 128 i); a stream that
// crosses a cut is "last" in one pass and "first" in the next. head = 0: state only. head = 1: logits of every token,
// row t of the logits. head = 2: logits of each stream's final token, row i for stream i (only the pass holding that
// token runs the head for it). `need` (head 1 only, may be NULL): a pass none of whose tokens has need[t] set runs no
// head, so its logits rows are not written. `stream_head` (head 2 only, may be NULL = every stream): only a stream with
// stream_head[i] set gets a head row, and its logits row counts the headed streams before it (the batcher's decode rows,
// followed by prefill segments without logits). Fills each pass's descriptor (zero past its last token) and head row count.
inline void pass_layout(const unsigned long long *tokens, int n, const unsigned long long *slots, const unsigned long long *lens,
                        int head, const unsigned char *need, std::vector<PassDesc> &passes, std::vector<int> &heads,
                        const unsigned char *stream_head = nullptr) {
    passes.assign((size_t)(n + kPfMaxTokens - 1) / kPfMaxTokens, PassDesc{});
    heads.assign(passes.size(), 0);
    int stream = 0, pos = 0;  // current stream, index of the next token inside it
    int ended = 0;            // streams whose final token lies in an earlier pass
    for (size_t i = 0; i < passes.size(); ++i) {
        PassDesc &h = passes[i];
        const int t0 = (int)i * kPfMaxTokens, T = std::min(kPfMaxTokens, n - t0);
        int H = 0;
        bool needed = need == nullptr;
        h.out_row0 = head == 1 ? t0 : ended;
        for (int t = 0; t < T; ++t) {
            if (need && need[t0 + t]) needed = true;
            while (pos == (int)lens[stream]) {
                ++stream;
                pos = 0;
            }
            const bool fin = pos + 1 == (int)lens[stream];
            const bool headed = fin && (!stream_head || stream_head[stream]);
            h.tokens[t] = tokens[t0 + t];
            h.desc[t] = (uint32_t)slots[stream] | (pos == 0 || t == 0 ? kDescFirst : 0u) | (fin || t == T - 1 ? kDescLast : 0u);
            if (head == 1 || (head == 2 && headed)) h.rows[H++] = t;
            if (headed) ++ended;
            ++pos;
        }
        heads[i] = needed ? H : 0;
    }
}

// The passes of a layout of n tokens (pass_layout's, possibly with snapshots added): per pass, upload it, then run it.
inline int prefill_passes(PrefillState &s, const Params &p, cudaStream_t st, const std::vector<PassDesc> &passes,
                          const std::vector<int> &heads, int n, float *logits) {
    int rc = prefill_init(s, p);
    if (rc) return rc;
    for (size_t i = 0; i < passes.size(); ++i) {
        PF_CK(cudaMemcpyAsync(s.pass, &passes[i], sizeof(PassDesc), cudaMemcpyHostToDevice, st));
        if ((rc = prefill_run(s, p, st, std::min(kPfMaxTokens, n - (int)i * kPfMaxTokens), heads[i], logits))) return rc;
    }
    return 0;
}

// A ragged forward (the layout and `head` of pass_layout): per pass, upload its layout, then run it. `logits` is a
// device buffer of at least n (head 1) / one per stream (head 2) rows.
inline int prefill_forward(PrefillState &s, const Params &p, cudaStream_t st, const unsigned long long *tokens, int n,
                           const unsigned long long *slots, const unsigned long long *lens, int head, float *logits,
                           const unsigned char *need = nullptr) {
    std::vector<PassDesc> passes;
    std::vector<int> heads;
    pass_layout(tokens, n, slots, lens, head, need, passes, heads);
    return prefill_passes(s, p, st, passes, heads, n, logits);
}

} // namespace rk
