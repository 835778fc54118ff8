// latbench.cu — ground-truth latencies of the building blocks of the token kernel's phase boundaries on the
// actual GPU, one warp, with the token kernel's shared-memory carve-out (227 KB -> almost no L1).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o latbench latbench.cu && ./latbench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ double wsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// a large body of straight-line dependent code (cold I-cache the first time)
template <int N> __device__ __noinline__ double cold_code(double x, double y) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
        x = fma(x, 1.0000001, y);
        y = fma(y, 0.9999999, x * 1e-9);
    }
    return x + y;
}

__global__ void k_lat(unsigned long long *buf, long long *out, double *dout, int iters) {
    extern __shared__ unsigned char smem[];
    const int lane = threadIdx.x & 31;
    if (threadIdx.x >= 32) return;
    long long t0, t1;
    double acc = (double)lane;
    // 1. %globaltimer read
    unsigned long long g = 0;
    t0 = clock64();
    for (int i = 0; i < 16; ++i) g ^= gtimer();
    t1 = clock64();
    if (lane == 0) out[0] = (t1 - t0) / 16;
    // 2. double shuffle-reduce (5 steps)
    t0 = clock64();
    for (int i = 0; i < 16; ++i) acc = wsum(acc) * 0.03125;
    t1 = clock64();
    if (lane == 0) out[1] = (t1 - t0) / 16;
    // 3. L2 round trip: dependent relaxed loads (pointer chase over 64 slots, 128-byte stride)
    unsigned long long idx = lane;
    t0 = clock64();
    for (int i = 0; i < 16; ++i) idx = ld_relaxed(buf + (idx & 63) * 16);
    t1 = clock64();
    if (lane == 0) out[2] = (t1 - t0) / 16;
    // 4. store -> load of the same address (relaxed, gpu scope)
    t0 = clock64();
    for (int i = 0; i < 16; ++i) {
        st_relaxed(buf + 2048 + lane, idx + i);
        idx += ld_relaxed(buf + 2048 + lane) & 1;
    }
    t1 = clock64();
    if (lane == 0) out[3] = (t1 - t0) / 16;
    // 5. local memory round trip (dynamic index defeats register promotion)
    {
        volatile double loc[32];
        for (int i = 0; i < 32; ++i) loc[i] = acc + i;
        int j = (int)(idx & 31);
        t0 = clock64();
        for (int i = 0; i < 16; ++i) j = ((int)loc[j] + i) & 31;
        t1 = clock64();
        if (lane == 0) out[4] = (t1 - t0) / 16;
        acc += j;
    }
    // 6. cold vs warm straight-line code: 2048 dependent DFMA pairs (~64 KB of SASS)
    t0 = clock64();
    acc = cold_code<2048>(acc, 1.0);
    t1 = clock64();
    if (lane == 0) out[5] = t1 - t0;
    t0 = clock64();
    acc = cold_code<2048>(acc, 1.0);
    t1 = clock64();
    if (lane == 0) out[6] = t1 - t0;
    // 7. a small cold function vs warm (96 DFMA pairs ~ 3 KB)
    t0 = clock64();
    acc = cold_code<96>(acc, 1.0);
    t1 = clock64();
    if (lane == 0) out[7] = t1 - t0;
    t0 = clock64();
    acc = cold_code<96>(acc, 1.0);
    t1 = clock64();
    if (lane == 0) out[8] = t1 - t0;
    // 8. double division, exp
    t0 = clock64();
    for (int i = 0; i < 16; ++i) acc = 1.0 / (acc + 1.5);
    t1 = clock64();
    if (lane == 0) out[9] = (t1 - t0) / 16;
    t0 = clock64();
    for (int i = 0; i < 16; ++i) acc = exp(acc * 0.5);
    t1 = clock64();
    if (lane == 0) out[10] = (t1 - t0) / 16;
    // 9. globaltimer resolution: ns between two distinct values
    unsigned long long a = gtimer(), b2;
    do { b2 = gtimer(); } while (b2 == a);
    if (lane == 0) out[11] = (long long)(b2 - a);
    dout[lane] = acc + (double)g + (double)idx + smem[lane];
}

int main() {
    unsigned long long *buf;
    long long *out, h[16] = {0};
    double *dout;
    cudaMalloc(&buf, 1 << 20);
    cudaMalloc(&out, 16 * 8);
    cudaMalloc(&dout, 32 * 8);
    unsigned long long hb[64 * 16];
    for (int i = 0; i < 64 * 16; ++i) hb[i] = (unsigned long long)((i / 16) * 7 + 3);
    cudaMemcpy(buf, hb, sizeof(hb), cudaMemcpyHostToDevice);
    cudaFuncSetAttribute(k_lat, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
    for (int rep = 0; rep < 2; ++rep) {
        k_lat<<<1, 64, 232448>>>(buf, out, dout, 16);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
            printf("error: %s\n", cudaGetErrorString(e));
            return 1;
        }
        cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
        printf("run %d (SM cycles): globaltimer read %lld | f64 warp-sum %lld | L2 dependent load %lld | st+ld same addr %lld | "
               "local mem round trip %lld | 64KB code cold %lld warm %lld | 3KB code cold %lld warm %lld | ddiv %lld | exp %lld | "
               "globaltimer tick %lld ns\n",
               rep, h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7], h[8], h[9], h[10], h[11]);
    }
    return 0;
}

// ---- part 2: the same f64 warp-sum inside the token kernel's environment, one ingredient at a time ---------------
// flags: 1 = 7 more warps blocked on a named barrier; 2 = a lane of warp 8 spinning on mbarrier.try_wait;
//        4 = setmaxnreg (consumers 232 / producer 40); 8 = bulk copies global->shared in flight (ring of 4 x 32 KB)
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__global__ void __launch_bounds__(384, 1) k_env(const unsigned char *src, long long *out, double *dout, int flags) {
    extern __shared__ __align__(128) unsigned char smem2[];
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem2 + 200000);
    volatile int *stop = reinterpret_cast<volatile int *>(smem2 + 200064);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(1));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar + 1)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        *stop = 0;
    }
    __syncthreads();
    if (warp >= 8) {
        if (flags & 4) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            if (flags & 8) { // stream 32 KB tiles into a 4-stage ring, no consumer: wait for each to land, go on
                uint32_t parity = 0;
                size_t off = 0;
                while (!*stop) {
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar + 1)), "r"(32768) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(smem2)),
                                 "l"(src + off), "r"(32768), "r"(smem_addr(bar + 1))
                                 : "memory");
                    uint32_t ok = 0;
                    while (!ok) {
                        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_addr(bar + 1)), "r"(parity) : "memory");
                    }
                    parity ^= 1;
                    off = (off + 32768 * 132) & ((1ull << 30) - 1);
                }
            } else if (flags & 2) { // spin on a barrier nobody completes
                uint32_t ok = 0;
                while (!ok && !*stop) {
                    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_addr(bar)), "r"(0) : "memory");
                }
            }
        }
        return;
    }
    if (flags & 4) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    if (warp > 0) {
        if (flags & 1) asm volatile("bar.sync 1, 256;" ::: "memory");
        return;
    }
    // warp 0: let the others settle, then time
    long long t0 = clock64();
    while (clock64() - t0 < 20000) {}
    double acc = (double)lane;
    t0 = clock64();
    for (int i = 0; i < 16; ++i) acc = wsum(acc) * 0.03125;
    long long t1 = clock64();
    // diverge (lane 0 does extra work), then sum again without and with __syncwarp
    if (lane == 0) acc += (double)(clock64() & 1);
    long long t2 = clock64();
    for (int i = 0; i < 16; ++i) acc = wsum(acc) * 0.03125;
    long long t3 = clock64();
    if (lane == 0) {
        out[0] = (t1 - t0) / 16;
        out[1] = (t3 - t2) / 16;
    }
    dout[lane] = acc;
    *stop = 1;
    if (flags & 1) asm volatile("bar.sync 1, 256;" ::: "memory");
}

struct Part2 {
    Part2() {
        unsigned char *src;
        long long *out, h[2];
        double *dout;
        cudaMalloc(&src, (1ull << 30) + (1 << 20));
        cudaMalloc(&out, 16);
        cudaMalloc(&dout, 256);
        cudaFuncSetAttribute(k_env, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
        for (int flags : {0, 1, 2, 3, 4, 7, 8, 9, 15}) {
            k_env<<<132, 384, 232448>>>(src, out, dout, flags);
            cudaError_t e = cudaDeviceSynchronize();
            if (e != cudaSuccess) {
                printf("flags %d error: %s\n", flags, cudaGetErrorString(e));
                break;
            }
            cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
            printf("env flags %2d: f64 warp-sum %lld cycles, after a lane-0 branch %lld cycles\n", flags, h[0], h[1]);
        }
    }
} part2_runs_before_main_returns;

// ---- part 3: the all-gather itself: every CTA reads the same `bytes` of exchanged data with `per` 16-byte strong loads
// per thread (256 threads), all CTAs at the same moment; with and without bulk copies streaming in the background.
__global__ void __launch_bounds__(384, 1) k_allgather(const unsigned char *src, const uint4 *vec, int groups, long long *out, int stream, int rotate) {
    extern __shared__ __align__(128) unsigned char smem3[];
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem3 + 200000);
    volatile int *stop = reinterpret_cast<volatile int *>(smem3 + 200064);
    const int warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        *stop = 0;
    }
    __syncthreads();
    if (warp >= 8) {
        if (warp == 8 && (threadIdx.x & 31) == 0 && stream) {
            uint32_t parity = 0;
            size_t off = (size_t)blockIdx.x * 32768;
            while (!*stop) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(32768 * stream) : "memory");
                for (int k = 0; k < stream; ++k)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(smem3 + 32768 * k)),
                                 "l"(src + off + (size_t)k * 32768 * 132), "r"(32768), "r"(smem_addr(bar))
                                 : "memory");
                uint32_t ok = 0;
                while (!ok) {
                    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
                }
                parity ^= 1;
                off = (off + (size_t)32768 * 132 * stream) & ((1ull << 30) - 1);
            }
        }
        return;
    }
    const int t = threadIdx.x;
    long long t0 = clock64();
    while (clock64() - t0 < 40000) {} // let the stream reach its steady state
    long long best = 1ll << 60, sum = 0;
    uint32_t acc = 0;
    for (int rep = 0; rep < 8; ++rep) {
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int rot = rotate ? (int)(((unsigned)groups * blockIdx.x) / gridDim.x) : 0;
        const long long a = clock64();
        uint4 f[20];
#pragma unroll
        for (int i = 0; i < 20; ++i) {
            int g = t + 256 * i + rot;
            if (g >= groups) g -= groups;
            if (t + 256 * i < groups) asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(f[i].x), "=r"(f[i].y), "=r"(f[i].z), "=r"(f[i].w) : "l"(vec + g) : "memory");
            else f[i] = make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int i = 0; i < 20; ++i) acc += f[i].x ^ f[i].w;
        asm volatile("" ::"r"(acc) : "memory");
        const long long b = clock64();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (b - a < best) best = b - a;
        sum += b - a;
        long long w0 = clock64();
        while (clock64() - w0 < 6000) {} // the CTAs drift apart and meet again like the token kernel's phases
    }
    if (t == 0) {
        out[2 * blockIdx.x] = sum / 8;
        out[2 * blockIdx.x + 1] = best + (acc & 1);
    }
    *stop = 1;
}

struct Part3 {
    Part3() {
        unsigned char *src;
        uint4 *vec;
        long long *out, h[2 * 132];
        cudaMalloc(&src, (1ull << 30) + (64 << 20));
        cudaMalloc(&vec, 1 << 20);
        cudaMalloc(&out, sizeof(h));
        cudaMemset(vec, 0, 1 << 20);
        cudaFuncSetAttribute(k_allgather, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
        for (int groups : {1024, 3072, 4096}) {
            for (int stream : {0, 1, 3}) {
                for (int rotate : {0, 1}) {
                    k_allgather<<<132, 384, 232448>>>(src, vec, groups, out, stream, rotate);
                    cudaError_t e = cudaDeviceSynchronize();
                    if (e != cudaSuccess) {
                        printf("allgather error: %s\n", cudaGetErrorString(e));
                        return;
                    }
                    cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
                    long long mean = 0, mx = 0;
                    for (int b = 0; b < 132; ++b) {
                        mean += h[2 * b];
                        if (h[2 * b] > mx) mx = h[2 * b];
                    }
                    printf("all-gather of %5d x 16 B by 132 CTAs, %d tiles streaming per SM, rotate %d: mean %lld cycles, slowest CTA %lld\n", groups,
                           stream, rotate, mean / 132, mx);
                }
            }
        }
    }
} part3_runs_before_main_returns;
