// stream_probe.cu — how fast the token kernel's weight stream can read HBM, and what it does to the latency of
// the exchange loads, as a function of the bytes each SM keeps in flight and of the bulk-copy size.
//
// Geometry of the token kernel (token_kernel.cuh, produce_token): one CTA per SM, one producer lane issuing 1-D
// bulk copies (L2::evict_first) into a ring of 5 x 32 KB stages, each CTA streaming its own contiguous rows.
// Here the eight consumer warps only release the stages, and a ninth warp times batches of 16-byte strong loads of
// L2-resident words - the loads gather() issues - while the stream runs.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o stream_probe stream_probe.cu && ./stream_probe [GiB]
// One line per setting: "stream budget=<B> sub=<B> gbs=<read GB/s> lat_ns_mean=.. lat_ns_p50=.. lat_ns_p90=.." (latency of
// one batch of 12 x 16-byte loads per lane, SM cycles at the device's rated clock)
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x)                                                                                                  \
    do {                                                                                                       \
        cudaError_t e_ = (x);                                                                                  \
        if (e_ != cudaSuccess) {                                                                               \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));                 \
            exit(1);                                                                                           \
        }                                                                                                      \
    } while (0)

constexpr int kStages = 5, kTile = 32768, kConsumerWarps = 8, kThreads = (kConsumerWarps + 2) * 32;
constexpr int kLatSamples = 64;   // timed batches per CTA
constexpr int kLatLoads = 12;     // 16-byte loads per lane and batch (3 x 4096 words over 256 threads, as gather())
constexpr int kLatWords = 32 * kLatLoads;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ bool test_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}

struct Args {
    const unsigned char *src;  // [grid][per_cta] bytes
    unsigned long long per_cta;
    const uint4 *words;        // L2-resident exchange words
    unsigned long long *lat;   // [grid][kLatSamples] SM cycles per batch (0: the stream ended first)
    unsigned int budget, sub;  // bytes in flight per SM (0: no stream), bulk-copy size
};

// The ring (5 x 32 KB) is cut into slots of `sub` bytes, each with its own full / empty barrier, so that the bytes in
// flight are known copy by copy: at most `budget` of them, and always one copy when none is.
constexpr int kMaxSlots = kStages * kTile / 4096;
__global__ void __launch_bounds__(kThreads, 1) k_stream(const Args a) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + kStages * kTile), *empty = full + kMaxSlots;
    volatile int *done = reinterpret_cast<volatile int *>(empty + kMaxSlots);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t nslots = kStages * kTile / a.sub;
    if (threadIdx.x == 0) {
        for (uint32_t i = 0; i < nslots; ++i) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(full + i)), "r"(1));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(empty + i)), "r"(kConsumerWarps));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        *done = 0;
    }
    __syncthreads();
    const unsigned long long ncopies = a.budget ? a.per_cta / a.sub : 0;
    const unsigned char *src = a.src + (size_t)blockIdx.x * a.per_cta;
    if (warp == kConsumerWarps) { // producer lane
        if (lane != 0) return;
        uint64_t pol;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        const uint32_t ring = smem_u32(smem), full0 = smem_u32(full), empty0 = smem_u32(empty);
        uint32_t st = 0, ph = 0, wst = 0, wph = 0;
        unsigned long long landed = 0;
        for (unsigned long long c = 0; c < ncopies; ++c) {
            for (;;) {
                while (landed < c && test_wait(full0 + 8 * wst, wph)) {
                    if (++wst == nslots) wst = 0, wph ^= 1;
                    ++landed;
                }
                const unsigned long long inflight = (c - landed) * a.sub;
                if (test_wait(empty0 + 8 * st, ph ^ 1) && (inflight == 0 || inflight + a.sub <= a.budget)) break;
                __nanosleep(40);
            }
            const uint32_t fb = full0 + 8 * st;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(fb), "r"(a.sub) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                         ::"r"(ring + st * a.sub), "l"(src + c * a.sub), "r"(a.sub), "r"(fb), "l"(pol) : "memory");
            if (++st == nslots) st = 0, ph ^= 1;
        }
        return;
    }
    if (warp == kConsumerWarps + 1) { // exchange-load timer
        const uint4 *w = a.words + (size_t)(blockIdx.x % 8) * kLatWords;
        uint32_t acc = 0;
        for (int s = 0; s < kLatSamples; ++s) {
            const long long w0 = clock64();
            while (clock64() - w0 < 4000) {} // the token kernel's exchanges are microseconds apart
            if (a.budget && *done) break;
            __syncwarp();
            const long long t0 = clock64();
            uint4 f[kLatLoads];
#pragma unroll
            for (int i = 0; i < kLatLoads; ++i)
                asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                             : "=r"(f[i].x), "=r"(f[i].y), "=r"(f[i].z), "=r"(f[i].w) : "l"(w + lane + 32 * i) : "memory");
#pragma unroll
            for (int i = 0; i < kLatLoads; ++i) acc += f[i].x ^ f[i].w;
            acc = __reduce_add_sync(0xffffffffu, acc); // every lane's loads have returned
            const long long t1 = clock64();
            if (lane == 0) a.lat[(size_t)blockIdx.x * kLatSamples + s] = (unsigned long long)(t1 - t0) + (acc == 0x7fffffffu);
        }
        return;
    }
    // consumer warps: release every slot as soon as it lands
    uint32_t st = 0, ph = 0;
    for (unsigned long long c = 0; c < ncopies; ++c) {
        while (!test_wait(smem_u32(full + st), ph)) {}
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(empty + st)) : "memory");
        if (++st == nslots) st = 0, ph ^= 1;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumerWarps * 32) : "memory");
    if (threadIdx.x == 0) *done = 1;
}

__global__ void k_ldg(const uint4 *src, unsigned long long n, uint32_t *sink) {
    uint32_t acc = 0;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        uint4 v;
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

static double median(std::vector<double> v) {
    std::sort(v.begin(), v.end());
    return v.empty() ? 0.0 : v[v.size() / 2];
}

int main(int argc, char **argv) {
    const double gib = argc > 1 ? atof(argv[1]) : 4.0;
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    const int grid = sms;
    int clock_khz = 0;
    CK(cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, dev));
    const double ghz = clock_khz / 1e6;
    const unsigned long long per_cta = ((unsigned long long)(gib * (1ull << 30)) / grid) / kTile * kTile;
    const unsigned long long total = per_cta * grid;
    printf("device %s, %d SMs, %.0f MHz; stream of %.2f GiB: %d CTAs x %llu bytes, ring %d x %d KB\n", prop.name, sms, clock_khz / 1e3,
           total / double(1ull << 30), grid, per_cta, kStages, kTile / 1024);
    unsigned char *src, *dst;
    uint4 *words;
    unsigned long long *lat;
    uint32_t *sink;
    CK(cudaMalloc(&src, total));
    CK(cudaMalloc(&dst, total / 2));
    CK(cudaMemset(src, 1, total));
    CK(cudaMalloc(&words, 8 * kLatWords * sizeof(uint4)));
    CK(cudaMemset(words, 0, 8 * kLatWords * sizeof(uint4)));
    CK(cudaMalloc(&lat, (size_t)grid * kLatSamples * 8));
    CK(cudaMalloc(&sink, 4));
    CK(cudaFuncSetAttribute(k_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448)); // the token kernel's carve-out
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    std::vector<unsigned long long> hl((size_t)grid * kLatSamples);

    auto run = [&](unsigned int budget, unsigned int sub) {
        Args a{src, per_cta, words, lat, budget, sub};
        std::vector<double> rates, lats;
        for (int rep = 0; rep < 3; ++rep) {
            CK(cudaMemset(lat, 0, (size_t)grid * kLatSamples * 8));
            CK(cudaEventRecord(e0));
            k_stream<<<grid, kThreads, 232448>>>(a);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaGetLastError());
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (budget) rates.push_back(total / (ms * 1e6));
            CK(cudaMemcpy(hl.data(), lat, hl.size() * 8, cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < hl.size(); ++i)
                if (rep > 0 && hl[i]) lats.push_back((double)hl[i] / ghz); // rep 0 warms up
        }
        std::vector<double> s = lats;
        std::sort(s.begin(), s.end());
        double mean = 0;
        for (double x : s) mean += x;
        mean = s.empty() ? 0 : mean / s.size();
        printf("stream budget=%u sub=%u gbs=%.1f lat_ns_mean=%.0f lat_ns_p50=%.0f lat_ns_p90=%.0f samples=%zu\n", budget, sub,
               budget ? median(rates) : 0.0, mean, s.empty() ? 0 : s[s.size() / 2], s.empty() ? 0 : s[s.size() * 9 / 10], s.size());
        fflush(stdout);
    };

    run(0, kTile); // exchange loads with nothing streaming
    for (unsigned int budget : {16384u, 32768u, 49152u, 65536u, 98304u, 131072u})
        for (unsigned int sub : {4096u, 8192u, 16384u, 32768u})
            if (sub <= budget) run(budget, sub);

    { // plain 128-bit loads over the same bytes
        std::vector<double> rates;
        for (int rep = 0; rep < 4; ++rep) {
            CK(cudaEventRecord(e0));
            k_ldg<<<sms * 4, 512>>>(reinterpret_cast<const uint4 *>(src), total / 16, sink);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaGetLastError());
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep) rates.push_back(total / (ms * 1e6));
        }
        printf("ldg128 gbs=%.1f\n", median(rates));
    }
    { // device-to-device copy: read rate (the same number of bytes is written)
        std::vector<double> rates;
        for (int rep = 0; rep < 4; ++rep) {
            CK(cudaEventRecord(e0));
            CK(cudaMemcpyAsync(dst, src, total / 2, cudaMemcpyDeviceToDevice));
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep) rates.push_back((total / 2) / (ms * 1e6));
        }
        printf("memcpy_d2d read_gbs=%.1f read+write_gbs=%.1f\n", median(rates), 2 * median(rates));
    }
    return 0;
}
