// quant_scale_probe — what the device computes for the two functions the float64 restatement (tests/numerics.py)
// has to reproduce bit for bit on the host: the quantiser's scale quant_scale(m) for every f32 mantissa of m in
// [1, 2) (the result scales exactly with the exponent: rcp.approx.ftz and the steps after it are scale-invariant
// for normal numbers), and expf(x) of the sigma(r) in the WKV on a grid of x in [-20, 20].
//
//   quant_scale_probe <out.bin>    writes 2^23 u32 inv bits, then 2^20 f32 x, then 2^20 f32 expf(-x)
#include <cstdio>
#include <vector>

#include "common.cuh"

constexpr unsigned kMant = 1u << 23;
constexpr unsigned kExp = 1u << 20;

__global__ void k_probe(uint32_t *inv, float *x, float *e) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < kMant) inv[i] = __float_as_uint(rk::quant_scale(__uint_as_float(0x3f800000u | i)));
    if (i < kExp) {
        const float xi = -20.0f + 40.0f * ((float)i / (float)kExp);
        x[i] = xi;
        e[i] = expf(-xi);
    }
}

int main(int argc, char **argv) {
    if (argc < 2) return 1;
    uint32_t *inv;
    float *x, *e;
    if (cudaMalloc(&inv, kMant * 4) || cudaMalloc(&x, kExp * 4) || cudaMalloc(&e, kExp * 4)) return 2;
    k_probe<<<kMant / 256, 256>>>(inv, x, e);
    std::vector<uint32_t> h(kMant + 2 * kExp);
    if (cudaMemcpy(h.data(), inv, kMant * 4, cudaMemcpyDeviceToHost) ||
        cudaMemcpy(h.data() + kMant, x, kExp * 4, cudaMemcpyDeviceToHost) ||
        cudaMemcpy(h.data() + kMant + kExp, e, kExp * 4, cudaMemcpyDeviceToHost))
        return 3;
    FILE *f = fopen(argv[1], "wb");
    if (!f || fwrite(h.data(), 4, h.size(), f) != h.size()) return 4;
    fclose(f);
    cudaFree(inv);
    cudaFree(x);
    cudaFree(e);
    return 0;
}
