// rwkv_oracle.cpp — CPU restatement of the reference's CUDA forward. TEST INFRASTRUCTURE.
//
// This file is the checker, never the product: only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / `--impl reference` legs may load it. The engine in
// rwkv-cpp-accelerated_b200/csrc/ does not link, include or call anything in oracle/.
//
// What it restates (all paths relative to harrisonvanderbyl/rwkv-cpp-accelerated):
//   orchestration + dtype flow     include/rwkv/cuda/rwkv.cu:493-593 (cuda_rwkv_parralel)
//   layernorm statistics           rwkv.cu:412-465 (addall, variance, meanvar), 40-57 (cuda_layernorm)
//   token shift                    rwkv.cu:351-392 (mixatt), 313-349 (mixffn)
//   uint8 dequant GEMV             rwkv.cu:58-100 (kernel_mm8_threec), 267-295 (kernelc_mm8_one)
//   WKV                            rwkv.cu:221-259 (kernel_wkvc_forward)
//   elementwise                    rwkv.cu:144-219 (setx, cuda_memset, cuda_relusquared, sigmoid), 394-410 (blockout)
//   file layout                    rwkv.cu:638-717 + include/rwkv/rwkv/rwkv.h:84,124-128
//
// Pinning status: the reference ships NO golden vectors for the forward (SURVEY.md 8c),
// so this oracle is pinned against the reference itself: oracle/_ref/ref_harness (the
// unmodified rwkv.cu + rwkv.h compiled for sm_90a by oracle/Makefile) is run on the
// GPU box on the same synthetic .bin and compared with this file in
// tests/test_parity_gpu.py::test_oracle_vs_reference_cuda. Where /root/reference or a
// GPU is unavailable that test skips and parity is "pinned by construction only".
//
// Deliberate, documented deviations from the CUDA reference (both inside its own
// run-to-run noise, because the reference reduces with fp32 atomicAdd in arbitrary order):
//   * split-K partial sums and layernorm partial sums are combined in ascending
//     block / thread order (one of the orders the reference may produce);
//   * libm exp/expf/sqrt instead of CUDA's libdevice versions (<= 2 ulp apart).
// Everything else keeps the reference's rounding points: f32 statistics, unbiased
// variance (E-1), no epsilon, FMA-contracted dequant `x*(w*r+o)`, the f32 round trip
// of the residual through the output projection, f64 WKV without max-shift.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <thread>

#include "../rwkv-cpp-accelerated_b200/csrc/binfmt.h"
#include "../include/rwkv/enums/enum.h"

namespace {

typedef unsigned long long ull;

constexpr ull kSplit = 16;   // MM8_ONE_JSPLIT  rwkv.cu:21
constexpr ull kEwBlock = 16; // EMBBLOCK: elements per thread in elementwise kernels, rwkv.cu:24
constexpr ull kVocab = binfmt::kVocab;

struct Model {
    ull L = 0, E = 0;
    void *map = nullptr;
    size_t map_bytes = 0;
    const uint8_t *t[binfmt::kNumTensors] = {};
    // scratch, named after the reference's buffers
    std::vector<double> x, buffer1, ffnk, ffnv;
    std::vector<float> buffer2, buffer3, buffer4, ffnr, kvr;
    int threads = 1;
};

// Column blocks of a GEMV are independent, so they may run on any number of host
// threads without changing a single bit of the result (cpu_baseline timing only).
template <class F> void parallel_blocks(int threads, long n, F &&fn) {
    if (threads <= 1 || n <= 1) {
        for (long i = 0; i < n; ++i) fn(i);
        return;
    }
    std::atomic<long> next{0};
    auto work = [&]() {
        for (;;) {
            const long i = next.fetch_add(1);
            if (i >= n) return;
            fn(i);
        }
    };
    std::vector<std::thread> pool;
    const int nt = threads < n ? threads : (int)n;
    for (int t = 1; t < nt; ++t) pool.emplace_back(work);
    work();
    for (auto &t : pool) t.join();
}

template <class T> const T *tensor(const Model &m, int i) { return reinterpret_cast<const T *>(m.t[i]); }

// ---- layernorm (rwkv.cu:412-465 + 40-57) -------------------------------------------
// addall: each CUDA thread sums its 16 consecutive doubles into a *float* accumulator
// (`accmini += a[i]` with accmini float -> round to f32 after every add), then the
// per-thread floats are atomically added into a float. variance: same shape, with the
// mean taken as float(mean_sum)/float(E) (float division, rwkv.cu:444).
void layernorm(const Model &m, const double *in, ull ln_row, double *out) {
    const ull E = m.E;
    const double *w = tensor<double>(m, LAYERNORMS) + ln_row * E;
    const double *b = w + E;
    float mean_acc = 0.0f;
    for (ull base = 0; base < E; base += kEwBlock) {
        float mini = 0.0f;
        for (ull c = 0; c < kEwBlock && base + c < E; ++c) mini = (float)((double)mini + in[base + c]);
        mean_acc += mini;
    }
    const float mean_f = mean_acc / (float)E; // `mean[token] / emb`: float / ull -> float
    float var_acc = 0.0f;
    for (ull base = 0; base < E; base += kEwBlock) {
        float mini = 0.0f;
        for (ull c = 0; c < kEwBlock && base + c < E; ++c) {
            const double d = in[base + c] - (double)mean_f;
            mini = (float)((double)mini + d * d);
        }
        var_acc += mini;
    }
    const double xmean = (double)mean_acc / (double)E;           // rwkv.cu:43
    const double x2 = (double)std::sqrt(var_acc / (float)(E - 1)); // rwkv.cu:44, float sqrt
    for (ull i = 0; i < E; ++i) out[i] = w[i] * ((in[i] - xmean) / x2) + b[i];
}

// ---- uint8 dequant GEMV (rwkv.cu:267-295 / 58-100) ------------------------------------
// y[k] += sum over 16 j-splits of ( f32 chain over j in split: acc = fma(x_j, fma(w,r,o), acc) ).
// XT is the activation type (double for kernelc_mm8_one<double>, float otherwise);
// the activation is cast to float per element (rwkv.cu:290).
template <class XT>
void mm8(const Model &m, ull N, ull M, const XT *x, const uint8_t *w, ull stride, float *y,
         const float *r, const float *o) {
    const ull chunk = (N + kSplit - 1) / kSplit;
    const ull KB = 512; // column block per task
    const long nblk = (long)((M + KB - 1) / KB);
    parallel_blocks(m.threads, nblk, [&](long blk) {
        const ull k0 = (ull)blk * KB, k1 = (k0 + KB < M) ? k0 + KB : M;
        float acc[KB];
        for (ull s = 0; s < kSplit; ++s) {
            const ull j0 = (s * chunk < N) ? s * chunk : N;
            const ull j1 = ((s + 1) * chunk < N) ? (s + 1) * chunk : N;
            for (ull k = 0; k < k1 - k0; ++k) acc[k] = 0.0f;
            for (ull j = j0; j < j1; ++j) {
                const float xj = (float)x[j];
                const float rj = r[j], oj = o[j];
                const uint8_t *wr = w + j * stride + k0;
                for (ull k = 0; k < k1 - k0; ++k)
                    acc[k] = std::fmaf(xj, std::fmaf((float)wr[k], rj, oj), acc[k]);
            }
            for (ull k = 0; k < k1 - k0; ++k) y[k0 + k] += acc[k];
        }
    });
}

void forward_one(Model &m, ull token, double *sxy, double *saa, double *sbb, double * /*spp*/,
                 double *sdd, float *logits) {
    const ull L = m.L, E = m.E;
    // rwkv.cu:513-524: embedding row (f32) -> buffer1 (f64) -> ln0 -> x
    const float *emb = tensor<float>(m, EMBED) + token * E;
    for (ull i = 0; i < E; ++i) m.buffer1[i] = (double)emb[i];
    layernorm(m, m.buffer1.data(), 0, m.x.data());

    for (ull l = 0; l < L; ++l) {
        // ---- attention block ---------------------------------------------------------
        layernorm(m, m.x.data(), 4 * l + 2, m.buffer1.data()); // rwkv.cu:535-537
        {                                                      // mixatt rwkv.cu:351-392
            const double *mk = tensor<double>(m, MIXK) + l * E, *mv = tensor<double>(m, MIXV) + l * E,
                         *mr = tensor<double>(m, MIXR) + l * E;
            double *st = sxy + l * E;
            for (ull i = 0; i < E; ++i) {
                const double rc = m.buffer1[i], dd = st[i];
                m.kvr[i] = (float)(mk[i] * rc + (1.0 - mk[i]) * dd);
                m.kvr[E + i] = (float)(mv[i] * rc + (1.0 - mv[i]) * dd);
                m.kvr[2 * E + i] = (float)(mr[i] * rc + (1.0 - mr[i]) * dd);
                st[i] = rc;
                m.buffer2[i] = m.buffer3[i] = m.buffer4[i] = 0.0f;
            }
        }
        // kernel_mm8_threec rwkv.cu:58-100: k,v,r
        mm8<float>(m, E, E, m.kvr.data(), tensor<uint8_t>(m, KM) + l * E * E, E, m.buffer2.data(),
                   tensor<float>(m, KR) + l * E, tensor<float>(m, O1) + l * E);
        mm8<float>(m, E, E, m.kvr.data() + E, tensor<uint8_t>(m, VM) + l * E * E, E, m.buffer3.data(),
                   tensor<float>(m, VR) + l * E, tensor<float>(m, O2) + l * E);
        mm8<float>(m, E, E, m.kvr.data() + 2 * E, tensor<uint8_t>(m, RM) + l * E * E, E,
                   m.buffer4.data(), tensor<float>(m, RR) + l * E, tensor<float>(m, O3) + l * E);
        { // kernel_wkvc_forward rwkv.cu:221-259 (unstabilised f64; pp untouched)
            const double *w = tensor<double>(m, DECAY) + l * E, *u = tensor<double>(m, BONUS) + l * E;
            double *aa = saa + l * E, *bb = sbb + l * E;
            for (ull i = 0; i < E; ++i) {
                const float kf = m.buffer2[i], rf = m.buffer4[i];
                const double vv = (double)m.buffer3[i];
                const double e1 = std::exp(u[i] + w[i] + (double)kf);
                const double wr1 = aa[i] + e1 * vv;
                const double wr2 = bb[i] + e1;
                double y = wr1 / wr2;
                y = (1.0 / (1.0 + (double)std::exp(-rf))) * y; // exp(float) overload, rwkv.cu:250
                m.buffer1[i] = y;
                const double ek = std::exp((double)kf), ew = std::exp(w[i]);
                aa[i] = (aa[i] + ek * vv) * ew;
                bb[i] = (bb[i] + ek) * ew;
            }
        }
        // rwkv.cu:548-553: residual goes through f32, the GEMV accumulates onto it
        for (ull i = 0; i < E; ++i) m.buffer2[i] = (float)m.x[i];
        mm8<double>(m, E, E, m.buffer1.data(), tensor<uint8_t>(m, ATTOUT) + l * E * E, E,
                    m.buffer2.data(), tensor<float>(m, ATTOUTR) + l * E, tensor<float>(m, ATTOUTO) + l * E);
        for (ull i = 0; i < E; ++i) m.x[i] = (double)m.buffer2[i];

        // ---- channel-mix (ffn) block ---------------------------------------------------
        layernorm(m, m.x.data(), 4 * (l + 1), m.buffer1.data()); // rwkv.cu:557-558
        {                                                        // mixffn rwkv.cu:313-349
            const double *mk = tensor<double>(m, FFNMIXK) + l * E, *mr = tensor<double>(m, FFNMIXV) + l * E;
            double *st = sdd + l * E;
            for (ull i = 0; i < E; ++i) {
                const double rc = m.buffer1[i], dd = st[i];
                m.ffnk[i] = mk[i] * rc + (1.0 - mk[i]) * dd;
                m.ffnv[i] = mr[i] * rc + (1.0 - mr[i]) * dd;
                st[i] = rc;
            }
        }
        for (ull i = 0; i < E; ++i) m.buffer2[i] = 0.0f; // rwkv.cu:566
        mm8<double>(m, E, E, m.ffnv.data(), tensor<uint8_t>(m, FFNR) + l * E * E, E, m.buffer2.data(),
                    tensor<float>(m, FFNRR) + l * E, tensor<float>(m, FFNRO) + l * E);
        for (ull i = 0; i < E; ++i) { // sigmoid rwkv.cu:199-219
            m.buffer4[i] = (float)(1.0 / (1.0 + std::exp(-(double)m.buffer2[i])));
            m.ffnr[4 * i] = m.ffnr[4 * i + 1] = m.ffnr[4 * i + 2] = m.ffnr[4 * i + 3] = 0.0f;
        }
        mm8<double>(m, E, 4 * E, m.ffnk.data(), tensor<uint8_t>(m, FFNK) + l * E * 4 * E, 4 * E,
                    m.ffnr.data(), tensor<float>(m, FFNKR) + l * E, tensor<float>(m, FFNKO) + l * E);
        for (ull i = 0; i < 4 * E; ++i) { // cuda_relusquared rwkv.cu:177-197
            float a = m.ffnr[i];
            a = a * (float)(a > 0);
            m.ffnr[i] = a * a;
            if (i % 4 == 0) m.buffer3[i / 4] = 0.0f;
        }
        mm8<float>(m, 4 * E, E, m.ffnr.data(), tensor<uint8_t>(m, FFNV) + l * 4 * E * E, E,
                   m.buffer3.data(), tensor<float>(m, FFNVR) + l * 4 * E, tensor<float>(m, FFNVO) + l * 4 * E);
        for (ull i = 0; i < E; ++i) m.x[i] = m.x[i] + (double)(m.buffer3[i] * m.buffer4[i]); // blockout rwkv.cu:407
    }
    // rwkv.cu:585-589: ln_out, head
    layernorm(m, m.x.data(), 4 * L + 2, m.buffer1.data());
    std::vector<float> &lg = m.buffer2;
    for (ull i = 0; i < kVocab; ++i) lg[i] = 0.0f;
    mm8<double>(m, E, kVocab, m.buffer1.data(), tensor<uint8_t>(m, HEAD), kVocab, lg.data(),
                tensor<float>(m, HEADR), tensor<float>(m, HEADO));
    if (logits) std::memcpy(logits, lg.data(), kVocab * sizeof(float));
}

} // namespace

extern "C" {

struct oracle_model;

oracle_model *oracle_load(const char *path) {
    int fd = open(path, O_RDONLY);
    if (fd < 0) return nullptr;
    struct stat st;
    if (fstat(fd, &st) != 0 || st.st_size < 16) {
        close(fd);
        return nullptr;
    }
    void *p = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (p == MAP_FAILED) return nullptr;
    const int64_t *hdr = (const int64_t *)p;
    Model *m = new Model;
    m->L = (ull)hdr[0];
    m->E = (ull)hdr[1];
    m->map = p;
    m->map_bytes = (size_t)st.st_size;
    if (m->L == 0 || m->E == 0 || binfmt::file_bytes(m->L, m->E) > (uint64_t)st.st_size) {
        munmap(p, m->map_bytes);
        delete m;
        return nullptr;
    }
    for (int i = 0; i < binfmt::kNumTensors; ++i)
        m->t[i] = (const uint8_t *)p + binfmt::offset(i, m->L, m->E);
    const ull E = m->E;
    m->x.assign(E, 0.0);
    m->buffer1.assign(E, 0.0);
    m->ffnk.assign(E, 0.0);
    m->ffnv.assign(E, 0.0);
    m->buffer2.assign(kVocab > E ? kVocab : E, 0.0f);
    m->buffer3.assign(E, 0.0f);
    m->buffer4.assign(E, 0.0f);
    m->ffnr.assign(4 * E, 0.0f);
    m->kvr.assign(3 * E, 0.0f);
    return (oracle_model *)m;
}

void oracle_free(oracle_model *h) {
    Model *m = (Model *)h;
    if (!m) return;
    if (m->map) munmap(m->map, m->map_bytes);
    delete m;
}

unsigned long long oracle_n_layers(oracle_model *h) { return ((Model *)h)->L; }
unsigned long long oracle_n_embed(oracle_model *h) { return ((Model *)h)->E; }

void oracle_set_threads(oracle_model *h, int threads) {
    Model *m = (Model *)h;
    m->threads = threads < 1 ? 1 : threads;
}

int oracle_max_threads(void) {
    const unsigned n = std::thread::hardware_concurrency();
    return n ? (int)n : 1;
}

// One token on caller-owned state (five arrays of n_layers*n_embed doubles, updated in
// place like the reference's RWKVState after getOutput). logits: 50277 floats or NULL.
void oracle_forward(oracle_model *h, unsigned long long token, double *xy, double *aa, double *bb,
                    double *pp, double *dd, float *logits) {
    forward_one(*(Model *)h, token, xy, aa, bb, pp, dd, logits);
}

// Residual stream after the last layer of the most recent forward (n_embed doubles);
// used by kernel-level parity tests.
const double *oracle_last_x(oracle_model *h) { return ((Model *)h)->x.data(); }

} // extern "C"
