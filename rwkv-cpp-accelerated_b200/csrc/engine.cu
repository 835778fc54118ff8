// engine.cu — host side of the H100 RWKV-v4 uint8 decode engine + the C ABI (include/rwkv_b200.h).
//
// Responsibilities:
//   * load a reference-format .bin (include/rwkv/cuda/rwkv.cu:638-717 semantics): each rank reads only
//     the slices of the matrices it streams, stages them through pinned memory, and repacks on the device
//     (transpose to [out][in], centre to s8, fold 128*r + o into one offset vector);
//   * keep state, embedding table, weights and logits resident in HBM;
//   * issue one token as ONE cooperative launch of the persistent token kernel (token_kernel.cuh);
//   * wire the exchange blocks of the ranks of a tensor-parallel group (CUDA IPC);
//   * measurement hooks used by bench.py.
//
// There is deliberately no CPU code path: every entry point that computes fails with an error when
// no sm_90 device is present.
#include <algorithm>
#include <cerrno>
#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <vector>

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cuda_runtime.h>

#include "../../include/rwkv/enums/enum.h"
#include "../../include/rwkv_b200.h"
#include "aux_kernels.cuh"
#include "beam.cuh"
#include "binfmt.h"
#include "generate.cuh"
#include "prefill.cuh"
#include "sampling.cuh"
#include "score.cuh"
#include "token_kernel.cuh"

namespace {

thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess)                                                                    \
            return fail(100 + (int)e__, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),  \
                        __FILE__, __LINE__);                                                       \
    } while (0)

// A device buffer that grows with the largest call and is freed with its owner (a failed free is ignored). grow() is
// called between calls, never with work in flight on the buffer: it never shrinks, frees the old block before
// allocating, and leaves cap 0 when the allocation fails.
template <class T> struct DevBuf {
    T *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr, o.cap = 0; }
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    int grow(size_t n) {
        if (n <= cap) return 0;
        release();
        CK(cudaMalloc((void **)&p, n * sizeof(T)));
        cap = n;
        return 0;
    }
};

const char *kKernelNames[1] = {"token"};

} // namespace

struct rwkv_b200_model {
    int device = 0;
    int sms = 0;
    int grid = 0;
    int cpl = 0;
    double *d_sample = nullptr, *h_sample = nullptr; // device sampler results {token, margin} per row, [max_gpt][2]
    double *d_u = nullptr;                            // the sampler's uniforms, [max_gpt]
    float *d_slogits = nullptr;       // [max_gpt][V] compact logits rows (forward_streams: one per stream)
    unsigned long long *d_next = nullptr; // [max_gpt] arg-max of each row of d_slogits
    unsigned long long stream_rows = 0;   // rows of d_slogits the last forward_streams call produced (0: none)
    size_t xch_bytes = 0;   // exchange block (peer-visible with tensor parallelism)
    bool tp_wired = false;  // peers' exchange blocks imported
    std::vector<void *> ipc_opened;
    unsigned long long L = 0, E = 0, max_gpt = 1;
    cudaStream_t stream = nullptr;
    rk::Params p{};
    size_t smem = 0;
    std::vector<void *> allocs;
    void *tensors[RWKV_B200_NUM_TENSORS] = {};
    double *spp = nullptr; // state_pp lives on the device only to honour the tensor table
    rk::Ctrl *h_ctrl = nullptr; // pinned [max_gpt]
    float *h_logits = nullptr;  // pinned [max_gpt][V]
    unsigned long long *h_next = nullptr;
    rk::Diag *h_diag = nullptr; // mapped pinned: the kernel's last words before a timeout trap
    int max_layers = -1;        // debug: run only the first n layers
    unsigned long long launches = 0;
    unsigned int epoch = 0, tk = 0; // exchange epochs (token_kernel.cuh); identical on every rank
    int tp_rank = 0, tp_size = 1;
    rk::PrefillState pf{};
    // generate_streams: per-stream records (device, and their pinned host mirror), the row map and the pass
    // descriptors are sized at load; the rest grows with the largest call and is freed with the model
    struct Gen {
        rk::GenStream *gs = nullptr, *h_gs = nullptr; // [max_gpt]
        int *row_stream = nullptr;                     // [max_gpt] stream of each row of the current group
        rk::PassDesc *passes = nullptr;                // [ceil(max_gpt / 128)] next step's passes (tensor cores)
        DevBuf<unsigned long long> out;                // [n_streams][max_new] emitted tokens
        DevBuf<unsigned long long> stop, ovr_tok;
        DevBuf<float> ovr_val;
        DevBuf<double> u;               // [group steps][rows] uniforms of the current group
        DevBuf<rwkv_b200_sampler> samp; // [n_streams] sampler of each stream (generate_streams_ex, sample_streams)
        DevBuf<float> pen_cnt;          // [n_streams][V] decayed counts of the emitted tokens (penalties only)
        DevBuf<unsigned char> pen_seen; // [n_streams][V] emitted in this call
        // generate_streams_logprobs: the results of each emitted token, and the model's rows of the step (raw mode with
        // penalties or overrides, which edit d_slogits in place)
        DevBuf<double> lp, top_lp;                 // [n_streams][max_new], [..][top_n]
        DevBuf<unsigned long long> rank, top_tok;  // [n_streams][max_new], [..][top_n]
        DevBuf<float> raw;                         // [rows][V]
        // generate_streams_constrained: each stream's automaton and state, and the record of a token without an edge
        DevBuf<rk::GenConstraint> gc;      // [n_streams]
        DevBuf<unsigned long long> fault;  // [3]
    } gen;
    // rwkv_b200_constraint_add: per id, the CSR on the host (the override check of a call) and one device block holding
    // the allow masks, then edge_start, the edge tokens and their targets
    struct Automaton {
        std::vector<unsigned long long> start; // [n_states + 1]
        std::vector<uint32_t> tok;             // [n_edges]
        DevBuf<unsigned char> dev;
        rk::GenConstraint view; // device pointers into dev, state 0
    };
    std::map<unsigned long long, Automaton> automata;
    unsigned long long next_automaton = 1;
    // score_streams: per scored row its d_slogits row and target in, its results out; grown with the largest call
    struct Score {
        DevBuf<int> rows;
        DevBuf<unsigned long long> tgt, rank, top_tok;
        DevBuf<double> lp, top_lp;
    } score;
    // beam_search: the beams' records live in gen.gs (beam j of group g is record g * B + j); the rest grows with the
    // largest call
    struct Beam {
        DevBuf<int> row0, groups;               // [G] step 0's row map, [G] the live groups of a host group
        DevBuf<unsigned long long> cand_tok;    // [rows][C]
        DevBuf<double> cand_lp, cum, P;         // [rows][C], [G * B], [N + 1]
        DevBuf<rk::BeamBack> back;              // [G][N][B]
        DevBuf<rk::BeamHyp> hyp;                // [G][K]
        DevBuf<int> n_hyp;                      // [G]
        DevBuf<unsigned long long> done, forks; // [G], [G * B][2]
    } beam;
};

namespace {

using M = rwkv_b200_model;

template <class T> int dmalloc(M *m, T **out, size_t count) {
    void *p = nullptr;
    CK(cudaMalloc(&p, count * sizeof(T) + 256));
    m->allocs.push_back(p);
    *out = reinterpret_cast<T *>(p);
    return 0;
}

int layers_to_run(const M *m) { return m->max_layers >= 0 && m->max_layers < (int)m->L ? m->max_layers : (int)m->L; }

// A failed synchronisation: if the kernel left a diagnostic record, say what it was waiting for.
int sync_failed(M *m, cudaError_t e, const char *what) {
    const rk::Diag *d = m->h_diag;
    if (d && d->code) {
        static const char *names[] = {"", "slice statistics", "activation vector", "offset sums", "peer partial sums",
                                      "sigmoid exchange", "completion flags", "arg-max candidates", "ring (full)", "ring (empty)",
                                      "cluster: limb planes free", "cluster: limb planes written"};
        return fail(100 + (int)e,
                    "%s failed: %s; token kernel timed out waiting for %s: rank %u cta %u thread %u layer %u kind %u "
                    "expected tag %u saw %u aux %llu (a peer rank that never launched, or a protocol bug)",
                    what, cudaGetErrorString(e), d->code < 12 ? names[d->code] : "?", d->rank, d->cta, d->thread, d->layer,
                    d->kind, d->expect, d->seen, d->aux);
    }
    return fail(100 + (int)e, "%s failed: %s", what, cudaGetErrorString(e));
}
#define SYNC(m)                                                          \
    do {                                                                 \
        cudaError_t e__ = cudaStreamSynchronize((m)->stream);            \
        if (e__ != cudaSuccess) return sync_failed((m), e__, "forward"); \
    } while (0)

// ---- kernel dispatch on the model width -------------------------------------------------
// CPL = 16-byte chunks per lane of an n_embed-byte row; FULL = n_embed == CPL * 512 (no tail predicates).
#define RK_CPLS(X) X(2) X(4) X(6) X(8) X(10)

const void *token_entry(int cpl, bool full, bool trace) {
#define X(A)                                                                                                          \
    if (cpl == A) {                                                                                                   \
        if (trace) return full ? (const void *)rk::k_token<A, true, true> : (const void *)rk::k_token<A, false, true>; \
        return full ? (const void *)rk::k_token<A, true, false> : (const void *)rk::k_token<A, false, false>;          \
    }
    RK_CPLS(X)
#undef X
    return nullptr;
}

int chunks_per_lane(unsigned long long seg_bytes) {
    int c = (int)((seg_bytes + 511) / 512);
    if (c < 2) c = 2;
    return (c + 1) & ~1;
}

// Ring geometry: a tile is eight row segments of n_embed bytes (one per consumer warp); as many stages
// as fit beside the limb planes.
void configure_ring(M *m) {
    rk::Params &p = m->p;
    p.tile_bytes = (int)(8 * m->E);
    p.stages = (int)std::min<size_t>(rk::kMaxStages, (rk::kSmemLimit - rk::smem_bytes(0, 0, p.plane_cap)) / p.tile_bytes);
    m->smem = rk::smem_bytes(p.stages, p.tile_bytes, p.plane_cap);
}

void fill_launch(int grid, int cluster, size_t smem, cudaLaunchConfig_t &cfg, cudaLaunchAttribute (&attrs)[2], cudaStream_t s) {
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(rk::kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    attrs[0].id = cudaLaunchAttributeCooperative;
    attrs[0].val.cooperative = 1;
    attrs[1].id = cudaLaunchAttributeClusterDimension;
    attrs[1].val.clusterDim.x = (unsigned int)cluster;
    attrs[1].val.clusterDim.y = 1;
    attrs[1].val.clusterDim.z = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = cluster > 1 ? 2 : 1;
}

int launch_token(M *m, int feed, bool greedy, const unsigned long long *stream, cudaStream_t s) {
    if (m->tp_size > 1 && !m->tp_wired)
        return fail(7, "tensor parallelism: call rwkv_b200_tp_import with every rank's handle before the first forward");
    rk::Params prm = m->p;
    prm.L_run = layers_to_run(m);
    prm.feed_mode = feed;
    prm.greedy = greedy ? 1 : 0;
    prm.stream = stream;
    prm.ep0 = m->epoch;
    prm.tk = ++m->tk;
    if (prm.tk == 0) prm.tk = ++m->tk; // tag 0 means "never written"
    m->epoch += (unsigned int)prm.L_run + 1u;
    void *args[] = {&prm};
    const bool full = m->E == (unsigned long long)m->cpl * 512ull;
    const void *fn = token_entry(m->cpl, full, m->p.trace != nullptr);
    if (!fn) return fail(3, "no kernel for %d chunks per lane", m->cpl);
    // cooperative: all CTAs resident together (they wait for each other's words); clusters of p.cluster CTAs share
    // the gather through distributed shared memory
    cudaLaunchConfig_t cfg{};
    cudaLaunchAttribute attrs[2];
    fill_launch(m->grid, m->p.cluster, m->smem, cfg, attrs, s);
    CK(cudaLaunchKernelExC(&cfg, fn, args));
    m->launches += 1;
    return 0;
}

// ---- loader --------------------------------------------------------------------------------
struct FileReader {
    int fd = -1;
    uint8_t *pin = nullptr;
    size_t pin_bytes = 0;
    ~FileReader() {
        if (fd >= 0) close(fd);
        if (pin) cudaFreeHost(pin);
    }
};

int read_exact(int fd, void *dst, size_t n, uint64_t off) {
    uint8_t *d = (uint8_t *)dst;
    while (n) {
        ssize_t got = pread(fd, d, n, (off_t)off);
        if (got < 0) {
            if (errno == EINTR) continue;
            return fail(4, "read error: %s", strerror(errno));
        }
        if (got == 0) return fail(4, "model file truncated");
        d += got;
        off += (uint64_t)got;
        n -= (size_t)got;
    }
    return 0;
}

// `rows` file rows of `row_stride` bytes starting at `off`; of each row the bytes [col0, col0 + cols)
// -> device dst, packed [rows][cols], through the pinned staging buffer. A rank of a tensor-parallel
// group reads only the columns / rows it streams.
int upload_rows(M *m, FileReader &fr, uint64_t off, size_t rows, size_t row_stride, size_t col0, size_t cols, void *dst) {
    uint8_t *d = (uint8_t *)dst;
    if (cols == row_stride) { // whole rows: one contiguous byte range
        size_t n = rows * cols;
        while (n) {
            const size_t c = std::min(n, fr.pin_bytes);
            int rc = read_exact(fr.fd, fr.pin, c, off);
            if (rc) return rc;
            CK(cudaMemcpyAsync(d, fr.pin, c, cudaMemcpyHostToDevice, m->stream));
            CK(cudaStreamSynchronize(m->stream));
            d += c;
            off += c;
            n -= c;
        }
        return 0;
    }
    if (cols > fr.pin_bytes) return fail(4, "row slice of %zu bytes exceeds the staging buffer", cols);
    const size_t per = fr.pin_bytes / cols;
    for (size_t r = 0; r < rows; r += per) {
        const size_t n = std::min(per, rows - r);
        for (size_t i = 0; i < n; ++i) {
            int rc = read_exact(fr.fd, fr.pin + i * cols, cols, off + (r + i) * row_stride + col0);
            if (rc) return rc;
        }
        CK(cudaMemcpyAsync(d + r * cols, fr.pin, n * cols, cudaMemcpyHostToDevice, m->stream));
        CK(cudaStreamSynchronize(m->stream));
    }
    return 0;
}

template <class T> int upload_tensor(M *m, FileReader &fr, int tid, T **out) {
    const size_t n = binfmt::elems(tid, m->L, m->E);
    int rc = dmalloc(m, out, n);
    if (rc) return rc;
    return upload_rows(m, fr, binfmt::offset(tid, m->L, m->E), 1, n * sizeof(T), 0, n * sizeof(T), *out);
}

// uint8 matrix family `tid`: `mats` matrices stored [rows_in][cols_out]; this rank keeps input rows
// [in0, in0 + nin) and output columns [out0, out0 + nout) -> int8 [nout][nin] per matrix.
int upload_matrix(M *m, FileReader &fr, int tid, size_t mats, size_t rows_in, size_t cols_out, size_t in0, size_t nin,
                  size_t out0, size_t nout, uint8_t *d_raw, int8_t **out) {
    int rc = dmalloc(m, out, mats * nin * nout);
    if (rc) return rc;
    const uint64_t base = binfmt::offset(tid, m->L, m->E);
    for (size_t i = 0; i < mats; ++i) {
        rc = upload_rows(m, fr, base + i * rows_in * cols_out + in0 * cols_out, nin, cols_out, out0, nout, d_raw);
        if (rc) return rc;
        dim3 g((unsigned)((nout + 63) / 64), (unsigned)((nin + 63) / 64));
        rk::k_transpose_xor<<<g, 256, 0, m->stream>>>(d_raw, nout, (int)nin, (int)nout, *out + i * nin * nout, nin, 0);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(m->stream));
    }
    return 0;
}

int centre(M *m, const float *r, const float *o, size_t n, const float **out) {
    float *oc = nullptr;
    int rc = dmalloc(m, &oc, n);
    if (rc) return rc;
    rk::k_centre_offsets<<<(unsigned)((n + 255) / 256), 256, 0, m->stream>>>(r, o, oc, n);
    CK(cudaGetLastError());
    *out = oc;
    return 0;
}

// Capacity checks of the per-CTA shared arrays for a grid of `grid` CTAs.
bool grid_fits(unsigned long long E, unsigned long long Er, unsigned long long Vr, int grid) {
    const unsigned long long g = (unsigned long long)grid;
    const unsigned long long ne = (E + g - 1) / g + 1, nc = (Er + g - 1) / g + 1, nk = (4 * Er + g - 1) / g + 1, nv = (Vr + g - 1) / g + 1;
    return grid >= 1 && grid <= rk::kMaxGrid && E >= g && ne <= (unsigned long long)rk::kMaxSlice &&
           nk <= 160 && nk + nc <= (unsigned long long)rk::kMaxRowsPerCta && 4 * ne <= (unsigned long long)rk::kMaxRowsPerCta &&
           3 * nc <= (unsigned long long)rk::kMaxRowsPerCta && nv <= (unsigned long long)rk::kMaxRowsPerCta;
}

// A grid of `grid` CTAs in clusters of `cluster`: divisibility, slice capacities, and - the CTAs wait for each
// other's words - that the device can hold all of them at once.
int check_grid(M *m, int grid, int cluster) {
    if (cluster != 1 && cluster != 2 && cluster != 4) return fail(1, "cluster must be 1, 2 or 4");
    if (grid < cluster || grid > m->sms || grid % cluster != 0)
        return fail(1, "grid=%d must be a multiple of cluster=%d and at most %d (the SM count)", grid, cluster, m->sms);
    if (!grid_fits(m->E, (unsigned long long)m->p.Er, (unsigned long long)m->p.Vr, grid))
        return fail(5, "a grid of %d CTAs does not fit n_embed=%llu", grid, m->E);
    if (cluster > 1) {
        cudaLaunchConfig_t cfg{};
        cudaLaunchAttribute attrs[2];
        fill_launch(grid, cluster, m->smem, cfg, attrs, m->stream);
        const bool full = m->E == (unsigned long long)m->cpl * 512ull;
        int nclusters = 0;
        CK(cudaOccupancyMaxActiveClusters(&nclusters, token_entry(m->cpl, full, m->p.trace != nullptr), &cfg));
        if (nclusters * cluster < grid)
            return fail(5, "the device holds %d clusters of %d CTAs at once; a grid of %d needs %d", nclusters, cluster, grid, grid / cluster);
    }
    return 0;
}

int do_load(M *m, const char *path, int quiet) {
    FileReader fr;
    fr.fd = open(path, O_RDONLY);
    if (fr.fd < 0) return fail(2, "Error opening file %s", path);
    int64_t hdr[2];
    int rc = read_exact(fr.fd, hdr, sizeof(hdr), 0);
    if (rc) return rc;
    m->L = (unsigned long long)hdr[0];
    m->E = (unsigned long long)hdr[1];
    const unsigned long long L = m->L, E = m->E, G = (unsigned long long)m->tp_size;
    if (!quiet) {
        printf("n_layers: %llu\nn_embed: %llu\n", L, E);
        fflush(stdout);
    }
    if (L == 0 || L > 4096 || E == 0 || E % 16 != 0 || E > 5120)
        return fail(5, "unsupported model shape: n_layers=%llu n_embed=%llu (need n_embed %% 16 == 0, <= 5120)", L, E);
    if (E % (16 * G) != 0)
        return fail(7, "tensor parallelism: n_embed=%llu is not a multiple of 16 x %llu ranks", E, G);
    struct stat st;
    if (fstat(fr.fd, &st) != 0 || (uint64_t)st.st_size < binfmt::file_bytes(L, E))
        return fail(4, "model file too short: %lld bytes, need %llu", (long long)st.st_size,
                    (unsigned long long)binfmt::file_bytes(L, E));

    CK(cudaSetDevice(m->device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, m->device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(6, "device %d is sm_%d%d; this engine is built for sm_90a only", m->device, prop.major, prop.minor);
    m->sms = prop.multiProcessorCount;
    m->grid = m->sms;
    CK(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    {
        int coop = 0;
        CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, m->device));
        if (!coop) return fail(6, "device does not support cooperative launch");
    }

    const unsigned long long Er = E / G;
    const unsigned long long V = binfmt::kVocab;
    const unsigned long long v_lo = V * (unsigned long long)m->tp_rank / G, v_hi = V * ((unsigned long long)m->tp_rank + 1) / G;
    const unsigned long long Vr = v_hi - v_lo;
    m->cpl = chunks_per_lane(E);
    rk::Params &p = m->p;
    p.L = (int)L;
    p.E = (int)E;
    p.G = (int)G;
    p.rank = m->tp_rank;
    p.Er = (int)Er;
    p.Vr = (int)Vr;
    p.vbase = (int)v_lo;
    p.plane_cap = (int)(12 * E);
    p.timeout_ms = G > 1 ? 60000u : 4000u;
    configure_ring(m);
    p.window = std::min(p.stages, 2);
    p.poll_first = 2;
    p.pf_dist = 4;
    p.bwindow = 1;
    p.vseg = G >= 4 ? 1 : G >= 2 ? 2 : 4; // 4E/G bytes per ffn-V row in segments of at most E bytes
    p.cluster = 1;
    if (p.stages < 2) return fail(5, "n_embed=%llu leaves no room for a two-stage ring", E);
    if (!grid_fits(E, Er, Vr, m->grid)) return fail(5, "a grid of %d CTAs does not fit n_embed=%llu", m->grid, E);
    const bool full = E == (unsigned long long)m->cpl * 512ull;
    for (int tr = 0; tr < 2; ++tr) {
        const void *fn = token_entry(m->cpl, full, tr != 0);
        if (!fn) return fail(3, "no kernel for %d chunks per lane", m->cpl);
        CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, rk::kSmemLimit));
    }

    fr.pin_bytes = 64u << 20;
    CK(cudaMallocHost((void **)&fr.pin, fr.pin_bytes));

    // The reference prints every tensor in file order (rwkv.cu:679); keep that UX.
    if (!quiet) {
        for (int t = 0; t < binfmt::kNumTensors; ++t) printf("loading: %s\n", binfmt::name(t));
        fflush(stdout);
    }

    // ---- small parameter tensors, reference dtype and shape (replicated on every rank) ----------
    float *emb, *kr, *vr, *rr, *o1, *o2, *o3, *aor, *aoo, *fkr, *fvr, *frr, *fko, *fvo, *fro, *hr, *ho;
    double *ln, *mixk, *mixv, *mixr, *fmk, *fmr, *decay, *bonus;
#define UP(tid, var)                                                                               \
    if ((rc = upload_tensor(m, fr, tid, &var))) return rc;                                          \
    m->tensors[tid] = var;
    UP(EMBED, emb) UP(LAYERNORMS, ln) UP(MIXK, mixk) UP(MIXV, mixv) UP(MIXR, mixr)
    UP(KR, kr) UP(VR, vr) UP(RR, rr) UP(O1, o1) UP(O2, o2) UP(O3, o3)
    UP(ATTOUTR, aor) UP(ATTOUTO, aoo) UP(FFNMIXK, fmk) UP(FFNMIXV, fmr)
    UP(FFNKR, fkr) UP(FFNVR, fvr) UP(FFNRR, frr) UP(FFNKO, fko) UP(FFNVO, fvo) UP(FFNRO, fro)
    UP(DECAY, decay) UP(BONUS, bonus) UP(HEADR, hr) UP(HEADO, ho)
#undef UP
    p.emb = emb; p.ln = ln; p.mixk = mixk; p.mixv = mixv; p.mixr = mixr; p.fmixk = fmk; p.fmixr = fmr;
    p.decay = decay; p.bonus = bonus;
    p.rk = kr; p.rv = vr; p.rr = rr; p.ro = aor; p.rfk = fkr; p.rfv = fvr; p.rfr = frr; p.rhead = hr;
    {
        double *ed = nullptr;
        if ((rc = dmalloc(m, &ed, (size_t)(L * E)))) return rc;
        rk::k_exp_table<<<(unsigned)((L * E + 255) / 256), 256, 0, m->stream>>>(decay, ed, (size_t)(L * E));
        CK(cudaGetLastError());
        p.expdecay = ed;
    }
    {
        std::vector<double> one(E, 1.0);
        double *d1 = nullptr;
        if ((rc = dmalloc(m, &d1, (size_t)E))) return rc;
        CK(cudaMemcpyAsync(d1, one.data(), E * sizeof(double), cudaMemcpyHostToDevice, m->stream));
        CK(cudaStreamSynchronize(m->stream));
        p.ones = d1;
    }
    if ((rc = centre(m, kr, o1, L * E, &p.ock))) return rc;
    if ((rc = centre(m, vr, o2, L * E, &p.ocv))) return rc;
    if ((rc = centre(m, rr, o3, L * E, &p.ocr))) return rc;
    if ((rc = centre(m, aor, aoo, L * E, &p.oco))) return rc;
    if ((rc = centre(m, fkr, fko, L * E, &p.ocfk))) return rc;
    if ((rc = centre(m, fvr, fvo, L * 4 * E, &p.ocfv))) return rc;
    if ((rc = centre(m, frr, fro, L * E, &p.ocfr))) return rc;
    if ((rc = centre(m, hr, ho, E, &p.ochead))) return rc;

    // ---- uint8 matrices: this rank's slices; stage raw, transpose + centre on the device ----------
    uint8_t *d_raw = nullptr;
    const size_t raw_bytes = std::max<size_t>(4 * Er * E, Vr * E);
    CK(cudaMalloc((void **)&d_raw, raw_bytes));
    const size_t c0 = (size_t)m->tp_rank * Er; // first channel of this rank
    int8_t *wk, *wv, *wr, *wo, *wfk, *wfv, *wfr, *whead;
    rc = upload_matrix(m, fr, KM, L, E, E, 0, E, c0, Er, d_raw, &wk);                         // column split
    if (!rc) rc = upload_matrix(m, fr, VM, L, E, E, 0, E, c0, Er, d_raw, &wv);
    if (!rc) rc = upload_matrix(m, fr, RM, L, E, E, 0, E, c0, Er, d_raw, &wr);
    if (!rc) rc = upload_matrix(m, fr, ATTOUT, L, E, E, c0, Er, 0, E, d_raw, &wo);             // row split
    if (!rc) rc = upload_matrix(m, fr, FFNK, L, E, 4 * E, 0, E, 4 * c0, 4 * Er, d_raw, &wfk);  // column split
    if (!rc) rc = upload_matrix(m, fr, FFNV, L, 4 * E, E, 4 * c0, 4 * Er, 0, E, d_raw, &wfv);  // row split
    if (!rc) rc = upload_matrix(m, fr, FFNR, L, E, E, 0, E, c0, Er, d_raw, &wfr);              // column split
    if (!rc) rc = upload_matrix(m, fr, HEAD, 1, E, V, 0, E, v_lo, Vr, d_raw, &whead);          // column split
    cudaFree(d_raw);
    if (rc) return rc;
    p.wk = wk; p.wv = wv; p.wr = wr; p.wo = wo; p.wfk = wfk; p.wfv = wfv; p.wfr = wfr; p.whead = whead;
    m->tensors[KM] = wk; m->tensors[VM] = wv; m->tensors[RM] = wr; m->tensors[ATTOUT] = wo;
    m->tensors[FFNK] = wfk; m->tensors[FFNV] = wfv; m->tensors[FFNR] = wfr; m->tensors[HEAD] = whead;

    // ---- state, activations, control ------------------------------------------------------------
    // The arrays the decode kernel reads and writes hold one slot more than max_gpt: generate_streams runs a finished
    // stream that still occupies a row on that scratch slot (index max_gpt). No public entry point reaches it.
    const size_t sn = (size_t)(L * E * m->max_gpt), sn1 = (size_t)(L * E * (m->max_gpt + 1));
    if ((rc = dmalloc(m, &p.sxy, sn1)) || (rc = dmalloc(m, &p.sdd, sn1)) || (rc = dmalloc(m, &m->spp, sn))) return rc;
    CK(cudaMemsetAsync(p.sxy, 0, sn1 * sizeof(double), m->stream));
    CK(cudaMemsetAsync(p.sdd, 0, sn1 * sizeof(double), m->stream));
    CK(cudaMemsetAsync(m->spp, 0, sn * sizeof(double), m->stream));
    double *b1, *fkb, *fvb;
    float *b3, *b4, *frb;
    if ((rc = dmalloc(m, &p.x, E)) || (rc = dmalloc(m, &p.ctrl, 1)) || (rc = dmalloc(m, &b1, E)) || (rc = dmalloc(m, &fkb, E)) ||
        (rc = dmalloc(m, &fvb, E)) || (rc = dmalloc(m, &b3, E)) || (rc = dmalloc(m, &b4, E)) || (rc = dmalloc(m, &frb, 4 * E)))
        return rc;
    CK(cudaMemsetAsync(p.ctrl, 0, sizeof(rk::Ctrl), m->stream));
    CK(cudaMemsetAsync(p.x, 0, E * sizeof(double), m->stream));
    // exchange block: one allocation, same layout on every rank (exchange.cuh)
    {
        size_t off = 256;
        auto take = [&](size_t bytes) {
            const size_t o = off;
            off = (off + bytes + 255) & ~(size_t)255;
            return o;
        };
        const size_t nb = (size_t)m->grid;
        for (int i = 0; i < 2; ++i) p.off_stat[i] = (unsigned int)take(rk::kRep * 2 * nb * sizeof(rk::TaggedDouble));
        for (int i = 0; i < 5; ++i) p.off_off[i] = (unsigned int)take(rk::kRep * 3 * nb * sizeof(rk::TaggedDouble));
        for (int i = 0; i < 5; ++i) p.off_max[i] = (unsigned int)take(rk::kRep * 3 * nb * 8);
        const size_t vlen[5] = {3 * E, Er, 2 * E, 4 * Er, E};
        for (int i = 0; i < 5; ++i) p.off_vec[i] = (unsigned int)take(vlen[i] * 4);
        for (int i = 0; i < 2; ++i) p.off_in[i] = (unsigned int)take(G * E * sizeof(rk::TaggedDouble));
        p.off_sr = (unsigned int)take(E * 8);
        p.off_arg = (unsigned int)take(G * nb * sizeof(rk::TaggedDouble));
        p.off_done = (unsigned int)take(G * nb * 8);
        p.off_logits = (unsigned int)take(V * 4);
        p.off_saa = take(sn1 * 8);
        p.off_sbb = take(sn1 * 8);
        m->xch_bytes = off;
        unsigned char *x = nullptr;
        if ((rc = dmalloc(m, &x, m->xch_bytes))) return rc;
        CK(cudaMemsetAsync(x, 0, m->xch_bytes, m->stream));
        for (int g = 0; g < rk::kMaxRanks; ++g) p.xch[g] = x; // peers are wired by rwkv_b200_tp_import
    }
    float *logits = reinterpret_cast<float *>(p.xch[0] + p.off_logits);
    double *saa = reinterpret_cast<double *>(p.xch[0] + p.off_saa), *sbb = reinterpret_cast<double *>(p.xch[0] + p.off_sbb);
    m->tensors[X] = p.x;
    m->tensors[STATEXY] = p.sxy; m->tensors[STATEAA] = saa; m->tensors[STATEBB] = sbb;
    m->tensors[STATEPP] = m->spp; m->tensors[STATEDD] = p.sdd;
    m->tensors[BUFFER1] = b1; m->tensors[BUFFER2] = logits; m->tensors[BUFFER3] = b3; m->tensors[BUFFER4] = b4;
    m->tensors[FFNKBUFFER] = fkb; m->tensors[FFNVBUFFER] = fvb; m->tensors[FFNRBUFFER] = frb;

    CK(cudaMallocHost((void **)&m->h_ctrl, sizeof(rk::Ctrl) * m->max_gpt));
    CK(cudaMallocHost((void **)&m->h_logits, sizeof(float) * V * m->max_gpt));
    CK(cudaMallocHost((void **)&m->h_next, sizeof(unsigned long long) * m->max_gpt));
    CK(cudaMallocHost((void **)&m->h_sample, 2 * sizeof(double) * m->max_gpt));
    if ((rc = dmalloc(m, &m->d_slogits, (size_t)V * m->max_gpt)) || (rc = dmalloc(m, &m->d_next, m->max_gpt)) ||
        (rc = dmalloc(m, &m->d_sample, 2 * m->max_gpt)) || (rc = dmalloc(m, &m->d_u, m->max_gpt)))
        return rc;
    if ((rc = dmalloc(m, &m->gen.gs, m->max_gpt)) || (rc = dmalloc(m, &m->gen.row_stream, m->max_gpt)) ||
        (rc = dmalloc(m, &m->gen.passes, (m->max_gpt + rk::kPfMaxTokens - 1) / rk::kPfMaxTokens)))
        return rc;
    CK(cudaMallocHost((void **)&m->gen.h_gs, sizeof(rk::GenStream) * m->max_gpt));
    CK(cudaHostAlloc((void **)&m->h_diag, sizeof(rk::Diag), cudaHostAllocMapped));
    memset(m->h_diag, 0, sizeof(rk::Diag));
    CK(cudaHostGetDevicePointer((void **)&p.diag, m->h_diag, 0));
    memset(m->h_logits, 0, sizeof(float) * V * m->max_gpt);
    CK(cudaStreamSynchronize(m->stream));
    return 0;
}

int check_model(const M *m) {
    if (!m) return fail(1, "null model handle");
    return 0;
}

float *dev_logits(M *m) { return reinterpret_cast<float *>(m->p.xch[m->tp_rank] + m->p.off_logits); }

// the reference applies the temperature as probs ^ uint8(1 / temp) (include/rwkv/sampler/typical.h)
int sample_exponent(float temp) { return temp != 1.0f ? (int)(unsigned char)(1.0 / (double)temp) : 1; }

// The five state arrays of one slot: xy, aa, bb, pp, dd ([L][E] doubles each at offset slot * L * E).
void slot_arrays(M *m, unsigned long long slot, double *(&a)[5]) {
    const size_t o = (size_t)(slot * m->L * m->E);
    double *base[5] = {m->p.sxy, (double *)m->tensors[STATEAA], (double *)m->tensors[STATEBB], m->spp, m->p.sdd};
    for (int i = 0; i < 5; ++i) a[i] = base[i] + o;
}

// Common checks of the multi-stream entry points.
int check_streams_model(M *m, const char *what) {
    int rc = check_model(m);
    if (rc) return rc;
    if (m->tp_size > 1) return fail(7, "%s: not supported with tensor parallelism", what);
    return 0;
}
int check_slot(M *m, const char *what, unsigned long long slot) {
    if (slot >= m->max_gpt) return fail(1, "%s: slot %llu >= max_gpt %llu", what, slot, m->max_gpt);
    return 0;
}

// n slots, each a slot of the model, none twice.
int check_slots(M *m, const char *what, const unsigned long long *slots, unsigned long long n) {
    std::vector<char> used(m->max_gpt, 0);
    for (unsigned long long i = 0; i < n; ++i) {
        if (int rc = check_slot(m, what, slots[i])) return rc;
        if (used[slots[i]]) return fail(1, "%s: slot %llu appears twice", what, slots[i]);
        used[slots[i]] = 1;
    }
    return 0;
}

// n token ids, each in the vocabulary; `of` names what index i counts ("first token 7 of stream 2").
int check_tokens(const char *what, const char *name, const unsigned long long *tokens, unsigned long long n,
                 const char *of = nullptr) {
    for (unsigned long long i = 0; i < n; ++i) {
        if (tokens[i] < binfmt::kVocab) continue;
        if (of) return fail(1, "%s: %s %llu of %s %llu out of range", what, name, tokens[i], of, i);
        return fail(1, "%s: %s %llu out of range", what, name, tokens[i]);
    }
    return 0;
}

// The model and the ragged token list of forward_streams and score_streams.
int check_ragged(M *m, const char *what, const unsigned long long *tokens, unsigned long long n_tokens,
                 const unsigned long long *slots, const unsigned long long *lengths, unsigned long long n_streams) {
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!tokens || !slots || !lengths || n_tokens == 0 || n_streams == 0) return fail(1, "%s: no tokens or no streams", what);
    if (n_tokens > m->max_gpt) return fail(1, "%s: %llu tokens > max_gpt %llu", what, n_tokens, m->max_gpt);
    if (n_streams > n_tokens) return fail(1, "%s: %llu streams for %llu tokens", what, n_streams, n_tokens);
    if ((rc = check_tokens(what, "token id", tokens, n_tokens)) || (rc = check_slots(m, what, slots, n_streams))) return rc;
    unsigned long long total = 0;
    for (unsigned long long i = 0; i < n_streams; ++i) {
        if (lengths[i] == 0 || lengths[i] > n_tokens) return fail(1, "%s: stream %llu has length %llu", what, i, lengths[i]);
        total += lengths[i];
    }
    if (total != n_tokens) return fail(1, "%s: the lengths add up to %llu, not n_tokens = %llu", what, total, n_tokens);
    return 0;
}

// Tensor cores or the decode kernel for a forward of n tokens: forward_streams' rule, which every call that has a
// choice follows (the multi-stream calls refuse tensor parallelism).
bool tensor_cores(const M *m, unsigned long long n) {
    return n >= (unsigned long long)m->pf.min_tokens && m->tp_size == 1 && rk::prefill_enabled(m->pf);
}

// Token by token through the decode kernel: stream i's lengths[i] tokens (stream-major) on slot slots[i]. Token t gets
// its own pinned control record (the source of a copy still in flight when the next token is queued). Its logits are
// copied (`kind`) to row(t, i, last) unless that is NULL; `last`: t is stream i's final token.
template <class Row>
int decode_tokens(M *m, const unsigned long long *tokens, const unsigned long long *slots, const unsigned long long *lengths,
                  unsigned long long n_streams, cudaMemcpyKind kind, Row row) {
    const size_t V = binfmt::kVocab;
    for (unsigned long long i = 0, t = 0; i < n_streams; ++i)
        for (unsigned long long k = 0; k < lengths[i]; ++k, ++t) {
            rk::Ctrl &c = m->h_ctrl[t];
            c.token = tokens[t];
            c.next = 0;
            c.slot = slots[i];
            c.pos = 0;
            CK(cudaMemcpyAsync(m->p.ctrl, &c, sizeof(rk::Ctrl), cudaMemcpyHostToDevice, m->stream));
            if (int rc = launch_token(m, 0, false, nullptr, m->stream)) return rc;
            if (float *dst = row(t, i, k + 1 == lengths[i])) CK(cudaMemcpyAsync(dst, dev_logits(m), V * sizeof(float), kind, m->stream));
        }
    return 0;
}

// The device sampler's picks {token, margin} of rows 0..n-1, read back with one synchronisation.
int read_samples(M *m, unsigned long long n, unsigned long long *tokens_out, double *margins_out) {
    CK(cudaMemcpyAsync(m->h_sample, m->d_sample, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    for (unsigned long long i = 0; i < n; ++i) {
        tokens_out[i] = (unsigned long long)m->h_sample[2 * i];
        if (margins_out) margins_out[i] = m->h_sample[2 * i + 1];
    }
    return 0;
}

// generate_streams enqueues this many steps between two looks at the streams' done flags: one synchronisation per
// group, and at most this many - 1 steps spent on streams that have finished.
constexpr unsigned long long kGenGroup = 16;

// Largest |presence| or |frequency| penalty accepted: penalised logits stay far inside the f32 range.
constexpr float kMaxPenalty = 1e6f;

// One step of generate_streams over `rows` rows on the decode kernel: each row on its stream's slot (or the scratch
// slot once the stream is done), its logits into row r of d_slogits. row_stream: the stream record of each row.
int gen_step_decode(M *m, int rows, const int *row_stream) {
    const size_t V = binfmt::kVocab;
    for (int r = 0; r < rows; ++r) {
        rk::k_gen_gate<<<1, 1, 0, m->stream>>>(m->gen.gs, row_stream, r, m->max_gpt, m->p.ctrl);
        CK(cudaGetLastError());
        int rc = launch_token(m, 0, false, nullptr, m->stream);
        if (rc) return rc;
        CK(cudaMemcpyAsync(m->d_slogits + (size_t)r * V, dev_logits(m), V * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
        m->launches += 1;
    }
    return 0;
}

// One step of generate_streams on the tensor cores: ceil(rows / 128) passes whose descriptors the previous step's
// feedback (or the group's upload) left in gen.passes; every row is a head row, so row r's logits land in d_slogits row r.
int gen_step_passes(M *m, int rows) {
    for (int p0 = 0, pi = 0; p0 < rows; p0 += rk::kPfMaxTokens, ++pi) {
        const int T = std::min(rk::kPfMaxTokens, rows - p0);
        CK(cudaMemcpyAsync(m->pf.pass, m->gen.passes + pi, sizeof(rk::PassDesc), cudaMemcpyDeviceToDevice, m->stream));
        int rc = rk::prefill_run(m->pf, m->p, m->stream, T, T, m->d_slogits);
        if (rc) return fail(rc, "%s", rk::prefill_error());
    }
    m->launches += rk::prefill_launches(m->pf);
    return 0;
}

// The passes of a step of `rows` one-token streams, row r on stream record rec[r] (its input token and slot), each row a
// head row: pass_layout's passes, uploaded to gen.passes in one copy.
int upload_step_passes(M *m, const int *rec, int rows) {
    std::vector<unsigned long long> tokens(rows), slots(rows), lens(rows, 1);
    for (int r = 0; r < rows; ++r) {
        tokens[r] = m->gen.h_gs[rec[r]].tok;
        slots[r] = m->gen.h_gs[rec[r]].slot;
    }
    std::vector<rk::PassDesc> passes;
    std::vector<int> heads;
    rk::pass_layout(tokens.data(), rows, slots.data(), lens.data(), 2, nullptr, passes, heads);
    CK(cudaMemcpyAsync(m->gen.passes, passes.data(), passes.size() * sizeof(rk::PassDesc), cudaMemcpyHostToDevice, m->stream));
    return 0;
}

// One stream's sampler. `history`: the call keeps the stream's emitted tokens (generate_streams_ex), so the penalties
// may be set; elsewhere they must be 0 and penalty_decay is not read.
int check_sampler(const char *what, unsigned long long s, const rwkv_b200_sampler &p, bool history) {
    if (!(p.temperature >= 0.0f && p.temperature <= FLT_MAX))
        return fail(1, "%s: stream %llu: temperature %g is not a finite value >= 0", what, s, p.temperature);
    if (!(p.top_p > 0.0f && p.top_p <= 1.0f)) return fail(1, "%s: stream %llu: top_p %g is outside (0, 1]", what, s, p.top_p);
    if (p.top_k > binfmt::kVocab) return fail(1, "%s: stream %llu: top_k %u > %llu", what, s, p.top_k, (unsigned long long)binfmt::kVocab);
    if (!history) {
        if (p.presence_penalty != 0.0f || p.frequency_penalty != 0.0f)
            return fail(1, "%s: stream %llu: presence_penalty and frequency_penalty must be 0 here (no token history; see "
                           "generate_streams_ex)", what, s);
        return 0;
    }
    if (!(fabsf(p.presence_penalty) <= kMaxPenalty))
        return fail(1, "%s: stream %llu: presence_penalty %g is not finite or exceeds %g in magnitude", what, s, p.presence_penalty, kMaxPenalty);
    if (!(fabsf(p.frequency_penalty) <= kMaxPenalty))
        return fail(1, "%s: stream %llu: frequency_penalty %g is not finite or exceeds %g in magnitude", what, s, p.frequency_penalty, kMaxPenalty);
    if (!(p.penalty_decay > 0.0f && p.penalty_decay <= 1.0f))
        return fail(1, "%s: stream %llu: penalty_decay %g is outside (0, 1]", what, s, p.penalty_decay);
    return 0;
}

// Override values of generate_streams_ex: finite or -inf, and not every token -inf (a repeated token keeps its last value).
int check_overrides(const char *what, const unsigned long long *tok, const float *val, unsigned long long n) {
    std::vector<char> masked(binfmt::kVocab, 0);
    for (unsigned long long i = 0; i < n; ++i) {
        if (!(std::isfinite(val[i]) || val[i] == -INFINITY))
            return fail(1, "%s: override value %g of token %llu is neither finite nor -inf", what, val[i], tok[i]);
        masked[tok[i]] = val[i] == -INFINITY;
    }
    if (n >= binfmt::kVocab && std::count(masked.begin(), masked.end(), 1) == (long)binfmt::kVocab)
        return fail(1, "%s: the overrides set every token to -inf", what);
    return 0;
}

// What generate_streams_logprobs asks for: the mode, top_n and the caller's result arrays.
struct LogprobRequest {
    int mode;
    unsigned top_n;
    double *logprobs_out;
    unsigned long long *ranks_out, *top_tokens_out;
    double *top_logprobs_out;
};

// What generate_streams_constrained adds: an automaton id per stream (or NULL), start states, final states.
struct ConstraintRequest {
    const unsigned long long *ids, *start_states;
    unsigned long long *states_out;
};

// The automaton of each stream of a constrained call (a zero record: none), refused before any work: unknown ids, start
// states out of range or without edges, and an automaton with a state whose every edge token the overrides set to -inf.
int check_constraints(M *m, const char *what, const ConstraintRequest &cq, unsigned long long n_streams,
                      const unsigned long long *override_tokens, const float *override_values, unsigned long long n_override,
                      std::vector<rk::GenConstraint> &out) {
    out.assign(n_streams, rk::GenConstraint{});
    if (!cq.ids) return 0;
    std::vector<char> masked(binfmt::kVocab, 0);
    for (unsigned long long i = 0; i < n_override; ++i) masked[override_tokens[i]] = override_values[i] == -INFINITY;
    std::vector<unsigned long long> seen;
    for (unsigned long long s = 0; s < n_streams; ++s) {
        const unsigned long long id = cq.ids[s];
        if (id == RWKV_B200_NO_CONSTRAINT) continue;
        const auto it = m->automata.find(id);
        if (it == m->automata.end()) return fail(1, "%s: stream %llu: constraint id %llu is unknown or removed", what, s, id);
        const M::Automaton &a = it->second;
        const unsigned long long n_states = a.start.size() - 1, q = cq.start_states ? cq.start_states[s] : 0;
        if (q >= n_states)
            return fail(1, "%s: stream %llu: start state %llu of constraint %llu is out of range (%llu states)", what, s, q, id,
                        n_states);
        if (a.start[q] == a.start[q + 1])
            return fail(1, "%s: stream %llu: start state %llu of constraint %llu has no edges (the automaton is complete there)",
                        what, s, q, id);
        out[s] = a.view;
        out[s].state = q;
        if (!n_override || std::find(seen.begin(), seen.end(), id) != seen.end()) continue;
        seen.push_back(id);
        for (unsigned long long p = 0; p < n_states; ++p) {
            bool open = a.start[p] == a.start[p + 1];
            for (unsigned long long e = a.start[p]; e < a.start[p + 1] && !open; ++e) open = !masked[a.tok[e]];
            if (!open)
                return fail(1, "%s: the overrides set every edge token of state %llu of constraint %llu to -inf", what, p, id);
        }
    }
    return 0;
}

// The body of generate_streams (samplers == NULL, `temp` and `u` pick the typical sampler or the arg-max), of
// generate_streams_ex (`ex`: every stream has its own sampler, or all pick the arg-max when samplers == NULL), of
// generate_streams_logprobs (generate_streams_ex with `lpq`: each emitted token is scored after its pick) and of
// generate_streams_constrained (with `cq`: token automata mask the rows after the overrides; `lpq` may be NULL).
int generate(M *m, const char *what, bool ex, const unsigned long long *slots, const unsigned long long *first_tokens,
             unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
             const unsigned long long *stop_tokens, unsigned long long n_stop, const unsigned long long *override_tokens,
             const float *override_values, unsigned long long n_override, float temp, const rwkv_b200_sampler *samplers,
             const double *u, unsigned long long *tokens_out, unsigned long long *lengths_out,
             const LogprobRequest *lpq = nullptr, const ConstraintRequest *cq = nullptr) {
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (lpq) {
        if (lpq->mode != RWKV_B200_LOGPROBS_RAW && lpq->mode != RWKV_B200_LOGPROBS_PROCESSED)
            return fail(1, "%s: logprob_mode %d is neither RWKV_B200_LOGPROBS_RAW (0) nor RWKV_B200_LOGPROBS_PROCESSED (1)", what,
                        lpq->mode);
        if (lpq->top_n > (unsigned)rk::kMaxTopN) return fail(1, "%s: top_n %u > %d", what, lpq->top_n, rk::kMaxTopN);
        if (!lpq->logprobs_out) return fail(1, "%s: logprobs_out is NULL", what);
        if (lpq->top_n && (!lpq->top_tokens_out || !lpq->top_logprobs_out))
            return fail(1, "%s: top_n = %u needs top_tokens_out and top_logprobs_out", what, lpq->top_n);
    }
    if (n_streams == 0) return fail(1, "%s: no streams", what);
    if (!slots || !first_tokens || !tokens_out || !lengths_out)
        return fail(1, "%s: null argument (slots, first_tokens, tokens_out and lengths_out are required)", what);
    if (n_stop && !stop_tokens) return fail(1, "%s: n_stop = %llu with NULL stop_tokens", what, n_stop);
    if (n_override && (!override_tokens || !override_values))
        return fail(1, "%s: n_override = %llu with NULL override_tokens or override_values", what, n_override);
    if (max_new == 0) return fail(1, "%s: max_new is 0", what);
    const size_t V = binfmt::kVocab;
    if ((rc = check_slots(m, what, slots, n_streams)) || (rc = check_tokens(what, "first token", first_tokens, n_streams, "stream")))
        return rc;
    for (unsigned long long i = 0; budgets && i < n_streams; ++i)
        if (budgets[i] == 0 || budgets[i] > max_new)
            return fail(1, "%s: budget %llu of stream %llu is outside 1..max_new = %llu", what, budgets[i], i, max_new);
    if ((rc = check_tokens(what, "stop token", stop_tokens, n_stop)) ||
        (rc = check_tokens(what, "override token", override_tokens, n_override)))
        return rc;
    bool pen = false; // some stream has a presence or frequency penalty
    if (ex) {
        if ((rc = check_overrides(what, override_tokens, override_values, n_override))) return rc;
        for (unsigned long long s = 0; samplers && s < n_streams; ++s) {
            if ((rc = check_sampler(what, s, samplers[s], true))) return rc;
            if (samplers[s].temperature > 0.0f && !u)
                return fail(1, "%s: u is NULL but stream %llu samples (temperature %g)", what, s, samplers[s].temperature);
            pen |= samplers[s].presence_penalty != 0.0f || samplers[s].frequency_penalty != 0.0f;
        }
    }
    if (u)
        for (unsigned long long i = 0; i < max_new * n_streams; ++i)
            if (!(u[i] >= 0.0 && u[i] < 1.0)) return fail(1, "%s: u[%llu] = %g is outside [0, 1)", what, i, u[i]);
    std::vector<rk::GenConstraint> hgc;
    if (cq && (rc = check_constraints(m, what, *cq, n_streams, override_tokens, override_values, n_override, hgc))) return rc;
    const bool constrained = std::any_of(hgc.begin(), hgc.end(), [](const rk::GenConstraint &c) { return c.mask != nullptr; });
    CK(cudaSetDevice(m->device));
    auto &g = m->gen;
    if (constrained && ((rc = g.gc.grow(n_streams)) || (rc = g.fault.grow(3)))) return rc;
    if (samplers && (rc = g.samp.grow(n_streams))) return rc;
    if (pen && ((rc = g.pen_cnt.grow(n_streams * V)) || (rc = g.pen_seen.grow(n_streams * V)))) return rc;
    if ((rc = g.out.grow(n_streams * max_new)) || (rc = g.stop.grow(n_stop)) || (rc = g.ovr_tok.grow(n_override)) ||
        (rc = g.ovr_val.grow(n_override)) || (u && (rc = g.u.grow(kGenGroup * m->max_gpt))))
        return rc;
    // raw mode reads the model's rows: d_slogits itself, or a copy taken before the penalties, overrides and mask edit it
    const bool raw_copy = lpq && lpq->mode == RWKV_B200_LOGPROBS_RAW && (pen || n_override || constrained);
    const size_t n_lp = (size_t)(n_streams * max_new), n_top = lpq ? n_lp * lpq->top_n : 0;
    if (lpq && ((rc = g.lp.grow(n_lp)) || (rc = g.rank.grow(n_lp)) || (rc = g.top_tok.grow(n_top)) || (rc = g.top_lp.grow(n_top)) ||
                (raw_copy && (rc = g.raw.grow(n_streams * V)))))
        return rc;
    // the path is chosen once, for n_streams tokens; a stream's numbers depend only on its row
    const bool tc = tensor_cores(m, n_streams);
    if (tc && (rc = rk::prefill_init(m->pf, m->p))) return fail(rc, "%s", rk::prefill_error());
    m->stream_rows = 0; // the compact logits rows no longer belong to a call the caller made

    rk::GenStream *hg = g.h_gs;
    for (unsigned long long s = 0; s < n_streams; ++s) hg[s] = rk::GenStream{slots[s], budgets ? budgets[s] : max_new, first_tokens[s], 0, 0};
    CK(cudaMemcpyAsync(g.gs, hg, n_streams * sizeof(rk::GenStream), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemsetAsync(g.out.p, 0, n_streams * max_new * sizeof(unsigned long long), m->stream));
    if (n_stop) CK(cudaMemcpyAsync(g.stop.p, stop_tokens, n_stop * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    if (n_override) {
        CK(cudaMemcpyAsync(g.ovr_tok.p, override_tokens, n_override * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(g.ovr_val.p, override_values, n_override * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    }
    if (samplers) CK(cudaMemcpyAsync(g.samp.p, samplers, n_streams * sizeof(rwkv_b200_sampler), cudaMemcpyHostToDevice, m->stream));
    if (constrained) {
        CK(cudaMemcpyAsync(g.gc.p, hgc.data(), n_streams * sizeof(rk::GenConstraint), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemsetAsync(g.fault.p, 0, 3 * sizeof(unsigned long long), m->stream));
    }
    if (pen) { // the history starts empty in every call: prompt tokens are not counted
        CK(cudaMemsetAsync(g.pen_cnt.p, 0, n_streams * V * sizeof(float), m->stream));
        CK(cudaMemsetAsync(g.pen_seen.p, 0, n_streams * V, m->stream));
    }
    if (lpq) { // all ones: NaN logprobs and RWKV_B200_NO_TARGET ranks and tokens wherever no token is emitted
        CK(cudaMemsetAsync(g.lp.p, 0xFF, n_lp * sizeof(double), m->stream));
        CK(cudaMemsetAsync(g.rank.p, 0xFF, n_lp * sizeof(unsigned long long), m->stream));
        if (n_top) {
            CK(cudaMemsetAsync(g.top_tok.p, 0xFF, n_top * sizeof(unsigned long long), m->stream));
            CK(cudaMemsetAsync(g.top_lp.p, 0xFF, n_top * sizeof(double), m->stream));
        }
    }
    std::vector<int> live(n_streams);
    for (unsigned long long s = 0; s < n_streams; ++s) live[s] = (int)s;
    std::vector<double> ug;
    const int exponent = sample_exponent(temp);
    for (unsigned long long step = 0; !live.empty() && step < max_new;) {
        // a group: the live streams are rows 0..rows-1; their inputs, and the uniforms of its steps, go up once
        const int rows = (int)live.size();
        const unsigned long long steps = std::min(kGenGroup, max_new - step);
        CK(cudaMemcpyAsync(g.row_stream, live.data(), rows * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        if (tc && (rc = upload_step_passes(m, live.data(), rows))) return rc;
        if (u) {
            ug.resize((size_t)steps * rows);
            for (unsigned long long k = 0; k < steps; ++k)
                for (int r = 0; r < rows; ++r) ug[k * rows + r] = u[(step + k) * n_streams + live[r]];
            CK(cudaMemcpyAsync(g.u.p, ug.data(), ug.size() * sizeof(double), cudaMemcpyHostToDevice, m->stream));
        }
        rk::GenFeedbackArgs fb{g.gs, g.row_stream, rows, u || samplers ? nullptr : m->d_next, m->d_sample, g.stop.p, (int)n_stop, g.out.p,
                               max_new, tc ? g.passes : nullptr, constrained ? g.gc.p : nullptr, g.fault.p};
        rk::GenLogprobArgs la{};
        if (lpq)
            la = rk::GenLogprobArgs{raw_copy ? g.raw.p : m->d_slogits, (int)V, g.gs, g.row_stream, fb.next, m->d_sample,
                                    lpq->mode == RWKV_B200_LOGPROBS_PROCESSED ? samplers ? g.samp.p : nullptr : nullptr,
                                    (int)lpq->top_n, max_new, g.lp.p, g.rank.p, g.top_tok.p, g.top_lp.p};
        const unsigned rb = (unsigned)((rows + 127) / 128);
        for (unsigned long long k = 0; k < steps; ++k) {
            if ((rc = tc ? gen_step_passes(m, rows) : gen_step_decode(m, rows, g.row_stream))) return rc;
            if (raw_copy)
                CK(cudaMemcpyAsync(g.raw.p, m->d_slogits, (size_t)rows * V * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
            if (pen) {
                const dim3 grid((unsigned)((V + rk::kPenaltyThreads - 1) / rk::kPenaltyThreads), (unsigned)rows);
                rk::k_gen_penalty<<<grid, rk::kPenaltyThreads, 0, m->stream>>>(m->d_slogits, (int)V, g.gs, g.row_stream, g.samp.p,
                                                                              g.pen_cnt.p, g.pen_seen.p);
                CK(cudaGetLastError());
                m->launches += 1;
            }
            if (n_override) {
                rk::k_gen_override<<<rb, 128, 0, m->stream>>>(m->d_slogits, (int)V, rows, g.ovr_tok.p, g.ovr_val.p, (int)n_override);
                CK(cudaGetLastError());
                m->launches += 1;
            }
            if (constrained) {
                const dim3 grid((unsigned)((V + rk::kMaskThreads - 1) / rk::kMaskThreads), (unsigned)rows);
                rk::k_gen_mask<<<grid, rk::kMaskThreads, 0, m->stream>>>(m->d_slogits, (int)V, g.gs, g.row_stream, g.gc.p);
                CK(cudaGetLastError());
                m->launches += 1;
            }
            if (samplers)
                rk::k_sample_nucleus<<<(unsigned)rows, rk::kNucThreads, 0, m->stream>>>(m->d_slogits, (int)V, g.samp.p, g.row_stream,
                                                                                       u ? g.u.p + k * rows : nullptr, m->d_sample);
            else if (u)
                rk::k_sample_typical<<<(unsigned)rows, rk::kSampleThreads, 0, m->stream>>>(m->d_slogits, V, (int)V, exponent,
                                                                                          g.u.p + k * rows, m->d_sample);
            else
                rk::k_argmax_rows<<<(unsigned)rows, rk::kArgmaxThreads, 0, m->stream>>>(m->d_slogits, (int)V, m->d_next);
            CK(cudaGetLastError());
            if (lpq) {
                rk::k_gen_logprob<<<(unsigned)rows, rk::kNucThreads, 0, m->stream>>>(la);
                CK(cudaGetLastError());
                m->launches += 1;
            }
            rk::k_gen_feedback<<<rb, 128, 0, m->stream>>>(fb);
            CK(cudaGetLastError());
            m->launches += 2;
        }
        // the end of a group: which streams are done (a few bytes, one synchronisation); drop them from the rows
        CK(cudaMemcpyAsync(hg, g.gs, n_streams * sizeof(rk::GenStream), cudaMemcpyDeviceToHost, m->stream));
        unsigned long long fault[3] = {0, 0, 0};
        if (constrained) CK(cudaMemcpyAsync(fault, g.fault.p, sizeof(fault), cudaMemcpyDeviceToHost, m->stream));
        SYNC(m);
        if (fault[0])
            return fail(8, "%s: stream %llu emitted token %llu, which has no edge out of state %llu of its constraint", what,
                        fault[0] - 1, fault[1], fault[2]);
        step += steps;
        live.erase(std::remove_if(live.begin(), live.end(), [&](int s) { return hg[s].done != 0; }), live.end());
    }
    CK(cudaMemcpyAsync(tokens_out, g.out.p, n_streams * max_new * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
    if (lpq) {
        CK(cudaMemcpyAsync(lpq->logprobs_out, g.lp.p, n_lp * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        if (lpq->ranks_out) CK(cudaMemcpyAsync(lpq->ranks_out, g.rank.p, n_lp * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        if (n_top) {
            CK(cudaMemcpyAsync(lpq->top_tokens_out, g.top_tok.p, n_top * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
            CK(cudaMemcpyAsync(lpq->top_logprobs_out, g.top_lp.p, n_top * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        }
    }
    if (constrained && cq->states_out)
        CK(cudaMemcpyAsync(hgc.data(), g.gc.p, n_streams * sizeof(rk::GenConstraint), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    for (unsigned long long s = 0; s < n_streams; ++s) lengths_out[s] = hg[s].len;
    if (cq && cq->states_out)
        for (unsigned long long s = 0; s < n_streams; ++s) cq->states_out[s] = hgc[s].mask ? hgc[s].state : 0;
    return 0;
}

// The body of rwkv_b200_beam_search: generate()'s group loop over beams. Step 0 has one row per group, later steps B
// rows per live group (group by group); each step is forward -> k_beam_expand -> k_beam_select -> k_beam_fork. At each
// host group's end the done flags come back and the done groups leave the rows; at the end the backpointers and the
// hypothesis lists come back once and the host rebuilds each hypothesis' tokens.
int beam(M *m, const unsigned long long *slots, const unsigned long long *first_tokens, unsigned long long n_groups,
         unsigned beams, unsigned long long max_new, const unsigned long long *stop_tokens, unsigned long long n_stop,
         double length_penalty, unsigned n_best, unsigned long long *tokens_out, unsigned long long *lengths_out,
         double *logprobs_out, double *scores_out, unsigned char *finished_out, double *token_logprobs_out) {
    const char *what = "beam_search";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!slots || !first_tokens || !tokens_out || !lengths_out || !logprobs_out || !scores_out || !finished_out)
        return fail(1, "%s: null argument (slots, first_tokens, tokens_out, lengths_out, logprobs_out, scores_out and "
                       "finished_out are required)", what);
    if (n_stop && !stop_tokens) return fail(1, "%s: n_stop = %llu with NULL stop_tokens", what, n_stop);
    if (n_groups == 0) return fail(1, "%s: no groups", what);
    if (beams == 0) return fail(1, "%s: beams is 0", what);
    if (n_stop > (unsigned long long)rk::kMaxTopN || beams + n_stop > (unsigned long long)rk::kMaxTopN)
        return fail(1, "%s: beams + n_stop = %u + %llu > %d", what, beams, n_stop, rk::kMaxTopN);
    if (n_best == 0 || n_best > beams) return fail(1, "%s: n_best %u is outside 1..beams = %u", what, n_best, beams);
    if (max_new == 0) return fail(1, "%s: max_new is 0", what);
    if (!std::isfinite(length_penalty)) return fail(1, "%s: length_penalty %g is not finite", what, length_penalty);
    if (n_groups > m->max_gpt) return fail(1, "%s: %llu groups > max_gpt %llu", what, n_groups, m->max_gpt);
    const size_t V = binfmt::kVocab;
    const unsigned long long G = n_groups, B = beams, K = n_best, N = max_new, C = B + n_stop;
    if ((rc = check_slots(m, what, slots, G * B)) || (rc = check_tokens(what, "first token", first_tokens, G, "group")) ||
        (rc = check_tokens(what, "stop token", stop_tokens, n_stop)))
        return rc;
    // the length penalties on the host, with the C library's pow: a host restatement gets the same bits
    if (N > ((unsigned long long)SIZE_MAX / sizeof(rk::BeamBack)) / (G * B))
        return fail(1, "%s: max_new = %llu: the backpointers of %llu beams do not fit in memory", what, N, G * B);
    std::vector<double> P;
    try {
        P.assign(N + 1, 0.0);
    } catch (const std::exception &) {
        return fail(9, "%s: out of host memory for max_new = %llu", what, N);
    }
    for (unsigned long long n = 1; n <= N; ++n) P[n] = pow((double)n, length_penalty);
    CK(cudaSetDevice(m->device));
    auto &g = m->gen;
    auto &bm = m->beam;
    if ((rc = g.stop.grow(n_stop)) || (rc = bm.row0.grow(G)) || (rc = bm.groups.grow(G)) || (rc = bm.cand_tok.grow(G * B * C)) ||
        (rc = bm.cand_lp.grow(G * B * C)) || (rc = bm.cum.grow(G * B)) || (rc = bm.P.grow(N + 1)) || (rc = bm.back.grow(G * N * B)) ||
        (rc = bm.hyp.grow(G * K)) || (rc = bm.n_hyp.grow(G)) || (rc = bm.done.grow(G)) || (rc = bm.forks.grow(2 * G * B)))
        return rc;
    // the path is chosen once, for G x B one-token streams
    const bool tc = tensor_cores(m, G * B);
    if (tc && (rc = rk::prefill_init(m->pf, m->p))) return fail(rc, "%s", rk::prefill_error());
    m->stream_rows = 0; // the compact logits rows no longer belong to a call the caller made

    rk::GenStream *hg = g.h_gs;
    for (unsigned long long s = 0; s < G * B; ++s) hg[s] = rk::GenStream{slots[s], N, s % B == 0 ? first_tokens[s / B] : 0, 0, 0};
    std::vector<int> row0(G), live(G);
    for (unsigned long long i = 0; i < G; ++i) {
        row0[i] = (int)(i * B);
        live[i] = (int)i;
    }
    CK(cudaMemcpyAsync(g.gs, hg, G * B * sizeof(rk::GenStream), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(bm.row0.p, row0.data(), G * sizeof(int), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(bm.P.p, P.data(), (N + 1) * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    if (n_stop) CK(cudaMemcpyAsync(g.stop.p, stop_tokens, n_stop * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemsetAsync(bm.cum.p, 0, G * B * sizeof(double), m->stream));
    CK(cudaMemsetAsync(bm.n_hyp.p, 0, G * sizeof(int), m->stream));
    CK(cudaMemsetAsync(bm.done.p, 0, G * sizeof(unsigned long long), m->stream));
    double *arr[5];
    slot_arrays(m, 0, arr);
    const size_t slot_len = (size_t)(m->L * m->E);
    const unsigned chunks = (unsigned)((slot_len + rk::kForkChunk - 1) / rk::kForkChunk);
    std::vector<unsigned long long> hdone(G, 0);
    std::vector<int> rs;
    for (unsigned long long step = 0; !live.empty() && step < N;) {
        // a host group: the live groups' beams are rows gi * B + j (step 0: row gi); their inputs go up once
        const int Gl = (int)live.size();
        const unsigned long long steps = std::min(kGenGroup, N - step);
        rs.resize((size_t)Gl * B);
        for (int gi = 0; gi < Gl; ++gi)
            for (unsigned long long j = 0; j < B; ++j) rs[gi * B + j] = (int)(live[gi] * B + j);
        CK(cudaMemcpyAsync(g.row_stream, rs.data(), rs.size() * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bm.groups.p, live.data(), Gl * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        if (tc && (rc = upload_step_passes(m, step == 0 ? row0.data() : rs.data(), step == 0 ? Gl : Gl * (int)B))) return rc;
        rk::BeamArgs ba{g.gs, bm.cum.p, bm.groups.p, bm.cand_tok.p, bm.cand_lp.p, (int)C, (int)B, (int)K, 0, 0, N, bm.P.p,
                        length_penalty < 0.0 ? 1 : 0, g.stop.p, (int)n_stop, bm.back.p, bm.hyp.p, bm.n_hyp.p, bm.done.p, bm.forks.p,
                        tc ? g.passes : nullptr};
        for (unsigned long long k = 0; k < steps; ++k) {
            const unsigned long long st = step + k;
            const int nb = st == 0 ? 1 : (int)B, rows = Gl * nb;
            const int *rmap = st == 0 ? bm.row0.p : g.row_stream;
            if ((rc = tc ? gen_step_passes(m, rows) : gen_step_decode(m, rows, rmap))) return rc;
            rk::k_beam_expand<<<(unsigned)rows, rk::kNucThreads, 0, m->stream>>>(m->d_slogits, (int)V, g.gs, rmap, (int)C,
                                                                                bm.cand_tok.p, bm.cand_lp.p);
            CK(cudaGetLastError());
            ba.step = (int)st;
            ba.nb = nb;
            rk::k_beam_select<<<(unsigned)Gl, rk::kBeamSelectThreads, 0, m->stream>>>(ba);
            CK(cudaGetLastError());
            m->launches += 2;
            if (st + 1 < N) { // after the last step every group is done and forks nothing
                rk::k_beam_fork<<<dim3((unsigned)(Gl * B), chunks, 5), rk::kForkThreads, 0, m->stream>>>(
                    bm.forks.p, arr[0], arr[1], arr[2], arr[3], arr[4], slot_len);
                CK(cudaGetLastError());
                m->launches += 1;
            }
        }
        // the end of a host group: which groups are done and the beams' records (one synchronisation)
        CK(cudaMemcpyAsync(hdone.data(), bm.done.p, G * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        CK(cudaMemcpyAsync(hg, g.gs, G * B * sizeof(rk::GenStream), cudaMemcpyDeviceToHost, m->stream));
        SYNC(m);
        step += steps;
        live.erase(std::remove_if(live.begin(), live.end(), [&](int gg) { return hdone[gg] != 0; }), live.end());
    }
    std::vector<rk::BeamHyp> hyp(G * K);
    std::vector<rk::BeamBack> back(G * N * B);
    CK(cudaMemcpyAsync(hyp.data(), bm.hyp.p, G * K * sizeof(rk::BeamHyp), cudaMemcpyDeviceToHost, m->stream));
    CK(cudaMemcpyAsync(back.data(), bm.back.p, G * N * B * sizeof(rk::BeamBack), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    // each hypothesis' tokens: its last token, then the backpointers of its beam from its step down to step 0
    const double nan = std::nan("");
    for (unsigned long long gg = 0; gg < G; ++gg)
        for (unsigned long long i = 0; i < K; ++i) {
            const rk::BeamHyp &h = hyp[gg * K + i];
            const size_t o = (size_t)(gg * K + i);
            unsigned long long *tok = tokens_out + o * N;
            double *tlp = token_logprobs_out ? token_logprobs_out + o * N : nullptr;
            for (unsigned long long t = 0; t < N; ++t) {
                tok[t] = 0;
                if (tlp) tlp[t] = nan;
            }
            tok[h.step] = h.tok;
            if (tlp) tlp[h.step] = h.lp;
            for (int s = h.step - 1, p = h.parent; s >= 0; --s) {
                const rk::BeamBack &bk = back[(gg * N + (unsigned long long)s) * B + (unsigned long long)p];
                tok[s] = bk.tok;
                if (tlp) tlp[s] = bk.lp;
                p = bk.parent;
            }
            lengths_out[o] = (unsigned long long)h.len;
            logprobs_out[o] = h.cum;
            scores_out[o] = h.score;
            finished_out[o] = (unsigned char)h.finished;
        }
    return 0;
}

} // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char *rwkv_b200_last_error(void) { return g_err.c_str(); }
int rwkv_b200_abi_version(void) { return 2; }

int rwkv_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int rwkv_b200_load_tp(const char *path, unsigned long long max_gpt, int device, int quiet, int tp_rank, int tp_size,
                      rwkv_b200_model **out, unsigned long long *n_layers, unsigned long long *n_embed) {
    if (!path || !out) return fail(1, "null argument");
    *out = nullptr;
    if (tp_size < 1 || tp_size > rk::kMaxRanks || tp_rank < 0 || tp_rank >= tp_size)
        return fail(7, "tensor parallelism: rank %d of %d is not supported (1..8 ranks)", tp_rank, tp_size);
    if (rwkv_b200_device_count() <= device || device < 0)
        return fail(6, "CUDA device %d not available (no CPU fallback exists)", device);
    M *m = new M;
    m->device = device;
    m->max_gpt = max_gpt ? max_gpt : 1;
    m->tp_rank = tp_rank;
    m->tp_size = tp_size;
    int rc = do_load(m, path, quiet);
    if (rc) {
        std::string keep = g_err;
        rwkv_b200_free(m);
        g_err = keep;
        return rc;
    }
    *out = m;
    if (n_layers) *n_layers = m->L;
    if (n_embed) *n_embed = m->E;
    return 0;
}

int rwkv_b200_load(const char *path, unsigned long long max_gpt, int device, int quiet, rwkv_b200_model **out,
                   unsigned long long *n_layers, unsigned long long *n_embed) {
    return rwkv_b200_load_tp(path, max_gpt, device, quiet, 0, 1, out, n_layers, n_embed);
}

void rwkv_b200_free(rwkv_b200_model *m) {
    if (!m) return;
    cudaSetDevice(m->device);
    if (m->stream) cudaStreamSynchronize(m->stream);
    rk::prefill_free(m->pf);
    for (void *p : m->ipc_opened) cudaIpcCloseMemHandle(p);
    for (void *p : m->allocs) cudaFree(p);
    if (m->h_ctrl) cudaFreeHost(m->h_ctrl);
    if (m->h_logits) cudaFreeHost(m->h_logits);
    if (m->h_next) cudaFreeHost(m->h_next);
    if (m->h_sample) cudaFreeHost(m->h_sample);
    if (m->h_diag) cudaFreeHost(m->h_diag);
    if (m->gen.h_gs) cudaFreeHost(m->gen.h_gs);
    if (m->stream) cudaStreamDestroy(m->stream);
    delete m; // frees the grow-only buffers and the automata
    cudaGetLastError(); // a context killed by a trap makes every call above fail; do not leave that as "last error"
}

void *rwkv_b200_tensor(rwkv_b200_model *m, int index) {
    if (!m || index < 0 || index >= RWKV_B200_NUM_TENSORS) return nullptr;
    return m->tensors[index];
}
unsigned long long rwkv_b200_n_layers(const rwkv_b200_model *m) { return m ? m->L : 0; }
unsigned long long rwkv_b200_n_embed(const rwkv_b200_model *m) { return m ? m->E : 0; }
unsigned long long rwkv_b200_max_gpt(const rwkv_b200_model *m) { return m ? m->max_gpt : 0; }

void *rwkv_b200_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (bytes == 0) bytes = 1;
    if (cudaMallocHost(&p, bytes) == cudaSuccess) return p;
    cudaGetLastError();
    // No driver (tokenizer-only use): tag the block so host_free knows it came from malloc.
    uint64_t *raw = (uint64_t *)malloc(bytes + 16);
    if (!raw) return nullptr;
    raw[0] = 0x6d616c6c6f636564ULL;
    return raw + 2;
}
void rwkv_b200_host_free(void *p) {
    if (!p) return;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeHost) {
        cudaFreeHost(p);
        return;
    }
    cudaGetLastError();
    uint64_t *raw = (uint64_t *)p - 2;
    if (raw[0] == 0x6d616c6c6f636564ULL) free(raw);
}

int rwkv_b200_state_upload(rwkv_b200_model *m, const double *xy, const double *aa, const double *bb,
                           const double *pp, const double *dd, unsigned long long slots) {
    int rc = check_model(m);
    if (rc) return rc;
    if (slots > m->max_gpt) return fail(1, "state_upload: %llu slots > max_gpt %llu", slots, m->max_gpt);
    CK(cudaSetDevice(m->device));
    const size_t n = (size_t)(m->L * m->E * slots) * sizeof(double);
    const double *src[5] = {xy, aa, bb, pp, dd};
    double *dst[5];
    slot_arrays(m, 0, dst);
    for (int i = 0; i < 5; ++i)
        if (src[i]) CK(cudaMemcpyAsync(dst[i], src[i], n, cudaMemcpyHostToDevice, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_state_download(rwkv_b200_model *m, double *xy, double *aa, double *bb, double *pp, double *dd,
                             unsigned long long slots) {
    int rc = check_model(m);
    if (rc) return rc;
    if (slots > m->max_gpt) return fail(1, "state_download: %llu slots > max_gpt %llu", slots, m->max_gpt);
    CK(cudaSetDevice(m->device));
    const size_t n = (size_t)(m->L * m->E * slots) * sizeof(double);
    double *dst[5] = {xy, aa, bb, pp, dd}, *src[5];
    slot_arrays(m, 0, src);
    for (int i = 0; i < 5; ++i)
        if (dst[i]) CK(cudaMemcpyAsync(dst[i], src[i], n, cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_state_zero(rwkv_b200_model *m) {
    int rc = check_model(m);
    if (rc) return rc;
    CK(cudaSetDevice(m->device));
    const size_t n = (size_t)(m->L * m->E * m->max_gpt) * sizeof(double);
    double *a[5];
    slot_arrays(m, 0, a);
    for (double *s : a) CK(cudaMemsetAsync(s, 0, n, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_forward(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n_tokens, int mode,
                      float *logits_out) {
    int rc = check_model(m);
    if (rc) return rc;
    if (!tokens || n_tokens == 0) return fail(1, "forward: no tokens");
    if (n_tokens > m->max_gpt) return fail(1, "Context too large, max context is %llu", m->max_gpt);
    CK(cudaSetDevice(m->device));
    const size_t V = binfmt::kVocab;
    for (unsigned long long t = 0; t < n_tokens; ++t)
        if (tokens[t] >= V) return fail(1, "token id %llu out of range", tokens[t]);
    m->stream_rows = 0;
    // GPT: one stream on slot 0; PARRALEL: n streams of one token on slots 0..n-1. Logits of every token.
    const bool par = mode == RWKV_B200_MODE_PARRALEL;
    std::vector<unsigned long long> slots(par ? n_tokens : 1), lens(par ? n_tokens : 1, par ? 1 : n_tokens);
    for (size_t i = 0; i < slots.size(); ++i) slots[i] = i;
    if (tensor_cores(m, n_tokens)) {
        if (par && n_tokens > (unsigned long long)rk::kPfMaxTokens)
            return fail(3, "batched prefill: PARRALEL chunks above 128 tokens are not supported");
        rc = rk::prefill_forward(m->pf, m->p, m->stream, tokens, (int)n_tokens, slots.data(), lens.data(), logits_out ? 1 : 0,
                                 m->d_slogits);
        if (rc) return fail(rc, "%s", rk::prefill_error());
        m->launches += rk::prefill_launches(m->pf);
        if (logits_out) CK(cudaMemcpyAsync(m->h_logits, m->d_slogits, n_tokens * V * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
    } else {
        // the logits of token t go to pinned row t
        const auto row = [&](unsigned long long t, unsigned long long, bool) { return logits_out ? m->h_logits + t * V : nullptr; };
        if ((rc = decode_tokens(m, tokens, slots.data(), lens.data(), slots.size(), cudaMemcpyDeviceToHost, row))) return rc;
    }
    SYNC(m);
    if (logits_out && logits_out != m->h_logits) memcpy(logits_out, m->h_logits, n_tokens * V * sizeof(float));
    return 0;
}

int rwkv_b200_forward_greedy(rwkv_b200_model *m, unsigned long long token, unsigned long long *next, float *logits_out) {
    int rc = check_model(m);
    if (rc) return rc;
    const size_t V = binfmt::kVocab;
    if (token >= V) return fail(1, "token id %llu out of range", token);
    CK(cudaSetDevice(m->device));
    m->stream_rows = 0;
    rk::Ctrl &c = m->h_ctrl[0];
    c.token = token;
    c.next = 0;
    c.slot = 0;
    c.pos = 0;
    CK(cudaMemcpyAsync(m->p.ctrl, &c, sizeof(rk::Ctrl), cudaMemcpyHostToDevice, m->stream));
    if ((rc = launch_token(m, 0, true, nullptr, m->stream))) return rc;
    CK(cudaMemcpyAsync(m->h_next, &m->p.ctrl->next, sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
    if (logits_out) CK(cudaMemcpyAsync(m->h_logits, dev_logits(m), V * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    if (next) *next = *m->h_next;
    if (logits_out && logits_out != m->h_logits) memcpy(logits_out, m->h_logits, V * sizeof(float));
    return 0;
}

float *rwkv_b200_logits_host(rwkv_b200_model *m) { return m ? m->h_logits : nullptr; }

int rwkv_b200_sample_typical(rwkv_b200_model *m, float temp, double u, unsigned long long *token, double *margin) {
    int rc = check_model(m);
    if (rc) return rc;
    if (!token) return fail(1, "null argument");
    CK(cudaSetDevice(m->device));
    CK(cudaMemcpyAsync(m->d_u, &u, sizeof(double), cudaMemcpyHostToDevice, m->stream));
    rk::k_sample_typical<<<1, rk::kSampleThreads, 0, m->stream>>>(dev_logits(m), 0, (int)binfmt::kVocab, sample_exponent(temp), m->d_u,
                                                                  m->d_sample);
    CK(cudaGetLastError());
    if ((rc = read_samples(m, 1, token, margin))) return rc;
    m->launches += 1;
    return 0;
}

int rwkv_b200_forward_streams(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n_tokens,
                              const unsigned long long *slots, const unsigned long long *lengths,
                              unsigned long long n_streams, float *logits_out, unsigned long long *next_out) {
    int rc = check_ragged(m, "forward_streams", tokens, n_tokens, slots, lengths, n_streams);
    if (rc) return rc;
    const size_t V = binfmt::kVocab;
    CK(cudaSetDevice(m->device));
    const bool head = logits_out || next_out;
    m->stream_rows = 0;
    if (tensor_cores(m, n_tokens)) {
        rc = rk::prefill_forward(m->pf, m->p, m->stream, tokens, (int)n_tokens, slots, lengths, head ? 2 : 0, m->d_slogits);
        if (rc) return fail(rc, "%s", rk::prefill_error());
        m->launches += rk::prefill_launches(m->pf);
    } else {
        // the last logits of a stream are copied into the compact buffer, so the arg-max and the sampler read the same
        // rows as after a batched pass
        const auto row = [&](unsigned long long, unsigned long long i, bool last) { return head && last ? m->d_slogits + i * V : nullptr; };
        if ((rc = decode_tokens(m, tokens, slots, lengths, n_streams, cudaMemcpyDeviceToDevice, row))) return rc;
    }
    if (next_out) {
        rk::k_argmax_rows<<<(unsigned)n_streams, rk::kArgmaxThreads, 0, m->stream>>>(m->d_slogits, (int)V, m->d_next);
        CK(cudaGetLastError());
        m->launches += 1;
        CK(cudaMemcpyAsync(m->h_next, m->d_next, n_streams * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
    }
    if (logits_out) CK(cudaMemcpyAsync(m->h_logits, m->d_slogits, n_streams * V * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    if (next_out) memcpy(next_out, m->h_next, n_streams * sizeof(unsigned long long));
    if (logits_out && logits_out != m->h_logits) memcpy(logits_out, m->h_logits, n_streams * V * sizeof(float));
    m->stream_rows = head ? n_streams : 0;
    return 0;
}

int rwkv_b200_sample_typical_streams(rwkv_b200_model *m, unsigned long long n_streams, float temp, const double *u,
                                     unsigned long long *tokens_out, double *margins_out) {
    int rc = check_streams_model(m, "sample_typical_streams");
    if (rc) return rc;
    if (!u || !tokens_out) return fail(1, "sample_typical_streams: null argument");
    if (m->stream_rows == 0) return fail(1, "sample_typical_streams: the last forward produced no per-stream logits (call forward_streams with logits or next)");
    if (n_streams != m->stream_rows)
        return fail(1, "sample_typical_streams: %llu rows asked, the last forward_streams produced %llu", n_streams, m->stream_rows);
    CK(cudaSetDevice(m->device));
    CK(cudaMemcpyAsync(m->d_u, u, n_streams * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    rk::k_sample_typical<<<(unsigned)n_streams, rk::kSampleThreads, 0, m->stream>>>(m->d_slogits, binfmt::kVocab, (int)binfmt::kVocab,
                                                                                   sample_exponent(temp), m->d_u, m->d_sample);
    CK(cudaGetLastError());
    if ((rc = read_samples(m, n_streams, tokens_out, margins_out))) return rc;
    m->launches += 1;
    return 0;
}

int rwkv_b200_generate_streams(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                               unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                               const unsigned long long *stop_tokens, unsigned long long n_stop,
                               const unsigned long long *override_tokens, const float *override_values,
                               unsigned long long n_override, float temp, const double *u, unsigned long long *tokens_out,
                               unsigned long long *lengths_out) {
    return generate(m, "generate_streams", false, slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop,
                    override_tokens, override_values, n_override, temp, nullptr, u, tokens_out, lengths_out);
}

int rwkv_b200_generate_streams_ex(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                  unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                  const unsigned long long *stop_tokens, unsigned long long n_stop,
                                  const unsigned long long *override_tokens, const float *override_values,
                                  unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                  unsigned long long *tokens_out, unsigned long long *lengths_out) {
    // without samplers every stream takes the arg-max and u is not read
    return generate(m, "generate_streams_ex", true, slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop,
                    override_tokens, override_values, n_override, 1.0f, samplers, samplers ? u : nullptr, tokens_out, lengths_out);
}

int rwkv_b200_generate_streams_logprobs(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                        unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                        const unsigned long long *stop_tokens, unsigned long long n_stop,
                                        const unsigned long long *override_tokens, const float *override_values,
                                        unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                        unsigned long long *tokens_out, unsigned long long *lengths_out, int logprob_mode,
                                        unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
                                        unsigned long long *top_tokens_out, double *top_logprobs_out) {
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    return generate(m, "generate_streams_logprobs", true, slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop,
                    override_tokens, override_values, n_override, 1.0f, samplers, samplers ? u : nullptr, tokens_out, lengths_out,
                    &lpq);
}

int rwkv_b200_constraint_add(rwkv_b200_model *m, unsigned long long n_states, const unsigned long long *edge_start,
                             const unsigned long long *edge_tokens, const unsigned long long *edge_next, unsigned long long *id) {
    const char *what = "constraint_add";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!edge_start || !id) return fail(1, "%s: null argument (edge_start and id are required)", what);
    if (n_states == 0 || n_states > RWKV_B200_MAX_CONSTRAINT_STATES)
        return fail(1, "%s: n_states = %llu is outside 1..%d", what, n_states, RWKV_B200_MAX_CONSTRAINT_STATES);
    if (edge_start[0] != 0) return fail(1, "%s: edge_start[0] = %llu, not 0", what, edge_start[0]);
    for (unsigned long long q = 0; q < n_states; ++q)
        if (edge_start[q + 1] < edge_start[q])
            return fail(1, "%s: edge_start decreases from state %llu to %llu (%llu > %llu)", what, q, q + 1, edge_start[q],
                        edge_start[q + 1]);
    const unsigned long long n_edges = edge_start[n_states];
    if (n_edges && (!edge_tokens || !edge_next)) return fail(1, "%s: %llu edges with NULL edge_tokens or edge_next", what, n_edges);
    for (unsigned long long q = 0; q < n_states; ++q)
        for (unsigned long long e = edge_start[q]; e < edge_start[q + 1]; ++e) {
            if (edge_tokens[e] >= binfmt::kVocab)
                return fail(1, "%s: state %llu: edge token %llu out of range", what, q, edge_tokens[e]);
            if (e > edge_start[q] && edge_tokens[e] <= edge_tokens[e - 1])
                return fail(1, "%s: state %llu: edge tokens are not strictly ascending (%llu after %llu)", what, q, edge_tokens[e],
                            edge_tokens[e - 1]);
            if (edge_next[e] >= n_states)
                return fail(1, "%s: state %llu: edge of token %llu leads to state %llu >= n_states %llu", what, q, edge_tokens[e],
                            edge_next[e], n_states);
        }
    // one block: the allow masks [n_states][kMaskWords] u32, edge_start [n_states + 1] u64, tokens and targets [n_edges] u32
    const size_t mask_bytes = (size_t)n_states * rk::kMaskWords * 4, start_bytes = (size_t)(n_states + 1) * 8;
    const size_t bytes = mask_bytes + start_bytes + (size_t)n_edges * 8;
    M::Automaton a;
    std::vector<unsigned char> blob;
    try {
        blob.assign(bytes, 0);
        a.start.assign(edge_start, edge_start + n_states + 1);
        a.tok.resize(n_edges);
    } catch (const std::bad_alloc &) {
        return fail(9, "%s: out of host memory for %llu states and %llu edges", what, n_states, n_edges);
    }
    uint32_t *mask = (uint32_t *)blob.data(), *tok = (uint32_t *)(blob.data() + mask_bytes + start_bytes), *next = tok + n_edges;
    memcpy(blob.data() + mask_bytes, edge_start, start_bytes);
    for (unsigned long long q = 0; q < n_states; ++q)
        for (unsigned long long e = edge_start[q]; e < edge_start[q + 1]; ++e) {
            const uint32_t t = (uint32_t)edge_tokens[e];
            mask[q * rk::kMaskWords + (t >> 5)] |= 1u << (t & 31);
            tok[e] = a.tok[e] = t;
            next[e] = (uint32_t)edge_next[e];
        }
    CK(cudaSetDevice(m->device));
    if ((rc = a.dev.grow(bytes))) return rc;
    const cudaError_t e = cudaMemcpy(a.dev.p, blob.data(), bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return fail(100 + (int)e, "%s: upload failed: %s", what, cudaGetErrorString(e));
    const unsigned char *d = a.dev.p;
    a.view = rk::GenConstraint{(const unsigned long long *)(d + mask_bytes), (const uint32_t *)(d + mask_bytes + start_bytes),
                               (const uint32_t *)(d + mask_bytes + start_bytes) + n_edges, (const uint32_t *)d, 0};
    *id = m->next_automaton++;
    m->automata.emplace(*id, std::move(a));
    return 0;
}

int rwkv_b200_constraint_remove(rwkv_b200_model *m, unsigned long long id) {
    int rc = check_model(m);
    if (rc) return rc;
    const auto it = m->automata.find(id);
    if (it == m->automata.end()) return fail(1, "constraint_remove: constraint id %llu is unknown or removed", id);
    CK(cudaSetDevice(m->device));
    m->automata.erase(it);
    return 0;
}

int rwkv_b200_generate_streams_constrained(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                           unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                           const unsigned long long *stop_tokens, unsigned long long n_stop,
                                           const unsigned long long *override_tokens, const float *override_values,
                                           unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                           unsigned long long *tokens_out, unsigned long long *lengths_out, int logprob_mode,
                                           unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
                                           unsigned long long *top_tokens_out, double *top_logprobs_out,
                                           const unsigned long long *constraint_ids, const unsigned long long *start_states,
                                           unsigned long long *states_out) {
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    const ConstraintRequest cq{constraint_ids, start_states, states_out};
    return generate(m, "generate_streams_constrained", true, slots, first_tokens, n_streams, max_new, budgets, stop_tokens,
                    n_stop, override_tokens, override_values, n_override, 1.0f, samplers, samplers ? u : nullptr, tokens_out,
                    lengths_out, logprobs_out ? &lpq : nullptr, &cq);
}

int rwkv_b200_beam_search(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                          unsigned long long n_groups, unsigned beams, unsigned long long max_new,
                          const unsigned long long *stop_tokens, unsigned long long n_stop, double length_penalty,
                          unsigned n_best, unsigned long long *tokens_out, unsigned long long *lengths_out,
                          double *logprobs_out, double *scores_out, unsigned char *finished_out,
                          double *token_logprobs_out) {
    return beam(m, slots, first_tokens, n_groups, beams, max_new, stop_tokens, n_stop, length_penalty, n_best, tokens_out,
                lengths_out, logprobs_out, scores_out, finished_out, token_logprobs_out);
}

int rwkv_b200_sample_streams(rwkv_b200_model *m, unsigned long long n_streams, const rwkv_b200_sampler *params, const double *u,
                             const float *logits, unsigned long long *tokens_out, double *margins_out) {
    const char *what = "sample_streams";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!params || !tokens_out) return fail(1, "%s: null argument (params and tokens_out are required)", what);
    if (n_streams == 0) return fail(1, "%s: no streams", what);
    const size_t V = binfmt::kVocab;
    if (logits) {
        if (n_streams > m->max_gpt) return fail(1, "%s: %llu rows of logits > max_gpt %llu", what, n_streams, m->max_gpt);
    } else {
        if (m->stream_rows == 0)
            return fail(1, "%s: the last forward produced no per-stream logits (call forward_streams with logits or next, or pass logits)", what);
        if (n_streams != m->stream_rows)
            return fail(1, "%s: %llu rows asked, the last forward_streams produced %llu", what, n_streams, m->stream_rows);
    }
    for (unsigned long long s = 0; s < n_streams; ++s) {
        if ((rc = check_sampler(what, s, params[s], false))) return rc;
        if (params[s].temperature > 0.0f && !u)
            return fail(1, "%s: u is NULL but stream %llu samples (temperature %g)", what, s, params[s].temperature);
        if (u && !(u[s] >= 0.0 && u[s] < 1.0)) return fail(1, "%s: u[%llu] = %g is outside [0, 1)", what, s, u[s]);
    }
    for (unsigned long long s = 0; logits && s < n_streams; ++s) {
        const float *row = logits + s * V;
        bool finite = false;
        for (size_t v = 0; v < V; ++v) {
            if (std::isnan(row[v]) || row[v] == INFINITY)
                return fail(1, "%s: logits[%llu][%zu] = %g (NaN and +inf are not allowed)", what, s, v, row[v]);
            finite |= std::isfinite(row[v]);
        }
        if (!finite) return fail(1, "%s: row %llu of the logits has no finite value", what, s);
    }
    CK(cudaSetDevice(m->device));
    auto &g = m->gen;
    if ((rc = g.samp.grow(n_streams))) return rc;
    CK(cudaMemcpyAsync(g.samp.p, params, n_streams * sizeof(rwkv_b200_sampler), cudaMemcpyHostToDevice, m->stream));
    if (u) CK(cudaMemcpyAsync(m->d_u, u, n_streams * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    if (logits) {
        m->stream_rows = 0; // the compact rows now hold the caller's logits, not those of the last forward_streams
        CK(cudaMemcpyAsync(m->d_slogits, logits, n_streams * V * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    }
    rk::k_sample_nucleus<<<(unsigned)n_streams, rk::kNucThreads, 0, m->stream>>>(m->d_slogits, (int)V, g.samp.p, nullptr,
                                                                                u ? m->d_u : nullptr, m->d_sample);
    CK(cudaGetLastError());
    if ((rc = read_samples(m, n_streams, tokens_out, margins_out))) return rc;
    m->launches += 1;
    return 0;
}

int rwkv_b200_score_streams(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n_tokens,
                            const unsigned long long *slots, const unsigned long long *lengths, unsigned long long n_streams,
                            const unsigned long long *targets, unsigned int top_n, double *logprobs_out,
                            unsigned long long *ranks_out, unsigned long long *top_tokens_out, double *top_logprobs_out) {
    const char *what = "score_streams";
    int rc = check_ragged(m, what, tokens, n_tokens, slots, lengths, n_streams);
    if (rc) return rc;
    if (!targets) return fail(1, "%s: targets is NULL (RWKV_B200_NO_TARGET marks a position that is not scored)", what);
    if (!logprobs_out) return fail(1, "%s: logprobs_out is NULL", what);
    if (top_n > (unsigned)rk::kMaxTopN) return fail(1, "%s: top_n %u > %d", what, top_n, rk::kMaxTopN);
    if (top_n && (!top_tokens_out || !top_logprobs_out))
        return fail(1, "%s: top_n = %u needs top_tokens_out and top_logprobs_out", what, top_n);
    const size_t V = binfmt::kVocab;
    // the scored positions: row j of the results is position pos[j], whose logits are row pos[j] of d_slogits
    std::vector<int> pos;
    std::vector<unsigned long long> tgt;
    std::vector<unsigned char> need(n_tokens, 0);
    for (unsigned long long i = 0, t = 0; i < n_streams; ++i)
        for (unsigned long long k = 0; k < lengths[i]; ++k, ++t) {
            if (targets[t] == RWKV_B200_NO_TARGET) continue;
            if (targets[t] >= V)
                return fail(1, "%s: targets[%llu] = %llu (stream %llu, position %llu) is neither a token id < %zu nor RWKV_B200_NO_TARGET",
                            what, t, targets[t], i, k, V);
            pos.push_back((int)t);
            tgt.push_back(targets[t]);
            need[t] = 1;
        }
    const size_t n = pos.size();
    CK(cudaSetDevice(m->device));
    m->stream_rows = 0; // the compact rows hold this call's scored positions, not per-stream logits
    auto &sc = m->score;
    if (n && ((rc = sc.rows.grow(n)) || (rc = sc.tgt.grow(n)) || (rc = sc.lp.grow(n)) || (rc = sc.rank.grow(n)) ||
              (rc = sc.top_tok.grow(n * top_n)) || (rc = sc.top_lp.grow(n * top_n))))
        return rc;
    if (tensor_cores(m, n_tokens)) {
        // logits of every token of a pass that holds a scored position, row t of d_slogits for token t
        rc = rk::prefill_forward(m->pf, m->p, m->stream, tokens, (int)n_tokens, slots, lengths, n ? 1 : 0, m->d_slogits, need.data());
        if (rc) return fail(rc, "%s", rk::prefill_error());
        m->launches += rk::prefill_launches(m->pf);
    } else {
        // a scored position's logits are copied into row t of d_slogits
        const auto row = [&](unsigned long long t, unsigned long long, bool) { return need[t] ? m->d_slogits + t * V : nullptr; };
        if ((rc = decode_tokens(m, tokens, slots, lengths, n_streams, cudaMemcpyDeviceToDevice, row))) return rc;
    }
    std::vector<double> lp(n), top_lp(n * top_n);
    std::vector<unsigned long long> rank(n), top_tok(n * top_n);
    if (n) {
        CK(cudaMemcpyAsync(sc.rows.p, pos.data(), n * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(sc.tgt.p, tgt.data(), n * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
        const rk::ScoreArgs a{m->d_slogits, (int)V, sc.rows.p, sc.tgt.p, (int)top_n, sc.lp.p, sc.rank.p, sc.top_tok.p, sc.top_lp.p};
        rk::k_logprob_rows<<<(unsigned)n, rk::kNucThreads, 0, m->stream>>>(a);
        CK(cudaGetLastError());
        m->launches += 1;
        CK(cudaMemcpyAsync(lp.data(), sc.lp.p, n * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        if (ranks_out) CK(cudaMemcpyAsync(rank.data(), sc.rank.p, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        if (top_n) {
            CK(cudaMemcpyAsync(top_tok.data(), sc.top_tok.p, n * top_n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
            CK(cudaMemcpyAsync(top_lp.data(), sc.top_lp.p, n * top_n * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        }
    }
    SYNC(m);
    const double nan = std::nan("");
    for (unsigned long long t = 0; t < n_tokens; ++t) {
        logprobs_out[t] = nan;
        if (ranks_out) ranks_out[t] = RWKV_B200_NO_TARGET;
        for (unsigned k = 0; k < top_n; ++k) {
            top_tokens_out[t * top_n + k] = RWKV_B200_NO_TARGET;
            top_logprobs_out[t * top_n + k] = nan;
        }
    }
    for (size_t j = 0; j < n; ++j) {
        const size_t t = (size_t)pos[j];
        logprobs_out[t] = lp[j];
        if (ranks_out) ranks_out[t] = rank[j];
        for (unsigned k = 0; k < top_n; ++k) {
            top_tokens_out[t * top_n + k] = top_tok[j * top_n + k];
            top_logprobs_out[t * top_n + k] = top_lp[j * top_n + k];
        }
    }
    return 0;
}

int rwkv_b200_slot_zero(rwkv_b200_model *m, unsigned long long slot) {
    int rc = check_streams_model(m, "slot_zero");
    if (rc || (rc = check_slot(m, "slot_zero", slot))) return rc;
    CK(cudaSetDevice(m->device));
    double *a[5];
    slot_arrays(m, slot, a);
    for (double *p : a) CK(cudaMemsetAsync(p, 0, (size_t)(m->L * m->E) * sizeof(double), m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_slot_copy(rwkv_b200_model *m, unsigned long long src, unsigned long long dst) {
    int rc = check_streams_model(m, "slot_copy");
    if (rc || (rc = check_slot(m, "slot_copy", src)) || (rc = check_slot(m, "slot_copy", dst))) return rc;
    if (src == dst) return 0;
    CK(cudaSetDevice(m->device));
    double *a[5], *b[5];
    slot_arrays(m, src, a);
    slot_arrays(m, dst, b);
    for (int i = 0; i < 5; ++i) CK(cudaMemcpyAsync(b[i], a[i], (size_t)(m->L * m->E) * sizeof(double), cudaMemcpyDeviceToDevice, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_slot_upload(rwkv_b200_model *m, unsigned long long slot, const double *xy, const double *aa, const double *bb,
                          const double *pp, const double *dd) {
    int rc = check_streams_model(m, "slot_upload");
    if (rc || (rc = check_slot(m, "slot_upload", slot))) return rc;
    CK(cudaSetDevice(m->device));
    double *a[5];
    slot_arrays(m, slot, a);
    const double *src[5] = {xy, aa, bb, pp, dd};
    for (int i = 0; i < 5; ++i)
        if (src[i]) CK(cudaMemcpyAsync(a[i], src[i], (size_t)(m->L * m->E) * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_slot_download(rwkv_b200_model *m, unsigned long long slot, double *xy, double *aa, double *bb, double *pp, double *dd) {
    int rc = check_streams_model(m, "slot_download");
    if (rc || (rc = check_slot(m, "slot_download", slot))) return rc;
    CK(cudaSetDevice(m->device));
    double *a[5];
    slot_arrays(m, slot, a);
    double *dst[5] = {xy, aa, bb, pp, dd};
    for (int i = 0; i < 5; ++i)
        if (dst[i]) CK(cudaMemcpyAsync(dst[i], a[i], (size_t)(m->L * m->E) * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_decode_timed(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n,
                           int teacher_forced, float *ms) {
    int rc = check_model(m);
    if (rc) return rc;
    if (!tokens || n == 0 || !ms) return fail(1, "decode_timed: bad arguments");
    CK(cudaSetDevice(m->device));
    const unsigned long long cnt = teacher_forced ? n : 1;
    for (unsigned long long i = 0; i < cnt; ++i)
        if (tokens[i] >= binfmt::kVocab) return fail(1, "token id %llu out of range", tokens[i]);
    unsigned long long *d_tok = nullptr;
    cudaEvent_t a = nullptr, b = nullptr;
    cudaError_t e = cudaMalloc((void **)&d_tok, cnt * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemcpy(d_tok, tokens, cnt * sizeof(unsigned long long), cudaMemcpyHostToDevice);
    rk::Ctrl c{tokens[0], tokens[0], 0, 0};
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e == cudaSuccess) e = cudaMemcpy(m->p.ctrl, &c, sizeof(rk::Ctrl), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaEventCreate(&a);
    if (e == cudaSuccess) e = cudaEventCreate(&b);
    if (e == cudaSuccess) e = cudaEventRecord(a, m->stream);
    rc = 0;
    for (unsigned long long i = 0; i < n && e == cudaSuccess && rc == 0; ++i)
        rc = launch_token(m, teacher_forced ? 2 : 1, !teacher_forced, d_tok, m->stream);
    if (e == cudaSuccess && rc == 0) e = cudaEventRecord(b, m->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
    if (e == cudaSuccess && rc == 0) e = cudaEventElapsedTime(ms, a, b);
    if (a) cudaEventDestroy(a);
    if (b) cudaEventDestroy(b);
    if (d_tok) cudaFree(d_tok);
    if (rc) return rc;
    if (e != cudaSuccess) return sync_failed(m, e, "decode_timed");
    return 0;
}

int rwkv_b200_kernel_count(void) { return 1; }
const char *rwkv_b200_kernel_name(int k) { return k == 0 ? kKernelNames[0] : ""; }

int rwkv_b200_profile(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n, float *ms_sum,
                      unsigned long long *launches, double *bytes) {
    int rc = check_model(m);
    if (rc) return rc;
    if (!tokens || !ms_sum || !launches || !bytes) return fail(1, "profile: bad arguments");
    CK(cudaSetDevice(m->device));
    ms_sum[0] = 0.f;
    launches[0] = 0;
    // algorithmic HBM bytes of one launch on this rank: its share of the weights + the vectors
    const double E = (double)m->E, V = (double)binfmt::kVocab, L = (double)m->L, G = (double)m->tp_size;
    bytes[0] = (13.0 * L * E * E + V * E) / G + ((double)binfmt::algorithmic_bytes_per_token(m->L, m->E) - (13.0 * L * E * E + V * E));
    cudaEvent_t a = nullptr, b = nullptr;
    CK(cudaEventCreate(&a));
    cudaError_t e = cudaEventCreate(&b);
    rc = 0;
    for (unsigned long long t = 0; t < n && e == cudaSuccess && rc == 0; ++t) {
        if (tokens[t] >= binfmt::kVocab) {
            rc = fail(1, "token id out of range");
            break;
        }
        rk::Ctrl c{tokens[t], 0, 0, 0};
        e = cudaMemcpyAsync(m->p.ctrl, &c, sizeof(rk::Ctrl), cudaMemcpyHostToDevice, m->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
        if (e == cudaSuccess) e = cudaEventRecord(a, m->stream);
        if (e == cudaSuccess) rc = launch_token(m, 0, true, nullptr, m->stream);
        if (e == cudaSuccess && rc == 0) e = cudaEventRecord(b, m->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
        float t_ms = 0.f;
        if (e == cudaSuccess && rc == 0) e = cudaEventElapsedTime(&t_ms, a, b);
        ms_sum[0] += t_ms;
        launches[0] += 1;
    }
    cudaEventDestroy(a);
    if (b) cudaEventDestroy(b);
    if (rc) return rc;
    if (e != cudaSuccess) return sync_failed(m, e, "profile");
    return 0;
}

unsigned long long rwkv_b200_launch_count(const rwkv_b200_model *m) { return m ? m->launches : 0; }

int rwkv_b200_set_option(rwkv_b200_model *m, const char *key, const char *value) {
    int rc = check_model(m);
    if (rc) return rc;
    if (!key || !value) return fail(1, "set_option: null");
    const std::string k = key;
    const int v = atoi(value);
    if (k == "trace") {
        if (v && !m->p.trace) {
            unsigned long long *t = nullptr;
            if (dmalloc(m, &t, (size_t)rk::kMaxGrid * rk::kTraceMax)) return fail(1, "trace alloc failed");
            cudaMemset(t, 0, (size_t)rk::kMaxGrid * rk::kTraceMax * 8);
            m->p.trace = t;
            unsigned long long *pt = nullptr;
            if (dmalloc(m, &pt, (size_t)2 * rk::kMaxGrid * rk::kTileTraceMax)) return fail(1, "trace alloc failed");
            cudaMemset(pt, 0, (size_t)2 * rk::kMaxGrid * rk::kTileTraceMax * 8);
            m->p.ptrace = pt;
        } else if (!v) {
            m->p.trace = nullptr;
            m->p.ptrace = nullptr;
        }
    } else if (k == "max_layers") m->max_layers = v;
    else if (k == "issue_gap") {
        if (v < 0 || v > 100000) return fail(1, "issue_gap is a cycle count in 0..100000");
        m->p.issue_gap = v;
    } else if (k == "window") {
        if (v < 1 || v > rk::kMaxStages) return fail(1, "window must be 1..%d", rk::kMaxStages);
        m->p.window = v;
    } else if (k == "cluster" || k == "grid") {
        const int c = k == "cluster" ? v : m->p.cluster, g = k == "grid" ? v : m->grid;
        if (int rc2 = check_grid(m, g, c)) return rc2;
        m->p.cluster = c;
        m->grid = g;
    } else if (k == "bwindow") {
        if (v < 1 || v > rk::kMaxStages) return fail(1, "bwindow must be 1..%d", rk::kMaxStages);
        m->p.bwindow = v;
    } else if (k == "pf_dist") {
        if (v < 0 || v > 64) return fail(1, "pf_dist is 0..64 tiles");
        m->p.pf_dist = v;
    } else if (k == "poll_first") {
        if (v < 0 || v > 2) return fail(1, "poll_first is 0, 1 or 2");
        m->p.poll_first = v;
    } else if (k == "dbg") {
        m->p.dbg = v;
    } else if (k == "timeout_ms") {
        if (v < 1) return fail(1, "timeout_ms must be positive");
        m->p.timeout_ms = (unsigned int)v;
    } else if (k == "stages") {
        if (v < 2 || v > rk::kMaxStages) return fail(1, "stages must be 2..%d", rk::kMaxStages);
        const size_t smem = rk::smem_bytes(v, m->p.tile_bytes, m->p.plane_cap);
        if (smem > (size_t)rk::kSmemLimit) return fail(1, "stages=%d needs %zu bytes of shared memory", v, smem);
        m->p.stages = v;
        m->smem = smem;
    } else if (k == "prefill") {
        m->pf.disabled = v == 0;
    } else if (k == "prefill_graph") {
        m->pf.use_graph = v != 0;
    } else if (k == "prefill_min") {
        if (v < 2) return fail(1, "prefill_min must be >= 2");
        m->pf.min_tokens = v;
    } else return fail(1, "unknown option '%s'", key);
    return 0;
}

// Debug/test hook: copy a named device vector to the host. Returns the element count.
long long rwkv_b200_debug_read(rwkv_b200_model *m, const char *name, void *dst, size_t dst_bytes) {
    if (check_model(m) || !name || !dst) return -1;
    cudaSetDevice(m->device);
    const std::string k = name;
    const void *src = nullptr;
    size_t bytes = 0, count = 0;
    const size_t E = m->E;
    if (k == "x") src = m->p.x, count = E, bytes = E * 8;
    else if (k == "logits") src = dev_logits(m), count = binfmt::kVocab, bytes = 4 * binfmt::kVocab;
    else if (k == "trace" && m->p.trace) src = m->p.trace, count = (size_t)m->grid * rk::kTraceMax, bytes = count * 8;
    else if (k == "ptrace" && m->p.ptrace) src = m->p.ptrace, count = (size_t)2 * m->grid * rk::kTileTraceMax, bytes = count * 8;
    else return -1;
    if (dst_bytes < bytes) return -1;
    if (cudaStreamSynchronize(m->stream) != cudaSuccess) return -1;
    if (cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (long long)count;
}

size_t rwkv_b200_tp_buffer_bytes(const rwkv_b200_model *m) { return m ? m->xch_bytes : 0; }

int rwkv_b200_tp_export(rwkv_b200_model *m, void *ipc_handle_64) {
    if (check_model(m) || !ipc_handle_64) return fail(1, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaSetDevice(m->device);
    CK(cudaStreamSynchronize(m->stream)); // the block is zero-filled before anybody maps it
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, m->p.xch[m->tp_rank]));
    memcpy(ipc_handle_64, &h, 64);
    return 0;
}

int rwkv_b200_tp_import(rwkv_b200_model *m, const void *ipc_handles) {
    if (check_model(m) || !ipc_handles) return fail(1, "null argument");
    if (m->tp_wired) return fail(7, "peer exchange blocks already imported");
    cudaSetDevice(m->device);
    const unsigned char *hs = static_cast<const unsigned char *>(ipc_handles);
    for (int g = 0; g < m->tp_size; ++g) {
        if (g == m->tp_rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, hs + 64 * (size_t)g, 64);
        void *ptr = nullptr;
        CK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        m->ipc_opened.push_back(ptr);
        m->p.xch[g] = static_cast<unsigned char *>(ptr);
    }
    m->tp_wired = true;
    return 0;
}

} // extern "C"
