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
#include <deque>
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
#include "index.cuh"
#include "prefill.cuh"
#include "prefix.cuh"
#include "prefix_index.h"
#include "sampling.cuh"
#include "score.cuh"
#include "speculate.cuh"
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

// The device buffers of a decode group (step_args, run_step): the model keeps one set for the one-shot generation calls
// and the batcher its own, so a call between runs leaves the batcher's requests alone. Each grows with its largest
// user; what a buffer holds is counted in streams (the one-shot calls) or lanes (the batcher).
struct StepBuffers {
    DevBuf<rk::GenStream> gs;          // stream records (the model's are sized at load)
    DevBuf<int> row_stream;            // [rows] the stream of each logits row (the model's are sized at load)
    DevBuf<rk::PassDesc> passes;       // the steps' passes (the model's: [ceil(max_gpt / 128)], zeroed at load)
    DevBuf<double> u;                  // [steps][rows] each row's uniform of a group's steps
    DevBuf<rwkv_b200_sampler> samp;    // [streams] each stream's sampler
    DevBuf<float> pen_cnt;             // [streams][V] decayed counts of the emitted tokens (penalties only)
    DevBuf<unsigned char> pen_seen;    // [streams][V] emitted in this call or request
    DevBuf<unsigned long long> out;    // [streams][max_new] emitted tokens (the batcher's: a ring per lane)
    // stop tokens and overrides: the call's lists, or each lane's by its CSR start ([lanes + 1]; the batcher only)
    DevBuf<unsigned long long> stop, stop_start, ovr_tok, ovr_start;
    DevBuf<float> ovr_val;
    DevBuf<rk::GenConstraint> gc;      // [streams] token automata
    DevBuf<unsigned long long> fault;  // [3] k_gen_feedback's and k_spec_accept's record of a token without an edge
    DevBuf<rk::GenStop> gst;           // [streams] stop sets
    // log-probabilities: the results of each emitted token, each lane's scoring (the batcher only), and the model's rows
    // of a step (raw mode with penalties, overrides or automata, which edit d_slogits in place)
    DevBuf<double> lp, top_lp;         // [streams][max_new], [..][top]
    DevBuf<unsigned long long> rank, top_tok;
    DevBuf<rk::LogprobLane> lp_lane;   // [lanes]
    DevBuf<float> raw;                 // [rows][V]
    // speculative streams: records, the live list, what k_spec_logprob scores ([rows]), histories, each row's automaton
    // state ([rows]), the copies home -> first slot ([streams][2]) and the streams' uniforms (SpecArgs::u)
    DevBuf<rk::SpecStream> ss;
    DevBuf<rk::SpecLive> live;
    DevBuf<rk::SpecScore> score;
    DevBuf<unsigned long long> hist, row_state, forks;
    DevBuf<double> su;
    DevBuf<rk::GenGuide> guide;        // [rows] each guided row's conditional row and scale (generate_streams_guided)
    DevBuf<rk::SpecDraft> ds;          // [streams] a draft model's records of a drafted call (generate_streams_drafted)
};

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
    unsigned long long launches = 0;
    unsigned int epoch = 0, tk = 0; // exchange epochs (token_kernel.cuh); identical on every rank
    int tp_rank = 0, tp_size = 1;
    rk::PrefillState pf{};
    // the one-shot generation calls (generate_streams*, generate_streams_speculative*, beam_search) and sample_streams:
    // the stream records (device, and their pinned host mirror [max_gpt]), the row map and the passes are sized at
    // load; the rest grows with the largest call and is freed with the model
    StepBuffers gen;
    rk::GenStream *h_gs = nullptr;
    // the speculative call's passes, sized by its own rule (streams of k + 1 rows never straddle a pass), so apart from
    // gen.passes, which must stay zeroed from load
    DevBuf<rk::PassDesc> spec_passes;
    // stop strings: the token bytes (rwkv_b200_token_bytes_set) and per set id its automaton (rwkv_b200_stop_set_add):
    // next [states][256] then hit [states] in one device block
    DevBuf<unsigned long long> tb_start; // [V + 1]
    DevBuf<unsigned char> tb_bytes;
    bool has_tb = false;
    struct StopSet {
        unsigned long long states = 0;
        DevBuf<uint32_t> dev;
    };
    std::map<unsigned long long, StopSet> stop_sets;
    unsigned long long next_stop_set = 1;
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
    rwkv_b200_batcher *batcher = nullptr; // the open batcher (at most one), closed by rwkv_b200_free
    // rwkv_b200_index_create: per id the rows [capacity][D] and live flags on the device, the flags and counts on the host
    struct Index {
        unsigned long long lb = 0, nl = 0, D = 0, capacity = 0, count = 0, live = 0;
        std::vector<unsigned char> alive; // [count]
        DevBuf<double> rows;
        DevBuf<unsigned char> d_alive;    // [capacity]
    };
    std::map<unsigned long long, Index> indexes;
    unsigned long long next_index = 1;
    // rwkv_b200_index_search: grown with the largest call
    struct IndexScratch {
        DevBuf<double> partial, l1, l2;            // [QB][block][G][2], [QB][count], [QB][count]
        DevBuf<unsigned long long> key[2], id[2];  // the selection's survivors, ping-pong
        DevBuf<unsigned long long> ent;            // [QB][k]
        DevBuf<double> o1, o2;                     // [QB][k]
    } isc;
    // rwkv_b200_adapter_add: per id its matrices in one device block and the record the passes read; per slot the bound
    // id (RWKV_B200_NO_ADAPTER: none; empty until the first binding) and, on the device, the bound record (rank 0: none)
    struct Adapter {
        DevBuf<float> data;
        rk::AdapterRec rec{};
    };
    std::map<unsigned long long, Adapter> adapters;
    unsigned long long next_adapter = 1;
    std::vector<unsigned long long> slot_ad;
    DevBuf<rk::AdapterRec> ad_table; // [max_gpt]
    std::vector<rwkv_b200_prefix_cache *> prefix_caches; // open caches, closed by rwkv_b200_free
};

// rwkv_b200_prefix_cache_open: the index on the host, the pool on the device, and the {entry, slot} pairs of a copy
struct rwkv_b200_prefix_cache {
    rwkv_b200_model *m = nullptr;
    prefix::Index index;
    unsigned long long block = 0;
    DevBuf<double> pool;               // xy, aa, bb, dd: each [capacity][L][E]
    DevBuf<unsigned long long> pairs;  // [max_gpt][2]
    explicit rwkv_b200_prefix_cache(size_t capacity) : index(capacity) {}
};

// rwkv_b200_batcher: the requests on the host, and per lane (0..rows-1, one per admitted request, reused) its stream
// record, sampler, penalty rows, stop tokens, overrides, automaton, log-probability choice and a ring of the current
// group's tokens (and their log-probabilities) on the device, in its own StepBuffers.
struct rwkv_b200_batcher {
    rwkv_b200_model *m = nullptr;
    int rows = 0, prefill_tokens = 0, max_pass = 0; // max_pass: passes of a step at most
    struct Req {
        unsigned long long slot = 0, max_new = 0;
        std::vector<unsigned long long> prompt, stop, tokens; // tokens: emitted so far
        std::vector<double> u;                                // empty: temperature 0
        rwkv_b200_sampler sampler{};
        int status = RWKV_B200_REQ_QUEUED;
        unsigned long long fed = 0; // tokens of prompt[0 .. n_prompt - 1) in the slot
        int lane = -1;
        // rwkv_b200_batcher_submit_ex: the overrides, the automaton (gc.mask == nullptr: none; gc.state is the current
        // state) and its id, and the scoring (lp.mode < 0: none) with the results of the emitted tokens so far
        std::vector<unsigned long long> ovr_tok;
        std::vector<float> ovr_val;
        rk::GenConstraint gc{};
        unsigned long long constraint_id = RWKV_B200_NO_CONSTRAINT;
        rk::LogprobLane lp{-1, 0};
        std::vector<double> logprobs, top_logprobs;             // [tokens], [tokens][lp.top_n]
        std::vector<unsigned long long> ranks, top_tokens;      // [tokens], [tokens][lp.top_n]
        // rwkv_b200_batcher_submit_stop: the stop set (gst.next == nullptr: none) with its match state and result
        rk::GenStop gst{};
        unsigned long long stop_set = RWKV_B200_NO_STOP_SET;
        // rwkv_b200_batcher_submit_spec: k drafts per step (0: none), the n-gram, the spare slots and the lookup context;
        // the steps that emitted a token and which of [slot, spares...] holds the conversation (home)
        unsigned draft = 0, ngram = 0;
        std::vector<unsigned long long> spares, context;
        unsigned long long steps = 0;
        int home = 0;
        // rwkv_b200_batcher_submit_prefix: the cache (nullptr: none) and the prompt tokens restored at admission
        rwkv_b200_prefix_cache *cache = nullptr;
        unsigned long long cached = 0;
    };
    std::map<unsigned long long, Req> reqs;
    unsigned long long next_id = 1;
    std::deque<unsigned long long> queue;     // queued ids, submission order
    std::vector<unsigned long long> admitted; // admitted ids, admission order
    std::vector<char> lane_used;              // [rows]
    // the lanes' device buffers: records, row map, samplers, stop tokens (CSR), the passes of a group's steps
    // ([kGenGroup][max_pass]) and its uniforms are sized at open; pen_cnt and pen_seen grow at the first request with
    // penalties; the overrides, automata, stop sets, scoring and speculative buffers at the first group whose decode
    // lanes use them
    StepBuffers bufs;
    // host mirrors, [rows] each: the lanes' records, automata (mask nullptr: none), scoring (mode < 0: none), stop sets
    // (next nullptr: none) and speculative records, and the group's rings of tokens and their results
    std::vector<rk::GenStream> h_gs;
    std::vector<rk::GenConstraint> h_gc;
    std::vector<rk::LogprobLane> h_lp;
    std::vector<rk::GenStop> h_gst;
    std::vector<rk::SpecStream> h_ss;
    std::vector<unsigned long long> h_out, h_rank, h_top_tok;
    std::vector<double> h_lpv, h_top_lp;
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

// A failed synchronisation: if the kernel left a diagnostic record, say what it was waiting for.
int sync_failed(M *m, cudaError_t e, const char *what) {
    const rk::Diag *d = m->h_diag;
    if (d && d->code) {
        static const char *names[] = {"", "slice statistics", "activation vector", "offset sums", "peer partial sums",
                                      "sigmoid exchange", "completion flags", "arg-max candidates", "ring (full)", "ring (empty)"};
        return fail(100 + (int)e,
                    "%s failed: %s; token kernel timed out waiting for %s: rank %u cta %u thread %u layer %u kind %u "
                    "expected tag %u saw %u aux %llu (a peer rank that never launched, or a protocol bug)",
                    what, cudaGetErrorString(e), d->code < 10 ? names[d->code] : "?", d->rank, d->cta, d->thread, d->layer,
                    d->kind, d->expect, d->seen, d->aux);
    }
    return fail(100 + (int)e, "%s failed: %s", what, cudaGetErrorString(e));
}
#define SYNC(m)                                                          \
    do {                                                                 \
        cudaError_t e__ = cudaStreamSynchronize((m)->stream);            \
        if (e__ != cudaSuccess) return sync_failed((m), e__, "forward"); \
    } while (0)
// Follows every <<<>>> launch that launch_count counts: its launch error, and one launch more.
#define LAUNCHED(m)             \
    do {                        \
        CK(cudaGetLastError()); \
        (m)->launches += 1;     \
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

void fill_launch(int grid, size_t smem, cudaLaunchConfig_t &cfg, cudaLaunchAttribute &attr, cudaStream_t s) {
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(rk::kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    attr.id = cudaLaunchAttributeCooperative;
    attr.val.cooperative = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
}

int launch_token(M *m, int feed, bool greedy, const unsigned long long *stream, cudaStream_t s) {
    if (m->tp_size > 1 && !m->tp_wired)
        return fail(7, "tensor parallelism: call rwkv_b200_tp_import with every rank's handle before the first forward");
    rk::Params prm = m->p;
    prm.feed_mode = feed;
    prm.greedy = greedy ? 1 : 0;
    prm.stream = stream;
    prm.ep0 = m->epoch;
    prm.tk = ++m->tk;
    if (prm.tk == 0) prm.tk = ++m->tk; // tag 0 means "never written"
    m->epoch += (unsigned int)prm.L + 1u;
    void *args[] = {&prm};
    const bool full = m->E == (unsigned long long)m->cpl * 512ull;
    const void *fn = token_entry(m->cpl, full, m->p.trace != nullptr);
    if (!fn) return fail(3, "no kernel for %d chunks per lane", m->cpl);
    // cooperative: all CTAs resident together (they wait for each other's words)
    cudaLaunchConfig_t cfg{};
    cudaLaunchAttribute attr;
    fill_launch(m->grid, m->smem, cfg, attr, s);
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

// A grid of `grid` CTAs: one CTA per SM at most (the CTAs wait for each other's words, so all of them must be
// resident at once) and the slice capacities.
int check_grid(M *m, int grid) {
    if (grid < 1 || grid > m->sms) return fail(1, "grid=%d must be 1..%d (the SM count)", grid, m->sms);
    if (!grid_fits(m->E, (unsigned long long)m->p.Er, (unsigned long long)m->p.Vr, grid))
        return fail(5, "a grid of %d CTAs does not fit n_embed=%llu", grid, m->E);
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
    // 12 KB copies, 2.5 tiles in flight while streaming, 1.25 while the CTAs exchange (80 / 40 KB at 7B): 3 % more
    // tokens/s at 7B than whole-tile copies, 2 and 1 tiles, on H100 SXM (DESIGN 4.1). Where a tile is at most 12 KB
    // the copies are whole tiles and the budgets admit 2 and 1 of them, as before.
    p.sub_bytes = std::min(12288, p.tile_bytes);
    p.budget = std::max(p.tile_bytes, std::min(p.stages * p.tile_bytes, 5 * p.tile_bytes / 2));
    p.qbudget = 5 * p.tile_bytes / 4;
    p.pf_dist = 4;
    p.vseg = G >= 4 ? 1 : G >= 2 ? 2 : 4; // 4E/G bytes per ffn-V row in segments of at most E bytes
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
    const size_t n_pass = (m->max_gpt + rk::kPfMaxTokens - 1) / rk::kPfMaxTokens;
    if ((rc = m->gen.gs.grow(m->max_gpt)) || (rc = m->gen.row_stream.grow(m->max_gpt)) || (rc = m->gen.passes.grow(n_pass)))
        return rc;
    // every pass of the generation calls starts zeroed: an upload fills the first step's passes, and k_beam_select and
    // k_gen_feedback then fill tokens, descriptors and row maps of passes no upload reached, so no snapshot field there
    // may hold leftover bytes
    CK(cudaMemsetAsync(m->gen.passes.p, 0, n_pass * sizeof(rk::PassDesc), m->stream));
    CK(cudaMallocHost((void **)&m->h_gs, sizeof(rk::GenStream) * m->max_gpt));
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

// The adapter bound to a slot, or RWKV_B200_NO_ADAPTER.
unsigned long long slot_binding(const M *m, unsigned long long slot) {
    return slot < m->slot_ad.size() ? m->slot_ad[slot] : RWKV_B200_NO_ADAPTER;
}
bool any_bound(const M *m, const unsigned long long *slots, unsigned long long n) {
    for (unsigned long long i = 0; i < n; ++i)
        if (slot_binding(m, slots[i]) != RWKV_B200_NO_ADAPTER) return true;
    return false;
}
// The slots of one conversation (a speculative stream, a beam group, a batcher request) hold it in turn, so they must
// all carry the same binding.
int check_same_binding(M *m, const char *what, const char *whose, unsigned long long index, const unsigned long long *slots,
                       unsigned long long n) {
    for (unsigned long long i = 1; i < n; ++i)
        if (slot_binding(m, slots[i]) != slot_binding(m, slots[0]))
            return fail(1, "%s: the slots of %s %llu are not bound to the same adapter (slot %llu and slot %llu)", what, whose,
                        index, slots[0], slots[i]);
    return 0;
}
// The decode kernel has no adapters: a call that runs on it refuses a bound slot.
int check_unbound(M *m, const char *what, const unsigned long long *slots, unsigned long long n) {
    for (unsigned long long i = 0; i < n; ++i)
        if (slot_binding(m, slots[i]) != RWKV_B200_NO_ADAPTER)
            return fail(1, "%s: slot %llu is bound to an adapter, which runs on the tensor cores only (use forward_streams)",
                        what, slots[i]);
    return 0;
}

// Tensor cores or the decode kernel for a forward of n tokens: forward_streams' rule, which every call that has a
// choice follows (the multi-stream calls refuse tensor parallelism). A call that names a bound slot (`bound`) takes the
// tensor cores whatever n, since adapters run there only.
bool tensor_cores(const M *m, unsigned long long n, bool bound = false) {
    return (bound || n >= (unsigned long long)m->pf.min_tokens) && m->tp_size == 1 && rk::prefill_enabled(m->pf);
}

// The adapter bit of a call's passes: set when one of its slots is bound (then the tensor cores are required); a call
// without bound slots enqueues exactly the passes it enqueues on a model without adapters.
int set_pass_adapters(M *m, const char *what, const unsigned long long *slots, unsigned long long n, bool &bound) {
    bound = any_bound(m, slots, n);
    m->pf.adapt = bound;
    m->pf.ad_table = m->ad_table.p;
    if (bound && !rk::prefill_enabled(m->pf))
        return fail(1, "%s: a slot bound to an adapter needs the tensor cores, and the \"prefill\" option is 0", what);
    return 0;
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
// Largest guidance scale accepted (rwkv_b200_generate_streams_guided): guided logits stay far inside the f32 range.
constexpr float kMaxGuidance = 100.0f;

// One step of generate_streams over `rows` rows on the decode kernel: each row on its stream's slot (or the scratch
// slot once the stream is done), its logits into row r of d_slogits. row_stream: the stream record of each row.
int gen_step_decode(M *m, int rows, const int *row_stream) {
    const size_t V = binfmt::kVocab;
    for (int r = 0; r < rows; ++r) {
        rk::k_gen_gate<<<1, 1, 0, m->stream>>>(m->gen.gs.p, row_stream, r, m->max_gpt, m->p.ctrl);
        LAUNCHED(m);
        int rc = launch_token(m, 0, false, nullptr, m->stream);
        if (rc) return rc;
        CK(cudaMemcpyAsync(m->d_slogits + (size_t)r * V, dev_logits(m), V * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
    }
    return 0;
}

// One step on the tensor cores: ceil(rows / per_pass) passes of per_pass rows (the last may be shorter) whose
// descriptors are in `passes` on the device (the previous step's feedback, the group's upload, or k_spec_draft). Pass i
// has heads[i] head rows (pass_layout's count); with heads NULL every row is a head row, so row r's logits land in
// d_slogits row r.
int gen_step_passes(M *m, const rk::PassDesc *passes, int rows, int per_pass, const int *heads = nullptr) {
    for (int p0 = 0, pi = 0; p0 < rows; p0 += per_pass, ++pi) {
        const int T = std::min(per_pass, rows - p0);
        CK(cudaMemcpyAsync(m->pf.pass, passes + pi, sizeof(rk::PassDesc), cudaMemcpyDeviceToDevice, m->stream));
        int rc = rk::prefill_run(m->pf, m->p, m->stream, T, heads ? heads[pi] : T, m->d_slogits);
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
        tokens[r] = m->h_gs[rec[r]].tok;
        slots[r] = m->h_gs[rec[r]].slot;
    }
    std::vector<rk::PassDesc> passes;
    std::vector<int> heads;
    rk::pass_layout(tokens.data(), rows, slots.data(), lens.data(), 2, nullptr, passes, heads);
    CK(cudaMemcpyAsync(m->gen.passes.p, passes.data(), passes.size() * sizeof(rk::PassDesc), cudaMemcpyHostToDevice, m->stream));
    return 0;
}

// k_beam_fork over n_pairs {source, destination} slot pairs in `forks` (device): it copies xy, aa, bb, pp and dd, or
// without `with_pp` xy, aa, bb and dd.
int fork_slots(M *m, const unsigned long long *forks, unsigned long long n_pairs, bool with_pp) {
    double *a[5];
    slot_arrays(m, 0, a);
    const size_t slot_len = (size_t)(m->L * m->E);
    const unsigned chunks = (unsigned)((slot_len + rk::kForkChunk - 1) / rk::kForkChunk);
    rk::k_beam_fork<<<dim3((unsigned)n_pairs, chunks, with_pp ? 5 : 4), rk::kForkThreads, 0, m->stream>>>(
        forks, a[0], a[1], a[2], with_pp ? a[3] : a[4], with_pp ? a[4] : nullptr, slot_len);
    LAUNCHED(m);
    return 0;
}

// One stream's sampler. `history`: the call keeps the stream's emitted tokens (generate_streams_ex), so the penalties
// may be set; elsewhere they must be 0 and penalty_decay is not read. `has_u`: the call was given uniforms, which a
// temperature above 0 needs.
int check_sampler(const char *what, unsigned long long s, const rwkv_b200_sampler &p, bool history, bool has_u) {
    if (!(p.temperature >= 0.0f && p.temperature <= FLT_MAX))
        return fail(1, "%s: stream %llu: temperature %g is not a finite value >= 0", what, s, p.temperature);
    if (!(p.top_p > 0.0f && p.top_p <= 1.0f)) return fail(1, "%s: stream %llu: top_p %g is outside (0, 1]", what, s, p.top_p);
    if (p.top_k > binfmt::kVocab) return fail(1, "%s: stream %llu: top_k %u > %llu", what, s, p.top_k, (unsigned long long)binfmt::kVocab);
    if (!history) {
        if (p.presence_penalty != 0.0f || p.frequency_penalty != 0.0f)
            return fail(1, "%s: stream %llu: presence_penalty and frequency_penalty must be 0 here (no token history; see "
                           "generate_streams_ex)", what, s);
    } else {
        if (!(fabsf(p.presence_penalty) <= kMaxPenalty))
            return fail(1, "%s: stream %llu: presence_penalty %g is not finite or exceeds %g in magnitude", what, s, p.presence_penalty, kMaxPenalty);
        if (!(fabsf(p.frequency_penalty) <= kMaxPenalty))
            return fail(1, "%s: stream %llu: frequency_penalty %g is not finite or exceeds %g in magnitude", what, s, p.frequency_penalty, kMaxPenalty);
        if (!(p.penalty_decay > 0.0f && p.penalty_decay <= 1.0f))
            return fail(1, "%s: stream %llu: penalty_decay %g is outside (0, 1]", what, s, p.penalty_decay);
    }
    if (p.temperature > 0.0f && !has_u) return fail(1, "%s: u is NULL but stream %llu samples (temperature %g)", what, s, p.temperature);
    return 0;
}

// The uniforms u[0..n-1] (none when u is NULL), each in [0, 1).
int check_uniforms(const char *what, const double *u, unsigned long long n) {
    for (unsigned long long i = 0; u && i < n; ++i)
        if (!(u[i] >= 0.0 && u[i] < 1.0)) return fail(1, "%s: u[%llu] = %g is outside [0, 1)", what, i, u[i]);
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

// A logprob_mode and top_n of generate_streams_logprobs or batcher_submit_ex.
int check_logprob_mode(const char *what, int mode, unsigned top_n) {
    if (mode != RWKV_B200_LOGPROBS_RAW && mode != RWKV_B200_LOGPROBS_PROCESSED)
        return fail(1, "%s: logprob_mode %d is neither RWKV_B200_LOGPROBS_RAW (0) nor RWKV_B200_LOGPROBS_PROCESSED (1)", what,
                    mode);
    if (top_n > (unsigned)rk::kMaxTopN) return fail(1, "%s: top_n %u > %d", what, top_n, rk::kMaxTopN);
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

// The stop set of each stream of a call with a stop request (a zero record: none), refused before any work: unknown ids,
// a set used before the model has token bytes, and start states out of range.
int check_stops(M *m, const char *what, const rwkv_b200_stop_request *sq, unsigned long long n_streams,
                std::vector<rk::GenStop> &out) {
    out.assign(n_streams, rk::GenStop{});
    if (!sq || !sq->set_ids) return 0;
    for (unsigned long long s = 0; s < n_streams; ++s) {
        const unsigned long long id = sq->set_ids[s];
        if (id == RWKV_B200_NO_STOP_SET) continue;
        const auto it = m->stop_sets.find(id);
        if (it == m->stop_sets.end()) return fail(1, "%s: stream %llu: stop set id %llu is unknown or removed", what, s, id);
        if (!m->has_tb)
            return fail(1, "%s: stream %llu: stop set %llu is used before the model has a token-bytes table "
                           "(rwkv_b200_token_bytes_set)", what, s, id);
        const M::StopSet &ss = it->second;
        const unsigned long long q = sq->start_states ? sq->start_states[s] : 0;
        if (q >= ss.states)
            return fail(1, "%s: stream %llu: start state %llu of stop set %llu is out of range (%llu states)", what, s, q, id,
                        ss.states);
        out[s] = rk::GenStop{ss.dev.p, ss.dev.p + ss.states * 256, m->tb_start.p, m->tb_bytes.p, q, 0, 0};
    }
    return 0;
}

// A call's stop results from the streams' final records (the request's NULL arrays are skipped).
void write_stops(const rwkv_b200_stop_request *sq, const std::vector<rk::GenStop> &st) {
    if (!sq) return;
    for (size_t s = 0; s < st.size(); ++s) {
        const bool on = st[s].next != nullptr;
        if (sq->states_out) sq->states_out[s] = on ? st[s].state : 0;
        if (sq->hit_out) sq->hit_out[s] = on ? st[s].match : 0;
        if (sq->tail_out) sq->tail_out[s] = on ? st[s].tail : 0;
    }
}

// The arguments the generate_streams calls and generate_streams_speculative share: the streams (their slots, first
// tokens, max_new and budgets), the stop tokens, overrides, samplers (NULL: none) and uniforms, and the results.
struct GenCall {
    const unsigned long long *slots, *first_tokens;
    unsigned long long n_streams, max_new;
    const unsigned long long *budgets, *stop_tokens;
    unsigned long long n_stop;
    const unsigned long long *override_tokens;
    const float *override_values;
    unsigned long long n_override;
    const rwkv_b200_sampler *samplers;
    const double *u;
    unsigned long long *tokens_out, *lengths_out;
};

// The checks of a GenCall whose streams name `per_stream` slots each. `values`: the override values are checked too.
int check_gen(M *m, const char *what, const GenCall &c, unsigned long long per_stream, bool values) {
    if (c.n_streams == 0) return fail(1, "%s: no streams", what);
    if (!c.slots || !c.first_tokens || !c.tokens_out || !c.lengths_out)
        return fail(1, "%s: null argument (slots, first_tokens, tokens_out and lengths_out are required)", what);
    if (c.n_stop && !c.stop_tokens) return fail(1, "%s: n_stop = %llu with NULL stop_tokens", what, c.n_stop);
    if (c.n_override && (!c.override_tokens || !c.override_values))
        return fail(1, "%s: n_override = %llu with NULL override_tokens or override_values", what, c.n_override);
    if (c.max_new == 0) return fail(1, "%s: max_new is 0", what);
    int rc;
    if ((rc = check_slots(m, what, c.slots, c.n_streams * per_stream)) ||
        (rc = check_tokens(what, "first token", c.first_tokens, c.n_streams, "stream")))
        return rc;
    for (unsigned long long i = 0; c.budgets && i < c.n_streams; ++i)
        if (c.budgets[i] == 0 || c.budgets[i] > c.max_new)
            return fail(1, "%s: budget %llu of stream %llu is outside 1..max_new = %llu", what, c.budgets[i], i, c.max_new);
    if ((rc = check_tokens(what, "stop token", c.stop_tokens, c.n_stop)) ||
        (rc = check_tokens(what, "override token", c.override_tokens, c.n_override)) ||
        (values && (rc = check_overrides(what, c.override_tokens, c.override_values, c.n_override))))
        return rc;
    for (unsigned long long s = 0; c.samplers && s < c.n_streams; ++s)
        if ((rc = check_sampler(what, s, c.samplers[s], true, c.u != nullptr))) return rc;
    return check_uniforms(what, c.u, c.max_new * c.n_streams);
}

// The buffers of a GenCall, grown and filled: gen.out zeroed, gen.stop, gen.ovr_tok, gen.ovr_val and gen.samp uploaded.
int upload_gen(M *m, const GenCall &c) {
    auto &g = m->gen;
    int rc;
    if ((rc = g.out.grow(c.n_streams * c.max_new)) || (rc = g.stop.grow(c.n_stop)) || (rc = g.ovr_tok.grow(c.n_override)) ||
        (rc = g.ovr_val.grow(c.n_override)) || (c.samplers && (rc = g.samp.grow(c.n_streams))))
        return rc;
    CK(cudaMemsetAsync(g.out.p, 0, c.n_streams * c.max_new * sizeof(unsigned long long), m->stream));
    if (c.n_stop) CK(cudaMemcpyAsync(g.stop.p, c.stop_tokens, c.n_stop * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    if (c.n_override) {
        CK(cudaMemcpyAsync(g.ovr_tok.p, c.override_tokens, c.n_override * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(g.ovr_val.p, c.override_values, c.n_override * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    }
    if (c.samplers) CK(cudaMemcpyAsync(g.samp.p, c.samplers, c.n_streams * sizeof(rwkv_b200_sampler), cudaMemcpyHostToDevice, m->stream));
    return 0;
}

// What a step does to its logits rows up to the pick, in this order: the penalties (pen_cnt set), the overrides
// (n_override > 0), the automaton masks (gc set), then one pick per row into d_sample: the nucleus sampler with each
// row's stream's sampler (samp set), the typical sampler (a step with uniforms), or else the arg-max into d_next. Row r
// of d_slogits belongs to stream record row_stream[r].
struct PickChain {
    const rk::GenStream *gs;
    const int *row_stream;
    const rwkv_b200_sampler *samp;
    float *pen_cnt;
    unsigned char *pen_seen;
    const unsigned long long *ovr_tok;
    const float *ovr_val;
    unsigned long long n_override;
    const rk::GenConstraint *gc;
    int exponent; // the typical sampler's
    // the batcher: each row's own overrides, ovr_*[ovr_start[s] .. ovr_start[s + 1]) of its stream s (n_override > 0
    // only says that some row has one); nullptr: all n_override for every row
    const unsigned long long *ovr_start;
    // speculative generation: the automaton state of each row (k_gen_mask's row_state); nullptr: each stream's state
    const unsigned long long *row_state;
};

// The chain on rows 0..rows-1 of d_slogits; u: the step's uniforms, one per row (NULL: none).
int pick_rows(M *m, const PickChain &pc, int rows, const double *u) {
    const size_t V = binfmt::kVocab;
    if (pc.pen_cnt) {
        const dim3 grid((unsigned)((V + rk::kPenaltyThreads - 1) / rk::kPenaltyThreads), (unsigned)rows);
        rk::k_gen_penalty<<<grid, rk::kPenaltyThreads, 0, m->stream>>>(m->d_slogits, (int)V, pc.gs, pc.row_stream, pc.samp, pc.pen_cnt,
                                                                      pc.pen_seen);
        LAUNCHED(m);
    }
    if (pc.n_override) {
        rk::k_gen_override<<<(unsigned)((rows + 127) / 128), 128, 0, m->stream>>>(m->d_slogits, (int)V, rows, pc.ovr_tok, pc.ovr_val,
                                                                                (int)pc.n_override, pc.row_stream, pc.ovr_start);
        LAUNCHED(m);
    }
    if (pc.gc) {
        const dim3 grid((unsigned)((V + rk::kMaskThreads - 1) / rk::kMaskThreads), (unsigned)rows);
        rk::k_gen_mask<<<grid, rk::kMaskThreads, 0, m->stream>>>(m->d_slogits, (int)V, pc.gs, pc.row_stream, pc.gc, pc.row_state);
        LAUNCHED(m);
    }
    if (pc.samp)
        rk::k_sample_nucleus<<<(unsigned)rows, rk::kNucThreads, 0, m->stream>>>(m->d_slogits, (int)V, pc.samp, pc.row_stream, u,
                                                                               m->d_sample);
    else if (u)
        rk::k_sample_typical<<<(unsigned)rows, rk::kSampleThreads, 0, m->stream>>>(m->d_slogits, V, (int)V, pc.exponent, u,
                                                                                  m->d_sample);
    else
        rk::k_argmax_rows<<<(unsigned)rows, rk::kArgmaxThreads, 0, m->stream>>>(m->d_slogits, (int)V, m->d_next);
    LAUNCHED(m);
    return 0;
}

// The log-probability request of generate_streams_logprobs and the calls after it, refused before any work.
int check_logprobs(const char *what, const LogprobRequest &lpq) {
    int rc;
    if ((rc = check_logprob_mode(what, lpq.mode, lpq.top_n))) return rc;
    if (!lpq.logprobs_out) return fail(1, "%s: logprobs_out is NULL", what);
    if (lpq.top_n && (!lpq.top_tokens_out || !lpq.top_logprobs_out))
        return fail(1, "%s: top_n = %u needs top_tokens_out and top_logprobs_out", what, lpq.top_n);
    return 0;
}

// What the steps of a call or of a batcher group enqueue besides the forward, and how their kernels read their inputs:
// derived from the call (check_features) or from the group's decode lanes (batcher_upload).
struct StepFlags {
    // samplers: every stream picks by its own sampler; uniforms: the rows draw uniforms (the typical sampler's, or the
    // samplers'); neither: the arg-max
    bool samplers = false, uniforms = false;
    // pen: some stream has a presence or frequency penalty; n_override: the overrides of the rows
    bool pen = false, constrained = false, stopped = false;
    unsigned long long n_override = 0;
    // scored, spec_scored: the one-token rows, the speculative rows are scored; raw: the scoring reads the model's rows
    // (the call's mode, or some batcher lane's); raw_copy (set_raw_copy): from a copy taken before the penalties,
    // overrides and masks edit d_slogits; top: the stride of the top arrays
    bool scored = false, spec_scored = false, raw = false, raw_copy = false;
    int top = 0;
    // guided: some stream has a guidance slot (k_gen_guide edits its row before the pick chain)
    bool guided = false;
};

// Raw log-probabilities read a copy of the model's rows when the guidance or the pick chain edits d_slogits.
void set_raw_copy(StepFlags &f) { f.raw_copy = f.raw && (f.pen || f.n_override || f.constrained || f.guided); }

// What a one-shot decoding call (generate() and speculate()) does besides emitting tokens: score them (lpq), follow
// token automata (cq) and stop sets (sq), and count penalties; each request is NULL when the call has none. Built by
// check_features, its buffers in m->gen readied by upload_features and its results written by finish_features.
struct CallFeatures : StepFlags {
    const LogprobRequest *lpq = nullptr;
    const ConstraintRequest *cq = nullptr;
    const rwkv_b200_stop_request *sq = nullptr;
    std::vector<rk::GenConstraint> gc; // each stream's automaton (a zero record: none)
    std::vector<rk::GenStop> st;       // each stream's stop set (a zero record: none)
    size_t n_lp = 0, n_top = 0; // entries of the log-probability and top arrays
};

// The automata and stop sets of a call's streams, checked against the model (the log-probability request is checked
// by the caller, where its message comes first), and the flags and sizes that follow from them.
int check_features(M *m, const char *what, const GenCall &c, const LogprobRequest *lpq, const ConstraintRequest *cq,
                   const rwkv_b200_stop_request *sq, CallFeatures &f) {
    const unsigned long long n = c.n_streams;
    f.lpq = lpq;
    f.cq = cq;
    f.sq = sq;
    f.samplers = c.samplers != nullptr;
    f.uniforms = c.u != nullptr;
    f.n_override = c.n_override;
    for (unsigned long long s = 0; c.samplers && s < n; ++s)
        f.pen |= c.samplers[s].presence_penalty != 0.0f || c.samplers[s].frequency_penalty != 0.0f;
    int rc;
    if (cq && (rc = check_constraints(m, what, *cq, n, c.override_tokens, c.override_values, c.n_override, f.gc))) return rc;
    f.constrained = std::any_of(f.gc.begin(), f.gc.end(), [](const rk::GenConstraint &gc) { return gc.mask != nullptr; });
    if ((rc = check_stops(m, what, sq, n, f.st))) return rc;
    f.stopped = std::any_of(f.st.begin(), f.st.end(), [](const rk::GenStop &st) { return st.next != nullptr; });
    f.scored = f.spec_scored = lpq != nullptr;
    f.raw = lpq && lpq->mode == RWKV_B200_LOGPROBS_RAW;
    set_raw_copy(f);
    f.top = lpq ? (int)lpq->top_n : 0;
    f.n_lp = (size_t)(n * c.max_new);
    f.n_top = lpq ? f.n_lp * lpq->top_n : 0;
    return 0;
}

// The feature buffers of m->gen grown for n_streams streams and steps of at most `rows` logits rows, then filled: the
// automata and stop sets uploaded, the fault record and penalty counts cleared, the result arrays set to all ones.
int upload_features(M *m, const CallFeatures &f, unsigned long long n_streams, size_t rows) {
    const size_t V = binfmt::kVocab;
    auto &g = m->gen;
    int rc;
    if ((f.constrained && ((rc = g.gc.grow(n_streams)) || (rc = g.fault.grow(3)))) || (f.stopped && (rc = g.gst.grow(n_streams))) ||
        (f.pen && ((rc = g.pen_cnt.grow(n_streams * V)) || (rc = g.pen_seen.grow(n_streams * V)))) ||
        (f.lpq && ((rc = g.lp.grow(f.n_lp)) || (rc = g.rank.grow(f.n_lp)) || (rc = g.top_tok.grow(f.n_top)) ||
                   (rc = g.top_lp.grow(f.n_top)) || (f.raw_copy && (rc = g.raw.grow(rows * V))))))
        return rc;
    if (f.constrained) {
        CK(cudaMemcpyAsync(g.gc.p, f.gc.data(), n_streams * sizeof(rk::GenConstraint), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemsetAsync(g.fault.p, 0, 3 * sizeof(unsigned long long), m->stream));
    }
    if (f.stopped) CK(cudaMemcpyAsync(g.gst.p, f.st.data(), n_streams * sizeof(rk::GenStop), cudaMemcpyHostToDevice, m->stream));
    if (f.pen) { // the history starts empty in every call: prompt tokens are not counted
        CK(cudaMemsetAsync(g.pen_cnt.p, 0, n_streams * V * sizeof(float), m->stream));
        CK(cudaMemsetAsync(g.pen_seen.p, 0, n_streams * V, m->stream));
    }
    if (f.lpq) { // all ones: NaN logprobs and RWKV_B200_NO_TARGET ranks and tokens wherever no token is emitted
        CK(cudaMemsetAsync(g.lp.p, 0xFF, f.n_lp * sizeof(double), m->stream));
        CK(cudaMemsetAsync(g.rank.p, 0xFF, f.n_lp * sizeof(unsigned long long), m->stream));
        if (f.n_top) {
            CK(cudaMemsetAsync(g.top_tok.p, 0xFF, f.n_top * sizeof(unsigned long long), m->stream));
            CK(cudaMemsetAsync(g.top_lp.p, 0xFF, f.n_top * sizeof(double), m->stream));
        }
    }
    return 0;
}

struct DraftStep;

// The arguments of a step's kernels; `raw` is where the step copies its model rows (nullptr: no copy).
struct StepArgs {
    PickChain pc;
    rk::GenLogprobArgs la;
    rk::SpecArgs sa;
    rk::GenFeedbackArgs fb;
    float *raw;
    // classifier-free guidance: n_guide guided rows of the step, each with its GenGuide (generate() sets them per group)
    const rk::GenGuide *guide;
    int n_guide;
    // speculative streams whose drafts come from a draft model (generate_streams_drafted); nullptr: prompt lookup
    DraftStep *draft;
};

// The arguments every step of a call or batcher group shares, over the buffers of `sb` as its upload readied them:
// each stream's tokens (and results) at [s][len % max_new], and n_stop stop tokens for every stream. Buffers only the
// batcher grows give each lane its own overrides (ovr_start), stop tokens (stop_start) and scoring (lp_lane: raw lanes
// read the copy, the others d_slogits with their sampler). The caller adds the shape of its steps: the one-token rows,
// the speculative k and uniform stride, the passes and the uniforms.
void step_args(M *m, StepBuffers &sb, const StepFlags &f, unsigned long long max_new, unsigned long long n_stop, StepArgs &a) {
    a = StepArgs{};
    const unsigned long long *next = f.samplers || f.uniforms ? nullptr : m->d_next;
    PickChain &pc = a.pc;
    pc.gs = sb.gs.p;
    pc.row_stream = sb.row_stream.p;
    pc.samp = f.samplers ? sb.samp.p : nullptr;
    pc.pen_cnt = f.pen ? sb.pen_cnt.p : nullptr;
    pc.pen_seen = sb.pen_seen.p;
    pc.ovr_tok = sb.ovr_tok.p;
    pc.ovr_val = sb.ovr_val.p;
    pc.n_override = f.n_override;
    pc.gc = f.constrained ? sb.gc.p : nullptr;
    pc.ovr_start = sb.ovr_start.p;
    rk::GenEmit &e = a.fb.emit;
    e.out = sb.out.p;
    e.max_new = max_new;
    e.stop = sb.stop.p;
    e.n_stop = (int)n_stop;
    e.stop_start = sb.stop_start.p;
    e.gc = f.constrained ? sb.gc.p : nullptr;
    e.fault = sb.fault.p;
    e.gst = f.stopped ? sb.gst.p : nullptr;
    a.raw = f.raw_copy ? sb.raw.p : nullptr;
    rk::GenLogprobArgs &la = a.la;
    la.lane = sb.lp_lane.p;
    la.raw = a.raw;
    la.logits = a.raw && !la.lane ? a.raw : m->d_slogits;
    la.V = (int)binfmt::kVocab;
    la.gs = sb.gs.p;
    la.row_stream = sb.row_stream.p;
    la.next = next;
    la.sample = m->d_sample;
    la.samp = la.lane || !f.raw ? pc.samp : nullptr;
    la.top_n = f.top;
    la.max_new = max_new;
    la.logprob = sb.lp.p;
    la.rank = sb.rank.p;
    la.top_tokens = sb.top_tok.p;
    la.top_logprobs = sb.top_lp.p;
    rk::SpecArgs &sa = a.sa;
    sa.ss = sb.ss.p;
    sa.live = sb.live.p;
    sa.hist = sb.hist.p;
    sa.u = f.uniforms ? sb.su.p : nullptr;
    sa.row_u = sb.u.p;
    sa.next = next;
    sa.sample = m->d_sample;
    sa.emit = e;
    sa.row_state = sb.row_state.p;
    sa.score = f.spec_scored ? sb.score.p : nullptr;
    a.fb.gs = sb.gs.p;
    a.fb.row_stream = sb.row_stream.p;
    a.fb.next = next;
    a.fb.sample = m->d_sample;
}

// One decoding step of generate(), speculate() and the batcher, enqueued in this order: k_spec_draft over n_spec
// speculative streams (with a.draft: draft_step, then k_spec_layout); the forward, on the tensor cores (fwd_rows tokens in passes of per_pass at `passes`, heads[i]
// head rows in pass i; heads NULL: every row a head row, whose head maps k_spec_draft writes) or, with passes NULL, on
// the decode kernel; nothing more when the step has no logits rows; the raw copy and the pick chain over `rows` rows
// with uniforms u, after k_gen_guide over the a.n_guide guided rows (their guidance rows follow the `rows` rows);
// k_gen_logprob and k_gen_feedback over the a.fb.rows one-token rows (rows 0..), then k_gen_guide_feedback;
// k_spec_accept, then k_spec_logprob over n_spec x (a.sa.k + 1) rows.
int draft_step(const DraftStep &d);

int run_step(M *m, const StepFlags &f, StepArgs &a, const rk::PassDesc *passes, int fwd_rows, int per_pass, const int *heads,
             int rows, int n_spec, const double *u) {
    const int plain = a.fb.rows;
    int rc;
    if (n_spec) {
        a.sa.heads = heads == nullptr;
        if (a.draft) {
            if ((rc = draft_step(*a.draft))) return rc;
            rk::k_spec_layout<<<(unsigned)n_spec, 32, 0, m->stream>>>(a.sa);
        } else {
            rk::k_spec_draft<<<(unsigned)n_spec, rk::kSpecDraftThreads, 0, m->stream>>>(a.sa);
        }
        LAUNCHED(m);
    }
    rc = passes ? gen_step_passes(m, passes, fwd_rows, per_pass, heads) : gen_step_decode(m, fwd_rows, a.pc.row_stream);
    if (rc || rows == 0) return rc;
    if (a.raw)
        CK(cudaMemcpyAsync(a.raw, m->d_slogits, (size_t)rows * binfmt::kVocab * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
    if (a.n_guide) {
        const dim3 grid((unsigned)((binfmt::kVocab + rk::kGuideThreads - 1) / rk::kGuideThreads), (unsigned)a.n_guide);
        rk::k_gen_guide<<<grid, rk::kGuideThreads, 0, m->stream>>>(m->d_slogits, (int)binfmt::kVocab, rows, a.guide);
        LAUNCHED(m);
    }
    if ((rc = pick_rows(m, a.pc, rows, u))) return rc;
    if (f.scored && plain) {
        rk::k_gen_logprob<<<(unsigned)plain, rk::kNucThreads, 0, m->stream>>>(a.la);
        LAUNCHED(m);
    }
    if (plain) {
        rk::k_gen_feedback<<<(unsigned)((plain + 127) / 128), 128, 0, m->stream>>>(a.fb);
        LAUNCHED(m);
    }
    if (a.n_guide) {
        rk::k_gen_guide_feedback<<<(unsigned)((a.n_guide + 127) / 128), 128, 0, m->stream>>>(a.fb.gs, a.fb.row_stream, plain,
                                                                                            a.n_guide, a.guide, a.fb.passes);
        LAUNCHED(m);
    }
    if (n_spec) {
        rk::k_spec_accept<<<(unsigned)n_spec, 32, 0, m->stream>>>(a.sa);
        LAUNCHED(m);
        if (f.spec_scored) {
            rk::k_spec_logprob<<<(unsigned)(n_spec * (a.sa.k + 1)), rk::kNucThreads, 0, m->stream>>>(a.sa, a.la);
            LAUNCHED(m);
        }
    }
    return 0;
}

// Enqueues the read-back of a group's automaton fault record into `fault` (with automata), read after the group's
// synchronisation: fault[0] - 1 is the stream that emitted token fault[1], which has no edge out of state
// fault[2] of its constraint.
int read_fault(M *m, const StepBuffers &sb, bool constrained, unsigned long long (&fault)[3]) {
    if (constrained) CK(cudaMemcpyAsync(fault, sb.fault.p, sizeof(fault), cudaMemcpyDeviceToHost, m->stream));
    return 0;
}

// The end of a group: `bytes` of stream records at `dev` come back into `host` with the automaton fault record, in one
// synchronisation; an emitted token without an edge fails the call.
int end_group(M *m, const char *what, const CallFeatures &f, void *host, const void *dev, size_t bytes) {
    unsigned long long fault[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, m->stream));
    if (int rc = read_fault(m, m->gen, f.constrained, fault)) return rc;
    SYNC(m);
    if (fault[0])
        return fail(8, "%s: stream %llu emitted token %llu, which has no edge out of state %llu of its constraint", what,
                    fault[0] - 1, fault[1], fault[2]);
    return 0;
}

// The end of a call: the tokens, scores, automaton states and stop records come back (one synchronisation) and go to
// the caller's arrays.
int finish_features(M *m, CallFeatures &f, const GenCall &c) {
    const auto &g = m->gen;
    const unsigned long long n_streams = c.n_streams;
    CK(cudaMemcpyAsync(c.tokens_out, g.out.p, n_streams * c.max_new * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
    if (const LogprobRequest *lpq = f.lpq) {
        CK(cudaMemcpyAsync(lpq->logprobs_out, g.lp.p, f.n_lp * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        if (lpq->ranks_out) CK(cudaMemcpyAsync(lpq->ranks_out, g.rank.p, f.n_lp * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        if (f.n_top) {
            CK(cudaMemcpyAsync(lpq->top_tokens_out, g.top_tok.p, f.n_top * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
            CK(cudaMemcpyAsync(lpq->top_logprobs_out, g.top_lp.p, f.n_top * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        }
    }
    if (f.constrained && f.cq->states_out)
        CK(cudaMemcpyAsync(f.gc.data(), g.gc.p, n_streams * sizeof(rk::GenConstraint), cudaMemcpyDeviceToHost, m->stream));
    if (f.stopped) CK(cudaMemcpyAsync(f.st.data(), g.gst.p, n_streams * sizeof(rk::GenStop), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    if (f.cq && f.cq->states_out)
        for (unsigned long long s = 0; s < n_streams; ++s) f.cq->states_out[s] = f.gc[s].mask ? f.gc[s].state : 0;
    write_stops(f.sq, f.st);
    return 0;
}

// The guidance of a guided call, refused before any work: NULL slots, NULL first tokens or scales while a slot is named,
// a guidance slot out of range, repeated or equal to a stream's slot, a first token out of the vocabulary, and a scale
// that is not finite or outside [0, 100]. The stream slots are checked already.
int check_guidance(M *m, const char *what, const GenCall &c, const rwkv_b200_guidance &gd) {
    if (!gd.slots) return fail(1, "%s: guidance with NULL slots", what);
    std::vector<char> used(m->max_gpt, 0); // 1: a stream's slot, 2: a guidance slot
    for (unsigned long long s = 0; s < c.n_streams; ++s) used[c.slots[s]] = 1;
    for (unsigned long long s = 0; s < c.n_streams; ++s) {
        const unsigned long long g = gd.slots[s];
        if (g == RWKV_B200_NO_GUIDANCE) continue;
        if (!gd.first_tokens || !gd.scales)
            return fail(1, "%s: stream %llu names guidance slot %llu with NULL first_tokens or scales", what, s, g);
        if (g >= m->max_gpt) return fail(1, "%s: stream %llu: guidance slot %llu >= max_gpt %llu", what, s, g, m->max_gpt);
        if (used[g] == 1) return fail(1, "%s: stream %llu: guidance slot %llu is the slot of a stream", what, s, g);
        if (used[g] == 2) return fail(1, "%s: stream %llu: guidance slot %llu appears twice", what, s, g);
        used[g] = 2;
        if (gd.first_tokens[s] >= binfmt::kVocab)
            return fail(1, "%s: stream %llu: guidance first token %llu out of range", what, s, gd.first_tokens[s]);
        const float w = gd.scales[s];
        if (!(w >= 0.0f && w <= kMaxGuidance))
            return fail(1, "%s: stream %llu: guidance scale %g is not a finite value in [0, %g]", what, s, w, kMaxGuidance);
    }
    return 0;
}

// The body of generate_streams (samplers == NULL, `temp` and `u` pick the typical sampler or the arg-max), of
// generate_streams_ex (`ex`: every stream has its own sampler, or all pick the arg-max when samplers == NULL), of
// generate_streams_logprobs (generate_streams_ex with `lpq`: each emitted token is scored after its pick) and of
// generate_streams_constrained (with `cq`: token automata mask the rows after the overrides; `lpq` may be NULL) and of
// generate_streams_stop (with `sq` as well: k_gen_feedback walks each emitted token through the stream's stop set) and
// of generate_streams_guided (with `gd`: a guided stream's guidance row runs on its guidance slot in the same forward,
// and k_gen_guide combines the two rows before the pick chain).
int generate(M *m, const char *what, bool ex, const GenCall &c, float temp, const LogprobRequest *lpq = nullptr,
             const ConstraintRequest *cq = nullptr, const rwkv_b200_stop_request *sq = nullptr,
             const rwkv_b200_guidance *gd = nullptr) {
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (lpq && (rc = check_logprobs(what, *lpq))) return rc;
    if ((rc = check_gen(m, what, c, 1, ex))) return rc;
    if (gd && (rc = check_guidance(m, what, c, *gd))) return rc;
    const unsigned long long n_streams = c.n_streams, max_new = c.max_new;
    // every slot the call names: the streams', then the guidance slots (stream record n_streams + j: guided stream j)
    std::vector<unsigned long long> named(c.slots, c.slots + n_streams);
    std::vector<int> guide_rec(n_streams, -1);
    for (unsigned long long s = 0; gd && s < n_streams; ++s)
        if (gd->slots[s] != RWKV_B200_NO_GUIDANCE) {
            guide_rec[s] = (int)named.size();
            named.push_back(gd->slots[s]);
        }
    const unsigned long long n_rec = named.size();
    bool bound;
    if ((rc = set_pass_adapters(m, what, named.data(), n_rec, bound))) return rc;
    CallFeatures f;
    if ((rc = check_features(m, what, c, lpq, cq, sq, f))) return rc;
    f.guided = n_rec > n_streams;
    set_raw_copy(f);
    CK(cudaSetDevice(m->device));
    auto &g = m->gen;
    if (c.u && (rc = g.u.grow(kGenGroup * m->max_gpt))) return rc;
    if (f.guided && (rc = g.guide.grow(n_rec - n_streams))) return rc;
    // the path is chosen once, for the rows of every stream and guidance slot; a stream's numbers depend only on its row
    const bool tc = tensor_cores(m, n_rec, bound);
    if (tc && (rc = rk::prefill_init(m->pf, m->p))) return fail(rc, "%s", rk::prefill_error());
    m->stream_rows = 0; // the compact logits rows no longer belong to a call the caller made

    rk::GenStream *hg = m->h_gs;
    for (unsigned long long s = 0; s < n_streams; ++s) {
        hg[s] = rk::GenStream{c.slots[s], c.budgets ? c.budgets[s] : max_new, c.first_tokens[s], 0, 0};
        if (guide_rec[s] >= 0) hg[guide_rec[s]] = rk::GenStream{gd->slots[s], hg[s].budget, gd->first_tokens[s], 0, 0};
    }
    CK(cudaMemcpyAsync(g.gs.p, hg, n_rec * sizeof(rk::GenStream), cudaMemcpyHostToDevice, m->stream));
    if ((rc = upload_gen(m, c)) || (rc = upload_features(m, f, n_streams, n_streams))) return rc;
    std::vector<int> live(n_streams), rs;
    for (unsigned long long s = 0; s < n_streams; ++s) live[s] = (int)s;
    std::vector<double> ug;
    std::vector<rk::GenGuide> guide;
    StepArgs a;
    step_args(m, g, f, max_new, c.n_stop, a);
    a.pc.exponent = sample_exponent(temp);
    a.fb.passes = tc ? g.passes.p : nullptr;
    a.guide = g.guide.p;
    for (unsigned long long step = 0; !live.empty() && step < max_new;) {
        // a group: the live streams are rows 0..rows-1, then the guidance rows of the live guided streams; their
        // inputs, and the uniforms of its steps, go up once
        const int rows = (int)live.size();
        const unsigned long long steps = std::min(kGenGroup, max_new - step);
        rs = live;
        guide.clear();
        for (int r = 0; r < rows; ++r)
            if (guide_rec[live[r]] >= 0) {
                rs.push_back(guide_rec[live[r]]);
                guide.push_back(rk::GenGuide{r, gd->scales[live[r]]});
            }
        const int fwd_rows = (int)rs.size();
        CK(cudaMemcpyAsync(g.row_stream.p, rs.data(), fwd_rows * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        if (!guide.empty())
            CK(cudaMemcpyAsync(g.guide.p, guide.data(), guide.size() * sizeof(rk::GenGuide), cudaMemcpyHostToDevice, m->stream));
        if (tc && (rc = upload_step_passes(m, rs.data(), fwd_rows))) return rc;
        if (c.u) {
            ug.resize((size_t)steps * rows);
            for (unsigned long long k = 0; k < steps; ++k)
                for (int r = 0; r < rows; ++r) ug[k * rows + r] = c.u[(step + k) * n_streams + live[r]];
            CK(cudaMemcpyAsync(g.u.p, ug.data(), ug.size() * sizeof(double), cudaMemcpyHostToDevice, m->stream));
        }
        a.fb.rows = rows;
        a.n_guide = (int)guide.size();
        for (unsigned long long k = 0; k < steps; ++k)
            if ((rc = run_step(m, f, a, a.fb.passes, fwd_rows, rk::kPfMaxTokens, nullptr, rows, 0, c.u ? g.u.p + k * rows : nullptr)))
                return rc;
        // the end of a group: which streams are done (a few bytes, one synchronisation); drop them (and their guidance
        // rows) from the rows
        if ((rc = end_group(m, what, f, hg, g.gs.p, n_rec * sizeof(rk::GenStream)))) return rc;
        step += steps;
        live.erase(std::remove_if(live.begin(), live.end(), [&](int s) { return hg[s].done != 0; }), live.end());
    }
    if ((rc = finish_features(m, f, c))) return rc;
    for (unsigned long long s = 0; s < n_streams; ++s) c.lengths_out[s] = hg[s].len;
    return 0;
}

// The copies home -> first slot of speculative streams that end with their conversation on a spare slot: {home, slot}
// pairs of xy, aa, bb and dd (pp: no tensor-core pass writes it).
int copy_home(M *m, StepBuffers &sb, const std::vector<unsigned long long> &forks) {
    int rc;
    if ((rc = sb.forks.grow(forks.size()))) return rc;
    CK(cudaMemcpyAsync(sb.forks.p, forks.data(), forks.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    return fork_slots(m, sb.forks.p, forks.size() / 2, false);
}

// What the speculative calls add to a GenCall: the drafts per step, the longest n-gram looked up, each stream's lookup
// context (tokens context[context_start[s] .. context_start[s + 1]); NULL context_start: none) and the result array of
// each stream's steps.
struct SpecRequest {
    unsigned draft, ngram;
    const unsigned long long *context_start, *context;
    unsigned long long *steps_out;
    const rwkv_b200_drafter *drafter; // generate_streams_drafted: the draft model instead of prompt lookup (no n-gram, no context)
};

// A drafted call's draft model and what each step enqueues there (speculate.cuh, "drafts from a draft model"): the
// kernels' arguments, the pick chain on the draft's rows (the call's sampler, overrides and automata; the draft's row
// map, row states and uniforms) and the head rows of each first pass.
struct DraftStep {
    M *dm = nullptr;
    rk::DraftArgs da{};
    PickChain pc{};
    const double *row_u = nullptr;
    std::vector<int> heads;
};

// One step's drafts on the draft model: k_draft_first, the first pass, then k times the pick chain and k_draft_pick,
// with the one-token pass of the next draft between them.
int draft_step(const DraftStep &d) {
    M *dm = d.dm;
    const rk::DraftArgs &da = d.da;
    const int n = da.n, W = da.k + 2;
    const unsigned blocks = (unsigned)((n + rk::kDraftThreads - 1) / rk::kDraftThreads);
    rk::k_draft_first<<<blocks, rk::kDraftThreads, 0, dm->stream>>>(da);
    LAUNCHED(dm);
    int rc = gen_step_passes(dm, da.first, n * W, da.per_first * W, d.heads.data());
    for (int i = 1; !rc && i <= da.k; ++i) {
        if ((rc = pick_rows(dm, d.pc, n, d.row_u))) return rc;
        rk::k_draft_pick<<<blocks, rk::kDraftThreads, 0, dm->stream>>>(da, i);
        LAUNCHED(dm);
        if (i < da.k) rc = gen_step_passes(dm, da.next, n, rk::kPfMaxTokens);
    }
    return rc;
}

// The drafter of a drafted call of S streams, refused before any work: a NULL handle, the target itself, another
// device, tensor parallelism, "prefill" 0, draft slots out of range or repeated, and a stream whose two draft slots are
// bound to different adapters. Then the draft's passes take its slots' adapters.
int check_drafter(M *m, const char *what, const rwkv_b200_drafter *dr, unsigned long long S) {
    if (!dr || !dr->model || !dr->slots) return fail(1, "%s: the drafter, its model or its slots is NULL", what);
    M *dm = dr->model;
    if (dm == m) return fail(1, "%s: the draft model is the target model", what);
    if (dm->device != m->device)
        return fail(1, "%s: the draft model is on device %d, the target on device %d", what, dm->device, m->device);
    if (dm->tp_size > 1) return fail(7, "%s: the draft model uses tensor parallelism", what);
    if (!rk::prefill_enabled(dm->pf)) return fail(1, "%s: the draft model needs the tensor cores (its \"prefill\" option is 0)", what);
    if (S > dm->max_gpt / 2)
        return fail(1, "%s: %llu streams x 2 draft slots > the draft model's max_gpt %llu", what, S, dm->max_gpt);
    const std::string dwhat = std::string(what) + ": draft model";
    int rc;
    if ((rc = check_slots(dm, dwhat.c_str(), dr->slots, 2 * S))) return rc;
    for (unsigned long long s = 0; s < S; ++s)
        if ((rc = check_same_binding(dm, dwhat.c_str(), "stream", s, dr->slots + 2 * s, 2))) return rc;
    bool bound;
    return set_pass_adapters(dm, dwhat.c_str(), dr->slots, 2 * S, bound);
}

// The draft model's buffers of a drafted call, after step_args: its records (D0, D1, nothing fed), its passes zeroed
// (k_draft_first and k_draft_pick fill tokens, descriptors and head maps only), D0 forked into D1, and the step's
// arguments over them.
int draft_setup(M *dm, const unsigned long long *slots, unsigned long long S, int k, const StepArgs &a, DraftStep &d) {
    auto &dg = dm->gen;
    const int per_first = rk::kPfMaxTokens / (k + 2), per_flush = rk::kPfMaxTokens / (k + 1);
    const size_t n_first = (S + per_first - 1) / per_first, n_next = (S + rk::kPfMaxTokens - 1) / rk::kPfMaxTokens;
    const size_t n_pass = std::max(n_first + n_next, (size_t)((S + per_flush - 1) / per_flush));
    int rc;
    if ((rc = dg.ds.grow(S)) || (rc = dm->spec_passes.grow(n_pass)) || (rc = dg.forks.grow(2 * S)) ||
        (a.sa.u && (rc = dg.u.grow(S))) || (a.pc.gc && (rc = dg.row_state.grow(S))))
        return rc;
    if ((rc = rk::prefill_init(dm->pf, dm->p))) return fail(rc, "%s", rk::prefill_error());
    dm->stream_rows = 0; // the draft's compact logits rows no longer belong to a call the caller made
    CK(cudaMemsetAsync(dm->spec_passes.p, 0, n_pass * sizeof(rk::PassDesc), dm->stream));
    std::vector<rk::SpecDraft> rec(S);
    for (unsigned long long s = 0; s < S; ++s) rec[s] = rk::SpecDraft{slots[2 * s], slots[2 * s + 1], 0};
    CK(cudaMemcpyAsync(dg.ds.p, rec.data(), S * sizeof(rk::SpecDraft), cudaMemcpyHostToDevice, dm->stream));
    // the first step's input continues D0's state on D1: the pairs {D0, D1} are the fork's {source, destination}
    CK(cudaMemcpyAsync(dg.forks.p, slots, 2 * S * sizeof(unsigned long long), cudaMemcpyHostToDevice, dm->stream));
    if ((rc = fork_slots(dm, dg.forks.p, S, false))) return rc;
    rk::DraftArgs &da = d.da;
    da.ss = a.sa.ss;
    da.live = a.sa.live;
    da.ds = dg.ds.p;
    da.hist = a.sa.hist;
    da.first = dm->spec_passes.p;
    da.next = dm->spec_passes.p + n_first;
    da.k = k;
    da.per_first = per_first;
    da.pick_next = a.sa.next ? dm->d_next : nullptr;
    da.pick_sample = dm->d_sample;
    da.u = a.sa.u;
    da.row_u = dg.u.p;
    da.u_stride = a.sa.u_stride;
    da.gc = a.pc.gc;
    da.row_state = dg.row_state.p;
    d.dm = dm;
    d.pc = a.pc;
    d.pc.row_stream = dg.row_stream.p;
    d.pc.row_state = a.pc.gc ? dg.row_state.p : nullptr;
    d.row_u = a.sa.u ? dg.u.p : nullptr;
    return 0;
}

// The call's end on the draft model: one pass without logits absorbs each stream's remaining tokens into D0.
int draft_flush(const DraftStep &d, unsigned long long S) {
    M *dm = d.dm;
    rk::DraftArgs da = d.da;
    const int W = da.k + 1;
    da.n = (int)S;
    da.per_first = rk::kPfMaxTokens / W;
    rk::k_draft_flush<<<(unsigned)((S + rk::kDraftThreads - 1) / rk::kDraftThreads), rk::kDraftThreads, 0, dm->stream>>>(da);
    LAUNCHED(dm);
    const std::vector<int> heads((S + da.per_first - 1) / da.per_first, 0);
    return gen_step_passes(dm, da.first, (int)S * W, da.per_first * W, heads.data());
}

// A draft model's work goes on the target's CUDA stream while the loan lasts, so the two models' launches keep one
// order without events or synchronisation.
struct StreamLoan {
    M *dm;
    cudaStream_t own;
    StreamLoan(M *d, cudaStream_t s) : dm(d), own(d ? d->stream : nullptr) {
        if (dm) dm->stream = s;
    }
    ~StreamLoan() {
        if (dm) dm->stream = own;
    }
};

// Speculative generation: generate()'s group loop with k + 1 rows per live stream. Each step is k_spec_draft -> passes
// -> pick_rows (overrides, automaton masks, pick) -> k_spec_accept (-> k_spec_logprob); at each group's end the records
// come back and the finished streams leave the rows. At the end a stream whose home is a spare has it copied to its first
// slot. With a stop request, k_spec_accept also walks each emitted token through the stream's stop set; with token
// automata, k_spec_draft gives each row its state and k_spec_accept advances the automaton; with logprobs_out, each
// emitted token is scored after k_spec_accept. With sr.drafter (generate_streams_drafted) each step's drafts come from
// the draft model's passes (draft_step) on this call's CUDA stream, and the call ends with draft_flush.
int speculate(M *m, const char *what, const GenCall &c, const SpecRequest &sr, const LogprobRequest *lpq,
              const ConstraintRequest *cq, const rwkv_b200_stop_request *sq) {
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (lpq && (rc = check_logprobs(what, *lpq))) return rc;
    const unsigned draft = sr.draft, ngram = sr.ngram;
    if (draft < 1 || draft > (unsigned)rk::kSpecMaxDraft) return fail(1, "%s: draft %u is outside 1..%d", what, draft, rk::kSpecMaxDraft);
    if (!sr.drafter && (ngram < 1 || ngram > (unsigned)rk::kSpecMaxNgram))
        return fail(1, "%s: ngram %u is outside 1..%d", what, ngram, rk::kSpecMaxNgram);
    if (!rk::prefill_enabled(m->pf)) return fail(1, "%s: needs the tensor cores (the \"prefill\" option is 0)", what);
    const unsigned long long K1 = draft + 1ull, S = c.n_streams, max_new = c.max_new;
    if (S > m->max_gpt / K1)
        return fail(1, "%s: %llu streams x %llu rows > max_gpt %llu", what, S, K1, m->max_gpt);
    // steps_out joins check_gen's required arrays, in its message
    if (S && (!c.slots || !c.first_tokens || !c.tokens_out || !c.lengths_out || !sr.steps_out))
        return fail(1, "%s: null argument (slots, first_tokens, tokens_out, lengths_out and steps_out are required)", what);
    if ((rc = check_gen(m, what, c, K1, true))) return rc;
    for (unsigned long long s = 0; s < S; ++s)
        if ((rc = check_same_binding(m, what, "stream", s, c.slots + s * K1, K1))) return rc;
    bool bound;
    if ((rc = set_pass_adapters(m, what, c.slots, S * K1, bound))) return rc;
    for (unsigned long long s = 0; c.samplers && s < S; ++s)
        if (c.samplers[s].presence_penalty != 0.0f || c.samplers[s].frequency_penalty != 0.0f)
            return fail(1, "%s: stream %llu: presence and frequency penalties are not supported (a row's counts would have "
                           "to include its own drafts)", what, s);
    const unsigned long long *context_start = sr.context_start, *context = sr.context;
    unsigned long long n_ctx = 0;
    if (context_start) {
        if (context_start[0] != 0) return fail(1, "%s: context_start[0] = %llu, not 0", what, context_start[0]);
        for (unsigned long long s = 0; s < S; ++s)
            if (context_start[s + 1] < context_start[s])
                return fail(1, "%s: context_start decreases from stream %llu to %llu (%llu > %llu)", what, s, s + 1,
                            context_start[s], context_start[s + 1]);
        n_ctx = context_start[S];
        if (n_ctx && !context) return fail(1, "%s: %llu context tokens with NULL context", what, n_ctx);
        if ((rc = check_tokens(what, "context token", context, n_ctx))) return rc;
    }
    CallFeatures f;
    if ((rc = check_features(m, what, c, lpq, cq, sq, f))) return rc;
    if (sr.drafter && (rc = check_drafter(m, what, sr.drafter, S))) return rc;
    const unsigned long long n_hist = n_ctx + S * (1 + max_new);
    CK(cudaSetDevice(m->device));
    auto &g = m->gen;
    const int per_pass = rk::kPfMaxTokens / (int)K1; // streams per pass: a stream's rows never straddle two passes
    const size_t n_pass = (size_t)((S + per_pass - 1) / per_pass);
    if ((rc = g.ss.grow(S)) || (rc = g.hist.grow(n_hist)) || (rc = g.live.grow(S)) || (rc = m->spec_passes.grow(n_pass)) ||
        (c.u && ((rc = g.su.grow(max_new * S)) || (rc = g.u.grow(S * K1)))) || (rc = g.forks.grow(2 * S)) ||
        (f.constrained && (rc = g.row_state.grow(S * K1))) || (lpq && (rc = g.score.grow(S * K1))))
        return rc;
    if ((rc = rk::prefill_init(m->pf, m->p))) return fail(rc, "%s", rk::prefill_error());
    m->stream_rows = 0; // the compact logits rows no longer belong to a call the caller made
    // k_spec_draft fills the tokens, descriptors and row maps only: the rest of each pass (no snapshots) stays zero
    CK(cudaMemsetAsync(m->spec_passes.p, 0, n_pass * sizeof(rk::PassDesc), m->stream));

    // the records and the histories: stream s's history starts with its context and its first token
    std::vector<rk::SpecStream> hs(S);
    std::vector<unsigned long long> hist(n_hist, 0); // stream s: its context, its first token, then room for max_new
    for (unsigned long long s = 0, h0 = 0; s < S; ++s) {
        rk::SpecStream &r = hs[s];
        r = rk::SpecStream{};
        for (unsigned long long i = 0; i < K1; ++i) r.slot[i] = c.slots[s * K1 + i];
        const unsigned long long c0 = context_start ? context_start[s] : 0, c1 = context_start ? context_start[s + 1] : 0;
        r.h0 = h0;
        r.hl = c1 - c0 + 1;
        r.budget = c.budgets ? c.budgets[s] : max_new;
        r.u0 = s;
        r.k = (int)draft;
        r.ngram = (int)ngram;
        std::copy(context + c0, context + c1, hist.begin() + h0);
        hist[h0 + c1 - c0] = c.first_tokens[s];
        h0 += r.hl + max_new;
    }
    CK(cudaMemcpyAsync(g.hist.p, hist.data(), n_hist * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(g.ss.p, hs.data(), S * sizeof(rk::SpecStream), cudaMemcpyHostToDevice, m->stream));
    if ((rc = upload_gen(m, c))) return rc;
    if (c.u) CK(cudaMemcpyAsync(g.su.p, c.u, max_new * S * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    if ((rc = upload_features(m, f, S, S * K1))) return rc;

    std::vector<int> live(S), rs;
    std::vector<rk::SpecLive> lv;
    for (unsigned long long s = 0; s < S; ++s) live[s] = (int)s;
    StepArgs a;
    step_args(m, g, f, max_new, c.n_stop, a);
    a.sa.k = (int)draft;
    a.sa.passes = m->spec_passes.p;
    a.sa.u_stride = S;
    if (f.constrained) a.pc.row_state = g.row_state.p;
    // a draft model works on this call's stream once its own earlier work is done
    M *dm = sr.drafter ? sr.drafter->model : nullptr;
    if (dm) CK(cudaStreamSynchronize(dm->stream));
    StreamLoan loan(dm, m->stream);
    DraftStep dstep;
    if (dm && (rc = draft_setup(dm, sr.drafter->slots, S, (int)draft, a, dstep))) return rc;
    a.draft = dm ? &dstep : nullptr;
    // each step emits at least one token per live stream, so max_new steps finish every stream
    for (unsigned long long step = 0; !live.empty() && step < max_new;) {
        const int n_live = (int)live.size(), rows = n_live * (int)K1;
        const unsigned long long steps = std::min(kGenGroup, max_new - step);
        rs.resize(rows);
        for (int r = 0; r < rows; ++r) rs[r] = live[r / (int)K1];
        lv.resize(n_live);
        for (int li = 0; li < n_live; ++li)
            lv[li] = rk::SpecLive{live[li], li * (int)K1, li / per_pass * rk::kPfMaxTokens + li % per_pass * (int)K1};
        CK(cudaMemcpyAsync(g.live.p, lv.data(), n_live * sizeof(rk::SpecLive), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(g.row_stream.p, rs.data(), rows * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        if (dm) { // draft row li is live stream live[li]'s; its first passes hold per_first streams each
            CK(cudaMemcpyAsync(dm->gen.row_stream.p, live.data(), n_live * sizeof(int), cudaMemcpyHostToDevice, m->stream));
            const int pf = dstep.da.per_first;
            dstep.da.n = n_live;
            dstep.heads.assign((n_live + pf - 1) / pf, pf);
            dstep.heads.back() = n_live - (int)(dstep.heads.size() - 1) * pf;
        }
        for (unsigned long long k = 0; k < steps; ++k)
            if ((rc = run_step(m, f, a, a.sa.passes, rows, per_pass * (int)K1, nullptr, rows, n_live, c.u ? g.u.p : nullptr)))
                return rc;
        // the end of a group: which streams are done and any token without an edge (one synchronisation); drop the
        // finished streams from the rows
        if ((rc = end_group(m, what, f, hs.data(), g.ss.p, S * sizeof(rk::SpecStream)))) return rc;
        step += steps;
        live.erase(std::remove_if(live.begin(), live.end(), [&](int s) { return hs[s].done != 0; }), live.end());
    }
    if (dm && (rc = draft_flush(dstep, S))) return rc;
    // a home on a spare: its xy, aa, bb and dd go to the first slot (pp: no forward writes it)
    std::vector<unsigned long long> forks;
    for (unsigned long long s = 0; s < S; ++s)
        if (hs[s].home != 0) {
            forks.push_back(hs[s].slot[hs[s].home]);
            forks.push_back(hs[s].slot[0]);
        }
    if (!forks.empty() && (rc = copy_home(m, g, forks))) return rc;
    if ((rc = finish_features(m, f, c))) return rc;
    for (unsigned long long s = 0; s < S; ++s) {
        c.lengths_out[s] = hs[s].len;
        sr.steps_out[s] = hs[s].steps;
    }
    return 0;
}

using B = rwkv_b200_batcher;
using PC = rwkv_b200_prefix_cache;
int prefix_copy(PC *c, const std::vector<unsigned long long> &pairs, bool restore);
void prefix_pool(const PC *c, double *(&pool)[4]);

int check_batcher(const B *b) {
    if (!b) return fail(1, "null batcher handle");
    return check_model(b->m);
}

// The batcher's request `id` into *out, after the handle checks; an unknown id is an error naming the call.
int find_req(B *b, const char *what, unsigned long long id, B::Req **out) {
    if (int rc = check_batcher(b)) return rc;
    const auto it = b->reqs.find(id);
    if (it == b->reqs.end()) return fail(1, "%s: request %llu is unknown or released", what, id);
    *out = &it->second;
    return 0;
}

// The unfinished request that holds `slot` as its slot or a spare (0: none).
unsigned long long slot_holder(const B *b, unsigned long long slot) {
    for (const auto &e : b->reqs) {
        const B::Req &o = e.second;
        if (o.status <= RWKV_B200_REQ_GENERATING &&
            (o.slot == slot || std::find(o.spares.begin(), o.spares.end(), slot) != o.spares.end()))
            return e.first;
    }
    return 0;
}

// A group boundary (the previous group's finished requests have left): queued requests are admitted in submission
// order while fewer than `rows` are admitted (each takes the lowest free lane: its record, sampler, penalty rows,
// automaton and scoring are reset), and every admitted request whose prefill is complete gets its decode row's records
// (stream, automaton, scoring). Returns the decode rows' lanes in admission order.
int batcher_boundary(B *b, std::vector<int> &dec) {
    M *m = b->m;
    const size_t V = binfmt::kVocab;
    auto &ad = b->admitted;
    std::map<PC *, std::vector<unsigned long long>> restores; // per cache, the {entry, slot} pairs of its admissions
    while (!b->queue.empty() && ad.size() < (size_t)b->rows) {
        const unsigned long long id = b->queue.front();
        b->queue.pop_front();
        B::Req &q = b->reqs[id];
        if (q.cache) { // the longest cached prefix of prompt[0 .. n_prompt - 1), restored before the group's passes
            long e = -1;
            prefix::Index &ix = q.cache->index;
            q.fed = q.cached = ix.lookup(slot_binding(m, q.slot), q.prompt.data(), q.prompt.size() - 1, &e);
            ix.stats().prefilled_tokens += q.prompt.size() - 1 - q.cached;
            restores[q.cache].insert(restores[q.cache].end(), {e >= 0 ? (unsigned long long)e : rk::kPrefixZero, q.slot});
        }
        q.lane = (int)(std::find(b->lane_used.begin(), b->lane_used.end(), 0) - b->lane_used.begin());
        b->lane_used[q.lane] = 1;
        q.status = RWKV_B200_REQ_PREFILLING;
        ad.push_back(id);
        b->h_gc[q.lane] = rk::GenConstraint{};
        b->h_lp[q.lane] = rk::LogprobLane{-1, 0};
        b->h_gst[q.lane] = rk::GenStop{};
        CK(cudaMemcpyAsync(b->bufs.samp.p + q.lane, &q.sampler, sizeof(rwkv_b200_sampler), cudaMemcpyHostToDevice, m->stream));
        if (q.sampler.presence_penalty != 0.0f || q.sampler.frequency_penalty != 0.0f) {
            int rc;
            if ((rc = b->bufs.pen_cnt.grow((size_t)b->rows * V)) || (rc = b->bufs.pen_seen.grow((size_t)b->rows * V))) return rc;
            CK(cudaMemsetAsync(b->bufs.pen_cnt.p + (size_t)q.lane * V, 0, V * sizeof(float), m->stream));
            CK(cudaMemsetAsync(b->bufs.pen_seen.p + (size_t)q.lane * V, 0, V, m->stream));
        }
    }
    for (auto &r : restores)
        if (int rc = prefix_copy(r.first, r.second, true)) return rc;
    dec.clear();
    for (unsigned long long id : ad) {
        B::Req &q = b->reqs[id];
        if (q.status == RWKV_B200_REQ_PREFILLING && q.fed + 1 == q.prompt.size()) {
            q.status = RWKV_B200_REQ_GENERATING;
            b->h_gs[q.lane] = rk::GenStream{q.slot, q.max_new, q.prompt.back(), 0, 0};
            b->h_gc[q.lane] = q.gc;
            b->h_lp[q.lane] = q.lp;
            b->h_gst[q.lane] = q.gst;
        }
        if (q.status == RWKV_B200_REQ_GENERATING) dec.push_back(q.lane);
    }
    // the lanes' lists in CSR over the lanes: the stop tokens of every admitted request, and the overrides of the decode
    // lanes, uploaded when one of them has some
    auto &bf = b->bufs;
    std::vector<const B::Req *> on(b->rows, nullptr);
    for (unsigned long long id : ad) on[b->reqs[id].lane] = &b->reqs[id];
    std::vector<unsigned long long> stop_start(b->rows + 1, 0), stop, ovr_start(b->rows + 1, 0), ovr_tok;
    std::vector<float> ovr_val;
    for (int l = 0; l < b->rows; ++l) {
        stop_start[l] = stop.size();
        ovr_start[l] = ovr_tok.size();
        if (const B::Req *q = on[l]) {
            stop.insert(stop.end(), q->stop.begin(), q->stop.end());
            if (q->status != RWKV_B200_REQ_GENERATING) continue;
            ovr_tok.insert(ovr_tok.end(), q->ovr_tok.begin(), q->ovr_tok.end());
            ovr_val.insert(ovr_val.end(), q->ovr_val.begin(), q->ovr_val.end());
        }
    }
    stop_start[b->rows] = stop.size();
    const size_t n_ovr = ovr_start[b->rows] = ovr_tok.size();
    int rc;
    if (n_ovr) {
        if ((rc = bf.ovr_tok.grow(n_ovr)) || (rc = bf.ovr_val.grow(n_ovr)) || (rc = bf.ovr_start.grow(b->rows + 1))) return rc;
        CK(cudaMemcpyAsync(bf.ovr_tok.p, ovr_tok.data(), n_ovr * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bf.ovr_val.p, ovr_val.data(), n_ovr * sizeof(float), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bf.ovr_start.p, ovr_start.data(), ovr_start.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice,
                           m->stream));
    }
    if ((rc = bf.stop.grow(stop.size()))) return rc;
    if (!stop.empty())
        CK(cudaMemcpyAsync(bf.stop.p, stop.data(), stop.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(bf.stop_start.p, stop_start.data(), stop_start.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice,
                       m->stream));
    return 0;
}

// A batcher group's host plan: each step's prefill segments, the decode rows and every step's passes.
struct GroupPlan {
    struct Seg {
        unsigned long long id, off, n;
    };
    std::vector<int> dec;                                 // the decode lanes, admission order (batcher_boundary)
    std::vector<std::vector<Seg>> segs;                   // [steps] each step's prefill segments
    std::map<unsigned long long, unsigned long long> fed; // each prefilling request's prompt tokens fed after the group
    std::vector<const B::Req *> of_lane;                  // [rows] the request of each lane
    std::vector<int> plain, rs;       // the one-token lanes (rows 0..Rp-1), the lane of each decode row
    std::vector<rk::SpecLive> sl;     // the speculative lanes
    int kmax = 0;                     // their largest k
    size_t ps = 0;                     // passes per step
    std::vector<rk::PassDesc> all;     // [steps][ps] every step's passes
    std::vector<int> step_rows;        // each step's tokens
    std::vector<std::vector<int>> H;   // each step's head rows per pass
    StepFlags f;                       // what the decode lanes use (batcher_upload)
    size_t W = 0, ring = 0;            // each lane's ring of tokens of the group, and all of them
    unsigned long long steps() const { return segs.size(); }
    int rows() const { return (int)rs.size(); } // logits rows of a step
};

// The host plan of a group of at most max_steps steps after its boundary (g.dec).
void batcher_plan(B *b, unsigned long long max_steps, GroupPlan &g) {
    // the prefill segments of each step: the budget goes to the prefilling requests in admission order
    for (unsigned long long id : b->admitted)
        if (b->reqs[id].status == RWKV_B200_REQ_PREFILLING) g.fed[id] = b->reqs[id].fed;
    for (unsigned long long k = 0; k < max_steps; ++k) {
        std::vector<GroupPlan::Seg> s;
        unsigned long long budget = (unsigned long long)b->prefill_tokens;
        for (unsigned long long id : b->admitted) {
            const B::Req &q = b->reqs[id];
            if (q.status != RWKV_B200_REQ_PREFILLING || budget == 0) continue;
            const unsigned long long take = std::min(budget, q.prompt.size() - 1 - g.fed[id]);
            if (take == 0) continue;
            s.push_back(GroupPlan::Seg{id, g.fed[id], take});
            g.fed[id] += take;
            budget -= take;
        }
        if (g.dec.empty() && s.empty()) break; // nothing left for this group's steps to do
        g.segs.push_back(std::move(s));
    }
    // the decode rows: the one-token lanes first (rows 0..Rp-1, where k_gen_feedback writes them), then k + 1 rows per
    // speculative lane, each lane's rows inside one pass: pad tokens (no head, no state stored) fill up a pass a lane
    // would straddle
    g.of_lane.assign(b->rows, nullptr);
    for (unsigned long long id : b->admitted) g.of_lane[b->reqs[id].lane] = &b->reqs[id];
    for (int l : g.dec)
        if (!g.of_lane[l]->draft) g.plain.push_back(l);
    g.rs = g.plain;
    std::vector<unsigned long long> dtok, dslot;
    std::vector<unsigned char> dhead;
    std::vector<int> pads;
    for (int l : g.plain) {
        dtok.push_back(b->h_gs[l].tok); // steps > 0: the feedback writes the pick over it
        dslot.push_back(b->h_gs[l].slot);
        dhead.push_back(1);
    }
    for (int l : g.dec) {
        const B::Req &q = *g.of_lane[l];
        if (!q.draft) continue;
        const int K1 = (int)q.draft + 1;
        g.kmax = std::max(g.kmax, (int)q.draft);
        while ((int)dtok.size() % rk::kPfMaxTokens + K1 > rk::kPfMaxTokens) {
            pads.push_back((int)dtok.size());
            dtok.push_back(0);
            dslot.push_back(q.slot);
            dhead.push_back(0);
        }
        g.sl.push_back(rk::SpecLive{l, (int)g.rs.size(), (int)dtok.size()});
        for (int i = 0; i < K1; ++i) { // k_spec_draft writes the tokens and descriptors
            g.rs.push_back(l);
            dtok.push_back(0);
            dslot.push_back(q.slot);
            dhead.push_back(1);
        }
    }
    // a speculative lane emits up to kGenGroup (k + 1) tokens in a group
    g.W = g.sl.empty() ? kGenGroup : kGenGroup * (rk::kSpecMaxDraft + 1);
    g.ring = (size_t)b->rows * g.W;
    // every step's layout: the decode rows, then the segments without a head
    const unsigned long long steps = g.steps();
    std::vector<std::vector<rk::PassDesc>> lay(steps);
    g.step_rows.resize(steps);
    g.H.resize(steps);
    g.ps = (size_t)b->max_pass;
    std::vector<PC *> snapped; // caches with entries pinned by this group's layouts
    for (unsigned long long k = 0; k < steps; ++k) {
        std::vector<unsigned long long> tokens(dtok), slots(dslot), lens(dtok.size(), 1);
        std::vector<unsigned char> head(dhead);
        std::vector<size_t> seg0; // each segment's first token in the step
        for (const GroupPlan::Seg &s : g.segs[k]) {
            const B::Req &q = b->reqs[s.id];
            seg0.push_back(tokens.size());
            tokens.insert(tokens.end(), q.prompt.begin() + (long)s.off, q.prompt.begin() + (long)(s.off + s.n));
            slots.push_back(q.slot);
            lens.push_back(s.n);
            head.push_back(0);
        }
        g.step_rows[k] = (int)tokens.size();
        rk::pass_layout(tokens.data(), g.step_rows[k], slots.data(), lens.data(), 2, nullptr, lay[k], g.H[k], head.data());
        for (int p : pads) lay[k][p / rk::kPfMaxTokens].desc[p % rk::kPfMaxTokens] &= ~rk::kDescLast;
        // snapshots of cached requests at block multiples and at n_prompt - 1 inside their segments. A pass carries one
        // pool: a snapshot into a second cache's pool in the same pass is skipped (and counted)
        for (size_t i = 0; i < g.segs[k].size(); ++i) {
            const GroupPlan::Seg &sg = g.segs[k][i];
            const B::Req &q = b->reqs[sg.id];
            if (!q.cache) continue;
            double *pool[4];
            prefix_pool(q.cache, pool);
            for (unsigned long long pos = sg.off + 1; pos <= sg.off + sg.n; ++pos) {
                if (pos % q.cache->block != 0 && pos + 1 != q.prompt.size()) continue;
                const size_t t = seg0[i] + (size_t)(pos - sg.off - 1);
                rk::PassDesc &pd = lay[k][t / rk::kPfMaxTokens];
                if (pd.pool[0] && pd.pool[0] != pool[0]) {
                    q.cache->index.stats().skipped += 1;
                    continue;
                }
                bool fresh = false;
                const long e = q.cache->index.take(slot_binding(b->m, q.slot), q.prompt.data(), (size_t)pos, &fresh);
                if (std::find(snapped.begin(), snapped.end(), q.cache) == snapped.end()) snapped.push_back(q.cache);
                if (e < 0 || !fresh) continue;
                pd.snap[t % rk::kPfMaxTokens] = (uint32_t)e + 1u;
                std::copy(pool, pool + 4, pd.pool);
            }
        }
        g.ps = std::max(g.ps, lay[k].size());
    }
    for (PC *c : snapped) c->index.unpin_all();
    g.all.resize(steps * g.ps);
    for (unsigned long long k = 0; k < steps; ++k) std::copy(lay[k].begin(), lay[k].end(), g.all.begin() + k * g.ps);
}

// The upload of a group: its passes, the decode lanes' records, row map and uniforms, and the buffers of the features
// they use (g.f), each enqueued only when one of them needs it.
int batcher_upload(B *b, GroupPlan &g) {
    M *m = b->m;
    auto &bf = b->bufs;
    const unsigned long long steps = g.steps();
    const int NR = g.rows(), Rp = (int)g.plain.size();
    int rc;
    if ((rc = bf.passes.grow(kGenGroup * g.ps)) || (rc = bf.row_stream.grow(NR)) || (rc = bf.u.grow(kGenGroup * NR)) ||
        (rc = bf.out.grow(g.ring)))
        return rc;
    b->h_out.resize(g.ring);
    CK(cudaMemcpyAsync(bf.passes.p, g.all.data(), g.all.size() * sizeof(rk::PassDesc), cudaMemcpyHostToDevice, m->stream));
    StepFlags &f = g.f;
    f.samplers = f.uniforms = true; // every lane has a sampler; a request without uniforms draws zeros
    for (int l : g.dec) {
        const B::Req &q = *g.of_lane[l];
        f.n_override += q.ovr_tok.size();
        f.pen |= q.sampler.presence_penalty != 0.0f || q.sampler.frequency_penalty != 0.0f;
        f.constrained |= q.gc.mask != nullptr;
        f.stopped |= q.gst.next != nullptr;
        if (q.lp.mode >= 0) {
            (q.draft ? f.spec_scored : f.scored) = true;
            f.raw |= q.lp.mode == RWKV_B200_LOGPROBS_RAW;
            if (q.lp.top_n) f.top = rk::kMaxTopN; // each lane's top entries at its own stride
        }
    }
    set_raw_copy(f);
    if (!g.dec.empty()) {
        CK(cudaMemcpyAsync(bf.gs.p, b->h_gs.data(), b->rows * sizeof(rk::GenStream), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bf.row_stream.p, g.rs.data(), NR * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        // uniforms [steps][NR]: one-token row r at step k draws with its request's u[len + k] (k_spec_draft writes the
        // speculative rows')
        std::vector<double> ug(steps * (size_t)NR, 0.0);
        for (int r = 0; r < Rp; ++r) {
            const rk::GenStream &gs = b->h_gs[g.plain[r]];
            const B::Req &q = *g.of_lane[g.plain[r]];
            for (unsigned long long k = 0; k < steps && !q.u.empty(); ++k)
                if (gs.len + k < q.max_new) ug[k * NR + r] = q.u[gs.len + k];
        }
        CK(cudaMemcpyAsync(bf.u.p, ug.data(), ug.size() * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    }
    const size_t V = binfmt::kVocab, top_ring = g.ring * f.top;
    if (f.constrained) {
        if ((rc = bf.gc.grow(b->rows)) || (rc = bf.fault.grow(3))) return rc;
        CK(cudaMemcpyAsync(bf.gc.p, b->h_gc.data(), b->rows * sizeof(rk::GenConstraint), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemsetAsync(bf.fault.p, 0, 3 * sizeof(unsigned long long), m->stream));
    }
    if (f.stopped) {
        if ((rc = bf.gst.grow(b->rows))) return rc;
        CK(cudaMemcpyAsync(bf.gst.p, b->h_gst.data(), b->rows * sizeof(rk::GenStop), cudaMemcpyHostToDevice, m->stream));
    }
    // the speculative lanes' records, histories (context ++ prompt ++ emitted, with room for the rest) and uniforms
    if (!g.sl.empty()) {
        std::vector<unsigned long long> hist;
        std::vector<double> su;
        for (const rk::SpecLive &e : g.sl) {
            const B::Req &q = *g.of_lane[e.s];
            rk::SpecStream &r = b->h_ss[e.s];
            r = rk::SpecStream{};
            r.slot[0] = q.slot;
            std::copy(q.spares.begin(), q.spares.end(), r.slot + 1);
            r.h0 = hist.size();
            hist.insert(hist.end(), q.context.begin(), q.context.end());
            hist.insert(hist.end(), q.prompt.begin(), q.prompt.end());
            hist.insert(hist.end(), q.tokens.begin(), q.tokens.end());
            r.hl = hist.size() - r.h0;
            hist.resize(hist.size() + q.max_new - q.tokens.size());
            r.budget = q.max_new;
            r.len = q.tokens.size();
            r.steps = q.steps;
            r.u0 = su.size();
            su.resize(su.size() + q.max_new, 0.0);
            std::copy(q.u.begin(), q.u.end(), su.begin() + (long)r.u0);
            r.home = q.home;
            r.k = (int)q.draft;
            r.ngram = (int)q.ngram;
        }
        if ((rc = bf.ss.grow(b->rows)) || (rc = bf.live.grow(b->rows)) || (rc = bf.hist.grow(hist.size())) ||
            (rc = bf.su.grow(su.size())) || (f.constrained && (rc = bf.row_state.grow(NR))) ||
            (f.spec_scored && (rc = bf.score.grow(g.sl.size() * (g.kmax + 1)))))
            return rc;
        CK(cudaMemcpyAsync(bf.ss.p, b->h_ss.data(), b->rows * sizeof(rk::SpecStream), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bf.live.p, g.sl.data(), g.sl.size() * sizeof(rk::SpecLive), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bf.hist.p, hist.data(), hist.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bf.su.p, su.data(), su.size() * sizeof(double), cudaMemcpyHostToDevice, m->stream));
        if (f.constrained) { // the one-token rows are masked by their lane's record; k_spec_draft writes the others
            const std::vector<unsigned long long> st(NR, rk::kStreamState);
            CK(cudaMemcpyAsync(bf.row_state.p, st.data(), NR * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
        }
    }
    // raw lanes read the model's rows: d_slogits itself, or a copy taken before the penalties, overrides and masks edit it
    if (f.scored || f.spec_scored) {
        if ((rc = bf.lp_lane.grow(b->rows)) || (rc = bf.lp.grow(g.ring)) || (rc = bf.rank.grow(g.ring)) ||
            (rc = bf.top_lp.grow(top_ring)) || (rc = bf.top_tok.grow(top_ring)) || (f.raw_copy && (rc = bf.raw.grow((size_t)NR * V))))
            return rc;
        CK(cudaMemcpyAsync(bf.lp_lane.p, b->h_lp.data(), b->rows * sizeof(rk::LogprobLane), cudaMemcpyHostToDevice, m->stream));
    }
    return 0;
}

// The end of a group: the lanes' records and the tokens of the group (with their results and the automata's states when
// a lane uses them) come back with one synchronisation and go to their requests; finished speculative requests have
// their home copied to their slot, and finished requests leave.
int batcher_collect(B *b, GroupPlan &g) {
    M *m = b->m;
    const auto &bf = b->bufs;
    const StepFlags &f = g.f;
    const size_t W = g.W, ring = g.ring, top_ring = ring * f.top;
    unsigned long long fault[3] = {0, 0, 0};
    if (!g.dec.empty()) {
        CK(cudaMemcpyAsync(b->h_gs.data(), bf.gs.p, b->rows * sizeof(rk::GenStream), cudaMemcpyDeviceToHost, m->stream));
        CK(cudaMemcpyAsync(b->h_out.data(), bf.out.p, ring * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
    }
    if (!g.sl.empty())
        CK(cudaMemcpyAsync(b->h_ss.data(), bf.ss.p, b->rows * sizeof(rk::SpecStream), cudaMemcpyDeviceToHost, m->stream));
    if (f.constrained)
        CK(cudaMemcpyAsync(b->h_gc.data(), bf.gc.p, b->rows * sizeof(rk::GenConstraint), cudaMemcpyDeviceToHost, m->stream));
    int rc;
    if ((rc = read_fault(m, bf, f.constrained, fault))) return rc;
    if (f.stopped) CK(cudaMemcpyAsync(b->h_gst.data(), bf.gst.p, b->rows * sizeof(rk::GenStop), cudaMemcpyDeviceToHost, m->stream));
    if (f.scored || f.spec_scored) {
        b->h_lpv.resize(ring);
        b->h_rank.resize(ring);
        b->h_top_lp.resize(top_ring);
        b->h_top_tok.resize(top_ring);
        CK(cudaMemcpyAsync(b->h_lpv.data(), bf.lp.p, ring * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        CK(cudaMemcpyAsync(b->h_rank.data(), bf.rank.p, ring * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        if (f.top) {
            CK(cudaMemcpyAsync(b->h_top_lp.data(), bf.top_lp.p, top_ring * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
            CK(cudaMemcpyAsync(b->h_top_tok.data(), bf.top_tok.p, top_ring * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        }
    }
    SYNC(m);
    if (fault[0]) {
        unsigned long long rid = 0;
        for (unsigned long long id : b->admitted)
            if (b->reqs[id].lane == (int)(fault[0] - 1)) rid = id;
        return fail(8, "batcher_run: request %llu emitted token %llu, which has no edge out of state %llu of its constraint", rid,
                    fault[1], fault[2]);
    }
    std::vector<unsigned long long> forks; // finished speculative requests whose home is a spare: home -> slot
    for (unsigned long long id : b->admitted) {
        B::Req &q = b->reqs[id];
        if (q.status == RWKV_B200_REQ_PREFILLING) {
            q.fed = g.fed[id];
            continue;
        }
        const rk::SpecStream &e = b->h_ss[q.lane];
        const unsigned long long len = q.draft ? e.len : b->h_gs[q.lane].len;
        for (unsigned long long j = q.tokens.size(); j < len; ++j) {
            const size_t x = (size_t)q.lane * W + j % W;
            q.tokens.push_back(b->h_out[x]);
            if (q.lp.mode < 0) continue;
            q.logprobs.push_back(b->h_lpv[x]);
            q.ranks.push_back(b->h_rank[x]);
            for (int t = 0; t < q.lp.top_n; ++t) {
                q.top_tokens.push_back(b->h_top_tok[x * rk::kMaxTopN + t]);
                q.top_logprobs.push_back(b->h_top_lp[x * rk::kMaxTopN + t]);
            }
        }
        if (q.gc.mask) q.gc.state = b->h_gc[q.lane].state;
        if (q.gst.next) q.gst = b->h_gst[q.lane];
        if (q.draft) {
            q.steps = e.steps;
            q.home = e.home;
        }
        if (q.draft ? e.done : b->h_gs[q.lane].done) {
            q.status = RWKV_B200_REQ_DONE;
            if (q.home) {
                forks.push_back(e.slot[q.home]);
                forks.push_back(q.slot);
                q.home = 0;
            }
        }
    }
    if (!forks.empty() && (rc = copy_home(m, b->bufs, forks))) return rc;
    // finished requests leave here, before the next boundary admits anyone (a caller may release them in between)
    auto &ad = b->admitted;
    ad.erase(std::remove_if(ad.begin(), ad.end(),
                            [&](unsigned long long id) {
                                const B::Req &q = b->reqs.at(id);
                                if (q.status != RWKV_B200_REQ_DONE) return false;
                                b->lane_used[q.lane] = 0;
                                return true;
                            }),
             ad.end());
    return 0;
}

// One group of at most `max_steps` steps (<= kGenGroup); *ran receives its length. The host lays out every step's
// passes in advance (prefill never depends on a pick) and uploads them once; the feedback of step k writes the decode
// rows' tokens and kDescLast bits into step k + 1's layout.
int batcher_group(B *b, unsigned long long max_steps, unsigned long long *ran) {
    M *m = b->m;
    GroupPlan g;
    int rc = batcher_boundary(b, g.dec);
    if (rc) return rc;
    *ran = 0;
    if (b->admitted.empty()) return 0;
    // the group's passes add adapter deltas when an admitted request's slot is bound (its spares share the binding)
    m->pf.adapt = false;
    m->pf.ad_table = m->ad_table.p;
    for (unsigned long long id : b->admitted) m->pf.adapt |= slot_binding(m, b->reqs[id].slot) != RWKV_B200_NO_ADAPTER;
    batcher_plan(b, max_steps, g);
    if ((rc = batcher_upload(b, g))) return rc;
    const unsigned long long steps = g.steps();
    const int NR = g.rows();
    auto &bf = b->bufs;
    StepArgs a;
    step_args(m, bf, g.f, g.W, 0, a);
    a.fb.rows = (int)g.plain.size();
    a.sa.k = g.kmax;
    a.sa.u_stride = 1;
    if (!g.sl.empty() && g.f.constrained) a.pc.row_state = bf.row_state.p;
    for (unsigned long long k = 0; k < steps; ++k) {
        rk::PassDesc *passes = bf.passes.p + k * g.ps;
        a.sa.passes = passes;
        a.sa.row_u = bf.u.p + k * NR;
        a.fb.passes = k + 1 < steps ? passes + g.ps : nullptr;
        if ((rc = run_step(m, g.f, a, passes, g.step_rows[k], rk::kPfMaxTokens, g.H[k].data(), NR, (int)g.sl.size(), a.sa.row_u)))
            return rc;
    }
    if ((rc = batcher_collect(b, g))) return rc;
    *ran = steps;
    return 0;
}

} // namespace

// =================================================================================================
// C ABI
// =================================================================================================
// ---- prefix state cache (csrc/prefix.cuh, csrc/prefix_index.h) -----------------------------------------------------
namespace {
// The base pointers of the pool's xy, aa, bb and dd arrays.
void prefix_pool(const PC *c, double *(&pool)[4]) {
    const size_t per = c->index.capacity() * (size_t)(c->m->L * c->m->E);
    for (int i = 0; i < 4; ++i) pool[i] = c->pool.p + i * per;
}

int check_cache(PC *c, const char *what) {
    if (!c) return fail(1, "%s: null prefix cache handle", what);
    return check_streams_model(c->m, what);
}

// k_prefix_copy over the {entry, slot} pairs (kPrefixZero: the zero state): restore = entry -> slot, else slot -> entry
int prefix_copy(PC *c, const std::vector<unsigned long long> &pairs, bool restore) {
    M *m = c->m;
    const unsigned long long n = pairs.size() / 2;
    if (n == 0) return 0;
    CK(cudaMemcpyAsync(c->pairs.p, pairs.data(), pairs.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    rk::PrefixCopyArgs a{};
    const size_t LE = (size_t)(m->L * m->E);
    prefix_pool(c, a.pool);
    slot_arrays(m, 0, a.slot);
    a.LE = LE;
    a.pairs = c->pairs.p;
    a.restore = restore ? 1 : 0;
    rk::k_prefix_copy<<<rk::prefix_copy_grid(LE, restore, n), rk::kPrefixThreads, 0, m->stream>>>(a);
    LAUNCHED(m);
    return 0;
}

// The ragged call of rwkv_b200_prefix_forward after its checks. The index changes before the device work is enqueued,
// so a call that fails after that point clears it: no entry may promise a state that was never written.
int prefix_forward(PC *c, const unsigned long long *tokens, const unsigned long long *slots, const unsigned long long *lengths,
                   unsigned long long S, bool head, std::vector<unsigned long long> &cached) {
    M *m = c->m;
    prefix::Index &ix = c->index;
    std::vector<unsigned long long> pairs(2 * S), rtok, rslot, rlen, off(S);
    std::vector<long> hit(S);
    for (unsigned long long s = 0, o = 0; s < S; o += lengths[s], ++s) {
        off[s] = o;
        cached[s] = ix.lookup(slot_binding(m, slots[s]), tokens + o, lengths[s] - (head ? 1 : 0), &hit[s]);
        pairs[2 * s] = hit[s] >= 0 ? (unsigned long long)hit[s] : rk::kPrefixZero;
        pairs[2 * s + 1] = slots[s];
        if (cached[s] == lengths[s]) continue; // state only and fully cached: no token runs
        rtok.insert(rtok.end(), tokens + o + cached[s], tokens + o + lengths[s]);
        rslot.push_back(slots[s]);
        rlen.push_back(lengths[s] - cached[s]);
    }
    const int n = (int)rtok.size();
    std::vector<rk::PassDesc> passes;
    std::vector<int> heads;
    if (n > 0) rk::pass_layout(rtok.data(), n, rslot.data(), rlen.data(), head ? 2 : 0, nullptr, passes, heads);
    // snapshots: the state after p tokens, for p in (cached, length] at multiples of the block and at the length
    for (unsigned long long s = 0, g0 = 0; s < S; ++s) {
        const unsigned long long r = cached[s], len = lengths[s];
        for (unsigned long long p = r + 1; p <= len; ++p) {
            if (p % c->block != 0 && p != len) continue;
            bool fresh = false;
            const long e = ix.take(slot_binding(m, slots[s]), tokens + off[s], (size_t)p, &fresh);
            if (e < 0 || !fresh) continue;
            const unsigned long long g = g0 + (p - r - 1); // its token in the remainder list
            passes[g / rk::kPfMaxTokens].snap[g % rk::kPfMaxTokens] = (uint32_t)e + 1u;
        }
        g0 += len - r;
    }
    ix.unpin_all();
    ix.stats().prefilled_tokens += (unsigned long long)n;
    for (rk::PassDesc &pd : passes) prefix_pool(c, pd.pool);
    int rc = prefix_copy(c, pairs, true);
    if (!rc && n > 0) {
        rc = rk::prefill_passes(m->pf, m->p, m->stream, passes, heads, n, m->d_slogits);
        if (rc) rc = fail(rc, "%s", rk::prefill_error());
        m->launches += rk::prefill_launches(m->pf);
    }
    if (rc) ix.clear();
    return rc;
}
} // namespace

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
    rwkv_b200_batcher_close(m->batcher);
    while (!m->prefix_caches.empty()) rwkv_b200_prefix_cache_close(m->prefix_caches.back());
    rk::prefill_free(m->pf);
    for (void *p : m->ipc_opened) cudaIpcCloseMemHandle(p);
    for (void *p : m->allocs) cudaFree(p);
    if (m->h_ctrl) cudaFreeHost(m->h_ctrl);
    if (m->h_logits) cudaFreeHost(m->h_logits);
    if (m->h_next) cudaFreeHost(m->h_next);
    if (m->h_sample) cudaFreeHost(m->h_sample);
    if (m->h_diag) cudaFreeHost(m->h_diag);
    if (m->h_gs) cudaFreeHost(m->h_gs);
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
    if ((rc = check_unbound(m, "forward", slots.data(), slots.size()))) return rc;
    m->pf.adapt = false;
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
    const unsigned long long slot0 = 0;
    if ((rc = check_unbound(m, "forward_greedy", &slot0, 1))) return rc;
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
    LAUNCHED(m);
    return read_samples(m, 1, token, margin);
}

int rwkv_b200_forward_streams(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n_tokens,
                              const unsigned long long *slots, const unsigned long long *lengths,
                              unsigned long long n_streams, float *logits_out, unsigned long long *next_out) {
    int rc = check_ragged(m, "forward_streams", tokens, n_tokens, slots, lengths, n_streams);
    if (rc) return rc;
    bool bound;
    if ((rc = set_pass_adapters(m, "forward_streams", slots, n_streams, bound))) return rc;
    const size_t V = binfmt::kVocab;
    CK(cudaSetDevice(m->device));
    const bool head = logits_out || next_out;
    m->stream_rows = 0;
    if (tensor_cores(m, n_tokens, bound)) {
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
        LAUNCHED(m);
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
    LAUNCHED(m);
    return read_samples(m, n_streams, tokens_out, margins_out);
}

int rwkv_b200_generate_streams(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                               unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                               const unsigned long long *stop_tokens, unsigned long long n_stop,
                               const unsigned long long *override_tokens, const float *override_values,
                               unsigned long long n_override, float temp, const double *u, unsigned long long *tokens_out,
                               unsigned long long *lengths_out) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, nullptr, u, tokens_out, lengths_out};
    return generate(m, "generate_streams", false, c, temp);
}

int rwkv_b200_generate_streams_ex(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                  unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                  const unsigned long long *stop_tokens, unsigned long long n_stop,
                                  const unsigned long long *override_tokens, const float *override_values,
                                  unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                  unsigned long long *tokens_out, unsigned long long *lengths_out) {
    // without samplers every stream takes the arg-max and u is not read
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    return generate(m, "generate_streams_ex", true, c, 1.0f);
}

int rwkv_b200_generate_streams_logprobs(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                        unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                        const unsigned long long *stop_tokens, unsigned long long n_stop,
                                        const unsigned long long *override_tokens, const float *override_values,
                                        unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                        unsigned long long *tokens_out, unsigned long long *lengths_out, int logprob_mode,
                                        unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
                                        unsigned long long *top_tokens_out, double *top_logprobs_out) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    return generate(m, "generate_streams_logprobs", true, c, 1.0f, &lpq);
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
    // the lane records of the model's batcher point into the automaton's device block
    if (const rwkv_b200_batcher *b = m->batcher)
        for (const auto &e : b->reqs)
            if (e.second.constraint_id == id && e.second.status <= RWKV_B200_REQ_GENERATING)
                return fail(1, "constraint_remove: constraint id %llu is named by unfinished request %llu of the model's batcher",
                            id, e.first);
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
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    const ConstraintRequest cq{constraint_ids, start_states, states_out};
    return generate(m, "generate_streams_constrained", true, c, 1.0f, logprobs_out ? &lpq : nullptr, &cq);
}

int rwkv_b200_token_bytes_set(rwkv_b200_model *m, const unsigned long long *start, const unsigned char *bytes) {
    const char *what = "token_bytes_set";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    const size_t V = binfmt::kVocab;
    if (!start) return fail(1, "%s: start is NULL", what);
    if (start[0] != 0) return fail(1, "%s: start[0] = %llu, not 0", what, start[0]);
    for (size_t v = 0; v < V; ++v)
        if (start[v + 1] < start[v])
            return fail(1, "%s: start decreases from token %zu to %zu (%llu > %llu)", what, v, v + 1, start[v], start[v + 1]);
    const unsigned long long n = start[V];
    if (n && !bytes) return fail(1, "%s: %llu bytes with NULL bytes", what, n);
    // the lane records of the model's batcher point into the table
    if (const rwkv_b200_batcher *b = m->batcher)
        for (const auto &e : b->reqs)
            if (e.second.gst.next && e.second.status <= RWKV_B200_REQ_GENERATING)
                return fail(1, "%s: unfinished request %llu of the model's batcher has a stop set", what, e.first);
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    if ((rc = m->tb_start.grow(V + 1)) || (rc = m->tb_bytes.grow(std::max<unsigned long long>(n, 1)))) {
        m->has_tb = false;
        return rc;
    }
    CK(cudaMemcpy(m->tb_start.p, start, (V + 1) * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    if (n) CK(cudaMemcpy(m->tb_bytes.p, bytes, n, cudaMemcpyHostToDevice));
    m->has_tb = true;
    return 0;
}

int rwkv_b200_stop_set_add(rwkv_b200_model *m, unsigned long long n_strings, const unsigned long long *string_start,
                           const unsigned char *bytes, unsigned long long *id) {
    const char *what = "stop_set_add";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!string_start || !bytes || !id) return fail(1, "%s: null argument (string_start, bytes and id are required)", what);
    if (n_strings == 0) return fail(1, "%s: no strings", what);
    if (string_start[0] != 0) return fail(1, "%s: string_start[0] = %llu, not 0", what, string_start[0]);
    for (unsigned long long i = 0; i < n_strings; ++i)
        if (string_start[i + 1] <= string_start[i]) return fail(1, "%s: string %llu is empty or its offsets decrease", what, i);
    if (string_start[n_strings] > RWKV_B200_MAX_STOP_BYTES)
        return fail(1, "%s: %llu bytes in total > %d", what, string_start[n_strings], RWKV_B200_MAX_STOP_BYTES);
    std::vector<uint32_t> next, hit;
    const uint32_t states = stopmatch::build(string_start, bytes, n_strings, next, hit);
    next.insert(next.end(), hit.begin(), hit.end()); // one block: next [states][256], then hit [states]
    M::StopSet ss;
    ss.states = states;
    CK(cudaSetDevice(m->device));
    if ((rc = ss.dev.grow(next.size()))) return rc;
    CK(cudaMemcpy(ss.dev.p, next.data(), next.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    *id = m->next_stop_set++;
    m->stop_sets.emplace(*id, std::move(ss));
    return 0;
}

int rwkv_b200_stop_set_remove(rwkv_b200_model *m, unsigned long long id) {
    int rc = check_model(m);
    if (rc) return rc;
    const auto it = m->stop_sets.find(id);
    if (it == m->stop_sets.end()) return fail(1, "stop_set_remove: stop set id %llu is unknown or removed", id);
    // the lane records of the model's batcher point into the set's device block
    if (const rwkv_b200_batcher *b = m->batcher)
        for (const auto &e : b->reqs)
            if (e.second.stop_set == id && e.second.status <= RWKV_B200_REQ_GENERATING)
                return fail(1, "stop_set_remove: stop set id %llu is named by unfinished request %llu of the model's batcher", id,
                            e.first);
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    m->stop_sets.erase(it);
    return 0;
}

int rwkv_b200_generate_streams_stop(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                    unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                    const unsigned long long *stop_tokens, unsigned long long n_stop,
                                    const unsigned long long *override_tokens, const float *override_values,
                                    unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                    unsigned long long *tokens_out, unsigned long long *lengths_out, int logprob_mode,
                                    unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
                                    unsigned long long *top_tokens_out, double *top_logprobs_out,
                                    const unsigned long long *constraint_ids, const unsigned long long *start_states,
                                    unsigned long long *states_out, const rwkv_b200_stop_request *stop) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    const ConstraintRequest cq{constraint_ids, start_states, states_out};
    return generate(m, stop ? "generate_streams_stop" : "generate_streams_constrained", true, c, 1.0f,
                    logprobs_out ? &lpq : nullptr, &cq, stop);
}

int rwkv_b200_generate_streams_guided(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                      unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                      const unsigned long long *stop_tokens, unsigned long long n_stop,
                                      const unsigned long long *override_tokens, const float *override_values,
                                      unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                      unsigned long long *tokens_out, unsigned long long *lengths_out, int logprob_mode,
                                      unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
                                      unsigned long long *top_tokens_out, double *top_logprobs_out,
                                      const unsigned long long *constraint_ids, const unsigned long long *start_states,
                                      unsigned long long *states_out, const rwkv_b200_stop_request *stop,
                                      const rwkv_b200_guidance *guidance) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    const ConstraintRequest cq{constraint_ids, start_states, states_out};
    const char *what = guidance ? "generate_streams_guided" : stop ? "generate_streams_stop" : "generate_streams_constrained";
    return generate(m, what, true, c, 1.0f, logprobs_out ? &lpq : nullptr, &cq, stop, guidance);
}

// Beam search: generate()'s group loop over beams. Step 0 has one row per group, later steps B rows per live group
// (group by group); each step is forward -> k_beam_expand -> k_beam_select -> k_beam_fork. At each host group's end the
// done flags come back and the done groups leave the rows; at the end the backpointers and the hypothesis lists come
// back once and the host rebuilds each hypothesis' tokens.
int rwkv_b200_beam_search(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                          unsigned long long n_groups, unsigned beams, unsigned long long max_new,
                          const unsigned long long *stop_tokens, unsigned long long n_stop, double length_penalty,
                          unsigned n_best, unsigned long long *tokens_out, unsigned long long *lengths_out,
                          double *logprobs_out, double *scores_out, unsigned char *finished_out,
                          double *token_logprobs_out) {
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
    for (unsigned long long g = 0; g < G; ++g)
        if ((rc = check_same_binding(m, what, "group", g, slots + g * B, B))) return rc;
    bool bound;
    if ((rc = set_pass_adapters(m, what, slots, G * B, bound))) return rc;
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
    const bool tc = tensor_cores(m, G * B, bound);
    if (tc && (rc = rk::prefill_init(m->pf, m->p))) return fail(rc, "%s", rk::prefill_error());
    m->stream_rows = 0; // the compact logits rows no longer belong to a call the caller made

    rk::GenStream *hg = m->h_gs;
    for (unsigned long long s = 0; s < G * B; ++s) hg[s] = rk::GenStream{slots[s], N, s % B == 0 ? first_tokens[s / B] : 0, 0, 0};
    std::vector<int> row0(G), live(G);
    for (unsigned long long i = 0; i < G; ++i) {
        row0[i] = (int)(i * B);
        live[i] = (int)i;
    }
    CK(cudaMemcpyAsync(g.gs.p, hg, G * B * sizeof(rk::GenStream), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(bm.row0.p, row0.data(), G * sizeof(int), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(bm.P.p, P.data(), (N + 1) * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    if (n_stop) CK(cudaMemcpyAsync(g.stop.p, stop_tokens, n_stop * sizeof(unsigned long long), cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemsetAsync(bm.cum.p, 0, G * B * sizeof(double), m->stream));
    CK(cudaMemsetAsync(bm.n_hyp.p, 0, G * sizeof(int), m->stream));
    CK(cudaMemsetAsync(bm.done.p, 0, G * sizeof(unsigned long long), m->stream));
    std::vector<unsigned long long> hdone(G, 0);
    std::vector<int> rs;
    for (unsigned long long step = 0; !live.empty() && step < N;) {
        // a host group: the live groups' beams are rows gi * B + j (step 0: row gi); their inputs go up once
        const int Gl = (int)live.size();
        const unsigned long long steps = std::min(kGenGroup, N - step);
        rs.resize((size_t)Gl * B);
        for (int gi = 0; gi < Gl; ++gi)
            for (unsigned long long j = 0; j < B; ++j) rs[gi * B + j] = (int)(live[gi] * B + j);
        CK(cudaMemcpyAsync(g.row_stream.p, rs.data(), rs.size() * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(bm.groups.p, live.data(), Gl * sizeof(int), cudaMemcpyHostToDevice, m->stream));
        if (tc && (rc = upload_step_passes(m, step == 0 ? row0.data() : rs.data(), step == 0 ? Gl : Gl * (int)B))) return rc;
        rk::BeamArgs ba{g.gs.p, bm.cum.p, bm.groups.p, bm.cand_tok.p, bm.cand_lp.p, (int)C, (int)B, (int)K, 0, 0, N, bm.P.p,
                        length_penalty < 0.0 ? 1 : 0, g.stop.p, (int)n_stop, bm.back.p, bm.hyp.p, bm.n_hyp.p, bm.done.p, bm.forks.p,
                        tc ? g.passes.p : nullptr};
        for (unsigned long long k = 0; k < steps; ++k) {
            const unsigned long long st = step + k;
            const int nb = st == 0 ? 1 : (int)B, rows = Gl * nb;
            const int *rmap = st == 0 ? bm.row0.p : g.row_stream.p;
            if ((rc = tc ? gen_step_passes(m, g.passes.p, rows, rk::kPfMaxTokens) : gen_step_decode(m, rows, rmap))) return rc;
            rk::k_beam_expand<<<(unsigned)rows, rk::kNucThreads, 0, m->stream>>>(m->d_slogits, (int)V, g.gs.p, rmap, (int)C,
                                                                                bm.cand_tok.p, bm.cand_lp.p);
            LAUNCHED(m);
            ba.step = (int)st;
            ba.nb = nb;
            rk::k_beam_select<<<(unsigned)Gl, rk::kBeamSelectThreads, 0, m->stream>>>(ba);
            LAUNCHED(m);
            // after the last step every group is done and forks nothing
            if (st + 1 < N && (rc = fork_slots(m, bm.forks.p, Gl * B, true))) return rc;
        }
        // the end of a host group: which groups are done and the beams' records (one synchronisation)
        CK(cudaMemcpyAsync(hdone.data(), bm.done.p, G * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        CK(cudaMemcpyAsync(hg, g.gs.p, G * B * sizeof(rk::GenStream), cudaMemcpyDeviceToHost, m->stream));
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

// The speculative entry points. A call that asks for none of an entry's features is named after the narrower entry
// that has only the features it uses.
int rwkv_b200_generate_streams_speculative_constrained(
    rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens, unsigned long long n_streams,
    unsigned long long max_new, const unsigned long long *budgets, const unsigned long long *stop_tokens, unsigned long long n_stop,
    const unsigned long long *override_tokens, const float *override_values, unsigned long long n_override,
    const rwkv_b200_sampler *samplers, const double *u, unsigned long long *tokens_out, unsigned long long *lengths_out,
    unsigned int draft, unsigned int ngram, const unsigned long long *context_start, const unsigned long long *context,
    unsigned long long *steps_out, int logprob_mode, unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
    unsigned long long *top_tokens_out, double *top_logprobs_out, const unsigned long long *constraint_ids,
    const unsigned long long *start_states, unsigned long long *states_out, const rwkv_b200_stop_request *sq) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    const ConstraintRequest cq{constraint_ids, start_states, states_out};
    return speculate(m, logprobs_out || constraint_ids ? "generate_streams_speculative_constrained"
                        : sq                           ? "generate_streams_speculative_stop"
                                                       : "generate_streams_speculative",
                     c, SpecRequest{draft, ngram, context_start, context, steps_out, nullptr}, logprobs_out ? &lpq : nullptr, &cq, sq);
}

int rwkv_b200_generate_streams_drafted(
    rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens, unsigned long long n_streams,
    unsigned long long max_new, const unsigned long long *budgets, const unsigned long long *stop_tokens, unsigned long long n_stop,
    const unsigned long long *override_tokens, const float *override_values, unsigned long long n_override,
    const rwkv_b200_sampler *samplers, const double *u, unsigned long long *tokens_out, unsigned long long *lengths_out,
    unsigned int draft, const rwkv_b200_drafter *drafter, unsigned long long *steps_out, int logprob_mode, unsigned int top_n,
    double *logprobs_out, unsigned long long *ranks_out, unsigned long long *top_tokens_out, double *top_logprobs_out,
    const unsigned long long *constraint_ids, const unsigned long long *start_states, unsigned long long *states_out,
    const rwkv_b200_stop_request *sq) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    const LogprobRequest lpq{logprob_mode, top_n, logprobs_out, ranks_out, top_tokens_out, top_logprobs_out};
    const ConstraintRequest cq{constraint_ids, start_states, states_out};
    static const rwkv_b200_drafter none{}; // a NULL drafter is refused with the other drafter checks
    return speculate(m, "generate_streams_drafted", c, SpecRequest{draft, 0, nullptr, nullptr, steps_out, drafter ? drafter : &none},
                     logprobs_out ? &lpq : nullptr, &cq, sq);
}

int rwkv_b200_generate_streams_speculative_stop(rwkv_b200_model *m, const unsigned long long *slots,
                                                const unsigned long long *first_tokens, unsigned long long n_streams,
                                                unsigned long long max_new, const unsigned long long *budgets,
                                                const unsigned long long *stop_tokens, unsigned long long n_stop,
                                                const unsigned long long *override_tokens, const float *override_values,
                                                unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                                unsigned long long *tokens_out, unsigned long long *lengths_out, unsigned int draft,
                                                unsigned int ngram, const unsigned long long *context_start,
                                                const unsigned long long *context, unsigned long long *steps_out,
                                                const rwkv_b200_stop_request *sq) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    return speculate(m, sq ? "generate_streams_speculative_stop" : "generate_streams_speculative", c,
                     SpecRequest{draft, ngram, context_start, context, steps_out, nullptr}, nullptr, nullptr, sq);
}

int rwkv_b200_generate_streams_speculative(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                                           unsigned long long n_streams, unsigned long long max_new, const unsigned long long *budgets,
                                           const unsigned long long *stop_tokens, unsigned long long n_stop,
                                           const unsigned long long *override_tokens, const float *override_values,
                                           unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                           unsigned long long *tokens_out, unsigned long long *lengths_out, unsigned int draft,
                                           unsigned int ngram, const unsigned long long *context_start,
                                           const unsigned long long *context, unsigned long long *steps_out) {
    const GenCall c{slots, first_tokens, n_streams, max_new, budgets, stop_tokens, n_stop, override_tokens, override_values,
                    n_override, samplers, samplers ? u : nullptr, tokens_out, lengths_out};
    return speculate(m, "generate_streams_speculative", c, SpecRequest{draft, ngram, context_start, context, steps_out, nullptr}, nullptr,
                     nullptr, nullptr);
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
    for (unsigned long long s = 0; s < n_streams; ++s)
        if ((rc = check_sampler(what, s, params[s], false, u != nullptr))) return rc;
    if ((rc = check_uniforms(what, u, n_streams))) return rc;
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
    LAUNCHED(m);
    return read_samples(m, n_streams, tokens_out, margins_out);
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
    bool bound;
    if ((rc = set_pass_adapters(m, what, slots, n_streams, bound))) return rc;
    CK(cudaSetDevice(m->device));
    m->stream_rows = 0; // the compact rows hold this call's scored positions, not per-stream logits
    auto &sc = m->score;
    if (n && ((rc = sc.rows.grow(n)) || (rc = sc.tgt.grow(n)) || (rc = sc.lp.grow(n)) || (rc = sc.rank.grow(n)) ||
              (rc = sc.top_tok.grow(n * top_n)) || (rc = sc.top_lp.grow(n * top_n))))
        return rc;
    if (tensor_cores(m, n_tokens, bound)) {
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
        LAUNCHED(m);
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

// ---- state indexes (csrc/index.cuh) ---------------------------------------------------------------------------------

// The multi-stream checks and the index of `id`.
// ---- adapters ----------------------------------------------------------------------------------------------------
// The input and output widths of projection k (RWKV_B200_AD_*).
static void adapter_dims(const M *m, int k, unsigned long long &in, unsigned long long &out) {
    in = k == RWKV_B200_AD_FFN_VALUE ? 4 * m->E : m->E;
    out = k == RWKV_B200_AD_FFN_KEY ? 4 * m->E : m->E;
}

int rwkv_b200_adapter_add(rwkv_b200_model *m, const rwkv_b200_adapter *desc, unsigned long long *id) {
    const char *what = "adapter_add";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!desc || !id) return fail(1, "%s: null argument", what);
    const unsigned long long r = desc->rank, L = m->L;
    if (r < 1 || r > RWKV_B200_MAX_ADAPTER_RANK) return fail(1, "%s: rank %llu is outside 1..%d", what, r, RWKV_B200_MAX_ADAPTER_RANK);
    if (!std::isfinite(desc->scale)) return fail(1, "%s: scale %g is not finite", what, desc->scale);
    size_t total = 0;
    for (int k = 0; k < RWKV_B200_AD_MATRICES; ++k) {
        if (!desc->A[k] != !desc->B[k]) return fail(1, "%s: matrix %d has only one of A and B", what, k);
        if (!desc->A[k]) continue;
        unsigned long long in, out;
        adapter_dims(m, k, in, out);
        const size_t na = (size_t)(L * r * in), nb = (size_t)(L * out * r);
        for (size_t i = 0; i < na; ++i)
            if (!std::isfinite(desc->A[k][i])) return fail(1, "%s: A of matrix %d has a non-finite value at %zu", what, k, i);
        for (size_t i = 0; i < nb; ++i)
            if (!std::isfinite(desc->B[k][i])) return fail(1, "%s: B of matrix %d has a non-finite value at %zu", what, k, i);
        total += na + nb;
    }
    if (total == 0) return fail(1, "%s: the adapter has no matrices", what);
    CK(cudaSetDevice(m->device));
    if ((rc = m->ad_table.grow(m->max_gpt))) return rc;
    if (m->slot_ad.empty()) { // the table starts all unbound (rank 0)
        CK(cudaMemsetAsync(m->ad_table.p, 0, m->max_gpt * sizeof(rk::AdapterRec), m->stream));
        m->slot_ad.assign(m->max_gpt, RWKV_B200_NO_ADAPTER);
    }
    M::Adapter a;
    if ((rc = a.data.grow(total))) return rc;
    a.rec.rank = (int)r;
    a.rec.scale = desc->scale;
    size_t o = 0;
    for (int k = 0; k < RWKV_B200_AD_MATRICES; ++k) {
        if (!desc->A[k]) continue;
        unsigned long long in, out;
        adapter_dims(m, k, in, out);
        const size_t na = (size_t)(L * r * in), nb = (size_t)(L * out * r);
        a.rec.A[k] = a.data.p + o;
        a.rec.B[k] = a.data.p + o + na;
        CK(cudaMemcpyAsync(a.data.p + o, desc->A[k], na * sizeof(float), cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(a.data.p + o + na, desc->B[k], nb * sizeof(float), cudaMemcpyHostToDevice, m->stream));
        o += na + nb;
    }
    SYNC(m);
    *id = m->next_adapter++;
    m->adapters.emplace(*id, std::move(a));
    return 0;
}

int rwkv_b200_adapter_remove(rwkv_b200_model *m, unsigned long long id) {
    const char *what = "adapter_remove";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    const auto it = m->adapters.find(id);
    if (it == m->adapters.end()) return fail(1, "%s: adapter id %llu is unknown or removed", what, id);
    for (unsigned long long s = 0; s < m->slot_ad.size(); ++s)
        if (m->slot_ad[s] == id) return fail(1, "%s: adapter %llu is still bound to slot %llu", what, id, s);
    CK(cudaSetDevice(m->device));
    SYNC(m); // no pass in flight still reads it
    m->adapters.erase(it);
    return 0;
}

int rwkv_b200_slot_adapter(rwkv_b200_model *m, unsigned long long slot, unsigned long long id) {
    const char *what = "slot_adapter";
    int rc = check_streams_model(m, what);
    if (rc || (rc = check_slot(m, what, slot))) return rc;
    const auto it = m->adapters.find(id);
    if (id != RWKV_B200_NO_ADAPTER && it == m->adapters.end()) return fail(1, "%s: adapter id %llu is unknown or removed", what, id);
    if (const rwkv_b200_batcher *b = m->batcher)
        for (const auto &kv : b->reqs) {
            const B::Req &q = kv.second;
            if (q.status > RWKV_B200_REQ_GENERATING) continue;
            if (q.slot == slot || std::find(q.spares.begin(), q.spares.end(), slot) != q.spares.end())
                return fail(1, "%s: slot %llu is held by batcher request %llu", what, slot, kv.first);
        }
    if (m->slot_ad.empty() && id == RWKV_B200_NO_ADAPTER) return 0; // nothing was ever bound
    CK(cudaSetDevice(m->device));
    if (m->slot_ad.empty()) return fail(1, "%s: no adapter table", what); // unreachable: an id exists only after an add
    const rk::AdapterRec rec = id == RWKV_B200_NO_ADAPTER ? rk::AdapterRec{} : it->second.rec;
    CK(cudaMemcpyAsync(m->ad_table.p + slot, &rec, sizeof(rec), cudaMemcpyHostToDevice, m->stream));
    SYNC(m); // the source is on this stack
    m->slot_ad[slot] = id;
    return 0;
}

static int find_index(M *m, const char *what, unsigned long long id, M::Index **out) {
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    const auto it = m->indexes.find(id);
    if (it == m->indexes.end()) return fail(1, "%s: index id %llu is unknown or freed", what, id);
    *out = &it->second;
    return 0;
}

// n entry ids, each added and not removed; with `once`, none twice.
static int check_entries(const M::Index &x, const char *what, const unsigned long long *entries, unsigned long long n,
                         bool once) {
    std::vector<char> seen(once ? x.count : 0, 0);
    for (unsigned long long i = 0; i < n; ++i) {
        const unsigned long long e = entries[i];
        if (e >= x.count) return fail(1, "%s: entry %llu was never added (%llu entries)", what, e, x.count);
        if (!x.alive[e]) return fail(1, "%s: entry %llu was removed", what, e);
        if (once && seen[e]) return fail(1, "%s: entry %llu appears twice", what, e);
        if (once) seen[e] = 1;
    }
    return 0;
}

// Room for n more entries.
static int check_room(const M::Index &x, const char *what, unsigned long long n) {
    if (n > x.capacity - x.count)
        return fail(1, "%s: %llu entries would pass the capacity %llu (%llu added)", what, n, x.capacity, x.count);
    return 0;
}

// Marks rows count .. count + n live (the copies into them are enqueued) and returns their ids.
static int index_append(M *m, M::Index &x, unsigned long long n, unsigned long long *entries_out) {
    CK(cudaMemsetAsync(x.d_alive.p + x.count, 1, n, m->stream));
    SYNC(m);
    x.alive.insert(x.alive.end(), n, 1);
    for (unsigned long long i = 0; i < n; ++i) entries_out[i] = x.count + i;
    x.count += n;
    x.live += n;
    return 0;
}

int rwkv_b200_index_create(rwkv_b200_model *m, unsigned long long layer_begin, unsigned long long n_layers,
                           unsigned long long capacity, unsigned long long *id) {
    const char *what = "index_create";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!id) return fail(1, "%s: id is NULL", what);
    if (n_layers == 0 || layer_begin >= m->L || n_layers > m->L - layer_begin)
        return fail(1, "%s: layers %llu .. %llu + %llu are not a non-empty range of the model's %llu layers", what, layer_begin,
                    layer_begin, n_layers, m->L);
    if (capacity == 0) return fail(1, "%s: capacity 0", what);
    const unsigned long long D = n_layers * m->E;
    if (capacity > (SIZE_MAX / sizeof(double)) / D) return fail(9, "%s: %llu entries of %llu doubles are too many", what, capacity, D);
    M::Index x;
    x.lb = layer_begin, x.nl = n_layers, x.D = D, x.capacity = capacity;
    CK(cudaSetDevice(m->device));
    if ((rc = x.rows.grow(capacity * D)) || (rc = x.d_alive.grow(capacity))) {
        const std::string e = g_err;
        cudaGetLastError(); // a failed allocation is not left behind as the last error
        return fail(rc, "%s: %llu entries of %llu bytes: %s", what, capacity, D * 8, e.c_str());
    }
    *id = m->next_index++;
    m->indexes.emplace(*id, std::move(x));
    return 0;
}

int rwkv_b200_index_free(rwkv_b200_model *m, unsigned long long id) {
    M::Index *x;
    int rc = find_index(m, "index_free", id, &x);
    if (rc) return rc;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    m->indexes.erase(id);
    return 0;
}

int rwkv_b200_index_add_slots(rwkv_b200_model *m, unsigned long long id, const unsigned long long *slots,
                              unsigned long long n, unsigned long long *entries_out) {
    const char *what = "index_add_slots";
    M::Index *x;
    int rc = find_index(m, what, id, &x);
    if (rc) return rc;
    if (!slots || !entries_out || n == 0) return fail(1, "%s: no slots (slots and entries_out are required)", what);
    for (unsigned long long i = 0; i < n; ++i)
        if ((rc = check_slot(m, what, slots[i]))) return rc;
    if ((rc = check_room(*x, what, n))) return rc;
    CK(cudaSetDevice(m->device));
    for (unsigned long long i = 0; i < n; ++i) {
        double *a[5];
        slot_arrays(m, slots[i], a);
        CK(cudaMemcpyAsync(x->rows.p + (x->count + i) * x->D, a[4] + x->lb * m->E, x->D * sizeof(double),
                           cudaMemcpyDeviceToDevice, m->stream));
    }
    return index_append(m, *x, n, entries_out);
}

int rwkv_b200_index_upload(rwkv_b200_model *m, unsigned long long id, const double *vectors, unsigned long long n,
                           unsigned long long *entries_out) {
    const char *what = "index_upload";
    M::Index *x;
    int rc = find_index(m, what, id, &x);
    if (rc) return rc;
    if (!vectors || !entries_out || n == 0) return fail(1, "%s: no vectors (vectors and entries_out are required)", what);
    if ((rc = check_room(*x, what, n))) return rc;
    for (unsigned long long i = 0; i < n * x->D; ++i)
        if (!std::isfinite(vectors[i]))
            return fail(1, "%s: element %llu of vector %llu is not finite", what, i % x->D, i / x->D);
    CK(cudaSetDevice(m->device));
    CK(cudaMemcpyAsync(x->rows.p + x->count * x->D, vectors, n * x->D * sizeof(double), cudaMemcpyHostToDevice, m->stream));
    return index_append(m, *x, n, entries_out);
}

int rwkv_b200_index_download(rwkv_b200_model *m, unsigned long long id, const unsigned long long *entries,
                             unsigned long long n, double *vectors_out) {
    const char *what = "index_download";
    M::Index *x;
    int rc = find_index(m, what, id, &x);
    if (rc) return rc;
    if (!entries || !vectors_out || n == 0) return fail(1, "%s: no entries (entries and vectors_out are required)", what);
    if ((rc = check_entries(*x, what, entries, n, false))) return rc;
    CK(cudaSetDevice(m->device));
    for (unsigned long long i = 0; i < n; ++i)
        CK(cudaMemcpyAsync(vectors_out + i * x->D, x->rows.p + entries[i] * x->D, x->D * sizeof(double),
                           cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_index_remove(rwkv_b200_model *m, unsigned long long id, const unsigned long long *entries,
                           unsigned long long n) {
    const char *what = "index_remove";
    M::Index *x;
    int rc = find_index(m, what, id, &x);
    if (rc) return rc;
    if (!entries || n == 0) return fail(1, "%s: no entries", what);
    if ((rc = check_entries(*x, what, entries, n, true))) return rc;
    std::vector<unsigned char> alive = x->alive;
    for (unsigned long long i = 0; i < n; ++i) alive[entries[i]] = 0;
    CK(cudaSetDevice(m->device));
    CK(cudaMemcpyAsync(x->d_alive.p, alive.data(), x->count, cudaMemcpyHostToDevice, m->stream));
    SYNC(m);
    x->alive.swap(alive);
    x->live -= n;
    return 0;
}

int rwkv_b200_index_search(rwkv_b200_model *m, unsigned long long id, const unsigned long long *query_slots,
                           unsigned long long n_queries, int metric, unsigned int k, unsigned long long *entries_out,
                           double *l1_out, double *l2_out, unsigned long long *found_out) {
    const char *what = "index_search";
    M::Index *x;
    int rc = find_index(m, what, id, &x);
    if (rc) return rc;
    if (!query_slots || !entries_out || !l1_out || !l2_out || !found_out)
        return fail(1, "%s: null argument (query_slots, entries_out, l1_out, l2_out and found_out are required)", what);
    if (n_queries == 0) return fail(1, "%s: no queries", what);
    if (metric != RWKV_B200_INDEX_L1 && metric != RWKV_B200_INDEX_L2) return fail(1, "%s: unknown metric %d", what, metric);
    if (k == 0 || k > RWKV_B200_MAX_NEIGHBOURS) return fail(1, "%s: k = %u is outside 1..%d", what, k, RWKV_B200_MAX_NEIGHBOURS);
    for (unsigned long long i = 0; i < n_queries; ++i)
        if ((rc = check_slot(m, what, query_slots[i]))) return rc;
    const unsigned long long N = x->count, D = x->D, QB = rk::kIdxQB;
    if (x->live == 0) {
        for (unsigned long long i = 0; i < n_queries * k; ++i) entries_out[i] = RWKV_B200_NO_ENTRY, l1_out[i] = l2_out[i] = NAN;
        for (unsigned long long i = 0; i < n_queries; ++i) found_out[i] = 0;
        return 0;
    }
    CK(cudaSetDevice(m->device));
    // segments, and an entry block that keeps the partial sums at 32 MiB at most
    const unsigned G = (unsigned)((D + rk::kIdxSeg - 1) / rk::kIdxSeg);
    const unsigned long long NB = std::max<unsigned long long>(1, std::min<unsigned long long>(N, (4ULL << 20) / (QB * G * 2)));
    auto pow2 = [](unsigned long long n) {
        int p = 1;
        while ((unsigned long long)p < n) p <<= 1;
        return p;
    };
    const int sort0 = pow2(std::min<unsigned long long>(N, rk::kIdxSelN));
    const unsigned long long chunks0 = (N + sort0 - 1) / sort0;
    M::IndexScratch &s = m->isc;
    if ((rc = s.partial.grow(QB * NB * G * 2)) || (rc = s.l1.grow(QB * N)) || (rc = s.l2.grow(QB * N)) ||
        (rc = s.key[0].grow(QB * chunks0 * k)) || (rc = s.key[1].grow(QB * chunks0 * k)) ||
        (rc = s.id[0].grow(QB * chunks0 * k)) || (rc = s.id[1].grow(QB * chunks0 * k)) || (rc = s.ent.grow(QB * k)) ||
        (rc = s.o1.grow(QB * k)) || (rc = s.o2.grow(QB * k))) {
        cudaGetLastError();
        return rc;
    }
    const int scan_smem = (int)(QB * rk::kIdxSeg * sizeof(double)), sel_smem = 2 * rk::kIdxSelN * (int)sizeof(unsigned long long);
    CK(cudaFuncSetAttribute(rk::k_index_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, scan_smem));
    CK(cudaFuncSetAttribute(rk::k_index_select, cudaFuncAttributeMaxDynamicSharedMemorySize, sel_smem));
    const double *dist = metric == RWKV_B200_INDEX_L1 ? s.l1.p : s.l2.p;
    for (unsigned long long b0 = 0; b0 < n_queries; b0 += QB) {
        const int nq = (int)std::min(QB, n_queries - b0);
        // the scan, one entry block at a time: enough CTAs of at least one row per warp to fill the GPU
        rk::IndexScanArgs a{};
        a.rows = x->rows.p, a.alive = x->d_alive.p, a.nq = nq, a.D = D, a.G = G, a.partial = s.partial.p;
        for (int q = 0; q < nq; ++q) {
            double *st[5];
            slot_arrays(m, query_slots[b0 + q], st);
            a.q[q] = st[4] + x->lb * m->E;
        }
        for (unsigned long long e0 = 0; e0 < N; e0 += NB) {
            const unsigned long long n = std::min(NB, N - e0);
            const unsigned long long target = (4ULL * m->sms + G - 1) / G;
            unsigned long long cy = std::min<unsigned long long>({(n + rk::kIdxWarps - 1) / rk::kIdxWarps, target, 65535});
            cy = std::max<unsigned long long>(cy, 1);
            a.e0 = e0, a.n = n, a.rows_per_cta = (n + cy - 1) / cy;
            cy = (n + a.rows_per_cta - 1) / a.rows_per_cta;
            rk::k_index_scan<<<dim3(G, (unsigned)cy), rk::kIdxWarps * 32, scan_smem, m->stream>>>(a);
            LAUNCHED(m);
            const unsigned long long t = (unsigned long long)nq * n;
            rk::k_index_combine<<<(unsigned)((t + 255) / 256), 256, 0, m->stream>>>(s.partial.p, x->d_alive.p, nq, e0, n, G,
                                                                                (double)m->E, s.l1.p, s.l2.p, N);
            LAUNCHED(m);
        }
        // the selection: passes over the survivors until one CTA per query holds them all
        const unsigned long long *ik = nullptr, *ii = nullptr;
        unsigned long long n = N;
        int pb = 0;
        for (;;) {
            const int sn = pow2(std::min<unsigned long long>(n, rk::kIdxSelN));
            const unsigned long long ch = (n + sn - 1) / sn;
            const rk::IndexSelArgs sa{dist, x->d_alive.p, N, ik, ii, n, (int)k, sn, s.key[pb].p, s.id[pb].p};
            rk::k_index_select<<<dim3((unsigned)ch, nq), rk::kIdxSelThreads, 2 * sn * sizeof(unsigned long long), m->stream>>>(sa);
            LAUNCHED(m);
            if (ch == 1) break;
            ik = s.key[pb].p, ii = s.id[pb].p, n = ch * k, pb ^= 1;
        }
        const int t = nq * (int)k;
        rk::k_index_finish<<<(t + 255) / 256, 256, 0, m->stream>>>(s.id[pb].p, s.l1.p, s.l2.p, N, nq, (int)k, s.ent.p, s.o1.p,
                                                                   s.o2.p);
        LAUNCHED(m);
        CK(cudaMemcpyAsync(entries_out + b0 * k, s.ent.p, t * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
        CK(cudaMemcpyAsync(l1_out + b0 * k, s.o1.p, t * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        CK(cudaMemcpyAsync(l2_out + b0 * k, s.o2.p, t * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        SYNC(m);
        for (int q = 0; q < nq; ++q) {
            unsigned long long f = 0;
            while (f < k && entries_out[(b0 + q) * k + f] != RWKV_B200_NO_ENTRY) ++f;
            found_out[b0 + q] = f;
        }
    }
    return 0;
}

int rwkv_b200_batcher_open(rwkv_b200_model *m, unsigned long long rows, unsigned long long prefill_tokens,
                           rwkv_b200_batcher **out) {
    const char *what = "batcher_open";
    int rc = check_streams_model(m, what);
    if (rc) return rc;
    if (!out) return fail(1, "%s: out is NULL", what);
    *out = nullptr;
    if (rows == 0 || rows > m->max_gpt) return fail(1, "%s: rows %llu is outside 1..max_gpt = %llu", what, rows, m->max_gpt);
    if (prefill_tokens == 0 || prefill_tokens > RWKV_B200_BATCHER_MAX_PREFILL)
        return fail(1, "%s: prefill_tokens %llu is outside 1..%llu", what, prefill_tokens, RWKV_B200_BATCHER_MAX_PREFILL);
    if (!rk::prefill_enabled(m->pf)) return fail(1, "%s: the batcher runs on the tensor cores, and \"prefill\" is 0", what);
    if (m->batcher) return fail(1, "%s: the model already has an open batcher", what);
    CK(cudaSetDevice(m->device));
    if ((rc = rk::prefill_init(m->pf, m->p))) return fail(rc, "%s", rk::prefill_error());
    B *b = new B;
    b->m = m;
    b->rows = (int)rows;
    b->prefill_tokens = (int)prefill_tokens;
    b->max_pass = (int)((rows + prefill_tokens + rk::kPfMaxTokens - 1) / rk::kPfMaxTokens);
    b->lane_used.assign(rows, 0);
    b->h_gs.assign(rows, rk::GenStream{});
    b->h_gc.assign(rows, rk::GenConstraint{});
    b->h_lp.assign(rows, rk::LogprobLane{-1, 0});
    b->h_gst.assign(rows, rk::GenStop{});
    b->h_ss.assign(rows, rk::SpecStream{});
    auto &bf = b->bufs;
    if ((rc = bf.gs.grow(rows)) || (rc = bf.row_stream.grow(rows)) || (rc = bf.passes.grow(kGenGroup * (size_t)b->max_pass)) ||
        (rc = bf.samp.grow(rows)) || (rc = bf.stop_start.grow(rows + 1)) || (rc = bf.out.grow(rows * kGenGroup)) ||
        (rc = bf.u.grow(kGenGroup * rows))) {
        delete b;
        return rc;
    }
    m->batcher = b;
    *out = b;
    return 0;
}

int rwkv_b200_batcher_submit_ex(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                unsigned long long *id) {
    const char *what = "batcher_submit";
    int rc = check_batcher(b);
    if (rc) return rc;
    if (!r || !id) return fail(1, "%s: null argument (the request and id are required)", what);
    if (r->n_prompt == 0 || !r->prompt) return fail(1, "%s: no prompt (n_prompt >= 1 tokens are required)", what);
    if (r->max_new == 0) return fail(1, "%s: max_new is 0", what);
    if (r->n_stop && !r->stop) return fail(1, "%s: n_stop = %llu with NULL stop", what, r->n_stop);
    const unsigned long long s = b->next_id; // the id it would get names it in messages
    if ((rc = check_slot(b->m, what, r->slot)) || (rc = check_tokens(what, "prompt token", r->prompt, r->n_prompt)) ||
        (rc = check_tokens(what, "stop token", r->stop, r->n_stop)) ||
        (rc = check_sampler(what, s, r->sampler, true, r->u != nullptr)) || (rc = check_uniforms(what, r->u, r->max_new)))
        return rc;
    std::vector<rk::GenConstraint> gc(1);
    if (x) {
        if (x->n_override && (!x->override_tokens || !x->override_values))
            return fail(1, "%s: n_override = %llu with NULL override_tokens or override_values", what, x->n_override);
        const ConstraintRequest cq{&x->constraint_id, &x->start_state, nullptr};
        if ((rc = check_tokens(what, "override token", x->override_tokens, x->n_override)) ||
            (rc = check_overrides(what, x->override_tokens, x->override_values, x->n_override)) ||
            (rc = check_constraints(b->m, what, cq, 1, x->override_tokens, x->override_values, x->n_override, gc)) ||
            (x->logprobs && (rc = check_logprob_mode(what, x->logprob_mode, x->top_n))))
            return rc;
    }
    if (const unsigned long long h = slot_holder(b, r->slot))
        return fail(1, "%s: slot %llu is held by unfinished request %llu", what, r->slot, h);
    B::Req q;
    q.slot = r->slot;
    q.max_new = r->max_new;
    q.prompt.assign(r->prompt, r->prompt + r->n_prompt);
    if (r->n_stop) q.stop.assign(r->stop, r->stop + r->n_stop);
    if (r->u) q.u.assign(r->u, r->u + r->max_new);
    q.sampler = r->sampler;
    if (x) {
        q.ovr_tok.assign(x->override_tokens, x->override_tokens + x->n_override);
        q.ovr_val.assign(x->override_values, x->override_values + x->n_override);
        q.gc = gc[0];
        if (q.gc.mask) q.constraint_id = x->constraint_id;
        if (x->logprobs) q.lp = rk::LogprobLane{x->logprob_mode, (int)x->top_n};
    }
    b->reqs[s] = std::move(q);
    b->queue.push_back(s);
    b->next_id += 1;
    *id = s;
    return 0;
}

int rwkv_b200_batcher_submit(rwkv_b200_batcher *b, const rwkv_b200_request *r, unsigned long long *id) {
    return rwkv_b200_batcher_submit_ex(b, r, nullptr, id);
}

int rwkv_b200_batcher_run(rwkv_b200_batcher *b, unsigned long long max_steps, unsigned long long *steps_run) {
    int rc = check_batcher(b);
    if (rc) return rc;
    if (steps_run) *steps_run = 0;
    if (!rk::prefill_enabled(b->m->pf)) return fail(1, "batcher_run: the batcher runs on the tensor cores, and \"prefill\" is 0");
    CK(cudaSetDevice(b->m->device));
    b->m->stream_rows = 0; // the compact logits rows no longer belong to a call the caller made
    for (unsigned long long done = 0; done < max_steps;) {
        unsigned long long ran = 0;
        if ((rc = batcher_group(b, std::min(kGenGroup, max_steps - done), &ran))) {
            // the caches of the admitted requests may name snapshots that were never written
            for (unsigned long long id : b->admitted)
                if (b->reqs[id].cache) b->reqs[id].cache->index.clear();
            return rc;
        }
        if (ran == 0) break;
        done += ran;
        if (steps_run) *steps_run = done;
    }
    return 0;
}

int rwkv_b200_batcher_read(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *tokens_out, unsigned long long cap,
                           unsigned long long *len, int *status) {
    B::Req *q = nullptr;
    if (int rc = find_req(b, "batcher_read", id, &q)) return rc;
    if (cap && !tokens_out) return fail(1, "batcher_read: cap = %llu with NULL tokens_out", cap);
    const size_t n = std::min<size_t>(cap, q->tokens.size());
    if (n) memcpy(tokens_out, q->tokens.data(), n * sizeof(unsigned long long));
    if (len) *len = q->tokens.size();
    if (status) *status = q->status;
    return 0;
}

int rwkv_b200_batcher_read_ex(rwkv_b200_batcher *b, unsigned long long id, unsigned long long cap,
                              unsigned long long *tokens_out, double *logprobs_out, unsigned long long *ranks_out,
                              unsigned long long *top_tokens_out, double *top_logprobs_out, unsigned long long *state_out,
                              unsigned long long *len, int *status) {
    const char *what = "batcher_read_ex";
    B::Req *q = nullptr;
    if (int rc = find_req(b, what, id, &q)) return rc;
    if (q->lp.mode < 0 && (logprobs_out || ranks_out || top_tokens_out || top_logprobs_out))
        return fail(1, "%s: request %llu has no log-probabilities (submit_ex with logprobs = 0 or without an extension)", what,
                    id);
    const size_t n = std::min<size_t>(cap, q->tokens.size()), nt = n * (size_t)std::max(q->lp.top_n, 0);
    if (tokens_out && n) memcpy(tokens_out, q->tokens.data(), n * sizeof(unsigned long long));
    if (logprobs_out && n) memcpy(logprobs_out, q->logprobs.data(), n * sizeof(double));
    if (ranks_out && n) memcpy(ranks_out, q->ranks.data(), n * sizeof(unsigned long long));
    if (top_tokens_out && nt) memcpy(top_tokens_out, q->top_tokens.data(), nt * sizeof(unsigned long long));
    if (top_logprobs_out && nt) memcpy(top_logprobs_out, q->top_logprobs.data(), nt * sizeof(double));
    if (state_out) *state_out = q->gc.mask ? q->gc.state : 0;
    if (len) *len = q->tokens.size();
    if (status) *status = q->status;
    return 0;
}

int rwkv_b200_batcher_submit_stop(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                  unsigned long long set_id, unsigned long long start_state, unsigned long long *id) {
    int rc = check_batcher(b);
    if (rc) return rc;
    const rwkv_b200_stop_request sq{&set_id, &start_state, nullptr, nullptr, nullptr};
    std::vector<rk::GenStop> gst;
    if ((rc = check_stops(b->m, "batcher_submit", &sq, 1, gst)) || (rc = rwkv_b200_batcher_submit_ex(b, r, x, id))) return rc;
    if (gst[0].next) {
        B::Req &q = b->reqs.at(*id);
        q.gst = gst[0];
        q.stop_set = set_id;
    }
    return 0;
}

int rwkv_b200_batcher_submit_spec(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                  unsigned long long set_id, unsigned long long start_state, const rwkv_b200_request_spec *spec,
                                  unsigned long long *id) {
    const char *what = "batcher_submit_spec";
    int rc = check_batcher(b);
    if (rc) return rc;
    if (spec) {
        M *m = b->m;
        if (!r) return fail(1, "%s: null argument (the request and id are required)", what);
        if (spec->draft < 1 || spec->draft > (unsigned)rk::kSpecMaxDraft)
            return fail(1, "%s: draft %u is outside 1..%d", what, spec->draft, rk::kSpecMaxDraft);
        if (spec->ngram < 1 || spec->ngram > (unsigned)rk::kSpecMaxNgram)
            return fail(1, "%s: ngram %u is outside 1..%d", what, spec->ngram, rk::kSpecMaxNgram);
        if (!spec->spare_slots) return fail(1, "%s: spare_slots is NULL", what);
        if (spec->n_context && !spec->context) return fail(1, "%s: %llu context tokens with NULL context", what, spec->n_context);
        if ((unsigned long long)b->rows * (spec->draft + 1ull) > m->max_gpt)
            return fail(1, "%s: rows %d x (draft %u + 1) > max_gpt %llu", what, b->rows, spec->draft, m->max_gpt);
        if (r->sampler.presence_penalty != 0.0f || r->sampler.frequency_penalty != 0.0f)
            return fail(1, "%s: presence and frequency penalties are not supported (a row's counts would have to include "
                           "its own drafts)", what);
        if ((rc = check_slots(m, what, spec->spare_slots, spec->draft)) ||
            (rc = check_tokens(what, "context token", spec->context, spec->n_context)))
            return rc;
        for (unsigned i = 0; i < spec->draft; ++i) {
            const unsigned long long z = spec->spare_slots[i];
            if (z == r->slot) return fail(1, "%s: spare slot %llu is the request's slot", what, z);
            if (const unsigned long long h = slot_holder(b, z))
                return fail(1, "%s: spare slot %llu is held by unfinished request %llu", what, z, h);
        }
        std::vector<unsigned long long> all(1, r->slot);
        all.insert(all.end(), spec->spare_slots, spec->spare_slots + spec->draft);
        if ((rc = check_same_binding(m, what, "request", b->next_id, all.data(), all.size()))) return rc;
    }
    if ((rc = rwkv_b200_batcher_submit_stop(b, r, x, set_id, start_state, id)) || !spec) return rc;
    B::Req &q = b->reqs.at(*id);
    q.draft = spec->draft;
    q.ngram = spec->ngram;
    q.spares.assign(spec->spare_slots, spec->spare_slots + spec->draft);
    if (spec->n_context) q.context.assign(spec->context, spec->context + spec->n_context);
    return 0;
}

int rwkv_b200_batcher_submit_prefix(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                    unsigned long long set_id, unsigned long long start_state,
                                    const rwkv_b200_request_spec *spec, rwkv_b200_prefix_cache *cache, unsigned long long *id) {
    int rc = check_batcher(b);
    if (rc) return rc;
    if (cache && std::find(b->m->prefix_caches.begin(), b->m->prefix_caches.end(), cache) == b->m->prefix_caches.end())
        return fail(1, "batcher_submit_prefix: the prefix cache is not an open cache of the batcher's model");
    if ((rc = rwkv_b200_batcher_submit_spec(b, r, x, set_id, start_state, spec, id)) || !cache) return rc;
    b->reqs.at(*id).cache = cache;
    return 0;
}

int rwkv_b200_batcher_read_prefix(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *cached) {
    B::Req *q = nullptr;
    if (int rc = find_req(b, "batcher_read_prefix", id, &q)) return rc;
    if (cached) *cached = q->cached;
    return 0;
}

int rwkv_b200_batcher_read_spec(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *steps) {
    B::Req *q = nullptr;
    if (int rc = find_req(b, "batcher_read_spec", id, &q)) return rc;
    if (!steps) return fail(1, "batcher_read_spec: steps is NULL");
    *steps = q->steps;
    return 0;
}

int rwkv_b200_batcher_read_stop(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *hit, unsigned long long *tail,
                                unsigned long long *state) {
    B::Req *q = nullptr;
    if (int rc = find_req(b, "batcher_read_stop", id, &q)) return rc;
    const rk::GenStop &g = q->gst;
    if (hit) *hit = g.next ? g.match : 0;
    if (tail) *tail = g.next ? g.tail : 0;
    if (state) *state = g.next ? g.state : 0;
    return 0;
}

int rwkv_b200_batcher_cancel(rwkv_b200_batcher *b, unsigned long long id) {
    B::Req *q = nullptr;
    if (int rc = find_req(b, "batcher_cancel", id, &q)) return rc;
    if (q->status > RWKV_B200_REQ_GENERATING) return fail(1, "batcher_cancel: request %llu has already ended", id);
    if (q->status == RWKV_B200_REQ_QUEUED) {
        b->queue.erase(std::find(b->queue.begin(), b->queue.end(), id));
    } else {
        if (q->home) { // the conversation is on a spare slot
            CK(cudaSetDevice(b->m->device));
            if (int rc = copy_home(b->m, b->bufs, {q->spares[q->home - 1], q->slot})) return rc;
            q->home = 0;
        }
        b->admitted.erase(std::find(b->admitted.begin(), b->admitted.end(), id));
        b->lane_used[q->lane] = 0;
    }
    q->status = RWKV_B200_REQ_CANCELLED;
    return 0;
}

int rwkv_b200_batcher_release(rwkv_b200_batcher *b, unsigned long long id) {
    B::Req *q = nullptr;
    if (int rc = find_req(b, "batcher_release", id, &q)) return rc;
    if (q->status <= RWKV_B200_REQ_GENERATING) return fail(1, "batcher_release: request %llu has not ended (cancel it first)", id);
    b->reqs.erase(id);
    return 0;
}

void rwkv_b200_batcher_close(rwkv_b200_batcher *b) {
    if (!b) return;
    if (b->m) {
        cudaSetDevice(b->m->device);
        cudaStreamSynchronize(b->m->stream);
        b->m->batcher = nullptr;
    }
    delete b;
}


int rwkv_b200_prefix_cache_open(rwkv_b200_model *m, unsigned long long capacity, unsigned long long block_tokens,
                                rwkv_b200_prefix_cache **out) {
    int rc = check_streams_model(m, "prefix_cache_open");
    if (rc) return rc;
    if (!out) return fail(1, "prefix_cache_open: null argument");
    if (!rk::prefill_enabled(m->pf)) return fail(1, "prefix_cache_open: the cache runs on the tensor cores, and the \"prefill\" option is 0");
    if (capacity == 0) return fail(1, "prefix_cache_open: capacity 0");
    if (block_tokens == 0 || block_tokens > RWKV_B200_BATCHER_MAX_PREFILL)
        return fail(1, "prefix_cache_open: block_tokens %llu outside 1..%llu", block_tokens, RWKV_B200_BATCHER_MAX_PREFILL);
    const size_t LE = (size_t)(m->L * m->E);
    if (capacity > SIZE_MAX / (4 * LE * sizeof(double))) return fail(1, "prefix_cache_open: capacity %llu is too large", capacity);
    CK(cudaSetDevice(m->device));
    PC *c = new (std::nothrow) PC((size_t)capacity);
    if (!c) return fail(1, "prefix_cache_open: out of host memory");
    c->m = m;
    c->block = block_tokens;
    if ((rc = c->pool.grow(4 * (size_t)capacity * LE)) || (rc = c->pairs.grow(2 * m->max_gpt))) {
        delete c;
        return rc;
    }
    m->prefix_caches.push_back(c);
    *out = c;
    return 0;
}

int rwkv_b200_prefix_cache_close(rwkv_b200_prefix_cache *c) {
    if (!c) return 0;
    M *m = c->m;
    if (m->batcher)
        for (const auto &e : m->batcher->reqs)
            if (e.second.cache == c && e.second.status <= RWKV_B200_REQ_GENERATING)
                return fail(1, "prefix_cache_close: unfinished batcher request %llu uses the cache", e.first);
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->stream); // passes and copies in flight may still write or read the pool
    m->prefix_caches.erase(std::find(m->prefix_caches.begin(), m->prefix_caches.end(), c));
    delete c;
    return 0;
}

int rwkv_b200_prefix_forward(rwkv_b200_prefix_cache *c, const unsigned long long *tokens, unsigned long long n_tokens,
                             const unsigned long long *slots, const unsigned long long *lengths, unsigned long long n_streams,
                             float *logits_out, unsigned long long *next_out, unsigned long long *cached_out) {
    const char *what = "prefix_forward";
    int rc = check_cache(c, what);
    if (rc) return rc;
    M *m = c->m;
    if ((rc = check_ragged(m, what, tokens, n_tokens, slots, lengths, n_streams))) return rc;
    if (!cached_out) return fail(1, "%s: null cached_out", what);
    if (!rk::prefill_enabled(m->pf)) return fail(1, "%s: the cache runs on the tensor cores, and the \"prefill\" option is 0", what);
    bool bound;
    if ((rc = set_pass_adapters(m, what, slots, n_streams, bound))) return rc;
    CK(cudaSetDevice(m->device));
    const size_t V = binfmt::kVocab;
    const bool head = logits_out || next_out;
    m->stream_rows = 0;
    std::vector<unsigned long long> cached(n_streams);
    if ((rc = prefix_forward(c, tokens, slots, lengths, n_streams, head, cached))) return rc;
    if (next_out) {
        rk::k_argmax_rows<<<(unsigned)n_streams, rk::kArgmaxThreads, 0, m->stream>>>(m->d_slogits, (int)V, m->d_next);
        LAUNCHED(m);
        CK(cudaMemcpyAsync(m->h_next, m->d_next, n_streams * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
    }
    if (logits_out) CK(cudaMemcpyAsync(m->h_logits, m->d_slogits, n_streams * V * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    if (next_out) memcpy(next_out, m->h_next, n_streams * sizeof(unsigned long long));
    if (logits_out && logits_out != m->h_logits) memcpy(logits_out, m->h_logits, n_streams * V * sizeof(float));
    std::copy(cached.begin(), cached.end(), cached_out);
    m->stream_rows = head ? n_streams : 0;
    return 0;
}

int rwkv_b200_prefix_insert(rwkv_b200_prefix_cache *c, unsigned long long slot, const unsigned long long *tokens,
                            unsigned long long n) {
    const char *what = "prefix_insert";
    int rc = check_cache(c, what);
    if (rc || (rc = check_slot(c->m, what, slot))) return rc;
    if (!tokens || n == 0) return fail(1, "%s: empty key", what);
    if ((rc = check_tokens(what, "token id", tokens, n))) return rc;
    M *m = c->m;
    CK(cudaSetDevice(m->device));
    bool fresh = false;
    const long e = c->index.take(slot_binding(m, slot), tokens, (size_t)n, &fresh);
    c->index.unpin_all(); // with nothing else pinned, some entry is always evictable
    if (e < 0) return fail(3, "%s: no entry could be taken", what);
    if ((rc = prefix_copy(c, {(unsigned long long)e, slot}, false))) {
        c->index.clear();
        return rc;
    }
    SYNC(m);
    return 0;
}

int rwkv_b200_prefix_download(rwkv_b200_prefix_cache *c, const unsigned long long *tokens, unsigned long long n, double *xy,
                              double *aa, double *bb, double *dd) {
    const char *what = "prefix_download";
    int rc = check_cache(c, what);
    if (rc) return rc;
    if (!tokens || n == 0) return fail(1, "%s: empty key", what);
    const long e = c->index.find(RWKV_B200_NO_ADAPTER, tokens, (size_t)n);
    if (e < 0) return fail(RWKV_B200_PREFIX_NOT_CACHED, "%s: no entry has this key", what);
    M *m = c->m;
    CK(cudaSetDevice(m->device));
    const size_t LE = (size_t)(m->L * m->E), per = c->index.capacity() * LE;
    double *dst[4] = {xy, aa, bb, dd};
    for (int i = 0; i < 4; ++i)
        if (dst[i]) CK(cudaMemcpyAsync(dst[i], c->pool.p + i * per + (size_t)e * LE, LE * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
    SYNC(m);
    return 0;
}

int rwkv_b200_prefix_clear(rwkv_b200_prefix_cache *c) {
    int rc = check_cache(c, "prefix_clear");
    if (rc) return rc;
    c->index.clear();
    return 0;
}

int rwkv_b200_prefix_stats(rwkv_b200_prefix_cache *c, struct rwkv_b200_prefix_stats *out) {
    int rc = check_cache(c, "prefix_stats");
    if (rc) return rc;
    if (!out) return fail(1, "prefix_stats: null argument");
    const prefix::Stats &s = c->index.stats();
    out->live = s.live;
    out->lookups = s.lookups;
    out->hit_tokens = s.hit_tokens;
    out->prefilled_tokens = s.prefilled_tokens;
    out->snapshots = s.snapshots;
    out->skipped = s.skipped;
    out->evictions = s.evictions;
    return 0;
}

int rwkv_b200_decode_timed(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n,
                           int teacher_forced, float *ms) {
    int rc = check_model(m);
    if (rc) return rc;
    if (!tokens || n == 0 || !ms) return fail(1, "decode_timed: bad arguments");
    const unsigned long long slot0 = 0;
    if ((rc = check_unbound(m, "decode_timed", &slot0, 1))) return rc;
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
    const unsigned long long slot0 = 0;
    if ((rc = check_unbound(m, "profile", &slot0, 1))) return rc;
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
    } else if (k == "sub_bytes") {
        if (v < 16 || v > m->p.tile_bytes || v % 16 != 0) return fail(1, "sub_bytes must be a multiple of 16 in 16..%d", m->p.tile_bytes);
        m->p.sub_bytes = v;
    } else if (k == "budget") { // a stage can always be filled outside an exchange
        if (v < m->p.tile_bytes || v > rk::kMaxStages * m->p.tile_bytes)
            return fail(1, "budget must be %d..%d bytes", m->p.tile_bytes, rk::kMaxStages * m->p.tile_bytes);
        m->p.budget = v;
    } else if (k == "qbudget") { // one copy is always allowed when nothing is in flight
        if (v < 0 || v > rk::kMaxStages * m->p.tile_bytes) return fail(1, "qbudget must be 0..%d bytes", rk::kMaxStages * m->p.tile_bytes);
        m->p.qbudget = v;
    } else if (k == "grid") {
        if (int rc2 = check_grid(m, v)) return rc2;
        m->grid = v;
    } else if (k == "pf_dist") {
        if (v < 0 || v > 64) return fail(1, "pf_dist is 0..64 tiles");
        m->p.pf_dist = v;
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
    if (k == "graph_records") { // tensor-core pass graphs recorded since load (a host counter)
        if (dst_bytes < sizeof(unsigned long long)) return -1;
        memcpy(dst, &m->pf.records, sizeof(unsigned long long));
        return 1;
    }
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
