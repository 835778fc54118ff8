// rwkv_hooks.cpp — the reference's six backend hooks, implemented on the H100 engine.
//
// The reference's host class (harrisonvanderbyl/rwkv-cpp-accelerated include/rwkv/rwkv/rwkv.h) talks to
// its CUDA backend through six C++-linkage functions declared at rwkv.h:63-122 and defined in
// include/rwkv/cuda/rwkv.cu:479-490 (setState), 467-477 (getOutput), 493-593 (cuda_rwkv_parralel),
// 595-628 (cuda_rwkv), 638-717 (load), 719-730 (freeTensors). A program that compiles against the
// REFERENCE's own, unmodified rwkv.h links against this translation unit + librwkv_b200 instead of
// rwkv.cu and runs on the H100 engine: same symbols (same mangled names), same argument meaning.
//
// How the 47-pointer calls map onto the engine: `load` fills the tensor table with the engine's device
// pointers (rwkv_b200_tensor), so every later call identifies its model by the pointer it passes for
// tensor X / STATEXY. The engine keeps embedding, weights and state resident and runs the whole token
// in one kernel, so the per-tensor pointers of cuda_rwkv_parralel are not dereferenced here.
//
// Built into librwkv_cuda.a by CMakeLists.txt; tests/test_boundary_gpu.py runs the reference's own
// RWKV::forward through it and checks the logits against the oracle.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../rwkv_b200.h"
#include "../enums/enum.h" // MODE and the tensor-index enum: part of the mangled signatures / the table order

namespace {

struct Bound {
    rwkv_b200_model *model;
    int **table;     // the caller's tensor table (RWKV::tensors)
    void *x, *sxy;   // device pointers that identify the model in later calls
    unsigned long long max_gpt;
};
std::mutex g_mu;
std::vector<Bound> g_bound;

Bound *find_by(void *x, void *sxy) {
    for (auto &b : g_bound)
        if ((x && b.x == x) || (sxy && b.sxy == sxy)) return &b;
    return nullptr;
}

[[noreturn]] void die(const char *what) {
    fprintf(stderr, "rwkv (H100 backend): %s: %s\n", what, rwkv_b200_last_error());
    exit(1);
}

} // namespace

// rwkv.h:63 / rwkv.cu:638 — load the model, fill ptrs[0..45] with device pointers, return {n_layers, n_embed}.
// A missing file prints a message and exits, as the reference does (rwkv.cu:641-645).
std::tuple<unsigned long long, unsigned long long> load(const std::string &filename, int **ptrs, unsigned long long maxGPT) {
    rwkv_b200_model *m = nullptr;
    unsigned long long L = 0, E = 0;
    if (rwkv_b200_load(filename.c_str(), maxGPT ? maxGPT : 1, 0, 0, &m, &L, &E) != 0) {
        printf("Error opening file %s: %s\n", filename.c_str(), rwkv_b200_last_error());
        exit(1);
    }
    for (int i = 0; i < RWKV_B200_NUM_TENSORS; ++i) ptrs[i] = static_cast<int *>(rwkv_b200_tensor(m, i));
    std::lock_guard<std::mutex> lk(g_mu);
    g_bound.push_back(Bound{m, ptrs, rwkv_b200_tensor(m, X), rwkv_b200_tensor(m, STATEXY), maxGPT ? maxGPT : 1});
    return std::make_tuple(L, E);
}

// rwkv.h:64 / rwkv.cu:479 — host state -> device state, `tokenlength` slots. (The reference's call site
// passes (n_layers, n_embed) in the opposite order of the declaration, rwkv.h:353; only the product is used.)
void setState(unsigned long long, unsigned long long, double *stateaa, double *, double *, double *, double *,
              double *instateaa, double *instatebb, double *instatecc, double *instatedd, double *instateee,
              unsigned long long tokenlength) {
    std::lock_guard<std::mutex> lk(g_mu);
    Bound *b = find_by(nullptr, stateaa);
    if (!b) {
        fprintf(stderr, "rwkv (H100 backend): setState on a state that load() did not create\n");
        exit(1);
    }
    if (rwkv_b200_state_upload(b->model, instateaa, instatebb, instatecc, instatedd, instateee, tokenlength) != 0) die("setState");
}

// rwkv.h:74 / rwkv.cu:467 — logits and state back to the host.
void getOutput(unsigned long long, unsigned long long, float *, double *statexyin, double *, double *, double *, double *,
               float *logitsout, double *statexyout, double *stateaaout, double *statebbout, double *stateppout,
               double *stateddout, unsigned long long tokenlength) {
    std::lock_guard<std::mutex> lk(g_mu);
    Bound *b = find_by(nullptr, statexyin);
    if (!b) {
        fprintf(stderr, "rwkv (H100 backend): getOutput on a state that load() did not create\n");
        exit(1);
    }
    // the forward left the logits of its `tokenlength` tokens in the engine's pinned buffer
    memcpy(logitsout, rwkv_b200_logits_host(b->model), sizeof(float) * RWKV_B200_VOCAB * tokenlength);
    if (rwkv_b200_state_download(b->model, statexyout, stateaaout, statebbout, stateppout, stateddout, tokenlength) != 0) die("getOutput");
}

// rwkv.h:77 / rwkv.cu:719
void freeTensors(int **ptrs) {
    std::lock_guard<std::mutex> lk(g_mu);
    for (size_t i = 0; i < g_bound.size(); ++i) {
        if (g_bound[i].table == ptrs) {
            rwkv_b200_free(g_bound[i].model);
            g_bound.erase(g_bound.begin() + (long)i);
            return;
        }
    }
}

// rwkv.h:104 / rwkv.cu:493 — the forward over `tokenlength` tokens.
void cuda_rwkv_parralel(unsigned long long, unsigned long long, unsigned long long *token, double *x,
                        float *, double *,
                        double *statexy, double *, double *, double *, double *,
                        double *, float *, float *, float *,
                        double *, double *, double *,
                        uint8_t *, uint8_t *, uint8_t *,
                        float *, float *, float *,
                        float *, float *, float *,
                        uint8_t *, float *, float *,
                        double *, double *,
                        uint8_t *, uint8_t *, uint8_t *,
                        float *, float *, float *,
                        float *, float *, float *,
                        double *, double *, float *,
                        double *, double *,
                        uint8_t *, float *, float *,
                        unsigned long long tokenlength, MODE mode) {
    Bound *b;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        b = find_by(x, statexy);
    }
    if (!b) {
        fprintf(stderr, "rwkv (H100 backend): forward on tensors that load() did not create\n");
        exit(1);
    }
    if (rwkv_b200_forward(b->model, token, tokenlength, mode == PARRALEL ? RWKV_B200_MODE_PARRALEL : RWKV_B200_MODE_GPT,
                          rwkv_b200_logits_host(b->model)) != 0)
        die("forward");
}

// rwkv.h:87 / rwkv.cu:595 — the single-token entry (unused by the reference's RWKV class; kept for the ABI).
void cuda_rwkv(unsigned long long n_layers, unsigned long long n_emb, unsigned long long token, double *x,
               float *embed, double *layernorms,
               double *statexy, double *stateaa, double *statebb, double *statepp, double *statedd,
               double *buffer1, float *buffer2, float *buffer3, float *buffer4,
               double *mixk, double *mixv, double *mixr,
               uint8_t *km, uint8_t *vm, uint8_t *rm,
               float *kr, float *vr, float *rr,
               float *o1, float *o2, float *o3,
               uint8_t *attout, float *attoutr, float *attouto,
               double *ffnmixk, double *ffnmixv,
               uint8_t *ffnk, uint8_t *ffnv, uint8_t *ffnr,
               float *ffnkr, float *ffnvr, float *ffnrr,
               float *ffnko, float *ffnvo, float *ffnro,
               double *ffnkbuffer, double *ffnvbuffer, float *ffnrbuffer,
               double *decay, double *bonus,
               uint8_t *head, float *headr, float *heado) {
    unsigned long long t = token;
    cuda_rwkv_parralel(n_layers, n_emb, &t, x, embed, layernorms, statexy, stateaa, statebb, statepp, statedd, buffer1, buffer2,
                       buffer3, buffer4, mixk, mixv, mixr, km, vm, rm, kr, vr, rr, o1, o2, o3, attout, attoutr, attouto, ffnmixk,
                       ffnmixv, ffnk, ffnv, ffnr, ffnkr, ffnvr, ffnrr, ffnko, ffnvo, ffnro, ffnkbuffer, ffnvbuffer, ffnrbuffer,
                       decay, bonus, head, headr, heado, 1, GPT);
}
