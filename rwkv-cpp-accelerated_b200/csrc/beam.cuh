// beam.cuh — device side of rwkv_b200_beam_search: beams are rows of generate_streams' step loop whose slot changes from
// step to step.
//
// A call runs G groups of B beams. Beam j of group g has the GenStream record g * B + j (its slot, its input token, its
// length and the group's done flag) and a cumulative log-probability. Each step of a host group is enqueued with no
// synchronisation inside it: forward (row r = a live beam; step 0 has one row per group, later steps B rows per live
// group, group by group), then
//   k_beam_expand  one CTA per row: the first C = B + n_stop tokens of the row's ranking with their log-probabilities,
//                  by logprob_row (score.cuh) with tau = 1, so every candidate is bit for bit what score_streams reports;
//   k_beam_select  one CTA per live group: orders the group's candidates, walks them (new beams, finished hypotheses),
//                  updates the hypothesis list, decides whether the group is done, assigns slots, and writes the next
//                  step's inputs (GenStream records, pass descriptors) and the forks;
//   k_beam_fork    copies a parent's five state arrays onto the free slot a forked beam takes.
// The rule is stated in include/rwkv_b200.h and DESIGN §4.3.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "generate.cuh"
#include "score.cuh"

namespace rk {

constexpr int kMaxBeams = kMaxTopN;                       // B + n_stop <= RWKV_B200_MAX_TOP_N
constexpr int kMaxBeamCands = kMaxBeams * kMaxTopN;       // candidates of one group and step: B * (B + n_stop) <= 400
constexpr int kBeamSelectThreads = 256;
constexpr int kForkThreads = 256;
constexpr int kForkChunk = kForkThreads * 8;              // doubles of one array one CTA of k_beam_fork copies

// One step of one beam: the beam it extends (its index among the group's previous beams), its token and that token's
// log-probability.
struct BeamBack {
    int parent;
    int pad;
    unsigned long long tok;
    double lp;
};

// A hypothesis: the beam with index `parent` among the beams that were live at step `step`, extended by `tok` (the stop
// token for a finished one). len = step + 1 tokens; cum = the sum of their log-probabilities; score = cum / P[len].
struct BeamHyp {
    double cum, score, lp;
    unsigned long long tok;
    int step, parent, len, finished;
};

struct BeamArgs {
    GenStream *gs;                   // [G * B] beam g * B + j
    double *cum;                     // [G * B] cumulative log-probability of each live beam
    const int *groups;               // [live groups] group of CTA gi of k_beam_select
    const unsigned long long *cand_tok; // [rows][C] candidates of each row (k_beam_expand)
    const double *cand_lp;           // [rows][C]
    int C, B, K;                     // candidates per row, beams, hypotheses kept
    int step;                        // this step, 0..N-1
    int nb;                          // live beams per group at this step: 1 at step 0, else B
    unsigned long long N;            // max_new
    const double *P;                 // [N + 1] length penalties, P[n] = pow(n, alpha)
    int neg_alpha;                   // alpha < 0: the bound of a live beam uses P[n + 1], else P[N]
    const unsigned long long *stop;  // [n_stop]
    int n_stop;
    BeamBack *back;                  // [G][N][B]
    BeamHyp *hyp;                    // [G][K] best first
    int *n_hyp;                      // [G]
    unsigned long long *done;        // [G]
    unsigned long long *forks;       // [live groups * B][2] {src slot, dst slot}; kNoFork: none
    PassDesc *passes;                // tensor-core path: the descriptors of the next step, else nullptr
};

constexpr unsigned long long kNoFork = ~0ull;

// One CTA of kNucThreads per row of the step: the first C tokens of the row's ranking, into cand_tok / cand_lp row r.
// A row of a done group returns at once (the whole CTA, before any barrier): its stream's record says done.
__global__ void __launch_bounds__(kNucThreads) k_beam_expand(const float *logits, int V, const GenStream *gs, const int *row_stream,
                                                             int C, unsigned long long *cand_tok, double *cand_lp) {
    const int r = blockIdx.x;
    if (gs[row_stream[r]].done) return;
    __shared__ double s_lp;
    __shared__ unsigned long long s_rank;
    logprob_row(logits + (size_t)r * V, V, 0, 1.0, C, &s_lp, &s_rank, cand_tok + (size_t)r * C, cand_lp + (size_t)r * C);
}

// Offer a hypothesis to a list of at most K held best first by (score descending, offer order ascending): it enters
// when fewer than K are held or its score is strictly above the worst one held (which it then replaces). Returns the
// new count.
__device__ __forceinline__ int beam_offer(BeamHyp *h, int n, int K, const BeamHyp &x) {
    if (n == K && !(x.score > h[K - 1].score)) return n;
    int i = n < K ? n++ : K - 1;
    while (i > 0 && h[i - 1].score < x.score) {
        h[i] = h[i - 1];
        --i;
    }
    h[i] = x;
    return n;
}

// One CTA per live group (CTA gi owns rows gi * nb .. gi * nb + nb - 1 of this step and gi * B .. gi * B + B - 1 of the
// next). Steps 3-9 of the rule.
__global__ void __launch_bounds__(kBeamSelectThreads) k_beam_select(const BeamArgs a) {
    const int gi = blockIdx.x, g = a.groups[gi], tid = threadIdx.x;
    const int B = a.B, C = a.C, nb = a.nb, n = nb * C;
    GenStream *gs = a.gs + (size_t)g * B;
    if (gs[0].done) return;
    // per candidate: c, its score as a finished hypothesis, and its bound (the last step: its score as an unfinished one)
    __shared__ double c_s[kMaxBeamCands], fin_s[kMaxBeamCands], bnd_s[kMaxBeamCands];
    __shared__ int order[kMaxBeamCands];
    __shared__ unsigned char is_stop[kMaxBeamCands];
    __shared__ int parent_s[kMaxBeams], free_of[kMaxBeams]; // new beam j: its parent; the free beam whose slot it takes, or -1
    __shared__ unsigned long long prev_slot[kMaxBeams], new_tok[kMaxBeams];
    __shared__ double new_lp[kMaxBeams], new_cum[kMaxBeams], new_bnd[kMaxBeams];
    __shared__ int s_done;

    const size_t row0 = (size_t)gi * nb * C;
    const int last = (unsigned long long)a.step + 1 == a.N; // the last step: the live beams become hypotheses
    for (int i = tid; i < n; i += kBeamSelectThreads) {
        const int b = i / C;
        const unsigned long long tok = a.cand_tok[row0 + i];
        const double c = a.cum[(size_t)g * B + b] + a.cand_lp[row0 + i];
        c_s[i] = c;
        fin_s[i] = c / a.P[a.step + 1];
        bnd_s[i] = c / (a.neg_alpha && last == 0 ? a.P[a.step + 2] : a.P[a.N]);
        bool st = false;
        for (int z = 0; z < a.n_stop; ++z) st |= a.stop[z] == tok;
        is_stop[i] = st ? 1 : 0;
    }
    for (int j = tid; j < B; j += kBeamSelectThreads) prev_slot[j] = gs[j].slot;
    __syncthreads();
    // order by (c descending, beam ascending, rank ascending): candidate i = b * C + rank, so the index breaks ties
    for (int i = tid; i < n; i += kBeamSelectThreads) {
        const double ci = c_s[i];
        int pos = 0;
        for (int u = 0; u < n; ++u) pos += c_s[u] > ci || (c_s[u] == ci && u < i);
        order[pos] = i;
    }
    __syncthreads();

    if (tid == 0) {
        BeamHyp *h = a.hyp + (size_t)g * a.K;
        int nh = a.n_hyp[g];
        int nnew = 0;
        for (int pos = 0; pos < n && nnew < B; ++pos) {
            const int i = order[pos], b = i / C;
            const unsigned long long tok = a.cand_tok[row0 + i];
            const double lp = a.cand_lp[row0 + i];
            if (is_stop[i]) {
                if (pos < B) {
                    nh = beam_offer(h, nh, a.K, BeamHyp{c_s[i], fin_s[i], lp, tok, a.step, b, a.step + 1, 1});
                }
                continue;
            }
            parent_s[nnew] = b;
            new_tok[nnew] = tok;
            new_lp[nnew] = lp;
            new_cum[nnew] = c_s[i];
            new_bnd[nnew] = bnd_s[i];
            ++nnew;
        }
        BeamBack *bk = a.back + ((size_t)g * a.N + a.step) * B;
        for (int j = 0; j < B; ++j) bk[j] = BeamBack{parent_s[j], 0, new_tok[j], new_lp[j]};
        bool done;
        if (last) {
            // the live beams are offered in order as unfinished hypotheses
            for (int j = 0; j < B; ++j)
                nh = beam_offer(h, nh, a.K, BeamHyp{new_cum[j], new_bnd[j], new_lp[j], new_tok[j], a.step, parent_s[j], (int)a.N, 0});
            done = true;
        } else {
            // exact: every log-probability is <= 0, so no extension of a live beam scores above its bound
            done = nh == a.K;
            for (int j = 0; j < B && done; ++j) done = new_bnd[j] <= h[a.K - 1].score;
        }
        a.n_hyp[g] = nh;
        // slots: a beam keeps its parent's slot if no earlier new beam took it, else takes the next free slot (a previous
        // beam without a child, ascending beam index) and a copy of the parent's state
        uint32_t taken = 0, child = 0; // bit p: previous beam p
        for (int j = 0; j < B; ++j) child |= 1u << parent_s[j];
        int free_at = 0;
        for (int j = 0; j < B; ++j) {
            const int p = parent_s[j];
            if (!((taken >> p) & 1u)) {
                taken |= 1u << p;
                free_of[j] = -1;
                continue;
            }
            while ((child >> free_at) & 1u) ++free_at;
            free_of[j] = free_at++;
        }
        s_done = done ? 1 : 0;
        if (done) a.done[g] = 1;
    }
    __syncthreads();
    const bool done = s_done != 0;
    // the next step's inputs; a done group's rows are frozen and it forks nothing
    for (int j = tid; j < B; j += kBeamSelectThreads) {
        const int p = parent_s[j], f = free_of[j];
        const unsigned long long slot = f < 0 ? prev_slot[p] : prev_slot[f];
        a.cum[(size_t)g * B + j] = new_cum[j];
        gs[j] = GenStream{slot, a.N, new_tok[j], (unsigned long long)a.step + 1, done ? 1ull : 0ull};
        unsigned long long *fk = a.forks + 2 * ((size_t)gi * B + j);
        fk[0] = prev_slot[p];
        fk[1] = f < 0 || done ? kNoFork : slot;
        if (a.passes) {
            const int r = gi * B + j;
            PassDesc &pd = a.passes[r / kPfMaxTokens];
            const int t = r % kPfMaxTokens;
            pd.tokens[t] = new_tok[j];
            pd.desc[t] = (uint32_t)slot | kDescFirst | (done ? 0u : kDescLast);
            pd.rows[t] = t;
            if (t == 0) pd.out_row0 = r;
        }
    }
}

// Grid (fork entries, chunks of kForkChunk doubles, 5 arrays): copy the chunk of array blockIdx.z of the source slot onto
// the destination slot. Unused entries exit at once. Sources and destinations of one step are disjoint (parents'
// slots, free slots), so the copies of a step run in any order.
__global__ void __launch_bounds__(kForkThreads) k_beam_fork(const unsigned long long *forks, double *a0, double *a1, double *a2,
                                                            double *a3, double *a4, size_t slot_len) {
    const unsigned long long dst = forks[2 * blockIdx.x + 1];
    if (dst == kNoFork) return;
    const unsigned long long src = forks[2 * blockIdx.x];
    const unsigned z = blockIdx.z;
    double *arr = z == 0 ? a0 : z == 1 ? a1 : z == 2 ? a2 : z == 3 ? a3 : a4;
    const double2 *s = reinterpret_cast<const double2 *>(arr + src * slot_len);
    double2 *d = reinterpret_cast<double2 *>(arr + dst * slot_len);
    const size_t n2 = slot_len / 2, i0 = (size_t)blockIdx.y * (kForkChunk / 2);
    for (size_t i = i0 + threadIdx.x; i < n2 && i < i0 + kForkChunk / 2; i += kForkThreads) d[i] = s[i];
}

} // namespace rk
