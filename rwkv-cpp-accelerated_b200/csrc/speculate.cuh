// speculate.cuh — device side of rwkv_b200_generate_streams_speculative and of the batcher's speculative lanes
// (rwkv_b200_batcher_submit_spec): prompt-lookup drafts verified in the tensor-core pass, so that a step can emit several
// tokens per stream with the bits of one-token-per-step generation.
//
// A call keeps one record per stream (SpecStream): its k + 1 slots, which of them is home (holds the conversation),
// its history (lookup context ++ first token ++ tokens emitted so far) and its length, budget and step count. Each step
// of a host group is enqueued with no synchronisation inside the group:
//   k_spec_draft   one CTA per live stream: the prompt-lookup drafts of the history (a block-parallel scan for the largest
//                  matching position per n-gram length, reduced by max, so the result does not depend on the schedule),
//                  then the step's layout: row 0 = the current input on the home slot (first | last), row i = draft i on
//                  the stream's i-th other slot (last), so every row stores its state in its own slot; and the uniform
//                  of each row for k_sample_nucleus;
//   forward        the tensor-core passes; a stream's k + 1 rows are consecutive head rows inside one pass (SpecLive);
//   k_gen_override, then k_sample_nucleus or k_argmax_rows on the rows (row_stream maps every row of s to s);
//   k_spec_accept  one CTA per live stream: the picks, the accepted prefix, the emitted tokens into the output (by
//                  gen_emit over SpecArgs::emit, the GenEmit of k_gen_feedback: budget, stops, automaton) and into the
//                  history, and the new home: the slot of the row that produced the last emitted token;
//   k_spec_logprob (with log-probabilities) one CTA per row: the emitted token of the row, if it emitted one, scored.
// With token automata, k_spec_draft also walks the drafts through the stream's automaton into a state per row, by which
// k_gen_mask masks the rows, and k_spec_accept advances the automaton by each emitted token (DESIGN §4.3).
// rwkv_b200_generate_streams_drafted takes the drafts from a draft model instead ("drafts from a draft model" below):
// k_spec_layout then lays out the rows of the drafts the draft model's passes stored in the record.
// The one-shot call gives every stream the same k and lays out floor(128 / (k + 1)) streams per pass, every row a head
// row, and k_spec_draft writes the passes' head maps. The batcher mixes streams of different k with one-token lanes
// (k_gen_feedback's) and prefill segments: the host lays out the head maps once per group, and each stream's outputs go
// to a ring of kGenGroup (kSpecMaxDraft + 1) entries per lane (`% max_new`, which leaves the one-shot index alone).
// At the end of the call, or when a batcher request ends, a stream whose home is not its first slot has the home's xy,
// aa, bb and dd copied to the first slot (k_beam_fork with four arrays). The rule is stated in include/rwkv_b200.h and
// DESIGN §4.3.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "generate.cuh"
#include "prefill.cuh"
#include "score.cuh"

namespace rk {

constexpr int kSpecMaxDraft = 15;   // k <= 15: a stream's k + 1 rows fit one warp and one pass
constexpr int kSpecMaxNgram = 8;
constexpr int kSpecDraftThreads = 256;

struct SpecStream {
    unsigned long long slot[kSpecMaxDraft + 1]; // the stream's k + 1 slots; slot[0] is the first slot
    unsigned long long row[kSpecMaxDraft + 1];  // this step's row tokens: [0] the input, [i] draft i
    unsigned long long h0, hl;                  // the history is hist[h0 .. h0 + hl); its last token is the next input
    unsigned long long budget, len, steps;      // tokens it may emit, tokens emitted, steps that emitted a token
    unsigned long long done;                    // 1 after a stop token or the budget
    unsigned long long u0;                      // row i of a step draws u[u0 + (len + i) * u_stride] (SpecArgs)
    int home;                                   // index into slot[] of the slot holding the conversation
    int k, ngram;                               // drafts per step (1..kSpecMaxDraft), longest n-gram looked up
};

// Where a live stream's rows lie in a step: its record, the logits row of its row 0 (rows row0 .. row0 + k), and the
// position of row 0 in the step's layout (pass pos0 / 128, token pos0 % 128; the k + 1 rows never straddle a pass).
struct SpecLive {
    int s, row0, pos0;
};

// What k_spec_logprob scores for row i of live stream li, at [li * (SpecArgs::k + 1) + i]: the row, its stream and the
// result entry of the token it emitted this step; s < 0: the row emitted nothing.
struct SpecScore {
    int r, s;
    unsigned long long o;
};

struct SpecArgs {
    SpecStream *ss;                  // [n_streams]
    const SpecLive *live;            // [live streams] CTA i's stream and rows
    int k;                           // the largest k of the live streams: k_spec_logprob's CTAs per stream, less one
    bool heads;                      // k_spec_draft writes the head maps (every row of a pass a head row, in order)
    unsigned long long *hist;        // the histories
    PassDesc *passes;                // the step's passes
    const double *u;                 // the uniforms, or nullptr
    double *row_u;                   // [rows] the uniform of each row (with u only)
    unsigned long long u_stride;
    const unsigned long long *next;  // arg-max per row, or nullptr when sampling
    const double *sample;            // {token, margin} per row when sampling
    // the emitted tokens and what ends a stream (generate.cuh); emit.gc is set with token automata, and then row_state
    // is the state of each row this step (kNoState: not masked)
    GenEmit emit;
    unsigned long long *row_state;   // [rows]
    SpecScore *score;                // [live streams][k + 1] with log-probabilities, else nullptr
};

// Draft rule: for n = ngram down to 1 with n < L, the largest j <= L - n - 1 with h[j .. j + n) == h[L - n .. L); the
// first n with such a j gives the proposal h[j + n .. min(j + n + k, L)], padded with its last token; no match at any n:
// k copies of h[L - 1]. Draft i (1-based) is then h[min(j + n + i - 1, L - 1)]. Returns j + n, or -1 without a match
// (and for a finished stream). Every thread of the CTA calls it.
__device__ __forceinline__ long long spec_propose(const SpecStream &g, const unsigned long long *h, long long L, bool live) {
    const int ngram = g.ngram, tid = threadIdx.x;
    __shared__ unsigned long long suf[kSpecMaxNgram]; // suf[i] = h[L - 1 - i]
    __shared__ int wmax[kSpecDraftThreads / 32];
    long long from = -1; // the proposal starts at h[from]
    if (live) {
        if (tid < ngram && tid < L) suf[tid] = h[L - 1 - tid];
        __syncthreads();
        for (int n = ngram; n >= 1 && from < 0; --n) {
            if (n >= L) continue;
            int best = -1;
            for (long long j = tid; j <= L - n - 1; j += kSpecDraftThreads) {
                bool eq = true;
                for (int i = 0; i < n && eq; ++i) eq = h[j + n - 1 - i] == suf[i];
                if (eq) best = (int)j;
            }
            best = __reduce_max_sync(0xffffffffu, best);
            if ((tid & 31) == 0) wmax[tid >> 5] = best;
            __syncthreads();
            for (int w = 0; w < kSpecDraftThreads / 32; ++w) best = max(best, wmax[w]);
            __syncthreads();
            if (best >= 0) from = best + n;
        }
    }
    return from;
}

// A step's layout for live stream lv, whatever proposed its drafts: thread tid <= k writes row tid's token
// (row_tok(tid): 0 the input, i draft i) into the record, the pass and its descriptor (row 0 on the home slot first |
// last, row i on the stream's i-th other slot last; a finished stream stores nothing), with a.heads the head map, and
// with uniforms the row's uniform; with token automata thread 0 walks the drafts into a state per row.
template <class RowTok>
__device__ __forceinline__ void spec_layout(const SpecArgs &a, const SpecLive lv, SpecStream &g, bool live, RowTok row_tok) {
    const int s = lv.s, tid = threadIdx.x, k = g.k;
    const unsigned long long tok = row_tok(tid);
    g.row[tid] = tok;
    const int r = lv.row0 + tid, pi = (lv.pos0 + tid) / kPfMaxTokens, t = (lv.pos0 + tid) % kPfMaxTokens;
    if (a.emit.gc && tid == 0) {
        // row 0 has the stream's state; row i is live while row i - 1 is, draft i has an edge out of its state and that
        // edge leads to a state with edges. A dead row cannot be emitted: with no edge, the pick of the masked row
        // i - 1 differs from draft i; at a complete state, emitting draft i ends the stream
        const GenConstraint &c = a.emit.gc[s];
        unsigned long long q = live && c.mask ? c.state : kNoState;
        a.row_state[r] = q;
        for (int i = 1; i <= k; ++i) {
            if (q != kNoState) {
                q = gen_edge(c, q, row_tok(i));
                if (q != kNoState && c.start[q] == c.start[q + 1]) q = kNoState;
            }
            a.row_state[r + i] = q;
        }
    }
    PassDesc &pd = a.passes[pi];
    pd.tokens[t] = tok;
    pd.desc[t] = (uint32_t)g.slot[(g.home + tid) % (k + 1)] | (tid == 0 ? kDescFirst : 0u) | (live ? kDescLast : 0u);
    if (a.heads) {
        pd.rows[t] = t;
        if (t == 0) pd.out_row0 = r;
    }
    if (a.u) { // a row past the budget is never emitted
        const unsigned long long pos = g.len + (unsigned long long)tid;
        a.row_u[r] = pos < g.budget ? a.u[g.u0 + pos * a.u_stride] : 0.0;
    }
}

// Prompt lookup: one CTA per live stream proposes (spec_propose) and lays out (spec_layout) its rows.
__global__ void __launch_bounds__(kSpecDraftThreads) k_spec_draft(const SpecArgs a) {
    const SpecLive lv = a.live[blockIdx.x];
    SpecStream &g = a.ss[lv.s];
    const unsigned long long *h = a.hist + g.h0;
    const long long L = (long long)g.hl;
    const bool live = g.done == 0;
    const long long from = spec_propose(g, h, L, live);
    if ((int)threadIdx.x > g.k) return;
    spec_layout(a, lv, g, live, [&](int i) { return i == 0 || from < 0 ? h[L - 1] : h[min(from + i - 1, L - 1)]; });
}

// ---- drafts from a draft model (rwkv_b200_generate_streams_drafted) ------------------------------------------------
// Each stream keeps two slots of the draft model: D0 holds the tokens the stream's home has absorbed (the history but
// its last token, h[0 .. fed) of this call so far), D1 is scratch. A step, before spec_layout, enqueues on the draft
// model (one CUDA stream with the target's work, no synchronisation):
//   k_draft_first  one thread per live stream: a segment of k + 2 positions, h[fed .. hl) then pads. h[fed .. hl - 1)
//                  (the tokens the home absorbed in the last step) starts on D0 (first) and stores into D0 (last at its
//                  end); h[hl - 1], the step's input, continues it and stores into D1 (last) and is the stream's head
//                  row. At the first step the segment is the input alone, first | last on D1, which the call forked
//                  from D0. Pads continue the segment and store nothing;
//   pass, then per draft i = 1..k: the pick chain on the draft's rows with the call's overrides, sampler, the row's
//   automaton state and the uniform of target row i - 1; k_draft_pick stores d_i into the stream record and, for
//   i < k, lays out pass i + 1: d_i first | last on D1, one token per stream;
//   k_spec_layout  the layout of the target's rows from the record's drafts.
// At the end of the call k_draft_flush lays out one pass without logits that absorbs each stream's h[fed .. hl - 1)
// into D0, so D0 ends with exactly the tokens the first slot absorbed. A finished stream stores nothing in any pass.
constexpr int kDraftThreads = 128;

struct SpecDraft {
    unsigned long long d0, d1; // the stream's draft slots
    unsigned long long fed;    // D0 holds the call's history h[0 .. fed)
};

struct DraftArgs {
    SpecStream *ss;                  // the target's stream records: history, budget, uniforms, drafts
    const SpecLive *live;            // [n_live] the live streams (only .s is read)
    SpecDraft *ds;                   // [n_streams]
    const unsigned long long *hist;
    PassDesc *first, *next;          // the first pass's descriptors, those of passes 2..k
    int n, k, per_first;             // live streams (all streams: k_draft_flush), drafts, streams per first pass
    const unsigned long long *pick_next; // the draft model's arg-max per row, or nullptr when sampling
    const double *pick_sample;       // its {token, margin} per row when sampling
    const double *u;                 // the call's uniforms (SpecArgs::u), or nullptr
    double *row_u;                   // [n_live] each draft row's uniform
    unsigned long long u_stride;
    const GenConstraint *gc;         // the call's automata, or nullptr
    unsigned long long *row_state;   // [n_live] each draft row's automaton state (with gc)
};

// The uniform of target row i of g this step (spec_layout's rule: 0 past the budget).
__device__ __forceinline__ double draft_u(const DraftArgs &a, const SpecStream &g, int i) {
    const unsigned long long pos = g.len + (unsigned long long)i;
    return pos < g.budget ? a.u[g.u0 + pos * a.u_stride] : 0.0;
}

__global__ void __launch_bounds__(kDraftThreads) k_draft_first(const DraftArgs a) {
    const int li = blockIdx.x * kDraftThreads + threadIdx.x;
    if (li >= a.n) return;
    const int s = a.live[li].s, W = a.k + 2;
    const SpecStream &g = a.ss[s];
    SpecDraft &d = a.ds[s];
    const unsigned long long *h = a.hist + g.h0, hl = g.hl;
    const bool live = g.done == 0;
    const int n = live ? (int)(hl - d.fed) : 0; // the segment: h[fed .. hl)
    const int j = li % a.per_first, t0 = j * W;
    PassDesc &pd = a.first[li / a.per_first];
    for (int t = 0; t < W; ++t) {
        uint32_t desc;
        if (!live) desc = (uint32_t)d.d1 | (t == 0 ? kDescFirst : 0u);
        else if (n == 1) desc = (uint32_t)d.d1 | (t == 0 ? kDescFirst | kDescLast : 0u);
        else if (t < n - 1) desc = (uint32_t)d.d0 | (t == 0 ? kDescFirst : 0u) | (t == n - 2 ? kDescLast : 0u);
        else desc = (uint32_t)d.d1 | (t == n - 1 ? kDescLast : 0u);
        pd.tokens[t0 + t] = t < n ? h[d.fed + t] : h[hl - 1];
        pd.desc[t0 + t] = desc;
    }
    pd.rows[j] = t0 + (live ? n - 1 : 0);
    if (j == 0) pd.out_row0 = li;
    if (live) d.fed = hl - 1;
    if (a.gc) a.row_state[li] = live && a.gc[s].mask ? a.gc[s].state : kNoState;
    if (a.u) a.row_u[li] = draft_u(a, g, 0);
}

// After draft i's pick: d_i into the record; for i < k, pass i + 1 (d_i on D1), the state and uniform of its row.
__global__ void __launch_bounds__(kDraftThreads) k_draft_pick(const DraftArgs a, int i) {
    const int li = blockIdx.x * kDraftThreads + threadIdx.x;
    if (li >= a.n) return;
    const int s = a.live[li].s;
    SpecStream &g = a.ss[s];
    const bool live = g.done == 0;
    const unsigned long long d = a.pick_next ? a.pick_next[li] : (unsigned long long)a.pick_sample[2 * li];
    if (live) g.row[i] = d;
    if (i == a.k) return;
    PassDesc &pd = a.next[li / kPfMaxTokens];
    const int t = li % kPfMaxTokens;
    pd.tokens[t] = d;
    pd.desc[t] = (uint32_t)a.ds[s].d1 | kDescFirst | (live ? kDescLast : 0u);
    pd.rows[t] = t;
    if (t == 0) pd.out_row0 = li;
    if (a.gc) {
        unsigned long long q = a.row_state[li];
        if (q != kNoState) {
            const GenConstraint &c = a.gc[s];
            q = gen_edge(c, q, d);
            if (q != kNoState && c.start[q] == c.start[q + 1]) q = kNoState;
        }
        a.row_state[li] = q;
    }
    if (a.u) a.row_u[li] = draft_u(a, g, i);
}

// The target's rows of a drafted step: spec_layout with the drafts k_draft_pick stored (one CTA per live stream).
__global__ void __launch_bounds__(32) k_spec_layout(const SpecArgs a) {
    const SpecLive lv = a.live[blockIdx.x];
    SpecStream &g = a.ss[lv.s];
    if ((int)threadIdx.x > g.k) return;
    const unsigned long long *h = a.hist + g.h0;
    const unsigned long long last = h[g.hl - 1];
    spec_layout(a, lv, g, g.done == 0, [&](int i) { return i == 0 ? last : g.row[i]; });
}

// The call's end: stream s (of a.n, every stream of the call) absorbs h[fed .. hl - 1) into D0, in k + 1 positions
// (a.per_first streams per pass, no head rows).
__global__ void __launch_bounds__(kDraftThreads) k_draft_flush(const DraftArgs a) {
    const int s = blockIdx.x * kDraftThreads + threadIdx.x;
    if (s >= a.n) return;
    const int W = a.k + 1;
    const SpecStream &g = a.ss[s];
    SpecDraft &d = a.ds[s];
    const unsigned long long *h = a.hist + g.h0, hl = g.hl;
    const int n = (int)(hl - 1 - d.fed), t0 = s % a.per_first * W;
    PassDesc &pd = a.first[s / a.per_first];
    for (int t = 0; t < W; ++t) {
        pd.tokens[t0 + t] = t < n ? h[d.fed + t] : h[hl - 1];
        pd.desc[t0 + t] = (uint32_t)d.d0 | (t == 0 ? kDescFirst : 0u) | (t == n - 1 ? kDescLast : 0u);
    }
    d.fed = hl - 1;
}

// One warp per live stream: lane i holds the pick p_i of row i; a = the leading i in 1..k with row[i] == p_{i - 1}.
// Lane 0 emits p_0 .. p_a by k_gen_feedback's rule (gen_emit) until one ends the stream, and moves home to the slot of
// the last row used. With `score`, it records what k_spec_logprob scores: row i emitted p_i at entry
// [s][(len + i) % max_new] (the one-shot index is below max_new; the batcher's is a ring), or nothing.
__global__ void __launch_bounds__(32) k_spec_accept(const SpecArgs a) {
    const SpecLive lv = a.live[blockIdx.x];
    const int s = lv.s, lane = threadIdx.x;
    SpecStream &g = a.ss[s];
    SpecScore *sc = a.score ? a.score + (size_t)blockIdx.x * (a.k + 1) : nullptr;
    if (g.done) {
        if (sc && lane <= a.k) sc[lane].s = -1;
        return;
    }
    const int k = g.k, r = lv.row0 + lane;
    unsigned long long p = 0;
    if (lane <= k) p = a.next ? a.next[r] : (unsigned long long)a.sample[2 * r];
    const unsigned long long prev = __shfl_up_sync(0xffffffffu, p, 1);
    const unsigned miss = __ballot_sync(0xffffffffu, lane >= 1 && (lane > k || g.row[lane] != prev));
    const int acc = __ffs((int)miss) - 2; // the first lane that misses is a + 1 (lane k + 1 always misses)
    __shared__ unsigned long long pk[kSpecMaxDraft + 1];
    if (lane <= k) pk[lane] = p;
    __syncwarp();
    if (lane != 0) return;
    unsigned long long len = g.len, hl = g.hl;
    int e = 0;
    bool stop = false;
    for (int i = 0; i <= acc && !stop; ++i) {
        const unsigned long long tok = pk[i];
        stop = gen_emit(a.emit, s, len, g.budget, tok);
        a.hist[g.h0 + hl] = tok;
        ++len;
        ++hl;
        e = i;
    }
    const unsigned long long max_new = a.emit.max_new;
    for (int i = 0; sc && i <= a.k; ++i) {
        const unsigned long long j = g.len + (unsigned long long)i;
        sc[i] = i <= e ? SpecScore{lv.row0 + i, s, (size_t)s * max_new + j % max_new} : SpecScore{0, -1, 0};
    }
    g.len = len;
    g.hl = hl;
    g.steps += 1;
    g.home = (g.home + e) % (k + 1);
    g.done = stop ? 1ull : 0ull;
}

// The log-probabilities of a step's emitted tokens, after k_spec_accept: CTA j of kNucThreads scores the token of
// score[j] by gen_logprob_at (generate_streams_logprobs' rule: raw or processed, and a batcher lane's own mode and
// top_n); a row that emitted nothing returns at once (the whole CTA).
__global__ void __launch_bounds__(kNucThreads) k_spec_logprob(const SpecArgs a, const GenLogprobArgs la) {
    const SpecScore c = a.score[blockIdx.x];
    if (c.s < 0) return;
    const int y = a.next ? (int)a.next[c.r] : (int)a.sample[2 * c.r];
    gen_logprob_at(la, c.s, c.r, y, (size_t)c.o);
}

} // namespace rk
