/* rwkv_b200.h — C ABI of the H100 (sm_90a) RWKV-v4 uint8 decode engine.
 *
 * This is the drop-in boundary: plain C, opaque handle, plain pointers and sizes,
 * no C++/torch types. Everything above it (include/rwkv/rwkv/rwkv.h, the pybind
 * module, bench.py via ctypes) is host glue; everything below it is hand-written
 * CUDA in rwkv-cpp-accelerated_b200/csrc/.
 *
 * Each entry point names the reference interface it replaces. Reference paths are
 * relative to harrisonvanderbyl/rwkv-cpp-accelerated:
 *   R.h  = include/rwkv/rwkv/rwkv.h      (backend hooks declared at R.h:63-122)
 *   R.cu = include/rwkv/cuda/rwkv.cu     (their CUDA implementation)
 *
 * Conventions: functions returning int return 0 on success and a non-zero code on
 * failure; rwkv_b200_last_error() then holds a message (thread-local). There is no
 * CPU fallback: without a usable sm_90 device every compute entry point fails.
 */
#ifndef RWKV_B200_H
#define RWKV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RWKV_B200_VOCAB 50277ULL
#define RWKV_B200_NUM_TENSORS 46

#define RWKV_B200_MODE_PARRALEL 0 /* enum MODE PARRALEL (include/rwkv/enums/enum.h:3) */
#define RWKV_B200_MODE_GPT 1      /* enum MODE GPT      (include/rwkv/enums/enum.h:4) */

typedef struct rwkv_b200_model rwkv_b200_model;

/* Last error message of the calling thread ("" if none). */
const char *rwkv_b200_last_error(void);

/* ABI version of this library (bumped on incompatible change). */
int rwkv_b200_abi_version(void);

/* Number of usable CUDA devices (0 if none / driver missing). Never throws. */
int rwkv_b200_device_count(void);

/* Load a reference-format model file onto `device` and repack it for decode.
 * Replaces `load(filename, ptrs, maxGPT)` (R.h:63, R.cu:638-717). The file layout is
 * 2 x int64 {n_layers, n_embed} followed by the 46 tensors in enum order
 * (converter/cpp_save_tensor.cpp:75-93). `max_gpt` is the number of state slots /
 * the longest token chunk a single forward may receive (R.h:281).
 * `quiet` = 0 prints the reference's "n_layers/n_embed/loading: <name>" lines.
 * Returns 0 and a handle in *out; non-zero if the file cannot be opened or parsed
 * (the reference calls exit(1) there, R.cu:641-645; the C++ wrapper keeps that). */
int rwkv_b200_load(const char *path, unsigned long long max_gpt, int device, int quiet,
                   rwkv_b200_model **out, unsigned long long *n_layers,
                   unsigned long long *n_embed);

/* Tensor-parallel load: this process is rank `tp_rank` of `tp_size` (1..8) ranks,
 * one GPU each, that decode ONE stream together (DESIGN.md section 7). Rank g owns the
 * att channels [g*E/G, (g+1)*E/G) and the ffn key channels [g*4E/G, ...): K, V, R, ffn-R,
 * ffn-K and the head are split by output channel, out-proj and ffn-V by input channel;
 * the loader reads and keeps only this rank's slices (1/G of every matrix; n_embed must
 * be a multiple of 16*G). The residual stream, layernorm and token shift are computed
 * identically on every rank; two in-kernel exchanges of partial sums per layer cross
 * NVLink. Every rank must make the same forward calls with the same tokens; all of them
 * receive the same logits and hold the complete recurrent state afterwards (state_download
 * works on any rank; state_upload must be given the same state on every rank).
 * `tp_size` = 1 is identical to rwkv_b200_load. After loading, wire the ranks with
 * rwkv_b200_tp_export / rwkv_b200_tp_import before the first forward. A rank that stops
 * calling makes the others fail with a time-out message (set_option "timeout_ms",
 * default 60000) instead of hanging. No reference counterpart (the reference is single-GPU). */
int rwkv_b200_load_tp(const char *path, unsigned long long max_gpt, int device, int quiet,
                      int tp_rank, int tp_size, rwkv_b200_model **out,
                      unsigned long long *n_layers, unsigned long long *n_embed);

/* Release every device and pinned-host allocation of the model.
 * Replaces `freeTensors(int**)` (R.h:77, R.cu:719-730). */
void rwkv_b200_free(rwkv_b200_model *m);

/* Device pointer that stands behind reference tensor-table slot `index`
 * (RWKV::tensors[index], R.h:249). State slots, scratch buffers and parameter
 * vectors keep the reference dtype and shape; the uint8 matrices are stored
 * repacked (row-major [out][in], value^0x80) — see DESIGN.md "HBM layout".
 * EMBED is a device pointer here (the reference keeps it on the host, R.cu:683). */
void *rwkv_b200_tensor(rwkv_b200_model *m, int index);

unsigned long long rwkv_b200_n_layers(const rwkv_b200_model *m);
unsigned long long rwkv_b200_n_embed(const rwkv_b200_model *m);
unsigned long long rwkv_b200_max_gpt(const rwkv_b200_model *m);

/* Pinned (page-locked) host memory for state mirrors / logits so copies are
 * asynchronous DMA. Falls back to malloc when no CUDA driver is present, so the
 * host API stays usable for tokenizer-only programs. */
void *rwkv_b200_host_alloc(size_t bytes);
void rwkv_b200_host_free(void *p);

/* Host -> device copy of the recurrent state, `slots` x n_layers x n_embed doubles per
 * array. Replaces `setState(...)` (R.h:64-66, R.cu:479-490). `pp` may be NULL
 * (the forward never reads or changes state_pp, R.cu:244,255). */
int rwkv_b200_state_upload(rwkv_b200_model *m, const double *xy, const double *aa,
                           const double *bb, const double *pp, const double *dd,
                           unsigned long long slots);

/* Device -> host copy of the recurrent state. Replaces the five state copies of
 * `getOutput(...)` (R.h:74-75, R.cu:472-476). NULL pointers are skipped. */
int rwkv_b200_state_download(rwkv_b200_model *m, double *xy, double *aa, double *bb,
                             double *pp, double *dd, unsigned long long slots);

/* Zero the device-resident state (what a fresh RWKVState holds, R.h:163-170). */
int rwkv_b200_state_zero(rwkv_b200_model *m);

/* One forward over `n_tokens` tokens on the device-resident state; blocks until the
 * logits are in `logits_out` (host, n_tokens x 50277 floats). One token = one launch of
 * the persistent token kernel; 8 tokens or more (one GPU; "prefill_min") run as int8
 * tensor-core GEMMs over the whole chunk with the weights streamed once per 128 tokens -
 * the same numbers; the chunk's launches are replayed as a CUDA graph per shape
 * (set_option "prefill" = "0" forces token by token, "prefill_graph" = "0" eager launches).
 * Replaces `cuda_rwkv_parralel(...)` + the logits copy of `getOutput`
 * (R.h:104-122, R.cu:493-593, 471). mode GPT: tokens are consumed in order on state
 * slot 0; mode PARRALEL: token t uses state slot t. n_tokens <= max_gpt. Both modes are special cases of
 * rwkv_b200_forward_streams (one stream on slot 0 / n_tokens streams of one token) with logits of every token.
 * `logits_out` may be NULL (state-only prefill: logits stay on the device). */
int rwkv_b200_forward(rwkv_b200_model *m, const unsigned long long *tokens,
                      unsigned long long n_tokens, int mode, float *logits_out);

/* Same as rwkv_b200_forward(.., 1 token, GPT) followed by an on-device argmax;
 * returns the arg-max token in *next. Used by greedy decode loops so only 8 bytes
 * cross PCIe per token. `logits_out` may be NULL. */
int rwkv_b200_forward_greedy(rwkv_b200_model *m, unsigned long long token,
                             unsigned long long *next, float *logits_out);

/* Pinned host buffer (max_gpt x 50277 floats) the engine copies logits into; passing
 * it as `logits_out` avoids one host-side memcpy. This is what RWKV::out points at. */
float *rwkv_b200_logits_host(rwkv_b200_model *m);

/* Test hook: copy a named device vector ("x" = residual stream after the last layer,
 * "logits", "trace", "ptrace") to `dst`. Returns the element count, or -1. */
long long rwkv_b200_debug_read(rwkv_b200_model *m, const char *name, void *dst, size_t dst_bytes);

/* --- measurement hooks (bench.py); not part of the reference surface ------------ */

/* Decode `n` tokens taken from `tokens` (host array, copied to HBM before timing) on
 * the resident state with no host<->device traffic inside the timed region; CUDA
 * events on the engine's stream bracket the whole run. Returns elapsed ms in *ms.
 * If `teacher_forced` is 0 only tokens[0] is used and each next token is the
 * on-device argmax of the previous logits. */
int rwkv_b200_decode_timed(rwkv_b200_model *m, const unsigned long long *tokens,
                           unsigned long long n, int teacher_forced, float *ms);

/* Number of distinct kernels in one single-token forward (1: the token kernel), and their names. */
int rwkv_b200_kernel_count(void);
const char *rwkv_b200_kernel_name(int k);

/* Run `n` single-token forwards with a CUDA-event pair around every launch.
 * ms_sum[k] = total ms spent in kernel class k, launches[k] = launch count,
 * bytes[k] = algorithmic HBM bytes of ONE launch of class k on this rank (its share of the
 * weights + the vectors). */
int rwkv_b200_profile(rwkv_b200_model *m, const unsigned long long *tokens,
                      unsigned long long n, float *ms_sum, unsigned long long *launches,
                      double *bytes);

/* Kernel launches issued by this model since load (for bench.py "gpu_launches"). */
unsigned long long rwkv_b200_launch_count(const rwkv_b200_model *m);

/* Device-side restatement of `typical(logits, temp, tau)` (R sampler/typical.h:20-58 as it actually
 * behaves, see include/rwkv/sampler/typical.h) on the logits of the LAST forward, which never leave
 * the GPU: probs = exp(l)/sum, probs ^ uint8(1/temp), cumulative sums, first index whose cumulative
 * probability reaches `u`, the uniform in [0,1) the caller drew from its generator
 * (std::generate_canonical<double,53> keeps the reference's random stream). `*margin` is the distance
 * of `u` to the nearest interval boundary; device sums are block reductions, so a caller that wants
 * the host's token in every case re-samples on the host when margin < 1e-9 (RWKV::sample does). */
int rwkv_b200_sample_typical(rwkv_b200_model *m, float temp, double u, unsigned long long *token,
                             double *margin);

/* --- multi-stream serving: independent conversations on their own state slots ------
 * No reference counterpart. One loaded model serves up to max_gpt conversations, each on its own state slot;
 * the weights are read once per pass for every live conversation. A caller either steps the conversations itself
 * (forward_streams, then the arg-max or sample_typical_streams) or hands the whole decode loop to the device
 * (generate_streams: many steps, picks and stop checks per call). Every entry point below returns
 * "not supported with tensor parallelism" when tp_size > 1, and validates its input before any work: a rejected
 * call leaves the state untouched. */

/* One ragged forward. `tokens` are stream-major: stream s owns lengths[s] consecutive tokens and advances state
 * slot slots[s]; its first token continues from what the slot holds. Slots are distinct and < max_gpt, lengths
 * >= 1 and add up to n_tokens <= max_gpt, token ids < 50277. A prompt chunk of one conversation and the next token
 * of the others may share one call. logits_out (host, [n_streams][50277]) receives each stream's logits after its
 * last token, next_out (host, [n_streams]) their arg-max taken on the device (first index on ties); both NULL =
 * state only (no head). Calls of prefill_min tokens or more run on the tensor cores in passes of at most 128
 * tokens (the same numbers, bit for bit, as each stream run alone there); shorter calls, and "prefill" = "0", run
 * token by token through the decode kernel. Slots not named are not touched. */
int rwkv_b200_forward_streams(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n_tokens,
                              const unsigned long long *slots, const unsigned long long *lengths,
                              unsigned long long n_streams, float *logits_out, unsigned long long *next_out);

/* rwkv_b200_sample_typical on each row of the last forward_streams call (which must have produced logits or
 * arg-maxes for exactly n_streams streams): row s draws with the uniform u[s] into tokens_out[s], margins_out[s]
 * (may be NULL). */
int rwkv_b200_sample_typical_streams(rwkv_b200_model *m, unsigned long long n_streams, float temp,
                                     const double *u, unsigned long long *tokens_out, double *margins_out);

/* Generate up to max_new tokens for each of n_streams conversations without returning to the host between steps.
 * Stream s continues on state slot slots[s]; its first input is first_tokens[s]. Each step feeds every live stream
 * its current token, picks the next one on the device, and emits it: arg-max when u == NULL (first index on ties),
 * else the typical sampler of rwkv_b200_sample_typical_streams with temp and the uniform u[step * n_streams + s]
 * (u: [max_new][n_streams], each in [0, 1)). Before each pick, logits[override_tokens[i]] = override_values[i]
 * (e.g. -99 on token 0 keeps a story from ending).
 * A stream stops after emitting a token in stop_tokens, or after budgets[s] tokens (NULL = max_new for every stream;
 * otherwise each in 1..max_new). The emitted stop token / last token is NOT fed: the slot ends where the equivalent
 * host loop (forward_streams, pick, append, check) would leave it, so a caller continues a conversation by feeding
 * tokens_out[s][lengths_out[s] - 1]. Emitted tokens and the slot states are bit for bit those of that loop run on the
 * same path: the tensor cores when n_streams >= prefill_min (and "prefill" is on), else the decode kernel; the path
 * does not change inside a call.
 * The device draw is final: unlike RWKV::sample, nothing re-samples on the host when the margin of u is below 1e-9.
 * tokens_out: [n_streams][max_new] host (entries past lengths_out[s] are 0); lengths_out: [n_streams] host.
 * Slots are distinct and < max_gpt, token ids < 50277, max_new >= 1; a count > 0 needs its array. After the call no
 * per-stream logits are held: rwkv_b200_sample_typical_streams is refused until the next forward_streams. */
int rwkv_b200_generate_streams(rwkv_b200_model *m, const unsigned long long *slots,
                               const unsigned long long *first_tokens, unsigned long long n_streams,
                               unsigned long long max_new, const unsigned long long *budgets,
                               const unsigned long long *stop_tokens, unsigned long long n_stop,
                               const unsigned long long *override_tokens, const float *override_values,
                               unsigned long long n_override, float temp, const double *u,
                               unsigned long long *tokens_out, unsigned long long *lengths_out);

/* A stream's sampler for rwkv_b200_sample_streams and rwkv_b200_generate_streams_ex. Per row of logits l:
 *  1. penalties (generate_streams_ex only): every token v the stream emitted earlier in the call has
 *     l[v] -= presence_penalty + frequency_penalty * cnt[v], in f32 with each operation rounded (no FMA), where cnt[v]
 *     is the decayed count: after each emitted token x, every count is multiplied by penalty_decay, then cnt[x] += 1.
 *     The history starts empty in every call; prompt tokens are not counted;
 *  2. the logit overrides, so an override value is final;
 *  3. temperature 0: the arg-max, first index on ties (what forward_streams' next_out holds); u is not read;
 *  4. temperature T > 0: p[v] = exp((l[v] - max l) / T) in double. Ranking tokens by l descending (ties: lower index
 *     first), the kept set is the first min(n_p, top_k) of them, n_p the smallest count whose mass reaches
 *     top_p * sum(p). The draw walks the kept tokens in vocabulary order and takes the first one with p > 0 whose
 *     cumulative share of the kept mass reaches u. The cut and the draw run on the device without a sort; outputs
 *     depend only on the row and the parameters (bit-deterministic). */
typedef struct rwkv_b200_sampler {
    float temperature;      /* 0 = arg-max (first index on ties); else > 0 */
    float top_p;            /* (0, 1]; 1 = no cut */
    unsigned int top_k;     /* 0 = no limit; <= 50277 */
    float presence_penalty; /* generate_streams_ex only (|x| <= 1e6); 0 elsewhere */
    float frequency_penalty;/* generate_streams_ex only (|x| <= 1e6); 0 elsewhere */
    float penalty_decay;    /* (0, 1]; generate_streams_ex only (not read elsewhere) */
} rwkv_b200_sampler;

/* Draw one token per row with per-row samplers params[s] (penalties must be 0) and uniforms u[s] in [0, 1) (u may be
 * NULL when every row has temperature 0). logits == NULL: the rows of the last forward_streams call, which must have
 * produced logits or arg-maxes for exactly n_streams streams. Otherwise the caller's host rows
 * ([n_streams][50277], n_streams <= max_gpt; no NaN or +inf, at least one finite value per row, -inf masks a token)
 * are sampled, e.g. after constrained decoding edited them; they replace the per-stream logits of the last forward,
 * so rwkv_b200_sample_typical_streams is refused until the next forward_streams. tokens_out[s] receives the token,
 * margins_out[s] (may be NULL) the distance of u to the edges of the token's cumulative interval (1 for temperature
 * 0): a caller with a host restatement of the rule can trust equal picks when the margin is >= 1e-9. */
int rwkv_b200_sample_streams(rwkv_b200_model *m, unsigned long long n_streams, const rwkv_b200_sampler *params,
                             const double *u, const float *logits, unsigned long long *tokens_out, double *margins_out);

/* rwkv_b200_generate_streams with a sampler per stream (samplers[n_streams]; NULL = arg-max for every stream, u not
 * read) in place of temp: greedy and sampled streams may share one call, and presence / frequency penalties apply to the
 * tokens each stream emits in this call. u: [max_new][n_streams] as for generate_streams; it may be NULL only if every
 * stream has temperature 0. Override values must be finite or -inf and may not set every token to -inf. Stops, budgets,
 * continuation, the forward path, untouched slots and the refusals are those of generate_streams; each step is bit for
 * bit forward_streams, the penalties in f32, the overrides, then rwkv_b200_sample_streams on those logits with the same
 * u. The penalty history ([n_streams][50277] counts and flags) is allocated at the first call that uses penalties. */
int rwkv_b200_generate_streams_ex(rwkv_b200_model *m, const unsigned long long *slots,
                                  const unsigned long long *first_tokens, unsigned long long n_streams,
                                  unsigned long long max_new, const unsigned long long *budgets,
                                  const unsigned long long *stop_tokens, unsigned long long n_stop,
                                  const unsigned long long *override_tokens, const float *override_values,
                                  unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                  unsigned long long *tokens_out, unsigned long long *lengths_out);

/* Scoring: how likely a text is under the model (perplexity, log-likelihood and multiple-choice evaluation, reranking,
 * prompt log-probabilities). A position without a target holds RWKV_B200_NO_TARGET; at most RWKV_B200_MAX_TOP_N top
 * alternatives per position. */
#define RWKV_B200_NO_TARGET 0xFFFFFFFFFFFFFFFFULL
#define RWKV_B200_MAX_TOP_N 20

/* A ragged forward that scores target tokens on the device. tokens, slots and lengths are those of
 * rwkv_b200_forward_streams, with the same validation and the same forward path: each slot advances by its tokens to the
 * same bits as forward_streams. targets[t] is the token expected after tokens[t], or RWKV_B200_NO_TARGET for a position
 * that is not scored (e.g. the context before a continuation; the last target of one chunk of a long document is the
 * first token of the next chunk). For a scored position, with l the f32 logits after tokens[t] and y = targets[t]:
 *   logprobs_out[t] = ((double)l[y] - m) - log(S), m = max l, S = sum exp((double)l[v] - m) in double, in a fixed order;
 *   ranks_out[t]    = the number of tokens ranked before y, ranking by l descending, ties by lower index, -0 with +0
 *                     (0 exactly when y is the arg-max that forward_streams' next_out reports);
 *   top_tokens_out[t][k], top_logprobs_out[t][k] (k < top_n <= RWKV_B200_MAX_TOP_N): the first top_n tokens of that
 *                     ranking, in order, with their logprobs by the same formula (bit for bit the logprob reported when
 *                     that token is the target).
 * An unscored position receives NaN, and RWKV_B200_NO_TARGET in its rank and top tokens (NaN top logprobs).
 * logprobs_out ([n_tokens]) and targets are required; ranks_out ([n_tokens]) may be NULL; top_tokens_out and
 * top_logprobs_out ([n_tokens][top_n]) are required when top_n > 0 and not read otherwise. The results depend only on
 * each row's logits, so they are deterministic, and a stream scores the same bits in any ragged call on the same path.
 * Only the results cross PCIe: 16 bytes per scored position plus the top entries. A call without any target is a
 * state-only forward; on the tensor cores a pass without a scored position runs no head. Refused before any work
 * (every slot untouched): the refusals of forward_streams, a target >= 50277 other than RWKV_B200_NO_TARGET,
 * top_n > RWKV_B200_MAX_TOP_N, missing arrays, and tensor parallelism. After the call no per-stream logits are held:
 * rwkv_b200_sample_typical_streams and rwkv_b200_sample_streams (without logits) are refused until the next
 * forward_streams. */
int rwkv_b200_score_streams(rwkv_b200_model *m, const unsigned long long *tokens, unsigned long long n_tokens,
                            const unsigned long long *slots, const unsigned long long *lengths,
                            unsigned long long n_streams, const unsigned long long *targets, unsigned int top_n,
                            double *logprobs_out, unsigned long long *ranks_out,
                            unsigned long long *top_tokens_out, double *top_logprobs_out);

/* Which row rwkv_b200_generate_streams_logprobs scores an emitted token on. */
#define RWKV_B200_LOGPROBS_RAW       0 /* the model's logits, before penalties and overrides (tau = 1) */
#define RWKV_B200_LOGPROBS_PROCESSED 1 /* the row the sampler read, divided by the stream's temperature */

/* rwkv_b200_generate_streams_ex that also reports how likely each emitted token was (completion logprobs and
 * top_logprobs, confidence displays, the sampling log-probabilities of RL rollouts), scored on the device after each
 * pick; only the results cross PCIe, once, at the end of the call. Every argument up to lengths_out, the emitted tokens,
 * the lengths, the slot states and every refusal are exactly those of rwkv_b200_generate_streams_ex: asking for
 * log-probabilities changes no token and no state bit.
 * Entry [s][k] (k < lengths_out[s]) describes the k-th token y stream s emitted, by the rule of
 * rwkv_b200_score_streams on a row l with a divisor tau:
 *   z[v] = ((double)l[v] - m) / tau, m = max l;  logprobs_out[s][k] = z[y] - log(sum_v exp(z[v]));
 *   ranks_out[s][k] and top_tokens_out[s][k][0..top_n) rank by l descending, ties by lower index, -0 with +0; each top
 *   entry carries its token's logprob by the same formula (bit for bit the logprob reported when it is emitted).
 * logprob_mode RWKV_B200_LOGPROBS_RAW: l is the model's logits row of the step, before penalties and overrides, and
 *   tau = 1: bit for bit what rwkv_b200_score_streams reports for that token after the same prefix on the same path.
 * logprob_mode RWKV_B200_LOGPROBS_PROCESSED: l is the row the sampler read, after penalties and overrides, and tau is
 *   the stream's temperature (1 for temperature 0 and when samplers == NULL): the distribution before the top-p /
 *   top-k cut, so a token outside the kept set still has a finite logprob.
 * Positions at or beyond lengths_out[s] receive NaN, and RWKV_B200_NO_TARGET in the rank and top tokens (NaN top
 * logprobs). logprobs_out ([n_streams][max_new]) is required; ranks_out (same shape) may be NULL; top_tokens_out and
 * top_logprobs_out ([n_streams][max_new][top_n]) are required when top_n > 0 and not read otherwise. Refused before any
 * work (every slot untouched): a logprob_mode other than the two above, top_n > RWKV_B200_MAX_TOP_N, missing arrays, and
 * every refusal of generate_streams_ex, tensor parallelism included. Each step runs one more kernel than
 * generate_streams_ex, plus, in raw mode with penalties or overrides, a device-to-device copy of the step's rows. The
 * typical sampler of rwkv_b200_generate_streams has no counterpart here. */
int rwkv_b200_generate_streams_logprobs(rwkv_b200_model *m, const unsigned long long *slots,
                                        const unsigned long long *first_tokens, unsigned long long n_streams,
                                        unsigned long long max_new, const unsigned long long *budgets,
                                        const unsigned long long *stop_tokens, unsigned long long n_stop,
                                        const unsigned long long *override_tokens, const float *override_values,
                                        unsigned long long n_override, const rwkv_b200_sampler *samplers,
                                        const double *u, unsigned long long *tokens_out,
                                        unsigned long long *lengths_out, int logprob_mode, unsigned int top_n,
                                        double *logprobs_out, unsigned long long *ranks_out,
                                        unsigned long long *top_tokens_out, double *top_logprobs_out);

/* Constrained generation: output that must follow a format (JSON with fixed keys, a number, a date, one of a few labels)
 * without returning to the host per step. A token automaton has n_states states; state q has the edges
 * (edge_tokens[e], edge_next[e]) for e in [edge_start[q], edge_start[q + 1]), sorted by token, no token twice in a state.
 * A state without edges is complete. A constrained stream carries its current state q, and each step is:
 *  1. the row passes through the penalties, then the logit overrides, exactly as in rwkv_b200_generate_streams_ex;
 *  2. mask: every token v without an edge out of q gets l[v] = -inf, after the overrides, so an override cannot re-enable
 *     a token the automaton forbids (the bits are those of numpy's row[~allowed] = -np.inf);
 *  3. the pick (arg-max or the sampler of rwkv_b200_sampler) runs on the masked row with the same u;
 *  4. after emitting y, q = next(q, y);
 *  5. if the new state has no edges the stream is done, like after a stop token: the emitted token is not fed.
 * Stop tokens and budgets still apply; whichever condition comes first ends the stream. The device keeps the CSR arrays
 * and one allow bitmask per state: ceil(50277 / 32) u32 words, 6288 bytes per state, plus 8 bytes per state and per
 * edge. The host keeps the CSR too (the override check below). Tools that build automata from regular expressions over
 * the tokenizer's bytes are in the Python package (constrain.py). */
#define RWKV_B200_NO_CONSTRAINT 0xFFFFFFFFFFFFFFFFULL /* constraint_ids entry of a stream without a constraint */
#define RWKV_B200_MAX_CONSTRAINT_STATES 65536

/* Upload a token automaton in CSR form (edge_start [n_states + 1], edge_tokens and edge_next [edge_start[n_states]]);
 * *id receives its id for rwkv_b200_generate_streams_constrained. Refused: n_states == 0 or >
 * RWKV_B200_MAX_CONSTRAINT_STATES, edge_start not starting at 0 or decreasing, an edge token >= 50277, tokens not strictly
 * ascending within a state, an edge_next >= n_states, and tensor parallelism. */
int rwkv_b200_constraint_add(rwkv_b200_model *m, unsigned long long n_states, const unsigned long long *edge_start,
                             const unsigned long long *edge_tokens, const unsigned long long *edge_next,
                             unsigned long long *id);
/* Free an automaton (an unknown or removed id is refused, and so is an id that an unfinished request of the model's
 * batcher names). rwkv_b200_free frees every automaton of the model. */
int rwkv_b200_constraint_remove(rwkv_b200_model *m, unsigned long long id);

/* rwkv_b200_generate_streams_logprobs with a token automaton per stream, by the rule above. constraint_ids[n_streams]:
 * an id of rwkv_b200_constraint_add, or RWKV_B200_NO_CONSTRAINT; NULL = no stream has a constraint. start_states
 * [n_streams]: each constrained stream's first state (NULL = state 0). states_out [n_streams] (may be NULL): each
 * constrained stream's final state (0 for the others), so a caller can continue a constrained generation in the next call
 * or check that it completed. logprobs_out == NULL: nothing is scored, and logprob_mode, top_n, ranks_out,
 * top_tokens_out and top_logprobs_out are not read. Streams without a constraint generate bit for bit as in
 * generate_streams_ex; with constraint_ids == NULL and logprobs_out == NULL the call is generate_streams_ex. Log-probabilities
 * in processed mode are taken on the masked row: the rank counts the tokens that rank before y (masked tokens rank last),
 * and a top entry past the allowed tokens is a masked token in index order with logprob -inf. Raw mode scores the model's
 * row. Refused before any work (every slot untouched): every refusal of generate_streams_logprobs (with logprobs_out
 * != NULL) or generate_streams_ex, an unknown or removed id, a start state out of range or without edges, and an automaton
 * with a state with edges whose every edge token this call's overrides set to -inf. Each step of a call with a constraint
 * runs one more kernel (k_gen_mask). A token emitted without an edge (a broken pick) fails the call at the end of its
 * 16-step group with a message naming the stream, the token and the state. */
int rwkv_b200_generate_streams_constrained(rwkv_b200_model *m, const unsigned long long *slots,
                                           const unsigned long long *first_tokens, unsigned long long n_streams,
                                           unsigned long long max_new, const unsigned long long *budgets,
                                           const unsigned long long *stop_tokens, unsigned long long n_stop,
                                           const unsigned long long *override_tokens, const float *override_values,
                                           unsigned long long n_override, const rwkv_b200_sampler *samplers,
                                           const double *u, unsigned long long *tokens_out,
                                           unsigned long long *lengths_out, int logprob_mode, unsigned int top_n,
                                           double *logprobs_out, unsigned long long *ranks_out,
                                           unsigned long long *top_tokens_out, double *top_logprobs_out,
                                           const unsigned long long *constraint_ids,
                                           const unsigned long long *start_states, unsigned long long *states_out);

/* Beam search on the device: the n_best best continuations of each of n_groups prompts (translation, summarisation,
 * extraction, n-best reranking). Group g owns the `beams` = B distinct slots slots[g * B .. g * B + B): slots[g * B]
 * holds the prompt state, the others are overwritten. Its first input is first_tokens[g] (the (slot, first_token)
 * convention of generate_streams). max_new = N, the stop tokens Z, length_penalty = alpha (any finite value) and
 * n_best = K (1 <= K <= B) are shared by every group; B + n_stop <= RWKV_B200_MAX_TOP_N. The rule, per group:
 *  1. Step 0 has one live beam: cum = 0, no tokens, input first_tokens[g] on slots[g * B]. Later steps have B live
 *     beams, j = 0..B-1.
 *  2. Expansion: each live beam's logits row l of the step gives the first B + n_stop tokens of the ranking (l
 *     descending, ties by lower index: the ranking of rwkv_b200_score_streams) with their logprobs by score_streams'
 *     formula, bit for bit what score_streams reports as top entries. A candidate's score is c = cum + logprob (double).
 *  3. The group's candidates are ordered by (c descending, beam index ascending, rank in its row ascending).
 *  4. Walk from position 0: a stop token at position < B is offered to the hypothesis list as a finished hypothesis (the
 *     beam's tokens and the stop token, len = that length, score = c / P[len]); a stop token at position >= B is skipped;
 *     every other token becomes the next new live beam until there are B of them (new beam j = the j-th such candidate).
 *  5. P[n] = pow((double)n, alpha) for n = 1..N, computed on the host by the C library's pow.
 *  6. The hypothesis list keeps the K best offered hypotheses by (score descending, offer order ascending); a new one
 *     enters only when fewer than K are held or its score is strictly above the worst one held.
 *  7. After the walk of step N - 1 the B live beams are offered in order j as unfinished hypotheses (len = N).
 *  8. A group is done when it holds K hypotheses and no live beam can beat the worst of them: a live beam with cum c and
 *     n tokens can score at most c / P[N] when alpha >= 0, and c / P[n + 1] when alpha < 0 (every logprob is <= 0). The
 *     result is exactly what running every group to N steps returns. A done group runs no more steps.
 *  9. Slots: after the walk, new beam j with parent p takes p's slot if no earlier new beam took it, else the next free
 *     slot: the slots of the previous beams without a child, in ascending beam index (at step 0: slots[g * B + 1 ..
 *     g * B + B), in that order), and a copy of the parent's state (rwkv_b200_slot_copy). A group that becomes done
 *     copies nothing, so its slots hold the states its last step's beams left (no slot holds a hypothesis' final state:
 *     a caller continues a hypothesis by feeding its text with forward_streams).
 * The forward path is forward_streams' rule for n_groups * beams one-token streams, chosen once per call.
 * Outputs, hypotheses best first, each group exactly n_best of them: tokens_out [n_groups][n_best][max_new] (0 past the
 * length), lengths_out [n_groups][n_best], logprobs_out [n_groups][n_best] (cum: the left-to-right double sum of the
 * token logprobs), scores_out [n_groups][n_best], finished_out [n_groups][n_best] (1: ended by a stop token), and, if
 * not NULL, token_logprobs_out [n_groups][n_best][max_new] (NaN past the length). Refused before any work (every slot
 * untouched): a missing required array, n_groups == 0, beams == 0, beams + n_stop > RWKV_B200_MAX_TOP_N, n_best == 0 or
 * > beams, max_new == 0, a slot out of range or repeated, a first or stop token >= 50277, a non-finite length_penalty,
 * and tensor parallelism. After the call no per-stream logits are held, as after generate_streams. */
int rwkv_b200_beam_search(rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens,
                          unsigned long long n_groups, unsigned beams, unsigned long long max_new,
                          const unsigned long long *stop_tokens, unsigned long long n_stop, double length_penalty,
                          unsigned n_best, unsigned long long *tokens_out, unsigned long long *lengths_out,
                          double *logprobs_out, double *scores_out, unsigned char *finished_out,
                          double *token_logprobs_out);

/* Speculative generation with prompt-lookup drafts: rwkv_b200_generate_streams_ex that may emit several tokens per stream
 * per step, with the same tokens. Every argument up to lengths_out is that of generate_streams_ex, except that each
 * stream names draft + 1 distinct slots: slots[n_streams][draft + 1]. slots[s][0] is the stream's first slot and holds
 * its conversation; the others are scratch, and their contents after the call are unspecified. draft = k (1..15) drafts
 * per step, ngram (1..8) the longest n-gram looked up. context_start [n_streams + 1] (CSR, context_start[0] = 0) and
 * context give each stream extra lookup tokens context[context_start[s] .. context_start[s + 1]) (e.g. the prompt, or a
 * document the answer quotes); context_start == NULL: none. steps_out [n_streams] receives the steps in which each
 * stream emitted a token, so lengths_out[s] / steps_out[s] is the stream's tokens per step.
 * The rule. h = context_s ++ [first_s] ++ the tokens stream s emitted so far in this call, L = len(h).
 *  1. Drafts: for n = ngram down to 1 with n < L, the largest j <= L - n - 1 with h[j .. j+n) == h[L-n .. L); the first
 *     n that has one gives the proposal h[j+n .. min(j+n+k, L)]. The k drafts d_1..d_k are the proposal padded by
 *     repeating its last token, or k copies of h[L-1] when no n matches.
 *  2. A step gives stream s k + 1 consecutive rows of one tensor-core pass: row 0 feeds its current input, row i feeds
 *     d_i. After the overrides, the pick p_i of row i uses the stream's sampler and the uniform u[(len + i) * n_streams
 *     + s], len = the tokens emitted before the step.
 *  3. a = the number of leading i in 1..k with d_i == p_(i-1). The step emits p_0 .. p_a in order, each with the stop and
 *     budget check of generate_streams; tokens after a stop or past the budget are dropped. The next input is the last
 *     emitted token, and the state continues from the slot of the row that produced it (emitted, not fed).
 * Because each row of a pass is exact and a stream's bits depend only on its own rows, the logits of row i are bit for
 * bit those generate_streams_ex computes at position len + i. So the emitted tokens, the lengths and the first slots'
 * xy, aa, bb and dd are bit for bit those of generate_streams_ex on the first slots with the same first tokens, budgets,
 * stops, overrides, samplers and u, run on the tensor cores, whatever the drafts are: drafts change the speed, never the
 * tokens. A first slot's pp is untouched (no forward writes it); slots no stream names are untouched. steps_out depends
 * only on the emitted tokens and the contexts, so a host can restate it exactly. Each step's passes hold floor(128 /
 * (draft + 1)) streams; streams leave the rows at 16-step group boundaries, as in generate_streams.
 * Refused before any work (every slot untouched): the refusals of generate_streams_ex, n_streams * (draft + 1) >
 * max_gpt, a slot repeated anywhere in slots, draft or ngram out of range, a missing steps_out, context offsets that do
 * not start at 0 or decrease, a context token >= 50277, a presence or frequency penalty, "prefill" set to 0, and tensor
 * parallelism. The call always runs on the tensor cores, whatever prefill_min is. After it no per-stream logits are held. */
int rwkv_b200_generate_streams_speculative(rwkv_b200_model *m, const unsigned long long *slots,
                                           const unsigned long long *first_tokens, unsigned long long n_streams,
                                           unsigned long long max_new, const unsigned long long *budgets,
                                           const unsigned long long *stop_tokens, unsigned long long n_stop,
                                           const unsigned long long *override_tokens, const float *override_values,
                                           unsigned long long n_override, const rwkv_b200_sampler *samplers,
                                           const double *u, unsigned long long *tokens_out,
                                           unsigned long long *lengths_out, unsigned int draft, unsigned int ngram,
                                           const unsigned long long *context_start, const unsigned long long *context,
                                           unsigned long long *steps_out);

/* Continuous batching: a batcher accepts requests at any time between runs and serves them together, so a request that
 * arrives while others generate starts at the next 16-step group instead of after the whole batch, and the rows freed
 * by finished requests are refilled at once. A request names a state slot, its prompt (n_prompt >= 1 tokens), max_new
 * >= 1, a sampler (penalties allowed), u[max_new] (NULL only at temperature 0) and its own stop tokens.
 *
 * The rule. For every request, the emitted tokens and the slot's final state are bit for bit what this sequence gives
 * when the request runs alone from the same slot state, both calls on the tensor cores:
 *   1. if n_prompt > 1: rwkv_b200_forward_streams of prompt[0 .. n_prompt - 1) on the slot, state only;
 *   2. rwkv_b200_generate_streams_ex of the one stream (slot, prompt[n_prompt - 1]) with max_new, the request's stop
 *      tokens, its sampler and its u.
 * This holds whatever the other requests are, when each was submitted, rows, prefill_tokens, the max_steps of each run,
 * and any cancellation of other requests. A request's penalty history starts empty at its first emitted token, as in
 * step 2. A cancelled request's tokens are a prefix of that sequence's tokens. Slots that no unfinished request names
 * are never written.
 * A request submitted with rwkv_b200_batcher_submit_ex may also carry logit overrides, a token automaton and
 * log-probabilities. Then step 2 is rwkv_b200_generate_streams_constrained of the one stream with, besides the above,
 * the request's overrides as the call's overrides, its constraint id and start state (or constraint_ids == NULL), and
 * its logprob_mode and top_n (or logprobs_out == NULL); without any of the three that call is generate_streams_ex, as
 * above. Its emitted tokens, the slot's final state, the log-probabilities, ranks and top entries and the final
 * automaton state are bit for bit that call's. Each step's order is the one-shot calls': forward, the copy of the
 * model's rows that raw mode reads (when some edit would change them), penalties, this request's overrides, its
 * automaton's mask, the pick, the scoring, the feedback. A request whose automaton reaches a state without edges ends
 * as RWKV_B200_REQ_DONE, like after a stop token (emitted, not fed). A cancelled request's log-probabilities are a
 * prefix of that call's, and its automaton state is the state after its emitted tokens. The rule rests on the ragged-pass invariant: a stream's bits depend only on its own rows and its
 * own predecessors, and cutting it across passes changes no bit.
 *
 * Scheduling (deterministic). A run is a series of groups of 16 steps (the last one of a run may be shorter), with one
 * synchronisation per group:
 *   - requests queue FIFO. At a group boundary finished requests leave first; queued requests are then admitted in
 *     submission order while fewer than `rows` are admitted;
 *   - an admitted request first prefills prompt[0 .. n_prompt - 1). Each step hands a budget of prefill_tokens prompt
 *     tokens to the prefilling requests in admission order, each taking as much of its remaining prompt as the budget
 *     allows, so the pass shape stays the same from step to step while prompt work lasts;
 *   - a request whose prefill is complete at a group boundary (at admission when n_prompt = 1) has a decode row for the
 *     whole group; its first input is prompt[n_prompt - 1]. Rows change only at group boundaries, so a request whose
 *     prefill completes inside a group waits up to 15 steps for its first token. A group without decode rows ends after
 *     its last step with prompt work;
 *   - a step is one set of tensor-core passes: the decode rows first (one token each, with logits), then the prefill
 *     segments (no logits), cut into passes of at most 128 tokens; then penalties, overrides, masks, the per-request sampler, scoring and the
 *     feedback that emits each row's token and writes it into the next step's passes.
 * At each group end the tokens emitted in the group come back, so rwkv_b200_batcher_read between runs sees a growing
 * prefix (streaming).
 *
 * The batcher always runs on the tensor cores: the rule is defined on that path. With only a few generating requests
 * the decode kernel of rwkv_b200_generate_streams is faster (at 7B: one stream 3.1 ms per step there, a tensor-core step
 * of 8 streams 10.3 ms, on an H100 SXM 80 GB at a 400 W power limit; tensor-core steps under 8 rows have not been
 * measured). Not available in the batcher: the typical sampler, admission inside a group, the decode-kernel path,
 * tensor parallelism, priorities and preemption.
 *
 * Other entry points may be called between runs, but must not name a slot held by an unfinished request (queued,
 * prefilling or generating); the batcher does not police that. rwkv_b200_free closes a model's open batcher, whose handle
 * is then invalid. */
typedef struct rwkv_b200_batcher rwkv_b200_batcher;
typedef struct rwkv_b200_request {
    unsigned long long slot;
    const unsigned long long *prompt; /* [n_prompt] */
    unsigned long long n_prompt;      /* >= 1 */
    unsigned long long max_new;       /* >= 1 */
    rwkv_b200_sampler sampler;
    const double *u;                  /* [max_new] uniforms in [0, 1), or NULL (temperature 0) */
    const unsigned long long *stop;   /* [n_stop] this request's stop tokens (emitted, not fed) */
    unsigned long long n_stop;
} rwkv_b200_request;

/* What rwkv_b200_batcher_submit_ex adds to a request (the rule above). */
typedef struct rwkv_b200_request_ex {
    const unsigned long long *override_tokens; /* [n_override] logit overrides, in order (a repeated token keeps its last) */
    const float *override_values;              /* [n_override] finite or -inf, not every token -inf */
    unsigned long long n_override;
    unsigned long long constraint_id;          /* an id of rwkv_b200_constraint_add, or RWKV_B200_NO_CONSTRAINT */
    unsigned long long start_state;            /* the automaton's first state (read with a constraint only) */
    int logprobs;                              /* 0: none; else every emitted token is scored */
    int logprob_mode;                          /* RWKV_B200_LOGPROBS_RAW or _PROCESSED (read when logprobs != 0) */
    unsigned int top_n;                        /* 0..RWKV_B200_MAX_TOP_N top entries per token (idem) */
} rwkv_b200_request_ex;

#define RWKV_B200_BATCHER_MAX_PREFILL 2048ULL /* prefill_tokens is 1..this */

/* Status of a request (rwkv_b200_batcher_read). */
#define RWKV_B200_REQ_QUEUED     0
#define RWKV_B200_REQ_PREFILLING 1 /* admitted, its prompt not yet fed or its decode row not yet begun */
#define RWKV_B200_REQ_GENERATING 2
#define RWKV_B200_REQ_DONE       3 /* a stop token or max_new tokens */
#define RWKV_B200_REQ_CANCELLED  4

/* Open the model's batcher: at most `rows` (1..max_gpt) admitted requests, prefill_tokens (1..
 * RWKV_B200_BATCHER_MAX_PREFILL) prompt tokens per step. Refused with tensor parallelism, with set_option "prefill" = 0,
 * and while the model has an open batcher (one per model). The batcher owns its device buffers; it shares only the
 * model's per-step scratch (logits rows and sampler results). */
int rwkv_b200_batcher_open(rwkv_b200_model *m, unsigned long long rows, unsigned long long prefill_tokens,
                           rwkv_b200_batcher **out);
/* Queue a request; *id receives its id (never 0). Copies every array (the caller may free them afterwards) and does
 * no device work. Refused: a slot out of range or named by an unfinished request of this batcher, n_prompt or max_new
 * of 0, a missing array, a token out of range, an invalid sampler (generate_streams_ex's checks), u NULL with a
 * temperature > 0, and a uniform outside [0, 1). */
int rwkv_b200_batcher_submit(rwkv_b200_batcher *b, const rwkv_b200_request *r, unsigned long long *id);
/* rwkv_b200_batcher_submit with the extension x (NULL: exactly rwkv_b200_batcher_submit). Refused as well, with nothing
 * queued and no id used: an override token out of range, an override value that is NaN or +inf, overrides that set
 * every token to -inf, n_override > 0 with a NULL array, an unknown or removed constraint id, a start state out of range
 * or without edges, overrides that set every edge token of some state of the automaton to -inf, and with logprobs a
 * logprob_mode other than the two or top_n > RWKV_B200_MAX_TOP_N. While the request is unfinished its automaton cannot
 * be removed (rwkv_b200_constraint_remove refuses). A group whose decode rows use none of these features enqueues
 * exactly what it would without them. */
int rwkv_b200_batcher_submit_ex(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                unsigned long long *id);
/* Run up to max_steps steps in groups of 16; stops early when nothing is queued or admitted. *steps_run (may be NULL)
 * receives the steps run. */
int rwkv_b200_batcher_run(rwkv_b200_batcher *b, unsigned long long max_steps, unsigned long long *steps_run);
/* The tokens a request has emitted so far: *len receives their count, tokens_out the first min(cap, *len) of them
 * (tokens_out may be NULL when cap is 0), *status its RWKV_B200_REQ_* status (len and status may be NULL). An unknown
 * or released id is refused. */
int rwkv_b200_batcher_read(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *tokens_out,
                           unsigned long long cap, unsigned long long *len, int *status);
/* rwkv_b200_batcher_read with the results of submit_ex: the first min(cap, *len) emitted tokens, their logprobs and
 * ranks, and top_tokens_out / top_logprobs_out [cap][top_n] (the request's top_n), as generate_streams_logprobs reports
 * them; *state_out the automaton's current state (0 without a constraint). Every array and pointer may be NULL (then it
 * is skipped); the log-probability arrays are refused for a request that is not scored. */
int rwkv_b200_batcher_read_ex(rwkv_b200_batcher *b, unsigned long long id, unsigned long long cap,
                              unsigned long long *tokens_out, double *logprobs_out, unsigned long long *ranks_out,
                              unsigned long long *top_tokens_out, double *top_logprobs_out,
                              unsigned long long *state_out, unsigned long long *len, int *status);
/* Cancel a queued, prefilling or generating request at once (calls are made between runs). A queued request's slot is
 * untouched; otherwise the slot holds the state after the tokens fed so far (its emitted tokens but the last one, as
 * after a stop token). Its tokens stay readable. A done or cancelled request, or an unknown id, is refused. */
int rwkv_b200_batcher_cancel(rwkv_b200_batcher *b, unsigned long long id);
/* Forget a done or cancelled request; anything else is refused. */
int rwkv_b200_batcher_release(rwkv_b200_batcher *b, unsigned long long id);
/* Close the batcher and free its buffers; unfinished requests are dropped where they stand. NULL is ignored. */
void rwkv_b200_batcher_close(rwkv_b200_batcher *b);

/* Stop strings: end a stream when the text it emits contains one of its stop strings ("\n\nUser:", "</answer>"), which
 * may start or end in the middle of a token and be spelled by many token sequences. A stop set is 1..n non-empty byte
 * strings of at most RWKV_B200_MAX_STOP_BYTES bytes in total. A stream with a set carries a match state; B is the byte
 * string of the tokens it emits in the call, each token's bytes as GPT2Tokenizer::decode({id}) gives them (the table of
 * rwkv_b200_token_bytes_set), prefixed by the text its start state carries over from an earlier call.
 *  1. The stream ends after the first emitted token t_j whose bytes complete an occurrence of a string of the set in B
 *     (the occurrence may begin in earlier tokens or in the carried text). t_j is emitted, not fed, like a stop token:
 *     it is in tokens_out and counts in the length, and the slot holds the state after t_(j-1) was fed.
 *  2. hit = 1 + the index of the matched string (among the strings ending at the earliest end byte, the lowest index),
 *     or 0 when the stream ended otherwise; tail = the bytes of t_j after the end of the occurrence; state = the final
 *     match state. So the text before the match is B[:len(B) - tail - len(string)].
 *  3. Stop tokens, budgets and token automata keep their meaning; whichever comes first ends the stream, and when a stop
 *     string and one of them end it on the same token, hit still reports the string.
 * The tokens and lengths are a prefix of the same call without stop sets, and each named slot holds bit for bit the state
 * of that call run with the stream's budget set to min(budget, j + 1). A stream without a set (RWKV_B200_NO_STOP_SET)
 * generates exactly as without this feature, and a call in which no stream has a set enqueues exactly what the call
 * without a stop request enqueues.
 * Match states: state q is the q-th distinct prefix of the set's strings in order of first appearance (0 the empty
 * prefix, then the prefixes of string 0 by length, then the new prefixes of string 1, and so on); the state after B is
 * the longest suffix of B that is a prefix of some string, and a start state q carries prefix q over. The device holds
 * each set as an Aho-Corasick DFA, next[states][256] and hit[states] in u32 (at most 4097 states, about 4 MB), and walks
 * each emitted token's bytes through it in the kernel that emits the token, stopping at the first byte that ends a
 * string. Not available: beam search, the typical sampler of rwkv_b200_generate_streams, seeding the state from prompt
 * text, and regular-expression patterns. */
#define RWKV_B200_NO_STOP_SET 0xFFFFFFFFFFFFFFFFULL /* set_ids entry of a stream without a stop set */
#define RWKV_B200_MAX_STOP_BYTES 4096

/* The bytes of every token: token v is bytes[start[v] .. start[v + 1]), v < 50277 (start: [50277 + 1], ascending from
 * 0). Uploaded once per model; a later call replaces the table. Refused: start not starting at 0 or decreasing, NULL
 * bytes with a non-empty table, tensor parallelism, and a replacement while an unfinished batcher request has a set. */
int rwkv_b200_token_bytes_set(rwkv_b200_model *m, const unsigned long long *start, const unsigned char *bytes);
/* Build and upload the automaton of a stop set: string i is bytes[string_start[i] .. string_start[i + 1]), i <
 * n_strings; *id receives its id. Refused: no strings, string_start not starting at 0, an empty string (or offsets that
 * decrease), more than RWKV_B200_MAX_STOP_BYTES bytes in total, and tensor parallelism. */
int rwkv_b200_stop_set_add(rwkv_b200_model *m, unsigned long long n_strings, const unsigned long long *string_start,
                           const unsigned char *bytes, unsigned long long *id);
/* Free a stop set (an unknown or removed id is refused, and so is one that an unfinished request of the model's batcher
 * names). rwkv_b200_free frees every set. */
int rwkv_b200_stop_set_remove(rwkv_b200_model *m, unsigned long long id);

/* What a generate call adds for stop strings, per stream. */
typedef struct rwkv_b200_stop_request {
    const unsigned long long *set_ids;      /* [n_streams] an id of rwkv_b200_stop_set_add or RWKV_B200_NO_STOP_SET; NULL: none */
    const unsigned long long *start_states; /* [n_streams] each stream's first match state; NULL: 0 */
    unsigned long long *states_out;         /* [n_streams] the final match state (0 without a set), or NULL */
    unsigned long long *hit_out;            /* [n_streams] hit by rule 2 (0 without a set), or NULL */
    unsigned long long *tail_out;           /* [n_streams] tail by rule 2 (0 unless hit), or NULL */
} rwkv_b200_stop_request;

/* rwkv_b200_generate_streams_constrained with stop strings by the rule above (stop == NULL: exactly that call).
 * Refused before any work (every slot untouched): every refusal of generate_streams_constrained, an unknown or removed set
 * id, a start state out of range, and a set used before the model has a token-bytes table. */
int rwkv_b200_generate_streams_stop(rwkv_b200_model *m, const unsigned long long *slots,
                                    const unsigned long long *first_tokens, unsigned long long n_streams,
                                    unsigned long long max_new, const unsigned long long *budgets,
                                    const unsigned long long *stop_tokens, unsigned long long n_stop,
                                    const unsigned long long *override_tokens, const float *override_values,
                                    unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u,
                                    unsigned long long *tokens_out, unsigned long long *lengths_out, int logprob_mode,
                                    unsigned int top_n, double *logprobs_out, unsigned long long *ranks_out,
                                    unsigned long long *top_tokens_out, double *top_logprobs_out,
                                    const unsigned long long *constraint_ids, const unsigned long long *start_states,
                                    unsigned long long *states_out, const rwkv_b200_stop_request *stop);

/* rwkv_b200_generate_streams_speculative with stop strings (stop == NULL: exactly that call). Each emitted token of a
 * step is walked in order, so a string that ends inside an accepted run of drafts ends the stream at that token. The
 * tokens, lengths, first slots and hit, tail and state are bit for bit those of rwkv_b200_generate_streams_stop on the
 * first slots, by the speculative rule. Refused as well: the stop refusals of rwkv_b200_generate_streams_stop. */
int rwkv_b200_generate_streams_speculative_stop(rwkv_b200_model *m, const unsigned long long *slots,
                                                const unsigned long long *first_tokens, unsigned long long n_streams,
                                                unsigned long long max_new, const unsigned long long *budgets,
                                                const unsigned long long *stop_tokens, unsigned long long n_stop,
                                                const unsigned long long *override_tokens, const float *override_values,
                                                unsigned long long n_override, const rwkv_b200_sampler *samplers,
                                                const double *u, unsigned long long *tokens_out,
                                                unsigned long long *lengths_out, unsigned int draft, unsigned int ngram,
                                                const unsigned long long *context_start, const unsigned long long *context,
                                                unsigned long long *steps_out, const rwkv_b200_stop_request *stop);

/* rwkv_b200_generate_streams_speculative_stop with log-probabilities and token automata: every argument up to steps_out
 * is that call's, the rest are those of rwkv_b200_generate_streams_stop with the same meaning. The tokens, lengths, the
 * first slots' xy, aa, bb and dd, logprobs_out, ranks_out, the top arrays, states_out and the stop hit, tail and state
 * are bit for bit those of rwkv_b200_generate_streams_stop on the first slots with the same arguments, run on the tensor
 * cores, whatever the drafts are; steps_out keeps the draft rule above. With logprobs_out == NULL and constraint_ids ==
 * NULL the call is rwkv_b200_generate_streams_speculative_stop and enqueues the same launches.
 * Rows of a constrained stream, q its automaton state at the start of a step: row 0 has state r_0 = q. For i = 1..k, row
 * i is live when row i - 1 is live, d_i has an edge out of r_(i-1) and the target of that edge has edges; its state r_i
 * is that target. The first row that fails this is dead, and so is every row after it. A live row is masked by its own
 * state after the overrides, as rule 2 of constrained generation masks a row; a dead row is not masked. A dead row is
 * never emitted: when d_i has no edge out of r_(i-1), the pick p_(i-1) on the masked row i - 1 is an allowed token, so
 * p_(i-1) != d_i and the step stops before row i; when d_i completes the automaton, emitting it (as p_(i-1)) ends the
 * stream. So every emitted row is masked exactly as generate_streams_constrained masks it, and no pick sees a row without
 * a finite value (the override check below keeps the live rows open).
 * Each emitted token runs through generate_streams_stop's checks in its order: the budget, the stop tokens, the automaton
 * (advance; end on a state without edges; a token without an edge fails the call at the end of its 16-step group with
 * generate_streams_constrained's message and code), then the stop strings. Emitted token p_i of a step is entry [s][len +
 * i] of the log-probability arrays, scored on row i: raw mode on the model's row (a copy of the step's rows is taken
 * before the overrides and masks when the call has either), processed mode on the row the pick read, divided by the
 * stream's temperature. Rows that emit no token are not scored. Each step runs k_gen_mask with automata and one scoring
 * kernel with logprobs_out.
 * Refused before any work (every slot untouched): every refusal of rwkv_b200_generate_streams_speculative_stop
 * (including presence and frequency penalties), those of rwkv_b200_generate_streams_logprobs with logprobs_out != NULL
 * (the mode, top_n > RWKV_B200_MAX_TOP_N, missing top arrays), and those of rwkv_b200_generate_streams_constrained (an
 * unknown or removed id, a start state out of range or without edges, overrides that set every edge token of a state to
 * -inf). */
int rwkv_b200_generate_streams_speculative_constrained(
    rwkv_b200_model *m, const unsigned long long *slots, const unsigned long long *first_tokens, unsigned long long n_streams,
    unsigned long long max_new, const unsigned long long *budgets, const unsigned long long *stop_tokens,
    unsigned long long n_stop, const unsigned long long *override_tokens, const float *override_values,
    unsigned long long n_override, const rwkv_b200_sampler *samplers, const double *u, unsigned long long *tokens_out,
    unsigned long long *lengths_out, unsigned int draft, unsigned int ngram, const unsigned long long *context_start,
    const unsigned long long *context, unsigned long long *steps_out, int logprob_mode, unsigned int top_n,
    double *logprobs_out, unsigned long long *ranks_out, unsigned long long *top_tokens_out, double *top_logprobs_out,
    const unsigned long long *constraint_ids, const unsigned long long *start_states, unsigned long long *states_out,
    const rwkv_b200_stop_request *stop);

/* rwkv_b200_batcher_submit_ex (x may be NULL) with a stop set: set_id (RWKV_B200_NO_STOP_SET: exactly submit_ex) and its
 * start state. The batcher rule's step 2 becomes rwkv_b200_generate_streams_stop of the one stream with the set and start
 * state; a request whose stop string matches ends as RWKV_B200_REQ_DONE. Refused as well, with nothing queued: an unknown
 * or removed set id, a start state out of range, and a model without a token-bytes table. While the request is
 * unfinished its set cannot be removed. */
int rwkv_b200_batcher_submit_stop(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                  unsigned long long set_id, unsigned long long start_state, unsigned long long *id);
/* A request's hit, tail and current match state by the rule above (0, 0, 0 without a set); each pointer may be NULL. A
 * cancelled request's state is the state after its emitted tokens. An unknown or released id is refused. */
int rwkv_b200_batcher_read_stop(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *hit,
                                unsigned long long *tail, unsigned long long *state);

/* Speculation in the batcher: a request may opt in to prompt-lookup drafts (rwkv_b200_generate_streams_speculative's
 * draft rule), so that a step emits several of its tokens where the drafts are right. Its lookup history is context ++
 * prompt ++ the tokens it has emitted.
 *   1. Bit for bit the plain batcher. The emitted tokens, log-probabilities, ranks, top entries, final automaton state,
 *      stop-string hit, tail and state, and the final state of `slot` are bit for bit what the same request gives
 *      without spec, so the batcher rule above holds for it unchanged, whatever the other traffic, rows,
 *      prefill_tokens, max_steps and cancellations are.
 *   2. Steps. rwkv_b200_batcher_read_spec's steps is the steps_out of rwkv_b200_generate_streams_speculative_* for the
 *      one stream with slots [slot, spare_slots...], first token prompt[n_prompt - 1], lookup context context ++
 *      prompt[0 .. n_prompt - 1), draft and ngram. Row i of a step draws with u[len + i], as in that call.
 *   3. Slots. When the request finishes, and at rwkv_b200_batcher_cancel, the state of the row holding the conversation
 *      is copied to slot (xy, aa, bb and dd), so cancel keeps its promise. The spare slots are scratch: their contents
 *      after the request are unspecified. Slots that no unfinished request names are never written.
 *   4. Scheduling. Admission, prefill budgets, 16-step groups and streaming reads are unchanged. The request's decode
 *      row becomes k + 1 consecutive rows inside one tensor-core pass (rows 1..k chain from row 0's state in the pass);
 *      the one-token rows come first, and pad tokens that store no state fill a pass a speculative request would
 *      straddle. A group whose decode rows do not speculate enqueues exactly what it enqueues without this feature.
 *   5. Refusals, with nothing queued and no id used: draft outside 1..15 or ngram outside 1..8, NULL spare_slots (or
 *      NULL context with n_context > 0), a spare slot out of range, repeated, equal to slot, or named (as slot or spare)
 *      by an unfinished request, a context token >= 50277, a presence or frequency penalty (as in the one-shot call:
 *      a row's counts would have to fold in its own drafts), rows x (draft + 1) > max_gpt, and every refusal of
 *      rwkv_b200_batcher_submit_stop. A request's slot is refused as well while an unfinished request names it as a
 *      spare. */
typedef struct rwkv_b200_request_spec {
    const unsigned long long *spare_slots; /* [draft] scratch slots; contents after the request are unspecified */
    unsigned int draft;                    /* k = 1..15 drafts per step */
    unsigned int ngram;                    /* 1..8, the longest n-gram looked up */
    const unsigned long long *context;     /* [n_context] extra lookup tokens placed before the prompt; may be NULL if 0 */
    unsigned long long n_context;
} rwkv_b200_request_spec;

/* rwkv_b200_batcher_submit_stop with speculation; spec == NULL is exactly submit_stop. */
int rwkv_b200_batcher_submit_spec(rwkv_b200_batcher *b, const rwkv_b200_request *r, const rwkv_b200_request_ex *x,
                                  unsigned long long set_id, unsigned long long start_state,
                                  const rwkv_b200_request_spec *spec, unsigned long long *id);
/* The steps in which a request emitted a token (0 for a request without speculation). An unknown or released id is
 * refused. */
int rwkv_b200_batcher_read_spec(rwkv_b200_batcher *b, unsigned long long id, unsigned long long *steps);

/* State of one slot: zero it (a new conversation), copy it onto another slot (fork a conversation), or move it
 * between the device and host arrays of n_layers x n_embed doubles each (NULL arrays are skipped). */
int rwkv_b200_slot_zero(rwkv_b200_model *m, unsigned long long slot);
int rwkv_b200_slot_copy(rwkv_b200_model *m, unsigned long long src, unsigned long long dst);
int rwkv_b200_slot_upload(rwkv_b200_model *m, unsigned long long slot, const double *xy, const double *aa,
                          const double *bb, const double *pp, const double *dd);
int rwkv_b200_slot_download(rwkv_b200_model *m, unsigned long long slot, double *xy, double *aa,
                            double *bb, double *pp, double *dd);

/* State indexes: store texts as their recurrent state in HBM and rank them against query slots, as
 * examples/vectordb does on the host.
 *  - Index. An index has a contiguous layer range [layer_begin, layer_begin + n_layers) and a fixed capacity of entries.
 *    Its vectors have D = n_layers * E f64 elements: the vector of slot s is that slot's dd array over those layers as
 *    stored (layer-major), bit for bit what rwkv_b200_slot_download returns for dd there. With every layer it is the
 *    statedd that examples/vectordb reads after loadContext.
 *  - Entries. Entries get ids 0, 1, 2, ... in the order they are added; adding appends and ids are never reused.
 *    rwkv_b200_index_remove marks entries so that they are never returned again; their rows are not reclaimed, so the
 *    capacity counts every add.
 *  - Distances. For a query vector a and an entry vector b, in f64 over the D elements:
 *      l1 = (sum_j |a_j - b_j|) / E          ("diff" in examples/vectordb)
 *      l2 = sqrt((sum_j (a_j - b_j)^2) / E)  ("euclid")
 *    The summation order is fixed and depends only on D: never on the index size, the entry's row, which entries are
 *    live, the number of queries or their batch, or k. So each distance is a function of the two vectors' bits alone.
 *    (examples/vectordb divides each term by E and accumulates in float; this is the same quantity without that
 *    rounding.)
 *  - Search. For each query the live entries are ranked by the chosen metric, ascending, ties to the lower id, a NaN
 *    distance after every number. The first min(k, live) entries (found_out) are returned with both distances;
 *    positions past found_out hold RWKV_B200_NO_ENTRY and NaN. entries_out, l1_out and l2_out are [n_queries][k].
 *  - Queries are state slots, so a query text is embedded by the same forward as the documents. A search reads those
 *    slots (a slot may appear more than once) and writes no slot; n_queries has no limit beyond memory (the queries
 *    are scanned in batches).
 * Refused before any work, changing neither the index nor any slot: a NULL handle or a missing array, an unknown or
 * freed index id, a layer range outside the model or n_layers == 0, capacity == 0 or a device allocation that fails,
 * an add that would pass the capacity (nothing is added), a slot >= max_gpt, a non-finite value in upload, an entry id
 * that was never added or was removed in download and remove (nothing is removed), a metric other than the two, k == 0
 * or k > RWKV_B200_MAX_NEIGHBOURS, n_queries == 0, and tensor parallelism. rwkv_b200_free frees every index. As for the
 * other multi-stream calls, the model's batcher does not police a slot named by one of its unfinished requests. */
#define RWKV_B200_INDEX_L1 0
#define RWKV_B200_INDEX_L2 1
#define RWKV_B200_MAX_NEIGHBOURS 256
#define RWKV_B200_NO_ENTRY 0xFFFFFFFFFFFFFFFFULL /* entries_out past found_out */
/* Allocate an index of `capacity` entries over layers [layer_begin, layer_begin + n_layers); *id receives its id. */
int rwkv_b200_index_create(rwkv_b200_model *m, unsigned long long layer_begin, unsigned long long n_layers,
                           unsigned long long capacity, unsigned long long *id);
/* Free an index and its device memory. */
int rwkv_b200_index_free(rwkv_b200_model *m, unsigned long long id);
/* Append the vectors of n slots (a device-to-device copy); entries_out [n] receives their ids. */
int rwkv_b200_index_add_slots(rwkv_b200_model *m, unsigned long long id, const unsigned long long *slots,
                              unsigned long long n, unsigned long long *entries_out);
/* Append n vectors given on the host, vectors [n][D]; entries_out [n] receives their ids. */
int rwkv_b200_index_upload(rwkv_b200_model *m, unsigned long long id, const double *vectors, unsigned long long n,
                           unsigned long long *entries_out);
/* The vectors of n live entries into vectors_out [n][D]. */
int rwkv_b200_index_download(rwkv_b200_model *m, unsigned long long id, const unsigned long long *entries,
                             unsigned long long n, double *vectors_out);
/* Remove n live entries (each at most once per call). */
int rwkv_b200_index_remove(rwkv_b200_model *m, unsigned long long id, const unsigned long long *entries,
                           unsigned long long n);
/* Rank the live entries for each query slot by `metric` (RWKV_B200_INDEX_L1 or _L2) and return the first k. */
int rwkv_b200_index_search(rwkv_b200_model *m, unsigned long long id, const unsigned long long *query_slots,
                           unsigned long long n_queries, int metric, unsigned int k, unsigned long long *entries_out,
                           double *l1_out, double *l2_out, unsigned long long *found_out);

/* LoRA adapters bound to state slots: serve many low-rank fine-tunes of one base model in the same tensor-core pass.
 *  - Adapter. A rank r in 1..RWKV_B200_MAX_ADAPTER_RANK, a scale s (alpha / r), and for any non-empty subset of the
 *    seven projections a pair A [n_layers][r][in] and B [n_layers][out][r] of f32 (row-major, copied at add). The
 *    projections are indexed by RWKV_B200_AD_*: att key, value, receptance and output (E -> E), ffn key (E -> 4E), ffn
 *    value (4E -> E) and ffn receptance (E -> E). The head and the embedding are not adapted.
 *  - Value. For a token whose slot is bound, each adapted projection's value is f32(S * tot + off + delta) instead of
 *    f32(S * tot + off), with delta_m = s * sum_i B[m][i] * h_i and h_i = sum_j A[i][j] * f_j, both in f64. f is the
 *    f32 activation the projection quantises, before the r-scaling and the 22-bit rounding: the token-shift mix for att
 *    key/value/receptance and ffn key/receptance, the WKV output rw for att output, and relu(k)^2 for ffn value. The
 *    summation orders are fixed, so delta depends only on the token's own f and its adapter: results are
 *    bit-deterministic and independent of the other tokens of a pass. A token whose slot is unbound, or whose adapter
 *    lacks a projection, gets exactly the bits it gets without adapters.
 *  - Bindings belong to slots, not to states: slot_copy, slot_zero, slot_upload, slot_download and the forks inside
 *    beam search and speculation move states only.
 *  - Path. Adapters run on the tensor cores only. A multi-stream call (forward_streams, score_streams, the
 *    generate_streams calls, beam search, speculation, the batcher) that names a bound slot runs on the tensor cores
 *    whatever its token count, and is refused when the "prefill" option is 0. rwkv_b200_forward, forward_greedy,
 *    decode_timed and profile (the decode kernel) refuse when a slot they touch is bound. A call that names no bound
 *    slot enqueues exactly the launches it does without adapters.
 *  - Refused before any work, with every slot and binding untouched: a speculative stream's slots, a beam group's
 *    slots, or a batcher request's slot and spare slots that do not all share one binding; binding or unbinding a slot
 *    held by a queued or admitted batcher request; removing an adapter that is still bound; a rank outside 1..64, an
 *    adapter without matrices, a matrix with only one of A and B, a non-finite value; an unknown id; any adapter call
 *    on a tensor-parallel model. The adapters live in device memory owned by the model (20 n_embed r n_layers floats
 *    with every projection) and rwkv_b200_free frees them. */
#define RWKV_B200_MAX_ADAPTER_RANK 64
#define RWKV_B200_NO_ADAPTER 0xFFFFFFFFFFFFFFFFULL /* rwkv_b200_slot_adapter: unbind */
#define RWKV_B200_AD_ATT_KEY 0
#define RWKV_B200_AD_ATT_VALUE 1
#define RWKV_B200_AD_ATT_RECEPTANCE 2
#define RWKV_B200_AD_ATT_OUTPUT 3
#define RWKV_B200_AD_FFN_KEY 4
#define RWKV_B200_AD_FFN_VALUE 5
#define RWKV_B200_AD_FFN_RECEPTANCE 6
#define RWKV_B200_AD_MATRICES 7
typedef struct {
    unsigned int rank;                       /* 1..RWKV_B200_MAX_ADAPTER_RANK */
    double scale;                            /* s = alpha / rank, finite */
    const float *A[RWKV_B200_AD_MATRICES];   /* [n_layers][rank][in] host arrays, or NULL: not adapted */
    const float *B[RWKV_B200_AD_MATRICES];   /* [n_layers][out][rank], NULL exactly where A is */
} rwkv_b200_adapter;
/* Copy an adapter to the device; *id receives its id (ids are never reused). */
int rwkv_b200_adapter_add(rwkv_b200_model *m, const rwkv_b200_adapter *desc, unsigned long long *id);
/* Free an adapter that no slot is bound to. */
int rwkv_b200_adapter_remove(rwkv_b200_model *m, unsigned long long id);
/* Bind `slot` to adapter `id`, or unbind it with RWKV_B200_NO_ADAPTER (in stream order: later calls see it). */
int rwkv_b200_slot_adapter(rwkv_b200_model *m, unsigned long long slot, unsigned long long id);

/* Engine knobs (all optional), key/value strings: "sub_bytes" (largest bulk copy of the
 * weight stream, a multiple of 16 up to one ring stage of 8 x n_embed bytes), "budget" /
 * "qbudget" (bytes of copies in flight per SM while streaming, at least one stage / while
 * the CTAs exchange vectors), "pf_dist" (tiles the L2
 * prefetch runs ahead), "stages" (ring depth), "timeout_ms", "trace", "prefill",
 * "prefill_min", "prefill_graph", "grid" (CTAs, at most the SM count). Returns non-zero for
 * an unknown key. */
int rwkv_b200_set_option(rwkv_b200_model *m, const char *key, const char *value);

/* --- tensor-parallel wiring (tp_size > 1 only) --------------------------------- */

/* Size in bytes of this rank's peer-visible exchange block (tagged activation vectors,
 * per-CTA records, inboxes of the cross-GPU partial sums, logits, WKV state); allocated by
 * the load. */
size_t rwkv_b200_tp_buffer_bytes(const rwkv_b200_model *m);
/* Export this rank's exchange buffer as a CUDA IPC handle (64 bytes). */
int rwkv_b200_tp_export(rwkv_b200_model *m, void *ipc_handle_64);
/* Import every rank's handle (tp_size x 64 bytes, own rank's entry ignored). */
int rwkv_b200_tp_import(rwkv_b200_model *m, const void *ipc_handles);

#ifdef __cplusplus
}
#endif
#endif /* RWKV_B200_H */
