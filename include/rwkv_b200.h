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
/* Free an automaton (an unknown or removed id is refused). rwkv_b200_free frees every automaton of the model. */
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

/* State of one slot: zero it (a new conversation), copy it onto another slot (fork a conversation), or move it
 * between the device and host arrays of n_layers x n_embed doubles each (NULL arrays are skipped). */
int rwkv_b200_slot_zero(rwkv_b200_model *m, unsigned long long slot);
int rwkv_b200_slot_copy(rwkv_b200_model *m, unsigned long long src, unsigned long long dst);
int rwkv_b200_slot_upload(rwkv_b200_model *m, unsigned long long slot, const double *xy, const double *aa,
                          const double *bb, const double *pp, const double *dd);
int rwkv_b200_slot_download(rwkv_b200_model *m, unsigned long long slot, double *xy, double *aa,
                            double *bb, double *pp, double *dd);

/* Engine knobs (all optional), key/value strings: "window" / "bwindow" (bulk copies in
 * flight per SM while streaming / while the CTAs exchange vectors), "pf_dist" (tiles the L2
 * prefetch runs ahead), "stages" (ring depth), "poll_first", "timeout_ms", "max_layers",
 * "trace", "prefill", "prefill_min", "prefill_graph", "grid" (CTAs, at most the SM count),
 * "cluster" (1, 2 or 4 CTAs share a gather through distributed shared memory; measured
 * without gain, default 1). Returns non-zero for an unknown key. */
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
