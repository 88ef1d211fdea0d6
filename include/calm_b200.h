/*
 * calm_b200.h -- C ABI of libcalm_b200.so, an H100 (sm_90a) backend for calm's
 * per-token forward() path.
 *
 * The first four functions ARE the reference's CUDA backend boundary: the
 * reference driver declares exactly these prototypes (reference src/run.c:22-25)
 * and the reference backend defines them extern "C" (src/infer.cu:69, 73, 743,
 * 761).  Linking the unmodified reference run.c/tensors.c/tokenizer.c/sampler.c
 * against this library instead of infer.cu gives a working `run` binary -- see
 * INTEGRATION.md.  Everything prefixed calm_b200_ is additive.
 *
 * Error behaviour follows the reference (infer.cu:12-20, 755): there are no
 * error codes; a CUDA failure or an unsupported configuration prints one line
 * to stderr and abort()s.  There is NO CPU fallback: without a usable sm_90
 * device prepare_cuda() aborts.
 *
 * Threading: one host thread, one model per process at a time (the reference
 * keeps global statics too, infer.cu:40-48).  calm_b200_release() makes the
 * library reusable for another model in the same process.
 */
#ifndef CALM_B200_H
#define CALM_B200_H

#include <stddef.h>
#include <stdint.h>

#include "calm_model.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ *
 * Reference boundary (names, arguments and protocol of the reference) *
 * ------------------------------------------------------------------ */

/* Copy `size` bytes of a model tensor to the device and return the device
 * pointer; the caller stores it in struct Weights (run.c:552-560).
 * Replaces reference infer.cu:69-71 (upload_cuda -> cuda_devicecopy :50-55). */
void* upload_cuda(void* host, size_t size);

/* One-time set-up after struct Weights holds device pointers: validates the
 * configuration, allocates activations and the KV cache (honouring
 * state.kvbits, run.c:534-540), allocates host-visible logits and stores them
 * in state.logits, builds the per-token launch plan.
 * Replaces reference infer.cu:73-131. */
void prepare_cuda(struct Transformer* transformer);

/* Run one token at position `pos`.  Returns a host-readable float[vocab_size]
 * valid until the next call (the caller may overwrite it, sampler.c:55-66), or
 * NULL without synchronising when flags & FF_UPDATE_KV_ONLY.
 * Replaces reference infer.cu:743-759 (forward_cuda -> forward<> :651-741). */
float* forward_cuda(struct Transformer* transformer, int token, int pos, unsigned flags);

/* Print the per-stage time / bandwidth table gathered so far (only when
 * profiling was enabled with CALM_B200_PERF=1 or CUDA_INJECTION64_PATH, as in
 * the reference).  Replaces reference infer.cu:761-801. */
void perf_cuda(void);

/* ------------------------------------------------------------------ *
 * Additive entry points                                               *
 * ------------------------------------------------------------------ */

#define CALM_B200_ABI_VERSION 1
int calm_b200_abi_version(void);

/* Select the CUDA device used by upload_cuda/prepare_cuda (default: env
 * CALM_B200_DEVICE, else 0 like reference infer.cu:79).  Call before upload. */
void calm_b200_set_device(int device);

/* Free a pointer returned by upload_cuda(). */
void calm_b200_free(void* device_ptr);

/* Free everything prepare_cuda() created for this transformer (the reference
 * never frees, run.c:636) so another model can be prepared in this process. */
void calm_b200_release(struct Transformer* transformer);

/* Tensor parallelism for models that do not fit (or should not sit on) one GPU -- the 70B shape of
 * BASELINE.json configs[4]; the reference has no counterpart (single device, infer.cu:79).  One process per GPU.
 * Rank 0 obtains a 128-byte NCCL id with calm_b200_tp_unique_id() and hands it to the other ranks by any means
 * (file, pipe, torch.distributed broadcast); every rank then calls calm_b200_tp_init(rank, world, id) BEFORE
 * prepare_cuda() and afterwards drives the library exactly as a single-GPU host does: upload the FULL tensors,
 * prepare, forward the same (token, pos) on every rank.  prepare_cuda() keeps this rank's 1/world of the query /
 * kv heads and of the FFN rows (row ranges of wq/wk/wv/w1/w3 in place, packed column ranges of wo/w2); each
 * forward sums the two partial projections per layer over NVLink (inside the CUDA graph) and every rank returns the full, identical logits.  Requires world | n_heads, n_kv_heads and 32*world |
 * hidden_dim; dense models.  libnccl.so.2 is bound with dlopen on first use.
 * calm_b200_tp_mode(): 0 = not tensor-parallel, 2 = the wo / w2 kernels sum their partials themselves through
 * CUDA-IPC-mapped peer memory (one-shot push all-reduce inside k_matres; default), 1 = ncclAllReduce between
 * kernels (peer mapping unavailable, or env CALM_B200_TP_FUSED=0). */
void calm_b200_tp_unique_id(void* out128);
void calm_b200_tp_init(int rank, int world, const void* id128);
int calm_b200_tp_world(void);
int calm_b200_tp_mode(void);


/* The prompt as ONE batched pass (the reference feeds prompt tokens one at a time through forward(.., FF_UPDATE_KV_ONLY),
 * run.c:206-209, README.md:80): n tokens at positions pos0 .. pos0+n-1 go through every layer together; the projections
 * are tensor-core GEMMs (wgmma.mma_async, accumulators in registers, weights dequantised on the fly, activations as an f16 hi + lo
 * pair so inputs keep 22 bits), attention is causal over the block and the cache.  Afterwards the KV cache holds what n
 * serial KV-only calls would have left (within the stated tolerance); no logits, no synchronisation with the host beyond
 * reading `tokens`.  Returns 1 when the batched pass ran, 0 when the model shape is not served by it (MoE, tensor
 * parallelism, dims not multiples of 128, head_dim other than 64 / 128, a block that would roll the cache over) and the
 * tokens were fed one by one instead -- same result either way.  A host integrates it by replacing the prompt loop:
 * forward_prefill_cuda(t, prompt, n - 1, 0); logits = forward_cuda(t, prompt[n - 1], n - 1, 0);  (INTEGRATION.md). */
int forward_prefill_cuda(struct Transformer* transformer, const int* tokens, int n, int pos0);

/* Score a token sequence: what the reference's study() computes one forward() at a time (run.c:291-308).
 * tokens[0 .. n-2] go through the batched prompt pass at positions pos0 .. pos0+n-2, and
 *   logprobs[i] = ln softmax(logits after tokens[i] at pos0+i)[tokens[i+1]],   i in [0, n-1).
 * The classifier runs over all n-1 rows on the tensor cores with the log-softmax fused into its epilogue, so the
 * [n-1][vocab] logits are never written.  Afterwards the KV cache holds exactly what forward_prefill_cuda(t, tokens, n-1,
 * pos0) leaves; the last token is only a target.  Every token, the target included, must be in the vocabulary.
 * Returns 1 when the tensor-core pass ran.  Returns 0 when the positions went one by one through the decode path (the
 * shapes forward_prefill_cuda does not serve, or pos0+n-1 > seq_len); both give the same values within the stated
 * tolerance (DESIGN.md s.6).  n < 2: nothing to score, the cache is untouched, returns 1.  Under tensor parallelism every
 * rank calls it with the same arguments, as with forward_cuda.  Perplexity over a text in chunks of m positions:
 * chunk c is calm_b200_score(t, tokens + c, m + 1, 0, out + c)  (INTEGRATION.md). */
int calm_b200_score(struct Transformer* transformer, const int* tokens, int n, int pos0, float* logprobs);

/* Score nseq independent sequences, each from position 0, packed into shared prompt-pass blocks.
 * Sequence i is tokens[off[i] .. off[i] + len[i]) and writes
 *   logprobs[off[i] + j] = ln softmax(logits after tokens[off[i] + j] at position j)[tokens[off[i] + j + 1]],  j in [0, len[i] - 1)
 * -- exactly what calm_b200_score(t, tokens + off[i], len[i], 0, logprobs + off[i]) writes.  Sequences may share their
 * boundary token (study()'s chunks: off = c * steps, len = steps + 1), but their output ranges must not overlap.
 * Slots of logprobs no sequence writes are left untouched.  Returns 1 when every sequence went through the tensor-core
 * pass, 0 when any went through the decode path.  The KV cache afterwards holds nothing a host can continue from.
 * Every token of tokens[0 .. n) must be in the vocabulary, and 0 <= off[i], off[i] + len[i] <= n; a sequence with
 * len[i] < 2 contributes nothing, nseq == 0 returns 1.  Many short sequences share one block of up to 2048 rows (DESIGN.md
 * s.6), so they fill the GPU where one call per sequence would leave most of it idle.  It equals calm_b200_score_context
 * with every ctx_len[i] == 0. */
int calm_b200_score_batch(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len,
                          int nseq, float* logprobs);

/* Score nseq sequences that each continue a context, packed into shared prompt-pass blocks with each context computed
 * once per block.  Sequence i is tokens[off[i] .. off[i] + len[i]); it continues the context
 * tokens[ctx_off[i] .. ctx_off[i] + ctx_len[i]) and writes
 *   logprobs[off[i] + j] = ln softmax(logits after tokens[off[i] + j] at position ctx_len[i] + j)[tokens[off[i] + j + 1]],
 *   j in [0, len[i] - 1)
 * -- exactly what calm_b200_score(t, ctx_i ++ seq_i, ctx_len[i] + len[i], 0, tmp) writes at tmp[ctx_len[i] + j].  The
 * first token of a sequence is an input only: for ln p(continuation | context), pass context[:-1] as the context and
 * context[-1:] ++ continuation as the sequence (INTEGRATION.md).  ctx_len[i] == 0 means no context, as in
 * calm_b200_score_batch.  Contexts are read only and may overlap anything; output ranges must not overlap, and slots of
 * logprobs no sequence writes are left untouched.  Sequences with the same (ctx_off[i], ctx_len[i]) share one copy of the
 * context's rows within a block; equal contents at different offsets are scored correctly but computed once per sequence.
 * Returns 1 when every sequence went through the tensor-core pass, 0 when any went through the decode path.  The KV cache
 * afterwards holds nothing a host can continue from.  Every token of tokens[0 .. n) must be in the vocabulary, and every
 * context and sequence must lie inside them; a sequence with len[i] < 2 contributes nothing (its context is not placed),
 * nseq == 0 returns 1.  A context with its sequence that does not fit one block of up to 2048 rows is scored alone by
 * calm_b200_score (DESIGN.md s.6). */
int calm_b200_score_context(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len, const int* off, const int* len, int nseq, float* logprobs);

/* The three scoring calls above, each also returning the greedy token at every scored position.  Each takes its
 * sibling's arguments plus `greedy` (not NULL), returns what the sibling returns and writes `logprobs` bit for bit as the
 * sibling does.  greedy[i] is written at exactly the slots where logprobs[i] is, other slots are left untouched, and
 *   greedy[i] = argmax over the vocabulary of the logits at the position logprobs[i] scores,
 * ties going to the lowest index (the reference's sample_argmax, sampler.c:34-42, and calm_b200_forward_argmax).  On the
 * tensor-core pass the logits are the fp32 classifier outputs the log-softmax is computed from, so the greedy token's
 * logit is the maximum that log-softmax subtracts; on the decode path they are the logits forward_cuda returns.
 * Uses: is_greedy of a loglikelihood request (every continuation token equals its position's greedy token), and
 * verifying draft tokens on a live cache with calm_b200_score_greedy at pos0 > 0 (INTEGRATION.md). */
int calm_b200_score_greedy(struct Transformer* transformer, const int* tokens, int n, int pos0, float* logprobs, int* greedy);
int calm_b200_score_batch_greedy(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq,
                                 float* logprobs, int* greedy);
int calm_b200_score_context_greedy(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                   const int* off, const int* len, int nseq, float* logprobs, int* greedy);

/* The three scoring calls above, each also returning the k most likely tokens at every scored position with their
 * log-probabilities (an OpenAI-style completion's logprobs=k; INTEGRATION.md).  Each takes its sibling's arguments plus
 * k, top_ids and top_logprobs, returns what the sibling returns and writes `logprobs` bit for bit as the sibling does.
 * For every slot i where logprobs[i] is written it writes top_ids[i*k + r] and top_logprobs[i*k + r], r in [0, k); other
 * slots are left untouched.  top_ids[i*k ..] are the k vocabulary indices with the largest logits at that position, by
 * logit descending, equal logits lowest index first (the reference's sample_argmax rule, sampler.c:34-42), so
 * top_ids[i*k] is what the _greedy sibling writes to greedy[i].  top_logprobs[i*k + r] = logit - M - ln S with the
 * maximum M and sum S that give logprobs[i], evaluated the same way: where top_ids[i*k + r] is the target,
 * top_logprobs[i*k + r] == logprobs[i] bit for bit, on the tensor-core pass and on the decode path alike.  The logits
 * are those the greedy siblings describe.  1 <= k <= min(CALM_B200_TOPK_MAX, vocab_size) and both arrays not NULL, or
 * the call aborts before any device work.  The first top-k call allocates the tile lists the merge reads:
 * 2048 x ceil(vocab_size / 128) x CALM_B200_TOPK_MAX x 8 bytes (328 MB at a 128256-token vocabulary; DESIGN.md s.6). */
#define CALM_B200_TOPK_MAX 20 /* the largest k a call accepts (the OpenAI API's top_logprobs limit) */
int calm_b200_score_topk(struct Transformer* transformer, const int* tokens, int n, int pos0, int k, float* logprobs, int* top_ids,
                         float* top_logprobs);
int calm_b200_score_batch_topk(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq, int k,
                               float* logprobs, int* top_ids, float* top_logprobs);
int calm_b200_score_context_topk(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                 const int* off, const int* len, int nseq, int k, float* logprobs, int* top_ids, float* top_logprobs);

/* forward + device-side greedy sample.  Returns argmax(logits) with the
 * reference's tie rule (lowest index, sampler.c:34-42).  The logits are still
 * written to state.logits. */
int calm_b200_forward_argmax(struct Transformer* transformer, int token, int pos);

/* Device-resident greedy decode: feeds token0 at pos0, then n_tokens-1 times the
 * argmax of the previous step, without a host round trip between tokens.
 * out_tokens[i] receives the token sampled after step i (n_tokens values).
 * This is what bench.py times as the in-HBM throughput. */
void calm_b200_decode_greedy(struct Transformer* transformer, int token0, int pos0, int n_tokens, int* out_tokens);

/* Verify draft tokens in one pass over the weights.  Feeds tokens[0 .. n) at positions pos0 .. pos0 + n - 1, writing
 * their cache slots, and sets greedy[i] to the argmax of the logits after tokens[i], ties going to the lowest index (the
 * rule of calm_b200_forward_argmax).  Slots past the prefix a caller accepts are scratch that later calls overwrite
 * (INTEGRATION.md).  Returns 1 when the short-block path ran (DESIGN.md s.6: the prompt pass's per-row kernels with a
 * GEMM that streams the weights over every SM).  Shapes the prompt pass does not serve (MoE, tensor parallelism, widths
 * not multiples of 128, head_dim other than 64 / 128) and blocks past seq_len take n calm_b200_forward_argmax calls
 * instead, with exactly their results, and return 0.  1 <= n <= CALM_B200_VERIFY_MAX and both arrays not NULL, or the
 * call aborts before any device work. */
#define CALM_B200_VERIFY_MAX 16
int calm_b200_verify_greedy(struct Transformer* transformer, const int* tokens, int n, int pos0, int* greedy);

/* Greedy decoding with prompt-lookup drafts.  tokens[0 .. n) is the sequence so far: the cache holds positions
 * [0, n - 1) and tokens[n - 1] is fed at n - 1, as calm_b200_decode_greedy(t, tokens[n - 1], n - 1, n_tokens, out)
 * feeds it.  Writes n_tokens greedy tokens to out_tokens and returns the model steps it ran (verify calls plus single
 * decode steps).  Each step looks up the last 3, else 2, else 1 tokens of tokens ++ emitted in the corpus: source[0 ..
 * n_source), or with source == NULL tokens ++ emitted itself (prompt lookup).  The rightmost occurrence that some token
 * follows wins, and up to max_draft (1 .. CALM_B200_VERIFY_MAX - 1) of the tokens after it are the drafts, fewer at the
 * corpus end, at seq_len and where fewer tokens are still wanted.  With drafts, one calm_b200_verify_greedy of the current
 * token and the drafts accepts the longest prefix that matches and emits the greedy token after it; without, one decode
 * step runs (calm_b200_forward_argmax), so a run that never matches emits calm_b200_decode_greedy's tokens.  Shapes the
 * verify call does not serve take decode steps only.  Afterwards cache slots [0, n - 1 + n_tokens) are valid, as after
 * calm_b200_decode_greedy; slots after them are scratch. */
int calm_b200_decode_lookup(struct Transformer* transformer, const int* tokens, int n, int n_tokens, const int* source, int n_source,
                            int max_draft, int* out_tokens);

/* Verify draft tokens by sampling (speculative sampling for deterministic drafts, DESIGN.md s.6).  Feeds tokens[0 .. n)
 * at pos0 .. pos0 + n - 1 and writes their cache slots, as calm_b200_verify_greedy does, and sets sampled[i] to the
 * reference's sample() (sampler.c:80-90) of the logits after tokens[i], drawn with the (i + 1)-th coin of *rng_state's
 * xorshift* generator (the coin calm_b200_decode_sample would use there).  With a accepted drafts -- the longest prefix
 * with sampled[i] == tokens[i + 1], i < n - 1 -- the caller emits sampled[0 .. a], and *rng_state is left advanced by
 * a + 1 draws, as a + 1 calls of calm_b200_forward_sample leave it.  Accepting a draft exactly when the target's own
 * sample equals it gives the target's distribution.  Returns 1 on the short-block path.  temperature == 0 or minp >= 1
 * is calm_b200_verify_greedy and leaves the generator alone, as sample() does.  The shapes and blocks verify_greedy does
 * not serve run n calm_b200_forward_sample calls on a copy of the state instead, with exactly their tokens, and return 0.
 * 1 <= n <= CALM_B200_VERIFY_MAX and no array NULL, or the call aborts before any device work.  The first call allocates
 * the logit rows and per-row sampler lists: 16 x vocab_size x 4 bytes and 16 x ceil(vocab_size / 1024) x 8 KB (8.2 MB
 * and 16.5 MB at a 128256-token vocabulary). */
int calm_b200_verify_sample(struct Transformer* transformer, const int* tokens, int n, int pos0, float temperature, float minp,
                            unsigned long long* rng_state, int* sampled);

/* calm_b200_decode_lookup's loop, draft rule, caps and end-of-cache handling with sampled tokens: a step with drafts is
 * one calm_b200_verify_sample, a step without is one calm_b200_forward_sample.  Writes n_tokens tokens, returns the model
 * steps, and leaves *rng_state where calm_b200_decode_sample of the same tokens leaves it: a run that never finds a
 * draft is calm_b200_decode_sample, bit for bit.  temperature == 0 or minp >= 1 is calm_b200_decode_lookup, and
 * rng_state must not be NULL. */
int calm_b200_decode_lookup_sample(struct Transformer* transformer, const int* tokens, int n, int n_tokens, const int* source,
                                   int n_source, int max_draft, float temperature, float minp, unsigned long long* rng_state,
                                   int* out_tokens);

/* Sample nseq continuations of one prompt together: every step is one pass over the weights for all of them, and the
 * prompt's cache entries are read once per step for all of them (DESIGN.md s.6).  The cache holds the prompt at
 * positions [0, pos0).  Each sequence b feeds token0 at pos0 and then its own sample n_tokens - 1 times, exactly as
 * calm_b200_decode_sample(t, token0, pos0, n_tokens, temperature, minp, &rng_states[b], ...) would, and
 * out_tokens[b * n_tokens + i] is its sample after step i; rng_states[b] is left advanced by n_tokens draws.
 * temperature == 0 or minp >= 1 makes every sequence the greedy stream and leaves the states alone, as sample() does.
 * Returns 1 on the new path.  Step j writes sequence b's entries to cache slot pos0 + j * nseq + b, so the call needs
 * pos0 + nseq * n_tokens <= seq_len; slots [0, pos0) stay bit for bit as they were and slots from pos0 on are scratch
 * (to continue one sequence, feed its tokens again from pos0: INTEGRATION.md).  Shapes the prompt pass does not serve
 * (as for calm_b200_verify_greedy) and calls past seq_len run calm_b200_decode_sample once per sequence, b = 0, 1, ..,
 * each from token0 at pos0, with exactly their tokens and states, and return 0.  1 <= nseq <= CALM_B200_SAMPLE_N_MAX,
 * n_tokens >= 0 and, for n_tokens > 0, neither array NULL, or the call aborts before any device work; n_tokens == 0
 * does nothing and returns 1.  The first call allocates what calm_b200_verify_sample allocates, 8 bytes per cache
 * position, and the attention's partials: 16 x n_heads x ceil((pos0 + n_tokens) / 128) x (head_dim + 2) x 4 bytes,
 * regrown when a later call needs more (8.5 MB for Llama-3-8B at 4096 positions). */
#define CALM_B200_SAMPLE_N_MAX 16 /* == VF_TOK, static_assert in engine.cu */
int calm_b200_decode_sample_n(struct Transformer* transformer, int token0, int pos0, int n_tokens, int nseq, float temperature, float minp,
                              unsigned long long* rng_states, int* out_tokens);

/* Sample nseq sequences that each continue their own prompt together: the prompts go through the prompt pass packed into
 * shared blocks, then every step is one pass over the weights for all of them (DESIGN.md s.6).  Prompt b is
 * tokens[off[b] .. off[b] + len[b]), len[b] >= 1, as in calm_b200_score_batch.  Sequence b is, by definition, what
 *   forward_prefill_cuda(t, prompt_b, len[b] - 1, 0);
 *   calm_b200_decode_sample(t, prompt_b[len[b] - 1], len[b] - 1, n_tokens, temperature, minp, &rng_states[b], ...);
 * give on a fresh cache, bit for bit: out_tokens[b * n_tokens + i] is its sample after step i, and rng_states[b] is left
 * advanced by n_tokens draws.  temperature == 0 or minp >= 1 makes every sequence its greedy stream and leaves the states
 * alone.  Returns 1 on the new path.  Prompt b's L_b = len[b] - 1 entries are placed at slots s_b .., each prompt taking
 * L_b rounded up to a multiple of 8 slots, packed in input order from slot 0 up to G = sum of those; step j writes
 * sequence b's entries to slot G + j * nseq + b, so the call needs G + nseq * n_tokens <= seq_len.  Shapes the prompt
 * pass does not serve (as for calm_b200_verify_greedy) and calls past seq_len run the pair above for b = 0, 1, .., with
 * exactly its tokens and states, and return 0.  The KV cache afterwards holds nothing a host can continue from (to
 * continue one sequence, feed its prompt and tokens again: INTEGRATION.md).  1 <= nseq <= CALM_B200_SAMPLE_N_MAX and
 * n_tokens >= 0, or the call aborts before any device work; n_tokens == 0 reads nothing else and returns 1.  Otherwise
 * no array may be NULL, every prompt must have len[b] >= 1 and lie inside tokens[0 .. n), and every token of
 * tokens[0 .. n) must be in the vocabulary, or the call aborts before any device work.  The first call allocates what
 * calm_b200_decode_sample_n allocates, with the attention's partials for ceil((max L_b + n_tokens) / 128) chunks, and
 * the prompt pass's buffers for min(G, 2048) rows. */
int calm_b200_decode_sample_batch(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq,
                                  int n_tokens, float temperature, float minp, unsigned long long* rng_states, int* out_tokens);

/* Beam search over one prompt: num_beams = B beams advance together, every step one pass over the weights for all of
 * them, the prompt's cache entries read once per step for all of them and each beam's generated entries read through its
 * ancestry, so no cache entry is ever copied (DESIGN.md s.6).  Hugging Face's generate(num_beams, length_penalty,
 * early_stopping, num_return_sequences) with eos_token_id = stop, at temperature 1 and without logit processors
 * (INTEGRATION.md).  The cache holds the prompt at slots [0, pos0); token0 is fed at pos0.
 *   Rows and slots.  Step j runs every live beam at RoPE position pos0 + j, row b writing cache slot pos0 + j * B + b;
 *     step 0 runs one row, fed token0, and every later step B rows.  The call needs pos0 + B * max_new <= seq_len; slots
 *     [0, pos0) are never written and slots from pos0 on are scratch afterwards.
 *   Candidates.  K = max(2, 1 + n_stop) * B (Hugging Face's, which leaves B candidates that are not stop tokens).  Each
 *     row takes its K best tokens, logit descending and the lowest id on ties, each with lp = l - M - ln S of the step's
 *     fp32 logits (calm_b200_decode_sample_queue_logprobs' log-probability, at temperature 1).  Beam b has a running fp32
 *     sum S_b, 0 at the start, and a candidate's score is c = S_b + lp, one fp32 add.  All rows' candidates are ordered
 *     by c descending, then beam ascending, then rank ascending, and the first K are walked in that order, q being the
 *     place in the walk.
 *   Walk.  A candidate whose token is in stop becomes a finished hypothesis when q < B and is skipped otherwise: the
 *     parent's tokens plus the stop token, raw sum c, score c / norm[max(1, j)] (the tokens before the stop).  Any other
 *     candidate becomes the next live beam, in walk order, until B are taken.  norm[L] = (float)pow((double)L,
 *     (double)length_penalty), computed on the host; every division is one IEEE fp32 division.
 *   Pool.  At most B finished hypotheses.  A new one enters while the pool holds fewer than B, or when its score is
 *     strictly greater than the worst; when the pool exceeds B the worst leaves, the earliest added among equal scores.
 *   Done.  After each step's walk, when the pool holds B: early_stopping 1 is done; early_stopping 0 is done when
 *     worst >= S_best / norm[j + 1], S_best the first live beam's sum (Hugging Face's default heuristic).  After max_new
 *     steps, if the call is not done, each live beam enters the pool, in beam order, with score S_b / norm[max_new].
 *   Outputs.  The pool sorted by score descending, the earliest added first among equal scores; for r < num_return,
 *     out_tokens[r * max_new ..] gets hypothesis r's tokens (stop token included), out_len[r] its length, out_scores[r]
 *     its score and, unless out_logprobs is NULL, out_logprobs[r * max_new ..] each token's lp; summed left to right in
 *     fp32 from 0 they give its raw sum bit for bit.  *steps gets the number of steps run.  Slots past out_len[r] and
 *     rows from num_return on are left untouched.
 * Returns 1 on this path.  MoE and tensor-parallel models, shapes the prompt pass does not serve (as for
 * calm_b200_verify_greedy) and calls past seq_len return 0, set *steps = 0 and do nothing else: a per-token fallback
 * would need a cache per beam (DESIGN.md s.8).  The call aborts before any device work when num_beams is outside
 * [1, CALM_B200_BEAM_MAX], K > CALM_B200_TOPK_MAX, num_return is outside [1, num_beams], max_new or n_stop is negative,
 * a stop id or token0 is outside the vocabulary, pos0 is negative, length_penalty is not finite, early_stopping is not
 * 0 or 1, or stop (with n_stop > 0), out_tokens, out_len, out_scores or steps is NULL.  max_new == 0 does nothing else
 * and returns 1.  The first call allocates what calm_b200_decode_sample_n allocates for ceil((pos0 + max_new) / 128)
 * chunks, the queue's top-k lists (calm_b200_decode_sample_queue_logprobs) and, regrown when a later call needs more,
 * 4 x B x max_new x (2 + 3 + 2 K) bytes of ancestry, backpointers and candidate lists. */
#define CALM_B200_BEAM_MAX 10
int calm_b200_decode_beam(struct Transformer* transformer, int token0, int pos0, int max_new, int num_beams, const int* stop, int n_stop,
                          float length_penalty, int early_stopping, int num_return, int* out_tokens, int* out_len, float* out_logprobs,
                          float* out_scores, int* steps);

/* Generate for a queue of nreq requests, at most max_rows (1 .. CALM_B200_SAMPLE_N_MAX) in flight, each with its own
 * length, sampling settings and generator, and admit new requests as rows finish (DESIGN.md s.6).  Request i's prompt is
 * tokens[off[i] .. off[i] + len[i]), len[i] >= 1, as in calm_b200_decode_sample_batch; it generates at most
 * max_new[i] >= 0 tokens at temperature[i] / minp[i] from rng_states[i].  stop[0 .. n_stop) is one list of stop ids shared
 * by all requests (NULL when n_stop == 0).  Request i writes its tokens to out_tokens[O_i ..], O_i = max_new[0] + .. +
 * max_new[i - 1], and its count to out_len[i]: the smaller of max_new[i] and 1 + the index of its first token in stop
 * (the stop token is emitted); out_tokens past out_len[i] are left untouched.  steps (may be NULL) receives the number of
 * steps the call ran, each one pass over the weights for the rows in flight.
 * Returns 1 on the new path: request i's tokens and its final rng_states[i] are then bit for bit those of
 * calm_b200_decode_sample_batch over its prompt alone (nseq = 1) with n_tokens = out_len[i], whatever the other requests,
 * max_rows, the admission order, the slots it was given or seq_len.  temperature[i] == 0 or minp[i] >= 1 makes request i
 * its greedy stream and leaves its state alone; max_new[i] == 0 gives out_len[i] = 0, and the request is never admitted.
 * Schedule.  Before every step the requests at the head of the queue are admitted in input order (no overtaking), while
 * a row is free and the placement below of the requests admitted so far before this step (a round), with the next one
 * added, fits.  A round's prompts go through the packed prompt pass together.  A step runs every request in flight once;
 * its rows are in admission order, and a request retires after the step that gave its max_new-th or its stop token.
 * Placement.  The cache slots [0, seq_len) are free at the start.  A round's placement, computed from the slots free
 * before the round, takes first one extent of the sum of ceil8(len[i] - 1) over its requests, at the lowest free start
 * that is a multiple of 8, holding their prompts packed in input order (request i's L_i = len[i] - 1 entries at slots
 * s_i ..); then, in input order, one extent of max_new[i] slots per request at the lowest free start (t_i ..).  Step j of
 * request i feeds its last token at RoPE position L_i + j and writes slot t_i + j.  A retiring request frees its
 * ceil8(L_i) prompt slots and its max_new[i] generated slots, and adjacent free slots merge.
 * Shapes the prompt pass does not serve (as for calm_b200_verify_greedy), and calls with a request whose
 * ceil8(len[i] - 1) + max_new[i] > seq_len, return 0: each request then runs in input order as forward_prefill_cuda of
 * its first len[i] - 1 tokens and calm_b200_forward_sample from its last token, token by token, until a stop token or
 * max_new[i] (decode_sample's stream, cut), and *steps = 0.  The call aborts before any device work when an array it
 * needs is NULL, max_rows is outside its range, nreq, n or n_stop is negative, a max_new is negative, a prompt is empty
 * or outside tokens[0 .. n), or a token of tokens[0 .. n) or a stop id is outside the vocabulary.  The KV cache
 * afterwards holds nothing a host can continue from.  The first call allocates what calm_b200_decode_sample_batch
 * allocates, and room for max_new[0] + .. + max_new[nreq - 1] tokens and nreq states, regrown by a larger call. */
int calm_b200_decode_sample_queue(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nreq,
                                  const int* max_new, const float* temperature, const float* minp, const int* stop, int n_stop,
                                  int max_rows, unsigned long long* rng_states, int* out_tokens, int* out_len, int* steps);

/* calm_b200_decode_sample_queue for requests whose prompts share prefixes: each shared context is computed once by the
 * prompt pass while its requests are in flight, and every step reads a context's whole chunks once for all of them
 * (DESIGN.md s.6).  Request i's prompt is the context tokens[ctx_off[i] .. ctx_off[i] + ctx_len[i]) followed by its own
 * tokens[off[i] .. off[i] + len[i]), len[i] >= 1; ctx_len[i] == 0 means no context.  Requests share a context exactly
 * when they name the same (ctx_off, ctx_len), as in calm_b200_score_context; equal contents at different offsets are
 * correct but computed separately.  Every other argument and output is calm_b200_decode_sample_queue's; prompt_rows
 * (may be NULL) receives the number of rows the call's prompt passes computed.
 * Returns 1 on the new path: request i's tokens and final rng_states[i] are then bit for bit those of
 * calm_b200_decode_sample_batch over its concatenated prompt alone (nseq = 1) with n_tokens = out_len[i], whatever the
 * other requests, which of them share its context, max_rows, the slots it was given or seq_len.
 * Schedule and placement.  calm_b200_decode_sample_queue's, with contexts: a context is resident from the round that
 * places it until it is released.  Admission: before every step the requests at the head of the queue are admitted in
 * input order while a row is free and the round's placement, computed from the slots free before the round, fits.  A
 * round's placement takes first one extent at the lowest free start that is a multiple of 8 holding, request by request
 * in input order, the request's context (ceil8(ctx_len[i]) slots, at RoPE positions 0 ..) unless that context is
 * resident or placed by an earlier request of the round, then its own prompt (ceil8(len[i] - 1) slots, at positions
 * ctx_len[i] ..); then, in input order, one extent of max_new[i] slots per request at the lowest free start.  A request
 * whose context is resident reads it there.  The extent goes through the packed prompt pass.  Release: after admission,
 * a resident context that no request in flight names (those admitted by the round included) frees its slots; if then
 * nothing is in flight, admission runs again on the empty cache.  Retire: a request retires after the step that gave its
 * max_new-th or its stop token and frees its own ceil8(len[i] - 1) prompt slots and its max_new[i] generated slots.
 * Step j of request i feeds its last token at RoPE position ctx_len[i] + len[i] - 1 + j and writes slot t_i + j.  With
 * every ctx_len 0 this is calm_b200_decode_sample_queue's rule exactly, and the call is that call.
 * Shapes the prompt pass does not serve, and calls with a request whose ceil8(ctx_len[i]) + ceil8(len[i] - 1) +
 * max_new[i] > seq_len, return 0: calm_b200_decode_sample_queue's fallback over each request's concatenated prompt,
 * with *steps = 0 and *prompt_rows = 0.  The call aborts before any device work where calm_b200_decode_sample_queue
 * does, and when a context lies outside tokens[0 .. n) or ctx_off / ctx_len is NULL. */
int calm_b200_decode_sample_queue_context(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                          const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                          const float* minp, const int* stop, int n_stop, int max_rows, unsigned long long* rng_states,
                                          int* out_tokens, int* out_len, int* steps, int* prompt_rows);

/* calm_b200_decode_sample_queue_context that also returns every generated token's log-probability and the k most likely
 * tokens at its step, with theirs (an OpenAI-style response's logprobs / top_logprobs, best_of, RL rollouts;
 * INTEGRATION.md).  ctx_off and ctx_len may both be NULL: no request has a context.
 * Unchanged outputs.  out_tokens, out_len, rng_states, steps, prompt_rows and the return value are bit for bit those of
 * calm_b200_decode_sample_queue_context with the same arguments (with no contexts, those of
 * calm_b200_decode_sample_queue), on the new path and on the fallback alike.
 * What the numbers are.  The model's own distribution, as in the scoring calls: the log-softmax of the step's fp32
 * logits at temperature 1 and without the min-p cut, whatever the request's temperature / minp.  A sampled token can
 * therefore have any log-probability and can lie outside the top k.
 * Where they go.  Request i's token of step j is out_tokens[O_i + j]; the same slot gets logprobs[O_i + j] = l[tok] - M
 * - ln S, with M and S the maximum and sum the scoring calls' merge gives that step's logits l (the expression of
 * calm_b200_score's logprobs), and for k >= 1 top_ids[(O_i + j)*k + r] and top_logprobs[(O_i + j)*k + r], r in [0, k),
 * by the _topk scoring calls' rule: logit descending, equal logits lowest index first, log-probabilities by the same
 * expression with the same M and S.  Where top_ids holds the emitted token, top_logprobs == logprobs bit for bit; a
 * greedy request's top_ids[.. + 0] is its token.  Slots past out_len[i] are left untouched.
 * Independence.  On the new path request i's logprobs / top_* do not depend on the other requests, max_rows, the slots
 * or seq_len, as its tokens do not: they come from the same logits.
 * Arguments.  0 <= k <= min(CALM_B200_TOPK_MAX, vocab_size); logprobs not NULL when any max_new[i] > 0, and top_ids /
 * top_logprobs not NULL when also k > 0 (either may be NULL when k == 0).  They hold max_new[0] + .. + max_new[nreq - 1]
 * and k times that entries.  Otherwise, and wherever calm_b200_decode_sample_queue_context aborts, the call aborts
 * before any device work.
 * Fallback (return 0; MoE, tensor parallelism, other shapes the prompt pass does not serve, requests that do not fit
 * seq_len): after each token of the queue's fallback, its device logits (those calm_b200_read_device_logits reads) go
 * through calm_b200_score's decode-path log-softmax in double and top-k, written as float.
 * The first call allocates what calm_b200_decode_sample_queue_context allocates, the step's tile lists for 16 rows:
 * 16 x ceil(vocab_size / 128) x CALM_B200_TOPK_MAX x 8 bytes (2.6 MB at a 128256-token vocabulary; not the scoring
 * calls' 2048-row lists), and room for the outputs, 4 + 8 k bytes per token of max_new[0] + .. + max_new[nreq - 1],
 * regrown by a larger call. */
int calm_b200_decode_sample_queue_logprobs(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                           const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                           const float* minp, const int* stop, int n_stop, int max_rows, unsigned long long* rng_states,
                                           int* out_tokens, int* out_len, int* steps, int* prompt_rows, int k, float* logprobs, int* top_ids,
                                           float* top_logprobs);

/* calm_b200_decode_sample_queue_logprobs where each request's logits first go through its own logit bias and presence,
 * frequency and repetition penalties (OpenAI's logit_bias / presence_penalty / frequency_penalty, the repetition_penalty
 * of Hugging Face generate; INTEGRATION.md).
 * Settings.  Request i has presence p = presence[i], frequency f = frequency[i], repetition r = repetition[i] (each
 * array may be NULL: 0, 0 and 1 for every request) and the bias list bias_ids / bias_val[bias_off[i] .. + bias_len[i]);
 * b(v) is the list's value for id v, 0 off the list.  bias_off and bias_len may both be NULL when n_bias == 0.
 * Processing.  At request i's step j, with l(v) the step's fp32 logit as calm_b200_decode_sample_queue_logprobs
 * computes it, c(v) how many of the request's tokens of steps 0 .. j-1 equal v (generated tokens only) and seen(v)
 * true when v is among the ctx_len[i] + len[i] tokens of ctx ++ prompt (the last one included) or c(v) > 0:
 *     l1 = (seen(v) && r != 1) ? (l > 0 ? l / r : l * r) : l
 *     a  = (b(v) - f * (float)c(v)) - (c(v) > 0 ? p : 0)
 *     l2 = (a == 0) ? l1 : l1 + a
 * each operation one IEEE fp32 operation rounded to nearest, with no contraction (numpy float32 gives the same bits).
 * l2 replaces l for everything the step does: a greedy request's token is the first maximum of l2, a sampled one's the
 * reference's sample() at its temperature / minp over l2, and logprobs / top_ids / top_logprobs are those of l2
 * (processed log-probabilities) by the _logprobs call's rules.
 * Neutral requests.  A request with p == 0, f == 0, r == 1 and an empty list is neutral: its outputs are the bits
 * calm_b200_decode_sample_queue_logprobs gives it, whatever shares its steps.
 * Arguments.  logprobs == NULL with k == 0: no log-probability work (the call then launches what
 * calm_b200_decode_sample_queue_context launches while no non-neutral request is in flight); otherwise the _logprobs
 * rules apply.  Contexts, the schedule, placement, stops, steps, prompt_rows and independence are the context call's:
 * request i's outputs do not depend on the other requests, max_rows, its slots, seq_len or an earlier call.  The call
 * aborts before any device work where calm_b200_decode_sample_queue_logprobs aborts, and when n_bias < 0, a bias list
 * lies outside [0, n_bias), a bias id is outside [0, vocab_size) or repeats within one list, a value is not finite,
 * |p|, |f| or |b| exceeds 1e6, or r lies outside [1e-6, 1e6] (bounds that keep every l2 finite).
 * Fallback (return 0; as the context call: MoE, tensor parallelism, shapes the prompt pass does not serve, requests
 * that do not fit seq_len).  A neutral request runs the context call's fallback.  A non-neutral one decodes on the
 * decode path and takes each step's device logits; the host applies the expression above and takes the first maximum
 * (greedy) or calls calm_b200_sample_logits with the request's state, and log-probabilities come from l2 in double as in
 * calm_b200_decode_sample_queue_logprobs' fallback.
 * Memory.  The first call with a non-neutral request allocates 16 lanes of 8 bytes per vocabulary entry, a count and
 * a bias row (16.4 MB at a 128256-token vocabulary), and room for the call's tokens and bias lists (4 bytes per token
 * of n, 8 per entry of n_bias), regrown by a larger call. */
int calm_b200_decode_sample_queue_penalties(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                            const int* off, const int* len, int nreq, const int* max_new, const float* temperature, const float* minp,
                                            const float* presence, const float* frequency, const float* repetition, const int* bias_off,
                                            const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias, const int* stop, int n_stop,
                                            int max_rows, unsigned long long* rng_states, int* out_tokens, int* out_len, int* steps,
                                            int* prompt_rows, int k, float* logprobs, int* top_ids, float* top_logprobs);

/* calm_b200_decode_sample_queue_penalties where each request may be constrained to a finite token automaton: structured
 * output (JSON mode, JSON schemas, regular expressions, guided choices; INTEGRATION.md "Structured output").
 * The automaton.  One for the whole call, with states 0 .. n_states-1 and W = ceil(vocab_size / 32) words per state:
 * allow[s*W + v/32] bit v%32 set means token v is allowed in state s (bits at or past vocab_size are 0).  After an
 * allowed token v the next state is exc_next[e] when exc_tok[e] == v for some e in [exc_off[s], exc_off[s+1]) (exc_tok
 * strictly ascending within a state, every listed token allowed in s), otherwise next_default[s].  A state with no
 * allowed token is final.
 * Start states.  start[i] == -1: request i is unconstrained; start == NULL: no request is (the call is then
 * calm_b200_decode_sample_queue_penalties exactly).  The automaton arrays are read only when some start[i] >= 0.
 * Processing.  At request i's step j in state s, with l2 the _penalties call's processed logit:
 *     l3(v) = l2(v) if v is allowed in s, otherwise -inf
 * and l3 replaces l2 for everything the step does: a greedy request's token is the first maximum of l3; logprobs is
 * l3[tok] - M - ln S over the allowed tokens, a masked token's log-probability -inf; when fewer than k tokens are
 * allowed, top_ids / top_logprobs hold -1 / -inf at the ranks past them.
 * Sampling.  A token whose l3 is -inf never survives the min-p cut (at minp == 0 the reference's
 * logit >= max + log(0) * T would keep it, and its rounding fallback could land on it).  With at most 2048 survivors the
 * drawn token is exactly the reference's sample() over the allowed tokens alone, in ascending id order; beyond 2048 it is
 * the device sampler's chunk-by-chunk rule over the full row with the masked entries left out.  One coin is drawn per
 * step, as without a constraint, also for a forced token (a state with one allowed token).
 * Retirement.  A request retires after the step that gives its max_new-th token, a stop token, or a token whose next
 * state is final; that token is emitted and counted in out_len.  out_state[i] (out_state may be NULL) receives the state
 * after the request's last token (start[i] when max_new[i] == 0), or -1 for an unconstrained request: a final state
 * tells a completed structure from one cut off by max_new.
 * Invariants.  An unconstrained request gets exactly the bits of the _penalties call, whatever shares its steps; with
 * start NULL or all -1 the call launches exactly what _penalties launches.  Request i's outputs do not depend on the
 * other requests, max_rows, its slots, seq_len or an earlier call.  The host follows each constrained request's state
 * from the step's tokens, which it reads back after each step with a constrained row, as it does with a stop list.
 * Aborts, before any device work: where calm_b200_decode_sample_queue_penalties aborts, and when n_states < 0, an
 * automaton array is NULL while some start[i] >= 0, a start lies outside [-1, n_states), allow has a bit set past the
 * vocabulary, exc_off[0] != 0 or exc_off decreases, an exception token is not strictly ascending or not allowed in its
 * state, an exception's next state lies outside [0, n_states), next_default[s] lies outside [-1, n_states), a state
 * allows a token outside its exception list while next_default[s] == -1, or a request with max_new > 0 starts in a
 * final state.
 * Fallback (return 0; as the _penalties call).  A constrained request decodes on the decode path and takes each step's
 * device logits; the host applies l2, then the mask, takes the first allowed maximum (greedy) or runs the masked sampler
 * kernels on the processed row with the request's state, and computes log-probabilities in double as the _logprobs
 * call's fallback does.
 * Memory.  A call with a constrained request uploads the bitmasks once, 4 W bytes per state (16 KB at a 128256-token
 * vocabulary), regrown by a larger call; the exception lists and default next states stay on the host.
 * Cost per call.  Nothing is kept between calls: each call with a constrained request checks the whole automaton on the
 * host (every bitmask word read and popcounted, every exception checked: n_states x W words, 16 MB for 1000 states at
 * 128256 tokens) and uploads every bitmask, before its first step.  A host that reuses a large automaton across many
 * short calls pays both every time; that cost has not been measured. */
int calm_b200_decode_sample_queue_constrained(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                              const int* off, const int* len, int nreq, const int* max_new, const float* temperature, const float* minp,
                                              const float* presence, const float* frequency, const float* repetition, const int* bias_off,
                                              const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias, const int* stop, int n_stop,
                                              int max_rows, unsigned long long* rng_states, int* out_tokens, int* out_len, int* steps,
                                              int* prompt_rows, int k, float* logprobs, int* top_ids, float* top_logprobs, int n_states,
                                              const uint32_t* allow, const int* next_default, const int* exc_off, const int* exc_tok,
                                              const int* exc_next, const int* start, int* out_state);

/* calm_b200_decode_sample_queue_constrained where each sampled request may also truncate its distribution to top-k
 * and top-p (nucleus) before the draw: top_k[i] (0 = off) and top_p[i] (1 = off), either array NULL meaning off for
 * every request (INTEGRATION.md "Top-k and top-p").
 * The rule.  At request i's step j, sampled (temperature T > 0, minp < 1), let l3 be the _constrained call's
 * processed and masked logits and M = max l3.
 *   Rank order: the allowed tokens (l3 != -inf) by l3 descending, equal logits lowest id first (the _topk calls' rule).
 *   Mass: q(v) = expf((l3(v) - M) / T), the exact fp32 value the sampler forms for a survivor, and
 *     m(v) = floor(q(v) * 2^40) as an unsigned 64-bit integer (m(argmax) = 2^40; sums are exact and associative).
 *   top_k = K > 0: keep the first K ranks.
 *   top_p = P < 1: with Z the total mass of the top-K set (of every allowed token when K is off) and
 *     target = ceil(Z * P) in exact integer arithmetic (P the fp32 value taken exactly), keep the shortest rank prefix
 *     of that set, at least one token, whose mass sum is >= target.  The nucleus is normalised over the top-k set:
 *     temperature -> top-k -> top-p -> min-p, Hugging Face's warper order and vLLM's top-k-then-top-p.
 *   Min-p: the reference's cut l >= M + log(minp) * T applies on top, unchanged; M is always kept.
 *   The draw: the survivors go through exactly the masked sampler (index order, the reference's fp32 additions, one
 *     coin per step): a truncated token behaves exactly like a token the automaton masked.
 * Greedy requests take the first maximum, which every truncation keeps: their top_k / top_p change nothing.
 * What truncation does not change: logprobs, top_ids and top_logprobs stay the _constrained call's, the model's
 * processed distribution at temperature 1 before min-p, top-k and top-p; penalty counts and automaton states
 * advance from the emitted token, as before.
 * Invariants.  A request with top_k 0 and top_p 1 gets the _constrained call's bits whatever shares its steps; with
 * top_k and top_p NULL, or all neutral, the call launches exactly what _constrained launches.  Request i's outputs do
 * not depend on the other requests, max_rows, its slots, seq_len or an earlier call.
 * Device work.  A step with a truncated sampled row runs k_sample_trunc_rows (one 8-CTA thread-block cluster per such
 * row: a radix select over its logits staged in shared memory) after the classifier, which writes -inf over the
 * row's dropped entries, then the masked sampler scan.  Truncation serves vocabularies up to 262144 tokens.
 * Aborts, before any device work: where _constrained aborts, and when a top_k is negative, a top_p is not finite or
 * outside (0, 1], or a request with max_new > 0 is sampled with top_k > 0 or top_p < 1 on a vocabulary larger than
 * 262144 tokens.
 * Fallback (return 0; as the _constrained call).  A truncated request decodes on the decode path; the host applies
 * l2 and the mask to each step's device logits and draws with calm_b200_sample_logits_truncated's kernels and the
 * request's state. */
int calm_b200_decode_sample_queue_truncated(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                            const int* off, const int* len, int nreq, const int* max_new, const float* temperature, const float* minp,
                                            const float* presence, const float* frequency, const float* repetition, const int* bias_off,
                                            const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias, const int* stop, int n_stop,
                                            int max_rows, unsigned long long* rng_states, int* out_tokens, int* out_len, int* steps,
                                            int* prompt_rows, int k, float* logprobs, int* top_ids, float* top_logprobs, int n_states,
                                            const uint32_t* allow, const int* next_default, const int* exc_off, const int* exc_tok,
                                            const int* exc_next, const int* start, int* out_state, const int* top_k, const float* top_p);

/* calm_b200_decode_sample_queue_truncated that fills the rows a step leaves free (16 per step, less the requests in
 * flight) with prompt-lookup drafts of the requests' own tokens, verified in the same step (DESIGN.md s.6; INTEGRATION.md
 * "Lookup drafts in the queue").  It takes every argument of the _truncated call, then max_draft, drafted and accepted.
 * Outputs.  out_tokens, out_len, rng_states, logprobs, top_ids, top_logprobs, out_state, prompt_rows and the return value
 * are bit for bit what calm_b200_decode_sample_queue_truncated gives with the same arguments; only *steps may be smaller.
 * *drafted (drafted may be NULL) receives the draft rows the call ran, *accepted (may be NULL) the drafts it accepted.
 * Slots past out_len[i] are left untouched, as in the _truncated call.
 * max_draft in [0, 15].  0: no drafts; the call launches exactly what _truncated launches and takes the same steps.
 * The draft rule (calm_b200_decode_lookup's with source == NULL).  Over request i's sequence ctx ++ prompt ++ its tokens so
 * far, the key is the last 3 tokens, else 2, else 1, and the draft is what follows the key's rightmost occurrence that
 * some token follows.
 * Which requests draft.  After a step's admission, the requests in flight in admission order each take up to
 * min(max_draft, max_new[i] - out_so_far - 1, rows still free of 16) draft rows, right after the request's own row.
 * The draft then stops before its first stop token, and for a constrained request before the first token its state
 * disallows and before the first token that leads to a final state: no draft row continues a finished request.  A
 * request with non-neutral penalties or bias never drafts.  max_rows counts requests, not rows.
 * Acceptance.  Draft row d of request i is the request at its step j + d, fed the draft's d-th token, and draws with the
 * coin after the d coins before it.  Row d + 1's token is accepted when row d's token equals it; the request emits the
 * tokens of its rows 0 .. a, a the accepted drafts, and draws one coin per emitted token.  Each emitted token is the one
 * the _truncated call gives at that step, since a row's result depends on its own keys, token, position and state alone.
 * Cost.  With max_draft > 0, every step copies its tokens and emitted flags back and synchronises, so that the host can
 * look up the next drafts.  Rejected draft rows leave cache slots and device-side outputs at or past the request's
 * position, which later steps overwrite; the host copies only each request's first out_len[i] outputs.
 * Aborts, before any device work: where the _truncated call aborts, and when max_draft is outside [0, 15].
 * Fallback (return 0; as the _truncated call): the _truncated call's fallback, with *steps, *drafted and *accepted 0. */
int calm_b200_decode_sample_queue_lookup(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                         const int* off, const int* len, int nreq, const int* max_new, const float* temperature, const float* minp,
                                         const float* presence, const float* frequency, const float* repetition, const int* bias_off,
                                         const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias, const int* stop, int n_stop,
                                         int max_rows, unsigned long long* rng_states, int* out_tokens, int* out_len, int* steps,
                                         int* prompt_rows, int k, float* logprobs, int* top_ids, float* top_logprobs, int n_states,
                                         const uint32_t* allow, const int* next_default, const int* exc_off, const int* exc_tok,
                                         const int* exc_next, const int* start, int* out_state, const int* top_k, const float* top_p,
                                         int max_draft, int* drafted, int* accepted);

/* The reference's sample() (sampler.c:80-90) on the device: temperature / min-p sampling with the reference's
 * xorshift* generator (sampler.c:7-17), no logits transfer and no host scan of the vocabulary per token.
 * temperature == 0 or minp >= 1 is greedy and leaves *rng_state alone, as in the reference.  Survivors are added
 * in index order like the reference does (exactly its additions up to 2048 survivors; chunk by chunk beyond).
 * decode_sample feeds token0 at pos0 and then n_tokens-1 times its own sample; out_tokens[i] = sample after step i.
 * The logits stay in HBM (calm_b200_read_device_logits copies the last step's); state.logits is not updated. */
void calm_b200_decode_sample(struct Transformer* transformer, int token0, int pos0, int n_tokens, float temperature, float minp,
                             unsigned long long* rng_state, int* out_tokens);
int calm_b200_forward_sample(struct Transformer* transformer, int token, int pos, float temperature, float minp, unsigned long long* rng_state);
void calm_b200_read_device_logits(float* out_vocab);

/* The same sampler kernels on logits supplied by the host (any vocabulary size, no model needed): returns the token,
 * advances *rng_state exactly as sample() does; *device_us (optional) = duration of the two sampler kernels. */
int calm_b200_sample_logits(const float* logits_host, int vocab, float temperature, float minp, unsigned long long* rng_state, float* device_us);

/* calm_b200_sample_logits with calm_b200_decode_sample_queue_truncated's top-k / top-p rule on one host row: chunk
 * maxima, k_sample_trunc_rows, the masked scan and the pick (a -inf logit never survives).  top_k 0 and top_p 1 mean
 * off; with both off the row still goes through the masked scan.  out_row (may be NULL) receives the row after
 * truncation, -inf at the dropped ids (for a greedy draw, the row unchanged).  Aborts when top_k < 0, top_p is not
 * finite or outside (0, 1], or a sampled draw with truncation has a vocabulary above 262144 tokens. */
int calm_b200_sample_logits_truncated(const float* logits_host, int vocab, float temperature, float minp, int top_k, float top_p,
                                      unsigned long long* rng_state, float* out_row, float* device_us);

/* Device timer on the library's stream (CUDA events): start, ..., stop -> ms. */
void calm_b200_timer_start(void);
float calm_b200_timer_stop(void);

/* The cudaStream_t all kernels of this library are launched on. */
void* calm_b200_stream(void);

/* Number of kernels this library has launched since load (bench "gpu_launches"). */
uint64_t calm_b200_launch_count(void);

/* Read back one KV-cache entry as floats in the reference's logical order
 * (kv_dim values each, reference infer.c:378-381); for parity tests. */
void calm_b200_read_kv(struct Transformer* transformer, int layer, int kv_pos, float* k_out, float* v_out);

/* (test aid) Copy one of the engine's buffers to the host as floats, after waiting for the library's stream, so a test
 * can check what each stage of the last token (or of the last prompt pass) wrote.  Returns the number of floats the
 * buffer holds; nothing is copied when `out` is NULL or `cap` is smaller than that.  `layer` is read by the two cache
 * selectors only.  With one layer nothing overwrites a stage's output before the token ends; with more, the
 * activation buffers hold the last layer's values.  No kernel is launched and nothing on the token path changes.
 *   X        float[dim]                   residual stream (after the last w2)
 *   XB       float[dim]                   the attention norm's output that parallel-norm models keep for the FFN
 *   Q        float[q_dim]                 rotated queries                          ATT  float[q_dim]  attention output
 *   HB       float[n_active][hidden]      gated FFN hidden vector (one row per active expert; dense models: one row)
 *   MOE_SEL  float[2 * n_active]          the router's experts (as floats), then their weights
 *   KEYS, VALUES  float[n_kv_heads][seq_len][head_dim]   one layer of the cache, every slot, decoded from fp16 / e5m2
 *   PF_X, PF_Q, PF_ATT, PF_HB   float[rows][dim | q_dim | q_dim | hidden]   the prompt pass's residual stream, rotated
 *            queries, attention output and FFN hidden matrix (the last two kept as f16 hi + lo pairs, summed here in
 *            float); rows = the pass's token tiles (a multiple of 128, at least n), of the last block of <= 2048 tokens
 *   PF_LOGITS  float[n][vocab]          the logit rows of the last calm_b200_verify_sample block that took the short-block
 *            path (n of its tokens), or of the last step of the last sampled calm_b200_decode_sample_n or
 *            calm_b200_decode_sample_batch call that took its new path (n = nseq, row b = sequence b), the values its
 *            sampler drew from, or of the last step of a calm_b200_decode_sample_queue call on its new path if that step
 *            sampled any row (n = the rows in flight).  After calm_b200_decode_sample_queue_penalties the rows of
 *            non-neutral requests hold their processed logits l2, the values the sampler drew from
 *   BEAM_IDS, BEAM_LOGPROBS  float[steps][B][K]   the last calm_b200_decode_beam call on its path: each step's rows'
 *            K best ids and their lp, as the walk read them (step 0's rows past row 0: id -1, lp -inf)
 *   BEAM_ANC  float[B][max_new]   that call's ancestry as its last step read it: entry [b][i] is the row of step i whose
 *            key row b read as its key pos0 + i (i <= steps - 1; the rest unspecified)
 *   After calm_b200_decode_sample_n or calm_b200_decode_sample_batch on its new path, the PF_* matrices hold the last
 *   step, row b = sequence b.  After calm_b200_decode_sample_queue on its new path, the PF_* matrices and PF_LOGITS hold
 *   the last step, with the rows in flight in admission order.  After calm_b200_decode_beam on its path, the PF_*
 *   matrices hold the last step, row b = live beam b. */
enum {
	CALM_B200_STATE_X = 0, CALM_B200_STATE_XB = 1, CALM_B200_STATE_Q = 2, CALM_B200_STATE_ATT = 3, CALM_B200_STATE_HB = 4,
	CALM_B200_STATE_MOE_SEL = 5, CALM_B200_STATE_KEYS = 6, CALM_B200_STATE_VALUES = 7,
	CALM_B200_STATE_PF_X = 8, CALM_B200_STATE_PF_Q = 9, CALM_B200_STATE_PF_ATT = 10, CALM_B200_STATE_PF_HB = 11,
	CALM_B200_STATE_PF_LOGITS = 12, CALM_B200_STATE_BEAM_IDS = 13, CALM_B200_STATE_BEAM_LOGPROBS = 14, CALM_B200_STATE_BEAM_ANC = 15
};
int calm_b200_read_state(int which, int layer, float* out, int cap);

/* (test aid) Overwrite with 0xFF bytes (NaN as f32, f16 and e5m2) every buffer whose previous contents must not influence
 * any later call, and the KV-cache slots [kv_from_pos, seq_len) of every layer and kv head (kv_from_pos >= seq_len: none).
 * Waits for the library's stream before and after.  Launches no kernel of the token path; changes no kernel.
 * What steers control flow, a wait or an address (token parameters, the attention's fold cells and counter, the
 * tensor-parallel exchange area, router and sampler state, index buffers, weights) is left alone: DESIGN.md s.3. */
void calm_b200_poison_state(struct Transformer* transformer, int kv_from_pos);

/* Fill the KV cache positions [0, n_pos) of every layer with a deterministic
 * pseudo-random pattern (bench: decode at a late position without running the
 * whole prefix). */
void calm_b200_fill_kv(struct Transformer* transformer, int n_pos, uint64_t seed);

/* Per-stage profiling at run time (what CALM_B200_PERF=1 enables from the start).  While on, every token runs the
 * PRODUCTION CUDA graph (same kernels, programmatic dependent launch) with one extra argument per launch: a stamp slot
 * into which the kernel folds min(start) / max(end) of its CTAs, read from %globaltimer -- the reference's coopstage
 * scheme (infer.cu:390-402), so perf_cuda() describes the path that produces the tokens, not an eager variant.
 * set_perf(1) clears the counters.  stage_stats() returns 0 past the last stage; totals are over all launches of that
 * stage since set_perf(1): milliseconds (first CTA past its dependency wait -> last CTA done), algorithmic bytes (the
 * reference's per-stage accounting, infer.cu:683-699) and launch count.  perf_token_ms(): mean span of a token, first
 * stamp to last (consecutive kernels overlap under PDL, so the stage sums can exceed it). */
void calm_b200_set_perf(int on);
int calm_b200_stage_stats(int stage, char* name, int name_cap, double* ms_total, double* bytes_total, long* launches);
double calm_b200_perf_token_ms(void);
/* (debug) 16 raw %globaltimer stamps the attention kernel of the middle layer left during the last profiled token. */
void calm_b200_debug_stamps(unsigned long long* out16);

/* Stand-alone run of the production matvec kernel: y[d] = W[d,n] . x[n] with W
 * in the `dbits` format at device pointer `w_device`; x and y are HOST arrays.
 * Returns the kernel's device time in milliseconds (mean over `iters` launches
 * after `warmup` launches).  Used by the unit parity tests (vs reference
 * infer.c:209-221) and by the per-kernel roofline bench. */
float calm_b200_matvec(int dbits, const void* w_device, const float* x_host, float* y_host, int n, int d, int warmup, int iters);

#ifdef __cplusplus
}
#endif

#endif /* CALM_B200_H */
