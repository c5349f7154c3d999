/*
 * b200t5.h - C ABI of libb200t5.so: T5 greedy generation on one NVIDIA H100 (sm_90a), the hot path of the
 * workshop's batch-inference loop. Two T5 architectures load: FLAN-T5 / T5 v1.1 (gated-GELU feed-forward, untied
 * lm_head) and the original T5 v1.0 (t5-small / t5-base / t5-large and their fine-tunes: ReLU feed-forward, lm_head
 * tied to the shared embedding, decoder output scaled by d_model ** -0.5). d_kv must be 64 (not t5-3b / t5-11b).
 *
 * What this boundary replaces in the reference (ray-project/anyscale-workshop-nyc-2023):
 * the reference has no FFI of its own; its plug-in seam is the Python attribute
 * `self.model` of HuggingFaceModelPredictor (NLP_workloads/Anyscale_job/predictor.py:27-37):
 *   - `checkpoint.get_model(model_cls, **kw)`   predictor.py:68   -> b200t5_create + b200t5_set_weight* + b200t5_finalize
 *   - `self.model.device`                       predictor.py:98   -> the `device` given to b200t5_create
 *   - `self.model.generate(**generate_kwargs)`  predictor.py:102  -> b200t5_generate / b200t5_generate_host
 * The arithmetic behind `generate` lives in the reference's pinned dependency
 * transformers==4.27.2 (requirements.txt:168): T5ForConditionalGeneration + greedy search.
 * INTEGRATION.md shows the ctypes binding a maintainer adds on the reference side.
 *
 * Two builds export this same ABI (csrc/Makefile), one per numerics contract of the dependency:
 *   libb200t5.so      torch_dtype=bfloat16: every eager op rounds to bf16 (SURVEY Appendix A.1-6)
 *   libb200t5_f16.so  torch_dtype=float16, the notebook's literal setting (Text_generation_with_FLAN_T5.ipynb,
 *                     BatchPredictor.from_checkpoint(..., torch_dtype=torch.float16)): fp16 roundings, the
 *                     feed-forward `wo` kept as an fp32 weight with an fp32 output (transformers'
 *                     _keep_in_fp32_modules = ["wo"]) and therefore an fp32 residual stream (Appendix A.7).
 * b200t5_set_weight converts whatever dtype it is given to the build's own types; b200t5_encode returns the
 * encoder output in the build's 2-byte type; the single-kernel test hooks exist in the bf16 build only.
 *
 * Conventions
 *   - every function returns 0 on success, a negative B200T5_E* code otherwise; the message
 *     is available from b200t5_last_error(handle) (or b200t5_last_global_error() when no
 *     handle exists yet). No C++ exception crosses this boundary.
 *   - the caller owns every buffer it passes in; weights are copied (and converted to bf16)
 *     into library-owned HBM by b200t5_set_weight, so the caller may free them afterwards.
 *   - the library owns its workspace, KV arenas and CUDA graphs; b200t5_destroy frees them.
 *   - a handle is not thread-safe (one call in flight); distinct handles are independent.
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).
 *   - there is no CPU fallback: every entry point that computes requires a CUDA device of
 *     compute capability 10.x and fails with B200T5_ENODEV otherwise.
 */
#ifndef B200T5_H_
#define B200T5_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200T5_OK 0
#define B200T5_EINVAL (-1)  /* bad argument / unsupported configuration */
#define B200T5_ENODEV (-2)  /* no sm_90 device */
#define B200T5_ECUDA (-3)   /* CUDA runtime / driver error */
#define B200T5_ESTATE (-4)  /* call order violated (e.g. generate before finalize) */
#define B200T5_ENOMEM (-5)

#define B200T5_DTYPE_BF16 0
#define B200T5_DTYPE_F16 1
#define B200T5_DTYPE_F32 2

typedef struct b200t5_ctx* b200t5_handle;

/* Mirrors the fields of transformers.T5Config the path depends on (config.json keys). */
typedef struct b200t5_config {
  int32_t vocab_size;          /* 32128 for FLAN-T5 */
  int32_t d_model;             /* 512 / 768 / 1024 */
  int32_t d_kv;                /* must be 64 */
  int32_t d_ff;                /* 1024 / 2048 / 2816 */
  int32_t num_heads;           /* 6 / 12 / 16 */
  int32_t num_layers;          /* encoder blocks */
  int32_t num_decoder_layers;  /* decoder blocks */
  int32_t relative_attention_num_buckets;   /* 32 */
  int32_t relative_attention_max_distance;  /* 128 */
  float layer_norm_epsilon;                 /* 1e-6 */
  int32_t pad_token_id;                     /* 0 */
  int32_t eos_token_id;                     /* 1 */
  int32_t decoder_start_token_id;           /* 0 */
  int32_t is_gated_gelu;          /* 1: feed_forward_proj "gated-gelu" (T5 v1.1 / FLAN-T5: wi_0, wi_1, wo);
                                   * 0: "relu" (T5 v1.0: wi, wo). Any other value: B200T5_EINVAL */
  int32_t scale_decoder_outputs;  /* 1: the final decoder norm's output is multiplied by fp32(d_model ** -0.5) and
                                   * rounded once more before the lm_head (transformers: unless the checkpoint's config
                                   * says tie_word_embeddings: false); 0: not. Any other value: B200T5_EINVAL */
} b200t5_config;

/* Greedy-generation controls: the subset of GenerationConfig the reference path uses
 * (predictor.predict(..., max_new_tokens=128), notebook line 908-913). */
typedef struct b200t5_gen_params {
  int32_t max_new_tokens;          /* >= 1 */
  int32_t min_new_tokens;          /* EOS is masked while fewer than this many tokens were generated */
  int32_t eos_token_id;            /* -1: take from config */
  int32_t pad_token_id;            /* -1: take from config */
  int32_t decoder_start_token_id;  /* -1: take from config */
  int32_t poll_interval;           /* steps between device->host "all rows finished" checks; <=0: 8 */
} b200t5_gen_params;

/* Greedy-mode logits processors (transformers GenerationConfig options of the same names; generation/logits_process.py),
 * applied in transformers' order to the lm_head logits rounded to the build's 2-byte type and widened to fp32:
 * encoder repetition penalty, repetition penalty, no-repeat n-grams, encoder no-repeat n-grams, bad words, the EOS mask
 * of min_new_tokens, suppressed tokens, begin-suppressed tokens; then the arg-max. Passing NULL instead of this struct
 * is the plain greedy path; so is a struct whose every field is a no-op. Host pointers, read during the call only. */
typedef struct b200t5_logits_params {
  double repetition_penalty;          /* 1.0 = off; > 0. Over the decoder ids so far, the start token included */
  double encoder_repetition_penalty;  /* 1.0 = off; > 0. Over the prompt's ids, padding positions included */
  int32_t no_repeat_ngram_size;          /* 0 = off; over the decoder ids, the start token included */
  int32_t encoder_no_repeat_ngram_size;  /* 0 = off; n-grams of the prompt's ids, padding included */
  const int32_t* suppress_tokens;        /* masked at every step */
  int32_t n_suppress_tokens;
  const int32_t* begin_suppress_tokens;  /* masked at the first generated position only */
  int32_t n_begin_suppress_tokens;
  const int32_t* eos_token_ids;  /* 1..16 ids: any of them finishes a row and all are masked while fewer than
                                  * min_new_tokens were generated; n_eos_token_ids == 0: gen_params' eos_token_id */
  int32_t n_eos_token_ids;
  const int32_t* bad_words_ids;      /* the sequences, concatenated */
  const int32_t* bad_words_offsets;  /* [n_bad_words + 1]: sequence i = bad_words_ids[offsets[i] .. offsets[i+1]) */
  int32_t n_bad_words;               /* a one-token sequence is banned at every step, except one equal to an EOS id,
                                      * which is dropped; a longer one bans its last token when the rest of it ends
                                      * the decoder ids */
} b200t5_logits_params;

/* Token log-probabilities of a call (the *_scored entry points). At every step the lm_head epilogue keeps, beside the
 * arg-max, the log-sum-exp of the step's processed fp32 scores (the act-rounded logits after the logits processors and
 * the EOS mask), so for the token t a row takes at step s
 *   token_logits[row][s]   = score[t]                                  (what the arg-max compared)
 *   token_logprobs[row][s] = score[t] - max - log(sum exp(score - max))  = log_softmax(score)[t]
 * without the [rows, vocab] scores ever reaching memory. Positions a row does not reach (after its EOS) hold 0, so the
 * sum of a row of token_logprobs is the log-likelihood of its sequence. Both arrays are fp32 [rows, max_new_tokens].
 * forced_ids (teacher forcing): instead of the arg-max, row r takes forced_ids[r][s] at step s, until its last label -
 * the position before the first -100 or forced_len - and not until an EOS; out_ids then echoes the labels and
 * token_logprobs are log p(label | prompt, earlier labels), what a cross-entropy loss sums. Every row needs at least
 * one label, labels lie in [0, vocab_size), -100 may only trail, 1 <= forced_len <= max_new_tokens, and logits
 * processors cannot be combined with forced_ids: B200T5_EINVAL otherwise.
 * The pointers are device pointers for b200t5_generate_scored and host pointers for the other two entry points. */
typedef struct b200t5_score_io {
  float* token_logprobs;      /* out, fp32 [rows, max_new_tokens]; 0 where the row has no token */
  float* token_logits;        /* out, may be NULL: the processed score of the chosen token */
  const int64_t* forced_ids;  /* in, may be NULL: [rows, forced_len], -100 after a row's last label */
  int32_t forced_len;         /* <= max_new_tokens */
} b200t5_score_io;

typedef struct b200t5_stats {
  float encoder_ms;       /* encoder + cross-KV projection of the last generate call (CUDA events) */
  float decode_ms;        /* decode loop of the last generate call (CUDA events) */
  int32_t decode_steps;   /* steps executed */
  int64_t kernel_launches;/* kernels launched by this library in the last generate call */
  double decode_algo_bytes;  /* algorithmic HBM bytes of the decode loop (SURVEY 8d model) */
  double encoder_flops;      /* encoder + cross-KV projection FLOPs */
  int32_t xattn_kernel;      /* decode cross-attention kernel of the last call: 0 per-thread-load, 1 TMA stream */
  int32_t row_chains;        /* row-chains the decode step was split into */
} b200t5_stats;

/* ---- lifecycle ---------------------------------------------------------------------- */
int b200t5_create(const b200t5_config* cfg, int device, b200t5_handle* out);
/* `name` is the Hugging Face state-dict key (e.g. "decoder.block.3.layer.1.EncDecAttention.q.weight"),
 * `dev_ptr` a device pointer on `device`, row-major with nn.Linear layout [out, in].
 * Unknown names that HF also ignores are accepted and dropped. */
int b200t5_set_weight(b200t5_handle h, const char* name, const void* dev_ptr, int dtype, const int64_t* shape,
                      int ndim);
/* Checks that every required tensor arrived, repacks (QKV concat, GeGLU interleave, cross-KV concat). A ReLU model
 * (is_gated_gelu 0) takes {encoder,decoder}.block.*.layer.*.DenseReluDense.wi.weight [d_ff, d_model] in place of
 * wi_0 / wi_1. Without lm_head.weight the lm_head is shared.weight (tied). */
int b200t5_finalize(b200t5_handle h);
int b200t5_destroy(b200t5_handle h);
const char* b200t5_last_error(b200t5_handle h);
const char* b200t5_last_global_error(void);

/* ---- the hot path ------------------------------------------------------------------- */
/* Device-resident variant. input_ids / attention_mask: int64 [B,S] on the device
 * (attention_mask may be NULL = all ones). out_ids: int64 [B, max_new_tokens+1], column 0 is the
 * decoder start token, rows are padded with pad_token_id after their EOS; out_len: int32 [B] =
 * tokens generated per row (including the EOS). Enqueued on `stream`; returns after the last
 * kernel was enqueued and the early-exit polling finished (the outputs are complete when the
 * stream is synchronised). */
int b200t5_generate(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                    const b200t5_gen_params* params, int64_t* out_ids, int32_t* out_len, void* stream);
/* Host-buffer variant (what a foreign-language host binds): copies inputs H2D, generates,
 * copies results D2H and synchronises. */
int b200t5_generate_host(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                         const b200t5_gen_params* params, int64_t* out_ids, int32_t* out_len);
/* Slot-pool (continuous-batching) variant for a caller that holds more than one batch: the driver loop of
 * BatchPredictor.predict (Text_generation_with_FLAN_T5.ipynb cell "predictor.predict(...)", NB:908-913) hands
 * every `batch_size` rows to predictor.py:102 separately, so each batch runs until its slowest row has finished.
 * Here N prompts (host int64 [N,S] buffers, attention_mask may be NULL) share `pool` decode slots (<= 0: 256):
 * a slot whose row has emitted EOS or max_new_tokens is refilled with the next prompt once at least `admit_min`
 * slots are free (<= 0: pool / 8); finished rows stop streaming their K/V at once. out_ids: host int64
 * [N, max_new_tokens+1], out_len: host int32 [N], row r = prompt r, same layout and - token for token - the same
 * values as b200t5_generate_host gives for that prompt in a `pool`-row batch. Synchronous. */
int b200t5_generate_stream(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int64_t N, int S,
                           const b200t5_gen_params* params, int pool, int admit_min, int64_t* out_ids,
                           int32_t* out_len);
/* The three entry points above with logits processors (`logits` may be NULL: the call is exactly the one above).
 * Every processor state lives in device memory, so the step graph captured for a set of active processors is replayed
 * whatever their values. Ids outside [0, vocab_size), an empty bad-word sequence, a penalty <= 0 or a negative n-gram
 * size fail with B200T5_EINVAL. */
int b200t5_generate_ex(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                       const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                       int32_t* out_len, void* stream);
int b200t5_generate_host_ex(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                            const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                            int32_t* out_len);
int b200t5_generate_stream_ex(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int64_t N, int S,
                              const b200t5_gen_params* params, const b200t5_logits_params* logits, int pool,
                              int admit_min, int64_t* out_ids, int32_t* out_len);
/* The three entry points above with token log-probabilities (`score` may be NULL: the call is exactly the one above,
 * same graphs, same number of kernel launches). rows = B, or N for the slot pool. A row's numbers do not depend on the
 * entry point, the batch or the slot it is decoded in: the three return bit-identical arrays for the same prompt. */
int b200t5_generate_scored(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                           const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                           int32_t* out_len, const b200t5_score_io* score, void* stream);
int b200t5_generate_host_scored(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                                int32_t* out_len, const b200t5_score_io* score);
int b200t5_generate_stream_scored(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int64_t N, int S,
                                  const b200t5_gen_params* params, const b200t5_logits_params* logits, int pool,
                                  int admit_min, int64_t* out_ids, int32_t* out_len, const b200t5_score_io* score);
int b200t5_get_stats(b200t5_handle h, b200t5_stats* out);

/* A decoder prompt (transformers' generate(decoder_input_ids=...)): b200t5_generate_scored whose rows start from the
 * decoder ids d = decoder_input_ids int64 [B, P] instead of the start token. The library takes d as given: d[b][0] is
 * the row's first decoder input, so a caller that follows transformers prepends the decoder start token itself (when
 * every row's first id differs from it). Every row starts unfinished whatever d holds; every prompt position is
 * attended to. The prompt's positions 0 .. P-2 run as one forward pass over B*(P-1) rows that fills the self-attention
 * cache; then max_new_tokens decode steps run from position P-1.
 *   out_ids: int64 [B, P + max_new_tokens] = d, then the generated tokens, then pad_token_id;
 *   out_len: int32 [B] = NEW tokens per row (EOS included), not counting the prompt;
 *   score (may be NULL): token_logprobs / token_logits fp32 [B, max_new_tokens], one column per new token.
 * min_new_tokens counts new tokens; begin_suppress_tokens apply at position P-1, the first generated one; the
 * repetition penalty and the n-gram bans see d. P == 1 with d[b][0] equal in every row is exactly
 * b200t5_generate_scored with that decoder start token: same kernels, same launch count, same bits.
 * B200T5_EINVAL for P < 1, decoder ids outside [0, vocab_size), P-1 + max_new_tokens > 4096 or score->forced_ids, and
 * for P >= 2 when B200T5_SK sets the feed-forward wi tile to other than 128 rows (the prefill is b200t5_forward's
 * decoder pass, which needs that tile), all before anything is enqueued.
 * decoder_input_ids is a HOST pointer in both entry points: the prompt is checked and staged on the host. The other
 * pointers are device pointers, and the call is enqueued on `stream` like b200t5_generate_scored. */
int b200t5_generate_prefixed(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                             const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                             int32_t* out_len, const b200t5_score_io* score, const int64_t* decoder_input_ids, int P,
                             void* stream);
/* The same with host buffers (as b200t5_generate_host_scored) for every pointer: synchronous. */
int b200t5_generate_host_prefixed(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                  const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                                  int32_t* out_len, const b200t5_score_io* score, const int64_t* decoder_input_ids, int P);

/* Beam search (transformers' GenerationMixin._beam_search with do_sample=False and one EOS id): each prompt decodes as
 * num_beams rows. Length penalty: a finished hypothesis of l generated tokens scores sum(log-probs) * fp32(1 / l**p),
 * the reciprocal taken in double. Ties: value descending, then token (beam * vocab + token across a prompt) ascending. */
typedef struct b200t5_beam_params {
  int32_t num_beams;             /* 2..16 */
  int32_t num_return_sequences;  /* 1..num_beams */
  double length_penalty;
  int32_t early_stopping;        /* 0 False, 1 True, 2 "never" */
} b200t5_beam_params;

/* Results of a beam call, n = num_return_sequences, row b*n + i = the i-th best hypothesis of prompt b. Device pointers
 * for b200t5_generate_beam, host pointers for b200t5_generate_host_beam. */
typedef struct b200t5_beam_io {
  int64_t* sequences;        /* out [B*n, max_new_tokens+1]: start token, the hypothesis (ending in EOS unless it reached
                              * max_new_tokens), then pad_token_id */
  int32_t* lengths;          /* out [B*n]: generated tokens of each hypothesis */
  float* sequences_scores;   /* out, may be NULL: [B*n] length-penalised scores */
  int64_t* beam_indices;     /* out, may be NULL: [B*n, max_new_tokens] beam of each step as b*num_beams + beam, -1 after
                              * the hypothesis ends */
  float* token_logprobs;     /* out, may be NULL: [B*n, max_new_tokens] each token's log-probability, 0 after the end */
} b200t5_beam_io;

/* Beam-search generate: input_ids / attention_mask as b200t5_generate; gen_params' min_new_tokens masks EOS as in greedy
 * decoding. The encoder and the cross-attention K/V projection run once per prompt; the decode step runs B*num_beams rows.
 * Parameters out of range return B200T5_EINVAL. Enqueued on `stream`, like b200t5_generate. */
int b200t5_generate_beam(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                         const b200t5_gen_params* params, const b200t5_beam_params* beam, const b200t5_beam_io* io,
                         void* stream);
/* The same with host buffers; synchronous. */
int b200t5_generate_host_beam(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                              const b200t5_gen_params* params, const b200t5_beam_params* beam, const b200t5_beam_io* io);
/* Bytes the self-attention cache reordering of the last beam call read and wrote (beam_reorder_kernel), and its steps. */
int b200t5_get_beam_stats(b200t5_handle h, double* reorder_bytes, int32_t* steps);

/* Teacher-forced forward pass (T5ForConditionalGeneration.forward with labels / decoder_input_ids, no cache): the encoder,
 * then the decoder over all T positions of every row at once - causal self-attention, cross-attention, feed-forward as
 * GEMMs over B*T rows - and the lm_head. Every product and attention keeps the rounding points of the decode step, so
 * the results agree with b200t5_decode_logits / the scored entry points within rounding, not bit for bit.
 * All pointers are device pointers; enqueued on `stream` like b200t5_generate (labels and decoder ids are read back to be
 * checked). input_ids / attention_mask as b200t5_generate. decoder_input_ids int64 [B,T], may be NULL when labels are
 * given: then transformers' _shift_right(labels) (the decoder start token, then labels[:, :-1] with -100 replaced by
 * the pad id). labels int64 [B,T], may be NULL: ids in [0, vocab_size) or -100 (ignored) anywhere in a row.
 * A row's results do not depend on the batch it sits in. Both inputs NULL, both outputs NULL, token_logprobs without
 * labels, ids out of range or T outside [1, 4096] return B200T5_EINVAL. */
typedef struct b200t5_forward_io {
  void* logits;           /* out, may be NULL: [B, T, vocab] in the build's 2-byte type */
  float* token_logprobs;  /* out, may be NULL: [B, T] log p(labels[b][t]); 0 where labels is -100; needs labels */
} b200t5_forward_io;
int b200t5_forward(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                   const int64_t* decoder_input_ids, const int64_t* labels, int T, const b200t5_forward_io* io,
                   void* stream);
/* Multiple-choice scoring (rank classification): b200t5_forward over R (prompt, candidate) rows whose prompts are shared.
 * The encoder and the cross-attention K/V projection run over the B prompts only; the decoder runs R*T rows, the
 * candidates of prompt b being rows row_offsets[b] .. row_offsets[b+1]-1, and each prompt's cross-attention runs all
 * its candidates' queries as one sequence against its keys (csrc/attention_decoder.cuh: decoder_cross_packed_kernel).
 * Every row gets the bits b200t5_forward gives it with that row's prompt repeated in its own row.
 * row_offsets is a HOST int32 [B+1] array: 0 first, strictly increasing, R = row_offsets[B]. labels int64 [R,T] (device)
 * as b200t5_forward's labels; the decoder input is transformers' _shift_right(labels). io: logits [R, T, vocab] and/or
 * token_logprobs [R, T]. b200t5_get_stats' encoder_flops then counts the B prompts once each. NULL pointers, offsets
 * that do not start at 0 or do not increase, R*num_heads > 65535, labels out of range or T outside [1, 4096] return
 * B200T5_EINVAL before anything is enqueued. */
int b200t5_forward_choices(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                           const int32_t* row_offsets, const int64_t* labels, int T, const b200t5_forward_io* io,
                           void* stream);

/* ---- measurement hooks (bench.py) --------------------------------------------------- */
/* Times the cross-attention decode kernel alone over the cross-KV arena of the last generate call, in launches of
 * `rows_per_launch` batch rows (0 = the whole batch; the step graph launches one row-chain at a time): reps sweeps
 * over all decoder layers, CUDA events on `stream`; returns the average launch duration and the algorithmic bytes
 * one launch must read (K+V rows of attended keys). A microbenchmark (back-to-back launches, nothing else on the
 * GPU); b200t5_get_xattn_profile gives the figure inside the step graph. */
int b200t5_bench_cross_attn(b200t5_handle h, int reps, int rows_per_launch, float* avg_ms_per_launch,
                            double* bytes_per_launch, void* stream);
/* Runtime options: what the B200T5_* environment variables set at create time, on a live handle (a sweep need not
 * reload the model). A change drops the execution plan; the next call re-captures the step graph. Names: "chains"
 * (row-chains per decode step, 0 = default), "xattn" (decode cross-attention: 0 = per-thread-load kernel, 1 = TMA stream kernel, 2 = per call by prompt fill),
 * "xattn_stages" (8 KB ring stages per CTA), "pdl", "admit_overlap", "sk_stages64", "sk_stages128" (pipeline stages of
 * the split-K decode GEMM tiles, 0 = default), "profile_xattn" (1 = every cross-attention launch inside the step graph
 * records %globaltimer stamps; never on in a timed region), "enc_gemm" (the 128 x 256 encoder GEMMs: 1 = default,
 * epilogue warps drain each tile while the next tile's MMAs run; 0 = the kernel whose epilogue follows each main loop;
 * bit-identical results; environment variable B200T5_ENC_GEMM at create time). Any other name returns B200T5_EINVAL. */
int b200t5_set_option(b200t5_handle h, const char* name, int value);
/* With "profile_xattn" on: mean in-situ duration (first CTA start to last CTA end) of the cross-attention launches the
 * step graph made since the option was set, how many there were, and the algorithmic bytes of one such launch; and,
 * per decoder layer and step, the time during which AT LEAST ONE of the row-chains' cross-attention launches was
 * running (the union of their intervals: the chains' launches may overlap each other) with the bytes the layer's
 * launches read together. bytes_per_layer / busy_us_per_layer is the HBM rate of the cross-attention stream as the
 * step runs it. */
int b200t5_get_xattn_profile(b200t5_handle h, double* avg_us_per_launch, int64_t* launches, double* bytes_per_launch,
                             double* busy_us_per_layer, double* bytes_per_layer);
/* lm_head + fused greedy arg-max exactly as the decode step runs them (csrc/gemm.cuh EpiLmHead<false, false> ->
 * finalize_step_kernel<false, false>):
 * x [M,K] and W [V,K] in the build's 2-byte type (device), `step` the decode position, EOS masked while
 * step < min_new. tokens: int64 [M] (device) = argmax_n act(x . W[n]) with torch.argmax's first-index tie rule
 * (transformers generation/utils.py:2762,2793; logits_process.py:225-233). Test hook. */
int b200t5_test_lm_argmax(int device, const void* x, const void* W, int M, int V, int K, int step, int eos, int min_new,
                          int64_t* tokens, void* stream);
/* One decode step of lm_head + logits processors + arg-max as the step graph runs them (csrc/gemm.cuh
 * EpiLmHead<true, false> -> finalize_step_kernel<true, false>, whatever `logits` holds): x [M,K] and W [V,K] as in
 * b200t5_test_lm_argmax; hist int64 [M, step+1] (device) the decoder ids so far (start token first), enc_ids int64
 * [M,S] (device) the prompts; eos is the EOS id when `logits` lists none.
 * tokens: int64 [M] (device); vals: fp32 [M,V] (device, may be NULL) the processed logits the arg-max ran on. Test hook;
 * both builds. */
int b200t5_test_lm_process(int device, const void* x, const void* W, int M, int V, int K, int step, int eos, int min_new,
                           const b200t5_logits_params* logits, const int64_t* hist, const int64_t* enc_ids, int S,
                           int64_t* tokens, float* vals, void* stream);
/* One decode step of a scored call as the step graph runs it (csrc/gemm.cuh EpiLmHead<kProc, true> ->
 * finalize_step_kernel<kProc, true>, kProc when `logits` has an active processor):
 * arguments as b200t5_test_lm_process, where `logits`, hist and enc_ids may be NULL (no processors); forced int64 [M]
 * (device, may be NULL) the tokens to take instead of the arg-max. tokens int64 [M], logprob and logit fp32 [M]
 * (device): the token taken, its log-probability and its processed score; vals as in b200t5_test_lm_process.
 * Test hook; both builds. */
int b200t5_test_lm_score(int device, const void* x, const void* W, int M, int V, int K, int step, int eos, int min_new,
                         const b200t5_logits_params* logits, const int64_t* hist, const int64_t* enc_ids, int S,
                         const int64_t* forced, int64_t* tokens, float* logprob, float* logit, float* vals, void* stream);

/* One beam step as the step graph runs it (csrc/beam.cuh: beam_row_kernel -> beam_select_kernel) on given fp32 logits
 * [B*k, V] (device) at decode position `step` of max_new_tokens T. In/out state (device): run_score fp32 [B*k]; fin
 * [B][16] records {float score; int32 t, par, tok; float lp; int32 flag} (a prompt's finished set, best first, k used);
 * heur int32 [B]. Out (device): lse fp32 [B*k]; cand_lp fp32 / cand_tok int32 [B*k][32] (each row's top 2k, best first);
 * parent int32 [B*k] (the row each row continues); token int32 [B*k]; retired int32 [B*k] (1: the row's prompt stopped).
 * Test hook; both builds. */
int b200t5_test_beam_step(int device, const float* logits, int B, int k, int V, int step, int T, int eos, int min_new,
                          double length_penalty, int early_stopping, float* run_score, void* fin, int32_t* heur, float* lse,
                          float* cand_lp, int32_t* cand_tok, int32_t* parent, int32_t* token, int32_t* retired, void* stream);
/* beam_reorder_kernel on a self-attention cache [planes][B*k][H][Tmax][64] of the build's 2-byte type (device): row r takes
 * positions 0..step of row parent[r] (int32 [B*k], device, within r's prompt). Test hook; both builds. */
int b200t5_test_beam_reorder(int device, void* kv, int planes, int B, int k, int H, int Tmax, int step, const int32_t* parent,
                             void* stream);
/* beam_replicate_kernel on a cross-attention K/V [planes][B*k][H][S][64] of the build's 2-byte type, extent int32 [B*k]
 * and key_ok uint8 [B*k][S] (device): rows b*k + j, j > 0, take the first extent[b*k] positions of row b*k, its extent and
 * its key_ok. Test hook; both builds. */
int b200t5_test_beam_replicate(int device, void* cross_kv, int32_t* extent, uint8_t* key_ok, int planes, int B, int k, int H, int S,
                               void* stream);
/* A whole beam search without the model, on the kernels the step graph runs: beam_init_kernel, then per step
 * beam_row_kernel -> beam_select_kernel on the fp32 logits [T][B*k][V] (device) of that step (rows of retired prompts
 * stop, as in b200t5_generate_beam; the search ends once every prompt has retired), then beam_output_kernel into io
 * (device pointers, layout of b200t5_beam_io with max_new_tokens T and num_return_sequences n). Out: steps (host) the
 * steps run; cand_lp fp32 / cand_tok int32 [T][B*k][32] (device, both NULL or neither) each live row's top 2k of each step,
 * as b200t5_test_beam_step; a retired row's entries are left as they were. Test hook; both builds. */
int b200t5_test_beam_search(int device, const float* logits, int B, int k, int V, int T, int eos, int min_new, double length_penalty,
                            int early_stopping, int n, int64_t start, int64_t pad, const b200t5_beam_io* io, int32_t* steps,
                            float* cand_lp, int32_t* cand_tok, void* stream);

/* ---- parity hooks (used by tests/ only) --------------------------------------------- */
/* Encoder last hidden state after the final RMSNorm, bf16 [B,S,d_model] (device). */
int b200t5_encode(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                  void* enc_out_bf16, void* stream);
/* Teacher-forced decode: decoder_input_ids int64 [B,T] (device) -> fp32 logits [B,T,vocab]
 * (device); logits are the bf16 lm_head outputs widened to fp32, as HF's `.float()` does. */
int b200t5_decode_logits(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                         const int64_t* decoder_input_ids, int T, float* logits, void* stream);
/* After a b200t5_generate_prefixed call with P >= 2 (and before any other call): decoder layer `layer`'s self-attention
 * cache at the prompt positions 0 .. P-2, as the prefill wrote it: kv_out [2][B][H][P-1][64] in the build's 2-byte
 * type (device), K then V. */
int b200t5_test_prefill_cache(b200t5_handle h, int layer, void* kv_out, void* stream);
/* T5Attention._relative_position_bucket for one offset (host-only, no GPU needed). */
int b200t5_relative_bucket(int relative_position, int bidirectional, int num_buckets, int max_distance);

/* Single-kernel hooks, in both builds: all pointers are device pointers. A 2-byte tensor is the build's activation
 * type (bf16 in libb200t5.so, fp16 in libb200t5_f16.so) unless noted. In the fp16 build the residual stream (the
 * residual C / R of the GEMMs, the RMSNorm input x) is fp32, and so is the GeGLU output (holding fp16 values). */
/* C[M,N] = act(A[M,K] W[N,K]^T) via the wgmma GEMM in one of the configurations the library launches:
 * bn = 512, the encoder configuration (128 x 256 tiles, weight in 128-row boxes) with mode 0 plain, 1 += residual R
 * (in C), 5 += residual as in decoder / encoder layer 0 (fp16 build: C = fp16(R + fp16(acc)), where mode 1 is
 * C = R + fp16(acc); bf16 build: same as 1), 2 GeGLU (W rows interleaved per 128, C is [M,N/2]), 6 ReLU
 * (C = relu(act(acc)) in the GeGLU output's type: the T5 v1.0 feed-forward input); or bn = 128 with mode 3, the fp32
 * logits of b200t5_decode_logits (C is float*), or mode 6, the ReLU product as the forward pass runs it (128 x 128
 * tiles). Anything else returns B200T5_EINVAL. pow_mode: the gelu table's (bf16 build; the fp16 build's epilogue has
 * no table). */
int b200t5_test_gemm(int device, const void* A, const void* W, void* C, int M, int N, int K, int bn, int mode,
                     int pow_mode, void* stream);
/* The 128 x 256 encoder GEMM as the encoder launches it; kernel 0 = the kernel whose epilogue follows each main loop,
 * 1 = the epilogue-overlapped kernel (option "enc_gemm"). mode 0 plain, 1 and 5 += residual R (in C), 2 GeGLU (W rows
 * interleaved per 128, C is [M,N/2]), 6 ReLU (as b200t5_test_gemm), 3 cross-attention K/V scatter: C is the arena [N/(H*64)][B][H][S][64] and row m
 * is position row_s[m] of prompt row_b[m] (both NULL: m = b*S + s, M = B*S). B, H, S are read in mode 3 only. */
int b200t5_test_enc_gemm(int device, const void* A, const void* W, void* C, int M, int N, int K, int kernel, int mode,
                         int pow_mode, const int* row_b, const int* row_s, int B, int H, int S, void* stream);
/* Same contract through the cluster split-K kernel the decode step uses (csrc/gemm_splitk.cuh):
 * bn in {64,128}; split in {1,2,4,8} CTAs per cluster along K (reduced automatically when K has
 * fewer 64-wide k-blocks); mode 0 plain, 1 and 5 += residual (in C), 2 GeGLU, 6 ReLU (as b200t5_test_gemm),
 * 4 decoder QKV: C is the q buffer [M, N/3] and `aux` the self-KV cache [2][M][H][Tmax][64] whose row `step` is
 * written. */
int b200t5_test_gemm_splitk(int device, const void* A, const void* W, void* C, int M, int N, int K, int bn, int split,
                            int mode, int pow_mode, void* aux, int Tmax, int step, void* stream);
/* fp16 build (libb200t5_f16.so) only: the fp32-weight feed-forward output projection (transformers keeps T5's `wo`
 * in fp32 under torch_dtype=float16), R += A . W^T computed as two tf32 tensor-core passes over W = W_hi + W_lo.
 * A [M,F] fp32 (fp16-representable values), W [N,F] fp32, R [M,N] fp32 in/out; kernel 0 = the encoder GEMM,
 * 1 = cluster split-K (decode; bn 64|128, split 1|2|4|8). The bf16 build returns B200T5_EINVAL. */
int b200t5_test_ffo(int device, const void* A, const void* W, void* R, int M, int N, int F, int kernel, int bn, int split,
                    void* stream);
int b200t5_test_rmsnorm(int device, const void* x, const void* w, void* y, int M, int d, float eps, void* stream);
/* The final decoder norm of a scale_decoder_outputs model: y = act(float(act(w * act(x * rsqrt(var + eps)))) * scale),
 * the last product in fp32 (scale = fp32(d_model ** -0.5) in the model). scale == 0 returns B200T5_EINVAL. */
int b200t5_test_rmsnorm_scaled(int device, const void* x, const void* w, void* y, int M, int d, float eps, float scale,
                               void* stream);
/* Decoder self-attention: self == 3 the 4-warp-per-(row, head) kernel the decode step runs; keys = t+1 with t = step, or, when extent is not NULL, t = extent[b] (int32 [B]: the
 * slot pool's per-row positions); dist_bias float [H][Tk]. Cross-attention: self == 0: extent int32 [B], key_ok uint8 [B][Tk];
 * self == 2: as 0 through the TMA stream kernel (csrc/attention_cross_stream.cuh), `step` = ring stages (0: 5);
 * same rounding points as self == 0, the fp32 accumulations in the tensor core's order. self == 1 returns
 * B200T5_EINVAL. */
int b200t5_test_attn_decode(int device, int self, const void* q, const void* K, const void* V, void* ctx, int B,
                            int H, int Tk, const int32_t* extent, const uint8_t* key_ok, int step,
                            const float* dist_bias, void* stream);
/* The mma.sync encoder attention; impl 0: rows b * S + i, impl 1: the packed-row addressing the encoder uses (row offsets
 * cu[b] = b * S), where query rows >= extent[b] are not written. */
int b200t5_test_encoder_attn(int device, const void* qkv, void* ctx, const float* rel_bias, const uint8_t* key_ok,
                             const int32_t* extent, int B, int S, int H, int impl, void* stream);
/* The decoder attentions of b200t5_forward (csrc/attention_decoder.cuh: decoder_attn_kernel), with the encoder attention's
 * rounding points. Self: qkv [B*T, 3*H*64] (q | k | v), causal, dist_bias float [H][T] indexed by i - j; T <= 4096.
 * Cross: q [B*T, H*64], kv [2][B][H][S][64] (one layer of the cross-K/V arena), keys masked by key_ok uint8 [B][S] and
 * extent int32 [B] (prep_mask's: a row without an attended key has extent S and attends uniformly). ctx [B*T, H*64]. */
int b200t5_test_decoder_self_attn(int device, const void* qkv, void* ctx, const float* dist_bias, int B, int T, int H,
                                  void* stream);
int b200t5_test_decoder_cross_attn(int device, const void* q, const void* kv, void* ctx, const uint8_t* key_ok,
                                   const int32_t* extent, int B, int T, int S, int H, void* stream);
/* The cross-attention of b200t5_forward_choices: q [qoff[B], H*64], prompt b's queries the rows qoff[b] .. qoff[b+1]-1
 * (qoff: DEVICE int32 [B+1], non-decreasing; read back for the grid), kv / key_ok / extent as above, ctx rows as q. */
int b200t5_test_decoder_cross_attn_packed(int device, const void* q, const void* kv, void* ctx, const uint8_t* key_ok,
                                          const int32_t* extent, const int32_t* qoff, int B, int S, int H, void* stream);
/* out[i] = act(gelu_new(gate[i]) * up[i]). mode 0: exactly the GeGLU epilogue's function (bf16 build: the exhaustive
 * gelu table; fp16 build: the op-by-op fp16 arithmetic with single-rounded pow); mode 2: the op-by-op arithmetic with
 * double-rounded pow (x*x*x in act_t); mode 1: same with single-rounded pow. */
int b200t5_test_geglu(int device, const void* gate, const void* up, void* out, int64_t n, int pow_mode,
                      void* stream);

const char* b200t5_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200T5_H_ */
