/*
 * b200t5.h - C ABI of libb200t5.so: FLAN-T5 (T5 v1.1, gated-GELU) greedy generation on one
 * NVIDIA H100 (sm_90a), the hot path of the workshop's batch-inference loop.
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
  int32_t is_gated_gelu;          /* must be 1 (feed_forward_proj == "gated-gelu") */
  int32_t scale_decoder_outputs;  /* must be 0 (tie_word_embeddings == false checkpoints) */
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
/* Checks that every required tensor arrived, repacks (QKV concat, GeGLU interleave, cross-KV concat). */
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
 * "xattn_stages" (8 KB ring stages per CTA), "xattn_late_pdl", "xattn_serialize", "xattn_l2pf", "pdl", "admit_overlap",
 * "sk_stages64", "sk_stages128" (pipeline stages of
 * the split-K decode GEMM tiles, 0 = default), "profile_xattn" (1 = every cross-attention launch inside the step graph
 * records %globaltimer stamps; never on in a timed region), "enc_gemm" (the 128 x 256 encoder GEMMs: 1 = default,
 * epilogue warps drain each tile while the next tile's MMAs run; 0 = the kernel whose epilogue follows each main loop;
 * bit-identical results; environment variable B200T5_ENC_GEMM at create time). */
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

/* ---- parity hooks (used by tests/ only) --------------------------------------------- */
/* Encoder last hidden state after the final RMSNorm, bf16 [B,S,d_model] (device). */
int b200t5_encode(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                  void* enc_out_bf16, void* stream);
/* Teacher-forced decode: decoder_input_ids int64 [B,T] (device) -> fp32 logits [B,T,vocab]
 * (device); logits are the bf16 lm_head outputs widened to fp32, as HF's `.float()` does. */
int b200t5_decode_logits(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                         const int64_t* decoder_input_ids, int T, float* logits, void* stream);
/* T5Attention._relative_position_bucket for one offset (host-only, no GPU needed). */
int b200t5_relative_bucket(int relative_position, int bidirectional, int num_buckets, int max_distance);

/* Single-kernel hooks, in both builds: all pointers are device pointers. A 2-byte tensor is the build's activation
 * type (bf16 in libb200t5.so, fp16 in libb200t5_f16.so) unless noted. In the fp16 build the residual stream (the
 * residual C / R of the GEMMs, the RMSNorm input x) is fp32, and so is the GeGLU output (holding fp16 values). */
/* C[M,N] = act(A[M,K] W[N,K]^T) via the wgmma GEMM; mode 0 plain, 1 += residual R (in C), 5 += residual as in
 * decoder / encoder layer 0 (fp16 build: C = fp16(R + fp16(acc)), where mode 1 is C = R + fp16(acc); bf16 build:
 * same as 1), 2 GeGLU (W rows interleaved per bn/2, C is [M,N/2]), 3 fp32 output (C is float*). bn in {32,64,128,256};
 * bn = 512 selects the encoder configuration (128 x 256 tiles, weight in 128-row boxes, GeGLU interleave per 128),
 * modes 0, 1, 2, 5. pow_mode: the gelu table's (bf16 build; the fp16 build's epilogue has no table). */
int b200t5_test_gemm(int device, const void* A, const void* W, void* C, int M, int N, int K, int bn, int mode,
                     int pow_mode, void* stream);
/* The 128 x 256 encoder GEMM as the encoder launches it; kernel 0 = the kernel whose epilogue follows each main loop,
 * 1 = the epilogue-overlapped kernel (option "enc_gemm"). mode 0 plain, 1 and 5 += residual R (in C), 2 GeGLU (W rows
 * interleaved per 128, C is [M,N/2]), 3 cross-attention K/V scatter: C is the arena [N/(H*64)][B][H][S][64] and row m
 * is position row_s[m] of prompt row_b[m] (both NULL: m = b*S + s, M = B*S). B, H, S are read in mode 3 only. */
int b200t5_test_enc_gemm(int device, const void* A, const void* W, void* C, int M, int N, int K, int kernel, int mode,
                         int pow_mode, const int* row_b, const int* row_s, int B, int H, int S, void* stream);
/* Same contract through the cluster split-K kernel the decode step uses (csrc/gemm_splitk.cuh):
 * bn in {64,128}; split in {1,2,4,8} CTAs per cluster along K (reduced automatically when K has
 * fewer 64-wide k-blocks); mode 0 plain, 1 and 5 += residual (in C), 2 GeGLU, 4 decoder QKV: C is the q
 * buffer [M, N/3] and `aux` the self-KV cache [2][M][H][Tmax][64] whose row `step` is written. */
int b200t5_test_gemm_splitk(int device, const void* A, const void* W, void* C, int M, int N, int K, int bn, int split,
                            int mode, int pow_mode, void* aux, int Tmax, int step, void* stream);
/* fp16 build (libb200t5_f16.so) only: the fp32-weight feed-forward output projection (transformers keeps T5's `wo`
 * in fp32 under torch_dtype=float16), R += A . W^T computed as two tf32 tensor-core passes over W = W_hi + W_lo.
 * A [M,F] fp32 (fp16-representable values), W [N,F] fp32, R [M,N] fp32 in/out; kernel 0 = the encoder GEMM,
 * 1 = cluster split-K (decode; bn 64|128, split 1|2|4|8). The bf16 build returns B200T5_EINVAL. */
int b200t5_test_ffo(int device, const void* A, const void* W, void* R, int M, int N, int F, int kernel, int bn, int split,
                    void* stream);
int b200t5_test_rmsnorm(int device, const void* x, const void* w, void* y, int M, int d, float eps, void* stream);
/* Decoder self-attention: self == 3 the 4-warp-per-(row, head) kernel the decode step runs, self == 1 the one-warp
 * variant (B200T5_SELF=warp); keys = t+1 with t = step, or, when extent is not NULL, t = extent[b] (int32 [B]: the
 * slot pool's per-row positions); dist_bias float [H][Tk]. Cross-attention: self == 0: extent int32 [B], key_ok uint8 [B][Tk];
 * self == 2: as 0 through the TMA stream kernel (csrc/attention_cross_stream.cuh), `step` = ring stages (0: 5);
 * same rounding points as self == 0, the fp32 accumulations in the tensor core's order. */
int b200t5_test_attn_decode(int device, int self, const void* q, const void* K, const void* V, void* ctx, int B,
                            int H, int Tk, const int32_t* extent, const uint8_t* key_ok, int step,
                            const float* dist_bias, void* stream);
/* The mma.sync encoder attention; impl 0: rows b * S + i, impl 1: the packed-row addressing the encoder uses (row offsets
 * cu[b] = b * S), where query rows >= extent[b] are not written. */
int b200t5_test_encoder_attn(int device, const void* qkv, void* ctx, const float* rel_bias, const uint8_t* key_ok,
                             const int32_t* extent, int B, int S, int H, int impl, void* stream);
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
