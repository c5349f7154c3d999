// libb200t5.so - C ABI (include/b200t5.h) over the sm_90a (H100) kernels in this directory.
// Host side: weight store + repacking, per-shape execution plans (workspace, TMA tensor
// maps, KV arenas, the CUDA graph of one decode step), the greedy loop.
//
// Reference path being replaced: HuggingFaceModelPredictor._predict_numpy ->
// model.generate() (NLP_workloads/Anyscale_job/predictor.py:97-102), whose arithmetic is
// transformers' T5ForConditionalGeneration + GenerationMixin._sample (greedy).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <optional>
#include <string>
#include <vector>

#include "../../include/b200t5.h"
#include "attention_decode.cuh"
#include "attention_cross_stream.cuh"
#include "attention_encoder.cuh"
#include "attention_decoder.cuh"
#include "beam.cuh"
#include "elementwise.cuh"
#include "gemm.cuh"
#include "gemm_splitk.cuh"
#include "gemm_2cta.cuh"

using namespace b200;

// ================================================================== error plumbing
static thread_local char g_err[512] = "";
static void set_gerr(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

struct b200t5_ctx;
static int fail(b200t5_ctx* h, int code, const char* fmt, ...);

#define CU_OK(h, expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return fail(h, B200T5_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// ================================================================== TMA tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}
// row-major [rows, cols] (cols contiguous) of 2-byte activations / weights, or (f32) of fp32 values for the tf32
// products of the fp16 build; box = 128 bytes of columns x box_rows rows, 128-B swizzle.
static bool make_tmap(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, bool f32 = false) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) {
    set_gerr("cuTensorMapEncodeTiled entry point not available");
    return false;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * (f32 ? 4u : 2u)};
  cuuint32_t box[2] = {f32 ? 32u : 64u, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                     : (B200T5_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  CUresult r = enc(tm, dt, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_gerr("cuTensorMapEncodeTiled failed with %d (rows=%llu cols=%llu box_rows=%u base=%p)", (int)r,
             (unsigned long long)rows, (unsigned long long)cols, box_rows, base);
    return false;
  }
  return true;
}

// ================================================================== small device helpers
DEVINL float load_as_float(const void* src, int dtype, size_t i) {
  if (dtype == B200T5_DTYPE_F32) return reinterpret_cast<const float*>(src)[i];
  if (dtype == B200T5_DTYPE_F16) return __half2float(reinterpret_cast<const __half*>(src)[i]);
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(src)[i]);
}
__global__ void convert_to_act_kernel(const void* src, int dtype, act_t* dst, size_t n) {
  size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) dst[i] = float2act(load_as_float(src, dtype, i));
}
#if B200T5_F16
// `wo` stays an fp32 weight (transformers' _keep_in_fp32_modules = ["wo"] under torch_dtype=float16)
__global__ void convert_to_f32_kernel(const void* src, int dtype, float* dst, size_t n) {
  size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) dst[i] = load_as_float(src, dtype, i);
}
// W [rows, K] fp32 -> W' [rows, 2*Kp] = [W_hi | W_lo], Kp = K rounded up to the 32-element k-block, both pieces
// exactly representable in tf32 (low 13 mantissa bits clear): W_hi = tf32_rn(W), W_lo = tf32_rn(W - W_hi) (the
// subtraction is exact), so A . W_hi^T + A . W_lo^T with fp32 accumulation carries ~22 of W's 24 significand bits.
DEVINL float tf32_rn(float x) {
  uint32_t u = __float_as_uint(x);
  u += 0x0FFFu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xFFFFE000u);
}
__global__ void split_tf32_kernel(const float* __restrict__ w, float* __restrict__ out, int rows, int K, int Kp) {
  size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t n = static_cast<size_t>(rows) * Kp;
  if (i >= n) return;
  const int r = static_cast<int>(i / Kp), k = static_cast<int>(i % Kp);
  const float v = k < K ? w[static_cast<size_t>(r) * K + k] : 0.f;
  const float hi = tf32_rn(v);
  out[static_cast<size_t>(r) * 2 * Kp + k] = hi;
  out[static_cast<size_t>(r) * 2 * Kp + Kp + k] = tf32_rn(v - hi);
}
#endif
// mode 0: the GeGLU epilogue's function (gemm.cuh gelu_epilogue); 1/2: op-by-op arithmetic with pow_mode 1/0
__global__ void geglu_elementwise_kernel(const act_t* gate, const act_t* up, act_t* out, long long n, int mode, GeluLut lut) {
  long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const float x = act2float(gate[i]);
  const float g = mode == 0 ? gelu_epilogue(x, lut.table, lut.lo, lut.hi) : gelu_new_act_exact(x, mode == 1 ? 1 : 0);
  out[i] = float2act(g * act2float(up[i]));
}
__global__ void build_gelu_table_kernel(uint16_t* full, int pow_mode) {
  const uint32_t bits = blockIdx.x * blockDim.x + threadIdx.x;  // every bf16 bit pattern
  if (bits >= 65536u) return;
  const float g = gelu_new_act_exact(__uint_as_float(bits << 16), pow_mode);
  full[bits] = static_cast<uint16_t>(__float_as_uint(g) >> 16);
}
__global__ void set_state_kernel(DecodeState* st, int step) {
  st->step = step;
  st->finished_rows = 0;
}

// ================================================================== model description
struct Cfg {
  int V, d, F, H, I, Le, Ld, nb, maxdist;
  float eps;
  int pad, eos, start;
  bool gated;       // feed-forward: gated-GELU (T5 v1.1 / FLAN-T5), else ReLU (T5 v1.0)
  float out_scale;  // scale_decoder_outputs: fp32(d_model ** -0.5) after the final decoder norm; 0 = none
};

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) {
    o.p = nullptr;
    o.bytes = 0;
  }
  cudaError_t alloc(size_t n) {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = n;
    return cudaMalloc(&p, n ? n : 16);
  }
  template <class T>
  T* as() const {
    return reinterpret_cast<T*>(p);
  }
};

struct EncLayerW {
  DevBuf ln0, ln1, wqkv, wo, wi, wff_o;  // wi interleaved for BN=256
  CUtensorMap tm_qkv, tm_o, tm_wi, tm_ffo;  // box of 128 weight rows: a 256-wide weight tile is loaded as two boxes
};
struct DecLayerW {
  DevBuf ln0, ln1, ln2, wqkv, wo, wcq, wco, wi, wff_o;  // wi interleaved per N-tile of the decode wi GEMM
  CUtensorMap tm_qkv, tm_o, tm_cq, tm_co, tm_wi, tm_ffo;
  // the same weights in boxes of 128 rows, for the 128 x 256 GEMMs of the forward pass (b200t5_forward)
  CUtensorMap tm2_qkv, tm2_o, tm2_cq, tm2_co, tm2_ffo;
  int wi_rows = 0;
};

constexpr int kMaxChains = 8;
constexpr int kStepsPerGraph = 8;

// Host form of a call's logits processors (b200t5_logits_params after validation; logits_process.cuh).
struct ProcHost {
  bool on = false;
  ProcCfg cfg{};
  std::vector<uint32_t> stat;        // [3][W]: suppressed + one-token bad words, begin-suppressed, EOS ids
  std::vector<int> bad_ids, bad_off;  // bad words of two or more tokens
};

// Device state of the processors for `rows` rows (logits_process.cuh: ProcDev). The step graph bakes these
// addresses: a reallocation means a new graph.
// Host form of a call's scoring request (b200t5_score_io after validation). `forced`: the labels padded with -100 to
// [rows, max_new_tokens], as the step kernels read them.
struct ScoreHost {
  bool on = false;
  std::vector<long long> forced;
};

struct ProcBufs {
  DevBuf cfg, seen, enc, banned, stat, list, cnt, enc_ids, bad_ids, bad_off;
  int rows = 0, S = 0, W = 0, ban_cap = 0;
  size_t n_bad_ids = 0, n_bad_off = 0;
  bool fits(int r, int s, int w, int cap, size_t nbi, size_t nbo) const {
    return cfg.p && rows == r && S == s && W == w && ban_cap >= cap && n_bad_ids >= nbi && n_bad_off >= nbo;
  }
  cudaError_t alloc(int r, int s, int w, int cap, size_t nbi, size_t nbo) {
    rows = r;
    S = s;
    W = w;
    ban_cap = cap;
    n_bad_ids = nbi;
    n_bad_off = nbo;
    const size_t bm = static_cast<size_t>(r) * w * 4;
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = cfg.alloc(sizeof(ProcCfg));
    if (e == cudaSuccess) e = seen.alloc(bm);
    if (e == cudaSuccess) e = enc.alloc(bm);
    if (e == cudaSuccess) e = banned.alloc(bm);
    if (e == cudaSuccess) e = stat.alloc(static_cast<size_t>(3) * w * 4);
    if (e == cudaSuccess) e = list.alloc(static_cast<size_t>(r) * cap * 4);
    if (e == cudaSuccess) e = cnt.alloc(static_cast<size_t>(r) * 4);
    if (e == cudaSuccess) e = enc_ids.alloc(static_cast<size_t>(r) * s * 4);
    if (e == cudaSuccess) e = bad_ids.alloc(nbi * 4);
    if (e == cudaSuccess) e = bad_off.alloc(nbo * 4);
    if (e != cudaSuccess && cfg.p) {  // fits() is false until a complete allocation
      cudaFree(cfg.p);
      cfg.p = nullptr;
    }
    return e;
  }
  ProcDev dev(int row0 = 0) const {
    ProcDev d;
    d.cfg = cfg.as<ProcCfg>();
    d.seen = seen.as<uint32_t>();
    d.enc = enc.as<uint32_t>();
    d.banned = banned.as<uint32_t>();
    d.stat = stat.as<uint32_t>();
    d.ban_list = list.as<int>();
    d.ban_cnt = cnt.as<int>();
    d.enc_ids = enc_ids.as<int>();
    d.bad_ids = bad_ids.as<int>();
    d.bad_off = bad_off.as<int>();
    d.ban_cap = ban_cap;
    d.S = S;
    d.W = W;
    d.row0 = row0;
    return d;
  }
  // a call's values; pageable sources: each copy has left the host buffer when it returns
  cudaError_t upload(const ProcHost& ph, cudaStream_t s) {
    cudaError_t e = cudaMemcpyAsync(cfg.p, &ph.cfg, sizeof(ProcCfg), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(stat.p, ph.stat.data(), ph.stat.size() * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && !ph.bad_ids.empty())
      e = cudaMemcpyAsync(bad_ids.p, ph.bad_ids.data(), ph.bad_ids.size() * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && !ph.bad_off.empty())
      e = cudaMemcpyAsync(bad_off.p, ph.bad_off.data(), ph.bad_off.size() * 4, cudaMemcpyHostToDevice, s);
    return e;
  }
};

// Beam-search state of a plan (beam.cuh), allocated by the first beam call. The step graph bakes these addresses.
// seq / len / score / bidx / lp: the host entry point's results, written by beam_output_kernel and copied to the caller.
struct BeamBufs {
  DevBuf logits, cand_lp, cand_tok, run_score, hist_par, hist_tok, hist_lp, fin, heur, parent, prm, len_scale, moved;
  DevBuf seq, len, score, bidx, lp;
  BeamDev dev(int rows) const {
    return BeamDev{prm.as<BeamParams>(), len_scale.as<float>(), logits.as<float>(), nullptr, cand_lp.as<float>(), cand_tok.as<int>(),
                   run_score.as<float>(), hist_par.as<int>(), hist_tok.as<int>(), hist_lp.as<float>(), fin.as<BeamFin>(), heur.as<int>(),
                   parent.as<int>(), rows};
  }
};

// What the step graph bakes in besides buffer addresses (the values of processors, labels and beam parameters are read
// from device memory at replay). A call whose mode differs from the one the graph was captured for re-captures it.
struct StepMode {
  long long eos = -1, pad = -1;
  int min_new = 0;
  bool pool = false;  // slot pool: per-slot positions and the pool's results; else one position for a static batch
  bool proc = false;  // logits processors: EpiLmHead<true, *>
  int score = 0;      // 0 plain head, 1 EpiLmHead<*, true> + finalize_step_kernel<*, true>, 2 those with teacher forcing
  int beam = 0;       // k > 0: the beam head (lm_head -> fp32 logits -> beam.cuh)
  bool xattn_stream = false;  // cross-attention kernel: the TMA stream kernel, else the per-thread-load kernel
  bool operator==(const StepMode& o) const {
    return eos == o.eos && pad == o.pad && min_new == o.min_new && pool == o.pool && proc == o.proc && score == o.score &&
           beam == o.beam && xattn_stream == o.xattn_stream;
  }
};

struct Plan {
  int B = 0, S = 0, Tmax = 0;
  int group = 1;  // rows per prompt (num_beams): the row-chains split on prompt boundaries
  int ws_S = 0;   // rows per prompt of the encoder workspace: S, or the forward pass's T when that is longer
  // encoder workspace, and the forward pass's decoder workspace once the cross-K/V projection has run
  DevBuf x, xn, qkv, ctx, hff;          // [B*ws_S, d], [B*ws_S, d], [B*ws_S, 3I], [B*ws_S, I], [B*ws_S, F]
  DevBuf key_ok, extent, enc_bias;      // uint8 [B,S], int [B], float [H][2S-1]
  DevBuf cu, row_b, row_s;              // packed encoder rows: int [B+1] offsets, int [B*S] row -> (prompt, position)
  int* h_cu = nullptr;                  // pinned copy of cu[B] (number of packed rows)
  int packed_rows = 0;                  // rows the last encoder pass ran on
  bool packed = false;
  DevBuf cross_kv;                      // [Ld][2][B][H][S][64]
  // decoder workspace
  DevBuf dx, dxn, dq, dctx, dh;         // [B,d], [B,d], [B,I], [B,I], [B,F]
  DevBuf self_kv;                       // [Ld][2][B][H][Tmax][64]
  DevBuf dec_bias;                      // float [H][Tmax]
  DevBuf pval, pidx;                    // [B][n_tiles]
  DevBuf state, unfinished, ids_dev, mask_dev;
  // what the decode kernels attend to: copies of extent / key_ok in which a finished row's extent drops to 0
  // (retired: its K/V are no longer streamed). In slot-pool mode they describe the slots' CURRENT prompts while
  // extent / key_ok describe the prompts of the encoder pass being admitted.
  DevBuf live_extent, live_key_ok;
  DevBuf xs_stamps, xs_acc;  // in-situ profile of the cross-attention launches: [Ld * chains][2] stamps / {ns, launches}, then [Ld][2] {busy ns, layers}
  // slot pool (b200t5_generate_stream): per-slot position and result row, admission lists
  DevBuf pos, out_row, admit;
  // A call's results, by row: ids [cap][Tmax+1] and lengths [cap]; for a scored call (allocated by the first one)
  // log-probabilities and processed scores [cap][Tmax], and the labels [cap][Tmax] of a teacher-forced one. `batch`
  // holds the static batch's B rows, `pool` the slot pool's N rows in input order (cap >= N: it only grows). The step
  // graph bakes these addresses: a reallocation drops it.
  struct Results {
    DevBuf ids, len, lp, lg, forced;
    size_t cap = 0;
  };
  Results batch, pool;
  Results& res() { return mode.pool ? pool : batch; }
  ProcBufs proc;                 // logits processors (allocated by the first call that uses them)
  DevBuf psum, fval, ftok;       // token log-probabilities (likewise): [B][n_tiles], [B], [B]
  BeamBufs beam;
  // the forward pass (b200t5_forward), allocated by its first call: the decoder ids int64 [B*T], the label columns
  // int32 [B*T] and a zero step; the causal bias float [H][fwd_T]; the lm_head partials when they do not fit in hff
  DevBuf fwd_ids, fwd_bias, fwd_part;
  int fwd_T = 0;
  // a call with a decoder prompt (b200t5_generate_prefixed): the prefill's ids int64 [B*(P-1)], then the prompt [B*P];
  // prompt_steps = P - 1 of the last such call (0 for any other call)
  DevBuf pre_ids;
  int prompt_steps = 0;
  StepMode mode;                 // what this call's steps run
  std::optional<StepMode> graph_mode;  // what the step graphs were captured for (none: re-capture)
  // after a reallocation of a buffer the step graph bakes: the next ensure_graph re-captures
  void invalidate_graph() { graph_mode.reset(); }
  long long rows_valid = 0;   // valid prompt tokens of the last encoder pass (packed rows)
  int* h_unf = nullptr;    // pinned: unfinished[B] read back every graph launch
  int* h_admit = nullptr;  // pinned: [3][B] = row_on flags, slots, rows
  int n_vtiles = 0;
  // tensor maps for activations (A operands)
  CUtensorMap tm_xn, tm_ctx, tm_hff;
  CUtensorMap tm_cross_kv;  // [Ld*2*B*H*S, 64] view of the cross-KV arena, box 64 x 64 keys (attention_cross_stream.cuh)
  // decode chains: the batch is cut into independent row ranges that run concurrently (one
  // stream each inside the step graph); every chain sees pointer-offset views of the same buffers
  struct Chain {
    int b0 = 0, nb = 0;
    CUtensorMap tm_dxn, tm_dctx, tm_dh;
  };
  int n_chains = 1;
  Chain chains[kMaxChains];
  // decode-step graph
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t gexec = nullptr;
  int graph_nodes = 0;
  // the same step captured kStepsPerGraph times back to back: one launch per 8 decode steps (= the poll interval)
  cudaGraph_t graph8 = nullptr;
  cudaGraphExec_t gexec8 = nullptr;
  // pinned staging for the host-buffer entry point and polling
  long long* h_ids = nullptr;
  long long* h_mask = nullptr;
  long long* h_out = nullptr;
  int* h_len = nullptr;
  DecodeState* h_state = nullptr;
  ~Plan() {
    if (gexec) cudaGraphExecDestroy(gexec);
    if (graph) cudaGraphDestroy(graph);
    if (gexec8) cudaGraphExecDestroy(gexec8);
    if (graph8) cudaGraphDestroy(graph8);
    if (h_ids) cudaFreeHost(h_ids);
    if (h_mask) cudaFreeHost(h_mask);
    if (h_out) cudaFreeHost(h_out);
    if (h_len) cudaFreeHost(h_len);
    if (h_state) cudaFreeHost(h_state);
    if (h_cu) cudaFreeHost(h_cu);
    if (h_unf) cudaFreeHost(h_unf);
    if (h_admit) cudaFreeHost(h_admit);
  }
};

struct b200t5_ctx {
  Cfg c;
  int device = 0;
  int num_sms = 132;
  bool finalized = false;
  int ffo_k = 0;  // K extent of the feed-forward output weight as stored (F, or 2 * round_up(F, 32) in the fp16 build)
  char err[512] = "";
  std::map<std::string, std::unique_ptr<DevBuf>> raw;  // HF name -> act_t copy (until finalize)
  std::map<std::string, std::unique_ptr<DevBuf>> raw_f32;  // fp16 build: fp32 copies of the `wo` weights
  std::map<std::string, std::vector<int64_t>> raw_shape;
  DevBuf shared, lm_head, enc_final_ln, dec_final_ln, enc_relbias, dec_relbias, wcrosskv;
  CUtensorMap tm_lm, tm_crosskv;
  std::vector<float> enc_relbias_h, dec_relbias_h;  // [nb][H] as float
  std::vector<EncLayerW> enc;
  std::vector<DecLayerW> dec;
  std::unique_ptr<Plan> plan;
  cudaStream_t cap_stream = nullptr, exec_stream = nullptr, enc_stream = nullptr;  // enc_stream: slot-pool admission encoder passes (lowest priority)
  cudaEvent_t enc_done_ev = nullptr, admitted_ev = nullptr;
  bool admit_overlap = true;  // B200T5_ADMIT_OVERLAP=0: admission encoder passes on the decode stream (round-1 behaviour)
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  bool ev_valid = false;
  bool use_pdl = true;
  GeluLut gelu_lut{nullptr, 0, 0};
  // decode GEMMs: cluster split-K tiles (gemm_splitk.cuh). {BN, wanted split} per product;
  // B200T5_SK="bn,s,bn,s,bn,s,bn,s" overrides (order: qkv, attention projections o/cq/co, wi, ffo).
  struct SkChoice {
    int bn, split;
  };
  // 128 x 256 encoder GEMMs through gemm_enc_ws_kernel (epilogue warps overlap the next tile's main loop) rather than
  // gemm_bf16_tn_kernel; bit-identical results. B200T5_ENC_GEMM, option "enc_gemm" 0|1.
  bool enc_gemm_ws = true;
  // Cross-attention of the decode step: the TMA-ring + mma.sync stream kernel (attention_cross_stream.cuh: small
  // footprint, shares the SMs with the other chain's GEMM CTAs; meant for batches whose prompts fill the window) or the
  // per-thread-load kernel (attention_decode.cuh: one short-lived CTA per (row, head), several per SM; meant for
  // ragged prompts). 2 = choose per call from
  // the batch's fill (valid prompt tokens / B*S >= kXattnStreamFill -> stream); B200T5_XATTN=ldg|stream|auto, option
  // "xattn" 0|1|2. The kernels differ only in the order of their fp32 accumulations (same tokens up to near-ties).
  int xattn_mode = 2;
  int xs_stages = 5;        // 8 KB ring stages per CTA (two CTAs per SM): B200T5_XS_STAGES
  bool profile_xattn = false;  // b200t5_set_option("profile_xattn"): stamp every cross-attention launch inside the step graph
  int sk_stages64 = 0, sk_stages128 = 0;  // pipeline stages of the split-K tiles (0 = default 4 / 3): B200T5_SK_STAGES="a,b"
  SkChoice sk_qkv{64, 2}, sk_proj{64, 4}, sk_wi{128, 2}, sk_ffo{64, 4};  // split-K choices per product (tools/sweep_decode.py)
  int chains_override = 0;
  cudaStream_t chain_streams[kMaxChains] = {};
  cudaEvent_t chain_ev[kMaxChains + 1] = {};
  // stats of the last generate
  int64_t launches = 0;
  int last_steps = 0;
  double last_decode_bytes = 0, last_enc_flops = 0;
};

static int fail(b200t5_ctx* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) snprintf(h->err, sizeof(h->err), "%s", buf);
  snprintf(g_err, sizeof(g_err), "%s", buf);
  return code;
}

static int check_device(b200t5_ctx* h, int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0)
    return fail(h, B200T5_ENODEV, "no CUDA device available (%s); libb200t5 has no CPU fallback",
                e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(h, B200T5_EINVAL, "device %d out of range (%d devices)", device, n);
  cudaDeviceProp p;
  CU_OK(h, cudaGetDeviceProperties(&p, device));
  if (p.major != 9)
    return fail(h, B200T5_ENODEV, "device %d is sm_%d%d; libb200t5 is built for sm_90a only", device, p.major, p.minor);
  CU_OK(h, cudaSetDevice(device));
  return p.multiProcessorCount;
}

// ================================================================== relative position buckets
// T5Attention._relative_position_bucket (modeling_t5.py:188-234), fp32 log + truncation.
extern "C" int b200t5_relative_bucket(int rel, int bidirectional, int num_buckets, int max_distance) {
  int ret = 0, n;
  if (bidirectional) {
    num_buckets /= 2;
    if (rel > 0) ret += num_buckets;
    n = rel < 0 ? -rel : rel;
  } else {
    n = rel < 0 ? -rel : 0;
  }
  const int max_exact = num_buckets / 2;
  if (n < max_exact) return ret + n;
  const float ratio = static_cast<float>(n) / static_cast<float>(max_exact);
  const float denom = static_cast<float>(log(static_cast<double>(max_distance) / static_cast<double>(max_exact)));
  const float scaled = logf(ratio) / denom * static_cast<float>(num_buckets - max_exact);
  int large = max_exact + static_cast<int>(scaled);
  if (large > num_buckets - 1) large = num_buckets - 1;
  return ret + large;
}

// ================================================================== GEMM dispatch
// The decode step's head, indexed [kProc][kScore]: the lm_head GEMM with its fused epilogue (gemm.cuh: EpiLmHead) and
// the kernel that merges the epilogue's partials (elementwise.cuh: finalize_step_kernel).
struct LmHead {
  cudaError_t (*gemm)(const CUtensorMap&, const CUtensorMap&, int, int, int, int, const LmHeadParams&, int, cudaStream_t, bool, int);
  void (*finalize)(FinalizeArgs);
  cudaError_t (*prepare)();
};
template <bool kProc, bool kScore>
constexpr LmHead lm_head_of() {
  return {launch_gemm<128, EpiLmHead<kProc, kScore>>, finalize_step_kernel<kProc, kScore>, prepare_gemm<128, EpiLmHead<kProc, kScore>>};
}
static const LmHead kLmHeads[2][2] = {{lm_head_of<false, false>(), lm_head_of<false, true>()},
                                      {lm_head_of<true, false>(), lm_head_of<true, true>()}};

// the head of M rows x N columns: tmA holds the rows' normalised activations [M, K], tmB the lm_head weight [N, K]
static cudaError_t run_lm_head(b200t5_ctx* h, bool proc, bool score, const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N,
                               int K, const LmHeadParams& ep, const FinalizeArgs& fa, cudaStream_t s, bool pdl) {
  const LmHead& lh = kLmHeads[proc][score];
  h->launches += 2;
  cudaError_t e = lh.gemm(tmA, tmB, M, N, K, 1, ep, h->num_sms, s, pdl, 0);
  if (e == cudaSuccess) e = launch_kernel(lh.finalize, dim3(M), dim3(128), 0, s, pdl, fa);
  return e;
}

// encoder GEMM, 128 x 256 tiles (gemm_2cta.cuh)
template <class Epi>
static cudaError_t run_gemm_2cta(b200t5_ctx* h, const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K,
                                 const typename Epi::Params& ep, cudaStream_t s) {
  h->launches++;
  if (h->enc_gemm_ws) return launch_gemm_enc_ws<Epi>(tmA, tmB, M, N, K, ep, h->num_sms, s);
  return launch_gemm_2cta<Epi>(tmA, tmB, M, N, K, ep, h->num_sms, s);
}

// split-K cluster GEMM (decode): Epi chosen by the caller, BN/split from the handle's choice
template <class Epi>
static cudaError_t run_gemm_sk(b200t5_ctx* h, const b200t5_ctx::SkChoice& ch, const CUtensorMap& tmA,
                               const CUtensorMap& tmB, int M, int N, int K, const typename Epi::Params& ep,
                               cudaStream_t s, bool pdl) {
  h->launches++;
  const int split = splitk_factor(K, ch.split);
  if (ch.bn == 128) return launch_gemm_splitk<128, Epi>(tmA, tmB, M, N, K, split, ep, s, pdl, 0, h->sk_stages128);
  return launch_gemm_splitk<64, Epi>(tmA, tmB, M, N, K, split, ep, s, pdl, 0, h->sk_stages64);
}

// Feed-forward output projection + residual. bf16 build: an ordinary 2-byte product. fp16 build: fp32 weight and
// fp32 output (HF keeps `wo` in fp32), computed as two tf32 passes over W' = [W_hi | W_lo] with the fp32 A operand
// (the GeGLU output) walked twice.
static cudaError_t run_ffo_2cta(b200t5_ctx* h, const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N,
                                const EpiResidual::Params& ep, cudaStream_t s) {
  h->launches++;
  if (!B200T5_F16 && h->enc_gemm_ws) return launch_gemm_enc_ws<EpiResidual>(tmA, tmB, M, N, h->ffo_k, ep, h->num_sms, s);
  return launch_gemm_2cta<EpiResidual, B200T5_F16 != 0>(tmA, tmB, M, N, h->ffo_k, ep, h->num_sms, s, B200T5_F16 ? h->ffo_k / 64 : 0);
}
static cudaError_t run_ffo_sk(b200t5_ctx* h, const b200t5_ctx::SkChoice& ch, const CUtensorMap& tmA, const CUtensorMap& tmB,
                              int M, int N, const EpiResidual::Params& ep, cudaStream_t s, bool pdl) {
  h->launches++;
  constexpr bool tf = B200T5_F16 != 0;
  const int split = splitk_factor(h->ffo_k, ch.split, tf ? kBK / 2 : kBK);
  const int akb = tf ? h->ffo_k / 64 : 0;
  if (ch.bn == 128) return launch_gemm_splitk<128, EpiResidual, tf>(tmA, tmB, M, N, h->ffo_k, split, ep, s, pdl, akb, h->sk_stages128);
  return launch_gemm_splitk<64, EpiResidual, tf>(tmA, tmB, M, N, h->ffo_k, split, ep, s, pdl, akb, h->sk_stages64);
}

// scale != 0: the rescaled final decoder norm of a T5 v1.0 checkpoint (rmsnorm_scaled_kernel), same launch shape
static cudaError_t run_rmsnorm(b200t5_ctx* h, const res_t* x, const act_t* w, act_t* y, int M, int d, float eps,
                               cudaStream_t s, bool pdl = false, float scale = 0.f) {
  if (h) h->launches++;
  const int wpb = 8;
  const int grid = (M + wpb - 1) / wpb;
  if (scale != 0.f) {
    if (d <= 1024) return launch_kernel(rmsnorm_scaled_kernel<4>, dim3(grid), dim3(wpb * 32), 0, s, pdl, x, w, y, M, d, eps, scale);
    if (d <= 4096) return launch_kernel(rmsnorm_scaled_kernel<16>, dim3(grid), dim3(wpb * 32), 0, s, pdl, x, w, y, M, d, eps, scale);
    return cudaErrorInvalidValue;
  }
  if (d <= 1024) return launch_kernel(rmsnorm_kernel<4>, dim3(grid), dim3(wpb * 32), 0, s, pdl, x, w, y, M, d, eps);
  if (d <= 4096) return launch_kernel(rmsnorm_kernel<16>, dim3(grid), dim3(wpb * 32), 0, s, pdl, x, w, y, M, d, eps);
  return cudaErrorInvalidValue;
}

static cudaError_t init_kernel_attrs() {
  cudaError_t e;
  if ((e = prepare_gemm<128, EpiStoreF32>()) != cudaSuccess) return e;
  for (const auto& row : kLmHeads)
    for (const LmHead& lh : row)
      if ((e = lh.prepare()) != cudaSuccess) return e;
  if ((e = prepare_gemm_2cta<EpiStore>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_2cta<EpiResidual>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_2cta<EpiGeglu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_2cta<EpiCrossKV>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_enc_ws<EpiStore>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_enc_ws<EpiResidual>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_enc_ws<EpiGeglu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_enc_ws<EpiCrossKV>()) != cudaSuccess) return e;
#define PREPSK(BN, EPI) \
  if ((e = prepare_gemm_splitk<BN, EPI>()) != cudaSuccess) return e;
  PREPSK(64, EpiStore) PREPSK(128, EpiStore) PREPSK(64, EpiResidual) PREPSK(128, EpiResidual)
  PREPSK(64, EpiQkvDecode) PREPSK(128, EpiQkvDecode) PREPSK(64, EpiGeglu) PREPSK(128, EpiGeglu)
#undef PREPSK
  if ((e = prepare_gemm_2cta<EpiResidual, B200T5_F16 != 0>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_splitk<64, EpiResidual, B200T5_F16 != 0>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_splitk<128, EpiResidual, B200T5_F16 != 0>()) != cudaSuccess) return e;
  // the teacher-forced forward pass (b200t5_forward): the GeGLU product on the decode packing, the lm_head variants
  if ((e = prepare_gemm<128, EpiGegluNarrow>()) != cudaSuccess) return e;
  // the ReLU feed-forward of T5 v1.0 checkpoints, in the encoder, the decode step and the forward pass
  if ((e = prepare_gemm_2cta<EpiRelu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_enc_ws<EpiRelu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_splitk<64, EpiRelu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm_splitk<128, EpiRelu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm<128, EpiRelu>()) != cudaSuccess) return e;
  if ((e = prepare_gemm<128, EpiLmLogits<false>>()) != cudaSuccess) return e;
  if ((e = prepare_gemm<128, EpiLmLogits<true>>()) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(decoder_attn_kernel<kAttnCausal>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)) != cudaSuccess)
    return e;
  if ((e = cudaFuncSetAttribute(decoder_attn_kernel<kAttnCross>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)) != cudaSuccess)
    return e;
  if ((e = cudaFuncSetAttribute(decoder_cross_packed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)) != cudaSuccess)
    return e;
  if ((e = cudaFuncSetAttribute(attn_cross_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(XsSmem::bytes(kXsMaxStages, 4096)))) != cudaSuccess)
    return e;
  return cudaFuncSetAttribute(encoder_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
}

// gelu_new over all 65536 bf16 inputs, evaluated once on the device with the exact op-by-op
// arithmetic; the host keeps only the magnitude window in which neither shortcut holds.
struct GeluLutOwner {
  DevBuf table;
  GeluLut lut{nullptr, 0, 0};
  int pow_mode = -1;
};
static GeluLutOwner g_gelu;  // one process drives one GPU

[[maybe_unused]] static int ensure_gelu_lut(b200t5_ctx* h, int pow_mode, GeluLut* out) {
  if (g_gelu.lut.table && g_gelu.pow_mode == pow_mode) {
    *out = g_gelu.lut;
    return B200T5_OK;
  }
  DevBuf full;
  CU_OK(h, full.alloc(65536 * 2));
  build_gelu_table_kernel<<<256, 256>>>(full.as<uint16_t>(), pow_mode);
  CU_OK(h, cudaGetLastError());
  std::vector<uint16_t> t(65536);
  CU_OK(h, cudaMemcpy(t.data(), full.p, 65536 * 2, cudaMemcpyDeviceToHost));
  auto half_bits = [](uint16_t xb) {  // bf16(0.5 * x) for a bf16 bit pattern, round-to-nearest-even
    uint32_t u = static_cast<uint32_t>(xb) << 16;
    float f;
    memcpy(&f, &u, 4);
    f *= 0.5f;
    memcpy(&u, &f, 4);
    u += 0x7FFFu + ((u >> 16) & 1u);
    return static_cast<uint16_t>(u >> 16);
  };
  int lo = 0;
  while (lo < 0x7F80 && t[lo] == half_bits(static_cast<uint16_t>(lo)) && t[0x8000 | lo] == half_bits(static_cast<uint16_t>(0x8000 | lo))) ++lo;
  int hi = 0x7F80;
  while (hi > lo && t[hi - 1] == static_cast<uint16_t>(hi - 1) && t[0x8000 | (hi - 1)] == 0x8000) --hi;
  const int n = hi - lo;
  if (n < 0 || 2 * n * 2 > kEpiSmemBytes) return fail(h, B200T5_ECUDA, "gelu table window [%#x,%#x) does not fit the epilogue scratch", lo, hi);
  std::vector<uint16_t> compact(((static_cast<size_t>(2) * (n > 0 ? n : 1) + 7) / 8) * 8 + 8, 0);
  for (int i = 0; i < n; ++i) {
    compact[i] = t[lo + i];
    compact[n + i] = t[0x8000 | (lo + i)];
  }
  CU_OK(h, g_gelu.table.alloc(compact.size() * 2));
  CU_OK(h, cudaMemcpy(g_gelu.table.p, compact.data(), compact.size() * 2, cudaMemcpyHostToDevice));
  g_gelu.lut = GeluLut{g_gelu.table.as<uint16_t>(), lo, hi};
  g_gelu.pow_mode = pow_mode;
  *out = g_gelu.lut;
  return B200T5_OK;
}

// ================================================================== lifecycle
extern "C" const char* b200t5_version(void) {
  return B200T5_F16 ? "b200t5 0.1 fp16 (sm_90a, wgmma/TMA)" : "b200t5 0.1 (sm_90a, wgmma/TMA)";
}
extern "C" const char* b200t5_last_global_error(void) { return g_err; }
extern "C" const char* b200t5_last_error(b200t5_handle h) { return h ? h->err : g_err; }

extern "C" int b200t5_create(const b200t5_config* cfg, int device, b200t5_handle* out) {
  if (!cfg || !out) return fail(nullptr, B200T5_EINVAL, "null argument");
  *out = nullptr;
  if (cfg->d_kv != 64) return fail(nullptr, B200T5_EINVAL, "d_kv=%d unsupported (kernels are specialised for 64)", cfg->d_kv);
  if (cfg->is_gated_gelu != 0 && cfg->is_gated_gelu != 1)
    return fail(nullptr, B200T5_EINVAL, "is_gated_gelu=%d: 1 = feed_forward_proj 'gated-gelu', 0 = 'relu'", cfg->is_gated_gelu);
  if (cfg->scale_decoder_outputs != 0 && cfg->scale_decoder_outputs != 1)
    return fail(nullptr, B200T5_EINVAL, "scale_decoder_outputs=%d: must be 0 or 1", cfg->scale_decoder_outputs);
  if (cfg->d_model % 8 || cfg->d_ff % 32 || cfg->d_model > 4096 || cfg->vocab_size < 2 || cfg->num_heads < 1 ||
      cfg->num_layers < 1 || cfg->num_decoder_layers < 1)
    return fail(nullptr, B200T5_EINVAL, "unsupported shape: d_model=%d d_ff=%d vocab=%d", cfg->d_model, cfg->d_ff, cfg->vocab_size);
  int sms = check_device(nullptr, device);
  if (sms < 0) return sms;
  b200t5_ctx* h = new (std::nothrow) b200t5_ctx();
  if (!h) return fail(nullptr, B200T5_ENOMEM, "out of host memory");
  h->c = Cfg{cfg->vocab_size, cfg->d_model, cfg->d_ff, cfg->num_heads, cfg->num_heads * 64, cfg->num_layers,
             cfg->num_decoder_layers, cfg->relative_attention_num_buckets, cfg->relative_attention_max_distance,
             cfg->layer_norm_epsilon, cfg->pad_token_id, cfg->eos_token_id, cfg->decoder_start_token_id,
             cfg->is_gated_gelu == 1,
             // transformers: sequence_output * (self.model_dim ** -0.5), a Python float taken as fp32 by the multiply
             cfg->scale_decoder_outputs ? static_cast<float>(pow(static_cast<double>(cfg->d_model), -0.5)) : 0.f};
  h->device = device;
  h->num_sms = sms;
  h->enc.resize(h->c.Le);
  h->dec.resize(h->c.Ld);
  const char* pdl_env = getenv("B200T5_PDL");
  h->use_pdl = pdl_env ? atoi(pdl_env) != 0 : true;
  if (const char* eg_env = getenv("B200T5_ENC_GEMM")) h->enc_gemm_ws = atoi(eg_env) != 0;
  if (const char* xa_env = getenv("B200T5_XATTN")) h->xattn_mode = strcmp(xa_env, "ldg") == 0 ? 0 : strcmp(xa_env, "stream") == 0 ? 1 : 2;
  if (const char* xs_env = getenv("B200T5_XS_STAGES")) {
    const int v = atoi(xs_env);
    if (v >= 2 && v <= kXsMaxStages) h->xs_stages = v;
  }
  if (const char* sk_env = getenv("B200T5_SK")) {
    int v[8];
    if (sscanf(sk_env, "%d,%d,%d,%d,%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3], &v[4], &v[5], &v[6], &v[7]) == 8) {
      b200t5_ctx::SkChoice* dst[4] = {&h->sk_qkv, &h->sk_proj, &h->sk_wi, &h->sk_ffo};
      for (int i = 0; i < 4; ++i) {
        dst[i]->bn = v[2 * i] == 128 ? 128 : 64;
        dst[i]->split = v[2 * i + 1] >= 8 ? 8 : (v[2 * i + 1] >= 4 ? 4 : (v[2 * i + 1] >= 2 ? 2 : 1));
      }
    }
  }
  if (const char* st_env = getenv("B200T5_SK_STAGES")) {
    int a = 0, b = 0;
    if (sscanf(st_env, "%d,%d", &a, &b) == 2) {
      h->sk_stages64 = a;
      h->sk_stages128 = b;
    }
  }
  const char* ch_env = getenv("B200T5_CHAINS");
  h->chains_override = ch_env ? atoi(ch_env) : 0;
  if (const char* ao_env = getenv("B200T5_ADMIT_OVERLAP")) h->admit_overlap = atoi(ao_env) != 0;
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // (lowest, highest)
  if (cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->exec_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithPriority(&h->enc_stream, cudaStreamNonBlocking, prio_lo) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->enc_done_ev, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->admitted_ev, cudaEventDisableTiming) != cudaSuccess) {
    delete h;
    return fail(nullptr, B200T5_ECUDA, "cudaStreamCreate failed");
  }
  {
    cudaError_t ke = init_kernel_attrs();
    if (ke != cudaSuccess) {
      delete h;
      return fail(nullptr, B200T5_ECUDA, "kernel attribute setup failed: %s", cudaGetErrorString(ke));
    }
  }
#if !B200T5_F16  // (the fp16 build evaluates gelu_new directly; the table indexes bf16 bit patterns)
  {
    int lrc = ensure_gelu_lut(nullptr, 0, &h->gelu_lut);
    if (lrc != B200T5_OK) {
      delete h;
      return lrc;
    }
  }
#endif
  {
    cudaError_t ce = cudaSuccess;
    for (int i = 0; i < 4 && ce == cudaSuccess; ++i) ce = cudaEventCreate(&h->ev[i]);
    for (int i = 0; i < kMaxChains && ce == cudaSuccess; ++i) ce = cudaStreamCreateWithFlags(&h->chain_streams[i], cudaStreamNonBlocking);
    for (int i = 0; i <= kMaxChains && ce == cudaSuccess; ++i) ce = cudaEventCreateWithFlags(&h->chain_ev[i], cudaEventDisableTiming);
    if (ce != cudaSuccess) {
      b200t5_destroy(h);
      return fail(nullptr, B200T5_ECUDA, "stream/event creation failed: %s", cudaGetErrorString(ce));
    }
  }
  *out = h;
  return B200T5_OK;
}

extern "C" int b200t5_destroy(b200t5_handle h) {
  if (!h) return B200T5_OK;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->plan.reset();
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  if (h->exec_stream) cudaStreamDestroy(h->exec_stream);
  if (h->enc_stream) cudaStreamDestroy(h->enc_stream);
  if (h->enc_done_ev) cudaEventDestroy(h->enc_done_ev);
  if (h->admitted_ev) cudaEventDestroy(h->admitted_ev);
  for (int i = 0; i < kMaxChains; ++i)
    if (h->chain_streams[i]) cudaStreamDestroy(h->chain_streams[i]);
  for (int i = 0; i <= kMaxChains; ++i)
    if (h->chain_ev[i]) cudaEventDestroy(h->chain_ev[i]);
  for (int i = 0; i < 4; ++i)
    if (h->ev[i]) cudaEventDestroy(h->ev[i]);
  delete h;
  return B200T5_OK;
}

extern "C" int b200t5_set_weight(b200t5_handle h, const char* name, const void* dev_ptr, int dtype,
                                 const int64_t* shape, int ndim) {
  if (!h || !name || !dev_ptr || !shape || ndim < 1 || ndim > 2) return fail(h, B200T5_EINVAL, "set_weight: bad argument");
  if (h->finalized) return fail(h, B200T5_ESTATE, "set_weight after finalize");
  if (dtype < 0 || dtype > 2) return fail(h, B200T5_EINVAL, "set_weight(%s): unknown dtype %d", name, dtype);
  CU_OK(h, cudaSetDevice(h->device));
  size_t n = 1;
  std::vector<int64_t> shp(shape, shape + ndim);
  for (int i = 0; i < ndim; ++i) {
    if (shape[i] <= 0) return fail(h, B200T5_EINVAL, "set_weight(%s): bad shape", name);
    n *= static_cast<size_t>(shape[i]);
  }
  std::unique_ptr<DevBuf> buf(new DevBuf());
  CU_OK(h, buf->alloc(n * sizeof(act_t)));
  if (dtype == (B200T5_F16 ? B200T5_DTYPE_F16 : B200T5_DTYPE_BF16)) {
    CU_OK(h, cudaMemcpy(buf->p, dev_ptr, n * sizeof(act_t), cudaMemcpyDeviceToDevice));
  } else {
    convert_to_act_kernel<<<1024, 256>>>(dev_ptr, dtype, buf->as<act_t>(), n);
    CU_OK(h, cudaGetLastError());
    CU_OK(h, cudaDeviceSynchronize());
  }
  h->raw[name] = std::move(buf);
  h->raw_shape[name] = shp;
#if B200T5_F16
  {
    const std::string nm(name);
    const std::string suffix = "DenseReluDense.wo.weight";
    if (nm.size() >= suffix.size() && nm.compare(nm.size() - suffix.size(), suffix.size(), suffix) == 0) {
      std::unique_ptr<DevBuf> f(new DevBuf());
      CU_OK(h, f->alloc(n * 4));
      convert_to_f32_kernel<<<1024, 256>>>(dev_ptr, dtype, f->as<float>(), n);
      CU_OK(h, cudaGetLastError());
      CU_OK(h, cudaDeviceSynchronize());
      h->raw_f32[nm] = std::move(f);
    }
  }
#endif
  return B200T5_OK;
}

// fetch a raw tensor, checking its shape
static act_t* take(b200t5_ctx* h, const std::string& name, int64_t r, int64_t c, int* rc) {
  auto it = h->raw.find(name);
  if (it == h->raw.end()) {
    *rc = fail(h, B200T5_ESTATE, "finalize: missing weight '%s'", name.c_str());
    return nullptr;
  }
  const auto& s = h->raw_shape[name];
  const bool ok = (c == 0) ? (s.size() == 1 && s[0] == r) : (s.size() == 2 && s[0] == r && s[1] == c);
  if (!ok) {
    *rc = fail(h, B200T5_EINVAL, "finalize: weight '%s' has the wrong shape", name.c_str());
    return nullptr;
  }
  return it->second->as<act_t>();
}

// dst[ntiles*bn, d]: per tile, bn/2 rows of wi_0 followed by the matching bn/2 rows of wi_1.
static int interleave_geglu(b200t5_ctx* h, const act_t* wi0, const act_t* wi1, DevBuf& dst, int F, int d, int bn,
                            int* rows_out) {
  const int half = bn / 2;
  const int ntiles = (F + half - 1) / half;
  CU_OK(h, dst.alloc(static_cast<size_t>(ntiles) * bn * d * sizeof(act_t)));
  CU_OK(h, cudaMemset(dst.p, 0, dst.bytes));
  for (int j = 0; j < ntiles; ++j) {
    const int rows = (j + 1) * half <= F ? half : F - j * half;
    act_t* base = dst.as<act_t>() + static_cast<size_t>(j) * bn * d;
    CU_OK(h, cudaMemcpy(base, wi0 + static_cast<size_t>(j) * half * d, static_cast<size_t>(rows) * d * sizeof(act_t), cudaMemcpyDeviceToDevice));
    CU_OK(h, cudaMemcpy(base + static_cast<size_t>(half) * d, wi1 + static_cast<size_t>(j) * half * d, static_cast<size_t>(rows) * d * sizeof(act_t), cudaMemcpyDeviceToDevice));
  }
  *rows_out = ntiles * bn;
  return B200T5_OK;
}

// Feed-forward output projection weight [d, F] as the GEMM kernels read it: a 2-byte copy (bf16 build) or the
// two tf32 pieces side by side, [d, 2 * round_up(F, 32)] fp32 (fp16 build).
static int build_ffo(b200t5_ctx* h, DevBuf& dst, const std::string& name, const act_t* src2, int d, int F, int* k_cols) {
#if B200T5_F16
  auto it = h->raw_f32.find(name);
  if (it == h->raw_f32.end()) return fail(h, B200T5_ESTATE, "finalize: missing fp32 copy of '%s'", name.c_str());
  const int Fp = (F + 31) / 32 * 32;
  CU_OK(h, dst.alloc(static_cast<size_t>(d) * 2 * Fp * 4));
  const size_t n = static_cast<size_t>(d) * Fp;
  split_tf32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256>>>(it->second->as<float>(), dst.as<float>(), d, F, Fp);
  CU_OK(h, cudaGetLastError());
  CU_OK(h, cudaDeviceSynchronize());
  *k_cols = 2 * Fp;
  (void)src2;
  return B200T5_OK;
#else
  *k_cols = F;
  CU_OK(h, dst.alloc(static_cast<size_t>(d) * F * sizeof(act_t)));
  CU_OK(h, cudaMemcpy(dst.p, src2, static_cast<size_t>(d) * F * sizeof(act_t), cudaMemcpyDeviceToDevice));
  return B200T5_OK;
#endif
}

static int clone_buf(b200t5_ctx* h, DevBuf& dst, const act_t* src, size_t n) {
  CU_OK(h, dst.alloc(n * sizeof(act_t)));
  CU_OK(h, cudaMemcpy(dst.p, src, n * sizeof(act_t), cudaMemcpyDeviceToDevice));
  return B200T5_OK;
}

// The feed-forward input weight(s) of one layer (`prefix` = "<side>.block.<l>.layer.<k>.DenseReluDense.") as the GEMMs
// with N-tiles of bn rows read them. Gated-GELU: wi_0 and wi_1 interleaved per tile (interleave_geglu), rows_out =
// the padded row count. ReLU (T5 v1.0): wi [F, d] as is, which every tile width reads in place (the tensor map's
// out-of-bounds rows load as zeros and no store reaches past F), rows_out = F.
static int pack_wi(b200t5_ctx* h, const std::string& prefix, DevBuf& dst, int bn, int* rows_out) {
  const int F = h->c.F, d = h->c.d;
  int rc = B200T5_OK;
  if (!h->c.gated) {
    const act_t* wi = take(h, prefix + "wi.weight", F, d, &rc);
    if (!wi) return rc;
    *rows_out = F;
    return clone_buf(h, dst, wi, static_cast<size_t>(F) * d);
  }
  const act_t* wi0 = take(h, prefix + "wi_0.weight", F, d, &rc);
  const act_t* wi1 = wi0 ? take(h, prefix + "wi_1.weight", F, d, &rc) : nullptr;
  if (!wi1) return rc;
  return interleave_geglu(h, wi0, wi1, dst, F, d, bn, rows_out);
}

#define TRY(expr)            \
  do {                       \
    int _rc = (expr);        \
    if (_rc != B200T5_OK) return _rc; \
  } while (0)
#define TMAP(h, tm, base, rows, cols, box) \
  do {                                     \
    if (!make_tmap(tm, base, rows, cols, box)) return fail(h, B200T5_ECUDA, "%s", g_err); \
  } while (0)
// the operands of the feed-forward output projection: 2-byte in the bf16 build, fp32 (tf32 MMA) in the fp16 build
#define TMAP_FFO(h, tm, base, rows, cols, box) \
  do {                                         \
    if (!make_tmap(tm, base, rows, cols, box, B200T5_F16 != 0)) return fail(h, B200T5_ECUDA, "%s", g_err); \
  } while (0)

extern "C" int b200t5_finalize(b200t5_handle h) {
  if (!h) return fail(nullptr, B200T5_EINVAL, "null handle");
  if (h->finalized) return B200T5_OK;
  CU_OK(h, cudaSetDevice(h->device));
  const Cfg& c = h->c;
  int rc = B200T5_OK;
  const int d = c.d, I = c.I, F = c.F;

  act_t* shared = take(h, "shared.weight", c.V, d, &rc);
  if (!shared) return rc;
  TRY(clone_buf(h, h->shared, shared, static_cast<size_t>(c.V) * d));
  // real FLAN-T5 checkpoints carry a separate lm_head; a checkpoint without one is tied
  const act_t* lm = h->raw.count("lm_head.weight") ? take(h, "lm_head.weight", c.V, d, &rc) : shared;
  if (!lm) return rc;
  TRY(clone_buf(h, h->lm_head, lm, static_cast<size_t>(c.V) * d));
  TMAP(h, &h->tm_lm, h->lm_head.p, c.V, d, 128);

  act_t* p;
  if (!(p = take(h, "encoder.final_layer_norm.weight", d, 0, &rc))) return rc;
  TRY(clone_buf(h, h->enc_final_ln, p, d));
  if (!(p = take(h, "decoder.final_layer_norm.weight", d, 0, &rc))) return rc;
  TRY(clone_buf(h, h->dec_final_ln, p, d));

  // relative attention bias tables -> host floats
  for (int side = 0; side < 2; ++side) {
    const std::string nm = std::string(side ? "decoder" : "encoder") + ".block.0.layer.0.SelfAttention.relative_attention_bias.weight";
    if (!(p = take(h, nm, c.nb, c.H, &rc))) return rc;
    std::vector<act_t> tmp(static_cast<size_t>(c.nb) * c.H);
    CU_OK(h, cudaMemcpy(tmp.data(), p, tmp.size() * sizeof(act_t), cudaMemcpyDeviceToHost));
    std::vector<float>& dst = side ? h->dec_relbias_h : h->enc_relbias_h;
    dst.resize(tmp.size());
    for (size_t i = 0; i < tmp.size(); ++i) dst[i] = act2float(tmp[i]);
  }

  char nm[256];
  for (int l = 0; l < c.Le; ++l) {
    EncLayerW& w = h->enc[l];
    auto key = [&](const char* suffix) {
      snprintf(nm, sizeof(nm), "encoder.block.%d.%s", l, suffix);
      return std::string(nm);
    };
    if (!(p = take(h, key("layer.0.layer_norm.weight"), d, 0, &rc))) return rc;
    TRY(clone_buf(h, w.ln0, p, d));
    if (!(p = take(h, key("layer.1.layer_norm.weight"), d, 0, &rc))) return rc;
    TRY(clone_buf(h, w.ln1, p, d));
    const act_t* q = take(h, key("layer.0.SelfAttention.q.weight"), I, d, &rc);
    const act_t* k = q ? take(h, key("layer.0.SelfAttention.k.weight"), I, d, &rc) : nullptr;
    const act_t* v = k ? take(h, key("layer.0.SelfAttention.v.weight"), I, d, &rc) : nullptr;
    if (!v) return rc;
    CU_OK(h, w.wqkv.alloc(static_cast<size_t>(3) * I * d * sizeof(act_t)));
    const size_t blk = static_cast<size_t>(I) * d;
    CU_OK(h, cudaMemcpy(w.wqkv.as<act_t>(), q, blk * 2, cudaMemcpyDeviceToDevice));
    CU_OK(h, cudaMemcpy(w.wqkv.as<act_t>() + blk, k, blk * 2, cudaMemcpyDeviceToDevice));
    CU_OK(h, cudaMemcpy(w.wqkv.as<act_t>() + 2 * blk, v, blk * 2, cudaMemcpyDeviceToDevice));
    if (!(p = take(h, key("layer.0.SelfAttention.o.weight"), d, I, &rc))) return rc;
    TRY(clone_buf(h, w.wo, p, static_cast<size_t>(d) * I));
    int wi_rows = 0;
    TRY(pack_wi(h, key("layer.1.DenseReluDense."), w.wi, 256, &wi_rows));
    if (!(p = take(h, key("layer.1.DenseReluDense.wo.weight"), d, F, &rc))) return rc;
    TRY(build_ffo(h, w.wff_o, key("layer.1.DenseReluDense.wo.weight"), p, d, F, &h->ffo_k));
    TMAP(h, &w.tm_qkv, w.wqkv.p, 3 * I, d, k2ctaBox);
    TMAP(h, &w.tm_o, w.wo.p, d, I, k2ctaBox);
    TMAP(h, &w.tm_wi, w.wi.p, wi_rows, d, k2ctaBox);
    TMAP_FFO(h, &w.tm_ffo, w.wff_o.p, d, h->ffo_k, k2ctaBox);
  }

  CU_OK(h, h->wcrosskv.alloc(static_cast<size_t>(c.Ld) * 2 * I * d * sizeof(act_t)));
  for (int l = 0; l < c.Ld; ++l) {
    DecLayerW& w = h->dec[l];
    auto key = [&](const char* suffix) {
      snprintf(nm, sizeof(nm), "decoder.block.%d.%s", l, suffix);
      return std::string(nm);
    };
    if (!(p = take(h, key("layer.0.layer_norm.weight"), d, 0, &rc))) return rc;
    TRY(clone_buf(h, w.ln0, p, d));
    if (!(p = take(h, key("layer.1.layer_norm.weight"), d, 0, &rc))) return rc;
    TRY(clone_buf(h, w.ln1, p, d));
    if (!(p = take(h, key("layer.2.layer_norm.weight"), d, 0, &rc))) return rc;
    TRY(clone_buf(h, w.ln2, p, d));
    const act_t* q = take(h, key("layer.0.SelfAttention.q.weight"), I, d, &rc);
    const act_t* k = q ? take(h, key("layer.0.SelfAttention.k.weight"), I, d, &rc) : nullptr;
    const act_t* v = k ? take(h, key("layer.0.SelfAttention.v.weight"), I, d, &rc) : nullptr;
    if (!v) return rc;
    const size_t blk = static_cast<size_t>(I) * d;
    CU_OK(h, w.wqkv.alloc(3 * blk * sizeof(act_t)));
    CU_OK(h, cudaMemcpy(w.wqkv.as<act_t>(), q, blk * 2, cudaMemcpyDeviceToDevice));
    CU_OK(h, cudaMemcpy(w.wqkv.as<act_t>() + blk, k, blk * 2, cudaMemcpyDeviceToDevice));
    CU_OK(h, cudaMemcpy(w.wqkv.as<act_t>() + 2 * blk, v, blk * 2, cudaMemcpyDeviceToDevice));
    if (!(p = take(h, key("layer.0.SelfAttention.o.weight"), d, I, &rc))) return rc;
    TRY(clone_buf(h, w.wo, p, static_cast<size_t>(d) * I));
    if (!(p = take(h, key("layer.1.EncDecAttention.q.weight"), I, d, &rc))) return rc;
    TRY(clone_buf(h, w.wcq, p, blk));
    const act_t* ck = take(h, key("layer.1.EncDecAttention.k.weight"), I, d, &rc);
    const act_t* cv = ck ? take(h, key("layer.1.EncDecAttention.v.weight"), I, d, &rc) : nullptr;
    if (!cv) return rc;
    CU_OK(h, cudaMemcpy(h->wcrosskv.as<act_t>() + (static_cast<size_t>(l) * 2 + 0) * blk, ck, blk * 2, cudaMemcpyDeviceToDevice));
    CU_OK(h, cudaMemcpy(h->wcrosskv.as<act_t>() + (static_cast<size_t>(l) * 2 + 1) * blk, cv, blk * 2, cudaMemcpyDeviceToDevice));
    if (!(p = take(h, key("layer.1.EncDecAttention.o.weight"), d, I, &rc))) return rc;
    TRY(clone_buf(h, w.wco, p, static_cast<size_t>(d) * I));
    int wi_rows = 0;
    // TMA box rows = the N-tile of the split-K kernel that will read the weight
    const int bn_qkv = h->sk_qkv.bn, bn_proj = h->sk_proj.bn, bn_wi = h->sk_wi.bn, bn_ffo = h->sk_ffo.bn;
    TRY(pack_wi(h, key("layer.2.DenseReluDense."), w.wi, bn_wi, &wi_rows));
    w.wi_rows = wi_rows;
    if (!(p = take(h, key("layer.2.DenseReluDense.wo.weight"), d, F, &rc))) return rc;
    TRY(build_ffo(h, w.wff_o, key("layer.2.DenseReluDense.wo.weight"), p, d, F, &h->ffo_k));
    TMAP(h, &w.tm_qkv, w.wqkv.p, 3 * I, d, bn_qkv);
    TMAP(h, &w.tm_o, w.wo.p, d, I, bn_proj);
    TMAP(h, &w.tm_cq, w.wcq.p, I, d, bn_proj);
    TMAP(h, &w.tm_co, w.wco.p, d, I, bn_proj);
    TMAP(h, &w.tm_wi, w.wi.p, wi_rows, d, bn_wi);
    TMAP_FFO(h, &w.tm_ffo, w.wff_o.p, d, h->ffo_k, bn_ffo);
    TMAP(h, &w.tm2_qkv, w.wqkv.p, 3 * I, d, k2ctaBox);
    TMAP(h, &w.tm2_o, w.wo.p, d, I, k2ctaBox);
    TMAP(h, &w.tm2_cq, w.wcq.p, I, d, k2ctaBox);
    TMAP(h, &w.tm2_co, w.wco.p, d, I, k2ctaBox);
    TMAP_FFO(h, &w.tm2_ffo, w.wff_o.p, d, h->ffo_k, k2ctaBox);
  }
  TMAP(h, &h->tm_crosskv, h->wcrosskv.p, static_cast<uint64_t>(c.Ld) * 2 * I, d, k2ctaBox);

  h->raw.clear();
  h->raw_f32.clear();
  h->raw_shape.clear();
  h->finalized = true;
  return B200T5_OK;
}


// ================================================================== plans
static int build_plan(b200t5_ctx* h, int B, int S, int Tmax, int group, int ws_S) {
  const Cfg& c = h->c;
  std::unique_ptr<Plan> pl(new Plan());
  pl->B = B;
  pl->S = S;
  pl->Tmax = Tmax;
  pl->group = group;
  pl->ws_S = ws_S;
  const size_t M = static_cast<size_t>(B) * S, Mw = static_cast<size_t>(B) * ws_S;
  const int d = c.d, I = c.I, F = c.F, H = c.H;
  CU_OK(h, pl->x.alloc(Mw * d * sizeof(res_t)));
  CU_OK(h, pl->xn.alloc(Mw * d * 2));
  CU_OK(h, pl->qkv.alloc(Mw * 3 * I * 2));
  CU_OK(h, pl->ctx.alloc(Mw * I * 2));
  CU_OK(h, pl->hff.alloc(Mw * F * sizeof(ffh_t)));
  CU_OK(h, pl->key_ok.alloc(M));
  CU_OK(h, pl->extent.alloc(static_cast<size_t>(B) * 4));
  CU_OK(h, pl->cu.alloc(static_cast<size_t>(B + 1) * 4));
  CU_OK(h, pl->row_b.alloc(M * 4));
  CU_OK(h, pl->row_s.alloc(M * 4));
  CU_OK(h, cudaMallocHost(&pl->h_cu, 16));
  CU_OK(h, pl->cross_kv.alloc(static_cast<size_t>(c.Ld) * 2 * M * I * 2));
  // finite everywhere: keys beyond a prompt's extent are never written, and the tensor-core decode attention
  // multiplies them by p = 0
  CU_OK(h, cudaMemset(pl->cross_kv.p, 0, pl->cross_kv.bytes));
  CU_OK(h, pl->dx.alloc(static_cast<size_t>(B) * d * sizeof(res_t)));
  CU_OK(h, pl->dxn.alloc(static_cast<size_t>(B) * d * 2));
  CU_OK(h, pl->dq.alloc(static_cast<size_t>(B) * I * 2));
  CU_OK(h, pl->dctx.alloc(static_cast<size_t>(B) * I * 2));
  CU_OK(h, pl->dh.alloc(static_cast<size_t>(B) * F * sizeof(ffh_t)));
  CU_OK(h, pl->self_kv.alloc(static_cast<size_t>(c.Ld) * 2 * B * I * Tmax * 2));
  pl->n_vtiles = (c.V + 127) / 128;
  CU_OK(h, pl->pval.alloc(static_cast<size_t>(B) * pl->n_vtiles * 4));
  CU_OK(h, pl->pidx.alloc(static_cast<size_t>(B) * pl->n_vtiles * 4));
  CU_OK(h, pl->state.alloc(sizeof(DecodeState)));
  CU_OK(h, pl->unfinished.alloc(static_cast<size_t>(B) * 4));
  CU_OK(h, pl->batch.ids.alloc(static_cast<size_t>(B) * (Tmax + 1) * 8));
  CU_OK(h, pl->batch.len.alloc(static_cast<size_t>(B) * 4));
  pl->batch.cap = static_cast<size_t>(B);
  CU_OK(h, pl->ids_dev.alloc(M * 8));
  CU_OK(h, pl->mask_dev.alloc(M * 8));
  CU_OK(h, cudaMallocHost(&pl->h_ids, M * 8));
  CU_OK(h, cudaMallocHost(&pl->h_mask, M * 8));
  CU_OK(h, cudaMallocHost(&pl->h_out, static_cast<size_t>(B) * (Tmax + 1) * 8));
  CU_OK(h, cudaMallocHost(&pl->h_len, static_cast<size_t>(B) * 4));
  CU_OK(h, cudaMallocHost(&pl->h_state, sizeof(DecodeState)));
  CU_OK(h, pl->live_extent.alloc(static_cast<size_t>(B) * 4));
  CU_OK(h, pl->live_key_ok.alloc(M));
  CU_OK(h, pl->pos.alloc(static_cast<size_t>(B) * 4));
  CU_OK(h, pl->out_row.alloc(static_cast<size_t>(B) * 4));
  CU_OK(h, pl->admit.alloc(static_cast<size_t>(3) * B * 4));
  CU_OK(h, cudaMemset(pl->pos.p, 0, pl->pos.bytes));
  CU_OK(h, pl->xs_stamps.alloc(static_cast<size_t>(c.Ld) * kMaxChains * 2 * 8));
  CU_OK(h, pl->xs_acc.alloc(static_cast<size_t>(c.Ld) * (kMaxChains + 1) * 2 * 8));
  CU_OK(h, cudaMemset(pl->xs_stamps.p, 0, pl->xs_stamps.bytes));
  CU_OK(h, cudaMemset(pl->xs_acc.p, 0, pl->xs_acc.bytes));
  CU_OK(h, cudaMemset(pl->out_row.p, 0, pl->out_row.bytes));
  CU_OK(h, cudaMallocHost(&pl->h_unf, static_cast<size_t>(B) * 4));
  CU_OK(h, cudaMallocHost(&pl->h_admit, static_cast<size_t>(3) * B * 4));

  // bias tables (values are the bf16 embedding entries widened to fp32)
  {
    std::vector<float> eb(static_cast<size_t>(H) * (2 * S - 1));
    for (int rel = -(S - 1); rel <= S - 1; ++rel) {
      const int bk = b200t5_relative_bucket(rel, 1, c.nb, c.maxdist);
      for (int hh = 0; hh < H; ++hh) eb[static_cast<size_t>(hh) * (2 * S - 1) + rel + S - 1] = h->enc_relbias_h[static_cast<size_t>(bk) * H + hh];
    }
    CU_OK(h, pl->enc_bias.alloc(eb.size() * 4));
    CU_OK(h, cudaMemcpy(pl->enc_bias.p, eb.data(), eb.size() * 4, cudaMemcpyHostToDevice));
    std::vector<float> db(static_cast<size_t>(H) * Tmax);
    for (int n = 0; n < Tmax; ++n) {
      const int bk = b200t5_relative_bucket(-n, 0, c.nb, c.maxdist);
      for (int hh = 0; hh < H; ++hh) db[static_cast<size_t>(hh) * Tmax + n] = h->dec_relbias_h[static_cast<size_t>(bk) * H + hh];
    }
    CU_OK(h, pl->dec_bias.alloc(db.size() * 4));
    CU_OK(h, cudaMemcpy(pl->dec_bias.p, db.data(), db.size() * 4, cudaMemcpyHostToDevice));
  }
  TMAP(h, &pl->tm_xn, pl->xn.p, Mw, d, 128);
  TMAP(h, &pl->tm_ctx, pl->ctx.p, Mw, I, 128);
  TMAP_FFO(h, &pl->tm_hff, pl->hff.p, Mw, F, 128);
  TMAP(h, &pl->tm_cross_kv, pl->cross_kv.p, static_cast<uint64_t>(c.Ld) * 2 * B * H * S, 64, kXsChunkKeys);
  CU_OK(h, cudaMemset(pl->ctx.p, 0, pl->ctx.bytes));  // padded query tiles are skipped: keep them finite
  {
    // chains of 128 rows (one M-tile per split-K GEMM): two for a 256-row batch, four for the slot pool's 512 rows
    // (three would give uneven M-tiles); B200T5_CHAINS overrides
    int nc = B >= 512 ? 4 : (B >= 128 ? 2 : 1);
    if (h->chains_override > 0) nc = h->chains_override;
    if (nc > kMaxChains) nc = kMaxChains;
    const int groups = B / group;  // a chain holds whole prompts (beam search: `group` rows each)
    if (nc > groups) nc = groups;
    pl->n_chains = nc;
    for (int i = 0; i < nc; ++i) {
      Plan::Chain& ch = pl->chains[i];
      ch.b0 = group * static_cast<int>(static_cast<long long>(groups) * i / nc);
      ch.nb = group * static_cast<int>(static_cast<long long>(groups) * (i + 1) / nc) - ch.b0;
      TMAP(h, &ch.tm_dxn, pl->dxn.as<act_t>() + static_cast<size_t>(ch.b0) * d, ch.nb, d, 128);
      TMAP(h, &ch.tm_dctx, pl->dctx.as<act_t>() + static_cast<size_t>(ch.b0) * I, ch.nb, I, 128);
      TMAP_FFO(h, &ch.tm_dh, pl->dh.as<ffh_t>() + static_cast<size_t>(ch.b0) * F, ch.nb, F, 128);
    }
  }
  h->plan = std::move(pl);
  return B200T5_OK;
}

// `ws`: rows per prompt the encoder workspace must hold besides S (a decoder prompt's prefill runs P - 1 rows per prompt)
static int ensure_plan(b200t5_ctx* h, int B, int S, int Tmax, int group = 1, int ws = 0) {
  if (h->plan && h->plan->B == B && h->plan->S == S && h->plan->Tmax == Tmax && h->plan->group == group && h->plan->ws_S >= ws)
    return B200T5_OK;
  CU_OK(h, cudaDeviceSynchronize());
  h->plan.reset();
  return build_plan(h, B, S, Tmax, group, std::max(S, ws));
}

// ================================================================== encoder
static int run_encoder(b200t5_ctx* h, const long long* ids, const long long* mask, cudaStream_t s, const int* row_on = nullptr) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  const int B = p.B, S = p.S, d = c.d, I = c.I, F = c.F, H = c.H;
  int M = B * S;
  prep_mask_kernel<<<B, 128, 0, s>>>(mask, p.key_ok.as<unsigned char>(), p.extent.as<int>(), B, S, row_on);
  h->launches++;
  // Variable-length packing: only rows below extent[b] are ever read downstream, so the encoder runs on those
  // (elementwise.cuh). The number of packed rows sizes the GEMM grids, hence one 4-byte read-back per call.
  p.packed = S <= kEncPackMaxS;
  if (row_on && !p.packed)
    return fail(h, B200T5_EINVAL, "slot-pool admission needs the packed encoder path (S <= %d)", kEncPackMaxS);
  const int* cu = nullptr;
  p.rows_valid = M;
  if (p.packed) {
    pack_offsets_kernel<<<1, 256, 0, s>>>(p.extent.as<int>(), p.cu.as<int>(), B);
    CU_OK(h, cudaMemcpyAsync(p.h_cu, p.cu.as<int>() + B, 4, cudaMemcpyDeviceToHost, s));
    CU_OK(h, cudaStreamSynchronize(s));
    M = *p.h_cu;
    p.rows_valid = M;
    cu = p.cu.as<int>();
    embed_rows_packed_kernel<<<dim3((S + 7) / 8, B), 256, 0, s>>>(ids, h->shared.as<act_t>(), p.x.as<res_t>(), cu, p.row_b.as<int>(),
                                                               p.row_s.as<int>(), S, d, c.V);
    h->launches += 2;
  } else {
    embed_rows_kernel<<<(M + 7) / 8, 256, 0, s>>>(ids, h->shared.as<act_t>(), p.x.as<res_t>(), M, d, c.V);
    h->launches++;
  }
  p.packed_rows = M;
  CU_OK(h, cudaGetLastError());
  const size_t attn_smem = encoder_attn_smem_bytes(S);
  if (attn_smem > 96 * 1024) return fail(h, B200T5_EINVAL, "encoder length S=%d too long for the attention kernel", S);
  const int wi_tiles = (F + 127) / 128;
  for (int l = 0; l < c.Le; ++l) {
    EncLayerW& w = h->enc[l];
    CU_OK(h, run_rmsnorm(h, p.x.as<res_t>(), w.ln0.as<act_t>(), p.xn.as<act_t>(), M, d, c.eps, s));
    {
      EpiStore::Params ep{p.qkv.as<act_t>(), 3 * I};
      CU_OK(h, run_gemm_2cta<EpiStore>(h, p.tm_xn, w.tm_qkv, M, 3 * I, d, ep, s));
    }
    encoder_attn_kernel<<<dim3((S + kEncQ - 1) / kEncQ, B * H), kEncThreads, attn_smem, s>>>(
        p.qkv.as<act_t>(), p.ctx.as<act_t>(), p.enc_bias.as<float>(), p.key_ok.as<unsigned char>(), p.extent.as<int>(), cu, S, H);
    h->launches++;
    CU_OK(h, cudaGetLastError());
    {
      EpiResidual::Params ep{p.x.as<res_t>(), p.x.as<res_t>(), d};
      ep.round_out = l == 0;  // (fp16 build) the stream is still fp16 before the first feed-forward block
      CU_OK(h, run_gemm_2cta<EpiResidual>(h, p.tm_ctx, w.tm_o, M, d, I, ep, s));
    }
    CU_OK(h, run_rmsnorm(h, p.x.as<res_t>(), w.ln1.as<act_t>(), p.xn.as<act_t>(), M, d, c.eps, s));
    if (c.gated) {
      EpiGeglu::Params ep{p.hff.as<ffh_t>(), F, h->gelu_lut};
      CU_OK(h, run_gemm_2cta<EpiGeglu>(h, p.tm_xn, w.tm_wi, M, wi_tiles * 256, d, ep, s));
    } else {
      CU_OK(h, run_gemm_2cta<EpiRelu>(h, p.tm_xn, w.tm_wi, M, F, d, EpiRelu::Params{p.hff.as<ffh_t>(), F}, s));
    }
    {
      EpiResidual::Params ep{p.x.as<res_t>(), p.x.as<res_t>(), d};
      ep.round_acc = B200T5_F16 ? 0 : 1;  // fp16 build: `wo` is an fp32 Linear, its output is not rounded
      ep.round_out = B200T5_F16 ? 0 : 1;
      CU_OK(h, run_ffo_2cta(h, p.tm_hff, w.tm_ffo, M, d, ep, s));
    }
  }
  CU_OK(h, run_rmsnorm(h, p.x.as<res_t>(), h->enc_final_ln.as<act_t>(), p.xn.as<act_t>(), M, d, c.eps, s));
  return B200T5_OK;
}

static int run_cross_kv(b200t5_ctx* h, cudaStream_t s) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  EpiCrossKV::Params ep{p.cross_kv.as<act_t>(), p.B, c.H, p.S};
  if (p.packed) {
    ep.row_b = p.row_b.as<int>();
    ep.row_s = p.row_s.as<int>();
  }
  const int M = p.packed ? p.packed_rows : p.B * p.S;
  CU_OK(h, run_gemm_2cta<EpiCrossKV>(h, p.tm_xn, h->tm_crosskv, M, c.Ld * 2 * c.I, c.d, ep, s));
  return B200T5_OK;
}

// ================================================================== one decode step
// One chain = rows [b0, b0+nb) of the batch through all decoder layers, the lm_head and the
// greedy bookkeeping. Rows are independent, so chains only share read-only state (weights, the
// step counter) and write disjoint row ranges of the same buffers.
struct ChainView {
  int b0, nb;
  res_t* dx;
  ffh_t* dh;
  act_t *dxn, *dq, *dctx;
  const Plan::Chain* ch;
};
static ChainView chain_view(b200t5_ctx* h, const Plan::Chain& ch) {
  Plan& p = *h->plan;
  const Cfg& c = h->c;
  ChainView v;
  v.b0 = ch.b0;
  v.nb = ch.nb;
  v.dx = p.dx.as<res_t>() + static_cast<size_t>(ch.b0) * c.d;
  v.dxn = p.dxn.as<act_t>() + static_cast<size_t>(ch.b0) * c.d;
  v.dq = p.dq.as<act_t>() + static_cast<size_t>(ch.b0) * c.I;
  v.dctx = p.dctx.as<act_t>() + static_cast<size_t>(ch.b0) * c.I;
  v.dh = p.dh.as<ffh_t>() + static_cast<size_t>(ch.b0) * c.F;
  v.ch = &ch;
  return v;
}

// layer l, up to and including the cross-attention query projection
static int chain_layer_pre(b200t5_ctx* h, cudaStream_t s, const ChainView& v, int l) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  const int B = p.B, d = c.d, I = c.I, H = c.H, T = p.Tmax;
  const bool pdl = h->use_pdl;
  // static batch: one position for all rows; slot pool: row b of the chain is at pos[b0 + b]
  const int sstride = p.mode.pool ? 1 : 0;
  const int* step = p.mode.pool ? p.pos.as<int>() + v.b0 : &p.state.as<DecodeState>()->step;
  DecLayerW& w = h->dec[l];
  // [kv][B][H][T][64]: a row offset of b0 is a pointer offset inside each kv plane
  act_t* skv = p.self_kv.as<act_t>() + l * (static_cast<size_t>(2) * B * I * T) + static_cast<size_t>(v.b0) * I * T;
  CU_OK(h, run_rmsnorm(h, v.dx, w.ln0.as<act_t>(), v.dxn, v.nb, d, c.eps, s, pdl));
  {
    EpiQkvDecode::Params ep{v.dq, skv, step, B, H, T, sstride};
    CU_OK(h, run_gemm_sk<EpiQkvDecode>(h, h->sk_qkv, v.ch->tm_dxn, w.tm_qkv, v.nb, 3 * I, d, ep, s, pdl));
  }
  // 4 warps per (row, head): two memory round trips whatever t is
  CU_OK(h, launch_kernel(attn_decode_kernel<true>, dim3(v.nb * H), dim3(kAttnDecThreads), T * sizeof(float), s, pdl, v.dq, skv,
                         skv + static_cast<size_t>(B) * I * T, v.dctx, H, T, nullptr, nullptr, step, p.dec_bias.as<float>(),
                         XsStamps{nullptr, 0}, sstride));
  h->launches++;
  {
    EpiResidual::Params ep{v.dx, v.dx, d};
    ep.round_out = l == 0;  // (fp16 build) the stream is still fp16 before the first feed-forward block
    CU_OK(h, run_gemm_sk<EpiResidual>(h, h->sk_proj, v.ch->tm_dctx, w.tm_o, v.nb, d, I, ep, s, pdl));
  }
  CU_OK(h, run_rmsnorm(h, v.dx, w.ln1.as<act_t>(), v.dxn, v.nb, d, c.eps, s, pdl));
  {
    EpiStore::Params ep{v.dq, I};
    CU_OK(h, run_gemm_sk<EpiStore>(h, h->sk_proj, v.ch->tm_dxn, w.tm_cq, v.nb, I, d, ep, s, pdl));
  }
  return B200T5_OK;
}

// One cross-attention launch over rows [b0, b0 + nb) of layer l (`q`, `ctx`, `ext`, `ok` are row-b0-relative).
// `slot` < 0: no in-situ stamps.
static cudaError_t launch_cross_attention(b200t5_ctx* h, cudaStream_t s, bool pdl, int l, int b0, int nb, const act_t* q,
                                          act_t* ctx, const int* ext, const unsigned char* ok, int slot) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  const int B = p.B, S = p.S, I = c.I;
  XsStamps st{slot >= 0 && p.xs_stamps.p ? p.xs_stamps.as<unsigned long long>() : nullptr, slot >= 0 ? slot : 0};
  if (p.mode.xattn_stream) {
    const int items = nb * c.H;
    const int k_row0 = ((l * 2) * B + b0) * c.H * S, v_row0 = ((l * 2 + 1) * B + b0) * c.H * S;
    return launch_kernel(attn_cross_stream_kernel, dim3(xs_grid(items, h->num_sms)), dim3(kXsThreads),
                         XsSmem::bytes(h->xs_stages, S), s, pdl, p.tm_cross_kv, p.tm_cross_kv, k_row0, v_row0, q, ctx, items, c.H,
                         S, ext, ok, h->xs_stages, st);
  }
  const act_t* kplane = p.cross_kv.as<act_t>() + l * (static_cast<size_t>(2) * B * I * S) + static_cast<size_t>(b0) * I * S;
  return launch_kernel(attn_decode_kernel<false>, dim3(nb * c.H), dim3(kAttnDecThreads), S * sizeof(float), s, pdl, q, kplane,
                       kplane + static_cast<size_t>(B) * I * S, ctx, c.H, S, ext, ok, nullptr, nullptr, st, 0);
}

// layer l, cross-attention over the encoder keys (the HBM-streaming kernel)
static int chain_layer_cross(b200t5_ctx* h, cudaStream_t s, const ChainView& v, int l, int chain_index) {
  Plan& p = *h->plan;
  const int S = p.S;
  CU_OK(h, launch_cross_attention(h, s, h->use_pdl, l, v.b0, v.nb, v.dq, v.dctx, p.live_extent.as<int>() + v.b0,
                                  p.live_key_ok.as<unsigned char>() + static_cast<size_t>(v.b0) * S,
                                  h->profile_xattn ? l * p.n_chains + chain_index : -1));
  h->launches++;
  return B200T5_OK;
}

// layer l, after the cross-attention: output projection and the feed-forward block
static int chain_layer_post(b200t5_ctx* h, cudaStream_t s, const ChainView& v, int l) {
  const Cfg& c = h->c;
  const int d = c.d, I = c.I, F = c.F;
  const bool pdl = h->use_pdl;
  DecLayerW& w = h->dec[l];
  {
    EpiResidual::Params ep{v.dx, v.dx, d};
    ep.round_out = l == 0;
    CU_OK(h, run_gemm_sk<EpiResidual>(h, h->sk_proj, v.ch->tm_dctx, w.tm_co, v.nb, d, I, ep, s, pdl));
  }
  CU_OK(h, run_rmsnorm(h, v.dx, w.ln2.as<act_t>(), v.dxn, v.nb, d, c.eps, s, pdl));
  if (c.gated) {
    EpiGeglu::Params ep{v.dh, F, h->gelu_lut};
    CU_OK(h, run_gemm_sk<EpiGeglu>(h, h->sk_wi, v.ch->tm_dxn, w.tm_wi, v.nb, w.wi_rows, d, ep, s, pdl));
  } else {
    CU_OK(h, run_gemm_sk<EpiRelu>(h, h->sk_wi, v.ch->tm_dxn, w.tm_wi, v.nb, F, d, EpiRelu::Params{v.dh, F}, s, pdl));
  }
  {
    EpiResidual::Params ep{v.dx, v.dx, d};
    ep.round_acc = B200T5_F16 ? 0 : 1;  // fp16 build: `wo` is an fp32 Linear, its output is not rounded
    ep.round_out = B200T5_F16 ? 0 : 1;
    CU_OK(h, run_ffo_sk(h, h->sk_ffo, v.ch->tm_dh, w.tm_ffo, v.nb, d, ep, s, pdl));
  }
  return B200T5_OK;
}

// final norm, lm_head and either the fused arg-max + greedy bookkeeping or fp32 logits (teacher forcing)
static int chain_head(b200t5_ctx* h, cudaStream_t s, const ChainView& v, float* logits_out, int ldl) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  const StepMode& m = p.mode;
  const int d = c.d, T = p.Tmax;
  const bool pdl = h->use_pdl;
  CU_OK(h, run_rmsnorm(h, v.dx, h->dec_final_ln.as<act_t>(), v.dxn, v.nb, d, c.eps, s, pdl, c.out_scale));
  if (logits_out) {
    EpiStoreF32::Params ep{logits_out + static_cast<size_t>(v.b0) * ldl, ldl};
    h->launches++;
    CU_OK(h, (launch_gemm<128, EpiStoreF32>(v.ch->tm_dxn, h->tm_lm, v.nb, c.V, d, 1, ep, h->num_sms, s, pdl)));
    return B200T5_OK;
  }
  const bool sm = m.pool;
  const Plan::Results& r = p.res();
  // result rows: b0.. of the static batch's, out_row[slot] of the slot pool's
  const size_t r0 = sm ? 0 : static_cast<size_t>(v.b0);
  LmHeadParams ep{};
  ep.pval = p.pval.as<float>() + static_cast<size_t>(v.b0) * p.n_vtiles;
  ep.pidx = p.pidx.as<int>() + static_cast<size_t>(v.b0) * p.n_vtiles;
  ep.n_tiles = p.n_vtiles;
  ep.step = sm ? p.pos.as<int>() + v.b0 : &p.state.as<DecodeState>()->step;
  ep.eos = static_cast<int>(m.eos);
  ep.min_new = m.min_new;
  ep.step_stride = sm ? 1 : 0;
  if (m.proc) ep.pd = p.proc.dev(v.b0);
  FinalizeArgs fa{ep.pval, ep.pidx, p.n_vtiles, p.state.as<DecodeState>(), p.unfinished.as<int>() + v.b0,
                  r.ids.as<long long>() + r0 * (T + 1), r.len.as<int>() + r0, T + 1, m.eos, m.pad, h->shared.as<act_t>(), v.dx, d,
                  p.live_extent.as<int>() + v.b0, sm ? p.pos.as<int>() + v.b0 : nullptr, sm ? p.out_row.as<int>() + v.b0 : nullptr,
                  T, ep.pd, ScoreDev()};
  if (m.score) {
    ep.psum = p.psum.as<float>() + static_cast<size_t>(v.b0) * p.n_vtiles;
    ep.fval = p.fval.as<float>() + v.b0;
    fa.sd = {ep.psum, ep.fval, p.ftok.as<int>() + v.b0, nullptr, r.lp.as<float>() + r0 * T, r.lg.as<float>() + r0 * T};
    if (m.score == 2) {
      ep.ftok = fa.sd.ftok;
      fa.sd.forced = r.forced.as<long long>() + r0 * T;
    }
  }
  CU_OK(h, run_lm_head(h, m.proc, m.score != 0, v.ch->tm_dxn, h->tm_lm, v.nb, c.V, d, ep, fa, s, pdl));
  return B200T5_OK;
}

// The beam bookkeeping of one step, after every chain's lm_head (beam.cuh).
static int run_beam_step(b200t5_ctx* h, cudaStream_t s) {
  Plan& p = *h->plan;
  const Cfg& c = h->c;
  const int rows = p.B, prompts = p.B / p.mode.beam;
  const BeamDev bd = p.beam.dev(rows);
  DecodeState* st = p.state.as<DecodeState>();
  CU_OK(h, launch_kernel(beam_row_kernel, dim3(rows), dim3(kBeamRowThreads), 0, s, false, bd, c.V, static_cast<const DecodeState*>(st),
                         static_cast<const int*>(p.unfinished.as<int>())));
  CU_OK(h, launch_kernel(beam_select_kernel, dim3(prompts), dim3(32), 0, s, false, bd, c.V, st, p.unfinished.as<int>(),
                         p.live_extent.as<int>(), static_cast<const act_t*>(h->shared.as<act_t>()), p.dx.as<res_t>(), c.d));
  CU_OK(h, launch_kernel(beam_reorder_kernel, dim3(c.Ld * 2 * c.H, prompts), dim3(kBeamReorderThreads), 0, s, false,
                         p.self_kv.as<act_t>(), bd, static_cast<const int*>(p.unfinished.as<int>()), static_cast<const DecodeState*>(st),
                         c.H, p.Tmax, p.beam.moved.as<unsigned long long>()));
  h->launches += 3;
  return B200T5_OK;
}

// All chains of one step. `fork` (used while capturing the step graph) runs the chains on their own streams, so
// that one chain's HBM-streaming cross-attention overlaps the other chain's latency-bound GEMM phases.
static int run_decode_step(b200t5_ctx* h, cudaStream_t s, bool fork, float* logits_out, int ldl) {
  Plan& p = *h->plan;
  const Cfg& c = h->c;
  const int nc = p.n_chains;
  ChainView v[kMaxChains];
  for (int i = 0; i < nc; ++i) v[i] = chain_view(h, p.chains[i]);
  if (!logits_out && p.mode.beam) {  // beam search: the lm_head stores the fp32 logits for beam_row_kernel
    logits_out = p.beam.logits.as<float>();
    ldl = c.V;
  }
  if (fork && nc > 1) {
    cudaStream_t cs[kMaxChains];
    cs[0] = s;
    for (int i = 1; i < nc; ++i) cs[i] = h->chain_streams[i];
    CU_OK(h, cudaEventRecord(h->chain_ev[0], s));
    for (int i = 1; i < nc; ++i) CU_OK(h, cudaStreamWaitEvent(cs[i], h->chain_ev[0], 0));
    for (int l = 0; l < c.Ld; ++l) {
      for (int i = 0; i < nc; ++i) {
        TRY(chain_layer_pre(h, cs[i], v[i], l));
        TRY(chain_layer_cross(h, cs[i], v[i], l, i));
        TRY(chain_layer_post(h, cs[i], v[i], l));
      }
    }
    for (int i = 0; i < nc; ++i) {
      TRY(chain_head(h, cs[i], v[i], logits_out, ldl));
      if (i > 0) {
        CU_OK(h, cudaEventRecord(h->chain_ev[i], cs[i]));
        CU_OK(h, cudaStreamWaitEvent(s, h->chain_ev[i], 0));
      }
    }
  } else {
    for (int i = 0; i < nc; ++i) {
      for (int l = 0; l < c.Ld; ++l) {
        TRY(chain_layer_pre(h, s, v[i], l));
        TRY(chain_layer_cross(h, s, v[i], l, i));
        TRY(chain_layer_post(h, s, v[i], l));
      }
      TRY(chain_head(h, s, v[i], logits_out, ldl));
    }
  }
  if (p.mode.beam && logits_out == p.beam.logits.as<float>()) TRY(run_beam_step(h, s));
  // joins every chain; not PDL-launched so that it sees all of them complete
  CU_OK(h, launch_kernel(advance_step_kernel, dim3(1), dim3(32), 0, s, false, p.state.as<DecodeState>(),
                         h->profile_xattn ? p.xs_stamps.as<unsigned long long>() : static_cast<unsigned long long*>(nullptr),
                         h->profile_xattn ? p.xs_acc.as<unsigned long long>() : static_cast<unsigned long long*>(nullptr),
                         c.Ld, nc));
  h->launches++;
  return B200T5_OK;
}

// Graphs of one decode step and of kStepsPerGraph steps, for p.mode. The cross-attention kernel is part of the mode:
// picked here from `fill` = valid prompt tokens / (B * S) of the batch at hand.
constexpr double kXattnStreamFill = 0.9;
static bool pick_xattn(const b200t5_ctx* h, double fill) {
  return h->xattn_mode == 2 ? fill >= kXattnStreamFill : h->xattn_mode != 0;
}
static int ensure_graph(b200t5_ctx* h, double fill) {
  Plan& p = *h->plan;
  p.mode.xattn_stream = pick_xattn(h, fill);
  if (p.graph_mode == p.mode) return B200T5_OK;
  p.invalidate_graph();
  if (p.gexec) cudaGraphExecDestroy(p.gexec);
  if (p.graph) cudaGraphDestroy(p.graph);
  if (p.gexec8) cudaGraphExecDestroy(p.gexec8);
  if (p.graph8) cudaGraphDestroy(p.graph8);
  p.gexec = p.gexec8 = nullptr;
  p.graph = p.graph8 = nullptr;
  for (int which = 0; which < 2; ++which) {
    const int reps = which ? kStepsPerGraph : 1;
    cudaGraph_t* g = which ? &p.graph8 : &p.graph;
    const int64_t before = h->launches;
    CU_OK(h, cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
    int rc = B200T5_OK;
    for (int r = 0; r < reps && rc == B200T5_OK; ++r) rc = run_decode_step(h, h->cap_stream, true, nullptr, 0);
    cudaError_t e = cudaStreamEndCapture(h->cap_stream, g);
    if (!which) p.graph_nodes = static_cast<int>(h->launches - before);
    h->launches = before;
    if (rc != B200T5_OK) return rc;
    CU_OK(h, e);
    CU_OK(h, cudaGraphInstantiate(which ? &p.gexec8 : &p.gexec, *g, 0));
  }
  p.graph_mode = p.mode;
  return B200T5_OK;
}

static int validate(b200t5_ctx* h, int B, int S, const b200t5_gen_params* gp) {
  if (!h) return fail(nullptr, B200T5_EINVAL, "null handle");
  if (!h->finalized) return fail(h, B200T5_ESTATE, "model not finalized");
  if (B < 1 || S < 1 || B > 65535) return fail(h, B200T5_EINVAL, "bad batch shape B=%d S=%d", B, S);
  if (gp && (gp->max_new_tokens < 1 || gp->max_new_tokens > 4096)) return fail(h, B200T5_EINVAL, "max_new_tokens=%d out of range", gp->max_new_tokens);
  return B200T5_OK;
}

// b200t5_logits_params -> ProcHost, with transformers' argument checks (ValueError there, B200T5_EINVAL here).
// NULL, or values that change nothing (penalties 1.0, n-gram sizes 0, no ids, EOS list = {eos}), leave ph->on false.
static int parse_logits_params(b200t5_ctx* h, int V, const b200t5_logits_params* lp, long long eos, ProcHost* ph) {
  *ph = ProcHost();
  if (!lp) return B200T5_OK;
  const int W = (V + 31) / 32;
  ProcCfg& c = ph->cfg;
  ph->stat.assign(static_cast<size_t>(3) * W, 0u);
  bool on = false;
  if (!(lp->repetition_penalty > 0) || !(lp->encoder_repetition_penalty > 0))
    return fail(h, B200T5_EINVAL, "repetition penalties must be > 0 (got %g, %g)", lp->repetition_penalty, lp->encoder_repetition_penalty);
  if (lp->repetition_penalty != 1.0) {
    c.rep_pen = 1;
    c.rep_neg = static_cast<float>(lp->repetition_penalty);
    c.rep_pos = static_cast<float>(1.0 / lp->repetition_penalty);
    on = true;
  }
  if (lp->encoder_repetition_penalty != 1.0) {
    c.enc_pen = 1;
    const double pe = 1.0 / lp->encoder_repetition_penalty;  // transformers stores the encoder penalty inverted
    c.enc_neg = static_cast<float>(pe);
    c.enc_pos = static_cast<float>(1.0 / pe);
    on = true;
  }
  if (lp->no_repeat_ngram_size < 0 || lp->encoder_no_repeat_ngram_size < 0)
    return fail(h, B200T5_EINVAL, "n-gram sizes must be >= 0");
  c.ngram = lp->no_repeat_ngram_size;
  c.enc_ngram = lp->encoder_no_repeat_ngram_size;
  on = on || c.ngram > 0 || c.enc_ngram > 0;
  auto mark = [&](int which, const int32_t* ids, int n, const char* what) -> int {
    if (n < 0 || (n > 0 && !ids)) return fail(h, B200T5_EINVAL, "bad %s list", what);
    for (int i = 0; i < n; ++i) {
      if (ids[i] < 0 || ids[i] >= V) return fail(h, B200T5_EINVAL, "%s id %d outside [0, %d)", what, ids[i], V);
      ph->stat[static_cast<size_t>(which) * W + (ids[i] >> 5)] |= 1u << (ids[i] & 31);
      on = true;
    }
    return B200T5_OK;
  };
  TRY(mark(0, lp->suppress_tokens, lp->n_suppress_tokens, "suppress_tokens"));
  TRY(mark(1, lp->begin_suppress_tokens, lp->n_begin_suppress_tokens, "begin_suppress_tokens"));
  if (lp->n_eos_token_ids < 0 || lp->n_eos_token_ids > kProcMaxEos || (lp->n_eos_token_ids > 0 && !lp->eos_token_ids))
    return fail(h, B200T5_EINVAL, "eos_token_ids: 0..%d ids", kProcMaxEos);
  if (lp->n_eos_token_ids == 0) {
    if (eos >= 0 && eos < V) c.eos[c.n_eos++] = static_cast<int>(eos);
  } else {
    for (int i = 0; i < lp->n_eos_token_ids; ++i) {
      const int e = lp->eos_token_ids[i];
      if (e < 0 || e >= V) return fail(h, B200T5_EINVAL, "eos id %d outside [0, %d)", e, V);
      if (e != eos) on = true;
      c.eos[c.n_eos++] = e;
    }
  }
  for (int i = 0; i < c.n_eos; ++i) ph->stat[static_cast<size_t>(2) * W + (c.eos[i] >> 5)] |= 1u << (c.eos[i] & 31);
  const int nb = lp->n_bad_words;
  if (nb < 0 || (nb > 0 && (!lp->bad_words_ids || !lp->bad_words_offsets)) || (nb > 0 && lp->bad_words_offsets[0] != 0))
    return fail(h, B200T5_EINVAL, "bad_words: bad offsets");
  for (int i = 0; i < nb; ++i) {
    const int lo = lp->bad_words_offsets[i], hi = lp->bad_words_offsets[i + 1];
    if (hi <= lo) return fail(h, B200T5_EINVAL, "bad_words: sequence %d is empty", i);
    for (int k = lo; k < hi; ++k)
      if (lp->bad_words_ids[k] < 0 || lp->bad_words_ids[k] >= V)
        return fail(h, B200T5_EINVAL, "bad_words: id %d outside [0, %d)", lp->bad_words_ids[k], V);
    if (hi - lo == 1) {
      const int tok = lp->bad_words_ids[lo];
      bool is_eos = false;
      for (int q = 0; q < c.n_eos; ++q) is_eos = is_eos || c.eos[q] == tok;
      if (is_eos) continue;  // transformers drops [eos] from bad_words_ids
      ph->stat[tok >> 5] |= 1u << (tok & 31);
    } else {
      if (ph->bad_off.empty()) ph->bad_off.push_back(0);
      ph->bad_ids.insert(ph->bad_ids.end(), lp->bad_words_ids + lo, lp->bad_words_ids + hi);
      ph->bad_off.push_back(static_cast<int>(ph->bad_ids.size()));
    }
    c.bad_add = 1;
    on = true;
  }
  c.n_bad = ph->bad_off.empty() ? 0 : static_cast<int>(ph->bad_off.size()) - 1;
  ph->on = on;
  return B200T5_OK;
}

// Make the plan's processor state fit this call and queue its values on `s` (before the step graph is captured or
// launched). A reallocation drops the step graph, which bakes the addresses.
static int setup_proc(b200t5_ctx* h, const ProcHost& ph, cudaStream_t s) {
  Plan& p = *h->plan;
  if (!ph.on) return B200T5_OK;
  const int W = (h->c.V + 31) / 32;
  const int cap = std::min(W * 32, p.Tmax + 1 + p.S + ph.cfg.n_bad);  // distinct bans of one step, at most
  if (!p.proc.fits(p.B, p.S, W, cap, ph.bad_ids.size(), ph.bad_off.size())) {
    CU_OK(h, cudaStreamSynchronize(s));
    CU_OK(h, p.proc.alloc(p.B, p.S, W, std::max(cap, p.proc.ban_cap), std::max<size_t>(ph.bad_ids.size(), 2 * p.proc.n_bad_ids),
                          std::max<size_t>(ph.bad_off.size(), 2 * p.proc.n_bad_off)));
    p.invalidate_graph();
  }
  CU_OK(h, p.proc.upload(ph, s));
  return B200T5_OK;
}

// b200t5_score_io -> ScoreHost for a call of `rows` rows and T = max_new_tokens. `host`: the struct's pointers are
// host pointers (else device pointers: the labels are read back to be checked). The destinations are set by the
// caller, which knows where the results must go.
static int parse_score(b200t5_ctx* h, const b200t5_score_io* sc, long long rows, int T, bool host, bool proc, ScoreHost* sh) {
  *sh = ScoreHost();
  if (!sc) return B200T5_OK;
  if (!sc->token_logprobs) return fail(h, B200T5_EINVAL, "score: token_logprobs is NULL");
  sh->on = true;
  if (!sc->forced_ids) return B200T5_OK;
  const int L = sc->forced_len;
  if (L < 1 || L > T) return fail(h, B200T5_EINVAL, "score: forced_len=%d outside [1, max_new_tokens=%d]", L, T);
  if (proc) return fail(h, B200T5_EINVAL, "score: forced_ids cannot be combined with logits processors");
  std::vector<long long> f(static_cast<size_t>(rows) * L);
  if (host) memcpy(f.data(), sc->forced_ids, f.size() * 8);
  else CU_OK(h, cudaMemcpy(f.data(), sc->forced_ids, f.size() * 8, cudaMemcpyDeviceToHost));
  sh->forced.assign(static_cast<size_t>(rows) * T, -100);
  for (long long r = 0; r < rows; ++r) {
    bool ended = false;
    for (int t = 0; t < L; ++t) {
      const long long v = f[static_cast<size_t>(r) * L + t];
      if (v == -100) {
        if (t == 0) return fail(h, B200T5_EINVAL, "score: row %lld of forced_ids has no label", r);
        ended = true;
        continue;
      }
      if (v < 0 || v >= h->c.V) return fail(h, B200T5_EINVAL, "score: forced id %lld outside [0, %d)", v, h->c.V);
      if (ended) return fail(h, B200T5_EINVAL, "score: row %lld of forced_ids has a label after -100", r);
      sh->forced[static_cast<size_t>(r) * T + t] = v;
    }
  }
  return B200T5_OK;
}

// Make the scoring buffers of the call's results (p.res(): the batch, or the slot pool at its capacity) fit this call
// and queue the labels on `s`. A new allocation drops the step graph, which bakes the addresses.
static int setup_score(b200t5_ctx* h, const ScoreHost& sh, cudaStream_t s) {
  Plan& p = *h->plan;
  if (!sh.on) return B200T5_OK;
  Plan::Results& r = p.res();
  const size_t n = r.cap * p.Tmax;
  if (!p.psum.p || !r.forced.p || r.forced.bytes != n * 8) {
    CU_OK(h, cudaStreamSynchronize(s));
    if (!p.psum.p) {
      CU_OK(h, p.psum.alloc(static_cast<size_t>(p.B) * p.n_vtiles * 4));
      CU_OK(h, p.fval.alloc(static_cast<size_t>(p.B) * 4));
      CU_OK(h, p.ftok.alloc(static_cast<size_t>(p.B) * 4));
      CU_OK(h, cudaMemset(p.fval.p, 0, p.fval.bytes));
    }
    CU_OK(h, r.lp.alloc(n * 4));
    CU_OK(h, r.lg.alloc(n * 4));
    CU_OK(h, r.forced.alloc(n * 8));
    p.invalidate_graph();
  }
  if (!sh.forced.empty()) CU_OK(h, cudaMemcpyAsync(r.forced.p, sh.forced.data(), sh.forced.size() * 8, cudaMemcpyHostToDevice, s));
  return B200T5_OK;
}

static void fill_stats_model(b200t5_ctx* h, int steps) {
  const Cfg& c = h->c;
  const Plan& p = *h->plan;
  // SURVEY 8(d): weights once per step + cross-KV + self-KV read/write, bf16.
  // (element count; the fp16 build's `wo` weights are fp32: counted twice)
  // feed-forward F x d matrices per layer: wi_0, wi_1, wo (gated-GELU) or wi, wo (ReLU)
  const double ff_mats = c.gated ? 3.0 : 2.0;
  const double wstep = static_cast<double>(c.Ld) * (6.0 * c.d * c.I + (ff_mats + (B200T5_F16 ? 1.0 : 0.0)) * c.d * c.F) +
                       static_cast<double>(c.V) * c.d;
  std::vector<int> ext(p.B, p.S);
  if (cudaMemcpy(ext.data(), p.extent.p, p.B * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
    ext.assign(p.B, p.S);  // statistics only: fall back to the padded length
  double sum_s = 0;
  for (int v : ext) sum_s += v;
  double bytes = 0;
  for (int t = 1; t <= steps; ++t)
    bytes += 2.0 * (wstep + static_cast<double>(c.Ld) * 2 * c.I * sum_s + static_cast<double>(c.Ld) * 2 * c.I * p.B * t +
                    static_cast<double>(c.Ld) * 2 * c.I * p.B);
  h->last_decode_bytes = bytes;
  // encoder + cross-KV projection FLOPs of the rows that matter (positions below extent[b]); for full-length
  // prompts this is SURVEY 8(d)'s figure, for padded ones it is the work the packed encoder actually does
  double sum_s2 = 0;
  for (int v : ext) sum_s2 += static_cast<double>(v) * v;
  h->last_enc_flops = 2.0 * c.Le * (4.0 * c.d * c.I + ff_mats * c.d * c.F) * sum_s + c.Le * 4.0 * sum_s2 * c.I +
                      2.0 * c.Ld * 2.0 * c.d * c.I * sum_s;
}

// A generate call's arguments after set_up_call: the special tokens and sizes every path resolves from them, the logits
// processors and the scoring request.
struct CallArgs {
  long long eos = 0, pad = 0, start = 0;
  int T = 0, min_new = 0;
  int first = 0;  // the first generated position: P - 1 after a decoder prompt of P ids, else 0
  ProcHost ph;
  ScoreHost sh;
  // The step mode of this call. A beam call's min_new_tokens lives in its BeamParams, not in the graph. The EOS mask
  // runs while step < first + min_new: after a decoder prompt the offset is baked into the graph, so a call with
  // another prompt length (and min_new_tokens > 0) re-captures it.
  StepMode mode(bool pool, int beam = 0) const {
    StepMode m;
    m.eos = eos;
    m.pad = pad;
    m.min_new = beam ? 0 : (min_new > 0 ? first + min_new : 0);
    m.pool = pool;
    m.proc = ph.on;
    m.score = sh.on ? (sh.forced.empty() ? 1 : 2) : 0;
    m.beam = beam;
    return m;
  }
};

// Checks a call of B rows (the slot pool: B slots) for `rows` prompts and resolves what it asks for. `host`: the pointers
// in `score` are host pointers.
static int set_up_call(b200t5_ctx* h, int B, int S, long long rows, const b200t5_gen_params* gp, const void* input_ids,
                       const void* out_ids, const void* out_len, const b200t5_logits_params* logits,
                       const b200t5_score_io* score, bool host, CallArgs* a) {
  TRY(validate(h, B, S, gp));
  if (!gp || !input_ids || !out_ids || !out_len) return fail(h, B200T5_EINVAL, "null argument");
  const Cfg& c = h->c;
  a->eos = gp->eos_token_id >= 0 ? gp->eos_token_id : c.eos;
  a->pad = gp->pad_token_id >= 0 ? gp->pad_token_id : c.pad;
  a->start = gp->decoder_start_token_id >= 0 ? gp->decoder_start_token_id : c.start;
  a->T = gp->max_new_tokens;
  a->min_new = gp->min_new_tokens > 0 ? gp->min_new_tokens : 0;
  TRY(parse_logits_params(h, c.V, logits, a->eos, &a->ph));
  CU_OK(h, cudaSetDevice(h->device));
  TRY(parse_score(h, score, rows, a->T, host, a->ph.on, &a->sh));
  if (a->start >= c.V || a->pad >= c.V) return fail(h, B200T5_EINVAL, "special token id out of range");
  return B200T5_OK;
}

// Queues the copy of the first n rows of the call's results (p.res()) to ids / len and, for a scored call, to lp / lg
// (lg may be NULL). `col0`: the scores start at column col0 of the plan's [rows][Tmax] arrays (a decoder prompt's
// first generated position) and are copied as [n][Tmax - col0].
static int copy_results(b200t5_ctx* h, size_t n, void* ids, void* len, void* lp, void* lg, cudaMemcpyKind kind, cudaStream_t s,
                        int col0 = 0) {
  Plan& p = *h->plan;
  const Plan::Results& r = p.res();
  const size_t T = static_cast<size_t>(p.Tmax);
  CU_OK(h, cudaMemcpyAsync(ids, r.ids.p, n * (T + 1) * 8, kind, s));
  CU_OK(h, cudaMemcpyAsync(len, r.len.p, n * 4, kind, s));
  if (p.mode.score && col0 > 0) {
    const size_t w = (T - col0) * 4;
    CU_OK(h, cudaMemcpy2DAsync(lp, w, r.lp.as<float>() + col0, T * 4, w, n, kind, s));
    if (lg) CU_OK(h, cudaMemcpy2DAsync(lg, w, r.lg.as<float>() + col0, T * 4, w, n, kind, s));
  } else if (p.mode.score) {
    CU_OK(h, cudaMemcpyAsync(lp, r.lp.p, n * T * 4, kind, s));
    if (lg) CU_OK(h, cudaMemcpyAsync(lg, r.lg.p, n * T * 4, kind, s));
  }
  return B200T5_OK;
}

// The start of a static batch's decoding, after its encoder pass: the decode kernels attend to live copies of extent /
// key_ok, and every row starts from the start token (`prompt`: from the decoder prompt [B][P] on the device).
static int begin_static_decode(b200t5_ctx* h, const CallArgs& a, cudaStream_t s, const long long* prompt = nullptr, int P = 1) {
  Plan& p = *h->plan;
  const int B = p.B;
  CU_OK(h, cudaMemcpyAsync(p.live_extent.p, p.extent.p, static_cast<size_t>(B) * 4, cudaMemcpyDeviceToDevice, s));
  CU_OK(h, cudaMemcpyAsync(p.live_key_ok.p, p.key_ok.p, static_cast<size_t>(B) * p.S, cudaMemcpyDeviceToDevice, s));
  if (prompt) {
    decode_init_prompt_kernel<<<B, 128, 0, s>>>(p.state.as<DecodeState>(), p.unfinished.as<int>(), p.batch.ids.as<long long>(),
                                                p.batch.len.as<int>(), p.Tmax + 1, B, prompt, P, a.pad, h->shared.as<act_t>(),
                                                p.dx.as<res_t>(), h->c.d);
    h->launches++;
    return B200T5_OK;
  }
  decode_init_kernel<<<B, 128, 0, s>>>(p.state.as<DecodeState>(), p.unfinished.as<int>(), p.batch.ids.as<long long>(),
                                       p.batch.len.as<int>(), a.T + 1, B, a.start, a.pad, h->shared.as<act_t>(), p.dx.as<res_t>(),
                                       h->c.d);
  h->launches++;
  return B200T5_OK;
}

// The T decode steps of a static batch, from the end of its encoder pass (ev[1]) to ev[2]. `early_exit`: stop at a
// poll once every row has finished.
static int run_static_steps(b200t5_ctx* h, const b200t5_gen_params* gp, int T, bool early_exit, cudaStream_t s) {
  Plan& p = *h->plan;
  const int poll = gp->poll_interval > 0 ? gp->poll_interval : 8;
  CU_OK(h, cudaGetLastError());
  CU_OK(h, cudaEventRecord(h->ev[1], s));
  int steps = 0;
  for (int t = 0; t < T; ++t) {
    if (t % kStepsPerGraph == 0 && t + kStepsPerGraph <= T && poll % kStepsPerGraph == 0) {
      // eight steps in one launch; the early-exit poll below happens on the same boundaries
      CU_OK(h, cudaGraphLaunch(p.gexec8, s));
      h->launches += static_cast<int64_t>(p.graph_nodes) * kStepsPerGraph;
      steps += kStepsPerGraph;
      t += kStepsPerGraph - 1;
    } else {
      CU_OK(h, cudaGraphLaunch(p.gexec, s));
      h->launches += p.graph_nodes;
      ++steps;
    }
    if ((t + 1) % poll == 0 && t + 1 < T && early_exit) {
      // every row finished (greedy: emitted EOS; beam: its prompt retired) -> the remaining steps would change nothing
      CU_OK(h, cudaMemcpyAsync(p.h_state, p.state.p, sizeof(DecodeState), cudaMemcpyDeviceToHost, s));
      CU_OK(h, cudaStreamSynchronize(s));
      if (p.h_state->finished_rows >= p.B) break;
    }
  }
  CU_OK(h, cudaEventRecord(h->ev[2], s));
  h->last_steps = steps;
  h->ev_valid = true;
  return B200T5_OK;
}

// A static batch of B rows; its results stay in the plan's buffers (copy_results).
static int generate_impl(b200t5_ctx* h, const long long* ids, const long long* mask, int B, int S, const b200t5_gen_params* gp,
                         const CallArgs& a, cudaStream_t s) {
  const int T = a.T;
  TRY(ensure_plan(h, B, S, T));
  Plan& p = *h->plan;
  p.mode = a.mode(false);
  TRY(setup_proc(h, a.ph, s));
  TRY(setup_score(h, a.sh, s));
  h->launches = 0;
  CU_OK(h, cudaEventRecord(h->ev[0], s));
  TRY(run_encoder(h, ids, mask, s));
  TRY(run_cross_kv(h, s));
  // (host-side capture, only when something baked into the graph changed; the GPU is busy with the encoder meanwhile)
  TRY(ensure_graph(h, static_cast<double>(p.rows_valid) / (static_cast<double>(B) * S)));
  TRY(begin_static_decode(h, a, s));
  if (p.mode.proc) {
    proc_reset_kernel<<<B, 128, 0, s>>>(p.proc.dev(), nullptr, ids, p.batch.ids.as<long long>(), T + 1, nullptr, 1);
    h->launches++;
  }
  if (p.mode.score) {
    score_reset_kernel<<<B, 128, 0, s>>>(p.batch.lp.as<float>(), p.batch.lg.as<float>(), static_cast<size_t>(B) * T, p.ftok.as<int>(),
                                         B, nullptr, nullptr, p.mode.score == 2 ? p.batch.forced.as<long long>() : nullptr, T);
    h->launches++;
  }
  return run_static_steps(h, gp, T, a.min_new < T, s);
}

extern "C" int b200t5_generate_scored(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                      const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                                      int32_t* out_len, const b200t5_score_io* score, void* stream) {
  CallArgs a;
  TRY(set_up_call(h, B, S, B, params, input_ids, out_ids, out_len, logits, score, false, &a));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TRY(generate_impl(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask), B, S,
                    params, a, s));
  return copy_results(h, static_cast<size_t>(B), out_ids, out_len, a.sh.on ? score->token_logprobs : nullptr,
                      a.sh.on ? score->token_logits : nullptr, cudaMemcpyDeviceToDevice, s);
}

extern "C" int b200t5_generate_ex(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                  const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                                  int32_t* out_len, void* stream) {
  return b200t5_generate_scored(h, input_ids, attention_mask, B, S, params, logits, out_ids, out_len, nullptr, stream);
}

extern "C" int b200t5_generate(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                               const b200t5_gen_params* params, int64_t* out_ids, int32_t* out_len, void* stream) {
  return b200t5_generate_ex(h, input_ids, attention_mask, B, S, params, nullptr, out_ids, out_len, stream);
}

extern "C" int b200t5_generate_host(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B,
                                    int S, const b200t5_gen_params* params, int64_t* out_ids, int32_t* out_len) {
  return b200t5_generate_host_ex(h, input_ids, attention_mask, B, S, params, nullptr, out_ids, out_len);
}

extern "C" int b200t5_generate_host_ex(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B,
                                       int S, const b200t5_gen_params* params, const b200t5_logits_params* logits,
                                       int64_t* out_ids, int32_t* out_len) {
  return b200t5_generate_host_scored(h, input_ids, attention_mask, B, S, params, logits, out_ids, out_len, nullptr);
}

extern "C" int b200t5_generate_host_scored(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B,
                                           int S, const b200t5_gen_params* params, const b200t5_logits_params* logits,
                                           int64_t* out_ids, int32_t* out_len, const b200t5_score_io* score) {
  CallArgs a;
  TRY(set_up_call(h, B, S, B, params, input_ids, out_ids, out_len, logits, score, true, &a));
  TRY(ensure_plan(h, B, S, a.T));
  Plan& p = *h->plan;
  cudaStream_t s = h->exec_stream;
  const size_t nb = static_cast<size_t>(B) * S * 8;
  memcpy(p.h_ids, input_ids, nb);
  CU_OK(h, cudaMemcpyAsync(p.ids_dev.p, p.h_ids, nb, cudaMemcpyHostToDevice, s));
  if (attention_mask) {
    memcpy(p.h_mask, attention_mask, nb);
    CU_OK(h, cudaMemcpyAsync(p.mask_dev.p, p.h_mask, nb, cudaMemcpyHostToDevice, s));
  }
  TRY(generate_impl(h, p.ids_dev.as<long long>(), attention_mask ? p.mask_dev.as<long long>() : nullptr, B, S, params, a, s));
  // ids and lengths through the pinned staging
  TRY(copy_results(h, static_cast<size_t>(B), p.h_out, p.h_len, a.sh.on ? score->token_logprobs : nullptr,
                   a.sh.on ? score->token_logits : nullptr, cudaMemcpyDeviceToHost, s));
  CU_OK(h, cudaStreamSynchronize(s));
  memcpy(out_ids, p.h_out, static_cast<size_t>(B) * (a.T + 1) * 8);
  memcpy(out_len, p.h_len, static_cast<size_t>(B) * 4);
  return B200T5_OK;
}

// ================================================================== beam search
// A beam call's parameters, for B prompts.
static int parse_beam(b200t5_ctx* h, const b200t5_beam_params* bp, int B) {
  if (!bp) return fail(h, B200T5_EINVAL, "null beam params");
  if (bp->num_beams < 2 || bp->num_beams > kBeamMax) return fail(h, B200T5_EINVAL, "num_beams=%d outside [2, %d]", bp->num_beams, kBeamMax);
  if (bp->num_return_sequences < 1 || bp->num_return_sequences > bp->num_beams)
    return fail(h, B200T5_EINVAL, "num_return_sequences=%d outside [1, num_beams=%d]", bp->num_return_sequences, bp->num_beams);
  if (bp->early_stopping < 0 || bp->early_stopping > 2) return fail(h, B200T5_EINVAL, "early_stopping=%d outside {0, 1, 2}", bp->early_stopping);
  if (!std::isfinite(bp->length_penalty)) return fail(h, B200T5_EINVAL, "length_penalty is not finite");
  const int rows = B * bp->num_beams;
  if (rows > 65535) return fail(h, B200T5_EINVAL, "B * num_beams = %d rows is too many", rows);
  return B200T5_OK;
}

// The plan's beam state and result staging, sized by the plan (B = prompts * k rows, Tmax): allocated once per plan.
static int ensure_beam_bufs(b200t5_ctx* h, Plan& p) {
  BeamBufs& b = p.beam;
  if (b.prm.p) return B200T5_OK;
  const size_t rows = static_cast<size_t>(p.B), T = static_cast<size_t>(p.Tmax), prompts = rows / p.group;
  CU_OK(h, b.seq.alloc(rows * (T + 1) * 8));
  CU_OK(h, b.len.alloc(rows * 4));
  CU_OK(h, b.score.alloc(rows * 4));
  CU_OK(h, b.bidx.alloc(rows * T * 8));
  CU_OK(h, b.lp.alloc(rows * T * 4));
  CU_OK(h, b.logits.alloc(rows * h->c.V * 4));
  CU_OK(h, b.cand_lp.alloc(rows * kBeamCand * 4));
  CU_OK(h, b.cand_tok.alloc(rows * kBeamCand * 4));
  CU_OK(h, b.run_score.alloc(rows * 4));
  CU_OK(h, b.hist_par.alloc(T * rows * 4));
  CU_OK(h, b.hist_tok.alloc(T * rows * 4));
  CU_OK(h, b.hist_lp.alloc(T * rows * 4));
  CU_OK(h, b.fin.alloc(prompts * kBeamMax * sizeof(BeamFin)));
  CU_OK(h, b.heur.alloc(prompts * 4));
  CU_OK(h, b.parent.alloc(rows * 4));
  CU_OK(h, b.len_scale.alloc(T * 4));
  CU_OK(h, b.moved.alloc(8));
  CU_OK(h, b.prm.alloc(sizeof(BeamParams)));
  p.invalidate_graph();
  return B200T5_OK;
}

// fp32(1 / (l ** length_penalty)) for l = 1..T, the reciprocal taken in double (oracle/beam.py: length_scale)
static std::vector<float> beam_len_scale(double length_penalty, int T) {
  std::vector<float> v(T);
  for (int l = 1; l <= T; ++l) v[l - 1] = static_cast<float>(1.0 / pow(static_cast<double>(l), length_penalty));
  return v;
}

// A static batch of B prompts as B * k decode rows; the results stay in the plan's beam state (beam_output_kernel).
// `ids` / `mask` are device buffers, or host buffers with kind = cudaMemcpyHostToDevice.
static int generate_beam_impl(b200t5_ctx* h, const long long* ids, const long long* mask, cudaMemcpyKind kind, int Bp, int S,
                              const b200t5_gen_params* gp, const b200t5_beam_params* bp, const CallArgs& a, cudaStream_t s) {
  const Cfg& c = h->c;
  const int T = a.T, k = bp->num_beams, rows = Bp * k;
  TRY(ensure_plan(h, rows, S, T, k));
  Plan& p = *h->plan;
  p.mode = a.mode(false, k);
  TRY(ensure_beam_bufs(h, p));
  const BeamDev bd = p.beam.dev(rows);
  const BeamParams prm{k, T, a.min_new, static_cast<int>(a.eos), bp->early_stopping, bp->early_stopping == 2 && bp->length_penalty > 0.0};
  const std::vector<float> ls = beam_len_scale(bp->length_penalty, T);
  CU_OK(h, cudaMemcpyAsync(p.beam.prm.p, &prm, sizeof(prm), cudaMemcpyHostToDevice, s));
  CU_OK(h, cudaMemcpyAsync(p.beam.len_scale.p, ls.data(), ls.size() * 4, cudaMemcpyHostToDevice, s));
  h->launches = 0;
  CU_OK(h, cudaEventRecord(h->ev[0], s));
  // The encoder runs on row b*k of each prompt only (the other rows have extent 0 in its pass, as in a slot-pool
  // admission); beam_replicate_kernel then gives the prompt's other rows its cross-attention K/V. The unpacked encoder
  // (S > kEncPackMaxS) takes no such row selection and runs every row.
  const bool packed = S <= kEncPackMaxS;
  const size_t rb = static_cast<size_t>(S) * 8;
  for (int j = 0; j < (packed ? 1 : k); ++j) {
    CU_OK(h, cudaMemcpy2DAsync(p.ids_dev.as<long long>() + static_cast<size_t>(j) * S, k * rb, ids, rb, rb, Bp, kind, s));
    if (mask) CU_OK(h, cudaMemcpy2DAsync(p.mask_dev.as<long long>() + static_cast<size_t>(j) * S, k * rb, mask, rb, rb, Bp, kind, s));
  }
  const int* row_on = nullptr;
  if (packed) {
    for (int r = 0; r < rows; ++r) p.h_admit[r] = r % k == 0;
    CU_OK(h, cudaMemcpyAsync(p.admit.p, p.h_admit, static_cast<size_t>(rows) * 4, cudaMemcpyHostToDevice, s));
    row_on = p.admit.as<int>();
  }
  TRY(run_encoder(h, p.ids_dev.as<long long>(), mask ? p.mask_dev.as<long long>() : nullptr, s, row_on));
  TRY(run_cross_kv(h, s));
  if (packed) {
    beam_replicate_kernel<<<dim3(c.Ld * 2 * c.H, rows), 256, 0, s>>>(p.cross_kv.as<act_t>(), p.extent.as<int>(), p.key_ok.as<unsigned char>(),
                                                                     rows, k, c.H, S);
    h->launches++;
  }
  const double valid = packed ? static_cast<double>(p.rows_valid) * k : static_cast<double>(p.rows_valid);
  TRY(ensure_graph(h, valid / (static_cast<double>(rows) * S)));
  TRY(begin_static_decode(h, a, s));
  beam_init_kernel<<<(std::max(rows, Bp * kBeamMax) + 255) / 256, 256, 0, s>>>(bd, Bp, k);
  h->launches++;
  CU_OK(h, cudaMemsetAsync(p.beam.moved.p, 0, 8, s));
  // a beam row finishes when its prompt retires: the prompt's finished set can no longer change
  return run_static_steps(h, gp, T, true, s);
}

static int beam_output(b200t5_ctx* h, int Bp, const b200t5_beam_params* bp, long long start, long long pad, int64_t* seq, int32_t* len,
                       float* sc, int64_t* bidx, float* lp, cudaStream_t s) {
  Plan& p = *h->plan;
  const int n = Bp * bp->num_return_sequences;
  beam_output_kernel<<<(n + 127) / 128, 128, 0, s>>>(p.beam.dev(p.B), Bp, bp->num_return_sequences, reinterpret_cast<long long*>(seq), len, sc,
                                                     reinterpret_cast<long long*>(bidx), lp, start, pad);
  h->launches++;
  CU_OK(h, cudaGetLastError());
  return B200T5_OK;
}

extern "C" int b200t5_generate_beam(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                    const b200t5_gen_params* params, const b200t5_beam_params* beam, const b200t5_beam_io* io,
                                    void* stream) {
  CallArgs a;
  if (!io) return fail(h, B200T5_EINVAL, "null beam io");
  TRY(set_up_call(h, B, S, B, params, input_ids, io->sequences, io->lengths, nullptr, nullptr, false, &a));
  TRY(parse_beam(h, beam, B));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TRY(generate_beam_impl(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask),
                         cudaMemcpyDeviceToDevice, B, S, params, beam, a, s));
  return beam_output(h, B, beam, a.start, a.pad, io->sequences, io->lengths, io->sequences_scores, io->beam_indices, io->token_logprobs, s);
}

extern "C" int b200t5_generate_host_beam(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                         const b200t5_gen_params* params, const b200t5_beam_params* beam, const b200t5_beam_io* io) {
  CallArgs a;
  if (!io) return fail(h, B200T5_EINVAL, "null beam io");
  TRY(set_up_call(h, B, S, B, params, input_ids, io->sequences, io->lengths, nullptr, nullptr, true, &a));
  TRY(parse_beam(h, beam, B));
  cudaStream_t s = h->exec_stream;
  TRY(ensure_plan(h, B * beam->num_beams, S, a.T, beam->num_beams));
  Plan& p = *h->plan;
  // the prompts through the pinned staging; the results through the plan's beam buffers
  const size_t nb = static_cast<size_t>(B) * S * 8;
  memcpy(p.h_ids, input_ids, nb);
  if (attention_mask) memcpy(p.h_mask, attention_mask, nb);
  TRY(generate_beam_impl(h, p.h_ids, attention_mask ? p.h_mask : nullptr, cudaMemcpyHostToDevice, B, S, params, beam, a, s));
  const BeamBufs& o = p.beam;
  TRY(beam_output(h, B, beam, a.start, a.pad, o.seq.as<int64_t>(), o.len.as<int32_t>(), o.score.as<float>(), o.bidx.as<int64_t>(),
                  o.lp.as<float>(), s));
  const size_t n = static_cast<size_t>(B) * beam->num_return_sequences, T = static_cast<size_t>(a.T);
  CU_OK(h, cudaMemcpyAsync(io->sequences, o.seq.p, n * (T + 1) * 8, cudaMemcpyDeviceToHost, s));
  CU_OK(h, cudaMemcpyAsync(io->lengths, o.len.p, n * 4, cudaMemcpyDeviceToHost, s));
  if (io->sequences_scores) CU_OK(h, cudaMemcpyAsync(io->sequences_scores, o.score.p, n * 4, cudaMemcpyDeviceToHost, s));
  if (io->beam_indices) CU_OK(h, cudaMemcpyAsync(io->beam_indices, o.bidx.p, n * T * 8, cudaMemcpyDeviceToHost, s));
  if (io->token_logprobs) CU_OK(h, cudaMemcpyAsync(io->token_logprobs, o.lp.p, n * T * 4, cudaMemcpyDeviceToHost, s));
  CU_OK(h, cudaStreamSynchronize(s));
  return B200T5_OK;
}

extern "C" int b200t5_get_beam_stats(b200t5_handle h, double* reorder_bytes, int32_t* steps) {
  if (!h || !reorder_bytes || !steps) return fail(h, B200T5_EINVAL, "null argument");
  if (!h->plan || !h->plan->beam.moved.p) return fail(h, B200T5_ESTATE, "no beam call yet");
  unsigned long long v = 0;
  CU_OK(h, cudaMemcpy(&v, h->plan->beam.moved.p, 8, cudaMemcpyDeviceToHost));
  *reorder_bytes = static_cast<double>(v);
  *steps = h->last_steps;
  return B200T5_OK;
}

// ================================================================== slot pool (continuous batching)
// N prompts through a pool of `pool` decode slots. A slot whose row has finished (EOS or max_new tokens) is
// retired at the next poll and refilled with the next prompt: an encoder pass over the newly admitted prompts
// only (packed rows; every other slot has extent 0 in that pass) writes their cross-KV into the slots' arena
// rows, then the same step graph as the static path runs with per-slot positions. Rows are independent in every
// kernel, so a prompt's tokens are bit-identical to what b200t5_generate returns for it in a `pool`-row batch.
// Replaces, for a caller that hands over more than one batch at a time, the per-batch generate() of
// predictor.py:102 under BatchPredictor.predict (NB:908-913): finished rows stop costing bandwidth and the
// pool stays full instead of draining to the slowest row of each 256-row batch.
extern "C" int b200t5_generate_stream(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int64_t N,
                                      int S, const b200t5_gen_params* gp, int pool, int admit_min, int64_t* out_ids,
                                      int32_t* out_len) {
  return b200t5_generate_stream_ex(h, input_ids, attention_mask, N, S, gp, nullptr, pool, admit_min, out_ids, out_len);
}

extern "C" int b200t5_generate_stream_ex(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int64_t N,
                                         int S, const b200t5_gen_params* gp, const b200t5_logits_params* logits, int pool,
                                         int admit_min, int64_t* out_ids, int32_t* out_len) {
  return b200t5_generate_stream_scored(h, input_ids, attention_mask, N, S, gp, logits, pool, admit_min, out_ids, out_len, nullptr);
}

extern "C" int b200t5_generate_stream_scored(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int64_t N,
                                             int S, const b200t5_gen_params* gp, const b200t5_logits_params* logits, int pool,
                                             int admit_min, int64_t* out_ids, int32_t* out_len, const b200t5_score_io* score) {
  if (N < 1 || N > (1ll << 30)) return fail(h, B200T5_EINVAL, "bad prompt count N=%lld", static_cast<long long>(N));
  if (pool < 1) pool = 256;
  if (pool > N) pool = static_cast<int>(N);
  CallArgs a;
  TRY(set_up_call(h, pool, S, N, gp, input_ids, out_ids, out_len, logits, score, true, &a));
  const Cfg& c = h->c;
  const int T = a.T;
  const int B = pool;
  if (admit_min < 1) admit_min = B >= 8 ? B / 8 : 1;
  const int poll = gp->poll_interval > 0 ? (gp->poll_interval > 64 ? 64 : gp->poll_interval) : kStepsPerGraph;
  TRY(ensure_plan(h, B, S, T));
  Plan& p = *h->plan;
  p.mode = a.mode(true);
  cudaStream_t s = h->exec_stream;
  Plan::Results& r = p.pool;
  if (r.cap < static_cast<size_t>(N)) {
    // the step graph bakes the result addresses: a larger result buffer means a new graph
    CU_OK(h, cudaStreamSynchronize(s));
    size_t cap = r.cap ? r.cap : 1024;
    while (cap < static_cast<size_t>(N)) cap *= 2;
    CU_OK(h, r.ids.alloc(cap * (T + 1) * 8));
    CU_OK(h, r.len.alloc(cap * 4));
    r.cap = cap;
    p.invalidate_graph();
  }
  TRY(setup_proc(h, a.ph, s));
  TRY(setup_score(h, a.sh, s));
  double fill = 1.0;
  if (attention_mask) {  // fill of the first prompts (up to four pools' worth): picks the cross-attention kernel
    const long long rows = N < 4LL * B ? N : 4LL * B;
    long long ones = 0;
    for (long long i = 0; i < rows * S; ++i) ones += attention_mask[i] != 0;
    fill = static_cast<double>(ones) / static_cast<double>(rows * S);
  }
  TRY(ensure_graph(h, fill));
  h->launches = 0;
  CU_OK(h, cudaEventRecord(h->ev[0], s));
  {
    const long long rows = N > B ? N : B;
    stream_init_kernel<<<static_cast<unsigned>(rows), 128, 0, s>>>(p.state.as<DecodeState>(), p.unfinished.as<int>(), p.pos.as<int>(),
                                                                  p.live_extent.as<int>(), r.ids.as<long long>(),
                                                                  r.len.as<int>(), T + 1, static_cast<int>(N), B, a.start, a.pad,
                                                                  h->shared.as<act_t>(), p.dx.as<res_t>(), c.d);
    h->launches++;
    if (p.mode.score) {  // every result position 0, no slot forced until it is admitted
      score_reset_kernel<<<1024, 128, 0, s>>>(r.lp.as<float>(), r.lg.as<float>(), static_cast<size_t>(N) * T,
                                              p.ftok.as<int>(), B, nullptr, nullptr, nullptr, T);
      h->launches++;
    }
    CU_OK(h, cudaGetLastError());
  }
  CU_OK(h, cudaEventRecord(h->ev[1], s));
  // Slot states: FREE -> (staged for an admission whose encoder pass is in flight) PENDING -> ACTIVE -> FREE.
  // The encoder pass of an admission runs on its own low-priority stream UNDER the decode steps of the slots that
  // are already active (its kernels touch only the encoder workspace and the arena rows of the pending slots, which
  // no decode kernel reads: their live extent is 0 until admit_slots_kernel starts them); the admitted slots join
  // at the next poll boundary. B200T5_ADMIT_OVERLAP=0 keeps everything on one stream (round-1 behaviour).
  enum : char { FREE = 0, PENDING = 1, ACTIVE = 2 };
  std::vector<char> state(B, FREE), stepped(B, 0);
  long long next = 0, done = 0;
  int active = 0, steps = 0, n_free = B;
  bool pending = false, enc_used = false;
  int pend_k = 0;
  double enc_flops = 0;
  int* row_on = p.h_admit;
  int* a_slot = p.h_admit + B;
  int* a_row = p.h_admit + 2 * B;
  const size_t row_bytes = static_cast<size_t>(S) * 8;
  auto admit_now = [&](int k) -> int {
    admit_slots_kernel<<<k, 128, 0, s>>>(p.admit.as<int>() + B, p.admit.as<int>() + 2 * B, p.unfinished.as<int>(), p.pos.as<int>(),
                                         p.out_row.as<int>(), p.extent.as<int>(), p.live_extent.as<int>(),
                                         p.key_ok.as<unsigned char>(), p.live_key_ok.as<unsigned char>(), S, a.start,
                                         h->shared.as<act_t>(), p.dx.as<res_t>(), c.d);
    h->launches++;
    if (p.mode.proc) {  // the admitted slots' processor state, from their prompts (still in ids_dev) and start token
      proc_reset_kernel<<<k, 128, 0, s>>>(p.proc.dev(), p.admit.as<int>() + B, p.ids_dev.as<long long>(),
                                          r.ids.as<long long>(), T + 1, p.out_row.as<int>(), 1);
      h->launches++;
    }
    if (p.mode.score == 2) {  // the admitted slots' first labels
      score_reset_kernel<<<(k + 127) / 128, 128, 0, s>>>(nullptr, nullptr, 0, p.ftok.as<int>(), k, p.admit.as<int>() + B,
                                                         p.admit.as<int>() + 2 * B, r.forced.as<long long>(), T);
      h->launches++;
    }
    CU_OK(h, cudaGetLastError());
    CU_OK(h, cudaEventRecord(h->admitted_ev, s));  // the staging buffers may be reused after this point
    for (int b = 0; b < B; ++b)
      if (state[b] == PENDING) state[b] = ACTIVE;
    active += k;
    return B200T5_OK;
  };
  while (done < N) {
    // ---- (a) an admission whose encoder pass ran under the previous round of decode steps: start its slots
    if (pending) {
      CU_OK(h, cudaStreamWaitEvent(s, h->enc_done_ev, 0));
      TRY(admit_now(pend_k));
      pending = false;
    }
    // ---- (b) `poll` decode steps for every slot (eight = one graph launch); queued BEFORE the next admission's
    //          encoder pass so that the two overlap
    const bool stepping = active > 0;
    for (int b = 0; b < B; ++b) stepped[b] = state[b] == ACTIVE;  // slots admitted later in this round have not stepped yet
    if (stepping) {
      if (poll % kStepsPerGraph == 0) {
        for (int r = 0; r < poll / kStepsPerGraph; ++r) CU_OK(h, cudaGraphLaunch(p.gexec8, s));
      } else {
        for (int r = 0; r < poll; ++r) CU_OK(h, cudaGraphLaunch(p.gexec, s));
      }
      h->launches += static_cast<int64_t>(p.graph_nodes) * poll;
      steps += poll;
      CU_OK(h, cudaMemcpyAsync(p.h_unf, p.unfinished.p, static_cast<size_t>(B) * 4, cudaMemcpyDeviceToHost, s));
    }
    // ---- (c) admission: the next k prompts go to the free slots
    const long long left = N - next;
    if (left > 0 && n_free > 0 && (active == 0 || n_free >= (left < admit_min ? left : admit_min))) {
      const bool overlap = h->admit_overlap && stepping;
      cudaStream_t es = overlap ? h->enc_stream : s;
      if (enc_used) CU_OK(h, cudaEventSynchronize(h->enc_done_ev));  // the pinned staging rows of the previous pass are free
      const int k = static_cast<int>(left < n_free ? left : n_free);
      int j = 0;
      for (int b = 0; b < B; ++b) {
        row_on[b] = 0;
        if (state[b] == FREE && j < k) {
          const long long r = next + j;
          row_on[b] = 1;
          a_slot[j] = b;
          a_row[j] = static_cast<int>(r);
          state[b] = PENDING;
          memcpy(p.h_ids + static_cast<size_t>(b) * S, input_ids + static_cast<size_t>(r) * S, row_bytes);
          if (attention_mask) memcpy(p.h_mask + static_cast<size_t>(b) * S, attention_mask + static_cast<size_t>(r) * S, row_bytes);
          ++j;
        }
      }
      n_free -= k;
      if (overlap) CU_OK(h, cudaStreamWaitEvent(es, h->admitted_ev, 0));  // the previous admit kernel has read `admit` / extent / key_ok
      const size_t nb = static_cast<size_t>(B) * row_bytes;
      CU_OK(h, cudaMemcpyAsync(p.ids_dev.p, p.h_ids, nb, cudaMemcpyHostToDevice, es));
      if (attention_mask) CU_OK(h, cudaMemcpyAsync(p.mask_dev.p, p.h_mask, nb, cudaMemcpyHostToDevice, es));
      CU_OK(h, cudaMemcpyAsync(p.admit.p, p.h_admit, static_cast<size_t>(3) * B * 4, cudaMemcpyHostToDevice, es));
      // rows that are not admitted keep stale ids / masks in the staging buffers: row_on switches them off
      TRY(run_encoder(h, p.ids_dev.as<long long>(), attention_mask ? p.mask_dev.as<long long>() : nullptr, es, p.admit.as<int>()));
      TRY(run_cross_kv(h, es));
      fill_stats_model(h, 0);
      enc_flops += h->last_enc_flops;
      next += k;
      if (overlap) {
        CU_OK(h, cudaEventRecord(h->enc_done_ev, es));
        enc_used = true;
        pending = true;
        pend_k = k;
      } else {
        TRY(admit_now(k));
      }
    }
    // ---- (d) which slots have finished
    if (stepping) {
      CU_OK(h, cudaStreamSynchronize(s));
      for (int b = 0; b < B; ++b) {
        if (state[b] == ACTIVE && stepped[b] && !p.h_unf[b]) {
          state[b] = FREE;
          ++n_free;
          --active;
          ++done;
        }
      }
    }
  }
  CU_OK(h, cudaEventRecord(h->ev[2], s));
  TRY(copy_results(h, static_cast<size_t>(N), out_ids, out_len, a.sh.on ? score->token_logprobs : nullptr,
                   a.sh.on ? score->token_logits : nullptr, cudaMemcpyDeviceToHost, s));
  CU_OK(h, cudaStreamSynchronize(s));
  h->last_steps = steps;
  h->last_decode_bytes = 0;  // not modelled for a pool whose occupancy varies
  h->last_enc_flops = enc_flops;
  h->ev_valid = true;
  return B200T5_OK;
}

extern "C" int b200t5_get_stats(b200t5_handle h, b200t5_stats* out) {
  if (!h || !out) return fail(h, B200T5_EINVAL, "null argument");
  memset(out, 0, sizeof(*out));
  if (!h->ev_valid || !h->plan) return fail(h, B200T5_ESTATE, "no generate call recorded");
  CU_OK(h, cudaSetDevice(h->device));
  CU_OK(h, cudaEventSynchronize(h->ev[2]));
  CU_OK(h, cudaEventElapsedTime(&out->encoder_ms, h->ev[0], h->ev[1]));
  CU_OK(h, cudaEventElapsedTime(&out->decode_ms, h->ev[1], h->ev[2]));
  out->decode_steps = h->last_steps;
  out->kernel_launches = h->launches;
  fill_stats_model(h, h->last_steps);
  out->decode_algo_bytes = h->last_decode_bytes;
  out->encoder_flops = h->last_enc_flops;
  out->xattn_kernel = h->plan->mode.xattn_stream ? 1 : 0;
  out->row_chains = h->plan->n_chains;
  return B200T5_OK;
}

// ================================================================== measurement hooks
// Times the roofline-setting kernel (cross-attention decode, D7) alone, on the cross-KV arena of the last
// generate call, in launches of `rows_per_launch` batch rows (0 = the whole batch; the step graph launches one
// chain's rows at a time): `reps` sweeps over all decoder layers (every launch streams a different slab, the sweep
// is far larger than L2), CUDA events on the launching stream. A microbenchmark: back-to-back launches with nothing
// else on the GPU. What the launches cost INSIDE the step graph is b200t5_get_xattn_profile's figure.
extern "C" int b200t5_bench_cross_attn(b200t5_handle h, int reps, int rows_per_launch, float* avg_ms_per_launch,
                                       double* bytes_per_launch, void* stream) {
  if (!h || !avg_ms_per_launch || !bytes_per_launch || reps < 1) return fail(h, B200T5_EINVAL, "bad argument");
  if (!h->plan) return fail(h, B200T5_ESTATE, "no plan: call generate first");
  CU_OK(h, cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Plan& p = *h->plan;
  const Cfg& c = h->c;
  const int rows = rows_per_launch > 0 && rows_per_launch < p.B ? rows_per_launch : p.B;
  int launches = 0;
  cudaError_t le = cudaSuccess;
  auto sweep = [&]() {
    launches = 0;
    for (int l = 0; l < c.Ld; ++l) {
      for (int b0 = 0; b0 < p.B; b0 += rows) {
        const int nb = p.B - b0 < rows ? p.B - b0 : rows;
        cudaError_t e = launch_cross_attention(h, s, false, l, b0, nb, p.dq.as<act_t>() + static_cast<size_t>(b0) * c.I,
                                               p.dctx.as<act_t>() + static_cast<size_t>(b0) * c.I, p.extent.as<int>() + b0,
                                               p.key_ok.as<unsigned char>() + static_cast<size_t>(b0) * p.S, -1);
        if (e != cudaSuccess) le = e;
        ++launches;
      }
    }
  };
  sweep();  // warm-up
  CU_OK(h, le);
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  struct EvGuard {
    cudaEvent_t &a, &b;
    ~EvGuard() {
      if (a) cudaEventDestroy(a);
      if (b) cudaEventDestroy(b);
    }
  } guard{e0, e1};
  CU_OK(h, cudaEventCreate(&e0));
  CU_OK(h, cudaEventCreate(&e1));
  CU_OK(h, cudaEventRecord(e0, s));
  for (int r = 0; r < reps; ++r) sweep();
  CU_OK(h, cudaEventRecord(e1, s));
  CU_OK(h, cudaEventSynchronize(e1));
  CU_OK(h, le);
  float ms = 0.f;
  CU_OK(h, cudaEventElapsedTime(&ms, e0, e1));
  CU_OK(h, cudaGetLastError());
  *avg_ms_per_launch = ms / (static_cast<float>(reps) * launches);
  std::vector<int> ext(p.B);
  CU_OK(h, cudaMemcpy(ext.data(), p.extent.p, p.B * 4, cudaMemcpyDeviceToHost));
  double sum_s = 0;
  for (int v : ext) sum_s += v;
  // K and V rows of every attended key, bf16; averaged over the launches of one layer
  *bytes_per_launch = 2.0 * 2.0 * c.I * sum_s / (static_cast<double>(launches) / c.Ld);
  return B200T5_OK;
}

// Runtime options (what the B200T5_* environment variables set at create time, changeable on a live handle so
// that a sweep does not reload the model). Any change drops the execution plan: the next call re-captures the
// step graph. Names: "chains" (row-chains per step, 0 = default), "xattn" (decode cross-attention: 0 = per-thread-load
// kernel, 1 = TMA stream kernel, 2 = per call by prompt fill), "xattn_stages", "pdl", "admit_overlap", "sk_stages64",
// "sk_stages128", "profile_xattn" (1 = every cross-attention launch inside the step graph stamps %globaltimer; read with
// b200t5_get_xattn_profile; off in any timed region), "enc_gemm" (128 x 256 encoder GEMMs: 1 = epilogue-overlapped
// kernel, 0 = the kernel whose epilogue follows each main loop).
extern "C" int b200t5_set_option(b200t5_handle h, const char* name, int value) {
  if (!h || !name) return fail(h, B200T5_EINVAL, "null argument");
  const std::string n(name);
  if (n == "chains") h->chains_override = value < 0 ? 0 : value;
  else if (n == "xattn") h->xattn_mode = value < 0 || value > 2 ? 2 : value;
  else if (n == "xattn_stages") {
    if (value < 2 || value > kXsMaxStages) return fail(h, B200T5_EINVAL, "xattn_stages must be in [2, %d]", kXsMaxStages);
    h->xs_stages = value;
  } else if (n == "pdl") h->use_pdl = value != 0;
  else if (n == "admit_overlap") h->admit_overlap = value != 0;
  else if (n == "sk_stages64") h->sk_stages64 = value;
  else if (n == "sk_stages128") h->sk_stages128 = value;
  else if (n == "profile_xattn") h->profile_xattn = value != 0;
  else if (n == "enc_gemm") h->enc_gemm_ws = value != 0;
  else return fail(h, B200T5_EINVAL, "unknown option '%s'", name);
  CU_OK(h, cudaSetDevice(h->device));
  CU_OK(h, cudaDeviceSynchronize());
  h->plan.reset();
  return B200T5_OK;
}

// Cross-attention launches of the step graph since profiling was switched on: their mean in-situ duration
// (first CTA's start to last CTA's end, %globaltimer), the number of launches seen, and the algorithmic bytes of
// one launch at the moment of the call (K and V rows of the keys the live rows still attend).
extern "C" int b200t5_get_xattn_profile(b200t5_handle h, double* avg_us_per_launch, int64_t* launches, double* bytes_per_launch,
                                        double* busy_us_per_layer, double* bytes_per_layer) {
  if (!h || !avg_us_per_launch || !launches || !bytes_per_launch || !busy_us_per_layer || !bytes_per_layer)
    return fail(h, B200T5_EINVAL, "null argument");
  if (!h->plan || !h->profile_xattn) return fail(h, B200T5_ESTATE, "profiling is off (b200t5_set_option(h, \"profile_xattn\", 1), then generate)");
  CU_OK(h, cudaSetDevice(h->device));
  CU_OK(h, cudaDeviceSynchronize());
  Plan& p = *h->plan;
  const int n = h->c.Ld * p.n_chains;
  std::vector<unsigned long long> acc(static_cast<size_t>(n + h->c.Ld) * 2);
  CU_OK(h, cudaMemcpy(acc.data(), p.xs_acc.p, acc.size() * 8, cudaMemcpyDeviceToHost));
  unsigned long long ns = 0, cnt = 0, busy = 0, layers = 0;
  for (int i = 0; i < n; ++i) {
    ns += acc[2 * i];
    cnt += acc[2 * i + 1];
  }
  for (int l = 0; l < h->c.Ld; ++l) {
    busy += acc[2 * (n + l)];
    layers += acc[2 * (n + l) + 1];
  }
  *avg_us_per_launch = cnt ? static_cast<double>(ns) / static_cast<double>(cnt) / 1e3 : 0.0;
  *busy_us_per_layer = layers ? static_cast<double>(busy) / static_cast<double>(layers) / 1e3 : 0.0;
  *launches = static_cast<int64_t>(cnt);
  std::vector<int> ext(p.B);
  CU_OK(h, cudaMemcpy(ext.data(), p.extent.p, p.B * 4, cudaMemcpyDeviceToHost));
  double sum_s = 0;
  for (int v : ext) sum_s += v;
  *bytes_per_layer = 2.0 * 2.0 * h->c.I * sum_s;
  *bytes_per_launch = *bytes_per_layer / p.n_chains;
  return B200T5_OK;
}

// ================================================================== parity hooks
extern "C" int b200t5_encode(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                             void* enc_out_bf16, void* stream) {
  TRY(validate(h, B, S, nullptr));
  if (!input_ids || !enc_out_bf16) return fail(h, B200T5_EINVAL, "null argument");
  CU_OK(h, cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int T = h->plan && h->plan->B == B && h->plan->S == S ? h->plan->Tmax : 1;
  TRY(ensure_plan(h, B, S, T));
  TRY(run_encoder(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask), s));
  if (h->plan->packed) {
    unpack_rows_kernel<<<dim3((S + 7) / 8, B), 256, 0, s>>>(h->plan->xn.as<act_t>(), h->plan->cu.as<int>(), static_cast<act_t*>(enc_out_bf16), S, h->c.d);
    CU_OK(h, cudaGetLastError());
  } else {
    CU_OK(h, cudaMemcpyAsync(enc_out_bf16, h->plan->xn.p, static_cast<size_t>(B) * S * h->c.d * 2, cudaMemcpyDeviceToDevice, s));
  }
  return B200T5_OK;
}

extern "C" int b200t5_decode_logits(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B,
                                    int S, const int64_t* decoder_input_ids, int T, float* logits, void* stream) {
  TRY(validate(h, B, S, nullptr));
  if (!input_ids || !decoder_input_ids || !logits || T < 1) return fail(h, B200T5_EINVAL, "bad argument");
  CU_OK(h, cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TRY(ensure_plan(h, B, S, T));
  Plan& p = *h->plan;
  const Cfg& c = h->c;
  TRY(run_encoder(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask), s));
  TRY(run_cross_kv(h, s));
  p.mode = StepMode();  // the step's head stores logits: only the cross-attention kernel matters
  p.mode.xattn_stream = pick_xattn(h, static_cast<double>(p.rows_valid) / (static_cast<double>(B) * S));
  CU_OK(h, cudaMemcpyAsync(p.live_extent.p, p.extent.p, static_cast<size_t>(B) * 4, cudaMemcpyDeviceToDevice, s));
  CU_OK(h, cudaMemcpyAsync(p.live_key_ok.p, p.key_ok.p, static_cast<size_t>(B) * S, cudaMemcpyDeviceToDevice, s));
  set_state_kernel<<<1, 1, 0, s>>>(p.state.as<DecodeState>(), 0);
  DevBuf col;
  CU_OK(h, col.alloc(static_cast<size_t>(B) * 8));
  for (int t = 0; t < T; ++t) {
    CU_OK(h, cudaMemcpy2DAsync(col.p, 8, reinterpret_cast<const long long*>(decoder_input_ids) + t, static_cast<size_t>(T) * 8, 8, B, cudaMemcpyDeviceToDevice, s));
    force_token_kernel<<<B, 128, 0, s>>>(col.as<long long>(), h->shared.as<act_t>(), p.dx.as<res_t>(), c.d);
    TRY(run_decode_step(h, s, false, logits + static_cast<size_t>(t) * c.V, T * c.V));
  }
  CU_OK(h, cudaStreamSynchronize(s));
  return B200T5_OK;
}

// ================================================================== teacher-forced forward pass
// The forward pass's GeGLU product: the decoder's wi is interleaved per 128-row tile for the split-K decode GEMM, so its
// B*T-row product runs 128 x 128 tiles that read that packing (the encoder's 128 x 256 tiles would need a second copy).
// A ReLU model's wi runs the same tiles through the same 128-row boxes with EpiRelu.
static cudaError_t run_geglu_fwd(b200t5_ctx* h, const CUtensorMap& tmA, const DecLayerW& w, int M, const EpiGeglu::Params& ep, cudaStream_t s) {
  h->launches++;
  if (!h->c.gated) return launch_gemm<128, EpiRelu>(tmA, w.tm_wi, M, h->c.F, h->c.d, 0, EpiRelu::Params{ep.out, ep.F}, h->num_sms, s);
  return launch_gemm<128, EpiGegluNarrow>(tmA, w.tm_wi, M, w.wi_rows, h->c.d, 0, ep, h->num_sms, s);
}

// The decoder layer stack over all B*T positions at once (T5Stack with is_decoder, no cache), from x = the embedded
// decoder ids to xn = the final RMSNorm, in the plan's encoder workspace; the epilogue flags of each product are the
// decode step's (chain_layer_pre / chain_layer_post). The products run the encoder's 128 x 256 GEMMs through the
// layer's 128-row-box tensor maps, except GeGLU (run_geglu_fwd).
// `prefill` (a decoder prompt's positions 0 .. T-1): each layer's K/V also go to cache positions 0 .. T-1
// (prefill_cache_kernel), and the pass ends at the last layer's K/V: nothing reads the prompt positions' outputs.
// `qoff` (b200t5_forward_choices): the decoder runs R rows of T positions for the plan's B prompts, prompt b's rows
// holding the query rows qoff[b] .. qoff[b+1]-1 (device int [B+1]), whose cross-attention is decoder_cross_packed_kernel
// over q_tiles tiles of 64 queries. Without it row b is prompt b (R = B).
static int run_decoder_forward(b200t5_ctx* h, int T, cudaStream_t s, bool prefill = false, int R = 0, const int* qoff = nullptr,
                               int q_tiles = 0) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  const int B = p.B, S = p.S, d = c.d, I = c.I, F = c.F, H = c.H;
  if (!qoff) R = B;
  const int M = R * T;
  res_t* x = p.x.as<res_t>();
  act_t* xn = p.xn.as<act_t>();
  act_t* qkv = p.qkv.as<act_t>();
  act_t* ctx = p.ctx.as<act_t>();
  const dim3 agrid((T + kEncQ - 1) / kEncQ, R * H);
  for (int l = 0; l < c.Ld; ++l) {
    DecLayerW& w = h->dec[l];
    CU_OK(h, run_rmsnorm(h, x, w.ln0.as<act_t>(), xn, M, d, c.eps, s));
    CU_OK(h, run_gemm_2cta<EpiStore>(h, p.tm_xn, w.tm2_qkv, M, 3 * I, d, EpiStore::Params{qkv, 3 * I}, s));
    if (prefill) {
      prefill_cache_kernel<<<M, 128, 0, s>>>(qkv, p.self_kv.as<act_t>() + static_cast<size_t>(l) * 2 * B * I * p.Tmax, T, B, H, p.Tmax);
      h->launches++;
      CU_OK(h, cudaGetLastError());
      if (l == c.Ld - 1) return B200T5_OK;
    }
    decoder_attn_kernel<kAttnCausal><<<agrid, kEncThreads, encoder_attn_smem_bytes(T), s>>>(
        qkv, nullptr, ctx, p.fwd_bias.as<float>(), nullptr, nullptr, R, T, T, H);
    h->launches++;
    CU_OK(h, cudaGetLastError());
    {
      EpiResidual::Params ep{x, x, d};
      ep.round_out = l == 0;  // (fp16 build) the stream is still fp16 before the first feed-forward block
      CU_OK(h, run_gemm_2cta<EpiResidual>(h, p.tm_ctx, w.tm2_o, M, d, I, ep, s));
    }
    CU_OK(h, run_rmsnorm(h, x, w.ln1.as<act_t>(), xn, M, d, c.eps, s));
    CU_OK(h, run_gemm_2cta<EpiStore>(h, p.tm_xn, w.tm2_cq, M, I, d, EpiStore::Params{qkv, I}, s));
    const act_t* kv = p.cross_kv.as<act_t>() + static_cast<size_t>(l) * 2 * B * I * S;
    if (qoff)
      decoder_cross_packed_kernel<<<dim3(q_tiles, B * H), kEncThreads, encoder_attn_smem_bytes(S), s>>>(
          qkv, kv, ctx, p.key_ok.as<unsigned char>(), p.extent.as<int>(), qoff, B, S, H);
    else
      decoder_attn_kernel<kAttnCross><<<agrid, kEncThreads, encoder_attn_smem_bytes(S), s>>>(
          qkv, kv, ctx, nullptr, p.key_ok.as<unsigned char>(), p.extent.as<int>(), B, T, S, H);
    h->launches++;
    CU_OK(h, cudaGetLastError());
    {
      EpiResidual::Params ep{x, x, d};
      ep.round_out = l == 0;
      CU_OK(h, run_gemm_2cta<EpiResidual>(h, p.tm_ctx, w.tm2_co, M, d, I, ep, s));
    }
    CU_OK(h, run_rmsnorm(h, x, w.ln2.as<act_t>(), xn, M, d, c.eps, s));
    CU_OK(h, run_geglu_fwd(h, p.tm_xn, w, M, EpiGeglu::Params{p.hff.as<ffh_t>(), F, h->gelu_lut}, s));
    {
      EpiResidual::Params ep{x, x, d};
      ep.round_acc = B200T5_F16 ? 0 : 1;  // fp16 build: `wo` is an fp32 Linear, its output is not rounded
      ep.round_out = B200T5_F16 ? 0 : 1;
      CU_OK(h, run_ffo_2cta(h, p.tm_hff, w.tm2_ffo, M, d, ep, s));
    }
  }
  CU_OK(h, run_rmsnorm(h, x, h->dec_final_ln.as<act_t>(), xn, M, d, c.eps, s, false, c.out_scale));
  return B200T5_OK;
}

// run_decoder_forward's GeGLU product (run_geglu_fwd) reads wi in the decode step's packing through 128-row boxes: it
// needs the default 128-row wi tile of the split-K decode GEMM (the tensor map's box, for a ReLU model too). Checked before anything is launched.
static int check_forward_wi(b200t5_ctx* h, const char* who) {
  if (h->sk_wi.bn != 128)
    return fail(h, B200T5_EINVAL, "%s: needs the feed-forward wi packed in 128-row tiles, but B200T5_SK set the wi tile to %d rows "
                "(unset B200T5_SK or give wi a bn of 128)", who, h->sk_wi.bn);
  return B200T5_OK;
}

// The forward pass's causal bias for T positions: dec_relbias by distance i - j, float [H][T], as the decode step's
// dec_bias (kept while T stays the same).
static int ensure_fwd_bias(b200t5_ctx* h, int T) {
  const Cfg& c = h->c;
  Plan& p = *h->plan;
  if (p.fwd_T == T) return B200T5_OK;
  std::vector<float> db(static_cast<size_t>(c.H) * T);
  for (int n = 0; n < T; ++n) {
    const int bk = b200t5_relative_bucket(-n, 0, c.nb, c.maxdist);
    for (int hh = 0; hh < c.H; ++hh) db[static_cast<size_t>(hh) * T + n] = h->dec_relbias_h[static_cast<size_t>(bk) * c.H + hh];
  }
  CU_OK(h, p.fwd_bias.alloc(db.size() * 4));
  CU_OK(h, cudaMemcpy(p.fwd_bias.p, db.data(), db.size() * 4, cudaMemcpyHostToDevice));
  p.fwd_T = T;
  return B200T5_OK;
}

// The teacher-forced pass of b200t5_forward and b200t5_forward_choices: the encoder and the cross-K/V projection over
// B prompts, then the decoder over R rows of T positions and the lm_head. `offs` (host int [B+1], b200t5_forward_choices)
// puts rows offs[b] .. offs[b+1]-1 on prompt b; NULL (b200t5_forward) puts row b on prompt b, R = B. `who` names the
// entry point in error messages.
static int forward_impl(b200t5_ctx* h, const char* who, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                        const int32_t* offs, const int64_t* decoder_input_ids, const int64_t* labels, int T,
                        const b200t5_forward_io* io, void* stream) {
  CU_OK(h, cudaSetDevice(h->device));
  const Cfg& c = h->c;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int R = offs ? offs[B] : B;
  const size_t M = static_cast<size_t>(R) * T;
  if (M > static_cast<size_t>(INT32_MAX) / 8) return fail(h, B200T5_EINVAL, "%s: %s*T too large", who, offs ? "R" : "B");
  // labels and decoder ids are read back and checked; without decoder ids they are transformers' _shift_right(labels)
  std::vector<long long> lab, dec(M);
  CU_OK(h, cudaStreamSynchronize(s));
  if (labels) {
    lab.resize(M);
    CU_OK(h, cudaMemcpy(lab.data(), labels, M * 8, cudaMemcpyDeviceToHost));
    for (long long v : lab)
      if (v != -100 && (v < 0 || v >= c.V)) return fail(h, B200T5_EINVAL, "%s: label %lld outside [0, %d) and not -100", who, v, c.V);
  }
  if (decoder_input_ids) {
    CU_OK(h, cudaMemcpy(dec.data(), decoder_input_ids, M * 8, cudaMemcpyDeviceToHost));
    for (long long v : dec)
      if (v < 0 || v >= c.V) return fail(h, B200T5_EINVAL, "%s: decoder id %lld outside [0, %d)", who, v, c.V);
  } else {
    if (c.start < 0 || c.start >= c.V || c.pad < 0 || c.pad >= c.V) return fail(h, B200T5_EINVAL, "%s: special token id out of range", who);
    for (size_t b = 0; b < static_cast<size_t>(R); ++b)
      for (int t = 0; t < T; ++t) {
        const long long v = t == 0 ? c.start : lab[b * T + t - 1];
        dec[b * T + t] = v == -100 ? c.pad : v;
      }
  }
  // the plan of (B, S): reused whatever its Tmax when its workspace holds the R*T decoder rows, else rebuilt with the
  // same Tmax (1 for a new shape: the forward pass has no self-attention cache)
  {
    const int ws = static_cast<int>(std::max<size_t>(S, (M + B - 1) / B));
    const bool same = h->plan && h->plan->B == B && h->plan->S == S && h->plan->group == 1;
    if (!same || h->plan->ws_S < ws) {
      const int Tm = same ? h->plan->Tmax : 1;
      CU_OK(h, cudaDeviceSynchronize());
      h->plan.reset();
      TRY(build_plan(h, B, S, Tm, 1, ws));
    }
  }
  Plan& p = *h->plan;
  const int nt = p.n_vtiles;
  // ids [M] int64, label columns [M] int32, one zero int (the lm_head's step: min_new is 0), then (choices) the query-row
  // offsets int [B+1]
  const size_t ids_bytes = M * 8 + M * 4 + 16 + (offs ? static_cast<size_t>(B + 1) * 4 : 0);
  if (p.fwd_ids.bytes < ids_bytes) CU_OK(h, p.fwd_ids.alloc(ids_bytes));
  long long* ids_dev = p.fwd_ids.as<long long>();
  int* ftok_dev = reinterpret_cast<int*>(ids_dev + M);
  int* zero_dev = ftok_dev + M;
  int* qoff_dev = zero_dev + 4;
  std::vector<int> ftok(M + 4, 0);
  for (size_t m = 0; m < M && labels; ++m) ftok[m] = lab[m] == -100 ? -1 : static_cast<int>(lab[m]);
  CU_OK(h, cudaMemcpyAsync(ids_dev, dec.data(), M * 8, cudaMemcpyHostToDevice, s));
  CU_OK(h, cudaMemcpyAsync(ftok_dev, ftok.data(), (M + 4) * 4, cudaMemcpyHostToDevice, s));
  int q_tiles = 0;
  std::vector<int> qoff;
  if (offs) {
    qoff.resize(B + 1);
    for (int b = 0; b <= B; ++b) qoff[b] = offs[b] * T;
    for (int b = 0; b < B; ++b) q_tiles = std::max(q_tiles, (qoff[b + 1] - qoff[b] + kEncQ - 1) / kEncQ);
    CU_OK(h, cudaMemcpyAsync(qoff_dev, qoff.data(), qoff.size() * 4, cudaMemcpyHostToDevice, s));
  }
  TRY(ensure_fwd_bias(h, T));
  // lm_head partials [M][n_tiles] x 3 + fval [M]: in hff (free after the last feed-forward block) when they fit
  const bool lp_on = io->token_logprobs != nullptr;
  const size_t part_bytes = lp_on ? M * (static_cast<size_t>(3) * nt + 1) * 4 : 0;
  float* part = p.hff.as<float>();
  if (part_bytes > p.hff.bytes) {
    if (p.fwd_part.bytes < part_bytes) CU_OK(h, p.fwd_part.alloc(part_bytes));
    part = p.fwd_part.as<float>();
  }
  h->launches = 0;
  CU_OK(h, cudaEventRecord(h->ev[0], s));
  TRY(run_encoder(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask), s));
  TRY(run_cross_kv(h, s));
  CU_OK(h, cudaEventRecord(h->ev[1], s));
  embed_rows_kernel<<<static_cast<unsigned>((M + 7) / 8), 256, 0, s>>>(ids_dev, h->shared.as<act_t>(), p.x.as<res_t>(), static_cast<int>(M), c.d, c.V);
  h->launches++;
  TRY(run_decoder_forward(h, T, s, false, R, offs ? qoff_dev : nullptr, q_tiles));
  LmHeadParams ep{};
  ep.pval = part;
  ep.pidx = reinterpret_cast<int*>(part + M * nt);
  ep.psum = part + 2 * M * nt;
  ep.fval = part + 3 * M * nt;
  ep.ftok = ftok_dev;
  ep.n_tiles = nt;
  ep.step = zero_dev;
  ep.eos = -1;
  ep.min_new = 0;
  h->launches++;
  if (io->logits) {
    const size_t ldc = static_cast<size_t>(c.V);
    if (lp_on) CU_OK(h, (launch_gemm<128, EpiLmLogits<true>>(p.tm_xn, h->tm_lm, static_cast<int>(M), c.V, c.d, 1,
                                                             EpiLmLogits<true>::Params{ep, static_cast<act_t*>(io->logits), ldc}, h->num_sms, s)));
    else CU_OK(h, (launch_gemm<128, EpiLmLogits<false>>(p.tm_xn, h->tm_lm, static_cast<int>(M), c.V, c.d, 1,
                                                        EpiLmLogits<false>::Params{ep, static_cast<act_t*>(io->logits), ldc}, h->num_sms, s)));
  } else {
    CU_OK(h, (launch_gemm<128, EpiLmHead<false, true>>(p.tm_xn, h->tm_lm, static_cast<int>(M), c.V, c.d, 1, ep, h->num_sms, s)));
  }
  if (lp_on) {
    forward_logprob_kernel<<<static_cast<unsigned>(M), 128, 0, s>>>(ep.pval, ep.psum, ep.fval, ftok_dev, nt, io->token_logprobs);
    h->launches++;
  }
  CU_OK(h, cudaGetLastError());
  CU_OK(h, cudaEventRecord(h->ev[2], s));
  h->last_steps = 0;
  h->ev_valid = true;
  return B200T5_OK;
}

extern "C" int b200t5_forward(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                              const int64_t* decoder_input_ids, const int64_t* labels, int T, const b200t5_forward_io* io,
                              void* stream) {
  TRY(validate(h, B, S, nullptr));
  if (!input_ids || !io) return fail(h, B200T5_EINVAL, "forward: null argument");
  if (!decoder_input_ids && !labels) return fail(h, B200T5_EINVAL, "forward: decoder_input_ids or labels is required");
  if (!io->logits && !io->token_logprobs) return fail(h, B200T5_EINVAL, "forward: neither logits nor token_logprobs requested");
  if (io->token_logprobs && !labels) return fail(h, B200T5_EINVAL, "forward: token_logprobs needs labels");
  if (T < 1 || T > 4096) return fail(h, B200T5_EINVAL, "forward: T=%d outside [1, 4096]", T);
  TRY(check_forward_wi(h, "forward"));
  return forward_impl(h, "forward", input_ids, attention_mask, B, S, nullptr, decoder_input_ids, labels, T, io, stream);
}

extern "C" int b200t5_forward_choices(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                      const int32_t* row_offsets, const int64_t* labels, int T, const b200t5_forward_io* io,
                                      void* stream) {
  TRY(validate(h, B, S, nullptr));
  if (!input_ids || !io || !row_offsets || !labels) return fail(h, B200T5_EINVAL, "forward_choices: null argument");
  if (!io->logits && !io->token_logprobs) return fail(h, B200T5_EINVAL, "forward_choices: neither logits nor token_logprobs requested");
  if (T < 1 || T > 4096) return fail(h, B200T5_EINVAL, "forward_choices: T=%d outside [1, 4096]", T);
  if (row_offsets[0] != 0) return fail(h, B200T5_EINVAL, "forward_choices: row_offsets[0] = %d, not 0", row_offsets[0]);
  for (int b = 0; b < B; ++b)
    if (row_offsets[b + 1] <= row_offsets[b])
      return fail(h, B200T5_EINVAL, "forward_choices: row_offsets not strictly increasing at prompt %d (%d, %d)", b, row_offsets[b],
                  row_offsets[b + 1]);
  if (static_cast<long long>(row_offsets[B]) * h->c.H > 65535)
    return fail(h, B200T5_EINVAL, "forward_choices: R*H = %lld exceeds 65535 (the causal self-attention's grid)",
                static_cast<long long>(row_offsets[B]) * h->c.H);
  TRY(check_forward_wi(h, "forward_choices"));
  return forward_impl(h, "forward_choices", input_ids, attention_mask, B, S, row_offsets, nullptr, labels, T, io, stream);
}

// ================================================================== decoder prompt
// generate(decoder_input_ids=d): a static batch whose decoding starts after a decoder prompt d [B][P] (start token
// included). The prompt's positions 0 .. P-2 run as one forward pass over B*(P-1) rows (run_decoder_forward with the
// cache sink), which leaves their K/V in the self-attention cache; then the step loop starts at t = P-1 with input
// d[P-1] (decode_init_prompt_kernel). Everything the steps index by position (cache, bias, result columns, score
// columns) is absolute, so the plan's Tmax is P-1 + max_new_tokens and the steps themselves are unchanged.

// The checks of a prefixed call and its prompt, host int64 [B][P] (checked and staged on the host: no stream sync).
static int read_prompt(b200t5_ctx* h, const int64_t* decoder_input_ids, int B, int P, const b200t5_gen_params* gp,
                       const b200t5_score_io* score, std::vector<long long>* d) {
  if (!decoder_input_ids) return fail(h, B200T5_EINVAL, "prefixed: decoder_input_ids is NULL");
  if (P < 1) return fail(h, B200T5_EINVAL, "prefixed: decoder prompt length P=%d < 1", P);
  if (P >= 2) TRY(check_forward_wi(h, "prefixed"));  // the prefill is run_decoder_forward
  if (gp && static_cast<long long>(P) - 1 + gp->max_new_tokens > 4096)
    return fail(h, B200T5_EINVAL, "prefixed: P-1 + max_new_tokens = %lld exceeds 4096", static_cast<long long>(P) - 1 + gp->max_new_tokens);
  if (score && score->forced_ids) return fail(h, B200T5_EINVAL, "prefixed: forced_ids cannot be combined with a decoder prompt");
  d->assign(decoder_input_ids, decoder_input_ids + static_cast<size_t>(B) * P);
  for (long long v : *d)
    if (v < 0 || v >= h->c.V) return fail(h, B200T5_EINVAL, "prefixed: decoder id %lld outside [0, %d)", v, h->c.V);
  return B200T5_OK;
}

// A prompt of one id shared by every row is the start token of an ordinary call.
static bool one_start(const std::vector<long long>& d, int P) {
  return P == 1 && std::all_of(d.begin(), d.end(), [&](long long v) { return v == d[0]; });
}

// A static batch of B rows after the decoder prompt d [B][P] (P > 1, or rows that start from different ids); its
// results stay in the plan's buffers (copy_results with col0 = P - 1).
static int generate_prefixed_impl(b200t5_ctx* h, const long long* ids, const long long* mask, int B, int S, const b200t5_gen_params* gp,
                                  CallArgs& a, const std::vector<long long>& d, int P, cudaStream_t s) {
  const Cfg& c = h->c;
  const int T = a.T, Tp = P - 1;
  TRY(ensure_plan(h, B, S, Tp + T, 1, Tp));
  Plan& p = *h->plan;
  a.first = Tp;
  a.ph.cfg.begin_t = Tp;
  p.mode = a.mode(false);
  TRY(setup_proc(h, a.ph, s));
  TRY(setup_score(h, a.sh, s));
  if (Tp > 0) TRY(ensure_fwd_bias(h, Tp));
  // the prefill's ids [B][Tp] (columns 0 .. P-2), then the prompt [B][P]
  std::vector<long long> staged(static_cast<size_t>(B) * (Tp + P));
  for (int b = 0; b < B; ++b)
    for (int t = 0; t < Tp; ++t) staged[static_cast<size_t>(b) * Tp + t] = d[static_cast<size_t>(b) * P + t];
  std::copy(d.begin(), d.end(), staged.begin() + static_cast<size_t>(B) * Tp);
  if (p.pre_ids.bytes < staged.size() * 8) CU_OK(h, p.pre_ids.alloc(staged.size() * 8));
  CU_OK(h, cudaMemcpyAsync(p.pre_ids.p, staged.data(), staged.size() * 8, cudaMemcpyHostToDevice, s));
  const long long* prompt = p.pre_ids.as<long long>() + static_cast<size_t>(B) * Tp;
  p.prompt_steps = Tp;
  h->launches = 0;
  CU_OK(h, cudaEventRecord(h->ev[0], s));
  TRY(run_encoder(h, ids, mask, s));
  TRY(run_cross_kv(h, s));
  TRY(ensure_graph(h, static_cast<double>(p.rows_valid) / (static_cast<double>(B) * S)));
  if (Tp > 0) {
    const int M = B * Tp;
    embed_rows_kernel<<<(M + 7) / 8, 256, 0, s>>>(p.pre_ids.as<long long>(), h->shared.as<act_t>(), p.x.as<res_t>(), M, c.d, c.V);
    h->launches++;
    TRY(run_decoder_forward(h, Tp, s, true));
  }
  TRY(begin_static_decode(h, a, s, prompt, P));
  if (p.mode.proc) {
    proc_reset_kernel<<<B, 128, 0, s>>>(p.proc.dev(), nullptr, ids, p.batch.ids.as<long long>(), p.Tmax + 1, nullptr, P);
    h->launches++;
  }
  if (p.mode.score) {
    score_reset_kernel<<<B, 128, 0, s>>>(p.batch.lp.as<float>(), p.batch.lg.as<float>(), static_cast<size_t>(B) * p.Tmax, p.ftok.as<int>(),
                                         B, nullptr, nullptr, nullptr, p.Tmax);
    h->launches++;
  }
  TRY(run_static_steps(h, gp, T, a.min_new < T, s));
  if (Tp > 0) {
    prompt_len_kernel<<<(B + 127) / 128, 128, 0, s>>>(p.batch.len.as<int>(), B, Tp);
    h->launches++;
    CU_OK(h, cudaGetLastError());
  }
  return B200T5_OK;
}

extern "C" int b200t5_generate_prefixed(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                        const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                                        int32_t* out_len, const b200t5_score_io* score, const int64_t* decoder_input_ids, int P,
                                        void* stream) {
  CallArgs a;
  TRY(set_up_call(h, B, S, B, params, input_ids, out_ids, out_len, logits, score, false, &a));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<long long> d;
  TRY(read_prompt(h, decoder_input_ids, B, P, params, score, &d));
  if (one_start(d, P)) {  // exactly b200t5_generate_scored with that start token
    a.start = d[0];
    TRY(generate_impl(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask), B, S,
                      params, a, s));
    return copy_results(h, static_cast<size_t>(B), out_ids, out_len, a.sh.on ? score->token_logprobs : nullptr,
                        a.sh.on ? score->token_logits : nullptr, cudaMemcpyDeviceToDevice, s);
  }
  TRY(generate_prefixed_impl(h, reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(attention_mask), B, S,
                             params, a, d, P, s));
  return copy_results(h, static_cast<size_t>(B), out_ids, out_len, a.sh.on ? score->token_logprobs : nullptr,
                      a.sh.on ? score->token_logits : nullptr, cudaMemcpyDeviceToDevice, s, P - 1);
}

extern "C" int b200t5_generate_host_prefixed(b200t5_handle h, const int64_t* input_ids, const int64_t* attention_mask, int B, int S,
                                             const b200t5_gen_params* params, const b200t5_logits_params* logits, int64_t* out_ids,
                                             int32_t* out_len, const b200t5_score_io* score, const int64_t* decoder_input_ids, int P) {
  CallArgs a;
  TRY(set_up_call(h, B, S, B, params, input_ids, out_ids, out_len, logits, score, true, &a));
  std::vector<long long> d;
  TRY(read_prompt(h, decoder_input_ids, B, P, params, score, &d));
  if (one_start(d, P)) {
    b200t5_gen_params gp = *params;
    gp.decoder_start_token_id = d[0];
    return b200t5_generate_host_scored(h, input_ids, attention_mask, B, S, &gp, logits, out_ids, out_len, score);
  }
  const int Tmax = P - 1 + a.T;
  TRY(ensure_plan(h, B, S, Tmax, 1, P - 1));
  Plan& p = *h->plan;
  cudaStream_t s = h->exec_stream;
  const size_t nb = static_cast<size_t>(B) * S * 8;
  memcpy(p.h_ids, input_ids, nb);
  CU_OK(h, cudaMemcpyAsync(p.ids_dev.p, p.h_ids, nb, cudaMemcpyHostToDevice, s));
  if (attention_mask) {
    memcpy(p.h_mask, attention_mask, nb);
    CU_OK(h, cudaMemcpyAsync(p.mask_dev.p, p.h_mask, nb, cudaMemcpyHostToDevice, s));
  }
  TRY(generate_prefixed_impl(h, p.ids_dev.as<long long>(), attention_mask ? p.mask_dev.as<long long>() : nullptr, B, S, params, a, d, P, s));
  TRY(copy_results(h, static_cast<size_t>(B), p.h_out, p.h_len, a.sh.on ? score->token_logprobs : nullptr,
                   a.sh.on ? score->token_logits : nullptr, cudaMemcpyDeviceToHost, s, P - 1));
  CU_OK(h, cudaStreamSynchronize(s));
  memcpy(out_ids, p.h_out, static_cast<size_t>(B) * (Tmax + 1) * 8);
  memcpy(out_len, p.h_len, static_cast<size_t>(B) * 4);
  return B200T5_OK;
}

extern "C" int b200t5_test_prefill_cache(b200t5_handle h, int layer, void* kv_out, void* stream) {
  if (!h || !h->plan || !kv_out) return fail(h, B200T5_EINVAL, "prefill cache: no plan or null argument");
  Plan& p = *h->plan;
  if (layer < 0 || layer >= h->c.Ld) return fail(h, B200T5_EINVAL, "prefill cache: layer %d outside [0, %d)", layer, h->c.Ld);
  if (p.prompt_steps < 1) return fail(h, B200T5_EINVAL, "prefill cache: the last call had no decoder prompt of two or more ids");
  CU_OK(h, cudaSetDevice(h->device));
  const size_t row = static_cast<size_t>(p.prompt_steps) * 64 * 2, pitch = static_cast<size_t>(p.Tmax) * 64 * 2;
  const act_t* src = p.self_kv.as<act_t>() + static_cast<size_t>(layer) * 2 * p.B * h->c.I * p.Tmax;
  CU_OK(h, cudaMemcpy2DAsync(kv_out, row, src, pitch, row, static_cast<size_t>(2) * p.B * h->c.H, cudaMemcpyDeviceToDevice,
                             static_cast<cudaStream_t>(stream)));
  return B200T5_OK;
}

// ================================================================== single-kernel hooks
[[maybe_unused]] static int hook_device(int device) {
  int sms = check_device(nullptr, device);
  if (sms < 0) return sms;
  cudaError_t e = init_kernel_attrs();
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "kernel attribute setup failed: %s", cudaGetErrorString(e));
  return sms;
}

// The GeGLU epilogue's gelu table, built with `pow_mode`; the fp16 build evaluates gelu_new directly and has none.
static int hook_gelu_lut(int pow_mode, GeluLut* lut) {
#if B200T5_F16
  (void)pow_mode;
  *lut = GeluLut{nullptr, 0, 0};
  return B200T5_OK;
#else
  return ensure_gelu_lut(nullptr, pow_mode, lut);
#endif
}

// C (res_t, in/out) += the product, as one residual phase of the stream: mode 1 after the first feed-forward block,
// mode 5 in layer 0 (fp16 build: the stream is still fp16 there, so the sum is rounded; bf16 build: same as mode 1).
static EpiResidual::Params hook_residual(void* C, int N, int mode) {
  EpiResidual::Params ep{static_cast<res_t*>(C), static_cast<const res_t*>(C), N};
  if (mode == 5) ep.round_out = 1;
  return ep;
}

extern "C" int b200t5_test_gemm(int device, const void* A, const void* W, void* C, int M, int N, int K, int bn, int mode,
                                int pow_mode, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (K % 8) return fail(nullptr, B200T5_EINVAL, "K must be a multiple of 8");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // bn 512: the encoder configuration (128 x 256 tiles, weight loaded in 128-row boxes, gemm_2cta.cuh), modes 0/1/2/5/6;
  // bn 128: the fp32 logits of b200t5_decode_logits, mode 3, or the forward pass's ReLU product (128 x 128 tiles), mode 6
  if (!((bn == 512 && (mode == 0 || mode == 1 || mode == 2 || mode == 5 || mode == 6)) || (bn == 128 && (mode == 3 || mode == 6))))
    return fail(nullptr, B200T5_EINVAL, "test_gemm: bn=512 with mode 0/1/2/5/6, or bn=128 with mode 3/6");
  CUtensorMap ta, tb;
  if (!make_tmap(&ta, A, M, K, 128) || !make_tmap(&tb, W, N, K, 128)) return fail(nullptr, B200T5_ECUDA, "%s", g_err);
  b200t5_ctx dummy;
  dummy.num_sms = sms;
  cudaError_t e = cudaErrorInvalidValue;
  if (mode == 0) {
    EpiStore::Params ep{static_cast<act_t*>(C), N};
    e = run_gemm_2cta<EpiStore>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 1 || mode == 5) {
    const EpiResidual::Params ep = hook_residual(C, N, mode);
    e = run_gemm_2cta<EpiResidual>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 2) {
    GeluLut lut;
    int lrc = hook_gelu_lut(pow_mode, &lut);
    if (lrc != B200T5_OK) return lrc;
    EpiGeglu::Params ep{static_cast<ffh_t*>(C), N / 2, lut};
    e = run_gemm_2cta<EpiGeglu>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 6) {
    const EpiRelu::Params ep{static_cast<ffh_t*>(C), N};
    e = bn == 512 ? run_gemm_2cta<EpiRelu>(&dummy, ta, tb, M, N, K, ep, s) : launch_gemm<128, EpiRelu>(ta, tb, M, N, K, 0, ep, sms, s);
  } else {
    EpiStoreF32::Params ep{static_cast<float*>(C), N};
    e = launch_gemm<128, EpiStoreF32>(ta, tb, M, N, K, 1, ep, sms, s);
  }
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "test_gemm(bn=%d, mode=%d): %s", bn, mode, cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_enc_gemm(int device, const void* A, const void* W, void* C, int M, int N, int K, int kernel,
                                    int mode, int pow_mode, const int* row_b, const int* row_s, int B, int H, int S,
                                    void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (K % 8) return fail(nullptr, B200T5_EINVAL, "K must be a multiple of 8");
  if (kernel != 0 && kernel != 1) return fail(nullptr, B200T5_EINVAL, "test_enc_gemm: kernel in {0, 1}");
  if (mode == 3 && (H < 1 || S < 1 || B < 1 || N % (H * 64) || (!row_b) != (!row_s) || (!row_b && M != B * S)))
    return fail(nullptr, B200T5_EINVAL, "test_enc_gemm: bad cross-KV arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUtensorMap ta, tb;
  if (!make_tmap(&ta, A, M, K, 128) || !make_tmap(&tb, W, N, K, k2ctaBox)) return fail(nullptr, B200T5_ECUDA, "%s", g_err);
  b200t5_ctx dummy;
  dummy.num_sms = sms;
  dummy.enc_gemm_ws = kernel == 1;
  cudaError_t e = cudaErrorInvalidValue;
  act_t* Cb = static_cast<act_t*>(C);
  if (mode == 0) {
    EpiStore::Params ep{Cb, N};
    e = run_gemm_2cta<EpiStore>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 1 || mode == 5) {
    const EpiResidual::Params ep = hook_residual(C, N, mode);
    e = run_gemm_2cta<EpiResidual>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 2) {
    GeluLut lut;
    int lrc = hook_gelu_lut(pow_mode, &lut);
    if (lrc != B200T5_OK) return lrc;
    EpiGeglu::Params ep{static_cast<ffh_t*>(C), N / 2, lut};
    e = run_gemm_2cta<EpiGeglu>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 3) {
    EpiCrossKV::Params ep{Cb, B, H, S, row_b, row_s};
    e = run_gemm_2cta<EpiCrossKV>(&dummy, ta, tb, M, N, K, ep, s);
  } else if (mode == 6) {
    e = run_gemm_2cta<EpiRelu>(&dummy, ta, tb, M, N, K, EpiRelu::Params{static_cast<ffh_t*>(C), N}, s);
  }
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "test_enc_gemm(kernel=%d, mode=%d): %s", kernel, mode, cudaGetErrorString(e));
  return B200T5_OK;
}

// lm_head + the decode step's head exactly as chain_head launches it, for M rows at position `step`: the head with
// processors when `proc` or `logits` has an active processor (the row state built by proc_reset_kernel from the
// decoder ids hist [M, step+1] and the prompts enc_ids [M, S]), scored when `score` (teacher-forced when `forced`
// holds each row's label). W doubles as the embedding table of the gather. `vals`: the columns' values, not written
// by the plain head.
static int test_lm_head(const char* name, int device, const void* x, const void* W, int M, int V, int K, int step, int eos,
                        int min_new, const b200t5_logits_params* logits, bool proc, const int64_t* hist, const int64_t* enc_ids,
                        int S, bool score, const int64_t* forced, int64_t* tokens, float* logprob, float* logit, float* vals,
                        void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (!x || !W || !tokens || M < 1 || V < 2 || K % 8 || step < 0 || (proc && (!hist || !enc_ids || S < 1)) ||
      (score && (!logprob || !logit)))
    return fail(nullptr, B200T5_EINVAL, "%s: bad argument", name);
  ProcHost ph;
  int rc = parse_logits_params(nullptr, V, logits, eos, &ph);
  if (rc != B200T5_OK) return rc;
  proc = proc || ph.on;
  if (proc && (!hist || !enc_ids || S < 1)) return fail(nullptr, B200T5_EINVAL, "%s: processors need hist and enc_ids", name);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUtensorMap ta, tb;
  if (!make_tmap(&ta, x, M, K, 128) || !make_tmap(&tb, W, V, K, 128)) return fail(nullptr, B200T5_ECUDA, "%s", g_err);
  // result arrays [M, T] with T = step + 1 columns (+ 1 when forced: a further label keeps the row going)
  const int n_tiles = (V + 127) / 128, T = step + 1, out_ld = T + 1, Wd = (V + 31) / 32;
  const size_t mt = static_cast<size_t>(M) * n_tiles * 4, m4 = static_cast<size_t>(M) * 4;
  DevBuf pval, pidx, st, unf, out, len, xn, ext, psum, fval, ftok, fids, lp, lg;
  ProcBufs pb;
  bool ok = pval.alloc(mt) == cudaSuccess && pidx.alloc(mt) == cudaSuccess && st.alloc(sizeof(DecodeState)) == cudaSuccess &&
            unf.alloc(m4) == cudaSuccess && out.alloc(static_cast<size_t>(M) * out_ld * 8) == cudaSuccess && len.alloc(m4) == cudaSuccess &&
            xn.alloc(static_cast<size_t>(M) * K * sizeof(res_t)) == cudaSuccess && ext.alloc(m4) == cudaSuccess;
  if (ok && proc)
    ok = pb.alloc(M, S, Wd, std::min(Wd * 32, step + 2 + S + ph.cfg.n_bad), ph.bad_ids.size(), ph.bad_off.size()) == cudaSuccess;
  if (ok && score)
    ok = psum.alloc(mt) == cudaSuccess && fval.alloc(m4) == cudaSuccess && ftok.alloc(m4) == cudaSuccess &&
         lp.alloc(static_cast<size_t>(M) * T * 4) == cudaSuccess && lg.alloc(static_cast<size_t>(M) * T * 4) == cudaSuccess;
  if (ok && score && forced) ok = fids.alloc(static_cast<size_t>(M) * T * 8) == cudaSuccess;
  if (!ok) return fail(nullptr, B200T5_ENOMEM, "%s: allocation failed", name);
  b200t5_ctx dummy;
  dummy.num_sms = sms;
  decode_init_kernel<<<M, 128, 0, s>>>(st.as<DecodeState>(), unf.as<int>(), out.as<long long>(), len.as<int>(), out_ld, M, 0, 0,
                                       static_cast<const act_t*>(W), xn.as<res_t>(), K);
  set_state_kernel<<<1, 1, 0, s>>>(st.as<DecodeState>(), step);
  cudaError_t e = cudaSuccess;
  if (proc) {
    e = cudaMemcpy2DAsync(out.p, static_cast<size_t>(out_ld) * 8, hist, static_cast<size_t>(step + 1) * 8,
                          static_cast<size_t>(step + 1) * 8, M, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = pb.upload(ph, s);
    if (e == cudaSuccess)
      proc_reset_kernel<<<M, 128, 0, s>>>(pb.dev(), nullptr, reinterpret_cast<const long long*>(enc_ids), out.as<long long>(),
                                          out_ld, nullptr, step + 1);
  }
  // the row's label of this step sits in column `step` of its [M, T] label rows; score_reset_kernel reads column 0
  if (e == cudaSuccess && score && forced)
    e = cudaMemcpy2DAsync(fids.as<long long>() + step, static_cast<size_t>(T) * 8, forced, 8, 8, M, cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess && score) {
    score_reset_kernel<<<M, 128, 0, s>>>(lp.as<float>(), lg.as<float>(), static_cast<size_t>(M) * T, ftok.as<int>(), M, nullptr, nullptr,
                                         forced ? fids.as<long long>() + step : nullptr, T);
    e = cudaGetLastError();
  }
  LmHeadParams ep{};
  ep.pval = pval.as<float>();
  ep.pidx = pidx.as<int>();
  ep.n_tiles = n_tiles;
  ep.step = &st.as<DecodeState>()->step;
  ep.eos = eos;
  ep.min_new = min_new;
  if (proc) ep.pd = pb.dev();
  ep.vals = vals;
  ep.ldv = V;
  FinalizeArgs fa{ep.pval, ep.pidx, n_tiles, st.as<DecodeState>(), unf.as<int>(), out.as<long long>(), len.as<int>(), out_ld, -1, 0,
                  static_cast<const act_t*>(W), xn.as<res_t>(), K, ext.as<int>(), nullptr, nullptr, T, ep.pd, ScoreDev()};
  if (score) {
    ep.psum = psum.as<float>();
    ep.fval = fval.as<float>();
    ep.ftok = forced ? ftok.as<int>() : nullptr;
    fa.sd = {ep.psum, ep.fval, ftok.as<int>(), forced ? fids.as<long long>() : nullptr, lp.as<float>(), lg.as<float>()};
  }
  if (e == cudaSuccess) e = run_lm_head(&dummy, proc, score, ta, tb, M, V, K, ep, fa, s, false);
  if (e == cudaSuccess)
    e = cudaMemcpy2DAsync(tokens, 8, out.as<long long>() + step + 1, static_cast<size_t>(out_ld) * 8, 8, M, cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess && score)
    e = cudaMemcpy2DAsync(logprob, 4, lp.as<float>() + step, static_cast<size_t>(T) * 4, 4, M, cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess && score)
    e = cudaMemcpy2DAsync(logit, 4, lg.as<float>() + step, static_cast<size_t>(T) * 4, 4, M, cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "%s: %s", name, cudaGetErrorString(e));
  return B200T5_OK;
}

// the plain head: the lowest-index arg-max tie rule
extern "C" int b200t5_test_lm_argmax(int device, const void* x, const void* W, int M, int V, int K, int step, int eos,
                                     int min_new, int64_t* tokens, void* stream) {
  return test_lm_head("test_lm_argmax", device, x, W, M, V, K, step, eos, min_new, nullptr, false, nullptr, nullptr, 0, false,
                      nullptr, tokens, nullptr, nullptr, nullptr, stream);
}

// the head with processors, whatever `logits` holds
extern "C" int b200t5_test_lm_process(int device, const void* x, const void* W, int M, int V, int K, int step, int eos,
                                      int min_new, const b200t5_logits_params* logits, const int64_t* hist,
                                      const int64_t* enc_ids, int S, int64_t* tokens, float* vals, void* stream) {
  return test_lm_head("test_lm_process", device, x, W, M, V, K, step, eos, min_new, logits, true, hist, enc_ids, S, false,
                      nullptr, tokens, nullptr, nullptr, vals, stream);
}

// the scored head, with processors when `logits` has an active one
extern "C" int b200t5_test_lm_score(int device, const void* x, const void* W, int M, int V, int K, int step, int eos,
                                    int min_new, const b200t5_logits_params* logits, const int64_t* hist,
                                    const int64_t* enc_ids, int S, const int64_t* forced, int64_t* tokens, float* logprob,
                                    float* logit, float* vals, void* stream) {
  return test_lm_head("test_lm_score", device, x, W, M, V, K, step, eos, min_new, logits, false, hist, enc_ids, S, true, forced,
                      tokens, logprob, logit, vals, stream);
}

extern "C" int b200t5_test_gemm_splitk(int device, const void* A, const void* W, void* C, int M, int N, int K, int bn,
                                       int split, int mode, int pow_mode, void* aux, int Tmax, int step, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (K % 8) return fail(nullptr, B200T5_EINVAL, "K must be a multiple of 8");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if ((bn != 64 && bn != 128) || (split != 1 && split != 2 && split != 4 && split != 8))
    return fail(nullptr, B200T5_EINVAL, "test_gemm_splitk: bn in {64,128}, split in {1,2,4,8}");
  CUtensorMap ta, tb;
  if (!make_tmap(&ta, A, M, K, 128) || !make_tmap(&tb, W, N, K, bn)) return fail(nullptr, B200T5_ECUDA, "%s", g_err);
  b200t5_ctx dummy;
  dummy.num_sms = sms;
  b200t5_ctx::SkChoice ch{bn, split};
  cudaError_t e = cudaErrorInvalidValue;
  act_t* Cb = static_cast<act_t*>(C);
  DevBuf st;
  if (mode == 0) {
    EpiStore::Params ep{Cb, N};
    e = run_gemm_sk<EpiStore>(&dummy, ch, ta, tb, M, N, K, ep, s, false);
  } else if (mode == 1 || mode == 5) {
    const EpiResidual::Params ep = hook_residual(C, N, mode);
    e = run_gemm_sk<EpiResidual>(&dummy, ch, ta, tb, M, N, K, ep, s, false);
  } else if (mode == 2) {
    GeluLut lut;
    int lrc = hook_gelu_lut(pow_mode, &lut);
    if (lrc != B200T5_OK) return lrc;
    EpiGeglu::Params ep{static_cast<ffh_t*>(C), N / 2, lut};
    e = run_gemm_sk<EpiGeglu>(&dummy, ch, ta, tb, M, N, K, ep, s, false);
  } else if (mode == 4) {
    if (!aux || N % 192 || Tmax <= step) return fail(nullptr, B200T5_EINVAL, "test_gemm_splitk: bad QKV arguments");
    if (st.alloc(sizeof(DecodeState)) != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "alloc");
    set_state_kernel<<<1, 1, 0, s>>>(st.as<DecodeState>(), step);
    EpiQkvDecode::Params ep{Cb, static_cast<act_t*>(aux), &st.as<DecodeState>()->step, M, N / 192, Tmax};
    e = run_gemm_sk<EpiQkvDecode>(&dummy, ch, ta, tb, M, N, K, ep, s, false);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  } else if (mode == 6) {
    e = run_gemm_sk<EpiRelu>(&dummy, ch, ta, tb, M, N, K, EpiRelu::Params{static_cast<ffh_t*>(C), N}, s, false);
  }
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "test_gemm_splitk(bn=%d, split=%d, mode=%d): %s", bn, split, mode, cudaGetErrorString(e));
  return B200T5_OK;
}

// fp16 build only: the fp32-weight feed-forward output projection, R += A . W^T, through the tf32 two-pass product
// (A [M,F] fp32 holding fp16 values, W [N,F] fp32, R [M,N] fp32 in/out). kernel 0: the encoder GEMM (gemm_2cta.cuh),
// 1: cluster split-K decode kernel (bn in {64,128}, split in {1,2,4,8}).
extern "C" int b200t5_test_ffo(int device, const void* A, const void* W, void* R, int M, int N, int F, int kernel, int bn,
                               int split, void* stream) {
#if !B200T5_F16
  return fail(nullptr, B200T5_EINVAL, "b200t5_test_ffo exists in the fp16 build only (libb200t5_f16.so)");
#else
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (F % 4 || N % 4) return fail(nullptr, B200T5_EINVAL, "F and N must be multiples of 4");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int Fp = (F + 31) / 32 * 32;
  DevBuf wsplit;
  if (wsplit.alloc(static_cast<size_t>(N) * 2 * Fp * 4) != cudaSuccess) return fail(nullptr, B200T5_ENOMEM, "alloc failed");
  const size_t n = static_cast<size_t>(N) * Fp;
  split_tf32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(static_cast<const float*>(W), wsplit.as<float>(), N, F, Fp);
  CUtensorMap ta, tb;
  const int box_b = kernel == 0 ? 128 : bn;
  if (!make_tmap(&ta, A, M, F, 128, true) || !make_tmap(&tb, wsplit.p, N, 2 * Fp, box_b, true))
    return fail(nullptr, B200T5_ECUDA, "%s", g_err);
  EpiResidual::Params ep{static_cast<float*>(R), static_cast<const float*>(R), N};
  ep.round_acc = 0;
  ep.round_out = 0;
  cudaError_t e;
  if (kernel == 0) {
    e = launch_gemm_2cta<EpiResidual, true>(ta, tb, M, N, 2 * Fp, ep, sms, s, Fp / 32);
  } else {
    const int sp = splitk_factor(2 * Fp, split, kBK / 2);
    e = bn == 128 ? launch_gemm_splitk<128, EpiResidual, true>(ta, tb, M, N, 2 * Fp, sp, ep, s, false, Fp / 32)
                  : launch_gemm_splitk<64, EpiResidual, true>(ta, tb, M, N, 2 * Fp, sp, ep, s, false, Fp / 32);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "test_ffo: %s", cudaGetErrorString(e));
  return B200T5_OK;
#endif
}

extern "C" int b200t5_test_beam_step(int device, const float* logits, int B, int k, int V, int step, int T, int eos, int min_new,
                                     double length_penalty, int early_stopping, float* run_score, void* fin, int32_t* heur, float* lse,
                                     float* cand_lp, int32_t* cand_tok, int32_t* parent, int32_t* token, int32_t* retired, void* stream) {
  int rc = hook_device(device);
  if (rc < 0) return rc;
  if (B < 1 || k < 1 || k > kBeamMax || V < 2 * k || step < 0 || step >= T || early_stopping < 0 || early_stopping > 2)
    return fail(nullptr, B200T5_EINVAL, "bad beam step arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int rows = B * k;
  DevBuf prm, ls, hp, ht, hl, st, unf;
  const BeamParams bp{k, T, min_new, eos, early_stopping, early_stopping == 2 && length_penalty > 0.0};
  const std::vector<float> lsv = beam_len_scale(length_penalty, T);
  const std::vector<int> ones(rows, 1);
  if (prm.alloc(sizeof(bp)) || ls.alloc(T * 4) || hp.alloc(static_cast<size_t>(T) * rows * 4) || ht.alloc(static_cast<size_t>(T) * rows * 4) ||
      hl.alloc(static_cast<size_t>(T) * rows * 4) || st.alloc(sizeof(DecodeState)) || unf.alloc(rows * 4))
    return fail(nullptr, B200T5_ECUDA, "allocation failed");
  CU_OK(nullptr, cudaMemcpy(prm.p, &bp, sizeof(bp), cudaMemcpyHostToDevice));
  CU_OK(nullptr, cudaMemcpy(ls.p, lsv.data(), T * 4, cudaMemcpyHostToDevice));
  CU_OK(nullptr, cudaMemcpy(unf.p, ones.data(), rows * 4, cudaMemcpyHostToDevice));
  set_state_kernel<<<1, 1, 0, s>>>(st.as<DecodeState>(), step);
  const BeamDev d{prm.as<BeamParams>(), ls.as<float>(), logits, lse, cand_lp, cand_tok, run_score, hp.as<int>(), ht.as<int>(), hl.as<float>(),
                  static_cast<BeamFin*>(fin), heur, parent, rows};
  beam_row_kernel<<<rows, kBeamRowThreads, 0, s>>>(d, V, st.as<DecodeState>(), unf.as<int>());
  beam_select_kernel<<<B, 32, 0, s>>>(d, V, st.as<DecodeState>(), unf.as<int>(), nullptr, nullptr, nullptr, 0);
  cudaError_t e = cudaMemcpyAsync(token, ht.as<int>() + static_cast<size_t>(step) * rows, rows * 4, cudaMemcpyDeviceToDevice, s);
  std::vector<int> u(rows);
  if (e == cudaSuccess) e = cudaMemcpyAsync(u.data(), unf.p, rows * 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  for (int& x : u) x = !x;
  if (e == cudaSuccess) e = cudaMemcpy(retired, u.data(), rows * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "beam step: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_beam_reorder(int device, void* kv, int planes, int B, int k, int H, int Tmax, int step, const int32_t* parent,
                                        void* stream) {
  int rc = hook_device(device);
  if (rc < 0) return rc;
  if (planes < 1 || B < 1 || k < 1 || k > kBeamMax || H < 1 || step < 0 || step >= Tmax) return fail(nullptr, B200T5_EINVAL, "bad reorder arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DevBuf prm, st, unf;
  const BeamParams bp{k, Tmax, 0, 0, 0, 0};
  const std::vector<int> ones(B * k, 1);
  if (prm.alloc(sizeof(bp)) || st.alloc(sizeof(DecodeState)) || unf.alloc(B * k * 4)) return fail(nullptr, B200T5_ECUDA, "allocation failed");
  CU_OK(nullptr, cudaMemcpy(prm.p, &bp, sizeof(bp), cudaMemcpyHostToDevice));
  CU_OK(nullptr, cudaMemcpy(unf.p, ones.data(), B * k * 4, cudaMemcpyHostToDevice));
  set_state_kernel<<<1, 1, 0, s>>>(st.as<DecodeState>(), step);
  BeamDev d{};
  d.prm = prm.as<BeamParams>();
  d.parent = const_cast<int*>(parent);
  d.rows = B * k;
  beam_reorder_kernel<<<dim3(planes * H, B), kBeamReorderThreads, 0, s>>>(static_cast<act_t*>(kv), d, unf.as<int>(), st.as<DecodeState>(), H, Tmax,
                                                                         nullptr);
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "beam reorder: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_beam_replicate(int device, void* cross_kv, int32_t* extent, uint8_t* key_ok, int planes, int B, int k, int H,
                                          int S, void* stream) {
  int rc = hook_device(device);
  if (rc < 0) return rc;
  if (planes < 1 || B < 1 || k < 1 || k > kBeamMax || H < 1 || S < 1 || B * k > 65535) return fail(nullptr, B200T5_EINVAL, "bad replicate arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  beam_replicate_kernel<<<dim3(planes * H, B * k), 256, 0, s>>>(static_cast<act_t*>(cross_kv), extent, key_ok, B * k, k, H, S);
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "beam replicate: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_beam_search(int device, const float* logits, int B, int k, int V, int T, int eos, int min_new,
                                       double length_penalty, int early_stopping, int n, int64_t start, int64_t pad,
                                       const b200t5_beam_io* io, int32_t* steps, float* cand_lp, int32_t* cand_tok, void* stream) {
  int rc = hook_device(device);
  if (rc < 0) return rc;
  if (B < 1 || k < 2 || k > kBeamMax || V < 2 * k || T < 1 || early_stopping < 0 || early_stopping > 2 || n < 1 || n > k || !io ||
      !io->sequences || !io->lengths || (cand_lp == nullptr) != (cand_tok == nullptr))
    return fail(nullptr, B200T5_EINVAL, "bad beam search arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int rows = B * k;
  DevBuf prm, ls, clp, ctk, rsc, hp, ht, hl, fin, heur, par, st, unf;
  const BeamParams bp{k, T, min_new, eos, early_stopping, early_stopping == 2 && length_penalty > 0.0};
  const std::vector<float> lsv = beam_len_scale(length_penalty, T);
  const std::vector<int> ones(rows, 1);
  const size_t hist = static_cast<size_t>(T) * rows * 4;
  if (prm.alloc(sizeof(bp)) || ls.alloc(T * 4) || clp.alloc(rows * kBeamCand * 4) || ctk.alloc(rows * kBeamCand * 4) || rsc.alloc(rows * 4) ||
      hp.alloc(hist) || ht.alloc(hist) || hl.alloc(hist) || fin.alloc(static_cast<size_t>(B) * kBeamMax * sizeof(BeamFin)) ||
      heur.alloc(B * 4) || par.alloc(rows * 4) || st.alloc(sizeof(DecodeState)) || unf.alloc(rows * 4))
    return fail(nullptr, B200T5_ECUDA, "allocation failed");
  CU_OK(nullptr, cudaMemcpy(prm.p, &bp, sizeof(bp), cudaMemcpyHostToDevice));
  CU_OK(nullptr, cudaMemcpy(ls.p, lsv.data(), T * 4, cudaMemcpyHostToDevice));
  CU_OK(nullptr, cudaMemcpy(unf.p, ones.data(), rows * 4, cudaMemcpyHostToDevice));
  BeamDev d{prm.as<BeamParams>(), ls.as<float>(), nullptr, nullptr, clp.as<float>(), ctk.as<int>(), rsc.as<float>(), hp.as<int>(), ht.as<int>(),
            hl.as<float>(), fin.as<BeamFin>(), heur.as<int>(), par.as<int>(), rows};
  beam_init_kernel<<<(std::max(rows, B * kBeamMax) + 255) / 256, 256, 0, s>>>(d, B, k);
  // the decode loop of run_static_steps without the model: one unfinished array for the whole search, and a stop
  // once every prompt has retired
  std::vector<int> u(rows);
  int ran = 0;
  cudaError_t e = cudaSuccess;
  for (int t = 0; t < T && e == cudaSuccess; ++t) {
    d.logits = logits + static_cast<size_t>(t) * rows * V;
    if (cand_lp != nullptr) {
      d.cand_lp = cand_lp + static_cast<size_t>(t) * rows * kBeamCand;
      d.cand_tok = cand_tok + static_cast<size_t>(t) * rows * kBeamCand;
    }
    set_state_kernel<<<1, 1, 0, s>>>(st.as<DecodeState>(), t);
    beam_row_kernel<<<rows, kBeamRowThreads, 0, s>>>(d, V, st.as<DecodeState>(), unf.as<int>());
    beam_select_kernel<<<B, 32, 0, s>>>(d, V, st.as<DecodeState>(), unf.as<int>(), nullptr, nullptr, nullptr, 0);
    ++ran;
    e = cudaMemcpyAsync(u.data(), unf.p, rows * 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (std::all_of(u.begin(), u.end(), [](int x) { return x == 0; })) break;
  }
  if (e == cudaSuccess) {
    beam_output_kernel<<<(B * n + 127) / 128, 128, 0, s>>>(d, B, n, reinterpret_cast<long long*>(io->sequences), io->lengths,
                                                            io->sequences_scores, reinterpret_cast<long long*>(io->beam_indices),
                                                            io->token_logprobs, start, pad);
    e = cudaStreamSynchronize(s);
  }
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "beam search: %s", cudaGetErrorString(e));
  if (steps != nullptr) *steps = ran;
  return B200T5_OK;
}

extern "C" int b200t5_test_rmsnorm(int device, const void* x, const void* w, void* y, int M, int d, float eps, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  cudaError_t e = run_rmsnorm(nullptr, static_cast<const res_t*>(x), static_cast<const act_t*>(w), static_cast<act_t*>(y), M, d, eps, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "rmsnorm: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_rmsnorm_scaled(int device, const void* x, const void* w, void* y, int M, int d, float eps, float scale,
                                          void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (!(scale != 0.f)) return fail(nullptr, B200T5_EINVAL, "test_rmsnorm_scaled: scale must be nonzero");
  cudaError_t e = run_rmsnorm(nullptr, static_cast<const res_t*>(x), static_cast<const act_t*>(w), static_cast<act_t*>(y), M, d, eps,
                              static_cast<cudaStream_t>(stream), false, scale);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "rmsnorm_scaled: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_attn_decode(int device, int self, const void* q, const void* K, const void* V, void* ctx,
                                       int B, int H, int Tk, const int32_t* extent, const uint8_t* key_ok, int step,
                                       const float* dist_bias, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (self == 1) return fail(nullptr, B200T5_EINVAL, "attn_decode: self in {0, 2, 3}");
  if (self == 3) {
    // the position: `step` for every row (static batch), or extent[b] for row b (slot pool, step_stride 1)
    DevBuf st;
    if (st.alloc(sizeof(DecodeState)) != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "alloc");
    set_state_kernel<<<1, 1, 0, s>>>(st.as<DecodeState>(), step);
    const int* pos = extent ? extent : &st.as<DecodeState>()->step;
    const int stride = extent ? 1 : 0;
    const act_t *qa = static_cast<const act_t*>(q), *Ka = static_cast<const act_t*>(K), *Va = static_cast<const act_t*>(V);
    attn_decode_kernel<true><<<B * H, kAttnDecThreads, Tk * sizeof(float), s>>>(
        qa, Ka, Va, static_cast<act_t*>(ctx), H, Tk, nullptr, nullptr, pos, dist_bias, XsStamps{nullptr, 0}, stride);
    cudaStreamSynchronize(s);
  } else if (self == 2) {  // the TMA stream kernel (attention_cross_stream.cuh); `step` = ring stages (0: 5)
    const int stages = step > 0 ? step : 5;
    if (stages < 2 || stages > kXsMaxStages || Tk > 4096) return fail(nullptr, B200T5_EINVAL, "attn_decode(stream): 2 <= stages <= %d, Tk <= 4096", kXsMaxStages);
    const int items = B * H;
    CUtensorMap tk, tv;
    if (!make_tmap(&tk, K, static_cast<uint64_t>(items) * Tk, 64, kXsChunkKeys) || !make_tmap(&tv, V, static_cast<uint64_t>(items) * Tk, 64, kXsChunkKeys))
      return fail(nullptr, B200T5_ECUDA, "%s", g_err);
    attn_cross_stream_kernel<<<xs_grid(items, sms), kXsThreads, XsSmem::bytes(stages, Tk), s>>>(
        tk, tv, 0, 0, static_cast<const act_t*>(q), static_cast<act_t*>(ctx), items, H, Tk, extent, key_ok, stages, XsStamps{nullptr, 0});
  } else {
    attn_decode_kernel<false><<<B * H, kAttnDecThreads, Tk * sizeof(float), s>>>(
        static_cast<const act_t*>(q), static_cast<const act_t*>(K), static_cast<const act_t*>(V), static_cast<act_t*>(ctx), H,
        Tk, extent, key_ok, nullptr, nullptr, XsStamps{nullptr, 0});
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "attn_decode: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_encoder_attn(int device, const void* qkv, void* ctx, const float* rel_bias,
                                        const uint8_t* key_ok, const int32_t* extent, int B, int S, int H, int impl,
                                        void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  // impl 1: the packed-row addressing the encoder uses (prompt b at rows cu[b] = b * S, only its extent computed)
  DevBuf cu;
  if (impl == 1) {
    std::vector<int> hcu(B);
    for (int b = 0; b < B; ++b) hcu[b] = b * S;
    if (cu.alloc(B * sizeof(int)) != cudaSuccess || cudaMemcpy(cu.p, hcu.data(), B * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess)
      return fail(nullptr, B200T5_ECUDA, "encoder_attn: offsets");
  }
  const size_t smem = encoder_attn_smem_bytes(S);
  cudaError_t e = smem <= 96 * 1024 ? cudaSuccess : cudaErrorInvalidValue;
  if (e == cudaSuccess) {
    encoder_attn_kernel<<<dim3((S + kEncQ - 1) / kEncQ, B * H), kEncThreads, smem, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const act_t*>(qkv), static_cast<act_t*>(ctx), rel_bias, key_ok, extent, impl == 1 ? cu.as<int>() : nullptr, S, H);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "encoder_attn: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_decoder_self_attn(int device, const void* qkv, void* ctx, const float* dist_bias, int B, int T, int H,
                                             void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (!qkv || !ctx || !dist_bias || B < 1 || H < 1 || T < 1 || T > 4096) return fail(nullptr, B200T5_EINVAL, "decoder_self_attn: bad argument");
  decoder_attn_kernel<kAttnCausal><<<dim3((T + kEncQ - 1) / kEncQ, B * H), kEncThreads, encoder_attn_smem_bytes(T), static_cast<cudaStream_t>(stream)>>>(
      static_cast<const act_t*>(qkv), nullptr, static_cast<act_t*>(ctx), dist_bias, nullptr, nullptr, B, T, T, H);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "decoder_self_attn: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_decoder_cross_attn(int device, const void* q, const void* kv, void* ctx, const uint8_t* key_ok,
                                              const int32_t* extent, int B, int T, int S, int H, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (!q || !kv || !ctx || !key_ok || !extent || B < 1 || H < 1 || T < 1 || S < 1 || encoder_attn_smem_bytes(S) > 96 * 1024)
    return fail(nullptr, B200T5_EINVAL, "decoder_cross_attn: bad argument");
  decoder_attn_kernel<kAttnCross><<<dim3((T + kEncQ - 1) / kEncQ, B * H), kEncThreads, encoder_attn_smem_bytes(S), static_cast<cudaStream_t>(stream)>>>(
      static_cast<const act_t*>(q), static_cast<const act_t*>(kv), static_cast<act_t*>(ctx), nullptr, key_ok, extent, B, T, S, H);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "decoder_cross_attn: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_decoder_cross_attn_packed(int device, const void* q, const void* kv, void* ctx, const uint8_t* key_ok,
                                                     const int32_t* extent, const int32_t* qoff, int B, int S, int H, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  if (!q || !kv || !ctx || !key_ok || !extent || !qoff || B < 1 || H < 1 || S < 1 || B * H > 65535 ||
      encoder_attn_smem_bytes(S) > 96 * 1024)
    return fail(nullptr, B200T5_EINVAL, "decoder_cross_attn_packed: bad argument");
  // the grid spans the longest prompt's query tiles: the offsets are read back
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<int> h_off(B + 1);
  cudaError_t e = cudaMemcpyAsync(h_off.data(), qoff, (B + 1) * sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "decoder_cross_attn_packed: %s", cudaGetErrorString(e));
  int tiles = 0;
  for (int b = 0; b < B; ++b) {
    if (h_off[b + 1] < h_off[b]) return fail(nullptr, B200T5_EINVAL, "decoder_cross_attn_packed: offsets decrease at %d", b);
    tiles = std::max(tiles, (h_off[b + 1] - h_off[b] + kEncQ - 1) / kEncQ);
  }
  if (tiles == 0) return B200T5_OK;
  decoder_cross_packed_kernel<<<dim3(tiles, B * H), kEncThreads, encoder_attn_smem_bytes(S), st>>>(
      static_cast<const act_t*>(q), static_cast<const act_t*>(kv), static_cast<act_t*>(ctx), key_ok, extent, qoff, B, S, H);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "decoder_cross_attn_packed: %s", cudaGetErrorString(e));
  return B200T5_OK;
}

extern "C" int b200t5_test_geglu(int device, const void* gate, const void* up, void* out, int64_t n, int pow_mode, void* stream) {
  const int sms = hook_device(device);
  if (sms < 0) return sms;
  GeluLut lut;
  int lrc = hook_gelu_lut(0, &lut);
  if (lrc != B200T5_OK) return lrc;
  geglu_elementwise_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const act_t*>(gate), static_cast<const act_t*>(up), static_cast<act_t*>(out), n, pow_mode, lut);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, B200T5_ECUDA, "geglu: %s", cudaGetErrorString(e));
  return B200T5_OK;
}
