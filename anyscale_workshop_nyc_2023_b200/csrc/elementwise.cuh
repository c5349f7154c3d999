// Memory-bound row kernels: embedding gather, T5 RMSNorm, mask preparation,
// per-step arg-max finalisation + stopping bookkeeping.
#pragma once
#include "logits_process.cuh"
#include "ptx.cuh"

namespace b200 {

// 8 consecutive residual-stream elements as floats (bf16 build: one 16-byte load; fp16 build: the stream is fp32)
DEVINL void load_res8(const res_t* p, float (&f)[8]) {
#if B200T5_F16
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
#else
  const uint4 v = *reinterpret_cast<const uint4*>(p);
  f[0] = act_lo(v.x); f[1] = act_hi(v.x); f[2] = act_lo(v.y); f[3] = act_hi(v.y);
  f[4] = act_lo(v.z); f[5] = act_hi(v.z); f[6] = act_lo(v.w); f[7] = act_hi(v.w);
#endif
}
// the same 8 elements written from a row of the embedding table (act_t values widen exactly)
DEVINL void store_res8_from_act(res_t* dst, const uint4& e) {
#if B200T5_F16
  reinterpret_cast<float4*>(dst)[0] = make_float4(act_lo(e.x), act_hi(e.x), act_lo(e.y), act_hi(e.y));
  reinterpret_cast<float4*>(dst)[1] = make_float4(act_lo(e.z), act_hi(e.z), act_lo(e.w), act_hi(e.w));
#else
  *reinterpret_cast<uint4*>(dst) = e;
#endif
}


// ---------------------------------------------------------------- embedding gather
// x[m, :] = E[ids[m], :]   (modeling_t5.py:682).  One warp per row, 16-B vectors.
__global__ void embed_rows_kernel(const long long* __restrict__ ids, const act_t* __restrict__ E,
                                  res_t* __restrict__ x, int M, int d, int vocab) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  long long id = ids[row];
  if (id < 0 || id >= vocab) id = 0;  // HF would raise an index error; ids are validated on the host
  const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(id) * d);
  res_t* dst = x + static_cast<size_t>(row) * d;
  for (int i = lane_id(); i < d / 8; i += 32) store_res8_from_act(dst + i * 8, src[i]);
}

// ---------------------------------------------------------------- packed (variable-length) encoder rows
// The reference pads every prompt to 512 tokens (JOB/utils.py:23-27) and HF runs the encoder over all of them.
// Rows at or beyond extent[b] (the last attended position + 1) are never read downstream - the keys are
// masked out of every attention and the cross-attention stops at extent[b] - so the encoder here runs on
// the valid rows only, packed back to back: row cu[b] + s holds position s of prompt b.
// One CTA: exclusive scan of extent[] -> cu[0..B]; cu[B] = number of packed rows.
__global__ void pack_offsets_kernel(const int* __restrict__ extent, int* __restrict__ cu, int B) {
  __shared__ int s_part[32];
  __shared__ int s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < B; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = i < B ? extent[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane_id() >= static_cast<uint32_t>(o)) x += y;
    }
    if (lane_id() == 31) s_part[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = threadIdx.x < (blockDim.x >> 5) ? s_part[threadIdx.x] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane_id() >= static_cast<uint32_t>(o)) w += y;
      }
      s_part[threadIdx.x] = w;  // inclusive over warps
    }
    __syncthreads();
    const int warp_off = (threadIdx.x >> 5) ? s_part[(threadIdx.x >> 5) - 1] : 0;
    const int incl = s_carry + warp_off + x;
    if (i < B) cu[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) cu[B] = s_carry;
}

// row tables for the packed layout + embedding gather: x[cu[b] + s, :] = E[ids[b, s], :]
__global__ void embed_rows_packed_kernel(const long long* __restrict__ ids, const act_t* __restrict__ E,
                                         res_t* __restrict__ x, const int* __restrict__ cu,
                                         int* __restrict__ row_b, int* __restrict__ row_s, int S, int d, int vocab) {
  const int b = blockIdx.y;
  const int n = cu[b + 1] - cu[b];
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= n) return;
  const int row = cu[b] + s;
  if (lane_id() == 0) {
    row_b[row] = b;
    row_s[row] = s;
  }
  long long id = ids[static_cast<size_t>(b) * S + s];
  if (id < 0 || id >= vocab) id = 0;
  const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(id) * d);
  res_t* dst = x + static_cast<size_t>(row) * d;
  for (int i = lane_id(); i < d / 8; i += 32) store_res8_from_act(dst + i * 8, src[i]);
}

// test hook: packed rows back to the padded [B*S, d] layout (rows beyond extent[b] are zero)
__global__ void unpack_rows_kernel(const act_t* __restrict__ xp, const int* __restrict__ cu,
                                   act_t* __restrict__ out, int S, int d) {
  const int b = blockIdx.y;
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= S) return;
  const int n = cu[b + 1] - cu[b];
  uint4* dst = reinterpret_cast<uint4*>(out + (static_cast<size_t>(b) * S + s) * d);
  const uint4* src = reinterpret_cast<const uint4*>(xp + static_cast<size_t>(cu[b] + s) * d);
  for (int i = lane_id(); i < d / 8; i += 32) dst[i] = s < n ? src[i] : make_uint4(0, 0, 0, 0);
}

// ---------------------------------------------------------------- T5 RMSNorm
// HF (modeling_t5.py:55-68), bf16 weights:
//   var = mean(float(x)^2)                      fp32
//   y1  = bf16( float(x) * rsqrt(var + eps) )   first rounding
//   y   = bf16( float(w) * float(y1) )          second rounding
// One warp per row; the row stays in registers between the two passes.
template <int kMaxVec>  // 8-element vectors per lane: d <= kMaxVec * 256
__global__ void rmsnorm_kernel(const res_t* __restrict__ x, const act_t* __restrict__ w,
                               act_t* __restrict__ y, int M, int d, float eps) {
  pdl_launch_dependents();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = lane_id();
  const int nvec = d >> 3;
  // the norm weights never depend on the previous kernel: fetch them before waiting for it
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4 wv[kMaxVec];
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) wv[i] = wr[idx];
  }
  pdl_wait();
  if (row >= M) return;
  const res_t* xr = x + static_cast<size_t>(row) * d;
  float v[kMaxVec][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      load_res8(xr + idx * 8, v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss = fmaf(v[i][j], v[i][j], ss);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = rsqrtf(ss * (1.0f / static_cast<float>(d)) + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + static_cast<size_t>(row) * d);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const uint32_t ws[4] = {wv[i].x, wv[i].y, wv[i].z, wv[i].w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float a = act_round(v[i][2 * j] * inv);
        const float b = act_round(v[i][2 * j + 1] * inv);
        o[j] = pack_act2(act_lo(ws[j]) * a, act_hi(ws[j]) * b);
      }
      yr[idx] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// ---------------------------------------------------------------- attention-mask preparation
// attention_mask int64 [B,S] -> key_ok uint8 [B,S] and extent[b] = 1 + index of the last
// attended key. A row with no attended key gets extent = S: every score is then
// finfo(bf16).min and the fp32 softmax is uniform over all S keys, exactly what
// HF's additive mask produces (masking_utils.py:610-612, modeling_t5.py:323-331).
// row_on (optional, slot pool admission): rows with row_on[b] == 0 are not part of this encoder pass at all:
// extent 0, so the packed encoder and the cross-KV projection never touch their rows.
__global__ void prep_mask_kernel(const long long* __restrict__ mask, unsigned char* __restrict__ key_ok,
                                 int* __restrict__ extent, int B, int S, const int* __restrict__ row_on = nullptr) {
  const int b = blockIdx.x;
  if (b >= B) return;
  if (row_on != nullptr && !row_on[b]) {
    for (int j = threadIdx.x; j < S; j += blockDim.x) key_ok[static_cast<size_t>(b) * S + j] = 0;
    if (threadIdx.x == 0) extent[b] = 0;
    return;
  }
  int last = -1;
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    const bool ok = mask == nullptr ? true : mask[static_cast<size_t>(b) * S + j] != 0;
    key_ok[static_cast<size_t>(b) * S + j] = ok ? 1 : 0;
    if (ok) last = j;
  }
  __shared__ int s_last;
  if (threadIdx.x == 0) s_last = -1;
  __syncthreads();
  atomicMax(&s_last, last);
  __syncthreads();
  if (threadIdx.x == 0) extent[b] = s_last < 0 ? S : s_last + 1;
}

// ---------------------------------------------------------------- decode state
struct DecodeState {
  int step;            // current decode position t (0-based)
  int finished_rows;   // rows that have emitted EOS
  int pad0, pad1;
};

// Start of generate(): x_dec[b] = E[decoder_start], out[b][0] = decoder_start, flags reset.
__global__ void decode_init_kernel(DecodeState* st, int* __restrict__ unfinished, long long* __restrict__ out_ids,
                                   int* __restrict__ out_len, int out_ld, int B, long long start_tok,
                                   long long pad_tok, const act_t* __restrict__ E,
                                   res_t* __restrict__ x, int d) {
  const int b = blockIdx.x;
  if (b == 0 && threadIdx.x == 0) {
    st->step = 0;
    st->finished_rows = 0;
  }
  if (b >= B) return;
  for (int j = threadIdx.x; j < out_ld; j += blockDim.x)
    out_ids[static_cast<size_t>(b) * out_ld + j] = j == 0 ? start_tok : pad_tok;
  if (threadIdx.x == 0) {
    unfinished[b] = 1;
    out_len[b] = 0;
  }
  const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(start_tok) * d);
  res_t* dst = x + static_cast<size_t>(b) * d;
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) store_res8_from_act(dst + i * 8, src[i]);
}

// ---------------------------------------------------------------- slot pool (b200t5_generate_stream)
// Start of a streamed run: result rows = [start, pad, ...], every slot idle (position 0, nothing to attend,
// decoder input = E[pad] so that idle slots compute on finite numbers).
__global__ void stream_init_kernel(DecodeState* st, int* __restrict__ unfinished, int* __restrict__ pos,
                                   int* __restrict__ live_extent, long long* __restrict__ out_ids,
                                   int* __restrict__ out_len, int out_ld, int N, int B, long long start_tok,
                                   long long pad_tok, const act_t* __restrict__ E, res_t* __restrict__ x,
                                   int d) {
  const int r = blockIdx.x;
  if (r == 0 && threadIdx.x == 0) {
    st->step = 0;
    st->finished_rows = 0;
  }
  if (r < N) {
    for (int j = threadIdx.x; j < out_ld; j += blockDim.x)
      out_ids[static_cast<size_t>(r) * out_ld + j] = j == 0 ? start_tok : pad_tok;
    if (threadIdx.x == 0) out_len[r] = 0;
  }
  if (r < B) {
    if (threadIdx.x == 0) {
      unfinished[r] = 0;
      pos[r] = 0;
      live_extent[r] = 0;
    }
    const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(pad_tok) * d);
    res_t* dst = x + static_cast<size_t>(r) * d;
    for (int i = threadIdx.x; i < d / 8; i += blockDim.x) store_res8_from_act(dst + i * 8, src[i]);
  }
}

// Admission of n prompts whose encoder pass has just run: slot slots[i] starts prompt rows[i] at position 0.
__global__ void admit_slots_kernel(const int* __restrict__ slots, const int* __restrict__ rows, int* __restrict__ unfinished,
                                   int* __restrict__ pos, int* __restrict__ out_row, const int* __restrict__ extent,
                                   int* __restrict__ live_extent, const unsigned char* __restrict__ key_ok,
                                   unsigned char* __restrict__ live_key_ok, int S, long long start_tok,
                                   const act_t* __restrict__ E, res_t* __restrict__ x, int d) {
  const int b = slots[blockIdx.x];
  if (threadIdx.x == 0) {
    unfinished[b] = 1;
    pos[b] = 0;
    out_row[b] = rows[blockIdx.x];
    live_extent[b] = extent[b];
  }
  for (int j = threadIdx.x; j < S; j += blockDim.x) live_key_ok[static_cast<size_t>(b) * S + j] = key_ok[static_cast<size_t>(b) * S + j];
  const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(start_tok) * d);
  res_t* dst = x + static_cast<size_t>(b) * d;
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) store_res8_from_act(dst + i * 8, src[i]);
}

// One CTA per row: reduce the per-tile (max, index) partials of the fused lm_head
// epilogue with the torch.argmax tie rule (lowest index), then HF's greedy
// bookkeeping (generation/utils.py:2793-2805):
//   tok = unfinished ? argmax : pad ; out[b, t+1] = tok ; unfinished &= tok != eos
// and fetch the embedding of tok as the next step's decoder input.
// A finished row is RETIRED: live_extent[b] = 0, so the cross-attention of the remaining steps no longer streams
// its K/V (its outputs are pad tokens whatever it computes).
// Slot-pool mode (pos != nullptr, b200t5_generate_stream): every slot has its own position pos[b] and writes to
// row out_row[b] of an [N, out_ld] result; a slot also finishes when it has emitted max_new tokens, idle slots
// (unfinished == 0) write nothing and stay at position 0.
// kProc (logits processors active): a row finishes on any of the call's EOS ids, and a row that goes on marks its
// token as seen and computes the bans of its next step (logits_process.cuh).
//
// kScore (token log-probabilities): the epilogue also left psum[b][i] = sum of expf(v - pval[b][i]) over tile i
// (gemm.cuh: EpiLmHead). They are merged in an order that depends on nothing but n_tiles and the 128-thread CTA -
// thread k adds tiles k, k + 128, ... in ascending order, the warp's lanes are folded by the xor tree, thread 0 adds the
// four warps in order:
//   M = max_i m_i,  S = sum_i s_i * expf(m_i - M),  lse = M + logf(S)
// so a row's numbers are bit-identical whichever row-chain, slot or batch it sits in. For an unfinished row at step t
//   logit[row][t] = v_tok,  logprob[row][t] = v_tok - lse          (fp32 [rows, max_new]; untouched positions stay 0)
// where v_tok = M for the arg-max token. Teacher forcing (sd.forced != nullptr, int64 [rows, max_new], -100 after a
// row's last label): tok = forced[row][t] instead of the arg-max, v_tok = fval[b] (written by the tile holding that
// column), and the row finishes after its last label, not on EOS; ftok[b] becomes the next step's forced column.
struct ScoreDev {
  const float* psum = nullptr;   // [B][n_tiles]
  const float* fval = nullptr;   // [B]
  int* ftok = nullptr;           // [B]
  const long long* forced = nullptr;  // [rows][max_new]
  float* logprob = nullptr;      // [rows][max_new]
  float* logit = nullptr;        // [rows][max_new]
};

struct FinalizeArgs {
  const float* pval;  // [B][n_tiles]
  const int* pidx;    // [B][n_tiles]
  int n_tiles;
  DecodeState* st;
  int* unfinished;
  long long* out_ids;  // [rows][out_ld]
  int* out_len;        // [rows]
  int out_ld;
  long long eos_tok, pad_tok;
  const act_t* E;  // embedding table
  res_t* x;        // [B][d]: the next step's decoder input
  int d;
  int* live_extent;
  int* pos;            // slot pool: per-slot positions, else nullptr
  const int* out_row;  // slot pool: per-slot result rows, else nullptr
  int max_new;
  ProcDev pd;   // kProc
  ScoreDev sd;  // kScore
};

template <bool kProc, bool kScore>
__global__ void finalize_step_kernel(const FinalizeArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const int t = a.pos != nullptr ? a.pos[b] : a.st->step;
  float best = -INFINITY;
  int bidx = 0x7fffffff;
  for (int i = threadIdx.x; i < a.n_tiles; i += blockDim.x) {
    const float v = a.pval[static_cast<size_t>(b) * a.n_tiles + i];
    const int ix = a.pidx[static_cast<size_t>(b) * a.n_tiles + i];
    if (v > best || (v == best && ix < bidx)) {
      best = v;
      bidx = ix;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (ov > best || (ov == best && oi < bidx)) {
      best = ov;
      bidx = oi;
    }
  }
  __shared__ float s_v[32];
  __shared__ int s_i[32];
  __shared__ long long s_tok;
  __shared__ int s_go;
  const int warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  if (lane_id() == 0) {
    s_v[warp] = best;
    s_i[warp] = bidx;
  }
  __syncthreads();
  float ssum = 0.f;
  if constexpr (kScore) {
    __shared__ float s_s[32];
    float mx = s_v[0];
    for (int w = 1; w < nwarp; ++w) mx = fmaxf(mx, s_v[w]);
    for (int i = threadIdx.x; i < a.n_tiles; i += blockDim.x)
      ssum += a.sd.psum[static_cast<size_t>(b) * a.n_tiles + i] * expf(a.pval[static_cast<size_t>(b) * a.n_tiles + i] - mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, o);
    if (lane_id() == 0) s_s[warp] = ssum;
    __syncthreads();
    if (threadIdx.x == 0)
      for (int w = 1; w < nwarp; ++w) ssum += s_s[w];
  }
  if (threadIdx.x == 0) {
    for (int w = 1; w < nwarp; ++w) {
      if (s_v[w] > best || (s_v[w] == best && s_i[w] < bidx)) {
        best = s_v[w];
        bidx = s_i[w];
      }
    }
    const int unf = a.unfinished[b];
    const int row = a.out_row != nullptr ? a.out_row[b] : b;
    long long tok = unf ? static_cast<long long>(bidx) : a.pad_tok;
    bool forced = false;
    if constexpr (kScore) {
      forced = a.sd.forced != nullptr;
      if (unf) {
        float v_tok = best;
        if (forced) {
          tok = a.sd.forced[static_cast<size_t>(row) * a.max_new + t];
          v_tok = a.sd.fval[b];
        }
        a.sd.logprob[static_cast<size_t>(row) * a.max_new + t] = v_tok - (best + logf(ssum));
        if (a.sd.logit != nullptr) a.sd.logit[static_cast<size_t>(row) * a.max_new + t] = v_tok;
      }
    }
    if (a.pos == nullptr || unf) a.out_ids[static_cast<size_t>(row) * a.out_ld + t + 1] = tok;
    bool fin = false;
    if (unf) {
      a.out_len[row] = t + 1;
      if (forced) {
        fin = t + 1 >= a.max_new || a.sd.forced[static_cast<size_t>(row) * a.max_new + t + 1] < 0;
        a.sd.ftok[b] = fin ? -1 : static_cast<int>(a.sd.forced[static_cast<size_t>(row) * a.max_new + t + 1]);
      } else {
        fin = (kProc ? proc_is_eos(*a.pd.cfg, tok) : tok == a.eos_tok) || (a.pos != nullptr && t + 1 >= a.max_new);
      }
      if (fin) {
        a.unfinished[b] = 0;
        a.live_extent[b] = 0;
        atomicAdd(&a.st->finished_rows, 1);
      }
    }
    if (a.pos != nullptr) a.pos[b] = (unf && !fin) ? t + 1 : 0;
    s_tok = (a.pos != nullptr && fin) ? a.pad_tok : tok;
    if constexpr (kProc) {
      s_go = unf && !fin;
      if (unf && !fin && a.pd.cfg->rep_pen) bit_set(a.pd.seen + static_cast<size_t>(a.pd.row0 + b) * a.pd.W, static_cast<int>(tok));
    }
  }
  __syncthreads();
  const uint4* src = reinterpret_cast<const uint4*>(a.E + static_cast<size_t>(s_tok) * a.d);
  res_t* dst = a.x + static_cast<size_t>(b) * a.d;
  for (int i = threadIdx.x; i < a.d / 8; i += blockDim.x) store_res8_from_act(dst + i * 8, src[i]);
  if constexpr (kProc) {
    // the row's decoder ids are now its result row up to column t + 1 (written above, visible after the barrier)
    if (s_go) proc_new_bans(a.pd, a.pd.row0 + b, a.out_ids + static_cast<size_t>(a.out_row != nullptr ? a.out_row[b] : b) * a.out_ld, t + 2, true);
  }
}

// Start of a scored call, and of every row of it. With logprob != nullptr: zero the n result elements (positions a
// row never reaches stay 0, so a row's sum is its log-likelihood). For i < n_set: slot slots[i] (nullptr: i) starts
// row rows[i] (nullptr: i) and takes its first forced column, -1 without teacher forcing (idle slots, start of a pool).
__global__ void score_reset_kernel(float* __restrict__ logprob, float* __restrict__ logit, size_t n, int* __restrict__ ftok,
                                   int n_set, const int* __restrict__ slots, const int* __restrict__ rows,
                                   const long long* __restrict__ forced, int forced_ld) {
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x, nth = static_cast<size_t>(gridDim.x) * blockDim.x;
  if (logprob != nullptr)
    for (size_t i = tid; i < n; i += nth) {
      logprob[i] = 0.f;
      logit[i] = 0.f;
    }
  for (size_t i = tid; i < static_cast<size_t>(n_set); i += nth) {
    const int row = rows != nullptr ? rows[i] : static_cast<int>(i);
    ftok[slots != nullptr ? slots[i] : i] = forced != nullptr ? static_cast<int>(forced[static_cast<size_t>(row) * forced_ld]) : -1;
  }
}

// End of a step (joins every chain). With in-situ profiling on, fold the cross-attention launch stamps of this
// step ({min start, max end} per launch, attention_decode.cuh: XsStamps; slot = layer * n_chains + chain) into
//   acc[slot]                = {sum of launch durations in ns, launches}               and
//   acc[n_slots + layer]     = {sum over steps of the time during which AT LEAST ONE of the layer's launches ran, layers}
// - the second is what the HBM stream of a layer costs the step when the chains' launches overlap each other.
__global__ void advance_step_kernel(DecodeState* st, unsigned long long* __restrict__ stamps,
                                    unsigned long long* __restrict__ acc, int n_layers, int n_chains) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) st->step += 1;
  if (stamps != nullptr) {
    const int n_slots = n_layers * n_chains;
    for (int l = threadIdx.x; l < n_layers; l += blockDim.x) {
      unsigned long long t0[8], t1[8];
      int n = 0;
      bool all = true;
      for (int c = 0; c < n_chains && c < 8; ++c) {
        const int i = l * n_chains + c;
        const unsigned long long a = stamps[2 * i], b = stamps[2 * i + 1];
        stamps[2 * i] = ~0ull;
        stamps[2 * i + 1] = 0;
        if (b > a && a != 0 && a != ~0ull) {  // (slots start zeroed: the first step after a plan is built is skipped)
          acc[2 * i] += b - a;
          acc[2 * i + 1] += 1;
          int k = n++;  // insertion sort by start time
          for (; k > 0 && t0[k - 1] > a; --k) {
            t0[k] = t0[k - 1];
            t1[k] = t1[k - 1];
          }
          t0[k] = a;
          t1[k] = b;
        } else {
          all = false;
        }
      }
      if (all && n > 0) {
        unsigned long long busy = 0, lo = t0[0], hi = t1[0];
        for (int k = 1; k < n; ++k) {
          if (t0[k] > hi) {
            busy += hi - lo;
            lo = t0[k];
            hi = t1[k];
          } else if (t1[k] > hi) {
            hi = t1[k];
          }
        }
        busy += hi - lo;
        acc[2 * (n_slots + l)] += busy;
        acc[2 * (n_slots + l) + 1] += 1;
      }
    }
  }
}

// teacher forcing (test hook): overwrite the next decoder input with a given token
__global__ void force_token_kernel(const long long* __restrict__ toks, const act_t* __restrict__ E,
                                   res_t* __restrict__ x, int d) {
  const int b = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(toks[b]) * d);
  res_t* dst = x + static_cast<size_t>(b) * d;
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) store_res8_from_act(dst + i * 8, src[i]);
}

}  // namespace b200
