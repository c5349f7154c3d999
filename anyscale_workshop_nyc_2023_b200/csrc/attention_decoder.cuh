// Decoder attention over all T positions of every row at once: the teacher-forced forward pass (b200t5_forward).
// Causal self-attention with T5's unidirectional relative-position bias, and cross-attention over a prompt's encoder
// keys in the cross-K/V arena, both on encoder_attn_kernel's tiles, helpers and rounding contract
// (attention_encoder.cuh).
#pragma once
#include "attention_encoder.cuh"

namespace b200 {

// The decoder's attentions over all T positions of every row at once (the teacher-forced forward pass), two-pass
// tiles with encoder_attn_kernel's tiling and rounding contract (SURVEY Appendix A.3):
//   kAttnCausal   unidirectional bias dist_bias[h][i - j], keys j > i masked (the decoder's self-attention over all
//                 T positions at once; T5Attention with is_decoder, modeling_t5.py:188-251);
//   kAttnCross    no bias, key mask key_ok (the decoder's cross-attention over a prompt's encoder keys).
constexpr int kAttnCausal = 1, kAttnCross = 2;

// One 64-query tile of one (row, head): q rows i0.. of qg (stride ldq), keys / values rows 0..ext-1 of kg / vg
// (stride ldkv), context rows to og (stride ldo). `rows` query rows exist; S is the length the bias table (kAttnCausal:
// T) or the mask row (kAttnCross: the prompt length) is sized for. kAttnCausal visits only the key chunks at or below the tile's diagonal:
// the chunks above it hold -inf scores only, which add exactly 0 to the sums.
template <int kKind>
DEVINL void attn_tile_2pass(uint8_t* dec_smem, const act_t* qg, int ldq, const act_t* kg, const act_t* vg, int ldkv, act_t* og,
                            int ldo, const float* __restrict__ bias, const unsigned char* __restrict__ ok_row, int ext, int rows,
                            int i0, int S, int h) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;

  uint8_t* sQ = dec_smem;                 // 8 KB
  uint8_t* sK = sQ + 8192;                // 2 x 8 KB
  uint8_t* sV = sK + 16384;               // 2 x 8 KB
  float* sBias = reinterpret_cast<float*>(sV + 16384);  // kAttnCausal: S + 64 floats, index j - (i - i0) + 63
  unsigned char* sOk = reinterpret_cast<unsigned char*>(sBias + S + 64);  // kAttnCross: S bytes
  const uint32_t sQ_u = smem_u32(sQ), sK_u = smem_u32(sK), sV_u = smem_u32(sV);

  int nchunks = (ext + kEncKC - 1) / kEncKC;
  if constexpr (kKind == kAttnCausal) nchunks = min(nchunks, i0 / kEncKC + 1);

  // bias slice or mask row (plain loads), Q tile + first K chunk (async)
  {
    if constexpr (kKind == kAttnCausal) {
      for (int x = threadIdx.x; x < S + 63; x += kEncThreads) {
        const int dist = i0 + 63 - x;  // i - j of (j = x - 63 + (i - i0))
        // j > i: -inf, the causal mask (HF adds finfo.min there: the same exp() = 0)
        sBias[x] = dist < 0 ? -INFINITY : (dist < S ? bias[static_cast<size_t>(h) * S + dist] : 0.f);
      }
    } else {
      for (int x = threadIdx.x; x < S; x += kEncThreads) sOk[x] = ok_row[x];
    }
  }
  load_tile_async(sQ_u, qg, ldq, i0, min(kEncQ, rows - i0));
  load_tile_async(sK_u, kg, ldkv, 0, min(kEncKC, ext));
  cp_async_commit();

  uint32_t qa[4][4];  // Q fragments for the 4 k-steps (d = 64)
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float oacc[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) oacc[nt][e] = 0.f;

  const int row_l0 = warp * 16 + g;  // local query rows of this thread: row_l0, row_l0 + 8

  for (int pass = 0; pass < 2; ++pass) {
    if (pass == 1) {
      // reduce the partial sums over the 4 lanes of a row, prefetch chunk 0 again (K and V)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
      }
      load_tile_async(sK_u, kg, ldkv, 0, min(kEncKC, ext));
      load_tile_async(sV_u, vg, ldkv, 0, min(kEncKC, ext));
      cp_async_commit();
    }
    for (int c = 0; c < nchunks; ++c) {
      const int buf = c & 1;
      if (c + 1 < nchunks) {
        const int r0 = (c + 1) * kEncKC;
        load_tile_async(sK_u + (buf ^ 1) * 8192, kg, ldkv, r0, min(kEncKC, ext - r0));
        if (pass == 1) load_tile_async(sV_u + (buf ^ 1) * 8192, vg, ldkv, r0, min(kEncKC, ext - r0));
        cp_async_commit();
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();

      if (pass == 0 && c == 0) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const int r = warp * 16 + (lane & 15);
          const int ch = kk * 2 + (lane >> 4);
          ldmatrix_x4(sQ_u + tile_off(r, ch), qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3]);
        }
      }

      // ---- S = Q K^T for this chunk: 16 x 64 per warp
      float sacc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) sacc[nt][e] = 0.f;
      const uint32_t kbase = sK_u + buf * 8192;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {  // pairs of n-tiles (16 keys)
          const int mi = lane >> 3;
          const int key = np * 16 + (mi >> 1) * 8 + (lane & 7);
          const int ch = kk * 2 + (mi & 1);
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(kbase + tile_off(key, ch), b0, b1, b2, b3);
          mma_act_16816(sacc[2 * np], qa[kk], b0, b1);
          mma_act_16816(sacc[2 * np + 1], qa[kk], b2, b3);
        }
      }

      // ---- scores -> bf16, + bias -> bf16, mask
      const int jc = c * kEncKC;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = jc + nt * 8 + tq * 2 + (e & 1);
          const int rl = row_l0 + (e >> 1) * 8;
          float s = act_round(sacc[nt][e]);
          if (j < ext) {
            if constexpr (kKind == kAttnCausal) {
              s = act_round(s + sBias[j - rl + 63]);
            } else if (!sOk[j]) {
              s = kActMin;
            }
          } else {
            s = -INFINITY;
          }
          sacc[nt][e] = s;
        }
      }

      if (pass == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float cm = -INFINITY;
#pragma unroll
          for (int nt = 0; nt < 8; ++nt) cm = fmaxf(cm, fmaxf(sacc[nt][2 * r], sacc[nt][2 * r + 1]));
          cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 1));
          cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 2));
          const float mn = fmaxf(m_run[r], cm);
          float add = 0.f;
#pragma unroll
          for (int nt = 0; nt < 8; ++nt) add += expf(sacc[nt][2 * r] - mn) + expf(sacc[nt][2 * r + 1] - mn);
          l_run[r] = l_run[r] * expf(m_run[r] - mn) + add;
          m_run[r] = mn;
        }
      } else {
        // ---- P = bf16(exp(s - max) / sum) as A fragments, O += P V
        const uint32_t vbase = sV_u + buf * 8192;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // 16 keys per k-step = n-tiles 2kk, 2kk+1 of S
          uint32_t pa[4];
          pa[0] = pack_act2(expf(sacc[2 * kk][0] - m_run[0]) / l_run[0], expf(sacc[2 * kk][1] - m_run[0]) / l_run[0]);
          pa[1] = pack_act2(expf(sacc[2 * kk][2] - m_run[1]) / l_run[1], expf(sacc[2 * kk][3] - m_run[1]) / l_run[1]);
          pa[2] = pack_act2(expf(sacc[2 * kk + 1][0] - m_run[0]) / l_run[0],
                              expf(sacc[2 * kk + 1][1] - m_run[0]) / l_run[0]);
          pa[3] = pack_act2(expf(sacc[2 * kk + 1][2] - m_run[1]) / l_run[1],
                              expf(sacc[2 * kk + 1][3] - m_run[1]) / l_run[1]);
#pragma unroll
          for (int dp = 0; dp < 4; ++dp) {  // pairs of d-tiles (16 dims)
            const int mi = lane >> 3;
            const int key = kk * 16 + (mi & 1) * 8 + (lane & 7);
            const int ch = dp * 2 + (mi >> 1);
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4_trans(vbase + tile_off(key, ch), b0, b1, b2, b3);
            mma_act_16816(oacc[2 * dp], pa, b0, b1);
            mma_act_16816(oacc[2 * dp + 1], pa, b2, b3);
          }
        }
      }
      __syncthreads();  // all warps done with buf before the next prefetch overwrites it
    }
  }

  // ---- write O (act_t) to og[i, d]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = i0 + row_l0 + r * 8;
    if (i < rows) {
      act_t* dst = og + static_cast<size_t>(i) * ldo + tq * 2;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
        *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack_act2(oacc[nt][2 * r], oacc[nt][2 * r + 1]);
    }
  }
}

// The decoder's attentions over T positions of every row at once (the teacher-forced forward pass):
//   kAttnCausal: qkv [B*T, 3I] from the fused self-attention QKV GEMM, dist_bias [H][T] (the decode step's dec_bias
//                table), every key below T exists; kv, key_ok and extent are unused.
//   kAttnCross:  q = qkv [B*T, I] (the cross-attention query projection), K / V of layer l in the cross-K/V arena
//                kv = [2][B][H][S][64] (EpiCrossKV), keys masked by key_ok [B][S] / extent [B] as in the decode step.
// ctx [B*T, I]. Grid (ceil(T / 64), B * H).
template <int kKind>
__global__ void __launch_bounds__(kEncThreads)
decoder_attn_kernel(const act_t* __restrict__ qkv, const act_t* __restrict__ kv, act_t* __restrict__ ctx,
                    const float* __restrict__ dist_bias, const unsigned char* __restrict__ key_ok,
                    const int* __restrict__ extent, int B, int T, int S, int H) {
  extern __shared__ __align__(128) uint8_t dec_smem[];
  const int I = H * 64;
  const int bh = blockIdx.y;
  const int b = bh / H, h = bh - b * H;
  const int i0 = blockIdx.x * kEncQ;
  const size_t row0 = static_cast<size_t>(b) * T;
  act_t* og = ctx + row0 * I + h * 64;
  if constexpr (kKind == kAttnCausal) {
    const act_t* qg = qkv + row0 * 3 * I + h * 64;
    attn_tile_2pass<kAttnCausal>(dec_smem, qg, 3 * I, qg + I, qg + 2 * I, 3 * I, og, I, dist_bias, nullptr, T, T, i0, T, h);
  } else {
    const size_t plane = static_cast<size_t>(B) * I * S;
    const act_t* kg = kv + (static_cast<size_t>(b) * H + h) * S * 64;
    attn_tile_2pass<kAttnCross>(dec_smem, qkv + row0 * I + h * 64, I, kg, kg + plane, 64, og, I, nullptr, key_ok + static_cast<size_t>(b) * S,
                                extent[b], T, i0, S, h);
  }
}

// The cross-attention of the multiple-choice forward pass (b200t5_forward_choices): the queries of all of prompt b's
// candidates are the contiguous rows qoff[b] .. qoff[b+1]-1 of q [*, I], tiled 64 at a time as one query sequence
// against prompt b's K/V in the cross-K/V arena kv = [2][B][H][S][64], keys masked by key_ok [B][S] / extent [B] as in
// kAttnCross. Cross-attention has no causal mask and no position bias, and every query row keeps its own softmax, so
// a row's result does not depend on which rows share its tile: each row gets the bits decoder_attn_kernel<kAttnCross>
// gives it against a private copy of the prompt's K/V, which is loaded here once per tile instead of once per candidate.
// ctx rows as q. Grid (tiles of the longest prompt's queries, B * H); CTAs past a prompt's queries exit.
__global__ void __launch_bounds__(kEncThreads)
decoder_cross_packed_kernel(const act_t* __restrict__ q, const act_t* __restrict__ kv, act_t* __restrict__ ctx,
                            const unsigned char* __restrict__ key_ok, const int* __restrict__ extent,
                            const int* __restrict__ qoff, int B, int S, int H) {
  extern __shared__ __align__(128) uint8_t dec_smem[];
  const int I = H * 64;
  const int bh = blockIdx.y;
  const int b = bh / H, h = bh - b * H;
  const int i0 = blockIdx.x * kEncQ;
  const int q0 = qoff[b], rows = qoff[b + 1] - q0;
  if (i0 >= rows) return;
  const size_t plane = static_cast<size_t>(B) * I * S;
  const act_t* kg = kv + (static_cast<size_t>(b) * H + h) * S * 64;
  attn_tile_2pass<kAttnCross>(dec_smem, q + static_cast<size_t>(q0) * I + h * 64, I, kg, kg + plane, 64,
                              ctx + static_cast<size_t>(q0) * I + h * 64, I, nullptr, key_ok + static_cast<size_t>(b) * S,
                              extent[b], rows, i0, S, h);
}

}  // namespace b200
