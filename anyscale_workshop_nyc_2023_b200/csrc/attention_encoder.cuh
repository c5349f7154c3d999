// Encoder self-attention with T5 relative-position bias and key-padding mask
// (modeling_t5.py:253-344; bias buckets :188-251, shared across layers :755-758).
//
// Warp-level mma.sync (m16n8k16, bf16 -> fp32) flash-style kernel that never materialises
// the [B,H,S,S] score tensor, but keeps HF's exact (non-online) rounding contract (SURVEY
// Appendix A.3) by running two passes over the keys: pass 1 computes the row max and
// sum(exp) over the bf16-rounded biased scores, pass 2 recomputes the identical scores,
// forms p = bf16(exp(s-max)/sum) and accumulates P.V in fp32. Recomputing Q K^T (d = 64)
// is cheaper than keeping a 64 x S fp32 score tile per CTA in registers or shared memory.
//
// qkv: [B*S, 3*I] bf16 from the fused QKV GEMM (q | k | v, head-major inside each).
// One CTA = 4 warps = 64 query rows of one (b,h); keys are visited in chunks of 64,
// only up to extent[b] (padded keys contribute exactly 0 after the fp32 softmax). Key rows at or beyond the extent
// are zero-filled, not loaded: in the packed layout they belong to the next prompt or were never written, and
// p = 0 times a NaN or Inf there would still poison P.V.
// Packed rows (cu != NULL): prompt b occupies rows cu[b] .. cu[b] + extent[b] - 1 of qkv and ctx, and only
// those query rows are computed and written.
// attention_decoder.cuh (attn_tile_2pass) repeats this kernel's two-pass loop for the decoder's forward-pass attentions:
// a change to the rounding contract here belongs there too. (A shared function changes this kernel's SASS.)
#pragma once
#include "attention_decode.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int kEncThreads = 128;
constexpr int kEncQ = 64;
constexpr int kEncKC = 64;
// Prompts up to this length run on packed rows (the slot pool admits prompts through the packed path only,
// modeling._POOL_MAX_S); longer ones run on all B*S rows.
constexpr int kEncPackMaxS = 512;

DEVINL void cp_async_16(uint32_t smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
DEVINL void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
DEVINL void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
DEVINL void mma_act_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      #if B200T5_F16
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
#else
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
#endif
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 64 rows x 128 B tile, 16-B chunks XOR-swizzled by (row & 7): conflict-free ldmatrix.
DEVINL uint32_t tile_off(int row, int chunk) { return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4)); }

// Load a 64x64 bf16 tile (rows row0.. of a [rows, ld] matrix at column col0) into swizzled smem.
DEVINL void load_tile_async(uint32_t smem_base, const act_t* g, int ld, int row0, int nrows_valid) {
  for (int i = threadIdx.x; i < 64 * 8; i += kEncThreads) {
    const int r = i >> 3, c = i & 7;
    const bool ok = r < nrows_valid;
    const act_t* src = g + static_cast<size_t>(row0 + (ok ? r : 0)) * ld + c * 8;
    cp_async_16(smem_base + tile_off(r, c), src, ok);
  }
}

__global__ void __launch_bounds__(kEncThreads)
encoder_attn_kernel(const act_t* __restrict__ qkv,     // [B*S, 3I]
                    act_t* __restrict__ ctx,           // [B*S, I]
                    const float* __restrict__ rel_bias,        // [H][2S-1], index j - i + S - 1
                    const unsigned char* __restrict__ key_ok,  // [B][S]
                    const int* __restrict__ extent,            // [B]
                    const int* __restrict__ cu,                // packed rows: prompt b starts at row cu[b] (NULL: b * S)
                    int S, int H) {
  extern __shared__ __align__(128) uint8_t enc_smem[];
  const int I = H * 64;
  const int ld = 3 * I;
  const int bh = blockIdx.y;
  const int b = bh / H, h = bh - b * H;
  const int i0 = blockIdx.x * kEncQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;

  uint8_t* sQ = enc_smem;                 // 8 KB
  uint8_t* sK = sQ + 8192;                // 2 x 8 KB
  uint8_t* sV = sK + 16384;               // 2 x 8 KB
  float* sBias = reinterpret_cast<float*>(sV + 16384);  // S + 64 floats: index j - (i - i0) + 63
  unsigned char* sOk = reinterpret_cast<unsigned char*>(sBias + S + 64);  // S bytes
  const uint32_t sQ_u = smem_u32(sQ), sK_u = smem_u32(sK), sV_u = smem_u32(sV);

  const int ext = extent[b];
  const int rows = cu ? ext : S;  // query rows of this prompt that exist in the layout
  if (i0 >= rows) return;
  const size_t row0 = cu ? static_cast<size_t>(cu[b]) : static_cast<size_t>(b) * S;
  const int nchunks = (ext + kEncKC - 1) / kEncKC;
  const act_t* qg = qkv + row0 * ld + h * 64;
  const act_t* kg = qg + I;
  const act_t* vg = qg + 2 * I;

  // bias slice + mask row (plain loads), Q tile + first K chunk (async)
  {
    const int lo = S - 64 - i0;  // rel index of (j=0, i=i0+63)
    for (int x = threadIdx.x; x < S + 63; x += kEncThreads) {
      const int idx = lo + x;
      sBias[x] = (idx >= 0 && idx < 2 * S - 1) ? rel_bias[static_cast<size_t>(h) * (2 * S - 1) + idx] : 0.f;
    }
    for (int x = threadIdx.x; x < S; x += kEncThreads) sOk[x] = key_ok[static_cast<size_t>(b) * S + x];
  }
  load_tile_async(sQ_u, qg, ld, i0, min(kEncQ, rows - i0));
  load_tile_async(sK_u, kg, ld, 0, min(kEncKC, ext));
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
      load_tile_async(sK_u, kg, ld, 0, min(kEncKC, ext));
      load_tile_async(sV_u, vg, ld, 0, min(kEncKC, ext));
      cp_async_commit();
    }
    for (int c = 0; c < nchunks; ++c) {
      const int buf = c & 1;
      if (c + 1 < nchunks) {
        const int r0 = (c + 1) * kEncKC;
        load_tile_async(sK_u + (buf ^ 1) * 8192, kg, ld, r0, min(kEncKC, ext - r0));
        if (pass == 1) load_tile_async(sV_u + (buf ^ 1) * 8192, vg, ld, r0, min(kEncKC, ext - r0));
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
            s = act_round(s + sBias[j - rl + 63]);
            if (!sOk[j]) s = kActMin;
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

  // ---- write O (bf16) to ctx[b*S + i, h*64 + d]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = i0 + row_l0 + r * 8;
    if (i < rows) {
      act_t* dst = ctx + (row0 + i) * I + h * 64 + tq * 2;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
        *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack_act2(oacc[nt][2 * r], oacc[nt][2 * r + 1]);
    }
  }
}

inline size_t encoder_attn_smem_bytes(int S) { return 8192 + 16384 + 16384 + (S + 64) * 4 + S + 16; }

}  // namespace b200
