// Persistent warp-specialised bf16 GEMM for sm_90a (H100):
//   D[M,N] = A[M,K] * W[N,K]^T      (both operands K-major, i.e. nn.Linear layout)
// TMA (128-B swizzle) -> smem ring -> wgmma (two consumer warpgroups, 64 tile rows each, fp32 accumulators in
// registers) -> accumulators staged as fp32 rows in shared memory -> the epilogue functor reads 32-column chunks of
// one row per thread, applies the fused epilogue and writes HBM directly.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (MMA, then epilogue), warp 8 = TMA producer.
// The staging tile aliases the pipeline ring: it is written once both warpgroups' MMAs of the tile have completed,
// and the producer starts the next tile's loads once every epilogue thread has read its rows. Tiles with BN <= 128
// keep a CTA near 100 KB so that two CTAs share an SM and one's epilogue overlaps the other's main loop.
//
// The epilogue functors are where the T5 rounding contract lives: HF eager bf16
// rounds every Linear output to bf16 before anything else touches it
// (transformers/models/t5/modeling_t5.py:277,298-299,338; SURVEY Appendix A.2),
// so each functor first rounds the fp32 accumulator to bf16 and only then fuses
// the residual add / GeGLU / KV scatter / arg-max.
#pragma once
#include "logits_process.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 288;     // 2 consumer warpgroups + 1 producer warp
constexpr int kGemmConsumers = 256;
constexpr int kEpiSmemBytes = 8192;  // per-CTA scratch the epilogue functor may stage tables in

template <int BN>
struct GemmCfg {
  static_assert(BN == 128 || BN == 256, "BN");
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = BN >= 256 ? 4 : (96 * 1024) / kStageBytes;
  static constexpr int kRingBytes = kStages * kStageBytes;
  static constexpr int kStageLd = BN + 4;  // floats per staged row; +4 keeps a warp's per-row 16-B reads conflict-free
  static constexpr int kStagingBytes = kBM * kStageLd * 4;
  static_assert(kStagingBytes <= kRingBytes, "the staged tile aliases the ring");
  static constexpr int kSmemBytes = kRingBytes + 1024 /*align*/ + 256 /*barriers*/ + kEpiSmemBytes;
  static constexpr int kCtasPerSm = BN <= 128 ? 2 : 1;
};

struct TileCoord {
  int m_tile, n_tile;
};
DEVINL TileCoord tile_coord(int tile, int tiles_m, int tiles_n, int m_fastest) {
  TileCoord c;
  if (m_fastest) {
    c.m_tile = tile % tiles_m;
    c.n_tile = tile / tiles_m;
  } else {
    c.n_tile = tile % tiles_n;
    c.m_tile = tile / tiles_n;
  }
  return c;
}

DEVINL void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kGemmConsumers) : "memory"); }

// One k-block (128 B of K per row) of this warpgroup's 64 x BN product: 4 wgmma of 32 B each.
template <int BN, bool kTf32>
DEVINL void wgmma_kblock(float (&acc)[BN / 2], uint32_t a_addr, uint32_t b_addr) {
  const uint64_t a_desc = make_desc_sw128_kmajor(a_addr);
  const uint64_t b_desc = make_desc_sw128_kmajor(b_addr);
#pragma unroll
  for (int k = 0; k < kBK / 16; ++k) wgmma_k32B<BN, kTf32>(acc, a_desc + 2 * k, b_desc + 2 * k);
}

// Writes a warpgroup's wgmma accumulators (rows row0 .. row0+63 of the tile) into the fp32 staging rows.
template <int BN>
DEVINL void stage_acc(float* stg, int row0, const float (&acc)[BN / 2]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(stg + r * GemmCfg<BN>::kStageLd + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(stg + (r + 8) * GemmCfg<BN>::kStageLd + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// kTf32 / a_kblocks: fp32 operands consumed as tf32 (the fp16 build's fp32-weight `wo` product): a k-block is 32
// elements (the same 128-byte rows), K counts the columns of W' = [W_hi | W_lo], and A has only a_kblocks k-blocks
// and is walked twice (kb % a_kblocks), so the accumulator receives A . W_hi^T + A . W_lo^T.
// kBBox: rows per TMA box of the weight tensor map (the weight tile is loaded in BN / kBBox boxes).
template <int BN, class Epi, bool kTf32 = false, int kBBox = BN>
__global__ void __launch_bounds__(kGemmThreads, GemmCfg<BN>::kCtasPerSm)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N,
                    int K, int m_fastest, typename Epi::Params ep, int a_kblocks) {
  using Cfg = GemmCfg<BN>;
  static_assert(BN % kBBox == 0, "box");
  constexpr int kbk = kTf32 ? kBK / 2 : kBK;  // elements per k-block (128 bytes)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kRingBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::kStages;
  uint64_t* stg_free = bars + 2 * Cfg::kStages;  // every epilogue thread has read the staged tile
  uint8_t* epi_smem = smem + Cfg::kRingBytes + 256;
  float* stg = reinterpret_cast<float*>(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (M + kBM - 1) / kBM;
  const int tiles_n = (N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int kblocks = (K + kbk - 1) / kbk;
  if (a_kblocks <= 0) a_kblocks = kblocks;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    mbar_init(stg_free, kGemmConsumers);
    mbar_fence_init();
  }
  __syncthreads();
  // PDL: everything above overlapped the previous kernel's tail. Each role waits for the previous
  // kernel (griddepcontrol.wait) only right before it first touches memory that kernel may have
  // written; the weights (B operand) never depend on it and are prefetched into L2 before the wait.

  if (warp == 8) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      if (static_cast<int>(blockIdx.x) < num_tiles) {
        const TileCoord tc0 = tile_coord(blockIdx.x, tiles_m, tiles_n, m_fastest);
        for (int kb = 0; kb < kblocks; ++kb)
          for (int p = 0; p < BN / kBBox; ++p) tma_prefetch_l2_2d(&tmB, kb * kbk, tc0.n_tile * BN + p * kBBox);
      }
      pdl_wait();
      int stage = 0;
      uint32_t phase = 0, sphase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        if (tile != static_cast<int>(blockIdx.x)) {
          mbar_wait(stg_free, sphase);  // the previous tile's staged accumulators (aliasing the ring) have been read
          sphase ^= 1u;
        }
        const TileCoord tc = tile_coord(tile, tiles_m, tiles_n, m_fastest);
        const int m0 = tc.m_tile * kBM, n0 = tc.n_tile * BN;
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u);
          uint8_t* sA = smem + stage * Cfg::kStageBytes;
          uint8_t* sB = sA + Cfg::kABytes;
          mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
          tma_load_2d(sA, &tmA, &full[stage], (kb % a_kblocks) * kbk, m0);
#pragma unroll
          for (int p = 0; p < BN / kBBox; ++p) tma_load_2d(sB + p * kBBox * 128, &tmB, &full[stage], kb * kbk, n0 + p * kBBox);
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups
    const int wg = warp >> 2;
    const int et = threadIdx.x;  // 0..255
    Epi::prologue(ep, epi_smem, et, kGemmConsumers);  // constant tables; overlaps the main loop
    pdl_wait();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord tc = tile_coord(tile, tiles_m, tiles_n, m_fastest);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStageBytes) + wg * 64 * 128;
        wgmma_fence_acc(acc);
        wgmma_fence();
        wgmma_kblock<BN, kTf32>(acc, a_addr, smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes));
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs are done: hand its stage back to the producer
        wgmma_fence_acc(acc);
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      // both warpgroups' MMAs are complete before the staging rows overwrite the ring
      consumers_sync();
      stage_acc<BN>(stg, wg * 64, acc);
      consumers_sync();
      const int row = et & (kBM - 1), part = et >> 7;
      const int m = tc.m_tile * kBM + row;
      const uint32_t waddr = (smem_u32(stg) >> 2) + static_cast<uint32_t>(row * Cfg::kStageLd);
      Epi::template run<BN>(ep, waddr, m, m < M, tc.n_tile, N, epi_smem, part, 2);
      mbar_arrive(stg_free);
    }
  }
}

// ======================================================================== epilogues
// Every functor works on CHUNKS: 32 consecutive fp32 accumulator columns of one output row
// (acc[] holds their bit patterns). `chunk_pre` fetches whatever the chunk needs that does not
// depend on the accumulator (so callers can issue it early); `chunk` applies the T5 rounding
// contract and writes HBM. Paired functors (GeGLU) consume two chunks: gate and up.
// The persistent kernel above feeds chunks from its staged accumulator rows (`run`); the split-K kernel
// (gemm_splitk.cuh) feeds them from the cluster-reduced partial sums.

DEVINL void round_pack_32(const uint32_t (&acc)[32], uint32_t (&out)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) out[i] = pack_act2(__uint_as_float(acc[2 * i]), __uint_as_float(acc[2 * i + 1]));
}

// Store 32 bf16 (64 B) to dst; columns [n0, n0+32) clipped to N in groups of 8.
DEVINL void store_row_chunk(act_t* dst, const uint32_t (&p)[16], int n0, int N) {
  uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    if (n0 + g * 8 + 8 <= N) d4[g] = make_uint4(p[4 * g], p[4 * g + 1], p[4 * g + 2], p[4 * g + 3]);
  }
}

// Store 32 fp32 (128 B) to dst, clipped to N in groups of 4.
DEVINL void store_row_chunk_f32(float* dst, const float (&v)[32], int n0, int N) {
  float4* d4 = reinterpret_cast<float4*>(dst);
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    if (n0 + g * 4 + 4 <= N) d4[g] = make_float4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]);
  }
}

struct NoPre {};

// Drives an unpaired functor over the BN columns of this thread's staged row, fetching the
// pre-operands of chunk c+1 before chunk c is processed.
// `part` of `parts`: the epilogue warp handles chunks [part*C/parts, (part+1)*C/parts) of the C = BN/32 chunks.
template <int BN, class Epi>
DEVINL void run_chunks(const typename Epi::Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N,
                                 const uint8_t* epi_smem, int part, int parts) {
  constexpr int C = BN / 32;
  const int c_lo = part * C / parts, c_hi = (part + 1) * C / parts;
  typename Epi::ChunkPre pre[2];
  if (m_ok && n_tile * BN + c_lo * 32 < N) Epi::chunk_pre(p, m, n_tile * BN + c_lo * 32, N, pre[0]);
#pragma unroll 1
  for (int c = c_lo; c < c_hi; c += 2) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (c + u < c_hi) {
        uint32_t acc[32];
        acc_ld_32(taddr + (c + u) * 32, acc);
        const int n0 = n_tile * BN + (c + u) * 32;
        if (m_ok && c + u + 1 < c_hi && n0 + 32 < N) Epi::chunk_pre(p, m, n0 + 32, N, pre[(u + 1) & 1]);
        if (m_ok && n0 < N) Epi::chunk(p, acc, m, n0, N, epi_smem, pre[u & 1]);
      }
    }
  }
}

// ---- plain store: C = bf16(acc)
struct EpiStore {
  struct Params {
    act_t* C;
    int ldc;
  };
  static constexpr bool kPaired = false;
  typedef NoPre ChunkPre;
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  static DEVINL void chunk_pre(const Params&, int, int, int, ChunkPre&) {}
  static DEVINL void chunk(const Params& p, const uint32_t (&acc)[32], int m, int n0, int N, const uint8_t*,
                           const ChunkPre&) {
    uint32_t o[16];
    round_pack_32(acc, o);
    store_row_chunk(p.C + static_cast<size_t>(m) * p.ldc + n0, o, n0, N);
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es,
                         int part, int parts) {
    run_chunks<BN, EpiStore>(p, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};

#if B200T5_F16
// ---- residual, fp16 build: the stream is fp32 (res_t = float) and torch's type promotion decides the arithmetic
// (modeling_t5.py T5LayerSelfAttention / T5LayerCrossAttention / T5LayerFF.forward):
//   attention output projection (fp16 Linear):  C = R + float(fp16(acc))            round_acc = 1
//     ... while the stream is still fp16, i.e. before the first feed-forward block:  C = fp16(R + fp16(acc))   round_out = 1
//   feed-forward `wo` (fp32 weight, fp32 output; _keep_in_fp32_modules): C = R + acc   round_acc = 0
struct EpiResidual {
  struct Params {
    res_t* C;
    const res_t* R;
    int ld;
    float* ss = nullptr;  // (fused RMSNorm is a bf16-build experiment)
    int ss_ld = 0;
    int round_acc = 1;
    int round_out = 0;
  };
  static constexpr bool kPaired = false;
  struct ChunkPre {
    float4 r[8];
  };
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  static DEVINL void chunk_pre(const Params& p, int m, int n0, int N, ChunkPre& pre) {
    const float4* r4 = reinterpret_cast<const float4*>(p.R + static_cast<size_t>(m) * p.ld + n0);
#pragma unroll
    for (int g = 0; g < 8; ++g) pre.r[g] = (n0 + g * 4 + 4 <= N) ? r4[g] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  static DEVINL void chunk(const Params& p, const uint32_t (&acc)[32], int m, int n0, int N, const uint8_t*,
                           const ChunkPre& pre) {
    float o[32];
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const float rw[4] = {pre.r[g].x, pre.r[g].y, pre.r[g].z, pre.r[g].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float y = __uint_as_float(acc[g * 4 + j]);
        if (p.round_acc) y = act_round(y);
        float v = rw[j] + y;
        if (p.round_out) v = act_round(v);
        o[g * 4 + j] = v;
      }
    }
    store_row_chunk_f32(p.C + static_cast<size_t>(m) * p.ld + n0, o, n0, N);
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es,
                         int part, int parts) {
    run_chunks<BN, EpiResidual>(p, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};
#else
// ---- residual: C = bf16( float(R) + float(bf16(acc)) )   (modeling_t5.py:375,406,149)
struct EpiResidual {
  struct Params {
    act_t* C;
    const act_t* R;
    int ld;
    // optional: sum of squares of the 32 outputs of each (row, chunk) -> ss[m * ss_ld + n0 / 32], for a
    // consumer GEMM that applies the following RMSNorm to its A operand (gemm_splitk.cuh, NormA)
    float* ss = nullptr;
    int ss_ld = 0;
    int round_acc = 1, round_out = 1;  // (fp16 build only; this build always rounds both)
  };
  static constexpr bool kPaired = false;
  struct ChunkPre {
    uint4 r[4];
  };
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  // The residual operand does not depend on the accumulator: it is fetched while the main loop /
  // the previous chunk is still in flight.
  static DEVINL void chunk_pre(const Params& p, int m, int n0, int N, ChunkPre& pre) {
    const uint4* r4 = reinterpret_cast<const uint4*>(p.R + static_cast<size_t>(m) * p.ld + n0);
#pragma unroll
    for (int g = 0; g < 4; ++g) pre.r[g] = (n0 + g * 8 + 8 <= N) ? r4[g] : make_uint4(0, 0, 0, 0);
  }
  static DEVINL void chunk(const Params& p, const uint32_t (&acc)[32], int m, int n0, int N, const uint8_t*,
                           const ChunkPre& pre) {
    uint32_t o[16];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const uint32_t rw[4] = {pre.r[g].x, pre.r[g].y, pre.r[g].z, pre.r[g].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float y0 = act_round(__uint_as_float(acc[g * 8 + 2 * j]));
        const float y1 = act_round(__uint_as_float(acc[g * 8 + 2 * j + 1]));
        o[g * 4 + j] = pack_act2(act_lo(rw[j]) + y0, act_hi(rw[j]) + y1);
      }
    }
    store_row_chunk(p.C + static_cast<size_t>(m) * p.ld + n0, o, n0, N);
    if (p.ss) {
      float sq = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (n0 + 2 * i + 2 <= N) {
          const float a = act_lo(o[i]), b = act_hi(o[i]);
          sq = fmaf(a, a, sq);
          sq = fmaf(b, b, sq);
        }
      }
      p.ss[static_cast<size_t>(m) * p.ss_ld + (n0 >> 5)] = sq;
    }
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es,
                         int part, int parts) {
    run_chunks<BN, EpiResidual>(p, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};

#endif

// gelu_new exactly as HF eager evaluates it on act_t tensors: every elementwise op rounds its
// result to act_t (transformers/activations.py:59-66; SURVEY Appendix A.5). On the GPU,
// torch.pow(x, 3.0) on a bf16 or an fp16 tensor is x*x*x in act_t arithmetic (two roundings,
// pow_mode 0; verified exhaustively against torch on the GPU for both types). pow_mode 1 rounds
// once: what torch on the CPU computes for fp16, which the fp16 oracle and its goldens follow.
DEVINL float gelu_new_act_exact(float x, int pow_mode) {
  const float half_x = act_round(0.5f * x);
  const float x3 = pow_mode == 0 ? act_round(act_round(x * x) * x) : act_round(x * x * x);
  const float t1 = act_round(0.044715f * x3);
  const float t2 = act_round(x + t1);
  const float t3 = act_round(0.7978845608028654f * t2);
  const float t4 = act_round(tanhf(t3));
  const float t5 = act_round(1.0f + t4);
  return act_round(half_x * t5);
}

// The input of gelu_new is itself a bf16 value, so the function has only 65536 possible
// arguments: it is tabulated once per device with the exact arithmetic above. Only magnitudes in
// [lo, hi) need the table (a few thousand entries, staged in shared memory by the epilogue);
// below lo the result is bf16(0.5*x) and above hi it is x (positive) or -0 (negative), which the
// host verifies entry by entry when it derives lo/hi from the full table (b200t5.cu).
struct GeluLut {
  const uint16_t* table;  // device: [2][hi - lo] bf16 bits, sign-major
  int lo, hi;             // magnitude bit patterns (bf16 bits & 0x7fff)
};

// Same function without divergent branches (the GEMM epilogue evaluates it 128 times per thread and tile):
// the three cases are computed side by side and selected.
DEVINL float gelu_from_lut_sel(float x, const uint16_t* lut, int lo, int n /* = hi - lo */) {
  const uint32_t bits = __float_as_uint(x) >> 16;
  const int mag = static_cast<int>(bits & 0x7FFFu);
  const bool neg = (bits >> 15) != 0;
  const int rel = mag - lo;
  const int idx = min(max(rel, 0), n - 1) + (neg ? n : 0);
  const float tab = __uint_as_float(static_cast<uint32_t>(lut[idx]) << 16);
  const float half = act_round(0.5f * x);
  float sat = neg ? (mag == 0x7F80 ? __int_as_float(0x7FC00000) : -0.0f) : x;
  sat = mag > 0x7F80 ? x : sat;
  return rel < 0 ? half : (rel >= n ? sat : tab);
}

DEVINL float gelu_from_lut(float x, const uint16_t* lut, int lo, int hi) {
  const uint32_t bits = __float_as_uint(x) >> 16;
  const int mag = static_cast<int>(bits & 0x7FFFu);
  const int neg = static_cast<int>(bits >> 15);
  if (mag < lo) return act_round(0.5f * x);  // tanh term rounds away: gelu_new(x) == bf16(0.5*x)
  if (mag >= hi) {
    if (mag > 0x7F80) return x;                     // NaN propagates
    if (!neg) return x;                             // tanh saturated: 0.5x * 2
    return mag == 0x7F80 ? __int_as_float(0x7FC00000) : -0.0f;  // 0.5x * (1 + -1): -inf*0 = NaN, else -0
  }
  return __uint_as_float(static_cast<uint32_t>(lut[neg * (hi - lo) + (mag - lo)]) << 16);
}

// gelu_new of an act_t value exactly as the GeGLU epilogue evaluates it (also run alone by b200t5_test_geglu):
// the fp16 build computes it op by op with the single-rounded pow of the oracle (CPU torch), which is one fp16 ulp
// away from CUDA torch on 15 of the 63,488 finite inputs (DESIGN.md 4b); the bf16 build reads the table `lut` (the
// epilogue's shared-memory copy), branch-free when the table is non-empty.
DEVINL float gelu_epilogue(float x, const uint16_t* lut, int lo, int hi) {
#if B200T5_F16
  return gelu_new_act_exact(x, 1);
#else
  return hi > lo ? gelu_from_lut_sel(x, lut, lo, hi - lo) : gelu_from_lut(x, lut, lo, hi);
#endif
}

// ---- GeGLU: tile columns [0,BN/2) are wi_0 (gate) features, [BN/2,BN) the matching
// wi_1 features (weights are interleaved per tile at finalize).
// EpiGegluNarrow below repeats this arithmetic for the forward pass: a change to the rounding here belongs there too.
//   out = bf16( gelu_new(bf16(gate)) * bf16(up) )          (modeling_t5.py:115-118)
struct EpiGeglu {
  struct Params {
    ffh_t* out;  // [M, F]
    int F;
    GeluLut lut;
  };
  static constexpr bool kPaired = true;
  typedef NoPre ChunkPre;
  // stage the gelu table (a few KB) with 16-byte loads; `nthreads` epilogue threads take part
  // (named barrier 2 is reserved for them)
  static DEVINL void prologue(const Params& p, uint8_t* epi_smem, int tid, int nthreads = 128) {
#if B200T5_F16
    return;  // fp16 build: gelu_new is evaluated directly (the table trick below indexes bf16 bit patterns)
#endif
    const int nvec = (2 * (p.lut.hi - p.lut.lo) * 2 + 15) / 16;
    const uint4* src = reinterpret_cast<const uint4*>(p.lut.table);
    uint4* dst = reinterpret_cast<uint4*>(epi_smem);
    for (int i = tid; i < nvec; i += nthreads) dst[i] = src[i];
    asm volatile("bar.sync 2, %0;" ::"r"(nthreads) : "memory");
  }
  // g/u: gate and up accumulators of features [f0, f0+32)
  static DEVINL void chunk2(const Params& p, const uint32_t (&g)[32], const uint32_t (&u)[32], int m, int f0,
                            const uint8_t* epi_smem) {
#if B200T5_F16
    // out = float(fp16(gelu_new(fp16 gate) * fp16 up)): the fp16 product cast up for the fp32 `wo` GEMM
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float x = act_round(__uint_as_float(g[i]));
      const float lin = act_round(__uint_as_float(u[i]));
      o[i] = act_round(gelu_epilogue(x, nullptr, 0, 0) * lin);
    }
    store_row_chunk_f32(p.out + static_cast<size_t>(m) * p.F + f0, o, f0, p.F);
#else
    const uint16_t* lut = reinterpret_cast<const uint16_t*>(epi_smem);
    uint32_t o[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      float r[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float x = act_round(__uint_as_float(g[2 * i + e]));
        const float lin = act_round(__uint_as_float(u[2 * i + e]));
        r[e] = gelu_epilogue(x, lut, p.lut.lo, p.lut.hi) * lin;
      }
      o[i] = pack_act2(r[0], r[1]);
    }
    store_row_chunk(p.out + static_cast<size_t>(m) * p.F + f0, o, f0, p.F);
#endif
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int /*N*/, const uint8_t* epi_smem,
                         int part, int parts) {
    constexpr int HALF = BN / 2;
    constexpr int C = HALF / 32;
#pragma unroll 1
    for (int c = part * C / parts; c < (part + 1) * C / parts; ++c) {
      uint32_t g[32], u[32];
      acc_ld_32(taddr + c * 32, g);
      acc_ld_32(taddr + HALF + c * 32, u);
      const int f0 = n_tile * HALF + c * 32;
      if (m_ok && f0 < p.F) chunk2(p, g, u, m, f0, epi_smem);
    }
  }
};

// ---- GeGLU of the teacher-forced forward pass (b200t5_forward): EpiGeglu's arithmetic and rounding, element for
// element, on the decode step's `wi` packing read in 128-wide tiles, eight features at a time instead of 32. The fp16
// build evaluates gelu_new op by op, and 32 gate + 32 up + 32 outputs per thread spill under this kernel's register
// budget; eight at a time do not.
struct EpiGegluNarrow {
  using Params = EpiGeglu::Params;
  static DEVINL void prologue(const Params& p, uint8_t* epi_smem, int tid, int nthreads = 128) {
    EpiGeglu::prologue(p, epi_smem, tid, nthreads);
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int /*N*/, const uint8_t* epi_smem,
                         int part, int parts) {
    constexpr int HALF = BN / 2;
    constexpr int C = HALF / 8;
#pragma unroll 1
    for (int c = part * C / parts; c < (part + 1) * C / parts; ++c) {
      const int f0 = n_tile * HALF + c * 8;
      if (!m_ok || f0 >= p.F) continue;  // F is a multiple of 32: a group of 8 is whole or absent
      uint32_t g[8], u[8];
#pragma unroll
      for (int v = 0; v < 2; ++v) {
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(g[4 * v]), "=r"(g[4 * v + 1]), "=r"(g[4 * v + 2]), "=r"(g[4 * v + 3])
                     : "r"((taddr + c * 8 + 4u * v) << 2) : "memory");
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u[4 * v]), "=r"(u[4 * v + 1]), "=r"(u[4 * v + 2]), "=r"(u[4 * v + 3])
                     : "r"((taddr + HALF + c * 8 + 4u * v) << 2) : "memory");
      }
#if B200T5_F16
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float x = act_round(__uint_as_float(g[i]));
        const float lin = act_round(__uint_as_float(u[i]));
        o[i] = act_round(gelu_epilogue(x, nullptr, 0, 0) * lin);
      }
      float4* dst = reinterpret_cast<float4*>(p.out + static_cast<size_t>(m) * p.F + f0);
      dst[0] = make_float4(o[0], o[1], o[2], o[3]);
      dst[1] = make_float4(o[4], o[5], o[6], o[7]);
#else
      const uint16_t* lut = reinterpret_cast<const uint16_t*>(epi_smem);
      uint32_t o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float r[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = act_round(__uint_as_float(g[2 * i + e]));
          const float lin = act_round(__uint_as_float(u[2 * i + e]));
          r[e] = gelu_epilogue(x, lut, p.lut.lo, p.lut.hi) * lin;
        }
        o[i] = pack_act2(r[0], r[1]);
      }
      *reinterpret_cast<uint4*>(p.out + static_cast<size_t>(m) * p.F + f0) = make_uint4(o[0], o[1], o[2], o[3]);
#endif
    }
  }
};

// ---- ReLU feed-forward of T5 v1.0 (T5DenseActDense, modeling_t5.py:84-100): out = relu(act(acc)), the A operand of
// `wo` in ffh_t (fp16 build: fp32 holding fp16 values, the cast up of transformers' forward). relu(act(x)) ==
// act(relu(x)), so the one rounding point is transformers': the output of `wi`. `wi` is stored as is ([F, d], no
// interleave), so N = F and the stores clip to it.
struct EpiRelu {
  struct Params {
    ffh_t* out;  // [M, ld]
    int ld;
  };
  static constexpr bool kPaired = false;
  typedef NoPre ChunkPre;
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  static DEVINL void chunk_pre(const Params&, int, int, int, ChunkPre&) {}
  static DEVINL float relu(float x) { return x < 0.f ? 0.f : x; }  // NaN propagates, as torch.relu
  static DEVINL void chunk(const Params& p, const uint32_t (&acc)[32], int m, int n0, int N, const uint8_t*,
                           const ChunkPre&) {
#if B200T5_F16
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = relu(act_round(__uint_as_float(acc[i])));
    store_row_chunk_f32(p.out + static_cast<size_t>(m) * p.ld + n0, o, n0, N);
#else
    uint32_t o[16];
#pragma unroll
    for (int i = 0; i < 16; ++i)
      o[i] = pack_act2(relu(act_round(__uint_as_float(acc[2 * i]))), relu(act_round(__uint_as_float(acc[2 * i + 1]))));
    store_row_chunk(p.out + static_cast<size_t>(m) * p.ld + n0, o, n0, N);
#endif
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es,
                         int part, int parts) {
    run_chunks<BN, EpiRelu>(p, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};

// ---- cross-attention K/V projection for all decoder layers at once (X1):
// row m = (b, s) of the encoder output; column n = ((layer*2 + kv)*H + h)*64 + d.
// Written straight into the decode arena  [layer][kv][B][H][S][64].
struct EpiCrossKV {
  struct Params {
    act_t* arena;
    int B, H, S;
    const int* row_b = nullptr;  // packed encoder rows: row m is position row_s[m] of prompt row_b[m]
    const int* row_s = nullptr;
  };
  static constexpr bool kPaired = false;
  typedef NoPre ChunkPre;
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  static DEVINL void chunk_pre(const Params&, int, int, int, ChunkPre&) {}
  static DEVINL void chunk(const Params& p, const uint32_t (&acc)[32], int m, int n0, int N, const uint8_t*,
                           const ChunkPre&) {
    const int b = p.row_b ? p.row_b[m] : m / p.S;
    const int s = p.row_s ? p.row_s[m] : m - b * p.S;
    const int hd = p.H * 64;
    const int lkv = n0 / hd;
    const int rem = n0 - lkv * hd;
    const int h = rem >> 6, d0 = rem & 63;
    uint32_t o[16];
    round_pack_32(acc, o);
    act_t* dst = p.arena + ((((static_cast<size_t>(lkv) * p.B + b) * p.H + h) * p.S + s) << 6) + d0;
    store_row_chunk(dst, o, n0, N);
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es,
                         int part, int parts) {
    run_chunks<BN, EpiCrossKV>(p, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};

// ---- decoder self-attention QKV for one new token: q -> q buffer, k/v appended in
// place at row *step of the preallocated cache [kv][B][H][Tmax][64] (replaces the
// torch.cat regrowth of transformers/cache_utils.py:119-120).
struct EpiQkvDecode {
  struct Params {
    act_t* q;      // [B, I]
    act_t* cache;  // this layer: [2][B][H][Tmax][64]
    const int* step;       // device scalar: current decode position t
    int B, H, Tmax;
    int step_stride = 0;   // 1 = slot pool: row m appends at its own position step[m]
  };
  static constexpr bool kPaired = false;
  typedef NoPre ChunkPre;
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  static DEVINL void chunk_pre(const Params&, int, int, int, ChunkPre&) {}
  static DEVINL void chunk(const Params& p, const uint32_t (&acc)[32], int m, int n0, int N, const uint8_t*,
                           const ChunkPre&) {
    const int I = p.H * 64;
    uint32_t o[16];
    round_pack_32(acc, o);
    act_t* dst;
    if (n0 < I) {
      dst = p.q + static_cast<size_t>(m) * I + n0;
    } else {
      const int t = p.step[m * p.step_stride];
      const int r = n0 - I;
      const int kv = r / I;
      const int rem = r - kv * I;
      const int h = rem >> 6, d0 = rem & 63;
      dst = p.cache + ((((static_cast<size_t>(kv) * p.B + m) * p.H + h) * p.Tmax + t) << 6) + d0;
    }
    store_row_chunk(dst, o, n0, N);
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es,
                         int part, int parts) {
    run_chunks<BN, EpiQkvDecode>(p, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};

// ---- lm_head epilogue of the decode step: logits never reach HBM. Each (row, n_tile) emits the max of its BN column
// values and the lowest column index attaining it (torch.argmax first-index contract; generation/utils.py:2762,2793);
// finalize_step_kernel merges the tiles. A row is not split: the first of the `parts` threads of each row takes it all.
//   kProc = false: a column's value is its logit rounded to act_t, EOS masked to -inf while step < min_new
//     (generation/logits_process.py:225-233).
//   kProc = true (logits_process.cuh): the logit after transformers' greedy processors. Each logit is rounded to act_t
//     and widened to fp32 (HF's `.to(torch.float32)`), then in HF's order: encoder repetition penalty, repetition
//     penalty (on the already penalised value), + 0 when bad words are active (HF adds a zero bias), and -inf where the
//     row's next-step bans, the static mask, the begin-suppress mask (step ProcCfg::begin_t, the first generated position) or the EOS
//     mask (step < min_new) has the
//     column's bit.
//   kScore (token log-probabilities): also, per (row, tile),
//     psum = sum_n expf(v_n - tile max)   (-inf columns add 0; an all -inf tile emits 0)
//     accumulated in ascending column order by the one thread that owns the row, so it does not depend on where the
//     row sits. The tile is read twice from the staged accumulators: once for the maximum, once for the sum. When the
//     step is teacher-forced, ftok[m] is the row's forced column (-1: none) and the tile that contains it writes its
//     value to fval[m].
// The arg-max and the log-sum-exp see the same fp32 number per column.
struct LmHeadParams {
  float* pval;  // [M, n_tiles]
  int* pidx;    // [M, n_tiles]
  int n_tiles;
  const int* step;
  int eos, min_new;
  int step_stride;  // 1 = slot pool: per-row positions
  ProcDev pd;       // kProc
  float* psum;      // kScore: [M, n_tiles]
  float* fval;      // kScore: [M]
  const int* ftok;  // kScore: [M], nullptr = the step is not teacher-forced
  float* vals;      // test hook only, else nullptr: the processed values [M, ldv]
  int ldv;
};

template <bool kProc, bool kScore>
struct EpiLmHead {
  using Params = LmHeadParams;
  // The plain head never writes `vals` (its test hook reads only tokens): a per-column test would cost the hot path.
  static constexpr bool kVals = kProc || kScore;
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  // What a processed row needs of the call's configuration, and the bitmap words of one 32-column chunk of it
  struct Row {
    bool enc_pen, rep_pen, bad_add;
    float en, ep, rn, rp;
    size_t rw;
    int t, begin_t;
  };
  struct Words {
    uint32_t ban, seen, enc;
  };
  static DEVINL Row row(const Params& p, int m, bool m_ok) {
    const ProcCfg& cf = *p.pd.cfg;
    Row r;
    r.enc_pen = cf.enc_pen;
    r.rep_pen = cf.rep_pen;
    r.bad_add = cf.bad_add;
    r.en = cf.enc_neg;
    r.ep = cf.enc_pos;
    r.rn = cf.rep_neg;
    r.rp = cf.rep_pos;
    r.rw = static_cast<size_t>(p.pd.row0 + m) * p.pd.W;
    r.t = m_ok ? p.step[m * p.step_stride] : 1;
    r.begin_t = cf.begin_t;
    return r;
  }
  static DEVINL Words words(const Params& p, const Row& r, bool m_ok, int n0) {
    const int W = p.pd.W, w = n0 >> 5;
    Words o{0, 0, 0};
    if (m_ok && w < W) {
      o.ban = p.pd.banned[r.rw + w] | p.pd.stat[w];
      if (r.t == r.begin_t) o.ban |= p.pd.stat[W + w];
      if (r.t < p.min_new) o.ban |= p.pd.stat[2 * W + w];
      if (r.rep_pen) o.seen = p.pd.seen[r.rw + w];
      if (r.enc_pen) o.enc = p.pd.enc[r.rw + w];
    }
    return o;
  }
  // the value of column n without processors: EOS masked by index
  static DEVINL float value(const Params& p, uint32_t acc, int n, int N, bool block_eos) {
    const float v = act_round(__uint_as_float(acc));
    return (n >= N || (block_eos && n == p.eos)) ? -INFINITY : v;
  }
  // ... and with processors: EOS masked by the bitmap
  static DEVINL float value(const Row& r, const Words& o, uint32_t acc, int j, int n, int N) {
    float v = act_round(__uint_as_float(acc));
    if ((o.enc >> j) & 1u) v = v < 0.f ? v * r.en : v * r.ep;
    if ((o.seen >> j) & 1u) v = v < 0.f ? v * r.rn : v * r.rp;
    if (r.bad_add) v = v + 0.f;
    if (n >= N || ((o.ban >> j) & 1u)) v = -INFINITY;
    return v;
  }
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t*, int part, int) {
    static_assert(BN % 32 == 0, "one bitmap word per 32 columns");
    if (part != 0) return;
    Row r{};
    bool block_eos = false;
    if constexpr (kProc) r = row(p, m, m_ok);
    else block_eos = m_ok && p.step[m * p.step_stride] < p.min_new;
    int forced = -1;
    if constexpr (kScore) forced = (m_ok && p.ftok != nullptr) ? p.ftok[m] : -1;
    float best = -INFINITY, sum = 0.f;
    int bidx = n_tile * BN;  // all -inf (cannot happen with finite logits) -> first column, like torch
#pragma unroll 1
    for (int pass = 0; pass < (kScore ? 2 : 1); ++pass) {
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        uint32_t acc[32];
        acc_ld_32(taddr + c * 32, acc);
        const int n0 = n_tile * BN + c * 32;
        Words o{0, 0, 0};
        if constexpr (kProc) o = words(p, r, m_ok, n0);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int n = n0 + j;
          float v;
          if constexpr (kProc) v = value(r, o, acc[j], j, n, N);
          else v = value(p, acc[j], n, N, block_eos);
          if (pass == 0) {
            if (v > best) {  // ascending scan + strict '>' keeps the lowest index among equal maxima
              best = v;
              bidx = n;
            }
            if constexpr (kScore)
              if (n == forced) p.fval[m] = v;
            if constexpr (kVals)
              if (p.vals != nullptr && m_ok && n < N) p.vals[static_cast<size_t>(m) * p.ldv + n] = v;
          } else if (v != -INFINITY) {
            sum += expf(v - best);
          }
        }
      }
    }
    if (m_ok) {
      p.pval[static_cast<size_t>(m) * p.n_tiles + n_tile] = best;
      p.pidx[static_cast<size_t>(m) * p.n_tiles + n_tile] = bidx;
      if constexpr (kScore) p.psum[static_cast<size_t>(m) * p.n_tiles + n_tile] = sum;
    }
  }
};

// ---- lm_head of the teacher-forced forward pass with logits requested: C [M, ldc] = act(acc), in the build's 2-byte
// type (HF's logits dtype; the act-rounded values are exact in it), and with kLabels also EpiLmHead<false, true>'s
// partials of the same values for the label columns lm.ftok.
template <bool kLabels>
struct EpiLmLogits {
  struct Params {
    LmHeadParams lm;
    act_t* C;
    size_t ldc;
  };
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t* es, int part, int parts) {
#pragma unroll 1
    for (int c = part * (BN / 32) / parts; c < (part + 1) * (BN / 32) / parts; ++c) {
      uint32_t acc[32];
      acc_ld_32(taddr + c * 32, acc);
      const int n0 = n_tile * BN + c * 32;
      if (m_ok && n0 < N) {
        act_t* dst = p.C + static_cast<size_t>(m) * p.ldc + n0;
        if (n0 + 32 <= N && p.ldc % 8 == 0) {
          uint32_t o[16];
          round_pack_32(acc, o);
          store_row_chunk(dst, o, n0, N);
        } else {
          for (int j = 0; j < 32 && n0 + j < N; ++j) dst[j] = float2act(__uint_as_float(acc[j]));
        }
      }
    }
    if constexpr (kLabels) EpiLmHead<false, true>::template run<BN>(p.lm, taddr, m, m_ok, n_tile, N, es, part, parts);
  }
};

// ---- fp32 logits store (test hook / teacher-forced parity): C = float(bf16(acc))
struct EpiStoreF32 {
  struct Params {
    float* C;
    int ldc;
  };
  static DEVINL void prologue(const Params&, uint8_t*, int, int = 128) {}
  template <int BN>
  static DEVINL void run(const Params& p, uint32_t taddr, int m, bool m_ok, int n_tile, int N, const uint8_t*, int part, int parts) {
#pragma unroll 1
    for (int c = part * (BN / 32) / parts; c < (part + 1) * (BN / 32) / parts; ++c) {
      uint32_t acc[32];
      acc_ld_32(taddr + c * 32, acc);
      const int n0 = n_tile * BN + c * 32;
      if (m_ok) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (n0 + j < N) p.C[static_cast<size_t>(m) * p.ldc + n0 + j] = act_round(__uint_as_float(acc[j]));
      }
    }
  }
};

// ======================================================================== host launch
// Opt in to the large dynamic shared memory carve-out once per process/device
// (done at b200t5_create so it never happens inside a stream capture).
template <int BN, class Epi, bool kTf32 = false, int kBBox = BN>
cudaError_t prepare_gemm() {
  return cudaFuncSetAttribute(gemm_bf16_tn_kernel<BN, Epi, kTf32, kBBox>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              GemmCfg<BN>::kSmemBytes);
}

// Launch with (optionally) the programmatic-stream-serialization attribute (PDL).
template <class... KArgs, class... Args>
cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                          Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// a_kblocks: see kTf32 at the kernel (0 = A spans all of K)
template <int BN, class Epi, bool kTf32 = false, int kBBox = BN>
cudaError_t launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, int m_fastest,
                        const typename Epi::Params& ep, int num_sms, cudaStream_t stream, bool pdl = false, int a_kblocks = 0) {
  using Cfg = GemmCfg<BN>;
  const int tiles = ((M + kBM - 1) / kBM) * ((N + BN - 1) / BN);
  const int slots = num_sms * Cfg::kCtasPerSm;
  const int grid = tiles < slots ? tiles : slots;
  return launch_kernel(gemm_bf16_tn_kernel<BN, Epi, kTf32, kBBox>, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, pdl,
                       tmA, tmB, M, N, K, m_fastest, ep, a_kblocks);
}

}  // namespace b200
