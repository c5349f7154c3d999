// Encoder GEMMs (M = packed prompt rows, tens of thousands):  D[M,N] = A[M,K] * W[N,K]^T  on 128 x 256 tiles.
//
// The encoder's tensor maps (EncLayerW::tm_*, tm_crosskv) have 128-row boxes for both operands; this configuration of the persistent
// wgmma kernel (gemm.cuh) loads each 256-row weight tile as two such boxes. A 128 x 256 tile is the largest the
// two consumer warpgroups hold in registers (128 fp32 accumulators per thread) and gives the best operand reuse
// per byte of shared memory: per k-block 48 KB are staged for 128 x 256 x 64 MACs.
//
// kTf32 (fp16 build, the fp32-weight `wo` product): both operands are fp32 in memory and consumed as tf32, a
// k-block is 32 elements (the same 128-byte rows) and K counts the columns of W' = [W_hi | W_lo], the two
// tf32 pieces of the fp32 weight side by side; A has only a_kblocks k-blocks and is walked twice (kb % a_kblocks),
// so the accumulator receives A . W_hi^T + A . W_lo^T.
#pragma once
#include "gemm.cuh"

namespace b200 {

constexpr int k2ctaBN = 256;
constexpr int k2ctaBox = 128;

template <class Epi, bool kTf32 = false>
cudaError_t prepare_gemm_2cta() {
  return prepare_gemm<k2ctaBN, Epi, kTf32, k2ctaBox>();
}

// a_kblocks: see kTf32 above (0 = A spans all of K). Tiles are visited n-fastest: the CTAs that run at the same
// time share the rows of A.
template <class Epi, bool kTf32 = false>
cudaError_t launch_gemm_2cta(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K,
                             const typename Epi::Params& ep, int num_sms, cudaStream_t stream, int a_kblocks = 0) {
  return launch_gemm<k2ctaBN, Epi, kTf32, k2ctaBox>(tmA, tmB, M, N, K, 0, ep, num_sms, stream, false, a_kblocks);
}

// ======================================================================== epilogue-overlapped encoder GEMM
// gemm_enc_ws_kernel<Epi>: the same 128 x 256 tiles, TMA boxes, wgmma sequence and n-fastest persistent tile order as
// the configuration above, so its fp32 accumulators are bit-identical. What differs is where the epilogue runs.
// One 48 KB-per-stage CTA fills an SM, so in the kernel above nothing hides the epilogue: the staged fp32 tile
// aliases the TMA ring and the main loop of the next tile waits for it. Here:
//   - every encoder epilogue (EpiStore, EpiResidual with round_acc, EpiGeglu, EpiCrossKV) first rounds the
//     accumulator to act_t, so the consumers round and write the tile into a 64 KB act_t staging buffer of its own,
//     outside the (now 3-stage) ring; the producer never waits on the epilogue;
//   - three epilogue warps drain the staged tile into HBM through the unchanged functor `chunk` / `chunk2` code while
//     the two consumer warpgroups run the next tile's MMAs. stg_full / stg_empty hand the buffer back and forth.
// Rounding a value that is already an act_t is exact, so each functor's arithmetic sees the same inputs as before.
//
// Warp roles (384 threads): warps 0..7 consumers (MMA + staging), warp 8 TMA producer, warps 9..11 epilogue.
constexpr int kEncWsThreads = 384;
constexpr int kEncWsEpiThreads = 96;
constexpr int kEncWsEpiWarp0 = 9;

struct EncWsCfg {
  static constexpr int kBN = k2ctaBN;
  static constexpr int kStages = 3;
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = kBN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRingBytes = kStages * kStageBytes;
  static constexpr int kStagingBytes = kBM * kBN * 2;  // act_t rows of 512 B, 16-B units swizzled (enc_stg_unit)
  static constexpr int kSmemBytes = kRingBytes + kStagingBytes + 1024 /*align*/ + 256 /*barriers*/ + kEpiSmemBytes;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

// Byte offset of 16-B unit u (8 act_t columns, 0..31) of staged row r. The XOR keeps three access patterns free of
// bank conflicts: the consumers' 4-byte fragment writes (one unit of 8 consecutive rows per warp instruction), the
// epilogue's 16-B reads of 8 chunks of one row (row-major items), and GeGLU's reads of 4 chunks of two adjacent rows.
DEVINL uint32_t enc_stg_unit(int r, int u) {
  const int f = ((u >> 3) & 3) ^ (((r & 1) << 1) | ((r >> 1) & 1) | (r & 4));
  return static_cast<uint32_t>(r * 512 + ((u ^ f) << 4));
}

// A warpgroup's accumulators (tile rows row0 .. row0+63) rounded to act_t into the staging rows.
DEVINL void enc_stage_act(uint32_t stg, int row0, const float (&acc)[k2ctaBN / 2]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const uint32_t w = 4u * (t & 3);
#pragma unroll
  for (int j = 0; j < k2ctaBN / 8; ++j) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + enc_stg_unit(r, j) + w), "r"(pack_act2(acc[4 * j], acc[4 * j + 1])) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + enc_stg_unit(r + 8, j) + w), "r"(pack_act2(acc[4 * j + 2], acc[4 * j + 3])) : "memory");
  }
}

// Staged columns [32 u0 / 4, +32) of row r (four units from u0) as fp32 bit patterns, the form the functors take.
DEVINL void enc_stg_ld_chunk(uint32_t stg, int r, int u0, uint32_t (&acc)[32]) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    uint32_t w[4];
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
                 : "r"(stg + enc_stg_unit(r, u0 + g))
                 : "memory");
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      acc[8 * g + 2 * k] = __float_as_uint(act_lo(w[k]));
      acc[8 * g + 2 * k + 1] = __float_as_uint(act_hi(w[k]));
    }
  }
}

// Epilogue thread e (0..95) drains one staged tile. Unpaired functors: item i = (row i / 8, chunk i % 8), so eight
// lanes cover one 512-B output row segment; the pre-operands (residual) of the thread's next item are fetched before
// the current item is processed, and those of its first item before the staged tile is waited for.
// GeGLU: item i = (row i / 4, feature chunk i % 4), gate columns in units [0, 16), up columns in [16, 32).
template <class Epi>
DEVINL void enc_ws_drain(const typename Epi::Params& p, uint32_t stg, int m0, int M, int n_tile, int N,
                         const uint8_t* es, int e, uint64_t* full, uint32_t parity) {
  if constexpr (Epi::kPaired) {
    mbar_wait(full, parity);
#pragma unroll 1
    for (int i = e; i < kBM * 4; i += kEncWsEpiThreads) {
      const int r = i >> 2, c = i & 3;
      const int m = m0 + r, f0 = n_tile * (k2ctaBN / 2) + c * 32;
      uint32_t g[32], u[32];
      enc_stg_ld_chunk(stg, r, 4 * c, g);
      enc_stg_ld_chunk(stg, r, 16 + 4 * c, u);
      if (m < M && f0 < p.F) Epi::chunk2(p, g, u, m, f0, es);
    }
  } else {
    constexpr int kItems = kBM * 8;
    typename Epi::ChunkPre pre[2];
    const int n_base = n_tile * k2ctaBN;
    if (m0 + (e >> 3) < M && n_base + (e & 7) * 32 < N) Epi::chunk_pre(p, m0 + (e >> 3), n_base + (e & 7) * 32, N, pre[0]);
    mbar_wait(full, parity);
#pragma unroll 1
    for (int i = e; i < kItems; i += 2 * kEncWsEpiThreads) {
#pragma unroll
      for (int v = 0; v < 2; ++v) {
        const int it = i + v * kEncWsEpiThreads;
        if (it < kItems) {
          const int nx = it + kEncWsEpiThreads;
          if (nx < kItems && m0 + (nx >> 3) < M && n_base + (nx & 7) * 32 < N)
            Epi::chunk_pre(p, m0 + (nx >> 3), n_base + (nx & 7) * 32, N, pre[(v + 1) & 1]);
          const int r = it >> 3, c = it & 7;
          const int m = m0 + r, n0 = n_base + c * 32;
          uint32_t acc[32];
          enc_stg_ld_chunk(stg, r, 4 * c, acc);
          if (m < M && n0 < N) Epi::chunk(p, acc, m, n0, N, es, pre[v]);
        }
      }
    }
  }
}

template <class Epi>
__global__ void __launch_bounds__(kEncWsThreads, 1)
gemm_enc_ws_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K,
                   typename Epi::Params ep) {
  using Cfg = EncWsCfg;
  constexpr int BN = Cfg::kBN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t stg = smem_u32(smem + Cfg::kRingBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kRingBytes + Cfg::kStagingBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::kStages;
  uint64_t* stg_full = bars + 2 * Cfg::kStages;   // both consumer warpgroups have staged the tile
  uint64_t* stg_empty = stg_full + 1;             // every epilogue thread has read it
  uint8_t* epi_smem = smem + Cfg::kRingBytes + Cfg::kStagingBytes + 256;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (M + kBM - 1) / kBM;
  const int tiles_n = (N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int kblocks = (K + kBK - 1) / kBK;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    mbar_init(stg_full, kGemmConsumers);
    mbar_init(stg_empty, kEncWsEpiThreads);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      if (static_cast<int>(blockIdx.x) < num_tiles) {
        const TileCoord tc0 = tile_coord(blockIdx.x, tiles_m, tiles_n, 0);
        for (int kb = 0; kb < kblocks; ++kb)
          for (int p = 0; p < BN / k2ctaBox; ++p) tma_prefetch_l2_2d(&tmB, kb * kBK, tc0.n_tile * BN + p * k2ctaBox);
      }
      pdl_wait();
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(tile, tiles_m, tiles_n, 0);
        const int m0 = tc.m_tile * kBM, n0 = tc.n_tile * BN;
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u);
          uint8_t* sA = smem + stage * Cfg::kStageBytes;
          uint8_t* sB = sA + Cfg::kABytes;
          mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
          tma_load_2d(sA, &tmA, &full[stage], kb * kBK, m0);
#pragma unroll
          for (int p = 0; p < BN / k2ctaBox; ++p) tma_load_2d(sB + p * k2ctaBox * 128, &tmB, &full[stage], kb * kBK, n0 + p * k2ctaBox);
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else if (warp >= kEncWsEpiWarp0) {
    // ------------------------------------------------------------ epilogue warps
    const int e = threadIdx.x - kEncWsEpiWarp0 * 32;
    Epi::prologue(ep, epi_smem, e, kEncWsEpiThreads);  // constant tables (named barrier 2 among these 96 threads)
    pdl_wait();
    uint32_t sphase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord tc = tile_coord(tile, tiles_m, tiles_n, 0);
      enc_ws_drain<Epi>(ep, stg, tc.m_tile * kBM, M, tc.n_tile, N, epi_smem, e, stg_full, sphase);
      mbar_arrive(stg_empty);
      sphase ^= 1u;
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups
    const int wg = warp >> 2;
    int stage = 0;
    uint32_t phase = 0, sphase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStageBytes) + wg * 64 * 128;
        wgmma_fence_acc(acc);
        wgmma_fence();
        wgmma_kblock<BN, false>(acc, a_addr, smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes));
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
      mbar_wait(stg_empty, sphase ^ 1u);  // the epilogue warps have read the previous tile
      enc_stage_act(stg, wg * 64, acc);
      mbar_arrive(stg_full);
      sphase ^= 1u;
    }
  }
}

template <class Epi>
cudaError_t prepare_gemm_enc_ws() {
  return cudaFuncSetAttribute(gemm_enc_ws_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, EncWsCfg::kSmemBytes);
}

// Every functor this kernel drives must round the accumulator to act_t first: the fp16 build's fp32 `wo` product
// (EpiResidual with round_acc = 0) stays on launch_gemm_2cta.
template <class Epi>
cudaError_t launch_gemm_enc_ws(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K,
                               const typename Epi::Params& ep, int num_sms, cudaStream_t stream) {
  if constexpr (std::is_same<Epi, EpiResidual>::value) {
    if (!ep.round_acc) return cudaErrorInvalidValue;
  }
  const int tiles = ((M + kBM - 1) / kBM) * ((N + k2ctaBN - 1) / k2ctaBN);
  const int grid = tiles < num_sms ? tiles : num_sms;
  return launch_kernel(gemm_enc_ws_kernel<Epi>, dim3(grid), dim3(kEncWsThreads), EncWsCfg::kSmemBytes, stream, false,
                       tmA, tmB, M, N, K, ep);
}

}  // namespace b200
