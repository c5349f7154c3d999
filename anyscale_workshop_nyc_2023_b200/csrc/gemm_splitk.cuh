// Split-K bf16 GEMM for the skinny decode-step products (M = batch rows <= a few hundred):
//   D[M,N] = A[M,K] * W[N,K]^T,  one 128 x BN output tile per CLUSTER, K cut across the
//   cluster's CTAs, partial sums reduced through distributed shared memory.
//
// Why: with M = 256 a decode GEMM has only (M/128)*(N/BN) output tiles, and every tile's CTA
// must pull (128 + BN) * K * 2 bytes through ONE SM. For N = 768, K = 2048 that is 650 KB per CTA
// on 12 of the 132 SMs. Cutting K over a cluster of S CTAs divides the per-SM bytes by S and
// multiplies the number of busy SMs by S; the reduction costs one DSMEM pass.
//
// Per CTA (288 threads, the roles of gemm.cuh): warp 8 = TMA producer (the weight slices do not
// depend on the previous kernel and are requested BEFORE griddepcontrol.wait), warps 0..7 = two
// consumer warpgroups, each running wgmma over 64 tile rows with fp32 accumulators in registers.
// Reduce-scatter by ROWS: rank r of the cluster owns tile rows [r*128/S, (r+1)*128/S); every
// consumer thread sends its accumulator fragments to the owner's `red` buffer slot [src rank][row]
// with st.shared::cluster, a cluster barrier (release/acquire) publishes the writes, and the owner
// sums the S partials in rank order (deterministic) and feeds 32-column chunks to the same epilogue
// functors the persistent GEMM uses (gemm.cuh), so the T5 rounding contract is shared.
//
// Footprint: the number of pipeline stages is a launch parameter, so that a CTA can be sized to fit on
// an SM next to the resident CTAs of the other row-chain's cross-attention stream (attention_cross_stream.cuh).
#pragma once
#include "gemm.cuh"

namespace b200 {

constexpr int kSkThreads = kGemmThreads;  // 2 consumer warpgroups + 1 producer warp
// Register cap: one split-K CTA (288 threads) must fit on an SM next to two CTAs of the other row-chain's
// cross-attention stream kernel (2 x 160 threads x 64 registers): (65536 - 20480) / 288 -> 152 per thread.
// Left to __launch_bounds__(288, 1), ptxas takes 168 and only one stream CTA fits beside the GEMM.
constexpr int kSkMaxRegs = 152;
constexpr int kSkMaxSplit = 8;
constexpr int kSkMaxStages = 4;

template <int BN>
struct SkCfg {
  static_assert(BN == 64 || BN == 128, "BN");
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kDefaultStages = BN == 64 ? 4 : 3;
  static constexpr int kRedLd = BN + 4;  // floats; +4 keeps the per-row v4 stores of a warp conflict-free
  static constexpr int kRedBytes = kBM * kRedLd * 4;  // [src rank][row of the owner] = 128 slots whatever the split
  // `epi`: the epilogue functor stages a table in shared memory (GeGLU); the others get no scratch, which is what
  // lets a BN = 64 CTA (131 KB) share an SM with two CTAs of the cross-attention stream (2 x 46 KB)
  static constexpr int smem_bytes(int stages, bool epi) {
    return stages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/ + kRedBytes + (epi ? kEpiSmemBytes : 0);
  }
  static constexpr int kMaxSmemBytes = smem_bytes(kSkMaxStages, true);
};

// ---------------------------------------------------------------- cluster PTX
DEVINL uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
DEVINL uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
DEVINL void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
DEVINL void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
DEVINL void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
DEVINL uint32_t mapa_shared(uint32_t cta_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(cta_addr), "r"(rank));
  return r;
}
DEVINL void st_cluster_v2(uint32_t addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

DEVINL void add32_smem(uint32_t (&acc)[32], const float* src) {
  const float4* r4 = reinterpret_cast<const float4*>(src);
#pragma unroll
  for (int v = 0; v < 8; ++v) {
    const float4 a = r4[v];
    acc[4 * v] = __float_as_uint(__uint_as_float(acc[4 * v]) + a.x);
    acc[4 * v + 1] = __float_as_uint(__uint_as_float(acc[4 * v + 1]) + a.y);
    acc[4 * v + 2] = __float_as_uint(__uint_as_float(acc[4 * v + 2]) + a.z);
    acc[4 * v + 3] = __float_as_uint(__uint_as_float(acc[4 * v + 3]) + a.w);
  }
}

// grid = (S, tiles_n, tiles_m), cluster = (S, 1, 1); S in {1,2,4,8} divides 128.
// kTf32 / a_kblocks: as in gemm.cuh (fp32 operands consumed as tf32, W' = [W_hi | W_lo], A walked twice).
template <int BN, class Epi, bool kTf32 = false>
__global__ void __maxnreg__(kSkMaxRegs)
gemm_splitk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N,
                   int K, typename Epi::Params ep, int a_kblocks, int stages) {
  using Cfg = SkCfg<BN>;
  constexpr int kbk = kTf32 ? kBK / 2 : kBK;  // elements per k-block (128 bytes)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + stages * Cfg::kStageBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kSkMaxStages;
  float* red = reinterpret_cast<float*>(smem + stages * Cfg::kStageBytes + 256);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int S = static_cast<int>(cluster_nctarank());
  const int rank = static_cast<int>(cluster_ctarank());
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(red) + Cfg::kRedBytes;
  const int n_tile = blockIdx.y, m_tile = blockIdx.z;
  const int kblocks = (K + kbk - 1) / kbk;
  if (a_kblocks <= 0) a_kblocks = kblocks;
  const int kb_per = (kblocks + S - 1) / S;
  const int kb0 = rank * kb_per;
  const int kb1 = (kb0 + kb_per) < kblocks ? (kb0 + kb_per) : kblocks;
  const int nkb = kb1 - kb0;  // host guarantees >= 1
  const int m0 = m_tile * kBM, n0t = n_tile * BN;

  pdl_launch_dependents();
  cluster_arrive_relaxed();  // #1: "this CTA runs" - peers wait for it before touching our shared memory
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      const int first = nkb < stages ? nkb : stages;
      // weights first: they never depend on the previous kernel
      for (int i = 0; i < first; ++i) {
        uint8_t* sA = smem + i * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full[i], Cfg::kStageBytes);
        tma_load_2d(sA + Cfg::kABytes, &tmB, &full[i], (kb0 + i) * kbk, n0t);
      }
      pdl_wait();
      for (int i = 0; i < first; ++i) tma_load_2d(smem + i * Cfg::kStageBytes, &tmA, &full[i], ((kb0 + i) % a_kblocks) * kbk, m0);
      int stage = first == stages ? 0 : first;
      uint32_t phase = first == stages ? 1u : 0u;
      for (int i = first; i < nkb; ++i) {
        mbar_wait(&empty[stage], phase ^ 1u);
        uint8_t* sA = smem + stage * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
        tma_load_2d(sA, &tmA, &full[stage], ((kb0 + i) % a_kblocks) * kbk, m0);
        tma_load_2d(sA + Cfg::kABytes, &tmB, &full[stage], (kb0 + i) * kbk, n0t);
        if (++stage == stages) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
    __syncwarp();
    cluster_wait_acquire();    // #1
    cluster_arrive_release();  // #2
    cluster_wait_acquire();
  } else {
    // ------------------------------------------------------------ consumer warpgroups: MMA, scatter, reduce + epilogue
    const int et = threadIdx.x;  // 0..255
    const int wg = warp >> 2;
    const int rows_per = kBM / S;
    if constexpr (Epi::kPaired) Epi::prologue(ep, epi_smem, et, kGemmConsumers);  // gelu table; overlaps the main loop
    constexpr int kChunks = Epi::kPaired ? BN / 64 : BN / 32;
    const int items = rows_per * kChunks;
    pdl_wait();
    // the first work item's accumulator-independent operands (residual row) are fetched now
    typename Epi::ChunkPre pre0;
    {
      const int rl = et / kChunks, c = et - rl * kChunks;
      const int m = m0 + rank * rows_per + rl;
      if constexpr (!Epi::kPaired) {
        if (et < items && m < M && n0t + c * 32 < N) Epi::chunk_pre(ep, m, n0t + c * 32, N, pre0);
      }
    }
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    {
      int stage = 0, prev = -1;
      uint32_t phase = 0;
      for (int i = 0; i < nkb; ++i) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStageBytes) + wg * 64 * 128;
        wgmma_fence_acc(acc);
        wgmma_fence();
        wgmma_kblock<BN, kTf32>(acc, a_addr, smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes));
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_acc(acc);
        if (prev >= 0 && (et & 127) == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == stages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
    }
    cluster_wait_acquire();  // #1: every CTA of the cluster is running, its `red` buffer may be written
    {
      // reduce-scatter by rows: tile row r goes to slot [rank][r % rows_per] of rank r / rows_per
      const int t = et & 127;
      const int rbase = wg * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
      const int c = 2 * (t & 3);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = rbase + 8 * half;
        const int dst_rank = row / rows_per;
        const int slot = rank * rows_per + (row - dst_rank * rows_per);
        const uint32_t dst = mapa_shared(smem_u32(red + static_cast<size_t>(slot) * Cfg::kRedLd + c), static_cast<uint32_t>(dst_rank));
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) st_cluster_v2(dst + 32 * j, acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
      }
    }
    cluster_arrive_release();  // #2: partials published
    cluster_wait_acquire();
#pragma unroll 1
    for (int it = et; it < items; it += kGemmConsumers) {
      const int rl = it / kChunks, c = it - rl * kChunks;
      const int m = m0 + rank * rows_per + rl;
      if (m >= M) continue;
      if constexpr (Epi::kPaired) {
        constexpr int HALF = BN / 2;
        const int f0 = n_tile * HALF + c * 32;
        if (f0 >= ep.F) continue;
        uint32_t g[32], u[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) g[j] = u[j] = 0u;
        for (int src = 0; src < S; ++src) {
          const float* base = red + static_cast<size_t>(src * rows_per + rl) * Cfg::kRedLd;
          add32_smem(g, base + c * 32);
          add32_smem(u, base + HALF + c * 32);
        }
        Epi::chunk2(ep, g, u, m, f0, epi_smem);
      } else {
        const int n0 = n0t + c * 32;
        if (n0 >= N) continue;
        typename Epi::ChunkPre pre;
        if (it == et) pre = pre0;
        else Epi::chunk_pre(ep, m, n0, N, pre);
        uint32_t acc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = 0u;
        for (int src = 0; src < S; ++src) add32_smem(acc, red + static_cast<size_t>(src * rows_per + rl) * Cfg::kRedLd + c * 32);
        Epi::chunk(ep, acc, m, n0, N, epi_smem, pre);
      }
    }
  }
}

template <int BN, class Epi, bool kTf32 = false>
cudaError_t prepare_gemm_splitk() {
  cudaError_t e = cudaFuncSetAttribute(gemm_splitk_kernel<BN, Epi, kTf32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SkCfg<BN>::kMaxSmemBytes);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(gemm_splitk_kernel<BN, Epi, kTf32>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
}

// Largest split in {8,4,2,1} not above `want` that leaves every rank at least one k-block.
inline int splitk_factor(int K, int want, int kbk = kBK) {
  const int kblocks = (K + kbk - 1) / kbk;
  for (int s = want; s > 1; s >>= 1) {
    const int per = (kblocks + s - 1) / s;
    if ((s - 1) * per < kblocks) return s;
  }
  return 1;
}

// stages: 0 = the tile's default (4 for BN = 64, 3 for BN = 128), otherwise 2..4
template <int BN, class Epi, bool kTf32 = false>
cudaError_t launch_gemm_splitk(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, int split,
                               const typename Epi::Params& ep, cudaStream_t stream, bool pdl, int a_kblocks = 0, int stages = 0) {
  using Cfg = SkCfg<BN>;
  if (stages < 2 || stages > kSkMaxStages) stages = Cfg::kDefaultStages;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(split, (N + BN - 1) / BN, (M + kBM - 1) / kBM);
  cfg.blockDim = dim3(kSkThreads);
  cfg.dynamicSmemBytes = Cfg::smem_bytes(stages, Epi::kPaired);
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  attr[na].id = cudaLaunchAttributeClusterDimension;
  attr[na].val.clusterDim.x = split;
  attr[na].val.clusterDim.y = 1;
  attr[na].val.clusterDim.z = 1;
  ++na;
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, gemm_splitk_kernel<BN, Epi, kTf32>, tmA, tmB, M, N, K, ep, a_kblocks, stages);
}

}  // namespace b200
