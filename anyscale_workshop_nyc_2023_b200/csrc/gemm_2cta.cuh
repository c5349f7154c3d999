// Encoder GEMMs (M = packed prompt rows, tens of thousands):  D[M,N] = A[M,K] * W[N,K]^T  on 128 x 256 tiles.
//
// The encoder's tensor maps (tm2_*) have 128-row boxes for both operands; this configuration of the persistent
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

}  // namespace b200
