// Single-query attention for the autoregressive decode step (HBM-bound streaming).
//
//   cross-attention (D7): q[b,h,:] against the S encoder keys of row b; bias is zero
//       plus the key-padding mask (modeling_t5.py:312-325). Reads the whole cross-KV
//       arena once per step: this kernel sets the decode roofline (SURVEY 8d).
//   self-attention  (D3): q against the t+1 cached keys, causal bucket bias taken from
//       a per-head table indexed by distance (modeling_t5.py:236-251, 319-321).
//
// Rounding contract (SURVEY Appendix A.3): s = bf16(q.k) ; s = bf16(s + bias) ;
// p = bf16( exp(s - max) / sum ) with max/sum in fp32 over the bf16 scores ;
// out = bf16( sum_j p_j v_j ) accumulated in fp32. Two streaming phases (K, then V)
// with the <= Tk scores parked in shared memory, so K and V are each read exactly once
// and the softmax is the exact (non-online) one HF computes.
//
// Layout: K and V are [B][H][Tk][64] bf16 (a (b,h) slab is contiguous: Tk*128 B).
// One CTA (4 warps) per (b,h); a key row (128 B) is read by 8 lanes x 16 B, so a warp
// load instruction covers 4 consecutive keys = 512 contiguous bytes.
#pragma once
#include "ptx.cuh"

namespace b200 {

#if B200T5_F16
constexpr float kActMin = -65504.0f;                // torch.finfo(torch.float16).min
#else
constexpr float kActMin = -3.3895313892515355e38f;  // torch.finfo(torch.bfloat16).min
#endif
constexpr int kAttnDecThreads = 128;
constexpr int kAttnDecUnroll = 8;

DEVINL float dot8(const uint4& kv, const float (&qf)[8]) {
  float s = act_lo(kv.x) * qf[0];
  s = fmaf(act_hi(kv.x), qf[1], s);
  s = fmaf(act_lo(kv.y), qf[2], s);
  s = fmaf(act_hi(kv.y), qf[3], s);
  s = fmaf(act_lo(kv.z), qf[4], s);
  s = fmaf(act_hi(kv.z), qf[5], s);
  s = fmaf(act_lo(kv.w), qf[6], s);
  s = fmaf(act_hi(kv.w), qf[7], s);
  return s;
}

// In-situ timing of the cross-attention launches inside the step graph (bench.py's roofline.frac): when `slots` is
// non-null every CTA folds its start / end %globaltimer into slot `slot` (min start, max end) and
// advance_step_kernel turns the slots into per-launch durations once per step. Null in the timed region.
struct XsStamps {
  unsigned long long* slots;  // [n_slots][2] = {min start, max end}
  int slot;
};

template <bool kSelf>
__global__ void __launch_bounds__(kAttnDecThreads)
attn_decode_kernel(const act_t* __restrict__ q,    // [B, H*64]
                   const act_t* __restrict__ Kc,   // [B][H][Tk][64]
                   const act_t* __restrict__ Vc,   // [B][H][Tk][64]
                   act_t* __restrict__ ctx,        // [B, H*64]
                   int H, int Tk,
                   const int* __restrict__ extent,            // cross: [B] keys to visit
                   const unsigned char* __restrict__ key_ok,  // cross: [B][Tk] 1 = attended
                   const int* __restrict__ step,              // self: device scalar t (or per-row positions)
                   const float* __restrict__ dist_bias,       // self: [H][Tk] bias by distance t-j
                   const XsStamps stamps,                     // cross: in-situ launch timing (slots == nullptr: off)
                   const int step_stride = 0) {               // self: 1 = slot pool, row b is at position step[b]
  extern __shared__ float s_scores[];  // Tk floats
  __shared__ float s_red[4][64];
  __shared__ float s_stat[8];

  pdl_launch_dependents();
  pdl_wait();
  unsigned long long t_start = 0;
  if (!kSelf && stamps.slots != nullptr && threadIdx.x == 0) t_start = global_timer_ns();
  const uint64_t stream_policy = l2_policy_evict_first();
  const int b = blockIdx.x / H, h = blockIdx.x - b * H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ks = lane >> 3, dg = lane & 7;
  const int t = kSelf ? step[b * step_stride] : 0;
  const int nkeys = kSelf ? t + 1 : extent[b];
  const size_t slab = (static_cast<size_t>(b) * H + h) * static_cast<size_t>(Tk) * 64;
  const act_t* Kp = Kc + slab + dg * 8;
  const act_t* Vp = Vc + slab + dg * 8;

  float qf[8];
  {
    const uint4 qv = *reinterpret_cast<const uint4*>(q + (static_cast<size_t>(b) * H + h) * 64 + dg * 8);
    qf[0] = act_lo(qv.x); qf[1] = act_hi(qv.x); qf[2] = act_lo(qv.y); qf[3] = act_hi(qv.y);
    qf[4] = act_lo(qv.z); qf[5] = act_hi(qv.z); qf[6] = act_lo(qv.w); qf[7] = act_hi(qv.w);
  }

  // ---------------- phase 1: scores
  // CTA-wide stride is 16 keys per step; kAttnDecUnroll independent 16-B loads in flight per thread.
  // (loop bound is warp-uniform: the shuffles below need all 32 lanes)
  for (int jb = warp * 4; jb < nkeys; jb += 16 * kAttnDecUnroll) {
    const int j0 = jb + ks;
    uint4 kv[kAttnDecUnroll];
#pragma unroll
    for (int u = 0; u < kAttnDecUnroll; ++u) {
      const int j = j0 + 16 * u;
      kv[u] = j < nkeys ? (kSelf ? ldg_nc_v4(Kp + static_cast<size_t>(j) * 64) : ldg_nc_v4_hint(Kp + static_cast<size_t>(j) * 64, stream_policy))
                        : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < kAttnDecUnroll; ++u) {
      const int j = j0 + 16 * u;
      float s = dot8(kv[u], qf);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      if (dg == 0 && j < nkeys) {
        s = act_round(s);
        if (kSelf) {
          s = act_round(s + dist_bias[h * Tk + (t - j)]);
        } else if (!key_ok[static_cast<size_t>(b) * Tk + j]) {
          s = kActMin;
        }
        s_scores[j] = s;
      }
    }
  }
  __syncthreads();

  // ---------------- softmax statistics over the bf16 scores (fp32, exact two-pass)
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nkeys; j += kAttnDecThreads) mx = fmaxf(mx, s_scores[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) s_stat[warp] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(s_stat[0], s_stat[1]), fmaxf(s_stat[2], s_stat[3]));
  float sum = 0.f;
  for (int j = threadIdx.x; j < nkeys; j += kAttnDecThreads) {
    const float e = expf(s_scores[j] - mx);
    s_scores[j] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) s_stat[4 + warp] = sum;
  __syncthreads();
  sum = (s_stat[4] + s_stat[5]) + (s_stat[6] + s_stat[7]);
  for (int j = threadIdx.x; j < nkeys; j += kAttnDecThreads) s_scores[j] = act_round(s_scores[j] / sum);
  __syncthreads();

  // ---------------- phase 2: out = P . V
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  for (int jb = warp * 4; jb < nkeys; jb += 16 * kAttnDecUnroll) {
    const int j0 = jb + ks;
    uint4 vv[kAttnDecUnroll];
    float p[kAttnDecUnroll];
#pragma unroll
    for (int u = 0; u < kAttnDecUnroll; ++u) {
      const int j = j0 + 16 * u;
      const bool ok = j < nkeys;
      vv[u] = ok ? (kSelf ? ldg_nc_v4(Vp + static_cast<size_t>(j) * 64) : ldg_nc_v4_hint(Vp + static_cast<size_t>(j) * 64, stream_policy))
                 : make_uint4(0, 0, 0, 0);
      p[u] = ok ? s_scores[j] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < kAttnDecUnroll; ++u) {
      acc[0] = fmaf(p[u], act_lo(vv[u].x), acc[0]);
      acc[1] = fmaf(p[u], act_hi(vv[u].x), acc[1]);
      acc[2] = fmaf(p[u], act_lo(vv[u].y), acc[2]);
      acc[3] = fmaf(p[u], act_hi(vv[u].y), acc[3]);
      acc[4] = fmaf(p[u], act_lo(vv[u].z), acc[4]);
      acc[5] = fmaf(p[u], act_hi(vv[u].z), acc[5]);
      acc[6] = fmaf(p[u], act_lo(vv[u].w), acc[6]);
      acc[7] = fmaf(p[u], act_hi(vv[u].w), acc[7]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], 8);
    acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], 16);
  }
  if (ks == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) s_red[warp][dg * 8 + e] = acc[e];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int d0 = threadIdx.x * 2;
    const float o0 = (s_red[0][d0] + s_red[1][d0]) + (s_red[2][d0] + s_red[3][d0]);
    const float o1 = (s_red[0][d0 + 1] + s_red[1][d0 + 1]) + (s_red[2][d0 + 1] + s_red[3][d0 + 1]);
    *reinterpret_cast<uint32_t*>(ctx + (static_cast<size_t>(b) * H + h) * 64 + d0) = pack_act2(o0, o1);
  }
  if (!kSelf && stamps.slots != nullptr && threadIdx.x == 0) {
    atomicMin(&stamps.slots[2 * stamps.slot], t_start);
    atomicMax(&stamps.slots[2 * stamps.slot + 1], static_cast<unsigned long long>(global_timer_ns()));
  }
}

}  // namespace b200
