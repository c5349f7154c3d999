// Cross-attention of the decode step (D7) as a TMA stream feeding the (legacy) tensor cores: the HBM roofline
// kernel, second design.
//
// attention_decode.cuh reads K/V with per-thread 16-byte loads and does the arithmetic on the CUDA cores: ~54 warp
// instructions per 512 bytes, i.e. ~60 % of an SM's issue slots at the HBM rate, and its bandwidth is proportional to
// the warps resident per SM. That is fine when it has the GPU to itself, but the decode step overlaps it with the
// latency-bound split-K GEMMs of the other row-chain, whose CTAs (44 K registers, up to ~165 KB of shared memory
// each) cannot co-reside with a full complement of attention CTAs and take their place.
//
// Here neither the bytes in flight nor the arithmetic depend on how many warps are resident:
//   * one producer lane per CTA streams the K and V slabs of the CTA's (row, head) items through a ring of 8 KB
//     shared-memory stages with TMA (cp.async.bulk.tensor.2d, 64 keys x 64 d per box, 128-byte swizzle, L2
//     evict-first; the chunk's 64 key_ok bytes ride along as a second bulk copy on the same mbarrier);
//   * four consumer warps compute out of shared memory with mma.sync.m16n8k16 (bf16 / fp16 inputs, fp32
//     accumulation): scores = K_chunk[64 x 64] . q as four 16-key tiles (one per warp), out = V_chunk^T[64 d x 64] . p
//     as four 16-d tiles (one per warp, accumulated over the whole item in registers), the vectors q and p occupying
//     column 0 of the B operand. ~25 warp instructions per 8 KB chunk and warp instead of ~220.
//     The tensor pipe runs at 1/8 utilisation by construction - irrelevant for a kernel that is bound by HBM; what
//     matters is that the issue slots are free (the CUDA-core arithmetic of attention_decode.cuh on the same ring is
//     issue-bound).
// Two CTAs per SM x `stages` x 8 KB are in flight whatever else is resident, the CTAs are persistent (grid sized so
// that every CTA gets the same number of items), and their footprint (2 x ~45 KB, 2 x 160 threads) leaves room for
// a split-K GEMM CTA of the other chain on the same SM.
//
// Rounding contract (SURVEY Appendix A.3) as in attention_decode.cuh: s = act(q.k) with fp32 accumulation; masked
// keys replaced by finfo.min; p = act(exp(s - max) / sum) from an exact two-pass fp32 softmax over the rounded scores;
// out = act(sum_j p_j v_j) with fp32 accumulation. Only the ORDER of the fp32 accumulations differs (the tensor core's
// instead of a sequential one), which no contract fixes: HF's own bmm does not either.
#pragma once
#include "attention_decode.cuh"

namespace b200 {

constexpr int kXsConsumerWarps = 4;
constexpr int kXsThreads = (kXsConsumerWarps + 1) * 32;  // + the producer warp
constexpr int kXsChunkKeys = 64;                         // 8 KB of K or V rows per ring stage
constexpr int kXsChunkBytes = kXsChunkKeys * 128;
constexpr int kXsMaxStages = 12;

struct XsSmem {
  // [stages][8 KB] ring (1024-byte aligned: swizzle atoms) | masks [stages][64] | scores f32 [Tk64] | p act [Tk64] |
  // stat [8] | q act [64] | full[stages] empty[stages]
  static __host__ __device__ int tk64(int Tk) { return (Tk + 63) & ~63; }
  static __host__ __device__ size_t bytes(int stages, int Tk) {
    return static_cast<size_t>(stages) * (kXsChunkBytes + 64) + static_cast<size_t>(tk64(Tk)) * 6 + 8 * 4 + 64 * 2 +
           2 * kXsMaxStages * 8 + 1024 /* alignment slack */;
  }
};

DEVINL void xs_bar_sync() { asm volatile("bar.sync 1, %0;" ::"r"(kXsConsumerWarps * 32) : "memory"); }  // the consumer warps only

// 2-D tiled TMA load with an L2 cache hint
DEVINL void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
DEVINL void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
DEVINL void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D (16x8 fp32) += A (16x16, row) * B (16x8, col), 2-byte inputs of the build's activation type
DEVINL void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
#if B200T5_F16
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
#else
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
#endif
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Release of a ring slot. The arrive is PREDICATED ON THE ACCUMULATOR of the last mma that consumed the slot: mma.sync
// has no memory semantics, so without a data dependency ptxas is free to schedule the arrive between the last
// ldmatrix and the mma that waits for it (it did: LDSM, SYNCS.ARRIVE, HMMA) - the slot is then handed back while the
// shared-memory read may still sit in the SM's memory queue, and with a GEMM CTA hammering shared memory on the same
// SM the refill occasionally won (run-to-run different tokens). The
// compare is never false (an mma produces the canonical NaN only), but ptxas cannot know that.
DEVINL void xs_release_slot(uint64_t* bar, float last_acc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %1, 0x7fc12345;\n"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n"
      "}"
      ::"r"(smem_u32(bar)), "r"(__float_as_uint(last_acc))
      : "memory");
}

// tmK / tmV: [rows, 64] views (box 64 x 64 rows, 128-byte swizzle) of the K and V planes; item `it` (= (row, head),
// chain-relative) owns rows k_row0 + it * Tk .. + Tk of tmK and v_row0 + it * Tk .. of tmV.
// <= 64 registers: two of these CTAs (20 K registers) and one split-K GEMM CTA (288 x 152, gemm_splitk.cuh) share an SM's 64 K
__global__ void __maxnreg__(64)
attn_cross_stream_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                         int k_row0, int v_row0,
                         const act_t* __restrict__ q,    // [B, H*64]
                         act_t* __restrict__ ctx,        // [B, H*64]
                         int n_items,                    // B * H
                         int H, int Tk,
                         const int* __restrict__ extent,            // [B] keys to visit (0 = retired row)
                         const unsigned char* __restrict__ key_ok,  // [B][Tk] 1 = attended
                         int stages, XsStamps stamps) {
  extern __shared__ uint8_t xs_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(xs_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_mask = ring + static_cast<size_t>(stages) * kXsChunkBytes;          // [stages][64]
  float* s_scores = reinterpret_cast<float*>(s_mask + static_cast<size_t>(stages) * 64);
  const int tk64 = XsSmem::tk64(Tk);
  act_t* s_p = reinterpret_cast<act_t*>(s_scores + tk64);                        // [tk64]
  float* s_stat = reinterpret_cast<float*>(s_p + tk64);                          // [8]
  act_t* s_q = reinterpret_cast<act_t*>(s_stat + 8);                             // [64]
  uint64_t* full = reinterpret_cast<uint64_t*>(s_q + 64);
  uint64_t* empty = full + kXsMaxStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kXsConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();
  // The dependent kernel (this chain's cross-attention output projection) is released when this CTA starts its LAST
  // item, not at once as everywhere else in the step: its CTAs would only sit on their SMs (~140 KB of shared memory
  // each) while this kernel streams, in the way of the OTHER chain's GEMMs, so its prologue overlaps the tail of the
  // stream only.
  // Everything above overlapped the previous kernel's tail; q / extent are that kernel's (or the previous step's) output
  pdl_wait();
  unsigned long long t_start = 0;
  if (stamps.slots != nullptr && threadIdx.x == 0) t_start = global_timer_ns();
  const int first = blockIdx.x, stride = gridDim.x;
  const int last_item = first + ((n_items - 1 - first) / stride) * stride;
  // The key_ok bytes of a K chunk travel with it (a second, 64-byte bulk copy on the same barrier) when the rows
  // are 16-byte aligned; otherwise the consumers read them from global memory.
  const bool mask_bulk = (Tk & 15) == 0;

  if (warp == kXsConsumerWarps) {
    // ------------------------------------------------------------ producer: K chunks then V chunks of every item
    if (lane == 0) {
      const uint64_t policy = l2_policy_evict_first();
      int stage = 0;
      uint32_t phase = 0;
      int n_next = first < n_items ? extent[first / H] : 0;
      for (int it = first; it < n_items; it += stride) {
        const int b = it / H;
        const int n = n_next;
        // (the next item's extent is fetched a whole item ahead: the ring holds < 2 us of stream, an L2 round trip
        // under load is of that order)
        if (it + stride < n_items) n_next = extent[(it + stride) / H];
#pragma unroll 1
        for (int kv = 0; kv < 2; ++kv) {
          const CUtensorMap* tm = kv ? &tmV : &tmK;
          const int row0 = (kv ? v_row0 : k_row0) + it * Tk;
          for (int k0 = 0; k0 < n; k0 += kXsChunkKeys) {
            const int keys = n - k0 < kXsChunkKeys ? n - k0 : kXsChunkKeys;
            const uint32_t mbytes = (kv == 0 && mask_bulk) ? static_cast<uint32_t>((keys + 15) & ~15) : 0u;
            mbar_wait(&empty[stage], phase ^ 1u);
            // a box is always 64 rows: rows beyond this item's keys belong to the next item / slab (finite values,
            // multiplied by p = 0) or lie beyond the tensor (zero fill)
            mbar_arrive_expect_tx(&full[stage], static_cast<uint32_t>(kXsChunkBytes) + mbytes);
            tma_load_2d_hint(ring + static_cast<size_t>(stage) * kXsChunkBytes, tm, &full[stage], 0, row0 + k0, policy);
            if (mbytes) bulk_load_1d(s_mask + stage * 64, key_ok + static_cast<size_t>(b) * Tk + k0, mbytes, &full[stage]);
            if (++stage == stages) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
    }
    return;  // (the copies complete on barriers the consumer warps wait on: the CTA outlives them)
  }

  // -------------------------------------------------------------- consumers
  const int gid = lane >> 2, tig = lane & 3;  // mma fragment coordinates: group (row) and thread in group
  const int tid = threadIdx.x;                // 0..127
  int stage = 0;
  uint32_t phase = 0;
  // ldmatrix row / 16-byte-unit provided by this lane (128-byte swizzle: physical unit = unit ^ (row & 7))
  //   Q K^T (A = K rows, not transposed): matrices (keys 0-7, d 0-7), (keys 8-15, d 0-7), (keys 0-7, d 8-15), (keys 8-15, d 8-15)
  const int a_row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;  // key row of this warp's 16-key tile
  const int a_unit = lane >> 4;                                      // + 2 * kstep
  //   P V (A = V^T, transposed load): matrices (keys 0-7, d 0-7), (keys 0-7, d 8-15), (keys 8-15, d 0-7), (keys 8-15, d 8-15)
  const int v_row = (lane & 7) + ((lane >> 4) & 1) * 8;              // + 16 * kstep (keys)
  const int v_unit = warp * 2 + ((lane >> 3) & 1);                   // this warp's 16-d tile
  // software pipeline over items: the next item's query is fetched while this one streams
  uint32_t q_next = 0;
  int nn = 0;
  auto fetch_q = [&](int it) -> uint32_t {  // 64 act_t = 32 words: one per lane of warp 0
    return warp == 0 ? reinterpret_cast<const uint32_t*>(q + static_cast<size_t>(it) * 64)[lane] : 0u;
  };
  if (first < n_items) {
    q_next = fetch_q(first);
    nn = extent[first / H];
  }
  for (int it = first; it < n_items; it += stride) {
    const int b = it / H;
    const int nkeys = nn;
    if (warp == 0) reinterpret_cast<uint32_t*>(s_q)[lane] = q_next;
    const int nxt = it + stride;
    if (nxt < n_items) {
      q_next = fetch_q(nxt);
      nn = extent[nxt / H];
    }
    if (it == last_item) pdl_launch_dependents();
    xs_bar_sync();  // s_q visible (and the previous item's s_p / s_scores no longer read)
    // B operand of Q K^T: q in column 0, i.e. in the lanes of group 0
    uint32_t qb[8];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      qb[2 * ks] = gid == 0 ? reinterpret_cast<const uint32_t*>(s_q)[ks * 8 + tig] : 0u;
      qb[2 * ks + 1] = gid == 0 ? reinterpret_cast<const uint32_t*>(s_q)[ks * 8 + 4 + tig] : 0u;
    }
    const unsigned char* ok_row = key_ok + static_cast<size_t>(b) * Tk;

    // ---------------- phase 1: scores of this warp's 16 keys of every 64-key chunk
    for (int k0 = 0; k0 < nkeys; k0 += kXsChunkKeys) {
      mbar_wait(&full[stage], phase);
      const uint32_t base = smem_u32(ring + static_cast<size_t>(stage) * kXsChunkBytes) + a_row * 128;
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t a[4];
        ldmatrix_x4(a, base + (((2 * ks + a_unit) ^ (a_row & 7)) << 4));
        mma_16816(acc, a, qb[2 * ks], qb[2 * ks + 1]);
      }
      if (tig == 0) {  // column 0: rows gid (acc[0]) and gid + 8 (acc[2]) of the tile
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int jl = warp * 16 + gid + 8 * hh;
          const int j = k0 + jl;
          if (j < nkeys) {
            const bool ok = mask_bulk ? s_mask[stage * 64 + jl] != 0 : ok_row[j] != 0;
            s_scores[j] = ok ? act_round(acc[2 * hh]) : kActMin;
          }
        }
      }
      __syncwarp();
      if (lane == 0) xs_release_slot(&empty[stage], acc[0]);
      if (++stage == stages) {
        stage = 0;
        phase ^= 1u;
      }
    }
    xs_bar_sync();

    // ---------------- softmax statistics over the rounded scores (fp32, exact two-pass)
    float mx = -INFINITY;
    for (int j = tid; j < nkeys; j += kXsConsumerWarps * 32) mx = fmaxf(mx, s_scores[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_stat[warp] = mx;
    xs_bar_sync();
    mx = fmaxf(fmaxf(s_stat[0], s_stat[1]), fmaxf(s_stat[2], s_stat[3]));
    float sum = 0.f;
    for (int j = tid; j < nkeys; j += kXsConsumerWarps * 32) {
      const float e = expf(s_scores[j] - mx);
      s_scores[j] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) s_stat[4 + warp] = sum;
    xs_bar_sync();
    sum = (s_stat[4] + s_stat[5]) + (s_stat[6] + s_stat[7]);
    // p in the activation type; zero beyond the row's keys up to the end of the last chunk (the V rows there
    // belong to somebody else)
    const int nk64 = (nkeys + kXsChunkKeys - 1) & ~(kXsChunkKeys - 1);
    for (int j = tid; j < nk64; j += kXsConsumerWarps * 32) s_p[j] = float2act(j < nkeys ? s_scores[j] / sum : 0.f);
    xs_bar_sync();

    // ---------------- phase 2: out[d] = sum_j p_j V[j][d] for this warp's 16 values of d
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 < nkeys; k0 += kXsChunkKeys) {
      mbar_wait(&full[stage], phase);
      const uint32_t base = smem_u32(ring + static_cast<size_t>(stage) * kXsChunkBytes);
      const uint32_t* pw = reinterpret_cast<const uint32_t*>(s_p + k0);  // pairs of p
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t a[4];
        const int row = ks * 16 + v_row;
        ldmatrix_x4_trans(a, base + row * 128 + ((v_unit ^ (row & 7)) << 4));
        const uint32_t b0 = gid == 0 ? pw[ks * 8 + tig] : 0u;
        const uint32_t b1 = gid == 0 ? pw[ks * 8 + 4 + tig] : 0u;
        mma_16816(o, a, b0, b1);
      }
      __syncwarp();
      if (lane == 0) xs_release_slot(&empty[stage], o[0]);
      if (++stage == stages) {
        stage = 0;
        phase ^= 1u;
      }
    }
    if (tig == 0) {
      act_t* dst = ctx + static_cast<size_t>(it) * 64 + warp * 16 + gid;
      dst[0] = float2act(o[0]);
      dst[8] = float2act(o[2]);
    }
  }
  if (first >= n_items) pdl_launch_dependents();  // no item
  if (stamps.slots != nullptr && threadIdx.x == 0) {
    atomicMin(&stamps.slots[2 * stamps.slot], t_start);
    atomicMax(&stamps.slots[2 * stamps.slot + 1], static_cast<unsigned long long>(global_timer_ns()));
  }
}

// grid: every CTA gets the same number of items (rounds = ceil(items / (2 * SMs)), CTAs = ceil(items / rounds))
inline int xs_grid(int n_items, int num_sms) {
  const int max_cta = 2 * num_sms;
  if (n_items <= max_cta) return n_items;
  const int rounds = (n_items + max_cta - 1) / max_cta;
  return (n_items + rounds - 1) / rounds;
}

}  // namespace b200
