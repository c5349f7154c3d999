// Greedy-mode logits processors on the device (transformers generation/logits_process.py, the greedy subset of
// GenerationMixin._get_logits_processor): encoder / decoder repetition penalties, decoder / encoder n-gram bans,
// bad-word sequences, several EOS ids, suppressed and begin-suppressed tokens.
//
// Everything a step needs lives in device memory, so the captured step graphs replay unchanged from call to call:
//   - ProcCfg: the values of this call (penalty multipliers, n-gram sizes, EOS ids);
//   - per row, V-bit bitmaps: `seen` (decoder ids so far, start token included), `enc` (the prompt's ids, padding
//     included) and `banned` (n-gram and multi-token bad-word bans of the NEXT step);
//   - shared by all rows: three V-bit masks `stat` = {suppress_tokens + one-token bad words, begin_suppress_tokens,
//     EOS ids};
//   - per row, the list of the tokens set in `banned` (so that the next update clears exactly those bits instead
//     of the whole bitmap) and the prompt's ids as int32.
// The fused lm_head epilogue (gemm.cuh: EpiLmHead<true, *>) applies them per 128-column tile; proc_new_bans runs at the
// end of finalize_step_kernel<true, *>, one CTA per row, once the row's token is known.
#pragma once
#include "ptx.cuh"

namespace b200 {

constexpr int kProcMaxEos = 16;

struct ProcCfg {
  // s < 0 ? s * neg : s * pos, with neg = fp32(p) and pos = fp32(1 / p), the reciprocal taken in double: torch's CUDA
  // `s * p` and `s / p` for a Python float p (the division by a CPU scalar is a multiplication by the reciprocal;
  // tests/test_logits_process_gpu.py pins the rounding). For the encoder penalty p = 1 / encoder_repetition_penalty,
  // as transformers stores it.
  float enc_neg, enc_pos, rep_neg, rep_pos;
  int enc_pen, rep_pen;  // 0 | 1
  int ngram, enc_ngram;  // 0 = off
  int n_bad;             // bad-word sequences of two or more tokens
  int bad_add;           // NoBadWordsLogitsProcessor is active: scores + bias turns -0.0 into +0.0 everywhere
  int n_eos;
  int eos[kProcMaxEos];
  int begin_t;  // the first generated position, where begin_suppress_tokens apply: 0, or P - 1 after a decoder prompt of P ids
};

struct ProcDev {
  const ProcCfg* cfg = nullptr;
  uint32_t* seen = nullptr;    // [B][W]
  uint32_t* enc = nullptr;     // [B][W]
  uint32_t* banned = nullptr;  // [B][W]
  const uint32_t* stat = nullptr;  // [3][W]
  int* ban_list = nullptr;     // [B][ban_cap]
  int* ban_cnt = nullptr;      // [B]
  int* enc_ids = nullptr;      // [B][S]
  const int* bad_ids = nullptr;  // multi-token bad words: sequence i = bad_ids[bad_off[i] .. bad_off[i+1])
  const int* bad_off = nullptr;
  int ban_cap = 0, S = 0, W = 0;
  int row0 = 0;  // first plan row of the launch (decode chains see row-offset views)
};

DEVINL void bit_set(uint32_t* words, int tok) { atomicOr(words + (tok >> 5), 1u << (tok & 31)); }

DEVINL bool proc_is_eos(const ProcCfg& c, long long tok) {
  for (int i = 0; i < c.n_eos; ++i)
    if (tok == c.eos[i]) return true;
  return false;
}

// Bans of the next step of row r, whose decoder ids so far are hist[0 .. L) (start token first); every thread of the
// CTA calls it. `clear`: unset the bits the previous update set first. Cost per row and step: the previous list's
// words, O(L n) for the decoder n-grams, O(S n) for the encoder n-grams, the bad words' total length.
//   no_repeat_ngram_size n:          hist[j .. j+n-1) == hist[L-n+1 .. L)  bans hist[j+n-1]   (nothing while L + 1 < n)
//   encoder_no_repeat_ngram_size n:  enc[j .. j+n-1)  == hist[L-n+1 .. L)  bans enc[j+n-1]    (nothing while L < n - 1)
//   bad word w of length k >= 2:     w[0 .. k-1)      == hist[L-k+1 .. L)  bans w[k-1]        (nothing while L < k)
DEVINL void proc_new_bans(const ProcDev& pd, int r, const long long* __restrict__ hist, int L, bool clear) {
  __shared__ int s_cnt;
  const ProcCfg& c = *pd.cfg;
  uint32_t* ban = pd.banned + static_cast<size_t>(r) * pd.W;
  int* list = pd.ban_list + static_cast<size_t>(r) * pd.ban_cap;
  if (clear) {
    const int old = pd.ban_cnt[r];
    for (int i = threadIdx.x; i < old; i += blockDim.x) ban[list[i] >> 5] = 0;  // every set bit is on the list
  }
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  auto add = [&](int tok) {
    const uint32_t bit = 1u << (tok & 31);
    if (!(atomicOr(ban + (tok >> 5), bit) & bit)) {
      const int k = atomicAdd(&s_cnt, 1);
      if (k < pd.ban_cap) list[k] = tok;
    }
  };
  const int n = c.ngram;
  if (n > 0) {
    for (int j = threadIdx.x; j <= L - n; j += blockDim.x) {
      bool eq = true;
      for (int k = 0; k < n - 1 && eq; ++k) eq = hist[j + k] == hist[L - n + 1 + k];
      if (eq) add(static_cast<int>(hist[j + n - 1]));
    }
  }
  const int e = c.enc_ngram;
  if (e > 0 && L >= e - 1) {
    const int* enc = pd.enc_ids + static_cast<size_t>(r) * pd.S;
    for (int j = threadIdx.x; j <= pd.S - e; j += blockDim.x) {
      bool eq = true;
      for (int k = 0; k < e - 1 && eq; ++k) eq = enc[j + k] == hist[L - e + 1 + k];
      if (eq) add(enc[j + e - 1]);
    }
  }
  for (int i = threadIdx.x; i < c.n_bad; i += blockDim.x) {
    const int lo = pd.bad_off[i], k = pd.bad_off[i + 1] - lo;
    if (k > L) continue;
    bool eq = true;
    for (int q = 0; q < k - 1 && eq; ++q) eq = pd.bad_ids[lo + q] == hist[L - k + 1 + q];
    if (eq) add(pd.bad_ids[lo + k - 1]);
  }
  __syncthreads();
  if (threadIdx.x == 0) pd.ban_cnt[r] = s_cnt < pd.ban_cap ? s_cnt : pd.ban_cap;
}

// Start of a row (static batch: every row after decode_init_kernel; slot pool: every admitted slot after
// admit_slots_kernel): clear its bitmaps, keep its prompt ids, mark the prompt's tokens and the L decoder ids of
// hist (the start token, or a call's decoder prompt; the test hook passes a longer history) and compute the bans of
// its first step.
// Row r = slots[blockIdx.x] (slots == nullptr: blockIdx.x); its history is row out_row[r] (nullptr: r) of hist_base.
__global__ void proc_reset_kernel(ProcDev pd, const int* __restrict__ slots, const long long* __restrict__ ids,
                                  const long long* __restrict__ hist_base, int hist_ld, const int* __restrict__ out_row,
                                  int L) {
  const int r = slots != nullptr ? slots[blockIdx.x] : static_cast<int>(blockIdx.x);
  const ProcCfg& c = *pd.cfg;
  uint32_t* seen = pd.seen + static_cast<size_t>(r) * pd.W;
  uint32_t* enc = pd.enc + static_cast<size_t>(r) * pd.W;
  uint32_t* ban = pd.banned + static_cast<size_t>(r) * pd.W;
  for (int i = threadIdx.x; i < pd.W; i += blockDim.x) {
    seen[i] = 0;
    enc[i] = 0;
    ban[i] = 0;
  }
  int* eids = pd.enc_ids + static_cast<size_t>(r) * pd.S;
  for (int j = threadIdx.x; j < pd.S; j += blockDim.x) eids[j] = static_cast<int>(ids[static_cast<size_t>(r) * pd.S + j]);
  __syncthreads();
  const long long* hist = hist_base + static_cast<size_t>(out_row != nullptr ? out_row[r] : r) * hist_ld;
  if (c.enc_pen)
    for (int j = threadIdx.x; j < pd.S; j += blockDim.x) bit_set(enc, eids[j]);
  if (c.rep_pen)
    for (int j = threadIdx.x; j < L; j += blockDim.x) bit_set(seen, static_cast<int>(hist[j]));
  __syncthreads();
  proc_new_bans(pd, r, hist, L, false);
}

}  // namespace b200
