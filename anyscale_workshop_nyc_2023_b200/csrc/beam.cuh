// Beam search on the decode rows (b200t5_generate_beam): transformers 5.5 GenerationMixin._beam_search with
// do_sample=False and one EOS id, restated in oracle/beam.py. Prompt b owns the k rows b*k .. b*k+k-1. Per step, after
// the lm_head has stored the act-rounded fp32 logits [rows, V] (EpiStoreF32):
//   beam_row_kernel     one CTA per row: lse, the min_new_tokens EOS mask, the top 2k of log_softmax
//   beam_select_kernel  one warp per prompt: top 2k of the k x 2k accumulated candidates, the next running beams,
//                       the finished set, the early-stop heuristic; next tokens, parents and decoder inputs
//   beam_reorder_kernel the self-attention cache rows follow their parents (in place)
// and once per call beam_output_kernel writes the returned hypotheses.
// Ties are broken as oracle/beam.py does: value descending, then index ascending (token within a row; beam * V + token
// across a prompt; list position in the running and finished selections).
#pragma once
#include "elementwise.cuh"

namespace b200 {

constexpr int kBeamMax = 16;             // num_beams <= 16
constexpr int kBeamCand = 2 * kBeamMax;  // candidate stride per row (2k <= 32: one warp holds a list)
constexpr int kBeamRowThreads = 256;
constexpr int kBeamReorderThreads = 128;
constexpr float kBeamNeg = -1.0e9f;      // transformers' penalty

// The values of a call, read from device memory so that the step graph does not depend on them.
struct BeamParams {
  int k;          // num_beams
  int T;          // max_new_tokens (max_length = T + 1)
  int min_new;    // EOS masked while step < min_new
  int eos;
  int early;      // early_stopping: 0 False, 1 True, 2 "never"
  int hyp_max;    // 1: the heuristic's best running score is scaled for length T (early "never", length_penalty > 0)
};

// One entry of a prompt's finished set: the hypothesis that ended at step t by taking token `tok` from running slot
// `par` (of that step), with log-probability lp and length-penalised score. t = -1: an empty placeholder.
struct BeamFin {
  float score;
  int t, par, tok;
  float lp;
  int flag;  // transformers' is_sent_finished
};

struct BeamDev {
  const BeamParams* prm;
  const float* len_scale;  // [T]: fp32(1 / (l ** length_penalty)) at index l - 1, the reciprocal taken in double
  const float* logits;     // [rows][V] act-rounded fp32 logits of this step
  float* lse;              // [rows] (test hook only, may be nullptr)
  float* cand_lp;          // [rows][kBeamCand] each row's top 2k by (log_prob + running score, token): log-probabilities
  int* cand_tok;           // [rows][kBeamCand] ... and tokens, best first
  float* run_score;        // [rows] running beam scores
  int* hist_par;           // [Tmax][rows]: running slot j of step s extended slot hist_par of that step ...
  int* hist_tok;           // ... with token hist_tok and log-probability hist_lp
  float* hist_lp;
  BeamFin* fin;            // [B][kBeamMax], sorted best first
  int* heur;               // [B] transformers' is_early_stop_heuristic_unsatisfied
  int* parent;             // [rows] the row whose cache row r takes before the next step
  int rows;
};

DEVINL bool beam_beats(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

// A warp-held list sorted best first: lane l < K holds entry l (value lv, key li, payload lp). Inserts (v, key, pay)
// when it beats entry K-1; the entries it beats form a suffix of the list, which moves down one lane.
DEVINL void beam_warp_insert(float& lv, int& li, int& lpay, float v, int key, int pay, int K) {
  const int lane = static_cast<int>(lane_id());
  const unsigned m = __ballot_sync(0xffffffffu, lane < K && beam_beats(v, key, lv, li));
  const float uv = __shfl_up_sync(0xffffffffu, lv, 1);
  const int ui = __shfl_up_sync(0xffffffffu, li, 1), up = __shfl_up_sync(0xffffffffu, lpay, 1);
  if (!m) return;
  const int pos = __ffs(m) - 1;
  if (lane > pos) {
    lv = uv;
    li = ui;
    lpay = up;
  } else if (lane == pos) {
    lv = v;
    li = key;
    lpay = pay;
  }
}

// Offers every lane's (v, key, pay) to the warp list (ok: the lane has an item).
DEVINL void beam_warp_offer(float& lv, int& li, int& lpay, float v, int key, int pay, bool ok, int K) {
  const float tv = __shfl_sync(0xffffffffu, lv, K - 1);
  const int ti = __shfl_sync(0xffffffffu, li, K - 1);
  unsigned q = __ballot_sync(0xffffffffu, ok && beam_beats(v, key, tv, ti));
  while (q) {
    const int src = __ffs(q) - 1;
    q &= q - 1;
    beam_warp_insert(lv, li, lpay, __shfl_sync(0xffffffffu, v, src), __shfl_sync(0xffffffffu, key, src),
                     __shfl_sync(0xffffffffu, pay, src), K);
  }
}

// One CTA per row. lse = M + log(S) with M the row maximum and S = sum exp(v - M), each reduced in an order that depends
// only on V and the block size (thread i takes columns i, i + 256, ... ascending, xor tree in the warp, warps in order),
// so a row's numbers do not depend on where it sits. log_probs = (v - M) - log(S) as torch's log_softmax, then the EOS
// column is -inf while step < min_new (after the lse: transformers' processor order). The row keeps its top 2k by
// (fl(log_prob + running score) desc, token asc): exactly the prompt-level order of beam_select_kernel restricted to
// the row, so the prompt's top 2k of all k x V candidates are always among the rows' lists, ties included.
__global__ void __launch_bounds__(kBeamRowThreads) beam_row_kernel(const BeamDev d, int V, const DecodeState* st,
                                                                   const int* __restrict__ unfinished) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  if (!unfinished[row]) return;
  const BeamParams prm = *d.prm;
  const int t = st->step, K = 2 * prm.k;
  const float* x = d.logits + static_cast<size_t>(row) * V;
  const int warp = threadIdx.x >> 5, lane = static_cast<int>(lane_id());
  constexpr int kWarps = kBeamRowThreads / 32;
  __shared__ float s_red[kWarps];
  __shared__ float s_v[kWarps][32];
  __shared__ int s_i[kWarps][32];
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += kBeamRowThreads) m = fmaxf(m, x[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = s_red[0];
  for (int w = 1; w < kWarps; ++w) m = fmaxf(m, s_red[w]);
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += kBeamRowThreads) s += expf(x[i] - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __syncthreads();
  if (lane == 0) s_red[warp] = s;
  __syncthreads();
  s = s_red[0];
  for (int w = 1; w < kWarps; ++w) s += s_red[w];
  const float ls = logf(s);
  if (d.lse != nullptr && threadIdx.x == 0) d.lse[row] = m + ls;
  const bool mask_eos = t < prm.min_new;
  const float rs = d.run_score[row];
  float lv = -INFINITY;  // accumulated score; the log-probability travels as the payload's bits
  int li = 0x7fffffff, lpay = 0;
  for (int base = warp * 32; base < V; base += kBeamRowThreads) {
    const int i = base + lane;
    float v = -INFINITY;
    if (i < V) v = (mask_eos && i == prm.eos) ? -INFINITY : (x[i] - m) - ls;
    beam_warp_offer(lv, li, lpay, v + rs, i, __float_as_int(v), i < V, K);
  }
  __shared__ int s_p[kWarps][32];
  s_v[warp][lane] = lv;
  s_i[warp][lane] = li;
  s_p[warp][lane] = lpay;
  __syncthreads();
  if (warp != 0) return;
  for (int w = 1; w < kWarps; ++w) beam_warp_offer(lv, li, lpay, s_v[w][lane], s_i[w][lane], s_p[w][lane], lane < K, K);
  if (lane < K) {
    d.cand_lp[static_cast<size_t>(row) * kBeamCand + lane] = __int_as_float(lpay);
    d.cand_tok[static_cast<size_t>(row) * kBeamCand + lane] = li;
  }
}

// One warp per prompt: steps c-g of _beam_search at step t (cur_len = t + 1, max_length = T + 1).
//  c. accumulated = log_prob + running score over the k rows' 2k candidates (the prompt's top 2k of all k x V lie among
//     them: beam_row_kernel ranks each row the same way), top 2k by (score, beam * V + token); a candidate hits the
//     stopping criteria on EOS or at t + 1 >= T
//  e. running beams: top k of score + hit * -1e9
//  f. finished set: top k of the old entries followed by the candidates, a candidate scored
//     score * len_scale[t] + (-1e9 unless it hit the criteria and is among the first k)
//  g. heuristic: best running score * len_scale (of t + 1, or T) > some (finished ? min finished score : -1e9)
// transformers also adds -1e9 to every candidate of a prompt whose heuristic has failed, or whose finished set is full
// with early_stopping=True: such a prompt can never change its finished set, so here it is retired instead - its rows
// stop (unfinished = 0, live_extent = 0) and no later kernel touches them.
// Row b*k + j then continues running slot j: parent[b*k + j], the token's embedding as its next decoder input.
__global__ void __launch_bounds__(32) beam_select_kernel(const BeamDev d, int V, DecodeState* st, int* __restrict__ unfinished,
                                                         int* __restrict__ live_extent, const act_t* __restrict__ E,
                                                         res_t* __restrict__ xdec, int dm) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const BeamParams prm = *d.prm;
  const int k = prm.k, K = 2 * k, r0 = b * k, t = st->step;
  if (!unfinished[r0]) return;
  const int lane = static_cast<int>(lane_id());
  __shared__ float s_acc[kBeamMax * kBeamCand];
  __shared__ BeamFin s_old[kBeamMax];
  __shared__ int s_next[kBeamMax];
  for (int e = lane; e < k * K; e += 32) {
    const int j = e / K, c = e % K;
    s_acc[e] = d.cand_lp[static_cast<size_t>(r0 + j) * kBeamCand + c] + d.run_score[r0 + j];
  }
  if (lane < k) s_old[lane] = d.fin[static_cast<size_t>(b) * kBeamMax + lane];
  __syncwarp();
  // c. the prompt's top 2k; key beam * V + token, payload the candidate's place e = j * K + c
  float lv = -INFINITY;
  int li = 0x7fffffff, le = 0;
  for (int base = 0; base < k * K; base += 32) {
    const int e = base + lane;
    const bool ok = e < k * K;
    const int j = ok ? e / K : 0;
    const int tok = ok ? d.cand_tok[static_cast<size_t>(r0 + j) * kBeamCand + e % K] : 0;
    beam_warp_offer(lv, li, le, ok ? s_acc[e] : -INFINITY, j * V + tok, e, ok, K);
  }
  const bool mine = lane < K;
  const int jc = le / K, tok = li - jc * V;
  const float lp = d.cand_lp[static_cast<size_t>(r0 + jc) * kBeamCand + le % K];
  const bool hit = tok == prm.eos || t + 1 >= prm.T;
  // e. running beams
  const float rval = hit ? lv + kBeamNeg : lv;
  int rank = 0;
  for (int l = 0; l < K; ++l) {
    const float o = __shfl_sync(0xffffffffu, rval, l);
    if (l != lane && beam_beats(o, l, rval, lane)) ++rank;
  }
  // f. finished set: old entries are 0..k-1, candidates k + c
  const bool did = hit && lane < k;
  float sc = lv * d.len_scale[t];
  sc = sc + (did ? 0.f : kBeamNeg);
  int frank = 0;
  for (int l = 0; l < K; ++l) {
    const float o = __shfl_sync(0xffffffffu, sc, l);
    if (mine && l != lane && beam_beats(o, k + l, sc, k + lane)) ++frank;
  }
  for (int o = 0; o < k; ++o)
    if (beam_beats(s_old[o].score, o, sc, k + lane)) ++frank;
  int orank = 0;  // rank of old entry `lane`
  if (lane < k) {
    for (int o = 0; o < k; ++o)
      if (o != lane && beam_beats(s_old[o].score, o, s_old[lane].score, lane)) ++orank;
  }
  for (int l = 0; l < K; ++l) {
    const float o = __shfl_sync(0xffffffffu, sc, l);
    if (lane < k && beam_beats(o, k + l, s_old[lane].score, lane)) ++orank;
  }
  BeamFin* fin = d.fin + static_cast<size_t>(b) * kBeamMax;
  if (lane < k && orank < k) fin[orank] = s_old[lane];
  if (mine && frank < k) fin[frank] = BeamFin{sc, t, jc, tok, lp, did ? 1 : 0};
  if (mine && rank < k) {
    const size_t h = static_cast<size_t>(t) * d.rows + r0 + rank;
    d.run_score[r0 + rank] = rval;
    d.hist_par[h] = jc;
    d.hist_tok[h] = tok;
    d.hist_lp[h] = lp;
    d.parent[r0 + rank] = r0 + jc;
    s_next[rank] = tok;
  }
  __syncwarp();
  // g. early-stop heuristic on the updated sets (read back what this warp just wrote)
  const float best = __shfl_sync(0xffffffffu, rval, __ffs(__ballot_sync(0xffffffffu, mine && rank == 0)) - 1);
  const float bs = best * (prm.hyp_max ? d.len_scale[prm.T - 1] : d.len_scale[t]);
  const BeamFin f = lane < k ? fin[lane] : BeamFin{0.f, 0, 0, 0, 0.f, 1};
  float mn = lane < k ? f.score : INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  const bool improve = __any_sync(0xffffffffu, lane < k && bs > (f.flag ? mn : kBeamNeg));
  const bool all_fin = __all_sync(0xffffffffu, f.flag != 0);
  const int heur = d.heur[b] && improve;
  if (lane == 0) d.heur[b] = heur;
  if (!heur || (prm.early == 1 && all_fin)) {
    if (lane < k) {
      unfinished[r0 + lane] = 0;
      if (live_extent != nullptr) live_extent[r0 + lane] = 0;
    }
    if (lane == 0) atomicAdd(&st->finished_rows, k);
    return;
  }
  if (E == nullptr) return;
  for (int j = 0; j < k; ++j) {
    const uint4* src = reinterpret_cast<const uint4*>(E + static_cast<size_t>(s_next[j]) * dm);
    res_t* dst = xdec + static_cast<size_t>(r0 + j) * dm;
    for (int i = lane; i < dm / 8; i += 32) store_res8_from_act(dst + i * 8, src[i]);
  }
}

// The self-attention cache [n_planes = Ld * 2][rows][H][Tmax][64] follows the beams: row r takes positions 0..t of row
// parent[r], within each prompt. CTA (plane * H + head, prompt); each thread owns one 16-byte chunk of one position at
// a time: it loads that chunk from every row some other row takes it from, then stores it to every row whose parent is
// another row. Rows that keep their own lineage are neither read nor written, so the permutation is done in place.
// `moved` (may be nullptr): bytes read and written, accumulated.
__global__ void __launch_bounds__(kBeamReorderThreads) beam_reorder_kernel(act_t* __restrict__ self_kv, const BeamDev d,
                                                                           const int* __restrict__ unfinished,
                                                                           const DecodeState* st, int H, int Tmax,
                                                                           unsigned long long* moved) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const int k = d.prm->k, r0 = b * k;
  if (!unfinished[r0]) return;
  __shared__ int s_par[kBeamMax];
  __shared__ int s_src[kBeamMax];
  __shared__ uint4 s_buf[kBeamMax][kBeamReorderThreads];
  if (threadIdx.x < k) s_par[threadIdx.x] = d.parent[r0 + threadIdx.x] - r0;
  __syncthreads();
  int n_dst = 0, n_src = 0;
  for (int j = 0; j < k; ++j) {
    if (s_par[j] != j) ++n_dst;
    bool src = false;
    for (int i = 0; i < k; ++i) src = src || (s_par[i] == j && i != j);
    if (threadIdx.x == 0) s_src[j] = src;
    n_src += src;
  }
  if (n_dst == 0) return;
  __syncthreads();
  const int plane = blockIdx.x / H, head = blockIdx.x % H;
  const int t = st->step;
  const size_t row_stride = static_cast<size_t>(H) * Tmax * 8;  // uint4 per row
  uint4* base = reinterpret_cast<uint4*>(self_kv) + (static_cast<size_t>(plane) * d.rows + r0) * row_stride +
                static_cast<size_t>(head) * Tmax * 8;
  const int n = (t + 1) * 8;
  for (int q = threadIdx.x; q < n; q += kBeamReorderThreads) {
    for (int j = 0; j < k; ++j)
      if (s_src[j]) s_buf[j][threadIdx.x] = base[j * row_stride + q];
    for (int j = 0; j < k; ++j)
      if (s_par[j] != j) base[j * row_stride + q] = s_buf[s_par[j]][threadIdx.x];
  }
  if (moved != nullptr && threadIdx.x == 0) atomicAdd(moved, static_cast<unsigned long long>(n_src + n_dst) * n * 16);
}

// Once per call: prompt b's k rows copy the cross-attention K/V, extent and key_ok of its row b*k (the only one the
// encoder ran on). CTA (plane * H + head, row).
__global__ void beam_replicate_kernel(act_t* __restrict__ cross_kv, int* __restrict__ extent, unsigned char* __restrict__ key_ok,
                                      int rows, int k, int H, int S) {
  const int r = blockIdx.y, j = r % k;
  if (j == 0) return;
  const int src = r - j;
  const int ext = extent[src];
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < S; i += blockDim.x) key_ok[static_cast<size_t>(r) * S + i] = key_ok[static_cast<size_t>(src) * S + i];
    if (threadIdx.x == 0) extent[r] = ext;
  }
  const int plane = blockIdx.x / H, head = blockIdx.x % H;
  const size_t row_stride = static_cast<size_t>(H) * S * 8;
  const uint4* from = reinterpret_cast<const uint4*>(cross_kv) + (static_cast<size_t>(plane) * rows + src) * row_stride + static_cast<size_t>(head) * S * 8;
  uint4* to = reinterpret_cast<uint4*>(cross_kv) + (static_cast<size_t>(plane) * rows + r) * row_stride + static_cast<size_t>(head) * S * 8;
  for (int i = threadIdx.x; i < ext * 8; i += blockDim.x) to[i] = from[i];
}

// Start of a beam call: running scores 0 for beam 0 and -1e9 for the others, empty finished sets, heuristic open.
__global__ void beam_init_kernel(const BeamDev d, int B, int k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * k) d.run_score[i] = i % k == 0 ? 0.f : kBeamNeg;
  if (i < B * kBeamMax) d.fin[i] = BeamFin{kBeamNeg, -1, 0, 0, 0.f, 0};
  if (i < B) d.heur[i] = 1;
}

// Once per call, one thread per returned hypothesis r = b * n + i (the i-th best finished entry of prompt b), walking
// its lineage back through the step history. seq [rows_out][T + 1]: start token, the hypothesis, pad; bidx and lp
// [rows_out][T] (may be nullptr): transformers' beam_indices (b * k + slot, -1 after the end) and the chosen tokens'
// log-probabilities (0 after the end); len [rows_out] = generated tokens; score (may be nullptr) = sequences_scores.
__global__ void beam_output_kernel(const BeamDev d, int B, int n, long long* __restrict__ seq, int* __restrict__ len,
                                   float* __restrict__ score, long long* __restrict__ bidx, float* __restrict__ lp,
                                   long long start, long long pad) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B * n) return;
  const int k = d.prm->k, T = d.prm->T, b = r / n;
  const BeamFin f = d.fin[static_cast<size_t>(b) * kBeamMax + r % n];
  const int L = f.t + 1;
  long long* sr = seq + static_cast<size_t>(r) * (T + 1);
  sr[0] = start;
  for (int s = L + 1; s <= T; ++s) sr[s] = pad;
  if (bidx != nullptr)
    for (int s = L; s < T; ++s) bidx[static_cast<size_t>(r) * T + s] = -1;
  if (lp != nullptr)
    for (int s = L; s < T; ++s) lp[static_cast<size_t>(r) * T + s] = 0.f;
  len[r] = L;
  if (score != nullptr) score[r] = f.score;
  int tok = f.tok, par = f.par;
  float l = f.lp;
  for (int s = L - 1; s >= 0; --s) {
    sr[s + 1] = tok;
    if (bidx != nullptr) bidx[static_cast<size_t>(r) * T + s] = b * k + par;
    if (lp != nullptr) lp[static_cast<size_t>(r) * T + s] = l;
    if (s > 0) {
      const size_t h = static_cast<size_t>(s - 1) * d.rows + b * k + par;
      tok = d.hist_tok[h];
      l = d.hist_lp[h];
      par = d.hist_par[h];
    }
  }
}

}  // namespace b200
