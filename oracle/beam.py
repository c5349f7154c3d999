"""Beam search in numpy: transformers 5.5 `GenerationMixin._beam_search` (generation/utils.py:3076-3410 and its helpers
_get_top_k_continuations, _get_running_beams_for_next_iteration, _update_finished_beams, _check_early_stop_heuristic,
_beam_search_has_unfinished_sequences) with do_sample=False and one EOS id, driving T5Oracle's decode step. What the
CUDA beam step (csrc/beam.cuh) must reproduce. TEST INFRASTRUCTURE, like the rest of this package.

Ties: torch.topk documents no order for equal values. Here, as in the CUDA kernels, candidates are ranked by value
descending, then by index ascending (flat index beam * V + token across a prompt, position in the list otherwise).

Besides the results, `beam_search` returns per prompt the smallest decision gap of its live steps: between consecutive
running picks and the first candidate left out (the set and the slots), between a candidate that hits the stopping
criteria and its neighbour across the first-k boundary, and between consecutive finished entries and the best one left
out. A prompt whose gap is tiny can legitimately come out differently under other rounding.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from oracle.scores import log_softmax

NEG = np.float32(-1.0e9)
_REAL = -5.0e8  # values below this carry a -1e9 penalty


def order(vals: np.ndarray) -> np.ndarray:
    """Indices of `vals` by value descending, then index ascending."""
    vals = np.asarray(vals, dtype=np.float32)
    return np.lexsort((np.arange(vals.size), -vals))


def length_scale(x, length: int, length_penalty: float, division: str = "reciprocal"):
    """x / (length ** length_penalty) on fp32 values: torch on CUDA multiplies by fp32(1 / p) with the reciprocal
    taken in double ("reciprocal", what libb200t5 does); torch on the CPU divides by fp32(p) ("true")."""
    p = float(length) ** float(length_penalty)
    x = np.asarray(x, dtype=np.float32)
    return (x * np.float32(1.0 / p) if division == "reciprocal" else x / np.float32(p)).astype(np.float32)


def fma32(a, b, c) -> np.ndarray:
    """fl(a * b + c) of fp32 values with one rounding, as a fused multiply-add computes it. The product is exact in
    double; TwoSum gives the error of the double sum, which decides the fp32 rounding only when that sum lies halfway
    between two fp32 values."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c)))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        z = s - p
        e = (p - (s - z)) + (c - z)
        r = s.astype(np.float32)
        other = np.nextafter(r, np.where(s > r, np.float32(np.inf), np.float32(-np.inf)))
        tie = np.isfinite(s) & (s != r) & (np.abs(s - r) == np.abs(other.astype(np.float64) - s)) & (e != 0)
        up = np.maximum(r, other)
        down = np.minimum(r, other)
    return np.where(tie, np.where(e > 0, up, down), r).astype(np.float32)


class BeamState:
    """Per-prompt state of `_beam_search` for B prompts of k beams and at most T new tokens."""

    def __init__(self, B: int, k: int, T: int, start: int, pad: int):
        self.B, self.k, self.T = B, k, T
        self.run_score = np.zeros((B, k), np.float32)
        self.run_score[:, 1:] = NEG
        self.run_seq = np.full((B, k, T + 1), pad, np.int64)
        self.run_seq[:, :, 0] = start
        self.run_bidx = np.full((B, k, T), -1, np.int64)
        self.run_lp = np.zeros((B, k, T), np.float32)
        self.fin_score = np.full((B, k), NEG, np.float32)
        self.fin_seq = self.run_seq.copy()
        self.fin_bidx = self.run_bidx.copy()
        self.fin_lp = self.run_lp.copy()
        self.fin_flag = np.zeros((B, k), bool)
        self.heur = np.ones(B, bool)  # is_early_stop_heuristic_unsatisfied
        self.live = np.ones(B, bool)  # what the device keeps decoding (a retired prompt can no longer change)
        self.gap = np.full(B, np.inf)


def step(st: BeamState, logp: np.ndarray, t: int, eos: int, length_penalty: float = 1.0, early_stopping=False,
         division: str = "reciprocal", fma: bool = False):
    """Steps c-g of one `_beam_search` iteration at decode step t (cur_len = t + 1, max_length = T + 1) for every
    prompt. logp: fp32 [B*k, V], the log-probabilities after the EOS mask. Returns the flat parent rows [B*k] the cache
    must be reordered by, and the next decoder tokens [B*k]. Also updates the decision gaps of live prompts.
    fma: a candidate's finished-set score is fl(score * fp32(1 / l**p) + penalty) with one rounding, as
    beam_select_kernel computes it (the compiler contracts it to an FFMA); transformers rounds the product first. The
    two differ only in scores that carry the -1e9 penalty."""
    B, k, T = st.B, st.k, st.T
    V = logp.shape[1]
    K = 2 * k
    parents = np.zeros(B * k, np.int64)
    tokens = np.zeros(B * k, np.int64)
    any_hit_all = True
    for b in range(B):
        lpb = logp[b * k:(b + 1) * k]
        acc = (lpb + st.run_score[b][:, None]).astype(np.float32).reshape(-1)
        o = order(acc)
        cand = o[:K]
        gaps = []
        beam, tok = cand // V, cand % V
        cval = acc[cand]
        cseq = st.run_seq[b][beam].copy()
        cseq[:, t + 1] = tok
        cbidx = st.run_bidx[b][beam].copy()
        cbidx[:, t] = b * k + beam
        clp = st.run_lp[b][beam].copy()
        clp[:, t] = lpb[beam, tok]
        hit = (tok == eos) | (t + 1 >= T)
        any_hit_all &= bool(hit.all())
        # e. running beams: candidates that hit a stopping criterion are pushed down by -1e9
        rval = (cval + hit.astype(np.float32) * NEG).astype(np.float32)
        ro = order(rval)
        sel = ro[:k]
        # the running picks, their order (the slots) and the first one left out
        real = [rval[i] for i in ro[:k + 1] if rval[i] > _REAL]
        gaps += [a - b for a, b in zip(real, real[1:])]
        if len(real) == k and acc.size > K:  # the next candidate that does not hit lies beyond the top 2k
            nxt = next((acc[i] for i in o[K:] if not ((i % V) == eos or t + 1 >= T)), None)
            gaps += [real[-1] - nxt] if nxt is not None else []
        # whether a candidate that hits is among the first k
        gaps += [cval[c] - cval[c + 1] for c in range(K - 1) if c + 1 <= k and hit[c] != hit[c + 1] and cval[c] > _REAL]
        # f. finished set
        did = hit & (np.arange(K) < k)
        full = bool(st.fin_flag[b].all()) and early_stopping is True
        if fma:
            s = fma32(cval, length_scale(1.0, t + 1, length_penalty, division), np.where(did, np.float32(0), NEG))
            s = (s + (NEG if full else np.float32(0))).astype(np.float32)
            s = (s + (np.float32(0) if st.heur[b] else NEG)).astype(np.float32)
        else:
            s = length_scale(cval, t + 1, length_penalty, division)
            s = (s + (NEG if full else np.float32(0))).astype(np.float32)
            s = (s + (np.float32(0) if st.heur[b] else NEG)).astype(np.float32)
            s = (s + np.where(did, np.float32(0), NEG)).astype(np.float32)
        merged = np.concatenate([st.fin_score[b], s])
        mo = order(merged)
        # the finished set, its order (the returned rows) and the best entry left out
        real = [merged[i] for i in mo[:k + 1] if merged[i] > _REAL]
        gaps += [a - b for a, b in zip(real, real[1:])]
        top = mo[:k]
        mseq = np.concatenate([st.fin_seq[b], cseq])
        mbidx = np.concatenate([st.fin_bidx[b], cbidx])
        mlp = np.concatenate([st.fin_lp[b], clp])
        mflag = np.concatenate([st.fin_flag[b], did])
        st.fin_seq[b], st.fin_bidx[b], st.fin_lp[b] = mseq[top], mbidx[top], mlp[top]
        st.fin_score[b], st.fin_flag[b] = merged[top], mflag[top]
        st.run_seq[b], st.run_bidx[b], st.run_lp[b] = cseq[sel], cbidx[sel], clp[sel]
        st.run_score[b] = rval[sel]
        parents[b * k:(b + 1) * k] = b * k + beam[sel]
        tokens[b * k:(b + 1) * k] = tok[sel]
        # g. early-stop heuristic at cur_len + 1
        hyp = T if (early_stopping == "never" and length_penalty > 0.0) else t + 1
        best = length_scale(st.run_score[b][:1], hyp, length_penalty, division)[0]
        worst = np.where(st.fin_flag[b], st.fin_score[b].min(), NEG)
        if st.live[b] and gaps:
            st.gap[b] = min(st.gap[b], float(min(gaps)))
        st.heur[b] = st.heur[b] and bool((best > worst).any())
        if not st.heur[b] or (early_stopping is True and st.fin_flag[b].all()):
            st.live[b] = False
    go_on = bool(st.heur.any()) and not (bool(st.fin_flag.all()) and early_stopping is True) and not any_hit_all
    return parents, tokens, go_on


def finalize(st: BeamState, n: int, pad: int):
    """The best n finished hypotheses per prompt, rows b*n + i: (sequences [B*n, 1+L'] padded with pad, lengths [B*n],
    sequences_scores [B*n], beam_indices [B*n, L'] padded with -1, token_logprobs [B*n, L'] padded with 0)."""
    seq = st.fin_seq[:, :n].reshape(st.B * n, -1)
    bidx = st.fin_bidx[:, :n].reshape(st.B * n, -1)
    lp = st.fin_lp[:, :n].reshape(st.B * n, -1)
    lens = (bidx >= 0).sum(axis=1)
    L = int(lens.max())
    seq = seq[:, :1 + L].copy()
    for r, n_r in enumerate(lens):
        seq[r, 1 + n_r:] = pad
    return seq, lens, st.fin_score[:, :n].reshape(-1).copy(), bidx[:, :L].copy(), lp[:, :L].copy()


def beam_search(oracle, input_ids, attention_mask=None, *, num_beams: int, max_new_tokens: int, min_new_tokens: int = 0,
                num_return_sequences: int = 1, length_penalty: float = 1.0, early_stopping=False,
                division: str = "reciprocal", stop_when_done: bool = True):
    """`generate(num_beams=k, ...)` of T5Oracle -> dict(sequences, lengths, sequences_scores, beam_indices,
    token_logprobs, gap). stop_when_done=False keeps decoding until max_new_tokens, which must not change anything."""
    sp = oracle.spec
    k, T = num_beams, max_new_tokens
    B = input_ids.shape[0]
    mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
    cache = oracle._init_cache(np.repeat(oracle.encode(input_ids, mask), k, axis=0), np.repeat(mask, k, axis=0))
    st = BeamState(B, k, T, sp.decoder_start_token_id, sp.pad_token_id)
    tok = np.full(B * k, sp.decoder_start_token_id, np.int64)
    for t in range(T):
        logp = log_softmax(oracle._decode_step(tok, cache).astype(np.float32))
        if t < min_new_tokens:
            logp[:, sp.eos_token_id] = -np.inf
        parents, tok, go_on = step(st, logp, t, sp.eos_token_id, length_penalty, early_stopping, division)
        for key in ("self_k", "self_v"):
            cache[key] = [c[parents] for c in cache[key]]
        if not go_on and stop_when_done:
            break
    seq, lens, scores, bidx, lp = finalize(st, num_return_sequences, sp.pad_token_id)
    return dict(sequences=seq, lengths=lens, sequences_scores=scores, beam_indices=bidx, token_logprobs=lp, gap=st.gap)


def hf_beam_kwargs(num_beams, num_return_sequences=1, length_penalty=1.0, early_stopping=False,
                   min_new_tokens: Optional[int] = None):
    kw = dict(num_beams=num_beams, num_return_sequences=num_return_sequences, length_penalty=length_penalty,
              early_stopping=early_stopping, do_sample=False)
    if min_new_tokens:
        kw["min_new_tokens"] = min_new_tokens
    return kw
