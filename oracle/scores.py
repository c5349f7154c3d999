"""Token log-probabilities in numpy: what the scored CUDA decode step (csrc/gemm.cuh EpiScore) must reproduce.

`generate` is oracle/logits_process.generate that also returns, per generated position, the chosen token's processed
score and its log-softmax over the step's processed scores (the two arrays transformers' compute_transition_scores
gives with normalize_logits=False / True); `score` is the teacher-forced counterpart: log p(label | prompt, earlier
labels) and the mean cross-entropy `T5ForConditionalGeneration(..., labels=...).loss`. Positions a row does not reach
(after its EOS, ignored labels) hold 0. TEST INFRASTRUCTURE, like the rest of this package.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from oracle.logits_process import Processors, process


def log_softmax(scores: np.ndarray) -> np.ndarray:
    """fp32, max-subtracted; -inf columns stay -inf."""
    s = scores.astype(np.float32)
    m = s.max(axis=-1, keepdims=True)
    e = np.exp(s - m, dtype=np.float32)
    return (s - m - np.log(e.sum(axis=-1, keepdims=True, dtype=np.float32))).astype(np.float32)


def generate(oracle, input_ids, attention_mask=None, max_new_tokens: int = 20, processors: Optional[Processors] = None,
             division: str = "reciprocal"):
    """-> (tokens int64 [B, 1+T'], token_logits fp32 [B, T'], token_logprobs fp32 [B, T'], margins [B, T'])."""
    proc = processors or Processors()
    sp = oracle.spec
    eos = list(proc.eos_token_id)
    B = input_ids.shape[0]
    mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
    cache = oracle._init_cache(oracle.encode(input_ids, mask), mask)
    out = np.full((B, 1), sp.decoder_start_token_id, dtype=np.int64)
    unfinished = np.ones(B, dtype=bool)
    logits_, logps, margins = [], [], []
    rows = np.arange(B)
    tok = out[:, 0]
    for _ in range(max_new_tokens):
        scores = process(oracle._decode_step(tok, cache).astype(np.float32), out, input_ids, proc, division)
        nxt = scores.argmax(axis=-1)
        top2 = np.partition(scores, -2, axis=-1)[:, -2:]
        margins.append(np.where(unfinished, top2[:, 1] - top2[:, 0], np.nan))
        logits_.append(np.where(unfinished, scores[rows, nxt], 0).astype(np.float32))
        logps.append(np.where(unfinished, log_softmax(scores)[rows, nxt], 0).astype(np.float32))
        nxt = np.where(unfinished, nxt, sp.pad_token_id)
        out = np.concatenate([out, nxt[:, None]], axis=1)
        unfinished &= ~np.isin(nxt, eos)
        tok = nxt
        if not unfinished.any():
            break
    return out, np.stack(logits_, axis=1), np.stack(logps, axis=1), np.stack(margins, axis=1)


def score(oracle, input_ids, attention_mask, labels):
    """labels int64 [B, L], -100 = ignored (trailing). -> (token_logprobs fp32 [B, L], loss)."""
    sp = oracle.spec
    B, L = labels.shape
    mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
    cache = oracle._init_cache(oracle.encode(input_ids, mask), mask)
    # T5's _shift_right: start token first, ignored positions fed as pad
    dec = np.concatenate([np.full((B, 1), sp.decoder_start_token_id, dtype=np.int64), np.where(labels == -100, sp.pad_token_id, labels)[:, :-1]], axis=1)
    out = np.zeros((B, L), dtype=np.float32)
    rows = np.arange(B)
    for t in range(L):
        lsm = log_softmax(oracle._decode_step(dec[:, t], cache).astype(np.float32))
        on = labels[:, t] != -100
        out[:, t] = np.where(on, lsm[rows, np.where(on, labels[:, t], 0)], 0)
    return out, float(-out.astype(np.float64).sum() / (labels != -100).sum())
