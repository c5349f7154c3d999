"""numpy restatement of transformers' greedy-mode logits processors (generation/logits_process.py, in the order
GenerationMixin._get_logits_processor builds them) and a greedy loop over T5Oracle that applies them.

The scores are the lm_head logits rounded to the compute dtype and widened to fp32, as HF's `.to(torch.float32)`:
  1. encoder_repetition_penalty over the prompt ids (padding included), once per distinct token, p = 1 / penalty;
  2. repetition_penalty over the decoder ids so far (start token included);
  3. no_repeat_ngram_size over the decoder ids (start token included);
  4. encoder_no_repeat_ngram_size over the n-grams of the prompt ids (padding included);
  5. bad_words_ids (a sequence equal to [eos] is dropped; the zero bias HF adds turns -0.0 into +0.0);
  6. the EOS mask while fewer than min_new_tokens tokens were generated;
  7. suppress_tokens, then begin_suppress_tokens at the first generated position;
  8. arg-max with the first-index tie rule.
`division`: torch on CUDA divides an fp32 tensor by a Python float p as a multiplication by fp32(1 / p), the
reciprocal taken in double ("reciprocal", what libb200t5 computes); torch on the CPU divides ("true").
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np


@dataclass
class Processors:
    repetition_penalty: float = 1.0
    encoder_repetition_penalty: float = 1.0
    no_repeat_ngram_size: int = 0
    encoder_no_repeat_ngram_size: int = 0
    bad_words_ids: Optional[List[List[int]]] = None
    suppress_tokens: Optional[Sequence[int]] = None
    begin_suppress_tokens: Optional[Sequence[int]] = None
    eos_token_id: List[int] = field(default_factory=lambda: [1])
    min_new_tokens: int = 0


def _penalise(x: np.ndarray, p: float, division: str) -> np.ndarray:
    p32 = np.float32(p)
    pos = x * np.float32(1.0 / p) if division == "reciprocal" else x / p32
    return np.where(x < 0, x * p32, pos).astype(np.float32)


def _ngram_bans(hist: Sequence[int], source: Sequence[int], n: int) -> List[int]:
    """Tokens that follow, in `source`, an (n-1)-gram equal to the last n-1 ids of `hist`."""
    L = len(hist)
    if L < n - 1:
        return []
    key = list(hist[L - n + 1:]) if n > 1 else []
    return [int(source[j + n - 1]) for j in range(len(source) - n + 1) if list(source[j:j + n - 1]) == key]


def process(scores: np.ndarray, dec_ids: np.ndarray, enc_ids: np.ndarray, proc: Processors,
            division: str = "reciprocal") -> np.ndarray:
    """scores fp32 [B,V] of the next position; dec_ids int [B,L] the decoder ids so far; enc_ids int [B,S]."""
    s = np.array(scores, dtype=np.float32, copy=True)
    B, V = s.shape
    L = dec_ids.shape[1]
    if proc.encoder_repetition_penalty != 1.0:
        for b in range(B):
            cols = np.unique(enc_ids[b])
            s[b, cols] = _penalise(s[b, cols], 1.0 / proc.encoder_repetition_penalty, division)
    if proc.repetition_penalty != 1.0:
        for b in range(B):
            cols = np.unique(dec_ids[b])
            s[b, cols] = _penalise(s[b, cols], proc.repetition_penalty, division)
    n = proc.no_repeat_ngram_size
    if n and L + 1 >= n:
        for b in range(B):
            s[b, _ngram_bans(dec_ids[b].tolist(), dec_ids[b].tolist(), n)] = -np.inf
    n = proc.encoder_no_repeat_ngram_size
    if n:
        for b in range(B):
            s[b, _ngram_bans(dec_ids[b].tolist(), enc_ids[b].tolist(), n)] = -np.inf
    if proc.bad_words_ids is not None:
        seqs = [list(w) for w in proc.bad_words_ids if not (len(w) == 1 and w[0] in proc.eos_token_id)]
        bias = np.zeros_like(s)
        for w in seqs:
            if len(w) == 1:
                bias[:, w[0]] = -np.inf
            elif len(w) <= L:
                for b in range(B):
                    if dec_ids[b, L - len(w) + 1:].tolist() == w[:-1]:
                        bias[b, w[-1]] = -np.inf
        s = (s + bias).astype(np.float32)
    if L - 1 < proc.min_new_tokens:
        s[:, proc.eos_token_id] = -np.inf
    if proc.suppress_tokens:
        s[:, list(proc.suppress_tokens)] = -np.inf
    if proc.begin_suppress_tokens and L == 1:
        s[:, list(proc.begin_suppress_tokens)] = -np.inf
    return s


def generate(oracle, input_ids, attention_mask=None, max_new_tokens: int = 20, processors: Optional[Processors] = None,
             return_margins: bool = False, division: str = "reciprocal"):
    """T5Oracle.generate with the processors applied to each step's logits (processors=None: plain greedy, EOS masked
    while fewer than min_new_tokens of the Processors were generated). Margins are top-1 minus top-2 of the PROCESSED
    scores (NaN once a row has finished)."""
    proc = processors or Processors()
    sp = oracle.spec
    eos = list(proc.eos_token_id)
    B = input_ids.shape[0]
    mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
    cache = oracle._init_cache(oracle.encode(input_ids, mask), mask)
    out = np.full((B, 1), sp.decoder_start_token_id, dtype=np.int64)
    unfinished = np.ones(B, dtype=bool)
    margins = []
    tok = out[:, 0]
    for _ in range(max_new_tokens):
        logits = oracle._decode_step(tok, cache).astype(np.float32)
        scores = process(logits, out, input_ids, proc, division)
        nxt = scores.argmax(axis=-1)
        if return_margins:
            top2 = np.partition(scores, -2, axis=-1)[:, -2:]
            margins.append(np.where(unfinished, top2[:, 1] - top2[:, 0], np.nan))
        nxt = np.where(unfinished, nxt, sp.pad_token_id)
        out = np.concatenate([out, nxt[:, None]], axis=1)
        unfinished &= ~np.isin(nxt, eos)
        tok = nxt
        if not unfinished.any():
            break
    if return_margins:
        return out, np.stack(margins, axis=1)
    return (out,)
