"""Greedy decoding after a decoder prompt (transformers' generate(decoder_input_ids=...)), restated on top of the numpy
oracle: T5Oracle._decode_step for the arithmetic and oracle.logits_process.process for the processors. TEST
INFRASTRUCTURE, imported by tests/test_prefix_*.py only.

transformers (generation/utils.py, 5.5):
  _prepare_decoder_input_ids_for_generation  the start token is prepended only when EVERY row's first id differs from it;
  _prepare_generated_length                  max_length / min_length count the prompt, *_new_tokens do not;
  MinNewTokensLengthLogitsProcessor          EOS masked while len(ids) - P < min_new_tokens;
  SuppressTokensAtBeginLogitsProcessor       begin_index = P: applies when len(ids) == P, the first generated position.
The prompt is teacher-forced through the decode step (its logits are dropped), every row starts unfinished, and the
processors see the prompt as decoder ids.
"""
from __future__ import annotations

import dataclasses
from typing import Optional

import numpy as np

from oracle.logits_process import Processors, process
from oracle.scores import log_softmax


def prepend_start(d: np.ndarray, start: int) -> np.ndarray:
    """transformers' rule: prepend the start token unless some row already begins with it."""
    d = np.asarray(d, dtype=np.int64)
    if (d[:, 0] != start).all():
        d = np.concatenate([np.full((d.shape[0], 1), start, dtype=np.int64), d], axis=1)
    return d


def generate(oracle, input_ids, attention_mask, decoder_input_ids, max_new_tokens: int, processors: Optional[Processors] = None,
             division: str = "reciprocal"):
    """Greedy search from the decoder prompt decoder_input_ids [B, P] (start token included, taken as given).
    -> (tokens int64 [B, P+T'], token_logits fp32 [B, T'], token_logprobs fp32 [B, T'], margins [B, T'])."""
    proc = processors or Processors()
    sp = oracle.spec
    eos = list(proc.eos_token_id)
    d = np.asarray(decoder_input_ids, dtype=np.int64)
    B, P = d.shape
    # process() counts generated tokens from a one-id prompt and suppresses begin tokens at length 1: shift the first
    # by P - 1 and apply the second here, at length P
    shifted = dataclasses.replace(proc, min_new_tokens=proc.min_new_tokens + P - 1 if proc.min_new_tokens else 0,
                                  begin_suppress_tokens=None)
    mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
    cache = oracle._init_cache(oracle.encode(input_ids, mask), mask)
    for t in range(P - 1):
        oracle._decode_step(d[:, t], cache)
    out = d.copy()
    unfinished = np.ones(B, dtype=bool)
    logits_, logps, margins = [], [], []
    rows = np.arange(B)
    tok = d[:, -1]
    for _ in range(max_new_tokens):
        scores = process(oracle._decode_step(tok, cache).astype(np.float32), out, input_ids, shifted, division)
        if proc.begin_suppress_tokens and out.shape[1] == P:
            scores[:, list(proc.begin_suppress_tokens)] = -np.inf
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


def prompt_cache(oracle, input_ids, attention_mask, decoder_input_ids):
    """The self-attention K and V of every decoder layer after teacher-forcing positions 0 .. P-2 of the prompt:
    lists of [B, H, P-1, 64]."""
    d = np.asarray(decoder_input_ids, dtype=np.int64)
    mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
    cache = oracle._init_cache(oracle.encode(input_ids, mask), mask)
    for t in range(d.shape[1] - 1):
        oracle._decode_step(d[:, t], cache)
    return cache["self_k"], cache["self_v"]
