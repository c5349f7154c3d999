"""The numpy logits processors (oracle/logits_process.py) against transformers' own processor classes, the argument
validation of the CUDA path's Python layer, and the ABI of the processor entry points. No GPU needed."""
import re
import subprocess

import numpy as np
import pytest

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.modeling import _eos_ids, logits_processor_args
from oracle.logits_process import Processors, process

V = 97


def _case(seed, B=5, L=9, S=13):
    rng = np.random.default_rng(seed)
    scores = (rng.standard_normal((B, V)) * 4).astype(np.float32)
    scores[0, :8] = -0.0  # signed zeros: the bad-words bias turns them into +0.0
    dec = rng.integers(0, 12, size=(B, L))
    dec[:, 0] = 0  # decoder start token = pad
    dec[1, 1:] = np.tile([3, 4, 5], L)[: L - 1]  # repeated n-grams
    enc = rng.integers(0, 12, size=(B, S))
    enc[:, -3:] = 0  # padding
    enc[2, :6] = [3, 4, 5, 3, 4, 6]
    return scores, dec, enc


def _hf(scores, dec, enc, proc):
    torch = pytest.importorskip("torch")
    lp = pytest.importorskip("transformers.generation.logits_process")
    s = torch.from_numpy(scores.copy())
    ids = torch.from_numpy(dec)
    encs = torch.from_numpy(enc)
    chain = []
    if proc.encoder_repetition_penalty != 1.0:
        chain.append(lp.EncoderRepetitionPenaltyLogitsProcessor(proc.encoder_repetition_penalty, encs))
    if proc.repetition_penalty != 1.0:
        chain.append(lp.RepetitionPenaltyLogitsProcessor(proc.repetition_penalty))
    if proc.no_repeat_ngram_size:
        chain.append(lp.NoRepeatNGramLogitsProcessor(proc.no_repeat_ngram_size))
    if proc.encoder_no_repeat_ngram_size:
        chain.append(lp.EncoderNoRepeatNGramLogitsProcessor(proc.encoder_no_repeat_ngram_size, encs))
    if proc.bad_words_ids is not None:
        chain.append(lp.NoBadWordsLogitsProcessor(proc.bad_words_ids, proc.eos_token_id))
    if proc.min_new_tokens:
        chain.append(lp.MinNewTokensLengthLogitsProcessor(1, proc.min_new_tokens, proc.eos_token_id))
    if proc.suppress_tokens:
        chain.append(lp.SuppressTokensLogitsProcessor(proc.suppress_tokens))
    if proc.begin_suppress_tokens:
        chain.append(lp.SuppressTokensAtBeginLogitsProcessor(proc.begin_suppress_tokens, 1))
    for p in chain:
        s = p(ids, s)
    return s.numpy()


PROCS = {
    "rep": Processors(repetition_penalty=1.3),
    "enc_rep": Processors(encoder_repetition_penalty=0.7),
    "ngram2": Processors(no_repeat_ngram_size=2),
    "ngram3": Processors(no_repeat_ngram_size=3),
    "ngram1": Processors(no_repeat_ngram_size=1),
    "enc_ngram3": Processors(encoder_no_repeat_ngram_size=3),
    "enc_ngram1": Processors(encoder_no_repeat_ngram_size=1),
    "bad": Processors(bad_words_ids=[[1], [7], [4, 5], [3, 4, 5, 3], [0, 9], [11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 2]]),
    "min_new": Processors(min_new_tokens=20, eos_token_id=[1, 6]),
    "suppress": Processors(suppress_tokens=[2, 3, 50], begin_suppress_tokens=[5, 6]),
    "all": Processors(repetition_penalty=1.2, encoder_repetition_penalty=1.5, no_repeat_ngram_size=2,
                      encoder_no_repeat_ngram_size=2, bad_words_ids=[[1], [9], [4, 5]], suppress_tokens=[10],
                      begin_suppress_tokens=[11], eos_token_id=[1, 2], min_new_tokens=3),
}


@pytest.mark.parametrize("name", list(PROCS))
@pytest.mark.parametrize("L", [1, 2, 9])
def test_numpy_processors_equal_transformers(name, L):
    proc = PROCS[name]
    for seed in range(3):
        scores, dec, enc = _case(seed, L=L)
        ours = process(scores, dec, enc, proc, division="true")  # torch on the CPU divides
        ref = _hf(scores, dec, enc, proc)
        assert ours.dtype == np.float32
        assert np.array_equal(ours.view(np.uint32), ref.view(np.uint32)), name


def test_reciprocal_division_is_within_two_ulps_of_true_division():
    scores, dec, enc = _case(7)
    a = process(scores, dec, enc, PROCS["all"], division="reciprocal")
    b = process(scores, dec, enc, PROCS["all"], division="true")
    fin = np.isfinite(a)
    assert (np.isfinite(b) == fin).all()
    diff = np.abs(a[fin].view(np.int32).astype(np.int64) - b[fin].view(np.int32).astype(np.int64))
    assert diff.max() <= 2  # one ulp per penalty; a token in both the prompt and the decoder ids gets two


def test_argument_validation_and_no_op_values():
    ok = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, suppress_tokens=[], encoder_repetition_penalty=1.0,
              encoder_no_repeat_ngram_size=0, begin_suppress_tokens=[])
    assert logits_processor_args(ok, None, 1, V) is None
    assert logits_processor_args({}, [1], 1, V) is None
    assert logits_processor_args({}, _eos_ids([1, 1]), 1, V) is None
    assert logits_processor_args({}, [1, 5], 1, V).params.n_eos_token_ids == 2
    a = logits_processor_args({"bad_words_ids": [[1], [4, 5], [6]]}, None, 1, V)
    assert a.params.n_bad_words == 2  # [eos] dropped
    for bad in ({"repetition_penalty": 0.0}, {"repetition_penalty": -1.0}, {"encoder_repetition_penalty": 0},
                {"no_repeat_ngram_size": -1}, {"encoder_no_repeat_ngram_size": -2}, {"bad_words_ids": []},
                {"bad_words_ids": [[]]}, {"bad_words_ids": [[V]]}, {"bad_words_ids": [[1]]}, {"bad_words_ids": [3]},
                {"suppress_tokens": [V]}, {"begin_suppress_tokens": [-1]}):
        with pytest.raises(ValueError):
            logits_processor_args(bad, None, 1, V)


NEW = ("b200t5_generate_ex", "b200t5_generate_host_ex", "b200t5_generate_stream_ex", "b200t5_test_lm_process")


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
def test_processor_symbols_are_exported_and_bound(flavour):
    path = _lib.LIB_PATHS[flavour]
    if not path.exists():
        pytest.skip(f"{path.name} not built")
    exported = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True).stdout
    for n in NEW:
        assert re.search(rf"\bT {n}\b", exported), f"{n} not exported by {path.name}"
        assert n in _lib.SIGNATURES
    assert _lib.SIGNATURES["b200t5_generate_ex"][1][6]._type_ is _lib.LogitsParams


def test_logits_params_struct_layout_matches_the_header():
    # two doubles, two int32, then (pointer, int32) x 3, two pointers and an int32, with natural alignment
    assert _lib.LogitsParams.repetition_penalty.offset == 0
    assert _lib.LogitsParams.no_repeat_ngram_size.offset == 16
    assert _lib.LogitsParams.suppress_tokens.offset == 24
    assert _lib.LogitsParams.n_bad_words.offset == 88
    assert _lib.C.sizeof(_lib.LogitsParams) == 96
