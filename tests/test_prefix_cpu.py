"""Decoder prompts (`generate(decoder_input_ids=...)`) without a GPU: the prompted greedy reference (tests/prefix_oracle.py
over the numpy oracle) against transformers' T5ForConditionalGeneration.generate on the CPU, the length arithmetic of
the Python layer against transformers', and the argument checks that run before the library is reached."""
import ctypes as C
import warnings

import numpy as np
import pytest

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from oracle import logits_process as olp
from oracle.t5_oracle import T5Oracle
import prefix_oracle as po  # tests/prefix_oracle.py (pytest puts this directory on sys.path)

torch = pytest.importorskip("torch")
pytest.importorskip("transformers")

TAU = 1e-3  # fp32 against fp32: a near-tie below this may go either way


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    from oracle.hf_anchor import load_hf_model

    cache = {}

    def get(spec_name, seed):
        if (spec_name, seed) not in cache:
            d = tmp_path_factory.mktemp(f"prefix_{spec_name}")
            save_checkpoint(d, SPECS[spec_name], seed=seed, dtype="F32")
            cache[spec_name, seed] = (load_hf_model(d), T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name]))
        return cache[spec_name, seed]

    return get


def _hf(hf, ids, mask, dec, **kw):
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return hf.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), decoder_input_ids=torch.from_numpy(dec),
                           do_sample=False, num_beams=1, **kw).numpy()


def _gated(ours, ref, margins, P):
    """Rows agree up to their first near-tie step; returns the rows that agree in full."""
    full = 0
    for b in range(ours.shape[0]):
        low = np.where(~(margins[b] > TAU) & ~np.isnan(margins[b]))[0]
        upto = P + (low[0] if low.size else margins.shape[1])
        w = min(upto, ours.shape[1], ref.shape[1])
        assert (ours[b, :w] == ref[b, :w]).all(), b
        full += int(ours.shape[1] == ref.shape[1] and (ours[b] == ref[b]).all())
    return full


def _batch(spec, B=5, S=12, P0=4, seed=0):
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=seed + 30, lengths="uniform")
    dec = np.random.default_rng(seed).integers(2, spec.vocab_size, size=(B, P0)).astype(np.int64)
    return ids, mask, dec


def _match(hf, orc, ids, mask, dec, T, proc=None, **kw):
    """transformers with `kw` against the prompted reference with T new tokens and `proc`."""
    spec = orc.spec
    want = _hf(hf, ids, mask, dec, **kw)
    d = po.prepend_start(dec, spec.decoder_start_token_id)
    ours, _, _, margins = po.generate(orc, ids, mask, d, T, proc or olp.Processors(eos_token_id=[spec.eos_token_id]), division="true")
    assert (want[:, : d.shape[1]] == d).all()
    return _gated(ours, want, margins, d.shape[1]), ours, want


@pytest.mark.parametrize("spec_name,seed", [("tiny", 1), ("mini", 2)])
def test_prepend_rule_and_greedy_match_transformers(pair, spec_name, seed):
    hf, orc = pair(spec_name, seed)
    spec = orc.spec
    ids, mask, dec = _batch(spec, seed=seed)
    full, ours, want = _match(hf, orc, ids, mask, dec, 10, max_new_tokens=10)
    assert want.shape[1] == 5 + ours.shape[1] - 5 and full >= 3
    # every row already starts with the start token: nothing is prepended
    dec0 = dec.copy()
    dec0[:, 0] = spec.decoder_start_token_id
    _match(hf, orc, ids, mask, dec0, 10, max_new_tokens=10)
    assert (_hf(hf, ids, mask, dec0, max_new_tokens=3)[:, :4] == dec0).all()
    # only some rows do: nothing is prepended either, and every row keeps its own first id
    mixed = dec.copy()
    mixed[0, 0] = spec.decoder_start_token_id
    assert (po.prepend_start(mixed, 0) == mixed).all()
    _match(hf, orc, ids, mask, mixed, 10, max_new_tokens=10)
    # a prompt holding EOS and pad: every row still starts unfinished
    odd = dec.copy()
    odd[1, 2] = spec.eos_token_id
    odd[2, -1] = spec.eos_token_id
    odd[3, 1] = spec.pad_token_id
    _match(hf, orc, ids, mask, odd, 8, max_new_tokens=8)


@pytest.mark.parametrize("kw,T,min_new", [(dict(max_new_tokens=7), 7, 0), (dict(max_length=12), 12 - 5, 0),
                                          (dict(max_length=12, min_length=10), 7, 5), (dict(max_new_tokens=9, min_new_tokens=6), 9, 6),
                                          (dict(max_new_tokens=9, min_length=8), 9, 3), (dict(), 20, 0)])
def test_lengths_match_transformers(pair, kw, T, min_new):
    """A prompt of P = 5 ids (start token prepended to four): max_length / min_length count it, *_new_tokens do not, and the
    default is transformers' own. EOS is boosted in the synthetic checkpoints, so the EOS mask shows in the tokens."""
    hf, orc = pair("tiny", 1)
    spec = orc.spec
    ids, mask, dec = _batch(spec, seed=3)
    proc = olp.Processors(eos_token_id=[spec.eos_token_id], min_new_tokens=min_new)
    _match(hf, orc, ids, mask, dec, T, proc, **kw)
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    gp = B200T5ForConditionalGeneration._gen_params(_Stub(), **kw, _prompt_len=5)
    assert (gp.max_new_tokens, gp.min_new_tokens) == (T, min_new)
    hf_len = _hf(hf, ids, mask, dec, eos_token_id=None, **kw).shape[1]
    assert hf_len == 5 + T


@pytest.mark.parametrize("name,kw", [("rep", dict(repetition_penalty=1.6)), ("ngram", dict(no_repeat_ngram_size=2)),
                                     ("begin", dict(begin_suppress_tokens=[1, 5, 9])),
                                     ("all", dict(repetition_penalty=1.3, no_repeat_ngram_size=3, begin_suppress_tokens=[2, 7],
                                                  suppress_tokens=[4], min_new_tokens=3))])
def test_processors_over_the_prompt_match_transformers(pair, name, kw):
    hf, orc = pair("tiny", 1)
    spec = orc.spec
    ids, mask, dec = _batch(spec, B=6, seed=5)
    dec[0, 1:3] = dec[0, 0]  # repeats inside the prompt: penalties and n-gram bans must see them
    dec[1] = [7, 8, 7, 8]
    T = 9
    proc = olp.Processors(eos_token_id=[spec.eos_token_id], **kw)
    _match(hf, orc, ids, mask, dec, T, proc, max_new_tokens=T, **kw)
    if name == "begin":  # the first new token is never a begin-suppressed one; later ones may be
        ours, _, _, _ = po.generate(orc, ids, mask, po.prepend_start(dec, 0), T, proc, division="true")
        assert not np.isin(ours[:, 5], [1, 5, 9]).any()


class _Stub:
    generation_config = type("G", (), {"max_length": 20})()


def test_gen_params_without_a_prompt_are_unchanged():
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration as M

    for kw, want in ((dict(), (19, 0)), (dict(max_length=9, min_length=4), (8, 3)), (dict(max_new_tokens=5, min_new_tokens=2), (5, 2))):
        gp = M._gen_params(_Stub(), **kw)
        assert (gp.max_new_tokens, gp.min_new_tokens) == want
    with pytest.raises(ValueError):
        M._gen_params(_Stub(), max_length=5, _prompt_len=5)  # transformers: the prompt leaves no room


class _Model:
    """The host-side surface of B200T5ForConditionalGeneration that argument handling reads (no GPU, no library)."""

    def __init__(self):
        from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration as M

        self.M = M
        self.config = type("C", (), {"vocab_size": 50})()
        self.generation_config = type("G", (), {"max_length": 20, "decoder_start_token_id": 0, "eos_token_id": 1, "pad_token_id": 0})()

    def prompt(self, d, B, start=None):
        return self.M._decoder_prompt(self, d, B, start)


def test_decoder_prompt_rule_and_checks():
    m = _Model()
    assert (m.prompt([[5, 6], [7, 8]], 2) == [[0, 5, 6], [0, 7, 8]]).all()
    assert (m.prompt(torch.tensor([[0, 6], [7, 8]]), 2) == [[0, 6], [7, 8]]).all()  # one row starts with it: kept as is
    assert (m.prompt([[3], [3]], 2, start=3) == [[3], [3]]).all()
    assert m.prompt(np.array([[4]], np.int32), 1).dtype == np.int64
    for bad in ([[1, 2]], [1, 2], [[]], np.zeros((2, 2), np.float32)):
        with pytest.raises(ValueError):
            m.prompt(bad, 2)
    for bad in ([[1, 50], [2, 3]], [[-1, 2], [2, 3]]):
        with pytest.raises(IndexError):
            m.prompt(bad, 2)


def test_unsupported_combinations_raise_before_the_library():
    """decoder_input_ids with beams, decoder_attention_mask, and the slot pool with a prompt: NotImplementedError naming
    the argument (the model needs no GPU to get there)."""
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration as M

    m = M.__new__(M)
    m.config = type("C", (), {"vocab_size": 50})()
    m.generation_config = type("G", (), {"max_length": 20, "decoder_start_token_id": 0, "eos_token_id": 1, "pad_token_id": 0})()
    ids = np.full((2, 4), 5, np.int64)
    with pytest.raises(NotImplementedError, match="decoder_input_ids"):
        m.generate(input_ids=ids, decoder_input_ids=[[3], [4]], num_beams=2)
    with pytest.raises(NotImplementedError, match="decoder_attention_mask"):
        m.generate(input_ids=ids, decoder_input_ids=[[3], [4]], decoder_attention_mask=[[1], [1]])
    with pytest.raises(NotImplementedError, match="decoder_attention_mask"):
        m.generate_host(ids, decoder_input_ids=[[3], [4]], decoder_attention_mask=[[1], [1]])
    with pytest.raises(NotImplementedError, match="decoder_input_ids"):
        m.generate_host(ids, decoder_input_ids=[[3], [4]], num_beams=2)
    with pytest.raises(NotImplementedError, match="decoder_input_ids"):
        m.generate_stream(ids, decoder_input_ids=[[3], [4]])
    with pytest.raises(ValueError):
        m.generate(input_ids=ids, decoder_input_ids=[[3]])
    with pytest.raises(IndexError):
        m.generate(input_ids=ids, decoder_input_ids=[[3], [99]])


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
def test_prefixed_entry_points_are_bound(flavour):
    lib = _lib.load(flavour)
    for name in ("b200t5_generate_prefixed", "b200t5_generate_host_prefixed", "b200t5_test_prefill_cache"):
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    # no handle: a loud error, not a crash
    assert lib.b200t5_test_prefill_cache(None, 0, C.c_void_p(1), None) == _lib.EINVAL
