"""Decoder prompts on the CUDA path (`generate(decoder_input_ids=...)`, b200t5_generate_prefixed) on an H100, both builds.

Anchors: a prompt of the start token alone is the ordinary call; the prefill's self-attention cache against the oracle's
K/V; tokens and log-probabilities against the oracle (gated at near-ties) and against transformers on this GPU; bits
across batch-mates, chunks, entry points and repeated calls; the first new token against step-by-step teacher forcing.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from oracle import logits_process as olp
from oracle.scores import log_softmax
from oracle.t5_oracle import T5Oracle
import prefix_oracle as po  # tests/prefix_oracle.py (pytest puts this directory on sys.path)

pytestmark = pytest.mark.gpu

TAU = {torch.bfloat16: 0.13, torch.float16: 0.03}  # margin gates / logit-error bounds of tests/test_scores_gpu.py
EMULATE = {torch.bfloat16: "bf16", torch.float16: "fp16"}
DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(spec_name, seed, dtype=torch.bfloat16):
        key = (spec_name, seed, dtype)
        if key not in cache:
            d = tmp_path_factory.mktemp(f"prefix_{spec_name}_{seed}")
            save_checkpoint(d, SPECS[spec_name], seed=seed)
            cache[key] = (B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=dtype), d)
        return cache[key]

    return get


_ORACLES = {}


def _oracle(spec_name, seed, dtype):
    key = (spec_name, seed, dtype)
    if key not in _ORACLES:
        _ORACLES[key] = T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate=EMULATE[dtype])
    return _ORACLES[key]


def _prompts(B, P0, vocab, seed):
    """[B, P0] answer prefixes that never start with the start token (0): the start token is prepended."""
    return np.random.default_rng(seed).integers(2, vocab, size=(B, P0)).astype(np.int64)


def _scored(model, ids, mask, dec, **kw):
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), decoder_input_ids=torch.from_numpy(dec),
                         return_dict_in_generate=True, output_scores=True, **kw)
    return out.sequences.cpu().numpy(), out.token_logprobs.cpu().numpy(), out.scores.token_logits.cpu().numpy()


def _compare_gated(toks, logp, ref_toks, ref_logp, margins, tau, P):
    """tests/test_scores_gpu.py's gate after a prompt of P ids: up to a row's first near-tie step the new tokens must
    agree; the numbers are compared while the tokens agree, within twice the logit error. Returns positions compared."""
    assert (toks[:, :P] == ref_toks[:, :P]).all()
    n = min(toks.shape[1], ref_toks.shape[1]) - P
    compared = 0
    for b in range(toks.shape[0]):
        m = margins[b, :n]
        ended = np.where(np.isnan(m))[0]
        live = ended[0] if ended.size else n
        low = np.where(~(m[:live] > tau))[0]
        gate = low[0] if low.size else live
        assert (toks[b, : P + gate] == ref_toks[b, : P + gate]).all(), b
        diff = np.where(toks[b, P: P + live] != ref_toks[b, P: P + live])[0]
        upto = diff[0] if diff.size else live
        assert np.abs(logp[b, :upto] - ref_logp[b, :upto]).max(initial=0) <= 2 * tau, b
        compared += upto
    return compared


def _launches(model):
    return int(model.stats()["kernel_launches"])


# ---------------------------------------------------------------- 1. P = 1 is the ordinary call
@DTYPES
def test_start_token_prompt_is_the_ordinary_call(models, dtype):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1, dtype)
    ids, mask = synthetic_token_batch(7, 24, spec.vocab_size, seed=3, lengths="uniform")
    ti, tm = torch.from_numpy(ids), torch.from_numpy(mask)
    start = np.zeros((7, 1), np.int64)
    for kw in (dict(), dict(repetition_penalty=1.3, no_repeat_ngram_size=2, begin_suppress_tokens=[5])):
        plain = model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=12, return_dict_in_generate=True, output_scores=True, **kw)
        n_plain = _launches(model)
        pre = model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=12, decoder_input_ids=torch.from_numpy(start),
                             return_dict_in_generate=True, output_scores=True, **kw)
        assert _launches(model) == n_plain
        assert torch.equal(plain.sequences, pre.sequences)
        assert torch.equal(plain.token_logprobs, pre.token_logprobs)
        assert torch.equal(plain.scores.token_logits, pre.scores.token_logits)
        seq = model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=12, **kw)
        seq_pre = model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=12, decoder_input_ids=start, **kw)
        assert torch.equal(seq, seq_pre) and torch.equal(seq, plain.sequences)


# ---------------------------------------------------------------- 2. the prefill's cache at kernel level
@DTYPES
@pytest.mark.parametrize("spec_name,seed,P0", [("tiny", 1, 5), ("mini", 2, 17)])
def test_prefill_cache_matches_the_oracle(models, dtype, spec_name, seed, P0):
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    B = 3
    ids, mask = synthetic_token_batch(B, 20, spec.vocab_size, seed=seed + 7, lengths="uniform")
    d = po.prepend_start(_prompts(B, P0, spec.vocab_size, seed), spec.decoder_start_token_id)
    P = d.shape[1]
    model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), decoder_input_ids=torch.from_numpy(d),
                   max_new_tokens=3)
    ks, vs = po.prompt_cache(_oracle(spec_name, seed, dtype), ids, mask, d)
    H = spec.num_heads
    for layer in range(spec.num_decoder_layers):
        got = torch.empty((2, B, H, P - 1, 64), dtype=dtype, device="cuda")
        rc = model._lib.b200t5_test_prefill_cache(model._h, layer, C.c_void_p(got.data_ptr()), None)
        assert rc == 0
        torch.cuda.synchronize()
        got = got.float().cpu().numpy()
        ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
        for kv, ref in ((0, ks[layer]), (1, vs[layer])):
            err = np.abs(got[kv] - ref)
            scale = np.abs(ref).max()
            print(f"{spec_name} {EMULATE[dtype]} layer {layer} {'KV'[kv]}: max {err.max() / scale:.2e} mean {err.mean() / scale:.2e} of {scale:.3g}")
            if layer == 0:  # the embedded prompt's norm and one product: accumulation order is the only difference
                assert err.max() <= 4 * ulp * scale, (kv, err.max(), scale)
            else:  # the layers below add their differences; a wrong position, head or layer would be off by ~scale
                assert err.max() <= 32 * ulp * scale and err.mean() <= 2 * ulp * scale, (layer, kv, err.max(), err.mean(), scale)


# ---------------------------------------------------------------- 3. tokens against the oracle and transformers
PROCS = {"plain": dict(), "rep_ngram": dict(repetition_penalty=1.3, no_repeat_ngram_size=2),
         "all": dict(repetition_penalty=1.3, encoder_repetition_penalty=0.9, no_repeat_ngram_size=3, encoder_no_repeat_ngram_size=3,
                     bad_words_ids=[[7], [5, 9]], suppress_tokens=[3], begin_suppress_tokens=[2], min_new_tokens=4)}
CASES = [("plain", 3, 14), ("rep_ngram", 3, 14), ("all", 3, 14), ("plain", 120, 24), ("all", 120, 24)]


@DTYPES
@pytest.mark.parametrize("spec_name,seed", [("tiny", 1), ("mini", 2)])
@pytest.mark.parametrize("name,P0,T", CASES)
def test_model_matches_the_oracle(models, dtype, spec_name, seed, name, P0, T):
    """(120, 24): the last positions pass 128, where the relative-position buckets saturate, across the prefill/decode
    boundary."""
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    kw = dict(PROCS[name])
    ids, mask = synthetic_token_batch(6, 16, spec.vocab_size, seed=41, lengths="uniform")
    d0 = _prompts(6, P0, spec.vocab_size, seed=P0)
    d0[1, 1] = spec.eos_token_id  # a prompt that holds EOS and pad: rows still start unfinished
    d0[2, 2] = spec.pad_token_id
    toks, logp, logit = _scored(model, ids, mask, d0, max_new_tokens=T, **kw)
    d = po.prepend_start(d0, spec.decoder_start_token_id)
    P = d.shape[1]
    assert toks.shape[1] <= P + T and (model.last_lengths.cpu().numpy() >= 1).all()
    min_new = kw.pop("min_new_tokens", 0)
    proc = olp.Processors(eos_token_id=[1], min_new_tokens=min_new, **kw)
    ref, ref_logit, ref_logp, margins = po.generate(_oracle(spec_name, seed, dtype), ids, mask, d, T, proc)
    assert _compare_gated(toks, logp, ref, ref_logp, margins, TAU[dtype], P) > 6
    assert _compare_gated(toks, logit, ref, ref_logit, margins, TAU[dtype], P) > 6
    # the plain call gives the scored call's tokens
    plain = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), decoder_input_ids=torch.from_numpy(d0),
                           max_new_tokens=T, min_new_tokens=min_new or None, **kw).cpu().numpy()
    assert np.array_equal(plain, toks)


def test_flan_t5_small_vs_hf_transition_scores(models):
    pytest.importorskip("transformers")
    from oracle.hf_anchor import hf_teacher_forced_logits, load_hf_model

    spec = SPECS["flan-t5-small"]
    model, ckpt = models("flan-t5-small", 3)
    B, S, T, P0 = 16, 96, 24, 6
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths="uniform")
    d0 = _prompts(B, P0, spec.vocab_size, seed=9)
    hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
    tids, tmask, tdec = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(d0).cuda()
    for kw in (dict(), dict(repetition_penalty=1.3, no_repeat_ngram_size=3)):
        with torch.no_grad():
            ref = hf.generate(input_ids=tids, attention_mask=tmask, decoder_input_ids=tdec, max_new_tokens=T, min_new_tokens=T,
                              do_sample=False, num_beams=1, return_dict_in_generate=True, output_scores=True, **kw)
            ref_logp = hf.compute_transition_scores(ref.sequences, ref.scores, normalize_logits=True).float().cpu().numpy()
            ref_logit = hf.compute_transition_scores(ref.sequences, ref.scores, normalize_logits=False).float().cpu().numpy()
        ref_toks = ref.sequences.cpu().numpy()
        P = ref_toks.shape[1] - T
        assert P == P0 + 1
        out = model.generate(input_ids=tids, attention_mask=tmask, decoder_input_ids=tdec, max_new_tokens=T, min_new_tokens=T,
                             return_dict_in_generate=True, output_scores=True, **kw)
        logp = model.compute_transition_scores(out.sequences, out.scores, normalize_logits=True).cpu().numpy()
        logit = model.compute_transition_scores(out.sequences, out.scores, normalize_logits=False).cpu().numpy()
        assert logp.shape == (B, T)
        lg = hf_teacher_forced_logits(hf, ids, mask, ref_toks[:, :-1])
        proc = olp.Processors(eos_token_id=[1], min_new_tokens=T + P - 1, **kw)
        margins = np.zeros((B, T))
        for t in range(T):
            s = olp.process(lg[:, P - 1 + t].astype(np.float32), ref_toks[:, : P + t], ids, proc)
            top2 = np.partition(s, -2, axis=-1)[:, -2:]
            margins[:, t] = top2[:, 1] - top2[:, 0]
        toks = out.sequences.cpu().numpy()
        n = _compare_gated(toks, logp, ref_toks, ref_logp, margins, TAU[torch.bfloat16], P)
        _compare_gated(toks, logit, ref_toks, ref_logit, margins, TAU[torch.bfloat16], P)
        print(f"flan-t5-small prefixed {kw or 'plain'}: {n} of {B * T} positions compared with transformers")
        assert n >= 2 * B


# ---------------------------------------------------------------- 4. bits
@DTYPES
def test_bits_across_batches_chunks_entry_points_and_replays(models, dtype):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1, dtype)
    B, T = 10, 16
    ids, mask = synthetic_token_batch(B, 28, spec.vocab_size, seed=13, lengths="uniform")
    d0 = _prompts(B, 9, spec.vocab_size, seed=4)
    ti, tm, td = torch.from_numpy(ids), torch.from_numpy(mask), torch.from_numpy(d0)
    kw = dict(max_new_tokens=T, return_dict_in_generate=True, output_scores=True)
    full = model.generate(input_ids=ti, attention_mask=tm, decoder_input_ids=td, **kw)
    launches = _launches(model)
    lens = model.last_lengths.cpu().numpy()
    seq, lp = full.sequences.cpu().numpy(), full.token_logprobs.cpu().numpy()
    # chunks: pool_size below B runs static chunks, never the slot pool
    pool = model.pool_size
    try:
        model.pool_size = 4
        ch = model.generate(input_ids=ti, attention_mask=tm, decoder_input_ids=td, **kw)
    finally:
        model.pool_size = pool
    assert np.array_equal(ch.sequences.cpu().numpy(), seq) and np.array_equal(ch.token_logprobs.cpu().numpy(), lp)
    # a row alone
    for b in (0, 7):
        one = model.generate(input_ids=ti[b:b + 1], attention_mask=tm[b:b + 1], decoder_input_ids=td[b:b + 1], **kw)
        n = one.sequences.shape[1]
        assert np.array_equal(one.sequences.cpu().numpy()[0], seq[b, :n]) and (seq[b, n:] == spec.pad_token_id).all()
        assert np.array_equal(one.token_logprobs.cpu().numpy()[0], lp[b, : n - d0.shape[1] - 1])
    # the host entry point
    hs, hl, hlp, hlg = model.generate_host(ids, mask, decoder_input_ids=d0, max_new_tokens=T, output_scores=True)
    assert np.array_equal(hs, seq) and np.array_equal(hlp, lp)
    assert np.array_equal(hl, lens) and (hl >= 1).all() and hl.max() == seq.shape[1] - d0.shape[1] - 1
    # replays after other kinds of calls on the same handle: same bits, same launches
    for other in (lambda: model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=T),
                  lambda: model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=T, repetition_penalty=1.2),
                  lambda: model.decode_logits(ti, tm, torch.from_numpy(po.prepend_start(d0, 0))),
                  lambda: model(input_ids=ti, attention_mask=tm, labels=td),
                  lambda: model.generate(input_ids=ti, attention_mask=tm, max_new_tokens=T, num_beams=2),
                  lambda: model.generate(input_ids=ti, attention_mask=tm, decoder_input_ids=td[:, :3], max_new_tokens=T, min_new_tokens=5)):
        other()
        again = model.generate(input_ids=ti, attention_mask=tm, decoder_input_ids=td, **kw)
        assert np.array_equal(again.sequences.cpu().numpy(), seq) and np.array_equal(again.token_logprobs.cpu().numpy(), lp)
        assert _launches(model) == launches


# ---------------------------------------------------------------- 5. prefill against step-by-step forcing
@DTYPES
@pytest.mark.parametrize("spec_name,seed,P0", [("tiny", 1, 6), ("mini", 2, 40)])
def test_first_token_matches_step_forcing(models, dtype, spec_name, seed, P0):
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    B = 8
    ids, mask = synthetic_token_batch(B, 32, spec.vocab_size, seed=17, lengths="uniform")
    d = po.prepend_start(_prompts(B, P0, spec.vocab_size, seed=23), spec.decoder_start_token_id)
    P = d.shape[1]
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), decoder_input_ids=torch.from_numpy(d),
                         max_new_tokens=1, min_new_tokens=1, return_dict_in_generate=True, output_scores=True)
    tok = out.sequences.cpu().numpy()[:, P]
    # the decode step's head rounds each logit to the compute type before its log-softmax
    lg = model.decode_logits(ids, mask, d)[:, P - 1].to(dtype).float().cpu().numpy()
    lg[:, spec.eos_token_id] = -np.inf  # min_new_tokens=1
    want = log_softmax(lg)[np.arange(B), tok]
    got = out.token_logprobs.cpu().numpy()[:, 0]
    # the two paths differ in accumulation order only; a flip of the arg-max needs a near-tie
    top2 = np.sort(lg, axis=-1)[:, -2:]
    close = top2[:, 1] - top2[:, 0] <= TAU[dtype]
    assert ((tok == lg.argmax(-1)) | close).all()
    assert np.abs(got - want).max() <= 2 * TAU[dtype]


# ---------------------------------------------------------------- 6. the prefill's precondition
def test_prompt_rejected_when_the_wi_tile_is_not_128_rows(tmp_path, monkeypatch):
    """The prefill is the forward pass's decoder stack, whose GeGLU product reads wi through 128-row boxes: with B200T5_SK
    giving wi another tile, a prompt of two or more ids is refused with B200T5_EINVAL before anything is launched, as
    b200t5_forward refuses it."""
    from anyscale_workshop_nyc_2023_b200 import _lib
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    spec = SPECS["tiny"]
    save_checkpoint(tmp_path, spec, seed=1)
    monkeypatch.setenv("B200T5_SK", "64,2,64,4,64,2,64,4")
    model = B200T5ForConditionalGeneration.from_pretrained(tmp_path, device_map="auto", torch_dtype=torch.bfloat16)
    ids, mask = synthetic_token_batch(3, 16, spec.vocab_size, seed=2, lengths="uniform")
    d0 = _prompts(3, 4, spec.vocab_size, seed=5)
    with pytest.raises(_lib.B200T5Error, match="B200T5_SK") as e:
        model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), decoder_input_ids=d0, max_new_tokens=4)
    assert e.value.code == _lib.EINVAL and "prefixed" in str(e.value)
    with pytest.raises(_lib.B200T5Error, match="B200T5_SK") as e:
        model.generate_host(ids, mask, decoder_input_ids=d0, max_new_tokens=4)
    assert e.value.code == _lib.EINVAL
