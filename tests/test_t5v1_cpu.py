"""CPU-only: the original T5 (v1.0) architecture - ReLU feed-forward, tied and rescaled head.

The oracle restatement (tests/t5v1_oracle.py) against transformers' T5ForConditionalGeneration on the same synthetic
checkpoints, the architecture check of modeling.py, and the roofline model's ReLU counts against a hand count."""
import json

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import roofline
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, param_names, save_checkpoint, synthetic_token_batch
from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits
from t5v1_oracle import load_hf_model, oracle_for

FLAN = ("tiny", "mini", "flan-t5-small", "flan-t5-base", "flan-t5-large")


@pytest.mark.parametrize("name", ["t5-tiny", "t5-tiny-untied", "t5-mini", "t5-small", "t5-base"])
def test_v1_specs(name):
    spec = SPECS[name]
    names = param_names(spec)
    cfg = spec.hf_config()
    assert cfg["feed_forward_proj"] == "relu" and cfg["dense_act_fn"] == "relu" and cfg["is_gated_act"] is False
    assert not any("wi_0" in k or "wi_1" in k for k in names)
    assert sum(k.endswith("DenseReluDense.wi.weight") for k in names) == spec.num_layers + spec.num_decoder_layers
    assert ("lm_head.weight" in names) == (name == "t5-tiny-untied")
    assert cfg["tie_word_embeddings"] is (name != "t5-tiny-untied")


def test_flan_specs_keep_their_architecture():
    for name in FLAN:
        cfg = SPECS[name].hf_config()
        assert cfg["feed_forward_proj"] == "gated-gelu" and cfg["tie_word_embeddings"] is False
        assert "lm_head.weight" in param_names(SPECS[name])


@pytest.mark.parametrize("name", ["t5-tiny", "t5-tiny-untied"])
def test_oracle_matches_transformers_fp32(tmp_path, name):
    spec = SPECS[name]
    save_checkpoint(tmp_path, spec, seed=3)
    hf = load_hf_model(tmp_path)
    assert hf.config.scale_decoder_outputs is (name == "t5-tiny")
    o = oracle_for(name, 3, emulate="fp32")
    ids, mask = synthetic_token_batch(4, 24, spec.vocab_size, seed=5, lengths="uniform")
    want = hf_generate(hf, ids, mask, max_new_tokens=10)
    (got,) = o.generate(ids, mask, max_new_tokens=10)
    assert got.shape == want.shape and (got == want).all()
    (forced,) = o.generate(ids, mask, max_new_tokens=10, min_new_tokens=10)
    logits = o.decode_logits(ids, mask, forced[:, :-1])
    ref = hf_teacher_forced_logits(hf, ids, mask, forced[:, :-1])
    assert np.abs(logits - ref).max() <= 1e-4


@pytest.mark.parametrize("name", ["t5-tiny", "t5-tiny-untied"])
@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_oracle_tracks_transformers_reduced_precision(tmp_path, name, mode):
    """Same rounding points as transformers eager in bf16 / fp16 (with the fp32 `wo`): greedy tokens are equal up to
    each row's first near-tie (the margin gate of the GPU tests) and the logits agree within the tolerance the FLAN
    oracle tests use."""
    spec = SPECS[name]
    save_checkpoint(tmp_path, spec, seed=3)
    dtype = torch.bfloat16 if mode == "bf16" else torch.float16
    hf = load_hf_model(tmp_path, dtype=dtype)
    o = oracle_for(name, 3, emulate=mode)
    ids, mask = synthetic_token_batch(4, 24, spec.vocab_size, seed=5, lengths="uniform")
    want = hf_generate(hf, ids, mask, max_new_tokens=10)
    got, margins = o.generate(ids, mask, max_new_tokens=10, return_margins=True)
    assert got.shape == want.shape
    tau = 0.13 if mode == "bf16" else 0.03
    for b in range(got.shape[0]):
        low = [s for s in range(margins.shape[1]) if not np.isnan(margins[b, s]) and not margins[b, s] > tau]
        upto = 1 + (low[0] if low else margins.shape[1])
        assert (got[b, :upto] == want[b, :upto]).all(), b
    logits = o.decode_logits(ids, mask, got[:, :-1])
    ref = hf_teacher_forced_logits(hf, ids, mask, got[:, :-1])
    err = np.abs(logits - ref)
    assert err.max() <= (0.13 if mode == "bf16" else 0.04)


def test_rescale_is_one_rounding_of_an_fp32_product():
    """The tied head's input is round(round(w * n) * fp32(d ** -0.5)): what torch computes for a 2-byte tensor times a
    Python float, which is not the product with the scale rounded to the 2-byte type first."""
    d = 768
    s = np.float32(d ** -0.5)
    rng = np.random.default_rng(0)
    for dtype in (torch.bfloat16, torch.float16):
        y = torch.from_numpy(rng.standard_normal(1 << 16).astype(np.float32)).to(dtype)
        want = (y * (d ** -0.5)).float().numpy()
        got = torch.from_numpy(y.float().numpy() * s).to(dtype).float().numpy()
        assert (got == want).all()


def _model_cls():
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    return B200T5ForConditionalGeneration


@pytest.mark.parametrize("ffp", ["gated-silu", "gelu", "silu", "gated-relu", "Relu"])
def test_unsupported_feed_forward_raises_before_the_library(tmp_path, monkeypatch, ffp):
    from anyscale_workshop_nyc_2023_b200 import _lib

    def no_library(*a, **k):  # pragma: no cover - reaching it is the failure
        raise AssertionError("the library was called")

    monkeypatch.setattr(_lib, "load", no_library)
    cfg = dict(SPECS["t5-tiny"].hf_config(), feed_forward_proj=ffp)
    with pytest.raises(ValueError, match=repr(ffp)):
        _model_cls()(cfg, torch.device("cuda", 0))
    save_checkpoint(tmp_path, SPECS["t5-tiny"], seed=0)
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match=repr(ffp)):
        _model_cls().from_pretrained(tmp_path)


def test_feed_forward_mapping():
    from anyscale_workshop_nyc_2023_b200.modeling import _is_gated_gelu

    assert _is_gated_gelu({"feed_forward_proj": "gated-gelu"}) == 1
    assert _is_gated_gelu({"feed_forward_proj": "relu"}) == 0
    assert _is_gated_gelu({}) == 0  # transformers' default, as in the original t5-small / t5-base configs


def test_roofline_relu_counts_by_hand():
    spec = SPECS["t5-base"]  # d = I = 768, F = 3072, 12 + 12 layers, V = 32128
    # per decoder layer: 6 d I attention weights + 2 d F feed-forward weights; + the lm_head
    w = 12 * (6 * 768 * 768 + 2 * 768 * 3072) + 32128 * 768
    assert roofline.step_weight_elements(spec) == w == 123_764_736
    # one step of 4 rows over 100 keys each: weights, cross K/V, self K/V read (t = 1) and written
    assert roofline.decode_bytes(spec, 4, 1, extents=[100] * 4) == 2.0 * (w + 12 * 2 * 768 * 400 + 12 * 2 * 768 * 4 * 2)
    # fp16 contract: `wo` (d x F per layer) counted twice
    assert roofline.decode_bytes(spec, 4, 1, extents=[100] * 4, fp32_wo=True) - roofline.decode_bytes(spec, 4, 1, extents=[100] * 4) == 2.0 * 12 * 768 * 3072
    # encoder: 2 (4 d I + 2 d F) per position and layer, attention 4 I S^2 per layer, cross K/V 2 * 2 d I per decoder layer
    enc = 2.0 * 12 * (4 * 768 * 768 + 2 * 768 * 3072) * 512 + 12 * 4.0 * 512 * 512 * 768 + 2.0 * 12 * 2.0 * 768 * 768 * 512
    assert roofline.encoder_flops(spec, 1, seq=512) == enc
    # forward pass, 2 rows x 4 positions: per position and decoder layer 2 (6 d I + 2 d F), the lm_head 2 d V; attention
    fwd = 8 * (12 * 2.0 * (6 * 768 * 768 + 2 * 768 * 3072) + 2.0 * 768 * 32128) + 12 * (2 * 2.0 * 768 * 4 * 5 + 4.0 * 768 * 4 * 200)
    assert roofline.decoder_forward_flops(spec, 2, 4, extents=[100, 100]) == fwd


def test_t5_base_and_flan_t5_base_feed_forward_are_the_same_size():
    v1, flan = SPECS["t5-base"], SPECS["flan-t5-base"]
    assert roofline.ff_matrices(v1) * v1.d_ff == roofline.ff_matrices(flan) * flan.d_ff == 3 * 2048
    assert roofline.step_weight_elements(v1) == roofline.step_weight_elements(flan)
