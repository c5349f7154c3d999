"""The original T5 (v1.0) on top of the numpy oracle and the transformers anchor. TEST INFRASTRUCTURE.

oracle/t5_oracle.py restates T5 v1.1 / FLAN-T5, the reference's model, and every existing test compares against it as
it is; it is left unchanged. A v1.0 checkpoint differs in two places, restated here at transformers' rounding points
(paths relative to site-packages/transformers/, line numbers of 5.5.0):

  ff          models/t5/modeling_t5.py:84-100     T5DenseActDense.forward: act(relu(wi x)), cast to `wo`'s dtype, wo
  rescale     models/t5/modeling_t5.py:1107-1108  sequence_output * (self.model_dim ** -0.5) when
              models/t5/configuration_t5.py:82    scale_decoder_outputs, i.e. unless the config says
                                                  tie_word_embeddings: false

The head is the shared embedding when the checkpoint has no lm_head.weight (T5Oracle already ties it).
"""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

from anyscale_workshop_nyc_2023_b200.synth import SPECS, load_state_dict_f32, make_state_dict
from oracle import hf_anchor
from oracle.t5_oracle import T5Oracle


class T5v1Oracle(T5Oracle):
    """T5Oracle for either architecture: spec.feed_forward_proj "relu" runs T5DenseActDense, and a tied spec scales
    the final decoder norm's output by fp32(d_model ** -0.5), rounded once in the compute dtype."""

    def __init__(self, state_dict, spec, emulate_bf16: bool = False, emulate=None):
        super().__init__(state_dict, spec, emulate_bf16=emulate_bf16, emulate=emulate)
        self.scale = np.float32(spec.d_model ** -0.5) if spec.tie_word_embeddings else None

    def ff(self, x, prefix):
        if spec_gated(self.spec):
            return super().ff(x, prefix)
        h = self.linear(x, f"{prefix}.DenseReluDense.wi.weight")
        h = np.where(h < 0, np.float32(0), h)  # relu of the rounded product: exact in any dtype
        if self.fp16:  # fp32 weight, input cast up, fp32 output (no rounding)
            return (h @ self.sd[f"{prefix}.DenseReluDense.wo.weight"].T).astype(np.float32)
        return self.linear(h, f"{prefix}.DenseReluDense.wo.weight")

    def rms_norm(self, x, name):
        y = super().rms_norm(x, name)
        if self.scale is not None and name == "decoder.final_layer_norm.weight":
            y = self.r(y * self.scale)
        return y


def spec_gated(spec) -> bool:
    return spec.feed_forward_proj == "gated-gelu"


def oracle_for(spec_name: str, seed: int, emulate: str = "bf16") -> T5v1Oracle:
    return T5v1Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate=emulate)


def load_hf_model(ckpt_dir, dtype=torch.float32, device="cpu"):
    """transformers.T5ForConditionalGeneration on a synthetic checkpoint of either architecture. A checkpoint with an
    lm_head.weight is hf_anchor.load_hf_model (the head untied after construction). A tied one is built from its
    config as saved, so that T5Config derives scale_decoder_outputs from it, and keeps the forced tie."""
    ckpt_dir = Path(ckpt_dir)
    sd32 = load_state_dict_f32(ckpt_dir)
    if "lm_head.weight" in sd32:
        return hf_anchor.load_hf_model(ckpt_dir, dtype=dtype, device=device)
    from transformers import T5Config, T5ForConditionalGeneration

    cfg = json.loads((ckpt_dir / "config.json").read_text())
    for k in ("architectures", "model_type", "torch_dtype", "dense_act_fn", "is_gated_act"):
        cfg.pop(k, None)
    config = T5Config(**cfg)
    assert config.scale_decoder_outputs
    config._attn_implementation = "eager"
    with torch.device("cpu"):
        model = T5ForConditionalGeneration(config)
    sd = {k: torch.from_numpy(np.array(v)) for k, v in sd32.items()}
    sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    sd["decoder.embed_tokens.weight"] = sd["shared.weight"]
    missing, unexpected = model.load_state_dict(sd, strict=False)
    missing = [m for m in missing if m != "lm_head.weight"]
    assert not missing and not unexpected, (missing, unexpected)
    assert model.lm_head.weight.data_ptr() == model.shared.weight.data_ptr()  # tied
    model = model.to(dtype=dtype, device=device).eval()
    if dtype == torch.float16:  # _keep_in_fp32_modules = ["wo"], as hf_anchor does
        for name, mod in model.named_modules():
            if name.endswith("DenseReluDense.wo"):
                mod.weight = torch.nn.Parameter(sd[f"{name}.weight"].to(device=device, dtype=torch.float32).clone(), requires_grad=False)
    model.generation_config.decoder_start_token_id = config.decoder_start_token_id
    model.generation_config.eos_token_id = config.eos_token_id
    model.generation_config.pad_token_id = config.pad_token_id
    return model
