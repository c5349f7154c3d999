"""Seeded synthetic assets: FLAN-T5-shaped checkpoints, Alpaca-schema prompts, token batches.

No FLAN-T5 weights, tokenizer model or Alpaca data exist offline (SURVEY section 0), so every
parity and benchmark input is generated here from numpy seeds. Checkpoints are written in the
Hugging Face directory format (``config.json`` + ``model.safetensors``), i.e. what
``checkpoint.get_model(model_cls)`` hands to ``model_cls.from_pretrained``
(reference: NLP_workloads/Anyscale_job/predictor.py:68), so the same directory loads into
``transformers.T5ForConditionalGeneration`` (the oracle anchor) and into
``B200T5ForConditionalGeneration``.
"""
from __future__ import annotations

import json
import struct
from dataclasses import asdict, dataclass
from pathlib import Path
from typing import Dict, Iterable, Optional, Tuple

import numpy as np


# --------------------------------------------------------------------------- bf16 <-> fp32 (numpy)
def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even fp32 -> bf16, returned as uint16 bit patterns."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    rounded = u + (np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1)))
    out = (rounded >> np.uint32(16)).astype(np.uint16)
    nan = np.isnan(x)
    if nan.any():
        out = np.where(nan, np.uint16(0x7FC0), out)
    return out


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    return (np.ascontiguousarray(b, dtype=np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)


def round_bf16(x: np.ndarray) -> np.ndarray:
    """fp32 array whose values are exactly representable in bf16 (RNE)."""
    return bf16_bits_to_f32(f32_to_bf16_bits(x))


# --------------------------------------------------------------------------- architectures
@dataclass(frozen=True)
class T5Spec:
    """The T5Config fields the path depends on (SURVEY Appendix C)."""

    name: str
    vocab_size: int = 32128
    d_model: int = 512
    d_kv: int = 64
    d_ff: int = 1024
    num_heads: int = 6
    num_layers: int = 8
    num_decoder_layers: int = 8
    relative_attention_num_buckets: int = 32
    relative_attention_max_distance: int = 128
    layer_norm_epsilon: float = 1e-6
    pad_token_id: int = 0
    eos_token_id: int = 1
    decoder_start_token_id: int = 0
    # synthetic-weight knob (not a T5Config field): multiplier on T5's own std of the attention query projections.
    # 1.0 = modeling_t5.py:_init_weights, attention scores of unit variance, as in a trained checkpoint. The two
    # test-sized models keep the 4.0 their committed golden fixtures were generated with (peaked attention on 2-3
    # layers and short prompts); on the 12-24-layer FLAN-T5 shapes with 512 keys that setting makes the network
    # numerically chaotic - stock transformers bf16 on GPU and on CPU rarely agree on an arg-max - so no
    # implementation can be compared with another one on it.
    q_init_gain: float = 1.0

    @property
    def inner_dim(self) -> int:
        return self.num_heads * self.d_kv

    def hf_config(self) -> dict:
        return {
            "architectures": ["T5ForConditionalGeneration"],
            "model_type": "t5",
            "vocab_size": self.vocab_size,
            "d_model": self.d_model,
            "d_kv": self.d_kv,
            "d_ff": self.d_ff,
            "num_heads": self.num_heads,
            "num_layers": self.num_layers,
            "num_decoder_layers": self.num_decoder_layers,
            "relative_attention_num_buckets": self.relative_attention_num_buckets,
            "relative_attention_max_distance": self.relative_attention_max_distance,
            "layer_norm_epsilon": self.layer_norm_epsilon,
            "dropout_rate": 0.1,
            "initializer_factor": 1.0,
            "feed_forward_proj": "gated-gelu",
            "dense_act_fn": "gelu_new",
            "is_gated_act": True,
            "is_encoder_decoder": True,
            "use_cache": True,
            "tie_word_embeddings": False,
            "pad_token_id": self.pad_token_id,
            "eos_token_id": self.eos_token_id,
            "decoder_start_token_id": self.decoder_start_token_id,
            "torch_dtype": "bfloat16",
        }


SPECS: Dict[str, T5Spec] = {
    # test-sized models (same kernels, seconds on the CPU oracle)
    "tiny": T5Spec("tiny", vocab_size=384, d_model=128, d_ff=256, num_heads=2, num_layers=2, num_decoder_layers=2, q_init_gain=4.0),
    "mini": T5Spec("mini", vocab_size=1000, d_model=256, d_ff=512, num_heads=3, num_layers=3, num_decoder_layers=2, q_init_gain=4.0),
    # the FLAN-T5 family (parameter counts 76.9 M / 247.5 M / 783.0 M untied)
    "flan-t5-small": T5Spec("flan-t5-small", d_model=512, d_ff=1024, num_heads=6, num_layers=8, num_decoder_layers=8),
    "flan-t5-base": T5Spec("flan-t5-base", d_model=768, d_ff=2048, num_heads=12, num_layers=12, num_decoder_layers=12),
    "flan-t5-large": T5Spec("flan-t5-large", d_model=1024, d_ff=2816, num_heads=16, num_layers=24, num_decoder_layers=24),
}


def param_names(spec: T5Spec) -> Dict[str, Tuple[int, ...]]:
    """HF state-dict keys and shapes (SURVEY Appendix G); nn.Linear layout [out, in]."""
    d, I, F, V, H = spec.d_model, spec.inner_dim, spec.d_ff, spec.vocab_size, spec.num_heads
    nb = spec.relative_attention_num_buckets
    out: Dict[str, Tuple[int, ...]] = {"shared.weight": (V, d), "lm_head.weight": (V, d)}
    for side, n_layers in (("encoder", spec.num_layers), ("decoder", spec.num_decoder_layers)):
        for i in range(n_layers):
            p = f"{side}.block.{i}.layer"
            for w in ("q", "k", "v"):
                out[f"{p}.0.SelfAttention.{w}.weight"] = (I, d)
            out[f"{p}.0.SelfAttention.o.weight"] = (d, I)
            if i == 0:
                out[f"{p}.0.SelfAttention.relative_attention_bias.weight"] = (nb, H)
            out[f"{p}.0.layer_norm.weight"] = (d,)
            ff = 1
            if side == "decoder":
                for w in ("q", "k", "v"):
                    out[f"{p}.1.EncDecAttention.{w}.weight"] = (I, d)
                out[f"{p}.1.EncDecAttention.o.weight"] = (d, I)
                out[f"{p}.1.layer_norm.weight"] = (d,)
                ff = 2
            out[f"{p}.{ff}.DenseReluDense.wi_0.weight"] = (F, d)
            out[f"{p}.{ff}.DenseReluDense.wi_1.weight"] = (F, d)
            out[f"{p}.{ff}.DenseReluDense.wo.weight"] = (d, F)
            out[f"{p}.{ff}.layer_norm.weight"] = (d,)
        out[f"{side}.final_layer_norm.weight"] = (d,)
    return out


def make_state_dict(spec: T5Spec, seed: int = 0, eos_boost: float = 2.5) -> Dict[str, np.ndarray]:
    """Seeded random weights, already rounded to bf16-representable fp32.

    Scales follow T5's own initialisation (modeling_t5.py:_init_weights; query projections times
    spec.q_init_gain) except that the untied lm_head is N(0, d^-1/2) with the EOS row boosted, which
    gives varied output lengths instead of the degenerate all-pad generations of the default init (SURVEY 8c).
    """
    rng = np.random.default_rng(seed)
    d, I, F = spec.d_model, spec.inner_dim, spec.d_ff
    sd: Dict[str, np.ndarray] = {}
    for name, shape in param_names(spec).items():
        if name.endswith("layer_norm.weight"):
            w = 1.0 + 0.1 * rng.standard_normal(shape)
        elif name == "shared.weight":
            w = rng.standard_normal(shape)
        elif name == "lm_head.weight":
            w = rng.standard_normal(shape) * d ** -0.5
            w[spec.eos_token_id] *= eos_boost
        elif name.endswith("relative_attention_bias.weight"):
            w = rng.standard_normal(shape) * 0.5
        elif ".q.weight" in name:
            w = rng.standard_normal(shape) * (d * spec.d_kv) ** -0.5 * spec.q_init_gain
        elif ".k.weight" in name or ".v.weight" in name or "wi_" in name:
            w = rng.standard_normal(shape) * d ** -0.5
        elif ".o.weight" in name:
            w = rng.standard_normal(shape) * I ** -0.5
        elif "wo.weight" in name:
            w = rng.standard_normal(shape) * F ** -0.5
        else:  # pragma: no cover
            raise KeyError(name)
        sd[name] = round_bf16(w.astype(np.float32))
    return sd


# --------------------------------------------------------------------------- safetensors (minimal reader/writer)
_ST_DTYPES = {"BF16": 2, "F16": 2, "F32": 4}


def write_safetensors(path: Path, tensors: Dict[str, np.ndarray], dtype: str = "BF16") -> None:
    header, blobs, off = {}, [], 0
    for name in sorted(tensors):
        a = np.ascontiguousarray(tensors[name], dtype=np.float32)
        if dtype == "BF16":
            raw = f32_to_bf16_bits(a).tobytes()
        elif dtype == "F16":
            raw = a.astype(np.float16).tobytes()
        elif dtype == "F32":
            raw = a.tobytes()
        else:
            raise ValueError(dtype)
        header[name] = {"dtype": dtype, "shape": list(a.shape), "data_offsets": [off, off + len(raw)]}
        off += len(raw)
        blobs.append(raw)
    header["__metadata__"] = {"format": "pt"}
    hj = json.dumps(header, separators=(",", ":")).encode()
    hj += b" " * ((8 - len(hj) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hj)))
        f.write(hj)
        for b in blobs:
            f.write(b)


def read_safetensors(path: Path) -> Dict[str, Tuple[str, Tuple[int, ...], np.ndarray]]:
    """name -> (dtype string, shape, raw little-endian array: uint16 for BF16, float16, float32)."""
    data = np.memmap(path, dtype=np.uint8, mode="r")
    (hlen,) = struct.unpack("<Q", bytes(data[:8]))
    header = json.loads(bytes(data[8: 8 + hlen]).decode())
    base = 8 + hlen
    out = {}
    for name, meta in header.items():
        if name == "__metadata__":
            continue
        dt, shape = meta["dtype"], tuple(meta["shape"])
        b, e = meta["data_offsets"]
        if dt not in _ST_DTYPES:
            raise ValueError(f"{name}: unsupported safetensors dtype {dt}")
        np_dt = {"BF16": np.uint16, "F16": np.float16, "F32": np.float32}[dt]
        arr = np.frombuffer(data[base + b: base + e], dtype=np_dt).reshape(shape)
        out[name] = (dt, shape, arr)
    return out


def load_state_dict_f32(ckpt_dir: Path) -> Dict[str, np.ndarray]:
    out = {}
    for name, (dt, _shape, arr) in read_safetensors(Path(ckpt_dir) / "model.safetensors").items():
        out[name] = bf16_bits_to_f32(arr) if dt == "BF16" else np.asarray(arr, dtype=np.float32)
    return out


def save_checkpoint(ckpt_dir: Path, spec: T5Spec, seed: int = 0, dtype: str = "BF16",
                    state_dict: Optional[Dict[str, np.ndarray]] = None) -> Path:
    ckpt_dir = Path(ckpt_dir)
    ckpt_dir.mkdir(parents=True, exist_ok=True)
    sd = state_dict if state_dict is not None else make_state_dict(spec, seed)
    write_safetensors(ckpt_dir / "model.safetensors", sd, dtype)
    (ckpt_dir / "config.json").write_text(json.dumps(spec.hf_config(), indent=1))
    gen = {
        "decoder_start_token_id": spec.decoder_start_token_id,
        "eos_token_id": spec.eos_token_id,
        "pad_token_id": spec.pad_token_id,
    }
    (ckpt_dir / "generation_config.json").write_text(json.dumps(gen, indent=1))
    (ckpt_dir / "b200t5_synth.json").write_text(json.dumps({"spec": asdict(spec), "seed": seed}, indent=1))
    return ckpt_dir


def spec_from_config(cfg: dict, name: str = "from-config") -> T5Spec:
    return T5Spec(
        name=name,
        vocab_size=cfg["vocab_size"], d_model=cfg["d_model"], d_kv=cfg["d_kv"], d_ff=cfg["d_ff"],
        num_heads=cfg["num_heads"], num_layers=cfg["num_layers"],
        num_decoder_layers=cfg.get("num_decoder_layers") or cfg["num_layers"],
        relative_attention_num_buckets=cfg.get("relative_attention_num_buckets", 32),
        relative_attention_max_distance=cfg.get("relative_attention_max_distance", 128),
        layer_norm_epsilon=cfg.get("layer_norm_epsilon", 1e-6),
        pad_token_id=cfg.get("pad_token_id", 0), eos_token_id=cfg.get("eos_token_id", 1),
        decoder_start_token_id=cfg.get("decoder_start_token_id", cfg.get("pad_token_id", 0)),
    )


# --------------------------------------------------------------------------- token batches and prompts
def synthetic_token_batch(B: int, S: int, vocab: int, seed: int, lengths: str = "uniform",
                          min_len: int = 2) -> Tuple[np.ndarray, np.ndarray]:
    """ids / attention_mask int64 [B,S] as the reference's tokenizer emits them: valid tokens
    uniform in [3, min(vocab, 32000)), the last valid token is EOS (1), right-padded with 0
    (JOB/utils.py:23-29 semantics; SURVEY 8d). lengths: "full" | "uniform" | "alpaca"."""
    rng = np.random.default_rng(seed)
    hi = min(vocab, 32000)
    ids = rng.integers(3, hi, size=(B, S), dtype=np.int64)
    if lengths == "full":
        lens = np.full(B, S, dtype=np.int64)
    elif lengths == "uniform":
        lens = rng.integers(min_len, S + 1, size=B)
    elif lengths == "alpaca":  # log-normal, median ~40 tokens, clipped to S
        lens = np.clip(np.round(np.exp(rng.normal(np.log(40.0), 0.6, size=B))), min_len, S).astype(np.int64)
    else:
        raise ValueError(lengths)
    pos = np.arange(S)[None, :]
    mask = (pos < lens[:, None]).astype(np.int64)
    ids = ids * mask
    ids[np.arange(B), lens - 1] = 1
    return ids, mask


_VERBS = ["Describe", "Explain", "Summarize", "List", "Translate", "Rewrite", "Classify", "Compare", "Generate", "Identify"]
_TOPICS = ["the water cycle", "a healthy breakfast", "the theory of relativity", "three primary colors", "a short poem",
           "the causes of inflation", "renewable energy", "a famous painting", "the rules of chess", "a job interview"]
_INPUTS = ["", "", "", "The quick brown fox jumps over the lazy dog.", "2, 4, 8, 16", "Paris is the capital of France.",
           "apples, oranges, bananas", "She sells sea shells by the sea shore."]


def synthetic_alpaca_rows(n: int, seed: int = 57) -> Dict[str, list]:
    """Column dict with the tatsu-lab/alpaca schema the notebook uses (instruction, input, output, text)."""
    rng = np.random.default_rng(seed)
    cols = {"instruction": [], "input": [], "output": [], "text": []}
    for _ in range(n):
        ins = f"{_VERBS[rng.integers(len(_VERBS))]} {_TOPICS[rng.integers(len(_TOPICS))]} in {int(rng.integers(1, 6))} sentences."
        inp = _INPUTS[rng.integers(len(_INPUTS))]
        out = f"{_TOPICS[rng.integers(len(_TOPICS))].capitalize()} is an example."
        cols["instruction"].append(ins)
        cols["input"].append(inp)
        cols["output"].append(out)
        cols["text"].append(f"### Instruction:\n{ins}\n\n### Input:\n{inp}\n\n### Response:\n{out}")
    return cols
