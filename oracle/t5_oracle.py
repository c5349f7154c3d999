"""CPU restatement (numpy) of the reference's hot path: T5 v1.1 encoder/decoder forward and the
greedy generation loop that `HuggingFaceModelPredictor._predict_numpy` runs through
`self.model.generate(**generate_kwargs)` (reference: NLP_workloads/Anyscale_job/predictor.py:97-102).

THIS IS TEST INFRASTRUCTURE. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import it; the product path (anyscale_workshop_nyc_2023_b200/) never does.

The arithmetic of the path is not in /root/reference: it lives in the reference's pinned,
un-vendored dependency transformers==4.27.2 (requirements.txt:168; this image carries 5.5.0, whose
T5 math is identical - SURVEY Appendix E). Each function cites the transformers source it restates
(paths relative to site-packages/transformers/, line numbers of 5.5.0):

  rms_norm            models/t5/modeling_t5.py:55-68      T5LayerNorm.forward
  gelu_new            activations.py:59-66                NewGELUActivation.forward
  relative_bucket     models/t5/modeling_t5.py:188-234    T5Attention._relative_position_bucket
  attention           models/t5/modeling_t5.py:253-344    T5Attention.forward
  ff                  models/t5/modeling_t5.py:115-132    T5DenseGatedActDense.forward
  encode / decode     models/t5/modeling_t5.py:424-498, 637-792   T5Block / T5Stack.forward
  logits              models/t5/modeling_t5.py:1107-1110  lm_head (no rescale for FLAN-T5)
  generate            generation/utils.py:2658-2841       GenerationMixin._sample (do_sample=False)
                      generation/logits_process.py:225-233  MinNewTokensLengthLogitsProcessor
                      generation/stopping_criteria.py:57-83,450-471  MaxLength / EosToken criteria

Pinning: the reference has no tests and no golden vectors for this path (SURVEY section 4), so the
oracle is pinned against outputs of the dependency itself, generated in the build container by
tests/golden/make_golden.py and committed as tests/golden/*.npz (token IDs and logits of
transformers' T5ForConditionalGeneration.generate on seeded synthetic checkpoints), plus the
known-answer vectors of SURVEY Appendix B (bucket tables, gelu_new values).

Three numerics modes:
  emulate_bf16=False  everything in fp32 (matches HF fp32 on CPU)
  emulate_bf16=True   fp32 arithmetic with a round-to-bf16 after every op where HF eager bf16
                      rounds (SURVEY Appendix A) - the contract the CUDA kernels implement.
  emulate="fp16"      the notebook's literal torch_dtype=torch.float16 (NB:882; SURVEY 8f row 1, Appendix A.7):
                      round-to-fp16 at the same points, EXCEPT that `wo` stays an fp32 weight with an fp32
                      output (`_keep_in_fp32_modules = ["wo"]`, modeling_t5.py; T5DenseGatedActDense.forward
                      casts its input up), so the residual stream is fp32 from the first feed-forward block
                      on (type promotion in T5LayerFF / T5LayerSelfAttention / T5LayerCrossAttention) and
                      T5LayerNorm rounds to fp16 only on its way out. The additive mask is finfo(fp16).min, and
                      fp16(score + mask) overflows to -inf exactly as in torch. The contract of
                      libb200t5_f16.so (DESIGN.md section 4b).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np

BF16_MIN = np.float32(-3.3895313892515355e38)
FP16_MIN = np.float32(-65504.0)
FP32_MIN = np.float32(np.finfo(np.float32).min)


def _round_bf16(x: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = (u + (np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1)))) & np.uint32(0xFFFF0000)
    return r.view(np.float32)


def _round_fp16(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        return np.asarray(x, dtype=np.float32).astype(np.float16).astype(np.float32)


def relative_bucket(rel: np.ndarray, bidirectional: bool, num_buckets: int = 32, max_distance: int = 128) -> np.ndarray:
    """T5Attention._relative_position_bucket; rel = memory_position - query_position (int array)."""
    rel = np.asarray(rel, dtype=np.int64)
    ret = np.zeros_like(rel)
    if bidirectional:
        num_buckets //= 2
        ret = ret + (rel > 0).astype(np.int64) * num_buckets
        n = np.abs(rel)
    else:
        n = -np.minimum(rel, 0)
    max_exact = num_buckets // 2
    is_small = n < max_exact
    with np.errstate(divide="ignore"):
        ratio = n.astype(np.float32) / np.float32(max_exact)
        scaled = np.log(ratio).astype(np.float32) / np.float32(math.log(max_distance / max_exact))
        scaled = scaled * np.float32(num_buckets - max_exact)
    large = max_exact + np.where(is_small, 0, scaled).astype(np.int64)  # truncation, as .to(torch.long)
    large = np.minimum(large, num_buckets - 1)
    return ret + np.where(is_small, n, large)


def gelu_new_f32(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.float32)
    c = np.float32(math.sqrt(2.0 / math.pi))
    return np.float32(0.5) * x * (np.float32(1.0) + np.tanh(c * (x + np.float32(0.044715) * (x * x * x))))


class T5Oracle:
    def __init__(self, state_dict: Dict[str, np.ndarray], spec, emulate_bf16: bool = False, emulate: Optional[str] = None):
        self.sd = {k: np.asarray(v, dtype=np.float32) for k, v in state_dict.items()}
        self.spec = spec
        self.mode = emulate if emulate is not None else ("bf16" if emulate_bf16 else "fp32")
        if self.mode not in ("fp32", "bf16", "fp16"):
            raise ValueError(self.mode)
        self.bf16 = self.mode != "fp32"  # "reduced precision": one rounding per eager op
        self.fp16 = self.mode == "fp16"
        self._round = {"fp32": lambda x: np.asarray(x, dtype=np.float32), "bf16": _round_bf16, "fp16": _round_fp16}[self.mode]
        if self.bf16:  # from_pretrained casts the fp32 checkpoint; in fp16 mode `wo` is kept in fp32
            self.sd = {k: (v if self.fp16 and k.endswith("DenseReluDense.wo.weight") else self._round(v)) for k, v in self.sd.items()}
        if "lm_head.weight" not in self.sd:  # tied checkpoint
            self.sd["lm_head.weight"] = self.sd["shared.weight"]
        self.H, self.dk = spec.num_heads, spec.d_kv
        self.mask_min = {"fp32": FP32_MIN, "bf16": BF16_MIN, "fp16": FP16_MIN}[self.mode]

    # ---- elementary ops with HF's rounding points
    def r(self, x):
        return self._round(x)

    def res_add(self, x, y):
        """Residual add under torch type promotion. x, y = (values, is_fp32). In fp16 mode the stream turns fp32 at
        the first feed-forward block (its `wo` output is fp32) and stays fp32; until then it is an fp16 add."""
        (xv, xf), (yv, yf) = x, y
        if self.fp16 and (xf or yf):
            return (xv.astype(np.float32) + yv.astype(np.float32)).astype(np.float32), True
        return self.r(xv + yv), False

    def linear(self, x, name):
        return self.r(x @ self.sd[name].T)

    def rms_norm(self, x, name):
        w = self.sd[name]
        var = np.mean(np.square(x.astype(np.float32)), axis=-1, keepdims=True, dtype=np.float32)
        y = self.r(x * (np.float32(1.0) / np.sqrt(var + np.float32(self.spec.layer_norm_epsilon))))
        return self.r(w * y)

    def gelu_new(self, x):
        if not self.bf16:
            return gelu_new_f32(x)
        r = self.r  # one rounding per eager op; torch.pow(x, 3.0) on bf16 is x*x*x in bf16 arithmetic
        half_x = r(np.float32(0.5) * x)
        # torch.pow(x, 3.0) on the CPU: bf16 -> x*x*x in bf16 arithmetic (two roundings); fp16 -> computed in fp32, one
        # rounding (measured against torch 2.11 on CPU: 0 mismatches over a 20001-point grid for the single rounding).
        # That is CPU behaviour: torch on the GPU rounds twice for fp16 too, one fp16 ulp of gelu_new away on 15 of the
        # 63,488 finite inputs (DESIGN.md 4b). The goldens and the CUDA library's fp16 build follow the CPU rounding.
        x3 = r(x * x * x) if self.fp16 else r(r(x * x) * x)
        t = r(np.float32(0.044715) * x3)
        t = r(x + t)
        t = r(np.float32(math.sqrt(2.0 / math.pi)) * t)
        t = r(np.tanh(t))
        t = r(np.float32(1.0) + t)
        return r(half_x * t)

    def ff(self, x, prefix):
        g = self.gelu_new(self.linear(x, f"{prefix}.DenseReluDense.wi_0.weight"))
        u = self.linear(x, f"{prefix}.DenseReluDense.wi_1.weight")
        h = self.r(g * u)
        if self.fp16:  # fp32 weight, input cast up, fp32 output (no rounding)
            return (h @ self.sd[f"{prefix}.DenseReluDense.wo.weight"].T).astype(np.float32)
        return self.linear(h, f"{prefix}.DenseReluDense.wo.weight")

    def _heads(self, x):  # [B,T,I] -> [B,H,T,dk]
        B, T, _ = x.shape
        return x.reshape(B, T, self.H, self.dk).transpose(0, 2, 1, 3)

    def _attend(self, q, k, v, bias_masked):
        """q [B,H,Tq,dk], k/v [B,H,Tk,dk], bias_masked broadcastable to [B,H,Tq,Tk] (already rounded)."""
        scores = self.r(np.matmul(q, k.transpose(0, 1, 3, 2)))  # no 1/sqrt(d) scaling (modeling_t5.py:308)
        scores = self.r(scores + bias_masked)
        m = scores.max(axis=-1, keepdims=True)
        e = np.exp((scores - m).astype(np.float32))
        p = self.r(e / e.sum(axis=-1, keepdims=True, dtype=np.float32))
        o = self.r(np.matmul(p, v))
        B, H, Tq, dk = o.shape
        return o.transpose(0, 2, 1, 3).reshape(B, Tq, H * dk)

    def _bias(self, side, q_pos, k_len):
        """[1,H,Tq,Tk] position bias for query positions q_pos (array) against keys 0..k_len-1."""
        table = self.sd[f"{side}.block.0.layer.0.SelfAttention.relative_attention_bias.weight"]  # [nb,H]
        rel = np.arange(k_len)[None, :] - np.asarray(q_pos)[:, None]
        bucket = relative_bucket(rel, bidirectional=(side == "encoder"),
                                 num_buckets=self.spec.relative_attention_num_buckets,
                                 max_distance=self.spec.relative_attention_max_distance)
        return table[bucket].transpose(2, 0, 1)[None]

    # ---- encoder
    def encode(self, input_ids: np.ndarray, attention_mask: Optional[np.ndarray] = None) -> np.ndarray:
        B, S = input_ids.shape
        mask = np.ones((B, S), dtype=np.int64) if attention_mask is None else attention_mask
        x = self.sd["shared.weight"][input_ids]
        add_mask = np.where(mask[:, None, None, :] != 0, np.float32(0), self.mask_min).astype(np.float32)
        pb = self.r(self._bias("encoder", np.arange(S), S) + add_mask)  # position_bias + mask (:323-325)
        xf = False  # is the residual stream fp32 (fp16 mode only)
        for i in range(self.spec.num_layers):
            p = f"encoder.block.{i}.layer"
            n = self.rms_norm(x, f"{p}.0.layer_norm.weight")
            q = self._heads(self.linear(n, f"{p}.0.SelfAttention.q.weight"))
            k = self._heads(self.linear(n, f"{p}.0.SelfAttention.k.weight"))
            v = self._heads(self.linear(n, f"{p}.0.SelfAttention.v.weight"))
            a = self.linear(self._attend(q, k, v, pb), f"{p}.0.SelfAttention.o.weight")
            x, xf = self.res_add((x, xf), (a, False))
            n = self.rms_norm(x, f"{p}.1.layer_norm.weight")
            x, xf = self.res_add((x, xf), (self.ff(n, f"{p}.1"), self.fp16))
        return self.rms_norm(x, "encoder.final_layer_norm.weight")

    # ---- decoder with KV cache
    def _init_cache(self, enc_out, mask):
        L = self.spec.num_decoder_layers
        cache = {"self_k": [None] * L, "self_v": [None] * L, "cross_k": [], "cross_v": [], "t": 0}
        for i in range(L):
            p = f"decoder.block.{i}.layer.1.EncDecAttention"
            cache["cross_k"].append(self._heads(self.linear(enc_out, f"{p}.k.weight")))
            cache["cross_v"].append(self._heads(self.linear(enc_out, f"{p}.v.weight")))
        cache["cross_bias"] = np.where(mask[:, None, None, :] != 0, np.float32(0), self.mask_min).astype(np.float32)
        return cache

    def _decode_step(self, tokens: np.ndarray, cache) -> np.ndarray:
        """tokens int64 [B] = decoder input at position t; returns logits [B,V]."""
        t = cache["t"]
        x = self.sd["shared.weight"][tokens][:, None, :]  # [B,1,d]
        self_bias = self.r(self._bias("decoder", np.array([t]), t + 1))  # + causal mask of zeros
        xf = False
        for i in range(self.spec.num_decoder_layers):
            p = f"decoder.block.{i}.layer"
            n = self.rms_norm(x, f"{p}.0.layer_norm.weight")
            q = self._heads(self.linear(n, f"{p}.0.SelfAttention.q.weight"))
            k = self._heads(self.linear(n, f"{p}.0.SelfAttention.k.weight"))
            v = self._heads(self.linear(n, f"{p}.0.SelfAttention.v.weight"))
            if t == 0:
                cache["self_k"][i], cache["self_v"][i] = k, v
            else:  # DynamicLayer.update: cat along the sequence axis (cache_utils.py:119-120)
                cache["self_k"][i] = np.concatenate([cache["self_k"][i], k], axis=2)
                cache["self_v"][i] = np.concatenate([cache["self_v"][i], v], axis=2)
            a = self._attend(q, cache["self_k"][i], cache["self_v"][i], self_bias)
            x, xf = self.res_add((x, xf), (self.linear(a, f"{p}.0.SelfAttention.o.weight"), False))
            n = self.rms_norm(x, f"{p}.1.layer_norm.weight")
            q = self._heads(self.linear(n, f"{p}.1.EncDecAttention.q.weight"))
            a = self._attend(q, cache["cross_k"][i], cache["cross_v"][i], cache["cross_bias"])
            x, xf = self.res_add((x, xf), (self.linear(a, f"{p}.1.EncDecAttention.o.weight"), False))
            n = self.rms_norm(x, f"{p}.2.layer_norm.weight")
            x, xf = self.res_add((x, xf), (self.ff(n, f"{p}.2"), self.fp16))
        x = self.rms_norm(x, "decoder.final_layer_norm.weight")
        cache["t"] = t + 1
        return self.linear(x[:, 0, :], "lm_head.weight")

    def decode_logits(self, input_ids, attention_mask, decoder_input_ids) -> np.ndarray:
        """Teacher-forced logits [B,T,V] for decoder_input_ids [B,T]."""
        mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
        cache = self._init_cache(self.encode(input_ids, mask), mask)
        out = [self._decode_step(decoder_input_ids[:, t], cache) for t in range(decoder_input_ids.shape[1])]
        return np.stack(out, axis=1)

    def generate(self, input_ids, attention_mask=None, max_new_tokens: int = 20, min_new_tokens: int = 0,
                 return_margins: bool = False) -> Tuple[np.ndarray, ...]:
        """Greedy search. Returns int64 [B, 1+T'] exactly as HF generate(): column 0 is the decoder
        start token, finished rows are padded, the loop stops when every row has emitted EOS.
        With return_margins also returns the top-1/top-2 logit gap per (row, step) (NaN once finished)."""
        sp = self.spec
        B = input_ids.shape[0]
        mask = np.ones_like(input_ids) if attention_mask is None else attention_mask
        cache = self._init_cache(self.encode(input_ids, mask), mask)
        out = np.full((B, 1), sp.decoder_start_token_id, dtype=np.int64)
        unfinished = np.ones(B, dtype=bool)
        margins = []
        tok = out[:, 0]
        for step in range(max_new_tokens):
            logits = self._decode_step(tok, cache).astype(np.float32)
            if step < min_new_tokens:
                logits[:, sp.eos_token_id] = -np.inf
            nxt = logits.argmax(axis=-1)  # first index among equal maxima, as torch.argmax
            if return_margins:
                top2 = np.partition(logits, -2, axis=-1)[:, -2:]
                margins.append(np.where(unfinished, top2[:, 1] - top2[:, 0], np.nan))
            nxt = np.where(unfinished, nxt, sp.pad_token_id)
            out = np.concatenate([out, nxt[:, None]], axis=1)
            unfinished &= nxt != sp.eos_token_id
            tok = nxt
            if not unfinished.any():
                break
        if return_margins:
            return out, np.stack(margins, axis=1)
        return (out,)
