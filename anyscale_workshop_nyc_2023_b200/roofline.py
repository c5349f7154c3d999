"""The algorithmic byte / FLOP model the roofline numbers are computed from (SURVEY section 8d), in Python.

The C library counts the same quantities while it runs (`b200t5_get_stats`: decode_algo_bytes, encoder_flops) and
`bench.py` divides them by CUDA-event times; this restatement exists so that the model itself is testable without a
GPU (tests/test_roofline_cpu.py pins it to SURVEY's table) and against the library (tests/test_model_gpu.py).
Element size 2 bytes (bf16 / fp16); activations, ids and logits are excluded, as in SURVEY 8d."""
from __future__ import annotations

import json
from pathlib import Path
from typing import Iterable, Optional, Tuple

# NVIDIA H100 SXM data sheet (a card allowed 700 W): HBM3 bandwidth and dense BF16 tensor throughput
H100_HBM_GBS = 3350.0
H100_BF16_TFLOPS = 989.0


def peaks(root: Path) -> Tuple[float, float, str]:
    """(HBM GB/s, bf16 TFLOP/s, source) the roofline fractions are taken against: the measured figures in
    `root / MEASURED_PEAKS.json` when that file exists, otherwise the H100 SXM data sheet."""
    f = Path(root) / "MEASURED_PEAKS.json"
    if f.exists():
        pk = json.loads(f.read_text())
        return float(pk["hbm_gbs"]), float(pk.get("bf16_tflops_sustained", H100_BF16_TFLOPS)), "measured (MEASURED_PEAKS.json)"
    return H100_HBM_GBS, H100_BF16_TFLOPS, "H100 SXM data sheet (HBM3 3.35 TB/s, dense BF16 989 TFLOP/s at 700 W)"


def step_weight_elements(spec) -> int:
    """W_step: decoder weights read once per decode step (self q,k,v,o + cross q,o + wi_0,wi_1,wo per layer, + lm_head);
    the cross k,v projections are prefill-only."""
    d, inner, f = spec.d_model, spec.inner_dim, spec.d_ff
    return spec.num_decoder_layers * (4 * d * inner + 2 * d * inner + 3 * d * f) + spec.vocab_size * d


def decode_bytes(spec, batch: int, steps: int, extents: Optional[Iterable[int]] = None, seq: Optional[int] = None,
                 fp32_wo: bool = False) -> float:
    """Bytes the greedy loop has to move for `steps` decode steps of a `batch`-row batch: weights once per step,
    the attended cross-KV rows (sum of extents) and the self-KV cache read (t rows at step t) and written (1 row).
    `fp32_wo`: the fp16 contract keeps `wo` in fp32 (4 bytes per weight)."""
    sum_s = float(sum(extents)) if extents is not None else float(batch) * float(seq)
    inner, ld = spec.inner_dim, spec.num_decoder_layers
    w = step_weight_elements(spec) + (ld * spec.d_model * spec.d_ff if fp32_wo else 0)
    total = 0.0
    for t in range(1, steps + 1):
        total += 2.0 * (w + ld * 2 * inner * sum_s + ld * 2 * inner * batch * t + ld * 2 * inner * batch)
    return total


def encoder_flops(spec, batch: int, extents: Optional[Iterable[int]] = None, seq: Optional[int] = None) -> float:
    """Encoder + cross-KV projection FLOPs over the positions that matter (below each row's extent)."""
    ext = list(extents) if extents is not None else [seq] * batch
    sum_s = float(sum(ext))
    sum_s2 = float(sum(e * e for e in ext))
    d, inner, f = spec.d_model, spec.inner_dim, spec.d_ff
    return (2.0 * spec.num_layers * (4 * d * inner + 3 * d * f) * sum_s + spec.num_layers * 4.0 * sum_s2 * inner
            + 2.0 * spec.num_decoder_layers * 2.0 * d * inner * sum_s)


def cross_attention_bytes_per_launch(spec, extents: Iterable[int]) -> float:
    """One launch of the roofline kernel: K and V rows (64 x 2 bytes per head) of every attended key."""
    return 2.0 * 2.0 * spec.inner_dim * float(sum(extents))
