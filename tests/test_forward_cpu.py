"""CPU-only: the FLOP count of the teacher-forced forward pass (roofline.decoder_forward_flops) against a hand count."""
import pytest

from anyscale_workshop_nyc_2023_b200 import roofline
from anyscale_workshop_nyc_2023_b200.synth import SPECS


def test_decoder_forward_flops_flan_t5_base():
    # FLAN-T5-base (d = I = 768, F = 2048, 12 decoder layers, V = 32128), 256 prompts of 512 tokens, 512 labels:
    #   products per layer and position  2 (6 * 768 * 768 + 3 * 768 * 2048)  = 16,515,072
    #   lm_head per position              2 * 768 * 32128                     = 49,348,608
    #   per position: 12 * 16,515,072 + 49,348,608 = 247,529,472; x 256 * 512 positions = 32,444,182,953,984
    #   causal self-attention  12 * 256 * 2 * 768 * 512 * 513                 =  1,239,366,500,352
    #   cross-attention        12 * 4 * 768 * 512 * (256 * 512)                =  2,473,901,162,496
    hand = 32_444_182_953_984 + 1_239_366_500_352 + 2_473_901_162_496
    assert roofline.decoder_forward_flops(SPECS["flan-t5-base"], 256, 512, seq=512) == hand
    assert hand / 1e12 == pytest.approx(36.16, abs=0.01)


def test_decoder_forward_flops_extents():
    spec = SPECS["flan-t5-base"]
    full = roofline.decoder_forward_flops(spec, 2, 7, extents=[512, 512])
    ragged = roofline.decoder_forward_flops(spec, 2, 7, extents=[512, 100])
    assert full - ragged == 12 * 4.0 * 768 * 7 * 412
    assert roofline.decoder_forward_flops(spec, 2, 7, seq=512) == full
