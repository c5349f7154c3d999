"""Token log-probabilities without a GPU: the numpy score oracle (oracle/scores.py) against transformers' own
compute_transition_scores and loss (tests/golden/scores.npz, written by tests/golden/make_golden_scores.py), the layout of
b200t5_score_io, and the argument validation of the Python layer."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.modeling import (GenerateOutput, TokenScores, generate_output_flags, score_labels)
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict
from oracle import scores as oscores
from oracle.logits_process import Processors
from oracle.t5_oracle import T5Oracle

ROOT = Path(__file__).resolve().parents[1]
GOLD = np.load(ROOT / "tests" / "golden" / "scores.npz")
CASES = {"tiny": (1, 12), "mini": (2, 16)}  # spec -> weight seed, max_new_tokens
PROC = Processors(repetition_penalty=1.3, no_repeat_ngram_size=2)
# logit tolerances of tests/test_oracle_cpu.py for the emulating modes
MODES = {"fp32": (None, 1e-4), "bf16": ("bf16", 0.13), "fp16": ("fp16", 0.04)}


def _oracle(spec_name, mode):
    seed, T = CASES[spec_name]
    spec = SPECS[spec_name]
    return T5Oracle(make_state_dict(spec, seed), spec, emulate=MODES[mode][0]), T


@pytest.mark.parametrize("proc", [False, True], ids=["plain", "proc"])
@pytest.mark.parametrize("spec_name", list(CASES))
def test_fp32_oracle_reproduces_transformers_transition_scores(spec_name, proc):
    o, T = _oracle(spec_name, "fp32")
    key = f"{spec_name}_fp32{'_proc' if proc else ''}"
    toks, logits, logps, _ = oscores.generate(o, GOLD[f"{spec_name}_ids"], GOLD[f"{spec_name}_mask"], T, PROC if proc else None)
    want = GOLD[f"{key}_tokens"]
    assert toks.shape == want.shape and (toks == want).all()
    live = np.cumsum(np.pad(want[:, 1:-1] == 1, ((0, 0), (1, 0))), axis=1) == 0  # up to and including the EOS
    assert np.abs(logps - GOLD[f"{key}_logprobs"])[live].max() <= 1e-4
    assert np.abs(logits - GOLD[f"{key}_logits"])[live].max() <= 1e-4
    assert (logps[~live] == 0).all() and (logits[~live] == 0).all()  # the convention: nothing after a row's EOS
    assert (logps <= 0).all()


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
@pytest.mark.parametrize("spec_name", list(CASES))
def test_emulating_oracles_track_transformers_transition_scores(spec_name, mode):
    o, T = _oracle(spec_name, mode)
    tol = MODES[mode][1]
    for suffix, proc in (("", None), ("_proc", PROC)):
        key = f"{spec_name}_{mode}{suffix}"
        toks, logits, logps, margins = oscores.generate(o, GOLD[f"{spec_name}_ids"], GOLD[f"{spec_name}_mask"], T, proc)
        want = GOLD[f"{key}_tokens"]
        n = min(toks.shape[1], want.shape[1]) - 1
        checked = 0
        for b in range(toks.shape[0]):
            # compare a row up to its first disagreement (a near-tie resolved the other way) or its EOS
            diff = np.nonzero(toks[b, 1:n + 1] != want[b, 1:n + 1])[0]
            upto = int(diff[0]) if diff.size else n
            eos = np.nonzero(want[b, 1:upto + 1] == 1)[0]
            upto = int(eos[0]) + 1 if eos.size else upto
            if diff.size:
                assert margins[b, diff[0]] <= 2 * tol, (b, diff[0], margins[b, diff[0]])
            # a log-probability moves by at most twice the largest logit error
            assert np.abs(logps[b, :upto] - GOLD[f"{key}_logprobs"][b, :upto]).max(initial=0) <= 2 * tol
            checked += upto
        assert checked >= toks.shape[0]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("spec_name", list(CASES))
def test_oracle_score_reproduces_transformers_loss(spec_name, mode):
    o, _ = _oracle(spec_name, mode)
    labels = GOLD[f"{spec_name}_labels"]
    tol = MODES[mode][1]
    lp, loss = oscores.score(o, GOLD[f"{spec_name}_ids"], GOLD[f"{spec_name}_mask"], labels)
    assert (lp[labels == -100] == 0).all()
    assert np.abs(lp - GOLD[f"{spec_name}_{mode}_label_logprobs"]).max() <= (1e-4 if mode == "fp32" else 2 * tol)
    # transformers' bf16 / fp16 loss is itself rounded to that type
    assert abs(loss - float(GOLD[f"{spec_name}_{mode}_loss"])) <= (1e-4 if mode == "fp32" else 2 * tol)


def test_log_softmax_keeps_banned_columns_at_minus_inf():
    s = np.array([[1.0, -np.inf, 3.0], [-np.inf, 2.0, -np.inf]], dtype=np.float32)
    l = oscores.log_softmax(s)
    assert np.isneginf(l[0, 1]) and l[1, 1] == 0.0 and not np.isnan(l).any()
    assert abs(np.exp(l[0, [0, 2]]).sum() - 1) < 1e-6


def test_score_io_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _lib.ScoreIO._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200t5.h"\nint main(void) { printf("%zu", sizeof(b200t5_score_io));\n'
                   + "".join(f'printf(" %zu", offsetof(b200t5_score_io, {f}));\n' for f in fields) + "return 0; }\n")
    exe = tmp_path / "layout"
    proc = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)],
                          capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.ScoreIO)] + [getattr(_lib.ScoreIO, f).offset for f in fields]
    header = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "b200t5.h").read_text(), flags=re.S)
    body = re.search(r"typedef struct b200t5_score_io \{(.*?)\}", header, flags=re.S).group(1)
    assert re.findall(r"(\w+);", body) == fields
    for name in ("b200t5_generate_scored", "b200t5_generate_host_scored", "b200t5_generate_stream_scored", "b200t5_test_lm_score"):
        assert name in _lib.SIGNATURES and re.search(rf"\b{name}\(", header)


def test_labels_are_validated_before_any_library_call():
    lab = score_labels(np.array([[5, 6, -100], [7, 8, 9]]), 10)
    assert lab.dtype == np.int64 and lab.shape == (2, 3)
    import torch

    assert (score_labels(torch.tensor([[1, -100]]), 10) == np.array([[1, -100]])).all()
    for bad in (None, np.array([1, 2]), np.zeros((2, 0), dtype=np.int64), np.array([[1.5, 2.0]]), np.array([[10, 1]]),
                np.array([[-1, 1]]), np.array([[-100, 1]]), np.array([[1, -100, 2]])):
        with pytest.raises(ValueError):
            score_labels(bad, 10)


def test_output_flags():
    assert generate_output_flags({}) == (False, False)
    assert generate_output_flags({"return_dict_in_generate": True, "output_scores": True, "output_logits": False}) == (True, True)
    for k in ("output_logits", "output_attentions", "output_hidden_states"):
        with pytest.raises(NotImplementedError):
            generate_output_flags({"return_dict_in_generate": True, k: True})
    out = GenerateOutput("seq")
    assert out.sequences == "seq" and out.scores is None and out.token_logprobs is None and out["sequences"] == "seq"
    sc = TokenScores(np.zeros((2, 3)), np.ones((2, 3)))
    assert len(sc) == 3 and GenerateOutput("seq", sc).token_logprobs is sc.token_logprobs
