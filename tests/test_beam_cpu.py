"""Beam search without a GPU: the numpy beam oracle (oracle/beam.py) against transformers' own generate(num_beams=...)
(tests/golden/beam.npz, written by tests/golden/make_golden_beam.py), the layouts of b200t5_beam_params / b200t5_beam_io,
and the argument checks of the Python layer."""
import ctypes as C
import json
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.modeling import MAX_BEAMS, beam_params
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict
from oracle.beam import beam_search
from oracle.t5_oracle import T5Oracle

ROOT = Path(__file__).resolve().parents[1]
GOLD = np.load(ROOT / "tests" / "golden" / "beam.npz")
CASES = [json.loads(str(c)) for c in GOLD["cases"]]
CKPT = {"tiny": (1, 12), "mini": (2, 16)}  # weight seed, max_new_tokens of make_golden_beam.py


def _run(i, **kw):
    name, k, n, lp, es, mn = CASES[i]
    seed, T = CKPT[name]
    o = T5Oracle(make_state_dict(SPECS[name], seed), SPECS[name])
    return beam_search(o, GOLD[f"{name}_ids"], GOLD[f"{name}_mask"], num_beams=k, max_new_tokens=T, min_new_tokens=mn,
                       num_return_sequences=n, length_penalty=lp, early_stopping=es, **kw)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c[0]}-k{c[1]}-n{c[2]}-lp{c[3]}-es{c[4]}-min{c[5]}" for c in CASES])
def test_fp32_oracle_reproduces_transformers_beam_search(i):
    r = _run(i, division="true")  # the golden ran on the CPU, where torch divides by the length penalty
    seq, bidx = GOLD[f"c{i}_sequences"], GOLD[f"c{i}_beam_indices"]
    assert r["sequences"].shape == seq.shape and (r["beam_indices"] == bidx).all()
    # transformers 5.5 fills a hypothesis' tail with EOS when pad_token_id is 0 (`pad or eos`); here it is pad_token_id
    inside = np.arange(seq.shape[1])[None, :] <= r["lengths"][:, None]
    assert (r["sequences"][inside] == seq[inside]).all() and (r["sequences"][~inside] == 0).all()
    assert (r["lengths"] == (bidx >= 0).sum(axis=1)).all()
    want = GOLD[f"c{i}_sequences_scores"]
    assert np.abs(r["sequences_scores"] - want).max() <= 1e-5 * np.maximum(1.0, np.abs(want)).max()
    assert np.abs(r["token_logprobs"] - GOLD[f"c{i}_token_logprobs"]).max() <= 1e-4


def test_golden_covers_the_contract():
    ks = {c[1] for c in CASES}
    assert ks == {2, 4} and {c[3] for c in CASES} >= {1.0, 0.0, 2.0, -0.5}
    assert {json.dumps(c[4]) for c in CASES} == {"false", "true", '"never"'}
    assert any(c[2] == 1 for c in CASES) and any(c[2] == c[1] for c in CASES) and any(c[5] > 0 for c in CASES)
    # natural EOS: some returned hypotheses end before max_new_tokens
    assert any(((GOLD[f"c{i}_beam_indices"] >= 0).sum(axis=1) < GOLD[f"c{i}_beam_indices"].shape[1]).any() for i in range(len(CASES)))


@pytest.mark.parametrize("i", [1, 3, 6])
def test_retiring_finished_prompts_changes_nothing(i):
    """The device retires a prompt whose heuristic failed or whose set is full under early_stopping=True; transformers
    keeps decoding it. Decoding every prompt to max_new_tokens gives the same results."""
    a, b = _run(i), _run(i, stop_when_done=False)
    for key in ("sequences", "lengths", "sequences_scores", "beam_indices", "token_logprobs"):
        assert np.array_equal(a[key], b[key]), key


def _layout(tmp_path, struct, cls):
    fields = [f for f, _ in cls._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200t5.h"\n'
                   f'int main(void) {{ printf("%zu", sizeof({struct}));\n'
                   + "".join(f'printf(" %zu", offsetof({struct}, {f}));\n' for f in fields) + "return 0; }\n")
    exe = tmp_path / "layout"
    proc = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)],
                          capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(cls)] + [getattr(cls, f).offset for f in fields]
    header = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "b200t5.h").read_text(), flags=re.S)
    body = re.search(rf"typedef struct {struct} \{{(.*?)\}}", header, flags=re.S).group(1)
    assert re.findall(r"(\w+);", body) == fields


def test_beam_structs_match_the_header(tmp_path):
    _layout(tmp_path, "b200t5_beam_params", _lib.BeamParams)
    _layout(tmp_path, "b200t5_beam_io", _lib.BeamIO)
    header = (ROOT / "include" / "b200t5.h").read_text()
    for name in ("b200t5_generate_beam", "b200t5_generate_host_beam", "b200t5_get_beam_stats", "b200t5_test_beam_step",
                 "b200t5_test_beam_reorder"):
        assert name in _lib.SIGNATURES and re.search(rf"\b{name}\(", header)


def test_beam_arguments_are_checked_before_any_library_call():
    V = 100
    assert beam_params(1, {}, None, 1, V) is None and beam_params(None, {"length_penalty": 2.0}, None, 1, V) is None
    p = beam_params(4, {"num_return_sequences": 2, "length_penalty": -0.5, "early_stopping": "never"}, [1], 1, V)
    assert (p.num_beams, p.num_return_sequences, p.length_penalty, p.early_stopping) == (4, 2, -0.5, 2)
    p = beam_params(2, {"early_stopping": True, "repetition_penalty": 1.0, "suppress_tokens": []}, None, 1, V)
    assert (p.num_return_sequences, p.length_penalty, p.early_stopping) == (1, 1.0, 1)
    for kw in ({"num_return_sequences": 5}, {"num_return_sequences": 0}, {"early_stopping": "sometimes"},
               {"early_stopping": 3}, {"length_penalty": float("nan")}):
        with pytest.raises(ValueError):
            beam_params(4, kw, None, 1, V)
    for nb in (0, -2, 2.5):
        with pytest.raises(ValueError):
            beam_params(nb, {}, None, 1, V)
    with pytest.raises(NotImplementedError, match="num_beams"):
        beam_params(MAX_BEAMS + 1, {}, None, 1, V)
    with pytest.raises(NotImplementedError, match="eos_token_id"):
        beam_params(4, {}, [1, 2], 1, V)
    for name, v in (("repetition_penalty", 1.3), ("no_repeat_ngram_size", 2), ("bad_words_ids", [[5]]), ("suppress_tokens", [7]),
                    ("encoder_repetition_penalty", 0.9), ("encoder_no_repeat_ngram_size", 3), ("begin_suppress_tokens", [3])):
        with pytest.raises(NotImplementedError, match=name):
            beam_params(4, {name: v}, None, 1, V)
