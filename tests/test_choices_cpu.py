"""Multiple-choice scoring (`score_choices`) without a GPU: the numpy oracle's teacher forcing over candidate targets
against transformers' `T5ForConditionalGeneration(..., labels=...)`, the three forms of `choices` and their validation
(choice_targets), the reduction to ChoiceScores (choice_scores), and the C declaration of b200t5_forward_choices."""
import re
from pathlib import Path

import numpy as np
import pytest

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from oracle import scores as oscores
from oracle.t5_oracle import T5Oracle

torch = pytest.importorskip("torch")

from anyscale_workshop_nyc_2023_b200.modeling import ChoiceScores, choice_scores, choice_targets  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
V = 100


def test_shared_forms():
    cands = [[5, 6, 7], [8], [9, 10]]
    want = np.array([[5, 6, 7], [8, -100, -100], [9, 10, -100]], np.int64)
    for form in (cands, want, torch.from_numpy(want), [np.array(c) for c in cands]):
        lab, counts = choice_targets(form, 4, V)
        assert lab.dtype == np.int64 and (lab == np.tile(want, (4, 1))).all()
        assert counts.tolist() == [3, 3, 3, 3]


def test_per_prompt_and_ragged_forms():
    per = np.array([[[1, 2], [3, -100]], [[4, -100], [5, 6]]], np.int64)
    lab, counts = choice_targets(per, 2, V)
    assert (lab == per.reshape(4, 2)).all() and counts.tolist() == [2, 2]
    lab, counts = choice_targets(torch.from_numpy(per), 2, V)
    assert (lab == per.reshape(4, 2)).all()
    ragged = [[[1, 2, 3]], [[4], [5, 6], [7]], [[8, 9]]]
    lab, counts = choice_targets(ragged, 3, V)
    assert counts.tolist() == [1, 3, 1]
    assert lab.tolist() == [[1, 2, 3], [4, -100, -100], [5, 6, -100], [7, -100, -100], [8, 9, -100]]


@pytest.mark.parametrize("bad", [
    [],                                            # no candidate
    [[1, 2], []],                                  # an empty candidate
    [[1, V]],                                      # id outside the vocabulary
    [[1, -100]],                                   # -100 in a list form
    [[1, -3]],
    np.array([[-100, 1]]),                         # -100 before the first token
    np.array([[1, -100, 2]]),                      # -100 before a token
    np.array([[1, V]]),
    np.zeros((0, 3), np.int64),
    np.array([[1.0, 2.0]]),                        # not integers
    np.zeros((2, 2, 2, 2), np.int64) + 1,          # too many dimensions
    np.ones((3, 2, 2), np.int64),                  # [B, C, L] with B != 2
    [[[1]], [[2]], [[3]]],                         # ragged, 3 lists for 2 prompts
    [[[1]], []],                                   # ragged, a prompt without candidates
])
def test_validation(bad):
    with pytest.raises(ValueError):
        choice_targets(bad, 2, V)


def test_scores_reduction_ties_and_normalize():
    # prompt 0: three candidates, 0 and 2 tie on the sum; prompt 1: one candidate (ragged, Cmax = 3)
    lab = np.array([[1, 2, -100], [3, -100, -100], [4, 5, 6], [7, 8, 9]], np.int64)
    tlp = torch.tensor([[-1.0, -1.0, 0], [-1.5, 0, 0], [-0.5, -0.5, -1.0], [-3.0, -2.0, -1.0]])
    r = choice_scores(tlp, lab, np.array([3, 1]))
    assert isinstance(r, ChoiceScores) and r["best"] is r.best
    assert r.token_logprobs.shape == (2, 3, 3) and r.lengths.dtype == torch.int32 and r.best.dtype == torch.int64
    assert r.lengths.tolist() == [[2, 1, 3], [3, 0, 0]]
    assert torch.equal(r.token_logprobs[0], tlp[:3]) and torch.equal(r.token_logprobs[1, 0], tlp[3])
    assert (r.token_logprobs[1, 1:] == 0).all()
    assert r.logprobs[0].tolist() == [-2.0, -1.5, -2.0] and r.logprobs[1, 0] == -6.0
    assert torch.isinf(r.logprobs[1, 1:]).all() and (r.logprobs[1, 1:] < 0).all()
    assert r.best.tolist() == [1, 0]
    n = choice_scores(tlp, lab, np.array([3, 1]), normalize=True)
    # means: -1.0, -1.5, -0.667: candidate 2; the absent ones are never chosen
    assert n.best.tolist() == [2, 0] and torch.equal(n.logprobs, r.logprobs)
    # exact ties go to the lowest index
    t = choice_scores(torch.tensor([[-1.0, -1.0], [-2.0, 0.0], [-2.0, 0.0]]), np.array([[1, 2], [1, -100], [1, -100]]), np.array([3]))
    assert t.best.tolist() == [0]
    tn = choice_scores(torch.tensor([[-1.0, -1.0], [-1.0, 0.0]]), np.array([[1, 2], [1, -100]]), np.array([2]), normalize=True)
    assert tn.best.tolist() == [0]


def test_log_likelihood_is_summed_in_double():
    L = 64
    tlp = torch.full((1, L), -0.1) + torch.linspace(0, 1e-3, L)
    r = choice_scores(tlp, np.ones((1, L), np.int64), np.array([1]))
    assert r.logprobs[0, 0].item() == np.float32(tlp.double().sum().item())


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    pytest.importorskip("transformers")
    from oracle.hf_anchor import load_hf_model

    spec = SPECS["tiny"]
    d = tmp_path_factory.mktemp("choices_tiny")
    save_checkpoint(d, spec, seed=1, dtype="F32")
    return load_hf_model(d), T5Oracle(make_state_dict(spec, 1), spec)


def test_oracle_teacher_forcing_matches_transformers_on_candidates(pair):
    """The oracle's restated teacher forcing (oracle.scores.score) on prompts repeated once per candidate equals
    transformers' per-token log-softmax of `model(..., labels=...)`, so it can anchor score_choices on the GPU."""
    hf, oracle = pair
    spec = SPECS["tiny"]
    B, S = 3, 14
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=5, lengths="uniform")
    rng = np.random.default_rng(3)
    ragged = [[list(rng.integers(2, spec.vocab_size, size=rng.integers(1, 6))) for _ in range(c)] for c in (2, 4, 1)]
    ragged = [[[int(t) for t in c] for c in g] for g in ragged]
    lab, counts = choice_targets(ragged, B, spec.vocab_size)
    rep_ids, rep_mask = np.repeat(ids, counts, 0), np.repeat(mask, counts, 0)
    ours, _ = oscores.score(oracle, rep_ids, rep_mask, lab)
    with torch.no_grad():
        out = hf(input_ids=torch.from_numpy(rep_ids), attention_mask=torch.from_numpy(rep_mask), labels=torch.from_numpy(lab))
    lsm = torch.log_softmax(out.logits.float(), -1)
    on = lab != -100
    ref = torch.gather(lsm, 2, torch.from_numpy(np.where(on, lab, 0))[..., None])[..., 0].numpy() * on
    assert np.abs(ours - ref).max() <= 1e-4
    r = choice_scores(torch.from_numpy(ours), lab, counts)
    r_hf = choice_scores(torch.from_numpy(ref.astype(np.float32)), lab, counts)
    gap = np.sort(r_hf.logprobs.numpy(), 1)
    sep = np.isinf(gap[:, -2]) | (gap[:, -1] - gap[:, -2] > 1e-3)
    assert (r.best.numpy() == r_hf.best.numpy())[sep].all()


def test_c_declaration_and_binding():
    h = (ROOT / "include" / "b200t5.h").read_text()
    decl = re.search(r"int b200t5_forward_choices\(([^)]*)\);", h)
    assert decl is not None
    args = [a.strip() for a in decl.group(1).split(",")]
    assert args == ["b200t5_handle h", "const int64_t* input_ids", "const int64_t* attention_mask", "int B", "int S",
                    "const int32_t* row_offsets", "const int64_t* labels", "int T", "const b200t5_forward_io* io", "void* stream"]
    assert len(_lib.SIGNATURES["b200t5_forward_choices"][1]) == len(args)
    hook = re.search(r"int b200t5_test_decoder_cross_attn_packed\(([^)]*)\);", h)
    assert hook is not None and len(_lib.SIGNATURES["b200t5_test_decoder_cross_attn_packed"][1]) == len(hook.group(1).split(","))
