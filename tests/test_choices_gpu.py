"""Multiple-choice scoring (`score_choices`, b200t5_forward_choices) on an H100.

Anchors: the packed cross-attention kernel bit for bit against decoder_attn_kernel<kAttnCross> on K/V replicated per
candidate; score_choices bit for bit against forward on the prompts repeated once per candidate; the numpy oracle and
transformers within the forward pass's tolerances; one encoder pass per prompt in stats(); and every other entry point
unchanged around a score_choices call.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.modeling import choice_scores, choice_targets
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir

pytestmark = pytest.mark.gpu

FLAVOUR = {torch.bfloat16: "bf16", torch.float16: "fp16"}
TAU = {torch.bfloat16: 0.13, torch.float16: 0.03}  # logit-error bounds of tests/test_forward_gpu.py
DTYPES = [pytest.param(torch.bfloat16, id="bf16"), pytest.param(torch.float16, id="fp16")]


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(spec_name, seed, dtype=torch.bfloat16):
        key = (spec_name, seed, dtype)
        if key not in cache:
            if spec_name == "flan-t5-base":
                d = checkpoint_dir(spec_name, seed)
            else:
                d = tmp_path_factory.mktemp(f"choices_{spec_name}_{seed}")
                save_checkpoint(d, SPECS[spec_name], seed=seed)
            cache[key] = (B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=dtype), d)
        return cache[key]

    return get


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# ------------------------------------------------------------------ kernel
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S", [1, 64, 130, 512])
def test_packed_cross_attention_kernel_bit_exact(dtype, S):
    """Prompts with 1, 2, 7 and 33 candidates of T = 5 positions: query tiles straddle prompt boundaries. Masks: trailing
    padding, holes, an all-masked prompt, a full one."""
    lib = _lib.load(FLAVOUR[dtype])
    H, T = 2, 5
    I = H * 64
    counts = np.array([1, 2, 7, 33])
    B = len(counts)
    R = int(counts.sum())
    g = torch.Generator(device="cuda").manual_seed(S)
    q = torch.randn(R * T, I, device="cuda", generator=g).to(dtype)
    kv = (torch.randn(2, B, H, S, 64, device="cuda", generator=g) * 0.5).to(dtype)
    rng = np.random.default_rng(S)
    mask = np.ones((B, S), np.int64)
    mask[0, rng.integers(max(1, S // 2), S + 1):] = 0
    mask[1, rng.choice(S, size=S // 3, replace=False)] = 0
    mask[2] = 0
    last = [np.nonzero(m)[0] for m in mask]
    ext = np.array([int(l[-1]) + 1 if l.size else S for l in last], np.int32)
    key_ok = torch.from_numpy(mask.astype(np.uint8)).cuda()
    extent = torch.from_numpy(ext).cuda()
    qoff = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32) * T).cuda()
    ctx = torch.full((R * T, I), float("nan"), dtype=dtype, device="cuda")
    _lib.check(lib.b200t5_test_decoder_cross_attn_packed(0, _ptr(q), _ptr(kv), _ptr(ctx), _ptr(key_ok), _ptr(extent), _ptr(qoff),
                                                         B, S, H, None), lib=lib)
    # the reference: every candidate a prompt of its own, with its prompt's K/V, mask and extent copied
    b_of = torch.from_numpy(np.repeat(np.arange(B), counts)).cuda()
    kv_rep, ok_rep, ext_rep = kv[:, b_of].contiguous(), key_ok[b_of].contiguous(), extent[b_of].contiguous()
    ref = torch.full_like(ctx, float("nan"))
    _lib.check(lib.b200t5_test_decoder_cross_attn(0, _ptr(q), _ptr(kv_rep), _ptr(ref), _ptr(ok_rep), _ptr(ext_rep), R, T, S, H, None),
               lib=lib)
    torch.cuda.synchronize()
    assert not torch.isnan(ctx.float()).any()
    assert torch.equal(ctx.view(torch.int16), ref.view(torch.int16))


# ------------------------------------------------------------------ model
def _forms(rng, B, C, V, Lmax):
    """The three forms of `choices` (the [B, C, L] one padded to Lmax columns)."""
    shared = [[int(t) for t in rng.integers(2, V, size=rng.integers(1, Lmax + 1))] for _ in range(C)]
    per = [[[int(t) for t in rng.integers(2, V, size=rng.integers(1, Lmax + 1))] for _ in range(C)] for _ in range(B)]
    per_arr = np.full((B, C, Lmax), -100, np.int64)
    for b in range(B):
        for c, cand in enumerate(per[b]):
            per_arr[b, c, :len(cand)] = cand
    ragged = [[[int(t) for t in rng.integers(2, V, size=rng.integers(1, Lmax + 1))] for _ in range(rng.integers(1, C + 2))]
              for _ in range(B)]
    return {"shared": shared, "per_prompt": torch.from_numpy(per_arr), "ragged": ragged}


def _expanded(model, ids, mask, choices):
    """forward on the prompts repeated once per candidate, with the candidates as labels: token_logprobs [R, L] and the
    labels [R, L]."""
    lab, counts = choice_targets(choices, ids.shape[0], model.config.vocab_size)
    rep = np.repeat(np.arange(ids.shape[0]), counts)
    out = model(input_ids=ids[rep], attention_mask=mask[rep], labels=lab, return_logits=False)
    return out.token_logprobs, lab, counts


def _check_against_expanded(res, tlp, lab, counts):
    off = np.concatenate([[0], np.cumsum(counts)])
    for b in range(len(counts)):
        for c in range(int(counts[b])):
            r = off[b] + c
            assert torch.equal(res.token_logprobs[b, c], tlp[r]), (b, c)
        assert (res.token_logprobs[b, counts[b]:] == 0).all() and (res.lengths[b, counts[b]:] == 0).all()
    want = choice_scores(tlp, lab, counts)
    assert torch.equal(res.lengths, want.lengths) and torch.equal(res.logprobs, want.logprobs) and torch.equal(res.best, want.best)
    lp = res.logprobs.cpu().numpy()
    for b in range(len(counts)):
        row = [float(np.float32(tlp[off[b] + c].double().sum().item())) for c in range(int(counts[b]))]
        assert lp[b, :counts[b]].tolist() == row and np.isneginf(lp[b, counts[b]:]).all()
        assert int(res.best[b]) == int(np.argmax(row))


MODEL_CASES = [("tiny", 1, 7, 40, 4, 6), ("mini", 2, 5, 70, 7, 9), ("flan-t5-base", 0, 4, 128, 4, 8)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("spec_name,seed,B,S,C,Lmax", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_bit_exact_against_the_expanded_forward(models, dtype, spec_name, seed, B, S, C, Lmax):
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=seed + 40, lengths="uniform")
    mask[-1, 3:] = 0
    rng = np.random.default_rng(B * 10 + C)
    for name, choices in _forms(rng, B, C, spec.vocab_size, Lmax).items():
        res = model.score_choices(ids, mask, choices)
        tlp, lab, counts = _expanded(model, ids, mask, choices)
        assert res.token_logprobs.shape == (B, int(counts.max()), lab.shape[1]), name
        _check_against_expanded(res, tlp, lab, counts)
        norm = model.score_choices(ids, mask, choices, normalize=True)
        assert torch.equal(norm.token_logprobs, res.token_logprobs)
        key = torch.where(res.lengths > 0, res.logprobs / res.lengths.clamp(min=1).float(), res.logprobs)
        assert torch.equal(norm.best, torch.argmax(key, 1))


def test_forms_agree_and_chunking_changes_nothing(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    B, S = 9, 30
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=8, lengths="uniform")
    rng = np.random.default_rng(5)
    shared = [[int(t) for t in rng.integers(2, spec.vocab_size, size=n)] for n in (1, 3, 2, 5)]
    arr = np.full((4, 5), -100, np.int64)
    for c, cand in enumerate(shared):
        arr[c, :len(cand)] = cand
    a = model.score_choices(ids, mask, shared)
    for other in (arr, torch.from_numpy(arr), np.tile(arr, (B, 1, 1)), [shared] * B):
        o = model.score_choices(ids, mask, other)
        assert torch.equal(o.token_logprobs, a.token_logprobs) and torch.equal(o.best, a.best)
    # ragged, with one prompt of 33 candidates; then chunks of 2 prompts, whose row bound splits that prompt's candidates
    ragged = [[[int(t) for t in rng.integers(2, spec.vocab_size, size=rng.integers(1, 6))] for _ in range(n)]
              for n in (1, 2, 33, 7, 1, 3, 2, 1, 4)]
    full = model.score_choices(ids, mask, ragged)
    old = model.pool_size
    try:
        model.pool_size = 2  # at most 2 prompts and 2 * S // L = 12 candidate rows per call
        ch = model.score_choices(ids, mask, ragged)
    finally:
        model.pool_size = old
    for f in ("token_logprobs", "lengths", "logprobs", "best"):
        assert torch.equal(getattr(ch, f), getattr(full, f)), f
    one = model.score_choices(ids[2:3], mask[2:3], [ragged[2]])
    assert torch.equal(one.token_logprobs[0], full.token_logprobs[2, :33])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("spec_name,seed", [("tiny", 1), ("mini", 2)])
def test_against_the_oracle(models, dtype, spec_name, seed):
    from oracle import scores as oscores
    from oracle.t5_oracle import T5Oracle

    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    B, S = 4, 24
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=seed + 3, lengths="uniform")
    rng = np.random.default_rng(seed)
    groups = [[[int(t) for t in rng.integers(2, spec.vocab_size, size=rng.integers(1, 7))] for _ in range(c)] for c in (3, 1, 4, 2)]
    res = model.score_choices(ids, mask, groups)
    lab, counts = choice_targets(groups, B, spec.vocab_size)
    rep = np.repeat(np.arange(B), counts)
    ref, _ = oscores.score(T5Oracle(make_state_dict(spec, seed), spec, emulate=FLAVOUR[dtype]), ids[rep], mask[rep], lab)
    off = np.concatenate([[0], np.cumsum(counts)])
    err = max(np.abs(res.token_logprobs[b, :counts[b]].cpu().numpy() - ref[off[b]:off[b + 1]]).max() for b in range(B))
    print(f"{spec_name} {FLAVOUR[dtype]}: score_choices vs oracle token log-probs max err {err:.4f}")
    assert err <= 2 * TAU[dtype]


@pytest.mark.parametrize("dtype", DTYPES)
def test_against_transformers(models, dtype):
    pytest.importorskip("transformers")
    from oracle.hf_anchor import load_hf_model

    spec = SPECS["tiny"]
    model, ckpt = models("tiny", 1, dtype)
    B, S = 16, 32
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=17, lengths="uniform")
    rng = np.random.default_rng(11)
    choices = [[int(t) for t in rng.integers(2, spec.vocab_size, size=n)] for n in (1, 2, 1, 3)]
    res = model.score_choices(ids, mask, choices)
    lab, counts = choice_targets(choices, B, spec.vocab_size)
    rep = np.repeat(np.arange(B), counts)
    hf = load_hf_model(ckpt)
    with torch.no_grad():
        out = hf(input_ids=torch.from_numpy(ids[rep]), attention_mask=torch.from_numpy(mask[rep]), labels=torch.from_numpy(lab))
    on = lab != -100
    lsm = torch.log_softmax(out.logits.float(), -1)
    ref = (torch.gather(lsm, 2, torch.from_numpy(np.where(on, lab, 0))[..., None])[..., 0] * torch.from_numpy(on)).float()
    ref_scores = choice_scores(ref, lab, counts)
    err = (res.token_logprobs.cpu() - ref_scores.token_logprobs).abs().max().item()
    print(f"tiny {FLAVOUR[dtype]}: score_choices vs transformers fp32 token log-probs max err {err:.4f}")
    assert err <= 2 * TAU[dtype]
    top2 = torch.topk(ref_scores.logprobs, 2, dim=1).values
    sep = (top2[:, 0] - top2[:, 1]) > 2 * TAU[dtype] * lab.shape[1]  # the per-token bound over a whole candidate
    print(f"  .best compared on {int(sep.sum())}/{B} prompts")
    assert sep.any()
    assert torch.equal(res.best.cpu()[sep], ref_scores.best[sep])


def test_one_encoder_pass_per_prompt(models):
    spec = SPECS["mini"]
    model, _ = models("mini", 2)
    B, S, C = 6, 48, 4
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=2, lengths="uniform")
    choices = [[5], [6, 7], [8, 9, 10], [11]]
    model.score_choices(ids, mask, choices)
    ours = model.stats()["encoder_flops"]
    model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=2)
    gen = model.stats()["encoder_flops"]
    rep = np.repeat(np.arange(B), C)
    model.generate(input_ids=torch.from_numpy(ids[rep]), attention_mask=torch.from_numpy(mask[rep]), max_new_tokens=2)
    expanded = model.stats()["encoder_flops"]
    assert ours == gen and expanded == pytest.approx(C * gen)


def test_other_entry_points_unchanged_around_score_choices(models):
    spec = SPECS["mini"]
    model, _ = models("mini", 2)
    ids, mask = synthetic_token_batch(8, 24, spec.vocab_size, seed=12, lengths="uniform")
    tids, tmask = torch.from_numpy(ids), torch.from_numpy(mask)
    labels = np.random.default_rng(0).integers(2, spec.vocab_size, size=(8, 6)).astype(np.int64)

    def run():
        res = []
        for kw in (dict(max_new_tokens=10), dict(max_new_tokens=10, return_dict_in_generate=True, output_scores=True),
                   dict(max_new_tokens=10, num_beams=3)):
            o = model.generate(input_ids=tids, attention_mask=tmask, **kw)
            seq = o.sequences if hasattr(o, "sequences") else o
            extra = o.token_logprobs.clone() if getattr(o, "token_logprobs", None) is not None else None
            res.append((seq.clone(), extra, int(model.stats()["kernel_launches"])))
        f = model(input_ids=ids, attention_mask=mask, labels=labels)
        res.append((f.logits.clone(), f.token_logprobs.clone(), int(model.stats()["kernel_launches"])))
        s = model.score(input_ids=tids, attention_mask=tmask, labels=torch.from_numpy(labels))
        res.append((s.token_logprobs.clone(), None, int(model.stats()["kernel_launches"])))
        return res

    first = run()
    # 33 candidates of up to 60 tokens per prompt: the call grows the workspace past the forward pass's
    rng = np.random.default_rng(1)
    model.score_choices(ids, mask, [[int(t) for t in rng.integers(2, spec.vocab_size, size=rng.integers(1, 61))] for _ in range(33)])
    second = run()
    for (a1, e1, n1), (a2, e2, n2) in zip(first, second):
        assert torch.equal(a1, a2) and n1 == n2
        assert (e1 is None) == (e2 is None) and (e1 is None or torch.equal(e1, e2))


def test_entry_point_validation(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    lib, h = model._lib, model._h
    B, S, T = 3, 10, 4
    ids = torch.randint(2, spec.vocab_size, (B, S), device="cuda")
    lab = torch.randint(2, spec.vocab_size, (6, T), device="cuda")
    logp = torch.empty((6, T), device="cuda")
    io = _lib.ForwardIO(logits=None, token_logprobs=logp.data_ptr())

    def call(offs, labels=lab, T=T, io=io):
        o = np.ascontiguousarray(offs, np.int32)
        return lib.b200t5_forward_choices(h, _ptr(ids), None, B, S, o.ctypes.data_as(C.c_void_p), _ptr(labels), T, C.byref(io), None)

    assert call([0, 1, 3, 6]) == _lib.OK
    for bad in ([1, 2, 3, 6], [0, 2, 2, 6], [0, 3, 2, 6]):
        assert call(bad) == _lib.EINVAL, bad
    assert call([0, 1, 3, 6], T=0) == _lib.EINVAL
    bad_lab = lab.clone()
    bad_lab[5, 3] = spec.vocab_size
    assert call([0, 1, 3, 6], labels=bad_lab) == _lib.EINVAL
    assert call([0, 1, 3, 6], io=_lib.ForwardIO(logits=None, token_logprobs=None)) == _lib.EINVAL
    with pytest.raises(IndexError):
        model.score_choices(np.full((2, 5), spec.vocab_size), None, [[1]])
    with pytest.raises(ValueError):
        model.score_choices(np.ones((2, 5), np.int64), np.ones((2, 4), np.int64), [[1]])
    with pytest.raises(ValueError):
        model.score_choices(np.ones((2, 5), np.int64), None, [[1, -100, 2]])
