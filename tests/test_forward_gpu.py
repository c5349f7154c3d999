"""The teacher-forced forward pass (`model(input_ids, attention_mask, labels=...)`, b200t5_forward) on an H100.

Anchors: the decoder attention kernels against a float64 reference with HF's rounding points; the committed HF goldens
(logits, label log-probabilities, loss); HF eager on this GPU against its own GPU-vs-CPU noise floor; and the step-loop
paths of this library (decode_logits, score) on the same inputs.
"""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, save_checkpoint, synthetic_token_batch

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden"
CASES = {"tiny_a": ("tiny", 1), "tiny_full": ("tiny", 1), "mini_a": ("mini", 2)}
# logit tolerances of tests/test_model_gpu.py
LOGIT_ATOL, LOGIT_MEAN = 0.5, 0.05
LOGIT_ATOL_FP16, LOGIT_MEAN_FP16 = 0.08, 0.008
TAU = {torch.bfloat16: 0.13, torch.float16: 0.03}  # logit-error bounds of tests/test_scores_gpu.py
FLAVOUR = {torch.bfloat16: "bf16", torch.float16: "fp16"}


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(spec_name, seed, dtype=torch.bfloat16):
        key = (spec_name, seed, dtype)
        if key not in cache:
            d = tmp_path_factory.mktemp(f"fwd_{spec_name}_{seed}")
            save_checkpoint(d, SPECS[spec_name], seed=seed)
            cache[key] = (B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=dtype), d)
        return cache[key]

    return get


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _round(x, dtype):
    return torch.as_tensor(x).to(dtype).double()


def _attn_ref(q, k, v, bias, ok, dtype):
    """float64 with HF's rounding points: act(q.k), act(+ bias), masked, fp32 softmax, act(p), fp32 P.V, act(out)."""
    s = _round(q.double() @ k.double().T, dtype)
    if bias is not None:
        s = _round(s + bias, dtype)
    s = torch.where(ok, s, torch.full_like(s, torch.finfo(dtype).min))
    p = torch.softmax(s.float(), -1).double()
    p = _round(p, dtype)
    return (p @ v.double()).to(dtype).double()


def _bucket(n, nb=32, md=128):
    return _lib.load().b200t5_relative_bucket(-n, 0, nb, md)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("B,T,H", [(2, 1, 2), (2, 77, 3), (1, 1024, 2), (3, 130, 1)])
def test_causal_self_attention_kernel(dtype, B, T, H):
    lib = _lib.load(FLAVOUR[dtype])
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T)
    I = H * 64
    qkv = (torch.randn(B * T, 3 * I, device="cuda", generator=g) * 0.5).to(dtype)
    table = torch.randn(32, H, generator=torch.Generator().manual_seed(3)).to(dtype).float()
    dist = torch.stack([table[_bucket(n)] for n in range(T)], 1).contiguous().cuda()  # [H][T]
    ctx = torch.full((B * T, I), float("nan"), dtype=dtype, device="cuda")
    _lib.check(lib.b200t5_test_decoder_self_attn(0, _ptr(qkv), _ptr(ctx), _ptr(dist), B, T, H, None), lib=lib)
    torch.cuda.synchronize()
    i = torch.arange(T)[:, None]
    j = torch.arange(T)[None, :]
    causal = (j <= i).cuda()
    bias = dist[:, (i - j).clamp(min=0)].double()  # [H][T][T]
    worst = 0.0
    for b in range(B):
        for h in range(H):
            rows = qkv[b * T:(b + 1) * T]
            ref = _attn_ref(rows[:, h * 64:(h + 1) * 64], rows[:, I + h * 64:I + (h + 1) * 64], rows[:, 2 * I + h * 64:2 * I + (h + 1) * 64],
                            bias[h], causal, dtype)
            got = ctx[b * T:(b + 1) * T, h * 64:(h + 1) * 64].double()
            worst = max(worst, (got - ref).abs().max().item())
    print(f"causal self-attention {FLAVOUR[dtype]} B={B} T={T} H={H}: max |err| {worst:.3g}")
    assert worst <= (2 ** -7 if dtype == torch.bfloat16 else 2 ** -10)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("B,T,S,H", [(3, 1, 40, 2), (3, 100, 70, 2), (2, 1024, 64, 1), (4, 33, 513, 2)])
def test_cross_attention_kernel(dtype, B, T, S, H):
    lib = _lib.load(FLAVOUR[dtype])
    g = torch.Generator(device="cuda").manual_seed(B * 7 + T + S)
    I = H * 64
    q = torch.randn(B * T, I, device="cuda", generator=g).to(dtype)
    kv = (torch.randn(2, B, H, S, 64, device="cuda", generator=g) * 0.5).to(dtype)
    rng = np.random.default_rng(T + S)
    mask = np.ones((B, S), np.int64)
    mask[0, rng.integers(S // 2, S):] = 0            # trailing padding
    mask[1, rng.choice(S, size=S // 3, replace=False)] = 0  # holes
    if B > 2:
        mask[2] = 0                                  # a prompt without any attended key
    key_ok = torch.from_numpy(mask.astype(np.uint8)).cuda()
    last = [np.nonzero(m)[0] for m in mask]
    extent = torch.tensor([int(l[-1]) + 1 if l.size else S for l in last], dtype=torch.int32, device="cuda")
    ctx = torch.full((B * T, I), float("nan"), dtype=dtype, device="cuda")
    _lib.check(lib.b200t5_test_decoder_cross_attn(0, _ptr(q), _ptr(kv), _ptr(ctx), _ptr(key_ok), _ptr(extent), B, T, S, H, None), lib=lib)
    torch.cuda.synchronize()
    worst = 0.0
    for b in range(B):
        ok = key_ok[b].bool()[None, :].expand(T, S)
        for h in range(H):
            ref = _attn_ref(q[b * T:(b + 1) * T, h * 64:(h + 1) * 64], kv[0, b, h], kv[1, b, h], None, ok, dtype)
            got = ctx[b * T:(b + 1) * T, h * 64:(h + 1) * 64].double()
            worst = max(worst, (got - ref).abs().max().item())
    print(f"cross-attention {FLAVOUR[dtype]} B={B} T={T} S={S} H={H}: max |err| {worst:.3g}")
    assert worst <= (2 ** -7 if dtype == torch.bfloat16 else 2 ** -10)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", list(CASES))
def test_golden_logits(models, case, dtype):
    spec_name, seed = CASES[case]
    sfx = "" if dtype == torch.bfloat16 else "_fp16"
    g = np.load(GOLD / f"{case}{sfx}.npz")
    model, _ = models(spec_name, seed, dtype)
    key = "bf16" if dtype == torch.bfloat16 else "fp16"
    dec_in = g[f"tokens_{key}"][:, :-1]  # the decoder inputs the golden logits were computed on
    out = model(input_ids=g["ids"], attention_mask=g["mask"], decoder_input_ids=dec_in)
    assert out.loss is None and out.token_logprobs is None and out.logits.dtype == dtype
    ref = g[f"logits_{key}"]
    err = np.abs(out.logits.float().cpu().numpy() - ref)
    atol, mean = (LOGIT_ATOL, LOGIT_MEAN) if dtype == torch.bfloat16 else (LOGIT_ATOL_FP16, LOGIT_MEAN_FP16)
    print(f"{case} {key}: forward logits max err {err.max():.4f} mean {err.mean():.5f}")
    assert err.max() <= atol and err.mean() <= mean


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("spec_name,seed,pre", [("tiny", 1, "tiny"), ("mini", 2, "mini")])
def test_golden_label_logprobs_and_loss(models, dtype, spec_name, seed, pre):
    z = np.load(GOLD / "scores.npz")
    model, _ = models(spec_name, seed, dtype)
    lab = z[f"{pre}_labels"]
    out = model(input_ids=z[f"{pre}_ids"], attention_mask=z[f"{pre}_mask"], labels=lab, return_logits=False)
    assert out.logits is None
    got = out.token_logprobs.cpu().numpy()
    want = z[f"{pre}_fp32_label_logprobs"]
    err = np.abs(got - want)
    print(f"{pre} {FLAVOUR[dtype]}: label log-probs max err {err.max():.4f}, loss {float(out.loss):.5f} vs {float(z[f'{pre}_fp32_loss']):.5f}")
    assert (got[lab == -100] == 0).all()
    assert err.max() <= 2 * TAU[dtype]
    assert abs(float(out.loss) - float(z[f"{pre}_fp32_loss"])) <= 2 * TAU[dtype]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_flan_t5_small_vs_hf_gpu(models, dtype):
    pytest.importorskip("transformers")
    from oracle.hf_anchor import load_hf_model

    spec = SPECS["flan-t5-small"]
    model, ckpt = models("flan-t5-small", 3, dtype)
    B, S, T = 16, 96, 24
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths="uniform")
    rng = np.random.default_rng(8)
    labels = rng.integers(2, spec.vocab_size, size=(B, T)).astype(np.int64)
    labels[rng.random((B, T)) < 0.15] = -100
    tl = torch.from_numpy(labels)

    def hf_run(device):
        hf = load_hf_model(ckpt, dtype=dtype, device=device)
        with torch.no_grad():
            fo = hf(input_ids=torch.from_numpy(ids).to(device), attention_mask=torch.from_numpy(mask).to(device), labels=tl.to(device))
        return fo.logits.float().cpu(), float(fo.loss)

    gpu_lg, gpu_loss = hf_run("cuda")
    cpu_lg, _ = hf_run("cpu")
    out = model(input_ids=ids, attention_mask=mask, labels=tl)
    ours = out.logits.float().cpu()
    err = (ours - gpu_lg).abs()
    floor = (gpu_lg - cpu_lg).abs()
    print(f"flan-t5-small {FLAVOUR[dtype]} forward logits vs HF-GPU max {err.max():.4f} mean {err.mean():.5f} | floor max "
          f"{floor.max():.4f} mean {floor.mean():.5f}; loss {float(out.loss):.5f} vs HF {gpu_loss:.5f}")
    assert err.mean() <= 1.15 * floor.mean() and err.max() <= 1.6 * floor.max()
    assert abs(float(out.loss) - gpu_loss) <= 2 * TAU[dtype] / 10


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_against_decode_logits_and_score(models, dtype):
    spec = SPECS["mini"]
    model, _ = models("mini", 2, dtype)
    B, S, T = 12, 70, 67
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=4, lengths="uniform")
    labels = np.random.default_rng(1).integers(2, spec.vocab_size, size=(B, T)).astype(np.int64)
    out = model(input_ids=ids, attention_mask=mask, labels=labels)
    dec_in = np.concatenate([np.zeros((B, 1), np.int64), labels[:, :-1]], 1)
    step = model.decode_logits(ids, mask, dec_in).cpu()
    lg_err = (out.logits.float().cpu() - step).abs()
    sc = model.score(input_ids=ids, attention_mask=mask, labels=labels)
    lp_err = (out.token_logprobs - sc.token_logprobs).abs()
    print(f"mini {FLAVOUR[dtype]}: forward vs decode_logits max {lg_err.max():.4f} mean {lg_err.mean():.5f}; "
          f"vs score() log-probs max {lp_err.max():.4f}; |loss - score loss| {abs(float(out.loss) - float(sc.loss)):.2e}")
    atol, mean = (LOGIT_ATOL, LOGIT_MEAN) if dtype == torch.bfloat16 else (LOGIT_ATOL_FP16, LOGIT_MEAN_FP16)
    assert lg_err.max() <= atol and lg_err.mean() <= mean
    assert lp_err.max() <= 2 * TAU[dtype]
    assert abs(float(out.loss) - float(sc.loss)) <= TAU[dtype] / 10


def test_semantics(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    B, S, T = 10, 30, 9
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=9, lengths="uniform")
    labels = np.random.default_rng(2).integers(2, spec.vocab_size, size=(B, T)).astype(np.int64)
    labels[:, 3] = -100  # holes in the middle
    labels[4, :] = -100
    a = model(input_ids=ids, attention_mask=mask, labels=labels)
    lp = a.token_logprobs.cpu().numpy()
    assert (lp[labels == -100] == 0).all() and (lp[labels != -100] < 0).all()
    want = -(lp.astype(np.float64).sum() / (labels != -100).sum())
    assert abs(float(a.loss) - want) <= 1e-6 * abs(want) and a["loss"] is a.loss
    # explicit decoder ids equal to the shifted labels: identical bits
    dec = np.concatenate([np.zeros((B, 1), np.int64), np.where(labels[:, :-1] == -100, 0, labels[:, :-1])], 1)
    b = model(input_ids=ids, attention_mask=mask, decoder_input_ids=dec, labels=labels)
    assert torch.equal(a.logits, b.logits) and torch.equal(a.token_logprobs, b.token_logprobs)
    # run to run
    c = model(input_ids=ids, attention_mask=mask, labels=labels)
    assert torch.equal(a.logits, c.logits) and torch.equal(a.token_logprobs, c.token_logprobs)
    # all labels ignored: NaN loss, as transformers
    assert np.isnan(float(model(input_ids=ids, attention_mask=mask, labels=np.full((B, T), -100)).loss))
    # a row's results do not depend on its batch; batches beyond pool_size run in chunks with the same bits
    one = model(input_ids=ids[2:3], attention_mask=mask[2:3], labels=labels[2:3])
    assert torch.equal(one.logits[0], a.logits[2]) and torch.equal(one.token_logprobs[0], a.token_logprobs[2])
    old = model.pool_size
    try:
        model.pool_size = 4
        ch = model(input_ids=ids, attention_mask=mask, labels=labels)
    finally:
        model.pool_size = old
    assert torch.equal(ch.logits, a.logits) and torch.equal(ch.token_logprobs, a.token_logprobs)
    with pytest.raises(ValueError):
        model(input_ids=ids, attention_mask=mask)
    for k in ("decoder_attention_mask", "encoder_outputs", "past_key_values", "output_attentions"):
        with pytest.raises(NotImplementedError):
            model(input_ids=ids, labels=labels, **{k: True})
    model(input_ids=ids, labels=labels, use_cache=False, return_dict=True)
    with pytest.raises(ValueError):
        model(input_ids=ids, attention_mask=mask[:, :-1], labels=labels)
    bad_ids = ids.copy()
    bad_ids[1, 2] = spec.vocab_size
    with pytest.raises(IndexError):
        model(input_ids=bad_ids, attention_mask=mask, labels=labels)
    bad = labels.copy()
    bad[0, 0] = spec.vocab_size
    with pytest.raises(_lib.B200T5Error):
        model(input_ids=ids, labels=bad)


def test_long_prompts_and_long_labels(models):
    """Prompts over 512 tokens (the unpacked encoder) and T > S against the step loop."""
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    for B, S, T in ((3, 600, 20), (2, 40, 300)):
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=S, lengths="uniform")
        dec = np.random.default_rng(T).integers(2, spec.vocab_size, size=(B, T)).astype(np.int64)
        out = model(input_ids=ids, attention_mask=mask, decoder_input_ids=dec)
        err = (out.logits.float().cpu() - model.decode_logits(ids, mask, dec).cpu()).abs()
        print(f"B={B} S={S} T={T}: forward vs decode_logits max {err.max():.4f} mean {err.mean():.5f}")
        assert err.max() <= LOGIT_ATOL and err.mean() <= LOGIT_MEAN


def test_generate_is_unchanged_around_a_forward(models):
    spec = SPECS["mini"]
    model, _ = models("mini", 2)
    ids, mask = synthetic_token_batch(8, 24, spec.vocab_size, seed=12, lengths="uniform")
    tids, tmask = torch.from_numpy(ids), torch.from_numpy(mask)
    calls = [dict(max_new_tokens=10), dict(max_new_tokens=10, return_dict_in_generate=True, output_scores=True),
             dict(max_new_tokens=10, num_beams=3)]

    def run():
        res = []
        for kw in calls:
            o = model.generate(input_ids=tids, attention_mask=tmask, **kw)
            seq = o.sequences if hasattr(o, "sequences") else o
            extra = o.token_logprobs.clone() if getattr(o, "token_logprobs", None) is not None else None
            res.append((seq.clone(), extra, int(model.stats()["kernel_launches"])))
        return res

    first = run()
    labels = np.random.default_rng(0).integers(2, spec.vocab_size, size=(8, 40)).astype(np.int64)
    model(input_ids=ids, attention_mask=mask, labels=labels)  # T > S: the forward grows the workspace
    second = run()
    for (s1, e1, n1), (s2, e2, n2) in zip(first, second):
        assert torch.equal(s1, s2) and n1 == n2
        assert (e1 is None) == (e2 is None) and (e1 is None or torch.equal(e1, e2))
