"""The original T5 (v1.0) on the CUDA path, on an H100: the ReLU feed-forward product in every GEMM configuration that
runs `wi` (EpiRelu), the rescaled final decoder norm (rmsnorm_scaled_kernel), and every model entry point on the
synthetic ReLU checkpoints (tied and rescaled head; t5-tiny-untied keeps an lm_head and no rescale), in both builds.

Anchors as in tests/test_model_gpu.py: the numpy oracle (tests/t5v1_oracle.py: oracle/t5_oracle.py with the ReLU
feed-forward and the rescale) under the margin-gated rule, and transformers eager on this GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import prefix_oracle as po  # tests/ is on sys.path under pytest
from anyscale_workshop_nyc_2023_b200 import _lib, roofline
from anyscale_workshop_nyc_2023_b200.synth import SPECS, save_checkpoint, synthetic_token_batch
from oracle import beam as obeam
from oracle import logits_process as olp
from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits
from oracle.scores import log_softmax
from t5v1_oracle import load_hf_model, oracle_for

pytestmark = pytest.mark.gpu

DEV = 0
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
FFH = {"bf16": torch.bfloat16, "fp16": torch.float32}  # ffh_t: the feed-forward buffer (fp32 holding fp16 values)
EPS = {"bf16": 2.0 ** -7, "fp16": 2.0 ** -10}
ABS = {"bf16": 1e-3, "fp16": 1e-3 / 8}
EXACT = {"bf16": 0.995, "fp16": 0.985}
TAU = {"bf16": 0.13, "fp16": 0.03}
MODE_RELU = 6
BUILDS = ["bf16", "fp16"]


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------ kernels
def check_relu(out, A, W, build):
    """out = relu(act(A W^T)) in ffh_t: within one ulp of torch's relu(round(fp32 product)), mostly bit-identical."""
    torch.cuda.synchronize()
    dt = DT[build]
    ref = torch.relu((A.float() @ W.float().T).to(dt)).float()
    o = out.float()
    assert (o == o.to(dt).float()).all()  # values of the build's 2-byte type
    assert (o >= 0).all()
    tol = EPS[build] * torch.maximum(o.abs(), ref.abs()) + ABS[build]
    assert ((o - ref).abs() <= tol).all()
    exact = (o == ref).float().mean().item()
    assert exact > EXACT[build], exact
    assert (o == 0).float().mean().item() > 0.3  # about half the products are negative


def operands(M, N, K, build, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = DT[build]
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.5).to(dt)
    return A, W, torch.full((M, N), float("nan"), device="cuda", dtype=FFH[build])


# (M, N = d_ff, K = d_model): partial M and N tiles, the t5-small / t5-base feed-forward shapes, many tiles per SM
ENC_SHAPES = [(128, 256, 64), (130, 352, 264), (300, 2048, 512), (4096, 3072, 768), (20000, 3072, 768)]


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("M,N,K", ENC_SHAPES)
def test_relu_encoder_gemms(build, M, N, K):
    """Both 128 x 256 encoder kernels (enc_gemm 0 and 1): bit-identical to each other, and torch's relu(A W^T)."""
    lib = _lib.load(build)
    torch.backends.cuda.matmul.allow_tf32 = False
    A, W, out0 = operands(M, N, K, build, M + N + K)
    out1 = out0.clone()
    for kernel, out in ((0, out0), (1, out1)):
        _lib.check(lib.b200t5_test_enc_gemm(DEV, P(A), P(W), P(out), M, N, K, kernel, MODE_RELU, 0, None, None, 0, 0, 0, None), None, lib)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1)
    check_relu(out1, A, W, build)


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("bn", [512, 128])
@pytest.mark.parametrize("M,N,K", [(130, 352, 264), (1000, 3072, 768)])
def test_relu_test_gemm(build, bn, M, N, K):
    """b200t5_test_gemm mode 6: the encoder configuration (bn 512) and the forward pass's 128 x 128 tiles (bn 128)."""
    lib = _lib.load(build)
    torch.backends.cuda.matmul.allow_tf32 = False
    A, W, out = operands(M, N, K, build, 7 * M + N + bn)
    _lib.check(lib.b200t5_test_gemm(DEV, P(A), P(W), P(out), M, N, K, bn, MODE_RELU, 0, None), None, lib)
    check_relu(out, A, W, build)


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("split", [1, 2, 4, 8])
@pytest.mark.parametrize("M,N,K", [(7, 2048, 512), (256, 3072, 768), (130, 352, 264)])
def test_relu_splitk_gemm(build, bn, split, M, N, K):
    """The decode step's cluster split-K GEMM at every tile width and split the plan can pick."""
    lib = _lib.load(build)
    torch.backends.cuda.matmul.allow_tf32 = False
    A, W, out = operands(M, N, K, build, M + 3 * N + bn + split)
    _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(out), M, N, K, bn, split, MODE_RELU, 0, None, 0, 0, None), None, lib)
    check_relu(out, A, W, build)


@pytest.mark.parametrize("build", BUILDS)
def test_other_modes_still_fail(build):
    lib = _lib.load(build)
    A, W, out = operands(128, 256, 64, build, 1)
    assert lib.b200t5_test_gemm(DEV, P(A), P(W), P(out), 128, 256, 64, 512, 7, 0, None) != 0
    assert lib.b200t5_test_gemm(DEV, P(A), P(W), P(out), 128, 256, 64, 128, 0, 0, None) != 0
    assert lib.b200t5_test_enc_gemm(DEV, P(A), P(W), P(out), 128, 256, 64, 1, 7, 0, None, None, 0, 0, 0, None) != 0
    assert lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(out), 128, 256, 64, 64, 1, 7, 0, None, 0, 0, None) != 0
    assert lib.b200t5_test_rmsnorm_scaled(DEV, P(A), P(W), P(out), 1, 64, 1e-6, 0.0, None) != 0


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("M,d", [(37, 128), (1000, 512), (130, 768), (64, 1024), (9, 2048)])
def test_rescaled_final_norm_bit_for_bit(build, M, d):
    """y = act(act(w * act(x * rsqrt(var + eps))) * s), s = fp32(d ** -0.5): the rescale is torch's `tensor * (d ** -0.5)`
    bit for bit on the unscaled kernel's output, and the whole norm agrees with torch's T5LayerNorm then the rescale."""
    lib = _lib.load(build)
    dt, res = DT[build], (torch.bfloat16 if build == "bf16" else torch.float32)
    g = torch.Generator(device="cuda").manual_seed(M * d)
    x = (torch.randn(M, d, device="cuda", generator=g) * 3).to(res)
    x[3 % M, :] = 0
    w = torch.randn(d, device="cuda", generator=g).to(dt)  # zero-mean weights, as the tied specs draw them
    y = torch.full((M, d), float("nan"), device="cuda", dtype=dt)
    ys = y.clone()
    s = d ** -0.5
    _lib.check(lib.b200t5_test_rmsnorm(DEV, P(x), P(w), P(y), M, d, 1e-6, None), None, lib)
    _lib.check(lib.b200t5_test_rmsnorm_scaled(DEV, P(x), P(w), P(ys), M, d, 1e-6, float(np.float32(s)), None), None, lib)
    torch.cuda.synchronize()
    assert torch.equal(ys, y * s)  # the rescale: one fp32 product of the 2-byte value, one rounding
    var = x.float().pow(2).mean(-1, keepdim=True)
    ref = (w * (x.float() * torch.rsqrt(var + 1e-6)).to(dt)) * s
    err = (ys.float() - ref.float()).abs()
    assert (err <= 3 * EPS[build] * torch.maximum(ys.float().abs(), ref.float().abs()) + 1e-6).all()
    assert (ys == ref).float().mean().item() > 0.99


# ------------------------------------------------------------------------------------------------ the model
@pytest.fixture(scope="module")
def models(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(name, seed, build):
        key = (name, seed, build)
        if key not in cache:
            d = tmp_path_factory.mktemp(f"ckpt_{name}_{seed}")
            save_checkpoint(d, SPECS[name], seed=seed)
            cache[key] = (B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=DT[build]), d)
        return cache[key]

    return get


def gated_rows(ours, ref, margins, tau):
    """Rows equal up to (excluding) their first step with an oracle margin <= tau; returns the count of such rows."""
    w = max(ours.shape[1], ref.shape[1])
    ours = np.pad(ours, ((0, 0), (0, w - ours.shape[1])))
    ref = np.pad(ref, ((0, 0), (0, w - ref.shape[1])))
    ok = 0
    for b in range(ours.shape[0]):
        low = [s for s in range(margins.shape[1]) if not np.isnan(margins[b, s]) and not margins[b, s] > tau]
        upto = 1 + (low[0] if low else margins.shape[1])
        ok += int((ours[b, :upto] == ref[b, :upto]).all())
    return ok


def chosen_within_tau(tokens, scores, first, tau, eos):
    """Every decision the CUDA path made is an arg-max of the oracle's scores along the CUDA path's own tokens up to
    tau: scores[b, t] are the (processed) scores of the position after tokens[b, t], and steps t >= first are checked
    until the row's EOS. Holds whatever near-ties decided, so every row is compared at every step. Returns the count."""
    n = 0
    for b in range(tokens.shape[0]):
        for t in range(first, tokens.shape[1] - 1):
            if t > first and tokens[b, t] == eos:
                break
            v = scores[b, t]
            assert v[tokens[b, t + 1]] >= v.max() - tau, (b, t, float(v.max() - v[tokens[b, t + 1]]))
            n += 1
    return n


MODELS = [("t5-tiny", 1), ("t5-mini", 2), ("t5-tiny-untied", 1)]


def batch(name, B=16, S=40, seed=5):
    return synthetic_token_batch(B, S, SPECS[name].vocab_size, seed=seed, lengths="uniform")


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("name,seed", MODELS)
def test_generate_matches_oracle_and_transformers(models, build, name, seed):
    model, ckpt = models(name, seed, build)
    ids, mask = batch(name)
    T = 16
    ours = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T).cpu().numpy()
    ref, margins = oracle_for(name, seed, emulate=build).generate(ids, mask, max_new_tokens=T, return_margins=True)
    assert gated_rows(ours, ref, margins, TAU[build]) == len(ids)
    # transformers on this GPU, forced length, gated on its own teacher-forced logits along its own path
    # (tests/test_model_gpu.py's rule for FLAN-T5)
    hf = load_hf_model(ckpt, dtype=DT[build], device="cuda")
    want = hf_generate(hf, ids, mask, T, min_new_tokens=T)
    forced = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T,
                            min_new_tokens=T).cpu().numpy()
    assert forced.shape == want.shape
    lg = hf_teacher_forced_logits(hf, ids, mask, want[:, :-1])
    lg[:, :, SPECS[name].eos_token_id] = -np.inf
    top2 = np.partition(lg, -2, axis=-1)[:, :, -2:]
    hf_margins = top2[:, :, 1] - top2[:, :, 0]
    n = gated_rows(forced, want, hf_margins, TAU[build])
    print(f"{name} {build}: {n}/{len(ids)} rows equal transformers on the GPU up to their first near-tie; "
          f"token agreement {(forced == want).mean():.3f}")
    assert n == len(ids)


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("name,seed", MODELS)
def test_forward_loss_and_logits_match_transformers(models, build, name, seed):
    model, ckpt = models(name, seed, build)
    ids, mask = batch(name, B=8)
    labels = synthetic_token_batch(8, 12, SPECS[name].vocab_size, seed=9, lengths="uniform")[0]
    labels[labels == 0] = -100
    out = model(input_ids=ids, attention_mask=mask, labels=labels)
    hf = load_hf_model(ckpt, dtype=DT[build], device="cuda")
    with torch.no_grad():
        ref = hf(input_ids=torch.from_numpy(ids).cuda(), attention_mask=torch.from_numpy(mask).cuda(), labels=torch.from_numpy(labels).cuda())
    err = (out.logits.float().cpu() - ref.logits.float().cpu()).abs()
    atol, mean = (0.5, 0.05) if build == "bf16" else (0.08, 0.008)
    assert err.max() <= atol and err.mean() <= mean
    assert float(out.loss) == pytest.approx(float(ref.loss), rel=2e-2)
    # score() decodes the same labels one position at a time: the same log-likelihoods within rounding
    sc = model.score(input_ids=ids, attention_mask=mask, labels=labels)
    assert float(sc.loss) == pytest.approx(float(out.loss), rel=2e-2)


@pytest.mark.parametrize("build", BUILDS)
def test_score_choices_equals_the_forward_pass_per_row(models, build):
    model, _ = models("t5-mini", 2, build)
    ids, mask = batch("t5-mini", B=6)
    choices = [[5, 6, 1], [17, 1], [9, 40, 41, 1]]
    res = model.score_choices(ids, mask, choices)
    lab = np.full((len(choices), 4), -100)
    for c, ch in enumerate(choices):
        lab[c, : len(ch)] = ch
    rep = np.repeat(np.arange(6), len(choices))
    fw = model(input_ids=ids[rep], attention_mask=mask[rep], labels=np.tile(lab, (6, 1)), return_logits=False)
    assert torch.equal(torch.as_tensor(res.token_logprobs).reshape(-1, 4).cpu(), torch.as_tensor(fw.token_logprobs).cpu())


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("name,seed,n", [("t5-tiny", 1, 1), ("t5-mini", 2, 2), ("t5-tiny-untied", 1, 1)])
def test_beam_search_matches_the_oracle(models, build, name, seed, n):
    """tests/test_beam_gpu.py's checks for FLAN-T5: every returned hypothesis is what the oracle computes along it (each
    token's log-probability, the length-penalised score, beam indices inside its prompt), and at least half the
    prompts' best hypotheses equal the oracle's; prompts without a near-tie decision equal it exactly."""
    model, _ = models(name, seed, build)
    spec, k, T, B = SPECS[name], 4, 12, 12
    ids, mask = batch(name, B=B, S=32, seed=41)
    o = oracle_for(name, seed, emulate=build)
    ref = obeam.beam_search(o, ids, mask, num_beams=k, max_new_tokens=T, num_return_sequences=n)
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T, num_beams=k,
                         num_return_sequences=n, return_dict_in_generate=True, output_scores=True)
    assert out.sequences.shape[0] == B * n
    tau = TAU[build]
    seq, sc, bidx = out.sequences.cpu().numpy(), out.sequences_scores.cpu().numpy(), out.beam_indices.cpu().numpy()
    tlp = out.scores.token_logprobs.cpu().numpy()
    L = (bidx >= 0).sum(axis=1)
    rows = np.arange(B * n) // n
    dec = np.where(np.arange(seq.shape[1] - 1)[None, :] < L[:, None], seq[:, :-1], 0)
    logp = np.stack([log_softmax(x) for x in o.decode_logits(ids[rows], mask[rows], dec)])
    want = np.take_along_axis(logp, seq[:, 1:, None], axis=2)[..., 0]
    live = np.arange(want.shape[1])[None, :] < L[:, None]
    assert np.abs(np.where(live, tlp - want, 0)).max() <= 2 * tau
    assert (tlp[~live] == 0).all() and (L >= 1).all() and (seq[np.arange(B * n), L] == spec.eos_token_id)[L < T].all()
    assert np.all(np.abs(sc - (want * live).sum(axis=1) / L.astype(np.float64)) <= 2 * tau)
    assert ((bidx // k == rows[:, None]) | ~live).all() and (bidx[~live] == -1).all()
    assert (np.diff(sc.reshape(B, n), axis=1) <= 0).all()
    safe = equal = 0
    for b in range(B):
        r = slice(b * n, b * n + n)
        Lr = (ref["beam_indices"][r] >= 0).sum(axis=1)
        w = 1 + int(Lr.max())
        same = np.array_equal(seq[r, :w], ref["sequences"][r, :w]) and np.array_equal(bidx[r, : w - 1], ref["beam_indices"][r, : w - 1])
        L0 = int(Lr[0])
        equal += int(np.array_equal(seq[b * n, : L0 + 1], ref["sequences"][b * n, : L0 + 1]))
        if ref["gap"][b] > tau:
            assert same, b
            safe += 1
    print(f"{name} {build} k={k} n={n}: {safe}/{B} prompts above the near-tie gap (all equal); {equal}/{B} best hypotheses equal")
    assert equal >= B // 2


@pytest.mark.parametrize("build", BUILDS)
def test_output_scores_decoder_prompts_and_processors(models, build):
    name, seed = "t5-mini", 2
    model, _ = models(name, seed, build)
    ids, mask = batch(name, B=8)
    o = oracle_for(name, seed, emulate=build)
    T = 10
    tau = TAU[build]
    eos = SPECS[name].eos_token_id
    # output_scores: the chosen tokens' log-probabilities are score() of the returned sequences (no EOS mask in either),
    # and the oracle's log-softmax along them
    g = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T,
                       return_dict_in_generate=True, output_scores=True)
    seq = g.sequences.cpu().numpy()
    tlp = np.asarray(g.scores.token_logprobs.cpu())
    lab = seq[:, 1:].copy()
    live = np.ones_like(lab, dtype=bool)
    for b in range(len(lab)):
        hit = np.where(lab[b] == eos)[0]
        if len(hit):
            lab[b, hit[0] + 1:] = -100
            live[b, hit[0] + 1:] = False
    sc = model.score(input_ids=ids, attention_mask=mask, labels=lab)
    assert np.allclose(tlp, np.asarray(sc.token_logprobs.cpu()), atol=1e-5)
    logp = np.stack([log_softmax(x) for x in o.decode_logits(ids, mask, seq[:, :-1])])
    want = np.take_along_axis(logp, seq[:, 1:, None], axis=2)[..., 0]
    assert np.abs(np.where(live, tlp - want, 0)).max() <= 2 * tau and (tlp[~live] == 0).all()
    # decoder prompts: gated against the prompted oracle, and every new token an arg-max of the oracle along the path
    d = np.stack([ids[:, 0] * 0, ids[:, 1], ids[:, 2]], 1)
    ours = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask),
                          decoder_input_ids=torch.from_numpy(d), max_new_tokens=T).cpu().numpy()
    ref, _, _, margins = po.generate(o, ids, mask, d, max_new_tokens=T)
    assert gated_rows(ours[:, 2:], ref[:, 2:], margins, tau) == len(ids)
    assert chosen_within_tau(ours, o.decode_logits(ids, mask, ours[:, :-1]), 2, tau, eos) >= len(ids)
    # logits processors: gated against the oracle's, and every decision an arg-max of the oracle's processed scores
    proc = olp.Processors(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=3)
    ours = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T,
                          repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=3).cpu().numpy()
    ref, margins = olp.generate(o, ids, mask, max_new_tokens=T, processors=proc, return_margins=True)
    assert gated_rows(ours, ref, margins, tau) == len(ids)
    raw = o.decode_logits(ids, mask, ours[:, :-1])
    processed = np.stack([olp.process(raw[:, t], ours[:, : t + 1], ids, proc) for t in range(raw.shape[1])], axis=1)
    assert chosen_within_tau(ours, processed, 0, tau, eos) >= len(ids) * 3


@pytest.mark.parametrize("build", BUILDS)
def test_slot_pool_equals_static_batches(models, build):
    model, _ = models("t5-tiny", 1, build)
    ids, mask = batch("t5-tiny", B=24, S=32, seed=77)
    T = 12
    pool, plen = model.generate_stream(ids, mask, pool=8, max_new_tokens=T)
    for c in range(3):
        rows = slice(8 * c, 8 * c + 8)
        st = model.generate(input_ids=torch.from_numpy(ids[rows]), attention_mask=torch.from_numpy(mask[rows]), max_new_tokens=T)
        st = st.cpu().numpy()
        assert (np.asarray(pool)[rows, : st.shape[1]] == st).all()


@pytest.mark.parametrize("build", BUILDS)
def test_batch_predictor_on_a_relu_checkpoint(build):
    from transformers import T5Tokenizer

    from anyscale_workshop_nyc_2023_b200 import rayshim
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir, make_batch_predictor

    ckpt = checkpoint_dir("t5-tiny", seed=1)
    tok = T5Tokenizer.from_pretrained(str(ckpt))
    ids, mask = batch("t5-tiny", B=8, S=32, seed=11)
    ds = rayshim.data.from_numpy({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()})
    bp = make_batch_predictor(ckpt, model_cls=B200T5ForConditionalGeneration, device_map="auto", torch_dtype=DT[build])
    pred = bp.predict(ds, batch_size=8, num_gpus_per_worker=1, max_new_tokens=12).to_pandas()
    model = bp._worker.predictor.model
    toks = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=12).cpu().numpy()
    assert pred["generated_output"].tolist() == tok.batch_decode(toks, skip_special_tokens=True)
    ref, margins = oracle_for("t5-tiny", 1, emulate=build).generate(ids, mask, max_new_tokens=12, return_margins=True)
    assert gated_rows(toks, ref, margins, TAU[build]) == 8


@pytest.mark.parametrize("build", BUILDS)
def test_library_counters_count_two_feed_forward_matrices(models, build):
    spec = SPECS["t5-mini"]
    model, _ = models("t5-mini", 2, build)
    ids, mask = synthetic_token_batch(7, 48, spec.vocab_size, seed=51, lengths="uniform")
    ext = mask.sum(axis=1).tolist()
    model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=9, min_new_tokens=9)
    st = model.stats()
    fp32_wo = build == "fp16"
    assert st["decode_algo_bytes"] == pytest.approx(roofline.decode_bytes(spec, 7, 9, extents=ext, fp32_wo=fp32_wo), rel=1e-9)
    assert st["encoder_flops"] == pytest.approx(roofline.encoder_flops(spec, 7, extents=ext), rel=1e-9)
