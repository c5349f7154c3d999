"""Beam search on the CUDA path (csrc/beam.cuh): the beam step and the cache reordering against torch and the numpy
oracle's step function, the model against the oracle and against transformers on the GPU, and the properties that need
no reference: every entry point, chunking, batch-mates and repeated runs give the same bits, the transition scores add
up to the sequence scores, and greedy calls are unchanged."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from oracle import beam as obeam
from oracle.scores import log_softmax
from oracle.t5_oracle import T5Oracle

pytestmark = pytest.mark.gpu

DEV = 0
TAU = {torch.bfloat16: 0.13, torch.float16: 0.03}  # the greedy tests' near-tie thresholds / logit-error bounds
FLAVOURS = ["bf16", "fp16"]
FIN = np.dtype([("score", "<f4"), ("t", "<i4"), ("par", "<i4"), ("tok", "<i4"), ("lp", "<f4"), ("flag", "<i4")])


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(spec_name, seed, dtype=torch.bfloat16):
        key = (spec_name, seed, dtype)
        if key not in cache:
            d = tmp_path_factory.mktemp(f"ckpt_{spec_name}_{seed}")
            save_checkpoint(d, SPECS[spec_name], seed=seed)
            cache[key] = (B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=dtype), d)
        return cache[key]

    return get


# ----------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("flavour", FLAVOURS)
@pytest.mark.parametrize("k,lp,es", [(4, 1.0, True), (2, 2.0, "never"), (3, -0.5, False)])
def test_beam_step_matches_torch_and_the_oracle_step(flavour, k, lp, es):
    lib = _lib.load(flavour)
    B, V, T, eos, min_new = 3, 1000, 6, 1, 1
    g = torch.Generator(device="cuda").manual_seed(k * 100 + V)
    st = obeam.BeamState(B, k, T, 0, 0)
    run_score = torch.from_numpy(st.run_score.reshape(-1).copy()).cuda()
    fin = np.zeros((B, 16), FIN)
    fin["score"], fin["t"] = -1e9, -1
    fin_d = torch.from_numpy(fin.view(np.uint8).copy()).cuda()
    heur = torch.ones(B, dtype=torch.int32, device="cuda")
    rows = B * k
    lse, cand_lp = torch.empty(rows, device="cuda"), torch.empty((rows, 32), device="cuda")
    cand_tok, parent, token, retired = (torch.empty(s, dtype=torch.int32, device="cuda") for s in ((rows, 32), rows, rows, rows))
    es_code = {False: 0, True: 1, "never": 2}[es]
    for t in range(T):
        logits = torch.randn(rows, V, device="cuda", generator=g) * 3
        logits[:, eos] += 4.0 + 2.0 * t  # hypotheses finish, the finished set fills up
        _lib.check(lib.b200t5_test_beam_step(DEV, P(logits), B, k, V, t, T, eos, min_new, lp, es_code, P(run_score), P(fin_d), P(heur),
                                             P(lse), P(cand_lp), P(cand_tok), P(parent), P(token), P(retired), None), lib=lib)
        torch.cuda.synchronize()
        want_lse = torch.logsumexp(logits.double(), dim=-1)
        assert torch.allclose(lse.double(), want_lse, atol=2e-5, rtol=0)
        lsm = torch.log_softmax(logits, dim=-1)
        if t < min_new:
            lsm[:, eos] = -float("inf")
        # each row's top 2k by (log_prob + running score desc, token asc): the prompt-level order within the row
        acc = (lsm.cpu().numpy() + st.run_score.reshape(-1)[:, None]).astype(np.float32)
        want_tok = np.stack([obeam.order(r)[:2 * k] for r in acc])
        assert np.array_equal(cand_tok[:, :2 * k].cpu().numpy(), want_tok)
        assert (cand_lp[:, :2 * k] - torch.gather(lsm, 1, torch.from_numpy(want_tok).long().cuda())).abs().max().item() <= 2e-5
        # the oracle's step on the kernel's own log-probabilities
        logp = lsm.cpu().numpy()
        ct, cl = cand_tok[:, :2 * k].cpu().numpy(), cand_lp[:, :2 * k].cpu().numpy()
        np.put_along_axis(logp, ct, cl, axis=1)
        live = st.live.copy()
        par, tok, _ = obeam.step(st, logp, t, eos, lp, es)
        ret = retired.cpu().numpy().reshape(B, k)
        assert (ret.all(axis=1) == ~st.live).all() and (ret.all(axis=1) | ~ret.any(axis=1)).all()
        f = fin_d.cpu().numpy().view(FIN).reshape(B, 16)[:, :k]
        for b in np.nonzero(live)[0]:
            sl = slice(b * k, b * k + k)
            assert (parent.cpu().numpy()[sl] == par[sl]).all() and (token.cpu().numpy()[sl] == tok[sl]).all()
            assert np.array_equal(run_score.cpu().numpy()[sl], st.run_score[b])
            assert np.array_equal(f["score"][b], st.fin_score[b]) and ((f["flag"][b] != 0) == st.fin_flag[b]).all()
            real = f["t"][b] >= 0
            assert (f["tok"][b][real] == st.fin_seq[b][real, f["t"][b][real] + 1]).all()
        assert ((heur.cpu().numpy() != 0) == st.heur)[live].all()


# FLAN-T5-base's 24 planes and 12 heads: (k, Tmax, step), steps whose (step + 1) * 8 chunks take the 128-thread loop
# 1 to 9 times
REORDER_CASES = {f"k{k}-T{T}-s{s}": (k, T, s) for k in (2, 5, 16) for T in (40, 129) for s in sorted({0, 15, 16, 127, T - 1}) if s < T}


@pytest.mark.parametrize("flavour", FLAVOURS)
@pytest.mark.parametrize("pmap", ["identity", "all_from_one", "cycle", *REORDER_CASES])
def test_reorder_matches_index_select(flavour, pmap):
    lib = _lib.load(flavour)
    dt = torch.bfloat16 if flavour == "bf16" else torch.float16
    if pmap in REORDER_CASES:  # parents drawn with replacement inside each prompt; prompt 0 keeps its own rows
        k, Tmax, step = REORDER_CASES[pmap]
        planes, B, H = 24, 3, 12
        rng = np.random.default_rng(Tmax * 100 + step * 10 + k)
        parent = torch.tensor([b * k + (j if b == 0 else int(rng.integers(k))) for b in range(B) for j in range(k)], dtype=torch.int32,
                              device="cuda")
    else:
        planes, B, k, H, Tmax, step = 4, 3, 4, 2, 16, 9
        base = {"identity": [0, 1, 2, 3], "all_from_one": [2, 2, 2, 2], "cycle": [1, 0, 3, 2]}[pmap]
        parent = torch.tensor([b * k + j for b in range(B) for j in base], dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(7)
    kv = (torch.randn(planes, B * k, H, Tmax, 64, device="cuda", generator=g)).to(dt)
    kv[:, :, :, step + 1:] = float("nan")  # positions the step has not reached: neither read nor written
    want = kv.clone()
    want[:, :, :, : step + 1] = kv.index_select(1, parent.long())[:, :, :, : step + 1]
    _lib.check(lib.b200t5_test_beam_reorder(DEV, P(kv), planes, B, k, H, Tmax, step, P(parent), None), lib=lib)
    torch.cuda.synchronize()
    assert torch.equal(kv.view(torch.int16), want.view(torch.int16))


# ----------------------------------------------------------------------------------------------------- model
# (model, seed, k, n, length_penalty, early_stopping, min_new_tokens, prompt lengths); "full" prompts fill the window,
# so the stream cross-attention kernel runs
BEAM_CASES = [("tiny", 1, 4, 1, 1.0, False, 0, "uniform"), ("tiny", 1, 2, 2, 2.0, "never", 3, "uniform"),
              ("mini", 2, 4, 4, 0.0, True, 0, "uniform"), ("mini", 2, 3, 1, -0.5, False, 0, "uniform"),
              ("mini", 2, 8, 1, 1.0, "never", 0, "uniform"), ("tiny", 1, 8, 8, 1.0, False, 2, "full"),
              ("tiny", 1, 16, 1, 0.0, True, 0, "full"), ("tiny", 1, 16, 16, 1.0, False, 0, "uniform"),
              ("mini", 2, 4, 2, 1.0, False, 0, "full")]


def _beam_case_id(c):
    return f"{c[0]}-k{c[2]}-n{c[3]}" + ("" if c[7] == "uniform" else f"-{c[7]}")


def _compare(out, ref, gaps, n, tau, lp):
    """Prompts whose oracle decision gap exceeds tau must agree exactly. Returns (such prompts, prompts whose best
    hypothesis agrees)."""
    seq, sc, bidx = (out.sequences.cpu().numpy(), out.sequences_scores.cpu().numpy(), out.beam_indices.cpu().numpy())
    safe = equal = 0
    for b in range(len(gaps)):
        rows = slice(b * n, b * n + n)
        L = (ref["beam_indices"][rows] >= 0).sum(axis=1)
        w = 1 + int(L.max())
        same = np.array_equal(seq[rows, :w], ref["sequences"][rows, :w]) and np.array_equal(bidx[rows, : w - 1], ref["beam_indices"][rows, : w - 1])
        b0 = b * n  # the best hypothesis
        L0 = int(L[0])
        equal += int(np.array_equal(seq[b0, : L0 + 1], ref["sequences"][b0, : L0 + 1]) and np.array_equal(bidx[b0, :L0], ref["beam_indices"][b0, :L0]))
        if gaps[b] > tau:
            assert same, b
            assert (np.abs(sc[rows] - ref["sequences_scores"][rows]) <= 2 * tau * L / L.astype(float) ** lp).all(), b
            safe += 1
    return safe, equal


@pytest.mark.parametrize("case", BEAM_CASES, ids=[_beam_case_id(c) for c in BEAM_CASES])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_model_matches_the_oracle(models, case, dtype):
    name, seed, k, n, lp, es, mn, lengths = case
    model, _ = models(name, seed, dtype)
    spec = SPECS[name]
    B, T = 12, 12
    ids, mask = synthetic_token_batch(B, 32, spec.vocab_size, seed=41 + k, lengths=lengths)
    o = T5Oracle(make_state_dict(spec, seed), spec, emulate="bf16" if dtype == torch.bfloat16 else "fp16")
    ref = obeam.beam_search(o, ids, mask, num_beams=k, max_new_tokens=T, min_new_tokens=mn, num_return_sequences=n,
                            length_penalty=lp, early_stopping=es)
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T, min_new_tokens=mn,
                         num_beams=k, num_return_sequences=n, length_penalty=lp, early_stopping=es, return_dict_in_generate=True,
                         output_scores=True)
    assert out.sequences.shape[0] == B * n and out.sequences.dtype == torch.long and out.sequences.device.type == "cuda"
    assert model.stats()["xattn_kernel"] == (1 if lengths == "full" else 0)  # 1: the stream kernel
    tau = TAU[dtype]
    # 1. Every returned hypothesis, whatever near-ties chose it, is what the oracle computes along it: each token's
    #    log-probability given the prompt and the hypothesis' own prefix (the EOS mask of min_new_tokens included), its
    #    length-penalised score, and beam indices inside its prompt. A fault in the K/V replication to rows j > 0, in the
    #    cache reordering or in the next decoder inputs changes these numbers.
    seq, sc, bidx = out.sequences.cpu().numpy(), out.sequences_scores.cpu().numpy(), out.beam_indices.cpu().numpy()
    tlp = out.scores.token_logprobs.cpu().numpy()
    L = (bidx >= 0).sum(axis=1)
    rows = np.arange(B * n) // n
    dec = np.where(np.arange(seq.shape[1] - 1)[None, :] < L[:, None], seq[:, :-1], 0)
    logp = np.stack([log_softmax(x) for x in o.decode_logits(ids[rows], mask[rows], dec)])
    logp[:, :mn, spec.eos_token_id] = -np.inf
    want = np.take_along_axis(logp, seq[:, 1:, None], axis=2)[..., 0]
    live = np.arange(want.shape[1])[None, :] < L[:, None]
    assert np.abs(np.where(live, tlp - want, 0)).max() <= 2 * tau
    assert (tlp[~live] == 0).all() and (L >= 1).all() and (seq[np.arange(B * n), L] == spec.eos_token_id)[L < T].all()
    assert np.all(np.abs(sc - (want * live).sum(axis=1) / L.astype(np.float64) ** lp) <= 2 * tau * L / L.astype(np.float64) ** lp)
    assert ((bidx // k == rows[:, None]) | ~live).all() and (bidx[~live] == -1).all()
    assert (np.diff(sc.reshape(B, n), axis=1) <= 0).all()  # best first
    # 2. Prompts with no near-tie decision (oracle gap > tau at every step) agree exactly; the others mostly do
    safe, equal = _compare(out, ref, ref["gap"], n, tau, lp)
    print(f"{name} k={k} n={n} {dtype}: {safe}/{B} prompts above the near-tie gap (all equal); {equal}/{B} best hypotheses equal")
    assert equal >= B // 2


def test_model_matches_transformers_on_the_gpu(models):
    from oracle.hf_anchor import load_hf_model

    model, d = models("mini", 2)
    spec = SPECS["mini"]
    ids, mask = synthetic_token_batch(12, 32, spec.vocab_size, seed=53, lengths="uniform")
    T = 12
    hf = load_hf_model(d, dtype=torch.bfloat16, device="cuda")
    with torch.no_grad():
        want = hf.generate(input_ids=torch.from_numpy(ids).cuda(), attention_mask=torch.from_numpy(mask).cuda(), max_new_tokens=T,
                           num_beams=4, do_sample=False, return_dict_in_generate=True, output_scores=True)
    ref = obeam.beam_search(T5Oracle(make_state_dict(spec, 2), spec, emulate="bf16"), ids, mask, num_beams=4, max_new_tokens=T)
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T, num_beams=4,
                         return_dict_in_generate=True)
    hs, hb = want.sequences.cpu().numpy(), want.beam_indices.cpu().numpy()
    seq, bidx = out.sequences.cpu().numpy(), out.beam_indices.cpu().numpy()
    equal = 0
    for b in range(len(ids)):
        L = int((hb[b] >= 0).sum())
        same = np.array_equal(seq[b, : L + 1], hs[b, : L + 1]) and np.array_equal(bidx[b, :L], hb[b, :L])
        assert same or not ref["gap"][b] > TAU[torch.bfloat16], b
        equal += int(same)
    print(f"vs transformers on the GPU: {equal}/{len(ids)} prompts equal")
    assert equal >= len(ids) // 2


def _beam(model, ids, mask, **kw):
    kw = dict(max_new_tokens=12, num_beams=4, num_return_sequences=2, return_dict_in_generate=True, output_scores=True) | kw
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw)
    return [t.cpu().numpy() for t in (out.sequences, out.sequences_scores, out.beam_indices, out.scores.token_logprobs)]


def test_entry_points_chunks_batch_mates_and_repeats_agree(models):
    model, _ = models("tiny", 1)
    spec = SPECS["tiny"]
    ids, mask = synthetic_token_batch(10, 24, spec.vocab_size, seed=61, lengths="uniform")
    a = _beam(model, ids, mask)
    assert all(np.array_equal(x, y) for x, y in zip(a, _beam(model, ids, mask)))  # repeated run
    h = model.generate_host(ids, mask, max_new_tokens=12, num_beams=4, num_return_sequences=2)
    assert all(np.array_equal(x, y) for x, y in zip((a[0], a[1], a[2], a[3]), (h[0], h[2], h[3], h[4])))
    # B * k > pool_size: static chunks of pool_size // k prompts, concatenated
    old = model.pool_size
    try:
        model.pool_size = 12  # chunks of 3 prompts
        c = _beam(model, ids, mask)
    finally:
        model.pool_size = old
    assert all(np.array_equal(x, y) for x, y in zip(a, c))
    # the prompt whose search runs longest, with batch-mates whose searches end (and retire their rows) earlier
    pool_ids, pool_mask = synthetic_token_batch(40, 24, spec.vocab_size, seed=62, lengths="uniform")
    es = dict(early_stopping=True, num_return_sequences=4)
    p = _beam(model, pool_ids, pool_mask, **es)
    longest = (p[2] >= 0).sum(axis=1).reshape(40, 4).max(axis=1)
    order = np.argsort(longest, kind="stable")
    target, mates = order[-1], order[:9]
    assert longest[mates].max() < longest[target]  # each mate's finished set was full, so it retired, before the target's
    x, m = np.concatenate([pool_ids[[target]], pool_ids[mates]]), np.concatenate([pool_mask[[target]], pool_mask[mates]])
    o = _beam(model, x, m, **es)
    W = 1 + int(longest[target])
    t4 = slice(4 * target, 4 * target + 4)
    assert np.array_equal(o[0][:4, :W], p[0][t4, :W]) and np.array_equal(o[1][:4], p[1][t4])
    assert np.array_equal(o[3][:4, : W - 1], p[3][t4, : W - 1])


@pytest.mark.parametrize("lp", [1.0, 0.0, 2.0])
def test_transition_scores_add_up_to_the_sequence_scores(models, lp):
    model, _ = models("mini", 2)
    ids, mask = synthetic_token_batch(6, 32, SPECS["mini"].vocab_size, seed=71, lengths="uniform")
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=12, num_beams=4,
                         num_return_sequences=4, length_penalty=lp, return_dict_in_generate=True, output_scores=True)
    ts = model.compute_transition_scores(out.sequences, out.scores, out.beam_indices)
    L = (out.beam_indices >= 0).sum(dim=1)
    assert (ts[out.beam_indices < 0] == 0).all()
    assert torch.allclose(ts.sum(dim=1) / L.double() ** lp, out.sequences_scores.double(), atol=1e-4, rtol=1e-5)


def test_greedy_calls_are_unchanged_by_a_beam_call(models):
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(8, 24, SPECS["tiny"].vocab_size, seed=81, lengths="uniform")
    a = dict(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=12)
    g0 = model.generate(**a).cpu().numpy()
    l0 = model.stats()["kernel_launches"]
    model.generate(**a, num_beams=4)
    g1 = model.generate(**a).cpu().numpy()
    assert np.array_equal(g0, g1) and model.stats()["kernel_launches"] == l0
    with pytest.raises(NotImplementedError):
        model.generate_stream(ids, mask, max_new_tokens=4, num_beams=2)
    with pytest.raises(NotImplementedError):
        model.generate(**a, num_beams=4, do_sample=True)
    with pytest.raises(NotImplementedError, match="repetition_penalty"):
        model.generate(**a, num_beams=4, repetition_penalty=1.2)
    with pytest.raises(ValueError):
        model.generate(**a, num_beams=2, num_return_sequences=3)


def test_batch_predictor_runs_beam_search(models):
    from transformers import T5Tokenizer

    from anyscale_workshop_nyc_2023_b200 import rayshim
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir, make_batch_predictor

    spec = SPECS["tiny"]
    ckpt = checkpoint_dir("tiny", seed=1)
    ids, mask = synthetic_token_batch(10, 24, spec.vocab_size, seed=91, lengths="uniform")
    ds = rayshim.data.from_numpy({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()})
    bp = make_batch_predictor(ckpt, device_map="auto", torch_dtype=torch.bfloat16)
    out = bp.predict(ds, batch_size=4, num_gpus_per_worker=1, max_scoring_workers=1, max_new_tokens=12, num_beams=4).to_pandas()
    model, _ = models("tiny", 1)
    tok = T5Tokenizer.from_pretrained(str(ckpt))
    want = []
    for lo in range(0, 10, 4):
        a = dict(input_ids=torch.from_numpy(ids[lo:lo + 4]), attention_mask=torch.from_numpy(mask[lo:lo + 4]), max_new_tokens=12)
        want += tok.batch_decode(model.generate(**a, num_beams=4), skip_special_tokens=True)
    assert out["generated_output"].tolist() == want
