"""Token log-probabilities on the CUDA path (csrc/gemm.cuh EpiLmHead<*, true>, finalize_step_kernel<*, true>): the fused
kernels against torch.log_softmax on the same GPU, the model against the numpy oracle and against transformers, and the
properties that need no reference: scoring changes no token and no launch of a plain call, every entry point returns the
same bits, and teacher-forced score() of a generation returns the generation's own numbers."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from oracle import logits_process as olp
from oracle import scores as oscores

pytestmark = pytest.mark.gpu

DEV = 0
TAU = {torch.bfloat16: 0.13, torch.float16: 0.03}  # margin gates / logit-error bounds of tests/test_model_gpu.py


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ----------------------------------------------------------------------------------------------------- kernel
def _params(d, keep):
    p = _lib.LogitsParams(repetition_penalty=d.get("repetition_penalty", 1.0),
                          encoder_repetition_penalty=d.get("encoder_repetition_penalty", 1.0),
                          no_repeat_ngram_size=d.get("no_repeat_ngram_size", 0),
                          encoder_no_repeat_ngram_size=d.get("encoder_no_repeat_ngram_size", 0))

    def arr(x):
        a = np.ascontiguousarray(x, dtype=np.int32)
        keep.append(a)
        return a.ctypes.data_as(C.c_void_p)

    for k in ("suppress_tokens", "begin_suppress_tokens"):
        if d.get(k):
            setattr(p, k, arr(d[k]))
            setattr(p, "n_" + k, len(d[k]))
    if d.get("eos"):
        p.eos_token_ids, p.n_eos_token_ids = arr(d["eos"]), len(d["eos"])
    if d.get("bad_words_ids"):
        bw = d["bad_words_ids"]
        p.bad_words_ids = arr([t for w in bw for t in w])
        p.bad_words_offsets = arr(np.cumsum([0] + [len(w) for w in bw]))
        p.n_bad_words = len(bw)
    return p


KPROCS = {  # the processor sets of tests/test_logits_process_gpu.py, and none
    "none": dict(),
    "rep": dict(repetition_penalty=1.3),
    "enc_rep": dict(encoder_repetition_penalty=1.7),
    "ngram": dict(no_repeat_ngram_size=2),
    "enc_ngram": dict(encoder_no_repeat_ngram_size=3),
    "bad": dict(bad_words_ids=[[5], [1], [2, 3], [3, 4, 2], [0, 7]]),
    "suppress": dict(suppress_tokens=[4, 9, 250], begin_suppress_tokens=[6, 8]),
    "all": dict(repetition_penalty=1.2, encoder_repetition_penalty=0.8, no_repeat_ngram_size=3,
                encoder_no_repeat_ngram_size=2, bad_words_ids=[[5], [2, 3]], suppress_tokens=[9],
                begin_suppress_tokens=[6], eos=[1, 11], min_new=True),
}


def _kernel_inputs(flavour, V, M, step, K=256, S=40):
    dt = torch.bfloat16 if flavour == "bf16" else torch.float16
    g = torch.Generator(device="cuda").manual_seed(M * 7 + step + V)
    x = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(V, K, device="cuda", generator=g) * 0.2).to(dt)
    W[3] = W[4]
    hist = torch.randint(0, 12, (M, step + 1), device="cuda", generator=g)
    hist[:, 0] = 0
    if step >= 4:
        hist[0, 1:5] = torch.tensor([2, 3, 2, 3])
    enc = torch.randint(0, 12, (M, S), device="cuda", generator=g)
    enc[:, S - 5:] = 0
    return x, W, hist, enc, K, S


def _lm_score(lib, x, W, V, K, step, min_new, params, hist, enc, S, forced=None, eos=1):
    M = x.shape[0]
    toks = torch.empty(M, dtype=torch.long, device="cuda")
    logp = torch.full((M,), float("nan"), device="cuda")
    logit = torch.full((M,), float("nan"), device="cuda")
    vals = torch.full((M, V), float("nan"), device="cuda")
    _lib.check(lib.b200t5_test_lm_score(DEV, P(x), P(W), M, V, K, step, eos, min_new, None if params is None else C.byref(params),
                                        P(hist), P(enc), S, P(forced), P(toks), P(logp), P(logit), P(vals), None), lib=lib)
    torch.cuda.synchronize()
    return toks, logp, logit, vals


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
@pytest.mark.parametrize("V", [1000, 32128])
@pytest.mark.parametrize("M", [1, 7, 256])
@pytest.mark.parametrize("step", [0, 5])
@pytest.mark.parametrize("name", list(KPROCS))
def test_kernel_matches_torch_log_softmax(flavour, V, M, step, name):
    lib = _lib.load(flavour)
    d = KPROCS[name]
    x, W, hist, enc, K, S = _kernel_inputs(flavour, V, M, step)
    min_new = step + 1 if d.get("min_new") else 0
    keep = []
    params = _params(d, keep) if d else None
    toks, logp, logit, vals = _lm_score(lib, x, W, V, K, step, min_new, params, hist, enc, S)
    # the same tokens and the same processed values as the hooks of the plain step
    ref_tok = torch.empty(M, dtype=torch.long, device="cuda")
    if d:
        ref_vals = torch.full((M, V), float("nan"), device="cuda")
        _lib.check(lib.b200t5_test_lm_process(DEV, P(x), P(W), M, V, K, step, 1, min_new, C.byref(params), P(hist), P(enc), S,
                                              P(ref_tok), P(ref_vals), None), lib=lib)
        torch.cuda.synchronize()
        assert torch.equal(vals.view(torch.int32), ref_vals.view(torch.int32))
    else:
        _lib.check(lib.b200t5_test_lm_argmax(DEV, P(x), P(W), M, V, K, step, 1, min_new, P(ref_tok), None), lib=lib)
        torch.cuda.synchronize()
    assert torch.equal(toks, ref_tok)
    assert not torch.isnan(vals).any()
    ref = torch.log_softmax(vals, -1).gather(1, toks[:, None])[:, 0]
    assert (logp - ref).abs().max().item() <= 2e-5
    assert torch.equal(logit, vals.gather(1, toks[:, None])[:, 0])
    assert (logp <= 0).all()


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
@pytest.mark.parametrize("V", [1000, 32128])
def test_kernel_forced_tokens(flavour, V):
    lib = _lib.load(flavour)
    M, step = 7, 5
    x, W, hist, enc, K, S = _kernel_inputs(flavour, V, M, step)
    keep = []
    params = _params(dict(suppress_tokens=[4, 9], repetition_penalty=1.3), keep)
    forced = torch.tensor([0, 4, V - 1, 127, 128, 9, 500], device="cuda")  # banned ones, tile edges, the last column
    toks, logp, logit, vals = _lm_score(lib, x, W, V, K, step, 0, params, hist, enc, S, forced)
    assert torch.equal(toks, forced)
    ref = torch.log_softmax(vals, -1).gather(1, forced[:, None])[:, 0]
    banned = torch.tensor([False, True, False, False, False, True, False], device="cuda")
    assert torch.isneginf(logp[banned]).all() and torch.isneginf(logit[banned]).all() and not torch.isnan(logp).any()
    assert (logp[~banned] - ref[~banned]).abs().max().item() <= 2e-5
    assert torch.equal(logit, vals.gather(1, forced[:, None])[:, 0])
    # without processors too
    toks, logp, logit, vals = _lm_score(lib, x, W, V, K, step, 0, None, None, None, 0, forced)
    assert torch.equal(toks, forced)
    assert (logp - torch.log_softmax(vals, -1).gather(1, forced[:, None])[:, 0]).abs().max().item() <= 2e-5


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
def test_kernel_single_allowed_column_has_log_probability_zero(flavour):
    lib = _lib.load(flavour)
    V, M, step = 1000, 7, 0
    x, W, hist, enc, K, S = _kernel_inputs(flavour, V, M, step)
    keep = []
    only = 777
    params = _params(dict(suppress_tokens=[t for t in range(V) if t != only]), keep)
    toks, logp, logit, vals = _lm_score(lib, x, W, V, K, step, 0, params, hist, enc, S, eos=only)
    assert (toks == only).all()
    assert torch.equal(logp, torch.zeros_like(logp))
    assert torch.equal(logit, vals[:, only])


# ----------------------------------------------------------------------------------------------------- models
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


def _oracle(spec_name, seed, dtype):
    from oracle.t5_oracle import T5Oracle

    return T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate="fp16" if dtype == torch.float16 else "bf16")


def _scored(model, ids, mask, **kw):
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), return_dict_in_generate=True,
                         output_scores=True, **kw)
    return out.sequences.cpu().numpy(), out.token_logprobs.cpu().numpy(), out.scores.token_logits.cpu().numpy()


def _compare_gated(toks, logp, ref_toks, ref_logp, margins, tau):
    """Up to a row's first near-tie step (margin <= tau) the tokens must agree. The numbers are compared for as long as
    the tokens do agree (the decoder has then seen the same inputs): a log-probability may differ by twice the logit
    error, once for the token's own score and once for the normaliser. Returns the number of positions compared."""
    n = min(toks.shape[1], ref_toks.shape[1]) - 1
    compared = 0
    for b in range(toks.shape[0]):
        m = margins[b, :n]
        ended = np.where(np.isnan(m))[0]
        live = ended[0] if ended.size else n
        low = np.where(~(m[:live] > tau))[0]
        gate = low[0] if low.size else live
        assert (toks[b, : gate + 1] == ref_toks[b, : gate + 1]).all(), b
        diff = np.where(toks[b, 1: live + 1] != ref_toks[b, 1: live + 1])[0]
        upto = diff[0] if diff.size else live
        assert np.abs(logp[b, :upto] - ref_logp[b, :upto]).max(initial=0) <= 2 * tau, b
        compared += upto
    return compared


MPROCS = {"plain": dict(), "rep_ngram": dict(repetition_penalty=1.3, no_repeat_ngram_size=2),
          "all": dict(repetition_penalty=1.3, encoder_repetition_penalty=0.9, no_repeat_ngram_size=3, encoder_no_repeat_ngram_size=3,
                      bad_words_ids=[[7], [5, 9]], suppress_tokens=[3], begin_suppress_tokens=[2])}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("spec_name,seed", [("tiny", 1), ("mini", 2)])
@pytest.mark.parametrize("name", list(MPROCS))
def test_model_matches_the_oracle(models, dtype, spec_name, seed, name):
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    kw = MPROCS[name]
    ids, mask = synthetic_token_batch(6, 16, spec.vocab_size, seed=41, lengths="uniform")
    T = 14
    toks, logp, logit = _scored(model, ids, mask, max_new_tokens=T, **kw)
    ref, ref_logit, ref_logp, margins = oscores.generate(_oracle(spec_name, seed, dtype), ids, mask, T,
                                                         olp.Processors(eos_token_id=[1], **kw) if kw else None)
    assert _compare_gated(toks, logp, ref, ref_logp, margins, TAU[dtype]) > 6
    assert _compare_gated(toks, logit, ref, ref_logit, margins, TAU[dtype]) > 6


def test_flan_t5_small_vs_hf_transition_scores_and_loss(models):
    pytest.importorskip("transformers")
    from oracle.hf_anchor import hf_teacher_forced_logits, load_hf_model

    spec = SPECS["flan-t5-small"]
    model, ckpt = models("flan-t5-small", 3)
    B, S, T = 16, 96, 24
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths="uniform")
    hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
    tids, tmask = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    for kw in (dict(), dict(repetition_penalty=1.3, no_repeat_ngram_size=3)):
        with torch.no_grad():
            ref = hf.generate(input_ids=tids, attention_mask=tmask, max_new_tokens=T, min_new_tokens=T, do_sample=False, num_beams=1,
                              return_dict_in_generate=True, output_scores=True, **kw)
            ref_logp = hf.compute_transition_scores(ref.sequences, ref.scores, normalize_logits=True).float().cpu().numpy()
            ref_logit = hf.compute_transition_scores(ref.sequences, ref.scores, normalize_logits=False).float().cpu().numpy()
        ref_toks = ref.sequences.cpu().numpy()
        out = model.generate(input_ids=tids, attention_mask=tmask, max_new_tokens=T, min_new_tokens=T, return_dict_in_generate=True,
                             output_scores=True, **kw)
        # the two-line transformers idiom, unchanged
        logp = model.compute_transition_scores(out.sequences, out.scores, normalize_logits=True).cpu().numpy()
        logit = model.compute_transition_scores(out.sequences, out.scores, normalize_logits=False).cpu().numpy()
        lg = hf_teacher_forced_logits(hf, ids, mask, ref_toks[:, :-1])
        proc = olp.Processors(eos_token_id=[1], min_new_tokens=T, **kw)
        margins = np.zeros((B, T))
        for t in range(T):
            s = olp.process(lg[:, t].astype(np.float32), ref_toks[:, : t + 1], ids, proc)
            top2 = np.partition(s, -2, axis=-1)[:, -2:]
            margins[:, t] = top2[:, 1] - top2[:, 0]
        toks = out.sequences.cpu().numpy()
        n = _compare_gated(toks, logp, ref_toks, ref_logp, margins, TAU[torch.bfloat16])
        _compare_gated(toks, logit, ref_toks, ref_logit, margins, TAU[torch.bfloat16])
        print(f"flan-t5-small {kw or 'plain'}: {n} of {B * T} positions compared with transformers")
        assert n >= 2 * B
    # score() against transformers' loss and per-token log-probabilities, ragged labels
    rng = np.random.default_rng(5)
    L = 12
    labels = rng.integers(2, spec.vocab_size, size=(B, L)).astype(np.int64)
    for b, k in enumerate(rng.integers(1, L + 1, size=B)):
        labels[b, k:] = -100
    with torch.no_grad():
        fo = hf(input_ids=tids, attention_mask=tmask, labels=torch.from_numpy(labels).cuda())
        lsm = torch.log_softmax(fo.logits.float(), -1)
    want = lsm.gather(2, torch.from_numpy(np.where(labels == -100, 0, labels)).cuda()[..., None])[..., 0].cpu().numpy()
    want = np.where(labels == -100, 0, want)
    res = model.score(input_ids=tids, attention_mask=tmask, labels=torch.from_numpy(labels))
    got = res.token_logprobs.cpu().numpy()
    assert got.shape == labels.shape and (got[labels == -100] == 0).all()
    assert np.abs(got - want).max() <= 2 * TAU[torch.bfloat16]
    assert abs(float(res.loss) - float(fo.loss.float())) <= 2 * TAU[torch.bfloat16]
    assert (res.lengths.cpu().numpy() == (labels != -100).sum(1)).all()


def _launches(model):
    return int(model.stats()["kernel_launches"])


@pytest.mark.parametrize("kw", [dict(), dict(repetition_penalty=1.3, no_repeat_ngram_size=2)], ids=["plain", "proc"])
def test_scoring_changes_no_token_and_no_launch_of_a_plain_call(models, kw):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(9, 20, spec.vocab_size, seed=8, lengths="uniform")
    a = dict(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=16, **kw)
    before = model.generate(**a)
    n_before = _launches(model)
    out = model.generate(**a, return_dict_in_generate=True, output_scores=True)
    assert _launches(model) == n_before + 1  # the reset of the result arrays; the step graph has as many nodes
    after = model.generate(**a)
    assert _launches(model) == n_before
    assert torch.equal(out.sequences, before) and torch.equal(after, before)
    no_scores = model.generate(**a, return_dict_in_generate=True)
    assert no_scores.scores is None and no_scores.token_logprobs is None and torch.equal(no_scores.sequences, before)
    assert _launches(model) == n_before
    assert torch.equal(model.generate(**a, output_scores=True), before)  # without return_dict_in_generate: the tensor, as transformers


def test_result_shape_and_conventions(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(32, 24, spec.vocab_size, seed=21, lengths="uniform")
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=20,
                         return_dict_in_generate=True, output_scores=True)
    seq, logp, logit = out.sequences.cpu().numpy(), out.token_logprobs.cpu().numpy(), out.scores.token_logits.cpu().numpy()
    assert out.token_logprobs.dtype == torch.float32 and out.token_logprobs.is_cuda
    assert logp.shape == (32, seq.shape[1] - 1) == logit.shape and len(out.scores) == logp.shape[1]
    lens = model.last_lengths.cpu().numpy()
    assert len(set(lens.tolist())) > 2  # rows end at different steps
    pos = np.arange(logp.shape[1])[None, :]
    assert (logp[pos >= lens[:, None]] == 0).all() and (logit[pos >= lens[:, None]] == 0).all()
    assert (logp[pos < lens[:, None]] < 0).all() and np.isfinite(logp).all()
    assert model.compute_transition_scores(out.sequences, out.scores, normalize_logits=False) is out.scores.token_logits
    assert model.compute_transition_scores(out.sequences, out.scores, normalize_logits=True) is out.token_logprobs
    with pytest.raises(TypeError):
        model.compute_transition_scores(out.sequences, (out.token_logprobs,))


def test_headline_shape_tokens_are_unchanged_by_scoring(models):
    spec = SPECS["flan-t5-base"]
    model, _ = models("flan-t5-base", 0)
    ids, mask = synthetic_token_batch(256, 512, spec.vocab_size, seed=0, lengths="full")
    a = dict(input_ids=torch.from_numpy(ids).cuda(), attention_mask=torch.from_numpy(mask).cuda(), max_new_tokens=128, min_new_tokens=128)
    plain = model.generate(**a)
    n_plain = _launches(model)
    out = model.generate(**a, return_dict_in_generate=True, output_scores=True)
    again = model.generate(**a, return_dict_in_generate=True, output_scores=True)
    assert torch.equal(out.sequences, plain)
    assert torch.equal(out.token_logprobs.view(torch.int32), again.token_logprobs.view(torch.int32))  # run to run
    assert out.token_logprobs.shape == (256, 128) and bool((out.token_logprobs < 0).all()) and bool(torch.isfinite(out.token_logprobs).all())
    assert torch.equal(model.generate(**a), plain) and _launches(model) == n_plain


def _static_rows(model, ids, mask, pool, **kw):
    """Row for row through generate_host and generate in `pool`-row batches (the last one padded with copies of its
    first row); both must return the same bits."""
    N, T = ids.shape[0], kw["max_new_tokens"]
    out = np.zeros((N, T + 1), dtype=np.int64)
    logp = np.zeros((N, T), dtype=np.float32)
    logit = np.zeros((N, T), dtype=np.float32)
    for lo in range(0, N, pool):
        hi = min(lo + pool, N)
        bi, bm = ids[lo:hi], mask[lo:hi]
        if hi - lo < pool:
            bi = np.concatenate([bi, np.repeat(bi[:1], pool - (hi - lo), 0)])
            bm = np.concatenate([bm, np.repeat(bm[:1], pool - (hi - lo), 0)])
        o, _, lp, lg = model.generate_host(bi, bm, output_scores=True, **kw)
        out[lo:hi, : o.shape[1]] = o[: hi - lo]
        logp[lo:hi, : lp.shape[1]] = lp[: hi - lo]
        logit[lo:hi, : lg.shape[1]] = lg[: hi - lo]
        d_seq, d_lp, d_lg = _scored(model, bi, bm, **kw)
        assert np.array_equal(d_seq, o) and np.array_equal(d_lp.view(np.int32), lp.view(np.int32))
        assert np.array_equal(d_lg.view(np.int32), lg.view(np.int32))
    return out, logp, logit


@pytest.mark.parametrize("admit", [4, 1])
@pytest.mark.parametrize("kw", [dict(), dict(repetition_penalty=1.4, no_repeat_ngram_size=2, eos_token_id=[1, 6])], ids=["plain", "proc"])
def test_entry_points_agree_bit_for_bit(models, admit, kw):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(150, 24, spec.vocab_size, seed=21, lengths="uniform")
    kw = dict(max_new_tokens=20, **kw)
    ref, ref_lp, ref_lg = _static_rows(model, ids, mask, 32, **kw)
    out, lens, lp, lg = model.generate_stream(ids, mask, pool=32, admit_min=admit, output_scores=True, **kw)
    assert len(set(lens.tolist())) > 3  # natural EOS: slots are refilled at different times
    w = out.shape[1]
    assert (out == ref[:, :w]).all()
    assert np.array_equal(lp.view(np.int32), ref_lp[:, : w - 1].view(np.int32))
    assert np.array_equal(lg.view(np.int32), ref_lg[:, : w - 1].view(np.int32))
    assert (ref_lp[:, w - 1:] == 0).all()
    out2, _, lp2, _ = model.generate_stream(ids, mask, pool=32, admit_min=admit, output_scores=True, **kw)
    assert np.array_equal(out2, out) and np.array_equal(lp2.view(np.int32), lp.view(np.int32))  # run to run
    plain, _ = model.generate_stream(ids, mask, pool=32, admit_min=admit, **kw)
    assert np.array_equal(plain, out)


def test_600_rows_through_the_slot_pool_and_static_chunks(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(600, 24, spec.vocab_size, seed=33, lengths="uniform")
    kw = dict(max_new_tokens=16)
    seq, lp, lg = _scored(model, ids, mask, **kw)  # > pool_size rows: the slot pool
    assert seq.shape[0] == 600 and np.array_equal(seq, model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw).cpu().numpy())
    for lo in (0, 256, 512):
        p_seq, p_lp, p_lg = _scored(model, ids[lo:lo + 256], mask[lo:lo + 256], **kw)  # static batches
        w = p_lp.shape[1]
        assert np.array_equal(p_lp.view(np.int32), lp[lo:lo + 256, :w].view(np.int32)) and (lp[lo:lo + 256, w:] == 0).all()
        assert np.array_equal(p_lg.view(np.int32), lg[lo:lo + 256, :w].view(np.int32))
    # prompts longer than the slot pool takes: static chunks of pool_size rows
    ids2, mask2 = synthetic_token_batch(300, 520, spec.vocab_size, seed=3, lengths="uniform")
    seq2, lp2, _ = _scored(model, ids2, mask2, max_new_tokens=10)
    a_seq, a_lp, _ = _scored(model, ids2[:256], mask2[:256], max_new_tokens=10)
    b_seq, b_lp, _ = _scored(model, ids2[256:], mask2[256:], max_new_tokens=10)
    assert np.array_equal(lp2[:256, : a_lp.shape[1]].view(np.int32), a_lp.view(np.int32))
    assert np.array_equal(lp2[256:, : b_lp.shape[1]].view(np.int32), b_lp.view(np.int32))
    assert np.array_equal(seq2[:256, : a_seq.shape[1]], a_seq) and np.array_equal(seq2[256:, : b_seq.shape[1]], b_seq)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_score_of_a_generation_returns_the_generations_own_numbers(models, dtype):
    spec = SPECS["mini"]
    model, _ = models("mini", 2, dtype)
    ids, mask = synthetic_token_batch(40, 20, spec.vocab_size, seed=8, lengths="uniform")
    seq, lp, _ = _scored(model, ids, mask, max_new_tokens=16)
    lens = model.last_lengths.cpu().numpy()
    labels = seq[:, 1:].copy()
    labels[np.arange(labels.shape[1])[None, :] >= lens[:, None]] = -100
    res = model.score(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), labels=torch.from_numpy(labels))
    assert np.array_equal(res.token_logprobs.cpu().numpy().view(np.int32), lp.view(np.int32))
    assert (res.lengths.cpu().numpy() == lens).all()
    assert abs(float(res.loss) + lp.astype(np.float64).sum() / lens.sum()) <= 1e-6 * abs(float(res.loss)) + 1e-6
    one = model.score(input_ids=torch.from_numpy(ids[:1]), attention_mask=torch.from_numpy(mask[:1]), labels=torch.from_numpy(labels[:1]))
    assert abs(float(one.token_logprobs.sum()) + float(one.loss) * int(lens[0])) <= 1e-4
    # more rows than one pool of slots: the same numbers through the slot pool
    old = model.pool_size, model.pool_slots
    model.pool_size = model.pool_slots = 16  # 40 rows through 16 slots: refills
    try:
        pooled = model.score(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), labels=torch.from_numpy(labels))
    finally:
        model.pool_size, model.pool_slots = old
    assert np.array_equal(pooled.token_logprobs.cpu().numpy().view(np.int32), lp.view(np.int32))


def test_validation(models):
    model, _ = models("tiny", 1)
    V = SPECS["tiny"].vocab_size
    ids = torch.ones((2, 8), dtype=torch.long)
    for k in ("output_logits", "output_attentions", "output_hidden_states"):
        with pytest.raises(NotImplementedError):
            model.generate(input_ids=ids, max_new_tokens=4, return_dict_in_generate=True, **{k: True})
        with pytest.raises(NotImplementedError):
            model.generate_host(ids.numpy(), max_new_tokens=4, **{k: True})
    for bad in ([[V, 1]], [[-100, 1]], [[1, -100, 2]], [[-3, 1]]):
        with pytest.raises(ValueError):
            model.score(input_ids=ids[:1], labels=torch.tensor(bad))
    with pytest.raises(ValueError):
        model.score(input_ids=ids, labels=torch.tensor([[1, 2]]))  # one row of labels for two prompts
    # the library checks what reaches it directly
    lib, h = model._lib, model._h
    gp = _lib.GenParams(max_new_tokens=4, min_new_tokens=0, eos_token_id=-1, pad_token_id=-1, decoder_start_token_id=-1, poll_interval=8)
    idn = np.ones((2, 8), dtype=np.int64)
    out, lens = np.zeros((2, 5), dtype=np.int64), np.zeros(2, dtype=np.int32)
    logp = np.zeros((2, 4), dtype=np.float32)
    keep = []
    lp = _params(dict(repetition_penalty=1.3), keep)

    def call(labels, forced_len=None, logits=None, stream=False, logprobs=logp):
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.int64)
        io = _lib.ScoreIO(token_logprobs=None if logprobs is None else logprobs.ctypes.data_as(C.c_void_p), token_logits=None,
                          forced_ids=None if lab is None else lab.ctypes.data_as(C.c_void_p),
                          forced_len=(lab.shape[1] if lab is not None else 0) if forced_len is None else forced_len)
        common = (h, idn.ctypes.data_as(C.c_void_p), None)
        tail = (out.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p), C.byref(io))
        if stream:
            return lib.b200t5_generate_stream_scored(*common, 2, 8, C.byref(gp), logits, 2, 0, *tail)
        return lib.b200t5_generate_host_scored(*common, 2, 8, C.byref(gp), logits, *tail)

    for stream in (False, True):
        assert call([[1, 2], [3, -100]], stream=stream) == _lib.OK
        assert call([[V, 2], [3, 4]], stream=stream) == _lib.EINVAL
        assert call([[1, -100, 2], [3, 4, 5]], stream=stream) == _lib.EINVAL
        assert call([[-100, 2], [3, 4]], stream=stream) == _lib.EINVAL
        assert call([[1, 2, 3, 4, 5], [1, 2, 3, 4, 5]], stream=stream) == _lib.EINVAL  # forced_len > max_new_tokens
        assert call([[1, 2], [3, 4]], forced_len=0, stream=stream) == _lib.EINVAL
        assert call([[1, 2], [3, 4]], logits=C.byref(lp), stream=stream) == _lib.EINVAL
        assert "logits processors" in _lib.last_error(h, lib)
        assert call(None, logprobs=None, stream=stream) == _lib.EINVAL
        assert call(None, logits=C.byref(lp), stream=stream) == _lib.OK
