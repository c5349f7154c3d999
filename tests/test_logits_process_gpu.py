"""Greedy logits processors on the CUDA path (csrc/logits_process.cuh, EpiLmHead<true, *>): the fused kernel against
transformers' processor classes run by torch on the same GPU, the model against the numpy oracle and against HF
generate, properties that need no reference, and the invariances of the three entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch
from oracle import logits_process as olp

pytestmark = pytest.mark.gpu

DEV = 0
TAU = 0.13  # margin gate in logit units, as tests/test_model_gpu.py


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ----------------------------------------------------------------------------------------------------- kernel
def _params(d, keep):
    """b200t5_logits_params from a dict of processor values; `keep` holds the arrays alive."""
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


def _torch_processors(d, V, enc, eos, min_new):
    from transformers.generation import logits_process as lp

    chain = []
    if d.get("encoder_repetition_penalty", 1.0) != 1.0:
        chain.append(lp.EncoderRepetitionPenaltyLogitsProcessor(d["encoder_repetition_penalty"], enc))
    if d.get("repetition_penalty", 1.0) != 1.0:
        chain.append(lp.RepetitionPenaltyLogitsProcessor(d["repetition_penalty"]))
    if d.get("no_repeat_ngram_size"):
        chain.append(lp.NoRepeatNGramLogitsProcessor(d["no_repeat_ngram_size"]))
    if d.get("encoder_no_repeat_ngram_size"):
        chain.append(lp.EncoderNoRepeatNGramLogitsProcessor(d["encoder_no_repeat_ngram_size"], enc))
    if d.get("bad_words_ids"):
        chain.append(lp.NoBadWordsLogitsProcessor(d["bad_words_ids"], eos))
    if min_new:
        chain.append(lp.MinNewTokensLengthLogitsProcessor(1, min_new, eos, device="cuda"))
    if d.get("suppress_tokens"):
        chain.append(lp.SuppressTokensLogitsProcessor(d["suppress_tokens"], device="cuda"))
    if d.get("begin_suppress_tokens"):
        chain.append(lp.SuppressTokensAtBeginLogitsProcessor(d["begin_suppress_tokens"], 1, device="cuda"))
    return chain


KPROCS = {
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


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
@pytest.mark.parametrize("V", [1000, 32128])
@pytest.mark.parametrize("M", [1, 7, 256])
@pytest.mark.parametrize("step", [0, 5])
@pytest.mark.parametrize("name", list(KPROCS))
def test_kernel_matches_hf_processors_on_the_gpu(flavour, V, M, step, name):
    pytest.importorskip("transformers")
    lib = _lib.load(flavour)
    dt = torch.bfloat16 if flavour == "bf16" else torch.float16
    d = KPROCS[name]
    K, S = 256, 40
    g = torch.Generator(device="cuda").manual_seed(M * 7 + step + V)
    x = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(V, K, device="cuda", generator=g) * 0.2).to(dt)
    W[3] = W[4]  # two equal columns: the first-index tie rule under processing
    hist = torch.randint(0, 12, (M, step + 1), device="cuda", generator=g)
    hist[:, 0] = 0
    if step >= 4:
        hist[0, 1:5] = torch.tensor([2, 3, 2, 3])  # a repeated n-gram and a bad-word prefix at the end
    enc = torch.randint(0, 12, (M, S), device="cuda", generator=g)
    enc[:, S - 5:] = 0  # padding
    eos_list = d.get("eos", [1])
    min_new = step + 1 if d.get("min_new") else 0
    keep = []
    raw = torch.full((M, V), float("nan"), device="cuda")
    tok0 = torch.empty(M, dtype=torch.long, device="cuda")
    noop = _lib.LogitsParams(repetition_penalty=1.0, encoder_repetition_penalty=1.0)
    _lib.check(lib.b200t5_test_lm_process(DEV, P(x), P(W), M, V, K, step, 1, 0, C.byref(noop), P(hist), P(enc), S,
                                          P(tok0), P(raw), None), lib=lib)
    vals = torch.full((M, V), float("nan"), device="cuda")
    toks = torch.empty(M, dtype=torch.long, device="cuda")
    _lib.check(lib.b200t5_test_lm_process(DEV, P(x), P(W), M, V, K, step, 1, min_new, C.byref(_params(d, keep)), P(hist),
                                          P(enc), S, P(toks), P(vals), None), lib=lib)
    torch.cuda.synchronize()
    assert torch.equal(tok0, raw.argmax(-1))
    if flavour == "bf16" and V == 1000:  # the unprocessed values are the lm_head GEMM's fp32 logits
        ref_raw = torch.full((M, V), float("nan"), device="cuda")
        _lib.check(lib.b200t5_test_gemm(DEV, P(x), P(W), P(ref_raw), M, V, K, 128, 3, 0, None), lib=lib)
        torch.cuda.synchronize()
        assert torch.equal(raw.view(torch.int32), ref_raw.view(torch.int32))
    ref = raw.clone()
    for p in _torch_processors(d, V, enc, eos_list, min_new):
        ref = p(hist, ref)
    assert torch.equal(vals.view(torch.int32), ref.view(torch.int32)), (vals != ref).sum().item()
    assert torch.equal(toks, ref.argmax(-1))


def test_kernel_rejects_bad_arguments():
    lib = _lib.load()
    x = torch.zeros(1, 64, dtype=torch.bfloat16, device="cuda")
    W = torch.zeros(100, 64, dtype=torch.bfloat16, device="cuda")
    hist = torch.zeros(1, 1, dtype=torch.long, device="cuda")
    tok = torch.zeros(1, dtype=torch.long, device="cuda")
    keep = []
    for d in (dict(repetition_penalty=0.0), dict(no_repeat_ngram_size=-1), dict(suppress_tokens=[100]),
              dict(bad_words_ids=[[3, 100]])):
        rc = lib.b200t5_test_lm_process(DEV, P(x), P(W), 1, 100, 64, 0, 1, 0, C.byref(_params(d, keep)), P(hist), P(hist),
                                        1, P(tok), None, None)
        assert rc == _lib.EINVAL


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

    if dtype == torch.float16:
        return T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate="fp16")
    return T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate_bf16=True)


def _pad_to(a, w, pad=0):
    return a if a.shape[1] >= w else np.concatenate([a, np.full((a.shape[0], w - a.shape[1]), pad, a.dtype)], 1)


def _gated(ours, ref, margins, tau=TAU):
    w = max(ours.shape[1], ref.shape[1])
    ours, ref = _pad_to(ours, w), _pad_to(ref, w)
    ok = 0
    for b in range(ours.shape[0]):
        m = margins[b]
        low = [s for s in np.where(~(m > tau))[0] if not np.isnan(m[s])]
        upto = 1 + (low[0] if low else m.shape[0])
        ok += int((ours[b, :upto] == ref[b, :upto]).all())
    return ok / ours.shape[0]


MPROCS = {
    "rep": dict(repetition_penalty=1.5),
    "enc_rep": dict(encoder_repetition_penalty=1.5),
    "ngram": dict(no_repeat_ngram_size=2),
    "enc_ngram": dict(encoder_no_repeat_ngram_size=2),
    "bad": dict(bad_words_ids=[[1], [7], [5, 9]]),
    "suppress": dict(suppress_tokens=[3, 4], begin_suppress_tokens=[1, 2]),
    "all": dict(repetition_penalty=1.3, encoder_repetition_penalty=0.9, no_repeat_ngram_size=3,
                encoder_no_repeat_ngram_size=3, bad_words_ids=[[7], [5, 9]], suppress_tokens=[3],
                begin_suppress_tokens=[2]),
}


def _oproc(kw, eos=(1,), min_new=0):
    return olp.Processors(eos_token_id=list(eos), min_new_tokens=min_new, **kw)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("spec_name,seed", [("tiny", 1), ("mini", 2)])
@pytest.mark.parametrize("name", list(MPROCS))
def test_model_matches_the_oracle(models, dtype, spec_name, seed, name):
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed, dtype)
    kw = MPROCS[name]
    ids, mask = synthetic_token_batch(6, 16, spec.vocab_size, seed=41, lengths="uniform")
    T = 14
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T,
                         **kw).cpu().numpy()
    ref, margins = olp.generate(_oracle(spec_name, seed, dtype), ids, mask, T, _oproc(kw), return_margins=True)
    assert _gated(out, ref, margins) == 1.0


def test_flan_t5_small_vs_hf_generate(models):
    pytest.importorskip("transformers")
    from oracle.hf_anchor import hf_teacher_forced_logits, load_hf_model

    spec = SPECS["flan-t5-small"]
    model, ckpt = models("flan-t5-small", 3)
    B, S, T = 16, 96, 24
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths="uniform")
    kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, encoder_no_repeat_ngram_size=4,
              bad_words_ids=[[7, 8], [100, 101, 102]], suppress_tokens=[3, 5])
    hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
    with torch.no_grad():
        ref = hf.generate(input_ids=torch.from_numpy(ids).cuda(), attention_mask=torch.from_numpy(mask).cuda(),
                          max_new_tokens=T, min_new_tokens=T, do_sample=False, num_beams=1, **kw).cpu().numpy()
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T,
                         min_new_tokens=T, **kw).cpu().numpy()
    assert out.shape == ref.shape
    lg = hf_teacher_forced_logits(hf, ids, mask, ref[:, :-1])
    proc = _oproc(kw, min_new=T)
    margins = np.zeros((B, T))
    for t in range(T):
        s = olp.process(lg[:, t].astype(np.float32), ref[:, : t + 1], ids, proc)
        top2 = np.partition(s, -2, axis=-1)[:, -2:]
        margins[:, t] = top2[:, 1] - top2[:, 0]
    print(f"flan-t5-small with processors vs HF: token agreement {(out == ref).mean():.3f}")
    assert _gated(out, ref, margins) == 1.0


def _has_repeated_ngram(row, n):
    grams = [tuple(row[i:i + n]) for i in range(len(row) - n + 1)]
    return len(grams) != len(set(grams))


def test_properties_without_a_reference(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(32, 24, spec.vocab_size, seed=5, lengths="uniform")
    bad = [[7, 8], [9, 10, 11], [12]]
    supp = [13, 14, 15]
    for n in (1, 2, 3):
        out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=40,
                             min_new_tokens=40, no_repeat_ngram_size=n, bad_words_ids=bad, suppress_tokens=supp).cpu().numpy()
        for row in out:
            assert not _has_repeated_ngram(row.tolist(), n)
            r = row.tolist()
            for w in bad:
                assert not any(r[i:i + len(w)] == w for i in range(len(r) - len(w) + 1))
            assert not set(r) & set(supp)


def test_no_op_values_are_plain_greedy(models):
    spec = SPECS["mini"]
    model, _ = models("mini", 2)
    ids, mask = synthetic_token_batch(9, 20, spec.vocab_size, seed=8, lengths="uniform")
    a = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=16).cpu().numpy()
    la = model.stats()["kernel_launches"]
    b = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=16,
                       repetition_penalty=1.0, encoder_repetition_penalty=1.0, no_repeat_ngram_size=0,
                       encoder_no_repeat_ngram_size=0, suppress_tokens=[], begin_suppress_tokens=[], eos_token_id=[1, 1]).cpu().numpy()
    assert np.array_equal(a, b) and model.stats()["kernel_launches"] == la


def _static_rows(model, ids, mask, pool, **kw):
    N, T = ids.shape[0], kw["max_new_tokens"]
    out = np.zeros((N, T + 1), dtype=np.int64)
    lens = np.zeros(N, dtype=np.int32)
    for lo in range(0, N, pool):
        hi = min(lo + pool, N)
        bi, bm = ids[lo:hi], mask[lo:hi]
        if hi - lo < pool:
            bi = np.concatenate([bi, np.repeat(bi[:1], pool - (hi - lo), 0)])
            bm = np.concatenate([bm, np.repeat(bm[:1], pool - (hi - lo), 0)])
        o, ln = model.generate_host(bi, bm, **kw)
        out[lo:hi, : o.shape[1]] = o[: hi - lo]
        lens[lo:hi] = ln[: hi - lo]
        dev = model.generate(input_ids=torch.from_numpy(bi), attention_mask=torch.from_numpy(bm), **kw).cpu().numpy()
        assert np.array_equal(dev, o)
    return out, lens


@pytest.mark.parametrize("admit", [4, 1])
def test_entry_points_agree_with_pool_refills(models, admit):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(150, 24, spec.vocab_size, seed=21, lengths="uniform")
    kw = dict(max_new_tokens=20, repetition_penalty=1.4, no_repeat_ngram_size=2, encoder_no_repeat_ngram_size=3,
              bad_words_ids=[[5, 9], [7]], suppress_tokens=[3], begin_suppress_tokens=[2], eos_token_id=[1, 6])
    ref, ref_len = _static_rows(model, ids, mask, 32, **kw)
    out, lens = model.generate_stream(ids, mask, pool=32, admit_min=admit, **kw)
    assert len(set(ref_len.tolist())) > 3
    assert (lens == ref_len).all()
    w = out.shape[1]
    assert (out == ref[:, :w]).all()
    # a plain call on the same handle afterwards is unaffected by the processor state
    plain, _ = model.generate_stream(ids, mask, pool=32, admit_min=admit, max_new_tokens=20)
    plain_ref, _ = _static_rows(model, ids, mask, 32, max_new_tokens=20)
    assert (plain == plain_ref[:, : plain.shape[1]]).all()


def test_static_chunks_beyond_256_rows(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(300, 520, spec.vocab_size, seed=3, lengths="uniform")
    kw = dict(max_new_tokens=10, repetition_penalty=1.3, no_repeat_ngram_size=2, encoder_no_repeat_ngram_size=2)
    full = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw).cpu().numpy()
    parts = [model.generate(input_ids=torch.from_numpy(ids[lo:hi]), attention_mask=torch.from_numpy(mask[lo:hi]), **kw).cpu().numpy()
             for lo, hi in ((0, 256), (256, 300))]
    w = full.shape[1]
    assert np.array_equal(full, np.concatenate([_pad_to(p, w) for p in parts]))


def test_eos_token_list_behaves_as_in_hf(models):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(8, 16, spec.vocab_size, seed=12, lengths="uniform")
    plain = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=24,
                           min_new_tokens=24).cpu().numpy()
    second = int(np.bincount(plain[:, 1:].ravel(), minlength=spec.vocab_size)[2:].argmax()) + 2  # a frequent token
    eos = [1, second]
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=24,
                         eos_token_id=eos).cpu().numpy()
    ref, margins = olp.generate(_oracle("tiny", 1, torch.bfloat16), ids, mask, 24, _oproc({}, eos=eos), return_margins=True)
    assert _gated(out, ref, margins) == 1.0
    for row in out:
        hits = [i for i in range(1, len(row)) if row[i] in eos]
        if hits:
            assert (row[hits[0] + 1:] == 0).all()
    forced = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=12,
                            min_new_tokens=12, eos_token_id=eos).cpu().numpy()
    assert not np.isin(forced[:, 1:], eos).any()


def test_batch_predictor_passes_processor_kwargs_through(models):
    from transformers import T5Tokenizer

    from anyscale_workshop_nyc_2023_b200 import rayshim
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir, make_batch_predictor

    spec = SPECS["tiny"]
    ckpt = checkpoint_dir("tiny", seed=1)
    ids, mask = synthetic_token_batch(10, 24, spec.vocab_size, seed=31, lengths="uniform")
    ds = rayshim.data.from_numpy({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()})
    bp = make_batch_predictor(ckpt, device_map="auto", torch_dtype=torch.bfloat16)
    out = bp.predict(ds, batch_size=4, num_gpus_per_worker=1, max_scoring_workers=1, max_new_tokens=12,
                     no_repeat_ngram_size=3).to_pandas()
    model, _ = models("tiny", 1)
    tok = T5Tokenizer.from_pretrained(str(ckpt))
    want = []
    for lo in range(0, 10, 4):
        a = dict(input_ids=torch.from_numpy(ids[lo:lo + 4]), attention_mask=torch.from_numpy(mask[lo:lo + 4]), max_new_tokens=12)
        want += tok.batch_decode(model.generate(**a, no_repeat_ngram_size=3), skip_special_tokens=True)
    assert out["generated_output"].tolist() == want


def test_validation(models):
    model, _ = models("tiny", 1)
    ids = torch.ones((2, 8), dtype=torch.long)
    V = SPECS["tiny"].vocab_size
    for kw in (dict(repetition_penalty=0.0), dict(encoder_repetition_penalty=-1.0), dict(no_repeat_ngram_size=-1),
               dict(encoder_no_repeat_ngram_size=-3), dict(bad_words_ids=[]), dict(bad_words_ids=[[]]),
               dict(bad_words_ids=[[V]]), dict(suppress_tokens=[V]), dict(begin_suppress_tokens=[-1])):
        with pytest.raises(ValueError):
            model.generate(input_ids=ids, max_new_tokens=4, **kw)
        with pytest.raises(ValueError):
            model.generate_host(ids.numpy(), max_new_tokens=4, **kw)
    with pytest.raises(NotImplementedError):
        model.generate(input_ids=ids, do_sample=True, no_repeat_ngram_size=2)
