"""End-to-end parity of the CUDA path (through libb200t5.so) on an H100.

Anchors, strongest first:
  1. committed golden fixtures: transformers' own generate()/forward on seeded checkpoints
     (tests/golden/make_golden.py, HF eager bf16 + fp32 on CPU);
  2. oracle/t5_oracle.py with bf16 rounding emulation (pinned to the same fixtures on CPU);
  3. HF eager bf16 on this GPU (same dtype, cuBLAS) when transformers is importable.

Token IDs are integers and must match exactly wherever the decision is not a numerical
near-tie: a (row, step) whose top-1/top-2 logit gap in the oracle is below TAU is a
coin-flip between implementations that differ only in fp32 accumulation order (SURVEY 7.3),
so rows are compared up to their first such step ("margin-gated"), and the ungated match
rate is printed. Logit tolerance: bf16 outputs, |err| <= LOGIT_ATOL (about 4 bf16 ulps at
the logit scale of these models), mean |err| <= LOGIT_MEAN.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200.synth import SPECS, make_state_dict, save_checkpoint, synthetic_token_batch

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden"
TAU = 0.13          # margin gate, in logit units (bf16 ulp at |logit| in [4,8) is 0.03125)
# Tolerances are set from the noise floor between independent bf16 implementations of the same
# forward (tools/diag_parity.py measures it: HF-bf16-GPU vs HF-bf16-CPU against ours vs HF-bf16-GPU).
# The 2-3 layer test models sit well below that floor.
LOGIT_ATOL = 0.5
LOGIT_MEAN = 0.05

CASES = {"tiny_a": ("tiny", 1, 12), "tiny_full": ("tiny", 1, 10), "mini_a": ("mini", 2, 16)}


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(spec_name, seed):
        key = (spec_name, seed)
        if key not in cache:
            d = tmp_path_factory.mktemp(f"ckpt_{spec_name}_{seed}")
            save_checkpoint(d, SPECS[spec_name], seed=seed)
            cache[key] = (B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=torch.bfloat16), d)
        return cache[key]

    return get


def oracle_for(spec_name, seed, emulate=True):
    from oracle.t5_oracle import T5Oracle

    return T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate_bf16=emulate)


def pad_to(a, width, pad=0):
    if a.shape[1] >= width:
        return a
    return np.concatenate([a, np.full((a.shape[0], width - a.shape[1]), pad, a.dtype)], axis=1)


def gated_prefix_match(ours, ref, margins, tau=TAU):
    """Rows must agree up to (excluding) the first step whose oracle margin is <= tau."""
    w = max(ours.shape[1], ref.shape[1])
    ours, ref = pad_to(ours, w), pad_to(ref, w)
    n_rows, gated_ok, full_ok = ours.shape[0], 0, 0
    for b in range(n_rows):
        m = margins[b]
        low = np.where(~(m > tau))[0]  # NaN (finished) counts as safe
        low = [s for s in low if not np.isnan(m[s])]
        first_low = low[0] if low else m.shape[0]
        upto = 1 + first_low  # column 0 is the start token; step s writes column s+1
        gated_ok += int((ours[b, :upto] == ref[b, :upto]).all())
        full_ok += int((ours[b] == ref[b]).all())
    return gated_ok / n_rows, full_ok / n_rows


@pytest.mark.parametrize("case", list(CASES))
def test_golden_generate(models, case):
    spec_name, seed, T = CASES[case]
    g = np.load(GOLD / f"{case}.npz")
    model, _ = models(spec_name, seed)
    out = model.generate(input_ids=torch.from_numpy(g["ids"]), attention_mask=torch.from_numpy(g["mask"]),
                         labels=torch.from_numpy(g["ids"]), max_new_tokens=T).cpu().numpy()
    orc = oracle_for(spec_name, seed)
    otoks, margins = orc.generate(g["ids"], g["mask"], max_new_tokens=T, return_margins=True)
    assert out[:, 0].tolist() == [0] * out.shape[0]
    gated_o, full_o = gated_prefix_match(out, otoks, margins)
    gated_h, full_h = gated_prefix_match(out, g["tokens_bf16"], margins)
    print(f"{case}: vs oracle gated={gated_o:.2f} full={full_o:.2f} | vs HF-bf16 golden gated={gated_h:.2f} full={full_h:.2f}")
    assert gated_o == 1.0 and gated_h == 1.0
    # forced length: min_new_tokens == max_new_tokens -> every row is exactly T tokens long
    forced = model.generate(input_ids=torch.from_numpy(g["ids"]), attention_mask=torch.from_numpy(g["mask"]),
                            max_new_tokens=T, min_new_tokens=T).cpu().numpy()
    assert forced.shape == (g["ids"].shape[0], T + 1)
    assert (forced[:, 1:] != SPECS[spec_name].eos_token_id).all()
    ftoks, fm = orc.generate(g["ids"], g["mask"], max_new_tokens=T, min_new_tokens=T, return_margins=True)
    gated_f, full_f = gated_prefix_match(forced, ftoks, fm)
    gated_fh, full_fh = gated_prefix_match(forced, g["forced_bf16"], fm)
    print(f"{case} forced: vs oracle gated={gated_f:.2f} full={full_f:.2f} | vs golden gated={gated_fh:.2f} full={full_fh:.2f}")
    assert gated_f == 1.0 and gated_fh == 1.0


@pytest.mark.parametrize("case", list(CASES))
def test_golden_logits_and_encoder(models, case):
    spec_name, seed, T = CASES[case]
    g = np.load(GOLD / f"{case}.npz")
    model, _ = models(spec_name, seed)
    valid = g["mask"].astype(bool)
    enc = model.encode(g["ids"], g["mask"]).float().cpu().numpy()
    e_err = np.abs(enc - g["enc_bf16"])[valid]
    print(f"{case}: encoder max err {e_err.max():.4f} mean {e_err.mean():.5f} (scale {np.abs(g['enc_bf16'])[valid].max():.2f})")
    assert e_err.max() <= 0.15 and e_err.mean() <= 0.01
    dec_in = g["tokens_bf16"][:, :-1]
    logits = model.decode_logits(g["ids"], g["mask"], dec_in).cpu().numpy()
    ref = g["logits_bf16"]
    # positions after a row's EOS are fed pad tokens in both; compare everything
    err = np.abs(logits - ref)
    print(f"{case}: logits max err {err.max():.4f} mean {err.mean():.5f} (scale {np.abs(ref).max():.2f})")
    assert err.max() <= LOGIT_ATOL and err.mean() <= LOGIT_MEAN


def test_host_entry_point_and_lengths(models):
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(7, 19, SPECS["tiny"].vocab_size, seed=5, lengths="uniform")
    dev = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=14).cpu().numpy()
    host, lens = model.generate_host(ids, mask, max_new_tokens=14)
    assert dev.shape == host.shape and (dev == host).all()
    eos, pad = 1, 0
    for b in range(ids.shape[0]):
        row = host[b, 1:]
        n = int(lens[b])
        assert (row[n:] == pad).all()
        assert (row[: max(n - 1, 0)] != eos).all()
        if n < row.shape[0]:
            assert row[n - 1] == eos
    st = model.stats()
    assert st["kernel_launches"] > 0 and st["decode_steps"] >= int(lens.max())


def test_default_max_length_and_validation(models):
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(2, 8, SPECS["tiny"].vocab_size, seed=6, lengths="full")
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), min_length=20)
    assert out.shape == (2, 20)  # HF default max_length=20 -> 19 new tokens + start token
    with pytest.raises(NotImplementedError):
        model.generate(input_ids=torch.from_numpy(ids), do_sample=True)
    with pytest.raises(IndexError):
        model.generate(input_ids=torch.full((1, 4), 10 ** 6))
    assert model.device.type == "cuda"


@pytest.mark.parametrize("B,S,lengths", [(1, 1, "full"), (3, 5, "uniform"), (9, 130, "uniform"), (2, 64, "full")])
def test_edge_shapes_vs_oracle(models, B, S, lengths):
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=B * 100 + S, lengths=lengths, min_len=1)
    T = 8
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T).cpu().numpy()
    otoks, margins = oracle_for("tiny", 1).generate(ids, mask, max_new_tokens=T, return_margins=True)
    gated, full = gated_prefix_match(out, otoks, margins)
    print(f"edge B={B} S={S}: gated={gated:.2f} full={full:.2f}")
    assert gated == 1.0


def test_mask_holes_and_fully_masked_row(models):
    """Non-prefix masks and an all-zero mask row follow HF's additive-mask semantics."""
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(4, 20, spec.vocab_size, seed=77, lengths="full")
    mask[1, 3:7] = 0
    mask[2, :] = 0
    T = 6
    orc = oracle_for("tiny", 1)
    dec = np.zeros((4, T), dtype=np.int64)
    dec[:, 1:] = np.random.default_rng(0).integers(3, spec.vocab_size, size=(4, T - 1))
    ref = orc.decode_logits(ids, mask, dec)
    got = model.decode_logits(ids, mask, dec).cpu().numpy()
    err = np.abs(got - ref)
    print(f"mask holes: logits max err {err.max():.4f} mean {err.mean():.5f}")
    assert err.max() <= LOGIT_ATOL and err.mean() <= LOGIT_MEAN


def test_no_attention_mask_equals_all_ones(models):
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(3, 12, SPECS["tiny"].vocab_size, seed=8, lengths="full")
    a = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=6)
    b = model.generate(input_ids=torch.from_numpy(ids), max_new_tokens=6)
    assert torch.equal(a, b)


def test_missing_attention_mask_is_inferred_from_pad_tokens_like_hf(models):
    """generate() without attention_mask: transformers masks the pad positions when the pad token occurs in the
    inputs and differs from EOS (GenerationMixin._prepare_attention_mask_for_generation). The predictor mirror and the
    reference predictor both allow mask-less input (feature_columns=["input_ids"])."""
    model, _ = models("tiny", 1)
    g = np.load(GOLD / "tiny_a.npz")
    ids, mask = g["ids"], g["mask"]
    assert (ids[mask == 0] == 0).all() and (mask == 0).any(), "the golden case is right-padded with pad id 0"
    T = CASES["tiny_a"][2]
    with_mask = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T)
    inferred = model.generate(input_ids=torch.from_numpy(ids), max_new_tokens=T)
    assert torch.equal(with_mask, inferred)
    host, _ = model.generate_host(ids, None, max_new_tokens=T)
    assert (host == with_mask.cpu().numpy()).all()
    gated, _ = gated_prefix_match(inferred.cpu().numpy(), g["tokens_bf16"],
                                  oracle_for("tiny", 1).generate(ids, mask, max_new_tokens=T, return_margins=True)[1])
    assert gated == 1.0
    # pad == eos: nothing can be inferred, every position is attended (HF's rule)
    all_ones = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.ones_like(torch.from_numpy(ids)),
                              max_new_tokens=T, pad_token_id=1)
    same_tok = model.generate(input_ids=torch.from_numpy(ids), max_new_tokens=T, pad_token_id=1)
    assert torch.equal(all_ones, same_tok)


def test_cross_attention_kernels_give_identical_tokens(models):
    """1, 2 and 3 row-chains and the knobs of the stream cross-attention kernel produce the same tokens (rows are independent
    in every kernel, the ring depth and the PDL trigger do not touch the arithmetic); the two cross-attention kernels
    differ only in the order of their fp32 accumulations, so they agree row for row up to the first near-tie step."""
    model, _ = models("mini", 2)
    spec = SPECS["mini"]
    ids, mask = synthetic_token_batch(150, 64, spec.vocab_size, seed=12, lengths="uniform")
    kw = dict(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=12)
    model.set_option("xattn", 0)
    base = model.generate(**kw).cpu()
    otoks, margins = oracle_for("mini", 2).generate(ids, mask, max_new_tokens=12, return_margins=True)
    try:
        for name, value in (("chains", 1), ("chains", 3), ("chains", 0)):
            model.set_option(name, value)
            assert torch.equal(model.generate(**kw).cpu(), base), (name, value)
        model.set_option("xattn", 1)
        stream = model.generate(**kw).cpu()
        gated, full = gated_prefix_match(stream.numpy(), otoks, margins)
        gated_b, _ = gated_prefix_match(stream.numpy(), base.numpy(), margins)
        print(f"stream kernel: vs oracle gated={gated:.2f} full={full:.2f}; vs per-thread-load kernel gated={gated_b:.2f} equal rows={gated_prefix_match(stream.numpy(), base.numpy(), margins)[1]:.2f}")
        assert gated == 1.0 and gated_b == 1.0
        for name, value in (("chains", 1), ("chains", 3), ("xattn_stages", 2), ("xattn_late_pdl", 0), ("xattn_serialize", 1), ("xattn_l2pf", 1)):
            model.set_option(name, value)
            assert torch.equal(model.generate(**kw).cpu(), stream), (name, value)
        model.set_option("xattn_l2pf", 0)
    finally:
        for name, value in (("xattn", 2), ("chains", 0), ("xattn_stages", 5), ("xattn_late_pdl", 1), ("xattn_serialize", 0)):
            model.set_option(name, value)


def test_cross_attention_kernel_is_chosen_from_the_prompt_fill(models):
    """Default ("xattn" = 2): the TMA stream kernel when the prompts fill the window (valid tokens / B*S >= 0.9), the
    per-thread-load kernel on ragged batches; 0 / 1 pin one of them. b200t5_get_stats reports what the last call ran."""
    model, _ = models("mini", 2)
    spec = SPECS["mini"]
    full = synthetic_token_batch(16, 64, spec.vocab_size, seed=5, lengths="full")
    ragged = synthetic_token_batch(16, 64, spec.vocab_size, seed=5, lengths="uniform")

    def kernel(batch):
        model.generate(input_ids=torch.from_numpy(batch[0]), attention_mask=torch.from_numpy(batch[1]), max_new_tokens=4)
        return model.stats()["xattn_kernel"]

    try:
        model.set_option("xattn", 2)
        assert kernel(full) == 1 and kernel(ragged) == 0 and kernel(full) == 1
        model.set_option("xattn", 0)
        assert kernel(full) == 0
        model.set_option("xattn", 1)
        assert kernel(ragged) == 1
    finally:
        model.set_option("xattn", 2)


def test_determinism_and_batch_invariance(models):
    """Same inputs -> identical tokens; a row's result does not depend on its batch neighbours
    (each (b,h) problem is independent and tile shapes do not change the per-row arithmetic)."""
    spec = SPECS["mini"]
    model, _ = models("mini", 2)
    ids, mask = synthetic_token_batch(6, 33, spec.vocab_size, seed=9, lengths="uniform")
    a = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=10, min_new_tokens=10).cpu()
    b = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=10, min_new_tokens=10).cpu()
    assert torch.equal(a, b)
    solo = model.generate(input_ids=torch.from_numpy(ids[2:3]), attention_mask=torch.from_numpy(mask[2:3]), max_new_tokens=10, min_new_tokens=10).cpu()
    assert torch.equal(a[2:3], solo)


def test_flan_t5_small_vs_hf_gpu(models):
    """Real FLAN-T5-small architecture; anchor = HF eager bf16 on this same GPU."""
    pytest.importorskip("transformers")
    from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits, load_hf_model

    spec = SPECS["flan-t5-small"]
    model, ckpt = models("flan-t5-small", 3)
    B, S, T = 16, 96, 24
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths="uniform")
    hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
    ref = hf_generate(hf, ids, mask, T, min_new_tokens=T)
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T, min_new_tokens=T).cpu().numpy()
    assert out.shape == ref.shape
    # margins from HF's own teacher-forced bf16 logits along HF's path
    lg = hf_teacher_forced_logits(hf, ids, mask, ref[:, :-1])
    lg[:, :, spec.eos_token_id] = -np.inf
    top2 = np.partition(lg, -2, axis=-1)[:, :, -2:]
    margins = top2[:, :, 1] - top2[:, :, 0]
    gated, full = gated_prefix_match(out, ref, margins)
    tok_rate = (out == ref).mean()
    print(f"flan-t5-small vs HF-bf16-GPU: gated rows={gated:.2f} ungated rows={full:.2f} token agreement={tok_rate:.3f}")
    ours_lg = model.decode_logits(ids, mask, ref[:, :-1]).cpu().numpy()
    gpu_lg = hf_teacher_forced_logits(hf, ids, mask, ref[:, :-1])
    cpu_lg = hf_teacher_forced_logits(load_hf_model(ckpt, dtype=torch.bfloat16, device="cpu"), ids, mask, ref[:, :-1])
    err = np.abs(ours_lg - gpu_lg)
    floor = np.abs(gpu_lg - cpu_lg)
    print(f"flan-t5-small teacher-forced logits: ours vs HF-bf16-GPU max {err.max():.4f} mean {err.mean():.5f} | "
          f"noise floor HF-bf16-GPU vs HF-bf16-CPU max {floor.max():.4f} mean {floor.mean():.5f}")
    assert gated == 1.0
    # the CUDA path must track the same-dtype GPU anchor as closely as two stock bf16 runs of the dependency (GPU vs
    # CPU) track each other (on the chaotic q_init_gain = 4 checkpoints of round 1 it was twice as close; on the
    # well-conditioned ones all three sit at the same rounding-noise level)
    assert err.mean() <= 1.15 * floor.mean() and err.max() <= 1.6 * floor.max()


def test_batch_predictor_api_single_gpu(models):
    """Notebook flow (:875-934) on the GPU through the shim: from_checkpoint -> predict -> to_pandas."""
    from anyscale_workshop_nyc_2023_b200 import rayshim
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir, make_batch_predictor

    spec = SPECS["tiny"]
    ckpt = checkpoint_dir("tiny", seed=1)
    ids, mask = synthetic_token_batch(10, 24, spec.vocab_size, seed=31, lengths="uniform")
    ds = rayshim.data.from_numpy({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()})
    bp = make_batch_predictor(ckpt, device_map="auto", torch_dtype=torch.bfloat16)
    out = bp.predict(ds, batch_size=4, num_gpus_per_worker=1, max_scoring_workers=1, max_new_tokens=8).to_pandas()
    assert len(out) == 10 and list(out.columns) == ["generated_output"]
    model, _ = models("tiny", 1)
    from transformers import T5Tokenizer

    tok = T5Tokenizer.from_pretrained(str(ckpt))
    want = []
    for lo in range(0, 10, 4):
        g = model.generate(input_ids=torch.from_numpy(ids[lo:lo + 4]), attention_mask=torch.from_numpy(mask[lo:lo + 4]), max_new_tokens=8)
        want += tok.batch_decode(g, skip_special_tokens=True)
    assert out["generated_output"].tolist() == want


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_batch_predictor_pool_two_gpus():
    """One scoring process per GPU, blocks dealt round-robin, results back in input order."""
    from anyscale_workshop_nyc_2023_b200 import rayshim
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir, make_batch_predictor

    spec = SPECS["tiny"]
    ckpt = checkpoint_dir("tiny", seed=1)
    ids, mask = synthetic_token_batch(24, 24, spec.vocab_size, seed=32, lengths="uniform")
    ds = rayshim.data.from_numpy({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()})
    bp = make_batch_predictor(ckpt, device_map="auto", torch_dtype=torch.bfloat16)
    one = bp.predict(ds, batch_size=4, num_gpus_per_worker=1, max_scoring_workers=1, max_new_tokens=8).to_pandas()
    two = bp.predict(ds, batch_size=4, num_gpus_per_worker=1, max_new_tokens=8).to_pandas()
    assert one["generated_output"].tolist() == two["generated_output"].tolist()


def _static_rows(model, ids, mask, pool, **kw):
    """Per-prompt tokens of the static path in `pool`-row batches (the last batch is filled up with copies of its
    first row, so every batch runs the same kernels as the slot pool does)."""
    N = ids.shape[0]
    T = kw["max_new_tokens"]
    out = np.zeros((N, T + 1), dtype=np.int64)
    lens = np.zeros(N, dtype=np.int32)
    for lo in range(0, N, pool):
        hi = min(lo + pool, N)
        bi, bm = ids[lo:hi], mask[lo:hi]
        if hi - lo < pool:
            fill = pool - (hi - lo)
            bi = np.concatenate([bi, np.repeat(bi[:1], fill, 0)])
            bm = np.concatenate([bm, np.repeat(bm[:1], fill, 0)])
        o, ln = model.generate_host(bi, bm, **kw)
        out[lo:hi, : o.shape[1]] = o[: hi - lo]
        lens[lo:hi] = ln[: hi - lo]
    return out, lens


@pytest.mark.parametrize("spec_name,seed,N,S,pool,T,admit", [
    ("tiny", 1, 150, 24, 32, 20, 0),     # several refill rounds, natural EOS
    ("mini", 2, 300, 40, 128, 16, 1),    # two row-chains, refill as soon as one slot is free
    ("tiny", 1, 20, 16, 64, 12, 0),      # fewer prompts than slots
])
def test_slot_pool_equals_static_batches(models, spec_name, seed, N, S, pool, T, admit):
    """Continuous batching (b200t5_generate_stream) is a scheduling change only: rows are independent in every
    kernel, so each prompt's tokens and length are bit-identical to the static path's."""
    spec = SPECS[spec_name]
    model, _ = models(spec_name, seed)
    ids, mask = synthetic_token_batch(N, S, spec.vocab_size, seed=21, lengths="uniform")
    kw = dict(max_new_tokens=T)
    ref, ref_len = _static_rows(model, ids, mask, min(pool, N), **kw)
    out, lens = model.generate_stream(ids, mask, pool=pool, admit_min=admit, **kw)
    assert len(set(ref_len.tolist())) > 3, "the workload should have varied natural lengths"
    assert (lens == ref_len).all()
    w = out.shape[1]
    assert w == int(ref_len.max()) + 1
    assert (out == ref[:, :w]).all() and (ref[:, w:] == 0).all()
    # and again: the pool state of a previous call must not leak into the next one
    out2, lens2 = model.generate_stream(ids[::-1].copy(), mask[::-1].copy(), pool=pool, admit_min=admit, **kw)
    assert (out2[::-1] == out).all() and (lens2[::-1] == lens).all()


def test_slot_pool_forced_length_and_generate_dispatch(models):
    """min_new_tokens == max_new_tokens: every slot runs to max_new and is then refilled; generate() itself
    switches to the slot pool for batches larger than model.pool_size; the static path still works afterwards
    (the step graph is re-captured when the mode changes)."""
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(70, 20, spec.vocab_size, seed=22, lengths="uniform")
    kw = dict(max_new_tokens=9, min_new_tokens=9)
    ref, ref_len = _static_rows(model, ids, mask, 16, **kw)
    assert (ref_len == 9).all()
    old = model.pool_size, model.pool_slots
    try:
        model.pool_size, model.pool_slots = 16, 16
        out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw).cpu().numpy()
        model.pool_slots = 64  # more slots than the static batches have rows: still the same tokens
        out64 = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw).cpu().numpy()
        assert (out64 == out).all()
    finally:
        model.pool_size, model.pool_slots = old
    assert out.shape == (70, 10) and (out == ref).all()
    again, _ = model.generate_host(ids[:16], mask[:16], **kw)
    assert (again == ref[:16]).all()


def test_finished_rows_are_retired_in_static_batches(models):
    """A row that has emitted EOS keeps producing pad tokens and stops reading its cross-KV (live extent 0):
    results equal the oracle-checked goldens' format (pads after EOS) and a solo run of each row."""
    spec = SPECS["tiny"]
    model, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(12, 24, spec.vocab_size, seed=23, lengths="uniform")
    out, lens = model.generate_host(ids, mask, max_new_tokens=24)
    assert lens.min() < lens.max()
    for b in (int(np.argmin(lens)), int(np.argmax(lens))):
        solo, sl = model.generate_host(ids[b:b + 1], mask[b:b + 1], max_new_tokens=24)
        assert int(sl[0]) == int(lens[b])
        assert (out[b, : solo.shape[1]] == solo[0]).all() and (out[b, solo.shape[1]:] == 0).all()


# ------------------------------------------------------------------------------------------------
# Parity AT THE BENCHED CONFIGURATIONS (BASELINE configs[1] / configs[3]): FLAN-T5-base, batch 256, 512-token prompts,
# 128 new tokens - the shapes bench.py times (128 x 256 encoder GEMM tiles at M = 131 072, the packed encoder attention, two
# 128-row decode chains, eight steps per graph launch, self-attention up to t = 127, 12-layer error accumulation).
# Anchor: transformers' own eager model in the same dtype ON THIS GPU, for a subset of rows (rows are independent of
# their batch neighbours, test_determinism_and_batch_invariance), reference call
# NLP_workloads/Anyscale_job/flan-t5-batch-inference.py:119-134.
def _headline_parity(model, ckpt, spec, dtype, B, S, T, lengths, rows, tau, tag):
    from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits, load_hf_model

    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=4242, lengths=lengths)
    sub = np.linspace(0, B - 1, rows).round().astype(int)  # rows of every chain
    hf = load_hf_model(ckpt, dtype=dtype, device="cuda")
    stats = {"tag": tag}
    for mode in ("forced", "natural"):
        kw = dict(max_new_tokens=T, **({"min_new_tokens": T} if mode == "forced" else {}))
        ours = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw).cpu().numpy()
        ref = hf_generate(hf, ids[sub], mask[sub], T, min_new_tokens=T if mode == "forced" else 0)
        # HF's own logits along HF's path -> margins; ours along the same path -> error and teacher-forced arg-max
        dec_in = pad_to(ref, T + 1)[:, :-1]
        hf_lg = hf_teacher_forced_logits(hf, ids[sub], mask[sub], dec_in)
        our_lg = model.decode_logits(ids[sub], mask[sub], dec_in).cpu().numpy()
        if mode == "forced":
            hf_lg[:, :, spec.eos_token_id] = -np.inf
            our_lg[:, :, spec.eos_token_id] = -np.inf
        live = np.ones(dec_in.shape, bool)
        for r in range(len(sub)):  # positions after a row's EOS are pad-fed in both: not part of the comparison
            e = np.where(ref[r, 1:] == spec.eos_token_id)[0]
            if len(e):
                live[r, e[0] + 1:] = False
        top2 = np.partition(hf_lg, -2, axis=-1)[:, :, -2:]
        margins = top2[:, :, 1] - top2[:, :, 0]
        agree = our_lg.argmax(-1) == hf_lg.argmax(-1)
        fin = np.isfinite(hf_lg) & np.isfinite(our_lg)
        err = np.abs(np.where(fin, our_lg - hf_lg, 0.0))
        safe = live & (margins > tau)
        gated_rows, full_rows = gated_prefix_match(ours[sub], ref, np.where(live, margins, np.nan), tau=tau)
        stats[mode] = {
            "tf_argmax_agreement": float(agree[live].mean()), "tf_argmax_agreement_gated": float(agree[safe].mean()),
            "gated_positions": int(safe.sum()), "positions": int(live.sum()),
            "free_running_rows_gated": gated_rows, "free_running_rows_ungated": full_rows,
            "free_running_token_agreement": float((pad_to(ours[sub], T + 1) == pad_to(ref, T + 1)).mean()),
            "logit_err_mean": float(err[live].mean()), "logit_err_max": float(err[live].max()),
            "logit_scale": float(np.abs(np.where(fin, hf_lg, 0.0)).max()),
            "lengths_ours": [int(x) for x in model.last_lengths.cpu().numpy()[sub][:8]],
        }
        if mode == "forced":
            assert ours.shape == (B, T + 1) and (ours[:, 1:] != spec.eos_token_id).all()
            cpu = load_hf_model(ckpt, dtype=dtype, device="cpu")
            k = min(8, len(sub))
            cpu_lg = hf_teacher_forced_logits(cpu, ids[sub[:k]], mask[sub[:k]], dec_in[:k])
            cpu_lg[:, :, spec.eos_token_id] = -np.inf
            floor = np.abs(np.where(np.isfinite(cpu_lg) & np.isfinite(hf_lg[:k]), cpu_lg - hf_lg[:k], 0.0))
            stats["floor_hf_gpu_vs_hf_cpu"] = {"logit_err_mean": float(floor.mean()), "logit_err_max": float(floor.max()),
                                               "tf_argmax_agreement": float((cpu_lg.argmax(-1) == hf_lg[:k].argmax(-1)).mean())}
            del cpu
    del hf
    torch.cuda.empty_cache()
    print("HEADLINE_PARITY " + json.dumps(stats))
    out_dir = Path(__file__).resolve().parents[1] / "gpurun_out"
    if out_dir.is_dir():
        with open(out_dir / "parity_headline.jsonl", "a") as f:
            f.write(json.dumps(stats) + "\n")
    return stats


# Floors asserted below: the UNGATED teacher-forced arg-max agreement with HF on the same GPU, i.e. how often two bf16
# implementations of the same 12-layer forward pick the same token when nothing is excluded.
UNGATED_FLOOR = {"bf16": 0.92, "fp16": 0.99}


@pytest.mark.timeout(600, method="thread")
@pytest.mark.parametrize("dtype_name,lengths", [("bf16", "full"), ("bf16", "alpaca"), ("fp16", "full")])
def test_headline_config_flan_t5_base_b256_s512_t128(models, models_fp16, dtype_name, lengths):
    pytest.importorskip("transformers")
    spec = SPECS["flan-t5-base"]
    if dtype_name == "bf16":
        model, ckpt = models("flan-t5-base", 0)
        dtype, tau = torch.bfloat16, TAU
    else:
        model = models_fp16("flan-t5-base", 0)
        ckpt = models("flan-t5-base", 0)[1]
        dtype, tau = torch.float16, TAU_FP16
    st = _headline_parity(model, ckpt, spec, dtype, 256, 512, 128, lengths, rows=24, tau=tau, tag=f"base-{dtype_name}-{lengths}")
    fl = st["floor_hf_gpu_vs_hf_cpu"]
    for mode in ("forced", "natural"):
        m = st[mode]
        assert m["tf_argmax_agreement_gated"] == 1.0, (mode, m)          # exact wherever the decision is not a near-tie
        assert m["free_running_rows_gated"] == 1.0, (mode, m)
        assert m["tf_argmax_agreement"] >= UNGATED_FLOOR[dtype_name], (mode, m)  # and nothing hides behind the gate
        # the CUDA path tracks the same-dtype GPU anchor as closely as two stock runs of the dependency (GPU vs CPU)
        # track each other: all three carry the same rounding noise (measured: ours 0.0149 / 0.0131 / 0.0011 mean
        # |dlogit| against floors of 0.0151 / 0.0158 / 0.0011)
        assert m["logit_err_mean"] <= 1.15 * fl["logit_err_mean"] and m["logit_err_max"] <= 1.6 * fl["logit_err_max"], (mode, m, fl)
        assert m["tf_argmax_agreement"] >= fl["tf_argmax_agreement"] - 0.02, (mode, m, fl)


def test_run_to_run_determinism_at_the_benched_shape(models):
    """Two row-chains, eight steps per graph launch, PDL-chained kernels on two streams: the same call must return
    the same tokens every time, forced length and natural EOS (retired rows), and the slot pool must equal the static
    batches row for row at this size too (tools/diag_determinism.py is the long form of this test)."""
    model, _ = models("flan-t5-base", 0)
    spec = SPECS["flan-t5-base"]
    ids, mask = synthetic_token_batch(512, 512, spec.vocab_size, seed=3, lengths="full")
    forced = [model.generate_host(ids[:256], mask[:256], max_new_tokens=32, min_new_tokens=32)[0] for _ in range(3)]
    assert all((forced[0] == f).all() for f in forced[1:])
    nat = []
    for _ in range(2):
        o, ln = model.generate_host(ids[:256], mask[:256], max_new_tokens=128)
        nat.append((pad_to(o, 129), ln))
    assert (nat[0][0] == nat[1][0]).all() and (nat[0][1] == nat[1][1]).all()
    assert len(set(nat[0][1].tolist())) > 5, "natural lengths should vary"
    pool, plen = model.generate_stream(ids, mask, pool=256, max_new_tokens=128)
    assert (pad_to(pool, 129)[:256] == nat[0][0]).all() and (plen[:256] == nat[0][1]).all()


@pytest.mark.timeout(900, method="thread")
def test_headline_config_flan_t5_large_b64(models):
    """BASELINE configs[3]'s model at a batch HF can anchor in seconds: 24 layers, d_model 1024, 16 heads."""
    pytest.importorskip("transformers")
    spec = SPECS["flan-t5-large"]
    model, ckpt = models("flan-t5-large", 0)
    st = _headline_parity(model, ckpt, spec, torch.bfloat16, 64, 512, 128, "full", rows=12, tau=TAU, tag="large-bf16-full")
    fl = st["floor_hf_gpu_vs_hf_cpu"]
    for mode in ("forced", "natural"):
        m = st[mode]
        assert m["tf_argmax_agreement_gated"] == 1.0 and m["free_running_rows_gated"] == 1.0, (mode, m)
        assert m["tf_argmax_agreement"] >= UNGATED_FLOOR["bf16"], (mode, m)
        assert m["logit_err_mean"] <= 1.15 * fl["logit_err_mean"], (mode, m, fl)


# ------------------------------------------------------------------------------------------------
# fp16 contract (libb200t5_f16.so): the notebook's literal torch_dtype=torch.float16 (NB:882) with transformers'
# fp32 `wo` and fp32 residual stream. Anchors: HF fp16 goldens (tests/golden/*_fp16.npz) and the oracle's fp16
# mode, which the CPU suite pins to those goldens. fp16 has 3 more mantissa bits than bf16, so the logit
# tolerances are tighter than the bf16 ones (ulp 0.0039-0.0078 at |logit| in [4, 16)).
TAU_FP16 = 0.03
LOGIT_ATOL_FP16 = 0.08
LOGIT_MEAN_FP16 = 0.008


@pytest.fixture(scope="module")
def models_fp16(tmp_path_factory):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration

    cache = {}

    def get(spec_name, seed):
        key = (spec_name, seed)
        if key not in cache:
            d = tmp_path_factory.mktemp(f"ckpt16_{spec_name}_{seed}")
            save_checkpoint(d, SPECS[spec_name], seed=seed)
            cache[key] = B200T5ForConditionalGeneration.from_pretrained(d, device_map="auto", torch_dtype=torch.float16)
        return cache[key]

    return get


def oracle_fp16(spec_name, seed):
    from oracle.t5_oracle import T5Oracle

    return T5Oracle(make_state_dict(SPECS[spec_name], seed), SPECS[spec_name], emulate="fp16")


@pytest.mark.parametrize("case", list(CASES))
def test_fp16_golden_generate(models_fp16, case):
    spec_name, seed, T = CASES[case]
    g = np.load(GOLD / f"{case}_fp16.npz")
    model = models_fp16(spec_name, seed)
    assert model.dtype == torch.float16
    out = model.generate(input_ids=torch.from_numpy(g["ids"]), attention_mask=torch.from_numpy(g["mask"]),
                         labels=torch.from_numpy(g["ids"]), max_new_tokens=T).cpu().numpy()
    orc = oracle_fp16(spec_name, seed)
    otoks, margins = orc.generate(g["ids"], g["mask"], max_new_tokens=T, return_margins=True)
    gated_o, full_o = gated_prefix_match(out, otoks, margins, tau=TAU_FP16)
    gated_h, full_h = gated_prefix_match(out, g["tokens_fp16"], margins, tau=TAU_FP16)
    print(f"{case} fp16: vs oracle gated={gated_o:.2f} full={full_o:.2f} | vs HF-fp16 golden gated={gated_h:.2f} full={full_h:.2f}")
    assert gated_o == 1.0 and gated_h == 1.0
    forced = model.generate(input_ids=torch.from_numpy(g["ids"]), attention_mask=torch.from_numpy(g["mask"]),
                            max_new_tokens=T, min_new_tokens=T).cpu().numpy()
    assert forced.shape == (g["ids"].shape[0], T + 1)
    ftoks, fm = orc.generate(g["ids"], g["mask"], max_new_tokens=T, min_new_tokens=T, return_margins=True)
    gated_f, full_f = gated_prefix_match(forced, ftoks, fm, tau=TAU_FP16)
    gated_fh, full_fh = gated_prefix_match(forced, g["forced_fp16"], fm, tau=TAU_FP16)
    print(f"{case} fp16 forced: vs oracle gated={gated_f:.2f} full={full_f:.2f} | vs golden gated={gated_fh:.2f} full={full_fh:.2f}")
    assert gated_f == 1.0 and gated_fh == 1.0


@pytest.mark.parametrize("case", list(CASES))
def test_fp16_golden_logits_and_encoder(models_fp16, case):
    spec_name, seed, T = CASES[case]
    g = np.load(GOLD / f"{case}_fp16.npz")
    model = models_fp16(spec_name, seed)
    valid = g["mask"].astype(bool)
    enc_t = model.encode(g["ids"], g["mask"])
    assert enc_t.dtype == torch.float16
    enc = enc_t.float().cpu().numpy()
    e_err = np.abs(enc - g["enc_fp16"])[valid]
    print(f"{case} fp16: encoder max err {e_err.max():.4f} mean {e_err.mean():.5f} (scale {np.abs(g['enc_fp16'])[valid].max():.2f})")
    assert e_err.max() <= 0.03 and e_err.mean() <= 0.002
    dec_in = g["tokens_fp16"][:, :-1]
    logits = model.decode_logits(g["ids"], g["mask"], dec_in).cpu().numpy()
    err = np.abs(logits - g["logits_fp16"])
    print(f"{case} fp16: logits max err {err.max():.4f} mean {err.mean():.5f} (scale {np.abs(g['logits_fp16']).max():.2f})")
    assert err.max() <= LOGIT_ATOL_FP16 and err.mean() <= LOGIT_MEAN_FP16
    assert (logits == logits.astype(np.float16).astype(np.float32)).all()  # fp16-rounded outputs


def test_fp16_and_bf16_models_coexist_and_pool(models, models_fp16):
    """Both libraries loaded in one process (separate handles); the slot pool in the fp16 build equals its static
    batches bit for bit, like the bf16 one."""
    spec = SPECS["tiny"]
    m16 = models_fp16("tiny", 1)
    mb, _ = models("tiny", 1)
    ids, mask = synthetic_token_batch(40, 20, spec.vocab_size, seed=31, lengths="uniform")
    kw = dict(max_new_tokens=12)
    ref, ref_len = _static_rows(m16, ids, mask, 16, **kw)
    out, lens = m16.generate_stream(ids, mask, pool=16, **kw)
    assert (lens == ref_len).all() and (out == ref[:, : out.shape[1]]).all()
    ob, _ = mb.generate_host(ids[:16], mask[:16], **kw)
    o16, _ = m16.generate_host(ids[:16], mask[:16], **kw)
    assert ob.shape[0] == o16.shape[0] == 16  # different contracts, both alive; tokens may legitimately differ


def test_fp16_flan_t5_small_vs_hf_gpu(models_fp16, tmp_path):
    """Real FLAN-T5-small architecture in the notebook's literal dtype; anchor = HF eager fp16 (fp32 `wo`) on this GPU.
    HF's fp32 `wo` Linear runs through cuBLAS fp32 there; ours through two tf32 passes over W_hi + W_lo."""
    pytest.importorskip("transformers")
    from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits, load_hf_model

    spec = SPECS["flan-t5-small"]
    model = models_fp16("flan-t5-small", 3)
    ckpt = tmp_path / "ckpt"
    save_checkpoint(ckpt, spec, seed=3)
    B, S, T = 16, 96, 24
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths="uniform")
    hf = load_hf_model(ckpt, dtype=torch.float16, device="cuda")
    assert hf.encoder.block[0].layer[1].DenseReluDense.wo.weight.dtype == torch.float32
    ref = hf_generate(hf, ids, mask, T, min_new_tokens=T)
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T, min_new_tokens=T).cpu().numpy()
    assert out.shape == ref.shape
    lg = hf_teacher_forced_logits(hf, ids, mask, ref[:, :-1])
    lg[:, :, spec.eos_token_id] = -np.inf
    top2 = np.partition(lg, -2, axis=-1)[:, :, -2:]
    margins = top2[:, :, 1] - top2[:, :, 0]
    gated, full = gated_prefix_match(out, ref, margins, tau=TAU_FP16)
    print(f"flan-t5-small fp16 vs HF-fp16-GPU: gated rows={gated:.2f} ungated rows={full:.2f} token agreement={(out == ref).mean():.3f}")
    ours_lg = model.decode_logits(ids, mask, ref[:, :-1]).cpu().numpy()
    gpu_lg = hf_teacher_forced_logits(hf, ids, mask, ref[:, :-1])
    cpu_lg = hf_teacher_forced_logits(load_hf_model(ckpt, dtype=torch.float16, device="cpu"), ids, mask, ref[:, :-1])
    err = np.abs(ours_lg - gpu_lg)
    floor = np.abs(gpu_lg - cpu_lg)
    print(f"flan-t5-small fp16 teacher-forced logits: ours vs HF-fp16-GPU max {err.max():.4f} mean {err.mean():.5f} | "
          f"noise floor HF-fp16-GPU vs HF-fp16-CPU max {floor.max():.4f} mean {floor.mean():.5f}")
    assert gated == 1.0
    assert err.mean() <= 1.15 * floor.mean() and err.max() <= 2.0 * floor.max()


def test_fp16_mask_holes_and_edge_shapes_vs_oracle(models_fp16):
    """fp16 build: a non-prefix mask (HF adds finfo(fp16).min, which can overflow to -inf; the kernels replace the
    score - both give probability 0 after the fp32 softmax), ragged lengths and a 1-token prompt against the oracle's
    fp16 mode. (A fully masked row is NaN in HF fp16 and is not part of the contract.)"""
    spec = SPECS["tiny"]
    model = models_fp16("tiny", 1)
    orc = oracle_fp16("tiny", 1)
    ids, mask = synthetic_token_batch(4, 20, spec.vocab_size, seed=77, lengths="full")
    mask[1, 3:7] = 0
    mask[3, 9:] = 0
    T = 6
    dec = np.zeros((4, T), dtype=np.int64)
    dec[:, 1:] = np.random.default_rng(0).integers(3, spec.vocab_size, size=(4, T - 1))
    ref = orc.decode_logits(ids, mask, dec)
    got = model.decode_logits(ids, mask, dec).cpu().numpy()
    err = np.abs(got - ref)
    print(f"fp16 mask holes: logits max err {err.max():.4f} mean {err.mean():.5f}")
    assert np.isfinite(got).all() and err.max() <= LOGIT_ATOL_FP16 and err.mean() <= LOGIT_MEAN_FP16
    for B, S, lengths in [(1, 1, "full"), (9, 130, "uniform")]:
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=5 + B, lengths=lengths)
        out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=8).cpu().numpy()
        otoks, margins = orc.generate(ids, mask, max_new_tokens=8, return_margins=True)
        gated, _ = gated_prefix_match(out, otoks, margins, tau=TAU_FP16)
        assert gated == 1.0, (B, S)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_long_prompts_beyond_the_packed_encoder(models, models_fp16, dtype):
    """S = 640 > 512: the encoder runs on unpacked rows (rows are packed for prompts up to 512 tokens); the slot pool,
    which needs the packed encoder, refuses such prompts loudly."""
    spec = SPECS["tiny"]
    model = models("tiny", 1)[0] if dtype == "bf16" else models_fp16("tiny", 1)
    orc = oracle_for("tiny", 1) if dtype == "bf16" else oracle_fp16("tiny", 1)
    tau = TAU if dtype == "bf16" else TAU_FP16
    ids, mask = synthetic_token_batch(3, 640, spec.vocab_size, seed=41, lengths="uniform", min_len=520)
    out = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=8).cpu().numpy()
    otoks, margins = orc.generate(ids, mask, max_new_tokens=8, return_margins=True)
    gated, full = gated_prefix_match(out, otoks, margins, tau=tau)
    print(f"S=640 {dtype}: gated={gated:.2f} full={full:.2f}")
    assert gated == 1.0
    from anyscale_workshop_nyc_2023_b200._lib import B200T5Error

    with pytest.raises(B200T5Error, match="packed encoder"):
        model.generate_stream(np.repeat(ids, 4, 0), np.repeat(mask, 4, 0), pool=4, max_new_tokens=4)
    # the handle is still usable afterwards
    again = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=8).cpu().numpy()
    assert (again == out).all()


def test_library_counters_equal_the_python_roofline_model(models, models_fp16):
    """b200t5_get_stats' decode_algo_bytes / encoder_flops (what bench.py divides by its CUDA-event times) are the
    SURVEY 8(d) model: the Python restatement (roofline.py, pinned to SURVEY's table on CPU) gives the same numbers
    for ragged prompts, in both builds."""
    from anyscale_workshop_nyc_2023_b200 import roofline

    spec = SPECS["mini"]
    ids, mask = synthetic_token_batch(7, 48, spec.vocab_size, seed=51, lengths="uniform")
    ext = mask.sum(axis=1).tolist()
    for model, fp32_wo in ((models("mini", 2)[0], False), (models_fp16("mini", 2), True)):
        model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=9, min_new_tokens=9)
        st = model.stats()
        assert int(st["decode_steps"]) == 9
        assert st["decode_algo_bytes"] == pytest.approx(roofline.decode_bytes(spec, 7, 9, extents=ext, fp32_wo=fp32_wo), rel=1e-9)
        assert st["encoder_flops"] == pytest.approx(roofline.encoder_flops(spec, 7, extents=ext), rel=1e-9)
        ca = model.bench_cross_attention(reps=1)
        assert ca["bytes_per_launch"] == pytest.approx(roofline.cross_attention_bytes_per_launch(spec, ext), rel=1e-9)
