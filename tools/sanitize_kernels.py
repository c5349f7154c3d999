"""Reduced-shape pass over every hand-written kernel family, meant to run under compute-sanitizer
(memcheck / racecheck / synccheck; SURVEY section 5): the mbarrier / DSMEM reduce-scatter / cluster-barrier /
PDL / bulk-copy-ring protocols at shapes small enough for the tools' 10-100x slowdown.

    compute-sanitizer --tool memcheck  python tools/sanitize_kernels.py
    compute-sanitizer --tool racecheck python tools/sanitize_kernels.py
    compute-sanitizer --tool synccheck python tools/sanitize_kernels.py

Each section also checks its result loosely, so a run doubles as a smoke test of the hooks."""
import ctypes as C
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200 import _lib  # noqa: E402
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

DEV = 0


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def rnd(*shape, scale=0.5, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def close(a, b, tol=0.05):
    err = (a.float() - b.float()).abs().max().item()
    assert err <= tol * (1 + b.float().abs().max().item()), err


def main():
    only = set(sys.argv[1:])
    lib = _lib.load()

    def section(name):
        on = not only or name in only
        if on:
            print("==", name, flush=True)
        return on

    if section("gemm"):
        for M, N, K in ((130, 264, 128), (300, 520, 128)):  # the encoder configuration (bn 512)
            A, W = rnd(M, K), rnd(N, K)
            out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
            _lib.check(lib.b200t5_test_gemm(DEV, P(A), P(W), P(out), M, N, K, 512, 0, 0, None))
            torch.cuda.synchronize()
            close(out, A.float() @ W.float().T)
    if section("enc_gemm"):
        # both 128 x 256 encoder kernels, every encoder epilogue; 18 x 8-9 tiles exceed the SM count, so some CTAs take
        # a second tile and the staging-buffer handshake turns over
        M, K, H, Bx, Sx = 2200, 64, 2, 4, 550
        A = rnd(M, K)
        for mode, N in ((0, 2056), (1, 2048), (2, 2048), (3, 2048)):
            W = rnd(N, K, seed=mode)
            outs = []
            for kernel in (0, 1):
                if mode == 3:
                    out = torch.zeros(N // (H * 64), Bx, H, Sx, 64, device="cuda", dtype=torch.bfloat16)
                else:
                    out = rnd(M, N // 2 if mode == 2 else N, seed=7)
                _lib.check(lib.b200t5_test_enc_gemm(DEV, P(A), P(W), P(out), M, N, K, kernel, mode, 0, None, None, Bx, H, Sx, None))
                torch.cuda.synchronize()
                outs.append(out)
            assert torch.equal(outs[0], outs[1])
    if section("splitk"):
        for bn, split, mode, (M, N, K) in ((64, 4, 0, (130, 192, 256)), (64, 2, 1, (37, 128, 128)), (128, 2, 0, (130, 264, 128)),
                                           (64, 8, 1, (256, 64, 512)), (64, 1, 0, (16, 64, 64)), (64, 2, 0, (8, 192, 64)),
                                           (64, 4, 0, (40, 96, 128))):
            A, W = rnd(M, K), rnd(N, K)
            R = rnd(M, N, seed=3)
            out = R.clone() if mode == 1 else torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
            _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(out), M, N, K, bn, split, mode, 0, None, 0, 0, None))
            torch.cuda.synchronize()
            ref = A.float() @ W.float().T
            close(out, ref + R.float() if mode == 1 else ref)
        # GeGLU (paired epilogue) and the QKV + KV-append epilogue
        M, F, K, bn = 70, 128, 128, 128
        A, W0, W1 = rnd(M, K), rnd(F, K, seed=1), rnd(F, K, seed=2)
        half = bn // 2
        Wi = torch.empty(2 * F, K, device="cuda", dtype=torch.bfloat16)
        Wi.view(F // half, 2, half, K)[:, 0] = W0.view(F // half, half, K)
        Wi.view(F // half, 2, half, K)[:, 1] = W1.view(F // half, half, K)
        out = torch.zeros(M, F, device="cuda", dtype=torch.bfloat16)
        _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(Wi), P(out), M, 2 * F, K, bn, 2, 2, 0, None, 0, 0, None))
        B, H, Tmax, step = 9, 2, 4, 1
        A, W = rnd(B, 64), rnd(3 * H * 64, 64)
        q = torch.zeros(B, H * 64, device="cuda", dtype=torch.bfloat16)
        cache = torch.zeros(2, B, H, Tmax, 64, device="cuda", dtype=torch.bfloat16)
        _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(q), B, 3 * H * 64, 64, 64, 1, 4, 0, P(cache), Tmax, step, None))
        torch.cuda.synchronize()
    if section("elementwise"):
        x, w = rnd(37, 256, scale=2), rnd(256)
        y = torch.empty_like(x)
        _lib.check(lib.b200t5_test_rmsnorm(DEV, P(x), P(w), P(y), 37, 256, 1e-6, None))
        xa, Wv = rnd(20, 64), rnd(1000, 64)
        toks = torch.zeros(20, device="cuda", dtype=torch.long)
        _lib.check(lib.b200t5_test_lm_argmax(DEV, P(xa), P(Wv), 20, 1000, 64, 0, 1, 2, P(toks), None))
        torch.cuda.synchronize()
        lg = (xa.float() @ Wv.float().T).bfloat16().float()
        lg[:, 1] = -float("inf")
        assert torch.equal(toks, lg.argmax(-1))
    if section("attention"):
        B, H, S = 5, 3, 130
        q, K, V = rnd(B, H, 64, scale=0.3), rnd(B, H, S, 64, scale=1.0, seed=1), rnd(B, H, S, 64, scale=1.0, seed=2)
        extent = torch.tensor([S, 1, 77, 0, 64], device="cuda", dtype=torch.int32)
        key_ok = (torch.arange(S, device="cuda")[None, :] < extent[:, None]).to(torch.uint8).contiguous()
        outs = []
        for impl, arg in ((0, 0), (2, 2), (2, 5)):
            ctx = torch.zeros(B, H * 64, device="cuda", dtype=torch.bfloat16)
            _lib.check(lib.b200t5_test_attn_decode(DEV, impl, P(q), P(K), P(V), P(ctx), B, H, S, P(extent), P(key_ok), arg, None, None))
            torch.cuda.synchronize()
            outs.append(ctx)
        assert torch.equal(outs[1], outs[2])
        close(outs[1], outs[0], 0.02)
        T, step = 40, 17
        Ks, Vs = rnd(B, H, T, 64, scale=1.0, seed=4), rnd(B, H, T, 64, scale=1.0, seed=5)
        bias = rnd(H, T).float().contiguous()
        ctx = torch.zeros(B, H * 64, device="cuda", dtype=torch.bfloat16)
        _lib.check(lib.b200t5_test_attn_decode(DEV, 3, P(q), P(Ks), P(Vs), P(ctx), B, H, T, None, None, step, P(bias), None))
        for impl, (Be, Se, He) in ((1, (2, 128, 2)), (1, (1, 200, 1)), (0, (1, 70, 2))):
            qkv = rnd(Be * Se, 3 * He * 64, scale=0.3)
            rb = rnd(He, 2 * Se - 1).float().contiguous()
            ok = torch.ones(Be, Se, device="cuda", dtype=torch.uint8)
            ext = torch.full((Be,), Se, device="cuda", dtype=torch.int32)
            ctx = torch.zeros(Be * Se, He * 64, device="cuda", dtype=torch.bfloat16)
            _lib.check(lib.b200t5_test_encoder_attn(DEV, P(qkv), P(ctx), P(rb), P(ok), P(ext), Be, Se, He, impl, None))
        torch.cuda.synchronize()
    if section("model"):
        # the whole step graph (PDL chains, two row-chains, finalize / advance) and the slot pool on the tiny model
        spec = SPECS["tiny"]
        for dtype in (torch.bfloat16, torch.float16):
            model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir("tiny", 1), torch_dtype=dtype)
            ids, mask = synthetic_token_batch(6, 24, spec.vocab_size, seed=2, lengths="uniform")
            a = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=4).cpu()
            model.set_option("chains", 2)
            b = model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=4).cpu()
            assert torch.equal(a, b)
            model.set_option("xattn", 1)  # the TMA-stream cross-attention kernel beside the other chain's GEMMs
            model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=4)
            ids2, mask2 = synthetic_token_batch(8, 192, spec.vocab_size, seed=4, lengths="full")
            model.generate(input_ids=torch.from_numpy(ids2), attention_mask=torch.from_numpy(mask2), max_new_tokens=3)
            model.set_option("profile_xattn", 1)  # %globaltimer stamps + the per-layer union fold in advance_step_kernel
            model.generate(input_ids=torch.from_numpy(ids2), attention_mask=torch.from_numpy(mask2), max_new_tokens=3)
            prof = model.xattn_profile()
            assert prof["launches"] > 0 and prof["busy_us_per_layer"] > 0
            model.set_option("profile_xattn", 0)
            model.set_option("xattn", 2)  # per call by prompt fill: full-length -> stream kernel, ragged -> per-thread loads
            model.generate(input_ids=torch.from_numpy(ids2), attention_mask=torch.from_numpy(mask2), max_new_tokens=3)
            assert model.stats()["xattn_kernel"] == 1
            model.set_option("xattn", 0)
            ids, mask = synthetic_token_batch(20, 24, spec.vocab_size, seed=3, lengths="uniform")
            model.generate_stream(ids, mask, pool=8, max_new_tokens=4)
            del model
    if section("logits_process"):
        # EpiLmHead<true, false> + finalize_step_kernel<true, false> + proc_reset_kernel through the hook (a V that is no multiple of
        # 32 or 128, bans at the vocabulary's end), then one small generate and one slot-pool run with every processor
        M, V, K, S, step = 20, 1000, 64, 30, 4
        xa, Wv = rnd(M, K), rnd(V, K)
        hist = torch.randint(0, V, (M, step + 1), device="cuda")
        enc = torch.randint(0, V, (M, S), device="cuda")
        keep = [torch.tensor([V - 1, 3], dtype=torch.int32), torch.tensor([2, V - 1, 998, 999], dtype=torch.int32),
                torch.tensor([0, 1, 4], dtype=torch.int32)]
        lp = _lib.LogitsParams(repetition_penalty=1.3, encoder_repetition_penalty=0.8, no_repeat_ngram_size=2,
                               encoder_no_repeat_ngram_size=2, suppress_tokens=keep[0].data_ptr(), n_suppress_tokens=2,
                               bad_words_ids=keep[1].data_ptr(), bad_words_offsets=keep[2].data_ptr(), n_bad_words=2)
        toks = torch.zeros(M, device="cuda", dtype=torch.long)
        vals = torch.zeros(M, V, device="cuda")
        _lib.check(lib.b200t5_test_lm_process(DEV, P(xa), P(Wv), M, V, K, step, 1, 0, C.byref(lp), P(hist), P(enc), S,
                                              P(toks), P(vals), None))
        torch.cuda.synchronize()
        assert torch.equal(toks, vals.argmax(-1)) and (vals[:, V - 1] == -float("inf")).all()
        spec = SPECS["tiny"]
        model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir("tiny", 1), torch_dtype=torch.bfloat16)
        ids, mask = synthetic_token_batch(6, 24, spec.vocab_size, seed=2, lengths="uniform")
        kw = dict(max_new_tokens=6, repetition_penalty=1.3, encoder_repetition_penalty=0.9, no_repeat_ngram_size=2,
                  encoder_no_repeat_ngram_size=3, bad_words_ids=[[5, 9], [7]], suppress_tokens=[3],
                  begin_suppress_tokens=[2], eos_token_id=[1, 6])
        model.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), **kw)
        ids, mask = synthetic_token_batch(20, 24, spec.vocab_size, seed=3, lengths="uniform")
        model.generate_stream(ids, mask, pool=8, **kw)
        del model
    print("sanitize_kernels: all sections ran", flush=True)


if __name__ == "__main__":
    main()
