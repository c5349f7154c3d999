"""Kernel parity in both builds at the edges the shape-parametrised suites do not reach.

`build` "bf16" is libb200t5.so, "fp16" libb200t5_f16.so (torch_dtype=float16: fp16 activations, an fp32 residual
stream, an fp32 GeGLU output holding fp16 values). Every reference is torch eager on the same GPU, rounding where HF
eager rounds:
- gelu_new over every input value, alone and inside every GEMM that runs the GeGLU epilogue, bit for bit (the fp16
  build with the single-rounded pow of CPU torch and the goldens, DESIGN.md 4b);
- fp16 overflow in the GEMM epilogues (inf, as torch gives, before HF's tensor-wide clamp);
- RMSNorm on an fp32 stream with rows beyond the fp16 range and rows below eps;
- fp16 attention with |q.k| in the thousands (T5 does not scale scores by 1/sqrt(d));
- decoder self-attention in both kernels, with one position for all rows or the slot pool's per-row positions."""
import ctypes as C
import math

import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = 0
BUILDS = ["bf16", "fp16"]
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}   # act_t
RES = {"bf16": torch.bfloat16, "fp16": torch.float32}  # res_t / ffh_t
EPS = {"bf16": 2.0 ** -7, "fp16": 2.0 ** -10}


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


@pytest.fixture
def lib(build):
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib.load(build)


def hf_gelu_new(x):
    """transformers' NewGELUActivation (activations.py:59-66), one rounding per op in x's dtype."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def gelu_new_single_pow(x):
    """The same with pow(x, 3.0) rounded once (x*x*x in fp32): CPU torch on fp16, which the oracle's goldens follow."""
    x3 = (x.float() * x.float() * x.float()).to(x.dtype)
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x3)))


def gelu_epilogue_ref(x, build):
    """What the GeGLU epilogue computes: torch on the GPU in the bf16 build, the single-rounded pow in the fp16 build
    (DESIGN.md 4b)."""
    return hf_gelu_new(x) if build == "bf16" else gelu_new_single_pow(x)


def all_values(dt, finite_only):
    bits = torch.arange(0, 65536, dtype=torch.int32, device="cuda").to(torch.int16)
    v = bits.view(dt)
    return v[torch.isfinite(v.float())] if finite_only else v


def same(a, b):
    """Elementwise: equal values (so +0 == -0), or the same NaN / inf positions."""
    a, b = a.float(), b.float()
    return (a == b) | (torch.isnan(a) & torch.isnan(b))


# ------------------------------------------------------------------------------------------------ gelu_new
@pytest.mark.parametrize("build", BUILDS)
def test_gelu_new_every_input_elementwise(lib, build):
    """Mode 0 runs the GeGLU epilogue's own gelu function (bf16: the branch-free table lookup, fp16: the op-by-op
    fp16 arithmetic), checked over every bit pattern, inf and NaN included. Mode 2, the op-by-op arithmetic with the
    double-rounded pow, must equal torch eager on this GPU in both builds: that is the rounding CUDA torch uses. The
    bf16 epilogue equals it; the fp16 epilogue keeps the single-rounded pow of CPU torch and the goldens, one ulp
    away on a handful of inputs (DESIGN.md 4b)."""
    dt = DT[build]
    x = all_values(dt, finite_only=False)
    ref = hf_gelu_new(x)
    one = torch.ones_like(x)
    out = {}
    for mode in (0, 1, 2):
        out[mode] = torch.empty_like(x)
        _lib.check(lib.b200t5_test_geglu(DEV, P(x), P(one), P(out[mode]), x.numel(), mode, None), None, lib)
        torch.cuda.synchronize()
    frac = {m: same(o, ref).float().mean().item() for m, o in out.items()}
    print(f"{build} gelu_new vs torch on this GPU over all 65536 inputs: epilogue {frac[0]:.6f}, single-rounded pow "
          f"{frac[1]:.6f} ({int(round((1 - frac[1]) * 65536))} differ), double-rounded pow {frac[2]:.6f}")
    assert frac[2] == 1.0, frac  # CUDA torch: x*x*x rounded twice, for bf16 and for fp16
    ok = same(out[0], gelu_epilogue_ref(x, build))
    assert ok.all(), x[~ok][:8].float().tolist()
    # the epilogue departs from torch exactly where the two pow roundings differ (none in bf16, 15 inputs in fp16)
    off = ~same(out[0], ref)
    assert torch.equal(off, ~same(out[1], out[2]) if build == "fp16" else torch.zeros_like(off)), off.sum().item()
    g = torch.Generator(device="cuda").manual_seed(7)
    up = torch.randn(x.numel(), device="cuda", generator=g).to(dt)
    res = torch.empty_like(x)
    _lib.check(lib.b200t5_test_geglu(DEV, P(x), P(up), P(res), x.numel(), 0, None), None, lib)
    torch.cuda.synchronize()
    assert same(res, gelu_epilogue_ref(x, build) * up).all()


# (hook, bn / kernel, split): every GEMM that launches EpiGeglu, with the width over which it interleaves gate / up rows
GEGLU_GEMMS = [("enc", 0, 0), ("enc", 1, 0), ("splitk", 64, 4), ("splitk", 128, 2)]


def geglu_half(hook, bn):
    return 128 if hook == "enc" else bn // 2


def run_geglu_gemm(lib, hook, bn, split, A, Wi, out, M, F, K):
    if hook == "enc":
        rc = lib.b200t5_test_enc_gemm(DEV, P(A), P(Wi), P(out), M, 2 * F, K, bn, 2, 0, None, None, 0, 0, 0, None)
    else:
        rc = lib.b200t5_test_gemm_splitk(DEV, P(A), P(Wi), P(out), M, 2 * F, K, bn, split, 2, 0, None, 0, 0, None)
    _lib.check(rc, None, lib)
    torch.cuda.synchronize()


def interleave(W0, W1, half):
    F, K = W0.shape
    n = F // half
    return torch.stack([W0.view(n, half, K), W1.view(n, half, K)], 1).reshape(2 * F, K).contiguous()


@pytest.mark.parametrize("hook,bn,split", GEGLU_GEMMS)
@pytest.mark.parametrize("build", BUILDS)
def test_gelu_new_every_input_through_the_geglu_gemms(lib, build, hook, bn, split):
    """A is the identity, so gate accumulator (m, f) is exactly W0[f, m]: W0 holds every finite input value once
    (only finite ones: 0 * inf in the K-sum would be NaN), and the epilogue's output must be bit-identical to torch's
    gelu_new(gate) * up (fp16: with the goldens' single-rounded pow), with up = 1 and with a random up."""
    dt = DT[build]
    K = F = M = 256
    vals = all_values(dt, finite_only=True)
    W0 = torch.zeros(F * K, device="cuda", dtype=dt)
    W0[: vals.numel()] = vals
    W0 = W0.view(F, K)
    A = torch.eye(M, K, device="cuda", dtype=dt)
    g = torch.Generator(device="cuda").manual_seed(bn + split)
    for W1 in (torch.ones(F, K, device="cuda", dtype=dt), torch.randn(F, K, device="cuda", generator=g).to(dt)):
        Wi = interleave(W0, W1, geglu_half(hook, bn))
        out = torch.full((M, F), float("nan"), device="cuda", dtype=RES[build])
        run_geglu_gemm(lib, hook, bn, split, A, Wi, out, M, F, K)
        ref = gelu_epilogue_ref(W0.T.contiguous(), build) * W1.T
        ok = same(out, ref)
        assert ok.all(), (ok.float().mean().item(), W0.T[~ok][:8].float().tolist(), out[~ok][:8].tolist(), ref[~ok][:8].float().tolist())


# ------------------------------------------------------------------------------------------------ fp16 overflow
def overflow_case(dt):
    """A [128, 64] x W [256, 64]: column n of row m is A[m,0] * W[n,0] + A[m,1] * W[n,1], every product exact in fp32.
    Half the columns go beyond +-65504 (fp16 inf), the rest stay finite."""
    M, N, K = 128, 256, 64
    A = torch.zeros(M, K, device="cuda", dtype=dt)
    A[:, 0] = 200.0
    A[:, 1] = torch.linspace(-4, 4, M, device="cuda").round().to(dt)
    W = torch.zeros(N, K, device="cuda", dtype=dt)
    W[:, 0] = torch.where(torch.arange(N, device="cuda") % 2 == 0, 400.0, 50.0).to(dt) * torch.where(torch.arange(N, device="cuda") % 4 < 2, 1.0, -1.0).to(dt)
    W[:, 1] = torch.arange(N, device="cuda").to(dt)
    return A, W, M, N, K


@pytest.mark.parametrize("hook,bn,split", [("gemm", 512, 0), ("enc", 0, 0), ("enc", 1, 0), ("splitk", 64, 4)])
def test_fp16_epilogues_overflow_to_inf_as_torch(hook, bn, split):
    """An fp16 Linear whose fp32 accumulator lies beyond 65504 gives +-inf in torch, and so must the store, the
    layer-0 residual (fp16 stream: the sum itself may overflow) and the GeGLU gate. (HF's T5Block then clamps inf
    over the whole tensor; DESIGN.md 4b explains why the fused epilogues do not.) The fp32-stream residual (mode 1)
    keeps a finite sum finite."""
    lib = _lib.load("fp16")
    dt = torch.float16
    A, W, M, N, K = overflow_case(dt)

    def gemm(Wt, out, mode, n):
        if hook == "gemm":
            rc = lib.b200t5_test_gemm(DEV, P(A), P(Wt), P(out), M, n, K, bn, mode, 0, None)
        elif hook == "enc":
            rc = lib.b200t5_test_enc_gemm(DEV, P(A), P(Wt), P(out), M, n, K, bn, mode, 0, None, None, 0, 0, 0, None)
        else:
            rc = lib.b200t5_test_gemm_splitk(DEV, P(A), P(Wt), P(out), M, n, K, bn, split, mode, 0, None, 0, 0, None)
        _lib.check(rc, None, lib)
        torch.cuda.synchronize()

    y = (A.float() @ W.float().T).to(dt)
    assert torch.isinf(y).float().mean().item() > 0.3 and torch.isfinite(y).float().mean().item() > 0.3
    out = torch.full((M, N), float("nan"), device="cuda", dtype=dt)
    gemm(W, out, 0, N)
    assert same(out, y).all()
    # residual: R holds fp16 values; 60000 + 10000 overflows fp16 but not fp32
    R = torch.where(torch.arange(N, device="cuda") % 3 == 0, 60000.0, -1.5).expand(M, N).contiguous()
    for mode in (5, 1):
        Cio = R.clone()
        gemm(W, Cio, mode, N)
        ref = (R + y.float()).to(dt).float() if mode == 5 else R + y.float()
        assert same(Cio, ref).all(), mode
    # sums that overflow only through the add (accumulator finite): mode 5 -> inf, mode 1 -> finite
    Ws = torch.zeros(N, K, device="cuda", dtype=dt)
    Ws[:, 0] = 50.0  # acc = 10000 for every column
    ys = (A.float() @ Ws.float().T).to(dt)
    for mode in (5, 1):
        Cio = R.clone()
        gemm(Ws, Cio, mode, N)
        ref = (R + ys.float()).to(dt).float() if mode == 5 else R + ys.float()
        assert same(Cio, ref).all(), mode
        assert torch.isinf(Cio).any().item() == (mode == 5)
    # GeGLU: gate beyond the range -> gelu_new(+inf) = inf, gelu_new(-inf) = NaN (-inf * 0), as in torch
    F = N // 2
    half = 128 if hook == "enc" or bn == 512 else bn // 2
    W0, W1 = W[:F], torch.ones(F, K, device="cuda", dtype=dt) * 0.005
    W1[:, 1:] = 0
    Wi = interleave(W0, W1, half)
    out = torch.full((M, F), 0.0, device="cuda", dtype=torch.float32)
    gemm(Wi, out, 2, 2 * F)
    gate = (A.float() @ W0.float().T).to(dt)
    up = (A.float() @ W1.float().T).to(dt)
    ref = hf_gelu_new(gate) * up
    assert torch.isnan(ref).any() and torch.isinf(ref).any()
    assert same(out, ref).all()


# ------------------------------------------------------------------------------------------------ RMSNorm, fp16
@pytest.mark.parametrize("M,d", [(37, 128), (1000, 512), (130, 768), (64, 1024), (9, 2048)])
def test_fp16_rmsnorm_on_the_fp32_stream(M, d):
    """T5LayerNorm with an fp32 input (the fp16 build's residual stream) and an fp16 weight: the variance and the
    scaling in fp32, one rounding to fp16, the weight product in fp16. Rows far beyond the fp16 range (the fp32 stream
    grows there in FLAN-T5's later layers) and rows so small that eps dominates the variance."""
    lib = _lib.load("fp16")
    g = torch.Generator(device="cuda").manual_seed(M + d)
    x = torch.randn(M, d, device="cuda", generator=g) * 3
    x[1::4] *= 4e4  # |x| up to ~5e5
    x[2::4] *= 1e-4  # variance below eps = 1e-6
    x[3, :] = 0.0
    w = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).half()
    y = torch.full((M, d), float("nan"), device="cuda", dtype=torch.float16)
    _lib.check(lib.b200t5_test_rmsnorm(DEV, P(x), P(w), P(y), M, d, 1e-6, None), None, lib)
    torch.cuda.synchronize()
    var = x.pow(2).mean(-1, keepdim=True)
    ref = w * (x * torch.rsqrt(var + 1e-6)).to(torch.float16)
    assert torch.isfinite(y.float()).all()
    # one ulp of the normalised value h (fp32 sums in another order) becomes up to two ulps of w * h
    assert (y.float() - ref.float()).abs().le(2 * EPS["fp16"] * torch.maximum(y.float().abs(), ref.float().abs()) + 1e-7).all()
    exact = (y == ref).float().mean().item()
    print(f"fp16 rmsnorm d={d} exact fraction {exact:.5f}")
    assert exact > 0.999, exact


# ------------------------------------------------------------------------------------------------ attention, fp16
def int_operand(*shape, g, lim=16):
    """Small integers: q.k is then exact in fp32 whatever the summation order, so the kernel's scores and torch's are
    the same numbers even at magnitudes where one fp16 ulp is 2 or 4."""
    return torch.randint(-lim, lim + 1, shape, device="cuda", generator=g).half()


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("B,S,H", [(2, 128, 2), (3, 200, 6), (2, 70, 3)])
def test_fp16_encoder_attention_large_scores(impl, B, S, H):
    lib = _lib.load("fp16")
    dt = torch.float16
    I = H * 64
    g = torch.Generator(device="cuda").manual_seed(S * H + impl)
    qkv = int_operand(B * S, 3 * I, g=g)
    qkv[:, 2 * I:] = torch.randn(B * S, I, device="cuda", generator=g).half()  # V
    rel = torch.randn(H, 2 * S - 1, device="cuda", generator=g).half().float().contiguous()
    lens = torch.randint(S // 2, S + 1, (B,), generator=torch.Generator().manual_seed(S))
    lens[0] = S
    ok = (torch.arange(S)[None, :] < lens[:, None]).cuda()
    ok[-1, 2] = False
    extent = (ok.float().cumsum(1).argmax(1) + 1).int()
    key_ok = ok.to(torch.uint8).contiguous()
    ctx = torch.full((B * S, I), float("nan"), device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_encoder_attn(DEV, P(qkv), P(ctx), P(rel), P(key_ok), P(extent), B, S, H, impl, None), None, lib)
    torch.cuda.synchronize()
    t = qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = t[0], t[1], t[2]
    raw = torch.matmul(q.float(), k.float().transpose(2, 3))
    assert raw.abs().max().item() > 1000
    scores = raw.to(dt)
    i = torch.arange(S, device="cuda")
    bias = rel[:, (i[None, :] - i[:, None]) + S - 1].to(dt)
    mask = torch.where(ok, 0.0, torch.finfo(dt).min).to(dt)[:, None, None, :]
    scores = scores + (bias[None] + mask)
    p = torch.softmax(scores.float(), dim=-1).to(dt)
    ref = torch.matmul(p.float(), v.float()).to(dt).permute(0, 2, 1, 3).reshape(B * S, I)
    rows = (torch.arange(S, device="cuda")[None, :] < extent[:, None]).reshape(-1) & ok.reshape(-1)
    out, refv = ctx[rows], ref[rows]
    assert torch.isfinite(out.float()).all()
    err = (out.float() - refv.float()).abs()
    assert (err <= 2 * EPS["fp16"] * refv.float().abs() + 2e-3).all(), err.max().item()
    exact = (out == refv).float().mean().item()
    print(f"fp16 encoder attention impl {impl} |q.k| up to {raw.abs().max().item():.0f}: exact fraction {exact:.5f}")
    assert exact > 0.95, exact


@pytest.mark.parametrize("impl,stages", [(0, 0), (2, 2), (2, 5), (2, 12)])
@pytest.mark.parametrize("B,H,S", [(4, 6, 512), (7, 3, 77), (64, 12, 200)])
def test_fp16_cross_attention_large_scores(impl, stages, B, H, S):
    lib = _lib.load("fp16")
    dt = torch.float16
    g = torch.Generator(device="cuda").manual_seed(B * S + stages)
    q = int_operand(B, H, 64, g=g)
    K = int_operand(B, H, S, 64, g=g)
    V = torch.randn(B, H, S, 64, device="cuda", generator=g).half()
    lens = torch.randint(1, S + 1, (B,), generator=torch.Generator().manual_seed(B))
    lens[0] = S
    ok = (torch.arange(S)[None, :] < lens[:, None])
    if lens[1] > 2:
        ok[1, 0] = False
    ok = ok.cuda()
    extent = lens.int().cuda()
    key_ok = ok.to(torch.uint8).contiguous()
    ctx = torch.full((B, H * 64), float("nan"), device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_attn_decode(DEV, impl, P(q), P(K), P(V), P(ctx), B, H, S, P(extent), P(key_ok), stages, None, None),
               None, lib)
    torch.cuda.synchronize()
    raw = torch.matmul(q.unsqueeze(2).float(), K.float().transpose(2, 3))
    assert raw.abs().max().item() > 1000
    mask = torch.where(ok, 0.0, torch.finfo(dt).min).to(dt)[:, None, None, :]
    p = torch.softmax((raw.to(dt) + mask).float(), dim=-1).to(dt)
    ref = torch.matmul(p.float(), V.float()).to(dt).reshape(B, H * 64)
    err = (ctx.float() - ref.float()).abs()
    assert torch.isfinite(ctx.float()).all()
    assert (err <= 2 * EPS["fp16"] * ref.float().abs() + 2e-3).all(), err.max().item()
    exact = (ctx == ref).float().mean().item()
    print(f"fp16 cross-attention impl {impl} stages {stages} |q.k| up to {raw.abs().max().item():.0f}: exact fraction {exact:.5f}")
    assert exact > 0.95, exact


# ------------------------------------------------------------------------------------------------ self-attention decode
def self_attn_ref(q, K, V, dist_bias, pos):
    """Row b attends to keys 0..pos[b] with the bias by distance dist_bias[h, pos[b] - j] (modeling_t5.py:236-251)."""
    dt = q.dtype
    out = []
    for b, t in enumerate(pos.tolist()):
        j = torch.arange(t + 1, device="cuda")
        scores = torch.matmul(q[b].unsqueeze(1).float(), K[b, :, : t + 1].float().transpose(1, 2)).to(dt)  # [H,1,t+1]
        scores = scores + dist_bias[:, t - j].to(dt).unsqueeze(1)
        p = torch.softmax(scores.float(), dim=-1).to(dt)
        out.append(torch.matmul(p.float(), V[b, :, : t + 1].float()).to(dt).reshape(-1))
    return torch.stack(out)


SELF_CASES = [  # B, H, Tmax: Tmax not a multiple of the kernels' 16-key stride
    (5, 6, 37), (8, 12, 100), (3, 16, 130), (4, 12, 128),
]


@pytest.mark.parametrize("kernel", [3])  # attn_decode_kernel<true>, the kernel the decode step runs
@pytest.mark.parametrize("B,H,T", SELF_CASES)
@pytest.mark.parametrize("build", BUILDS)
def test_self_attention_decode_positions(lib, build, kernel, B, H, T):
    """One position for every row (step 0, a middle step, Tmax - 1) and per-row positions as the slot pool runs them
    (extent = positions, step_stride 1), mixing 0, middle positions and Tmax - 1. Cache rows past a row's position
    hold NaN: reading one would show in the output."""
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(B * T + H + kernel)
    q = (torch.randn(B, H, 64, device="cuda", generator=g) * 0.3).to(dt)
    Kc = torch.randn(B, H, T, 64, device="cuda", generator=g).to(dt)
    Vc = torch.randn(B, H, T, 64, device="cuda", generator=g).to(dt)
    dist_bias = torch.randn(H, T, device="cuda", generator=g).to(dt).float().contiguous()
    per_row = torch.tensor([0, T - 1, T // 2, 1, T - 2, 5, T - 1, 0][:B], dtype=torch.int32, device="cuda")
    cases = [(s, None) for s in (0, T // 3, T - 1)] + [(None, per_row)]
    for step, pos in cases:
        pos_all = pos if pos is not None else torch.full((B,), step, dtype=torch.int32, device="cuda")
        live = torch.arange(T, device="cuda")[None, None, :] <= pos_all.long()[:, None, None]  # [B,1,T]
        K = torch.where(live[..., None], Kc, torch.full_like(Kc, float("nan")))
        V = torch.where(live[..., None], Vc, torch.full_like(Vc, float("nan")))
        ctx = torch.full((B, H * 64), float("nan"), device="cuda", dtype=dt)
        _lib.check(lib.b200t5_test_attn_decode(DEV, kernel, P(q), P(K), P(V), P(ctx), B, H, T, P(pos), None,
                                               step if step is not None else 0, P(dist_bias), None), None, lib)
        torch.cuda.synchronize()
        ref = self_attn_ref(q, K, V, dist_bias, pos_all)
        assert torch.isfinite(ctx.float()).all(), (step, pos_all.tolist())
        err = (ctx.float() - ref.float()).abs()
        assert (err <= 2 * EPS[build] * ref.float().abs() + 2e-3).all(), (step, err.max().item())
        exact = (ctx == ref).float().mean().item()
        assert exact > 0.95, (step, exact)
