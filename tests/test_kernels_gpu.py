"""Per-kernel parity on an H100: every CUDA kernel is called through the C ABI (include/b200t5.h)
and compared with a plain PyTorch restatement of the same op that rounds where HF eager rounds
(SURVEY Appendix A). Tolerances are written next to each assertion.

Most tests run in both builds: `build` "bf16" is libb200t5.so, "fp16" libb200t5_f16.so (torch_dtype=float16, with an
fp32 residual stream). The reference then computes in that build's activation dtype; a bf16 case keeps the test id
it had before the fp16 cases were added."""
import ctypes as C
import math

import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = 0
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}   # the build's activation dtype (act_t)
RES = {"bf16": torch.bfloat16, "fp16": torch.float32}  # its residual stream / GeGLU output dtype (res_t, ffh_t)
EPS = {"bf16": 2.0 ** -7, "fp16": 2.0 ** -10}         # one ulp relative to the value
ABS = {"bf16": 1e-3, "fp16": 1e-3 / 8}                # absolute floor for cancelled sums, scaled with the precision
# floor on the fraction of a single-rounded GEMM output that is bit-identical to torch's: an fp32 sum that lands near a
# rounding boundary flips under another accumulation order, and fp16's boundaries are 8x denser than bf16's
# (measured on an H100: fp16 >= 0.990 at K = 2048)
EXACT = {"bf16": 0.995, "fp16": 0.985}


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def in_builds(cases, modes=None):
    """Each case in both builds (and, with `modes`, in each mode, the first being the historical one): the bf16 case
    of the first mode keeps its historical id, the others get "-fp16" / "-mode<m>" suffixes."""
    out = []
    for c in cases:
        c = c if isinstance(c, tuple) else (c,)
        cid = "-".join(str(v) for v in c)
        for build in ("bf16", "fp16"):
            bid = cid if build == "bf16" else f"{cid}-fp16"
            if modes is None:
                out.append(pytest.param(*c, build, id=bid))
            else:
                out += [pytest.param(*c, build, m, id=bid if i == 0 else f"{bid}-mode{m}") for i, m in enumerate(modes)]
    return out


@pytest.fixture
def build():
    return "bf16"


@pytest.fixture
def lib(build):
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib.load(build)


def ulp_close(a, b, ulps=1.0, build="bf16"):
    """Tensors equal up to `ulps` units in the last place (of the build's dtype) of the larger magnitude."""
    a, b = a.float(), b.float()
    tol = ulps * EPS[build] * torch.maximum(a.abs(), b.abs()) + 1e-30
    return ((a - b).abs() <= tol)


@pytest.mark.parametrize("M,N,K,bn,build", in_builds([
    (128, 256, 64, 256), (128, 256, 128, 256), (256, 512, 768, 256), (300, 520, 264, 256),
    (4096, 2304, 768, 256), (8, 2304, 768, 64), (256, 768, 768, 32), (256, 768, 2048, 32),
    (256, 1000, 512, 128), (200, 136, 64, 64),
    # bn = 512: the encoder configuration (128 x 256 tiles, weight tile loaded as two 128-row TMA boxes)
    (256, 256, 64, 512), (512, 768, 768, 512), (4096, 2304, 768, 512), (300, 520, 264, 512), (1000, 1000, 2048, 512),
]))
def test_gemm_store(lib, M, N, K, bn, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.5).to(dt)
    Cout = torch.full((M, N), float("nan"), device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_gemm(DEV, P(A), P(W), P(Cout), M, N, K, bn, 0, 0, None), None, lib)
    torch.cuda.synchronize()
    ref32 = A.float() @ W.float().T
    assert torch.isfinite(Cout.float()).all()
    # fp32 accumulation, one rounding to act_t: within 1 ulp of the rounded fp32 reference
    ok = ulp_close(Cout, ref32.to(dt), 1.0, build) | ((Cout.float() - ref32).abs() <= ABS[build])
    assert ok.all(), f"max err {(Cout.float() - ref32).abs().max().item()}"
    exact = (Cout == ref32.to(dt)).float().mean().item()
    print(f"{build} store exact fraction {exact:.5f}")
    assert exact > EXACT[build], exact


def residual_case(M, N, K, build, mode, seed=11):
    """A, W in the build's dtype and R in its stream dtype; returns (A, W, R, reference of the residual phase `mode`)."""
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.2).to(dt)
    R = torch.randn(M, N, device="cuda", generator=g).to(RES[build])
    if mode == 5:
        R = R.to(dt).to(RES[build])  # layer 0: the stream still holds act_t values
    y = (A.float() @ W.float().T).to(dt)
    if build == "bf16" or mode == 5:
        ref = (R.float() + y.float()).to(dt)  # x + Linear(...): two roundings (modeling_t5.py:375)
    else:
        ref = R + y.float()  # fp32 stream + fp16 Linear output: torch promotes, one fp32 add
    return A, W, R, y, ref


def check_residual(Cio, y, ref, build, mode):
    # the Linear output may differ by one ulp of |y| (fp32 accumulation order); after the add
    # that is an absolute error of ulp(y), not a relative one of the (possibly cancelled) sum
    tol = EPS[build] * (y.float().abs() + ref.float().abs()) + ABS[build]
    assert ((Cio.float() - ref.float()).abs() <= tol).all()
    if mode == 5 or build == "bf16":
        assert torch.equal(Cio.float().to(DT[build]).float(), Cio.float())  # the sum is rounded to act_t
    exact = (Cio == ref).float().mean().item()
    print(f"{build} residual mode {mode} exact fraction {exact:.5f}")
    assert exact > 0.99, exact


@pytest.mark.parametrize("M,N,K,bn,build,mode", in_builds([(256, 768, 768, 32), (384, 512, 1024, 256), (130, 264, 128, 256),
                                                           (4096, 768, 2048, 512), (130, 264, 128, 512)], modes=(1, 5)))
def test_gemm_residual(lib, M, N, K, bn, build, mode):
    """mode 1: C = R + act(acc) (fp16 build: fp32 stream); mode 5: the layer-0 phase, C = act(R + act(acc))."""
    A, W, R, y, ref = residual_case(M, N, K, build, mode)
    Cio = R.clone()
    _lib.check(lib.b200t5_test_gemm(DEV, P(A), P(W), P(Cio), M, N, K, bn, mode, 0, None), None, lib)
    torch.cuda.synchronize()
    check_residual(Cio, y, ref, build, mode)


def hf_gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def epilogue_gelu_new(x, build):
    """gelu_new as the build's GeGLU epilogue computes it: HF eager on the GPU in bf16; in fp16 with pow(x, 3.0) rounded
    once (x*x*x in fp32), as CPU torch and the goldens do, one ulp from CUDA torch on 15 inputs (DESIGN.md 4b)."""
    if build == "bf16":
        return hf_gelu_new(x)
    x3 = (x.float() * x.float() * x.float()).to(x.dtype)
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x3)))


def all_bf16_values():
    bits = torch.arange(0, 65536, dtype=torch.int32, device="cuda").to(torch.int16)
    v = bits.view(torch.bfloat16)
    return v[torch.isfinite(v.float())]


def test_geglu_exhaustive(lib):
    """gelu_new over every finite bf16 input must be bit-identical to HF eager on this GPU."""
    x = all_bf16_values()
    ref = hf_gelu_new(x)  # eager bf16: one rounding per op (transformers/activations.py:59-66)
    one = torch.ones_like(x)
    res = {}
    for mode in (0, 1, 2):  # 0 = engine path (table), 2 = op-by-op arithmetic behind the table, 1 = single-rounded pow
        out = torch.empty_like(x)
        _lib.check(lib.b200t5_test_geglu(DEV, P(x), P(one), P(out), x.numel(), mode, None))
        torch.cuda.synchronize()
        res[mode] = (out.view(torch.int16) == ref.view(torch.int16)) | (out.float() == ref.float())
    frac = {m: r.float().mean().item() for m, r in res.items()}
    print("geglu exact-match fraction per pow_mode:", frac)
    assert frac[0] == 1.0 and frac[2] == 1.0, frac  # the engine's path is bit-identical to HF eager on this GPU
    # with a non-trivial multiplier
    g = torch.Generator(device="cuda").manual_seed(3)
    up = torch.randn(x.numel(), device="cuda", generator=g).bfloat16()
    out = torch.empty_like(x)
    _lib.check(lib.b200t5_test_geglu(DEV, P(x), P(up), P(out), x.numel(), 0, None))
    torch.cuda.synchronize()
    ref2 = hf_gelu_new(x) * up
    assert ((out.float() == ref2.float()) | (out.view(torch.int16) == ref2.view(torch.int16))).all()


@pytest.mark.parametrize("M,F,K,bn,build", in_builds([(256, 2048, 768, 64), (512, 1024, 512, 256), (100, 160, 128, 64), (4096, 2048, 768, 512)]))
def test_gemm_geglu(lib, M, F, K, bn, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(5)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W0 = (torch.randn(F, K, device="cuda", generator=g) * 0.1).to(dt)
    W1 = (torch.randn(F, K, device="cuda", generator=g) * 0.1).to(dt)
    tile = 256 if bn == 512 else bn  # the pair kernel's tile is 256 wide
    half = tile // 2
    ntiles = (F + half - 1) // half
    Wi = torch.zeros(ntiles * tile, K, device="cuda", dtype=dt)
    for j in range(ntiles):
        rows = min(half, F - j * half)
        Wi[j * tile: j * tile + rows] = W0[j * half: j * half + rows]
        Wi[j * tile + half: j * tile + half + rows] = W1[j * half: j * half + rows]
    out = torch.full((M, F), float("nan"), device="cuda", dtype=RES[build])
    # N passed = 2F so that the hook derives F = N/2; padded tile rows are zero weights
    assert ntiles * tile == 2 * F or F % half != 0
    _lib.check(lib.b200t5_test_gemm(DEV, P(A), P(Wi), P(out), M, 2 * F if F % half == 0 else ntiles * tile, K, bn, 2, 0, None), None, lib)
    torch.cuda.synchronize()
    if F % half != 0:
        pytest.skip("ragged F is exercised end-to-end only")
    gate = (A.float() @ W0.float().T).to(dt)
    lin = (A.float() @ W1.float().T).to(dt)
    ref = epilogue_gelu_new(gate, build) * lin
    assert torch.isfinite(out.float()).all()
    assert torch.equal(out.to(dt).float(), out.float())  # fp16 build: fp32 storage of fp16 values
    close = ulp_close(out, ref, 2.0, build) | ((out.float() - ref.float()).abs() < 1e-6)
    assert close.float().mean().item() > 0.999
    exact = (out == ref).float().mean().item()
    print(f"{build} geglu exact fraction {exact:.5f}")
    assert exact > 0.98, exact


SK_SHAPES = [
    # M, N, K, bn, split   (the decode-step products of FLAN-T5-base/small/large and ragged edges)
    (256, 768, 768, 64, 4), (256, 768, 2048, 64, 4), (256, 768, 2048, 64, 8), (256, 2304, 768, 128, 4),
    (64, 768, 768, 64, 4), (8, 512, 384, 64, 4), (8, 512, 384, 64, 8), (130, 1024, 2816, 64, 4),
    (256, 1000, 512, 128, 2), (200, 136, 64, 64, 4), (256, 768, 768, 64, 1), (100, 264, 1024, 128, 8),
]


@pytest.mark.parametrize("M,N,K,bn,split,build", in_builds(SK_SHAPES))
def test_gemm_splitk_store(lib, M, N, K, bn, split, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K + split)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.5).to(dt)
    Cout = torch.full((M, N), float("nan"), device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(Cout), M, N, K, bn, split, 0, 0, None, 0, 0, None), None, lib)
    torch.cuda.synchronize()
    ref32 = A.float() @ W.float().T
    assert torch.isfinite(Cout.float()).all()
    # fp32 partial sums added in rank order, one rounding to bf16: within 1 bf16 ulp of the fp32 reference
    ok = ulp_close(Cout, ref32.to(dt), 1.0, build) | ((Cout.float() - ref32).abs() <= ABS[build])
    assert ok.all(), f"max err {(Cout.float() - ref32).abs().max().item()}"
    exact = (Cout == ref32.to(dt)).float().mean().item()
    print(f"{build} split-K store exact fraction {exact:.5f}")
    assert exact > EXACT[build], exact
    # deterministic: the reduction order is fixed
    C2 = torch.empty_like(Cout)
    _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(C2), M, N, K, bn, split, 0, 0, None, 0, 0, None), None, lib)
    torch.cuda.synchronize()
    assert torch.equal(Cout, C2)


@pytest.mark.parametrize("M,N,K,bn,split,build,mode", in_builds([(256, 768, 768, 64, 4), (256, 768, 2048, 64, 8), (130, 264, 128, 128, 2),
                                                                 (37, 512, 1024, 64, 4)], modes=(1, 5)))
def test_gemm_splitk_residual(lib, M, N, K, bn, split, build, mode):
    A, W, R, y, ref = residual_case(M, N, K, build, mode)
    Cio = R.clone()
    _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(Cio), M, N, K, bn, split, mode, 0, None, 0, 0, None), None, lib)
    torch.cuda.synchronize()
    check_residual(Cio, y, ref, build, mode)


@pytest.mark.parametrize("M,F,K,bn,split,build", in_builds([(256, 2048, 768, 128, 2), (256, 2048, 768, 64, 4), (64, 1024, 512, 128, 4), (100, 2816, 1024, 64, 2)]))
def test_gemm_splitk_geglu(lib, M, F, K, bn, split, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(5)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W0 = (torch.randn(F, K, device="cuda", generator=g) * 0.1).to(dt)
    W1 = (torch.randn(F, K, device="cuda", generator=g) * 0.1).to(dt)
    half = bn // 2
    assert F % half == 0
    ntiles = F // half
    Wi = torch.zeros(ntiles * bn, K, device="cuda", dtype=dt)
    Wi.view(ntiles, 2, half, K)[:, 0] = W0.view(ntiles, half, K)
    Wi.view(ntiles, 2, half, K)[:, 1] = W1.view(ntiles, half, K)
    out = torch.full((M, F), float("nan"), device="cuda", dtype=RES[build])
    _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(Wi), P(out), M, 2 * F, K, bn, split, 2, 0, None, 0, 0, None), None, lib)
    torch.cuda.synchronize()
    gate = (A.float() @ W0.float().T).to(dt)
    lin = (A.float() @ W1.float().T).to(dt)
    ref = epilogue_gelu_new(gate, build) * lin
    assert torch.isfinite(out.float()).all()
    assert torch.equal(out.to(dt).float(), out.float())
    close = ulp_close(out, ref, 2.0, build) | ((out.float() - ref.float()).abs() < 1e-6)
    assert close.float().mean().item() > 0.999
    exact = (out == ref).float().mean().item()
    print(f"{build} split-K geglu exact fraction {exact:.5f}")
    assert exact > 0.98, exact


@pytest.mark.parametrize("B,H,K,bn,split,Tmax,step,build", in_builds([(256, 12, 768, 128, 4, 16, 5), (8, 6, 512, 64, 4, 8, 0), (70, 16, 1024, 128, 2, 4, 3)]))
def test_gemm_splitk_qkv_append(lib, B, H, K, bn, split, Tmax, step, build):
    """q -> [B, I]; k/v rows appended in place at cache[kv][b][h][step] (replaces cache_utils.py:119-120)."""
    dt = DT[build]
    I = H * 64
    g = torch.Generator(device="cuda").manual_seed(B + H)
    A = (torch.randn(B, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(3 * I, K, device="cuda", generator=g) * 0.3).to(dt)
    q = torch.full((B, I), float("nan"), device="cuda", dtype=dt)
    cache = torch.zeros(2, B, H, Tmax, 64, device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_gemm_splitk(DEV, P(A), P(W), P(q), B, 3 * I, K, bn, split, 4, 0, P(cache), Tmax, step, None), None, lib)
    torch.cuda.synchronize()
    ref = (A.float() @ W.float().T).to(dt)
    rq, rk, rv = ref[:, :I], ref[:, I:2 * I].view(B, H, 64), ref[:, 2 * I:].view(B, H, 64)
    assert (ulp_close(q, rq, 1.0, build) | ((q.float() - rq.float()).abs() <= ABS[build])).all()
    assert (ulp_close(cache[0, :, :, step], rk, 1.0, build) | ((cache[0, :, :, step].float() - rk.float()).abs() <= ABS[build])).all()
    assert (ulp_close(cache[1, :, :, step], rv, 1.0, build) | ((cache[1, :, :, step].float() - rv.float()).abs() <= ABS[build])).all()
    other = [t for t in range(Tmax) if t != step]
    assert (cache[:, :, :, other] == 0).all()  # no other cache row is touched


def test_gemm_logits_f32(lib, build):
    dt = DT[build]
    M, N, K = 256, 1000, 512
    g = torch.Generator(device="cuda").manual_seed(9)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.5).to(dt)
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
    _lib.check(lib.b200t5_test_gemm(DEV, P(A), P(W), P(out), M, N, K, 128, 3, 0, None), None, lib)
    torch.cuda.synchronize()
    ref = (A.float() @ W.float().T).to(dt).float()
    assert (out == out.to(dt).float()).all()  # values are act_t-representable
    assert (ulp_close(out, ref, 1.0, build) | ((out - ref).abs() <= ABS[build])).all()
    exact = (out == ref).float().mean().item()
    print(f"{build} fp32 logits exact fraction {exact:.5f}")
    assert exact > EXACT[build], exact


def test_gemm_logits_f32_fp16():
    """test_gemm_logits_f32 in the fp16 build (the bf16 case above keeps its historical id)."""
    torch.backends.cuda.matmul.allow_tf32 = False
    test_gemm_logits_f32(_lib.load("fp16"), "fp16")


def rmsnorm_ref(x, w):
    """T5LayerNorm.forward (modeling_t5.py:55-68): x in the stream dtype (fp32 in the fp16 build), w in act_t."""
    var = x.float().pow(2).mean(-1, keepdim=True)
    h = (x * torch.rsqrt(var + 1e-6)).to(w.dtype)
    return w * h


@pytest.mark.parametrize("M,d,build", in_builds([(256, 768), (1000, 512), (37, 1024), (64, 128)]))
def test_rmsnorm(lib, M, d, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(d)
    x = (torch.randn(M, d, device="cuda", generator=g) * 3).to(RES[build])
    w = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(dt)
    y = torch.empty(M, d, device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_rmsnorm(DEV, P(x), P(w), P(y), M, d, 1e-6, None), None, lib)
    torch.cuda.synchronize()
    ref = rmsnorm_ref(x, w)
    assert ulp_close(y, ref, 1.0, build).all()
    exact = (y == ref).float().mean().item()
    print(f"{build} rmsnorm exact fraction {exact:.5f}")
    assert exact > 0.999, exact


def torch_attn_decode(q, K, V, bias_add):
    """q [B,H,64], K/V [B,H,T,64], bias_add [B,H,T] (already bias+mask), all in the build's dtype."""
    dt = q.dtype
    scores = torch.matmul(q.unsqueeze(2).float(), K.float().transpose(2, 3)).to(dt)  # [B,H,1,T]
    scores = scores + bias_add.unsqueeze(2)
    p = torch.softmax(scores.float(), dim=-1).to(dt)
    return torch.matmul(p.float(), V.float()).to(dt).squeeze(2)


def mask_add_of(ok, dt):
    """HF's additive key mask: 0 where attended, finfo(dt).min where not (modeling_t5.py, extended attention mask)."""
    return torch.where(ok, 0.0, torch.finfo(dt).min).to(dt)


@pytest.mark.parametrize("impl", [0, 2])  # 0: per-thread-load kernel (attention_decode.cuh), 2: bulk-copy stream kernel (attention_cross_stream.cuh)
@pytest.mark.parametrize("B,H,S,build", in_builds([(4, 6, 512), (3, 2, 77), (16, 12, 256), (40, 12, 512), (5, 3, 130)]))
def test_cross_attn_decode(lib, B, H, S, impl, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(B * S)
    q = (torch.randn(B, H, 64, device="cuda", generator=g) * 0.3).to(dt)
    K = torch.randn(B, H, S, 64, device="cuda", generator=g).to(dt)
    V = torch.randn(B, H, S, 64, device="cuda", generator=g).to(dt)
    lens = torch.randint(1, S + 1, (B,), generator=torch.Generator().manual_seed(1))
    lens[0] = S
    ok = (torch.arange(S)[None, :] < lens[:, None])
    ok[1, 0] = False  # a hole inside the attended prefix
    if B > 2 and build == "bf16":
        ok[2, :] = False  # fully masked row -> uniform attention over all S keys (HF bf16 behaviour; NaN in fp16)
    ok = ok.cuda()
    extent = torch.where(ok.any(1), ok.float().cumsum(1).argmax(1) + 1, torch.tensor(S, device="cuda")).int()
    key_ok = ok.to(torch.uint8).contiguous()
    ctx = torch.empty(B, H * 64, device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_attn_decode(DEV, impl, P(q), P(K), P(V), P(ctx), B, H, S, P(extent), P(key_ok), 0, None, None), None, lib)
    torch.cuda.synchronize()
    mask_add = mask_add_of(ok, dt)[:, None, :].expand(B, H, S)
    ref = torch_attn_decode(q, K, V, mask_add).reshape(B, H * 64)
    err = (ctx.float() - ref.float()).abs()
    # fp32 accumulation-order noise only: within 2 ulps of |value| or 2e-3 absolute
    assert (err <= 2 * EPS[build] * ref.float().abs() + 2e-3).all(), err.max().item()
    exact = (ctx == ref).float().mean().item()
    print(f"{build} cross-attention impl {impl} exact fraction {exact:.5f}")
    assert exact > 0.97, exact


@pytest.mark.parametrize("stages", [2, 5, 12])
@pytest.mark.parametrize("B,H,S,build", in_builds([(256, 12, 512), (7, 3, 77), (64, 16, 200), (300, 12, 64), (5, 3, 513), (2, 1, 1)]))
def test_cross_attn_stream_kernel_matches_the_per_thread_load_kernel(lib, B, H, S, stages, build):
    """The TMA-stream / mma.sync kernel against the per-thread-load kernel on the same inputs: same rounding points, only
    the order of the fp32 accumulations differs (tensor core vs sequential), so the outputs agree to 2 bf16 ulps and are
    bit-identical in all but a few percent of the elements. Ragged extents, mask holes, retired rows (extent 0),
    persistent CTAs with several items each (B*H > 2 * SMs), every ring depth, S not a multiple of the 64-key chunk
    or of 16 (mask bytes read from global memory instead of riding the ring)."""
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(B * S + stages)
    q = (torch.randn(B, H, 64, device="cuda", generator=g) * 0.3).to(dt)
    K = torch.randn(B, H, S, 64, device="cuda", generator=g).to(dt)
    V = torch.randn(B, H, S, 64, device="cuda", generator=g).to(dt)
    lens = torch.randint(1, S + 1, (B,), generator=torch.Generator().manual_seed(2))
    lens[0] = S
    ok = (torch.arange(S)[None, :] < lens[:, None])
    if S > 4:
        ok[B // 2, 1:3] = False
    extent = lens.clone().int()
    if B > 3:
        extent[3] = 0  # a retired row: nothing is read, the output is zero
    extent, key_ok = extent.cuda(), ok.to(torch.uint8).cuda().contiguous()
    out = []
    for impl, arg in ((0, 0), (2, stages)):
        ctx = torch.full((B, H * 64), float("nan"), device="cuda", dtype=dt)
        _lib.check(lib.b200t5_test_attn_decode(DEV, impl, P(q), P(K), P(V), P(ctx), B, H, S, P(extent), P(key_ok), arg, None, None), None, lib)
        torch.cuda.synchronize()
        out.append(ctx)
    assert torch.isfinite(out[1].float()).all()
    # A score whose fp32 value sits on a bf16 rounding boundary can round differently under the two accumulation
    # orders; on a row with few keys that moves p (and the output) by up to a bf16 ulp of the SCORE, not of the
    # output. Such flips are rare: bound their number and their size, and hold everything else to 2 ulps.
    diff = (out[0].float() - out[1].float()).abs()
    within = ulp_close(out[0], out[1], 2.0, build) | (diff <= 2e-3)
    print(f"{build} stream vs per-thread-load: equal {(out[0] == out[1]).float().mean().item():.4f}, beyond 2 ulp {(~within).float().mean().item():.2e}, max |diff| {diff.max().item():.4f}")
    assert (~within).float().mean().item() <= 2e-4 and diff.max().item() <= 0.06
    assert (out[0] == out[1]).float().mean().item() > 0.9
    # and both against the fp32 restatement with HF's rounding points (as test_cross_attn_decode)
    okb = key_ok.bool()
    mask_add = mask_add_of(okb, dt)[:, None, :].expand(B, H, S)
    keep = (extent > 0) & okb.any(1)
    ref = torch_attn_decode(q, K, V, mask_add).reshape(B, H * 64)
    for o in out:
        err = (o.float() - ref.float()).abs()[keep]
        tol = 2 * EPS[build] * ref.float().abs()[keep] + 2e-3
        assert (err > tol).float().mean().item() <= 2e-4 and err.max().item() <= 0.06
    if B > 3:
        assert (out[1][3] == 0).all()
    # deterministic
    again = torch.empty_like(out[1])
    _lib.check(lib.b200t5_test_attn_decode(DEV, 2, P(q), P(K), P(V), P(again), B, H, S, P(extent), P(key_ok), stages, None, None), None, lib)
    torch.cuda.synchronize()
    assert torch.equal(again.view(torch.int16), out[1].view(torch.int16))


def _argmax_case(lib, x, W, step, eos, min_new):
    M, K = x.shape
    V = W.shape[0]
    toks = torch.full((M,), -7, device="cuda", dtype=torch.long)
    _lib.check(lib.b200t5_test_lm_argmax(DEV, P(x), P(W), M, V, K, step, eos, min_new, P(toks), None), None, lib)
    torch.cuda.synchronize()
    logits = (x.float() @ W.float().T).to(x.dtype).float()  # the lm_head output is rounded to act_t before the arg-max
    if step < min_new:
        logits[:, eos] = -float("inf")
    return toks, logits


def test_fused_argmax_lowest_index_tie_rule(lib, build):
    """torch.argmax returns the FIRST index among equal maxima (transformers generation/utils.py:2762,2793). The fused
    path reduces in three places: inside a 32-column chunk, across the chunks of a 128-column tile (EpiLmHead),
    across tiles and warps (finalize_step_kernel). Exact ties are constructed in all of them, including across the
    last, partial tile of V = 32128 = 251 * 128 and against the masked EOS column."""
    dt = DT[build]
    K, V, M = 64, 32128, 160
    g = torch.Generator(device="cuda").manual_seed(0)
    W = (torch.randn(V, K, device="cuda", generator=g) * 0.05).to(dt)
    x = torch.zeros(M, K, device="cuda", dtype=dt)
    x[:, 0] = 1.0  # logit(n) = W[n, 0] exactly (one product, exact in fp32, act_t in -> act_t out)
    W[:, 0] = (torch.randn(V, device="cuda", generator=g) * 0.5).to(dt).clamp(-3, 3)
    W[:, 1:] = 0
    top = 8.0
    ties = {
        0: [5, 17],                    # same 32-column chunk
        1: [40, 100],                  # same tile, different chunks
        2: [300, 20000],               # different tiles
        3: [127, 128],                 # adjacent columns across a tile boundary
        4: [32000, 32127],             # inside the last tile
        5: [31999, 32127, 7],          # three-way, lowest index far from the others
        6: [1, 2],                     # EOS (= 1) is one of the maxima: blocked while step < min_new, wins afterwards
        7: [0, 32127],                 # first and last column
    }
    Wt = W.clone()
    rows = sorted(ties)
    # every row needs its own tie pattern: give row r the vector e_{r+1} instead and put the pattern in column r+1
    x.zero_()
    for r in range(M):
        x[r, 0] = 1.0
    for r in rows:
        x[r, 0] = 0.0
        x[r, r + 1] = 1.0
        Wt[:, r + 1] = W[:, 0]
        for n in ties[r]:
            Wt[n, r + 1] = top
    for step, min_new in ((0, 4), (4, 4), (9, 0)):
        toks, logits = _argmax_case(lib, x, Wt, step, 1, min_new)
        ref = logits.argmax(dim=-1)  # torch: first index among equal maxima
        assert torch.equal(toks, ref), (step, min_new, toks[:10].tolist(), ref[:10].tolist())
        for r in rows:
            want = min(n for n in ties[r] if not (step < min_new and n == 1))
            assert int(toks[r]) == want, (r, step, int(toks[r]), want)
    # rows >= 8 share one logit vector: all equal, whatever tile row / CTA they sit in
    toks, _ = _argmax_case(lib, x, Wt, 0, 1, 0)
    assert len(set(toks[8:].tolist())) == 1


def test_fused_argmax_lowest_index_tie_rule_fp16():
    """test_fused_argmax_lowest_index_tie_rule in the fp16 build (the bf16 case above keeps its historical id)."""
    test_fused_argmax_lowest_index_tie_rule(_lib.load("fp16"), "fp16")


@pytest.mark.parametrize("V,K,M,build", in_builds([(32128, 768, 256), (1000, 512, 37), (384, 128, 130)]))
def test_fused_argmax_random_with_quantised_ties(lib, V, K, M, build):
    """Random activations against a head quantised so coarsely that many columns share the row maximum exactly."""
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(V + K)
    W = torch.randint(-1, 2, (V, K), device="cuda", generator=g).to(dt)  # {-1, 0, 1}
    # six non-zero activations per row: integer logits in [-6, 6], so the row maximum is shared by many columns
    x = torch.zeros(M, K, device="cuda", dtype=dt)
    cols = torch.rand(M, K, device="cuda", generator=g).argsort(dim=1)[:, :6]
    x.scatter_(1, cols, (torch.randint(0, 2, (M, 6), device="cuda", generator=g) * 2 - 1).to(dt))
    for step, min_new in ((0, 0), (2, 5)):
        toks, logits = _argmax_case(lib, x, W, step, 1, min_new)
        n_ties = (logits == logits.max(dim=-1, keepdim=True).values).sum(-1)
        assert (n_ties > 1).float().mean().item() > 0.2, "the case should contain exact ties"
        assert torch.equal(toks, logits.argmax(dim=-1))


@pytest.mark.parametrize("B,H,T,step,build", in_builds([(4, 6, 128, 0), (4, 6, 128, 5), (8, 12, 128, 127), (3, 2, 40, 33)]))
def test_self_attn_decode(lib, B, H, T, step, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(T + step)
    q = (torch.randn(B, H, 64, device="cuda", generator=g) * 0.3).to(dt)
    K = torch.randn(B, H, T, 64, device="cuda", generator=g).to(dt)
    V = torch.randn(B, H, T, 64, device="cuda", generator=g).to(dt)
    dist_bias = torch.randn(H, T, device="cuda", generator=g).to(dt).float().contiguous()
    ctx = torch.empty(B, H * 64, device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_attn_decode(DEV, 1, P(q), P(K), P(V), P(ctx), B, H, T, None, None, step, P(dist_bias), None), None, lib)
    torch.cuda.synchronize()
    n = step + 1
    j = torch.arange(n, device="cuda")
    bias = dist_bias[:, step - j].to(dt)[None].expand(B, H, n)
    ref = torch_attn_decode(q, K[:, :, :n], V[:, :, :n], bias).reshape(B, H * 64)
    err = (ctx.float() - ref.float()).abs()
    assert (err <= 2 * EPS[build] * ref.float().abs() + 2e-3).all(), err.max().item()
    assert (ctx == ref).float().mean().item() > 0.97


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("B,S,H,build", in_builds([(2, 128, 2), (3, 200, 6), (2, 512, 12), (1, 64, 1), (2, 70, 3), (4, 384, 2)]))
def test_encoder_attn(lib, B, S, H, impl, build):
    dt = DT[build]
    I = H * 64
    g = torch.Generator(device="cuda").manual_seed(S + H)
    qkv = (torch.randn(B * S, 3 * I, device="cuda", generator=g) * 0.5).to(dt)
    rel = torch.randn(H, 2 * S - 1, device="cuda", generator=g).to(dt).float().contiguous()
    lens = torch.randint(1, S + 1, (B,), generator=torch.Generator().manual_seed(2))
    lens[0] = S
    ok = (torch.arange(S)[None, :] < lens[:, None]).cuda()
    if B > 1 and lens[1] > 3:
        ok[1, 1] = False
    extent = (ok.float().cumsum(1).argmax(1) + 1).int()
    key_ok = ok.to(torch.uint8).contiguous()
    ctx = torch.full((B * S, I), float("nan"), device="cuda", dtype=dt)
    _lib.check(lib.b200t5_test_encoder_attn(DEV, P(qkv), P(ctx), P(rel), P(key_ok), P(extent), B, S, H, impl, None), None, lib)
    torch.cuda.synchronize()
    # torch restatement of T5Attention.forward (modeling_t5.py:308-337)
    t = qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)  # [3,B,H,S,64]
    q, k, v = t[0], t[1], t[2]
    scores = torch.matmul(q.float(), k.float().transpose(2, 3)).to(dt)
    i = torch.arange(S, device="cuda")
    bias = rel[:, (i[None, :] - i[:, None]) + S - 1].to(dt)  # [H,S,S] index j-i+S-1
    mask = mask_add_of(ok, dt)[:, None, None, :]
    pb = bias[None] + mask
    scores = scores + pb
    p = torch.softmax(scores.float(), dim=-1).to(dt)
    ref = torch.matmul(p.float(), v.float()).to(dt).permute(0, 2, 1, 3).reshape(B * S, I)
    # padded query rows are never observed downstream (with packed-row addressing, impl 1, they are not computed)
    valid_rows = (torch.arange(S, device="cuda")[None, :] < extent[:, None]).reshape(-1) & ok.reshape(-1)
    out, refv = ctx[valid_rows], ref[valid_rows]
    assert torch.isfinite(out.float()).all()
    err = (out.float() - refv.float()).abs()
    assert (err <= 2 * EPS[build] * refv.float().abs() + 3e-3).all(), err.max().item()
    exact = (out == refv).float().mean().item()
    print(f"{build} encoder attention impl {impl} exact fraction {exact:.5f}")
    assert exact > 0.95, exact


# ------------------------------------------------------------------------------------------------ fp16 build
@pytest.mark.parametrize("M,N,F,kernel,bn,split", [
    (512, 768, 2048, 0, 0, 0),      # encoder shape, encoder GEMM configuration
    (300, 520, 1000, 0, 0, 0),      # ragged everything; F not a multiple of the 32-element k-block
    (256, 768, 2048, 1, 64, 4),     # decode shape, cluster split-K
    (128, 512, 1024, 1, 128, 2),
    (37, 136, 96, 1, 64, 8),        # more ranks than k-blocks allow -> the factor is reduced
])
def test_fp32_weight_ffo_via_two_tf32_passes(M, N, F, kernel, bn, split):
    """`wo` under torch_dtype=float16 is an fp32 Linear (transformers keeps it in fp32): R += A . W^T with fp32 W.
    The tensor cores only offer tf32 (10 mantissa bits); the library multiplies by W_hi and W_lo, both tf32-exact,
    in one K-loop. Error metric: max |err| / sum_k |a||w| against an fp64 product; it grows with K (the tensor
    core's fp32 accumulation truncates) and must stay far below a single tf32 pass (8e-5 .. 2.5e-4) and the fp16
    rounding (4.9e-4) that follows it in T5LayerNorm."""
    lib16 = _lib.load("fp16")
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + 7 * F)
    A = (torch.randn(M, F, device="cuda", generator=g)).half().float()          # fp16 values, as the GeGLU epilogue writes them
    W = torch.randn(N, F, device="cuda", generator=g) * 0.05                     # full fp32 mantissas
    R0 = torch.randn(M, N, device="cuda", generator=g)
    R = R0.clone()
    _lib.check(lib16.b200t5_test_ffo(DEV, P(A), P(W), P(R), M, N, F, kernel, bn, split, None), None, lib16)
    ref = R0.double() + A.double() @ W.double().t()
    scale = (A.double().abs() @ W.double().abs().t()).clamp_min(1e-30)  # sum |a||w|: the natural error scale of a dot product
    err = ((R.double() - ref).abs() / scale).max().item()
    torch.backends.cuda.matmul.allow_tf32 = False
    fp32_err = (((R0 + A @ W.t()).double() - ref).abs() / scale).max().item()
    w_tf32 = (W.view(torch.int32) & -8192).view(torch.float32)  # one tf32 pass: W truncated to 10 mantissa bits
    one_pass_err = (((R0.double() + A.double() @ w_tf32.double().t()) - ref).abs() / scale).max().item()
    print(f"ffo M={M} N={N} F={F} kernel={kernel}: rel err two-pass {err:.2e} | torch fp32 {fp32_err:.2e} | single tf32 pass {one_pass_err:.2e}")
    assert err <= 5e-6 and err <= 0.05 * one_pass_err, (err, fp32_err, one_pass_err)
    # and the bf16 build refuses the hook loudly
    assert _lib.load().b200t5_test_ffo(DEV, P(A), P(W), P(R), M, N, F, kernel, bn, split, None) == _lib.EINVAL
