"""The two 128 x 256 encoder GEMM kernels (csrc/gemm_2cta.cuh) on an H100: gemm_enc_ws_kernel, whose epilogue warps
drain each tile while the next tile's MMAs run, must give bit-identical outputs to gemm_bf16_tn_kernel (option
"enc_gemm" 1 vs 0) for every encoder epilogue, and both must stay within the usual tolerances of a torch reference.
Tile counts run from 1 to far above the 132 SMs, so the staging buffer and its barriers turn over many times.
The kernel tests run in both builds ("bf16": libb200t5.so, "fp16": libb200t5_f16.so, with its fp32 residual stream and
fp32 GeGLU output); a bf16 case keeps the test id it had before the fp16 cases were added."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import _lib
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch

pytestmark = pytest.mark.gpu

DEV = 0


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


DT = {"bf16": torch.bfloat16, "fp16": torch.float16}   # the build's activation dtype
RES = {"bf16": torch.bfloat16, "fp16": torch.float32}  # its residual stream / GeGLU output dtype
EPS = {"bf16": 2.0 ** -7, "fp16": 2.0 ** -10}         # one ulp relative to the value
ABS = {"bf16": 1e-3, "fp16": 1e-3 / 8}
EXACT = {"bf16": 0.995, "fp16": 0.985}  # bit-identical fraction of a single rounding (fp16's boundaries are 8x denser)


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


def alpaca_extents(B=256, S=512):
    _, mask = synthetic_token_batch(B, S, SPECS["flan-t5-base"].vocab_size, seed=1, lengths="alpaca")
    return mask.sum(1).astype(np.int64)


ALPACA_M = int(alpaca_extents().sum())  # packed encoder rows of the alpaca-length bench batch


def rnd(*shape, scale, g, dt=torch.bfloat16):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dt)


def run_both(lib, A, W, make_out, M, N, K, mode, row_b=None, row_s=None, B=0, H=0, S=0):
    outs = []
    for kernel in (0, 1):
        out = make_out()
        _lib.check(lib.b200t5_test_enc_gemm(DEV, P(A), P(W), P(out), M, N, K, kernel, mode, 0, P(row_b), P(row_s), B, H, S, None),
                   None, lib)
        torch.cuda.synchronize()
        outs.append(out)
    return outs


def within_one_ulp(out, ref32, build="bf16"):
    """fp32 accumulation in another order, one rounding: within one ulp of the rounded fp32 reference."""
    ref = ref32.to(DT[build]).float()
    tol = EPS[build] * torch.maximum(out.float().abs(), ref.abs()) + ABS[build]
    exact = (out.float() == ref).float().mean().item()
    print(f"{build} exact fraction {exact:.5f}")
    return ((out.float() - ref).abs() <= tol).all() and exact > EXACT[build]


# (M, N, K): tiles = ceil(M/128) * ceil(N/256) = 1, 6, 9, 132 (one per SM), 288, 9 * 72, ...
@pytest.mark.parametrize("M,N,K,build", in_builds([(128, 256, 64), (130, 520, 264), (300, 768, 768), (1408, 3072, 768),
                                                     (4096, 2304, 768), (4096, 4096, 2048), (ALPACA_M, 18432, 768)]))
def test_store_bit_exact(lib, M, N, K, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + 7 * K)
    A, W = rnd(M, K, scale=0.5, g=g, dt=dt), rnd(N, K, scale=0.5, g=g, dt=dt)
    old, new = run_both(lib, A, W, lambda: torch.full((M, N), float("nan"), device="cuda", dtype=dt), M, N, K, 0)
    assert torch.equal(old, new)
    assert within_one_ulp(new, A.float() @ W.float().T, build)


@pytest.mark.parametrize("M,N,K,build,mode", in_builds([(300, 256, 64), (130, 520, 264), (4096, 768, 768), (4096, 768, 2048),
                                                          (ALPACA_M, 768, 768), (ALPACA_M, 768, 2048)], modes=(1, 5)))
def test_residual_bit_exact(lib, M, N, K, build, mode):
    """mode 1: C = R + act(acc) (fp16 build: fp32 stream); mode 5: the layer-0 phase, C = act(R + act(acc))."""
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(11 + M + N + K)
    A, W = rnd(M, K, scale=0.5, g=g, dt=dt), rnd(N, K, scale=0.2, g=g, dt=dt)
    R = torch.randn(M, N, device="cuda", generator=g).to(RES[build])
    if mode == 5:
        R = R.to(dt).to(RES[build])  # layer 0: the stream still holds act_t values
    old, new = run_both(lib, A, W, lambda: R.clone(), M, N, K, mode)
    assert torch.equal(old, new)
    y = (A.float() @ W.float().T).to(dt)
    ref = (R.float() + y.float()).to(dt) if (build == "bf16" or mode == 5) else R + y.float()
    tol = EPS[build] * (y.float().abs() + ref.float().abs()) + ABS[build]  # one ulp of the Linear output survives the add
    assert ((new.float() - ref.float()).abs() <= tol).all()
    if mode == 5:
        assert torch.equal(new.to(dt).float(), new.float())
    exact = (new == ref).float().mean().item()
    print(f"{build} residual mode {mode} exact fraction {exact:.5f}")
    assert exact > 0.99, exact


def hf_gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * torch.pow(x, 3.0))))


def epilogue_gelu_new(x, build):
    """gelu_new as the build's GeGLU epilogue computes it: HF eager on the GPU in bf16; in fp16 with pow(x, 3.0) rounded
    once (x*x*x in fp32), as CPU torch and the goldens do, one ulp from CUDA torch on 15 inputs (DESIGN.md 4b)."""
    if build == "bf16":
        return hf_gelu_new(x)
    x3 = (x.float() * x.float() * x.float()).to(x.dtype)
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x3)))


@pytest.mark.parametrize("M,F,K,build", in_builds([(130, 256, 64), (300, 1152, 264), (4096, 2048, 768), (ALPACA_M, 2048, 768)]))
def test_geglu_bit_exact(lib, M, F, K, build):
    dt = DT[build]
    g = torch.Generator(device="cuda").manual_seed(5 + M + F)
    A = rnd(M, K, scale=0.5, g=g, dt=dt)
    W0, W1 = rnd(F, K, scale=0.1, g=g, dt=dt), rnd(F, K, scale=0.1, g=g, dt=dt)
    Wi = torch.stack([W0.view(F // 128, 128, K), W1.view(F // 128, 128, K)], 1).reshape(2 * F, K).contiguous()
    old, new = run_both(lib, A, Wi, lambda: torch.full((M, F), float("nan"), device="cuda", dtype=RES[build]), M, 2 * F, K, 2)
    assert torch.equal(old, new)
    assert torch.equal(new.to(dt).float(), new.float())  # fp16 build: fp32 storage of fp16 values
    gate = (A.float() @ W0.float().T).to(dt)
    lin = (A.float() @ W1.float().T).to(dt)
    ref = epilogue_gelu_new(gate, build) * lin
    err = (new.float() - ref.float()).abs()
    close = err <= 2.0 * EPS[build] * torch.maximum(new.float().abs(), ref.float().abs()) + 1e-6
    assert close.float().mean().item() > 0.999
    exact = (new == ref).float().mean().item()
    print(f"{build} geglu exact fraction {exact:.5f}")
    assert exact > 0.98, exact


@pytest.mark.parametrize("packed,build", in_builds([False, True]))
def test_cross_kv_bit_exact(lib, packed, build):
    dt = DT[build]
    H, K = 12, 768
    if packed:  # the alpaca-length bench batch: rows of 256 prompts packed back to back
        B, S = 256, 512
        ext = torch.from_numpy(alpaca_extents(B, S)).cuda()
        row_b = torch.repeat_interleave(torch.arange(B, device="cuda"), ext).int()
        row_s = torch.cat([torch.arange(int(e), device="cuda") for e in ext.tolist()]).int()
        N = 24 * H * 64  # 12 decoder layers x (K, V)
    else:
        B, S = 2, 150
        row_b = row_s = None
        N = 4 * H * 64
    M = int(row_b.numel()) if packed else B * S
    g = torch.Generator(device="cuda").manual_seed(M)
    A, W = rnd(M, K, scale=0.5, g=g, dt=dt), rnd(N, K, scale=0.5, g=g, dt=dt)
    L2 = N // (H * 64)
    old, new = run_both(lib, A, W, lambda: torch.zeros(L2, B, H, S, 64, device="cuda", dtype=dt), M, N, K, 3,
                        row_b, row_s, B, H, S)
    assert torch.equal(old, new)
    rb = row_b.long() if packed else torch.arange(M, device="cuda") // S
    rs = row_s.long() if packed else torch.arange(M, device="cuda") % S
    got = new[:, rb, :, rs, :]  # [M, L2, H, 64]
    assert within_one_ulp(got.reshape(M, N), A.float() @ W.float().T, build)
    if packed:  # positions past a prompt's extent are never written
        del got
        new[:, rb, :, rs, :] = 0
        assert not new.any()


# ------------------------------------------------------------------ model level, both libraries
@pytest.fixture(scope="module", params=[torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def base_model(request):
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir("flan-t5-base", 0), torch_dtype=request.param)
    yield model
    model.set_option("enc_gemm", 1)
    del model
    torch.cuda.empty_cache()


@pytest.mark.parametrize("lengths", ["full", "alpaca"])
def test_model_encode_and_generate_bit_exact(base_model, lengths):
    B, S = 256, 512
    ids, mask = synthetic_token_batch(B, S, SPECS["flan-t5-base"].vocab_size, seed=1, lengths=lengths)
    ids_t, mask_t = torch.from_numpy(ids), torch.from_numpy(mask)
    enc, tok = {}, {}
    for setting in (0, 1):
        base_model.set_option("enc_gemm", setting)
        enc[setting] = base_model.encode(ids_t, mask_t)
        tok[setting] = base_model.generate(input_ids=ids_t, attention_mask=mask_t, max_new_tokens=24).cpu()
    assert torch.equal(enc[0], enc[1])
    assert torch.equal(tok[0], tok[1])
