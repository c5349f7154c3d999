"""Where the encoder's time goes: one encoder pass of FLAN-T5 at the bench shape, per kernel family, from
torch.profiler CUDA kernel records, with the FLOPs and bytes of each product and its share of the dense BF16 peak.

    python tools/profile_encoder.py [--lengths full alpaca] [--enc-gemm 0 1] [--reps 3] [--json OUT]

The cross-attention K/V projection runs in generate, not in encode; it is timed through the single-kernel hook
(b200t5_test_enc_gemm, cross-K/V scatter with packed row maps) at the same M, N, K. With several --enc-gemm settings the
settings alternate within each repetition (option "enc_gemm"), and every figure is the median over repetitions.
Bytes are the algorithmic ones: A and W read once, the output written once, the residual read once."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
from pathlib import Path

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200 import _lib  # noqa: E402
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.roofline import H100_BF16_TFLOPS  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

FAMILIES = ["rmsnorm", "qkv", "attention", "o", "wi (geglu)", "wo", "cross-kv", "other"]


def kernel_records(prof):
    """(start_us, duration_us, name) of every CUDA kernel in the trace, in launch order."""
    out = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start:
            out.append((e.time_range.start, e.time_range.end - e.time_range.start, e.name))
    out.sort()
    return out


def classify(records):
    """Kernel family -> summed microseconds. The two residual products alternate within a layer: O, then wo."""
    t = dict.fromkeys(FAMILIES, 0.0)
    n_res = 0
    for _, dur, name in records:
        if "rmsnorm" in name:
            fam = "rmsnorm"
        elif "encoder_attn" in name:
            fam = "attention"
        elif "EpiCrossKV" in name:
            fam = "cross-kv"
        elif "EpiGeglu" in name:
            fam = "wi (geglu)"
        elif "EpiResidual" in name:
            fam = "o" if n_res % 2 == 0 else "wo"
            n_res += 1
        elif "EpiStore" in name:
            fam = "qkv"
        else:
            fam = "other"
        t[fam] += dur
    return t


def work(spec, extents, fp32_wo):
    """Family -> (FLOP, bytes) of the whole encoder pass over the packed rows."""
    M = float(sum(extents))
    d, inner, f, L = spec.d_model, spec.inner_dim, spec.d_ff, spec.num_layers

    def gemm(n, k, res=False, w_bytes=2):
        return 2.0 * M * n * k, 2.0 * M * k + w_bytes * n * k + 2.0 * M * n * (2 if res else 1)

    out = {
        "qkv": gemm(3 * inner, d),
        "o": gemm(d, inner, res=True),
        "wi (geglu)": (2.0 * M * 2 * f * d, 2.0 * M * d + 2.0 * 2 * f * d + 2.0 * M * f),
        "wo": gemm(d, f, res=True, w_bytes=4 if fp32_wo else 2),
        "attention": (4.0 * inner * float(sum(e * e for e in extents)), 2.0 * M * 3 * inner + 2.0 * M * inner),
        "rmsnorm": (0.0, 2 * (2.0 * M * d + 2.0 * M * d)),
    }
    out = {k: (v[0] * L, v[1] * L) for k, v in out.items()}
    ld = spec.num_decoder_layers
    out["cross-kv"] = (2.0 * M * ld * 2 * inner * d, 2.0 * M * d + 2.0 * ld * 2 * inner * d + 2.0 * M * ld * 2 * inner)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--lengths", nargs="+", default=["full", "alpaca"])
    ap.add_argument("--enc-gemm", nargs="+", type=int, default=[1], help="option enc_gemm settings to alternate")
    ap.add_argument("--dtype", choices=["bf16", "fp16"], default="bf16")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="write the results here as well")
    args = ap.parse_args()

    spec = SPECS[args.model]
    dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(args.model, 0), torch_dtype=dtype)
    lib = _lib.load()  # the bf16 library's single-kernel hooks (cross-K/V projection)
    print(f"device: {torch.cuda.get_device_name(0)}", flush=True)

    results = {}
    for lengths in args.lengths:
        ids, mask = synthetic_token_batch(args.batch, args.seq, spec.vocab_size, seed=1, lengths=lengths)
        extents = mask.sum(1).astype(np.int64)
        M = int(extents.sum())
        ids_t, mask_t = torch.from_numpy(ids), torch.from_numpy(mask)
        # cross-K/V projection operands at the encoder's shape (values do not matter for time)
        H, N, K = spec.num_heads, spec.num_decoder_layers * 2 * spec.inner_dim, spec.d_model
        g = torch.Generator(device="cuda").manual_seed(0)
        A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
        W = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
        ext_t = torch.from_numpy(extents).cuda()
        row_b = torch.repeat_interleave(torch.arange(args.batch, device="cuda"), ext_t).int()
        row_s = (torch.arange(M, device="cuda") - torch.repeat_interleave(torch.cumsum(ext_t, 0) - ext_t, ext_t)).int()
        arena = torch.empty(N // (H * 64), args.batch, H, args.seq, 64, device="cuda", dtype=torch.bfloat16)

        def cross_kv(setting):
            _lib.check(lib.b200t5_test_enc_gemm(0, C.c_void_p(A.data_ptr()), C.c_void_p(W.data_ptr()), C.c_void_p(arena.data_ptr()),
                                                M, N, K, setting, 3, 0, C.c_void_p(row_b.data_ptr()), C.c_void_p(row_s.data_ptr()),
                                                args.batch, H, args.seq, None))

        per = {s: [] for s in args.enc_gemm}
        for rep in range(args.reps):
            order = args.enc_gemm if rep % 2 == 0 else list(reversed(args.enc_gemm))
            for setting in order:
                model.set_option("enc_gemm", setting)
                model.encode(ids_t, mask_t)  # warm: plan, modules
                cross_kv(setting)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    model.encode(ids_t, mask_t)
                    cross_kv(setting)
                    torch.cuda.synchronize()
                per[setting].append(classify(kernel_records(prof)))
        w = work(spec, extents.tolist(), fp32_wo=args.dtype == "fp16")
        results[lengths] = {"packed_rows": M, "settings": {}}
        print(f"\n== {args.model} {args.dtype} B={args.batch} S={args.seq} lengths={lengths}: {M} packed rows, "
              f"median of {args.reps} (kernel time, torch.profiler)")
        print(f"{'family':<12}" + "".join(f"{'enc_gemm=' + str(s) + ' ms':>18}" for s in args.enc_gemm)
              + f"{'GFLOP':>10}{'MB':>10}" + "".join(f"{'TFLOP/s (' + str(s) + ')':>15}{'of 989':>8}" for s in args.enc_gemm))
        med = {s: {f: statistics.median(r[f] for r in per[s]) / 1e3 for f in FAMILIES} for s in args.enc_gemm}
        for f in FAMILIES:
            flop, nbytes = w.get(f, (0.0, 0.0))
            row = f"{f:<12}" + "".join(f"{med[s][f]:>18.3f}" for s in args.enc_gemm) + f"{flop / 1e9:>10.0f}{nbytes / 1e6:>10.0f}"
            for s in args.enc_gemm:
                tf = flop / (med[s][f] * 1e-3) / 1e12 if med[s][f] > 0 and flop > 0 else 0.0
                row += f"{tf:>15.1f}{tf / H100_BF16_TFLOPS:>8.3f}"
            print(row)
        for s in args.enc_gemm:
            enc_ms = sum(v for f, v in med[s].items() if f != "cross-kv")
            gemm_ms = sum(med[s][f] for f in ("qkv", "o", "wi (geglu)", "wo", "cross-kv"))
            print(f"enc_gemm={s}: encoder kernels {enc_ms:.2f} ms + cross-kv {med[s]['cross-kv']:.2f} ms; "
                  f"GEMMs {gemm_ms:.2f} ms, attention {med[s]['attention']:.2f} ms")
            results[lengths]["settings"][str(s)] = {"median_ms": med[s], "runs_ms": [{f: r[f] / 1e3 for f in FAMILIES} for r in per[s]]}
        results[lengths]["work"] = {f: {"flop": v[0], "bytes": v[1]} for f, v in w.items()}
        del arena, A, W
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        Path(args.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
