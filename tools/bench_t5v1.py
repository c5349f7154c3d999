"""T5 v1.0 against FLAN-T5 at the same size: the t5-base shape (ReLU feed-forward, d_ff 3072, tied and rescaled head)
against flan-t5-base (gated-GELU, d_ff 2048), 256 prompts of 512 tokens, 128 forced new tokens (min_new_tokens =
max_new_tokens), alternating runs of the two in one process. Their feed-forward blocks have the same FLOPs and weight
bytes per layer (2 * 768 * 3072 = 3 * 768 * 2048), so the two should cost the same. Reports, per model, the median ms
per batch, the encoder ms (encoder + cross-K/V projection, CUDA events) and its TFLOP/s (the library's encoder_flops),
and the decode ms; then transformers' eager bf16 generate on the t5-base shape on the same GPU (loaded with
`T5ForConditionalGeneration.from_pretrained`, as a user would). `--profile` then runs one call of each model under
torch.profiler and splits its kernel time by GEMM kernel and epilogue (the 128 x 256 encoder GEMMs with EpiRelu /
EpiGeglu for `wi`, EpiResidual for the attention output and `wo`; the split-K decode GEMMs likewise), which is where
the two models differ. The card's name and power limit are printed with the numbers.

    python tools/bench_t5v1.py [--runs 3] [--batch 256] [--seq 512] [--new 128] [--no-hf] [--profile] [--json OUT]
"""
import argparse
import json
import re
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out or "unknown"


def kernel_split(model, ids, mask, kw):
    """{kernel family + epilogue: ms} of one generate call under torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.generate(input_ids=ids, attention_mask=mask, **kw)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if not us:
            continue
        m = re.search(r"(gemm_\w+_kernel)<([^>]*?)(Epi\w+)", e.key)
        if m:
            tile = "<256>" if "256" in m.group(2) else ("<128>" if "128" in m.group(2) else ("<64>" if "64" in m.group(2) else ""))
            name = f"{m.group(1)}{tile} {m.group(3)}"
        else:
            name = "other kernels"
        out[name] = out.get(name, 0.0) + us / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the H100"
    names = ("t5-base", "flan-t5-base")
    models = {n: B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(n), device_map="auto", torch_dtype=torch.bfloat16)
              for n in names}
    ids, mask = synthetic_token_batch(a.batch, a.seq, SPECS["t5-base"].vocab_size, seed=3, lengths="full")
    ids, mask = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    kw = dict(max_new_tokens=a.new, min_new_tokens=a.new)
    res = {n: {"ms": [], "encoder_ms": [], "decode_ms": [], "encoder_tflops": []} for n in names}
    for n in names:  # warm-up: plans, graphs, module loads
        models[n].generate(input_ids=ids, attention_mask=mask, **kw)
    for _ in range(a.runs):
        for n in names:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = models[n].generate(input_ids=ids, attention_mask=mask, **kw)
            torch.cuda.synchronize()
            ms = 1e3 * (time.perf_counter() - t0)
            st = models[n].stats()
            assert out.shape[1] == a.new + 1
            res[n]["ms"].append(ms)
            res[n]["encoder_ms"].append(st["encoder_ms"])
            res[n]["decode_ms"].append(st["decode_ms"])
            res[n]["encoder_tflops"].append(st["encoder_flops"] / (st["encoder_ms"] * 1e-3) / 1e12)
    summary = {"card": card(), "batch": a.batch, "seq": a.seq, "new_tokens": a.new, "runs": a.runs}
    print(f"card: {summary['card']}; {a.batch} prompts x {a.seq} tokens, {a.new} forced new tokens, median of {a.runs} alternated runs")
    for n in names:
        med = {k: statistics.median(v) for k, v in res[n].items()}
        summary[n] = med
        print(f"{n:14s} {med['ms']:9.1f} ms/batch  encoder {med['encoder_ms']:7.1f} ms ({med['encoder_tflops']:6.1f} TFLOP/s)  "
              f"decode {med['decode_ms']:8.1f} ms")
    r = summary["t5-base"]["ms"] / summary["flan-t5-base"]["ms"]
    print(f"t5-base / flan-t5-base: {r:.3f} (encoder {summary['t5-base']['encoder_ms'] / summary['flan-t5-base']['encoder_ms']:.3f}, "
          f"decode {summary['t5-base']['decode_ms'] / summary['flan-t5-base']['decode_ms']:.3f})")
    if a.profile:
        split = {n: kernel_split(models[n], ids, mask, kw) for n in names}
        summary["kernel_ms"] = split
        keys = sorted(set(split[names[0]]) | set(split[names[1]]), key=lambda k: -max(split[names[0]].get(k, 0), split[names[1]].get(k, 0)))
        print(f"torch.profiler, one call each, kernel ms: {'':40s} {names[0]:>12s} {names[1]:>12s}")
        for k in keys:
            print(f"  {k:74s} {split[names[0]].get(k, 0.0):12.2f} {split[names[1]].get(k, 0.0):12.2f}")
        print(f"  {'total':74s} {sum(split[names[0]].values()):12.2f} {sum(split[names[1]].values()):12.2f}")
    if not a.no_hf:
        from transformers import T5ForConditionalGeneration

        del models
        torch.cuda.empty_cache()
        hf = T5ForConditionalGeneration.from_pretrained(str(checkpoint_dir("t5-base")), dtype=torch.bfloat16).to("cuda").eval()
        with torch.no_grad():
            hf.generate(input_ids=ids[:8], attention_mask=mask[:8], max_new_tokens=4, do_sample=False)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hf.generate(input_ids=ids, attention_mask=mask, do_sample=False, num_beams=1, **kw)
            torch.cuda.synchronize()
        summary["transformers_eager_bf16_ms"] = 1e3 * (time.perf_counter() - t0)
        print(f"transformers eager bf16 generate, t5-base shape: {summary['transformers_eager_bf16_ms']:.1f} ms/batch (one run)")
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
