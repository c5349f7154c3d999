"""Cost of the teacher-forced forward pass (`model(input_ids, attention_mask, labels=...)`, b200t5_forward) at the
notebook's evaluation shape: FLAN-T5-base, 256 prompts of 512 tokens, labels of 512 (the prompts themselves, as the
notebook's Trainer evaluates) and of 128 tokens. Alternating three runs of each: forward for the loss only, forward
with logits, score() on the same labels (the step loop), and transformers' eager bf16 `model(...).loss` on the same GPU.
Reports ms per batch, label positions per second and TFLOP/s (roofline.decoder_forward_flops + encoder_flops) against
the 989 TFLOP/s dense BF16 data-sheet figure, the loss differences, and the label lengths at which score() is faster.
`--profile` runs one loss-only forward under torch.profiler instead and prints the per-kernel breakdown. The card's
name and power limit are printed with the numbers.

    python tools/bench_forward.py [--runs 3] [--batch 256] [--seq 512] [--labels 512,128] [--no-hf] [--profile] [--json OUT]
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200 import roofline  # noqa: E402
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return out or "unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--labels", default="512,128")
    ap.add_argument("--crossover", default="1,2,4,8,16,32", help="label lengths at which forward and score() are compared")
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_forward.py measures on a GPU; none found")
    print("card:", card())
    spec = SPECS[a.model]
    ckpt = checkpoint_dir(a.model, 0)
    model = B200T5ForConditionalGeneration.from_pretrained(ckpt, torch_dtype=torch.bfloat16)
    ids, mask = synthetic_token_batch(a.batch, a.seq, spec.vocab_size, seed=0, lengths="full")
    ids_t, mask_t = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()

    def labels_of(L):
        lab = np.full((a.batch, L), -100, np.int64)
        n = min(L, a.seq)
        lab[:, :n] = np.where(mask[:, :n] != 0, ids[:, :n], -100)
        return torch.from_numpy(lab).cuda()

    if a.profile:
        lab = labels_of(int(a.labels.split(",")[0]))
        model(input_ids=ids_t, attention_mask=mask_t, labels=lab, return_logits=False)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            model(input_ids=ids_t, attention_mask=mask_t, labels=lab, return_logits=False)
            torch.cuda.synchronize()
        rows = [(e.key, e.device_time_total / 1e3, e.count) for e in prof.key_averages() if e.device_time_total > 0]
        total = sum(r[1] for r in rows)
        print(f"per-kernel breakdown, loss-only forward, labels {lab.shape[1]} (total {total:.1f} ms of kernel time):")
        for k, ms, n in sorted(rows, key=lambda r: -r[1])[:20]:
            print(f"  {ms:9.2f} ms {100 * ms / total:5.1f} %  x{n:4d}  {k[:110]}")
        return

    hf = None
    if not a.no_hf:
        from oracle.hf_anchor import load_hf_model
        hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
    ext = [int(m.nonzero()[0][-1]) + 1 for m in mask]
    results = {"card": card(), "shapes": []}
    for L in [int(x) for x in a.labels.split(",")]:
        lab = labels_of(L)
        flops = roofline.decoder_forward_flops(spec, a.batch, L, extents=ext) + roofline.encoder_flops(spec, a.batch, extents=ext)
        paths = {"forward (loss)": lambda: model(input_ids=ids_t, attention_mask=mask_t, labels=lab, return_logits=False).loss,
                 "forward (loss + logits)": lambda: model(input_ids=ids_t, attention_mask=mask_t, labels=lab).loss,
                 "score()": lambda: model.score(input_ids=ids_t, attention_mask=mask_t, labels=lab).loss}
        if hf is not None:
            def hf_loss():
                with torch.no_grad():
                    return hf(input_ids=ids_t, attention_mask=mask_t, labels=lab).loss
            paths["HF eager bf16"] = hf_loss
        times = {k: [] for k in paths}
        losses = {}
        for k, fn in paths.items():  # warm-up
            losses[k] = float(fn())
        for _ in range(a.runs):
            for k, fn in paths.items():
                ms, _ = timed(fn)
                times[k].append(ms)
        print(f"\nFLAN-T5 {a.model}: {a.batch} prompts x {a.seq} tokens, {L} labels; {flops / 1e12:.2f} TFLOP (decoder + lm_head + encoder)")
        shape = {"labels": L, "tflop": flops / 1e12, "paths": {}}
        for k, ts in times.items():
            med = statistics.median(ts)
            pos = a.batch * L / (med / 1e3)
            tf = flops / (med / 1e3) / 1e12
            print(f"  {k:26s} {med:9.1f} ms (runs {', '.join(f'{t:.1f}' for t in ts)})  {pos:12.0f} label positions/s  "
                  f"{tf:6.1f} TFLOP/s = {100 * tf / PEAK_TFLOPS:4.1f} % of {PEAK_TFLOPS:.0f}   loss {losses[k]:.5f}")
            shape["paths"][k] = {"ms": ts, "loss": losses[k]}
        print(f"  |loss_forward - loss_score| = {abs(losses['forward (loss)'] - losses['score()']):.3g}"
              + (f"   |loss_forward - loss_HF| = {abs(losses['forward (loss)'] - losses['HF eager bf16']):.3g}" if hf is not None else ""))
        results["shapes"].append(shape)
        del lab
        torch.cuda.empty_cache()
    print("\ncrossover (median of two runs each):")
    cross = []
    for L in [int(x) for x in a.crossover.split(",")]:
        lab = labels_of(L)
        f = lambda: model(input_ids=ids_t, attention_mask=mask_t, labels=lab, return_logits=False).loss  # noqa: E731
        s = lambda: model.score(input_ids=ids_t, attention_mask=mask_t, labels=lab).loss  # noqa: E731
        f(), s()
        tf = statistics.median([timed(f)[0] for _ in range(2)])
        ts = statistics.median([timed(s)[0] for _ in range(2)])
        print(f"  labels {L:4d}: forward {tf:8.1f} ms   score() {ts:8.1f} ms   {'score() faster' if ts < tf else 'forward faster'}")
        cross.append({"labels": L, "forward_ms": tf, "score_ms": ts})
    results["crossover"] = cross
    if a.json:
        Path(a.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
