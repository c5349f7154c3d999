"""Cost of a decoder prompt (`generate(decoder_input_ids=...)`, b200t5_generate_prefixed) at the README's decode shape:
FLAN-T5-base, 256 prompts of 512 tokens, decoder prompts of P ids (start token included), then 64 new tokens with EOS
masked (min_new_tokens = max_new_tokens), so every row runs every step.

For each P the prefixed call is compared with the same call without a prompt and max_new_tokens = P-1 + 64: that call
runs the P-1 extra decode steps step-forcing the prompt would run, on the same plan (same Tmax), so it costs exactly
what step-forcing costs. Three alternated runs of each, in one process. A second loop reads the library's CUDA events:
`stats()["encoder_ms"]` spans the encoder pass up to the first decode step, which for a prefixed call also holds the
prompt's embedding, the prefill and the prompt's start-of-decoding kernel, so the difference of the two calls' median
spans is the cost the prompt adds before the first step (not events placed around the prefill alone).
`--profile` instead runs one prefixed call per P under torch.profiler (a run of its own) and prints the prefill's
kernels: every GPU activity after the cross-K/V projection (the last `EpiCrossKV` GEMM) and before
`decode_init_prompt_kernel`, with each kernel's summed time, their span and the idle time inside the span. The card's
name and power limit are printed with the numbers.

    python tools/bench_prefix.py [--runs 3] [--batch 256] [--seq 512] [--new 64] [--prompts 2,8,32,64] [--profile] [--json OUT]
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
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402


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


def gpu_activities(prof):
    """(name, start us, duration us) of every GPU activity of a profile, in start order."""
    out = []
    for e in prof.events():
        if getattr(e, "device_type", None) == torch.autograd.DeviceType.CUDA:
            out.append((e.name, e.time_range.start, e.time_range.end - e.time_range.start))
    if not out:  # kineto's own records
        for e in prof.profiler.kineto_results.events():
            if e.device_type() == torch.autograd.DeviceType.CUDA:
                out.append((e.name(), e.start_ns() / 1e3, e.duration_ns() / 1e3))
    return sorted(out, key=lambda r: r[1])


def profile_prefill(model, call, P):
    call()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    acts = gpu_activities(prof)
    xkv = [i for i, r in enumerate(acts) if "EpiCrossKV" in r[0]]
    init = [i for i, r in enumerate(acts) if "decode_init_prompt_kernel" in r[0]]
    if not xkv or not init:
        print(f"P = {P}: could not find the prefill's bounds among {len(acts)} GPU activities")
        return None
    win = acts[xkv[-1] + 1: init[0]]
    if not win:
        print(f"P = {P}: no GPU activity between the cross-K/V projection and decode_init_prompt_kernel")
        return None
    busy = sum(r[2] for r in win)
    span = win[-1][1] + win[-1][2] - win[0][1]
    per = {}
    for name, _, dur in win:
        n, t = per.get(name, (0, 0.0))
        per[name] = (n + 1, t + dur)
    print(f"\nP = {P}: prefill = {len(win)} GPU activities, {busy / 1e3:.3f} ms of kernel time in a {span / 1e3:.3f} ms span "
          f"({(span - busy) / 1e3:.3f} ms idle)")
    for name, (n, t) in sorted(per.items(), key=lambda kv: -kv[1][1]):
        print(f"  {t / 1e3:8.3f} ms {100 * t / busy:5.1f} %  x{n:3d}  {name[:110]}")
    return {"P": P, "busy_ms": busy / 1e3, "span_ms": span / 1e3, "kernels": {k: {"n": n, "ms": t / 1e3} for k, (n, t) in per.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--prompts", default="2,8,32,64", help="decoder prompt lengths P, start token included")
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prefix.py measures on a GPU; none found")
    print("card:", card())
    spec = SPECS[a.model]
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(a.model, 0), torch_dtype=torch.bfloat16)
    ids, mask = synthetic_token_batch(a.batch, a.seq, spec.vocab_size, seed=0, lengths="full")
    ids_t, mask_t = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    rng = np.random.default_rng(1)
    results = {"card": card(), "batch": a.batch, "seq": a.seq, "new": a.new, "shapes": []}
    if a.profile:
        results["profiles"] = []
        for P in [int(x) for x in a.prompts.split(",")]:
            d = np.concatenate([np.zeros((a.batch, 1), np.int64), rng.integers(3, spec.vocab_size, size=(a.batch, P - 1))], axis=1)
            call = lambda: model.generate(input_ids=ids_t, attention_mask=mask_t, decoder_input_ids=d, max_new_tokens=a.new,  # noqa: E731
                                          min_new_tokens=a.new)
            results["profiles"].append(profile_prefill(model, call, P))
        if a.json:
            Path(a.json).write_text(json.dumps(results, indent=1))
        return
    print(f"FLAN-T5 {a.model}: {a.batch} prompts x {a.seq} tokens, decoder prompt of P ids, then {a.new} forced new tokens")
    for P in [int(x) for x in a.prompts.split(",")]:
        d = np.concatenate([np.zeros((a.batch, 1), np.int64), rng.integers(3, spec.vocab_size, size=(a.batch, P - 1))], axis=1)
        T2 = P - 1 + a.new
        paths = {
            "prefill + decode": lambda: model.generate(input_ids=ids_t, attention_mask=mask_t, decoder_input_ids=d, max_new_tokens=a.new,
                                                       min_new_tokens=a.new),
            "step-forced": lambda: model.generate(input_ids=ids_t, attention_mask=mask_t, max_new_tokens=T2, min_new_tokens=T2),
        }
        times = {k: [] for k in paths}
        for fn in paths.values():  # warm-up: plan, graphs
            fn()
        for _ in range(a.runs):
            for k, fn in paths.items():
                times[k].append(timed(fn)[0])
        # what the prompt adds before the first step: encoder_ms (CUDA events from the encoder to the first decode step)
        # with and without it
        enc = {k: [] for k in paths}
        for _ in range(a.runs):
            for k, fn in paths.items():
                fn()
                enc[k].append(model.stats()["encoder_ms"])
        prefill = statistics.median(enc["prefill + decode"]) - statistics.median(enc["step-forced"])
        med = {k: statistics.median(ts) for k, ts in times.items()}
        print(f"\nP = {P}: {P - 1} prompt positions per row")
        for k, ts in times.items():
            print(f"  {k:18s} {med[k]:9.1f} ms (runs {', '.join(f'{t:.1f}' for t in ts)})")
        verdict = "prefill faster" if med["prefill + decode"] < med["step-forced"] else "step-forcing faster or equal"
        print(f"  saved {med['step-forced'] - med['prefill + decode']:8.1f} ms ({verdict});  added before the first step {prefill:.2f} ms "
              f"(encoder-span events {statistics.median(enc['prefill + decode']):.2f} vs {statistics.median(enc['step-forced']):.2f} ms)")
        results["shapes"].append({"P": P, "ms": times, "encoder_ms": enc, "added_before_first_step_ms": prefill})
    if a.json:
        Path(a.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
