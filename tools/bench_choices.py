"""Cost of multiple-choice scoring (rank classification) at FLAN-T5-base scale: 256 synthetic prompts of 512 tokens, each
with C candidates of 1 to 8 tokens (C = 4, then C = 16). Alternating three runs of each path on the same GPU:
  score_choices            one encoder pass per prompt, the candidates as decoder rows (b200t5_forward_choices);
  forward (repeated)       model(...) on the prompts repeated C times with the candidates as labels, return_logits=False;
  score() (repeated)       the step-loop scorer on the same repeated batch;
  HF eager bf16            transformers' model(..., labels=...) on the same repeated batch, in batches of 256 rows.
Reports the median ms per call, the speedup of score_choices and how far its token log-probabilities are from the other
paths' (score_choices and forward must agree bit for bit). `--profile` runs one score_choices and one repeated forward
under torch.profiler and splits their kernel time into encoder, cross-K/V projection, decoder and lm_head. The card's
name, power limit and clocks are printed with the numbers.

    python tools/bench_choices.py [--runs 3] [--batch 256] [--seq 512] [--choices 4,16] [--no-hf] [--profile] [--json OUT]
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
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration, choice_targets  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

HF_ROWS = 256  # rows per transformers call: the repeated batch of C = 16 would not fit its eager attention at once


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out or "unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def phases(prof):
    """Kernel time by phase, from the kernels in launch order: each call's encoder runs up to its cross-K/V projection
    (EpiCrossKV), its decoder from there to the lm_head (EpiLmHead) and forward_logprob_kernel; anything after an lm_head
    starts the next call (a chunked forward makes several)."""
    evs = [e for e in prof.events() if str(getattr(e, "device_type", "")).endswith("CUDA")]
    evs.sort(key=lambda e: e.time_range.start)
    out = {"encoder": 0.0, "cross-K/V projection": 0.0, "decoder": 0.0, "lm_head": 0.0}
    phase = "encoder"
    for e in evs:
        if "EpiCrossKV" in e.name:
            phase = "cross-K/V projection"
        elif phase == "cross-K/V projection":
            phase = "decoder"
        if "EpiLmHead" in e.name or "forward_logprob" in e.name:
            phase = "lm_head"
        elif phase == "lm_head":
            phase = "encoder"
        out[phase] += e.time_range.elapsed_us() / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--choices", default="4,16")
    ap.add_argument("--max-len", type=int, default=8)
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_choices.py measures on a GPU; none found")
    print("card (name, power limit, max SM clock, max memory clock):", card())
    spec = SPECS[a.model]
    ckpt = checkpoint_dir(a.model, 0)
    model = B200T5ForConditionalGeneration.from_pretrained(ckpt, torch_dtype=torch.bfloat16)
    ids, mask = synthetic_token_batch(a.batch, a.seq, spec.vocab_size, seed=0, lengths="full")
    ids_t, mask_t = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    rng = np.random.default_rng(0)

    def workload(C):
        cands = np.full((a.batch, C, a.max_len), -100, np.int64)
        for b in range(a.batch):
            for c in range(C):
                n = int(rng.integers(1, a.max_len + 1))
                cands[b, c, :n] = rng.integers(2, spec.vocab_size, size=n)
        lab, counts = choice_targets(cands, a.batch, spec.vocab_size)
        rep = torch.from_numpy(np.repeat(np.arange(a.batch), counts)).cuda()
        return torch.from_numpy(cands).cuda(), torch.from_numpy(lab).cuda(), ids_t[rep].contiguous(), mask_t[rep].contiguous()

    if a.profile:
        cands, lab, rids, rmask = workload(int(a.choices.split(",")[0]))
        runs = {"score_choices": lambda: model.score_choices(ids_t, mask_t, cands),
                "forward (repeated)": lambda: model(input_ids=rids, attention_mask=rmask, labels=lab, return_logits=False)}
        for name, fn in runs.items():
            fn()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            split = phases(prof)
            total = sum(split.values())
            print(f"\n{name}, C = {cands.shape[1]}: {total:.2f} ms of kernel time")
            for k, ms in split.items():
                print(f"  {k:22s} {ms:8.2f} ms {100 * ms / max(total, 1e-9):5.1f} %")
            rows = [(e.key, e.device_time_total / 1e3, e.count) for e in prof.key_averages() if e.device_time_total > 0]
            for k, ms, n in sorted(rows, key=lambda r: -r[1])[:8]:
                print(f"    {ms:8.2f} ms x{n:4d}  {k[:100]}")
        return

    hf = None
    if not a.no_hf:
        from oracle.hf_anchor import load_hf_model
        hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
    results = {"card": card(), "batch": a.batch, "seq": a.seq, "shapes": []}
    for C in [int(x) for x in a.choices.split(",")]:
        cands, lab, rids, rmask = workload(C)
        on = lab != -100

        def hf_logprobs():
            out = []
            with torch.no_grad():
                for lo in range(0, rids.shape[0], HF_ROWS):
                    sl = slice(lo, lo + HF_ROWS)
                    lg = hf(input_ids=rids[sl], attention_mask=rmask[sl], labels=lab[sl]).logits
                    lsm = torch.log_softmax(lg.float(), -1)
                    out.append(torch.gather(lsm, 2, torch.where(on[sl], lab[sl], 0)[..., None])[..., 0] * on[sl])
            return torch.cat(out)

        paths = {"score_choices": lambda: model.score_choices(ids_t, mask_t, cands).token_logprobs.reshape(-1, lab.shape[1]),
                 "forward (repeated)": lambda: model(input_ids=rids, attention_mask=rmask, labels=lab, return_logits=False).token_logprobs,
                 "score() (repeated)": lambda: model.score(input_ids=rids, attention_mask=rmask, labels=lab).token_logprobs}
        if hf is not None:
            paths["HF eager bf16 (repeated)"] = hf_logprobs
        times = {k: [] for k in paths}
        outs = {k: fn().float() for k, fn in paths.items()}  # warm-up, and the results compared below
        for _ in range(a.runs):
            for k, fn in paths.items():
                fn()  # score() runs the slot pool, whose execution plan the next path would otherwise rebuild inside its timed call
                times[k].append(timed(fn)[0])
        base = outs["score_choices"]
        med = {k: statistics.median(ts) for k, ts in times.items()}
        print(f"\n{a.model}: {a.batch} prompts x {a.seq} tokens, C = {C} candidates of 1 to {a.max_len} tokens "
              f"({a.batch * C} candidate rows)")
        shape = {"choices": C, "paths": {}}
        for k, ts in times.items():
            diff = (outs[k] - base).abs().max().item()
            print(f"  {k:26s} {med[k]:9.1f} ms (runs {', '.join(f'{t:.1f}' for t in ts)})  "
                  f"x{med[k] / med['score_choices']:6.2f} of score_choices   max |token log-prob - score_choices| {diff:.3g}")
            shape["paths"][k] = {"ms": ts, "max_abs_diff": diff}
        results["shapes"].append(shape)
        del cands, lab, rids, rmask, outs
        torch.cuda.empty_cache()
    if a.json:
        Path(a.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
