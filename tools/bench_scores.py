"""Cost of token log-probabilities at the headline shape (FLAN-T5-base, 256 x 512 -> 128 tokens, forced length): decode
time and tokens/s of plain and scored greedy decode (generate(..., return_dict_in_generate=True, output_scores=True)),
alternating three runs of each in one process, the launches of each, and the share of the lm_head GEMM and of the
finalize kernel in each mode from torch.profiler (a run of its own). The card's name and power limit are printed with
the numbers.

    python tools/bench_scores.py [--runs 3] [--batch 256] [--seq 512] [--new 128] [--json OUT]
"""
import argparse
import json
import re
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

SCORED = dict(return_dict_in_generate=True, output_scores=True)
# kernel-name patterns (demangled or mangled template arguments <kProc, kScore>) -> label
TAGS = ((r"EpiLmHead(<false, true>|ILb0ELb1E)", "lm_head (EpiLmHead<false, true>)"),
        (r"EpiLmHead(<false, false>|ILb0ELb0E)", "lm_head (EpiLmHead<false, false>)"),
        (r"finalize_step_kernel(<false, true>|ILb0ELb1E)", "finalize_step_kernel<false, true>"),
        (r"finalize_step_kernel(<false, false>|ILb0ELb0E)", "finalize_step_kernel<false, false>"),
        ("score_reset_kernel", "score_reset_kernel"))


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scores.py measures on a GPU; none found")
    spec = SPECS[a.model]
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(a.model, 0), torch_dtype=torch.bfloat16)
    ids, mask = synthetic_token_batch(a.batch, a.seq, spec.vocab_size, seed=0, lengths="full")
    ids_t, mask_t = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()

    def run(kw):
        out = model.generate(input_ids=ids_t, attention_mask=mask_t, max_new_tokens=a.new, min_new_tokens=a.new, **kw)
        torch.cuda.synchronize()
        st = model.stats()
        return out, st["decode_ms"], st["kernel_launches"]

    settings = {"plain": {}, "scored": SCORED}
    warm = {name: run(kw)[0] for name, kw in settings.items()}  # plans, graphs, result buffers
    same_tokens = bool(torch.equal(warm["plain"], warm["scored"].sequences))
    res = {k: [] for k in settings}
    launches = {}
    for _ in range(a.runs):
        for name, kw in settings.items():
            _, ms, nl = run(kw)
            res[name].append(ms)
            launches[name] = nl
    toks = a.batch * a.new
    share = {}
    for name, kw in settings.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run(kw)
        total, parts = 0.0, {}
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            total += t
            for frag, label in TAGS:
                if re.search(frag, ev.key):
                    parts[label] = parts.get(label, 0.0) + t
                    break
        share[name] = {"gpu_ms": total / 1e3, **{k: {"ms": v / 1e3, "share": v / total} for k, v in parts.items()}}
    summary = {
        "shape": f"{a.model} {a.batch}x{a.seq}->{a.new} forced length, bf16",
        "gpu": torch.cuda.get_device_name(),
        "power_limit": power_limit(),
        "same_tokens": same_tokens,
        "decode_ms": res,
        "decode_ms_median": {k: statistics.median(v) for k, v in res.items()},
        "tokens_per_s": {k: toks / (statistics.median(v) / 1e3) for k, v in res.items()},
        "overhead": statistics.median(res["scored"]) / statistics.median(res["plain"]) - 1.0,
        "kernel_launches": launches,
        "profile": share,
    }
    print(json.dumps(summary, indent=1))
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
