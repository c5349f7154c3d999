"""Cost of the greedy logits processors at the headline shape (FLAN-T5-base, 256 x 512 -> 128 tokens, forced length):
decode time and tokens/s with no processors and with repetition_penalty=1.2, no_repeat_ngram_size=3, alternating
three runs of each, and the processor kernels' share of the decode time from torch.profiler.

    python tools/bench_logits_process.py [--runs 3] [--batch 256] [--seq 512] [--new 128] [--json OUT]
"""
import argparse
import json
import re
import statistics
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

PROC = dict(repetition_penalty=1.2, no_repeat_ngram_size=3)
# kernel-name patterns (demangled or mangled template arguments <kProc, kScore>) -> label
TAGS = (("proc_reset_kernel", "proc_reset_kernel"),
        (r"EpiLmHead(<true, false>|ILb1ELb0E)", "lm_head (EpiLmHead<true, false>)"),
        (r"EpiLmHead(<false, false>|ILb0ELb0E)", "lm_head (EpiLmHead<false, false>)"),
        (r"finalize_step_kernel(<true, false>|ILb1ELb0E)", "finalize_step_kernel<true, false>"),
        (r"finalize_step_kernel(<false, false>|ILb0ELb0E)", "finalize_step_kernel<false, false>"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    spec = SPECS[a.model]
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(a.model, 0), torch_dtype=torch.bfloat16)
    ids, mask = synthetic_token_batch(a.batch, a.seq, spec.vocab_size, seed=0, lengths="full")
    ids_t, mask_t = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()

    def run(kw):
        out = model.generate(input_ids=ids_t, attention_mask=mask_t, max_new_tokens=a.new, min_new_tokens=a.new, **kw)
        torch.cuda.synchronize()
        st = model.stats()
        return out, st["decode_ms"], st["kernel_launches"]

    settings = {"none": {}, "processors": PROC}
    for kw in settings.values():  # warm-up: plans, graphs, processor state
        run(kw)
    res = {k: [] for k in settings}
    launches = {}
    for _ in range(a.runs):
        for name, kw in settings.items():
            _, ms, nl = run(kw)
            res[name].append(ms)
            launches[name] = nl
    toks = a.batch * a.new
    # share of the call's GPU time: proc_reset_kernel, the lm_head with processors and finalize_step_kernel<true, false>
    # (which computes the bans), against the same kernels of the plain step
    share = {}
    for name, kw in settings.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run(kw)
        total, parts = 0.0, {}
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            total += t
            for pat, key in TAGS:
                if re.search(pat, ev.key):
                    parts[key] = parts.get(key, 0.0) + t
                    break
        share[name] = {k: v / total for k, v in parts.items()}
    summary = {
        "shape": f"{a.model} {a.batch}x{a.seq}->{a.new} forced length, bf16",
        "gpu": torch.cuda.get_device_name(),
        "decode_ms": {k: v for k, v in res.items()},
        "decode_ms_median": {k: statistics.median(v) for k, v in res.items()},
        "tokens_per_s": {k: toks / (statistics.median(v) / 1e3) for k, v in res.items()},
        "overhead": statistics.median(res["processors"]) / statistics.median(res["none"]) - 1.0,
        "kernel_launches": launches,
        "profile_share": share,
    }
    print(json.dumps(summary, indent=1))
    if a.json:
        Path(a.json).write_text(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
