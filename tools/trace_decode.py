"""Kernel timeline of a few decode steps on an H100 (CUPTI via torch.profiler: every kernel in the
process is traced, including the graph-launched ones of libb200t5). Writes gpurun_out/trace_<tag>.json
with (name, start_us, dur_us, stream) tuples; analyse with tools/analyze_trace.py."""
import json
import os
import sys
from pathlib import Path

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "default"
    model_name = os.environ.get("TRACE_MODEL", "flan-t5-base")
    B, S, T = int(os.environ.get("TRACE_B", 256)), int(os.environ.get("TRACE_S", 512)), int(os.environ.get("TRACE_T", 12))
    spec = SPECS[model_name]
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(model_name, 0))
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=1, lengths="full")
    ids, mask = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    for _ in range(2):
        model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=T, min_new_tokens=T)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=T, min_new_tokens=T)
        torch.cuda.synchronize()
    ev = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            ev.append({"name": e.name[:100], "start": e.time_range.start, "dur": e.time_range.end - e.time_range.start,
                       "stream": getattr(e, "device_index", 0)})
    out = ROOT / "gpurun_out" / f"trace_{tag}.json"
    out.parent.mkdir(exist_ok=True)
    prof.export_chrome_trace(str(ROOT / "gpurun_out" / f"chrome_{tag}.json"))
    out.write_text(json.dumps(ev))
    print(tag, len(ev), "events", model.stats())


if __name__ == "__main__":
    main()
