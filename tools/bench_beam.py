"""Cost of beam search at the headline shape (FLAN-T5-base, 64 prompts x 512 -> 128 tokens, num_beams=4: 256 decode rows):
ms per batch and decode ms of the beam path with forced length (min_new_tokens=128) and with natural EOS, and of greedy
decoding on 256 prompts (the same row count), alternating three runs of each in one process. Also: the bytes
beam_reorder_kernel moved per step (counted on the device), the torch.profiler share of the lm_head store and of the
three beam kernels (a run of its own), and transformers' eager bf16 generate(num_beams=4) on the same 64 prompts with the
rate at which its best hypotheses' tokens agree with ours. The card's name and power limit are printed with the numbers.

    python tools/bench_beam.py [--runs 3] [--prompts 64] [--beams 4] [--seq 512] [--new 128] [--no-hf] [--json OUT]
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

TAGS = (("EpiStoreF32", "lm_head store (EpiStoreF32)"), ("beam_row_kernel", "beam_row_kernel"),
        ("beam_select_kernel", "beam_select_kernel"), ("beam_reorder_kernel", "beam_reorder_kernel"))


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
    ap.add_argument("--prompts", type=int, default=64)
    ap.add_argument("--beams", type=int, default=4)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_beam.py measures on a GPU; none found")
    spec = SPECS[a.model]
    ckpt = checkpoint_dir(a.model, 0)
    model = B200T5ForConditionalGeneration.from_pretrained(ckpt, torch_dtype=torch.bfloat16)
    rows = a.prompts * a.beams
    model.pool_size = max(model.pool_size, rows)  # one static batch of all prompts
    ids, mask = synthetic_token_batch(rows, a.seq, spec.vocab_size, seed=0, lengths="full")
    ids_t, mask_t = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    bids, bmask = ids_t[: a.prompts].contiguous(), mask_t[: a.prompts].contiguous()

    def run(name):
        kw = dict(max_new_tokens=a.new)
        if name == "greedy":
            x, m = ids_t, mask_t
            kw["min_new_tokens"] = a.new
        else:
            x, m = bids, bmask
            kw["num_beams"] = a.beams
            if name == "beam_forced":
                kw["min_new_tokens"] = a.new
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = model.generate(input_ids=x, attention_mask=m, **kw)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        st = model.stats()
        extra = model.beam_stats() if name != "greedy" else {}
        return out, ms, st["decode_ms"], st["decode_steps"], extra

    names = ("beam_forced", "beam_eos", "greedy")
    warm = {n: run(n)[0] for n in names}  # plans, graphs
    res = {n: {"batch_ms": [], "decode_ms": [], "steps": None, "reorder_bytes_per_step": None} for n in names}
    for _ in range(a.runs):
        for n in names:
            _, ms, dms, steps, extra = run(n)
            res[n]["batch_ms"].append(ms)
            res[n]["decode_ms"].append(dms)
            res[n]["steps"] = steps
            if extra:
                res[n]["reorder_bytes_per_step"] = extra["reorder_bytes"] / max(1, extra["steps"])
    # cross-attention K/V one step streams, for scale: Ld * 2 * rows * H * S * 64 * 2 bytes
    xkv = spec.num_decoder_layers * 2 * rows * spec.num_heads * a.seq * 64 * 2
    share = {}
    for n in ("beam_forced", "greedy"):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run(n)
        total, parts = 0.0, {}
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            total += t
            for frag, label in TAGS:
                if re.search(frag, ev.key):
                    parts[label] = parts.get(label, 0.0) + t
                    break
        share[n] = {"gpu_ms": total / 1e3, **{k: {"ms": v / 1e3, "share": v / total} for k, v in parts.items()}}
    summary = {
        "shape": f"{a.model} {a.prompts} prompts x {a.beams} beams ({rows} rows), {a.seq}->{a.new}, bf16; greedy on {rows} prompts",
        "gpu": torch.cuda.get_device_name(),
        "power_limit": power_limit(),
        "runs": res,
        "median_batch_ms": {n: statistics.median(v["batch_ms"]) for n, v in res.items()},
        "median_decode_ms": {n: statistics.median(v["decode_ms"]) for n, v in res.items()},
        "cross_kv_bytes_per_step": xkv,
        "reorder_vs_cross_kv": {n: res[n]["reorder_bytes_per_step"] / xkv for n in ("beam_forced", "beam_eos")},
        "profile": share,
    }
    if not a.no_hf:
        from oracle.hf_anchor import load_hf_model

        hf = load_hf_model(ckpt, dtype=torch.bfloat16, device="cuda")
        with torch.no_grad():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref = hf.generate(input_ids=bids, attention_mask=bmask, max_new_tokens=a.new, num_beams=a.beams, do_sample=False,
                              return_dict_in_generate=True)
            torch.cuda.synchronize()
            hf_ms = (time.perf_counter() - t0) * 1e3
        ours = warm["beam_eos"]
        L = (ref.beam_indices >= 0).sum(dim=1)  # HF fills a hypothesis' tail with EOS: compare its own tokens only
        W = min(ours.shape[1], ref.sequences.shape[1]) - 1
        pos = torch.arange(W, device=L.device)[None, :] < L[:, None]
        agree = ((ours[:, 1:W + 1] == ref.sequences[:, 1:W + 1]) & pos).sum().item() / max(1, pos.sum().item())
        summary["hf_eager_bf16"] = {"batch_ms": hf_ms, "token_agreement": agree,
                                    "rows_equal": float(((ours[:, 1:W + 1] == ref.sequences[:, 1:W + 1]) | ~pos).all(dim=1).float().mean())}
    print(json.dumps(summary, indent=1))
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
