"""Decode-step knob sweep on one H100 without reloading the model: every configuration is a set of
b200t5_set_option values; for each, the decode loop and encoder times (CUDA events inside the library) of a few
forced-length generate calls and the in-situ duration of the cross-attention launches (%globaltimer stamps).

    python tools/sweep_decode.py [--model flan-t5-base] [--batch 256] [--configs "chains=1;chains=2,xattn=0;..."]

Writes gpurun_out/sweep_decode.json and prints one line per configuration."""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200 import roofline  # noqa: E402
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

DEFAULTS = {"chains": 0, "xattn": 2, "xattn_serialize": 0, "xattn_l2pf": 0, "xattn_stages": 5, "xattn_late_pdl": 1, "pdl": 1, "sk_stages64": 0, "sk_stages128": 0}
DEFAULT_CONFIGS = ("chains=1,xattn=0;chains=2,xattn=0;chains=1;chains=2;chains=3;chains=4;"
                   "chains=2,xattn_late_pdl=0;chains=2,xattn_stages=4;chains=2,xattn_stages=6,sk_stages64=3,sk_stages128=2;"
                   "chains=2,xattn_stages=8,sk_stages64=2,sk_stages128=2;chains=3,xattn_stages=4;chains=2,sk_stages64=3")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="flan-t5-base")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--lengths", default="full")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default=DEFAULT_CONFIGS)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    spec = SPECS[a.model]
    model = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir(a.model, 0))
    model.pool_size = max(model.pool_size, a.batch)
    ids, mask = synthetic_token_batch(a.batch, a.seq, spec.vocab_size, seed=1, lengths=a.lengths)
    ids, mask = torch.from_numpy(ids).cuda(), torch.from_numpy(mask).cuda()
    kw = dict(input_ids=ids, attention_mask=mask, max_new_tokens=a.new, min_new_tokens=a.new)
    results, base_tokens = [], None
    for cfg in a.configs.split(";"):
        opts = dict(DEFAULTS)
        for kv in filter(None, cfg.split(",")):
            k, v = kv.split("=")
            opts[k.strip()] = int(v)
        for k, v in opts.items():
            model.set_option(k, v)
        try:
            out = model.generate(**kw)
            model.generate(**kw)
            dec, enc = [], []
            for _ in range(a.reps):
                out = model.generate(**kw)
                st = model.stats()
                dec.append(st["decode_ms"])
                enc.append(st["encoder_ms"])
            rec = {"config": cfg, "decode_ms": min(dec), "decode_ms_all": dec, "encoder_ms": min(enc), "launches": st["kernel_launches"],
                   "decode_frac_of_hbm": st["decode_algo_bytes"] / (min(dec) / 1e3) / 1e9 / roofline.peaks(ROOT)[0]}
            toks = out.cpu()
            if base_tokens is None:
                base_tokens = toks
            rec["tokens_equal_first_config"] = bool(torch.equal(toks, base_tokens))
            if not a.no_profile:
                model.set_option("profile_xattn", 1)
                model.generate(**kw)
                p = model.xattn_profile()
                model.set_option("profile_xattn", 0)
                rec["xattn_in_situ_us"] = p["us_per_launch"]
                rec["xattn_in_situ_gbs"] = p["bytes_per_launch"] / max(p["us_per_launch"], 1e-9) / 1e3
                rec["xattn_launches"] = p["launches"]
                rec["xattn_busy_us_per_layer"] = p["busy_us_per_layer"]
                rec["xattn_layer_gbs"] = p["bytes_per_layer"] / max(p["busy_us_per_layer"], 1e-9) / 1e3
        except Exception as e:  # noqa: BLE001 - keep sweeping; a CUDA fault poisons the context and shows up below
            rec = {"config": cfg, "error": f"{type(e).__name__}: {e}"}
        print(json.dumps(rec), flush=True)
        results.append(rec)
    out_dir = ROOT / "gpurun_out"
    out_dir.mkdir(exist_ok=True)
    (out_dir / "sweep_decode.json").write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
