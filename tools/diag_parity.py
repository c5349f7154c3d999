"""Noise-floor calibration on an H100: how far apart are independent bf16 implementations of the
same T5 forward?  ours (CUDA kernels) / HF eager bf16 on GPU (cuBLAS) / HF eager bf16 on CPU,
all measured against HF fp32 on CPU ("truth"). Writes gpurun_out/diag_parity.json."""
import json
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, save_checkpoint, synthetic_token_batch  # noqa: E402
from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits, load_hf_model  # noqa: E402


def stats(a, b):
    e = np.abs(a - b)
    return {"max": float(e.max()), "mean": float(e.mean()), "exact": float((a == b).mean())}


def main():
    out = {}
    for spec_name, B, S, T, lengths in [("tiny", 6, 24, 12, "uniform"), ("flan-t5-small", 16, 96, 24, "uniform"),
                                        ("flan-t5-small", 8, 128, 16, "full")]:
        spec = SPECS[spec_name]
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=21, lengths=lengths)
        with tempfile.TemporaryDirectory() as d:
            save_checkpoint(d, spec, seed=3)
            ours = B200T5ForConditionalGeneration.from_pretrained(d)
            hf_gpu = load_hf_model(d, dtype=torch.bfloat16, device="cuda")
            hf_cpu = load_hf_model(d, dtype=torch.bfloat16, device="cpu")
            hf_32 = load_hf_model(d, dtype=torch.float32, device="cpu")
            ref_tok = hf_generate(hf_32, ids, mask, T, min_new_tokens=T)
            dec_in = ref_tok[:, :-1]
            L = {
                "ours": ours.decode_logits(ids, mask, dec_in).cpu().numpy(),
                "hf_gpu": hf_teacher_forced_logits(hf_gpu, ids, mask, dec_in),
                "hf_cpu": hf_teacher_forced_logits(hf_cpu, ids, mask, dec_in),
                "fp32": hf_teacher_forced_logits(hf_32, ids, mask, dec_in),
            }
            valid = mask.astype(bool)
            with torch.no_grad():
                E = {
                    "ours": ours.encode(ids, mask).float().cpu().numpy()[valid],
                    "hf_gpu": hf_gpu.encoder(input_ids=torch.from_numpy(ids).cuda(), attention_mask=torch.from_numpy(mask).cuda()).last_hidden_state.float().cpu().numpy()[valid],
                    "hf_cpu": hf_cpu.encoder(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask)).last_hidden_state.float().numpy()[valid],
                    "fp32": hf_32.encoder(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask)).last_hidden_state.float().numpy()[valid],
                }
            key = f"{spec_name}_B{B}_S{S}_{lengths}"
            res = {"logit_scale": float(np.abs(L["fp32"]).max()), "enc_scale": float(np.abs(E["fp32"]).max())}
            for a, b in [("ours", "fp32"), ("hf_gpu", "fp32"), ("hf_cpu", "fp32"), ("ours", "hf_gpu"), ("ours", "hf_cpu"), ("hf_gpu", "hf_cpu")]:
                res[f"logits {a} vs {b}"] = stats(L[a], L[b])
                res[f"enc {a} vs {b}"] = stats(E[a], E[b])
            # argmax agreement with fp32 truth along the fp32 path
            for a in ("ours", "hf_gpu", "hf_cpu"):
                la = L[a].copy()
                la[:, :, spec.eos_token_id] = -np.inf
                lt = L["fp32"].copy()
                lt[:, :, spec.eos_token_id] = -np.inf
                res[f"argmax {a} vs fp32"] = float((la.argmax(-1) == lt.argmax(-1)).mean())
            for a, b in [("ours", "hf_gpu"), ("ours", "hf_cpu"), ("hf_gpu", "hf_cpu")]:
                la, lb = L[a].copy(), L[b].copy()
                la[:, :, spec.eos_token_id] = -np.inf
                lb[:, :, spec.eos_token_id] = -np.inf
                res[f"argmax {a} vs {b}"] = float((la.argmax(-1) == lb.argmax(-1)).mean())
            out[key] = res
            print(key, json.dumps(res, indent=1))
            del ours, hf_gpu
            torch.cuda.empty_cache()
    Path(ROOT / "gpurun_out").mkdir(exist_ok=True)
    (ROOT / "gpurun_out" / "diag_parity.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
