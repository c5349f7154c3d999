"""Generates tests/golden/beam.npz: transformers' own beam search (`generate(num_beams=...)`, fp32, CPU) on the seeded
synthetic tiny / mini checkpoints, the fixture of tests/test_beam_cpu.py. The other goldens are not touched. Re-run with:
    python tests/golden/make_golden_beam.py

Per case: sequences, sequences_scores, beam_indices and compute_transition_scores(sequences, scores, beam_indices).
The cases cover k in {2, 4} with n = 1 and n = k, length_penalty in {1.0, 0.0, 2.0, -0.5}, the three early_stopping
values and min_new_tokens; the checkpoints' EOS boost gives hypotheses that end before max_new_tokens.
"""
import json
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch
import transformers

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from anyscale_workshop_nyc_2023_b200.synth import SPECS, save_checkpoint, synthetic_token_batch  # noqa: E402
from oracle.hf_anchor import load_hf_model  # noqa: E402

CHECKPOINTS = {"tiny": (1, 4, 24, 12, 301), "mini": (2, 4, 40, 16, 303)}  # weight seed, B, S, max_new, input seed
# spec, num_beams, num_return_sequences, length_penalty, early_stopping, min_new_tokens
CASES = [("tiny", 2, 1, 1.0, False, 0), ("tiny", 2, 2, 0.0, True, 0), ("tiny", 4, 1, 2.0, "never", 0),
         ("tiny", 4, 4, -0.5, False, 5), ("mini", 4, 1, 1.0, False, 0), ("mini", 2, 2, 2.0, "never", 3),
         ("mini", 4, 4, 0.0, True, 0), ("mini", 2, 1, -0.5, "never", 0), ("mini", 4, 2, 1.0, True, 6)]


@torch.no_grad()
def main():
    res = {"cases": np.array([json.dumps(c) for c in CASES])}
    for spec_name, (wseed, B, S, T, iseed) in CHECKPOINTS.items():
        spec = SPECS[spec_name]
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, iseed, "uniform")
        res[f"{spec_name}_ids"], res[f"{spec_name}_mask"] = ids, mask
        with tempfile.TemporaryDirectory() as d:
            save_checkpoint(d, spec, seed=wseed)
            m = load_hf_model(d, dtype=torch.float32)
            for i, (name, k, n, lp, es, mn) in enumerate(CASES):
                if name != spec_name:
                    continue
                kw = dict(num_beams=k, num_return_sequences=n, length_penalty=lp, early_stopping=es, do_sample=False)
                if mn:
                    kw["min_new_tokens"] = mn
                out = m.generate(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T,
                                 return_dict_in_generate=True, output_scores=True, **kw)
                res[f"c{i}_sequences"] = out.sequences.numpy()
                res[f"c{i}_sequences_scores"] = out.sequences_scores.float().numpy()
                res[f"c{i}_beam_indices"] = out.beam_indices.numpy()
                res[f"c{i}_token_logprobs"] = m.compute_transition_scores(out.sequences, out.scores, out.beam_indices).float().numpy()
    res["meta"] = np.array([f"torch={torch.__version__} transformers={transformers.__version__}"])
    np.savez_compressed(Path(__file__).resolve().parent / "beam.npz", **res)
    print({k: v.shape for k, v in res.items() if k != "meta"})


if __name__ == "__main__":
    main()
