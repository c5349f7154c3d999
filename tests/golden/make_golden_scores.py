"""Generates tests/golden/scores.npz: transformers' own token scores on the seeded synthetic tiny / mini checkpoints
(CPU, nothing is downloaded), the fixture of tests/test_scores_cpu.py. The other goldens are not touched. Re-run with:
    python tests/golden/make_golden_scores.py

Per case and dtype tag (fp32, bf16, fp16), plain and with repetition_penalty=1.3, no_repeat_ngram_size=2 ("_proc"):
generate(return_dict_in_generate=True, output_scores=True) and compute_transition_scores(normalize_logits=False / True);
and model(input_ids, attention_mask, labels).loss with the per-token log-probabilities for ragged labels.
"""
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

CASES = [("tiny", 1, 6, 24, 12, 201), ("mini", 2, 5, 40, 16, 203)]  # spec, weight seed, B, S, max_new, input seed
PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=2)


def ragged_labels(B, L, vocab, seed):
    rng = np.random.default_rng(seed)
    lab = rng.integers(2, vocab, size=(B, L)).astype(np.int64)
    for b, n in enumerate(rng.integers(1, L + 1, size=B)):
        lab[b, n:] = -100
    lab[0, :] = np.where(lab[0] == -100, 3, lab[0])  # one full row
    return lab


@torch.no_grad()
def main_scores():
    res = {}
    for spec_name, wseed, B, S, T, iseed in CASES:
        spec = SPECS[spec_name]
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, iseed, "uniform")
        labels = ragged_labels(B, 7, spec.vocab_size, iseed + 1)
        res[f"{spec_name}_ids"], res[f"{spec_name}_mask"], res[f"{spec_name}_labels"] = ids, mask, labels
        with tempfile.TemporaryDirectory() as d:
            save_checkpoint(d, spec, seed=wseed)
            for tag, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16), ("fp16", torch.float16)):
                m = load_hf_model(d, dtype=dtype)
                tids, tmask = torch.from_numpy(ids), torch.from_numpy(mask)
                for suffix, kw in (("", {}), ("_proc", PROC)):
                    out = m.generate(input_ids=tids, attention_mask=tmask, max_new_tokens=T, do_sample=False, num_beams=1,
                                     return_dict_in_generate=True, output_scores=True, **kw)
                    key = f"{spec_name}_{tag}{suffix}"
                    res[f"{key}_tokens"] = out.sequences.numpy()
                    res[f"{key}_logits"] = m.compute_transition_scores(out.sequences, out.scores, normalize_logits=False).float().numpy()
                    res[f"{key}_logprobs"] = m.compute_transition_scores(out.sequences, out.scores, normalize_logits=True).float().numpy()
                fo = m(input_ids=tids, attention_mask=tmask, labels=torch.from_numpy(labels))
                lsm = torch.log_softmax(fo.logits.float(), dim=-1)
                tl = torch.gather(lsm, 2, torch.from_numpy(np.where(labels == -100, 0, labels))[..., None])[..., 0]
                res[f"{spec_name}_{tag}_label_logprobs"] = torch.where(torch.from_numpy(labels == -100), torch.zeros(()), tl).numpy()
                res[f"{spec_name}_{tag}_loss"] = np.array(float(fo.loss.float()))
    res["meta"] = np.array([f"torch={torch.__version__} transformers={transformers.__version__} proc={PROC}"])
    np.savez_compressed(Path(__file__).resolve().parent / "scores.npz", **res)
    print({k: v.shape for k, v in res.items() if k != "meta"})


if __name__ == "__main__":
    main_scores()
