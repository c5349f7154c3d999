"""Generates tests/golden/*.npz by running the reference's own dependency (transformers'
T5ForConditionalGeneration.generate, eager attention) on seeded synthetic checkpoints, in the
build container (CPU). Re-run with:  python tests/golden/make_golden.py   (--fp16: only the *_fp16.npz files)
The fixtures pin oracle/t5_oracle.py; they are environment-stamped (torch / transformers versions).

    B200T5_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden.py --reference-predictor

runs the reference's own NLP_workloads/Anyscale_job/predictor.py and utils.py, unmodified, through the shim on the
inputs of tests/test_reference_predictor_cpu.py and stores what they return in reference_predictor.npz (strings and
token arrays only; nothing of the reference's code).
"""
import sys
from pathlib import Path

import numpy as np
import torch
import transformers

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from anyscale_workshop_nyc_2023_b200.synth import SPECS, save_checkpoint, synthetic_token_batch  # noqa: E402
from oracle.hf_anchor import hf_generate, hf_teacher_forced_logits, load_hf_model  # noqa: E402

CASES = [  # name, spec, weight seed, B, S, max_new, input seed, lengths
    ("tiny_a", "tiny", 1, 6, 24, 12, 101, "uniform"),
    ("tiny_full", "tiny", 1, 4, 16, 10, 102, "full"),
    ("mini_a", "mini", 2, 5, 40, 16, 103, "uniform"),
]


def main_fp16():
    """fp16 goldens (the notebook's literal torch_dtype, NB:882) in their own files, so that the fp32/bf16 fixtures
    above stay byte-identical: tests/golden/<case>_fp16.npz."""
    import tempfile

    out_dir = Path(__file__).resolve().parent
    for name, spec_name, wseed, B, S, T, iseed, lengths in CASES:
        spec = SPECS[spec_name]
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, iseed, lengths)
        with tempfile.TemporaryDirectory() as d:
            save_checkpoint(d, spec, seed=wseed)
            m = load_hf_model(d, dtype=torch.float16)
            assert m.encoder.block[0].layer[1].DenseReluDense.wo.weight.dtype == torch.float32
            toks = hf_generate(m, ids, mask, T)
            res = {"ids": ids, "mask": mask, "tokens_fp16": toks, "forced_fp16": hf_generate(m, ids, mask, T, min_new_tokens=T),
                   "logits_fp16": hf_teacher_forced_logits(m, ids, mask, toks[:, :-1]).astype(np.float32)}
            with torch.no_grad():
                enc = m.encoder(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask)).last_hidden_state
            res["enc_fp16"] = enc.float().numpy()
        res["meta"] = np.array([f"spec={spec_name} wseed={wseed} max_new={T} torch={torch.__version__} transformers={transformers.__version__} wo=fp32"])
        np.savez_compressed(out_dir / f"{name}_fp16.npz", **res)
        print(name + "_fp16", {k: v.shape for k, v in res.items() if k != "meta"})


def main():
    import tempfile

    out_dir = Path(__file__).resolve().parent
    torch.manual_seed(0)
    for name, spec_name, wseed, B, S, T, iseed, lengths in CASES:
        spec = SPECS[spec_name]
        ids, mask = synthetic_token_batch(B, S, spec.vocab_size, iseed, lengths)
        with tempfile.TemporaryDirectory() as d:
            save_checkpoint(d, spec, seed=wseed)
            res = {"ids": ids, "mask": mask}
            for tag, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
                m = load_hf_model(d, dtype=dtype)
                toks = hf_generate(m, ids, mask, T)
                forced = hf_generate(m, ids, mask, T, min_new_tokens=T)
                res[f"tokens_{tag}"] = toks
                res[f"forced_{tag}"] = forced
                res[f"logits_{tag}"] = hf_teacher_forced_logits(m, ids, mask, toks[:, :-1]).astype(np.float32)
                with torch.no_grad():
                    enc = m.encoder(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask)).last_hidden_state
                res[f"enc_{tag}"] = enc.float().numpy()
        res["meta"] = np.array([f"spec={spec_name} wseed={wseed} max_new={T} torch={torch.__version__} transformers={transformers.__version__}"])
        np.savez_compressed(out_dir / f"{name}.npz", **res)
        print(name, {k: v.shape for k, v in res.items() if k != "meta"})


def main_reference_predictor():
    """tests/golden/reference_predictor.npz; the inputs and calls are those of tests/test_reference_predictor_cpu.py."""
    import pandas as pd

    from anyscale_workshop_nyc_2023_b200 import rayshim, refsource
    from anyscale_workshop_nyc_2023_b200.preprocess import make_preprocess_function
    from anyscale_workshop_nyc_2023_b200.synth import synthetic_alpaca_rows
    from anyscale_workshop_nyc_2023_b200.workload import ASSETS, checkpoint_dir

    if refsource.reference_root() is None:
        raise SystemExit("set B200T5_REFERENCE_ROOT to a checkout of the reference")
    rayshim.install()
    from ray.data.preprocessors import BatchMapper
    from ray.train.batch_predictor import BatchPredictor
    from transformers import T5Tokenizer

    from anyscale_workshop_nyc_2023_b200.rayshim.train import HuggingFaceCheckpoint

    class HFOnCpu:  # model_cls: the dependency's own model on CPU, kwargs as the notebook passes them
        @staticmethod
        def from_pretrained(path, **kw):
            assert kw.get("torch_dtype") is torch.float16 and kw.get("device_map") == "auto"
            return load_hf_model(path, dtype=torch.float32, device="cpu")

    Ref = refsource.load_reference_predictor_module().HuggingFaceModelPredictor
    out = {}
    # flan-t5-batch-inference.py:119-138 with the unmodified class
    ckpt = checkpoint_dir("tiny", seed=1)
    ds = rayshim.data.from_huggingface(synthetic_alpaca_rows(11)).limit(10)
    fn = make_preprocess_function(str(ckpt), max_length=32, lean=False)
    checkpoint = HuggingFaceCheckpoint.from_directory(str(ckpt))
    checkpoint.set_preprocessor(BatchMapper(fn, batch_format="pandas", batch_size=4096))
    bp = BatchPredictor.from_checkpoint(checkpoint=checkpoint, predictor_cls=Ref, model_cls=HFOnCpu, tokenizer=T5Tokenizer,
                                        use_gpu=False, device_map="auto", torch_dtype=torch.float16)
    pred = bp.predict(ds, num_gpus_per_worker=0, batch_size=4, max_new_tokens=7).to_pandas()
    out["flow_generated_output"] = np.array(pred["generated_output"].tolist(), dtype=str)
    # _predict_numpy on the four argument patterns of the hot path
    model = load_hf_model(ckpt)
    tok = T5Tokenizer.from_pretrained(str(ckpt))
    ids, mask = synthetic_token_batch(6, 20, SPECS["tiny"].vocab_size, seed=17, lengths="uniform")
    cases = [
        ({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()}, dict(max_new_tokens=6)),
        ({"input_ids": ids, "attention_mask": mask, "labels": ids.copy(), "junk": ids}, dict(feature_columns=["input_ids", "attention_mask"], max_new_tokens=4)),
        ({"input_ids": ids, "attention_mask": mask}, dict()),
        ({"input_ids": ids, "attention_mask": mask}, dict(max_new_tokens=5, min_new_tokens=5)),
    ]
    ref = Ref(model, tokenizer=tok)
    for i, (data, kw) in enumerate(cases):
        df = ref._predict_numpy({k: v.copy() for k, v in data.items()}, **kw)
        out[f"predict_case{i}"] = np.array(df["generated_output"].tolist(), dtype=str)
    # utils.py:6-33 with its hub tokenizer download pointed at the local tokenizer files
    utils = refsource.load_reference_utils_module()
    real = T5Tokenizer.from_pretrained
    utils.T5Tokenizer.from_pretrained = classmethod(lambda cls, name, *a, **k: real(str(ASSETS / "tokenizer"), *a, **k))
    batch = pd.DataFrame(synthetic_alpaca_rows(40, seed=5))[["instruction", "input"]]
    for k, v in utils.preprocess_function(batch).items():
        out[f"preprocess_{k}"] = np.asarray(v)
    np.savez_compressed(Path(__file__).resolve().parent / "reference_predictor.npz", **out)
    print("reference_predictor", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    if "--reference-predictor" in sys.argv:
        main_reference_predictor()
    elif "--fp16" in sys.argv:
        main_fp16()
    else:
        main()
        main_fp16()
