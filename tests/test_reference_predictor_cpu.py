"""CPU-only: this package's mirror of the reference's hot-path file against what the reference's OWN code returned.

`NLP_workloads/Anyscale_job/predictor.py:14-106` (HuggingFaceModelPredictor) and `utils.py:6-33`
(preprocess_function), unmodified and driven through the shim, were run once on the inputs below; their outputs are
stored in tests/golden/reference_predictor.npz (strings and token arrays, nothing of the reference's code). The
equalities pinned here and on the GPU:

    reference predictor + HF model  ==  direct HF generate                    (golden, here)
    reference predictor             ==  this package's mirror, same model      (golden, here)
    mirror + CUDA model             ==  CUDA generate == HF on the same GPU    (tests/test_model_gpu.py)

Flow reproduced: flan-t5-batch-inference.py:119-138 (from_checkpoint -> predict -> to_pandas -> join).
"""
from pathlib import Path

import numpy as np
import pandas as pd
import pytest
import torch

from anyscale_workshop_nyc_2023_b200 import rayshim
from anyscale_workshop_nyc_2023_b200.preprocess import make_preprocess_function
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_alpaca_rows, synthetic_token_batch
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir

GOLDEN = np.load(Path(__file__).resolve().parent / "golden" / "reference_predictor.npz")


class HFOnCpu:
    """model_cls stand-in with from_pretrained(dir, **kw): the dependency's own model on CPU (what
    `T5ForConditionalGeneration` is in the reference script, minus the hub download)."""

    @staticmethod
    def from_pretrained(path, **kw):
        from oracle.hf_anchor import load_hf_model

        assert kw.get("torch_dtype") is torch.float16 and kw.get("device_map") == "auto"  # forwarded untouched (NB:881-882)
        return load_hf_model(path, dtype=torch.float32, device="cpu")


def test_reference_script_flow_matches_the_reference_class_output():
    """BatchPredictor.from_checkpoint(checkpoint=..., predictor_cls=<predictor class>, model_cls=..., tokenizer=T5Tokenizer,
    use_gpu=..., device_map="auto", torch_dtype=torch.float16) -> predict(ds, num_gpus_per_worker=..., batch_size=...,
    max_new_tokens=...) -> to_pandas -> join, as flan-t5-batch-inference.py:119-138: the mirror class returns what the
    reference's unmodified class returned in this flow (golden), which is what the dependency generates directly."""
    rayshim.install()  # `import ray` resolves to the shim, as for the reference script
    from ray.data.preprocessors import BatchMapper
    from ray.train.batch_predictor import BatchPredictor
    from transformers import T5Tokenizer

    from anyscale_workshop_nyc_2023_b200.rayshim.train import HuggingFaceCheckpoint
    from oracle.hf_anchor import hf_generate, load_hf_model

    from anyscale_workshop_nyc_2023_b200.predictor import HuggingFaceModelPredictor as Mirror

    ckpt = checkpoint_dir("tiny", seed=1)
    use_gpu = False
    validation_dataset = rayshim.data.from_huggingface(synthetic_alpaca_rows(11)).limit(10)
    fn = make_preprocess_function(str(ckpt), max_length=32, lean=False)  # the reference's own tokenizer call
    checkpoint = HuggingFaceCheckpoint.from_directory(str(ckpt))
    checkpoint.set_preprocessor(BatchMapper(fn, batch_format="pandas", batch_size=4096))
    predictor = BatchPredictor.from_checkpoint(checkpoint=checkpoint, predictor_cls=Mirror, model_cls=HFOnCpu,
                                               tokenizer=T5Tokenizer, use_gpu=use_gpu, device_map="auto", torch_dtype=torch.float16)
    prediction = predictor.predict(validation_dataset, num_gpus_per_worker=int(use_gpu), batch_size=4, max_new_tokens=7)
    input_data_pd = validation_dataset.to_pandas()
    prediction_pd = prediction.to_pandas()
    outputs = input_data_pd.join(prediction_pd, how="inner").head(n=7)
    assert len(outputs) == 7 and "generated_output" in outputs.columns and "instruction" in outputs.columns
    # row for row what the dependency generates directly for the same tokenised prompts
    enc = fn(input_data_pd)
    model = load_hf_model(ckpt)
    tok = T5Tokenizer.from_pretrained(str(ckpt))
    want = []
    for lo in range(0, 10, 4):
        want += tok.batch_decode(hf_generate(model, enc["input_ids"][lo:lo + 4], enc["attention_mask"][lo:lo + 4], 7), skip_special_tokens=True)
    assert prediction_pd["generated_output"].tolist() == want
    assert GOLDEN["flow_generated_output"].tolist() == want


def test_mirror_predictor_equals_the_reference_predictor():
    """Same model, same inputs, same kwargs through both classes: identical DataFrames - for the dict-of-columns input
    of the hot path, with `labels` present (JOB/utils.py:31), with feature_columns, and for max_length-default calls."""
    from transformers import T5Tokenizer

    from anyscale_workshop_nyc_2023_b200.predictor import HuggingFaceModelPredictor as Mirror
    from oracle.hf_anchor import load_hf_model

    ckpt = checkpoint_dir("tiny", seed=1)
    model = load_hf_model(ckpt)
    tok = T5Tokenizer.from_pretrained(str(ckpt))
    ids, mask = synthetic_token_batch(6, 20, SPECS["tiny"].vocab_size, seed=17, lengths="uniform")
    mir = Mirror(model, tokenizer=tok)
    cases = [
        ({"input_ids": ids, "attention_mask": mask, "labels": ids.copy()}, dict(max_new_tokens=6)),
        ({"input_ids": ids, "attention_mask": mask, "labels": ids.copy(), "junk": ids}, dict(feature_columns=["input_ids", "attention_mask"], max_new_tokens=4)),
        ({"input_ids": ids, "attention_mask": mask}, dict()),  # GenerationConfig default max_length = 20
        ({"input_ids": ids, "attention_mask": mask}, dict(max_new_tokens=5, min_new_tokens=5)),
    ]
    for i, (data, kw) in enumerate(cases):
        b = mir._predict_numpy({k: v.copy() for k, v in data.items()}, **kw)
        assert list(b.columns) == ["generated_output"]
        assert GOLDEN[f"predict_case{i}"].tolist() == b["generated_output"].tolist()
    # the classmethod: same constructor contract (tokenizer class resolved through the checkpoint)
    from anyscale_workshop_nyc_2023_b200.rayshim.train import HuggingFaceCheckpoint

    ck = HuggingFaceCheckpoint.from_directory(str(ckpt))
    for cls in (Mirror,):
        p = cls.from_checkpoint(ck, HFOnCpu, tokenizer=T5Tokenizer, use_gpu=False, device_map="auto", torch_dtype=torch.float16)
        assert p.use_gpu is False and p.tokenizer.__class__.__name__ == "T5Tokenizer" and p.get_preprocessor() is None


def test_reference_preprocess_function_equals_the_mirror():
    """utils.py:6-33 hard-codes `T5Tokenizer.from_pretrained("google/flan-t5-base")` (a hub download); with that one
    call pointed at the local tokenizer files the unmodified function produced the golden arrays, and this package's
    lean mirror produces identical ones."""
    from anyscale_workshop_nyc_2023_b200.workload import ASSETS

    batch = pd.DataFrame(synthetic_alpaca_rows(40, seed=5))[["instruction", "input"]]
    mir = make_preprocess_function(str(ASSETS / "tokenizer"))(batch)
    assert set(mir) == {"input_ids", "attention_mask", "labels"}
    for k in mir:
        assert np.array_equal(GOLDEN[f"preprocess_{k}"], mir[k]), k
