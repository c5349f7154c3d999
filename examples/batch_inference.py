"""The workshop's batch-inference cells (NLP_workloads/Text_generation/Model_finetuning_and_batch_inference.ipynb,
cells at :260-296 preprocess, :875-883 BatchPredictor.from_checkpoint, :908-913 predict, :934 join) as one script,
with the ONE edit the drop-in asks for: `model_cls`.

    python examples/batch_inference.py --model-cls b200            # H100 path (needs an H100)
    python examples/batch_inference.py --model-cls hf --n 8        # the dependency's own model on CPU (reference path)

Ray is not installable offline, so `import ray` resolves to the in-repo shim (rayshim.install()), which serves exactly
the calls these cells make. Checkpoints are synthetic (seeded random weights of the FLAN-T5 architecture).
"""
import argparse
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from anyscale_workshop_nyc_2023_b200 import rayshim  # noqa: E402

rayshim.install()

import ray  # noqa: E402
from ray.data.preprocessors import BatchMapper  # noqa: E402
from ray.train.batch_predictor import BatchPredictor  # noqa: E402
from ray.train.huggingface import HuggingFaceCheckpoint  # noqa: E402
from transformers import T5Tokenizer  # noqa: E402

from anyscale_workshop_nyc_2023_b200.predictor import HuggingFaceModelPredictor  # noqa: E402
from anyscale_workshop_nyc_2023_b200.preprocess import make_preprocess_function  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import synthetic_alpaca_rows  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402


class HFModelOnCpu:
    """`model_cls` of the reference path: transformers' T5ForConditionalGeneration (untied head, see oracle/hf_anchor.py)."""

    @staticmethod
    def from_pretrained(path, **kw):
        from oracle.hf_anchor import load_hf_model  # the example's CPU leg only; the CUDA path never imports oracle/

        return load_hf_model(path, dtype=torch.float32, device="cpu")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-cls", default="b200", choices=["b200", "hf"])
    ap.add_argument("--model", default=None, help="flan-t5-small | flan-t5-base | flan-t5-large | tiny (default: base on H100, tiny on CPU)")
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--batch-size", type=int, default=4096, help="rows handed to the predictor at once; > 256 uses the slot pool")
    ap.add_argument("--max-new-tokens", type=int, default=128)
    ap.add_argument("--torch-dtype", default="bfloat16", choices=["bfloat16", "float16"])
    a = ap.parse_args()
    on_gpu = a.model_cls == "b200"
    model_name = a.model or ("flan-t5-base" if on_gpu else "tiny")
    ckpt_dir = checkpoint_dir(model_name, seed=0)

    ray.init()
    ds = ray.data.from_huggingface(synthetic_alpaca_rows(a.n))                       # NB: load_dataset(...) -> from_huggingface
    batch_mapper = BatchMapper(make_preprocess_function(str(ckpt_dir)), batch_format="pandas")  # NB:296
    checkpoint = HuggingFaceCheckpoint.from_directory(str(ckpt_dir))
    checkpoint.set_preprocessor(batch_mapper)
    if on_gpu:
        from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration as model_cls
    else:
        model_cls = HFModelOnCpu
    predictor = BatchPredictor.from_checkpoint(                                        # NB:875-883
        checkpoint=checkpoint, predictor_cls=HuggingFaceModelPredictor, model_cls=model_cls, tokenizer=T5Tokenizer,
        use_gpu=on_gpu, device_map="auto", torch_dtype=getattr(torch, a.torch_dtype))
    t0 = time.perf_counter()
    prediction = predictor.predict(ds, num_gpus_per_worker=int(on_gpu), batch_size=a.batch_size,  # NB:908-913
                                   max_new_tokens=a.max_new_tokens)
    dt = time.perf_counter() - t0
    input_data_pd = ds.to_pandas()
    prediction_pd = prediction.to_pandas()
    joined = input_data_pd.join(prediction_pd, how="inner")                            # NB:934
    print(joined[["instruction", "generated_output"]].head(3).to_string(max_colwidth=60))
    print(f"{len(joined)} prompts in {dt:.2f} s ({len(joined) / dt:.1f} prompts/s) with model_cls={model_cls.__name__}")
    ray.shutdown()


if __name__ == "__main__":
    main()
