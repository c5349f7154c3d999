"""Host-side mirror of the reference's plug-in: `HuggingFaceModelPredictor`.

Interface source: NLP_workloads/Anyscale_job/predictor.py:14-106 (identical copy in the notebook,
Model_finetuning_and_batch_inference.ipynb:760-852). Names, argument meaning and error behaviour
are kept so the notebook cells run unchanged; the body is written for the CUDA path:

  * columns are staged through pinned host memory (one set of buffers per calling thread) and copied with
    non-blocking H2D copies; a batch larger than the model's pool of decode slots is handed over in HOST memory
    (the slot pool admits prompts from host buffers as slots free up: no copy to the device and back);
    `labels` - which the reference's preprocessor emits as a copy of `input_ids`
    (JOB/utils.py:31) and `generate` ignores - is not shipped to the device;
  * works with any `model` exposing `.device` and `.generate(**kw) -> LongTensor[B, 1+T]`
    (B200T5ForConditionalGeneration, or transformers' own model for the CPU baseline).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import threading

import numpy as np
import pandas as pd
import torch

try:  # real Ray if present, otherwise the in-repo shim (Ray cannot be installed offline)
    from ray.train.predictor import Predictor
except Exception:  # pragma: no cover - exercised when ray is absent
    from .rayshim.train import Predictor

_NOT_MODEL_INPUTS = ("labels",)


class HuggingFaceModelPredictor(Predictor):
    """Ray AIR predictor that turns tokenised prompts into generated text.

    Args mirror the reference: `model` (anything with `.generate`), `tokenizer` (for
    `batch_decode`), `preprocessor` (AIR preprocessor applied by `Predictor.predict`), `use_gpu`.
    """

    def __init__(self, model: Any, tokenizer: Optional[Any] = None, preprocessor: Optional[Any] = None,
                 use_gpu: bool = False) -> None:
        super().__init__(preprocessor)
        self.model = model
        self.tokenizer = tokenizer
        self.use_gpu = use_gpu
        self._pinned: Dict[Any, torch.Tensor] = {}

    @classmethod
    def from_checkpoint(cls, checkpoint: Any, model_cls: Any, *, tokenizer: Optional[Any] = None,
                        use_gpu: bool = False, **get_model_kwargs: Any) -> "HuggingFaceModelPredictor":
        """`checkpoint` needs get_model / get_tokenizer / get_preprocessor (AIR HuggingFaceCheckpoint
        duck type). A tokenizer *class* is resolved through the checkpoint; an instance is used as is;
        None falls back to AutoTokenizer like the reference."""
        if not tokenizer:
            from transformers import AutoTokenizer

            tokenizer = AutoTokenizer
        if isinstance(tokenizer, type):
            tokenizer = checkpoint.get_tokenizer(tokenizer)
        model = checkpoint.get_model(model_cls, **get_model_kwargs)
        return cls(model, tokenizer=tokenizer, preprocessor=checkpoint.get_preprocessor(), use_gpu=use_gpu)

    def _to_device(self, name: str, arr: np.ndarray) -> torch.Tensor:
        device = torch.device(self.model.device)
        t = torch.from_numpy(np.ascontiguousarray(arr))
        if device.type != "cuda":
            return t.to(device)
        key = (name, threading.get_ident())  # two scoring threads may alternate on one predictor (rayshim/train.py)
        buf = self._pinned.get(key)
        if buf is None or buf.shape != t.shape or buf.dtype != t.dtype:
            buf = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            self._pinned[key] = buf
        buf.copy_(t)
        return buf.to(device, non_blocking=True)

    def _predict_numpy(self, data: Dict[str, Any], feature_columns: Optional[List[str]] = None,
                       **generate_kwargs: Any) -> pd.DataFrame:
        """`data`: dict of already-tokenised columns (input_ids, attention_mask[, labels]) as numpy
        arrays [B, S]; returns a DataFrame with the single column "generated_output"."""
        if isinstance(data, np.ndarray):
            data = {"input_ids": data}
        if feature_columns:
            data = {k: v for k, v in data.items() if k in feature_columns}
        on_gpu = torch.device(self.model.device).type == "cuda"
        first = next(iter(data.values()), None)
        host_ok = getattr(self.model, "takes_host_batches", None)
        if on_gpu and host_ok is not None and getattr(first, "ndim", 0) == 2 and host_ok(first.shape[0], first.shape[1]):
            tensors = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in data.items() if k not in _NOT_MODEL_INPUTS}
        else:
            tensors = {k: self._to_device(k, v) for k, v in data.items() if not (on_gpu and k in _NOT_MODEL_INPUTS)}
        outputs = self.model.generate(**{**tensors, **generate_kwargs})
        texts = self.tokenizer.batch_decode(outputs, skip_special_tokens=True)
        return pd.DataFrame(texts, columns=["generated_output"])
