"""Synthetic workload assembly shared by bench.py, __graft_entry__.smoke() and the tests:
a FLAN-T5-shaped checkpoint directory (weights + tokenizer files, i.e. what the reference's
`result.checkpoint` directory contains) and the BatchPredictor wired to the CUDA model class."""
from __future__ import annotations

import os
import shutil
import tempfile
from pathlib import Path
from typing import Optional

from .synth import SPECS, save_checkpoint

ASSETS = Path(__file__).resolve().parent / "assets"


def checkpoint_dir(spec_name: str, seed: int = 0, root: Optional[str] = None) -> Path:
    """Create (once) and return a synthetic checkpoint directory for `spec_name`. The directory name carries the user
    id: in a shared temporary directory another user's (private) checkpoint is neither readable nor replaceable."""
    root = Path(root or os.environ.get("B200T5_CKPT_ROOT", tempfile.gettempdir()))
    d = root / f"b200t5_ckpt_{spec_name}_seed{seed}_q{SPECS[spec_name].q_init_gain:g}_u{os.getuid()}"
    marker = d / ".complete"
    if not marker.exists():
        tmp = Path(tempfile.mkdtemp(prefix=d.name + ".", dir=root))
        save_checkpoint(tmp, SPECS[spec_name], seed=seed)
        for f in (ASSETS / "tokenizer").iterdir():
            shutil.copy(f, tmp / f.name)
        (tmp / ".complete").write_text("ok")
        try:
            os.replace(tmp, d)
        except OSError:  # another process won the race
            shutil.rmtree(tmp, ignore_errors=True)
    return d


def make_batch_predictor(ckpt: Path, model_cls=None, preprocessor=None, **model_kwargs):
    """`BatchPredictor.from_checkpoint(...)` exactly as notebook :875-883 calls it, with
    `model_cls` defaulting to the CUDA class."""
    from transformers import T5Tokenizer

    from .predictor import HuggingFaceModelPredictor
    from .rayshim.train import BatchPredictor, HuggingFaceCheckpoint

    if model_cls is None:
        from .modeling import B200T5ForConditionalGeneration as model_cls
    checkpoint = HuggingFaceCheckpoint.from_directory(str(ckpt))
    if preprocessor is not None:
        checkpoint.set_preprocessor(preprocessor)
    return BatchPredictor.from_checkpoint(checkpoint=checkpoint, predictor_cls=HuggingFaceModelPredictor,
                                          model_cls=model_cls, tokenizer=T5Tokenizer, **model_kwargs)
