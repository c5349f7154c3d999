"""Loading the reference's OWN hot-path sources, unmodified, when its checkout is present.

`NLP_workloads/Anyscale_job/predictor.py` (HuggingFaceModelPredictor, :14-106) and `utils.py`
(preprocess_function, :6-33) are plain Python whose only obstacle offline is `import ray` at module top
(predictor.py:7). With the shim registered under the name `ray` (rayshim.install()) they import as they are,
straight from a reference checkout - nothing is copied into this repository. A checkout is used only where
$B200T5_REFERENCE_ROOT names one, so callers must handle `None`:

  * bench.py's CPU arm uses it when available (`cpu_baseline.kind == "reference"`), the mirror otherwise ("port").
"""
from __future__ import annotations

import importlib.util
import os
import sys
from pathlib import Path
from types import ModuleType
from typing import Optional

_JOB_DIR = Path("NLP_workloads") / "Anyscale_job"


def reference_root() -> Optional[Path]:
    env = os.environ.get("B200T5_REFERENCE_ROOT")
    if not env:
        return None
    root = Path(env)
    try:
        return root if (root / _JOB_DIR / "predictor.py").is_file() else None
    except OSError:  # not readable by this user
        return None


def _load(path: Path, name: str) -> ModuleType:
    from . import rayshim

    rayshim.install()
    spec = importlib.util.spec_from_file_location(name, str(path))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)  # the file itself, unmodified
    return mod


def load_reference_predictor_module() -> Optional[ModuleType]:
    """The reference's predictor.py as a module (its `HuggingFaceModelPredictor` is the class the notebook passes as
    `predictor_cls`), or None when the checkout is absent."""
    root = reference_root()
    if root is None:
        return None
    name = "_reference_anyscale_job_predictor"
    return sys.modules.get(name) or _load(root / _JOB_DIR / "predictor.py", name)


def load_reference_utils_module() -> Optional[ModuleType]:
    root = reference_root()
    if root is None:
        return None
    name = "_reference_anyscale_job_utils"
    return sys.modules.get(name) or _load(root / _JOB_DIR / "utils.py", name)
