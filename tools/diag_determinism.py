"""Diagnostic: run-to-run determinism and static-vs-pool identity of natural-EOS generation at the bench shape, per
cross-attention kernel / option set (one process, b200t5_set_option)."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration  # noqa: E402
from anyscale_workshop_nyc_2023_b200.synth import SPECS, synthetic_token_batch  # noqa: E402
from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir  # noqa: E402

m = B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir("flan-t5-base", 0))
ids, mask = synthetic_token_batch(512, 512, 32128, seed=3, lengths="full")
T = 128


def static(n=256):
    outs = []
    for lo in range(0, ids.shape[0], n):
        o, ln = m.generate_host(ids[lo:lo + n], mask[lo:lo + n], max_new_tokens=T)
        outs.append(np.pad(o, ((0, 0), (0, T + 1 - o.shape[1]))))
    return np.concatenate(outs)


ref = None
CONFIGS = sys.argv[1].split(";") if len(sys.argv) > 1 else ("xattn=0", "xattn=1", "xattn=1,chains=1", "xattn=1,pdl=0", "xattn=1,xattn_stages=2")
for opts in CONFIGS:
    for k in ("xattn=0", "chains=0", "pdl=1", "xattn_stages=5", "sk_stages64=0", "sk_stages128=0"):
        a, b = k.split("=")
        m.set_option(a, int(b))
    for kv in opts.split(","):
        a, b = kv.split("=")
        m.set_option(a, int(b))
    before = [m.generate_host(ids[:256], mask[:256], max_new_tokens=32, min_new_tokens=32)[0] for _ in range(3)]
    print(f"{opts:32s} forced-32 BEFORE any natural-EOS run: rows differing {[int((before[0] != f).any(1).sum()) for f in before[1:]]}", flush=True)
    runs = [static() for _ in range(3)] if "--forced-only" not in sys.argv else [np.zeros((1, 1)), np.zeros((1, 1))]
    forced = []
    for _ in range(4):
        o, _ln = m.generate_host(ids[:256], mask[:256], max_new_tokens=32, min_new_tokens=32)
        forced.append(o)
    same = [bool((runs[0] == r).all()) for r in runs[1:]]
    rows_diff = int((runs[0] != runs[1]).any(1).sum())
    if "--forced-only" in sys.argv:
        pool = runs[0]
    else:
        pool, _ = m.generate_stream(ids, mask, pool=256, max_new_tokens=T)
        pool = np.pad(pool, ((0, 0), (0, T + 1 - pool.shape[1])))
    print(f"{opts:32s} static runs identical: {same} (rows differing run0/run1: {rows_diff}); pool == static: {bool((pool == runs[0]).all())} "
          f"(rows differing: {int((pool != runs[0]).any(1).sum())}); tokens {int((runs[0] != 0).sum())}; forced-32 identical: {[bool((forced[0] == f).all()) for f in forced[1:]]} (rows differing {[int((forced[0] != f).any(1).sum()) for f in forced[1:]]})", flush=True)
    if ref is None:
        ref = runs[0]
