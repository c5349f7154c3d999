"""The step graph's cache across every kind of call. The graph bakes in what a call's steps run (StepMode in
csrc/b200t5.cu); a call on the same plan replays it or re-captures it. One handle runs each kind of call on one
(B, S, T) plan, then the same calls in reverse order, so every call follows a different predecessor the second time.
Each must give the bits, kernel launches and decode steps of its first run."""
import numpy as np
import pytest
import torch

from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration
from anyscale_workshop_nyc_2023_b200.synth import SPECS, save_checkpoint, synthetic_token_batch

pytestmark = pytest.mark.gpu


def test_every_call_kind_repeats_its_results_after_any_other(tmp_path):
    spec = SPECS["tiny"]
    save_checkpoint(tmp_path, spec, seed=1)
    model = B200T5ForConditionalGeneration.from_pretrained(tmp_path, device_map="auto", torch_dtype=torch.bfloat16)
    B, S, T = 8, 24, 12
    ids, mask = synthetic_token_batch(B, S, spec.vocab_size, seed=101, lengths="uniform")
    rng = np.random.default_rng(102)
    labels = rng.integers(2, spec.vocab_size, size=(B, T))
    labels[::2, T - 3:] = -100  # every other row's labels end early
    dec = rng.integers(2, spec.vocab_size, size=(B, T))
    a = dict(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), max_new_tokens=T)

    def arrays(*ts):
        return [t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t) for t in ts]

    def scored():
        o = model.generate(**a, return_dict_in_generate=True, output_scores=True)
        return arrays(o.sequences, o.scores.token_logprobs, o.scores.token_logits)

    calls = {
        "generate": lambda: arrays(model.generate(**a)),
        "processors": lambda: arrays(model.generate(**a, repetition_penalty=1.3)),
        "scores": scored,
        "score": lambda: (lambda r: arrays(r.token_logprobs, r.lengths))(model.score(a["input_ids"], a["attention_mask"], labels)),
        "pool": lambda: arrays(*model.generate_stream(ids, mask, pool=B, max_new_tokens=T)),
        "host": lambda: arrays(*model.generate_host(ids, mask, max_new_tokens=T)),
        "decode_logits": lambda: arrays(model.decode_logits(ids, mask, dec)),
        "beam": lambda: arrays(model.generate(**a, num_beams=2)),  # a plan of B * 2 rows, then back to B rows
    }
    order = ["generate", "processors", "scores", "score", "pool", "host", "decode_logits", "beam", "generate"]
    first = {}
    for name in order + order[::-1]:
        got = calls[name]()
        st = None
        if name != "decode_logits":  # (not a generate call: no statistics of its own)
            s = model.stats()
            st = {k: s[k] for k in ("kernel_launches", "decode_steps", "xattn_kernel")}
        if name not in first:
            first[name] = (got, st)
            continue
        want, want_st = first[name]
        assert [(x.dtype, x.shape) for x in got] == [(x.dtype, x.shape) for x in want], name
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got, want)), name
        assert st == want_st, (name, st, want_st)
