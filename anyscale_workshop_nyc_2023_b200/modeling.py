"""`B200T5ForConditionalGeneration`: the object the reference predictor holds as ``self.model``.

The reference's seam is duck-typed (NLP_workloads/Anyscale_job/predictor.py):
    checkpoint.get_model(model_cls, **get_model_kwargs)   :68   -> model_cls.from_pretrained(dir, **kw)
    self.model.device                                      :98
    self.model.generate(**generate_kwargs) -> LongTensor   :102  (consumed by tokenizer.batch_decode :104)
so passing ``model_cls=B200T5ForConditionalGeneration`` to ``BatchPredictor.from_checkpoint``
(notebook lines 875-883) swaps the Hugging Face eager model for the sm_90a kernels behind
libb200t5.so without touching the predictor.

PyTorch is used for device memory and streams only; all arithmetic runs in the CUDA library.
There is no CPU path: constructing the model without an H100 raises.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import threading
import warnings
from pathlib import Path
from types import SimpleNamespace
from typing import Any, Dict, Optional

import numpy as np
import torch

from . import _lib
from .synth import read_safetensors

_POOL_MAX_S = 512  # the slot pool admits prompts through the packed encoder (csrc: kEncPackMaxS)
_HF_DEFAULT_MAX_LENGTH = 20  # GenerationConfig default the notebook's single-prompt cell relies on (NB:577)

_IGNORED_WEIGHTS = ("decoder.block.0.layer.1.EncDecAttention.relative_attention_bias.weight",)
_ALIASES = ("encoder.embed_tokens.weight", "decoder.embed_tokens.weight")


# transformers' greedy-mode logits processors the CUDA path applies (b200t5_logits_params, csrc/logits_process.cuh)
LOGITS_PROCESSOR_KWARGS = ("repetition_penalty", "encoder_repetition_penalty", "no_repeat_ngram_size",
                           "encoder_no_repeat_ngram_size", "bad_words_ids", "suppress_tokens", "begin_suppress_tokens")


class _LogitsArgs:
    """A validated set of logits processors: the C struct plus the arrays its pointers refer to."""

    def __init__(self, params: _lib.LogitsParams, arrays, eos_ids):
        self.params = params
        self._arrays = arrays  # keeps the buffers the struct points to alive
        self.eos_ids = eos_ids

    def ref(self):
        return C.byref(self.params)


def _eos_ids(eos_token_id):
    """eos_token_id as a list without repeats (None stays None)."""
    if eos_token_id is None:
        return None
    if isinstance(eos_token_id, torch.Tensor):
        eos_token_id = eos_token_id.tolist()
    if isinstance(eos_token_id, (list, tuple)):
        if not eos_token_id:
            raise ValueError("eos_token_id must not be an empty list")
        return list(dict.fromkeys(int(e) for e in eos_token_id))
    return [int(eos_token_id)]


def _id_list(name, v, vocab_size):
    ids = [int(t) for t in (v.tolist() if isinstance(v, torch.Tensor) else v)]
    bad = [t for t in ids if t < 0 or t >= vocab_size]
    if bad:
        raise ValueError(f"`{name}` contains ids outside [0, {vocab_size}): {bad}")
    return ids


def logits_processor_args(kw: Dict[str, Any], eos_ids, default_eos: int, vocab_size: int) -> Optional[_LogitsArgs]:
    """Validate the processor kwargs of a generate call as transformers does (ValueError where its processors raise)
    and build b200t5_logits_params. Returns None when nothing would change greedy decoding: no-op values
    (repetition_penalty=1.0, no_repeat_ngram_size=0, suppress_tokens=[], ...) count as absent, as in transformers."""
    p = _lib.LogitsParams(repetition_penalty=1.0, encoder_repetition_penalty=1.0)
    arrays = []
    active = False

    def arr(ids):
        a = np.ascontiguousarray(ids, dtype=np.int32)
        arrays.append(a)
        return a.ctypes.data_as(C.c_void_p)

    for name in ("repetition_penalty", "encoder_repetition_penalty"):
        v = kw.get(name)
        if v is None:
            continue
        v = float(v)
        if not v > 0:
            raise ValueError(f"`{name}` has to be a strictly positive float, but is {v}")
        setattr(p, name, v)
        active = active or v != 1.0
    for name in ("no_repeat_ngram_size", "encoder_no_repeat_ngram_size"):
        v = kw.get(name)
        if v is None:
            continue
        if isinstance(v, bool) or int(v) != v or v < 0:
            raise ValueError(f"`{name}` has to be a non-negative integer, but is {v}")
        setattr(p, name, int(v))
        active = active or int(v) > 0
    for name, ptr, cnt in (("suppress_tokens", "suppress_tokens", "n_suppress_tokens"),
                           ("begin_suppress_tokens", "begin_suppress_tokens", "n_begin_suppress_tokens")):
        v = kw.get(name)
        if v is None:
            continue
        ids = _id_list(name, v, vocab_size)
        if ids:
            setattr(p, ptr, arr(ids))
            setattr(p, cnt, len(ids))
            active = True
    eos_list = eos_ids if eos_ids else [default_eos]
    bw = kw.get("bad_words_ids")
    if bw is not None:
        if not isinstance(bw, (list, tuple)) or len(bw) == 0:
            raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bw}.")
        if any(not isinstance(w, (list, tuple)) for w in bw):
            raise ValueError(f"`bad_words_ids` has to be a list of lists, but is {bw}.")
        seqs = []
        for w in bw:
            ids = _id_list("bad_words_ids", w, vocab_size)
            if not ids:
                raise ValueError(f"`bad_words_ids` contains an empty sequence: {bw}")
            if len(ids) == 1 and ids[0] in eos_list:
                continue  # transformers drops [eos] (NoBadWordsLogitsProcessor)
            seqs.append(ids)
        if not seqs:  # transformers: the remaining sequence bias must not be empty
            raise ValueError(f"`bad_words_ids` bans nothing but the EOS token: {bw}")
        off = np.cumsum([0] + [len(w) for w in seqs])
        p.bad_words_ids = arr([t for w in seqs for t in w])
        p.bad_words_offsets = arr(off)
        p.n_bad_words = len(seqs)
        active = True
    if eos_ids is not None and len(eos_ids) > 1:
        if len(eos_ids) > 16:
            raise ValueError("at most 16 eos_token_id values are supported")
        p.eos_token_ids = arr(eos_ids)
        p.n_eos_token_ids = len(eos_ids)
        active = True
    return _LogitsArgs(p, arrays, eos_list) if active else None


class TokenScores:
    """What `generate(..., output_scores=True)` returns as `.scores`: per generated position, the chosen token's
    processed score (`token_logits`) and its log-softmax (`token_logprobs`), fp32 [B, T'], 0 after a row's EOS.
    NOT transformers' tuple of T' tensors [B, vocab]: the fused lm_head epilogue never writes the vocabulary-wide
    scores. `compute_transition_scores` accepts it in place of that tuple."""

    def __init__(self, token_logprobs, token_logits):
        self.token_logprobs = token_logprobs
        self.token_logits = token_logits

    def __len__(self):
        return int(self.token_logprobs.shape[1])


class GenerateOutput:
    """`generate(..., return_dict_in_generate=True)`: `.sequences` is the tensor a plain call returns, `.scores` a
    TokenScores (None without output_scores=True), `.token_logprobs` a shortcut to scores.token_logprobs."""

    def __init__(self, sequences, scores: Optional[TokenScores] = None):
        self.sequences = sequences
        self.scores = scores
        self.token_logprobs = None if scores is None else scores.token_logprobs

    def __getitem__(self, key):
        return getattr(self, key)


def generate_output_flags(kw: Dict[str, Any]):
    """(return_dict_in_generate, output_scores) of a generate call. The outputs the CUDA path cannot give raise
    instead of being dropped."""
    for k in ("output_logits", "output_attentions", "output_hidden_states"):
        if kw.get(k):
            raise NotImplementedError(f"generate({k}=True) is not supported by the CUDA path")
    return bool(kw.get("return_dict_in_generate")), bool(kw.get("output_scores"))


def score_labels(labels, vocab_size: int) -> np.ndarray:
    """Validate `labels` of score() as int64 [B, L]: ids in [0, vocab_size) or -100, every row with at least one
    label, -100 only after a row's last label (teacher forcing stops there)."""
    if labels is None:
        raise ValueError("labels is required")
    lab = np.ascontiguousarray(labels.detach().cpu().numpy() if isinstance(labels, torch.Tensor) else labels)
    if lab.ndim != 2 or lab.shape[1] < 1 or lab.dtype.kind not in "iu":
        raise ValueError(f"labels must be integers [batch, length >= 1], got {lab.dtype} {lab.shape}")
    lab = lab.astype(np.int64)
    ignored = lab == -100
    if ((lab < 0) & ~ignored).any() or (lab >= vocab_size).any():
        raise ValueError(f"labels contain ids outside [0, {vocab_size}) other than -100")
    if ignored[:, 0].any():
        raise ValueError("every row of labels needs at least one label")
    if (ignored[:, :-1] & ~ignored[:, 1:]).any():
        raise ValueError("labels: -100 may only follow a row's last label")
    return lab


def _chk(model, rc: int, handle=None) -> None:
    _lib.check(rc, handle, model._lib)


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class B200T5ForConditionalGeneration:
    """FLAN-T5 greedy generation on one H100. API subset of transformers.T5ForConditionalGeneration
    that the workshop's predictor and notebook cells touch."""

    main_input_name = "input_ids"

    def __init__(self, config: Dict[str, Any], device: torch.device, compute_dtype: torch.dtype = torch.bfloat16):
        if device.type != "cuda":
            raise RuntimeError("B200T5ForConditionalGeneration runs on an H100 only; there is no CPU fallback")
        if compute_dtype not in (torch.bfloat16, torch.float16):
            raise ValueError(f"compute dtype must be bfloat16 or float16, got {compute_dtype}")
        # one shared library per numerics contract: bf16 everywhere, or the notebook's literal torch_dtype=float16
        # (NB:882) with transformers' fp32 `wo` / fp32 residual stream (SURVEY Appendix A.7)
        self._dtype = compute_dtype
        self._lib = _lib.load("fp16" if compute_dtype == torch.float16 else "bf16")
        self._device = device
        self.config = SimpleNamespace(**config)
        self.generation_config = SimpleNamespace(
            max_length=_HF_DEFAULT_MAX_LENGTH,
            eos_token_id=config.get("eos_token_id", 1),
            pad_token_id=config.get("pad_token_id", 0),
            decoder_start_token_id=config.get("decoder_start_token_id", config.get("pad_token_id", 0)),
        )
        ffp = config.get("feed_forward_proj", "gated-gelu")
        cfg = _lib.Config(
            vocab_size=config["vocab_size"], d_model=config["d_model"], d_kv=config["d_kv"], d_ff=config["d_ff"],
            num_heads=config["num_heads"], num_layers=config["num_layers"],
            num_decoder_layers=config.get("num_decoder_layers") or config["num_layers"],
            relative_attention_num_buckets=config.get("relative_attention_num_buckets", 32),
            relative_attention_max_distance=config.get("relative_attention_max_distance", 128),
            layer_norm_epsilon=config.get("layer_norm_epsilon", 1e-6),
            pad_token_id=self.generation_config.pad_token_id,
            eos_token_id=self.generation_config.eos_token_id,
            decoder_start_token_id=self.generation_config.decoder_start_token_id,
            is_gated_gelu=1 if ffp == "gated-gelu" else 0,
            # HF decides "scale decoder outputs" from tie_word_embeddings (configuration_t5.py:82)
            scale_decoder_outputs=0 if config.get("tie_word_embeddings", True) is False else 1,
        )
        h = C.c_void_p()
        index = device.index if device.index is not None else torch.cuda.current_device()
        _chk(self, self._lib.b200t5_create(C.byref(cfg), index, C.byref(h)))
        self._h = h
        self._index = index
        self.last_lengths: Optional[torch.Tensor] = None
        # generate() switches to the continuous-batching path for batches larger than pool_size; that path runs
        # pool_slots decode slots (tools/bench_stream.py measures the choice)
        self.pool_size = int(os.environ.get("B200T5_POOL", "256"))
        # one handle = one execution plan: calls are serialised. Two host threads may alternate on it (the detokenise /
        # DataFrame tail of block i overlaps the GPU part of block i+1: rayshim/train.py:_overlap_tail).
        self._gpu_lock = threading.RLock()
        self.pool_slots = int(os.environ.get("B200T5_POOL_SLOTS", "512"))

    # ------------------------------------------------------------------ loading
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, device_map=None, torch_dtype=None,
                        dtype=None, device=None, **kwargs) -> "B200T5ForConditionalGeneration":
        """Load a Hugging Face T5 directory (config.json + model.safetensors | pytorch_model.bin).

        `device_map="auto"` / `torch_dtype=` are accepted as the notebook passes them (NB:881-882).
        torch_dtype=bfloat16 (default) and torch_dtype=float16 select the two numerics contracts the library
        implements; float16 is transformers' mode for T5: fp16 weights and activations, `wo` kept in fp32, fp32
        residual stream from the first feed-forward block on. float32 is honoured as "load and round to
        bfloat16" with a warning.
        """
        path = Path(pretrained_model_name_or_path)
        if not (path / "config.json").exists():
            raise FileNotFoundError(f"{path} is not a Hugging Face checkpoint directory (no config.json); "
                                    "hub downloads are not available offline")
        want = dtype if dtype is not None else torch_dtype
        compute = torch.float16 if want in (torch.float16, "float16", "half") else torch.bfloat16
        if want not in (None, torch.bfloat16, "bfloat16", "auto", torch.float16, "float16", "half"):
            warnings.warn(f"B200T5ForConditionalGeneration computes in bfloat16 or float16; requested {want} weights "
                          "are rounded to bfloat16 on load", stacklevel=2)
        if not torch.cuda.is_available():
            raise RuntimeError("no CUDA device: B200T5ForConditionalGeneration has no CPU fallback")
        if device is None:
            if device_map is None or device_map in ("auto", "balanced", "sequential"):
                device = torch.device("cuda", torch.cuda.current_device())  # one replica per process/GPU
            elif isinstance(device_map, dict):
                device = torch.device(next(iter(device_map.values())))
            else:
                device = torch.device(device_map)
        if torch.device(device).type == "cuda" and torch.device(device).index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        config = json.loads((path / "config.json").read_text())
        model = cls(config, device, compute)
        model._load_weights(path)
        return model

    def _load_weights(self, path: Path) -> None:
        st = path / "model.safetensors"
        tensors: Dict[str, torch.Tensor] = {}
        if st.exists():
            for name, (dt, shape, arr) in read_safetensors(st).items():
                a = np.array(arr)  # copy out of the memmap
                if dt == "BF16":
                    t = torch.from_numpy(a.view(np.int16)).view(torch.bfloat16)
                else:
                    t = torch.from_numpy(a)
                tensors[name] = t
        elif (path / "pytorch_model.bin").exists():
            tensors = torch.load(path / "pytorch_model.bin", map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"{path}: neither model.safetensors nor pytorch_model.bin found")
        self.load_state_dict(tensors)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        codes = {torch.bfloat16: _lib.DTYPE_BF16, torch.float16: _lib.DTYPE_F16, torch.float32: _lib.DTYPE_F32}
        with torch.cuda.device(self._index):
            for name, t in state_dict.items():
                if name in _IGNORED_WEIGHTS or name in _ALIASES:
                    continue
                if t.dtype not in codes:
                    t = t.float()
                dev = t.to(self._device).contiguous()
                shape = (C.c_int64 * dev.dim())(*dev.shape)
                _chk(self, self._lib.b200t5_set_weight(self._h, name.encode(), _ptr(dev), codes[dev.dtype], shape,
                                                       dev.dim()), self._h)
                del dev
            _chk(self, self._lib.b200t5_finalize(self._h), self._h)
        return SimpleNamespace(missing_keys=[], unexpected_keys=[])

    # ------------------------------------------------------------------ nn.Module-ish surface
    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def dtype(self) -> torch.dtype:
        return self._dtype

    def eval(self):
        return self

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (str, torch.device)) and torch.device(a) != self._device and torch.device(a).type != "cuda":
                raise RuntimeError("B200T5ForConditionalGeneration cannot be moved off the GPU")
        return self

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                self._lib.b200t5_destroy(h)
            except Exception:
                pass
            self._h = None

    # ------------------------------------------------------------------ generation
    def _gen_params(self, max_new_tokens, max_length, min_new_tokens, min_length, eos_token_id, pad_token_id,
                    decoder_start_token_id, poll_interval) -> _lib.GenParams:
        # GenerationMixin._prepare_generated_length (generation/utils.py:1619-1639): the decoder
        # prompt is the single start token, so max_length = max_new_tokens + 1.
        if max_new_tokens is None:
            max_length = self.generation_config.max_length if max_length is None else max_length
            max_new_tokens = int(max_length) - 1
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        if min_new_tokens is None:
            min_new_tokens = max(int(min_length) - 1, 0) if min_length else 0
        if isinstance(eos_token_id, (list, tuple, torch.Tensor)):
            eos_token_id = _eos_ids(eos_token_id)[0]  # the rest go to the logits processors (_logits_args)
        return _lib.GenParams(
            max_new_tokens=int(max_new_tokens), min_new_tokens=int(min(min_new_tokens, max_new_tokens)),
            eos_token_id=-1 if eos_token_id is None else int(eos_token_id),
            pad_token_id=-1 if pad_token_id is None else int(pad_token_id),
            decoder_start_token_id=-1 if decoder_start_token_id is None else int(decoder_start_token_id),
            poll_interval=int(poll_interval),
        )

    def _logits_args(self, kw: Dict[str, Any], eos_token_id) -> Optional[_LogitsArgs]:
        default_eos = self.generation_config.eos_token_id
        return logits_processor_args(kw, _eos_ids(eos_token_id), default_eos, self.config.vocab_size)

    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, *, max_new_tokens=None, max_length=None,
                 min_new_tokens=None, min_length=None, eos_token_id=None, pad_token_id=None,
                 decoder_start_token_id=None, do_sample=False, num_beams=1, poll_interval=8,
                 **unused) -> torch.LongTensor:
        """Greedy `generate`: returns int64 [B, 1+T'] on `self.device`, column 0 the decoder start
        token, rows padded after their EOS, T' = steps until every row finished (<= max_new_tokens).
        `labels` (which the reference passes, JOB/utils.py:31) and other HF kwargs that do not
        change greedy decoding are accepted and ignored, as HF itself does (generation/utils.py:583).
        transformers' greedy logits processors are applied on the GPU: repetition_penalty,
        encoder_repetition_penalty, no_repeat_ngram_size, encoder_no_repeat_ngram_size, bad_words_ids,
        suppress_tokens, begin_suppress_tokens, and eos_token_id given as a list.
        return_dict_in_generate=True returns a GenerateOutput (`.sequences` = that tensor); with output_scores=True its
        `.scores` / `.token_logprobs` carry each generated token's processed score and log-probability, computed in
        the lm_head epilogue (see TokenScores, compute_transition_scores). output_logits / output_attentions /
        output_hidden_states raise NotImplementedError."""
        if input_ids is None:
            input_ids = unused.pop("inputs", None)
        if input_ids is None:
            raise ValueError("input_ids is required")
        if do_sample or (num_beams is not None and num_beams != 1):
            raise NotImplementedError("only greedy decoding (do_sample=False, num_beams=1) is implemented")
        for k in ("temperature", "top_k", "top_p", "num_return_sequences"):
            v = unused.get(k)
            if v is not None and not (isinstance(v, (int, float)) and v == 1):
                raise NotImplementedError(f"generate({k}=...) is not supported by the CUDA path")
        for k in ("logits_processor", "stopping_criteria", "forced_bos_token_id", "decoder_input_ids", "encoder_outputs"):
            if unused.get(k) is not None:  # (may be tensors: no truth-value tests)
                raise NotImplementedError(f"generate({k}=...) is not supported by the CUDA path")
        as_dict, want_scores = generate_output_flags(unused)
        gp = self._gen_params(max_new_tokens, max_length, min_new_tokens, min_length, eos_token_id, pad_token_id,
                              decoder_start_token_id, poll_interval)
        lp = self._logits_args(unused, eos_token_id)
        host = torch.as_tensor(input_ids)
        if host.dim() != 2:
            raise ValueError(f"input_ids must be [batch, seq], got {tuple(host.shape)}")
        if as_dict:
            if not want_scores:  # the unchanged greedy call, wrapped
                return GenerateOutput(self.generate(input_ids=input_ids, attention_mask=attention_mask, max_new_tokens=gp.max_new_tokens,
                                                    min_new_tokens=gp.min_new_tokens, eos_token_id=eos_token_id, pad_token_id=pad_token_id,
                                                    decoder_start_token_id=decoder_start_token_id, poll_interval=poll_interval,
                                                    **{k: unused[k] for k in LOGITS_PROCESSOR_KWARGS if k in unused}))
            seq, _, logp, logit = self._run_scored(host, attention_mask, gp, lp, None)
            return GenerateOutput(seq, TokenScores(logp, logit))
        if self.takes_host_batches(host.shape[0], host.shape[1]) and host.device.type == "cpu":
            # more rows than one pool of decode slots, still in host memory: the slot pool admits prompts from host
            # buffers as slots free up, so nothing is copied to the device (and back) up front
            return self._generate_pool_from_host(host, attention_mask, gp, lp)
        ids, mask = self._device_inputs(host, attention_mask, gp, lp)
        B, S = ids.shape
        if B > self.pool_size:
            if self.takes_host_batches(B, S):
                # more rows than one pool of decode slots: continuous batching, same tokens row for row. The pool
                # admits prompts from host memory as slots free up (its entry point takes host buffers).
                out_np, _ = self.generate_stream(ids.cpu().numpy(), None if mask is None else mask.cpu().numpy(), _gen_params=gp,
                                                 _logits=lp)
                return torch.from_numpy(out_np).to(self._device)
            # prompts the slot pool cannot take (it needs the packed encoder, S <= 512): static batches
            outs = [self._generate_static(ids[lo:lo + self.pool_size], None if mask is None else mask[lo:lo + self.pool_size], gp, lp)
                    for lo in range(0, B, self.pool_size)]
            width = max(o.shape[1] for o in outs)
            pad = gp.pad_token_id if gp.pad_token_id >= 0 else self.generation_config.pad_token_id
            return torch.cat([torch.nn.functional.pad(o, (0, width - o.shape[1]), value=pad) for o in outs], dim=0)
        return self._generate_static(ids, mask, gp, lp)

    def compute_transition_scores(self, sequences, scores, beam_indices=None, normalize_logits: bool = False):
        """transformers' GenerationMixin.compute_transition_scores for the `.scores` of this model's generate: the
        chosen tokens' log-probabilities (normalize_logits=True) or processed scores (False), fp32 [B, T']. One
        deviation: positions after a row's EOS are 0 (transformers reports the score of the pad token it fed)."""
        if not isinstance(scores, TokenScores):
            raise TypeError("scores must be the `.scores` of this model's generate(..., output_scores=True)")
        if beam_indices is not None:
            raise NotImplementedError("beam search is not implemented")
        return scores.token_logprobs if normalize_logits else scores.token_logits

    @torch.no_grad()
    def score(self, input_ids, attention_mask=None, labels=None):
        """Teacher-forced log-likelihood of given targets, `T5ForConditionalGeneration(input_ids, attention_mask,
        labels=labels)` without the logits: labels int64 [B, L], -100 after a row's last label. Returns
        `.token_logprobs` fp32 [B, L] = log p(label | prompt, earlier labels) (0 at ignored positions), `.lengths` (labels
        per row) and `.loss` = -sum / count over all labels, transformers' mean cross-entropy. More rows than
        `pool_size` go through the slot pool; each (prompt, target) pair is a row."""
        lab = score_labels(labels, self.config.vocab_size)
        gp = _lib.GenParams(max_new_tokens=lab.shape[1], min_new_tokens=0, eos_token_id=-1, pad_token_id=-1,
                            decoder_start_token_id=-1, poll_interval=8)
        host = torch.as_tensor(input_ids)
        if host.dim() != 2 or host.shape[0] != lab.shape[0]:
            raise ValueError(f"input_ids must be [batch, seq] with one row per row of labels, got {tuple(host.shape)}")
        _, lens, logp, _ = self._run_scored(host, attention_mask, gp, None, lab)
        count = int((lab != -100).sum())
        return SimpleNamespace(token_logprobs=logp, lengths=lens, loss=-(logp.double().sum() / count).float())

    def _run_scored(self, host: torch.Tensor, attention_mask, gp, lp, labels: Optional[np.ndarray]):
        """generate's routing (static batch, slot pool, static chunks) for a scored call: (sequences [B, 1+T'],
        lengths [B], token_logprobs [B, T'], token_logits [B, T']) on the device. With `labels` the call is
        teacher-forced and T' = labels.shape[1]."""
        ids, mask = self._device_inputs(host, attention_mask, gp, lp)
        B, S = ids.shape
        T = gp.max_new_tokens
        if B > self.pool_size and self.takes_host_batches(B, S):
            out, lens, logp, logit = self.generate_stream(ids.cpu().numpy(), None if mask is None else mask.cpu().numpy(),
                                                          _gen_params=gp, _logits=lp, _labels=labels, output_scores=True)
            out, lens, logp, logit = (torch.from_numpy(np.ascontiguousarray(a)).to(self._device) for a in (out, lens, logp, logit))
        else:
            parts = [self._generate_static(ids[lo:lo + self.pool_size], None if mask is None else mask[lo:lo + self.pool_size], gp, lp,
                                           score=True, labels=None if labels is None else labels[lo:lo + self.pool_size])
                     for lo in range(0, B, self.pool_size)]
            out, lens, logp, logit = (torch.cat([p[i] for p in parts], dim=0) for i in range(4))
        steps = T if labels is not None else int(lens.max().item())
        return out[:, : steps + 1], lens, logp[:, :steps], logit[:, :steps]

    def _score_io(self, logp, logit, labels):
        """b200t5_score_io over two result arrays and optional labels (torch tensors or numpy arrays, all on the side
        the entry point expects); returns the struct and what must stay alive with it."""
        ptr = (lambda a: C.c_void_p(a.data_ptr())) if isinstance(logp, torch.Tensor) else (lambda a: a.ctypes.data_as(C.c_void_p))
        io = _lib.ScoreIO(token_logprobs=ptr(logp), token_logits=ptr(logit), forced_ids=None if labels is None else ptr(labels),
                          forced_len=0 if labels is None else int(labels.shape[1]))
        return io, (logp, logit, labels)

    def _check_inputs(self, ids, mask) -> None:
        """input_ids (a torch tensor or a numpy array) within [0, vocab_size), and attention_mask (None: not given) of
        the same shape."""
        V = self.config.vocab_size
        bad = False
        if isinstance(ids, torch.Tensor):
            if ids.numel():
                lo, hi = torch.aminmax(ids)  # one kernel, one synchronisation
                bad = bool(((lo < 0) | (hi >= V)).item())
        elif ids.size:
            bad = int(ids.min()) < 0 or int(ids.max()) >= V
        if bad:
            raise IndexError("input_ids contain token ids outside [0, vocab_size)")
        if mask is not None and mask.shape != ids.shape:
            raise ValueError("attention_mask shape must match input_ids")

    def _device_inputs(self, host: torch.Tensor, attention_mask, gp, lp):
        """input_ids and attention_mask as contiguous int64 tensors on the model's device, checked; without an
        attention_mask the inferred one (None: attend everywhere)."""
        ids = host.to(device=self._device, dtype=torch.long).contiguous()
        mask = None
        if attention_mask is not None:
            mask = torch.as_tensor(attention_mask).to(device=self._device, dtype=torch.long).contiguous()
        self._check_inputs(ids, mask)
        return ids, (self._infer_attention_mask(ids, gp, lp) if mask is None else mask)

    def takes_host_batches(self, B: int, S: int) -> bool:
        """True when a [B, S] batch would go through the slot pool, whose entry point takes HOST buffers: a caller that
        still has the batch in host memory (predictor.py) hands it over as it is."""
        return B > self.pool_size and S <= _POOL_MAX_S and os.environ.get("B200T5_STREAM", "1") != "0"

    def _generate_pool_from_host(self, ids: torch.Tensor, attention_mask, gp, lp=None) -> torch.Tensor:
        ids_np = np.ascontiguousarray(ids.numpy(), dtype=np.int64)
        mask_np = None
        if attention_mask is not None:
            mask_np = np.ascontiguousarray(torch.as_tensor(attention_mask).cpu().numpy(), dtype=np.int64)
        self._check_inputs(ids_np, mask_np)
        if mask_np is None:
            mask_np = self._infer_mask_np(ids_np, gp, lp)
        out_np, _ = self.generate_stream(ids_np, mask_np, _gen_params=gp, _logits=lp)
        return torch.from_numpy(out_np).to(self._device)

    def _pad_is_eos(self, gp, lp) -> bool:
        pad = gp.pad_token_id if gp.pad_token_id >= 0 else self.generation_config.pad_token_id
        eos = gp.eos_token_id if gp.eos_token_id >= 0 else self.generation_config.eos_token_id
        return pad is None or pad == eos or (lp is not None and pad in lp.eos_ids)

    def _infer_attention_mask(self, ids: torch.Tensor, gp, lp=None) -> Optional[torch.Tensor]:
        """GenerationMixin._prepare_attention_mask_for_generation (transformers generation/utils.py): without an
        attention_mask the pad positions are masked when the pad token occurs in the inputs and is not an EOS
        token; otherwise every position is attended (None = all ones for the library)."""
        pad = gp.pad_token_id if gp.pad_token_id >= 0 else self.generation_config.pad_token_id
        if self._pad_is_eos(gp, lp):
            return None
        is_pad = ids == pad
        if not bool(is_pad.any().item()):
            return None
        return (~is_pad).to(torch.long).contiguous()

    def _generate_static(self, ids: torch.Tensor, mask: Optional[torch.Tensor], gp, lp=None, score: bool = False, labels=None):
        B, S = ids.shape
        ids = ids.contiguous()
        mask = None if mask is None else mask.contiguous()
        T = gp.max_new_tokens
        with torch.cuda.device(self._index):
            out = torch.empty((B, T + 1), dtype=torch.long, device=self._device)
            lens = torch.empty((B,), dtype=torch.int32, device=self._device)
            stream = torch.cuda.current_stream(self._device)
            with self._gpu_lock:
                io = None
                if score:  # full-width results: (ids [B, T+1], lengths, token_logprobs [B, T], token_logits [B, T])
                    logp = torch.empty((B, T), dtype=torch.float32, device=self._device)
                    logit = torch.empty((B, T), dtype=torch.float32, device=self._device)
                    forced = None if labels is None else torch.from_numpy(np.ascontiguousarray(labels)).to(self._device)
                    io, _keep = self._score_io(logp, logit, forced)
                _chk(self, self._lib.b200t5_generate_scored(self._h, _ptr(ids), _ptr(mask), B, S, C.byref(gp),
                                                            None if lp is None else lp.ref(), _ptr(out), _ptr(lens),
                                                            None if io is None else C.byref(io), C.c_void_p(stream.cuda_stream)),
                     self._h)
                self.last_lengths = lens
                if score:
                    torch.cuda.current_stream(self._device).synchronize()
                    return out, lens, logp, logit
                steps = int(lens.max().item())  # synchronises; HF returns exactly the steps it ran
        return out[:, : steps + 1]

    def _infer_mask_np(self, ids: np.ndarray, gp, lp=None) -> Optional[np.ndarray]:
        pad = gp.pad_token_id if gp.pad_token_id >= 0 else self.generation_config.pad_token_id
        if self._pad_is_eos(gp, lp) or not (ids == pad).any():
            return None
        return np.ascontiguousarray(ids != pad, dtype=np.int64)

    def generate_host(self, input_ids: np.ndarray, attention_mask: Optional[np.ndarray] = None, **kw):
        """numpy in / numpy out through b200t5_generate_host_scored (the foreign-host entry point):
        H2D copy, generation, D2H copy and synchronisation all happen inside the library. Takes the logits
        processor kwargs `generate` takes. With output_scores=True it returns (ids, lengths, token_logprobs,
        token_logits), the last two fp32 [B, T']."""
        gp = self._gen_params(kw.get("max_new_tokens"), kw.get("max_length"), kw.get("min_new_tokens"),
                              kw.get("min_length"), kw.get("eos_token_id"), kw.get("pad_token_id"),
                              kw.get("decoder_start_token_id"), kw.get("poll_interval", 8))
        lp = self._logits_args(kw, kw.get("eos_token_id"))
        ids = np.ascontiguousarray(input_ids, dtype=np.int64)
        B, S = ids.shape
        mask = self._infer_mask_np(ids, gp, lp) if attention_mask is None else np.ascontiguousarray(attention_mask, dtype=np.int64)
        out = np.empty((B, gp.max_new_tokens + 1), dtype=np.int64)
        lens = np.empty((B,), dtype=np.int32)
        want_scores = generate_output_flags(kw)[1]
        with self._gpu_lock:
            mp = None if mask is None else mask.ctypes.data_as(C.c_void_p)
            io = None
            if want_scores:  # -> (ids, lengths, token_logprobs, token_logits), numpy
                logp = np.empty((B, gp.max_new_tokens), dtype=np.float32)
                logit = np.empty((B, gp.max_new_tokens), dtype=np.float32)
                io, _keep = self._score_io(logp, logit, None)
            _chk(self, self._lib.b200t5_generate_host_scored(self._h, ids.ctypes.data_as(C.c_void_p), mp, B, S, C.byref(gp),
                                                             None if lp is None else lp.ref(), out.ctypes.data_as(C.c_void_p),
                                                             lens.ctypes.data_as(C.c_void_p), None if io is None else C.byref(io)),
                 self._h)
        steps = int(lens.max())
        if want_scores:
            return out[:, : steps + 1], lens, logp[:, :steps], logit[:, :steps]
        return out[:, : steps + 1], lens

    def generate_stream(self, input_ids: np.ndarray, attention_mask: Optional[np.ndarray] = None, *, pool: Optional[int] = None,
                        admit_min: int = 0, _gen_params=None, _logits=None, _labels=None, **kw):
        """N prompts through a pool of decode slots (b200t5_generate_stream): a slot whose row has finished is
        refilled with the next prompt, so short answers do not wait for the slowest row of a fixed batch as they do
        when BatchPredictor hands `generate` one batch at a time (NB:908-913 -> JOB/predictor.py:102). Returns
        (int64 [N, 1+T'], int32 lengths [N]) with the rows in input order; every row equals what `generate` returns
        for that prompt. Takes the logits processor kwargs `generate` takes. With output_scores=True it returns (ids,
        lengths, token_logprobs, token_logits), the last two fp32 [N, T'] (b200t5_generate_stream_scored)."""
        gp = _gen_params or self._gen_params(kw.get("max_new_tokens"), kw.get("max_length"), kw.get("min_new_tokens"),
                                             kw.get("min_length"), kw.get("eos_token_id"), kw.get("pad_token_id"),
                                             kw.get("decoder_start_token_id"), kw.get("poll_interval", 8))
        lp = _logits if _gen_params is not None else self._logits_args(kw, kw.get("eos_token_id"))
        ids = np.ascontiguousarray(input_ids, dtype=np.int64)
        if ids.ndim != 2:
            raise ValueError(f"input_ids must be [batch, seq], got {ids.shape}")
        N, S = ids.shape
        mask = None if attention_mask is None else np.ascontiguousarray(attention_mask, dtype=np.int64)
        self._check_inputs(ids, mask)
        if mask is None:
            mask = self._infer_mask_np(ids, gp, lp)
        out = np.empty((N, gp.max_new_tokens + 1), dtype=np.int64)
        lens = np.empty((N,), dtype=np.int32)
        want_scores = generate_output_flags(kw)[1]
        with self._gpu_lock:
            mp = None if mask is None else mask.ctypes.data_as(C.c_void_p)
            io = None
            if want_scores:
                logp = np.empty((N, gp.max_new_tokens), dtype=np.float32)
                logit = np.empty((N, gp.max_new_tokens), dtype=np.float32)
                io, _keep = self._score_io(logp, logit, None if _labels is None else np.ascontiguousarray(_labels, dtype=np.int64))
            _chk(self, self._lib.b200t5_generate_stream_scored(self._h, ids.ctypes.data_as(C.c_void_p), mp, N, S, C.byref(gp),
                                                               None if lp is None else lp.ref(), int(pool or self.pool_slots),
                                                               int(admit_min), out.ctypes.data_as(C.c_void_p),
                                                               lens.ctypes.data_as(C.c_void_p), None if io is None else C.byref(io)),
                 self._h)
        self.last_lengths = torch.from_numpy(lens)
        steps = int(lens.max())
        if want_scores:
            return out[:, : steps + 1], lens, logp[:, :steps], logit[:, :steps]
        return out[:, : steps + 1], lens

    def stats(self) -> Dict[str, float]:
        s = _lib.Stats()
        _chk(self, self._lib.b200t5_get_stats(self._h, C.byref(s)), self._h)
        return {k: getattr(s, k) for k, _ in _lib.Stats._fields_}

    def bench_cross_attention(self, reps: int = 5, rows_per_launch: int = 0) -> Dict[str, float]:
        """Average launch time of the cross-attention decode kernel ALONE on the last call's KV arena, in launches of
        `rows_per_launch` rows (0 = the whole batch). A microbenchmark; `xattn_profile` is the in-situ figure."""
        ms, nbytes = C.c_float(), C.c_double()
        with torch.cuda.device(self._index):
            stream = torch.cuda.current_stream(self._device)
            _chk(self, self._lib.b200t5_bench_cross_attn(self._h, reps, int(rows_per_launch), C.byref(ms), C.byref(nbytes),
                                                         C.c_void_p(stream.cuda_stream)), self._h)
        return {"ms_per_launch": ms.value, "bytes_per_launch": nbytes.value}

    def set_option(self, name: str, value: int) -> None:
        """Runtime knob of the library (include/b200t5.h: b200t5_set_option); drops the execution plan."""
        _chk(self, self._lib.b200t5_set_option(self._h, name.encode(), int(value)), self._h)

    def xattn_profile(self) -> Dict[str, float]:
        """In-situ timing of the cross-attention launches of the step graph since set_option("profile_xattn", 1): per
        launch, and per layer as the union of the row-chains' (possibly overlapping) launches."""
        us, n, nbytes, busy, lbytes = C.c_double(), C.c_int64(), C.c_double(), C.c_double(), C.c_double()
        _chk(self, self._lib.b200t5_get_xattn_profile(self._h, C.byref(us), C.byref(n), C.byref(nbytes), C.byref(busy),
                                                      C.byref(lbytes)), self._h)
        return {"us_per_launch": us.value, "launches": int(n.value), "bytes_per_launch": nbytes.value,
                "busy_us_per_layer": busy.value, "bytes_per_layer": lbytes.value}

    # ------------------------------------------------------------------ parity hooks (tests)
    @torch.no_grad()
    def encode(self, input_ids, attention_mask=None) -> torch.Tensor:
        ids = torch.as_tensor(input_ids).to(self._device, torch.long).contiguous()
        mask = None if attention_mask is None else torch.as_tensor(attention_mask).to(self._device, torch.long).contiguous()
        B, S = ids.shape
        out = torch.empty((B, S, self.config.d_model), dtype=self._dtype, device=self._device)
        with torch.cuda.device(self._index):
            stream = torch.cuda.current_stream(self._device)
            _chk(self, self._lib.b200t5_encode(self._h, _ptr(ids), _ptr(mask), B, S, _ptr(out),
                                               C.c_void_p(stream.cuda_stream)), self._h)
            torch.cuda.synchronize(self._device)
        return out

    @torch.no_grad()
    def decode_logits(self, input_ids, attention_mask, decoder_input_ids) -> torch.Tensor:
        ids = torch.as_tensor(input_ids).to(self._device, torch.long).contiguous()
        mask = None if attention_mask is None else torch.as_tensor(attention_mask).to(self._device, torch.long).contiguous()
        dec = torch.as_tensor(decoder_input_ids).to(self._device, torch.long).contiguous()
        B, S = ids.shape
        T = dec.shape[1]
        out = torch.empty((B, T, self.config.vocab_size), dtype=torch.float32, device=self._device)
        with torch.cuda.device(self._index):
            stream = torch.cuda.current_stream(self._device)
            _chk(self, self._lib.b200t5_decode_logits(self._h, _ptr(ids), _ptr(mask), B, S, _ptr(dec), T, _ptr(out),
                                                      C.c_void_p(stream.cuda_stream)), self._h)
        return out
