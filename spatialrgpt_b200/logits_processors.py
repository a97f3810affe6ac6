"""HF's logits processors behind generate(repetition_penalty=, no_repeat_ngram_size=, bad_words_ids=, min_length=, min_new_tokens=):
the kwargs' validation, their mapping to one processor spec, and the spec's device encoding (csrc/logits_process.cu runs it).

Semantics (transformers generation/logits_process.py and generation/utils.py; DESIGN.md §3 lists where 4.37.2 differs):
  * the history is the generated tokens only: the reference calls HF with inputs_embeds, so HF's input_ids start empty;
  * order: repetition penalty, no-repeat n-gram, bad words, minimum length (min_length, min_new_tokens), then sampling's warpers;
  * bad_words_ids equal to [eos] are dropped; a minimum length without an EOS id is a no-op;
  * min_length L counts the prompt: m = max(L - S, 0) with S the inputs_embeds length; min_new_tokens wins over it.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

F_PENALTY, F_NGRAM, F_BAD, F_MINLEN = 1, 2, 4, 8
SPEC_HEAD = 5  # flags, n-gram size, minimum new tokens, n_eos, n_bad


def eos_list(eos_token_id) -> List[int]:
    if eos_token_id is None:
        return []
    if isinstance(eos_token_id, (list, tuple, set)):
        return [int(e) for e in eos_token_id]
    if hasattr(eos_token_id, "tolist"):
        v = eos_token_id.tolist()
        return [int(e) for e in (v if isinstance(v, list) else [v])]
    return [int(eos_token_id)]


def parse(repetition_penalty=None, no_repeat_ngram_size=None, bad_words_ids=None, min_new_tokens=None, min_length=None, eos_token_id=None,
          vocab_size: Optional[int] = None) -> Optional[dict]:
    """Validates the processor kwargs of one generate() call (ValueError for what HF rejects) and returns the spec, or None when every
    option is neutral (penalty 1.0, n-gram size 0, no minimum, no bad words).  ``min_length`` stays unresolved until the prompt length
    is known (resolve_min_length)."""
    spec = {}
    if repetition_penalty is not None:
        p = float(repetition_penalty)
        if not p > 0:
            raise ValueError(f"`repetition_penalty` has to be a strictly positive float, but is {repetition_penalty}")
        if p != 1.0:
            spec["repetition_penalty"] = p
    if no_repeat_ngram_size is not None:
        if isinstance(no_repeat_ngram_size, bool) or int(no_repeat_ngram_size) != no_repeat_ngram_size or no_repeat_ngram_size < 0:
            raise ValueError(f"`no_repeat_ngram_size` has to be a strictly positive integer, but is {no_repeat_ngram_size}")
        if no_repeat_ngram_size > 0:
            spec["no_repeat_ngram_size"] = int(no_repeat_ngram_size)
    eos = eos_list(eos_token_id)
    if bad_words_ids is not None:
        if not isinstance(bad_words_ids, list) or len(bad_words_ids) == 0:
            raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bad_words_ids}.")
        if any(not isinstance(seq, list) or len(seq) == 0 for seq in bad_words_ids):
            raise ValueError(f"`bad_words_ids` has to be a list of non-empty lists, but is {bad_words_ids}.")
        for seq in bad_words_ids:
            for t in seq:
                if isinstance(t, bool) or not isinstance(t, (int, np.integer)) or t < 0:
                    raise ValueError(f"Each list in `bad_words_ids` has to be a list of positive integers, but is {bad_words_ids}.")
                if vocab_size is not None and t >= vocab_size:
                    raise ValueError(f"The model vocabulary size is {vocab_size}, but the token {t} of `bad_words_ids` is outside it")
        seqs = [[int(t) for t in seq] for seq in bad_words_ids if not any(seq == [e] for e in eos)]  # HF drops [eos]
        if seqs:
            spec["bad_words_ids"] = seqs
    for name, v in (("min_new_tokens", min_new_tokens), ("min_length", min_length)):
        if v is not None:
            if isinstance(v, bool) or int(v) != v:
                raise ValueError(f"`{name}` has to be an integer, but is {v}")
            if v > 0 and eos and not (name == "min_length" and min_new_tokens is not None):  # min_new_tokens (even 0) wins; without
                spec[name] = int(v)                                                             # an EOS id HF builds no such processor
    if not spec:
        return None
    spec["eos_token_ids"] = eos
    return spec


def resolve_min_length(spec: Optional[dict], prompt_len: int) -> Optional[dict]:
    """The decoder's spec: min_length L -> min_new_tokens max(L - S, 0) (HF _prepare_generated_length subtracts the inputs_embeds
    length S), unless min_new_tokens is given, which wins.  None when nothing is left to do."""
    if spec is None:
        return None
    out = {k: v for k, v in spec.items() if k != "min_length"}
    if "min_new_tokens" not in out and "min_length" in spec:
        m = max(spec["min_length"] - int(prompt_len), 0)
        if m > 0:
            out["min_new_tokens"] = m
    return out if set(out) - {"eos_token_ids"} else None


def encode(spec: dict):
    """(fparams float32 [penalty, 1 / penalty], ints int32 [flags, n, m, n_eos, n_bad, eos..., bad offsets..., bad tokens...]).  1 / penalty
    is the double reciprocal rounded to fp32: ATen's CUDA division by a Python scalar multiplies by that (DESIGN.md §3)."""
    p = float(spec.get("repetition_penalty", 1.0))
    fparams = np.array([np.float32(p), np.float32(1.0 / p)], dtype=np.float32)
    flags = 0
    flags |= F_PENALTY if "repetition_penalty" in spec else 0
    flags |= F_NGRAM if "no_repeat_ngram_size" in spec else 0
    bad = spec.get("bad_words_ids") or []
    flags |= F_BAD if bad else 0
    eos = list(spec.get("eos_token_ids") or [])
    m = int(spec.get("min_new_tokens", 0))
    flags |= F_MINLEN if m > 0 and eos else 0
    offs = np.cumsum([0] + [len(s) for s in bad]).tolist()
    ints = [flags, int(spec.get("no_repeat_ngram_size", 0)), m, len(eos), len(bad)] + eos + offs + [t for s in bad for t in s]
    return fparams, np.array(ints, dtype=np.int32)


def process_np(scores: np.ndarray, hist: Sequence[int], spec: dict, true_division: bool = False) -> np.ndarray:
    """numpy restatement of the kernel on one fp32 row (the tests pin it to transformers' processor classes).  ``true_division``:
    divide by the penalty as torch does on the CPU, instead of multiplying by fp32(1 / penalty) as ATen does on the GPU."""
    x = np.array(scores, dtype=np.float32).copy()
    hist = [int(t) for t in hist]
    n = len(hist)
    if "repetition_penalty" in spec:
        p = np.float32(spec["repetition_penalty"])
        inv = np.float32(1.0 / float(spec["repetition_penalty"]))
        for t in set(hist):
            x[t] = x[t] * p if x[t] < 0 else (x[t] / p if true_division else x[t] * inv)
    g = spec.get("no_repeat_ngram_size", 0)
    kill = set()
    if g:
        for i in range(0, n - g + 1):
            if hist[i:i + g - 1] == hist[n - g + 1:]:
                kill.add(hist[i + g - 1])
    bad = spec.get("bad_words_ids") or []
    if bad:
        bias = np.zeros_like(x)
        for s in bad:
            if len(s) == 1 or (len(s) <= n and hist[n - len(s) + 1:] == s[:-1]):
                bias[s[-1]] = -np.inf
        x = x + bias
    if n < spec.get("min_new_tokens", 0):
        kill.update(spec.get("eos_token_ids") or [])
    for t in kill:
        x[t] = -np.inf
    return x
