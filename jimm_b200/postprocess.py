"""Zero-shot / classification epilogue on the GPU: what the reference's examples compute in JAX after the forward path.

    probs, order = zero_shot(model(images, text))        # examples/clip_inference.py:46-51 for every image row
    values, indices = top_k(model(images, text), 5)      # the first 5 of that order, without sorting the row
    probs = pair_probabilities(siglip(images, text))     # sigmoid of SigLIP's biased logits
    labels = classify(vit(images))                       # examples/vit_inference.py:58
"""

from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib

_INT32_MAX = 2**31 - 1  # rows and columns are C ints, and the order holds int32 column indices


def _checked(logits: torch.Tensor) -> torch.Tensor:
    """The logits as a [rows, cols] CUDA tensor (1-D taken as one row), checked before anything is allocated."""
    if not isinstance(logits, torch.Tensor) or not logits.is_cuda:
        raise _lib.JimmError("postprocess expects the CUDA logits tensor the model returned; there is no CPU fallback")
    if logits.ndim == 1:
        logits = logits[None]
    if logits.ndim != 2:
        raise ValueError(f"expected logits of shape [rows, cols], got {tuple(logits.shape)}")
    if logits.shape[0] > _INT32_MAX or logits.shape[1] > _INT32_MAX:
        raise ValueError(f"postprocess takes at most {_INT32_MAX} rows and columns, got {tuple(logits.shape)}")
    return logits


def _rows(logits: torch.Tensor) -> torch.Tensor:
    """fp32 rows as the library reads them, `ld` floats apart with unit column stride: 16-bit logits cast, expanded (stride-0) or
    overlapping rows copied."""
    x = logits.to(torch.float32)
    rows, cols = x.shape
    if x.stride(1) != 1 or (rows > 1 and not cols <= x.stride(0) <= _INT32_MAX):
        x = x.contiguous()
    return x


def _stream(x: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)


def _run(logits: torch.Tensor, mode: int, want_probs: bool, want_order: bool, want_argmax: bool):
    x = _rows(_checked(logits))
    rows, cols = x.shape
    lib = _lib.load()
    with torch.cuda.device(x.device):
        probs = torch.empty((rows, cols), dtype=torch.float32, device=x.device) if want_probs else None
        order = torch.empty((rows, cols), dtype=torch.int32, device=x.device) if want_order else None
        amax = torch.empty((rows,), dtype=torch.int32, device=x.device) if want_argmax else None
        p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
        _lib.check(lib.jimm_postprocess(p(x), rows, cols, x.stride(0) if rows > 1 else cols, mode, p(probs), cols, p(order), p(amax),
                                        _stream(x)))
    return probs, order, amax


def zero_shot(logits: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per row: `exp(s) / sum(exp(s))` and `argsort(s)[::-1]` (examples/clip_inference.py:47,49)."""
    probs, order, _ = _run(logits, 0, True, True, False)
    return probs, order


def pair_probabilities(logits: torch.Tensor) -> torch.Tensor:
    """SigLIP: independent probability of every (image, text) pair, `sigmoid(logits)`."""
    return _run(logits, 1, True, False, False)[0]


def classify(logits: torch.Tensor) -> torch.Tensor:
    """`argmax(logits, -1)` (examples/vit_inference.py:58): first maximum per row, int32."""
    return _run(logits, 0, False, False, True)[2]


def top_k(logits: torch.Tensor, k: int, probs: bool = False):
    """The best k columns of each row: `values, indices` ([rows, k] fp32 and int32 on the logits' device), and with probs=True also
    the softmax probabilities there.  Bit for bit, indices is `zero_shot(logits)[1][:, :k]` (equal scores larger index first, every
    NaN first, -0 tied with +0), values is `logits.gather(1, indices)` in fp32 and the probabilities are `zero_shot(logits)[0]` at
    those columns -- without sorting the row: for k <= 1024 a radix select finds the k-th key and only the k survivors are sorted.
    Inputs as zero_shot takes them; 1 <= k <= cols."""
    logits = _checked(logits)
    rows, cols = logits.shape
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= cols:
        raise ValueError(f"top_k: k must be an int in 1 .. {cols} (the columns), got {k!r}")
    x = _rows(logits)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        values = torch.empty((rows, k), dtype=torch.float32, device=x.device)
        indices = torch.empty((rows, k), dtype=torch.int32, device=x.device)
        pr = torch.empty((rows, k), dtype=torch.float32, device=x.device) if probs else None
        p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
        _lib.check(lib.jimm_topk(p(x), rows, cols, x.stride(0) if rows > 1 else cols, k, p(values), p(indices), p(pr), _stream(x)))
    return (values, indices, pr) if probs else (values, indices)
