"""Zero-shot / classification epilogue on the GPU: what the reference's examples compute in JAX after the forward path.

    probs, order = zero_shot(model(images, text))        # examples/clip_inference.py:46-51 for every image row
    probs = pair_probabilities(siglip(images, text))     # sigmoid of SigLIP's biased logits
    labels = classify(vit(images))                       # examples/vit_inference.py:58
"""

from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib

_INT32_MAX = 2**31 - 1  # rows and columns are C ints, and the order holds int32 column indices


def _run(logits: torch.Tensor, mode: int, want_probs: bool, want_order: bool, want_argmax: bool):
    if not isinstance(logits, torch.Tensor) or not logits.is_cuda:
        raise _lib.JimmError("postprocess expects the CUDA logits tensor the model returned; there is no CPU fallback")
    if logits.ndim == 1:
        logits = logits[None]
    if logits.ndim != 2:
        raise ValueError(f"expected logits of shape [rows, cols], got {tuple(logits.shape)}")
    rows, cols = logits.shape
    if rows > _INT32_MAX or cols > _INT32_MAX:  # before the cast / copy below allocates anything
        raise ValueError(f"postprocess takes at most {_INT32_MAX} rows and columns, got {tuple(logits.shape)}")
    x = logits.to(torch.float32)
    # the library reads rows `ld` floats apart with unit column stride: expanded (stride-0) or overlapping rows are copied first
    if x.stride(1) != 1 or (rows > 1 and not cols <= x.stride(0) <= _INT32_MAX):
        x = x.contiguous()
    lib = _lib.load()
    with torch.cuda.device(x.device):
        probs = torch.empty((rows, cols), dtype=torch.float32, device=x.device) if want_probs else None
        order = torch.empty((rows, cols), dtype=torch.int32, device=x.device) if want_order else None
        amax = torch.empty((rows,), dtype=torch.int32, device=x.device) if want_argmax else None
        p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
        _lib.check(lib.jimm_postprocess(p(x), rows, cols, x.stride(0) if rows > 1 else cols, mode, p(probs), cols, p(order), p(amax),
                                        C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
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
