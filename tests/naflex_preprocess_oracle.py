"""CPU oracle of the SigLIP 2 NaFlex image front-end: transformers' `Siglip2ImageProcessorPil` restated with the pieces of
oracle/preprocess_oracle.py (Pillow's 8-bit resize, rescale + normalise) -- the size rule, the resize to each frame's own patch
grid, the (py, px, c) patchify, the zero padding rows and the attention mask.  Pinned against the processor itself and the
committed fixture tests/golden/preprocess_siglip2_naflex.npz (tests/test_naflex_preprocess_oracle.py)."""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np

import preprocess_oracle as PO


def siglip2_config(resample: int = PO.BILINEAR) -> PO.PreprocessConfig:
    """The Siglip2 processors' rescale / normalise settings (size comes from the patch budget, per image)."""
    return PO.PreprocessConfig(height=0, width=0, resample=resample, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))


def naflex_size(h: int, w: int, patch: int, max_num_patches: int, eps: float = 1e-5) -> Tuple[int, int]:
    """transformers' `get_image_size_for_max_num_patches`: the binary search over the scale, in Python floats (IEEE doubles)."""
    def scaled(scale, size):
        return max(patch, math.ceil(size * scale / patch) * patch)

    lo, hi = eps / 10, 100.0
    while (hi - lo) >= eps:
        scale = (lo + hi) / 2
        th, tw = scaled(scale, h), scaled(scale, w)
        if (th / patch) * (tw / patch) <= max_num_patches:
            lo = scale
        else:
            hi = scale
    return int(scaled(lo, h)), int(scaled(lo, w))


def pil_resize_u8(img: np.ndarray, out_h: int, out_w: int, resample: int, rows: int = 128) -> np.ndarray:
    """PO.pil_resize_u8 with each pass run over `rows` rows at a time: the same bytes (every output row depends on its own window
    only) in bounded memory, for camera-sized frames."""
    h, w, _ = img.shape
    fv, cv, kv = PO.resample_coeffs(h, out_h, resample)
    out = img
    if out_w != w:
        fh, _, kh = PO.resample_coeffs(w, out_w, resample)
        y0, y1 = int(fv[0]), int(fv[-1] + cv[-1])
        out = np.concatenate([PO._pass(img[a:min(a + rows, y1)], fh, kh, axis=1) for a in range(y0, y1, rows)])
        fv = fv - y0
    if out_h != h:
        out = np.concatenate([PO._pass(out, fv[a:a + rows], kv[a:a + rows], axis=0) for a in range(0, out_h, rows)])
    return np.ascontiguousarray(out)


def naflex_preprocess(img: np.ndarray, patch: int, max_num_patches: int, cfg: PO.PreprocessConfig):
    """uint8 [H, W, 3] -> (float32 patch rows [gh * gw, patch * patch * 3] in (py, px, c) order, (gh, gw))."""
    h, w, _ = img.shape
    th, tw = naflex_size(h, w, patch, max_num_patches)
    out = pil_resize_u8(img, th, tw, cfg.resample) if (th, tw) != (h, w) else img
    x = PO.rescale_normalize(out, cfg)
    gh, gw = th // patch, tw // patch
    rows = x.reshape(gh, patch, gw, patch, 3).transpose(0, 2, 1, 3, 4).reshape(gh * gw, patch * patch * 3)
    return np.ascontiguousarray(rows), (gh, gw)


def naflex_batch(imgs, patch: int, max_num_patches: int, cfg: PO.PreprocessConfig):
    """The processor's three outputs for a list of frames: pixel_values [B, N, P*P*3] (zero padding rows), pixel_attention_mask
    int32 [B, N], spatial_shapes int64 [B, 2]."""
    B, K = len(imgs), patch * patch * 3
    pv = np.zeros((B, max_num_patches, K), np.float32)
    mask = np.zeros((B, max_num_patches), np.int32)
    shapes = np.zeros((B, 2), np.int64)
    for b, img in enumerate(imgs):
        rows, (gh, gw) = naflex_preprocess(img, patch, max_num_patches, cfg)
        pv[b, :len(rows)] = rows
        mask[b, :len(rows)] = 1
        shapes[b] = (gh, gw)
    return pv, mask, shapes


def hf_processor(patch: int, max_num_patches: int, resample: int = PO.BILINEAR):
    from transformers import Siglip2ImageProcessorPil

    return Siglip2ImageProcessorPil(patch_size=patch, max_num_patches=max_num_patches, resample=resample)


def hf_batch(proc, imgs, max_num_patches: int = None):
    """Siglip2ImageProcessorPil on uint8 frames, as numpy (pixel_values, pixel_attention_mask, spatial_shapes)."""
    from PIL import Image

    kw = {} if max_num_patches is None else {"max_num_patches": max_num_patches}
    r = proc(images=[Image.fromarray(i) for i in imgs], return_tensors="np", **kw)
    return np.asarray(r["pixel_values"]), np.asarray(r["pixel_attention_mask"]), np.asarray(r["spatial_shapes"])
