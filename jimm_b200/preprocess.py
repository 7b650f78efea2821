"""GPU image front-end: the HuggingFace image processor the reference's examples run on the host, as one CUDA kernel.

    proc = ImagePreprocessor.from_pretrained("path/to/checkpoint_dir")      # reads preprocessor_config.json
    proc = ImagePreprocessor.clip(224)                                      # or the stock settings of a model family
    pixels_nhwc = proc(uint8_images, dtype=torch.float16)                   # [B,H,W,3] uint8 -> [B,h,w,3] on the GPU
    logits = model(pixels_nhwc)

Replaces `processor(images=image, return_tensors="np")["pixel_values"]` followed by `jnp.transpose(..., (0, 2, 3, 1))`
(examples/vit_inference.py:27-37, examples/clip_inference.py:35-38): Pillow resize (bilinear / bicubic, antialiased) ->
centre crop -> rescale -> normalise, bit-exact with transformers' PIL processors (see include/jimm_b200.h, csrc/preprocess.cu).
Constructor keywords follow `preprocessor_config.json` / the HF processors' kwargs.
"""

from __future__ import annotations

import ctypes as C
import json
import os
from typing import Optional, Sequence, Union

import numpy as np
import torch

from . import _lib

BILINEAR, BICUBIC = 2, 3
_OUT_CODE = {torch.float32: _lib.F32, torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _size_fields(size, default_to_square: bool = True) -> dict:
    """HF `get_size_dict`: a legacy integer size is square for ViTImageProcessor / SiglipImageProcessor (default_to_square=True) and the
    shortest edge for CLIPImageProcessor (default_to_square=False)."""
    if isinstance(size, int):
        return {"height": size, "width": size} if default_to_square else {"shortest_edge": size}
    if isinstance(size, (tuple, list)):
        return {"height": int(size[0]), "width": int(size[1])}
    if isinstance(size, dict):
        if "shortest_edge" in size and size["shortest_edge"]:
            if size.get("longest_edge"):
                raise ValueError("size with both shortest_edge and longest_edge is not part of the ViT / CLIP / SigLIP front-ends")
            return {"shortest_edge": int(size["shortest_edge"])}
        if size.get("height") and size.get("width"):
            return {"height": int(size["height"]), "width": int(size["width"])}
    raise ValueError(f"Size must contain 'height' and 'width' keys, or a 'shortest_edge' key. Got {size}.")


def _config(size=None, crop_size=None, resample: int = BILINEAR, do_center_crop: Optional[bool] = None,
            rescale_factor: float = 1 / 255, image_mean: Sequence[float] = (0.5, 0.5, 0.5), image_std: Sequence[float] = (0.5, 0.5, 0.5),
            do_resize: bool = True, do_rescale: bool = True, do_normalize: bool = True, default_to_square: bool = True) -> _lib.PreprocConfig:
    """jimm_preproc_config_t of ImagePreprocessor's keywords (checked here; no GPU needed)."""
    if not (do_resize and do_rescale and do_normalize):
        raise ValueError("the GPU front-end implements the full resize -> rescale -> normalize pipeline of the reference's examples")
    if int(resample) not in (BILINEAR, BICUBIC):
        raise ValueError(f"resample must be PIL BILINEAR (2) or BICUBIC (3), got {resample}")
    if len(image_mean) != 3 or len(image_std) != 3:
        raise ValueError("mean must have 3 elements if it is an iterable")
    if not all(image_std):
        raise ValueError("std evaluated to zero, leading to division by zero.")
    f = _size_fields(size if size is not None else {"height": 224, "width": 224}, default_to_square)
    cfg = _lib.PreprocConfig()
    cfg.height, cfg.width, cfg.shortest_edge = f.get("height", 0), f.get("width", 0), f.get("shortest_edge", 0)
    if do_center_crop is None:
        do_center_crop = crop_size is not None
    if do_center_crop:
        c = _size_fields(crop_size if not isinstance(crop_size, int) else (crop_size, crop_size))
        if "height" not in c:
            raise ValueError(f"The size dictionary must have keys 'height' and 'width'. Got {crop_size}")
        cfg.crop_h, cfg.crop_w = c["height"], c["width"]
    cfg.resample = int(resample)
    cfg.rescale_factor = float(rescale_factor)
    cfg.mean = (C.c_float * 3)(*[float(v) for v in image_mean])
    cfg.std = (C.c_float * 3)(*[float(v) for v in image_std])
    return cfg


class ImagePreprocessor:
    """Mirror of `ViTImageProcessor` / `CLIPImageProcessor` / `SiglipImageProcessor` for uint8 RGB batches on the GPU."""

    def __init__(self, size=None, crop_size=None, resample: int = BILINEAR, do_center_crop: Optional[bool] = None,
                 rescale_factor: float = 1 / 255, image_mean: Sequence[float] = (0.5, 0.5, 0.5),
                 image_std: Sequence[float] = (0.5, 0.5, 0.5), do_resize: bool = True, do_rescale: bool = True,
                 do_normalize: bool = True, device: Optional[int] = None, default_to_square: bool = True, **unused):
        cfg = _config(size, crop_size, resample, do_center_crop, rescale_factor, image_mean, image_std, do_resize, do_rescale,
                      do_normalize, default_to_square)
        if not torch.cuda.is_available():
            raise _lib.JimmError("jimm_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
        self.cfg = cfg
        self.handle = C.c_void_p()
        _lib.check(self.lib.jimm_preproc_create(C.byref(cfg), self.device.index, C.byref(self.handle)))

    # ---- stock settings of the three model families (their preprocessor_config.json) ----
    @classmethod
    def vit(cls, size: int = 224, **kw):
        return cls(size={"height": size, "width": size}, resample=BILINEAR, **kw)

    @classmethod
    def siglip(cls, size: int = 224, **kw):
        return cls(size={"height": size, "width": size}, resample=BICUBIC, **kw)

    @classmethod
    def clip(cls, size: int = 224, **kw):
        return cls(size={"shortest_edge": size}, crop_size={"height": size, "width": size}, resample=BICUBIC,
                   image_mean=OPENAI_CLIP_MEAN, image_std=OPENAI_CLIP_STD, **kw)

    @classmethod
    def from_pretrained(cls, path: str, **kw):
        """Read `preprocessor_config.json` from a checkpoint directory (or the file itself)."""
        f = os.path.join(path, "preprocessor_config.json") if os.path.isdir(path) else path
        if not os.path.exists(f):
            raise ValueError(f"preprocessor_config.json not found at {path}")
        with open(f) as fh:
            c = json.load(fh)
        keys = ("size", "crop_size", "resample", "do_center_crop", "rescale_factor", "image_mean", "image_std", "do_resize",
                "do_rescale", "do_normalize")
        args = {k: c[k] for k in keys if k in c and c[k] is not None}
        # integer `size`: CLIPImageProcessor reads it as the shortest edge, ViT / SigLIP processors as a square
        args["default_to_square"] = "clip" not in str(c.get("image_processor_type", "")).lower()
        args.update(kw)
        return cls(**args)

    def output_size(self, height: int, width: int):
        oh, ow = C.c_int(), C.c_int()
        _lib.check(self.lib.jimm_preproc_output_size(self.handle, int(height), int(width), C.byref(oh), C.byref(ow)))
        return oh.value, ow.value

    def __call__(self, images: Union[torch.Tensor, np.ndarray, Sequence], dtype: torch.dtype = torch.float32) -> torch.Tensor:
        """uint8 RGB [B,H,W,3] (or one [H,W,3] image, or a list of images of possibly different sizes) -> CUDA [B,h,w,3]."""
        if dtype not in _OUT_CODE:
            raise ValueError(f"unsupported output dtype {dtype}")
        if isinstance(images, (list, tuple)):
            outs = [self(im, dtype) for im in images]
            return torch.cat(outs, 0)
        x = images if isinstance(images, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(images))
        if x.dtype != torch.uint8:
            raise ValueError(f"expected uint8 RGB images, got {x.dtype}")
        if x.ndim == 3:
            x = x[None]
        if x.ndim != 4 or x.shape[3] != 3:
            raise ValueError(f"expected images of shape [batch, height, width, 3], got {tuple(x.shape)}")
        B, H, W, _ = x.shape
        oh, ow = self.output_size(H, W)
        with torch.cuda.device(self.device):
            xd = x.to(self.device, non_blocking=True).contiguous()
            out = torch.empty((B, oh, ow, 3), dtype=dtype, device=self.device)
            _lib.check(self.lib.jimm_preproc_run(self.handle, C.c_void_p(xd.data_ptr()), B, H, W, C.c_void_p(out.data_ptr()),
                                                 _OUT_CODE[dtype], C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
            xd.record_stream(torch.cuda.current_stream(self.device))
        return out

    def close(self):
        if getattr(self, "handle", None):
            self.lib.jimm_preproc_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def resample_coeffs(in_size: int, out_size: int, resample: int):
    """Host-only: Pillow's window starts, window lengths and fixed-point weights as the library computes them (test hook)."""
    lib = _lib.load()
    ks = C.c_int()
    _lib.check(lib.jimm_k_resample_coeffs(in_size, out_size, resample, C.byref(ks), None, None, None, 0))
    first = np.zeros(out_size, np.int32)
    count = np.zeros(out_size, np.int32)
    kk = np.zeros((out_size, ks.value), np.int32)
    _lib.check(lib.jimm_k_resample_coeffs(in_size, out_size, resample, C.byref(ks), first.ctypes.data_as(C.c_void_p),
                                          count.ctypes.data_as(C.c_void_p), kk.ctypes.data_as(C.c_void_p), kk.size))
    return first, count, kk


FUSED, TWO_PASS = 0, 1


def plan(height: int, width: int, **config):
    """Host-only: how the library runs height x width frames under ImagePreprocessor(**config) -- (path, tier, TY, smem): FUSED with
    TY output rows per CTA and smem bytes of shared memory chosen under budget tier 0 / 1 / 2 (72 / 110 / 200 KB), or TWO_PASS
    (-1, 8, 0).  Raises ValueError for a size the front-end refuses (test hook)."""
    lib = _lib.load()
    cfg = _config(**config)
    path, tier, ty, smem = C.c_int(), C.c_int(), C.c_int(), C.c_longlong()
    _lib.check(lib.jimm_k_preproc_plan(C.byref(cfg), int(height), int(width), C.byref(path), C.byref(tier), C.byref(ty), C.byref(smem)))
    return path.value, tier.value, ty.value, smem.value


def naflex_grid(height: int, width: int, patch_size: int = 16, max_num_patches: int = 256):
    """Host-only: the patch grid (rows, columns) of transformers' Siglip2 size rule (get_image_size_for_max_num_patches) for a
    height x width frame.  Raises ValueError for a frame the front-end refuses or a grid of more than max_num_patches patches."""
    gh, gw = C.c_int(), C.c_int()
    _lib.check(_lib.load().jimm_preproc_naflex_grid(int(patch_size), int(max_num_patches), int(height), int(width), C.byref(gh),
                                                     C.byref(gw)))
    return gh.value, gw.value


class NaFlexPreprocessor:
    """Mirror of transformers' `Siglip2ImageProcessor` (PIL backend) for uint8 RGB frames of any size on the GPU: each frame resized to
    its own patch grid under the max_num_patches budget, rescaled, normalised and written as patch rows, every frame of a call in
    one set of launches (csrc/preprocess.cu).  The result is the processor's three tensors, bit for bit, so it also feeds a
    HuggingFace model."""

    def __init__(self, patch_size: int = 16, max_num_patches: int = 256, resample: int = BILINEAR, rescale_factor: float = 1 / 255,
                 image_mean: Sequence[float] = (0.5, 0.5, 0.5), image_std: Sequence[float] = (0.5, 0.5, 0.5), device: Optional[int] = None,
                 do_resize: bool = True, do_rescale: bool = True, do_normalize: bool = True, **unused):
        if not (do_resize and do_rescale and do_normalize):
            raise ValueError("the GPU front-end implements the full resize -> rescale -> normalize pipeline of the Siglip2 processor")
        if int(resample) not in (BILINEAR, BICUBIC):
            raise ValueError(f"resample must be PIL BILINEAR (2) or BICUBIC (3), got {resample}")
        if len(image_mean) != 3 or len(image_std) != 3:
            raise ValueError("mean must have 3 elements if it is an iterable")
        if not all(image_std):
            raise ValueError("std evaluated to zero, leading to division by zero.")
        if int(patch_size) < 1 or int(max_num_patches) < 1:
            raise ValueError(f"patch_size and max_num_patches must be at least 1, got {patch_size} and {max_num_patches}")
        cfg = _lib.PreprocConfig()
        cfg.resample = int(resample)
        cfg.rescale_factor = float(rescale_factor)
        cfg.mean = (C.c_float * 3)(*[float(v) for v in image_mean])
        cfg.std = (C.c_float * 3)(*[float(v) for v in image_std])
        self.patch_size, self.max_num_patches = int(patch_size), int(max_num_patches)
        if not torch.cuda.is_available():
            raise _lib.JimmError("jimm_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
        self.cfg = cfg
        self.handle = C.c_void_p()
        _lib.check(self.lib.jimm_preproc_create_naflex(C.byref(cfg), self.patch_size, self.device.index, C.byref(self.handle)))

    @classmethod
    def from_pretrained(cls, path: str, **kw):
        """Read a Siglip2 `preprocessor_config.json` from a checkpoint directory (or the file itself)."""
        f = os.path.join(path, "preprocessor_config.json") if os.path.isdir(path) else path
        if not os.path.exists(f):
            raise ValueError(f"preprocessor_config.json not found at {path}")
        with open(f) as fh:
            c = json.load(fh)
        keys = ("patch_size", "max_num_patches", "resample", "rescale_factor", "image_mean", "image_std", "do_resize", "do_rescale",
                "do_normalize")
        args = {k: c[k] for k in keys if k in c and c[k] is not None}
        args.update(kw)
        return cls(**args)

    def grid(self, height: int, width: int, max_num_patches: Optional[int] = None):
        """The (rows, columns) patch grid of a height x width frame (the size rule; host only)."""
        return naflex_grid(height, width, self.patch_size, self.max_num_patches if max_num_patches is None else max_num_patches)

    def __call__(self, frames: Union[torch.Tensor, np.ndarray, Sequence], dtype: torch.dtype = torch.float32,
                 max_num_patches: Optional[int] = None) -> dict:
        """uint8 RGB frames -- a [B, H, W, 3] batch, one [H, W, 3] frame, or a list of [H, W, 3] frames of different sizes, on the host or
        CUDA -- -> {"pixel_values": CUDA [B, max_num_patches, P*P*3] of dtype, "pixel_attention_mask": CUDA int32 [B, max_num_patches],
        "spatial_shapes": CPU int64 [B, 2]}.  max_num_patches: the processor's per-call keyword (default: the constructor's)."""
        if dtype not in _OUT_CODE:
            raise ValueError(f"unsupported output dtype {dtype}")
        N = self.max_num_patches if max_num_patches is None else int(max_num_patches)
        if isinstance(frames, (list, tuple)):
            xs = [f if isinstance(f, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(f)) for f in frames]
            xs = [x[0] if x.ndim == 4 and x.shape[0] == 1 else x for x in xs]
        else:
            x = frames if isinstance(frames, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(frames))
            xs = [x] if x.ndim == 3 else list(x) if x.ndim == 4 else [x]
        for i, x in enumerate(xs):
            if x.dtype != torch.uint8:
                raise ValueError(f"frame {i}: expected uint8 RGB, got {x.dtype}")
            if x.ndim != 3 or x.shape[2] != 3:
                raise ValueError(f"frame {i}: expected shape [height, width, 3], got {tuple(x.shape)}")
        B, P = len(xs), self.patch_size
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device)
            if isinstance(frames, torch.Tensor) and frames.ndim == 4:
                xd = frames.to(self.device, non_blocking=True).contiguous()
                ds = list(xd) if B else []
            else:
                ds = [x.to(self.device, non_blocking=True).contiguous() for x in xs]
            pv = torch.empty((B, N, P * P * 3), dtype=dtype, device=self.device)
            mask = torch.empty((B, N), dtype=torch.int32, device=self.device)
            grid = (C.c_int * max(2 * B, 1))()
            if B:
                _lib.check(self.lib.jimm_preproc_run_naflex(
                    self.handle, (C.c_void_p * B)(*[d.data_ptr() for d in ds]), B, (C.c_int * B)(*[d.shape[0] for d in ds]),
                    (C.c_int * B)(*[d.shape[1] for d in ds]), N, C.c_void_p(pv.data_ptr()), _OUT_CODE[dtype], C.c_void_p(mask.data_ptr()),
                    grid, C.c_void_p(st.cuda_stream)))
                for d in ds:
                    d.record_stream(st)
        shapes = torch.tensor(list(grid)[:2 * B], dtype=torch.int64).reshape(B, 2)
        return {"pixel_values": pv, "pixel_attention_mask": mask, "spatial_shapes": shapes}

    def close(self):
        if getattr(self, "handle", None):
            self.lib.jimm_preproc_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def resample_coeffs_device(in_size: int, out_size: int, resample: int):
    """Pillow's tables as the NaFlex front-end builds them on the GPU (test hook): (first, count, kk) as resample_coeffs returns."""
    lib = _lib.load()
    ks = C.c_int()
    _lib.check(lib.jimm_k_resample_coeffs(in_size, out_size, resample, C.byref(ks), None, None, None, 0))
    first = np.zeros(out_size, np.int32)
    count = np.zeros(out_size, np.int32)
    kk = np.zeros((out_size, ks.value), np.int32)
    _lib.check(lib.jimm_k_resample_coeffs_device(in_size, out_size, resample, first.ctypes.data_as(C.c_void_p),
                                                 count.ctypes.data_as(C.c_void_p), kk.ctypes.data_as(C.c_void_p), kk.size))
    return first, count, kk
