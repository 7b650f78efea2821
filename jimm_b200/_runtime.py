"""Native model handle: drives jimm_model_create -> set_param x N -> finalize, and the forward entry points, for the
Python mirror classes.  PyTorch is used only for device memory, streams and torch.distributed plumbing."""

from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from .nn import LazyParam

_TORCH_TO_CODE = {torch.float32: _lib.F32, torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _as_tensor(x, what: str) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x))
    if hasattr(x, "__dlpack__"):
        return torch.from_dlpack(x)
    return torch.as_tensor(np.asarray(x))


class PendingResult:
    """Result of an asynchronously dispatched forward: `.result()` waits for that call's work only."""

    def __init__(self, tensor: torch.Tensor, event, keep=None):
        self._tensor, self._event, self._keep = tensor, event, keep

    def done(self) -> bool:
        return self._event is None or self._event.query()

    def result(self) -> torch.Tensor:
        if self._event is not None:
            self._event.synchronize()
            self._event = self._keep = None
        return self._tensor


class NativeModel:
    """One opaque jimm_model_t on one GPU."""

    def __init__(self, cfg: _lib.Config, params: Dict[str, torch.Tensor], max_batch: int, device: Optional[int] = None,
                 max_tokens: int = 0):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.JimmError("jimm_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        self.cfg = cfg
        self.handle = C.c_void_p()
        _lib.check(self.lib.jimm_model_create(C.byref(cfg), self.device_index, C.byref(self.handle)))
        try:
            keep = []  # the borrowed buffers stay alive until finalize has streamed them to the GPU
            for name, t in params.items():
                flags = 0
                if isinstance(t, LazyParam):  # a view of checkpoint memory, possibly the (out, in) transpose of the flax kernel
                    shape_t, flags, t = t.shape, (_lib.PARAM_TRANSPOSED if t.transposed else 0), t.base
                else:
                    shape_t = tuple(t.shape)
                t = t.detach()
                if t.dtype not in _TORCH_TO_CODE:
                    t = t.to(torch.float32)
                if t.is_cuda or not t.is_contiguous():
                    t = t.contiguous().cpu()
                keep.append(t)
                shape = (C.c_int64 * max(len(shape_t), 1))(*shape_t)
                _lib.check(self.lib.jimm_model_set_param_ref(self.handle, name.encode(), C.c_void_p(t.data_ptr()), shape, len(shape_t),
                                                              _TORCH_TO_CODE[t.dtype], flags))
            if max_tokens > 0:
                _lib.check(self.lib.jimm_model_set_max_tokens(self.handle, int(max_tokens)))
            _lib.check(self.lib.jimm_model_finalize(self.handle, int(max_batch)))
        except Exception:
            self.lib.jimm_model_destroy(self.handle)
            self.handle = None
            raise
        self.max_batch = int(max_batch)
        vo, to = C.c_int(), C.c_int()
        _lib.check(self.lib.jimm_model_output_dim(self.handle, C.byref(vo), C.byref(to)))
        self.vision_out, self.text_out = vo.value, to.value
        self._comm = None
        self.preproc = None  # ImagePreprocessor for uint8 inputs (set by the owning model's set_preprocessor)

    def images_per_call(self, height: int, width: int) -> int:
        """Images of height x width one chunk of an interpolate_pos_encoding call runs on this handle (0: one does not fit)."""
        n = C.c_int()
        _lib.check(self.lib.jimm_model_images_per_call(self.handle, int(height), int(width), C.byref(n)))
        return n.value

    def side_stream(self) -> torch.cuda.Stream:
        """Copy stream for host inputs of the multi-GPU dual path."""
        if getattr(self, "_side", None) is None:
            self._side = torch.cuda.Stream(self.device)
        return self._side

    def close(self):
        if getattr(self, "handle", None):
            self.lib.jimm_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- input normalisation ----
    def _prep_images(self, x, interpolate: bool = False) -> torch.Tensor:
        """interpolate: HF's interpolate_pos_encoding -- any image size of at least one patch is accepted."""
        x = _as_tensor(x, "image")
        if x.ndim != 4:
            raise ValueError(f"expected images of shape [batch, height, width, channels], got {tuple(x.shape)}")
        c = self.cfg
        if x.dtype == torch.uint8:
            # raw RGB frames: need the attached image front-end (model.set_preprocessor); any frame size it maps to the model's input
            if self.preproc is None:
                raise ValueError("uint8 images need an image front-end: call model.set_preprocessor(ImagePreprocessor...) first, "
                                 "or pass normalised float pixel values")
            if x.shape[3] != 3:
                raise ValueError(f"expected uint8 RGB frames [B,H,W,3], got {tuple(x.shape)}")
            oh, ow = self.preproc.output_size(x.shape[1], x.shape[2])
            if interpolate:
                self._check_grid(oh, ow)
            elif (oh, ow) != (c.img_size, c.img_size):
                raise ValueError(f"the image front-end maps {x.shape[1]}x{x.shape[2]} frames to {oh}x{ow}, the model takes {c.img_size}x{c.img_size}")
            return x.contiguous()
        if interpolate:
            if x.shape[3] != c.in_ch:
                raise ValueError(f"expected NHWC images [B,H,W,{c.in_ch}], got {tuple(x.shape)}")
            self._check_grid(x.shape[1], x.shape[2])
        elif x.shape[1] != c.img_size or x.shape[2] != c.img_size or x.shape[3] != c.in_ch:
            raise ValueError(f"expected NHWC images [B,{c.img_size},{c.img_size},{c.in_ch}], got {tuple(x.shape)}")
        if x.dtype not in _TORCH_TO_CODE:
            x = x.to(torch.float32)
        return x.contiguous()

    def _check_grid(self, h: int, w: int):
        P = self.cfg.patch
        if h < P or w < P:
            raise ValueError(f"interpolate_pos_encoding: a {h}x{w} image is smaller than one {P}x{P} patch")

    def _off_grid(self, x: torch.Tensor, interpolate: bool) -> bool:
        """True when an interpolate_pos_encoding call's (prepared) images are not the native size: the *_hw entry points run it."""
        if not interpolate:
            return False
        hw = self.preproc.output_size(x.shape[1], x.shape[2]) if x.dtype == torch.uint8 else (x.shape[1], x.shape[2])
        return tuple(hw) != (self.cfg.img_size, self.cfg.img_size)

    def _device_images(self, x: torch.Tensor) -> torch.Tensor:
        """Prepared images on this GPU in a tower input type (uint8 frames through the image front-end)."""
        xd = x.to(self.device, non_blocking=True)
        return self.preproc(xd, dtype=self._operand_dtype()) if xd.dtype == torch.uint8 else xd

    def _prep_ids(self, t) -> torch.Tensor:
        t = _as_tensor(t, "text")
        if t.ndim != 2:
            raise ValueError(f"expected token ids of shape [batch, context_length], got {tuple(t.shape)}")
        return t.to(torch.int32).contiguous()

    # ---- forward ----
    def vision(self, x, encode: bool = False, interpolate: bool = False) -> torch.Tensor:
        """VisionTransformer.__call__ / encode_image.  CUDA input -> async CUDA output; host input -> host output.
        interpolate: HF's interpolate_pos_encoding (images of any size; see jimm_vit_forward_hw)."""
        x = self._prep_images(x, interpolate)
        if self._off_grid(x, interpolate):
            return self._vision_hw(x, encode)
        B = x.shape[0]
        fn_dev = self.lib.jimm_encode_image if encode else self.lib.jimm_vit_forward
        if x.is_cuda:
            if x.dtype == torch.uint8:  # device frames: front-end kernel, then the tower, on the current stream
                x = self.preproc(x, dtype=self._operand_dtype())
            with torch.cuda.device(self.device):
                out = torch.empty((B, self.vision_out), dtype=torch.float32, device=self.device)
                _lib.check(fn_dev(self.handle, C.c_void_p(x.data_ptr()), _TORCH_TO_CODE[x.dtype], B, C.c_void_p(out.data_ptr()),
                                  C.c_void_p(_stream_ptr(self.device))))
            return out
        return self._vision_host(x, encode).result()

    def vision_async(self, x, encode: bool = False, interpolate: bool = False) -> "PendingResult":
        """Host input: enqueue H2D + forward + D2H and return without synchronising (JAX-style asynchronous dispatch);
        `.result()` waits for this call only.  Back-to-back calls pipeline: the copies of call k+1 run under the towers of
        call k.  The caller keeps `x` alive and unmodified until the result is taken.  Host images off the native size
        (interpolate=True) run synchronously."""
        x = self._prep_images(x, interpolate)
        if x.is_cuda or self._off_grid(x, interpolate):
            return PendingResult(self.vision(x, encode, interpolate), None)
        return self._vision_host(x, encode)

    def _vision_hw(self, x: torch.Tensor, encode: bool) -> torch.Tensor:
        """A vision call at a size other than the native one: host images are copied to the GPU here and the result back."""
        B = x.shape[0]
        fn = self.lib.jimm_encode_image_hw if encode else self.lib.jimm_vit_forward_hw
        with torch.cuda.device(self.device):
            xd = self._device_images(x)
            out = torch.empty((B, self.vision_out), dtype=torch.float32, device=self.device)
            _lib.check(fn(self.handle, C.c_void_p(xd.data_ptr()), _TORCH_TO_CODE[xd.dtype], B, xd.shape[1], xd.shape[2],
                          C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr(self.device))))
        return out if x.is_cuda else out.cpu()

    # ---- packed lists of images of different sizes (jimm_vit_forward_packed) ----
    def _prep_image_list(self, images, interpolate: bool):
        """Each element of a list / tuple as one prepared image [H, W, C] (a leading batch dimension of 1 is dropped), all of one
        dtype and on one device; the checks of _prep_images, per image."""
        xs = []
        for i, x in enumerate(images):
            x = _as_tensor(x, "image")
            if x.ndim == 4 and x.shape[0] == 1:
                x = x[0]
            if x.ndim != 3:
                raise ValueError(f"image {i} of the list: expected [height, width, channels] or [1, height, width, channels], got {tuple(x.shape)}")
            xs.append(x)
        if len({x.dtype for x in xs}) > 1:
            raise ValueError(f"the images of a list must share one dtype, got {sorted({str(x.dtype) for x in xs})}")
        if len({x.device for x in xs}) > 1:
            raise ValueError(f"the images of a list must be on one device, got {sorted({str(x.device) for x in xs})}")
        return [self._prep_images(x[None], interpolate)[0] for x in xs]

    def _vision_packed_dev(self, images, encode: bool, interpolate: bool):
        """The rows of a list of images on this GPU (fp32 [len, out_dim]) and whether the inputs were host memory."""
        xs = self._prep_image_list(images, interpolate)
        B = len(xs)
        host = B > 0 and not xs[0].is_cuda
        with torch.cuda.device(self.device):
            out = torch.empty((B, self.vision_out), dtype=torch.float32, device=self.device)
            if B == 0:
                return out, True
            # uint8 frames go through the image front-end one at a time (their output sizes differ)
            xd = [self._device_images(x[None])[0].contiguous() for x in xs]
            ptrs = (C.c_void_p * B)(*[x.data_ptr() for x in xd])
            hs = (C.c_int * B)(*[x.shape[0] for x in xd])
            ws = (C.c_int * B)(*[x.shape[1] for x in xd])
            fn = self.lib.jimm_encode_image_packed if encode else self.lib.jimm_vit_forward_packed
            _lib.check(fn(self.handle, ptrs, _TORCH_TO_CODE[xd[0].dtype], B, hs, ws, C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr(self.device))))
            if not host:
                cur = torch.cuda.current_stream(self.device)
                for x in xd:  # freshly made device copies are freed only after the call's work
                    x.record_stream(cur)
        return out, host

    def vision_packed(self, images, encode: bool = False, interpolate: bool = False) -> torch.Tensor:
        """A list / tuple of images of different sizes in one call: their tokens packed into one stream (variable-length
        attention).  Row i is the result of the call on images[i] alone.  CUDA inputs -> CUDA output without a host synchronisation;
        host inputs -> host output."""
        out, host = self._vision_packed_dev(images, encode, interpolate)
        return out.cpu() if host else out

    def dual_packed(self, images, text, interpolate: bool = False) -> torch.Tensor:
        """CLIP.__call__ / SigLIP.__call__ on a list of images of different sizes."""
        ids = self._prep_ids(text)
        ie, host = self._vision_packed_dev(images, True, interpolate)
        host = host and not ids.is_cuda
        with torch.cuda.device(self.device):
            te = self.text(ids.to(self.device, non_blocking=True))
            out = self.logits(ie, te)
        return out.cpu() if host else out

    def _operand_dtype(self) -> torch.dtype:
        return {_lib.F32: torch.float32, _lib.F16: torch.float16, _lib.BF16: torch.bfloat16, _lib.F8E4M3: torch.float16}[self.cfg.compute_dtype]

    def _vision_host(self, x: torch.Tensor, encode: bool) -> "PendingResult":
        B = x.shape[0]
        fn_dev = self.lib.jimm_encode_image if encode else self.lib.jimm_vit_forward
        # host path: H2D + forward + D2H enqueued by the library on the current stream
        with torch.cuda.device(self.device):
            # fresh pinned result (torch's caching host allocator makes this cheap); no CPU-side tensor op on this path: an
            # intra-op OpenMP team on a CPU-quota-limited box costs milliseconds
            out = torch.empty((B, self.vision_out), dtype=torch.float32, pin_memory=True)
            cur = torch.cuda.current_stream(self.device)
            if x.dtype == torch.uint8 and not encode:
                # raw frames: bytes over PCIe, front-end + tower in the library's sliced copy/compute pipeline
                _lib.check(self.lib.jimm_vit_forward_host_u8(self.handle, self.preproc.handle, C.c_void_p(x.data_ptr()), B, x.shape[1], x.shape[2],
                                                             C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr(self.device))))
            elif encode:
                xd = x.to(self.device, non_blocking=True)
                if xd.dtype == torch.uint8:
                    xd = self.preproc(xd, dtype=self._operand_dtype())
                od = torch.empty((B, self.vision_out), dtype=torch.float32, device=self.device)
                _lib.check(fn_dev(self.handle, C.c_void_p(xd.data_ptr()), _TORCH_TO_CODE[xd.dtype], B, C.c_void_p(od.data_ptr()),
                                  C.c_void_p(_stream_ptr(self.device))))
                out.copy_(od, non_blocking=True)
            else:
                _lib.check(self.lib.jimm_vit_forward_host(self.handle, C.c_void_p(x.data_ptr()), _TORCH_TO_CODE[x.dtype], B,
                                                          C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr(self.device))))
            ev = torch.cuda.Event()
            ev.record(cur)
        return PendingResult(out, ev, keep=x)

    def text(self, ids) -> torch.Tensor:
        ids = self._prep_ids(ids)
        host = not ids.is_cuda
        B, T = ids.shape
        with torch.cuda.device(self.device):
            idd = ids.to(self.device, non_blocking=True)
            out = torch.empty((B, self.text_out), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.jimm_encode_text(self.handle, C.c_void_p(idd.data_ptr()), B, T, C.c_void_p(out.data_ptr()),
                                                 C.c_void_p(_stream_ptr(self.device))))
            if host:
                out = out.cpu()
        return out

    def dual_encode(self, x: torch.Tensor, ids: torch.Tensor):
        """encode_image + encode_text of device-resident inputs with the two towers running concurrently (jimm_dual_encode)."""
        Bi, (Bt, T) = x.shape[0], ids.shape
        with torch.cuda.device(self.device):
            if x.dtype == torch.uint8:  # raw frames: the image front-end first (model.set_preprocessor)
                x = self.preproc(x, dtype=self._operand_dtype())
            ie = torch.empty((Bi, self.vision_out), dtype=torch.float32, device=self.device)
            te = torch.empty((Bt, self.text_out), dtype=torch.float32, device=self.device)
            # images of the native size run exactly as jimm_dual_encode; others only reach here with interpolate_pos_encoding
            _lib.check(self.lib.jimm_dual_encode_hw(self.handle, C.c_void_p(x.data_ptr()), _TORCH_TO_CODE[x.dtype], Bi, x.shape[1], x.shape[2],
                                                    C.c_void_p(ids.data_ptr()), Bt, T, C.c_void_p(ie.data_ptr()), C.c_void_p(te.data_ptr()),
                                                    C.c_void_p(_stream_ptr(self.device))))
        return ie, te

    def logits(self, img_e: torch.Tensor, txt_e: torch.Tensor) -> torch.Tensor:
        with torch.cuda.device(self.device):
            img_e = img_e.to(self.device, torch.float32).contiguous()
            txt_e = txt_e.to(self.device, torch.float32).contiguous()
            Bi, Bt = img_e.shape[0], txt_e.shape[0]
            out = torch.empty((Bi, Bt), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.jimm_contrastive_logits(self.handle, C.c_void_p(img_e.data_ptr()), Bi, C.c_void_p(txt_e.data_ptr()), Bt,
                                                        C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr(self.device))))
        return out

    def dual(self, image, text, interpolate: bool = False) -> torch.Tensor:
        """CLIP.__call__ / SigLIP.__call__ on one GPU."""
        x = self._prep_images(image, interpolate)
        ids = self._prep_ids(text)
        Bi, (Bt, T) = x.shape[0], ids.shape
        with torch.cuda.device(self.device):
            if self._off_grid(x, interpolate):
                xd, idd = self._device_images(x), ids.to(self.device, non_blocking=True)
                out = torch.empty((Bi, Bt), dtype=torch.float32, device=self.device)
                _lib.check(self.lib.jimm_dual_forward_hw(self.handle, C.c_void_p(xd.data_ptr()), _TORCH_TO_CODE[xd.dtype], Bi, xd.shape[1],
                                                         xd.shape[2], C.c_void_p(idd.data_ptr()), Bt, T, C.c_void_p(out.data_ptr()),
                                                         C.c_void_p(_stream_ptr(self.device))))
                return out if (x.is_cuda or ids.is_cuda) else out.cpu()
            if x.dtype == torch.uint8:
                # raw RGB frames (model.set_preprocessor): bytes over PCIe, the image front-end on the GPU, then both towers concurrently
                host_in = not x.is_cuda and not ids.is_cuda
                xd = self.preproc(x.to(self.device, non_blocking=True), dtype=self._operand_dtype())
                idd = ids.to(self.device, non_blocking=True)
                out = torch.empty((Bi, Bt), dtype=torch.float32, device=self.device)
                _lib.check(self.lib.jimm_dual_forward(self.handle, C.c_void_p(xd.data_ptr()), _TORCH_TO_CODE[xd.dtype], Bi,
                                                      C.c_void_p(idd.data_ptr()), Bt, T, C.c_void_p(out.data_ptr()),
                                                      C.c_void_p(_stream_ptr(self.device))))
                if not host_in:
                    return out
                out_h = torch.empty((Bi, Bt), dtype=torch.float32, pin_memory=True)
                out_h.copy_(out, non_blocking=True)
                torch.cuda.current_stream(self.device).synchronize()
                return out_h
            if not x.is_cuda and not ids.is_cuda:
                out = torch.empty((Bi, Bt), dtype=torch.float32, pin_memory=True)
                _lib.check(self.lib.jimm_dual_forward_host(self.handle, C.c_void_p(x.data_ptr()), _TORCH_TO_CODE[x.dtype], Bi,
                                                           C.c_void_p(ids.data_ptr()), Bt, T, C.c_void_p(out.data_ptr()),
                                                           C.c_void_p(_stream_ptr(self.device))))
                torch.cuda.current_stream(self.device).synchronize()
                return out
            xd, idd = x.to(self.device, non_blocking=True), ids.to(self.device, non_blocking=True)
            out = torch.empty((Bi, Bt), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.jimm_dual_forward(self.handle, C.c_void_p(xd.data_ptr()), _TORCH_TO_CODE[xd.dtype], Bi,
                                                  C.c_void_p(idd.data_ptr()), Bt, T, C.c_void_p(out.data_ptr()),
                                                  C.c_void_p(_stream_ptr(self.device))))
        return out

    # ---- multi-GPU contrastive head (one process per GPU; torch.distributed is the control plane) ----
    def comm_setup(self, max_rows_per_rank: int, group=None):
        import torch.distributed as dist

        rank, world = dist.get_rank(group), dist.get_world_size(group)
        handle = C.create_string_buffer(64)
        _lib.check(self.lib.jimm_comm_init(self.handle, rank, world, int(max_rows_per_rank), handle))
        handles = [None] * world
        dist.all_gather_object(handles, bytes(handle.raw), group=group)
        _lib.check(self.lib.jimm_comm_connect(self.handle, b"".join(handles)))
        dist.barrier(group)
        self._comm = (rank, world, int(max_rows_per_rank))

    def comm_logits(self, img_e: torch.Tensor, txt_e: torch.Tensor) -> torch.Tensor:
        """Fused normalise + NVLink peer scatter + local logits row block [B_local, world*B_local]."""
        if self._comm is None:
            raise _lib.JimmError("comm_setup() has not been called")
        rank, world, _ = self._comm
        with torch.cuda.device(self.device):
            img_e = img_e.to(self.device, torch.float32).contiguous()
            txt_e = txt_e.to(self.device, torch.float32).contiguous()
            B = img_e.shape[0]
            if txt_e.shape[0] != B:
                raise ValueError("multi-GPU contrastive head needs equal image/text batch per rank")
            out = torch.empty((B, world * B), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.jimm_comm_contrastive_logits(self.handle, C.c_void_p(img_e.data_ptr()), C.c_void_p(txt_e.data_ptr()), B,
                                                             C.c_void_p(out.data_ptr()), C.c_void_p(_stream_ptr(self.device))))
        return out


class NativeSubModule:
    """Native handle of a bare Transformer / TransformerEncoder (kind ENCODER) or MultiHeadAttentionPoolingHead (kind MAPHEAD): the
    same kernels and block orchestration as inside a tower, on [batch, seq, hidden] activations."""

    def __init__(self, cfg: _lib.Config, params: Dict[str, torch.Tensor], max_batch: int):
        self.native = NativeModel(cfg, params, max_batch)
        self.kind, self.max_seq, self.max_batch, self.D = cfg.kind, cfg.ctx_len, int(max_batch), cfg.v_width

    def close(self):
        self.native.close()

    def __call__(self, x) -> torch.Tensor:
        n = self.native
        x = _as_tensor(x, "activations")
        if x.ndim != 3 or x.shape[2] != self.D:
            raise ValueError(f"expected activations of shape [batch, seq, {self.D}], got {tuple(x.shape)}")
        host = not x.is_cuda
        B, S, D = x.shape
        with torch.cuda.device(n.device):
            xd = x.to(n.device, torch.float32, non_blocking=True).contiguous()
            st = C.c_void_p(_stream_ptr(n.device))
            if self.kind == _lib.KIND_ENCODER:
                out = torch.empty((B, S, D), dtype=torch.float32, device=n.device)
                _lib.check(n.lib.jimm_encoder_forward(n.handle, C.c_void_p(xd.data_ptr()), B, S, C.c_void_p(out.data_ptr()), st))
            else:
                out = torch.empty((B, D), dtype=torch.float32, device=n.device)
                _lib.check(n.lib.jimm_map_head_forward(n.handle, C.c_void_p(xd.data_ptr()), B, S, C.c_void_p(out.data_ptr()), st))
            xd.record_stream(torch.cuda.current_stream(n.device))
        return out.cpu() if host else out


def activation(x, act: int) -> torch.Tensor:
    """Elementwise activation kernel (1 tanh-GELU, 2 QuickGELU) on a CUDA tensor; fp32 result."""
    x = _as_tensor(x, "x")
    if not x.is_cuda:
        raise _lib.JimmError("jimm_b200 runs on CUDA tensors only (there is no CPU fallback)")
    lib = _lib.load()
    with torch.cuda.device(x.device):
        xd = x.to(torch.float32).contiguous()
        y = torch.empty_like(xd)
        _lib.check(lib.jimm_k_activation(C.c_void_p(xd.data_ptr()), C.c_void_p(y.data_ptr()), xd.numel(), int(act), C.c_void_p(_stream_ptr(x.device))))
    return y


def grid_tokens(cfg: _lib.Config, height: int, width: int) -> int:
    """Tokens per image of a vision tower on height x width images: the patches (trailing pixels dropped) and the CLS token."""
    return (int(height) // cfg.patch) * (int(width) // cfg.patch) + (1 if cfg.pooling == _lib.POOL_CLS else 0)


def default_max_batch() -> int:
    return int(os.environ.get("JIMM_MAX_BATCH", "256"))
