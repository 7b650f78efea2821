"""Native model handle: drives jimm_model_create -> set_param x N -> finalize, and the forward entry points, for the
Python mirror classes.  PyTorch is used only for device memory, streams and torch.distributed plumbing."""

from __future__ import annotations

import ctypes as C
import math
import numbers
import os
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib
from .nn import LazyParam

_TORCH_TO_CODE = {torch.float32: _lib.F32, torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}


def _as_tensor(x) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x))
    if hasattr(x, "__dlpack__"):
        return torch.from_dlpack(x)
    return torch.as_tensor(np.asarray(x))


def _call(lib, device: torch.device, name: str, *args):
    """Library entry point `name` on `args` and the current stream of `device`, with `device` current: tensors are passed as their
    data pointers, torch dtypes as dtype codes."""
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else _TORCH_TO_CODE[a] if isinstance(a, torch.dtype) else a for a in args]
    with torch.cuda.device(device):
        _lib.check(getattr(lib, name)(*args, torch.cuda.current_stream(device).cuda_stream))


class Images(NamedTuple):
    """The images of one vision call, checked and prepared once (prep_images)."""

    x: Union[torch.Tensor, List[torch.Tensor]]  # [B, H, W, C], or a list of [H, W, C], or NaFlex patch rows [B, N, P*P*C] (grid)
    host: bool  # host memory: the result goes back to the host
    u8: bool  # raw RGB frames for the image front-end
    hw: Optional[Tuple[int, int]]  # the (height, width) the tower sees; for a list the one with the most tokens (None: empty list)
    trained: bool  # hw is the trained size
    grid: Optional[List[Tuple[int, int]]] = None  # NaFlex patch rows: each sample's patch grid (rows, columns)


def _prep_batch(x, cfg: _lib.Config, preproc, interpolate: bool):
    """One [B, H, W, C] batch, checked and made contiguous, and the (height, width) the tower sees."""
    x = _as_tensor(x)
    if x.ndim != 4:
        raise ValueError(f"expected images of shape [batch, height, width, channels], got {tuple(x.shape)}")
    _, h, w, ch = x.shape
    S = cfg.img_size
    if x.dtype == torch.uint8:
        # raw RGB frames: need the attached image front-end (model.set_preprocessor); any frame size it maps to the model's input
        if preproc is None:
            raise ValueError("uint8 images need an image front-end: call model.set_preprocessor(ImagePreprocessor...) first, "
                             "or pass normalised float pixel values")
        if ch != 3:
            raise ValueError(f"expected uint8 RGB frames [B,H,W,3], got {tuple(x.shape)}")
        hw = preproc.output_size(h, w)
        if not interpolate and hw != (S, S):
            raise ValueError(f"the image front-end maps {h}x{w} frames to {hw[0]}x{hw[1]}, the model takes {S}x{S}")
    else:
        if interpolate and ch != cfg.in_ch:
            raise ValueError(f"expected NHWC images [B,H,W,{cfg.in_ch}], got {tuple(x.shape)}")
        if not interpolate and (h != S or w != S or ch != cfg.in_ch):
            raise ValueError(f"expected NHWC images [B,{S},{S},{cfg.in_ch}], got {tuple(x.shape)}")
        hw = (h, w)
        if x.dtype not in _TORCH_TO_CODE:
            x = x.to(torch.float32)
    if interpolate and min(hw) < cfg.patch:
        raise ValueError(f"interpolate_pos_encoding: a {hw[0]}x{hw[1]} image is smaller than one {cfg.patch}x{cfg.patch} patch")
    return x.contiguous(), hw


def prep_images(images, cfg: _lib.Config, preproc, interpolate: bool) -> Images:
    """The input step of every vision call: a [B, H, W, C] batch, or a list / tuple of [H, W, C] (or [1, H, W, C]) images of one dtype
    on one device, checked against the model and the image front-end `preproc`.  interpolate: HF's interpolate_pos_encoding -- any
    image size of at least one patch is accepted."""
    if not isinstance(images, (list, tuple)):
        x, hw = _prep_batch(images, cfg, preproc, interpolate)
        return Images(x, not x.is_cuda, x.dtype == torch.uint8, hw, hw == (cfg.img_size, cfg.img_size))
    xs = []
    for i, x in enumerate(images):
        x = _as_tensor(x)
        if x.ndim == 4 and x.shape[0] == 1:
            x = x[0]
        if x.ndim != 3:
            raise ValueError(f"image {i} of the list: expected [height, width, channels] or [1, height, width, channels], got {tuple(x.shape)}")
        xs.append(x)
    if len({x.dtype for x in xs}) > 1:
        raise ValueError(f"the images of a list must share one dtype, got {sorted({str(x.dtype) for x in xs})}")
    if len({x.device for x in xs}) > 1:
        raise ValueError(f"the images of a list must be on one device, got {sorted({str(x.device) for x in xs})}")
    prepped = [_prep_batch(x[None], cfg, preproc, interpolate) for x in xs]
    hw = max((hw for _, hw in prepped), key=lambda s: grid_tokens(cfg, *s), default=None)
    xs = [x[0] for x, _ in prepped]
    return Images(xs, not xs or not xs[0].is_cuda, bool(xs) and xs[0].dtype == torch.uint8, hw, hw == (cfg.img_size, cfg.img_size))


def prep_patches(pixel_values, spatial_shapes, pixel_attention_mask, cfg: _lib.Config) -> Images:
    """The input step of a SigLIP 2 NaFlex call on the HF processor's output: pixel_values [B, N, P*P*C] (each row a patch flattened in
    (py, px, c) order), spatial_shapes [B, 2] integer (patch rows, patch columns) with 1 <= rows * columns <= N, and optionally
    pixel_attention_mask [B, N], which must be the prefix mask the shapes imply (sample b's first rows * columns entries set).  The
    masked rows are never read, so the mask itself is not needed."""
    x = _as_tensor(pixel_values)
    K = cfg.patch * cfg.patch * cfg.in_ch
    if x.ndim != 3 or x.shape[2] != K:
        raise ValueError(f"expected pixel_values of shape [batch, max_num_patches, {K}] (patch {cfg.patch}, {cfg.in_ch} channels), "
                         f"got {tuple(x.shape)}")
    B, N = x.shape[0], x.shape[1]
    ss = _as_tensor(spatial_shapes)
    if tuple(ss.shape) != (B, 2) or ss.dtype.is_floating_point or ss.dtype.is_complex or ss.dtype == torch.bool:
        raise ValueError(f"expected integer spatial_shapes of shape [{B}, 2] (patch rows, patch columns), got {tuple(ss.shape)} {ss.dtype}")
    grid = [(int(h), int(w)) for h, w in ss.tolist()]
    for i, (h, w) in enumerate(grid):
        if h < 1 or w < 1 or h * w > N:
            raise ValueError(f"sample {i}: spatial shape {h}x{w} needs 1 .. {N} (max_num_patches) patch rows")
    if pixel_attention_mask is not None:
        mk = _as_tensor(pixel_attention_mask)
        n = torch.tensor([h * w for h, w in grid], dtype=torch.long)
        if tuple(mk.shape) != (B, N) or not torch.equal(mk.cpu() != 0, torch.arange(N)[None, :] < n[:, None]):
            raise ValueError("pixel_attention_mask is not the mask spatial_shapes implies (each sample's first rows * columns patches)")
    if x.dtype not in _TORCH_TO_CODE:
        x = x.to(torch.float32)
    hw = max(((h * cfg.patch, w * cfg.patch) for h, w in grid), key=lambda s: grid_tokens(cfg, *s), default=None)
    return Images(x.contiguous(), not x.is_cuda, False, hw, False, grid)


class Texts(NamedTuple):
    """The token sequences of one text call on a list, checked and concatenated once (prep_texts)."""

    ids: torch.Tensor  # int32 [sum of the lengths]: the sequences one after another, on the device they came from
    lens: List[int]
    host: bool  # host memory: the result goes back to the host


def prep_texts(texts, context_length: int) -> Texts:
    """The input step of a text call on a list / tuple of token sequences of different lengths: each a 1-D (or [1, L]) integer torch
    tensor (CUDA or host), numpy array or Python list of ints, 1 <= L <= context_length, all on one device.  They are concatenated
    into one int32 tensor on that device, so host input crosses to the GPU in one copy."""
    # A zero-shot classifier passes tens of thousands of short prompts: the per-sequence work stays in Python attribute reads, and the
    # concatenation and the cast to int32 are one operation each for the whole list.
    xs, lens = [], []
    for i, t in enumerate(texts):
        t = _as_tensor(t)
        if t.ndim == 2 and t.shape[0] == 1:
            t = t[0]
        if t.ndim != 1:
            raise ValueError(f"sequence {i} of the list: expected token ids of shape [length] or [1, length], got {tuple(t.shape)}")
        n = t.shape[0]
        if not 1 <= n <= context_length:
            raise ValueError(f"sequence {i} of the list: length {n} outside 1 .. context_length={context_length}")
        xs.append(t)
        lens.append(int(n))
    for i, t in enumerate(xs):
        if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
            raise ValueError(f"sequence {i} of the list: token ids must be integers, got {t.dtype}")
    if len({x.device for x in xs}) > 1:
        raise ValueError(f"the sequences of a list must be on one device, got {sorted({str(x.device) for x in xs})}")
    ids = torch.cat(xs).to(torch.int32) if xs else torch.empty(0, dtype=torch.int32)
    return Texts(ids.contiguous(), lens, not ids.is_cuda)


_TOKEN_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


class TokenLayers(NamedTuple):
    """The requests of a per-token call (prep_layers) or of an attention call (prep_blocks), checked once."""

    codes: List[int]  # the distinct requests as the library takes them: layers 0 .. L or LAYER_FINAL; blocks 0 .. L-1 or ATTN_MAP
    index: List[int]  # request i is codes[index[i]]
    single: bool  # one request (an int or None), not a list / tuple
    dtype: torch.dtype


def prep_layers(layers, num_layers: int, dtype) -> TokenLayers:
    """The layer step of a per-token call on a tower of num_layers blocks: `layers` is one request or a list / tuple of them, each an int
    k in [-(L+1), L] (x_k, the residual stream after k blocks, negative k counting from the end as Python indexing does: -1 is x_L) or
    None (the final-normed tokens); dtype the output type, float32, float16 or bfloat16."""
    L = int(num_layers)
    if dtype not in _TOKEN_DTYPES:
        raise ValueError(f"hidden states come as torch.float32, torch.float16 or torch.bfloat16, got dtype={dtype}")
    single = layers is None or not isinstance(layers, (list, tuple))
    reqs = [layers] if single else list(layers)
    if not reqs:
        raise ValueError("layers: an empty list requests nothing; pass an int, None or a non-empty list of them")
    codes, index = [], []
    for k in reqs:
        if k is None:
            c = _lib.LAYER_FINAL
        elif isinstance(k, (int, np.integer)) and not isinstance(k, bool):
            k = int(k)
            if not -(L + 1) <= k <= L:
                raise ValueError(f"layer {k} outside [-{L + 1}, {L}] for a tower of {L} blocks (0 is the embeddings, {L} the last block)")
            c = k % (L + 1)
        else:
            raise ValueError(f"a layer request is an int or None, got {k!r}")
        if c not in codes:
            codes.append(c)
        index.append(codes.index(c))
    return TokenLayers(codes, index, single, dtype)


def prep_blocks(blocks, num_layers: int, dtype, map_head: bool) -> TokenLayers:
    """The block step of an attention call on a tower of num_layers blocks: `blocks` is an int k in [-L, L-1] (block k's self-attention
    weights, negative k counting from the end), "map" (the MAP head's probe weights; map_head: the tower has one), None (every block in
    order, HF's `attentions` tuple, "map" not included) or a list / tuple of these; dtype the output type, float32, float16 or bfloat16.
    One int or "map" gives one result; None or a list gives a tuple."""
    L = int(num_layers)
    if dtype not in _TOKEN_DTYPES:
        raise ValueError(f"attention weights come as torch.float32, torch.float16 or torch.bfloat16, got dtype={dtype}")
    single = blocks is not None and not isinstance(blocks, (list, tuple))
    reqs = [blocks] if single else list(range(L)) if blocks is None else list(blocks)
    if not reqs:
        raise ValueError("blocks: an empty list requests nothing; pass an int, \"map\", None or a non-empty list of them")
    codes, index = [], []
    for k in reqs:
        if isinstance(k, str) and k == "map":
            if not map_head:
                raise ValueError('blocks="map": the tower has no MAP head (CLS-pooled vision towers and text towers)')
            c = _lib.ATTN_MAP
        elif isinstance(k, (int, np.integer)) and not isinstance(k, bool):
            k = int(k)
            if not -L <= k <= L - 1:
                raise ValueError(f"block {k} outside [-{L}, {L - 1}] for a tower of {L} blocks")
            c = k % L
        else:
            raise ValueError(f'a block request is an int or "map" (or None for every block, alone), got {k!r}')
        if c not in codes:
            codes.append(c)
        index.append(codes.index(c))
    return TokenLayers(codes, index, single, dtype)


def prep_ids(t) -> torch.Tensor:
    """A [B, T] token-id tensor as the library takes it: int32, contiguous."""
    t = _as_tensor(t)
    if t.ndim != 2:
        raise ValueError(f"expected token ids of shape [batch, context_length], got {tuple(t.shape)}")
    return t.to(torch.int32).contiguous()


def tokens_result(toks, req: TokenLayers, pooled, return_pooled: bool):
    """What a per-token call returns: one result per request (a tuple for a list of requests), and the pooled output when asked."""
    res = toks[req.index[0]] if req.single else tuple(toks[i] for i in req.index)
    return (res, pooled) if return_pooled else res


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

    def _device_images(self, x):
        """Prepared images on this GPU in a tower input type: host images copied over, uint8 frames through the image front-end (one
        at a time for a list; their output sizes differ)."""
        if isinstance(x, list):
            return [self._device_images(t[None])[0].contiguous() for t in x]
        xd = x.to(self.device, non_blocking=True)
        return self.preproc(xd, dtype=self._operand_dtype()) if xd.dtype == torch.uint8 else xd

    def _operand_dtype(self) -> torch.dtype:
        return {_lib.F32: torch.float32, _lib.F16: torch.float16, _lib.BF16: torch.bfloat16, _lib.F8E4M3: torch.float16}[self.cfg.compute_dtype]

    def _run(self, name: str, *args):
        """Entry point `name` on this handle (see _call)."""
        _call(self.lib, self.device, name, self.handle, *args)

    def _back(self, out: torch.Tensor, host: bool, keep=None) -> PendingResult:
        """A call's result as its caller gets it: `out` as it is for device inputs; for host inputs a pinned host tensor (`out` itself
        when the library wrote it there, else a copy queued behind the call) and the event that marks it filled.  `keep` stays
        referenced until the result is taken."""
        if not host:
            return PendingResult(out, None)
        if out.is_cuda:
            # fresh pinned result (torch's caching host allocator makes this cheap); no CPU-side tensor op on the host path: an
            # intra-op OpenMP team on a CPU-quota-limited box costs milliseconds
            out = torch.empty(out.shape, dtype=out.dtype, pin_memory=True).copy_(out, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        return PendingResult(out, ev, keep)

    # ---- forward ----
    def vision(self, x, encode: bool = False, interpolate: bool = False, wait: bool = True):
        """VisionTransformer.__call__ / encode_image on Images, or on a tensor / list prepared here.  CUDA input -> async CUDA output;
        host input -> host output.  interpolate: HF's interpolate_pos_encoding (images of any size; see jimm_vit_forward_hw); a list
        runs in one packed call (jimm_vit_forward_packed).  wait=False returns a PendingResult: host images of the trained size are
        left in flight (JAX-style asynchronous dispatch: back-to-back calls pipeline, the copies of call k+1 run under the towers of
        call k, and the caller keeps the images alive and unmodified until the result is taken); any other input comes back
        finished."""
        im = x if isinstance(x, Images) else prep_images(x, self.cfg, self.preproc, interpolate)
        if im.host and im.trained and not encode and not isinstance(im.x, list):
            # host path: H2D + forward + D2H enqueued by the library on the current stream, into a pinned result (uint8 frames: bytes
            # over PCIe, front-end + tower in the library's sliced copy/compute pipeline)
            B = len(im.x)
            out = torch.empty((B, self.vision_out), dtype=torch.float32, pin_memory=True)
            if im.u8:
                self._run("jimm_vit_forward_host_u8", self.preproc.handle, im.x, B, im.x.shape[1], im.x.shape[2], out)
            else:
                self._run("jimm_vit_forward_host", im.x, im.x.dtype, B, out)
            res = self._back(out, True, keep=im.x)
            return res if not wait else res.result()
        res = self._back(self._vision_dev(im, encode), im.host, keep=im.x).result()
        return res if wait else PendingResult(res, None)

    def _image_inputs(self, im: Images, xd):
        """The arguments of a vision call on im's images xd (on this GPU) up to `out` / `req`: the input form ("patches": NaFlex rows,
        "packed": a list, "trained" / "dense": a batch of the trained size or not), the ctypes argument tuple (a batch's with H and W)
        and each sample's token count (None for a batch).  Freshly made device copies of list images are freed only after the call's
        work."""
        B = len(xd)
        if im.grid is not None:
            return "patches", (xd, xd.dtype, B, xd.shape[1], (C.c_int * (2 * B))(*[v for hw in im.grid for v in hw])), [h * w for h, w in im.grid]
        if isinstance(xd, list):
            if not im.host:
                for t in xd:
                    t.record_stream(torch.cuda.current_stream(self.device))
            args = ((C.c_void_p * B)(*[t.data_ptr() for t in xd]), xd[0].dtype if B else torch.float32, B,
                    (C.c_int * B)(*[t.shape[0] for t in xd]), (C.c_int * B)(*[t.shape[1] for t in xd]))
            return "packed", args, [grid_tokens(self.cfg, t.shape[0], t.shape[1]) for t in xd]
        return "trained" if im.trained else "dense", (xd, xd.dtype, B, xd.shape[1], xd.shape[2]), None

    def _vision_dev(self, im: Images, encode: bool) -> torch.Tensor:
        """The vision call on the images on this GPU (host images copied over): fp32 [B, out_dim] on this GPU."""
        xd = self._device_images(im.x)
        B = len(xd)
        out = torch.empty((B, self.vision_out), dtype=torch.float32, device=self.device)
        form, args, _ = self._image_inputs(im, xd)
        name = "jimm_encode_image" if encode else "jimm_vit_forward"
        if form == "trained":
            self._run(name, *args[:3], out)
        elif form == "dense":
            self._run(name + "_hw", *args, out)
        elif B:
            self._run("jimm_encode_image_patches" if form == "patches" else name + "_packed", *args, out)
        return out

    def _texts(self, text) -> Union[torch.Tensor, Texts]:
        """The text input of a call: Texts for a list / tuple of sequences (or Texts already), else the [B, T] ids tensor."""
        if isinstance(text, Texts):
            return text
        if isinstance(text, (list, tuple)):
            return prep_texts(text, self.cfg.ctx_len)
        return prep_ids(text)

    def _text_inputs(self, ids: Union[torch.Tensor, Texts]):
        """The arguments of a text call on a [B, T] ids tensor or on Texts up to `out` / `req`, the ids copied to this GPU: the ctypes
        argument tuple, each sequence's length (None for a tensor) and whether the result goes back to the host."""
        if isinstance(ids, Texts):
            B = len(ids.lens)
            return (ids.ids.to(self.device, non_blocking=True), B, (C.c_int * max(B, 1))(*ids.lens)), ids.lens, ids.host
        B, T = ids.shape
        return (ids.to(self.device, non_blocking=True), B, T), None, not ids.is_cuda

    def _text_dev(self, ids: Union[torch.Tensor, Texts]) -> torch.Tensor:
        """encode_text of a [B, T] ids tensor, or of Texts in one packed call (jimm_encode_text_packed): fp32 [B, E] on this GPU."""
        args, lens, _ = self._text_inputs(ids)
        out = torch.empty((args[1], self.text_out), dtype=torch.float32, device=self.device)
        if lens is None:
            self._run("jimm_encode_text", *args, out)
        elif lens:
            self._run("jimm_encode_text_packed", *args, out)
        return out

    def text(self, ids) -> torch.Tensor:
        """encode_text of a [B, T] ids tensor, or of a list of sequences of different lengths (one packed call).  CUDA input -> CUDA
        output; host input -> host output."""
        ids = self._texts(ids)
        return self._back(self._text_dev(ids), ids.host if isinstance(ids, Texts) else not ids.is_cuda).result()

    # ---- per-token hidden states and attention weights ----
    def _sink_call(self, name: str, struct, inputs, shapes, req: TokenLayers, B: int, pooled_dim: int, pooled: bool, host: bool):
        """Entry point `name` (jimm_image_tokens* / jimm_text_tokens* with struct TokensReq, jimm_image_attn* / jimm_text_attn* with
        AttnReq) on `inputs`: per distinct request i one output of req.dtype shaped by shapes[i] -- a tuple for a dense batch, or a list
        of per-sample shapes, views of one packed buffer in sample order -- and the fp32 [B, pooled_dim] pooled output when asked (else
        None).  host: the results come back to the host."""
        outs = [torch.empty(sum(math.prod(x) for x in ([sh] if isinstance(sh, tuple) else sh)), dtype=req.dtype, device=self.device)
                for sh in shapes]
        pool = torch.empty((B, pooled_dim), dtype=torch.float32, device=self.device) if pooled else None
        if B:
            n = len(req.codes)
            r = struct(n, (C.c_int * n)(*req.codes), (C.c_void_p * n)(*[o.data_ptr() for o in outs]), _TORCH_TO_CODE[req.dtype])
            self._run(name, *inputs, C.byref(r), pool if pooled else None)
        if host:
            outs = [self._back(o, True).result() for o in outs]
            pool = self._back(pool, True).result() if pool is not None else None
        res = []
        for o, sh in zip(outs, shapes):
            if isinstance(sh, tuple):
                res.append(o.view(sh))
            else:
                res.append([p.view(x) for p, x in zip(torch.split(o, [math.prod(x) for x in sh]), sh)] if sh else [])
        return res, pool

    @staticmethod
    def _sink_shapes(attn: bool, req: TokenLayers, B: int, S, counts, D: int, H: int):
        """Each request's output shape (see _sink_call) for B samples of S tokens each (counts None) or of counts[b] tokens: hidden
        states [S, D] per sample; attention weights [H, S, S], or [H, 1, S] for the MAP head's."""
        def one(c, n):
            return (n, D) if not attn else (H, 1, n) if c == _lib.ATTN_MAP else (H, n, n)
        return [(B, *one(c, S)) if counts is None else [one(c, n) for n in counts] for c in req.codes]

    def _image_sink(self, im: Images, req: TokenLayers, pooled: bool, attn: bool):
        xd = self._device_images(im.x)
        B = len(xd)
        form, args, counts = self._image_inputs(im, xd)
        name = ("jimm_image_attn" if attn else "jimm_image_tokens") + {"patches": "_patches", "packed": "_packed"}.get(form, "")
        S = grid_tokens(self.cfg, xd.shape[1], xd.shape[2]) if counts is None else None
        shapes = self._sink_shapes(attn, req, B, S, counts, self.cfg.v_width, self.cfg.v_heads)
        return self._sink_call(name, _lib.AttnReq if attn else _lib.TokensReq, args, shapes, req, B, self.vision_out, pooled, im.host)

    def _text_sink(self, ids, req: TokenLayers, pooled: bool, attn: bool):
        args, lens, host = self._text_inputs(self._texts(ids))
        B = args[1]
        name = ("jimm_text_attn" if attn else "jimm_text_tokens") + ("" if lens is None else "_packed")
        shapes = self._sink_shapes(attn, req, B, args[2] if lens is None else None, lens, self.cfg.t_width, self.cfg.t_heads)
        return self._sink_call(name, _lib.AttnReq if attn else _lib.TokensReq, args, shapes, req, B, self.text_out, pooled, host)

    def image_tokens(self, im: Images, req: TokenLayers, pooled: bool = False):
        """Hidden states of the vision tower on prepared images: per distinct request [B, S, D] for a batch, a list of [S_i, D] views of
        one packed [sum S_i, D] buffer for a list or NaFlex patch rows; and the pooled output (the vision call's result) when asked.
        Host images are copied over and run eagerly; their results come back to the host."""
        return self._image_sink(im, req, pooled, False)

    def text_tokens(self, ids, req: TokenLayers, pooled: bool = False):
        """Hidden states of the text tower on a [B, T] ids tensor (per distinct request [B, T, D]) or on Texts (a list of [L_i, D] views
        of one packed [sum L_i, D] buffer); and the pooled output (encode_text's result) when asked.  Host ids give host results."""
        return self._text_sink(ids, req, pooled, False)

    def image_attn(self, im: Images, req: TokenLayers, pooled: bool = False):
        """Attention weights of the vision tower on prepared images (req from prep_blocks): per distinct request [B, H, S, S] for a batch
        ([B, H, 1, S] for the MAP head's), a list of [H, S_i, S_i] ([H, 1, S_i]) views of one packed buffer for a list or NaFlex patch
        rows; and the pooled output when asked.  Host images give host results."""
        return self._image_sink(im, req, pooled, True)

    def text_attn(self, ids, req: TokenLayers, pooled: bool = False):
        """Attention weights of the text tower on a [B, T] ids tensor ([B, H, T, T] per distinct request) or on Texts (a list of
        [H, L_i, L_i] views of one packed buffer); and the pooled output when asked.  Host ids give host results."""
        return self._text_sink(ids, req, pooled, True)

    def dual_encode(self, x: torch.Tensor, ids: torch.Tensor):
        """encode_image + encode_text of device-resident inputs with the two towers running concurrently (jimm_dual_encode)."""
        x = self._device_images(x)
        Bi, (Bt, T) = x.shape[0], ids.shape
        ie = torch.empty((Bi, self.vision_out), dtype=torch.float32, device=self.device)
        te = torch.empty((Bt, self.text_out), dtype=torch.float32, device=self.device)
        # images of the native size run exactly as jimm_dual_encode; others only reach here with interpolate_pos_encoding
        self._run("jimm_dual_encode_hw", x, x.dtype, Bi, x.shape[1], x.shape[2], ids, Bt, T, ie, te)
        return ie, te

    def logits(self, img_e: torch.Tensor, txt_e: torch.Tensor) -> torch.Tensor:
        img_e = img_e.to(self.device, torch.float32).contiguous()
        txt_e = txt_e.to(self.device, torch.float32).contiguous()
        Bi, Bt = img_e.shape[0], txt_e.shape[0]
        out = torch.empty((Bi, Bt), dtype=torch.float32, device=self.device)
        self._run("jimm_contrastive_logits", img_e, Bi, txt_e, Bt, out)
        return out

    def _embeddings(self, name: str, x) -> torch.Tensor:
        """A [rows, E] embedding set of a search or an index, checked: float32 / float16 / bfloat16, at most 2^31 - 1 rows."""
        t = _as_tensor(x)
        E = self.text_out
        if t.ndim != 2 or t.shape[1] != E:
            raise ValueError(f"search: expected {name} of shape [rows, {E}] (the model's embedding width), got {tuple(t.shape)}")
        if t.dtype not in _TORCH_TO_CODE:
            raise ValueError(f"search: {name} must be float32, float16 or bfloat16, got {t.dtype}")
        if t.shape[0] > 2**31 - 1:
            raise ValueError(f"search: at most {2**31 - 1} {name} rows, got {t.shape[0]}")
        return t

    @staticmethod
    def _search_k(k, N: int) -> int:
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= min(N, 1024):
            raise ValueError(f"search: k must be an int in 1 .. min(gallery rows={N}, 1024), got {k!r}")
        return int(k)

    def search(self, queries, gallery, k: int):
        """The k best gallery rows of each query by the model's score (jimm_search): fp32 [Q, k] scores and int32 [Q, k] indices,
        bit for bit the top_k of the logits matrix the contrastive head would give for the two sets.  Both [*, E] embedding sets of
        float32 / float16 / bfloat16 on the device or the host; the result is on the host when both were."""
        q, g = self._embeddings("queries", queries), self._embeddings("gallery", gallery)
        Q, N = q.shape[0], g.shape[0]
        k = self._search_k(k, N)
        host = not q.is_cuda and not g.is_cuda
        qd = q.to(self.device, torch.float32, non_blocking=True).contiguous()
        gd = g.to(self.device, torch.float32, non_blocking=True).contiguous()
        values = torch.empty((Q, k), dtype=torch.float32, device=self.device)
        indices = torch.empty((Q, k), dtype=torch.int32, device=self.device)
        self._run("jimm_search", qd, Q, gd, N, k, values, indices)
        return self._back(values, host).result(), self._back(indices, host).result()

    def index(self, gallery=None) -> "GalleryIndex":
        """A gallery index on this handle (jimm_index_create), holding `gallery`'s rows when given; it raises once this handle is
        closed."""
        return GalleryIndex(lambda: self, gallery)

    def dual(self, images, text, interpolate: bool = False) -> torch.Tensor:
        """CLIP.__call__ / SigLIP.__call__ on one GPU, on Images or on a tensor / list prepared here, and on a [B, T] ids tensor or a
        list of token sequences (Texts).  The result is on the host when the images and the ids were.  A list of sequences runs the
        vision call, the packed text call and the logits one after another on the current stream."""
        im = images if isinstance(images, Images) else prep_images(images, self.cfg, self.preproc, interpolate)
        ids = self._texts(text)
        if isinstance(ids, Texts):
            out = self.logits(self._vision_dev(im, True), self._text_dev(ids))
            return self._back(out, im.host and ids.host).result()
        host = im.host and not ids.is_cuda
        Bi, (Bt, T) = len(im.x), ids.shape
        if isinstance(im.x, list) or im.grid is not None:
            out = self.logits(self._vision_dev(im, True), self._text_dev(ids))
        elif host and im.trained and not im.u8:
            # float pixels and ids: the library's pipeline copies both in and the logits out
            out = torch.empty((Bi, Bt), dtype=torch.float32, pin_memory=True)
            self._run("jimm_dual_forward_host", im.x, im.x.dtype, Bi, ids, Bt, T, out)
        else:
            xd, idd = self._device_images(im.x), ids.to(self.device, non_blocking=True)
            out = torch.empty((Bi, Bt), dtype=torch.float32, device=self.device)
            if im.trained:
                self._run("jimm_dual_forward", xd, xd.dtype, Bi, idd, Bt, T, out)
            else:
                self._run("jimm_dual_forward_hw", xd, xd.dtype, Bi, xd.shape[1], xd.shape[2], idd, Bt, T, out)
        return self._back(out, host).result()

    # ---- multi-GPU contrastive head (one process per GPU; torch.distributed is the control plane) ----
    def comm_setup(self, max_rows_per_rank: int, group=None):
        import torch.distributed as dist

        from .dist import exchange_handles

        rank, world = dist.get_rank(group), dist.get_world_size(group)
        handle = C.create_string_buffer(64)
        _lib.check(self.lib.jimm_comm_init(self.handle, rank, world, int(max_rows_per_rank), handle))
        _lib.check(self.lib.jimm_comm_connect(self.handle, exchange_handles(handle.raw, group)))
        dist.barrier(group)
        self._comm = (rank, world, int(max_rows_per_rank))

    def comm_logits(self, img_e: torch.Tensor, txt_e: torch.Tensor) -> torch.Tensor:
        """Fused normalise + NVLink peer scatter + local logits row block [B_local, world*B_local]."""
        if self._comm is None:
            raise _lib.JimmError("comm_setup() has not been called")
        rank, world, _ = self._comm
        img_e = img_e.to(self.device, torch.float32).contiguous()
        txt_e = txt_e.to(self.device, torch.float32).contiguous()
        B = img_e.shape[0]
        if txt_e.shape[0] != B:
            raise ValueError("multi-GPU contrastive head needs equal image/text batch per rank")
        out = torch.empty((B, world * B), dtype=torch.float32, device=self.device)
        self._run("jimm_comm_contrastive_logits", img_e, txt_e, B, out)
        return out


class KMeans(NamedTuple):
    """The result of GalleryIndex.kmeans, on the index's device."""

    centroids: torch.Tensor  # fp32 [C, E], unit rows: the centroids the last assignment step used
    assign: torch.Tensor  # int32 [len(index)]: each row's cluster, -1 for rows that take no part
    scores: torch.Tensor  # fp32 [len(index)]: each row's score against its centroid, -inf where assign is -1
    counts: torch.Tensor  # int64 [C]: rows per cluster under assign
    iterations: int  # assignment steps run (<= iters)


class GalleryIndex:
    """A gallery normalised once and kept on the GPU (jimm_index_*): search(queries, k) is NativeModel.search(queries, every row added
    so far, k) on the model's current handle, bit for bit; range_search(queries, threshold) and pairs(threshold) give every score at or
    above a threshold.  remove(ids) drops rows from every later call, keep= restricts one call to a subset of the rows, and compact()
    renumbers the live rows and frees the removed ones.  `native` returns that handle: a model's `native` method, which rebuilds it
    when its parameters or batch bound change.  Each add / search rebinds the index to the handle `native` gives (jimm_index_rebind,
    same width and device; the stored rows stay), so it scores with the model's current logit_scale / logit_bias and never reads a
    handle the model has destroyed.  Holding `native` keeps the model alive."""

    def __init__(self, native: Callable[[], NativeModel], gallery=None):
        self._native = native
        m = native()
        self._bound, self._lib, self._device, self._width = m, m.lib, m.device, m.text_out
        self.handle = C.c_void_p()
        _lib.check(m.lib.jimm_index_create(m.handle, C.byref(self.handle)))
        self._rows = 0
        if gallery is not None:
            self.add(gallery)

    def _model(self) -> NativeModel:
        """The handle the index scores with now, bound to it."""
        if not self.handle:
            raise _lib.JimmError("gallery index: closed")
        m = self._native()
        if not m.handle:
            raise _lib.JimmError("gallery index: its model handle has been closed")
        if m is not self._bound:
            _lib.check(self._lib.jimm_index_rebind(self.handle, m.handle))
            self._bound = m
        return m

    def add(self, rows) -> "GalleryIndex":
        """Append [n, E] embeddings (float32 / float16 / bfloat16, device or host); their indices continue from len(self)."""
        m = self._model()
        g = m._embeddings("gallery", rows)
        n = g.shape[0]
        if self._rows + n > 2**31 - 1:
            raise ValueError(f"index: at most {2**31 - 1} rows, {self._rows} + {n} given")
        gd = g.to(m.device, torch.float32, non_blocking=True).contiguous()
        _call(m.lib, m.device, "jimm_index_add", self.handle, gd, n)
        self._rows += n
        return self

    def __len__(self) -> int:
        """Every row ever added (removed ones included) since the last compact(): the next add numbers its rows from here."""
        return self._rows

    @property
    def num_live(self) -> int:
        """The rows not removed."""
        if not self.handle:
            raise _lib.JimmError("gallery index: closed")
        live = C.c_longlong()
        _lib.check(self._lib.jimm_index_live(self.handle, C.byref(live)))
        return live.value

    def _row_tensor(self, x, what: str) -> torch.Tensor:
        """x (an int, a sequence, a numpy array or a torch tensor, on the host or the index's device) as a 1-D tensor, checked for its
        device; an empty sequence is int64."""
        if isinstance(x, torch.Tensor):
            t = x
        else:
            a = np.asarray(x)
            if a.size == 0:
                a = a.astype(np.int64)
            if a.dtype.kind not in "biu":
                raise ValueError(f"index: {what} must be integers or bools, got {a.dtype}")
            t = torch.from_numpy(np.ascontiguousarray(a))
        if t.is_cuda and t.device != self._device:
            raise ValueError(f"index: {what} is on {t.device}, the index on {self._device}")
        return t.reshape(-1)

    def _row_ids(self, t: torch.Tensor, what: str) -> torch.Tensor:
        """Integer row ids, each in 0 .. len(self) - 1, as int32 on the index's device."""
        if t.dtype == torch.bool or t.dtype.is_floating_point or t.dtype.is_complex:
            raise ValueError(f"index: {what} must be integer row ids, got {t.dtype}")
        t = t.to(torch.int64)
        if t.numel() > 0:
            lo, hi = int(t.min()), int(t.max())
            if lo < 0 or hi >= self._rows:
                raise ValueError(f"index: {what} must be row ids in 0 .. {self._rows - 1}, got {lo} .. {hi}")
        return t.to(self._device, torch.int32, non_blocking=True).contiguous()

    def _keep(self, keep) -> Optional[torch.Tensor]:
        """keep as a bool mask [len(self)] on the index's device (its memory is the byte mask the C calls take), or None."""
        if keep is None:
            return None
        t = self._row_tensor(keep, "keep")
        if t.dtype == torch.bool:
            if t.numel() != self._rows:
                raise ValueError(f"index: a keep mask must have one entry per row ({self._rows}), got {t.numel()}")
            return t.to(self._device, non_blocking=True).contiguous()
        ids = self._row_ids(t, "keep")
        mask = torch.zeros(self._rows, dtype=torch.bool, device=self._device)
        mask[ids.long()] = True
        return mask

    def remove(self, ids) -> int:
        """Remove rows by id (an int, a sequence, a numpy array or an integer tensor, host or device): every later call skips them.
        Returns the rows newly removed (duplicates and rows already removed count once / not at all).  Row numbers are not reused,
        and removed rows keep their memory until compact()."""
        if not self.handle:
            raise _lib.JimmError("gallery index: closed")
        ids = self._row_ids(self._row_tensor(ids, "ids"), "ids")
        removed = C.c_longlong()
        _call(self._lib, self._device, "jimm_index_remove", self.handle, ids, ids.numel(), C.byref(removed))
        return removed.value

    def compact(self) -> torch.Tensor:
        """Drop the removed rows and renumber the live ones in their order, in new storage of their size.  Returns the old-to-new
        map: int64 [len(self) before] on the index's device, -1 for a removed row."""
        if not self.handle:
            raise _lib.JimmError("gallery index: closed")
        old_to_new = torch.empty(self._rows, dtype=torch.int32, device=self._device)
        _call(self._lib, self._device, "jimm_index_compact", self.handle, old_to_new)
        self._rows = self.num_live
        return old_to_new.to(torch.int64)

    def search(self, queries, k: int, keep=None):
        """The k best rows of the index for each query: fp32 [Q, k] scores and int32 [Q, k] row indices, on the host when the queries
        were.  Only live rows are searched, and of those only the ones keep selects (a bool mask [len(self)] or row ids, host or
        device): bit for bit model.search against those rows alone, with their row numbers.  With fewer than k such rows, the columns
        past them hold (-inf, -1)."""
        m = self._model()
        q = m._embeddings("queries", queries)
        k = m._search_k(k, self._rows)
        mask = self._keep(keep)
        Q = q.shape[0]
        qd = q.to(m.device, torch.float32, non_blocking=True).contiguous()
        values = torch.empty((Q, k), dtype=torch.float32, device=m.device)
        indices = torch.empty((Q, k), dtype=torch.int32, device=m.device)
        if mask is None:
            _call(m.lib, m.device, "jimm_index_search", self.handle, qd, Q, k, values, indices, None)
        else:
            _call(m.lib, m.device, "jimm_index_search_keep", self.handle, qd, Q, k, mask, values, indices, None)
        host = not q.is_cuda
        return m._back(values, host).result(), m._back(indices, host).result()

    def kmeans(self, n_clusters: int, iters: int = 20, init=None, seed: int = 0, keep=None) -> "KMeans":
        """Spherical k-means over the stored rows (jimm_index_kmeans): at most `iters` assignment steps of each row to its best centroid
        by cosine (the model's logit_scale and logit_bias play no part), each followed by the mean of every cluster's rows summed in
        fixed point, so the result is the same bits on every run.  A row takes part when it is live, selected by keep (as in search)
        and finite and non-zero; the others get assign -1 and score -inf.  init: None (rows sampled from `seed`), n_clusters integer row
        ids (host or device, each a row that takes part), or a float32 / float16 / bfloat16 [n_clusters, E] tensor of vectors (host or
        the index's device).  Stops early when an assignment repeats the previous one.  Returns a KMeans on the index's device."""
        if not self.handle:
            raise _lib.JimmError("gallery index: closed")
        for name, v, lo, hi in (("n_clusters", n_clusters, 1, 65536), ("iters", iters, 1, 2**31 - 1), ("seed", seed, 0, 2**64 - 1)):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
                raise ValueError(f"index kmeans: {name} must be an int in {lo} .. {hi}, got {v!r}")
        Cn, E = int(n_clusters), self._width
        vectors = ids = None
        if init is not None:
            t = _as_tensor(init)
            if t.is_cuda and t.device != self._device:
                raise ValueError(f"index kmeans: init is on {t.device}, the index on {self._device}")
            if t.dtype.is_floating_point:
                if t.dtype not in _TORCH_TO_CODE or tuple(t.shape) != (Cn, E):
                    raise ValueError(f"index kmeans: init vectors must be float32 / float16 / bfloat16 of shape [{Cn}, {E}], got {t.dtype} "
                                     f"{tuple(t.shape)}")
                vectors = t.to(self._device, torch.float32, non_blocking=True).contiguous()
            else:
                if t.ndim != 1 or t.numel() != Cn:
                    raise ValueError(f"index kmeans: init must be {Cn} row ids or a [{Cn}, {E}] float tensor, got {t.dtype} {tuple(t.shape)}")
                ids = self._row_ids(t, "init ids")
        mask = self._keep(keep)
        centroids = torch.empty((Cn, E), dtype=torch.float32, device=self._device)
        assign = torch.empty(self._rows, dtype=torch.int32, device=self._device)
        scores = torch.empty(self._rows, dtype=torch.float32, device=self._device)
        counts = torch.empty(Cn, dtype=torch.int64, device=self._device)
        steps = C.c_int()
        _call(self._lib, self._device, "jimm_index_kmeans", self.handle, Cn, vectors, ids, int(seed), int(iters), mask, centroids, assign,
              scores, counts, C.byref(steps), None)
        return KMeans(centroids, assign, scores, counts, steps.value)

    @staticmethod
    def _threshold(threshold) -> float:
        """A threshold on the model's score scale as a Python float; the C call rounds it to fp32 (nearest) once."""
        if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real):
            raise ValueError(f"index: the threshold must be a real number, got {threshold!r}")
        try:
            t = float(threshold)
        except OverflowError:  # an integer beyond every float: fp32 rounds it to an infinity
            t = math.copysign(math.inf, threshold)
        if math.isnan(t):
            raise ValueError("index: the threshold is NaN")
        return t

    def _hits(self, m: NativeModel, name: str, *args):
        """Run jimm_index_range_search / jimm_index_pairs and copy its jimm_hits_t into device tensors: offsets int64 [rows + 1], scores
        fp32 [total] and indices int32 [total]."""
        h = C.c_void_p()
        _call(m.lib, m.device, name, self.handle, *args, C.byref(h), None)
        try:
            rows, total = C.c_int(), C.c_longlong()
            _lib.check(m.lib.jimm_hits_size(h, C.byref(rows), C.byref(total)))
            offsets = torch.empty(rows.value + 1, dtype=torch.int64, device=m.device)
            scores = torch.empty(total.value, dtype=torch.float32, device=m.device)
            indices = torch.empty(total.value, dtype=torch.int32, device=m.device)
            _call(m.lib, m.device, "jimm_hits_copy", h, offsets, scores, indices)
        finally:
            with torch.cuda.device(m.device):
                m.lib.jimm_hits_destroy(h)
        return offsets, scores, indices

    def range_search(self, queries, threshold, keep=None):
        """Every row of the index whose score against each query is >= threshold (a real number on the model's score scale,
        exp(logit_scale) * cos + logit_bias, rounded to fp32), in CSR: offsets int64 [Q + 1], scores fp32 [nnz] and row indices int32
        [nnz], each query's hits in ascending row order; on the host when the queries were.  Bit for bit the entries >= threshold of the
        score matrix model.search ranks; a NaN score is never a hit.  Only live rows that keep selects (as in search) are hits."""
        m = self._model()
        q = m._embeddings("queries", queries)
        t = self._threshold(threshold)
        mask = self._keep(keep)
        Q = q.shape[0]
        qd = q.to(m.device, torch.float32, non_blocking=True).contiguous()
        if mask is None:
            out = self._hits(m, "jimm_index_range_search", qd, Q, t)
        else:
            out = self._hits(m, "jimm_index_range_search_keep", qd, Q, t, mask)
        host = not q.is_cuda
        return tuple(m._back(x, host).result() for x in out)

    def pairs(self, threshold, keep=None):
        """Every pair of stored rows i < j whose score is >= threshold: `i, j, scores` (int32, int32, fp32), ordered by i then j, on the
        device.  The upper triangle of range_search(every raw row added, threshold), without the raw rows.  Both rows of a pair are
        live and selected by keep (as in search)."""
        m = self._model()
        t = self._threshold(threshold)
        mask = self._keep(keep)
        if mask is None:
            offsets, scores, j = self._hits(m, "jimm_index_pairs", t)
        else:
            offsets, scores, j = self._hits(m, "jimm_index_pairs_keep", t, mask)
        rows = offsets.numel() - 1
        i = torch.repeat_interleave(torch.arange(rows, dtype=torch.int32, device=m.device), offsets.diff(), output_size=j.numel())
        return i, j, scores

    def close(self):
        """Free the stored rows (jimm_index_destroy reads only the index's own device, never the model)."""
        if getattr(self, "handle", None):
            with torch.cuda.device(self._device):
                self._lib.jimm_index_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


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
        x = _as_tensor(x)
        if x.ndim != 3 or x.shape[2] != self.D:
            raise ValueError(f"expected activations of shape [batch, seq, {self.D}], got {tuple(x.shape)}")
        B, S, D = x.shape
        xd = x.to(n.device, torch.float32, non_blocking=True).contiguous()
        if self.kind == _lib.KIND_ENCODER:
            out = torch.empty((B, S, D), dtype=torch.float32, device=n.device)
            n._run("jimm_encoder_forward", xd, B, S, out)
        else:
            out = torch.empty((B, D), dtype=torch.float32, device=n.device)
            n._run("jimm_map_head_forward", xd, B, S, out)
        xd.record_stream(torch.cuda.current_stream(n.device))
        return n._back(out, not x.is_cuda).result()


def activation(x, act: int) -> torch.Tensor:
    """Elementwise activation kernel (1 tanh-GELU, 2 QuickGELU) on a CUDA tensor; fp32 result."""
    x = _as_tensor(x)
    if not x.is_cuda:
        raise _lib.JimmError("jimm_b200 runs on CUDA tensors only (there is no CPU fallback)")
    xd = x.to(torch.float32).contiguous()
    y = torch.empty_like(xd)
    _call(_lib.load(), x.device, "jimm_k_activation", xd, y, xd.numel(), int(act))
    return y


def grid_tokens(cfg: _lib.Config, height: int, width: int) -> int:
    """Tokens per image of a vision tower on height x width images: the patches (trailing pixels dropped) and the CLS token."""
    return (int(height) // cfg.patch) * (int(width) // cfg.patch) + (1 if cfg.pooling == _lib.POOL_CLS else 0)


def default_max_batch() -> int:
    return int(os.environ.get("JIMM_MAX_BATCH", "256"))
