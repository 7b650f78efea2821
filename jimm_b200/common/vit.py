"""Mirror of jimm.common.vit (reference: src/jimm/common/vit.py): VisionTransformerBase and
MultiHeadAttentionPoolingHead with the reference's constructor kwargs and parameter tree.  `__call__` runs the whole
tower in the CUDA library (patchify + wgmma GEMMs + flash attention + LayerNorm + CLS|MAP pooling)."""

from __future__ import annotations

from typing import Dict, Optional

import torch

from .. import _lib, nn
from .._runtime import Images, NativeModel, default_max_batch, grid_tokens, prep_blocks, prep_images, prep_layers, tokens_result
from .transformer import Transformer, _SubModuleRunner, g_wrap


class MultiHeadAttentionPoolingHead(_SubModuleRunner, nn.Module):
    """common/vit.py:12-101.  Inside a tower it is evaluated as part of the tower forward (probe query precomputed at finalize, k/v
    projection GEMM over all tokens, single-query attention, LN + MLP + residual); called on its own it runs the same kernels through
    jimm_map_head_forward."""

    def __init__(self, hidden_size: int, intermediate_size: int, num_heads: int, layernorm_epsilon: float = 1e-6, rngs=None,
                 dtype=None, param_dtype=None, mesh=None):
        nn.Module.__init__(self)
        self._sub_init(dtype)
        if intermediate_size <= 0 or intermediate_size % 8:
            raise ValueError(f"MAP head intermediate_size {intermediate_size}: the GEMM kernels take a positive multiple of 8")
        g = nn._gen(rngs)
        object.__setattr__(self, "layernorm_epsilon", layernorm_epsilon)
        object.__setattr__(self, "_dims", (hidden_size, num_heads, intermediate_size))
        self.add_param("probe", nn.zeros((1, 1, hidden_size)))
        self.add_child("attn", nn.MultiHeadAttention(num_heads, hidden_size, rngs=g_wrap(g)))
        self.add_child("layernorm", nn.LayerNorm(hidden_size, layernorm_epsilon))
        # nnx.Sequential [Linear, gelu, Linear] -> param indices 0 and 2 (:65-85)
        self.add_child("mlp", nn.Sequential(nn.Linear(hidden_size, intermediate_size, rngs=g_wrap(g)), None,
                                            nn.Linear(intermediate_size, hidden_size, rngs=g_wrap(g))))

    def _sub_config(self, max_seq):
        D, H, M = self._dims
        cfg = _lib.Config()
        cfg.kind = _lib.KIND_MAPHEAD
        cfg.v_width, cfg.v_heads, cfg.v_mlp, cfg.v_layers = D, H, M, 0
        cfg.v_eps_outer = cfg.v_eps_block = float(self.layernorm_epsilon)
        cfg.ctx_len = int(max_seq)
        cfg.compute_dtype = self._sub_dtype
        return cfg

    def __call__(self, hidden_state):
        """[batch, seq, hidden] -> [batch, hidden] (common/vit.py:87-101)."""
        return self._run(hidden_state)


class _NativeOwner:
    """Mixin for top-level runnable models: lazily builds (and rebuilds when parameters or the batch bound change) the
    native handle from the flat parameter tree."""

    def _native_init(self, dtype):
        object.__setattr__(self, "_native", None)
        object.__setattr__(self, "_preproc", None)
        object.__setattr__(self, "_compute_dtype", nn.compute_dtype_code(dtype))
        object.__setattr__(self, "_max_batch", default_max_batch())
        object.__setattr__(self, "_max_tokens", 0)  # vision tokens per sample of the workspace (0: the native count)

    @staticmethod
    def _release_native(n):
        """Free a native handle.  If it owns an NVLink gather buffer, the peers have it mapped through CUDA IPC and may still be storing
        into it: every rank rebuilds at the same point of the program (same batch on every rank), so all of them drain their streams
        and meet at a barrier before anybody frees."""
        if getattr(n, "_comm", None) is not None:
            import torch.distributed as dist

            if dist.is_available() and dist.is_initialized():
                torch.cuda.synchronize(n.device)
                dist.barrier()
        n.close()

    def _invalidate(self):
        n = getattr(self, "_native", None)
        if n is not None:
            self._release_native(n)
        object.__setattr__(self, "_native", None)

    def _native_config(self) -> _lib.Config:
        raise NotImplementedError

    def native(self, batch: int = 1, require: bool = False, hw=None) -> NativeModel:
        """Native handle whose workspace holds `max_batch` samples per call; larger vision / text batches are chunked by
        the library, the contrastive head needs the whole batch resident (`require=True`).  hw: the (height, width) of the images of
        an interpolate_pos_encoding call; the handle is rebuilt with a larger token budget only when the library reports that one
        such image does not fit (a call whose images merely fit fewer at a time runs in smaller chunks).  A raised budget is kept
        for later rebuilds.  An image past a limit no budget lifts (the MAP head's sequence limit) raises ValueError from
        images_per_call: an existing handle is kept as it is, and a handle built for this call is dropped with its budget."""
        n = self._native
        if n is not None and (not require or batch <= n.max_batch) and (hw is None or n.images_per_call(*hw) > 0):
            return n
        if n is not None:
            self._release_native(n)
        mb = max(self._max_batch, int(batch) if require else 1)
        cfg = self._native_config()
        # any jimm_model_set_max_tokens budget of at least ceil(tokens / max_batch) holds one image of that many tokens
        need = -(-grid_tokens(cfg, *hw) // mb) if hw is not None else 0
        budget = self._max_tokens
        if need > max(self._max_tokens, grid_tokens(cfg, cfg.img_size, cfg.img_size)):  # more tokens than the workspace rows
            object.__setattr__(self, "_max_tokens", need)
        n = self._build_native(mb)
        try:
            fits = hw is None or n.images_per_call(*hw) > 0
        except ValueError:
            object.__setattr__(self, "_max_tokens", budget)
            self._invalidate()
            raise
        if not fits:  # enough rows, but not the bytes of its padded patch rows
            self._release_native(n)
            object.__setattr__(self, "_max_tokens", max(self._max_tokens, need))
            n = self._build_native(mb)
        return n

    def _build_native(self, mb: int) -> NativeModel:
        n = NativeModel(self._native_config(), self.flat_params(raw=True), mb, max_tokens=self._max_tokens)
        n.preproc = self._preproc
        object.__setattr__(self, "_native", n)
        return n

    def _images(self, images, interpolate_pos_encoding: bool) -> Images:
        """The image-input step (prep_images) on this model's config and image front-end, before any handle is built."""
        n = self._native
        return prep_images(images, n.cfg if n is not None else self._native_config(), self._preproc, interpolate_pos_encoding)

    def _vision(self, images, interpolate_pos_encoding: bool, encode: bool = False, wait: bool = True, **inputs):
        """A vision call (NativeModel.vision) on a [B, H, W, C] batch or a list / tuple of images of different sizes (one packed
        call).  The handle is rebuilt only when the largest image of an interpolate_pos_encoding call does not fit it.  `inputs`: the
        further image inputs a model's _images takes (SigLIP 2 NaFlex's spatial_shapes / pixel_attention_mask)."""
        im = self._images(images, interpolate_pos_encoding, **inputs)
        return self.native(hw=im.hw if interpolate_pos_encoding else None).vision(im, encode=encode, wait=wait)

    def _vision_tokens(self, images, layers, dtype, return_pooled: bool, interpolate_pos_encoding: bool, attn: bool = False, **inputs):
        """A per-token vision call (NativeModel.image_tokens) or, attn, an attention call (NativeModel.image_attn, `layers` being the
        blocks) on the inputs _vision takes.  The requests, the dtype and the images are checked before any handle is built, and the
        handle is chosen (or rebuilt) as for the pooled call."""
        cfg = self._native_config()
        req = prep_blocks(layers, cfg.v_layers, dtype, cfg.pooling == _lib.POOL_MAP) if attn else prep_layers(layers, cfg.v_layers, dtype)
        im = self._images(images, interpolate_pos_encoding, **inputs)
        n = self.native(hw=im.hw if interpolate_pos_encoding else None)
        toks, pooled = (n.image_attn if attn else n.image_tokens)(im, req, return_pooled)
        return tokens_result(toks, req, pooled, return_pooled)

    def set_max_image_size(self, height: int, width: int):
        """Size the vision workspace for interpolate_pos_encoding calls on images up to height x width: `max_batch` such images run
        in one chunk, and no call on them rebuilds the handle.  The default holds `max_batch` images of the native size (larger
        images then run fewer at a time)."""
        object.__setattr__(self, "_max_tokens", grid_tokens(self._native_config(), height, width))
        self._invalidate()
        return self

    def set_preprocessor(self, preprocessor):
        """Attach a `jimm_b200.preprocess.ImagePreprocessor`: the model then also accepts raw uint8 RGB frames [B,H,W,3] (host or
        CUDA) -- examples/vit_inference.py:27-37's `processor(images=...)` + transpose runs on the GPU, and host batches cross PCIe
        as bytes instead of fp32 pixel values.  A `NaFlexPreprocessor` goes with SigLIP 2 NaFlex models only, at the model's patch
        size (ValueError otherwise)."""
        from ..preprocess import NaFlexPreprocessor

        if isinstance(preprocessor, NaFlexPreprocessor):
            if not getattr(self, "naflex", False):
                raise ValueError("a NaFlexPreprocessor feeds SigLIP 2 NaFlex models (SigLIP(..., naflex=True)) only; use ImagePreprocessor")
            patch = self._native_config().patch
            if preprocessor.patch_size != patch:
                raise ValueError(f"the NaFlex front-end cuts {preprocessor.patch_size}-pixel patches, the model takes {patch}-pixel patches")
        object.__setattr__(self, "_preproc", preprocessor)
        if self._native is not None:
            self._native.preproc = preprocessor
        return self

    def set_max_batch(self, max_batch: int):
        """Bound of samples per native call (workspace is sized for it at finalize)."""
        object.__setattr__(self, "_max_batch", int(max_batch))
        self._invalidate()
        return self


def tower_config_fields(cfg: _lib.Config, *, img_size, patch_size, in_channels, hidden_size, num_layers, num_heads, mlp_dim,
                        pooling_type, use_quick_gelu, use_pre_norm, use_patch_bias, layernorm_epsilon):
    cfg.img_size, cfg.patch, cfg.in_ch = img_size, patch_size, in_channels
    cfg.v_width, cfg.v_layers, cfg.v_heads, cfg.v_mlp = hidden_size, num_layers, num_heads, mlp_dim
    cfg.pooling = _lib.POOL_CLS if pooling_type == "CLS" else _lib.POOL_MAP
    cfg.pre_norm, cfg.patch_bias = int(use_pre_norm), int(use_patch_bias)
    cfg.v_act = _lib.ACT_QUICK_GELU if use_quick_gelu else _lib.ACT_GELU_TANH
    cfg.v_eps_outer = layernorm_epsilon
    cfg.v_eps_block = 1e-6  # Transformer default; VisionTransformerBase never forwards its epsilon (common/vit.py:193-204)
    return cfg


class VisionTransformerBase(_NativeOwner, nn.Module):
    """common/vit.py:104-248.  map_mlp_dim: the MAP head's MLP width; None is the reference's 4 * hidden_size (common/vit.py:175),
    HF SigLIP checkpoints use the tower's intermediate_size."""

    def __init__(self, img_size: int, patch_size: int, in_channels: int, hidden_size: int, num_layers: int, num_heads: int,
                 mlp_dim: int, pooling_type: str = "CLS", dropout_rate: float = 0.0, use_quick_gelu: bool = False,
                 use_pre_norm: bool = False, use_patch_bias: bool = True, layernorm_epsilon: float = 1e-5, rngs=None, dtype=None,
                 param_dtype=None, mesh=None, map_mlp_dim: Optional[int] = None):
        nn.Module.__init__(self)
        self._native_init(dtype)
        g = nn._gen(rngs)
        n_patches = (img_size // patch_size) ** 2
        hp = dict(img_size=img_size, patch_size=patch_size, in_channels=in_channels, hidden_size=hidden_size, num_layers=num_layers,
                  num_heads=num_heads, mlp_dim=mlp_dim, pooling_type=pooling_type, use_quick_gelu=use_quick_gelu,
                  use_pre_norm=use_pre_norm, use_patch_bias=use_patch_bias, layernorm_epsilon=layernorm_epsilon)
        object.__setattr__(self, "_hp", hp)
        object.__setattr__(self, "use_pre_norm", use_pre_norm)
        object.__setattr__(self, "pooling_type", pooling_type)
        object.__setattr__(self, "dropout_rate", dropout_rate)
        self.add_child("patch_embeddings", nn.Conv(in_channels, hidden_size, (patch_size, patch_size), use_patch_bias, g_wrap(g)))
        if pooling_type == "CLS":
            self.add_param("cls_token", nn.zeros((1, 1, hidden_size)))
            pos = nn.truncated_normal(g, (1, n_patches + 1, hidden_size), 0.02)
        elif pooling_type == "MAP":
            pos = nn.truncated_normal(g, (1, n_patches, hidden_size), 0.02)
            self.add_child("MAPHead", MultiHeadAttentionPoolingHead(hidden_size, map_mlp_dim or 4 * hidden_size, num_heads,
                                                                      layernorm_epsilon, rngs=g_wrap(g)))
        else:
            raise ValueError("pooling_type must be either MAP or CLS.")  # common/vit.py:178
        self.add_param("position_embeddings", pos)
        if use_pre_norm:
            self.add_child("ln_pre", nn.LayerNorm(hidden_size, layernorm_epsilon))
        self.add_child("transformer", Transformer(width=hidden_size, mlp_dim=mlp_dim, layers=num_layers, num_heads=num_heads,
                                                  dropout_rate=dropout_rate, use_quick_gelu=use_quick_gelu, rngs=g_wrap(g)))
        self.add_child("ln_post", nn.LayerNorm(hidden_size, layernorm_epsilon))

    def _native_config(self) -> _lib.Config:
        cfg = _lib.Config()
        cfg.kind = _lib.KIND_TOWER
        tower_config_fields(cfg, **self._hp)
        cfg.num_classes = 0
        cfg.compute_dtype = self._compute_dtype
        return cfg

    def __call__(self, img, interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """[batch, height, width, channels] -> [batch, hidden_size] (CLS token or MAP head output).  interpolate_pos_encoding
        (HuggingFace's keyword): images of any size of at least one patch, the position embeddings resampled bicubically to the
        patch grid.  A list / tuple of images [H_i, W_i, C] (or [1, H_i, W_i, C]) of different sizes runs in one packed call; row i
        is the result of images[i] alone."""
        return self._vision(img, interpolate_pos_encoding)

    def forward_async(self, img, interpolate_pos_encoding: bool = False):
        """Asynchronous dispatch for host inputs (the reference's calls return before the device finishes, examples/vit_inference.py:54
        only blocks when it reads the logits): returns a `PendingResult`; back-to-back calls overlap their copies with compute.  A
        list of images runs as in __call__, synchronously for host images."""
        return self._vision(img, interpolate_pos_encoding, wait=False)

    def forward_tokens(self, img, layers=None, *, dtype=torch.float32, return_pooled: bool = False, interpolate_pos_encoding: bool = False):
        """Per-token hidden states (HF's output_hidden_states) of the inputs __call__ takes.  layers: an int k in [-(L+1), L] -- x_k, the
        fp32 residual stream after k blocks (0: the embeddings, after ln_pre when the tower has it; negative k counts from the end, -1 is
        x_L) -- or None, the final-normed tokens ln_post(x_L); or a list / tuple of these, giving a tuple in request order.  Each result
        is [batch, S, hidden_size] of `dtype` (float32, float16 or bfloat16), S = patches (+1 CLS, first), patches row-major; a list of
        images gives a list of [S_i, hidden_size].  Without None or return_pooled only the blocks up to the deepest request run.
        return_pooled: also return __call__'s result on the same input, bit for bit: (tokens, pooled)."""
        return self._vision_tokens(img, layers, dtype, return_pooled, interpolate_pos_encoding)

    def forward_attentions(self, img, blocks=None, *, dtype=torch.float32, return_pooled: bool = False, interpolate_pos_encoding: bool = False):
        """Self-attention weights (HF's output_attentions) of the inputs __call__ takes.  blocks: an int k in [-L, L-1] -- block k's
        softmax(q k^T / sqrt(d)) per head, computed in fp32 on the q / k the forward's attention reads (negative k counts from the end)
        -- or "map" on a MAP-pooled tower, its pooling head's probe weights (the weights the pooled output sums the tokens with); None
        gives every block in order, a tuple like HF's `attentions`; a list / tuple of these gives a tuple in request order.  Each result
        is [batch, heads, S, S] ("map": [batch, heads, 1, S]) of `dtype` (float32, float16 or bfloat16), S the tokens as forward_tokens
        orders them; a list of images gives a list of [heads, S_i, S_i].  Without "map" or return_pooled only the blocks up to the
        deepest request run.  return_pooled: also return __call__'s result on the same input, bit for bit: (weights, pooled)."""
        return self._vision_tokens(img, blocks, dtype, return_pooled, interpolate_pos_encoding, attn=True)
