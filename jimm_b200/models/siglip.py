"""Mirror of jimm.models.siglip (reference: src/jimm/models/siglip.py), and SigLIP 2 NaFlex checkpoints on the same parameter tree."""

from __future__ import annotations

import math
from typing import Optional

import torch

from .. import _lib, nn
from ..common.transformer import g_wrap
from ..common import hf_loader as L
from ..common.utils import load_params_and_config
from .._runtime import _as_tensor, prep_patches
from ..common.vit import VisionTransformerBase, tower_config_fields
from ._dual import DualTower, build_text_tower


class SigLIP(DualTower):
    """models/siglip.py:15-174.

    naflex=True: the vision tower of a SigLIP 2 NaFlex checkpoint (HF `Siglip2Model`).  The parameter tree is SigLIP's, with a
    (image_resolution / vision_patch_size)^2-row position table; every image keeps its own aspect ratio and patch grid, and the table is
    resampled to that grid with F.interpolate(mode="bilinear", align_corners=False, antialias=True).  encode_image / __call__ then take the
    HF processor's `pixel_values` [B, max_num_patches, P*P*3] with `spatial_shapes` [B, 2] (and optionally its `pixel_attention_mask`),
    or NHWC images of any size of at least one patch (a list for different sizes), trailing pixels dropped.

    vision_heads, vision_mlp_dim, text_mlp_dim, vision_quick_gelu, text_quick_gelu: the architecture of checkpoints that depart from the
    reference's rule (vision_width // 64 heads, MLPs 4x the width, tanh GELU), such as so400m (16 heads of 72 and MLPs 4304 wide on
    both towers).  The MAP head's MLP is vision_mlp_dim wide, as in HF's SigLIP; its GELU is always tanh.  None / the defaults are the
    reference's values."""

    def __init__(self, image_resolution: int, vision_layers: int, vision_width: int, vision_patch_size: int, context_length: int,
                 vocab_size: int, transformer_width: int, transformer_heads: int, transformer_layers: int, rngs=None,
                 dtype=torch.float32, param_dtype=torch.float32, mesh=None, naflex: bool = False, vision_heads: Optional[int] = None,
                 vision_mlp_dim: Optional[int] = None, text_mlp_dim: Optional[int] = None, vision_quick_gelu: bool = False,
                 text_quick_gelu: bool = False):
        if naflex and image_resolution % vision_patch_size:
            raise ValueError(f"naflex: image_resolution {image_resolution} must be a multiple of vision_patch_size {vision_patch_size} "
                             "(the position table is a square grid of patches)")
        if vision_quick_gelu:
            raise ValueError("vision_quick_gelu: the MAP head runs the tanh GELU, so the vision tower of SigLIP cannot be QuickGELU")
        self._init_common(image_resolution, vision_layers, vision_width, vision_patch_size, context_length, vocab_size,
                          transformer_width, transformer_heads, transformer_layers, dtype, vision_heads=vision_heads,
                          vision_mlp_dim=vision_mlp_dim, text_mlp_dim=text_mlp_dim, vision_quick_gelu=vision_quick_gelu,
                          text_quick_gelu=text_quick_gelu)
        object.__setattr__(self, "naflex", bool(naflex))
        g = nn._gen(rngs)
        # models/siglip.py:59-78: MAP pooling, patch bias, tanh-GELU, eps 1e-6
        self.add_child("vision_model", VisionTransformerBase(
            img_size=image_resolution, patch_size=vision_patch_size, in_channels=3, hidden_size=vision_width,
            num_layers=vision_layers, num_heads=self.vision_heads, mlp_dim=self.vision_mlp_dim, use_pre_norm=False,
            use_patch_bias=True, use_quick_gelu=False, pooling_type="MAP", layernorm_epsilon=1e-6, dtype=dtype, rngs=g_wrap(g),
            map_mlp_dim=self.vision_mlp_dim))
        build_text_tower(self, g, head_bias=True, layernorm_epsilon=1e-6, attn_mask=None)
        self.add_param("logit_scale", nn.ones(()))
        self.add_param("logit_bias", nn.ones(()))

    def _native_config(self) -> _lib.Config:
        cfg = _lib.Config()
        cfg.kind = _lib.KIND_SIGLIP_NAFLEX if self.naflex else _lib.KIND_SIGLIP
        tower_config_fields(cfg, **self.vision_model._hp)
        cfg.num_classes = 0
        # text: no mask, tanh-GELU, ln_final eps 1e-6 (:104), last-token pooling (:151), Linear head with bias (:111-119,152)
        return self._text_config(cfg, causal=0, pool=_lib.TPOOL_LAST, head_bias=1, eps_outer=1e-6)

    # ---- SigLIP 2 NaFlex inputs ----
    def _images(self, images, interpolate_pos_encoding: bool, spatial_shapes=None, pixel_attention_mask=None):
        """The image input of a call: on a NaFlex model the HF processor's pixel_values with spatial_shapes (prep_patches), or images of
        any size; otherwise as for SigLIP."""
        if spatial_shapes is None and pixel_attention_mask is None:
            return super()._images(images, interpolate_pos_encoding or self.naflex)
        if not self.naflex:
            raise ValueError("spatial_shapes / pixel_attention_mask are inputs of SigLIP 2 NaFlex models (SigLIP(..., naflex=True))")
        if spatial_shapes is None:
            raise ValueError("pixel_attention_mask needs the spatial_shapes it was made for")
        n = self._native
        return prep_patches(images, spatial_shapes, pixel_attention_mask, n.cfg if n is not None else self._native_config())

    def _frames(self, image, spatial_shapes, pixel_attention_mask) -> bool:
        """Whether a call's image input is uint8 RGB frames for the attached NaFlex front-end: a [B, H, W, 3] batch or a list of
        [H, W, 3] frames on a NaFlex model.  Such frames with a fixed-size ImagePreprocessor attached are a ValueError: it would not
        give each image its own patch grid."""
        if not self.naflex or spatial_shapes is not None or pixel_attention_mask is not None:
            return False
        first = image[0] if isinstance(image, (list, tuple)) and len(image) else image
        if isinstance(first, (list, tuple)) or _as_tensor(first).dtype != torch.uint8:
            return False
        from ..preprocess import NaFlexPreprocessor

        if not isinstance(self._preproc, NaFlexPreprocessor):
            raise ValueError("uint8 frames into a SigLIP 2 NaFlex model need model.set_preprocessor(NaFlexPreprocessor(...)): a fixed-size "
                             "ImagePreprocessor does not give each image its own patch grid")
        return True

    def _frames_call(self, frames, fn):
        """fn(pixel_values, spatial_shapes) on uint8 frames in chunks of max_batch: one front-end call per chunk, in the model's operand
        dtype, so the intermediate holds at most max_batch x max_num_patches patch rows.  The chunks' results are joined in order, and
        come back to the host for host frames."""
        xs = frames if isinstance(frames, (list, tuple)) else _as_tensor(frames)
        if not isinstance(xs, (list, tuple)) and xs.ndim == 3:
            xs = xs[None]
        first = xs[0] if len(xs) else None
        host = first is not None and not _as_tensor(first).is_cuda
        dtype = {_lib.F32: torch.float32, _lib.BF16: torch.bfloat16}.get(self._compute_dtype, torch.float16)
        parts = []
        for b0 in range(0, max(len(xs), 1), self._max_batch):
            r = self._preproc(xs[b0:b0 + self._max_batch], dtype=dtype)
            parts.append(fn(r["pixel_values"], r["spatial_shapes"]))
        return _host(_join(parts)) if host else _join(parts)

    def encode_image(self, image, interpolate_pos_encoding: bool = False, spatial_shapes=None, pixel_attention_mask=None) -> torch.Tensor:
        """As DualTower.encode_image.  On a NaFlex model: `image` is the HF processor's pixel_values [B, N, P*P*3] when spatial_shapes
        [B, 2] = (patch rows, patch columns) is given -- sample b's first rows_b * cols_b rows are its patches, the rest padding that is
        never read; a pixel_attention_mask, if given, must be the prefix mask those shapes imply (ValueError otherwise) -- or, with a
        NaFlexPreprocessor attached, uint8 RGB frames (a [B, H, W, 3] batch or a list of frames of any sizes), which the front-end turns
        into exactly those inputs; else NHWC images of any size (interpolate_pos_encoding is implied)."""
        if self._frames(image, spatial_shapes, pixel_attention_mask):
            return self._frames_call(image, lambda pv, ss: self.encode_image(pv, spatial_shapes=ss))
        return self._vision(image, interpolate_pos_encoding or self.naflex, encode=True, spatial_shapes=spatial_shapes,
                            pixel_attention_mask=pixel_attention_mask)

    def encode_image_tokens(self, image, layers=None, *, dtype=torch.float32, return_pooled: bool = False, interpolate_pos_encoding: bool = False,
                            spatial_shapes=None, pixel_attention_mask=None):
        """As DualTower.encode_image_tokens, with the NaFlex image inputs of encode_image: on pixel_values with spatial_shapes each
        sample's result is [rows_b * cols_b, D] (no CLS token), its patches row-major; uint8 frames as encode_image takes them."""
        if self._frames(image, spatial_shapes, pixel_attention_mask):
            return self._frames_call(image, lambda pv, ss: self.encode_image_tokens(pv, layers, dtype=dtype, return_pooled=return_pooled,
                                                                                    spatial_shapes=ss))
        return self._vision_tokens(image, layers, dtype, return_pooled, interpolate_pos_encoding or self.naflex, spatial_shapes=spatial_shapes,
                                   pixel_attention_mask=pixel_attention_mask)

    def encode_image_attentions(self, image, blocks=None, *, dtype=torch.float32, return_pooled: bool = False,
                                interpolate_pos_encoding: bool = False, spatial_shapes=None, pixel_attention_mask=None):
        """As DualTower.encode_image_attentions, with the NaFlex image inputs of encode_image: on pixel_values with spatial_shapes each
        sample's result is [heads, n_b, n_b] ("map": [heads, 1, n_b]), n_b = rows_b * cols_b its patches, row-major; uint8 frames as
        encode_image takes them."""
        if self._frames(image, spatial_shapes, pixel_attention_mask):
            return self._frames_call(image, lambda pv, ss: self.encode_image_attentions(pv, blocks, dtype=dtype, return_pooled=return_pooled,
                                                                                        spatial_shapes=ss))
        return self._vision_tokens(image, blocks, dtype, return_pooled, interpolate_pos_encoding or self.naflex, attn=True,
                                   spatial_shapes=spatial_shapes, pixel_attention_mask=pixel_attention_mask)

    def __call__(self, image, text, spatial_shapes=None, pixel_attention_mask=None, interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """As DualTower.__call__, with the NaFlex image inputs of encode_image (single process only).  uint8 frames: the logits of
        encode_image(frames) against encode_text(text)."""
        if self._frames(image, spatial_shapes, pixel_attention_mask):
            ie, te = self.encode_image(image), self.encode_text(text)
            n = self.native(max(len(ie), len(te)), require=True)
            out = n.logits(ie, te)
            return out.cpu() if not ie.is_cuda and not te.is_cuda else out
        return self._dual_call(image, text, interpolate_pos_encoding or self.naflex, spatial_shapes=spatial_shapes,
                               pixel_attention_mask=pixel_attention_mask)

    @classmethod
    def from_pretrained(cls, model_name_or_path: str, use_pytorch: bool = False, mesh=None, dtype=torch.float32) -> "SigLIP":
        """Load a HF `SiglipModel` checkpoint (models/siglip.py:176-385): shapes always inferred from the tensors, except
        `image_size`, which must come from config["vision_config"] (:210), and each tower's heads, MLP width and hidden_act, which come
        from config["vision_config"] / config["text_config"] (hf_loader.tower_arch).  A SigLIP 2 NaFlex checkpoint (`Siglip2Model`: a 2-D
        `patch_embedding.weight`, the Linear over flattened (py, px, c) patches) loads as SigLIP(..., naflex=True): patch_size from
        config["vision_config"], image_resolution = sqrt(num_patches) * patch_size."""
        hf, config = load_params_and_config(model_name_or_path, use_pytorch)

        def depth(tower, suffix):
            return max((int(k.split(".")[3]) + 1 for k in hf if k.startswith(f"{tower}.encoder.layers.") and k.endswith(suffix)), default=0)

        pw = hf["vision_model.embeddings.patch_embedding.weight"]
        naflex = pw.ndim == 2
        if naflex:
            vision_width, vision_patch = pw.shape[0], int(config["vision_config"]["patch_size"])
            num_patches = hf["vision_model.embeddings.position_embedding.weight"].shape[0]
            g = math.isqrt(num_patches)
            if g * g != num_patches:
                raise ValueError(f"SigLIP 2 NaFlex checkpoint: num_patches = {num_patches} position rows is not a square grid")
            image_resolution = g * vision_patch
        else:
            vision_width, vision_patch = pw.shape[0], pw.shape[3]
            image_resolution = config["vision_config"]["image_size"]
        vocab_size, text_width = hf["text_model.embeddings.token_embedding.weight"].shape
        v_layers, t_layers = depth("vision_model", ".mlp.fc2.bias"), depth("text_model", ".self_attn.q_proj.weight")
        v_heads, v_mlp, v_quick = L.tower_arch(config["vision_config"], "vision_config", vision_width, hf, "vision_model", "gelu_pytorch_tanh")
        t_heads, t_mlp, t_quick = L.tower_arch(config.get("text_config", {}), "text_config", text_width, hf, "text_model", "gelu_pytorch_tanh")
        with nn.deferred_init():  # every parameter is replaced below
            model = cls(image_resolution=image_resolution, vision_layers=v_layers, vision_width=vision_width,
                        vision_patch_size=vision_patch, context_length=hf["text_model.embeddings.position_embedding.weight"].shape[0],
                        vocab_size=vocab_size, transformer_width=text_width, transformer_heads=t_heads, transformer_layers=t_layers,
                        mesh=mesh, dtype=dtype, param_dtype=dtype, naflex=naflex, vision_heads=v_heads, vision_mlp_dim=v_mlp,
                        text_mlp_dim=t_mlp, vision_quick_gelu=v_quick, text_quick_gelu=t_quick)
        v, mh = "vision_model.", "vision_model.MAPHead."
        rules = [
            ("logit_scale", "logit_scale", L.ASIS),                                      # (1,) -> ()          models/siglip.py:322-323
            ("logit_bias", "logit_bias", L.ASIS),
            ("positional_embedding", "text_model.embeddings.position_embedding.weight", L.ASIS),
            ("token_embedding.embedding", "text_model.embeddings.token_embedding.weight", L.ASIS),
            ("ln_final.scale", "text_model.final_layer_norm.weight", L.ASIS),
            ("ln_final.bias", "text_model.final_layer_norm.bias", L.ASIS),
            ("text_projection.kernel", "text_model.head.weight", L.LINEAR),
            ("text_projection.bias", "text_model.head.bias", L.ASIS),
            (v + "patch_embeddings.kernel", v + "embeddings.patch_embedding.weight", L.PATCH_LINEAR if naflex else L.CONV),
            (v + "patch_embeddings.bias", v + "embeddings.patch_embedding.bias", L.ASIS),
            (v + "position_embeddings", v + "embeddings.position_embedding.weight", L.ASIS),  # (S,D) -> (1,S,D)    :320-321
            (v + "ln_post.scale", v + "post_layernorm.weight", L.ASIS),
            (v + "ln_post.bias", v + "post_layernorm.bias", L.ASIS),
            (mh + "probe", v + "head.probe", L.ASIS),
            (mh + "layernorm.scale", v + "head.layernorm.weight", L.ASIS),
            (mh + "layernorm.bias", v + "head.layernorm.bias", L.ASIS),
            (mh + "mlp.layers.0.kernel", v + "head.mlp.fc1.weight", L.LINEAR),
            (mh + "mlp.layers.0.bias", v + "head.mlp.fc1.bias", L.ASIS),
            (mh + "mlp.layers.2.kernel", v + "head.mlp.fc2.weight", L.LINEAR),
            (mh + "mlp.layers.2.bias", v + "head.mlp.fc2.bias", L.ASIS),
            (mh + "attn.out.kernel", v + "head.attention.out_proj.weight", L.OUT_W),
            (mh + "attn.out.bias", v + "head.attention.out_proj.bias", L.ASIS),
        ]
        # the MAP head's q/k/v live packed in one (3D, D) / (3D) pair: row blocks 0, 1, 2 (models/siglip.py:249-256,352-363)
        for i, role in enumerate(("query", "key", "value")):
            rules.append((mh + f"attn.{role}.kernel", v + "head.attention.in_proj_weight", L.QKV_W, (i, 3)))
            rules.append((mh + f"attn.{role}.bias", v + "head.attention.in_proj_bias", L.QKV_B, (i, 3)))
        for i in range(t_layers):
            rules += L.block_rules(f"text_model.blocks.layers.{i}.", f"text_model.encoder.layers.{i}.", L.CLIP_BLOCK)
        for i in range(v_layers):
            rules += L.block_rules(f"{v}transformer.blocks.layers.{i}.", f"{v}encoder.layers.{i}.", L.CLIP_BLOCK)
        L.apply_mapping(model, hf, rules, missing="strict", shape_error=ValueError, what="SigLIP ")
        return model


def _join(parts):
    """The results of a call's chunks as one result: tensors concatenated, per-sample lists chained, tuples joined per position."""
    a = parts[0]
    if isinstance(a, torch.Tensor):
        return torch.cat(parts) if len(parts) > 1 else a
    if isinstance(a, list):
        return [x for p in parts for x in p]
    return tuple(_join([p[i] for p in parts]) for i in range(len(a)))


def _host(r):
    if isinstance(r, torch.Tensor):
        return r.cpu()
    return [_host(x) for x in r] if isinstance(r, list) else tuple(_host(x) for x in r)
