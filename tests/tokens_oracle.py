"""CPU restatement of the per-token hidden states of the vision and text towers, on jimm_oracle's layers.

x_k is a tower's residual stream after k of its L blocks: x_0 the embeddings (vision: patch embedding + position table, CLS row first
on CLS towers, after ln_pre when the tower has it; text: token embedding + positions), x_L what the final norm reads.  Each function here
returns the list [x_0, ..., x_L, final], `final` being the final-normed tokens: ln_post(x_L) for a vision tower, ln_final(x_L) for a
text tower -- the tensors the pooled calls pool from.  The arithmetic is jimm_oracle's, step for step: the last entry's pooled row is
what jimm_oracle's pooled functions pool.
"""

from __future__ import annotations

from typing import List

import torch

import jimm_oracle as O
import naflex_oracle as NF


def _blocks(p: O.Params, prefix: str, x, layers, num_heads, use_quick_gelu, mask, sem: O.Semantics) -> List[torch.Tensor]:
    """[x_0, ..., x_L] of O.transformer (common/transformer.py:171-196), block eps 1e-6 unless sem overrides it."""
    eps = sem.block_eps if sem.block_eps is not None else 1e-6
    xs = [x]
    for i in range(layers):
        xs.append(O.transformer_encoder(p, f"{prefix}blocks.layers.{i}.", xs[-1], num_heads, eps, use_quick_gelu, mask, sem))
    return xs


def vision_hidden(p: O.Params, prefix: str, img, cfg: O.TowerCfg, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    """O.vision_tower up to its pooling head: [x_0, ..., x_L, ln_post(x_L)], each [B, S, D]."""
    x = O.patch_embed(p, prefix, img, cfg, sem)
    B = x.shape[0]
    if cfg.pooling_type == "CLS":
        x = torch.cat([O._prm(p[prefix + "cls_token"], sem).expand(B, -1, -1), x], dim=1)
    x = O._out(x + O._prm(p[prefix + "position_embeddings"], sem), sem)
    if cfg.use_pre_norm:
        x = O.layer_norm(x, p[prefix + "ln_pre.scale"], p[prefix + "ln_pre.bias"], cfg.layernorm_epsilon, sem)
    xs = _blocks(p, prefix + "transformer.", x, cfg.num_layers, cfg.num_heads, cfg.use_quick_gelu, None, sem)
    return xs + [O.layer_norm(xs[-1], p[prefix + "ln_post.scale"], p[prefix + "ln_post.bias"], cfg.layernorm_epsilon, sem)]


def vit_hidden(p: O.Params, cfg: O.ViTCfg, img, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    return vision_hidden(p, "encoder.", img, cfg.tower(), sem)


def clip_image_hidden(p: O.Params, cfg: O.DualCfg, img, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    return vision_hidden(p, "vision_model.", img, cfg.clip_tower(), sem)


def siglip_image_hidden(p: O.Params, cfg: O.DualCfg, img, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    return vision_hidden(p, "vision_model.", img, cfg.siglip_tower(), sem)


def _text_hidden(p: O.Params, cfg: O.DualCfg, text, kind: str, sem: O.Semantics) -> List[torch.Tensor]:
    """O.clip_encode_text / O.siglip_encode_text up to the pooling: [x_0, ..., x_L, ln_final(x_L)], each [B, T, D]."""
    seq = text.shape[1]
    x = O._prm(p["token_embedding.embedding"][text], sem)
    x = O._out(x + O._prm(p["positional_embedding"][:seq], sem), sem)
    mask = torch.tril(torch.ones(cfg.context_length, cfg.context_length, dtype=x.dtype)) if kind == "clip" else None
    xs = _blocks(p, "text_model.", x, cfg.transformer_layers, cfg.transformer_heads, cfg.text_quick(kind), mask, sem)
    eps = 1e-5 if kind == "clip" else 1e-6  # models/clip.py:117, models/siglip.py:104
    return xs + [O.layer_norm(xs[-1], p["ln_final.scale"], p["ln_final.bias"], eps, sem)]


def clip_text_hidden(p: O.Params, cfg: O.DualCfg, text, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    return _text_hidden(p, cfg, text, "clip", sem)


def siglip_text_hidden(p: O.Params, cfg: O.DualCfg, text, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    return _text_hidden(p, cfg, text, "siglip", sem)


def naflex_hidden(p: O.Params, cfg: O.DualCfg, pixel_values, spatial_shapes, sem: O.Semantics = O.JIMM) -> List[List[torch.Tensor]]:
    """SigLIP 2 NaFlex on the processor's pixel_values: per sample b, [x_0, ..., x_L, ln_post(x_L)], each [gh_b * gw_b, D] (the position
    table resampled to the sample's grid, as naflex_oracle.encode_patches does)."""
    t = NF.naflex_tower(cfg)
    P, g, k = t.patch_size, t.img_size // t.patch_size, "vision_model.position_embeddings"
    out = []
    for b, (gh, gw) in enumerate(torch.as_tensor(spatial_shapes).tolist()):
        img = NF.rows_to_image(pixel_values[b, : gh * gw], gh, gw, P)[None]
        pb = {**p, k: NF.resample_pos_aa(p[k], g, gh, gw)}
        out.append([x[0] for x in vision_hidden(pb, "vision_model.", img, t, sem)])
    return out
