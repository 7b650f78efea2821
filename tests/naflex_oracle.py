"""CPU restatement of the SigLIP 2 NaFlex vision tower (HF `Siglip2Model`) for the tests, on jimm_oracle's SigLIP tower.

NaFlex differs from SigLIP in three places, all before the encoder:
  - the patch embedding is a Linear over flattened patches, each row in (py, px, c) order (Siglip2ImageProcessor's
    reshape(C, gh, P, gw, P).permute(1, 3, 2, 4, 0)); that is the conv kernel reshaped, so a sample's patch rows are the pixels of a
    (gh*P) x (gw*P) image and jimm_oracle's patch embedding of that image is the same GEMM;
  - the g x g position table is resampled to each sample's patch grid (gh, gw) with F.interpolate(mode="bilinear",
    align_corners=False, antialias=True) -- in fp32 and cast back to the parameters' dtype, as Siglip2VisionEmbeddings does on the CPU;
  - samples are padded to max_num_patches rows and pixel_attention_mask hides the padding from attention and the MAP head.  Here each
    sample runs on its own, which is what the mask computes.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import check_vs_hf as H
import jimm_oracle as O


def image_to_rows(img: torch.Tensor, P: int) -> torch.Tensor:
    """NHWC image [H, W, C] -> patch rows [(H // P) * (W // P), P*P*C], row-major over the grid, each row in (py, px, c) order (the
    processor's convert_image_to_patches; trailing pixels that do not fill a patch dropped)."""
    H, W, C = img.shape
    gh, gw = H // P, W // P
    return img[: gh * P, : gw * P].reshape(gh, P, gw, P, C).permute(0, 2, 1, 3, 4).reshape(gh * gw, P * P * C)


def rows_to_image(rows: torch.Tensor, gh: int, gw: int, P: int) -> torch.Tensor:
    """The inverse of image_to_rows: gh*gw patch rows -> the NHWC image [gh*P, gw*P, C] they cut into."""
    C = rows.shape[-1] // (P * P)
    return rows.reshape(gh, gw, P, P, C).permute(0, 2, 1, 3, 4).reshape(gh * P, gw * P, C)


def pad_batch(images, P: int, max_num_patches: int, fill: float = 0.0):
    """NHWC images of their own sizes -> (pixel_values [B, max_num_patches, P*P*C], spatial_shapes [B, 2], pixel_attention_mask [B, N]),
    the layout Siglip2ImageProcessor returns; padding rows hold `fill`."""
    rows = [image_to_rows(x, P) for x in images]
    C = images[0].shape[-1]
    pv = torch.full((len(images), max_num_patches, P * P * C), fill, dtype=images[0].dtype)
    mask = torch.zeros((len(images), max_num_patches), dtype=torch.int32)
    for b, r in enumerate(rows):
        pv[b, : r.shape[0]] = r
        mask[b, : r.shape[0]] = 1
    shapes = torch.tensor([[x.shape[0] // P, x.shape[1] // P] for x in images], dtype=torch.int64)
    return pv, shapes, mask


def resample_pos_aa(pos: torch.Tensor, g: int, gh: int, gw: int) -> torch.Tensor:
    """pos [1, g*g, D] -> [1, gh*gw, D]: Siglip2VisionEmbeddings.resize_positional_embeddings for one sample."""
    D = pos.shape[-1]
    grid = pos[0].reshape(g, g, D).permute(2, 0, 1).unsqueeze(0).to(torch.float32)
    r = F.interpolate(grid, size=(gh, gw), mode="bilinear", align_corners=False, antialias=True)
    return r[0].reshape(D, gh * gw).T.reshape(1, gh * gw, D).to(pos.dtype)


def naflex_tower(cfg: O.DualCfg) -> O.TowerCfg:
    return cfg.siglip_tower()


def encode_patches(p: O.Params, cfg: O.DualCfg, pixel_values: torch.Tensor, spatial_shapes, sem=O.JIMM) -> torch.Tensor:
    """SigLIP 2 NaFlex get_image_features(pixel_values, pixel_attention_mask, spatial_shapes).pooler_output: [B, D]."""
    t = naflex_tower(cfg)
    P, g, k = t.patch_size, t.img_size // t.patch_size, "vision_model.position_embeddings"
    out = []
    for b, (gh, gw) in enumerate(torch.as_tensor(spatial_shapes).tolist()):
        img = rows_to_image(pixel_values[b, : gh * gw], gh, gw, P)[None]
        pb = {**p, k: resample_pos_aa(p[k], g, gh, gw)}
        out.append(O.vision_tower(pb, "vision_model.", img, t, sem))
    return torch.cat(out)


def encode_images(p: O.Params, cfg: O.DualCfg, images, sem=O.JIMM) -> torch.Tensor:
    """NaFlex image embeddings of NHWC images of their own sizes (trailing pixels dropped)."""
    P = cfg.vision_patch_size
    return torch.cat([encode_patches(p, cfg, image_to_rows(x, P)[None], [[x.shape[0] // P, x.shape[1] // P]], sem) for x in images])


def forward(p: O.Params, cfg: O.DualCfg, pixel_values, spatial_shapes, text, sem=O.JIMM) -> torch.Tensor:
    """Siglip2Model(...).logits_per_image."""
    return O.contrastive_logits(encode_patches(p, cfg, pixel_values, spatial_shapes, sem), O.siglip_encode_text(p, cfg, text, sem),
                                p["logit_scale"], p["logit_bias"], sem)


def hf_to_flax_siglip2(sd, cfg: O.DualCfg) -> O.Params:
    """HF Siglip2Model state dict -> SigLIP's flax parameter tree: jimm_oracle's SigLIP transforms, with the patch Linear weight
    (D, P*P*C) unflattened to the (P, P, C, D) kernel."""
    k = "vision_model.embeddings.patch_embedding.weight"
    w = sd[k]
    P, D = cfg.vision_patch_size, w.shape[0]
    C = w.shape[1] // (P * P)
    o = O.hf_to_flax_siglip({**sd, k: w.new_zeros((D, C, P, P))}, cfg)
    o["vision_model.patch_embeddings.kernel"] = w.T.reshape(P, P, C, D).contiguous()
    return o


def dual_cfg(cfg) -> O.DualCfg:
    """O.DualCfg of a Siglip2Config (image_resolution = sqrt(num_patches) * patch_size)."""
    t, v = cfg.text_config, cfg.vision_config
    g = math.isqrt(v.num_patches)
    return O.DualCfg(image_resolution=g * v.patch_size, vision_layers=v.num_hidden_layers, vision_width=v.hidden_size,
                     vision_patch_size=v.patch_size, context_length=t.max_position_embeddings, vocab_size=t.vocab_size,
                     transformer_width=t.hidden_size, transformer_heads=t.num_attention_heads, transformer_layers=t.num_hidden_layers,
                     **H.arch_fields(cfg))


def tiny_siglip2_config():
    """The tiny NaFlex config of the golden fixture: a 16 x 16 position table at patch 4, width 64 (one head of 64), two vision layers
    and one text layer, so the checkpoint stays under 1 MB."""
    from transformers import Siglip2Config

    return Siglip2Config(
        text_config=dict(hidden_size=64, num_attention_heads=1, num_hidden_layers=1, intermediate_size=256,
                         max_position_embeddings=16, vocab_size=100, projection_size=64),
        vision_config=dict(hidden_size=64, num_attention_heads=1, num_hidden_layers=2, intermediate_size=256,
                           num_patches=256, patch_size=4),
    )


# (patch rows, patch columns) of the fixture's padded batch at max_num_patches 256: the table's own grid, below 16 on an axis (the
# antialias branch), above, non-square, one row, and both axes downscaled
GOLDEN_SHAPES = [(16, 16), (8, 24), (20, 12), (1, 37), (5, 5), (32, 8), (7, 30)]
GOLDEN_MAX_PATCHES = 256
