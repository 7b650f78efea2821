"""CPU restatement of interpolate_pos_encoding for the tests: the oracle's towers on images of any size.

HuggingFace's ViTEmbeddings / CLIPVisionEmbeddings / SiglipVisionEmbeddings.interpolate_pos_encoding view the patch rows of the
position table ([g*g, D], after the CLS row if there is one) as a [D, g, g] image, resample it with
torch.nn.functional.interpolate(mode="bicubic", align_corners=False) to the image's patch grid (H // P, W // P), and keep the CLS row.
Here that table replaces the trained one in a copy of the parameters, in the parameters' dtype, and jimm_oracle's forwards run
unchanged (their patch embedding already drops the trailing pixels, like the VALID conv).  jimm_oracle itself is the parity
yardstick of the native size and stays as it is."""

from __future__ import annotations

import torch
import torch.nn.functional as F

import jimm_oracle as O


def resample_pos(pos: torch.Tensor, g: int, gh: int, gw: int, cls: bool) -> torch.Tensor:
    """pos [1, (1 +) g*g, D] -> [1, (1 +) gh*gw, D]: the patch rows resampled bicubically, tokens row-major over (gh, gw)."""
    if (gh, gw) == (g, g):
        return pos
    off = 1 if cls else 0
    D = pos.shape[-1]
    grid = pos[0, off:].reshape(g, g, D).permute(2, 0, 1).unsqueeze(0)
    r = F.interpolate(grid, size=(gh, gw), mode="bicubic", align_corners=False)
    return torch.cat([pos[:, :off], r[0].permute(1, 2, 0).reshape(1, gh * gw, D)], 1)


def with_grid(p: O.Params, prefix: str, tower: O.TowerCfg, H: int, W: int) -> O.Params:
    """A copy of p whose position table fits H x W images."""
    P, k = tower.patch_size, prefix + "position_embeddings"
    return {**p, k: resample_pos(p[k], tower.img_size // P, H // P, W // P, tower.pooling_type == "CLS")}


def vision_tower(p, prefix, img, cfg: O.TowerCfg, sem=O.JIMM, interpolate_pos_encoding=False):
    if interpolate_pos_encoding:
        p = with_grid(p, prefix, cfg, img.shape[1], img.shape[2])
    return O.vision_tower(p, prefix, img, cfg, sem)


def vit_forward(p, cfg: O.ViTCfg, img, sem=O.JIMM, interpolate_pos_encoding=False):
    if interpolate_pos_encoding:
        p = with_grid(p, "encoder.", cfg.tower(), img.shape[1], img.shape[2])
    return O.vit_forward(p, cfg, img, sem)


def _dual(fn, tower):
    def run(p, cfg: O.DualCfg, img, *rest, sem=O.JIMM, interpolate_pos_encoding=False):
        if interpolate_pos_encoding:
            p = with_grid(p, "vision_model.", tower(cfg), img.shape[1], img.shape[2])
        return fn(p, cfg, img, *rest, sem)

    return run


clip_encode_image = _dual(O.clip_encode_image, O.DualCfg.clip_tower)
clip_forward = _dual(O.clip_forward, O.DualCfg.clip_tower)
siglip_encode_image = _dual(O.siglip_encode_image, O.DualCfg.siglip_tower)
siglip_forward = _dual(O.siglip_forward, O.DualCfg.siglip_tower)
