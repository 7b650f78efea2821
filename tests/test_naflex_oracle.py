"""CPU: the SigLIP 2 NaFlex restatement (tests/naflex_oracle.py) against HuggingFace Siglip2Model, the committed fixture, and the
loader / input checks of SigLIP(..., naflex=True) that run before any GPU work."""

import math
import os

import numpy as np
import pytest
import torch

import check_vs_hf as H
import jimm_oracle as O
import naflex_oracle as N


def _hf_model(dtype=torch.float64, seed=0):
    from transformers import Siglip2Model

    torch.manual_seed(seed)
    m = H.perturb_(Siglip2Model(N.tiny_siglip2_config())).eval().to(dtype)
    with torch.no_grad():
        m.logit_scale.fill_(2.3)
        m.logit_bias.fill_(-1.7)
    return m


def test_oracle_matches_hf_fp64_padded_mixed_shapes():
    """A batch padded to max_num_patches with grids below, at and above the 16 x 16 table, non-square and one row: the oracle runs
    each sample alone, HF runs the padded batch under pixel_attention_mask."""
    m = _hf_model()
    oc = N.dual_cfg(m.config)
    P = oc.vision_patch_size
    g = torch.Generator().manual_seed(5)
    imgs = [torch.rand((h * P, w * P, 3), generator=g, dtype=torch.float64) * 2 - 1 for h, w in N.GOLDEN_SHAPES]
    pv, shapes, mask = N.pad_batch(imgs, P, N.GOLDEN_MAX_PATCHES, fill=0.7)
    txt = O.synthetic_tokens(5, oc.context_length, oc.vocab_size, "siglip")
    p = N.hf_to_flax_siglip2({k: v.detach() for k, v in m.state_dict().items()}, oc)
    with torch.no_grad():
        kw = dict(pixel_values=pv, pixel_attention_mask=mask, spatial_shapes=shapes)
        ref_i, ref_t = m.get_image_features(**kw).pooler_output, m.get_text_features(input_ids=txt).pooler_output
        ref_l = m(input_ids=txt, **kw).logits_per_image
        out_i = N.encode_patches(p, oc, pv, shapes)
        out_t = O.siglip_encode_text(p, oc, txt)
        out_l = N.forward(p, oc, pv, shapes, txt)
    assert H.rel(out_i, ref_i) < 1e-9 and H.rel(out_t, ref_t) < 1e-9 and H.rel(out_l, ref_l) < 1e-9
    # the NHWC form of the same pixels
    assert H.rel(N.encode_images(p, oc, imgs), ref_i) < 1e-9


def test_resample_identity_at_table_grid():
    pos = torch.randn((1, 256, 40))
    assert torch.equal(N.resample_pos_aa(pos, 16, 16, 16), pos)


def test_golden_naflex(golden_dir):
    from safetensors.torch import load_file

    d = os.path.join(golden_dir, "tiny_siglip2_naflex")
    io = dict(np.load(os.path.join(d, "io.npz")))
    sd = load_file(os.path.join(d, "model.safetensors"))
    oc = O.DualCfg(64, 2, 64, 4, 16, 100, 64, 1, 1)
    p = O.cast_params(N.hf_to_flax_siglip2(sd, oc), torch.float64)
    pv, shapes = torch.from_numpy(io["pixel_values"]).double(), torch.from_numpy(io["spatial_shapes"])
    txt = torch.from_numpy(io["tokens"]).long()
    assert [tuple(s) for s in shapes.tolist()] == N.GOLDEN_SHAPES
    np.testing.assert_allclose(N.encode_patches(p, oc, pv, shapes).float().numpy(), io["hf_image_embeds"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(O.siglip_encode_text(p, oc, txt).float().numpy(), io["hf_text_embeds"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(N.forward(p, oc, pv, shapes, txt).float().numpy(), io["hf_logits"], rtol=0, atol=1e-4)


def test_from_pretrained_naflex_tree(golden_dir):
    from safetensors.torch import load_file

    from jimm_b200 import _lib
    from jimm_b200.models import SigLIP

    path = os.path.join(golden_dir, "tiny_siglip2_naflex", "model.safetensors")
    m = SigLIP.from_pretrained(path)
    oc = O.DualCfg(64, 2, 64, 4, 16, 100, 64, 1, 1)
    flat, ref = m.flat_params(), N.hf_to_flax_siglip2(load_file(path), oc)
    assert set(flat) == set(ref), set(flat) ^ set(ref)
    for k, v in ref.items():
        assert tuple(flat[k].shape) == tuple(v.shape) and torch.equal(flat[k], v.to(torch.float32)), k
    assert m.naflex and (m.image_resolution, m.vision_patch_size, m.vision_width) == (64, 4, 64)
    cfg = m._native_config()
    assert cfg.kind == _lib.KIND_SIGLIP_NAFLEX and cfg.img_size == 64 and cfg.patch == 4
    assert cfg.pooling == _lib.POOL_MAP and cfg.pre_norm == 0 and cfg.patch_bias == 1


def test_from_pretrained_naflex_non_square_table(golden_dir, tmp_path):
    import shutil

    from safetensors.torch import load_file, save_file

    from jimm_b200.models import SigLIP

    d = os.path.join(golden_dir, "tiny_siglip2_naflex")
    sd = load_file(os.path.join(d, "model.safetensors"))
    k = "vision_model.embeddings.position_embedding.weight"
    sd[k] = sd[k][:250].contiguous()
    assert math.isqrt(250) ** 2 != 250
    save_file(sd, str(tmp_path / "model.safetensors"))
    shutil.copy(os.path.join(d, "config.json"), tmp_path / "config.json")
    with pytest.raises(ValueError, match="not a square grid"):
        SigLIP.from_pretrained(str(tmp_path / "model.safetensors"))


def test_naflex_input_checks(golden_dir):
    """Refused in the input step, before a native handle is built (so on a machine without a GPU too)."""
    from jimm_b200.models import SigLIP

    d = os.path.join(golden_dir, "tiny_siglip2_naflex")
    io = dict(np.load(os.path.join(d, "io.npz")))
    m = SigLIP.from_pretrained(os.path.join(d, "model.safetensors"))
    pv, shapes, mask = io["pixel_values"], io["spatial_shapes"], io["pixel_attention_mask"]
    bad = mask.copy()
    bad[1, 200] = 1  # sample 1 is 8 x 24 = 192 patches
    with pytest.raises(ValueError, match="pixel_attention_mask"):
        m.encode_image(pv, spatial_shapes=shapes, pixel_attention_mask=bad)
    with pytest.raises(ValueError, match="pixel_attention_mask"):
        m(pv, io["tokens"], spatial_shapes=shapes, pixel_attention_mask=bad)
    bad = mask.copy()
    bad[3, 0] = 0
    with pytest.raises(ValueError, match="pixel_attention_mask"):
        m.encode_image(pv, spatial_shapes=shapes, pixel_attention_mask=bad)
    big = shapes.copy()
    big[0] = (17, 16)  # 272 patches > max_num_patches 256
    with pytest.raises(ValueError, match="max_num_patches"):
        m.encode_image(pv, spatial_shapes=big)
    zero = shapes.copy()
    zero[2] = (0, 5)
    with pytest.raises(ValueError, match="spatial shape"):
        m.encode_image(pv, spatial_shapes=zero)
    with pytest.raises(ValueError, match="pixel_values"):
        m.encode_image(pv[:, :, :40], spatial_shapes=shapes)
    with pytest.raises(ValueError, match="needs the spatial_shapes"):
        m.encode_image(pv, pixel_attention_mask=mask)
    plain = SigLIP.from_pretrained(os.path.join(golden_dir, "tiny_siglip", "model.safetensors"))
    assert not plain.naflex
    with pytest.raises(ValueError, match="NaFlex"):
        plain.encode_image(pv, spatial_shapes=shapes)
    with pytest.raises(ValueError, match="multiple of vision_patch_size"):
        SigLIP(62, 1, 128, 4, 16, 100, 128, 2, 1, naflex=True)
