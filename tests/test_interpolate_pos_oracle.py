"""CPU: the interpolate_pos_encoding oracle (tests/interp_oracle.py) against HuggingFace's interpolate_pos_encoding=True on tiny
random-init ViT, CLIP and SigLIP models in float64, and its resampler against F.interpolate."""

import pytest
import torch
import torch.nn.functional as F

import check_vs_hf as H
import interp_oracle as I
import jimm_oracle as O

# tiny models: 32 x 32 images, patch 8 -> a 4 x 4 trained grid
SIZES = [(40, 48), (24, 24), (36, 36)]  # up-sampled and non-square | down-sampled | floors to the trained grid


def _img(B, h, w, dtype=torch.float64):
    g = torch.Generator().manual_seed(h * 1000 + w)
    return torch.rand((B, h, w, 3), generator=g, dtype=torch.float32).to(dtype) * 2 - 1


@pytest.mark.parametrize("hw", SIZES)
def test_vit_matches_hf(hw):
    from transformers import ViTForImageClassification

    torch.manual_seed(0)
    cfg = H.tiny_vit_config()
    m = H.perturb_(ViTForImageClassification(cfg)).eval().to(torch.float64)
    oc = O.ViTCfg(num_classes=cfg.num_labels, img_size=cfg.image_size, patch_size=cfg.patch_size, num_layers=cfg.num_hidden_layers,
                  num_heads=cfg.num_attention_heads, mlp_dim=cfg.intermediate_size, hidden_size=cfg.hidden_size)
    p = O.hf_to_flax_vit({k: v.detach() for k, v in m.state_dict().items()}, oc.num_layers, oc.num_heads)
    img = _img(2, *hw)
    sem = O.Semantics(gelu="erf", block_eps=cfg.layer_norm_eps)
    with torch.no_grad():
        ref = m(pixel_values=img.permute(0, 3, 1, 2), interpolate_pos_encoding=True).logits
        out = I.vit_forward(p, oc, img, sem, interpolate_pos_encoding=True)
    assert H.rel(out, ref) < 1e-9
    if hw == (36, 36):
        with torch.no_grad():
            assert torch.equal(out, O.vit_forward(p, oc, img, sem))


@pytest.mark.parametrize("hw", SIZES)
def test_clip_matches_hf(hw):
    from transformers import CLIPModel

    torch.manual_seed(0)
    cfg = H.tiny_clip_config()
    m = H.perturb_(CLIPModel(cfg)).eval().to(torch.float64)
    oc = H._dual_cfg(cfg)
    p = O.hf_to_flax_clip({k: v.detach() for k, v in m.state_dict().items()}, oc)
    img = _img(3, *hw)
    txt = O.synthetic_tokens(4, oc.context_length, oc.vocab_size, "clip")
    sem = O.Semantics(block_eps=cfg.vision_config.layer_norm_eps)
    with torch.no_grad():
        ref = m(pixel_values=img.permute(0, 3, 1, 2), input_ids=txt, interpolate_pos_encoding=True).logits_per_image
        out = I.clip_forward(p, oc, img, txt, sem=sem, interpolate_pos_encoding=True)
    assert H.rel(out, ref) < 1e-9
    if hw == (36, 36):
        with torch.no_grad():
            assert torch.equal(out, O.clip_forward(p, oc, img, txt, sem))


@pytest.mark.parametrize("hw", SIZES)
def test_siglip_matches_hf(hw):
    from transformers import SiglipModel

    torch.manual_seed(0)
    cfg = H.tiny_siglip_config()
    m = H.perturb_(SiglipModel(cfg)).eval().to(torch.float64)
    with torch.no_grad():
        m.logit_scale.fill_(2.3)
        m.logit_bias.fill_(-1.7)
    oc = H._dual_cfg(cfg)
    p = O.hf_to_flax_siglip({k: v.detach() for k, v in m.state_dict().items()}, oc)
    img = _img(3, *hw)
    txt = O.synthetic_tokens(4, oc.context_length, oc.vocab_size, "siglip")
    pix = img.permute(0, 3, 1, 2)
    with torch.no_grad():
        ref_i = m.vision_model(pixel_values=pix, interpolate_pos_encoding=True).pooler_output
        ref_l = m(pixel_values=pix, input_ids=txt, interpolate_pos_encoding=True).logits_per_image
        ie = I.siglip_encode_image(p, oc, img, interpolate_pos_encoding=True)
        lg = I.siglip_forward(p, oc, img, txt, interpolate_pos_encoding=True)
    assert H.rel(ie, ref_i) < 1e-9 and H.rel(lg, ref_l) < 1e-9
    if hw == (36, 36):
        with torch.no_grad():
            assert torch.equal(ie, O.siglip_encode_image(p, oc, img))


@pytest.mark.parametrize("cls", [True, False])
@pytest.mark.parametrize("g,gh,gw", [(14, 24, 24), (14, 7, 7), (14, 18, 10), (16, 32, 32), (1, 3, 5), (4, 4, 4)])
def test_resampler_is_f_interpolate(cls, g, gh, gw):
    D, off = 32, int(cls)
    pos = torch.randn((1, off + g * g, D), generator=torch.Generator().manual_seed(g * 100 + gh), dtype=torch.float64)
    out = I.resample_pos(pos, g, gh, gw, cls)
    ref = F.interpolate(pos[0, off:].T.reshape(1, D, g, g), size=(gh, gw), mode="bicubic", align_corners=False)
    assert torch.equal(out[0, off:], ref[0].reshape(D, gh * gw).T)
    assert torch.equal(out[0, :off], pos[0, :off])
    # the native grid is the table itself, and so is resampling to it
    assert torch.equal(I.resample_pos(pos, g, g, g, cls), pos)
    same = F.interpolate(pos[0, off:].T.reshape(1, D, g, g), size=(g, g), mode="bicubic", align_corners=False)
    assert torch.equal(same[0].reshape(D, g * g).T, pos[0, off:])
