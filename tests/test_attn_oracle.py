"""CPU: the attention weights of the oracle (tests/attn_oracle.py) against HuggingFace eager attention with output_attentions=True in
fp64 on the golden fixtures, the MAP head's probe weights against HF's pooling head (nn.MultiheadAttention with need_weights=True,
average_attn_weights=False), and the argument checks of the attention calls, which run before any native handle is built."""

import os

import numpy as np
import pytest
import torch

import attn_oracle as AO
import check_vs_hf as H
import jimm_oracle as O
import naflex_oracle as NF

TOL = 1e-9  # relative, fp64: ViT's eager softmax runs in the model's dtype
# HF's CLIP / SigLIP / SigLIP 2 eager attention takes its softmax in fp32 whatever the model's dtype (softmax(..., dtype=torch.float32)),
# so their weights -- and every later block's input -- carry fp32 rounding even in an fp64 model
TOL_F32_SOFTMAX = 1e-6


def _close(a, b, tol=TOL_F32_SOFTMAX):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert H.rel(a, b) < tol, H.rel(a, b)


def _hf(cls, golden_dir, name):
    m = cls.from_pretrained(os.path.join(golden_dir, name), attn_implementation="eager").eval().double()
    return m, dict(np.load(os.path.join(golden_dir, name, "io.npz")))


def _sd(m):
    return {k: v.detach() for k, v in m.state_dict().items()}


def _tower(m, name):
    """m's vision_model / text_model wrapped as HF's Siglip*VisionModel / *TextModel, which collect the attentions (CLIP's sub-modules
    return them as they are)."""
    import transformers

    sub = getattr(m, name)
    cls = type(m).__name__.replace("Model", "VisionModel" if name == "vision_model" else "TextModel")
    if cls.startswith("CLIP"):
        return sub
    w = getattr(transformers, cls)(getattr(m.config, name.replace("_model", "_config"))).eval().double()
    setattr(w, name, sub)
    return w


def _map_hf(head, x):
    """HF's MAP head weights on its input x [B, S, D]: [B, H, 1, S]."""
    probe = head.probe.repeat(x.shape[0], 1, 1)
    return head.attention(probe, x, x, need_weights=True, average_attn_weights=False)[1]


def test_vit_attentions_match_hf(golden_dir):
    from transformers import ViTForImageClassification

    m, io = _hf(ViTForImageClassification, golden_dir, "tiny_vit")
    c = m.config
    oc = O.ViTCfg(num_classes=c.num_labels, img_size=c.image_size, patch_size=c.patch_size, num_layers=c.num_hidden_layers,
                  num_heads=c.num_attention_heads, mlp_dim=c.intermediate_size, hidden_size=c.hidden_size)
    p = O.hf_to_flax_vit(_sd(m), oc.num_layers, oc.num_heads)
    img = torch.from_numpy(io["images"]).double()
    with torch.no_grad():
        r = m.vit(pixel_values=img.permute(0, 3, 1, 2), output_attentions=True)
        blocks, mw = AO.vit_attn(p, oc, img, O.Semantics(gelu="erf", block_eps=c.layer_norm_eps))
    assert mw is None and len(blocks) == len(r.attentions) == oc.num_layers
    for a, b in zip(blocks, r.attentions):
        _close(a, b, TOL)


def _dual(golden_dir, kind):
    from transformers import CLIPModel, SiglipModel

    m, io = _hf(CLIPModel if kind == "clip" else SiglipModel, golden_dir, f"tiny_{kind}")
    oc = H._dual_cfg(m.config)
    p = (O.hf_to_flax_clip if kind == "clip" else O.hf_to_flax_siglip)(_sd(m), oc)
    return m, io, oc, p, H.hf_semantics(m.config)


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_vision_attentions_match_hf(golden_dir, kind):
    m, io, oc, p, sem = _dual(golden_dir, kind)
    img = torch.from_numpy(io["images"]).double()
    with torch.no_grad():
        r = _tower(m, "vision_model")(pixel_values=img.permute(0, 3, 1, 2), output_attentions=True)
        blocks, mw = (AO.clip_image_attn if kind == "clip" else AO.siglip_image_attn)(p, oc, img, sem)
    assert len(blocks) == len(r.attentions) == oc.vision_layers
    for a, b in zip(blocks, r.attentions):
        _close(a, b)
    if kind == "clip":
        assert mw is None
        return
    with torch.no_grad():
        ref = _map_hf(m.vision_model.head, r.last_hidden_state)
    assert mw.shape == (img.shape[0], oc.v_heads, 1, (oc.image_resolution // oc.vision_patch_size) ** 2)
    _close(mw, ref)
    # the pooled row is the MAP weights' sum over the value rows, as O.map_head computes it
    assert torch.allclose(mw.sum(-1), torch.ones_like(mw.sum(-1)), rtol=0, atol=1e-12)


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_text_attentions_match_hf(golden_dir, kind):
    m, io, oc, p, sem = _dual(golden_dir, kind)
    txt = torch.from_numpy(io["tokens"]).long()
    with torch.no_grad():
        r = _tower(m, "text_model")(input_ids=txt, output_attentions=True)
        blocks = (AO.clip_text_attn if kind == "clip" else AO.siglip_text_attn)(p, oc, txt, sem)
    assert len(blocks) == len(r.attentions) == oc.transformer_layers
    for a, b in zip(blocks, r.attentions):
        _close(a, b)
        if kind == "clip":  # causal: exactly 0 above the diagonal, in HF and in the oracle
            up = torch.triu(torch.ones(a.shape[-1], a.shape[-1], dtype=torch.bool), 1)
            assert (a[..., up] == 0).all() and (b[..., up] == 0).all()


def test_naflex_attentions_match_hf(golden_dir):
    from transformers import Siglip2Model

    m, io = _hf(Siglip2Model, golden_dir, "tiny_siglip2_naflex")
    oc = NF.dual_cfg(m.config)
    p = NF.hf_to_flax_siglip2(_sd(m), oc)
    pv, shapes, mask = (torch.from_numpy(io[k]) for k in ("pixel_values", "spatial_shapes", "pixel_attention_mask"))
    with torch.no_grad():
        r = _tower(m, "vision_model")(pixel_values=pv.double(), pixel_attention_mask=mask, spatial_shapes=shapes, output_attentions=True)
        ours = AO.naflex_attn(p, oc, pv.double(), shapes, H.hf_semantics(m.config))
    for b, (blocks, mw) in enumerate(ours):
        n = int(shapes[b].prod())
        for a, ref in zip(blocks, r.attentions):
            _close(a, ref[b, :, :n, :n])
            assert (ref[b, :, :n, n:] == 0).all()  # HF's padding columns carry no weight
        with torch.no_grad():
            _close(mw, _map_hf(m.vision_model.head, r.last_hidden_state[b:b + 1, :n])[0])


def test_oracle_weights_are_the_oracle_attention():
    """The weights times the values are O.multi_head_attention's output before its out projection, in jimm semantics."""
    oc = O.DualCfg(32, 2, 64, 8, 8, 50, 64, 1, 2)
    p = O.random_dual_params(oc, "siglip", seed=2, dtype=torch.float64)
    x = torch.randn(2, 16, 64, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    pre = "vision_model.transformer.blocks.layers.0.attn."
    w = AO.attention_weights(p, pre, x, x, oc.v_heads)
    D, Hh, d = p[pre + "value.kernel"].shape
    v = (x @ p[pre + "value.kernel"].reshape(D, Hh * d) + p[pre + "value.bias"].reshape(-1)).reshape(2, 16, Hh, d).permute(0, 2, 1, 3)
    o = (w @ v).permute(0, 2, 1, 3).reshape(2, 16, Hh * d) @ p[pre + "out.kernel"].reshape(Hh * d, D) + p[pre + "out.bias"]
    assert torch.allclose(o, O.multi_head_attention(p, pre, x, x, oc.v_heads), rtol=0, atol=1e-12)


# ---- argument checks of the attention calls (no GPU: they must raise before a handle is built) ----
def test_prep_blocks_resolves_requests():
    from jimm_b200._lib import ATTN_MAP
    from jimm_b200._runtime import prep_blocks

    r = prep_blocks(None, 3, torch.float32, False)
    assert not r.single and r.codes == [0, 1, 2] and r.index == [0, 1, 2]
    r = prep_blocks(-1, 3, torch.float16, False)
    assert r.single and r.codes == [2]
    r = prep_blocks("map", 3, torch.float32, True)
    assert r.single and r.codes == [ATTN_MAP]
    r = prep_blocks([-3, "map", 2, 0, -1], 3, torch.bfloat16, True)
    assert not r.single and r.codes == [0, ATTN_MAP, 2] and r.index == [0, 1, 2, 0, 2]
    assert not prep_blocks((1,), 3, torch.float32, False).single
    for bad in (3, -4, 1.0, True, "1", "MAP", [], [0, 7], [None]):
        with pytest.raises(ValueError):
            prep_blocks(bad, 3, torch.float32, True)
    with pytest.raises(ValueError):
        prep_blocks("map", 3, torch.float32, False)  # no MAP head
    for dt in (torch.float64, torch.int32, torch.float8_e4m3fn):
        with pytest.raises(ValueError):
            prep_blocks(0, 3, dt, False)


def test_model_methods_check_before_any_handle():
    from jimm_b200.common.vit import VisionTransformerBase
    from jimm_b200.models import CLIP, SigLIP, VisionTransformer

    vit = VisionTransformer(num_classes=4, img_size=32, patch_size=8, num_layers=2, num_heads=2, mlp_dim=64, hidden_size=64)
    img = torch.zeros(1, 32, 32, 3)
    for kw in (dict(blocks=2), dict(blocks=-3), dict(blocks="map"), dict(blocks=[0, 9]), dict(dtype=torch.float64), dict(blocks="x")):
        with pytest.raises(ValueError):
            vit.forward_attentions(img, **kw)
    with pytest.raises(ValueError):
        vit.forward_attentions(torch.zeros(1, 16, 16, 3))  # the existing input error: not the trained size
    tower = VisionTransformerBase(32, 8, 3, 64, 2, 2, 64)
    with pytest.raises(ValueError):
        tower.forward_attentions(img, blocks="map")  # CLS-pooled
    clip = CLIP(32, 2, 64, 8, 8, 50, 64, 1, 2)
    with pytest.raises(ValueError):
        clip.encode_image_attentions(img, blocks="map")
    with pytest.raises(ValueError):
        clip.encode_text_attentions(torch.zeros(2, 8, dtype=torch.long), blocks="map")
    with pytest.raises(ValueError):
        clip.encode_text_attentions(torch.zeros(2, 9, dtype=torch.long))  # longer than context_length
    sig = SigLIP(32, 2, 64, 8, 8, 50, 64, 1, 2)
    with pytest.raises(ValueError):
        sig.encode_image_attentions(img, blocks=[0, 2])
    with pytest.raises(ValueError):
        sig.encode_image_attentions(img, spatial_shapes=torch.tensor([[4, 4]]))  # NaFlex inputs on a SigLIP model
    with pytest.raises(ValueError):
        sig.encode_text_attentions(torch.zeros(1, 8, dtype=torch.long), dtype=torch.int8)
    for m in (vit, tower, clip, sig):
        assert m._native is None
