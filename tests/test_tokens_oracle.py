"""CPU: the per-token hidden states of the oracle (tests/tokens_oracle.py) against HuggingFace output_hidden_states=True in fp64, and the
argument checks of the per-token calls, which run before any native handle is built.

HF mapping (hidden_states[k] is x_k in every family):
  ViT, SigLIP / SigLIP 2 vision, CLIP / SigLIP text: last_hidden_state is the final-normed tokens (layer None);
  CLIP vision: hidden_states[0] is after pre_layrnorm, and last_hidden_state is x_L (layer -1): HF does not apply post_layernorm to
  the tokens, only to the pooled CLS row."""

import pytest
import torch

import check_vs_hf as H
import jimm_oracle as O
import naflex_oracle as NF
import tokens_oracle as TO

TOL = 1e-9  # relative, fp64: the layouts, masks and norms are exact


def _check(xs, hidden_states, last, last_index):
    assert len(xs) == len(hidden_states) + 1
    for k, (a, b) in enumerate(zip(xs, hidden_states)):
        assert H.rel(a, b) < TOL, (k, H.rel(a, b))
    assert H.rel(xs[last_index], last) < TOL, H.rel(xs[last_index], last)


def test_vit_hidden_states_match_hf():
    from transformers import ViTForImageClassification

    torch.manual_seed(0)
    cfg = H.tiny_vit_config()
    m = H.perturb_(ViTForImageClassification(cfg)).eval().double()
    oc = O.ViTCfg(num_classes=cfg.num_labels, img_size=cfg.image_size, patch_size=cfg.patch_size, num_layers=cfg.num_hidden_layers,
                  num_heads=cfg.num_attention_heads, mlp_dim=cfg.intermediate_size, hidden_size=cfg.hidden_size)
    p = O.hf_to_flax_vit({k: v.detach() for k, v in m.state_dict().items()}, oc.num_layers, oc.num_heads)
    img = O.synthetic_images(2, cfg.image_size, dtype=torch.float64)
    with torch.no_grad():
        r = m.vit(pixel_values=img.permute(0, 3, 1, 2), output_hidden_states=True)
        xs = TO.vit_hidden(p, oc, img, O.Semantics(gelu="erf", block_eps=cfg.layer_norm_eps))
    _check(xs, r.hidden_states, r.last_hidden_state, -1)
    # the final-normed CLS row is what the classifier reads
    with torch.no_grad():
        logits = O.vit_forward(p, oc, img, O.Semantics(gelu="erf", block_eps=cfg.layer_norm_eps))
    assert H.rel(O.linear(xs[-1][:, 0], p["classifier.kernel"], p["classifier.bias"]), logits) < TOL


def _tower(m, name):
    """m's vision_model / text_model with output_hidden_states wired: SigLIP's sub-modules collect hidden states only under their
    SiglipVisionModel / SiglipTextModel wrappers (CLIP's return them as they are)."""
    import transformers

    sub = getattr(m, name)
    cls = type(m).__name__.replace("Model", "VisionModel" if name == "vision_model" else "TextModel")
    if cls.startswith("CLIP"):
        return sub
    w = getattr(transformers, cls)(getattr(m.config, name.replace("_model", "_config"))).eval().double()
    setattr(w, name, sub)
    return w


def _dual(kind):
    from transformers import CLIPModel, SiglipModel

    torch.manual_seed(0)
    cfg = H.tiny_clip_config() if kind == "clip" else H.tiny_siglip_config()
    m = H.perturb_((CLIPModel if kind == "clip" else SiglipModel)(cfg)).eval().double()
    oc = H._dual_cfg(cfg)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    p = O.hf_to_flax_clip(sd, oc) if kind == "clip" else O.hf_to_flax_siglip(sd, oc)
    return m, cfg, oc, p, H.hf_semantics(cfg)


def test_clip_vision_hidden_states_match_hf():
    m, cfg, oc, p, sem = _dual("clip")
    img = O.synthetic_images(2, oc.image_resolution, dtype=torch.float64)
    with torch.no_grad():
        r = m.vision_model(pixel_values=img.permute(0, 3, 1, 2), output_hidden_states=True)
        xs = TO.clip_image_hidden(p, oc, img, sem)
        pooled = O.clip_encode_image(p, oc, img, sem)
    _check(xs, r.hidden_states, r.last_hidden_state, -2)  # last_hidden_state is x_L, not post-normed
    assert H.rel(xs[-1][:, 0], r.pooler_output) < TOL  # post_layernorm of the CLS row
    assert H.rel(O.linear(xs[-1][:, 0], p["visual_projection.kernel"]), pooled) < TOL


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_text_hidden_states_match_hf(kind):
    m, cfg, oc, p, sem = _dual(kind)
    txt = O.synthetic_tokens(3, oc.context_length, oc.vocab_size, kind)
    with torch.no_grad():
        r = _tower(m, "text_model")(input_ids=txt, output_hidden_states=True)
        xs = (TO.clip_text_hidden if kind == "clip" else TO.siglip_text_hidden)(p, oc, txt, sem)
        pooled = (O.clip_encode_text if kind == "clip" else O.siglip_encode_text)(p, oc, txt, sem)
    _check(xs, r.hidden_states, r.last_hidden_state, -1)
    rows = txt.argmax(-1) if kind == "clip" else torch.full((txt.shape[0],), txt.shape[1] - 1)
    f = xs[-1][torch.arange(txt.shape[0]), rows]
    head = O.linear(f, p["text_projection.kernel"], p.get("text_projection.bias"))
    assert H.rel(head, pooled) < TOL


def test_siglip_vision_hidden_states_match_hf():
    m, cfg, oc, p, sem = _dual("siglip")
    img = O.synthetic_images(2, oc.image_resolution, dtype=torch.float64)
    with torch.no_grad():
        r = _tower(m, "vision_model")(pixel_values=img.permute(0, 3, 1, 2), output_hidden_states=True)
        xs = TO.siglip_image_hidden(p, oc, img, sem)
    _check(xs, r.hidden_states, r.last_hidden_state, -1)
    assert H.rel(O.map_head(p, "vision_model.MAPHead.", xs[-1], oc.v_heads, 1e-6, sem), r.pooler_output) < TOL


def test_naflex_hidden_states_match_hf():
    from transformers import Siglip2Model

    torch.manual_seed(0)
    cfg = NF.tiny_siglip2_config()
    m = H.perturb_(Siglip2Model(cfg)).eval().double()
    oc = NF.dual_cfg(cfg)
    p = NF.hf_to_flax_siglip2({k: v.detach() for k, v in m.state_dict().items()}, oc)
    P = oc.vision_patch_size
    g = torch.Generator().manual_seed(5)
    images = [torch.randn(h * P, w * P, 3, generator=g, dtype=torch.float64) for h, w in [(16, 16), (8, 24), (5, 7)]]
    pv, shapes, mask = NF.pad_batch(images, P, 256)
    with torch.no_grad():
        r = _tower(m, "vision_model")(pixel_values=pv, pixel_attention_mask=mask, spatial_shapes=shapes, output_hidden_states=True)
        hs = TO.naflex_hidden(p, oc, pv, shapes, H.hf_semantics(cfg))
    for b, xs in enumerate(hs):
        n = int(shapes[b].prod())
        _check(xs, [h[b, :n] for h in r.hidden_states], r.last_hidden_state[b, :n], -1)


def test_oracle_pooled_calls_pool_the_last_entry():
    """The final-normed tokens are what jimm semantics pools, in every family."""
    oc = O.DualCfg(32, 2, 64, 8, 8, 50, 64, 1, 2)
    img = O.synthetic_images(2, 32, dtype=torch.float64)
    for kind in ("clip", "siglip"):
        p = O.random_dual_params(oc, kind, seed=2, dtype=torch.float64)
        txt = O.synthetic_tokens(2, 8, 50, kind)
        if kind == "clip":
            xs = TO.clip_image_hidden(p, oc, img)
            assert torch.allclose(O.linear(xs[-1][:, 0], p["visual_projection.kernel"]), O.clip_encode_image(p, oc, img), rtol=0, atol=1e-12)
            ts = TO.clip_text_hidden(p, oc, txt)
            f = ts[-1][torch.arange(2), txt.argmax(-1)]
            assert torch.allclose(O.linear(f, p["text_projection.kernel"]), O.clip_encode_text(p, oc, txt), rtol=0, atol=1e-12)
        else:
            xs = TO.siglip_image_hidden(p, oc, img)
            assert torch.allclose(O.map_head(p, "vision_model.MAPHead.", xs[-1], oc.v_heads, 1e-6), O.siglip_encode_image(p, oc, img),
                                  rtol=0, atol=1e-12)
            ts = TO.siglip_text_hidden(p, oc, txt)
            head = O.linear(ts[-1][:, -1], p["text_projection.kernel"], p["text_projection.bias"])
            assert torch.allclose(head, O.siglip_encode_text(p, oc, txt), rtol=0, atol=1e-12)


# ---- argument checks of the per-token calls (no GPU: they must raise before a handle is built) ----
def test_prep_layers_resolves_requests():
    from jimm_b200._lib import LAYER_FINAL
    from jimm_b200._runtime import prep_layers

    r = prep_layers(None, 4, torch.float32)
    assert r.single and r.codes == [LAYER_FINAL] and r.index == [0]
    r = prep_layers(-1, 4, torch.float16)
    assert r.single and r.codes == [4]
    r = prep_layers([-2, 0, None, 4, -1, -5], 4, torch.bfloat16)
    assert not r.single and r.codes == [3, 0, LAYER_FINAL, 4] and r.index == [0, 1, 2, 3, 3, 1]
    assert not prep_layers((1,), 4, torch.float32).single  # a tuple of one request gives a tuple
    for bad in (5, -6, 1.0, True, "1", [], [0, 7]):
        with pytest.raises(ValueError):
            prep_layers(bad, 4, torch.float32)
    for dt in (torch.float64, torch.int32, torch.float8_e4m3fn):
        with pytest.raises(ValueError):
            prep_layers(0, 4, dt)


def test_tokens_result_forms():
    from jimm_b200._runtime import prep_layers, tokens_result

    toks = ["a", "b"]
    assert tokens_result(toks, prep_layers(1, 3, torch.float32)._replace(codes=[1], index=[1]), None, False) == "b"
    assert tokens_result(toks, prep_layers([1, 2, 1], 3, torch.float32), "p", True) == (("a", "b", "a"), "p")


def test_model_methods_check_before_any_handle():
    from jimm_b200.models import CLIP, SigLIP, VisionTransformer
    from jimm_b200.common.vit import VisionTransformerBase

    vit = VisionTransformer(num_classes=4, img_size=32, patch_size=8, num_layers=2, num_heads=2, mlp_dim=64, hidden_size=64)
    img = torch.zeros(1, 32, 32, 3)
    for kw in (dict(layers=3), dict(layers=-4), dict(layers=[0, 9]), dict(dtype=torch.float64), dict(layers="x")):
        with pytest.raises(ValueError):
            vit.forward_tokens(img, **kw)
    with pytest.raises(ValueError):
        vit.forward_tokens(torch.zeros(1, 16, 16, 3))  # the existing input error: not the trained size
    tower = VisionTransformerBase(32, 8, 3, 64, 2, 2, 64)
    with pytest.raises(ValueError):
        tower.forward_tokens(img, layers=3)
    clip = CLIP(32, 2, 64, 8, 8, 50, 64, 1, 2)
    with pytest.raises(ValueError):
        clip.encode_image_tokens(img, layers=-4)
    with pytest.raises(ValueError):
        clip.encode_text_tokens(torch.zeros(2, 8, dtype=torch.long), layers=3)
    with pytest.raises(ValueError):
        clip.encode_text_tokens(torch.zeros(2, 9, dtype=torch.long))  # longer than context_length
    with pytest.raises(ValueError):
        clip.encode_text_tokens(torch.zeros(8, dtype=torch.long))  # not [B, T]
    with pytest.raises(ValueError):
        clip.encode_text_tokens([torch.zeros(9, dtype=torch.long)])
    sig = SigLIP(32, 2, 64, 8, 8, 50, 64, 1, 2)
    with pytest.raises(ValueError):
        sig.encode_image_tokens(img, spatial_shapes=torch.tensor([[4, 4]]))  # NaFlex inputs on a SigLIP model
    with pytest.raises(ValueError):
        sig.encode_text_tokens(torch.zeros(1, 8, dtype=torch.long), dtype=torch.int8)
    for m in (vit, tower, clip, sig):
        assert m._native is None
