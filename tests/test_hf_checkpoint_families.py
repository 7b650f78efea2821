"""HF checkpoints of each CLIP / SigLIP family at their real tower widths: from_pretrained must build the architecture the checkpoint
declares (heads, MLP widths, the MAP head's MLP width and each tower's activation), not the reference's rule of width // 64 heads,
MLPs 4x the width and one activation per class.  The families (check_vs_hf.FAMILIES) are random-init HF models at the real widths with
2 + 2 layers and 4 x 4 patch grids, perturbed and written with save_pretrained:

  openai-clip-b32 (control)   vision 768 / 12 heads / MLP 3072 / quick_gelu    text 512 / 8 / 2048 / quick_gelu
  openclip-vit-h14            vision 1280 / 16 (d 80) / 5120 / gelu            text 1024 / 16 / 4096 / gelu
  openclip-vit-g14            vision 1408 / 16 (d 88) / 6144 / gelu            text 1024 / 16 / 4096 / gelu
  siglip-base (control)       vision 768 / 12 / 3072                            text 768 / 12 / 3072
  siglip-so400m               vision 1152 / 16 (d 72) / 4304, MAP MLP 4304     text 1152 / 16 / 4304
  siglip2-giant-opt           vision 1536 / 16 (d 96) / 6144                    text 1152 / 16 / 4304, head 1152 -> 1536
  siglip2-so400m-naflex       Siglip2Model, vision as so400m at patch 16 with a 16 x 16 position table, text as so400m

- CPU: the native config read back from from_pretrained; the oracle against HF's fp64 forward in HF semantics; the old rule moves the
  oracle's output far past the GPU bounds.  giant-opt's text head projects to the vision width, which the native text tower (its
  projection as wide as the tower) does not run: from_pretrained refuses it, and only the oracle tests take it.
- GPU: from_pretrained against the fp64 oracle in every compute dtype; a coarse bound against HF itself, which a wrong activation mapping
  breaks; the control families bit for bit against the constructor; NaFlex on Siglip2ImageProcessor's output; so400m at full depth."""

import dataclasses

import numpy as np
import pytest
import torch

import check_vs_hf as H
import jimm_oracle as O
import naflex_oracle as N
from gpu_util import check_parity, record_parity

FAMILIES = list(H.FAMILIES)
CHANGED = ["openclip-vit-h14", "openclip-vit-g14", "siglip-so400m", "siglip2-giant-opt"]  # where the reference's rule is wrong
CONTROLS = ["openai-clip-b32", "siglip-base"]
UNLOADABLE = ["siglip2-giant-opt"]

TOL = 1e-3          # the model parity bars of test_parity_gpu.py
LOGITS_TOL = 2e-3
BF16_VS_SAME = 8e-3
# The project runs the tanh GELU where HF's "gelu" is erf, and CLIP's blocks use the reference's LayerNorm eps 1e-6 where HF uses 1e-5.
# The oracle in project semantics against HF's fp64 forward, measured on the CPU (test_project_semantics_gap_to_hf): image / text embeds
# 2.9e-6 / 7.7e-4 (openai-clip-b32, eps only), 1.0e-4 / 8.0e-4 (openclip-vit-h14), 1.1e-4 / 9.6e-4 (openclip-vit-g14), below 1e-14 for
# the SigLIP families.  A GPU embedding must stay within HF_BOUND, about 3x the largest gap, of HF's; QuickGELU in place of the tanh
# GELU moves the h14 / g14 oracle embeddings by 4.9e-3 - 1.3e-2.
HF_GAP = 9.6e-4
HF_BOUND = 3e-3
# The old rule moves the oracle's image embeds by 3.1e-2 (g14) to 2.0e-1 (giant-opt), at least 20x the GPU bound.  Its text embeds
# move by 1.2e-2 (g14) to 4.1e-1 (giant-opt): the CLIP text towers already took their heads from the config, so only the activation
# moves them there, by 12x the GPU bound.
MOVE_IMAGE = 20 * TOL
MOVE_TEXT = 10 * TOL

NAFLEX_SIZES = [(120, 360), (200, 200), (300, 150)]  # (height, width): wide, square and tall


def _kind(name):
    return H.FAMILIES[name][0]


class Family:
    """One family's checkpoint on disk, its fp64 HF model and the oracle's config and parameters."""

    def __init__(self, name, root, seed=0):
        from transformers import CLIPModel, Siglip2Model, SiglipModel

        self.name, self.kind = name, _kind(name)
        self.cfg = H.family_config(name)
        torch.manual_seed(seed)
        cls = {"clip": CLIPModel, "siglip": SiglipModel, "siglip2": Siglip2Model}[self.kind]
        m = H.perturb_(cls(self.cfg)).eval()
        if self.kind != "clip":
            with torch.no_grad():
                m.logit_scale.fill_(2.3)
                m.logit_bias.fill_(-1.7)
        m.save_pretrained(str(root), safe_serialization=True)
        self.path = str(root / "model.safetensors")
        sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
        self.hf = m.to(torch.float64)
        if self.kind == "siglip2":
            self.oc = N.dual_cfg(self.cfg)
            self.params = N.hf_to_flax_siglip2(sd, self.oc)
        else:
            self.oc = H._dual_cfg(self.cfg)
            self.params = (O.hf_to_flax_clip if self.kind == "clip" else O.hf_to_flax_siglip)(sd, self.oc)
        oc = self.oc
        if self.kind == "siglip2":
            P = oc.vision_patch_size
            g = torch.Generator().manual_seed(11)
            imgs = [torch.rand((h // P * P, w // P * P, 3), generator=g) * 2 - 1 for h, w in ((64, 96), (80, 48))]
            self.images = N.pad_batch(imgs, P, (oc.image_resolution // P) ** 2)[:2]  # (pixel_values, spatial_shapes)
        else:
            self.images = O.synthetic_images(2, oc.image_resolution, seed=12)
        self.tokens = O.synthetic_tokens(3, oc.context_length, oc.vocab_size, "clip" if self.kind == "clip" else "siglip", seed=13)

    def load(self, dtype=torch.float32):
        from jimm_b200.models import CLIP, SigLIP

        return (CLIP if self.kind == "clip" else SigLIP).from_pretrained(self.path, dtype=dtype)

    def oracle(self, sem=O.JIMM, params=None, oc=None):
        """(image embeds, text embeds, logits) of the oracle in fp64."""
        p = O.cast_params(params or self.params, torch.float64)
        oc = oc or self.oc
        with torch.no_grad():
            if self.kind == "clip":
                img = self.images.double()
                ie, te = O.clip_encode_image(p, oc, img, sem), O.clip_encode_text(p, oc, self.tokens, sem)
                return ie, te, O.contrastive_logits(ie, te, p["logit_scale"], None, sem)
            if self.kind == "siglip":
                ie = O.siglip_encode_image(p, oc, self.images.double(), sem)
            else:
                pv, shapes = self.images
                ie = N.encode_patches(p, oc, pv.double(), shapes, sem)
            te = O.siglip_encode_text(p, oc, self.tokens, sem)
            return ie, te, O.contrastive_logits(ie, te, p["logit_scale"], p["logit_bias"], sem)

    def reference(self):
        """(image embeds, text embeds, logits) of the HF model in fp64."""
        with torch.no_grad():
            if self.kind == "siglip2":
                pv, shapes = self.images
                mask = (torch.arange(pv.shape[1])[None] < shapes.prod(-1)[:, None]).to(torch.int32)
                kw = dict(pixel_values=pv.double(), spatial_shapes=shapes, pixel_attention_mask=mask)
            else:
                kw = dict(pixel_values=self.images.double().permute(0, 3, 1, 2))
            ie = self.hf.get_image_features(**kw).pooler_output
            te = self.hf.get_text_features(input_ids=self.tokens).pooler_output
            return ie, te, self.hf(input_ids=self.tokens, **kw).logits_per_image

    def run(self, model):
        """(image embeds, text embeds, logits) of a jimm_b200 model on the GPU."""
        txt = self.tokens.cuda()
        if self.kind == "siglip2":
            pv, shapes = self.images
            img, kw = pv.cuda(), dict(spatial_shapes=shapes)
        else:
            img, kw = self.images.cuda(), {}
        return model.encode_image(img, **kw), model.encode_text(txt), model(img, txt, **kw)


@pytest.fixture(scope="module", params=FAMILIES)
def family(request, tmp_path_factory):
    return Family(request.param, tmp_path_factory.mktemp(request.param))


def _named(request_family, names):
    if request_family.name not in names:
        pytest.skip(f"{request_family.name} is not one of {names}")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_from_pretrained_builds_the_declared_architecture(family):
    """(a) Heads, MLP widths, the MAP head's MLP width and each tower's activation as the checkpoint's config.json declares them."""
    from jimm_b200 import _lib

    if family.name in UNLOADABLE:
        with pytest.raises(ValueError, match="text_projection"):
            family.load()
        return
    m = family.load()
    cfg = m._native_config()
    v, t = family.cfg.vision_config, family.cfg.text_config
    act = lambda a: _lib.ACT_QUICK_GELU if a == "quick_gelu" else _lib.ACT_GELU_TANH
    got = dict(v_heads=cfg.v_heads, v_mlp=cfg.v_mlp, v_act=cfg.v_act, t_heads=cfg.t_heads, t_mlp=cfg.t_mlp, t_act=cfg.t_act)
    want = dict(v_heads=v.num_attention_heads, v_mlp=v.intermediate_size, v_act=act(v.hidden_act), t_heads=t.num_attention_heads,
                t_mlp=t.intermediate_size, t_act=act(t.hidden_act))
    assert got == want
    if family.kind != "clip":
        assert tuple(m.flat_param_shapes()["vision_model.MAPHead.mlp.layers.0.kernel"]) == (v.hidden_size, v.intermediate_size)
    flat = m.flat_params()
    assert set(flat) == set(family.params), set(flat) ^ set(family.params)
    for k, ref in family.params.items():
        assert tuple(flat[k].shape) == tuple(ref.shape), k
        assert torch.equal(flat[k], ref.float()), k


def test_oracle_matches_hf_fp64(family):
    """(b) In HF semantics (erf GELU where HF declares "gelu", HF's LayerNorm eps) the oracle is HF's forward."""
    out = family.oracle(H.hf_semantics(family.cfg))
    for what, a, r in zip(("image_embeds", "text_embeds", "logits"), out, family.reference()):
        assert H.rel(a, r) < 1e-5, (family.name, what, H.rel(a, r))


def test_project_semantics_gap_to_hf(family):
    """The gap HF_BOUND rests on: the oracle in project semantics (tanh GELU, the reference's eps) against HF's fp64 forward."""
    for what, a, r in zip(("image_embeds", "text_embeds"), family.oracle(), family.reference()):
        gap = H.rel(a, r)
        record_parity(f"{family.name} oracle (project semantics)", what, "float64", "HF fp64", None, gap)
        assert gap < 1.05 * HF_GAP, (family.name, what, gap)


def test_old_rule_moves_the_oracle(family):
    """(c) Heads width // 64 on the vision tower (and on SigLIP's text tower) and CLIP's QuickGELU on both towers, the rule the loaders
    used to apply, move the embeddings far past the GPU bound (MOVE_IMAGE, MOVE_TEXT).  The MLP widths stay the checkpoint's: the oracle
    reads them from the weights."""
    _named(family, CHANGED)
    oc = family.oc
    old = dict(vision_heads=None, vision_quick_gelu=None, text_quick_gelu=None)
    if family.kind != "clip":
        old["transformer_heads"] = oc.transformer_width // 64
    oc_old = dataclasses.replace(oc, **old)
    sd = {k: v.detach() for k, v in family.hf.state_dict().items()}
    p_old = (O.hf_to_flax_clip if family.kind == "clip" else O.hf_to_flax_siglip)(sd, oc_old)
    for what, a, r in zip(("image_embeds", "text_embeds", "logits"), family.oracle(params=p_old, oc=oc_old), family.oracle()):
        moved = H.rel(a, r)
        record_parity(f"{family.name} old rule", what, "float64", "oracle", None, moved)
        if what != "logits":
            assert moved > (MOVE_IMAGE if what == "image_embeds" else MOVE_TEXT), (family.name, what, moved)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_from_pretrained_against_oracle(family):
    """(d) fp32 (tf32 operands) and fp16 within the project's bars of the fp64 oracle in project semantics, bf16 of the same-rounding
    oracle; FP8 reported.  (e) fp32 embeddings within HF_BOUND of HF's own fp64 forward."""
    _named(family, [n for n in FAMILIES if n not in UNLOADABLE])
    ref = family.oracle()
    same_bf16 = family.oracle(O.Semantics(operand_round="bf16"))
    hf = family.reference()
    names = ("image_embeds", "text_embeds", "logits")
    for dtype in (torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn):
        out = family.run(family.load(dtype))
        case = f"from_pretrained {family.name}"
        for what, a, r, s, h in zip(names, out, ref, same_bf16, hf):
            bound = LOGITS_TOL if what == "logits" else TOL
            if dtype == torch.bfloat16:
                check_parity(case, what, dtype, "same-rounding", a, s, BF16_VS_SAME)
            elif dtype == torch.float8_e4m3fn:
                check_parity(case, what, dtype, "fp64 oracle", a, r, None)
            else:
                check_parity(case, what, dtype, "fp64 oracle", a, r, bound)
            if dtype == torch.float32 and what != "logits":
                check_parity(case, what, dtype, "HF fp64", a, h, HF_BOUND)


@pytest.mark.gpu
def test_controls_match_the_constructor(family):
    """(f) For checkpoints the reference's rule fits, from_pretrained gives the bits of the constructor with the reference's defaults
    and the same parameters."""
    _named(family, CONTROLS)
    from jimm_b200.models import CLIP, SigLIP

    oc = family.oc
    for dtype in (torch.float32, torch.float16):
        ctor = (CLIP if family.kind == "clip" else SigLIP)(
            image_resolution=oc.image_resolution, vision_layers=oc.vision_layers, vision_width=oc.vision_width,
            vision_patch_size=oc.vision_patch_size, context_length=oc.context_length, vocab_size=oc.vocab_size,
            transformer_width=oc.transformer_width, transformer_heads=oc.transformer_heads, transformer_layers=oc.transformer_layers,
            dtype=dtype)
        for k, v in family.params.items():
            ctor.set_flat_param(k, v.float())
        for what, a, b in zip(("image_embeds", "text_embeds", "logits"), family.run(family.load(dtype)), family.run(ctor)):
            assert torch.equal(a, b), (family.name, dtype, what)


@pytest.mark.gpu
def test_naflex_so400m_on_processor_output(family):
    """(g) The so400m NaFlex family on Siglip2ImageProcessor(patch_size=16, max_num_patches=256)'s output for three images of different
    aspect ratios, against HF Siglip2Model in fp64."""
    _named(family, ["siglip2-so400m-naflex"])
    from transformers import Siglip2ImageProcessor

    g = np.random.default_rng(14)
    imgs = [g.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in NAFLEX_SIZES]
    enc = Siglip2ImageProcessor(patch_size=16, max_num_patches=256)(images=imgs, return_tensors="pt")
    pv, shapes, mask = enc["pixel_values"], enc["spatial_shapes"], enc["pixel_attention_mask"]
    assert len({tuple(s) for s in shapes.tolist()}) == 3
    txt = family.tokens
    with torch.no_grad():
        kw = dict(pixel_values=pv.double(), spatial_shapes=shapes, pixel_attention_mask=mask)
        ref = (family.hf.get_image_features(**kw).pooler_output, family.hf.get_text_features(input_ids=txt).pooler_output,
               family.hf(input_ids=txt, **kw).logits_per_image)
    for dtype in (torch.float32, torch.float16):
        m = family.load(dtype)
        out = (m.encode_image(pv.cuda(), spatial_shapes=shapes, pixel_attention_mask=mask.cuda()), m.encode_text(txt.cuda()),
               m(pv.cuda(), txt.cuda(), spatial_shapes=shapes, pixel_attention_mask=mask.cuda()))
        for what, a, r in zip(("image_embeds", "text_embeds", "logits"), out, ref):
            check_parity("so400m NaFlex on Siglip2ImageProcessor output", what, dtype, "HF Siglip2Model fp64", a, r,
                         LOGITS_TOL if what == "logits" else TOL)


@pytest.mark.gpu
def test_siglip_so400m_full_depth():
    """(h) so400m at its HF architecture and full 27 + 27 layers (16 heads of 72 and MLPs 4304 wide on both towers, MAP MLP 4304), fp16,
    two images and two texts, against the fp64 oracle."""
    from jimm_b200.models import SigLIP

    oc = O.DualCfg(224, 27, 1152, 14, 64, 32000, 1152, 16, 27, vision_heads=16, vision_mlp=4304, text_mlp=4304, map_mlp=4304)
    p = O.random_dual_params(oc, "siglip", seed=103)
    p64 = O.cast_params(p, torch.float64)
    img, txt = O.synthetic_images(2, 224, seed=15), O.synthetic_tokens(2, 64, 32000, "siglip", seed=16)
    with torch.no_grad():
        ref_i, ref_t = O.siglip_encode_image(p64, oc, img.double()), O.siglip_encode_text(p64, oc, txt)
        ref = O.contrastive_logits(ref_i, ref_t, p64["logit_scale"], p64["logit_bias"])
    m = SigLIP(image_resolution=224, vision_layers=27, vision_width=1152, vision_patch_size=14, context_length=64, vocab_size=32000,
               transformer_width=1152, transformer_heads=16, transformer_layers=27, dtype=torch.float16, vision_heads=16,
               vision_mlp_dim=4304, text_mlp_dim=4304)
    for k, v in p.items():
        m.set_flat_param(k, v)
    case = "SigLIP so400m HF architecture, 27+27 layers"
    check_parity(case, "image_embeds", torch.float16, "fp64", m.encode_image(img.cuda()), ref_i, TOL)
    check_parity(case, "text_embeds", torch.float16, "fp64", m.encode_text(txt.cuda()), ref_t, TOL)
    check_parity(case, "logits", torch.float16, "fp64", m(img.cuda(), txt.cuda()), ref, LOGITS_TOL)
