"""Pin the oracle against HuggingFace transformers (offline mirror of the reference's own tests).

TEST INFRASTRUCTURE ONLY (see oracle/jimm_oracle.py header).

The reference's tests (tests/test_vit.py, tests/test_clip.py, tests/test_siglip.py)
compare jimm against HF PyTorch models on downloaded weights.  There is no
network here, so the same comparison runs on random-init HF models built from
configs, with zero/one-initialised parameters perturbed so every bias / LN /
cls / probe path is exercised.  Two checks per model:

  hf   semantics (erf-GELU where HF uses it, HF eps everywhere)  -> must agree <= 1e-5:
       proves the layout transforms, head split, patch order, pooling, masks.
  jimm semantics (tanh-GELU, block eps 1e-6)                      -> must meet the
       reference's own tolerance (0.05 / 1e-1 / 1e-2).

Run:  python oracle/check_vs_hf.py [--full]
"""

from __future__ import annotations

import os
import sys

os.environ.setdefault("HF_HUB_OFFLINE", "1")
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jimm_oracle as O  # noqa: E402


def perturb_(model, seed=7):
    """Make zero/one-initialised params non-trivial (biases, LN, cls token, probe, logit scale/bias)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.ndim <= 1 or "cls_token" in name or "class_embedding" in name or "probe" in name or "position_embedding" in name:
                if "logit_scale" in name or "logit_bias" in name:
                    continue
                scale = 0.1 if ("norm" in name.lower() or "layrnorm" in name) else 0.05
                p.add_(torch.randn(p.shape, generator=g) * scale)
    return model


def tiny_vit_config(**kw):
    from transformers import ViTConfig

    base = dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256, image_size=32,
                patch_size=8, num_labels=10, hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    base.update(kw)
    return ViTConfig(**base)


def tiny_clip_config():
    from transformers import CLIPConfig

    return CLIPConfig(
        text_config=dict(hidden_size=128, num_attention_heads=2, num_hidden_layers=2, intermediate_size=512,
                         max_position_embeddings=16, vocab_size=100, eos_token_id=99, bos_token_id=98, pad_token_id=1,
                         projection_dim=128),
        vision_config=dict(hidden_size=128, num_attention_heads=2, num_hidden_layers=2, intermediate_size=512,
                           image_size=32, patch_size=8, projection_dim=128),
        projection_dim=128,
    )


def tiny_siglip_config():
    from transformers import SiglipConfig

    return SiglipConfig(
        text_config=dict(hidden_size=128, num_attention_heads=2, num_hidden_layers=2, intermediate_size=512,
                         max_position_embeddings=16, vocab_size=100, projection_size=128),
        vision_config=dict(hidden_size=128, num_attention_heads=2, num_hidden_layers=2, intermediate_size=512,
                           image_size=32, patch_size=8),
    )


# HF checkpoint families at their real tower widths: model class, vision (width, heads, MLP width, hidden_act, patch) and text (width,
# heads, MLP width, hidden_act).  family_config builds one at a small depth and image size.
FAMILIES = {
    "openai-clip-b32": ("clip", (768, 12, 3072, "quick_gelu", 32), (512, 8, 2048, "quick_gelu")),
    "openclip-vit-h14": ("clip", (1280, 16, 5120, "gelu", 14), (1024, 16, 4096, "gelu")),
    "openclip-vit-g14": ("clip", (1408, 16, 6144, "gelu", 14), (1024, 16, 4096, "gelu")),
    "siglip-base": ("siglip", (768, 12, 3072, "gelu_pytorch_tanh", 16), (768, 12, 3072, "gelu_pytorch_tanh")),
    "siglip-so400m": ("siglip", (1152, 16, 4304, "gelu_pytorch_tanh", 14), (1152, 16, 4304, "gelu_pytorch_tanh")),
    "siglip2-giant-opt": ("siglip", (1536, 16, 6144, "gelu_pytorch_tanh", 16), (1152, 16, 4304, "gelu_pytorch_tanh")),
    "siglip2-so400m-naflex": ("siglip2", (1152, 16, 4304, "gelu_pytorch_tanh", 16), (1152, 16, 4304, "gelu_pytorch_tanh")),
}


def family_config(name, vision_layers=2, text_layers=2, grid=4, context_length=16, vocab_size=100):
    """The HF config of FAMILIES[name] with `grid` x `grid` patches per image (NaFlex: a 16 x 16 position table)."""
    from transformers import CLIPConfig, Siglip2Config, SiglipConfig

    kind, (vw, vh, vm, va, P), (tw, th, tm, ta) = FAMILIES[name]
    v = dict(hidden_size=vw, num_attention_heads=vh, intermediate_size=vm, hidden_act=va, num_hidden_layers=vision_layers, patch_size=P)
    t = dict(hidden_size=tw, num_attention_heads=th, intermediate_size=tm, hidden_act=ta, num_hidden_layers=text_layers,
             max_position_embeddings=context_length, vocab_size=vocab_size)
    if kind == "clip":
        return CLIPConfig(text_config=dict(t, eos_token_id=vocab_size - 1, bos_token_id=vocab_size - 2, pad_token_id=1),
                          vision_config=dict(v, image_size=grid * P), projection_dim=tw)
    t["projection_size"] = vw  # SigLIP's text head projects to the vision width (1152 -> 1536 in giant-opt)
    if kind == "siglip":
        return SiglipConfig(text_config=t, vision_config=dict(v, image_size=grid * P))
    return Siglip2Config(text_config=t, vision_config=dict(v, num_patches=256))  # the 16 x 16 table of the NaFlex checkpoints


def hf_semantics(cfg) -> O.Semantics:
    """The oracle in HF semantics: erf GELU on the towers whose hidden_act is "gelu", HF's LayerNorm eps in the blocks."""
    acts = {cfg.vision_config.hidden_act, cfg.text_config.hidden_act} - {"quick_gelu"}
    assert len(acts) <= 1, f"one GELU form for both towers, got {acts}"
    return O.Semantics(gelu="erf" if acts == {"gelu"} else "tanh", block_eps=cfg.vision_config.layer_norm_eps)


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def check_vit(cfg=None, B=2, dtype=torch.float64, seed=0):
    from transformers import ViTForImageClassification

    torch.manual_seed(seed)
    cfg = cfg or tiny_vit_config()
    m = perturb_(ViTForImageClassification(cfg)).eval().to(dtype)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    oc = O.ViTCfg(num_classes=cfg.num_labels, img_size=cfg.image_size, patch_size=cfg.patch_size, num_layers=cfg.num_hidden_layers,
                  num_heads=cfg.num_attention_heads, mlp_dim=cfg.intermediate_size, hidden_size=cfg.hidden_size)
    p = O.hf_to_flax_vit(sd, oc.num_layers, oc.num_heads)
    img = O.synthetic_images(B, cfg.image_size, dtype=dtype)
    with torch.no_grad():
        ref = m(pixel_values=img.permute(0, 3, 1, 2)).logits
        hf_sem = O.Semantics(gelu="erf" if cfg.hidden_act == "gelu" else "tanh", block_eps=cfg.layer_norm_eps)
        out_hf = O.vit_forward(p, oc, img, hf_sem)
        out_jimm = O.vit_forward(p, oc, img)
    return dict(hf_abs=float((out_hf - ref).abs().max()), hf_rel=rel(out_hf, ref),
                jimm_abs=float((out_jimm - ref).abs().max()), jimm_rel=rel(out_jimm, ref),
                argmax_equal=bool((out_jimm.argmax(-1) == ref.argmax(-1)).all()))


def _dual_cfg(cfg) -> O.DualCfg:
    t, v = cfg.text_config, cfg.vision_config
    return O.DualCfg(image_resolution=v.image_size, vision_layers=v.num_hidden_layers, vision_width=v.hidden_size,
                     vision_patch_size=v.patch_size, context_length=t.max_position_embeddings, vocab_size=t.vocab_size,
                     transformer_width=t.hidden_size, transformer_heads=t.num_attention_heads,
                     transformer_layers=t.num_hidden_layers, **arch_fields(cfg))


def arch_fields(cfg) -> dict:
    """The DualCfg fields a HF config declares beyond the reference's rule: heads, MLP widths (the MAP head's is the vision tower's,
    as in HF's SigLIP) and each tower's activation."""
    t, v = cfg.text_config, cfg.vision_config
    return dict(vision_heads=v.num_attention_heads, vision_mlp=v.intermediate_size, text_mlp=t.intermediate_size,
                map_mlp=v.intermediate_size, vision_quick_gelu=v.hidden_act == "quick_gelu", text_quick_gelu=t.hidden_act == "quick_gelu")


def check_clip(cfg=None, B=3, dtype=torch.float64, seed=0):
    from transformers import CLIPModel

    torch.manual_seed(seed)
    cfg = cfg or tiny_clip_config()
    m = perturb_(CLIPModel(cfg)).eval().to(dtype)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    oc = _dual_cfg(cfg)
    p = O.hf_to_flax_clip(sd, oc)
    img = O.synthetic_images(B, oc.image_resolution, dtype=dtype)
    txt = O.synthetic_tokens(B + 1, oc.context_length, oc.vocab_size, "clip")
    sem = hf_semantics(cfg)
    with torch.no_grad():
        ref = m(pixel_values=img.permute(0, 3, 1, 2), input_ids=txt).logits_per_image
        ref_i, ref_t = m.get_image_features(pixel_values=img.permute(0, 3, 1, 2)).pooler_output, m.get_text_features(input_ids=txt).pooler_output
        out_hf = O.clip_forward(p, oc, img, txt, sem)
        ie, te = O.clip_encode_image(p, oc, img, sem), O.clip_encode_text(p, oc, txt, sem)
        out_jimm = O.clip_forward(p, oc, img, txt)
    return dict(hf_abs=float((out_hf - ref).abs().max()), hf_rel=rel(out_hf, ref), img_rel=rel(ie, ref_i), txt_rel=rel(te, ref_t),
                jimm_abs=float((out_jimm - ref).abs().max()), jimm_rel=rel(out_jimm, ref))


def check_siglip(cfg=None, B=3, dtype=torch.float64, seed=0):
    from transformers import SiglipModel

    torch.manual_seed(seed)
    cfg = cfg or tiny_siglip_config()
    m = perturb_(SiglipModel(cfg)).eval().to(dtype)
    with torch.no_grad():
        m.logit_scale.fill_(2.3)
        m.logit_bias.fill_(-1.7)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    oc = _dual_cfg(cfg)
    p = O.hf_to_flax_siglip(sd, oc)
    img = O.synthetic_images(B, oc.image_resolution, dtype=dtype)
    txt = O.synthetic_tokens(B + 1, oc.context_length, oc.vocab_size, "siglip")
    with torch.no_grad():
        out = m(pixel_values=img.permute(0, 3, 1, 2), input_ids=txt)
        sem = hf_semantics(cfg)
        ie, te, lg = O.siglip_encode_image(p, oc, img, sem), O.siglip_encode_text(p, oc, txt, sem), O.siglip_forward(p, oc, img, txt, sem)
        # HF returns the un-normalised pooled outputs from the sub-models; image_embeds/text_embeds are normalised
        ref_i = m.vision_model(pixel_values=img.permute(0, 3, 1, 2)).pooler_output
        ref_t = m.text_model(input_ids=txt).pooler_output
    return dict(img_rel=rel(ie, ref_i), txt_rel=rel(te, ref_t), logits_abs=float((lg - out.logits_per_image).abs().max()),
                logits_rel=rel(lg, out.logits_per_image))


def main():
    full = "--full" in sys.argv
    print("tiny ViT   ", check_vit())
    print("tiny CLIP  ", check_clip())
    print("tiny SigLIP", check_siglip())
    if full:
        from transformers import CLIPConfig, SiglipConfig, ViTConfig

        print("ViT-B/16   ", check_vit(ViTConfig(num_labels=1000), B=2, dtype=torch.float32))
        print("CLIP-B/32  ", check_clip(CLIPConfig(), B=2, dtype=torch.float32))
        print("SigLIP-B/16", check_siglip(SiglipConfig(), B=2, dtype=torch.float32))


if __name__ == "__main__":
    main()
