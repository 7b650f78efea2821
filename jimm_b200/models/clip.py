"""Mirror of jimm.models.clip (reference: src/jimm/models/clip.py)."""

from __future__ import annotations

from typing import Optional

import torch

from .. import _lib, nn
from ..common.transformer import g_wrap
from ..common import hf_loader as L
from ..common.utils import load_params_and_config
from ..common.vit import VisionTransformerBase, tower_config_fields
from ._dual import DualTower, build_text_tower


class CLIP(DualTower):
    """models/clip.py:15-188.

    vision_heads, vision_mlp_dim, text_mlp_dim, vision_quick_gelu, text_quick_gelu: the architecture of checkpoints that depart from the
    reference's rule (vision_width // 64 heads, MLPs 4x the width, QuickGELU on both towers), such as OpenCLIP's ViT-H/14 (16 heads of
    80, tanh GELU where HF declares hidden_act "gelu").  None / the defaults are the reference's values."""

    def __init__(self, image_resolution: int, vision_layers: int, vision_width: int, vision_patch_size: int, context_length: int,
                 vocab_size: int, transformer_width: int, transformer_heads: int, transformer_layers: int, rngs=None,
                 dtype=torch.float32, param_dtype=torch.float32, mesh=None, vision_heads: Optional[int] = None,
                 vision_mlp_dim: Optional[int] = None, text_mlp_dim: Optional[int] = None, vision_quick_gelu: bool = True,
                 text_quick_gelu: bool = True):
        self._init_common(image_resolution, vision_layers, vision_width, vision_patch_size, context_length, vocab_size,
                          transformer_width, transformer_heads, transformer_layers, dtype, vision_heads=vision_heads,
                          vision_mlp_dim=vision_mlp_dim, text_mlp_dim=text_mlp_dim, vision_quick_gelu=vision_quick_gelu,
                          text_quick_gelu=text_quick_gelu)
        g = nn._gen(rngs)
        object.__setattr__(self, "attn_mask", torch.tril(torch.ones(context_length, context_length)))  # :62
        # models/clip.py:64-81: pre-norm, no patch bias, QuickGELU, CLS, eps 1e-5
        self.add_child("vision_model", VisionTransformerBase(
            img_size=image_resolution, patch_size=vision_patch_size, in_channels=3, hidden_size=vision_width,
            num_layers=vision_layers, num_heads=self.vision_heads, mlp_dim=self.vision_mlp_dim, use_pre_norm=True, use_patch_bias=False,
            use_quick_gelu=self.vision_quick_gelu, pooling_type="CLS", layernorm_epsilon=1e-5, dtype=dtype, rngs=g_wrap(g)))
        self.add_child("visual_projection", nn.Linear(vision_width, transformer_width, use_bias=False, rngs=g_wrap(g)))
        build_text_tower(self, g, head_bias=False, layernorm_epsilon=1e-6, attn_mask=self.attn_mask)
        self.add_param("logit_scale", nn.ones(()))

    def _native_config(self) -> _lib.Config:
        cfg = _lib.Config()
        cfg.kind = _lib.KIND_CLIP
        tower_config_fields(cfg, **self.vision_model._hp)
        cfg.num_classes = 0
        # text: causal tril mask (:62,:98), QuickGELU (:99), ln_final eps 1e-5 (:117), EOT = argmax(ids) pooling (:164), bias-free projection (:166)
        return self._text_config(cfg, causal=1, pool=_lib.TPOOL_EOT_ARGMAX, head_bias=0, eps_outer=1e-5)

    @classmethod
    def from_pretrained(cls, model_name_or_path: str, use_pytorch: bool = False, mesh=None, dtype=torch.float32) -> "CLIP":
        """Load a HF `CLIPModel` checkpoint (models/clip.py:190-416).  Heads, MLP widths and hidden_act of each tower come from
        config.json's vision_config / text_config (hf_loader.tower_arch); without a config.json, heads are width // 64, the MLP widths
        those of the fc1 weights and both towers QuickGELU."""
        hf, config = load_params_and_config(model_name_or_path, use_pytorch)
        if config == {}:
            if use_pytorch:
                raise ValueError(f"Configuration could not be loaded for PyTorch model {model_name_or_path}")
            # no config.json: the architecture from the tensor shapes (models/clip.py:213-252); head width 64 on both towers

            def depth(tower):
                return max((int(k.split(".")[3]) + 1 for k in hf if k.startswith(f"{tower}.encoder.layers.") and k.endswith(".self_attn.q_proj.weight")),
                           default=0)

            tok = hf["text_model.embeddings.token_embedding.weight"]
            vw = hf["vision_model.embeddings.class_embedding"].shape[0]
            vp = hf["vision_model.embeddings.patch_embedding.weight"].shape[2]
            grid = int((hf["vision_model.embeddings.position_embedding.weight"].shape[0] - 1) ** 0.5)
            config = {
                "text_config": {"hidden_size": tok.shape[1], "num_attention_heads": tok.shape[1] // 64, "num_hidden_layers": depth("text_model"),
                                "max_position_embeddings": hf["text_model.embeddings.position_embedding.weight"].shape[0], "vocab_size": tok.shape[0]},
                "vision_config": {"hidden_size": vw, "num_attention_heads": vw // 64, "num_hidden_layers": depth("vision_model"),
                                  "image_size": grid * vp, "patch_size": vp},
            }
        tc, vc = config["text_config"], config["vision_config"]
        v_heads, v_mlp, v_quick = L.tower_arch(vc, "vision_config", vc["hidden_size"], hf, "vision_model", "quick_gelu")
        t_heads, t_mlp, t_quick = L.tower_arch(tc, "text_config", tc["hidden_size"], hf, "text_model", "quick_gelu")
        with nn.deferred_init():  # every parameter is replaced below (and asserted to be)
            model = cls(image_resolution=vc["image_size"], vision_layers=vc["num_hidden_layers"], vision_width=vc["hidden_size"],
                        vision_patch_size=vc["patch_size"], context_length=tc["max_position_embeddings"], vocab_size=tc["vocab_size"],
                        transformer_width=tc["hidden_size"], transformer_heads=t_heads, transformer_layers=tc["num_hidden_layers"],
                        mesh=mesh, dtype=dtype, param_dtype=dtype, vision_heads=v_heads, vision_mlp_dim=v_mlp, text_mlp_dim=t_mlp,
                        vision_quick_gelu=v_quick, text_quick_gelu=t_quick)
        v = "vision_model."
        rules = [
            ("logit_scale", "logit_scale", L.ASIS),
            ("positional_embedding", "text_model.embeddings.position_embedding.weight", L.ASIS),
            ("token_embedding.embedding", "text_model.embeddings.token_embedding.weight", L.ASIS),
            ("ln_final.scale", "text_model.final_layer_norm.weight", L.ASIS),
            ("ln_final.bias", "text_model.final_layer_norm.bias", L.ASIS),
            ("text_projection.kernel", "text_projection.weight", L.LINEAR),
            (v + "cls_token", v + "embeddings.class_embedding", L.ASIS),               # (D) -> (1,1,D)      models/clip.py:358-359
            (v + "position_embeddings", v + "embeddings.position_embedding.weight", L.ASIS),  # (S,D) -> (1,S,D)    :360-361
            (v + "patch_embeddings.kernel", v + "embeddings.patch_embedding.weight", L.CONV),
            (v + "ln_pre.scale", v + "pre_layrnorm.weight", L.ASIS),                   # [sic] HF's spelling
            (v + "ln_pre.bias", v + "pre_layrnorm.bias", L.ASIS),
            (v + "ln_post.scale", v + "post_layernorm.weight", L.ASIS),
            (v + "ln_post.bias", v + "post_layernorm.bias", L.ASIS),
            ("visual_projection.kernel", "visual_projection.weight", L.LINEAR),
        ]
        for i in range(tc["num_hidden_layers"]):
            rules += L.block_rules(f"text_model.blocks.layers.{i}.", f"text_model.encoder.layers.{i}.", L.CLIP_BLOCK)
        for i in range(vc["num_hidden_layers"]):
            rules += L.block_rules(f"{v}transformer.blocks.layers.{i}.", f"{v}encoder.layers.{i}.", L.CLIP_BLOCK)
        # models/clip.py:343-345 skips table entries that are absent on either side, then insists that nothing is left over (:405-414)
        L.apply_mapping(model, hf, rules, missing="skip", shape_error=ValueError, what="CLIP ")
        return model
