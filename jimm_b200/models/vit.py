"""Mirror of jimm.models.vit (reference: src/jimm/models/vit.py): VisionTransformer with the reference's constructor,
`__call__` and `from_pretrained`, running on the H100 CUDA library."""

from __future__ import annotations

import os

import torch

from .. import _lib, nn
from ..common.transformer import g_wrap
from ..common import hf_loader as L
from ..common.utils import load_params_and_config
from ..common.vit import VisionTransformerBase, _NativeOwner, tower_config_fields


class VisionTransformer(_NativeOwner, nn.Module):
    """Vision Transformer for image classification (models/vit.py:16-103)."""

    def __init__(self, num_classes: int = 1000, in_channels: int = 3, img_size: int = 224, patch_size: int = 16, num_layers: int = 12,
                 num_heads: int = 12, mlp_dim: int = 3072, hidden_size: int = 768, dropout_rate: float = 0.1,
                 use_quick_gelu: bool = False, do_classification: bool = True, dtype=torch.float32, param_dtype=torch.float32,
                 rngs=None, mesh=None) -> None:
        nn.Module.__init__(self)
        self._native_init(dtype)
        g = nn._gen(rngs)
        object.__setattr__(self, "do_classification", do_classification)
        object.__setattr__(self, "num_classes", num_classes)
        object.__setattr__(self, "dtype", dtype)
        # models/vit.py:61-78: CLS pooling, no pre-norm, patch bias, layernorm_epsilon=1e-12
        self.add_child("encoder", VisionTransformerBase(
            img_size=img_size, patch_size=patch_size, in_channels=in_channels, hidden_size=hidden_size, num_layers=num_layers,
            num_heads=num_heads, mlp_dim=mlp_dim, dropout_rate=dropout_rate, use_quick_gelu=use_quick_gelu, use_pre_norm=False,
            use_patch_bias=True, layernorm_epsilon=1e-12, rngs=g_wrap(g), dtype=dtype, param_dtype=param_dtype, mesh=mesh))
        if do_classification:
            self.add_child("classifier", nn.Linear(hidden_size, num_classes, rngs=g_wrap(g)))

    def _native_config(self) -> _lib.Config:
        cfg = _lib.Config()
        cfg.kind = _lib.KIND_VIT
        tower_config_fields(cfg, **self.encoder._hp)
        cfg.num_classes = self.num_classes if self.do_classification else 0
        cfg.compute_dtype = self._compute_dtype
        return cfg

    def __call__(self, x, interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """[batch, height, width, channels] -> logits [batch, num_classes] (models/vit.py:91-103).

        Inference semantics (dropout is the identity), like the reference after `.eval()`.  interpolate_pos_encoding (HuggingFace's
        keyword): images of any size of at least one patch, the position embeddings resampled bicubically to the patch grid.  A
        list / tuple of images [H_i, W_i, C] (or [1, H_i, W_i, C]) of different sizes runs in one packed call; row i is the result of
        x[i] alone."""
        return self._vision(x, interpolate_pos_encoding)

    def forward_async(self, x, interpolate_pos_encoding: bool = False):
        """Asynchronous dispatch for host inputs (JAX dispatches asynchronously; examples/vit_inference.py:54-58 only blocks when
        it reads the logits): returns a `PendingResult`; back-to-back calls overlap their H2D copies with the previous forward.  A
        list of images runs as in __call__, synchronously for host images."""
        return self._vision(x, interpolate_pos_encoding, wait=False)

    def forward_tokens(self, x, layers=None, *, dtype=torch.float32, return_pooled: bool = False, interpolate_pos_encoding: bool = False):
        """Per-token hidden states of the encoder (HF's output_hidden_states; VisionTransformerBase.forward_tokens), on the inputs
        __call__ takes.  return_pooled: also return the logits __call__ gives on the same input, bit for bit: (tokens, logits)."""
        return self._vision_tokens(x, layers, dtype, return_pooled, interpolate_pos_encoding)

    def forward_attentions(self, x, blocks=None, *, dtype=torch.float32, return_pooled: bool = False, interpolate_pos_encoding: bool = False):
        """Self-attention weights of the encoder's blocks (HF's output_attentions; VisionTransformerBase.forward_attentions), on the
        inputs __call__ takes.  return_pooled: also return the logits __call__ gives on the same input, bit for bit: (weights, logits)."""
        return self._vision_tokens(x, blocks, dtype, return_pooled, interpolate_pos_encoding, attn=True)

    @classmethod
    def from_pretrained(cls, model_name_or_path: str, use_pytorch: bool = False, mesh=None, dtype=torch.float32) -> "VisionTransformer":
        """Load a HF `ViTForImageClassification` checkpoint (models/vit.py:105-273): same config parsing, shape
        inference without a config, HF->flax name map, layout transforms and strict visit checks."""
        hf, config = load_params_and_config(model_name_or_path, use_pytorch)
        if config:
            dims = dict(hidden_size=config["hidden_size"], num_layers=config["num_hidden_layers"], num_heads=config["num_attention_heads"],
                        mlp_dim=config["intermediate_size"], patch_size=config["patch_size"], img_size=config["image_size"],
                        num_classes=len(config["id2label"]) if "id2label" in config else config.get("num_labels", 1000))
            act = config.get("hidden_act", "gelu")
            if act not in ("gelu", "quick_gelu"):
                print(f"Warning: Unexpected hidden_act '{act}' in config, defaulting to standard GELU.")
            dims["use_quick_gelu"] = act == "quick_gelu"
        elif not use_pytorch and os.path.isfile(model_name_or_path):
            # no config.json beside the file: read the architecture off the tensor shapes (models/vit.py:142-166; heads = width / 64)
            width = hf["vit.embeddings.cls_token"].shape[-1]
            patch = hf["vit.embeddings.patch_embeddings.projection.weight"].shape[2]
            grid = int((hf["vit.embeddings.position_embeddings"].shape[1] - 1) ** 0.5)
            depth = 1 + max((int(k.split(".")[3]) for k in hf if k.startswith("vit.encoder.layer.")), default=-1)
            dims = dict(hidden_size=width, num_layers=depth, num_heads=width // 64, mlp_dim=hf["vit.encoder.layer.0.intermediate.dense.weight"].shape[0],
                        patch_size=patch, img_size=grid * patch, num_classes=hf["classifier.bias"].shape[0], use_quick_gelu=False)
        else:
            raise ValueError(f"Could not load or infer configuration for {model_name_or_path}")

        with nn.deferred_init():  # every parameter is replaced below (and asserted to be)
            model = cls(mesh=mesh, dtype=dtype, param_dtype=dtype, **dims)
        rules = [
            ("encoder.cls_token", "vit.embeddings.cls_token", L.ASIS),
            ("encoder.position_embeddings", "vit.embeddings.position_embeddings", L.ASIS),
            ("encoder.patch_embeddings.kernel", "vit.embeddings.patch_embeddings.projection.weight", L.CONV),
            ("encoder.patch_embeddings.bias", "vit.embeddings.patch_embeddings.projection.bias", L.ASIS),
            ("classifier.kernel", "classifier.weight", L.LINEAR),
            ("classifier.bias", "classifier.bias", L.ASIS),
            ("encoder.ln_post.scale", "vit.layernorm.weight", L.ASIS),
            ("encoder.ln_post.bias", "vit.layernorm.bias", L.ASIS),
        ]
        for i in range(dims["num_layers"]):
            rules += L.block_rules(f"encoder.transformer.blocks.layers.{i}.", f"vit.encoder.layer.{i}.", L.VIT_BLOCK)
        # strictness of models/vit.py:225-268: both names must exist, shapes must agree, nothing may be left over on either side
        L.apply_mapping(model, hf, rules, missing="assert", shape_error=AssertionError, what="")
        return model
