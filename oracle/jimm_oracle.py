"""CPU oracle for the jimm ViT / CLIP / SigLIP inference forward path.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it.  Nothing under ``jimm_b200/`` imports this module; the
product path fails loudly when the CUDA library is missing.

What it is
----------
A plain torch-CPU (fp64 or fp32) restatement of the reference's forward
semantics, function by function, each citing the reference file:line it follows
(paths relative to the reference repository's root).  The arithmetic of the reference lives in
un-vendored third-party code -- flax 0.10.6 (uv.lock:332-333) on jax/jaxlib
0.6.2 (uv.lock:586-587) -- so the layer semantics (nnx.Linear, nnx.LayerNorm
with use_fast_variance, nnx.MultiHeadAttention, nnx.Conv, nnx.gelu == tanh
approximation, nnx.Embed) are restated from that library's published behaviour.

Pinning status
--------------
JAX/flax are not installable in this image, so the reference itself cannot be
executed: **parity is unpinned at the flax boundary**.  What pins the oracle
instead (tests/test_oracle_vs_hf.py, oracle/check_vs_hf.py):
  * the reference's own tests compare against HuggingFace transformers
    (tests/test_vit.py:49-52 <0.05, tests/test_clip.py:48 atol 1e-1,
    tests/test_siglip.py:36,52,69 atol 1e-2).  The oracle is run on random-init
    HF models through the reference's HF->flax layout transforms (restated in
    ``hf_to_flax_*`` below) and must meet those tolerances in *jimm semantics*
    and <=1e-5 in *HF semantics* (``gelu="erf"``, HF eps), which proves every
    transpose / head split / patch order / pooling choice;
  * committed golden fixtures under tests/golden/ (tiny HF checkpoints + HF
    outputs + oracle outputs, made by tests/golden/make_golden.py).

Parameter trees are flat dicts keyed by the reference's flax paths joined with
"." (e.g. ``encoder.transformer.blocks.layers.0.attn.query.kernel``) holding
torch tensors in the reference's layouts (SURVEY.md section 8b table).
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch

Params = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------- #
# operand rounding emulation (sets per-dtype expectations for the CUDA path)
# --------------------------------------------------------------------------- #
def _round_tf32(x: torch.Tensor) -> torch.Tensor:
    """Round-to-nearest-even to 10 explicit mantissa bits (tf32 operand format)."""
    xi = x.to(torch.float32).contiguous().view(torch.int32)
    bias = ((xi >> 13) & 1) + 0x0FFF
    xi = (xi + bias) & ~0x1FFF
    return xi.view(torch.float32)


def round_operand(x: torch.Tensor, mode: Optional[str]) -> torch.Tensor:
    """Emulate tensor-core operand rounding; accumulation stays in x.dtype."""
    if mode is None:
        return x
    dt = x.dtype
    if mode == "fp16":
        return x.to(torch.float16).to(dt)
    if mode == "bf16":
        return x.to(torch.bfloat16).to(dt)
    if mode == "tf32":
        return _round_tf32(x).to(dt)
    raise ValueError(mode)


@dataclass
class Semantics:
    """Knobs that exist ONLY so the oracle can be pinned against HF transformers.

    jimm semantics (the parity target) are the defaults."""

    gelu: str = "tanh"  # nnx.gelu default approximate=True (common/transformer.py:90, common/vit.py:75)
    block_eps: Optional[float] = None  # None -> Transformer default 1e-6 (common/transformer.py:142)
    operand_round: Optional[str] = None  # None | "fp16" | "bf16" | "tf32"
    # flax `dtype=` semantics ([flax-knowledge], flax 0.10.6 nnx/nn/linear.py, normalization.py, attention.py): with
    # dtype=bf16 every layer promotes its inputs AND parameters to bf16 (promote_dtype) and returns a bf16 array, so the
    # residual stream, every bias add, every activation and the softmax are rounded to bf16; only the LayerNorm statistics
    # are computed in fp32.  That is the path examples/vit_inference.py:14-21 takes (from_pretrained(..., dtype=jnp.bfloat16),
    # models/vit.py:181-182 also sets param_dtype=dtype).  act_round="bf16" (with operand_round="bf16") restates it: every
    # op output below goes through _out().  The dot_general accumulates in fp32 and rounds once (XLA CPU), softmax is
    # rounded after the normalisation only (XLA fuses the elementwise chain in fp32) -- both are statements about the
    # absent third-party library, see the header.
    act_round: Optional[str] = None  # None | "bf16" | "fp16"


JIMM = Semantics()
FLAX_BF16 = Semantics(operand_round="bf16", act_round="bf16")


def _out(x: torch.Tensor, sem: "Semantics") -> torch.Tensor:
    """Round a layer output to the flax compute dtype (identity in fp32 semantics)."""
    return x if sem.act_round is None else round_operand(x, sem.act_round)


def _prm(x: torch.Tensor, sem: "Semantics") -> torch.Tensor:
    """A parameter as the layer sees it after promote_dtype (biases, LN scale/bias, cls, pos, scalars)."""
    return x if sem.act_round is None else round_operand(x, sem.act_round)


# --------------------------------------------------------------------------- #
# flax.nnx layer semantics
# --------------------------------------------------------------------------- #
def linear(x, kernel, bias=None, sem: Semantics = JIMM):
    """nnx.Linear: y = x @ kernel (+ bias); kernel is (in, out)."""
    y = _out(round_operand(x, sem.operand_round) @ round_operand(kernel, sem.operand_round), sem)
    return y if bias is None else _out(y + _prm(bias, sem), sem)


def layer_norm(x, scale, bias, eps, sem: "Semantics" = None):
    """nnx.LayerNorm with use_fast_variance=True: var = max(0, E[x^2] - E[x]^2); statistics in fp32 whatever `dtype`."""
    sem = sem or JIMM
    mean = x.mean(-1, keepdim=True)
    mean2 = (x * x).mean(-1, keepdim=True)
    var = torch.clamp(mean2 - mean * mean, min=0.0)
    return _out((x - mean) * torch.rsqrt(var + eps) * _prm(scale, sem) + _prm(bias, sem), sem)


def gelu_tanh(x):
    """jax.nn.gelu(approximate=True)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x * x * x)))


def quickgelu(x):
    """common/transformer.py:12-19."""
    return x * torch.sigmoid(1.702 * x)


def _act(x, use_quick_gelu: bool, sem: Semantics):
    if use_quick_gelu:
        return _out(quickgelu(x), sem)
    if sem.gelu == "erf":
        return torch.nn.functional.gelu(x)
    return _out(gelu_tanh(x), sem)


def multi_head_attention(p: Params, prefix: str, xq, xkv, num_heads: int, mask=None, sem: Semantics = JIMM):
    """nnx.MultiHeadAttention (common/transformer.py:67-79, common/vit.py:42-53).

    query/key/value kernels (D,H,d), biases (H,d); out kernel (H,d,D), bias (D).
    softmax((q/sqrt(d)) k^T masked) v; mask non-zero == keep."""
    Wq, Wk, Wv = p[prefix + "query.kernel"], p[prefix + "key.kernel"], p[prefix + "value.kernel"]
    D, H, d = Wq.shape
    assert H == num_heads
    r = lambda t: round_operand(t, sem.operand_round)
    o_ = lambda t: _out(t, sem)
    q = o_(o_(r(xq) @ r(Wq.reshape(D, H * d))) + _prm(p[prefix + "query.bias"].reshape(H * d), sem))
    k = o_(o_(r(xkv) @ r(Wk.reshape(D, H * d))) + _prm(p[prefix + "key.bias"].reshape(H * d), sem))
    v = o_(o_(r(xkv) @ r(Wv.reshape(D, H * d))) + _prm(p[prefix + "value.bias"].reshape(H * d), sem))
    B, Sq, _ = q.shape
    Sk = k.shape[1]
    q = o_(q.reshape(B, Sq, H, d).permute(0, 2, 1, 3) / math.sqrt(d))
    k = k.reshape(B, Sk, H, d).permute(0, 2, 1, 3)
    v = v.reshape(B, Sk, H, d).permute(0, 2, 1, 3)
    w = o_(r(q) @ r(k).transpose(-1, -2))  # [B,H,Sq,Sk]
    if mask is not None:
        w = torch.where(mask != 0, w, torch.finfo(w.dtype).min)
    w = o_(torch.softmax(w, dim=-1))
    o = o_(r(w) @ r(v))  # [B,H,Sq,d]
    o = o.permute(0, 2, 1, 3).reshape(B, Sq, H * d)
    Wo = p[prefix + "out.kernel"].reshape(H * d, D)
    return o_(o_(r(o) @ r(Wo)) + _prm(p[prefix + "out.bias"], sem))


# --------------------------------------------------------------------------- #
# common/transformer.py
# --------------------------------------------------------------------------- #
def transformer_encoder(p: Params, prefix: str, x, num_heads, eps, use_quick_gelu, mask, sem: Semantics = JIMM):
    """TransformerEncoder.__call__ (common/transformer.py:116-132)."""
    if mask is not None:
        s = min(x.shape[1], mask.shape[0])  # :125-129
        mask = mask[:s, :s]
    h = layer_norm(x, p[prefix + "norm1.scale"], p[prefix + "norm1.bias"], eps, sem)
    x = _out(x + multi_head_attention(p, prefix + "attn.", h, h, num_heads, mask, sem), sem)  # :130
    h = layer_norm(x, p[prefix + "norm2.scale"], p[prefix + "norm2.bias"], eps, sem)
    h = linear(h, p[prefix + "mlp.layers.0.kernel"], p[prefix + "mlp.layers.0.bias"], sem)
    h = _act(h, use_quick_gelu, sem)
    h = linear(h, p[prefix + "mlp.layers.3.kernel"], p[prefix + "mlp.layers.3.bias"], sem)
    return _out(x + h, sem)  # :131


def transformer(p: Params, prefix: str, x, layers, num_heads, use_quick_gelu, mask=None, eps=1e-6, sem: Semantics = JIMM):
    """Transformer.__call__ (common/transformer.py:171-196).  eps default 1e-6 (:142)."""
    if sem.block_eps is not None:
        eps = sem.block_eps
    for i in range(layers):
        x = transformer_encoder(p, f"{prefix}blocks.layers.{i}.", x, num_heads, eps, use_quick_gelu, mask, sem)
    return x


# --------------------------------------------------------------------------- #
# common/vit.py
# --------------------------------------------------------------------------- #
def map_head(p: Params, prefix: str, x, num_heads, eps, sem: Semantics = JIMM):
    """MultiHeadAttentionPoolingHead.__call__ (common/vit.py:87-101)."""
    B = x.shape[0]
    probe = _prm(p[prefix + "probe"], sem).expand(B, -1, -1)  # :96
    y = multi_head_attention(p, prefix + "attn.", probe, x, num_heads, None, sem)  # :97
    residual = y
    y = layer_norm(y, p[prefix + "layernorm.scale"], p[prefix + "layernorm.bias"], eps, sem)
    h = linear(y, p[prefix + "mlp.layers.0.kernel"], p[prefix + "mlp.layers.0.bias"], sem)
    h = torch.nn.functional.gelu(h) if sem.gelu == "erf" else _out(gelu_tanh(h), sem)  # nnx.gelu :75
    h = linear(h, p[prefix + "mlp.layers.2.kernel"], p[prefix + "mlp.layers.2.bias"], sem)
    return _out(residual + h, sem)[:, 0]  # :100-101


@dataclass
class TowerCfg:
    """ctor kwargs of VisionTransformerBase (common/vit.py:107-126)."""

    img_size: int
    patch_size: int
    in_channels: int
    hidden_size: int
    num_layers: int
    num_heads: int
    mlp_dim: int
    pooling_type: str = "CLS"
    use_quick_gelu: bool = False
    use_pre_norm: bool = False
    use_patch_bias: bool = True
    layernorm_epsilon: float = 1e-5
    map_mlp: Optional[int] = None  # MAP head MLP width; None: 4 * hidden_size (common/vit.py:175)


def patch_embed(p: Params, prefix: str, img, cfg: TowerCfg, sem: Semantics = JIMM):
    """nnx.Conv NHWC x HWIO, stride P, VALID (common/vit.py:153-165, :228-230)
    == GEMM [B*n, P*P*C] x [P*P*C, D], A-row order (kh, kw, c)."""
    B, Hh, Ww, C = img.shape
    P = cfg.patch_size
    gh, gw = Hh // P, Ww // P
    x = img[:, : gh * P, : gw * P, :].reshape(B, gh, P, gw, P, C).permute(0, 1, 3, 2, 4, 5).reshape(B, gh * gw, P * P * C)
    K = p[prefix + "patch_embeddings.kernel"].reshape(P * P * C, -1)
    y = _out(round_operand(x, sem.operand_round) @ round_operand(K, sem.operand_round), sem)
    if cfg.use_patch_bias:
        y = _out(y + _prm(p[prefix + "patch_embeddings.bias"], sem), sem)
    return y


def vision_tower(p: Params, prefix: str, img, cfg: TowerCfg, sem: Semantics = JIMM):
    """VisionTransformerBase.__call__ (common/vit.py:216-248)."""
    if cfg.pooling_type not in ("CLS", "MAP"):
        raise ValueError("pooling_type must be either MAP or CLS.")  # :178
    x = patch_embed(p, prefix, img, cfg, sem)
    B = x.shape[0]
    if cfg.pooling_type == "CLS":
        cls = _prm(p[prefix + "cls_token"], sem).expand(B, -1, -1)  # :232
        x = torch.cat([cls, x], dim=1)  # :233
    x = _out(x + _prm(p[prefix + "position_embeddings"], sem), sem)  # :236
    if cfg.use_pre_norm:
        x = layer_norm(x, p[prefix + "ln_pre.scale"], p[prefix + "ln_pre.bias"], cfg.layernorm_epsilon, sem)  # :239
    # dropout is identity in eval (:241)
    # NOTE quirk 2: the Transformer is built WITHOUT layernorm_epsilon (:193-204) -> block eps 1e-6
    x = transformer(p, prefix + "transformer.", x, cfg.num_layers, cfg.num_heads, cfg.use_quick_gelu, None, 1e-6, sem)
    x = layer_norm(x, p[prefix + "ln_post.scale"], p[prefix + "ln_post.bias"], cfg.layernorm_epsilon, sem)  # :244
    if cfg.pooling_type == "CLS":
        return x[:, 0]  # :246
    return map_head(p, prefix + "MAPHead.", x, cfg.num_heads, cfg.layernorm_epsilon, sem)  # :248


# --------------------------------------------------------------------------- #
# models/vit.py
# --------------------------------------------------------------------------- #
@dataclass
class ViTCfg:
    """ctor kwargs of VisionTransformer (models/vit.py:23-40)."""

    num_classes: int = 1000
    in_channels: int = 3
    img_size: int = 224
    patch_size: int = 16
    num_layers: int = 12
    num_heads: int = 12
    mlp_dim: int = 3072
    hidden_size: int = 768
    use_quick_gelu: bool = False
    do_classification: bool = True

    def tower(self) -> TowerCfg:
        # models/vit.py:61-78: CLS, no pre-norm, patch bias, eps 1e-12
        return TowerCfg(self.img_size, self.patch_size, self.in_channels, self.hidden_size, self.num_layers, self.num_heads,
                        self.mlp_dim, "CLS", self.use_quick_gelu, False, True, 1e-12)


def vit_forward(p: Params, cfg: ViTCfg, img, sem: Semantics = JIMM):
    """VisionTransformer.__call__ (models/vit.py:91-103)."""
    x = vision_tower(p, "encoder.", img, cfg.tower(), sem)
    if cfg.do_classification:
        return linear(x, p["classifier.kernel"], p["classifier.bias"], sem)
    return x


# --------------------------------------------------------------------------- #
# models/clip.py, models/siglip.py
# --------------------------------------------------------------------------- #
@dataclass
class DualCfg:
    """ctor kwargs shared by CLIP (models/clip.py:16-31) and SigLIP (models/siglip.py:16-31)."""

    image_resolution: int
    vision_layers: int
    vision_width: int
    vision_patch_size: int
    context_length: int
    vocab_size: int
    transformer_width: int
    transformer_heads: int
    transformer_layers: int
    # HF checkpoints that depart from the reference's rule; None is the rule: vision heads vision_width // 64 (models/clip.py:60,
    # models/siglip.py:59), MLPs 4x the width (the MAP head's too, common/vit.py:175), QuickGELU on CLIP's towers and tanh GELU on SigLIP's
    vision_heads: Optional[int] = None
    vision_mlp: Optional[int] = None
    text_mlp: Optional[int] = None
    map_mlp: Optional[int] = None
    vision_quick_gelu: Optional[bool] = None
    text_quick_gelu: Optional[bool] = None

    @property
    def v_heads(self) -> int:
        return self.vision_heads or self.vision_width // 64

    @property
    def t_mlp(self) -> int:
        return self.text_mlp or 4 * self.transformer_width

    def text_quick(self, kind: str) -> bool:
        return (kind == "clip") if self.text_quick_gelu is None else self.text_quick_gelu

    def clip_tower(self) -> TowerCfg:
        # models/clip.py:60-81
        quick = True if self.vision_quick_gelu is None else self.vision_quick_gelu
        return TowerCfg(self.image_resolution, self.vision_patch_size, 3, self.vision_width, self.vision_layers,
                        self.v_heads, self.vision_mlp or self.vision_width * 4, "CLS", quick, True, False, 1e-5)

    def siglip_tower(self) -> TowerCfg:
        # models/siglip.py:59-78
        quick = False if self.vision_quick_gelu is None else self.vision_quick_gelu
        return TowerCfg(self.image_resolution, self.vision_patch_size, 3, self.vision_width, self.vision_layers,
                        self.v_heads, self.vision_mlp or self.vision_width * 4, "MAP", quick, False, True, 1e-6, self.map_mlp)


def clip_encode_image(p: Params, cfg: DualCfg, img, sem: Semantics = JIMM):
    """CLIP.encode_image (models/clip.py:135-146)."""
    f = vision_tower(p, "vision_model.", img, cfg.clip_tower(), sem)
    return linear(f, p["visual_projection.kernel"], None, sem)


def clip_encode_text(p: Params, cfg: DualCfg, text, sem: Semantics = JIMM):
    """CLIP.encode_text (models/clip.py:148-167)."""
    seq = text.shape[1]
    x = _prm(p["token_embedding.embedding"][text], sem)  # :159
    x = _out(x + _prm(p["positional_embedding"][:seq], sem), sem)  # :160
    mask = torch.tril(torch.ones(cfg.context_length, cfg.context_length, dtype=x.dtype))  # :62
    x = transformer(p, "text_model.", x, cfg.transformer_layers, cfg.transformer_heads, cfg.text_quick("clip"), mask, 1e-6, sem)  # :161 (eps not forwarded :92-104)
    x = layer_norm(x, p["ln_final.scale"], p["ln_final.bias"], 1e-5, sem)  # :162 (:117)
    eot = text.argmax(dim=-1)  # :164
    x = x[torch.arange(x.shape[0]), eot]
    return _out(round_operand(x, sem.operand_round) @ round_operand(p["text_projection.kernel"], sem.operand_round), sem)  # :166


def contrastive_logits(img_f, txt_f, logit_scale, logit_bias=None, sem: Semantics = JIMM):
    """models/clip.py:183-187 / models/siglip.py:169-173 (no epsilon in the norms).  In flax-bf16 semantics the features
    arrive as bf16 arrays, so the norm, the division, exp(logit_scale) and the matmul each return bf16."""
    o_ = lambda t: _out(t, sem)
    i = o_(img_f / o_(torch.linalg.norm(img_f, dim=-1, keepdim=True)))
    t = o_(txt_f / o_(torch.linalg.norm(txt_f, dim=-1, keepdim=True)))
    logits = o_(o_(o_(torch.exp(_prm(logit_scale, sem))) * i) @ t.T)
    return logits if logit_bias is None else o_(logits + _prm(logit_bias, sem))


def clip_forward(p: Params, cfg: DualCfg, img, text, sem: Semantics = JIMM):
    """CLIP.__call__ (models/clip.py:169-188)."""
    return contrastive_logits(clip_encode_image(p, cfg, img, sem), clip_encode_text(p, cfg, text, sem), p["logit_scale"], None, sem)


def siglip_encode_image(p: Params, cfg: DualCfg, img, sem: Semantics = JIMM):
    """SigLIP.encode_image (models/siglip.py:123-133)."""
    return vision_tower(p, "vision_model.", img, cfg.siglip_tower(), sem)


def siglip_encode_text(p: Params, cfg: DualCfg, text, sem: Semantics = JIMM):
    """SigLIP.encode_text (models/siglip.py:135-153)."""
    seq = text.shape[1]
    x = _prm(p["token_embedding.embedding"][text], sem)
    x = _out(x + _prm(p["positional_embedding"][:seq], sem), sem)
    x = transformer(p, "text_model.", x, cfg.transformer_layers, cfg.transformer_heads, cfg.text_quick("siglip"), None, 1e-6, sem)  # :81-92 eps 1e-6
    x = layer_norm(x, p["ln_final.scale"], p["ln_final.bias"], 1e-6, sem)  # :104
    return linear(x[:, -1, :], p["text_projection.kernel"], p["text_projection.bias"], sem)  # :151-152


def siglip_forward(p: Params, cfg: DualCfg, img, text, sem: Semantics = JIMM):
    """SigLIP.__call__ (models/siglip.py:155-174)."""
    return contrastive_logits(siglip_encode_image(p, cfg, img, sem), siglip_encode_text(p, cfg, text, sem),
                              p["logit_scale"], p["logit_bias"], sem)


# --------------------------------------------------------------------------- #
# HF checkpoint -> flax-path parameter tree (the reference's from_pretrained transforms)
# --------------------------------------------------------------------------- #
def _qkv_w(w, H):  # (D_out, D_in) -> (D, H, d)   models/vit.py:241-243
    D = w.shape[1]
    return w.T.reshape(D, H, w.shape[0] // H)


def _out_w(w, H):  # (D, H*d) -> (H, d, D)        models/vit.py:246-248
    return w.T.reshape(H, w.shape[1] // H, w.shape[0])


def hf_to_flax_vit(sd: Dict[str, torch.Tensor], num_layers: int, num_heads: int) -> Params:
    """models/vit.py:192-250."""
    o: Params = {}
    o["encoder.cls_token"] = sd["vit.embeddings.cls_token"]
    o["encoder.position_embeddings"] = sd["vit.embeddings.position_embeddings"]
    o["encoder.patch_embeddings.kernel"] = sd["vit.embeddings.patch_embeddings.projection.weight"].permute(2, 3, 1, 0)  # :239-240
    o["encoder.patch_embeddings.bias"] = sd["vit.embeddings.patch_embeddings.projection.bias"]
    o["classifier.kernel"] = sd["classifier.weight"].T
    o["classifier.bias"] = sd["classifier.bias"]
    o["encoder.ln_post.scale"] = sd["vit.layernorm.weight"]
    o["encoder.ln_post.bias"] = sd["vit.layernorm.bias"]
    for i in range(num_layers):
        f = f"encoder.transformer.blocks.layers.{i}."
        h = f"vit.encoder.layer.{i}."
        for y in ("query", "key", "value"):
            o[f + f"attn.{y}.kernel"] = _qkv_w(sd[h + f"attention.attention.{y}.weight"], num_heads)
            o[f + f"attn.{y}.bias"] = sd[h + f"attention.attention.{y}.bias"].reshape(num_heads, -1)
        o[f + "attn.out.kernel"] = _out_w(sd[h + "attention.output.dense.weight"], num_heads)
        o[f + "attn.out.bias"] = sd[h + "attention.output.dense.bias"]
        o[f + "mlp.layers.0.kernel"] = sd[h + "intermediate.dense.weight"].T
        o[f + "mlp.layers.0.bias"] = sd[h + "intermediate.dense.bias"]
        o[f + "mlp.layers.3.kernel"] = sd[h + "output.dense.weight"].T
        o[f + "mlp.layers.3.bias"] = sd[h + "output.dense.bias"]
        o[f + "norm1.scale"] = sd[h + "layernorm_before.weight"]
        o[f + "norm1.bias"] = sd[h + "layernorm_before.bias"]
        o[f + "norm2.scale"] = sd[h + "layernorm_after.weight"]
        o[f + "norm2.bias"] = sd[h + "layernorm_after.bias"]
    return {k: v.contiguous() for k, v in o.items()}


def _dual_blocks(o: Params, sd, flax_prefix: str, hf_prefix: str, layers: int, heads: int):
    """models/clip.py:286-334 / models/siglip.py:258-306 + transforms clip.py:362-390."""
    for i in range(layers):
        f = f"{flax_prefix}blocks.layers.{i}."
        h = f"{hf_prefix}encoder.layers.{i}."
        for fl, hf in (("query", "q_proj"), ("key", "k_proj"), ("value", "v_proj")):
            o[f + f"attn.{fl}.kernel"] = _qkv_w(sd[h + f"self_attn.{hf}.weight"], heads)
            o[f + f"attn.{fl}.bias"] = sd[h + f"self_attn.{hf}.bias"].reshape(heads, -1)
        o[f + "attn.out.kernel"] = _out_w(sd[h + "self_attn.out_proj.weight"], heads)
        o[f + "attn.out.bias"] = sd[h + "self_attn.out_proj.bias"]
        o[f + "norm1.scale"] = sd[h + "layer_norm1.weight"]
        o[f + "norm1.bias"] = sd[h + "layer_norm1.bias"]
        o[f + "norm2.scale"] = sd[h + "layer_norm2.weight"]
        o[f + "norm2.bias"] = sd[h + "layer_norm2.bias"]
        o[f + "mlp.layers.0.kernel"] = sd[h + "mlp.fc1.weight"].T
        o[f + "mlp.layers.0.bias"] = sd[h + "mlp.fc1.bias"]
        o[f + "mlp.layers.3.kernel"] = sd[h + "mlp.fc2.weight"].T
        o[f + "mlp.layers.3.bias"] = sd[h + "mlp.fc2.bias"]


def hf_to_flax_clip(sd, cfg: DualCfg) -> Params:
    """models/clip.py:269-396."""
    o: Params = {}
    o["logit_scale"] = sd["logit_scale"]
    o["positional_embedding"] = sd["text_model.embeddings.position_embedding.weight"]
    o["token_embedding.embedding"] = sd["text_model.embeddings.token_embedding.weight"]
    o["ln_final.scale"] = sd["text_model.final_layer_norm.weight"]
    o["ln_final.bias"] = sd["text_model.final_layer_norm.bias"]
    o["text_projection.kernel"] = sd["text_projection.weight"].T
    o["vision_model.cls_token"] = sd["vision_model.embeddings.class_embedding"].reshape(1, 1, -1)  # :358-359
    pe = sd["vision_model.embeddings.position_embedding.weight"]
    o["vision_model.position_embeddings"] = pe.reshape(1, *pe.shape)  # :360-361
    o["vision_model.patch_embeddings.kernel"] = sd["vision_model.embeddings.patch_embedding.weight"].permute(2, 3, 1, 0)
    o["vision_model.ln_pre.scale"] = sd["vision_model.pre_layrnorm.weight"]
    o["vision_model.ln_pre.bias"] = sd["vision_model.pre_layrnorm.bias"]
    o["vision_model.ln_post.scale"] = sd["vision_model.post_layernorm.weight"]
    o["vision_model.ln_post.bias"] = sd["vision_model.post_layernorm.bias"]
    o["visual_projection.kernel"] = sd["visual_projection.weight"].T
    _dual_blocks(o, sd, "text_model.", "text_model.", cfg.transformer_layers, cfg.transformer_heads)
    _dual_blocks(o, sd, "vision_model.transformer.", "vision_model.", cfg.vision_layers, cfg.v_heads)
    return {k: v.contiguous() for k, v in o.items()}


def hf_to_flax_siglip(sd, cfg: DualCfg) -> Params:
    """models/siglip.py:228-366."""
    o: Params = {}
    o["logit_scale"] = sd["logit_scale"].squeeze()  # :322-323
    o["logit_bias"] = sd["logit_bias"].squeeze()
    o["positional_embedding"] = sd["text_model.embeddings.position_embedding.weight"]
    o["token_embedding.embedding"] = sd["text_model.embeddings.token_embedding.weight"]
    o["ln_final.scale"] = sd["text_model.final_layer_norm.weight"]
    o["ln_final.bias"] = sd["text_model.final_layer_norm.bias"]
    o["text_projection.kernel"] = sd["text_model.head.weight"].T
    o["text_projection.bias"] = sd["text_model.head.bias"]
    v = "vision_model."
    o[v + "patch_embeddings.kernel"] = sd[v + "embeddings.patch_embedding.weight"].permute(2, 3, 1, 0)
    o[v + "patch_embeddings.bias"] = sd[v + "embeddings.patch_embedding.bias"]
    pe = sd[v + "embeddings.position_embedding.weight"]
    o[v + "position_embeddings"] = pe.reshape(1, *pe.shape)
    o[v + "ln_post.scale"] = sd[v + "post_layernorm.weight"]
    o[v + "ln_post.bias"] = sd[v + "post_layernorm.bias"]
    H = cfg.v_heads
    m = v + "MAPHead."
    o[m + "probe"] = sd[v + "head.probe"]
    o[m + "layernorm.scale"] = sd[v + "head.layernorm.weight"]
    o[m + "layernorm.bias"] = sd[v + "head.layernorm.bias"]
    o[m + "mlp.layers.0.kernel"] = sd[v + "head.mlp.fc1.weight"].T
    o[m + "mlp.layers.0.bias"] = sd[v + "head.mlp.fc1.bias"]
    o[m + "mlp.layers.2.kernel"] = sd[v + "head.mlp.fc2.weight"].T
    o[m + "mlp.layers.2.bias"] = sd[v + "head.mlp.fc2.bias"]
    qw, kw, vw = torch.chunk(sd[v + "head.attention.in_proj_weight"], 3, dim=0)  # :352-357
    qb, kb, vb = torch.chunk(sd[v + "head.attention.in_proj_bias"], 3, dim=0)  # :358-363
    for name, w, b in (("query", qw, qb), ("key", kw, kb), ("value", vw, vb)):
        o[m + f"attn.{name}.kernel"] = _qkv_w(w, H)
        o[m + f"attn.{name}.bias"] = b.reshape(H, -1)
    o[m + "attn.out.kernel"] = _out_w(sd[v + "head.attention.out_proj.weight"], H)
    o[m + "attn.out.bias"] = sd[v + "head.attention.out_proj.bias"]
    _dual_blocks(o, sd, "text_model.", "text_model.", cfg.transformer_layers, cfg.transformer_heads)
    _dual_blocks(o, sd, "vision_model.transformer.", "vision_model.", cfg.vision_layers, H)
    return {k: v_.contiguous() for k, v_ in o.items()}


def cast_params(p: Params, dtype) -> Params:
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in p.items()}


# --------------------------------------------------------------------------- #
# random-init parameter trees with the reference's init distributions (SURVEY 8c),
# biases / LN / cls / probe perturbed so bias-handling bugs are visible.
# --------------------------------------------------------------------------- #
def _xavier(g, *shape, fan_in, fan_out):
    a = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(*shape, generator=g, dtype=torch.float64) * 2 - 1) * a


def _small(g, *shape, s=0.02):
    return torch.randn(*shape, generator=g, dtype=torch.float64) * s


def _rand_blocks(o: Params, g, prefix, layers, D, H, M):
    d = D // H
    for i in range(layers):
        f = f"{prefix}blocks.layers.{i}."
        for y in ("query", "key", "value"):
            o[f + f"attn.{y}.kernel"] = _xavier(g, D, H, d, fan_in=D, fan_out=D)
            o[f + f"attn.{y}.bias"] = _small(g, H, d)
        o[f + "attn.out.kernel"] = _xavier(g, H, d, D, fan_in=D, fan_out=D)
        o[f + "attn.out.bias"] = _small(g, D)
        for n in ("norm1", "norm2"):
            o[f + n + ".scale"] = 1.0 + _small(g, D, s=0.1)
            o[f + n + ".bias"] = _small(g, D, s=0.1)
        o[f + "mlp.layers.0.kernel"] = _xavier(g, D, M, fan_in=D, fan_out=M)
        o[f + "mlp.layers.0.bias"] = _small(g, M)
        o[f + "mlp.layers.3.kernel"] = _xavier(g, M, D, fan_in=M, fan_out=D)
        o[f + "mlp.layers.3.bias"] = _small(g, D)


def _rand_tower(o: Params, g, prefix, t: TowerCfg):
    D, P, C = t.hidden_size, t.patch_size, t.in_channels
    n = (t.img_size // P) ** 2
    o[prefix + "patch_embeddings.kernel"] = _xavier(g, P, P, C, D, fan_in=P * P * C, fan_out=D)
    if t.use_patch_bias:
        o[prefix + "patch_embeddings.bias"] = _small(g, D)
    if t.pooling_type == "CLS":
        o[prefix + "cls_token"] = _small(g, 1, 1, D, s=0.5)
        o[prefix + "position_embeddings"] = _small(g, 1, n + 1, D, s=0.2)
    else:
        o[prefix + "position_embeddings"] = _small(g, 1, n, D, s=0.2)
        m = prefix + "MAPHead."
        d = D // t.num_heads
        o[m + "probe"] = _small(g, 1, 1, D, s=0.5)
        for y in ("query", "key", "value"):
            o[m + f"attn.{y}.kernel"] = _xavier(g, D, t.num_heads, d, fan_in=D, fan_out=D)
            o[m + f"attn.{y}.bias"] = _small(g, t.num_heads, d)
        o[m + "attn.out.kernel"] = _xavier(g, t.num_heads, d, D, fan_in=D, fan_out=D)
        o[m + "attn.out.bias"] = _small(g, D)
        o[m + "layernorm.scale"] = 1.0 + _small(g, D, s=0.1)
        o[m + "layernorm.bias"] = _small(g, D, s=0.1)
        M = t.map_mlp or 4 * D
        o[m + "mlp.layers.0.kernel"] = _xavier(g, D, M, fan_in=D, fan_out=M)
        o[m + "mlp.layers.0.bias"] = _small(g, M)
        o[m + "mlp.layers.2.kernel"] = _xavier(g, M, D, fan_in=M, fan_out=D)
        o[m + "mlp.layers.2.bias"] = _small(g, D)
    if t.use_pre_norm:
        o[prefix + "ln_pre.scale"] = 1.0 + _small(g, D, s=0.1)
        o[prefix + "ln_pre.bias"] = _small(g, D, s=0.1)
    o[prefix + "ln_post.scale"] = 1.0 + _small(g, D, s=0.1)
    o[prefix + "ln_post.bias"] = _small(g, D, s=0.1)
    _rand_blocks(o, g, prefix + "transformer.", t.num_layers, D, t.num_heads, t.mlp_dim)


def random_vit_params(cfg: ViTCfg, seed=0, dtype=torch.float32) -> Params:
    g = torch.Generator().manual_seed(seed)
    o: Params = {}
    _rand_tower(o, g, "encoder.", cfg.tower())
    if cfg.do_classification:
        o["classifier.kernel"] = _xavier(g, cfg.hidden_size, cfg.num_classes, fan_in=cfg.hidden_size, fan_out=cfg.num_classes)
        o["classifier.bias"] = _small(g, cfg.num_classes)
    return cast_params(o, dtype)


def random_tower_params(t: TowerCfg, seed=0, dtype=torch.float32, prefix="") -> Params:
    g = torch.Generator().manual_seed(seed)
    o: Params = {}
    _rand_tower(o, g, prefix, t)
    return cast_params(o, dtype)


def random_dual_params(cfg: DualCfg, kind: str, seed=0, dtype=torch.float32) -> Params:
    g = torch.Generator().manual_seed(seed)
    o: Params = {}
    Dt, T, V = cfg.transformer_width, cfg.context_length, cfg.vocab_size
    if kind == "clip":
        _rand_tower(o, g, "vision_model.", cfg.clip_tower())
        o["visual_projection.kernel"] = _xavier(g, cfg.vision_width, Dt, fan_in=cfg.vision_width, fan_out=Dt)
        o["text_projection.kernel"] = _xavier(g, Dt, Dt, fan_in=Dt, fan_out=Dt)
        o["logit_scale"] = torch.tensor(2.6592, dtype=torch.float64)
    elif kind == "siglip":
        _rand_tower(o, g, "vision_model.", cfg.siglip_tower())
        o["text_projection.kernel"] = _xavier(g, Dt, Dt, fan_in=Dt, fan_out=Dt)
        o["text_projection.bias"] = _small(g, Dt)
        o["logit_scale"] = torch.tensor(2.3, dtype=torch.float64)
        o["logit_bias"] = torch.tensor(-1.7, dtype=torch.float64)
    else:
        raise ValueError(kind)
    o["token_embedding.embedding"] = _small(g, V, Dt, s=0.3)
    o["positional_embedding"] = _small(g, T, Dt, s=0.1)
    o["ln_final.scale"] = 1.0 + _small(g, Dt, s=0.1)
    o["ln_final.bias"] = _small(g, Dt, s=0.1)
    _rand_blocks(o, g, "text_model.", cfg.transformer_layers, Dt, cfg.transformer_heads, cfg.t_mlp)
    return cast_params(o, dtype)


def synthetic_images(B, img, C=3, seed=1234, dtype=torch.float32):
    """SURVEY 8d: standard normal NHWC."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, img, img, C, generator=g, dtype=torch.float32).to(dtype)


def synthetic_tokens(B, T, V, kind: str, seed=4321):
    """SURVEY 8d: ids uniform in [1, V-2]; CLIP rows get one EOT = V-1 at a random position >= 1."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, V - 1, (B, T), generator=g, dtype=torch.int64)
    if kind == "clip":
        pos = torch.randint(1, T, (B,), generator=g)
        ids[torch.arange(B), pos] = V - 1
    return ids
