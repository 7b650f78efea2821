"""Attention head widths other than 64: any multiple of 8 from 8 to 128 (d = width / heads).

- CPU: jimm_model_create accepts the configurations that need it (the SigLIP so400m notebook model, d = 72 in its text tower; the
  MNIST ViT of the reference's training example, d = 16; a bare encoder at d = 80) and refuses d = 12, d = 136 and widths that the
  heads do not divide.  The oracle matches HuggingFace at d = 80 (ViT) and d = 72 (SigLIP), so it is a fair judge there.
- GPU kernels: jimm_k_attention_hd against exact fp64 softmax attention and against a tile-faithful fp64 restatement of the
  kernel, with neighbouring heads holding large values (a missing zero fill of the padded columns would pick them up); the
  reverse walk, 16-bit and tf32 outputs bit for bit against the fp32 forward output; rows past B * S untouched.  d = 64 through
  jimm_k_attention_hd is jimm_k_attention_ex bit for bit.  jimm_k_map_attention_hd against fp64.
- GPU models against the oracle: the MNIST ViT, the so400m SigLIP (2+2 layers and the full 27+27), a ViT-H/14-shaped tower in CLS
  and MAP pooling, a bare Transformer and MAP head at d = 72, and VisionTransformer.from_pretrained on a d = 80 HF checkpoint."""

import ctypes
import math

import pytest
import torch

import jimm_oracle as O
from attn_oracle import EXACT_TOL, _attn_ref, _check_tile_faithful
from gpu_util import BF16, CODE, F16, F32, check, check_parity, ptr, stream
from test_kernel_paths_gpu import SENTINEL, TF32, rna_tf32 as _rna_tf32

DEV = "cuda"
SMS = 132
TOL = 1e-3  # the model parity bars of test_parity_gpu.py
LOGITS_TOL = 2e-3
BF16_VS_SAME = 8e-3
BF16_VS_FP32 = 1.5e-2


# ---------------------------------------------------------------------------------------------------------------- CPU: model creation
def _cfg(kind, width, heads, t_width=0, t_heads=0, img=(224, 14, 3), sub_ctx=0):
    from jimm_b200 import _lib

    cfg = _lib.Config()
    cfg.kind, cfg.pooling, cfg.compute_dtype = kind, 0, 1
    cfg.img_size, cfg.patch, cfg.in_ch = img
    cfg.v_width, cfg.v_heads, cfg.v_layers, cfg.v_mlp = width, heads, 2, 4 * width
    cfg.ctx_len, cfg.vocab, cfg.t_width, cfg.t_heads, cfg.t_layers, cfg.t_mlp = (sub_ctx or 64), 32000, t_width, t_heads, 2, 4 * t_width
    return cfg


def _create(lib, cfg):
    h = ctypes.c_void_p()
    rc = lib.jimm_model_create(ctypes.byref(cfg), 0, ctypes.byref(h))
    if rc == 0:
        lib.jimm_model_destroy(h)
    return rc, lib.jimm_last_error().decode()


ACCEPTED = {
    "so400m_siglip": (2, 1152, 18, 1152, 16),  # vision 1152 / 18 = 64, text 1152 / 16 = 72
    "mnist_vit": (0, 512, 32, 0, 0, (28, 7, 1)),  # 16
    "encoder_d80": (4, 1280, 16, 0, 0),  # 80
    "map_head_d72": (5, 1152, 16, 0, 0),  # 72
}


@pytest.mark.parametrize("name", list(ACCEPTED))
def test_create_accepts_head_widths(lib, name):
    """The configurations get past validation: on a host without a GPU they fail at the device check, not with JIMM_EINVAL."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: the GPU tests below create these models")
    rc, msg = _create(lib, _cfg(*ACCEPTED[name]))
    assert rc == -2, (rc, msg)
    assert "no CPU fallback" in msg or "CUDA" in msg, msg


REFUSED = {
    "vision_d12": ((0, 96, 8, 0, 0), "vision head_dim: width 96 / heads 8 = 12"),
    "vision_d136": ((0, 272, 2, 0, 0), "vision head_dim: width 272 / heads 2 = 136"),
    "vision_indivisible": ((0, 200, 3, 0, 0), "vision head_dim: width 200 / heads 3"),
    "text_d12": ((2, 128, 2, 96, 8), "text head_dim: width 96 / heads 8 = 12"),
    "text_indivisible": ((1, 128, 2, 200, 3), "text head_dim: width 200 / heads 3"),
    "encoder_d136": ((4, 272, 2, 0, 0), "head_dim: width 272 / heads 2 = 136"),
    "map_head_d4": ((5, 32, 8, 0, 0), "head_dim: width 32 / heads 8 = 4"),
}


@pytest.mark.parametrize("name", list(REFUSED))
def test_create_refuses_head_widths(lib, name):
    (kind, w, h, tw, th), text = REFUSED[name]
    rc, msg = _create(lib, _cfg(kind, w, h, tw, th))
    assert rc == -1, (rc, msg)
    assert text in msg and "multiples of 8 from 8 to 128" in msg, msg


# ---------------------------------------------------------------------------------------------------------------- CPU: oracle vs HF
def test_oracle_matches_hf_vit_d80():
    import check_vs_hf as H

    r = H.check_vit(H.tiny_vit_config(hidden_size=160, num_attention_heads=2, intermediate_size=320))
    assert r["hf_rel"] < 1e-9, r
    assert r["jimm_abs"] < 0.05 and r["argmax_equal"], r


def test_oracle_matches_hf_siglip_text_d72():
    """Both towers 144 wide with two heads: d = 72 in the text tower and (144 // 64 = 2 heads) in the vision tower."""
    import check_vs_hf as H
    from transformers import SiglipConfig

    cfg = SiglipConfig(
        text_config=dict(hidden_size=144, num_attention_heads=2, num_hidden_layers=2, intermediate_size=576, max_position_embeddings=16,
                         vocab_size=100, projection_size=144),
        vision_config=dict(hidden_size=144, num_attention_heads=2, num_hidden_layers=2, intermediate_size=576, image_size=32, patch_size=8),
    )
    r = H.check_siglip(cfg)
    assert r["img_rel"] < 1e-9 and r["txt_rel"] < 1e-9 and r["logits_rel"] < 1e-9, r


# ---------------------------------------------------------------------------------------------------------------- GPU: attention kernel
def _qkv(B, S, H, d, dtype, seed):
    """Odd heads hold values 6x larger than even ones: a padded column that is not zero-filled reads the next head's (or for the last
    q head, the first k head's) values into Q K^T."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B * S, 3, H, d, generator=g)
    x[:, :, 1::2] *= 6.0
    x[:, :, 0::2] *= 1.5
    return x.reshape(B * S, 3 * H * d).to(DEV).to(dtype)


def attention_hd(lib, qkv, out, out_code, B, S, H, d, causal, reverse=0):
    check(lib, lib.jimm_k_attention_hd(ptr(qkv), CODE[qkv.dtype], ptr(out), out_code, B, S, H, d, causal, reverse, stream()))


OUT_TYPES = {torch.float16: [(torch.float16, F16), (torch.float32, TF32)], torch.bfloat16: [(torch.bfloat16, BF16)]}
HEAD_DIMS = [8, 16, 32, 40, 72, 80, 96, 128]


def _run_all_outputs(lib, qkv, B, S, H, d, causal, io):
    """fp32 forward output; every other output type and the reverse walk bit for bit against it; rows past B * S untouched."""
    D = H * d
    f32 = torch.empty(B * S, D, device=DEV)
    attention_hd(lib, qkv, f32, F32, B, S, H, d, causal)
    for dt, code in [(torch.float32, F32)] + OUT_TYPES[io]:
        want = f32 if code == F32 else _rna_tf32(f32) if code == TF32 else f32.to(dt)
        for reverse in (0, 1):
            buf = torch.full((B * S + 65, D), SENTINEL, dtype=dt, device=DEV)
            attention_hd(lib, qkv, buf, code, B, S, H, d, causal, reverse)
            torch.cuda.synchronize()
            assert torch.equal(buf[: B * S], want), (d, code, reverse)
            assert bool((buf[B * S:].float() == SENTINEL).all()), (d, code, reverse, "rows past B * S written")
    return f32


@pytest.mark.gpu
@pytest.mark.parametrize("io", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("S", [1, 17, 64, 77, 197, 257, 577])
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_attention_hd(lib, d, S, causal, io):
    B, H = 3, 3
    qkv = _qkv(B, S, H, d, io, seed=1000 * d + S + 7 * causal)
    f32 = _run_all_outputs(lib, qkv, B, S, H, d, causal, io)
    case = f"attention d={d} B={B} S={S} H={H} causal={causal}"
    check_parity(case, "out", io, "exact fp64", f32, _attn_ref(qkv, B, S, H, d, causal), EXACT_TOL[io])
    _check_tile_faithful(case, f32, qkv, B, S, H, d, causal)


@pytest.mark.gpu
@pytest.mark.parametrize("io", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("d,H,S,causal", [(80, 16, 257, 0), (72, 16, 64, 0), (16, 32, 17, 0), (128, 8, 577, 0), (72, 16, 77, 1),
                                          (40, 12, 197, 0), (96, 12, 197, 1)])
def test_attention_hd_more_ctas_than_sms(lib, d, H, S, causal, io):
    """At least two CTAs per SM at the models' shapes (ViT-H/14 at 224: S = 257, 16 heads of 80; so400m text: 64 tokens, 16 heads of
    72; the MNIST ViT: 17 tokens, 32 heads of 16)."""
    B = max(2, math.ceil(2 * SMS / (math.ceil(S / 64) * H)))
    qkv = _qkv(B, S, H, d, io, seed=d * S + H)
    f32 = _run_all_outputs(lib, qkv, B, S, H, d, causal, io)
    case = f"attention d={d} B={B} S={S} H={H} causal={causal}"
    check_parity(case, "out", io, "exact fp64", f32, _attn_ref(qkv, B, S, H, d, causal), EXACT_TOL[io])
    _check_tile_faithful(case, f32, qkv, B, S, H, d, causal)


@pytest.mark.gpu
@pytest.mark.parametrize("io", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("H", [12, 16])
@pytest.mark.parametrize("S,causal", [(50, 0), (197, 0), (77, 1), (256, 0), (576, 0), (577, 0), (1024, 0)])
def test_hd64_is_attention_ex(lib, S, causal, H, io):
    """d = 64 through jimm_k_attention_hd gives the bits of jimm_k_attention_ex, at the shapes of test_attention_as_run."""
    B = max(2, math.ceil(2 * SMS / (math.ceil(S / 64) * H)))
    D = H * 64
    g = torch.Generator(device="cpu").manual_seed(S + H)
    qkv = (torch.randn(B * S, 3 * D, generator=g) * 1.5).to(DEV).to(io)
    for dt, code in [(torch.float32, F32)] + OUT_TYPES[io]:
        for reverse in (0, 1):
            a = torch.full((B * S, D), SENTINEL, dtype=dt, device=DEV)
            b = torch.full((B * S, D), SENTINEL, dtype=dt, device=DEV)
            attention_hd(lib, qkv, a, code, B, S, H, 64, causal, reverse)
            check(lib, lib.jimm_k_attention_ex(ptr(qkv), CODE[io], ptr(b), code, B, S, H, causal, reverse, stream()))
            torch.cuda.synchronize()
            assert torch.equal(a, b), (code, reverse)


@pytest.mark.gpu
def test_attention_hd_rejects_bad_widths(lib):
    qkv = torch.zeros(4, 3 * 2 * 12, dtype=torch.float16, device=DEV)
    out = torch.zeros(4, 2 * 12, dtype=torch.float16, device=DEV)
    for d in (0, 4, 12, 136):
        assert lib.jimm_k_attention_hd(ptr(qkv), F16, ptr(out), F16, 1, 4, 2, d, 0, 0, stream()) == -1
        assert b"head_dim" in lib.jimm_last_error()
        assert lib.jimm_k_map_attention_hd(ptr(out), ptr(qkv), F16, ptr(out), F16, 1, 4, 2, d, stream()) == -1


# ---------------------------------------------------------------------------------------------------------------- GPU: MAP attention
@pytest.mark.gpu
@pytest.mark.parametrize("S", [17, 256, 729])
@pytest.mark.parametrize("d", [16, 72, 80, 128])
def test_map_attention_hd(lib, d, S):
    """fp32 output against fp64; 16-bit and tf32 outputs are the fp32 output rounded, bit for bit; rows past B untouched."""
    H, B = 16, 40
    D = H * d
    g = torch.Generator(device="cpu").manual_seed(d * S)
    q = (torch.randn(D, generator=g) * 0.5).to(DEV)
    kv = torch.randn(B * S, 2, H, d, generator=g)
    kv[:, :, 1::2] *= 6.0  # neighbouring heads large, as above
    kv = kv.reshape(B * S, 2 * D).to(DEV)
    for io, outs in ((torch.float16, [(torch.float16, F16), (torch.float32, TF32)]), (torch.bfloat16, [(torch.bfloat16, BF16)])):
        kvt = kv.to(io)
        f32 = torch.empty(B, D, device=DEV)
        check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kvt), CODE[io], ptr(f32), F32, B, S, H, d, stream()))
        k, v = kvt.double().reshape(B, S, 2, H, d).permute(2, 0, 3, 1, 4)
        w = torch.softmax((q.double().reshape(1, H, 1, d) / math.sqrt(d)) @ k.transpose(-1, -2), -1)
        ref = (w @ v).reshape(B, D)
        check_parity(f"MAP attention d={d} B={B} S={S} H={H}", "pooled", io, "exact fp64", f32, ref, 2e-5)
        for dt, code in outs:
            out = torch.full((B + 3, D), SENTINEL, dtype=dt, device=DEV)
            check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kvt), CODE[io], ptr(out), code, B, S, H, d, stream()))
            torch.cuda.synchronize()
            assert torch.equal(out[:B], _rna_tf32(f32) if code == TF32 else f32.to(dt)), (io, code)
            assert bool((out[B:].float() == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------------- GPU: models
def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


@pytest.mark.gpu
def test_mnist_vit_d16():
    """The model of the reference's examples/vit_training.py (28 x 28 x 1, patch 7, 512 wide, 32 heads of 16), inference."""
    from jimm_b200.models import VisionTransformer

    oc = O.ViTCfg(num_classes=10, in_channels=1, img_size=28, patch_size=7, num_layers=2, num_heads=32, mlp_dim=2048, hidden_size=512)
    p = O.random_vit_params(oc, seed=71)
    img = O.synthetic_images(6, 28, C=1)
    with torch.no_grad():
        ref = O.vit_forward(p, oc, img)
        ref_same = O.vit_forward(p, oc, img, O.Semantics(operand_round="bf16"))
    case = "MNIST ViT 2x512, 32 heads of 16"
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        m = _set(VisionTransformer(num_classes=10, in_channels=1, img_size=28, patch_size=7, num_layers=2, num_heads=32, mlp_dim=2048,
                                   hidden_size=512, dtype=dtype), p).eval()
        out = m(img.cuda())
        assert out.shape == (6, 10)
        if dtype == torch.bfloat16:
            check_parity(case, "logits", dtype, "same-rounding", out, ref_same, BF16_VS_SAME)
            check_parity(case, "logits", dtype, "fp32", out, ref, BF16_VS_FP32)
        else:
            check_parity(case, "logits", dtype, "fp32", out, ref, TOL)


SO400M = (224, 1152, 14, 64, 32000, 1152, 16)  # image_resolution, vision_width, patch, context_length, vocab, text width, text heads


def _so400m(layers):
    r, vw, ps, ctx, voc, tw, th = SO400M
    return O.DualCfg(r, layers, vw, ps, ctx, voc, tw, th, layers)


def _so400m_model(layers, dtype):
    from jimm_b200.models import SigLIP

    r, vw, ps, ctx, voc, tw, th = SO400M
    return SigLIP(image_resolution=r, vision_layers=layers, vision_width=vw, vision_patch_size=ps, context_length=ctx, vocab_size=voc,
                  transformer_width=tw, transformer_heads=th, transformer_layers=layers, dtype=dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_siglip_so400m_notebook_reduced_depth(dtype):
    """The reference's examples/siglip_inference.ipynb model (vision 1152 / 18 heads of 64, text 1152 / 16 heads of 72) at 2+2 layers."""
    cfg = _so400m(2)
    p = O.random_dual_params(cfg, "siglip", seed=73)
    img, txt = O.synthetic_images(2, 224, seed=3), O.synthetic_tokens(3, 64, 32000, "siglip", seed=4)
    sem = O.Semantics(operand_round="bf16") if dtype == torch.bfloat16 else O.JIMM
    with torch.no_grad():
        ref_i, ref_t = O.siglip_encode_image(p, cfg, img), O.siglip_encode_text(p, cfg, txt)
        ref = O.siglip_forward(p, cfg, img, txt)
        if dtype == torch.bfloat16:
            same_i, same_t = O.siglip_encode_image(p, cfg, img, sem), O.siglip_encode_text(p, cfg, txt, sem)
            same = O.siglip_forward(p, cfg, img, txt, sem)
    m = _set(_so400m_model(2, dtype), p)
    emb_i, emb_t, out = m.encode_image(img.cuda()), m.encode_text(txt.cuda()), m(img.cuda(), txt.cuda())
    assert out.shape == (2, 3)
    case = "SigLIP so400m notebook, 2+2 layers"
    if dtype == torch.float16:
        check_parity(case, "image_embeds", dtype, "fp32", emb_i, ref_i, TOL)
        check_parity(case, "text_embeds", dtype, "fp32", emb_t, ref_t, TOL)
        check_parity(case, "logits", dtype, "fp32", out, ref, LOGITS_TOL)
    else:
        for what, a, s, r in (("image_embeds", emb_i, same_i, ref_i), ("text_embeds", emb_t, same_t, ref_t), ("logits", out, same, ref)):
            check_parity(case, what, dtype, "same-rounding", a, s, BF16_VS_SAME)
            check_parity(case, what, dtype, "fp32", a, r, BF16_VS_FP32)


@pytest.mark.gpu
def test_siglip_so400m_notebook_full_depth():
    """The same model at its full 27+27 layers, fp16, two images and two texts."""
    cfg = _so400m(27)
    p = O.random_dual_params(cfg, "siglip", seed=79)
    img, txt = O.synthetic_images(2, 224, seed=5), O.synthetic_tokens(2, 64, 32000, "siglip", seed=6)
    with torch.no_grad():
        ref_i, ref_t = O.siglip_encode_image(p, cfg, img), O.siglip_encode_text(p, cfg, txt)
        ref = O.contrastive_logits(ref_i, ref_t, p["logit_scale"], p["logit_bias"])
    m = _set(_so400m_model(27, torch.float16), p)
    case = "SigLIP so400m notebook, 27+27 layers"
    check_parity(case, "image_embeds", torch.float16, "fp32", m.encode_image(img.cuda()), ref_i, TOL)
    check_parity(case, "text_embeds", torch.float16, "fp32", m.encode_text(txt.cuda()), ref_t, TOL)
    check_parity(case, "logits", torch.float16, "fp32", m(img.cuda(), txt.cuda()), ref, LOGITS_TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("pooling", ["CLS", "MAP"])
def test_vit_h14_tower(pooling):
    """A ViT-H/14-shaped VisionTransformerBase (1280 wide, 16 heads of 80, patch 14 at 224: 256 or 257 tokens), 2 layers; MAP pooling
    runs the MAP head at d = 80."""
    from jimm_b200.common.vit import VisionTransformerBase

    kw = dict(img_size=224, patch_size=14, in_channels=3, hidden_size=1280, num_layers=2, num_heads=16, mlp_dim=5120, pooling_type=pooling,
              layernorm_epsilon=1e-6)
    t = O.TowerCfg(**kw)
    p = O.random_tower_params(t, seed=83)
    img = O.synthetic_images(3, 224, seed=8)
    with torch.no_grad():
        ref = O.vision_tower(p, "", img, t)
    for dtype in (torch.float16, torch.float32):
        m = _set(VisionTransformerBase(**kw, dtype=dtype), p)
        out = m(img.cuda())
        assert out.shape == (3, 1280)
        check_parity(f"ViT-H/14 tower 2x1280, {pooling}", "pooled", dtype, "fp32", out, ref, TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_bare_transformer_d72(causal):
    """Transformer.__call__ (jimm_encoder_forward) at 144 wide, 2 heads of 72, causal and not."""
    from jimm_b200.common.transformer import Transformer

    D, M, H, L, T = 144, 576, 2, 2, 40
    g = torch.Generator().manual_seed(89)
    p = {}
    O._rand_blocks(p, g, "", L, D, H, M)
    p = O.cast_params(p, torch.float32)
    mask = torch.tril(torch.ones(T, T)) if causal else None
    x = torch.randn(5, 33, D, generator=g)
    with torch.no_grad():
        ref = O.transformer(p, "", x, L, H, False, mask, 1e-5)
    for dtype in (torch.float16, torch.float32):
        t = _set(Transformer(D, M, L, H, layernorm_epsilon=1e-5, attn_mask=mask, dtype=dtype), p)
        check_parity(f"bare Transformer 2x144, heads of 72, causal={causal}", "activations", dtype, "fp32", t(x.cuda()), ref, TOL)


@pytest.mark.gpu
def test_bare_map_head_d72():
    """MultiHeadAttentionPoolingHead.__call__ (jimm_map_head_forward) at 1152 wide, 16 heads of 72."""
    from jimm_b200.common.vit import MultiHeadAttentionPoolingHead

    D, H = 1152, 16
    t = O.TowerCfg(32, 8, 3, D, 0, H, 4 * D, "MAP", layernorm_epsilon=1e-6)
    p = {k[len("MAPHead."):]: v for k, v in O.random_tower_params(t, seed=97).items() if k.startswith("MAPHead.")}
    x = torch.randn(6, 64, D, generator=torch.Generator().manual_seed(98))
    with torch.no_grad():
        ref = O.map_head(p, "", x, H, 1e-6)
    for dtype in (torch.float16, torch.float32):
        h = _set(MultiHeadAttentionPoolingHead(D, 4 * D, H, 1e-6, dtype=dtype), p)
        out = h(x.cuda())
        assert out.shape == (6, D)
        check_parity("bare MAP head 1152, heads of 72", "pooled", dtype, "fp32", out, ref, TOL)


@pytest.mark.gpu
def test_from_pretrained_hf_vit_d80(tmp_path):
    """VisionTransformer.from_pretrained on a random-init HF ViT with 2 heads of 80, saved with its config.json: the heads come from
    num_attention_heads, and the model matches the oracle on hf_to_flax_vit of the same weights."""
    import check_vs_hf as H
    from transformers import ViTForImageClassification

    from jimm_b200.models import VisionTransformer

    torch.manual_seed(101)
    cfg = H.tiny_vit_config(hidden_size=160, num_attention_heads=2, intermediate_size=640)
    hf = H.perturb_(ViTForImageClassification(cfg)).eval()
    hf.save_pretrained(str(tmp_path), safe_serialization=True)
    sd = {k: v.detach() for k, v in hf.state_dict().items()}
    oc = O.ViTCfg(num_classes=cfg.num_labels, img_size=cfg.image_size, patch_size=cfg.patch_size, num_layers=cfg.num_hidden_layers,
                  num_heads=2, mlp_dim=cfg.intermediate_size, hidden_size=160)
    p = O.hf_to_flax_vit(sd, oc.num_layers, 2)
    img = O.synthetic_images(4, cfg.image_size, seed=9)
    with torch.no_grad():
        ref = O.vit_forward(p, oc, img)
    for dtype in (torch.float16, torch.float32):
        m = VisionTransformer.from_pretrained(str(tmp_path / "model.safetensors"), dtype=dtype)
        out = m(img.cuda())
        assert out.shape == (4, cfg.num_labels)
        check_parity("from_pretrained HF ViT 2x160, heads of 80", "logits", dtype, "fp32", out, ref, TOL)
