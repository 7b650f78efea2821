"""GPU: interpolate_pos_encoding -- the vision towers on images of any size, the position table resampled bicubically to the patch
grid (jimm_k_tokens_init_interp, jimm_*_hw) -- against the interpolating CPU oracle (tests/interp_oracle.py)."""

import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import fp8_oracle as F8
import interp_oracle as I
import jimm_oracle as O
from gpu_util import check, check_parity, ptr, rel_err, stream

pytestmark = pytest.mark.gpu
TOL = 1e-3
BF16_VS_SAME = 8e-3
LOGITS_TOL = 2e-3  # contrastive logits amplify the embedding error by exp(logit_scale), as in test_parity_gpu.py


def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


# ------------------------------------------------------------------ kernel
@pytest.mark.parametrize("D", [64, 768, 1024])
@pytest.mark.parametrize("cls", [True, False])
@pytest.mark.parametrize("g,gh,gw", [(14, 24, 24), (14, 7, 7), (14, 18, 10), (16, 32, 32), (1, 3, 5), (14, 14, 14)])
def test_tokens_init_interp_kernel(lib, g, gh, gw, cls, D):
    off, B = int(cls), 3
    gen = torch.Generator().manual_seed(g * 7 + gh + D)
    pos = torch.randn((off + g * g, D), generator=gen) * 0.2
    c = torch.randn(D, generator=gen) if cls else None
    x = torch.full((B, off + gh * gw, D), float("nan"), device="cuda")
    cd, pd = (c.cuda() if cls else None), pos.cuda()  # held until the kernel has run
    check(lib, lib.jimm_k_tokens_init_interp(ptr(cd), ptr(pd), g, D, ptr(x), B, gh, gw, stream()))
    torch.cuda.synchronize()
    ref = I.resample_pos(pos[None], g, gh, gw, cls)[0].clone()
    if cls:
        ref[0] += c
    out = x.cpu()
    for b in range(B):
        assert torch.equal(out[b], out[0])
    if (gh, gw) == (g, g):  # the trained grid: the bytes tokens_init writes (pos, cls + pos[0])
        assert torch.equal(out[0], ref)
    else:
        err = float((out[0] - ref).abs().max())
        assert err <= 1e-6 * float(pos.abs().max()), err


# ------------------------------------------------------------------ models against the interpolating oracle
@pytest.fixture(scope="module")
def vitb16():
    cfg = O.ViTCfg()
    return cfg, O.random_vit_params(cfg, seed=0)


@pytest.mark.parametrize("hw", [(384, 384), (288, 160)])
def test_vit_b16(vitb16, hw):
    from jimm_b200.models import VisionTransformer

    cfg, p = vitb16
    img = O.synthetic_images(4, max(hw))[:, : hw[0], : hw[1]].contiguous()
    with torch.no_grad():
        ref = I.vit_forward(p, cfg, img, interpolate_pos_encoding=True)
        ref_bf = I.vit_forward(p, cfg, img, O.Semantics(operand_round="bf16"), interpolate_pos_encoding=True)
    case = f"ViT-B/16@{hw[0]}x{hw[1]} B=4 interpolate_pos_encoding"
    for dtype in (torch.float16, torch.float32, torch.bfloat16):
        m = _set(VisionTransformer(dtype=dtype), p).eval()
        out = m(img.cuda(), interpolate_pos_encoding=True)
        if dtype == torch.bfloat16:
            check_parity(case, "logits", dtype, "same-rounding", out, ref_bf, BF16_VS_SAME)
            continue
        check_parity(case, "logits", dtype, "fp32", out, ref, TOL)
        assert torch.equal(out.argmax(-1).cpu(), ref.argmax(-1))


def test_patch14_tower_280():
    """Patch 14 (zero-padded patch-GEMM K, 588 -> 592) at 280 x 280: a 20 x 20 grid from a 16 x 16 table."""
    from jimm_b200.common.vit import VisionTransformerBase

    t = O.TowerCfg(img_size=224, patch_size=14, in_channels=3, hidden_size=256, num_layers=2, num_heads=4, mlp_dim=1024, pooling_type="CLS",
                   use_quick_gelu=True, use_pre_norm=True, use_patch_bias=False, layernorm_epsilon=1e-5)
    p = O.random_tower_params(t, seed=31)
    img = O.synthetic_images(3, 280)
    with torch.no_grad():
        ref = I.vision_tower(p, "", img, t, interpolate_pos_encoding=True)
    for dtype in (torch.float16, torch.float32):
        m = _set(VisionTransformerBase(img_size=224, patch_size=14, in_channels=3, hidden_size=256, num_layers=2, num_heads=4, mlp_dim=1024,
                                       pooling_type="CLS", use_quick_gelu=True, use_pre_norm=True, use_patch_bias=False,
                                       layernorm_epsilon=1e-5, dtype=dtype), p)
        check_parity("tower patch 14 @280 interpolate_pos_encoding", "pooled", dtype, "fp32", m(img.cuda(), interpolate_pos_encoding=True), ref, TOL)


@pytest.fixture(scope="module")
def siglip_b16():
    cfg = O.DualCfg(256, 2, 768, 16, 64, 1000, 768, 12, 2)  # SigLIP-B/16 @256 shapes, 2 layers per tower
    return cfg, O.random_dual_params(cfg, "siglip", seed=9)


SAME_BF16 = O.Semantics(operand_round="bf16")


def _dual_dtypes(case, make, img, txt, enc_ref, enc_same, logits_ref, argmax=False):
    """A dual model in fp16, fp32 (tf32) and bf16: embeddings and logits against the fp32 oracle, bf16 embeddings against the oracle
    with bf16 operand rounding."""
    for dtype in (torch.float16, torch.float32, torch.bfloat16):
        m = make(dtype)
        ie = m.encode_image(img.cuda(), interpolate_pos_encoding=True)
        if dtype == torch.bfloat16:
            check_parity(case, "image_embeds", dtype, "same-rounding", ie, enc_same, BF16_VS_SAME)
            continue
        check_parity(case, "image_embeds", dtype, "fp32", ie, enc_ref, TOL)
        out = m(img.cuda(), txt.cuda(), interpolate_pos_encoding=True)
        check_parity(case, "logits", dtype, "fp32", out, logits_ref, LOGITS_TOL)
        if argmax:
            assert torch.equal(out.argmax(-1).cpu(), logits_ref.argmax(-1))


@pytest.mark.parametrize("size", [384, 224])
def test_siglip_b16(siglip_b16, size):
    from jimm_b200.models import SigLIP

    cfg, p = siglip_b16
    img, txt = O.synthetic_images(3, size), O.synthetic_tokens(4, 64, 1000, "siglip")
    with torch.no_grad():
        ref_i = I.siglip_encode_image(p, cfg, img, interpolate_pos_encoding=True)
        same_i = I.siglip_encode_image(p, cfg, img, sem=SAME_BF16, interpolate_pos_encoding=True)
        ref = I.siglip_forward(p, cfg, img, txt, interpolate_pos_encoding=True)
    _dual_dtypes(f"SigLIP-B/16 shapes @{size} (MAP head), 2+2 layers, interpolate_pos_encoding",
                 lambda dt: _set(SigLIP(256, 2, 768, 16, 64, 1000, 768, 12, 2, dtype=dt), p), img, txt, ref_i, same_i, ref)


def test_clip_b32_336():
    """336 / 32 = 10.5: the grid floors to 10 x 10 from the trained 7 x 7."""
    from jimm_b200.models import CLIP

    cfg = O.DualCfg(224, 2, 768, 32, 77, 1000, 512, 8, 2)
    p = O.random_dual_params(cfg, "clip", seed=7)
    img, txt = O.synthetic_images(3, 336), O.synthetic_tokens(4, 77, 1000, "clip")
    with torch.no_grad():
        ref_i = I.clip_encode_image(p, cfg, img, interpolate_pos_encoding=True)
        same_i = I.clip_encode_image(p, cfg, img, sem=SAME_BF16, interpolate_pos_encoding=True)
        ref = I.clip_forward(p, cfg, img, txt, interpolate_pos_encoding=True)
    _dual_dtypes("CLIP-B/32 shapes @336, 2+2 layers, interpolate_pos_encoding",
                 lambda dt: _set(CLIP(224, 2, 768, 32, 77, 1000, 512, 8, 2, dtype=dt), p), img, txt, ref_i, same_i, ref, argmax=True)


@pytest.mark.parametrize("kind", ["vit", "clip", "siglip"])
def test_golden_tiny_40x48(golden_dir, kind):
    import check_vs_hf as H
    import transformers
    from safetensors.torch import load_file

    from jimm_b200.models import CLIP, SigLIP, VisionTransformer

    d = os.path.join(golden_dir, f"tiny_{kind}")
    path = os.path.join(d, "model.safetensors")
    sd = load_file(path)
    with open(os.path.join(d, "config.json")) as f:
        hc = json.load(f)
    img = (torch.rand((3, 40, 48, 3), generator=torch.Generator().manual_seed(40)) * 2 - 1)
    if kind == "vit":
        c = transformers.ViTConfig(**hc)
        oc = O.ViTCfg(num_classes=c.num_labels, img_size=c.image_size, patch_size=c.patch_size, num_layers=c.num_hidden_layers,
                      num_heads=c.num_attention_heads, mlp_dim=c.intermediate_size, hidden_size=c.hidden_size)
        p = O.hf_to_flax_vit(sd, oc.num_layers, oc.num_heads)
        run_ref = lambda sem: I.vit_forward(p, oc, img, sem, interpolate_pos_encoding=True)
        run = lambda dt: VisionTransformer.from_pretrained(path, dtype=dt)(img.cuda(), interpolate_pos_encoding=True)
    else:
        c = (transformers.CLIPConfig if kind == "clip" else transformers.SiglipConfig)(**hc)
        oc = H._dual_cfg(c)
        fn = I.clip_encode_image if kind == "clip" else I.siglip_encode_image
        p = (O.hf_to_flax_clip if kind == "clip" else O.hf_to_flax_siglip)(sd, oc)
        run_ref = lambda sem: fn(p, oc, img, sem=sem, interpolate_pos_encoding=True)
        cls = CLIP if kind == "clip" else SigLIP
        run = lambda dt: cls.from_pretrained(path, dtype=dt).encode_image(img.cuda(), interpolate_pos_encoding=True)
    with torch.no_grad():
        ref, same = run_ref(O.JIMM), run_ref(SAME_BF16)
    case, what = f"golden tiny_{kind} @40x48 interpolate_pos_encoding", "logits" if kind == "vit" else "image_embeds"
    for dtype in (torch.float16, torch.float32, torch.bfloat16):
        out = run(dtype)
        if dtype == torch.bfloat16:
            check_parity(case, what, dtype, "same-rounding", out, same, BF16_VS_SAME)
            continue
        check_parity(case, what, dtype, "fp32", out, ref, TOL)
        if kind == "vit":
            assert torch.equal(out.argmax(-1).cpu(), ref.argmax(-1))


# ------------------------------------------------------------------ same bits where nothing should change
def _small_vit(dtype=torch.float16, seed=1):
    from jimm_b200.models import VisionTransformer

    cfg = O.ViTCfg(num_classes=12, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=1024, hidden_size=256)
    p = O.random_vit_params(cfg, seed=seed)
    mk = lambda: _set(VisionTransformer(num_classes=12, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=1024,
                                        hidden_size=256, dtype=dtype), p).eval()
    return cfg, p, mk


def test_native_size_is_the_default_call(vitb16):
    from jimm_b200.models import VisionTransformer

    cfg, p = vitb16
    m = _set(VisionTransformer(dtype=torch.float16), p).eval()
    img = O.synthetic_images(4, 224).cuda()
    assert torch.equal(m(img, interpolate_pos_encoding=True), m(img))


def test_graph_replay_never_crosses_grids(vitb16, monkeypatch):
    """ViT-B/16 at 224 (native), 384 and 288 x 160 interleaved on one handle, at a batch in the CUDA-graph range: every call gives
    the bits of a handle without graphs (native calls replay their graph, off-grid calls never do)."""
    from jimm_b200.models import VisionTransformer

    cfg, p = vitb16
    sizes = [(224, 224), (384, 384), (288, 160)]
    imgs = {hw: O.synthetic_images(4, max(hw), seed=hw[0])[:, : hw[0], : hw[1]].contiguous().cuda() for hw in sizes}
    monkeypatch.setenv("JIMM_GRAPH_MAX_BATCH", "0")
    plain = _set(VisionTransformer(dtype=torch.float16), p).eval()
    want = {hw: plain(x, interpolate_pos_encoding=True) for hw, x in imgs.items()}
    monkeypatch.delenv("JIMM_GRAPH_MAX_BATCH")
    m = _set(VisionTransformer(dtype=torch.float16), p).eval()
    for _ in range(4):
        for hw, x in imgs.items():
            assert torch.equal(m(x, interpolate_pos_encoding=True), want[hw]), hw


# ------------------------------------------------------------------ chunking and the token budget
def test_chunking_and_budget(vitb16):
    from jimm_b200.models import VisionTransformer

    cfg, p = vitb16
    img = O.synthetic_images(20, 384)
    with torch.no_grad():
        ref = I.vit_forward(p, cfg, img, interpolate_pos_encoding=True)
    # max_batch 8 at 197 tokens: 1576 tokens, two 577-token images per chunk
    a = _set(VisionTransformer(dtype=torch.float16), p).eval().set_max_batch(8)(img.cuda(), interpolate_pos_encoding=True)
    b = _set(VisionTransformer(dtype=torch.float16), p).eval().set_max_batch(8).set_max_image_size(384, 384)(img.cuda(), interpolate_pos_encoding=True)
    check_parity("ViT-B/16@384 B=20, 2 images per chunk", "logits", torch.float16, "fp32", a, ref, TOL)
    check_parity("ViT-B/16@384 B=20, 8 images per chunk", "logits", torch.float16, "fp32", b, ref, TOL)
    assert rel_err(a, b) < 1e-3


def test_one_image_over_budget():
    from jimm_b200 import _lib

    cfg, p, mk = _small_vit()
    m = mk().set_max_batch(1)  # 17 tokens in all
    x = O.synthetic_images(2, 160).cuda()  # 101 tokens per image
    n = m.native()
    assert n.images_per_call(160, 160) == 0 and n.images_per_call(64, 64) == 1
    lib = _lib.load()
    out = torch.empty((2, 12), device="cuda")
    rc = lib.jimm_vit_forward_hw(n.handle, C.c_void_p(x.data_ptr()), _lib.F32, 2, 160, 160, C.c_void_p(out.data_ptr()), stream())
    msg = lib.jimm_last_error().decode()
    assert rc == -1 and "101 tokens" in msg and "jimm_model_set_max_tokens" in msg, msg
    # the Python classes rebuild the handle with a budget that holds one such image ...
    got = m(x, interpolate_pos_encoding=True)
    assert m.native() is not n and m.native().images_per_call(160, 160) == 1
    with torch.no_grad():
        check_parity("small ViT @160 after a budget rebuild", "logits", torch.float16, "fp32", got,
                     I.vit_forward(p, cfg, x.cpu(), interpolate_pos_encoding=True), TOL)
    # ... and keep it when a later rebuild (here a larger batch bound) replaces the handle
    m.set_max_batch(2)
    n2 = m.native()
    assert n2.images_per_call(160, 160) == 2
    assert rel_err(m(x, interpolate_pos_encoding=True), got) < 1e-3 and m.native() is n2  # no further rebuild


def test_rebuild_for_padded_patch_rows():
    """A CLS tower whose patch count (64) is a multiple of 32 and whose MLP is narrower than a patch row (64 < 16*16*3): a 48 x 688
    image has 3 x 43 = 129 patches and 130 tokens, which the default workspace of 2 x 65 rows holds, but its 160 padded patch rows do
    not fit the 128 the default sized.  The library says so, and the Python class rebuilds rather than failing."""
    from jimm_b200.common.vit import VisionTransformerBase

    t = O.TowerCfg(img_size=128, patch_size=16, in_channels=3, hidden_size=64, num_layers=1, num_heads=1, mlp_dim=64, pooling_type="CLS")
    p = O.random_tower_params(t, seed=13)
    m = _set(VisionTransformerBase(img_size=128, patch_size=16, in_channels=3, hidden_size=64, num_layers=1, num_heads=1, mlp_dim=64,
                                   pooling_type="CLS", dtype=torch.float16), p).set_max_batch(2)
    assert m.native().images_per_call(48, 688) == 0
    x = O.synthetic_images(3, 688)[:, :48].contiguous()
    out = m(x.cuda(), interpolate_pos_encoding=True)
    assert m.native().images_per_call(48, 688) >= 1
    with torch.no_grad():
        check_parity("tower 64-wide @48x688, padded patch rows", "pooled", torch.float16, "fp32", out,
                     I.vision_tower(p, "", x, t, interpolate_pos_encoding=True), TOL)


# ------------------------------------------------------------------ inputs
def test_host_and_numpy_inputs():
    cfg, p, mk = _small_vit()
    m = mk()
    img = O.synthetic_images(3, 96)
    dev = m(img.cuda(), interpolate_pos_encoding=True)
    for x in (img.pin_memory(), img, img.numpy()):
        out = m(x, interpolate_pos_encoding=True)
        assert not out.is_cuda and torch.equal(out, dev.cpu())
    assert torch.equal(m.forward_async(img, interpolate_pos_encoding=True).result(), dev.cpu())


def test_uint8_frames_through_the_front_end():
    from jimm_b200.models import SigLIP
    from jimm_b200.preprocess import ImagePreprocessor

    cfg = O.DualCfg(256, 2, 256, 16, 16, 300, 256, 4, 2)
    p = O.random_dual_params(cfg, "siglip", seed=3)
    m = _set(SigLIP(256, 2, 256, 16, 16, 300, 256, 4, 2, dtype=torch.float16), p)
    pre = ImagePreprocessor.siglip(384)
    m.set_preprocessor(pre)
    frames = torch.randint(0, 256, (2, 300, 420, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5))
    want = m.encode_image(pre(frames, dtype=torch.float16), interpolate_pos_encoding=True)
    assert torch.equal(m.encode_image(frames.cuda(), interpolate_pos_encoding=True), want)
    assert torch.equal(m.encode_image(frames, interpolate_pos_encoding=True), want.cpu())


# ------------------------------------------------------------------ fallback paths and compute modes
@pytest.mark.parametrize("env", [("JIMM_GEMM_IMPL", "simt"), ("JIMM_EPI_MODE_RES", "0")])
def test_fallback_paths(monkeypatch, env):
    cfg, p, mk = _small_vit()
    x = O.synthetic_images(3, 112)[:, :, :80].contiguous().cuda()
    a = mk()(x, interpolate_pos_encoding=True)
    monkeypatch.setenv(*env)
    b = mk()(x, interpolate_pos_encoding=True)
    assert rel_err(b, a) < 1e-3
    with torch.no_grad():
        check_parity(f"small ViT @112x80 {env[0]}={env[1]}", "logits", torch.float16, "fp32", b,
                     I.vit_forward(p, cfg, x.cpu(), interpolate_pos_encoding=True), TOL)


def test_fp8_at_384(vitb16):
    from jimm_b200.models import VisionTransformer

    cfg, p = vitb16
    img = O.synthetic_images(2, 384)
    pd = {k: v.double() for k, v in p.items()}
    with torch.no_grad(), F8.active():
        ref8 = I.vit_forward(pd, cfg, img.double(), F8.FP8, interpolate_pos_encoding=True)
        ref32 = I.vit_forward(pd, cfg, img.double(), interpolate_pos_encoding=True)
    out = _set(VisionTransformer(dtype=torch.float8_e4m3fn), p).eval()(img.cuda(), interpolate_pos_encoding=True)
    check_parity("ViT-B/16@384 B=2 interpolate_pos_encoding", "logits", "float8_e4m3fn", "FP8 oracle", out, ref8,
                 F8_SHARE * rel_err(ref8, ref32))


F8_SHARE = 0.5  # the FP8 model bound of test_fp8_gpu.py (ORACLE_SHARE): half the FP8 oracle's own distance to fp32


# ------------------------------------------------------------------ errors
def test_errors():
    from jimm_b200 import _lib

    cfg, p, mk = _small_vit()
    m = mk()
    with pytest.raises(ValueError, match="expected NHWC images"):
        m(O.synthetic_images(2, 96).cuda())  # the default keyword keeps the native-size check
    with pytest.raises(ValueError, match="smaller than one 16x16 patch"):
        m(O.synthetic_images(2, 64)[:, :12].contiguous().cuda(), interpolate_pos_encoding=True)
    x = torch.zeros((1, 12, 64, 3), device="cuda")
    out = torch.empty((1, 12), device="cuda")
    lib = _lib.load()
    rc = lib.jimm_vit_forward_hw(m.native().handle, C.c_void_p(x.data_ptr()), _lib.F32, 1, 12, 64, C.c_void_p(out.data_ptr()), stream())
    assert rc == -1 and "smaller than one" in lib.jimm_last_error().decode()
