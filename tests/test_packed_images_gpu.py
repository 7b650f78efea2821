"""GPU: lists of images of different sizes in one call -- their tokens packed into one stream (jimm_k_attention_packed,
jimm_k_map_attention_packed, jimm_*_packed, the list inputs of the model classes).  Row i of a packed call must be the bits of the call
on image i alone, and within the 1e-3 bar of the interpolating oracle (tests/interp_oracle.py)."""

import ctypes as C

import numpy as np
import pytest
import torch

import interp_oracle as I
import jimm_oracle as O
from gpu_util import BF16, F16, F32, TORCH, check, check_parity, ptr, stream

pytestmark = pytest.mark.gpu
TOL = 1e-3
TF32 = 3
PAIRS = [(F16, F16), (F16, F32), (F16, TF32), (BF16, BF16), (BF16, F32)]
LENS = [1, 63, 64, 65, 197, 577, 1025, 50]
PAD = 5  # rows after the last sample: outside every sample, they must stay as filled


def _offsets(lens):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return off, torch.from_numpy(off).cuda()


def _out_dtype(code):
    return torch.float32 if code == TF32 else TORCH[code]


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("io,ot", PAIRS)
@pytest.mark.parametrize("hd", [8, 64, 72, 128])
def test_attention_packed_kernel(lib, hd, io, ot, reverse):
    H = 2
    D = H * hd
    off, off_d = _offsets(LENS)
    T = int(off[-1])
    g = torch.Generator().manual_seed(hd * 10 + io * 3 + ot)
    qkv = torch.randn((T + PAD, 3 * D), generator=g).to(TORCH[io]).cuda()
    out = torch.full((T + PAD, D), float("nan"), dtype=_out_dtype(ot), device="cuda")
    check(lib, lib.jimm_k_attention_packed(ptr(qkv), io, ptr(out), ot, ptr(off_d), len(LENS), max(LENS), H, hd, reverse, stream()))
    for b, S in enumerate(LENS):
        o = int(off[b])
        ref = torch.full((S, D), float("nan"), dtype=_out_dtype(ot), device="cuda")
        check(lib, lib.jimm_k_attention_hd(ptr(qkv[o:o + S]), io, ptr(ref), ot, 1, S, H, hd, 0, reverse, stream()))
        assert torch.equal(out[o:o + S], ref), f"sample {b} (S={S})"
    assert torch.isnan(out[T:]).all()


@pytest.mark.parametrize("io,ot", PAIRS)
@pytest.mark.parametrize("hd", [8, 64, 72, 128])
def test_map_attention_packed_kernel(lib, hd, io, ot):
    H = 2
    D = H * hd
    off, off_d = _offsets(LENS)
    T = int(off[-1])
    g = torch.Generator().manual_seed(hd * 10 + io * 3 + ot + 1)
    q = torch.randn(D, generator=g).cuda()
    kv = torch.randn((T + PAD, 2 * D), generator=g).to(TORCH[io]).cuda()
    out = torch.full((len(LENS) + 1, D), float("nan"), dtype=_out_dtype(ot), device="cuda")
    check(lib, lib.jimm_k_map_attention_packed(ptr(q), ptr(kv), io, ptr(out), ot, ptr(off_d), len(LENS), max(LENS), H, hd, stream()))
    for b, S in enumerate(LENS):
        o = int(off[b])
        ref = torch.full((1, D), float("nan"), dtype=_out_dtype(ot), device="cuda")
        check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kv[o:o + S]), io, ptr(ref), ot, 1, S, H, hd, stream()))
        assert torch.equal(out[b:b + 1], ref), f"sample {b} (S={S})"
    assert torch.isnan(out[len(LENS):]).all()


# ------------------------------------------------------------------ models
def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


def _images(sizes, seed, C=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn((h, w, C), generator=g) for h, w in sizes]


# trained size 64 at P = 16: the trained size, larger, smaller, non-square, one patch, trailing pixels (230 x 170 -> 14 x 10 patches) and a
# repeated size
SIZES_P16 = [(64, 64), (96, 80), (32, 48), (16, 16), (230, 170), (48, 112), (96, 80)]
DTYPES = [torch.float16, torch.bfloat16, torch.float32, torch.float8_e4m3fn]


def _vit_small():
    cfg = O.ViTCfg(num_classes=10, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=512, hidden_size=128)
    p = O.random_vit_params(cfg, seed=11)

    def make(dtype=torch.float16):
        from jimm_b200.models import VisionTransformer

        return _set(VisionTransformer(num_classes=10, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=512, hidden_size=128,
                                      dtype=dtype), p).eval()

    return cfg, p, make


def _rows_equal_singles(m, imgs, packed, **kw):
    for i, x in enumerate(imgs):
        one = m(x[None].cuda(), interpolate_pos_encoding=True, **kw)
        assert torch.equal(packed[i:i + 1], one), f"image {i} {tuple(x.shape)}"


def _parity(case, dtype, packed, refs):
    if dtype in (torch.float16, torch.float32):
        check_parity(case, "rows", dtype, "fp32", packed, torch.cat(refs), TOL)


@pytest.mark.parametrize("dtype", DTYPES)
def test_vit_cls_classifier(dtype):
    cfg, p, make = _vit_small()
    imgs = _images(SIZES_P16, 1)
    m = make(dtype)
    packed = m([x.cuda() for x in imgs], interpolate_pos_encoding=True)
    assert packed.is_cuda and packed.shape == (len(imgs), 10)
    _rows_equal_singles(m, imgs, packed)
    with torch.no_grad():
        refs = [I.vit_forward(p, cfg, x[None], interpolate_pos_encoding=True) for x in imgs]
    _parity("small ViT (CLS + classifier) packed list of 7 sizes", dtype, packed, refs)


@pytest.mark.parametrize("dtype", DTYPES)
def test_tower_map(dtype):
    from jimm_b200.common.vit import VisionTransformerBase

    kw = dict(img_size=64, patch_size=8, in_channels=3, hidden_size=256, num_layers=2, num_heads=4, mlp_dim=1024, pooling_type="MAP",
              use_quick_gelu=False, use_pre_norm=False, use_patch_bias=True, layernorm_epsilon=1e-6)
    t = O.TowerCfg(**kw)
    p = O.random_tower_params(t, seed=12)
    sizes = [(64, 64), (80, 96), (24, 40), (8, 8), (115, 85), (40, 56), (80, 96)]
    imgs = _images(sizes, 2)
    m = _set(VisionTransformerBase(**kw, dtype=dtype), p)
    packed = m([x.cuda() for x in imgs], interpolate_pos_encoding=True)
    _rows_equal_singles(m, imgs, packed)
    with torch.no_grad():
        refs = [I.vision_tower(p, "", x[None], t, interpolate_pos_encoding=True) for x in imgs]
    _parity("tower (MAP head) packed list of 7 sizes", dtype, packed, refs)


DUAL = O.DualCfg(64, 2, 128, 16, 16, 100, 128, 4, 2)


@pytest.mark.parametrize("dtype", DTYPES)
def test_clip_encode_image(dtype):
    """CLIP's tower: pre-norm, no patch bias, QuickGELU, visual projection."""
    from jimm_b200.models import CLIP

    p = O.random_dual_params(DUAL, "clip", seed=13)
    imgs = _images(SIZES_P16, 3)
    m = _set(CLIP(64, 2, 128, 16, 16, 100, 128, 4, 2, dtype=dtype), p)
    packed = m.encode_image([x.cuda() for x in imgs], interpolate_pos_encoding=True)
    for i, x in enumerate(imgs):
        assert torch.equal(packed[i:i + 1], m.encode_image(x[None].cuda(), interpolate_pos_encoding=True)), i
    with torch.no_grad():
        refs = [I.clip_encode_image(p, DUAL, x[None], interpolate_pos_encoding=True) for x in imgs]
    _parity("CLIP (pre-norm, QuickGELU) encode_image packed list of 7 sizes", dtype, packed, refs)


@pytest.mark.parametrize("dtype", DTYPES)
def test_siglip_call_with_text(dtype):
    from jimm_b200.models import SigLIP

    p = O.random_dual_params(DUAL, "siglip", seed=14)
    imgs = _images(SIZES_P16, 4)
    txt = O.synthetic_tokens(3, 16, 100, "siglip")
    m = _set(SigLIP(64, 2, 128, 16, 16, 100, 128, 4, 2, dtype=dtype), p)
    packed = m([x.cuda() for x in imgs], txt.cuda(), interpolate_pos_encoding=True)
    assert packed.shape == (len(imgs), 3)
    for i, x in enumerate(imgs):
        assert torch.equal(packed[i:i + 1], m(x[None].cuda(), txt.cuda(), interpolate_pos_encoding=True)), i
    emb = m.encode_image([x.cuda() for x in imgs], interpolate_pos_encoding=True)
    with torch.no_grad():
        refs = [I.siglip_encode_image(p, DUAL, x[None], interpolate_pos_encoding=True) for x in imgs]
    _parity("SigLIP (MAP head) encode_image packed list of 7 sizes", dtype, emb, refs)


def test_vit_b16():
    from jimm_b200.models import VisionTransformer

    cfg = O.ViTCfg()
    p = O.random_vit_params(cfg, seed=0)
    sizes = [(224, 224), (288, 160), (160, 224), (16, 16), (230, 170), (288, 160)]
    imgs = _images(sizes, 5)
    m = _set(VisionTransformer(dtype=torch.float16), p).eval()
    packed = m([x.cuda() for x in imgs], interpolate_pos_encoding=True)
    _rows_equal_singles(m, imgs, packed)
    with torch.no_grad():
        refs = [I.vit_forward(p, cfg, x[None], interpolate_pos_encoding=True) for x in imgs]
    _parity("ViT-B/16 packed list of 6 sizes", torch.float16, packed, refs)


# ------------------------------------------------------------------ chunking, rebuilds, calls in flight
def test_chunks_give_the_same_bytes():
    cfg, p, make = _vit_small()
    imgs = [x.cuda() for x in _images(SIZES_P16 + [(64, 48), (80, 80)], 6)]
    one = make()
    one.set_max_batch(16).set_max_image_size(230, 170)
    ref = one(imgs, interpolate_pos_encoding=True)
    small = make()
    small.set_max_batch(2).set_max_image_size(230, 170)  # 2 images per chunk at most: 9 images take 5 chunks
    assert torch.equal(small(imgs, interpolate_pos_encoding=True), ref)
    tight = make()
    tight.set_max_batch(16)  # the default budget, 16 x 17 tokens, holds 290 tokens in two chunks
    assert torch.equal(tight(imgs, interpolate_pos_encoding=True), ref)


def test_one_rebuild_for_an_image_too_large(monkeypatch):
    from jimm_b200.common.vit import _NativeOwner

    cfg, p, make = _vit_small()
    m = make()
    m.set_max_batch(2)
    small = [x.cuda() for x in _images([(64, 64), (32, 48)], 7)]
    m(small, interpolate_pos_encoding=True)
    built = []
    orig = _NativeOwner._build_native
    monkeypatch.setattr(_NativeOwner, "_build_native", lambda self, mb: built.append(mb) or orig(self, mb))
    big = small + [x.cuda() for x in _images([(320, 256)], 8)]  # 321 tokens; the handle holds 2 x 17
    out = m(big, interpolate_pos_encoding=True)
    assert len(built) == 1
    m(big, interpolate_pos_encoding=True)
    assert len(built) == 1
    for i, x in enumerate(big):
        assert torch.equal(out[i:i + 1], m(x[None], interpolate_pos_encoding=True))


def test_c_entry_refuses_an_image_too_large():
    from jimm_b200 import _lib

    cfg, p, make = _vit_small()
    m = make()
    m.set_max_batch(2)
    n = m.native()
    x = torch.zeros((320, 256, 3), device="cuda")
    y = torch.zeros((64, 64, 3), device="cuda")
    out = torch.full((2, 10), float("nan"), device="cuda")
    ptrs = (C.c_void_p * 2)(y.data_ptr(), x.data_ptr())
    hs, ws = (C.c_int * 2)(64, 320), (C.c_int * 2)(64, 256)
    lib = _lib.load()
    rc = lib.jimm_vit_forward_packed(n.handle, ptrs, _lib.F32, 2, hs, ws, C.c_void_p(out.data_ptr()), stream())
    assert rc == -1 and "needs 321 tokens" in lib.jimm_last_error().decode()
    torch.cuda.synchronize()
    assert torch.isnan(out).all()  # refused before anything was enqueued


def test_two_calls_in_flight():
    cfg, p, make = _vit_small()
    m = make()
    a = [x.cuda() for x in _images([(96, 80), (16, 16), (64, 64), (230, 170)], 9)]
    b = [x.cuda() for x in _images([(32, 48), (48, 112), (48, 112)], 10)]
    ra = m(a, interpolate_pos_encoding=True).clone()
    torch.cuda.synchronize()
    rb = m(b, interpolate_pos_encoding=True).clone()
    torch.cuda.synchronize()
    oa = m(a, interpolate_pos_encoding=True)
    ob = m(b, interpolate_pos_encoding=True)
    torch.cuda.synchronize()
    assert torch.equal(oa, ra) and torch.equal(ob, rb)


# ------------------------------------------------------------------ inputs
def test_host_and_numpy_lists():
    cfg, p, make = _vit_small()
    m = make()
    imgs = _images(SIZES_P16, 11)
    dev = m([x.cuda() for x in imgs], interpolate_pos_encoding=True)
    for lst in (imgs, [x.numpy() for x in imgs], tuple(x[None] for x in imgs)):
        out = m(lst, interpolate_pos_encoding=True)
        assert not out.is_cuda and torch.equal(out, dev.cpu())
    res = m.forward_async(imgs, interpolate_pos_encoding=True).result()
    assert torch.equal(res, dev.cpu())


def test_uint8_frames_without_centre_crop():
    from jimm_b200.preprocess import ImagePreprocessor

    cfg, p, make = _vit_small()
    m = make()
    m.set_preprocessor(ImagePreprocessor(size={"shortest_edge": 64}, do_center_crop=False))
    g = torch.Generator().manual_seed(12)
    frames = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in [(120, 200), (64, 64), (300, 150), (99, 77)]]
    packed = m([f.cuda() for f in frames], interpolate_pos_encoding=True)
    for i, f in enumerate(frames):
        assert torch.equal(packed[i:i + 1], m(f[None].cuda(), interpolate_pos_encoding=True)), i
    assert torch.equal(m(frames, interpolate_pos_encoding=True), packed.cpu())


# ------------------------------------------------------------------ errors
def test_errors():
    cfg, p, make = _vit_small()
    m = make()
    a = torch.zeros((64, 64, 3), device="cuda")
    with pytest.raises(ValueError, match="one dtype"):
        m([a, a.half()], interpolate_pos_encoding=True)
    with pytest.raises(ValueError, match="one device"):
        m([a, a.cpu()], interpolate_pos_encoding=True)
    with pytest.raises(ValueError, match="expected NHWC"):
        m([a, torch.zeros((64, 64, 4), device="cuda")], interpolate_pos_encoding=True)
    with pytest.raises(ValueError, match="smaller than one 16x16 patch"):
        m([a, torch.zeros((12, 64, 3), device="cuda")], interpolate_pos_encoding=True)
    with pytest.raises(ValueError, match="expected NHWC"):
        m([a, torch.zeros((96, 64, 3), device="cuda")])  # without interpolate_pos_encoding every image is at the trained size
    assert torch.equal(m([a, a]), m(torch.stack([a, a])))
    empty = m([], interpolate_pos_encoding=True)
    assert empty.shape == (0, 10) and empty.dtype == torch.float32
