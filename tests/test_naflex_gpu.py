"""GPU: SigLIP 2 NaFlex -- the antialiased bilinear position resample (jimm_k_tokens_add_interp_packed / jimm_k_tokens_init_interp_ex,
mode 1) against F.interpolate(antialias=True), the gather of HF patch rows (jimm_k_patch_rows_packed), and the model on the golden
fixture: parity with HF Siglip2Model, bit equalities between its input forms, chunking and refused calls."""

import ctypes as C
import os

import numpy as np
import pytest
import torch

import naflex_oracle as N
from gpu_util import BF16, F16, F32, TORCH, check, check_parity, ptr, rel_err, stream

pytestmark = pytest.mark.gpu
TOL = 1e-3
BF16_TOL = 8e-3
TF32 = 3
AA = 1  # resampling mode: antialiased bilinear
GRIDS = [(1, 1), (1, 37), (7, 16), (11, 23), (16, 16), (32, 8), (40, 40), (64, 4)]


def _offsets(lens):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return off, torch.from_numpy(off).cuda()


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("D", [64, 200, 768, 1152])
def test_pos_resample_vs_interpolate(lib, D):
    g = 16
    pos = torch.randn((g * g, D), generator=torch.Generator().manual_seed(D))
    pos_d = pos.cuda()
    lens = [gh * gw for gh, gw in GRIDS]
    off, off_d = _offsets(lens)
    gw_d = torch.tensor([gw for _, gw in GRIDS], dtype=torch.int32, device="cuda")
    x = torch.zeros((int(off[-1]) + 3, D), device="cuda")
    x[-3:] = 5.0  # rows outside every image stay as filled
    check(lib, lib.jimm_k_tokens_add_interp_packed(None, ptr(pos_d), g, D, ptr(x), ptr(off_d), ptr(gw_d), len(GRIDS), max(lens), AA, stream()))
    for b, (gh, gw) in enumerate(GRIDS):
        got = x[off[b]:off[b + 1]]
        ref = N.resample_pos_aa(pos[None], g, gh, gw)[0]
        err = rel_err(got.cpu(), ref)
        assert err < 1e-6, f"grid {gh}x{gw} D={D}: rel err {err:.2e}"
        one = torch.full((gh * gw, D), float("nan"), device="cuda")
        check(lib, lib.jimm_k_tokens_init_interp_ex(None, ptr(pos_d), g, D, ptr(one), 1, gh, gw, AA, stream()))
        assert torch.equal(one, got), f"grid {gh}x{gw}: the per-image and packed kernels differ"
        if (gh, gw) == (g, g):
            assert torch.equal(got.cpu(), pos)  # the identity, bit for bit
    assert torch.equal(x[-3:], torch.full((3, D), 5.0, device="cuda"))


def test_pos_resample_bicubic_mode_unchanged(lib):
    """Mode 0 of the new packed entry point is the bicubic resample of jimm_k_tokens_init_interp, bit for bit."""
    g, D = 16, 128
    pos_d = torch.randn((g * g, D), generator=torch.Generator().manual_seed(1)).cuda()
    lens = [gh * gw for gh, gw in GRIDS]
    off, off_d = _offsets(lens)
    gw_d = torch.tensor([gw for _, gw in GRIDS], dtype=torch.int32, device="cuda")
    x = torch.zeros((int(off[-1]), D), device="cuda")
    check(lib, lib.jimm_k_tokens_add_interp_packed(None, ptr(pos_d), g, D, ptr(x), ptr(off_d), ptr(gw_d), len(GRIDS), max(lens), 0, stream()))
    for b, (gh, gw) in enumerate(GRIDS):
        one = torch.full((gh * gw, D), float("nan"), device="cuda")
        check(lib, lib.jimm_k_tokens_init_interp(None, ptr(pos_d), g, D, ptr(one), 1, gh, gw, stream()))
        assert torch.equal(one, x[off[b]:off[b + 1]])


@pytest.mark.parametrize("P,hw", [(4, (28, 120)), (16, (70, 50)), (14, (42, 29))])
def test_patchify_rows_are_processor_rows(lib, P, hw):
    """patchify writes each patch row in (py, px, c) order: the rows of Siglip2ImageProcessor's convert_image_to_patches."""
    img = torch.randn((*hw, 3), generator=torch.Generator().manual_seed(P))
    gh, gw = hw[0] // P, hw[1] // P
    out = torch.full((gh * gw, P * P * 3), float("nan"), device="cuda")
    check(lib, lib.jimm_k_patchify(ptr(img.cuda()), F32, 1, hw[0], hw[1], 3, P, ptr(out), F32, stream()))
    assert torch.equal(out.cpu(), N.image_to_rows(img, P))


@pytest.mark.parametrize("out_code", [F32, F16, BF16, TF32])
@pytest.mark.parametrize("in_code", [F32, F16, BF16])
def test_patch_rows_gather_equals_patchify(lib, in_code, out_code):
    """The patch rows of a padded pixel_values batch land in the packed operand with the bits patchify gives on the same pixels; padding
    rows (NaN here) are never read and the pad columns are zeros."""
    P, Nmax, ldk = 4, 256, 56
    K = P * P * 3
    g = torch.Generator().manual_seed(in_code * 4 + out_code)
    imgs = [torch.randn((h * P, w * P, 3), generator=g).to(TORCH[in_code]) for h, w in N.GOLDEN_SHAPES]
    pv, _, _ = N.pad_batch(imgs, P, Nmax, fill=float("nan"))
    lens = [h * w for h, w in N.GOLDEN_SHAPES]
    off, off_d = _offsets(lens)
    odt = torch.float32 if out_code == TF32 else TORCH[out_code]
    out = torch.full((int(off[-1]) + 4, ldk), 7.0, dtype=odt, device="cuda")
    check(lib, lib.jimm_k_patch_rows_packed(ptr(pv.cuda()), in_code, Nmax, K, ptr(off_d), len(imgs), max(lens), ptr(out), out_code, ldk, stream()))
    for b, x in enumerate(imgs):
        ref = torch.full((lens[b], ldk), float("nan"), dtype=odt, device="cuda")
        check(lib, lib.jimm_k_patchify_ex(ptr(x.cuda()), in_code, 1, x.shape[0], x.shape[1], 3, P, ptr(ref), out_code, 0, ldk, stream()))
        assert torch.equal(out[off[b]:off[b + 1]], ref), f"sample {b}"
    assert torch.all(out[: int(off[-1]), K:] == 0)
    assert torch.all(out[int(off[-1]):] == 7.0)


# ------------------------------------------------------------------ model on the golden fixture
def _fixture(golden_dir):
    d = os.path.join(golden_dir, "tiny_siglip2_naflex")
    return os.path.join(d, "model.safetensors"), dict(np.load(os.path.join(d, "io.npz")))


def _model(path, dtype):
    from jimm_b200.models import SigLIP

    m = SigLIP.from_pretrained(path, dtype=dtype)
    assert m.naflex
    return m


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn])
def test_golden_parity_vs_hf(golden_dir, dtype):
    path, io = _fixture(golden_dir)
    m = _model(path, dtype)
    pv, shapes, mask = torch.from_numpy(io["pixel_values"]).cuda(), io["spatial_shapes"], io["pixel_attention_mask"]
    txt = torch.from_numpy(io["tokens"]).cuda()
    ie = m.encode_image(pv, spatial_shapes=shapes, pixel_attention_mask=mask)
    te = m.encode_text(txt)
    lg = m(pv, txt, spatial_shapes=shapes, pixel_attention_mask=mask)
    assert ie.shape == (7, 64) and lg.shape == (7, 5)
    # bf16 operands carry 8 significant bits (unit roundoff 3.9e-3), so bf16 against an fp32 model gets the project's bf16 bound; FP8 is
    # outside the parity of the other modes: reported only
    bound = {torch.float32: TOL, torch.float16: TOL, torch.bfloat16: BF16_TOL, torch.float8_e4m3fn: None}[dtype]
    case = "golden tiny_siglip2_naflex, padded mixed shapes"
    check_parity(case, "image_embeds", dtype, "HF Siglip2Model fp32", ie, io["hf_image_embeds"], bound)
    check_parity(case, "text_embeds", dtype, "HF Siglip2Model fp32", te, io["hf_text_embeds"], bound)
    check_parity(case, "logits", dtype, "HF Siglip2Model fp32", lg, io["hf_logits"], bound)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_input_forms_give_the_same_bits(golden_dir, dtype):
    path, io = _fixture(golden_dir)
    m = _model(path, dtype)
    pv, shapes, mask = torch.from_numpy(io["pixel_values"]), io["spatial_shapes"], io["pixel_attention_mask"]
    P = m.vision_patch_size
    ie = m.encode_image(pv.cuda(), spatial_shapes=shapes, pixel_attention_mask=mask)
    # host pixel_values, no mask
    assert torch.equal(m.encode_image(pv, spatial_shapes=shapes).cuda(), ie)
    # padding rows full of NaN change no bit
    pv_nan = pv.clone()
    for b, (h, w) in enumerate(shapes.tolist()):
        pv_nan[b, h * w:] = float("nan")
    assert torch.equal(m.encode_image(pv_nan.cuda(), spatial_shapes=shapes), ie)
    # each sample alone, as pixel_values with its own N
    for b, (h, w) in enumerate(shapes.tolist()):
        one = m.encode_image(pv[b:b + 1, : h * w].cuda(), spatial_shapes=shapes[b:b + 1])
        assert torch.equal(one, ie[b:b + 1]), f"sample {b} ({h}x{w})"
    # the same pixels as NHWC images: a list (packed call), and each image as a batch of one (the *_hw calls; 64 x 64 is img_size)
    imgs = [N.rows_to_image(pv[b, : h * w], h, w, P) for b, (h, w) in enumerate(shapes.tolist())]
    assert torch.equal(m.encode_image([x.cuda() for x in imgs]), ie)
    for b, x in enumerate(imgs):
        assert torch.equal(m.encode_image(x[None].cuda()), ie[b:b + 1]), f"image {b} {tuple(x.shape)}"
    # trailing pixels that do not fill a patch are dropped
    wide = torch.cat([imgs[1], torch.randn((imgs[1].shape[0], 3, 3))], 1)
    assert torch.equal(m.encode_image([wide.cuda()]), ie[1:2])
    # the dual call: pixel_values, and one image through jimm_dual_forward_hw
    txt = torch.from_numpy(io["tokens"]).cuda()
    lg = m(pv.cuda(), txt, spatial_shapes=shapes)
    assert torch.equal(lg, m.native().logits(ie, m.encode_text(txt)))
    assert torch.equal(m(imgs[3][None].cuda(), txt), lg[3:4])


def test_chunking_matches_single_samples(golden_dir):
    """More samples than max_batch, and samples past the token budget (max_batch x 256 tokens): the chunks equal the per-sample calls."""
    path, _ = _fixture(golden_dir)
    m = _model(path, torch.float16).set_max_batch(4)
    shapes = [(32, 32), (16, 16), (8, 8), (40, 25), (1, 1), (12, 20), (3, 50), (16, 16), (9, 9)]
    imgs = [torch.randn((h * 4, w * 4, 3), generator=torch.Generator().manual_seed(i)) for i, (h, w) in enumerate(shapes)]
    pv, ss, _ = N.pad_batch(imgs, 4, 1024, fill=float("nan"))
    out = m.encode_image(pv.cuda(), spatial_shapes=ss)
    assert m.native().max_batch == 4
    for b, (h, w) in enumerate(shapes):
        one = m.encode_image(pv[b:b + 1, : h * w].cuda(), spatial_shapes=ss[b:b + 1])
        assert torch.equal(one, out[b:b + 1]), f"sample {b} ({h}x{w})"
    assert torch.equal(m.encode_image([x.cuda() for x in imgs]), out)


def test_refused_calls_enqueue_nothing(lib, golden_dir):
    from jimm_b200.models import SigLIP

    path, io = _fixture(golden_dir)
    m = _model(path, torch.float16)
    pv = torch.from_numpy(io["pixel_values"]).cuda()
    B, Nmax = pv.shape[0], pv.shape[1]
    n = m.native()
    out = torch.full((B, 64), float("nan"), device="cuda")

    def call(handle, grid):
        g = (C.c_int * (2 * B))(*[v for hw in grid for v in hw])
        torch.cuda.synchronize()
        n0 = lib.jimm_launch_count()
        rc = lib.jimm_encode_image_patches(handle, ptr(pv), F32, B, Nmax, g, ptr(out), stream())
        torch.cuda.synchronize()
        assert lib.jimm_launch_count() == n0
        return rc

    good = [tuple(s) for s in io["spatial_shapes"].tolist()]
    assert call(n.handle, [(17, 16)] + good[1:]) == -1  # 272 > N = 256
    assert "more than its N" in lib.jimm_last_error().decode()
    assert call(n.handle, good[:3] + [(0, 4)] + good[4:]) == -1
    plain = SigLIP.from_pretrained(os.path.join(golden_dir, "tiny_siglip", "model.safetensors"), dtype=torch.float16)
    assert call(plain.native().handle, good) == -1
    assert "not a SigLIP 2 NaFlex" in lib.jimm_last_error().decode()
    assert torch.isnan(out).all()
    with pytest.raises(ValueError):
        m.encode_image(pv, spatial_shapes=np.array([(17, 16)] + good[1:]))
