"""The image front-end at the frame sizes cameras and phones produce (1080p, 4K UHD, 12 MP, 24 MP, 8K, both orientations), at tiny and
extreme aspect ratios, and past 65535 images per call, against oracle/preprocess_oracle.py (or Pillow's own resize, which
test_oracle_resize_matches_pillow pins the oracle to): fp32 bit for bit, fp16 / bf16 equal to the round-to-nearest-even cast of the
fp32 reference.

Sizes whose fused plan does not fit in shared memory run in two passes through a global 8-bit intermediate (csrc/preprocess.cu).
The CPU tests pin the planner through its host-only hook: sizes that fitted keep their plan, the sizes that did not fit get the
two-pass path, and the GPU cases below cover every (budget tier, TY) plan the planner chooses."""
import functools

import numpy as np
import pytest
import torch

import preprocess_oracle as P

gpu = pytest.mark.gpu

KINDS = {
    "vit": (lambda s: dict(size={"height": s, "width": s}, resample=P.BILINEAR), P.PreprocessConfig.vit),
    "siglip": (lambda s: dict(size={"height": s, "width": s}, resample=P.BICUBIC), P.PreprocessConfig.siglip),
    "clip": (lambda s: dict(size={"shortest_edge": s}, crop_size={"height": s, "width": s}, resample=P.BICUBIC), P.PreprocessConfig.clip),
}
FRONT_ENDS = [("vit", 224), ("clip", 224), ("clip", 336), ("siglip", 224), ("siglip", 384), ("siglip", 512)]
# 1080p, 4K UHD, 12 MP (4:3 phone), 3000 x 4000, 24 MP, 8K UHD; each in landscape and portrait
FRAMES = [(1080, 1920), (2160, 3840), (3024, 4032), (3000, 4000), (4000, 6000), (4320, 7680)]
FRAMES = FRAMES + [(w, h) for h, w in FRAMES]
CAMERA_CASES = [(h, w, kind, size) for h, w in FRAMES for kind, size in FRONT_ENDS]

# Plans of the fused kernel (tier, TY, shared-memory bytes) before the two-pass path existed: the 14 sizes of
# test_preprocess_gpu.py's CASES, the golden-fixture sizes, and every camera frame whose plan fitted.
FUSED_PLANS = [
    ("vit", 224, 480, 640, 0, 16, 57664), ("vit", 224, 224, 224, 0, 32, 35136), ("vit", 224, 37, 53, 0, 32, 13568),
    ("vit", 384, 500, 333, 0, 16, 50592), ("clip", 224, 480, 640, 0, 16, 63168), ("clip", 224, 640, 480, 0, 16, 59328),
    ("clip", 224, 333, 500, 0, 32, 65088), ("clip", 224, 224, 224, 0, 32, 46336), ("siglip", 256, 480, 640, 0, 16, 66080),
    ("siglip", 224, 100, 80, 0, 32, 31456), ("siglip", 512, 1080, 1920, 2, 16, 169760), ("vit", 32, 3, 3, 0, 32, 1728),
    ("clip", 75, 301, 227, 0, 32, 40392), ("siglip", 50, 2000, 35, 2, 16, 144360),
    ("vit", 48, 61, 83, 0, 32, 12016), ("vit", 48, 48, 48, 0, 32, 7856), ("vit", 48, 30, 100, 0, 32, 8944),
    ("clip", 40, 61, 83, 0, 32, 12232), ("clip", 40, 90, 57, 0, 32, 10864), ("clip", 40, 40, 40, 0, 32, 8560),
    ("siglip", 64, 61, 83, 0, 32, 13472), ("siglip", 64, 200, 150, 0, 32, 30688), ("siglip", 64, 20, 24, 0, 32, 8224),
    ("vit", 224, 1080, 1920, 2, 32, 181280), ("vit", 224, 1920, 1080, 2, 16, 149728),
    ("clip", 224, 1080, 1920, 2, 32, 202560), ("clip", 224, 1920, 1080, 2, 32, 182464),
    ("clip", 336, 1080, 1920, 2, 16, 153600), ("clip", 336, 1920, 1080, 2, 32, 184784),
    ("siglip", 224, 1080, 1920, 2, 16, 165536), ("siglip", 224, 1920, 1080, 2, 16, 189184),
    ("siglip", 384, 1080, 1920, 2, 16, 170912), ("siglip", 384, 1920, 1080, 2, 16, 195872),
    ("siglip", 512, 1080, 1920, 2, 16, 169760), ("siglip", 512, 1920, 1080, 2, 16, 194464),
    ("vit", 224, 2160, 3840, 2, 4, 182720), ("vit", 224, 3840, 2160, 2, 4, 163296), ("vit", 224, 3024, 4032, 2, 2, 187328),
    ("vit", 224, 4032, 3024, 2, 4, 194144), ("vit", 224, 3000, 4000, 2, 4, 204032), ("vit", 224, 4000, 3000, 2, 4, 193504),
    ("clip", 224, 2160, 3840, 2, 2, 196288), ("clip", 224, 3840, 2160, 2, 8, 194944), ("clip", 224, 4000, 3000, 2, 1, 202208),
    ("clip", 336, 2160, 3840, 2, 2, 193552), ("clip", 336, 3840, 2160, 2, 8, 191536),
    ("siglip", 224, 3840, 2160, 2, 2, 199648), ("siglip", 384, 3840, 2160, 2, 1, 194080), ("siglip", 512, 3840, 2160, 2, 2, 201632),
]
_FUSED_CAMERA = {(k, s, h, w) for k, s, h, w, *_ in FUSED_PLANS}
# every camera cell whose fused plan did not fit (the front-end refused these: "needs N bytes of shared memory")
REFUSED_BEFORE = [(h, w, k, s) for h, w, k, s in CAMERA_CASES if (k, s, h, w) not in _FUSED_CAMERA]

# Frames that reach the (tier, TY) plans no camera cell above reaches
TIER_CASES = [(640, 1, "siglip", 224), (1080, 1, "siglip", 224), (1, 1920, "siglip", 224)]
# Tiny and extreme shapes: upscaling from 1-3 pixels, one-pixel-wide frames (CLIP resizes 1 x 3000 to 224 x 672000 before the crop),
# a 89600-wide CLIP pre-crop resize, and a tall narrow SigLIP frame
EXTREME_CASES = ([(n, n, k, 512) for n in (1, 2, 3) for k in ("vit", "clip", "siglip")] +
                 [(1, 3000, k, 224) for k in KINDS] + [(3000, 1, k, 224) for k in KINDS] +
                 [(10, 4000, "clip", 224), (4000, 10, "clip", 224), (4000, 35, "siglip", 224)])
# Wide windows over narrow outputs: more than 127 four-tap groups per output column, which the fused kernel's packed window
# descriptor cannot hold (it ran these and wrote zeros); they take the two-pass path.
WIDE_WINDOW_CASES = [(32, 4500, {"size": {"height": 32, "width": 32}, "resample": P.BICUBIC}),
                     (8, 5000, {"size": {"height": 8, "width": 12}, "resample": P.BILINEAR}),
                     (16, 4000, {"size": {"height": 16, "width": 30}, "resample": P.BICUBIC})]


def _kw(kind, size):
    return KINDS[kind][0](size)


def _cfg(kind, size):
    return KINDS[kind][1](size)


def _plan(h, w, **kw):
    from jimm_b200 import preprocess as pp

    return pp.plan(h, w, **kw)


# ---------------------------------------------------------------- references
def _geometry(cfg, h, w):
    rh, rw = P.resized_size(cfg, h, w)
    oh, ow = cfg.crop_h or rh, cfg.crop_w or rw
    return rh, rw, (rh - oh) // 2, (rw - ow) // 2, oh, ow


def _pillow_ref(img, cfg):
    """Pillow's Image.resize, then the centre crop and the oracle's rescale / normalise."""
    from PIL import Image

    h, w, _ = img.shape
    rh, rw, top, left, oh, ow = _geometry(cfg, h, w)
    r = np.asarray(Image.fromarray(img).resize((rw, rh), resample=cfg.resample)) if (rh, rw) != (h, w) else img
    return P.rescale_normalize(r[top:top + oh, left:left + ow], cfg)


def _cropped_ref(img, cfg):
    """P.preprocess evaluated for the kept rows and columns only: the oracle's tables sliced to the crop and its passes over them (the
    full pre-crop resize of a one-pixel-wide CLIP frame would not fit in memory), the vertical pass 16 output rows at a time (its
    gather holds every tap of every output row)."""
    h, w, _ = img.shape
    rh, rw, top, left, oh, ow = _geometry(cfg, h, w)
    out = img
    if rw != w:
        fh, _, kh = P.resample_coeffs(w, rw, cfg.resample)
        out = P._pass(out, fh[left:left + ow], kh[left:left + ow], axis=1)
    else:
        out = out[:, left:left + ow]
    if rh != h:
        fv, _, kv = P.resample_coeffs(h, rh, cfg.resample)
        fv, kv = fv[top:top + oh], kv[top:top + oh]
        out = np.concatenate([P._pass(out, fv[i:i + 16], kv[i:i + 16], axis=0) for i in range(0, oh, 16)])
    else:
        out = out[top:top + oh]
    return P.rescale_normalize(out, cfg)


@functools.lru_cache(maxsize=2)
def _frames(h, w, n=2, seed=0):
    """n camera-sized uint8 frames: 16 x 16 blocks of random level plus noise, with saturated rows and columns so that the bicubic
    lobes hit both clamps.  Cheap at 8K (numpy uint8 throughout)."""
    rng = np.random.default_rng(seed * 7919 + h * 31 + w)
    base = rng.integers(0, 128, (n, (h + 15) // 16, (w + 15) // 16, 3), dtype=np.uint8)
    img = np.repeat(np.repeat(base, 16, axis=1), 16, axis=2)[:, :h, :w]
    img = img + rng.integers(0, 128, (n, h, w, 3), dtype=np.uint8)
    img[:, ::11] = 255
    img[:, :, ::13] = 0
    return np.ascontiguousarray(img)


# ---------------------------------------------------------------- CPU: the planner
@pytest.mark.parametrize("kind,size,h,w,tier,ty,smem", FUSED_PLANS)
def test_fitting_sizes_keep_their_fused_plan(lib, kind, size, h, w, tier, ty, smem):
    assert _plan(h, w, **_kw(kind, size)) == (0, tier, ty, smem)


def test_sizes_that_did_not_fit_get_the_two_pass_plan(lib):
    assert len(REFUSED_BEFORE) == 46
    for h, w, kind, size in REFUSED_BEFORE:
        assert _plan(h, w, **_kw(kind, size)) == (1, -1, 8, 0), (h, w, kind, size)
    for h, w, kw in WIDE_WINDOW_CASES:
        assert _plan(h, w, **kw)[0] == 1, (h, w, kw)


def test_gpu_cases_cover_every_plan(lib):
    """Every (path, tier, TY) the planner chooses over a grid of frame sizes and the stock front-ends occurs among the GPU cases."""
    edges = [1, 3, 16, 35, 64, 100, 224, 333, 480, 640, 720, 1080, 1440, 1920, 2160, 3000, 3024, 3840, 4000, 4032, 4320, 6000, 7680]
    chosen = set()
    for kind, size in FRONT_ENDS + [("vit", 32), ("siglip", 64), ("clip", 64), ("siglip", 256)]:
        for h in edges:
            for w in edges:
                try:
                    chosen.add(_plan(h, w, **_kw(kind, size))[:3])
                except ValueError:  # CLIP crop larger than a tiny resized edge
                    pass
    covered = {_plan(h, w, **_kw(k, s))[:3] for h, w, k, s in CAMERA_CASES + TIER_CASES + EXTREME_CASES}
    assert {(0, 0, 32), (0, 2, 1), (1, -1, 8)} <= chosen
    assert chosen <= covered, sorted(chosen - covered)


def test_remaining_limits_are_refused_with_their_message(lib):
    with pytest.raises(ValueError, match=r"at most 2\^31 - 1 bytes"):
        _plan(30000, 24000, **_kw("vit", 224))
    with pytest.raises(ValueError, match=r"at most 16777216 pixels per edge"):
        _plan(1, 80000, **_kw("clip", 224))  # CLIP: 224 x 17920000 before the crop
    with pytest.raises(ValueError, match="centre crop"):
        _plan(8, 8, size={"height": 16, "width": 16}, crop_size={"height": 32, "width": 32})
    with pytest.raises(ValueError, match=r"8-bit intermediate of 2160216000 bytes per image"):
        _plan(40000, 10, size={"height": 40000, "width": 18000}, resample=P.BILINEAR)  # (40000 + 4) rows x 54000 bytes
    assert _plan(24000, 29826, **_kw("vit", 224))[0] == 1  # 2^31 - 1 - 1152 bytes: still taken
    assert _plan(1, 74898, **_kw("clip", 224))[0] == 1  # 224 x 16777152
    assert _plan(39000, 10, size={"height": 39000, "width": 18000}, resample=P.BILINEAR)[0] == 1  # 2106216000 bytes


def test_cropped_reference_matches_oracle():
    for h, w, kind, size in [(37, 53, "clip", 24), (90, 57, "clip", 40), (61, 83, "siglip", 64), (3, 3, "vit", 32), (1, 30, "clip", 8)]:
        img = _frames(h, w, 1)[0]
        assert np.array_equal(_cropped_ref(img, _cfg(kind, size)), P.preprocess(img, _cfg(kind, size))), (h, w, kind)


# ---------------------------------------------------------------- GPU: the kernels
def _proc(kind, size):
    from jimm_b200.preprocess import ImagePreprocessor

    return getattr(ImagePreprocessor, kind)(size)


@gpu
@pytest.mark.parametrize("h,w,kind,size", CAMERA_CASES + TIER_CASES)
def test_camera_frames_bit_exact(lib, h, w, kind, size):
    n = 1 if h * w > 13_000_000 else 2
    imgs = _frames(h, w)[:n]
    cfg = _cfg(kind, size)
    ref = np.stack([_pillow_ref(im, cfg) for im in imgs])
    out = _proc(kind, size)(torch.from_numpy(imgs).cuda(), dtype=torch.float32).cpu().numpy()
    assert out.shape == ref.shape
    assert np.array_equal(out, ref), (np.count_nonzero(out != ref), _plan(h, w, **_kw(kind, size)))


@gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("h,w,kind,size", [(2160, 3840, "siglip", 384), (4032, 3024, "clip", 224), (4320, 7680, "vit", 224),
                                           (3840, 2160, "clip", 336)])
def test_camera_frames_half_outputs(lib, h, w, kind, size, dtype):
    imgs = _frames(h, w)[:1]
    ref = torch.from_numpy(_pillow_ref(imgs[0], _cfg(kind, size)))[None].to(dtype)
    out = _proc(kind, size)(torch.from_numpy(imgs).cuda(), dtype=dtype)
    assert out.dtype == dtype and torch.equal(out.cpu(), ref)


@gpu
@pytest.mark.parametrize("h,w,kind,size", EXTREME_CASES)
def test_tiny_and_extreme_shapes(lib, h, w, kind, size):
    imgs = _frames(h, w)
    ref = np.stack([_cropped_ref(im, _cfg(kind, size)) for im in imgs])
    out = _proc(kind, size)(torch.from_numpy(imgs).cuda(), dtype=torch.float32).cpu().numpy()
    assert out.shape == ref.shape and np.array_equal(out, ref)


@gpu
@pytest.mark.parametrize("h,w,kw", WIDE_WINDOW_CASES)
def test_wide_windows_bit_exact(lib, h, w, kw):
    from jimm_b200.preprocess import ImagePreprocessor

    imgs = _frames(h, w)
    cfg = P.PreprocessConfig(height=kw["size"]["height"], width=kw["size"]["width"], resample=kw["resample"])
    ref = np.stack([P.preprocess(im, cfg) for im in imgs])
    out = ImagePreprocessor(**kw)(torch.from_numpy(imgs).cuda(), dtype=torch.float32).cpu().numpy()
    assert np.array_equal(out, ref), np.count_nonzero(out != ref)


@gpu
@pytest.mark.parametrize("offset", [0, 5])
def test_more_than_65535_images(lib, offset):
    """65540 frames of 8 x 8 -> 4 x 4: two launches, the second starting at image 65532 -- from a 16-byte aligned base and from one 5
    bytes off it."""
    from jimm_b200.preprocess import ImagePreprocessor

    B = 65540
    imgs = np.random.default_rng(1).integers(0, 256, (B, 8, 8, 3), dtype=np.uint8)
    # the oracle's two passes over the whole batch at once (rows of all images, then columns of all images)
    fh, _, kh = P.resample_coeffs(8, 4, P.BILINEAR)
    x = P._pass(imgs.reshape(B * 8, 8, 3), fh, kh, axis=1).reshape(B, 8, 4, 3)
    x = P._pass(x.transpose(1, 0, 2, 3).reshape(8, B * 4, 3), fh, kh, axis=0).reshape(4, B, 4, 3).transpose(1, 0, 2, 3)
    cfg = P.PreprocessConfig.vit(4)
    ref = P.rescale_normalize(x, cfg)
    for i in (0, 65531, 65532, B - 1):
        assert np.array_equal(ref[i], P.preprocess(imgs[i], cfg))
    flat = torch.zeros(imgs.size + offset, dtype=torch.uint8, device="cuda")
    flat[offset:] = torch.from_numpy(imgs).reshape(-1).cuda()
    out = ImagePreprocessor.vit(4)(flat[offset:].view(B, 8, 8, 3), dtype=torch.float32).cpu().numpy()
    assert np.array_equal(out, ref), np.nonzero((out != ref).reshape(B, -1).any(1))[0][:8]


@gpu
def test_two_streams_share_one_handle(lib):
    """Two-pass calls of different sizes in flight on two streams on one handle: each call has its own intermediate."""
    proc = _proc("siglip", 384)
    cfg = _cfg("siglip", 384)
    a, b = _frames(2160, 3840), _frames(3024, 4032)
    assert _plan(2160, 3840, **_kw("siglip", 384))[0] == 1 and _plan(3024, 4032, **_kw("siglip", 384))[0] == 1
    ra = np.stack([_pillow_ref(im, cfg) for im in a])
    rb = np.stack([_pillow_ref(im, cfg) for im in b])
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for _ in range(3):
        with torch.cuda.stream(s1):
            oa = proc(da, dtype=torch.float32)
        with torch.cuda.stream(s2):
            ob = proc(db, dtype=torch.float32)
        outs.append((oa, ob))
    torch.cuda.synchronize()
    for oa, ob in outs:
        assert np.array_equal(oa.cpu().numpy(), ra) and np.array_equal(ob.cpu().numpy(), rb)


@gpu
def test_two_pass_unaligned_input_and_odd_output_width(lib):
    """The two-pass path with the input pointer off the 16-byte grid and an output row length that breaks the vector stores."""
    from jimm_b200.preprocess import ImagePreprocessor

    kw = dict(size={"height": 45, "width": 37}, resample=P.BICUBIC, image_mean=(0.1, 0.2, 0.3), image_std=(0.9, 0.8, 0.7))
    assert _plan(30, 9000, **kw)[0] == 1
    imgs = _frames(30, 9000)
    flat = torch.zeros(imgs.size + 5, dtype=torch.uint8, device="cuda")
    flat[5:] = torch.from_numpy(imgs).reshape(-1).cuda()
    proc = ImagePreprocessor(**kw)
    cfg = P.PreprocessConfig(height=45, width=37, resample=P.BICUBIC, mean=(0.1, 0.2, 0.3), std=(0.9, 0.8, 0.7))
    ref = torch.from_numpy(np.stack([P.preprocess(im, cfg) for im in imgs]))
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        assert torch.equal(proc(flat[5:].view(imgs.shape), dtype=dt).cpu(), ref.to(dt)), dt


# Tall narrow frames whose 8-bit intermediate is tens of MB per image (every row, 676 bytes each), so a call runs several chunks of
# images -- 2 and 3 per chunk -- and an output of 225 x 225 x 3 samples per image starts every chunk after the first off the
# vector-store grid of the output pointer.  The reference is the oracle, not the installed Pillow: for these shapes (horizontal axis
# upscaled, vertical one reduced) Pillow 12 runs the vertical pass first, which rounds differently, while the processors the
# front-end mirrors are pinned to Pillow 11.3, whose horizontal-then-vertical order the oracle restates.
CHUNKED_CASES = [(40000, 2, 5), (30000, 3, 7)]


@gpu
@pytest.mark.parametrize("h,w,B", CHUNKED_CASES)
def test_two_pass_chunks(lib, h, w, B):
    from jimm_b200.preprocess import ImagePreprocessor

    kw = dict(size={"height": 225, "width": 225}, resample=P.BICUBIC)
    assert _plan(h, w, **kw)[0] == 1
    per_image = h * 676
    assert 2 <= (64 << 20) // per_image < B - 1  # at least three chunks
    imgs = _frames(h, w, B)
    cfg = P.PreprocessConfig(height=225, width=225, resample=P.BICUBIC)
    ref = torch.from_numpy(np.stack([_cropped_ref(im, cfg) for im in imgs]))
    flat = torch.zeros(imgs.size + 5, dtype=torch.uint8, device="cuda")
    flat[5:] = torch.from_numpy(imgs).reshape(-1).cuda()
    proc = ImagePreprocessor(**kw)
    for x in (flat[5:].view(imgs.shape), torch.from_numpy(imgs).cuda()):
        for dt in (torch.float32, torch.float16):
            assert torch.equal(proc(x, dtype=dt).cpu(), ref.to(dt)), dt


@gpu
def test_misaligned_output_pointer_is_refused(lib):
    """The kernels store four samples at once: an output pointer off that grid is refused, not written."""
    import ctypes as C

    proc = _proc("vit", 8)
    x = torch.zeros((2, 16, 16, 3), dtype=torch.uint8, device="cuda")
    out = torch.zeros(2 * 8 * 8 * 3 + 4, device="cuda")
    for dtype, off in ((0, 4), (0, 8), (1, 4)):
        rc = lib.jimm_preproc_run(proc.handle, C.c_void_p(x.data_ptr()), 2, 16, 16, C.c_void_p(out.data_ptr() + off), dtype, None)
        assert rc == -1 and "aligned" in lib.jimm_last_error().decode()
    torch.cuda.synchronize()
    assert not out.any()


@gpu
def test_refused_size_fails_in_output_size_and_run(lib):
    import ctypes as C

    proc = _proc("clip", 224)
    with pytest.raises(ValueError, match="pixels per edge"):
        proc.output_size(1, 80000)
    with pytest.raises(ValueError, match="pixels per edge"):
        proc(np.zeros((1, 1, 80000, 3), np.uint8))
    out = torch.empty(3 * 224 * 224, device="cuda")
    x = torch.zeros(80000 * 3, dtype=torch.uint8, device="cuda")
    assert lib.jimm_preproc_run(proc.handle, C.c_void_p(x.data_ptr()), 1, 1, 80000, C.c_void_p(out.data_ptr()), 0, None) == -1
    from jimm_b200.preprocess import ImagePreprocessor

    wide = ImagePreprocessor(size={"height": 40000, "width": 18000})
    with pytest.raises(ValueError, match="8-bit intermediate"):
        wide.output_size(40000, 10)


# ---------------------------------------------------------------- GPU: through the models
CAMERA_PAIR = [(2160, 3840), (4032, 3024)]


def _vit(max_batch):
    from jimm_b200.models import VisionTransformer

    torch.manual_seed(0)
    return VisionTransformer(num_classes=10, img_size=224, patch_size=32, num_layers=2, num_heads=2, mlp_dim=256, hidden_size=128,
                             dtype=torch.float16).eval().set_max_batch(max_batch)


@gpu
def test_camera_frames_through_vit():
    """uint8 camera frames into a ViT with a SigLIP-style front-end (two passes at both sizes): device frames, pinned host frames
    (the library's sliced copy / front-end / tower pipeline), a list of mixed sizes, and small-batch graph replay -- each equal to
    front-end-then-model bit for bit."""
    from jimm_b200 import _lib
    from jimm_b200.preprocess import ImagePreprocessor

    lib = _lib.load()
    m = _vit(4)
    proc = ImagePreprocessor.siglip(224)
    m.set_preprocessor(proc)
    px = {}
    for h, w in CAMERA_PAIR:
        assert proc.output_size(h, w) == (224, 224) and _plan(h, w, **_kw("siglip", 224))[0] == 1
        frames = torch.from_numpy(_frames(h, w))
        px[h, w] = proc(frames.cuda(), dtype=torch.float16)
        ref = m(px[h, w])
        assert torch.equal(m(frames.cuda()), ref)
        assert torch.equal(m(frames.pin_memory()), ref.cpu())
        replays = lib.jimm_graph_replay_count()
        for _ in range(3):
            assert torch.equal(m(frames[:1].pin_memory()), ref[:1].cpu())
        assert lib.jimm_graph_replay_count() > replays
    mixed = [torch.from_numpy(_frames(h, w)[0]) for h, w in CAMERA_PAIR]
    ref = m([px[hw][0] for hw in CAMERA_PAIR])
    assert torch.equal(m([f.cuda() for f in mixed]), ref)
    assert torch.equal(m([f.pin_memory() for f in mixed]), ref.cpu())


@gpu
def test_camera_frames_through_clip():
    from jimm_b200 import _lib
    from jimm_b200.models import CLIP
    from jimm_b200.preprocess import ImagePreprocessor

    torch.manual_seed(0)
    m = CLIP(image_resolution=224, vision_layers=2, vision_width=128, vision_patch_size=32, context_length=16, vocab_size=100,
             transformer_width=64, transformer_heads=1, transformer_layers=2, dtype=torch.float16).eval().set_max_batch(4)
    proc = ImagePreprocessor.clip(224)
    m.set_preprocessor(proc)
    ids = torch.randint(1, 100, (2, 16), dtype=torch.int32)
    lib = _lib.load()
    embs = {}
    for h, w in CAMERA_PAIR:
        frames = torch.from_numpy(_frames(h, w))
        px = proc(frames.cuda(), dtype=torch.float16)
        ref = m(px, ids.cuda())
        assert torch.equal(m(frames.cuda(), ids.cuda()), ref)
        replays = lib.jimm_graph_replay_count()
        for _ in range(3):
            assert torch.equal(m(frames.pin_memory(), ids), ref.cpu())
        assert lib.jimm_graph_replay_count() > replays
        embs[h, w] = m.encode_image(px)
        assert torch.equal(m.encode_image(frames.pin_memory()), embs[h, w].cpu())
    mixed = [torch.from_numpy(_frames(h, w)[0]) for h, w in CAMERA_PAIR]
    ref = m.encode_image([proc(f.cuda(), dtype=torch.float16)[0] for f in mixed])
    assert torch.equal(m.encode_image([f.cuda() for f in mixed]), ref)


@gpu
def test_refused_frames_fail_before_any_work():
    """A frame size the front-end refuses raises ValueError before the model rebuilds its handle, stages a byte or launches a kernel,
    through the Python model and through the host-frame C entry point (whose byte staging would hold max_batch such frames)."""
    import ctypes as C

    from jimm_b200 import _lib
    from jimm_b200.preprocess import ImagePreprocessor

    lib = _lib.load()
    m = _vit(4096)
    m.set_preprocessor(ImagePreprocessor.clip(224))
    ok = torch.from_numpy(_frames(480, 640)[:1]).pin_memory()
    m(ok)  # build the handle, grow the staging for 480 x 640 frames
    n0 = m._native
    frame = torch.zeros((1, 1, 80000, 3), dtype=torch.uint8).pin_memory()  # CLIP: 224 x 17920000 before the crop
    torch.cuda.synchronize()
    launches, free0 = lib.jimm_launch_count(), torch.cuda.mem_get_info()[0]
    with pytest.raises(ValueError, match="pixels per edge"):
        m(frame)
    with pytest.raises(ValueError, match="pixels per edge"):
        m(frame.cuda())
    assert m._native is n0
    out = torch.empty((1, 10), dtype=torch.float32, pin_memory=True)
    rc = lib.jimm_vit_forward_host_u8(n0.handle, m._preproc.handle, C.c_void_p(frame.data_ptr()), 1, 1, 80000, C.c_void_p(out.data_ptr()),
                                      None)
    torch.cuda.synchronize()
    assert rc == -1 and "pixels per edge" in _lib.last_error()
    assert lib.jimm_launch_count() == launches
    # 4096 x 240 KB of staging would have been allocated had the call got past the size check
    assert torch.cuda.mem_get_info()[0] > free0 - (512 << 20)
    assert torch.equal(m(ok), m(ok.cuda()).cpu())


@gpu
def test_sliced_host_frames_into_an_odd_input_size():
    """Host frames large enough for the library's two-slice copy pipeline, into a model whose input (15 x 15 x 3 samples) is odd: every
    slice's front-end output starts on the grid of the vector stores, and the result equals front-end-then-model bit for bit."""
    from jimm_b200.models import VisionTransformer
    from jimm_b200.preprocess import ImagePreprocessor

    torch.manual_seed(0)
    m = VisionTransformer(num_classes=10, img_size=15, patch_size=5, num_layers=2, num_heads=2, mlp_dim=256, hidden_size=128,
                          dtype=torch.float16).eval().set_max_batch(160)
    proc = ImagePreprocessor.vit(15)
    m.set_preprocessor(proc)
    frames = torch.from_numpy(_frames(400, 400, 160))  # 77 MB of bytes: copied in two slices
    ref = m(proc(frames.cuda(), dtype=torch.float16))
    assert torch.equal(m(frames.pin_memory()), ref.cpu())
