"""GPU: which library entry points each public call reaches, in order, for every placement, type and size of its inputs; how many
handles it builds; and what it returns.  A recording wrapper around the loaded library (installed before any model is built) logs the
forward entry points, the image front-end (jimm_preproc_run) and jimm_model_finalize, and forwards every call unchanged.  A host
result must equal the result of the same call on CUDA inputs bit for bit.  The multi-GPU contrastive call is covered by
test_multigpu_gpu.py and test_interpolate_pos_multigpu_gpu.py."""

import pytest
import torch

pytestmark = pytest.mark.gpu

FIN = "jimm_model_finalize"
PRE = "jimm_preproc_run"
RECORDED = {FIN, PRE, "jimm_vit_forward", "jimm_encode_image", "jimm_encode_text", "jimm_contrastive_logits", "jimm_dual_encode",
            "jimm_dual_forward", "jimm_vit_forward_hw", "jimm_encode_image_hw", "jimm_dual_encode_hw", "jimm_dual_forward_hw",
            "jimm_vit_forward_packed", "jimm_encode_image_packed", "jimm_encoder_forward", "jimm_map_head_forward",
            "jimm_vit_forward_host", "jimm_dual_forward_host", "jimm_vit_forward_host_u8", "jimm_comm_contrastive_logits"}
S = 64  # trained size of every model here (patch 16)
B = 3


class _Recorder:
    def __init__(self, lib, log):
        self._lib, self._log = lib, log

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in RECORDED:
            return fn

        def call(*args):
            self._log.append(name)
            return fn(*args)

        return call


@pytest.fixture
def log(monkeypatch):
    from jimm_b200 import _lib, build

    build.build()
    calls = []
    rec = _Recorder(_lib.load(), calls)
    monkeypatch.setattr(_lib, "load", lambda: rec)
    return calls


def _front_end():
    """Shortest edge to 64, no crop: a 64 x 64 frame stays at the trained size, a 64 x 96 frame does not."""
    from jimm_b200.preprocess import ImagePreprocessor

    return ImagePreprocessor(size={"shortest_edge": S}, do_center_crop=False)


def _model(kind, front_end=True):
    from jimm_b200 import Rngs
    from jimm_b200.common.vit import VisionTransformerBase
    from jimm_b200.models import CLIP, SigLIP, VisionTransformer

    if kind == "vit":
        m = VisionTransformer(num_classes=10, img_size=S, patch_size=16, num_layers=2, num_heads=4, mlp_dim=512, hidden_size=128,
                              dtype=torch.float16, rngs=Rngs(0)).eval()
    elif kind == "map":
        m = VisionTransformerBase(img_size=S, patch_size=16, in_channels=3, hidden_size=128, num_layers=2, num_heads=4, mlp_dim=512,
                                  pooling_type="MAP", layernorm_epsilon=1e-6, dtype=torch.float16, rngs=Rngs(0))
    else:
        m = {"clip": CLIP, "siglip": SigLIP}[kind](S, 2, 128, 16, 16, 100, 128, 4, 2, dtype=torch.float16, rngs=Rngs(1))
    if front_end:
        m.set_preprocessor(_front_end())
    return m


def _images(b, h, w, seed):
    return torch.randn((b, h, w, 3), generator=torch.Generator().manual_seed(seed))


def _frames(b, h, w, seed):
    return torch.randint(0, 256, (b, h, w, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))


def _ids(b, seed=7):
    return torch.randint(1, 99, (b, 16), generator=torch.Generator().manual_seed(seed))


def _call(log, fn, want, cuda, shape, builds=0):
    """fn() reaches exactly the entry points `want`, builds `builds` handles and returns an fp32 tensor of `shape` on the GPU (cuda)
    or the host."""
    log.clear()
    out = fn()
    assert [c for c in log if c != FIN] == want
    assert log.count(FIN) == builds
    assert out.is_cuda == cuda and out.dtype == torch.float32 and tuple(out.shape) == tuple(shape), (out.device, out.dtype, out.shape)
    return out


def _host_forms(x):
    return [x, x.pin_memory(), x.numpy()]


# ------------------------------------------------------------------ ViT / VisionTransformerBase: __call__ and forward_async
@pytest.mark.parametrize("kind", ["vit", "map"])
def test_vision_call(log, kind):
    m = _model(kind)
    log.clear()
    od = m.native().vision_out
    assert log == [FIN]
    fwd, hw, packed = "jimm_vit_forward", "jimm_vit_forward_hw", "jimm_vit_forward_packed"

    # trained size: CUDA float (with and without interpolate_pos_encoding), CUDA uint8, host float, host uint8
    x = _images(B, S, S, 1)
    dev = _call(log, lambda: m(x.cuda()), [fwd], True, (B, od))
    assert torch.equal(_call(log, lambda: m(x.cuda(), interpolate_pos_encoding=True), [fwd], True, (B, od)), dev)
    for xh in _host_forms(x):
        assert torch.equal(_call(log, lambda: m(xh), ["jimm_vit_forward_host"], False, (B, od)), dev.cpu())
    assert torch.equal(_call(log, lambda: m(x, interpolate_pos_encoding=True), ["jimm_vit_forward_host"], False, (B, od)), dev.cpu())
    fr = _frames(B, S, S, 2)
    dev8 = _call(log, lambda: m(fr.cuda()), [PRE, fwd], True, (B, od))
    for fh in (fr, fr.pin_memory()):
        assert torch.equal(_call(log, lambda: m(fh), ["jimm_vit_forward_host_u8"], False, (B, od)), dev8.cpu())

    # other sizes with interpolate_pos_encoding, any placement
    y = _images(B, 80, 96, 3)
    devy = _call(log, lambda: m(y.cuda(), interpolate_pos_encoding=True), [hw], True, (B, od))
    for yh in _host_forms(y):
        assert torch.equal(_call(log, lambda: m(yh, interpolate_pos_encoding=True), [hw], False, (B, od)), devy.cpu())
    fy = _frames(B, S, 96, 4)
    devfy = _call(log, lambda: m(fy.cuda(), interpolate_pos_encoding=True), [PRE, hw], True, (B, od))
    assert torch.equal(_call(log, lambda: m(fy, interpolate_pos_encoding=True), [PRE, hw], False, (B, od)), devfy.cpu())

    # lists: one packed call, uint8 frames through the front-end one at a time; an empty list gives [0, out] on the host
    lst = [_images(1, h, w, 5 + i)[0] for i, (h, w) in enumerate([(S, S), (80, 96), (32, 48)])]
    devl = _call(log, lambda: m([t.cuda() for t in lst], interpolate_pos_encoding=True), [packed], True, (3, od))
    for lh in (lst, [t.pin_memory() for t in lst], [t.numpy() for t in lst], tuple(t[None] for t in lst)):
        assert torch.equal(_call(log, lambda: m(lh, interpolate_pos_encoding=True), [packed], False, (3, od)), devl.cpu())
    fl = [_frames(1, h, w, 9 + i)[0] for i, (h, w) in enumerate([(S, S), (S, 96)])]
    devfl = _call(log, lambda: m([t.cuda() for t in fl], interpolate_pos_encoding=True), [PRE, PRE, packed], True, (2, od))
    assert torch.equal(_call(log, lambda: m(fl, interpolate_pos_encoding=True), [PRE, PRE, packed], False, (2, od)), devfl.cpu())
    ref2 = m(x[:2].cuda())
    assert torch.equal(_call(log, lambda: m([x[0].cuda(), x[1].cuda()]), [packed], True, (2, od)), ref2)
    _call(log, lambda: m([], interpolate_pos_encoding=True), [], False, (0, od))

    # forward_async: host images of the trained size are left in flight; every other input comes back finished
    p = m.forward_async(x.pin_memory())
    assert log[-1] == "jimm_vit_forward_host" and torch.equal(p.result(), dev.cpu())
    p = m.forward_async(fr.pin_memory())
    assert log[-1] == "jimm_vit_forward_host_u8" and torch.equal(p.result(), dev8.cpu())
    for arg, ref, last in ((x.cuda(), dev, fwd), (y, devy.cpu(), hw), (lst, devl.cpu(), packed)):
        log.clear()
        p = m.forward_async(arg, interpolate_pos_encoding=True)
        assert p.done() and log[-1] == last and torch.equal(p.result(), ref)
    assert FIN not in log


def test_vision_rebuilds(log):
    m = _model("vit")
    m.set_max_batch(2)
    od = 10
    x = _images(1, S, S, 1).cuda()
    _call(log, lambda: m(x), ["jimm_vit_forward"], True, (1, od), builds=1)
    big = _images(1, 320, 256, 2).cuda()  # 321 tokens; the handle holds 2 x 17
    out = _call(log, lambda: m(big, interpolate_pos_encoding=True), ["jimm_vit_forward_hw"], True, (1, od), builds=1)
    _call(log, lambda: m(big, interpolate_pos_encoding=True), ["jimm_vit_forward_hw"], True, (1, od))
    m.set_max_batch(3)  # a later rebuild keeps the raised budget
    lst = [x[0], big[0]]
    packed = _call(log, lambda: m(lst, interpolate_pos_encoding=True), ["jimm_vit_forward_packed"], True, (2, od), builds=1)
    assert torch.equal(packed[1:], out)


# ------------------------------------------------------------------ CLIP / SigLIP
@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_encode_image_and_text(log, kind):
    m = _model(kind)
    n = m.native()
    od, ot = n.vision_out, n.text_out
    enc, hw, packed = "jimm_encode_image", "jimm_encode_image_hw", "jimm_encode_image_packed"

    x = _images(B, S, S, 1)
    dev = _call(log, lambda: m.encode_image(x.cuda()), [enc], True, (B, od))
    assert torch.equal(_call(log, lambda: n.vision(x.cuda(), encode=True), [enc], True, (B, od)), dev)
    for xh in _host_forms(x):
        assert torch.equal(_call(log, lambda: m.encode_image(xh), [enc], False, (B, od)), dev.cpu())
    fr = _frames(B, S, S, 2)
    dev8 = _call(log, lambda: m.encode_image(fr.cuda()), [PRE, enc], True, (B, od))
    assert torch.equal(_call(log, lambda: m.encode_image(fr.pin_memory()), [PRE, enc], False, (B, od)), dev8.cpu())

    y = _images(B, 80, 96, 3)
    devy = _call(log, lambda: m.encode_image(y.cuda(), interpolate_pos_encoding=True), [hw], True, (B, od))
    assert torch.equal(_call(log, lambda: m.encode_image(y, interpolate_pos_encoding=True), [hw], False, (B, od)), devy.cpu())
    fy = _frames(B, S, 96, 4)
    devfy = _call(log, lambda: m.encode_image(fy.cuda(), interpolate_pos_encoding=True), [PRE, hw], True, (B, od))
    assert torch.equal(_call(log, lambda: m.encode_image(fy, interpolate_pos_encoding=True), [PRE, hw], False, (B, od)), devfy.cpu())

    lst = [_images(1, h, w, 5 + i)[0] for i, (h, w) in enumerate([(S, S), (80, 96), (32, 48)])]
    devl = _call(log, lambda: m.encode_image([t.cuda() for t in lst], interpolate_pos_encoding=True), [packed], True, (3, od))
    assert torch.equal(_call(log, lambda: m.encode_image([t.numpy() for t in lst], interpolate_pos_encoding=True), [packed], False, (3, od)),
                       devl.cpu())
    fl = [_frames(1, S, 96, 9)[0], _frames(1, S, S, 10)[0]]
    devfl = _call(log, lambda: m.encode_image([t.cuda() for t in fl], interpolate_pos_encoding=True), [PRE, PRE, packed], True, (2, od))
    assert torch.equal(_call(log, lambda: m.encode_image(fl, interpolate_pos_encoding=True), [PRE, PRE, packed], False, (2, od)), devfl.cpu())

    ids = _ids(4)
    devt = _call(log, lambda: m.encode_text(ids.cuda()), ["jimm_encode_text"], True, (4, ot))
    assert torch.equal(_call(log, lambda: n.text(ids.to(torch.int32).cuda()), ["jimm_encode_text"], True, (4, ot)), devt)
    for ih in (ids, ids.pin_memory(), ids.numpy()):
        assert torch.equal(_call(log, lambda: m.encode_text(ih), ["jimm_encode_text"], False, (4, ot)), devt.cpu())


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_dual_call(log, kind):
    m = _model(kind)
    m.native()
    bt = 4
    ids = _ids(bt)
    idc = ids.cuda()
    shape = (B, bt)

    # trained size
    x = _images(B, S, S, 1)
    dev = _call(log, lambda: m(x.cuda(), idc), ["jimm_dual_forward"], True, shape)
    assert torch.equal(_call(log, lambda: m(x.cuda(), idc, interpolate_pos_encoding=True), ["jimm_dual_forward"], True, shape), dev)
    for xh, ih in ((x, ids), (x.pin_memory(), ids.to(torch.int32).pin_memory()), (x.numpy(), ids.numpy())):
        assert torch.equal(_call(log, lambda: m(xh, ih), ["jimm_dual_forward_host"], False, shape), dev.cpu())
    assert torch.equal(_call(log, lambda: m(x, idc), ["jimm_dual_forward"], True, shape), dev)  # host images, CUDA ids
    assert torch.equal(_call(log, lambda: m(x.cuda(), ids), ["jimm_dual_forward"], True, shape), dev)  # CUDA images, host ids
    fr = _frames(B, S, S, 2)
    dev8 = _call(log, lambda: m(fr.cuda(), idc), [PRE, "jimm_dual_forward"], True, shape)
    assert torch.equal(_call(log, lambda: m(fr.pin_memory(), ids.pin_memory()), [PRE, "jimm_dual_forward"], False, shape), dev8.cpu())
    assert torch.equal(_call(log, lambda: m(fr, idc), [PRE, "jimm_dual_forward"], True, shape), dev8)

    # other sizes
    y = _images(B, 80, 96, 3)
    devy = _call(log, lambda: m(y.cuda(), idc, interpolate_pos_encoding=True), ["jimm_dual_forward_hw"], True, shape)
    assert torch.equal(_call(log, lambda: m(y, ids, interpolate_pos_encoding=True), ["jimm_dual_forward_hw"], False, shape), devy.cpu())
    assert torch.equal(_call(log, lambda: m(y, idc, interpolate_pos_encoding=True), ["jimm_dual_forward_hw"], True, shape), devy)
    assert torch.equal(_call(log, lambda: m(y.cuda(), ids, interpolate_pos_encoding=True), ["jimm_dual_forward_hw"], True, shape), devy)
    fy = _frames(B, S, 96, 4)
    devfy = _call(log, lambda: m(fy.cuda(), idc, interpolate_pos_encoding=True), [PRE, "jimm_dual_forward_hw"], True, shape)
    assert torch.equal(_call(log, lambda: m(fy, ids, interpolate_pos_encoding=True), [PRE, "jimm_dual_forward_hw"], False, shape), devfy.cpu())

    # lists
    seq = ["jimm_encode_image_packed", "jimm_encode_text", "jimm_contrastive_logits"]
    lst = [_images(1, h, w, 5 + i)[0] for i, (h, w) in enumerate([(S, S), (80, 96), (32, 48)])]
    devl = _call(log, lambda: m([t.cuda() for t in lst], idc, interpolate_pos_encoding=True), seq, True, (3, bt))
    assert torch.equal(_call(log, lambda: m(lst, ids, interpolate_pos_encoding=True), seq, False, (3, bt)), devl.cpu())
    assert torch.equal(_call(log, lambda: m(lst, idc, interpolate_pos_encoding=True), seq, True, (3, bt)), devl)
    fl = [_frames(1, S, 96, 9)[0], _frames(1, S, S, 10)[0]]
    devfl = _call(log, lambda: m([t.cuda() for t in fl], idc, interpolate_pos_encoding=True), [PRE, PRE] + seq, True, (2, bt))
    assert torch.equal(_call(log, lambda: m(fl, ids.numpy(), interpolate_pos_encoding=True), [PRE, PRE] + seq, False, (2, bt)), devfl.cpu())


# ------------------------------------------------------------------ bare sub-modules
@pytest.mark.parametrize("kind", ["encoder", "map_head"])
def test_sub_module(log, kind):
    from jimm_b200 import Rngs
    from jimm_b200.common.transformer import Transformer
    from jimm_b200.common.vit import MultiHeadAttentionPoolingHead

    if kind == "encoder":
        m, fwd, shape = Transformer(width=64, mlp_dim=256, layers=2, num_heads=4, rngs=Rngs(0)), "jimm_encoder_forward", (2, 10, 64)
    else:
        m, fwd, shape = MultiHeadAttentionPoolingHead(64, 256, 4, rngs=Rngs(0)), "jimm_map_head_forward", (2, 64)
    x = torch.randn((2, 10, 64), generator=torch.Generator().manual_seed(3))
    dev = _call(log, lambda: m(x.cuda()), [fwd], True, shape, builds=1)
    for xh in _host_forms(x):
        assert torch.equal(_call(log, lambda: m(xh), [fwd], False, shape), dev.cpu())


# ------------------------------------------------------------------ refused inputs
def _on_gpu(x):
    return x.cuda() if isinstance(x, torch.Tensor) else [t.cuda() for t in x]


INVALID = [
    ("rank", lambda: _images(B, S, S, 0)[0], False, "expected images of shape \\[batch, height, width, channels\\]"),
    ("channels", lambda: torch.zeros((B, S, S, 4)), False, "expected NHWC images \\[B,64,64,3\\]"),
    ("channels interpolate", lambda: torch.zeros((B, S, S, 4)), True, "expected NHWC images \\[B,H,W,3\\]"),
    ("size", lambda: torch.zeros((B, 80, S, 3)), False, "expected NHWC images \\[B,64,64,3\\]"),
    ("below a patch", lambda: torch.zeros((B, 12, S, 3)), True, "a 12x64 image is smaller than one 16x16 patch"),
    ("frames channels", lambda: torch.zeros((B, S, S, 4), dtype=torch.uint8), True, "expected uint8 RGB frames"),
    ("frames off the trained size", lambda: torch.zeros((B, S, 96, 3), dtype=torch.uint8), False,
     "the image front-end maps 64x96 frames to 64x96, the model takes 64x64"),
    ("list rank", lambda: [torch.zeros((S, S, 3)), torch.zeros((S, 3))], True, "image 1 of the list: expected \\[height, width, channels\\]"),
    ("list dtypes", lambda: [torch.zeros((S, S, 3)), torch.zeros((S, S, 3), dtype=torch.float16)], True, "must share one dtype"),
    ("list devices", lambda: [torch.zeros((S, S, 3)), torch.zeros((S, S, 3)).cuda()], True, "must be on one device"),
    ("list channels", lambda: [torch.zeros((S, S, 3)), torch.zeros((S, S, 4))], True, "expected NHWC images \\[B,H,W,3\\]"),
    ("list below a patch", lambda: [torch.zeros((S, S, 3)), torch.zeros((S, 8, 3))], True, "smaller than one 16x16 patch"),
    ("list off the trained size", lambda: [torch.zeros((S, S, 3)), torch.zeros((80, S, 3))], False, "expected NHWC images \\[B,64,64,3\\]"),
]


@pytest.mark.parametrize("kind", ["vit", "clip"])
@pytest.mark.parametrize("case,make,interp,msg", INVALID, ids=[c[0] for c in INVALID])
def test_refused_images(log, kind, case, make, interp, msg):
    m = _model(kind)
    ids = _ids(B)
    calls = [lambda x: m(x, interpolate_pos_encoding=interp)] if kind == "vit" else [
        lambda x: m.encode_image(x, interpolate_pos_encoding=interp), lambda x: m(x, ids, interpolate_pos_encoding=interp)]
    for fn in calls:
        for x in (make(), _on_gpu(make())) if case != "list devices" else (make(),):
            with pytest.raises(ValueError, match=msg):
                fn(x)
    assert not [c for c in log if c != FIN]  # nothing ran


@pytest.mark.parametrize("kind", ["vit", "clip"])
def test_frames_need_a_front_end(log, kind):
    m = _model(kind, front_end=False)
    fr = _frames(B, S, S, 1)
    for x in (fr, fr.cuda()):
        for interp in (False, True):
            with pytest.raises(ValueError, match="uint8 images need an image front-end"):
                m(x, interpolate_pos_encoding=interp) if kind == "vit" else m.encode_image(x, interpolate_pos_encoding=interp)
            with pytest.raises(ValueError, match="uint8 images need an image front-end"):
                m([x[0]], interpolate_pos_encoding=interp) if kind == "vit" else m([x[0]], _ids(1), interpolate_pos_encoding=interp)
    assert not [c for c in log if c != FIN]
