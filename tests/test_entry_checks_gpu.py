"""GPU: the checks of the forward entry points (include/jimm_b200.h, "check their arguments in one order").

A refusal table over the ten image and the four text entry points: every check each one runs, and one call with two faults per boundary
between two steps, which pins the documented order.  A refused call returns -1 with the expected message, launches nothing and leaves
its NaN-filled outputs as they were."""

import ctypes as C
import os

import numpy as np
import pytest
import torch

import jimm_oracle as O
from gpu_util import ptr, stream

pytestmark = pytest.mark.gpu
L = 2


def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


@pytest.fixture(scope="module")
def env(golden_dir):
    from jimm_b200 import _lib
    from jimm_b200._runtime import NativeModel
    from jimm_b200.models import CLIP, SigLIP, VisionTransformer

    vcfg = O.ViTCfg(num_classes=16, img_size=64, patch_size=16, num_layers=L, num_heads=4, mlp_dim=512, hidden_size=256)
    vit = _set(VisionTransformer(num_classes=16, img_size=64, patch_size=16, num_layers=L, num_heads=4, mlp_dim=512, hidden_size=256,
                                 dtype=torch.float16), O.random_vit_params(vcfg, seed=0))
    dcfg = O.DualCfg(64, L, 128, 16, 16, 100, 128, 2, L)
    clip = _set(CLIP(64, L, 128, 16, 16, 100, 128, 2, L, dtype=torch.float16), O.random_dual_params(dcfg, "clip", seed=1))
    d = os.path.join(golden_dir, "tiny_siglip2_naflex")
    nf = SigLIP.from_pretrained(os.path.join(d, "model.safetensors"), dtype=torch.float16)
    io = dict(np.load(os.path.join(d, "io.npz")))
    # a bare encoder: a handle with neither tower
    cfg = _lib.Config()
    cfg.kind, cfg.v_width, cfg.v_heads, cfg.v_mlp, cfg.v_layers, cfg.v_act = _lib.KIND_ENCODER, 64, 1, 128, 1, _lib.ACT_GELU_TANH
    cfg.v_eps_block = cfg.v_eps_outer = 1e-6
    cfg.ctx_len = 8
    p = {}
    O._rand_blocks(p, torch.Generator().manual_seed(3), "", 1, 64, 1, 128)
    enc = NativeModel(cfg, O.cast_params(p, torch.float32), 2)
    models = (vit, clip, nf, enc)  # the handles live as long as their models
    lib = _lib.load()
    hv, hc, hn = (m.native().handle for m in models[:3])
    img = O.synthetic_images(2, 64).cuda()
    ids = O.synthetic_tokens(2, 16, 100, "clip").to(torch.int32).cuda()
    pv = torch.from_numpy(io["pixel_values"][:2]).cuda()
    good = [v for hw in io["spatial_shapes"][:2].tolist() for v in hw]
    sink = torch.full((4096, 256), float("nan"), device="cuda")
    out = torch.full((2, 128), float("nan"), device="cuda")

    def req(layer):
        return C.byref(_lib.TokensReq(1, (C.c_int * 1)(layer), (C.c_void_p * 1)(sink.data_ptr()), 0))

    ints = lambda *v: (C.c_int * len(v))(*v)  # noqa: E731
    imgs = (C.c_void_p * 2)(img.data_ptr(), img.data_ptr())
    return dict(lib=lib, hv=hv, hc=hc, hn=hn, he=enc.handle, img=ptr(img), ids=ptr(ids), pv=ptr(pv), N=pv.shape[1], grid=ints(*good),
                imgs=imgs, HW=ints(64, 64), sink=sink, out=out, req=req, ints=ints, models=models)


# Each image entry point as f(e, handle, img, dtype, B, out, req, shape): img is its input (a batch, a list or NaFlex rows) and shape its
# per-form sizes (H, W for a batch, the (H, W) arrays for a list, the grid for NaFlex rows); None takes the entry point's good value.
def _image_calls():
    def dense(name, vit, tokens, hw=True):
        def f(e, h, img, dt, B, out, req, shape):
            H, W = (64, 64) if shape is None else shape
            if tokens:
                return getattr(e["lib"], name)(h, img, dt, B, H, W, req, out, stream())
            if hw:
                return getattr(e["lib"], name)(h, img, dt, B, H, W, out, stream())
            return getattr(e["lib"], name)(h, img, dt, B, out, stream())
        return dict(fn=f, form="dense", vit=vit, tokens=tokens, hw=hw or tokens)

    def lst(name, vit, tokens):
        def f(e, h, img, dt, B, out, req, shape):
            H, W = (e["HW"], e["HW"]) if shape is None else shape
            args = (h, img, dt, B, H, W) + ((req,) if tokens else ())
            return getattr(e["lib"], name)(*args, out, stream())
        return dict(fn=f, form="list", vit=vit, tokens=tokens)

    def rows(name, tokens):
        def f(e, h, img, dt, B, out, req, shape):
            args = (h, img, dt, B, e["N"], e["grid"] if shape is None else shape) + ((req,) if tokens else ())
            return getattr(e["lib"], name)(*args, out, stream())
        return dict(fn=f, form="rows", vit=False, tokens=tokens)

    return {
        "jimm_vit_forward": dense("jimm_vit_forward", True, False, hw=False),
        "jimm_encode_image": dense("jimm_encode_image", False, False, hw=False),
        "jimm_vit_forward_hw": dense("jimm_vit_forward_hw", True, False),
        "jimm_encode_image_hw": dense("jimm_encode_image_hw", False, False),
        "jimm_image_tokens": dense("jimm_image_tokens", False, True),
        "jimm_vit_forward_packed": lst("jimm_vit_forward_packed", True, False),
        "jimm_encode_image_packed": lst("jimm_encode_image_packed", False, False),
        "jimm_image_tokens_packed": lst("jimm_image_tokens_packed", False, True),
        "jimm_encode_image_patches": rows("jimm_encode_image_patches", False),
        "jimm_image_tokens_patches": rows("jimm_image_tokens_patches", True),
    }


IMAGE = _image_calls()


def _refused(e, call, msg):
    torch.cuda.synchronize()
    n0 = e["lib"].jimm_launch_count()
    rc = call()
    torch.cuda.synchronize()
    err = e["lib"].jimm_last_error().decode()
    assert rc == -1, (rc, err)
    assert msg in err, (msg, err)
    assert e["lib"].jimm_launch_count() == n0, "a refused call launched kernels"
    assert torch.isnan(e["out"]).all() and torch.isnan(e["sink"]).all(), "a refused call wrote its outputs"


@pytest.mark.parametrize("name", list(IMAGE))
def test_image_entry_refusals(env, name):
    e, c = env, IMAGE[name]
    good_h = e["hn"] if c["form"] == "rows" else e["hv"] if c["vit"] else e["hc"]
    good_in = {"dense": e["img"], "list": e["imgs"], "rows": e["pv"]}[c["form"]]
    out, req = ptr(e["out"]), e["req"](0)

    def call(h=good_h, img=good_in, dt=0, B=2, out=out, req=req, shape=None):
        return lambda: c["fn"](e, h, img, dt, B, out, req, shape)

    bad_shape = {"dense": (8, 64), "list": (e["ints"](64, 8), e["HW"]), "rows": e["ints"](17, 16, 4, 4)}[c["form"]]
    shape_msg = {"dense": "smaller than one", "list": "smaller than one", "rows": "more than its N"}[c["form"]]
    bad_tower = e["hc"] if c["vit"] or c["form"] == "rows" else e["he"]
    tower_msg = "not a SigLIP 2 NaFlex" if c["form"] == "rows" else "on a dual-tower model" if c["vit"] else "model has no vision tower"
    null = f"{name}: null argument"

    # 1. the handle
    _refused(e, call(h=None), "null model")
    _refused(e, call(B=-1), "negative batch")
    # 2. the image dtype
    _refused(e, call(dt=7), "bad image dtype 7")
    # 3. the tower
    _refused(e, call(h=bad_tower), tower_msg)
    # 4. the request
    if c["tokens"]:
        _refused(e, call(req=None), f"{name}: null request")
        _refused(e, call(req=e["req"](9)), "asks for layer 9")
    # 5. null arguments: the inputs always, out on the pooled calls
    _refused(e, call(img=None), null)
    if not c["tokens"]:
        _refused(e, call(out=None), null)
    if c["form"] == "list":
        _refused(e, call(shape=(None, e["HW"])), null)
    if c["form"] == "rows":
        _refused(e, call(shape=C.POINTER(C.c_int)()), null)
    # 6. the shapes
    if c["form"] != "dense" or c["hw"]:
        _refused(e, call(shape=bad_shape), shape_msg)
    if c["form"] == "list":
        _refused(e, call(img=(C.c_void_p * 2)(e["imgs"][0], None)), "image 1 is a null pointer")
    if c["form"] == "rows":
        _refused(e, call(shape=e["ints"](0, 4, 4, 4)), "each edge from 1 up")

    # two faults, one per boundary: the earlier step reports
    _refused(e, call(B=-1, dt=7), "negative batch")                                   # 1 | 2
    _refused(e, call(dt=7, h=bad_tower), "bad image dtype 7")                         # 2 | 3
    if c["tokens"]:
        _refused(e, call(h=bad_tower, req=e["req"](9)), tower_msg)                   # 3 | 4
    else:
        _refused(e, call(h=bad_tower, img=None), tower_msg)                          # 3 | 5
    if c["tokens"]:
        _refused(e, call(req=e["req"](9), img=None), "asks for layer 9")              # 4 | 5
    if c["form"] != "dense" or c["hw"]:
        _refused(e, call(img=None, shape=bad_shape), null)                             # 5 | 6

    # a per-token call's pooled output is optional; B = 0 takes null inputs
    if c["tokens"]:
        torch.cuda.synchronize()
        assert c["fn"](e, good_h, good_in, 0, 2, None, req, None) == 0
        torch.cuda.synchronize()
        e["sink"].fill_(float("nan"))
    assert c["fn"](e, good_h, None, 0, 0, None, req, None) == 0


TEXT = {
    "jimm_encode_text": (False, False),
    "jimm_encode_text_packed": (True, False),
    "jimm_text_tokens": (False, True),
    "jimm_text_tokens_packed": (True, True),
}


@pytest.mark.parametrize("name", list(TEXT))
def test_text_entry_refusals(env, name):
    e = env
    packed, tokens = TEXT[name]
    fn = getattr(e["lib"], name)
    out = ptr(e["out"])
    good_shape = e["ints"](5, 16) if packed else 16
    bad_shape = e["ints"](5, 0) if packed else 17
    shape_msg = "length 0 outside" if packed else "sequence length 17 outside (0, context_length=16]"

    def call(h=e["hc"], ids=e["ids"], B=2, shape=good_shape, out=out, req=e["req"](0)):
        return lambda: fn(h, ids, B, shape, *((req,) if tokens else ()), out, stream())

    null = f"{name}: null argument"
    _refused(e, call(h=None), "null model")                                            # 1
    _refused(e, call(B=-1), "negative batch")
    _refused(e, call(h=e["hv"]), "no text tower")                                      # 3
    if tokens:                                                                          # 4
        _refused(e, call(req=None), f"{name}: null request")
        _refused(e, call(req=e["req"](9)), "asks for layer 9")
    _refused(e, call(ids=None), null)                                                   # 5
    if packed:
        _refused(e, call(shape=None), null)
    if not tokens:
        _refused(e, call(out=None), null)
    _refused(e, call(shape=bad_shape), shape_msg)                                       # 6

    _refused(e, call(B=-1, h=e["hv"]), "negative batch")                               # 1 | 3
    if tokens:
        _refused(e, call(h=e["hv"], req=e["req"](9)), "no text tower")                 # 3 | 4
        _refused(e, call(req=e["req"](9), ids=None), "asks for layer 9")               # 4 | 5
    else:
        _refused(e, call(h=e["hv"], ids=None), "no text tower")                        # 3 | 5
    _refused(e, call(ids=None, shape=bad_shape), null)                                  # 5 | 6

    if tokens:
        torch.cuda.synchronize()
        assert fn(e["hc"], e["ids"], 2, good_shape, e["req"](0), None, stream()) == 0
        torch.cuda.synchronize()
        e["sink"].fill_(float("nan"))
    assert fn(e["hc"], None, 0, good_shape, *((e["req"](0),) if tokens else ()), None, stream()) == 0
