"""GPU: per-token hidden states (forward_tokens / encode_image_tokens / encode_text_tokens, jimm_image_tokens* / jimm_text_tokens*).

The copy kernel against torch's casts; every layer against the CPU oracle (tests/tokens_oracle.py) at the project's bars, recorded in
PARITY.md; return_pooled against the pooled calls bit for bit on every input form; the pooled calls' bits, launch counts and graph
replays unchanged by token calls; packed rows equal to each sample alone; the early exit against a model of fewer blocks; 16-bit
outputs against the fp32 output's casts; the PDL ordering of the copy; and refused calls enqueuing nothing."""

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import jimm_oracle as O
import naflex_oracle as NF
import tokens_oracle as TO
from gpu_util import check, check_parity, ptr, stream

pytestmark = pytest.mark.gpu
TOL = 1e-3  # north_star: 1e-3 relative vs the fp32 oracle
BF16_VS_SAME = 8e-3  # bf16 operands, against the oracle with the same operand rounding
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = 3  # blocks of the test towers
LAYERS = [0, 1, L - 1, L, None]
BAR = {torch.float32: TOL, torch.float16: TOL, torch.bfloat16: BF16_VS_SAME, torch.float8_e4m3fn: None}
ROUND = {torch.float32: "tf32", torch.float16: "fp16", torch.bfloat16: "bf16", torch.float8_e4m3fn: None}


def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


def _name(k):
    return "final" if k is None else f"x_{k}"


# ------------------------------------------------------------------ the copy kernel
@pytest.mark.parametrize("D", [8, 64, 264, 768, 1152, 2048])
@pytest.mark.parametrize("out_type", [0, 1, 2])
def test_tokens_out_kernel(lib, D, out_type):
    dt = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16}[out_type]
    g = torch.Generator().manual_seed(D)
    for rows in (1, 3, 257, 1001):
        x = torch.randn((rows, D), generator=g) * 300
        x[0, :4] = torch.tensor([70000.0, -1e-30, 65519.0, 3.0e38])  # fp16 overflow, subnormal, the fp16 rounding edge, bf16 range
        x = x.cuda()
        out = torch.full((rows + 2, D), 7, dtype=dt, device="cuda")
        check(lib, lib.jimm_k_tokens_out(ptr(x), rows, D, ptr(out), out_type, stream()))
        torch.cuda.synchronize()
        ref = x.to(dt)
        iv = torch.int32 if dt == torch.float32 else torch.int16
        assert torch.equal(out[:rows].view(iv), ref.view(iv)), (D, rows)
        assert (out[rows:] == 7).all(), "rows past the end were written"


# ------------------------------------------------------------------ models
def _vit(dtype, layers=L, params=None):
    from jimm_b200.models import VisionTransformer

    cfg = O.ViTCfg(num_classes=16, img_size=64, patch_size=16, num_layers=L, num_heads=4, mlp_dim=512, hidden_size=256)
    p = params if params is not None else O.random_vit_params(cfg, seed=0, dtype=torch.float64)
    m = VisionTransformer(num_classes=16, img_size=64, patch_size=16, num_layers=layers, num_heads=4, mlp_dim=512, hidden_size=256, dtype=dtype)
    _set(m, {k: v for k, v in p.items() if not k.startswith("encoder.transformer.blocks.layers.") or int(k.split(".")[4]) < layers})
    return m, cfg, p


DCFG = O.DualCfg(64, L, 128, 16, 16, 100, 128, 2, L)


def _dual(kind, dtype):
    from jimm_b200.models import CLIP, SigLIP

    p = O.random_dual_params(DCFG, kind, seed=1, dtype=torch.float64)
    m = (CLIP if kind == "clip" else SigLIP)(64, L, 128, 16, 16, 100, 128, 2, L, dtype=dtype)
    return _set(m, p), p


def _naflex(golden_dir, dtype):
    from safetensors.torch import load_file

    from jimm_b200.models import SigLIP

    d = os.path.join(golden_dir, "tiny_siglip2_naflex")
    m = SigLIP.from_pretrained(os.path.join(d, "model.safetensors"), dtype=dtype)
    cfg = NF.dual_cfg(NF.tiny_siglip2_config())
    p = O.cast_params(NF.hf_to_flax_siglip2(load_file(os.path.join(d, "model.safetensors")), cfg), torch.float64)
    return m, cfg, p, dict(np.load(os.path.join(d, "io.npz")))


def _check_layers(case, dtype, outs, refs, same=None):
    """outs[i] (CUDA, request LAYERS[i]) against refs (fp32 oracle, [x_0 .. x_L, final]) and, for bf16, same (the same-rounding
    oracle); FP8 reported only."""
    for k, o in zip(LAYERS, outs):
        r = refs[-1] if k is None else refs[k]
        if dtype == torch.bfloat16:
            rs = same[-1] if k is None else same[k]
            check_parity(case, f"tokens {_name(k)}", dtype, "same-rounding", o, rs, BF16_VS_SAME)
            check_parity(case, f"tokens {_name(k)}", dtype, "fp32", o, r, None)
        else:
            check_parity(case, f"tokens {_name(k)}", dtype, "fp32", o, r, BAR[dtype])


# ------------------------------------------------------------------ parity against the oracle
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn])
def test_parity_vit(dtype):
    m, cfg, p = _vit(dtype)
    img = O.synthetic_images(3, 64)
    with torch.no_grad():
        refs = TO.vit_hidden(p, cfg, img.double())
        same = TO.vit_hidden(p, cfg, img.double(), O.Semantics(operand_round=ROUND[dtype])) if dtype == torch.bfloat16 else None
    outs = m.forward_tokens(img.cuda(), LAYERS)
    assert isinstance(outs, tuple) and all(o.shape == (3, 17, 256) and o.dtype == torch.float32 for o in outs)
    _check_layers("ViT 3x256 (CLS, no ln_pre) 64px B=3", dtype, outs, refs, same)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn])
@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_parity_dual(kind, dtype):
    m, p = _dual(kind, dtype)
    img = O.synthetic_images(2, 64)
    txt = O.synthetic_tokens(3, 16, 100, kind)
    vis = TO.clip_image_hidden if kind == "clip" else TO.siglip_image_hidden
    txh = TO.clip_text_hidden if kind == "clip" else TO.siglip_text_hidden
    sem = O.Semantics(operand_round=ROUND[dtype])
    with torch.no_grad():
        ri, rt = vis(p, DCFG, img.double()), txh(p, DCFG, txt)
        si, st = (vis(p, DCFG, img.double(), sem), txh(p, DCFG, txt, sem)) if dtype == torch.bfloat16 else (None, None)
    oi = m.encode_image_tokens(img.cuda(), LAYERS)
    ot = m.encode_text_tokens(txt.cuda(), LAYERS)
    S = 16 + (kind == "clip")
    assert all(o.shape == (2, S, 128) for o in oi) and all(o.shape == (3, 16, 128) for o in ot)
    tower = "CLS, ln_pre" if kind == "clip" else "MAP"
    _check_layers(f"{kind.upper()} vision 3x128 ({tower}) 64px B=2", dtype, oi, ri, si)
    _check_layers(f"{kind.upper()} text 3x128 T=16 B=3", dtype, ot, rt, st)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn])
def test_parity_naflex(golden_dir, dtype):
    m, cfg, p, io = _naflex(golden_dir, dtype)
    pv, shapes = torch.from_numpy(io["pixel_values"]), io["spatial_shapes"]
    Lv = cfg.vision_layers
    layers = [0, 1, Lv - 1, Lv, None]
    with torch.no_grad():
        refs = TO.naflex_hidden(p, cfg, pv.double(), shapes)
        same = TO.naflex_hidden(p, cfg, pv.double(), shapes, O.Semantics(operand_round="bf16")) if dtype == torch.bfloat16 else None
    outs = m.encode_image_tokens(pv.cuda(), layers, spatial_shapes=shapes)
    for i, k in enumerate(layers):
        assert [o.shape[0] for o in outs[i]] == [h * w for h, w in shapes.tolist()]
        j = -1 if k is None else k
        o, r = torch.cat(outs[i]), torch.cat([x[j] for x in refs])
        case = "golden tiny_siglip2_naflex vision, padded mixed shapes"
        if dtype == torch.bfloat16:
            check_parity(case, f"tokens {_name(k)}", dtype, "same-rounding", o, torch.cat([x[j] for x in same]), BF16_VS_SAME)
            check_parity(case, f"tokens {_name(k)}", dtype, "fp32", o, r, None)
        else:
            check_parity(case, f"tokens {_name(k)}", dtype, "fp32", o, r, BAR[dtype])


def test_parity_fused_layernorm(monkeypatch):
    """JIMM_FUSE_LN=1 (read when a handle is built): the out-proj / FC2 epilogues normalise the rows they complete."""
    monkeypatch.setenv("JIMM_FUSE_LN", "1")
    m, cfg, p = _vit(torch.float16)
    img = O.synthetic_images(3, 64)
    with torch.no_grad():
        refs = TO.vit_hidden(p, cfg, img.double())
    _check_layers("ViT 3x256 64px B=3, JIMM_FUSE_LN=1", torch.float16, m.forward_tokens(img.cuda(), LAYERS), refs)
    pooled = m(img.cuda())
    assert torch.equal(m.forward_tokens(img.cuda(), 1, return_pooled=True)[1], pooled)


# ------------------------------------------------------------------ return_pooled: the pooled calls' bits on every input form
def test_return_pooled_bits_vision():
    m, _, _ = _vit(torch.float16)
    g = torch.Generator().manual_seed(3)
    small = torch.randn((4, 64, 64, 3), generator=g).cuda()
    for _ in range(3):  # the pooled call of B = 4 is graph-replayed from its second call on
        ref = m(small)
    for layers in (0, None, [2, None]):
        assert torch.equal(m.forward_tokens(small, layers, return_pooled=True)[1], ref)
    # host input: host results
    toks, pooled = m.forward_tokens(small.cpu(), 1, return_pooled=True)
    assert not toks.is_cuda and not pooled.is_cuda and torch.equal(pooled, ref.cpu())
    assert torch.equal(toks, m.forward_tokens(small, 1).cpu())
    # interpolate_pos_encoding at another size
    hw = torch.randn((3, 48, 80, 3), generator=g).cuda()
    toks, pooled = m.forward_tokens(hw, [0, None], return_pooled=True, interpolate_pos_encoding=True)
    assert toks[0].shape == (3, 1 + 3 * 5, 256) and torch.equal(pooled, m(hw, interpolate_pos_encoding=True))
    # a packed list
    lst = [torch.randn((h, w, 3), generator=g).cuda() for h, w in [(64, 64), (32, 96), (80, 48)]]
    toks, pooled = m.forward_tokens(lst, None, return_pooled=True, interpolate_pos_encoding=True)
    assert [t.shape[0] for t in toks] == [17, 13, 16] and torch.equal(pooled, m(lst, interpolate_pos_encoding=True))
    # B past max_batch
    m.set_max_batch(4)
    big = torch.randn((9, 64, 64, 3), generator=g).cuda()
    toks, pooled = m.forward_tokens(big, [L, None], return_pooled=True)
    assert torch.equal(pooled, m(big))
    one = [m.forward_tokens(big[i:i + 1], [L, None]) for i in range(9)]
    for j in range(2):
        assert torch.equal(toks[j], torch.cat([o[j] for o in one]))


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_return_pooled_bits_dual(kind):
    m, _ = _dual(kind, torch.float16)
    img = O.synthetic_images(5, 64).cuda()
    txt = O.synthetic_tokens(6, 16, 100, kind).cuda()
    for _ in range(3):
        ri, rt = m.encode_image(img), m.encode_text(txt)
    assert torch.equal(m.encode_image_tokens(img, 1, return_pooled=True)[1], ri)
    assert torch.equal(m.encode_text_tokens(txt, [0, None], return_pooled=True)[1], rt)
    seqs = [txt[i, : 4 + 2 * i] for i in range(6)]
    toks, pooled = m.encode_text_tokens(seqs, [1, None], return_pooled=True)
    assert torch.equal(pooled, m.encode_text(seqs))
    for i, s in enumerate(seqs):  # packed rows equal the sequence alone
        alone = m.encode_text_tokens(s[None], [1, None])
        for j in range(2):
            assert torch.equal(toks[j][i], alone[j][0]), (i, j)
    # host ids
    toks, pooled = m.encode_text_tokens(txt.cpu(), None, return_pooled=True)
    assert not toks.is_cuda and torch.equal(pooled, rt.cpu())


def test_return_pooled_bits_naflex(golden_dir):
    m, cfg, p, io = _naflex(golden_dir, torch.float16)
    pv, shapes = torch.from_numpy(io["pixel_values"]).cuda(), io["spatial_shapes"]
    ref = m.encode_image(pv, spatial_shapes=shapes)
    toks, pooled = m.encode_image_tokens(pv, [1, None], return_pooled=True, spatial_shapes=shapes)
    assert torch.equal(pooled, ref)
    P = cfg.vision_patch_size
    for b, (h, w) in enumerate(shapes.tolist()):  # each sample alone, as pixel_values and as the NHWC image its rows cut
        one = m.encode_image_tokens(pv[b:b + 1, : h * w], [1, None], spatial_shapes=shapes[b:b + 1])
        img = NF.rows_to_image(pv[b, : h * w].cpu(), h, w, P)[None].cuda()
        hwc = m.encode_image_tokens(img, [1, None])
        for j in range(2):
            assert torch.equal(toks[j][b], one[j][0]) and torch.equal(toks[j][b], hwc[j][0]), (b, j)


# ------------------------------------------------------------------ the pooled calls are unchanged
def test_pooled_calls_unchanged_by_token_calls(lib):
    m, p = _dual("clip", torch.float16)
    img = O.synthetic_images(4, 64).cuda()
    txt = O.synthetic_tokens(4, 16, 100, "clip").cuda()

    def launches(fn):
        torch.cuda.synchronize()
        n0, g0 = lib.jimm_launch_count(), lib.jimm_graph_replay_count()
        out = fn()
        torch.cuda.synchronize()
        return out, lib.jimm_launch_count() - n0, lib.jimm_graph_replay_count() - g0

    calls = [lambda: m.encode_image(img), lambda: m.encode_text(txt), lambda: m(img, txt)]
    for fn in calls:  # first call eager, second captured, later ones replayed
        fn(), fn()
    before = [launches(fn) for fn in calls]
    for _, n, r in before:
        assert r >= 1  # replayed
    for _ in range(2):
        _, n, r = launches(lambda: m.encode_image_tokens(img, [0, 2, None], return_pooled=True))
        assert r == 0 and n > 0
        _, n, r = launches(lambda: m.encode_text_tokens(txt, [1, None], return_pooled=True))
        assert r == 0 and n > 0
    after = [launches(fn) for fn in calls]
    for (o0, n0, r0), (o1, n1, r1) in zip(before, after):
        assert torch.equal(o0, o1) and n0 == n1 and r0 == r1


# ------------------------------------------------------------------ packed = alone, chunking past max_batch and the token budget
def test_packed_chunks_put_rows_at_their_offsets():
    m, _, _ = _vit(torch.float32)
    m.set_max_batch(2)  # the token budget: 2 x 17 rows per chunk
    g = torch.Generator().manual_seed(4)
    sizes = [(64, 64), (16, 16), (96, 96), (32, 64), (64, 64), (48, 16), (16, 112)]
    lst = [torch.randn((h, w, 3), generator=g).cuda() for h, w in sizes]
    toks = m.forward_tokens(lst, [0, 2, None], interpolate_pos_encoding=True)
    for i, x in enumerate(lst):
        alone = m.forward_tokens(x[None], [0, 2, None], interpolate_pos_encoding=True)
        for j in range(3):
            assert torch.equal(toks[j][i], alone[j][0]), (sizes[i], j)
    assert toks[0][0].untyped_storage().data_ptr() == toks[0][-1].untyped_storage().data_ptr()  # views of one packed buffer


def test_text_packed_chunks_past_the_budget():
    m, _ = _dual("clip", torch.float16)
    m.set_max_batch(2)  # 2 x 16 token rows per chunk
    txt = O.synthetic_tokens(7, 16, 100, "clip")
    seqs = [txt[i, : n].cuda() for i, n in enumerate([16, 3, 9, 16, 1, 12, 7])]
    toks = m.encode_text_tokens(seqs, [2, None])
    for i, s in enumerate(seqs):
        alone = m.encode_text_tokens(s[None], [2, None])
        for j in range(2):
            assert torch.equal(toks[j][i], alone[j][0]), (i, j)
    dense = m.encode_text_tokens(txt.cuda(), [2, None])  # 7 rows of 16 past max_batch: chunks of 2
    for i in range(7):
        alone = m.encode_text_tokens(txt[i:i + 1].cuda(), [2, None])
        for j in range(2):
            assert torch.equal(dense[j][i], alone[j][0])


# ------------------------------------------------------------------ early exit
def test_early_exit_bits_and_launches(lib):
    full, cfg, p = _vit(torch.float16)
    img = O.synthetic_images(3, 64).cuda()

    def launches(m, k):
        torch.cuda.synchronize()
        n0 = lib.jimm_launch_count()
        out = m.forward_tokens(img, k)
        torch.cuda.synchronize()
        return out, lib.jimm_launch_count() - n0

    full.native()  # the handle is built (and its weights uploaded) outside the counted calls
    counts = {}
    for k in range(L + 1):
        out, counts[k] = launches(full, k)
        if 0 < k < L:
            part, _, _ = _vit(torch.float16, layers=k, params=p)
            assert torch.equal(out, launches(part, k)[0]), k
    per_block = counts[L] - counts[L - 1]
    assert per_block == 7  # LayerNorm, QKV, attention, out-projection, LayerNorm, FC1, FC2
    for k in range(L + 1):
        assert counts[L] - counts[k] == (L - k) * per_block, counts


# ------------------------------------------------------------------ 16-bit outputs are the fp32 output's casts
@pytest.mark.parametrize("kind", ["vit", "clip"])
def test_16bit_outputs_equal_fp32_casts(kind):
    if kind == "vit":
        m, _, _ = _vit(torch.float16)
        img = O.synthetic_images(3, 64).cuda()
        run = lambda dt: m.forward_tokens(img, LAYERS, dtype=dt)
    else:
        m, _ = _dual("clip", torch.bfloat16)
        txt = O.synthetic_tokens(3, 16, 100, "clip").cuda()
        run = lambda dt: m.encode_text_tokens(txt, LAYERS, dtype=dt)
    ref = run(torch.float32)
    for dt in (torch.float16, torch.bfloat16):
        out = run(dt)
        for k, o, r in zip(LAYERS, out, ref):
            assert o.dtype == dt and torch.equal(o.view(torch.int16), r.to(dt).view(torch.int16)), (kind, dt, k)


# ------------------------------------------------------------------ ordering: the copy waits for the block that wrote x
_PDL_SCRIPT = r"""
import sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/oracle")
import jimm_oracle as O
from jimm_b200.models import VisionTransformer
p = O.random_vit_params(O.ViTCfg(), seed=0)
m = VisionTransformer(dtype=torch.float16)
for k, v in p.items():
    m.set_flat_param(k, v)
img = O.synthetic_images(8, 224).cuda()
torch.save([t.cpu() for t in m.forward_tokens(img, [0, 1, 6, 12, None], dtype=torch.float16)], sys.argv[2])
"""


def test_pdl_off_gives_the_same_bits(tmp_path):
    """JIMM_PDL is read once per process: a fresh interpreter with it off against one with the default."""
    outs = []
    for pdl in ("0", "1"):
        f = tmp_path / f"pdl{pdl}.pt"
        env = dict(os.environ, JIMM_PDL=pdl)
        r = subprocess.run([sys.executable, "-c", _PDL_SCRIPT, ROOT, str(f)], env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(torch.load(f))
    for a, b in zip(*outs):
        assert a.shape == (8, 197, 768) and torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------ refusals
def test_refused_calls_enqueue_nothing(lib, golden_dir):
    from jimm_b200._lib import TokensReq

    vit, _, _ = _vit(torch.float16)
    clip, _ = _dual("clip", torch.float16)
    nf, _, _, io = _naflex(golden_dir, torch.float16)
    hv, hc, hn = vit.native().handle, clip.native().handle, nf.native().handle
    img = O.synthetic_images(2, 64).cuda()
    ids = O.synthetic_tokens(2, 16, 100, "clip").to(torch.int32).cuda()
    buf = torch.full((4096, 256), float("nan"), device="cuda")
    pooled = torch.full((2, 16), float("nan"), device="cuda")

    def req(layers, dtype=0, out=None, n=None):
        outs = out if out is not None else [buf.data_ptr()] * len(layers)
        k = len(layers)
        return TokensReq(k if n is None else n, (C.c_int * max(k, 1))(*layers), (C.c_void_p * max(k, 1))(*outs), dtype)

    def refused(fn, msg=""):
        torch.cuda.synchronize()
        n0 = lib.jimm_launch_count()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == -1 and lib.jimm_launch_count() == n0
        assert msg in lib.jimm_last_error().decode(), lib.jimm_last_error().decode()

    im = lambda h, r, H=64, W=64: lambda: lib.jimm_image_tokens(h, ptr(img), 0, 2, H, W, C.byref(r), ptr(pooled), stream())
    refused(im(hv, req([L + 1])), "outside 0 .. 3")
    refused(im(hv, req([-2])), "outside 0 .. 3")
    refused(im(hv, req([0], n=0)), "layer requests")
    refused(im(hv, req([0] * (L + 3))), "layer requests")
    refused(im(hv, req([0], dtype=3)), "output dtype")
    refused(im(hv, req([0], dtype=4)), "output dtype")
    refused(im(hv, req([0], out=[0])), "null or not 16-byte aligned")
    refused(im(hv, req([0], out=[buf.data_ptr() + 4])), "null or not 16-byte aligned")
    refused(lambda: lib.jimm_image_tokens(hv, ptr(img), 0, 2, 64, 64, None, ptr(pooled), stream()), "null request")
    refused(im(hv, req([0]), H=8, W=64), "smaller than one")  # the pooled call's refusals
    refused(lambda: lib.jimm_image_tokens(hv, ptr(img), 7, 2, 64, 64, C.byref(req([0])), ptr(pooled), stream()), "bad image dtype")
    refused(lambda: lib.jimm_text_tokens(hv, ptr(ids), 2, 16, C.byref(req([0])), None, stream()), "no text tower")
    refused(lambda: lib.jimm_text_tokens(hc, ptr(ids), 2, 17, C.byref(req([0])), None, stream()), "context_length")
    refused(lambda: lib.jimm_text_tokens(hc, ptr(ids), 2, 16, C.byref(req([L + 1])), None, stream()), "outside 0 .. 3")
    lens = (C.c_int * 2)(5, 0)
    refused(lambda: lib.jimm_text_tokens_packed(hc, ptr(ids), 2, lens, C.byref(req([0])), None, stream()), "length 0")
    H2, W2 = (C.c_int * 2)(64, 8), (C.c_int * 2)(64, 64)
    ptrs = (C.c_void_p * 2)(img.data_ptr(), img.data_ptr())
    refused(lambda: lib.jimm_image_tokens_packed(hv, ptrs, 0, 2, H2, W2, C.byref(req([0])), None, stream()), "smaller than one")
    pv = torch.from_numpy(io["pixel_values"]).cuda()
    good = [v for hw in io["spatial_shapes"].tolist() for v in hw]
    B, N = pv.shape[0], pv.shape[1]
    bad = (C.c_int * (2 * B))(*([17, 16] + good[2:]))
    refused(lambda: lib.jimm_image_tokens_patches(hn, ptr(pv), 0, B, N, bad, C.byref(req([0])), None, stream()), "more than its N")
    okg = (C.c_int * (2 * B))(*good)
    refused(lambda: lib.jimm_image_tokens_patches(hc, ptr(pv), 0, B, N, okg, C.byref(req([0])), None, stream()), "not a SigLIP 2 NaFlex")
    refused(lambda: lib.jimm_image_tokens_patches(hn, ptr(pv), 0, B, N, okg, C.byref(req([3])), None, stream()), "outside 0 .. 2")
    assert torch.isnan(buf).all() and torch.isnan(pooled).all()
