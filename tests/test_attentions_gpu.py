"""GPU: attention weights (forward_attentions / encode_image_attentions / encode_text_attentions, jimm_image_attn* / jimm_text_attn*).

The probs kernel against an fp64 softmax of the same qkv bits at every head width, sequence length, mask, layout and dtype; the MAP
head's probe weights likewise; every block and the MAP weights against the CPU oracle (tests/attn_oracle.py) at the project's bars,
recorded in PARITY.md; return_pooled against the pooled calls bit for bit on every input form; the pooled calls' bits, launch counts and
graph replays unchanged by attention calls; packed samples equal to each sample alone; the early exit; host results; the PDL ordering;
a NaN image leaving its neighbours alone; one request of more than 2^31 elements; and refused calls enqueuing nothing."""

import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import attn_oracle as AO
import jimm_oracle as O
import naflex_oracle as NF
from gpu_util import CODE, check, check_parity, ptr, stream

pytestmark = pytest.mark.gpu
# Twice the hidden-state bars (1e-3; bf16 8e-3 against the same-rounding oracle): the weights of block k carry the rounding of every
# block before it, and the softmax turns an absolute score error e into a relative weight error e.  Block 0, whose input matches the
# oracle's, stays near 1e-4 in fp32 / fp16; the third block of the test towers reaches 1.1e-3 in fp16 and 8.1e-3 in bf16 (H100).
TOL = 2e-3
BF16_VS_SAME = 1.6e-2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = 3  # blocks of the test towers
BAR = {torch.float32: TOL, torch.float16: TOL, torch.bfloat16: BF16_VS_SAME, torch.float8_e4m3fn: None}
ROUND = {torch.float32: "tf32", torch.float16: "fp16", torch.bfloat16: "bf16", torch.float8_e4m3fn: None}
QK = {torch.float32: "fp16", torch.float16: "fp16", torch.bfloat16: "bf16", torch.float8_e4m3fn: "fp16"}  # the attention I/O type


def _same(dtype):
    """The oracle rounded as the CUDA path of `dtype` rounds: GEMM operands, and q / k in the attention I/O type its weights are
    computed on (fp16 even in the fp32 mode, so the plain fp32 oracle differs from them by about 1e-3)."""
    return AO.AttnSemantics(operand_round=ROUND[dtype], qk_round=QK[dtype])


# ------------------------------------------------------------------ the probs kernel
def _probs_ref(qkv, B, S, H, d, causal, lens=None):
    """fp64 softmax((q / sqrt(d)) k^T masked) of the qkv bits, flattened in the output layout (sample b from H * sum S_j^2 on)."""
    x = qkv.double()
    lens = lens or [S] * B
    out, r0 = [], 0
    for n in lens:
        q = x[r0:r0 + n, : H * d].reshape(n, H, d).permute(1, 0, 2)
        k = x[r0:r0 + n, H * d: 2 * H * d].reshape(n, H, d).permute(1, 0, 2)
        s = q @ k.transpose(1, 2) / math.sqrt(d)
        if causal:
            s = s.masked_fill(torch.triu(torch.ones(n, n, dtype=torch.bool, device=x.device), 1), float("-inf"))
        out.append(torch.softmax(s, -1).reshape(-1))
        r0 += n
    return torch.cat(out)


def _probs(lib, qkv, out_dt, B, S, H, d, causal, lens=None, pad=64):
    """jimm_k_attn_probs into a buffer with `pad` sentinel elements past its end: (output, sentinel tail)."""
    n = H * (sum(x * x for x in lens) if lens else B * S * S)
    buf = torch.full((n + pad,), float("nan"), dtype=out_dt, device="cuda")
    seq = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device="cuda") if lens else None
    check(lib, lib.jimm_k_attn_probs(ptr(qkv), CODE[qkv.dtype], ptr(buf), CODE[out_dt], ptr(seq), len(lens) if lens else B,
                                     max(lens) if lens else S, H, d, int(causal), stream()))
    torch.cuda.synchronize()
    return buf[:n], buf[n:]


def _check_probs(out, ref, lens, H, causal):
    assert torch.allclose(out.double(), ref, rtol=1e-4, atol=2e-6), float((out.double() - ref).abs().max())
    r0 = 0
    for n in lens:
        p = out[r0: r0 + H * n * n].view(H, n, n)
        assert torch.allclose(p.double().sum(-1), torch.ones(H, n, dtype=torch.float64, device="cuda"), rtol=0, atol=1e-5)
        if causal:
            assert (p[:, torch.triu(torch.ones(n, n, dtype=torch.bool, device="cuda"), 1)] == 0).all()
        r0 += H * n * n


@pytest.mark.parametrize("d", [8, 16, 24, 40, 64, 72, 80, 96, 128])
def test_probs_kernel(lib, d):
    H = 2
    g = torch.Generator(device="cuda").manual_seed(d)
    for S in (1, 2, 63, 64, 65, 197, 257, 577, 1025):
        for io in (torch.float16, torch.bfloat16):
            for causal in (False, True):
                for lens in (None, [S, 1, S // 2 + 1, 65]):
                    B = 2 if lens is None else len(lens)
                    rows = B * S if lens is None else sum(lens)
                    qkv = (torch.randn((rows, 3 * H * d), generator=g, device="cuda") * 1.5).to(io)
                    ref = _probs_ref(qkv, B, S, H, d, causal, lens)
                    f32, tail = _probs(lib, qkv, torch.float32, B, S, H, d, causal, lens)
                    assert torch.isnan(tail).all(), "elements past the output were written"
                    _check_probs(f32, ref, lens or [S] * B, H, causal)
                    for dt in (torch.float16, torch.bfloat16):  # 16-bit outputs: the fp32 output rounded to nearest even
                        o16, tail = _probs(lib, qkv, dt, B, S, H, d, causal, lens)
                        assert torch.isnan(tail).all() and torch.equal(o16.view(torch.int16), f32.to(dt).view(torch.int16)), (S, dt)
                    if lens:  # each packed sample is the dense call on that sample alone
                        r0, e0 = 0, 0
                        for n in lens:
                            alone, _ = _probs(lib, qkv[r0:r0 + n], torch.float32, 1, n, H, d, causal)
                            assert torch.equal(f32[e0:e0 + H * n * n], alone), (S, n)
                            r0, e0 = r0 + n, e0 + H * n * n


def test_probs_kernel_past_2_31_elements(lib):
    """One fp16 dense request of B * H * S^2 > 2^31 elements: the rows around element 2^31 and the last row against fp64."""
    B, H, S, d = 8, 16, 4097, 64
    assert B * H * S * S > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn((B * S, 3 * H * d), generator=g, device="cuda").half()
    out, tail = _probs(lib, qkv, torch.float16, B, S, H, d, False)
    assert torch.isnan(tail).all()
    row = 2 ** 31 // S
    for r in (row - 1, row, row + 1, B * H * S - 1):
        b, h, q = r // (H * S), (r // S) % H, r % S
        x = qkv[b * S:(b + 1) * S].double()
        qv = x[q, h * d:(h + 1) * d]
        k = x[:, H * d + h * d: H * d + (h + 1) * d]
        ref = torch.softmax(k @ qv / math.sqrt(d), 0)
        got = out[r * S:(r + 1) * S].double()
        assert torch.allclose(got, ref, rtol=2e-3, atol=1e-6), (r, float((got - ref).abs().max()))
    del out


@pytest.mark.parametrize("d", [8, 64, 72, 128])
def test_map_probs_kernel(lib, d):
    H = 3
    g = torch.Generator(device="cuda").manual_seed(d)
    for S in (1, 63, 257, 1025):
        for lens in (None, [S, 1, S // 2 + 1]):
            B = 2 if lens is None else len(lens)
            rows = B * S if lens is None else sum(lens)
            q = torch.randn((H * d,), generator=g, device="cuda")
            kv = torch.randn((rows, 2 * H * d), generator=g, device="cuda").half()
            seq = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device="cuda") if lens else None
            pooled = torch.empty((B, H * d), device="cuda")
            plain = torch.empty((B, H * d), device="cuda")
            probs = torch.full((H * rows + 16,), float("nan"), device="cuda")
            Smax = max(lens) if lens else S
            check(lib, lib.jimm_k_map_attention_probs(ptr(q), ptr(kv), 1, ptr(pooled), 0, ptr(seq), B, Smax, H, d, ptr(probs), 0, stream()))
            check(lib, lib.jimm_k_map_attention_probs(ptr(q), ptr(kv), 1, ptr(plain), 0, ptr(seq), B, Smax, H, d, None, 0, stream()))
            torch.cuda.synchronize()
            assert torch.equal(pooled, plain) and torch.isnan(probs[H * rows:]).all()
            r0 = 0
            for n in lens or [S] * B:
                k = kv[r0:r0 + n, : H * d].double().view(n, H, d)
                ref = torch.softmax(torch.einsum("nhd,hd->hn", k, q.double().view(H, d)) / math.sqrt(d), -1)
                got = probs[H * r0: H * (r0 + n)].view(H, n)
                assert torch.allclose(got.double(), ref, rtol=1e-4, atol=1e-6)
                r0 += n
            for pt in (1, 2):  # 16-bit weights are the fp32 weights rounded to nearest even
                dt = {1: torch.float16, 2: torch.bfloat16}[pt]
                p16 = torch.empty((H * rows,), dtype=dt, device="cuda")
                check(lib, lib.jimm_k_map_attention_probs(ptr(q), ptr(kv), 1, ptr(plain), 0, ptr(seq), B, Smax, H, d, ptr(p16), pt, stream()))
                torch.cuda.synchronize()
                assert torch.equal(p16.view(torch.int16), probs[: H * rows].to(dt).view(torch.int16))


# ------------------------------------------------------------------ models
def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


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


def _parity(case, what, dtype, out, ref, same):
    """Asserted against the same-rounding oracle (fp32 / fp16 at 1e-3, bf16 at BF16_VS_SAME), the plain fp32 oracle reported."""
    if same is not None:
        check_parity(case, what, dtype, "same-rounding", out, same, BAR[dtype])
    check_parity(case, what, dtype, "fp32", out, ref, None)


def _check_all(case, dtype, outs, refs, same, map_out=None):
    """outs: block 0 .. L-1 weights (CUDA); refs / same: (blocks, map) of the fp32 / same-rounding oracle."""
    for k, o in enumerate(outs):
        _parity(case, f"attentions block {k}", dtype, o, refs[0][k], same[0][k] if same else None)
    if map_out is not None:
        _parity(case, "attentions MAP head", dtype, map_out, refs[1], same[1] if same else None)


DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn]


@pytest.mark.parametrize("dtype", DTYPES)
def test_parity_vit(dtype):
    m, cfg, p = _vit(dtype)
    img = O.synthetic_images(3, 64)
    with torch.no_grad():
        refs = AO.vit_attn(p, cfg, img.double())
        same = AO.vit_attn(p, cfg, img.double(), _same(dtype)) if BAR[dtype] else None
    outs = m.forward_attentions(img.cuda())
    assert isinstance(outs, tuple) and len(outs) == L and all(o.shape == (3, 4, 17, 17) and o.dtype == torch.float32 for o in outs)
    _check_all("ViT 3x256 (CLS, no ln_pre) 64px B=3", dtype, outs, refs, same)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_parity_dual(kind, dtype):
    m, p = _dual(kind, dtype)
    img = O.synthetic_images(2, 64)
    txt = O.synthetic_tokens(3, 16, 100, kind)
    vis = AO.clip_image_attn if kind == "clip" else AO.siglip_image_attn
    txa = AO.clip_text_attn if kind == "clip" else AO.siglip_text_attn
    sem = _same(dtype)
    with torch.no_grad():
        ri, rt = vis(p, DCFG, img.double()), (txa(p, DCFG, txt), None)
        si, st = (vis(p, DCFG, img.double(), sem), (txa(p, DCFG, txt, sem), None)) if BAR[dtype] else (None, None)
    blocks = list(range(L)) + (["map"] if kind == "siglip" else [])
    oi = m.encode_image_attentions(img.cuda(), blocks)
    ot = m.encode_text_attentions(txt.cuda())
    S = 16 + (kind == "clip")
    assert all(o.shape == (2, 2, S, S) for o in oi[:L]) and all(o.shape == (3, 2, 16, 16) for o in ot)
    tower = "CLS, ln_pre" if kind == "clip" else "MAP"
    _check_all(f"{kind.upper()} vision 3x128 ({tower}) 64px B=2", dtype, oi[:L], ri, si, oi[L] if kind == "siglip" else None)
    _check_all(f"{kind.upper()} text 3x128 T=16 B=3", dtype, ot, rt, st)
    if kind == "clip":
        up = torch.triu(torch.ones(16, 16, dtype=torch.bool, device="cuda"), 1)
        assert all((o[..., up] == 0).all() for o in ot)
    else:
        assert oi[L].shape == (2, 2, 1, 16)


@pytest.mark.parametrize("dtype", DTYPES)
def test_parity_naflex(golden_dir, dtype):
    m, cfg, p, io = _naflex(golden_dir, dtype)
    pv, shapes = torch.from_numpy(io["pixel_values"]), io["spatial_shapes"]
    Lv = cfg.vision_layers
    with torch.no_grad():
        refs = AO.naflex_attn(p, cfg, pv.double(), shapes)
        same = AO.naflex_attn(p, cfg, pv.double(), shapes, _same(dtype)) if BAR[dtype] else None
    outs = m.encode_image_attentions(pv.cuda(), list(range(Lv)) + ["map"], spatial_shapes=shapes)
    case = "golden tiny_siglip2_naflex vision, padded mixed shapes"
    for i in range(Lv + 1):
        n = [h * w for h, w in shapes.tolist()]
        assert [tuple(o.shape) for o in outs[i]] == [(1, 1 if i == Lv else k, k) for k in n]
        o = torch.cat([x.reshape(-1) for x in outs[i]])
        pick = (lambda r: r[0][i]) if i < Lv else (lambda r: r[1])
        r = torch.cat([pick(x).reshape(-1) for x in refs])
        s = torch.cat([pick(x).reshape(-1) for x in same]) if same else None
        _parity(case, f"attentions {'MAP head' if i == Lv else f'block {i}'}", dtype, o, r, s)


# ------------------------------------------------------------------ return_pooled, input forms, packed = alone
def test_return_pooled_bits_vision():
    m, _, _ = _vit(torch.float16)
    g = torch.Generator().manual_seed(3)
    small = torch.randn((4, 64, 64, 3), generator=g).cuda()
    for _ in range(3):  # the pooled call of B = 4 is graph-replayed from its second call on
        ref = m(small)
    for blocks in (0, None, [2, 0]):
        assert torch.equal(m.forward_attentions(small, blocks, return_pooled=True)[1], ref)
    # host input: host results
    w, pooled = m.forward_attentions(small.cpu(), 1, return_pooled=True)
    assert not w.is_cuda and not pooled.is_cuda and torch.equal(pooled, ref.cpu())
    assert torch.equal(w, m.forward_attentions(small, 1).cpu())
    # interpolate_pos_encoding at another size
    hw = torch.randn((3, 48, 80, 3), generator=g).cuda()
    w, pooled = m.forward_attentions(hw, [0, 2], return_pooled=True, interpolate_pos_encoding=True)
    assert w[0].shape == (3, 4, 16, 16) and torch.equal(pooled, m(hw, interpolate_pos_encoding=True))
    # a packed list: each image's weights are its call alone
    lst = [torch.randn((h, w_, 3), generator=g).cuda() for h, w_ in [(64, 64), (32, 96), (80, 48)]]
    w, pooled = m.forward_attentions(lst, [1, 2], return_pooled=True, interpolate_pos_encoding=True)
    assert [t.shape for t in w[0]] == [(4, 17, 17), (4, 13, 13), (4, 16, 16)] and torch.equal(pooled, m(lst, interpolate_pos_encoding=True))
    assert w[0][0].untyped_storage().data_ptr() == w[0][-1].untyped_storage().data_ptr()  # views of one packed buffer
    for i, x in enumerate(lst):
        alone = m.forward_attentions(x[None], [1, 2], interpolate_pos_encoding=True)
        for j in range(2):
            assert torch.equal(w[j][i], alone[j][0]), (i, j)
    # B past max_batch and the packed token budget
    m.set_max_batch(2)
    big = torch.randn((5, 64, 64, 3), generator=g).cuda()
    w, pooled = m.forward_attentions(big, [0, 2], return_pooled=True)
    assert torch.equal(pooled, m(big))
    for i in range(5):
        alone = m.forward_attentions(big[i:i + 1], [0, 2])
        assert torch.equal(w[0][i], alone[0][0]) and torch.equal(w[1][i], alone[1][0])
    lst = [torch.randn((h, w_, 3), generator=g).cuda() for h, w_ in [(64, 64), (16, 16), (96, 96), (32, 64), (48, 16)]]
    w = m.forward_attentions(lst, 1, interpolate_pos_encoding=True)
    for i, x in enumerate(lst):
        assert torch.equal(w[i], m.forward_attentions(x[None], 1, interpolate_pos_encoding=True)[0])


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_return_pooled_bits_dual(kind):
    m, _ = _dual(kind, torch.float16)
    img = O.synthetic_images(5, 64).cuda()
    txt = O.synthetic_tokens(6, 16, 100, kind).cuda()
    for _ in range(3):
        ri, rt = m.encode_image(img), m.encode_text(txt)
    blocks = [1, "map"] if kind == "siglip" else 1
    assert torch.equal(m.encode_image_attentions(img, blocks, return_pooled=True)[1], ri)
    assert torch.equal(m.encode_text_attentions(txt, [0, 2], return_pooled=True)[1], rt)
    if kind == "siglip":  # the MAP weights without the pooled output: the head stops after its attention
        assert torch.equal(m.encode_image_attentions(img, "map"), m.encode_image_attentions(img, "map", return_pooled=True)[0])
    seqs = [txt[i, : 4 + 2 * i] for i in range(6)]
    w, pooled = m.encode_text_attentions(seqs, [1, 2], return_pooled=True)
    assert torch.equal(pooled, m.encode_text(seqs))
    for i, s in enumerate(seqs):  # packed samples equal the sequence alone
        alone = m.encode_text_attentions(s[None], [1, 2])
        for j in range(2):
            assert w[j][i].shape == (2, len(s), len(s)) and torch.equal(w[j][i], alone[j][0]), (i, j)
    # host ids
    w, pooled = m.encode_text_attentions(txt.cpu(), None, return_pooled=True)
    assert not w[0].is_cuda and torch.equal(pooled, rt.cpu())
    # past max_batch: dense and packed chunks
    m.set_max_batch(2)
    dense = m.encode_text_attentions(txt, 2)
    packed = m.encode_text_attentions(seqs, 2)
    for i in range(6):
        assert torch.equal(dense[i], m.encode_text_attentions(txt[i:i + 1], 2)[0])
        assert torch.equal(packed[i], m.encode_text_attentions(seqs[i][None], 2)[0])


def test_naflex_bits(golden_dir):
    m, cfg, p, io = _naflex(golden_dir, torch.float16)
    pv, shapes = torch.from_numpy(io["pixel_values"]).cuda(), io["spatial_shapes"]
    ref = m.encode_image(pv, spatial_shapes=shapes)
    w, pooled = m.encode_image_attentions(pv, [1, "map"], return_pooled=True, spatial_shapes=shapes)
    assert torch.equal(pooled, ref)
    P = cfg.vision_patch_size
    for b, (h, w_) in enumerate(shapes.tolist()):  # each sample alone, as pixel_values and as the NHWC image its rows cut
        one = m.encode_image_attentions(pv[b:b + 1, : h * w_], [1, "map"], spatial_shapes=shapes[b:b + 1])
        img = NF.rows_to_image(pv[b, : h * w_].cpu(), h, w_, P)[None].cuda()
        hwc = m.encode_image_attentions(img, [1, "map"])
        for j in range(2):
            assert torch.equal(w[j][b], one[j][0]) and torch.equal(w[j][b], hwc[j][0]), (b, j)


def test_nan_image_leaves_packed_neighbours():
    m, _, _ = _vit(torch.float16)
    g = torch.Generator().manual_seed(9)
    lst = [torch.randn((h, w, 3), generator=g).cuda() for h, w in [(64, 64), (32, 96), (80, 48)]]
    clean = m.forward_attentions(lst, [0, 2], interpolate_pos_encoding=True)
    bad = [lst[0], torch.full_like(lst[1], float("nan")), lst[2]]
    dirty = m.forward_attentions(bad, [0, 2], interpolate_pos_encoding=True)
    for j in range(2):
        assert torch.equal(dirty[j][0], clean[j][0]) and torch.equal(dirty[j][2], clean[j][2])
        assert torch.isnan(dirty[j][1]).all()


# ------------------------------------------------------------------ the pooled calls are unchanged; early exit; 16-bit outputs
def _launches(lib, fn):
    torch.cuda.synchronize()
    n0, g0 = lib.jimm_launch_count(), lib.jimm_graph_replay_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.jimm_launch_count() - n0, lib.jimm_graph_replay_count() - g0


def test_pooled_calls_unchanged_by_attention_calls(lib):
    m, p = _dual("siglip", torch.float16)
    img = O.synthetic_images(4, 64).cuda()
    txt = O.synthetic_tokens(4, 16, 100, "siglip").cuda()
    calls = [lambda: m.encode_image(img), lambda: m.encode_text(txt), lambda: m(img, txt)]
    for fn in calls:  # first call eager, second captured, later ones replayed
        fn(), fn()
    before = [_launches(lib, fn) for fn in calls]
    assert all(r >= 1 for _, _, r in before)
    for _ in range(2):
        _, n, r = _launches(lib, lambda: m.encode_image_attentions(img, [0, 2, "map"], return_pooled=True))
        assert r == 0 and n > 0
        _, n, r = _launches(lib, lambda: m.encode_text_attentions(txt, None, return_pooled=True))
        assert r == 0 and n > 0
    after = [_launches(lib, fn) for fn in calls]
    for (o0, n0, r0), (o1, n1, r1) in zip(before, after):
        assert torch.equal(o0, o1) and n0 == n1 and r0 == r1


def test_early_exit(lib):
    full, cfg, p = _vit(torch.float16)
    img = O.synthetic_images(3, 64).cuda()
    full.native()
    counts = {}
    for k in range(L):
        out, counts[k], _ = _launches(lib, lambda: full.forward_attentions(img, k))
        if k < L - 1:  # against a model of k + 1 blocks
            part, _, _ = _vit(torch.float16, layers=k + 1, params=p)
            assert torch.equal(out, part.forward_attentions(img, k)), k
    for k in range(1, L):
        assert counts[k] - counts[k - 1] == 7  # LayerNorm, QKV, attention, out-projection, LayerNorm, FC1, FC2
    _, two, _ = _launches(lib, lambda: full.forward_attentions(img, [0, 1]))
    assert two == counts[1] + 1  # one probs launch per request


@pytest.mark.parametrize("kind", ["vit", "clip"])
def test_16bit_outputs_equal_fp32_casts(kind):
    if kind == "vit":
        m, _, _ = _vit(torch.float16)
        img = O.synthetic_images(3, 64).cuda()
        run = lambda dt: m.forward_attentions(img, None, dtype=dt)
    else:
        m, _ = _dual("clip", torch.bfloat16)
        txt = O.synthetic_tokens(3, 16, 100, "clip").cuda()
        run = lambda dt: m.encode_text_attentions(txt, None, dtype=dt)
    ref = run(torch.float32)
    for dt in (torch.float16, torch.bfloat16):
        for k, (o, r) in enumerate(zip(run(dt), ref)):
            assert o.dtype == dt and torch.equal(o.view(torch.int16), r.to(dt).view(torch.int16)), (kind, dt, k)


# ------------------------------------------------------------------ ordering: the probs kernel reads qkv before FC1 overwrites it
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
torch.save([t.cpu() for t in m.forward_attentions(img, [0, 5, 11], dtype=torch.float16)], sys.argv[2])
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
        assert a.shape == (8, 12, 197, 197) and torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------ refusals
def test_refused_calls_enqueue_nothing(lib, golden_dir):
    from jimm_b200._lib import ATTN_MAP, AttnReq

    vit, _, _ = _vit(torch.float16)
    clip, _ = _dual("clip", torch.float16)
    sig, _ = _dual("siglip", torch.float16)
    nf, _, _, io = _naflex(golden_dir, torch.float16)
    hv, hc, hs, hn = vit.native().handle, clip.native().handle, sig.native().handle, nf.native().handle
    img = O.synthetic_images(2, 64).cuda()
    ids = O.synthetic_tokens(2, 16, 100, "clip").to(torch.int32).cuda()
    buf = torch.full((1 << 16,), float("nan"), device="cuda")
    pooled = torch.full((2, 16), float("nan"), device="cuda")

    def req(blocks, dtype=0, out=None, n=None):
        outs = out if out is not None else [buf.data_ptr()] * len(blocks)
        k = len(blocks)
        return AttnReq(k if n is None else n, (C.c_int * max(k, 1))(*blocks), (C.c_void_p * max(k, 1))(*outs), dtype)

    def refused(fn, msg=""):
        torch.cuda.synchronize()
        n0 = lib.jimm_launch_count()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == -1 and lib.jimm_launch_count() == n0
        assert msg in lib.jimm_last_error().decode(), lib.jimm_last_error().decode()

    im = lambda h, r, H=64, W=64: lambda: lib.jimm_image_attn(h, ptr(img), 0, 2, H, W, C.byref(r), ptr(pooled), stream())
    refused(im(hv, req([L])), "outside 0 .. 2")
    refused(im(hv, req([-3])), "outside 0 .. 2")
    refused(im(hv, req([ATTN_MAP])), "without a MAP head")  # CLS tower
    refused(im(hv, req([0], n=0)), "attention requests")
    refused(im(hv, req([0] * (L + 2))), "attention requests")
    refused(im(hv, req([0], dtype=3)), "output dtype")
    refused(im(hv, req([0], dtype=4)), "output dtype")
    refused(im(hv, req([0], out=[0])), "null or not 16-byte aligned")
    refused(im(hv, req([0], out=[buf.data_ptr() + 4])), "null or not 16-byte aligned")
    refused(lambda: lib.jimm_image_attn(hv, ptr(img), 0, 2, 64, 64, None, ptr(pooled), stream()), "null request")
    refused(im(hv, req([0]), H=8, W=64), "smaller than one")  # the pooled call's refusals
    refused(im(hs, req([ATTN_MAP]), H=8, W=64), "smaller than one")
    refused(lambda: lib.jimm_image_attn(hv, ptr(img), 7, 2, 64, 64, C.byref(req([0])), ptr(pooled), stream()), "bad image dtype")
    refused(lambda: lib.jimm_image_attn(hv, None, 0, 2, 64, 64, C.byref(req([0])), ptr(pooled), stream()), "null argument")
    refused(lambda: lib.jimm_text_attn(hv, ptr(ids), 2, 16, C.byref(req([0])), None, stream()), "no text tower")
    refused(lambda: lib.jimm_text_attn(hc, ptr(ids), 2, 17, C.byref(req([0])), None, stream()), "context_length")
    refused(lambda: lib.jimm_text_attn(hc, ptr(ids), 2, 16, C.byref(req([L])), None, stream()), "outside 0 .. 2")
    refused(lambda: lib.jimm_text_attn(hs, ptr(ids), 2, 16, C.byref(req([ATTN_MAP])), None, stream()), "without a MAP head")
    lens = (C.c_int * 2)(5, 0)
    refused(lambda: lib.jimm_text_attn_packed(hc, ptr(ids), 2, lens, C.byref(req([0])), None, stream()), "length 0")
    H2, W2 = (C.c_int * 2)(64, 8), (C.c_int * 2)(64, 64)
    ptrs = (C.c_void_p * 2)(img.data_ptr(), img.data_ptr())
    refused(lambda: lib.jimm_image_attn_packed(hv, ptrs, 0, 2, H2, W2, C.byref(req([0])), None, stream()), "smaller than one")
    pv = torch.from_numpy(io["pixel_values"]).cuda()
    good = [v for hw in io["spatial_shapes"].tolist() for v in hw]
    B, N = pv.shape[0], pv.shape[1]
    bad = (C.c_int * (2 * B))(*([17, 16] + good[2:]))
    refused(lambda: lib.jimm_image_attn_patches(hn, ptr(pv), 0, B, N, bad, C.byref(req([ATTN_MAP])), None, stream()), "more than its N")
    okg = (C.c_int * (2 * B))(*good)
    refused(lambda: lib.jimm_image_attn_patches(hc, ptr(pv), 0, B, N, okg, C.byref(req([0])), None, stream()), "not a SigLIP 2 NaFlex")
    refused(lambda: lib.jimm_image_attn_patches(hn, ptr(pv), 0, B, N, okg, C.byref(req([2])), None, stream()), "outside 0 .. 1")
    assert torch.isnan(buf).all() and torch.isnan(pooled).all()
