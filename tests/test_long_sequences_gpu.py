"""GPU: attention, MAP pooling and position resampling at the 1k to 57k tokens of 512 to 2048 px images (interpolate_pos_encoding,
packed lists), where the kernels run 17 to 900 key tiles per online softmax, the MAP scores fill most of shared memory and the
bicubic grids are several times the trained table.

- jimm_k_attention_hd at S = 1025 .. 8464 (4097 = 64 x 64 + 1: one real key and 63 clamped copies of it in the last tile) against
  exact fp64 and the tile-faithful fp64 restatement, on random inputs and on inputs with one dominant key (first tile, middle, last
  key); every output type and the reverse walk bit for bit; jimm_k_attention_packed with a 4097-token sample among 30 short ones.
- jimm_k_map_attention_hd / _packed up to the device's limit (its opt-in shared memory / 4 - 1152 tokens), refused one past it
  before any launch.
- jimm_k_tokens_init_interp on grids up to 128 x 64 and 1 x 300 from 14 x 14 / 16 x 16 tables, and the packed position add through a
  packed model call.
- Models against the interpolating oracle (tests/interp_oracle.py), 2 layers: ViT-B/16 at 1024 x 1024 (4097 tokens), a SigLIP-B/16-
  shaped MAP tower (256 wide) at 1472 x 1472 (8464 tokens), and a MAP tower at 1920 x 1920 (57600 tokens, past the MAP limit) that is
  refused up front while the same size runs on a CLS tower.

The fp64 references are computed one head at a time, so a test peaks at a few GB of device memory."""

import ctypes as C
import gc
import math

import pytest
import torch

import interp_oracle as I
import jimm_oracle as O
from gpu_util import BF16, CODE, F16, F32, TORCH, check, check_parity, ptr, record_parity, rel_err, stream
from attn_oracle import EXACT_TOL, _attn_ref, _attn_tile_ref, _check_tile_faithful
from test_head_dims import _qkv, _run_all_outputs
from test_kernel_paths_gpu import SENTINEL, TF32, rna_tf32

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-3
BF16_VS_SAME = 8e-3
MAP_TOL = 2e-5  # test_head_dims.test_map_attention_hd


@pytest.fixture(autouse=True)
def _free_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _map_limit():
    """The longest sequence the MAP head's attention takes: its scores, after 128 + 1024 floats, in the opt-in shared memory."""
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin // 4 - 1152


def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


# ------------------------------------------------------------------ attention kernel
def _peaked_qkv(B, S, H, d, io, seed, key):
    """_qkv's inputs with one dominant key: every query shares a component u, and key `key` of every sample is 3 u."""
    x = _qkv(B, S, H, d, torch.float32, seed).reshape(B, S, 3, H, d)
    u = torch.randn(H, d, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
    x[:, :, 0] += 2 * u
    x[:, key, 1] = 3 * u
    return x.reshape(B * S, 3 * H * d).to(io)


def _per_head(fn, qkv, B, S, H, d, causal):
    """fn (an fp64 restatement) one head at a time: [B * S, H * d] fp64."""
    x = qkv.reshape(B * S, 3, H, d)
    return torch.cat([fn(x[:, :, h].reshape(B * S, 3 * d), B, S, 1, d, causal) for h in range(H)], 1)


def _check_long(case, out, qkv, B, S, H, d, causal):
    """out (fp32) against exact fp64 and against the tile-faithful fp64."""
    io = qkv.dtype
    check_parity(case, "out", io, "exact fp64", out, _per_head(_attn_ref, qkv, B, S, H, d, causal), EXACT_TOL[io])
    _check_tile_faithful(case, out, qkv, B, S, H, d, causal, ref=_per_head(_attn_tile_ref, qkv, B, S, H, d, causal))


LONG_S = [1025, 2048, 2305, 4097, 8464]
IOS = pytest.mark.parametrize("io", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])


@IOS
@pytest.mark.parametrize("S", LONG_S)
@pytest.mark.parametrize("d", [64, 72, 80, 128])
def test_attention_long(lib, d, S, io):
    B, H = (2 if S < 4000 else 1), 2
    qkv = _qkv(B, S, H, d, io, seed=31 * d + S)
    f32 = _run_all_outputs(lib, qkv, B, S, H, d, 0, io)
    _check_long(f"long attention d={d} B={B} S={S} H={H}", f32, qkv, B, S, H, d, 0)


@IOS
@pytest.mark.parametrize("d", [64, 72, 80, 128])
def test_attention_long_causal(lib, d, io):
    B, S, H = 2, 2048, 2
    qkv = _qkv(B, S, H, d, io, seed=37 * d + 1)
    f32 = _run_all_outputs(lib, qkv, B, S, H, d, 1, io)
    _check_long(f"long attention d={d} B={B} S={S} H={H} causal", f32, qkv, B, S, H, d, 1)


@IOS
@pytest.mark.parametrize("peak", ["first", "mid", "last"])
@pytest.mark.parametrize("S", [1025, 4097, 8464])
@pytest.mark.parametrize("d", [64, 80])
def test_attention_long_peaked(lib, d, S, peak, io):
    """One key dominates every query's scores: at key 5 (the first tile, before the running maximum settles), mid-sequence, or at
    S - 1 (alone in its tile at S = 1025 and 4097)."""
    B, H = 1, 2
    key = {"first": 5, "mid": S // 2 + 3, "last": S - 1}[peak]
    qkv = _peaked_qkv(B, S, H, d, io, seed=41 * d + S, key=key)
    f32 = _run_all_outputs(lib, qkv, B, S, H, d, 0, io)
    _check_long(f"long attention d={d} S={S} H={H} dominant key {peak}", f32, qkv, B, S, H, d, 0)


SHORT = [1, 2, 7, 17, 31, 50, 63, 64, 65, 77, 96, 100, 127, 128, 129, 150, 160, 191, 192, 193, 196, 197, 3, 33, 97, 145, 180, 12, 111, 170]
PAIRS = [(F16, F16), (F16, F32), (F16, TF32), (BF16, BF16), (BF16, F32)]


def _out_dtype(code):
    return torch.float32 if code == TF32 else TORCH[code]


@pytest.mark.parametrize("io,ot", PAIRS)
@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("order", ["long_first", "long_last"])
def test_attention_packed_long(lib, order, d, io, ot):
    """A 4097-token sample among 30 of 1 to 197 tokens: each sample gives the bits of its _hd call and matches fp64."""
    H = 2
    D = H * d
    lens = [4097] + SHORT if order == "long_first" else SHORT + [4097]
    off = [0]
    for n in lens:
        off.append(off[-1] + n)
    T = off[-1]
    g = torch.Generator().manual_seed(d * 7 + io * 3 + ot)
    qkv = torch.randn((T + 5, 3 * D), generator=g).to(TORCH[io]).to(DEV)
    out = torch.full((T + 5, D), float("nan"), dtype=_out_dtype(ot), device=DEV)
    off_d = torch.tensor(off, dtype=torch.int32, device=DEV)
    check(lib, lib.jimm_k_attention_packed(ptr(qkv), io, ptr(out), ot, ptr(off_d), len(lens), max(lens), H, d, 0, stream()))
    worst = 0.0
    for b, S in enumerate(lens):
        o = off[b]
        one = torch.full((S, D), float("nan"), dtype=_out_dtype(ot), device=DEV)
        check(lib, lib.jimm_k_attention_hd(ptr(qkv[o:o + S]), io, ptr(one), ot, 1, S, H, d, 0, 0, stream()))
        assert torch.equal(out[o:o + S], one), f"sample {b} (S={S})"
        worst = max(worst, rel_err(out[o:o + S], _per_head(_attn_ref, qkv[o:o + S], 1, S, H, d, 0)))
    assert torch.isnan(out[T:]).all()
    record_parity(f"packed attention d={d} 4097 + 30 short ({order}) out={ot}", "out", str(TORCH[io]).replace("torch.", ""), "exact fp64",
                  EXACT_TOL[TORCH[io]], worst)
    assert worst < EXACT_TOL[TORCH[io]], worst


# ------------------------------------------------------------------ MAP attention kernel
def _map_inputs(B, S, H, d, probe, seed):
    """q fp32 [H d] and kv fp32 [B S, 2 H d], neighbouring heads large; probe "flat": q = 0 (equal weights on every key), "last": the
    last key of every sample dominates."""
    g = torch.Generator().manual_seed(seed)
    kv = torch.randn(B, S, 2, H, d, generator=g)
    kv[:, :, :, 1::2] *= 6.0
    if probe == "flat":
        q = torch.zeros(H, d)
    else:
        u = torch.randn(H, d, generator=g)
        q, kv[:, -1, 0] = 2 * u, 3 * u
    return q.reshape(-1).to(DEV), kv.reshape(B * S, 2 * H * d).to(DEV)


def _map_ref(q, kvt, B, S, H, d):
    k, v = kvt.double().reshape(B, S, 2, H, d).permute(2, 0, 3, 1, 4)
    w = torch.softmax((q.double().reshape(1, H, 1, d) / math.sqrt(d)) @ k.transpose(-1, -2), -1)
    return (w @ v).reshape(B, H * d)


MAP_S = [4096, 8192, 8193, 8464, 16384, "limit"]


@pytest.mark.parametrize("probe", ["flat", "last"])
@pytest.mark.parametrize("S", MAP_S)
def test_map_attention_long(lib, S, probe):
    """fp32 output against fp64; 16-bit and tf32 outputs the fp32 output rounded; the packed form, a 37-token sample before this one,
    gives each sample the bits of its _hd call."""
    S = _map_limit() if S == "limit" else S
    B, H, d = 2, 4, 64
    D = H * d
    q, kv = _map_inputs(B, S, H, d, probe, seed=S + (probe == "last"))
    for io, outs in ((torch.float16, [(torch.float16, F16), (torch.float32, TF32)]), (torch.bfloat16, [(torch.bfloat16, BF16)])):
        kvt = kv.to(io)
        f32 = torch.empty(B, D, device=DEV)
        check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kvt), CODE[io], ptr(f32), F32, B, S, H, d, stream()))
        check_parity(f"MAP attention d={d} B={B} S={S} H={H} probe {probe}", "pooled", io, "exact fp64", f32, _map_ref(q, kvt, B, S, H, d), MAP_TOL)
        for dt, code in outs:
            out = torch.full((B + 3, D), SENTINEL, dtype=dt, device=DEV)
            check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kvt), CODE[io], ptr(out), code, B, S, H, d, stream()))
            torch.cuda.synchronize()
            assert torch.equal(out[:B], rna_tf32(f32) if code == TF32 else f32.to(dt)), (io, code)
            assert bool((out[B:].float() == SENTINEL).all())
        lens = [37, S]
        pk = torch.cat([kvt[:37], kvt[S:]])  # sample 1 of kv after 37 rows of sample 0
        off = torch.tensor([0, 37, 37 + S], dtype=torch.int32, device=DEV)
        out = torch.full((3, D), SENTINEL, dtype=torch.float32, device=DEV)
        check(lib, lib.jimm_k_map_attention_packed(ptr(q), ptr(pk), CODE[io], ptr(out), F32, ptr(off), 2, S, H, d, stream()))
        one = torch.empty(1, D, device=DEV)
        check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(pk[:37]), CODE[io], ptr(one), F32, 1, 37, H, d, stream()))
        torch.cuda.synchronize()
        assert torch.equal(out[0:1], one) and torch.equal(out[1:2], f32[1:2]), io
        assert bool((out[2:] == SENTINEL).all())
        del kvt, pk


def test_map_attention_past_the_limit(lib):
    S, H, d = _map_limit() + 1, 4, 64
    D = H * d
    kv = torch.zeros((S, 2 * D), dtype=torch.float16, device=DEV)
    q = torch.zeros(D, device=DEV)
    out = torch.full((2, D), SENTINEL, device=DEV)
    off = torch.tensor([0, S], dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    n0 = lib.jimm_launch_count()
    assert lib.jimm_k_map_attention_hd(ptr(q), ptr(kv), F16, ptr(out), F32, 1, S, H, d, stream()) == -1
    msg = lib.jimm_last_error().decode()
    assert f"S={S} too large" in msg and f"at most {S - 1} tokens" in msg, msg
    assert lib.jimm_k_map_attention_packed(ptr(q), ptr(kv), F16, ptr(out), F32, ptr(off), 1, S, H, d, stream()) == -1
    assert f"S={S} too large" in lib.jimm_last_error().decode()
    torch.cuda.synchronize()
    assert lib.jimm_launch_count() == n0
    assert bool((out == SENTINEL).all())


# ------------------------------------------------------------------ position resampling
GRIDS = [(14, 73, 73), (16, 92, 92), (14, 128, 64), (16, 1, 300), (16, 300, 1)]


@pytest.mark.parametrize("cls", [True, False])
@pytest.mark.parametrize("g,gh,gw", GRIDS)
def test_tokens_init_interp_large_grids(lib, g, gh, gw, cls):
    """Against F.interpolate in fp64.  The bound is 1e-6 max|pos| (test_interpolate_pos_gpu.py) or twice PyTorch's own fp32 distance
    from fp64, whichever is larger: at 14 -> 73 and 16 -> 92 the fp32 source coordinate (scale (dst + 0.5) - 0.5, near g) is off by
    up to an ulp of g, and PyTorch's fp32 result is itself 1.1e-6 to 1.3e-6 max|pos| from fp64."""
    off, B, D = int(cls), 2, 768
    gen = torch.Generator().manual_seed(g * 7 + gh + gw)
    pos = torch.randn((off + g * g, D), generator=gen) * 0.2
    c = torch.randn(D, generator=gen) if cls else None
    x = torch.full((B, off + gh * gw, D), float("nan"), device=DEV)
    cd, pd = (c.to(DEV) if cls else None), pos.to(DEV)
    check(lib, lib.jimm_k_tokens_init_interp(ptr(cd), ptr(pd), g, D, ptr(x), B, gh, gw, stream()))
    torch.cuda.synchronize()
    refs = {}
    for dt in (torch.float32, torch.float64):
        r = I.resample_pos(pos[None].to(dt), g, gh, gw, cls)[0].clone()
        if cls:
            r[0] += c.to(dt)
        refs[dt] = r
    out = x.cpu()
    assert torch.equal(out[1], out[0])
    pmax = float(pos.abs().max())
    err64 = float((out[0].double() - refs[torch.float64]).abs().max())
    torch32 = float((refs[torch.float32].double() - refs[torch.float64]).abs().max())
    bound = max(1e-6 * pmax, 2 * torch32)
    case = f"tokens_init_interp {g}x{g} -> {gh}x{gw} cls={cls} (abs error over max abs pos)"
    record_parity(case, "tokens", "float32", "F.interpolate bicubic fp32", None, float((out[0] - refs[torch.float32]).abs().max()) / pmax)
    record_parity(case, "tokens", "float32", "F.interpolate bicubic fp64", bound / pmax, err64 / pmax)
    assert err64 <= bound, (err64 / pmax, torch32 / pmax)


def _tiny_tower(img, patch, pooling, seed):
    from jimm_b200.common.vit import VisionTransformerBase

    kw = dict(img_size=img, patch_size=patch, in_channels=3, hidden_size=64, num_layers=1, num_heads=1, mlp_dim=256, pooling_type=pooling,
              layernorm_epsilon=1e-6)
    t = O.TowerCfg(**kw)
    p = O.random_tower_params(t, seed=seed)
    return t, p, (lambda dtype=torch.float16: _set(VisionTransformerBase(**kw, dtype=dtype), p))


@pytest.mark.parametrize("pooling", ["CLS", "MAP"])
@pytest.mark.parametrize("g", [14, 16])
def test_packed_position_add_large_grids(g, pooling):
    """The packed call resamples every image's table in one kernel (tokens_add_interp_packed); each row is the bits of the image's
    own call, whose table tokens_init_interp writes."""
    P = 16
    sizes = [(gh * P, gw * P) for gg, gh, gw in GRIDS if gg == g] + [(g * P, g * P)]
    _, _, make = _tiny_tower(g * P, P, pooling, seed=g)
    m = make()
    gen = torch.Generator().manual_seed(g)
    imgs = [torch.randn((h, w, 3), generator=gen).to(DEV) for h, w in sizes]
    packed = m(imgs, interpolate_pos_encoding=True)
    for i, x in enumerate(imgs):
        assert torch.equal(packed[i:i + 1], m(x[None], interpolate_pos_encoding=True)), sizes[i]


# ------------------------------------------------------------------ models
def test_vit_b16_1024():
    """ViT-B/16 shapes, 2 layers, at 1024 x 1024: 4097 tokens from a 14 x 14 table."""
    from jimm_b200.models import VisionTransformer

    cfg = O.ViTCfg(num_layers=2)
    p = O.random_vit_params(cfg, seed=3)
    img = O.synthetic_images(2, 1024, seed=4)
    with torch.no_grad():
        ref = I.vit_forward(p, cfg, img, interpolate_pos_encoding=True)
        same = I.vit_forward(p, cfg, img, O.Semantics(operand_round="bf16"), interpolate_pos_encoding=True)
    case = "ViT-B/16 2 layers @1024x1024 (4097 tokens) B=2 interpolate_pos_encoding"
    for dtype in (torch.float16, torch.float32, torch.bfloat16):
        m = _set(VisionTransformer(num_layers=2, dtype=dtype), p).eval()
        out = m(img.cuda(), interpolate_pos_encoding=True)
        if dtype == torch.bfloat16:
            check_parity(case, "logits", dtype, "same-rounding", out, same, BF16_VS_SAME)
        else:
            check_parity(case, "logits", dtype, "fp32", out, ref, TOL)
            assert torch.equal(out.argmax(-1).cpu(), ref.argmax(-1))
        del m


SIGLIP = O.DualCfg(224, 2, 256, 16, 16, 100, 256, 4, 2)  # SigLIP-B/16 shapes at 256 wide (4 heads of 64), 2 + 2 layers


def _siglip(p, dtype):
    from jimm_b200.models import SigLIP

    return _set(SigLIP(224, 2, 256, 16, 16, 100, 256, 4, 2, dtype=dtype), p)


def test_siglip_map_tower_1472():
    """8464 tokens (92 x 92 from a 14 x 14 table) into the MAP head: past the MAP attention's former 8192-token limit."""
    p = O.random_dual_params(SIGLIP, "siglip", seed=5)
    img = O.synthetic_images(1, 1472, seed=6)
    with torch.no_grad():
        ref = I.siglip_encode_image(p, SIGLIP, img, interpolate_pos_encoding=True)
    case = "SigLIP-B/16-shaped tower 2x256 @1472x1472 (8464 tokens, MAP head)"
    for dtype in (torch.float16, torch.float32):
        m = _siglip(p, dtype)
        check_parity(case, "image_embeds", dtype, "fp32", m.encode_image(img.cuda(), interpolate_pos_encoding=True), ref, TOL)
        if dtype == torch.float16:
            gen = torch.Generator().manual_seed(7)
            imgs = [img[0].cuda(), torch.randn((224, 224, 3), generator=gen).cuda(), torch.randn((64, 512, 3), generator=gen).cuda()]
            packed = m.encode_image(imgs, interpolate_pos_encoding=True)
            for i, x in enumerate(imgs):
                assert torch.equal(packed[i:i + 1], m.encode_image(x[None], interpolate_pos_encoding=True)), tuple(x.shape)
        del m


def test_map_tower_past_the_limit():
    """A 64-wide MAP tower at 1920 x 1920 with patch 8: 240 x 240 = 57600 tokens, past the MAP limit.  Refused before anything is
    enqueued, by every entry point, with a message that is not the "raise the budget" one; the Python class raises ValueError and
    keeps its handle.  The same size runs on a CLS tower: only the MAP head has the limit."""
    from jimm_b200 import _lib

    limit = _map_limit()
    H = W = 1920
    tokens = (H // 8) * (W // 8)
    assert tokens > limit
    _, _, make = _tiny_tower(64, 8, "MAP", seed=8)
    m = make().set_max_batch(1).set_max_image_size(H, W)  # a workspace that holds the image: only the MAP limit refuses it
    n = m.native()
    lib = _lib.load()
    x = torch.zeros((1, H, W, 3), device=DEV)
    small = torch.zeros((64, 64, 3), device=DEV)
    out = torch.full((2, 64), float("nan"), device=DEV)
    ptrs = (C.c_void_p * 2)(small.data_ptr(), x.data_ptr())
    hs, ws = (C.c_int * 2)(64, H), (C.c_int * 2)(64, W)
    torch.cuda.synchronize()
    n0 = lib.jimm_launch_count()
    got = []
    for fn in (lib.jimm_encode_image_hw, lib.jimm_vit_forward_hw):
        got.append((fn(n.handle, C.c_void_p(x.data_ptr()), _lib.F32, 1, H, W, C.c_void_p(out.data_ptr()), stream()), lib.jimm_last_error().decode()))
    for fn in (lib.jimm_encode_image_packed, lib.jimm_vit_forward_packed):
        got.append((fn(n.handle, ptrs, _lib.F32, 2, hs, ws, C.c_void_p(out.data_ptr()), stream()), lib.jimm_last_error().decode()))
    torch.cuda.synchronize()
    assert lib.jimm_launch_count() == n0, "kernels were launched before the refusal"
    assert torch.isnan(out).all()
    for rc, msg in got:
        assert rc == -1 and f"{tokens} tokens" in msg and f"at most {limit} tokens" in msg, (rc, msg)
    k = C.c_int(-7)
    assert lib.jimm_model_images_per_call(n.handle, H, W, C.byref(k)) == -1
    msg = lib.jimm_last_error().decode()
    assert f"{tokens} tokens" in msg and f"at most {limit} tokens" in msg and "raise the budget" not in msg, msg
    assert lib.jimm_model_images_per_call(n.handle, 64, 64, C.byref(k)) == 0 and k.value >= 1
    with pytest.raises(ValueError, match=f"{tokens} tokens"):
        m(x, interpolate_pos_encoding=True)
    with pytest.raises(ValueError, match=f"{tokens} tokens"):
        m([small, x[0]], interpolate_pos_encoding=True)
    assert m.native() is n
    # a handle built for the call itself is dropped, and the budget stays as it was
    fresh = make()
    with pytest.raises(ValueError, match=f"{tokens} tokens"):
        fresh(x, interpolate_pos_encoding=True)
    assert fresh._max_tokens == 0 and fresh.native().images_per_call(64, 64) >= 1
    del m, fresh, n
    # the CLS tower at the same size (57601 tokens) runs
    _, _, make_cls = _tiny_tower(64, 8, "CLS", seed=9)
    c = make_cls()
    y = c(torch.randn((1, H, W, 3), generator=torch.Generator().manual_seed(10)).to(DEV), interpolate_pos_encoding=True)
    assert y.shape == (1, 64) and bool(torch.isfinite(y).all())


def test_map_head_handle_past_the_limit():
    """A bare MAP head is refused at finalize for a ctx_len past the limit, and runs at the limit and below afterwards."""
    from jimm_b200.common.vit import MultiHeadAttentionPoolingHead

    D, Hh = 64, 1
    t = O.TowerCfg(32, 8, 3, D, 0, Hh, 4 * D, "MAP", layernorm_epsilon=1e-6)
    p = {k[len("MAPHead."):]: v for k, v in O.random_tower_params(t, seed=11).items() if k.startswith("MAPHead.")}
    h = _set(MultiHeadAttentionPoolingHead(D, 4 * D, Hh, 1e-6, dtype=torch.float16), p)
    limit = _map_limit()
    with pytest.raises(ValueError, match=f"ctx_len: {limit + 1} tokens"):
        h(torch.zeros((1, limit + 1, D), device=DEV))
    x = torch.randn((1, limit, D), generator=torch.Generator().manual_seed(12))
    with torch.no_grad():
        ref = O.map_head(p, "", x, Hh, 1e-6)
    check_parity(f"bare MAP head 64 wide at S={limit}", "pooled", torch.float16, "fp32", h(x.to(DEV)), ref, TOL)
