"""FP8 compute mode (dtype=torch.float8_e4m3fn): float16 everywhere except the QKV and FC1 GEMMs of every encoder block, which run
on e4m3 operands with power-of-two scales per token row and per output channel (tests/fp8_oracle.py states the numerics).

- CPU: the dtype names; jimm_model_create refuses tower widths that are not multiples of 16 and names the width.
- GPU kernels: the e4m3 LayerNorm and the weight quantiser give the oracle quantiser's bytes and scales bit for bit (the LayerNorm
  against the same kernel's fp32 output); the e4m3 GEMM against fp64 on the dequantised operands, with M / N / K tails, N ending a
  256-column tile at each store-box boundary, bias / GELU / QuickGELU and f16 / bf16 / f32 / tf32 outputs; the reverse walk and a
  plan of more rows give the same bits; rows >= roundup(M, 16) keep their sentinel.
- GPU models: each model's distance to the FP8 oracle is at most half of that oracle's distance to the fp32 oracle; graph replay,
  batch chunking, host inputs, JIMM_FUSE_LN, one stream and a transposed weight hand-off give the same bits."""

import ctypes

import pytest
import torch

import fp8_oracle as F
import jimm_oracle as O
from gpu_util import CODE, check, check_parity, ptr, record_parity, rel_err, stream
from test_kernel_paths_gpu import SENTINEL, TF32

DEV = "cuda"
E4M3 = 4  # jimm_dtype JIMM_F8E4M3
# A model's distance to the FP8 oracle, as a share of that oracle's own distance to the fp32 oracle.  Measured on an H100: 0.04 (ViT-L/16
# MAP, 2 layers) to 0.33 (bare 3-layer Transformer, whose K = 128 GEMMs have nothing to promote).  The distance does not come from the
# GEMM: the fp16 attention's last-bit differences from the fp64 oracle move a few LayerNorm outputs across an e4m3 rounding boundary,
# each such flip is a whole e4m3 step, and the flips of one block feed the next.
ORACLE_SHARE = 0.5


def _u8(q):
    return q.view(torch.uint8)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_dtype_names():
    from jimm_b200 import _lib, nn

    assert nn.compute_dtype_code(torch.float8_e4m3fn) == _lib.F8E4M3 == E4M3
    assert nn.compute_dtype_code("float8_e4m3fn") == E4M3
    assert nn.compute_dtype_code("jnp.float8_e4m3fn") == E4M3
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        nn.compute_dtype_code(torch.float8_e5m2)


def _create(lib, kind, width, heads, t_width=0, t_heads=0):
    from jimm_b200 import _lib

    cfg = _lib.Config()
    cfg.kind, cfg.pooling, cfg.compute_dtype = kind, 0, E4M3
    cfg.img_size, cfg.patch, cfg.in_ch = 224, 16, 3
    cfg.v_width, cfg.v_heads, cfg.v_layers, cfg.v_mlp = width, heads, 2, 4 * width
    cfg.ctx_len, cfg.vocab, cfg.t_width, cfg.t_heads, cfg.t_layers, cfg.t_mlp = 64, 1000, t_width, t_heads, 2, 4 * t_width
    h = ctypes.c_void_p()
    rc = lib.jimm_model_create(ctypes.byref(cfg), 0, ctypes.byref(h))
    if rc == 0:
        lib.jimm_model_destroy(h)
    return rc, lib.jimm_last_error().decode()


@pytest.mark.parametrize("kind,w,h,tw,th,text", [(0, 200, 25, 0, 0, "vision width 200"), (1, 256, 4, 200, 25, "text width 200"),
                                                 (4, 200, 25, 0, 0, "model width 200"), (5, 72, 9, 0, 0, "model width 72")])
def test_create_refuses_width_not_multiple_of_16(lib, kind, w, h, tw, th, text):
    rc, msg = _create(lib, kind, w, h, tw, th)
    assert rc == -1, (rc, msg)
    assert text in msg and "multiple of 16" in msg, msg


# ---------------------------------------------------------------------------------------------------------------- GPU: LayerNorm
def _ln_input(rows, D, gscale, zero_bias, seed):
    """Row 0 is all zeros (with a zero bias its normalised row is zero); the other rows have deviations from 2^-40 to 2^0, so with a
    small eps their normalised values run from ~2^-20 |scale| to |scale|."""
    g = torch.Generator().manual_seed(seed)
    dev = torch.pow(2.0, torch.linspace(-40, 0, rows)).unsqueeze(1)
    x = torch.randn(rows, D, generator=g) * dev
    x[0] = 0
    scale = torch.randn(D, generator=g) * gscale
    bias = torch.zeros(D) if zero_bias else torch.randn(D, generator=g) * gscale * 0.5
    return x.to(DEV), scale.to(DEV), bias.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("gscale", [2.0 ** -20, 1.0, 2.0 ** 20], ids=["g2^-20", "g1", "g2^20"])
@pytest.mark.parametrize("eps", [1e-12, 1e-6, 1e-5])
@pytest.mark.parametrize("D", [64, 768, 1024, 1152, 2048])  # <= 1024: 8 float4 per lane; above: 16
def test_layernorm_e4m3(lib, D, eps, gscale):
    rows = 333
    x, scale, bias = _ln_input(rows, D, gscale, zero_bias=eps == 1e-12, seed=D)
    y = torch.empty(rows, D, device=DEV)
    check(lib, lib.jimm_k_layernorm_ex(ptr(x), D, 1, 0, None, ptr(scale), ptr(bias), eps, ptr(y), 0, D, rows, D, 0, stream()))
    q_ref, s_ref = F.quantize_rows(y.cpu())
    for rev in (0, 1):
        q = torch.full((rows + 5, D), 0x55, dtype=torch.uint8, device=DEV)
        s = torch.full((rows + 5,), -1.0, device=DEV)
        check(lib, lib.jimm_k_layernorm_e4m3(ptr(x), D, ptr(scale), ptr(bias), eps, ptr(q), D, ptr(s), rows, D, rev, stream()))
        torch.cuda.synchronize()
        assert torch.equal(q[:rows].cpu(), _u8(q_ref)), f"reverse={rev}: e4m3 bytes differ from the oracle quantiser"
        assert torch.equal(s[:rows].cpu(), s_ref), f"reverse={rev}: row scales differ from the oracle"
        assert bool((q[rows:] == 0x55).all()) and bool((s[rows:] == -1).all()), "rows past `rows` were written"
    if eps == 1e-12:  # zero bias: row 0 normalises to zeros, the others span about 2^-20 |scale| .. |scale|
        amax = y.abs().amax(-1).cpu()
        assert float(amax[0]) == 0 and float(s_ref[0]) == 1.0
        assert float(amax[1:].min()) < 2.0 ** -17 * gscale and float(amax.max()) > gscale


# ---------------------------------------------------------------------------------------------------------------- GPU: weight quantiser
def _rows_with_spread(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * torch.pow(2.0, torch.randint(-20, 21, (N, 1), generator=g).float())
    w[0] = 0
    w[1] = 0
    w[1, 5] = 448.0 * 2.0 ** -3  # amax exactly 448 x a power of two: s = 2^-3, the element becomes 448
    w[2, :] = 0.5 * (2.0 ** -9 + 2.0 ** -8)  # constant row 0.75 x 2^-8: s = 2^-17, every element 384
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("N,K", [(2304, 768), (3072, 1024), (100, 2048), (7, 12)])
def test_weight_quantiser(lib, N, K):
    w = _rows_with_spread(N, K, seed=N)
    q_ref, s_ref = F.quantize_rows(w)
    wd = w.to(DEV)
    q = torch.empty(N, K, dtype=torch.uint8, device=DEV)
    s = torch.empty(N, device=DEV)
    check(lib, lib.jimm_k_quantize_e4m3(ptr(wd), K, N, K, ptr(q), K, ptr(s), stream()))
    torch.cuda.synchronize()
    assert torch.equal(q.cpu(), _u8(q_ref))
    assert torch.equal(s.cpu(), s_ref)
    assert float(s_ref[0]) == 1.0 and float(s_ref[1]) == 2.0 ** -3 and int(q[1, 5]) == 0x7E


# ---------------------------------------------------------------------------------------------------------------- GPU: GEMM
def _mk8(M, N, K, seed):
    """e4m3 A [M, K], B [N, K] with per-row scales spanning 2^-4..2^3 (device; products stay inside fp16), and their dequantised fp64
    values (CPU)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g) * torch.pow(2.0, torch.randint(-4, 4, (M, 1), generator=g).float())
    b = torch.randn(N, K, generator=g) * torch.pow(2.0, torch.randint(-4, 4, (N, 1), generator=g).float())
    qa, sa = F.quantize_rows(a)
    qb, sb = F.quantize_rows(b)
    return (_u8(qa).to(DEV), sa.to(DEV), _u8(qb).to(DEV), sb.to(DEV)), F.dequant(qa, sa), F.dequant(qb, sb)


def gemm8(lib, ops, out, *, M=None, plan_M=0, bias=None, act=0, out_code=None, mode=2, reverse=0, impl=0):
    A, sa, B, sb = ops
    N, K = B.shape
    M = A.shape[0] if M is None else M
    return lib.jimm_k_gemm_e4m3(impl, ptr(A), A.stride(0), ptr(B), B.stride(0), M, N, K, ptr(sa), ptr(sb), ptr(bias), act, ptr(out),
                                CODE[out.dtype] if out_code is None else out_code, out.stride(0), mode, plan_M, reverse, stream())


ACTS = [lambda v: v, lambda v: O.gelu_tanh(v), lambda v: O.quickgelu(v)]
# One rounding of the output type plus the e4m3 MMA's accumulation error (test_fp8_accumulation_error)
OUT_TOL8 = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2, torch.float32: 1e-3, TF32: 1.5e-3}


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "gelu", "quickgelu"])
@pytest.mark.parametrize("M", [200, 3001])
@pytest.mark.parametrize("out_t,N", [(torch.float16, n) for n in (64, 128, 192, 320, 2296)] + [(torch.bfloat16, 192)]
                         + [(torch.float32, n) for n in (32, 96, 160, 224, 288)] + [(TF32, 224)],
                         ids=lambda v: {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32", TF32: "tf32"}.get(v, str(v)))
def test_gemm_e4m3(lib, out_t, N, M, act):
    """Columns >= N and rows >= roundup(M, 16) keep their sentinel; the rest is act(fp64 product of the dequantised operands + bias)
    at one output rounding; the reverse walk and a plan of more rows write the same bits."""
    K, ldo = 1008, N + 64  # K tail: 1008 = 7 x 128 + 112 (e4m3 rows must be 16-byte multiples)
    ops, Ad, Bd = _mk8(M, N, K, seed=N + M)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(N)).to(DEV)
    ref = ACTS[act](Ad @ Bd.T + bias.double().cpu())
    dt = torch.float32 if out_t == TF32 else out_t
    code = TF32 if out_t == TF32 else CODE[out_t]
    r16 = (M + 15) // 16 * 16
    outs = []
    for rev, plan_M in ((0, 0), (1, 0), (0, M + 100)):
        out = torch.full((M + 48, ldo), SENTINEL, dtype=dt, device=DEV)
        A = ops[0] if plan_M == 0 else torch.cat([ops[0], torch.zeros(100, K, dtype=torch.uint8, device=DEV)])
        sa = ops[1] if plan_M == 0 else torch.cat([ops[1], torch.ones(100, device=DEV)])
        check(lib, gemm8(lib, (A, sa, ops[2], ops[3]), out, M=M, plan_M=plan_M, bias=bias, act=act, out_code=code, reverse=rev))
        torch.cuda.synchronize()
        assert bool((out[:, N:].float() == SENTINEL).all()), "columns >= N were written"
        assert bool((out[r16:].float() == SENTINEL).all()), "rows >= roundup(M, 16) were written"
        err = rel_err(out[:M, :N].cpu(), ref)
        assert err < OUT_TOL8[out_t], f"rev={rev} plan_M={plan_M}: rel err {err:.2e}"
        outs.append(out[:M])
    assert torch.equal(outs[0], outs[1]), "reverse walk differs from the forward walk"
    assert torch.equal(outs[0], outs[2]), "a plan of more rows differs"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
def test_gemm_e4m3_simt_and_lsu(lib, mode):
    """The SIMT bisection kernel and the LSU epilogue (mode 0) compute the same function."""
    M, N, K = 300, 520, 768
    ops, Ad, Bd = _mk8(M, N, K, seed=3)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(4)).to(DEV)
    ref = O.gelu_tanh(Ad @ Bd.T + bias.double().cpu())
    for impl in (0, 1):
        out = torch.full((M, N), SENTINEL, device=DEV)
        check(lib, gemm8(lib, ops, out, bias=bias, act=1, mode=mode, impl=impl))
        torch.cuda.synchronize()
        assert rel_err(out.cpu(), ref) < OUT_TOL8[torch.float32], f"impl={impl} mode={mode}"


@pytest.mark.gpu
def test_gemm_e4m3_refuses_other_epilogues(lib):
    M, N, K = 64, 128, 256
    A = torch.zeros(M, K, dtype=torch.uint8, device=DEV)
    B = torch.zeros(N, K, dtype=torch.uint8, device=DEV)
    x = torch.zeros(M, N, device=DEV)
    rc = lib.jimm_k_gemm(0, E4M3, ptr(A), K, ptr(B), K, M, N, K, None, 0, None, ptr(x), N, ptr(x), 0, N, 0, 0, 0, 2, stream())
    assert rc == -1 and "e4m3" in lib.jimm_last_error().decode()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [768, 1024, 1152, 2048])
def test_fp8_accumulation_error(lib, K):
    """fp32 output of the e4m3 GEMM against fp64 on the same (exactly representable) operands: the MMA's accumulation error alone.
    Recorded per K; the bound is about 3x the worst value measured on an H100 (6.8e-5 at K = 768, 4.0e-5 at K = 2048, with the K-slab
    promotion of gemm_wgmma_kernel; without it the e4m3 wgmma gave 4.3e-4 to 5.2e-4)."""
    M, N = 2048, 2304
    ops, Ad, Bd = _mk8(M, N, K, seed=K)
    out = torch.empty(M, N, device=DEV)
    check(lib, gemm8(lib, ops, out))
    torch.cuda.synchronize()
    ref = Ad @ Bd.T
    # error per element relative to the sum of |products| (the scale an fp32 accumulation error is proportional to)
    mag = Ad.abs() @ Bd.abs().T
    per = float(((out.cpu().double() - ref).abs() / mag).max())
    record_parity(f"e4m3 GEMM {M}x{N}x{K}", "accumulation error / sum|a b|", "e4m3", "fp64", None, per)
    assert per < ACC_BOUND, f"K={K}: max |err| / sum|a b| = {per:.2e}"


ACC_BOUND = 2e-4


# ---------------------------------------------------------------------------------------------------------------- GPU: models
def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


def _fp64(p):
    return {k: v.to(torch.float64) for k, v in p.items()}


def _judge(case, what, out, ref8, ref32):
    """out vs the FP8 oracle, at most ORACLE_SHARE of the FP8 oracle's own distance to the fp32 oracle."""
    d_mode = rel_err(ref8, ref32)
    record_parity(case, what, "float8_e4m3fn", "fp32 (FP8 oracle)", None, d_mode)
    check_parity(case, what, "float8_e4m3fn", "FP8 oracle", out, ref8, ORACLE_SHARE * d_mode)


@pytest.fixture(scope="module")
def vitb16_fp8():
    cfg = O.ViTCfg()
    p = O.random_vit_params(cfg, seed=0)
    img = O.synthetic_images(2, 224)
    pd, imgd = _fp64(p), img.double()
    with torch.no_grad(), F.active():
        ref8 = O.vit_forward(pd, cfg, imgd, F.FP8)
        ref32 = O.vit_forward(pd, cfg, imgd)
    return cfg, p, img, ref8, ref32


@pytest.mark.gpu
def test_vit_b16_fp8(vitb16_fp8):
    from jimm_b200.models import VisionTransformer

    cfg, p, img, ref8, ref32 = vitb16_fp8
    m = _set(VisionTransformer(dtype=torch.float8_e4m3fn), p).eval()
    out = m(img.cuda())
    _judge("ViT-B/16@224 B=2", "logits", out, ref8, ref32)
    assert torch.equal(m(img), out.cpu())  # host input


@pytest.mark.gpu
def test_vit_l16_384_map_fp8():
    from jimm_b200.common.vit import VisionTransformerBase

    t = O.TowerCfg(img_size=384, patch_size=16, in_channels=3, hidden_size=1024, num_layers=2, num_heads=16, mlp_dim=4096,
                   pooling_type="MAP", layernorm_epsilon=1e-6)
    p = O.random_tower_params(t, seed=5)
    img = O.synthetic_images(2, 384)
    with torch.no_grad(), F.active():
        ref8 = O.vision_tower(_fp64(p), "", img.double(), t, F.FP8)
        ref32 = O.vision_tower(_fp64(p), "", img.double(), t)
    m = _set(VisionTransformerBase(img_size=384, patch_size=16, in_channels=3, hidden_size=1024, num_layers=2, num_heads=16, mlp_dim=4096,
                                   pooling_type="MAP", layernorm_epsilon=1e-6, dtype=torch.float8_e4m3fn), p)
    _judge("ViT-L/16@384 MAP, 2 layers", "pooled", m(img.cuda()), ref8, ref32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_dual_tower_medium_fp8(kind, monkeypatch):
    from jimm_b200.models import CLIP, SigLIP

    tw = 128 if kind == "clip" else 256
    cfg = O.DualCfg(image_resolution=64, vision_layers=2, vision_width=256, vision_patch_size=16, context_length=20, vocab_size=300,
                    transformer_width=tw, transformer_heads=tw // 64, transformer_layers=2)
    p = O.random_dual_params(cfg, kind, seed=11)
    img, txt = O.synthetic_images(6, 64), O.synthetic_tokens(9, 20, 300, kind)
    enc_i, enc_t = (O.clip_encode_image, O.clip_encode_text) if kind == "clip" else (O.siglip_encode_image, O.siglip_encode_text)
    pd, imgd = _fp64(p), img.double()
    with torch.no_grad(), F.active():
        ri8, rt8 = enc_i(pd, cfg, imgd, F.FP8), enc_t(pd, cfg, txt, F.FP8)
        ri32, rt32 = enc_i(pd, cfg, imgd), enc_t(pd, cfg, txt)
    cls = CLIP if kind == "clip" else SigLIP
    m = _set(cls(64, 2, 256, 16, 20, 300, tw, tw // 64, 2, dtype=torch.float8_e4m3fn), p)
    case = f"dual medium {kind} 2x256/2x{tw}"
    _judge(case, "image_embeds", m.encode_image(img.cuda()), ri8, ri32)
    _judge(case, "text_embeds", m.encode_text(txt.cuda()), rt8, rt32)
    out = m(img.cuda(), txt.cuda())
    assert torch.equal(m(img, txt.to(torch.int32)), out.cpu())  # host inputs
    monkeypatch.setenv("JIMM_DUAL_STREAMS", "0")  # read when the native model is created
    m1 = _set(cls(64, 2, 256, 16, 20, 300, tw, tw // 64, 2, dtype=torch.float8_e4m3fn), p)
    assert torch.equal(m1(img.cuda(), txt.cuda()), out), "one stream differs from two"


@pytest.mark.gpu
@pytest.mark.parametrize("causal,quick", [(False, False), (True, True)])
def test_transformer_fp8(causal, quick):
    from jimm_b200.common.transformer import Transformer

    D, M, H, L, T = 128, 512, 2, 3, 20
    g = torch.Generator().manual_seed(41)
    p = {}
    O._rand_blocks(p, g, "", L, D, H, M)
    p = O.cast_params(p, torch.float32)
    mask = torch.tril(torch.ones(T, T)) if causal else None
    x = torch.randn(5, 13, D, generator=g)
    with torch.no_grad(), F.active():
        ref8 = O.transformer(_fp64(p), "", x.double(), L, H, quick, mask, 1e-5, F.FP8)
        ref32 = O.transformer(_fp64(p), "", x.double(), L, H, quick, mask, 1e-5)
    t = _set(Transformer(D, M, L, H, layernorm_epsilon=1e-5, attn_mask=mask, use_quick_gelu=quick, dtype=torch.float8_e4m3fn), p)
    # the encoder returns the residual stream, whose first rows carry the input: judge the update x_out - x_in
    out = t(x.cuda()).cpu().double()
    _judge(f"bare Transformer 3x128 causal={causal}", "activations - input", out - x.double(), ref8 - x.double(), ref32 - x.double())


SMALL = dict(num_classes=16, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=1024, hidden_size=256)


@pytest.mark.gpu
def test_fp8_same_bits_across_paths(monkeypatch):
    """Graph replay, batch chunking, host inputs, JIMM_FUSE_LN=1 and a transposed (HF-layout) weight hand-off give the same bits."""
    from jimm_b200.models import VisionTransformer
    from jimm_b200.nn import LazyParam

    p = O.random_vit_params(O.ViTCfg(**SMALL), seed=2)
    img = O.synthetic_images(8, 64, seed=3)
    m = _set(VisionTransformer(**SMALL, dtype=torch.float8_e4m3fn), p).eval()
    x = img.cuda()
    ref = m(x)
    small = [m(x[:4]) for _ in range(4)]  # eager, capture, replays
    for o in small:
        assert torch.equal(o, ref[:4]), "graph replay differs"
    assert torch.equal(m(img), ref.cpu()), "host input differs"
    m.set_max_batch(3)
    assert torch.equal(m(x), ref), "chunked batch differs"
    # HF (out, in) layout of every kernel of the blocks: the quantiser reads the same fp32 rows
    mt = VisionTransformer(**SMALL, dtype=torch.float8_e4m3fn).eval()
    for k, v in p.items():
        v = v.to(torch.float32)
        if ".blocks." in k and k.endswith(".kernel"):
            K = v.shape[0] if "attn.out" not in k else v.shape[0] * v.shape[1]
            mt.set_flat_param(k, LazyParam(v.reshape(K, -1).T.contiguous(), v.shape, transposed=True))
        else:
            mt.set_flat_param(k, v)
    assert torch.equal(mt(x), ref), "transposed hand-off differs"
    monkeypatch.setenv("JIMM_FUSE_LN", "1")
    mf = _set(VisionTransformer(**SMALL, dtype=torch.float8_e4m3fn), p).eval()
    assert torch.equal(mf(x), ref), "JIMM_FUSE_LN=1 differs"


@pytest.mark.gpu
def test_fp8_simt_bisection_path(monkeypatch):
    """JIMM_GEMM_IMPL=simt in FP8 mode: the same function up to fp32 summation order, which the e4m3 rounding of the LayerNorm
    outputs amplifies as between the model and its oracle (8.7e-3 measured on an H100)."""
    from jimm_b200.models import VisionTransformer

    p = O.random_vit_params(O.ViTCfg(**SMALL), seed=2)
    x = O.synthetic_images(3, 64, seed=3).cuda()
    a = _set(VisionTransformer(**SMALL, dtype=torch.float8_e4m3fn), p)(x)
    monkeypatch.setenv("JIMM_GEMM_IMPL", "simt")
    b = _set(VisionTransformer(**SMALL, dtype=torch.float8_e4m3fn), p)(x)
    assert rel_err(b, a) < 2.5e-2
