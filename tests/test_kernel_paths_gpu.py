"""GPU: the GEMM and patchify as the forward pass runs them, through jimm_k_gemm_ex / jimm_k_patchify_ex: more tiles than SMs on every
store epilogue, the reverse tile walk, plans built for more rows than are run, the token-scatter patch embedding, the tf32 (type 3)
stores and the padded patch layout.  References are fp64 on operands already rounded to the operand type; wherever two runs do the
same arithmetic, they must agree bit for bit."""

import math

import pytest
import torch

from gpu_util import CODE, F16, F32, check, gelu_tanh, ptr, quick_gelu, rel_err, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
TF32 = 3  # type code 3 of the jimm_k_* entry points: fp32 rounded to tf32
ACTS = [lambda v: v, gelu_tanh, quick_gelu]
SENTINEL = -768.0  # exact in fp16 / bf16 / tf32: marks memory a kernel must not write
D_LN = 768  # a width the fused LayerNorm takes (6 x 128)


def rna_tf32(x):
    """fp32 -> tf32 the way the kernels' cvt.rna.tf32.f32 rounds: to nearest, ties AWAY from zero (the oracle's _round_tf32
    rounds ties to even, so it is not the reference for bitwise checks).  Adding half an ulp to the magnitude bits and
    truncating carries into the exponent correctly."""
    u = x.contiguous().view(torch.int32)
    return ((u + 0x1000) & ~0x1FFF).view(torch.float32)


def _mk(M, N, K, dtype, seed=0):
    """A [M, K], B [N, K] in the operand type (torch.float32 = tf32 operands) and their exact fp64 values."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(DEV)
    B = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(DEV)
    A, B = (rna_tf32(A), rna_tf32(B)) if dtype == torch.float32 else (A.to(dtype), B.to(dtype))
    return A, B, A.double(), B.double()


def _randn(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


def gemm_ex(lib, A, Bw, out, *, M=None, plan_M=0, bias=None, act=0, residual=None, out_code=None, mode=2, reverse=0, tok=(0, 0, 0),
            ln=None):
    """jimm_k_gemm_ex; A holds the plan's rows (plan_M or M of them).  ln = (scale, bias, eps, ln_out, ln_code, counters).  Returns rc."""
    N, K = Bw.shape
    M = A.shape[0] if M is None else M
    ls, lb, eps, lo, lcode, cnt = ln if ln is not None else (None, None, 0.0, None, 0, None)
    return lib.jimm_k_gemm_ex(0, CODE[A.dtype], ptr(A), A.stride(0), ptr(Bw), Bw.stride(0), M, N, K, ptr(bias), act, None, ptr(residual),
                              0 if residual is None else residual.stride(0), ptr(out), CODE[out.dtype] if out_code is None else out_code,
                              out.stride(0), 0, 0, 0, mode, plan_M, reverse, *tok, ptr(ls), ptr(lb), eps, ptr(lo), lcode,
                              0 if lo is None else lo.stride(0), ptr(cnt), stream())


def _canvas(rows, cols, dtype):
    return torch.full((rows, cols), SENTINEL, dtype=dtype, device=DEV)


def _untouched(t):
    return bool((t.float() == SENTINEL).all())


OUT_TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2, torch.float32: 3e-5, TF32: 1e-3}  # one rounding of the output type
OPS = [torch.float16, torch.bfloat16, torch.float32]


# ---- more tiles than SMs on the plain-store epilogues ---------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2296, 2300])
@pytest.mark.parametrize("out_t", [torch.float16, torch.bfloat16, torch.float32, TF32], ids=["f16", "bf16", "f32", "tf32"])
@pytest.mark.parametrize("op", OPS, ids=["f16", "bf16", "tf32"])
def test_multi_tile_store_epilogues(lib, op, out_t, N):
    """24 x 18 = 432 tiles (> 3 per CTA on 132 SMs) with ragged M, N and K tails: each CTA reuses its double-buffered store boxes across
    tiles.  Columns N..ldo and rows >= M of the output are never written.  N = 2300 ends 16-bit rows inside a 16-byte chunk, where the
    TMA store would write past N: those shapes must take the LSU epilogue."""
    M, K, ldo = 3000, 1000, 2320
    A, B, Ad, Bd = _mk(M, N, K, op, seed=10)
    bias = _randn(N, seed=11)
    base = Ad @ Bd.T + bias.double()
    dt = torch.float32 if out_t == TF32 else out_t
    code = TF32 if out_t == TF32 else CODE[out_t]
    for act in (0, 1, 2):
        ref = ACTS[act](base)
        for mode in (2, 0):
            buf = _canvas(M + 40, ldo, dt)
            check(lib, gemm_ex(lib, A, B, buf, M=M, bias=bias, act=act, out_code=code, mode=mode))
            got = buf[:M, :N]
            assert rel_err(got, ref) < OUT_TOL[out_t], (act, mode, rel_err(got, ref))
            assert _untouched(buf[:, N:]), (act, mode, "columns between N and ldo written")
            assert _untouched(buf[M:]), (act, mode, "rows >= M written")


# ---- reverse tile walk ----------------------------------------------------------------------------------------------------------------
def _nk(kind):
    return (2296, 520) if kind in ("store_f16", "store_tf32", "generic") else (D_LN, 264)


def _run_kind(lib, kind, op, reverse, A, M, plan_M=0, seed=20):
    """One GEMM of epilogue `kind` on M rows of A (output buffers as tall as A, same inputs for a given seed); returns the tensors it
    may write (and the fused LayerNorm's counters)."""
    g_M = A.shape[0]
    N, K = _nk(kind)
    _, B, _, _ = _mk(8, N, K, op, seed=seed + 1)
    bias = _randn(N, seed=seed + 2)
    if kind in ("store_f16", "store_tf32", "generic"):
        out = _canvas(g_M, N + 20, torch.float16 if kind == "store_f16" else torch.float32)
        code = {"store_f16": F16, "store_tf32": TF32, "generic": F32}[kind]
        check(lib, gemm_ex(lib, A, B, out, M=M, plan_M=plan_M, bias=bias, act=1, out_code=code, mode=0 if kind == "generic" else 2,
                           reverse=reverse))
        return (out,)
    x = _randn(g_M, N, seed=seed + 3) * 2 + 0.5
    if kind == "reduce_add":
        check(lib, gemm_ex(lib, A, B, x, M=M, plan_M=plan_M, bias=bias, residual=x, reverse=reverse))
        return (x,)
    scale, lbias = _randn(N, seed=seed + 4), _randn(N, seed=seed + 5)
    h = _canvas(g_M, N, op)
    cnt = torch.zeros(g_M // 32 + 2, dtype=torch.int32, device=DEV)
    check(lib, gemm_ex(lib, A, B, x, M=M, plan_M=plan_M, bias=bias, residual=x, reverse=reverse,
                       ln=(scale, lbias, 1e-6, h, CODE[op], cnt)))
    return x, h, cnt


@pytest.mark.parametrize("kind,op", [("store_f16", torch.float16), ("store_tf32", torch.bfloat16), ("generic", torch.float32),
                                     ("reduce_add", torch.bfloat16), ("fused_ln", torch.float16), ("fused_ln", torch.float32)])
def test_reverse_walk_is_bitwise_equal(lib, kind, op):
    """run_encoder alternates the tile direction of every GEMM: walking the tiles from the end gives the same bits.  Multi-tile shapes
    (M = 6000: 47 row tiles x 18 or 6 column tiles)."""
    N, K = _nk(kind)
    A, _, _, _ = _mk(6000, N, K, op, seed=20)
    fwd = _run_kind(lib, kind, op, 0, A, 6000)
    rev = _run_kind(lib, kind, op, 1, A, 6000)
    torch.cuda.synchronize()
    for a, b in zip(fwd, rev):
        assert torch.equal(a, b), kind
    if kind == "fused_ln":
        assert int(rev[2].abs().sum()) == 0, "fused LayerNorm counters not back at zero"


# ---- plan rows > run rows -------------------------------------------------------------------------------------------------------------
PLAN_M = 4000
RUN_MS = [1, 15, 16, 17, 127, 128, 129, 1000, PLAN_M]


@pytest.mark.parametrize("kind,op", [("store_f16", torch.float16), ("store_tf32", torch.float32), ("generic", torch.bfloat16),
                                     ("reduce_add", torch.float16), ("fused_ln", torch.bfloat16), ("fused_ln", torch.float32)])
def test_plan_rows_exceed_run_rows(lib, kind, op):
    """Plans are built once for the largest batch and run on fewer rows.  The A rows >= M hold NaN (stale workspace).  Rows < M are the
    bits of a plan built for exactly M; the generic epilogue writes no row >= M, the TMA epilogues none >= roundup(M, 16), the fused
    LayerNorm normalises rows < M only and leaves its counters at zero."""
    N, K = _nk(kind)
    A0, _, _, _ = _mk(PLAN_M, N, K, op, seed=30)
    for M in RUN_MS:
        A = A0.clone()
        A[M:] = float("nan")
        big = _run_kind(lib, kind, op, M % 2, A, M, plan_M=PLAN_M, seed=30)
        exact = _run_kind(lib, kind, op, 0, A, M, plan_M=M, seed=30)  # its tensor maps end at row M: it writes no row >= M
        torch.cuda.synchronize()
        written = M if kind == "generic" else (M + 15) // 16 * 16
        for i, (b, e) in enumerate(zip(big, exact)):
            if kind == "fused_ln" and i == 2:
                assert int(b.abs().sum()) == 0 and int(e.abs().sum()) == 0, (M, "counters not back at zero")
                continue
            assert torch.equal(b[:M], e[:M]), (M, i, "rows < M differ from a plan built for exactly M")
            last = M if (kind == "fused_ln" and i == 1) else written  # i == 1: the normalised rows
            assert torch.equal(b[last:], e[last:]), (M, i, f"rows >= {last} written")
            if kind != "reduce_add" and not (kind == "fused_ln" and i == 0):  # the output canvases start as SENTINEL
                assert _untouched(b[last:]), (M, i, "rows beyond the contract written")


# ---- token-scatter patch embedding ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", OPS, ids=["f16", "bf16", "tf32"])
@pytest.mark.parametrize("n", [49, 196, 256, 576])
@pytest.mark.parametrize("tok_off", [0, 1], ids=["map", "cls"])
def test_token_scatter_patch_epilogue(lib, tok_off, n, op):
    """The default patch embedding: A rows (sample, padded patch) reduce-added through the 3-D tensor map into the position-initialised
    residual stream x[b, p + tok_off].  Pad rows of A and the samples beyond the run are NaN; the CLS row, the samples beyond the run and
    the rows past the last sample keep their bits.  More tiles than SMs; the plan is built for three more samples than are run."""
    D, K = 768, 592  # patch 14 x 3 channels, padded to 592
    n_pad = (n + 31) // 32 * 32
    S = n + tok_off
    B = max(2, 6000 // n_pad)
    plan_B = B + 3
    A, W, Ad, Wd = _mk(plan_B * n_pad, D, K, op, seed=n + tok_off)
    A3 = A.view(plan_B, n_pad, K)
    A3[:, n:] = float("nan")
    A3[B:] = float("nan")
    bias = _randn(D, seed=41)
    init = _randn(plan_B * S + 8, D, seed=42)
    x = init.clone()
    check(lib, gemm_ex(lib, A, W, x, M=B * n_pad, plan_M=plan_B * n_pad, bias=bias, residual=x, tok=(n_pad, tok_off, S)))
    torch.cuda.synchronize()
    touched = torch.zeros(x.shape[0], dtype=torch.bool, device=DEV)
    touched[: plan_B * S].view(plan_B, S)[:B, tok_off:] = True
    y = Ad.view(plan_B, n_pad, K)[:B, :n] @ Wd.T + bias.double()
    ref = init.double()[: plan_B * S].view(plan_B, S, D)[:B, tok_off:] + y
    got = x[: plan_B * S].view(plan_B, S, D)[:B, tok_off:]
    assert rel_err(got, ref) < 2e-5, rel_err(got, ref)
    assert torch.equal(x[~touched], init[~touched]), "a row the patch GEMM must not touch changed"


def test_token_scatter_rejects_malformed_arguments(lib):
    """tok_pad not a multiple of 16, or not dividing the plan's or the run's rows: -1 with a message, nothing launched."""
    D, K = 256, 64
    A, W, _, _ = _mk(4 * 64, D, K, torch.float16, seed=50)
    x = _randn(4 * 65, D, seed=51)
    x0 = x.clone()
    torch.cuda.synchronize()
    launches = lib.jimm_launch_count()
    for M, plan_M, tok in ((4 * 56, 0, (56, 1, 57)), (4 * 64, 4 * 64 + 32, (64, 1, 65)), (3 * 64 + 32, 4 * 64, (64, 1, 65))):
        rc = gemm_ex(lib, A, W, x, M=M, plan_M=plan_M, residual=x, tok=tok)
        assert rc == -1 and b"token scatter" in lib.jimm_last_error(), (M, plan_M, tok, rc)
    torch.cuda.synchronize()
    assert lib.jimm_launch_count() == launches
    assert torch.equal(x, x0)


# ---- tf32 stores are rounded (type 3 == rna(type 0) of the same call) ----------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gemm_tma", "gemm_generic", "attention", "layernorm", "patchify", "patchify_generic", "fused_ln"])
def test_tf32_store_is_rna_of_fp32(lib, kind):
    if kind in ("gemm_tma", "gemm_generic"):
        M, N, K = 1500, 1000, 400
        A, B, _, _ = _mk(M, N, K, torch.float32, seed=60)
        bias = _randn(N, seed=61)
        mode = 2 if kind == "gemm_tma" else 0
        f32, t32 = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
        check(lib, gemm_ex(lib, A, B, f32, bias=bias, act=2, mode=mode))
        check(lib, gemm_ex(lib, A, B, t32, bias=bias, act=2, mode=mode, out_code=TF32))
    elif kind == "attention":
        Bn, S, H = 3, 197, 2
        qkv = (_randn(Bn * S, 3 * H * 64, seed=62) * 1.5).half()
        f32, t32 = torch.empty(Bn * S, H * 64, device=DEV), torch.empty(Bn * S, H * 64, device=DEV)
        check(lib, lib.jimm_k_attention(ptr(qkv), F16, ptr(f32), F32, Bn, S, H, 0, stream()))
        check(lib, lib.jimm_k_attention(ptr(qkv), F16, ptr(t32), TF32, Bn, S, H, 0, stream()))
    elif kind == "layernorm":
        rows, D = 333, 768
        x = _randn(rows, D, seed=63) * 3 + 1.5
        sc, bi = _randn(D, seed=64), _randn(D, seed=65)
        f32, t32 = torch.empty(rows, D, device=DEV), torch.empty(rows, D, device=DEV)
        check(lib, lib.jimm_k_layernorm(ptr(x), D, 1, 0, None, ptr(sc), ptr(bi), 1e-6, ptr(f32), F32, D, rows, D, stream()))
        check(lib, lib.jimm_k_layernorm(ptr(x), D, 1, 0, None, ptr(sc), ptr(bi), 1e-6, ptr(t32), TF32, D, rows, D, stream()))
    elif kind in ("patchify", "patchify_generic"):
        Bn, P, C = 2, (16 if kind == "patchify" else 14), 3
        img = 4 * P
        x = _randn(Bn, img, img, C, seed=66)
        u = x.view(torch.int32)
        u[:, ::3] = (u[:, ::3] & ~0x1FFF) | 0x1000  # exact ties: rna rounds them away from zero, round-to-even would not always
        rows, k = Bn * 16, P * P * C
        f32, t32 = torch.empty(rows, k, device=DEV), torch.empty(rows, k, device=DEV)
        check(lib, lib.jimm_k_patchify(ptr(x), F32, Bn, img, img, C, P, ptr(f32), F32, stream()))
        check(lib, lib.jimm_k_patchify(ptr(x), F32, Bn, img, img, C, P, ptr(t32), TF32, stream()))
        assert not torch.equal(f32, t32)
    else:  # fused LayerNorm of the fp32 (tf32) mode vs the LayerNorm kernel's fp32 store on the same x
        M, N, K = 2000, D_LN, 256
        A, B, _, _ = _mk(M, N, K, torch.float32, seed=67)
        bias, sc, bi = _randn(N, seed=68), _randn(N, seed=69), _randn(N, seed=70)
        x0 = _randn(M, N, seed=71) * 2 + 0.5
        x_ref = x0.clone()
        check(lib, gemm_ex(lib, A, B, x_ref, bias=bias, residual=x_ref))
        f32 = torch.empty(M, N, device=DEV)
        check(lib, lib.jimm_k_layernorm(ptr(x_ref), N, 1, 0, None, ptr(sc), ptr(bi), 1e-6, ptr(f32), F32, N, M, N, stream()))
        x, t32 = x0.clone(), torch.empty(M, N, device=DEV)
        cnt = torch.zeros(M // 32 + 2, dtype=torch.int32, device=DEV)
        check(lib, gemm_ex(lib, A, B, x, bias=bias, residual=x, ln=(sc, bi, 1e-6, t32, TF32, cnt)))
        torch.cuda.synchronize()
        assert torch.equal(x, x_ref)
    torch.cuda.synchronize()
    assert torch.isfinite(f32).all()
    assert torch.equal(t32, rna_tf32(f32)), kind


@pytest.mark.parametrize("K", [8, 200, 592, 1000])
def test_tf32_operand_k_tails(lib, K):
    """tf32 operands, K not a multiple of the 32-element k-block (592: the padded patch-14 GEMM); both epilogues, ragged M and N."""
    M, N = 333, 520
    A, B, Ad, Bd = _mk(M, N, K, torch.float32, seed=K)
    ref = Ad @ Bd.T
    for mode in (2, 0):
        out = torch.empty(M, N, device=DEV)
        check(lib, gemm_ex(lib, A, B, out, mode=mode))
        assert rel_err(out, ref) < 2e-5, (mode, rel_err(out, ref))


@pytest.mark.parametrize("op,K", [(torch.float16, 100), (torch.bfloat16, 36), (torch.float32, 98)], ids=["f16", "bf16", "tf32"])
def test_operand_k_tail_inside_16_bytes(lib, op, K):
    """K x element size not a multiple of 16 bytes, rows strided to the next 16 bytes: the columns past K (NaN here) are not operands."""
    M, N = 300, 264
    ld = (K + 7) // 8 * 8
    A, B, Ad, Bd = _mk(M, N, K, op, seed=90)
    Ap = torch.full((M, ld), float("nan"), dtype=op, device=DEV)
    Bp = torch.full((N, ld), float("nan"), dtype=op, device=DEV)
    Ap[:, :K], Bp[:, :K] = A, B
    ref = Ad @ Bd.T
    for mode in (2, 0):
        out = torch.empty(M, N, device=DEV)
        check(lib, gemm_ex(lib, Ap[:, :K], Bp[:, :K], out, mode=mode))
        assert rel_err(out, ref) < 2e-5, (mode, rel_err(out, ref))


# ---- padded patchify -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_t", [torch.float16, torch.bfloat16, TF32], ids=["f16", "bf16", "tf32"])
@pytest.mark.parametrize("in_t", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("C", [1, 3, 4])  # 1, 3: generic kernel (ldk 200, 592); 4: vectorised kernel (784 columns, no pad)
def test_patchify_padded_layout(lib, C, in_t, out_t):
    """The patch GEMM's A operand: rows_per_sample = n_pad, row stride ldk = roundup(P*P*C, 8).  The valid region is the torch
    reshape bit for bit, pad columns are exactly 0, pad rows keep their NaN; H != W and a remainder row of pixels the VALID conv
    drops."""
    Bn, P, H, W = 3, 14, 100, 112
    gh, gw = H // P, W // P
    n = gh * gw
    n_pad = (n + 31) // 32 * 32
    PPC = P * P * C
    ldk = (PPC + 7) // 8 * 8
    x = (_randn(Bn, H, W, C, seed=C) * 2).to(in_t)
    dt = torch.float32 if out_t == TF32 else out_t
    out = torch.full((Bn * n_pad, ldk), float("nan"), dtype=dt, device=DEV)
    code = TF32 if out_t == TF32 else CODE[out_t]
    check(lib, lib.jimm_k_patchify_ex(ptr(x), CODE[in_t], Bn, H, W, C, P, ptr(out), code, n_pad, ldk, stream()))
    torch.cuda.synchronize()
    ref = x[:, : gh * P, : gw * P].reshape(Bn, gh, P, gw, P, C).permute(0, 1, 3, 2, 4, 5).reshape(Bn, n, PPC).float()
    ref = rna_tf32(ref) if out_t == TF32 else ref.to(out_t)
    o = out.view(Bn, n_pad, ldk)
    assert torch.equal(o[:, :n, :PPC], ref)
    assert torch.equal(o[:, :n, PPC:], torch.zeros_like(o[:, :n, PPC:])), "pad columns not zero"
    assert torch.isnan(o[:, n:].float()).all(), "pad rows written"


def test_patchify_rejects_too_few_rows_per_sample(lib):
    x = torch.zeros(2, 28, 28, 3, device=DEV)
    out = torch.zeros(8, 592, device=DEV)
    assert lib.jimm_k_patchify_ex(ptr(x), F32, 2, 28, 28, 3, 14, ptr(out), F32, 3, 592, stream()) == -1
    assert b"rows_per_sample" in lib.jimm_last_error()


# ---- generic epilogue with a separate residual (MAP-head fc2) ------------------------------------------------------------------------
@pytest.mark.parametrize("out_t", [torch.float32, torch.float16], ids=["f32", "f16"])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("mode", [0, 2])  # mode 2 falls back to the generic epilogue: the residual is not the output
def test_generic_separate_residual(lib, mode, act, out_t):
    """out = act(A B^T + bias) + residual with residual != out and ldr != ldo; the residual keeps its bits, columns N..ldo stay
    untouched.  Multi-tile and ragged."""
    M, N, K = 1000, 700, 3072
    A, B, Ad, Bd = _mk(M, N, K, torch.bfloat16, seed=80)
    bias = _randn(N, seed=81)
    res_buf = _randn(M, N + 36, seed=82)
    res = res_buf[:, :N]
    res0 = res_buf.clone()
    out = _canvas(M, N + 12, out_t)
    check(lib, gemm_ex(lib, A, B, out, bias=bias, act=act, residual=res, mode=mode))
    torch.cuda.synchronize()
    ref = ACTS[act](Ad @ Bd.T + bias.double()) + res.double()
    assert rel_err(out[:, :N], ref) < OUT_TOL[out_t], rel_err(out[:, :N], ref)
    assert _untouched(out[:, N:])
    assert torch.equal(res_buf, res0)
