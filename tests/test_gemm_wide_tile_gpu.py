"""GPU: the GEMM's 128 x 256 output tile where its shape shows.  A 256-column tile is stored as four 64-column boxes (16-bit outputs) or
eight 32-column boxes (32-bit outputs); widths that end a tile at each box boundary must write exactly the columns < N.  The fused
LayerNorm counts a row group complete when all N columns are added, also when the group's last column tile is partial (N = 384,
1152).  Tile counts run from below the SM count to several waves.  References are fp64 on operands already rounded to the operand
type; the reverse tile walk must give the bits of the forward walk."""

import pytest
import torch

from gpu_util import CODE, check, ptr, rel_err, stream
from test_kernel_paths_gpu import OUT_TOL, SENTINEL, TF32, _mk, _randn, gemm_ex

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("M", [200, 3001])  # 2 row tiles (< 1 wave) / 24 row tiles (several waves at N = 2296)
@pytest.mark.parametrize("out_t,N", [(torch.float16, n) for n in (64, 128, 192, 320, 2296)] + [(torch.bfloat16, 192)]
                         + [(torch.float32, n) for n in (32, 96, 160, 224, 288)] + [(TF32, n) for n in (32, 224)],
                         ids=lambda v: {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32", TF32: "tf32"}.get(v, str(v)))
@pytest.mark.parametrize("op", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "tf32"])
def test_wide_tile_box_boundaries(lib, op, out_t, N, M):
    """Columns >= N and rows >= roundup(M, 16) keep their sentinel; the rest is the fp64 product + bias at one output rounding.  The
    reverse tile walk writes the same bits."""
    K, ldo = 320, N + 64
    A, B, Ad, Bd = _mk(M, N, K, op, seed=N + M)
    bias = _randn(N, seed=N)
    ref = Ad @ Bd.T + bias.double()
    dt = torch.float32 if out_t == TF32 else out_t
    code = TF32 if out_t == TF32 else CODE[out_t]
    outs = []
    for rev in (0, 1):
        out = torch.full((M + 48, ldo), SENTINEL, dtype=dt, device=DEV)
        check(lib, gemm_ex(lib, A, B, out, bias=bias, out_code=code, reverse=rev))
        torch.cuda.synchronize()
        r16 = (M + 15) // 16 * 16
        assert bool((out[:, N:].float() == SENTINEL).all()), "columns >= N were written"
        assert bool((out[r16:].float() == SENTINEL).all()), "rows >= roundup(M, 16) were written"
        err = rel_err(out[:M, :N], ref)
        assert err < OUT_TOL[out_t], f"rel err {err:.2e}"
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), "reverse walk differs from the forward walk"


@pytest.mark.parametrize("N", [384, 1152, 768, 1024])  # last column tile partial (384, 1152) / whole tiles
@pytest.mark.parametrize("M", [100, 4000])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "tf32"])
def test_wide_tile_fused_layernorm(lib, dtype, M, N):
    """x += A B^T + bias with the fused LayerNorm: x equal to the unfused reduce-add, the normalised rows equal to the LayerNorm kernel on
    that x, the counters back at zero; the reverse walk gives the same bits."""
    K = 256
    A, B, _, _ = _mk(M, N, K, dtype, seed=N)
    bias = _randn(N, seed=1)
    x0 = _randn(M, N, seed=2) * 2 + 0.5
    scale, lbias = _randn(N, seed=3), _randn(N, seed=4)
    x_ref = x0.clone()
    check(lib, gemm_ex(lib, A, B, x_ref, bias=bias, residual=x_ref))
    h_ref = torch.empty(M, N, dtype=dtype, device=DEV)
    check(lib, lib.jimm_k_layernorm(ptr(x_ref), N, 1, 0, None, ptr(scale), ptr(lbias), 1e-6, ptr(h_ref), CODE[dtype], N, M, N, stream()))
    cnt = torch.zeros(M // 32 + 2, dtype=torch.int32, device=DEV)
    hs = []
    for rev in (0, 1):
        x = x0.clone()
        h = torch.full((M, N), 7.0, dtype=dtype, device=DEV)
        check(lib, gemm_ex(lib, A, B, x, bias=bias, residual=x, reverse=rev, ln=(scale, lbias, 1e-6, h, CODE[dtype], cnt)))
        torch.cuda.synchronize()
        assert torch.equal(x, x_ref), f"reverse={rev}: residual stream differs from the unfused kernel"
        tol = {torch.float32: 1e-3, torch.float16: 1e-3, torch.bfloat16: 8e-3}[dtype]
        assert rel_err(h, h_ref) < tol, f"reverse={rev}: fused LayerNorm differs from the LayerNorm kernel: {rel_err(h, h_ref):.2e}"
        assert int(cnt.abs().sum()) == 0, "completion counters not reset"
        hs.append(h)
    assert torch.equal(hs[0], hs[1]), "reverse walk differs from the forward walk"
