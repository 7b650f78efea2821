"""CPU: the FP8 oracle's quantiser (tests/fp8_oracle.py) against torch.float8_e4m3fn, and its Semantics knob."""

import torch

import fp8_oracle as F
import jimm_oracle as O


def _all_finite_e4m3():
    v = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).to(torch.float64)
    return torch.sort(v[torch.isfinite(v)].unique()).values  # -448 .. 448, one zero


def test_round_e4m3_matches_torch_on_grid_and_ties():
    grid = _all_finite_e4m3()
    assert float(grid.max()) == 448.0 and float(grid[grid > 0].min()) == 2.0 ** -9
    mids = (grid[1:] + grid[:-1]) / 2  # every tie between neighbours, subnormal ones included
    quarter = grid[:-1] + (grid[1:] - grid[:-1]) / 4
    for y in (grid, mids, quarter, torch.tensor([2.0 ** -10, 2.0 ** -11, 3 * 2.0 ** -11, -2.0 ** -10, 0.0, -0.0, 447.9, 448.0])):
        y32 = y.to(torch.float32)  # these values are fp32-exact
        assert torch.equal(y32.to(torch.float64), y)
        want = y32.to(torch.float8_e4m3fn).to(torch.float64)
        assert torch.equal(F.round_e4m3(y), want), y[F.round_e4m3(y) != want][:8]
    g = torch.Generator().manual_seed(0)
    r = (torch.randn(100000, generator=g) * torch.pow(2.0, torch.randint(-12, 9, (100000,), generator=g).float())).clamp(-448, 448)
    assert torch.equal(F.round_e4m3(r.double()), r.to(torch.float8_e4m3fn).to(torch.float64))


def _brute_scale(a: float) -> float:
    if a == 0:
        return 1.0
    k = -126
    while a / 2.0 ** k > 448.0:
        k += 1
    return 2.0 ** k


def test_row_scales_and_bytes():
    rows = []
    for j in (-20, -3, 0, 5, 20):
        base = torch.linspace(-1, 1, 64, dtype=torch.float32)
        rows.append(base * 448.0 * 2.0 ** j)  # amax exactly 448 x 2^j: s = 2^j, the end elements become +-448
        rows.append(base * 448.0 * 2.0 ** j * 1.0001)  # just above: s = 2^(j + 1)
        rows.append(base * 2.0 ** j * 0.3)
    rows.append(torch.zeros(64))  # zero row: s = 1, zero bytes
    rows.append(torch.full((64,), 2.0 ** -140))  # fp32 subnormal row: k clamps at -126
    x = torch.stack(rows)
    q, s = F.quantize_rows(x)
    for i in range(x.shape[0]):
        assert float(s[i]) == _brute_scale(float(x[i].abs().max())) or (i == x.shape[0] - 1 and float(s[i]) == 2.0 ** -126), i
    assert torch.equal(q, (x / s.unsqueeze(1)).to(torch.float8_e4m3fn))
    assert float(q[0].to(torch.float32).abs().max()) == 448.0 and float(s[0]) == 2.0 ** -20
    assert float(s[1]) == 2.0 ** -19
    assert float(s[-2]) == 1.0 and int(q[-2].view(torch.uint8).abs().max()) == 0


def test_fp8_semantics_knob_moves_only_qkv_and_fc1():
    """Without `active()` (or with fp8=False) the FP8 Semantics is the fp16 oracle; with it, the result moves by e4m3-sized errors."""
    D, M, H, L = 128, 512, 2, 2
    g = torch.Generator().manual_seed(1)
    p = {}
    O._rand_blocks(p, g, "", L, D, H, M)
    p = {k: v.to(torch.float64) for k, v in O.cast_params(p, torch.float32).items()}
    x = torch.randn(2, 9, D, generator=g, dtype=torch.float64)
    f16 = O.transformer(p, "", x, L, H, False, None, 1e-6, O.Semantics(operand_round="fp16"))
    with F.active():
        off = O.transformer(p, "", x, L, H, False, None, 1e-6, F.Fp8Semantics(operand_round="fp16", fp8=False))
        on = O.transformer(p, "", x, L, H, False, None, 1e-6, F.FP8)
    assert torch.equal(off, f16)
    d = float(((on - x) - (f16 - x)).abs().max() / (f16 - x).abs().max())
    assert 1e-3 < d < 0.2, d
