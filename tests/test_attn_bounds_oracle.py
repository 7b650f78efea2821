"""CPU: the attention bounds of attn_bounds hold for fp32 emulations of the kernels on every input family, and catch mutants of them,
two of which the older tolerance checks pass (a probability flush below 2^-20 and one output column off by 2^-10)."""

import math

import pytest
import torch

import attn_bounds as AB
from attn_oracle import _check_tile_faithful
from bounds_util import assert_within

C_QK = AB.C_QK[torch.float16]
SHAPES = [(2, 129, 3, 72, False), (2, 200, 3, 24, True), (1, 65, 3, 128, False), (2, 63, 3, 8, True)]


def _inputs(family, B, S, H, d, seed=1):
    io = torch.bfloat16 if family == "big" else torch.float16
    qkv = AB.make_qkv(family, B, S, H, d, io, seed)
    return io, qkv, AB.split_qkv(qkv, B, S, H, d)


def _ratio(out, ref, bound):
    return float(((out.double() - ref).abs() / bound).max())


@pytest.mark.parametrize("family", AB.FAMILIES)
def test_emulations_within_bound(family):
    """emulate_probs and emulate_flash (fp32 output) within probs_ref_bound / flash_ref_bound at every element."""
    for B, S, H, d, causal in SHAPES:
        io, _, (q, k, v) = _inputs(family, B, S, H, d)
        case = f"emulated {family} B={B} S={S} H={H} d={d} causal={causal}"
        P, bound = AB.probs_ref_bound(q, k, causal, C_QK)
        assert_within(case, "probs", AB.emulate_probs(q, k, causal), P, bound)
        o, bound = AB.flash_ref_bound(q, k, v, causal, C_QK, io, "f32")
        assert_within(case, "flash output", AB.emulate_flash(q, k, v, causal, io), o, bound)


def test_sink_reaches_below_the_subnormals():
    """The sink family puts probabilities across fp32's subnormal range and below 2^-149, where the emulation returns 0 within the floor."""
    _, _, (q, k, _) = _inputs("sink", 2, 129, 3, 72)
    P, bound = AB.probs_ref_bound(q, k, False, C_QK)
    pe = AB.emulate_probs(q, k, False).double()
    assert float(P[P > 0].min()) < 2.0 ** -149 and bool(((P > 2.0 ** -149) & (P < 2.0 ** -126)).any())
    assert bool((pe[P < 2.0 ** -150] == 0).all())
    assert_within("emulated sink", "probs", pe, P, bound)


def _old_allclose(out, ref):
    """test_attentions_gpu's elementwise check of jimm_k_attn_probs."""
    return torch.allclose(out.double(), ref, rtol=1e-4, atol=2e-6)


def _old_row_sums(out):
    """test_attentions_gpu's row-sum check of jimm_k_attn_probs."""
    return torch.allclose(out.double().sum(-1), torch.ones(out.shape[:-1], dtype=torch.float64), rtol=0, atol=1e-5)


@pytest.mark.parametrize("mutant,family", [("flush", "sink"), ("scale", "flat"), ("dp_scale", "mild"), ("no_alpha_l", "late")])
def test_probs_mutants_fail_the_bound(mutant, family):
    """Each mutant of emulate_probs fails the bound.  The flush of p < 2^-20 passes both older checks (allclose and row sums); the
    2^-14 scaling passes the allclose (only the row sums see it)."""
    B, S, H, d = 2, 200, 3, 72
    _, _, (q, k, _) = _inputs(family, B, S, H, d)
    P, bound = AB.probs_ref_bound(q, k, False, C_QK)
    out = AB.emulate_probs(q, k, False, mutant=mutant)
    assert _ratio(out, P, bound) > 1.0, mutant
    with pytest.raises(AssertionError, match=r"\|out - ref\| / bound = .* at \("):
        assert_within(f"mutant {mutant}", "probs", out, P, bound)
    if mutant == "flush":
        assert _old_allclose(out, P) and _old_row_sums(out)
    if mutant == "scale":
        assert _old_allclose(out, P) and not _old_row_sums(out)


def _flash_layout(o, B, S, H, d):
    """[B H, S, d] -> the kernel's [B S, H d]."""
    return o.reshape(B, H, S, d).permute(0, 2, 1, 3).reshape(B * S, H * d)


@pytest.mark.parametrize("mutant,family", [("column", "colscale"), ("dp_scale", "mild"), ("no_alpha_l", "late")])
def test_flash_mutants_fail_the_bound(mutant, family):
    """Each mutant of emulate_flash fails the bound.  One column 2^-10 off, on the columns scaled by 2^-12 (odd: no cancellation),
    passes the older tile-faithful check (per-row error relative to the row's largest |ref|)."""
    B, S, H, d = 2, 200, 3, 72
    io, qkv, (q, k, v) = _inputs(family, B, S, H, d)
    o, bound = AB.flash_ref_bound(q, k, v, False, C_QK, io, "f32")
    out = AB.emulate_flash(q, k, v, False, io, mutant=mutant, col=1)
    assert _ratio(out, o, bound) > 1.0, mutant
    if mutant == "column":
        assert float(v[..., 1].abs().max()) < 2.0 ** -9 < 2.0 ** 9 < float(v[..., -1].abs().max())
        _check_tile_faithful("mutant column", _flash_layout(out, B, S, H, d), qkv, B, S, H, d, False)


def test_rho_is_exact_for_a_shifted_key():
    """_rho on one key with an exponent error bound e and exact others: the bound 2^e / (1 - P_j + P_j 2^-e) - 1 covers the actual
    relative move of P^_j when that key's exponent is off by exactly e, 2^e / (1 - P_j + P_j 2^e) - 1."""
    P = torch.tensor([[0.5, 0.3, 0.2]], dtype=torch.float64)
    e = 1e-3
    E = torch.tensor([[e, 0.0, 0.0]], dtype=torch.float64)
    rho = AB._rho(P, E, torch.ones_like(P, dtype=torch.bool))
    exact = 2 ** e / (0.5 + 0.5 * 2 ** e) - 1
    assert rho[0, 0] >= exact and math.isclose(float(rho[0, 0]), 2 ** e / (0.5 + 0.5 * 2 ** -e) - 1, rel_tol=1e-12)
