"""CPU restatement of the FP8 compute mode (dtype=torch.float8_e4m3fn) for the tests.

The mode is dtype=float16 except that the QKV and FC1 GEMMs of every encoder block run on float8 e4m3 operands:
  - scales are powers of two, one per A row (token) and one per B row (output channel): for a row with absolute maximum a > 0,
    s = 2^k with the smallest integer k such that a / s <= 448 (k >= -126, so s stays a normal fp32); s = 1 when a = 0;
  - an element x is stored as e4m3(x / s), rounded to nearest even; x / s is exact and never exceeds 448;
  - the GEMM accumulates the e4m3 products and returns acc * (s_row * s_col) + bias.
The A row is the block LayerNorm's fp32 output, the B row the weight's fp32 row.  Everything else keeps the oracle's fp16 operand
rounding.  `FP8` is the Semantics knob; `active()` lets jimm_oracle's encoder blocks honour it (the oracle module itself is the
parity yardstick of the other modes and stays as it is)."""

from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass
from unittest import mock

import torch

import jimm_oracle as O

E4M3_MAX = 448.0


def e4m3_scale(amax: torch.Tensor) -> torch.Tensor:
    """Row scales s = 2^k (fp32) from row absolute maxima, from the exponent bits (frexp is exact)."""
    a = amax.to(torch.float64)
    m, e = torch.frexp(a)  # a = m 2^e, m in [0.5, 1); a <= 448 2^k = 0.875 2^(9 + k)
    k = e.to(torch.int64) - 9 + (m > 0.875).to(torch.int64)
    k = torch.where(a > 0, torch.clamp(k, min=-126), torch.zeros_like(k))
    k = torch.where(torch.isinf(a), torch.full_like(k, 255), k)  # an infinite row: s = inf, the row dequantises to NaN
    return torch.ldexp(torch.ones_like(a), k.to(torch.float64)).to(torch.float32)


def round_e4m3(y: torch.Tensor) -> torch.Tensor:
    """Round to the nearest e4m3 value (ties to even), saturating at +-448; fp64 in, fp64 out.  Normal numbers have 3 mantissa bits
    below the leading one; below 2^-6 the spacing is the subnormal step 2^-9."""
    y = y.to(torch.float64)
    a = y.abs()
    _, e = torch.frexp(a)  # leading bit 2^(e - 1)
    quantum = torch.ldexp(torch.ones_like(a), (torch.clamp(e - 1, min=-6) - 3).to(torch.float64))
    r = torch.clamp(torch.round(a / quantum) * quantum, max=E4M3_MAX)  # torch.round: half to even
    return torch.copysign(r, y)


def quantize_rows(x: torch.Tensor):
    """fp32 rows -> (float8_e4m3fn values, fp32 scales [rows]), as the LayerNorm kernel and the weight quantiser store them."""
    x = x.to(torch.float32)
    s = e4m3_scale(torch.where(torch.isnan(x), 0.0, x.abs()).amax(-1))  # NaN does not count towards the maximum (fmaxf on the device)
    q = round_e4m3(x / s.unsqueeze(-1))  # division by a power of two: exact (also into fp32 subnormals, as on the device)
    return q.to(torch.float8_e4m3fn), s


def dequant(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    return q.to(torch.float64) * s.to(torch.float64).unsqueeze(-1)


def fp8_linear(h: torch.Tensor, w_nk: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """e4m3 GEMM: h [..., K] (quantised per row from its fp32 value), w_nk [N, K] (quantised per row); exact products and sum."""
    hq = dequant(*quantize_rows(h))
    wq = dequant(*quantize_rows(w_nk))
    return hq.to(h.dtype) @ wq.to(h.dtype).T + bias.to(h.dtype)


@dataclass
class Fp8Semantics(O.Semantics):
    fp8: bool = True  # QKV and FC1 of every encoder block on e4m3 operands; operand_round everywhere else


FP8 = Fp8Semantics(operand_round="fp16")


def _block(p, prefix, x, num_heads, eps, use_quick_gelu, mask, sem):
    """TransformerEncoder.__call__ with the FP8 mode's QKV and FC1 (the rest as jimm_oracle.transformer_encoder, act_round None)."""
    if mask is not None:
        s = min(x.shape[1], mask.shape[0])
        mask = mask[:s, :s]
    r = lambda t: O.round_operand(t, sem.operand_round)
    a = prefix + "attn."
    h = O.layer_norm(x, p[prefix + "norm1.scale"], p[prefix + "norm1.bias"], eps, sem)
    Wq, Wk, Wv = p[a + "query.kernel"], p[a + "key.kernel"], p[a + "value.kernel"]
    D, H, d = Wq.shape
    w_qkv = torch.cat([W.reshape(D, H * d).T for W in (Wq, Wk, Wv)], 0)  # the fused [3D, D] K-major operand
    b_qkv = torch.cat([p[a + n + ".bias"].reshape(H * d) for n in ("query", "key", "value")])
    qkv = fp8_linear(h, w_qkv, b_qkv)
    q, k, v = qkv.split(H * d, dim=-1)
    B, S, _ = q.shape
    q = q.reshape(B, S, H, d).permute(0, 2, 1, 3) / math.sqrt(d)
    k = k.reshape(B, S, H, d).permute(0, 2, 1, 3)
    v = v.reshape(B, S, H, d).permute(0, 2, 1, 3)
    w = r(q) @ r(k).transpose(-1, -2)
    if mask is not None:
        w = torch.where(mask != 0, w, torch.finfo(w.dtype).min)
    o = r(torch.softmax(w, dim=-1)) @ r(v)
    o = o.permute(0, 2, 1, 3).reshape(B, S, H * d)
    x = x + r(o) @ r(p[a + "out.kernel"].reshape(H * d, D)) + p[a + "out.bias"]
    h = O.layer_norm(x, p[prefix + "norm2.scale"], p[prefix + "norm2.bias"], eps, sem)
    h = fp8_linear(h, p[prefix + "mlp.layers.0.kernel"].T, p[prefix + "mlp.layers.0.bias"])
    h = O._act(h, use_quick_gelu, sem)
    h = O.linear(h, p[prefix + "mlp.layers.3.kernel"], p[prefix + "mlp.layers.3.bias"], sem)
    return x + h


@contextlib.contextmanager
def active():
    """Inside: jimm_oracle's forwards run `_block` for every encoder block whose Semantics has fp8 set."""
    orig = O.transformer_encoder

    def te(p, prefix, x, num_heads, eps, use_quick_gelu, mask, sem=O.JIMM):
        if getattr(sem, "fp8", False):
            return _block(p, prefix, x, num_heads, eps, use_quick_gelu, mask, sem)
        return orig(p, prefix, x, num_heads, eps, use_quick_gelu, mask, sem)

    with mock.patch.object(O, "transformer_encoder", te):
        yield
