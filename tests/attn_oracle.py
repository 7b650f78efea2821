"""CPU restatement of the attention weights of the vision and text towers (HF output_attentions), on jimm_oracle's layers.

Block k's weights are softmax((q / sqrt(d)) k^T masked) per head, with q and k what O.multi_head_attention computes from
norm1(x_k), x_k the residual stream entering block k (tokens_oracle's hidden states): [B, H, S, S].  The MAP head's weights are the
same softmax with its probe as the query and ln_post(x_L) as the keys: [B, H, 1, S], the weights its pooled output sums with.  The
arithmetic is jimm_oracle's, step for step (O.multi_head_attention stops right after the softmax here).
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

import jimm_oracle as O
import naflex_oracle as NF
import tokens_oracle as TO
from gpu_util import record_parity


@dataclass
class AttnSemantics(O.Semantics):
    """O.Semantics with q and k rounded to `qk_round` ("fp16" / "bf16") before the scores: the attention I/O type the CUDA path stores
    its qkv buffer in (fp16 in the fp32 and fp16 compute modes, bf16 in bf16 mode), on which its weights are defined.  The MAP head's
    probe query stays fp32 there; only its keys are rounded."""

    qk_round: Optional[str] = None


def attention_weights(p: O.Params, prefix: str, xq, xkv, num_heads: int, mask=None, sem: O.Semantics = O.JIMM, round_q: bool = True) -> torch.Tensor:
    """The softmax of O.multi_head_attention(p, prefix, xq, xkv, num_heads, mask, sem): [B, H, Sq, Sk].  With AttnSemantics.qk_round, k
    (and q when round_q) are rounded to it first."""
    Wq, Wk = p[prefix + "query.kernel"], p[prefix + "key.kernel"]
    D, H, d = Wq.shape
    assert H == num_heads
    r = lambda t: O.round_operand(t, sem.operand_round)
    o_ = lambda t: O._out(t, sem)
    q = o_(o_(r(xq) @ r(Wq.reshape(D, H * d))) + O._prm(p[prefix + "query.bias"].reshape(H * d), sem))
    k = o_(o_(r(xkv) @ r(Wk.reshape(D, H * d))) + O._prm(p[prefix + "key.bias"].reshape(H * d), sem))
    qk = getattr(sem, "qk_round", None)
    if qk is not None:
        q = O.round_operand(q, qk) if round_q else q
        k = O.round_operand(k, qk)
    B, Sq, _ = q.shape
    Sk = k.shape[1]
    q = o_(q.reshape(B, Sq, H, d).permute(0, 2, 1, 3) / math.sqrt(d))
    k = k.reshape(B, Sk, H, d).permute(0, 2, 1, 3)
    w = o_(r(q) @ r(k).transpose(-1, -2))
    if mask is not None:
        w = torch.where(mask != 0, w, torch.finfo(w.dtype).min)
    return o_(torch.softmax(w, dim=-1))


def _blocks(p: O.Params, prefix: str, xs, num_heads: int, mask, sem: O.Semantics) -> List[torch.Tensor]:
    """Block k's weights for k = 0 .. L-1, xs = [x_0, ..., x_L, ...] (block eps 1e-6 unless sem overrides it)."""
    eps = sem.block_eps if sem.block_eps is not None else 1e-6
    out = []
    for i in range(len(xs) - 2):
        bp = f"{prefix}blocks.layers.{i}."
        m = mask[: xs[i].shape[1], : xs[i].shape[1]] if mask is not None else None
        h = O.layer_norm(xs[i], p[bp + "norm1.scale"], p[bp + "norm1.bias"], eps, sem)
        out.append(attention_weights(p, bp + "attn.", h, h, num_heads, m, sem))
    return out


def map_weights(p: O.Params, prefix: str, final, num_heads: int, sem: O.Semantics = O.JIMM) -> torch.Tensor:
    """The MAP head's probe weights over the final-normed tokens `final` [B, S, D]: [B, H, 1, S] (O.map_head's attention)."""
    probe = O._prm(p[prefix + "probe"], sem).expand(final.shape[0], -1, -1)
    return attention_weights(p, prefix + "attn.", probe, final, num_heads, None, sem, round_q=False)


def vision_attn(p: O.Params, prefix: str, img, cfg: O.TowerCfg, sem: O.Semantics = O.JIMM) -> Tuple[List[torch.Tensor], Optional[torch.Tensor]]:
    """([block 0 .. L-1 weights, each [B, H, S, S]], the MAP head's [B, H, 1, S] or None on a CLS tower)."""
    xs = TO.vision_hidden(p, prefix, img, cfg, sem)
    blocks = _blocks(p, prefix + "transformer.", xs, cfg.num_heads, None, sem)
    mw = map_weights(p, prefix + "MAPHead.", xs[-1], cfg.num_heads, sem) if cfg.pooling_type == "MAP" else None
    return blocks, mw


def vit_attn(p: O.Params, cfg: O.ViTCfg, img, sem: O.Semantics = O.JIMM):
    return vision_attn(p, "encoder.", img, cfg.tower(), sem)


def clip_image_attn(p: O.Params, cfg: O.DualCfg, img, sem: O.Semantics = O.JIMM):
    return vision_attn(p, "vision_model.", img, cfg.clip_tower(), sem)


def siglip_image_attn(p: O.Params, cfg: O.DualCfg, img, sem: O.Semantics = O.JIMM):
    return vision_attn(p, "vision_model.", img, cfg.siglip_tower(), sem)


def _text_attn(p: O.Params, cfg: O.DualCfg, text, kind: str, sem: O.Semantics) -> List[torch.Tensor]:
    xs = (TO.clip_text_hidden if kind == "clip" else TO.siglip_text_hidden)(p, cfg, text, sem)
    mask = torch.tril(torch.ones(cfg.context_length, cfg.context_length, dtype=xs[0].dtype)) if kind == "clip" else None
    return _blocks(p, "text_model.", xs, cfg.transformer_heads, mask, sem)


def clip_text_attn(p: O.Params, cfg: O.DualCfg, text, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    """Block 0 .. L-1 weights of the causal CLIP text tower, each [B, H, T, T] (0 above the diagonal)."""
    return _text_attn(p, cfg, text, "clip", sem)


def siglip_text_attn(p: O.Params, cfg: O.DualCfg, text, sem: O.Semantics = O.JIMM) -> List[torch.Tensor]:
    return _text_attn(p, cfg, text, "siglip", sem)


def naflex_attn(p: O.Params, cfg: O.DualCfg, pixel_values, spatial_shapes, sem: O.Semantics = O.JIMM):
    """SigLIP 2 NaFlex on the processor's pixel_values: per sample b, ([block weights [H, n_b, n_b]], MAP weights [H, 1, n_b]),
    n_b = gh_b * gw_b (the position table resampled to the sample's grid, as naflex_oracle.encode_patches does)."""
    t = NF.naflex_tower(cfg)
    P, g, k = t.patch_size, t.img_size // t.patch_size, "vision_model.position_embeddings"
    out = []
    for b, (gh, gw) in enumerate(torch.as_tensor(spatial_shapes).tolist()):
        img = NF.rows_to_image(pixel_values[b, : gh * gw], gh, gw, P)[None]
        pb = {**p, k: NF.resample_pos_aa(p[k], g, gh, gw)}
        blocks, mw = vision_attn(pb, "vision_model.", img, t, sem)
        out.append(([w[0] for w in blocks], mw[0]))
    return out


# ---------------------------------------------------------------------------------------------------------------- the attention kernel
# fp64 references of one attention call on the fused qkv buffer [B * S, 3 * H * d] (q, k, v of head h at columns h d, D + h d, 2 D + h d),
# for the kernel tests: exact softmax attention, and the attention kernel's own steps restated in fp64.
def _scale_log2(d):
    """The kernel's fp32 constant: fl(fl(1 / sqrt(d)) * fl(log2 e))."""
    return float(torch.tensor(1.0 / math.sqrt(d), dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32))


def _attn_ref(qkv, B, S, H, d, causal):
    q, k, v = qkv.double().reshape(B, S, 3, H, d).permute(2, 0, 3, 1, 4)
    w = (q / math.sqrt(d)) @ k.transpose(-1, -2)
    if causal:
        w = w.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=qkv.device)), float("-inf"))
    return (torch.softmax(w, -1) @ v).permute(0, 2, 1, 3).reshape(B * S, H * d)


def _attn_tile_ref(qkv, B, S, H, d, causal):
    """attention_kernel restated in fp64: 64-key tiles from key 0, a running row maximum m of the raw scores q.k, alpha =
    exp2((m_old - m_new) c), p = exp2(s c - m_new c), l = l alpha + sum(p) with p unrounded, o = o alpha + round(p) . v, with p
    rounded to the operand type as the kernel packs it for the P.V MMA (c = _scale_log2(d)).  A causal row sees no key past itself, so
    the tiles after its own add nothing (alpha = 1, p = 0) and need no special case."""
    c = _scale_log2(d)
    q, k, v = qkv.double().reshape(B, S, 3, H, d).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2)
    if causal:
        s = s.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=qkv.device)), float("-inf"))
    m = torch.full((B, H, S, 1), float("-inf"), dtype=torch.float64, device=qkv.device)
    l = torch.zeros_like(m)
    o = torch.zeros(B, H, S, d, dtype=torch.float64, device=qkv.device)
    for k0 in range(0, S, 64):
        sj = s[..., k0:k0 + 64]
        m_new = torch.maximum(m, sj.amax(-1, keepdim=True))
        alpha = torch.exp2((m - m_new) * c)  # m = -inf on the first tile: alpha = 0
        p = torch.exp2(sj * c - m_new * c)
        l = l * alpha + p.sum(-1, keepdim=True)
        o = o * alpha + p.to(qkv.dtype).double() @ v[..., k0:k0 + 64, :]
        m = m_new
    return (o / l).permute(0, 2, 1, 3).reshape(B * S, H * d)


# Worst values over seven runs of test_attention, test_attention_split_variant and test_attention_lazy_rescale_path (inputs are
# unseeded) on an H100 80GB HBM3 at a 400 W power limit: per row 6.5e-4 (fp16) and 3.9e-3 (bf16), bias 1.3e-6 and 4.0e-6.  The
# per-row floor is one ulp of P on a row's dominant key: the kernel's fp32 p and the fp64 p now and then round to neighbouring
# operand values.  Those flips have no sign, so the bias is their sampling noise (largest for bf16 at small S); a P packer that
# truncates instead of rounding moved it to 3.5e-5 .. 1.9e-3 (unchanged only at S = 1, where most p are exactly 1).  Per-row bounds
# are 3x, bias bounds 4-5x the worst value.
TILE_ROW_TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}
TILE_BIAS_TOL = {torch.float16: 5e-6, torch.bfloat16: 2e-5}
EXACT_TOL = {torch.float16: 3e-3, torch.bfloat16: 2e-2}  # against _attn_ref


def _check_tile_faithful(case, out, qkv, B, S, H, d, causal, ref=None):
    """The fp32 output against _attn_tile_ref (or `ref`, the same computed another way): the largest error of any (sample, head, query
    row) relative to that row's largest |ref|, and the mean error along sign(ref) relative to mean |ref| (a P packer that truncates
    instead of rounding to nearest biases every output towards zero by about half an ulp of the operand type)."""
    ref = (_attn_tile_ref(qkv, B, S, H, d, causal) if ref is None else ref).reshape(B, S, H, d)
    e = out.double().reshape(B, S, H, d) - ref
    row = float((e.abs().amax(-1) / ref.abs().amax(-1)).max())
    bias = float((e * ref.sign()).mean() / ref.abs().mean())
    dn = str(qkv.dtype).replace("torch.", "")
    record_parity(case, "per-row", dn, "tile-faithful fp64", TILE_ROW_TOL[qkv.dtype], row)
    record_parity(case, "bias", dn, "tile-faithful fp64", TILE_BIAS_TOL[qkv.dtype], abs(bias))
    assert row < TILE_ROW_TOL[qkv.dtype], (case, "per-row", row)
    assert abs(bias) < TILE_BIAS_TOL[qkv.dtype], (case, "bias", bias)
