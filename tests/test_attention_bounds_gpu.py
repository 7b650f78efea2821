"""The attention kernels checked element by element against fp64: |out - ref| <= bound at every probability and every output, with
the bounds of attn_bounds (derived there from each kernel's steps), on the input families of attn_bounds.make_qkv.

- test_score_accumulation_constant measures c_qk, the accumulation constant of score_tile's wgmma, through jimm_k_attn_probs itself.
- jimm_k_attn_probs (fp32 output; the 16-bit outputs are tested bit for bit as casts of it), dense and packed, causal and not.
- jimm_k_attention_hd (f32, tf32, f16, bf16 outputs; reverse 0 and 1, which must give the same bits) and jimm_k_attention_packed_ex.
- jimm_k_map_attention_hd, jimm_k_map_attention_packed and jimm_k_map_attention_probs (pooled output and probe weights).
Shapes: the towers' (S = 197 / H 12 / d 64, 257 / 16 / 80, 577 / 16 / 64, 729 / 16 / 72, the causal CLIP text tower at 77 and the
SigLIP text tower at 64), the key-tile edges S = 1, 2, 63, 64, 65, 127, 129 at d = 8 .. 128 (every padded width), packed samples of
1, 63, 64, 65 and 200 tokens, and one long row (S = 4096; the MAP head 8192).  A failure names the worst element as (sample, head,
row, key or column) with out, ref and bound.
"""

import math

import numpy as np
import pytest
import torch

import attn_bounds as AB
from bounds_util import OUT, assert_within
from gpu_util import CODE, F32, check, ptr, record_parity, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
IOS = [torch.float16, torch.bfloat16]
IO_ID = {torch.float16: "f16", torch.bfloat16: "bf16"}
FLASH_OUT = {torch.float16: ["f32", "tf32", "f16"], torch.bfloat16: ["f32", "bf16"]}
MAP_OUT = {torch.float16: "f16", torch.bfloat16: "bf16"}
D_ALL = [8, 24, 40, 64, 72, 80, 88, 112, 128]
# (B, S, H, d, causal)
TOWERS = [(2, 197, 12, 64, False), (1, 257, 16, 80, False), (1, 577, 16, 64, False), (1, 729, 16, 72, False), (2, 77, 8, 64, True),
          (2, 64, 12, 64, False)]
EDGES = [(2, S, 3, d, causal) for S, d in zip([1, 2, 63, 64, 65, 127, 129], [8, 24, 40, 88, 112, 128, 72]) for causal in (False, True)]
LONG = [(1, 4096, 1, 64, False)]
LENS = [1, 63, 64, 65, 200]
PACKED = [(88, False), (40, True)]  # (d, causal)


def _cases(family, io):
    if family == "big" and io != torch.bfloat16:
        pytest.skip("q and k beyond fp16's range: bf16 only")
    return TOWERS + EDGES + LONG


def _qkv(family, B, S, H, d, io, seed):
    return AB.make_qkv(family, B, S, H, d, io, seed).to(DEV)


def _offsets(lens):
    return torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)


def _samples(qkv, lens, H, d):
    """(q, k, v) [H, n, d] of each packed sample."""
    r0 = 0
    for n in lens:
        yield AB.split_qkv(qkv[r0:r0 + n], 1, n, H, d)
        r0 += n


# ---------------------------------------------------------------------------------------------------------------- c_qk
def _two_key_rows(d, H, B, io, seed):
    """Per (sample, head): two keys whose products with q cancel between the two halves of the head dims, so |s| << a while the
    accumulator's partial sums reach a / 2 halfway.  Dim i and i + d/2 of q are both x_i; of key j, y_ji and round(-y_ji + 0.05 z_ji)
    with sign(y) = sign(x) (x, y, z ~ N(0, 1) x 8, 8, 1 rounded to io, full mantissas): s_j is a few units, a_j thousands."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, H, d // 2, generator=g) * 8).to(io).float()
    q = torch.cat([x, x], -1)
    ks = []
    for _ in range(2):
        y = ((torch.randn(B, H, d // 2, generator=g) * 8).abs() * x.sign()).to(io).float()
        y2 = (-y + 0.05 * torch.randn(B, H, d // 2, generator=g)).to(io).float()
        ks.append(torch.cat([y, y2], -1))
    q = q[:, None].expand(B, 2, H, d)
    k = torch.stack(ks, 1)
    v = torch.zeros_like(k)
    return torch.stack([q, k, v], 2).reshape(B * 2, 3 * H * d).to(io)


@pytest.mark.parametrize("io", IOS, ids=IO_ID.get)
def test_score_accumulation_constant(lib, io):
    """Rows of two live keys, jimm_k_attn_probs with fp32 output: log2(P^_1 / P^_0) = fl(s^_1 c) - fl(s^_0 c) up to exp2f's and the
    products' roundings (a few u, 1e-6 in log2 units), so (s^_1 - s^_0) - (s_1 - s_0) is read to about u |s c| / c, far below
    c_qk (a_0 + a_1).  Worst |that| / (a_0 + a_1) over d = 8 .. 128 (read-out noise included, so an overestimate): recorded per d and
    asserted below attn_bounds.C_QK."""
    B, H = 8, 32
    worst = 0.0
    for d in D_ALL:
        qkv = _two_key_rows(d, H, B, io, seed=d).to(DEV)
        out = torch.empty(B * H * 4, device=DEV)
        check(lib, lib.jimm_k_attn_probs(ptr(qkv), CODE[io], ptr(out), F32, None, B, 2, H, d, 0, stream()))
        torch.cuda.synchronize()
        p = out.double().view(B, H, 2, 2)
        q, k, _ = AB.split_qkv(qkv, B, 2, H, d)
        s = (q @ k.transpose(-1, -2)).view(B, H, 2, 2)
        a = (q.abs() @ k.abs().transpose(-1, -2)).view(B, H, 2, 2)
        assert bool((p > 2.0 ** -126).all()), "both keys must stay normal for the read-out"
        got = torch.log2(p[..., 1] / p[..., 0]) / AB._scale_log2(d)
        per = float(((got - (s[..., 1] - s[..., 0])).abs() / (a[..., 0] + a[..., 1])).max())
        record_parity(f"score_tile d={d}", "score error / (a_0 + a_1)", IO_ID[io], "fp64", AB.C_QK[io], per)
        worst = max(worst, per)
    print(f"c_qk measured {IO_ID[io]}: {worst:.3e}")
    assert worst < AB.C_QK[io], (IO_ID[io], worst)


# ---------------------------------------------------------------------------------------------------------------- jimm_k_attn_probs
def _probs(lib, qkv, B, S, H, d, causal, lens=None):
    n = H * (sum(x * x for x in lens) if lens else B * S * S)
    out = torch.full((n,), float("nan"), device=DEV)
    seq = _offsets(lens) if lens else None
    check(lib, lib.jimm_k_attn_probs(ptr(qkv), CODE[qkv.dtype], ptr(out), F32, ptr(seq), len(lens) if lens else B, max(lens) if lens else S,
                                     H, d, int(causal), stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("family", AB.FAMILIES)
@pytest.mark.parametrize("io", IOS, ids=IO_ID.get)
def test_probs_bound(lib, io, family):
    """jimm_k_attn_probs, fp32 output: every probability within probs_ref_bound, dense (shape (sample, head, row, key)) and packed."""
    c_qk = AB.C_QK[io]
    for i, (B, S, H, d, causal) in enumerate(_cases(family, io)):
        qkv = _qkv(family, B, S, H, d, io, seed=i)
        out = _probs(lib, qkv, B, S, H, d, causal)
        q, k, _ = AB.split_qkv(qkv, B, S, H, d)
        P, bound = AB.probs_ref_bound(q, k, causal, c_qk)
        shape = (B, H, S, S)
        assert_within(f"attn_probs {family} B={B} S={S} H={H} d={d} causal={causal}", "P", out.view(shape), P.view(shape), bound.view(shape),
                      IO_ID[io])
    for d, causal in PACKED:
        H = 3
        qkv = _qkv(family, 1, sum(LENS), H, d, io, seed=d)
        out = _probs(lib, qkv, len(LENS), max(LENS), H, d, causal, LENS)
        e0 = 0
        for b, (q, k, _) in enumerate(_samples(qkv, LENS, H, d)):
            n = q.shape[1]
            P, bound = AB.probs_ref_bound(q, k, causal, c_qk)
            assert_within(f"attn_probs packed {family} lens={LENS} H={H} d={d} causal={causal}", f"P of sample {b}",
                          out[e0:e0 + H * n * n].view(H, n, n), P, bound, IO_ID[io])
            e0 += H * n * n


# ---------------------------------------------------------------------------------------------------------------- flash attention
def _flash(lib, qkv, out_t, B, S, H, d, causal, reverse=0, lens=None):
    dt, code, _, _ = OUT[out_t]
    rows = sum(lens) if lens else B * S
    out = torch.full((rows, H * d), float("nan"), dtype=dt, device=DEV)
    if lens:
        check(lib, lib.jimm_k_attention_packed_ex(ptr(qkv), CODE[qkv.dtype], ptr(out), code, ptr(_offsets(lens)), len(lens), max(lens), H, d,
                                                  int(causal), reverse, stream()))
    else:
        check(lib, lib.jimm_k_attention_hd(ptr(qkv), CODE[qkv.dtype], ptr(out), code, B, S, H, d, int(causal), reverse, stream()))
    torch.cuda.synchronize()
    return out


def _heads(o, n, H, d):
    """[n, H d] -> [H, n, d]."""
    return o.reshape(n, H, d).permute(1, 0, 2)


@pytest.mark.parametrize("family", AB.FAMILIES)
@pytest.mark.parametrize("io", IOS, ids=IO_ID.get)
def test_flash_bound(lib, io, family):
    """jimm_k_attention_hd to every output type the io type takes: every output within flash_ref_bound (shape (sample, head, row,
    column)); reverse = 1 gives reverse = 0's bits.  jimm_k_attention_packed_ex the same per packed sample."""
    c_qk = AB.C_QK[io]
    for i, (B, S, H, d, causal) in enumerate(_cases(family, io)):
        qkv = _qkv(family, B, S, H, d, io, seed=i)
        q, k, v = AB.split_qkv(qkv, B, S, H, d)
        for out_t in FLASH_OUT[io]:
            o, bound = AB.flash_ref_bound(q, k, v, causal, c_qk, io, out_t)
            out = _flash(lib, qkv, out_t, B, S, H, d, causal)
            got = out.view(B, S, H, d).permute(0, 2, 1, 3)
            shape = (B, H, S, d)
            assert_within(f"attention {family} B={B} S={S} H={H} d={d} causal={causal}", f"out {out_t}", got, o.view(shape), bound.view(shape),
                          IO_ID[io])
            assert torch.equal(_flash(lib, qkv, out_t, B, S, H, d, causal, reverse=1), out), "reverse = 1 changed the bits"
    for d, causal in PACKED:
        H = 3
        qkv = _qkv(family, 1, sum(LENS), H, d, io, seed=d)
        for out_t in FLASH_OUT[io]:
            out = _flash(lib, qkv, out_t, 0, 0, H, d, causal, lens=LENS)
            r0 = 0
            for b, (q, k, v) in enumerate(_samples(qkv, LENS, H, d)):
                n = q.shape[1]
                o, bound = AB.flash_ref_bound(q, k, v, causal, c_qk, io, out_t)
                assert_within(f"attention packed {family} lens={LENS} H={H} d={d} causal={causal}", f"out {out_t} of sample {b}",
                              _heads(out[r0:r0 + n], n, H, d), o, bound, IO_ID[io])
                r0 += n


# ---------------------------------------------------------------------------------------------------------------- MAP head
MAP_CASES = [(2, 197, 12, 64), (1, 257, 16, 80), (1, 577, 16, 64), (1, 729, 16, 72)] + \
            [(2, S, 3, d) for S, d in zip([1, 2, 63, 64, 65, 127, 129], [8, 24, 40, 88, 112, 128, 72])] + [(1, 8192, 2, 64)]


def _map_inputs(family, B, S, H, d, io, seed):
    """The probe: q of the family's first row in fp32, moved off the io grid (x (1 + 2^-13)); kv: the family's k and v."""
    qkv = _qkv(family, B, S, H, d, io, seed)
    q = (qkv[0, : H * d].float() * (1 + 2.0 ** -13)).contiguous()
    return q, qkv[:, H * d:].contiguous()


def _map(lib, q, kv, io, out_t, B, S, H, d, lens=None, probs=False):
    dt, code, _, _ = OUT[out_t]
    rows = sum(lens) if lens else B * S
    nb = len(lens) if lens else B
    out = torch.full((nb, H * d), float("nan"), dtype=dt, device=DEV)
    pr = torch.full((H * rows,), float("nan"), device=DEV) if probs else None
    seq = _offsets(lens) if lens else None
    if probs:
        check(lib, lib.jimm_k_map_attention_probs(ptr(q), ptr(kv), CODE[io], ptr(out), code, ptr(seq), nb, max(lens) if lens else S, H, d,
                                                  ptr(pr), F32, stream()))
    elif lens:
        check(lib, lib.jimm_k_map_attention_packed(ptr(q), ptr(kv), CODE[io], ptr(out), code, ptr(seq), nb, max(lens), H, d, stream()))
    else:
        check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kv), CODE[io], ptr(out), code, B, S, H, d, stream()))
    torch.cuda.synchronize()
    return out, pr


@pytest.mark.parametrize("family", AB.FAMILIES)
@pytest.mark.parametrize("io", IOS, ids=IO_ID.get)
def test_map_bound(lib, io, family):
    """jimm_k_map_attention_hd (fp32 and the io type out) and jimm_k_map_attention_probs: pooled outputs within map_ref_bound (shape
    (sample, head, column)), probe weights (sample, head, key); jimm_k_map_attention_packed per packed sample.  The weights call's
    pooled output has the plain call's bits."""
    if family == "big" and io != torch.bfloat16:
        pytest.skip("q and k beyond fp16's range: bf16 only")
    for i, (B, S, H, d) in enumerate(MAP_CASES):
        q, kv = _map_inputs(family, B, S, H, d, io, seed=i)
        k, v = (t.double().reshape(B, S, H, d).permute(0, 2, 1, 3).reshape(B * H, S, d) for t in kv.split(H * d, 1))
        case = f"map {family} B={B} S={S} H={H} d={d}"
        for out_t in ("f32", MAP_OUT[io]):
            P, pb, o, ob = AB.map_ref_bound(q.view(H, d), k, v, io, out_t)
            out, _ = _map(lib, q, kv, io, out_t, B, S, H, d)
            assert_within(case, f"pooled {out_t}", out.view(B, H, d), o.view(B, H, d), ob.view(B, H, d), IO_ID[io])
        out2, pr = _map(lib, q, kv, io, "f32", B, S, H, d, probs=True)
        P, pb, o, ob = AB.map_ref_bound(q.view(H, d), k, v, io, "f32")
        assert_within(case, "probe weights", pr.view(B, H, S), P.view(B, H, S), pb.view(B, H, S), IO_ID[io])
        assert torch.equal(out2, _map(lib, q, kv, io, "f32", B, S, H, d)[0])
    H, d = 3, 72
    q, kv = _map_inputs(family, 1, sum(LENS), H, d, io, seed=99)
    out, _ = _map(lib, q, kv, io, "f32", 0, 0, H, d, lens=LENS)
    r0 = 0
    for b, n in enumerate(LENS):
        k, v = (t.double().reshape(n, H, d).permute(1, 0, 2) for t in kv[r0:r0 + n].split(H * d, 1))
        _, _, o, ob = AB.map_ref_bound(q.view(H, d), k, v, io, "f32")
        assert_within(f"map packed {family} lens={LENS} H={H} d={d}", f"pooled f32 of sample {b}", out[b].view(H, d), o, ob, IO_ID[io])
        r0 += n
