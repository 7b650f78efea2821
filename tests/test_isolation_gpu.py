"""GPU: one non-finite or overflowing input changes no other result.  A poisoned sample (NaN, +inf, -inf, or a finite value that
overflows the 16-bit operand) must leave every other sample of the same call bit for bit as the clean call left it, in the batched
and the packed kernels, in the models, and in every later call on the same handle.  The poisoned sample's own non-finite pattern is
compared with an fp64 reference, which also shows that the poison went through the kernel.  Bytes no kernel may read (plan rows past
the run, columns between K and lda, rows past the packed stream) are filled with NaN and must not change a bit."""

import math

import numpy as np
import pytest
import torch

import fp8_oracle as F
import jimm_oracle as O
import preprocess_oracle as P
from gpu_util import BF16, CODE, F16, F32, TORCH, check, ptr, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
TF32 = 3
NAN, INF = float("nan"), float("inf")
POISONS = ["nan", "inf", "-inf", "big"]


def poison_value(kind, dtype=torch.float32):
    """'big' is finite in fp32 but overflows the 16-bit operand: 7e4 for fp16; 1e30 for bf16 and fp32, whose squares and products
    overflow the fp32 arithmetic downstream.  Written into an fp16 operand, 7e4 rounds to inf and repeats the 'inf' case; it is a finite
    overflow where the input is fp32 (the models' pixels, the LayerNorm's residual stream)."""
    return {"nan": NAN, "inf": INF, "-inf": -INF}.get(kind, 7e4 if dtype == torch.float16 else 1e30)


def _randn(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


def _bad(t):
    return ~torch.isfinite(t.float() if t.dtype != torch.float64 else t)


def _same(a, b):
    """Bitwise equality that treats NaN like any other bit pattern."""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _offsets(lens):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return off, torch.from_numpy(off).to(DEV)


def _out_dtype(code):
    return torch.float32 if code == TF32 else TORCH[code]


def gemm_ex(lib, A, Bw, out, *, M=None, plan_M=0, bias=None, act=0, residual=None, out_code=None, mode=2, tok=(0, 0, 0), ln=None):
    """jimm_k_gemm_ex; ln = (scale, bias, eps, ln_out, ln_code, counters)."""
    N, K = Bw.shape
    M = A.shape[0] if M is None else M
    ls, lb, eps, lo, lcode, cnt = ln if ln is not None else (None, None, 0.0, None, 0, None)
    return lib.jimm_k_gemm_ex(0, CODE[A.dtype], ptr(A), A.stride(0), ptr(Bw), Bw.stride(0), M, N, K, ptr(bias), act, None, ptr(residual),
                              0 if residual is None else residual.stride(0), ptr(out), CODE[out.dtype] if out_code is None else out_code,
                              out.stride(0), 0, 0, 0, mode, plan_M, 0, *tok, ptr(ls), ptr(lb), eps, ptr(lo), lcode,
                              0 if lo is None else lo.stride(0), ptr(cnt), stream())


# ====================================================================================================================== attention
def _attn_ref(qkv, S, H, d, causal):
    """One sample in fp64, strictly causal: 0 x = 0 for every key a row does not attend to, so a non-finite value reaches exactly
    the (row, column) outputs whose softmax weight on it is not zero."""
    q, k, v = qkv.double().reshape(S, 3, H, d).permute(1, 2, 0, 3)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(d)
    if causal:
        s = s.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=qkv.device)), -INF)
    p = torch.softmax(s, -1)
    vbad = ~torch.isfinite(v)
    out = p @ torch.where(vbad, torch.zeros_like(v), v)
    out = out.masked_fill(((p != 0).double() @ vbad.double()) > 0, NAN)
    return out.permute(1, 0, 2).reshape(S, H * d)


def _check_own(out, qkv_s, S, H, d, causal, part, r, c):
    """The poisoned sample's non-finite pattern against _attn_ref.  The causal kernel multiplies the diagonal 64-key tile's P by its
    whole V tile in one MMA, so a non-finite V value at key r also reaches, as 0 x inf / 0 x NaN, the rows of its 64-row block before
    r, in its own column only (the fp64 reference's matmul would spread it to every row).  Nothing else may differ."""
    ref_bad = _bad(_attn_ref(qkv_s, S, H, d, causal))
    bad = _bad(out)
    assert part == 1 or bool(ref_bad.any()), "a non-finite q or v value reaches no output of the reference"
    assert bool((bad >= ref_bad).all()), "a non-finite the reference has is missing: the poison did not reach the output"
    extra = bad & ~ref_bad
    if causal and part == 2:
        allowed = torch.zeros_like(extra)
        allowed[(r // 64) * 64:r, c - 2 * H * d] = True
        extra &= ~allowed
    assert not bool(extra.any()), f"non-finite outputs the reference does not have: rows {extra.any(1).nonzero().flatten().tolist()[:8]}"


def _attention(lib, qkv, io, ot, B, S, H, d, causal):
    out = torch.full((B * S, H * d), NAN, dtype=_out_dtype(ot), device=DEV)
    check(lib, lib.jimm_k_attention_hd(ptr(qkv), io, ptr(out), ot, B, S, H, d, causal, 0, stream()))
    return out


@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("io", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("d", [64, 72, 128])
@pytest.mark.parametrize("S", [1, 63, 65, 197, 577])
def test_attention_poisoned_sample(lib, S, d, io, causal):
    """Poison one element of q (middle row), k or v (first row: what a clamp past the previous sample's end would read; last row: the
    row the partial key tile is clamped to) of the first, middle or last sample: the other samples keep their bits in both output
    types, the poisoned one has the reference's non-finite pattern."""
    B, H = 3, 2
    D = H * d
    dt = TORCH[io]
    qkv0 = (_randn(B * S, 3 * D, seed=S * 7 + d + io) * 1.5).to(dt)
    ots = (io, F32)
    clean = {ot: _attention(lib, qkv0, io, ot, B, S, H, d, causal) for ot in ots}
    for b in (0, B // 2, B - 1):
        rows = slice(b * S, (b + 1) * S)
        others = torch.ones(B * S, dtype=torch.bool, device=DEV)
        others[rows] = False
        for part, r in [(0, S // 2)] + [(p, r) for p in (1, 2) for r in sorted({0, S - 1})]:
            c = part * D + hd_col(H, d)
            for kind in POISONS:
                qkv = qkv0.clone()
                qkv[b * S + r, c] = poison_value(kind, dt)
                for ot in ots:
                    out = _attention(lib, qkv, io, ot, B, S, H, d, causal)
                    assert _same(out[others], clean[ot][others]), (b, part, kind, ot, "a clean sample changed")
                    own = out[rows]
                    finite = bool(torch.isfinite(qkv[b * S + r, c].float()))
                    if part != 1:  # a key whose score ends at -inf or whose weight rounds to 0 may change nothing
                        assert not _same(own, clean[ot][rows]), (b, part, kind, "the poison changed nothing")
                    if not finite and ot == F32:
                        _check_own(own, qkv[rows], S, H, d, causal, part, r, c)


def hd_col(H, d):
    return (H - 1) * d + d - 1  # the last column of the last head


LENS_P = [40, 64, 100, 64, 7, 130, 65, 64]  # neighbours shorter than, as long as and longer than one 64-row tile
PAD = 5


@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("io", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("d", [64, 72])
def test_attention_packed_poisoned_neighbours(lib, d, io, causal):
    """Packed samples: poison the first and the last row of sample j in q, k or v (the first row of the sample after j is what a clamp
    past j's end would read); every other sample keeps its bits, j has the reference's pattern.  The rows past seq_off[B] hold NaN
    instead of zeros without changing a bit, and stay unwritten."""
    H = 2
    D = H * d
    dt = TORCH[io]
    off, off_d = _offsets(LENS_P)
    T = int(off[-1])
    nB, mS = len(LENS_P), max(LENS_P)
    qkv0 = (_randn(T + PAD, 3 * D, seed=d + io + causal) * 1.5).to(dt)
    qkv0[T:] = 0

    def run(qkv):
        out = torch.full((T + PAD, D), -3.0, dtype=torch.float32, device=DEV)
        check(lib, lib.jimm_k_attention_packed_ex(ptr(qkv), io, ptr(out), F32, ptr(off_d), nB, mS, H, d, causal, 0, stream()))
        return out

    clean = run(qkv0)
    tail = qkv0.clone()
    tail[T:] = NAN
    got = run(tail)
    assert _same(got, clean) and bool((got[T:] == -3.0).all()), "rows past seq_off[B] were read or written"
    for j, S in enumerate(LENS_P):
        rows = slice(int(off[j]), int(off[j + 1]))
        others = torch.ones(T + PAD, dtype=torch.bool, device=DEV)
        others[rows] = False
        for part in range(3):
            c = part * D + hd_col(H, d)
            for r in sorted({0, S - 1}):
                for kind in ("nan", "inf"):
                    qkv = qkv0.clone()
                    qkv[int(off[j]) + r, c] = poison_value(kind, dt)
                    out = run(qkv)
                    assert _same(out[others], clean[others]), (j, part, r, kind, "a neighbouring sample changed")
                    _check_own(out[rows], qkv[rows], S, H, d, causal, part, r, c)


def _map_ref(q, kv, S, H, d):
    k, v = kv.double().reshape(S, 2, H, d).permute(1, 2, 0, 3)
    p = torch.softmax((q.double().reshape(H, 1, d) / math.sqrt(d)) @ k.transpose(-1, -2), -1)
    return (p @ v).reshape(H * d)


@pytest.mark.parametrize("packed", [False, True], ids=["batched", "packed"])
@pytest.mark.parametrize("io", [F16, BF16], ids=["f16", "bf16"])
def test_map_attention_poisoned_sample(lib, io, packed):
    """MAP pooling: poison the first or the last key / value row of one sample; the other samples' pooled rows keep their bits."""
    H, d = 2, 64
    D = H * d
    dt = TORCH[io]
    lens = [40, 64, 100, 7, 65] if packed else [65] * 5
    off, off_d = _offsets(lens)
    T = int(off[-1])
    nB = len(lens)
    q = _randn(D, seed=5)
    kv0 = _randn(T + PAD, 2 * D, seed=6 + io).to(dt)

    def run(kv):
        out = torch.full((nB, D), -3.0, device=DEV)
        if packed:
            check(lib, lib.jimm_k_map_attention_packed(ptr(q), ptr(kv), io, ptr(out), F32, ptr(off_d), nB, max(lens), H, d, stream()))
        else:
            check(lib, lib.jimm_k_map_attention_hd(ptr(q), ptr(kv), io, ptr(out), F32, nB, lens[0], H, d, stream()))
        return out

    clean = run(kv0)
    tail = kv0.clone()
    tail[T:] = NAN
    assert _same(run(tail), clean), "rows past the last sample were read"
    for j, S in enumerate(lens):
        o = int(off[j])
        for part in range(2):
            c = part * D + hd_col(H, d)
            for r in (0, S - 1):
                for kind in POISONS:
                    kv = kv0.clone()
                    kv[o + r, c] = poison_value(kind, dt)
                    out = run(kv)
                    keep = torch.arange(nB, device=DEV) != j
                    assert _same(out[keep], clean[keep]), (j, part, r, kind, "another sample's pooled row changed")
                    assert not _same(out[j], clean[j]), (j, part, r, kind, "the poison changed nothing")
                    if not bool(torch.isfinite(kv[o + r, c].float())):
                        assert _same(_bad(out[j]), _bad(_map_ref(q, kv[o:o + S], S, H, d))), (j, part, r, kind)


# ====================================================================================================================== LayerNorm
def _ln_ref(x, scale, bias, eps):
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = (xd * xd).mean(-1, keepdim=True) - mean * mean
    return (xd - mean) * torch.rsqrt(var + eps) * scale.double() + bias.double()


@pytest.mark.parametrize("gather", ["rows", "offset", "index"])
@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("ot", [F32, F16, BF16, TF32], ids=["f32", "f16", "bf16", "tf32"])
def test_layernorm_poisoned_row(lib, ot, reverse, gather):
    """One poisoned element in a source row (alone, and at the end of a 32-row group): the other output rows keep their bits; the
    poisoned row is non-finite wherever the fp64 reference is.  'offset' and 'index' normalise one gathered row per sample."""
    D, G = 768, 5
    rows = 70
    x0 = _randn(rows * G, D, seed=ot + 10 * reverse) * 2 + 0.5
    scale, bias = _randn(D, seed=1), _randn(D, seed=2)
    idx = torch.randint(0, G, (rows,), generator=torch.Generator().manual_seed(3), dtype=torch.int32).to(DEV)
    group, row_off, index = {"rows": (1, 0, None), "offset": (G, G - 1, None), "index": (G, 0, idx)}[gather]
    n = rows if gather != "rows" else rows * G
    src = torch.arange(n, device=DEV) * group + (idx[:n].long() if index is not None else row_off)

    def run(x):
        out = torch.full((n, D), -3.0, dtype=_out_dtype(ot), device=DEV)
        check(lib, lib.jimm_k_layernorm_ex(ptr(x), D, group, row_off, ptr(index), ptr(scale), ptr(bias), 1e-6, ptr(out), ot, D, n, D,
                                           reverse, stream()))
        return out

    clean = run(x0)
    for r in (0, 31, n - 1):
        for kind in POISONS:
            x = x0.clone()
            x[src[r], 7] = poison_value(kind)
            out = run(x)
            keep = torch.arange(n, device=DEV) != r
            assert _same(out[keep], clean[keep]), (r, kind, "another row changed")
            if kind == "big":
                assert not _same(out[r], clean[r])
            else:
                assert bool(_bad(out[r]).all()) and bool(_bad(_ln_ref(x[src[r]], scale, bias, 1e-6)).all()), (r, kind)


def test_layernorm_e4m3_poisoned_rows(lib):
    """FP8 LayerNorm: a row of +inf, a row of NaN, a row with one +inf and a row with one -inf.  The other rows keep their bytes and
    row scales; each poisoned row dequantises to non-finite values wherever the fp64 LayerNorm is non-finite, which is everywhere."""
    rows, D = 100, 768
    x0 = _randn(rows, D, seed=20) * 2 + 0.5
    scale, bias = _randn(D, seed=21), _randn(D, seed=22)

    def run(x):
        q = torch.full((rows, D), 0x55, dtype=torch.uint8, device=DEV)
        s = torch.full((rows,), -1.0, device=DEV)
        check(lib, lib.jimm_k_layernorm_e4m3(ptr(x), D, ptr(scale), ptr(bias), 1e-6, ptr(q), D, ptr(s), rows, D, 0, stream()))
        return q, s

    q0, s0 = run(x0)
    x = x0.clone()
    poisoned = [3, 31, 32, 99]
    x[3] = INF
    x[31] = NAN
    x[32, 100] = INF
    x[99, 0] = -INF
    q, s = run(x)
    keep = torch.ones(rows, dtype=torch.bool, device=DEV)
    keep[poisoned] = False
    assert _same(q[keep], q0[keep]) and _same(s[keep], s0[keep]), "a clean row's bytes or scale changed"
    deq = F.dequant(q.view(torch.float8_e4m3fn).cpu(), s.cpu())
    for r in poisoned:
        assert bool(_bad(_ln_ref(x[r], scale, bias, 1e-6)).all())
        assert bool(_bad(deq[r]).all()), (r, f"row dequantises to finite values (scale {float(s[r])})")
    # the oracle quantiser of the same fp32 LayerNorm rows: an infinite row absolute maximum gives an infinite scale there too
    y = torch.empty(rows, D, device=DEV)
    check(lib, lib.jimm_k_layernorm_ex(ptr(x), D, 1, 0, None, ptr(scale), ptr(bias), 1e-6, ptr(y), F32, D, rows, D, 0, stream()))
    _, s_ref = F.quantize_rows(y.cpu())
    assert torch.equal(s.cpu(), s_ref), "row scales differ from the oracle quantiser"


# ====================================================================================================================== GEMM
KINDS = ["store_f16", "generic", "reduce_add", "fused_ln", "token_scatter"]


def _gemm_kind(lib, kind, A, W, x0, bias, M, plan_M=0, ln_w=None):
    """One GEMM of epilogue `kind`; returns the tensors it writes."""
    N = W.shape[0]
    if kind in ("store_f16", "generic"):
        out = torch.full((A.shape[0], N + 24), -3.0, dtype=torch.float16 if kind == "store_f16" else torch.float32, device=DEV)
        check(lib, gemm_ex(lib, A, W, out[:, :N], M=M, plan_M=plan_M, bias=bias, act=1, mode=2 if kind == "store_f16" else 0))
        return (out,)
    x = x0.clone()
    if kind == "reduce_add":
        check(lib, gemm_ex(lib, A, W, x, M=M, plan_M=plan_M, bias=bias, residual=x))
        return (x,)
    if kind == "token_scatter":  # samples of n = 40 patches padded to 48 rows, written to tokens 1 .. 40 of 41
        check(lib, gemm_ex(lib, A, W, x, M=M, plan_M=plan_M, bias=bias, residual=x, tok=(48, 1, 41)))
        return (x,)
    h = torch.full((A.shape[0], N), -3.0, dtype=A.dtype, device=DEV)
    cnt = torch.zeros(A.shape[0] // 32 + 2, dtype=torch.int32, device=DEV)
    check(lib, gemm_ex(lib, A, W, x, M=M, plan_M=plan_M, bias=bias, residual=x, ln=(ln_w[0], ln_w[1], 1e-6, h, CODE[A.dtype], cnt)))
    return x, h


def _out_rows(kind, r):
    """Output rows of A row r (the token-scatter epilogue moves row p of sample b to token p + 1)."""
    if kind == "token_scatter":
        b, p = divmod(r, 48)
        return [b * 41 + p + 1] if p < 40 else []
    return [r]


@pytest.mark.parametrize("op", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "tf32"])
@pytest.mark.parametrize("kind", KINDS)
def test_gemm_poisoned_row(lib, kind, op):
    """One poisoned A row (first, inside a 128-row tile and a 32-row LayerNorm group, last) changes that output row only; a poisoned
    weight row changes that output column only.  Plans for more rows than run with NaN past M, a strided A with NaN between K and
    lda and NaN pad rows of the patch operand give the clean bits."""
    nS, extra = 7, 96  # the plan holds two samples of the token scatter more than are run
    M = nS * 48 if kind == "token_scatter" else 300
    N, K, lda = 768, 264, 280
    plan_M = M + extra
    Abuf = torch.full((plan_M, lda), NAN, dtype=op, device=DEV)  # columns K .. lda of every row: NaN
    Abuf[:, :K] = _randn(plan_M, K, seed=30).to(op)
    Abuf[M:, :K] = 0
    if kind == "token_scatter":
        Abuf[:M].view(nS, 48, lda)[:, 40:] = NAN  # pad rows of each sample
    A0 = Abuf[:, :K]
    W0 = (_randn(N, K, seed=31) / math.sqrt(K)).to(op)
    bias = _randn(N, seed=32)
    x0 = _randn((nS * 41 if kind == "token_scatter" else M) + extra, N, seed=33)
    ln_w = (_randn(N, seed=34), _randn(N, seed=35))
    clean = _gemm_kind(lib, kind, A0, W0, x0, bias, M, plan_M=plan_M, ln_w=ln_w)
    stale = Abuf.clone()
    stale[M:] = NAN  # plan rows past M
    # the TMA epilogues may also store rows M .. m16 - 1, which no caller reads; the generic epilogue stores rows < M only
    m16 = M if kind == "generic" else (M + 15) // 16 * 16
    for what, A in (("rows past M", stale[:, :K]), ("columns between K and lda", A0.contiguous())):
        for a, b in zip(_gemm_kind(lib, kind, A, W0, x0, bias, M, plan_M=plan_M, ln_w=ln_w), clean):
            assert _same(a[:M], b[:M]) and _same(a[m16:], b[m16:]), f"{what} changed the result"
    # first row, inside a 128-row tile and a 32-row LayerNorm group, and both 8-row halves of the last 16-row group
    rs = [0, 37, 47, 48, M - 1] if kind == "token_scatter" else [0, 37, 63, 130, M - 9, M - 1]
    for r in rs:
        for kind_p in POISONS:
            A = Abuf.clone()
            A[r, 11] = poison_value(kind_p, op)
            got = _gemm_kind(lib, kind, A[:, :K], W0, x0, bias, M, plan_M=plan_M, ln_w=ln_w)
            orows = _out_rows(kind, r)
            for t, c in zip(got, clean):
                keep = torch.ones(t.shape[0], dtype=torch.bool, device=DEV)
                keep[orows] = False
                assert _same(t[keep], c[keep]), (r, kind_p, "another output row changed")
                for o in orows:
                    if bool(torch.isfinite(A[r, 11].float())):
                        assert not _same(t[o], c[o]), (r, kind_p)
                    else:
                        assert bool(_bad(t[o][:N]).all()), (r, kind_p, "the poisoned row is not non-finite")
            if kind in ("store_f16", "generic"):
                assert bool((got[0][:, N:] == -3.0).all()), "columns between N and ldo written"
    for n in (0, 130, N - 1):  # a poisoned weight row: that output column only
        W = W0.clone()
        W[n, 5] = NAN
        got = _gemm_kind(lib, kind, A0, W, x0, bias, M, plan_M=plan_M, ln_w=ln_w)
        t, c = got[0], clean[0]
        keep = torch.ones(t.shape[1], dtype=torch.bool, device=DEV)
        keep[n] = False
        written = torch.tensor(sorted({o for r in range(M) for o in _out_rows(kind, r)}), device=DEV)
        if kind == "fused_ln":  # the LayerNorm of a row with a NaN is NaN: the residual stream is the one to check
            assert _same(t[:, keep], c[:, keep]) and bool(_bad(t[written, n]).all())
        else:
            assert _same(t[:, keep], c[:, keep]), (n, "another output column changed")
            assert bool(_bad(t[written, n]).all()), (n, "the poisoned column is not non-finite")


def test_gemm_e4m3_poisoned_row(lib):
    """FP8 GEMM: A rows quantised per row; one row with NaN, one with +inf.  The other output rows keep their bits, the poisoned ones
    are non-finite."""
    M, N, K = 300, 768, 256
    a = _randn(M, K, seed=40)
    w = _randn(N, K, seed=41) / 16
    bias = _randn(N, seed=42)

    def quant(src):
        q = torch.empty(src.shape, dtype=torch.uint8, device=DEV)
        s = torch.empty(src.shape[0], device=DEV)
        check(lib, lib.jimm_k_quantize_e4m3(ptr(src), K, src.shape[0], K, ptr(q), K, ptr(s), stream()))
        return q, s

    wq, ws = quant(w)

    def run(src):
        aq, as_ = quant(src)
        out = torch.full((M, N), -3.0, dtype=torch.float16, device=DEV)
        check(lib, lib.jimm_k_gemm_e4m3(0, ptr(aq), K, ptr(wq), K, M, N, K, ptr(as_), ptr(ws), ptr(bias), 0, ptr(out), F16, N, 2, 0, 0,
                                        stream()))
        return out

    clean = run(a)
    x = a.clone()
    x[37, 3] = NAN
    x[130, 200] = INF
    out = run(x)
    keep = torch.ones(M, dtype=torch.bool, device=DEV)
    keep[[37, 130]] = False
    assert _same(out[keep], clean[keep])
    assert bool(_bad(out[37]).all()) and bool(_bad(out[130]).all())


# ====================================================================================================================== front end
@pytest.mark.parametrize("in_t", [torch.float32, torch.float16], ids=["f32", "f16"])
@pytest.mark.parametrize("C", [1, 3, 4])
def test_patchify_poisoned_image(lib, C, in_t):
    """The padded patch operand: a poisoned pixel changes that image's patch element only; pad columns stay 0, pad rows unwritten."""
    Bn, P, H, W = 3, 14, 100, 112
    gh, gw = H // P, W // P
    n = gh * gw
    n_pad = (n + 31) // 32 * 32
    ldk = (P * P * C + 7) // 8 * 8
    x0 = _randn(Bn, H, W, C, seed=C).to(in_t)

    PPC = P * P * C  # C = 3: 588 values padded to 592 columns; C = 4: 784, no pad

    def run(x):
        out = torch.full((Bn * n_pad, ldk), NAN, dtype=torch.float16, device=DEV)
        check(lib, lib.jimm_k_patchify_ex(ptr(x), CODE[in_t], Bn, H, W, C, P, ptr(out), F16, n_pad, ldk, stream()))
        o = out.view(Bn, n_pad, ldk)
        assert bool((o[:, :n, PPC:] == 0).all()), "pad columns not zero"  # the patch GEMM multiplies them by the weight's zero columns
        assert bool(torch.isnan(o[:, n:]).all()), "pad rows written"
        return out

    clean = run(x0)
    for b in range(Bn):
        for kind in POISONS:
            x = x0.clone()
            x[b, 20, 33, C - 1] = poison_value(kind)
            out = run(x)
            diff = ~(out.view(torch.int16) == clean.view(torch.int16))
            row, col = b * n_pad + (20 // P) * gw + 33 // P, (20 % P) * P * C + (33 % P) * C + C - 1
            assert diff.sum() == 1 and bool(diff[row, col]), (b, kind)
            assert bool(_bad(out[row, col])), (b, kind)


def test_tokens_init_interp_ignores_stale_output(lib):
    """The position-initialised stream is written, not added to: NaN left in x by an earlier call changes nothing."""
    g, D, B, gh, gw = 4, 128, 3, 5, 7
    cls, pos = _randn(D, seed=50), _randn(1 + g * g, D, seed=51)
    out = []
    for fill in (0.0, NAN):
        x = torch.full((B + 1, 1 + gh * gw, D), fill, device=DEV)
        check(lib, lib.jimm_k_tokens_init_interp(ptr(cls), ptr(pos), g, D, ptr(x), B, gh, gw, stream()))
        out.append(x)
    assert _same(out[0][:B], out[1][:B]) and bool(torch.isnan(out[1][B]).all())


def test_embed_packed_extreme_ids(lib):
    """Out-of-range and negative ids in one sequence are clamped to the table and change no other sequence."""
    lens = [7, 64, 3, 77]
    V, D, T_ctx = 50, 128, 77
    off, off_d = _offsets(lens)
    T = int(off[-1])
    g = torch.Generator().manual_seed(60)
    ids0 = torch.randint(0, V, (T,), generator=g, dtype=torch.int32).to(DEV)
    table, pos = _randn(V, D, seed=61), _randn(T_ctx, D, seed=62)

    def run(ids):
        x = torch.full((T + PAD, D), -3.0, device=DEV)
        check(lib, lib.jimm_k_embed_packed(ptr(ids), ptr(table), ptr(pos), ptr(x), ptr(off_d), len(lens), T, D, V, stream()))
        return x

    clean = run(ids0)
    ids = ids0.clone()
    ids[int(off[1]) + 5], ids[int(off[1]) + 6] = 2 ** 31 - 1, -(2 ** 31)
    x = run(ids)
    keep = torch.ones(T + PAD, dtype=torch.bool, device=DEV)
    keep[int(off[1]) + 5:int(off[1]) + 7] = False
    assert _same(x[keep], clean[keep]) and torch.isfinite(x[:T]).all()
    assert torch.equal(x[int(off[1]) + 5], table[V - 1] + pos[5]) and torch.equal(x[int(off[1]) + 6], table[0] + pos[6])


def test_l2_normalize_and_logits_poisoned_rows(lib):
    """A zero row and a NaN row of image embeddings: only those rows of the logits may be non-finite, the NaN one is."""
    Bi, Bt, E = 9, 11, 96
    ie0, te = _randn(Bi, E, seed=70), _randn(Bt, E, seed=71)
    sc, bs = torch.tensor([2.3], device=DEV), torch.tensor([-1.7], device=DEV)

    def run(ie):
        i_n, t_n = torch.empty_like(ie), torch.empty_like(te)
        check(lib, lib.jimm_k_l2_normalize(ptr(ie), ptr(i_n), E, Bi, E, stream()))
        check(lib, lib.jimm_k_l2_normalize(ptr(te), ptr(t_n), E, Bt, E, stream()))
        out = torch.empty(Bi, Bt, device=DEV)
        check(lib, lib.jimm_k_logits(ptr(i_n), ptr(t_n), ptr(sc), ptr(bs), ptr(out), Bi, Bt, E, Bt, stream()))
        return out

    clean = run(ie0)
    ie = ie0.clone()
    ie[2] = 0
    ie[5] = NAN
    out = run(ie)
    keep = torch.ones(Bi, dtype=torch.bool, device=DEV)
    keep[[2, 5]] = False
    assert _same(out[keep], clean[keep])
    assert bool(_bad(out[5]).all())


def test_postprocess_non_finite_rows(lib):
    """Rows mixing NaN, +-inf and -0: order and argmax bit-exact against the oracle (NaN sorts first once reversed, the first NaN is
    the argmax, -0 ties +0); the clean rows are those of a clean call."""
    from jimm_b200.postprocess import classify, zero_shot

    x = torch.randn(6, 40, generator=torch.Generator().manual_seed(80)) * 4
    x[1, [3, 9]] = NAN
    x[2, [0, 5]] = INF
    x[2, 6] = -INF
    x[3, [2, 4]] = torch.tensor([-0.0, 0.0])
    x[3, [6, 8]] = torch.tensor([0.0, -0.0])  # -0 ties +0 in either order: the larger index comes first
    x[3, 10] = -INF
    x[4] = NAN
    x[5, [1, 30]] = torch.tensor([INF, NAN])
    _, order = zero_shot(x.cuda())
    _, ref_o = P.zero_shot_oracle(x.numpy())
    assert np.array_equal(order.cpu().numpy(), ref_o)
    assert np.array_equal(classify(x.cuda()).cpu().numpy(), P.classify_oracle(x.numpy()))
    clean = x.clone()
    clean[1:] = 0
    probs, order = zero_shot(x.cuda())
    p0, o0 = zero_shot(clean.cuda())
    assert _same(probs[0], p0[0]) and torch.equal(order[0], o0[0])


# ====================================================================================================================== models
def _set(model, params):
    for k, v in params.items():
        model.set_flat_param(k, v.to(torch.float32))
    return model


def _vit_small(dtype=torch.float16):
    from jimm_b200.models import VisionTransformer

    p = O.random_vit_params(O.ViTCfg(num_classes=10, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=512, hidden_size=128),
                            seed=11)
    return lambda: _set(VisionTransformer(num_classes=10, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=512, hidden_size=128,
                                          dtype=dtype), p).eval()


def _map_tower(dtype=torch.float16):
    from jimm_b200.common.vit import VisionTransformerBase

    # patch 14: rows of 588 values, padded to 592 columns
    kw = dict(img_size=56, patch_size=14, in_channels=3, hidden_size=256, num_layers=2, num_heads=4, mlp_dim=1024, pooling_type="MAP",
              use_quick_gelu=False, use_pre_norm=False, use_patch_bias=True, layernorm_epsilon=1e-6)
    p = O.random_tower_params(O.TowerCfg(**kw), seed=12)
    return lambda: _set(VisionTransformerBase(**kw, dtype=dtype), p)


DUAL = O.DualCfg(64, 2, 128, 16, 16, 100, 128, 4, 2)


def _dual(kind, dtype=torch.float16):
    from jimm_b200.models import CLIP, SigLIP

    p = O.random_dual_params(DUAL, kind, seed=13)
    return lambda: _set((CLIP if kind == "clip" else SigLIP)(64, 2, 128, 16, 16, 100, 128, 4, 2, dtype=dtype), p)


def _imgs(B, h=64, w=64, seed=0):
    return torch.randn((B, h, w, 3), generator=torch.Generator().manual_seed(seed))


def _poisoned(x, i, kind):
    y = x.clone()
    y[i, 5, 7, 1] = poison_value(kind)
    return y


def _rows_isolated(out, clean, i, what, need_bad=True):
    keep = torch.ones(out.shape[0], dtype=torch.bool, device=out.device)
    keep[i] = False
    assert _same(out[keep], clean[keep]), f"{what}: a clean row changed"
    if need_bad:
        assert bool(_bad(out[i]).any()), f"{what}: the poisoned row is finite"
    else:
        assert not _same(out[i], clean[i]), f"{what}: the poison changed nothing"


def _vision_cases(m, call, B, seed, kinds=POISONS, idx=None, size=64):
    x = _imgs(B, size, size, seed=seed).cuda()
    clean = call(m, x).clone()
    for i in (idx if idx is not None else (0, B // 2, B - 1)):
        for kind in kinds:
            out = call(m, _poisoned(x, i, kind))
            _rows_isolated(out, clean, i, f"B={B} image {i} {kind}")
    return clean


@pytest.mark.parametrize("B", [4, 40, 20], ids=["graph", "eager", "chunked"])
def test_vit_poisoned_image(B):
    """A small ViT: B = 4 replays a CUDA graph from its second call, B = 40 runs eagerly, B = 20 on a handle for 8 runs in three chunks.
    One poisoned image changes its own logits only."""
    m = _vit_small()()
    if B == 20:
        m.set_max_batch(8)
    clean = _vision_cases(m, lambda m, x: m(x), B, seed=B)
    assert _same(m(_imgs(B, seed=B).cuda()), clean), "a clean call after poisoned ones changed"


def test_vit_b16_poisoned_image():
    from jimm_b200.models import VisionTransformer

    m = _set(VisionTransformer(dtype=torch.float16), O.random_vit_params(O.ViTCfg(), seed=0)).eval()
    x = _imgs(4, 224, 224, seed=1).cuda()
    clean = m(x).clone()
    for kind in ("nan", "big"):
        _rows_isolated(m(_poisoned(x, 2, kind)), clean, 2, f"ViT-B/16 {kind}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.float8_e4m3fn], ids=["f16", "fp8"])
def test_map_tower_poisoned_image(dtype):
    _vision_cases(_map_tower(dtype)(), lambda m, x: m(x), 6, seed=2, size=56)


def test_vit_fp8_poisoned_image():
    _vision_cases(_vit_small(torch.float8_e4m3fn)(), lambda m, x: m(x), 6, seed=3)


@pytest.mark.parametrize("streams", ["1", "0"])
@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_dual_poisoned_image_and_prompt(kind, streams, monkeypatch):
    """encode_image, encode_text and the joint call: a poisoned image changes its own embedding and its own row of logits only; a
    prompt of extreme ids changes its own embedding and its own column only."""
    monkeypatch.setenv("JIMM_DUAL_STREAMS", streams)
    m = _dual(kind)()
    x = _imgs(5, seed=4).cuda()
    txt = O.synthetic_tokens(6, 16, 100, kind, seed=5).to(torch.int32).cuda()
    ci, ct, cl = m.encode_image(x).clone(), m.encode_text(txt).clone(), m(x, txt).clone()
    for kind_p in POISONS:
        xp = _poisoned(x, 3, kind_p)
        _rows_isolated(m.encode_image(xp), ci, 3, f"encode_image {kind_p}")
        _rows_isolated(m(xp, txt), cl, 3, f"logits {kind_p}")
    tp = txt.clone()
    tp[2, 4], tp[2, 9] = 2 ** 31 - 1, -(2 ** 31)
    _rows_isolated(m.encode_text(tp), ct, 2, "encode_text extreme ids", need_bad=False)
    _rows_isolated(m(x, tp).T, cl.T, 2, "logits extreme ids", need_bad=False)


def test_packed_image_list_poisoned():
    """A packed list of images of different sizes at interpolated positions: a poisoned image changes its own row only."""
    m = _vit_small()()
    g = torch.Generator().manual_seed(6)
    imgs = [torch.randn((h, w, 3), generator=g).cuda() for h, w in [(64, 64), (96, 80), (32, 48), (16, 16), (48, 112)]]
    clean = m(imgs, interpolate_pos_encoding=True).clone()
    for i in range(len(imgs)):
        for kind in POISONS:
            lst = list(imgs)
            lst[i] = imgs[i].clone()
            lst[i][3, 5, 0] = poison_value(kind)
            _rows_isolated(m(lst, interpolate_pos_encoding=True), clean, i, f"packed image {i} {kind}")


def test_packed_text_list_extreme_ids():
    m = _dual("clip")()
    g = torch.Generator().manual_seed(7)
    seqs = [torch.randint(1, 98, (L,), generator=g) for L in (3, 16, 9, 2, 12)]
    for s in seqs:
        s[-1] = 99
    clean = m.encode_text([s.cuda() for s in seqs]).clone()
    for i in range(len(seqs)):
        lst = [s.clone().cuda() for s in seqs]
        lst[i][0] = 2 ** 31 - 1 if i % 2 else -(2 ** 31)
        _rows_isolated(m.encode_text(lst), clean, i, f"packed text {i}", need_bad=False)


def test_host_path_poisoned_image():
    """forward_async on host images: a poisoned image changes its own row only, and the next host call is clean."""
    m = _vit_small()()
    x = _imgs(6, seed=8)
    clean = m.forward_async(x).result().clone()
    out = m.forward_async(_poisoned(x, 4, "nan")).result()
    _rows_isolated(out, clean, 4, "host path")
    assert _same(m.forward_async(x).result(), clean)


# ====================================================================================================================== across calls
def _all_poisoned(B, seed, px):
    x = _imgs(B, px, px, seed=seed)
    for i in range(B):
        x[i, :, :, i % 3] = poison_value(POISONS[i % 4])
    return x.cuda()


@pytest.mark.parametrize("model", ["vit", "map", "clip"])
def test_poisoned_call_leaves_nothing_behind(model):
    """A handle for 8 images first runs 8 poisoned ones, which leaves NaN / inf in every workspace row; then a smaller batch, a batch at
    another resolution, a packed list, a graph-replayed B = 4 and a host call each give the bits of a handle that never saw it."""
    make = {"vit": _vit_small(), "map": _map_tower(), "clip": _dual("clip")}[model]
    call = (lambda m, x, **kw: m.encode_image(x, **kw)) if model == "clip" else (lambda m, x, **kw: m(x, **kw))
    g = torch.Generator().manual_seed(9)
    px, o = (56, 42) if model == "map" else (64, 48)
    small = _imgs(3, px, px, seed=10).cuda()
    other = _imgs(8, o, o, seed=11).cuda()
    lst = [torch.randn((h, w, 3), generator=g).cuda() for h, w in [(px, px), (o - 14, o), (o, 16)]]
    four = _imgs(4, px, px, seed=12).cuda()
    host = _imgs(5, px, px, seed=13)

    def cases(m):
        return [call(m, small), call(m, other, interpolate_pos_encoding=True), call(m, lst, interpolate_pos_encoding=True), call(m, four),
                call(m, host)]

    used = make().set_max_batch(8)
    call(used, four)  # the first call of B = 4 runs eagerly; the one in cases() is captured and replayed
    out = call(used, _all_poisoned(8, 14, px))
    assert bool(_bad(out).any(-1).all()), "the poisoned batch is not non-finite in every row"
    if model == "clip":
        bad_t = O.synthetic_tokens(8, 16, 100, "clip", seed=15).to(torch.int32)
        bad_t[:, 3] = 2 ** 31 - 1
        used.encode_text(bad_t.cuda())
    got = cases(used)
    fresh = make().set_max_batch(8)
    call(fresh, four)
    ref = cases(fresh)
    for name, a, b in zip(["smaller batch", "other resolution", "packed list", "graph B=4", "host call"], got, ref):
        assert _same(a, b), f"{model}: {name} differs after a poisoned call"
