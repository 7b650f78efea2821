"""GEMM epilogues, activations and LayerNorm checked element by element: |out - ref| <= bound at EVERY element, with ref in fp64 and a
bound derived per element from the operation's error model (assert_within), rather than max|out - ref| <= tol * max|ref| over the
whole tensor.  A max-normalised tolerance is set by the largest output and cannot see an error in an element that is small next to
it: the activations' negative tails, LayerNorm outputs near the row mean, outputs near zero.

- CPU: assert_within passes an exact result and flags one perturbed element.
- jimm_k_activation (act 0, 1, 2) on an fp32 sweep of every binade, the specials, a dense grid and the flush thresholds, and the public
  common.transformer.quickgelu on fp16 / bf16 / strided input.
- jimm_k_gemm_ex / jimm_k_gemm / jimm_k_gemm_e4m3: every epilogue (TMA stores, LSU, SIMT, row-add with row remap, separate residual,
  in-place reduce-add, token scatter, the e4m3 scaled stores) x {none, GELU, QuickGELU}, on pre-activations spread over about
  [-12, 12]; ragged multi-wave shapes and the QKV / FC1 / FC2 shapes of real towers.
- jimm_k_layernorm / jimm_k_layernorm_e4m3 and the fused LayerNorm of the reduce-add GEMM (N = 128 and 256 included) against an fp64
  LayerNorm of the residual rows the kernel read; the fused path's refusal of the widths it does not take.

Error model of one GEMM element (u = 2^-24, the fp32 unit roundoff):
    bound = slope * (c_acc * sum_k |a_k b_k| + u |pre|) + act_err(pre) + u_out |ref| + u * (sum of |terms| added in fp32) + eta_out
- sum_k |a_k b_k| in fp64 over the operands as passed (rounded to the operand type; e4m3: dequantised).  c_acc is the tensor-core
  accumulation constant of the operand type (C_ACC, measured by test_accumulation_constant); the SIMT kernel's serial fp32 FMA
  chain has the classical c_acc = K u.
- u |pre|: the fp32 addition of the bias to the accumulator.  slope = max |act'|: 1, 1.13 (GELU, max 1.1290), 1.1 (QuickGELU,
  max 1.0998).
- act_err: the activation's own error (see act_bound), including its flush to zero: |pre| 2^-126.
- u_out: the output type's unit roundoff; eta_out: half its smallest subnormal step (the rounding model's underflow term; 2^-25 for
  fp16, at most 2^-134 for the others).
"""

import math

import numpy as np
import pytest
import torch

import fp8_oracle as F
from bounds_util import OUT, U, assert_within
from gpu_util import CODE, F16, check, gemm, ptr, record_parity, stream
from test_fp8_gpu import gemm8
from test_kernel_paths_gpu import SENTINEL, gemm_ex, rna_tf32

DEV = "cuda"
LOG2E = 1.0 / math.log(2.0)
OPS = ["f16", "bf16", "tf32"]
OP_DTYPE = {"f16": torch.float16, "bf16": torch.bfloat16, "tf32": torch.float32}
SLOPE = [1.0, 1.13, 1.1]
# Tensor-core accumulation constants, max |out - sum a b| / sum |a b| per element: about 4x the worst value test_accumulation_constant
# measured on an H100 80GB HBM3 (700 W power limit) over K = 768 .. 5120: f16 7.5e-7, bf16 7.2e-7, tf32 1.56e-6 (all at K = 5120),
# e4m3 5.8e-5 (K = 768; the K-slab promotion keeps it from growing with K).
C_ACC = {"f16": 3e-6, "bf16": 3e-6, "tf32": 6e-6, "e4m3": 2.4e-4}


# ---------------------------------------------------------------------------------------------------------------- the per-element check
def test_assert_within_flags_one_element():
    """CPU: an exact result passes with ratio 0; one element off by 1.5 x its bound fails and the message names it; NaN fails."""
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(37, 53, generator=g, dtype=torch.float64)
    bound = 1e-6 * ref.abs() + 1e-30
    assert assert_within("self-test", "exact", ref.clone(), ref, bound) == 0.0
    out = ref + 0.5 * bound
    assert abs(assert_within("self-test", "half the bound", out, ref, bound) - 0.5) < 1e-6
    out[17, 29] = ref[17, 29] + 1.5 * bound[17, 29]
    with pytest.raises(AssertionError, match=r"= 1\.5 at \(17, 29\)"):
        assert_within("self-test", "one perturbed element", out, ref, bound)
    out = ref.clone()
    out[3, 4] = float("nan")
    with pytest.raises(AssertionError, match=r"at \(3, 4\): out=nan"):
        assert_within("self-test", "NaN", out, ref, bound)


# ---------------------------------------------------------------------------------------------------------------- activations in fp64
def act_ref(x, act):
    """fp64 reference.  GELU: 0.5 x (1 + tanh(u)) == x sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3); the sigmoid form is used
    because 1 + tanh(u) cancels in fp64 once u < -19, where the tail is still far above fp32's flush threshold."""
    if act == 0:
        return x
    if act == 1:
        return x * torch.sigmoid(2.0 * math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3))
    return x * torch.sigmoid(1.702 * x)


def act_z(x, act):
    """The exponent the kernel computes (common.cuh): act(x) = x / (1 + 2^z)."""
    if act == 1:
        return -2.0 * math.sqrt(2.0 / math.pi) * LOG2E * x * (1.0 + 0.044715 * x * x)
    return -1.702 * LOG2E * x


K_ACT = 8.0


def act_bound(x, y, act):
    """Bound on |kernel act(x) - act(x)| for an exact fp32 argument x, y = act(x) in fp64:
        K_ACT u (1 + w |z|) |y| + |x| 2^-126 + 2^-150,    w = 2^z / (1 + 2^z),  K_ACT = 8.
    The kernel computes y' = x * rcp(1 + ex2(z')).  z' carries the roundings of the folded fp32 constants and of its own arithmetic:
    GELU c0 (3 roundings), c1 = c0 * 0.044715f (5), x*x, the fma and x*w (3 more): |z' - z| <= 8u|z|; QuickGELU 4u|z|.  2^z' =
    2^z (1 + ln2 (z' - z)) (1 + e_ex2) with |e_ex2| <= 2 ulp = 4u (ex2.approx.f32); 1 + 2^z' is one rounding (u); rcp.approx.f32 is
    within 1 ulp (2u); x * r one more (u).  A relative error e of 2^z moves 1 / (1 + 2^z) by w e, so
        |y' / y - 1| <= w (4u + 5.6u|z|) + 4u <= 8u (1 + w|z|).
    The relative form (|y|, not |x|) is what lets the tail be checked down to the flush region.  Flush: rcp.approx.ftz returns 0 once
    1 + 2^z' > 2^126 (z' >= 126), and 2^z' overflows to inf at z' >= 128, so y' = 0 while |y| <= |x| 2^-126.  The fp32 product x * r
    underflows into the subnormals with an absolute error of at most 2^-150."""
    z = act_z(x, act)
    w = torch.sigmoid(z * math.log(2.0))
    rel = K_ACT * U * (1.0 + w * z.abs()) * y.abs()
    return torch.where(y == 0, torch.zeros_like(rel), rel) + x.abs() * 2.0 ** -126 + 2.0 ** -150


# ---------------------------------------------------------------------------------------------------------------- activation kernel
N_BIG = 3 * 2 ** 20 + 5


def _crossings():
    """fp32 x at which each activation's z crosses +-126 and +-128, with 4 float neighbours on each side."""
    c0 = -2.0 * math.sqrt(2.0 / math.pi) * LOG2E
    xs = []
    for zt in (126.0, 128.0, -126.0, -128.0):
        xs.append(zt / (-1.702 * LOG2E))
        r = [v.real for v in np.roots([c0 * 0.044715, 0.0, c0, -zt]) if abs(v.imag) < 1e-9]
        xs += r
    out = []
    for x in np.array(xs, dtype=np.float32):
        v = x
        for _ in range(5):
            v = np.nextafter(v, np.float32(-np.inf))
        for _ in range(9):
            v = np.nextafter(v, np.float32(np.inf))
            out.append(v)
    return np.array(out, dtype=np.float32)


def _sweep():
    """N_BIG fp32 values, specials first: +-0, +-inf, NaN; the flush thresholds; every binade 2^-149 .. 2^127 of both signs with several
    mantissas (the low ones round into the subnormals); then a dense grid over [-60, 60]."""
    rng = np.random.default_rng(0)
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], dtype=np.float32)
    mant = np.concatenate([[1.0, 1.0 + 2.0 ** -23, 1.25, 1.5, 1.75, 2.0 - 2.0 ** -23], rng.uniform(1, 2, 3)])
    e = np.arange(-149, 128)
    binades = (np.ldexp(mant[None, :], e[:, None]).reshape(-1)).astype(np.float32)
    binades = np.stack([binades, -binades], 1).reshape(-1)
    head = np.concatenate([special, _crossings(), binades])
    dense = np.linspace(-60.0, 60.0, N_BIG - head.size).astype(np.float32)
    return torch.from_numpy(np.concatenate([head, dense]))


_SWEEP = None


def sweep():
    global _SWEEP
    if _SWEEP is None:
        _SWEEP = _sweep()
    return _SWEEP


def activation(lib, x, act, pad=0):
    y = torch.full((x.numel() + pad,), SENTINEL, device=DEV)
    check(lib, lib.jimm_k_activation(ptr(x), ptr(y), x.numel(), act, stream()))
    torch.cuda.synchronize()
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "gelu", "quickgelu"])
@pytest.mark.parametrize("n", [0, 1, 255, 257, N_BIG])
def test_activation_kernel(lib, n, act):
    """y = act(x) within act_bound at every finite x; NaN -> NaN, +inf -> +inf, -inf -> what fp64 torch gives on the same formula
    (NaN: -inf * sigmoid(-inf) = -inf * 0; intended, the formula has no limit to agree on); act 0 returns the input's bits; the
    n + 64 elements after y[n - 1] keep their sentinel."""
    xc = sweep()[:n]
    x = xc.to(DEV)
    y = activation(lib, x, act, pad=64)
    assert bool((y[n:] == SENTINEL).all()), "elements past n were written"
    y = y[:n].cpu()
    if act == 0:
        assert torch.equal(y.view(torch.int32), xc.view(torch.int32))
        return
    fin = torch.isfinite(xc)
    xd = xc.double()
    ref = act_ref(xd, act)
    for v in (float("nan"), float("-inf")):
        sel = torch.isnan(xc) if v != v else xc == v
        assert bool(torch.isnan(y[sel]).all()) and bool(torch.isnan(ref[sel]).all()), (v, y[sel])
    sel = xc == float("inf")
    assert bool((y[sel] == float("inf")).all())
    if int(fin.sum()):
        bound = act_bound(xd[fin], ref[fin], act)
        assert_within(f"jimm_k_activation act={act} n={n}", "elementwise", y[fin], ref[fin], bound)
        # The ratio above is set where the absolute terms are tight (subnormal x * 0.5, the flush at z = 126); report the one where
        # the relative term is the bound too: normal outputs away from the flush threshold.
        rel = (ref[fin].abs() >= 2.0 ** -126) & (act_z(xd[fin], act) < 120)
        if int(rel.sum()):
            assert_within(f"jimm_k_activation act={act} n={n}", "elementwise, normal y, z < 120", y[fin][rel], ref[fin][rel], bound[rel])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["f16", "bf16", "strided_f32"])
def test_public_quickgelu(lib, kind):
    """common.transformer.quickgelu on fp16, bf16 and a non-contiguous fp32 view: the bits of jimm_k_activation(act 2) on
    x.float().contiguous(), in x's shape."""
    from jimm_b200.common.transformer import quickgelu

    base = sweep()[5:].view(-1)[: 6 * 1000 * 37].view(6, 1000, 37).to(DEV)  # finite values (the specials stripped)
    x = {"f16": base.half(), "bf16": base.bfloat16(), "strided_f32": base.transpose(0, 2)[::2]}[kind]
    assert kind != "strided_f32" or not x.is_contiguous()
    y = quickgelu(x)
    assert y.shape == x.shape and y.dtype == torch.float32
    xf = x.float().contiguous()
    want = activation(lib, xf.view(-1), 2).view(x.shape)
    assert torch.equal(y.contiguous().view(torch.int32), want.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------- GEMM operands
class Case:
    """Operands whose pre-activations spread over about [-12, 12]: row i of A scaled by f_i in [0.02, 2.5] and a bias spread over
    [-6, 6], so every row has a negative tail and the low-f rows sit near zero or near their bias.  pre = A B^T + bias and
    S = |A| |B|^T in fp64 on the operands as passed."""

    def __init__(self, M, N, K, op, seed):
        g = torch.Generator().manual_seed(seed)
        f = torch.empty(M, 1).uniform_(0.02, 2.5, generator=g)
        a = torch.randn(M, K, generator=g) * f
        b = torch.randn(N, K, generator=g) / math.sqrt(K)
        self.bias = (torch.rand(N, generator=g) * 12 - 6).to(DEV)
        self.op = op
        if op == "e4m3":
            qa, sa = F.quantize_rows(a)
            qb, sb = F.quantize_rows(b)
            self.ops = (qa.view(torch.uint8).to(DEV), sa.to(DEV), qb.view(torch.uint8).to(DEV), sb.to(DEV))
            Ad, Bd = F.dequant(qa, sa).to(DEV), F.dequant(qb, sb).to(DEV)
        else:
            dt = OP_DTYPE[op]
            self.A, self.B = (rna_tf32(a.to(DEV)), rna_tf32(b.to(DEV))) if op == "tf32" else (a.to(DEV, dt), b.to(DEV, dt))
            Ad, Bd = self.A.double(), self.B.double()
        self.M, self.N, self.K = M, N, K
        self.pre = Ad @ Bd.T + self.bias.double()
        self.S = Ad.abs() @ Bd.abs().T

    def run(self, lib, out, *, act=0, out_code=None, mode=2, impl=0, residual=None):
        if self.op == "e4m3":
            return check(lib, gemm8(lib, self.ops, out, bias=self.bias, act=act, out_code=out_code, mode=mode, impl=impl))
        if impl == 1:
            return gemm(lib, self.A, self.B, bias=self.bias, act=act, residual=residual, out=out, impl=1, mode=mode)
        return check(lib, gemm_ex(lib, self.A, self.B, out, bias=self.bias, act=act, out_code=out_code, mode=mode, residual=residual))

    def bound(self, act, out_t, ref, c_acc=None, added=None):
        """The module docstring's bound for act(pre) (+ the fp32 terms `added`, as the sum of their magnitudes) stored as out_t."""
        c = C_ACC[self.op] if c_acc is None else c_acc
        _, _, u_out, eta = OUT[out_t]
        b = SLOPE[act] * (c * self.S + U * self.pre.abs()) + u_out * ref.abs() + eta
        if act:
            b = b + act_bound(self.pre, act_ref(self.pre, act), act)
        if added is not None:
            b = b + U * added
        return b


_CASES = {}


def case(M, N, K, op, seed):
    key = (M, N, K, op, seed)
    if key not in _CASES:
        _CASES.clear()  # one at a time: the fp64 products of a tower shape are 100 MB
        _CASES[key] = Case(M, N, K, op, seed)
    return _CASES[key]


def _canvas(rows, cols, dt):
    return torch.full((rows, cols), SENTINEL, dtype=dt, device=DEV)


def _untouched(t):
    return bool((t.float() == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------------- GEMM: c_acc
@pytest.mark.gpu
@pytest.mark.parametrize("K", [768, 1008, 4304, 5120])
@pytest.mark.parametrize("op", OPS + ["e4m3"])
def test_accumulation_constant(lib, op, K):
    """fp32 output of the plain TMA store, no bias or activation: max |out - sum a b| / sum |a b| is the accumulation constant c_acc
    of the operand type's wgmma (e4m3: with the K-slab promotion).  Recorded per K; asserted below C_ACC."""
    M, N = 1154, 1024
    c = case(M, N, K, op, seed=K)
    out = torch.empty(M, N, device=DEV)
    if op == "e4m3":
        check(lib, gemm8(lib, c.ops, out))
    else:
        check(lib, gemm_ex(lib, c.A, c.B, out))
    torch.cuda.synchronize()
    exact = c.pre - c.bias.double()
    per = float(((out.double() - exact).abs() / c.S).max())
    record_parity(f"GEMM {M}x{N}x{K}", "accumulation error / sum|a b|", op, "fp64", C_ACC[op], per)
    assert per < C_ACC[op], f"{op} K={K}: max |err| / sum|a b| = {per:.3e} >= c_acc {C_ACC[op]:.1e}"


# ---------------------------------------------------------------------------------------------------------------- GEMM: plain stores
@pytest.mark.gpu
@pytest.mark.parametrize("out_t", list(OUT))
@pytest.mark.parametrize("op", OPS + ["e4m3"])
def test_store_epilogues(lib, op, out_t):
    """TMA store (mode 2) and LSU (mode 0) x {none, GELU, QuickGELU}, 3001 x 2296 x 1008: 24 x 9 tiles (e4m3: 47 x 9), more than
    one wave on 132 SMs, ragged in M, N and K.  Columns N .. ldo and rows >= roundup(M, 16) keep their sentinel."""
    M, N, K, ldo = 3001, 2296, 1008, 2320
    c = case(M, N, K, op, seed=1)
    dt, code, _, _ = OUT[out_t]
    r16 = (M + 15) // 16 * 16
    for act in (0, 1, 2):
        ref = act_ref(c.pre, act)
        bnd = c.bound(act, out_t, ref)
        for mode in (2, 0):
            buf = _canvas(M + 40, ldo, dt)
            c.run(lib, buf, act=act, out_code=code, mode=mode)
            torch.cuda.synchronize()
            assert_within(f"{op} GEMM {M}x{N}x{K} mode={mode} act={act}", f"store {out_t}", buf[:M, :N], ref, bnd, op)
            assert _untouched(buf[:, N:]), (act, mode, "columns between N and ldo written")
            assert _untouched(buf[r16:]), (act, mode, "rows >= roundup(M, 16) written")


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS + ["e4m3"])
def test_simt_epilogue(lib, op):
    """The SIMT kernel (impl 1): a serial fp32 FMA chain per element, c_acc = K u (the classical gamma_K bound), stores in f32 and
    bf16, x {none, GELU, QuickGELU}."""
    M, N, K = 300, 520, 768
    c = case(M, N, K, op, seed=2)
    for out_t in ("f32", "bf16"):
        dt, code, _, _ = OUT[out_t]
        for act in (0, 1, 2):
            ref = act_ref(c.pre, act)
            out = _canvas(M, N, dt)
            c.run(lib, out, act=act, out_code=code, mode=0, impl=1)
            torch.cuda.synchronize()
            assert_within(f"{op} SIMT GEMM {M}x{N}x{K} act={act}", f"store {out_t}", out, ref, c.bound(act, out_t, ref, c_acc=K * U), op)


# ---------------------------------------------------------------------------------------------------------------- GEMM: generic epilogue
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])  # mode 2 falls back to the generic epilogue (row-add, row remap)
@pytest.mark.parametrize("op", OPS)
def test_rowadd_row_remap(lib, op, mode):
    """The patch GEMM's generic epilogue: out[b * 197 + p + 1] = act(A[b * 196 + p] B^T + bias) + rowadd[p + 1]; row 0 of each sample
    (the CLS row) keeps its sentinel.  f32 and bf16 outputs, x {none, GELU, QuickGELU}."""
    rows_in, rows_out, row_off, nb = 196, 197, 1, 9
    M, N, K = rows_in * nb, 776, 592
    c = case(M, N, K, op, seed=3)
    rowadd = torch.randn(rows_out, N, generator=torch.Generator().manual_seed(4)).to(DEV)
    add = rowadd[row_off: row_off + rows_in].double().repeat(nb, 1)
    dst = (torch.arange(M, device=DEV) // rows_in) * rows_out + torch.arange(M, device=DEV) % rows_in + row_off
    for out_t in ("f32", "bf16"):
        dt = OUT[out_t][0]
        for act in (0, 1, 2):
            a = act_ref(c.pre, act)
            ref = a + add
            out = _canvas(nb * rows_out, N, dt)
            check(lib, lib.jimm_k_gemm(0, CODE[c.A.dtype], ptr(c.A), K, ptr(c.B), K, M, N, K, ptr(c.bias), act, ptr(rowadd), None, 0,
                                       ptr(out), OUT[out_t][1], N, rows_in, rows_out, row_off, mode, stream()))
            torch.cuda.synchronize()
            assert_within(f"{op} GEMM rowadd+remap mode={mode} act={act}", f"store {out_t}", out[dst], ref,
                          c.bound(act, out_t, ref, added=a.abs() + add.abs()), op)
            assert _untouched(out.view(nb, rows_out, N)[:, :row_off]), "rows outside the remap written"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])  # mode 2 falls back to the generic epilogue: the residual is not the output
@pytest.mark.parametrize("op", OPS)
def test_separate_residual(lib, op, mode):
    """out = act(A B^T + bias) + residual with residual != out (the MAP head's fc2); the residual keeps its bits, columns N .. ldo
    their sentinel."""
    M, N, K = 1000, 700, 3072
    c = case(M, N, K, op, seed=5)
    res_buf = torch.randn(M, N + 36, generator=torch.Generator().manual_seed(6)).to(DEV) * 4
    res = res_buf[:, :N]
    res0 = res_buf.clone()
    for out_t in ("f32", "f16"):
        dt, code, _, _ = OUT[out_t]
        for act in (0, 1, 2):
            a = act_ref(c.pre, act)
            ref = a + res.double()
            out = _canvas(M, N + 12, dt)
            check(lib, gemm_ex(lib, c.A, c.B, out, bias=c.bias, act=act, residual=res, mode=mode, out_code=code))
            torch.cuda.synchronize()
            assert_within(f"{op} GEMM residual mode={mode} act={act}", f"store {out_t}", out[:, :N], ref,
                          c.bound(act, out_t, ref, added=a.abs() + res.double().abs()), op)
            assert _untouched(out[:, N:])
            assert torch.equal(res_buf, res0)


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS)
def test_inplace_reduce_add(lib, op):
    """x += act(A B^T + bias) in place: act none takes the TMA reduce-add (the add done in L2), GELU the generic epilogue (an
    activation with a residual); rows >= M of x keep their bits."""
    M, N, K = 3001, 1152, 1000
    c = case(M, N, K, op, seed=7)
    x0 = torch.randn(M + 30, N, generator=torch.Generator().manual_seed(8)).to(DEV) * 3 + 1
    for act in (0, 1):
        x = x0.clone()
        check(lib, gemm_ex(lib, c.A, c.B, x, M=M, bias=c.bias, act=act, residual=x))
        torch.cuda.synchronize()
        a = act_ref(c.pre, act)
        ref = x0[:M].double() + a
        assert_within(f"{op} GEMM in-place reduce-add act={act}", "x", x[:M], ref, c.bound(act, "f32", ref, added=a.abs() + x0[:M].double().abs()), op)
        assert torch.equal(x[M:], x0[M:])


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("tok_off", [0, 1], ids=["map", "cls"])
def test_token_scatter(lib, tok_off, op):
    """The patch embedding's token scatter: A row b * n_pad + p reduce-added into x[b, p + tok_off]; pad rows of A are NaN, the CLS
    rows and the rows past the last sample keep their bits."""
    n, D, K = 196, 768, 592
    n_pad, S = 224, 196 + tok_off
    nb = 12
    M = nb * n_pad
    c = case(M, D, K, op, seed=9 + tok_off)
    A = c.A.clone()
    A.view(nb, n_pad, K)[:, n:] = float("nan")
    init = torch.randn(nb * S + 8, D, generator=torch.Generator().manual_seed(10)).to(DEV)
    x = init.clone()
    check(lib, gemm_ex(lib, A, c.B, x, bias=c.bias, residual=x, tok=(n_pad, tok_off, S)))
    torch.cuda.synchronize()
    pre = c.pre.view(nb, n_pad, D)[:, :n]
    S_ = c.S.view(nb, n_pad, D)[:, :n]
    x0 = init[: nb * S].view(nb, S, D)[:, tok_off:].double()
    ref = x0 + pre
    got = x[: nb * S].view(nb, S, D)[:, tok_off:]
    bound = C_ACC[op] * S_ + U * pre.abs() + U * (x0.abs() + pre.abs()) + U * ref.abs() + 2.0 ** -150
    assert_within(f"{op} token scatter tok_off={tok_off}", "x", got, ref, bound, op)
    touched = torch.zeros(x.shape[0], dtype=torch.bool, device=DEV)
    touched[: nb * S].view(nb, S)[:, tok_off:] = True
    assert torch.equal(x[~touched], init[~touched])


# ---------------------------------------------------------------------------------------------------------------- GEMM: tower shapes
TOWERS = {768: 3072, 1024: 4096, 1152: 4304, 1280: 5120}  # width -> MLP width


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS + ["e4m3"])
@pytest.mark.parametrize("D", list(TOWERS))
def test_tower_projection_shapes(lib, D, op):
    """M = 2 x 577 tokens through the projections of a real tower, with the epilogue the encoder gives each: QKV (D -> 3D) stored
    in the operand type (e4m3: f16), FC1 (D -> MLP) with GELU and with QuickGELU, FC2 (MLP -> D) reduce-added into the fp32
    residual stream (not e4m3: the FP8 mode runs FC2 in fp16)."""
    M, mlp = 2 * 577, TOWERS[D]
    out_t = "f16" if op == "e4m3" else op
    dt, code, _, _ = OUT[out_t]
    for name, N, K, acts in (("qkv", 3 * D, D, (0,)), ("fc1", mlp, D, (1, 2))):
        c = case(M, N, K, op, seed=D + N)
        for act in acts:
            ref = act_ref(c.pre, act)
            out = _canvas(M, N, dt)
            c.run(lib, out, act=act, out_code=code)
            torch.cuda.synchronize()
            assert_within(f"{op} D={D} {name} {M}x{N}x{K} act={act}", f"store {out_t}", out, ref, c.bound(act, out_t, ref), op)
    if op == "e4m3":
        return
    c = case(M, D, mlp, op, seed=D + mlp + 1)
    x0 = torch.randn(M, D, generator=torch.Generator().manual_seed(D)).to(DEV) * 2
    x = x0.clone()
    check(lib, gemm_ex(lib, c.A, c.B, x, bias=c.bias, residual=x))
    torch.cuda.synchronize()
    ref = x0.double() + c.pre
    assert_within(f"{op} D={D} fc2 {M}x{D}x{mlp}", "x", x, ref, c.bound(0, "f32", ref, added=x0.double().abs() + c.pre.abs()), op)


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
def ln_rows(rows, D, seed):
    """Residual-stream rows of four kinds, cycling: plain (N(0.5, 4)); a mean 20 .. 60 times the spread; one outlier channel of
    |x| 50 .. 200 (as in CLIP-L streams); quiet rows of spread 3e-3, whose variance is of the order of eps (eps is observable)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, D, generator=g)
    k = torch.arange(rows) % 4
    sign = torch.where(torch.rand(rows, generator=g) < 0.5, -1.0, 1.0)
    s = torch.empty(rows).uniform_(0.5, 1.5, generator=g)
    r = torch.empty(rows).uniform_(20, 60, generator=g)
    x[k == 0] = x[k == 0] * 2 + 0.5
    x[k == 1] = (x * s[:, None] + (sign * r * s)[:, None])[k == 1]
    out_v = sign * torch.empty(rows).uniform_(50, 200, generator=g)
    oc = torch.randint(0, D, (rows,), generator=g)
    i2 = torch.nonzero(k == 2).squeeze(1)
    x[i2, oc[i2]] = out_v[i2]
    x[k == 3] = x[k == 3] * 3e-3
    return x


def ln_ref_bound(x, g, b, eps, u_out, eta):
    """fp64 LayerNorm of the fp32 rows x and the bound on the kernel's error.  The kernel (one warp per row; the fused path the same
    arithmetic): s = sum x, s2 = sum x^2 in fp32, each lane summing its D / 128 float4 (3 adds inside one) then a 5-level shuffle
    tree, so every term passes through at most n = D / 128 + 8 roundings: |ds| <= n u sum|x|, |ds2| <= (n + 1) u sum x^2.
    mean = s * fl(1/D): |dmean| <= (n + 2) u E|x|.  var = max(0, s2/D - mean^2) (flax's fast variance):
    |dvar| <= (n + 3) u E[x^2] + (2n + 5) u mean^2 + u var <= (3n + 9) u E[x^2] -- the cancellation that makes rows with a large mean
    the hard case.  rstd = rsqrtf(var + eps) (2 ulp, 4u; the add u): |drstd| / rstd <= (1 - dvar / (var + eps))^-1/2 - 1 + 6u.
    y = (x - mean) rstd g + b: (x - mean), the two products, and the final add relative to |y|:
        bound = |g| rstd (|dmean| + |x - mean| (|drstd| / rstd + 4u)) + (u + u_out) |y| + eta_out."""
    D = x.shape[-1]
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    ref = (x - mean) * rstd * g.double() + b.double()
    n = math.ceil(D / 128) + 8
    dmean = (n + 2) * U * x.abs().mean(-1, keepdim=True)
    dvar = (3 * n + 9) * U * (x * x).mean(-1, keepdim=True)
    q = dvar / (var + eps)
    assert bool((q < 0.5).all()), "rows too ill-conditioned for a first-order bound"
    drel = (1.0 - q) ** -0.5 - 1.0 + 6 * U
    bound = g.double().abs() * rstd * (dmean + (x - mean).abs() * (drel + 4 * U)) + (U + u_out) * ref.abs() + eta
    return ref, bound


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("D", [128, 768, 1024, 1280, 2048])
def test_layernorm(lib, D, eps):
    """jimm_k_layernorm to f32, tf32, f16 and bf16, and jimm_k_layernorm_e4m3 dequantised with its row scales (e4m3: u_out = 2^-4,
    eta = 2^-10 x the row scale)."""
    rows = 1003
    x = ln_rows(rows, D, seed=D).to(DEV)
    gen = torch.Generator().manual_seed(D + 1)
    sc = (torch.randn(D, generator=gen) * 1.5).to(DEV)
    bi = (torch.randn(D, generator=gen) * 0.5).to(DEV)
    for out_t in ("f32", "tf32", "f16", "bf16"):
        dt, code, u_out, eta = OUT[out_t]
        y = torch.empty(rows, D, dtype=dt, device=DEV)
        check(lib, lib.jimm_k_layernorm(ptr(x), D, 1, 0, None, ptr(sc), ptr(bi), eps, ptr(y), code, D, rows, D, stream()))
        torch.cuda.synchronize()
        ref, bound = ln_ref_bound(x, sc, bi, eps, u_out, eta)
        assert_within(f"LayerNorm {rows}x{D} eps={eps}", f"out {out_t}", y, ref, bound)
    q = torch.empty(rows, D, dtype=torch.uint8, device=DEV)
    s = torch.empty(rows, device=DEV)
    check(lib, lib.jimm_k_layernorm_e4m3(ptr(x), D, ptr(sc), ptr(bi), eps, ptr(q), D, ptr(s), rows, D, 0, stream()))
    torch.cuda.synchronize()
    deq = q.view(torch.float8_e4m3fn).double() * s.double()[:, None]
    ref, bound = ln_ref_bound(x, sc, bi, eps, 2.0 ** -4, 0.0)
    assert_within(f"LayerNorm {rows}x{D} eps={eps}", "out e4m3 (dequantised)", deq, ref, bound + 2.0 ** -10 * s.double()[:, None])


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("N", [128, 256, 768, 1152])
def test_fused_layernorm(lib, N, op):
    """x += A B^T + bias, then the fused LayerNorm of each completed 32-row group in the operand type, at M = 16, 100 and 4000 and
    both tile walks: x within the reduce-add bound; the normalised rows within ln_ref_bound of an fp64 LayerNorm of the x the GEMM
    left (read back from the GPU); rows >= M of the LayerNorm output keep their sentinel; the counters are back at zero."""
    K, eps = 256, 1e-5
    out_t = op
    dt, code, u_out, eta = OUT[out_t]
    gen = torch.Generator().manual_seed(N)
    sc = (torch.randn(N, generator=gen) * 1.5).to(DEV)
    lb = (torch.randn(N, generator=gen) * 0.5).to(DEV)
    for M in (16, 100, 4000):
        c = case(M, N, K, op, seed=N + M)
        x0 = ln_rows(M + 32, N, seed=M).to(DEV)
        # small updates (the rows keep their kind: quiet rows stay quiet): A and bias scaled by 1e-4 in the exact arithmetic below
        A = (c.A.float() * 1e-4).to(c.A.dtype) if op != "tf32" else rna_tf32(c.A * 1e-4)
        bias = c.bias * 1e-4
        Ad = A.double()
        pre = Ad @ c.B.double().T + bias.double()
        S = Ad.abs() @ c.B.double().abs().T
        for rev in (0, 1):
            x = x0.clone()
            h = _canvas(M + 32, N, dt)
            cnt = torch.zeros(M // 32 + 2, dtype=torch.int32, device=DEV)
            check(lib, gemm_ex(lib, A, c.B, x, M=M, bias=bias, residual=x, reverse=rev, ln=(sc, lb, eps, h, code, cnt)))
            torch.cuda.synchronize()
            case_ = f"{op} fused LayerNorm M={M} N={N} reverse={rev}"
            ref = x0[:M].double() + pre
            bx = C_ACC[op] * S + U * pre.abs() + U * (x0[:M].double().abs() + pre.abs()) + U * ref.abs() + 2.0 ** -150
            assert_within(case_, "x", x[:M], ref, bx, op)
            assert torch.equal(x[M:], x0[M:])
            yref, yb = ln_ref_bound(x[:M], sc, lb, eps, u_out, eta)
            assert_within(case_, f"LayerNorm out {out_t}", h[:M], yref, yb, op)
            assert _untouched(h[M:]), "LayerNorm rows >= M written"
            assert int(cnt.abs().sum()) == 0, "counters not back at zero"


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1280, 1536, 2048])
def test_fused_layernorm_refuses_wide_rows(lib, N):
    """Rows of 10, 12 and 16 x 128 are left to the LayerNorm kernel: -1 with the message, nothing launched, x untouched."""
    M, K = 64, 128
    A = torch.randn(M, K, device=DEV).half()
    B = torch.randn(N, K, device=DEV).half()
    x = torch.randn(M, N, device=DEV)
    x0 = x.clone()
    sc, lb = torch.ones(N, device=DEV), torch.zeros(N, device=DEV)
    h = torch.empty(M, N, dtype=torch.float16, device=DEV)
    cnt = torch.zeros(M // 32 + 2, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    launches = lib.jimm_launch_count()
    rc = gemm_ex(lib, A, B, x, residual=x, ln=(sc, lb, 1e-5, h, F16, cnt))
    assert rc == -1 and b"does not take the fused LayerNorm path" in lib.jimm_last_error(), rc
    torch.cuda.synchronize()
    assert lib.jimm_launch_count() == launches
    assert torch.equal(x, x0)
