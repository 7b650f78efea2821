"""fp64 references of the attention kernels and per-element bounds on their error, derived from each kernel's own steps.

Everything is computed from the operands the kernel read (the fp16 / bf16 qkv, widened to fp64; the MAP head's fp32 probe), per
(sample x head) row r and key j, with c* = log2(e) / sqrt(d) the exact scale and c = _scale_log2(d) the kernel's fp32 one:
    s_j = q.k_j,  a_j = sum_i |q_i k_ij|,  m = max_j s_j,  t_j = (s_j - m) c*,  P_j = 2^t_j / sum 2^t,  o = sum_j P_j v_j,
    w = sum_j P_j |v_j|.
The bounds take the form
    |P^_j - P_j| <= rho_j P_j + floor                                   (probabilities)
    |o^ - o|     <= sum_j rho'_j P_j |v_j| + rel |o| + floor terms      (outputs; (P rho') @ |v| per element)
No other absolute term is allowed: a probability of 1e-30 is checked to its relative bound.

How rho_j is built (probs_bound).  Each key's contribution reaches the kernel's result as 2^(x_j) times multiplicative roundings, and
every rounding is written as an exponent error E_j (log2 units, E_j >= |x_j - t_j - shift|, the shift common to the row).  A relative
rounding r becomes -log2(1 - r).  Then P^_j = 2^(t_j + e_j) / sum_k P_k 2^(e_k) (|e_k| <= E_k) lies within
    2^(-E_j) / sum_k P_k 2^(E_k)  ..  2^(E_j) / sum_k P_k 2^(-E_k)
of P_j, which gives rho_j exactly (no first-order step).  Errors shared by every key of a row (the row maximum's own score error, which
the kernel subtracts from every key alike) cancel there and are not counted.

Terms of E_j for the wgmma kernels (attention_kernel and attn_probs_kernel share score_tile and softmax_step):
- scores: |s^_j - s_j| <= c_qk a_j (score_tile's wgmma; c_qk measured by test_score_accumulation_constant), times c.
- scale: |c - c*| |s_j - m|.
- the fp32 exponent fl(s^_j c) - fl(m c) (one fma or a product and a difference), and the fp32 product m c itself:
  u (|s_j c| + 2 M c + |t_j|), with M the largest |s| of the row (every running maximum the kernel uses is one of the scores).  This is
  the term a large common offset exercises.
- exp2f: 2 ulp (CUDA C Programming Guide, table of single-precision maths functions, exp2f: 2 ulp; the build has no -ftz, so it keeps
  subnormal results), 4u relative.
- alpha = exp2f(fl(fl(m_old - m_new) c)), once per key tile after the key's own: the exponent's two roundings add at most
  2u (m_new - m_old) c per rescale, and the maxima only rise, so their sum over the later tiles is at most 2u |t_j|; each rescale also
  brings exp2f's 4u and the multiply's u, (T - 1) of them for T key tiles.
Row terms (rel_row, the same for every key of the row): the row sum l, 16 fp32 additions per thread per 64-key tile in softmax_step,
one alpha multiply per tile and the two quad shuffles of row_inv_sum: all terms positive, so gamma_n l with n = 17 T + 2; 1 / l one
rounding (u); attn_probs_kernel's p * (1 / l) one more (u).  Floor: exp2f's 2 ulp of a subnormal result and the product's rounding into
the subnormals, 4 x 2^-149.

The flash kernel's output (flash_ref_bound) adds, per key: P rounded to the operand type for the P.V MMA, u_op = 2^-11 (fp16) or 2^-8
(bf16) relative, or, where p is below the operand type's normal range, an absolute min(eta_op, p) (eta_op = 2^-25 for fp16's subnormal
step, 2^-134 for bf16; in P units eta_op / l, l >= 1); the P.V accumulation c_pv = c_qk + 9 u T (four chained k16 wgmmas per key
tile, each adding into the fp32 accumulator with one truncation, 2u, and the alpha rescale of o, u per tile), on sum_j P^_j |v_j|.
Row terms: l as above, 1 / l and o * (1 / l) (2u), then the output type's rounding u_out |o| + eta_out (bounds_util.OUT).

The MAP head (map_attention_kernel, SIMT, natural-log units, q the fp32 probe) is bounded by map_ref_bound:
- scores: sq_i = fl(q_i qscale), qscale = fl(1 / sqrt(d)); s^ = an fmaf chain of d terms: (gamma_d + u) qscale a_j, plus
  |qscale - 1 / sqrt(d)| a_j.
- x_j = fl(s^_j - bmax): u |x_j|; __expf(x): 2 + floor(1.17 |x|) ulp (the same table's __expf entry), (4 + 2.34 |x|) u relative, and
  results below 2^-126 are flushed to zero (ex2.approx.ftz): floor 2^-126 (+ 2^-149 for p / bsum's rounding).
- bsum: a strided per-thread chain of ceil(S / 256) terms, a 5-level warp tree and a sum of 8 partials: gamma_n, n = ceil(S/256) + 13;
  the probabilities p / bsum one rounding.
- output: a per-warp fmaf chain over ceil(S / 8) keys and a sum of 8 partials, gamma_(ceil(S/8) + 8) on sum_j P^_j |v_j|; v / bsum (u);
  the output rounding; the flushed keys add min(2^-126, P_j) |v_j|.

emulate_probs / emulate_flash follow the kernels' step order in fp32 on the CPU (64-key tiles, online m and l with the quad's four
partial sums, the fp32 s c - m c, P rounded to the operand type before P.V, the fp32 accumulator).  They do not claim the kernels'
bits; they exist to test the bounds, and their mutants to show what the bounds catch.
"""

import math

import torch

from attn_oracle import _scale_log2
from bounds_util import OUT, U

LOG2E = 1.0 / math.log(2.0)
KT = 64  # keys per tile of the wgmma kernels
# operand type: (unit roundoff, half the smallest subnormal step)
OP = {torch.float16: (2.0 ** -11, 2.0 ** -25), torch.bfloat16: (2.0 ** -8, 2.0 ** -134)}
# Score accumulation constant of score_tile, max |s^ - s| / a per score.  test_score_accumulation_constant measured, on an H100 80GB
# HBM3 (700 W power limit) over d = 8 .. 128, on scores whose partial sums reach a / 2 before cancelling: fp16 9.9e-8, bf16 4.1e-8.
# Both operand types give exact products to the same fp32 accumulator, so one constant serves both: 4e-7, about 4x the larger value.
# The offset family (one dominant product and d - 1 small ones) reaches 0.63 of it in fp16, i.e. about 2.5e-7: the cancelling rows
# are not the accumulator's worst case.  Not the GEMM's C_ACC: K here is d <= 128 and the instruction is m64n64k16.
C_QK = {torch.float16: 4e-7, torch.bfloat16: 4e-7}
FLOOR_WGMMA = 4 * 2.0 ** -149
FLOOR_MAP = 2.0 ** -126 + 2.0 ** -149


def padded_head_dim(d):
    """attention.cu's padded width: d runs at the smallest of 16, 32, 64, 80, 96, 128 that holds it."""
    return next(w for w in (16, 32, 64, 80, 96, 128) if d <= w)


def gamma(n):
    return n * U / (1 - n * U)


def _log2_rel(r):
    """A relative rounding r as an exponent error: 2^(-E) <= 1 - r and 1 + r <= 2^E."""
    return -torch.log2(1.0 - torch.as_tensor(r, dtype=torch.float64)) if torch.is_tensor(r) else -math.log2(1.0 - r)


def split_qkv(qkv, B, S, H, d):
    """The fused [B * S, 3 H d] buffer as q, k, v [B * H, S, d] in fp64."""
    q, k, v = qkv.double().reshape(B, S, 3, H, d).permute(2, 0, 3, 1, 4)
    return q.reshape(B * H, S, d), k.reshape(B * H, S, d), v.reshape(B * H, S, d)


def _scores(q, k, causal):
    s = q @ k.transpose(-1, -2)
    a = q.abs() @ k.abs().transpose(-1, -2)
    valid = torch.ones_like(s, dtype=torch.bool)
    if causal:
        valid = torch.tril(valid)
    return s.masked_fill(~valid, float("-inf")), a.masked_fill(~valid, 0.0), valid


def _rho(P, E, valid):
    """Relative bound of P^_j from the exponent errors E (module docstring): the larger side of 2^(+-E_j) / sum_k P_k 2^(-+E_k)."""
    E = torch.where(valid, E, torch.zeros_like(E))
    hi = torch.exp2(E) / (P * torch.exp2(-E)).sum(-1, keepdim=True)
    lo = torch.exp2(-E) / (P * torch.exp2(E)).sum(-1, keepdim=True)
    return torch.maximum(hi - 1.0, 1.0 - lo)


def probs_bound(q, k, causal, c_qk):
    """The wgmma kernels' softmax: (P, rho, l, rel_row, T).  P [N, S, S] fp64 (0 on masked keys); rho the per-key relative bound before
    the row terms rel_row (l's sum and reciprocal: attention_kernel and attn_probs_kernel both have them); l = sum_j 2^t_j (>= 1); T key
    tiles."""
    S, d = q.shape[-2], q.shape[-1]
    T = (S + KT - 1) // KT
    c, cs = _scale_log2(d), LOG2E / math.sqrt(d)
    s, a, valid = _scores(q, k, causal)
    m = s.amax(-1, keepdim=True)
    t = (s - m) * cs
    p = torch.exp2(t)
    l = p.sum(-1, keepdim=True)
    P = p / l
    sv = torch.where(valid, s, torch.zeros_like(s))
    tv = torch.where(valid, t, torch.zeros_like(t))
    Mc = (sv.abs().amax(-1, keepdim=True) + c_qk * a.amax(-1, keepdim=True)) * c
    E = (c * c_qk * a + abs(c - cs) * tv.abs() / cs
         + U * (sv.abs() * c + 2 * Mc + tv.abs()) + 2 * U * tv.abs()
         + _log2_rel(4 * U) + (T - 1) * _log2_rel(5 * U))
    rho = _rho(P, E, valid)
    rel_row = gamma(17 * T + 2) + U
    return P, rho, l, rel_row, T


def probs_ref_bound(q, k, causal, c_qk):
    """attn_probs_kernel with fp32 output: (P, bound) [N, S, S]."""
    P, rho, _, rel_row, _ = probs_bound(q, k, causal, c_qk)
    rel = (1 + rho) * (1 + rel_row) * (1 + U) - 1  # rel_row: l and 1 / l; U: p * (1 / l)
    return P, rel * P + FLOOR_WGMMA


def flash_ref_bound(q, k, v, causal, c_qk, io, out_t):
    """attention_kernel with output type out_t: (o, bound) [N, S, d]."""
    P, rho, l, rel_row, T = probs_bound(q, k, causal, c_qk)
    u_op, eta_op = OP[io]
    c_pv = c_qk + 9 * U * T
    av = v.abs()
    o = P @ v
    Pr = (1 + rho) * P  # upper bound on P^
    A = (rho * P + u_op * Pr + c_pv * (1 + u_op) * Pr) @ av + torch.minimum(eta_op / l, Pr) @ av
    _, _, u_out, eta_out = OUT[out_t]
    rel = (1 + rel_row) * (1 + U) - 1  # l, 1 / l; U: o * (1 / l)
    err = A + rel * (o.abs() + A)
    return o, err + u_out * (o.abs() + err) + eta_out


def map_ref_bound(q, k, v, io, out_t):
    """map_attention_kernel: q [H, d] the fp32 probe, k and v [N = B H, S, d] (head n % H uses q[n % H]): (P [N, S], bound, o [N, d],
    bound)."""
    N, S, d = k.shape
    H = q.shape[0]
    qd = q.double().repeat(N // H, 1)[:, None, :]  # [N, 1, d]
    s = (qd * k).sum(-1) / math.sqrt(d)
    a = (qd.abs() * k.abs()).sum(-1)
    qscale = float(torch.tensor(1.0 / math.sqrt(d), dtype=torch.float32))
    m = s.amax(-1, keepdim=True)
    x = s - m
    p = torch.exp(x)
    P = p / p.sum(-1, keepdim=True)
    ds = (gamma(d) + U) * qscale * a + abs(qscale - 1.0 / math.sqrt(d)) * a
    E = LOG2E * (ds + U * x.abs()) + _log2_rel((4 + 2.34 * x.abs()) * U)
    rho = _rho(P, E, torch.ones_like(P, dtype=torch.bool))
    rel_sum = gamma((S + 255) // 256 + 13)
    p_bound = ((1 + rho) * (1 + rel_sum) * (1 + U) - 1) * P + FLOOR_MAP
    Pr = (1 + rho) * P
    av = v.abs()
    o = (P[:, None, :] @ v)[:, 0]
    A = ((rho * P + gamma((S + 7) // 8 + 8) * Pr)[:, None, :] @ av)[:, 0] + (torch.minimum(torch.full_like(P, FLOOR_MAP), Pr)[:, None, :] @ av)[:, 0]
    rel = (1 + rel_sum) * (1 + U) - 1
    err = A + rel * (o.abs() + A)
    _, _, u_out, eta_out = OUT[out_t]
    return P, p_bound, o, err + u_out * (o.abs() + err) + eta_out


# ---------------------------------------------------------------------------------------------------------------- fp32 emulations (CPU)
def _f32(x):
    return torch.tensor(x, dtype=torch.float32)


def _tiles(q, k, causal, c):
    """The masked fp32 score tiles [N, S, 64] (keys past S at -inf), each score rounded once from fp64 as the MMA's fp32 result."""
    s = (q @ k.transpose(-1, -2)).float()
    S = s.shape[-1]
    if causal:
        s = s.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool)), float("-inf"))
    T = (S + KT - 1) // KT
    s = torch.nn.functional.pad(s, (0, T * KT - S), value=float("-inf"))
    return [s[..., j * KT:(j + 1) * KT] for j in range(T)]


def _softmax_step(s, m_run, l_run, c, rescale_l=True):
    """softmax_step in fp32: s [N, S, 64] -> p; m_run [N, S]; l_run [N, S, 4] (the quad's partial sums: thread t4 holds keys
    8 nt + 2 t4 + {0, 1}).  Returns (p, alpha)."""
    mnew = torch.maximum(m_run, s.amax(-1))
    muse = torch.where(mnew == float("-inf"), torch.zeros_like(mnew), mnew)
    alpha = torch.exp2((m_run - muse) * c)
    moff = muse * c
    if rescale_l:
        l_run = l_run * alpha[..., None]
    p = torch.exp2(s * c - moff[..., None])
    pq = p.reshape(*p.shape[:-1], 8, 4, 2)
    for nt in range(8):
        l_run = l_run + (pq[..., nt, :, 0] + pq[..., nt, :, 1])
    return p, alpha, mnew, l_run


def _inv_sum(l_run):
    return 1.0 / ((l_run[..., 0] + l_run[..., 1]) + (l_run[..., 2] + l_run[..., 3]))


def emulate_probs(q, k, causal, mutant=None):
    """attn_probs_kernel in fp32: P^ [N, S, S].  mutant: None, "flush" (p < 2^-20 -> 0), "scale" (every p x (1 + 2^-14)), "dp_scale"
    (scale_log2 of the padded width), "no_alpha_l" (l not rescaled on the second tile)."""
    d = q.shape[-1]
    c = _f32(_scale_log2(padded_head_dim(d) if mutant == "dp_scale" else d))
    tiles = _tiles(q, k, causal, c)
    N, S = q.shape[0], q.shape[1]
    m_run = torch.full((N, S), float("-inf"))
    l_run = torch.zeros(N, S, 4)
    for j, s in enumerate(tiles):
        _, _, m_run, l_run = _softmax_step(s, m_run, l_run, c, rescale_l=not (mutant == "no_alpha_l" and j == 1))
    inv = _inv_sum(l_run)
    moff = torch.where(m_run == float("-inf"), torch.zeros_like(m_run), m_run) * c
    p = torch.cat([torch.exp2(s * c - moff[..., None]) * inv[..., None] for s in tiles], -1)[..., :S]
    if mutant == "flush":
        p = torch.where(p < 2.0 ** -20, torch.zeros_like(p), p)
    if mutant == "scale":
        p = p * _f32(1 + 2.0 ** -14)
    return p


def emulate_flash(q, k, v, causal, io, mutant=None, col=0):
    """attention_kernel in fp32 with fp32 output: o^ [N, S, d].  P is rounded to io before P.V, each tile's P.V is added to the fp32
    accumulator with one rounding.  mutant: None, "column" (output column `col` x (1 + 2^-10)), "dp_scale", "no_alpha_l"."""
    d = q.shape[-1]
    c = _f32(_scale_log2(padded_head_dim(d) if mutant == "dp_scale" else d))
    tiles = _tiles(q, k, causal, c)
    N, S = q.shape[0], q.shape[1]
    vp = torch.nn.functional.pad(v, (0, 0, 0, len(tiles) * KT - S))
    m_run = torch.full((N, S), float("-inf"))
    l_run = torch.zeros(N, S, 4)
    o = torch.zeros(N, S, d)
    for j, s in enumerate(tiles):
        p, alpha, m_run, l_run = _softmax_step(s, m_run, l_run, c, rescale_l=not (mutant == "no_alpha_l" and j == 1))
        o = o * alpha[..., None]
        o = (o.double() + p.to(io).double() @ vp[:, j * KT:(j + 1) * KT]).float()
    o = o * _inv_sum(l_run)[..., None]
    if mutant == "column":
        o[..., col] = o[..., col] * _f32(1 + 2.0 ** -10)
    return o


# ---------------------------------------------------------------------------------------------------------------- input families
FAMILIES = ["mild", "flat", "sink", "offset", "late", "colscale", "big"]


def make_qkv(family, B, S, H, d, io, seed):
    """The fused qkv [B * S, 3 H d] of one input family, in io (CPU; values representable in io by construction: the cast is exact
    or rounds to what the kernel reads, and the references use the rounded values).
    - mild: randn x 1.5.
    - flat: even heads q = 0, odd heads every key equal: P = 1 / S.
    - sink: one key per row 30, 60, 90 or 120 logits ((head + sample) % 4) above the rest: key 0 in even samples, key S - 1 (the
      ragged last tile) in odd ones; the other probabilities lie in about 1e-12 .. 1e-53, across fp32's subnormals and below 2^-149.
    - offset: every score of a row about K_r +- 3 with |K_r c| up to 400 (q and k share a large first component).
    - late: the scores rise along the key axis, so the row maximum rises at every key tile.
    - colscale: v's columns scaled by 2^-12 .. 2^12; keys in identical pairs, with even columns of v opposite within a pair, so those
      outputs cancel to about 0 while sum P |v| stays large.
    - big (bf16 only): q beyond fp16's range and k below it (x 2^24 / x 2^-24, odd heads x 2^20 / x 2^-16)."""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, S, H, d, generator=g) for _ in range(3))
    q, k = q * 1.5, k * 1.5
    rd = math.sqrt(d)
    c = _scale_log2(d)
    if family == "flat":
        q[:, :, 0::2] = 0.0
        k[:, :, 1::2] = k[:, :1, 1::2]
    elif family == "sink":
        q0 = torch.randn(H, d, generator=g)
        q = q0 + 0.1 * torch.randn(B, S, H, d, generator=g)
        k = 0.5 * k / 1.5
        for h in range(H):
            for b in range(B):
                delta = (30.0, 60.0, 90.0, 120.0)[(h + b) % 4]
                k[b, 0 if b % 2 == 0 else S - 1, h] = q0[h] * (delta * rd / float(q0[h] @ q0[h]))
    elif family == "offset":
        off = math.sqrt(400.0 / c)
        q, k = q / 3, k / 3
        q[..., 0] = off * (2 * torch.rand(B, S, H, generator=g) - 1)
        k[..., 0] = off
    elif family == "late":
        u = torch.nn.functional.normalize(torch.randn(H, d, generator=g), dim=-1)
        rise = torch.minimum(torch.arange(S) * (3.0 / KT), torch.arange(S) * (40.0 / max(S, 1)))  # logits
        q = q * 0.2 + u * 8.0
        k = k * 0.2 + u * (rise * rd / 8.0).reshape(1, S, 1, 1)
    elif family == "colscale":
        k[:, 1::2] = k[:, 0:(S // 2) * 2:2]
        scale = torch.exp2(torch.round(torch.linspace(-12.0, 12.0, d)))
        v = v * scale
        v[:, 1::2, :, 0::2] = -v[:, 0:(S // 2) * 2:2, :, 0::2]
    elif family == "big":
        assert io == torch.bfloat16
        q[:, :, 0::2] *= 2.0 ** 24
        k[:, :, 0::2] *= 2.0 ** -24
        q[:, :, 1::2] *= 2.0 ** 20
        k[:, :, 1::2] *= 2.0 ** -16
    else:
        assert family == "mild", family
    return torch.stack([q, k, v], dim=2).reshape(B * S, 3 * H * d).to(io)
