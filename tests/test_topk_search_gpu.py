"""GPU tests of top-k selection and gallery search, bit for bit.

  * postprocess.top_k against the order prefix of the numpy oracle and of zero_shot on the GPU, at widths from 1 column to 2^20
    (one CTA per row up to 32768 columns, segments and a merge beyond), with the value patterns of the wide zero_shot tests (ties,
    signed zeros, NaN / inf, all-NaN rows), every k from 1 through the select's largest (1024) and past it (the full sort's
    prefix); values and probabilities against the gathered logits and zero_shot's probabilities as int32 bit patterns.
  * CLIP.search / SigLIP.search against top_k of the matrix the jimm_k_l2_normalize + jimm_k_logits test hooks compute from the
    same embeddings with the model's logit_scale / logit_bias, and through the public calls (model(x, t) and its transpose), at
    gallery sizes up to 2^23 rows, whose [8192, 2^23] score matrix (256 GiB) does not fit on the device."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import preprocess_oracle as P
from test_postprocess_wide_gpu import PATTERNS, _row

pytestmark = pytest.mark.gpu

WIDTHS = [1, 63, 64, 4095, 4096, 4097, 21843, 25000, 65537, 2**20]
KS = [1, 5, 100, 1024, 1025]
LOG_SCALE, BIAS = math.log(100.0), -10.0


def _bits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _launches():
    from jimm_b200 import _lib

    return _lib.load().jimm_launch_count()


def _check_topk(xd, ref_order, ks, what):
    """top_k of the CUDA logits xd at each k against ref_order's prefix (numpy) and zero_shot on the GPU."""
    from jimm_b200.postprocess import top_k, zero_shot

    zp, zo = zero_shot(xd)
    x32 = xd.to(torch.float32)
    if x32.ndim == 1:
        x32 = x32[None]
    for k in sorted({min(k, x32.shape[1]) for k in ks}):
        v, i, p = top_k(xd, k, probs=True)
        assert v.dtype == torch.float32 and i.dtype == torch.int32 and tuple(i.shape) == (x32.shape[0], k), what
        ic = i.cpu()
        if ref_order is not None:
            o = ref_order[:, :k]
            bad = np.nonzero((ic.numpy() != o).any(axis=1))[0]
            assert bad.size == 0, f"{what} k={k}: indices differ from the oracle in rows {bad[:8].tolist()}"
        assert torch.equal(ic, zo[:, :k].cpu()), f"{what} k={k}: indices differ from zero_shot's order"
        assert _bits(v, x32.gather(1, i.long())), f"{what} k={k}: values are not the logits at the indices"
        assert _bits(p, zp.gather(1, i.long())), f"{what} k={k}: probs are not zero_shot's at the indices"
        v2, i2 = top_k(xd, k)
        assert _bits(v2, v) and torch.equal(i2, i), f"{what} k={k}: probs=False changes the selection"


@pytest.mark.parametrize("cols", WIDTHS)
def test_top_k_widths_and_patterns(cols):
    x = np.stack([_row(p, cols, np.random.default_rng(1000 + r)) for r, p in enumerate(PATTERNS)])
    _, ref = P.zero_shot_oracle(x)
    _check_topk(torch.from_numpy(x).cuda(), ref, KS + [cols], f"cols={cols}")


@pytest.mark.parametrize("rows,cols", [(1, 21843), (3, 4097), (3, 65537), (256, 21843), (256, 4095)])
def test_top_k_rows(rows, cols):
    rng = np.random.default_rng(rows * 7 + cols)
    x = np.stack([_row(PATTERNS[r % len(PATTERNS)], cols, rng) for r in range(rows)])
    _, ref = P.zero_shot_oracle(x)
    _check_topk(torch.from_numpy(x).cuda(), ref, [1, 5, 100, 1024, 1025], f"rows={rows} cols={cols}")


def test_top_k_5000_captions():
    """[5000, 25000]: every row against zero_shot on the GPU, 16 sampled rows against the numpy oracle."""
    g = torch.Generator(device="cuda").manual_seed(5)
    xd = torch.randn(5000, 25000, device="cuda", generator=g) * 4
    xd[1::7] = torch.round(xd[1::7])  # rows full of ties
    sample = torch.linspace(0, 4999, 16).long()
    _, ref = P.zero_shot_oracle(xd[sample].cpu().numpy())
    from jimm_b200.postprocess import top_k

    _check_topk(xd, None, [5, 100], "5000x25000")
    for k in (5, 100, 1024):
        _, i = top_k(xd, k)
        assert np.array_equal(i[sample].cpu().numpy(), ref[:, :k]), f"k={k}: sampled rows differ from the oracle"


def test_top_k_input_forms():
    """A column-slice view, an expanded row, a 1-D row and fp16 logits: top_k reads what zero_shot reads."""
    rng = np.random.default_rng(3)
    base = torch.from_numpy(np.stack([_row(p, 30000, rng) for p in PATTERNS])).cuda()
    view = base[:, 7:7 + 25000]
    _check_topk(view, P.zero_shot_oracle(view.cpu().numpy())[1], [1, 5, 100, 1024, 1025], "column slice")
    exp = base[2:3, :4097].expand(5, 4097)
    _check_topk(exp, P.zero_shot_oracle(exp.cpu().numpy())[1], [1, 100, 4097], "expanded row")
    row = base[0, :21843]
    _check_topk(row, P.zero_shot_oracle(row[None].cpu().numpy())[1], [5, 1024], "1-D row")
    h = (torch.randn(4, 65537, device="cuda") * 3).half()
    _check_topk(h, P.zero_shot_oracle(h.float().cpu().numpy())[1], [1, 5, 1024, 1025], "fp16")


def test_top_k_refusals_launch_nothing():
    from jimm_b200.postprocess import top_k

    x = torch.randn(3, 50, device="cuda")
    n = _launches()
    for k in (0, 51, -1, True, 2.0):
        with pytest.raises(ValueError):
            top_k(x, k)
    with pytest.raises(Exception):
        top_k(x.cpu(), 5)
    assert _launches() == n, "a refused call launched a kernel"


# ---- search ----
def _model(kind, E):
    """A 1-layer fp16 CLIP / SigLIP at random init with both towers E wide (SigLIP's image embedding is its vision width), logit_scale
    = log 100 and, for SigLIP, logit_bias = -10."""
    from jimm_b200.models import CLIP, SigLIP

    m = (CLIP if kind == "clip" else SigLIP)(32, 1, E, 16, 8, 64, E, E // 64, 1, dtype=torch.float16)
    m.set_flat_param("logit_scale", torch.tensor(LOG_SCALE))
    if kind == "siglip":
        m.set_flat_param("logit_bias", torch.tensor(BIAS))
    return m


_MODELS = {}


def _get(kind, E):
    if (kind, E) not in _MODELS:
        _MODELS[(kind, E)] = _model(kind, E)
    return _MODELS[(kind, E)]


def _hook_logits(m, q, g):
    """The score matrix from the test hooks: l2_normalize both sides, then the logits kernel with the model's scale and bias."""
    from jimm_b200 import _lib

    lib = _lib.load()
    E = q.shape[1]
    qn, gn = torch.empty_like(q), torch.empty_like(g)
    out = torch.empty((q.shape[0], g.shape[0]), dtype=torch.float32, device="cuda")
    scale = m.logit_scale.float().reshape(1).cuda()
    bias = m.logit_bias.float().reshape(1).cuda() if "logit_bias" in m._params else None
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    _lib.check(lib.jimm_k_l2_normalize(p(q), p(qn), E, q.shape[0], E, st))
    _lib.check(lib.jimm_k_l2_normalize(p(g), p(gn), E, g.shape[0], E, st))
    _lib.check(lib.jimm_k_logits(p(qn), p(gn), p(scale), p(bias), p(out), q.shape[0], g.shape[0], E, g.shape[0], st))
    return out


def _emb(n, E, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, E, device="cuda", generator=g)


def _gallery_with_specials(N, E, seed):
    """N rows with duplicated rows (exact ties), a NaN row, an inf row and an all-zero row (NaN scores) where N allows."""
    x = _emb(N, E, seed)
    if N >= 8:
        x[N // 2] = x[1]
        x[N - 1] = x[0]
        x[3, 5] = float("nan")
        x[4, 0] = float("inf")
        x[5] = 0.0
    return x


SEARCH_SHAPES = [(1, 1), (7, 63), (64, 64), (65, 65), (1000, 4097), (64, 25000), (7, 2**20), (65, 2**20), (1000, 25000)]


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.parametrize("Q,N", SEARCH_SHAPES)
def test_search_matches_hook_logits(kind, Q, N):
    from jimm_b200.postprocess import top_k

    E = 64
    m = _get(kind, E)
    g = _gallery_with_specials(N, E, seed=Q + N)
    q = _emb(Q, E, seed=7 * Q + N) * 3.0
    q[0] = g[N // 2]  # a query equal to a gallery row (and, for N >= 8, to its duplicate)
    if Q >= 4:
        q[2] = float("nan")
        q[3] = 0.0
    logits = _hook_logits(m, q, g)
    for k in sorted({min(k, N) for k in (1, 5, 100, 1024)}):
        v, i = m.search(q, g, k)
        rv, ri = top_k(logits, k)
        assert torch.equal(i, ri), f"{kind} Q={Q} N={N} k={k}: indices differ from top_k of the hook logits"
        assert _bits(v, rv), f"{kind} Q={Q} N={N} k={k}: scores differ from the hook logits"


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_search_through_public_calls(kind):
    """search(encode_image(x), encode_text(t)) == top_k(model(x, t)); the other way round == top_k(model(x, t).T); host inputs and
    16-bit embeddings give the bits of their fp32 device form."""
    from jimm_b200.postprocess import top_k

    m = _get(kind, 256)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(6, 32, 32, 3, generator=g).cuda()
    t = torch.randint(0, 64, (40, 8), generator=g, dtype=torch.int32).cuda()
    logits = m(x, t)
    ie, te = m.encode_image(x), m.encode_text(t)
    for k in (1, 5, 40):
        v, i = m.search(ie, te, k)
        rv, ri = top_k(logits, k)
        assert torch.equal(i, ri) and _bits(v, rv), f"{kind} k={k}: image -> text search differs from top_k(model(x, t))"
    for k in (1, 6):
        v, i = m.search(te, ie, k)
        rv, ri = top_k(logits.T, k)
        assert torch.equal(i, ri) and _bits(v, rv), f"{kind} k={k}: text -> image search differs from top_k(model(x, t).T)"
    v, i = m.search(ie, te, 5)
    hv, hi = m.search(ie.cpu(), te.cpu(), 5)
    assert not hv.is_cuda and torch.equal(hi, i.cpu()) and _bits(hv, v), "host inputs"
    for dt in (torch.float16, torch.bfloat16):
        a, b = ie.to(dt), te.to(dt)
        v16, i16 = m.search(a, b, 5)
        r32 = m.search(a.float(), b.float(), 5)
        assert torch.equal(i16, r32[1]) and _bits(v16, r32[0]), f"{dt} embeddings"


def test_search_concurrent_streams():
    """Two streams searching on one handle at once give the bits of the same searches one after the other."""
    m = _get("siglip", 64)
    jobs = [(_emb(300, 64, 1), _gallery_with_specials(70000, 64, 2), 100), (_emb(129, 64, 3), _gallery_with_specials(40000, 64, 4), 1024)]
    seq = [m.search(q, g, k) for q, g, k in jobs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    cur = torch.cuda.current_stream()
    out = []
    for s, (q, g, k) in zip(streams, jobs):
        s.wait_stream(cur)
        with torch.cuda.stream(s):
            out.append(m.search(q, g, k))
    for s in streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for (v, i), (rv, ri) in zip(out, seq):
        assert torch.equal(i, ri) and _bits(v, rv)


def test_search_refusals_launch_nothing():
    from jimm_b200 import _lib

    m = _get("clip", 64)
    q, g = _emb(4, 64, 1), _emb(2000, 64, 2)
    m.search(q, g, 1)  # the handle exists before counting
    n = _launches()
    for args in [(q, g, 0), (q, g[:5], 6), (q, g, 1025), (q[:, :63], g, 5), (q, g[:, :32], 5), (q, g, True)]:
        with pytest.raises(ValueError):
            m.search(*args)
    nat = m.native()
    vals = torch.empty((4, 8), device="cuda")
    idx = torch.empty((4, 8), dtype=torch.int32, device="cuda")
    for N, k in [(2000, 0), (5, 6), (2000, 1025)]:
        rc = nat.lib.jimm_search(nat.handle, C.c_void_p(q.data_ptr()), 4, C.c_void_p(g.data_ptr()), N, k, C.c_void_p(vals.data_ptr()),
                                 C.c_void_p(idx.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -1, (N, k, rc)  # JIMM_EINVAL
    assert _launches() == n, "a refused call launched a kernel"


def test_search_gallery_past_device_memory():
    """Q = 8192 queries against N = 2^23 gallery rows at E = 256: 8 GiB of gallery and a 256 GiB score matrix, which no device holds.
    16 sampled queries against top_k of their [16, N] hook logits."""
    from jimm_b200.postprocess import top_k

    m = _get("siglip", 256)
    Q, N, E, k = 8192, 2**23, 256, 10
    g = torch.empty((N, E), device="cuda")
    for c in range(0, N, 2**20):  # generated in slices: randn's own temporaries stay small
        g[c:c + 2**20] = _emb(2**20, E, seed=100 + c // 2**20)
    g[N - 1] = g[12345]
    q = _emb(Q, E, seed=9)
    q[17] = g[12345]
    v, i = m.search(q, g, k)
    torch.cuda.synchronize()
    rows = torch.cat([torch.tensor([17]), torch.linspace(0, Q - 1, 15).long()])
    rv, ri = top_k(_hook_logits(m, q[rows.cuda()], g), k)
    assert torch.equal(i[rows.cuda()], ri) and _bits(v[rows.cuda()], rv)
    assert set(i[17, :2].tolist()) == {12345, N - 1} and i[17, 0].item() == N - 1, "the exact tie comes out larger index first"
