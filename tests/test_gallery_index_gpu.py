"""GPU tests of the gallery index (model.index / jimm_index_*), bit for bit against model.search.

  * Identity: index.search(q, k) against model.search(q, gallery, k) -- scores as int32 bit patterns, indices equal -- for CLIP and
    SigLIP (bias -10) at E = 256, 512, 768 and 1152, at N from k to 2^20 + 3 rows (the seed block alone, one row past it, many screened
    chunks), Q across the 2048-query chunk edge and k from 1 to 1024; fp16 / bf16 and host inputs; both directions through the public
    calls; an index built by several adds against the concatenated gallery.
  * Bound-hostile galleries through the same identity: clustered embeddings, exact duplicate rows (which must overflow the screen's
    candidate lists and fall back), rows placed 1e-6 .. 1e-3 in cosine around each query's k-th score, zero / NaN / inf rows and
    queries, and rows near fp32 underflow whose normalised norm is not 1.
  * The screen screens: on Gaussian data at 2^20 rows, fewer than 1 % of the rows per query are rescored and nothing falls back.
  * The tensor-core term of the screen's bound: the fp16 wgmma GEMM (jimm_k_gemm, the screen's mainloop) against fp64 on adversarial
    operands, |a - r| <= c_tc sum |q^ g^| with c_tc = E kTcAccumPerK, read from jimm_b200/csrc/gemm.cuh.
  * The index follows its model: after the model rebuilds its native handle (a larger batch, set_flat_param) a search binds to the
    new handle and equals model.search with the current logit_scale; an index of a closed bare handle raises.
  * Refusals raise ValueError (or return JIMM_EINVAL) and launch nothing."""
import ctypes as C
import math
import os
import re

import pytest
import torch

from gpu_util import check, gemm, ptr, stream

pytestmark = pytest.mark.gpu

LOG_SCALE, BIAS = math.log(100.0), -10.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tc_per_k():
    """kTcAccumPerK as jimm_b200/csrc/gemm.cuh defines it: the c_tc / E the screen's bound uses."""
    src = open(os.path.join(ROOT, "jimm_b200", "csrc", "gemm.cuh")).read()
    m = re.search(r"constexpr double kTcAccumPerK = (0x[0-9a-fA-F.]+p[-+]?\d+);", src)
    assert m, "kTcAccumPerK not found in gemm.cuh"
    return float.fromhex(m.group(1))


def _bits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _launches():
    from jimm_b200 import _lib

    return _lib.load().jimm_launch_count()


_MODELS = {}


def _new_model(kind, E, heads=None):
    """A 1-layer fp16 CLIP / SigLIP at random init with both towers E wide (heads of 64 unless given), logit_scale = log 100 and, for
    SigLIP, logit_bias = -10."""
    from jimm_b200.models import CLIP, SigLIP

    h = heads or E // 64
    m = (CLIP if kind == "clip" else SigLIP)(32, 1, E, 16, 8, 64, E, h, 1, dtype=torch.float16, vision_heads=h)
    m.set_flat_param("logit_scale", torch.tensor(LOG_SCALE))
    if kind == "siglip":
        m.set_flat_param("logit_bias", torch.tensor(BIAS))
    return m


def _get(kind, E, heads=None):
    if (kind, E) not in _MODELS:
        _MODELS[(kind, E)] = _new_model(kind, E, heads)
    return _MODELS[(kind, E)]


def _emb(n, E, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, E, device="cuda", generator=g)


def _search_stats(index, q, k):
    """index.search through the C entry point, with its jimm_search_stats."""
    from jimm_b200 import _lib

    index._model()  # bind to the model's current handle, as index.search does
    Q = q.shape[0]
    qd = q.to("cuda", torch.float32).contiguous()
    v = torch.empty((Q, k), device="cuda")
    i = torch.empty((Q, k), dtype=torch.int32, device="cuda")
    st = _lib.SearchStats()
    check(_lib.load(), _lib.load().jimm_index_search(index.handle, ptr(qd), Q, k, ptr(v), ptr(i), C.byref(st), stream()))
    torch.cuda.synchronize()
    return v, i, st


def _same(m, index, q, g, ks, what):
    """index.search == model.search at each k; returns the stats of the last k."""
    st = None
    for k in ks:
        v, i, st = _search_stats(index, q, k)
        rv, ri = m.search(q, g, k)
        bad = (i != ri).any(dim=1).nonzero().flatten()
        assert bad.numel() == 0, f"{what} k={k}: indices differ in queries {bad[:8].tolist()}"
        assert _bits(v, rv), f"{what} k={k}: scores differ"
        pv, pi = index.search(q, k)  # the public call gives the same
        assert torch.equal(pi, i) and _bits(pv, v), f"{what} k={k}: index.search differs from jimm_index_search"
    return st


# ---- identity ----
SMALL = [(1, 1, [1]), (5, 5, [5]), (100, 100, [1, 100]), (1024, 1024, [1024]), (2047, 63, [1, 5, 63]), (2049, 32768, [1, 100, 1024]),
         (3, 32769, [1, 5, 1024]), (5000, 40000, [5, 100])]


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.parametrize("Q,N,ks", SMALL)
def test_identity_small(kind, Q, N, ks):
    E = 256
    m = _get(kind, E)
    g, q = _emb(N, E, seed=N), _emb(Q, E, seed=Q + 1) * 2.0
    st = _same(m, m.index(g), q, g, ks, f"{kind} Q={Q} N={N}")
    if N > 32768:
        assert st.chunks_screened > 0


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.parametrize("E", [256, 512, 768, 1152])
def test_identity_large(kind, E):
    """2^20 + 3 rows: the seed block and 16 screened chunks, the last one 3 rows wide; 2049 queries: two query chunks."""
    m = _get(kind, E)
    N, Q = 2**20 + 3, 2049
    g, q = _emb(N, E, seed=E), _emb(Q, E, seed=E + 1)
    q[7] = g[N - 1]
    st = _same(m, m.index(g), q, g, [1, 100] if E != 768 else [5, 1024], f"{kind} E={E}")
    assert st.chunks_screened == 2 * 16


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_identity_width_not_multiple_of_16(kind):
    """E = 520 (5 heads of 104): the logits kernel's last K step is zero-padded, and the rescorer reproduces it."""
    m = _get(kind, 520, heads=5)
    g, q = _emb(32768 + 70000, 520, seed=52), _emb(700, 520, seed=53)
    g[40000] = 0.0
    q[3] = g[90000]
    st = _same(m, m.index(g), q, g, [1, 7, 100], f"{kind} E=520")
    assert st.chunks_screened > 0 and st.rows_rescored > 0


def test_identity_5000_queries():
    m = _get("siglip", 768)
    N = 2**20 + 3
    g, q = _emb(N, 768, seed=3), _emb(5000, 768, seed=4)
    _same(m, m.index(g), q, g, [100], "5000 x 2^20")


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_both_directions_and_input_forms(kind):
    """index(encode_text(t)).search(encode_image(x)) == top_k(model(x, t)); the other way round == top_k(model(x, t).T); fp16 / bf16 and
    host inputs give model.search's bits, host queries give host results."""
    from jimm_b200.postprocess import top_k

    m = _get(kind, 256)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(6, 32, 32, 3, generator=g).cuda()
    t = torch.randint(0, 64, (40, 8), generator=g, dtype=torch.int32).cuda()
    logits = m(x, t)
    ie, te = m.encode_image(x), m.encode_text(t)
    for k in (1, 5, 40):
        v, i = m.index(te).search(ie, k)
        rv, ri = top_k(logits, k)
        assert torch.equal(i, ri) and _bits(v, rv), f"{kind} k={k}: image -> text differs from top_k(model(x, t))"
    v, i = m.index(ie).search(te, 6)
    rv, ri = top_k(logits.T, 6)
    assert torch.equal(i, ri) and _bits(v, rv), f"{kind}: text -> image differs from top_k(model(x, t).T)"
    # the same through screened chunks: a large gallery of the text side
    G = torch.cat([_emb(70000, 256, seed=5), te])
    v, i = m.index(G).search(ie, 5)
    rv, ri = m.search(ie, G, 5)
    assert torch.equal(i, ri) and _bits(v, rv)
    G16, q16 = G.to(torch.bfloat16), ie.to(torch.float16)
    index = m.index(G16)
    for qq in (q16, q16.cpu(), ie.cpu()):
        v, i = index.search(qq, 5)
        rv, ri = m.search(qq.cuda(), G16, 5)
        assert v.is_cuda == qq.is_cuda and i.is_cuda == qq.is_cuda, "results go to the host exactly when the queries are there"
        assert torch.equal(i.cpu(), ri.cpu()) and _bits(v, rv), f"queries {qq.dtype} on {qq.device}"
    v, i = m.index(G.cpu()).search(ie, 5)
    rv, ri = m.search(ie, G, 5)
    assert torch.equal(i, ri) and _bits(v, rv), "host gallery"


def test_several_adds():
    m = _get("clip", 512)
    parts = [_emb(n, 512, seed=n) for n in (1, 40000, 777, 300000, 5)]
    index = m.index(parts[0])
    for p in parts[1:]:
        index.add(p)
    g = torch.cat(parts)
    assert len(index) == g.shape[0]
    q = _emb(300, 512, seed=9)
    q[0] = parts[3][17]
    _same(m, index, q, g, [1, 50], "adds")


# ---- bound-hostile data ----
def _clustered(centroids, n, noise, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.randint(0, centroids.shape[0], (n,), device="cuda", generator=gen)
    return centroids[lab] + noise * torch.randn(n, centroids.shape[1], device="cuda", generator=gen)


@pytest.mark.parametrize("noise", [0.3, 0.01])
def test_clustered(noise):
    """300 centroids plus noise: each query has thousands of rows within a few 1e-3 of its k-th score."""
    m = _get("siglip", 768)
    c = _emb(300, 768, seed=1)
    g, q = _clustered(c, 2**20, noise, seed=2), _clustered(c, 1000, noise, seed=3)
    _same(m, m.index(g), q, g, [5, 100], f"clustered noise={noise}")


def test_duplicates_fall_back():
    """Every row after the seed block is one of two rows: the screen passes every copy (exact ties, broken by index), the candidate
    lists overflow and those (query, chunk) pairs take the exact block step."""
    m = _get("clip", 256)
    base = _emb(32768, 256, seed=1)
    dup = _emb(2, 256, seed=2)
    g = torch.cat([base, dup[torch.arange(100000, device="cuda") % 2]])
    q = torch.cat([dup, _emb(30, 256, seed=3)])
    st = _same(m, m.index(g), q, g, [1, 100, 1024], "duplicates")
    assert st.fallbacks > 0


def test_rows_around_the_kth_score():
    """Rows whose cosine with a query sits 1e-6 .. 1e-3 above or below that query's k-th cosine, appended after the seed block and
    after a screened chunk."""
    E, k = 768, 10
    m = _get("siglip", E)
    g = _emb(2**17, E, seed=1)
    q = _emb(64, E, seed=2)
    v, _ = m.search(q, g, k)
    cos_k = ((v[:, k - 1].double() - BIAS) / 100.0)
    qn = torch.nn.functional.normalize(q.double(), dim=1)
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(3)
    for d in (1e-6, 3e-6, 1e-5, 1e-4, 1e-3):
        for sgn in (1.0, -1.0):
            c = (cos_k + sgn * d).clamp(-1, 1)[:, None]
            u = torch.randn(q.shape[0], E, device="cuda", generator=gen, dtype=torch.float64)
            u = torch.nn.functional.normalize(u - (u * qn).sum(1, keepdim=True) * qn, dim=1)
            rows.append((c * qn + (1 - c * c).sqrt() * u).float())
    near = torch.cat(rows)
    G = torch.cat([g[:40000], near, g[40000:], near])
    _same(m, m.index(G), q, G, [k, 1, 100], "near the k-th score")


def test_nonfinite_and_zero_rows_and_queries():
    m = _get("siglip", 512)
    g = _emb(100000, 512, seed=1)
    for r in (5, 40000, 99999):
        g[r] = 0.0
    g[50000, 3] = float("nan")
    g[70000, 0] = float("inf")
    g[80000, 1] = -float("inf")
    g[90000] = 1e30  # the sum of squares overflows: the normalised row is all zeros
    q = _emb(40, 512, seed=2)
    q[1] = 0.0
    q[2, 4] = float("nan")
    q[3, 0] = float("inf")
    q[4] = g[60000]
    _same(m, m.index(g), q, g, [1, 5, 100], "non-finite")


@pytest.mark.parametrize("k", [1, 3, 5])
def test_nan_kth_score_still_screens(k):
    """Three zero rows in the seed block score NaN against every query, and NaN ranks first: at k <= 3 the running k-th score is NaN.
    Only rows that can score NaN (non-finite bound) may still enter, so the screen keeps those alone and nothing falls back."""
    m = _get("siglip", 256)
    g = _emb(32768 + 140000, 256, seed=61)
    g[[10, 20000, 30000]] = 0.0
    g[100000] = 0.0  # a later NaN row, which enters ahead of the earlier ones (equal keys, larger index first)
    q = _emb(500, 256, seed=62)
    st = _same(m, m.index(g), q, g, [k], f"NaN k-th k={k}")
    assert st.fallbacks == 0
    if k <= 3:  # the k-th is NaN: each query rescores the one zero row past the seed block and nothing else
        assert st.rows_rescored == 500, st.rows_rescored


def test_rows_near_underflow():
    """Rows whose squares are fp32 subnormals or flush: l2_normalize does not bring them to norm 1."""
    E = 768
    m = _get("clip", E)
    g = _emb(70000, E, seed=1)
    tiny = _emb(4000, E, seed=2)
    g[33000:34000] = tiny[:1000] * 3e-23
    g[40000:41000] = tiny[1000:2000] * 1e-21
    g[50000:51000] = tiny[2000:3000] * 1e-23
    g[50000:51000, :8] = 1e-19
    g[60000:61000] = tiny[3000:4000] * 1e-22
    from jimm_b200 import _lib  # the normalised norms really are off 1

    gn = torch.empty(4000, E, device="cuda")
    src = torch.cat([g[33000:34000], g[40000:41000], g[50000:51000], g[60000:61000]]).contiguous()
    check(_lib.load(), _lib.load().jimm_k_l2_normalize(ptr(src), ptr(gn), E, 4000, E, stream()))
    norms = gn.double().norm(dim=1)
    assert ((norms - 1).abs() > 1e-3).any()
    q = torch.cat([_emb(20, E, seed=3), g[33000:33010], g[50000:50010]])
    _same(m, m.index(g), q, g, [1, 10, 100], "underflow")


# ---- the screen screens ----
@pytest.mark.parametrize("k", [5, 100])
def test_screen_rescores_few_rows(k):
    E, N, Q = 768, 2**20, 2048
    m = _get("clip", E)
    g, q = _emb(N, E, seed=21), _emb(Q, E, seed=22)
    index = m.index(g)
    _, _, st = _search_stats(index, q, k)
    per_query = st.rows_rescored / Q
    print(f"\nGaussian 2^20 x {E}, k={k}: {per_query:.1f} rows rescored per query, {st.fallbacks} fallbacks, {st.chunks_screened} chunks")
    assert st.fallbacks == 0
    assert per_query < 0.01 * N


# ---- the tensor-core term of the bound ----
def _adversarial(E, M, seed):
    """fp16 operand pairs (rows of A, rows of B): cancelling runs, mixed exponents, one dominant product, Gaussian."""
    gen = torch.Generator().manual_seed(seed)
    fam = []
    a = torch.ones(M, E, dtype=torch.float64)
    b = torch.ones(M, E, dtype=torch.float64)
    b[:, E // 2:] = -1.0
    a[:, :E // 2] += torch.rand(M, E // 2, generator=gen, dtype=torch.float64) * 2**-8
    fam.append(("cancel", a, b))
    e = torch.randint(-14, 8, (M, E), generator=gen).double()
    a = torch.randn(M, E, generator=gen, dtype=torch.float64) * torch.pow(2.0, e)
    b = torch.randn(M, E, generator=gen, dtype=torch.float64) * torch.pow(2.0, torch.randint(-14, 8, (M, E), generator=gen).double())
    fam.append(("mixed exponents", a, b))
    a = torch.randn(M, E, generator=gen, dtype=torch.float64) * 2**-6
    b = torch.randn(M, E, generator=gen, dtype=torch.float64) * 2**-6
    a[:, 0], b[:, 0] = 200.0, 200.0
    a[:, 1], b[:, 1] = 200.0, -200.0
    fam.append(("dominant pair", a, b))
    a = torch.randn(M, E, generator=gen, dtype=torch.float64) / math.sqrt(E)
    b = torch.randn(M, E, generator=gen, dtype=torch.float64) / math.sqrt(E)
    fam.append(("gaussian unit", a, b))
    # a partial sum that grows to a large value and then cancels down, under a running sum of small products
    a = torch.randn(M, E, generator=gen, dtype=torch.float64) * 2**-10
    b = torch.randn(M, E, generator=gen, dtype=torch.float64) * 2**-10
    a[:, :16], b[:, :16] = 64.0, 1.0
    a[:, E - 16:], b[:, E - 16:] = 64.0, -1.0
    fam.append(("grow then cancel", a, b))
    return [(n, a.half(), b.half()) for n, a, b in fam]


@pytest.mark.parametrize("E", [256, 520, 768, 1152])
def test_tensor_core_accumulation_term(lib, E):
    worst = 0.0
    c_tc_per_k = _tc_per_k()
    for name, a, b in _adversarial(E, 256, seed=E):
        A, B = a.cuda(), b.cuda()
        out = gemm(lib, A, B, out_dtype=torch.float32, mode=2)
        torch.cuda.synchronize()
        ref = a.double() @ b.double().T  # exact products, fp64 sums
        tot = a.double().abs() @ b.double().abs().T
        err = (out.double().cpu() - ref).abs()
        ratio = (err / (E * c_tc_per_k * tot).clamp_min(1e-300)).max().item()
        worst = max(worst, ratio)
        print(f"\nE={E} {name}: max |a - r| / (c_tc sum |q g|) = {ratio:.3f}")
        assert ratio <= 1.0, f"E={E} {name}: the fp16 wgmma's accumulation exceeds c_tc = E x {c_tc_per_k!r} (ratio {ratio:.3f})"
    print(f"E={E}: largest ratio {worst:.3f}")


# ---- refusals ----
def test_refusals_launch_nothing():
    from jimm_b200 import _lib

    m = _get("clip", 256)
    g, q = _emb(2000, 256, seed=1), _emb(4, 256, seed=2)
    index = m.index(g)
    index.search(q, 1)  # everything exists before counting
    small = m.index(_emb(3, 256, seed=3))
    n = _launches()
    for args in [(q, 0), (q, 2001), (q, 1025), (q, True), (q, 2.0), (q[:, :255], 5), (q.to(torch.float64), 5), (q.to(torch.int32), 5)]:
        with pytest.raises(ValueError):
            index.search(*args)
    for rows in (g[:, :128], g.to(torch.float64), g[0]):
        with pytest.raises(ValueError):
            index.add(rows)
    with pytest.raises(ValueError):
        m.index(g[:, :200])
    with pytest.raises(ValueError):
        small.search(q, 4)
    lib = _lib.load()
    vals = torch.empty((4, 8), device="cuda")
    idx = torch.empty((4, 8), dtype=torch.int32, device="cuda")
    for k in (0, 2001, 1025):
        rc = lib.jimm_index_search(index.handle, ptr(q), 4, k, ptr(vals), ptr(idx), None, stream())
        assert rc == -1, (k, rc)
    assert lib.jimm_index_add(index.handle, ptr(g), -1, stream()) == -1
    assert _launches() == n, "a refused call launched a kernel"
    assert len(index) == 2000


# ---- the index follows its model ----
def test_index_follows_model_rebuilds():
    """A rebuild of the model's native handle -- a call with more samples than its max_batch, set_flat_param of logit_scale -- frees the
    handle the index was built on.  The next search binds to the new handle and gives model.search's bits with the current scale;
    adding rows still works; closing the index after the rebuilds reads no freed handle."""
    m = _new_model("siglip", 256)
    g, q = _emb(32768 + 50000, 256, seed=71), _emb(40, 256, seed=72)
    index = m.index(g)
    _same(m, index, q, g, [5], "before")
    v0, _ = index.search(q, 5)
    n0 = m.native()
    mb = n0.max_batch
    gen = torch.Generator().manual_seed(73)
    x = torch.randn(mb + 1, 32, 32, 3, generator=gen).cuda()
    t = torch.randint(0, 64, (mb + 1, 8), generator=gen, dtype=torch.int32).cuda()
    m(x, t)
    assert m.native() is not n0 and not n0.handle, "the call did not rebuild the handle"
    _same(m, index, q, g, [5, 100], "after a batch rebuild")
    n1 = m.native()
    m.set_flat_param("logit_scale", torch.tensor(math.log(30.0)))
    assert not n1.handle
    _same(m, index, q, g, [5], "after set_flat_param")
    v1, _ = index.search(q, 5)
    assert not torch.equal(v0, v1), "the new logit_scale is not in the scores"
    more = _emb(1000, 256, seed=74)
    index.add(more)
    _same(m, index, q, torch.cat([g, more]), [5], "add after the rebuilds")
    index.close()
    with pytest.raises(Exception):
        index.search(q, 5)


def test_index_of_a_closed_handle_raises():
    from jimm_b200 import _lib

    m = _new_model("clip", 256)
    g, q = _emb(5000, 256, seed=81), _emb(8, 256, seed=82)
    bare = m.native().index(g)  # bound to this handle alone
    rv, ri = m.search(q, g, 5)
    v, i = bare.search(q, 5)
    assert torch.equal(i, ri) and _bits(v, rv)
    m.set_flat_param("logit_scale", torch.tensor(math.log(20.0)))  # frees that handle
    with pytest.raises(_lib.JimmError):
        bare.search(q, 5)
    with pytest.raises(_lib.JimmError):
        bare.add(g[:10])
    bare.close()
