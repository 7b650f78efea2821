"""GPU tests of the gallery index's threshold search (index.range_search / jimm_index_range_search) and near-duplicate pairs
(index.pairs / jimm_index_pairs), bit for bit against the score matrix of the jimm_k_l2_normalize + jimm_k_logits test hooks.

  * Identity: CSR offsets and indices equal, scores equal as int32 bit patterns, for CLIP and SigLIP (bias -10) at E = 256, 768 and
    1152, N from 1 to 2^20 + 3, Q across the 2048-query chunk edge, thresholds giving about 0, 3, 100 and 5000 hits per query (the
    last overflows the screen's lists and takes the exact block step), and the special thresholds: a present score (the tie is a hit),
    +-inf, FLT_MAX, -0.0, +0.0 and the smallest subnormal.
  * Bound-hostile data through the same identity: clustered rows, exact duplicates, zero / NaN / inf rows and queries (a NaN score is
    never a hit), rows near fp32 underflow, and a non-finite or tiny logit_scale (every row is scored exactly).
  * Pairs: the upper triangle of range_search(all rows), directly against the hook matrix, a symmetric full mask; N = 0 and 1 give
    nothing.
  * Agreement with index.search, the screen screening (under 1 % of the rows rescored), offsets past 2^31 hits, the model handle
    followed after rebuilds, input forms, repeatability, and refusals that launch nothing."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gpu_util import ptr, stream

pytestmark = pytest.mark.gpu

LOG_SCALE, BIAS = math.log(100.0), -10.0
FLT_MAX = float(np.finfo(np.float32).max)
TINY = float(np.finfo(np.float32).smallest_subnormal)
_MODELS = {}


def _new_model(kind, E):
    from jimm_b200.models import CLIP, SigLIP

    h = E // 64
    m = (CLIP if kind == "clip" else SigLIP)(32, 1, E, 16, 8, 64, E, h, 1, dtype=torch.float16, vision_heads=h)
    m.set_flat_param("logit_scale", torch.tensor(LOG_SCALE))
    if kind == "siglip":
        m.set_flat_param("logit_bias", torch.tensor(BIAS))
    return m


def _get(kind, E):
    if (kind, E) not in _MODELS:
        _MODELS[(kind, E)] = _new_model(kind, E)
    return _MODELS[(kind, E)]


def _emb(n, E, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, E, device="cuda", generator=g)


def _lib():
    from jimm_b200 import _lib as L

    return L


def _normalised(x):
    L = _lib()
    x = x.to("cuda", torch.float32).contiguous()
    out = torch.empty_like(x)
    for r0 in range(0, x.shape[0], 2**20):
        n = min(2**20, x.shape[0] - r0)
        L.check(L.load().jimm_k_l2_normalize(ptr(x[r0:]), ptr(out[r0:]), x.shape[1], n, x.shape[1], stream()))
    return out


def _hook_rows(m, qn, gn):
    """The hook score matrix of normalised queries qn against normalised rows gn (jimm_k_logits with the model's scale and bias)."""
    L = _lib()
    out = torch.empty((qn.shape[0], gn.shape[0]), dtype=torch.float32, device="cuda")
    scale = m.logit_scale.float().reshape(1).cuda()
    bias = m.logit_bias.float().reshape(1).cuda() if "logit_bias" in m._params else None
    E = qn.shape[1]
    L.check(L.load().jimm_k_logits(ptr(qn), ptr(gn), ptr(scale), ptr(bias), ptr(out), qn.shape[0], gn.shape[0], E, gn.shape[0], stream()))
    return out


def _row_chunks(Q, N):
    step = max(1, min(2048, (1 << 28) // max(N, 1)))
    return [(r0, min(Q, r0 + step)) for r0 in range(0, Q, step)]


def _ref_csr(m, q, g, threshold, upper=False):
    """CSR of hook(q, g) >= fp32(threshold) (upper: only columns j > i), computed in row chunks."""
    t = torch.tensor(threshold, dtype=torch.float32, device="cuda")
    qn, gn = _normalised(q), _normalised(g)
    counts, scores, idx = [], [], []
    for r0, r1 in _row_chunks(q.shape[0], g.shape[0]):
        Lm = _hook_rows(m, qn[r0:r1], gn)
        mask = Lm >= t
        if upper:
            mask &= torch.arange(g.shape[0], device="cuda")[None, :] > torch.arange(r0, r1, device="cuda")[:, None]
        counts.append(mask.sum(1))
        scores.append(Lm[mask])
        idx.append(mask.nonzero()[:, 1].to(torch.int32))
        del Lm, mask
    offsets = torch.zeros(q.shape[0] + 1, dtype=torch.int64, device="cuda")
    if counts:
        offsets[1:] = torch.cat(counts).cumsum(0)
    return offsets, torch.cat(scores) if scores else torch.empty(0, device="cuda"), torch.cat(idx) if idx else torch.empty(0, dtype=torch.int32, device="cuda")


def _thresholds(m, q, g, hits):
    """Thresholds giving about `hits` hits per query, from the hook scores of the first 64 queries (0: their largest score)."""
    s = _hook_rows(m, _normalised(q[:64]), _normalised(g)).flatten()
    s = s[~s.isnan()].sort(descending=True).values
    rows = min(64, q.shape[0])
    return [s[min(max(h * rows - 1, 0), s.numel() - 1)].item() for h in hits]


def _bits_equal(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _assert_csr(got, ref, what):
    go, gs, gi = got
    ro, rs, ri = ref
    go, ro = go.cpu(), ro.cpu()
    if not torch.equal(go, ro):
        bad = (go != ro).nonzero().flatten()
        raise AssertionError(f"{what}: offsets differ first at row {bad[0].item()} ({go[bad[0]].item()} vs {ro[bad[0]].item()})")
    assert torch.equal(gi.cpu(), ri.cpu()), f"{what}: indices differ"
    assert _bits_equal(gs, rs), f"{what}: scores differ"


def _range_stats(index, q, threshold):
    """index.range_search through the C entry points, with its jimm_search_stats."""
    L = _lib()
    lib = L.load()
    index._model()
    qd = q.to("cuda", torch.float32).contiguous()
    h = C.c_void_p()
    st = L.SearchStats()
    L.check(lib.jimm_index_range_search(index.handle, ptr(qd), qd.shape[0], threshold, C.byref(h), C.byref(st), stream()))
    rows, total = C.c_int(), C.c_longlong()
    L.check(lib.jimm_hits_size(h, C.byref(rows), C.byref(total)))
    o = torch.empty(rows.value + 1, dtype=torch.int64, device="cuda")
    s = torch.empty(total.value, device="cuda")
    i = torch.empty(total.value, dtype=torch.int32, device="cuda")
    L.check(lib.jimm_hits_copy(h, ptr(o), ptr(s), ptr(i), stream()))
    L.check(lib.jimm_hits_destroy(h))
    return (o, s, i), st


def _check(m, index, q, g, thresholds, what):
    """range_search == the hook CSR at each threshold (through the C call and the public one); returns the stats of each."""
    stats = []
    for t in thresholds:
        got, st = _range_stats(index, q, t)
        _assert_csr(got, _ref_csr(m, q, g, t), f"{what} t={t!r}")
        pub = index.range_search(q, t)
        assert all(torch.equal(a, b) for a, b in zip(pub, got)), f"{what} t={t!r}: index.range_search differs from the C call"
        stats.append(st)
    return stats


# ---- identity ----
SIZES = [(1, 1), (5, 5), (2047, 1), (1, 65536), (2049, 65536), (2047, 65537), (3, 65537)]


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.parametrize("Q,N", SIZES)
def test_identity_small(kind, Q, N):
    E = 256
    m = _get(kind, E)
    g, q = _emb(N, E, seed=N), _emb(Q, E, seed=Q + 1) * 2.0
    ts = _thresholds(m, q, g, [0, 3, 100, 5000])
    stats = _check(m, m.index(g), q, g, ts, f"{kind} Q={Q} N={N}")
    if N >= 65536:
        assert stats[-1].fallbacks > 0, "5000 hits per query in one chunk must overflow the screen's lists"


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.parametrize("E", [256, 768, 1152])
def test_identity_large(kind, E):
    """2^20 + 3 rows: 17 screened chunks, the last 3 rows wide; 2049 queries: two query chunks.  5000 hits spread over 17 chunks fit
    the screen's lists; 80000 (about 5000 per chunk) overflow them."""
    m = _get(kind, E)
    N, Q = 2**20 + 3, 2049
    g, q = _emb(N, E, seed=E), _emb(Q, E, seed=E + 1)
    q[7] = g[N - 1]
    ts = _thresholds(m, q, g, [0, 3, 100, 5000, 80000])
    stats = _check(m, m.index(g), q, g, ts, f"{kind} E={E}")
    assert all(s.chunks_screened == 2 * 17 for s in stats)
    assert stats[-1].fallbacks > 0


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_special_thresholds(kind):
    """A threshold equal to a present score (the tie is a hit), the infinities, FLT_MAX, both zeros and the smallest subnormal, on
    data with exact zero and NaN scores."""
    E = 256
    m = _get(kind, E)
    g = _emb(70000, E, seed=31)
    g[100:200, 0] = 0.0
    g[300] = 0.0  # NaN scores
    q = _emb(40, E, seed=32)
    q[0] = 0.0
    q[0, 0] = 1.0  # one-hot: exact zero accumulators against rows 100 .. 199, so CLIP scores exact +0
    index = m.index(g)
    L = _hook_rows(m, _normalised(q[:3]), _normalised(g))
    present = L[1, 12345].item()
    _check(m, index, q, g, [present, math.inf, -math.inf, FLT_MAX, -FLT_MAX, -0.0, 0.0, TINY, -TINY], kind)
    o, s, i = index.range_search(q[1:2], present)
    assert (i == 12345).any(), "a score equal to the threshold is a hit"


# ---- bound-hostile data ----
def _clustered(centroids, n, noise, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.randint(0, centroids.shape[0], (n,), device="cuda", generator=gen)
    return centroids[lab] + noise * torch.randn(n, centroids.shape[1], device="cuda", generator=gen)


@pytest.mark.parametrize("noise", [0.3, 0.01])
def test_clustered(noise):
    m = _get("siglip", 768)
    c = _emb(300, 768, seed=1)
    g, q = _clustered(c, 2**18, noise, seed=2), _clustered(c, 500, noise, seed=3)
    _check(m, m.index(g), q, g, _thresholds(m, q, g, [3, 100, 5000]), f"clustered noise={noise}")


def test_duplicates_and_nonfinite():
    m = _get("clip", 512)
    base = _emb(40000, 512, seed=1)
    dup = _emb(2, 512, seed=2)
    g = torch.cat([base, dup[torch.arange(100000, device="cuda") % 2]])
    for r in (5, 40000, 99999):
        g[r] = 0.0
    g[50000, 3] = float("nan")
    g[70000, 0] = float("inf")
    g[80000, 1] = -float("inf")
    g[90000] = 1e30  # the sum of squares overflows: the normalised row is all zeros
    q = torch.cat([dup, _emb(30, 512, seed=3)])
    q[3] = 0.0
    q[4, 4] = float("nan")
    q[5, 0] = float("inf")
    stats = _check(m, m.index(g), q, g, _thresholds(m, q, g, [3, 100]) + [0.0], "duplicates and non-finite")
    assert stats[0].fallbacks > 0, "the duplicate rows overflow the screen's lists"


def test_rows_near_underflow():
    E = 768
    m = _get("clip", E)
    g = _emb(70000, E, seed=1)
    tiny = _emb(4000, E, seed=2)
    g[33000:34000] = tiny[:1000] * 3e-23
    g[40000:41000] = tiny[1000:2000] * 1e-21
    g[50000:51000] = tiny[2000:3000] * 1e-23
    g[50000:51000, :8] = 1e-19
    g[60000:61000] = tiny[3000:4000] * 1e-22
    q = torch.cat([_emb(20, E, seed=3), g[33000:33010], g[50000:50010]])
    _check(m, m.index(g), q, g, _thresholds(m, q, g, [3, 100]), "underflow")


@pytest.mark.parametrize("log_scale", [float("inf"), float("nan"), -100.0])
def test_nonfinite_or_tiny_scale(log_scale):
    """exp(logit_scale) non-finite or below 2^-60: the accumulator bound is -inf and every row is scored exactly."""
    m = _new_model("siglip", 256)
    m.set_flat_param("logit_scale", torch.tensor(log_scale))
    g, q = _emb(70000, 256, seed=41), _emb(10, 256, seed=42)
    _check(m, m.index(g), q, g, [-10.0, BIAS, 0.0, -math.inf], f"logit_scale={log_scale}")


# ---- pairs ----
def _pairs_from_csr(o, s, i):
    rows = o.numel() - 1
    r = torch.repeat_interleave(torch.arange(rows, device=o.device, dtype=torch.int32), o.diff())
    return r, i, s


@pytest.mark.parametrize("N", [2, 2049, 70000, 2**18 + 5])
def test_pairs_upper_triangle(N):
    E = 256
    m = _get("siglip", E)
    g = _emb(N, E, seed=N)
    if N > 10:
        g[N // 2] = g[1]  # an exact duplicate pair
    cuts = sorted({0, N // 3, N // 2 + 1, N})
    index = m.index(g[: cuts[1]])
    for a, b in zip(cuts[1:], cuts[2:]):
        index.add(g[a:b])
    assert len(index) == N
    for t in _thresholds(m, g, g, [2, 50]):
        i, j, s = index.pairs(t)
        o, rs, ri = index.range_search(g, t)
        up = ri > torch.repeat_interleave(torch.arange(N, device="cuda", dtype=torch.int32), o.diff())
        ri_, rj, rsc = [x[up] for x in _pairs_from_csr(o, rs, ri)]
        assert torch.equal(i, ri_) and torch.equal(j, rj) and _bits_equal(s, rsc), f"N={N} t={t}: pairs != upper triangle of range_search"
        assert i.dtype == torch.int32 and j.dtype == torch.int32 and s.dtype == torch.float32 and i.is_cuda
        if N == 70000:
            ro, rsc2, rj2 = _ref_csr(m, g, g, t, upper=True)
            ri2 = torch.repeat_interleave(torch.arange(N, device="cuda", dtype=torch.int32), ro.diff())
            assert torch.equal(i, ri2) and torch.equal(j, rj2) and _bits_equal(s, rsc2), f"N={N} t={t}: pairs != hook matrix"
        if N == 2049:  # the full mask of the hook matrix is symmetric, and so are its scores
            Lm = _hook_rows(m, _normalised(g), _normalised(g))
            assert torch.equal(Lm.view(torch.int32), Lm.T.contiguous().view(torch.int32))
            assert torch.equal((Lm >= t), (Lm >= t).T)


def test_pairs_of_tiny_indexes():
    m = _get("clip", 256)
    for N in (0, 1):
        index = m.index(_emb(N, 256, seed=5)) if N else m.index()
        for t in (-math.inf, 0.0):
            i, j, s = index.pairs(t)
            assert i.numel() == j.numel() == s.numel() == 0
    o, s, i = m.index().range_search(_emb(3, 256, seed=6), -math.inf)
    assert o.tolist() == [0, 0, 0, 0] and s.numel() == 0 and i.numel() == 0, "an empty index gives all-zero offsets"
    o, s, i = m.index(_emb(10, 256, seed=7)).range_search(_emb(0, 256, seed=8), -math.inf)
    assert o.tolist() == [0] and s.numel() == 0


# ---- agreement with index.search ----
def test_contains_search():
    m = _get("siglip", 768)
    g, q = _emb(200000, 768, seed=51), _emb(16, 768, seed=52)
    index = m.index(g)
    for k in (1, 10, 100):
        v, ix = index.search(q, k)
        for r in range(q.shape[0]):
            o, s, i = index.range_search(q[r:r + 1], v[r, k - 1].item())
            got = dict(zip(i.tolist(), s.view(torch.int32).tolist()))
            assert all(a in got for a in ix[r].tolist()), f"k={k} query {r}: search's rows missing"
            assert all(got[a] == b for a, b in zip(ix[r].tolist(), v[r].view(torch.int32).tolist())), f"k={k} query {r}: score bits"


# ---- the screen screens ----
def test_screen_rescores_few_rows():
    E, N, Q = 768, 2**20, 2048
    m = _get("clip", E)
    g, q = _emb(N, E, seed=21), _emb(Q, E, seed=22)
    index = m.index(g)
    (t,) = _thresholds(m, q, g, [10])
    (o, _, _), st = _range_stats(index, q, t)
    per_query = st.rows_rescored / Q
    print(f"\nGaussian 2^20 x {E}, ~10 hits: {per_query:.1f} rows rescored per query, {o[-1].item() / Q:.1f} hits, {st.fallbacks} fallbacks")
    assert st.fallbacks == 0
    assert per_query < 0.01 * N


# ---- int64 offsets ----
def test_offsets_past_2_to_31():
    torch.cuda.empty_cache()
    E, N, Q = 256, 2**20 + 1, 2048
    m = _get("clip", E)
    g, q = _emb(N, E, seed=61), _emb(Q, E, seed=62)
    index = m.index(g)
    o, s, i = index.range_search(q, -math.inf)
    assert o[-1].item() == Q * N and Q * N > 2**31
    assert torch.equal(o, torch.arange(Q + 1, device="cuda", dtype=torch.int64) * N)
    gn = _normalised(g)
    for r in (0, 1, 1023, 2046, 2047):
        a, b = o[r].item(), o[r + 1].item()
        ref = _hook_rows(m, _normalised(q[r:r + 1]), gn)[0]
        assert torch.equal(i[a:b], torch.arange(N, device="cuda", dtype=torch.int32)), f"row {r}: indices"
        assert _bits_equal(s[a:b], ref), f"row {r}: scores"
    del o, s, i


# ---- lifetime and inputs ----
def test_follows_model_and_input_forms():
    m = _new_model("siglip", 256)
    g, q = _emb(70000, 256, seed=71), _emb(40, 256, seed=72)
    index = m.index(g)
    (t,) = _thresholds(m, q, g, [20])
    a = index.range_search(q, t)
    b = index.range_search(q, t)
    assert all(x.dtype == y.dtype and torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(a, b)), "a repeat differs"
    m.set_flat_param("logit_scale", torch.tensor(math.log(30.0)))
    _check(m, index, q, g, [t - 5.0], "after set_flat_param")
    m.set_max_batch(7)
    _check(m, index, q, g, [t - 5.0], "after set_max_batch")
    pi, pj, ps = index.pairs(t)
    ro, rs, rj = _ref_csr(m, g, g, t, upper=True)
    assert torch.equal(pj, rj) and _bits_equal(ps, rs), "pairs after the rebuilds"
    for qq in (q.cpu(), q.to(torch.float16), q.to(torch.bfloat16), q.to(torch.bfloat16).cpu()):
        o, s, i = index.range_search(qq, t)
        assert o.is_cuda == qq.is_cuda and s.is_cuda == qq.is_cuda and i.is_cuda == qq.is_cuda
        _assert_csr((o, s, i), _ref_csr(m, qq.cuda().float(), g, t), f"queries {qq.dtype} on {qq.device}")
    index.close()
    from jimm_b200 import _lib as L

    with pytest.raises(L.JimmError):
        index.range_search(q, t)
    with pytest.raises(L.JimmError):
        index.pairs(t)


# ---- refusals ----
def test_refusals_launch_nothing():
    L = _lib()
    lib = L.load()
    m = _get("clip", 256)
    g, q = _emb(2000, 256, seed=1), _emb(4, 256, seed=2)
    index = m.index(g)
    index.range_search(q, 0.0)  # everything exists before counting
    index.pairs(0.0)
    n = lib.jimm_launch_count()
    for t in (float("nan"), np.float32("nan"), "1.0", torch.tensor(1.0), True, 1 + 2j, None):
        with pytest.raises(ValueError):
            index.range_search(q, t)
        with pytest.raises(ValueError):
            index.pairs(t)
    for qq in (q[:, :255], q.to(torch.float64), q.to(torch.int32), q[0]):
        with pytest.raises(ValueError):
            index.range_search(qq, 0.0)
    h = C.c_void_p()
    assert lib.jimm_index_range_search(index.handle, ptr(q), 4, float("nan"), C.byref(h), None, stream()) == -1
    assert lib.jimm_index_pairs(index.handle, float("nan"), C.byref(h), None, stream()) == -1
    assert lib.jimm_index_range_search(None, ptr(q), 4, 0.0, C.byref(h), None, stream()) == -1
    assert lib.jimm_index_range_search(index.handle, None, 4, 0.0, C.byref(h), None, stream()) == -1
    assert lib.jimm_index_range_search(index.handle, ptr(q), -1, 0.0, C.byref(h), None, stream()) == -1
    assert lib.jimm_index_range_search(index.handle, ptr(q), 4, 0.0, None, None, stream()) == -1
    assert lib.jimm_index_pairs(None, 0.0, C.byref(h), None, stream()) == -1
    assert lib.jimm_index_pairs(index.handle, 0.0, None, None, stream()) == -1
    rows, total = C.c_int(), C.c_longlong()
    assert lib.jimm_hits_size(None, C.byref(rows), C.byref(total)) == -1
    assert lib.jimm_hits_copy(None, None, None, None, stream()) == -1
    assert lib.jimm_hits_destroy(None) == 0
    assert lib.jimm_launch_count() == n, "a refused call launched a kernel"
    index.close()
    with pytest.raises(L.JimmError):
        index.range_search(q, 0.0)
