"""GPU tests of removing rows from a gallery index and searching a subset of its rows (index.remove, index.compact, keep=), bit for bit
against the same calls on the allowed rows alone.

Notation: raw = every row ever added, A = the ascending ids of a call's allowed rows (live and kept), nA = len(A), twin = an index of raw
with nothing removed.
  * search: the first min(k, nA) columns of index.search(q, k, keep) equal model.search(q, raw[A], min(k, nA)) with indices mapped
    through A -- scores as int32 bit patterns -- and the rest are (-inf, -1).  CLIP and SigLIP, N below the seed block and across
    several screen chunks, E = 256, 768 and 1152, filters from every row to none, masks and id lists, host and device.
  * removals: search equals search(keep=live) and the identity above; repeated removals count nothing; add numbers from len(index);
    num_live; the live rows survive a model rebuild.
  * range_search and pairs equal the twin's with the entries outside A dropped, under removals and filters, including thresholds
    so low that queries take the exact fallback.
  * traps: zero and non-finite rows that are removed or filtered out never appear; duplicates overflowing the screen list with half
    of them filtered out fall back and stay exact.
  * compact: the map, and every call after it equals the call before it with indices mapped.
  * no change: with nothing removed and keep=None the calls launch exactly as many kernels as before.
  * refusals raise ValueError (or return JIMM_EINVAL) and launch nothing."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gpu_util import check, ptr, stream

pytestmark = pytest.mark.gpu

LOG_SCALE, BIAS = math.log(100.0), -10.0


def _bits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _launches():
    from jimm_b200 import _lib

    return _lib.load().jimm_launch_count()


_MODELS = {}


def _new_model(kind, E):
    """A 1-layer fp16 CLIP / SigLIP at random init with both towers E wide, logit_scale = log 100 and, for SigLIP, logit_bias = -10."""
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


def _ref_search(m, q, raw, A, k):
    """model.search over raw[A], indices through A, padded with (-inf, -1) past nA."""
    Q, nA = q.shape[0], A.numel()
    v = torch.full((Q, k), -math.inf, device="cuda")
    i = torch.full((Q, k), -1, dtype=torch.int32, device="cuda")
    kk = min(k, nA)
    if kk > 0:
        rv, ri = m.search(q, raw[A], kk)
        v[:, :kk] = rv
        i[:, :kk] = A[ri.long()].to(torch.int32)
    return v, i


def _check_search(m, index, q, raw, A, ks, what, keep="mask"):
    """index.search(q, k, keep) against _ref_search for each k that fits len(index); keep given as A's mask or ids (or None)."""
    N = len(index)
    if keep == "mask":
        kp = torch.zeros(N, dtype=torch.bool, device="cuda")
        kp[A] = True
    elif keep == "ids":
        kp = A
    else:
        kp = None
    for k in ks:
        if k > min(N, 1024):
            continue
        v, i = index.search(q, k, keep=kp)
        rv, ri = _ref_search(m, q, raw, A, k)
        bad = (i != ri).any(dim=1).nonzero().flatten()
        assert bad.numel() == 0, f"{what} k={k}: indices differ in queries {bad[:8].tolist()}"
        assert _bits(v, rv), f"{what} k={k}: scores differ"


def _filters(N, seed):
    """(name, ascending allowed ids) for the filters of the identity tests."""
    gen = torch.Generator().manual_seed(seed)
    r = torch.rand(N, generator=gen)
    lo = max(0, min(65536, N) - 3000)
    hi = min(N, lo + 80000) if N > 65536 else min(N, lo + 2000)
    out = [("all", torch.arange(N)), ("half", (r < 0.5).nonzero().flatten()), ("1%", (r < 0.01).nonzero().flatten()),
           ("one", torch.tensor([int(N * 0.37)])), ("first", torch.tensor([0])), ("last", torch.tensor([N - 1])),
           ("block", torch.arange(lo, hi)), ("empty", torch.zeros(0, dtype=torch.int64))]
    return [(n, a.to("cuda")) for n, a in out]


# ---- identity 1: search over the allowed rows ----
@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.parametrize("N,E", [(5000, 256), (2**18 + 5, 768), (70001, 1152)])
def test_search_identity(kind, N, E):
    m = _get(kind, E)
    raw, q = _emb(N, E, seed=N + E), _emb(37, E, seed=7) * 2.0
    index = m.index(raw)
    for j, (name, A) in enumerate(_filters(N, seed=N)):
        ks = [1, 5, 100, 1024] if name in ("half", "all") or N == 5000 else [5, 100]
        form = ("mask", "ids")[j % 2]
        _check_search(m, index, q, raw, A, ks, f"{kind} N={N} E={E} {name} {form}", keep=form)
    # host keep, as a mask and as a list of ids
    A = _filters(N, seed=N)[2][1]
    kp = torch.zeros(N, dtype=torch.bool)
    kp[A.cpu()] = True
    v, i = index.search(q, 5, keep=kp)
    rv, ri = _ref_search(m, q, raw, A, 5)
    assert torch.equal(i, ri) and _bits(v, rv), "host mask"
    v, i = index.search(q, 5, keep=A.tolist())
    assert torch.equal(i, ri) and _bits(v, rv), "host id list"
    v, i = index.search(q, 5, keep=A.cpu().numpy())
    assert torch.equal(i, ri) and _bits(v, rv), "numpy ids"


def test_padding_and_duplicate_ids():
    """Fewer allowed rows than k: the columns past them are (-inf, -1).  Ids in any order and repeated select the same rows."""
    m = _get("siglip", 256)
    raw, q = _emb(3000, 256, seed=11), _emb(9, 256, seed=12)
    index = m.index(raw)
    A = torch.tensor([5, 17, 2999], device="cuda")
    v, i = index.search(q, 10, keep=torch.tensor([2999, 5, 17, 5, 2999], device="cuda"))
    rv, ri = _ref_search(m, q, raw, A, 10)
    assert torch.equal(i, ri) and _bits(v, rv)
    assert (i[:, 3:] == -1).all() and torch.isneginf(v[:, 3:]).all() and (i[:, :3] >= 0).all()
    v, i = index.search(q.cpu(), 4, keep=[])  # host queries, empty filter: all padding, on the host
    assert not v.is_cuda and (i == -1).all() and torch.isneginf(v).all()


# ---- removals ----
def test_remove_then_search():
    m = _get("clip", 256)
    N = 70000
    raw, q = _emb(N, 256, seed=21), _emb(40, 256, seed=22)
    index = m.index(raw)
    assert index.num_live == N
    gen = torch.Generator().manual_seed(23)
    rem = torch.randperm(N, generator=gen)[: N // 3]
    assert index.remove(rem.cuda()) == N // 3
    assert index.remove(rem[:100].numpy()) == 0, "rows already removed count nothing"
    assert index.remove([int(rem[0]), int(rem[0])]) == 0
    gone = set(rem.tolist())
    extra = [x for x in range(N) if x not in gone][:2]
    assert index.remove([extra[0], extra[0], extra[1]]) == 2, "a duplicate id counts once"
    assert index.remove(extra[0]) == 0
    assert index.num_live == N - N // 3 - 2 and len(index) == N
    live = torch.ones(N, dtype=torch.bool, device="cuda")
    live[rem.cuda()] = False
    live[extra] = False
    A = live.nonzero().flatten()
    _check_search(m, index, q, raw, A, [1, 5, 100, 1024], "after removals", keep=None)
    for k in (5, 100):
        v, i = index.search(q, k)
        kv, ki = index.search(q, k, keep=live)
        assert torch.equal(i, ki) and _bits(v, kv), "search != search(keep=live)"
    # a filter on top of the removals: the allowed rows are live and kept
    kp = torch.rand(N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(24)) < 0.2
    v, i = index.search(q, 100, keep=kp)
    rv, ri = _ref_search(m, q, raw, (live & kp).nonzero().flatten(), 100)
    assert torch.equal(i, ri) and _bits(v, rv), "removals and a filter"
    # add after remove: new rows are live and numbered from len(index)
    more = _emb(500, 256, seed=25)
    index.add(more)
    assert len(index) == N + 500 and index.num_live == N - N // 3 - 2 + 500
    raw2 = torch.cat([raw, more])
    A2 = torch.cat([A, torch.arange(N, N + 500, device="cuda")])
    _check_search(m, index, q, raw2, A2, [5, 100], "add after remove", keep=None)
    assert index.remove(N + 3) == 1
    _check_search(m, index, q, raw2, A2[A2 != N + 3], [5], "remove of an added row", keep=None)


def test_remove_everything():
    m = _get("siglip", 256)
    raw, q = _emb(40000, 256, seed=31), _emb(5, 256, seed=32)
    index = m.index(raw)
    assert index.remove(torch.arange(40000)) == 40000 and index.num_live == 0
    v, i = index.search(q, 7)
    assert (i == -1).all() and torch.isneginf(v).all()
    o, s, j = index.range_search(q, -math.inf)
    assert o.tolist() == [0] * 6 and s.numel() == 0
    a, b, s = index.pairs(-math.inf)
    assert a.numel() == b.numel() == s.numel() == 0


def test_live_rows_follow_model_rebuilds():
    m = _new_model("siglip", 256)
    N = 32768 + 50000
    raw, q = _emb(N, 256, seed=41), _emb(30, 256, seed=42)
    index = m.index(raw)
    rem = torch.arange(0, N, 3, device="cuda")
    index.remove(rem)
    live = torch.ones(N, dtype=torch.bool, device="cuda")
    live[rem] = False
    A = live.nonzero().flatten()
    _check_search(m, index, q, raw, A, [5], "before", keep=None)
    n0 = m.native()
    m.set_flat_param("logit_scale", torch.tensor(math.log(30.0)))
    assert m.native() is not n0
    _check_search(m, index, q, raw, A, [5, 100], "after a rebuild", keep=None)
    assert index.num_live == A.numel()


# ---- identities 2 and 3: range search and pairs against a twin ----
def _filter_csr(o, s, i, allowed):
    keep = allowed[i.long()]
    rows = o.numel() - 1
    r = torch.repeat_interleave(torch.arange(rows, device=o.device), o.diff())
    cnt = torch.bincount(r[keep], minlength=rows)
    return torch.cat([torch.zeros(1, dtype=torch.int64, device=o.device), cnt.cumsum(0)]), s[keep], i[keep]


def _same_csr(got, ref, what):
    assert torch.equal(got[0].cpu(), ref[0].cpu()), f"{what}: offsets differ"
    assert torch.equal(got[2].cpu(), ref[2].cpu()), f"{what}: indices differ"
    assert _bits(got[1], ref[1]), f"{what}: scores differ"


def _thresholds(twin, q, ks):
    """Scores at each query's k-th best, medianed: thresholds with about k hits per query."""
    return [float(twin.search(q, k)[0][:, -1].median()) for k in ks]


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_range_search_identity(kind):
    m = _get(kind, 256)
    N = 140001
    raw, q = _emb(N, 256, seed=51), _emb(2100, 256, seed=52)  # across the 2048-query chunk
    twin, index = m.index(raw), m.index(raw)
    gen = torch.Generator(device="cuda").manual_seed(53)
    live = torch.rand(N, device="cuda", generator=gen) >= 0.1
    index.remove((~live).nonzero().flatten())
    assert index.num_live == int(live.sum())
    kp = torch.rand(N, device="cuda", generator=gen) < 0.5
    low = -30.0 if kind == "siglip" else 0.0  # about half the rows clear it: every (query, chunk) list overflows
    for t in _thresholds(twin, q, [3, 300]) + [low]:
        qq = q if t != low else q[:40]
        ref = twin.range_search(qq, t)
        _same_csr(index.range_search(qq, t), _filter_csr(*ref, live), f"{kind} t={t} removals")
        _same_csr(index.range_search(qq, t, keep=kp), _filter_csr(*ref, live & kp), f"{kind} t={t} removals and filter")
        _same_csr(twin.range_search(qq, t, keep=kp.nonzero().flatten().cpu()), _filter_csr(*ref, kp), f"{kind} t={t} filter")


def _same_pairs(got, ref, what):
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), f"{what}: pairs differ"
    assert _bits(got[2], ref[2]), f"{what}: scores differ"


@pytest.mark.parametrize("N,low", [(9000, True), (140001, False)])
def test_pairs_identity(N, low):
    m = _get("siglip", 256)
    raw = _emb(N, 256, seed=N)
    gen = torch.Generator(device="cuda").manual_seed(61)
    src = torch.randint(0, N, (N // 50,), device="cuda", generator=gen)
    dst = torch.randint(0, N, (N // 50,), device="cuda", generator=gen)
    raw[dst] = raw[src] + 0.01 * torch.randn(dst.numel(), 256, device="cuda", generator=gen)  # planted near-duplicates
    twin, index = m.index(raw), m.index(raw)
    live = torch.rand(N, device="cuda", generator=gen) >= 0.25
    index.remove((~live).nonzero().flatten())
    kp = torch.rand(N, device="cuda", generator=gen) < 0.6
    ts = [-20.0] if low else [float(m.search(raw[:64], raw, 2)[0][:, -1].min()), 80.0]
    for t in ts:
        i, j, s = twin.pairs(t)
        assert i.numel() > 0
        for what, allowed, idx, keep in [("removals", live, index, None), ("filter", kp, twin, kp), ("both", live & kp, index, kp.nonzero().flatten())]:
            ok = allowed[i.long()] & allowed[j.long()]
            _same_pairs(idx.pairs(t, keep=keep), (i[ok], j[ok], s[ok]), f"N={N} t={t} {what}")


# ---- traps ----
def test_removed_and_filtered_nonfinite_rows_never_appear():
    """Zero and non-finite rows have norm bound +inf and pass every screen; NaN ranks first.  Removed or filtered out, they never appear."""
    m = _get("clip", 256)
    N = 100000
    raw, q = _emb(N, 256, seed=71), _emb(20, 256, seed=72)
    bad = torch.tensor([3, 40000, 70001, 99999], device="cuda")
    raw[bad[0]] = 0.0
    raw[bad[1]] = math.nan
    raw[bad[2], 7] = math.inf
    raw[bad[3]] = 0.0
    index = m.index(raw)
    v, i = index.search(q, 5)
    assert torch.isin(i, bad.to(torch.int32)).any(), "the bad rows rank first when present"
    index.remove(bad[:2])
    kp = torch.ones(N, dtype=torch.bool, device="cuda")
    kp[bad[2:]] = False
    live = torch.ones(N, dtype=torch.bool, device="cuda")
    live[bad[:2]] = False
    A = (live & kp).nonzero().flatten()
    for k in (1, 5, 100):
        v, i = index.search(q, k, keep=kp)
        rv, ri = _ref_search(m, q, raw, A, k)
        assert torch.equal(i, ri) and _bits(v, rv), f"k={k}"
        assert not torch.isin(i, bad.to(torch.int32)).any()
        assert not torch.isnan(v).any()
    o, s, j = index.range_search(q, -math.inf, keep=kp)
    assert not torch.isin(j, bad.to(torch.int32)).any() and o[-1] == 20 * A.numel()
    a, b, s = index.pairs(-math.inf, keep=torch.arange(0, 200, device="cuda"))
    assert not torch.isin(a, bad.to(torch.int32)).any() and not torch.isin(b, bad.to(torch.int32)).any()


def _search_keep_stats(index, q, k, keep):
    from jimm_b200 import _lib

    index._model()
    Q = q.shape[0]
    qd = q.to("cuda", torch.float32).contiguous()
    v = torch.empty((Q, k), device="cuda")
    i = torch.empty((Q, k), dtype=torch.int32, device="cuda")
    st = _lib.SearchStats()
    check(_lib.load(), _lib.load().jimm_index_search_keep(index.handle, ptr(qd), Q, k, ptr(keep) if keep is not None else None, ptr(v), ptr(i),
                                                          C.byref(st), stream()))
    torch.cuda.synchronize()
    return v, i, st


def test_filtered_duplicates_fall_back():
    """Every row after the seed block is one of two rows, and half of those copies are filtered out: the kept copies still overflow the
    screen's lists, the fallback block step runs over allowed rows only, and the seed counts only allowed rows."""
    m = _get("clip", 256)
    base = _emb(32768, 256, seed=81)
    dup = _emb(2, 256, seed=82)
    raw = torch.cat([base, dup[torch.arange(100000, device="cuda") % 2]])
    q = torch.cat([dup, _emb(30, 256, seed=83)])
    index = m.index(raw)
    N = raw.shape[0]
    gen = torch.Generator(device="cuda").manual_seed(84)
    kp = torch.rand(N, device="cuda", generator=gen) < 0.5
    kp[:32768] = torch.rand(32768, device="cuda", generator=gen) < 0.9
    A = kp.nonzero().flatten()
    for k in (1, 100, 1024):
        v, i, st = _search_keep_stats(index, q, k, kp)
        rv, ri = _ref_search(m, q, raw, A, k)
        assert torch.equal(i, ri) and _bits(v, rv), f"k={k}"
        assert not torch.isin(i, (~kp).nonzero().flatten().to(torch.int32)).any()
        assert st.fallbacks > 0, f"k={k}: no fallback"


# ---- identity 4: compact ----
def test_compact():
    m = _get("siglip", 256)
    N = 140001
    raw, q = _emb(N, 256, seed=91), _emb(50, 256, seed=92)
    index = m.index(raw)
    gen = torch.Generator(device="cuda").manual_seed(93)
    dead = (torch.rand(N, device="cuda", generator=gen) < 0.3).nonzero().flatten()
    index.remove(dead)
    t = float(index.search(q, 20)[0][:, -1].median())
    tp = float(m.search(raw[:64], raw, 2)[0][:, -1].min())
    before = [index.search(q, k) for k in (5, 100)]
    rbefore = index.range_search(q, t)
    pbefore = index.pairs(tp)
    live = index.num_live
    mp = index.compact()
    assert mp.dtype == torch.int64 and mp.is_cuda and mp.numel() == N
    alive = torch.ones(N, dtype=torch.bool, device="cuda")
    alive[dead] = False
    assert (mp[~alive] == -1).all() and torch.equal(mp[alive], torch.arange(live, device="cuda"))
    assert len(index) == live and index.num_live == live
    for (v0, i0), k in zip(before, (5, 100)):
        v, i = index.search(q, k)
        assert torch.equal(i.long(), mp[i0.long()]) and _bits(v, v0), f"search k={k} after compact"
    o, s, i = index.range_search(q, t)
    assert torch.equal(o, rbefore[0]) and torch.equal(i.long(), mp[rbefore[2].long()]) and _bits(s, rbefore[1])
    a, b, s = index.pairs(tp)
    assert torch.equal(a.long(), mp[pbefore[0].long()]) and torch.equal(b.long(), mp[pbefore[1].long()]) and _bits(s, pbefore[2])
    # add after compact, then an index with nothing removed compacts to the identity
    more = _emb(300, 256, seed=94)
    index.add(more)
    assert len(index) == live + 300
    _check_search(m, index, q, torch.cat([raw[alive], more]), torch.arange(live + 300, device="cuda"), [5], "add after compact", keep=None)
    ident = index.compact()
    assert torch.equal(ident, torch.arange(live + 300, device="cuda"))
    empty = m.index()
    assert empty.compact().numel() == 0


# ---- identity 5: nothing removed, no filter ----
def test_unfiltered_calls_launch_as_before():
    from jimm_b200 import _lib

    m = _get("clip", 256)
    raw, q = _emb(70000, 256, seed=101), _emb(10, 256, seed=102)
    index = m.index(raw)
    index.search(q, 5)

    def count(f):
        n = _launches()
        f()
        torch.cuda.synchronize()
        return _launches() - n

    plain = count(lambda: index.search(q, 5))
    assert count(lambda: index.search(q, 5, keep=None)) == plain
    r = count(lambda: index.range_search(q, 50.0))
    assert count(lambda: index.range_search(q, 50.0, keep=None)) == r
    p = count(lambda: index.pairs(90.0))
    assert count(lambda: index.pairs(90.0, keep=None)) == p
    lib = _lib.load()
    v = torch.empty((10, 5), device="cuda")
    i = torch.empty((10, 5), dtype=torch.int32, device="cuda")
    qd = q.contiguous()
    c = count(lambda: check(lib, lib.jimm_index_search(index.handle, ptr(qd), 10, 5, ptr(v), ptr(i), None, stream())))
    assert c == plain
    assert count(lambda: check(lib, lib.jimm_index_search_keep(index.handle, ptr(qd), 10, 5, None, ptr(v), ptr(i), None, stream()))) == plain
    assert count(lambda: index.search(q, 5, keep=torch.ones(70000, dtype=torch.bool))) > plain, "a filter lists the allowed rows"
    index.compact()  # nothing removed: the same rows, the same code
    assert count(lambda: index.search(q, 5)) == plain
    assert index.remove([]) == 0
    assert count(lambda: index.search(q, 5)) == plain


# ---- refusals ----
def test_refusals_launch_nothing():
    from jimm_b200 import _lib

    m = _get("clip", 256)
    raw, q = _emb(2000, 256, seed=111), _emb(4, 256, seed=112)
    index = m.index(raw)
    index.search(q, 1)
    n = _launches()
    bad_keeps = [torch.ones(1999, dtype=torch.bool), torch.ones(2001, dtype=torch.bool, device="cuda"), torch.ones(2000),
                 np.ones(2000, dtype=np.float32), [0.5], [2000], [-1], torch.tensor([0, 2000], device="cuda"), ["a"]]
    for kp in bad_keeps:
        with pytest.raises(ValueError):
            index.search(q, 5, keep=kp)
        with pytest.raises(ValueError):
            index.range_search(q, 0.0, keep=kp)
        with pytest.raises(ValueError):
            index.pairs(0.0, keep=kp)
    for ids in ([2000], -1, torch.tensor([5, -3]), torch.tensor([1.0]), torch.ones(3, dtype=torch.bool), np.array([0.0]), [1.5]):
        with pytest.raises(ValueError):
            index.remove(ids)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            index.search(q, 5, keep=torch.ones(2000, dtype=torch.bool, device="cuda:1"))
        with pytest.raises(ValueError):
            index.remove(torch.tensor([0], device="cuda:1"))
    lib = _lib.load()
    removed = C.c_longlong()
    live = C.c_longlong()
    ids = torch.tensor([1, 2], dtype=torch.int32, device="cuda")
    assert lib.jimm_index_remove(None, ptr(ids), 2, C.byref(removed), stream()) == -1
    assert lib.jimm_index_remove(index.handle, ptr(ids), -1, C.byref(removed), stream()) == -1
    assert lib.jimm_index_remove(index.handle, None, 2, C.byref(removed), stream()) == -1
    assert lib.jimm_index_remove(index.handle, ptr(ids), 2, None, stream()) == -1
    assert lib.jimm_index_live(None, C.byref(live)) == -1
    assert lib.jimm_index_live(index.handle, None) == -1
    assert lib.jimm_index_compact(None, None, stream()) == -1
    v = torch.empty((4, 8), device="cuda")
    i = torch.empty((4, 8), dtype=torch.int32, device="cuda")
    kp = torch.ones(2000, dtype=torch.bool, device="cuda")
    for k in (0, 2001, 1025):
        assert lib.jimm_index_search_keep(index.handle, ptr(q), 4, k, ptr(kp), ptr(v), ptr(i), None, stream()) == -1
    h = C.c_void_p()
    assert lib.jimm_index_range_search_keep(index.handle, ptr(q), 4, math.nan, ptr(kp), C.byref(h), None, stream()) == -1
    assert lib.jimm_index_pairs_keep(index.handle, 0.0, ptr(kp), None, None, stream()) == -1
    assert _launches() == n, "a refused call launched a kernel"
    assert index.num_live == 2000 and len(index) == 2000
    # an id out of range on the device is found on the device: JIMM_EINVAL, and nothing is removed
    ids = torch.tensor([1, 2000], dtype=torch.int32, device="cuda")
    assert lib.jimm_index_remove(index.handle, ptr(ids), 2, C.byref(removed), stream()) == -1
    assert index.num_live == 2000
    assert index.remove(1) == 1 and index.num_live == 1999
    index.close()
    for f in (lambda: index.remove(0), lambda: index.compact(), lambda: index.num_live, lambda: index.search(q, 1, keep=[0])):
        with pytest.raises(_lib.JimmError):
            f()
