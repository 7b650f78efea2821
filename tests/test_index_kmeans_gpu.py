"""GPU tests of spherical k-means over a gallery index (index.kmeans / jimm_index_kmeans), bit for bit against kmeans_oracle.py run on the
library's own hooks.

The oracle takes the stored rows (jimm_k_l2_normalize of the raw rows), keeps the clusterable ones (allowed, finite, norm bound <= 2),
and runs each step through the hooks: jimm_k_l2_normalize of the means, jimm_k_logits at logit_scale 0 and no bias in row chunks,
top_k(., 1), then numpy for the fixed-point sums.  Centroids and scores are compared as int32 bit patterns; assignments, counts and
iterations must be equal.
  * identity: CLIP and SigLIP (bias -10) at E = 256, 768 and 1152, N from 1000 to 2^18 + 5 (across the 2048-row chunks), C in {1, 7,
    255, 256, 257, 1000, 32769, 65536}, iters 1 to 5, sampled, id and vector inits, several seeds;
  * clustered data converges before iters, with the screen rescoring a small fraction of C per row and no fallbacks;
  * hostile rows (zero, NaN, inf, subnormal-sum, duplicates), duplicate init ids, a cluster whose mean is exactly zero;
  * keep= and remove() equal k-means on an index of the allowed rows alone; compact() through its map;
  * repeatability, and search / range_search / pairs unchanged (bits and launches) around a k-means call;
  * refusals."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import kmeans_oracle as ko
from gpu_util import ptr, stream

pytestmark = pytest.mark.gpu

LOG_SCALE, BIAS = math.log(100.0), -10.0


def _lib():
    from jimm_b200 import _lib as L

    return L


def _launches():
    return _lib().load().jimm_launch_count()


def _bits(a, b):
    a, b = torch.as_tensor(a).detach().cpu().contiguous(), torch.as_tensor(b).detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


_MODELS = {}


def _get(kind, E):
    """A 1-layer fp16 CLIP / SigLIP at random init, logit_scale = log 100 and, for SigLIP, logit_bias = -10."""
    if (kind, E) not in _MODELS:
        from jimm_b200.models import CLIP, SigLIP

        h = E // 64
        m = (CLIP if kind == "clip" else SigLIP)(32, 1, E, 16, 8, 64, E, h, 1, dtype=torch.float16, vision_heads=h)
        m.set_flat_param("logit_scale", torch.tensor(LOG_SCALE))
        if kind == "siglip":
            m.set_flat_param("logit_bias", torch.tensor(BIAS))
        _MODELS[(kind, E)] = m
    return _MODELS[(kind, E)]


def _emb(n, E, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, E, device="cuda", generator=g)


# ---- the hooks ----
def _normalize(x):
    """jimm_k_l2_normalize of fp32 rows (numpy or device tensor) -> device tensor."""
    L = _lib()
    x = torch.as_tensor(x).to("cuda", torch.float32).contiguous()
    out = torch.empty_like(x)
    E = x.shape[1]
    for r0 in range(0, x.shape[0], 1 << 20):
        n = min(1 << 20, x.shape[0] - r0)
        L.check(L.load().jimm_k_l2_normalize(ptr(x[r0:]), ptr(out[r0:]), E, n, E, stream()))
    return out


def _normalize_np(m):
    return _normalize(m).cpu().numpy()


def _assign_np(x, c):
    """Each row's best centroid: jimm_k_logits at logit_scale 0 (exp(0) = 1) and no bias, then top_k(., 1)."""
    from jimm_b200.postprocess import top_k

    L = _lib()
    xd = torch.as_tensor(x).to("cuda").contiguous()
    cd = torch.as_tensor(c).to("cuda").contiguous()
    n, Cn, E = xd.shape[0], cd.shape[0], xd.shape[1]
    zero = torch.zeros(1, device="cuda")
    a = np.empty(n, dtype=np.int32)
    s = np.empty(n, dtype=np.float32)
    step = max(1, min(n, (1 << 27) // Cn))
    for r0 in range(0, n, step):
        r = min(step, n - r0)
        out = torch.empty((r, Cn), dtype=torch.float32, device="cuda")
        L.check(L.load().jimm_k_logits(ptr(xd[r0:]), ptr(cd), ptr(zero), None, ptr(out), r, Cn, E, Cn, stream()))
        v, i = top_k(out, 1)
        a[r0:r0 + r] = i[:, 0].cpu().numpy()
        s[r0:r0 + r] = v[:, 0].cpu().numpy()
    return a, s


def _stored(raw):
    """The index's stored rows (numpy fp32) and which of them are clusterable (finite, norm bound <= 2)."""
    x = _normalize(raw).cpu().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        nb = np.sqrt((x.astype(np.float64) ** 2).sum(axis=1)) * (1 + 2.0**-30)
    return x, np.isfinite(x).all(axis=1) & (nb <= 2)


def _oracle(raw, Cn, iters, init=None, seed=0, allowed=None):
    """(centroids, assign [N], scores [N], counts, iterations) of the definition on raw's stored rows."""
    x, ok = _stored(raw)
    N = x.shape[0]
    if allowed is not None:
        ok = ok & allowed
    ids = np.flatnonzero(ok)
    if init is None:
        m0 = x[ko.sample_init(ids, seed, Cn)]
    elif isinstance(init, np.ndarray) and init.dtype.kind in "iu":
        m0 = x[init]
    else:
        m0 = torch.as_tensor(init).float().cpu().numpy()
    c, a, s, it = ko.kmeans(x[ids], m0, iters, _normalize_np, _assign_np)
    assign = np.full(N, -1, dtype=np.int32)
    scores = np.full(N, -np.inf, dtype=np.float32)
    assign[ids], scores[ids] = a, s
    return c, assign, scores, np.bincount(a, minlength=Cn).astype(np.int64), it


def _check(res, ref, what):
    c, a, s, n, it = ref
    assert res.iterations == it, f"{what}: {res.iterations} steps, oracle {it}"
    assert np.array_equal(res.assign.cpu().numpy(), a), f"{what}: assignments differ"
    assert _bits(res.centroids, torch.from_numpy(c)), f"{what}: centroids differ"
    assert _bits(res.scores, torch.from_numpy(s)), f"{what}: scores differ"
    assert np.array_equal(res.counts.cpu().numpy(), n), f"{what}: counts differ"
    for t in (res.centroids, res.assign, res.scores, res.counts):
        assert t.is_cuda


def _init(kind_of_init, N, Cn, E, seed):
    rng = np.random.default_rng(seed)
    if kind_of_init == "ids":
        return rng.choice(N, Cn, replace=Cn > N)
    if kind_of_init == "vectors":
        return _emb(Cn, E, seed + 99)
    return None


# ---- identity ----
CASES = [
    ("clip", 256, 5000, 7, 5, "sampled", 0),
    ("siglip", 256, 5000, 1, 3, "ids", 1),
    ("clip", 768, 2**18 + 5, 1000, 4, "sampled", 2),
    ("siglip", 768, 70001, 255, 3, "vectors", 3),
    ("clip", 1152, 20000, 257, 2, "sampled", 4),
    ("siglip", 1152, 9000, 256, 5, "ids", 5),
    ("clip", 768, 2049, 1000, 1, "sampled", 6),
    ("siglip", 256, 4097, 16, 5, "sampled", 2**64 - 1),
    ("clip", 256, 70000, 32769, 2, "sampled", 7),
    ("siglip", 256, 66000, 65536, 2, "vectors", 8),
]


@pytest.mark.parametrize("kind,E,N,Cn,iters,init,seed", CASES)
def test_kmeans_identity(kind, E, N, Cn, iters, init, seed):
    m = _get(kind, E)
    raw = _emb(N, E, seed=N + E + Cn)
    index = m.index(raw)
    it = _init(init, N, Cn, E, seed % 1000)
    res = index.kmeans(Cn, iters=iters, init=it, seed=seed)
    _check(res, _oracle(raw, Cn, iters, it, seed), f"{kind} E={E} N={N} C={Cn} iters={iters} {init} seed={seed}")
    if init == "vectors":  # the same vectors from the host and in fp16 / bf16 give the float32 of those values
        for v in (it.cpu(), it.half(), it.bfloat16()):
            r2 = index.kmeans(Cn, iters=iters, init=v, seed=seed)
            _check(r2, _oracle(raw, Cn, iters, v.float(), seed), f"init {v.dtype} {v.device}")


def _kmeans_c(index, Cn, iters, init_ids=None, init_vectors=None, seed=0):
    """jimm_index_kmeans directly, returning (rc, stats, iterations)."""
    L = _lib()
    N = len(index)
    out = [torch.empty((Cn, index._width), device="cuda"), torch.empty(N, dtype=torch.int32, device="cuda"),
           torch.empty(N, device="cuda"), torch.empty(Cn, dtype=torch.int64, device="cuda")]
    st, steps = L.SearchStats(), C.c_int()
    rc = L.load().jimm_index_kmeans(index.handle, Cn, ptr(init_vectors), ptr(init_ids), seed, iters, None, *[ptr(t) for t in out], C.byref(steps),
                                    C.byref(st), stream())
    torch.cuda.synchronize()
    return rc, st, steps.value


def test_clustered_converges_and_screens():
    """1000 planted centres: started from one row of each, the assignment repeats before iters, the screen keeps few centroids per
    row, and nothing falls back."""
    E, N, Cn = 768, 2**18, 1000
    m = _get("clip", E)
    g = torch.Generator(device="cuda").manual_seed(5)
    centres = torch.randn(Cn, E, device="cuda", generator=g)
    lab = torch.randint(0, Cn, (N,), device="cuda", generator=g)
    raw = centres[lab] + 0.3 * torch.randn(N, E, device="cuda", generator=g)
    index = m.index(raw)
    lab_np = lab.cpu().numpy()
    first = np.array([np.flatnonzero(lab_np == j)[0] for j in range(Cn)])
    res = index.kmeans(Cn, iters=20, init=first)
    assert res.iterations < 20
    _check(res, _oracle(raw, Cn, 20, first), "clustered")
    rc, st, steps = _kmeans_c(index, Cn, 20, init_ids=torch.from_numpy(first).int().cuda())
    assert rc == 0 and steps == res.iterations
    per_row = st.rows_rescored / (N * steps)
    print(f"clustered: {steps} steps, {per_row:.2f} centroids rescored per row and step (C = {Cn}), {st.fallbacks} fallbacks, "
          f"{st.chunks_screened} chunks")
    assert st.fallbacks == 0 and st.chunks_screened == steps * math.ceil(N / 2048)
    assert per_row < 0.02 * Cn


def test_hostile_rows():
    """Zero, NaN, inf and subnormal-sum rows take no part (-1, -inf, never counted); exact duplicates cluster together."""
    E, N = 256, 3000
    m = _get("siglip", E)
    raw = _emb(N, E, seed=11)
    raw[10] = 0
    raw[20, 5] = float("nan")
    raw[30, 7] = float("inf")
    raw[40] = 1e-30  # its sum of squares underflows in fp32
    raw[50:60] = raw[49]
    index = m.index(raw)
    bad = [10, 20, 30, 40]
    for init in (None, np.array([49, 50, 0, 1, 2, 3, 4])):
        res = index.kmeans(7, iters=4, init=init, seed=3)
        _check(res, _oracle(raw, 7, 4, init, 3), f"hostile init={init}")
        a = res.assign.cpu()
        assert (a[bad] == -1).all() and torch.isinf(res.scores.cpu()[bad]).all()
        assert int(res.counts.sum()) == N - len(bad)
        assert len(set(a[49:60].tolist())) == 1


def test_duplicate_init_ids_and_zero_mean():
    E = 256
    m = _get("clip", E)
    raw = _emb(500, E, seed=12)
    index = m.index(raw)
    init = np.array([5, 5, 9])
    res = index.kmeans(3, iters=1, init=init)
    _check(res, _oracle(raw, 3, 1, init), "duplicate init ids, one step")
    assert int(res.counts[0]) == 0  # equal scores go to the larger cluster
    res = index.kmeans(3, iters=5, init=init)
    _check(res, _oracle(raw, 3, 5, init), "duplicate init ids")
    # rows v and -v, one cluster: the mean is exactly zero, so the centroid stays l2_normalize(v) and the assignment repeats
    v = _emb(1, E, seed=13)
    idx2 = m.index(torch.cat([v, -v]))
    res = idx2.kmeans(1, iters=5, init=[0])
    _check(res, _oracle(torch.cat([v, -v]), 1, 5, np.array([0])), "zero mean")
    assert res.iterations == 2 and _bits(res.centroids, _normalize(_normalize(v)))


def test_keep_remove_compact():
    E, N, Cn = 256, 20000, 300
    m = _get("siglip", E)
    raw = _emb(N, E, seed=21)
    V = _emb(Cn, E, seed=22)
    A = torch.rand(N, generator=torch.Generator().manual_seed(3)) < 0.5
    Ad = A.cuda()
    ref = m.index(raw[Ad]).kmeans(Cn, iters=4, init=V)
    index = m.index(raw)

    def same(res, what, ids=None):
        a = res.assign.cpu()
        ids = torch.nonzero(A).flatten() if ids is None else ids
        assert res.iterations == ref.iterations, what
        assert torch.equal(a[ids], ref.assign.cpu()), what
        assert (a[~A] == -1).all() if a.numel() == N else True, what
        assert _bits(res.centroids, ref.centroids) and _bits(res.scores.cpu()[ids], ref.scores.cpu()), what
        assert torch.equal(res.counts.cpu(), ref.counts.cpu()), what

    same(index.kmeans(Cn, iters=4, init=V, keep=Ad), "keep mask")
    same(index.kmeans(Cn, iters=4, init=V, keep=torch.nonzero(A).flatten().tolist()), "keep ids")
    index.remove(torch.nonzero(~A).flatten())
    same(index.kmeans(Cn, iters=4, init=V), "after remove")
    old_to_new = index.compact()
    res = index.kmeans(Cn, iters=4, init=V)
    assert len(index) == int(A.sum())
    same(res, "after compact", ids=torch.arange(len(index)))
    assert torch.equal(old_to_new.cpu()[A], torch.arange(len(index)))


def test_repeatable_and_isolated():
    E, N = 768, 40000
    m = _get("clip", E)
    raw = _emb(N, E, seed=31)
    q = _emb(100, E, seed=32)
    index = m.index(raw)

    def calls():
        n0 = _launches()
        out = [index.search(q, 10), index.range_search(q, 3.0), index.pairs(30.0)]
        torch.cuda.synchronize()
        return out, _launches() - n0

    before, nb = calls()
    r1 = index.kmeans(600, iters=3, seed=1)
    r2 = index.kmeans(600, iters=3, seed=1)
    after, na = calls()
    assert nb == na
    for x, y in zip(before, after):
        for s, t in zip(x, y):
            assert _bits(s.float() if s.dtype != torch.float32 else s, t.float() if t.dtype != torch.float32 else t)
    for s, t in zip(r1, r2):
        if isinstance(s, torch.Tensor):
            assert torch.equal(s.cpu().view(torch.uint8), t.cpu().view(torch.uint8))
    assert r1.iterations == r2.iterations


def test_refusals():
    from jimm_b200 import _lib as L

    E = 256
    m = _get("clip", E)
    raw = _emb(100, E, seed=41)
    raw[3] = 0
    index = m.index(raw)
    n0 = _launches()
    for kw in (dict(n_clusters=0), dict(n_clusters=65537), dict(n_clusters=True), dict(n_clusters=4, iters=0), dict(n_clusters=4, seed=-1),
               dict(n_clusters=4, init=[1, 2, 3]), dict(n_clusters=4, init=[1, 2, 3, 100]), dict(n_clusters=4, init=[1, 2, 3, -1]),
               dict(n_clusters=4, init=torch.zeros(4, E + 8)), dict(n_clusters=4, init=torch.zeros(4, E, dtype=torch.float64)),
               dict(n_clusters=4, init=torch.ones(4, dtype=torch.bool)), dict(n_clusters=4, keep=torch.ones(99, dtype=torch.bool)),
               dict(n_clusters=4, keep=[100])):
        with pytest.raises(ValueError):
            index.kmeans(**kw)
    assert _launches() == n0, "a refusal before any launch launched"
    # checked on the device: more sampled clusters than clusterable rows, a zero row as an init id, a zero init vector
    for kw in (dict(n_clusters=100), dict(n_clusters=4, init=[0, 1, 2, 3]), dict(n_clusters=4, init=torch.zeros(4, E)),
               dict(n_clusters=50, keep=torch.arange(40))):
        with pytest.raises(ValueError):
            index.kmeans(**kw)
    # both inits at the C entry point
    rc, _, _ = _kmeans_c(index, 2, 3, init_ids=torch.tensor([0, 1], dtype=torch.int32, device="cuda"), init_vectors=_emb(2, E, 1))
    assert rc == -1
    index.close()
    with pytest.raises(L.JimmError):
        index.kmeans(4)
