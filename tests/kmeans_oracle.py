"""Reference of GalleryIndex.kmeans in numpy: the initial sampling, the fixed-point update and the loop around them, with the normalise and
assignment steps passed in (the GPU tests pass the library's own hooks, the CPU tests float64 numpy).

Definition (INTEGRATION.md, "Clustering (k-means)"):
  * keys: 1 + (splitmix64(seed + id) >> 41) * 2^-23 for the clusterable rows' ascending ids; cluster j starts from the row at the j-th
    position of top_k(keys, C), equal keys to the larger position first.
  * update: S_j[e] = sum over the rows of cluster j of rint(x[e] * 2^30) in int64; m_j = fp32(fp64(S_j) * 2^-30 / fp64(n_j)); a cluster
    with no rows, or whose new mean normalises to a non-finite row, keeps its previous mean and centroid.
  * loop: c_t = normalize(m_t); a_t = assign(x, c_t); stop when t + 1 == iters or t > 0 and a_t == a_{t-1}."""
import numpy as np

MASK64 = (1 << 64) - 1


def splitmix64(x):
    """The first output of splitmix64 with state x (uint64 array or int): the mix of x + 0x9e3779b97f4a7c15."""
    z = (np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def sample_keys(ids, seed: int):
    """float32 keys in [1, 2) of the clusterable rows ids (ascending)."""
    ids = np.asarray(ids, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = splitmix64(np.uint64(seed & MASK64) + ids)
    m = (z >> np.uint64(41)).astype(np.uint32)
    return (np.uint32(0x3F800000) | m).view(np.float32)


def top_k_positions(keys, C: int):
    """The first C positions of keys in descending order, equal keys larger position first (top_k's order)."""
    pos = np.arange(keys.size)
    return np.lexsort((-pos, -keys.astype(np.float64)))[:C]


def sample_init(ids, seed: int, C: int):
    """Row ids of the sampled initial means."""
    ids = np.asarray(ids)
    return ids[top_k_positions(sample_keys(ids, seed), C)]


def fixed_sums(x, assign, C: int):
    """S int64 [C, E] and n int64 [C] of the rows x (float32 [n, E], |x| <= 2) assigned to each cluster."""
    q = np.rint(x.astype(np.float64) * 2.0**30).astype(np.int64)
    S = np.zeros((C, x.shape[1]), dtype=np.int64)
    np.add.at(S, assign, q)
    n = np.bincount(assign, minlength=C).astype(np.int64)
    return S, n


def means(S, n, m_old):
    """fp32(fp64(S) * 2^-30 / n) for the clusters with rows, m_old for the others."""
    m = m_old.copy()
    has = n > 0
    m[has] = (S[has].astype(np.float64) * 2.0**-30 / n[has, None].astype(np.float64)).astype(np.float32)
    return m


def update(x, assign, m, c, normalize):
    """m_{t+1} and c_{t+1} from the assignment: a cluster with no rows or a non-finite new centroid keeps m_t and c_t."""
    C = m.shape[0]
    S, n = fixed_sums(x, assign, C)
    m_new = means(S, n, m)
    c_new = normalize(m_new)
    bad = ~np.isfinite(c_new).all(axis=1)
    m_new[bad], c_new[bad] = m[bad], c[bad]
    return m_new, c_new


def kmeans(x, m0, iters: int, normalize, assign_fn):
    """The loop on the clusterable rows x (float32 [n, E]) from the initial means m0 (float32 [C, E]): (centroids, assign, scores,
    iterations).  normalize(m) -> float32 rows; assign_fn(x, c) -> (int cluster [n], float32 score [n])."""
    m = np.asarray(m0, dtype=np.float32).copy()
    c = normalize(m)
    if not np.isfinite(c).all():
        raise ValueError("initial centroids with a non-finite l2_normalize")
    prev = None
    for t in range(iters):
        a, s = assign_fn(x, c)
        if t + 1 == iters or (t > 0 and np.array_equal(a, prev)):
            return c, a, s, t + 1
        m, c = update(x, a, m, c, normalize)
        prev = a
    raise AssertionError("unreachable")


def normalize64(m):
    """l2_normalize in float64, rounded to float32: the CPU tests' stand-in for the kernel."""
    m64 = m.astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (m64 / np.sqrt((m64 * m64).sum(axis=1, keepdims=True))).astype(np.float32)


def assign64(x, c):
    """Best cluster by float64 cosine, equal scores to the larger cluster: the CPU tests' stand-in for the screened search."""
    s = x.astype(np.float64) @ c.astype(np.float64).T
    a = s.shape[1] - 1 - np.argmax(s[:, ::-1], axis=1)
    return a.astype(np.int32), s[np.arange(s.shape[0]), a].astype(np.float32)
