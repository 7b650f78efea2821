"""CPU tests of the k-means reference (kmeans_oracle.py): the sampling keys, the fixed-point update and the loop."""
import numpy as np

import kmeans_oracle as ko


def test_splitmix64_known_values():
    # the first outputs of the reference splitmix64 generator seeded with 0 and with 1234567
    assert int(ko.splitmix64(0)) == 0xE220A8397B1DCDAF
    assert int(ko.splitmix64(1234567)) == 6457827717110365317
    # seed + id wraps modulo 2^64
    assert ko.sample_keys([0], 2**64 - 1)[0] == ko.sample_keys([1], 2**64 - 2)[0]


def test_sample_keys_range_and_bits():
    ids = np.arange(10000)
    k = ko.sample_keys(ids, 7)
    assert k.dtype == np.float32 and (k >= 1).all() and (k < 2).all()
    z = ko.splitmix64(np.uint64(7) + ids.astype(np.uint64))
    assert np.array_equal(k.astype(np.float64), 1 + (z >> np.uint64(41)).astype(np.float64) * 2.0**-23)
    assert len(np.unique(k)) > 9900


def test_sample_ties_to_larger_position():
    keys = np.array([1.5, 1.25, 1.5, 1.75, 1.25], dtype=np.float32)
    assert ko.top_k_positions(keys, 5).tolist() == [3, 2, 0, 4, 1]
    ids = np.array([3, 8, 20, 21, 40])
    got = ko.sample_init(ids, 11, 3)
    assert len(set(got.tolist())) == 3 and set(got.tolist()) <= set(ids.tolist())


def test_fixed_point_mean_against_float64():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((5000, 64)) / 8).astype(np.float32)
    a = rng.integers(0, 7, 5000)
    S, n = ko.fixed_sums(x, a, 7)
    for j in range(7):
        ref = x[a == j].astype(np.float64).mean(axis=0)
        pre = S[j].astype(np.float64) * 2.0**-30 / n[j]
        assert np.abs(pre - ref).max() <= 2.0**-30  # each term rounds by at most 2^-31, so the mean errs by at most that
    # values that are multiples of 2^-30 sum exactly
    q = rng.integers(-(2**23), 2**23, (300, 16)).astype(np.float64) * 2.0**-30
    xq = q.astype(np.float32)
    assert np.array_equal(xq.astype(np.float64), q)
    S, n = ko.fixed_sums(xq, np.zeros(300, dtype=np.int64), 1)
    assert np.array_equal(S[0], np.rint(q * 2.0**30).astype(np.int64).sum(axis=0))
    m = ko.means(S, n, np.zeros((1, 16), np.float32))
    assert np.array_equal(m[0], (q.sum(axis=0) / 300).astype(np.float32))


def test_rint_ties_to_even():
    x = np.array([[2.0**-31, 3 * 2.0**-31, -(2.0**-31)]], dtype=np.float32)
    S, _ = ko.fixed_sums(x, np.zeros(1, dtype=np.int64), 1)
    assert S[0].tolist() == [0, 2, 0]


def test_overflow_bound_at_two():
    # |x| <= 2: each term is at most 2^31, so even 2^31 - 1 rows of 2 stay below 2^62 < 2^63
    x = np.full((4, 8), 2.0, dtype=np.float32)
    x[1] = -2.0
    S, n = ko.fixed_sums(x, np.zeros(4, dtype=np.int64), 1)
    assert S[0].tolist() == [2**32] * 8 and n[0] == 4
    assert (2**31 - 1) * 2**31 < 2**62


def test_keep_previous_rules():
    m = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float32)
    c = ko.normalize64(m)
    v = np.array([0.6, 0.8, 0.0], dtype=np.float32)
    x = np.stack([v, -v, np.array([0, 0.6, 0.8], np.float32)])
    a = np.array([0, 0, 1])  # cluster 0's mean is exactly zero, cluster 2 is empty
    m_new, c_new = ko.update(x, a, m, c, ko.normalize64)
    assert np.array_equal(m_new[0], m[0]) and np.array_equal(c_new[0], c[0])
    assert np.array_equal(m_new[2], m[2]) and np.array_equal(c_new[2], c[2])
    assert np.array_equal(m_new[1], x[2])


def test_loop_on_separated_data():
    rng = np.random.default_rng(3)
    centres = ko.normalize64(rng.standard_normal((5, 32)).astype(np.float32))
    lab = rng.integers(0, 5, 400)
    x = ko.normalize64(centres[lab] + 0.05 * rng.standard_normal((400, 32)).astype(np.float32))
    init = np.array([np.flatnonzero(lab == j)[0] for j in range(5)])
    c, a, s, it = ko.kmeans(x, x[init], 20, ko.normalize64, ko.assign64)
    assert np.array_equal(a, lab) and it == 2
    assert np.array_equal(ko.assign64(x, c)[0], a)
    # iters = 1: the initial centroids only
    c1, a1, _, it1 = ko.kmeans(x, x[init], 1, ko.normalize64, ko.assign64)
    assert it1 == 1 and np.array_equal(c1, ko.normalize64(x[init]))
    # large margins: the fixed-point loop reaches the same assignment as one in float64 throughout
    m = x[init].astype(np.float64)
    for _ in range(3):
        cc = m / np.linalg.norm(m, axis=1, keepdims=True)
        aa = np.argmax(x.astype(np.float64) @ cc.T, axis=1)
        m = np.stack([x[aa == j].astype(np.float64).mean(axis=0) for j in range(5)])
    assert np.array_equal(aa, a)


def test_duplicate_init_larger_cluster_takes_ties():
    x = ko.normalize64(np.array([[1, 0], [0.9, 0.1], [0, 1]], dtype=np.float32))
    _, a, _, _ = ko.kmeans(x, x[[0, 0, 2]], 1, ko.normalize64, ko.assign64)
    assert a.tolist() == [1, 1, 2]
    c, _, _, _ = ko.kmeans(x, x[[0, 0, 2]], 2, ko.normalize64, ko.assign64)
    assert np.array_equal(c[0], ko.normalize64(x[[0]])[0])  # cluster 0 was empty and kept its centroid
