"""GPU tests of the zero-shot / classification epilogue at the widths real label and caption counts reach: an ImageNet-21k head
(21843 classes), COCO's 25000 captions, a gallery of 2^20 embeddings.  Rows wider than 4096 columns are sorted as 4096-key runs
merged in global memory; the values below put ties, signed zeros, NaN and infinities on both sides of the run boundaries the merge
has to join.  Order and argmax are bit-exact against numpy (stable argsort reversed, first maximum); probabilities within the
suite's bars: softmax rtol 2e-5 against the fp64-summed oracle, sigmoid rtol 2e-6 against fp64."""
import numpy as np
import pytest
import torch

import preprocess_oracle as P

pytestmark = pytest.mark.gpu

RUN = 4096  # columns per shared-memory run of the wide path
WIDTHS = [4095, 4096, 4097, 8191, 8192, 8193, 21843, 25000, 65537]
NAN, INF = float("nan"), float("inf")


def _spots(cols):
    """Three column positions each in the first run, a middle run and the last run (the same run below three runs; positions past
    a narrow row wrap around)."""
    mid = (cols // RUN // 2) * RUN
    return [tuple(p % cols for p in s) for s in [(3, 100, min(RUN, cols) - 1), (mid, mid + 7, mid + 2000), (cols - 1, cols - 5, cols - 300)]]


def _row(pattern, cols, rng):
    """One fp32 row of `cols` values following `pattern`; every pattern is defined at every width from 1 column on."""
    x = (rng.standard_normal(cols) * 8).astype(np.float32)
    if pattern == "randn":
        pass
    elif pattern == "levels":  # 16 distinct values: every run boundary splits ties
        x = ((rng.integers(0, 16, cols) - 8) * 0.75).astype(np.float32)
    elif pattern == "equal":
        x[:] = 0.25
    elif pattern == "ascending":
        x.sort()
    elif pattern == "descending":
        x = np.sort(x)[::-1].copy()
    elif pattern == "signed_zero":  # +0 / -0 interleaved in two different runs, and around the first run boundary
        for lo, hi in ((50, RUN - 50), (cols - RUN + 40, cols), (RUN - 20, min(RUN + 20, cols))):
            idx = np.arange(max(lo, 0), min(hi, cols), 3)
            x[idx] = np.where(np.arange(idx.size) % 2 == 0, 0.0, -0.0).astype(np.float32)
    elif pattern == "nonfinite":  # NaN (both signs), +inf and -inf in the first, a middle and the last run
        for a, b, c in _spots(cols):
            x[a], x[b], x[c] = NAN, INF, -INF
        x[(_spots(cols)[1][0] + 1) % cols] = -NAN
        x[(cols - 2) % cols] = INF
    elif pattern == "dup_max":  # the maximum in the first and the last run: argmax is the first copy
        m = x.max() + 1.0
        x[[11 % cols, (cols - 2) % cols]] = m
    elif pattern == "all_nan":
        x[:] = NAN
    else:
        raise AssertionError(pattern)
    return x


PATTERNS = ["randn", "levels", "equal", "ascending", "descending", "signed_zero", "nonfinite", "dup_max", "all_nan"]


def _matrix(rows, cols, patterns, seed):
    rng = np.random.default_rng(seed)
    return np.stack([_row(patterns[r % len(patterns)], cols, rng) for r in range(rows)])


def _check(x, what=""):
    """zero_shot, classify and pair_probabilities of the [rows, cols] fp32 array x against the oracles."""
    from jimm_b200.postprocess import classify, pair_probabilities, zero_shot

    xd = torch.from_numpy(x).cuda()
    probs, order = zero_shot(xd)
    amax = classify(xd)
    sig = pair_probabilities(xd)
    ref_p, ref_o = P.zero_shot_oracle(x)
    o = order.cpu().numpy()
    bad = np.nonzero((o != ref_o).any(axis=1))[0]
    assert bad.size == 0, f"{what}: order differs in rows {bad[:8].tolist()}, first column {int(np.argmax(o[bad[0]] != ref_o[bad[0]]))}"
    assert np.array_equal(amax.cpu().numpy(), P.classify_oracle(x)), what
    np.testing.assert_allclose(probs.cpu().numpy(), ref_p, rtol=2e-5, atol=1e-30, err_msg=what)
    with np.errstate(over="ignore"):
        ref_s = 1.0 / (1.0 + np.exp(-x.astype(np.float64)))
    np.testing.assert_allclose(sig.cpu().numpy(), ref_s, rtol=2e-6, atol=1e-30, err_msg=what)
    return probs, order, amax


@pytest.mark.parametrize("cols", WIDTHS)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_pattern_at_width(lib, pattern, cols):
    """Three rows of one pattern (each its own draw) at each width around and beyond one run."""
    _check(_matrix(3, cols, [pattern], seed=cols * 17 + PATTERNS.index(pattern)), f"{pattern} [3, {cols}]")


@pytest.mark.parametrize("cols", WIDTHS)
@pytest.mark.parametrize("rows", [1, 64])
def test_rows_at_width(lib, rows, cols):
    """1 and 64 rows at each width, the rows cycling through every pattern (64 rows: each pattern seven times over)."""
    pats = PATTERNS if rows > 1 else [PATTERNS[WIDTHS.index(cols) % len(PATTERNS)]]
    _check(_matrix(rows, cols, pats, seed=rows * 1000 + cols), f"[{rows}, {cols}]")


@pytest.mark.parametrize("pattern", ["randn", "levels", "nonfinite", "signed_zero"])
def test_one_row_of_2pow20_plus_3(lib, pattern):
    """A gallery of 2^20 + 3 embeddings: nine merge passes, the last run three columns long."""
    _check(_matrix(1, 2**20 + 3, [pattern], seed=20), pattern)


def test_retrieval_score_matrix(lib):
    """256 queries against 25000 captions: 100 x cosine similarity of unit embeddings, CLIP's logit scale."""
    g = torch.Generator().manual_seed(5)
    q = torch.nn.functional.normalize(torch.randn(256, 64, generator=g), dim=-1)
    c = torch.nn.functional.normalize(torch.randn(25000, 64, generator=g), dim=-1)
    c[12345] = c[7]  # a duplicated caption: equal scores in two different runs of every row
    _check((100.0 * q @ c.T).numpy(), "retrieval [256, 25000]")


@pytest.mark.parametrize("cols", [1, 2, 31, 32, 33, 255, 256, 257, 1000, 2048, 2049, 4000])
def test_narrow_widths(lib, cols):
    """At most 4096 columns the row is sorted in its own CTA's shared memory, as before the wide path existed."""
    _check(_matrix(9, cols, PATTERNS, seed=cols), f"[9, {cols}]")


def test_argmax_of_a_21k_class_vit(lib):
    """classify(model(images)) on an ImageNet-21k-sized head equals the oracle's argmax of the same logits."""
    import jimm_oracle as O
    from jimm_b200.models import VisionTransformer
    from jimm_b200.postprocess import classify

    kw = dict(num_classes=21843, img_size=32, patch_size=16, num_layers=1, num_heads=2, mlp_dim=256, hidden_size=128)
    m = VisionTransformer(**kw, dtype=torch.float16).eval()
    for k, v in O.random_vit_params(O.ViTCfg(**kw), seed=3).items():
        m.set_flat_param(k, v)
    logits = m(torch.randn(6, 32, 32, 3, generator=torch.Generator().manual_seed(4)).cuda())
    assert logits.shape == (6, 21843)
    assert np.array_equal(classify(logits).cpu().numpy(), P.classify_oracle(logits.float().cpu().numpy()))


def test_input_forms(lib):
    """A column slice (ld > cols), a transposed tensor, a stride-0 expanded tensor and 16-bit logits: each the oracle's answer on the
    fp32 values the call sees."""
    from jimm_b200.postprocess import classify, zero_shot

    def same(xd, what):
        ref_p, ref_o = P.zero_shot_oracle(xd.float().cpu().numpy())
        probs, order = zero_shot(xd)
        assert np.array_equal(order.cpu().numpy(), ref_o), what
        assert np.array_equal(classify(xd).cpu().numpy(), P.classify_oracle(xd.float().cpu().numpy())), what
        np.testing.assert_allclose(probs.cpu().numpy(), ref_p, rtol=2e-5, atol=1e-30, err_msg=what)

    base = torch.from_numpy(_matrix(3, 30000, ["levels", "randn", "nonfinite"], seed=9)).cuda()
    same(base[:, 1234:26234], "column slice, ld 30000 > cols 25000")
    same(torch.from_numpy(_matrix(3, 25000, ["randn"], seed=10)).cuda().T.contiguous().T, "transposed")
    same(torch.from_numpy(_matrix(25000, 3, ["levels"], seed=11)).cuda().T, "transposed view [3, 25000]")
    one = torch.from_numpy(_matrix(1, 25000, ["levels"], seed=12)).cuda()
    same(one.expand(4, 25000), "stride-0 expanded rows")
    same(one[0].expand(5, 25000), "stride-0 expanded 1-D row")
    f = torch.from_numpy(_matrix(3, 21843, ["randn", "dup_max", "nonfinite"], seed=13)).cuda()
    same(f.half(), "fp16 logits")
    same(f.bfloat16(), "bf16 logits")


def test_non_default_stream(lib):
    """A call on a side stream gives the default stream's bits."""
    from jimm_b200.postprocess import classify, zero_shot

    x = torch.from_numpy(_matrix(8, 25000, PATTERNS, seed=14)).cuda()
    p0, o0 = zero_shot(x)
    a0 = classify(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        p1, o1 = zero_shot(x)
        a1 = classify(x)
    s.synchronize()
    assert torch.equal(p0.view(torch.int32), p1.view(torch.int32))
    assert torch.equal(o0, o1) and torch.equal(a0, a1)


@pytest.mark.parametrize("poison", ["nan", "inf"])
def test_poisoned_row_leaves_the_others(lib, poison):
    """[4, 21843]: a row of NaN or inf changes no other row's order, argmax or probabilities."""
    from jimm_b200.postprocess import classify, zero_shot

    clean = torch.from_numpy(_matrix(4, 21843, ["levels", "randn", "signed_zero", "dup_max"], seed=15)).cuda()
    x = clean.clone()
    x[2] = NAN if poison == "nan" else INF
    x[1, 20000] = -INF if poison == "inf" else NAN  # and one more poisoned element in another row
    pc, oc = zero_shot(clean)
    ac = classify(clean)
    px, ox = zero_shot(x)
    ax = classify(x)
    keep = [0, 3]
    assert torch.equal(px[keep].view(torch.int32), pc[keep].view(torch.int32))
    assert torch.equal(ox[keep], oc[keep]) and torch.equal(ax[keep], ac[keep])
    assert bool(torch.isnan(px[2]).all())
    ref_p, ref_o = P.zero_shot_oracle(x.cpu().numpy())
    assert np.array_equal(ox.cpu().numpy(), ref_o)
    assert np.array_equal(ax.cpu().numpy(), P.classify_oracle(x.cpu().numpy()))
