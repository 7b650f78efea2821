"""GPU tests of the zero-shot / classification epilogue kernel against its oracle: integer outputs (order, argmax) bit-exact
including ties, probabilities within fp32 summation error."""
import numpy as np
import pytest
import torch

import preprocess_oracle as P

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows,cols", [(1, 6), (7, 1), (5, 1000), (3, 4096), (256, 256), (2, 33)])
def test_zero_shot_matches_oracle(lib, rows, cols):
    from jimm_b200.postprocess import classify, pair_probabilities, zero_shot

    g = torch.Generator().manual_seed(rows * 31 + cols)
    x = torch.randn(rows, cols, generator=g) * 8.0
    if cols > 4:  # ties, signed zeros
        x[:, 1] = x[:, 3]
        x[0, 0], x[0, 2] = 0.0, -0.0
        x[:, cols - 1] = x.max(dim=1).values  # duplicate maximum: argmax must return the first one
    ref_p, ref_o = P.zero_shot_oracle(x.numpy())
    probs, order = zero_shot(x.cuda())
    assert np.array_equal(order.cpu().numpy(), ref_o)
    np.testing.assert_allclose(probs.cpu().numpy(), ref_p, rtol=2e-5, atol=1e-30)
    assert np.array_equal(classify(x.cuda()).cpu().numpy(), P.classify_oracle(x.numpy()))
    sig = pair_probabilities(x.cuda()).cpu().numpy()
    np.testing.assert_allclose(sig, 1.0 / (1.0 + np.exp(-x.numpy().astype(np.float64))), rtol=2e-6, atol=1e-30)


def test_overflow_strided_and_wide_input(lib):
    """The example's softmax is un-shifted: logits above ~88.7 overflow to inf and the row becomes NaN, as in the reference.  A
    column slice keeps its row stride; 5000 columns take the wide path."""
    from jimm_b200.postprocess import classify, zero_shot

    x = torch.tensor([[100.0, 1.0, 2.0], [3.0, 2.0, 1.0]])
    probs, order = zero_shot(x.cuda())
    assert torch.isnan(probs[0, 0]) and probs[0, 1] == 0
    ref_p, _ = P.zero_shot_oracle(x.numpy())
    assert np.isnan(ref_p[0, 0]) and ref_p[0, 1] == 0
    assert order.cpu().tolist() == [[0, 2, 1], [0, 1, 2]]
    big = torch.randn(4, 10).cuda()
    view = big[:, :6]  # row stride 10
    ref_p, ref_o = P.zero_shot_oracle(view.cpu().numpy())
    p2, o2 = zero_shot(view)
    assert np.array_equal(o2.cpu().numpy(), ref_o)
    np.testing.assert_allclose(p2.cpu().numpy(), ref_p, rtol=2e-5)
    wide = torch.randn(2, 5000, generator=torch.Generator().manual_seed(50)) * 8.0  # past the 4096 columns one CTA sorts
    wide[:, 4500] = wide[:, 17]  # a tie across the two sorted runs
    ref_p, ref_o = P.zero_shot_oracle(wide.numpy())
    p3, o3 = zero_shot(wide.cuda())
    assert np.array_equal(o3.cpu().numpy(), ref_o)
    np.testing.assert_allclose(p3.cpu().numpy(), ref_p, rtol=2e-5, atol=1e-30)
    assert np.array_equal(classify(wide.cuda()).cpu().numpy(), P.classify_oracle(wide.numpy()))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_wider_than_int32_refused_before_any_allocation(lib, dtype):
    """2^31 columns do not fit the int32 order: refused before the wrapper casts, copies or allocates anything.  The stride-0
    expanded input costs no memory itself, and a contiguous fp32 copy of it would take 8 GB."""
    from jimm_b200.postprocess import classify, pair_probabilities, zero_shot

    x = torch.zeros(1, dtype=dtype, device="cuda").expand(3, 2**31)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    for fn in (zero_shot, classify, pair_probabilities):
        with pytest.raises(ValueError, match="2147483647"):
            fn(x)
    assert torch.cuda.max_memory_allocated() == before
