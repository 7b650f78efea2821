"""CPU: the input step of a text call on a list of token sequences (prep_texts) -- concatenation, offsets, dtypes, the [1, L] form and
every refusal, all before any handle exists."""

import numpy as np
import pytest
import torch

from jimm_b200._runtime import Texts, prep_texts

CTX = 77


def test_concatenates_in_order_as_int32():
    seqs = [torch.tensor([49406, 320, 49407]), np.array([1, 2], dtype=np.int64), [5, 6, 7, 8], torch.tensor([[9]], dtype=torch.int16)]
    t = prep_texts(seqs, CTX)
    assert isinstance(t, Texts)
    assert t.lens == [3, 2, 4, 1]
    assert t.ids.dtype == torch.int32 and t.ids.is_contiguous() and t.ids.ndim == 1
    assert t.ids.tolist() == [49406, 320, 49407, 1, 2, 5, 6, 7, 8, 9]
    assert t.host
    off = np.concatenate([[0], np.cumsum(t.lens)])
    for i, s in enumerate(seqs):
        assert t.ids[off[i]:off[i + 1]].tolist() == torch.as_tensor(np.asarray(s)).reshape(-1).tolist()


def test_tuple_uint8_numpy_int32_and_the_bounds():
    t = prep_texts((np.arange(CTX, dtype=np.int32), torch.tensor([7], dtype=torch.uint8)), CTX)
    assert t.lens == [CTX, 1]
    assert t.ids.tolist() == list(range(CTX)) + [7]


def test_out_of_range_ids_pass_through():
    # the embedding clamps them on the GPU, as the [B, T] call does
    t = prep_texts([[-5, 100000]], CTX)
    assert t.ids.tolist() == [-5, 100000]


def test_empty_list():
    t = prep_texts([], CTX)
    assert t.lens == [] and t.ids.numel() == 0 and t.ids.dtype == torch.int32 and t.host


@pytest.mark.parametrize("bad, match", [
    ([torch.tensor([1, 2]), torch.tensor([], dtype=torch.int64)], "sequence 1 of the list: length 0"),
    ([[]], "length 0"),
    ([torch.arange(CTX + 1)], f"length {CTX + 1} outside 1 .. context_length={CTX}"),
    ([torch.zeros((2, 3), dtype=torch.int64)], r"shape \[length\] or \[1, length\], got \(2, 3\)"),
    ([torch.zeros((1, 1, 3), dtype=torch.int64)], r"got \(1, 1, 3\)"),
    ([torch.tensor(3)], r"got \(\)"),
    ([torch.tensor([1.0, 2.0])], "must be integers, got torch.float32"),
    ([np.array([1.5])], "must be integers"),
    ([torch.tensor([True, False])], "must be integers, got torch.bool"),
    ([torch.tensor([1, 2], device="meta"), torch.tensor([1, 2])], "one device"),
])
def test_refusals(bad, match):
    with pytest.raises(ValueError, match=match):
        prep_texts(bad, CTX)


def test_refused_before_a_handle_is_built(monkeypatch):
    """The model classes run the input step before they build (or rebuild) their native handle."""
    from jimm_b200.common.vit import _NativeOwner
    from jimm_b200.models import CLIP, SigLIP

    def no_build(self, mb):
        raise AssertionError("a handle was built")

    monkeypatch.setattr(_NativeOwner, "_build_native", no_build)
    for cls in (CLIP, SigLIP):
        m = cls(32, 1, 64, 16, 16, 100, 64, 1, 1)
        with pytest.raises(ValueError, match="length 17 outside"):
            m.encode_text([torch.arange(3), torch.arange(17)])
        with pytest.raises(ValueError, match="length 0"):
            m(torch.zeros((1, 32, 32, 3)), [torch.arange(3), []])
