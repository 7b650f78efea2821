"""CPU tests of the SigLIP 2 NaFlex front-end's host side: the library's size rule (jimm_preproc_naflex_grid) against transformers'
get_image_size_for_max_num_patches, its refusals, and the NaFlex oracle (tests/naflex_preprocess_oracle.py) against
Siglip2ImageProcessorPil and the committed fixture."""
import os

import numpy as np
import pytest

import naflex_preprocess_oracle as NP
import preprocess_oracle as PO

BUDGETS = (1, 16, 64, 196, 256, 576, 784, 1024, 4096)
# the frames of the front-end's checks: upscaling and downscaling, strips, camera sizes
FRAMES = [(480, 640), (17, 3000), (1000, 1000), (224, 224), (16, 16), (7, 9), (1080, 1920), (333, 77), (1, 1), (1, 30000), (30000, 1),
          (2160, 3840), (3000, 4000)]


def _grid(lib, patch, n, h, w):
    import ctypes as C

    gh, gw = C.c_int(), C.c_int()
    rc = lib.jimm_preproc_naflex_grid(patch, n, h, w, C.byref(gh), C.byref(gw))
    return rc, (gh.value, gw.value)


def test_size_rule_matches_hf(lib):
    from transformers.models.siglip2.image_processing_pil_siglip2 import get_image_size_for_max_num_patches as hf_size

    # every pair at one budget and both patch sizes; the first 2000 at every budget
    rng = np.random.default_rng(2024)
    # half uniform over 1 .. 20000 per edge, half log-uniform (small frames and strips)
    uni = rng.integers(1, 20001, size=(10000, 2))
    log = np.exp(rng.uniform(0, np.log(20000), size=(10000, 2))).astype(np.int64).clip(1, 20000)
    pairs = np.concatenate([uni, log])
    assert len(pairs) >= 20000
    for i, (h, w) in enumerate(pairs.tolist()):
        for patch in (14, 16):
            n = BUDGETS[(i + patch) % len(BUDGETS)] if i >= 2000 else None
            for n in ([n] if n is not None else BUDGETS):
                th, tw = hf_size(h, w, patch, n)
                assert NP.naflex_size(h, w, patch, n) == (th, tw)
                rc, g = _grid(lib, patch, n, h, w)
                if (th // patch) * (tw // patch) > n:
                    assert rc == -1, (h, w, patch, n)
                else:
                    assert rc == 0 and g == (th // patch, tw // patch), (h, w, patch, n, g, th, tw)


def test_size_rule_refusals(lib):
    from transformers.models.siglip2.image_processing_pil_siglip2 import get_image_size_for_max_num_patches as hf_size

    assert _grid(lib, 0, 256, 100, 100)[0] == -1
    assert "patch size" in lib.jimm_last_error().decode()
    assert _grid(lib, 16, 0, 100, 100)[0] == -1
    assert "max_num_patches" in lib.jimm_last_error().decode()
    for h, w in ((0, 10), (10, 0), (-1, 5)):
        assert _grid(lib, 16, 256, h, w)[0] == -1
    # H x W x 3 of 2^31 bytes or more: refused; one byte less: accepted
    assert _grid(lib, 16, 256, 2, (2 ** 31) // 6 + 1)[0] == -1
    assert "2^31" in lib.jimm_last_error().decode()
    assert _grid(lib, 16, 256, 1, (2 ** 31 - 1) // 3)[0] == 0
    # the processor's grid of a 1 x 100,000,000 strip at 4 patches is 1 x 7: refused, naming the grid
    th, tw = hf_size(1, 100_000_000, 16, 4)
    assert (th // 16, tw // 16) == (1, 7)
    assert _grid(lib, 16, 4, 1, 100_000_000)[0] == -1
    assert "1x7" in lib.jimm_last_error().decode()
    assert _grid(lib, 16, 4, 100_000_000, 1)[0] == -1


@pytest.mark.parametrize("n", [64, 256, 1024])
def test_oracle_matches_siglip2_processor(n):
    proc = NP.hf_processor(16, n)
    cfg = NP.siglip2_config()
    imgs = [PO.synthetic_u8_images(1, h, w, seed=11 + i)[0] for i, (h, w) in enumerate(FRAMES)]
    for i, img in enumerate(imgs):
        pv, mask, shapes = NP.hf_batch(proc, [img])
        opv, omask, oshapes = NP.naflex_batch([img], 16, n, cfg)
        assert np.array_equal(shapes, oshapes), (FRAMES[i], shapes, oshapes)
        assert np.array_equal(mask, omask), FRAMES[i]
        assert pv.dtype == np.float32 and np.array_equal(pv, opv), FRAMES[i]


def test_oracle_matches_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "preprocess_siglip2_naflex.npz"))
    P = int(z["patch"])
    imgs = [z[f"img{i}"] for i in range(len([k for k in z.files if k.startswith("img")]))]
    for n in z["max_num_patches"].tolist():
        pv, mask, shapes = NP.naflex_batch(imgs, P, n, NP.siglip2_config())
        assert np.array_equal(pv, z[f"pixel_values_{n}"])
        assert np.array_equal(mask, z[f"pixel_attention_mask_{n}"])
        assert np.array_equal(shapes, z[f"spatial_shapes_{n}"])
    assert z["pixel_attention_mask_16"].min() == 0 and z["pixel_attention_mask_64"].min() == 0  # the fixture has padding rows
