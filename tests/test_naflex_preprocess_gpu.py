"""GPU: the SigLIP 2 NaFlex image front-end (jimm_preproc_run_naflex) -- device-built tables against make_table, frames from 1x1 to 8K
and strips against the CPU oracle (bit-exact fp32, RNE fp16 / bf16) on every path the planner reports, ragged calls against each frame
alone, two streams on one handle, refusals that enqueue nothing, and the model fed by it on the tiny_siglip2_naflex fixture."""
import ctypes as C
import os
import random
import threading

import numpy as np
import pytest
import torch

import naflex_preprocess_oracle as NP
import preprocess_oracle as PO
from gpu_util import check_parity

pytestmark = pytest.mark.gpu
F32, F16, BF16 = 0, 1, 2
FRAMES = [(1, 1), (7, 9), (16, 16), (224, 224), (333, 77), (480, 640), (1080, 1920), (2160, 3840), (3024, 4032), (7680, 4320),
          (1, 30000), (30000, 1)]
BUDGETS = (64, 256, 1024)


@pytest.fixture(scope="module")
def frames():
    return {hw: PO.synthetic_u8_images(1, *hw, seed=hw[0] * 7 + hw[1])[0] for hw in FRAMES}


def _front_end(patch):
    from jimm_b200.preprocess import NaFlexPreprocessor

    return NaFlexPreprocessor(patch_size=patch)


def _raw(pre, ptrs, H, W, N, pv, code, mask, grid=None, stream=None):
    """jimm_preproc_run_naflex on explicit pointers; returns the status."""
    B = len(ptrs)
    st = stream if stream is not None else torch.cuda.current_stream()
    return pre.lib.jimm_preproc_run_naflex(pre.handle, (C.c_void_p * max(B, 1))(*ptrs), B, (C.c_int * max(B, 1))(*H),
                                           (C.c_int * max(B, 1))(*W), N, C.c_void_p(pv), code, C.c_void_p(mask), grid,
                                           C.c_void_p(st.cuda_stream))


def test_device_tables_equal_make_table(frames):
    from jimm_b200.preprocess import naflex_grid, resample_coeffs, resample_coeffs_device

    pairs = set()
    for h, w in FRAMES:
        for P in (16, 14, 4):
            for n in BUDGETS:
                gh, gw = naflex_grid(h, w, P, n)
                pairs |= {(h, gh * P), (w, gw * P)}
    for resample in (PO.BILINEAR, PO.BICUBIC):
        for i, o in sorted(pairs):
            ref = resample_coeffs(i, o, resample)
            got = resample_coeffs_device(i, o, resample)
            for a, b in zip(ref, got):
                assert np.array_equal(a, b), (i, o, resample)


def test_planner_paths_covered():
    """Every path the planner gives the frames below at the budgets below -- the three fused tiers and the two-pass path -- occurs."""
    from jimm_b200.preprocess import naflex_grid, plan

    seen = {}
    for h, w in FRAMES:
        for P in (16, 14, 4):
            for n in BUDGETS:
                gh, gw = naflex_grid(h, w, P, n)
                path, tier, _, _ = plan(h, w, size={"height": gh * P, "width": gw * P}, resample=PO.BILINEAR)
                seen.setdefault((path, tier), (h, w, P, n))
    assert {(0, 0), (0, 1), (0, 2), (1, -1)} <= set(seen), seen


@pytest.mark.parametrize("P", [16, 14, 4])
def test_frames_match_oracle(frames, P):
    pre = _front_end(P)
    cfg = NP.siglip2_config()
    imgs = [frames[hw] for hw in FRAMES]
    for n in BUDGETS:
        ref_pv, ref_mask, ref_shapes = NP.naflex_batch(imgs, P, n, cfg)
        out = {}
        for dt in (torch.float32, torch.float16, torch.bfloat16):
            r = pre([torch.from_numpy(i).cuda() for i in imgs], dtype=dt, max_num_patches=n)
            assert r["pixel_values"].dtype == dt and r["spatial_shapes"].device.type == "cpu" and r["spatial_shapes"].dtype == torch.int64
            assert torch.equal(r["spatial_shapes"], torch.from_numpy(ref_shapes)), (P, n)
            assert torch.equal(r["pixel_attention_mask"].cpu(), torch.from_numpy(ref_mask)), (P, n)
            out[dt] = r["pixel_values"]
        f32 = out[torch.float32].cpu()
        for b, hw in enumerate(FRAMES):
            assert torch.equal(f32[b], torch.from_numpy(ref_pv[b])), (hw, P, n)  # padding rows included: exactly zero
        for dt in (torch.float16, torch.bfloat16):
            assert torch.equal(out[dt].cpu(), f32.to(dt)), (dt, P, n)


def test_ragged_call_equals_each_frame_alone(frames):
    """A list call equals each frame alone, bit for bit: fused and two-pass frames mixed, repeats, any order, frame pointers at every
    byte offset modulo 16."""
    P, n = 16, 1024
    pre = _front_end(P)
    sizes = [(2160, 3840), (480, 640), (1080, 1920), (333, 77), (2160, 3840), (3024, 4032), (7, 9), (1, 30000), (480, 640)]
    alone = {hw: pre([frames[hw]], dtype=torch.float16, max_num_patches=n) for hw in set(sizes)}
    for trial in range(3):
        order = sizes[:]
        random.Random(trial).shuffle(order)
        # every frame at its own misalignment inside one byte buffer
        offs, total = [], 0
        for k, hw in enumerate(order):
            total += (k * 5 + trial + 1) % 16
            offs.append(total)
            total += frames[hw].size
        buf = torch.zeros(total + 16, dtype=torch.uint8, device="cuda")
        for o, hw in zip(offs, order):
            buf[o:o + frames[hw].size] = torch.from_numpy(frames[hw].reshape(-1)).cuda()
        N, K = n, P * P * 3
        pv = torch.full((len(order), N, K), float("nan"), dtype=torch.float16, device="cuda")
        mask = torch.full((len(order), N), -1, dtype=torch.int32, device="cuda")
        grid = (C.c_int * (2 * len(order)))()
        rc = _raw(pre, [buf.data_ptr() + o for o in offs], [h for h, _ in order], [w for _, w in order], n, pv.data_ptr(), F16,
                  mask.data_ptr(), grid)
        assert rc == 0, pre.lib.jimm_last_error()
        for b, hw in enumerate(order):
            assert torch.equal(pv[b], alone[hw]["pixel_values"][0]), (trial, b, hw)
            assert torch.equal(mask[b], alone[hw]["pixel_attention_mask"][0])
            assert (grid[2 * b], grid[2 * b + 1]) == tuple(alone[hw]["spatial_shapes"][0].tolist())


def test_two_streams_on_one_handle(frames):
    P, n = 16, 256
    pre = _front_end(P)
    lists = [[frames[hw] for hw in ((480, 640), (2160, 3840), (333, 77))], [frames[hw] for hw in ((1080, 1920), (7680, 4320), (1, 1))]]
    ref = [pre(x, dtype=torch.bfloat16) for x in lists]
    dev = [[torch.from_numpy(f).cuda() for f in x] for x in lists]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    res = [[None] * 4, [None] * 4]

    def drive(k):
        with torch.cuda.stream(streams[k]):
            for it in range(4):
                res[k][it] = pre(dev[k], dtype=torch.bfloat16)

    threads = [threading.Thread(target=drive, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    for k in range(2):
        for r in res[k]:
            assert torch.equal(r["pixel_values"], ref[k]["pixel_values"])
            assert torch.equal(r["pixel_attention_mask"], ref[k]["pixel_attention_mask"])


def test_refusals_enqueue_nothing():
    from jimm_b200 import _lib
    from jimm_b200.preprocess import ImagePreprocessor

    P, n = 16, 64
    pre = _front_end(P)
    img = torch.zeros((64, 64, 3), dtype=torch.uint8, device="cuda")
    pv = torch.full((2, n, P * P * 3), float("nan"), device="cuda")
    pv16 = torch.full((2, n, P * P * 3 + 4), float("nan"), dtype=torch.float16, device="cuda")
    mask = torch.full((2, n + 1), -7, dtype=torch.int32, device="cuda")
    p0 = img.data_ptr()
    cases = {
        "null frame pointer": ([p0, 0], [64, 64], [64, 64], n, pv.data_ptr(), F32, mask.data_ptr()),
        "null pixel_values": ([p0, p0], [64, 64], [64, 64], n, 0, F32, mask.data_ptr()),
        "bad dtype": ([p0, p0], [64, 64], [64, 64], n, pv.data_ptr(), 7, mask.data_ptr()),
        "misaligned fp32 output": ([p0, p0], [64, 64], [64, 64], n, pv.data_ptr() + 4, F32, mask.data_ptr()),
        "misaligned fp16 output": ([p0, p0], [64, 64], [64, 64], n, pv16.data_ptr() + 2, F16, mask.data_ptr()),
        "misaligned mask": ([p0, p0], [64, 64], [64, 64], n, pv.data_ptr(), F32, mask.data_ptr() + 2),
        "max_num_patches 0": ([p0, p0], [64, 64], [64, 64], 0, pv.data_ptr(), F32, mask.data_ptr()),
        "empty frame": ([p0, p0], [64, 0], [64, 64], n, pv.data_ptr(), F32, mask.data_ptr()),
        "2^31-byte frame": ([p0, p0], [64, 2], [64, 2 ** 30], n, pv.data_ptr(), F32, mask.data_ptr()),
        "strip past the budget": ([p0, p0], [64, 1], [64, 100_000_000], 4, pv.data_ptr(), F32, mask.data_ptr()),
    }
    torch.cuda.synchronize()
    for what, args in cases.items():
        n0 = pre.lib.jimm_launch_count()
        assert _raw(pre, *args) == -1, what
        assert pre.lib.jimm_launch_count() == n0, what
        assert pre.lib.jimm_last_error().decode(), what
    torch.cuda.synchronize()
    assert torch.isnan(pv).all() and torch.isnan(pv16).all() and (mask == -7).all()
    assert _raw(pre, [], [], [], n, 0, F32, 0) == 0  # B = 0: a no-op
    # the handle kinds do not mix
    fixed = ImagePreprocessor.siglip(64)
    assert _raw(fixed, [p0], [64], [64], n, pv.data_ptr(), F32, mask.data_ptr()) == -1
    assert "jimm_preproc_create_naflex" in fixed.lib.jimm_last_error().decode()
    assert pre.lib.jimm_preproc_run(pre.handle, C.c_void_p(p0), 1, 64, 64, C.c_void_p(pv.data_ptr()), F32, None) == -1
    oh, ow = C.c_int(), C.c_int()
    assert pre.lib.jimm_preproc_output_size(pre.handle, 64, 64, C.byref(oh), C.byref(ow)) == -1
    cfg = _lib.PreprocConfig()
    cfg.resample, cfg.rescale_factor = 2, 1 / 255
    cfg.std = (C.c_float * 3)(0.5, 0.5, 0.5)
    cfg.height = 224
    h = C.c_void_p()
    assert pre.lib.jimm_preproc_create_naflex(C.byref(cfg), 16, 0, C.byref(h)) == -1
    torch.cuda.synchronize()
    assert torch.isnan(pv).all() and (mask == -7).all()


# ------------------------------------------------------------------ the model fed by the front-end
MODEL_FRAMES = [(37, 53), (64, 64), (9, 70), (50, 11), (3, 5), (100, 75), (1, 200)]


def _model(golden_dir, dtype):
    from jimm_b200.models import SigLIP
    from jimm_b200.preprocess import NaFlexPreprocessor

    m = SigLIP.from_pretrained(os.path.join(golden_dir, "tiny_siglip2_naflex", "model.safetensors"), dtype=dtype)
    m.set_preprocessor(NaFlexPreprocessor(patch_size=m.vision_patch_size, max_num_patches=256))
    return m


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_model_on_frames_equals_model_on_processor_output(golden_dir, dtype):
    m = _model(golden_dir, dtype)
    imgs = [PO.synthetic_u8_images(1, h, w, seed=50 + i)[0] for i, (h, w) in enumerate(MODEL_FRAMES)]
    pv, mask, ss = NP.hf_batch(NP.hf_processor(4, 256), imgs)
    pvd = torch.from_numpy(pv).cuda()
    txt = torch.from_numpy(np.load(os.path.join(golden_dir, "tiny_siglip2_naflex", "io.npz"))["tokens"]).cuda()
    dev = [torch.from_numpy(i).cuda() for i in imgs]
    ref = m.encode_image(pvd, spatial_shapes=ss)
    assert torch.equal(m.encode_image(dev), ref)
    assert torch.equal(m.encode_image(imgs).cuda(), ref)  # host frames: host result
    assert torch.equal(m(dev, txt), m(pvd, txt, spatial_shapes=ss))
    toks = m.encode_image_tokens(dev, [1, None], return_pooled=True)
    rtoks = m.encode_image_tokens(pvd, [1, None], return_pooled=True, spatial_shapes=ss)
    assert torch.equal(toks[1], rtoks[1])
    for a, b in zip(toks[0], rtoks[0]):
        assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))
    att = m.encode_image_attentions(dev, "map")
    ratt = m.encode_image_attentions(pvd, "map", spatial_shapes=ss)
    assert len(att) == len(ratt) and all(torch.equal(x, y) for x, y in zip(att, ratt))
    # a same-size batch tensor, and a list longer than max_batch (three chunks)
    sq = torch.from_numpy(np.stack([PO.synthetic_u8_images(1, 40, 60, seed=90 + i)[0] for i in range(5)])).cuda()
    rs = NP.hf_batch(NP.hf_processor(4, 256), list(sq.cpu().numpy()))
    assert torch.equal(m.encode_image(sq), m.encode_image(torch.from_numpy(rs[0]).cuda(), spatial_shapes=rs[2]))
    m.set_max_batch(3)
    assert torch.equal(m.encode_image(dev), m.encode_image(pvd, spatial_shapes=ss))
    chunked = m.encode_image_tokens(dev, 1)
    assert len(chunked) == len(imgs) and all(torch.equal(x, y) for x, y in zip(chunked, rtoks[0][0]))
    # against HF Siglip2Model on the processor's output
    from transformers import Siglip2Model

    hf = Siglip2Model.from_pretrained(os.path.join(golden_dir, "tiny_siglip2_naflex")).eval()
    with torch.no_grad():
        r = hf.get_image_features(pixel_values=torch.from_numpy(pv), pixel_attention_mask=torch.from_numpy(mask),
                                  spatial_shapes=torch.from_numpy(ss))
    r = getattr(r, "pooler_output", r)
    bound = 8e-3 if dtype == torch.bfloat16 else 1e-3
    check_parity("tiny_siglip2_naflex on uint8 frames through the NaFlex front-end", "image_embeds", dtype, "HF Siglip2Model fp32",
                 m.encode_image(dev), r, bound)


def test_model_front_end_checks(golden_dir):
    from jimm_b200.models import SigLIP
    from jimm_b200.preprocess import ImagePreprocessor, NaFlexPreprocessor

    m = _model(golden_dir, torch.float32)
    with pytest.raises(ValueError, match="patch"):
        m.set_preprocessor(NaFlexPreprocessor(patch_size=16))
    m.set_preprocessor(ImagePreprocessor.siglip(64))
    with pytest.raises(ValueError, match="NaFlexPreprocessor"):
        m.encode_image([np.zeros((20, 20, 3), np.uint8)])
    s = SigLIP(64, 2, 128, 16, 16, 100, 128, 4, 2)
    with pytest.raises(ValueError, match="NaFlex"):
        s.set_preprocessor(NaFlexPreprocessor(patch_size=16))
