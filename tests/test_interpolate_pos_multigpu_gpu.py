"""GPU (needs >= 2 H100s; skipped otherwise): SigLIP with interpolate_pos_encoding=True under torch.distributed -- one process per
GPU, 384 x 384 images on a tower trained at 256 -- against the single-GPU call and the interpolating oracle, in the style of
tests/test_multigpu_gpu.py."""

import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for d in (root, os.path.join(root, "oracle"), os.path.join(root, "tests")):
        sys.path.insert(0, d)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist

    import interp_oracle as I
    import jimm_oracle as O
    from jimm_b200 import dist as jd
    from jimm_b200.models import SigLIP
    from jimm_b200.preprocess import ImagePreprocessor

    jd.init_from_env("nccl")
    cfg = O.DualCfg(256, 2, 256, 16, 20, 300, 256, 4, 2)
    p = O.random_dual_params(cfg, "siglip", seed=11)
    Bg = 4 * world
    img, txt = O.synthetic_images(Bg, 384), O.synthetic_tokens(Bg, 20, 300, "siglip")
    with torch.no_grad():
        ref = I.siglip_forward(p, cfg, img, txt, interpolate_pos_encoding=True)
    m = SigLIP(256, 2, 256, 16, 20, 300, 256, 4, 2, dtype=torch.float16)
    for k, v in p.items():
        m.set_flat_param(k, v)
    lo, hi = jd.shard_range(Bg, rank, world)
    m.set_comm("off")
    full = m(img.cuda(), txt.cuda(), interpolate_pos_encoding=True).cpu()
    errs = []
    for mode in ("peer", "peer", "nccl"):
        m.set_comm(mode)
        out = m(img[lo:hi].cuda(), txt[lo:hi].cuda(), interpolate_pos_encoding=True)
        assert out.shape == (hi - lo, Bg)
        if mode == "peer":
            assert torch.equal(out.cpu(), full[lo:hi]), "sharded interpolate_pos_encoding call differs from the single-GPU call"
        else:
            assert float((out.cpu() - full[lo:hi]).abs().max()) < 1e-4
        errs.append(float((out.cpu().double() - ref[lo:hi].double()).abs().max() / ref.abs().max()))
    m.set_comm("peer")
    # host inputs: the images are copied on a side stream while the text tower runs, then the off-grid vision call
    out_h = m(img[lo:hi].pin_memory(), txt[lo:hi].to(torch.int32).pin_memory(), interpolate_pos_encoding=True)
    assert not out_h.is_cuda and torch.equal(out_h, full[lo:hi])
    # raw uint8 frames through a 384 front-end, device and host: the same bits as front-end-then-model
    proc = ImagePreprocessor.siglip(384)
    m.set_preprocessor(proc)
    frames = torch.randint(0, 256, (Bg, 300, 420, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)[lo:hi].contiguous()
    ref_u8 = m(proc(frames.cuda(), dtype=torch.float16), txt[lo:hi].cuda(), interpolate_pos_encoding=True)
    assert torch.equal(m(frames.cuda(), txt[lo:hi].cuda(), interpolate_pos_encoding=True), ref_u8)
    assert torch.equal(m(frames.pin_memory(), txt[lo:hi].to(torch.int32).pin_memory(), interpolate_pos_encoding=True), ref_u8.cpu())
    # a handle rebuild on every rank at once (4 images of 256 tokens hold no 1296-token 576 x 576 image), the gather buffer re-made
    m.set_max_batch(hi - lo)
    big = O.synthetic_images(Bg, 576, seed=9)
    with torch.no_grad():
        ref_big = I.siglip_forward(p, cfg, big, txt, interpolate_pos_encoding=True)
    out_b = m(big[lo:hi].cuda(), txt[lo:hi].cuda(), interpolate_pos_encoding=True)
    errs.append(float((out_b.cpu().double() - ref_big[lo:hi].double()).abs().max() / ref_big.abs().max()))
    torch.cuda.synchronize()
    dist.barrier()
    q.put((rank, errs))
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_sharded_siglip_384():
    world = min(torch.cuda.device_count(), 2)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=500) for _ in range(world))
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    from gpu_util import record_parity

    for rank, errs in res:
        # logits carry the fp16 towers' error amplified by exp(logit_scale) (tests/test_parity_gpu.py LOGITS_TOL)
        record_parity(f"multi-GPU SigLIP @384 interpolate_pos_encoding, world {world}, rank {rank}", "logits row block", "float16", "fp32",
                      2e-3, max(errs))
        assert all(e < 2e-3 for e in errs), (rank, errs)
