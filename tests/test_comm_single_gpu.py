"""GPU (one H100): the multi-GPU contrastive head -- the fused normalise + peer-store + flag + logits kernel of csrc/comm.cu and the
distributed call of the CLIP / SigLIP mirrors (_call_distributed -> _distributed_logits -> comm_setup / comm_logits) -- at world 1.

comm_init(world = 1) marks itself connected, and the kernel still runs all four phases: it normalises this rank's rows into its own
gather buffer, publishes its own epoch flag, waits on it and computes the [B, B] logits block with the single-GPU head's logits_tile.
So the claim the multi-GPU tests make, that the fused head gives the single-GPU head's bits, is checked here on one GPU:

  * the fused head against jimm_contrastive_logits bit for bit (int32 views, so NaN payloads count), at text widths E = 64 .. 1152
    and B_local from 1 to max_rows, and against an fp64 reference under a componentwise worst-case bound;
  * the gather buffer's rows against l2_normalize's bits, and the two parity buffers alternating;
  * hundreds of calls enqueued back to back (epoch flags, the CTA ticket counter, parity reuse);
  * zero and non-finite rows (NaN in the row / column they poison, nothing else changed);
  * _call_distributed on device, pinned host, uint8 and resampled-position inputs against the single-process call;
  * refusals that launch nothing, and comm_setup / handle rebuilds that leak no device memory.

Each check runs in a spawned process with a single-rank gloo group on a file:// store under the test's tmp_path (no port, nothing
outlives the test).  World 1 is not full coverage: rank offsets (rank * B_local), stores into peer buffers, flags published across
ranks, and the B_local-mismatch and timeout reports need two or more GPUs and stay with tests/test_multigpu_gpu.py."""

import ctypes as C
import math
import os
import queue
import time
import traceback

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

WIDTHS = [64, 256, 512, 768, 1152]  # E = txt.D
MAX_ROWS = 300  # >= 256, and not a multiple of the 64-row tile
ROWS = [1, 2, 63, 64, 65, 128, 129, MAX_ROWS]
LOG_SCALE, BIAS = math.log(100.0), -10.0  # not the constructors' 1.0 / 1.0: swapping or reordering them shows
U = 2.0 ** -24  # unit roundoff of fp32
C_NORM = 2.0  # the constant c of the fp64 bound (derived in test_fused_head_against_fp64)


# ---- spawned single-rank process group ----
def _child(fn, store, args, q):
    import torch.distributed as dist

    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", init_method="file://" + store, rank=0, world_size=1)
        try:
            res = fn(*args)
            torch.cuda.synchronize()
        finally:
            dist.destroy_process_group()
        q.put(("ok", res))
    except BaseException:
        q.put(("error", traceback.format_exc()))


def _in_group(tmp_path, fn, *args, timeout=600):
    """fn(*args) in a spawned process that is a rank-0-of-1 gloo group; its return value, or the test fails with its traceback."""
    store = str(tmp_path / "pg_store")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_child, args=(fn, store, args, q))
    p.start()
    deadline = time.monotonic() + timeout
    try:
        while True:
            try:
                status, res = q.get(timeout=5)
                break
            except queue.Empty:
                if not p.is_alive():
                    pytest.fail(f"the worker exited with code {p.exitcode} without a result")
                if time.monotonic() > deadline:
                    pytest.fail(f"the worker gave no result within {timeout} s")
        p.join(120)
        assert p.exitcode == 0, p.exitcode
    finally:
        if p.is_alive():
            p.kill()
            p.join()
        if os.path.exists(store):
            os.remove(store)
    if status != "ok":
        pytest.fail("worker failed:\n" + res)
    return res


# ---- helpers run inside the worker ----
def _bits(a, b):
    """Same shape and the same fp32 bit patterns (NaN payloads included)."""
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _dual(kind, E):
    """A 1-layer fp16 CLIP / SigLIP at random init with text width E (the comm head's row width), logit_scale = log 100 and, for
    SigLIP, logit_bias = -10; its native handle holds MAX_ROWS rows and has its gather buffer set up."""
    from jimm_b200.models import CLIP, SigLIP

    m = (CLIP if kind == "clip" else SigLIP)(32, 1, 64, 16, 8, 64, E, E // 64, 1, dtype=torch.float16)
    m.set_flat_param("logit_scale", torch.tensor(LOG_SCALE))
    if kind == "siglip":
        m.set_flat_param("logit_bias", torch.tensor(BIAS))
    n = m.native(MAX_ROWS, require=True)
    n.comm_setup(MAX_ROWS)
    return m, n


def _rows(B, E, seed, scaled=True):
    """[B, E] fp32 standard normal rows on the GPU; scaled: row r multiplied by 2^k_r, k_r in [-30, 30] (the first two rows 2^30 and
    2^-30).  Squares and sums of such rows stay normal fp32, so the scale is exact through the norm."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, E, generator=g)
    if scaled:
        k = torch.randint(-30, 31, (B,), generator=g)
        k[: min(B, 2)] = torch.tensor([30, -30])[: min(B, 2)]
        x = x * torch.tensor([2.0 ** int(v) for v in k]).reshape(B, 1)
    return x.cuda()


def _scale_f32():
    return math.exp(float(torch.tensor(LOG_SCALE, dtype=torch.float32)))  # exp of the stored fp32 parameter, in fp64


def _fp64(ie, te, bias):
    """exp(s) * (i/|i|)(t/|t|)^T + b in fp64, and sum_k |i^_k t^_k| per element."""
    i, t = ie.double(), te.double()
    i_n, t_n = i / i.norm(dim=1, keepdim=True), t / t.norm(dim=1, keepdim=True)
    return _scale_f32() * (i_n @ t_n.T) + bias, i_n.abs() @ t_n.abs().T


def _l2_normalize(lib, x):
    from gpu_util import check, ptr, stream

    out = torch.empty_like(x)
    check(lib, lib.jimm_k_l2_normalize(ptr(x), ptr(out), x.shape[1], x.shape[0], x.shape[1], stream()))
    return out


def _gathered(n, rows):
    """(device address, row stride, copy of rows [0, rows) of the gather buffer jimm_comm_gathered reports)."""
    p, ld = C.c_void_p(), C.c_int()
    rc = n.lib.jimm_comm_gathered(n.handle, C.byref(p), C.byref(ld))
    assert rc == 0, n.lib.jimm_last_error()

    class _View:  # a zero-copy view of library memory, through the CUDA array interface torch reads
        __cuda_array_interface__ = dict(shape=(rows, ld.value), typestr="<f4", data=(p.value, False), strides=None, version=2)

    return p.value, ld.value, torch.as_tensor(_View(), device="cuda").clone()


# ---- 1 + 2: fused head = single-GPU head, bit for bit; both against fp64 ----
def _w_heads(kind):
    bias = BIAS if kind == "siglip" else 0.0
    achieved = {}
    for E in WIDTHS:
        m, n = _dual(kind, E)
        worst = 0.0
        for B in ROWS:
            ie, te = _rows(B, E, seed=E + B), _rows(B, E, seed=10_000 + E + B)
            out = n.comm_logits(ie, te)
            single = n.logits(ie, te)
            assert out.shape == (B, B)
            assert _bits(out, single), (kind, E, B, "fused head differs from jimm_contrastive_logits")
            ref, absdot = _fp64(ie, te, bias)
            diff = (out.double() - ref).abs()
            bound = _scale_f32() * C_NORM * E * U * absdot + 2.0 ** -23 * ref.abs()
            bad = diff > bound
            assert not bad.any(), (kind, E, B, int(bad.sum()), float((diff / bound).max()))
            worst = max(worst, float((diff / (_scale_f32() * absdot)).max()))
            # a power-of-two row scale scales the norm exactly: no logit bit may change, in either head
            si = torch.tensor([2.0 ** (2 * (r % 9) - 8) for r in range(B)], device="cuda").reshape(B, 1)
            st = torch.tensor([2.0 ** (9 - 3 * (r % 7)) for r in range(B)], device="cuda").reshape(B, 1)
            assert _bits(n.comm_logits(ie * si, te * st), out), (kind, E, B, "fused head: a power-of-two row scale changed a bit")
            assert _bits(n.logits(ie * si, te * st), single), (kind, E, B, "single-GPU head: a power-of-two row scale changed a bit")
        assert n.lib.jimm_comm_status(n.handle) == 0
        achieved[E] = worst
        m._invalidate()
    return achieved


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.timeout(900)
def test_fused_head_against_fp64(kind, tmp_path):
    """The fused head equals jimm_contrastive_logits bit for bit at every E and B_local, and both are within a componentwise
    worst-case bound of ref = exp(s) * i^ t^T + b computed in fp64 (i^ = i/|i|, u = 2^-24):

        |out - ref| <= exp(s) * c * E * u * sum_k |i^_k t^_k|  +  2u * |ref|,   c = 2.

    Derivation.  |ss^ - ss| <= g_n ss with n = ceil(E/32) + 5 roundings (a lane's FMA chain over E/32 squares, then a 5-level warp
    tree; all terms are non-negative), g_n = n u / (1 - n u).  sqrtf and the division round once each, so every normalised element
    carries a relative error e <= g_n / 2 + 2u + O(u^2) <= (E/64 + 5) u + O(u^2).  The k-ascending FMA chain of the dot product adds
    at most g_E * sum|a_k b_k| (E roundings).  With both operands perturbed, |acc - i^.t^| <= (2e + g_E) sum|i^ t^| + O(u^2)
    = (33E/32 + 10) u sum + O(u^2).  expf is within 2 ulp, a relative 4u, and |i^.t^| <= sum, so the scaled product is within
    exp(s) (33E/32 + 14) u sum + O(E^2 u^2) of exp(s) i^.t^.  The final sc * acc + b rounds at most twice (once if contracted to an
    FMA): u exp(s) sum for the product, u |out| <= u |ref| + O(E u^2) for the sum.  For E >= 16, 33E/32 + 15 <= 2E with room left for
    the O(E^2 u^2) terms (E u < 1e-4 here), and u |ref| <= 2u |ref|.  So the bound holds for every input without overflow or
    underflow, whatever the data, and cannot be flaky.  Rows scaled by 2^+-30 keep every square and sum a normal fp32 number.

    The achieved max |diff| / (exp(s) sum|i^ t^|) is recorded per width."""
    from gpu_util import record_parity

    achieved = _in_group(tmp_path, _w_heads, kind)
    for E, a in achieved.items():
        # no '|' in the labels: they become cells of PARITY.md's table
        record_parity(f"multi-GPU {kind} head, world 1, E {E}, B_local 1..{MAX_ROWS}",
                      "logits, max abs(diff) / (exp(s) sum abs(i^ t^))", "float32", "fp64", C_NORM * E * U, a)


# ---- 3: gather buffer and parity buffers ----
def _w_gathered(kind):
    for E in (64, 768, 1152):
        m, n = _dual(kind, E)
        addrs = []
        for call, B in enumerate((65, MAX_ROWS, 1, 129)):
            ie, te = _rows(B, E, seed=3 * call + E), _rows(B, E, seed=3 * call + E + 1)
            out = n.comm_logits(ie, te)
            torch.cuda.synchronize()
            addr, ld, g = _gathered(n, B)
            assert ld == 2 * E, (E, ld)
            assert _bits(g[:, :E], _l2_normalize(n.lib, ie)), (E, B, "image rows of the gather buffer")
            assert _bits(g[:, E:], _l2_normalize(n.lib, te)), (E, B, "text rows of the gather buffer")
            assert _bits(out, n.logits(ie, te))
            addrs.append(addr)
        buf_bytes = MAX_ROWS * 2 * E * 4  # one parity buffer: world * max_rows * 2E floats
        assert addrs[0] != addrs[1] and addrs[2] == addrs[0] and addrs[3] == addrs[1], addrs
        assert abs(addrs[1] - addrs[0]) == buf_bytes, (addrs, buf_bytes)
        m._invalidate()


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.timeout(600)
def test_gather_buffer_rows_and_parity(kind, tmp_path):
    """After a synchronised call, rows [0, B) of jimm_comm_gathered's buffer are l2_normalize's bits, image rows in columns [0, E),
    text rows in [E, 2E), at row stride 2E; consecutive calls alternate between the two parity buffers, one buffer apart."""
    _in_group(tmp_path, _w_gathered, kind)


# ---- 4: back-to-back epochs ----
def _w_back_to_back(kind, E, calls):
    m, n = _dual(kind, E)
    cycle = (1, 64, 65, MAX_ROWS)
    gen = torch.Generator(device="cuda").manual_seed(7)
    ins = [(torch.randn(B, E, device="cuda", generator=gen), torch.randn(B, E, device="cuda", generator=gen))
           for B in (cycle[c % len(cycle)] for c in range(calls))]
    torch.cuda.synchronize()
    launches = n.lib.jimm_launch_count()
    outs = [n.comm_logits(ie, te) for ie, te in ins]  # no synchronisation between the calls
    assert n.lib.jimm_launch_count() - launches == calls
    torch.cuda.synchronize()
    assert n.lib.jimm_comm_status(n.handle) == 0, n.lib.jimm_last_error()
    for c, ((ie, te), out) in enumerate(zip(ins, outs)):
        assert _bits(out, n.logits(ie, te)), (kind, E, c, ie.shape[0])
    m._invalidate()


@pytest.mark.parametrize("kind,E", [("clip", 512), ("siglip", 1152)])
@pytest.mark.timeout(600)
def test_back_to_back_epochs(kind, E, tmp_path):
    """512 calls enqueued without a synchronisation, each with fresh inputs and its own output, B_local cycling through 1, 64, 65 and
    max_rows: every result is its single-GPU reference bit for bit and the status word stays 0.  Covers the CTA ticket counter
    (epoch * gridDim.x - 1), the epoch flags and the reuse of the two parity buffers over many epochs."""
    _in_group(tmp_path, _w_back_to_back, kind, E, 512)


# ---- 5: zero and non-finite rows ----
def _w_nonfinite(kind):
    bias = BIAS if kind == "siglip" else 0.0
    B = 129
    poison_i = {0: "zero", 63: "nan", 64: "inf", 128: "-inf"}
    poison_t = {1: "-inf", 64: "zero", 65: "nan", 100: "inf"}

    def poison(x, where):
        x = x.clone()
        for r, kind_ in where.items():
            if kind_ == "zero":
                x[r] = 0.0
            else:
                x[r, r % x.shape[1]] = {"nan": float("nan"), "inf": float("inf"), "-inf": float("-inf")}[kind_]
        return x

    for E in (64, 1152):
        m, n = _dual(kind, E)
        ie, te = _rows(B, E, seed=1 + E), _rows(B, E, seed=2 + E)
        clean = n.comm_logits(ie, te)
        pi, pt = poison(ie, poison_i), poison(te, poison_t)
        out, single = n.comm_logits(pi, pt), n.logits(pi, pt)
        assert _bits(out, single), (kind, E, "fused head differs from the single-GPU head on poisoned rows")
        ref, _ = _fp64(pi, pt, bias)  # the reference's unguarded x / |x|: 0/0 and inf/inf are NaN
        assert torch.equal(torch.isnan(out).cpu(), torch.isnan(ref).cpu()), (kind, E)
        rows = torch.ones(B, dtype=torch.bool)
        cols = torch.ones(B, dtype=torch.bool)
        rows[list(poison_i)] = False
        cols[list(poison_t)] = False
        assert torch.isnan(out.cpu()[~rows]).all() and torch.isnan(out.cpu()[:, ~cols]).all()
        keep = rows[:, None] & cols[None, :]
        assert _bits(out.cpu()[keep], clean.cpu()[keep]), (kind, E, "a poisoned row changed another logit")
        assert _bits(n.comm_logits(ie, te), clean), (kind, E, "the call after a poisoned one differs")
        assert n.lib.jimm_comm_status(n.handle) == 0
        m._invalidate()


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.timeout(600)
def test_zero_and_nonfinite_rows(kind, tmp_path):
    """An all-zero row and rows holding NaN / +inf / -inf give the single-GPU head's bits: NaN across the logits row (image) or column
    (text) they poison, as the fp64 x / |x| does.  Every other logit keeps the clean call's bits, and so does the next call."""
    _in_group(tmp_path, _w_nonfinite, kind)


# ---- 6: the distributed call at world 1 ----
def _w_distributed(kind):
    import jimm_oracle as O
    from jimm_b200.models import CLIP, SigLIP
    from jimm_b200.preprocess import ImagePreprocessor

    tw = 128 if kind == "clip" else 256
    cfg = O.DualCfg(64, 2, 256, 16, 20, 300, tw, tw // 64, 2)
    p = O.random_dual_params(cfg, kind, seed=11)
    p["logit_scale"] = torch.tensor(LOG_SCALE, dtype=torch.float64)
    if kind == "siglip":
        p["logit_bias"] = torch.tensor(BIAS, dtype=torch.float64)
    B = 8
    img, txt = O.synthetic_images(B, 64), O.synthetic_tokens(B, 20, 300, kind)
    with torch.no_grad():
        ref = (O.clip_forward if kind == "clip" else O.siglip_forward)(p, cfg, img, txt)
    m = (CLIP if kind == "clip" else SigLIP)(64, 2, 256, 16, 20, 300, tw, tw // 64, 2, dtype=torch.float16)
    for k, v in p.items():
        m.set_flat_param(k, v)

    def single(*a, **kw):
        return m.set_comm("off")(*a, **kw)

    def fused(*a, **kw):
        return m.set_comm("peer")._call_distributed(*a, **kw)

    errs = []
    # device images, three repeated calls (both parity buffers, and one reused)
    want = single(img.cuda(), txt.cuda())
    for _ in range(3):
        out = fused(img.cuda(), txt.cuda())
        assert m._native._comm is not None, "the distributed call did not take the fused head"
        assert out.is_cuda and _bits(out, want), (kind, "device images")
        errs.append(float((out.cpu().double() - ref.double()).abs().max() / ref.double().abs().max()))
    # pinned host float images and host ids: ids first, images on the side stream
    ih, th = img.pin_memory(), txt.to(torch.int32).pin_memory()
    out_h = fused(ih, th)
    assert not out_h.is_cuda and _bits(out_h, single(ih, th)) and _bits(out_h, want), (kind, "host images")
    errs.append(float((out_h.double() - ref.double()).abs().max() / ref.double().abs().max()))
    # raw uint8 frames through the image front-end, on the device and pinned on the host
    m.set_preprocessor(ImagePreprocessor.clip(64) if kind == "clip" else ImagePreprocessor.siglip(64))
    frames = torch.randint(0, 256, (B, 64, 64, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    want_u8 = single(frames.cuda(), txt.cuda())
    assert _bits(fused(frames.cuda(), txt.cuda()), want_u8), (kind, "device uint8 frames")
    out_u8 = fused(frames.pin_memory(), th)
    assert not out_u8.is_cuda and _bits(out_u8, want_u8), (kind, "host uint8 frames")
    # interpolate_pos_encoding at a size other than the trained 64 x 64
    x = torch.randn(B, 48, 80, 3, generator=torch.Generator().manual_seed(9))
    for _ in range(2):
        out_i = fused(x.cuda(), txt.cuda(), interpolate_pos_encoding=True)
        assert _bits(out_i, single(x.cuda(), txt.cuda(), interpolate_pos_encoding=True)), (kind, "interpolate_pos_encoding")
    assert m._native.lib.jimm_comm_status(m._native.handle) == 0
    m._invalidate()
    return errs


@pytest.mark.parametrize("kind", ["clip", "siglip"])
@pytest.mark.timeout(900)
def test_distributed_call_at_world_one(kind, tmp_path):
    """_call_distributed (which __call__ takes only at world > 1) equals the single-process call bit for bit on device images (three
    calls), pinned host float images with host ids, device and pinned host uint8 frames, and interpolate_pos_encoding at 48 x 80; and
    is within LOGITS_TOL of the fp32 oracle."""
    from gpu_util import record_parity
    from test_parity_gpu import LOGITS_TOL

    errs = _in_group(tmp_path, _w_distributed, kind)
    record_parity(f"multi-GPU {kind} head, world 1, distributed call", "logits", "float16", "fp32", LOGITS_TOL, max(errs))
    assert max(errs) < LOGITS_TOL, errs


# ---- 7: lifecycle and refusals ----
def _w_refusals():
    from jimm_b200 import _lib
    from jimm_b200.models import CLIP, VisionTransformer

    E = 64
    m = CLIP(32, 1, 64, 16, 8, 64, E, 1, 1, dtype=torch.float16)
    m.set_flat_param("logit_scale", torch.tensor(LOG_SCALE))
    n = m.native(MAX_ROWS, require=True)
    lib, h = n.lib, n.handle
    vit = VisionTransformer(num_classes=16, img_size=32, patch_size=16, num_layers=1, num_heads=1, mlp_dim=128, hidden_size=64,
                            dtype=torch.float16)
    nv = vit.native()  # built (weights packed on the GPU) before the launches are counted
    ie, te = _rows(MAX_ROWS + 1, E, seed=1), _rows(MAX_ROWS + 1, E, seed=2)
    hbuf = C.create_string_buffer(64)
    p, ld = C.c_void_p(), C.c_int()
    torch.cuda.synchronize()
    launches = lib.jimm_launch_count()

    # before any set-up: no gather buffer, and comm_logits is refused
    assert lib.jimm_comm_gathered(h, C.byref(p), C.byref(ld)) == -4 and "not initialised" in _lib.last_error()
    assert lib.jimm_comm_status(h) == 0
    with pytest.raises(_lib.JimmError, match="comm_setup"):
        n.comm_logits(ie[:8], te[:8])
    # bad world / rank / rows leave the handle without a gather buffer
    for rank, world, rows in ((0, 0, MAX_ROWS), (0, 17, MAX_ROWS), (-1, 1, MAX_ROWS), (1, 1, MAX_ROWS), (0, 1, 0)):
        assert lib.jimm_comm_init(h, rank, world, rows, hbuf) == -1, (rank, world, rows)
        assert "bad arguments" in _lib.last_error()
        assert lib.jimm_comm_gathered(h, C.byref(p), C.byref(ld)) == -4, (rank, world, rows)
    # a ViT handle has no text tower
    assert nv.lib.jimm_comm_init(nv.handle, 0, 1, MAX_ROWS, hbuf) == -1 and "no text tower" in _lib.last_error()
    assert nv.lib.jimm_comm_gathered(nv.handle, C.byref(p), C.byref(ld)) == -4
    assert lib.jimm_launch_count() == launches, "a refused call launched a kernel"
    vit._invalidate()

    n.comm_setup(MAX_ROWS)
    out = n.comm_logits(ie[:65], te[:65])
    assert lib.jimm_launch_count() - launches == 1, "one comm call is one launch of the fused kernel"
    assert _bits(out, n.logits(ie[:65], te[:65]))
    assert lib.jimm_comm_gathered(h, C.byref(p), None) == 0
    buf = p.value
    torch.cuda.synchronize()
    launches = lib.jimm_launch_count()
    # B_local outside (0, max_rows]
    for rows in (0, MAX_ROWS + 1):
        with pytest.raises(ValueError, match="B_local"):
            n.comm_logits(ie[:rows], te[:rows])
    # a second init on the same handle: -4, the buffer kept
    assert lib.jimm_comm_init(h, 0, 1, MAX_ROWS, hbuf) == -4 and "already initialised" in _lib.last_error()
    assert lib.jimm_comm_gathered(h, C.byref(p), None) == 0 and p.value == buf
    assert lib.jimm_launch_count() == launches, "a refused call launched a kernel"
    assert lib.jimm_comm_status(h) == 0
    # and the next good call still gives the single-GPU head's bits
    for B in (1, 129, MAX_ROWS):
        assert _bits(n.comm_logits(ie[:B], te[:B]), n.logits(ie[:B], te[:B])), B
    assert lib.jimm_comm_status(h) == 0
    m._invalidate()


@pytest.mark.timeout(600)
def test_comm_refusals_launch_nothing(tmp_path):
    """comm_logits before comm_setup (JimmError), B_local of 0 or past max_rows (ValueError), a second jimm_comm_init on one handle
    (-4), jimm_comm_init with a bad world, rank or row count or on a ViT handle (-1), jimm_comm_gathered before init (-4): each
    returns its status and launches nothing, and the next good call gives the single-GPU head's bits."""
    _in_group(tmp_path, _w_refusals)


def _w_rebuild(rebuilds):
    E = 1152
    m, n = _dual("siglip", E)
    ie, te = _rows(MAX_ROWS, E, seed=3), _rows(MAX_ROWS, E, seed=4)
    first = n.comm_logits(ie, te).cpu()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(rebuilds):
        m._invalidate()  # _release_native: synchronise, barrier, close (comm_destroy)
        n = m.native(MAX_ROWS, require=True)
        n.comm_setup(MAX_ROWS)
        assert _bits(n.comm_logits(ie, te), first)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free1 = torch.cuda.mem_get_info()[0]
    gather = 2 * MAX_ROWS * 2 * E * 4 + 4096  # both parity buffers and the flags
    m._invalidate()
    return free0, free1, gather


@pytest.mark.timeout(600)
def test_comm_setup_rebuilds_do_not_leak(tmp_path):
    """20 handle rebuilds after comm_setup, each set up again: free device memory comes back to its starting value within one gather
    buffer (a comm_destroy that kept the buffer would lose 20 of them)."""
    free0, free1, gather = _in_group(tmp_path, _w_rebuild, 20)
    assert free0 - free1 <= gather, (free0, free1, gather)
