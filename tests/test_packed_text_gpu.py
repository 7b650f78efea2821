"""GPU: lists of token sequences of different lengths in one text-tower call -- their tokens packed into one stream
(jimm_k_attention_packed_ex with the causal mask, jimm_k_embed_packed, jimm_encode_text_packed, the list inputs of CLIP / SigLIP).  Row i
of a packed call must be the bits of the call on sequence i alone; for CLIP also the bits of the padded call on the row the sequence was
cut from after its EOT; and within the 1e-3 bar of the oracle."""

import ctypes as C

import numpy as np
import pytest
import torch

import jimm_oracle as O
from gpu_util import BF16, F16, F32, TORCH, check, check_parity, ptr, stream

pytestmark = pytest.mark.gpu
TOL = 1e-3
TF32 = 3
PAIRS = [(F16, F16), (F16, F32), (F16, TF32), (BF16, BF16), (BF16, F32)]
LENS = [1, 7, 63, 64, 65, 77, 128, 200]
PAD = 5  # rows after the last sample: outside every sample, they must stay as filled


def _offsets(lens):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return off, torch.from_numpy(off).cuda()


def _out_dtype(code):
    return torch.float32 if code == TF32 else TORCH[code]


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("io,ot", PAIRS)
@pytest.mark.parametrize("hd", [8, 64, 72, 128])
def test_attention_packed_causal_kernel(lib, hd, io, ot, reverse):
    H = 2
    D = H * hd
    off, off_d = _offsets(LENS)
    T = int(off[-1])
    g = torch.Generator().manual_seed(hd * 10 + io * 3 + ot + 7)
    qkv = torch.randn((T + PAD, 3 * D), generator=g).to(TORCH[io]).cuda()
    out = torch.full((T + PAD, D), float("nan"), dtype=_out_dtype(ot), device="cuda")
    check(lib, lib.jimm_k_attention_packed_ex(ptr(qkv), io, ptr(out), ot, ptr(off_d), len(LENS), max(LENS), H, hd, 1, reverse, stream()))
    for b, S in enumerate(LENS):
        o = int(off[b])
        ref = torch.full((S, D), float("nan"), dtype=_out_dtype(ot), device="cuda")
        check(lib, lib.jimm_k_attention_hd(ptr(qkv[o:o + S]), io, ptr(ref), ot, 1, S, H, hd, 1, reverse, stream()))
        assert torch.equal(out[o:o + S], ref), f"sample {b} (S={S})"
    assert torch.isnan(out[T:]).all()


@pytest.mark.parametrize("hd", [64, 72])
def test_attention_packed_ex_non_causal_is_the_packed_call(lib, hd):
    H, io, ot = 2, F16, F16
    D = H * hd
    off, off_d = _offsets(LENS)
    T = int(off[-1])
    qkv = torch.randn((T, 3 * D), generator=torch.Generator().manual_seed(hd)).half().cuda()
    a = torch.full((T, D), float("nan"), dtype=torch.float16, device="cuda")
    b = a.clone()
    check(lib, lib.jimm_k_attention_packed_ex(ptr(qkv), io, ptr(a), ot, ptr(off_d), len(LENS), max(LENS), H, hd, 0, 0, stream()))
    check(lib, lib.jimm_k_attention_packed(ptr(qkv), io, ptr(b), ot, ptr(off_d), len(LENS), max(LENS), H, hd, 0, stream()))
    assert torch.equal(a, b)


def test_embed_packed_kernel(lib):
    lens = [1, 7, 77, 3, 64, 2, 77]
    V, D, Tctx = 50, 132, 77
    off, off_d = _offsets(lens)
    T = int(off[-1])
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(-20, V + 20, (T + PAD,), generator=g, dtype=torch.int32).cuda()
    assert (ids[:T] < 0).any() and (ids[:T] >= V).any()  # the clamping is exercised at both ends
    table = torch.randn((V, D), generator=g).cuda()
    pos = torch.randn((Tctx, D), generator=g).cuda()
    x = torch.full((T + PAD, D), float("nan"), device="cuda")
    check(lib, lib.jimm_k_embed_packed(ptr(ids), ptr(table), ptr(pos), ptr(x), ptr(off_d), len(lens), T, D, V, stream()))
    for b, L in enumerate(lens):
        o = int(off[b])
        ref = torch.full((L, D), float("nan"), device="cuda")
        check(lib, lib.jimm_k_embed(ptr(ids[o:o + L]), ptr(table), ptr(pos), ptr(ref), 1, L, D, V, stream()))
        assert torch.equal(x[o:o + L], ref), f"sequence {b} (L={L})"
    assert torch.isnan(x[T:]).all()


# ------------------------------------------------------------------ models
DT = O.DualCfg(32, 1, 128, 16, 77, 1000, 128, 2, 2)  # SigLIP has no visual projection: equal tower widths
EOT = DT.vocab_size - 1  # the largest id: CLIP pools at the first maximum
DTYPES = [torch.float16, torch.bfloat16, torch.float32, torch.float8_e4m3fn]


def _model(kind, dtype=torch.float16, seed=0):
    from jimm_b200.models import CLIP, SigLIP

    p = O.random_dual_params(DT, kind, seed=seed)
    m = (CLIP if kind == "clip" else SigLIP)(32, 1, 128, 16, 77, 1000, 128, 2, 2, dtype=dtype)
    for k, v in p.items():
        m.set_flat_param(k, v.to(torch.float32))
    return p, m


def _tokens(g, n):
    return torch.randint(1, EOT - 1, (n,), generator=g)


def _clip_seqs(seed):
    """Lengths 1 .. 77 (13 twice), EOT last; then EOT in the middle (tokens after it), first, and tied (the first one pools)."""
    g = torch.Generator().manual_seed(seed)
    seqs = []
    for L in [1, 2, 13, 63, 64, 65, 77, 13]:
        s = _tokens(g, L)
        s[-1] = EOT
        seqs.append(s)
    s = _tokens(g, 40)
    s[17] = EOT
    seqs.append(s)
    s = _tokens(g, 20)
    s[0] = EOT
    seqs.append(s)
    s = _tokens(g, 30)
    s[9] = s[21] = EOT
    seqs.append(s)
    return seqs


def _siglip_seqs(seed):
    g = torch.Generator().manual_seed(seed)
    return [_tokens(g, L) for L in [1, 2, 13, 63, 64, 65, 77, 13]]


def _rows_equal_singles(m, seqs, packed):
    for i, s in enumerate(seqs):
        assert torch.equal(packed[i:i + 1], m.encode_text(s[None].cuda())), f"sequence {i} (L={len(s)})"


def _oracle_rows(fn, p, seqs):
    with torch.no_grad():
        return torch.cat([fn(p, DT, s[None].long()) for s in seqs])


@pytest.mark.parametrize("dtype", DTYPES)
def test_clip_encode_text(dtype):
    p, m = _model("clip", dtype, seed=21)
    seqs = _clip_seqs(1)
    packed = m.encode_text([s.cuda() for s in seqs])
    assert packed.is_cuda and packed.dtype == torch.float32 and packed.shape == (len(seqs), 128)
    # (a) each row is the call on that sequence alone
    _rows_equal_singles(m, seqs, packed)
    # (b) padded rows cut just after their EOT: the padded call's rows (tokens after the EOT never reach the pooled row)
    g = torch.Generator().manual_seed(2)
    padded = torch.randint(1, EOT - 1, (8, 77), generator=g)
    for i, e in enumerate([0, 5, 12, 63, 64, 76, 40]):
        padded[i, e] = EOT
    padded[7, 10] = padded[7, 50] = EOT  # tied maximum: cut after the first
    cut = [r[: int(r.argmax()) + 1] for r in padded]
    assert [len(c) for c in cut] == [1, 6, 13, 64, 65, 77, 41, 11]
    assert torch.equal(m.encode_text([c.cuda() for c in cut]), m.encode_text(padded.cuda()))
    # (c) the oracle on each sequence at its own length
    if dtype in (torch.float16, torch.float32):
        check_parity("small CLIP text (128 wide, 2 layers) packed list of 11 sequences, lengths 1-77", "rows", dtype, "fp32", packed,
                     _oracle_rows(O.clip_encode_text, p, seqs), TOL)


@pytest.mark.parametrize("dtype", DTYPES)
def test_siglip_encode_text(dtype):
    p, m = _model("siglip", dtype, seed=22)
    seqs = _siglip_seqs(3)
    packed = m.encode_text([s.cuda() for s in seqs])
    assert packed.shape == (len(seqs), 128)
    _rows_equal_singles(m, seqs, packed)
    if dtype in (torch.float16, torch.float32):
        check_parity("small SigLIP text (128 wide, 2 layers) packed list of 8 sequences, lengths 1-77", "rows", dtype, "fp32", packed,
                     _oracle_rows(O.siglip_encode_text, p, seqs), TOL)


# ------------------------------------------------------------------ chunking, launches, calls in flight
def test_chunks_give_the_same_bytes():
    seqs = [s.cuda() for s in _clip_seqs(4)]
    g = torch.Generator().manual_seed(5)
    lens = [3] * 20 + [77] * 8 + [2] * 12 + [70, 9] * 10  # 60 sequences: 20 short ones share a chunk, the 77s break on tokens
    more = [_tokens(g, L) for L in lens]
    for s in more:
        s[-1] = EOT
    seqs = [s.cuda() for s in more] + seqs
    _, small = _model("clip", seed=23)
    small.set_max_batch(4)  # 4 x 77 = 308 token rows per chunk
    _, big = _model("clip", seed=23)
    big.set_max_batch(64)  # every sequence in one chunk
    assert torch.equal(small.encode_text(seqs), big.encode_text(seqs))


def test_launches_do_not_grow_with_the_sequences(lib):
    _, m = _model("clip", seed=24)
    g = torch.Generator().manual_seed(6)
    few = [_tokens(g, L).cuda() for L in [5, 12, 9]]
    many = [_tokens(g, int(L)).cuda() for L in torch.randint(1, 31, (200,), generator=g)]
    m.encode_text(few)
    m.encode_text(many)
    torch.cuda.synchronize()
    n0 = lib.jimm_launch_count()
    m.encode_text(few)
    n1 = lib.jimm_launch_count()
    m.encode_text(many)
    n2 = lib.jimm_launch_count()
    assert n1 - n0 == n2 - n1 > 0


def _images(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn((h, w, 3), generator=g) for h, w in sizes]


@pytest.mark.parametrize("kind", ["clip", "siglip"])
def test_call_with_a_text_list(kind):
    _, m = _model(kind, seed=25)
    seqs = [s.cuda() for s in (_clip_seqs(7) if kind == "clip" else _siglip_seqs(7))]
    img = O.synthetic_images(3, 32).cuda()
    out = m(img, seqs)
    assert out.is_cuda and out.shape == (3, len(seqs))
    assert torch.equal(out, m.native().logits(m.encode_image(img), m.encode_text(seqs)))
    imgs = [x.cuda() for x in _images([(32, 32), (48, 16), (16, 64)], 8)]
    out = m(imgs, seqs, interpolate_pos_encoding=True)
    assert torch.equal(out, m.native().logits(m.encode_image(imgs, interpolate_pos_encoding=True), m.encode_text(seqs)))


def test_host_lists_give_host_results():
    _, m = _model("clip", seed=26)
    seqs = _clip_seqs(9)
    dev = m.encode_text([s.cuda() for s in seqs])
    for lst in (seqs, [s.numpy() for s in seqs], [s.tolist() for s in seqs], tuple(s[None] for s in seqs)):
        out = m.encode_text(lst)
        assert not out.is_cuda and torch.equal(out, dev.cpu())
    img = O.synthetic_images(2, 32)
    logits = m(img, seqs)
    assert not logits.is_cuda and torch.equal(logits, m(img.cuda(), [s.cuda() for s in seqs]).cpu())


def test_calls_in_flight():
    _, m = _model("clip", seed=27)
    a = [s.cuda() for s in _clip_seqs(10)]
    b = [s.cuda() for s in _clip_seqs(11)[::-1]]
    imgs = [x.cuda() for x in _images([(48, 32), (16, 16), (32, 32)], 12)]
    ra = m.encode_text(a).clone()
    torch.cuda.synchronize()
    rb = m.encode_text(b).clone()
    torch.cuda.synchronize()
    ri = m.encode_image(imgs, interpolate_pos_encoding=True).clone()
    torch.cuda.synchronize()
    oa = m.encode_text(a)
    ob = m.encode_text(b)
    oi = m.encode_image(imgs, interpolate_pos_encoding=True)
    torch.cuda.synchronize()
    assert torch.equal(oa, ra) and torch.equal(ob, rb) and torch.equal(oi, ri)


# ------------------------------------------------------------------ errors
def test_errors(monkeypatch):
    _, m = _model("clip", seed=28)
    a = torch.arange(1, 6).cuda()
    with pytest.raises(ValueError, match="length 0"):
        m.encode_text([a, a[:0]])
    with pytest.raises(ValueError, match="length 78 outside"):
        m.encode_text([a, torch.ones(78, dtype=torch.int64, device="cuda")])
    with pytest.raises(ValueError, match="one device"):
        m.encode_text([a, a.cpu()])
    with pytest.raises(ValueError, match=r"\[1, length\]"):
        m.encode_text([a, torch.stack([a, a])])
    empty = m.encode_text([])
    assert empty.shape == (0, 128) and empty.dtype == torch.float32
    img = O.synthetic_images(1, 32).cuda()
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(ValueError, match="list of token sequences is not supported by the multi-GPU"):
        m(img, [a])


def test_c_entry_refuses_before_enqueueing(lib):
    from jimm_b200.models import VisionTransformer

    _, m = _model("clip", seed=29)
    n = m.native()
    ids = torch.arange(1, 100, dtype=torch.int32, device="cuda")
    out = torch.full((2, 128), float("nan"), device="cuda")
    for lens in ([5, 0], [5, 78], [-1, 5]):
        rc = lib.jimm_encode_text_packed(n.handle, ptr(ids), 2, (C.c_int * 2)(*lens), ptr(out), stream())
        assert rc == -1 and "outside (0, context_length=77]" in lib.jimm_last_error().decode()
    vit = VisionTransformer(num_classes=10, img_size=32, patch_size=16, num_layers=1, num_heads=2, mlp_dim=256, hidden_size=64,
                            dtype=torch.float16)
    rc = lib.jimm_encode_text_packed(vit.native().handle, ptr(ids), 2, (C.c_int * 2)(5, 5), ptr(out), stream())
    assert rc == -1 and "no text tower" in lib.jimm_last_error().decode()
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
