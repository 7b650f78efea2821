"""GPU: checkpoint ingestion -- the cast / transpose / staging code every real checkpoint goes through at finalize.

Kernel level, through jimm_k_upload_rows / jimm_k_upload_kernel (the loops of finalize over a staging ring of 32 MiB slots): every
(stored dtype, output type) cast is bit-equal to torch's cast of the same values (tf32: round to nearest, ties away), in the flax
(K, N) and the transposed [N, K] layouts, with pad columns and neighbouring rows left alone, at sizes that split a tensor into several
ring chunks -- a flax kernel whose chunks start off the transpose kernel's 32-row grid, a token table, a row longer than a slot, and
a slot reused behind its event while the stream is still busy.

Model level: a checkpoint whose values are representable in its stored dtype gives the same output bits whichever way it is handed
over (fp32 flax tensors, the copying jimm_model_set_param, from_pretrained on safetensors -- transposed and zero-copy -- and on
pytorch_model.bin), for every stored dtype and compute mode, on real-size ViT-B/16, CLIP-B/32 and SigLIP-B/16 checkpoints and a bare
encoder block with a 1408 x 6144 MLP.  Each family is anchored once against an independent reference."""

import ctypes as C
import gc
import shutil

import pytest
import torch

import jimm_oracle as O
from fp8_oracle import quantize_rows
from gpu_util import check, check_parity, ptr, stream
from test_kernel_paths_gpu import rna_tf32

pytestmark = pytest.mark.gpu
F32, F16, BF16, TF32 = 0, 1, 2, 3
SRC = {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}
OUT = {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16, TF32: torch.float32}
SENTINEL = -768.0  # exact in every output type: marks memory an upload must not write
CHUNK = 32 << 20  # bytes of one staging slot


@pytest.fixture(scope="module")
def lib():
    from jimm_b200 import _lib

    return _lib.load()


def ref_cast(x, out_code):
    """torch's cast of x's values to the output type (CPU); tf32 as the kernels round it (cvt.rna)."""
    v = x.float()
    return rna_tf32(v) if out_code == TF32 else v.to(OUT[out_code])


def bits(t):
    return t.contiguous().view({4: torch.int32, 2: torch.int16}[t.element_size()]).cpu()


def assert_bit_equal(got, want, what=""):
    got, want = got.cpu(), want.cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    assert torch.equal(gn, wn), f"{what}: NaN positions differ"
    bad = (bits(got) != bits(want)) & ~wn
    if bad.any():
        i = bad.flatten().nonzero()[0].item()
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first at flat index {i}: got {got.flatten()[i].item()!r} "
                             f"want {want.flatten()[i].item()!r}")


def upload_rows(lib, host, out, ldd=None, s=None):
    rows, K = host.shape
    check(lib, lib.jimm_k_upload_rows(ptr(host), {v: k for k, v in SRC.items()}[host.dtype], rows, K, ptr(out[0]), out[1], ldd or K,
                                      s or stream()))


def upload_kernel(lib, host, K, N, transposed, out, ldd=None, n0=0, s=None):
    check(lib, lib.jimm_k_upload_kernel(ptr(host), {v: k for k, v in SRC.items()}[host.dtype], K, N, int(transposed), ptr(out[0]), out[1],
                                        ldd or K, n0, s or stream()))


def dev_out(rows, cols, code, fill=SENTINEL):
    return torch.full((rows, cols), fill, dtype=OUT[code], device="cuda"), code


# ------------------------------------------------------------------------------------------------------------------ exact casts
def special_values():
    """fp32 values at the edges of the casts (as stored in the checkpoint dtype they may change; the reference casts what is stored)."""
    tie11 = 1.0 + 2.0 ** -11  # half an fp16 / tf32 ulp above 1: RNE -> 1, RNA -> 1 + 2^-10
    tie8 = 1.0 + 2.0 ** -8  # half a bf16 ulp above 1
    odd11 = 1.0 + 3 * 2.0 ** -11  # a tie with an odd lower neighbour: both round up
    v = [tie11, -tie11, odd11, -odd11, tie8, -tie8, 1.0 + 3 * 2.0 ** -8, 3.0 * tie11, 1e-3 * tie11,
         2.0 ** -24, 3 * 2.0 ** -24, -(2.0 ** -20), 2.0 ** -14 - 2.0 ** -24, 2.0 ** -25, 0.0, -0.0,  # fp16 subnormals, +-0
         65504.0, 65519.0, 65520.0, -65520.0, 70000.0, 1e5, -3e38, 1e30,  # above the fp16 range: +-inf in fp16
         float("inf"), float("-inf"), float("nan"), -float("nan")]
    return torch.tensor(v, dtype=torch.float32)


def cast_inputs(src_code, n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.cat([special_values(), torch.randn(n, generator=g) * 3, torch.rand(n, generator=g) * 2 ** -12])
    # RNE / RNA disagreements for every target: random mantissas with the dropped bits forced to exactly one half
    ties = torch.randn(512, generator=g).view(torch.int32)
    x = torch.cat([x, ((ties & ~0x1FFF) | 0x1000).view(torch.float32), ((ties & ~0xFFFF) | 0x8000).view(torch.float32)])
    return x.to(SRC[src_code])


@pytest.mark.parametrize("src", [F32, F16, BF16])
@pytest.mark.parametrize("out", [F32, F16, BF16, TF32])
def test_casts_bit_exact(lib, src, out):
    """Every (stored dtype, output type) pair, through the row copy and both kernel layouts, equals torch's cast of the stored
    values: RNE to fp16 / bf16 (bf16 above 65504 -> +-inf in fp16), RNA to tf32, subnormals and signed zeros kept, NaN stays NaN."""
    x = cast_inputs(src)
    K = 97
    x = x[: x.numel() // K * K].reshape(-1, K).contiguous()
    R = x.shape[0]
    want = ref_cast(x, out)
    d = dev_out(R, K, out)
    upload_rows(lib, x, d)
    assert_bit_equal(d[0], want, "rows")
    # the same values as a (K, N) = (R, K) flax kernel and as its transpose: both give the [N, K] operand x.T
    d = dev_out(K, R, out)
    upload_kernel(lib, x, R, K, False, d)
    assert_bit_equal(d[0], want.T.contiguous(), "flax kernel")
    d = dev_out(K, R, out)
    upload_kernel(lib, x.T.contiguous(), R, K, True, d)
    assert_bit_equal(d[0], want.T.contiguous(), "transposed kernel")


# ---------------------------------------------------------------------------------------------------------------------- layouts
@pytest.mark.parametrize("out", [F16, TF32])
@pytest.mark.parametrize("transposed", [False, True])
def test_kernel_layout_padding_and_offset(lib, out, transposed):
    """K, N off the 32 x 32 tile grid, ldd > K (pad columns keep the caller's sentinel) and n0 > 0 into a fused operand (the
    q | k | v projections): the other rows are untouched."""
    K, N, ldd, n0, Ntot = 45, 77, 56, 77, 3 * 77
    g = torch.Generator().manual_seed(1)
    w = torch.randn(K, N, generator=g).to(torch.bfloat16)  # flax (K, N)
    host = w.T.contiguous() if transposed else w
    d = dev_out(Ntot, ldd, out)
    upload_kernel(lib, host, K, N, transposed, d, ldd=ldd, n0=n0)
    got = d[0].cpu()
    want = torch.full((Ntot, ldd), SENTINEL, dtype=OUT[out])
    want[n0:n0 + N, :K] = ref_cast(w.T.contiguous(), out)
    assert_bit_equal(got, want)
    # rows with a pitch: pad columns untouched
    x = torch.randn(33, 45, generator=g)
    d = dev_out(33, 64, out)
    upload_rows(lib, x, d, ldd=64)
    want = torch.full((33, 64), SENTINEL, dtype=OUT[out])
    want[:, :45] = ref_cast(x, out)
    assert_bit_equal(d[0].cpu(), want)


def test_rejects_bad_arguments(lib):
    x = torch.zeros(4, 8)
    d = torch.zeros(4, 8, device="cuda")
    assert lib.jimm_k_upload_rows(ptr(x), F32, 4, 8, ptr(d), F32, 7, stream()) == -1  # ldd < K
    assert lib.jimm_k_upload_kernel(ptr(x), 5, 4, 8, 0, ptr(d), F32, 8, 0, stream()) == -1  # bad source type
    assert lib.jimm_k_upload_kernel(ptr(x), F32, 4, 8, 0, ptr(d), 4, 8, 0, stream()) == -1  # e4m3 is not an upload type


# ------------------------------------------------------------------------------------------------------ sizes that split into chunks
def _rand(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(dtype)


@pytest.mark.parametrize("K,N,dtype,out,transposed", [
    (1408, 6144, torch.float32, TF32, False),  # 24 KiB rows: chunks of 1365 rows, the second starts at k0 = 1365 (not a multiple of 32)
    (1408, 6144, torch.float32, F16, True),
    (2048, 12288, torch.bfloat16, BF16, False),  # also 1365 rows per chunk
    (2048, 12288, torch.bfloat16, F16, True),
    (3000, 6144, torch.float32, F32, False),  # three chunks: the first slot is reused
])
def test_kernel_chunks(lib, K, N, dtype, out, transposed):
    w = _rand((K, N), dtype, seed=K + N)
    assert K * N * w.element_size() > CHUNK
    host = w.T.contiguous() if transposed else w
    d = dev_out(N, K, out)
    upload_kernel(lib, host, K, N, transposed, d)
    assert_bit_equal(d[0], ref_cast(w.T.contiguous(), out), f"{K}x{N} {dtype} transposed={transposed}")


@pytest.mark.parametrize("rows,K,dtype,out", [
    (49408, 512, torch.float16, F16),  # CLIP-B/32 token table as fp16: two chunks
    (49408, 512, torch.bfloat16, TF32),
    (49408, 512, torch.float32, F32),  # as fp32: four chunks
    (1, (8 << 20) + 4099, torch.float32, F32),  # one row longer than a slot: split along the row
    (1, (20 << 20) + 5, torch.float32, TF32),  # three pieces of one row
    (1, (16 << 20) + 3, torch.bfloat16, F32),
])
def test_rows_chunks(lib, rows, K, dtype, out):
    x = _rand((rows, K), dtype, seed=rows + K)
    d = dev_out(rows, K, out)
    upload_rows(lib, x, d)
    assert_bit_equal(d[0], ref_cast(x, out), f"{rows}x{K} {dtype}")


def test_slot_reuse_waits_for_a_busy_stream(lib):
    """Five chunks through two slots while the stream is still busy with earlier work: the host copy of chunk i + 2 into a slot must
    wait until the device has consumed chunk i from it."""
    w = _rand((5 * 1365 - 100, 6144), torch.float32, seed=5)
    x = _rand((49408 * 2, 512), torch.float32, seed=6)
    s = torch.cuda.Stream()
    d1, d2 = dev_out(6144, w.shape[0], F32), dev_out(x.shape[0], 512, F16)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)  # ~0.1 s of device time ahead of the copies
        upload_kernel(lib, w, w.shape[0], 6144, False, d1, s=C.c_void_p(s.cuda_stream))
        torch.cuda._sleep(200_000_000)
        upload_rows(lib, x, d2, s=C.c_void_p(s.cuda_stream))
    s.synchronize()
    assert_bit_equal(d1[0], w.T.contiguous(), "kernel behind a busy stream")
    assert_bit_equal(d2[0], x.half(), "table behind a busy stream")


# ----------------------------------------------------------------------------------------------------------- e4m3 weight quantiser
def test_e4m3_weights_same_from_either_hand_off(lib):
    """FP8 mode packs a weight to fp32 [N, K] rows, then quantises each row: a transposed bf16 hand-off and a flax fp32 hand-off of the
    same values give the same bytes and scales, which are the reference quantiser's."""
    K, N = 1408, 6144
    w16 = _rand((K, N), torch.bfloat16, seed=9) * 0.05
    outs = []
    for host, transposed in ((w16.T.contiguous(), True), (w16.float(), False)):
        f32 = dev_out(N, K, F32)
        upload_kernel(lib, host, K, N, transposed, f32)
        q = torch.empty((N, K), dtype=torch.uint8, device="cuda")
        sc = torch.empty(N, dtype=torch.float32, device="cuda")
        check(lib, lib.jimm_k_quantize_e4m3(ptr(f32[0]), K, N, K, ptr(q), K, ptr(sc), stream()))
        outs.append((q.cpu(), sc.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    rq, rs = quantize_rows(w16.float().T.contiguous())
    assert torch.equal(outs[0][0], rq.view(torch.uint8)) and torch.equal(outs[0][1], rs)


# -------------------------------------------------------------------------------------------------- models at real size, every hand-off
COMPUTE = {"fp32": F32, "fp16": F16, "bf16": BF16, "e4m3": 4}
STORED = (torch.float32, torch.float16, torch.bfloat16)
TOL = 1e-3


class CopyingNativeModel:
    """A native handle whose parameters go through jimm_model_set_param (the library keeps its own copy) in flax layout and the
    checkpoint's dtype; forwards are NativeModel's."""

    def __new__(cls, cfg, params, max_batch, dtype):
        from jimm_b200 import _lib
        from jimm_b200._runtime import NativeModel

        n = NativeModel.__new__(NativeModel)
        n.lib, n.cfg, n.device_index, n.device = _lib.load(), cfg, 0, torch.device("cuda", 0)
        n.handle = C.c_void_p()
        _lib.check(n.lib.jimm_model_create(C.byref(cfg), 0, C.byref(n.handle)))
        code = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}[dtype]
        for name, v in params.items():
            t = (v.materialize() if hasattr(v, "materialize") else v).to(dtype).contiguous()
            shape = (C.c_int64 * max(t.ndim, 1))(*t.shape)
            _lib.check(n.lib.jimm_model_set_param(n.handle, name.encode(), C.c_void_p(t.data_ptr()), shape, t.ndim, code))
            del t  # the library holds its own copy
        _lib.check(n.lib.jimm_model_finalize(n.handle, max_batch))
        vo, to = C.c_int(), C.c_int()
        _lib.check(n.lib.jimm_model_output_dim(n.handle, C.byref(vo), C.byref(to)))
        n.max_batch, n.vision_out, n.text_out, n._comm, n.preproc = max_batch, vo.value, to.value, None, None
        return n


def _cfg(cfg, compute):
    c = type(cfg)()
    C.memmove(C.byref(c), C.byref(cfg), C.sizeof(cfg))
    c.compute_dtype = compute
    return c


def _save_checkpoint(hf_model, d, dtype):
    from safetensors.torch import save_file

    d.mkdir(parents=True)
    sd = {k: (v.detach().to(dtype) if v.is_floating_point() else v.detach()).contiguous() for k, v in hf_model.state_dict().items()}
    save_file(sd, str(d / "model.safetensors"))
    torch.save(sd, str(d / "pytorch_model.bin"))
    hf_model.config.to_json_file(str(d / "config.json"))
    return sd


def _hand_offs(cls, d, dtype):
    """(native config, {hand-off: (parameters, handle constructor)}, fp32 flax parameters) of the checkpoint in directory d, stored
    as `dtype`.  The fp32 flax tensors are what set_flat_param hands over."""
    from jimm_b200._runtime import NativeModel

    st = cls.from_pretrained(str(d / "model.safetensors"))
    pt = cls.from_pretrained(str(d), use_pytorch=True)
    raw = st.flat_params(raw=True)
    k = next(n for n, v in raw.items() if getattr(v, "transposed", False))
    assert raw[k].base.dtype == dtype and pt.flat_params(raw=True)[k].base.dtype == dtype  # zero-copy: the stored dtype reaches the library
    flat = st.flat_params()
    return st._native_config(), {
        "flax fp32 (set_flat_param)": (flat, NativeModel),
        "jimm_model_set_param copy": (raw, lambda cfg, p, mb: CopyingNativeModel(cfg, p, mb, dtype)),
        "from_pretrained safetensors": (raw, NativeModel),
        "from_pretrained pytorch_model.bin": (pt.flat_params(raw=True), NativeModel),
    }, flat


def _same_bits_every_hand_off(cfg, hand_offs, run, what):
    """For every compute mode: the outputs of every hand-off are bit-equal.  Returns {compute: outputs of the first hand-off}."""
    first = {}
    for cname, code in COMPUTE.items():
        outs = {}
        for hname, (params, make) in hand_offs.items():
            n = make(_cfg(cfg, code), params, 4)
            try:
                outs[hname] = [o.cpu() for o in run(n)]
            finally:
                n.close()
        base_name, base = next(iter(outs.items()))
        for hname, o in outs.items():
            for i, (a, b) in enumerate(zip(o, base)):
                assert torch.isfinite(a).all(), f"{what} [{cname}] {hname}: output {i} not finite"
                assert torch.equal(a, b), f"{what} [{cname}]: output {i} of '{hname}' differs from '{base_name}' (max |d| {(a - b).abs().max():.3e})"
        first[cname] = base
    return first


def _family(tmp_path, hf_model, cls, run, what):
    """Save hf_model in every stored dtype (one at a time, deleted after use) and check the hand-off invariant; returns the fp32
    checkpoint's outputs per compute mode and its flax parameters."""
    anchor = None
    try:
        for dtype in STORED:
            d = tmp_path / str(dtype).replace("torch.", "")
            _save_checkpoint(hf_model, d, dtype)
            cfg, hand_offs, flat = _hand_offs(cls, d, dtype)
            outs = _same_bits_every_hand_off(cfg, hand_offs, run, f"{what} stored {dtype}")
            if dtype == torch.float32:
                anchor = (outs, flat)
            del hand_offs
            gc.collect()
            shutil.rmtree(d)
    finally:
        shutil.rmtree(tmp_path, ignore_errors=True)
    return anchor


def _hf_seeded(build, seed):
    from check_vs_hf import perturb_

    torch.manual_seed(seed)
    return perturb_(build()).eval()


def test_vit_b16_every_hand_off(tmp_path):
    from transformers import ViTConfig, ViTForImageClassification

    from jimm_b200.models import VisionTransformer

    hf = _hf_seeded(lambda: ViTForImageClassification(ViTConfig(num_labels=1000)), 0)
    img = O.synthetic_images(2, 224, seed=11)
    outs, flat = _family(tmp_path, hf, VisionTransformer, lambda n: [n.vision(img.cuda())], "ViT-B/16@224")
    del hf
    cfg = O.ViTCfg()
    with torch.no_grad():
        ref = O.vit_forward(flat, cfg, img)
    for c, dt in (("fp32", torch.float32), ("fp16", torch.float16)):
        check_parity("ViT-B/16@224 from a HF checkpoint", "logits", dt, "fp32", outs[c][0], ref, TOL)


def test_clip_b32_every_hand_off(tmp_path):
    from transformers import CLIPConfig, CLIPModel

    from jimm_b200.models import CLIP

    hf = _hf_seeded(lambda: CLIPModel(CLIPConfig()), 1)  # vision 12 x 768 P32 @224, text 12 x 512, T = 77, V = 49408
    assert hf.config.text_config.vocab_size == 49408 and hf.config.text_config.max_position_embeddings == 77
    img = O.synthetic_images(2, 224, seed=12)
    txt = O.synthetic_tokens(3, 77, 49408, "clip", seed=13)

    def run(n):
        ie, te = n.vision(img.cuda(), encode=True), n.text(txt)
        return [ie, te, n.logits(ie, te)]

    outs, flat = _family(tmp_path, hf, CLIP, run, "CLIP-B/32")
    del hf
    cfg = O.DualCfg(224, 12, 768, 32, 77, 49408, 512, 8, 12)
    with torch.no_grad():
        ref_i, ref_t = O.clip_encode_image(flat, cfg, img), O.clip_encode_text(flat, cfg, txt)
    for c, dt in (("fp32", torch.float32), ("fp16", torch.float16)):
        check_parity("CLIP-B/32 from a HF checkpoint", "image_embeds", dt, "fp32", outs[c][0], ref_i, TOL)
        check_parity("CLIP-B/32 from a HF checkpoint", "text_embeds", dt, "fp32", outs[c][1], ref_t, TOL)


def test_siglip_b16_every_hand_off(tmp_path):
    """SigLIP-B/16 @224 with the MAP head (its packed in_proj split three ways) and the text head, anchored against HuggingFace's own
    forward in fp64 (jimm's and HF's semantics coincide for SigLIP)."""
    from transformers import SiglipConfig, SiglipModel

    from jimm_b200.models import SigLIP

    hf = _hf_seeded(lambda: SiglipModel(SiglipConfig()), 2)
    with torch.no_grad():
        hf.logit_scale.fill_(2.3)
        hf.logit_bias.fill_(-1.7)
    img = O.synthetic_images(2, 224, seed=14)
    txt = O.synthetic_tokens(3, 64, 32000, "siglip", seed=15)

    def run(n):
        ie, te = n.vision(img.cuda(), encode=True), n.text(txt)
        return [ie, te, n.logits(ie, te)]

    outs, _ = _family(tmp_path, hf, SigLIP, run, "SigLIP-B/16")
    hf = hf.double()
    with torch.no_grad():
        ref_i = hf.vision_model(pixel_values=img.double().permute(0, 3, 1, 2)).pooler_output
        ref_t = hf.text_model(input_ids=txt.long()).pooler_output
    for c, dt in (("fp32", torch.float32), ("fp16", torch.float16)):
        check_parity("SigLIP-B/16@224 from a HF checkpoint", "image_embeds", dt, "HF fp64", outs[c][0], ref_i, TOL)
        check_parity("SigLIP-B/16@224 from a HF checkpoint", "text_embeds", dt, "HF fp64", outs[c][1], ref_t, TOL)


def test_encoder_1408x6144_every_hand_off():
    """A bare encoder block with the 1408 x 6144 MLP, so FC1's flax kernel is split into ring chunks at k0 = 1365 inside a model."""
    from jimm_b200 import _lib
    from jimm_b200._runtime import NativeModel, NativeSubModule
    from jimm_b200.nn import LazyParam

    D, M, H, S = 1408, 6144, 16, 40
    g = torch.Generator().manual_seed(21)
    p = {}
    O._rand_blocks(p, g, "", 1, D, H, M)
    p = O.cast_params(p, torch.float32)
    x = torch.randn(2, S, D, generator=g)
    cfg = _lib.Config()
    cfg.kind, cfg.v_width, cfg.v_heads, cfg.v_mlp, cfg.v_layers, cfg.v_act = _lib.KIND_ENCODER, D, H, M, 1, _lib.ACT_GELU_TANH
    cfg.v_eps_block = cfg.v_eps_outer = 1e-6
    cfg.ctx_len = S

    def transposed(params, dtype):  # kernels as the [N, K] transpose of their (K, N) view, like a HF (out, in) weight
        out = {}
        for k, v in params.items():
            v = v.to(dtype)
            if k.endswith(".kernel"):
                K = v.shape[0] if not k.endswith("out.kernel") else v.shape[0] * v.shape[1]
                out[k] = LazyParam(v.reshape(K, -1).T.contiguous(), v.shape, transposed=True)
            else:
                out[k] = v.float()
        return out

    def sub(n):
        s = NativeSubModule.__new__(NativeSubModule)
        s.native, s.kind, s.max_seq, s.max_batch, s.D = n, cfg.kind, S, 2, D
        return s

    anchor = None
    for dtype in STORED:
        pd = {k: v.to(dtype).float() for k, v in p.items()}  # values representable in the stored dtype
        hand_offs = {
            "flax fp32": (pd, NativeModel),
            "jimm_model_set_param copy": (pd, lambda c, q, mb: CopyingNativeModel(c, q, mb, dtype)),
            "transposed zero-copy": (transposed(pd, dtype), NativeModel),
        }
        outs = _same_bits_every_hand_off(cfg, hand_offs, lambda n: [sub(n)(x.cuda())], f"encoder 1408/6144 stored {dtype}")
        if dtype == torch.float32:
            anchor = outs
    with torch.no_grad():
        ref = O.transformer_encoder(p, "blocks.layers.0.", x, H, 1e-6, False, None)
    for c, dt in (("fp32", torch.float32), ("fp16", torch.float16)):
        check_parity("bare TransformerEncoder 1408/6144 (chunked FC1)", "activations", dt, "fp32", anchor[c][0], ref, TOL)
