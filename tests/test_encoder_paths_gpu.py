"""The other half of every encoder block as the forward pass runs it: attention, MAP attention, LayerNorm and the text towers'
pooling, through jimm_k_attention_ex / jimm_k_layernorm_ex (the encoder's reverse walk) at the models' shapes and output types.

- Wherever two runs do the same fp32 arithmetic they must agree bit for bit: the reverse walk with the forward walk, a 16-bit
  output with the fp32 output of the same kernel rounded to nearest even, a tf32 output with rna_tf32 of it, an in-place or
  gathered LayerNorm with the dense one.
- LayerNorm rows with a variance near eps, and whole models whose every LayerNorm input has a variance near 3e-6, so that any
  epsilon in the model (1e-12, 1e-6, 1e-5) being swapped for another shows in the output.
- CLIP's end-of-text pooling with the padding HuggingFace tokenizers produce: many EOT ids per row, the first one wins."""

import math

import pytest
import torch

import jimm_oracle as O
from gpu_util import BF16, CODE, F16, F32, check, check_parity, ptr, rel_err, stream
from test_kernel_paths_gpu import SENTINEL, TF32, rna_tf32

DEV = "cuda"
SMS = 132
TOL = 1e-3  # the model parity bar (test_parity_gpu.py)


def _randn(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


def _untouched(t):
    return bool((t.float() == SENTINEL).all())


# ---- attention as run_encoder runs it ------------------------------------------------------------------------------------------------
def attention_ex(lib, qkv, out, out_code, B, S, H, causal, reverse):
    check(lib, lib.jimm_k_attention_ex(ptr(qkv), CODE[qkv.dtype], ptr(out), out_code, B, S, H, causal, reverse, stream()))


OUT_TYPES = {torch.float16: [(torch.float16, F16), (torch.float32, TF32)], torch.bfloat16: [(torch.bfloat16, BF16)]}


@pytest.mark.gpu
@pytest.mark.parametrize("io", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("H", [12, 16])
@pytest.mark.parametrize("S,causal", [(50, 0), (197, 0), (77, 1), (256, 0), (576, 0), (577, 0), (1024, 0)],
                         ids=["vit_b32", "vit_b16", "clip_text", "siglip_256", "siglip_576", "vit_l16_384", "s1024"])
def test_attention_as_run(lib, S, causal, H, io):
    """At least two CTAs per SM.  The fp32 output of the forward walk is the reference: it is close to exact softmax attention; the
    reverse walk gives the same bits for every output type; 16-bit outputs are it rounded to nearest even, tf32 outputs rna_tf32 of
    it.  The rows of the output buffer past B * S keep their bits."""
    B = max(2, math.ceil(2 * SMS / (math.ceil(S / 64) * H)))
    D = H * 64
    qkv = (_randn(B * S, 3 * D, seed=S + H) * 1.5).to(io)
    f32 = torch.empty(B * S, D, device=DEV)
    attention_ex(lib, qkv, f32, F32, B, S, H, causal, 0)
    q, k, v = qkv.double().reshape(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    w = (q / 8.0) @ k.transpose(-1, -2)
    if causal:
        w = w.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=DEV)), float("-inf"))
    ref = (torch.softmax(w, -1) @ v).permute(0, 2, 1, 3).reshape(B * S, D)
    assert rel_err(f32, ref) < (3e-3 if io == torch.float16 else 2e-2), rel_err(f32, ref)
    for dt, code in [(torch.float32, F32)] + OUT_TYPES[io]:
        want = f32 if code == F32 else rna_tf32(f32) if code == TF32 else f32.to(dt)
        for reverse in (0, 1):
            buf = torch.full((B * S + 70, D), SENTINEL, dtype=dt, device=DEV)
            attention_ex(lib, qkv, buf, code, B, S, H, causal, reverse)
            torch.cuda.synchronize()
            assert torch.equal(buf[: B * S], want), (code, reverse)
            assert _untouched(buf[B * S:]), (code, reverse, "rows past B * S written")


# ---- MAP-head attention ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("probe", ["flat", "peaked"])
@pytest.mark.parametrize("H", [12, 16])
@pytest.mark.parametrize("S", [196, 256, 576, 729, 1024])
def test_map_attention_as_run(lib, S, H, probe):
    """run_map_head stores the pooled row in the compute type: f16 -> f16, f16 -> tf32 (fp32 mode) and bf16 -> bf16, bit for bit
    the fp32 output of the same kernel rounded.  The fp32 outputs against fp64 for a flat probe (softmax near uniform) and a sharply
    peaked one (one key per sample and head scores about 14 above every other)."""
    B, D = 64, H * 64
    g = torch.Generator(device="cpu").manual_seed(S * H)
    kv = torch.randn(B, S, 2, H, 64, generator=g)
    u = torch.nn.functional.normalize(torch.randn(H, 64, generator=g), dim=-1)
    if probe == "flat":
        q = torch.randn(H, 64, generator=g) * 0.05
    else:
        kv[:, :, 0] *= 0.5
        hot = torch.randint(0, S, (B, H), generator=g)
        for h in range(H):
            kv[torch.arange(B), hot[:, h], 0, h] = u[h] * 4.0
        q = u * 48.0  # (q / 8) . k = 24 on the hot key, N(0, 9) elsewhere
    q = q.reshape(D).to(DEV)
    kv = kv.reshape(B * S, 2 * D).to(DEV)
    for io, outs in ((torch.float16, [(torch.float16, F16), (torch.float32, TF32)]), (torch.bfloat16, [(torch.bfloat16, BF16)])):
        kvt = kv.to(io)
        f32 = torch.empty(B, D, device=DEV)
        check(lib, lib.jimm_k_map_attention(ptr(q), ptr(kvt), CODE[io], ptr(f32), F32, B, S, H, stream()))
        k, v = kvt.double().reshape(B, S, 2, H, 64).permute(2, 0, 3, 1, 4)
        w = torch.softmax((q.double().reshape(1, H, 1, 64) / 8.0) @ k.transpose(-1, -2), -1)
        if probe == "peaked":
            assert float(w.amax(-1).min()) > 0.999
        ref = (w @ v).reshape(B, D)
        assert rel_err(f32, ref) < 2e-5, (io, rel_err(f32, ref))
        for dt, code in outs:
            out = torch.full((B + 3, D), SENTINEL, dtype=dt, device=DEV)
            check(lib, lib.jimm_k_map_attention(ptr(q), ptr(kvt), CODE[io], ptr(out), code, B, S, H, stream()))
            torch.cuda.synchronize()
            assert torch.equal(out[:B], rna_tf32(f32) if code == TF32 else f32.to(dt)), (io, code)
            assert _untouched(out[B:])


# ---- LayerNorm ------------------------------------------------------------------------------------------------------------------------
def layernorm_ex(lib, x, out, out_code, eps, scale, bias, *, rows=None, group=1, row_off=0, index=None, reverse=0):
    D = scale.shape[0]
    rows = x.shape[0] if rows is None else rows
    check(lib, lib.jimm_k_layernorm_ex(ptr(x), x.stride(0), group, row_off, ptr(index), ptr(scale), ptr(bias), eps, ptr(out), out_code,
                                       out.stride(0), rows, D, reverse, stream()))


LN_OUTS = [(torch.float32, F32), (torch.float32, TF32), (torch.float16, F16), (torch.bfloat16, BF16)]
LN_IDS = ["f32", "tf32", "f16", "bf16"]


def _fast_var_ln(x, scale, bias, eps):
    """nnx.LayerNorm(use_fast_variance=True) in fp64 on the fp32 input."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = ((xd * xd).mean(-1, keepdim=True) - mean * mean).clamp_min(0)
    return (xd - mean) * torch.rsqrt(var + eps) * scale.double() + bias.double()


@pytest.mark.gpu
@pytest.mark.parametrize("out", LN_OUTS, ids=LN_IDS)
@pytest.mark.parametrize("D", [768, 1024, 1280, 1664, 2048])
def test_layernorm_reverse_and_in_place(lib, D, out):
    """The reverse row walk gives the bits of the forward walk; in place (out == x, fp32: ln_pre) the bits of out of place.  1280,
    1664 and 2048 take the 16-vector register path (2048 is its last width); results against fp64."""
    dt, code = out
    rows = 3001
    x = _randn(rows, D, seed=D) * 3 + 1.5
    scale, bias = _randn(D, seed=D + 1), _randn(D, seed=D + 2)
    fwd = torch.full((rows + 9, D), SENTINEL, dtype=dt, device=DEV)
    rev = fwd.clone()
    layernorm_ex(lib, x, fwd, code, 1e-6, scale, bias, rows=rows)
    layernorm_ex(lib, x, rev, code, 1e-6, scale, bias, rows=rows, reverse=1)
    torch.cuda.synchronize()
    assert torch.equal(fwd, rev)
    assert _untouched(fwd[rows:])
    ref = _fast_var_ln(x, scale, bias, 1e-6)
    tol = {F32: 2e-5, TF32: 1e-3, F16: 1e-3, BF16: 8e-3}[code]
    assert rel_err(fwd[:rows], ref) < tol, rel_err(fwd[:rows], ref)
    if code in (F32, TF32):
        for reverse in (0, 1):
            y = x.clone()
            layernorm_ex(lib, y, y, code, 1e-6, scale, bias, reverse=reverse)
            torch.cuda.synchronize()
            assert torch.equal(y, fwd[:rows]), reverse


@pytest.mark.gpu
@pytest.mark.parametrize("out", LN_OUTS[1:], ids=LN_IDS[1:])
@pytest.mark.parametrize("D", [768, 1280, 2048])
def test_layernorm_pooled_gathers(lib, D, out):
    """The pooled LayerNorms read one row per sample: group = S with row_off = 0 (CLS token: ViT, CLIP vision), row_off = S - 1
    (SigLIP text), and row_index (CLIP EOT).  Each gives the bits of the dense kernel on the gathered rows, in both walks."""
    dt, code = out
    B, S = 300, 77
    x = _randn(B * S, D, seed=D + 3) * 2 - 0.5
    scale, bias = _randn(D, seed=D + 4), _randn(D, seed=D + 5)
    idx = torch.randint(0, S, (B,), generator=torch.Generator().manual_seed(D), dtype=torch.int32).to(DEV)
    x3 = x.view(B, S, D)
    for off, index, rows in ((0, None, x3[:, 0]), (S - 1, None, x3[:, S - 1]), (0, idx, x3[torch.arange(B, device=DEV), idx.long()])):
        dense = torch.empty(B, D, dtype=dt, device=DEV)
        layernorm_ex(lib, rows.contiguous(), dense, code, 1e-5, scale, bias)
        for reverse in (0, 1):
            got = torch.full((B + 5, D), SENTINEL, dtype=dt, device=DEV)
            layernorm_ex(lib, x, got, code, 1e-5, scale, bias, rows=B, group=S, row_off=off, index=index, reverse=reverse)
            torch.cuda.synchronize()
            assert torch.equal(got[:B], dense), (off, index is not None, reverse)
            assert _untouched(got[B:])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [256, 768, 1280, 2048])
@pytest.mark.parametrize("eps", [1e-12, 1e-6, 1e-5])
def test_layernorm_variance_near_eps(lib, eps, D):
    """Rows whose variance lies in [0.1, 10] * eps: rsqrt(var + eps) differs there from rsqrt(max(var, eps)) or any other eps by
    several percent.  Row means within two standard deviations of zero (the fast-variance formula cancels no more than that)."""
    rows = 512
    g = torch.Generator(device="cpu").manual_seed(D)
    z = torch.randn(rows, D, generator=g, dtype=torch.float64)
    z = (z - z.mean(-1, keepdim=True)) / z.std(-1, correction=0, keepdim=True)
    var = eps * 10 ** (torch.rand(rows, 1, generator=g, dtype=torch.float64) * 2 - 1)
    mean = (torch.rand(rows, 1, generator=g, dtype=torch.float64) * 4 - 2) * var.sqrt()
    x = (z * var.sqrt() + mean).float().to(DEV)
    scale, bias = _randn(D, seed=D + 6), _randn(D, seed=D + 7)
    out = torch.empty(rows, D, device=DEV)
    layernorm_ex(lib, x, out, F32, eps, scale, bias)
    ref = _fast_var_ln(x, scale, bias, eps)
    xd = x.double()
    v = (xd * xd).mean(-1) - xd.mean(-1) ** 2
    assert float(v.min()) > 0.09 * eps and float(v.max()) < 11 * eps
    assert rel_err(out, ref) < 2e-5, rel_err(out, ref)


# ---- every LayerNorm epsilon observable at model level --------------------------------------------------------------------------------
# Two-layer models, fp32 (tf32) mode.  The embeddings and the CLIP pre-norm's scale and bias (EMBED) are scaled by the first factor
# of EPS_SCALE, the kernels and biases of every projection that adds into a LayerNorm input (attention out, FC2, the MAP head's
# attention out: RESIDUAL) by the second, so each LayerNorm sees rows of variance about 1e-6 .. 1e-5: there 1e-12, 1e-6 and 1e-5
# give clearly different outputs.  fp16 is left out: the scaled weights fall below fp16's normal range.
EPS_SCALE = {"vit": (1.5e-3, 2e-3), "clip_image": (2.5e-3, 1e-3), "clip_text": (2.5e-3, 2e-3), "siglip_image": (1.5e-3, 2e-3),
             "siglip_text": (2.5e-3, 1e-3)}
EPS_USED = (1e-12, 1e-6, 1e-5)
EMBED = ("patch_embeddings.kernel", "patch_embeddings.bias", "position_embeddings", "cls_token", "ln_pre.scale", "ln_pre.bias",
         "token_embedding.embedding", "positional_embedding")
RESIDUAL = ("attn.out.kernel", "attn.out.bias", "mlp.layers.3.kernel", "mlp.layers.3.bias")
VIT = O.ViTCfg(num_classes=10, img_size=32, patch_size=8, num_layers=2, num_heads=2, mlp_dim=512, hidden_size=128)
DUAL = {"clip": O.DualCfg(64, 2, 256, 16, 20, 300, 128, 2, 2), "siglip": O.DualCfg(64, 2, 256, 16, 20, 300, 256, 4, 2)}
_LAYER_NORM = O.layer_norm


def _eps_case(kind):
    """(scaled parameters, input, oracle forward, CUDA model forward)."""
    from jimm_b200.models import CLIP, SigLIP, VisionTransformer

    if kind == "vit":
        p = O.random_vit_params(VIT, seed=51)
        x = O.synthetic_images(4, 32, seed=52)
        fwd = lambda: O.vit_forward(p, VIT, x)  # noqa: E731
        model = lambda: VisionTransformer(num_classes=10, img_size=32, patch_size=8, num_layers=2, num_heads=2, mlp_dim=512,  # noqa: E731
                                          hidden_size=128, dtype=torch.float32)
        run = lambda m: m(x.cuda())  # noqa: E731
    else:
        dual, tower = kind.split("_")
        cfg = DUAL[dual]
        p = O.random_dual_params(cfg, dual, seed=53)
        x = O.synthetic_images(4, 64, seed=54) if tower == "image" else O.synthetic_tokens(5, 20, 300, dual, seed=55)
        fn = {("clip", "image"): O.clip_encode_image, ("clip", "text"): O.clip_encode_text, ("siglip", "image"): O.siglip_encode_image,
              ("siglip", "text"): O.siglip_encode_text}[dual, tower]
        fwd = lambda: fn(p, cfg, x)  # noqa: E731
        model = lambda: (CLIP if dual == "clip" else SigLIP)(64, 2, 256, 16, 20, 300, cfg.transformer_width, cfg.transformer_heads, 2,  # noqa: E731
                                                             dtype=torch.float32)
        run = lambda m: m.encode_image(x.cuda()) if tower == "image" else m.encode_text(x.cuda())  # noqa: E731
    for k in p:
        if k.endswith(EMBED):
            p[k] = p[k] * EPS_SCALE[kind][0]
        elif k.endswith(RESIDUAL):
            p[k] = p[k] * EPS_SCALE[kind][1]
    return p, fwd, model, run


def _record_layer_norms(monkeypatch, change=None):
    """Replace jimm_oracle.layer_norm by one that records (eps, smallest and largest row variance) of every call; change = (i, eps')
    runs call i with eps' instead."""
    calls = []

    def ln(x, scale, bias, eps, sem=None):
        xd = x.double()
        var = (xd * xd).mean(-1) - xd.mean(-1) ** 2
        calls.append((eps, float(var.min()), float(var.max())))
        if change is not None and len(calls) - 1 == change[0]:
            eps = change[1]
        return _LAYER_NORM(x, scale, bias, eps, sem)

    monkeypatch.setattr(O, "layer_norm", ln)
    return calls


@pytest.mark.parametrize("kind", list(EPS_SCALE))
def test_every_layernorm_epsilon_moves_the_oracle(kind, monkeypatch):
    """The premise of test_every_layernorm_epsilon_at_model_level, checked on the oracle (CPU).  Every LayerNorm input row has a
    variance within [0.1, 10] * eps (for the 1e-12 norms: * 1e-6, the epsilon they could be mistaken for).  Running any single
    LayerNorm with its epsilon times 10, or with any other epsilon the models use, moves the output by at least 20x the parity bar.
    (1e-12 times 10 is left out: at a variance where 1e-6 is visible, 1e-11 cannot be.)"""
    p, fwd, _, _ = _eps_case(kind)
    with torch.no_grad():
        calls = _record_layer_norms(monkeypatch)
        ref = fwd()
        assert len(calls) >= 5
        for i, (eps, vmin, vmax) in enumerate(calls):
            e = max(eps, 1e-6)
            assert 0.1 * e <= vmin and vmax <= 10 * e, (kind, i, eps, vmin, vmax)
            for alt in [e for e in EPS_USED if e != eps] + ([eps * 10] if eps >= 1e-6 else []):
                _record_layer_norms(monkeypatch, (i, alt))
                moved = rel_err(fwd(), ref)
                assert moved >= 20 * TOL, (kind, i, eps, alt, moved)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(EPS_SCALE))
def test_every_layernorm_epsilon_at_model_level(kind):
    """ViT (outer 1e-12, blocks 1e-6), CLIP (vision pre / post norm 1e-5, text ln_final 1e-5, blocks 1e-6) and SigLIP (all 1e-6,
    MAP head included) against the oracle at the parity bar, with every LayerNorm input at variance near its eps: any LayerNorm given
    another epsilon would miss the bar by 20x or more (test_every_layernorm_epsilon_moves_the_oracle)."""
    p, fwd, model, run = _eps_case(kind)
    with torch.no_grad():
        ref = fwd()
    m = model()
    for k, v in p.items():
        m.set_flat_param(k, v.to(torch.float32))
    check_parity(f"every LayerNorm eps observable, {kind}", "output", torch.float32, "fp32", run(m), ref, TOL)


# ---- CLIP end-of-text pooling with HuggingFace padding --------------------------------------------------------------------------------
EOT_FIRST = [5, 31, 32, 40, 63, 64, 76, 1]  # 76 = T - 1 alone; 1: EOT from position 1 to the end


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_clip_eot_pooling_with_padding(dtype):
    """CLIP pools the first end-of-text token (jnp.argmax: the first maximum).  HuggingFace tokenizers pad with the EOT id, so rows
    hold it from their first EOT to the end; the argmax kernel's 32 lanes then see ties, and the first EOT at or after position 32
    ties with later ones in other lanes.  Against the oracle (torch.argmax returns the first maximum too).  Under the causal mask a
    row's pooled token sees nothing after it, so cutting the rows at the last first-EOT gives the same embeddings bit for bit."""
    from jimm_b200.models import CLIP

    T, V = 77, 1000
    cfg = O.DualCfg(32, 1, 128, 16, T, V, 256, 4, 2)
    p = O.random_dual_params(cfg, "clip", seed=61)
    g = torch.Generator().manual_seed(62)
    ids = torch.randint(1, V - 1, (len(EOT_FIRST), T), generator=g)
    for r, e in enumerate(EOT_FIRST):
        ids[r, e:] = V - 1
    with torch.no_grad():
        ref = O.clip_encode_text(p, cfg, ids)
    m = CLIP(32, 1, 128, 16, T, V, 256, 4, 2, dtype=dtype)
    for k, v in p.items():
        m.set_flat_param(k, v.to(torch.float32))
    full = m.encode_text(ids.cuda())
    check_parity("CLIP text, EOT padding", "text_embeds", dtype, "fp32", full, ref, TOL)
    cut = [r for r, e in enumerate(EOT_FIRST) if e < T - 1]
    Tc = max(EOT_FIRST[r] for r in cut) + 1
    sub = ids[cut].cuda()
    assert torch.equal(m.encode_text(sub[:, :Tc].contiguous()), m.encode_text(sub))
