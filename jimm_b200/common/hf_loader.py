"""HuggingFace checkpoint -> the reference's flax parameter tree, without touching the bytes on the CPU.

The reference's `from_pretrained` (models/vit.py:192-268, models/clip.py:269-416, models/siglip.py:228-385) walks a {flax path: HF name}
table, applies a layout transform per entry and checks that every parameter on both sides is accounted for.  The tables stay in the
model files (they are the contract); this module applies them.  Kernels are NOT transposed here: a HuggingFace `(out, in)` weight is
wrapped in a `LazyParam(transposed=True)` -- it already is the K-major operand the GEMMs read -- and handed to the CUDA library by
pointer; biases / norms / embeddings stay views of the checkpoint memory in their stored dtype."""

from __future__ import annotations

from typing import Callable, Dict, Iterable, Optional, Set, Tuple

import torch

from ..nn import LazyParam

# per-entry transform kinds
ASIS = "asis"          # same element order, possibly a different rank (cls token, position table, squeezed scalars)
LINEAR = "linear"      # nn.Linear weight (out, in)            -> nnx.Linear kernel (in, out)
QKV_W = "qkv_w"        # q/k/v projection weight (H*d, D)      -> (D, H, d)
QKV_B = "qkv_b"        # q/k/v projection bias (H*d)           -> (H, d)
OUT_W = "out_w"        # attention output weight (D, H*d)      -> (H, d, D)
CONV = "conv"          # patch conv weight (D, C, P, P)        -> HWIO (P, P, C, D)
PATCH_LINEAR = "patch_linear"  # SigLIP 2 NaFlex patch Linear weight (D, P*P*C), columns in (py, px, c) order -> HWIO (P, P, C, D)

KNOWN_UNUSED = {"text_model.embeddings.position_ids", "vision_model.embeddings.position_ids"}  # models/vit.py:262-265


def convert(t: torch.Tensor, kind: str, flax_shape: Tuple[int, ...], rows: Optional[Tuple[int, int]] = None):
    """The flax-layout value of HF tensor `t` (optionally its row block rows=(i, n): the i-th of n equal chunks along dim 0, for the packed
    MAP-head in_proj tensors, models/siglip.py:352-363), or None when the shapes cannot match."""
    if rows is not None:
        i, n = rows
        if t.shape[0] % n:
            return None
        step = t.shape[0] // n
        t = t[i * step:(i + 1) * step]
    numel = 1
    for d in flax_shape:
        numel *= d
    if kind == CONV:
        if t.ndim != 4:
            return None
        v = t.permute(2, 3, 1, 0)
        return v if tuple(v.shape) == tuple(flax_shape) else None
    if kind == PATCH_LINEAR:  # the (P*P*C, D) view of the HWIO kernel, transposed: the K-major operand as stored
        if t.ndim != 2 or tuple(t.shape) != (flax_shape[-1], numel // flax_shape[-1]):
            return None
        return LazyParam(t if t.is_contiguous() else t.contiguous(), flax_shape, transposed=True)
    if kind in (LINEAR, QKV_W, OUT_W):
        if t.ndim != 2 or t.numel() != numel:
            return None
        if kind == LINEAR and tuple(t.shape) != (flax_shape[1], flax_shape[0]):
            return None
        if kind == QKV_W and tuple(t.shape) != (flax_shape[1] * flax_shape[2], flax_shape[0]):
            return None
        if kind == OUT_W and tuple(t.shape) != (flax_shape[2], flax_shape[0] * flax_shape[1]):
            return None
        return LazyParam(t if t.is_contiguous() else t.contiguous(), flax_shape, transposed=True)
    if t.numel() != numel:
        return None
    if kind == QKV_B and (t.ndim != 1 or len(flax_shape) != 2):
        return None
    if t.numel() >= 1 << 16:  # large tables (token embedding): keep the view, no fp32 copy on the host
        return LazyParam(t if t.is_contiguous() else t.contiguous(), flax_shape, transposed=False)
    return t.reshape(flax_shape)


def shape_of(v) -> Tuple[int, ...]:
    return tuple(v.shape)


def apply_mapping(model, hf: Dict[str, torch.Tensor], rules: Iterable[Tuple], *, missing: str, shape_error: Callable[[str], Exception],
                  what: str) -> None:
    """rules: (flax_path, hf_name, kind[, rows]).  missing = "assert" (ViT: both names must exist, models/vit.py:229-232) | "skip"
    (CLIP: entries absent on either side are skipped, models/clip.py:343-345) | "strict" (SigLIP).  Afterwards every flax parameter must
    have been visited and every HF tensor used (except the known position_ids buffers)."""
    want = model.flat_param_shapes()
    unvisited: Set[str] = set(want)
    used: Set[str] = set()
    for rule in rules:
        dst, src, kind = rule[0], rule[1], rule[2]
        rows = rule[3] if len(rule) > 3 else None
        if missing == "skip" and (dst not in want or src not in hf):
            continue
        if missing == "assert":
            assert dst in want, dst
            assert src in hf, f"HF key '{src}' (from Flax key {dst}) not found in loaded weights."
        used.add(src)
        unvisited.discard(dst)
        v = convert(hf[src], kind, want[dst], rows)
        if v is None:
            got = tuple(hf[src].shape)
            raise shape_error(f"Shape mismatch for {dst} (Flax) vs {src} (HF): {want[dst]} (expected) != {got} (HF tensor, transform '{kind}')")
        model.set_flat_param(dst, v)
    assert len(unvisited) == 0, f"Some Flax {what}model parameters were not visited: {sorted(unvisited)}"
    unexpected = set(hf) - used - KNOWN_UNUSED
    assert len(unexpected) == 0, f"Some unexpected HuggingFace checkpoint parameters were not used: {sorted(unexpected)}"


def tower_arch(tower_config: dict, field: str, width: int, hf: Dict[str, torch.Tensor], prefix: str, default_act: str):
    """(heads, MLP width, use_quick_gelu) of one `width`-wide tower of a HF CLIP / SigLIP checkpoint from its `field` ("vision_config" /
    "text_config") dict.  A key the dict lacks takes its default: heads width // 64, the MLP width of the `prefix` tower's first fc1
    weight, hidden_act `default_act`.  hidden_act "quick_gelu" is QuickGELU; "gelu", "gelu_new" and "gelu_pytorch_tanh" run the tanh
    GELU, as VisionTransformer.from_pretrained maps "gelu"; any other value raises ValueError."""
    fc1 = hf.get(f"{prefix}.encoder.layers.0.mlp.fc1.weight")
    heads = int(tower_config.get("num_attention_heads", width // 64))
    mlp = int(tower_config.get("intermediate_size", fc1.shape[0] if fc1 is not None else 4 * width))
    act = tower_config.get("hidden_act", default_act)
    if act not in ("quick_gelu", "gelu", "gelu_new", "gelu_pytorch_tanh"):
        raise ValueError(f"{field}.hidden_act = {act!r} is not supported: the towers run 'quick_gelu' or the tanh GELU "
                         "('gelu', 'gelu_new', 'gelu_pytorch_tanh')")
    return heads, mlp, act == "quick_gelu"


def block_rules(flax_base: str, hf_base: str, names: Dict[str, str]):
    """The 16 entries of one encoder block.  `names` maps the role to the HF sub-path (they differ between ViT and CLIP / SigLIP)."""
    r = []
    for role in ("query", "key", "value"):
        r.append((flax_base + f"attn.{role}.kernel", hf_base + names[role] + ".weight", QKV_W))
        r.append((flax_base + f"attn.{role}.bias", hf_base + names[role] + ".bias", QKV_B))
    r.append((flax_base + "attn.out.kernel", hf_base + names["out"] + ".weight", OUT_W))
    r.append((flax_base + "attn.out.bias", hf_base + names["out"] + ".bias", ASIS))
    for flax_n, role in (("norm1", "ln1"), ("norm2", "ln2")):
        r.append((flax_base + flax_n + ".scale", hf_base + names[role] + ".weight", ASIS))
        r.append((flax_base + flax_n + ".bias", hf_base + names[role] + ".bias", ASIS))
    for idx, role in ((0, "fc1"), (3, "fc2")):
        r.append((flax_base + f"mlp.layers.{idx}.kernel", hf_base + names[role] + ".weight", LINEAR))
        r.append((flax_base + f"mlp.layers.{idx}.bias", hf_base + names[role] + ".bias", ASIS))
    return r


VIT_BLOCK = {"query": "attention.attention.query", "key": "attention.attention.key", "value": "attention.attention.value",
             "out": "attention.output.dense", "ln1": "layernorm_before", "ln2": "layernorm_after", "fc1": "intermediate.dense", "fc2": "output.dense"}
CLIP_BLOCK = {"query": "self_attn.q_proj", "key": "self_attn.k_proj", "value": "self_attn.v_proj", "out": "self_attn.out_proj",
              "ln1": "layer_norm1", "ln2": "layer_norm2", "fc1": "mlp.fc1", "fc2": "mlp.fc2"}
