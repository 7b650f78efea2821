"""Minimal module system mirroring the parts of flax.nnx the reference uses on the forward path: a parameter tree
whose flat paths equal the reference's `nnx.to_flat_state(nnx.state(model, nnx.Param))` keys, `eval()` / `train()`,
and seeded initialisers with the reference's distributions.  Parameters live on the host as fp32 torch tensors in
the reference's (flax) layouts; the device copy is packed by the CUDA library at finalize time."""

from __future__ import annotations

import math
from typing import Dict, Iterator, List, Optional, Tuple

import torch

from . import _lib


class Rngs:
    """Stand-in for `nnx.Rngs(seed)`: one seeded torch generator drawn from in construction order."""

    def __init__(self, seed: int = 0, **_ignored):
        self.seed = int(seed)
        self._gen = torch.Generator().manual_seed(self.seed)

    def params(self) -> torch.Generator:
        return self._gen


def _gen(rngs) -> torch.Generator:
    if rngs is None:
        return Rngs(0).params()
    if isinstance(rngs, Rngs):
        return rngs.params()
    if isinstance(rngs, int):
        return Rngs(rngs).params()
    seed = getattr(rngs, "seed", 0)
    return Rngs(seed if isinstance(seed, int) else 0).params()


# ---- initialisers (same distributions as the reference: common/vit.py:163-171, common/transformer.py:64-78) ----
_SKIP_INIT = False


class deferred_init:
    """Inside this context the random initialisers only allocate: `from_pretrained` overwrites every parameter (and asserts that
    it did, like the reference's visit checks), so drawing 86 M random numbers first is 60 % of the loader's time for nothing."""

    def __enter__(self):
        global _SKIP_INIT
        self._prev, _SKIP_INIT = _SKIP_INIT, True
        return self

    def __exit__(self, *exc):
        global _SKIP_INIT
        _SKIP_INIT = self._prev
        return False


def xavier_uniform(g, shape, fan_in, fan_out):
    if _SKIP_INIT:
        return torch.empty(shape, dtype=torch.float32)
    a = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1) * a


def truncated_normal(g, shape, stddev=0.02):
    if _SKIP_INIT:
        return torch.empty(shape, dtype=torch.float32)
    t = torch.empty(shape, dtype=torch.float32)
    torch.nn.init.trunc_normal_(t, mean=0.0, std=1.0, a=-2.0, b=2.0, generator=g)
    return t * stddev


def zeros(shape):
    return torch.zeros(shape, dtype=torch.float32)


def ones(shape):
    return torch.ones(shape, dtype=torch.float32)


_DTYPE_NAMES = {"float32": _lib.F32, "float16": _lib.F16, "bfloat16": _lib.BF16, "half": _lib.F16, "float": _lib.F32,
                "float8_e4m3fn": _lib.F8E4M3}


def compute_dtype_code(dtype) -> int:
    """Accept torch / numpy / jax.numpy dtypes or strings (the reference's `dtype: DTypeLike`).

    float8_e4m3fn selects the FP8 mode: float16 everywhere except the QKV and FC1 GEMMs of each encoder block, which run on e4m3
    operands with power-of-two scales per token row and per output channel (parameters stay as loaded on the host; the weights are
    quantised on the GPU).  It is not held to the 1e-3 parity of the other modes."""
    if dtype is None:
        return _lib.F32
    if isinstance(dtype, int) and dtype in (_lib.F32, _lib.F16, _lib.BF16, _lib.F8E4M3):
        return dtype
    name = getattr(dtype, "__name__", None) or getattr(dtype, "name", None) or str(dtype)
    name = name.replace("torch.", "").replace("jnp.", "")
    if name in _DTYPE_NAMES:
        return _DTYPE_NAMES[name]
    raise ValueError(f"Unsupported dtype {dtype!r}: expected float32, float16, bfloat16 or float8_e4m3fn")


class LazyParam:
    """A parameter whose value is a VIEW of checkpoint memory (e.g. the mmap of a safetensors file) in its stored dtype:
        transposed=False:  flax value = base.reshape(shape)
        transposed=True :  base is the 2-D [N, K] transpose of the flax kernel's (K, N) view -- a HuggingFace (out, in) weight as stored;
                           flax value = base.T.reshape(shape)  (models/vit.py:241-250)
    Nothing is converted or copied on the CPU: the CUDA library receives the pointer (jimm_model_set_param_ref) and casts / packs on
    the GPU.  `materialize()` produces the fp32 tensor in the reference's layout for code that wants to look at the value."""

    __slots__ = ("base", "shape", "transposed")

    def __init__(self, base: torch.Tensor, shape, transposed: bool = False):
        self.base, self.shape, self.transposed = base, tuple(int(d) for d in shape), bool(transposed)

    def materialize(self) -> torch.Tensor:
        t = self.base.to(torch.float32)
        if self.transposed:
            t = t.reshape(t.shape[0], -1).T
        return t.reshape(self.shape).contiguous()


class Module:
    """Parameter-tree node.  Leaves are torch fp32 CPU tensors (or `LazyParam` views of a checkpoint); children are Modules."""

    def __init__(self):
        object.__setattr__(self, "_params", {})
        object.__setattr__(self, "_children", {})
        object.__setattr__(self, "_training", True)

    # -- tree construction --
    def add_param(self, name: str, value: torch.Tensor):
        self._params[name] = value.detach().to(torch.float32).contiguous()

    def add_child(self, name, module: "Module"):
        self._children[str(name)] = module
        return module

    def __getattr__(self, name):
        ch = object.__getattribute__(self, "_children")
        if name in ch:
            return ch[name]
        pr = object.__getattribute__(self, "_params")
        if name in pr:
            v = pr[name]
            return v.materialize() if isinstance(v, LazyParam) else v
        raise AttributeError(f"{type(self).__name__!s} has no attribute {name!r}")

    # -- flat state (== the reference's flat-state keys joined with '.') --
    def flat_params(self, prefix: str = "", raw: bool = False) -> Dict[str, torch.Tensor]:
        """{flax path: fp32 tensor in the reference's layout}; raw=True keeps `LazyParam` entries as they are (the native hand-off)."""
        out: Dict[str, torch.Tensor] = {}
        for k, v in self._params.items():
            out[prefix + k] = v if raw or not isinstance(v, LazyParam) else v.materialize()
        for k, c in self._children.items():
            out.update(c.flat_params(prefix + k + ".", raw))
        return out

    def flat_param_shapes(self, prefix: str = "") -> Dict[str, Tuple[int, ...]]:
        out: Dict[str, Tuple[int, ...]] = {}
        for k, v in self._params.items():
            out[prefix + k] = tuple(v.shape)
        for k, c in self._children.items():
            out.update(c.flat_param_shapes(prefix + k + "."))
        return out

    def set_flat_param(self, path: str, value):
        parts = path.split(".")
        node = self
        for p in parts[:-1]:
            node = node._children[p]
        if parts[-1] not in node._params:
            raise KeyError(path)
        node._params[parts[-1]] = value if isinstance(value, LazyParam) else value.detach().to(torch.float32).contiguous()
        self._invalidate()

    def _invalidate(self):
        pass

    # -- nnx.Module API used by the reference's scripts (examples/vit_inference.py:22, examples/vit_training.py:215) --
    def eval(self):
        self._set_training(False)
        return self

    def train(self):
        self._set_training(True)
        return self

    def _set_training(self, flag: bool):
        object.__setattr__(self, "_training", flag)
        for c in self._children.values():
            c._set_training(flag)

    @property
    def training(self) -> bool:
        return self._training


class ModuleList(Module):
    def __init__(self, modules: List[Module]):
        super().__init__()
        for i, m in enumerate(modules):
            self.add_child(i, m)

    def __getitem__(self, i):
        return self._children[str(i)]

    def __len__(self):
        return len(self._children)

    def __iter__(self) -> Iterator[Module]:
        return iter(self._children.values())


class Sequential(Module):
    """nnx.Sequential: children live under `layers.{i}`; non-module entries (activations, dropout) keep their index."""

    def __init__(self, *layers):
        super().__init__()
        holder = Module()
        for i, l in enumerate(layers):
            if isinstance(l, Module):
                holder.add_child(i, l)
        self.add_child("layers", holder)


class Linear(Module):
    """nnx.Linear parameter holder: kernel (in, out), bias (out)."""

    def __init__(self, in_features, out_features, use_bias=True, rngs=None):
        super().__init__()
        g = _gen(rngs)
        self.add_param("kernel", xavier_uniform(g, (in_features, out_features), in_features, out_features))
        if use_bias:
            self.add_param("bias", zeros((out_features,)))


class LayerNorm(Module):
    def __init__(self, num_features, epsilon=1e-6, rngs=None):
        super().__init__()
        object.__setattr__(self, "epsilon", epsilon)
        self.add_param("scale", ones((num_features,)))
        self.add_param("bias", zeros((num_features,)))


class _Proj(Module):
    def __init__(self, kshape, bshape, fan_in, fan_out, g):
        super().__init__()
        self.add_param("kernel", xavier_uniform(g, kshape, fan_in, fan_out))
        self.add_param("bias", zeros(bshape))


class MultiHeadAttention(Module):
    """nnx.MultiHeadAttention parameter holder: query/key/value kernels (D,H,d), out kernel (H,d,D)."""

    def __init__(self, num_heads, in_features, rngs=None):
        super().__init__()
        g = _gen(rngs)
        D, H = in_features, num_heads
        if D % H != 0:
            raise ValueError(f"Memory dimension ({D}) must be divisible by 'num_heads' heads ({H}).")
        d = D // H
        for name in ("query", "key", "value"):
            self.add_child(name, _Proj((D, H, d), (H, d), D, D, g))
        self.add_child("out", _Proj((H, d, D), (D,), D, D, g))


class Conv(Module):
    """nnx.Conv parameter holder: kernel (P,P,C,D) HWIO, bias (D)."""

    def __init__(self, in_features, out_features, kernel_size, use_bias=True, rngs=None):
        super().__init__()
        g = _gen(rngs)
        kh, kw = kernel_size
        self.add_param("kernel", xavier_uniform(g, (kh, kw, in_features, out_features), kh * kw * in_features, kh * kw * out_features))
        if use_bias:
            self.add_param("bias", zeros((out_features,)))


class Embed(Module):
    def __init__(self, num_embeddings, features, rngs=None):
        super().__init__()
        g = _gen(rngs)
        self.add_param("embedding", xavier_uniform(g, (num_embeddings, features), num_embeddings, features))
