"""Mirror of jimm.common.transformer (reference: src/jimm/common/transformer.py): same class names, constructor kwargs, parameter
tree and `__call__`.  The arithmetic of a block runs inside the CUDA library (LayerNorm -> fused QKV wgmma GEMM -> wgmma
attention -> out-proj GEMM + residual -> LayerNorm -> FC1 GEMM + GELU -> FC2 GEMM + residual): inside a tower it is driven by
VisionTransformerBase / CLIP / SigLIP; called on their own, `Transformer` / `TransformerEncoder` build a native handle of just
that stack (jimm_encoder_forward) and run the same kernels on [batch, seq, hidden] activations."""

from __future__ import annotations

import torch

from .. import _lib, nn


def quickgelu(x) -> torch.Tensor:
    """x * sigmoid(1.702 x) (common/transformer.py:12-19) as a CUDA kernel (jimm_k_activation); inside the towers the same function is
    the FC1 GEMM's fused epilogue."""
    from .._runtime import activation

    return activation(x, 2)


def _is_causal_mask(mask) -> bool:
    """The only mask the reference builds is `jnp.tril(jnp.ones((T, T)))` (models/clip.py:62); non-zero = keep."""
    m = torch.as_tensor(mask.tolist() if hasattr(mask, "tolist") and not isinstance(mask, torch.Tensor) else mask)
    if m.ndim != 2 or m.shape[0] != m.shape[1]:
        return False
    return bool(torch.equal(m != 0, torch.tril(torch.ones_like(m, dtype=torch.bool))))


class _SubModuleRunner:
    """Lazily builds (and rebuilds when parameters / batch / sequence bounds change) the native handle of a bare block stack."""

    def _sub_init(self, dtype):
        object.__setattr__(self, "_sub", None)
        object.__setattr__(self, "_sub_dtype", nn.compute_dtype_code(dtype))

    def _invalidate(self):
        if getattr(self, "_sub", None) is not None:
            self._sub.close()
        object.__setattr__(self, "_sub", None)

    def _sub_config(self, max_seq: int) -> _lib.Config:
        raise NotImplementedError

    def _sub_params(self):
        return self.flat_params()

    def _run(self, x):
        from .._runtime import NativeSubModule, default_max_batch

        if getattr(x, "ndim", None) != 3:
            raise ValueError(f"expected activations of shape [batch, seq, hidden], got {tuple(getattr(x, 'shape', ()))}")
        B, S = int(x.shape[0]), int(x.shape[1])
        sub = self._sub
        if sub is None or S > sub.max_seq:
            if sub is not None:  # dropped first: a refused rebuild (a sequence past the MAP head's limit) leaves no closed handle behind
                self._invalidate()
            # workspace for `rows` tokens: batches beyond that are chunked by the library
            mb = max(1, min(default_max_batch(), max(1, 65536 // S)))
            sub = NativeSubModule(self._sub_config(S), self._sub_params(), mb)
            object.__setattr__(self, "_sub", sub)
        return sub(x)


def _encoder_config(width, mlp_dim, layers, num_heads, eps, use_quick_gelu, attn_mask, dtype_code, max_seq) -> _lib.Config:
    if attn_mask is not None and not _is_causal_mask(attn_mask):
        raise NotImplementedError("attention masks other than the lower-triangular (causal) mask the reference builds (models/clip.py:62) "
                                  "are not supported by the attention kernels")
    cfg = _lib.Config()
    cfg.kind = _lib.KIND_ENCODER
    cfg.v_width, cfg.v_layers, cfg.v_heads, cfg.v_mlp = width, layers, num_heads, mlp_dim
    cfg.v_act = _lib.ACT_QUICK_GELU if use_quick_gelu else _lib.ACT_GELU_TANH
    cfg.v_eps_block = cfg.v_eps_outer = float(eps)
    cfg.t_causal = int(attn_mask is not None)
    cfg.ctx_len = int(max_seq)
    cfg.compute_dtype = dtype_code
    return cfg


class TransformerEncoder(_SubModuleRunner, nn.Module):
    """common/transformer.py:22-132."""

    def __init__(self, hidden_size: int, mlp_dim: int, num_heads: int, layernorm_epsilon=1e-5, dropout_rate: float = 0.0,
                 attn_mask=None, use_quick_gelu: bool = False, dtype=None, param_dtype=None, rngs=None, mesh=None) -> None:
        nn.Module.__init__(self)
        self._sub_init(dtype)
        object.__setattr__(self, "attn_mask", attn_mask)
        object.__setattr__(self, "layernorm_epsilon", layernorm_epsilon)
        object.__setattr__(self, "use_quick_gelu", use_quick_gelu)
        object.__setattr__(self, "_dims", (hidden_size, mlp_dim, num_heads))
        g = nn._gen(rngs)
        self.add_child("norm1", nn.LayerNorm(hidden_size, layernorm_epsilon))
        self.add_child("attn", nn.MultiHeadAttention(num_heads, hidden_size, rngs=g_wrap(g)))
        self.add_child("norm2", nn.LayerNorm(hidden_size, layernorm_epsilon))
        # nnx.Sequential [Linear, act, Dropout, Linear, Dropout] -> param indices 0 and 3 (:92-114)
        self.add_child("mlp", nn.Sequential(nn.Linear(hidden_size, mlp_dim, rngs=g_wrap(g)), None, None,
                                            nn.Linear(mlp_dim, hidden_size, rngs=g_wrap(g)), None))

    def _sub_config(self, max_seq):
        D, M, H = self._dims
        return _encoder_config(D, M, 1, H, self.layernorm_epsilon, self.use_quick_gelu, self.attn_mask, self._sub_dtype, max_seq)

    def _sub_params(self):
        return {"blocks.layers.0." + k: v for k, v in self.flat_params().items()}  # a stack of one block

    def __call__(self, x):
        """[batch, seq, hidden] -> [batch, seq, hidden] (common/transformer.py:116-132): x + attn(norm1(x)), then x + mlp(norm2(x)); the mask,
        when given, is sliced to the sequence length like the reference (:125-129)."""
        return self._run(x)


class _G(nn.Rngs):
    def __init__(self, g):
        self.seed = 0
        self._gen = g


def g_wrap(g):
    return _G(g)


class Transformer(_SubModuleRunner, nn.Module):
    """common/transformer.py:135-196.  NOTE the default layernorm_epsilon=1e-6 (:142) is what every tower gets, because
    VisionTransformerBase and CLIP never forward their own epsilon (SURVEY.md quirk 2)."""

    def __init__(self, width: int, mlp_dim: int, layers: int, num_heads: int, layernorm_epsilon=1e-6, dropout_rate: float = 0.0,
                 attn_mask=None, use_quick_gelu: bool = False, dtype=None, param_dtype=None, rngs=None, mesh=None):
        nn.Module.__init__(self)
        self._sub_init(dtype)
        for k, v in dict(width=width, layers=layers, num_heads=num_heads, dropout_rate=dropout_rate, mlp_dim=mlp_dim,
                         layernorm_epsilon=layernorm_epsilon, use_quick_gelu=use_quick_gelu, attn_mask=attn_mask).items():
            object.__setattr__(self, k, v)
        g = nn._gen(rngs)
        blocks = nn.Module()
        blocks.add_child("layers", nn.ModuleList([
            TransformerEncoder(width, mlp_dim, num_heads, layernorm_epsilon, dropout_rate, attn_mask, use_quick_gelu, dtype,
                               param_dtype, g_wrap(g), mesh) for _ in range(layers)]))
        self.add_child("blocks", blocks)

    def _sub_config(self, max_seq):
        return _encoder_config(self.width, self.mlp_dim, self.layers, self.num_heads, self.layernorm_epsilon, self.use_quick_gelu, self.attn_mask,
                               self._sub_dtype, max_seq)

    def __call__(self, x):
        """[batch, seq, width] -> [batch, seq, width]: the blocks in order (common/transformer.py:190-196)."""
        return self._run(x)
