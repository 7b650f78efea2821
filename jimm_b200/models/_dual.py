"""Shared machinery of the CLIP / SigLIP mirrors: text-tower parameter tree, native config, multi-GPU contrastive head."""

from __future__ import annotations

import torch

from .. import _lib, nn
from .._runtime import GalleryIndex, Texts, _call, prep_blocks, prep_ids, prep_layers, prep_texts, tokens_result
from ..common.transformer import Transformer, g_wrap
from ..common.vit import _NativeOwner, tower_config_fields


class DualTower(_NativeOwner, nn.Module):
    """Base of CLIP and SigLIP: holds the shared attributes and the encode / call plumbing."""

    _kind = None

    def _init_common(self, image_resolution, vision_layers, vision_width, vision_patch_size, context_length, vocab_size,
                     transformer_width, transformer_heads, transformer_layers, dtype, *, vision_heads, vision_mlp_dim, text_mlp_dim,
                     vision_quick_gelu, text_quick_gelu):
        """The shared attributes.  vision_heads / vision_mlp_dim / text_mlp_dim None: the reference's rule, vision_width // 64 heads
        (models/clip.py:60, models/siglip.py:59) and MLPs 4x the width."""
        nn.Module.__init__(self)
        self._native_init(dtype)
        for k, v in dict(image_resolution=image_resolution, vision_layers=vision_layers, vision_width=vision_width,
                         vision_patch_size=vision_patch_size, context_length=context_length, vocab_size=vocab_size,
                         transformer_width=transformer_width, transformer_heads=transformer_heads,
                         transformer_layers=transformer_layers, dtype=dtype, vision_heads=vision_heads or vision_width // 64,
                         vision_mlp_dim=vision_mlp_dim or 4 * vision_width, text_mlp_dim=text_mlp_dim or 4 * transformer_width,
                         vision_quick_gelu=bool(vision_quick_gelu), text_quick_gelu=bool(text_quick_gelu)).items():
            object.__setattr__(self, k, v)
        object.__setattr__(self, "_comm_mode", None)

    def _text_config(self, cfg: _lib.Config, *, causal, pool, head_bias, eps_outer):
        cfg.ctx_len, cfg.vocab, cfg.t_width = self.context_length, self.vocab_size, self.transformer_width
        cfg.t_heads, cfg.t_layers, cfg.t_mlp = self.transformer_heads, self.transformer_layers, self.text_mlp_dim
        cfg.t_act = _lib.ACT_QUICK_GELU if self.text_quick_gelu else _lib.ACT_GELU_TANH
        cfg.t_causal, cfg.t_pool, cfg.t_head_bias = causal, pool, head_bias
        cfg.t_eps_outer = eps_outer
        cfg.t_eps_block = 1e-6  # Transformer default (common/transformer.py:142); CLIP does not forward 1e-5 (models/clip.py:92-104)
        cfg.compute_dtype = self._compute_dtype
        return cfg

    # ---- reference API ----
    def encode_image(self, image, interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """interpolate_pos_encoding (HuggingFace's keyword): images of any size of at least one patch, the position embeddings
        resampled bicubically to the patch grid.  A list / tuple of images of different sizes runs in one packed call; row i is the
        embedding of image[i] alone."""
        return self._vision(image, interpolate_pos_encoding, encode=True)

    def _texts(self, text):
        """The text input step (prep_texts) for a list / tuple of token sequences, before any handle is built; a tensor as it is."""
        return prep_texts(text, self.context_length) if isinstance(text, (list, tuple)) else text

    def encode_text(self, text) -> torch.Tensor:
        """[B, T] token ids -> [B, E].  A list / tuple of token sequences of different lengths (each 1-D or [1, L], a tensor, numpy
        array or list of ints, 1 <= L <= context_length) runs in one packed call that skips the padding: row i is
        encode_text(text[i][None]), the call at T = len(text[i]).  For CLIP that is also the row of the padded call when text[i] is the
        padded row cut just after its EOT (its first maximum id): nothing after the EOT reaches the pooled token.  SigLIP pools the last
        token, so a list gives each sequence at its own length, not the padded embedding its checkpoint was trained on."""
        text = self._texts(text)
        return self.native().text(text) if isinstance(text, Texts) else self.native(text.shape[0]).text(text)

    def encode_image_tokens(self, image, layers=None, *, dtype=torch.float32, return_pooled: bool = False,
                            interpolate_pos_encoding: bool = False):
        """Per-token hidden states of the vision tower (HF's output_hidden_states) on the inputs encode_image takes: as
        VisionTransformerBase.forward_tokens, None being ln_post(x_L).  return_pooled: also return encode_image's result, bit for bit."""
        return self._vision_tokens(image, layers, dtype, return_pooled, interpolate_pos_encoding)

    def encode_text_tokens(self, text, layers=None, *, dtype=torch.float32, return_pooled: bool = False):
        """Per-token hidden states of the text tower on the inputs encode_text takes.  layers: an int k in [-(L+1), L] -- x_k, the fp32
        residual stream after k blocks (0: token embedding + positions; -1 is x_L) -- or None, the final-normed tokens ln_final(x_L); or a
        list / tuple of these, giving a tuple in request order.  Each result is [batch, T, width] of `dtype` (float32, float16 or
        bfloat16), every row as computed, those after an EOT or padding included; a list of sequences gives a list of [L_i, width].
        Without None or return_pooled only the blocks up to the deepest request run.  return_pooled: also return encode_text's result,
        bit for bit: (tokens, pooled)."""
        return self._text_tokens(text, prep_layers(layers, self.transformer_layers, dtype), return_pooled, False)

    def encode_image_attentions(self, image, blocks=None, *, dtype=torch.float32, return_pooled: bool = False,
                                interpolate_pos_encoding: bool = False):
        """Self-attention weights of the vision tower (HF's output_attentions) on the inputs encode_image takes: as
        VisionTransformerBase.forward_attentions ("map" on SigLIP's MAP head).  return_pooled: also return encode_image's result, bit
        for bit."""
        return self._vision_tokens(image, blocks, dtype, return_pooled, interpolate_pos_encoding, attn=True)

    def encode_text_attentions(self, text, blocks=None, *, dtype=torch.float32, return_pooled: bool = False):
        """Self-attention weights of the text tower (HF's output_attentions) on the inputs encode_text takes.  blocks: an int k in
        [-L, L-1], None (every block in order, a tuple) or a list / tuple of ints, giving a tuple in request order.  Each result is
        [batch, heads, T, T] of `dtype` (float32, float16 or bfloat16), every row as computed, those after an EOT or padding included;
        CLIP's text tower is causal, its entries above the diagonal 0.  A list of sequences gives a list of [heads, L_i, L_i].  Without
        return_pooled only the blocks up to the deepest request run.  return_pooled: also return encode_text's result, bit for bit."""
        return self._text_tokens(text, prep_blocks(blocks, self.transformer_layers, dtype, False), return_pooled, True)

    def _text_tokens(self, text, req, return_pooled: bool, attn: bool):
        """A per-token (NativeModel.text_tokens) or, attn, attention call (NativeModel.text_attn) of request req on the text inputs,
        checked before any handle is built."""
        text = self._texts(text)
        if not isinstance(text, Texts):
            text = prep_ids(text)
            if not 1 <= text.shape[1] <= self.context_length:
                raise ValueError(f"sequence length {text.shape[1]} outside 1 .. context_length={self.context_length}")
        n = self.native()
        toks, pooled = (n.text_attn if attn else n.text_tokens)(text, req, return_pooled)
        return tokens_result(toks, req, pooled, return_pooled)

    def __call__(self, image, text, interpolate_pos_encoding: bool = False) -> torch.Tensor:
        """Similarity logits.  Single process: [B_img, B_txt].  Under torch.distributed (one process per GPU, batch sharded
        over ranks like the reference's P("batch") inputs, examples/clip_inference.py:41-42): this rank's row block
        [B_local, world*B_local], embeddings exchanged over NVLink peer memory inside the fused logits kernel.
        interpolate_pos_encoding: as in encode_image.  `image` may be a list of images of different sizes and `text` a list of token
        sequences of different lengths, as in encode_text (single process only)."""
        return self._dual_call(image, text, interpolate_pos_encoding)

    def _dual_call(self, image, text, interpolate_pos_encoding: bool, **inputs):
        """__call__, with the further image inputs a model's _images takes (SigLIP 2 NaFlex's spatial_shapes / pixel_attention_mask;
        single process only)."""
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 and self._comm_mode != "off":
            if isinstance(image, (list, tuple)):
                raise ValueError("a list of images is not supported by the multi-GPU contrastive call; pass one [B, H, W, C] tensor per rank")
            if isinstance(text, (list, tuple)):
                raise ValueError("a list of token sequences is not supported by the multi-GPU contrastive call; pass one [B, T] tensor per rank")
            if any(v is not None for v in inputs.values()):
                raise ValueError("NaFlex pixel_values (spatial_shapes / pixel_attention_mask) are not supported by the multi-GPU contrastive "
                                 "call; pass one [B, H, W, C] tensor per rank")
            return self._call_distributed(image, text, interpolate_pos_encoding)
        im = self._images(image, interpolate_pos_encoding, **inputs)
        text = self._texts(text)
        Bt = len(text.lens) if isinstance(text, Texts) else text.shape[0]
        n = self.native(max(len(im.x), Bt), require=True, hw=im.hw if interpolate_pos_encoding else None)
        return n.dual(im, text)

    def search(self, queries, gallery, k: int):
        """Top-k retrieval without the score matrix: for each query embedding its k best gallery embeddings by this model's logit,
        `scores, indices` ([Q, k] fp32 and int32).  queries [Q, E] and gallery [N, E] are encode_image / encode_text outputs, either
        side either tower, fp32 / fp16 / bf16 on the device or the host (host results when both are on the host).  Bit for bit,
        search(encode_image(x), encode_text(t), k) == top_k(model(x, t), k) and search(encode_text(t), encode_image(x), k) ==
        top_k(model(x, t).T, k), at any Q and N; 1 <= k <= min(N, 1024).  Single GPU."""
        return self.native().search(queries, gallery, k)

    def index(self, gallery=None):
        """A gallery index: `gallery` ([N, E] embeddings as search takes them, fp32 / fp16 / bf16, device or host) normalised once and
        kept on the GPU.  `index.add(rows)` appends (indices continue), `len(index)` counts the rows, and `index.search(queries, k)`
        equals search(queries, every row added so far, k) bit for bit, with host results for host queries.  Each search screens the
        gallery on the tensor cores in fp16 and scores exactly only the rows that can still reach the best k.  The index keeps this
        model alive and follows its native handle: after a rebuild (a larger batch, set_flat_param, ...) the next add / search binds
        the stored rows to the new handle, so results stay equal to search with the model's current logit_scale / logit_bias.
        Single GPU; widths as the model has them (multiples of 8)."""
        return GalleryIndex(self.native, gallery)

    def set_comm(self, mode: str):
        """'peer' (default, fused NVLink peer-store kernel) | 'nccl' (torch.distributed all_gather baseline) | 'off'."""
        if mode not in ("peer", "nccl", "off"):
            raise ValueError(mode)
        object.__setattr__(self, "_comm_mode", mode)
        return self

    def _call_distributed(self, image, text, interpolate_pos_encoding: bool = False) -> torch.Tensor:
        import torch.distributed as dist

        im = self._images(image, interpolate_pos_encoding)
        x, B = im.x, len(im.x)
        n = self.native(B, require=True, hw=im.hw if interpolate_pos_encoding else None)
        ids = prep_ids(text)
        with torch.cuda.device(n.device):
            cur = torch.cuda.current_stream(n.device)
            # host inputs: the ids go first (H2D copies share one engine), the images follow on a side stream and land while
            # the text tower runs -- the same overlap as the single-GPU host path (csrc/model.cu jimm_dual_forward_host)
            ids_d = ids if ids.is_cuda else ids.to(n.device, non_blocking=True)
            if x.is_cuda:
                x_d = x
            else:
                side = n.side_stream()
                side.wait_stream(cur)
                with torch.cuda.stream(side):
                    x_d = x.to(n.device, non_blocking=True)
            if x.is_cuda:
                ie, te = n.dual_encode(x_d, ids_d)  # both towers concurrently (text forked onto the library's side stream)
            elif im.u8:
                # raw frames are a quarter of the bytes: take the short copy up front and run the two towers concurrently
                cur.wait_stream(side)
                x_d.record_stream(cur)
                ie, te = n.dual_encode(x_d, ids_d)
            else:
                te = n.text(ids_d)
                cur.wait_stream(side)
                x_d.record_stream(cur)
                ie = n.vision(x_d, encode=True, interpolate=interpolate_pos_encoding)
            return n._back(self._distributed_logits(n, ie, te, B), im.host and not ids.is_cuda).result()

    def _distributed_logits(self, n, ie, te, B) -> torch.Tensor:
        import torch.distributed as dist

        if (self._comm_mode or "peer") == "peer":
            if n._comm is None or n._comm[2] < B:
                n.comm_setup(max(B, n.max_batch))
            return n.comm_logits(ie, te)
        # NCCL baseline: normalise locally, all-gather the packed [B, 2E] buffer, logits for the local rows
        world = dist.get_world_size()
        i_n = ie / torch.linalg.norm(ie, dim=-1, keepdim=True)
        t_n = te / torch.linalg.norm(te, dim=-1, keepdim=True)
        gathered = torch.empty((world * B, t_n.shape[1]), dtype=torch.float32, device=n.device)
        dist.all_gather_into_tensor(gathered, t_n.contiguous())
        scale = self.logit_scale.to(n.device).reshape(1)
        bias = self.logit_bias.to(n.device).reshape(1) if "logit_bias" in self._params else None
        out = torch.empty((B, world * B), dtype=torch.float32, device=n.device)
        _call(n.lib, n.device, "jimm_k_logits", i_n, gathered, scale, bias, out, B, world * B, t_n.shape[1], world * B)
        return out


def build_text_tower(model: DualTower, g, *, head_bias: bool, layernorm_epsilon, attn_mask):
    Dt, T, V = model.transformer_width, model.context_length, model.vocab_size
    model.add_child("text_model", Transformer(width=Dt, mlp_dim=model.text_mlp_dim, layers=model.transformer_layers,
                                              num_heads=model.transformer_heads, dropout_rate=0.0, attn_mask=attn_mask,
                                              use_quick_gelu=model.text_quick_gelu,
                                              layernorm_epsilon=layernorm_epsilon, rngs=g_wrap(g)))
    model.add_child("token_embedding", nn.Embed(V, Dt, rngs=g_wrap(g)))
    model.add_param("positional_embedding", nn.truncated_normal(g, (T, Dt), 0.02))
    model.add_child("ln_final", nn.LayerNorm(Dt))
    model.add_child("text_projection", nn.Linear(Dt, Dt, use_bias=head_bias, rngs=g_wrap(g)))
