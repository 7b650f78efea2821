/* jimm_b200 -- C ABI of the H100-native ViT / CLIP / SigLIP inference forward path.
 *
 * The reference (pythoncrazy/jimm) has no FFI boundary: its boundary is the Python class surface
 * (src/jimm/models/{vit,clip,siglip}.py, src/jimm/common/{vit,transformer}.py).  This header is the C-ABI
 * underneath the drop-in Python mirror in jimm_b200/ (ctypes binding: jimm_b200/_lib.py; the stub a reference
 * maintainer would add is shown in INTEGRATION.md).  Each entry point cites the reference interface it replaces.
 *
 * Conventions
 *   - one opaque jimm_model_t per GPU; a handle is not thread-safe, distinct handles are;
 *   - every call returns 0 on success or a negative jimm_status; the message is in jimm_last_error() (thread-local);
 *   - "device" pointers are CUDA device pointers on the model's GPU; "host" pointers are CPU memory (pinned memory
 *     makes the copies asynchronous);
 *   - all work is enqueued on the caller's stream (a cudaStream_t passed as void*; NULL = default stream) and the call
 *     returns without synchronising, like JAX's asynchronous dispatch (examples/vit_inference.py:54);
 *   - images are NHWC (tests/test_vit.py:46), token ids int32 [B,T];
 *   - no C++ exceptions cross this boundary.
 */
#ifndef JIMM_B200_H_
#define JIMM_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define JIMM_API __attribute__((visibility("default")))
#else
#define JIMM_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct jimm_model jimm_model_t;

enum jimm_status { JIMM_OK = 0, JIMM_EINVAL = -1, JIMM_ECUDA = -2, JIMM_EDRIVER = -3, JIMM_ESTATE = -4, JIMM_ENOMEM = -5 };
/* JIMM_F8E4M3 is valid only as jimm_config_t.compute_dtype (see there). */
enum jimm_dtype { JIMM_F32 = 0, JIMM_F16 = 1, JIMM_BF16 = 2, JIMM_I32 = 3, JIMM_F8E4M3 = 4 };
enum jimm_kind {
  JIMM_VIT = 0, JIMM_CLIP = 1, JIMM_SIGLIP = 2, JIMM_TOWER = 3 /* bare VisionTransformerBase */,
  JIMM_ENCODER = 4 /* bare Transformer / TransformerEncoder stack (common/transformer.py:22-196) */,
  JIMM_MAPHEAD = 5 /* bare MultiHeadAttentionPoolingHead (common/vit.py:12-101) */,
  JIMM_SIGLIP_NAFLEX = 6 /* SigLIP 2 NaFlex: SigLIP whose vision tower takes each image at its own patch grid, see jimm_encode_image_patches */
};
enum jimm_pool { JIMM_POOL_CLS = 0, JIMM_POOL_MAP = 1 };
enum jimm_act { JIMM_GELU_TANH = 0, JIMM_QUICK_GELU = 1 };
enum jimm_text_pool { JIMM_TPOOL_EOT_ARGMAX = 0, JIMM_TPOOL_LAST = 1 };

/* Mirrors the constructor kwargs of VisionTransformer (models/vit.py:23-40), VisionTransformerBase
 * (common/vit.py:107-126), CLIP (models/clip.py:16-31) and SigLIP (models/siglip.py:16-31). */
typedef struct jimm_config {
  int kind;                               /* jimm_kind */
  /* vision tower */
  int img_size, patch, in_ch, v_width, v_layers, v_heads, v_mlp;
  int pooling;                            /* jimm_pool */
  int pre_norm, patch_bias, v_act;        /* use_pre_norm, use_patch_bias, use_quick_gelu */
  float v_eps_outer;                      /* ln_pre / ln_post / MAP layernorm: 1e-12 ViT | 1e-5 CLIP | 1e-6 SigLIP */
  float v_eps_block;                      /* encoder-block LayerNorm eps: 1e-6 (common/transformer.py:142; never overridden) */
  int num_classes;                        /* ViT classifier width; 0 = no classifier (do_classification=False) */
  /* text tower (CLIP / SigLIP) */
  int ctx_len, vocab, t_width, t_heads, t_layers, t_mlp;
  int t_act, t_causal, t_pool, t_head_bias;
  float t_eps_outer, t_eps_block;
  /* numerics */
  int compute_dtype;                      /* jimm_dtype of the tensor-core operands: F32 (tf32 MMA) | F16 | BF16 | F8E4M3;
                                             accumulation, residual stream, LN statistics, softmax, logits are fp32.
                                             F8E4M3: F16 except that the QKV and FC1 GEMMs of every encoder block take float8 e4m3
                                             operands, scaled by a power of two per token row (from the block LayerNorm) and per
                                             output channel (from the weight row, at finalize); tower widths must be multiples of 16.
                                             Not within the 1e-3 parity of the other modes. */
} jimm_config_t;

JIMM_API const char* jimm_last_error(void);
/* ABI version of this header (bumped on any signature change). */
JIMM_API int jimm_abi_version(void);

/* -- lifecycle: replaces Module.__init__ + from_pretrained's parameter hand-off (models/vit.py:171-257) ----------- */
JIMM_API int jimm_model_create(const jimm_config_t* cfg, int device, jimm_model_t** out);
/* Hand one parameter over in the reference's flax layout, keyed by the reference's flat-state path joined with '.'
 * (e.g. "encoder.transformer.blocks.layers.0.attn.query.kernel", shape (D,H,d); SURVEY.md 8b table).
 * `host` is read during the call.  dtype: JIMM_F32 | JIMM_F16 | JIMM_BF16. */
JIMM_API int jimm_model_set_param(jimm_model_t* m, const char* flax_path, const void* host, const int64_t* shape, int ndim, int dtype);
/* Zero-copy hand-off: `host` is BORROWED and must stay valid and unchanged until jimm_model_finalize returns (e.g. the mmap of a
 * safetensors file).  `shape` is still the reference's flax shape.  flags & JIMM_PARAM_TRANSPOSED: the memory holds the 2-D transpose
 * [N, K] of the flax kernel's (K, N) view -- a HuggingFace (out, in) weight exactly as stored in the checkpoint, i.e. the transform
 * `W.T.reshape(...)` of models/vit.py:241-250 is NOT applied by the caller; that is already the K-major operand layout of the GEMMs,
 * so finalize only casts it.  Casts, transposes and packing run on the GPU; bytes go through a pinned staging ring; finalize
 * synchronises once. */
enum jimm_param_flags { JIMM_PARAM_TRANSPOSED = 1 };
JIMM_API int jimm_model_set_param_ref(jimm_model_t* m, const char* flax_path, const void* host, const int64_t* shape, int ndim, int dtype,
                                      int flags);
/* Pack weights (fused [3D,D] QKV, K-major operands, dtype cast), build TMA descriptors, size the workspace for
 * `max_batch` samples per call.  Fails (JIMM_ESTATE) naming the first missing / unexpected / mis-shaped parameter --
 * the analogue of the reference's strict visit checks (models/vit.py:229-232,259-268). */
JIMM_API int jimm_model_finalize(jimm_model_t* m, int max_batch);
/* Token budget of the vision workspace for the *_hw entry points, called before finalize: the workspace then holds
 * max_batch x max(tokens_per_sample, the native count (img_size / patch)^2 (+1)) tokens (a token is a patch, or the CLS token), and
 * any one image of up to that many tokens fits it.  Without this call the budget is max_batch x the native count, and an image of
 * another size may need more room than its token count says (its padded patch rows).  Vision models only. */
JIMM_API int jimm_model_set_max_tokens(jimm_model_t* m, int tokens_per_sample);
/* Images of H x W that one chunk of a *_hw call runs on this handle: max_batch on the trained patch grid, otherwise as many as the
 * workspace holds, up to max_batch; 0 when one image does not fit (the *_hw call then returns JIMM_EINVAL; a larger
 * jimm_model_set_max_tokens budget would fit it).  JIMM_EINVAL itself, with a message naming the tokens and the limit, for an image
 * of a MAP-pooled tower with more patches than the MAP head's attention pools: it holds one score per token in shared memory, so a
 * device with 227 KB of opt-in shared memory per block (H100) takes at most 56960 tokens, and no budget lifts that. */
JIMM_API int jimm_model_images_per_call(const jimm_model_t* m, int H, int W, int* images);
JIMM_API int jimm_model_destroy(jimm_model_t* m);
/* Introspection used by the Python mirror. */
JIMM_API int jimm_model_output_dim(const jimm_model_t* m, int* vision_out, int* text_out);
JIMM_API int jimm_model_max_batch(const jimm_model_t* m);

/* -- forward: device-resident inputs/outputs ---------------------------------------------------------------------- */
/* The forward calls on device inputs (jimm_vit_forward*, jimm_encode_image*, jimm_encode_text*, jimm_image_tokens*, jimm_text_tokens*,
 * jimm_image_attn*, jimm_text_attn*) check their arguments in one order and report the first fault, before anything is enqueued:
 *   1. the handle: not null, finalized (else JIMM_ESTATE), B >= 0;
 *   2. the image dtype (image calls);
 *   3. the tower: a vision / text tower, a ViT / tower handle for jimm_vit_forward*, a JIMM_SIGLIP_NAFLEX handle for the *_patches calls;
 *   4. the request of a per-token or attention call;
 *   5. when B > 0, null arguments ("<call>: null argument"): the inputs, and out on the pooled calls (pooled stays optional);
 *   6. the shapes: image sizes, NaFlex patch grids, the workspace and the MAP head's sequence limit; sequence lengths;
 *   7. the handle's device is made current.
 * Every refusal is JIMM_EINVAL unless stated. */
/* VisionTransformer.__call__ (models/vit.py:91-103) / VisionTransformerBase.__call__ (common/vit.py:216-248).
 * img: device NHWC [B,img,img,in_ch] of in_dtype; out: device fp32 [B, num_classes | v_width]. */
JIMM_API int jimm_vit_forward(jimm_model_t* m, const void* img, int in_dtype, int B, float* out, void* stream);
/* CLIP.encode_image (models/clip.py:135-146) / SigLIP.encode_image (models/siglip.py:123-133); out fp32 [B,E]. */
JIMM_API int jimm_encode_image(jimm_model_t* m, const void* img, int in_dtype, int B, float* out, void* stream);
/* CLIP.encode_text (models/clip.py:148-167) / SigLIP.encode_text (models/siglip.py:135-153); ids device int32 [B,T]. */
JIMM_API int jimm_encode_text(jimm_model_t* m, const int32_t* ids, int B, int T, float* out, void* stream);
/* L2-normalise + exp(logit_scale) * I . T^T (+ logit_bias) (models/clip.py:183-187, models/siglip.py:169-173).
 * img_e fp32 [Bi,E], txt_e fp32 [Bt,E] (un-normalised encoder outputs), logits fp32 [Bi,Bt] row stride Bt. */
JIMM_API int jimm_contrastive_logits(jimm_model_t* m, const float* img_e, int Bi, const float* txt_e, int Bt, float* logits, void* stream);
/* encode_image + encode_text of one CLIP / SigLIP call with the two (independent) towers running CONCURRENTLY: the text tower is forked onto
 * a side stream and joined back into `stream`, so the idle SMs of one tower's GEMM tail rounds are filled by the other tower.
 * img_e fp32 [Bi,E], txt_e fp32 [Bt,E] (un-normalised, as jimm_encode_image / jimm_encode_text return them). */
JIMM_API int jimm_dual_encode(jimm_model_t* m, const void* img, int in_dtype, int Bi, const int32_t* ids, int Bt, int T, float* img_e, float* txt_e,
                     void* stream);
/* CLIP.__call__ / SigLIP.__call__ (models/clip.py:169-188, models/siglip.py:155-174) on one GPU. */
JIMM_API int jimm_dual_forward(jimm_model_t* m, const void* img, int in_dtype, int Bi, const int32_t* ids, int Bt, int T, float* logits,
                      void* stream);
/* The four calls above for images of any size H x W >= patch (HF's interpolate_pos_encoding=True): img is device NHWC [B,H,W,in_ch].
 * The patch grid is (H / patch) x (W / patch), trailing pixels that do not fill a patch dropped (the VALID conv).  On a grid other
 * than the trained g x g, the patch rows of the position table are resampled bicubically to it (torch.nn.functional.interpolate,
 * mode="bicubic", align_corners=False), the CLS row kept, tokens row-major over the grid.  At H == W == img_size each call is its
 * twin above.  Other sizes run eagerly (no CUDA-graph replay) in chunks of min(max_batch, budget / tokens) images, the budget being
 * the workspace's max_batch x tokens-per-sample (jimm_model_set_max_tokens); an image that alone does not fit, or that is past the MAP
 * head's sequence limit (jimm_model_images_per_call), is JIMM_EINVAL before anything is enqueued. */
JIMM_API int jimm_vit_forward_hw(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, float* out, void* stream);
JIMM_API int jimm_encode_image_hw(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, float* out, void* stream);
JIMM_API int jimm_dual_encode_hw(jimm_model_t* m, const void* img, int in_dtype, int Bi, int H, int W, const int32_t* ids, int Bt, int T,
                                 float* img_e, float* txt_e, void* stream);
JIMM_API int jimm_dual_forward_hw(jimm_model_t* m, const void* img, int in_dtype, int Bi, int H, int W, const int32_t* ids, int Bt, int T,
                                  float* logits, void* stream);
/* B images of different sizes in one call.  imgs: host array of B device pointers, image i NHWC [H[i], W[i], in_ch], contiguous;
 * H, W: host int arrays, read during the call; out: device fp32 [B, out_dim].  Image i's row equals the *_hw call on that image alone.
 * The tokens of consecutive images are packed into one stream (variable-length attention): the images are walked in order, and a new
 * chunk starts when the next image would pass max_batch images, the token budget or the workspace bytes (counted as for the *_hw
 * calls).  An image that alone does not fit, or that is past the MAP head's sequence limit, is JIMM_EINVAL with the *_hw message,
 * before anything is enqueued.  Packed calls run
 * eagerly and return without synchronising; back-to-back calls on one stream are safe. */
JIMM_API int jimm_vit_forward_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W, float* out, void* stream);
JIMM_API int jimm_encode_image_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W, float* out, void* stream);
/* SigLIP 2 NaFlex (kind JIMM_SIGLIP_NAFLEX; config as JIMM_SIGLIP with img_size = g * patch, g * g the position table's rows, MAP pooling,
 * no pre-norm, patch bias).  Every vision call on this kind resamples the g x g position table to the image's patch grid with
 * F.interpolate(mode="bilinear", align_corners=False, antialias=True) instead of bicubically -- at img_size x img_size the table itself,
 * so jimm_encode_image is the plain SigLIP tower -- and the *_hw and *_packed calls above run on it unchanged.
 * jimm_encode_image_patches takes the HuggingFace Siglip2ImageProcessor's output as it is: patches device [B, N, patch*patch*in_ch] of
 * in_dtype (pixel_values; each row a patch flattened in (py, px, c) order), grid host int [B][2] = (gh, gw) (spatial_shapes), read during
 * the call.  Sample b's rows 0 .. gh*gw - 1 are its patches, row-major over its grid; the rows after them (the processor's padding, what
 * pixel_attention_mask marks 0) are never read.  out: device fp32 [B, v_width]; row b equals jimm_encode_image_packed on the gh*patch x
 * gw*patch image with those patches.  Chunks, the token budget and the MAP head's limit are those of jimm_encode_image_packed.  A grid
 * edge < 1, gh*gw > N, a null argument or a model of another kind is JIMM_EINVAL before anything is enqueued. */
JIMM_API int jimm_encode_image_patches(jimm_model_t* m, const void* patches, int in_dtype, int B, int N, const int* grid, float* out, void* stream);
/* B token sequences of different lengths in one jimm_encode_text call.  ids: device int32, the B sequences one after another; len: host
 * int array [B], read during the call, every length in 1 .. ctx_len; out: device fp32 [B, E].  Row i equals jimm_encode_text on sequence
 * i alone (T = len[i]): positions restart at 0 in every sequence, CLIP's causal mask and EOT argmax are taken within it, SigLIP pools its
 * last token.  (For CLIP that is also the row of a padded call whenever sequence i is that row cut just after its first maximum id.)
 * The tokens of consecutive sequences are packed into one stream (variable-length attention); a chunk takes the sequences in order while
 * their tokens fit max_batch x ctx_len rows, up to 65535 sequences.  A bad length, a null argument or a model without a text tower is
 * JIMM_EINVAL before anything is enqueued.  Runs eagerly and returns without synchronising; back-to-back calls on one stream are safe. */
JIMM_API int jimm_encode_text_packed(jimm_model_t* m, const int32_t* ids, int B, const int* len, float* out, void* stream);

/* -- per-token hidden states (HF output_hidden_states) of the vision and text towers ---------------------------------------------
 * With x_k the fp32 residual stream after k of a tower's L blocks: layer k in 0 .. L returns x_k (x_0: the embeddings -- vision: patch
 * embedding + position table, resampled on another grid, CLS row first on CLS towers, after ln_pre when the tower has it; text: token
 * embedding + positions); JIMM_LAYER_FINAL returns the final-normed tokens, ln_post(x_L) (vision) / ln_final(x_L) (text).  Rows: per
 * image its S = gh*gw (+1 CLS) tokens in the order the tower holds them (CLS, then patches row-major); per sequence its T tokens, those
 * after an EOT or padding as computed.  Each request j writes out[j]: a device buffer [rows, D] row-major, contiguous, 16-byte aligned,
 * of out_dtype (JIMM_F32: the residual stream's bits; JIMM_F16 / JIMM_BF16: those rounded to nearest even); rows = B * S (dense), the
 * sum of the samples' token counts (packed, in sample order).  pooled (device fp32 [B, out_dim], or NULL for none) receives exactly
 * what the matching pooled call writes: jimm_vit_forward* on a ViT / tower handle, jimm_encode_image* / jimm_encode_text* on a dual one.
 * Without JIMM_LAYER_FINAL and pooled, only max(k) blocks run.  These calls never replay a CUDA graph and leave the graph cache as it
 * is; they allocate nothing.  A bad request (n outside 1 .. L + 2, a layer outside 0 .. L and not JIMM_LAYER_FINAL, a bad out_dtype,
 * a null or misaligned pointer) and every refusal of the matching pooled call is JIMM_EINVAL before anything is enqueued. */
#define JIMM_LAYER_FINAL (-1)
typedef struct jimm_tokens_req {
  int n;                                   /* requests, 1 .. L + 2 */
  const int* layers;                       /* host [n]: each 0 .. L, or JIMM_LAYER_FINAL */
  void* const* out;                        /* host [n] of device buffers: [rows, D] row-major, contiguous */
  int out_dtype;                           /* JIMM_F32 / JIMM_F16 / JIMM_BF16 */
} jimm_tokens_req_t;
/* The vision tower on images as jimm_vit_forward_hw / jimm_encode_image_hw take them (H == W == img_size: the trained size). */
JIMM_API int jimm_image_tokens(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, const jimm_tokens_req_t* req, float* pooled,
                               void* stream);
/* ... on images of different sizes as jimm_vit_forward_packed / jimm_encode_image_packed take them */
JIMM_API int jimm_image_tokens_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W,
                                      const jimm_tokens_req_t* req, float* pooled, void* stream);
/* ... on HF NaFlex patch rows as jimm_encode_image_patches takes them (kind JIMM_SIGLIP_NAFLEX); sample b has gh*gw rows */
JIMM_API int jimm_image_tokens_patches(jimm_model_t* m, const void* patches, int in_dtype, int B, int N, const int* grid,
                                       const jimm_tokens_req_t* req, float* pooled, void* stream);
/* The text tower on ids as jimm_encode_text / jimm_encode_text_packed take them */
JIMM_API int jimm_text_tokens(jimm_model_t* m, const int32_t* ids, int B, int T, const jimm_tokens_req_t* req, float* pooled, void* stream);
JIMM_API int jimm_text_tokens_packed(jimm_model_t* m, const int32_t* ids, int B, const int* len, const jimm_tokens_req_t* req, float* pooled,
                                     void* stream);

/* -- attention weights (HF output_attentions) of the vision and text towers, and the MAP head's probe weights ------------------------
 * Block k (0 .. L-1) gives softmax(q k^T / sqrt(d)) of each of its H heads, computed in fp32 on the q / k its attention reads (the qkv
 * buffer in the attention I/O type: fp16, or bf16 in bf16 mode).  Each request j writes out[j], a device buffer, contiguous, 16-byte
 * aligned, of out_dtype (JIMM_F32; JIMM_F16 / JIMM_BF16: the fp32 weights rounded to nearest even): per sample b its [H, S_b, S_b]
 * weights, row-major (query rows, key columns), sample b from element H * sum_{j<b} S_j^2 on -- [B, H, S, S] for a dense call.  The
 * CLIP text tower is causal: the entries above the diagonal are 0.  JIMM_ATTN_MAP (MAP-pooled vision towers) gives the MAP head's
 * probe weights, the ones its pooled output sums with: per sample [H, 1, S_b], sample b from element H * sum_{j<b} S_j on.  Rows and
 * samples are those of jimm_image_tokens* / jimm_text_tokens*; sample b of a packed call equals the call on that sample alone.
 * pooled (device fp32 [B, out_dim], or NULL) receives exactly what the matching pooled call writes.  Without JIMM_ATTN_MAP and pooled,
 * only the blocks up to the deepest request run.  These calls never replay a CUDA graph, leave the graph cache as it is and allocate
 * nothing.  A bad request (n outside 1 .. L + 1, a block outside 0 .. L-1 and not JIMM_ATTN_MAP, JIMM_ATTN_MAP on a CLS-pooled or a
 * text tower, a bad out_dtype, a null or misaligned pointer) and every refusal of the matching pooled call is JIMM_EINVAL before
 * anything is enqueued, in the order stated above the forward calls (the request is step 4). */
#define JIMM_ATTN_MAP (-2)
typedef struct jimm_attn_req {
  int n;                                   /* requests, 1 .. L + 1 */
  const int* blocks;                       /* host [n]: each 0 .. L-1, or JIMM_ATTN_MAP */
  void* const* out;                        /* host [n] of device buffers, 16-byte aligned */
  int out_dtype;                           /* JIMM_F32 / JIMM_F16 / JIMM_BF16 */
} jimm_attn_req_t;
/* The vision tower on images as jimm_image_tokens takes them */
JIMM_API int jimm_image_attn(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, const jimm_attn_req_t* req, float* pooled,
                             void* stream);
/* ... as jimm_image_tokens_packed takes them */
JIMM_API int jimm_image_attn_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W,
                                    const jimm_attn_req_t* req, float* pooled, void* stream);
/* ... as jimm_image_tokens_patches takes them (kind JIMM_SIGLIP_NAFLEX) */
JIMM_API int jimm_image_attn_patches(jimm_model_t* m, const void* patches, int in_dtype, int B, int N, const int* grid, const jimm_attn_req_t* req,
                                     float* pooled, void* stream);
/* The text tower on ids as jimm_text_tokens / jimm_text_tokens_packed take them */
JIMM_API int jimm_text_attn(jimm_model_t* m, const int32_t* ids, int B, int T, const jimm_attn_req_t* req, float* pooled, void* stream);
JIMM_API int jimm_text_attn_packed(jimm_model_t* m, const int32_t* ids, int B, const int* len, const jimm_attn_req_t* req, float* pooled,
                                   void* stream);

/* -- forward of a bare sub-module (kinds JIMM_ENCODER / JIMM_MAPHEAD; config fields used: v_width, v_heads, v_mlp, v_layers, v_act,
 *    v_eps_block, v_eps_outer, t_causal (attn_mask = tril), ctx_len = max tokens per sample, compute_dtype; parameters keyed
 *    "blocks.layers.{i}.<...>" resp. "probe", "attn.<...>", "layernorm.<...>", "mlp.layers.{0,2}.<...>") ---------------------------- */
/* Transformer.__call__ / TransformerEncoder.__call__ (common/transformer.py:116-132,190-196): x, out device fp32 [B,S,D]. */
JIMM_API int jimm_encoder_forward(jimm_model_t* m, const float* x, int B, int S, float* out, void* stream);
/* MultiHeadAttentionPoolingHead.__call__ (common/vit.py:87-101): x device fp32 [B,S,D] -> out device fp32 [B,D].  A ctx_len past the
 * MAP head's sequence limit (jimm_model_images_per_call) is JIMM_EINVAL at jimm_model_finalize; so is a MAP-pooled tower whose
 * trained image size is. */
JIMM_API int jimm_map_head_forward(jimm_model_t* m, const float* x, int B, int S, float* out, void* stream);

/* -- forward: HOST buffers (the reference-facing call: host->device copy, forward, device->host copy, all enqueued on
 *    `stream`; the caller synchronises the stream before reading `out`).  examples/vit_inference.py:52-58. ----------- */
JIMM_API int jimm_vit_forward_host(jimm_model_t* m, const void* img_host, int in_dtype, int B, float* out_host, void* stream);
JIMM_API int jimm_dual_forward_host(jimm_model_t* m, const void* img_host, int in_dtype, int Bi, const int32_t* ids_host, int Bt, int T,
                           float* logits_host, void* stream);
/* The whole examples/vit_inference.py:27-58 pipeline from raw frames: host uint8 RGB [B,H,W,3] -> (bytes over PCIe, a quarter of the
 * fp32 pixel values) -> image front-end `pre` on the GPU (see jimm_preproc_* below; its output size must equal the model's input) ->
 * tower -> host fp32 [B, num_classes | v_width].  Same slicing / stream semantics as jimm_vit_forward_host. */
typedef struct jimm_preproc jimm_preproc_t;
JIMM_API int jimm_vit_forward_host_u8(jimm_model_t* m, jimm_preproc_t* pre, const uint8_t* img_host, int B, int H, int W, float* out_host,
                                      void* stream);

/* -- multi-GPU contrastive head: one process per GPU, embeddings exchanged over NVLink peer memory ------------------- */
/* Allocate this rank's symmetric gather buffer ([world*max_rows, 2E] fp32 + flags) and export its IPC handle
 * (64 bytes).  The handles of all ranks are exchanged by the caller (torch.distributed / any out-of-band channel). */
JIMM_API int jimm_comm_init(jimm_model_t* m, int rank, int world, int max_rows_per_rank, unsigned char* handle_out /*[64]*/);
JIMM_API int jimm_comm_connect(jimm_model_t* m, const unsigned char* handles /*[world*64]*/);
/* Fused: L2-normalise the local [B_local,E] image/text embeddings, store them straight into every peer's gather buffer
 * over NVLink (st.global on mapped peer pointers), device-side flag barrier, then the local rank's logits row block
 * logits_local fp32 [B_local, world*B_local] = exp(scale) * I_local . T_all^T (+ bias).  No host synchronisation. */
JIMM_API int jimm_comm_contrastive_logits(jimm_model_t* m, const float* img_e, const float* txt_e, int B_local, float* logits_local,
                                 void* stream);
/* The device-side wait for the peers is bounded (JIMM_COMM_TIMEOUT_MS, default 10 s) and every rank must pass the same B_local: a
 * missing or mismatched peer yields NaN logits and a sticky error, returned here (after the stream has been synchronised) and by the
 * next jimm_comm_contrastive_logits call. */
JIMM_API int jimm_comm_status(jimm_model_t* m);
/* Device pointer to this rank's gathered, normalised [world*B_local, 2E] buffer (valid after the call above). */
JIMM_API int jimm_comm_gathered(jimm_model_t* m, float** gathered, int* row_stride);

/* -- per-kernel entry points (device pointers; used by tests/ so every kernel is individually
 *    parity- and profile-testable; SURVEY.md 8b) -------------------------------------------------------------------
 * Type codes of these entry points: 0 fp32 | 1 fp16 | 2 bf16 | 3 fp32 rounded to tf32 (round to nearest, ties away from zero;
 * the operand format of the fp32 compute mode).  Here 3 is NOT JIMM_I32. */
/* C[M,N] = epi(A[M,K] . B[N,K]^T): impl 0 = wgmma/TMA kernel, 1 = SIMT cross-check.
 * act: 0 none | 1 gelu_tanh | 2 quick_gelu; epi_mode 0 / 1 LSU stores | 2 TMA stores; rows_in>0 remaps output rows. */
JIMM_API int jimm_k_gemm(int impl, int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* bias, int act,
                const float* rowadd, const float* residual, int ldr, void* out, int out_type, int ldo, int rows_in, int rows_out,
                int row_off, int epi_mode, void* stream);
/* x[M,N] += A . B^T + bias through the fp32 reduce-add epilogue, then -- fused -- ln_out = LayerNorm(x) row by row
 * as the last column tile of each 32-row group completes (the out-proj / FC2 + following norm of common/transformer.py:130-131).
 * counters: device int32 [M/32 + 1], zero on entry (left zero on exit).  ln_out_type JIMM_F32 stores tf32-rounded fp32. */
JIMM_API int jimm_k_gemm_residual_ln(int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* bias, float* x, int ldx,
                            const float* ln_scale, const float* ln_bias, float eps, void* ln_out, int ln_out_type, int ln_ldo, int* counters,
                            void* stream);
/* Both of the above, as the forward pass runs the GEMM (the two are this call with the extra arguments at their defaults):
 *   plan_M (0 = M): the rows the plan (its tensor maps) is built for; M <= plan_M rows are run.  With M < plan_M the TMA epilogues
 *     (epi_mode 2) may write rows [M, roundup(M, 16)) of the output; rows >= roundup(M, 16) are never written.
 *   reverse: walk the tiles from the last one (same result).
 *   tok_pad > 0: token scatter of the patch embedding: A row b * tok_pad + p is reduce-added into out[b, p + tok_off, :] of an fp32
 *     [M / tok_pad, tok_S, N] tensor (residual == out, epi_mode 2, tok_pad a multiple of 16 dividing M and plan_M); rows
 *     p + tok_off >= tok_S are dropped.
 *   ln_counters != NULL: fused LayerNorm of jimm_k_gemm_residual_ln (ln_* arguments as there; needs the fp32 reduce-add). */
JIMM_API int jimm_k_gemm_ex(int impl, int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* bias, int act,
                            const float* rowadd, const float* residual, int ldr, void* out, int out_type, int ldo, int rows_in, int rows_out,
                            int row_off, int epi_mode, int plan_M, int reverse, int tok_pad, int tok_off, int tok_S, const float* ln_scale,
                            const float* ln_bias, float ln_eps, void* ln_out, int ln_out_type, int ln_ldo, int* ln_counters, void* stream);
JIMM_API int jimm_k_layernorm(const float* x, int ldx, int group, int row_off, const int32_t* row_index, const float* scale, const float* bias,
                     float eps, void* out, int out_type, int ldy, int rows, int D, void* stream);
JIMM_API int jimm_k_attention(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int causal, void* stream);
/* jimm_k_layernorm / jimm_k_attention as the encoder runs them (each of the two is its _ex call with reverse = 0):
 *   reverse: walk the rows (LayerNorm) or the samples (attention) from the last one; the result is the same, bit for bit. */
JIMM_API int jimm_k_layernorm_ex(const float* x, int ldx, int group, int row_off, const int32_t* row_index, const float* scale, const float* bias,
                                 float eps, void* out, int out_type, int ldy, int rows, int D, int reverse, void* stream);
JIMM_API int jimm_k_attention_ex(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int causal, int reverse,
                                 void* stream);
/* FP8 (e4m3) pieces of the F8E4M3 compute mode.  An e4m3 matrix is one byte per element (row strides in elements = bytes); a scale
 * vector holds one fp32 power of two per row, s = 2^k with k the smallest integer such that max|row| / s <= 448 (s = 1 for a zero row,
 * k >= -126); elements are stored as e4m3(x / s), rounded to nearest even.
 * jimm_k_layernorm_e4m3: the dense per-row LayerNorm of jimm_k_layernorm_ex (group 1, row_off 0) with an e4m3 output [rows, ldy] and
 *   row_scale fp32 [rows]; the row's scale comes from its fp32 normalised values.
 * jimm_k_gemm_e4m3: out = act(A . B^T * (a_scale[row] * b_scale[col]) + bias), A e4m3 [M, K], B e4m3 [N, K], a_scale [plan_M],
 *   b_scale [N] (8-byte aligned); out_type 0 fp32 | 1 fp16 | 2 bf16 | 3 tf32; impl, epi_mode, plan_M, reverse as jimm_k_gemm_ex.
 * jimm_k_quantize_e4m3: the weight quantiser of finalize: rows of an fp32 [rows, K] matrix (row stride lds) -> e4m3 [rows, ldo]
 *   and row_scale [rows]; K, lds and ldo multiples of 4. */
JIMM_API int jimm_k_layernorm_e4m3(const float* x, int ldx, const float* scale, const float* bias, float eps, void* out, int ldy,
                                   float* row_scale, int rows, int D, int reverse, void* stream);
JIMM_API int jimm_k_gemm_e4m3(int impl, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* a_scale,
                              const float* b_scale, const float* bias, int act, void* out, int out_type, int ldo, int epi_mode, int plan_M,
                              int reverse, void* stream);
JIMM_API int jimm_k_quantize_e4m3(const float* src, int lds, int rows, int K, void* out, int ldo, float* row_scale, void* stream);
JIMM_API int jimm_k_map_attention(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, void* stream);
/* jimm_k_attention_ex / jimm_k_map_attention for heads of head_dim columns (D = H * head_dim; the two are these calls with
 * head_dim = 64).  head_dim: a multiple of 8 from 8 to 128.  Softmax scale 1 / sqrt(head_dim). */
JIMM_API int jimm_k_attention_hd(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, int causal,
                                 int reverse, void* stream);
JIMM_API int jimm_k_map_attention_hd(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim,
                                     void* stream);
/* Packed forms of the two above (non-causal): seq_off device int32 [B + 1], sample b = rows seq_off[b] .. seq_off[b+1]-1 of the packed
 * [rows, 3D] qkv / [rows, 2D] kv (and of out [rows, D] for attention; out [B, D] for MAP), every length >= 1 and <= max_S.  Each
 * sample's result is the bits of the _hd call on that sample alone; rows outside every sample are not written. */
JIMM_API int jimm_k_attention_packed(const void* qkv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int max_S, int H,
                                     int head_dim, int reverse, void* stream);
JIMM_API int jimm_k_map_attention_packed(const float* q, const void* kv, int io_type, void* out, int out_type, const int32_t* seq_off, int B,
                                         int max_S, int H, int head_dim, void* stream);
/* jimm_k_attention_packed with a causal mask when causal != 0 (key <= query, counted from each sample's first row); jimm_k_attention_packed
 * is this call with causal = 0.  Each sample's rows are the bits of jimm_k_attention_hd(..., causal, ...) on that sample alone. */
JIMM_API int jimm_k_attention_packed_ex(const void* qkv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int max_S, int H,
                                        int head_dim, int causal, int reverse, void* stream);
/* The attention weights of jimm_k_attention_hd / jimm_k_attention_packed_ex (HF output_attentions): softmax((q/sqrt(d)) k^T masked) in
 * fp32, written as out_type JIMM_F32 / JIMM_F16 / JIMM_BF16 (the fp32 value rounded to nearest even).  out: sample b's [H, S_b, S_b] block,
 * row-major, from element H * sum_{j<b} S_j^2 on (dense, seq_off NULL: S_b = S); causal: the entries above the diagonal are 0. */
JIMM_API int jimm_k_attn_probs(const void* qkv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int S, int H, int head_dim,
                               int causal, void* stream);
/* jimm_k_map_attention_hd (seq_off NULL) / jimm_k_map_attention_packed that also writes the weights its output sums with, probs
 * [B, H, 1, S] of probs_type (packed: sample b's [H, 1, S_b] from element H * seq_off[b] on); probs NULL is the plain call. */
JIMM_API int jimm_k_map_attention_probs(const float* q, const void* kv, int io_type, void* out, int out_type, const int32_t* seq_off, int B,
                                        int S, int H, int head_dim, void* probs, int probs_type, void* stream);
JIMM_API int jimm_k_patchify(const void* img, int in_type, int B, int H, int W, int C, int P, void* out, int out_type, void* stream);
/* jimm_k_patchify into the patch GEMM's padded layout: rows_per_sample (0 = patches per image; more = pad rows per sample, left
 * untouched) and ldk (row stride in elements, 0 = P*P*C; more = pad columns, written as zeros). */
JIMM_API int jimm_k_patchify_ex(const void* img, int in_type, int B, int H, int W, int C, int P, void* out, int out_type, int rows_per_sample,
                                int ldk, void* stream);
/* y = act(x) elementwise on device fp32 (act: 1 tanh-GELU == nnx.gelu, 2 QuickGELU == common/transformer.py:12-19). */
JIMM_API int jimm_k_activation(const float* x, float* y, long long n, int act, void* stream);
/* Initial residual stream of a tower on a gh x gw patch grid, for a position table trained on a g x g grid: x fp32 [B, (1 +) gh*gw, D];
 * row 0 = cls + pos[0] when cls (fp32 [D]) is not NULL, the patch rows the bicubic resampling of pos's g x g patch rows described at
 * jimm_vit_forward_hw (pos fp32 [(1 +) g*g, D]); D a multiple of 4.  (gh, gw) == (g, g) gives the table itself, bit for bit. */
JIMM_API int jimm_k_tokens_init_interp(const float* cls, const float* pos, int g, int D, float* x, int B, int gh, int gw, void* stream);
/* jimm_k_tokens_init_interp with the resampling chosen by mode: 0 bicubic (jimm_k_tokens_init_interp itself), 1 antialiased bilinear
 * (F.interpolate(mode="bilinear", align_corners=False, antialias=True), the NaFlex rule; up to g table rows per axis). */
JIMM_API int jimm_k_tokens_init_interp_ex(const float* cls, const float* pos, int g, int D, float* x, int B, int gh, int gw, int mode,
                                          void* stream);
/* The position add of a packed vision call: image b is rows seq_off[b] .. seq_off[b+1]-1 of x fp32 [rows, D] (seq_off device int32 [B + 1]),
 * its grid (n_b / gw[b]) x gw[b] (gw device int32 [B]; n_b its rows less the CLS row when cls is not NULL).  The CLS row is set to cls +
 * pos[0]; each patch row gets += the table resampled as jimm_k_tokens_init_interp_ex (mode) gives it.  max_S: the most rows of one image. */
JIMM_API int jimm_k_tokens_add_interp_packed(const float* cls, const float* pos, int g, int D, float* x, const int32_t* seq_off, const int32_t* gw,
                                             int B, int max_S, int mode, void* stream);
/* The patch-GEMM operand of jimm_encode_image_patches: patches [B, N, K] of in_type (0 fp32 | 1 fp16 | 2 bf16), sample b's rows 0 .. n_b - 1
 * (n_b = seq_off[b+1] - seq_off[b] <= max_rows <= N) -> rows seq_off[b] + r of out [*, ldk] of out_type (0 fp32 | 1 fp16 | 2 bf16 | 3 tf32),
 * columns K .. ldk - 1 written as zeros; other rows of out untouched, other rows of patches never read. */
JIMM_API int jimm_k_patch_rows_packed(const void* patches, int in_type, int N, int K, const int32_t* seq_off, int B, int max_rows, void* out,
                                      int out_type, int ldk, void* stream);
JIMM_API int jimm_k_embed(const int32_t* ids, const float* table, const float* pos, float* x, int B, int T, int D, int vocab, void* stream);
/* jimm_k_embed on B sequences packed as for jimm_k_attention_packed (seq_off device int32 [B + 1], T_total = seq_off[B] rows of ids and
 * x): x[r] = table[clamp(ids[r], 0, vocab - 1)] + pos[r - seq_off[b]] for the rows r of sequence b, whose positions restart at 0. */
JIMM_API int jimm_k_embed_packed(const int32_t* ids, const float* table, const float* pos, float* x, const int32_t* seq_off, int B, int T_total,
                                 int D, int vocab, void* stream);
/* The copy of the per-token calls: out[r, :] = x[r, :] for r < rows, x fp32 [rows, D] and out [rows, D] of out_type (0 fp32: the same
 * bits | 1 fp16 | 2 bf16: round to nearest even), both contiguous and 16-byte aligned, D a multiple of 8; nothing after rows * D
 * elements of out is written. */
JIMM_API int jimm_k_tokens_out(const float* x, long long rows, int D, void* out, int out_type, void* stream);
JIMM_API int jimm_k_l2_normalize(const float* x, float* out, int ldo, int B, int E, void* stream);
JIMM_API int jimm_k_logits(const float* img, const float* txt, const float* logit_scale, const float* logit_bias, float* logits, int Bi, int Bt,
                  int E, int ldl, void* stream);
/* Checkpoint ingestion as jimm_model_finalize runs it: host memory of src_type (0 fp32 | 1 fp16 | 2 bf16) is streamed through a
 * pinned staging ring in chunks of at most 32 MiB, cast on the device to out_type (0 fp32 | 1 fp16 | 2 bf16 round to nearest even |
 * 3 tf32 round to nearest, ties away) and written to device memory dst.  The ring belongs to the call, which returns once its last
 * chunk has been written.
 * jimm_k_upload_rows: rows of K elements, row-major -> dst[r * ldd + k] (ldd >= K); a single row longer than a chunk (rows = 1,
 *   ldd = K) is split along K.
 * jimm_k_upload_kernel: a kernel's (K, N) view -> rows n0 .. n0 + N - 1 of the K-major operand dst [*, ldd] (ldd >= K):
 *   dst[(n0 + n) * ldd + k] = value (k, n).  host holds the (K, N) matrix row-major (flax layout, transposed = 0) or its [N, K]
 *   transpose (a HuggingFace (out, in) weight, transposed = 1).  Columns K .. ldd - 1 and other rows are not written. */
JIMM_API int jimm_k_upload_rows(const void* host, int src_type, long long rows, long long K, void* dst, int out_type, long long ldd, void* stream);
JIMM_API int jimm_k_upload_kernel(const void* host, int src_type, int K, int N, int transposed, void* dst, int out_type, long long ldd, int n0,
                                  void* stream);
/* ---- image front-end (SURVEY.md 8f.1): the HuggingFace image processor the reference's examples run on the host ----
 * Replaces `processor(images=..., return_tensors="np")["pixel_values"]` + the NCHW->NHWC transpose of
 * examples/vit_inference.py:27-37, examples/clip_inference.py:35-38 (transformers 4.53.0 slow processors on Pillow 11.3.0,
 * uv.lock:2679,1573): Pillow 8-bit resize with antialiasing (bilinear | bicubic) -> optional centre crop -> rescale ->
 * normalise, written NHWC in the dtype the tower consumes.  Bit-exact with that pipeline (integer resampling, IEEE fp32
 * rescale/normalise).  Mirrors `preprocessor_config.json`: size {height,width} | {shortest_edge}, crop_size, resample,
 * rescale_factor, image_mean, image_std. */
typedef struct jimm_preproc_config {
  int height, width;        /* exact output size (ViT, SigLIP: size = {height, width}) ... */
  int shortest_edge;        /* ... or, when non-zero, resize the shortest edge to this keeping the aspect ratio (CLIP) */
  int crop_h, crop_w;       /* centre crop after the resize (CLIP crop_size); 0 = none */
  int resample;             /* PIL code: 2 bilinear, 3 bicubic */
  double rescale_factor;    /* 1/255 */
  float mean[3], std[3];    /* image_mean, image_std */
} jimm_preproc_config_t;
JIMM_API int jimm_preproc_create(const jimm_preproc_config_t* cfg, int device, jimm_preproc_t** out);
/* Output size of H x W frames.  Refuses (JIMM_EINVAL) exactly the sizes jimm_preproc_run refuses: frames of H x W x 3 >= 2^31 bytes,
 * a resized image (before the crop) of more than 2^24 pixels per edge, a crop larger than the resized image. */
JIMM_API int jimm_preproc_output_size(const jimm_preproc_t* p, int H, int W, int* out_h, int* out_w);
/* img: device uint8 [B,H,W,3] (same-sized RGB images); out: device [B,out_h,out_w,3] of out_dtype (JIMM_F32 | JIMM_F16 | JIMM_BF16),
 * aligned to four samples (16 bytes for JIMM_F32, 8 for the 16-bit types; JIMM_EINVAL otherwise).
 * Sizes whose one-kernel plan does not fit in shared memory (4K, 12 MP, 8K frames into the bicubic front-ends) run in two passes
 * through an 8-bit intermediate allocated in stream order per call, at most 64 MB per chunk of images; same bytes. */
JIMM_API int jimm_preproc_run(jimm_preproc_t* p, const uint8_t* img, int B, int H, int W, void* out, int out_dtype, void* stream);
JIMM_API int jimm_preproc_destroy(jimm_preproc_t* p);
/* ---- SigLIP 2 NaFlex front-end: transformers' Siglip2ImageProcessor (PIL backend) on the GPU ----
 * Every frame gets its own output size from the patch budget, is resized with Pillow's 8-bit arithmetic, rescaled, normalised and
 * written as patch rows, bit-exact with the processor's pixel_values / pixel_attention_mask / spatial_shapes.
 * jimm_preproc_naflex_grid (host only, no handle, no GPU): the processor's size rule (get_image_size_for_max_num_patches) in double
 *   precision -- the patch grid gh x gw of an H x W frame (output size gh*patch x gw*patch).  JIMM_EINVAL for patch < 1,
 *   max_num_patches < 1, an edge < 1, H x W x 3 >= 2^31 bytes, or a grid of more than max_num_patches patches (extreme strips,
 *   for which the processor itself emits more rows than max_num_patches).
 * jimm_preproc_create_naflex: cfg's resample (2 bilinear | 3 bicubic), rescale_factor, mean and std; height, width, shortest_edge,
 *   crop_h and crop_w must be 0.  jimm_preproc_run and jimm_preproc_output_size refuse such a handle; jimm_preproc_run_naflex
 *   refuses a fixed-size one.
 * jimm_preproc_run_naflex: imgs a host array of B device pointers, image i contiguous uint8 RGB [H[i], W[i], 3] at any alignment;
 *   pixel_values device [B, max_num_patches, patch*patch*3] of out_dtype (JIMM_F32 | JIMM_F16 | JIMM_BF16, aligned as for
 *   jimm_preproc_run), each row a patch in (py, px, c) order, sample b's rows gh*gw .. max_num_patches - 1 zero; mask (nullable)
 *   device int32 [B, max_num_patches], 1 on the patch rows; grid (nullable) host int [B][2] = (gh, gw), written before the call
 *   returns.  fp16 / bf16 are the fp32 values rounded to nearest even.  Every refusal (JIMM_EINVAL) happens before anything is
 *   enqueued; B = 0 is a no-op.  The call never waits for the stream: Pillow's tables are built on the device into scratch
 *   allocated in stream order, plus an 8-bit intermediate of at most 64 MB per chunk for frames whose fused plan does not fit in
 *   shared memory. */
JIMM_API int jimm_preproc_naflex_grid(int patch, int max_num_patches, int H, int W, int* gh, int* gw);
JIMM_API int jimm_preproc_create_naflex(const jimm_preproc_config_t* cfg, int patch, int device, jimm_preproc_t** out);
JIMM_API int jimm_preproc_run_naflex(jimm_preproc_t* p, const uint8_t* const* imgs, int B, const int* H, const int* W, int max_num_patches,
                                     void* pixel_values, int out_dtype, int32_t* mask, int* grid, void* stream);
/* Host-only test entry: Pillow's resampling windows and 22-bit fixed-point weights for one axis. */
JIMM_API int jimm_k_resample_coeffs(int in_size, int out_size, int resample, int* ksize, int* first, int* count, int* kk, int kk_capacity);
/* Test entry: the same tables as built on the device by the NaFlex front-end (first, count [out_size], kk [out_size][ksize] on the host;
 * synchronises). */
JIMM_API int jimm_k_resample_coeffs_device(int in_size, int out_size, int resample, int* first, int* count, int* kk, int kk_capacity);
/* Host-only test entry: the plan jimm_preproc_run uses for H x W frames.  path 0: one fused kernel with TY output rows per CTA, smem
 * bytes of shared memory, chosen under shared-memory budget tier 0 / 1 / 2 (72 / 110 / 200 KB); path 1: two passes (tier -1, smem 0). */
JIMM_API int jimm_k_preproc_plan(const jimm_preproc_config_t* cfg, int H, int W, int* path, int* tier, int* TY, long long* smem);
/* ---- zero-shot / classification epilogue (SURVEY.md 8f.3): what the examples compute in JAX after the forward ----
 * logits: device fp32 [rows, cols] (leading dimension ld).  mode 0: probs = exp(x) / sum(exp(x)) per row, un-shifted like
 * examples/clip_inference.py:47; mode 1: probs = sigmoid(x) (SigLIP pair probabilities).  order (nullable, int32 [rows, cols]):
 * `argsort(x)[::-1]` per row -- descending, equal scores with the larger index first (examples/clip_inference.py:49);
 * argmax (nullable, int32 [rows]): first maximum per row (examples/vit_inference.py:58).  Any cols: the order of a row wider than
 * 4096 columns is sorted in scratch allocated in stream order on `stream` (cudaMallocAsync / cudaFreeAsync), 16 bytes per column
 * per row (8 when cols <= 8192), for at most 256 MB of rows at a time (or one row, if a row needs more). */
JIMM_API int jimm_postprocess(const float* logits, int rows, int cols, int ld, int mode, float* probs, int ldp, int32_t* order, int32_t* argmax,
                              void* stream);
/* Top-k of each logits row (1 <= k <= cols): indices (int32 [rows, k]) are the first k columns of jimm_postprocess's order -- equal
 * scores larger index first, every NaN above +inf, -0 tied with +0 -- values (fp32 [rows, k]) the logits at those columns, bit for
 * bit, and probs (nullable, fp32 [rows, k]) mode 0's probabilities there, bit for bit.  k <= 1024: a row of up to 32768 columns is
 * selected in one CTA from one read (radix select, then a sort of the k survivors); a wider row keeps k candidates per 8192-column
 * segment in scratch (8 k bytes per segment per row, at most 256 MB of rows at a time) and merges them.  k > 1024: the prefix of the
 * full order, sorted in scratch (4 bytes per column per row, at most 256 MB of rows at a time, plus the sort's own).  Scratch is
 * allocated in stream order on `stream`. */
JIMM_API int jimm_topk(const float* logits, int rows, int cols, int ld, int k, float* values, int32_t* indices, float* probs, void* stream);
/* Gallery search of a CLIP / SigLIP model: for each of the Q queries (device fp32 [Q, E], un-normalised embeddings as
 * jimm_encode_image / jimm_encode_text return them) its k best gallery rows (device fp32 [N, E], the other tower's embeddings) by
 * the model's own score, as jimm_topk would pick them from the [Q, N] jimm_contrastive_logits matrix -- values fp32 [Q, k], indices
 * int32 [Q, k] -- bit for bit, without that matrix: scores go through bounded score blocks in stream-ordered scratch (under 0.5 GB
 * at E <= 1024 for any N).  E is the model's embedding width; 1 <= k <= min(N, 1024). */
JIMM_API int jimm_search(jimm_model_t* m, const float* queries, int Q, const float* gallery, int N, int k, float* values, int32_t* indices,
                         void* stream);
/* Gallery index of a CLIP / SigLIP model: a gallery normalised once and kept on the device, searched many times.
 * jimm_index_create: an empty index for m's embedding width E (a multiple of 8 up to 8192, which every model width is) on m's device.
 *   jimm_index_add and jimm_index_search read the model the index is bound to (its logit_scale / logit_bias at every search), so that
 *   model must outlive every such call.
 * jimm_index_rebind: binds the index to another model of the same width on the same device (JIMM_EINVAL otherwise), e.g. the handle
 *   rebuilt from the same parameters; the stored rows stay.  After the bound model is destroyed, only jimm_index_rebind and
 *   jimm_index_destroy may be called.
 * jimm_index_add: appends n rows (device fp32 [n, E], un-normalised embeddings as jimm_search's gallery); row numbering continues.
 *   The index stores each row normalised by the contrastive head's l2_normalize (fp32), an fp16 copy and an upper bound on the
 *   normalised row's norm: 6 E + 4 bytes per row, in storage that grows geometrically.  At most 2^31 - 1 rows in all.
 * jimm_index_search: jimm_search(m, queries, Q, all rows added so far, N, k, ...) bit for bit, 1 <= k <= min(N, 1024).  Each query's
 *   exact best k over the first 32768 rows seeds a threshold; the other rows are screened in fp16 on the tensor cores against it with a
 *   proven error bound, and only the rows that can still reach the best k are scored exactly (see INTEGRATION.md, "Gallery index").
 *   stats (nullable, host) receives the work done.  The call waits for `stream` once per screened chunk of 65536 rows.
 * Adds and searches on different streams must be ordered by the caller.  jimm_index_destroy waits for the index's device; it never
 * reads the model. */
typedef struct jimm_index jimm_index_t;
typedef struct jimm_search_stats {
  long long rows_rescored;    /* (query, row) pairs the screen passed and the rescorer scored exactly */
  long long fallbacks;        /* (query, screen chunk) pairs that passed too many rows and went through the exact block step */
  long long chunks_screened;  /* screen launches: (query chunk of up to 2048, gallery chunk of up to 65536) pairs */
} jimm_search_stats;
JIMM_API int jimm_index_create(jimm_model_t* m, jimm_index_t** out);
JIMM_API int jimm_index_rebind(jimm_index_t* idx, jimm_model_t* m);
JIMM_API int jimm_index_add(jimm_index_t* idx, const float* rows, int n, void* stream);
JIMM_API int jimm_index_search(jimm_index_t* idx, const float* queries, int Q, int k, float* values, int32_t* indices, jimm_search_stats* stats,
                               void* stream);
JIMM_API int jimm_index_destroy(jimm_index_t* idx);
/* Threshold search of a gallery index.  Scores are the ones jimm_index_search ranks (fp32, on the model's score scale: exp(logit_scale)
 * cos + logit_bias); a pair is a hit when its score >= threshold in IEEE order (a NaN score never is; -0 >= +0).  threshold must not be
 * NaN (JIMM_EINVAL); +inf and -inf are allowed.
 * jimm_index_range_search: for each of the Q queries (device fp32 [Q, E], as jimm_index_search takes them) every row added so far whose
 *   score is >= threshold, in ascending row order.  Rows: Q.
 * jimm_index_pairs: for each stored row i every stored row j > i whose score against it is >= threshold (score(i, j) and score(j, i) are
 *   the same bits), in ascending j.  Rows: the rows added so far.
 * Both screen in fp16 on the tensor cores against a fixed accumulator bound and rescore the survivors exactly, as jimm_index_search
 *   does; stats (nullable, host) receives the work done.  They wait for `stream` once per screened chunk of 65536 rows and once per
 *   chunk of 2048 query rows, size the result from the counts and return it in *out, a jimm_hits_t the caller destroys.  If the hits
 *   do not fit in device memory the call returns JIMM_ENOMEM, names the hits reached, frees what it allocated in stream order and sets
 *   *out to NULL; the index is unchanged.  Device memory: 8 bytes per hit and 8 per row in the result, and as much again for one
 *   query chunk's staged hits while it runs.
 * jimm_hits_size: the result's rows and hits (host values, no wait).
 * jimm_hits_copy: CSR into caller memory (device or host): offsets int64 [rows + 1] (offsets[0] = 0), scores fp32 [total], indices
 *   int32 [total] (the row numbers of the hits), enqueued on `stream`.
 * jimm_hits_destroy: waits for the result's device, then frees it. */
typedef struct jimm_hits jimm_hits_t;
JIMM_API int jimm_index_range_search(jimm_index_t* idx, const float* queries, int Q, float threshold, jimm_hits_t** out,
                                     jimm_search_stats* stats, void* stream);
JIMM_API int jimm_index_pairs(jimm_index_t* idx, float threshold, jimm_hits_t** out, jimm_search_stats* stats, void* stream);
JIMM_API int jimm_hits_size(const jimm_hits_t* h, int* rows, long long* total);
JIMM_API int jimm_hits_copy(const jimm_hits_t* h, int64_t* offsets, float* scores, int32_t* indices, void* stream);
JIMM_API int jimm_hits_destroy(jimm_hits_t* h);
/* Removing rows and searching a subset of a gallery index.  A row keeps its number from jimm_index_add until jimm_index_compact, removed
 * or not, and numbers are never reused.
 * jimm_index_remove: marks rows ids (device int32 [n], any order, duplicates allowed) removed; *removed (host) = the rows newly removed.
 *   An id outside 0 .. rows - 1 is JIMM_EINVAL and removes nothing.  Waits for `stream` once.  Removed rows keep their memory.
 * jimm_index_live: *live = the rows not removed (host, no wait).
 * jimm_index_search_keep / _range_search_keep / _pairs_keep: the calls above over the allowed rows -- the live rows with keep[r] != 0
 *   (keep: device bytes [rows], a bool tensor's memory; NULL keeps every row) -- bit for bit the same call on an index holding only
 *   those rows, with results in the index's row numbers.  Pairs need both rows allowed, and their result still has one row per stored
 *   row.  A search with fewer than k allowed rows pads each query's outputs past them with (-inf, -1); k's limit is unchanged.  With
 *   keep NULL and no row removed they run exactly as the calls without _keep; those calls are these with keep NULL, so after a
 *   removal they too see only the live rows.  Otherwise each call first lists the allowed rows (4 bytes each, one more wait for
 *   `stream`) and reads them through a buffer of 65536 rows, (6 E + 4) bytes each; rows_rescored counts allowed rows only.
 * jimm_index_compact: drops the removed rows: the live ones are renumbered 0 .. live - 1 in order, into new storage of exactly that
 *   size (the old one freed in stream order).  old_to_new (nullable, device int32 [rows before]) gets each row's new number, -1 for a
 *   removed row.  JIMM_ENOMEM leaves the index as it was. */
JIMM_API int jimm_index_remove(jimm_index_t* idx, const int32_t* ids, int n, long long* removed, void* stream);
JIMM_API int jimm_index_live(const jimm_index_t* idx, long long* live);
JIMM_API int jimm_index_search_keep(jimm_index_t* idx, const float* queries, int Q, int k, const uint8_t* keep, float* values, int32_t* indices,
                                    jimm_search_stats* stats, void* stream);
JIMM_API int jimm_index_range_search_keep(jimm_index_t* idx, const float* queries, int Q, float threshold, const uint8_t* keep, jimm_hits_t** out,
                                          jimm_search_stats* stats, void* stream);
JIMM_API int jimm_index_pairs_keep(jimm_index_t* idx, float threshold, const uint8_t* keep, jimm_hits_t** out, jimm_search_stats* stats,
                                   void* stream);
JIMM_API int jimm_index_compact(jimm_index_t* idx, int32_t* old_to_new, void* stream);
/* Spherical k-means over the stored rows of a gallery index.  The rows are the normalised rows jimm_index_add stored.  A row takes part
 * when it is live, kept (keep as jimm_index_search_keep) and its norm bound is at most 2 (zero, non-finite and subnormal-sum rows are
 * not); the others get assign -1 and score -inf.  score(x, c) = jimm_k_logits(x, c) at logit_scale 0 (exp(0) = 1) and no bias: the
 * cosine, whatever the model's logit_scale and logit_bias.  Initial means m_0 [C, E]: init_vectors (device fp32 [C, E]), the stored rows
 * init_ids (device int32 [C], each a row that takes part, repeats allowed), or, both NULL, the rows at the first C positions of
 * top_k(keys, C) with key 1 + (splitmix64(seed + id) >> 41) 2^-23 for the rows taking part in ascending id (splitmix64(x): the first
 * output of the generator with state x).  Step t = 0, 1, ..: c_t = l2_normalize(m_t); a_t = each row's best cluster (top_k at k = 1:
 * equal scores to the larger cluster); stop when t + 1 == iters or t > 0 and a_t == a_{t-1}; else m_{t+1}[j] = fp32(fp64(S_j) 2^-30 /
 * n_j), S_j[e] = sum over the n_j rows x of cluster j of rint(x[e] 2^30) in int64 (exact, so independent of order), keeping m_t[j] when
 * n_j = 0 or l2_normalize(m_{t+1}[j]) is not finite.  Outputs (device): centroids fp32 [C, E] = the c_t of the last step, assign int32
 * [rows], scores fp32 [rows] (each row's score against its centroid), counts int64 [C] (rows per cluster under assign); *iterations
 * (host) = the steps run.  stats sums jimm_index_search's counters over the steps.  JIMM_EINVAL before any launch for C outside 1 ..
 * 65536, iters < 1 or both inits given; after a check on the device and before any output is written for init ids that do not take
 * part (or are outside 0 .. rows - 1), initial centroids whose l2_normalize is not finite, or sampling more clusters than rows taking
 * part.  Memory, in stream order: 8 C E bytes of sums, 18 C E + 20 C bytes of means, centroids and their fp16 copies, 16 bytes per row
 * taking part, and a search's scratch per step.  Waits for `stream` to list the rows, to check the initial centroids, once per step
 * and once per screened chunk of 2048 rows. */
JIMM_API int jimm_index_kmeans(jimm_index_t* idx, int C, const float* init_vectors, const int32_t* init_ids, unsigned long long seed, int iters,
                               const uint8_t* keep, float* centroids, int32_t* assign, float* scores, int64_t* counts, int* iterations,
                               jimm_search_stats* stats, void* stream);
/* Micro-benchmark (not on the product path): TMA fill bandwidth from L2 with `cluster` CTAs per cluster.  mode 0: every CTA loads
 * its own 16 KB tiles; 1: the CTAs of a cluster load the same tile each; 2: same tile, each loads 1/cluster of it and multicasts. */
JIMM_API int jimm_k_l2_probe(const void* buf, int rows, int mode, int cluster, int iters, float* ms, void* stream);
/* Live timing of the dominant kernel (the wgmma GEMM) inside a forward: between begin and end every GEMM launch is
 * bracketed by CUDA events on the launch stream; end synchronises and returns the summed device time (ms), the
 * algorithmic FLOPs (2*M*N*K per launch) and the number of launches.  Used by bench.py's roofline object. */
JIMM_API int jimm_profile_begin(jimm_model_t* m);
JIMM_API int jimm_profile_end(jimm_model_t* m, double* gemm_ms, double* gemm_flops, long long* gemm_launches);
/* Count of kernel launches issued by this library since process start (bench.py's gpu_launches). */
JIMM_API long long jimm_launch_count(void);
/* Count of tower forwards replayed from a captured CUDA graph (batches <= JIMM_GRAPH_MAX_BATCH, default 32, from the
 * second call of a shape on); their kernels are included in jimm_launch_count. */
JIMM_API long long jimm_graph_replay_count(void);

#ifdef __cplusplus
}
#endif
#endif /* JIMM_B200_H_ */
