// Host-callable launchers for the non-GEMM kernels of the forward path (elementwise.cu, attention.cu).
// All enqueue on `stream` and return 0 / negative status (message via jimm_last_error()).
// `reverse`: walk the rows / tiles / items from the end.  Consecutive kernels of an encoder block alternate direction so each
// one starts on the data its producer wrote LAST -- the part still resident in the 50 MB L2 (the activations are 77-310 MB).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gemm.cuh"

struct jimm_hits;  // the C ABI's jimm_hits_t (postprocess.cu)

namespace jimm {

// nnx.LayerNorm (fast variance, fp32 statistics) over fp32 rows.  SURVEY 8a row a3.
//   src row for output r:  r * group + (row_index ? row_index[r] : row_off)      (row stride ldx elements)
//   out[r, :] (type out_type, row stride ldy) = (x - mean) * rsqrt(max(0, E[x^2]-mean^2) + eps) * scale + bias
//   out_type DT_E4M3: out[r, :] = e4m3(y / s_r), row_scale[r] = s_r (power of two from the row's absolute maximum; ldy in bytes)
int layernorm_run(const float* x, int ldx, int group, int row_off, const int* row_index, const float* scale, const float* bias,
                  float eps, void* out, int out_type, int ldy, int rows, int D, cudaStream_t stream, int reverse = 0,
                  float* row_scale = nullptr);

// Weight quantiser of the FP8 compute mode: each row of an fp32 [rows, K] matrix (row stride lds) -> e4m3 row of out (row stride ldo
// bytes) and its scale row_scale[r], by the same rule as the e4m3 LayerNorm.  One warp per row.
int quantize_rows_e4m3_run(const float* src, int lds, int rows, int K, void* out, int ldo, float* row_scale, cudaStream_t stream);

// Patchify: NHWC image (in_type fp32/fp16/bf16) -> A matrix [B*gh*gw, P*P*C] of out_type, row order (b,gy,gx), column
// order (ky,kx,c) == the HWIO kernel reshape (common/vit.py:153-165,228-230).  128-bit loads.
int patchify_run(const void* img, int in_type, int B, int H, int W, int C, int P, void* out, int out_type, cudaStream_t stream,
                 int rows_per_sample = 0 /* 0 = gh*gw; larger = padded row count per sample (pad rows untouched) */,
                 int ldk = 0 /* row stride in elements; 0 = P*P*C; larger = zero-padded K (any P / C through the generic kernel) */);

// x[b, s, :] = pos[s, :] (+ cls for s == 0)   -- initial value of the residual stream; the patch GEMM then reduce-adds the
// patch embeddings into rows tok_off.. (common/vit.py:231-236)
int tokens_init_run(float* x, const float* cls, const float* pos, int B, int S, int D, cudaStream_t stream);

// How the position table is resampled to another patch grid: bicubic (HF's interpolate_pos_encoding) or antialiased bilinear (SigLIP 2
// NaFlex); both F.interpolate with align_corners=False.
enum PosInterp : int { POS_BICUBIC = 0, POS_BILINEAR_AA = 1 };

// tokens_init_run on a gh x gw patch grid for a table trained on a g x g grid: x[b, 0, :] = cls + pos[0] (cls != null), and the patch
// rows (row-major over (gh, gw)) are the resampling (mode: PosInterp) of pos's g x g patch rows, computed on the fly from 16 table rows
// each (bicubic) or the rows under the antialias window (up to g per axis).  x: fp32 [B, gh*gw (+1), D]; at (gh, gw) == (g, g) the same
// bits as tokens_init_run in either mode.
int tokens_init_interp_run(float* x, const float* cls, const float* pos, int g, int D, int B, int gh, int gw, int mode, cudaStream_t stream);

// Packed form of tokens_init_interp_run for B images of different grids, after the patch GEMM: image b is rows seq_off[b] ..
// seq_off[b + 1] - 1 of x (device int32 [B + 1]), its grid is (n_b / gw[b]) x gw[b] (gw: device int32 [B]).  Its CLS row (cls != null) is
// set to cls + pos[0]; every patch row, which holds that patch's embedding, gets the resampled table row added -- the bits the
// per-image path gives by reduce-adding the embedding onto the table.  max_S: the longest image's rows.
int tokens_add_interp_packed_run(float* x, const float* cls, const float* pos, int g, int D, const int* seq_off, const int* gw, int B, int max_S,
                                 int mode, cudaStream_t stream);

// The patch-GEMM operand of a packed call from HuggingFace NaFlex patch rows: pv [B, N, K] of in_type (K = P*P*C in (py, px, c) order, the
// order patchify writes), sample b's rows 0 .. n_b - 1 (n_b = seq_off[b + 1] - seq_off[b] <= max_rows <= N; seq_off device int32 [B + 1])
// -> rows seq_off[b] + r of out [*, ldk] in out_type, columns K .. ldk - 1 zeros.  The other rows of pv are never read.
int patch_rows_packed_run(const void* pv, int in_type, int N, int K, const int* seq_off, int B, int max_rows, void* out, int out_type, int ldk,
                          cudaStream_t stream);

// x[b, 0, :] = cls + pos[0]   (common/vit.py:231-236), fp32 residual stream [B, S, D]
int cls_row_run(float* x, const float* cls, const float* pos, int B, int S, int D, cudaStream_t stream);

// x[b,t,:] = table[ids[b,t], :] + pos[t, :]   (models/clip.py:159-160, models/siglip.py:146-147)
int embed_run(const int32_t* ids, const float* table, const float* pos, float* x, int B, int T, int D, int vocab, cudaStream_t stream);

// Packed form of embed_run for B sequences of different lengths: sequence b is rows seq_off[b] .. seq_off[b + 1] - 1 of ids / x
// (seq_off: device int32 [B + 1], rows = seq_off[B]), its positions restart at 0: x[r, :] = table[ids[r], :] + pos[r - seq_off[b], :].
int embed_packed_run(const int32_t* ids, const float* table, const float* pos, float* x, const int* seq_off, int B, int rows, int D, int vocab,
                     cudaStream_t stream);

// idx[b] = first argmax_t ids[b, t]    (models/clip.py:164)
int argmax_ids_run(const int32_t* ids, int* idx, int B, int T, cudaStream_t stream);
// Packed form over the sequences of embed_packed_run: row[b] = seq_off[b] + first argmax_t ids[seq_off[b] + t] (an absolute row)
int argmax_ids_packed_run(const int32_t* ids, const int* seq_off, int* row, int B, cudaStream_t stream);

// rows /= ||row||_2  (no epsilon; models/clip.py:183-184), fp32 [B,E] -> out (row stride ldo)
int l2_normalize_run(const float* x, float* out, int ldo, int B, int E, cudaStream_t stream);

// logits[i,j] = exp(logit_scale) * <img[i], txt[j]> (+ logit_bias)   fp32 SIMT (models/clip.py:186-187, models/siglip.py:172-173)
int logits_run(const float* img, const float* txt, const float* logit_scale, const float* logit_bias, float* logits, int Bi, int Bt,
               int E, int ldl, cudaStream_t stream);

// postprocess.cu.  Top-k of each logits row: the first k entries of jimm_postprocess's order (1 <= k <= cols), their values and,
// probs non-null, their softmax probabilities -- bit for bit.  Scratch is allocated in stream order on `stream`.
int topk_run(const float* logits, int rows, int cols, int ld, int k, float* values, int32_t* indices, float* probs, cudaStream_t stream);
// Top-k of each query's scores against the gallery (1 <= k <= min(N, 1024)) with no [Q, N] buffer: every score is the one
// l2_normalize_run + logits_run give for that pair (queries on the image side, gallery on the text side, or the other way round).
int search_run(const float* queries, int Q, const float* gallery, int N, int E, const float* logit_scale, const float* logit_bias, int k,
               float* values, int32_t* indices, cudaStream_t stream);

// Gallery index (postprocess.cu): rows of width E (a multiple of 8 up to 8192, as every model width is) normalised once and stored with
// an fp16 copy and per-row norm bounds; a search screens them on the tensor cores and rescores the survivors exactly, and gives search_run's bits for the same queries against
// every row added so far (1 <= k <= min(rows, 1024)).  The store's memory is allocated in stream order on the add's stream; the caller
// orders adds and searches on different streams.  stats (nullable, zeroed by the caller): rows rescored, (query, chunk) pairs that fell
// back to the exact block step, and chunks screened.  A search waits for its stream once per screened chunk.
struct GalleryStore;
int gallery_create(int E, GalleryStore** out);
long long gallery_rows(const GalleryStore* g);
int gallery_width(const GalleryStore* g);
int gallery_add(GalleryStore* g, const float* rows, int n, cudaStream_t stream);
// keep (nullable): device bytes [rows], nonzero keeps the row.  A search runs over the allowed rows -- live and kept -- as if they were
// the only rows, and with fewer than k of them the slots past the last are (-inf, -1).  With no filter and no removed rows it runs
// exactly as before any removal existed; otherwise it waits for its stream once more, to size the allowed rows.
int gallery_search(const GalleryStore* g, const float* queries, int Q, const float* logit_scale, const float* logit_bias, int k, const uint8_t* keep,
                   float* values, int32_t* indices, long long* stats, cudaStream_t stream);
void gallery_destroy(GalleryStore* g);
// Removed rows keep their number and their storage until gallery_compact.  gallery_remove: clears the live bit of ids[0 .. n) (device,
// each in 0 .. rows - 1, else JIMM_EINVAL and nothing is removed); *removed = the rows newly removed.  Waits for its stream once.
// gallery_compact: drops the removed rows into new storage of exactly the live rows, in order, and writes old_to_new (nullable, device
// [rows]: the new number, -1 for a removed row).  On failure the store is unchanged.
long long gallery_live(const GalleryStore* g);
int gallery_remove(GalleryStore* g, const int* ids, int n, long long* removed, cudaStream_t stream);
int gallery_compact(GalleryStore* g, int32_t* old_to_new, cudaStream_t stream);
// Every (query, stored row) pair whose score is >= threshold, in CSR (jimm_hits, postprocess.cu), each row's hits in ascending stored-row
// order: the Q queries against every stored row, or (pairs) the stored rows against the later ones, Q = rows.  The same screen and
// rescore as gallery_search with the threshold fixed; stats as there.  The call waits for its stream once per screened chunk and once
// per chunk of kSearchRows queries.  On failure *out is null and everything allocated is freed in stream order.
// keep as gallery_search: only allowed rows are hits, and for pairs both rows of a pair are allowed; the pairs result still has a
// row for every stored row.
int gallery_range(const GalleryStore* g, const float* queries, int Q, bool pairs, float threshold, const float* logit_scale,
                  const float* logit_bias, const uint8_t* keep, jimm_hits** out, long long* stats, cudaStream_t stream);
// Spherical k-means over the clusterable rows (live, kept, norm bound <= 2) with C clusters (1 .. 65536) and at most iters assignment
// steps; init: vectors (device fp32 [C, E]), row ids (device int32 [C]) or, both null, sampled from seed.  Outputs on the device:
// centroids fp32 [C, E], assign int32 / scores fp32 [rows] (-1 / -inf for rows that take no part), counts int64 [C]; *iterations
// (host).  stats as gallery_search, summed over the steps.  JIMM_EINVAL for init ids that are not clusterable, initial centroids with a
// non-finite l2_normalize, or more sampled clusters than clusterable rows, before any output is written.  Waits for its stream to size
// the rows, to check the initial centroids, once per screened chunk and once per step.
int gallery_kmeans(const GalleryStore* g, int C, const float* init_vectors, const int32_t* init_ids, unsigned long long seed, int iters,
                   const uint8_t* keep, float* centroids, int32_t* assign, float* scores, int64_t* counts, int* iterations, long long* stats,
                   cudaStream_t stream);

// dst[n*K + k] = cast(src[k*N + n])   (flax (in,out) kernel -> K-major [N,K] operand)
int transpose_cast_run(const float* src, int K, int N, void* dst, int out_type, int ldd, cudaStream_t stream);
int cast_run(const float* src, void* dst, int out_type, size_t n, cudaStream_t stream);

// Per-token hidden states: out[r, :] = x[r, :] for rows r < rows of a contiguous fp32 [rows, D] residual stream, out contiguous of
// out_type DT_F32 (a bit copy) | DT_F16 | DT_BF16 (round to nearest even).  D a multiple of 8, x and out 16-byte aligned; nothing past
// rows * D elements of out is written.  Launched with PDL: it waits for its stream predecessor before it reads x.
int tokens_out_run(const float* x, size_t rows, int D, void* out, int out_type, cudaStream_t stream);

// ---- checkpoint ingestion (pack.cu) ----
// rows of K elements of src_type (DT_F32 | DT_F16 | DT_BF16), row-major -> dst[r * ldd + k] of out_type
int pack_rows_run(const void* src, int src_type, size_t rows, size_t K, void* dst, int out_type, size_t ldd, cudaStream_t stream);
// kc rows (starting at row k0) of a (K, N) row-major matrix of src_type -> dst[n * ldd + k0 + k] of out_type (K-major operand)
int pack_transpose_run(const void* src, int src_type, int kc, int N, void* dst, int out_type, size_t ldd, int k0, cudaStream_t stream);
// two pinned host slots + two device slots: memcpy of chunk i+1 overlaps the DMA and the pack kernel of chunk i
struct UploadRing {
  static constexpr size_t kCap = static_cast<size_t>(32) << 20;
  void* pinned[2] = {nullptr, nullptr};
  void* dev[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  bool busy[2] = {false, false};
  int cur = 0;
  bool ready = false;
  int init();
  void destroy();
  int stage(const void* src, size_t bytes, cudaStream_t s, void** dptr);  // host -> pinned slot -> device slot (async); *dptr = device slot
  int commit(cudaStream_t s);                                              // after the consuming kernel has been enqueued
};
// The chunked host -> device loops of finalize, through `ring` on stream s (a chunk is at most one ring slot):
//   upload_rows: rows of K src_type elements (row-major host memory) -> dst[r * ldd + k] of out_type; a single row longer than a slot
//     (rows == 1, ldd == K) is split along K.
//   upload_kernel: a kernel's (K, N) view -- host memory holding it row-major (the flax layout) or, transposed, its [N, K] transpose --
//     into rows n0 .. n0 + N - 1 of the K-major operand dst [*, ldd] of out_type; columns K .. ldd - 1 are not written.
int upload_rows(UploadRing& ring, const void* host, int src_type, size_t rows, size_t K, void* dst, int out_type, size_t ldd, cudaStream_t s);
int upload_kernel(UploadRing& ring, const void* host, int src_type, int K, int N, bool transposed, void* dst, int out_type, size_t ldd, int n0,
                  cudaStream_t s);
int activation_run(const float* x, float* y, size_t n, int act /* 0 none, 1 gelu_tanh, 2 quick_gelu */, cudaStream_t stream);

// Multi-head softmax attention over the fused qkv buffer [B*S, 3D] (q | k | v, H heads of head_dim d; D = H d).  SURVEY 8a row a5.
//   o[b*S+s, h*d+j] = softmax_k((q/sqrt(d)) k^T  masked) v ; causal: key <= query.  d a multiple of 8 in [8, 128].
//   io_type fp16/bf16; out_type fp16/bf16/fp32/tf32
int attention_run(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, int causal, cudaStream_t stream,
                  int reverse = 0);

// attention_run over B samples of different lengths packed into one [rows, 3D] qkv / [rows, D] out: sample b is rows seq_off[b] ..
// seq_off[b + 1] - 1 (seq_off: device int32 [B + 1]), max_S >= every length.  causal: key <= query within each sample.  Each sample's
// rows are the bits attention_run gives on that sample alone.
int attention_packed_run(const void* qkv, int io_type, void* out, int out_type, const int* seq_off, int B, int max_S, int H, int head_dim,
                         int causal, cudaStream_t stream, int reverse = 0);

// The attention weights attention_run computes (HF output_attentions): p[b, h, q, k] = softmax_k((q/sqrt(d)) k^T masked) in fp32, written as
// out_type DT_F32 | DT_F16 | DT_BF16 (round to nearest even).  out: sample b's [H, S_b, S_b] block starts at element H * sum_{j<b} S_j^2,
// row-major; causal: the entries above the diagonal are 0.  seq_off null: B samples of S rows; else packed as in attention_packed_run
// (S = max_S).  io_type fp16/bf16.  Launched with PDL: it waits for its stream predecessor before it reads qkv.
int attn_probs_run(const void* qkv, int io_type, void* out, int out_type, const int* seq_off, int B, int S, int H, int head_dim, int causal,
                   cudaStream_t stream);

// MAP-head attention with a single (input-independent) probe query (common/vit.py:96-97).
//   q: fp32 [H*d] (already projected + biased), kv: [B*S, 2D] (k | v) io_type, out [B, D] out_type; d as attention_run
//   probs (optional): the weights the output sums with, [B, H, 1, S] of probs_type DT_F32 | DT_F16 | DT_BF16
int map_attention_run(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, cudaStream_t stream,
                      void* probs = nullptr, int probs_type = DT_F32);
// map_attention_run on samples packed as in attention_packed_run (kv: [rows, 2D]); out [B, D]; probs: sample b's [H, 1, S_b] from element
// H * seq_off[b] on
int map_attention_packed_run(const float* q, const void* kv, int io_type, void* out, int out_type, const int* seq_off, int B, int max_S, int H,
                             int head_dim, cudaStream_t stream, void* probs = nullptr, int probs_type = DT_F32);
// The longest sequence the MAP-head attention takes on `device` (its scores live in shared memory): into *max_S; 0 or an error code.
int map_attention_max_seq(int device, int* max_S);

}  // namespace jimm
