// Per-kernel entry points of the C ABI (jimm_k_*, include/jimm_b200.h): each launches one kernel family on caller-owned buffers, with
// no model handle, so tests can check a kernel on its own.
#include <mutex>

#include "../../include/jimm_b200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

namespace jimm {
extern std::mutex g_capture_mu;  // model.cu: held by every phase that must not overlap a graph capture (pinned staging among them)
}  // namespace jimm

using namespace jimm;

extern "C" {

int jimm_k_gemm_ex(int impl, int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* bias, int act,
                   const float* rowadd, const float* residual, int ldr, void* out, int out_type, int ldo, int rows_in, int rows_out,
                   int row_off, int epi_mode, int plan_M, int reverse, int tok_pad, int tok_off, int tok_S, const float* ln_scale,
                   const float* ln_bias, float ln_eps, void* ln_out, int ln_out_type, int ln_ldo, int* ln_counters, void* stream) {
  if (plan_M <= 0) plan_M = M;
  if (M <= 0 || M > plan_M) { set_last_error("jimm_k_gemm_ex: need 0 < M <= plan_M (M=%d plan_M=%d)", M, plan_M); return JIMM_EINVAL; }
  GemmEpilogue e;
  e.bias = bias; e.act = act; e.rowadd = rowadd; e.residual = residual; e.ldr = ldr; e.out = out; e.out_type = out_type; e.ldo = ldo;
  e.rows_in = rows_in; e.rows_out = rows_out; e.row_off = row_off; e.mode = epi_mode;
  e.tok_pad = tok_pad; e.tok_off = tok_off; e.tok_S = tok_S;
  if (ln_counters) {  // fp32 operands: the normalised rows are the next GEMM's tf32 operand
    e.ln_scale = ln_scale; e.ln_bias = ln_bias; e.ln_out = ln_out; e.ln_out_type = ln_out_type == JIMM_F32 ? DT_TF32 : ln_out_type; e.ln_ldo = ln_ldo;
    e.ln_eps = ln_eps; e.ln_cnt = ln_counters;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (impl == 1) {
    if (plan_M != M || reverse || tok_pad || ln_counters) {
      set_last_error("jimm_k_gemm_ex: the SIMT GEMM has no plan rows, reverse walk, token scatter or fused LayerNorm");
      return JIMM_EINVAL;
    }
    return gemm_simt_run(dtype, A, lda, B, ldb, M, N, K, e, s);
  }
  GemmPlan p;
  if (int rc = gemm_plan_init(&p, dtype, A, lda, B, ldb, plan_M, N, K, e)) return rc;
  if (ln_counters && !gemm_fuses_ln(&p, M)) {
    set_last_error("gemm: this shape does not take the fused LayerNorm path (needs N = 128 x {1,2,3,4,6,8,9}, aligned operands, "
                   "LayerNorm output in the operand type)");
    return JIMM_EINVAL;
  }
  return gemm_plan_run(&p, M, s, reverse);
}
int jimm_k_gemm(int impl, int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* bias, int act,
                const float* rowadd, const float* residual, int ldr, void* out, int out_type, int ldo, int rows_in, int rows_out,
                int row_off, int epi_mode, void* stream) {
  return jimm_k_gemm_ex(impl, dtype, A, lda, B, ldb, M, N, K, bias, act, rowadd, residual, ldr, out, out_type, ldo, rows_in, rows_out, row_off,
                        epi_mode, M, 0, 0, 0, 0, nullptr, nullptr, 0.f, nullptr, 0, 0, nullptr, stream);
}
int jimm_k_gemm_residual_ln(int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* bias, float* x, int ldx,
                            const float* ln_scale, const float* ln_bias, float eps, void* ln_out, int ln_out_type, int ln_ldo, int* counters,
                            void* stream) {
  if (!counters) { set_last_error("jimm_k_gemm_residual_ln: null counters"); return JIMM_EINVAL; }
  return jimm_k_gemm_ex(0, dtype, A, lda, B, ldb, M, N, K, bias, 0, nullptr, x, ldx, x, JIMM_F32, ldx, 0, 0, 0, 2, M, 0, 0, 0, 0, ln_scale,
                        ln_bias, eps, ln_out, ln_out_type, ln_ldo, counters, stream);
}
int jimm_k_layernorm_ex(const float* x, int ldx, int group, int row_off, const int32_t* row_index, const float* scale, const float* bias,
                        float eps, void* out, int out_type, int ldy, int rows, int D, int reverse, void* stream) {
  return layernorm_run(x, ldx, group, row_off, row_index, scale, bias, eps, out, out_type, ldy, rows, D, static_cast<cudaStream_t>(stream), reverse);
}
int jimm_k_layernorm(const float* x, int ldx, int group, int row_off, const int32_t* row_index, const float* scale, const float* bias,
                     float eps, void* out, int out_type, int ldy, int rows, int D, void* stream) {
  return jimm_k_layernorm_ex(x, ldx, group, row_off, row_index, scale, bias, eps, out, out_type, ldy, rows, D, 0, stream);
}
int jimm_k_layernorm_e4m3(const float* x, int ldx, const float* scale, const float* bias, float eps, void* out, int ldy, float* row_scale,
                          int rows, int D, int reverse, void* stream) {
  return layernorm_run(x, ldx, 1, 0, nullptr, scale, bias, eps, out, DT_E4M3, ldy, rows, D, static_cast<cudaStream_t>(stream), reverse,
                       row_scale);
}
int jimm_k_gemm_e4m3(int impl, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const float* a_scale, const float* b_scale,
                     const float* bias, int act, void* out, int out_type, int ldo, int epi_mode, int plan_M, int reverse, void* stream) {
  if (plan_M <= 0) plan_M = M;
  if (M <= 0 || M > plan_M) { set_last_error("jimm_k_gemm_e4m3: need 0 < M <= plan_M (M=%d plan_M=%d)", M, plan_M); return JIMM_EINVAL; }
  if (out_type < DT_F32 || out_type > DT_TF32) { set_last_error("jimm_k_gemm_e4m3: bad output type %d", out_type); return JIMM_EINVAL; }
  GemmEpilogue e;
  e.bias = bias; e.act = act; e.out = out; e.out_type = out_type; e.ldo = ldo; e.mode = epi_mode;
  e.a_scale = a_scale; e.b_scale = b_scale;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (impl == 1) {
    if (plan_M != M || reverse) { set_last_error("jimm_k_gemm_e4m3: the SIMT GEMM has no plan rows or reverse walk"); return JIMM_EINVAL; }
    return gemm_simt_run(DT_E4M3, A, lda, B, ldb, M, N, K, e, s);
  }
  GemmPlan p;
  if (int rc = gemm_plan_init(&p, DT_E4M3, A, lda, B, ldb, plan_M, N, K, e)) return rc;
  return gemm_plan_run(&p, M, s, reverse);
}
int jimm_k_quantize_e4m3(const float* src, int lds, int rows, int K, void* out, int ldo, float* row_scale, void* stream) {
  return quantize_rows_e4m3_run(src, lds, rows, K, out, ldo, row_scale, static_cast<cudaStream_t>(stream));
}
int jimm_k_attention_hd(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, int causal, int reverse,
                        void* stream) {
  return attention_run(qkv, io_type, out, out_type, B, S, H, head_dim, causal, static_cast<cudaStream_t>(stream), reverse);
}
int jimm_k_attention_ex(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int causal, int reverse, void* stream) {
  return jimm_k_attention_hd(qkv, io_type, out, out_type, B, S, H, 64, causal, reverse, stream);
}
int jimm_k_attention(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int causal, void* stream) {
  return jimm_k_attention_ex(qkv, io_type, out, out_type, B, S, H, causal, 0, stream);
}
int jimm_k_map_attention_hd(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, void* stream) {
  return map_attention_run(q, kv, io_type, out, out_type, B, S, H, head_dim, static_cast<cudaStream_t>(stream));
}
int jimm_k_attention_packed_ex(const void* qkv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int max_S, int H,
                               int head_dim, int causal, int reverse, void* stream) {
  return attention_packed_run(qkv, io_type, out, out_type, seq_off, B, max_S, H, head_dim, causal, static_cast<cudaStream_t>(stream), reverse);
}
int jimm_k_attention_packed(const void* qkv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int max_S, int H, int head_dim,
                            int reverse, void* stream) {
  return jimm_k_attention_packed_ex(qkv, io_type, out, out_type, seq_off, B, max_S, H, head_dim, 0, reverse, stream);
}
int jimm_k_map_attention_packed(const float* q, const void* kv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int max_S,
                                int H, int head_dim, void* stream) {
  return map_attention_packed_run(q, kv, io_type, out, out_type, seq_off, B, max_S, H, head_dim, static_cast<cudaStream_t>(stream));
}
int jimm_k_attn_probs(const void* qkv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int S, int H, int head_dim, int causal,
                      void* stream) {
  if (B > 0 && S > 0 && (!qkv || !out)) { set_last_error("jimm_k_attn_probs: null argument"); return JIMM_EINVAL; }
  return attn_probs_run(qkv, io_type, out, out_type, seq_off, B, S, H, head_dim, causal, static_cast<cudaStream_t>(stream));
}
int jimm_k_map_attention_probs(const float* q, const void* kv, int io_type, void* out, int out_type, const int32_t* seq_off, int B, int S, int H,
                               int head_dim, void* probs, int probs_type, void* stream) {
  if (seq_off) return map_attention_packed_run(q, kv, io_type, out, out_type, seq_off, B, S, H, head_dim, static_cast<cudaStream_t>(stream), probs, probs_type);
  return map_attention_run(q, kv, io_type, out, out_type, B, S, H, head_dim, static_cast<cudaStream_t>(stream), probs, probs_type);
}
int jimm_k_map_attention(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, void* stream) {
  return jimm_k_map_attention_hd(q, kv, io_type, out, out_type, B, S, H, 64, stream);
}
int jimm_k_patchify_ex(const void* img, int in_type, int B, int H, int W, int C, int P, void* out, int out_type, int rows_per_sample, int ldk,
                       void* stream) {
  return patchify_run(img, in_type, B, H, W, C, P, out, out_type, static_cast<cudaStream_t>(stream), rows_per_sample, ldk);
}
int jimm_k_patchify(const void* img, int in_type, int B, int H, int W, int C, int P, void* out, int out_type, void* stream) {
  return jimm_k_patchify_ex(img, in_type, B, H, W, C, P, out, out_type, 0, 0, stream);
}
int jimm_k_activation(const float* x, float* y, long long n, int act, void* stream) {
  if (n < 0 || (n > 0 && (!x || !y))) { set_last_error("jimm_k_activation: bad arguments"); return JIMM_EINVAL; }
  return activation_run(x, y, static_cast<size_t>(n), act, static_cast<cudaStream_t>(stream));
}
int jimm_k_tokens_init_interp_ex(const float* cls, const float* pos, int g, int D, float* x, int B, int gh, int gw, int mode, void* stream) {
  return tokens_init_interp_run(x, cls, pos, g, D, B, gh, gw, mode, static_cast<cudaStream_t>(stream));
}
int jimm_k_tokens_init_interp(const float* cls, const float* pos, int g, int D, float* x, int B, int gh, int gw, void* stream) {
  return jimm_k_tokens_init_interp_ex(cls, pos, g, D, x, B, gh, gw, POS_BICUBIC, stream);
}
int jimm_k_tokens_add_interp_packed(const float* cls, const float* pos, int g, int D, float* x, const int32_t* seq_off, const int32_t* gw, int B,
                                    int max_S, int mode, void* stream) {
  if (B > 0 && (!pos || !x || !seq_off || !gw || g <= 0)) { set_last_error("jimm_k_tokens_add_interp_packed: null argument or empty table"); return JIMM_EINVAL; }
  return tokens_add_interp_packed_run(x, cls, pos, g, D, seq_off, gw, B, max_S, mode, static_cast<cudaStream_t>(stream));
}
int jimm_k_patch_rows_packed(const void* patches, int in_type, int N, int K, const int32_t* seq_off, int B, int max_rows, void* out, int out_type,
                             int ldk, void* stream) {
  if (B > 0 && (!patches || !seq_off || !out)) { set_last_error("jimm_k_patch_rows_packed: null argument"); return JIMM_EINVAL; }
  return patch_rows_packed_run(patches, in_type, N, K, seq_off, B, max_rows, out, out_type, ldk, static_cast<cudaStream_t>(stream));
}
int jimm_k_embed(const int32_t* ids, const float* table, const float* pos, float* x, int B, int T, int D, int vocab, void* stream) {
  return embed_run(ids, table, pos, x, B, T, D, vocab, static_cast<cudaStream_t>(stream));
}
int jimm_k_embed_packed(const int32_t* ids, const float* table, const float* pos, float* x, const int32_t* seq_off, int B, int T_total, int D,
                        int vocab, void* stream) {
  return embed_packed_run(ids, table, pos, x, seq_off, B, T_total, D, vocab, static_cast<cudaStream_t>(stream));
}
int jimm_k_tokens_out(const float* x, long long rows, int D, void* out, int out_type, void* stream) {
  if (rows < 0 || (rows > 0 && (!x || !out))) { set_last_error("jimm_k_tokens_out: bad arguments"); return JIMM_EINVAL; }
  return tokens_out_run(x, static_cast<size_t>(rows), D, out, out_type, static_cast<cudaStream_t>(stream));
}
int jimm_k_l2_normalize(const float* x, float* out, int ldo, int B, int E, void* stream) {
  return l2_normalize_run(x, out, ldo, B, E, static_cast<cudaStream_t>(stream));
}
int jimm_k_logits(const float* img, const float* txt, const float* logit_scale, const float* logit_bias, float* logits, int Bi, int Bt,
                  int E, int ldl, void* stream) {
  return logits_run(img, txt, logit_scale, logit_bias, logits, Bi, Bt, E, ldl, static_cast<cudaStream_t>(stream));
}

// checkpoint ingestion as finalize runs it, through a staging ring of this call's own (freed, its last chunk done, before returning)
static int check_upload_types(const char* fn, const void* host, void* dst, int src_type, int out_type) {
  if (!host || !dst) { set_last_error("%s: null pointer", fn); return JIMM_EINVAL; }
  if (src_type < DT_F32 || src_type > DT_BF16 || out_type < DT_F32 || out_type > DT_TF32) {
    set_last_error("%s: bad type codes (src %d, out %d)", fn, src_type, out_type);
    return JIMM_EINVAL;
  }
  return 0;
}
int jimm_k_upload_rows(const void* host, int src_type, long long rows, long long K, void* dst, int out_type, long long ldd, void* stream) {
  if (int rc = check_upload_types("jimm_k_upload_rows", host, dst, src_type, out_type)) return rc;
  if (rows < 0 || K < 0 || ldd < K) { set_last_error("jimm_k_upload_rows: bad shape (rows %lld, K %lld, ldd %lld)", rows, K, ldd); return JIMM_EINVAL; }
  std::lock_guard<std::mutex> no_capture(g_capture_mu);  // pinned staging ring
  UploadRing ring;
  const int rc = upload_rows(ring, host, src_type, static_cast<size_t>(rows), static_cast<size_t>(K), dst, out_type, static_cast<size_t>(ldd),
                             static_cast<cudaStream_t>(stream));
  ring.destroy();
  return rc;
}
int jimm_k_upload_kernel(const void* host, int src_type, int K, int N, int transposed, void* dst, int out_type, long long ldd, int n0, void* stream) {
  if (int rc = check_upload_types("jimm_k_upload_kernel", host, dst, src_type, out_type)) return rc;
  if (K < 0 || N < 0 || n0 < 0 || ldd < K) { set_last_error("jimm_k_upload_kernel: bad shape (K %d, N %d, ldd %lld, n0 %d)", K, N, ldd, n0); return JIMM_EINVAL; }
  std::lock_guard<std::mutex> no_capture(g_capture_mu);  // pinned staging ring
  UploadRing ring;
  const int rc = upload_kernel(ring, host, src_type, K, N, transposed != 0, dst, out_type, static_cast<size_t>(ldd), n0,
                               static_cast<cudaStream_t>(stream));
  ring.destroy();
  return rc;
}

}  // extern "C"
