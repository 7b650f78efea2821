// Host-side interface of the wgmma/TMA GEMM (gemm.cu).
//
//   C[M,N] = epilogue( A[M,K] . B[N,K]^T )      A, B K-major ("TN"), fp32 accumulate in registers
//
// This one kernel serves every dense contraction on the jimm forward path
// (SURVEY.md 8a rows a1,a4,a6,a7,a9,a10): patch-embed, fused QKV, attention
// out-projection (+residual), MLP FC1 (+GELU/QuickGELU), FC2 (+residual), MAP-head
// k/v + MLP, classifier / projections.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace jimm {

// DT_TF32: stored as fp32 with the value rounded (to nearest) to tf32 -- the operand format of the fp32 compute mode, so the
// tensor core's truncation of the low 13 mantissa bits is exact.  Only ever an internal buffer / operand type.
// DT_E4M3: float8 e4m3 (fn) operand with power-of-two scales kept beside it (one per A row, one per B row); the FP8 compute mode's
// QKV / FC1 operands.
enum DType : int { DT_F32 = 0, DT_F16 = 1, DT_BF16 = 2, DT_TF32 = 3, DT_E4M3 = 4 };
enum Act : int { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_QUICK_GELU = 2 };

inline size_t dtype_size(int dt) { return (dt == DT_F32 || dt == DT_TF32) ? 4 : dt == DT_E4M3 ? 1 : 2; }

// Output tile of one CTA (M rows x N columns).  A GEMM runs ceil(M / GEMM_TILE_M) x ceil(N / GEMM_TILE_N) tiles on at most one CTA per
// SM, so its time goes in waves of that many tiles.
constexpr int GEMM_TILE_M = 128;
constexpr int GEMM_TILE_N = 256;

struct GemmEpilogue {
  const float* bias = nullptr;      // [N] fp32, added per output column
  int act = ACT_NONE;               // applied after bias
  const float* rowadd = nullptr;    // fp32 [*, N]; row (r % rows_in + row_off) added (position embeddings)
  const float* residual = nullptr;  // fp32, indexed like the output (out_row, ldr); may alias out
  int ldr = 0;
  void* out = nullptr;
  int out_type = DT_F32;
  int ldo = 0;                                   // output row stride (elements)
  // Token-scatter form of the fp32 reduce-add epilogue (patch embedding): A rows are (sample, padded patch index) with
  // tok_pad rows per sample (multiple of 16, dividing M); row (b, p) is ADDED to out[b, p + tok_off, :] of a [B, tok_S, N] tensor through a
  // 3-D tensor map (rows p + tok_off >= tok_S are clipped by TMA, so the pad rows p >= tok_S - tok_off of A are never added).
  // Requires residual == out, fp32 (pre-initialised with pos-emb), and the TMA epilogue: gemm_plan_init fails otherwise.
  int tok_pad = 0, tok_off = 0, tok_S = 0;
  int reverse = 0;  // walk the M tiles from the end (L2-resident part of the A operand first; see kernels.cuh)
  int rows_in = 0, rows_out = 0, row_off = 0;    // out_row = (r / rows_in) * rows_out + r % rows_in + row_off (rows_in == 0: identity)
  // 2: TMA epilogue (swizzled smem box -> cp.async.bulk.tensor store, cp.reduce .add for the fp32 residual stream; needs
  //    no rowadd / row remap and residual == out, 16-byte aligned out / ldo and N x element size) -- falls back to 0 when not applicable;
  // 0 / 1: LSU stores straight from the accumulator registers (any shape, row remap, row-add, residual read)
  int mode = 2;
  // Fused LayerNorm of the UPDATED residual rows (fp32 reduce-add epilogue only): when the last column tile of a 32-row group has
  // been added, the CTA that completed it normalises those rows (nnx.LayerNorm fast variance,
  // common/transformer.py:130-131: the norm that follows `x + attn(...)` / `x + mlp(...)`) and writes them as the next GEMM's A operand.
  // ln_cnt: int32 [ceil(M/32)] completion counters, zero before the first launch (the kernel resets them).  ln_out may alias this
  // GEMM's A operand (rows whose tiles are all done are no longer read).
  const float* ln_scale = nullptr;
  const float* ln_bias = nullptr;
  void* ln_out = nullptr;
  int ln_out_type = DT_F16, ln_ldo = 0;
  float ln_eps = 1e-6f;
  int* ln_cnt = nullptr;
  // DT_E4M3 operands only (required there, ignored otherwise): fp32 dequantisation scales, a_scale [rows of A] and b_scale [N];
  // the accumulator is multiplied by a_scale[row] * b_scale[col] before the bias.  FP8 plans take the plain stores only (bias,
  // activation; no residual, row remap, row-add, token scatter or fused LayerNorm).
  const float* a_scale = nullptr;
  const float* b_scale = nullptr;
};

// Screening epilogue of the gallery index (fp16 operands; see epilogue_screen in gemm.cu): no output is written.  Column j of row i is
// kept when acc_ij + delta_ij >= t[i] (or the comparison is unordered), delta_ij = c1 nq[i] ng[j] + c2 (nq[i] + ng[j]) + c3 at K = E
// (screen_bound); a kept j goes to list[i * cap + atomicAdd(&cnt[i], 1)] when that slot is below cap.  cnt[i] > cap afterwards means
// row i's list overflowed.
struct GemmScreen {
  const float* t = nullptr;   // [M] per-row thresholds
  const float* nq = nullptr;  // [M] row norm bounds of A
  const float* ng = nullptr;  // [N] row norm bounds of B
  int* cnt = nullptr;         // [M] zero before the launch
  int* list = nullptr;        // [M, cap] column indices
  int cap = 0;
};

// c_tc / E: the bound on the fp16 wgmma's accumulation error per unit of sum |q^ g^| and of K (measured by the GPU tests)
constexpr double kTcAccumPerK = 0x1p-22;

// The screen's bound delta = c1 nq ng + c2 (nq + ng) + c3 on |fp16 wgmma sum - fp32 fmaf chain| at width E (derivation at
// epilogue_screen, gemm.cu), each constant rounded up by 2^-20 relative.
struct ScreenBound {
  float c1, c2, c3;
};
__host__ __device__ inline ScreenBound screen_bound(int E) {
  const double u = 0x1p-11, s = 0x1p-25 * sqrt(static_cast<double>(E)), gam = E * 0x1p-24 / (1.0 - E * 0x1p-24), ctc = E * kTcAccumPerK;
  const double up = 1.0 + 0x1p-20;
  return {static_cast<float>((2 * u + u * u + gam + ctc * (1 + u) * (1 + u)) * up), static_cast<float>(((1 + 2 * u) * s + ctc * (1 + u) * s) * up),
          static_cast<float>((E * 0x1p-50 + ctc * s * s) * up)};
}

struct GemmPlan {
  CUtensorMap map_a, map_b, map_c;  // map_c: output (mode 2 only)
  int M = 0, N = 0, K = 0;
  int dtype = DT_F16;  // operand type: DT_F16 / DT_BF16 / DT_F32 (tf32 MMA) / DT_E4M3
  GemmEpilogue epi;
};

// Build TMA descriptors for A [M,K] (row stride lda elements) and B [N,K] (row stride ldb).
// Returns 0 or a negative status (message in jimm_last_error()).
int gemm_plan_init(GemmPlan* plan, int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K,
                   const GemmEpilogue& epi);
// Enqueue on `stream`; M may be overridden (<= planned M) to run on fewer rows of the same buffers.  Rows < M are the same bits a
// plan built for exactly M rows gives.  The tensor maps still span the planned rows, so with M < planned M:
//   - the generic epilogue (mode 0 / 1) writes no row >= M;
//   - the TMA epilogues (mode 2) store / reduce-add whole 16-row boxes: rows [M, roundup(M, 16)) of the output (the residual
//     stream for the reduce-add) receive values computed from whatever A holds there; rows >= roundup(M, 16) are never written.
//     A token-scatter plan runs whole samples (M % tok_pad == 0), so its boxes never pass M.
//   - the fused LayerNorm normalises rows < M only.
int gemm_plan_run(const GemmPlan* plan, int M_override, cudaStream_t stream, int reverse = 0);

// Simple SIMT reference GEMM (debug / bring-up cross-check on the GPU; never on the product path
// unless JIMM_GEMM_IMPL=simt is set for bisection).
int gemm_simt_run(int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const GemmEpilogue& epi,
                  cudaStream_t stream);

// The screen of the gallery index: fp16 A [M, K] . B [N, K]^T (both K-major, row stride K, 16-byte aligned) on the same mainloop, ring,
// tiles and schedule as every other 16-bit GEMM, through the GemmScreen epilogue.
int gemm_screen_run(const void* A, int M, const void* B, int N, int K, const GemmScreen& screen, cudaStream_t stream);

// 1 when gemm_plan_run(plan, M_override) will apply the plan's fused LayerNorm (fp32 reduce-add epilogue)
int gemm_fuses_ln(const GemmPlan* plan, int M_override);

int device_sm_count();

}  // namespace jimm
