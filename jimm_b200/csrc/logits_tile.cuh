// fp32 64x64 logits tile shared by the single-GPU logits kernel (elementwise.cu) and the fused
// normalise + peer-scatter + logits kernel (comm.cu).  256 threads, 4x4 micro-tile per thread, K step 16.
//
// The operands arrive as one 128-bit load per thread and K step (row r = thread / 4, four consecutive k), are transposed into shared
// memory (k-major, row stride 68 floats = 17 x 16 B so that a thread's four i / four j values are ONE 128-bit shared load each), and the
// next step's global loads are issued before the current step's FMAs.  The accumulation order per output element is k ascending in
// one FMA chain, so the fused multi-GPU head stays bit-identical to the single-GPU one.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace jimm {

static constexpr int LOGITS_LDS = 68;  // shared-memory row stride (floats)

// The logit of one pair from its dot-product accumulator: one fused multiply-add, fl(sc * acc + bs), rounded once.  The gallery
// index's rescorer (postprocess.cu) computes its scores through this same function, so they are these bits.
__device__ __forceinline__ float logit_value(float sc, float acc, float bs) { return __fmaf_rn(sc, acc, bs); }

// out[i, j] = sc * <A[i, :E], B[j, :E]> + bs   for the 64x64 tile at (i0, j0); row strides lda / ldb / ldl (elements).
// CG_LOADS: read the operands with ld.global.cg (data written by peer GPUs into local memory; bypass L1).
template <bool CG_LOADS>
__device__ __forceinline__ void logits_tile(const float* __restrict__ A, size_t lda, const float* __restrict__ B, size_t ldb,
                                            float* __restrict__ out, size_t ldl, int Bi, int Bt, int E, int i0, int j0, float sc,
                                            float bs, float (*As)[LOGITS_LDS], float (*Bs)[LOGITS_LDS]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lr = threadIdx.x >> 2, lk = (threadIdx.x & 3) * 4;  // loader: row of the tile, first of its four k
  const bool vec = (E & 3) == 0 && (lda & 3) == 0 && (ldb & 3) == 0 && ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15) == 0;
  const float* arow = A + static_cast<size_t>(i0 + lr) * lda;
  const float* brow = B + static_cast<size_t>(j0 + lr) * ldb;
  const bool a_ok = i0 + lr < Bi, b_ok = j0 + lr < Bt;
  auto ld1 = [](const float* p) { return CG_LOADS ? __ldcg(p) : *p; };
  auto ld4 = [](const float* p) { return CG_LOADS ? __ldcg(reinterpret_cast<const float4*>(p)) : *reinterpret_cast<const float4*>(p); };
  auto load = [&](int k0, float4& a4, float4& b4) {
    const int k = k0 + lk;
    a4 = make_float4(0.f, 0.f, 0.f, 0.f);
    b4 = a4;
    if (vec) {  // E % 4 == 0: k < E implies k + 3 < E
      if (a_ok && k < E) a4 = ld4(arow + k);
      if (b_ok && k < E) b4 = ld4(brow + k);
    } else {
      if (a_ok) {
        if (k < E) a4.x = ld1(arow + k);
        if (k + 1 < E) a4.y = ld1(arow + k + 1);
        if (k + 2 < E) a4.z = ld1(arow + k + 2);
        if (k + 3 < E) a4.w = ld1(arow + k + 3);
      }
      if (b_ok) {
        if (k < E) b4.x = ld1(brow + k);
        if (k + 1 < E) b4.y = ld1(brow + k + 1);
        if (k + 2 < E) b4.z = ld1(brow + k + 2);
        if (k + 3 < E) b4.w = ld1(brow + k + 3);
      }
    }
  };
  float acc[4][4] = {};
  float4 a4, b4;
  load(0, a4, b4);
  for (int k0 = 0; k0 < E; k0 += 16) {
    As[lk][lr] = a4.x; As[lk + 1][lr] = a4.y; As[lk + 2][lr] = a4.z; As[lk + 3][lr] = a4.w;
    Bs[lk][lr] = b4.x; Bs[lk + 1][lr] = b4.y; Bs[lk + 2][lr] = b4.z; Bs[lk + 3][lr] = b4.w;
    __syncthreads();
    if (k0 + 16 < E) load(k0 + 16, a4, b4);  // in flight during the FMAs below
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a[4] = {av.x, av.y, av.z, av.w}, b[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int w = 0; w < 4; ++w) acc[u][w] = fmaf(a[u], b[w], acc[u][w]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int i = i0 + ty * 4 + u, j = j0 + tx * 4 + w;
      if (i < Bi && j < Bt) out[static_cast<size_t>(i) * ldl + j] = logit_value(sc, acc[u][w], bs);
    }
}

}  // namespace jimm
