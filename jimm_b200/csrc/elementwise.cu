// HBM-bound kernels of the forward path: LayerNorm, patchify, CLS row, token embedding, pooling helpers,
// L2-normalise, fp32 logits, weight packing.  128-bit vectorised loads/stores, warp-shuffle reductions.
#include <limits.h>
#include <stdio.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "kernels.cuh"
#include "logits_tile.cuh"

namespace jimm {

// ------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row kept in registers (D <= 2048), fp32 statistics.
// OutT = __nv_fp8_e4m3: the normalised fp32 row y is quantised to e4m3 as y / s, s = 2^k from the row's absolute maximum
// (e4m3_scale_exp), and s goes to row_scale[r] -- the FP8 compute mode's QKV / FC1 A operand with its row scales.
// ------------------------------------------------------------------------------------------
template <typename OutT, int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, size_t ldx, int group, int row_off, const int* __restrict__ row_index,
                 const float* __restrict__ scale, const float* __restrict__ bias, float eps, OutT* __restrict__ out, size_t ldy,
                 int rows, int D, int reverse, float* __restrict__ row_scale) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  pdl_wait();
  if (warp >= rows) return;
  if (reverse) warp = rows - 1 - warp;
  const size_t src_row = static_cast<size_t>(warp) * group + (row_index ? row_index[warp] : row_off);
  const float4* xr = reinterpret_cast<const float4*>(x + src_row * ldx);
  const int nv = D >> 2;
  float4 v[MAXV];
  float s = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nv) {
      v[i] = xr[idx];
      s += v[i].x + v[i].y + v[i].z + v[i].w;
      s2 += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
    }
  }
  s = warp_sum(s);
  s2 = warp_sum(s2);
  const float inv_d = 1.0f / static_cast<float>(D);
  const float mean = s * inv_d;
  const float var = fmaxf(s2 * inv_d - mean * mean, 0.0f);  // flax use_fast_variance=True
  const float rstd = rsqrtf(var + eps);
  const float4* sc = reinterpret_cast<const float4*>(scale);
  const float4* bi = reinterpret_cast<const float4*>(bias);
  OutT* orow = out + static_cast<size_t>(warp) * ldy;
  if constexpr (std::is_same<OutT, __nv_fp8_e4m3>::value) {
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nv) {
        const float4 g = __ldg(sc + idx), b = __ldg(bi + idx);
        v[i].x = (v[i].x - mean) * rstd * g.x + b.x;
        v[i].y = (v[i].y - mean) * rstd * g.y + b.y;
        v[i].z = (v[i].z - mean) * rstd * g.z + b.z;
        v[i].w = (v[i].w - mean) * rstd * g.w + b.w;
        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
      }
    }
    const int k = e4m3_scale_exp(warp_max(amax));
    const float inv_s = ldexpf(1.0f, -k);
    if (lane == 0) row_scale[warp] = ldexpf(1.0f, k);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nv)
        reinterpret_cast<uint32_t*>(orow)[idx] = e4m3x4_rn(v[i].x * inv_s, v[i].y * inv_s, v[i].z * inv_s, v[i].w * inv_s);
    }
  } else {
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nv) {
      const float4 g = __ldg(sc + idx), b = __ldg(bi + idx);
      float4 y;
      y.x = (v[i].x - mean) * rstd * g.x + b.x;
      y.y = (v[i].y - mean) * rstd * g.y + b.y;
      y.z = (v[i].z - mean) * rstd * g.z + b.z;
      y.w = (v[i].w - mean) * rstd * g.w + b.w;
      if constexpr (std::is_same<OutT, tf32_t>::value) {
        reinterpret_cast<float4*>(orow)[idx] = make_float4(round_tf32(y.x), round_tf32(y.y), round_tf32(y.z), round_tf32(y.w));
      } else if constexpr (sizeof(OutT) == 4) {
        reinterpret_cast<float4*>(orow)[idx] = y;
      } else if constexpr (sizeof(OutT) == 2) {
        uint2 p;
        constexpr int ot = std::is_same<OutT, __half>::value ? 1 : 2;
        p.x = pack2(y.x, y.y, ot);
        p.y = pack2(y.z, y.w, ot);
        reinterpret_cast<uint2*>(orow)[idx] = p;
      }
    }
  }
  }
}

template <typename OutT>
static int ln_launch(const float* x, int ldx, int group, int row_off, const int* row_index, const float* scale, const float* bias,
                     float eps, void* out, int ldy, int rows, int D, cudaStream_t stream, int reverse, float* row_scale = nullptr) {
  const int threads = 256, wpb = threads / 32;
  const int grid = (rows + wpb - 1) / wpb;
  const int nv = D / 4;
  if (nv <= 32 * 8)
    JIMM_CUDA_CHECK(launch_k(layernorm_kernel<OutT, 8>, dim3(grid), dim3(threads), 0, stream, 1, true, x, ldx, group, row_off, row_index, scale, bias, eps,
                             static_cast<OutT*>(out), ldy, rows, D, reverse, row_scale));
  else
    JIMM_CUDA_CHECK(launch_k(layernorm_kernel<OutT, 16>, dim3(grid), dim3(threads), 0, stream, 1, true, x, ldx, group, row_off, row_index, scale, bias, eps,
                             static_cast<OutT*>(out), ldy, rows, D, reverse, row_scale));
  note_launch();
  return 0;
}

int layernorm_run(const float* x, int ldx, int group, int row_off, const int* row_index, const float* scale, const float* bias,
                  float eps, void* out, int out_type, int ldy, int rows, int D, cudaStream_t stream, int reverse, float* row_scale) {
  if (D % 4 != 0 || D > 2048 || ldx % 4 != 0 || ldy % 4 != 0) {
    set_last_error("layernorm: D=%d must be a multiple of 4 and <= 2048 (ldx=%d ldy=%d)", D, ldx, ldy);
    return -1;
  }
  if (out_type == DT_E4M3 && row_scale == nullptr) { set_last_error("layernorm: e4m3 output needs a row-scale vector"); return -1; }
  if (rows <= 0) return 0;
  if (out_type == DT_E4M3)
    return ln_launch<__nv_fp8_e4m3>(x, ldx, group, row_off, row_index, scale, bias, eps, out, ldy, rows, D, stream, reverse, row_scale);
  if (out_type == DT_F32) return ln_launch<float>(x, ldx, group, row_off, row_index, scale, bias, eps, out, ldy, rows, D, stream, reverse);
  if (out_type == DT_TF32) return ln_launch<tf32_t>(x, ldx, group, row_off, row_index, scale, bias, eps, out, ldy, rows, D, stream, reverse);
  if (out_type == DT_F16) return ln_launch<__half>(x, ldx, group, row_off, row_index, scale, bias, eps, out, ldy, rows, D, stream, reverse);
  return ln_launch<__nv_bfloat16>(x, ldx, group, row_off, row_index, scale, bias, eps, out, ldy, rows, D, stream, reverse);
}

// ------------------------------------------------------------------------------------------
// Patchify: each thread moves 4 consecutive source elements (one 128-bit load for fp32 input).
// ------------------------------------------------------------------------------------------
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
patchify_kernel(const InT* __restrict__ img, OutT* __restrict__ out, int B, int H, int W, int C, int P, int gh, int gw, int per_img4, int rps) {
  // blockIdx.y = image, 32-bit index arithmetic inside the image (64-bit divisions of a flat index make this kernel XU-bound)
  const int i4 = blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= per_img4) return;
  const int b = blockIdx.y;
  const int rem = i4 * 4;
  const int WC = W * C, PC = P * C;
  const size_t e = static_cast<size_t>(b) * H * WC + rem;
  const int y = rem / WC, xc = rem - y * WC;
  const int gx = xc / PC, kc = xc - gx * PC;
  const int gy = y / P, ky = y - gy * P;
  if (gy >= gh || gx >= gw) return;  // VALID conv drops the remainder
  float v[4];
  if constexpr (sizeof(InT) == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(img + e));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    const uint2 t = __ldg(reinterpret_cast<const uint2*>(img + e));
    const InT* h = reinterpret_cast<const InT*>(&t);
    for (int j = 0; j < 4; ++j) v[j] = to_float(h[j]);
  }
  const size_t dst = (static_cast<size_t>(b) * rps + static_cast<size_t>(gy) * gw + gx) * (static_cast<size_t>(P) * PC) +
                     static_cast<size_t>(ky) * PC + kc;
  if constexpr (std::is_same<OutT, tf32_t>::value) {
    *reinterpret_cast<float4*>(out + dst) = make_float4(round_tf32(v[0]), round_tf32(v[1]), round_tf32(v[2]), round_tf32(v[3]));
  } else if constexpr (sizeof(OutT) == 4) {
    *reinterpret_cast<float4*>(out + dst) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    constexpr int ot = std::is_same<OutT, __half>::value ? 1 : 2;
    uint2 p;
    p.x = pack2(v[0], v[1], ot);
    p.y = pack2(v[2], v[3], ot);
    *reinterpret_cast<uint2*>(out + dst) = p;
  }
}

template <typename InT>
static int patchify_dispatch(const void* img, int B, int H, int W, int C, int P, void* out, int out_type, cudaStream_t stream, int rps) {
  const int gh = H / P, gw = W / P;
  if (rps <= 0) rps = gh * gw;
  const int per_img4 = H * W * C / 4;
  const int threads = 256;
  const InT* in = static_cast<const InT*>(img);
  for (int b0 = 0; b0 < B; b0 += 65535) {  // grid.y limit
    const int nb = B - b0 < 65535 ? B - b0 : 65535;
    const dim3 grid(static_cast<unsigned>((per_img4 + threads - 1) / threads), static_cast<unsigned>(nb));
    const InT* src = in + static_cast<size_t>(b0) * H * W * C;
    const size_t ooff = static_cast<size_t>(b0) * rps * P * P * C;
    if (out_type == DT_F32) patchify_kernel<InT, float><<<grid, threads, 0, stream>>>(src, static_cast<float*>(out) + ooff, nb, H, W, C, P, gh, gw, per_img4, rps);
    else if (out_type == DT_TF32) patchify_kernel<InT, tf32_t><<<grid, threads, 0, stream>>>(src, static_cast<tf32_t*>(out) + ooff, nb, H, W, C, P, gh, gw, per_img4, rps);
    else if (out_type == DT_F16) patchify_kernel<InT, __half><<<grid, threads, 0, stream>>>(src, static_cast<__half*>(out) + ooff, nb, H, W, C, P, gh, gw, per_img4, rps);
    else patchify_kernel<InT, __nv_bfloat16><<<grid, threads, 0, stream>>>(src, static_cast<__nv_bfloat16*>(out) + ooff, nb, H, W, C, P, gh, gw, per_img4, rps);
  }
  JIMM_LAUNCH_CHECK();
  return 0;
}

// Generic form (any patch size / channel count, zero-padded K): one thread per OUTPUT element (b, patch, k), k in [0, ldk); columns
// k >= P*P*C are written as zeros so that the row stride ldk can be rounded up to the 16 bytes TMA needs (patch 14 x 3 channels = 588
// elements -> 592: every ViT-L/14 / H/14 CLIP and patch14 SigLIP checkpoint the reference loads).
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
patchify_generic_kernel(const InT* __restrict__ img, OutT* __restrict__ out, int H, int W, int C, int P, int gh, int gw, int rps, int ldk,
                        size_t total) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = static_cast<int>(i % ldk);
  const size_t r = i / ldk;
  const int n = gh * gw;
  const int b = static_cast<int>(r / n), pt = static_cast<int>(r - static_cast<size_t>(b) * n);
  const int gy = pt / gw, gx = pt - gy * gw;
  float v = 0.f;
  const int PC = P * C;
  if (k < P * PC) {
    const int ky = k / PC, kc = k - ky * PC;  // (kh, kw, c) order == the HWIO kernel reshape
    v = to_float(img[(static_cast<size_t>(b) * H + gy * P + ky) * W * C + static_cast<size_t>(gx) * PC + kc]);
  }
  out[(static_cast<size_t>(b) * rps + pt) * ldk + k] = from_float<OutT>(v);
}

template <typename InT>
static int patchify_generic_dispatch(const void* img, int B, int H, int W, int C, int P, void* out, int out_type, cudaStream_t stream, int rps, int ldk) {
  const int gh = H / P, gw = W / P;
  if (rps <= 0) rps = gh * gw;
  const size_t total = static_cast<size_t>(B) * gh * gw * ldk;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  const InT* in = static_cast<const InT*>(img);
  if (out_type == DT_F32) patchify_generic_kernel<InT, float><<<grid, 256, 0, stream>>>(in, static_cast<float*>(out), H, W, C, P, gh, gw, rps, ldk, total);
  else if (out_type == DT_TF32) patchify_generic_kernel<InT, tf32_t><<<grid, 256, 0, stream>>>(in, static_cast<tf32_t*>(out), H, W, C, P, gh, gw, rps, ldk, total);
  else if (out_type == DT_F16) patchify_generic_kernel<InT, __half><<<grid, 256, 0, stream>>>(in, static_cast<__half*>(out), H, W, C, P, gh, gw, rps, ldk, total);
  else patchify_generic_kernel<InT, __nv_bfloat16><<<grid, 256, 0, stream>>>(in, static_cast<__nv_bfloat16*>(out), H, W, C, P, gh, gw, rps, ldk, total);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ldk: row stride of `out` in elements (0 = P*P*C).  The vectorised kernel needs P*C and W*C to be multiples of 4 and an unpadded row.
int patchify_run(const void* img, int in_type, int B, int H, int W, int C, int P, void* out, int out_type, cudaStream_t stream, int rows_per_sample,
                 int ldk) {
  if (B <= 0) return 0;
  const int PPC = P * P * C;
  if (ldk <= 0) ldk = PPC;
  if (ldk < PPC) { set_last_error("patchify: row stride %d < patch_size^2*channels %d", ldk, PPC); return -1; }
  if (rows_per_sample != 0 && rows_per_sample < (H / P) * (W / P)) {
    set_last_error("patchify: rows_per_sample %d < patches per image %d", rows_per_sample, (H / P) * (W / P));
    return -1;
  }
  if ((P * C) % 4 != 0 || (W * C) % 4 != 0 || ldk != PPC) {
    if (in_type == DT_F32) return patchify_generic_dispatch<float>(img, B, H, W, C, P, out, out_type, stream, rows_per_sample, ldk);
    if (in_type == DT_F16) return patchify_generic_dispatch<__half>(img, B, H, W, C, P, out, out_type, stream, rows_per_sample, ldk);
    return patchify_generic_dispatch<__nv_bfloat16>(img, B, H, W, C, P, out, out_type, stream, rows_per_sample, ldk);
  }
  if (in_type == DT_F32) return patchify_dispatch<float>(img, B, H, W, C, P, out, out_type, stream, rows_per_sample);
  if (in_type == DT_F16) return patchify_dispatch<__half>(img, B, H, W, C, P, out, out_type, stream, rows_per_sample);
  return patchify_dispatch<__nv_bfloat16>(img, B, H, W, C, P, out, out_type, stream, rows_per_sample);
}

// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tokens_init_kernel(float4* __restrict__ x, const float4* __restrict__ cls, const float4* __restrict__ pos, size_t total4, int SD4, int D4) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int r = static_cast<int>(i % SD4);  // position inside the sample
  float4 v = __ldg(pos + r);
  if (cls != nullptr && r < D4) {
    const float4 c = __ldg(cls + r);
    v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w;
  }
  x[i] = v;
}
int tokens_init_run(float* x, const float* cls, const float* pos, int B, int S, int D, cudaStream_t stream) {
  if (B <= 0) return 0;
  if (D % 4 != 0) { set_last_error("tokens_init: D must be a multiple of 4"); return -1; }
  const size_t total4 = static_cast<size_t>(B) * S * D / 4;
  tokens_init_kernel<<<static_cast<unsigned>((total4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(cls),
                                                                                         reinterpret_cast<const float4*>(pos), total4, S * D / 4, D / 4);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// Bicubic resampling of the position table (torch.nn.functional.interpolate(mode="bicubic", align_corners=False), the operation
// HF's interpolate_pos_encoding applies): source index and Keys' cubic weights (A = -0.75) of output index `dst` along an axis
// of `in` -> `out` samples, with PyTorch's float operations in PyTorch's order.  The _rn intrinsics keep nvcc from contracting them
// into FMAs.  At out == in the weights are exactly (0, 1, 0, 0).
__device__ __forceinline__ void bicubic_taps(int in, int out, int dst, int (&idx)[4], float (&w)[4]) {
  const float scale = static_cast<float>(in) / static_cast<float>(out);
  const float real = __fsub_rn(__fmul_rn(scale, __fadd_rn(static_cast<float>(dst), 0.5f)), 0.5f);
  const int i0 = min(static_cast<int>(floorf(real)), in - 1);
  const float t = fminf(fmaxf(__fsub_rn(real, static_cast<float>(i0)), 0.f), 1.f);
  constexpr float A = -0.75f;
  auto cc1 = [](float x) { return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, x), A + 3.f), x), x), 1.f); };
  auto cc2 = [](float x) {
    return __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x), 5.f * A), x), 8.f * A), x), 4.f * A);
  };
  const float u = __fsub_rn(1.f, t);
  w[0] = cc2(__fadd_rn(t, 1.f));
  w[1] = cc1(t);
  w[2] = cc1(u);
  w[3] = cc2(__fadd_rn(u, 1.f));
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = max(min(i0 - 1 + k, in - 1), 0);
}

// Antialiased bilinear resampling (torch.nn.functional.interpolate(mode="bilinear", align_corners=False, antialias=True), the operation
// SigLIP 2 NaFlex applies to its position table; PyTorch's _upsample_bilinear2d_aa weight rule) along an axis of `in` -> `out` samples:
// output index `dst` reads taps i0 .. i1 - 1, each weighted by the triangle filter stretched by max(scale, 1) and normalised by the sum.
// Downscaling reads up to `in` taps (all of them for out = 1).  At out == in the taps are (dst, dst + 1) with weights exactly (1, 0).
struct AaAxis {
  int i0, i1;
  float center, invscale, total;
  __device__ __forceinline__ float raw(int j) const {
    const float x = fabsf(__fmul_rn(__fadd_rn(__fsub_rn(static_cast<float>(j), center), 0.5f), invscale));
    return x < 1.f ? __fsub_rn(1.f, x) : 0.f;
  }
  __device__ __forceinline__ float weight(int j) const { return __fdiv_rn(raw(j), total); }
};
__device__ __forceinline__ AaAxis aa_axis(int in, int out, int dst) {
  AaAxis a;
  const float scale = __fdiv_rn(static_cast<float>(in), static_cast<float>(out));
  const float support = scale >= 1.f ? scale : 1.f;
  a.invscale = scale >= 1.f ? __fdiv_rn(1.f, scale) : 1.f;
  a.center = __fmul_rn(scale, __fadd_rn(static_cast<float>(dst), 0.5f));
  a.i0 = max(static_cast<int>(__fadd_rn(__fsub_rn(a.center, support), 0.5f)), 0);
  a.i1 = min(static_cast<int>(__fadd_rn(__fadd_rn(a.center, support), 0.5f)), in);
  a.total = 0.f;
  for (int j = a.i0; j < a.i1; ++j) a.total = __fadd_rn(a.total, a.raw(j));
  return a;
}

__device__ __forceinline__ float4 mul4(float4 p, float w) { return make_float4(__fmul_rn(p.x, w), __fmul_rn(p.y, w), __fmul_rn(p.z, w), __fmul_rn(p.w, w)); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w)); }

// Row r of the initial residual stream of a gh x gw grid, columns 4 c .. 4 c + 3: cls + pos[0] for the CLS row (cls != null), else
// the resampling (Mode: bicubic or antialiased bilinear) of pos's g x g patch rows.
template <int Mode>
__device__ __forceinline__ float4 interp_token(const float4* __restrict__ cls, const float4* __restrict__ pos, int g, int D4, int gh, int gw, int r,
                                               int c) {
  const int off = cls != nullptr ? 1 : 0;
  float4 v;
  if (r < off) {
    const float4 a = __ldg(pos + c), b = __ldg(cls + c);
    v = make_float4(b.x + a.x, b.y + a.y, b.z + a.z, b.w + a.w);
  } else if (Mode == POS_BILINEAR_AA) {
    const int q = r - off, gy = q / gw, gx = q - gy * gw;
    const AaAxis ay = aa_axis(g, gh, gy), ax = aa_axis(g, gw, gx);
    const float4* src = pos + static_cast<size_t>(off) * D4 + c;
    // sum over rows of (sum over columns of tap * wx) * wy, each sum in tap order: PyTorch's separable accumulation.  Zero-weight taps
    // are skipped (each sum starts at its first weighted tap), so the (g, g) resample returns the table itself.
    bool first_row = true;
    for (int a = ay.i0; a < ay.i1; ++a) {
      const float wy = ay.weight(a);
      if (wy == 0.f) continue;
      const float4* row = src + static_cast<size_t>(a) * g * D4;
      float4 h = make_float4(0.f, 0.f, 0.f, 0.f);
      bool first_col = true;
      for (int b = ax.i0; b < ax.i1; ++b) {
        const float wx = ax.weight(b);
        if (wx == 0.f) continue;
        const float4 t = mul4(__ldg(row + static_cast<size_t>(b) * D4), wx);
        h = first_col ? t : add4(h, t);
        first_col = false;
      }
      v = first_row ? mul4(h, wy) : add4(v, mul4(h, wy));
      first_row = false;
    }
  } else {
    const int q = r - off, gy = q / gw, gx = q - gy * gw;
    int iy[4], ix[4];
    float wy[4], wx[4];
    bicubic_taps(g, gh, gy, iy, wy);
    bicubic_taps(g, gw, gx, ix, wx);
    const float4* src = pos + static_cast<size_t>(off) * D4 + c;
    // sum over rows of (sum over columns of tap * wx) * wy, each sum in tap order: PyTorch's separable accumulation
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const float4* row = src + static_cast<size_t>(iy[a]) * g * D4;
      float4 h = __ldg(row + static_cast<size_t>(ix[0]) * D4);
      h = make_float4(__fmul_rn(h.x, wx[0]), __fmul_rn(h.y, wx[0]), __fmul_rn(h.z, wx[0]), __fmul_rn(h.w, wx[0]));
#pragma unroll
      for (int b = 1; b < 4; ++b) {
        const float4 p = __ldg(row + static_cast<size_t>(ix[b]) * D4);
        h.x = __fadd_rn(h.x, __fmul_rn(p.x, wx[b])); h.y = __fadd_rn(h.y, __fmul_rn(p.y, wx[b]));
        h.z = __fadd_rn(h.z, __fmul_rn(p.z, wx[b])); h.w = __fadd_rn(h.w, __fmul_rn(p.w, wx[b]));
      }
      if (a == 0) {
        v = make_float4(__fmul_rn(h.x, wy[0]), __fmul_rn(h.y, wy[0]), __fmul_rn(h.z, wy[0]), __fmul_rn(h.w, wy[0]));
      } else {
        v.x = __fadd_rn(v.x, __fmul_rn(h.x, wy[a])); v.y = __fadd_rn(v.y, __fmul_rn(h.y, wy[a]));
        v.z = __fadd_rn(v.z, __fmul_rn(h.z, wy[a])); v.w = __fadd_rn(v.w, __fmul_rn(h.w, wy[a]));
      }
    }
  }
  return v;
}

// One thread per (token r, 4 columns): the value is the same for every sample, so it is computed once and stored B times.
template <int Mode>
__global__ void __launch_bounds__(256)
tokens_init_interp_kernel(float4* __restrict__ x, const float4* __restrict__ cls, const float4* __restrict__ pos, int g, int D4, int B,
                          int gh, int gw, int S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * D4) return;
  const int r = i / D4, c = i - r * D4;
  const float4 v = interp_token<Mode>(cls, pos, g, D4, gh, gw, r, c);
  const size_t SD4 = static_cast<size_t>(S) * D4;
  for (int b = 0; b < B; ++b) x[b * SD4 + i] = v;
}

// blockIdx.y = image; one thread per (token r of the image, 4 columns)
template <int Mode>
__global__ void __launch_bounds__(256)
tokens_add_interp_packed_kernel(float4* __restrict__ x, const float4* __restrict__ cls, const float4* __restrict__ pos, int g, int D4,
                                const int* __restrict__ seq_off, const int* __restrict__ gw_of) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const int row0 = seq_off[b], S = seq_off[b + 1] - row0;
  if (i >= S * D4) return;
  const int r = i / D4, c = i - r * D4;
  const int gw = gw_of[b], gh = (S - (cls != nullptr ? 1 : 0)) / gw;
  const float4 v = interp_token<Mode>(cls, pos, g, D4, gh, gw, r, c);
  float4* dst = x + static_cast<size_t>(row0) * D4 + i;
  if (cls != nullptr && r == 0) {
    *dst = v;
  } else {  // table + embedding: the per-image path reduce-adds the embedding onto the table, and fp32 addition commutes
    const float4 e = *dst;
    *dst = make_float4(v.x + e.x, v.y + e.y, v.z + e.z, v.w + e.w);
  }
}

static int check_interp_mode(const char* fn, int mode) {
  if (mode != POS_BICUBIC && mode != POS_BILINEAR_AA) { set_last_error("%s: bad resampling mode %d", fn, mode); return -1; }
  return 0;
}

int tokens_add_interp_packed_run(float* x, const float* cls, const float* pos, int g, int D, const int* seq_off, const int* gw, int B, int max_S,
                                 int mode, cudaStream_t stream) {
  if (B <= 0) return 0;
  if (check_interp_mode("tokens_add_interp_packed", mode)) return -1;
  if (D % 4 != 0) { set_last_error("tokens_add_interp_packed: D must be a multiple of 4"); return -1; }
  if (B > 65535) { set_last_error("tokens_add_interp_packed: %d images exceed the grid", B); return -1; }
  const int D4 = D / 4, n = max_S * D4;
  const dim3 grid((n + 255) / 256, B);
  auto kernel = mode == POS_BILINEAR_AA ? tokens_add_interp_packed_kernel<POS_BILINEAR_AA> : tokens_add_interp_packed_kernel<POS_BICUBIC>;
  kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(cls), reinterpret_cast<const float4*>(pos), g, D4,
                                   seq_off, gw);
  JIMM_LAUNCH_CHECK();
  return 0;
}

int tokens_init_interp_run(float* x, const float* cls, const float* pos, int g, int D, int B, int gh, int gw, int mode, cudaStream_t stream) {
  if (B <= 0) return 0;
  if (check_interp_mode("tokens_init_interp", mode)) return -1;
  if (D % 4 != 0) { set_last_error("tokens_init_interp: D must be a multiple of 4"); return -1; }
  if (g <= 0 || gh <= 0 || gw <= 0) { set_last_error("tokens_init_interp: empty grid (g=%d, output %dx%d)", g, gh, gw); return -1; }
  const int S = gh * gw + (cls != nullptr ? 1 : 0), D4 = D / 4;
  const int n = S * D4;
  auto kernel = mode == POS_BILINEAR_AA ? tokens_init_interp_kernel<POS_BILINEAR_AA> : tokens_init_interp_kernel<POS_BICUBIC>;
  kernel<<<(n + 255) / 256, 256, 0, stream>>>(reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(cls), reinterpret_cast<const float4*>(pos),
                                              g, D4, B, gh, gw, S);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// Patch rows of the HuggingFace NaFlex processor ([B, N, K] pixel_values, sample b's first n_b rows valid) into the packed patch-GEMM
// operand: blockIdx.y = sample, one thread per (row, column) of its n_b = seq_off[b + 1] - seq_off[b] rows; columns K .. ldk - 1 are zeros.
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
patch_rows_packed_kernel(const InT* __restrict__ pv, OutT* __restrict__ out, const int* __restrict__ seq_off, int N, int K, int ldk) {
  const int b = blockIdx.y;
  const int row0 = seq_off[b];
  const size_t total = static_cast<size_t>(seq_off[b + 1] - row0) * ldk;
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int r = static_cast<int>(i / ldk), k = static_cast<int>(i % ldk);
  const float v = k < K ? to_float(pv[(static_cast<size_t>(b) * N + r) * K + k]) : 0.f;
  out[static_cast<size_t>(row0 + r) * ldk + k] = from_float<OutT>(v);
}

template <typename InT>
static void patch_rows_packed_launch(const void* pv, void* out, int out_type, const int* seq_off, int B, int max_rows, int N, int K, int ldk,
                                     cudaStream_t stream) {
  const dim3 grid(static_cast<unsigned>((static_cast<size_t>(max_rows) * ldk + 255) / 256), B);
  const InT* in = static_cast<const InT*>(pv);
  if (out_type == DT_F32) patch_rows_packed_kernel<InT, float><<<grid, 256, 0, stream>>>(in, static_cast<float*>(out), seq_off, N, K, ldk);
  else if (out_type == DT_TF32) patch_rows_packed_kernel<InT, tf32_t><<<grid, 256, 0, stream>>>(in, static_cast<tf32_t*>(out), seq_off, N, K, ldk);
  else if (out_type == DT_F16) patch_rows_packed_kernel<InT, __half><<<grid, 256, 0, stream>>>(in, static_cast<__half*>(out), seq_off, N, K, ldk);
  else patch_rows_packed_kernel<InT, __nv_bfloat16><<<grid, 256, 0, stream>>>(in, static_cast<__nv_bfloat16*>(out), seq_off, N, K, ldk);
}

int patch_rows_packed_run(const void* pv, int in_type, int N, int K, const int* seq_off, int B, int max_rows, void* out, int out_type, int ldk,
                          cudaStream_t stream) {
  if (B <= 0 || max_rows <= 0) return 0;
  if (in_type < DT_F32 || in_type > DT_BF16 || out_type < DT_F32 || out_type > DT_TF32) {
    set_last_error("patch_rows_packed: bad type codes (in %d, out %d)", in_type, out_type);
    return -1;
  }
  if (K <= 0 || ldk < K || max_rows > N) { set_last_error("patch_rows_packed: bad shape (N %d, K %d, ldk %d, max_rows %d)", N, K, ldk, max_rows); return -1; }
  if (B > 65535) { set_last_error("patch_rows_packed: %d samples exceed the grid", B); return -1; }
  if (in_type == DT_F32) patch_rows_packed_launch<float>(pv, out, out_type, seq_off, B, max_rows, N, K, ldk, stream);
  else if (in_type == DT_F16) patch_rows_packed_launch<__half>(pv, out, out_type, seq_off, B, max_rows, N, K, ldk, stream);
  else patch_rows_packed_launch<__nv_bfloat16>(pv, out, out_type, seq_off, B, max_rows, N, K, ldk, stream);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
__global__ void cls_row_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos, int B, size_t SD, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * D) return;
  const int b = i / D, d = i - b * D;
  x[static_cast<size_t>(b) * SD + d] = cls[d] + pos[d];
}
int cls_row_run(float* x, const float* cls, const float* pos, int B, int S, int D, cudaStream_t stream) {
  if (B <= 0) return 0;
  const int n = B * D;
  cls_row_kernel<<<(n + 255) / 256, 256, 0, stream>>>(x, cls, pos, B, static_cast<size_t>(S) * D, D);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// x[r, :] = table[clamp(ids[r]), :] + pos[t, :] by one warp
__device__ __forceinline__ void embed_row(const int32_t* __restrict__ ids, const float* __restrict__ table, const float* __restrict__ pos,
                                          float* __restrict__ x, int r, int t, int D4, int vocab, int lane) {
  int id = ids[r];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);  // jnp take clamps out-of-range indices
  const float4* e = reinterpret_cast<const float4*>(table) + static_cast<size_t>(id) * D4;
  const float4* p = reinterpret_cast<const float4*>(pos) + static_cast<size_t>(t) * D4;
  float4* o = reinterpret_cast<float4*>(x) + static_cast<size_t>(r) * D4;
  for (int i = lane; i < D4; i += 32) {
    const float4 a = __ldg(e + i), b = __ldg(p + i);
    o[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

__global__ void __launch_bounds__(256)
embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table, const float* __restrict__ pos, float* __restrict__ x,
             int rows, int T, int D4, int vocab) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  embed_row(ids, table, pos, x, warp, warp % T, D4, vocab, lane);
}
int embed_run(const int32_t* ids, const float* table, const float* pos, float* x, int B, int T, int D, int vocab, cudaStream_t stream) {
  if (D % 4 != 0) { set_last_error("embed: D must be a multiple of 4"); return -1; }
  const int rows = B * T;
  if (rows <= 0) return 0;
  embed_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(ids, table, pos, x, rows, T, D / 4, vocab);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// one warp per row; the row's sequence is the last b with seq_off[b] <= row (binary search over the B + 1 offsets)
__global__ void __launch_bounds__(256)
embed_packed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table, const float* __restrict__ pos, float* __restrict__ x,
                    const int* __restrict__ seq_off, int B, int rows, int D4, int vocab) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seq_off[mid] <= warp) lo = mid;
    else hi = mid - 1;
  }
  embed_row(ids, table, pos, x, warp, warp - seq_off[lo], D4, vocab, lane);
}
int embed_packed_run(const int32_t* ids, const float* table, const float* pos, float* x, const int* seq_off, int B, int rows, int D, int vocab,
                     cudaStream_t stream) {
  if (D % 4 != 0) { set_last_error("embed_packed: D must be a multiple of 4"); return -1; }
  if (B <= 0 || rows <= 0) return 0;
  if (!seq_off) { set_last_error("embed_packed: null seq_off"); return -1; }
  embed_packed_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(ids, table, pos, x, seq_off, B, rows, D / 4, vocab);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// first argmax of ids[0 .. T-1] by one warp: the largest id, the lowest position among equal ones
__device__ __forceinline__ int warp_argmax_ids(const int32_t* __restrict__ ids, int T, int lane) {
  int best = INT_MIN, bi = 0x7fffffff;
  for (int t = lane; t < T; t += 32) {
    const int v = ids[t];
    if (v > best) { best = v; bi = t; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, best, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  return bi;
}

__global__ void argmax_ids_kernel(const int32_t* __restrict__ ids, int* __restrict__ idx, int B, int T) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const int bi = warp_argmax_ids(ids + static_cast<size_t>(warp) * T, T, lane);
  if (lane == 0) idx[warp] = bi;
}
int argmax_ids_run(const int32_t* ids, int* idx, int B, int T, cudaStream_t stream) {
  if (B <= 0) return 0;
  argmax_ids_kernel<<<(B + 7) / 8, 256, 0, stream>>>(ids, idx, B, T);
  JIMM_LAUNCH_CHECK();
  return 0;
}

__global__ void argmax_ids_packed_kernel(const int32_t* __restrict__ ids, const int* __restrict__ seq_off, int* __restrict__ row, int B) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const int r0 = seq_off[warp];
  const int bi = warp_argmax_ids(ids + r0, seq_off[warp + 1] - r0, lane);
  if (lane == 0) row[warp] = r0 + bi;
}
int argmax_ids_packed_run(const int32_t* ids, const int* seq_off, int* row, int B, cudaStream_t stream) {
  if (B <= 0) return 0;
  argmax_ids_packed_kernel<<<(B + 7) / 8, 256, 0, stream>>>(ids, seq_off, row, B);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
__global__ void l2_normalize_kernel(const float* __restrict__ x, float* __restrict__ out, size_t ldo, int B, int E) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const float* r = x + static_cast<size_t>(warp) * E;
  float s = 0.f;
  for (int i = lane; i < E; i += 32) s += r[i] * r[i];
  s = warp_sum(s);
  const float n = sqrtf(s);
  for (int i = lane; i < E; i += 32) out[static_cast<size_t>(warp) * ldo + i] = r[i] / n;
}
int l2_normalize_run(const float* x, float* out, int ldo, int B, int E, cudaStream_t stream) {
  if (B <= 0) return 0;
  l2_normalize_kernel<<<(B + 7) / 8, 256, 0, stream>>>(x, out, ldo, B, E);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// fp32 logits: 64x64 tile per CTA, 16x16 threads, 4x4 micro-tile, K step 16.  Full fp32 FMA (no tensor cores):
// 2*B^2*E is micro-seconds of work and the parity budget is spent elsewhere.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
logits_kernel(const float* __restrict__ img, const float* __restrict__ txt, const float* __restrict__ logit_scale,
              const float* __restrict__ logit_bias, float* __restrict__ out, int Bi, int Bt, int E, size_t ldl) {
  __shared__ __align__(16) float As[16][LOGITS_LDS], Bs[16][LOGITS_LDS];
  const float sc = expf(*logit_scale);
  const float bs = logit_bias ? *logit_bias : 0.f;
  logits_tile<false>(img, E, txt, E, out, ldl, Bi, Bt, E, blockIdx.y * 64, blockIdx.x * 64, sc, bs, As, Bs);
}
int logits_run(const float* img, const float* txt, const float* logit_scale, const float* logit_bias, float* logits, int Bi, int Bt,
               int E, int ldl, cudaStream_t stream) {
  if (Bi <= 0 || Bt <= 0) return 0;
  dim3 grid((Bt + 63) / 64, (Bi + 63) / 64);
  logits_kernel<<<grid, 256, 0, stream>>>(img, txt, logit_scale, logit_bias, logits, Bi, Bt, E, ldl);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// weight packing (runs once at finalize)
// ------------------------------------------------------------------------------------------
template <typename OutT>
__global__ void transpose_cast_kernel(const float* __restrict__ src, int K, int N, OutT* __restrict__ dst, size_t ldd) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? src[static_cast<size_t>(k) * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K) dst[static_cast<size_t>(n) * ldd + k] = from_float<OutT>(tile[threadIdx.x][i]);
  }
}
int transpose_cast_run(const float* src, int K, int N, void* dst, int out_type, int ldd, cudaStream_t stream) {
  dim3 block(32, 8), grid((N + 31) / 32, (K + 31) / 32);
  if (out_type == DT_F32) transpose_cast_kernel<float><<<grid, block, 0, stream>>>(src, K, N, static_cast<float*>(dst), ldd);
  else if (out_type == DT_TF32) transpose_cast_kernel<tf32_t><<<grid, block, 0, stream>>>(src, K, N, static_cast<tf32_t*>(dst), ldd);
  else if (out_type == DT_F16) transpose_cast_kernel<__half><<<grid, block, 0, stream>>>(src, K, N, static_cast<__half*>(dst), ldd);
  else transpose_cast_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>(src, K, N, static_cast<__nv_bfloat16*>(dst), ldd);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// FP8 weight quantiser (finalize): one warp per row of K fp32 values; K, lds, ldo multiples of 4.
__global__ void __launch_bounds__(256)
quantize_rows_e4m3_kernel(const float* __restrict__ src, size_t lds, int rows, int K4, uint32_t* __restrict__ out, size_t ldo4,
                          float* __restrict__ row_scale) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float4* r = reinterpret_cast<const float4*>(src + static_cast<size_t>(warp) * lds);
  float amax = 0.f;
  for (int i = lane; i < K4; i += 32) {
    const float4 v = r[i];
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  const int k = e4m3_scale_exp(warp_max(amax));
  const float inv_s = ldexpf(1.0f, -k);
  if (lane == 0) row_scale[warp] = ldexpf(1.0f, k);
  uint32_t* o = out + static_cast<size_t>(warp) * ldo4;
  for (int i = lane; i < K4; i += 32) {
    const float4 v = r[i];
    o[i] = e4m3x4_rn(v.x * inv_s, v.y * inv_s, v.z * inv_s, v.w * inv_s);
  }
}
int quantize_rows_e4m3_run(const float* src, int lds, int rows, int K, void* out, int ldo, float* row_scale, cudaStream_t stream) {
  if (K <= 0 || K % 4 != 0 || lds % 4 != 0 || ldo % 4 != 0 || lds < K || ldo < K) {
    set_last_error("quantize_rows_e4m3: K=%d, lds=%d and ldo=%d must be multiples of 4 with lds, ldo >= K", K, lds, ldo);
    return -1;
  }
  if (rows <= 0) return 0;
  quantize_rows_e4m3_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(src, lds, rows, K / 4, static_cast<uint32_t*>(out), ldo / 4, row_scale);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// standalone activation (API parity for jimm.common.transformer.quickgelu; inside the towers the activation is the FC1 epilogue)
__global__ void activation_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, int act) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) y[i] = act == 2 ? quick_gelu(x[i]) : (act == 1 ? gelu_tanh(x[i]) : x[i]);
}
int activation_run(const float* x, float* y, size_t n, int act, cudaStream_t stream) {
  if (n == 0) return 0;
  activation_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(x, y, n, act);
  JIMM_LAUNCH_CHECK();
  return 0;
}

template <typename OutT>
__global__ void cast_kernel(const float* __restrict__ src, OutT* __restrict__ dst, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = from_float<OutT>(src[i]);
}
int cast_run(const float* src, void* dst, int out_type, size_t n, cudaStream_t stream) {
  if (n == 0) return 0;
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  if (out_type == DT_F32) cast_kernel<float><<<grid, 256, 0, stream>>>(src, static_cast<float*>(dst), n);
  else if (out_type == DT_TF32) cast_kernel<tf32_t><<<grid, 256, 0, stream>>>(src, static_cast<tf32_t*>(dst), n);
  else if (out_type == DT_F16) cast_kernel<__half><<<grid, 256, 0, stream>>>(src, static_cast<__half*>(dst), n);
  else cast_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(src, static_cast<__nv_bfloat16*>(dst), n);
  JIMM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// Per-token hidden states: fp32 residual-stream rows -> the caller's buffer.  Each thread moves 8 elements per step (two 16-byte
// loads; one 16-byte store for 16-bit outputs, two for fp32).  Launched with PDL between two encoder blocks, so it waits for the
// previous block's FC2 reduce-add before it reads x -- every thread, before any exit, so the kernel never completes ahead of its
// producer.
// ------------------------------------------------------------------------------------------
template <typename OutT>
__global__ void __launch_bounds__(256)
tokens_out_kernel(const float4* __restrict__ x, OutT* __restrict__ out, size_t n8) {
  pdl_launch_dependents();
  pdl_wait();
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 a = x[2 * i], b = x[2 * i + 1];
    if constexpr (sizeof(OutT) == 4) {
      reinterpret_cast<float4*>(out)[2 * i] = a;
      reinterpret_cast<float4*>(out)[2 * i + 1] = b;
    } else {
      constexpr int ot = std::is_same<OutT, __half>::value ? 1 : 2;
      uint4 p;
      p.x = pack2(a.x, a.y, ot);
      p.y = pack2(a.z, a.w, ot);
      p.z = pack2(b.x, b.y, ot);
      p.w = pack2(b.z, b.w, ot);
      reinterpret_cast<uint4*>(out)[i] = p;
    }
  }
}

int tokens_out_run(const float* x, size_t rows, int D, void* out, int out_type, cudaStream_t stream) {
  if (D <= 0 || D % 8 != 0 || (out_type != DT_F32 && out_type != DT_F16 && out_type != DT_BF16)) {
    set_last_error("tokens_out: D=%d must be a positive multiple of 8 and the output type fp32 / fp16 / bf16 (got %d)", D, out_type);
    return -1;
  }
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) % 16 != 0) {
    set_last_error("tokens_out: x and out must be 16-byte aligned");
    return -1;
  }
  if (rows == 0) return 0;
  const size_t n8 = rows * static_cast<size_t>(D) / 8;
  const unsigned grid = static_cast<unsigned>(std::min<size_t>((n8 + 255) / 256, static_cast<size_t>(device_sm_count()) * 8));
  const float4* x4 = reinterpret_cast<const float4*>(x);
  if (out_type == DT_F32) JIMM_CUDA_CHECK(launch_k(tokens_out_kernel<float>, dim3(grid), dim3(256), 0, stream, 1, true, x4, static_cast<float*>(out), n8));
  else if (out_type == DT_F16) JIMM_CUDA_CHECK(launch_k(tokens_out_kernel<__half>, dim3(grid), dim3(256), 0, stream, 1, true, x4, static_cast<__half*>(out), n8));
  else JIMM_CUDA_CHECK(launch_k(tokens_out_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, stream, 1, true, x4, static_cast<__nv_bfloat16*>(out), n8));
  note_launch();
  return 0;
}

}  // namespace jimm
