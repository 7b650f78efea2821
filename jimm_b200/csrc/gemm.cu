// Persistent, warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   C[M,N] = epi( A[M,K] . B[N,K]^T ),  A/B K-major fp16 | bf16 | fp32(tf32) | e4m3, fp32 accumulate in registers.
//
// One kernel, gemm_wgmma_kernel<T, OUT, ACT>, with two K-slab bodies: m64n256 wgmmas accumulating straight into registers (16-bit,
// tf32), and for e4m3 (FP8 compute mode) 64 x 256 tiles whose slabs are summed from zero and promoted into fp32 registers, with row /
// column scales in the epilogue (see "e4m3 operands" below).
//
// CTA = 384 threads (three warpgroups), 1 CTA / SM, grid = min(#tiles, #SMs), static round-robin 128 x 256 tile schedule (n fastest).
//   warpgroup 0, warp 0 : TMA producer (one lane): 4-stage smem ring of {A 128x128B, B 256x128B} tiles (48 KB), SWIZZLE_128B
//   warpgroup 0, warps 1-3: idle, or LayerNorm workers of the fused-LayerNorm epilogue
//   warpgroups 1, 2     : consumers, 64 rows each (e4m3: 128 columns each): wgmma.mma_async from shared memory, one wgmma group in
//                         flight while the previous stage is released; then the epilogue straight from the accumulator registers.
//                         While they run it, the producer is already filling the ring for their next tile.
// 128 x 256 rather than 128 x 128: a k-slab of 128 B fills (128 + 256) x 128 B of shared memory from L2 for 2 x 128 x 256 x 64 FLOP
// (fp16), 85 FLOP per byte instead of 64, and the two consumer warpgroups read one B slab per 2 x 64 x 256 instead of 2 x 64 x 128
// outputs.  The 128 fp32 accumulators per consumer thread do not fit in the 168 registers each of 384 threads starts with, so the
// warpgroups trade registers with setmaxnreg (PRODUCER_REGS / CONSUMER_REGS below).
// Two mbarrier arrays: smem full (TMA transaction bytes) / empty (one arrive per consumer warp).
//
// Epilogues are compile-time specialised (a run-time branch on dtype / activation inside the unrolled loops costs registers and
// instruction-cache misses):
//   OUT_H16 / OUT_BF16 / OUT_TF32 / OUT_F32 + ACT {none, tanh-GELU, QuickGELU}: each warp packs its 16 rows into 16 x 128 B
//       swizzled boxes in smem (double-buffered) and stores them with cp.async.bulk.tensor (bounds clipped by the tensor map).
//   OUT_F32_ADD: the fp32 residual stream x += acc + bias through cp.reduce.async.bulk.tensor .add (done in L2; the SM
//       never reads the residual).
//   OUT_GENERIC: everything else (position-embedding row-add + row remap of the patch GEMM, heads with unaligned N,
//       fp32 stores to caller buffers): LSU stores from the registers, run-time flags.
//   OUT_SCREEN: the gallery index's screen (fp16 only): no output, each (row, column) whose score may reach the row's threshold is
//       appended to the row's candidate list (see "screening epilogue").
//
// Reference ops served (SURVEY.md 8a): a1 patch-embed conv-as-GEMM (common/vit.py:153-165,228-236),
// a4 fused q/k/v projections (common/transformer.py:67-79), a6 out-proj + residual (:130),
// a7 MLP (:90-114,131), a9 MAP-head linears (common/vit.py:42-85), a10 classifier / projections
// (models/vit.py:81-89, models/clip.py:82-90,166, models/siglip.py:111-119).
#include "gemm.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"

namespace jimm {

static constexpr int BM = GEMM_TILE_M;  // two consumer warpgroups x 64 rows
static constexpr int BN = GEMM_TILE_N;  // one m64n256 wgmma per consumer warpgroup and K step
static_assert(BM == 128 && BN == 256, "the warp roles and the wgmma shape below are written for 128 x 256 tiles");
static constexpr int STAGES = 4;  // a 48 KB stage is 1024 tensor-core clocks of work (fp16)
static constexpr int A_STAGE_BYTES = BM * 128;
static constexpr int B_STAGE_BYTES = BN * 128;
static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
static constexpr int EPI_WARPS = 8;                                       // warps 4..11
static constexpr int EPI_BOX_ROWS = 16;                                   // one warp's rows of the tile
static constexpr int EPI_BUF_BYTES = EPI_BOX_ROWS * 128;                  // one 16-row x 128-byte swizzled TMA-store box
static constexpr int EPI_BUFS = 2;                                        // per warp: box i + 1 is packed while box i is stored
static constexpr int EPI_STAGE_BYTES = EPI_WARPS * EPI_BUFS * EPI_BUF_BYTES;  // 32 KB
static constexpr int NUM_THREADS = 384;
static constexpr int KERNEL_REGS = 168;  // per thread at launch: 64 K registers / 384 threads, in the allocation unit of 8

enum OutKind : int { OUT_GENERIC = 0, OUT_H16 = 1, OUT_BF16 = 2, OUT_TF32 = 3, OUT_F32_ADD = 4, OUT_F32 = 5, OUT_SCREEN = 6 };

struct EpiDev {
  const float* bias;
  const float* rowadd;
  const float* residual;
  void* out;
  int act, ldr, out_type, ldo, rows_in, rows_out, row_off, mode;
  int M, N;
  int reverse;
  int tok_pad, tok_off;  // > 0: 3-D token-scatter reduce-add (see GemmEpilogue)
  // fused LayerNorm of completed row groups (see GemmEpilogue)
  const float* ln_scale;
  const float* ln_bias;
  void* ln_out;
  int* ln_cnt;
  int ln_out_type, ln_ldo;
  float ln_eps;
  const float* a_scale;  // e4m3 operands: dequantisation scales (see GemmEpilogue)
  const float* b_scale;
  // OUT_SCREEN reads its GemmScreen from the fields above (gemm_screen_run): t = bias, nq = a_scale, ng = b_scale, cnt = ln_cnt,
  // list = out, cap = ldo.  The struct keeps its size, so every other kernel's parameters keep their offsets.
};

template <int ACT>
__device__ __forceinline__ float act_ct(float v) {
  if constexpr (ACT == ACT_GELU_TANH) return gelu_tanh(v);
  else if constexpr (ACT == ACT_QUICK_GELU) return quick_gelu(v);
  else return v;
}
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ACT_GELU_TANH) return gelu_tanh(v);
  if (act == ACT_QUICK_GELU) return quick_gelu(v);
  return v;
}

__device__ __forceinline__ void remap_row(const EpiDev& e, int row, int& out_row, int& add_row) {
  if (e.rows_in > 0) {
    int b = row / e.rows_in, p = row - b * e.rows_in;
    out_row = b * e.rows_out + p + e.row_off;
    add_row = p + e.row_off;
  } else {
    out_row = row;
    add_row = row;
  }
}

__device__ __forceinline__ void store1(const EpiDev& e, int out_row, int col, float v) {
  size_t off = static_cast<size_t>(out_row) * e.ldo + col;
  if (e.out_type == DT_F32) static_cast<float*>(e.out)[off] = v;
  else if (e.out_type == DT_TF32) static_cast<float*>(e.out)[off] = round_tf32(v);
  else if (e.out_type == DT_F16) static_cast<__half*>(e.out)[off] = __float2half_rn(v);
  else static_cast<__nv_bfloat16*>(e.out)[off] = __float2bfloat16_rn(v);
}

template <typename T>
struct Traits;  // DTYPE: the operand's DType; KIND: wgmma_m64n256_ss operand kind
template <>
struct Traits<__half> {
  static constexpr int DTYPE = DT_F16, KIND = 0;
};
template <>
struct Traits<__nv_bfloat16> {
  static constexpr int DTYPE = DT_BF16, KIND = 1;
};
template <>
struct Traits<float> {
  static constexpr int DTYPE = DT_TF32, KIND = 2;
};
template <>
struct Traits<__nv_fp8_e4m3> {
  static constexpr int DTYPE = DT_E4M3;
};
template <typename T>
constexpr bool kScaled = std::is_same<T, __nv_fp8_e4m3>::value;  // the accumulator is multiplied by a_scale[row] * b_scale[col]

// Rows of one CTA tile: e4m3 tiles are half height (see "e4m3 operands").  The kernel, the grid size and the A tensor map's box read it.
constexpr int tile_rows(int dtype) { return dtype == DT_E4M3 ? 64 : BM; }

// ---- fused LayerNorm of completed 32-row groups (reduce-add epilogue) --------------------------------------------------------------
// Who normalises: NOT the consumer warps, whose next tile would wait for them.  The consumer warps only PUBLISH (wait for their
// reduce-adds, bump the group's counter, and the one that completes a group pushes its index into a shared-memory ring); the producer
// warpgroup's otherwise idle warps 1-3 pop indices and normalise, off the MMA / epilogue critical path.  The rows are read back with
// ld.global.cg (they were just reduce-added in L2; L1 is bypassed) in batches whose loads are all issued back to back, double-buffered
// in registers.  Same arithmetic as layernorm_kernel (elementwise.cu): fp32, var = max(0, E[x^2] - E[x]^2).  NV = D / 128 float4 per
// lane per row.
static constexpr int ACT_FUSE_LN = 7;  // internal marker in the kernel's ACT slot (OUT_F32_ADD has no activation)
static constexpr int LNQ = 240;        // ring slots
struct LnQueue {
  int head, tail, done, pad;
  int slot[LNQ];  // -1 = empty, else a row-group index
};

template <typename OutT, int NV>
__device__ __forceinline__ void ln_rows_nv(const EpiDev& e, int row0, int lane) {
  constexpr int R0 = 8 / NV;
  constexpr int R = R0 < 1 ? 1 : R0;  // rows per batch: <= 8 float4 per lane per buffer (the LayerNorm warps hold PRODUCER_REGS)
  constexpr bool DOUBLE = NV <= 8;    // wider rows: one buffer (a row's loads still go out back to back)
  const float inv_d = 1.0f / static_cast<float>(NV * 128);
  const float4* sc = reinterpret_cast<const float4*>(e.ln_scale);
  const float4* bi = reinterpret_cast<const float4*>(e.ln_bias);
  const float* xbase = static_cast<const float*>(e.out);
  const int ldx = e.ldo, ldh = e.ln_ldo;
  const float eps = e.ln_eps;
  OutT* hbase = static_cast<OutT*>(e.ln_out);
  const int rows = min(32, e.M - row0);
  float4 a[R][NV];
  float4 b[DOUBLE ? R : 1][DOUBLE ? NV : 1];
#define JIMM_LN_LOAD(buf, r0_)                                                                                          \
  _Pragma("unroll") for (int i = 0; i < R; ++i) { /* unconditional (row clamped): the buffers stay in registers */     \
    const float4* xr = reinterpret_cast<const float4*>(xbase + static_cast<size_t>(row0 + min((r0_) + i, rows - 1)) * ldx); \
    _Pragma("unroll") for (int j = 0; j < NV; ++j) buf[i][j] = __ldcg(xr + lane + 32 * j);                              \
  }
#define JIMM_LN_PROCESS(buf, r0_)                                                                                       \
  _Pragma("unroll") for (int i = 0; i < R; ++i) {                                                                       \
    if ((r0_) + i < rows) {                                                                                             \
      float s = 0.f, s2 = 0.f;                                                                                          \
      _Pragma("unroll") for (int j = 0; j < NV; ++j) {                                                                  \
        const float4 v = buf[i][j];                                                                                     \
        s += v.x + v.y + v.z + v.w;                                                                                     \
        s2 += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;                                                            \
      }                                                                                                                 \
      s = warp_sum(s);                                                                                                  \
      s2 = warp_sum(s2);                                                                                                \
      const float mean = s * inv_d;                                                                                     \
      const float rstd = rsqrtf(fmaxf(s2 * inv_d - mean * mean, 0.0f) + eps);                                           \
      OutT* orow = hbase + static_cast<size_t>(row0 + (r0_) + i) * ldh;                                                 \
      _Pragma("unroll") for (int j = 0; j < NV; ++j) {                                                                  \
        const int idx = lane + 32 * j;                                                                                  \
        const float4 v = buf[i][j], g = __ldg(sc + idx), bb = __ldg(bi + idx);                                          \
        float4 y;                                                                                                       \
        y.x = (v.x - mean) * rstd * g.x + bb.x;                                                                         \
        y.y = (v.y - mean) * rstd * g.y + bb.y;                                                                         \
        y.z = (v.z - mean) * rstd * g.z + bb.z;                                                                         \
        y.w = (v.w - mean) * rstd * g.w + bb.w;                                                                         \
        if constexpr (std::is_same<OutT, float>::value) {                                                               \
          reinterpret_cast<float4*>(orow)[idx] = make_float4(round_tf32(y.x), round_tf32(y.y), round_tf32(y.z), round_tf32(y.w)); \
        } else {                                                                                                        \
          uint2 pk;                                                                                                     \
          constexpr int ot = std::is_same<OutT, __half>::value ? DT_F16 : DT_BF16;                                      \
          pk.x = pack2(y.x, y.y, ot);                                                                                   \
          pk.y = pack2(y.z, y.w, ot);                                                                                   \
          reinterpret_cast<uint2*>(orow)[idx] = pk;                                                                     \
        }                                                                                                               \
      }                                                                                                                 \
    }                                                                                                                   \
  }
  if constexpr (DOUBLE) {
    JIMM_LN_LOAD(a, 0)
#pragma unroll 1
    for (int r0 = 0; r0 < rows; r0 += 2 * R) {
      JIMM_LN_LOAD(b, r0 + R)
      JIMM_LN_PROCESS(a, r0)
      JIMM_LN_LOAD(a, r0 + 2 * R)
      JIMM_LN_PROCESS(b, r0 + R)
    }
  } else {
#pragma unroll 1
    for (int r0 = 0; r0 < rows; r0 += R) {
      JIMM_LN_LOAD(a, r0)
      JIMM_LN_PROCESS(a, r0)
    }
  }
#undef JIMM_LN_LOAD
#undef JIMM_LN_PROCESS
}

// OutT = the GEMM's operand type (the normalised rows are the next GEMM's A operand; float = tf32-rounded fp32)
template <typename OutT>
__device__ __forceinline__ void ln_rows_dispatch(const EpiDev& e, int row0, int lane) {
  switch (e.N >> 7) {  // gemm_fuses_ln() admits exactly these widths
    case 1: ln_rows_nv<OutT, 1>(e, row0, lane); break;
    case 2: ln_rows_nv<OutT, 2>(e, row0, lane); break;
    case 3: ln_rows_nv<OutT, 3>(e, row0, lane); break;
    case 4: ln_rows_nv<OutT, 4>(e, row0, lane); break;
    case 6: ln_rows_nv<OutT, 6>(e, row0, lane); break;
    case 8: ln_rows_nv<OutT, 8>(e, row0, lane); break;
    case 9: ln_rows_nv<OutT, 9>(e, row0, lane); break;
    default: break;
  }
}

// Epilogue side (lane 0 of a consumer warp): this thread's reduce-adds of `cols` columns into its 16 rows of row group `rg` have been
// ISSUED; wait for their completion, publish, and if that completes the rows (all N columns of both 16-row halves added, by whichever
// CTAs handled the other column tiles) queue the group for this CTA's LayerNorm warps.
__device__ __forceinline__ void ln_publish(const EpiDev& e, LnQueue* q, int rg, int cols) {
  tma_store_wait_all();  // the bulk reduce-adds of this thread are complete (performed in L2) ...
  __threadfence();       // ... and ordered before the counter update (release; cumulative over what this thread observed)
  const int old = atomicAdd(e.ln_cnt + rg, cols);
  if (old + cols == 2 * e.N) {
    e.ln_cnt[rg] = 0;  // self-cleaning for the next launch
    __threadfence();   // acquire side: the other contributors' adds are ordered before the consumer's loads
    const int t = atomicAdd(&q->tail, 1);
    volatile int* s = &q->slot[t % LNQ];
    while (*s != -1) __nanosleep(64);  // ring full: the consumers always make progress
    *s = rg;
  }
}

// LayerNorm warp: pop row groups until every epilogue warp of this CTA has finished publishing and the ring is drained.
template <typename OutT>
__device__ __forceinline__ void ln_worker(const EpiDev& e, LnQueue* q, int lane) {
  for (;;) {
    int rg = -2;
    if (lane == 0) {
      const int t = atomicAdd(&q->head, 1);
      volatile int* s = &q->slot[t % LNQ];
      for (;;) {
        if (*s >= 0) {
          const int v = atomicExch(&q->slot[t % LNQ], -1);
          if (v >= 0) { rg = v; break; }
        }
        // `done` is bumped after a warp's last push (tail already final for that warp): once all have, tickets >= tail get nothing
        if (*reinterpret_cast<volatile int*>(&q->done) == EPI_WARPS && t >= *reinterpret_cast<volatile int*>(&q->tail)) break;
        __nanosleep(256);
      }
      __threadfence();
    }
    rg = __shfl_sync(0xffffffffu, rg, 0);
    if (rg < 0) return;
    ln_rows_dispatch<OutT>(e, rg * 32, lane);
  }
}

// ---- TMA epilogue of one consumer warp: its 16 rows x BN columns, thread (g = lane / 4, t = lane % 4) holds rows g and g + 8,
// columns 8 j + 2 t (+1) of the wgmma accumulator.  16-bit outputs: 64 columns per 16 x 128 B box; 32-bit outputs: 32 columns.
// NC: the warp's columns (BN, or 128 for e4m3), acc[NC / 2] its accumulators
template <int OUT, int ACT, bool SCALED, int NC>
__device__ __forceinline__ void epilogue_tma(const CUtensorMap* map_c, const EpiDev& epi, const float (&acc)[NC / 2], uint8_t* tbuf0, int lane,
                                             int row_base, int n_tile0, uint32_t& box_count) {
  constexpr bool OUT16 = (OUT == OUT_H16 || OUT == OUT_BF16);
  constexpr int ES = OUT16 ? 2 : 4;
  constexpr int COLS_PER_BOX = 128 / ES;
  constexpr int JB = COLS_PER_BOX / 8;  // accumulator n-blocks per box
  const int g = lane >> 2, t = lane & 3;
  float sa0 = 1.f, sa1 = 1.f;  // row scales of rows g and g + 8 (rows >= M of the last box read row M - 1's: never stored past the box)
  if constexpr (SCALED) {
    sa0 = __ldg(epi.a_scale + min(row_base + g, epi.M - 1));
    sa1 = __ldg(epi.a_scale + min(row_base + g + 8, epi.M - 1));
  }
#pragma unroll
  for (int s = 0; s < NC / COLS_PER_BOX; ++s) {
    const int n0 = n_tile0 + s * COLS_PER_BOX;
    if (n0 >= epi.N) break;
    uint8_t* tbuf = tbuf0 + (box_count & (EPI_BUFS - 1)) * EPI_BUF_BYTES;
    ++box_count;
    if (lane == 0) tma_store_wait_read1();  // the box that last used this buffer has been read out of smem
    __syncwarp();
#pragma unroll
    for (int jj = 0; jj < JB; ++jj) {
      const int j = s * JB + jj;
      const int col = n0 + jj * 8 + 2 * t;
      float2 b2 = make_float2(0.f, 0.f);
      if (epi.bias != nullptr && col < epi.N) b2 = __ldg(reinterpret_cast<const float2*>(epi.bias + col));
      float a0 = acc[4 * j], a1 = acc[4 * j + 1], a2 = acc[4 * j + 2], a3 = acc[4 * j + 3];
      if constexpr (SCALED) {  // products of two powers of two: exact, in any order
        float2 s2 = make_float2(0.f, 0.f);
        if (col < epi.N) s2 = __ldg(reinterpret_cast<const float2*>(epi.b_scale + col));
        a0 *= sa0 * s2.x; a1 *= sa0 * s2.y; a2 *= sa1 * s2.x; a3 *= sa1 * s2.y;
      }
      const float v0 = act_ct<ACT>(a0 + b2.x), v1 = act_ct<ACT>(a1 + b2.y);
      const float v2 = act_ct<ACT>(a2 + b2.x), v3 = act_ct<ACT>(a3 + b2.y);
      const int byte = (jj * 8 + 2 * t) * ES;
      // 128-byte swizzle: 16-byte chunk c of row r lives at chunk c ^ (r % 8); rows g and g + 8 share r % 8 = g
      const int off = ((((byte >> 4) ^ g)) << 4) + (byte & 15);
      uint8_t* p0 = tbuf + g * 128 + off;
      uint8_t* p1 = p0 + 8 * 128;
      if constexpr (OUT16) {
        *reinterpret_cast<uint32_t*>(p0) = pack2(v0, v1, OUT == OUT_H16 ? 1 : 2);
        *reinterpret_cast<uint32_t*>(p1) = pack2(v2, v3, OUT == OUT_H16 ? 1 : 2);
      } else if constexpr (OUT == OUT_TF32) {
        *reinterpret_cast<float2*>(p0) = make_float2(round_tf32(v0), round_tf32(v1));
        *reinterpret_cast<float2*>(p1) = make_float2(round_tf32(v2), round_tf32(v3));
      } else {
        *reinterpret_cast<float2*>(p0) = make_float2(v0, v1);
        *reinterpret_cast<float2*>(p1) = make_float2(v2, v3);
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      const uint32_t tbuf_u32 = smem_u32(tbuf);
      if constexpr (OUT == OUT_F32_ADD) {
        if (epi.tok_pad > 0) {
          const int b = row_base / epi.tok_pad;
          tma_reduce_add_3d(map_c, tbuf_u32, n0, row_base - b * epi.tok_pad + epi.tok_off, b);
        } else {
          tma_reduce_add_2d(map_c, tbuf_u32, n0, row_base);
        }
      } else {
        tma_store_2d(map_c, tbuf_u32, n0, row_base);
      }
      tma_store_commit();
    }
  }
}

// ---- generic LSU epilogue (run-time flags; any N, row remap, row-add, residual read) ---------------------------------
template <bool SCALED, int NC>
__device__ __forceinline__ void epilogue_generic(const EpiDev& epi, const float (&acc)[NC / 2], int lane, int row_base, int n_tile0) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row_base + g + 8 * h;
    if (row >= epi.M) continue;
    int out_row, add_row;
    remap_row(epi, row, out_row, add_row);
    float sa = 1.f;
    if constexpr (SCALED) sa = __ldg(epi.a_scale + row);
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) {
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int col = n_tile0 + 8 * j + 2 * t + q;
        if (col < epi.N) {
          float v = acc[4 * j + 2 * h + q];
          if constexpr (SCALED) v *= sa * __ldg(epi.b_scale + col);
          if (epi.bias) v += __ldg(epi.bias + col);
          v = apply_act(v, epi.act);
          if (epi.rowadd) v += __ldg(epi.rowadd + static_cast<size_t>(add_row) * epi.N + col);
          if (epi.residual) v += epi.residual[static_cast<size_t>(out_row) * epi.ldr + col];
          store1(epi, out_row, col, v);
        }
      }
    }
  }
}

// ---- screening epilogue of the gallery index (fp16 operands) ------------------------------------------------------------------------
// A row i is a normalised query q (fp32) rounded to fp16 as q^, B row j a normalised gallery row g rounded as g^; nq >= ||q||_2 and
// ng >= ||g||_2 are the index's norm bounds (+inf for a row with a non-finite value, whose fp16 copy is zeros).  The exact score's
// accumulator is acc = the fp32 fmaf chain of q_k g_k, k ascending (logits_tile); the screen holds a = the wgmma's sum of q^_k g^_k.
// delta >= |a - acc|, with u = 2^-11 (fp16 unit roundoff), s = 2^-25 sqrt(E) and E = K:
//   * the fp16 operands: q^_k = q_k (1 + e) + h with |e| <= u, |h| <= 2^-25 (half the fp16 subnormal step), likewise g^_k, so
//     |sum q^ g^ - sum q g| <= (2u + u^2) sum |q g| + (1 + 2u) 2^-25 (sum |q| + sum |g|) + E 2^-50
//                           <= (2u + u^2) nq ng + (1 + 2u) s (nq + ng) + E 2^-50              (Cauchy-Schwarz, sum |q| <= sqrt(E) ||q||);
//   * the fmaf chain, one rounding per step: |acc - sum q g| <= gamma_E sum |q g| <= gamma_E nq ng, gamma_E = E 2^-24 / (1 - E 2^-24);
//   * the tensor core's own accumulation, not assumed to be IEEE: |a - sum q^ g^| <= c_tc sum |q^ g^| <= c_tc nq^ ng^ with
//     nq^ = (1 + u) nq + s >= ||q^||, so <= c_tc ((1 + u)^2 nq ng + (1 + u) s (nq + ng) + s^2).  c_tc = E 2^-22; the GPU tests measure
//     the fp16 wgmma's accumulation against that constant on adversarial operands.
// So delta = c1 nq ng + c2 (nq + ng) + c3 with c1 = 2u + u^2 + gamma_E + c_tc (1 + u)^2, c2 = (1 + 2u) s + c_tc (1 + u) s and
// c3 = E 2^-50 + c_tc s^2, computed in double and rounded up by 2^-20 relative (screen_bound, gemm.cuh), which covers the
// four fp32 roundings of the expression below.  At E = 768: c1 = 1.2e-3.  Then acc >= t implies a + delta >= acc >= t, and
// fl(a + delta) >= t (t is a float, rounding is monotone): a row is dropped only if acc < t.  A non-finite bound makes delta +inf or
// NaN, and `!(a + delta < t)` keeps the row.
template <int NC>
__device__ __forceinline__ void epilogue_screen(const EpiDev& epi, const float (&acc)[NC / 2], int lane, int row_base, int n_tile0, int K) {
  const ScreenBound c = screen_bound(K);
  int* list = static_cast<int*>(epi.out);
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row_base + g + 8 * h;
    if (row >= epi.M) continue;
    const float t = __ldg(epi.bias + row), nq = __ldg(epi.a_scale + row);
    const float d0 = c.c1 * nq, d1 = c.c2 * nq + c.c3;
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) {
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int col = n_tile0 + 8 * j + 2 * t4 + q;
        if (col < epi.N) {
          const float ng = __ldg(epi.b_scale + col);
          const float delta = fmaf(d0, ng, fmaf(c.c2, ng, d1));
          if (!(acc[4 * j + 2 * h + q] + delta < t)) {
            const int pos = atomicAdd(epi.ln_cnt + row, 1);
            if (pos < epi.ldo) list[static_cast<size_t>(row) * epi.ldo + pos] = col;
          }
        }
      }
    }
  }
}

// ---- e4m3 operands ---------------------------------------------------------------------------------------------------------------
// The e4m3 wgmma does not accumulate in full fp32: its sums of products lose low-order bits (about 5e-4 of sum |a b| at K = 768..2048
// on an H100, measured with m64n256k32), which puts an FP8 model at about a third of its whole FP8 error away from an exact-accumulation
// restatement.  So each 128-deep K slab (four m64n128k32 wgmmas) is accumulated from zero and then added to fp32 registers ("promotion").
// The 64 promoted sums plus 64 accumulators per thread fit where m64n256 would need 256, so the CTA tile is 64 x 256: both consumer
// warpgroups take the same 64 A rows, warpgroup wg columns [128 wg, 128 wg + 128) of the B tile.  That is gemm_wgmma_kernel's e4m3
// slab body and tile split; the ring (A stages keep their 128-row spacing and hold 64 rows), barriers, register split, tile walk and
// epilogues are shared.  e4m3 plans take the plain-store epilogues only, never the fused LayerNorm.

template <typename T, int OUT, int ACT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const __grid_constant__ CUtensorMap map_c, const EpiDev epi, int K) {
  constexpr bool SCALED = kScaled<T>;  // e4m3: promoted K slabs, scaled epilogue
  constexpr int BK = 128 / sizeof(T);  // one 128-byte swizzle atom along K per stage
  constexpr int UK = 32 / sizeof(T);   // wgmma K (16 for 16-bit, 8 for tf32, 32 for e4m3)
  constexpr int TM = tile_rows(Traits<T>::DTYPE);
  constexpr int STAGE_TX = TM * 128 + B_STAGE_BYTES;  // bytes one stage's TMA loads bring
  // Consumer warpgroup wg's part of the tile starts wg * WG_DM rows and wg * WG_DN columns in: the 16-bit / tf32 tile is split by
  // rows, the e4m3 tile by columns.  Each consumer warp holds 16 rows x NC columns.
  constexpr int WG_DM = SCALED ? 0 : 64;
  constexpr int WG_DN = SCALED ? 128 : 0;
  constexpr int NC = BN - WG_DN;
  constexpr bool FUSE_LN = OUT == OUT_F32_ADD && ACT == ACT_FUSE_LN;  // see "fused LayerNorm" above
  constexpr int EPI_ACT = ACT == ACT_FUSE_LN ? static_cast<int>(ACT_NONE) : ACT;
  // Registers per thread of the producer warpgroup / of each consumer warpgroup after setmaxnreg.  The consumers hold 128
  // accumulators (e4m3: 64 plus 64 promoted sums); the producer's TMA lane needs few.  The fused LayerNorm's workers live in the
  // producer warpgroup and keep up to 64 registers of row data (ln_rows_nv) plus the scale / bias they load, while its consumers'
  // reduce-add epilogue is the leanest.
  // Chosen from ptxas -v: splits without spills.  The three warpgroups share the CTA's launch allocation of KERNEL_REGS per thread
  // (checked at launch).
  constexpr int PRODUCER_REGS = FUSE_LN ? 152 : 40;
  constexpr int CONSUMER_REGS = FUSE_LN ? 176 : 232;
  static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= NUM_THREADS * KERNEL_REGS, "register split exceeds the CTA's allocation");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* epi_stage = smem + STAGES * STAGE_BYTES;
  LnQueue* lnq = reinterpret_cast<LnQueue*>(epi_stage + EPI_STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(lnq + 1);  // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                     // [STAGES]

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int M = epi.M, N = epi.N;
  const int m_tiles = (M + TM - 1) / TM, n_tiles = (N + BN - 1) / BN;
  const int num_tiles = m_tiles * n_tiles;
  const int num_kb = (K + BK - 1) / BK;

  pdl_launch_dependents();
  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    if constexpr (OUT != OUT_GENERIC && OUT != OUT_SCREEN) tma_prefetch_desc(&map_c);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EPI_WARPS);
    }
    fence_barrier_init();
  }
  if constexpr (FUSE_LN) {
    if (warp_idx == 1) {
      for (int i = lane; i < LNQ; i += 32) lnq->slot[i] = -1;
      if (lane == 0) lnq->head = lnq->tail = lnq->done = 0;
    }
  }
  __syncthreads();
  pdl_wait();  // everything above (barrier init, descriptor prefetch) overlapped the previous kernel's tail

  if (warp_idx < 4) {
    setmaxnreg<KERNEL_REGS, PRODUCER_REGS>();
    if (warp_idx == 0) {
      // ===================== TMA producer =====================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          const int tv = epi.reverse ? num_tiles - 1 - tile : tile;
          const int m_blk = tv / n_tiles, n_blk = tv - m_blk * n_tiles;
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], STAGE_TX);
            tma_load_2d(smem_a + stage * A_STAGE_BYTES, &map_a, &full_bar[stage], kb * BK, m_blk * TM);
            tma_load_2d(smem_b + stage * B_STAGE_BYTES, &map_b, &full_bar[stage], kb * BK, n_blk * BN);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else if constexpr (FUSE_LN) {
      ln_worker<T>(epi, lnq, lane);
    }
  } else {
    // ===================== consumers: mainloop + epilogue =====================
    setmaxnreg<KERNEL_REGS, CONSUMER_REGS>();
    const int wg = (warp_idx - 4) >> 2;  // consumer warpgroup: rows [64 wg, 64 wg + 64) of the tile (e4m3: 128 columns)
    const int wq = warp_idx & 3;         // warp within the warpgroup: rows [16 wq, 16 wq + 16) of those
    uint8_t* tbuf0 = epi_stage + (warp_idx - 4) * EPI_BUFS * EPI_BUF_BYTES;
    int stage = 0;
    uint32_t phase = 0, box_count = 0;
    int ln_rg = -1, ln_cols = 0;  // row group / column count of this warp's previous tile, not yet published (fused LayerNorm)
    float acc[NC / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int tv = epi.reverse ? num_tiles - 1 - tile : tile;
      const int m_blk = tv / n_tiles, n_blk = tv - m_blk * n_tiles;
      int prev = -1;
      if constexpr (SCALED) {
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) acc[i] = 0.f;
      }
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = make_wgmma_desc_sw128(smem_u32(smem_a + stage * A_STAGE_BYTES + wg * WG_DM * 128));
        const uint64_t bdesc = make_wgmma_desc_sw128(smem_u32(smem_b + stage * B_STAGE_BYTES + wg * WG_DN * 128));
        if constexpr (SCALED) {
          // the slab's sum from zero; once its wgmmas have retired, the stage goes back to the producer and the sum is promoted
          float slab[NC / 2];
          wgmma_fence_operands(slab);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)  // descriptors advance by 32 bytes (>> 4) per wgmma K step
            wgmma_m64n128k32_e4m3_ss(slab, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k), k != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operands(slab);
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
          for (int i = 0; i < NC / 2; ++i) acc[i] += slab[i];
        } else {
          wgmma_fence_operands(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)  // descriptors advance by 32 bytes (>> 4) per wgmma K step
            wgmma_m64n256_ss<Traits<T>::KIND>(acc, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k), (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_fence_operands(acc);
          if (prev >= 0) {
            wgmma_wait<1>();  // the previous stage's wgmmas have retired: hand its smem back to the producer
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
          }
          prev = stage;
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if constexpr (!SCALED) {
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }

      const int row_base = m_blk * TM + wg * WG_DM + wq * 16;
      const int n_tile0 = n_blk * BN + wg * WG_DN;
      if constexpr (OUT == OUT_GENERIC) {
        epilogue_generic<SCALED, NC>(epi, acc, lane, row_base, n_tile0);
      } else if constexpr (OUT == OUT_SCREEN) {
        epilogue_screen<NC>(epi, acc, lane, row_base, n_tile0, K);
      } else {
        // split by columns, a consumer warpgroup's columns can lie wholly past N
        if (row_base < M && (WG_DN == 0 || n_tile0 < N))
          epilogue_tma<OUT, EPI_ACT, SCALED, NC>(&map_c, epi, acc, tbuf0, lane, row_base, n_tile0, box_count);
        if constexpr (FUSE_LN) {
          // Publishing is deferred by one tile: the PREVIOUS tile's reduce-adds were issued a whole mainloop ago, so waiting for them
          // costs nothing.  Both 16-row halves of a 32-row group publish, also a half that lies beyond M.
          if (lane == 0 && ln_rg >= 0) ln_publish(epi, lnq, ln_rg, ln_cols);
          ln_rg = (row_base & ~31) < M ? row_base >> 5 : -1;
          ln_cols = min(BN, N - n_tile0);
        }
      }
    }
    if constexpr (FUSE_LN) {
      if (lane == 0) {
        if (ln_rg >= 0) ln_publish(epi, lnq, ln_rg, ln_cols);
        __threadfence_block();
        atomicAdd(&lnq->done, 1);
      }
    }
    if constexpr (OUT != OUT_GENERIC && OUT != OUT_SCREEN) {
      if (lane == 0) tma_store_wait_all();
    }
  }
}

// ------------------------------------------------------------------------------------------
// SIMT reference GEMM (bring-up cross-check / JIMM_GEMM_IMPL=simt bisection only)
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void gemm_simt_kernel(const T* __restrict__ A, int lda, const T* __restrict__ B, int ldb, int K, EpiDev epi) {
  __shared__ float As[16][17], Bs[16][17];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int row = blockIdx.y * 16 + ty, col = blockIdx.x * 16 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
    const int ar = blockIdx.y * 16 + ty, ak = k0 + tx;
    As[ty][tx] = (ar < epi.M && ak < K) ? to_float(A[static_cast<size_t>(ar) * lda + ak]) : 0.f;
    const int br = blockIdx.x * 16 + ty, bk = k0 + tx;
    Bs[ty][tx] = (br < epi.N && bk < K) ? to_float(B[static_cast<size_t>(br) * ldb + bk]) : 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc += As[ty][k] * Bs[tx][k];
    __syncthreads();
  }
  if (row < epi.M && col < epi.N) {
    int out_row, add_row;
    remap_row(epi, row, out_row, add_row);
    float v = acc;
    if constexpr (kScaled<T>) v *= epi.a_scale[row] * epi.b_scale[col];
    if (epi.bias) v += epi.bias[col];
    v = apply_act(v, epi.act);
    if (epi.rowadd) v += epi.rowadd[static_cast<size_t>(add_row) * epi.N + col];
    if (epi.residual) v += epi.residual[static_cast<size_t>(out_row) * epi.ldr + col];
    store1(epi, out_row, col, v);
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_STAGE_BYTES + static_cast<int>(sizeof(LnQueue)) + 2 * STAGES * 8 + 1024;
static_assert(SMEM_BYTES <= 232448, "exceeds 227 KB of shared memory");
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static std::atomic<PFN_encodeTiled> fn{nullptr};  // handles finalized in several threads may resolve it at once (same pointer)
  if (PFN_encodeTiled f = fn.load(std::memory_order_acquire)) return f;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
    set_last_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn.store(reinterpret_cast<PFN_encodeTiled>(p), std::memory_order_release);
  return reinterpret_cast<PFN_encodeTiled>(p);
}

static CUtensorMapDataType tensor_map_dtype(int dtype) {
  switch (dtype) {
    case DT_F32:
    case DT_TF32: return CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    case DT_F16: return CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    case DT_E4M3: return CU_TENSOR_MAP_DATA_TYPE_UINT8;
    default: return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  }
}

// 2-D tensor map over a row-major [rows, cols] matrix (K-major operands: cols = K): dims {cols, rows}, box {128 B worth of columns,
// box_rows}, SWIZZLE_128B, zero OOB fill.
int make_tensor_map_2d(CUtensorMap* map, int dtype, const void* ptr, int rows, int cols, int ld, int box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -3;
  const size_t es = dtype_size(dtype);
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * es};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / es), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (strides[0] & 15) != 0) {
    set_last_error("gemm: operand pointer/stride must be 16-byte aligned (ptr=%p, ld=%d)", ptr, ld);
    return -1;
  }
  CUresult r = enc(map, tensor_map_dtype(dtype), 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rows=%d cols=%d ld=%d)", static_cast<int>(r), rows, cols, ld);
    return -3;
  }
  return 0;
}

// 3-D tensor map over out[B, S, N] (dims {N, S, B}), box {128 B of columns, 16 rows, 1}, SWIZZLE_128B: rows >= S are clipped,
// so a 16-row box never spills into the next sample.
static int make_tensor_map_3d(CUtensorMap* map, int dtype, const void* ptr, int B, int S, int N, int ld) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -3;
  const size_t es = dtype_size(dtype);
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(N), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(B)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld) * es, static_cast<cuuint64_t>(S) * ld * es};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(128 / es), EPI_BOX_ROWS, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, tensor_map_dtype(dtype), 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled(3d) failed: CUresult %d", static_cast<int>(r)); return -3; }
  return 0;
}

int device_sm_count() {  // of the CURRENT device (cached per device: a process may drive several GPUs)
  // threads driving distinct handles may fill an entry at once: they compute the same value, and the atomic makes that defined
  static std::atomic<int> sms[DeviceOnce::kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= DeviceOnce::kMaxDevices) dev = 0;
  int n = sms[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    const char* env = getenv("JIMM_NUM_SMS");
    if (env && atoi(env) > 0) n = atoi(env);
    sms[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

static int check_epi(const GemmEpilogue& e, int N) {
  if (e.out == nullptr) { set_last_error("gemm: null output"); return -1; }
  if (e.ldo < N) { set_last_error("gemm: ldo (%d) < N (%d)", e.ldo, N); return -1; }
  return 0;
}
// e4m3 operands take the plain-store epilogues only (bias, activation; modes 0 / 1 / 2) and need both scale vectors
static int check_e4m3_epi(const GemmEpilogue& e) {
  if (e.a_scale == nullptr || e.b_scale == nullptr) { set_last_error("gemm: e4m3 operands need row scales for A and B"); return -1; }
  if ((reinterpret_cast<uintptr_t>(e.b_scale) & 7) != 0) { set_last_error("gemm: the B scales must be 8-byte aligned"); return -1; }
  if (e.residual || e.rowadd || e.rows_in != 0 || e.tok_pad != 0 || e.ln_cnt) {
    set_last_error("gemm: e4m3 operands support bias and activation epilogues only (no residual, row-add, row remap, token scatter or "
                   "fused LayerNorm)");
    return -1;
  }
  return 0;
}
int gemm_plan_init(GemmPlan* plan, int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K,
                   const GemmEpilogue& epi) {
  if (M <= 0 || N <= 0 || K <= 0) { set_last_error("gemm: bad shape %dx%dx%d", M, N, K); return -1; }
  if (int rc = check_epi(epi, N)) return rc;
  if (dtype == DT_E4M3) {
    if (int rc = check_e4m3_epi(epi)) return rc;
  }
  // the token scatter exists only as the TMA reduce-add: every other epilogue would ignore tok_* and write the plain row layout
  if (epi.tok_pad != 0) {
    if (epi.tok_pad < 0 || epi.tok_pad % EPI_BOX_ROWS != 0 || M % epi.tok_pad != 0 || epi.tok_off < 0 || epi.tok_S <= 0) {
      set_last_error("gemm: token scatter needs tok_pad a positive multiple of %d dividing M (tok_pad=%d M=%d tok_off=%d tok_S=%d)", EPI_BOX_ROWS,
                     epi.tok_pad, M, epi.tok_off, epi.tok_S);
      return -1;
    }
    if (epi.residual != epi.out || epi.ldr != epi.ldo || epi.out_type != DT_F32) {
      set_last_error("gemm: token scatter reduce-adds into an fp32 output that is also the residual");
      return -1;
    }
  }
  if (int rc = make_tensor_map_2d(&plan->map_a, dtype, A, M, K, lda, tile_rows(dtype))) return rc;
  if (int rc = make_tensor_map_2d(&plan->map_b, dtype, B, N, K, ldb, BN)) return rc;
  plan->M = M; plan->N = N; plan->K = K; plan->dtype = dtype; plan->epi = epi;
  memset(&plan->map_c, 0, sizeof(plan->map_c));
  if (plan->epi.mode == 2) {
    const size_t es = dtype_size(epi.out_type);
    // N * es % 16: where a row ends inside a 16-byte chunk, the TMA store wrote columns past N (fp16 / bf16 output, N = 2300,
    // ldo = 2320, on an H100); with ldo > N they belong to the caller.  Such N take the LSU epilogue.
    const bool ok = epi.rowadd == nullptr && epi.rows_in == 0 && (static_cast<size_t>(N) * es) % 16 == 0 &&
                    (epi.residual == nullptr || (epi.residual == epi.out && epi.ldr == epi.ldo && epi.out_type == DT_F32)) &&
                    (static_cast<size_t>(epi.ldo) * es) % 16 == 0 && (reinterpret_cast<uintptr_t>(epi.out) & 15) == 0 &&
                    (epi.bias == nullptr || ((reinterpret_cast<uintptr_t>(epi.bias) & 15) == 0 && N % 4 == 0)) &&
                    !(epi.residual && epi.act != ACT_NONE);
    if (ok && epi.tok_pad > 0) {
      if (int rc = make_tensor_map_3d(&plan->map_c, DT_F32, epi.out, M / epi.tok_pad, epi.tok_S, N, epi.ldo)) return rc;
    } else if (ok) {
      if (int rc = make_tensor_map_2d(&plan->map_c, epi.out_type, epi.out, M, N, epi.ldo, EPI_BOX_ROWS)) return rc;
    } else {
      plan->epi.mode = 0;
    }
  }
  if (epi.tok_pad > 0 && plan->epi.mode != 2) {
    set_last_error("gemm: the token scatter needs the TMA epilogue (mode 2, no activation, 16-byte aligned output / bias, N %% 4 == 0)");
    return -1;
  }
  return 0;
}

static EpiDev to_dev(const GemmEpilogue& e, int M, int N) {
  EpiDev d;
  d.bias = e.bias; d.rowadd = e.rowadd; d.residual = e.residual; d.out = e.out;
  d.act = e.act; d.ldr = e.ldr; d.out_type = e.out_type; d.ldo = e.ldo;
  d.rows_in = e.rows_in; d.rows_out = e.rows_out; d.row_off = e.row_off; d.mode = e.mode;
  d.M = M; d.N = N;
  d.tok_pad = e.tok_pad; d.tok_off = e.tok_off;
  d.reverse = e.reverse;
  d.ln_scale = e.ln_scale; d.ln_bias = e.ln_bias; d.ln_out = e.ln_out; d.ln_cnt = e.ln_cnt;
  d.ln_out_type = e.ln_out_type; d.ln_ldo = e.ln_ldo; d.ln_eps = e.ln_eps;
  d.a_scale = e.a_scale; d.b_scale = e.b_scale;
  return d;
}

template <typename T, int OUT, int ACT>
static int launch_one(const GemmPlan* p, int M, cudaStream_t stream) {
  constexpr auto kernel = gemm_wgmma_kernel<T, OUT, ACT>;
  constexpr int TM = tile_rows(Traits<T>::DTYPE);
  if (int rc = smem_opt_in<kernel>(SMEM_BYTES)) return rc;
  static DeviceOnce regs_checked;
  if (int rc = regs_checked.run([&]() -> int {
        // setmaxnreg moves registers within the launch allocation: with fewer than KERNEL_REGS per thread, an increase would wait forever
        cudaFuncAttributes fa;
        JIMM_CUDA_CHECK(cudaFuncGetAttributes(&fa, kernel));
        if (fa.numRegs != KERNEL_REGS) {
          set_last_error("gemm: kernel compiled with %d registers per thread, the warpgroup register split assumes %d", fa.numRegs, KERNEL_REGS);
          return -2;
        }
        return 0;
      }))
    return rc;
  const int tiles = ((M + TM - 1) / TM) * ((p->N + BN - 1) / BN);
  const int grid = tiles < device_sm_count() ? tiles : device_sm_count();
  JIMM_CUDA_CHECK(launch_k(kernel, dim3(grid), dim3(NUM_THREADS), SMEM_BYTES, stream, 1, true, p->map_a, p->map_b, p->map_c,
                           to_dev(p->epi, M, p->N), p->K));
  note_launch();
  return 0;
}

template <typename T, int OUT>
static int launch_act(const GemmPlan* p, int M, cudaStream_t stream) {
  switch (p->epi.act) {
    case ACT_GELU_TANH: return launch_one<T, OUT, ACT_GELU_TANH>(p, M, stream);
    case ACT_QUICK_GELU: return launch_one<T, OUT, ACT_QUICK_GELU>(p, M, stream);
    default: return launch_one<T, OUT, ACT_NONE>(p, M, stream);
  }
}

template <typename T>
static int launch_tc(const GemmPlan* p, int M, cudaStream_t stream) {
  const GemmEpilogue& e = p->epi;
  if (e.mode != 2) return launch_one<T, OUT_GENERIC, ACT_NONE>(p, M, stream);
  if constexpr (!kScaled<T>) {  // gemm_plan_init gives e4m3 plans no residual
    if (e.residual) return gemm_fuses_ln(p, M) ? launch_one<T, OUT_F32_ADD, ACT_FUSE_LN>(p, M, stream) : launch_one<T, OUT_F32_ADD, ACT_NONE>(p, M, stream);
  }
  switch (e.out_type) {
    case DT_F16: return launch_act<T, OUT_H16>(p, M, stream);
    case DT_BF16: return launch_act<T, OUT_BF16>(p, M, stream);
    case DT_TF32: return launch_act<T, OUT_TF32>(p, M, stream);
    default: return launch_act<T, OUT_F32>(p, M, stream);
  }
}

// Will gemm_plan_run(p, M) normalise the finished rows itself (GemmEpilogue::ln_*)?  Same predicate as launch_one.
int gemm_fuses_ln(const GemmPlan* p, int /*M_override: any row count*/) {
  const int nv = p->N >> 7;
  // ln_rows_dispatch's widths; 1280, 1536 and 2048 (nv = 10, 12, 16) are left to the LayerNorm kernel: their row buffers do not fit in
  // the LayerNorm warps' PRODUCER_REGS without spilling
  const bool width_ok = p->N % 128 == 0 && (nv <= 4 || nv == 6 || nv == 8 || nv == 9);
  // the normalised rows are written in this GEMM's operand type (they are the next GEMM's A operand)
  const int want = p->dtype == DT_F16 ? DT_F16 : p->dtype == DT_BF16 ? DT_BF16 : DT_TF32;
  return p->epi.ln_cnt != nullptr && p->epi.ln_out_type == want && width_ok && p->epi.mode == 2 && p->epi.residual != nullptr && p->epi.tok_pad == 0;
}

int gemm_plan_run(const GemmPlan* p0, int M_override, cudaStream_t stream, int reverse) {
  const int M = (M_override > 0 && M_override <= p0->M) ? M_override : p0->M;
  if (p0->epi.tok_pad > 0 && M % p0->epi.tok_pad != 0) {
    set_last_error("gemm: token scatter runs whole samples (M=%d, tok_pad=%d)", M, p0->epi.tok_pad);
    return -1;
  }
  GemmPlan local;
  const GemmPlan* p = p0;
  if (reverse != p0->epi.reverse) { local = *p0; local.epi.reverse = reverse; p = &local; }
  switch (p->dtype) {
    case DT_F16: return launch_tc<__half>(p, M, stream);
    case DT_BF16: return launch_tc<__nv_bfloat16>(p, M, stream);
    case DT_F32:
    case DT_TF32: return launch_tc<float>(p, M, stream);
    case DT_E4M3: return launch_tc<__nv_fp8_e4m3>(p, M, stream);
  }
  set_last_error("gemm: bad dtype %d", p->dtype);
  return -1;
}

int gemm_screen_run(const void* A, int M, const void* B, int N, int K, const GemmScreen& screen, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) { set_last_error("gemm screen: bad shape %dx%dx%d", M, N, K); return -1; }
  if (!screen.t || !screen.nq || !screen.ng || !screen.cnt || !screen.list || screen.cap < 1) {
    set_last_error("gemm screen: null threshold, bound, counter or list, or cap < 1");
    return -1;
  }
  GemmPlan p;
  if (int rc = make_tensor_map_2d(&p.map_a, DT_F16, A, M, K, K, tile_rows(DT_F16))) return rc;
  if (int rc = make_tensor_map_2d(&p.map_b, DT_F16, B, N, K, K, BN)) return rc;
  memset(&p.map_c, 0, sizeof(p.map_c));
  p.M = M; p.N = N; p.K = K; p.dtype = DT_F16;
  // the screen travels in the epilogue fields epilogue_screen reads (see EpiDev)
  p.epi.mode = 0;
  p.epi.bias = screen.t; p.epi.a_scale = screen.nq; p.epi.b_scale = screen.ng; p.epi.ln_cnt = screen.cnt;
  p.epi.out = screen.list; p.epi.ldo = screen.cap;
  return launch_one<__half, OUT_SCREEN, ACT_NONE>(&p, M, stream);
}

int gemm_simt_run(int dtype, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const GemmEpilogue& epi,
                  cudaStream_t stream) {
  if (int rc = check_epi(epi, N)) return rc;
  if (dtype == DT_E4M3) {
    if (int rc = check_e4m3_epi(epi)) return rc;
  }
  dim3 block(16, 16), grid((N + 15) / 16, (M + 15) / 16);
  EpiDev d = to_dev(epi, M, N);
  if (dtype == DT_F16) gemm_simt_kernel<__half><<<grid, block, 0, stream>>>(static_cast<const __half*>(A), lda, static_cast<const __half*>(B), ldb, K, d);
  else if (dtype == DT_BF16) gemm_simt_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>(static_cast<const __nv_bfloat16*>(A), lda, static_cast<const __nv_bfloat16*>(B), ldb, K, d);
  else if (dtype == DT_E4M3) gemm_simt_kernel<__nv_fp8_e4m3><<<grid, block, 0, stream>>>(static_cast<const __nv_fp8_e4m3*>(A), lda, static_cast<const __nv_fp8_e4m3*>(B), ldb, K, d);
  else gemm_simt_kernel<float><<<grid, block, 0, stream>>>(static_cast<const float*>(A), lda, static_cast<const float*>(B), ldb, K, d);
  JIMM_LAUNCH_CHECK();
  return 0;
}

}  // namespace jimm
