// Softmax attention kernels (SURVEY.md 8a row a5, a9).
//
// attention_kernel: flash-style fused softmax(q k^T / sqrt(d)) v over the fused qkv buffer, for any head width d that is a
// multiple of 8 up to 128 (64 in the CLIP / SigLIP vision towers, models/clip.py:60, models/siglip.py:59; 72 in the SigLIP
// so400m text tower, 80 in ViT-H/14, 16 in small ViTs).  One CTA = one warpgroup = 64 query rows of one (sample, head); warp w
// owns rows 16 w .. 16 w + 15; K/V streamed in 64-key tiles through a double-buffered cp.async ring.  The kernel is compiled for
// a padded width DP (padded_head_dim: 16, 32, 64, 80, 96, 128); every tile is 64 rows x DP columns in a swizzled layout
// (HeadTile), with columns d .. DP-1 zero-filled, so the tensor cores read it in place: S = Q K^T is wgmma m64n64k16 with both
// operands in shared memory (K-major), O += P V is wgmma m64nDPk16 with P straight from the score registers (A fragment) and V
// in shared memory (MN-major).  Scores and probabilities never leave registers; fp32 online softmax with warp-quad shuffles.
//
// map_attention_kernel: MAP-head pooling attention with a single precomputed probe query (common/vit.py:96-97), any head
// width the flash kernel takes.
#include <cmath>
#include <type_traits>

#include "common.cuh"
#include "kernels.cuh"

namespace jimm {

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

template <typename T>
__device__ __forceinline__ uint32_t pack_pair(float a, float b) {
  if constexpr (std::is_same<T, __half>::value) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}

static constexpr int QT = 64;   // query rows per CTA
static constexpr int KT = 64;   // keys per pipeline stage

// Shared-memory layout of a 64-row tile of one head, padded to DP columns (DP a multiple of 16).  A row is 2 DP bytes, split into
// NB column blocks of SW bytes (SW = 128, 64 or 32: the widest swizzle that divides the row).  Block b holds columns
// [b SW / 2, (b + 1) SW / 2) of all 64 rows, SW bytes per row, in the SW-byte swizzle layout; blocks are 64 SW bytes apart.
// DP = 64 is one 128-byte-swizzled block of 64 x 128 B.
template <int DP>
struct HeadTile {
  static_assert(DP % 16 == 0 && DP >= 16 && DP <= 128, "padded head width");
  static constexpr int ROWB = DP * 2;
  static constexpr int SW = ROWB % 128 == 0 ? 128 : ROWB % 64 == 0 ? 64 : 32;
  static constexpr int NB = ROWB / SW;
  static constexpr int CH = SW / 16;        // 16-byte chunks per block row
  static constexpr int NCH = DP / 8;        // 16-byte chunks per row
  static constexpr int BYTES = QT * ROWB;   // QT == KT
  static constexpr int SMEM = 5 * BYTES;    // Q + double-buffered K and V
  // byte offset of 16-byte chunk `ch` (columns 8 ch .. 8 ch + 7) of row `row`
  static __device__ __forceinline__ uint32_t off(uint32_t row, uint32_t ch) {
    const uint32_t blk = ch / CH, cb = ch % CH;
    return blk * (QT * SW) + row * SW + ((cb ^ ((row * SW >> 7) & (CH - 1))) << 4);
  }
  // wgmma descriptor offset (16-byte units) of head dims 16 ks .. 16 ks + 15 of a K-major tile
  static __device__ __forceinline__ uint64_t kstep(int ks) { return static_cast<uint64_t>(((ks * 32) / SW * (QT * SW) + (ks * 32) % SW) >> 4); }
};

// 16-byte cp.async that reads src_bytes (16 or 0) from global memory and zero-fills the rest
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes));
}

// Copy a 64-row tile of one head (rows s0.. ; row stride `ld` elements; d columns) into the HeadTile<DP> layout; columns d .. DP-1
// are zero-filled (cp.async reads no bytes for them), so they add nothing to Q K^T.  Rows >= S are clamped to S-1 (their scores
// are masked / their outputs are never stored).
template <typename T, int DP>
__device__ __forceinline__ void load_tile(uint32_t smem_base, const T* __restrict__ gbase, size_t ld, int s0, int S, int d, int tid) {
  using L = HeadTile<DP>;
#pragma unroll
  for (int i = 0; i < L::NCH * QT / 128; ++i) {
    const uint32_t c = tid + i * 128;  // unsigned: the division and modulo fold to shifts and masks
    const uint32_t row = c / L::NCH, ch = c % L::NCH;
    int s = s0 + static_cast<int>(row);
    s = s < S ? s : S - 1;
    const bool in = static_cast<int>(ch * 8) < d;
    const T* src = gbase + static_cast<size_t>(s) * ld + (in ? ch * 8 : 0);
    cp_async16_zfill(smem_base + L::off(row, ch), src, in ? 16u : 0u);
  }
}

// Shared memory of a CTA: static up to 48 KB, else dynamic (opted in by attn_launch_k, 1 KB of slack for the 1024-byte alignment).
template <int BYTES, bool STATIC = (BYTES <= 48 * 1024)>
struct AttnSmem {
  static __device__ __forceinline__ uint8_t* get() {
    __shared__ __align__(1024) uint8_t smem[BYTES];  // 1024-aligned: the swizzle atoms of the wgmma operands
    return smem;
  }
};
template <int BYTES>
struct AttnSmem<BYTES, false> {
  static __device__ __forceinline__ uint8_t* get() {
    extern __shared__ uint8_t smem_raw[];
    return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  }
};

// The rows of sample b: rows row0 .. row0 + S - 1 of qkv / out.  Dense: B samples of S_arg rows each.  PACKED: sample b is rows
// seq_off[b] .. seq_off[b + 1] - 1 (read after pdl_wait: the offsets may come from the previous kernel).
template <bool PACKED>
__device__ __forceinline__ void sample_rows(int b, int S_arg, const int* __restrict__ seq_off, size_t& row0, int& S) {
  if constexpr (PACKED) {
    row0 = static_cast<size_t>(seq_off[b]);
    S = seq_off[b + 1] - seq_off[b];
  } else {
    row0 = static_cast<size_t>(b) * S_arg;
    S = S_arg;
  }
}

// S = Q K^T of one 64-key tile (64 x 64 per warpgroup, both operands K-major in shared memory): this warp's 16 query rows in the
// m16n8 accumulator layout, s[n-block][e] = the score of row g + 8 (e >> 1) and key 8 n-block + 2 t4 + (e & 1) (g = lane / 4, t4 = lane % 4).
template <typename T, int DP>
__device__ __forceinline__ void score_tile(float (&s)[8][4], uint64_t qdesc, uint32_t sK) {
  using L = HeadTile<DP>;
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  float (&s_acc)[32] = reinterpret_cast<float (&)[32]>(s);
  const uint64_t kdesc = make_wgmma_desc<L::SW>(sK, 16);
#pragma unroll
  for (int i = 0; i < 32; ++i) s_acc[i] = 0.f;
  wgmma_fence_operands(s_acc);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < DP / 16; ++ks)  // 16 head dims (32 B) per step
    wgmma_m64n64k16_ss<BF16>(s_acc, qdesc + L::kstep(ks), kdesc + L::kstep(ks), ks != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operands(s_acc);
}

// Scores of keys at or past S, and (CAUSAL) of keys above the diagonal, to -inf.  k0: the tile's first key, q0: the CTA's first query
// row, row_lo: this thread's first row (the other is row_lo + 8).  Tiles with no such key are left alone.
template <bool CAUSAL>
__device__ __forceinline__ void mask_tile(float (&s)[8][4], int k0, int q0, int row_lo, int t4, int S) {
  if ((k0 + KT > S) || (CAUSAL && (k0 + KT - 1 > q0))) {
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + nt * 8 + t4 * 2 + (e & 1);
        const int qrow = row_lo + (e >> 1) * 8;
        const bool ok = key < S && (!CAUSAL || key <= qrow);
        if (!ok) s[nt][e] = -INFINITY;
      }
    }
  }
}

// One online-softmax step over a masked score tile, for this thread's two rows: the row max (over the quad that shares the rows)
// updates m_run, s becomes p = exp2(s scale_log2 - m_run scale_log2) in place, and l_run, this thread's share of the row sums, is
// rescaled to the new max and adds the tile's p.  Returns alpha, the factor that rescaled l_run (and must rescale what else the earlier
// tiles summed).  A row with every key masked so far keeps m_run = -inf and gets p = 0.
__device__ __forceinline__ float2 softmax_step(float (&s)[8][4], float (&m_run)[2], float (&l_run)[2], float scale_log2) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
    mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
  }
  float alpha[2], moff[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float mnew = fmaxf(m_run[r], mx[r]);
    const float muse = (mnew == -INFINITY) ? 0.f : mnew;
    alpha[r] = exp2f((m_run[r] - muse) * scale_log2);  // m_run = -inf -> 0
    m_run[r] = mnew;
    moff[r] = muse * scale_log2;
    l_run[r] *= alpha[r];
  }
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    s[nt][0] = exp2f(s[nt][0] * scale_log2 - moff[0]);
    s[nt][1] = exp2f(s[nt][1] * scale_log2 - moff[0]);
    s[nt][2] = exp2f(s[nt][2] * scale_log2 - moff[1]);
    s[nt][3] = exp2f(s[nt][3] * scale_log2 - moff[1]);
    l_run[0] += s[nt][0] + s[nt][1];
    l_run[1] += s[nt][2] + s[nt][3];
  }
  return make_float2(alpha[0], alpha[1]);
}

// 1 / l of one of this thread's rows: l, this thread's share of the row sum, added over the quad that shares the row
__device__ __forceinline__ float row_inv_sum(float l) {
  l += __shfl_xor_sync(0xffffffffu, l, 1);
  l += __shfl_xor_sync(0xffffffffu, l, 2);
  return 1.0f / l;
}

// Head width d (a multiple of 8, d <= DP); the tiles are padded to DP columns with zeros.  scale_log2 = log2(e) / sqrt(d).
// PACKED: sample b is rows seq_off[b] .. seq_off[b + 1] - 1 of qkv / out (S_arg unused); query tiles past a sample's end exit at once.
template <typename T, typename OutT, bool CAUSAL, int DP, bool PACKED = false>
__global__ void __launch_bounds__(128)
attention_kernel(const T* __restrict__ qkv, OutT* __restrict__ out, int S_arg, int H, int d, float scale_log2, int reverse,
                 const int* __restrict__ seq_off) {
  using L = HeadTile<DP>;
  uint8_t* smem = AttnSmem<L::SMEM>::get();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = reverse ? static_cast<int>(gridDim.z) - 1 - static_cast<int>(blockIdx.z) : static_cast<int>(blockIdx.z);
  const int D = H * d;
  const size_t ld = static_cast<size_t>(3) * D;
  if constexpr (PACKED) {
    pdl_launch_dependents();
    pdl_wait();  // the offsets may come from the previous kernel
  }
  size_t row0;
  int S;
  sample_rows<PACKED>(b, S_arg, seq_off, row0, S);
  if (PACKED && qt * QT >= S) return;
  const T* base = qkv + row0 * ld + h * d;
  const T* gq = base;
  const T* gk = base + D;
  const T* gv = base + 2 * D;
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK0 = sQ + L::BYTES;
  const uint32_t sV0 = sK0 + 2 * L::BYTES;
  const int q0 = qt * QT;
  if constexpr (!PACKED) {
    pdl_launch_dependents();
    pdl_wait();
  }
  int n_kv = (S + KT - 1) / KT;
  if (CAUSAL) n_kv = min(n_kv, qt + 1);

  load_tile<T, DP>(sQ, gq, ld, q0, S, d, tid);
  load_tile<T, DP>(sK0, gk, ld, 0, S, d, tid);
  load_tile<T, DP>(sV0, gv, ld, 0, S, d, tid);
  cp_async_commit();

  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  const uint64_t qdesc = make_wgmma_desc<L::SW>(sQ, 16);
  float o[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int g = lane >> 2, t4 = lane & 3;
  const int row_lo = q0 + warp * 16 + g;  // this thread's two query rows: row_lo, row_lo + 8

  for (int j = 0; j < n_kv; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile<T, DP>(sK0 + (buf ^ 1) * L::BYTES, gk, ld, (j + 1) * KT, S, d, tid);
      load_tile<T, DP>(sV0 + (buf ^ 1) * L::BYTES, gv, ld, (j + 1) * KT, S, d, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();  // this thread's cp.async writes -> visible to the tensor cores' (async proxy) reads
    __syncthreads();
    const uint32_t sK = sK0 + buf * L::BYTES, sV = sV0 + buf * L::BYTES;

    float s[8][4];
    score_tile<T, DP>(s, qdesc, sK);
    mask_tile<CAUSAL>(s, j * KT, q0, row_lo, t4, S);
    const float2 alpha = softmax_step(s, m_run, l_run, scale_log2);
#pragma unroll
    for (int nt = 0; nt < DP / 8; ++nt) {
      o[nt][0] *= alpha.x; o[nt][1] *= alpha.x;
      o[nt][2] *= alpha.y; o[nt][3] *= alpha.y;
    }
    // ---- O += P V: A = P (keys 16 kk .. 16 kk + 15 of this warp's rows), B = V rows of those keys (MN-major, 16 rows per step) ----
    uint32_t pf[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pf[kk][0] = pack_pair<T>(s[2 * kk][0], s[2 * kk][1]);
      pf[kk][1] = pack_pair<T>(s[2 * kk][2], s[2 * kk][3]);
      pf[kk][2] = pack_pair<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pf[kk][3] = pack_pair<T>(s[2 * kk + 1][2], s[2 * kk + 1][3]);
    }
    float (&o_acc)[DP / 2] = reinterpret_cast<float (&)[DP / 2]>(o);
    const uint64_t vdesc = make_wgmma_desc<L::SW>(sV, L::NB > 1 ? QT * L::SW : 16);
    wgmma_fence_operands(o_acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64nNk16_rs<BF16, DP>(o_acc, pf[kk], vdesc + static_cast<uint64_t>(kk * (16 * L::SW >> 4)));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(o_acc);
    __syncthreads();  // everyone done with buf before it is refilled two iterations later
  }

  // ---- finalise: O /= l, store columns < d ----
  const float inv[2] = {row_inv_sum(l_run[0]), row_inv_sum(l_run[1])};
  OutT* obase = out + row0 * D + h * d;
  if constexpr (sizeof(OutT) == 2) {
    // stage this warp's 16 x DP tile through its (now free) Q rows so the global stores are whole 16-byte chunks of a row
    uint8_t* sq = smem;
#pragma unroll
    for (int nt = 0; nt < DP / 8; ++nt) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = warp * 16 + g + r * 8;
        const int ch = nt;  // 8 columns (16 B) per n-tile
        const uint32_t v = pack_pair<OutT>(o[nt][2 * r] * inv[r], o[nt][2 * r + 1] * inv[r]);
        *reinterpret_cast<uint32_t*>(sq + L::off(row, ch) + t4 * 4) = v;
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < L::NCH / 2; ++i) {  // 16 rows x NCH chunks, 32 per step
      const uint32_t c = i * 32 + lane;
      const int row = warp * 16 + static_cast<int>(c / L::NCH), ch = static_cast<int>(c % L::NCH);
      const int srow = q0 + row;
      if (srow < S && ch * 8 < d) {
        const uint4 v = *reinterpret_cast<const uint4*>(sq + L::off(row, ch));
        *reinterpret_cast<uint4*>(obase + static_cast<size_t>(srow) * D + ch * 8) = v;
      }
    }
  } else {
#pragma unroll
    for (int nt = 0; nt < DP / 8; ++nt) {
      if (nt * 8 >= d) break;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int srow = row_lo + r * 8;
        if (srow < S) {
          float2 v = make_float2(o[nt][2 * r] * inv[r], o[nt][2 * r + 1] * inv[r]);
          if constexpr (std::is_same<OutT, tf32_t>::value) v = make_float2(round_tf32(v.x), round_tf32(v.y));
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(obase) + static_cast<size_t>(srow) * D + nt * 8 + t4 * 2) = v;
        }
      }
    }
  }
}

// The padded widths compiled: d is run at the smallest of them >= d.  16, 32, 64 and 128 are exact for the common head widths; 80
// serves ViT-H / SigLIP so400m-text widths (80, 72) and 96 widths 88 and 96.  Widths 40-56 run at 64 and 104-120 at 128.
static int padded_head_dim(int d) { return d <= 16 ? 16 : d <= 32 ? 32 : d <= 64 ? 64 : d <= 80 ? 80 : d <= 96 ? 96 : 128; }

// The softmax scale 1 / sqrt(d) (flax: query / sqrt(depth)) times log2(e), in fp32: 0.125f * log2(e) for d = 64.
static float attn_scale_log2(int d) { return static_cast<float>(1.0 / std::sqrt(static_cast<double>(d))) * 1.4426950408889634f; }

// Calls f(CAUSAL, DP, PACKED), each a std::integral_constant: the compiled variant of a wgmma attention kernel that runs head width d,
// causal or not, on B samples of S rows each (seq_off null) or in the packed form (S = the longest sample, sample b = rows seq_off[b]
// .. seq_off[b + 1] - 1).  Packed and causal: the query tile, the key count n_kv and the mask are all relative to the sample's first
// row (row0), so each sample is masked as it is alone.
template <typename F>
static int attn_variant(int d, int causal, const int* seq_off, F&& f) {
  auto at_width = [&](auto c, auto p) -> int {
    switch (padded_head_dim(d)) {
      case 16: return f(c, std::integral_constant<int, 16>{}, p);
      case 32: return f(c, std::integral_constant<int, 32>{}, p);
      case 64: return f(c, std::integral_constant<int, 64>{}, p);
      case 80: return f(c, std::integral_constant<int, 80>{}, p);
      case 96: return f(c, std::integral_constant<int, 96>{}, p);
      default: return f(c, std::integral_constant<int, 128>{}, p);
    }
  };
  if (seq_off && causal) return at_width(std::true_type{}, std::true_type{});
  if (seq_off) return at_width(std::false_type{}, std::true_type{});
  if (causal) return at_width(std::true_type{}, std::false_type{});
  return at_width(std::false_type{}, std::false_type{});
}

// Launches Kernel, one warpgroup CTA per 64 query rows of each (sample, head), with SMEM bytes of shared memory: static up to 48 KB,
// else dynamic (opted in, with 1 KB of slack for AttnSmem's 1024-byte alignment).
template <auto Kernel, int SMEM, typename... Args>
static int attn_launch_k(int B, int S, int H, cudaStream_t stream, Args... args) {
  constexpr int dyn = SMEM <= 48 * 1024 ? 0 : SMEM + 1024;
  if constexpr (dyn > 0) {
    if (int rc = smem_opt_in<Kernel>(dyn)) return rc;
  }
  JIMM_CUDA_CHECK(launch_k(Kernel, dim3((S + QT - 1) / QT, H, B), dim3(128), dyn, stream, 1, true, args...));
  note_launch();
  return 0;
}

template <typename T>
struct Type {
  using type = T;
};
// Calls f(Type<T>{}, Type<OutT>{}) for the (io, out) dtype pairs of the flash and MAP kernels.
template <typename F>
static int io_out_dispatch(const char* name, int io_type, int out_type, F&& f) {
  if (io_type == DT_F16 && out_type == DT_F16) return f(Type<__half>{}, Type<__half>{});
  if (io_type == DT_F16 && out_type == DT_F32) return f(Type<__half>{}, Type<float>{});
  if (io_type == DT_F16 && out_type == DT_TF32) return f(Type<__half>{}, Type<tf32_t>{});
  if (io_type == DT_BF16 && out_type == DT_BF16) return f(Type<__nv_bfloat16>{}, Type<__nv_bfloat16>{});
  if (io_type == DT_BF16 && out_type == DT_F32) return f(Type<__nv_bfloat16>{}, Type<float>{});
  set_last_error("%s: unsupported dtype combination io=%d out=%d", name, io_type, out_type);
  return -1;
}

static bool head_dim_ok(int d) { return d >= 8 && d <= 128 && d % 8 == 0; }

static int attn_dispatch(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, int causal, cudaStream_t stream,
                         int reverse, const int* seq_off) {
  if (!head_dim_ok(head_dim)) { set_last_error("attention: head_dim %d is not a multiple of 8 in [8, 128]", head_dim); return -1; }
  if (B <= 0 || S <= 0) return 0;
  if (B > 65535 || H > 65535) { set_last_error("attention: grid too large (B=%d H=%d)", B, H); return -1; }
  return io_out_dispatch("attention", io_type, out_type, [&](auto io, auto o) {
    using T = typename decltype(io)::type;
    using OutT = typename decltype(o)::type;
    return attn_variant(head_dim, causal, seq_off, [&](auto c, auto dp, auto p) {
      constexpr int DP = decltype(dp)::value;
      return attn_launch_k<attention_kernel<T, OutT, decltype(c)::value, DP, decltype(p)::value>, HeadTile<DP>::SMEM>(
          B, S, H, stream, static_cast<const T*>(qkv), static_cast<OutT*>(out), S, H, head_dim, attn_scale_log2(head_dim), reverse, seq_off);
    });
  });
}

int attention_run(const void* qkv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, int causal, cudaStream_t stream, int reverse) {
  return attn_dispatch(qkv, io_type, out, out_type, B, S, H, head_dim, causal, stream, reverse, nullptr);
}

int attention_packed_run(const void* qkv, int io_type, void* out, int out_type, const int* seq_off, int B, int max_S, int H, int head_dim,
                         int causal, cudaStream_t stream, int reverse) {
  if (!seq_off) { set_last_error("attention_packed: null seq_off"); return -1; }
  return attn_dispatch(qkv, io_type, out, out_type, B, max_S, H, head_dim, causal, stream, reverse, seq_off);
}

// ------------------------------------------------------------------------------------------
// Attention weights (HF output_attentions): softmax(q k^T / sqrt(d)) of one block, written out.
// ------------------------------------------------------------------------------------------
// One CTA = one warpgroup = 64 query rows of one (sample, head), the tiles, descriptors and S = Q K^T of attention_kernel.  Two passes over
// the sample's 64-key tiles: the first keeps the fp32 online row max m and sum l (exp2 with scale_log2, as attention_kernel does), the
// second recomputes each score tile and writes p = exp2(s c - m) / l.  Each warp stages its 16 x 64 tile in shared memory and writes it
// as row segments of consecutive keys: rows are S elements long, so no store can assume more than the element's alignment.  Causal:
// key tiles entirely above the diagonal are written as zeros without being computed.  Rows q >= S and keys >= S are never stored.
// out: sample b's [H, S_b, S_b] block starts at element H * sum_{j<b} S_j^2 (dense: b * H * S^2); every offset is 64-bit.
template <int DP, int OUTB>
struct ProbsSmem {
  static constexpr int STAGE_LD = OUTB == 4 ? 72 : 36;  // 32-bit words per staged row (64 fp32 or 64 16-bit + padding: no bank conflicts)
  static constexpr int STAGE = QT * STAGE_LD * 4;
  static constexpr int BYTES = 3 * HeadTile<DP>::BYTES + STAGE;  // Q + double-buffered K + the staged output tile
};

template <typename T, typename OutT, bool CAUSAL, int DP, bool PACKED>
__global__ void __launch_bounds__(128)
attn_probs_kernel(const T* __restrict__ qkv, OutT* __restrict__ out, int S_arg, int H, int d, float scale_log2, const int* __restrict__ seq_off) {
  using L = HeadTile<DP>;
  using PS = ProbsSmem<DP, static_cast<int>(sizeof(OutT))>;
  uint8_t* smem = AttnSmem<PS::BYTES>::get();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = H * d;
  const size_t ld = static_cast<size_t>(3) * D;
  uint32_t* stage = reinterpret_cast<uint32_t*>(smem + 3 * L::BYTES);
  pdl_launch_dependents();
  pdl_wait();  // qkv is the QKV GEMM's output (and the offsets may come from the previous kernel)
  size_t row0;
  int S;
  sample_rows<PACKED>(b, S_arg, seq_off, row0, S);
  size_t obase = static_cast<size_t>(b) * H * S_arg * S_arg;
  if constexpr (PACKED) {
    if (qt * QT >= S) return;
    // H * sum_{j<b} S_j^2, reduced over the CTA
    unsigned long long acc = 0;
    for (int j = tid; j < b; j += 128) {
      const unsigned long long n = static_cast<unsigned long long>(seq_off[j + 1] - seq_off[j]);
      acc += n * n;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    unsigned long long* red = reinterpret_cast<unsigned long long*>(stage);  // free until pass 2
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    obase = static_cast<size_t>(H) * (red[0] + red[1] + red[2] + red[3]);
  }
  obase += static_cast<size_t>(h) * S * S;
  const T* gq = qkv + row0 * ld + h * d;
  const T* gk = gq + D;
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK0 = sQ + L::BYTES;
  const int q0 = qt * QT;
  const int n_all = (S + KT - 1) / KT;
  const int n_kv = CAUSAL ? min(n_all, qt + 1) : n_all;  // the tiles with a key at or below the diagonal

  const uint64_t qdesc = make_wgmma_desc<L::SW>(sQ, 16);
  const int g = lane >> 2, t4 = lane & 3;
  const int row_lo = q0 + warp * 16 + g;  // this thread's two query rows: row_lo, row_lo + 8

  // S = Q K^T of key tile j, masked.  The K tile of step j of a pass is in buffer j & 1; the next one is prefetched while this one is used.
  auto scores = [&](int j, float (&s)[8][4]) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile<T, DP>(sK0 + (buf ^ 1) * L::BYTES, gk, ld, (j + 1) * KT, S, d, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    score_tile<T, DP>(s, qdesc, sK0 + buf * L::BYTES);
    __syncthreads();  // every warp is done reading buf before it is refilled by the next step's prefetch
    mask_tile<CAUSAL>(s, j * KT, q0, row_lo, t4, S);
  };

  // ---- pass 1: row max and sum (the flash kernel's softmax steps; p and alpha are not needed) ----
  load_tile<T, DP>(sQ, gq, ld, q0, S, d, tid);
  load_tile<T, DP>(sK0, gk, ld, 0, S, d, tid);
  cp_async_commit();
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  for (int j = 0; j < n_kv; ++j) {
    float s[8][4];
    scores(j, s);
    softmax_step(s, m_run, l_run, scale_log2);
  }
  float inv[2], moff[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    inv[r] = row_inv_sum(l_run[r]);
    moff[r] = (m_run[r] == -INFINITY ? 0.f : m_run[r]) * scale_log2;
  }

  // ---- pass 2: the probabilities, staged per warp and stored as row segments ----
  uint32_t* wst = stage + warp * 16 * PS::STAGE_LD;
  OutT* orow = out + obase + static_cast<size_t>(q0 + warp * 16) * S;  // this warp's first row
  const int rows = min(16, S - (q0 + warp * 16));                       // this warp's rows inside the sample (may be <= 0)
  load_tile<T, DP>(sK0, gk, ld, 0, S, d, tid);
  cp_async_commit();
  for (int j = 0; j < n_all; ++j) {
    const int k0 = j * KT, cols = min(KT, S - k0);
    if (j < n_kv) {
      float s[8][4];
      scores(j, s);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float p0 = exp2f(s[nt][2 * r] * scale_log2 - moff[r]) * inv[r];
          const float p1 = exp2f(s[nt][2 * r + 1] * scale_log2 - moff[r]) * inv[r];
          const int srow = g + r * 8, c = nt * 8 + t4 * 2;
          if constexpr (sizeof(OutT) == 4) *reinterpret_cast<float2*>(wst + srow * PS::STAGE_LD + c) = make_float2(p0, p1);
          else wst[srow * PS::STAGE_LD + c / 2] = pack_pair<OutT>(p0, p1);
        }
      }
      __syncwarp();
      for (int r = 0; r < rows; ++r) {
        OutT* dst = orow + static_cast<size_t>(r) * S + k0;
        const OutT* src = reinterpret_cast<const OutT*>(wst + r * PS::STAGE_LD);
        if (lane < cols) dst[lane] = src[lane];
        if (lane + 32 < cols) dst[lane + 32] = src[lane + 32];
      }
      __syncwarp();  // the staged tile is read before the next one overwrites it
    } else {  // causal: every key of the tile is above the diagonal
      const OutT z = from_float<OutT>(0.f);
      for (int r = 0; r < rows; ++r) {
        OutT* dst = orow + static_cast<size_t>(r) * S + k0;
        if (lane < cols) dst[lane] = z;
        if (lane + 32 < cols) dst[lane + 32] = z;
      }
    }
  }
}

template <typename T, typename OutT>
static int probs_launch(const void* qkv, void* out, int B, int S, int H, int d, int causal, cudaStream_t stream, const int* seq_off) {
  return attn_variant(d, causal, seq_off, [&](auto c, auto dp, auto p) {
    constexpr int DP = decltype(dp)::value;
    return attn_launch_k<attn_probs_kernel<T, OutT, decltype(c)::value, DP, decltype(p)::value>, ProbsSmem<DP, static_cast<int>(sizeof(OutT))>::BYTES>(
        B, S, H, stream, static_cast<const T*>(qkv), static_cast<OutT*>(out), S, H, d, attn_scale_log2(d), seq_off);
  });
}

template <typename T>
static int probs_out(const void* qkv, void* out, int out_type, int B, int S, int H, int d, int causal, cudaStream_t stream, const int* seq_off) {
  if (out_type == DT_F32) return probs_launch<T, float>(qkv, out, B, S, H, d, causal, stream, seq_off);
  if (out_type == DT_F16) return probs_launch<T, __half>(qkv, out, B, S, H, d, causal, stream, seq_off);
  return probs_launch<T, __nv_bfloat16>(qkv, out, B, S, H, d, causal, stream, seq_off);
}

int attn_probs_run(const void* qkv, int io_type, void* out, int out_type, const int* seq_off, int B, int S, int H, int head_dim, int causal,
                   cudaStream_t stream) {
  if (!head_dim_ok(head_dim)) { set_last_error("attn_probs: head_dim %d is not a multiple of 8 in [8, 128]", head_dim); return -1; }
  if (out_type != DT_F32 && out_type != DT_F16 && out_type != DT_BF16) { set_last_error("attn_probs: output dtype %d", out_type); return -1; }
  if (B <= 0 || S <= 0) return 0;
  if (B > 65535 || H > 65535) { set_last_error("attn_probs: grid too large (B=%d H=%d)", B, H); return -1; }
  if (io_type == DT_F16) return probs_out<__half>(qkv, out, out_type, B, S, H, head_dim, causal, stream, seq_off);
  if (io_type == DT_BF16) return probs_out<__nv_bfloat16>(qkv, out, out_type, B, S, H, head_dim, causal, stream, seq_off);
  set_last_error("attn_probs: qkv dtype %d; the attention I/O is fp16 or bf16", io_type);
  return -1;
}

// ------------------------------------------------------------------------------------------
// MAP-head attention: one CTA (256 threads) per (sample, head); scores in smem; HBM-bound on K/V.
// ------------------------------------------------------------------------------------------
// PACKED: sample b is rows seq_off[b] .. seq_off[b + 1] - 1 of kv (S_arg: the longest sample, which the scores' smem is sized for)
template <typename T, typename OutT, bool PACKED = false>
__global__ void __launch_bounds__(256)
map_attention_kernel(const float* __restrict__ q, const T* __restrict__ kv, OutT* __restrict__ out, int S_arg, int H, int d, float qscale,
                     const int* __restrict__ seq_off, void* __restrict__ probs, int probs_type) {
  extern __shared__ float sm[];
  float* sq = sm;              // [128]
  float* red = sm + 128;       // [8 * 128] cross-group reduction / [8] block reductions
  float* sc = sm + 128 + 1024; // [S]
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int D = H * d;
  const size_t ld = static_cast<size_t>(2) * D;
  int S = S_arg;
  size_t row0 = static_cast<size_t>(b) * S_arg;
  if constexpr (PACKED) {
    row0 = static_cast<size_t>(seq_off[b]);
    S = seq_off[b + 1] - seq_off[b];
  }
  const T* kbase = kv + row0 * ld + h * d;
  const T* vbase = kbase + D;
  if (tid < d) sq[tid] = q[h * d + tid] * qscale;  // query / sqrt(depth)
  __syncthreads();
  // scores
  float lmax = -INFINITY;
  for (int s = tid; s < S; s += 256) {
    const uint4* kr = reinterpret_cast<const uint4*>(kbase + static_cast<size_t>(s) * ld);
    float acc = 0.f;
#pragma unroll 8
    for (int c = 0; c < d / 8; ++c) {
      const uint4 u = __ldg(kr + c);
      const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = fmaf(to_float(e[i]), sq[c * 8 + i], acc);
    }
    sc[s] = acc;
    lmax = fmaxf(lmax, acc);
  }
  lmax = warp_max(lmax);
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  float bmax = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) bmax = fmaxf(bmax, red[w]);
  __syncthreads();
  float lsum = 0.f;
  for (int s = tid; s < S; s += 256) {
    const float p = __expf(sc[s] - bmax);
    sc[s] = p;
    lsum += p;
  }
  lsum = warp_sum(lsum);
  if (lane == 0) red[warp] = lsum;
  __syncthreads();
  float bsum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) bsum += red[w];
  __syncthreads();
  if (probs) {  // the weights the output sums with, [B, H, 1, S]: sample b from element H * (its first token row) on
    const size_t pb = row0 * H + static_cast<size_t>(h) * S;
    for (int s = tid; s < S; s += 256) {
      const float p = sc[s] / bsum;
      if (probs_type == DT_F32) static_cast<float*>(probs)[pb + s] = p;
      else if (probs_type == DT_F16) static_cast<__half*>(probs)[pb + s] = __float2half_rn(p);
      else static_cast<__nv_bfloat16*>(probs)[pb + s] = __float2bfloat16_rn(p);
    }
  }
  // output: warp = key group, lane = dim pairs lane and lane + 32 (columns 2 lane, 2 lane + 1 and 64 more)
  float a[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int s = warp; s < S; s += 8) {
    const float p = sc[s];
    const uint32_t* vr = reinterpret_cast<const uint32_t*>(vbase + static_cast<size_t>(s) * ld);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (2 * (lane + 32 * j) < d) {
        const uint32_t u = __ldg(vr + lane + 32 * j);
        const T* e = reinterpret_cast<const T*>(&u);
        a[j][0] = fmaf(p, to_float(e[0]), a[j][0]);
        a[j][1] = fmaf(p, to_float(e[1]), a[j][1]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int c = 2 * (lane + 32 * j);
    if (c < d) {
      red[warp * 128 + c] = a[j][0];
      red[warp * 128 + c + 1] = a[j][1];
    }
  }
  __syncthreads();
  if (tid < d) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += red[w * 128 + tid];
    out[static_cast<size_t>(b) * D + h * d + tid] = from_float<OutT>(v / bsum);
  }
}

// The scores of a sample sit in shared memory after 128 + 1024 floats of probe and reductions: the longest sequence is what the
// device's opt-in shared memory per block holds (56960 tokens at the 227 KB of an H100).
static constexpr int kMapSmemFloats = 128 + 1024;
int map_attention_max_seq(int device, int* max_S) {
  int optin = 0;
  JIMM_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  *max_S = optin / static_cast<int>(sizeof(float)) - kMapSmemFloats;
  return 0;
}

// smem_max: the bytes of the longest sequence map_attention_max_seq allows on this device, which the kernel is opted in to once
template <typename T, typename OutT, bool PACKED>
static int map_launch_k(const float* q, const void* kv, void* out, int B, int S, int H, int d, cudaStream_t stream, const int* seq_off, void* probs,
                        int probs_type, int smem_max) {
  constexpr auto kernel = map_attention_kernel<T, OutT, PACKED>;
  const size_t smem = (kMapSmemFloats + S) * sizeof(float);
  if (smem > 48 * 1024) {
    if (int rc = smem_opt_in<kernel>(smem_max)) return rc;
  }
  const float qscale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(d)));  // 0.125f for d = 64
  kernel<<<dim3(H, B), 256, smem, stream>>>(q, static_cast<const T*>(kv), static_cast<OutT*>(out), S, H, d, qscale, seq_off, probs, probs_type);
  JIMM_LAUNCH_CHECK();
  return 0;
}

static int map_dispatch(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, cudaStream_t stream,
                        const int* seq_off, void* probs, int probs_type) {
  if (!head_dim_ok(head_dim)) { set_last_error("map_attention: head_dim %d is not a multiple of 8 in [8, 128]", head_dim); return -1; }
  if (B <= 0) return 0;
  int dev = 0, max_S = 0;
  JIMM_CUDA_CHECK(cudaGetDevice(&dev));
  if (int rc = map_attention_max_seq(dev, &max_S)) return rc;
  if (S > max_S) { set_last_error("map_attention: S=%d too large (the scores of a sample live in shared memory: at most %d tokens on device %d)", S, max_S, dev); return -1; }
  if (probs && probs_type != DT_F32 && probs_type != DT_F16 && probs_type != DT_BF16) {
    set_last_error("map_attention: probs dtype %d", probs_type);
    return -1;
  }
  const int smem_max = (kMapSmemFloats + max_S) * static_cast<int>(sizeof(float));
  return io_out_dispatch("map_attention", io_type, out_type, [&](auto io, auto o) {
    using T = typename decltype(io)::type;
    using OutT = typename decltype(o)::type;
    if (seq_off) return map_launch_k<T, OutT, true>(q, kv, out, B, S, H, head_dim, stream, seq_off, probs, probs_type, smem_max);
    return map_launch_k<T, OutT, false>(q, kv, out, B, S, H, head_dim, stream, nullptr, probs, probs_type, smem_max);
  });
}

int map_attention_run(const float* q, const void* kv, int io_type, void* out, int out_type, int B, int S, int H, int head_dim, cudaStream_t stream,
                      void* probs, int probs_type) {
  return map_dispatch(q, kv, io_type, out, out_type, B, S, H, head_dim, stream, nullptr, probs, probs_type);
}

int map_attention_packed_run(const float* q, const void* kv, int io_type, void* out, int out_type, const int* seq_off, int B, int max_S, int H,
                             int head_dim, cudaStream_t stream, void* probs, int probs_type) {
  if (!seq_off) { set_last_error("map_attention_packed: null seq_off"); return -1; }
  return map_dispatch(q, kv, io_type, out, out_type, B, max_S, H, head_dim, stream, seq_off, probs, probs_type);
}

}  // namespace jimm
