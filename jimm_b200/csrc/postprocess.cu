// Zero-shot / classification epilogue (SURVEY.md 8f.3): what the reference's examples do in JAX after the forward path.
//   examples/clip_inference.py:46-51   scores = logits[0]; softmax = exp(scores) / sum(exp(scores)); order = argsort(scores)[::-1]
//   examples/vit_inference.py:58       predicted = argmax(logits, -1)
//   SigLIP (sigmoid loss, models/siglip.py:169-174 logits + bias): per-pair probability = sigmoid(logit)
// One CTA per row of logits: probabilities (fp32, the example's un-shifted exp / sum) and the argmax (a block reduction); the full
// descending order of a row of up to 4096 columns is sorted in the same CTA's shared memory.  Wider rows are sorted in global
// scratch: 4096-key runs sorted in shared memory, then merged pairwise in global memory (merge path, one CTA per 2048 outputs).
// Integer outputs are exact, including ties: argsort is stable ascending and then reversed, so equal scores come out with the
// LARGER index first; argmax returns the first maximum.  Both follow from 64-bit keys (order_key << 32 | index): they are unique,
// so any correct descending sort of them is numpy's stable argsort reversed, and the maximum of (order_key, -index) is the first
// maximum.
#include <algorithm>

#include "../../include/jimm_b200.h"
#include "common.cuh"

namespace jimm {
namespace {

constexpr int kThreads = 256;
constexpr int kRunCols = 4096;                               // keys sorted in one CTA's shared memory (32 KB)
constexpr int kMergeItems = 8;                               // outputs per thread of a merge
constexpr int kMergeTile = kThreads * kMergeItems;           // outputs per merge CTA; divides 2 * kRunCols
constexpr size_t kScratchBytes = static_cast<size_t>(256) << 20;  // wide-row keys per group of rows (at least one row's)

static_assert((2 * kRunCols) % kMergeTile == 0, "a merge tile must not span two pairs of runs");

using u64 = unsigned long long;

// Monotonic map float -> uint32 (larger float = larger key); -0 is folded into +0 and every NaN into the canonical quiet NaN,
// which sorts above +inf (numpy / jnp sort NaN last in ascending order, i.e. first once reversed).
__device__ __forceinline__ uint32_t order_key(float v) {
  uint32_t u = __float_as_uint(v);
  if (v != v) u = 0x7fc00000u;
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Every real element's key is > 0 (the smallest, -inf, maps to 0x007fffff << 32), so 0 pads a run and sorts after it.
__device__ __forceinline__ u64 sort_key(const float* x, long long i) {
  return (static_cast<u64>(order_key(x[i])) << 32) | static_cast<uint32_t>(i);
}

// Bitonic sort of n (a power of two) keys in shared memory, descending, by the whole CTA.
__device__ void bitonic_sort_desc(u64* keys, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += kThreads) {
        const int l = i ^ j;
        if (l > i) {
          const u64 a = keys[i], b = keys[l];
          const bool desc = (i & k) == 0;
          if (desc ? a < b : a > b) {
            keys[i] = b;
            keys[l] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(kThreads) postprocess_kernel(const float* __restrict__ logits, int cols, int ld, int mode, float* __restrict__ probs,
                                                             int ldp, int32_t* __restrict__ order, int32_t* __restrict__ argmax, int npow2) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  u64* keys = reinterpret_cast<u64*>(smem_raw);  // [npow2] (key << 32 | index), sorted descending; only when order is set
  __shared__ float red[kThreads / 32];
  __shared__ u64 red_max[kThreads / 32];
  __shared__ float total;
  const int row = blockIdx.x, tid = threadIdx.x;
  const float* x = logits + static_cast<size_t>(row) * ld;

  // ---- probabilities ----
  if (probs) {
    float* p = probs + static_cast<size_t>(row) * ldp;
    if (mode == 1) {
      for (long long i = tid; i < cols; i += kThreads) p[i] = 1.0f / (1.0f + expf(-x[i]));
    } else {
      float s = 0.f;
      for (long long i = tid; i < cols; i += kThreads) s += expf(x[i]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if ((tid & 31) == 0) red[tid >> 5] = s;
      __syncthreads();
      if (tid == 0) {
        float t = 0.f;
        for (int w = 0; w < kThreads / 32; ++w) t += red[w];
        total = t;
      }
      __syncthreads();
      const float t = total;
      for (long long i = tid; i < cols; i += kThreads) p[i] = expf(x[i]) / t;
    }
  }

  // ---- argmax: maximum of (order_key, -index), i.e. the first maximum, and the first NaN of a row that has one ----
  if (argmax) {
    u64 best = 0;
    for (long long i = tid; i < cols; i += kThreads)
      best = max(best, (static_cast<u64>(order_key(x[i])) << 32) | (0xffffffffu - static_cast<uint32_t>(i)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((tid & 31) == 0) red_max[tid >> 5] = best;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kThreads / 32; ++w) best = max(best, red_max[w]);
      argmax[row] = static_cast<int32_t>(0xffffffffu - static_cast<uint32_t>(best & 0xffffffffu));
    }
  }
  if (!order) return;

  // ---- descending order of a row of at most kRunCols columns: bitonic sort of its keys in shared memory ----
  for (int i = tid; i < npow2; i += kThreads) keys[i] = i < cols ? sort_key(x, i) : 0ull;
  __syncthreads();
  bitonic_sort_desc(keys, npow2);
  for (int i = tid; i < cols; i += kThreads) order[static_cast<size_t>(row) * cols + i] = static_cast<int32_t>(keys[i] & 0xffffffffu);
}

// ---- wide rows: grid (runs, rows of the group) ----
// Run r of a row holds its columns [r * kRunCols, (r + 1) * kRunCols), sorted descending into keys[row * cols + ...].
__global__ void __launch_bounds__(kThreads) sort_runs_kernel(const float* __restrict__ logits, int cols, int ld, u64* __restrict__ keys_out) {
  __shared__ u64 keys[kRunCols];
  const float* x = logits + static_cast<size_t>(blockIdx.y) * ld;
  const long long base = static_cast<long long>(blockIdx.x) * kRunCols;
  const int n = static_cast<int>(min(static_cast<long long>(kRunCols), cols - base));
  for (int i = threadIdx.x; i < kRunCols; i += kThreads) keys[i] = i < n ? sort_key(x, base + i) : 0ull;
  __syncthreads();
  bitonic_sort_desc(keys, kRunCols);
  u64* out = keys_out + static_cast<size_t>(blockIdx.y) * cols + base;
  for (int i = threadIdx.x; i < n; i += kThreads) out[i] = keys[i];
}

// Merge path of two descending runs of unique keys: how many of the first k merged keys come from a[0, na).
__device__ __forceinline__ long long merge_split(const u64* a, long long na, const u64* b, long long nb, long long k) {
  long long lo = max(0ll, k - nb), hi = min(k, na);
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] > b[k - 1 - mid]) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// One merge pass over every row of the group (grid: (ceil(cols / kMergeTile), rows)): sorted runs of `width` keys, pairwise, into
// runs of 2 * width.  The CTA owns outputs [k0, k1) of one pair (width is a multiple of kMergeTile, so no tile spans two pairs):
// it finds where they start and end in both runs, stages those keys in shared memory, and each thread merges kMergeItems of them.
// The last pass writes the low words (the column indices) to `order` instead of keys to `dst`.
__global__ void __launch_bounds__(kThreads) merge_kernel(const u64* __restrict__ src, int cols, long long width, u64* __restrict__ dst,
                                                       int32_t* __restrict__ order) {
  __shared__ u64 tile[kMergeTile];
  __shared__ long long split[2];
  const int tid = threadIdx.x;
  const size_t row_off = static_cast<size_t>(blockIdx.y) * cols;
  const long long t0 = static_cast<long long>(blockIdx.x) * kMergeTile;
  const long long base = t0 / (2 * width) * (2 * width);
  const long long na = min(width, cols - base), nb = max(0ll, min(width, cols - base - na));
  const u64* a = src + row_off + base;
  const u64* b = a + na;
  const long long k0 = t0 - base, k1 = min(k0 + kMergeTile, na + nb);
  if (tid < 2) split[tid] = merge_split(a, na, b, nb, tid == 0 ? k0 : k1);
  __syncthreads();
  const long long i0 = split[0], j0 = k0 - i0;
  const int ta = static_cast<int>(split[1] - i0), n = static_cast<int>(k1 - k0);
  for (int i = tid; i < n; i += kThreads) tile[i] = i < ta ? a[i0 + i] : b[j0 + i - ta];
  __syncthreads();

  u64 out[kMergeItems];
  const int d = tid * kMergeItems;
  if (d < n) {
    const u64* sa = tile;
    const u64* sb = tile + ta;
    const int tb = n - ta;
    int ia = static_cast<int>(merge_split(sa, ta, sb, tb, d)), ib = d - ia;
#pragma unroll
    for (int m = 0; m < kMergeItems; ++m) {
      if (d + m < n) {
        const bool take_a = ib >= tb || (ia < ta && sa[ia] > sb[ib]);
        out[m] = take_a ? sa[ia++] : sb[ib++];
      }
    }
  }
  __syncthreads();  // every thread has read its inputs from the tile
  if (d < n) {
#pragma unroll
    for (int m = 0; m < kMergeItems; ++m)
      if (d + m < n) tile[d + m] = out[m];
  }
  __syncthreads();
  if (order) {
    int32_t* o = order + row_off + base + k0;
    for (int i = tid; i < n; i += kThreads) o[i] = static_cast<int32_t>(tile[i] & 0xffffffffu);
  } else {
    u64* o = dst + row_off + base + k0;
    for (int i = tid; i < n; i += kThreads) o[i] = tile[i];
  }
}

// Order of rows wider than kRunCols.  Keys live in scratch allocated in stream order for this call: one buffer when a single merge
// pass finishes the row, two (ping-pong) otherwise, for as many rows at a time as fit in kScratchBytes (at least one).
int sort_wide_rows(const float* logits, int rows, int cols, int ld, int32_t* order, cudaStream_t st) {
  int passes = 0;
  for (long long w = kRunCols; w < cols; w *= 2) ++passes;
  const size_t row_bytes = static_cast<size_t>(cols) * sizeof(u64) * (passes > 1 ? 2 : 1);
  const int group = static_cast<int>(std::min<size_t>(std::max<size_t>(kScratchBytes / row_bytes, 1), std::min(rows, 65535)));
  u64* scratch = nullptr;
  JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), group * row_bytes, st));
  u64* buf[2] = {scratch, passes > 1 ? scratch + static_cast<size_t>(group) * cols : nullptr};
  const unsigned runs = static_cast<unsigned>((static_cast<long long>(cols) + kRunCols - 1) / kRunCols);
  const unsigned tiles = static_cast<unsigned>((static_cast<long long>(cols) + kMergeTile - 1) / kMergeTile);
  auto run_group = [&](int r0, int g) -> int {
    JIMM_CUDA_CHECK(launch_k(sort_runs_kernel, dim3(runs, g), dim3(kThreads), 0, st, 1, false, logits + static_cast<size_t>(r0) * ld, cols, ld,
                             buf[0]));
    note_launch();
    int cur = 0;
    long long w = kRunCols;
    for (int p = 0; p < passes; ++p, w *= 2, cur ^= 1) {
      const bool last = p == passes - 1;
      JIMM_CUDA_CHECK(launch_k(merge_kernel, dim3(tiles, g), dim3(kThreads), 0, st, 1, false, buf[cur], cols, w, last ? nullptr : buf[cur ^ 1],
                               last ? order + static_cast<size_t>(r0) * cols : nullptr));
      note_launch();
    }
    return 0;
  };
  int rc = 0;
  for (int r0 = 0; r0 < rows && rc == 0; r0 += group) rc = run_group(r0, std::min(group, rows - r0));
  const cudaError_t fe = cudaFreeAsync(scratch, st);
  if (rc == 0 && fe != cudaSuccess) { set_last_error("cudaFreeAsync -> %s", cudaGetErrorString(fe)); return JIMM_ECUDA; }
  return rc;
}

}  // namespace
}  // namespace jimm

using namespace jimm;

extern "C" int jimm_postprocess(const float* logits, int rows, int cols, int ld, int mode, float* probs, int ldp, int32_t* order, int32_t* argmax,
                                void* stream) {
  if (rows < 0 || cols <= 0 || ld < cols || (probs && ldp < cols)) { set_last_error("bad shape rows=%d cols=%d ld=%d ldp=%d", rows, cols, ld, ldp); return JIMM_EINVAL; }
  if (mode != 0 && mode != 1) { set_last_error("mode must be 0 (softmax) or 1 (sigmoid), got %d", mode); return JIMM_EINVAL; }
  if (!logits) { set_last_error("null logits"); return JIMM_EINVAL; }
  if (rows == 0) return 0;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool wide = cols > kRunCols;
  int32_t* row_order = wide ? nullptr : order;  // a narrow row's order is sorted by the row's own CTA
  if (probs || argmax || row_order) {
    int npow2 = 1;
    if (row_order)
      while (npow2 < cols) npow2 <<= 1;
    const size_t smem = row_order ? static_cast<size_t>(npow2) * sizeof(unsigned long long) : 0;
    JIMM_CUDA_CHECK(launch_k(postprocess_kernel, dim3(rows), dim3(kThreads), smem, st, 1, false, logits, cols, ld, mode, probs, ldp, row_order,
                             argmax, npow2));
    note_launch();
  }
  if (order && wide) return sort_wide_rows(logits, rows, cols, ld, order, st);
  return 0;
}
