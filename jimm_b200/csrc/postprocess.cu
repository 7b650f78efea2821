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
#include <cfloat>
#include <vector>

#include "../../include/jimm_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "logits_tile.cuh"

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

struct KeyIsValue {
  __device__ __forceinline__ u64 operator()(u64 v) const { return v; }
};

// Bitonic sort of n (a power of two) keys in shared memory, descending by key(.), by the whole CTA.
template <typename Key = KeyIsValue>
__device__ void bitonic_sort_desc(u64* keys, int n, Key key = {}) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += kThreads) {
        const int l = i ^ j;
        if (l > i) {
          const u64 a = keys[i], b = keys[l];
          const bool desc = (i & k) == 0;
          if (desc ? key(a) < key(b) : key(a) > key(b)) {
            keys[i] = b;
            keys[l] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

// Softmax denominator of a row: sum of exp(x[i]), per-thread strided sums reduced by a shuffle tree per warp and the warps' sums in
// order by thread 0.  Called by the whole CTA; every thread gets the total.  zero_shot's probabilities and top_k's are both
// exp(x) / this sum, so they agree bit for bit.
__device__ __forceinline__ float row_exp_sum(const float* __restrict__ x, int cols, float* red, float* total) {
  const int tid = threadIdx.x;
  float s = 0.f;
  for (long long i = tid; i < cols; i += kThreads) s += expf(x[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    *total = t;
  }
  __syncthreads();
  return *total;
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
      const float t = row_exp_sum(x, cols, red, &total);
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

// ---- top-k: the first k entries of the descending order, selected without sorting the row ----
// A candidate is (float bits << 32 | column): the value as stored (-0 and NaN payloads included) and its column.  Its sort key is the
// order's (order_key << 32 | column), so candidates compare exactly like the full sort's keys; kPadCand (column 0xffffffff, never a
// real column) has key 0, below every real one.
constexpr int kSelectMaxK = 1024;   // largest k selected in shared memory; beyond it top_k takes the prefix of the full sort
constexpr int kRowCols = 32768;     // rows up to this wide are selected in one CTA from one read (128 KB of keys)
constexpr int kSegCols = 8192;      // wider rows: segments of this many columns, k candidates each, then one merge
constexpr u64 kPadCand = 0xffffffffull;

struct CandKey {
  __device__ __forceinline__ u64 operator()(u64 c) const {
    const uint32_t col = static_cast<uint32_t>(c & 0xffffffffu);
    return col == 0xffffffffu ? 0ull : (static_cast<u64>(order_key(__uint_as_float(static_cast<uint32_t>(c >> 32)))) << 32) | col;
  }
};

struct SelectSmem {
  uint32_t hist[kThreads / 32][256];  // one histogram per warp: fewer collisions on the shared atomics
  uint32_t digit, remaining;
  int count;
  float red[kThreads / 32], total;
};

// The k-th largest of n unique 64-bit keys key(i), 1 <= k <= n: one 8-bit digit per pass from the top, each pass a histogram of the
// keys that share the digits chosen so far.  Every key's low word (a column) is below 2^lo_bits, so the passes over its higher
// digits (all zero) are skipped.
template <typename Key>
__device__ u64 radix_select(Key key, long long n, int k, int lo_bits, SelectSmem& s) {
  static_assert(kThreads == 256, "one bin per thread");
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  u64 prefix = 0, mask = 0;
  uint32_t remaining = static_cast<uint32_t>(k);
  for (int shift = 56; shift >= 0; shift -= 8) {
    if (shift < 32 && shift >= lo_bits) continue;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) s.hist[w][tid] = 0;
    __syncthreads();
    for (long long i = tid; i < n; i += kThreads) {
      const u64 v = key(i);
      if ((v & mask) == prefix) atomicAdd(&s.hist[warp][(v >> shift) & 255], 1u);
    }
    __syncthreads();
    uint32_t t = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) t += s.hist[w][tid];
    __syncthreads();
    s.hist[0][tid] = t;
    __syncthreads();
    if (warp == 0) {  // lane l holds bins 255 - 8l down to 248 - 8l; find the bin where the count from the top reaches `remaining`
      uint32_t c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += (c[j] = s.hist[0][255 - 8 * lane - j]);
      uint32_t inc = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
      }
      uint32_t acc = inc - sum;
      if (acc < remaining && remaining <= inc) {
        int d = -1;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (d < 0) {
            if (acc + c[j] >= remaining) d = j;
            else acc += c[j];
          }
        }
        s.digit = 255 - 8 * lane - d;
        s.remaining = remaining - acc;
      }
    }
    __syncthreads();
    prefix |= static_cast<u64>(s.digit) << shift;
    mask |= 0xffull << shift;
    remaining = s.remaining;
  }
  return prefix;
}

// The candidates cand(i) of the keys key(i) >= kth (the min(n, k) best when kth is the k-th key, or every one when kth is 0) into
// surv[], padded with kPadCand to npow2 (a power of two >= k) and sorted descending.
template <typename Key, typename Cand>
__device__ void collect_sorted(Key key, Cand cand, long long n, u64 kth, int k, int npow2, u64* surv, SelectSmem& s) {
  if (threadIdx.x == 0) s.count = 0;
  __syncthreads();
  for (long long i = threadIdx.x; i < n; i += kThreads)
    if (key(i) >= kth) surv[atomicAdd(&s.count, 1)] = cand(i);
  for (long long i = min(n, static_cast<long long>(k)) + threadIdx.x; i < npow2; i += kThreads) surv[i] = kPadCand;
  __syncthreads();
  bitonic_sort_desc(surv, npow2, CandKey{});
}

// The first k sorted candidates of a row: as candidates into cand_out, or as values (the stored bits), columns and, when probs is
// set, exp(value) / total -- zero_shot's probability at that column.
__device__ void emit_row(const u64* surv, int k, u64* cand_out, float* values, int32_t* indices, float* probs, float total) {
  for (int i = threadIdx.x; i < k; i += kThreads) {
    const u64 c = surv[i];
    if (cand_out) {
      cand_out[i] = c;
    } else {
      const float v = __uint_as_float(static_cast<uint32_t>(c >> 32));
      values[i] = v;
      indices[i] = static_cast<int32_t>(c & 0xffffffffu);
      if (probs) probs[i] = expf(v) / total;
    }
  }
}

// grid (segments, rows): segment s of row r is the columns [s * seg, min((s + 1) * seg, cols)) of x's row r, numbered from col_base.
// Its keys are staged once in shared memory; its k best (all of them, padded, when it is narrower) go to cand + r * cand_ld + s * k,
// or -- cand null, one segment spanning the row -- straight to the row's outputs (row stride k).
__global__ void __launch_bounds__(kThreads) topk_segment_kernel(const float* __restrict__ logits, int cols, int ld, int seg, int k, int col_base,
                                                              int lo_bits, int npow2, u64* __restrict__ cand, long long cand_ld,
                                                              float* __restrict__ values, int32_t* __restrict__ indices, float* __restrict__ probs) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  u64* surv = reinterpret_cast<u64*>(smem_raw);                   // [npow2]
  uint32_t* keys = reinterpret_cast<uint32_t*>(surv + npow2);     // [seg]
  __shared__ SelectSmem s;
  const int row = blockIdx.y;
  const float* x = logits + static_cast<size_t>(row) * ld;
  const int c0 = blockIdx.x * seg;
  const int n = min(seg, cols - c0);
  for (int i = threadIdx.x; i < n; i += kThreads) keys[i] = order_key(x[c0 + i]);
  __syncthreads();
  const uint32_t base = static_cast<uint32_t>(col_base + c0);
  auto key = [&](long long i) { return (static_cast<u64>(keys[i]) << 32) | (base + static_cast<uint32_t>(i)); };
  auto cand_of = [&](long long i) { return (static_cast<u64>(__float_as_uint(x[c0 + i])) << 32) | (base + static_cast<uint32_t>(i)); };
  const u64 kth = n > k ? radix_select(key, n, k, lo_bits, s) : 0ull;
  collect_sorted(key, cand_of, n, kth, k, npow2, surv, s);
  if (cand) {
    emit_row(surv, k, cand + row * cand_ld + static_cast<long long>(blockIdx.x) * k, nullptr, nullptr, nullptr, 0.f);
  } else {
    const float t = probs ? row_exp_sum(x, cols, s.red, &s.total) : 0.f;
    const size_t o = static_cast<size_t>(row) * k;
    emit_row(surv, k, nullptr, values + o, indices + o, probs ? probs + o : nullptr, t);
  }
}

// grid (rows): the k best of the n candidates at cand + r * cand_ld (at least k of them real), to out_cand + r * cand_ld (which may
// be where they came from: every read is done before the first write) or, out_cand null, to the outputs (row stride k); probs
// need the logits row x (cols wide, stride ld) for the softmax denominator.
__global__ void __launch_bounds__(kThreads) topk_merge_kernel(const u64* cand, long long cand_ld, long long n, int k, int lo_bits, int npow2,
                                                            u64* out_cand, const float* __restrict__ logits, int cols, int ld,
                                                            float* __restrict__ values, int32_t* __restrict__ indices, float* __restrict__ probs) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  u64* surv = reinterpret_cast<u64*>(smem_raw);  // [npow2]
  __shared__ SelectSmem s;
  const int row = blockIdx.x;
  const u64* c = cand + row * cand_ld;
  auto key = [&](long long i) { return CandKey{}(c[i]); };
  auto cand_of = [&](long long i) { return c[i]; };
  collect_sorted(key, cand_of, n, radix_select(key, n, k, lo_bits, s), k, npow2, surv, s);
  if (out_cand) {
    emit_row(surv, k, out_cand + row * cand_ld, nullptr, nullptr, nullptr, 0.f);
  } else {
    const float t = probs ? row_exp_sum(logits + static_cast<size_t>(row) * ld, cols, s.red, &s.total) : 0.f;
    const size_t o = static_cast<size_t>(row) * k;
    emit_row(surv, k, nullptr, values + o, indices + o, probs ? probs + o : nullptr, t);
  }
}

// grid (rows): the first k columns of each row's full order (k > kSelectMaxK), with their values and probabilities.
__global__ void __launch_bounds__(kThreads) topk_gather_kernel(const int32_t* __restrict__ order, int cols, const float* __restrict__ logits, int ld,
                                                             int k, float* __restrict__ values, int32_t* __restrict__ indices, float* __restrict__ probs) {
  __shared__ float red[kThreads / 32], total;
  const int row = blockIdx.x;
  const float* x = logits + static_cast<size_t>(row) * ld;
  const float t = probs ? row_exp_sum(x, cols, red, &total) : 0.f;
  const size_t o = static_cast<size_t>(row) * k;
  for (int i = threadIdx.x; i < k; i += kThreads) {
    const int32_t j = order[static_cast<size_t>(row) * cols + i];
    const float v = x[j];
    values[o + i] = v;
    indices[o + i] = j;
    if (probs) probs[o + i] = expf(v) / t;
  }
}

int bit_width(long long cols) {  // bits of the largest column index, cols - 1
  int b = 0;
  while ((1ll << b) < cols) ++b;
  return b;
}

int pow2_at_least(int k) {
  int p = 1;
  while (p < k) p <<= 1;
  return p;
}

// Segment kernel over rows [0, rows) of `logits` in grid-sized groups; shared memory for `seg`-column segments and k survivors.
int launch_segments(const float* logits, int rows, int cols, int ld, int seg, int k, int col_base, int lo_bits, u64* cand, long long cand_ld,
                    float* values, int32_t* indices, float* probs, cudaStream_t st) {
  const int npow2 = pow2_at_least(k);
  const size_t smem = static_cast<size_t>(npow2) * sizeof(u64) + static_cast<size_t>(seg) * sizeof(uint32_t);
  if (const int rc = smem_opt_in<topk_segment_kernel>(kSelectMaxK * sizeof(u64) + kRowCols * sizeof(uint32_t))) return rc;
  const unsigned segs = static_cast<unsigned>((static_cast<long long>(cols) + seg - 1) / seg);
  for (int r0 = 0; r0 < rows; r0 += 65535) {
    const int g = std::min(65535, rows - r0);
    const size_t o = static_cast<size_t>(r0) * k;
    JIMM_CUDA_CHECK(launch_k(topk_segment_kernel, dim3(segs, g), dim3(kThreads), smem, st, 1, false, logits + static_cast<size_t>(r0) * ld, cols, ld,
                             seg, k, col_base, lo_bits, npow2, cand ? cand + r0 * cand_ld : nullptr, cand_ld, cand ? nullptr : values + o,
                             cand ? nullptr : indices + o, cand || !probs ? nullptr : probs + o));
    note_launch();
  }
  return 0;
}

int launch_merge(const u64* cand, int rows, long long cand_ld, long long n, int k, int lo_bits, u64* out_cand, const float* logits, int cols, int ld,
                 float* values, int32_t* indices, float* probs, cudaStream_t st) {
  const int npow2 = pow2_at_least(k);
  JIMM_CUDA_CHECK(launch_k(topk_merge_kernel, dim3(rows), dim3(kThreads), static_cast<size_t>(npow2) * sizeof(u64), st, 1, false, cand, cand_ld, n,
                           k, lo_bits, npow2, out_cand, logits, cols, ld, values, indices, probs));
  note_launch();
  return 0;
}

int free_scratch(void* p, cudaStream_t st, int rc) {
  const cudaError_t fe = cudaFreeAsync(p, st);
  if (rc == 0 && fe != cudaSuccess) { set_last_error("cudaFreeAsync -> %s", cudaGetErrorString(fe)); return JIMM_ECUDA; }
  return rc;
}

// The exact block step of a search: the scores of qn normalised queries nq against gn normalised gallery rows ng (gallery rows g0 ..
// g0 + gn - 1) through the contrastive head's logits kernel into `block` [qn, gn], reduced to k candidates per segment in each cand row
// after slot 0, and merged into slot 0, the row's running best k (first: there is none yet).  last: the merge writes values / indices
// (row stride k) instead.
constexpr int kSearchRows = 2048, kSearchCols = 32768;  // one score block: queries x gallery rows
static_assert(kSearchCols % kSegCols == 0 && kSearchCols >= kSelectMaxK, "a chunk is whole segments and holds k candidates");

int block_step(const float* nq, int qn, const float* ng, int gn, int g0, int E, const float* logit_scale, const float* logit_bias, int k, int lo,
               float* block, u64* cand, long long cand_ld, bool first, bool last, float* values, int32_t* indices, cudaStream_t st) {
  const long long segs = (gn + kSegCols - 1) / kSegCols;
  int rc = logits_run(nq, ng, logit_scale, logit_bias, block, qn, gn, E, gn, st);
  if (rc == 0) rc = launch_segments(block, qn, gn, gn, kSegCols, k, g0, lo, cand + k, cand_ld, nullptr, nullptr, nullptr, st);
  if (rc == 0)
    rc = launch_merge(first ? cand + k : cand, qn, cand_ld, (first ? 0 : k) + segs * k, k, lo, last ? nullptr : cand, nullptr, 0, 0,
                      last ? values : nullptr, last ? indices : nullptr, nullptr, st);
  return rc;
}

}  // namespace

int topk_run(const float* logits, int rows, int cols, int ld, int k, float* values, int32_t* indices, float* probs, cudaStream_t st) {
  if (k > kSelectMaxK) {  // the prefix of the full order, sorted in scratch for as many rows at a time as fit in kScratchBytes
    const int group = static_cast<int>(std::min<size_t>(std::max<size_t>(kScratchBytes / (static_cast<size_t>(cols) * sizeof(int32_t)), 1), rows));
    int32_t* order = nullptr;
    JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&order), static_cast<size_t>(group) * cols * sizeof(int32_t), st));
    int rc = 0;
    for (int r0 = 0; r0 < rows && rc == 0; r0 += group) {
      const int g = std::min(group, rows - r0);
      const float* x = logits + static_cast<size_t>(r0) * ld;
      const size_t o = static_cast<size_t>(r0) * k;
      rc = jimm_postprocess(x, g, cols, ld, 0, nullptr, cols, order, nullptr, st);
      if (rc == 0) {
        const cudaError_t e = launch_k(topk_gather_kernel, dim3(g), dim3(kThreads), 0, st, 1, false, order, cols, x, ld, k, values + o, indices + o,
                                       probs ? probs + o : nullptr);
        if (e != cudaSuccess) { set_last_error("topk_gather_kernel -> %s", cudaGetErrorString(e)); rc = JIMM_ECUDA; }
        else note_launch();
      }
    }
    return free_scratch(order, st, rc);
  }
  const int lo = bit_width(cols);
  if (cols <= kRowCols) return launch_segments(logits, rows, cols, ld, cols, k, 0, lo, nullptr, 0, values, indices, probs, st);
  // wider rows: k candidates per segment in scratch, for as many rows at a time as fit in kScratchBytes, then one merge per row
  const long long segs = (static_cast<long long>(cols) + kSegCols - 1) / kSegCols, cand_ld = segs * k;
  const size_t row_bytes = static_cast<size_t>(cand_ld) * sizeof(u64);
  const int group = static_cast<int>(std::min<size_t>(std::max<size_t>(kScratchBytes / row_bytes, 1), std::min(rows, 65535)));
  u64* cand = nullptr;
  JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&cand), group * row_bytes, st));
  int rc = 0;
  for (int r0 = 0; r0 < rows && rc == 0; r0 += group) {
    const int g = std::min(group, rows - r0);
    const float* x = logits + static_cast<size_t>(r0) * ld;
    const size_t o = static_cast<size_t>(r0) * k;
    rc = launch_segments(x, g, cols, ld, kSegCols, k, 0, lo, cand, cand_ld, nullptr, nullptr, nullptr, st);
    if (rc == 0) rc = launch_merge(cand, g, cand_ld, cand_ld, k, lo, nullptr, x, cols, ld, values + o, indices + o, probs ? probs + o : nullptr, st);
  }
  return free_scratch(cand, st, rc);
}

// Gallery search: the scores of a chunk of queries against a chunk of gallery rows are the contrastive head's own -- the same
// l2_normalize and logits kernels, so every score is the bit pattern model(x, t) holds at that (image, text) pair -- written to a
// bounded score block and reduced at once to k candidates per (query, segment).  Each query's candidate row holds its running best
// k in slot 0 and the current chunk's segments after it; one merge per gallery chunk folds them back into slot 0, and the last one
// writes the outputs.  Scratch is the same for every N: kSearchRows x (E + kSearchCols) floats, kSearchCols x E floats and
// kSearchRows x (1 + kSearchCols / kSegCols) x k candidates -- at most about 450 MB at E = 768 and k = 1024.  The block costs 8 bytes
// of memory traffic per score against 2E FMA flops, so the search stays bound by the FMAs.
int search_run(const float* queries, int Q, const float* gallery, int N, int E, const float* logit_scale, const float* logit_bias, int k,
               float* values, int32_t* indices, cudaStream_t st) {
  const int qc = std::min(Q, kSearchRows), gc = std::min(N, kSearchCols);
  const long long cand_ld = (1 + (gc + kSegCols - 1) / kSegCols) * static_cast<long long>(k);
  const size_t cand_bytes = (static_cast<size_t>(qc) * cand_ld * sizeof(u64) + 255) / 256 * 256;  // the float rows start 16-byte aligned
  const size_t floats = static_cast<size_t>(qc) * E + static_cast<size_t>(gc) * E + static_cast<size_t>(qc) * gc;
  u64* cand = nullptr;
  JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&cand), cand_bytes + floats * sizeof(float), st));
  float* nq = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(cand) + cand_bytes);
  float* ng = nq + static_cast<size_t>(qc) * E;
  float* block = ng + static_cast<size_t>(gc) * E;
  const int lo = bit_width(N);
  int rc = 0;
  for (int q0 = 0; q0 < Q && rc == 0; q0 += qc) {
    const int qn = std::min(qc, Q - q0);
    rc = l2_normalize_run(queries + static_cast<size_t>(q0) * E, nq, E, qn, E, st);
    for (int g0 = 0; g0 < N && rc == 0; g0 += gc) {
      const int gn = std::min(gc, N - g0);
      const size_t o = static_cast<size_t>(q0) * k;
      if (rc == 0) rc = l2_normalize_run(gallery + static_cast<size_t>(g0) * E, ng, E, gn, E, st);
      if (rc == 0)
        rc = block_step(nq, qn, ng, gn, g0, E, logit_scale, logit_bias, k, lo, block, cand, cand_ld, g0 == 0, N - g0 == gn, values + o,
                        indices + o, st);
    }
  }
  return free_scratch(cand, st, rc);
}

// ---- gallery index: normalised rows stored once, screened on the tensor cores in fp16, survivors rescored exactly ----
// A search gives the bits search_run gives for the same queries against every row added so far.  Per chunk of kSearchRows queries:
//   1. the queries are normalised by l2_normalize_run, and get an fp16 copy and a norm bound (prep_rows_kernel);
//   2. seed: the first min(N, kSearchCols) stored rows go through block_step, the exact block step of search_run, which gives each
//      query a running exact best k;
//   3. each query's threshold t_i (threshold_kernel) is a lower bound on the accumulator of any row that can still enter its best k;
//   4. the other rows are screened kScreenCols at a time by the fp16 GEMM with the screening epilogue (gemm.cu, which also derives the
//      bound delta on |fp16 wgmma sum - fp32 accumulator|): a row survives when a + delta >= t_i;
//   5. the survivors are rescored exactly (rescore_kernel: the fmaf chain and logit_value of logits_tile) and merged into the best k,
//      and t_i is recomputed, so later chunks are screened harder.  A query with more than kScreenCap survivors in a chunk falls back to
//      block_step on that chunk.
// Dropped rows provably score below the running k-th; every other row is scored by the logits kernel's own arithmetic, on the stored
// normalised rows -- the bits search_run computes -- so the result is search_run's.
namespace {

constexpr int kScreenCols = 65536;  // gallery rows per screen launch
constexpr int kScreenCap = 4096;    // survivors kept per query and screen chunk; more fall back to the exact block step
constexpr float kMaxBound = 1024.f;  // rows of larger norm are treated as non-finite (their fp16 copy could overflow)

// One warp per row of x (normalised, fp32 [n, E]): the fp16 copy h and bound[r] >= ||x_r||_2, the sum of squares taken in double (each
// square exact, E <= 8192 additions: relative error below 2^-39) and rounded up by 2^-30.  A row with a non-finite value or a norm above
// kMaxBound gets bound +inf and zeros in h: it passes every screen and is always scored exactly.
__global__ void __launch_bounds__(256) prep_rows_kernel(const float* __restrict__ x, int n, int E, __half* __restrict__ h,
                                                        float* __restrict__ bound) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* r = x + row * E;
  double s = 0.0;
  bool finite = true;
  for (int i = lane; i < E; i += 32) {
    const float v = r[i];
    finite = finite && isfinite(v);
    s += static_cast<double>(v) * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float nb = __double2float_ru(sqrt(s) * (1.0 + 0x1p-30));
  const bool ok = __all_sync(0xffffffffu, finite) && nb <= kMaxBound;
  __half* hr = h + row * E;
  for (int i = lane; i < E; i += 32) hr[i] = ok ? __float2half_rn(r[i]) : __float2half_rn(0.f);
  if (lane == 0) bound[row] = ok ? nb : INFINITY;
}

int prep_rows_run(const float* x, int n, int E, __half* h, float* bound, cudaStream_t st) {
  if (n <= 0) return 0;
  JIMM_CUDA_CHECK(launch_k(prep_rows_kernel, dim3(static_cast<unsigned>((n + 7) / 8)), dim3(256), 0, st, 1, false, x, n, E, h, bound));
  note_launch();
  return 0;
}

// t[i] for each of qn queries from its running k-th score s_k (slot k - 1 of its sorted candidate row).  A row enters the best k only if
// its score s = fl(sc acc + bs) (logit_value: one rounding) is >= s_k -- a tie enters too, since a later row has the larger index.
// Rounding to nearest is monotone, so s >= s_k needs sc acc + bs >= s_k - 2^-24 |s_k| - 2^-150, i.e. (sc > 0)
//   acc >= (s_k - bs) / sc - (2^-24 |s_k| + 2^-150) / sc.
// t = (s_k - bs) / sc - m in double, m = 2^-20 (|s_k| + |bs|) / sc + 2^-20, then rounded down to fp32.  The double arithmetic errs by
// under 2^-50 (|s_k| + |bs|) / sc, and with sc >= 2^-60 the 2^-150 / sc term is below 2^-90, so m covers both with room to spare and
// t <= that lower bound.  Non-finite s_k, with sc and bs finite:
//   * s_k = +inf: s = +inf needs sc acc + bs >= FLT_MAX, so s_k = FLT_MAX in the formula gives a valid (weaker) bound;
//   * s_k NaN (NaN ranks above every number, so the running best k is all NaN): a number can no longer enter, only another NaN score.
//     With sc and bs finite, fl(sc acc + bs) is NaN only if acc is, which needs a non-finite value in the query or the row; the index
//     gives such a row or query norm bound +inf, and delta is then +inf or NaN, which passes any t.  So t = +inf: only those rows survive;
//   * s_k = -inf: every row ties or beats it, t = -inf.
// If sc or bs is not finite, or sc < 2^-60, t = -inf: every row survives and the chunk goes exact.
// The same bound serves a fixed threshold (range search): a row is a hit only if its score is >= s_k := the threshold.
__device__ __forceinline__ float acc_lower_bound(float sk, float sc, float bs) {
  float ti = -INFINITY;
  if (isfinite(sc) && isfinite(bs)) {
    if (isnan(sk)) {
      ti = INFINITY;
    } else if (sk != -INFINITY && sc >= 0x1p-60f) {
      const double s = fmin(static_cast<double>(sk), static_cast<double>(FLT_MAX));
      const double a = fabs(s) + fabs(static_cast<double>(bs));
      const double td = (s - bs) / sc - (0x1p-20 * a / sc + 0x1p-20);
      ti = __double2float_rd(td);
    }
  }
  return ti;
}

__global__ void threshold_kernel(const u64* __restrict__ cand, long long cand_ld, int qn, int k, const float* __restrict__ logit_scale,
                                 const float* __restrict__ logit_bias, float* __restrict__ t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= qn) return;
  const float sk = __uint_as_float(static_cast<uint32_t>(cand[i * cand_ld + k - 1] >> 32));
  const float sc = expf(*logit_scale);
  const float bs = logit_bias ? *logit_bias : 0.f;
  t[i] = acc_lower_bound(sk, sc, bs);
}

// After a screen: per query whose list overflowed (cnt > cap) its index in ovl; info[0] = the largest count of the others, info[1] =
// the number of overflowed queries, info[2] = the others' counts summed.  One CTA.
__global__ void __launch_bounds__(1024) screen_info_kernel(const int* __restrict__ cnt, int qn, int cap, int* __restrict__ ovl, int* __restrict__ info) {
  __shared__ int smax, snov, ssum;
  if (threadIdx.x == 0) smax = snov = ssum = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < qn; i += blockDim.x) {
    const int c = cnt[i];
    if (c > cap) {
      ovl[atomicAdd(&snov, 1)] = i;
    } else if (c > 0) {
      atomicMax(&smax, c);
      atomicAdd(&ssum, c);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) { info[0] = smax; info[1] = snov; info[2] = ssum; }
}

// The exact score of normalised query row qrow (shared memory) against stored row grow: the fmaf chain over k ascending of
// logits_tile and logit_value with the same sc and bs as logits_kernel.
__device__ __forceinline__ float rescore_value(const float* qrow, const float* __restrict__ grow, int E, const float* __restrict__ logit_scale,
                                               const float* __restrict__ logit_bias) {
  const float4* g = reinterpret_cast<const float4*>(grow);  // E % 4 == 0 (checked by gallery_create)
  float acc = 0.f;
  for (int e = 0; e < E; e += 4) {
    const float4 v = __ldg(g + e / 4);
    acc = fmaf(qrow[e], v.x, acc);
    acc = fmaf(qrow[e + 1], v.y, acc);
    acc = fmaf(qrow[e + 2], v.z, acc);
    acc = fmaf(qrow[e + 3], v.w, acc);
  }
  if (E % 16 != 0) acc = fmaf(0.f, 0.f, acc);  // logits_tile's zero-padded last K step (turns a -0 into +0)
  const float sc = expf(*logit_scale);
  const float bs = logit_bias ? *logit_bias : 0.f;
  return logit_value(sc, acc, bs);
}

// grid (ceil(width / 128), qn): slot s < width of query i's candidates after its running best k.  A surviving row j of the chunk
// (list[i][s], s < cnt[i] <= cap) gets its exact score (rescore_value) as the candidate (score bits << 32 | g0 + j); other slots get
// kPadCand.
__global__ void __launch_bounds__(128) rescore_kernel(const float* __restrict__ nq, const float* __restrict__ ng, int E, const int* __restrict__ cnt,
                                                      const int* __restrict__ list, int cap, int width, int g0, const float* __restrict__ logit_scale,
                                                      const float* __restrict__ logit_bias, u64* __restrict__ cand, long long cand_ld, int k) {
  extern __shared__ __align__(16) float qrow[];  // [E]
  const int i = blockIdx.y;
  const float* q = nq + static_cast<size_t>(i) * E;
  for (int e = threadIdx.x; e < E; e += blockDim.x) qrow[e] = q[e];
  __syncthreads();
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= width) return;
  const int c = cnt[i];
  u64 out = kPadCand;
  if (c <= cap && s < c) {
    const int j = list[static_cast<size_t>(i) * cap + s];
    const float v = rescore_value(qrow, ng + static_cast<size_t>(j) * E, E, logit_scale, logit_bias);
    out = (static_cast<u64>(__float_as_uint(v)) << 32) | static_cast<uint32_t>(g0 + j);
  }
  cand[i * cand_ld + k + s] = out;
}

// grid (nover): copy overflowed query ovl[r]'s normalised row and running best k into row r of fq / fcand (to_chunk), or the best k back.
__global__ void __launch_bounds__(256) fallback_copy_kernel(const int* __restrict__ ovl, int E, int k, float* nq, float* fq, u64* cand,
                                                            long long cand_ld, u64* fcand, long long fcand_ld, int to_chunk) {
  const int r = blockIdx.x, i = ovl[r];
  if (to_chunk) {
    for (int e = threadIdx.x; e < E; e += blockDim.x) fq[static_cast<size_t>(r) * E + e] = nq[static_cast<size_t>(i) * E + e];
    for (int s = threadIdx.x; s < k; s += blockDim.x) fcand[r * fcand_ld + s] = cand[i * cand_ld + s];
  } else {
    for (int s = threadIdx.x; s < k; s += blockDim.x) cand[i * cand_ld + s] = fcand[r * fcand_ld + s];
  }
}

// ---- range search: every row whose score is >= a fixed threshold ----
constexpr int kRangeThreads = kThreads;  // bitonic_sort_desc strides by kThreads

struct KeyAscending {  // bitonic_sort_desc by this key sorts ascending
  __device__ __forceinline__ u64 operator()(u64 v) const { return ~v; }
};

// Exclusive prefix sum of v over the CTA (blockDim.x a multiple of 32, at most 1024), in thread order; *total gets the sum.  Every
// thread of the CTA calls it; *total may be read until the next call.
template <typename T>
__device__ T block_exclusive_scan(T v, T* warp_sums, T* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[w] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    T run = 0;
    for (int i = 0; i < nw; ++i) {
      const T s = warp_sums[i];
      warp_sums[i] = run;
      run += s;
    }
    *total = run;
  }
  __syncthreads();
  const T r = warp_sums[w] + x - v;
  __syncthreads();
  return r;
}

// t[i] = acc_lower_bound(threshold) for each of qn rows: a row whose accumulator is below t scores below the threshold.
__global__ void range_threshold_kernel(int qn, float threshold, const float* __restrict__ logit_scale, const float* __restrict__ logit_bias,
                                       float* __restrict__ t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= qn) return;
  t[i] = acc_lower_bound(threshold, expf(*logit_scale), logit_bias ? *logit_bias : 0.f);
}

// After a screen of gn rows, one CTA: each query's staging room pos[i] (exclusive prefix sum of cnt[i], or of gn when its list overflowed
// (cnt[i] > cap)), the overflowed queries in ascending order in ovl, info[0] = their number, info[1] = the summed room, info[2] = the
// summed counts of the others (rows rescored) and info[3] = the largest of those counts.
__global__ void __launch_bounds__(1024) range_info_kernel(const int* __restrict__ cnt, int qn, int cap, int gn, int* __restrict__ ovl,
                                                          int* __restrict__ pos, int* __restrict__ info) {
  __shared__ int warp_sums[32], total, smax;
  if (threadIdx.x == 0) smax = 0;
  __syncthreads();
  int room = 0, nover = 0, rescored = 0;
  for (int b = 0; b < qn; b += blockDim.x) {
    const int i = b + threadIdx.x;
    const int c = i < qn ? cnt[i] : 0;
    const bool over = c > cap;
    if (!over && c > 0) atomicMax(&smax, c);
    const int p = block_exclusive_scan(over ? gn : c, warp_sums, &total);
    if (i < qn) pos[i] = room + p;
    room += total;
    const int o = block_exclusive_scan(over ? 1 : 0, warp_sums, &total);
    if (over) ovl[nover + o] = i;
    nover += total;
    block_exclusive_scan(over ? 0 : c, warp_sums, &total);
    rescored += total;
  }
  if (threadIdx.x == 0) { info[0] = nover; info[1] = room; info[2] = rescored; info[3] = smax; }
}

// Keeps the hits of one round of blockDim.x candidates, in thread order: hit (score v, row j) goes to out[base + its rank].  Returns the
// round's number of hits.
__device__ __forceinline__ int keep_hits(bool hit, float v, int j, float* __restrict__ out_score, int32_t* __restrict__ out_index, long long base,
                                         int* warp_sums, int* total) {
  const int r = block_exclusive_scan(hit ? 1 : 0, warp_sums, total);
  if (hit) { out_score[base + r] = v; out_index[base + r] = j; }
  return *total;
}

// grid (qn): query i's screen survivors in chunk g0 (list[i][s], s < cnt[i] <= cap) sorted ascending in shared memory, scored by
// rescore_value, and those with score >= threshold -- and, pairs (row0 >= 0), stored row g0 + j > row0 + i -- written in row order to
// the staging at pos[i]; count[i] = their number.  An overflowed query (cnt[i] > cap) is left to range_block_kernel.
__global__ void __launch_bounds__(kRangeThreads) range_rescore_kernel(const float* __restrict__ nq, const float* __restrict__ ng, int E,
                                                                      const int* __restrict__ cnt, const int* __restrict__ list, int cap, int g0,
                                                                      int row0, float threshold, const float* __restrict__ logit_scale,
                                                                      const float* __restrict__ logit_bias, const int* __restrict__ pos,
                                                                      float* __restrict__ st_score, int32_t* __restrict__ st_index,
                                                                      int* __restrict__ count) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* qrow = reinterpret_cast<float*>(smem_raw);                  // [E]
  u64* keys = reinterpret_cast<u64*>(smem_raw + static_cast<size_t>(E) * sizeof(float));  // [npow2]: row, then score bits << 32 | row
  __shared__ int warp_sums[32], total;
  const int i = blockIdx.x;
  const int c = cnt[i];
  if (c > cap || c == 0) return;  // the block step takes an overflowed query; count[i] stays 0 for an empty one
  int npow2 = 1;
  while (npow2 < c) npow2 <<= 1;
  for (int e = threadIdx.x; e < E; e += blockDim.x) qrow[e] = nq[static_cast<size_t>(i) * E + e];
  for (int s = threadIdx.x; s < npow2; s += blockDim.x) keys[s] = s < c ? static_cast<u64>(list[static_cast<size_t>(i) * cap + s]) : ~0ull;
  __syncthreads();
  bitonic_sort_desc(keys, npow2, KeyAscending{});  // ascending rows, the padding (~0) last
  for (int s = threadIdx.x; s < c; s += blockDim.x) {
    const int j = static_cast<int>(keys[s]);
    const float v = rescore_value(qrow, ng + static_cast<size_t>(j) * E, E, logit_scale, logit_bias);
    keys[s] = (static_cast<u64>(__float_as_uint(v)) << 32) | static_cast<uint32_t>(j);
  }
  __syncthreads();
  long long base = pos[i];
  for (int s0 = 0; s0 < c; s0 += blockDim.x) {
    const int s = s0 + threadIdx.x;
    const u64 kv = s < c ? keys[s] : 0ull;
    const float v = __uint_as_float(static_cast<uint32_t>(kv >> 32));
    const int j = g0 + static_cast<int>(static_cast<uint32_t>(kv));
    const bool hit = s < c && v >= threshold && (row0 < 0 || j > row0 + i);
    base += keep_hits(hit, v, j, st_score, st_index, base, warp_sums, &total);
  }
  if (threadIdx.x == 0) count[i] = static_cast<int>(base - pos[i]);
}

// grid (nover): row r of the exact score block [nover, cols] (query ovl[r], stored rows col0 ..) -- the entries >= threshold, and for
// pairs (row0 >= 0) those of stored row col0 + c > row0 + ovl[r], in column order, appended to the query's staging after the count[i]
// hits its earlier pieces of the chunk left there.
__global__ void __launch_bounds__(kRangeThreads) range_block_kernel(const float* __restrict__ block, int cols, const int* __restrict__ ovl, int col0,
                                                                    int row0, float threshold, const int* __restrict__ pos,
                                                                    float* __restrict__ st_score, int32_t* __restrict__ st_index,
                                                                    int* __restrict__ count) {
  __shared__ int warp_sums[32], total;
  const int r = blockIdx.x, i = ovl[r];
  const float* x = block + static_cast<size_t>(r) * cols;
  long long base = static_cast<long long>(pos[i]) + count[i];
  for (int c0 = 0; c0 < cols; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x;
    const float v = c < cols ? x[c] : 0.f;
    const bool hit = c < cols && v >= threshold && (row0 < 0 || col0 + c > row0 + i);
    base += keep_hits(hit, v, col0 + c, st_score, st_index, base, warp_sums, &total);
  }
  if (threadIdx.x == 0) count[i] = static_cast<int>(base - pos[i]);
}

// One CTA, at the end of a query chunk: with count[c * qn + i] the hits of query i in gallery chunk c, offsets[i] = base + the hits of
// the queries before i (offsets[qn] = base + all of them) and dst[c * qn + i] = where the hits of (i, c) go: after offsets[i] and the
// query's hits in chunks before c.
__global__ void __launch_bounds__(1024) range_offsets_kernel(const int* __restrict__ count, int nch, int qn, long long base,
                                                             long long* __restrict__ offsets, long long* __restrict__ dst) {
  __shared__ long long warp_sums[32], total;
  long long run = base;
  for (int b = 0; b < qn; b += blockDim.x) {
    const int i = b + threadIdx.x;
    long long n = 0;
    if (i < qn)
      for (int c = 0; c < nch; ++c) n += count[static_cast<size_t>(c) * qn + i];
    const long long o = run + block_exclusive_scan(n, warp_sums, &total);
    if (i < qn) {
      offsets[i] = o;
      long long d = o;
      for (int c = 0; c < nch; ++c) {
        dst[static_cast<size_t>(c) * qn + i] = d;
        d += count[static_cast<size_t>(c) * qn + i];
      }
    }
    run += total;
  }
  if (threadIdx.x == 0) offsets[qn] = run;
}

// grid (qn): the count[i] staged hits of query i in one gallery chunk, from pos[i] to the result at dst[i] - base.
__global__ void __launch_bounds__(kRangeThreads) range_gather_kernel(const float* __restrict__ st_score, const int32_t* __restrict__ st_index,
                                                                     const int* __restrict__ pos, const int* __restrict__ count,
                                                                     const long long* __restrict__ dst, long long base, float* __restrict__ score,
                                                                     int32_t* __restrict__ index) {
  const int i = blockIdx.x, n = count[i];
  const long long from = pos[i], to = dst[i] - base;
  for (int s = threadIdx.x; s < n; s += blockDim.x) {
    score[to + s] = st_score[from + s];
    index[to + s] = st_index[from + s];
  }
}

// ---- removed rows and filters: a call runs over its allowed rows, the live rows it keeps, numbered 0 .. nA - 1 in ascending row order ----
// The screen GEMM and the exact kernels read those rows through a chunk buffer (gather_rows_kernel), so they run unchanged on
// positions, and the positions go back to row ids at the end: the map is monotone, so every order and tie rule carries over.
constexpr int kAllowRows = 8192;  // rows per CTA of the allowed-id passes: 256 threads, one 32-row word each

constexpr float kClusterBound = 2.f;  // k-means takes the rows whose norm bound is at most this: |x[e]| <= 2, so x[e] 2^30 fits 32 bits

// Bit b: row 32 w + b (< n) is live (live null: every row is), kept (keep null: every row is; else the byte is nonzero) and, bound
// non-null, clusterable (bound <= kClusterBound).
__device__ __forceinline__ uint32_t allowed_word(const uint32_t* __restrict__ live, const uint8_t* __restrict__ keep, const float* __restrict__ bound,
                                                 long long n, long long w) {
  const long long r0 = w * 32;
  if (r0 >= n) return 0u;
  const int nb = static_cast<int>(min(n - r0, 32ll));
  uint32_t m = live ? live[w] : 0xffffffffu;
  if (nb < 32) m &= (1u << nb) - 1u;
  if (keep) {
    uint32_t kb = 0;
    for (int b = 0; b < nb; ++b) kb |= (keep[r0 + b] ? 1u : 0u) << b;
    m &= kb;
  }
  if (bound) {
    uint32_t bb = 0;
    for (int b = 0; b < nb; ++b) bb |= (bound[r0 + b] <= kClusterBound ? 1u : 0u) << b;
    m &= bb;
  }
  return m;
}

// grid (ceil(n / kAllowRows)): count[b] = the allowed rows among block b's kAllowRows.
__global__ void __launch_bounds__(256) allowed_count_kernel(const uint32_t* __restrict__ live, const uint8_t* __restrict__ keep,
                                                            const float* __restrict__ bound, long long n, int* __restrict__ count) {
  __shared__ int warp_sums[32], total;
  const long long w = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  block_exclusive_scan(__popc(allowed_word(live, keep, bound, n, w)), warp_sums, &total);
  if (threadIdx.x == 0) count[blockIdx.x] = total;
}

// One CTA: start[b] = the allowed rows before block b (exclusive prefix sum of count over nb blocks), start[nb] = all of them.
__global__ void __launch_bounds__(1024) allowed_scan_kernel(const int* __restrict__ count, int nb, int* __restrict__ start) {
  __shared__ int warp_sums[32], total;
  int run = 0;
  for (int b0 = 0; b0 < nb; b0 += blockDim.x) {
    const int b = b0 + threadIdx.x;
    const int o = block_exclusive_scan(b < nb ? count[b] : 0, warp_sums, &total);
    if (b < nb) start[b] = run + o;
    run += total;
  }
  if (threadIdx.x == 0) start[nb] = run;
}

// grid as allowed_count_kernel: block b's allowed rows, ascending, to ids[start[b] ..].
__global__ void __launch_bounds__(256) allowed_scatter_kernel(const uint32_t* __restrict__ live, const uint8_t* __restrict__ keep,
                                                              const float* __restrict__ bound, long long n, const int* __restrict__ start,
                                                              int* __restrict__ ids) {
  __shared__ int warp_sums[32], total;
  const long long w = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  uint32_t m = allowed_word(live, keep, bound, n, w);
  int at = start[blockIdx.x] + block_exclusive_scan(__popc(m), warp_sums, &total);
  for (; m; m &= m - 1) ids[at++] = static_cast<int>(w * 32 + __ffs(m) - 1);
}

// One warp per row r < pn: stored row ids[r] -- its normalised fp32 row, fp16 copy and bound -- to row r of rows, half and bound, in
// 16-byte pieces (E % 8 == 0).
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ g_rows, const __half* __restrict__ g_half,
                                                          const float* __restrict__ g_bound, const int* __restrict__ ids, int pn, int E,
                                                          float* __restrict__ rows, __half* __restrict__ half, float* __restrict__ bound) {
  const int r = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= pn) return;
  const size_t j = static_cast<size_t>(ids[r]);
  const float4* fs = reinterpret_cast<const float4*>(g_rows + j * E);
  float4* fd = reinterpret_cast<float4*>(rows + static_cast<size_t>(r) * E);
  for (int e = lane; e < E / 4; e += 32) fd[e] = __ldg(fs + e);
  const uint4* hs = reinterpret_cast<const uint4*>(g_half + j * E);
  uint4* hd = reinterpret_cast<uint4*>(half + static_cast<size_t>(r) * E);
  for (int e = lane; e < E / 8; e += 32) hd[e] = __ldg(hs + e);
  if (lane == 0) bound[r] = g_bound[j];
}

// The outputs of a search over positions: index p < na becomes row ids[p]; a padding slot (index -1, from kPadCand, or any slot when
// na == 0) becomes (-inf, -1).
__global__ void __launch_bounds__(256) search_ids_kernel(float* __restrict__ values, int32_t* __restrict__ indices, long long n,
                                                         const int* __restrict__ ids, int na) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = indices[i];
  if (p >= 0 && p < na) {
    indices[i] = ids[p];
  } else {
    values[i] = -INFINITY;
    indices[i] = -1;
  }
}

// index[i] = ids[index[i]] for the n hits of a range search or pairs call over positions.
__global__ void __launch_bounds__(256) hits_ids_kernel(int32_t* __restrict__ index, long long n, const int* __restrict__ ids) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) index[i] = ids[index[i]];
}

// Pairs over positions, query rows q0 .. q0 + qn - 1 (offsets pos_off [qn + 1]), to stored rows lo .. lo + R - 1: the offset of row r
// is the one of the first position p with ids[p] >= r, so a row that is not allowed gets no hits.  R + 1 threads.
__global__ void __launch_bounds__(256) pairs_rows_kernel(const int* __restrict__ ids, int q0, int qn, int lo, int R,
                                                         const long long* __restrict__ pos_off, long long* __restrict__ row_off) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x > R) return;
  const long long r = static_cast<long long>(lo) + x;
  int a = q0, b = q0 + qn;  // lower bound of r in ids[q0 .. q0 + qn)
  while (a < b) {
    const int c = (a + b) >> 1;
    if (ids[c] < r) a = c + 1;
    else b = c;
  }
  row_off[x] = pos_off[a - q0];
}

// The ids of a removal, n of them: info[0] counts those outside [0, rows).
__global__ void __launch_bounds__(256) remove_check_kernel(const int* __restrict__ ids, int n, long long rows, unsigned long long* __restrict__ info) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (ids[i] < 0 || ids[i] >= rows)) atomicAdd(info, 1ull);
}

// Unless remove_check_kernel found a bad id (info[0] != 0): clears bit ids[i] of live, and info[1] counts the bits that were set.
__global__ void __launch_bounds__(256) remove_kernel(const int* __restrict__ ids, int n, uint32_t* __restrict__ live, unsigned long long* __restrict__ info) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || info[0] != 0) return;
  const uint32_t bit = 1u << (ids[i] & 31);
  if (atomicAnd(live + (ids[i] >> 5), ~bit) & bit) atomicAdd(info + 1, 1ull);
}

// old_to_new[ids[p]] = p for the na live rows (the others were set to -1).
__global__ void __launch_bounds__(256) compact_map_kernel(const int* __restrict__ ids, int na, int32_t* __restrict__ old_to_new) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < na) old_to_new[ids[p]] = p;
}

int alloc_async(void** p, size_t bytes, const char* what, cudaStream_t st) {
  const cudaError_t e = cudaMallocAsync(p, bytes, st);
  if (e == cudaSuccess) return 0;
  cudaGetLastError();
  *p = nullptr;
  set_last_error("index: %s of %zu bytes -> %s", what, bytes, cudaGetErrorString(e));
  return e == cudaErrorMemoryAllocation ? JIMM_ENOMEM : JIMM_ECUDA;
}

int launched(cudaError_t e, const char* what) {
  if (e == cudaSuccess) { note_launch(); return 0; }
  set_last_error("%s -> %s", what, cudaGetErrorString(e));
  return JIMM_ECUDA;
}

}  // namespace

struct GalleryStore {
  int E = 0;
  long long n = 0, cap = 0;
  float* rows = nullptr;   // [cap, E] normalised by l2_normalize_run: the bits search_run computes
  __half* half = nullptr;  // [cap, E] fp16 copy, the screen's B operand
  float* bound = nullptr;  // [cap] norm bounds (prep_rows_kernel)
  // Removed rows: bit r of live is clear.  The bitset exists from the first removal to the next compaction, [ceil(cap / 32)] words
  // with every bit past n set, so added rows are live as they are.  removed counts the clear bits below n.
  uint32_t* live = nullptr;
  long long removed = 0;
};

namespace {

long long live_words(long long rows) { return (rows + 31) / 32; }

// The ascending ids of the live rows that keep keeps (device bytes [n], nonzero keeps; null keeps every row) and, clusterable, whose
// norm bound is at most kClusterBound, in *ids, allocated in stream order for the caller to free (null when there are none), and their
// number in *na.  Waits for the stream once.
int allowed_ids(const GalleryStore* g, const uint8_t* keep, int** ids, int* na, cudaStream_t st, bool clusterable = false) {
  *ids = nullptr;
  *na = 0;
  if (g->n == 0) return 0;
  const int nb = static_cast<int>((g->n + kAllowRows - 1) / kAllowRows);
  int* count = nullptr;
  if (int rc = alloc_async(reinterpret_cast<void**>(&count), (2 * static_cast<size_t>(nb) + 1) * sizeof(int), "allowed-row counts", st)) return rc;
  int* start = count + nb;
  const float* bound = clusterable ? g->bound : nullptr;
  auto run = [&]() -> int {
    if (int e = launched(launch_k(allowed_count_kernel, dim3(nb), dim3(256), 0, st, 1, false, g->live, keep, bound, g->n, count), "allowed_count_kernel"))
      return e;
    if (int e = launched(launch_k(allowed_scan_kernel, dim3(1), dim3(1024), 0, st, 1, false, count, nb, start), "allowed_scan_kernel")) return e;
    JIMM_CUDA_CHECK(cudaMemcpyAsync(na, start + nb, sizeof(int), cudaMemcpyDeviceToHost, st));
    JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
    if (*na == 0) return 0;
    if (int e = alloc_async(reinterpret_cast<void**>(ids), static_cast<size_t>(*na) * sizeof(int), "allowed-row ids", st)) return e;
    return launched(launch_k(allowed_scatter_kernel, dim3(nb), dim3(256), 0, st, 1, false, g->live, keep, bound, g->n, start, *ids),
                    "allowed_scatter_kernel");
  };
  const int rc = run();
  if (rc != 0 && *ids) {
    cudaFreeAsync(*ids, st);
    *ids = nullptr;
  }
  return free_scratch(count, st, rc);
}

// Allowed rows p0 .. p0 + pn - 1 (ids[p0 ..]) into the chunk buffer rows / half / bound.
int gather_rows(const GalleryStore* g, const int* ids, int pn, float* rows, __half* half, float* bound, cudaStream_t st) {
  if (pn <= 0) return 0;
  return launched(launch_k(gather_rows_kernel, dim3(static_cast<unsigned>((pn + 7) / 8)), dim3(256), 0, st, 1, false, g->rows, g->half, g->bound,
                           ids, pn, g->E, rows, half, bound),
                  "gather_rows_kernel");
}

// The rows a search or range search reads: every stored row (ids null), or the allowed rows ids[0 .. n) through a chunk buffer of
// kScreenCols rows.  rows / half / bound point at positions p0 .. of the view after at(p0, pn).
struct RowView {
  const GalleryStore* g;
  const int* ids;
  int n;
  float* buf_rows;
  __half* buf_half;
  float* buf_bound;
  float* rows = nullptr;
  __half* half = nullptr;
  float* bound = nullptr;
  int at(int p0, int pn, cudaStream_t st) {
    if (!ids) {
      rows = g->rows + static_cast<size_t>(p0) * g->E;
      half = g->half + static_cast<size_t>(p0) * g->E;
      bound = g->bound + p0;
      return 0;
    }
    rows = buf_rows;
    half = buf_half;
    bound = buf_bound;
    return gather_rows(g, ids + p0, pn, buf_rows, buf_half, buf_bound, st);
  }
};

}  // namespace

int gallery_create(int E, GalleryStore** out) {
  if (E <= 0 || E % 8 != 0 || E > 1024 * 8) { set_last_error("index: embedding width %d must be a multiple of 8 in 8 .. 8192", E); return JIMM_EINVAL; }
  *out = new GalleryStore();
  (*out)->E = E;
  return 0;
}

long long gallery_rows(const GalleryStore* g) { return g->n; }

int gallery_width(const GalleryStore* g) { return g->E; }

int gallery_add(GalleryStore* g, const float* rows, int n, cudaStream_t st) {
  if (n <= 0) return 0;
  const int E = g->E;
  const long long need = g->n + n;
  if (need > g->cap) {  // grow geometrically: copy the stored rows over, free the old storage in stream order
    const long long cap = std::max(need, std::max(2 * g->cap, 1024ll));
    float* r = nullptr;
    __half* h = nullptr;
    float* b = nullptr;
    uint32_t* l = nullptr;
    auto fail = [&](cudaError_t e, const char* what) {
      cudaGetLastError();
      if (r) cudaFreeAsync(r, st);
      if (h) cudaFreeAsync(h, st);
      if (b) cudaFreeAsync(b, st);
      if (l) cudaFreeAsync(l, st);
      set_last_error("index: %s growing to %lld rows of width %d -> %s", what, cap, E, cudaGetErrorString(e));
      return e == cudaErrorMemoryAllocation ? JIMM_ENOMEM : JIMM_ECUDA;
    };
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&r), static_cast<size_t>(cap) * E * sizeof(float), st);
    if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void**>(&h), static_cast<size_t>(cap) * E * sizeof(__half), st);
    if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void**>(&b), static_cast<size_t>(cap) * sizeof(float), st);
    if (e == cudaSuccess && g->live) e = cudaMallocAsync(reinterpret_cast<void**>(&l), live_words(cap) * sizeof(uint32_t), st);
    if (e != cudaSuccess) return fail(e, "allocation");
    if (g->n > 0) {
      e = cudaMemcpyAsync(r, g->rows, static_cast<size_t>(g->n) * E * sizeof(float), cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(h, g->half, static_cast<size_t>(g->n) * E * sizeof(__half), cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(b, g->bound, static_cast<size_t>(g->n) * sizeof(float), cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) return fail(e, "copy");
    }
    if (l) {  // the new words live, then the old ones over them (their bits past n are set)
      e = cudaMemsetAsync(l, 0xff, live_words(cap) * sizeof(uint32_t), st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(l, g->live, live_words(g->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) return fail(e, "copy");
    }
    if (g->rows) {  // the new storage holds every row from here on
      cudaFreeAsync(g->rows, st);
      cudaFreeAsync(g->half, st);
      cudaFreeAsync(g->bound, st);
    }
    if (l) {
      cudaFreeAsync(g->live, st);
      g->live = l;
    }
    g->rows = r; g->half = h; g->bound = b; g->cap = cap;
  }
  constexpr int kPiece = 1 << 20;  // rows per l2_normalize_run (its warp index is an int)
  for (int r0 = 0; r0 < n; r0 += kPiece) {
    const int m = std::min(kPiece, n - r0);
    const size_t at = static_cast<size_t>(g->n + r0);
    if (int rc = l2_normalize_run(rows + static_cast<size_t>(r0) * E, g->rows + at * E, E, m, E, st)) return rc;
    if (int rc = prep_rows_run(g->rows + at * E, m, E, g->half + at * E, g->bound + at, st)) return rc;
  }
  g->n = need;
  return 0;
}

void gallery_destroy(GalleryStore* g) {
  if (!g) return;
  cudaDeviceSynchronize();  // cudaFree does not wait for the work still using stream-ordered allocations
  cudaFree(g->rows);
  cudaFree(g->half);
  cudaFree(g->bound);
  cudaFree(g->live);
  delete g;
}

long long gallery_live(const GalleryStore* g) { return g->n - g->removed; }

int gallery_remove(GalleryStore* g, const int* ids, int n, long long* removed, cudaStream_t st) {
  *removed = 0;
  if (n == 0) return 0;
  if (!g->live) {  // the first removal: every row live, and every bit past n set
    const long long words = live_words(g->cap);
    if (int rc = alloc_async(reinterpret_cast<void**>(&g->live), words * sizeof(uint32_t), "live bitset", st)) return rc;
    JIMM_CUDA_CHECK(cudaMemsetAsync(g->live, 0xff, words * sizeof(uint32_t), st));
  }
  unsigned long long* info = nullptr;
  if (int rc = alloc_async(reinterpret_cast<void**>(&info), 2 * sizeof(unsigned long long), "removal counts", st)) return rc;
  unsigned long long h[2] = {0, 0};
  auto run = [&]() -> int {
    JIMM_CUDA_CHECK(cudaMemsetAsync(info, 0, 2 * sizeof(unsigned long long), st));
    const dim3 grid((n + 255) / 256);
    if (int e = launched(launch_k(remove_check_kernel, grid, dim3(256), 0, st, 1, false, ids, n, g->n, info), "remove_check_kernel")) return e;
    if (int e = launched(launch_k(remove_kernel, grid, dim3(256), 0, st, 1, false, ids, n, g->live, info), "remove_kernel")) return e;
    JIMM_CUDA_CHECK(cudaMemcpyAsync(h, info, sizeof(h), cudaMemcpyDeviceToHost, st));
    JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
    if (h[0] != 0) {
      set_last_error("index remove: %llu of %d ids outside 0 .. %lld", h[0], n, g->n - 1);
      return JIMM_EINVAL;
    }
    return 0;
  };
  const int rc = free_scratch(info, st, run());
  if (rc == 0) {
    g->removed += static_cast<long long>(h[1]);
    *removed = static_cast<long long>(h[1]);
  }
  return rc;
}

int gallery_compact(GalleryStore* g, int32_t* old_to_new, cudaStream_t st) {
  const int E = g->E;
  int* ids = nullptr;
  int na = 0;
  if (g->removed == 0) {  // nothing to drop: the storage stays, the map is the identity
    if (old_to_new && g->n > 0) {
      if (int rc = allowed_ids(g, nullptr, &ids, &na, st)) return rc;
      const int rc = launched(launch_k(compact_map_kernel, dim3((na + 255) / 256), dim3(256), 0, st, 1, false, ids, na, old_to_new),
                              "compact_map_kernel");
      return free_scratch(ids, st, rc);
    }
    return 0;
  }
  if (int rc = allowed_ids(g, nullptr, &ids, &na, st)) return rc;
  float* r = nullptr;
  __half* h = nullptr;
  float* b = nullptr;
  auto run = [&]() -> int {
    if (na > 0) {
      if (int e = alloc_async(reinterpret_cast<void**>(&r), static_cast<size_t>(na) * E * sizeof(float), "compacted rows", st)) return e;
      if (int e = alloc_async(reinterpret_cast<void**>(&h), static_cast<size_t>(na) * E * sizeof(__half), "compacted fp16 rows", st)) return e;
      if (int e = alloc_async(reinterpret_cast<void**>(&b), static_cast<size_t>(na) * sizeof(float), "compacted bounds", st)) return e;
      constexpr int kPiece = 1 << 20;
      for (int p0 = 0; p0 < na; p0 += kPiece) {
        const size_t at = static_cast<size_t>(p0);
        if (int e = gather_rows(g, ids + p0, std::min(kPiece, na - p0), r + at * E, h + at * E, b + at, st)) return e;
      }
    }
    if (old_to_new) {
      JIMM_CUDA_CHECK(cudaMemsetAsync(old_to_new, 0xff, static_cast<size_t>(g->n) * sizeof(int32_t), st));
      if (na > 0)
        if (int e = launched(launch_k(compact_map_kernel, dim3((na + 255) / 256), dim3(256), 0, st, 1, false, ids, na, old_to_new),
                             "compact_map_kernel"))
          return e;
    }
    return 0;
  };
  const int rc = run();
  if (ids) cudaFreeAsync(ids, st);
  if (rc != 0) {  // the index stays as it was
    if (r) cudaFreeAsync(r, st);
    if (h) cudaFreeAsync(h, st);
    if (b) cudaFreeAsync(b, st);
    return rc;
  }
  cudaFreeAsync(g->rows, st);
  cudaFreeAsync(g->half, st);
  cudaFreeAsync(g->bound, st);
  cudaFreeAsync(g->live, st);
  g->rows = r; g->half = h; g->bound = b; g->live = nullptr;
  g->n = g->cap = na;
  g->removed = 0;
  return 0;
}

namespace {

// gallery_search over the N rows of a view: every stored row (ids null) or the allowed rows ids[0 .. N), whose positions the outputs
// then hold.  The queries are raw rows, normalised and prepared here, or (qrows non-null) rows already normalised with their fp16 copies
// and bounds, read through qrows in chunks of kSearchRows.  The first min(N, seed_cols) rows seed each chunk's best k exactly.
int search_rows(const GalleryStore* g, const int* ids, int N, const float* queries, RowView* qrows, int Q, int seed_cols, const float* logit_scale,
                const float* logit_bias, int k, float* values, int32_t* indices, long long* stats, cudaStream_t st) {
  const int E = g->E;
  const int qc = std::min(Q, kSearchRows), seed = std::min(N, seed_cols);
  const bool screen = N > seed;
  const long long seed_ld = k + (seed + kSegCols - 1) / kSegCols * static_cast<long long>(k);
  const long long cand_ld = screen ? k + std::max<long long>(kScreenCap, kSearchCols / kSegCols * static_cast<long long>(k)) : seed_ld;
  const long long fcand_ld = k + kSearchCols / kSegCols * static_cast<long long>(k);
  // scratch: 256-byte aligned pieces of one stream-ordered allocation
  size_t off = 0;
  auto piece = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) / 256 * 256; return at; };
  const size_t o_cand = piece(static_cast<size_t>(qc) * cand_ld * sizeof(u64));
  const size_t o_nq = qrows ? 0 : piece(static_cast<size_t>(qc) * E * sizeof(float));
  // the seed block, and with a screen the fallback's kSearchCols pieces
  const size_t o_block = piece(static_cast<size_t>(qc) * (screen ? std::min(N, kSearchCols) : seed) * sizeof(float));
  size_t o_fcand = 0, o_fq = 0, o_hq = 0, o_nbq = 0, o_t = 0, o_cnt = 0, o_ovl = 0, o_list = 0, o_info = 0;
  if (screen) {
    o_fcand = piece(static_cast<size_t>(qc) * fcand_ld * sizeof(u64));
    o_fq = piece(static_cast<size_t>(qc) * E * sizeof(float));
    o_hq = qrows ? 0 : piece(static_cast<size_t>(qc) * E * sizeof(__half));
    o_nbq = qrows ? 0 : piece(static_cast<size_t>(qc) * sizeof(float));
    o_t = piece(static_cast<size_t>(qc) * sizeof(float));
    o_cnt = piece(static_cast<size_t>(qc) * sizeof(int));
    o_ovl = piece(static_cast<size_t>(qc) * sizeof(int));
    o_list = piece(static_cast<size_t>(qc) * kScreenCap * sizeof(int));
    o_info = piece(4 * sizeof(int));
  }
  const int vc = ids ? std::min(N, kScreenCols) : 0;  // the view's chunk buffer
  const size_t o_vrows = piece(static_cast<size_t>(vc) * E * sizeof(float));
  const size_t o_vhalf = piece(static_cast<size_t>(vc) * E * sizeof(__half));
  const size_t o_vbound = piece(static_cast<size_t>(vc) * sizeof(float));
  uint8_t* base = nullptr;
  JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&base), off, st));
  RowView view{g, ids, N, reinterpret_cast<float*>(base + o_vrows), reinterpret_cast<__half*>(base + o_vhalf), reinterpret_cast<float*>(base + o_vbound)};
  u64* cand = reinterpret_cast<u64*>(base + o_cand);
  float* nq = qrows ? nullptr : reinterpret_cast<float*>(base + o_nq);
  float* block = reinterpret_cast<float*>(base + o_block);
  u64* fcand = reinterpret_cast<u64*>(base + o_fcand);
  float* fq = reinterpret_cast<float*>(base + o_fq);
  __half* hq = qrows ? nullptr : reinterpret_cast<__half*>(base + o_hq);
  float* nbq = qrows ? nullptr : reinterpret_cast<float*>(base + o_nbq);
  float* t = reinterpret_cast<float*>(base + o_t);
  int* cnt = reinterpret_cast<int*>(base + o_cnt);
  int* ovl = reinterpret_cast<int*>(base + o_ovl);
  int* list = reinterpret_cast<int*>(base + o_list);
  int* info = reinterpret_cast<int*>(base + o_info);
  GemmScreen sd;
  sd.t = t; sd.cnt = cnt; sd.list = list; sd.cap = kScreenCap;
  const int lo = bit_width(N);
  int rc = 0;
  auto threshold = [&](int qn) -> int {
    JIMM_CUDA_CHECK(launch_k(threshold_kernel, dim3((qn + 255) / 256), dim3(256), 0, st, 1, false, cand, cand_ld, qn, k, logit_scale, logit_bias, t));
    note_launch();
    return 0;
  };
  // Gallery rows g0 .. g0 + gn - 1 against the current qn queries: screen, rescore the survivors, send overflowed queries through the
  // exact block step, tighten the thresholds.  Every error is returned, so the caller frees the scratch.
  auto screen_chunk = [&](int qn, int g0) -> int {
    const int gn = std::min(kScreenCols, N - g0);
    if (int e = view.at(g0, gn, st)) return e;
    sd.ng = view.bound;
    JIMM_CUDA_CHECK(cudaMemsetAsync(cnt, 0, static_cast<size_t>(qn) * sizeof(int), st));
    if (int e = gemm_screen_run(hq, qn, view.half, gn, E, sd, st)) return e;
    JIMM_CUDA_CHECK(launch_k(screen_info_kernel, dim3(1), dim3(1024), 0, st, 1, false, cnt, qn, kScreenCap, ovl, info));
    note_launch();
    int h[3];
    JIMM_CUDA_CHECK(cudaMemcpyAsync(h, info, sizeof(h), cudaMemcpyDeviceToHost, st));
    JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
    const int width = h[0], nover = h[1];
    if (stats) { stats[0] += h[2]; stats[1] += nover; stats[2] += 1; }
    if (width > 0) {
      JIMM_CUDA_CHECK(launch_k(rescore_kernel, dim3((width + 127) / 128, qn), dim3(128), static_cast<size_t>(E) * sizeof(float), st, 1, false, nq,
                               view.rows, E, cnt, list, kScreenCap, width, g0, logit_scale, logit_bias, cand, cand_ld, k));
      note_launch();
      if (int e = launch_merge(cand, qn, cand_ld, k + width, k, lo, cand, nullptr, 0, 0, nullptr, nullptr, nullptr, st)) return e;
    }
    if (nover > 0) {  // those queries' chunk goes through the exact block step, in kSearchCols pieces
      JIMM_CUDA_CHECK(launch_k(fallback_copy_kernel, dim3(nover), dim3(256), 0, st, 1, false, ovl, E, k, nq, fq, cand, cand_ld, fcand, fcand_ld, 1));
      note_launch();
      for (int s0 = 0; s0 < gn; s0 += kSearchCols)
        if (int e = block_step(fq, nover, view.rows + static_cast<size_t>(s0) * E, std::min(kSearchCols, gn - s0), g0 + s0, E, logit_scale,
                               logit_bias, k, lo, block, fcand, fcand_ld, false, false, nullptr, nullptr, st))
          return e;
      JIMM_CUDA_CHECK(launch_k(fallback_copy_kernel, dim3(nover), dim3(256), 0, st, 1, false, ovl, E, k, nq, fq, cand, cand_ld, fcand, fcand_ld, 0));
      note_launch();
    }
    return width > 0 || nover > 0 ? threshold(qn) : 0;
  };
  for (int q0 = 0; q0 < Q && rc == 0; q0 += qc) {
    const int qn = std::min(qc, Q - q0);
    const size_t o = static_cast<size_t>(q0) * k;
    if (qrows) {
      rc = qrows->at(q0, qn, st);
      nq = qrows->rows;
      hq = qrows->half;
      nbq = qrows->bound;
    } else {
      rc = l2_normalize_run(queries + static_cast<size_t>(q0) * E, nq, E, qn, E, st);
    }
    if (rc == 0) rc = view.at(0, seed, st);
    if (rc == 0) rc = block_step(nq, qn, view.rows, seed, 0, E, logit_scale, logit_bias, k, lo, block, cand, cand_ld, true, !screen, values + o, indices + o, st);
    if (!screen) continue;
    if (rc == 0 && !qrows) rc = prep_rows_run(nq, qn, E, hq, nbq, st);
    sd.nq = nbq;
    if (rc == 0) rc = threshold(qn);
    for (int g0 = seed; g0 < N && rc == 0; g0 += kScreenCols) rc = screen_chunk(qn, g0);
    if (rc == 0) rc = launch_merge(cand, qn, cand_ld, k, k, lo, nullptr, nullptr, 0, 0, values + o, indices + o, nullptr, st);
  }
  return free_scratch(base, st, rc);
}

}  // namespace

int gallery_search(const GalleryStore* g, const float* queries, int Q, const float* logit_scale, const float* logit_bias, int k, const uint8_t* keep,
                   float* values, int32_t* indices, long long* stats, cudaStream_t st) {
  if (!keep && g->removed == 0)
    return search_rows(g, nullptr, static_cast<int>(g->n), queries, nullptr, Q, kSearchCols, logit_scale, logit_bias, k, values, indices, stats, st);
  // over the allowed rows' positions, then to row ids; with fewer than k of them the slots past the last are padding
  int* ids = nullptr;
  int na = 0;
  if (int rc = allowed_ids(g, keep, &ids, &na, st)) return rc;
  int rc = na == 0 ? 0 : search_rows(g, ids, na, queries, nullptr, Q, kSearchCols, logit_scale, logit_bias, k, values, indices, stats, st);
  const long long n = static_cast<long long>(Q) * k;
  if (rc == 0 && n > 0)
    rc = launched(launch_k(search_ids_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st, 1, false, values, indices, n, ids, na),
                  "search_ids_kernel");
  return ids ? free_scratch(ids, st, rc) : rc;
}

// ---- k-means: spherical k-means over the clusterable rows (allowed, norm bound <= kClusterBound) ----
// Assignment is a gallery search at k = 1 with the roles turned: the rows are the queries (already normalised, with fp16 copies and
// bounds) and the centroids a small gallery, normalised and prepared once per step, seeded exactly by their first kKmeansSeedCols and
// screened beyond.  Scores are logit_value(1, acc, 0): a device 0.0f as logit_scale (expf(0) = 1) and no bias.  The update sums the rows
// of each cluster in fixed point, S[j][e] = sum rint(x[e] 2^30) in int64, so every order of the sums gives the same integers, and the
// mean is fp32(fp64(S) 2^-30 / n_j).
namespace {

constexpr int kKmeansSeedCols = 256;  // centroids scored exactly before the screen: the threshold's seed
constexpr int kSumRows = 64;          // sorted rows per CTA of kmeans_sum_kernel

// splitmix64's first output for the state x: the mix of x + the golden-ratio increment.
__device__ __forceinline__ u64 splitmix64(u64 x) {
  u64 z = x + 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// keys[p] = 1 + (splitmix64(seed + id) >> 41) 2^-23 for the clusterable row id = ids[p] (ids null: p): a float in [1, 2).
__global__ void __launch_bounds__(256) kmeans_keys_kernel(const int* __restrict__ ids, int na, u64 seed, float* __restrict__ keys) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= na) return;
  const u64 id = static_cast<u64>(ids ? ids[p] : p);
  keys[p] = __uint_as_float(0x3f800000u | static_cast<uint32_t>(splitmix64(seed + id) >> 41));
}

// One warp per cluster j < C: stored row sel[j] (through map when non-null) into m[j], if it is a clusterable row of the n stored rows;
// otherwise *bad counts it and m[j] is not written.
__global__ void __launch_bounds__(256) kmeans_gather_kernel(const int* __restrict__ sel, const int* __restrict__ map, int C, const float* __restrict__ rows,
                                                            const float* __restrict__ bound, const uint32_t* __restrict__ live,
                                                            const uint8_t* __restrict__ keep, long long n, int E, float* __restrict__ m,
                                                            int* __restrict__ bad) {
  const int j = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (j >= C) return;
  long long id = sel[j];
  if (map && id >= 0) id = map[id];
  const bool ok = id >= 0 && id < n && (!live || ((live[id >> 5] >> (id & 31)) & 1u)) && (!keep || keep[id]) && bound[id] <= kClusterBound;
  if (!ok) {
    if (lane == 0) atomicAdd(bad, 1);
    return;
  }
  const float4* s = reinterpret_cast<const float4*>(rows + static_cast<size_t>(id) * E);
  float4* d = reinterpret_cast<float4*>(m + static_cast<size_t>(j) * E);
  for (int e = lane; e < E / 4; e += 32) d[e] = s[e];
}

// One warp per centroid j < C of c (l2_normalize of m_new).  If one of its values is not finite: m_old null (the initial centroids), *bad
// counts it; otherwise the cluster keeps its previous mean and centroid: m_new[j] = m_old[j], c[j] = c_old[j].
__global__ void __launch_bounds__(256) kmeans_finite_kernel(float* __restrict__ c, int C, int E, float* __restrict__ m_new, const float* __restrict__ m_old,
                                                            const float* __restrict__ c_old, int* __restrict__ bad) {
  const int j = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (j >= C) return;
  const size_t r = static_cast<size_t>(j) * E;
  bool finite = true;
  for (int e = lane; e < E; e += 32) finite = finite && isfinite(c[r + e]);
  if (__all_sync(0xffffffffu, finite)) return;
  if (!m_old) {
    if (lane == 0) atomicAdd(bad, 1);
    return;
  }
  for (int e = lane; e < E; e += 32) {
    m_new[r + e] = m_old[r + e];
    c[r + e] = c_old[r + e];
  }
}

// *changed += the positions p < n where a[p] != b[p].
__global__ void __launch_bounds__(256) kmeans_changed_kernel(const int32_t* __restrict__ a, const int32_t* __restrict__ b, int n, int* __restrict__ changed) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int d = __syncthreads_count(p < n && a[p] != b[p]);
  if (threadIdx.x == 0 && d > 0) atomicAdd(changed, d);
}

// Called by every lane of the warp: the lanes holding the same cluster j >= 0 add their number to at[j] with one atomic, so a large
// cluster does not serialise the warp on one address.  Returns this lane's slot: the old at[j] + its rank among those lanes (lanes
// with j < 0 add nothing).
template <typename T>
__device__ __forceinline__ T warp_claim(T* at, int j) {
  const unsigned peers = __match_any_sync(0xffffffffu, j);
  const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
  T base = 0;
  if (lane == leader && j >= 0) base = atomicAdd(at + j, static_cast<T>(__popc(peers)));
  base = __shfl_sync(peers, base, leader);
  return base + static_cast<T>(__popc(peers & ((1u << lane) - 1u)));
}

// n[a[p]] += 1 for each position p < na.
__global__ void __launch_bounds__(256) kmeans_count_kernel(const int32_t* __restrict__ a, int na, int* __restrict__ n) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  warp_claim(n, p < na ? a[p] : -1);
}

// Counting sort of the positions by cluster: order[cursor[a[p]]++] = p (cursor starts at each cluster's first slot).
__global__ void __launch_bounds__(256) kmeans_order_kernel(const int32_t* __restrict__ a, int na, int* __restrict__ cursor, int* __restrict__ order) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = p < na ? a[p] : -1;
  const int slot = warp_claim(cursor, j);
  if (j >= 0) order[slot] = p;
}

// S[j][e] += rint(x[e] 2^30) over the rows x of cluster j, for kSumRows positions of order per CTA (sorted by cluster): each thread sums
// its elements of a run of one cluster in an int64 and adds it with one atomic when the cluster changes.  x[e] 2^30 is exact (a power
// of two scaling) and |x[e]| <= 2, so each term fits 32 bits and each sum stays below 2^62; integer sums do not depend on their order.
__global__ void __launch_bounds__(256) kmeans_sum_kernel(const int* __restrict__ order, const int32_t* __restrict__ a, const int* __restrict__ ids,
                                                         const float* __restrict__ rows, int E, int na, unsigned long long* __restrict__ S) {
  __shared__ int srow[kSumRows], sj[kSumRows];
  const int r0 = blockIdx.x * kSumRows, nr = min(kSumRows, na - r0);
  for (int r = threadIdx.x; r < nr; r += blockDim.x) {
    const int p = order[r0 + r];
    sj[r] = a[p];
    srow[r] = ids ? ids[p] : p;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    long long acc = 0;
    int cur = sj[0];
    for (int r = 0; r < nr; ++r) {
      if (sj[r] != cur) {
        atomicAdd(S + static_cast<size_t>(cur) * E + e, static_cast<unsigned long long>(acc));
        acc = 0;
        cur = sj[r];
      }
      acc += __float2ll_rn(rows[static_cast<size_t>(srow[r]) * E + e] * 0x1p30f);
    }
    atomicAdd(S + static_cast<size_t>(cur) * E + e, static_cast<unsigned long long>(acc));
  }
}

// m_new = fp32_rn(fp64_rn(S) 2^-30 / fp64(n_j)) for the clusters with rows; the others keep m_old.
__global__ void __launch_bounds__(256) kmeans_mean_kernel(const long long* __restrict__ S, const int* __restrict__ n, const float* __restrict__ m_old,
                                                          float* __restrict__ m_new, int C, int E) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(C) * E) return;
  const int cnt = n[i / E];
  m_new[i] = cnt > 0 ? __double2float_rn(__ddiv_rn(__ll2double_rn(S[i]) * 0x1p-30, static_cast<double>(cnt))) : m_old[i];
}

// Every stored row r < n: assign -1, score -inf (the rows that take no part keep these).
__global__ void __launch_bounds__(256) kmeans_clear_kernel(int32_t* __restrict__ assign, float* __restrict__ scores, long long n) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n) return;
  assign[r] = -1;
  scores[r] = -INFINITY;
}

// Position p < na to its row id = ids[p] (ids null: p): assign and score, and counts[a[p]] += 1.
__global__ void __launch_bounds__(256) kmeans_out_kernel(const int32_t* __restrict__ a, const float* __restrict__ v, const int* __restrict__ ids, int na,
                                                         int32_t* __restrict__ assign, float* __restrict__ scores, unsigned long long* __restrict__ counts) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = p < na ? a[p] : -1;
  warp_claim(counts, j);
  if (j < 0) return;
  const int id = ids ? ids[p] : p;
  assign[id] = j;
  scores[id] = v[p];
}

unsigned blocks_of(long long n, int per) { return static_cast<unsigned>((n + per - 1) / per); }

}  // namespace

int gallery_kmeans(const GalleryStore* g, int C, const float* init_vectors, const int32_t* init_ids, unsigned long long seed, int iters,
                   const uint8_t* keep, float* centroids, int32_t* assign, float* scores, int64_t* counts, int* iterations, long long* stats,
                   cudaStream_t st) {
  const int E = g->E;
  const long long rows = g->n;
  const bool sampled = !init_vectors && !init_ids;
  // the clusterable rows' ids; when that is every stored row, positions are row ids and the rows are read in place
  int* ids = nullptr;
  int na = 0;
  if (int rc = allowed_ids(g, keep, &ids, &na, st, true)) return rc;
  if (ids && na == rows) {
    cudaFreeAsync(ids, st);
    ids = nullptr;
  }
  if (sampled && C > na) {
    set_last_error("index kmeans: %d clusters sampled from %d clusterable rows", C, na);
    return ids ? free_scratch(ids, st, JIMM_EINVAL) : JIMM_EINVAL;
  }
  const size_t CE = static_cast<size_t>(C) * E, NA = static_cast<size_t>(na);
  const int qc = std::min(std::max(na, 1), kSearchRows);
  size_t off = 0;
  auto piece = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) / 256 * 256; return at; };
  const size_t o_S = piece(CE * sizeof(long long));
  const size_t o_m = piece(2 * CE * sizeof(float));
  const size_t o_c = piece(2 * CE * sizeof(float));
  const size_t o_ch = piece(CE * sizeof(__half));
  const size_t o_cb = piece(static_cast<size_t>(C) * sizeof(float));
  const size_t o_n = piece((3 * static_cast<size_t>(C) + 1) * sizeof(int));  // n [C], start [C + 1], cursor [C]
  const size_t o_a = piece(2 * NA * sizeof(int32_t));
  const size_t o_v = piece(NA * sizeof(float));
  const size_t o_ord = piece(NA * sizeof(int));
  const size_t o_keys = piece(sampled ? NA * sizeof(float) : 0);
  const size_t o_sel = piece(sampled ? 2 * static_cast<size_t>(C) * sizeof(int) : 0);
  const size_t o_qr = piece(ids ? static_cast<size_t>(qc) * E * sizeof(float) : 0);
  const size_t o_qh = piece(ids ? static_cast<size_t>(qc) * E * sizeof(__half) : 0);
  const size_t o_qb = piece(ids ? static_cast<size_t>(qc) * sizeof(float) : 0);
  const size_t o_info = piece(4 * sizeof(int));  // zero (the logit_scale 0.0f), bad ids, bad vectors, changed
  uint8_t* base = nullptr;
  if (int rc = alloc_async(reinterpret_cast<void**>(&base), off, "k-means scratch", st)) return ids ? free_scratch(ids, st, rc) : rc;
  long long* S = reinterpret_cast<long long*>(base + o_S);
  float* m[2] = {reinterpret_cast<float*>(base + o_m), reinterpret_cast<float*>(base + o_m) + CE};
  float* c[2] = {reinterpret_cast<float*>(base + o_c), reinterpret_cast<float*>(base + o_c) + CE};
  __half* ch = reinterpret_cast<__half*>(base + o_ch);
  float* cb = reinterpret_cast<float*>(base + o_cb);
  int* n = reinterpret_cast<int*>(base + o_n);
  int* start = n + C;
  int* cursor = start + C + 1;
  int32_t* abuf = reinterpret_cast<int32_t*>(base + o_a);
  float* vals = reinterpret_cast<float*>(base + o_v);
  int* order = reinterpret_cast<int*>(base + o_ord);
  float* keys = reinterpret_cast<float*>(base + o_keys);
  int* sel = reinterpret_cast<int*>(base + o_sel);
  int* info = reinterpret_cast<int*>(base + o_info);
  const float* zero = reinterpret_cast<const float*>(info);
  RowView qv{g, ids, na, reinterpret_cast<float*>(base + o_qr), reinterpret_cast<__half*>(base + o_qh), reinterpret_cast<float*>(base + o_qb)};
  auto run = [&]() -> int {
    JIMM_CUDA_CHECK(cudaMemsetAsync(info, 0, 4 * sizeof(int), st));
    // m_0 and c_0, checked on the device
    if (init_vectors) {
      JIMM_CUDA_CHECK(cudaMemcpyAsync(m[0], init_vectors, CE * sizeof(float), cudaMemcpyDeviceToDevice, st));
    } else {
      const int* from = init_ids;
      const int* map = nullptr;
      if (sampled) {  // the rows at the positions of top_k(keys, C), ties to the larger position
        if (int e = launched(launch_k(kmeans_keys_kernel, dim3(blocks_of(na, 256)), dim3(256), 0, st, 1, false, ids, na, seed, keys),
                             "kmeans_keys_kernel"))
          return e;
        if (int e = topk_run(keys, 1, na, na, C, reinterpret_cast<float*>(sel + C), sel, nullptr, st)) return e;
        from = sel;
        map = ids;
      }
      if (int e = launched(launch_k(kmeans_gather_kernel, dim3(blocks_of(C, 8)), dim3(256), 0, st, 1, false, from, map, C, g->rows, g->bound, g->live,
                                    keep, rows, E, m[0], info + 1),
                           "kmeans_gather_kernel"))
        return e;
    }
    if (int e = l2_normalize_run(m[0], c[0], E, C, E, st)) return e;
    if (int e = launched(launch_k(kmeans_finite_kernel, dim3(blocks_of(C, 8)), dim3(256), 0, st, 1, false, c[0], C, E, nullptr, nullptr, nullptr,
                                  info + 2),
                         "kmeans_finite_kernel"))
      return e;
    int h[2];
    JIMM_CUDA_CHECK(cudaMemcpyAsync(h, info + 1, sizeof(h), cudaMemcpyDeviceToHost, st));
    JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
    if (h[0] != 0) {
      set_last_error("index kmeans: %d of %d init ids are not clusterable rows (live, kept, finite and not zero)", h[0], C);
      return JIMM_EINVAL;
    }
    if (h[1] != 0) {
      set_last_error("index kmeans: %d of %d initial centroids have a non-finite l2_normalize", h[1], C);
      return JIMM_EINVAL;
    }
    int cur = 0, t = 0;
    for (;; ++t) {
      int32_t* a = abuf + (t & 1) * NA;
      int32_t* prev = abuf + ((t + 1) & 1) * NA;
      if (int e = prep_rows_run(c[cur], C, E, ch, cb, st)) return e;
      GalleryStore cs;
      cs.E = E; cs.n = C; cs.cap = C; cs.rows = c[cur]; cs.half = ch; cs.bound = cb;
      if (na > 0)
        if (int e = search_rows(&cs, nullptr, C, nullptr, &qv, na, kKmeansSeedCols, zero, nullptr, 1, vals, a, stats, st)) return e;
      if (t + 1 == iters) break;
      if (t > 0) {
        int changed = 0;
        if (na > 0 && launched(launch_k(kmeans_changed_kernel, dim3(blocks_of(na, 256)), dim3(256), 0, st, 1, false, a, prev, na, info + 3),
                               "kmeans_changed_kernel"))
          return JIMM_ECUDA;
        JIMM_CUDA_CHECK(cudaMemcpyAsync(&changed, info + 3, sizeof(int), cudaMemcpyDeviceToHost, st));
        JIMM_CUDA_CHECK(cudaMemsetAsync(info + 3, 0, sizeof(int), st));
        JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
        if (changed == 0) break;  // the next means would be these bits again
      }
      // m_{t+1}: the rows sorted by cluster (counting sort), summed in fixed point, divided; c_{t+1} = l2_normalize(m_{t+1}), and a
      // cluster whose new centroid is not finite keeps m_t and c_t
      JIMM_CUDA_CHECK(cudaMemsetAsync(n, 0, static_cast<size_t>(C) * sizeof(int), st));
      JIMM_CUDA_CHECK(cudaMemsetAsync(S, 0, CE * sizeof(long long), st));
      if (na > 0) {
        if (int e = launched(launch_k(kmeans_count_kernel, dim3(blocks_of(na, 256)), dim3(256), 0, st, 1, false, a, na, n), "kmeans_count_kernel")) return e;
        if (int e = launched(launch_k(allowed_scan_kernel, dim3(1), dim3(1024), 0, st, 1, false, n, C, start), "allowed_scan_kernel")) return e;
        JIMM_CUDA_CHECK(cudaMemcpyAsync(cursor, start, static_cast<size_t>(C) * sizeof(int), cudaMemcpyDeviceToDevice, st));
        if (int e = launched(launch_k(kmeans_order_kernel, dim3(blocks_of(na, 256)), dim3(256), 0, st, 1, false, a, na, cursor, order), "kmeans_order_kernel"))
          return e;
        if (int e = launched(launch_k(kmeans_sum_kernel, dim3(blocks_of(na, kSumRows)), dim3(256), 0, st, 1, false, order, a, ids, g->rows, E, na,
                                      reinterpret_cast<unsigned long long*>(S)),
                             "kmeans_sum_kernel"))
          return e;
      }
      if (int e = launched(launch_k(kmeans_mean_kernel, dim3(blocks_of(static_cast<long long>(CE), 256)), dim3(256), 0, st, 1, false, S, n, m[cur],
                                    m[cur ^ 1], C, E),
                           "kmeans_mean_kernel"))
        return e;
      if (int e = l2_normalize_run(m[cur ^ 1], c[cur ^ 1], E, C, E, st)) return e;
      if (int e = launched(launch_k(kmeans_finite_kernel, dim3(blocks_of(C, 8)), dim3(256), 0, st, 1, false, c[cur ^ 1], C, E, m[cur ^ 1], m[cur],
                                    c[cur], info + 2),
                           "kmeans_finite_kernel"))
        return e;
      cur ^= 1;
    }
    // the outputs: c_t, a_t scattered to row ids, counts of a_t
    int32_t* a = abuf + (t & 1) * NA;
    JIMM_CUDA_CHECK(cudaMemcpyAsync(centroids, c[cur], CE * sizeof(float), cudaMemcpyDeviceToDevice, st));
    JIMM_CUDA_CHECK(cudaMemsetAsync(counts, 0, static_cast<size_t>(C) * sizeof(int64_t), st));
    if (rows > 0 && launched(launch_k(kmeans_clear_kernel, dim3(blocks_of(rows, 256)), dim3(256), 0, st, 1, false, assign, scores, rows),
                             "kmeans_clear_kernel"))
      return JIMM_ECUDA;
    if (na > 0 && launched(launch_k(kmeans_out_kernel, dim3(blocks_of(na, 256)), dim3(256), 0, st, 1, false, a, vals, ids, na, assign, scores,
                                    reinterpret_cast<unsigned long long*>(counts)),
                           "kmeans_out_kernel"))
      return JIMM_ECUDA;
    *iterations = t + 1;
    return 0;
  };
  const int rc = run();
  if (ids) cudaFreeAsync(ids, st);
  return free_scratch(base, st, rc);
}

}  // namespace jimm

// The hits of one range search or pairs call, in CSR: one segment per query chunk, each in its own device storage.
struct jimm_hits {
  struct Segment {
    int rows = 0;                   // rows of the segment; its offsets [rows + 1] count from the first row of the result
    long long start = 0, nnz = 0;   // offsets[0] and the segment's hits
    long long* offsets = nullptr;   // device
    float* scores = nullptr;        // device: scores fp32 [nnz], then indices int32 [nnz]
  };
  int device = 0, rows = 0;
  long long total = 0;
  std::vector<Segment> segs;
};

namespace jimm {

void hits_free(jimm_hits* h, cudaStream_t st) {  // in stream order
  for (auto& s : h->segs) {
    cudaFreeAsync(s.offsets, st);
    if (s.scores) cudaFreeAsync(s.scores, st);
  }
  delete h;
}

int gallery_range(const GalleryStore* g, const float* queries, int Q, bool pairs, float threshold, const float* logit_scale,
                  const float* logit_bias, const uint8_t* keep, jimm_hits** out, long long* stats, cudaStream_t st) {
  const int E = g->E;
  *out = nullptr;
  int device = 0;
  JIMM_CUDA_CHECK(cudaGetDevice(&device));
  // A filter or removed rows: the call runs over the N allowed rows' positions (ids), then maps the hits and, for pairs, the result's
  // rows back to row ids.
  const bool filtered = keep || g->removed > 0;
  int* ids = nullptr;
  int N = static_cast<int>(g->n);
  if (filtered)
    if (int rc = allowed_ids(g, keep, &ids, &N, st)) return rc;
  if (pairs) Q = N;
  jimm_hits* hits = new jimm_hits();
  hits->device = device;
  hits->rows = Q;
  if (Q == 0 && !(pairs && filtered)) {
    if (ids) cudaFreeAsync(ids, st);
    *out = hits;
    return 0;
  }
  const int qc = std::max(std::min(Q, kSearchRows), 1), nch = (N + kScreenCols - 1) / kScreenCols;
  // scratch: 256-byte aligned pieces of one stream-ordered allocation
  size_t off = 0;
  auto piece = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) / 256 * 256; return at; };
  const bool qbuf = !pairs || filtered;  // the queries, or the allowed stored rows of a pairs call, are staged in nq / hq / nbq
  const size_t o_nq = qbuf ? piece(static_cast<size_t>(qc) * E * sizeof(float)) : 0;
  const size_t o_hq = qbuf ? piece(static_cast<size_t>(qc) * E * sizeof(__half)) : 0;
  const size_t o_nbq = qbuf ? piece(static_cast<size_t>(qc) * sizeof(float)) : 0;
  const int vc = ids ? std::min(N, kScreenCols) : 0;  // the gallery view's chunk buffer
  const size_t o_vrows = piece(static_cast<size_t>(vc) * E * sizeof(float));
  const size_t o_vhalf = piece(static_cast<size_t>(vc) * E * sizeof(__half));
  const size_t o_vbound = piece(static_cast<size_t>(vc) * sizeof(float));
  const size_t o_fq = piece(static_cast<size_t>(qc) * E * sizeof(float));
  const size_t o_block = piece(static_cast<size_t>(qc) * std::min(N, kSearchCols) * sizeof(float));
  const size_t o_t = piece(static_cast<size_t>(qc) * sizeof(float));
  const size_t o_cnt = piece(static_cast<size_t>(qc) * sizeof(int));
  const size_t o_ovl = piece(static_cast<size_t>(qc) * sizeof(int));
  const size_t o_list = piece(static_cast<size_t>(qc) * kScreenCap * sizeof(int));
  const size_t o_info = piece(4 * sizeof(int));
  const size_t o_pos = piece(static_cast<size_t>(nch) * qc * sizeof(int));
  const size_t o_count = piece(static_cast<size_t>(nch) * qc * sizeof(int));
  const size_t o_dst = piece(static_cast<size_t>(nch) * qc * sizeof(long long));
  uint8_t* base = nullptr;
  std::vector<float*> stage(nch, nullptr);  // per gallery chunk: staged scores [room], then indices [room], of the current query chunk
  std::vector<int> stage_room(nch, 0);
  long long done = 0;                       // hits of the query chunks before the current one
  auto free_stage = [&]() {
    for (auto& p : stage) {
      if (p) cudaFreeAsync(p, st);
      p = nullptr;
    }
    std::fill(stage_room.begin(), stage_room.end(), 0);
  };
  // every failure frees what the call allocated, in stream order
  auto fail = [&](int rc) {
    free_stage();
    hits_free(hits, st);
    if (ids) cudaFreeAsync(ids, st);
    return base ? free_scratch(base, st, rc) : rc;
  };
  auto alloc = [&](void** p, size_t bytes, const char* what) -> int {
    const cudaError_t e = cudaMallocAsync(p, bytes, st);
    if (e == cudaSuccess) return 0;
    cudaGetLastError();
    *p = nullptr;
    set_last_error("%s: %s of %zu bytes after %lld hits -> %s", pairs ? "pairs" : "range search", what, bytes, done, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? JIMM_ENOMEM : JIMM_ECUDA;
  };
  if (int rc = alloc(reinterpret_cast<void**>(&base), off, "scratch")) return fail(rc);
  float* nq = reinterpret_cast<float*>(base + o_nq);
  __half* hq = reinterpret_cast<__half*>(base + o_hq);
  float* nbq = reinterpret_cast<float*>(base + o_nbq);
  float* fq = reinterpret_cast<float*>(base + o_fq);
  float* block = reinterpret_cast<float*>(base + o_block);
  float* t = reinterpret_cast<float*>(base + o_t);
  int* cnt = reinterpret_cast<int*>(base + o_cnt);
  int* ovl = reinterpret_cast<int*>(base + o_ovl);
  int* list = reinterpret_cast<int*>(base + o_list);
  int* info = reinterpret_cast<int*>(base + o_info);
  int* pos = reinterpret_cast<int*>(base + o_pos);
  int* count = reinterpret_cast<int*>(base + o_count);
  long long* dst = reinterpret_cast<long long*>(base + o_dst);
  RowView view{g, ids, N, reinterpret_cast<float*>(base + o_vrows), reinterpret_cast<__half*>(base + o_vhalf), reinterpret_cast<float*>(base + o_vbound)};
  RowView qview{g, ids, N, nq, hq, nbq};  // pairs: the query rows
  GemmScreen sd;
  sd.t = t; sd.cnt = cnt; sd.list = list; sd.cap = kScreenCap;
  const int max_smem = static_cast<int>(8192 * sizeof(float) + kScreenCap * sizeof(u64));
  if (int rc = smem_opt_in<range_rescore_kernel>(max_smem)) return fail(rc);
  auto check_launch = [&](cudaError_t e, const char* what) -> int {
    if (e == cudaSuccess) { note_launch(); return 0; }
    set_last_error("%s -> %s", what, cudaGetErrorString(e));
    return JIMM_ECUDA;
  };
  // Query rows q0 .. q0 + qn - 1 (normalised in qrows, fp16 copies qh, bounds qb) against gallery chunk c: screen, then the survivors'
  // hits (rescored) and the overflowed queries' hits (exact block step) staged in row order, their counts in count[c * qn + i].
  auto range_chunk = [&](int qn, int q0, float* qrows, const __half* qh, int c) -> int {
    const int g0 = c * kScreenCols, gn = std::min(kScreenCols, N - g0);
    if (pairs && g0 + gn - 1 <= q0) return 0;  // no row of the chunk lies above any query row's diagonal
    const int row0 = pairs ? q0 : -1;
    int* pos_c = pos + static_cast<size_t>(c) * qn;
    int* count_c = count + static_cast<size_t>(c) * qn;
    if (int e = view.at(g0, gn, st)) return e;
    sd.ng = view.bound;
    JIMM_CUDA_CHECK(cudaMemsetAsync(cnt, 0, static_cast<size_t>(qn) * sizeof(int), st));
    if (int e = gemm_screen_run(qh, qn, view.half, gn, E, sd, st)) return e;
    if (int e = check_launch(launch_k(range_info_kernel, dim3(1), dim3(1024), 0, st, 1, false, cnt, qn, kScreenCap, gn, ovl, pos_c, info),
                             "range_info_kernel"))
      return e;
    int h[4];
    JIMM_CUDA_CHECK(cudaMemcpyAsync(h, info, sizeof(h), cudaMemcpyDeviceToHost, st));
    JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
    const int nover = h[0], room = h[1], rescored = h[2], widest = h[3];
    if (stats) { stats[0] += rescored; stats[1] += nover; stats[2] += 1; }
    if (room == 0) return 0;
    if (int e = alloc(reinterpret_cast<void**>(&stage[c]), static_cast<size_t>(room) * (sizeof(float) + sizeof(int32_t)), "staging")) return e;
    stage_room[c] = room;
    float* ss = stage[c];
    int32_t* si = reinterpret_cast<int32_t*>(ss + room);
    if (widest > 0) {
      const size_t smem = static_cast<size_t>(E) * sizeof(float) + static_cast<size_t>(pow2_at_least(widest)) * sizeof(u64);
      if (int e = check_launch(launch_k(range_rescore_kernel, dim3(qn), dim3(kRangeThreads), smem, st, 1, false, qrows, view.rows, E, cnt, list, kScreenCap, g0, row0, threshold, logit_scale,
                                        logit_bias, pos_c, ss, si, count_c),
                               "range_rescore_kernel"))
        return e;
    }
    if (nover > 0) {  // those queries' chunk goes through the exact block step, in kSearchCols pieces
      if (int e = check_launch(launch_k(fallback_copy_kernel, dim3(nover), dim3(256), 0, st, 1, false, ovl, E, 0, qrows, fq, nullptr, 0ll,
                                        nullptr, 0ll, 1),
                               "fallback_copy_kernel"))
        return e;
      for (int s0 = 0; s0 < gn; s0 += kSearchCols) {
        const int pw = std::min(kSearchCols, gn - s0);
        if (int e = logits_run(fq, view.rows + static_cast<size_t>(s0) * E, logit_scale, logit_bias, block, nover, pw, E, pw, st)) return e;
        if (int e = check_launch(launch_k(range_block_kernel, dim3(nover), dim3(kRangeThreads), 0, st, 1, false, block, pw, ovl, g0 + s0, row0,
                                          threshold, pos_c, ss, si, count_c),
                                 "range_block_kernel"))
          return e;
      }
    }
    return 0;
  };
  // The end of a query chunk: offsets from the counts, then the staged hits gathered into the chunk's segment in (query, row) order.
  auto assemble = [&](int qn) -> int {
    jimm_hits::Segment seg;
    seg.rows = qn;
    seg.start = done;
    if (int e = alloc(reinterpret_cast<void**>(&seg.offsets), static_cast<size_t>(qn + 1) * sizeof(long long), "result offsets")) return e;
    hits->segs.push_back(seg);
    jimm_hits::Segment& sg = hits->segs.back();
    if (int e = check_launch(launch_k(range_offsets_kernel, dim3(1), dim3(1024), 0, st, 1, false, count, nch, qn, done, sg.offsets, dst),
                             "range_offsets_kernel"))
      return e;
    long long end = 0;
    JIMM_CUDA_CHECK(cudaMemcpyAsync(&end, sg.offsets + qn, sizeof(end), cudaMemcpyDeviceToHost, st));
    JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
    sg.nnz = end - done;
    if (sg.nnz > 0) {
      if (int e = alloc(reinterpret_cast<void**>(&sg.scores), static_cast<size_t>(sg.nnz) * (sizeof(float) + sizeof(int32_t)), "result")) return e;
      int32_t* idx = reinterpret_cast<int32_t*>(sg.scores + sg.nnz);
      for (int c = 0; c < nch; ++c) {
        if (!stage[c]) continue;
        const int* pos_c = pos + static_cast<size_t>(c) * qn;
        const int* count_c = count + static_cast<size_t>(c) * qn;
        const float* ss = stage[c];
        const int32_t* si = reinterpret_cast<const int32_t*>(ss + stage_room[c]);
        if (int e = check_launch(launch_k(range_gather_kernel, dim3(qn), dim3(kRangeThreads), 0, st, 1, false, ss, si, pos_c, count_c,
                                          dst + static_cast<size_t>(c) * qn, done, sg.scores, idx),
                                 "range_gather_kernel"))
          return e;
      }
      if (ids && check_launch(launch_k(hits_ids_kernel, dim3(static_cast<unsigned>((sg.nnz + 255) / 256)), dim3(256), 0, st, 1, false, idx,
                                       sg.nnz, ids),
                              "hits_ids_kernel"))
        return JIMM_ECUDA;
    }
    done = end;
    return 0;
  };
  // Filtered pairs: the result's rows are the stored rows 0 .. g->n - 1, so segment s of query positions q0 .. q0 + qn - 1 becomes the
  // stored rows after the previous segment's up to its last allowed row (the last segment: up to the end), those not allowed empty.
  auto pairs_rows = [&]() -> int {
    const int rows = static_cast<int>(g->n);
    if (hits->segs.empty()) {  // no allowed row
      jimm_hits::Segment seg;
      seg.rows = rows;
      if (int e = alloc(reinterpret_cast<void**>(&seg.offsets), static_cast<size_t>(rows + 1) * sizeof(long long), "result offsets")) return e;
      hits->segs.push_back(seg);
      JIMM_CUDA_CHECK(cudaMemsetAsync(seg.offsets, 0, static_cast<size_t>(rows + 1) * sizeof(long long), st));
    } else {
      const size_t ns = hits->segs.size();
      std::vector<int> last(ns, rows - 1);  // the last allowed row of each segment but the last
      for (size_t s = 0; s + 1 < ns; ++s)
        JIMM_CUDA_CHECK(cudaMemcpyAsync(&last[s], ids + s * qc + hits->segs[s].rows - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
      JIMM_CUDA_CHECK(cudaStreamSynchronize(st));
      int lo = 0;
      for (size_t s = 0; s < ns; ++s) {
        jimm_hits::Segment& sg = hits->segs[s];
        const int R = last[s] + 1 - lo;
        long long* ro = nullptr;
        if (int e = alloc(reinterpret_cast<void**>(&ro), static_cast<size_t>(R + 1) * sizeof(long long), "result offsets")) return e;
        if (int e = check_launch(launch_k(pairs_rows_kernel, dim3((R + 256) / 256), dim3(256), 0, st, 1, false, ids, static_cast<int>(s * qc), sg.rows,
                                          lo, R, sg.offsets, ro),
                                 "pairs_rows_kernel")) {
          cudaFreeAsync(ro, st);
          return e;
        }
        cudaFreeAsync(sg.offsets, st);
        sg.offsets = ro;
        sg.rows = R;
        lo += R;
      }
    }
    hits->rows = rows;
    return 0;
  };
  if (int rc = check_launch(launch_k(range_threshold_kernel, dim3((qc + 255) / 256), dim3(256), 0, st, 1, false, qc, threshold, logit_scale,
                                     logit_bias, t),
                            "range_threshold_kernel"))
    return fail(rc);
  for (int q0 = 0; q0 < Q; q0 += qc) {
    const int qn = std::min(qc, Q - q0);
    float* qrows = nq;
    const __half* qh = hq;
    int rc = 0;
    if (pairs) {  // the stored rows themselves: normalised, with their fp16 copies and bounds
      rc = qview.at(q0, qn, st);
      qrows = qview.rows;
      qh = qview.half;
      sd.nq = qview.bound;
    } else {
      sd.nq = nbq;
      rc = l2_normalize_run(queries + static_cast<size_t>(q0) * E, nq, E, qn, E, st);
      if (rc == 0) rc = prep_rows_run(nq, qn, E, hq, nbq, st);
    }
    if (rc == 0 && nch > 0) {
      const cudaError_t e = cudaMemsetAsync(count, 0, static_cast<size_t>(nch) * qn * sizeof(int), st);
      if (e != cudaSuccess) { set_last_error("cudaMemsetAsync -> %s", cudaGetErrorString(e)); rc = JIMM_ECUDA; }
    }
    for (int c = 0; c < nch && rc == 0; ++c) rc = range_chunk(qn, q0, qrows, qh, c);
    if (rc == 0) rc = assemble(qn);
    if (rc != 0) return fail(rc);
    free_stage();
  }
  if (pairs && filtered)
    if (int rc = pairs_rows()) return fail(rc);
  hits->total = done;
  *out = hits;
  if (ids) cudaFreeAsync(ids, st);
  return free_scratch(base, st, 0);
}

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

extern "C" int jimm_topk(const float* logits, int rows, int cols, int ld, int k, float* values, int32_t* indices, float* probs, void* stream) {
  if (rows < 0 || cols <= 0 || ld < cols) { set_last_error("top_k: bad shape rows=%d cols=%d ld=%d", rows, cols, ld); return JIMM_EINVAL; }
  if (k < 1 || k > cols) { set_last_error("top_k: k=%d outside 1 .. cols=%d", k, cols); return JIMM_EINVAL; }
  if (rows > 0 && (!logits || !values || !indices)) { set_last_error("top_k: null logits, values or indices"); return JIMM_EINVAL; }
  if (rows == 0) return 0;
  return topk_run(logits, rows, cols, ld, k, values, indices, probs, static_cast<cudaStream_t>(stream));
}

extern "C" int jimm_hits_size(const jimm_hits_t* h, int* rows, long long* total) {
  if (!h || !rows || !total) { set_last_error("hits: null handle, rows or total"); return JIMM_EINVAL; }
  *rows = h->rows;
  *total = h->total;
  return 0;
}

extern "C" int jimm_hits_copy(const jimm_hits_t* h, int64_t* offsets, float* scores, int32_t* indices, void* stream) {
  if (!h || !offsets || (h->total > 0 && (!scores || !indices))) { set_last_error("hits copy: null handle, offsets, scores or indices"); return JIMM_EINVAL; }
  JIMM_CUDA_CHECK(cudaSetDevice(h->device));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (h->segs.empty()) JIMM_CUDA_CHECK(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st));
  long long row = 0;
  for (const auto& s : h->segs) {  // consecutive segments share one offset: the first's last is the next one's first
    JIMM_CUDA_CHECK(cudaMemcpyAsync(offsets + row, s.offsets, static_cast<size_t>(s.rows + 1) * sizeof(int64_t), cudaMemcpyDefault, st));
    if (s.nnz > 0) {
      JIMM_CUDA_CHECK(cudaMemcpyAsync(scores + s.start, s.scores, static_cast<size_t>(s.nnz) * sizeof(float), cudaMemcpyDefault, st));
      JIMM_CUDA_CHECK(cudaMemcpyAsync(indices + s.start, s.scores + s.nnz, static_cast<size_t>(s.nnz) * sizeof(int32_t), cudaMemcpyDefault, st));
    }
    row += s.rows;
  }
  return 0;
}

extern "C" int jimm_hits_destroy(jimm_hits_t* h) {
  if (!h) return 0;
  JIMM_CUDA_CHECK(cudaSetDevice(h->device));
  cudaDeviceSynchronize();  // cudaFree does not wait for the work still using stream-ordered allocations
  for (auto& s : h->segs) {
    cudaFree(s.offsets);
    if (s.scores) cudaFree(s.scores);
  }
  delete h;
  return 0;
}
