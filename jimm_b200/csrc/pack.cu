// Checkpoint ingestion on the device (SURVEY.md 8f.2; reference: from_pretrained's layout transforms, models/vit.py:239-250,
// models/clip.py:356-396, models/siglip.py:318-366, and the `.numpy()` hand-off of common/utils.py:55-99).
//
// Parameters arrive as host pointers in their checkpoint dtype (fp32 | fp16 | bf16): either the reference's flax layout (kernel viewed
// (K, N) row-major) or -- zero-copy from a HuggingFace file -- its 2-D transpose (N, K), which is exactly the K-major operand layout the
// GEMMs read, so the double transpose HF -> flax -> packed collapses into a cast.  Bytes go through a two-slot pinned staging ring
// (the CPU memcpy of chunk i+1 runs under the DMA + pack kernel of chunk i), the cast / transpose / K-padding happen on the GPU, and
// nothing synchronises the stream until finalize ends.
#include <string.h>

#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

#define JIMM_TRY_RC(expr) do { int _rc = (expr); if (_rc != 0) return _rc; } while (0)

namespace jimm {

template <typename T>
__device__ __forceinline__ float src_to_float(T v) { return to_float(v); }

// dst[r * ldd + k] = cast(src[r * K + k]): row-preserving cast-copy (transposed-reference operands, fp32 vectors with ldd == K)
template <typename SrcT, typename OutT>
__global__ void __launch_bounds__(256) pack_rows_kernel(const SrcT* __restrict__ src, size_t rows, size_t K, OutT* __restrict__ dst, size_t ldd) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * K) return;
  const size_t r = i / K, k = i - r * K;
  dst[r * ldd + k] = from_float<OutT>(src_to_float(src[i]));
}

// src: kc rows of a (K, N) row-major matrix starting at row k0 -> dst[n * ldd + k0 + k] (K-major operand), 32 x 32 smem tiles
template <typename SrcT, typename OutT>
__global__ void pack_transpose_kernel(const SrcT* __restrict__ src, int kc, int N, OutT* __restrict__ dst, size_t ldd, int k0) {
  __shared__ float tile[32][33];
  const int kb = blockIdx.y * 32, nb = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = kb + i, n = nb + threadIdx.x;
    tile[i][threadIdx.x] = (k < kc && n < N) ? src_to_float(src[static_cast<size_t>(k) * N + n]) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = nb + i, k = kb + threadIdx.x;
    if (n < N && k < kc) dst[static_cast<size_t>(n) * ldd + k0 + k] = from_float<OutT>(tile[threadIdx.x][i]);
  }
}

template <typename SrcT>
static int rows_dispatch(const void* src, size_t rows, size_t K, void* dst, int out_type, size_t ldd, cudaStream_t s) {
  const size_t n = rows * K;
  if (n == 0) return 0;
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  const SrcT* p = static_cast<const SrcT*>(src);
  if (out_type == DT_F32) pack_rows_kernel<SrcT, float><<<grid, 256, 0, s>>>(p, rows, K, static_cast<float*>(dst), ldd);
  else if (out_type == DT_TF32) pack_rows_kernel<SrcT, tf32_t><<<grid, 256, 0, s>>>(p, rows, K, static_cast<tf32_t*>(dst), ldd);
  else if (out_type == DT_F16) pack_rows_kernel<SrcT, __half><<<grid, 256, 0, s>>>(p, rows, K, static_cast<__half*>(dst), ldd);
  else pack_rows_kernel<SrcT, __nv_bfloat16><<<grid, 256, 0, s>>>(p, rows, K, static_cast<__nv_bfloat16*>(dst), ldd);
  JIMM_LAUNCH_CHECK();
  return 0;
}
int pack_rows_run(const void* src, int src_type, size_t rows, size_t K, void* dst, int out_type, size_t ldd, cudaStream_t s) {
  if (src_type == DT_F16) return rows_dispatch<__half>(src, rows, K, dst, out_type, ldd, s);
  if (src_type == DT_BF16) return rows_dispatch<__nv_bfloat16>(src, rows, K, dst, out_type, ldd, s);
  return rows_dispatch<float>(src, rows, K, dst, out_type, ldd, s);
}

template <typename SrcT>
static int transpose_dispatch(const void* src, int kc, int N, void* dst, int out_type, size_t ldd, int k0, cudaStream_t s) {
  if (kc <= 0 || N <= 0) return 0;
  dim3 block(32, 8), grid((N + 31) / 32, (kc + 31) / 32);
  const SrcT* p = static_cast<const SrcT*>(src);
  if (out_type == DT_F32) pack_transpose_kernel<SrcT, float><<<grid, block, 0, s>>>(p, kc, N, static_cast<float*>(dst), ldd, k0);
  else if (out_type == DT_TF32) pack_transpose_kernel<SrcT, tf32_t><<<grid, block, 0, s>>>(p, kc, N, static_cast<tf32_t*>(dst), ldd, k0);
  else if (out_type == DT_F16) pack_transpose_kernel<SrcT, __half><<<grid, block, 0, s>>>(p, kc, N, static_cast<__half*>(dst), ldd, k0);
  else pack_transpose_kernel<SrcT, __nv_bfloat16><<<grid, block, 0, s>>>(p, kc, N, static_cast<__nv_bfloat16*>(dst), ldd, k0);
  JIMM_LAUNCH_CHECK();
  return 0;
}
int pack_transpose_run(const void* src, int src_type, int kc, int N, void* dst, int out_type, size_t ldd, int k0, cudaStream_t s) {
  if (src_type == DT_F16) return transpose_dispatch<__half>(src, kc, N, dst, out_type, ldd, k0, s);
  if (src_type == DT_BF16) return transpose_dispatch<__nv_bfloat16>(src, kc, N, dst, out_type, ldd, k0, s);
  return transpose_dispatch<float>(src, kc, N, dst, out_type, ldd, k0, s);
}

// ---- two-slot pinned staging ring ------------------------------------------------------------------------------------------
int UploadRing::init() {
  for (int i = 0; i < 2; ++i) {
    JIMM_CUDA_CHECK(cudaHostAlloc(&pinned[i], kCap, cudaHostAllocDefault));
    JIMM_CUDA_CHECK(cudaMalloc(&dev[i], kCap));
    JIMM_CUDA_CHECK(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    busy[i] = false;
  }
  ready = true;
  return 0;
}
void UploadRing::destroy() {
  if (!ready) return;
  for (int i = 0; i < 2; ++i) {
    if (busy[i]) cudaEventSynchronize(ev[i]);
    cudaFreeHost(pinned[i]);
    cudaFree(dev[i]);
    cudaEventDestroy(ev[i]);
  }
  ready = false;
}
int UploadRing::stage(const void* src, size_t bytes, cudaStream_t s, void** dptr) {
  if (!ready) JIMM_TRY_RC(init());
  if (bytes > kCap) { set_last_error("upload ring: chunk of %zu bytes exceeds the slot", bytes); return -1; }
  if (busy[cur]) { JIMM_CUDA_CHECK(cudaEventSynchronize(ev[cur])); busy[cur] = false; }  // the pack kernel that read this slot is done
  memcpy(pinned[cur], src, bytes);
  JIMM_CUDA_CHECK(cudaMemcpyAsync(dev[cur], pinned[cur], bytes, cudaMemcpyHostToDevice, s));
  *dptr = dev[cur];
  return 0;
}
int UploadRing::commit(cudaStream_t s) {
  JIMM_CUDA_CHECK(cudaEventRecord(ev[cur], s));
  busy[cur] = true;
  cur ^= 1;
  return 0;
}

// ---- host -> device packing through the ring (finalize, and the jimm_k_upload_* test entry points) ------------------------------
int upload_rows(UploadRing& ring, const void* host, int src_type, size_t rows, size_t K, void* dst, int out_type, size_t ldd, cudaStream_t s) {
  const size_t es = dtype_size(src_type), row_bytes = K * es;
  if (row_bytes == 0 || rows == 0) return 0;
  const uint8_t* src = static_cast<const uint8_t*>(host);
  const size_t out_es = dtype_size(out_type);
  if (row_bytes > UploadRing::kCap) {  // a single very long row (flat vectors): split it into pieces
    if (rows != 1 || ldd != K) { set_last_error("upload: row of %zu bytes exceeds the staging slot", row_bytes); return -1; }
    const size_t per = UploadRing::kCap / es;
    for (size_t k0 = 0; k0 < K; k0 += per) {
      const size_t kc = K - k0 < per ? K - k0 : per;
      void* d = nullptr;
      JIMM_TRY_RC(ring.stage(src + k0 * es, kc * es, s, &d));
      JIMM_TRY_RC(pack_rows_run(d, src_type, 1, kc, static_cast<uint8_t*>(dst) + k0 * out_es, out_type, kc, s));
      JIMM_TRY_RC(ring.commit(s));
    }
    return 0;
  }
  const size_t per = UploadRing::kCap / row_bytes;
  for (size_t r0 = 0; r0 < rows; r0 += per) {
    const size_t rc = rows - r0 < per ? rows - r0 : per;
    void* d = nullptr;
    JIMM_TRY_RC(ring.stage(src + r0 * row_bytes, rc * row_bytes, s, &d));
    JIMM_TRY_RC(pack_rows_run(d, src_type, rc, K, static_cast<uint8_t*>(dst) + r0 * ldd * out_es, out_type, ldd, s));
    JIMM_TRY_RC(ring.commit(s));
  }
  return 0;
}

int upload_kernel(UploadRing& ring, const void* host, int src_type, int K, int N, bool transposed, void* dst_base, int out_type, size_t ldd,
                  int n0, cudaStream_t s) {
  if (K <= 0 || N <= 0) return 0;
  uint8_t* dst = static_cast<uint8_t*>(dst_base) + static_cast<size_t>(n0) * ldd * dtype_size(out_type);
  if (transposed) return upload_rows(ring, host, src_type, N, K, dst, out_type, ldd, s);  // already [N, K]: cast-copy
  const size_t row_bytes = static_cast<size_t>(N) * dtype_size(src_type);
  if (row_bytes > UploadRing::kCap) { set_last_error("upload: kernel row of %zu bytes exceeds the staging slot", row_bytes); return -1; }
  // K is split into chunks of whole (K, N) rows; a chunk starts at row k0 of the kernel (not a multiple of the kernel's 32-row tile)
  const int per = static_cast<int>(UploadRing::kCap / row_bytes);
  const uint8_t* src = static_cast<const uint8_t*>(host);
  for (int k0 = 0; k0 < K; k0 += per) {
    const int kc = K - k0 < per ? K - k0 : per;
    void* d = nullptr;
    JIMM_TRY_RC(ring.stage(src + static_cast<size_t>(k0) * row_bytes, static_cast<size_t>(kc) * row_bytes, s, &d));
    JIMM_TRY_RC(pack_transpose_run(d, src_type, kc, N, dst, out_type, ldd, k0, s));
    JIMM_TRY_RC(ring.commit(s));
  }
  return 0;
}

}  // namespace jimm
