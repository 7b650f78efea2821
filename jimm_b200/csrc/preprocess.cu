// Image front-end on the GPU (SURVEY.md 8f.1): what the reference's examples run on the host before the forward path
// (examples/vit_inference.py:27-37, examples/clip_inference.py:35-38): HuggingFace image processor = Pillow 8-bit resize
// (bilinear / bicubic with antialiasing) -> optional centre crop -> rescale by 1/255 -> per-channel normalise -> NHWC.
//
// One fused kernel, input read once and output written once.  A CTA owns TY output rows of one image:
//   1. the input rows its vertical taps need go, one warp per row (coalesced 16-byte loads into a per-warp row buffer, no
//      CTA-wide synchronisation), through the horizontal pass, for the cropped columns only, into an 8-bit tile in shared
//      memory -- Pillow's temporary image, never written to HBM;
//   2. the vertical pass reads that tile four bytes per thread, and each resulting 8-bit sample goes through a 768-entry
//      table (channel, value) -> normalised float, then to the output dtype.
// Sizes whose plan does not fit in shared memory (4K and larger frames into the bicubic front-ends) run the same two passes as two
// kernels through an 8-bit intermediate in global memory (hpass_kernel, vpass_kernel); the planner (plan_size) is host-only.
// All arithmetic is Pillow's: int32 fixed point with 22 fractional bits, taps and weights from the same double-precision
// recipe, so the result is bit-exact (oracle/preprocess_oracle.py restates it and is pinned against Pillow itself).
// HBM-bound byte work: algorithmic bytes = H*W*3 read + oh*ow*3*sizeof(out) written per image.
#include <algorithm>
#include <cmath>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/jimm_b200.h"
#include "common.cuh"

#define JIMM_TRY(expr)          \
  do {                          \
    const int _rc = (expr);     \
    if (_rc != 0) return _rc;   \
  } while (0)

namespace jimm {
namespace {

constexpr int kPrecisionBits = 32 - 8 - 2;
constexpr int kThreads = 256;

// ---- host: Pillow's coefficient recipe (Resample.c precompute_coeffs + normalize_coeffs_8bpc) ----
double filter_bilinear(double x) {
  if (x < 0.0) x = -x;
  return x < 1.0 ? 1.0 - x : 0.0;
}
double filter_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

struct ResampleTable {
  int ksize = 0, kpad = 0;            // Pillow's window capacity; the same rounded up to a multiple of 4
  std::vector<int> first, count, kk;  // kk[out][ksize]

  // Device layout: rows padded with zero weights to kpad taps so the kernels run groups of four taps without a tail (a zero
  // weight makes whatever byte it meets irrelevant).
  std::vector<int> padded(int stride) const {
    const size_t n = first.size();
    std::vector<int> p(n * stride, 0);
    for (size_t i = 0; i < n; ++i)
      for (int k = 0; k < ksize; ++k) p[i * stride + k] = kk[i * ksize + k];
    return p;
  }
  // Row stride for shared memory: an odd number of 16-byte units, so a warp's int4 reads of consecutive rows are conflict-free.
  int smem_stride() const { return (kpad / 4) % 2 ? kpad : kpad + 4; }
};

// Windows of output coordinates [begin, end) (default: all of them), stored from index 0: the front-end builds only the cropped
// range, so its tables cost what the output needs whatever the size of the resize before the crop.  weights = false computes the
// window bounds only (kk stays empty): what the planner reads, without a filter evaluation.
ResampleTable make_table(int in_size, int out_size, int resample, int begin = 0, int end = -1, bool weights = true) {
  if (end < 0) end = out_size;
  double (*f)(double) = resample == 3 ? filter_bicubic : filter_bilinear;
  const double fsupport = resample == 3 ? 2.0 : 1.0;
  const double scale = static_cast<double>(in_size) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = fsupport * filterscale;
  ResampleTable t;
  t.ksize = static_cast<int>(std::ceil(support)) * 2 + 1;
  t.kpad = (t.ksize + 3) / 4 * 4;
  t.first.assign(end - begin, 0);
  t.count.assign(end - begin, 0);
  if (weights) t.kk.assign(static_cast<size_t>(end - begin) * t.ksize, 0);
  std::vector<double> w(weights ? t.ksize : 0);
  const double ss = 1.0 / filterscale;
  for (int xx = begin; xx < end; ++xx) {
    const double center = 0.0 + (xx + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    t.first[xx - begin] = xmin;
    t.count[xx - begin] = xmax;
    if (!weights) continue;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = f((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    for (int x = 0; x < xmax; ++x) {
      const double k = ww != 0.0 ? w[x] / ww : w[x];
      t.kk[static_cast<size_t>(xx - begin) * t.ksize + x] =
          k < 0 ? static_cast<int>(-0.5 + k * (1 << kPrecisionBits)) : static_cast<int>(0.5 + k * (1 << kPrecisionBits));
    }
  }
  return t;
}

struct KernelArgs {
  const uint8_t* img;
  void* out;
  const float* lut;                    // [3][256] normalised value of an 8-bit sample
  const int *hfirst, *hcount, *hk;     // horizontal tables of the cropped columns
  const int *vfirst, *vcount, *vk;     // vertical tables of the cropped rows
  int H, W, oh, ow, hks, hstride, vks;  // hks / vks: taps rounded up to a multiple of 4; hstride: row stride of hk
  int TY;                              // output rows per CTA
  int rowb;                            // bytes per tile row (ow*3 rounded up to 4)
  int stage_bytes;                     // one warp's row buffer (W*3 + 32, rounded to 16)
  int vec_ok;                          // img is 16-byte aligned
  int P, gw;                           // patch-row store: patch size, patches per grid row
};

// Where vertical_pass stores: NHWC [B, oh, ow, 3] (the fixed-size front-end), or NaFlex patch rows (one sample's [gh * gw, P*P*3],
// each row a patch flattened in (py, px, c) order).
enum { kNhwc = 0, kPatchRows = 1 };

__device__ __forceinline__ int clip8(int acc) {
  const int v = acc >> kPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

template <typename OUT>
__device__ __forceinline__ OUT to_out(float v);
template <> __device__ __forceinline__ float to_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __half to_out<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 to_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename OUT>
__device__ __forceinline__ void store4(OUT* dst, const OUT (&v)[4]) {
  if constexpr (sizeof(OUT) == 4) {
    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    uint2 pk;
    pk.x = static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&v[0])) | (static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&v[1])) << 16);
    pk.y = static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&v[2])) | (static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&v[3])) << 16);
    *reinterpret_cast<uint2*>(dst) = pk;
  }
}

// Vertical pass + normalise + store of output rows [yo0, yo1) of image b (NHWC; patch rows: a.out is the sample's first row), from
// the 8-bit horizontal-pass rows in tile32 (input rows from in_y0 on, rowb bytes apart): four consecutive samples per thread, four
// taps per step.
template <typename OUT, int LAYOUT>
__device__ __forceinline__ void vertical_pass(const KernelArgs& a, const uint32_t* tile32, int in_y0, int yo0, int yo1, int b) {
  const int tid = threadIdx.x;
  const int words = a.rowb / 4;
  const int n_el = a.ow * 3;
  OUT* out = static_cast<OUT*>(a.out);
  for (int it = tid; it < (yo1 - yo0) * words; it += kThreads) {
    const int r = it / words, wd = it - r * words;
    const int yo = yo0 + r;
    const uint32_t* tp = tile32 + (a.vfirst[yo] - in_y0) * words + wd;
    const int vgroups = (a.vcount[yo] + 3) >> 2;
    const int4* kp = reinterpret_cast<const int4*>(a.vk + static_cast<size_t>(yo) * a.vks);
    int acc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = 1 << (kPrecisionBits - 1);
    for (int g = 0; g < vgroups; ++g) {
      const int4 k = __ldg(kp + g);
      const uint32_t t0 = tp[(4 * g) * words], t1 = tp[(4 * g + 1) * words], t2 = tp[(4 * g + 2) * words], t3 = tp[(4 * g + 3) * words];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[j] += static_cast<int>((t0 >> (8 * j)) & 255u) * k.x;
        acc[j] += static_cast<int>((t1 >> (8 * j)) & 255u) * k.y;
        acc[j] += static_cast<int>((t2 >> (8 * j)) & 255u) * k.z;
        acc[j] += static_cast<int>((t3 >> (8 * j)) & 255u) * k.w;
      }
    }
    const int e0 = wd * 4;
    OUT v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = (e0 + j) % 3;
      v[j] = to_out<OUT>(__ldg(a.lut + c * 256 + clip8(acc[j])));
    }
    if constexpr (LAYOUT == kNhwc) {
      const size_t base = (static_cast<size_t>(b) * a.oh + yo) * n_el + e0;
      if (e0 + 3 < n_el && (base * sizeof(OUT)) % (4 * sizeof(OUT)) == 0) {
        store4(out + base, v);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < n_el) out[base + j] = v[j];
      }
    } else {
      // one pixel row of a patch is a run of 3P contiguous elements: (yo, e) -> patch row (yo / P) * gw + e / 3P, column
      // (yo % P) * 3P + e % 3P; the four samples go out as one vector when they fall inside one run at an aligned address
      const int run = 3 * a.P;
      const size_t row0 = static_cast<size_t>(yo / a.P) * a.gw * run * a.P + static_cast<size_t>(yo % a.P) * run;
      const int pc = e0 / run, w0 = e0 - pc * run;
      const size_t base = row0 + static_cast<size_t>(pc) * run * a.P + w0;
      if (w0 + 3 < run && reinterpret_cast<uintptr_t>(out + base) % (4 * sizeof(OUT)) == 0) {
        store4(out + base, v);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int e = e0 + j, pj = e / run;
          if (e < n_el) out[row0 + static_cast<size_t>(pj) * run * a.P + (e - pj * run)] = v[j];
        }
      }
    }
  }
}

// One CTA's work of the fused kernel: output rows [ty * TY, ty * TY + TY) of image b, smem the dynamic shared memory.
template <typename OUT, int LAYOUT>
__device__ __forceinline__ void fused_tile(const KernelArgs& a, uint8_t* smem, int b, int ty) {
  int* hk_s = reinterpret_cast<int*>(smem);                 // [ow][hstride]
  int* hfirst_s = hk_s + a.ow * a.hstride;  // byte offset of the window in a row | number of four-tap groups << 24
  uint8_t* stage = reinterpret_cast<uint8_t*>(hfirst_s + a.ow);
  stage += (16 - (reinterpret_cast<uintptr_t>(stage) & 15)) & 15;
  uint8_t* tile = stage + static_cast<size_t>(kThreads / 32) * a.stage_bytes;  // stage = one row buffer per warp

  const int tid = threadIdx.x;
  const int yo0 = ty * a.TY;
  const int yo1 = min(yo0 + a.TY, a.oh);
  const int in_y0 = a.vfirst[yo0];
  const int in_y1 = a.vfirst[yo1 - 1] + a.vcount[yo1 - 1];

  {
    const int4* src = reinterpret_cast<const int4*>(a.hk);
    int4* dst = reinterpret_cast<int4*>(hk_s);
    for (int i = tid; i < a.ow * a.hstride / 4; i += kThreads) dst[i] = __ldg(src + i);
    for (int i = tid; i < a.ow; i += kThreads) hfirst_s[i] = (a.hfirst[i] * 3) | (((a.hcount[i] + 3) >> 2) << 24);
  }

  const size_t row_bytes = static_cast<size_t>(a.W) * 3;
  const uint8_t* img_b = a.img + static_cast<size_t>(b) * a.H * row_bytes;
  __syncthreads();
  // ---- horizontal pass: one warp per input row, no CTA-wide synchronisation (warps hide each other's load latency) ----
  const int warp = tid >> 5, lane = tid & 31;
  uint8_t* wb = stage + static_cast<size_t>(warp) * a.stage_bytes;
  const uint32_t* wb32 = reinterpret_cast<const uint32_t*>(wb);
  for (int row = warp; row < in_y1 - in_y0; row += kThreads / 32) {
    const uint8_t* src = img_b + static_cast<size_t>(in_y0 + row) * row_bytes;
    const int bytes = static_cast<int>(row_bytes);
    const int mis = a.vec_ok ? static_cast<int>(reinterpret_cast<uintptr_t>(src) & 15) : 0;  // data starts at wb + mis
    if (a.vec_ok) {
      const int head = (16 - mis) & 15;  // bytes before the first aligned vector
      const int nvec = bytes > head ? (bytes - head) / 16 : 0;
      const uint4* vsrc = reinterpret_cast<const uint4*>(src + head);
      uint4* vdst = reinterpret_cast<uint4*>(wb + mis + head);
      for (int i = lane; i < nvec; i += 32) vdst[i] = __ldg(vsrc + i);
      const int tail0 = head + nvec * 16;
      for (int i = lane; i < head && i < bytes; i += 32) wb[mis + i] = __ldg(src + i);
      for (int i = tail0 + lane; i < bytes; i += 32) wb[mis + i] = __ldg(src + i);
    } else {
      for (int i = lane; i < bytes; i += 32) wb[i] = __ldg(src + i);
    }
    __syncwarp();
    uint8_t* trow = tile + static_cast<size_t>(row) * a.rowb;
    for (int xo = lane; xo < a.ow; xo += 32) {
      // The window is a run of RGB bytes from an arbitrary byte offset: read aligned words, realign them with funnel shifts;
      // four taps = twelve bytes = three realigned words (R0 G0 B0 R1 | G1 B1 R2 G2 | B2 R3 G3 B3) and one int4 of weights.
      const int fg = hfirst_s[xo];
      const int start = (fg & 0xffffff) + mis, hgroups = fg >> 24;
      const uint32_t* wp = wb32 + (start >> 2);
      const uint32_t sh = (start & 3) * 8;
      const int4* kp = reinterpret_cast<const int4*>(hk_s + xo * a.hstride);
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      uint32_t prev = wp[0];
      for (int g = 0; g < hgroups; ++g) {
        const uint32_t w1 = wp[3 * g + 1], w2 = wp[3 * g + 2], w3 = wp[3 * g + 3];
        const int4 k = kp[g];
        const uint32_t s0 = __funnelshift_r(prev, w1, sh), s1 = __funnelshift_r(w1, w2, sh), s2 = __funnelshift_r(w2, w3, sh);
        prev = w3;
        a0 += static_cast<int>(s0 & 255u) * k.x;
        a1 += static_cast<int>((s0 >> 8) & 255u) * k.x;
        a2 += static_cast<int>((s0 >> 16) & 255u) * k.x;
        a0 += static_cast<int>(s0 >> 24) * k.y;
        a1 += static_cast<int>(s1 & 255u) * k.y;
        a2 += static_cast<int>((s1 >> 8) & 255u) * k.y;
        a0 += static_cast<int>((s1 >> 16) & 255u) * k.z;
        a1 += static_cast<int>(s1 >> 24) * k.z;
        a2 += static_cast<int>(s2 & 255u) * k.z;
        a0 += static_cast<int>((s2 >> 8) & 255u) * k.w;
        a1 += static_cast<int>((s2 >> 16) & 255u) * k.w;
        a2 += static_cast<int>(s2 >> 24) * k.w;
      }
      trow[xo * 3] = static_cast<uint8_t>(clip8(a0));
      trow[xo * 3 + 1] = static_cast<uint8_t>(clip8(a1));
      trow[xo * 3 + 2] = static_cast<uint8_t>(clip8(a2));
    }
    __syncwarp();
  }
  __syncthreads();
  vertical_pass<OUT, LAYOUT>(a, reinterpret_cast<const uint32_t*>(tile), in_y0, yo0, yo1, b);
}

template <typename OUT>
__global__ void __launch_bounds__(kThreads) preprocess_kernel(const KernelArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  fused_tile<OUT, kNhwc>(a, smem, blockIdx.y, blockIdx.x);
}

// Two-pass path for sizes whose fused plan does not fit in shared memory (Resample.c's own order): the horizontal pass writes the
// 8-bit intermediate -- the same clipped bytes the fused kernel keeps in its tile -- to global memory, one CTA per input row of one
// image, for the cropped columns and the rows the cropped output reads only; vertical_pass then reads it from there.
struct PassArgs {
  KernelArgs k;
  uint8_t* mid;  // [images][rows][rowb] bytes, plus zero-weight tap slack after the last image
  int y0, rows;  // input rows [y0, y0 + rows) of each image
  int b0;        // first image of this chunk: k.img and k.out stay the call's base pointers, so the vector stores' alignment
                 // test in vertical_pass sees the absolute output index
};

// Horizontal pass of one input row src into its intermediate row dst, one thread per output pixel.
__device__ __forceinline__ void hpass_row(const KernelArgs& a, const uint8_t* src, uint8_t* dst) {
  const long long last = (a.W - 1) * 3LL;  // zero-weight taps past the window may run past the row: read its last pixel instead
  for (int xo = threadIdx.x; xo < a.ow; xo += kThreads) {
    const long long x0 = a.hfirst[xo] * 3LL;  // 64-bit: the padded taps may pass 2^31 in a row of nearly 2^31 bytes
    const int hgroups = (a.hcount[xo] + 3) >> 2;
    const int4* kp = reinterpret_cast<const int4*>(a.hk + static_cast<size_t>(xo) * a.hstride);
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int g = 0; g < hgroups; ++g) {
      const int4 k4 = __ldg(kp + g);
      const int kw[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint8_t* px = src + min(x0 + (4 * g + j) * 3, last);
        a0 += static_cast<int>(__ldg(px)) * kw[j];
        a1 += static_cast<int>(__ldg(px + 1)) * kw[j];
        a2 += static_cast<int>(__ldg(px + 2)) * kw[j];
      }
    }
    dst[xo * 3] = static_cast<uint8_t>(clip8(a0));
    dst[xo * 3 + 1] = static_cast<uint8_t>(clip8(a1));
    dst[xo * 3 + 2] = static_cast<uint8_t>(clip8(a2));
  }
}

__global__ void __launch_bounds__(kThreads) hpass_kernel(const PassArgs p) {
  const KernelArgs& a = p.k;
  const int row = blockIdx.x, b = blockIdx.y;
  hpass_row(a, a.img + (static_cast<size_t>(p.b0 + b) * a.H + p.y0 + row) * a.W * 3, p.mid + (static_cast<size_t>(b) * p.rows + row) * a.rowb);
}

template <typename OUT>
__global__ void __launch_bounds__(kThreads) vpass_kernel(const PassArgs p) {
  const int b = blockIdx.y;
  const int yo0 = blockIdx.x * p.k.TY;
  const int yo1 = min(yo0 + p.k.TY, p.k.oh);
  const uint32_t* tile32 = reinterpret_cast<const uint32_t*>(p.mid + static_cast<size_t>(b) * p.rows * p.k.rowb);
  vertical_pass<OUT, kNhwc>(p.k, tile32, p.y0, yo0, yo1, p.b0 + b);
}

struct DevTable {
  int ksize = 0, stride = 0;
  int *first = nullptr, *count = nullptr, *kk = nullptr;
};

enum { kFused = 0, kTwoPass = 1 };
constexpr long long kMaxFrameBytes = (1LL << 31) - 1;  // H * W * 3 of one frame
constexpr int kMaxResizedEdge = 1 << 24;               // each edge of the resized image before the crop: keeps pre-crop coordinates far inside int
constexpr size_t kMidChunkBytes = size_t(64) << 20;    // two-pass intermediate of one chunk of images
constexpr int kFusedImages = 65532;                   // images per fused launch
constexpr int kTwoPassTY = 8;                          // output rows per CTA of the two-pass vertical kernel

struct SizePlan {
  int rh = 0, rw = 0, top = 0, left = 0, oh = 0, ow = 0;
  DevTable h, v;
  int path = kFused;
  int tier = -1;  // fused: index of the shared-memory budget the plan was chosen under
  int TY = 0, tile_rows = 0, rowb = 0, stage_bytes = 0;
  size_t smem = 0;
  int mid_y0 = 0, mid_rows = 0;  // two-pass: the input rows [mid_y0, mid_y0 + mid_rows) the cropped output reads
};

}  // namespace
}  // namespace jimm

using namespace jimm;

struct jimm_preproc {
  jimm_preproc_config_t cfg;
  int device = 0;
  int naflex_patch = 0;  // > 0: a NaFlex handle (jimm_preproc_create_naflex), its patch size; the output size is per image
  float* lut = nullptr;
  mutable std::mutex mu;  // guards plans and allocs: one handle may be driven from several threads
  std::map<std::pair<int, int>, SizePlan> plans;
  std::vector<void*> allocs;
};

namespace {

int upload(jimm_preproc* p, const std::vector<int>& v, int** out) {
  void* d = nullptr;
  JIMM_CUDA_CHECK(cudaMalloc(&d, v.size() * sizeof(int)));
  p->allocs.push_back(d);
  JIMM_CUDA_CHECK(cudaMemcpy(d, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice));
  *out = static_cast<int*>(d);
  return 0;
}

int resized_size(const jimm_preproc_config_t& c, int H, int W, int* rh, int* rw) {
  double h = c.height, w = c.width;
  if (c.shortest_edge) {
    // transformers get_resize_output_image_size(size=shortest_edge, default_to_square=False)
    const int s = W <= H ? W : H, l = W <= H ? H : W;
    const double new_long = static_cast<double>(c.shortest_edge) * l / s;
    if (W <= H) { w = c.shortest_edge; h = new_long; } else { h = c.shortest_edge; w = new_long; }
  }
  if (h >= kMaxResizedEdge + 1.0 || w >= kMaxResizedEdge + 1.0) {
    set_last_error("resize %dx%d -> %.0fx%.0f: the front-end resizes to at most %d pixels per edge before the crop", H, W, std::floor(h),
                   std::floor(w), kMaxResizedEdge);
    return JIMM_EINVAL;
  }
  *rh = static_cast<int>(h);
  *rw = static_cast<int>(w);
  return 0;
}

int check_cfg(const jimm_preproc_config_t* c) {
  if (!c) { set_last_error("null preprocessing config"); return JIMM_EINVAL; }
  if (c->resample != 2 && c->resample != 3) { set_last_error("resample must be 2 (bilinear) or 3 (bicubic), got %d", c->resample); return JIMM_EINVAL; }
  if (!c->shortest_edge && (c->height <= 0 || c->width <= 0)) { set_last_error("size needs height and width, or shortest_edge"); return JIMM_EINVAL; }
  if ((c->crop_h > 0) != (c->crop_w > 0)) { set_last_error("crop needs both height and width"); return JIMM_EINVAL; }
  for (int i = 0; i < 3; ++i)
    if (c->std[i] == 0.f) { set_last_error("std evaluated to zero, leading to division by zero."); return JIMM_EINVAL; }
  return 0;
}

// The plan of one frame size, on the host only (jimm_preproc_output_size and the plan test hook run it without a GPU): output
// geometry, Pillow's tables and the path.  Fused when the kernel's shared memory fits one of its budgets; otherwise two passes
// through a global 8-bit intermediate.  A size is refused only past the limits checked here (INTEGRATION.md).
int plan_size(const jimm_preproc_config_t& c, int H, int W, SizePlan* out, ResampleTable* th_out, ResampleTable* tv_out, bool weights = true) {
  if (H <= 0 || W <= 0) { set_last_error("bad image size %dx%d", H, W); return JIMM_EINVAL; }
  if (static_cast<long long>(H) * W * 3 > kMaxFrameBytes) {
    set_last_error("frame %dx%d is %lld bytes: the front-end takes frames of at most 2^31 - 1 bytes (H x W x 3)", H, W,
                   static_cast<long long>(H) * W * 3);
    return JIMM_EINVAL;
  }
  SizePlan s;
  JIMM_TRY(resized_size(c, H, W, &s.rh, &s.rw));
  s.oh = c.crop_h ? c.crop_h : s.rh;
  s.ow = c.crop_w ? c.crop_w : s.rw;
  if (s.oh > s.rh || s.ow > s.rw) {
    set_last_error("centre crop %dx%d larger than the resized image %dx%d", s.oh, s.ow, s.rh, s.rw);
    return JIMM_EINVAL;
  }
  s.top = (s.rh - s.oh) / 2;
  s.left = (s.rw - s.ow) / 2;
  ResampleTable& th = *th_out;
  ResampleTable& tv = *tv_out;
  th = make_table(W, s.rw, c.resample, s.left, s.left + s.ow, weights);
  tv = make_table(H, s.rh, c.resample, s.top, s.top + s.oh, weights);
  s.h.ksize = th.kpad;
  s.h.stride = th.smem_stride();
  s.v.ksize = s.v.stride = tv.kpad;
  s.rowb = (s.ow * 3 + 3) / 4 * 4;
  // fused: one warp's row buffer holds a whole input row, and a window descriptor packs its four-tap group count in 7 bits
  const size_t row_bytes = static_cast<size_t>(W) * 3;
  int hgroups = 0;
  for (int xo = 0; xo < s.ow; ++xo) hgroups = std::max(hgroups, (th.count[xo] + 3) >> 2);
  if (row_bytes + 3 * th.kpad + 48 <= 64 * 1024 && hgroups < 128) {
    // shared-memory budget: horizontal tables for the cropped columns + staging group + 8-bit tile
    const size_t tables = (static_cast<size_t>(s.ow) * s.h.stride + s.ow) * sizeof(int) + 16;
    s.stage_bytes = static_cast<int>((row_bytes + 15 + 3 * th.kpad + 8 + 15) / 16 * 16);  // alignment shift + zero-weight taps past the row + word read-ahead
    // Largest tile of output rows (<= 32) that fits three CTAs per SM; when that leaves fewer than 16 rows (wide inputs, large
    // outputs) the halo rows recomputed per tile dominate, so trade occupancy for a taller tile: two CTAs, then one.
    const size_t budgets[3] = {72 * 1024, 110 * 1024, 200 * 1024};
    for (int bi = 0; bi < 3; ++bi) {
      s.tier = bi;
      for (s.TY = 32; s.TY >= 1; s.TY /= 2) {
        int rows = 0;  // worst-case number of input rows one tile of TY output rows touches
        for (int y0 = 0; y0 < s.oh; y0 += s.TY) {
          const int y1 = (y0 + s.TY < s.oh ? y0 + s.TY : s.oh) - 1;
          const int r = tv.first[y1] + tv.count[y1] - tv.first[y0];
          rows = r > rows ? r : rows;
        }
        s.tile_rows = rows;
        s.smem = tables + static_cast<size_t>(kThreads / 32) * s.stage_bytes + static_cast<size_t>(rows + tv.kpad) * s.rowb + 16;  // zero-weight taps may run past the last row
        if (s.smem <= budgets[bi] || s.TY == 1) break;
      }
      if (s.smem <= budgets[bi] && (s.TY >= 16 || s.TY >= s.oh)) break;
    }
    if (s.smem <= 200 * 1024) {
      *out = s;
      return 0;
    }
  }
  s.path = kTwoPass;
  s.tier = -1;
  s.TY = kTwoPassTY;
  s.tile_rows = s.stage_bytes = 0;
  s.smem = 0;
  s.mid_y0 = tv.first[0];
  s.mid_rows = tv.first[s.oh - 1] + tv.count[s.oh - 1] - s.mid_y0;
  const size_t mid_bytes = static_cast<size_t>(s.mid_rows + tv.kpad) * s.rowb;  // the vertical pass indexes one image's rows in int
  if (mid_bytes > static_cast<size_t>(kMaxFrameBytes)) {
    set_last_error("resize %dx%d -> %dx%d needs an 8-bit intermediate of %zu bytes per image: the front-end's limit is 2^31 - 1", H, W,
                   s.rh, s.rw, mid_bytes);
    return JIMM_EINVAL;
  }
  *out = s;
  return 0;
}

int get_plan(jimm_preproc* p, int H, int W, SizePlan** out) {
  std::lock_guard<std::mutex> lock(p->mu);
  auto it = p->plans.find({H, W});
  if (it != p->plans.end()) { *out = &it->second; return 0; }
  SizePlan s;
  ResampleTable th, tv;
  JIMM_TRY(plan_size(p->cfg, H, W, &s, &th, &tv));
  JIMM_TRY(upload(p, th.first, &s.h.first));
  JIMM_TRY(upload(p, th.count, &s.h.count));
  JIMM_TRY(upload(p, th.padded(s.h.stride), &s.h.kk));
  JIMM_TRY(upload(p, tv.first, &s.v.first));
  JIMM_TRY(upload(p, tv.count, &s.v.count));
  JIMM_TRY(upload(p, tv.padded(s.v.stride), &s.v.kk));
  auto ins = p->plans.emplace(std::make_pair(H, W), s);
  *out = &ins.first->second;  // map nodes never move: the pointer stays valid while other sizes are added
  return 0;
}

template <typename OUT>
int launch(const KernelArgs& a, const SizePlan& s, int B, cudaStream_t stream) {
  if (int rc = smem_opt_in<preprocess_kernel<OUT>>(200 * 1024)) return rc;
  const dim3 grid((s.oh + s.TY - 1) / s.TY, B);
  JIMM_CUDA_CHECK(launch_k(preprocess_kernel<OUT>, grid, dim3(kThreads), s.smem, stream, 1, false, a));
  note_launch();
  return 0;
}

template <typename OUT>
int launch_two_pass(const PassArgs& pa, const SizePlan& s, int B, cudaStream_t stream) {
  JIMM_CUDA_CHECK(launch_k(hpass_kernel, dim3(s.mid_rows, B), dim3(kThreads), 0, stream, 1, false, pa));
  note_launch();
  JIMM_CUDA_CHECK(launch_k(vpass_kernel<OUT>, dim3((s.oh + s.TY - 1) / s.TY, B), dim3(kThreads), 0, stream, 1, false, pa));
  note_launch();
  return 0;
}

// All B images of one size: the fused kernel, up to 65532 images per launch; or the two passes, whose intermediate is allocated in
// stream order for this call alone, so that calls in flight on other streams of the same handle never share it, and sized for a
// chunk of images rather than the batch.  (The device's default pool returns it to the driver at each synchronisation unless
// the application raises the pool's release threshold; the cost of that has not been measured.)
template <typename OUT>
int run_sized(const SizePlan& s, KernelArgs a, int B, cudaStream_t st) {
  const uint8_t* img = a.img;
  OUT* out = static_cast<OUT*>(a.out);
  const size_t in_image = static_cast<size_t>(a.H) * a.W * 3, out_image = static_cast<size_t>(s.oh) * s.ow * 3;
  if (s.path == kFused) {
    // 65532 images per launch (the grid's y limit is 65535): a multiple of four, so every launch's output pointer keeps the
    // alignment of `out` that the kernel's vector stores test relative to it
    for (int b0 = 0; b0 < B; b0 += kFusedImages) {
      a.img = img + static_cast<size_t>(b0) * in_image;
      a.out = out + static_cast<size_t>(b0) * out_image;
      JIMM_TRY(launch<OUT>(a, s, std::min(B - b0, kFusedImages), st));
    }
    return 0;
  }
  const size_t mid_image = static_cast<size_t>(s.mid_rows) * s.rowb;
  const int chunk = static_cast<int>(std::min<size_t>(std::max<size_t>(kMidChunkBytes / mid_image, 1), std::min(B, 65535)));
  PassArgs pa;
  pa.k = a;
  pa.y0 = s.mid_y0;
  pa.rows = s.mid_rows;
  pa.mid = nullptr;
  pa.b0 = 0;
  // + zero-weight taps of the last image's last rows, which may run past its intermediate
  JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&pa.mid), chunk * mid_image + static_cast<size_t>(s.v.ksize) * s.rowb, st));
  int rc = 0;
  for (int b0 = 0; b0 < B && rc == 0; b0 += chunk) {
    pa.b0 = b0;
    rc = launch_two_pass<OUT>(pa, s, std::min(B - b0, chunk), st);
  }
  const cudaError_t fe = cudaFreeAsync(pa.mid, st);
  if (rc == 0 && fe != cudaSuccess) { set_last_error("cudaFreeAsync -> %s", cudaGetErrorString(fe)); return JIMM_ECUDA; }
  return rc;
}


}  // namespace
namespace jimm {
namespace {

// ---- SigLIP 2 NaFlex: every image at its own output size, written as patch rows, all images of a call in ragged launches ----
// A call's images become flat lists of work items (the CTAs of the fused kernel: (image, output-row tile); of the two passes:
// (image, input row) and (image, tile)); each CTA finds its image by a binary search over the per-image descriptors, which travel
// as the launch's __grid_constant__ parameter (chunks of kNfImages images).  Pillow's tables are built on the device for every
// call into scratch allocated in stream order: the handle keeps nothing per frame size, and the host never waits for the stream.

// The size rule of transformers' Siglip2 processors (get_image_size_for_max_num_patches), in double precision: a binary search
// for the largest scale whose patch-rounded size has at most max_num_patches patches.  Plain IEEE double arithmetic, as Python's
// floats (the host compiler contracts no FMA here: x86-64 without -mfma).
int naflex_grid(int patch, int max_num_patches, int H, int W, int* gh, int* gw) {
  if (patch < 1) { set_last_error("NaFlex patch size %d: must be at least 1", patch); return JIMM_EINVAL; }
  if (max_num_patches < 1) { set_last_error("max_num_patches %d: must be at least 1", max_num_patches); return JIMM_EINVAL; }
  if (H <= 0 || W <= 0) { set_last_error("bad image size %dx%d", H, W); return JIMM_EINVAL; }
  if (static_cast<long long>(H) * W * 3 > kMaxFrameBytes) {
    set_last_error("frame %dx%d is %lld bytes: the front-end takes frames of at most 2^31 - 1 bytes (H x W x 3)", H, W,
                   static_cast<long long>(H) * W * 3);
    return JIMM_EINVAL;
  }
  auto scaled = [patch](double scale, int size) -> long long {
    const long long s = static_cast<long long>(std::ceil(size * scale / patch)) * patch;
    return s > patch ? s : patch;
  };
  const double eps = 1e-5;
  double lo = eps / 10, hi = 100.0;
  while (hi - lo >= eps) {
    const double scale = (lo + hi) / 2;
    const long long th = scaled(scale, H), tw = scaled(scale, W);
    const double n = (static_cast<double>(th) / patch) * (static_cast<double>(tw) / patch);
    if (n <= max_num_patches) lo = scale; else hi = scale;
  }
  const long long rows = scaled(lo, H) / patch, cols = scaled(lo, W) / patch;
  if (rows * cols > max_num_patches) {
    set_last_error("frame %dx%d: the NaFlex size rule gives a %lldx%lld patch grid, more than max_num_patches = %d", H, W, rows, cols,
                   max_num_patches);
    return JIMM_EINVAL;
  }
  *gh = static_cast<int>(rows);
  *gw = static_cast<int>(cols);
  return 0;
}

struct NfImage {
  const uint8_t* img;  // the frame, [H, W, 3]
  void* out;           // the sample's first patch row
  long long tab;       // its tables in the call's table scratch (ints): hfirst, hcount [ow4], hk [ow][hstride], vfirst, vcount [oh4], vk [oh][vks]
  long long mid;       // two-pass: its intermediate in the chunk's buffer (bytes)
  int H, W, oh, ow;
  int hstride, vks, TY, rowb, stage_bytes;
  int mid_y0, mid_rows;
  int item0;  // its first work item in this launch
  int vec_ok;
};
constexpr int kNfImages = 320;
struct NfLaunch {
  const float* lut;
  int* tables;
  uint8_t* mid;
  int n, P, resample;
  NfImage d[kNfImages];
};
static_assert(sizeof(NfLaunch) <= 32764, "kernel parameters are limited to 32764 bytes");

inline __host__ __device__ int round4(int n) { return (n + 3) & ~3; }
inline long long nf_table_ints(int oh, int ow, int hstride, int vks) {
  return 2LL * round4(ow) + static_cast<long long>(ow) * hstride + 2LL * round4(oh) + static_cast<long long>(oh) * vks;
}

__device__ __forceinline__ int nf_find(const NfLaunch& L, int item) {
  int lo = 0, hi = L.n - 1;
  while (lo < hi) {
    const int m = (lo + hi + 1) >> 1;
    if (L.d[m].item0 <= item) lo = m; else hi = m - 1;
  }
  return lo;
}

__device__ __forceinline__ KernelArgs nf_args(const NfLaunch& L, const NfImage& d) {
  KernelArgs a;
  const int* t = L.tables + d.tab;
  a.img = d.img;
  a.out = d.out;
  a.lut = L.lut;
  a.hfirst = t;
  a.hcount = t + round4(d.ow);
  a.hk = t + 2 * round4(d.ow);
  a.vfirst = a.hk + static_cast<size_t>(d.ow) * d.hstride;
  a.vcount = a.vfirst + round4(d.oh);
  a.vk = a.vcount + round4(d.oh);
  a.H = d.H; a.W = d.W; a.oh = d.oh; a.ow = d.ow; a.hks = d.hstride; a.hstride = d.hstride; a.vks = d.vks;
  a.TY = d.TY; a.rowb = d.rowb; a.stage_bytes = d.stage_bytes; a.vec_ok = d.vec_ok;
  a.P = L.P;
  a.gw = d.ow / L.P;
  return a;
}

// Pillow's filters and make_table's recipe with every double operation rounded on its own (__d*_rn): no FMA contraction moves a
// weight, so the device tables equal the host's bit for bit.
__device__ __forceinline__ double nf_filter(double x, int resample) {
  if (x < 0.0) x = -x;
  if (resample == 3) {
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
    return 0.0;
  }
  return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// Window and weights of output coordinate xx of one axis; the row of kk is padded with zero weights to `stride` taps.
__device__ void nf_axis(int in_size, int out_size, int resample, int xx, int stride, int* first, int* count, int* kk) {
  const double fsupport = resample == 3 ? 2.0 : 1.0;
  const double scale = __ddiv_rn(static_cast<double>(in_size), static_cast<double>(out_size));
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(fsupport, filterscale);
  const double ss = __ddiv_rn(1.0, filterscale);
  const double center = __dadd_rn(0.0, __dmul_rn(__dadd_rn(static_cast<double>(xx), 0.5), scale));
  int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, support), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, support), 0.5));
  if (xmax > in_size) xmax = in_size;
  xmax -= xmin;
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x)
    ww = __dadd_rn(ww, nf_filter(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss), resample));
  int* row = kk + static_cast<size_t>(xx) * stride;
  for (int x = 0; x < stride; ++x) {
    int v = 0;
    if (x < xmax) {
      const double w = nf_filter(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss), resample);
      const double k = ww != 0.0 ? __ddiv_rn(w, ww) : w;
      const double f = __dmul_rn(k, static_cast<double>(1 << kPrecisionBits));
      v = k < 0 ? static_cast<int>(__dadd_rn(-0.5, f)) : static_cast<int>(__dadd_rn(0.5, f));
    }
    row[x] = v;
  }
  first[xx] = xmin;
  count[xx] = xmax;
}

// One thread per output coordinate of every image (its ow columns, then its oh rows); items count coordinates here.
__global__ void __launch_bounds__(kThreads) nf_tables_kernel(const __grid_constant__ NfLaunch L, int items) {
  const int g = blockIdx.x * kThreads + threadIdx.x;
  if (g >= items) return;
  const NfImage& d = L.d[nf_find(L, g)];
  int* t = L.tables + d.tab;
  const int c = g - d.item0;
  if (c < d.ow) {
    nf_axis(d.W, d.ow, L.resample, c, d.hstride, t, t + round4(d.ow), t + 2 * round4(d.ow));
  } else {
    int* v = t + 2 * round4(d.ow) + static_cast<size_t>(d.ow) * d.hstride;
    nf_axis(d.H, d.oh, L.resample, c - d.ow, d.vks, v, v + round4(d.oh), v + 2 * round4(d.oh));
  }
}

// Three CTAs per SM (the occupancy of the 72 KB tier): with the bound ptxas keeps the descriptor's fields in registers instead of
// spilling one.
template <typename OUT>
__global__ void __launch_bounds__(kThreads, 3) nf_fused_kernel(const __grid_constant__ NfLaunch L) {
  extern __shared__ __align__(16) uint8_t smem[];
  const NfImage& d = L.d[nf_find(L, blockIdx.x)];
  const KernelArgs a = nf_args(L, d);
  fused_tile<OUT, kPatchRows>(a, smem, 0, blockIdx.x - d.item0);
}

__global__ void __launch_bounds__(kThreads) nf_hpass_kernel(const __grid_constant__ NfLaunch L) {
  const NfImage& d = L.d[nf_find(L, blockIdx.x)];
  const KernelArgs a = nf_args(L, d);
  const int row = blockIdx.x - d.item0;
  hpass_row(a, d.img + (static_cast<size_t>(d.mid_y0) + row) * d.W * 3, L.mid + d.mid + static_cast<size_t>(row) * d.rowb);
}

template <typename OUT>
__global__ void __launch_bounds__(kThreads) nf_vpass_kernel(const __grid_constant__ NfLaunch L) {
  const NfImage& d = L.d[nf_find(L, blockIdx.x)];
  const KernelArgs a = nf_args(L, d);
  const int yo0 = (blockIdx.x - d.item0) * d.TY;
  vertical_pass<OUT, kPatchRows>(a, reinterpret_cast<const uint32_t*>(L.mid + d.mid), d.mid_y0, yo0, min(yo0 + d.TY, d.oh), 0);
}

// The padding rows (zeros) and pixel_attention_mask of a chunk of samples, one launch: sample blockIdx.y has npatch[y] patches.
constexpr int kPadImages = 7680;
struct NfPad {
  uint8_t* out;   // the chunk's first sample
  int32_t* mask;  // nullable
  long long sample_bytes, row_bytes;
  int maxp, vec;  // vec: sample_bytes, row_bytes and out allow 16-byte stores
  int npatch[kPadImages];
};
static_assert(sizeof(NfPad) <= 32764, "kernel parameters are limited to 32764 bytes");

__global__ void __launch_bounds__(kThreads) nf_pad_kernel(const __grid_constant__ NfPad p) {
  const int b = blockIdx.y, np = p.npatch[b];
  const long long t0 = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x, step = static_cast<long long>(gridDim.x) * kThreads;
  uint8_t* o = p.out + b * p.sample_bytes + np * p.row_bytes;
  const long long bytes = (p.maxp - np) * p.row_bytes;
  if (p.vec) {
    for (long long i = t0; i < bytes / 16; i += step) reinterpret_cast<uint4*>(o)[i] = make_uint4(0, 0, 0, 0);
  } else {
    for (long long i = t0; i < bytes / 2; i += step) reinterpret_cast<uint16_t*>(o)[i] = 0;  // rows are 2-byte multiples
  }
  if (p.mask)
    for (long long j = t0; j < p.maxp; j += step) p.mask[static_cast<long long>(b) * p.maxp + j] = j < np ? 1 : 0;
}

}  // namespace
}  // namespace jimm
namespace {

struct NfWork {
  int i;  // index in the call
  SizePlan s;
  long long tab = 0, mid = 0;
};

NfImage nf_image(const NfWork& w, const uint8_t* img, void* out, int H, int W) {
  NfImage d;
  d.img = img;
  d.out = out;
  d.tab = w.tab;
  d.mid = w.mid;
  d.H = H; d.W = W; d.oh = w.s.oh; d.ow = w.s.ow;
  d.hstride = w.s.h.stride; d.vks = w.s.v.ksize; d.TY = w.s.TY; d.rowb = w.s.rowb; d.stage_bytes = w.s.stage_bytes;
  d.mid_y0 = w.s.mid_y0; d.mid_rows = w.s.mid_rows;
  d.item0 = 0;
  d.vec_ok = (reinterpret_cast<uintptr_t>(img) & 15) == 0;
  return d;
}

// Launches `kernel` over the work items of images ws[0 .. n) in chunks of kNfImages: items(w) of each, in order.  per_thread: the
// items are threads (the table kernel) rather than CTAs.  smem: dynamic shared memory of a chunk (the largest plan's).
template <bool per_thread, typename K, typename Items>
int nf_launch(K kernel, NfLaunch& L, const std::vector<const NfWork*>& ws, const std::vector<NfImage>& all, Items items, bool want_smem,
              cudaStream_t st) {
  for (size_t c0 = 0; c0 < ws.size(); c0 += kNfImages) {
    L.n = static_cast<int>(std::min<size_t>(kNfImages, ws.size() - c0));
    long long total = 0;
    size_t smem = 0;
    for (int k = 0; k < L.n; ++k) {
      const NfWork& w = *ws[c0 + k];
      L.d[k] = all[w.i];
      L.d[k].tab = w.tab;
      L.d[k].mid = w.mid;
      L.d[k].item0 = static_cast<int>(total);
      total += items(w);
      smem = std::max(smem, w.s.smem);
    }
    if (total == 0) continue;
    if (total > (per_thread ? (1LL << 31) - 1 - kThreads : (1LL << 31) - 1)) {
      set_last_error("NaFlex front-end: %lld work items in one launch", total);
      return JIMM_EINVAL;
    }
    const unsigned grid = per_thread ? static_cast<unsigned>((total + kThreads - 1) / kThreads) : static_cast<unsigned>(total);
    if constexpr (per_thread) {
      JIMM_CUDA_CHECK(launch_k(kernel, dim3(grid), dim3(kThreads), 0, st, 1, false, L, static_cast<int>(total)));
    } else {
      JIMM_CUDA_CHECK(launch_k(kernel, dim3(grid), dim3(kThreads), want_smem ? smem : 0, st, 1, false, L));
    }
    note_launch();
  }
  return 0;
}

// The work of one checked NaFlex call: tables, padding and mask, then the fused images per shared-memory tier and the two-pass
// images per chunk of intermediates.
template <typename OUT>
int nf_enqueue(const jimm_preproc* p, std::vector<NfWork>& work, const std::vector<NfImage>& all, int B, int maxp, void* pixel_values,
               int32_t* mask, cudaStream_t st) {
  JIMM_TRY(smem_opt_in<nf_fused_kernel<OUT>>(200 * 1024));
  const int P = p->naflex_patch;
  long long tab_ints = 0;
  for (NfWork& w : work) {
    w.tab = tab_ints;
    tab_ints += nf_table_ints(w.s.oh, w.s.ow, w.s.h.stride, w.s.v.ksize);
  }
  // two-pass images: chunks whose intermediates fit kMidChunkBytes (at least one image each), in call order
  std::vector<std::vector<const NfWork*>> mid_chunks;
  size_t mid_bytes = 0, chunk_bytes = 0, slack = 0;
  for (NfWork& w : work) {
    if (w.s.path != kTwoPass) continue;
    const size_t b = static_cast<size_t>(w.s.mid_rows) * w.s.rowb;
    if (mid_chunks.empty() || chunk_bytes + b > kMidChunkBytes || mid_chunks.back().size() == static_cast<size_t>(kNfImages)) {
      mid_chunks.emplace_back();
      chunk_bytes = 0;
    }
    w.mid = static_cast<long long>(chunk_bytes);
    chunk_bytes += b;
    mid_chunks.back().push_back(&w);
    mid_bytes = std::max(mid_bytes, chunk_bytes);
    slack = std::max(slack, static_cast<size_t>(w.s.v.ksize) * w.s.rowb);  // zero-weight taps past an intermediate's last rows
  }
  NfLaunch L;
  L.lut = p->lut;
  L.mid = nullptr;
  L.P = P;
  L.resample = p->cfg.resample;
  int* tables = nullptr;
  JIMM_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&tables), static_cast<size_t>(tab_ints) * sizeof(int), st));
  L.tables = tables;
  if (mid_bytes) {
    if (cudaMallocAsync(reinterpret_cast<void**>(&L.mid), mid_bytes + slack, st) != cudaSuccess) {
      cudaFreeAsync(tables, st);
      set_last_error("cudaMallocAsync of a %zu-byte NaFlex intermediate failed", mid_bytes + slack);
      return JIMM_ENOMEM;
    }
  }
  int rc = 0;
  auto run = [&]() -> int {
    std::vector<const NfWork*> every;
    for (const NfWork& w : work) every.push_back(&w);
    JIMM_TRY(nf_launch<true>(nf_tables_kernel, L, every, all, [](const NfWork& w) { return static_cast<long long>(w.s.oh) + w.s.ow; },
                             false, st));
    const size_t es = sizeof(OUT);
    NfPad pad;
    pad.row_bytes = static_cast<long long>(P) * P * 3 * es;
    pad.sample_bytes = pad.row_bytes * maxp;
    pad.maxp = maxp;
    for (int b0 = 0; b0 < B; b0 += kPadImages) {
      const int n = std::min(B - b0, kPadImages);
      pad.out = static_cast<uint8_t*>(pixel_values) + b0 * pad.sample_bytes;
      pad.mask = mask ? mask + static_cast<long long>(b0) * maxp : nullptr;
      pad.vec = pad.row_bytes % 16 == 0 && reinterpret_cast<uintptr_t>(pad.out) % 16 == 0;
      long long most = maxp;  // the mask's entries, or the 16- / 2-byte stores of the largest padding
      for (int k = 0; k < n; ++k) {
        const NfWork& w = work[b0 + k];
        pad.npatch[k] = (w.s.oh / P) * (w.s.ow / P);
        most = std::max(most, (maxp - pad.npatch[k]) * pad.row_bytes / (pad.vec ? 16 : 2));
      }
      const unsigned gx = static_cast<unsigned>(std::min<long long>((most + kThreads - 1) / kThreads, 64));
      JIMM_CUDA_CHECK(launch_k(nf_pad_kernel, dim3(gx, n), dim3(kThreads), 0, st, 1, false, pad));
      note_launch();
    }
    for (int tier = 0; tier < 3; ++tier) {
      std::vector<const NfWork*> ws;
      for (const NfWork& w : work)
        if (w.s.path == kFused && w.s.tier == tier) ws.push_back(&w);
      JIMM_TRY(nf_launch<false>(nf_fused_kernel<OUT>, L, ws, all,
                                [](const NfWork& w) { return static_cast<long long>((w.s.oh + w.s.TY - 1) / w.s.TY); }, true, st));
    }
    for (const auto& ws : mid_chunks) {
      JIMM_TRY(nf_launch<false>(nf_hpass_kernel, L, ws, all, [](const NfWork& w) { return static_cast<long long>(w.s.mid_rows); }, false, st));
      JIMM_TRY(nf_launch<false>(nf_vpass_kernel<OUT>, L, ws, all,
                                [](const NfWork& w) { return static_cast<long long>((w.s.oh + w.s.TY - 1) / w.s.TY); }, false, st));
    }
    return 0;
  };
  rc = run();
  const cudaError_t f1 = cudaFreeAsync(tables, st);
  const cudaError_t f2 = L.mid ? cudaFreeAsync(L.mid, st) : cudaSuccess;
  if (rc == 0 && (f1 != cudaSuccess || f2 != cudaSuccess)) {
    set_last_error("cudaFreeAsync -> %s", cudaGetErrorString(f1 != cudaSuccess ? f1 : f2));
    return JIMM_ECUDA;
  }
  return rc;
}

// The rescale / normalise table of a handle (both kinds): transformers rescale + normalize of one 8-bit sample,
// float32(float64(v) * factor), then (x - float32(mean)) / float32(std).
int make_lut(jimm_preproc* p, const jimm_preproc_config_t* cfg) {
  std::vector<float> lut(3 * 256);
  for (int c = 0; c < 3; ++c)
    for (int v = 0; v < 256; ++v) {
      const float x = static_cast<float>(static_cast<double>(v) * cfg->rescale_factor);
      volatile float d = x - cfg->mean[c];  // volatile: keep the two roundings separate
      lut[c * 256 + v] = d / cfg->std[c];
    }
  void* d = nullptr;
  if (cudaMalloc(&d, lut.size() * sizeof(float)) != cudaSuccess) { set_last_error("cudaMalloc failed"); return JIMM_ENOMEM; }
  p->lut = static_cast<float*>(d);
  p->allocs.push_back(d);
  if (cudaMemcpy(d, lut.data(), lut.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
    set_last_error("cudaMemcpy failed");
    return JIMM_ECUDA;
  }
  return 0;
}

}  // namespace

extern "C" {

int jimm_preproc_create(const jimm_preproc_config_t* cfg, int device, jimm_preproc_t** out) {
  JIMM_TRY(check_cfg(cfg));
  if (!out) { set_last_error("null output handle"); return JIMM_EINVAL; }
  JIMM_CUDA_CHECK(cudaSetDevice(device));
  jimm_preproc* p = new jimm_preproc();
  p->cfg = *cfg;
  p->device = device;
  if (const int rc = make_lut(p, cfg)) {
    for (void* d : p->allocs) cudaFree(d);
    delete p;
    return rc;
  }
  *out = p;
  return 0;
}

int jimm_preproc_create_naflex(const jimm_preproc_config_t* cfg, int patch, int device, jimm_preproc_t** out) {
  if (!cfg || !out) { set_last_error("jimm_preproc_create_naflex: null argument"); return JIMM_EINVAL; }
  if (cfg->resample != 2 && cfg->resample != 3) { set_last_error("resample must be 2 (bilinear) or 3 (bicubic), got %d", cfg->resample); return JIMM_EINVAL; }
  if (cfg->height || cfg->width || cfg->shortest_edge || cfg->crop_h || cfg->crop_w) {
    set_last_error("a NaFlex front-end sizes every image by its patch budget: height, width, shortest_edge, crop_h and crop_w must be 0");
    return JIMM_EINVAL;
  }
  for (int i = 0; i < 3; ++i)
    if (cfg->std[i] == 0.f) { set_last_error("std evaluated to zero, leading to division by zero."); return JIMM_EINVAL; }
  if (patch < 1) { set_last_error("NaFlex patch size %d: must be at least 1", patch); return JIMM_EINVAL; }
  JIMM_CUDA_CHECK(cudaSetDevice(device));
  jimm_preproc* p = new jimm_preproc();
  p->cfg = *cfg;
  p->device = device;
  p->naflex_patch = patch;
  if (const int rc = make_lut(p, cfg)) {
    for (void* d : p->allocs) cudaFree(d);
    delete p;
    return rc;
  }
  *out = p;
  return 0;
}

int jimm_preproc_naflex_grid(int patch, int max_num_patches, int H, int W, int* gh, int* gw) {
  int r = 0, c = 0;
  JIMM_TRY(naflex_grid(patch, max_num_patches, H, W, &r, &c));
  if (gh) *gh = r;
  if (gw) *gw = c;
  return 0;
}

int jimm_preproc_run_naflex(jimm_preproc_t* p, const uint8_t* const* imgs, int B, const int* H, const int* W, int max_num_patches,
                            void* pixel_values, int out_dtype, int32_t* mask, int* grid, void* stream) {
  if (!p) { set_last_error("jimm_preproc_run_naflex: null argument"); return JIMM_EINVAL; }
  if (!p->naflex_patch) {
    set_last_error("jimm_preproc_run_naflex: the handle has a fixed output size (jimm_preproc_create); NaFlex calls need a handle from "
                   "jimm_preproc_create_naflex");
    return JIMM_EINVAL;
  }
  if (B < 0) { set_last_error("jimm_preproc_run_naflex: batch %d", B); return JIMM_EINVAL; }
  if (B == 0) return 0;
  if (!imgs || !H || !W || !pixel_values) { set_last_error("jimm_preproc_run_naflex: null argument"); return JIMM_EINVAL; }
  if (max_num_patches < 1) { set_last_error("max_num_patches %d: must be at least 1", max_num_patches); return JIMM_EINVAL; }
  if (out_dtype < JIMM_F32 || out_dtype > JIMM_BF16) { set_last_error("bad output dtype %d", out_dtype); return JIMM_EINVAL; }
  const size_t es = out_dtype == JIMM_F32 ? 4 : 2;
  if (reinterpret_cast<uintptr_t>(pixel_values) % (4 * es)) {
    set_last_error("pixel_values must be %zu-byte aligned for this dtype", 4 * es);
    return JIMM_EINVAL;
  }
  if (reinterpret_cast<uintptr_t>(mask) % 4) { set_last_error("mask must be 4-byte aligned"); return JIMM_EINVAL; }
  const int P = p->naflex_patch;
  const size_t sample = static_cast<size_t>(max_num_patches) * P * P * 3 * es;
  std::vector<NfWork> work(B);
  std::vector<NfImage> all(B);
  std::vector<int> shapes(2 * static_cast<size_t>(B));
  for (int i = 0; i < B; ++i) {
    auto refuse = [i]() {
      const std::string m = last_error_message();
      set_last_error("image %d: %s", i, m.c_str());
      return JIMM_EINVAL;
    };
    if (!imgs[i]) { set_last_error("image %d: null frame pointer", i); return JIMM_EINVAL; }
    int gh = 0, gw = 0;
    if (naflex_grid(P, max_num_patches, H[i], W[i], &gh, &gw)) return refuse();
    const long long th = static_cast<long long>(gh) * P, tw = static_cast<long long>(gw) * P;
    if (th > kMaxResizedEdge || tw > kMaxResizedEdge) {
      set_last_error("image %d: resize %dx%d -> %lldx%lld: the front-end resizes to at most %d pixels per edge", i, H[i], W[i], th, tw,
                     kMaxResizedEdge);
      return JIMM_EINVAL;
    }
    jimm_preproc_config_t c = p->cfg;
    c.height = static_cast<int>(th);
    c.width = static_cast<int>(tw);
    ResampleTable tx, ty;
    if (plan_size(c, H[i], W[i], &work[i].s, &tx, &ty, false)) return refuse();
    work[i].i = i;
    all[i] = nf_image(work[i], imgs[i], static_cast<uint8_t*>(pixel_values) + i * sample, H[i], W[i]);
    shapes[2 * i] = gh;
    shapes[2 * i + 1] = gw;
  }
  if (grid) std::copy(shapes.begin(), shapes.end(), grid);
  JIMM_CUDA_CHECK(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (out_dtype == JIMM_F32) return nf_enqueue<float>(p, work, all, B, max_num_patches, pixel_values, mask, st);
  if (out_dtype == JIMM_F16) return nf_enqueue<__half>(p, work, all, B, max_num_patches, pixel_values, mask, st);
  return nf_enqueue<__nv_bfloat16>(p, work, all, B, max_num_patches, pixel_values, mask, st);
}

int jimm_preproc_output_size(const jimm_preproc_t* p, int H, int W, int* out_h, int* out_w) {
  if (!p) { set_last_error("bad arguments"); return JIMM_EINVAL; }
  if (p->naflex_patch) {
    set_last_error("jimm_preproc_output_size: a NaFlex handle sizes every image by its patch budget; use jimm_preproc_naflex_grid");
    return JIMM_EINVAL;
  }
  SizePlan s;
  bool known = false;
  {
    std::lock_guard<std::mutex> lock(p->mu);
    auto it = p->plans.find({H, W});
    if (it != p->plans.end()) { s = it->second; known = true; }
  }
  if (!known) {  // the planner jimm_preproc_run uses: a size it would refuse is refused here, before a caller stages anything
    ResampleTable th, tv;
    JIMM_TRY(plan_size(p->cfg, H, W, &s, &th, &tv));
  }
  if (out_h) *out_h = s.oh;
  if (out_w) *out_w = s.ow;
  return 0;
}

int jimm_preproc_run(jimm_preproc_t* p, const uint8_t* img, int B, int H, int W, void* out, int out_dtype, void* stream) {
  if (!p || !img || !out) { set_last_error("null argument"); return JIMM_EINVAL; }
  if (p->naflex_patch) {
    set_last_error("jimm_preproc_run: a NaFlex handle has no fixed output size; use jimm_preproc_run_naflex");
    return JIMM_EINVAL;
  }
  if (B <= 0) return 0;
  if (out_dtype < JIMM_F32 || out_dtype > JIMM_BF16) { set_last_error("bad output dtype %d", out_dtype); return JIMM_EINVAL; }
  // the kernels store four samples at once wherever the index allows: out must be aligned for that
  const size_t vec_bytes = out_dtype == JIMM_F32 ? 16 : 8;
  if (reinterpret_cast<uintptr_t>(out) % vec_bytes) {
    set_last_error("output pointer must be %zu-byte aligned for this dtype", vec_bytes);
    return JIMM_EINVAL;
  }
  JIMM_CUDA_CHECK(cudaSetDevice(p->device));
  SizePlan* s = nullptr;
  JIMM_TRY(get_plan(p, H, W, &s));
  KernelArgs a;
  a.img = img;
  a.out = out;
  a.lut = p->lut;
  a.hfirst = s->h.first;  // tables of the cropped columns and rows only
  a.hcount = s->h.count;
  a.hk = s->h.kk;
  a.vfirst = s->v.first;
  a.vcount = s->v.count;
  a.vk = s->v.kk;
  a.H = H; a.W = W; a.oh = s->oh; a.ow = s->ow; a.hks = s->h.ksize; a.hstride = s->h.stride; a.vks = s->v.ksize;
  a.TY = s->TY; a.rowb = s->rowb; a.stage_bytes = s->stage_bytes;
  a.vec_ok = (reinterpret_cast<uintptr_t>(img) & 15) == 0;
  a.P = a.gw = 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (out_dtype == JIMM_F32) return run_sized<float>(*s, a, B, st);
  if (out_dtype == JIMM_F16) return run_sized<__half>(*s, a, B, st);
  return run_sized<__nv_bfloat16>(*s, a, B, st);
}

int jimm_preproc_destroy(jimm_preproc_t* p) {
  if (!p) return 0;
  cudaSetDevice(p->device);
  for (void* d : p->allocs) cudaFree(d);
  delete p;
  return 0;
}

// Host-only: the resampling tables, for the CPU test that pins them to the oracle's.
int jimm_k_resample_coeffs(int in_size, int out_size, int resample, int* ksize, int* first, int* count, int* kk, int kk_capacity) {
  if (in_size <= 0 || out_size <= 0 || (resample != 2 && resample != 3)) { set_last_error("bad arguments"); return JIMM_EINVAL; }
  ResampleTable t = make_table(in_size, out_size, resample);
  if (ksize) *ksize = t.ksize;
  if (first) for (int i = 0; i < out_size; ++i) first[i] = t.first[i];
  if (count) for (int i = 0; i < out_size; ++i) count[i] = t.count[i];
  if (kk) {
    if (kk_capacity < out_size * t.ksize) { set_last_error("kk buffer too small: %d < %d", kk_capacity, out_size * t.ksize); return JIMM_EINVAL; }
    for (int i = 0; i < out_size * t.ksize; ++i) kk[i] = t.kk[i];
  }
  return 0;
}

// Device tables of the NaFlex front-end for one axis, read back for the test that pins them to make_table's.  The table kernel
// builds both axes of an in_size x in_size -> out_size x out_size image; the two must agree, and the zero-weight padding of each
// row must be zero.  Synchronises (a test hook).
int jimm_k_resample_coeffs_device(int in_size, int out_size, int resample, int* first, int* count, int* kk, int kk_capacity) {
  if (in_size <= 0 || out_size <= 0 || (resample != 2 && resample != 3) || !first || !count || !kk) {
    set_last_error("bad arguments");
    return JIMM_EINVAL;
  }
  const ResampleTable t = make_table(in_size, out_size, resample, 0, -1, false);
  if (kk_capacity < static_cast<long long>(out_size) * t.ksize) { set_last_error("kk buffer too small: %d < %d", kk_capacity, out_size * t.ksize); return JIMM_EINVAL; }
  NfWork w;
  w.i = 0;
  w.s.oh = w.s.ow = out_size;
  w.s.h.stride = w.s.v.ksize = t.kpad;
  static NfLaunch L;  // 28 KB: off the stack
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  L.lut = nullptr;
  L.mid = nullptr;
  L.n = 1;
  L.P = 1;
  L.resample = resample;
  L.d[0] = nf_image(w, nullptr, nullptr, in_size, in_size);
  const long long ints = nf_table_ints(out_size, out_size, t.kpad, t.kpad);
  JIMM_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&L.tables), ints * sizeof(int)));
  std::vector<int> h(ints);
  cudaError_t e = launch_k(nf_tables_kernel, dim3((2 * out_size + kThreads - 1) / kThreads), dim3(kThreads), 0, nullptr, 1, false, L,
                           2 * out_size);
  if (e == cudaSuccess) e = cudaMemcpy(h.data(), L.tables, ints * sizeof(int), cudaMemcpyDeviceToHost);
  cudaFree(L.tables);
  if (e != cudaSuccess) { set_last_error("jimm_k_resample_coeffs_device: %s", cudaGetErrorString(e)); return JIMM_ECUDA; }
  note_launch();
  const int o4 = round4(out_size);
  const int* hf = h.data();
  const int* vf = hf + 2 * o4 + static_cast<size_t>(out_size) * t.kpad;
  for (int i = 0; i < out_size; ++i) {
    const int* row = hf + 2 * o4 + static_cast<size_t>(i) * t.kpad;
    const int* vrow = vf + 2 * o4 + static_cast<size_t>(i) * t.kpad;
    if (hf[i] != vf[i] || hf[o4 + i] != vf[o4 + i] || !std::equal(row, row + t.kpad, vrow)) {
      set_last_error("jimm_k_resample_coeffs_device: the two axes' tables differ at output %d", i);
      return JIMM_EINVAL;
    }
    first[i] = hf[i];
    count[i] = hf[o4 + i];
    for (int k = 0; k < t.kpad; ++k) {
      if (k < t.ksize) kk[static_cast<size_t>(i) * t.ksize + k] = row[k];
      else if (row[k] != 0) { set_last_error("jimm_k_resample_coeffs_device: non-zero padding tap in row %d", i); return JIMM_EINVAL; }
    }
  }
  return 0;
}

// Host-only: the plan jimm_preproc_run would use for H x W frames, for the CPU tests that pin the planner.
int jimm_k_preproc_plan(const jimm_preproc_config_t* cfg, int H, int W, int* path, int* tier, int* TY, long long* smem) {
  JIMM_TRY(check_cfg(cfg));
  SizePlan s;
  ResampleTable th, tv;
  JIMM_TRY(plan_size(*cfg, H, W, &s, &th, &tv));
  if (path) *path = s.path;
  if (tier) *tier = s.tier;
  if (TY) *TY = s.TY;
  if (smem) *smem = static_cast<long long>(s.smem);
  return 0;
}

}  // extern "C"
