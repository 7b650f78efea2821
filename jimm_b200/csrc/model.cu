// Model state, weight packing, forward orchestration and the C ABI (include/jimm_b200.h).
//
// Host-side structure mirrors the reference's module tree:
//   Tower (VisionTransformerBase, common/vit.py:104-248)  -> patch GEMM, cls/pos, [ln_pre], L x Block, ln_post, CLS | MAP head
//   Block (TransformerEncoder, common/transformer.py:22-132)
//   TextTower (nnx.Embed + Transformer + ln_final + pooling; models/clip.py:148-167, models/siglip.py:135-153)
//   heads (classifier / visual_projection / text_projection; contrastive logits)
// All arithmetic is in the kernels of gemm.cu / attention.cu / elementwise.cu / comm.cu; there is no CPU fallback.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <map>
#include <tuple>
#include <memory>
#include <utility>
#include <string>
#include <vector>

#include "../../include/jimm_b200.h"
#include "comm.cuh"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

namespace jimm {

// ------------------------------------------------------------------------------------------
// error + launch accounting
// ------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error_message() { return g_err; }
static std::atomic<long long> g_launches{0};
static std::atomic<long long> g_graph_replays{0};
// Small-batch forwards are captured in cudaStreamCaptureModeRelaxed, so CUDA does not stop another thread's potentially unsafe calls
// (cudaMalloc / cudaFree / cudaHostAlloc / cudaFreeHost / device or legacy-stream synchronisation) while a capture is open, and their
// effect on it is undefined.  Distinct handles may live in distinct threads: the library's own such phases -- finalize, destroy, the
// growth of a host-path staging buffer -- hold this lock, and a capture only starts when it can take it (otherwise that call runs
// eagerly and a later one captures).  The ingestion test entry points (kernel_api.cu) take it too.
std::mutex g_capture_mu;
static thread_local long long t_launches = 0;  // launches of the calling thread (what a capture on it recorded)
void note_launch() {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  ++t_launches;
}
int pdl_enabled() {
  static const int v = [] { const char* env = getenv("JIMM_PDL"); return env ? atoi(env) : 1; }();  // thread-safe static init
  return v;
}

#define JIMM_TRY(expr)          \
  do {                          \
    int _rc = (expr);           \
    if (_rc != 0) return _rc;   \
  } while (0)

// ------------------------------------------------------------------------------------------
// small RAII-free device memory pool (freed in model destroy)
// ------------------------------------------------------------------------------------------
struct DevPool {
  std::vector<void*> ptrs;
  size_t bytes = 0;
  int alloc(void** out, size_t n) {
    if (n == 0) n = 16;
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, n);
    if (e != cudaSuccess) {
      set_last_error("cudaMalloc(%zu bytes) failed: %s", n, cudaGetErrorString(e));
      return JIMM_ENOMEM;
    }
    ptrs.push_back(p);
    bytes += n;
    *out = p;
    return 0;
  }
  template <typename T>
  int alloc(T** out, size_t n) {
    void* p = nullptr;
    JIMM_TRY(alloc(&p, n));
    *out = static_cast<T*>(p);
    return 0;
  }
  void release() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
    bytes = 0;
  }
};

struct HostParam {
  std::vector<int64_t> shape;   // the reference's flax shape
  std::vector<float> data;      // owned fp32 copy (jimm_model_set_param) ...
  const void* ref = nullptr;    // ... or a borrowed host pointer (jimm_model_set_param_ref), valid until finalize returns
  int dtype = DT_F32;           // element type behind ptr()
  bool transposed = false;      // ref holds the 2-D transpose [N, K] of the flax kernel's (K, N) view (a HuggingFace (out, in) weight as is)
  bool used = false;
  size_t n = 0;
  size_t numel() const { return n; }
  const void* ptr() const { return ref ? ref : static_cast<const void*>(data.data()); }
  size_t esize() const { return dtype == DT_F32 ? 4 : 2; }
  float at(size_t i) const {  // host-side read of element i of the STORED order
    if (dtype == DT_F32) return static_cast<const float*>(ptr())[i];
    const uint16_t h = static_cast<const uint16_t*>(ptr())[i];
    if (dtype == DT_BF16) { uint32_t u = static_cast<uint32_t>(h) << 16; float f; memcpy(&f, &u, 4); return f; }
    return __half2float(*reinterpret_cast<const __half*>(&h));
  }
};

struct LinearW {
  void* w = nullptr;   // [N, K] compute dtype, K-major (e4m3 for the FP8 mode's QKV / FC1)
  float* b = nullptr;  // [N] fp32 or null
  float* ws = nullptr; // [N] fp32 row scales of an e4m3 w, else null
  int N = 0, K = 0;
};
struct LNW {
  float* scale = nullptr;
  float* bias = nullptr;
};
struct BlockW {
  LNW norm1, norm2;
  LinearW qkv, out, fc1, fc2;
  GemmPlan p_qkv, p_out, p_fc1, p_fc2;
};

struct EncoderCfg {  // one Transformer stack
  int D = 0, H = 0, M = 0, L = 0, act = 0, causal = 0;
  float eps = 1e-6f;
};

struct Encoder {
  EncoderCfg c;
  std::vector<BlockW> blocks;
};

struct VisionTower {
  bool present = false;
  int img = 0, P = 0, C = 0, D = 0, n = 0, n_pad = 0, S = 0, pooling = 0, pre_norm = 0, patch_bias = 0;
  int Kp = 0;  // patch GEMM K = P*P*C rounded up to a multiple of 8 (16-byte rows for TMA; the pad columns are zeros on both operands)
  bool patch_scatter = false;  // patch GEMM reduce-adds into the pos-initialised residual stream through a 3-D TMA map
  int interp = POS_BICUBIC;    // how the position table is resampled to another patch grid (antialiased bilinear for SigLIP 2 NaFlex)
  float eps_outer = 1e-5f;
  Encoder enc;
  LinearW patch;
  float* cls = nullptr;
  float* pos = nullptr;  // [S, D]
  LNW ln_pre, ln_post;
  // MAP head
  float* map_q = nullptr;  // [D] fp32: probe . Wq + bq (input independent)
  LinearW map_kv, map_out, map_fc1, map_fc2;
  LNW map_ln;
  // head after pooling (classifier / visual_projection); N == 0 -> none
  LinearW head;
  GemmPlan p_patch, p_head, p_map_kv, p_map_out, p_map_fc1, p_map_fc2;
  // packed calls (jimm_vit_forward_packed): plain fp32 acc + bias over patch rows laid out like the tokens they become (a CLS row's
  // A row is never written and its output is overwritten), straight into the residual stream
  GemmPlan p_patch_packed;
};

struct TextTower {
  bool present = false;
  int T = 0, V = 0, D = 0, pool = 0;
  float eps_outer = 1e-5f;
  Encoder enc;
  float* table = nullptr;  // [V, D] fp32
  float* pos = nullptr;    // [T, D] fp32
  LNW ln_final;
  LinearW head;  // text_projection
  GemmPlan p_head;
  GemmPlan p_head_packed;  // packed calls (jimm_encode_text_packed): the pooled rows of up to TextWs::pk_seqs sequences, read from enc.h
};

struct EncBufs {  // the activation buffers one encoder stack works in, for `rows` rows of width D (alloc_stack)
  float* x = nullptr;     // fp32 residual stream [rows, D]
  void* h = nullptr;      // LN out / attention out (compute dtype) [rows, D]
  void* big = nullptr;    // qkv | mlp hidden, and in the vision tower patches | MAP k,v (aliased; disjoint lifetimes; big_bytes)
  int* ln_cnt = nullptr;  // completion counters of the fused LayerNorm (one per 32 rows, zero between launches; null = LayerNorm stays a kernel)
  void* h8 = nullptr;     // FP8 mode: e4m3 block LayerNorm out [rows, D] (QKV / FC1 A operand) and its row scales [rows]; null otherwise
  float* sa = nullptr;
};

// The text tower has its own residual stream / activation buffers so that the two towers of CLIP / SigLIP can run CONCURRENTLY on two
// streams (they are independent until the contrastive head): the tail rounds of one tower's persistent GEMMs and its small kernels are
// filled by the other tower's CTAs instead of leaving SMs idle.
struct TextWs {
  EncBufs enc;            // [Bmax*T, Dt]
  void* pooled = nullptr; // [Bmax, Dt]
  int* idx = nullptr;     // [Bmax] EOT positions
  // packed calls: int32 token offsets [pk_seqs + 1] and pooled rows [pk_seqs] of the sequences of a chunk.  A chunk holds as many
  // sequences as fit the Bmax*T token rows, up to the attention grid's 65535 samples.  Apart from ws.pk_meta, so that a packed text call
  // on the text side stream may overlap a packed image call.
  int* pk_meta = nullptr;
  int pk_seqs = 0;
};

struct Workspace {
  EncBufs enc;            // [Tmax, D] (ws_rows x D), ws.big ws_big bytes
  void* pooled = nullptr; // [Bmax, D] compute dtype
  float* feat = nullptr;  // [Bmax, D] fp32 (MAP attention out-proj / residual)
  void* mid2 = nullptr;   // [Bmax, M] compute dtype (MAP MLP hidden, M = vis.map_fc1.N)
  float* emb_i = nullptr; // [Bmax, E] fp32 encoder outputs
  float* emb_t = nullptr;
  float* nrm_i = nullptr; // normalised
  float* nrm_t = nullptr;
  void* in_img = nullptr; // host-path staging: image batch (fp32 worst case)
  uint8_t* in_u8 = nullptr;  // host-path staging of raw uint8 RGB frames (jimm_vit_forward_host_u8); grown on demand
  size_t in_u8_bytes = 0;
  int32_t* in_ids = nullptr;
  float* out_dev = nullptr;  // host-path staging for results
  size_t out_dev_elems = 0;
  int* pk_meta = nullptr;    // packed calls: int32 token offsets [Bmax + 1] and grid widths [Bmax] of the images of a chunk
};

// A vision forward on a patch grid other than the trained one (jimm_vit_forward_hw & co.): gh x gw patches, S tokens per image, the
// patch GEMM for this grid and the most images the workspace holds at once.  Host-side state only (tensor maps into the workspace).
struct PatchGrid {
  int gh = 0, gw = 0, n = 0, n_pad = 0, S = 0, chunk = 0;
  GemmPlan patch;
};

}  // namespace jimm

using namespace jimm;

struct jimm_model {
  jimm_config_t cfg;
  int device = 0;
  bool finalized = false;
  int max_batch = 0;
  int max_tokens = 0;        // jimm_model_set_max_tokens: vision tokens per sample the workspace holds (the native count when lower)
  size_t ws_rows = 0;        // residual-stream rows of the vision workspace (x, h, ln_cnt, h8 / sa, the encoder plans' M)
  size_t ws_big = 0;         // bytes of ws.big
  static constexpr size_t kMaxGrids = 16;
  std::map<std::pair<int, int>, PatchGrid> grids;  // off-grid plans by (gh, gw), built on first use
  int cdt = DT_F16;    // compute dtype of GEMM operands
  int adt = DT_F16;    // dtype of the qkv / MAP-kv buffers consumed by the attention kernels (16-bit even in fp32 mode)
  // FP8 compute mode (JIMM_F8E4M3): cdt / adt are fp16, except that the QKV and FC1 GEMMs of every encoder block take e4m3 operands
  // with power-of-two scales per A row (written by the block LayerNorms) and per weight row (computed at finalize)
  bool f8 = false;
  std::map<std::string, HostParam> host;
  DevPool pool;
  VisionTower vis;
  TextTower txt;
  float* logit_scale = nullptr;
  float* logit_bias = nullptr;
  Workspace ws;
  TextWs wt;
  // two-stream execution of the dual towers (JIMM_DUAL_STREAMS=0 disables): text tower on `text_stream`, forked from / joined to the
  // caller's stream with events
  bool dual_streams = true;
  cudaStream_t text_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  float* graph_out_t = nullptr;  // text-tower twin of graph_out
  CommState comm;
  cudaStream_t copy_stream = nullptr;            // host path: H2D of chunk i+1 overlaps the forward of chunk i
  static constexpr int kHostSlices = 4;
  cudaEvent_t ev_copied[kHostSlices] = {};
  cudaEvent_t ev_consumed[kHostSlices] = {};
  cudaEvent_t ev_start = nullptr;
  // Back-to-back host-path calls on one stream are ordered slot by slot (a slot is free again once its slice has been through
  // patchify), so the copies of call k+1 run under the towers of call k: the asynchronous-dispatch pipeline of the reference.
  bool host_chain = false;            // the last toucher of the staging buffer was jimm_vit_forward_host ...
  cudaStream_t host_chain_stream = nullptr;  // ... on this stream ...
  int host_chain_sizes[kHostSlices] = {};    // ... with this slice layout
  int host_chain_kind = 0;                   // ... 0: float images into in_img, 1: uint8 frames into in_u8 (+ front-end into in_img)
  bool slot_recorded[kHostSlices] = {};
  bool prof_on = false;
  std::vector<cudaEvent_t> prof_ev;
  size_t prof_used = 0;
  double prof_flops = 0.0;
  long long prof_launches = 0;
  int epi_mode_16 = 2;  // epilogue mode for 16-bit no-residual outputs (2 = TMA store)
  int epi_mode_res = 2; // epilogue mode for fp32 residual outputs (2 = TMA reduce-add into the residual stream)
  bool l2_alternate = true;  // JIMM_L2_ALTERNATE=0 disables the alternating walk direction
  // JIMM_FUSE_LN=1: the out-proj / FC2 GEMMs normalise the rows they complete (gemm.cu, "fused LayerNorm").  Off by default: it removes
  // two launches per block, but the row read-back competes with the GEMM's own TMA traffic for L2 bandwidth.  Kept for A/B runs and
  // covered by tests.
  bool fuse_ln = false;
  bool simt = false;    // JIMM_GEMM_IMPL=simt: bisection aid, routes every GEMM through the SIMT cross-check kernel
  // CUDA-graph replay of a whole tower for small batches (launch-bound regime; config 1 is B=4): the second call of a
  // (tower, batch, dtype | length) shape is stream-captured from fixed staging buffers, later calls replay it.
  struct GraphEntry {
    cudaGraphExec_t exec = nullptr;
    long long launches = 0;
    int seen = 0;
  };
  std::map<std::tuple<int, int, int>, GraphEntry> graphs;
  int graph_max_batch = 32;  // JIMM_GRAPH_MAX_BATCH (0 disables)
  float* graph_out = nullptr;  // [graph_max_batch, max(vision out, E)]
  cudaStream_t capture_stream = nullptr;
};

namespace jimm {

static size_t cdt_size(const jimm_model* m) { return dtype_size(m->cdt); }

// CLIP, SigLIP and SigLIP 2 NaFlex: a vision and a text tower and the contrastive head
static bool dual_kind(int kind) { return kind == JIMM_CLIP || kind == JIMM_SIGLIP || kind == JIMM_SIGLIP_NAFLEX; }

// The buffers of an encoder stack over `rows` rows of width D, with `big` bytes of b->big.
static int alloc_stack(jimm_model* m, size_t rows, size_t D, size_t big, EncBufs* b) {
  *b = EncBufs{};
  JIMM_TRY(m->pool.alloc(&b->x, rows * D * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&b->h, rows * D * cdt_size(m)));
  JIMM_TRY(m->pool.alloc(&b->big, big));
  // zeroed completion counters of the fused LayerNorm; not in FP8 mode, where the block LayerNorms write e4m3 rows with a row scale,
  // which only the LayerNorm kernel computes
  if (m->fuse_ln && !m->simt && m->epi_mode_res == 2 && !m->f8) {
    const size_t n = (rows + 31) / 32 + 1;
    JIMM_TRY(m->pool.alloc(&b->ln_cnt, n * sizeof(int)));
    JIMM_CUDA_CHECK(cudaMemset(b->ln_cnt, 0, n * sizeof(int)));
  }
  if (m->f8) {
    JIMM_TRY(m->pool.alloc(&b->h8, rows * D));
    JIMM_TRY(m->pool.alloc(&b->sa, rows * sizeof(float)));
  }
  return 0;
}

// Bytes of the vision tower's ws.big for a chunk of T tokens whose patch-GEMM operand has patch_rows rows.  The buffer holds one phase
// at a time: the patch operand, the 16-bit qkv, the MLP hidden layer or the MAP head's 16-bit k | v.  Finalize sizes ws.big with it and
// every chunk is admitted by it (grid_chunk, packed_fit), so no chunk outgrows the allocation.
static size_t big_bytes(const jimm_model* m, size_t T, size_t patch_rows) {
  const VisionTower& v = m->vis;
  const size_t cs = cdt_size(m), D = v.D;
  size_t b = std::max({patch_rows * v.Kp * cs, T * 3 * D * 2, T * v.enc.c.M * cs});
  if (v.pooling == JIMM_POOL_MAP) b = std::max(b, T * 2 * D * 2);
  return b;
}

// ------------------------------------------------------------------------------------------
// parameter upload / packing helpers (finalize)
// ------------------------------------------------------------------------------------------
struct Packer {
  jimm_model* m;
  UploadRing ring;
  cudaStream_t stream = 0;
  bool f32_tmp = false;  // pack weights as fp32 into a temporary buffer (the e4m3 quantiser's input), see e4m3()
  int wtype() const { return f32_tmp ? DT_F32 : m->cdt; }

  // one synchronisation for the whole finalize
  void done() {
    cudaStreamSynchronize(stream);
    ring.destroy();
  }

  HostParam* find(const std::string& name, std::initializer_list<int64_t> shape) {
    auto it = m->host.find(name);
    if (it == m->host.end()) {
      set_last_error("finalize: parameter '%s' was never set (the reference asserts every flax param is visited, models/vit.py:259)", name.c_str());
      return nullptr;
    }
    HostParam& hp = it->second;
    std::vector<int64_t> want(shape);
    if (hp.shape != want) {
      std::string got, exp;
      for (auto d : hp.shape) got += std::to_string(d) + ",";
      for (auto d : want) exp += std::to_string(d) + ",";
      set_last_error("finalize: shape mismatch for '%s': expected (%s) got (%s)", name.c_str(), exp.c_str(), got.c_str());
      return nullptr;
    }
    hp.used = true;
    return &hp;
  }

  // `rows` rows of K stored elements -> dst[r * ldd + k] of out_type, streamed through the ring in row chunks
  int rows_to_device(const HostParam* hp, size_t rows, size_t K, void* dst, int out_type, size_t ldd) {
    return upload_rows(ring, hp->ptr(), hp->dtype, rows, K, dst, out_type, ldd, stream);
  }

  // fp32 vector / tensor uploaded element for element (biases, LayerNorm, cls, pos, embedding table, scalars)
  int upload_f32(const std::string& name, std::initializer_list<int64_t> shape, float** out) {
    HostParam* hp = find(name, shape);
    if (!hp) return JIMM_ESTATE;
    if (hp->transposed) { set_last_error("finalize: '%s' cannot be handed over transposed", name.c_str()); return JIMM_EINVAL; }
    void* d = nullptr;
    JIMM_TRY(m->pool.alloc(&d, hp->numel() * sizeof(float)));
    // 2-D tensors go row by row so that a long table streams through the ring in row chunks
    const size_t K = hp->shape.empty() ? 1 : static_cast<size_t>(hp->shape.back());
    const size_t rows = K ? hp->numel() / K : 0;
    JIMM_TRY(rows_to_device(hp, rows, K, d, DT_F32, K));
    *out = static_cast<float*>(d);
    return 0;
  }
  int upload_ln(const std::string& prefix, int D, LNW* ln) {
    JIMM_TRY(upload_f32(prefix + ".scale", {D}, &ln->scale));
    JIMM_TRY(upload_f32(prefix + ".bias", {D}, &ln->bias));
    return 0;
  }
  // flax kernel viewed as (K, N) row-major  ->  rows [n0, n0+N) of a packed [Ntot, ldd] K-major operand (ldd >= K: zero-padded K)
  int pack_kernel(const std::string& name, std::initializer_list<int64_t> shape, int K, int N, void* dst_base, int n0, int ldd = 0) {
    if (ldd <= 0) ldd = K;
    HostParam* hp = find(name, shape);
    if (!hp) return JIMM_ESTATE;
    if (hp->numel() != static_cast<size_t>(K) * N) { set_last_error("finalize: '%s' numel mismatch", name.c_str()); return JIMM_ESTATE; }
    return upload_kernel(ring, hp->ptr(), hp->dtype, K, N, hp->transposed, dst_base, wtype(), ldd, n0, stream);
  }
  int alloc_linear(LinearW* lw, int N, int K, bool bias) {
    lw->N = N; lw->K = K;
    if (f32_tmp) JIMM_CUDA_CHECK(cudaMallocAsync(&lw->w, static_cast<size_t>(N) * K * sizeof(float), stream));  // freed by e4m3()
    else JIMM_TRY(m->pool.alloc(&lw->w, static_cast<size_t>(N) * K * cdt_size(m)));
    if (bias) {
      void* b = nullptr;
      JIMM_TRY(m->pool.alloc(&b, static_cast<size_t>(N) * sizeof(float)));
      lw->b = static_cast<float*>(b);
    }
    return 0;
  }
  int upload_bias_at(const std::string& name, std::initializer_list<int64_t> shape, float* dst, size_t count) {
    HostParam* hp = find(name, shape);
    if (!hp) return JIMM_ESTATE;
    if (hp->numel() != count) { set_last_error("finalize: '%s' numel mismatch", name.c_str()); return JIMM_ESTATE; }
    return rows_to_device(hp, 1, count, dst, DT_F32, count);
  }
  // element (k, n) of a kernel's flax (K, N) view, whatever its stored order
  static float kn(const HostParam* hp, size_t k, size_t n, size_t K, size_t N) { return hp->transposed ? hp->at(n * K + k) : hp->at(k * N + n); }
  // nnx.Linear: kernel (K,N), optional bias (N)
  int linear(const std::string& prefix, int K, int N, bool bias, LinearW* lw) {
    JIMM_TRY(alloc_linear(lw, N, K, bias));
    JIMM_TRY(pack_kernel(prefix + ".kernel", {K, N}, K, N, lw->w, 0));
    if (bias) JIMM_TRY(upload_bias_at(prefix + ".bias", {N}, lw->b, N));
    return 0;
  }
  // nnx.MultiHeadAttention projections -> fused operand; names: subset of {"query","key","value"}
  int fused_proj(const std::string& attn_prefix, const std::vector<std::string>& names, int D, int H, LinearW* lw) {
    const int d = D / H;
    const int N = D * static_cast<int>(names.size());
    JIMM_TRY(alloc_linear(lw, N, D, true));
    for (size_t i = 0; i < names.size(); ++i) {
      JIMM_TRY(pack_kernel(attn_prefix + "." + names[i] + ".kernel", {D, H, d}, D, D, lw->w, static_cast<int>(i) * D));
      JIMM_TRY(upload_bias_at(attn_prefix + "." + names[i] + ".bias", {H, d}, lw->b + i * D, D));
    }
    return 0;
  }
  int out_proj(const std::string& attn_prefix, int D, int H, LinearW* lw) {
    const int d = D / H;
    JIMM_TRY(alloc_linear(lw, D, D, true));
    JIMM_TRY(pack_kernel(attn_prefix + ".out.kernel", {H, d, D}, D, D, lw->w, 0));
    JIMM_TRY(upload_bias_at(attn_prefix + ".out.bias", {D}, lw->b, D));
    return 0;
  }
  // MultiHeadAttentionPoolingHead parameters (common/vit.py:27-85) under `mp`
  int map_head(const std::string& mp, int D, int H, VisionTower* v) {
    const int d = D / H;
    JIMM_TRY(fused_proj(mp + "attn", {"key", "value"}, D, H, &v->map_kv));
    JIMM_TRY(out_proj(mp + "attn", D, H, &v->map_out));
    JIMM_TRY(upload_ln(mp + "layernorm", D, &v->map_ln));
    // the MLP width is that of the staged (D, M) fc1 kernel: 4 * D in the reference's towers (common/vit.py:175), the checkpoint's
    // intermediate_size in HF SigLIP (4304 in so400m)
    auto fc1 = m->host.find(mp + "mlp.layers.0.kernel");
    const int M = fc1 != m->host.end() && fc1->second.shape.size() == 2 ? static_cast<int>(fc1->second.shape[1]) : 4 * D;
    if (M <= 0 || M % 8 != 0) {
      set_last_error("MAP head mlp width %d (%smlp.layers.0.kernel): must be a positive multiple of 8", M, mp.c_str());
      return JIMM_EINVAL;
    }
    JIMM_TRY(linear(mp + "mlp.layers.0", D, M, true, &v->map_fc1));
    JIMM_TRY(linear(mp + "mlp.layers.2", M, D, true, &v->map_fc2));
    // probe query is input independent: q = probe . Wq + bq  (common/vit.py:96-97), done once on the host in fp64
    HostParam* probe = find(mp + "probe", {1, 1, D});
    HostParam* wq = find(mp + "attn.query.kernel", {D, H, d});
    HostParam* bq = find(mp + "attn.query.bias", {H, d});
    if (!probe || !wq || !bq) return JIMM_ESTATE;
    std::vector<float> q(D);
    for (int o = 0; o < D; ++o) {
      double acc = bq->at(o);
      for (int i = 0; i < D; ++i) acc += static_cast<double>(probe->at(i)) * kn(wq, i, o, D, D);
      q[o] = static_cast<float>(acc);
    }
    void* dq = nullptr;
    JIMM_TRY(m->pool.alloc(&dq, D * sizeof(float)));
    JIMM_CUDA_CHECK(cudaMemcpy(dq, q.data(), D * sizeof(float), cudaMemcpyHostToDevice));
    v->map_q = static_cast<float*>(dq);
    return 0;
  }
  // FP8 mode: `pack` (which packs one linear layer through alloc_linear / pack_kernel) runs with fp32 weights into a temporary
  // buffer, then each [N, K] row is quantised to e4m3 with its power-of-two scale (quantize_rows_e4m3_run) -- the same bytes from a
  // flax-layout and from a transposed hand-off, since both pack to the same fp32 rows.
  template <typename F>
  int e4m3(LinearW* lw, F&& pack) {
    f32_tmp = true;
    const int rc = pack();
    f32_tmp = false;
    void* f32 = lw->w;
    lw->w = nullptr;
    if (rc) {
      if (f32) cudaFreeAsync(f32, stream);
      return rc;
    }
    void* q = nullptr;
    void* sc = nullptr;
    JIMM_TRY(m->pool.alloc(&q, static_cast<size_t>(lw->N) * lw->K));
    JIMM_TRY(m->pool.alloc(&sc, static_cast<size_t>(lw->N) * sizeof(float)));
    lw->w = q;
    lw->ws = static_cast<float*>(sc);
    JIMM_TRY(quantize_rows_e4m3_run(static_cast<const float*>(f32), lw->K, lw->N, lw->K, q, lw->K, lw->ws, stream));
    JIMM_CUDA_CHECK(cudaFreeAsync(f32, stream));
    return 0;
  }
  int encoder(const std::string& prefix, Encoder* enc) {
    const EncoderCfg& c = enc->c;
    enc->blocks.resize(c.L);
    for (int i = 0; i < c.L; ++i) {
      const std::string f = prefix + "blocks.layers." + std::to_string(i) + ".";
      BlockW& b = enc->blocks[i];
      JIMM_TRY(upload_ln(f + "norm1", c.D, &b.norm1));
      JIMM_TRY(upload_ln(f + "norm2", c.D, &b.norm2));
      auto qkv = [&]() { return fused_proj(f + "attn", {"query", "key", "value"}, c.D, c.H, &b.qkv); };
      JIMM_TRY(m->f8 ? e4m3(&b.qkv, qkv) : qkv());
      JIMM_TRY(out_proj(f + "attn", c.D, c.H, &b.out));
      auto fc1 = [&]() { return linear(f + "mlp.layers.0", c.D, c.M, true, &b.fc1); };
      JIMM_TRY(m->f8 ? e4m3(&b.fc1, fc1) : fc1());
      JIMM_TRY(linear(f + "mlp.layers.3", c.M, c.D, true, &b.fc2));
    }
    return 0;
  }
};

// ------------------------------------------------------------------------------------------
// GEMM dispatch (plan-based wgmma path; optional SIMT bisection path)
// ------------------------------------------------------------------------------------------
static int run_gemm(jimm_model* m, const GemmPlan& p, const void* A, int lda, const LinearW& w, int M, cudaStream_t s, int reverse = 0) {
  if (M <= 0) return 0;
  if (m->simt) return gemm_simt_run(p.dtype, A, lda, w.w, w.K, M, p.N, p.K, p.epi, s);
  if (!m->prof_on) return gemm_plan_run(&p, M, s, reverse);
  if (m->prof_used + 2 > m->prof_ev.size()) {
    for (int i = 0; i < 256; ++i) {
      cudaEvent_t e;
      JIMM_CUDA_CHECK(cudaEventCreate(&e));
      m->prof_ev.push_back(e);
    }
  }
  JIMM_CUDA_CHECK(cudaEventRecord(m->prof_ev[m->prof_used], s));
  JIMM_TRY(gemm_plan_run(&p, M, s, reverse));
  JIMM_CUDA_CHECK(cudaEventRecord(m->prof_ev[m->prof_used + 1], s));
  m->prof_used += 2;
  m->prof_flops += 2.0 * M * static_cast<double>(p.N) * p.K;
  m->prof_launches += 1;
  return 0;
}

static GemmEpilogue epi_plain(const LinearW& w, int act, void* out, int out_type, int ldo, int mode) {
  GemmEpilogue e;
  e.bias = w.b; e.act = act; e.out = out; e.out_type = out_type; e.ldo = ldo; e.mode = mode;
  return e;
}
static GemmEpilogue epi_residual(const LinearW& w, float* x, int ld, int mode) {
  GemmEpilogue e;
  e.bias = w.b; e.residual = x; e.ldr = ld; e.out = x; e.out_type = DT_F32; e.ldo = ld; e.mode = mode;
  return e;
}

static int plan_encoder(jimm_model* m, Encoder* enc, int Tmax, const EncBufs& ws) {
  const EncoderCfg& c = enc->c;
  const int act = c.act == JIMM_QUICK_GELU ? ACT_QUICK_GELU : ACT_GELU_TANH;
  // x + attn(norm1(x)) is followed by norm2, x + mlp(norm2(x)) by the NEXT block's norm1 (common/transformer.py:130-131): the residual
  // GEMMs normalise the rows they complete and write the next GEMM's A operand, so only the first norm1 of a stack is a kernel
  auto with_ln = [&](GemmEpilogue e, const LNW& ln) {
    if (ws.ln_cnt) { e.ln_scale = ln.scale; e.ln_bias = ln.bias; e.ln_out = ws.h; e.ln_out_type = m->cdt; e.ln_ldo = c.D; e.ln_eps = c.eps; e.ln_cnt = ws.ln_cnt; }
    return e;
  };
  // QKV / FC1 read the block LayerNorm's output: e4m3 with row scales in FP8 mode
  const int ln_t = m->f8 ? DT_E4M3 : m->cdt;
  void* ln_h = m->f8 ? ws.h8 : ws.h;
  auto scaled = [&](GemmEpilogue e, const LinearW& w) {
    if (m->f8) { e.a_scale = ws.sa; e.b_scale = w.ws; }
    return e;
  };
  for (size_t bi = 0; bi < enc->blocks.size(); ++bi) {
    BlockW& b = enc->blocks[bi];
    // QKV: h[T,D] x Wqkv[3D,D]^T + b -> qkv (16-bit) [T,3D]
    JIMM_TRY(gemm_plan_init(&b.p_qkv, ln_t, ln_h, c.D, b.qkv.w, c.D, Tmax, 3 * c.D, c.D,
                            scaled(epi_plain(b.qkv, ACT_NONE, ws.big, m->adt, 3 * c.D, m->epi_mode_16), b.qkv)));
    // out-proj: attn[T,D] x Wo[D,D]^T + bo + x -> x
    JIMM_TRY(gemm_plan_init(&b.p_out, m->cdt, ws.h, c.D, b.out.w, c.D, Tmax, c.D, c.D, with_ln(epi_residual(b.out, ws.x, c.D, m->epi_mode_res), b.norm2)));
    // FC1: h x W1^T + b1 -> act -> mid [T,M]
    JIMM_TRY(gemm_plan_init(&b.p_fc1, ln_t, ln_h, c.D, b.fc1.w, c.D, Tmax, c.M, c.D,
                            scaled(epi_plain(b.fc1, act, ws.big, m->cdt, c.M, m->epi_mode_16), b.fc1)));
    // FC2: mid x W2^T + b2 + x -> x
    GemmEpilogue e2 = epi_residual(b.fc2, ws.x, c.D, m->epi_mode_res);
    if (bi + 1 < enc->blocks.size()) e2 = with_ln(e2, enc->blocks[bi + 1].norm1);
    JIMM_TRY(gemm_plan_init(&b.p_fc2, m->cdt, ws.big, c.M, b.fc2.w, c.M, Tmax, c.D, c.M, e2));
  }
  return 0;
}

static int plan_map_head(jimm_model* m, int Bm, int Tv) {
  VisionTower& v = m->vis;
  Workspace& ws = m->ws;
  const int D = v.D, M = v.map_fc1.N;
  JIMM_TRY(gemm_plan_init(&v.p_map_kv, m->cdt, ws.enc.h, D, v.map_kv.w, D, Tv, 2 * D, D, epi_plain(v.map_kv, ACT_NONE, ws.enc.big, m->adt, 2 * D, m->epi_mode_16)));
  JIMM_TRY(gemm_plan_init(&v.p_map_out, m->cdt, ws.pooled, D, v.map_out.w, D, Bm, D, D, epi_plain(v.map_out, ACT_NONE, ws.feat, DT_F32, D, 0)));
  JIMM_TRY(gemm_plan_init(&v.p_map_fc1, m->cdt, ws.pooled, D, v.map_fc1.w, D, Bm, M, D, epi_plain(v.map_fc1, ACT_GELU_TANH, ws.mid2, m->cdt, M, 0)));
  GemmEpilogue e = epi_plain(v.map_fc2, ACT_NONE, ws.out_dev, DT_F32, D, 0);
  e.residual = ws.feat; e.ldr = D;
  JIMM_TRY(gemm_plan_init(&v.p_map_fc2, m->cdt, ws.mid2, M, v.map_fc2.w, M, Bm, D, M, e));
  return 0;
}

// The patch GEMM of up to `images` images of n patches (n_pad when padded to 32 rows) and S tokens, writing the residual stream ws.x.
// Token scatter: it reduce-adds each patch row into its token row, onto the position rows already there.  Otherwise it maps patch rows
// to token rows (leaving the CLS row) and adds `pos` (the trained table) or, when pos is null, the resampled table already in ws.x.
static int plan_patch(jimm_model* m, int n, int n_pad, int S, int images, const float* pos, GemmPlan* p) {
  const VisionTower& v = m->vis;
  float* x = m->ws.enc.x;
  const int off = v.pooling == JIMM_POOL_CLS ? 1 : 0;
  GemmEpilogue e;
  e.bias = v.patch.b; e.out = x; e.out_type = DT_F32; e.ldo = v.D;
  if (v.patch_scatter) {
    e.residual = x; e.ldr = v.D; e.mode = 2; e.tok_pad = n_pad; e.tok_off = off; e.tok_S = S;
  } else {
    if (pos) e.rowadd = pos;
    else { e.residual = x; e.ldr = v.D; }
    e.mode = 0; e.rows_in = n; e.rows_out = S; e.row_off = off;
  }
  JIMM_TRY(gemm_plan_init(p, m->cdt, m->ws.enc.big, v.Kp, v.patch.w, v.Kp, images * (v.patch_scatter ? n_pad : n), v.D, v.Kp, e));
  if (v.patch_scatter && p->epi.mode != 2) { set_last_error("patch GEMM: token-scatter epilogue unavailable"); return JIMM_EINVAL; }
  return 0;
}

// B samples of different lengths packed into T rows: sample b is rows seq_off[b] .. seq_off[b + 1] - 1 (device), max_S the longest
struct PackedRows {
  const int* seq_off;
  int T, max_S;
};

// Where a per-token call (jimm_image_tokens* / jimm_text_tokens*) puts the hidden states of one chunk: request j copies x_layers[j]
// (JIMM_LAYER_FINAL: the final-normed tokens) into out[j] from output row row0 on.  An attention call (jimm_image_attn* /
// jimm_text_attn*) instead writes block ablocks[j]'s weights into aout[j] from element H * sq0 on (JIMM_ATTN_MAP: the MAP head's probe
// weights, from element H * row0 on).  run_encoder runs `blocks` blocks; the pooling tail runs only when the call asked for the pooled
// output too, or for the MAP head's weights.
struct TokenSink {
  int n = 0;
  const int* layers = nullptr;
  void* const* out = nullptr;
  int out_type = DT_F32;
  size_t row0 = 0;             // the chunk's first output row
  int blocks = 0;              // max(requested layer), or every block for JIMM_LAYER_FINAL / a pooled output
  const LNW* ln = nullptr;     // the final norm: ln_post (vision) / ln_final (text)
  float eps = 0.f;
  int an = 0;                  // attention requests
  const int* ablocks = nullptr;
  void* const* aout = nullptr;
  int aout_type = DT_F32;
  bool map = false;            // one of them is JIMM_ATTN_MAP
  size_t sq0 = 0;              // sum of S_b^2 over the samples before the chunk
  TokenSink at(size_t r, size_t sq) const { TokenSink t = *this; t.row0 = r; t.sq0 = sq; return t; }
};

// The requests of `sink` for layer k (JIMM_LAYER_FINAL: the final norm) on the T rows of x
static int sink_rows(const TokenSink& sink, int k, const float* x, int T, int D, cudaStream_t s) {
  for (int j = 0; j < sink.n; ++j) {
    if (sink.layers[j] != k) continue;
    void* dst = static_cast<uint8_t*>(sink.out[j]) + sink.row0 * D * dtype_size(sink.out_type);
    if (k == JIMM_LAYER_FINAL) JIMM_TRY(layernorm_run(x, D, 1, 0, nullptr, sink.ln->scale, sink.ln->bias, sink.eps, dst, sink.out_type, D, T, D, s));
    else JIMM_TRY(tokens_out_run(x, static_cast<size_t>(T), D, dst, sink.out_type, s));
  }
  return 0;
}

// The attention requests of `sink` for block bi, on the qkv that block's attention read
static int sink_attn(const TokenSink& sink, int bi, const void* qkv, int adt, const EncoderCfg& c, int B, int S, const PackedRows* pk, cudaStream_t s) {
  for (int j = 0; j < sink.an; ++j) {
    if (sink.ablocks[j] != bi) continue;
    void* dst = static_cast<uint8_t*>(sink.aout[j]) + sink.sq0 * c.H * dtype_size(sink.aout_type);
    JIMM_TRY(attn_probs_run(qkv, adt, dst, sink.aout_type, pk ? pk->seq_off : nullptr, B, pk ? pk->max_S : S, c.H, c.D / c.H, c.causal, s));
  }
  return 0;
}

// x: fp32 [B*S, D] residual stream in ws.x (pk: the packed rows instead).  TransformerEncoder.__call__ x L (common/transformer.py:116-132,190-196).
// sink: also copy the requested layers out, and run only sink->blocks blocks.
static int run_encoder(jimm_model* m, Encoder* enc, int B, int S, cudaStream_t s, const EncBufs& ws, const PackedRows* pk = nullptr,
                       const TokenSink* sink = nullptr) {
  const EncoderCfg& c = enc->c;
  const int T = pk ? pk->T : B * S;
  const int nblocks = sink ? sink->blocks : static_cast<int>(enc->blocks.size());
  if (sink) JIMM_TRY(sink_rows(*sink, 0, ws.x, T, c.D, s));
  // Boustrophedon schedule: every kernel walks its rows / tiles / items in the direction opposite to its producer, so it
  // starts on the data written last -- the part of the 77-310 MB activation still resident in the 50 MB L2.
  int dir = m->l2_alternate ? 1 : 0;  // the patch GEMM / embedding kernels ran forward -> the first LayerNorm runs backward
  auto flip = [&]() { const int d = dir; if (m->l2_alternate) dir ^= 1; return d; };
  bool h_ready = false;  // ws.h already holds norm1(x) of the coming block (written by the previous block's FC2 epilogue)
  const int ln_t = m->f8 ? DT_E4M3 : m->cdt;  // the block LayerNorms feed QKV / FC1 (see plan_encoder)
  void* ln_h = m->f8 ? ws.h8 : ws.h;
  for (int bi = 0; bi < nblocks; ++bi) {
    BlockW& b = enc->blocks[bi];
    if (!h_ready) JIMM_TRY(layernorm_run(ws.x, c.D, 1, 0, nullptr, b.norm1.scale, b.norm1.bias, c.eps, ln_h, ln_t, c.D, T, c.D, s, flip(), ws.sa));
    JIMM_TRY(run_gemm(m, b.p_qkv, ln_h, c.D, b.qkv, T, s, flip()));
    if (pk) JIMM_TRY(attention_packed_run(ws.big, m->adt, ws.h, m->cdt, pk->seq_off, B, pk->max_S, c.H, c.D / c.H, c.causal, s, flip()));
    else JIMM_TRY(attention_run(ws.big, m->adt, ws.h, m->cdt, B, S, c.H, c.D / c.H, c.causal, s, flip()));
    if (sink) JIMM_TRY(sink_attn(*sink, bi, ws.big, m->adt, c, B, S, pk, s));  // before FC1 overwrites ws.big
    JIMM_TRY(run_gemm(m, b.p_out, ws.h, c.D, b.out, T, s, flip()));  // + residual (+ norm2 -> ws.h when fused)
    if (m->simt || !gemm_fuses_ln(&b.p_out, T))
      JIMM_TRY(layernorm_run(ws.x, c.D, 1, 0, nullptr, b.norm2.scale, b.norm2.bias, c.eps, ln_h, ln_t, c.D, T, c.D, s, flip(), ws.sa));
    JIMM_TRY(run_gemm(m, b.p_fc1, ln_h, c.D, b.fc1, T, s, flip()));
    JIMM_TRY(run_gemm(m, b.p_fc2, ws.big, c.M, b.fc2, T, s, flip()));  // + residual (+ the next block's norm1 -> ws.h when fused)
    h_ready = !m->simt && gemm_fuses_ln(&b.p_fc2, T);
    if (sink) JIMM_TRY(sink_rows(*sink, bi + 1, ws.x, T, c.D, s));
  }
  if (sink) JIMM_TRY(sink_rows(*sink, JIMM_LAYER_FINAL, ws.x, T, c.D, s));
  return 0;
}

// MultiHeadAttentionPoolingHead.__call__ (common/vit.py:87-101) on the tokens in ws.h (compute dtype, [B*S, D], or the packed rows pk);
// out fp32 [B, D].  sink: each JIMM_ATTN_MAP request also receives the probe weights; without out the head stops after its attention.
static int run_map_head(jimm_model* m, int B, int S, float* out, cudaStream_t s, const PackedRows* pk = nullptr, const TokenSink* sink = nullptr) {
  VisionTower& v = m->vis;
  Workspace& ws = m->ws;
  const int D = v.D, T = pk ? pk->T : B * S, H = v.enc.c.H, d = v.enc.c.D / v.enc.c.H;
  JIMM_TRY(run_gemm(m, v.p_map_kv, ws.enc.h, D, v.map_kv, T, s));                                    // k | v  [T, 2D]
  auto attend = [&](void* probs, int probs_type) -> int {                                            // [B, D]
    if (pk) return map_attention_packed_run(v.map_q, ws.enc.big, m->adt, ws.pooled, m->cdt, pk->seq_off, B, pk->max_S, H, d, s, probs, probs_type);
    return map_attention_run(v.map_q, ws.enc.big, m->adt, ws.pooled, m->cdt, B, S, H, d, s, probs, probs_type);
  };
  bool probed = false;
  for (int j = 0; sink && j < sink->an; ++j) {
    if (sink->ablocks[j] != JIMM_ATTN_MAP) continue;
    JIMM_TRY(attend(static_cast<uint8_t*>(sink->aout[j]) + sink->row0 * H * dtype_size(sink->aout_type), sink->aout_type));
    probed = true;
  }
  if (!probed) JIMM_TRY(attend(nullptr, DT_F32));
  if (!out) return 0;
  JIMM_TRY(run_gemm(m, v.p_map_out, ws.pooled, D, v.map_out, B, s));                                 // -> feat fp32 [B, D]
  JIMM_TRY(layernorm_run(ws.feat, D, 1, 0, nullptr, v.map_ln.scale, v.map_ln.bias, v.eps_outer, ws.pooled, m->cdt, D, B, D, s));
  JIMM_TRY(run_gemm(m, v.p_map_fc1, ws.pooled, D, v.map_fc1, B, s));                                 // gelu -> mid2 [B, M]
  GemmPlan p = v.p_map_fc2;  // + bias + residual(feat) -> out fp32 [B, D]
  p.epi.out = out;
  return run_gemm(m, p, ws.mid2, v.map_fc1.N, v.map_fc2, B, s);
}

// ln_post + the pooling head of B samples of S tokens (pk: the packed rows instead) in ws.x.  CLS: ln_post is per-row and only row 0 of
// each sample is consumed (common/vit.py:244-246): every S-th row, or the packed offsets as row index (group 0).  MAP: ln_post of every
// row, then the MAP head (common/vit.py:87-101).  out: fp32 [B, out_dim]
static int run_pool(jimm_model* m, int B, int S, float* out, cudaStream_t s, const PackedRows* pk = nullptr, const TokenSink* sink = nullptr) {
  VisionTower& v = m->vis;
  Workspace& ws = m->ws;
  const int D = v.D;
  if (v.pooling == JIMM_POOL_MAP) {
    JIMM_TRY(layernorm_run(ws.enc.x, D, 1, 0, nullptr, v.ln_post.scale, v.ln_post.bias, v.eps_outer, ws.enc.h, m->cdt, D, pk ? pk->T : B * S, D, s));
    return run_map_head(m, B, S, out, s, pk, sink);
  }
  const int group = pk ? 0 : S;
  const int* row_index = pk ? pk->seq_off : nullptr;
  if (v.head.N == 0) return layernorm_run(ws.enc.x, D, group, 0, row_index, v.ln_post.scale, v.ln_post.bias, v.eps_outer, out, DT_F32, D, B, D, s);
  JIMM_TRY(layernorm_run(ws.enc.x, D, group, 0, row_index, v.ln_post.scale, v.ln_post.bias, v.eps_outer, ws.pooled, m->cdt, D, B, D, s));
  GemmPlan p = v.p_head;
  p.epi.out = out;
  return run_gemm(m, p, ws.pooled, D, v.head, B, s);
}

// The vision tower after the patch embedding, on B samples of S tokens (pk: the packed rows instead) in ws.x: ln_pre, the encoder and,
// unless a token or attention call (sink) asked for no pooled output and no MAP weights, the pooling head into out.
static int vision_tail(jimm_model* m, int B, int S, float* out, cudaStream_t s, const PackedRows* pk, const TokenSink* sink) {
  VisionTower& v = m->vis;
  float* x = m->ws.enc.x;
  if (v.pre_norm)
    JIMM_TRY(layernorm_run(x, v.D, 1, 0, nullptr, v.ln_pre.scale, v.ln_pre.bias, v.eps_outer, x, DT_F32, v.D, pk ? pk->T : B * S, v.D, s));
  JIMM_TRY(run_encoder(m, &v.enc, B, S, s, m->ws.enc, pk, sink));
  if (sink && !out && !sink->map) return 0;
  return run_pool(m, B, S, out, s, pk, sink);
}

// VisionTransformerBase.__call__ (common/vit.py:216-248) + the model's head.  img: [B, H, W, C]; grid: null for the trained patch
// grid, else the grid of H x W (position table resampled).  out: fp32 [B, out_dim]
static int run_vision(jimm_model* m, const void* img, int in_dtype, int B, int H, int W, const PatchGrid* grid, float* out, cudaStream_t s,
                      const TokenSink* sink = nullptr) {
  VisionTower& v = m->vis;
  float* x = m->ws.enc.x;
  void* big = m->ws.enc.big;
  const int D = v.D, S = grid ? grid->S : v.S, n = v.n;
  const float* cls = v.pooling == JIMM_POOL_CLS ? v.cls : nullptr;
  // patch embed + pos (+cls)
  if (grid) {
    // resampled pos (+cls) first; the patch GEMM adds onto it (token scatter, or a residual-reading epilogue with row remap)
    JIMM_TRY(tokens_init_interp_run(x, cls, v.pos, v.img / v.P, D, B, grid->gh, grid->gw, v.interp, s));
    const int rows = v.patch_scatter ? grid->n_pad : grid->n;
    JIMM_TRY(patchify_run(img, in_dtype, B, H, W, v.C, v.P, big, m->cdt, s, v.patch_scatter ? grid->n_pad : 0, v.Kp));
    JIMM_TRY(run_gemm(m, grid->patch, big, v.patch.K, v.patch, B * rows, s));
  } else if (v.patch_scatter) {
    JIMM_TRY(tokens_init_run(x, cls, v.pos, B, S, D, s));
    JIMM_TRY(patchify_run(img, in_dtype, B, H, W, v.C, v.P, big, m->cdt, s, v.n_pad, v.Kp));
    JIMM_TRY(run_gemm(m, v.p_patch, big, v.patch.K, v.patch, B * v.n_pad, s));
  } else {
    JIMM_TRY(patchify_run(img, in_dtype, B, H, W, v.C, v.P, big, m->cdt, s, 0, v.Kp));
    JIMM_TRY(run_gemm(m, v.p_patch, big, v.patch.K, v.patch, B * n, s));
    if (cls) JIMM_TRY(cls_row_run(x, v.cls, v.pos, B, S, D, s));
  }
  return vision_tail(m, B, S, out, s, nullptr, sink);
}

// The pixels of a vision call, in one of three forms:
//   IMG_DENSE: img [B, H, W, C], every image H x W (native: the trained size, which image_call fills in);
//   IMG_LIST:  B NHWC images imgs[b] of Hs[b] x Ws[b];
//   IMG_ROWS:  the HuggingFace NaFlex patch rows of B samples, img = patches [B, N, P*P*C], of which sample b's first gh * gw rows are
//              its patches, (gh, gw) = (grid[2b], grid[2b + 1]); image_call points Hs, Ws at the sizes the grids cut.
enum ImageForm { IMG_DENSE, IMG_LIST, IMG_ROWS };
struct ImageSrc {
  ImageForm form = IMG_DENSE;
  const void* img = nullptr;
  const void* const* imgs = nullptr;
  int H = 0, W = 0;
  bool native = false;
  const int* Hs = nullptr;
  const int* Ws = nullptr;
  const int* grid = nullptr;
  int N = 0;
  size_t sample_bytes = 0;  // IMG_DENSE / IMG_ROWS: bytes of one sample (image_call fills it in)
  static ImageSrc dense(const void* img, int H, int W) { ImageSrc s; s.img = img; s.H = H; s.W = W; return s; }
  static ImageSrc trained(const void* img) { ImageSrc s; s.img = img; s.native = true; return s; }
  static ImageSrc list(const void* const* imgs, const int* H, const int* W) { ImageSrc s; s.form = IMG_LIST; s.imgs = imgs; s.Hs = H; s.Ws = W; return s; }
  static ImageSrc rows(const void* patches, int N, const int* grid) { ImageSrc s; s.form = IMG_ROWS; s.img = patches; s.N = N; s.grid = grid; return s; }
  ImageSrc from(int b0) const {  // the samples from b0 on
    ImageSrc p = *this;
    if (imgs) p.imgs += b0;
    else p.img = static_cast<const uint8_t*>(img) + b0 * sample_bytes;
    if (Hs) { p.Hs += b0; p.Ws += b0; }
    if (grid) p.grid += 2 * b0;
    return p;
  }
};

// Uploads the offsets tok[0 .. B] of a packed chunk and one int per sequence, col(b), to meta [2B + 1].  The copy is stream-ordered from
// pageable memory, which is staged before the call returns: an earlier call or chunk on this stream has read its own offsets before this
// copy lands.
template <typename F>
static int upload_offsets(int* meta, const int* tok, int B, F&& col, cudaStream_t s) {
  std::vector<int> h(2 * static_cast<size_t>(B) + 1);
  for (int b = 0; b <= B; ++b) h[b] = tok[b];
  for (int b = 0; b < B; ++b) h[B + 1 + b] = col(b);
  JIMM_CUDA_CHECK(cudaMemcpyAsync(meta, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  return 0;
}

// run_vision on B images of different sizes (src: IMG_LIST or IMG_ROWS) packed into one token stream: image b is token rows tok[b] ..
// tok[b + 1] - 1 (host offsets, tok[0] = 0), max_S the most tokens of one image.  Every kernel works row by row or, given the offsets,
// image by image, so row b of out is the bits run_vision gives on image b alone.
static int run_vision_packed(jimm_model* m, const ImageSrc& src, int in_dtype, int B, const int* tok, int max_S, float* out, cudaStream_t s,
                             const TokenSink* sink) {
  VisionTower& v = m->vis;
  Workspace& ws = m->ws;
  const int T = tok[B], off = v.pooling == JIMM_POOL_CLS ? 1 : 0;
  JIMM_TRY(upload_offsets(ws.pk_meta, tok, B, [&](int b) { return src.Ws[b] / v.P; }, s));
  const PackedRows pk{ws.pk_meta, T, max_S};
  const size_t row_bytes = static_cast<size_t>(v.Kp) * cdt_size(m);
  if (src.form == IMG_ROWS) {  // NaFlex patch rows: no CLS token, so patch rows are token rows
    JIMM_TRY(patch_rows_packed_run(src.img, in_dtype, src.N, v.P * v.P * v.C, pk.seq_off, B, max_S, ws.enc.big, m->cdt, v.Kp, s));
  } else {
    for (int b = 0; b < B; ++b)
      JIMM_TRY(patchify_run(src.imgs[b], in_dtype, 1, src.Hs[b], src.Ws[b], v.C, v.P, static_cast<uint8_t*>(ws.enc.big) + (tok[b] + off) * row_bytes,
                            m->cdt, s, 0, v.Kp));
  }
  JIMM_TRY(run_gemm(m, v.p_patch_packed, ws.enc.big, v.Kp, v.patch, T, s));
  JIMM_TRY(tokens_add_interp_packed_run(ws.enc.x, off ? v.cls : nullptr, v.pos, v.img / v.P, v.D, pk.seq_off, ws.pk_meta + B + 1, B, max_S,
                                        v.interp, s));
  return vision_tail(m, B, 0, out, s, &pk, sink);
}

// CLIP.encode_text (models/clip.py:148-167) / SigLIP.encode_text (models/siglip.py:135-153).  out fp32 [B, Dt]
static int run_text(jimm_model* m, const int32_t* ids, int B, int T, float* out, cudaStream_t s, const TokenSink* sink = nullptr) {
  TextTower& t = m->txt;
  TextWs& ws = m->wt;
  JIMM_TRY(embed_run(ids, t.table, t.pos, ws.enc.x, B, T, t.D, t.V, s));
  JIMM_TRY(run_encoder(m, &t.enc, B, T, s, ws.enc, nullptr, sink));
  if (sink && !out) return 0;
  if (t.pool == JIMM_TPOOL_EOT_ARGMAX) {
    JIMM_TRY(argmax_ids_run(ids, ws.idx, B, T, s));
    JIMM_TRY(layernorm_run(ws.enc.x, t.D, T, 0, ws.idx, t.ln_final.scale, t.ln_final.bias, t.eps_outer, ws.pooled, m->cdt, t.D, B, t.D, s));
  } else {
    JIMM_TRY(layernorm_run(ws.enc.x, t.D, T, T - 1, nullptr, t.ln_final.scale, t.ln_final.bias, t.eps_outer, ws.pooled, m->cdt, t.D, B, t.D, s));
  }
  GemmPlan p = t.p_head;
  p.epi.out = out;
  JIMM_TRY(run_gemm(m, p, ws.pooled, t.D, t.head, B, s));
  return 0;
}

// run_text on B token sequences of different lengths packed into one stream: sequence b is rows tok[b] .. tok[b + 1] - 1 of ids (host
// offsets, tok[0] = 0), max_S the longest.  Positions restart at 0 in every sequence and the causal mask (CLIP) is taken within it; every
// other kernel works row by row, so row b of out is the bits run_text gives on sequence b alone.
static int run_text_packed(jimm_model* m, const int32_t* ids, int B, const int* tok, int max_S, float* out, cudaStream_t s,
                           const TokenSink* sink) {
  TextTower& t = m->txt;
  TextWs& ws = m->wt;
  // The pooled rows follow the offsets: each sequence's last row (SigLIP's last-token pooling); CLIP's EOT rows overwrite them on the device.
  JIMM_TRY(upload_offsets(ws.pk_meta, tok, B, [&](int b) { return tok[b + 1] - 1; }, s));
  const PackedRows pk{ws.pk_meta, tok[B], max_S};
  int* rows = ws.pk_meta + B + 1;
  JIMM_TRY(embed_packed_run(ids, t.table, t.pos, ws.enc.x, pk.seq_off, B, pk.T, t.D, t.V, s));
  JIMM_TRY(run_encoder(m, &t.enc, B, 0, s, ws.enc, &pk, sink));
  if (sink && !out) return 0;
  if (t.pool == JIMM_TPOOL_EOT_ARGMAX) JIMM_TRY(argmax_ids_packed_run(ids, pk.seq_off, rows, B, s));
  // ln_final of the pooled rows only (group 0: the rows by index), into ws.enc.h -- free once the encoder has run -- for the head GEMM
  JIMM_TRY(layernorm_run(ws.enc.x, t.D, 0, 0, rows, t.ln_final.scale, t.ln_final.bias, t.eps_outer, ws.enc.h, m->cdt, t.D, B, t.D, s));
  GemmPlan p = t.p_head_packed;
  p.epi.out = out;
  return run_gemm(m, p, ws.enc.h, t.D, t.head, B, s);
}

static int check_ready(const jimm_model* m, int B) {
  if (!m) { set_last_error("null model"); return JIMM_EINVAL; }
  if (!m->finalized) { set_last_error("model not finalized"); return JIMM_ESTATE; }
  if (B < 0) { set_last_error("negative batch"); return JIMM_EINVAL; }
  return 0;
}
static int set_device(const jimm_model* m) {
  JIMM_CUDA_CHECK(cudaSetDevice(m->device));
  return 0;
}

// argument checks shared by the entry points
static int check_image_dtype(int in_dtype) {
  if (in_dtype < JIMM_F32 || in_dtype > JIMM_BF16) { set_last_error("bad image dtype %d", in_dtype); return JIMM_EINVAL; }
  return 0;
}
// a vision tower and, for a jimm_vit_forward* call (vit_fn names it), a ViT-only model
static int check_vision(const jimm_model* m, const char* vit_fn) {
  if (!m->vis.present) { set_last_error("model has no vision tower"); return JIMM_EINVAL; }
  if (vit_fn && m->cfg.kind != JIMM_VIT && m->cfg.kind != JIMM_TOWER) {
    set_last_error("%s on a dual-tower model; use the jimm_encode_image* / jimm_dual_* calls", vit_fn);
    return JIMM_EINVAL;
  }
  return 0;
}
static int check_text(const jimm_model* m) {
  if (!m->txt.present) { set_last_error("model has no text tower"); return JIMM_EINVAL; }
  return 0;
}
static int check_text_len(const jimm_model* m, int T) {
  if (T <= 0 || T > m->txt.T) { set_last_error("sequence length %d outside (0, context_length=%d]", T, m->txt.T); return JIMM_EINVAL; }
  return 0;
}
static int check_patch(const jimm_model* m, int H, int W) {
  if (H < m->vis.P || W < m->vis.P) { set_last_error("image %dx%d is smaller than one %dx%d patch", H, W, m->vis.P, m->vis.P); return JIMM_EINVAL; }
  return 0;
}

// every length of a packed text call in 1 .. context_length
static int check_lens(const jimm_model* m, int B, const int* len) {
  for (int b = 0; b < B; ++b) {
    if (len[b] <= 0 || len[b] > m->txt.T) {
      set_last_error("sequence %d: length %d outside (0, context_length=%d]", b, len[b], m->txt.T);
      return JIMM_EINVAL;
    }
  }
  return 0;
}

// fn(b0, nb) on consecutive chunks [b0, b0 + nb) of B items, at most `chunk` each
template <typename F>
static int for_chunks(int B, int chunk, F&& fn) {
  for (int b0 = 0; b0 < B; b0 += chunk) JIMM_TRY(fn(b0, std::min(chunk, B - b0)));
  return 0;
}

static int vision_out_dim(const jimm_model* m) { return m->vis.head.N > 0 ? m->vis.head.N : m->vis.D; }

// ------------------------------------------------------------------------------------------
// CUDA-graph replay for small batches
// ------------------------------------------------------------------------------------------
static void graphs_release(jimm_model* m) {
  for (auto& kv : m->graphs)
    if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  m->graphs.clear();
}

// Runs `body` (which enqueues a tower on `s`, reading and writing fixed workspace buffers only) eagerly the first time a key is
// seen, captures it into a graph the second time, and replays the graph afterwards.  Any capture problem disables graphs for
// the model and falls back to the eager launches -- the same kernels either way.
template <typename F>
static int run_graphed(jimm_model* m, std::tuple<int, int, int> key, cudaStream_t s, F&& body) {
  if (m->graph_max_batch <= 0 || m->prof_on || m->simt) return body(s);
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone) {  // the caller is capturing already
    cudaGetLastError();
    return body(s);
  }
  jimm_model::GraphEntry& e = m->graphs[key];
  if (e.exec) {
    JIMM_CUDA_CHECK(cudaGraphLaunch(e.exec, s));
    g_launches.fetch_add(e.launches, std::memory_order_relaxed);
    g_graph_replays.fetch_add(1, std::memory_order_relaxed);
    return 0;
  }
  if (e.seen++ == 0) return body(s);
  // another thread is in finalize / destroy (see g_capture_mu): run eagerly now, capture on a later call
  std::unique_lock<std::mutex> capture_lock(g_capture_mu, std::try_to_lock);
  if (!capture_lock.owns_lock()) return body(s);
  // Capture on a private stream: the caller's stream may be the legacy default stream, which cannot be captured; nothing
  // executes during capture, and the instantiated graph is launched on the caller's stream.
  if (!m->capture_stream && cudaStreamCreateWithFlags(&m->capture_stream, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    m->graph_max_batch = 0;
    return body(s);
  }
  const long long l0 = t_launches;
  if (cudaStreamBeginCapture(m->capture_stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    cudaGetLastError();
    m->graph_max_batch = 0;
    return body(s);
  }
  const int rc = body(m->capture_stream);
  cudaGraph_t g = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(m->capture_stream, &g);
  const long long captured = t_launches - l0;  // this thread's launches only: other threads' eager launches did run
  g_launches.fetch_sub(captured, std::memory_order_relaxed);  // captured launches have not run
  cudaGraphExec_t exec = nullptr;
  if (rc == 0 && ce == cudaSuccess && g && cudaGraphInstantiate(&exec, g, 0) == cudaSuccess) {
    cudaGraphDestroy(g);
    e.exec = exec;
    e.launches = captured;
    JIMM_CUDA_CHECK(cudaGraphLaunch(e.exec, s));
    g_launches.fetch_add(e.launches, std::memory_order_relaxed);
    g_graph_replays.fetch_add(1, std::memory_order_relaxed);
    return 0;
  }
  if (g) cudaGraphDestroy(g);
  cudaGetLastError();
  m->graph_max_batch = 0;
  if (rc != 0) return rc;
  return body(s);
}

// Vision tower of one chunk.  Small chunks go through the graph: input staged into ws.in_img, result from m->graph_out.
static int exec_vision(jimm_model* m, const void* img, int in_dtype, int n, float* out, cudaStream_t s) {
  const int px = m->vis.img;
  if (n <= 0 || n > m->graph_max_batch || !m->graph_out) return run_vision(m, img, in_dtype, n, px, px, nullptr, out, s);
  const size_t bytes = static_cast<size_t>(n) * m->vis.img * m->vis.img * m->vis.C * dtype_size(in_dtype);
  if (img != m->ws.in_img) {
    m->host_chain = false;  // the staging buffer is written outside the host path's slot protocol
    JIMM_CUDA_CHECK(cudaMemcpyAsync(m->ws.in_img, img, bytes, cudaMemcpyDeviceToDevice, s));
  }
  JIMM_TRY(run_graphed(m, std::make_tuple(0, n, in_dtype), s, [&](cudaStream_t cs) { return run_vision(m, m->ws.in_img, in_dtype, n, px, px, nullptr, m->graph_out, cs); }));
  JIMM_CUDA_CHECK(cudaMemcpyAsync(out, m->graph_out, static_cast<size_t>(n) * vision_out_dim(m) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}

static int exec_text(jimm_model* m, const int32_t* ids, int n, int T, float* out, cudaStream_t s) {
  if (n <= 0 || n > m->graph_max_batch || !m->graph_out_t) return run_text(m, ids, n, T, out, s);
  if (ids != m->ws.in_ids) JIMM_CUDA_CHECK(cudaMemcpyAsync(m->ws.in_ids, ids, static_cast<size_t>(n) * T * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  JIMM_TRY(run_graphed(m, std::make_tuple(1, n, T), s, [&](cudaStream_t cs) { return run_text(m, m->ws.in_ids, n, T, m->graph_out_t, cs); }));
  JIMM_CUDA_CHECK(cudaMemcpyAsync(out, m->graph_out_t, static_cast<size_t>(n) * m->txt.D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}

// JIMM_EINVAL when samples of S tokens are more than the MAP head's attention pools on the handle's device (map_attention_max_seq): it
// keeps one score per token in shared memory, so no token budget lifts this limit.  `what` names the sample in the message.
static int map_seq_fits(const jimm_model* m, size_t S, const char* what) {
  int max_S = 0;
  JIMM_TRY(map_attention_max_seq(m->device, &max_S));
  if (S <= static_cast<size_t>(max_S)) return 0;
  set_last_error("%s: %zu tokens, more than the MAP head's attention pools on device %d (at most %d tokens per sample: one score per "
                 "token in shared memory)", what, S, m->device, max_S);
  return JIMM_EINVAL;
}

// After packing: every parameter that was set must have been used (`what` names the handle in the message).  Drops the host copies.
static int check_all_used(jimm_model* m, const char* what) {
  for (auto& kv : m->host) {
    if (!kv.second.used) {
      set_last_error("finalize: unexpected parameter '%s' was set but is not part of this %s", kv.first.c_str(), what);
      return JIMM_ESTATE;
    }
  }
  m->host.clear();
  return 0;
}

// The vision workspace, or a bare sub-module's: the encoder stack over Tv rows with `big` bytes of ws.big, the pooled rows and MAP head
// buffers of Bm samples, and the result staging of out_elems floats.
static int alloc_workspace(jimm_model* m, size_t Bm, size_t Tv, size_t big, size_t out_elems) {
  Workspace& ws = m->ws;
  const size_t D = m->vis.D, cs = cdt_size(m);
  JIMM_TRY(alloc_stack(m, Tv, D, big, &ws.enc));
  JIMM_TRY(m->pool.alloc(&ws.pooled, Bm * D * cs));
  JIMM_TRY(m->pool.alloc(&ws.feat, Bm * D * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&ws.mid2, Bm * m->vis.map_fc1.N * cs));
  ws.out_dev_elems = out_elems;
  JIMM_TRY(m->pool.alloc(&ws.out_dev, out_elems * sizeof(float)));
  m->ws_rows = Tv;
  m->ws_big = big;
  return 0;
}

// Handle of a bare sub-module (kind JIMM_ENCODER: Transformer, parameters "blocks.layers.{i}.*", common/transformer.py:135-196;
// kind JIMM_MAPHEAD: MultiHeadAttentionPoolingHead, parameters "probe", "attn.*", "layernorm.*", "mlp.layers.{0,2}.*",
// common/vit.py:12-101).  cfg: v_width / v_heads / v_mlp / v_layers / v_act / v_eps_block (block LN) / v_eps_outer (MAP LN) / t_causal,
// ctx_len = max tokens per sample.  The same kernels and orchestration as inside a tower (run_encoder / run_map_head).
static int finalize_sub(jimm_model* m, int max_batch) {
  const jimm_config_t& c = m->cfg;
  if (c.kind == JIMM_MAPHEAD) JIMM_TRY(map_seq_fits(m, static_cast<size_t>(c.ctx_len), "MAP head ctx_len"));
  VisionTower& v = m->vis;
  v.present = false;
  v.D = c.v_width; v.S = c.ctx_len; v.n = v.S; v.pooling = JIMM_POOL_MAP; v.eps_outer = c.v_eps_outer;
  v.enc.c.D = c.v_width; v.enc.c.H = c.v_heads; v.enc.c.M = c.v_mlp; v.enc.c.L = c.kind == JIMM_ENCODER ? c.v_layers : 0;
  v.enc.c.act = c.v_act; v.enc.c.causal = c.t_causal; v.enc.c.eps = c.v_eps_block;
  Packer pk{m};
  const int rc = c.kind == JIMM_ENCODER ? pk.encoder("", &v.enc) : pk.map_head("", v.D, c.v_heads, &v);
  pk.done();
  JIMM_TRY(rc);
  JIMM_TRY(check_all_used(m, "module"));
  const size_t Bm = max_batch, Tv = Bm * v.S;
  JIMM_TRY(alloc_workspace(m, Bm, Tv, big_bytes(m, Tv, 0), Bm * v.D));
  if (c.kind == JIMM_ENCODER) JIMM_TRY(plan_encoder(m, &v.enc, static_cast<int>(Tv), m->ws.enc));
  else JIMM_TRY(plan_map_head(m, static_cast<int>(Bm), static_cast<int>(Tv)));
  JIMM_CUDA_CHECK(cudaDeviceSynchronize());
  m->graph_max_batch = 0;
  m->max_batch = max_batch;
  m->finalized = true;
  return 0;
}

// Uploads and packs every parameter of a ViT / tower / CLIP / SigLIP handle whose towers finalize has configured.  The caller runs
// pk.done() whatever the result.
static int pack_model(jimm_model* m, Packer& pk) {
  const jimm_config_t& c = m->cfg;
  const bool dual = dual_kind(c.kind);
  const std::string vp = c.kind == JIMM_VIT ? "encoder." : (dual ? "vision_model." : "");
  VisionTower& v = m->vis;
  const int D = v.D, PPC0 = c.patch * c.patch * c.in_ch;
  JIMM_TRY(pk.alloc_linear(&v.patch, D, v.Kp, c.patch_bias != 0));
  if (v.Kp != PPC0) JIMM_CUDA_CHECK(cudaMemsetAsync(v.patch.w, 0, static_cast<size_t>(D) * v.Kp * cdt_size(m), pk.stream));
  JIMM_TRY(pk.pack_kernel(vp + "patch_embeddings.kernel", {c.patch, c.patch, c.in_ch, D}, PPC0, D, v.patch.w, 0, v.Kp));
  if (c.patch_bias) JIMM_TRY(pk.upload_bias_at(vp + "patch_embeddings.bias", {D}, v.patch.b, D));
  if (v.pooling == JIMM_POOL_CLS) JIMM_TRY(pk.upload_f32(vp + "cls_token", {1, 1, D}, &v.cls));
  JIMM_TRY(pk.upload_f32(vp + "position_embeddings", {1, v.S, D}, &v.pos));
  if (c.pre_norm) JIMM_TRY(pk.upload_ln(vp + "ln_pre", D, &v.ln_pre));
  JIMM_TRY(pk.upload_ln(vp + "ln_post", D, &v.ln_post));
  JIMM_TRY(pk.encoder(vp + "transformer.", &v.enc));
  if (v.pooling == JIMM_POOL_MAP) JIMM_TRY(pk.map_head(vp + "MAPHead.", D, c.v_heads, &v));
  if (c.kind == JIMM_VIT && c.num_classes > 0) JIMM_TRY(pk.linear("classifier", D, c.num_classes, true, &v.head));
  else if (c.kind == JIMM_CLIP) JIMM_TRY(pk.linear("visual_projection", D, c.t_width, false, &v.head));
  if (!dual) return 0;
  TextTower& t = m->txt;
  JIMM_TRY(pk.upload_f32("token_embedding.embedding", {t.V, t.D}, &t.table));
  JIMM_TRY(pk.upload_f32("positional_embedding", {t.T, t.D}, &t.pos));
  JIMM_TRY(pk.upload_ln("ln_final", t.D, &t.ln_final));
  JIMM_TRY(pk.encoder("text_model.", &t.enc));
  JIMM_TRY(pk.linear("text_projection", t.D, t.D, c.t_head_bias != 0, &t.head));
  JIMM_TRY(pk.upload_f32("logit_scale", {}, &m->logit_scale));
  if (c.kind != JIMM_CLIP) JIMM_TRY(pk.upload_f32("logit_bias", {}, &m->logit_bias));
  return 0;
}

}  // namespace jimm

// ==========================================================================================
// C ABI
// ==========================================================================================
extern "C" {

const char* jimm_last_error(void) { return g_err; }
int jimm_abi_version(void) { return 1; }
long long jimm_launch_count(void) { return g_launches.load(); }
long long jimm_graph_replay_count(void) { return g_graph_replays.load(); }

// The attention kernels take head widths (width / heads) that are multiples of 8 from 8 to 128.
static int check_heads(const char* tower, int width, int heads) {
  const int hd = heads > 0 ? width / heads : 0;
  if (heads <= 0 || width % heads != 0 || hd % 8 != 0 || hd < 8 || hd > 128) {
    set_last_error("%shead_dim: width %d / heads %d = %s%d; supported head widths are multiples of 8 from 8 to 128 (width divisible by heads)", tower,
                   width, heads, heads > 0 && width % heads == 0 ? "" : "non-integer ", hd);
    return JIMM_EINVAL;
  }
  return 0;
}

int jimm_model_create(const jimm_config_t* cfg, int device, jimm_model_t** out) {
  if (!cfg || !out) { set_last_error("jimm_model_create: null argument"); return JIMM_EINVAL; }
  if (cfg->kind < JIMM_VIT || cfg->kind > JIMM_SIGLIP_NAFLEX) { set_last_error("bad kind %d", cfg->kind); return JIMM_EINVAL; }
  const bool sub = cfg->kind == JIMM_ENCODER || cfg->kind == JIMM_MAPHEAD;  // a bare Transformer / MultiHeadAttentionPoolingHead
  if (cfg->pooling != JIMM_POOL_CLS && cfg->pooling != JIMM_POOL_MAP) {
    set_last_error("pooling_type must be either MAP or CLS.");  // common/vit.py:178
    return JIMM_EINVAL;
  }
  const bool dual = dual_kind(cfg->kind);
  if (check_heads(sub ? "" : "vision ", cfg->v_width, cfg->v_heads) || (dual && check_heads("text ", cfg->t_width, cfg->t_heads))) return JIMM_EINVAL;
  const int cd = cfg->compute_dtype;
  if (cd != JIMM_F32 && cd != JIMM_F16 && cd != JIMM_BF16 && cd != JIMM_F8E4M3) { set_last_error("bad compute_dtype %d", cd); return JIMM_EINVAL; }
  // FP8: an e4m3 [T, width] operand's rows are width bytes, and TMA rows are multiples of 16 bytes
  if (cd == JIMM_F8E4M3 && (cfg->v_width % 16 != 0 || (dual && cfg->t_width % 16 != 0))) {
    const bool vis = cfg->v_width % 16 != 0;
    set_last_error("float8_e4m3fn compute: %s width %d must be a multiple of 16 (the e4m3 QKV / FC1 operand rows are width bytes)",
                   vis ? (sub ? "model" : "vision") : "text", vis ? cfg->v_width : cfg->t_width);
    return JIMM_EINVAL;
  }
  if (sub && cfg->ctx_len <= 0) { set_last_error("sub-module handle: ctx_len (max tokens per sample) must be positive"); return JIMM_EINVAL; }
  if (!sub && (cfg->patch <= 0 || cfg->img_size < cfg->patch || cfg->in_ch <= 0)) {
    set_last_error("unsupported patch/img/channels (%d/%d/%d)", cfg->patch, cfg->img_size, cfg->in_ch);
    return JIMM_EINVAL;
  }
  // SigLIP 2 NaFlex is SigLIP's tower (MAP head, no pre-norm, patch bias) on a g x g position table, img_size = g * patch
  if (cfg->kind == JIMM_SIGLIP_NAFLEX && (cfg->pooling != JIMM_POOL_MAP || cfg->pre_norm != 0 || cfg->patch_bias != 1 || cfg->img_size % cfg->patch != 0)) {
    set_last_error("SigLIP 2 NaFlex: needs MAP pooling, pre_norm 0, patch_bias 1 and img_size a multiple of patch (got pooling %d, pre_norm %d, "
                   "patch_bias %d, img_size %d, patch %d)", cfg->pooling, cfg->pre_norm, cfg->patch_bias, cfg->img_size, cfg->patch);
    return JIMM_EINVAL;
  }
  // limits of the kernels, reported at construction (not on the first forward): widths are TMA rows (16-byte multiples), LayerNorm keeps
  // a row in registers
  if (cfg->v_width % 8 != 0 || cfg->v_mlp % 8 != 0 || cfg->v_width > 2048) {
    set_last_error("vision width %d / mlp %d: must be multiples of 8 and width <= 2048", cfg->v_width, cfg->v_mlp);
    return JIMM_EINVAL;
  }
  if (dual && (cfg->t_width % 8 != 0 || cfg->t_mlp % 8 != 0 || cfg->t_width > 2048)) {
    set_last_error("text width %d / mlp %d: must be multiples of 8 and width <= 2048", cfg->t_width, cfg->t_mlp);
    return JIMM_EINVAL;
  }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_last_error("no CUDA device available (%s): jimm_b200 has no CPU fallback", cudaGetErrorString(e));
    return JIMM_ECUDA;
  }
  if (device < 0 || device >= ndev) { set_last_error("bad device %d (have %d)", device, ndev); return JIMM_EINVAL; }
  cudaDeviceProp prop;
  JIMM_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_last_error("device %d is sm_%d%d; jimm_b200 kernels are sm_90a (H100) only", device, prop.major, prop.minor);
    return JIMM_ECUDA;
  }
  jimm_model* m = new jimm_model();
  m->cfg = *cfg;
  m->device = device;
  m->f8 = cfg->compute_dtype == JIMM_F8E4M3;
  // fp32 mode: operands rounded to tf32 when produced; FP8 mode: fp16 outside QKV / FC1
  m->cdt = cfg->compute_dtype == JIMM_F32 ? DT_TF32 : m->f8 ? DT_F16 : cfg->compute_dtype;
  m->adt = cfg->compute_dtype == JIMM_BF16 ? DT_BF16 : DT_F16;
  const char* env = getenv("JIMM_GEMM_IMPL");
  m->simt = env && strcmp(env, "simt") == 0;
  if ((env = getenv("JIMM_L2_ALTERNATE"))) m->l2_alternate = atoi(env) != 0;
  if ((env = getenv("JIMM_GRAPH_MAX_BATCH"))) m->graph_max_batch = atoi(env) > 0 ? atoi(env) : 0;
  if ((env = getenv("JIMM_DUAL_STREAMS"))) m->dual_streams = atoi(env) != 0;
  if ((env = getenv("JIMM_FUSE_LN"))) m->fuse_ln = atoi(env) != 0;
  if ((env = getenv("JIMM_EPI_MODE_16"))) m->epi_mode_16 = atoi(env);
  if ((env = getenv("JIMM_EPI_MODE_RES"))) m->epi_mode_res = atoi(env);
  *out = m;
  return 0;
}

// jimm_model_set_param (fn; an owned copy, ref null) and jimm_model_set_param_ref (a borrowed host pointer, ref = host)
static int add_param(jimm_model_t* m, const char* fn, const char* flax_path, const void* host, const void* ref, const int64_t* shape, int ndim,
                     int dtype, bool transposed) {
  if (!m || !flax_path || !host || (ndim > 0 && !shape)) { set_last_error("jimm_model_%s: null argument", fn); return JIMM_EINVAL; }
  if (m->finalized) { set_last_error("model already finalized"); return JIMM_ESTATE; }
  if (dtype < JIMM_F32 || dtype > JIMM_BF16) { set_last_error("%s: unsupported dtype %d", fn, dtype); return JIMM_EINVAL; }
  HostParam hp;
  hp.n = 1;
  for (int i = 0; i < ndim; ++i) {
    if (shape[i] < 0) { set_last_error("negative dim"); return JIMM_EINVAL; }
    hp.shape.push_back(shape[i]);
    hp.n *= static_cast<size_t>(shape[i]);
  }
  hp.dtype = dtype;  // kept in the caller's element type: the cast happens on the GPU at finalize
  hp.ref = ref;
  hp.transposed = transposed;
  if (transposed && ndim < 2) { set_last_error("%s: '%s': only kernels (ndim >= 2) can be handed over transposed", fn, flax_path); return JIMM_EINVAL; }
  if (!ref) {
    const size_t bytes = hp.n * hp.esize();
    hp.data.resize((bytes + 3) / 4);
    memcpy(hp.data.data(), host, bytes);
  }
  m->host[flax_path] = std::move(hp);
  return 0;
}

int jimm_model_set_param(jimm_model_t* m, const char* flax_path, const void* host, const int64_t* shape, int ndim, int dtype) {
  return add_param(m, "set_param", flax_path, host, nullptr, shape, ndim, dtype, false);
}

int jimm_model_set_param_ref(jimm_model_t* m, const char* flax_path, const void* host, const int64_t* shape, int ndim, int dtype, int flags) {
  return add_param(m, "set_param_ref", flax_path, host, host, shape, ndim, dtype, (flags & JIMM_PARAM_TRANSPOSED) != 0);
}

int jimm_model_finalize(jimm_model_t* m, int max_batch) {
  if (!m) { set_last_error("null model"); return JIMM_EINVAL; }
  if (m->finalized) { set_last_error("model already finalized"); return JIMM_ESTATE; }
  if (max_batch <= 0) { set_last_error("max_batch must be positive"); return JIMM_EINVAL; }
  std::lock_guard<std::mutex> no_capture(g_capture_mu);  // allocations, pinned staging and synchronisation follow
  JIMM_TRY(set_device(m));
  const jimm_config_t& c = m->cfg;
  if (c.kind == JIMM_ENCODER || c.kind == JIMM_MAPHEAD) return finalize_sub(m, max_batch);
  if (c.pooling == JIMM_POOL_MAP) {
    const size_t g = static_cast<size_t>(c.img_size / c.patch);
    JIMM_TRY(map_seq_fits(m, g * g, "the trained image size"));
  }
  const bool dual = dual_kind(c.kind);

  // ---- towers ----
  VisionTower& v = m->vis;
  v.present = true;
  v.img = c.img_size; v.P = c.patch; v.C = c.in_ch; v.D = c.v_width;
  v.n = (c.img_size / c.patch) * (c.img_size / c.patch);
  v.pooling = c.pooling; v.pre_norm = c.pre_norm; v.patch_bias = c.patch_bias; v.eps_outer = c.v_eps_outer;
  v.S = v.n + (v.pooling == JIMM_POOL_CLS ? 1 : 0);
  v.n_pad = ((v.n + 31) / 32) * 32;
  v.patch_scatter = !m->simt && m->epi_mode_res == 2;
  v.interp = c.kind == JIMM_SIGLIP_NAFLEX ? POS_BILINEAR_AA : POS_BICUBIC;
  v.Kp = (c.patch * c.patch * c.in_ch + 7) / 8 * 8;  // K of the patch GEMM, zero-padded (patch 14: 588 -> 592)
  v.enc.c.D = c.v_width; v.enc.c.H = c.v_heads; v.enc.c.M = c.v_mlp; v.enc.c.L = c.v_layers;
  v.enc.c.act = c.v_act; v.enc.c.causal = 0; v.enc.c.eps = c.v_eps_block;
  TextTower& t = m->txt;
  if (dual) {
    t.present = true;
    t.T = c.ctx_len; t.V = c.vocab; t.D = c.t_width; t.pool = c.t_pool; t.eps_outer = c.t_eps_outer;
    t.enc.c.D = c.t_width; t.enc.c.H = c.t_heads; t.enc.c.M = c.t_mlp; t.enc.c.L = c.t_layers;
    t.enc.c.act = c.t_act; t.enc.c.causal = c.t_causal; t.enc.c.eps = c.t_eps_block;
  }
  Packer pk{m};
  const int rc = pack_model(m, pk);
  pk.done();  // one synchronisation for the whole upload, whatever its result
  JIMM_TRY(rc);
  JIMM_TRY(check_all_used(m, "model"));

  // ---- workspace ----
  Workspace& ws = m->ws;
  const int D = v.D;
  const size_t cs = cdt_size(m), Bm = max_batch;
  // token budget: max_batch x the native token count, or x jimm_model_set_max_tokens when that is larger
  const size_t Tv = Bm * std::max(m->max_tokens, v.S);
  // patch rows: max_batch images of the trained grid (rows padded to a multiple of 32 per image) or, under a token budget, the padded
  // rows of one image of up to Tv tokens
  size_t patch_rows = Bm * v.n_pad;
  if (m->max_tokens > 0) patch_rows = std::max(patch_rows, (Tv + 31) / 32 * 32);
  const size_t E = dual ? t.D : vision_out_dim(m);
  JIMM_TRY(alloc_workspace(m, Bm, Tv, big_bytes(m, Tv, patch_rows), std::max(dual ? Bm * Bm : Bm * vision_out_dim(m), Bm * E)));
  if (dual) {  // the text tower's own buffers (it runs concurrently with the vision tower)
    const size_t Tt = Bm * t.T;
    JIMM_TRY(alloc_stack(m, Tt, t.D, std::max(Tt * 3 * t.D * 2, Tt * t.enc.c.M * cs), &m->wt.enc));
    JIMM_TRY(m->pool.alloc(&m->wt.pooled, Bm * t.D * cs));
    JIMM_TRY(m->pool.alloc(&m->wt.idx, Bm * sizeof(int)));
    JIMM_TRY(m->pool.alloc(&ws.in_ids, Bm * t.T * sizeof(int32_t)));
    m->wt.pk_seqs = static_cast<int>(std::min<size_t>(Tt, 65535));  // one token each at most; the attention grid's z limit
    JIMM_TRY(m->pool.alloc(&m->wt.pk_meta, (2 * static_cast<size_t>(m->wt.pk_seqs) + 1) * sizeof(int)));
  }
  JIMM_TRY(m->pool.alloc(&ws.emb_i, Bm * E * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&ws.emb_t, Bm * E * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&ws.nrm_i, Bm * E * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&ws.nrm_t, Bm * E * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&ws.in_img, Bm * v.img * v.img * v.C * sizeof(float)));
  JIMM_TRY(m->pool.alloc(&ws.pk_meta, (2 * Bm + 1) * sizeof(int)));
  if (m->graph_max_batch > 0) {
    const size_t gw = std::max(static_cast<size_t>(vision_out_dim(m)), E);
    const size_t gb = std::min(static_cast<size_t>(m->graph_max_batch), Bm);
    JIMM_TRY(m->pool.alloc(&m->graph_out, gb * gw * sizeof(float)));
    if (dual) JIMM_TRY(m->pool.alloc(&m->graph_out_t, gb * gw * sizeof(float)));
  }

  // ---- GEMM plans (TMA descriptors bound to the fixed workspace / weight buffers) ----
  JIMM_TRY(plan_patch(m, v.n, v.n_pad, v.S, max_batch, v.pos, &v.p_patch));
  {  // as many patch rows as the token budget and ws.big hold (packed_fit keeps a chunk's rows within both)
    const size_t rows = std::min(Tv, m->ws_big / (static_cast<size_t>(v.Kp) * cs));
    JIMM_TRY(gemm_plan_init(&v.p_patch_packed, m->cdt, ws.enc.big, v.Kp, v.patch.w, v.Kp, static_cast<int>(rows), D, v.Kp,
                            epi_plain(v.patch, ACT_NONE, ws.enc.x, DT_F32, D, 2)));
  }
  JIMM_TRY(plan_encoder(m, &v.enc, static_cast<int>(Tv), ws.enc));
  if (v.head.N > 0)
    JIMM_TRY(gemm_plan_init(&v.p_head, m->cdt, ws.pooled, D, v.head.w, D, static_cast<int>(Bm), v.head.N, D,
                            epi_plain(v.head, ACT_NONE, ws.out_dev, DT_F32, v.head.N, 0)));
  if (v.pooling == JIMM_POOL_MAP) JIMM_TRY(plan_map_head(m, static_cast<int>(Bm), static_cast<int>(Tv)));
  if (dual) {
    JIMM_TRY(plan_encoder(m, &t.enc, static_cast<int>(Bm) * t.T, m->wt.enc));
    JIMM_TRY(gemm_plan_init(&t.p_head, m->cdt, m->wt.pooled, t.D, t.head.w, t.D, static_cast<int>(Bm), t.D, t.D,
                            epi_plain(t.head, ACT_NONE, ws.out_dev, DT_F32, t.D, 0)));
    JIMM_TRY(gemm_plan_init(&t.p_head_packed, m->cdt, m->wt.enc.h, t.D, t.head.w, t.D, m->wt.pk_seqs, t.D, t.D,
                            epi_plain(t.head, ACT_NONE, ws.out_dev, DT_F32, t.D, 0)));
  }
  JIMM_CUDA_CHECK(cudaDeviceSynchronize());
  m->max_batch = max_batch;
  m->finalized = true;
  return 0;
}

int jimm_model_set_max_tokens(jimm_model_t* m, int tokens_per_sample) {
  if (!m) { set_last_error("null model"); return JIMM_EINVAL; }
  if (m->finalized) { set_last_error("jimm_model_set_max_tokens: call it before jimm_model_finalize"); return JIMM_ESTATE; }
  if (m->cfg.kind == JIMM_ENCODER || m->cfg.kind == JIMM_MAPHEAD) {
    set_last_error("jimm_model_set_max_tokens: sub-module handles take their token count from ctx_len");
    return JIMM_EINVAL;
  }
  if (tokens_per_sample <= 0) { set_last_error("jimm_model_set_max_tokens: tokens_per_sample must be positive (got %d)", tokens_per_sample); return JIMM_EINVAL; }
  m->max_tokens = tokens_per_sample;
  return 0;
}

int jimm_model_destroy(jimm_model_t* m) {
  if (!m) return 0;
  std::lock_guard<std::mutex> no_capture(g_capture_mu);  // device synchronisation and frees follow
  cudaSetDevice(m->device);
  cudaDeviceSynchronize();
  comm_destroy(&m->comm);
  graphs_release(m);
  if (m->capture_stream) cudaStreamDestroy(m->capture_stream);
  if (m->text_stream) { cudaStreamDestroy(m->text_stream); cudaEventDestroy(m->ev_fork); cudaEventDestroy(m->ev_join); }
  for (cudaEvent_t e : m->prof_ev) cudaEventDestroy(e);
  if (m->copy_stream) {
    cudaStreamDestroy(m->copy_stream);
    for (int i = 0; i < jimm_model::kHostSlices; ++i) { cudaEventDestroy(m->ev_copied[i]); cudaEventDestroy(m->ev_consumed[i]); }
    cudaEventDestroy(m->ev_start);
  }
  if (m->ws.in_u8) cudaFree(m->ws.in_u8);
  m->pool.release();
  delete m;
  return 0;
}

int jimm_model_output_dim(const jimm_model_t* m, int* vision_out, int* text_out) {
  if (!m) { set_last_error("null model"); return JIMM_EINVAL; }
  if (vision_out) *vision_out = m->cfg.kind == JIMM_VIT && m->cfg.num_classes > 0 ? m->cfg.num_classes
                                : (m->cfg.kind == JIMM_CLIP ? m->cfg.t_width : m->cfg.v_width);
  if (text_out) *text_out = m->cfg.t_width;
  return 0;
}
int jimm_model_max_batch(const jimm_model_t* m) { return m ? m->max_batch : 0; }

// ---- forward, device buffers ----
// How many images of a gh x gw patch grid one chunk of an off-grid call runs: max_batch, or fewer when the token-sized buffers (x, h,
// ln_cnt, h8 / sa: ws_rows rows) or ws.big (big_bytes) hold fewer.  0: one image does not fit.
static size_t grid_chunk(const jimm_model* m, int gh, int gw) {
  const VisionTower& v = m->vis;
  const size_t n = static_cast<size_t>(gh) * gw, S = n + (v.pooling == JIMM_POOL_CLS ? 1 : 0), n_pad = (n + 31) / 32 * 32;
  return std::min({static_cast<size_t>(m->max_batch), m->ws_rows / S, m->ws_big / big_bytes(m, S, v.patch_scatter ? n_pad : n)});
}

// JIMM_EINVAL for an H x W image that alone does not fit the vision workspace
static int image_too_large(const jimm_model* m, int H, int W) {
  const VisionTower& v = m->vis;
  const int gh = H / v.P, gw = W / v.P, off = v.pooling == JIMM_POOL_CLS ? 1 : 0;
  set_last_error("a %dx%d image needs %zu tokens (%dx%d patches%s), more than fit this handle's vision workspace (%zu tokens in all); "
                 "raise the budget with jimm_model_set_max_tokens before jimm_model_finalize", H, W, static_cast<size_t>(gh) * gw + off, gh, gw,
                 off ? " + CLS" : "", m->ws_rows);
  return JIMM_EINVAL;
}

// JIMM_EINVAL for an H x W image past the MAP head's sequence limit (map_seq_fits); 0 for a CLS tower
static int image_map_fits(const jimm_model* m, int H, int W) {
  const VisionTower& v = m->vis;
  if (v.pooling != JIMM_POOL_MAP) return 0;
  char what[64];
  snprintf(what, sizeof what, "a %dx%d image (%dx%d patches)", H, W, H / v.P, W / v.P);
  return map_seq_fits(m, static_cast<size_t>(H / v.P) * (W / v.P), what);
}

// H x W images cut into the trained patch grid (they differ from the trained size in the trailing pixels at most)
static bool trained_grid(const VisionTower& v, int H, int W) { return H / v.P == v.img / v.P && W / v.P == v.img / v.P; }

// The off-grid state for H x W images: the patch grid, how many images a chunk runs (grid_chunk) and the patch GEMM plan for that many.
// The plan is host-side tensor maps only, so the cache is simply dropped when full.
static int get_grid(jimm_model* m, int H, int W, PatchGrid** out) {
  const VisionTower& v = m->vis;
  const int gh = H / v.P, gw = W / v.P;
  auto it = m->grids.find(std::make_pair(gh, gw));
  if (it != m->grids.end()) { *out = &it->second; return 0; }
  JIMM_TRY(image_map_fits(m, H, W));
  const size_t chunk = grid_chunk(m, gh, gw);
  if (chunk == 0) return image_too_large(m, H, W);
  PatchGrid g;
  g.gh = gh; g.gw = gw; g.n = gh * gw; g.n_pad = (g.n + 31) / 32 * 32; g.S = g.n + (v.pooling == JIMM_POOL_CLS ? 1 : 0);
  g.chunk = static_cast<int>(chunk);
  JIMM_TRY(plan_patch(m, g.n, g.n_pad, g.S, g.chunk, nullptr, &g.patch));  // adds onto the resampled table already in x
  if (m->grids.size() >= jimm_model::kMaxGrids) m->grids.clear();
  *out = &(m->grids[std::make_pair(gh, gw)] = g);
  return 0;
}

// Vision forward of B images of src.H x src.W (IMG_DENSE) on the patch grid `grid` (null: the trained grid).  The native size goes through
// exec_vision (graphs, staging); other sizes run eagerly.  A token call (sink) always runs eagerly, its chunk of images from b0 on writing
// from output row b0 * S on; out may then be null.
static int vision_chunks(jimm_model* m, const ImageSrc& src, int in_dtype, int B, const PatchGrid* grid, float* out, cudaStream_t s,
                         const TokenSink* sink = nullptr) {
  const VisionTower& v = m->vis;
  const bool native = src.H == v.img && src.W == v.img;
  const int od = vision_out_dim(m);
  return for_chunks(B, grid ? grid->chunk : m->max_batch, [&](int b0, int nb) {
    const void* img = src.from(b0).img;
    float* dst = out ? out + static_cast<size_t>(b0) * od : nullptr;
    if (native && !sink) return exec_vision(m, img, in_dtype, nb, dst, s);
    const size_t S = grid ? grid->S : v.S;
    const TokenSink at = sink ? sink->at(b0 * S, b0 * S * S) : TokenSink{};
    return run_vision(m, img, in_dtype, nb, src.H, src.W, grid, dst, s, sink ? &at : nullptr);
  });
}

int jimm_model_images_per_call(const jimm_model_t* m, int H, int W, int* images) {
  JIMM_TRY(check_ready(m, 0));
  if (!images) { set_last_error("jimm_model_images_per_call: null argument"); return JIMM_EINVAL; }
  JIMM_TRY(check_vision(m, nullptr));
  JIMM_TRY(check_patch(m, H, W));
  const VisionTower& v = m->vis;
  const bool trained = trained_grid(v, H, W);
  if (!trained) JIMM_TRY(image_map_fits(m, H, W));
  *images = trained ? m->max_batch : static_cast<int>(grid_chunk(m, H / v.P, W / v.P));
  return 0;
}

// Does a chunk of T packed tokens fit the vision workspace?  The token-sized buffers hold ws_rows rows, and ws.big the chunk's phases
// (big_bytes), with the patch-GEMM operand laid out by token: T rows.  One image fits whenever grid_chunk says so, except where its
// token-layout patch rows (S rather than the padded n_pad) outgrow every other term of a handle without a set_max_tokens budget.
static bool packed_fit(const jimm_model* m, size_t T) { return T <= m->ws_rows && big_bytes(m, T, T) <= m->ws_big; }

// sum of (tok[b + 1] - tok[b])^2 over the samples of a packed chunk's offsets: what an attention call's outputs advance by, per head
static size_t sum_squares(const std::vector<int>& tok) {
  size_t n = 0;
  for (size_t b = 0; b + 1 < tok.size(); ++b) n += static_cast<size_t>(tok[b + 1] - tok[b]) * (tok[b + 1] - tok[b]);
  return n;
}

// B images of different sizes (IMG_LIST / IMG_ROWS): chunks of consecutive images, each as many as fit (packed_fit, at most max_batch),
// run packed.  A token call (sink): each chunk writes from its first token row on; out may then be null.
static int vision_packed(jimm_model* m, const ImageSrc& src, int in_dtype, int B, float* out, cudaStream_t s, const TokenSink* sink) {
  const VisionTower& v = m->vis;
  const int off = v.pooling == JIMM_POOL_CLS ? 1 : 0;
  const int od = vision_out_dim(m);
  std::vector<int> tok;
  size_t t0 = 0, sq0 = 0;  // the chunk's first token row; the sum of S_b^2 over the samples before it
  for (int b0 = 0; b0 < B;) {
    tok.assign(1, 0);
    int b1 = b0, max_S = 0;
    while (b1 < B && b1 - b0 < m->max_batch) {
      const int S = (src.Hs[b1] / v.P) * (src.Ws[b1] / v.P) + off;
      if (!packed_fit(m, static_cast<size_t>(tok.back()) + S)) break;
      tok.push_back(tok.back() + S);
      max_S = std::max(max_S, S);
      ++b1;
    }
    float* dst = out ? out + static_cast<size_t>(b0) * od : nullptr;
    const TokenSink at = sink ? sink->at(t0, sq0) : TokenSink{};
    JIMM_TRY(run_vision_packed(m, src.from(b0), in_dtype, b1 - b0, tok.data(), max_S, dst, s, sink ? &at : nullptr));
    t0 += tok.back();
    sq0 += sum_squares(tok);
    b0 = b1;
  }
  return 0;
}

// A token call (sink) runs eagerly, the chunk from sequence b0 on writing from output row b0 * T on; out may then be null.
static int text_chunks(jimm_model* m, const int32_t* ids, int B, int T, float* out, cudaStream_t s, const TokenSink* sink = nullptr) {
  return for_chunks(B, m->max_batch, [&](int b0, int nb) {
    const int32_t* src = ids + static_cast<size_t>(b0) * T;
    float* dst = out ? out + static_cast<size_t>(b0) * m->txt.D : nullptr;
    if (!sink) return exec_text(m, src, nb, T, dst, s);
    const TokenSink at = sink->at(static_cast<size_t>(b0) * T, static_cast<size_t>(b0) * T * T);
    return run_text(m, src, nb, T, dst, s, &at);
  });
}

// B token sequences of lengths len[b] (ids: their concatenation): chunks of consecutive sequences, each as many as the text workspace's
// max_batch x context_length token rows hold (at most pk_seqs), run packed.  The chunks are cut by tokens, not by sequences: short
// prompts fill a chunk with several times max_batch sequences, and its GEMMs with as many rows as a padded call of max_batch.
// A token call (sink): each chunk writes from its first row of ids on; out may then be null.
static int text_packed(jimm_model* m, const int32_t* ids, int B, const int* len, float* out, cudaStream_t s, const TokenSink* sink) {
  const int budget = m->max_batch * m->txt.T;
  std::vector<int> tok;
  size_t r0 = 0, sq0 = 0;  // the chunk's first row of ids; the sum of len^2 over the sequences before it
  for (int b0 = 0; b0 < B;) {
    tok.assign(1, 0);
    int b1 = b0, max_S = 0;
    while (b1 < B && b1 - b0 < m->wt.pk_seqs && tok.back() + len[b1] <= budget) {
      tok.push_back(tok.back() + len[b1]);
      max_S = std::max(max_S, len[b1]);
      ++b1;
    }
    float* dst = out ? out + static_cast<size_t>(b0) * m->txt.D : nullptr;
    const TokenSink at = sink ? sink->at(r0, sq0) : TokenSink{};
    JIMM_TRY(run_text_packed(m, ids + r0, b1 - b0, tok.data(), max_S, dst, s, sink ? &at : nullptr));
    r0 += tok.back();
    sq0 += sum_squares(tok);
    b0 = b1;
  }
  return 0;
}

// ---- the forward calls on device inputs ----
// The request of a per-token call (fn names it) on the tower with encoder `enc` and final norm (ln, eps), as the sink of its chunks.
// pooled: the call writes the pooled output too, so every block runs.
static int tokens_sink(const char* fn, const jimm_tokens_req_t* req, const Encoder& enc, const LNW& ln, float eps, bool pooled, TokenSink* sink) {
  const int L = enc.c.L;
  if (!req || !req->layers || !req->out) { set_last_error("%s: null request", fn); return JIMM_EINVAL; }
  if (req->n < 1 || req->n > L + 2) { set_last_error("%s: %d layer requests, outside 1 .. L + 2 = %d", fn, req->n, L + 2); return JIMM_EINVAL; }
  if (req->out_dtype != JIMM_F32 && req->out_dtype != JIMM_F16 && req->out_dtype != JIMM_BF16) {
    set_last_error("%s: output dtype %d; hidden states are JIMM_F32, JIMM_F16 or JIMM_BF16", fn, req->out_dtype);
    return JIMM_EINVAL;
  }
  int blocks = pooled ? L : 0;
  for (int j = 0; j < req->n; ++j) {
    const int k = req->layers[j];
    if (k != JIMM_LAYER_FINAL && (k < 0 || k > L)) {
      set_last_error("%s: request %d asks for layer %d, outside 0 .. %d (or JIMM_LAYER_FINAL)", fn, j, k, L);
      return JIMM_EINVAL;
    }
    if (!req->out[j] || reinterpret_cast<uintptr_t>(req->out[j]) % 16 != 0) {
      set_last_error("%s: output buffer %d is null or not 16-byte aligned", fn, j);
      return JIMM_EINVAL;
    }
    blocks = std::max(blocks, k == JIMM_LAYER_FINAL ? L : k);
  }
  *sink = TokenSink{};
  sink->n = req->n;
  sink->layers = req->layers;
  sink->out = req->out;
  sink->out_type = req->out_dtype;
  sink->blocks = blocks;
  sink->ln = &ln;
  sink->eps = eps;
  return 0;
}

// The request of an attention call (fn names it) on the tower with encoder `enc` (map_head: the tower pools with a MAP head), as the
// sink of its chunks.  pooled or a JIMM_ATTN_MAP request: every block runs.
static int attn_sink(const char* fn, const jimm_attn_req_t* req, const Encoder& enc, bool map_head, bool pooled, TokenSink* sink) {
  const int L = enc.c.L;
  if (!req || !req->blocks || !req->out) { set_last_error("%s: null request", fn); return JIMM_EINVAL; }
  if (req->n < 1 || req->n > L + 1) { set_last_error("%s: %d attention requests, outside 1 .. L + 1 = %d", fn, req->n, L + 1); return JIMM_EINVAL; }
  if (req->out_dtype != JIMM_F32 && req->out_dtype != JIMM_F16 && req->out_dtype != JIMM_BF16) {
    set_last_error("%s: output dtype %d; attention weights are JIMM_F32, JIMM_F16 or JIMM_BF16", fn, req->out_dtype);
    return JIMM_EINVAL;
  }
  int blocks = pooled ? L : 0;
  bool map = false;
  for (int j = 0; j < req->n; ++j) {
    const int k = req->blocks[j];
    if (k == JIMM_ATTN_MAP) {
      if (!map_head) { set_last_error("%s: request %d asks for JIMM_ATTN_MAP on a tower without a MAP head", fn, j); return JIMM_EINVAL; }
      map = true;
    } else if (k < 0 || k >= L) {
      set_last_error("%s: request %d asks for block %d, outside 0 .. %d (or JIMM_ATTN_MAP)", fn, j, k, L - 1);
      return JIMM_EINVAL;
    }
    if (!req->out[j] || reinterpret_cast<uintptr_t>(req->out[j]) % 16 != 0) {
      set_last_error("%s: output buffer %d is null or not 16-byte aligned", fn, j);
      return JIMM_EINVAL;
    }
    blocks = std::max(blocks, k == JIMM_ATTN_MAP ? L : k + 1);
  }
  *sink = TokenSink{};
  sink->an = req->n;
  sink->ablocks = req->blocks;
  sink->aout = req->out;
  sink->aout_type = req->out_dtype;
  sink->map = map;
  sink->blocks = blocks;
  return 0;
}

// The kinds of forward call: the pooled output (jimm_encode_*), the same on a ViT / tower handle only (jimm_vit_forward*), the hidden
// states of a request with the pooled output optional (jimm_image_tokens* / jimm_text_tokens*), and the attention weights of a request,
// the same (jimm_image_attn* / jimm_text_attn*)
enum CallKind { CALL_ENCODE, CALL_VIT, CALL_TOKENS, CALL_ATTN };

static int null_argument(const char* fn) {
  set_last_error("%s: null argument", fn);
  return JIMM_EINVAL;
}

// The shape step of a vision call (fn names it), which fills in src's sizes.  IMG_DENSE: images of at least one patch, and off the
// trained grid its plan (*grid; null on the trained grid).  IMG_ROWS: every sample's grid within its N rows, the image sizes it cuts
// written to cut.  IMG_LIST and IMG_ROWS: every image present, of at least one patch, within the MAP head's limit and alone fitting
// a packed chunk.
static int image_shapes(jimm_model* m, const char* fn, ImageSrc* src, int in_dtype, int B, std::vector<int>* cut, PatchGrid** grid) {
  const VisionTower& v = m->vis;
  *grid = nullptr;
  if (src->form == IMG_DENSE) {
    if (src->native) src->H = src->W = v.img;
    JIMM_TRY(check_patch(m, src->H, src->W));
    if (!trained_grid(v, src->H, src->W)) JIMM_TRY(get_grid(m, src->H, src->W, grid));
    src->sample_bytes = static_cast<size_t>(src->H) * src->W * v.C * dtype_size(in_dtype);
    return 0;
  }
  if (src->form == IMG_ROWS) {
    cut->resize(2 * static_cast<size_t>(B));
    for (int b = 0; b < B; ++b) {
      const int gh = src->grid[2 * b], gw = src->grid[2 * b + 1];
      if (gh < 1 || gw < 1 || gh > INT32_MAX / v.P || gw > INT32_MAX / v.P) {
        set_last_error("%s: sample %d has a %dx%d patch grid (each edge from 1 up)", fn, b, gh, gw);
        return JIMM_EINVAL;
      }
      if (static_cast<int64_t>(gh) * gw > src->N) {
        set_last_error("%s: sample %d has a %dx%d patch grid, %lld patches, more than its N = %d rows", fn, b, gh, gw,
                       static_cast<long long>(gh) * gw, src->N);
        return JIMM_EINVAL;
      }
      (*cut)[b] = gh * v.P;
      (*cut)[B + b] = gw * v.P;
    }
    src->Hs = cut->data();
    src->Ws = cut->data() + B;
    src->sample_bytes = static_cast<size_t>(src->N) * v.P * v.P * v.C * dtype_size(in_dtype);
  }
  const int off = v.pooling == JIMM_POOL_CLS ? 1 : 0;
  for (int b = 0; b < B; ++b) {
    const int H = src->Hs[b], W = src->Ws[b];
    if (src->imgs && !src->imgs[b]) { set_last_error("packed call: image %d is a null pointer", b); return JIMM_EINVAL; }
    if (H < v.P || W < v.P) { set_last_error("image %d: %dx%d is smaller than one %dx%d patch", b, H, W, v.P, v.P); return JIMM_EINVAL; }
    JIMM_TRY(image_map_fits(m, H, W));
    if (!packed_fit(m, static_cast<size_t>(H / v.P) * (W / v.P) + off)) return image_too_large(m, H, W);
  }
  return 0;
}

// Every vision call on device images (fn names it): the checks in the order include/jimm_b200.h states, then the chunker of the form.
static int image_call(jimm_model* m, const char* fn, CallKind kind, ImageSrc src, int in_dtype, int B, float* out, const jimm_tokens_req_t* req,
                      void* stream, const jimm_attn_req_t* areq = nullptr) {
  JIMM_TRY(check_ready(m, B));
  JIMM_TRY(check_image_dtype(in_dtype));
  if (src.form != IMG_ROWS) {
    JIMM_TRY(check_vision(m, kind == CALL_VIT ? fn : nullptr));
  } else if (m->cfg.kind != JIMM_SIGLIP_NAFLEX) {
    set_last_error("%s: the model is not a SigLIP 2 NaFlex handle (kind %d); use jimm_encode_image_packed", fn, m->cfg.kind);
    return JIMM_EINVAL;
  }
  TokenSink sink;
  if (kind == CALL_TOKENS) JIMM_TRY(tokens_sink(fn, req, m->vis.enc, m->vis.ln_post, m->vis.eps_outer, out != nullptr, &sink));
  if (kind == CALL_ATTN) JIMM_TRY(attn_sink(fn, areq, m->vis.enc, m->vis.pooling == JIMM_POOL_MAP, out != nullptr, &sink));
  const bool sinks = kind == CALL_TOKENS || kind == CALL_ATTN;
  const bool inputs = src.form == IMG_LIST ? src.imgs && src.Hs && src.Ws : src.img && (src.form == IMG_DENSE || src.grid);
  if (B > 0 && (!inputs || (!sinks && !out))) return null_argument(fn);
  std::vector<int> cut;
  PatchGrid* grid = nullptr;
  JIMM_TRY(image_shapes(m, fn, &src, in_dtype, B, &cut, &grid));
  JIMM_TRY(set_device(m));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const TokenSink* sk = sinks ? &sink : nullptr;
  if (src.form == IMG_DENSE) return vision_chunks(m, src, in_dtype, B, grid, out, s, sk);
  return vision_packed(m, src, in_dtype, B, out, s, sk);
}

// The token ids of a text call: B sequences of T ids each (ids [B, T]), or, packed, of len[b] ids one after another
struct TextSrc {
  const int32_t* ids;
  int T;
  const int* len;
  bool packed;
};

// Every text call on device ids (fn names it), on the pattern of image_call
static int text_call(jimm_model* m, const char* fn, CallKind kind, const TextSrc& src, int B, float* out, const jimm_tokens_req_t* req,
                     void* stream, const jimm_attn_req_t* areq = nullptr) {
  JIMM_TRY(check_ready(m, B));
  JIMM_TRY(check_text(m));
  TokenSink sink;
  if (kind == CALL_TOKENS) JIMM_TRY(tokens_sink(fn, req, m->txt.enc, m->txt.ln_final, m->txt.eps_outer, out != nullptr, &sink));
  if (kind == CALL_ATTN) JIMM_TRY(attn_sink(fn, areq, m->txt.enc, false, out != nullptr, &sink));
  const bool sinks = kind == CALL_TOKENS || kind == CALL_ATTN;
  if (B > 0 && (!src.ids || (src.packed && !src.len) || (!sinks && !out))) return null_argument(fn);
  JIMM_TRY(src.packed ? check_lens(m, B, src.len) : check_text_len(m, src.T));
  JIMM_TRY(set_device(m));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const TokenSink* sk = sinks ? &sink : nullptr;
  if (src.packed) return text_packed(m, src.ids, B, src.len, out, s, sk);
  return text_chunks(m, src.ids, B, src.T, out, s, sk);
}

int jimm_vit_forward(jimm_model_t* m, const void* img, int in_dtype, int B, float* out, void* stream) {
  return image_call(m, "jimm_vit_forward", CALL_VIT, ImageSrc::trained(img), in_dtype, B, out, nullptr, stream);
}

int jimm_encode_image(jimm_model_t* m, const void* img, int in_dtype, int B, float* out, void* stream) {
  return image_call(m, "jimm_encode_image", CALL_ENCODE, ImageSrc::trained(img), in_dtype, B, out, nullptr, stream);
}

int jimm_vit_forward_hw(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, float* out, void* stream) {
  return image_call(m, "jimm_vit_forward_hw", CALL_VIT, ImageSrc::dense(img, H, W), in_dtype, B, out, nullptr, stream);
}

int jimm_encode_image_hw(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, float* out, void* stream) {
  return image_call(m, "jimm_encode_image_hw", CALL_ENCODE, ImageSrc::dense(img, H, W), in_dtype, B, out, nullptr, stream);
}

int jimm_vit_forward_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W, float* out, void* stream) {
  return image_call(m, "jimm_vit_forward_packed", CALL_VIT, ImageSrc::list(imgs, H, W), in_dtype, B, out, nullptr, stream);
}

int jimm_encode_image_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W, float* out, void* stream) {
  return image_call(m, "jimm_encode_image_packed", CALL_ENCODE, ImageSrc::list(imgs, H, W), in_dtype, B, out, nullptr, stream);
}

// HuggingFace NaFlex patch rows: sample b is the (gh*P) x (gw*P) image of its first gh*gw rows, run through the packed chunker
int jimm_encode_image_patches(jimm_model_t* m, const void* patches, int in_dtype, int B, int N, const int* grid, float* out, void* stream) {
  return image_call(m, "jimm_encode_image_patches", CALL_ENCODE, ImageSrc::rows(patches, N, grid), in_dtype, B, out, nullptr, stream);
}

int jimm_encode_text(jimm_model_t* m, const int32_t* ids, int B, int T, float* out, void* stream) {
  return text_call(m, "jimm_encode_text", CALL_ENCODE, TextSrc{ids, T, nullptr, false}, B, out, nullptr, stream);
}

int jimm_encode_text_packed(jimm_model_t* m, const int32_t* ids, int B, const int* len, float* out, void* stream) {
  return text_call(m, "jimm_encode_text_packed", CALL_ENCODE, TextSrc{ids, 0, len, true}, B, out, nullptr, stream);
}

int jimm_image_tokens(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, const jimm_tokens_req_t* req, float* pooled, void* stream) {
  return image_call(m, "jimm_image_tokens", CALL_TOKENS, ImageSrc::dense(img, H, W), in_dtype, B, pooled, req, stream);
}

int jimm_image_tokens_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W, const jimm_tokens_req_t* req,
                             float* pooled, void* stream) {
  return image_call(m, "jimm_image_tokens_packed", CALL_TOKENS, ImageSrc::list(imgs, H, W), in_dtype, B, pooled, req, stream);
}

int jimm_image_tokens_patches(jimm_model_t* m, const void* patches, int in_dtype, int B, int N, const int* grid, const jimm_tokens_req_t* req,
                              float* pooled, void* stream) {
  return image_call(m, "jimm_image_tokens_patches", CALL_TOKENS, ImageSrc::rows(patches, N, grid), in_dtype, B, pooled, req, stream);
}

int jimm_text_tokens(jimm_model_t* m, const int32_t* ids, int B, int T, const jimm_tokens_req_t* req, float* pooled, void* stream) {
  return text_call(m, "jimm_text_tokens", CALL_TOKENS, TextSrc{ids, T, nullptr, false}, B, pooled, req, stream);
}

int jimm_text_tokens_packed(jimm_model_t* m, const int32_t* ids, int B, const int* len, const jimm_tokens_req_t* req, float* pooled, void* stream) {
  return text_call(m, "jimm_text_tokens_packed", CALL_TOKENS, TextSrc{ids, 0, len, true}, B, pooled, req, stream);
}

int jimm_image_attn(jimm_model_t* m, const void* img, int in_dtype, int B, int H, int W, const jimm_attn_req_t* req, float* pooled, void* stream) {
  return image_call(m, "jimm_image_attn", CALL_ATTN, ImageSrc::dense(img, H, W), in_dtype, B, pooled, nullptr, stream, req);
}

int jimm_image_attn_packed(jimm_model_t* m, const void* const* imgs, int in_dtype, int B, const int* H, const int* W, const jimm_attn_req_t* req,
                           float* pooled, void* stream) {
  return image_call(m, "jimm_image_attn_packed", CALL_ATTN, ImageSrc::list(imgs, H, W), in_dtype, B, pooled, nullptr, stream, req);
}

int jimm_image_attn_patches(jimm_model_t* m, const void* patches, int in_dtype, int B, int N, const int* grid, const jimm_attn_req_t* req,
                            float* pooled, void* stream) {
  return image_call(m, "jimm_image_attn_patches", CALL_ATTN, ImageSrc::rows(patches, N, grid), in_dtype, B, pooled, nullptr, stream, req);
}

int jimm_text_attn(jimm_model_t* m, const int32_t* ids, int B, int T, const jimm_attn_req_t* req, float* pooled, void* stream) {
  return text_call(m, "jimm_text_attn", CALL_ATTN, TextSrc{ids, T, nullptr, false}, B, pooled, nullptr, stream, req);
}

int jimm_text_attn_packed(jimm_model_t* m, const int32_t* ids, int B, const int* len, const jimm_attn_req_t* req, float* pooled, void* stream) {
  return text_call(m, "jimm_text_attn_packed", CALL_ATTN, TextSrc{ids, 0, len, true}, B, pooled, nullptr, stream, req);
}

int jimm_contrastive_logits(jimm_model_t* m, const float* img_e, int Bi, const float* txt_e, int Bt, float* logits, void* stream) {
  JIMM_TRY(check_ready(m, Bi));
  JIMM_TRY(check_text(m));
  if (Bi > m->max_batch || Bt > m->max_batch) { set_last_error("contrastive_logits: batch (%d,%d) exceeds max_batch %d", Bi, Bt, m->max_batch); return JIMM_EINVAL; }
  JIMM_TRY(set_device(m));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int E = m->txt.D;
  JIMM_TRY(l2_normalize_run(img_e, m->ws.nrm_i, E, Bi, E, s));
  JIMM_TRY(l2_normalize_run(txt_e, m->ws.nrm_t, E, Bt, E, s));
  return logits_run(m->ws.nrm_i, m->ws.nrm_t, m->logit_scale, m->logit_bias, logits, Bi, Bt, E, Bt, s);
}

int jimm_search(jimm_model_t* m, const float* queries, int Q, const float* gallery, int N, int k, float* values, int32_t* indices, void* stream) {
  JIMM_TRY(check_ready(m, Q));
  JIMM_TRY(check_text(m));
  if (N < 1 || k < 1 || k > N || k > 1024) { set_last_error("search: k=%d outside 1 .. min(N=%d, 1024)", k, N); return JIMM_EINVAL; }
  if (!gallery || (Q > 0 && (!queries || !values || !indices))) { set_last_error("search: null queries, gallery, values or indices"); return JIMM_EINVAL; }
  JIMM_TRY(set_device(m));
  if (Q == 0) return 0;
  return search_run(queries, Q, gallery, N, m->txt.D, m->logit_scale, m->logit_bias, k, values, indices, static_cast<cudaStream_t>(stream));
}

// The gallery index: the model it scores with, the device its rows live on and the stored rows (postprocess.cu owns their formats).
// Only add and search read m; destroy needs the device alone, so an index outlives a model it has been rebound away from.
struct jimm_index {
  jimm_model* m = nullptr;
  int device = 0;
  GalleryStore* store = nullptr;
};

int jimm_index_create(jimm_model_t* m, jimm_index_t** out) {
  JIMM_TRY(check_ready(m, 0));
  JIMM_TRY(check_text(m));
  if (!out) { set_last_error("index: null output handle"); return JIMM_EINVAL; }
  GalleryStore* store = nullptr;
  JIMM_TRY(gallery_create(m->txt.D, &store));
  *out = new jimm_index{m, m->device, store};
  return 0;
}

int jimm_index_rebind(jimm_index_t* idx, jimm_model_t* m) {
  if (!idx) { set_last_error("index: null handle"); return JIMM_EINVAL; }
  JIMM_TRY(check_ready(m, 0));
  JIMM_TRY(check_text(m));
  if (m->device != idx->device || m->txt.D != gallery_width(idx->store)) {
    set_last_error("index rebind: the model (device %d, width %d) does not match the index (device %d, width %d)", m->device, m->txt.D,
                   idx->device, gallery_width(idx->store));
    return JIMM_EINVAL;
  }
  idx->m = m;
  return 0;
}

int jimm_index_add(jimm_index_t* idx, const float* rows, int n, void* stream) {
  if (!idx) { set_last_error("index: null handle"); return JIMM_EINVAL; }
  if (n < 0 || (n > 0 && !rows)) { set_last_error("index add: n=%d rows=%p", n, static_cast<const void*>(rows)); return JIMM_EINVAL; }
  if (gallery_rows(idx->store) + n > 2147483647ll) {
    set_last_error("index add: %lld + %d rows exceed 2^31 - 1", gallery_rows(idx->store), n);
    return JIMM_EINVAL;
  }
  JIMM_TRY(set_device(idx->m));
  return gallery_add(idx->store, rows, n, static_cast<cudaStream_t>(stream));
}

int jimm_index_search(jimm_index_t* idx, const float* queries, int Q, int k, float* values, int32_t* indices, jimm_search_stats* stats, void* stream) {
  return jimm_index_search_keep(idx, queries, Q, k, nullptr, values, indices, stats, stream);
}

int jimm_index_search_keep(jimm_index_t* idx, const float* queries, int Q, int k, const uint8_t* keep, float* values, int32_t* indices,
                           jimm_search_stats* stats, void* stream) {
  if (!idx) { set_last_error("index: null handle"); return JIMM_EINVAL; }
  jimm_model* m = idx->m;
  JIMM_TRY(check_ready(m, Q));
  const long long N = gallery_rows(idx->store);
  if (N < 1 || k < 1 || k > N || k > 1024) { set_last_error("search: k=%d outside 1 .. min(N=%lld, 1024)", k, N); return JIMM_EINVAL; }
  if (Q > 0 && (!queries || !values || !indices)) { set_last_error("search: null queries, values or indices"); return JIMM_EINVAL; }
  JIMM_TRY(set_device(m));
  long long st[3] = {0, 0, 0};
  const int rc = Q == 0 ? 0 : gallery_search(idx->store, queries, Q, m->logit_scale, m->logit_bias, k, keep, values, indices, st,
                                             static_cast<cudaStream_t>(stream));
  if (stats) { stats->rows_rescored = st[0]; stats->fallbacks = st[1]; stats->chunks_screened = st[2]; }
  return rc;
}

// Shared checks and dispatch of jimm_index_range_search (queries) and jimm_index_pairs (queries null, Q = 0).
static int index_range(jimm_index_t* idx, const float* queries, int Q, bool pairs, float threshold, const uint8_t* keep, jimm_hits_t** out,
                       jimm_search_stats* stats, void* stream) {
  const char* what = pairs ? "pairs" : "range search";
  if (!idx) { set_last_error("index: null handle"); return JIMM_EINVAL; }
  if (!out) { set_last_error("%s: null output handle", what); return JIMM_EINVAL; }
  *out = nullptr;
  jimm_model* m = idx->m;
  JIMM_TRY(check_ready(m, Q));
  if (threshold != threshold) { set_last_error("%s: the threshold is NaN", what); return JIMM_EINVAL; }
  if (Q > 0 && !queries) { set_last_error("%s: null queries", what); return JIMM_EINVAL; }
  JIMM_TRY(set_device(m));
  long long st[3] = {0, 0, 0};
  const int rc = gallery_range(idx->store, queries, Q, pairs, threshold, m->logit_scale, m->logit_bias, keep, out, st, static_cast<cudaStream_t>(stream));
  if (stats) { stats->rows_rescored = st[0]; stats->fallbacks = st[1]; stats->chunks_screened = st[2]; }
  return rc;
}

int jimm_index_range_search(jimm_index_t* idx, const float* queries, int Q, float threshold, jimm_hits_t** out, jimm_search_stats* stats,
                            void* stream) {
  return index_range(idx, queries, Q, false, threshold, nullptr, out, stats, stream);
}

int jimm_index_pairs(jimm_index_t* idx, float threshold, jimm_hits_t** out, jimm_search_stats* stats, void* stream) {
  return index_range(idx, nullptr, 0, true, threshold, nullptr, out, stats, stream);
}

int jimm_index_range_search_keep(jimm_index_t* idx, const float* queries, int Q, float threshold, const uint8_t* keep, jimm_hits_t** out,
                                 jimm_search_stats* stats, void* stream) {
  return index_range(idx, queries, Q, false, threshold, keep, out, stats, stream);
}

int jimm_index_pairs_keep(jimm_index_t* idx, float threshold, const uint8_t* keep, jimm_hits_t** out, jimm_search_stats* stats, void* stream) {
  return index_range(idx, nullptr, 0, true, threshold, keep, out, stats, stream);
}

// Removal and compaction touch only the stored rows, so they need the index's device, not its model.
int jimm_index_remove(jimm_index_t* idx, const int32_t* ids, int n, long long* removed, void* stream) {
  if (!idx || !removed) { set_last_error("index remove: null handle or count"); return JIMM_EINVAL; }
  if (n < 0 || (n > 0 && !ids)) { set_last_error("index remove: n=%d ids=%p", n, static_cast<const void*>(ids)); return JIMM_EINVAL; }
  JIMM_CUDA_CHECK(cudaSetDevice(idx->device));
  return gallery_remove(idx->store, ids, n, removed, static_cast<cudaStream_t>(stream));
}

int jimm_index_live(const jimm_index_t* idx, long long* live) {
  if (!idx || !live) { set_last_error("index live: null handle or count"); return JIMM_EINVAL; }
  *live = gallery_live(idx->store);
  return 0;
}

int jimm_index_compact(jimm_index_t* idx, int32_t* old_to_new, void* stream) {
  if (!idx) { set_last_error("index: null handle"); return JIMM_EINVAL; }
  JIMM_CUDA_CHECK(cudaSetDevice(idx->device));
  return gallery_compact(idx->store, old_to_new, static_cast<cudaStream_t>(stream));
}

// k-means reads only the stored rows (scores at unit scale and zero bias), so like removal it needs the index's device, not its model.
int jimm_index_kmeans(jimm_index_t* idx, int C, const float* init_vectors, const int32_t* init_ids, unsigned long long seed, int iters,
                      const uint8_t* keep, float* centroids, int32_t* assign, float* scores, int64_t* counts, int* iterations,
                      jimm_search_stats* stats, void* stream) {
  if (!idx) { set_last_error("index: null handle"); return JIMM_EINVAL; }
  if (C < 1 || C > 65536) { set_last_error("index kmeans: n_clusters=%d outside 1 .. 65536", C); return JIMM_EINVAL; }
  if (iters < 1) { set_last_error("index kmeans: iters=%d must be at least 1", iters); return JIMM_EINVAL; }
  if (init_vectors && init_ids) { set_last_error("index kmeans: give init vectors or init ids, not both"); return JIMM_EINVAL; }
  if (!centroids || !counts || !iterations || (gallery_rows(idx->store) > 0 && (!assign || !scores))) {
    set_last_error("index kmeans: null centroids, assign, scores, counts or iterations");
    return JIMM_EINVAL;
  }
  JIMM_CUDA_CHECK(cudaSetDevice(idx->device));
  long long st[3] = {0, 0, 0};
  const int rc = gallery_kmeans(idx->store, C, init_vectors, init_ids, seed, iters, keep, centroids, assign, scores, counts, iterations, st,
                                static_cast<cudaStream_t>(stream));
  if (stats) { stats->rows_rescored = st[0]; stats->fallbacks = st[1]; stats->chunks_screened = st[2]; }
  return rc;
}

int jimm_index_destroy(jimm_index_t* idx) {
  if (!idx) return 0;
  JIMM_CUDA_CHECK(cudaSetDevice(idx->device));
  gallery_destroy(idx->store);
  delete idx;
  return 0;
}

// Fork the text tower onto the model's side stream (ordered after everything already enqueued on `s`), returning the stream it runs
// on; join_text() makes `s` wait for it.  Profiling (per-GEMM events) and JIMM_DUAL_STREAMS=0 keep the towers on one stream.
static int fork_text(jimm_model* m, cudaStream_t s, cudaStream_t* ts) {
  *ts = s;
  if (!m->dual_streams || m->prof_on) return 0;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone) { cudaGetLastError(); return 0; }
  if (!m->text_stream) {
    JIMM_CUDA_CHECK(cudaStreamCreateWithFlags(&m->text_stream, cudaStreamNonBlocking));
    JIMM_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_fork, cudaEventDisableTiming));
    JIMM_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_join, cudaEventDisableTiming));
  }
  JIMM_CUDA_CHECK(cudaEventRecord(m->ev_fork, s));
  JIMM_CUDA_CHECK(cudaStreamWaitEvent(m->text_stream, m->ev_fork, 0));
  *ts = m->text_stream;
  return 0;
}
static int join_text(jimm_model* m, cudaStream_t s, cudaStream_t ts) {
  if (ts == s) return 0;
  JIMM_CUDA_CHECK(cudaEventRecord(m->ev_join, ts));
  JIMM_CUDA_CHECK(cudaStreamWaitEvent(s, m->ev_join, 0));
  return 0;
}

// encode_image + encode_text of one call, the two towers running concurrently (device inputs); img_e fp32 [Bi,E], txt_e fp32 [Bt,E].
int jimm_dual_encode_hw(jimm_model_t* m, const void* img, int in_dtype, int Bi, int H, int W, const int32_t* ids, int Bt, int T, float* img_e,
                        float* txt_e, void* stream) {
  JIMM_TRY(check_ready(m, Bi));
  JIMM_TRY(check_text(m));
  JIMM_TRY(check_image_dtype(in_dtype));
  JIMM_TRY(check_text_len(m, T));
  ImageSrc src = ImageSrc::dense(img, H, W);
  std::vector<int> cut;
  PatchGrid* grid = nullptr;
  JIMM_TRY(image_shapes(m, "jimm_dual_encode_hw", &src, in_dtype, Bi, &cut, &grid));  // refuse the images before the text tower runs
  JIMM_TRY(set_device(m));
  cudaStream_t s = static_cast<cudaStream_t>(stream), ts = s;
  JIMM_TRY(fork_text(m, s, &ts));
  JIMM_TRY(text_chunks(m, ids, Bt, T, txt_e, ts));
  JIMM_TRY(vision_chunks(m, src, in_dtype, Bi, grid, img_e, s));
  return join_text(m, s, ts);
}

int jimm_dual_encode(jimm_model_t* m, const void* img, int in_dtype, int Bi, const int32_t* ids, int Bt, int T, float* img_e, float* txt_e,
                     void* stream) {
  JIMM_TRY(check_ready(m, Bi));
  return jimm_dual_encode_hw(m, img, in_dtype, Bi, m->vis.img, m->vis.img, ids, Bt, T, img_e, txt_e, stream);
}

int jimm_dual_forward_hw(jimm_model_t* m, const void* img, int in_dtype, int Bi, int H, int W, const int32_t* ids, int Bt, int T, float* logits,
                         void* stream) {
  JIMM_TRY(check_ready(m, Bi));
  if (Bi > m->max_batch || Bt > m->max_batch) { set_last_error("dual_forward: batch (%d,%d) exceeds max_batch %d", Bi, Bt, m->max_batch); return JIMM_EINVAL; }
  JIMM_TRY(jimm_dual_encode_hw(m, img, in_dtype, Bi, H, W, ids, Bt, T, m->ws.emb_i, m->ws.emb_t, stream));
  return jimm_contrastive_logits(m, m->ws.emb_i, Bi, m->ws.emb_t, Bt, logits, stream);
}

int jimm_dual_forward(jimm_model_t* m, const void* img, int in_dtype, int Bi, const int32_t* ids, int Bt, int T, float* logits,
                      void* stream) {
  JIMM_TRY(check_ready(m, Bi));
  return jimm_dual_forward_hw(m, img, in_dtype, Bi, m->vis.img, m->vis.img, ids, Bt, T, logits, stream);
}

// ---- forward of a bare sub-module (device buffers) ----
static int check_sub(jimm_model_t* m, int kind, int B, int S, const void* x, const void* out) {
  JIMM_TRY(check_ready(m, B));
  if (m->cfg.kind != kind) { set_last_error("this handle is not a %s", kind == JIMM_ENCODER ? "Transformer (JIMM_ENCODER)" : "MAP head (JIMM_MAPHEAD)"); return JIMM_EINVAL; }
  if (S <= 0 || S > m->vis.S) { set_last_error("sequence length %d outside (0, %d]", S, m->vis.S); return JIMM_EINVAL; }
  if (!x || !out) { set_last_error("null buffer"); return JIMM_EINVAL; }
  return set_device(m);
}

int jimm_encoder_forward(jimm_model_t* m, const float* x, int B, int S, float* out, void* stream) {
  JIMM_TRY(check_sub(m, JIMM_ENCODER, B, S, x, out));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t row = static_cast<size_t>(S) * m->vis.D;
  return for_chunks(B, m->max_batch, [&](int b0, int nb) {
    JIMM_CUDA_CHECK(cudaMemcpyAsync(m->ws.enc.x, x + b0 * row, nb * row * sizeof(float), cudaMemcpyDeviceToDevice, s));
    JIMM_TRY(run_encoder(m, &m->vis.enc, nb, S, s, m->ws.enc));
    JIMM_CUDA_CHECK(cudaMemcpyAsync(out + b0 * row, m->ws.enc.x, nb * row * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return 0;
  });
}

int jimm_map_head_forward(jimm_model_t* m, const float* x, int B, int S, float* out, void* stream) {
  JIMM_TRY(check_sub(m, JIMM_MAPHEAD, B, S, x, out));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t row = static_cast<size_t>(S) * m->vis.D;
  return for_chunks(B, m->max_batch, [&](int b0, int nb) {
    JIMM_TRY(cast_run(x + b0 * row, m->ws.enc.h, m->cdt, nb * row, s));  // the head's inputs are GEMM operands: compute dtype
    return run_map_head(m, nb, S, out + static_cast<size_t>(b0) * m->vis.D, s);
  });
}

// ---- forward, host buffers ----
static int ensure_copy_stream(jimm_model* m) {
  if (m->copy_stream) return 0;
  JIMM_CUDA_CHECK(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < jimm_model::kHostSlices; ++i) {
    JIMM_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_copied[i], cudaEventDisableTiming));
    JIMM_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_consumed[i], cudaEventDisableTiming));
  }
  JIMM_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_start, cudaEventDisableTiming));
  return 0;
}

// Slice schedule of one super-chunk of nb images on the host path.  Two slices: a head slice whose H2D copy is the only exposed
// one, chosen between nb/head_div and nb/3 so that BOTH slices quantise well into waves of GEMM tiles (a badly chosen
// split costs an extra wave in every GEMM).  JIMM_HOST_SLICES (comma separated sizes) overrides it for experiments.
static void host_slices(const jimm_model* m, int nb, int* sizes, size_t bytes_per_image = 0) {
  for (int i = 0; i < jimm_model::kHostSlices; ++i) sizes[i] = 0;
  sizes[0] = nb;
  if (const char* env = getenv("JIMM_HOST_SLICES")) {
    int k = 0, acc = 0;
    for (const char* q = env; *q && k < jimm_model::kHostSlices - 1;) {
      const int v = atoi(q);
      if (v <= 0 || acc + v >= nb) break;
      sizes[k++] = v;
      acc += v;
      while (*q && *q != ',') ++q;
      if (*q == ',') ++q;
    }
    sizes[k] = nb - acc;
    return;
  }
  if (nb < 128) return;
  // Slicing hides all but the first slice's copy but costs GEMM waves and launches: only worth it when the whole copy is long.  Raw
  // uint8 frames (38 MB for 256 x 224 x 224 x 3) go in one piece.
  if (bytes_per_image && static_cast<size_t>(nb) * bytes_per_image < (static_cast<size_t>(64) << 20)) return;
  static const int head_div = [] { const char* env = getenv("JIMM_HOST_HEAD_DIV"); return (env && atoi(env) > 0) ? atoi(env) : 4; }();
  const int S = m->vis.S, D = m->vis.D, Mm = m->vis.enc.c.M;
  const int sms = device_sm_count();
  auto cost = [&](int n) {
    const long mt = (static_cast<long>(n) * S + GEMM_TILE_M - 1) / GEMM_TILE_M;
    auto rounds = [&](int N) { return (mt * ((N + GEMM_TILE_N - 1) / GEMM_TILE_N) + sms - 1) / sms; };
    return static_cast<double>(D) * rounds(3 * D) + static_cast<double>(D) * rounds(D) + static_cast<double>(D) * rounds(Mm) +
           static_cast<double>(Mm) * rounds(D);
  };
  int best = nb / head_div;
  double best_cost = 1e30;
  for (int c0 = nb / head_div; c0 <= nb / 3; ++c0) {
    const double cst = cost(c0) + cost(nb - c0) + 1e-3 * c0 * D;  // tie-break towards the smaller exposed copy
    if (cst < best_cost) { best_cost = cst; best = c0; }
  }
  sizes[0] = best;
  sizes[1] = nb - best;
}

// Host-buffer vision forward.  pre == nullptr: img_host holds NHWC images of in_dtype at the model's resolution.  pre != nullptr:
// img_host holds raw uint8 RGB frames [B,Hin,Win,3]; each slice is copied as bytes (4x fewer than fp32 pixels), run through the image
// front-end on the compute stream (resize / crop / rescale / normalise into the tower's operand dtype) and then through the tower.
static int vit_forward_host_impl(jimm_model_t* m, const void* img_host, int in_dtype, int B, float* out_host, cudaStream_t s,
                                 jimm_preproc_t* pre, int Hin, int Win) {
  JIMM_TRY(ensure_copy_stream(m));
  const size_t img_elems = static_cast<size_t>(m->vis.img) * m->vis.img * m->vis.C;
  const size_t src_bytes = pre ? static_cast<size_t>(Hin) * Win * 3 : img_elems * dtype_size(in_dtype);  // per image, on the host
  const int tower_dtype = pre ? (m->cdt == DT_TF32 ? JIMM_F32 : m->cdt) : in_dtype;
  const int od = vision_out_dim(m);
  const int kind = pre ? 1 : 0;
  if (pre) {
    const size_t need = static_cast<size_t>(m->max_batch) * src_bytes;
    if (need > m->ws.in_u8_bytes) {  // first call (or larger frames): grow the byte staging buffer
      std::lock_guard<std::mutex> no_capture(g_capture_mu);
      JIMM_CUDA_CHECK(cudaDeviceSynchronize());
      if (m->ws.in_u8) cudaFree(m->ws.in_u8);
      m->ws.in_u8 = nullptr; m->ws.in_u8_bytes = 0;
      JIMM_CUDA_CHECK(cudaMalloc(&m->ws.in_u8, need));
      m->ws.in_u8_bytes = need;
      m->host_chain = false;
    }
  }
  // Sliced pipeline per super-chunk of <= max_batch images: slice i+1 is copied on the side stream while slice i is in the
  // tower, and the next super-chunk's first copy overlaps this one's last forward.  The slices partition the staging buffer
  // (max_batch images), one event pair each; one D2H of the super-chunk's result at its end.
  return for_chunks(B, m->max_batch, [&](int b0, int nb) {
    int sizes[jimm_model::kHostSlices];
    host_slices(m, nb, sizes, src_bytes);
    if (pre && img_elems % 4) {
      // the front-end writes each slice at off * img_elems floats and needs that 16 bytes aligned (8 for 16-bit outputs): with an odd
      // image size, start every slice at a multiple of four images
      for (int i = 0; i + 1 < jimm_model::kHostSlices && sizes[i + 1] > 0; ++i) {
        const int r = sizes[i] % 4;
        sizes[i] -= r;
        sizes[i + 1] += r;
      }
    }
    bool same_layout = m->host_chain && m->host_chain_stream == s && m->host_chain_kind == kind;
    for (int i = 0; i < jimm_model::kHostSlices; ++i) same_layout = same_layout && sizes[i] == m->host_chain_sizes[i];
    if (!same_layout) {
      // earlier work on the caller's stream may still read the staging buffer in another layout: order the copies after all of it
      JIMM_CUDA_CHECK(cudaEventRecord(m->ev_start, s));
      JIMM_CUDA_CHECK(cudaStreamWaitEvent(m->copy_stream, m->ev_start, 0));
      for (int i = 0; i < jimm_model::kHostSlices; ++i) {
        // ... and after the slices of an earlier host call, which may have run on another stream
        if (m->slot_recorded[i]) JIMM_CUDA_CHECK(cudaStreamWaitEvent(m->copy_stream, m->ev_consumed[i], 0));
        m->slot_recorded[i] = false;
        m->host_chain_sizes[i] = sizes[i];
      }
      m->host_chain = true;
      m->host_chain_stream = s;
      m->host_chain_kind = kind;
    }
    int off = 0;
    for (int slot = 0; slot < jimm_model::kHostSlices; ++slot) {
      const int n = sizes[slot];
      if (n <= 0) continue;
      uint8_t* img_dst = static_cast<uint8_t*>(m->ws.in_img) + static_cast<size_t>(off) * img_elems * sizeof(float);
      uint8_t* copy_dst = pre ? m->ws.in_u8 + static_cast<size_t>(off) * src_bytes : img_dst;
      float* out_d = m->ws.out_dev + static_cast<size_t>(off) * od;
      if (m->slot_recorded[slot]) JIMM_CUDA_CHECK(cudaStreamWaitEvent(m->copy_stream, m->ev_consumed[slot], 0));
      JIMM_CUDA_CHECK(cudaMemcpyAsync(copy_dst, static_cast<const uint8_t*>(img_host) + static_cast<size_t>(b0 + off) * src_bytes, n * src_bytes,
                                      cudaMemcpyHostToDevice, m->copy_stream));
      JIMM_CUDA_CHECK(cudaEventRecord(m->ev_copied[slot], m->copy_stream));
      JIMM_CUDA_CHECK(cudaStreamWaitEvent(s, m->ev_copied[slot], 0));
      if (pre) {
        if (int rc = jimm_preproc_run(pre, copy_dst, n, Hin, Win, img_dst, tower_dtype, s)) return rc;
        // the byte staging slice is free as soon as the front-end has read it: the next call's copy runs under THIS call's tower
        // (the front-end's output slice is only rewritten by the next call's front-end, which is stream-ordered after this tower)
        JIMM_CUDA_CHECK(cudaEventRecord(m->ev_consumed[slot], s));
      }
      JIMM_TRY(exec_vision(m, img_dst, tower_dtype, n, out_d, s));
      if (!pre) JIMM_CUDA_CHECK(cudaEventRecord(m->ev_consumed[slot], s));
      m->slot_recorded[slot] = true;
      off += n;
    }
    JIMM_CUDA_CHECK(cudaMemcpyAsync(out_host + static_cast<size_t>(b0) * od, m->ws.out_dev, static_cast<size_t>(nb) * od * sizeof(float),
                                    cudaMemcpyDeviceToHost, s));
    return 0;
  });
}

int jimm_vit_forward_host(jimm_model_t* m, const void* img_host, int in_dtype, int B, float* out_host, void* stream) {
  JIMM_TRY(check_ready(m, B));
  JIMM_TRY(check_image_dtype(in_dtype));
  JIMM_TRY(check_vision(m, "jimm_vit_forward_host"));
  JIMM_TRY(set_device(m));
  return vit_forward_host_impl(m, img_host, in_dtype, B, out_host, static_cast<cudaStream_t>(stream), nullptr, 0, 0);
}

int jimm_vit_forward_host_u8(jimm_model_t* m, jimm_preproc_t* pre, const uint8_t* img_host, int B, int H, int W, float* out_host, void* stream) {
  JIMM_TRY(check_ready(m, B));
  if (!pre || !img_host || !out_host) { set_last_error("jimm_vit_forward_host_u8: null argument"); return JIMM_EINVAL; }
  JIMM_TRY(check_vision(m, "jimm_vit_forward_host_u8"));
  if (m->vis.C != 3) { set_last_error("the image front-end produces 3-channel images; the model takes %d", m->vis.C); return JIMM_EINVAL; }
  int oh = 0, ow = 0;
  if (int rc = jimm_preproc_output_size(pre, H, W, &oh, &ow)) return rc;
  if (oh != m->vis.img || ow != m->vis.img) {
    set_last_error("front-end output %dx%d for %dx%d frames does not match the model's %dx%d input", oh, ow, H, W, m->vis.img, m->vis.img);
    return JIMM_EINVAL;
  }
  JIMM_TRY(set_device(m));
  return vit_forward_host_impl(m, img_host, JIMM_F32, B, out_host, static_cast<cudaStream_t>(stream), pre, H, W);
}

int jimm_dual_forward_host(jimm_model_t* m, const void* img_host, int in_dtype, int Bi, const int32_t* ids_host, int Bt, int T,
                           float* logits_host, void* stream) {
  JIMM_TRY(check_ready(m, Bi));
  JIMM_TRY(check_text(m));
  if (Bi > m->max_batch || Bt > m->max_batch) { set_last_error("dual_forward_host: batch (%d,%d) exceeds max_batch %d", Bi, Bt, m->max_batch); return JIMM_EINVAL; }
  JIMM_TRY(check_image_dtype(in_dtype));
  JIMM_TRY(check_text_len(m, T));
  JIMM_TRY(set_device(m));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  JIMM_TRY(ensure_copy_stream(m));
  const size_t img_elems = static_cast<size_t>(m->vis.img) * m->vis.img * m->vis.C;
  const size_t img_bytes = img_elems * dtype_size(in_dtype);
  const int E = m->txt.D;
  // The (large) image copy goes to the side stream while the caller's stream takes the token ids and runs the text tower,
  // which hides it (CLIP-B/32 B=256: copy 2.8 ms, text tower 2.8 ms; measured 5.94 ms end to end against 5.85 ms device
  // resident).  Slicing the images as well only costs GEMM waves here (6.3 ms with 64+192), so it is one slice unless
  // JIMM_HOST_SLICES asks otherwise.
  // The token ids go first: H2D copies share one copy engine, so ids submitted after the images would queue behind them and
  // hold the text tower back.
  m->host_chain = false;
  JIMM_CUDA_CHECK(cudaEventRecord(m->ev_start, s));
  JIMM_CUDA_CHECK(cudaStreamWaitEvent(m->copy_stream, m->ev_start, 0));
  cudaStream_t ts = s;
  JIMM_TRY(fork_text(m, s, &ts));  // ids copy + text tower on the side stream, concurrently with the image copy and the vision tower
  JIMM_CUDA_CHECK(cudaMemcpyAsync(m->ws.in_ids, ids_host, static_cast<size_t>(Bt) * T * sizeof(int32_t), cudaMemcpyHostToDevice, ts));
  int sizes[jimm_model::kHostSlices] = {Bi, 0, 0, 0};
  if (getenv("JIMM_HOST_SLICES")) host_slices(m, Bi, sizes);
  int off = 0;
  for (int slot = 0; slot < jimm_model::kHostSlices; ++slot) {
    const int n = sizes[slot];
    if (n <= 0) continue;
    uint8_t* dst = static_cast<uint8_t*>(m->ws.in_img) + static_cast<size_t>(off) * img_elems * sizeof(float);
    JIMM_CUDA_CHECK(cudaMemcpyAsync(dst, static_cast<const uint8_t*>(img_host) + static_cast<size_t>(off) * img_bytes, n * img_bytes,
                                    cudaMemcpyHostToDevice, m->copy_stream));
    JIMM_CUDA_CHECK(cudaEventRecord(m->ev_copied[slot], m->copy_stream));
    off += n;
  }
  JIMM_TRY(exec_text(m, m->ws.in_ids, Bt, T, m->ws.emb_t, ts));
  off = 0;
  for (int slot = 0; slot < jimm_model::kHostSlices; ++slot) {
    const int n = sizes[slot];
    if (n <= 0) continue;
    const uint8_t* src = static_cast<const uint8_t*>(m->ws.in_img) + static_cast<size_t>(off) * img_elems * sizeof(float);
    JIMM_CUDA_CHECK(cudaStreamWaitEvent(s, m->ev_copied[slot], 0));
    JIMM_TRY(exec_vision(m, src, in_dtype, n, m->ws.emb_i + static_cast<size_t>(off) * E, s));
    off += n;
  }
  JIMM_TRY(join_text(m, s, ts));
  JIMM_TRY(jimm_contrastive_logits(m, m->ws.emb_i, Bi, m->ws.emb_t, Bt, m->ws.out_dev, stream));
  JIMM_CUDA_CHECK(cudaMemcpyAsync(logits_host, m->ws.out_dev, static_cast<size_t>(Bi) * Bt * sizeof(float), cudaMemcpyDeviceToHost, s));
  return 0;
}

// ---- multi-GPU contrastive head ----
int jimm_comm_init(jimm_model_t* m, int rank, int world, int max_rows_per_rank, unsigned char* handle_out) {
  JIMM_TRY(check_ready(m, 0));
  JIMM_TRY(check_text(m));
  JIMM_TRY(set_device(m));
  return comm_init(&m->comm, rank, world, max_rows_per_rank, m->txt.D, handle_out);
}
int jimm_comm_connect(jimm_model_t* m, const unsigned char* handles) {
  JIMM_TRY(check_ready(m, 0));
  JIMM_TRY(set_device(m));
  return comm_connect(&m->comm, handles);
}
int jimm_comm_contrastive_logits(jimm_model_t* m, const float* img_e, const float* txt_e, int B_local, float* logits_local, void* stream) {
  JIMM_TRY(check_ready(m, B_local));
  JIMM_TRY(set_device(m));
  return comm_contrastive_logits(&m->comm, img_e, txt_e, B_local, m->logit_scale, m->logit_bias, logits_local, static_cast<cudaStream_t>(stream));
}
int jimm_comm_status(jimm_model_t* m) {
  if (!m) { set_last_error("null model"); return JIMM_EINVAL; }
  return comm_status(&m->comm);
}
int jimm_comm_gathered(jimm_model_t* m, float** gathered, int* row_stride) {
  if (!m || !m->comm.ready) { set_last_error("comm not initialised"); return JIMM_ESTATE; }
  if (gathered) *gathered = m->comm.local_buf;
  if (row_stride) *row_stride = 2 * m->comm.E;
  return 0;
}

int jimm_profile_begin(jimm_model_t* m) {
  JIMM_TRY(check_ready(m, 0));
  m->prof_on = true;
  m->prof_used = 0;
  m->prof_flops = 0.0;
  m->prof_launches = 0;
  return 0;
}
int jimm_profile_end(jimm_model_t* m, double* gemm_ms, double* gemm_flops, long long* gemm_launches) {
  JIMM_TRY(check_ready(m, 0));
  JIMM_TRY(set_device(m));
  m->prof_on = false;
  JIMM_CUDA_CHECK(cudaDeviceSynchronize());
  double ms = 0.0;
  for (size_t i = 0; i + 1 < m->prof_used; i += 2) {
    float t = 0.f;
    JIMM_CUDA_CHECK(cudaEventElapsedTime(&t, m->prof_ev[i], m->prof_ev[i + 1]));
    ms += t;
  }
  if (gemm_ms) *gemm_ms = ms;
  if (gemm_flops) *gemm_flops = m->prof_flops;
  if (gemm_launches) *gemm_launches = m->prof_launches;
  m->prof_used = 0;
  return 0;
}

}  // extern "C"
