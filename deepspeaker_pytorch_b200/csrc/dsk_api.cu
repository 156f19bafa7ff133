// libdsk.so — host side: engine handle, TMA descriptor construction, launch plans and the C ABI
// declared in include/dsk.h.  No torch types; raw device pointers + cudaStream_t only.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <map>
#include <numeric>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/dsk.h"
#include "aam_kernels.cuh"
#include "ge2e_kernels.cuh"
#include "conv_umma.cuh"
#include "conv3x3_halo.cuh"
#include "conv1_umma.cuh"
#include "fbank_kernels.cuh"
#include "vad_kernels.cuh"
#include "augment_kernels.cuh"
#include "cluster_kernels.cuh"
#include "head_kernels.cuh"
#include "loss_kernels.cuh"
#include "metric_kernels.cuh"
#include "plda_kernels.cuh"
#include "score_kernels.cuh"
#include "simt_kernels.cuh"
#include "spectral_kernels.cuh"
#include "supcon_kernels.cuh"
#include "train_kernels.cuh"
#include "vbx_kernels.cuh"
#include "wgrad_umma.cuh"

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t e_ = (expr);                                                                        \
    if (e_ != cudaSuccess)                                                                          \
      return fail(DSK_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

#define KERNEL_CHECK()                                                                              \
  do {                                                                                              \
    cudaError_t e_ = cudaGetLastError();                                                            \
    if (e_ != cudaSuccess)                                                                          \
      return fail(DSK_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

// Launch with the programmatic-stream-serialization attribute (PDL). Only for kernels that call pdl_wait().
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 16-bit tensor map, 128B swizzle, zero OOB fill. dims/strides innermost first; strides[i] is the byte
// stride of dim i+1.
int make_tmap(CUtensorMap* out, bool bf16, const void* ptr, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, bool f32 = false, bool swizzle128 = true) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(DSK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i < rank - 1) gs[i] = strides_bytes[i];
  }
  CUresult r = fn(out, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                           : (bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16), rank,
                  const_cast<void*>(ptr), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::string d;
    for (int i = 0; i < rank; ++i) d += std::to_string(dims[i]) + "/" + std::to_string(box[i]) + " ";
    return fail(DSK_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims/box %s)", (int)r, rank,
                d.c_str());
  }
  return DSK_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute: remember (kernel, device) pairs, not kernels.
int ensure_smem_optin(const void* kern, int bytes) {
  static std::map<std::pair<const void*, int>, int> done;
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  auto key = std::make_pair(kern, dev);
  auto it = done.find(key);
  if (it != done.end() && it->second >= bytes) return DSK_OK;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done[key] = bytes;
  return DSK_OK;
}

struct ConvLaunch {
  CUtensorMap tmA, tmB, tmOut, tmRes;
  dsk::ConvParams p;
  int n_tile = 0;
  int grid = 0;
  bool bf16 = false;  // operand type the tensor maps were encoded for (launch_conv instantiates the kernel for it)
  bool out_f32 = false;
};

struct WgradLaunch {
  CUtensorMap tmG, tmX;
  dsk::WgradParams p;
  int n_tile = 0;
  int grid = 0;
};

struct HaloLaunch {
  CUtensorMap tmIn, tmW, tmOut;
  dsk::HaloParams p;
  int n_tile = 0;
  int ksize = 3;  // 3: the 3x3 tap plan (HaloPlan<1>), 5: the parity-planar 5x5 s2 plan (HaloPlan<2>)
  int grid = 0;
  int smem = 0;
};

struct LayerCfg {
  int cin, cout, ksize, stride;
};

// What every cached plan of the tensor-core cosine and Gram ops holds besides its buffers' pointers and GEMM
// descriptors: the key it was built for and its one device buffer (arena_alloc).  plan_acquire rebuilds a plan when the
// key changes; release() frees the buffer and empties the plan (empty key, no buffer, no descriptors).
template <typename Plan, int KeyLen>
struct CachedPlan {
  std::array<int, KeyLen> key{};
  uint8_t* buf = nullptr;
  cudaError_t release() {
    const cudaError_t e = cudaFree(buf);
    static_cast<Plan&>(*this) = Plan();
    return e;
  }
};

// Cached plan of the all-pairs ops for one (N, D) and anchor row range [row0, row0 + rows): E rounded to 16 bit in the
// handle's operand type, the squared norms of the rounded rows and the Gram G = E16[row0 : row0 + rows_pad] E16^T.
// Npad: N rounded up to 128; Epad: the rows of E16 the Gram's "pixel" view can read (rows >= N are zero).
struct AllpairsPlan : CachedPlan<AllpairsPlan, 4> {  // key (N, D, row0, rows)
  int Npad = 0, Epad = 0;
  uint16_t* e16 = nullptr;   // [Epad][D]
  float* gram = nullptr;     // [rows_pad][Npad]
  float* norms = nullptr;    // [Epad]
  std::vector<ConvLaunch> gemm;
};

// Cached plan of the AAM-softmax op for one (N, C, D): fp16 hi/lo operand images, fp32 GEMM outputs and workspaces, and
// the descriptors of its three GEMMs.  Np / Cp: N and C rounded up to 128 (the GEMM's pixel tile).
struct AamPlan : CachedPlan<AamPlan, 3> {  // key (N, C, D)
  int N = 0, C = 0, D = 0, Np = 0, Cp = 0;
  uint16_t *ea = nullptr, *wb = nullptr;     // forward operands: E^ [Np][3D] (A side), W^ [Cp][3D] (B side)
  uint16_t *et = nullptr, *wt = nullptr;     // backward B operands, transposed: E^T [D][3Np], W^T [D][3Cp]
  uint16_t *da = nullptr, *dt = nullptr;     // backward A operands: dcos [Np][3Cp], dcos^T [Cp][3Np] (K-sliced)
  float *nrm_e = nullptr, *nrm_w = nullptr;  // [Np], [Cp]
  float *gcos = nullptr, *dcos = nullptr;    // [Np][Cp]
  float *rinv = nullptr, *cinv = nullptr;    // [Np], [Cp]: inverse power-of-two scales of dcos's rows / columns
  int sc = 0, sn = 0;                        // K slices of the two backward GEMMs: ceil(Cp / kAamSlice), ceil(Np / ...)
  float *ge = nullptr, *gw = nullptr;        // [sc][Np][D], [sn][Cp][D]: the slices' scaled gradients w.r.t. E^ and W^
  float* row_loss = nullptr;                 // [Np]
  std::vector<ConvLaunch> fwd, ge_gemm, gw_gemm;
};

// Cached plan of the GE2E ops for one (N, P, D, row0, rows): the AAM op's hi/lo operand images and GEMMs with the P
// speaker centroids in place of the class weights - the cosines and gE^ = dcos C^ for the rows x P block of the row
// range [row0, row0 + rows), the centroid gradient gC^ = dcos^T E^ over all N rows - plus GE2E's own buffers.  Np, Rp,
// Cp: N, rows and P rounded up to 128 (the GEMM's pixel tile).
struct Ge2ePlan : CachedPlan<Ge2ePlan, 5> {  // key (N, P, D, row0, rows)
  int N = 0, P = 0, D = 0, Np = 0, Rp = 0, Cp = 0;
  int sc = 0, sn = 0;                        // K slices of gE^ and gC^: ceil(Cp / kAamSlice), ceil(Np / kAamSlice)
  float* cent = nullptr;                     // [P][D] inclusive centroids (mean of the normalised rows)
  double* nr64 = nullptr;                    // [N] fp64 row norms
  float *nrm_e = nullptr, *nrm_c = nullptr;  // [N], [P] fp32 norms of the rows and the centroids
  uint16_t *ea = nullptr, *cb = nullptr;     // forward operands: E^ of the range [Rp][3D] (A side), C^ [Cp][3D] (B side)
  uint16_t *et = nullptr, *ct = nullptr;     // backward B operands, transposed: E^T [D][3Np] (all rows), C^T [D][3Cp]
  uint16_t *da = nullptr, *dt = nullptr;     // backward A operands: the range's dcos [Rp][3Cp], dcos^T [Cp][3Np]
  float* gcos = nullptr;                     // [Rp][Cp] the range's GEMM cosines
  float* dcos = nullptr;                     // [Np][Cp] the whole batch's dcos, zero-padded
  float *rinv = nullptr, *cinv = nullptr;    // [Rp], [Cp]: inverse power-of-two scales of dcos's rows / columns
  float *ge = nullptr, *gc = nullptr;        // [sc][Rp][D], [sn][Cp][D]: the slices' scaled gradients w.r.t. E^, C^
  float* gcent = nullptr;                    // [P][D] the gradient w.r.t. the inclusive centroids
  float* own = nullptr;                      // [Rp][D] gê of the range: the target's direct term, then the whole row
  float* xg = nullptr;                       // [N][D] each row's exclusive-centroid term, shared by the other members
  float* ones = nullptr;                     // [Rp] = 1 (the un-scaling factor of gê)
  // the whole-batch ops' intermediates (only in a plan for the range (0, N)): row losses [N], the target column's dcos
  // [N] and the per-row shares of dL/dw and dL/db [2][N]; their dcos goes straight to dcos / da / rinv above
  float *row_loss = nullptr, *tdc = nullptr;
  double* part = nullptr;
  std::vector<ConvLaunch> fwd, ge_gemm, gc_gemm;
};

// Cached plan of the cosine-scoring ops for one (Nc, D, chunk): the fp16 hi/lo operand images of a row chunk of E and of
// the cohort, their norms, the chunk's fp32 cosines and the descriptors of the one GEMM.  Np: Nc rounded up to 128.
struct ScorePlan : CachedPlan<ScorePlan, 3> {  // key (Nc, D, chunk)
  int D = 0, chunk = 0, Np = 0;
  uint16_t *ea = nullptr, *cb = nullptr;     // E^ chunk [chunk][3D] (A side), cohort^ [Np][3D] (B side)
  float *nrm_e = nullptr, *nrm_c = nullptr;  // [chunk], [Np]
  float* cos = nullptr;                      // [chunk][Np]
  std::vector<ConvLaunch> gemm;
};

// One part of a plan's buffer: the pointer arena_alloc sets and the part's size in bytes (0 allowed)
struct ArenaPart {
  template <typename T>
  ArenaPart(T** p, size_t n) : slot(reinterpret_cast<void**>(p)), bytes(n) {}
  void** slot;
  size_t bytes;
};

// One cudaMalloc for all parts of a plan, each at a 256-byte aligned offset, zeroed on `s` once here (padding that no
// kernel writes stays zero).  *buf receives the allocation, which the plan's release() frees.
int arena_alloc(uint8_t** buf, std::initializer_list<ArenaPart> parts, cudaStream_t s) {
  const auto aligned = [](size_t n) { return (n + 255) / 256 * 256; };
  size_t bytes = 0;
  for (const ArenaPart& p : parts) bytes += aligned(p.bytes);
  CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(buf), bytes));
  CUDA_TRY(cudaMemsetAsync(*buf, 0, bytes, s));
  bytes = 0;
  for (const ArenaPart& p : parts) {
    *p.slot = *buf + bytes;
    bytes += aligned(p.bytes);
  }
  return DSK_OK;
}

// Make the cached plan P current for `key`.  A plan built for another key is rebuilt: `s` is synchronised (its kernels
// may still use the old buffer), P released, then build() allocates P's buffer and builds its GEMM descriptors.  A failed
// build leaves P released.  A call whose key matches never synchronises.
template <typename Plan, typename Build>
int plan_acquire(Plan& P, const decltype(Plan::key)& key, cudaStream_t s, Build build) {
  if (P.buf && P.key == key) return DSK_OK;
  CUDA_TRY(cudaStreamSynchronize(s));
  CUDA_TRY(P.release());
  if (const int rc = build()) {
    P.release();
    return rc;
  }
  P.key = key;
  return DSK_OK;
}

// conv index i = 3*stage + {0: 5x5 s2 entry conv, 1,2: 3x3 block convs}
LayerCfg layer_cfg(int i) {
  static const int ch[4] = {64, 128, 256, 512};
  const int st = i / 3, k = i % 3;
  if (k == 0) return {st == 0 ? 1 : ch[st - 1], ch[st], 5, 2};
  return {ch[st], ch[st], 3, 1};
}

}  // namespace

struct dsk_handle_s {
  int device = 0;
  bool bf16 = false;
  int num_sms = 132;
  bool weights_loaded = false;
  bool eval_packed = false;           // false after dsk_load_weights_train: only the training path's operand images are current
  int emb = 512;
  long weights_epoch = 0;             // bumped by every dsk_load_weights
  dsk_handle_s* src = nullptr;        // dsk_share_weights: the handle whose packed weights this one borrows
  long seen_epoch = -1;
  // packed parameters
  void* wpk[DSK_NUM_CONV] = {};       // 16-bit [tap][cout][cin]   (conv1: nullptr)
  void* wpk_dgrad[DSK_NUM_CONV] = {}; // 16-bit [tap][cin][cout] for the data gradient (rotated for stride 1)
  void* wpk_planar[DSK_NUM_CONV] = {}; // 16-bit [plane-major tap][cout][cin] for the halo form of the 5x5 s2 convs
  int* planar_perm = nullptr;         // device copy of the plane-major tap order
  float* conv1_w = nullptr;           // fp32 [64][25]
  uint16_t* conv1_img = nullptr;      // pre-swizzled hi/lo split operand image of conv1_umma_kernel (16 KB)
  float* scale[DSK_NUM_CONV] = {};    // folded eval BN
  std::vector<float> scale_host[DSK_NUM_CONV], bias_host[DSK_NUM_CONV];  // host copies for the halo kernels' parameters
  bool host_affine_valid = false;
  float* bias[DSK_NUM_CONV] = {};
  float* fc_wq = nullptr;             // fp32 [E][w*512+c]
  const float* fc_b = nullptr;        // borrowed (valid until next load_weights)
  dsk_weights w = {};                 // borrowed parameter pointers (train mode reads gamma/beta, updates running stats)
  // workspace
  void* ws = nullptr;
  size_t ws_bytes = 0;
  // plans keyed by (B, T)
  struct Plan {
    int B = 0, T = 0;
    std::vector<void*> act;  // 12 activation buffers (16-bit NHWC), index = conv index
    float* pooled = nullptr;
    float* fc_out = nullptr;
    float* fc_part = nullptr;  // [kFcSplit][B][E] K-slice partial sums of the fc layer
    std::vector<HaloLaunch> halo;  // index = conv index (0 unused): the 5x5 s2 and 3x3 s1 convs (padded layout)
    // The 15 launches of a forward as one CUDA graph (captured from the second call of a shape on; programmatic
    // dependent-launch edges included): one cudaGraphLaunch per forward instead of 15 kernel launches.  Only the input
    // and output pointers differ between calls: they are patched into the first / last kernel node.
    bool warm = false, graph_failed = false;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t gexec = nullptr;
    cudaGraphNode_t node_first = nullptr, node_last = nullptr;
    const float* g_x = nullptr;
    float* g_emb = nullptr;
    Plan() = default;
    Plan(const Plan&) = delete;
    Plan& operator=(const Plan&) = delete;
    Plan(Plan&& o) noexcept { *this = std::move(o); }
    Plan& operator=(Plan&& o) noexcept {
      B = o.B; T = o.T; act = std::move(o.act); pooled = o.pooled; fc_out = o.fc_out; fc_part = o.fc_part;
      halo = std::move(o.halo); warm = o.warm; graph_failed = o.graph_failed;
      graph = o.graph; gexec = o.gexec; node_first = o.node_first; node_last = o.node_last; g_x = o.g_x; g_emb = o.g_emb;
      o.graph = nullptr; o.gexec = nullptr;
      return *this;
    }
    void reset_graph() {
      if (gexec) cudaGraphExecDestroy(gexec);
      if (graph) cudaGraphDestroy(graph);
      gexec = nullptr;
      graph = nullptr;
      graph_failed = false;
    }
    ~Plan() { reset_graph(); }
  };
  std::map<std::pair<int, int>, Plan> plans;
  // training
  float* ones = nullptr;   // [512] = 1
  float* zeros = nullptr;  // [512] = 0
  float loss_scale = 0.f;  // 0 = automatic
  bool defer_stats = false;  // dsk_set_defer_running_stats: train forwards record batch statistics, the caller commits them in order
  std::vector<dsk_train_ctx_s*> ctx_pool;
  AllpairsPlan allpairs;       // cached all-pairs Gram plan (the batch-hard and tensor-core top-k ops)
  AamPlan aam;                 // cached AAM-softmax plan (its own slot: a step may use both ops)
  Ge2ePlan ge2e;               // cached GE2E plan (its own slot: a step may sum the GE2E and AAM losses)
  AamPlan supcon;              // cached supervised-contrastive plan: the AAM plan for (N, N, D), in a slot of its own
  ScorePlan score;             // cached cosine-scoring plan (its own slot: evaluation runs between training steps)
  ScorePlan search;            // cached gallery-search plan (its own slot: searches alternate with cohort statistics)
  bool use_graph = true;       // DSK_GRAPH=0: always launch the forward kernel by kernel
  bool bwd_capture_on = false; // debug: dsk_debug_set_backward_capture
  dsk_backward_capture bwd_capture = {};
  // optional per-launch timing (dsk_set_profiling): events recorded around every kernel of a forward
  int profiling = 0;  // 0 off, 1 per launch, 2 per section
  std::vector<cudaEvent_t> events;
  int n_marks = 0;
};

// Everything one train-mode forward saves for its backward (one per a/p/n call, train_triplet.py:215).
struct dsk_train_ctx_s {
  int B = 0, T = 0;                    // shape the launch descriptors are currently bound to (B <= cap)
  int cap = 0;                         // utterances the buffers were sized for
  size_t bytes = 0;
  bool in_use = false;
  bool forward_done = false;
  const float* x = nullptr;            // borrowed: the caller keeps the input alive until backward
  uint8_t* base = nullptr;             // one allocation
  float* raw[DSK_NUM_CONV] = {};       // conv outputs before BN (fp32 NHWC: BN must see unrounded values)
  void* y[DSK_NUM_CONV] = {};          // after BN (+res) + clip (16-bit NHWC)
  float* mean[DSK_NUM_CONV] = {};
  float* rstd[DSK_NUM_CONV] = {};
  float* unb[DSK_NUM_CONV] = {};       // unbiased batch variance (what the running_var update consumes)
  bool stats_pending = false;          // the forward defers the running-statistics update (set at its start, both modes):
                                       // dsk_train_ctx_commit_stats owes it
  float *pooled = nullptr, *fc_out = nullptr, *fc_part = nullptr, *inv_norm = nullptr;
  float *scale_t = nullptr, *shift_t = nullptr, *partial = nullptr, *coef = nullptr;
  float *g_fc = nullptr, *dP = nullptr, *dwacc = nullptr, *c1part = nullptr;
  float* ls = nullptr;                 // {S, 1/S}: this backward's loss scale, chosen on the device (loss_scale_kernel)
  void *gA = nullptr, *gB = nullptr, *G = nullptr, *gres = nullptr;
  ConvLaunch conv[DSK_NUM_CONV];       // forward convs 1..11 (raw output, no epilogue math)
  ConvLaunch dgrad[DSK_NUM_CONV][4];
  int n_dgrad[DSK_NUM_CONV] = {};
  WgradLaunch wgrad[DSK_NUM_CONV];
  // synchronised BatchNorm (dsk_sync_*): the staged forward or backward in progress
  int sync_dir = 0;                    // 0 none, 1 forward, 2 backward
  int sync_stage = 0;                  // forward: the layer whose records are out; backward: 12 (loss scale), then 11..0
  bool sync_fwd = false;               // this context's forward ran with synchronised statistics
  float* rec = nullptr;                // this stage's records of the B local utterances
  long long* mtot = nullptr;           // [12] global pixel count of each layer's statistics
  float* emb_out = nullptr;            // borrowed: where the forward's tail writes the embeddings
  dsk_grads grads = {};                // the backward's output pointers
};

namespace {

constexpr int kStatBlocksMax = 592;  // partial rows per 64-channel group of the BatchNorm reductions (4 blocks per SM: the
                                     // single-block finalize kernels walk these rows, ~8 us each at 1200)
// K-split count of the weight-gradient GEMM of a layer (>= 2 work items per SM), before the per-batch cap
int wgrad_ksplit_bound(int num_sms, int cout, int cin, int taps) {
  const bool swapped = cout == 64;
  const int n_tile = swapped ? 64 : (cin >= 128 ? 128 : 64);
  const int items0 = swapped ? (taps + 1) / 2 : taps * (cout / 128) * (cin / n_tile);
  return (2 * num_sms + items0 - 1) / items0;
}

// Choose the pixel box (wt, hb, nb) with wt*hb*nb == total that wastes the fewest rows.
void choose_tile(int B, int Hout, int Wout, int total, int& wt, int& hb, int& nb) {
  wt = Wout < total ? Wout : total;
  const int rows = total / wt;  // h*n rows per tile
  long best = -1;
  hb = 1;
  nb = rows;
  for (int h = rows; h >= 1; h >>= 1) {
    const int n = rows / h;
    const long padded = static_cast<long>((Hout + h - 1) / h) * h * ((B + n - 1) / n) * n;
    if (best < 0 || padded < best) {
      best = padded;
      hb = h;
      nb = n;
    }
  }
}

template <int N_TILE, bool BF16, bool OUT_F32>
int launch_conv_t(const ConvLaunch& L, cudaStream_t s) {
  auto kern = dsk::conv_umma_kernel<N_TILE, BF16, OUT_F32>;
  if (int rc = ensure_smem_optin(reinterpret_cast<const void*>(kern), dsk::ConvSmem<N_TILE>::kTotal)) return rc;
  CUDA_TRY(launch_pdl(kern, dim3(L.grid), dim3(dsk::kConvThreads), dsk::ConvSmem<N_TILE>::kTotal, s, L.tmA, L.tmB, L.tmOut, L.tmRes, L.p));
  return DSK_OK;
}

template <bool BF16, bool OUT_F32>
int launch_conv_n(const ConvLaunch& L, cudaStream_t s) {
  switch (L.n_tile) {
    case 64: return launch_conv_t<64, BF16, OUT_F32>(L, s);
    case 128: return launch_conv_t<128, BF16, OUT_F32>(L, s);
  }
  return fail(DSK_ERR_INVALID, "unsupported N tile %d", L.n_tile);
}

// Launch a conv or GEMM descriptor built by build_conv_core, on the kernel instantiated for what it was built for
int launch_conv(const ConvLaunch& L, cudaStream_t s) {
  if (L.bf16) return L.out_f32 ? launch_conv_n<true, true>(L, s) : launch_conv_n<true, false>(L, s);
  return L.out_f32 ? launch_conv_n<false, true>(L, s) : launch_conv_n<false, false>(L, s);
}

// A 5-D TMA view (dims innermost first; str[i] = byte stride of dim i+1) of a 16-bit tensor.
struct View5 {
  const void* ptr;
  uint64_t dims[5];
  uint64_t str[4];
};

// NHWC tensor as (c, w, 1, h, n)
View5 nhwc_view(const void* ptr, int B, int H, int W, int C) {
  View5 v;
  v.ptr = ptr;
  v.dims[0] = C; v.dims[1] = W; v.dims[2] = 1; v.dims[3] = H; v.dims[4] = B;
  v.str[0] = 2ull * C; v.str[1] = 2ull * W * C; v.str[2] = 2ull * W * C; v.str[3] = 2ull * H * W * C;
  return v;
}
// NHWC tensor with even H, W as parity view (pw*C + c, w/2, h&1, h/2, n): what a stride-2 conv reads / its
// data-gradient writes.
View5 nhwc_parity_view(const void* ptr, int B, int H, int W, int C) {
  View5 v;
  v.ptr = ptr;
  v.dims[0] = 2ull * C; v.dims[1] = W / 2; v.dims[2] = 2; v.dims[3] = H / 2; v.dims[4] = B;
  v.str[0] = 4ull * C; v.str[1] = 2ull * W * C; v.str[2] = 4ull * W * C; v.str[3] = 2ull * H * W * C;
  return v;
}

struct TapTable {
  int n = 0;
  int16_t c[dsk::kMaxTaps];
  int8_t w[dsk::kMaxTaps], dw[dsk::kMaxTaps], ph[dsk::kMaxTaps], dh[dsk::kMaxTaps];
  void add(int c_, int w_, int dw_, int ph_, int dh_) {
    c[n] = (int16_t)c_; w[n] = (int8_t)w_; dw[n] = (int8_t)dw_; ph[n] = (int8_t)ph_; dh[n] = (int8_t)dh_;
    ++n;
  }
};

// Generic builder: out[pixel grid Hgrid x Wgrid x B][n_out] = epilogue( sum_taps A(tap-shifted)[.., k] * Wt[tap][n_out][k] ).
int build_conv_core(const dsk_handle_s* h, ConvLaunch* L, const View5& a, const void* wpk, int k_ch, int n_out,
                    int w_slices, const View5& o, const void* res, int B, int Hgrid, int Wgrid, const TapTable& taps,
                    int flags, float clip_hi, const float* scale, const float* bias, int out_c_base, int out_ph,
                    bool out_f32 = false, bool f16 = false) {
  if (out_f32 && (flags != 0)) return fail(DSK_ERR_INVALID, "conv: fp32 output supports neither residual nor clip");
  L->out_f32 = out_f32;
  if (k_ch % 64 || n_out % 64 || k_ch < 64 || n_out < 64 || n_out > 512)
    return fail(DSK_ERR_INVALID, "conv: channel counts must be multiples of 64 and <= 512 outputs (got %d, %d)", k_ch, n_out);
  if (Wgrid > 128 || 128 % Wgrid) return fail(DSK_ERR_INVALID, "conv: output width %d must divide 128", Wgrid);
  const bool bf = h->bf16 && !f16;  // f16: fp16 operands whatever the handle's type
  L->bf16 = bf;
  dsk::ConvParams& p = L->p;
  memset(&p, 0, sizeof(p));
  choose_tile(B, Hgrid, Wgrid, 128, p.wt, p.hb, p.nb);
  p.tiles_w = (Wgrid + p.wt - 1) / p.wt;
  p.tiles_h = (Hgrid + p.hb - 1) / p.hb;
  p.tiles_n = (B + p.nb - 1) / p.nb;
  const int tiles_m = p.tiles_w * p.tiles_h * p.tiles_n;
  // N tile: minimise the number of waves over the SMs; ties go to the smaller tile (more SMs busy).  No 256-channel
  // tile: its 64 x 256 fp32 accumulator slice per consumer warpgroup does not fit the registers.
  int n_tile = 64;
  long best_waves = -1;
  for (int cand : {64, 128}) {
    if (n_out % cand) continue;
    const long tiles = static_cast<long>(tiles_m) * (n_out / cand);
    const long waves = (tiles + h->num_sms - 1) / h->num_sms;
    if (best_waves < 0 || waves < best_waves) {
      best_waves = waves;
      n_tile = cand;
    }
  }
  L->n_tile = n_tile;
  p.tiles_c = n_out / n_tile;
  p.taps = taps.n;
  p.cin_chunks = k_ch / 64;
  p.cout = n_out;
  p.flags = flags;
  p.clip_hi = clip_hi;
  p.scale = scale;
  p.bias = bias;
  p.out_c_base = out_c_base;
  p.out_ph = out_ph;
  for (int t = 0; t < taps.n; ++t) {
    p.tap_c[t] = taps.c[t];
    p.tap_w[t] = taps.w[t];
    p.tap_dw[t] = taps.dw[t];
    p.tap_ph[t] = taps.ph[t];
    p.tap_dh[t] = taps.dh[t];
  }
  const int num_tiles = tiles_m * p.tiles_c;
  L->grid = num_tiles < h->num_sms ? num_tiles : h->num_sms;
  uint32_t boxA[5] = {64, (uint32_t)p.wt, 1, (uint32_t)p.hb, (uint32_t)p.nb};
  int rc = make_tmap(&L->tmA, bf, a.ptr, 5, a.dims, a.str, boxA);
  if (rc) return rc;
  uint64_t wd[3] = {(uint64_t)k_ch, (uint64_t)n_out, (uint64_t)w_slices};
  uint64_t ws[2] = {2ull * k_ch, 2ull * k_ch * n_out};
  uint32_t wb[3] = {64, (uint32_t)n_tile, 1};
  rc = make_tmap(&L->tmB, bf, wpk, 3, wd, ws, wb);
  if (rc) return rc;
  if (out_f32) {
    uint64_t str4[4] = {o.str[0] * 2, o.str[1] * 2, o.str[2] * 2, o.str[3] * 2};  // the view was built for 2-byte elements
    uint32_t boxO[5] = {32, (uint32_t)p.wt, 1, (uint32_t)p.hb, (uint32_t)p.nb};
    rc = make_tmap(&L->tmOut, bf, o.ptr, 5, o.dims, str4, boxO, true);
    if (rc) return rc;
    return make_tmap(&L->tmRes, bf, o.ptr, 5, o.dims, str4, boxO, true);
  }
  rc = make_tmap(&L->tmOut, bf, o.ptr, 5, o.dims, o.str, boxA);
  if (rc) return rc;
  return make_tmap(&L->tmRes, bf, (flags & dsk::CONV_RESIDUAL) ? res : o.ptr, 5, o.dims, o.str, boxA);
}

// Forward conv layer on NHWC 16-bit tensors (3x3 s1 p1 or 5x5 s2 p2).
int build_conv(const dsk_handle_s* h, ConvLaunch* L, const void* in, const void* wpk, const float* scale,
               const float* bias, const void* res, void* out, int B, int Hin, int Win, int cin, int cout, int ksize,
               int stride, int flags, float clip_hi, bool out_f32 = false) {
  if (!((ksize == 3 && stride == 1) || (ksize == 5 && stride == 2)))
    return fail(DSK_ERR_INVALID, "conv: only 3x3 s1 p1 and 5x5 s2 p2 are supported (got k=%d s=%d)", ksize, stride);
  if (stride == 2 && ((Hin & 1) || (Win & 1)))
    return fail(DSK_ERR_INVALID, "conv: stride-2 input must have even H and W (got %d x %d)", Hin, Win);
  if (cin % 64 || cin < 64) return fail(DSK_ERR_INVALID, "conv: cin must be a multiple of 64 (got %d)", cin);
  const int Hout = Hin / stride, Wout = Win / stride;
  TapTable tt;
  for (int r = 0; r < ksize; ++r)
    for (int s = 0; s < ksize; ++s) {
      if (stride == 1)
        tt.add(0, r * ksize + s, s - 1, 0, r - 1);
      else  // input col = 2*w - 2 + s -> (w2 = w + floor((s-2)/2), parity = s & 1); same for rows
        tt.add((s & 1) * cin, r * ksize + s, (s - 2) >> 1, r & 1, (r - 2) >> 1);
    }
  const View5 a = stride == 1 ? nhwc_view(in, B, Hin, Win, cin) : nhwc_parity_view(in, B, Hin, Win, cin);
  const View5 o = nhwc_view(out, B, Hout, Wout, cout);
  return build_conv_core(h, L, a, wpk, cin, cout, ksize * ksize, o, res, B, Hout, Wout, tt, flags, clip_hi, scale, bias,
                         0, 0, out_f32);
}

// Data gradient of a 3x3 s1 p1 conv: g_in = conv(G, rot180(W)^T) (+ res).  G (B,H,W,cout) -> g_in (B,H,W,cin).
int build_dgrad_s1(const dsk_handle_s* h, ConvLaunch* L, const void* G, const void* wpk_dgrad, const void* res,
                   void* gin, int B, int H, int W, int cin, int cout) {
  TapTable tt;
  for (int r = 0; r < 3; ++r)
    for (int s = 0; s < 3; ++s) tt.add(0, r * 3 + s, s - 1, 0, r - 1);
  return build_conv_core(h, L, nhwc_view(G, B, H, W, cout), wpk_dgrad, cout, cin, 9, nhwc_view(gin, B, H, W, cin), res,
                         B, H, W, tt, res ? dsk::CONV_RESIDUAL : 0, 0.f, nullptr, nullptr, 0, 0);
}

// Data gradient of a 5x5 s2 p2 conv, parity class (ph, pw) of the input pixels:
//   g_in[2*h2+ph][2*w2+pw] = sum_{r = ph (mod 2), s = pw (mod 2)} G[h2 + (ph+2-r)/2][w2 + (pw+2-s)/2] . W[:, :, r, s]
// G (B,Hout,Wout,cout) -> g_in (B,2*Hout,2*Wout,cin) written through its parity view.
int build_dgrad_s2(const dsk_handle_s* h, ConvLaunch* L, const void* G, const void* wpk_dgrad, void* gin, int B,
                   int Hout, int Wout, int cin, int cout, int ph, int pw) {
  TapTable tt;
  for (int r = ph; r < 5; r += 2)
    for (int s = pw; s < 5; s += 2) tt.add(0, r * 5 + s, (pw + 2 - s) / 2, 0, (ph + 2 - r) / 2);
  return build_conv_core(h, L, nhwc_view(G, B, Hout, Wout, cout), wpk_dgrad, cout, cin, 25,
                         nhwc_parity_view(gin, B, 2 * Hout, 2 * Wout, cin), nullptr, B, Hout, Wout, tt, 0, 0.f, nullptr,
                         nullptr, pw * cin, ph);
}

// ---- weight gradient --------------------------------------------------------------------------------------------
// dW[tap][cout][cin] += G (x) X over the output pixel grid (B x Hout x Wout).  G: NHWC gradient w.r.t. the raw conv
// output; X: the conv's NHWC input (B, Hin, Win, cin).  ksize/stride as the forward conv.
int build_wgrad(const dsk_handle_s* h, WgradLaunch* L, const void* G, const void* X, int B, int Hin, int Win, int cout,
                int cin, int ksize, int stride, float* dwacc) {
  const bool bf = h->bf16;
  dsk::WgradParams& p = L->p;
  memset(&p, 0, sizeof(p));
  const int Hout = Hin / stride, Wout = Win / stride;
  if (Wout > 128 || 128 % Wout) return fail(DSK_ERR_INVALID, "wgrad: output width %d must divide 128", Wout);
  choose_tile(B, Hout, Wout, 128, p.wt, p.hb, p.nb);
  p.chunks_w = (Wout + p.wt - 1) / p.wt;
  p.chunks_h = (Hout + p.hb - 1) / p.hb;
  p.chunks_n = (B + p.nb - 1) / p.nb;
  p.taps = ksize * ksize;
  p.cout = cout;
  p.cin = cin;
  p.swapped = cout == 64 ? 1 : 0;
  if (p.swapped && cin != 64) return fail(DSK_ERR_INVALID, "wgrad: cout == 64 requires cin == 64");
  const int n_tile = p.swapped ? 64 : (cin >= 128 ? 128 : 64);
  L->n_tile = n_tile;
  p.co_tiles = p.swapped ? 1 : cout / 128;
  p.ci_tiles = p.swapped ? 1 : cin / n_tile;
  p.dw = dwacc;
  for (int r = 0; r < ksize; ++r)
    for (int s = 0; s < ksize; ++s) {
      const int t = r * ksize + s;
      if (stride == 1) {
        p.tap_c[t] = 0;
        p.tap_dw[t] = (int8_t)(s - 1);
        p.tap_ph[t] = 0;
        p.tap_dh[t] = (int8_t)(r - 1);
      } else {
        p.tap_c[t] = (int16_t)((s & 1) * cin);
        p.tap_dw[t] = (int8_t)((s - 2) >> 1);
        p.tap_ph[t] = (int8_t)(r & 1);
        p.tap_dh[t] = (int8_t)((r - 2) >> 1);
      }
    }
  const int total_chunks = p.chunks_w * p.chunks_h * p.chunks_n;
  const int items0 = (p.swapped ? (p.taps + 1) / 2 : p.taps) * p.co_tiles * p.ci_tiles;
  int ksplit = (2 * h->num_sms + items0 - 1) / items0;
  const int max_split = total_chunks / 4 > 0 ? total_chunks / 4 : 1;
  if (ksplit > max_split) ksplit = max_split;
  if (ksplit < 1) ksplit = 1;
  p.ksplit = ksplit;
  p.slice_elems = static_cast<long>(p.taps) * cout * cin;
  const int items = items0 * ksplit;
  L->grid = items < h->num_sms ? items : h->num_sms;
  const View5 g = nhwc_view(G, B, Hout, Wout, cout);
  const View5 x = stride == 1 ? nhwc_view(X, B, Hin, Win, cin) : nhwc_parity_view(X, B, Hin, Win, cin);
  uint32_t box[5] = {64, (uint32_t)p.wt, 1, (uint32_t)p.hb, (uint32_t)p.nb};
  int rc = make_tmap(&L->tmG, bf, g.ptr, 5, g.dims, g.str, box);
  if (rc) return rc;
  return make_tmap(&L->tmX, bf, x.ptr, 5, x.dims, x.str, box);
}

template <int N_TILE, bool BF16>
int launch_wgrad_t(const WgradLaunch& L, cudaStream_t s) {
  auto kern = dsk::wgrad_umma_kernel<N_TILE, BF16>;
  if (int rc = ensure_smem_optin(reinterpret_cast<const void*>(kern), dsk::WgradSmem<N_TILE>::kTotal)) return rc;
  kern<<<L.grid, dsk::kWgradThreads, dsk::WgradSmem<N_TILE>::kTotal, s>>>(L.tmG, L.tmX, L.p);
  KERNEL_CHECK();
  return DSK_OK;
}

int launch_wgrad(const dsk_handle_s* h, const WgradLaunch& L, cudaStream_t s) {
  if (h->bf16) {
    switch (L.n_tile) {
      case 64: return launch_wgrad_t<64, true>(L, s);
      case 128: return launch_wgrad_t<128, true>(L, s);
    }
  } else {
    switch (L.n_tile) {
      case 64: return launch_wgrad_t<64, false>(L, s);
      case 128: return launch_wgrad_t<128, false>(L, s);
    }
  }
  return fail(DSK_ERR_INVALID, "unsupported wgrad N tile %d", L.n_tile);
}

// ---- zero-padded NHWC layout of the eval forward (see conv3x3_halo.cuh) ---------------------------------------------
// rows: 1 leading pad + N*(H+1) (each image followed by one pad row) + slack for the last tile's halo / overrun
long padded_positions(int N, int H, int W) {
  const long rows = 1 + static_cast<long>(N) * (H + 1) + (128 + W + 3 + W) / (W + 1) + 2;
  return rows * (W + 1);
}
size_t padded_bytes(int N, int H, int W, int C) { return static_cast<size_t>(padded_positions(N, H, W)) * C * 2; }

// The GEMMs of the cached plans: O (rows_pad x n_total fp32) = A (rows_pad x K) B^T (n_total x K), both 16-bit row-major
// images (f16: fp16 operands whatever the handle's type).  Rows of A are the "pixels" (W = 128, H = rows_pad / 128), rows
// of B the "output channels", <= 512 per launch; one tap.
int build_gemm(const dsk_handle_s* h, std::vector<ConvLaunch>* out, const uint16_t* A, int rows_pad, const uint16_t* B,
               int n_total, int K, float* O, bool f16) {
  TapTable tt;
  tt.add(0, 0, 0, 0, 0);
  for (int c0 = 0; c0 < n_total; c0 += 512) {
    ConvLaunch L;
    const int rc = build_conv_core(h, &L, nhwc_view(A, 1, rows_pad / 128, 128, K), B + static_cast<size_t>(c0) * K, K,
                                   n_total - c0 < 512 ? n_total - c0 : 512, 1, nhwc_view(O, 1, rows_pad / 128, 128, n_total),
                                   nullptr, 1, rows_pad / 128, 128, tt, 0, 0.f, nullptr, nullptr, c0, 0, true, f16);
    if (rc) return rc;
    out->push_back(L);
  }
  return DSK_OK;
}

// A backward product of the cosine ops over a K dimension of Kp (a multiple of 128) with fp16 operands, split K
// deterministically: one build_gemm per kAamSlice-wide K slice, slice k of the K-sliced A image ([rows_pad][3w] at
// k kAamSlice 3 rows_pad) times slice k of the transposed image Bt ([D][3w]) into its own output O + k rows_pad D.
int build_sliced_gemm(const dsk_handle_s* h, std::vector<ConvLaunch>* out, const uint16_t* A, int rows_pad,
                      const uint16_t* Bt, int D, int Kp, float* O) {
  const size_t ks = dsk::kAamSlice;
  for (int k = 0; k * dsk::kAamSlice < Kp; ++k) {
    const int w = Kp - k * dsk::kAamSlice < dsk::kAamSlice ? Kp - k * dsk::kAamSlice : dsk::kAamSlice;
    if (int rc = build_gemm(h, out, A + k * ks * 3 * rows_pad, rows_pad, Bt + k * ks * 3 * D, D, 3 * w,
                            O + static_cast<size_t>(k) * rows_pad * D, true))
      return rc;
  }
  return DSK_OK;
}

// Packed tap order of the parity-planar 5x5 s2 conv: plane (ph, pw) major, then r, then s. slot -> original r*5+s.
void planar_tap_order(int* perm /*[25]*/) {
  int n = 0;
  for (int ph = 0; ph < 2; ++ph)
    for (int pw = 0; pw < 2; ++pw)
      for (int r = ph; r < 5; r += 2)
        for (int s = pw; s < 5; s += 2) perm[n++] = r * 5 + s;
}

// device per-channel affine -> host vectors (plan build / single-op entry points only: synchronises the device)
int fetch_affine(const float* scale_d, const float* bias_d, int n, std::vector<float>* sc, std::vector<float>* bi) {
  sc->assign(n, 1.0f);
  bi->assign(n, 0.0f);
  CUDA_TRY(cudaDeviceSynchronize());
  if (scale_d) CUDA_TRY(cudaMemcpy(sc->data(), scale_d, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (bias_d) CUDA_TRY(cudaMemcpy(bi->data(), bias_d, n * sizeof(float), cudaMemcpyDeviceToHost));
  return DSK_OK;
}

// Halo-reuse conv on the padded layout (conv3x3_halo.cuh).  ksize 3 (stride 1, C -> C, input = standard padded
// layout of the same geometry) or ksize 5 (stride 2, input = parity-planar padded layout at the OUTPUT geometry).
// (N, H, W) is the OUTPUT geometry.  out_planar: write the output parity-planar (it feeds a stride-2 conv).
int build_halo(const dsk_handle_s* h, HaloLaunch* L, const void* in, const void* wpk, const float* scale_host,
               const float* bias_host, const void* res, void* out, int N, int H, int W, int cin, int cout, int ksize,
               int flags, float clip_hi, int out_planar) {
  if (cin % 64 || cin < 64 || cout % 64 || cout < 64 || cout > 512)
    return fail(DSK_ERR_INVALID, "halo conv: channel counts must be multiples of 64 (got %d -> %d)", cin, cout);
  if (ksize != 3 && ksize != 5) return fail(DSK_ERR_INVALID, "halo conv: ksize must be 3 or 5");
  if (ksize == 3 && cin != cout) return fail(DSK_ERR_INVALID, "halo conv: the 3x3 form needs cin == cout");
  if (W > 34) return fail(DSK_ERR_INVALID, "halo conv: W must be <= 34 (got %d)", W);
  if (out_planar && ((H & 1) || (W & 1))) return fail(DSK_ERR_INVALID, "halo conv: planar output needs even H, W");
  if (out_planar && ksize != 3) return fail(DSK_ERR_INVALID, "halo conv: planar output is written by the 3x3 form only");
  const bool bf = h->bf16;
  dsk::HaloParams& p = L->p;
  memset(&p, 0, sizeof(p));
  p.W = W; p.H = H; p.N = N;
  p.q_begin = W + 1;
  const long q_end = static_cast<long>(N) * (H + 1) * (W + 1);   // one past the last real pixel position
  const int n_tile = cout == 64 ? 64 : 128;
  const int tm = dsk::HaloSmem<128>::kTileRows;  // positions per tile
  p.tiles_m = static_cast<int>((q_end - p.q_begin + tm - 1) / tm);
  const int tpb = 3;  // taps per weight box
  L->n_tile = n_tile;
  L->ksize = ksize;
  p.tiles_c = cout / n_tile;
  p.chunks = cin / 64;
  p.cout = cout;
  p.flags = flags;
  p.clip_hi = clip_hi;
  for (int i = 0; i < cout; ++i) {
    p.scale_c[i] = scale_host ? scale_host[i] : 1.0f;
    p.bias_c[i] = bias_host ? bias_host[i] : 0.0f;
  }
  p.pitch_magic = static_cast<unsigned long long>((static_cast<unsigned __int128>(1) << 64) / static_cast<unsigned>(W + 1)) + 1ull;
  p.img_magic = static_cast<unsigned long long>((static_cast<unsigned __int128>(1) << 64) / static_cast<unsigned>(H + 1)) + 1ull;
  const long npos = padded_positions(N, H, W);
  // the kernel's positions, tile indices and TMA row coordinates are 32-bit signed (four planes for the 5x5 input)
  if (npos * (ksize == 5 ? 4 : 1) >= (1l << 31))
    return fail(DSK_ERR_INVALID, "halo conv: %ld padded positions exceed 32-bit indexing (N %d, H %d, W %d)", npos, N, H, W);
  int ntaps_total;
  if (ksize == 3) {
    ntaps_total = 9;
    p.nboxes = 9 / tpb;
    p.plane_positions = 0;
    for (int b = 0; b < p.nboxes; ++b) {
      p.box_plane[b] = 0;
      p.box_first[b] = b == 0;
      p.box_wtap[b] = (int16_t)(tpb * b);
    }
  } else {
    ntaps_total = 25;
    p.plane_positions = static_cast<int>(npos);
    int slot = 0, nb = 0;
    for (int pl = 0; pl < 4; ++pl) {
      const int ph = pl >> 1, pw = pl & 1;
      const int cnt = (ph ? 2 : 3) * (pw ? 2 : 3);
      for (int t0 = 0; t0 < cnt; t0 += tpb, ++nb) {
        p.box_plane[nb] = (int8_t)pl;
        p.box_first[nb] = t0 == 0;
        p.box_wtap[nb] = (int16_t)(slot + t0);
      }
      slot += cnt;
    }
    p.nboxes = nb;  // 3 + 2 + 2 + 2 = 9 three-tap boxes
  }
  // all weight boxes of a CTA fit the B ring and every tile of the CTA uses the same ones: load them once
  p.b_resident = (p.chunks == 1 && p.tiles_c == 1 && p.nboxes <= 3 && n_tile == 64) ? 1 : 0;
  p.res_ptr = (flags & dsk::CONV_RESIDUAL) ? static_cast<const uint16_t*>(res) : nullptr;
  p.out_planar = out_planar;
  if (out_planar) {
    p.out_ptr = static_cast<uint16_t*>(out);
    p.out_plane_positions = static_cast<int>(padded_positions(N, H / 2, W / 2));
    p.out_C = cout;
  }
  // shared-memory carve: two output staging tiles; the residual is read from global memory (HaloParams::res_ptr), so
  // everything else goes to the operand rings - weight boxes, the latency-critical stream, first (48 KB each at
  // N_TILE = 128): the deepest ring that fits in 227 KB
  {
    const int halo_rows = tm + 2 * W + 4;
    p.a_stage_bytes = (halo_rows * 128 + 1023) / 1024 * 1024;
    const int b_bytes = tpb * n_tile * 128;
    const int fixed = dsk::HaloSmem<128>::kFixedBytes;  // the same for every tile width
    const int limit = 227 * 1024;
    p.a_stages = n_tile == 64 ? 3 : 2;
    p.stg_bufs = 2;
    int nb = (limit - fixed - p.a_stages * p.a_stage_bytes - p.stg_bufs * 16384) / b_bytes;
    p.b_stages = nb > dsk::kHaloMaxStages ? dsk::kHaloMaxStages : nb;
    if (p.b_resident) p.b_stages = 3;
    if (p.b_stages < 2) return fail(DSK_ERR_INVALID, "halo conv: shared memory does not fit");
    L->smem = p.a_stages * p.a_stage_bytes + p.b_stages * b_bytes + p.stg_bufs * 16384 + fixed;
  }
  const int num_tiles = p.tiles_m * p.tiles_c;
  L->grid = num_tiles < h->num_sms ? num_tiles : h->num_sms;
  const uint64_t in_pos = static_cast<uint64_t>(npos) * (ksize == 5 ? 4 : 1);
  uint64_t idims[2] = {(uint64_t)cin, in_pos};
  uint64_t istr[1] = {2ull * cin};
  uint32_t box_in[2] = {64, (uint32_t)(tm + 2 * W + 4)};
  int rc = make_tmap(&L->tmIn, bf, in, 2, idims, istr, box_in);
  if (rc) return rc;
  uint64_t wd[3] = {(uint64_t)cin, (uint64_t)cout, (uint64_t)ntaps_total};
  uint64_t ws[2] = {2ull * cin, 2ull * cin * cout};
  uint32_t wb[3] = {64, (uint32_t)n_tile, (uint32_t)tpb};
  rc = make_tmap(&L->tmW, bf, wpk, 3, wd, ws, wb);
  if (rc) return rc;
  // output: standard padded layout of the output geometry (with a planar output the map is unused but must be valid:
  // point it at the residual or the input)
  uint64_t odims[2] = {(uint64_t)cout, (uint64_t)npos};
  uint64_t ostr[1] = {2ull * cout};
  uint32_t box_out[2] = {64, (uint32_t)tm};
  const void* out_map = out_planar ? ((flags & dsk::CONV_RESIDUAL) ? res : in) : out;
  return make_tmap(&L->tmOut, bf, out_map, 2, odims, ostr, box_out);
}

template <int N_TILE, bool BF16, int KIND>
int launch_halo_t(const HaloLaunch& L, cudaStream_t s) {
  auto kern = dsk::conv3x3_halo_kernel<N_TILE, BF16, KIND>;
  if (int rc = ensure_smem_optin(reinterpret_cast<const void*>(kern), 227 * 1024)) return rc;
  CUDA_TRY(launch_pdl(kern, dim3(L.grid), dim3(dsk::kHaloThreads), L.smem, s, L.tmIn, L.tmW, L.tmOut, L.p));
  return DSK_OK;
}

// one instantiation per (tile width, operand type, tap plan): each carries only the code it runs
template <int N_TILE>
int launch_halo_v(const dsk_handle_s* h, const HaloLaunch& L, cudaStream_t s) {
  const bool k5 = L.ksize == 5;
  if (h->bf16) return k5 ? launch_halo_t<N_TILE, true, 2>(L, s) : launch_halo_t<N_TILE, true, 1>(L, s);
  return k5 ? launch_halo_t<N_TILE, false, 2>(L, s) : launch_halo_t<N_TILE, false, 1>(L, s);
}

int launch_halo(const dsk_handle_s* h, const HaloLaunch& L, cudaStream_t s) {
  return L.n_tile == 64 ? launch_halo_v<64>(h, L, s) : launch_halo_v<128>(h, L, s);
}

int check_handle(dsk_handle h) {
  if (!h) return fail(DSK_ERR_INVALID, "null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  return DSK_OK;
}

template <typename T>
int dev_alloc(T** p, size_t n) {
  CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  return DSK_OK;
}

// per-utterance element counts of the 12 activation tensors at time length T
void act_shape(int i, int T, int& H, int& W, int& C) {
  const int st = i / 3;
  H = T >> (st + 1);
  W = 64 >> (st + 1);
  C = 64 << st;
}

int get_plan(dsk_handle h, int B, int T, cudaStream_t s, dsk_handle_s::Plan** out) {
  auto key = std::make_pair(B, T);
  auto it = h->plans.find(key);
  if (it != h->plans.end()) {
    *out = &it->second;
    return DSK_OK;
  }
  // A new shape: (re)allocate the workspace for it alone and rebuild all plans lazily.
  // Eval activations use the zero-padded NHWC layout (conv3x3_halo.cuh); pads are zeroed here once and are
  // never overwritten with anything but zeros.
  size_t bytes = 0;
  size_t off[DSK_NUM_CONV];
  for (int i = 0; i < DSK_NUM_CONV; ++i) {
    int H, W, C;
    act_shape(i, T, H, W, C);
    off[i] = bytes;
    // a block output that feeds a stride-2 conv (i = 2, 5, 8) is stored parity-planar (4 planes at half res)
    const bool planar = (i % 3 == 2) && i < DSK_NUM_CONV - 1;
    const size_t b = planar ? 4 * padded_bytes(B, H / 2, W / 2, C) : padded_bytes(B, H, W, C);
    bytes += ((b + 1023) / 1024) * 1024;
  }
  const size_t act_bytes = bytes;
  const size_t off_pooled = bytes;
  bytes += static_cast<size_t>(B) * 2048 * 4;
  const size_t off_fc = bytes;
  bytes += static_cast<size_t>(B) * h->emb * 4;
  const size_t off_fc_part = bytes;
  bytes += static_cast<size_t>(dsk::kFcSplit) * B * h->emb * 4;
  if (bytes > h->ws_bytes) {
    // drop cached plans: their descriptors point into the old workspace
    h->plans.clear();
    if (h->ws) CUDA_TRY(cudaFree(h->ws));
    h->ws = nullptr;
    h->ws_bytes = 0;
    CUDA_TRY(cudaMalloc(&h->ws, bytes));
    h->ws_bytes = bytes;
  } else {
    // the workspace is shared by all shapes, but the pad positions differ per shape: plans of other shapes would
    // find non-zero pads after this one ran, so only one shape is cached at a time
    h->plans.clear();
  }
  // Ordered on the caller's stream: after the forwards this lane still has in flight on it (they read / write the old
  // shape's pads) and before the new shape's first kernel.  (A NULL-stream memset would be unordered against the
  // non-blocking streams PyTorch hands out.)
  CUDA_TRY(cudaMemsetAsync(h->ws, 0, act_bytes, s));
  dsk_handle_s::Plan pl;
  pl.B = B;
  pl.T = T;
  pl.act.resize(DSK_NUM_CONV);
  uint8_t* base = static_cast<uint8_t*>(h->ws);
  for (int i = 0; i < DSK_NUM_CONV; ++i) pl.act[i] = base + off[i];
  pl.pooled = reinterpret_cast<float*>(base + off_pooled);
  pl.fc_out = reinterpret_cast<float*>(base + off_fc);
  pl.fc_part = reinterpret_cast<float*>(base + off_fc_part);
  pl.halo.resize(DSK_NUM_CONV);
  if (!h->host_affine_valid) {  // once per weight load: host copy of the folded BN affine for the kernel parameters
    for (int i = 1; i < DSK_NUM_CONV; ++i) {
      int rc2 = fetch_affine(h->scale[i], h->bias[i], layer_cfg(i).cout, &h->scale_host[i], &h->bias_host[i]);
      if (rc2) return rc2;
    }
    h->host_affine_valid = true;
  }
  for (int i = 1; i < DSK_NUM_CONV; ++i) {
    const LayerCfg c = layer_cfg(i);
    const int k = i % 3;
    int Ho, Wo, Co;
    act_shape(i, T, Ho, Wo, Co);
    int rc;
    if (k == 0) {
      rc = build_halo(h, &pl.halo[i], pl.act[i - 1], h->wpk_planar[i], h->scale_host[i].data(), h->bias_host[i].data(), nullptr, pl.act[i], B, Ho, Wo,
                      c.cin, c.cout, 5, dsk::CONV_CLIP, 20.0f, 0);
    } else {
      const void* res = (k == 2) ? pl.act[i - 2] : nullptr;  // block output adds the block input
      const int flags = dsk::CONV_CLIP | (k == 2 ? dsk::CONV_RESIDUAL : 0);
      const int out_planar = (k == 2 && i < DSK_NUM_CONV - 1) ? 1 : 0;
      rc = build_halo(h, &pl.halo[i], pl.act[i - 1], h->wpk[i], h->scale_host[i].data(), h->bias_host[i].data(), res, pl.act[i], B, Ho, Wo, c.cin,
                      c.cout, 3, flags, 20.0f, out_planar);
    }
    if (rc) return rc;
  }
  auto ins = h->plans.emplace(key, std::move(pl));
  *out = &ins.first->second;
  return DSK_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char* dsk_last_error(void) { return g_err.c_str(); }
int32_t dsk_version(void) { return 100; }

int32_t dsk_create(dsk_handle* out, int32_t device, int32_t operand) {
  if (!out) return fail(DSK_ERR_INVALID, "dsk_create: out is null");
  if (operand != DSK_F16 && operand != DSK_BF16) return fail(DSK_ERR_INVALID, "dsk_create: bad operand type %d", operand);
  CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(DSK_ERR_ARCH, "dsk_create: device %d is sm_%d%d; this library contains sm_90a code only", device,
                prop.major, prop.minor);
  dsk_handle h = new dsk_handle_s();
  h->device = device;
  h->bf16 = operand == DSK_BF16;
  h->num_sms = prop.multiProcessorCount;
  {
    const char* e = getenv("DSK_GRAPH");
    h->use_graph = !(e && e[0] == '0');
  }
  {
    std::vector<float> one(512, 1.0f);
    if (cudaMalloc(reinterpret_cast<void**>(&h->ones), 512 * 4) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&h->zeros), 512 * 4) != cudaSuccess ||
        cudaMemcpy(h->ones, one.data(), 512 * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemset(h->zeros, 0, 512 * 4) != cudaSuccess) {
      delete h;
      return fail(DSK_ERR_CUDA, "dsk_create: device allocation failed");
    }
  }
  *out = h;
  return DSK_OK;
}

int32_t dsk_destroy(dsk_handle h) {
  if (!h) return DSK_OK;
  cudaSetDevice(h->device);
  if (!h->src) {  // a borrower's parameter pointers belong to its source
    for (int i = 0; i < DSK_NUM_CONV; ++i) {
      cudaFree(h->wpk[i]);
      cudaFree(h->wpk_dgrad[i]);
      cudaFree(h->wpk_planar[i]);
      cudaFree(h->scale[i]);
      cudaFree(h->bias[i]);
    }
    cudaFree(h->conv1_w);
    cudaFree(h->conv1_img);
    cudaFree(h->planar_perm);
    cudaFree(h->fc_wq);
  }
  cudaFree(h->ws);
  h->allpairs.release();
  h->aam.release();
  h->ge2e.release();
  h->supcon.release();
  h->score.release();
  h->search.release();
  cudaFree(h->ones);
  cudaFree(h->zeros);
  for (dsk_train_ctx_s* c : h->ctx_pool) {
    cudaFree(c->base);
    delete c;
  }
  for (cudaEvent_t e : h->events) cudaEventDestroy(e);
  delete h;
  return DSK_OK;
}

namespace {
int load_weights_impl(dsk_handle h, const dsk_weights* w, void* stream, bool train_only);
}
int32_t dsk_load_weights(dsk_handle h, const dsk_weights* w, void* stream) { return load_weights_impl(h, w, stream, false); }
int32_t dsk_load_weights_train(dsk_handle h, const dsk_weights* w, void* stream) { return load_weights_impl(h, w, stream, true); }

namespace {
int load_weights_impl(dsk_handle h, const dsk_weights* w, void* stream, bool train_only) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!w) return fail(DSK_ERR_INVALID, "dsk_load_weights: null weights");
  if (w->embedding_size <= 0 || w->embedding_size % 64)
    return fail(DSK_ERR_INVALID, "dsk_load_weights: embedding_size must be a positive multiple of 64");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->src) return fail(DSK_ERR_STATE, "dsk_load_weights: this handle borrows its weights (dsk_share_weights)");
  if (h->weights_loaded && h->emb != w->embedding_size) return fail(DSK_ERR_INVALID, "embedding_size changed");
  ++h->weights_epoch;
  // eval plans carry the folded BN affine in their kernel parameters (and their graphs borrowed parameter pointers)
  h->plans.clear();
  h->host_affine_valid = false;
  h->emb = w->embedding_size;
  h->eval_packed = !train_only;
  dsk::PackTrainTable tbl{};
  int nblk = 0;
  for (int i = 0; i < DSK_NUM_CONV; ++i) {
    const LayerCfg c = layer_cfg(i);
    const int taps = c.ksize * c.ksize;
    const long n = static_cast<long>(c.cout) * c.cin * taps;
    if (!w->conv_w[i] || !w->bn_gamma[i] || !w->bn_beta[i] || !w->bn_running_mean[i] || !w->bn_running_var[i])
      return fail(DSK_ERR_INVALID, "dsk_load_weights: null parameter pointer for conv/bn %d", i);
    if (train_only) {
      // the training path reads only wpk / wpk_dgrad / conv1_w / fc_wq: one table-driven launch below
      tbl.w[i] = w->conv_w[i];
      if (i == 0) {
        if (!h->conv1_w) {
          rc = dev_alloc(&h->conv1_w, 64 * 25);
          if (rc) return rc;
        }
        tbl.conv1_dst = h->conv1_w;
        continue;
      }
      if (!h->wpk[i]) {
        CUDA_TRY(cudaMalloc(&h->wpk[i], n * 2));
        CUDA_TRY(cudaMalloc(&h->wpk_dgrad[i], n * 2));
      }
      tbl.fwd[i] = static_cast<uint16_t*>(h->wpk[i]);
      tbl.dgrad[i] = static_cast<uint16_t*>(h->wpk_dgrad[i]);
      tbl.cout[i] = c.cout, tbl.cin[i] = c.cin, tbl.taps[i] = taps, tbl.rotate[i] = c.stride == 1;
      tbl.first_block[i] = nblk;
      nblk += (c.cout / dsk::kPackCo) * (c.cin / dsk::kPackCi);
      tbl.first_block[i + 1] = nblk;
      continue;
    }
    if (!h->scale[i]) {
      rc = dev_alloc(&h->scale[i], c.cout);
      if (rc) return rc;
      rc = dev_alloc(&h->bias[i], c.cout);
      if (rc) return rc;
    }
    dsk::bn_fold_kernel<<<(c.cout + 127) / 128, 128, 0, s>>>(w->bn_gamma[i], w->bn_beta[i], w->bn_running_mean[i],
                                                             w->bn_running_var[i], 1e-5f, h->scale[i], h->bias[i],
                                                             c.cout);
    KERNEL_CHECK();
    if (i == 0) {
      if (!h->conv1_w) {
        rc = dev_alloc(&h->conv1_w, 64 * 25);
        if (rc) return rc;
      }
      CUDA_TRY(cudaMemcpyAsync(h->conv1_w, w->conv_w[0], 64 * 25 * sizeof(float), cudaMemcpyDeviceToDevice, s));
      if (!h->conv1_img) CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&h->conv1_img), dsk::kConv1ImgHalfs * 2));
      if (h->bf16) dsk::pack_conv1_umma_kernel<true><<<32, 256, 0, s>>>(h->conv1_w, h->conv1_img);
      else dsk::pack_conv1_umma_kernel<false><<<32, 256, 0, s>>>(h->conv1_w, h->conv1_img);
      KERNEL_CHECK();
      continue;
    }
    if (!h->wpk[i]) {
      CUDA_TRY(cudaMalloc(&h->wpk[i], n * 2));
      CUDA_TRY(cudaMalloc(&h->wpk_dgrad[i], n * 2));
    }
    const int blocks = static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    if (h->bf16) {
      dsk::pack_conv_weight_kernel<true><<<blocks, 256, 0, s>>>(w->conv_w[i], (uint16_t*)h->wpk[i], c.cout, c.cin, taps);
      dsk::pack_conv_weight_dgrad_kernel<true><<<blocks, 256, 0, s>>>(w->conv_w[i], (uint16_t*)h->wpk_dgrad[i], c.cout, c.cin, taps, c.stride == 1);
    } else {
      dsk::pack_conv_weight_kernel<false><<<blocks, 256, 0, s>>>(w->conv_w[i], (uint16_t*)h->wpk[i], c.cout, c.cin, taps);
      dsk::pack_conv_weight_dgrad_kernel<false><<<blocks, 256, 0, s>>>(w->conv_w[i], (uint16_t*)h->wpk_dgrad[i], c.cout, c.cin, taps, c.stride == 1);
    }
    KERNEL_CHECK();
    if (c.stride == 2) {
      if (!h->planar_perm) {
        int perm[25];
        planar_tap_order(perm);
        rc = dev_alloc(&h->planar_perm, 25);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpy(h->planar_perm, perm, sizeof(perm), cudaMemcpyHostToDevice));
      }
      if (!h->wpk_planar[i]) CUDA_TRY(cudaMalloc(&h->wpk_planar[i], n * 2));
      if (h->bf16)
        dsk::pack_conv_weight_perm_kernel<true><<<blocks, 256, 0, s>>>(w->conv_w[i], (uint16_t*)h->wpk_planar[i], c.cout, c.cin, taps, h->planar_perm);
      else
        dsk::pack_conv_weight_perm_kernel<false><<<blocks, 256, 0, s>>>(w->conv_w[i], (uint16_t*)h->wpk_planar[i], c.cout, c.cin, taps, h->planar_perm);
      KERNEL_CHECK();
    }
  }
  if (train_only) {
    if (h->bf16) dsk::pack_train_weights_kernel<true><<<nblk + 1, 256, 0, s>>>(tbl);
    else dsk::pack_train_weights_kernel<false><<<nblk + 1, 256, 0, s>>>(tbl);
    KERNEL_CHECK();
  }
  if (!w->fc_w || !w->fc_b) return fail(DSK_ERR_INVALID, "dsk_load_weights: null fc pointer");
  if (!h->fc_wq) {
    rc = dev_alloc(&h->fc_wq, static_cast<size_t>(h->emb) * 2048);
    if (rc) return rc;
  }
  dsk::pack_fc_weight_kernel<<<1024, 256, 0, s>>>(w->fc_w, h->fc_wq, h->emb, 512, 4);
  KERNEL_CHECK();
  h->fc_b = w->fc_b;
  h->w = *w;
  h->weights_loaded = true;
  return DSK_OK;
}
}  // namespace

int32_t dsk_share_weights(dsk_handle h, dsk_handle src) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!src || src == h || src->src) return fail(DSK_ERR_INVALID, "dsk_share_weights: bad source handle");
  if (h->weights_loaded && !h->src) return fail(DSK_ERR_STATE, "dsk_share_weights: the handle already owns weights");
  if (h->device != src->device || h->bf16 != src->bf16)
    return fail(DSK_ERR_INVALID, "dsk_share_weights: device / operand type differ from the source");
  h->src = src;
  h->seen_epoch = -1;
  return DSK_OK;
}

namespace {

// a borrowing handle picks up the source's current parameter pointers; its plans (which bake the folded BN affine
// into kernel parameters) are rebuilt.  Plan building synchronises the device (fetch_affine), which also orders this
// handle's stream after the source's repack kernels.
void adopt_shared_weights(dsk_handle h) {
  dsk_handle_s* s = h->src;
  if (!s || h->seen_epoch == s->weights_epoch) return;
  for (int i = 0; i < DSK_NUM_CONV; ++i) {
    h->wpk[i] = s->wpk[i];
    h->wpk_dgrad[i] = s->wpk_dgrad[i];
    h->wpk_planar[i] = s->wpk_planar[i];
    h->scale[i] = s->scale[i];
    h->bias[i] = s->bias[i];
  }
  h->conv1_w = s->conv1_w;
  h->conv1_img = s->conv1_img;
  h->planar_perm = s->planar_perm;
  h->fc_wq = s->fc_wq;
  h->fc_b = s->fc_b;
  h->w = s->w;
  h->emb = s->emb;
  h->weights_loaded = s->weights_loaded;
  h->eval_packed = s->eval_packed;
  h->plans.clear();
  h->host_affine_valid = false;
  h->seen_epoch = s->weights_epoch;
}

// conv1: tensor map over the input batch (64 bins, T frames, B utterances; box = the 11 frames x 64 bins of one tile,
// out-of-bounds rows zero) and the persistent grid (<= 4 CTAs per SM, the same number of tiles for every CTA)
int conv1_launch_geometry(const dsk_handle_s* h, const float* x, int B, int T, CUtensorMap* tm, int* grid, int* n_tiles) {
  const uint64_t dims[3] = {64, static_cast<uint64_t>(T), static_cast<uint64_t>(B)};
  const uint64_t strides[2] = {64 * sizeof(float), static_cast<uint64_t>(T) * 64 * sizeof(float)};
  const uint32_t box[3] = {64, static_cast<uint32_t>(dsk::kConv1PatchRows), 1};
  int rc = make_tmap(tm, false, x, 3, dims, strides, box, /*f32=*/true, /*swizzle128=*/false);
  if (rc) return rc;
  const int nt = B * (T / 2 / 4);
  const int per_cta = (nt + 4 * h->num_sms - 1) / (4 * h->num_sms);
  *n_tiles = nt;
  *grid = (nt + per_cta - 1) / per_cta;
  return DSK_OK;
}

// the 15 launches of one eval forward on stream s
int enqueue_forward(dsk_handle h, dsk_handle_s::Plan* pl, const float* x, int B, int T, float* emb, cudaStream_t s) {
  int rc = 0;
  h->n_marks = 0;
  // profiling level 1: an event after every launch; level 2: only at the section boundaries (conv1 | the 11
  // tensor-core convs | tail), so the conv chain runs back to back exactly as in production
  auto mark = [&](bool boundary = false) {
    if (!h->profiling || (h->profiling == 2 && !boundary)) return;
    if (h->n_marks >= static_cast<int>(h->events.size())) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      h->events.push_back(e);
    }
    cudaEventRecord(h->events[h->n_marks++], s);
  };
  mark(true);
  // conv1 (+bn1 +clip): persistent CTAs, the fbank rows of each tile staged by TMA
  {
    CUtensorMap tmX;
    int grid = 0, n_tiles = 0;
    rc = conv1_launch_geometry(h, x, B, T, &tmX, &grid, &n_tiles);
    if (rc) return rc;
    if (h->bf16) {
      if (int rc2 = ensure_smem_optin(reinterpret_cast<const void*>(dsk::conv1_umma_kernel<true>), dsk::kConv1SmemBytes)) return rc2;
      CUDA_TRY(launch_pdl(dsk::conv1_umma_kernel<true>, dim3(grid), dim3(dsk::kConv1Threads), dsk::kConv1SmemBytes, s, tmX,
                          (const uint4*)h->conv1_img, (const float*)h->scale[0], (const float*)h->bias[0], (uint16_t*)pl->act[0], T, n_tiles, 20.0f));
    } else {
      if (int rc2 = ensure_smem_optin(reinterpret_cast<const void*>(dsk::conv1_umma_kernel<false>), dsk::kConv1SmemBytes)) return rc2;
      CUDA_TRY(launch_pdl(dsk::conv1_umma_kernel<false>, dim3(grid), dim3(dsk::kConv1Threads), dsk::kConv1SmemBytes, s, tmX,
                          (const uint4*)h->conv1_img, (const float*)h->scale[0], (const float*)h->bias[0], (uint16_t*)pl->act[0], T, n_tiles, 20.0f));
    }
    mark(true);
  }
  for (int i = 1; i < DSK_NUM_CONV; ++i) {
    rc = launch_halo(h, pl->halo[i], s);
    if (rc) return rc;
    mark(i == DSK_NUM_CONV - 1);
  }
  // tail
  {
    const int H4 = T / 16, WC = 4 * 512;
    if (h->bf16)
      CUDA_TRY(launch_pdl(dsk::pool_time_kernel<true>, dim3(B, WC / 512), dim3(256), 0, s, (const uint16_t*)pl->act[11],
                          pl->pooled, H4, WC, 512, 1));
    else
      CUDA_TRY(launch_pdl(dsk::pool_time_kernel<false>, dim3(B, WC / 512), dim3(256), 0, s, (const uint16_t*)pl->act[11],
                          pl->pooled, H4, WC, 512, 1));
    mark();
    const int fc_smem = (dsk::kFcUtt + dsk::kFcFeat) * dsk::kFcPitch * 4;
    if (int rc2 = ensure_smem_optin(reinterpret_cast<const void*>(dsk::fc_kernel), fc_smem)) return rc2;
    dim3 g((B + dsk::kFcUtt - 1) / dsk::kFcUtt, h->emb / dsk::kFcFeat, dsk::kFcSplit);
    CUDA_TRY(launch_pdl(dsk::fc_kernel, g, dim3(256), fc_smem, s, (const float*)pl->pooled, (const float*)h->fc_wq,
                        pl->fc_part, B, 2048, h->emb));
    mark();
    CUDA_TRY(launch_pdl(dsk::l2norm_kernel, dim3(B), dim3(512), 0, s, (const float*)pl->fc_part, (int)dsk::kFcSplit,
                        (const float*)h->fc_b, pl->fc_out, emb, (float*)nullptr, B, h->emb, 10.0f));
    mark(true);
  }
  return DSK_OK;
}

void conv1_node_params(dsk_handle h, dsk_handle_s::Plan* pl, int B, int T, cudaKernelNodeParams* kp) {
  memset(kp, 0, sizeof(*kp));
  kp->func = h->bf16 ? reinterpret_cast<void*>(dsk::conv1_umma_kernel<true>) : reinterpret_cast<void*>(dsk::conv1_umma_kernel<false>);
  const int nt = B * (T / 2 / 4);
  const int per_cta = (nt + 4 * h->num_sms - 1) / (4 * h->num_sms);
  kp->gridDim = dim3((nt + per_cta - 1) / per_cta);
  kp->blockDim = dim3(dsk::kConv1Threads);
  kp->sharedMemBytes = dsk::kConv1SmemBytes;
}

// Capture the forward into a graph (stream capture keeps the programmatic-launch edges).  Any failure just leaves the
// plan on the kernel-by-kernel path.
void build_forward_graph(dsk_handle h, dsk_handle_s::Plan* pl, const float* x, int B, int T, float* emb, cudaStream_t s) {
  pl->graph_failed = true;  // until proven otherwise
  // the legacy default stream cannot be captured: forwards issued on it stay on the kernel-by-kernel path
  if (s == nullptr || s == cudaStreamLegacy) return;
  if (cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  const int rc = enqueue_forward(h, pl, x, B, T, emb, s);
  cudaGraph_t g = nullptr;
  const cudaError_t e = cudaStreamEndCapture(s, &g);
  if (rc || e != cudaSuccess || !g) {
    cudaGetLastError();
    if (g) cudaGraphDestroy(g);
    return;
  }
  size_t n = 0;
  if (cudaGraphGetNodes(g, nullptr, &n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    cudaGraphDestroy(g);
    return;
  }
  std::vector<cudaGraphNode_t> nodes(n);
  cudaGraphGetNodes(g, nodes.data(), &n);
  cudaKernelNodeParams c1;
  conv1_node_params(h, pl, B, T, &c1);
  cudaGraphNode_t first = nullptr, last = nullptr;
  for (size_t i = 0; i < n; ++i) {
    cudaGraphNodeType t;
    if (cudaGraphNodeGetType(nodes[i], &t) != cudaSuccess || t != cudaGraphNodeTypeKernel) continue;
    cudaKernelNodeParams kp;
    if (cudaGraphKernelNodeGetParams(nodes[i], &kp) != cudaSuccess) continue;
    if (kp.func == c1.func) first = nodes[i];
    if (kp.func == reinterpret_cast<void*>(dsk::l2norm_kernel)) last = nodes[i];
  }
  cudaGraphExec_t ex = nullptr;
  if (!first || !last || cudaGraphInstantiate(&ex, g, 0) != cudaSuccess) {
    cudaGetLastError();
    cudaGraphDestroy(g);
    return;
  }
  pl->graph = g;
  pl->gexec = ex;
  pl->node_first = first;
  pl->node_last = last;
  pl->g_x = x;
  pl->g_emb = emb;
  pl->graph_failed = false;
}

// patch the input / output pointers of the instantiated graph
int retarget_forward_graph(dsk_handle h, dsk_handle_s::Plan* pl, const float* x, int B, int T, float* emb) {
  if (x != pl->g_x) {
    cudaKernelNodeParams kp;
    conv1_node_params(h, pl, B, T, &kp);
    alignas(64) CUtensorMap tmX;   // the input pointer lives inside the tensor map: re-encode it for this batch
    int grid = 0, n_tiles = 0;
    int rc = conv1_launch_geometry(h, x, B, T, &tmX, &grid, &n_tiles);
    if (rc) return rc;
    const uint4* wimg = reinterpret_cast<const uint4*>(h->conv1_img);
    const float *sc = h->scale[0], *bi = h->bias[0];
    uint16_t* out = static_cast<uint16_t*>(pl->act[0]);
    int Tv = T;
    float clip = 20.0f;
    void* args[8] = {&tmX, &wimg, &sc, &bi, &out, &Tv, &n_tiles, &clip};
    kp.kernelParams = args;
    CUDA_TRY(cudaGraphExecKernelNodeSetParams(pl->gexec, pl->node_first, &kp));
    pl->g_x = x;
  }
  if (emb != pl->g_emb) {
    cudaKernelNodeParams kp;
    memset(&kp, 0, sizeof(kp));
    kp.func = reinterpret_cast<void*>(dsk::l2norm_kernel);
    kp.gridDim = dim3(B);
    kp.blockDim = dim3(512);
    const float* part = pl->fc_part;
    int nsplit = dsk::kFcSplit;
    const float* fb = h->fc_b;
    float* y = pl->fc_out;
    float* inv = nullptr;
    int Bv = B, E = h->emb;
    float alpha = 10.0f;
    void* args[9] = {&part, &nsplit, &fb, &y, &emb, &inv, &Bv, &E, &alpha};
    kp.kernelParams = args;
    CUDA_TRY(cudaGraphExecKernelNodeSetParams(pl->gexec, pl->node_last, &kp));
    pl->g_emb = emb;
  }
  return DSK_OK;
}

}  // namespace

int32_t dsk_rescnn_forward(dsk_handle h, const float* x, int32_t B, int32_t T, float* emb, int32_t mode,
                           void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  adopt_shared_weights(h);
  if (!h->weights_loaded) return fail(DSK_ERR_STATE, "dsk_rescnn_forward: call dsk_load_weights first");
  if (!h->eval_packed)
    return fail(DSK_ERR_STATE, "dsk_rescnn_forward: the weights were loaded with dsk_load_weights_train (training operand "
                               "images only); call dsk_load_weights before an eval forward");
  if (!x || !emb || B <= 0) return fail(DSK_ERR_INVALID, "dsk_rescnn_forward: bad arguments");
  if (T < 16 || T % 16) return fail(DSK_ERR_INVALID, "dsk_rescnn_forward: T must be a positive multiple of 16 (got %d)", T);
  if (mode != DSK_EVAL) return fail(DSK_ERR_INVALID, "dsk_rescnn_forward: use dsk_rescnn_forward_train for batch-statistics BN");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk_handle_s::Plan* pl;
  rc = get_plan(h, B, T, s, &pl);
  if (rc) return rc;
  if (h->use_graph && !h->profiling && pl->warm) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &cs) != cudaSuccess) cudaGetLastError();
    if (cs == cudaStreamCaptureStatusNone) {  // inside a caller's capture the plain launches are what gets recorded
      if (!pl->gexec && !pl->graph_failed) build_forward_graph(h, pl, x, B, T, emb, s);
      if (pl->gexec) {
        rc = retarget_forward_graph(h, pl, x, B, T, emb);
        if (rc) return rc;
        CUDA_TRY(cudaGraphLaunch(pl->gexec, s));
        return DSK_OK;
      }
    }
  }
  pl->warm = true;  // the first call of a shape also sets the one-time function attributes, outside any capture
  return enqueue_forward(h, pl, x, B, T, emb, s);
}

int32_t dsk_set_profiling(dsk_handle h, int32_t enable) {
  if (!h) return fail(DSK_ERR_INVALID, "null handle");
  h->profiling = enable < 0 ? 0 : (enable > 2 ? 2 : enable);
  h->n_marks = 0;
  return DSK_OK;
}

int32_t dsk_get_launch_times(dsk_handle h, float* ms_out, int32_t cap, int32_t* n_out) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!ms_out || !n_out) return fail(DSK_ERR_INVALID, "dsk_get_launch_times: null output");
  const int n = h->n_marks > 0 ? h->n_marks - 1 : 0;
  if (n > cap) return fail(DSK_ERR_INVALID, "dsk_get_launch_times: need room for %d values", n);
  if (n > 0) CUDA_TRY(cudaEventSynchronize(h->events[h->n_marks - 1]));
  for (int i = 0; i < n; ++i) CUDA_TRY(cudaEventElapsedTime(&ms_out[i], h->events[i], h->events[i + 1]));
  *n_out = n;
  return DSK_OK;
}


// ---- training ---------------------------------------------------------------------------------------------------
static int stat_blocks(long M, int C) {
  long gx = kStatBlocksMax / (C / 64);
  const long need = (M + 31) / 32;
  if (gx > need) gx = need;
  return gx < 1 ? 1 : static_cast<int>(gx);
}

// the backward's gradient w.r.t. y[i]: gA and gB alternate from layer 11's (gA) down, so the dgrad of layer i reads G
// and writes grad_buf(c, i - 1) while grad_buf(c, i) is still live
static void* grad_buf(const dsk_train_ctx_s* c, int i) { return (DSK_NUM_CONV - 1 - i) % 2 == 0 ? c->gA : c->gB; }

// Buffers of a train context are sized for `cap` utterances; the launch descriptors (TMA maps, tile counts) are bound
// to the batch size of the current forward (ctx_bind), so one context serves every B <= cap of the same T: the
// reference's hard-triplet branch re-forwards a different number of selected triplets every step
// (train_triplet.py:262-279) and must not allocate a fresh context per distinct count.
static int ctx_bind(dsk_handle h, dsk_train_ctx_s* c, int B);

static int ctx_create(dsk_handle h, int cap, int T, cudaStream_t s, dsk_train_ctx_s** out) {
  dsk_train_ctx_s* c = new dsk_train_ctx_s();
  c->cap = cap;
  c->T = T;
  const int B = cap;
  size_t bytes = 0;
  auto take = [&](size_t n) {
    const size_t o = bytes;
    bytes += (n + 1023) / 1024 * 1024;
    return o;
  };
  size_t o_raw[DSK_NUM_CONV], o_y[DSK_NUM_CONV], o_mean[DSK_NUM_CONV], o_rstd[DSK_NUM_CONV], o_unb[DSK_NUM_CONV];
  size_t max_act = 0;
  for (int i = 0; i < DSK_NUM_CONV; ++i) {
    int H, W, C;
    act_shape(i, T, H, W, C);
    const size_t act = static_cast<size_t>(B) * H * W * C * 2;
    if (act > max_act) max_act = act;
    o_raw[i] = take(2 * act);
    o_y[i] = take(act);
    o_mean[i] = take(C * 4);
    o_rstd[i] = take(C * 4);
    o_unb[i] = take(C * 4);
  }
  const size_t o_pooled = take(static_cast<size_t>(B) * 2048 * 4), o_fc = take(static_cast<size_t>(B) * h->emb * 4);
  const size_t o_fc_part = take(static_cast<size_t>(dsk::kFcSplit) * B * h->emb * 4);
  const size_t o_inv = take(B * 4), o_sc = take(512 * 4), o_sh = take(512 * 4), o_ls = take(2 * 4);
  const size_t o_part = take(static_cast<size_t>(kStatBlocksMax) * 4 * 512 * 4), o_coef = take(3 * 512 * 4);
  const size_t o_gfc = take(static_cast<size_t>(B) * h->emb * 4), o_dP = take(static_cast<size_t>(B) * 2048 * 4);
  size_t dw_bytes = 0;  // [ksplit][tap][cout][cin] fp32 slices of the largest layer
  for (int i = 1; i < DSK_NUM_CONV; ++i) {
    const LayerCfg lc = layer_cfg(i);
    const int taps = lc.ksize * lc.ksize;
    const size_t need = static_cast<size_t>(wgrad_ksplit_bound(h->num_sms, lc.cout, lc.cin, taps)) * taps * lc.cout * lc.cin * 4;
    if (need > dw_bytes) dw_bytes = need;
  }
  const size_t o_dw = take(dw_bytes), o_c1 = take(static_cast<size_t>(B) * ((T / 2 + 7) / 8) * 1600 * 4);
  const size_t o_gA = take(max_act), o_gB = take(max_act), o_G = take(max_act), o_gres = take(max_act);
  const size_t o_rec = take(static_cast<size_t>(B) * (3 * 512 + 1) * 4), o_mtot = take(DSK_NUM_CONV * 8);
  if (cudaMalloc(reinterpret_cast<void**>(&c->base), bytes) != cudaSuccess) {
    cudaGetLastError();
    delete c;
    return fail(DSK_ERR_CUDA, "train context: cudaMalloc of %zu bytes failed", bytes);
  }
  c->bytes = bytes;
  CUDA_TRY(cudaMemsetAsync(c->base, 0, bytes, s));
  uint8_t* b = c->base;
  for (int i = 0; i < DSK_NUM_CONV; ++i) {
    c->raw[i] = reinterpret_cast<float*>(b + o_raw[i]);
    c->y[i] = b + o_y[i];
    c->mean[i] = reinterpret_cast<float*>(b + o_mean[i]);
    c->rstd[i] = reinterpret_cast<float*>(b + o_rstd[i]);
    c->unb[i] = reinterpret_cast<float*>(b + o_unb[i]);
  }
  c->pooled = reinterpret_cast<float*>(b + o_pooled);
  c->fc_out = reinterpret_cast<float*>(b + o_fc);
  c->fc_part = reinterpret_cast<float*>(b + o_fc_part);
  c->inv_norm = reinterpret_cast<float*>(b + o_inv);
  c->scale_t = reinterpret_cast<float*>(b + o_sc);
  c->shift_t = reinterpret_cast<float*>(b + o_sh);
  c->ls = reinterpret_cast<float*>(b + o_ls);
  c->partial = reinterpret_cast<float*>(b + o_part);
  c->coef = reinterpret_cast<float*>(b + o_coef);
  c->g_fc = reinterpret_cast<float*>(b + o_gfc);
  c->dP = reinterpret_cast<float*>(b + o_dP);
  c->dwacc = reinterpret_cast<float*>(b + o_dw);
  c->c1part = reinterpret_cast<float*>(b + o_c1);
  c->gA = b + o_gA;
  c->gB = b + o_gB;
  c->G = b + o_G;
  c->gres = b + o_gres;
  c->rec = reinterpret_cast<float*>(b + o_rec);
  c->mtot = reinterpret_cast<long long*>(b + o_mtot);
  *out = c;
  return DSK_OK;
}

// (re)build the launch descriptors for batch size B (every tensor is a contiguous [B][H][W][C] prefix of its buffer)
static int ctx_bind(dsk_handle h, dsk_train_ctx_s* c, int B) {
  if (c->B == B) return DSK_OK;
  const int T = c->T;
  c->B = 0;
  for (int i = 1; i < DSK_NUM_CONV; ++i) {
    const LayerCfg lc = layer_cfg(i);
    int Hi, Wi, Ci, Ho, Wo, Co;
    act_shape(i - 1, T, Hi, Wi, Ci);
    act_shape(i, T, Ho, Wo, Co);
    int rc = build_conv(h, &c->conv[i], c->y[i - 1], h->wpk[i], nullptr, nullptr, nullptr, c->raw[i], B, Hi, Wi, lc.cin,
                        lc.cout, lc.ksize, lc.stride, 0, 0.f, true);
    if (rc) return rc;
    void* g_out = grad_buf(c, i - 1);
    if (lc.stride == 1) {
      const void* res = (i % 3 == 1) ? c->gres : nullptr;  // skip connection joins at the block input
      rc = build_dgrad_s1(h, &c->dgrad[i][0], c->G, h->wpk_dgrad[i], res, g_out, B, Ho, Wo, lc.cin, lc.cout);
      c->n_dgrad[i] = 1;
    } else {
      for (int cls = 0; cls < 4 && !rc; ++cls)
        rc = build_dgrad_s2(h, &c->dgrad[i][cls], c->G, h->wpk_dgrad[i], g_out, B, Ho, Wo, lc.cin, lc.cout, cls >> 1, cls & 1);
      c->n_dgrad[i] = 4;
    }
    if (rc) return rc;
    rc = build_wgrad(h, &c->wgrad[i], c->G, c->y[i - 1], B, Hi, Wi, lc.cout, lc.cin, lc.ksize, lc.stride, c->dwacc);
    if (rc) return rc;
  }
  c->B = B;
  return DSK_OK;
}

// A free context of the same T with room for B utterances (the smallest such), else a new one of capacity B after
// returning the idle contexts it makes redundant (smaller capacity or another T) to the driver: the pool holds the
// contexts a step has in flight at once (3 for a triplet step), not one per batch size ever seen.
static int ctx_acquire(dsk_handle h, int B, int T, cudaStream_t s, dsk_train_ctx_s** out) {
  dsk_train_ctx_s* best = nullptr;
  for (dsk_train_ctx_s* cand : h->ctx_pool)
    if (!cand->in_use && cand->T == T && cand->cap >= B && (!best || cand->cap < best->cap)) best = cand;
  if (!best) {
    for (size_t i = 0; i < h->ctx_pool.size();) {
      dsk_train_ctx_s* c = h->ctx_pool[i];
      if (!c->in_use && (c->T != T || c->cap < B)) {
        CUDA_TRY(cudaFree(c->base));  // synchronises the device: nothing still reads the buffers
        delete c;
        h->ctx_pool.erase(h->ctx_pool.begin() + i);
      } else {
        ++i;
      }
    }
    int rc = ctx_create(h, B, T, s, &best);
    if (rc) return rc;
    h->ctx_pool.push_back(best);
  }
  int rc = ctx_bind(h, best, B);
  if (rc) return rc;
  best->sync_dir = 0;
  best->sync_fwd = false;
  *out = best;
  return DSK_OK;
}

int32_t dsk_set_loss_scale(dsk_handle h, float scale) {
  if (!h) return fail(DSK_ERR_INVALID, "null handle");
  if (scale < 0.f) return fail(DSK_ERR_INVALID, "loss scale must be >= 0 (0 = automatic)");
  h->loss_scale = scale;
  return DSK_OK;
}

// ---- dsk_debug_set_backward_capture: copies of the backward's intermediate tensors -----------------------------------
static int capture_copy(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (dst) CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s));
  return DSK_OK;
}

// the l2-norm backward's input and output
static int capture_gfc(dsk_handle h, const dsk_train_ctx_s* c, cudaStream_t s) {
  if (!h->bwd_capture_on) return DSK_OK;
  const size_t n = static_cast<size_t>(c->B) * h->emb * 4;
  int rc = capture_copy(h->bwd_capture.g_fc, c->g_fc, n, s);
  return rc ? rc : capture_copy(h->bwd_capture.fc_out, c->fc_out, n, s);
}

// the loss scale and the fc input gradient
static int capture_head(dsk_handle h, const dsk_train_ctx_s* c, cudaStream_t s) {
  if (!h->bwd_capture_on) return DSK_OK;
  int rc = capture_copy(h->bwd_capture.loss_scale, c->ls, 2 * 4, s);
  return rc ? rc : capture_copy(h->bwd_capture.dP, c->dP, static_cast<size_t>(c->B) * 2048 * 4, s);
}

// layer i's BatchNorm backward: its input gradient gy (before) or its outputs G and gres (after)
static int capture_layer(dsk_handle h, const dsk_train_ctx_s* c, int i, bool after, cudaStream_t s) {
  if (!h->bwd_capture_on) return DSK_OK;
  int H, W, C;
  act_shape(i, c->T, H, W, C);
  const size_t bytes = static_cast<size_t>(c->B) * H * W * C * 2;
  if (!after) return capture_copy(h->bwd_capture.gy[i], grad_buf(c, i), bytes, s);
  int rc = capture_copy(h->bwd_capture.G[i], c->G, bytes, s);
  return (rc || i % 3 != 2) ? rc : capture_copy(h->bwd_capture.gres[i], c->gres, bytes, s);
}

int32_t dsk_debug_set_backward_capture(dsk_handle h, const dsk_backward_capture* cap) {
  if (!h) return fail(DSK_ERR_INVALID, "null handle");
  h->bwd_capture_on = cap != nullptr;
  h->bwd_capture = cap ? *cap : dsk_backward_capture{};
  return DSK_OK;
}

// ---- the train-mode layer sequence ------------------------------------------------------------------------------
// Each step below is the only code on the training path that launches its kernels: the default forward and backward,
// the synchronised stages and the per-op BatchNorm entry points are sequences of these calls.  Where a step takes
// `gathered`, a non-null pointer selects the synchronised statistics (the gathered records of N utterances of all
// ranks) and null the statistics of this batch alone.

// layer i's conv into raw[i]: conv1 from the input features, else the bound conv of y[i-1]
static int train_conv(dsk_handle h, const dsk_train_ctx_s* c, int i, cudaStream_t s) {
  if (i > 0) return launch_conv(c->conv[i], s);
  dsk::conv1_kernel<false, true><<<c->B * ((c->T / 2 + 7) / 8), 256, 0, s>>>(c->x, h->conv1_w, h->ones, h->zeros, c->raw[0],
                                                                            c->T, 0, 0.f, 0);
  KERNEL_CHECK();
  return DSK_OK;
}

// BatchNorm batch statistics of raw [M][C] from these M rows alone: mean, rstd, the apply's scale / shift, the unbiased
// variance (unb may be null) and, if update, the running statistics.  partial holds stat_blocks(M, C) * 4 * C floats.
static int bn_local_stats(const float* raw, long M, int C, const float* gamma, const float* beta, float* running_mean,
                          float* running_var, float* mean, float* rstd, float* scale, float* shift, float* unb, int update,
                          float* partial, cudaStream_t s) {
  const int gx = stat_blocks(M, C);
  dsk::bn_stats_partial_kernel<<<dim3(gx, C / 64), 256, 0, s>>>(raw, M, C, partial);
  KERNEL_CHECK();
  dsk::bn_finalize_kernel<<<(C + 31) / 32, 1024, 0, s>>>(partial, raw, gx, C, M, gamma, beta, running_mean, running_var, 0.1f,
                                                         1e-5f, mean, rstd, scale, shift, unb, update);
  KERNEL_CHECK();
  return DSK_OK;
}

// BatchNorm apply + residual (res may be null) + clip: raw fp32 -> y 16-bit
static int bn_apply(bool bf16, const float* raw, const float* scale, const float* shift, const void* res, void* y, long M,
                    int C, cudaStream_t s) {
  auto kern = bf16 ? dsk::bn_apply_kernel<true> : dsk::bn_apply_kernel<false>;
  kern<<<dim3(static_cast<unsigned>((M + 63) / 64), C / 64), 256, 0, s>>>(raw, scale, shift, (const uint16_t*)res,
                                                                          (uint16_t*)y, M, C, 20.0f);
  KERNEL_CHECK();
  return DSK_OK;
}

// layer i's batch statistics, then its BatchNorm + residual + clip into y[i]
static int train_bn_forward(dsk_handle h, dsk_train_ctx_s* c, int i, const float* gathered, int N, cudaStream_t s) {
  int H, W, C;
  act_shape(i, c->T, H, W, C);
  const long M = static_cast<long>(c->B) * H * W;
  const dsk_weights& w = h->w;
  const int update = c->stats_pending ? 0 : 1;
  int rc = DSK_OK;
  if (gathered) {
    dsk::bn_record_finalize_kernel<<<(C + 31) / 32, 1024, 0, s>>>(
        gathered, N, C, w.bn_gamma[i], w.bn_beta[i], w.bn_running_mean[i], w.bn_running_var[i], 0.1f, 1e-5f, c->mean[i],
        c->rstd[i], c->scale_t, c->shift_t, c->unb[i], c->mtot + i, update);
    KERNEL_CHECK();
  } else {
    rc = bn_local_stats(c->raw[i], M, C, w.bn_gamma[i], w.bn_beta[i], w.bn_running_mean[i], w.bn_running_var[i], c->mean[i],
                        c->rstd[i], c->scale_t, c->shift_t, c->unb[i], update, c->partial, s);
  }
  const void* res = (i % 3 == 2) ? c->y[i - 2] : nullptr;
  return rc ? rc : bn_apply(h->bf16, c->raw[i], c->scale_t, c->shift_t, res, c->y[i], M, C, s);
}

// the tail after layer 11: time pooling, fc as K-slice partial sums, then bias + l2 norm into emb_out
static int train_tail(dsk_handle h, dsk_train_ctx_s* c, cudaStream_t s) {
  const int B = c->B, H4 = c->T / 16, WC = 4 * 512;
  auto pool = h->bf16 ? dsk::pool_time_kernel<true> : dsk::pool_time_kernel<false>;
  pool<<<dim3(B, WC / 512), 256, 0, s>>>((const uint16_t*)c->y[11], c->pooled, H4, WC, 512, 0);
  KERNEL_CHECK();
  const int fc_smem = (dsk::kFcUtt + dsk::kFcFeat) * dsk::kFcPitch * 4;
  int rc = ensure_smem_optin(reinterpret_cast<const void*>(dsk::fc_kernel), fc_smem);
  if (rc) return rc;
  dim3 g((B + dsk::kFcUtt - 1) / dsk::kFcUtt, h->emb / dsk::kFcFeat, dsk::kFcSplit);
  dsk::fc_kernel<<<g, 256, fc_smem, s>>>(c->pooled, h->fc_wq, c->fc_part, B, 2048, h->emb);
  KERNEL_CHECK();
  dsk::l2norm_kernel<<<B, 512, 0, s>>>(c->fc_part, dsk::kFcSplit, h->fc_b, c->fc_out, c->emb_out, c->inv_norm, B, h->emb, 10.0f);
  KERNEL_CHECK();
  return DSK_OK;
}

// The loss scale of this backward from the n values of absmax_src (the local g_fc, or the gathered per-utterance maxima):
// explicit (dsk_set_loss_scale), 1 for bf16 operands, else chosen on the device.  Then the fc and pooling backward into
// the gy of layer 11.
static int head_backward(dsk_handle h, dsk_train_ctx_s* c, const float* absmax_src, long n, const dsk_grads* g,
                         cudaStream_t s) {
  const int B = c->B, E = h->emb, H4 = c->T / 16;
  dsk::loss_scale_kernel<<<1, 1024, 0, s>>>(absmax_src, n, h->loss_scale > 0.f ? h->loss_scale : (h->bf16 ? 1.0f : 0.0f), c->ls);
  KERNEL_CHECK();
  dsk::fc_bwd_weight_kernel<<<dim3(E / 8, 2048 / 256), 256, 0, s>>>(c->g_fc, c->pooled, g->fc_w, g->fc_b, B, 2048, E, 512, 4);
  KERNEL_CHECK();
  dsk::fc_bwd_input_kernel<<<dim3(B, 2048 / 256), 256, E * 4, s>>>(c->g_fc, h->fc_wq, c->dP, 2048, E);
  KERNEL_CHECK();
  int rc = capture_head(h, c, s);
  if (rc) return rc;
  auto pool = h->bf16 ? dsk::pool_bwd_kernel<true> : dsk::pool_bwd_kernel<false>;
  pool<<<B, 256, 0, s>>>(c->dP, (uint16_t*)grad_buf(c, DSK_NUM_CONV - 1), H4, 2048, 1.0f / H4, c->ls);
  KERNEL_CHECK();
  return DSK_OK;
}

// BatchNorm backward coefficients from these M rows alone: dgamma, dbeta (times inv_scale, and times the 1/S of dyn when
// set) and the apply's coef [3][C].  partial holds stat_blocks(M, C) * 2 * C floats.
static int bn_bwd_local_coef(bool bf16, const void* gy, const void* y, const float* raw, const float* mean, const float* rstd,
                             long M, int C, const float* gamma, float inv_scale, const float* dyn, float* dgamma,
                             float* dbeta, float* coef, float* partial, cudaStream_t s) {
  const int gx = stat_blocks(M, C);
  auto reduce = bf16 ? dsk::bn_bwd_reduce_kernel<true> : dsk::bn_bwd_reduce_kernel<false>;
  reduce<<<dim3(gx, C / 64), 256, 0, s>>>((const uint16_t*)gy, (const uint16_t*)y, raw, mean, rstd, M, C, 20.0f, partial);
  KERNEL_CHECK();
  dsk::bn_bwd_finalize_kernel<<<(C + 31) / 32, 1024, 0, s>>>(partial, gx, C, M, gamma, rstd, inv_scale, dgamma, dbeta, coef, dyn);
  KERNEL_CHECK();
  return DSK_OK;
}

// BatchNorm backward apply: gy (w.r.t. y) -> G (w.r.t. raw) and gres (w.r.t. the residual; may be null)
static int bn_bwd_apply(bool bf16, const void* gy, const void* y, const float* raw, const float* mean, const float* rstd,
                        const float* coef, void* G, void* gres, long M, int C, cudaStream_t s) {
  auto kern = bf16 ? dsk::bn_bwd_apply_kernel<true> : dsk::bn_bwd_apply_kernel<false>;
  kern<<<dim3(static_cast<unsigned>((M + 63) / 64), C / 64), 256, 0, s>>>(
      (const uint16_t*)gy, (const uint16_t*)y, raw, mean, rstd, coef, (uint16_t*)G, (uint16_t*)gres, M, C, 20.0f);
  KERNEL_CHECK();
  return DSK_OK;
}

// layer i's BatchNorm backward, its weight gradient and, for i > 0, the data gradient into the gy of layer i-1
static int train_bn_backward(dsk_handle h, dsk_train_ctx_s* c, int i, const float* gathered, int N, const dsk_grads* g,
                             cudaStream_t s) {
  const bool bf = h->bf16;
  const int B = c->B, T = c->T;
  int H, W, C;
  act_shape(i, T, H, W, C);
  const long M = static_cast<long>(B) * H * W;
  const void* gy = grad_buf(c, i);
  int rc = capture_layer(h, c, i, false, s);
  if (rc) return rc;
  if (gathered) {
    dsk::bn_bwd_record_finalize_kernel<<<(C + 31) / 32, 1024, 0, s>>>(gathered, N, c->rec, B, C, c->mtot + i, h->w.bn_gamma[i],
                                                                      c->rstd[i], c->ls, g->bn_gamma[i], g->bn_beta[i], c->coef);
    KERNEL_CHECK();
  } else {
    rc = bn_bwd_local_coef(bf, gy, c->y[i], c->raw[i], c->mean[i], c->rstd[i], M, C, h->w.bn_gamma[i], 1.0f, c->ls,
                           g->bn_gamma[i], g->bn_beta[i], c->coef, c->partial, s);
    if (rc) return rc;
  }
  void* gres = (i % 3 == 2) ? c->gres : nullptr;
  if ((rc = bn_bwd_apply(bf, gy, c->y[i], c->raw[i], c->mean[i], c->rstd[i], c->coef, c->G, gres, M, C, s))) return rc;
  if ((rc = capture_layer(h, c, i, true, s))) return rc;
  if (i == 0) {
    const int nblk = B * ((T / 2 + 7) / 8);
    auto part = bf ? dsk::conv1_wgrad_partial_kernel<true> : dsk::conv1_wgrad_partial_kernel<false>;
    part<<<nblk, 256, 0, s>>>((const uint16_t*)c->G, c->x, B, T, c->c1part);
    KERNEL_CHECK();
    dsk::sum_partials_kernel<<<(1600 + 31) / 32, 1024, 0, s>>>(c->c1part, nblk, 1600, 1.0f, g->conv_w[0], c->ls);
    KERNEL_CHECK();
    return DSK_OK;
  }
  const LayerCfg lc = layer_cfg(i);
  const int taps = lc.ksize * lc.ksize;
  const size_t n = static_cast<size_t>(taps) * lc.cout * lc.cin;
  if ((rc = launch_wgrad(h, c->wgrad[i], s))) return rc;
  dsk::unpack_wgrad_kernel<<<static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096), 256, 0, s>>>(
      c->dwacc, g->conv_w[i], lc.cout, lc.cin, taps, 1.0f, c->wgrad[i].p.ksplit, c->wgrad[i].p.slice_elems, c->ls);
  KERNEL_CHECK();
  for (int k = 0; k < c->n_dgrad[i] && !rc; ++k) rc = launch_conv(c->dgrad[i][k], s);
  return rc;
}

int32_t dsk_rescnn_forward_train(dsk_handle h, const float* x, int32_t B, int32_t T, float* emb, dsk_train_ctx* ctx_out,
                                 void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!h->weights_loaded) return fail(DSK_ERR_STATE, "dsk_rescnn_forward_train: call dsk_load_weights first");
  if (!x || !emb || !ctx_out || B <= 0) return fail(DSK_ERR_INVALID, "dsk_rescnn_forward_train: bad arguments");
  if (T < 16 || T % 16) return fail(DSK_ERR_INVALID, "dsk_rescnn_forward_train: T must be a positive multiple of 16 (got %d)", T);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk_train_ctx_s* c = nullptr;
  rc = ctx_acquire(h, B, T, s, &c);
  if (rc) return rc;
  c->in_use = true;
  c->forward_done = false;
  c->stats_pending = h->defer_stats;
  c->x = x;
  c->emb_out = emb;
  for (int i = 0; i < DSK_NUM_CONV; ++i)
    if ((rc = train_conv(h, c, i, s)) || (rc = train_bn_forward(h, c, i, nullptr, 0, s))) return rc;
  if ((rc = train_tail(h, c, s))) return rc;
  c->forward_done = true;
  *ctx_out = c;
  return DSK_OK;
}

int32_t dsk_set_defer_running_stats(dsk_handle h, int32_t on) {
  if (!h) return fail(DSK_ERR_INVALID, "null handle");
  h->defer_stats = on != 0;
  return DSK_OK;
}

int32_t dsk_train_ctx_commit_stats(dsk_handle h, dsk_train_ctx c, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->forward_done) return fail(DSK_ERR_STATE, "dsk_train_ctx_commit_stats: context has no pending forward");
  if (!c->stats_pending) return DSK_OK;  // that forward already updated the running statistics itself
  dsk::BnCommitParams p;
  for (int i = 0; i < DSK_NUM_CONV; ++i) {
    int H, W, C;
    act_shape(i, c->T, H, W, C);
    p.mean[i] = c->mean[i];
    p.unbiased[i] = c->unb[i];
    p.running_mean[i] = h->w.bn_running_mean[i];
    p.running_var[i] = h->w.bn_running_var[i];
    p.C[i] = C;
  }
  p.momentum = 0.1f;
  dsk::bn_running_commit_kernel<<<dim3(4, DSK_NUM_CONV), 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  KERNEL_CHECK();
  c->stats_pending = false;
  return DSK_OK;
}

int32_t dsk_rescnn_backward(dsk_handle h, dsk_train_ctx c, const float* grad_emb, const dsk_grads* g, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->in_use || !c->forward_done) return fail(DSK_ERR_STATE, "dsk_rescnn_backward: context has no pending forward");
  if (c->sync_fwd) return fail(DSK_ERR_STATE, "dsk_rescnn_backward: a synchronised forward needs dsk_sync_backward_begin");
  if (!grad_emb || !g) return fail(DSK_ERR_INVALID, "dsk_rescnn_backward: null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::l2norm_bwd_kernel<<<c->B, 128, 0, s>>>(c->fc_out, c->inv_norm, grad_emb, c->g_fc, h->emb, 10.0f);
  KERNEL_CHECK();
  if ((rc = capture_gfc(h, c, s)) || (rc = head_backward(h, c, c->g_fc, static_cast<long>(c->B) * h->emb, g, s))) return rc;
  for (int i = DSK_NUM_CONV - 1; i >= 0; --i)
    if ((rc = train_bn_backward(h, c, i, nullptr, 0, g, s))) return rc;
  c->forward_done = false;
  c->in_use = false;
  return DSK_OK;
}

int32_t dsk_train_ctx_read(dsk_handle h, dsk_train_ctx c, int32_t which, int32_t layer, float* out_nchw, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->forward_done) return fail(DSK_ERR_STATE, "dsk_train_ctx_read: context has no pending forward");
  if (layer < 0 || layer >= DSK_NUM_CONV || !out_nchw || which < 0 || which > 1)
    return fail(DSK_ERR_INVALID, "dsk_train_ctx_read: bad arguments");
  int H, W, C;
  act_shape(layer, c->T, H, W, C);
  const long n = static_cast<long>(c->B) * C * H * W;
  const int blocks = static_cast<int>((n + 255) / 256 < 65535 ? (n + 255) / 256 : 65535);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (which == 0)
    dsk::nhwc_f32_to_nchw_kernel<<<blocks, 256, 0, s>>>(c->raw[layer], out_nchw, c->B, C, H * W);
  else if (h->bf16)
    dsk::nhwc16_to_nchw_kernel<true><<<blocks, 256, 0, s>>>((const uint16_t*)c->y[layer], out_nchw, c->B, C, H * W);
  else
    dsk::nhwc16_to_nchw_kernel<false><<<blocks, 256, 0, s>>>((const uint16_t*)c->y[layer], out_nchw, c->B, C, H * W);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_debug_backward_plan(dsk_handle h, dsk_train_ctx c, int32_t layer, int32_t* out) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->B) return fail(DSK_ERR_STATE, "dsk_debug_backward_plan: context is not bound to a batch");
  if (layer < 0 || layer >= DSK_NUM_CONV || !out) return fail(DSK_ERR_INVALID, "dsk_debug_backward_plan: bad arguments");
  int H, W, C;
  act_shape(layer, c->T, H, W, C);
  out[0] = out[1] = 0;
  if (layer > 0) {
    const dsk::WgradParams& p = c->wgrad[layer].p;
    const int chunks = p.chunks_w * p.chunks_h * p.chunks_n;
    out[0] = p.ksplit;
    out[1] = (chunks + p.ksplit - 1) / p.ksplit;
  }
  out[2] = stat_blocks(static_cast<long>(c->B) * H * W, C);
  return DSK_OK;
}

int32_t dsk_debug_train_tiles(dsk_handle h, dsk_train_ctx c, int32_t layer, int32_t* out) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->B) return fail(DSK_ERR_STATE, "dsk_debug_train_tiles: context is not bound to a batch");
  if (layer < 0 || layer >= DSK_NUM_CONV || !out) return fail(DSK_ERR_INVALID, "dsk_debug_train_tiles: bad arguments");
  for (int k = 0; k < 6; ++k) out[k] = 0;
  if (layer == 0) return DSK_OK;
  const dsk::ConvParams& f = c->conv[layer].p;
  for (int k = 0; k < c->n_dgrad[layer]; ++k) {  // built on the forward's output grid: the same box, or a bug
    const dsk::ConvParams& d = c->dgrad[layer][k].p;
    if (d.wt != f.wt || d.hb != f.hb || d.nb != f.nb)
      return fail(DSK_ERR_STATE, "dsk_debug_train_tiles: layer %d data-gradient conv %d tiles %dx%dx%d, forward %dx%dx%d",
                  layer, k, d.wt, d.hb, d.nb, f.wt, f.hb, f.nb);
  }
  const dsk::WgradParams& w = c->wgrad[layer].p;
  out[0] = f.wt;
  out[1] = f.hb;
  out[2] = f.nb;
  out[3] = w.wt;
  out[4] = w.hb;
  out[5] = w.nb;
  return DSK_OK;
}

int32_t dsk_debug_read_eval_activation(dsk_handle h, int32_t layer, void* dst, int64_t dst_bytes, int32_t* planar_out,
                                       void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (layer < 0 || layer >= DSK_NUM_CONV || !dst || !planar_out)
    return fail(DSK_ERR_INVALID, "dsk_debug_read_eval_activation: bad arguments");
  // get_plan keeps at most one shape, and dsk_load_weights drops it
  if (h->plans.empty()) return fail(DSK_ERR_STATE, "dsk_debug_read_eval_activation: no eval forward plan is cached");
  const dsk_handle_s::Plan& pl = h->plans.begin()->second;
  int H, W, C;
  act_shape(layer, pl.T, H, W, C);
  // the layout get_plan chose for this buffer
  const bool planar = (layer % 3 == 2) && layer < DSK_NUM_CONV - 1;
  const size_t bytes = planar ? 4 * padded_bytes(pl.B, H / 2, W / 2, C) : padded_bytes(pl.B, H, W, C);
  if (dst_bytes < 0 || static_cast<size_t>(dst_bytes) != bytes)
    return fail(DSK_ERR_INVALID, "dsk_debug_read_eval_activation: layer %d holds %zu bytes, dst_bytes is %lld", layer, bytes,
                static_cast<long long>(dst_bytes));
  CUDA_TRY(cudaMemcpyAsync(dst, pl.act[layer], bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
  *planar_out = planar ? 1 : 0;
  return DSK_OK;
}

int32_t dsk_train_ctx_release(dsk_handle h, dsk_train_ctx c) {
  if (!h || !c) return fail(DSK_ERR_INVALID, "dsk_train_ctx_release: null argument");
  c->in_use = false;
  c->forward_done = false;
  return DSK_OK;
}

// ---- synchronised BatchNorm: the train forward and backward as resumable stages -----------------------------------
// Each stage ends where this rank's per-utterance records (train_kernels.cuh) are ready; the caller gathers every rank's
// records in rank order and resumes with them.  The stages run the steps of the train-mode layer sequence above, with
// the batch statistics, the backward coefficients and the loss scale taken from the gathered records.

// fp32 words of one utterance's record at the current stage
static long sync_rec_words(const dsk_train_ctx_s* c) {
  if (c->sync_dir == 2 && c->sync_stage == DSK_NUM_CONV) return 1;  // max |dL/d(fc out)|
  int H, W, C;
  act_shape(c->sync_stage, c->T, H, W, C);
  return c->sync_dir == 1 ? 3L * C + 1 : 2L * C;
}

static void sync_fwd_records(dsk_train_ctx_s* c, int i, cudaStream_t s) {
  int H, W, C;
  act_shape(i, c->T, H, W, C);
  dsk::bn_utt_record_kernel<<<dim3(c->B, C / 64), 256, 0, s>>>(c->raw[i], H * W, C, c->rec);
}

static void sync_bwd_records(dsk_handle h, dsk_train_ctx_s* c, int i, cudaStream_t s) {
  int H, W, C;
  act_shape(i, c->T, H, W, C);
  const uint16_t* gy = (const uint16_t*)grad_buf(c, i);
  dim3 g(c->B, C / 64);
  if (h->bf16)
    dsk::bn_bwd_utt_record_kernel<true><<<g, 256, 0, s>>>(gy, (const uint16_t*)c->y[i], c->raw[i], c->mean[i], c->rstd[i],
                                                          H * W, C, 20.0f, c->rec);
  else
    dsk::bn_bwd_utt_record_kernel<false><<<g, 256, 0, s>>>(gy, (const uint16_t*)c->y[i], c->raw[i], c->mean[i], c->rstd[i],
                                                           H * W, C, 20.0f, c->rec);
}

// forward of layer i up to its records
static int sync_fwd_conv(dsk_handle h, dsk_train_ctx_s* c, int i, cudaStream_t s) {
  int rc = train_conv(h, c, i, s);
  if (rc) return rc;
  sync_fwd_records(c, i, s);
  KERNEL_CHECK();
  return DSK_OK;
}

// layer i's global statistics from the gathered records, its BatchNorm + residual + clip, then the next layer's conv
// and records or the tail
static int sync_fwd_stage(dsk_handle h, dsk_train_ctx_s* c, const float* gathered, int N, cudaStream_t s, int* more) {
  const int i = c->sync_stage;
  int rc = train_bn_forward(h, c, i, gathered, N, s);
  if (rc) return rc;
  if (i + 1 < DSK_NUM_CONV) {
    c->sync_stage = i + 1;
    *more = 1;
    return sync_fwd_conv(h, c, i + 1, s);
  }
  if ((rc = train_tail(h, c, s))) return rc;
  c->sync_dir = 0;
  c->forward_done = true;
  *more = 0;
  return DSK_OK;
}

// stage 12: the loss scale from the gathered maxima, the fc / pooling backward and layer 11's records.  Stage i: layer i's
// coefficients from the gathered records, the BatchNorm backward, its weight gradient, then the data gradient and layer
// i-1's records (i > 0).
static int sync_bwd_stage(dsk_handle h, dsk_train_ctx_s* c, const float* gathered, int N, cudaStream_t s, int* more) {
  const int i = c->sync_stage;
  int rc = i == DSK_NUM_CONV ? head_backward(h, c, gathered, N, &c->grads, s)
                             : train_bn_backward(h, c, i, gathered, N, &c->grads, s);
  if (rc) return rc;
  if (i == 0) {
    c->sync_dir = 0;
    c->forward_done = false;
    c->in_use = false;
    *more = 0;
    return DSK_OK;
  }
  c->sync_stage = i - 1;
  sync_bwd_records(h, c, i - 1, s);
  KERNEL_CHECK();
  *more = 1;
  return DSK_OK;
}

int32_t dsk_sync_forward_begin(dsk_handle h, const float* x, int32_t B, int32_t T, float* emb, dsk_train_ctx* ctx_out,
                               void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!h->weights_loaded) return fail(DSK_ERR_STATE, "dsk_sync_forward_begin: call dsk_load_weights first");
  if (!x || !emb || !ctx_out || B <= 0) return fail(DSK_ERR_INVALID, "dsk_sync_forward_begin: bad arguments");
  if (T < 16 || T % 16) return fail(DSK_ERR_INVALID, "dsk_sync_forward_begin: T must be a positive multiple of 16 (got %d)", T);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk_train_ctx_s* c = nullptr;
  rc = ctx_acquire(h, B, T, s, &c);
  if (rc) return rc;
  c->in_use = true;
  c->forward_done = false;
  c->stats_pending = h->defer_stats;
  c->x = x;
  c->emb_out = emb;
  c->sync_dir = 1;
  c->sync_stage = 0;
  c->sync_fwd = true;
  rc = sync_fwd_conv(h, c, 0, s);
  if (rc) {
    c->in_use = false;
    c->sync_dir = 0;
    return rc;
  }
  *ctx_out = c;
  return DSK_OK;
}

int32_t dsk_sync_backward_begin(dsk_handle h, dsk_train_ctx c, const float* grad_emb, const dsk_grads* g, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->in_use || !c->forward_done || !c->sync_fwd || c->sync_dir)
    return fail(DSK_ERR_STATE, "dsk_sync_backward_begin: context has no finished synchronised forward");
  if (!grad_emb || !g) return fail(DSK_ERR_INVALID, "dsk_sync_backward_begin: null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::l2norm_bwd_kernel<<<c->B, 128, 0, s>>>(c->fc_out, c->inv_norm, grad_emb, c->g_fc, h->emb, 10.0f);
  KERNEL_CHECK();
  if ((rc = capture_gfc(h, c, s))) return rc;
  dsk::row_absmax_kernel<<<c->B, 128, 0, s>>>(c->g_fc, h->emb, c->rec);
  KERNEL_CHECK();
  c->grads = *g;
  c->sync_dir = 2;
  c->sync_stage = DSK_NUM_CONV;
  return DSK_OK;
}

int32_t dsk_sync_records(dsk_handle h, dsk_train_ctx c, void** ptr, int64_t* bytes) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!ptr || !bytes) return fail(DSK_ERR_INVALID, "dsk_sync_records: null argument");
  if (!c || !c->in_use || !c->sync_dir) return fail(DSK_ERR_STATE, "dsk_sync_records: no synchronised stage in progress");
  *ptr = c->rec;
  *bytes = static_cast<int64_t>(c->B) * sync_rec_words(c) * 4;
  return DSK_OK;
}

int32_t dsk_sync_stage(dsk_handle h, dsk_train_ctx c, const void* gathered, int32_t n_total, int32_t* more, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!c || !c->in_use || !c->sync_dir) return fail(DSK_ERR_STATE, "dsk_sync_stage: no synchronised stage in progress");
  if (!gathered || !more || n_total < c->B)
    return fail(DSK_ERR_INVALID, "dsk_sync_stage: need the gathered records of n_total >= %d utterances", c->B);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const float* gr = static_cast<const float*>(gathered);
  return c->sync_dir == 1 ? sync_fwd_stage(h, c, gr, n_total, s, more) : sync_bwd_stage(h, c, gr, n_total, s, more);
}


// ---- per-op entry points for unit tests of the backward building blocks -------------------------------------------
int32_t dsk_conv2d_dgrad_nhwc(dsk_handle h, const void* G, const float* w_oihw, const void* res, void* gin, int32_t B,
                              int32_t Hin, int32_t Win, int32_t cin, int32_t cout, int32_t ksize, int32_t stride,
                              void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!G || !w_oihw || !gin) return fail(DSK_ERR_INVALID, "dsk_conv2d_dgrad_nhwc: null pointer");
  if (!((ksize == 3 && stride == 1) || (ksize == 5 && stride == 2)))
    return fail(DSK_ERR_INVALID, "dgrad: only 3x3 s1 p1 and 5x5 s2 p2 are supported");
  if (stride == 2 && res) return fail(DSK_ERR_INVALID, "dgrad: residual only with stride 1");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int taps = ksize * ksize;
  const long n = static_cast<long>(cout) * cin * taps;
  void* wpk = nullptr;
  CUDA_TRY(cudaMallocAsync(&wpk, n * 2, s));
  const int blocks = static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  if (h->bf16) dsk::pack_conv_weight_dgrad_kernel<true><<<blocks, 256, 0, s>>>(w_oihw, (uint16_t*)wpk, cout, cin, taps, stride == 1);
  else dsk::pack_conv_weight_dgrad_kernel<false><<<blocks, 256, 0, s>>>(w_oihw, (uint16_t*)wpk, cout, cin, taps, stride == 1);
  KERNEL_CHECK();
  const int Hout = Hin / stride, Wout = Win / stride;
  ConvLaunch L;
  if (stride == 1) {
    rc = build_dgrad_s1(h, &L, G, wpk, res, gin, B, Hin, Win, cin, cout);
    if (!rc) rc = launch_conv(L, s);
  } else {
    for (int cls = 0; cls < 4 && !rc; ++cls) {
      rc = build_dgrad_s2(h, &L, G, wpk, gin, B, Hout, Wout, cin, cout, cls >> 1, cls & 1);
      if (!rc) rc = launch_conv(L, s);
    }
  }
  CUDA_TRY(cudaFreeAsync(wpk, s));
  return rc;
}

int32_t dsk_conv2d_wgrad_nhwc(dsk_handle h, const void* G, const void* X, float* dw_oihw, int32_t B, int32_t Hin,
                              int32_t Win, int32_t cin, int32_t cout, int32_t ksize, int32_t stride, float mult,
                              void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!G || !X || !dw_oihw) return fail(DSK_ERR_INVALID, "dsk_conv2d_wgrad_nhwc: null pointer");
  if (!((ksize == 3 && stride == 1) || (ksize == 5 && stride == 2)))
    return fail(DSK_ERR_INVALID, "wgrad: only 3x3 s1 p1 and 5x5 s2 p2 are supported");
  if (cin % 64 || cout % 64) return fail(DSK_ERR_INVALID, "wgrad: channel counts must be multiples of 64");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int taps = ksize * ksize;
  const size_t n = static_cast<size_t>(taps) * cout * cin;
  float* acc = nullptr;
  WgradLaunch L;
  rc = build_wgrad(h, &L, G, X, B, Hin, Win, cout, cin, ksize, stride, nullptr);
  if (rc) return rc;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&acc), n * 4 * L.p.ksplit, s));
  L.p.dw = acc;
  rc = launch_wgrad(h, L, s);
  if (!rc) {
    dsk::unpack_wgrad_kernel<<<static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096), 256, 0, s>>>(
        acc, dw_oihw, cout, cin, taps, mult, L.p.ksplit, L.p.slice_elems);
    KERNEL_CHECK();
  }
  CUDA_TRY(cudaFreeAsync(acc, s));
  return rc;
}

// BatchNorm(train) + optional residual + clip on an NHWC tensor viewed as [M][C]: raw fp32 -> y 16-bit, plus the
// saved mean / rstd (running stats updated in place).
int32_t dsk_bn_act_train_forward(dsk_handle h, const float* raw, const float* gamma, const float* beta,
                                 float* running_mean, float* running_var, const void* res, void* y, float* mean,
                                 float* rstd, int64_t M, int32_t C, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!raw || !gamma || !beta || !running_mean || !running_var || !y || !mean || !rstd || C % 64 || C > 512 || M <= 0)
    return fail(DSK_ERR_INVALID, "dsk_bn_act_train_forward: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* tmp = nullptr;
  const int gx = stat_blocks(M, C);
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&tmp), (static_cast<size_t>(gx) * 4 * C + 2 * C) * 4, s));
  float *partial = tmp, *sc = tmp + static_cast<size_t>(gx) * 4 * C, *sh = sc + C;
  rc = bn_local_stats(raw, M, C, gamma, beta, running_mean, running_var, mean, rstd, sc, sh, nullptr, 1, partial, s);
  if (!rc) rc = bn_apply(h->bf16, raw, sc, sh, res, y, M, C, s);
  CUDA_TRY(cudaFreeAsync(tmp, s));
  return rc;
}

// Backward of the above: gy (16-bit, w.r.t. y) -> G (16-bit, w.r.t. raw), gres (16-bit, w.r.t. res; may be NULL),
// dgamma, dbeta (fp32, multiplied by inv_scale).
int32_t dsk_bn_act_train_backward(dsk_handle h, const void* gy, const void* y, const float* raw, const float* gamma,
                                  const float* mean, const float* rstd, void* G, void* gres, float* dgamma,
                                  float* dbeta, int64_t M, int32_t C, float inv_scale, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!gy || !y || !raw || !gamma || !mean || !rstd || !G || !dgamma || !dbeta || C % 64 || C > 512 || M <= 0)
    return fail(DSK_ERR_INVALID, "dsk_bn_act_train_backward: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* tmp = nullptr;
  const int gx = stat_blocks(M, C);
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&tmp), (static_cast<size_t>(gx) * 2 * C + 3 * C) * 4, s));
  float *partial = tmp, *coef = tmp + static_cast<size_t>(gx) * 2 * C;
  rc = bn_bwd_local_coef(h->bf16, gy, y, raw, mean, rstd, M, C, gamma, inv_scale, nullptr, dgamma, dbeta, coef, partial, s);
  if (!rc) rc = bn_bwd_apply(h->bf16, gy, y, raw, mean, rstd, coef, G, gres, M, C, s);
  CUDA_TRY(cudaFreeAsync(tmp, s));
  return rc;
}

// dsk_bn_act_train_forward with the statistics of the synchronised path: B utterances of HW pixels each (M = B HW rows),
// one record per utterance, combined by the record finalize as if gathered from any split of the B utterances.
int32_t dsk_bn_act_sync_train_forward(dsk_handle h, const float* raw, const float* gamma, const float* beta,
                                      float* running_mean, float* running_var, const void* res, void* y, float* mean,
                                      float* rstd, int32_t B, int32_t HW, int32_t C, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!raw || !gamma || !beta || !running_mean || !running_var || !y || !mean || !rstd || C % 64 || C > 512 || B <= 0 ||
      HW <= 0)
    return fail(DSK_ERR_INVALID, "dsk_bn_act_sync_train_forward: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* tmp = nullptr;
  const size_t rec_words = static_cast<size_t>(B) * (3 * C + 1);
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&tmp), (rec_words + 2 * C) * 4, s));
  float *rec = tmp, *sc = tmp + rec_words, *sh = sc + C;
  dsk::bn_utt_record_kernel<<<dim3(B, C / 64), 256, 0, s>>>(raw, HW, C, rec);
  KERNEL_CHECK();
  dsk::bn_record_finalize_kernel<<<(C + 31) / 32, 1024, 0, s>>>(rec, B, C, gamma, beta, running_mean, running_var, 0.1f, 1e-5f,
                                                                mean, rstd, sc, sh, nullptr, nullptr, 1);
  KERNEL_CHECK();
  rc = bn_apply(h->bf16, raw, sc, sh, res, y, static_cast<long>(B) * HW, C, s);
  CUDA_TRY(cudaFreeAsync(tmp, s));
  return rc;
}

int32_t dsk_conv3x3_padded(dsk_handle h, const void* in, const void* w_packed, const float* scale, const float* bias,
                           const void* res, void* out, int32_t N, int32_t H, int32_t W, int32_t C, int32_t flags,
                           float clip_hi, int32_t out_planar, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!in || !w_packed || !out) return fail(DSK_ERR_INVALID, "dsk_conv3x3_padded: null pointer");
  if ((flags & dsk::CONV_RESIDUAL) && !res) return fail(DSK_ERR_INVALID, "dsk_conv3x3_padded: residual flag without res");
  HaloLaunch L;
  std::vector<float> sc_h, bi_h;
  rc = fetch_affine(scale, bias, C, &sc_h, &bi_h);
  if (rc) return rc;
  rc = build_halo(h, &L, in, w_packed, scale ? sc_h.data() : nullptr, bias ? bi_h.data() : nullptr, res, out, N, H, W, C, C, 3,
                  flags, clip_hi, out_planar);
  if (rc) return rc;
  return launch_halo(h, L, static_cast<cudaStream_t>(stream));
}

int32_t dsk_conv5x5s2_planar(dsk_handle h, const void* in_planar, const float* w_oihw, const float* scale,
                             const float* bias, void* out, int32_t N, int32_t Hout, int32_t Wout, int32_t cin,
                             int32_t cout, int32_t flags, float clip_hi, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!in_planar || !w_oihw || !out) return fail(DSK_ERR_INVALID, "dsk_conv5x5s2_planar: null pointer");
  if (flags & dsk::CONV_RESIDUAL) return fail(DSK_ERR_INVALID, "dsk_conv5x5s2_planar: no residual on this path");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long n = static_cast<long>(cout) * cin * 25;
  void* wpk = nullptr;
  int* perm_d = nullptr;
  int perm[25];
  planar_tap_order(perm);
  CUDA_TRY(cudaMallocAsync(&wpk, n * 2, s));
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&perm_d), sizeof(perm), s));
  CUDA_TRY(cudaMemcpyAsync(perm_d, perm, sizeof(perm), cudaMemcpyHostToDevice, s));
  const int blocks = static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  if (h->bf16) dsk::pack_conv_weight_perm_kernel<true><<<blocks, 256, 0, s>>>(w_oihw, (uint16_t*)wpk, cout, cin, 25, perm_d);
  else dsk::pack_conv_weight_perm_kernel<false><<<blocks, 256, 0, s>>>(w_oihw, (uint16_t*)wpk, cout, cin, 25, perm_d);
  KERNEL_CHECK();
  CUDA_TRY(cudaStreamSynchronize(s));  // perm[] is a stack array
  HaloLaunch L;
  std::vector<float> sc_h, bi_h;
  rc = fetch_affine(scale, bias, cout, &sc_h, &bi_h);
  if (!rc)
    rc = build_halo(h, &L, in_planar, wpk, scale ? sc_h.data() : nullptr, bias ? bi_h.data() : nullptr, nullptr, out, N, Hout,
                    Wout, cin, cout, 5, flags, clip_hi, 0);
  if (!rc) rc = launch_halo(h, L, s);
  CUDA_TRY(cudaFreeAsync(wpk, s));
  CUDA_TRY(cudaFreeAsync(perm_d, s));
  return rc;
}

int64_t dsk_padded_positions(int32_t N, int32_t H, int32_t W) { return padded_positions(N, H, W); }

int32_t dsk_conv2d_nhwc(dsk_handle h, const void* in, const void* w_packed, const float* scale, const float* bias,
                        const void* res, void* out, int32_t B, int32_t Hin, int32_t Win, int32_t cin, int32_t cout,
                        int32_t ksize, int32_t stride, int32_t flags, float clip_hi, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!in || !w_packed || !out) return fail(DSK_ERR_INVALID, "dsk_conv2d_nhwc: null pointer");
  if ((flags & dsk::CONV_RESIDUAL) && !res) return fail(DSK_ERR_INVALID, "dsk_conv2d_nhwc: residual flag without res");
  ConvLaunch L;
  rc = build_conv(h, &L, in, w_packed, scale, bias, res, out, B, Hin, Win, cin, cout, ksize, stride, flags, clip_hi);
  if (rc) return rc;
  return launch_conv(L, static_cast<cudaStream_t>(stream));
}

int32_t dsk_pack_conv_weight(dsk_handle h, const float* w_oihw, void* w_packed, int32_t cout, int32_t cin,
                             int32_t ksize, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  const long n = static_cast<long>(cout) * cin * ksize * ksize;
  const int blocks = static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->bf16)
    dsk::pack_conv_weight_kernel<true><<<blocks, 256, 0, s>>>(w_oihw, (uint16_t*)w_packed, cout, cin, ksize * ksize);
  else
    dsk::pack_conv_weight_kernel<false><<<blocks, 256, 0, s>>>(w_oihw, (uint16_t*)w_packed, cout, cin, ksize * ksize);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_nchw_f32_to_nhwc16(dsk_handle h, const float* in, void* out, int32_t B, int32_t C, int32_t H, int32_t W,
                               void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  const long n = static_cast<long>(B) * C * H * W;
  const int blocks = static_cast<int>((n + 255) / 256 < 65535 ? (n + 255) / 256 : 65535);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->bf16)
    dsk::nchw_to_nhwc16_kernel<true><<<blocks, 256, 0, s>>>(in, (uint16_t*)out, B, C, H * W);
  else
    dsk::nchw_to_nhwc16_kernel<false><<<blocks, 256, 0, s>>>(in, (uint16_t*)out, B, C, H * W);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_nhwc16_to_nchw_f32(dsk_handle h, const void* in, float* out, int32_t B, int32_t C, int32_t H, int32_t W,
                               void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  const long n = static_cast<long>(B) * C * H * W;
  const int blocks = static_cast<int>((n + 255) / 256 < 65535 ? (n + 255) / 256 : 65535);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->bf16)
    dsk::nhwc16_to_nchw_kernel<true><<<blocks, 256, 0, s>>>((const uint16_t*)in, out, B, C, H * W);
  else
    dsk::nhwc16_to_nchw_kernel<false><<<blocks, 256, 0, s>>>((const uint16_t*)in, out, B, C, H * W);
  KERNEL_CHECK();
  return DSK_OK;
}

// ---- distances / loss / selection -----------------------------------------------------------------
static inline float pd_eps(int D) { return static_cast<float>(1e-4 / static_cast<double>(D)); }
int32_t dsk_allpairs_topk(const float* E, const int64_t* labels, int32_t N, int32_t D, int32_t k, int64_t* idx,
                          float* val, void* stream);

int32_t dsk_pairwise_distance(const float* x1, const float* x2, int32_t B, int32_t D, float* out, void* stream) {
  if (!x1 || !x2 || !out || B <= 0 || D <= 0) return fail(DSK_ERR_INVALID, "dsk_pairwise_distance: bad arguments");
  dsk::pairwise_distance_kernel<<<(B + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(x1, x2, B, D, pd_eps(D), out);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_pairwise_distance_bwd(const float* x1, const float* x2, const float* dist, const float* grad_out,
                                  int32_t B, int32_t D, float* grad_x1, float* grad_x2, void* stream) {
  if (!x1 || !x2 || !dist || !grad_out || B <= 0 || D <= 0)
    return fail(DSK_ERR_INVALID, "dsk_pairwise_distance_bwd: bad arguments");
  const long n = static_cast<long>(B) * D;
  dsk::pairwise_distance_bwd_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x1, x2, dist, grad_out, B, D, grad_x1, grad_x2);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_triplet_loss(const float* a, const float* p, const float* n, int32_t B, int32_t D, float margin,
                         float* loss, float* d_p, float* d_n, void* stream) {
  if (!a || !p || !n || !loss || !d_p || !d_n || B <= 0 || D <= 0)
    return fail(DSK_ERR_INVALID, "dsk_triplet_loss: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::triplet_dist_kernel<<<(B + 7) / 8, 256, 0, s>>>(a, p, n, B, D, pd_eps(D), d_p, d_n);
  KERNEL_CHECK();
  dsk::hinge_mean_kernel<<<1, 1024, 0, s>>>(d_p, d_n, B, margin, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_triplet_loss_bwd(const float* a, const float* p, const float* n, const float* d_p, const float* d_n,
                             const float* grad_loss, int32_t B, int32_t D, float margin, float* ga, float* gp,
                             float* gn, void* stream) {
  if (!a || !p || !n || !d_p || !d_n || !grad_loss || !ga || !gp || !gn || B <= 0 || D <= 0)
    return fail(DSK_ERR_INVALID, "dsk_triplet_loss_bwd: bad arguments");
  const long cnt = static_cast<long>(B) * D;
  dsk::triplet_loss_bwd_kernel<<<(cnt + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      a, p, n, d_p, d_n, grad_loss, B, D, margin, ga, gp, gn);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_margin_select(const float* d_p, const float* d_n, int32_t B, float margin, int64_t* idx,
                          int32_t* count, void* stream) {
  if (!d_p || !d_n || !idx || !count || B <= 0) return fail(DSK_ERR_INVALID, "dsk_margin_select: bad arguments");
  dsk::margin_select_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(d_p, d_n, B, margin, idx, count);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_gather_rows(const float* src, const int64_t* idx, const int32_t* count, int32_t max_rows,
                        int64_t row_elems, float* out, void* stream) {
  if (!src || !idx || !count || !out || max_rows <= 0 || row_elems <= 0)
    return fail(DSK_ERR_INVALID, "dsk_gather_rows: bad arguments");
  dsk::gather_rows_kernel<<<max_rows, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, idx, count, row_elems, out);
  KERNEL_CHECK();
  return DSK_OK;
}

// The tensor-core Gram of the all-pairs ops for the anchor rows [row0, row0 + rows): (re)builds the plan cached in the
// handle for (N, D, row0, rows) - buffers and the Gram GEMM descriptors - then rounds E to 16 bit, takes the squared
// norms of the rounded rows and runs G = E16[row0 : row0 + rows_pad] E16^T (rows_pad x Npad) on `s`.  A rebuild
// synchronises `s`: a caller that alternates row ranges pays it on every change.
static int allpairs_gram(dsk_handle h, const float* E, int N, int D, int row0, int rows, cudaStream_t s,
                         const float** G_out, const float** norms_out, int* Npad_out) {
  AllpairsPlan& A = h->allpairs;
  int rc = plan_acquire(A, {N, D, row0, rows}, s, [&]() -> int {
    const int rows_pad = (rows + 127) / 128 * 128;
    A.Npad = (N + 127) / 128 * 128;
    // the "pixel" view reads rows_pad rows of E16 from row0, which may run past Npad
    A.Epad = row0 + rows_pad > A.Npad ? row0 + rows_pad : A.Npad;
    if (int rc = arena_alloc(&A.buf, {{&A.e16, A.Epad * D * 2ull}, {&A.gram, 1ull * rows_pad * A.Npad * 4},
                                      {&A.norms, A.Epad * 4ull}}, s))
      return rc;
    // the anchor rows of E16 against all its rows, K = D, in the handle's operand type
    return build_gemm(h, &A.gemm, A.e16 + static_cast<size_t>(row0) * D, rows_pad, A.e16, A.Npad, D, A.gram, false);
  });
  if (rc) return rc;
  if (h->bf16) dsk::allpairs_prep_kernel<true><<<A.Epad, 128, 0, s>>>(E, N, D, A.e16, A.norms);
  else dsk::allpairs_prep_kernel<false><<<A.Epad, 128, 0, s>>>(E, N, D, A.e16, A.norms);
  KERNEL_CHECK();
  for (size_t i = 0; i < A.gemm.size() && !rc; ++i) rc = launch_conv(A.gemm[i], s);
  *G_out = A.gram;
  *norms_out = A.norms;
  *Npad_out = A.Npad;
  return rc;
}

// unit roundoff of the 16-bit operand format of the Gram
static inline float allpairs_unit_roundoff(dsk_handle h) { return h->bf16 ? 1.0f / 256.0f : 1.0f / 2048.0f; }

int32_t dsk_allpairs_topk_tc(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D, int32_t k,
                             int64_t* idx, float* val, void* stream) {
  int rc = check_handle(h);
  if (rc) return rc;
  if (!E || !labels || !idx || !val || N <= 0 || D <= 0 || k <= 0 || k > N)
    return fail(DSK_ERR_INVALID, "dsk_allpairs_topk_tc: bad arguments");
  if (D % 64 || k > 8) return dsk_allpairs_topk(E, labels, N, D, k, idx, val, stream);  // exact CUDA-core path
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const float *G = nullptr, *norms = nullptr;
  int Npad = 0;
  rc = allpairs_gram(h, E, N, D, 0, N, s, &G, &norms, &Npad);
  if (!rc) {
    const float u = allpairs_unit_roundoff(h);
    dsk::allpairs_select_refine_kernel<false><<<(N + 7) / 8, 256, 0, s>>>(E, G, norms, labels, N, Npad, 0, N, D, pd_eps(D),
                                                                           k, u, idx, val);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(DSK_ERR_CUDA, "kernel launch failed: %s", cudaGetErrorString(e));
  }
  return rc;
}

static inline bool batch_hard_bad_range(int N, int row0, int rows) {
  return N < 2 || N > DSK_BATCH_HARD_MAX_N || row0 < 0 || rows < 1 || row0 > N - rows;
}

int32_t dsk_batch_hard_select_rows(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D,
                                   int32_t row0, int32_t rows, int64_t* pos_idx, int64_t* neg_idx, float* d_ap,
                                   float* d_an, uint8_t* valid, void* stream) {
  if (!E || !labels || !pos_idx || !neg_idx || !d_ap || !d_an || !valid || D <= 0 || batch_hard_bad_range(N, row0, rows))
    return fail(DSK_ERR_INVALID, "dsk_batch_hard_select_rows: bad arguments (N must be 2..%d, 0 <= row0, 1 <= rows, "
                "row0 + rows <= N; got N %d, row0 %d, rows %d)", DSK_BATCH_HARD_MAX_N, N, row0, rows);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const float eps = pd_eps(D);
  const int blocks = (rows + 7) / 8;
  if (h && D % 64 == 0) {  // tensor-core Gram + exact refinement of the negative
    int rc = check_handle(h);
    if (rc) return rc;
    const float *G = nullptr, *norms = nullptr;
    int Npad = 0;
    rc = allpairs_gram(h, E, N, D, row0, rows, s, &G, &norms, &Npad);
    if (rc) return rc;
    if (row0 == 0 && rows == N)
      dsk::allpairs_select_refine_kernel<false><<<blocks, 256, 0, s>>>(E, G, norms, labels, N, Npad, 0, N, D, eps, 1,
                                                                        allpairs_unit_roundoff(h), neg_idx, d_an);
    else
      dsk::allpairs_select_refine_kernel<true><<<blocks, 256, 0, s>>>(E, G, norms, labels, N, Npad, row0, rows, D, eps, 1,
                                                                       allpairs_unit_roundoff(h), neg_idx, d_an);
    KERNEL_CHECK();
    dsk::batch_hard_positive_kernel<false><<<blocks, 256, 0, s>>>(E, nullptr, labels, N, row0, rows, D, eps, pos_idx,
                                                                   d_ap, d_an, valid);
    KERNEL_CHECK();
  } else {  // exact CUDA-core rows x N distance matrix (the same bits)
    float* S = nullptr;
    CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&S), static_cast<size_t>(rows) * N * sizeof(float), s));
    dim3 g((N + 63) / 64, (rows + 63) / 64);
    dsk::allpairs_sqdist_kernel<<<g, 256, 0, s>>>(E, N, D, row0, rows, S);
    KERNEL_CHECK();
    dsk::topk_rows_kernel<<<blocks, 256, 0, s>>>(S, labels, N, row0, rows, eps, 1, neg_idx, d_an);
    KERNEL_CHECK();
    dsk::batch_hard_positive_kernel<true><<<blocks, 256, 0, s>>>(E, S, labels, N, row0, rows, D, eps, pos_idx, d_ap, d_an,
                                                                  valid);
    KERNEL_CHECK();
    CUDA_TRY(cudaFreeAsync(S, s));
  }
  return DSK_OK;
}

int32_t dsk_batch_hard_mean(const float* d_ap, const float* d_an, const uint8_t* valid, int32_t N, float margin,
                            float* loss, void* stream) {
  if (!d_ap || !d_an || !valid || !loss || N < 2 || N > DSK_BATCH_HARD_MAX_N)
    return fail(DSK_ERR_INVALID, "dsk_batch_hard_mean: bad arguments (N must be 2..%d, got %d)", DSK_BATCH_HARD_MAX_N, N);
  dsk::batch_hard_mean_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(d_ap, d_an, valid, N, margin, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_batch_hard_triplet(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D, float margin,
                               float* loss, int64_t* pos_idx, int64_t* neg_idx, float* d_ap, float* d_an,
                               uint8_t* valid, void* stream) {
  if (!E || !labels || !loss || !pos_idx || !neg_idx || !d_ap || !d_an || !valid || D <= 0 || N < 2 ||
      N > DSK_BATCH_HARD_MAX_N)
    return fail(DSK_ERR_INVALID, "dsk_batch_hard_triplet: bad arguments (N must be 2..%d, got %d)", DSK_BATCH_HARD_MAX_N, N);
  const int rc = dsk_batch_hard_select_rows(h, E, labels, N, D, 0, N, pos_idx, neg_idx, d_ap, d_an, valid, stream);
  return rc ? rc : dsk_batch_hard_mean(d_ap, d_an, valid, N, margin, loss, stream);
}

int32_t dsk_batch_hard_triplet_bwd_rows(const float* E, const int64_t* pos_idx, const int64_t* neg_idx,
                                        const float* d_ap, const float* d_an, const uint8_t* valid, int32_t N,
                                        int32_t D, int32_t row0, int32_t rows, float margin, const float* grad_loss,
                                        float* gE_rows, void* stream) {
  if (!E || !pos_idx || !neg_idx || !d_ap || !d_an || !grad_loss || !valid || !gE_rows || D <= 0 ||
      batch_hard_bad_range(N, row0, rows))
    return fail(DSK_ERR_INVALID, "dsk_batch_hard_triplet_bwd_rows: bad arguments (N must be 2..%d, 0 <= row0, "
                "1 <= rows, row0 + rows <= N; got N %d, row0 %d, rows %d)", DSK_BATCH_HARD_MAX_N, N, row0, rows);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* coef = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&coef), sizeof(float), s));
  dsk::batch_hard_coef_kernel<<<1, 1024, 0, s>>>(valid, N, grad_loss, coef);
  KERNEL_CHECK();
  dsk::batch_hard_bwd_kernel<<<rows, 128, 0, s>>>(E, pos_idx, neg_idx, d_ap, d_an, valid, N, D, row0, margin, coef,
                                                  gE_rows);
  KERNEL_CHECK();
  CUDA_TRY(cudaFreeAsync(coef, s));
  return DSK_OK;
}

int32_t dsk_batch_hard_triplet_bwd(const float* E, const int64_t* pos_idx, const int64_t* neg_idx, const float* d_ap,
                                   const float* d_an, int32_t N, int32_t D, float margin, const float* grad_loss,
                                   const uint8_t* valid, float* gE, void* stream) {
  if (!E || !pos_idx || !neg_idx || !d_ap || !d_an || !grad_loss || !valid || !gE || D <= 0 || N < 2 ||
      N > DSK_BATCH_HARD_MAX_N)
    return fail(DSK_ERR_INVALID, "dsk_batch_hard_triplet_bwd: bad arguments (N must be 2..%d, got %d)", DSK_BATCH_HARD_MAX_N, N);
  return dsk_batch_hard_triplet_bwd_rows(E, pos_idx, neg_idx, d_ap, d_an, valid, N, D, 0, N, margin, grad_loss, gE,
                                         stream);
}

int32_t dsk_allpairs_topk(const float* E, const int64_t* labels, int32_t N, int32_t D, int32_t k, int64_t* idx,
                          float* val, void* stream) {
  if (!E || !labels || !idx || !val || N <= 0 || D <= 0 || k <= 0 || k > N)
    return fail(DSK_ERR_INVALID, "dsk_allpairs_topk: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* S = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&S), static_cast<size_t>(N) * N * sizeof(float), s));
  dim3 g((N + 63) / 64, (N + 63) / 64);
  dsk::allpairs_sqdist_kernel<<<g, 256, 0, s>>>(E, N, D, 0, N, S);
  KERNEL_CHECK();
  dsk::topk_rows_kernel<<<(N + 7) / 8, 256, 0, s>>>(S, labels, N, 0, N, pd_eps(D), k, idx, val);
  KERNEL_CHECK();
  CUDA_TRY(cudaFreeAsync(S, s));
  return DSK_OK;
}

// ---- additive angular margin softmax ------------------------------------------------------------------------------
// The GEMMs of the cosine ops (AAM-softmax, GE2E, scoring) take fp16 operands whatever the handle's type: a bf16 hi/lo
// split keeps 16 bits, not 22.

// The AAM plan in slot P of h (h->aam) for (N, C, D).  A rebuild synchronises `s` (buffers in use are freed).
static int aam_plan(dsk_handle h, AamPlan& P, int N, int C, int D, cudaStream_t s, AamPlan** out) {
  *out = &P;
  return plan_acquire(P, {N, C, D}, s, [&]() -> int {
    const int Np = (N + 127) / 128 * 128, Cp = (C + 127) / 128 * 128;
    P.N = N;
    P.C = C;
    P.D = D;
    P.Np = Np;
    P.Cp = Cp;
    P.sc = (Cp + dsk::kAamSlice - 1) / dsk::kAamSlice;
    P.sn = (Np + dsk::kAamSlice - 1) / dsk::kAamSlice;
    const size_t d3 = 3ull * D;
    int rc = arena_alloc(&P.buf, {{&P.ea, Np * d3 * 2},                {&P.wb, Cp * d3 * 2},
                                  {&P.et, Np * d3 * 2},                {&P.wt, Cp * d3 * 2},
                                  {&P.da, 3ull * Np * Cp * 2},         {&P.dt, 3ull * Np * Cp * 2},
                                  {&P.nrm_e, Np * 4ull},               {&P.nrm_w, Cp * 4ull},
                                  {&P.gcos, 1ull * Np * Cp * 4},       {&P.dcos, 1ull * Np * Cp * 4},
                                  {&P.rinv, Np * 4ull},                {&P.cinv, Cp * 4ull},
                                  {&P.ge, 1ull * P.sc * Np * D * 4},   {&P.gw, 1ull * P.sn * Cp * D * 4},
                                  {&P.row_loss, Np * 4ull}}, s);
    if (!rc) rc = build_gemm(h, &P.fwd, P.ea, Np, P.wb, Cp, 3 * D, P.gcos, true);  // cos = E^ W^T, K = 3D
    // gE^ = dcos W^ (K = 3Cp) and gW^ = dcos^T E^ (K = 3Np)
    if (!rc) rc = build_sliced_gemm(h, &P.ge_gemm, P.da, Np, P.wt, D, Cp, P.ge);
    if (!rc) rc = build_sliced_gemm(h, &P.gw_gemm, P.dt, Cp, P.et, D, Np, P.gw);
    return rc;
  });
}

static int aam_check(dsk_handle h, bool ptrs_ok, int N, int C, int K, int D, float margin, float scale, int topk,
                     float topk_margin, const char* what) {
  if (!ptrs_ok || N < 1 || C < 2 || K < 1 || K > DSK_AAM_MAX_SUBCENTRES ||
      static_cast<int64_t>(C) * K > DSK_AAM_MAX_C || D < 64 || D % 64 || !std::isfinite(margin) || margin < 0.f ||
      !std::isfinite(scale) || !(scale > 0.f) || topk < 0 || topk > C - 1 || topk > DSK_AAM_MAX_TOPK ||
      !std::isfinite(topk_margin) || topk_margin < 0.f)
    return fail(DSK_ERR_INVALID, "%s: bad arguments (need non-null pointers, N >= 1, C >= 2, 1 <= K <= %d, C K <= %d, D "
                "a positive multiple of 64, finite margin >= 0 and scale > 0, 0 <= topk <= min(C - 1, %d), finite "
                "topk_margin >= 0; got N %d, C %d, K %d, D %d, margin %g, scale %g, topk %d, topk_margin %g)", what,
                DSK_AAM_MAX_SUBCENTRES, DSK_AAM_MAX_C, DSK_AAM_MAX_TOPK, N, C, K, D, margin, scale, topk, topk_margin);
  return check_handle(h);
}

static dsk::AamMargin aam_margin(float margin, float scale, float topk_margin) {
  const double m = margin, pi = 3.14159265358979323846;
  return {static_cast<float>(std::cos(m)), static_cast<float>(std::sin(m)), static_cast<float>(std::cos(pi - m)),
          static_cast<float>(std::sin(pi - m) * m), scale, static_cast<float>(std::cos(double(topk_margin))),
          static_cast<float>(std::sin(double(topk_margin)))};
}

// Rows X[0, n) (D wide) of one operand of a cosine GEMM: their norms nrm (taken by cos_prep when `norm`, else already
// there), and the hi/lo images cos_prep writes of them, padded with zero rows to n_pad: `img` row-major [n_pad][3D],
// `imgT` transposed and K-sliced (either may be NULL).
struct CosRows {
  const float* X;
  int n, n_pad;
  float* nrm;
  bool norm;
  uint16_t *img, *imgT;
};

// Operand prep of a cosine GEMM on `s`: the norms of the A-side rows a and the B-side rows b, then their images.  Either
// side may be NULL.
static int cos_prep(int D, const CosRows* a, const CosRows* b, cudaStream_t s) {
  for (const CosRows* r : {a, b})
    if (r && r->norm) {
      dsk::aam_norm_kernel<<<(r->n + 7) / 8, 256, 0, s>>>(r->X, r->n, D, r->nrm);
      KERNEL_CHECK();
    }
  for (const CosRows* r : {a, b})
    if (r && (r->img || r->imgT)) {
      dsk::aam_split_kernel<<<dim3(D / 64, r->n_pad / 32), 256, 0, s>>>(r->X, r->nrm, r->n, r->n_pad, D, r == a ? 1 : 0,
                                                                        r->img, r->imgT);
      KERNEL_CHECK();
    }
  return DSK_OK;
}

// norms of E and W, and their hi/lo operand images (forward: row-major; backward: transposed)
static int aam_prep(const AamPlan& P, const float* E, const float* W, bool backward, cudaStream_t s) {
  const CosRows e{E, P.N, P.Np, P.nrm_e, true, backward ? nullptr : P.ea, backward ? P.et : nullptr};
  const CosRows w{W, P.C, P.Cp, P.nrm_w, true, backward ? nullptr : P.wb, backward ? P.wt : nullptr};
  return cos_prep(P.D, &e, &w, s);
}

static int aam_forward(dsk_handle h, const float* E, const float* W, const int64_t* labels, int N, int C, int K, int D,
                       float margin, float scale, int topk, float topk_margin, float* loss, float* cos, float* lse,
                       uint8_t* sub, int32_t* top, void* stream, const char* what) {
  int rc = aam_check(h, E && W && labels && loss && cos && lse && (K == 1 || sub) && (topk == 0 || top), N, C, K, D,
                     margin, scale, topk, topk_margin, what);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AamPlan* P = nullptr;
  if ((rc = aam_plan(h, h->aam, N, C * K, D, s, &P))) return rc;
  if ((rc = aam_prep(*P, E, W, false, s))) return rc;
  for (const ConvLaunch& L : P->fwd)
    if ((rc = launch_conv(L, s))) return rc;
  dsk::aam_rows_kernel<<<N, 256, 0, s>>>(P->gcos, P->Cp, E, W, D, labels, C, K, topk,
                                         aam_margin(margin, scale, topk_margin), cos, sub, top, lse, P->row_loss);
  KERNEL_CHECK();
  dsk::mean_rows_kernel<<<1, 1024, 0, s>>>(P->row_loss, N, N, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

static int aam_backward(dsk_handle h, const float* E, const float* W, const int64_t* labels, const float* cos,
                        const float* lse, const uint8_t* sub, const int32_t* top, int N, int C, int K, int D,
                        float margin, float scale, int topk, float topk_margin, const float* grad_loss, float* gE,
                        float* gW, void* stream, const char* what) {
  int rc = aam_check(h, E && W && labels && cos && lse && grad_loss && gE && gW && (K == 1 || sub) && (topk == 0 || top),
                     N, C, K, D, margin, scale, topk, topk_margin, what);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AamPlan* P = nullptr;
  if ((rc = aam_plan(h, h->aam, N, C * K, D, s, &P))) return rc;
  if ((rc = aam_prep(*P, E, W, true, s))) return rc;
  dsk::aam_dcos_kernel<<<P->Np, 256, 0, s>>>(cos, sub, top, lse, labels, N, C, K, P->Cp, topk,
                                             aam_margin(margin, scale, topk_margin), grad_loss, P->dcos, P->da, P->rinv);
  KERNEL_CHECK();
  dsk::aam_dcos_t_kernel<<<P->Cp / 32, 256, 0, s>>>(P->dcos, P->Np, P->Cp, P->dt, P->cinv);
  KERNEL_CHECK();
  for (const ConvLaunch& L : P->ge_gemm)
    if ((rc = launch_conv(L, s))) return rc;
  for (const ConvLaunch& L : P->gw_gemm)
    if ((rc = launch_conv(L, s))) return rc;
  dsk::aam_normalize_bwd_kernel<<<(N + 7) / 8, 256, 0, s>>>(E, P->nrm_e, P->ge, P->sc, static_cast<long>(P->Np) * D,
                                                            P->rinv, N, D, gE);
  KERNEL_CHECK();
  dsk::aam_normalize_bwd_kernel<<<(C * K + 7) / 8, 256, 0, s>>>(W, P->nrm_w, P->gw, P->sn,
                                                                static_cast<long>(P->Cp) * D, P->cinv, C * K, D, gW);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_aam_softmax_sc(dsk_handle h, const float* E, const float* W, const int64_t* labels, int32_t N, int32_t C,
                           int32_t K, int32_t D, float margin, float scale, int32_t topk, float topk_margin, float* loss,
                           float* cos, float* lse, uint8_t* sub, int32_t* top, void* stream) {
  return aam_forward(h, E, W, labels, N, C, K, D, margin, scale, topk, topk_margin, loss, cos, lse, sub, top, stream,
                     "dsk_aam_softmax_sc");
}

int32_t dsk_aam_softmax_sc_bwd(dsk_handle h, const float* E, const float* W, const int64_t* labels, const float* cos,
                               const float* lse, const uint8_t* sub, const int32_t* top, int32_t N, int32_t C, int32_t K,
                               int32_t D, float margin, float scale, int32_t topk, float topk_margin,
                               const float* grad_loss, float* gE, float* gW, void* stream) {
  return aam_backward(h, E, W, labels, cos, lse, sub, top, N, C, K, D, margin, scale, topk, topk_margin, grad_loss, gE,
                      gW, stream, "dsk_aam_softmax_sc_bwd");
}

int32_t dsk_aam_softmax(dsk_handle h, const float* E, const float* W, const int64_t* labels, int32_t N, int32_t C,
                        int32_t D, float margin, float scale, float* loss, float* cos, float* lse, void* stream) {
  return aam_forward(h, E, W, labels, N, C, 1, D, margin, scale, 0, 0.f, loss, cos, lse, nullptr, nullptr, stream,
                     "dsk_aam_softmax");
}

int32_t dsk_aam_softmax_bwd(dsk_handle h, const float* E, const float* W, const int64_t* labels, const float* cos,
                            const float* lse, int32_t N, int32_t C, int32_t D, float margin, float scale,
                            const float* grad_loss, float* gE, float* gW, void* stream) {
  return aam_backward(h, E, W, labels, cos, lse, nullptr, nullptr, N, C, 1, D, margin, scale, 0, 0.f, grad_loss, gE, gW,
                      stream, "dsk_aam_softmax_bwd");
}

int32_t dsk_aam_subcentre_cos(const float* E, const float* W, const int64_t* labels, int32_t N, int32_t C, int32_t K,
                              int32_t D, float* out, void* stream) {
  if (!E || !W || !labels || !out || N < 1 || C < 1 || K < 1 || K > DSK_AAM_MAX_SUBCENTRES || D < 1 ||
      static_cast<int64_t>(C) * K > INT32_MAX)
    return fail(DSK_ERR_INVALID, "dsk_aam_subcentre_cos: bad arguments (need non-null pointers, N >= 1, C >= 1, "
                "1 <= K <= %d, D >= 1; got N %d, C %d, K %d, D %d)", DSK_AAM_MAX_SUBCENTRES, N, C, K, D);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::aam_subcentre_cos_kernel<<<N, 256, 0, s>>>(E, W, labels, C, K, D, out);
  KERNEL_CHECK();
  return DSK_OK;
}

// ---- the class-sharded AAM-softmax --------------------------------------------------------------------------------
// The shard [c0, c1) of C classes: 0 <= c0 < c1 <= C, c0 a multiple of 128 and c1 one too unless it is C, (c1 - c0) K
// within the per-call cap; the other arguments as aam_check.  R ranks, nb record blocks (stages 3 and 4).
static int aam_shard_check(bool ptrs_ok, int R, int N, int C, int c0, int c1, int K, int D, float margin, float scale,
                           int topk, float topk_margin, const char* what) {
  const int B = dsk::kAamShardBlock;
  if (!ptrs_ok || R < 1 || N < 1 || C < 2 || K < 1 || K > DSK_AAM_MAX_SUBCENTRES || c0 < 0 || c0 % B || c1 <= c0 ||
      c1 > C || (c1 % B && c1 != C) || static_cast<int64_t>(c1 - c0) * K > DSK_AAM_MAX_C || D < 64 || D % 64 ||
      !std::isfinite(margin) || margin < 0.f || !std::isfinite(scale) || !(scale > 0.f) || topk < 0 || topk > C - 1 ||
      topk > DSK_AAM_MAX_TOPK || !std::isfinite(topk_margin) || topk_margin < 0.f)
    return fail(DSK_ERR_INVALID, "%s: bad arguments (need non-null pointers, R >= 1, N >= 1, C >= 2, 1 <= K <= %d, a "
                "class range 0 <= c0 < c1 <= C with c0 and c1 (unless c1 = C) multiples of %d and (c1 - c0) K <= %d, D a "
                "positive multiple of 64, finite margin >= 0 and scale > 0, 0 <= topk <= min(C - 1, %d), finite "
                "topk_margin >= 0; got R %d, N %d, C %d, c0 %d, c1 %d, K %d, D %d, margin %g, scale %g, topk %d, "
                "topk_margin %g)", what, DSK_AAM_MAX_SUBCENTRES, B, DSK_AAM_MAX_C, DSK_AAM_MAX_TOPK, R, N, C, c0, c1, K,
                D, margin, scale, topk, topk_margin);
  return DSK_OK;
}

int32_t dsk_aam_shard_cos(dsk_handle h, const float* E, const float* W, const int64_t* labels, int32_t N, int32_t C,
                          int32_t c0, int32_t c1, int32_t K, int32_t D, int32_t topk, float* cos, uint8_t* sub,
                          uint64_t* keys, void* stream) {
  int rc = aam_shard_check(E && W && labels && cos && (K == 1 || sub) && (topk == 0 || keys), 1, N, C, c0, c1, K, D,
                           0.f, 1.f, topk, 0.f, "dsk_aam_shard_cos");
  if (rc || (rc = check_handle(h))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int Cr = c1 - c0;
  AamPlan* P = nullptr;
  if ((rc = aam_plan(h, h->aam, N, Cr * K, D, s, &P))) return rc;
  if ((rc = aam_prep(*P, E, W, false, s))) return rc;
  for (const ConvLaunch& L : P->fwd)
    if ((rc = launch_conv(L, s))) return rc;
  dsk::aam_shard_cos_kernel<<<N, 256, 0, s>>>(P->gcos, P->Cp, E, W, D, labels, c0, Cr, K, topk, cos, sub,
                                              reinterpret_cast<unsigned long long*>(keys));
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_aam_shard_merge(const float* cos, const int64_t* labels, const uint64_t* keys, int32_t R, int32_t N,
                            int32_t C, int32_t c0, int32_t c1, int32_t topk, float margin, float scale,
                            float topk_margin, int32_t* top, uint64_t* thr, float* mloc, void* stream) {
  if (int rc = aam_shard_check(cos && labels && mloc && (topk == 0 || (keys && top && thr)), R, N, C, c0, c1, 1, 64,
                               margin, scale, topk, topk_margin, "dsk_aam_shard_merge"))
    return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::aam_shard_merge_kernel<<<N, 256, 0, s>>>(cos, labels, reinterpret_cast<const unsigned long long*>(keys), R, N, c0,
                                                c1 - c0, topk, aam_margin(margin, scale, topk_margin), top,
                                                reinterpret_cast<unsigned long long*>(thr), mloc);
  KERNEL_CHECK();
  return DSK_OK;
}

static bool aam_shard_nb_ok(int nb, int c0, int c1) {
  return nb >= (c1 - c0 + dsk::kAamShardBlock - 1) / dsk::kAamShardBlock && nb <= 1 << 20;
}

int32_t dsk_aam_shard_partials(const float* cos, const int64_t* labels, const uint64_t* thr, const float* maxima,
                               int32_t R, int32_t N, int32_t C, int32_t c0, int32_t c1, int32_t topk, int32_t nb,
                               float margin, float scale, float topk_margin, float* m, float* rec, void* stream) {
  if (int rc = aam_shard_check(cos && labels && maxima && m && rec && (topk == 0 || thr), R, N, C, c0, c1, 1, 64, margin,
                               scale, topk, topk_margin, "dsk_aam_shard_partials"))
    return rc;
  if (!aam_shard_nb_ok(nb, c0, c1))
    return fail(DSK_ERR_INVALID, "dsk_aam_shard_partials: nb %d is not in [ceil((c1 - c0) / %d), 2^20] for c0 %d, c1 %d",
                nb, dsk::kAamShardBlock, c0, c1);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::aam_shard_partials_kernel<<<N, dsk::kAamShardBlock, 0, s>>>(
      cos, labels, reinterpret_cast<const unsigned long long*>(thr), maxima, R, N, c0, c1 - c0, topk, nb,
      aam_margin(margin, scale, topk_margin), m, rec);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_aam_shard_finish(const float* rec, const float* m, const int64_t* labels, int32_t R, int32_t N, int32_t C,
                             int32_t nb, float* loss, float* lse, float* row_loss, float* den, void* stream) {
  if (!rec || !m || !labels || !loss || !lse || !row_loss || !den || R < 1 || N < 1 || C < 2 || nb < 1 ||
      nb > 1 << 20 || static_cast<int64_t>(R) * nb * dsk::kAamShardBlock < C)
    return fail(DSK_ERR_INVALID, "dsk_aam_shard_finish: bad arguments (need non-null pointers, R >= 1, N >= 1, C >= 2, "
                "1 <= nb <= 2^20 with R nb %d >= C; got R %d, N %d, C %d, nb %d)", dsk::kAamShardBlock, R, N, C, nb);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::aam_shard_finish_kernel<<<(N + 7) / 8, 256, 0, s>>>(rec, m, labels, R, N, C, nb, lse, row_loss, den);
  KERNEL_CHECK();
  dsk::mean_rows_kernel<<<1, 1024, 0, s>>>(row_loss, N, N, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_aam_shard_bwd(dsk_handle h, const float* E, const float* W, const int64_t* labels, const float* cos,
                          const uint8_t* sub, const uint64_t* thr, const float* m, const float* den, int32_t N,
                          int32_t C, int32_t c0, int32_t c1, int32_t K, int32_t D, float margin, float scale,
                          int32_t topk, float topk_margin, const float* grad_loss, float* gW, float* gE_part,
                          void* stream) {
  int rc = aam_shard_check(E && W && labels && cos && (K == 1 || sub) && (topk == 0 || thr) && m && den && grad_loss &&
                               gW && gE_part, 1, N, C, c0, c1, K, D, margin, scale, topk, topk_margin,
                           "dsk_aam_shard_bwd");
  if (rc || (rc = check_handle(h))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int CK = (c1 - c0) * K;
  AamPlan* P = nullptr;
  if ((rc = aam_plan(h, h->aam, N, CK, D, s, &P))) return rc;
  if ((rc = aam_prep(*P, E, W, true, s))) return rc;
  dsk::aam_shard_dcos_kernel<<<P->Np, 256, 0, s>>>(cos, sub, reinterpret_cast<const unsigned long long*>(thr), m, den,
                                                   labels, N, c0, c1 - c0, K, P->Cp, topk,
                                                   aam_margin(margin, scale, topk_margin), grad_loss, P->dcos, P->da,
                                                   P->rinv);
  KERNEL_CHECK();
  dsk::aam_dcos_t_kernel<<<P->Cp / 32, 256, 0, s>>>(P->dcos, P->Np, P->Cp, P->dt, P->cinv);
  KERNEL_CHECK();
  for (const ConvLaunch& L : P->ge_gemm)
    if ((rc = launch_conv(L, s))) return rc;
  for (const ConvLaunch& L : P->gw_gemm)
    if ((rc = launch_conv(L, s))) return rc;
  const size_t nd = static_cast<size_t>(N) * D;
  dsk::aam_shard_gpart_kernel<<<static_cast<unsigned>((nd + 255) / 256), 256, 0, s>>>(
      P->ge, P->sc, static_cast<size_t>(P->Np) * D, P->rinv, N, D, gE_part);
  KERNEL_CHECK();
  dsk::aam_normalize_bwd_kernel<<<(CK + 7) / 8, 256, 0, s>>>(W, P->nrm_w, P->gw, P->sn, static_cast<long>(P->Cp) * D,
                                                             P->cinv, CK, D, gW);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_aam_shard_bwd_rows(const float* E, const float* parts, int32_t R, int32_t n, int32_t D, float* gE,
                               void* stream) {
  if (!E || !parts || !gE || R < 1 || n < 1 || D < 1)
    return fail(DSK_ERR_INVALID, "dsk_aam_shard_bwd_rows: bad arguments (need non-null pointers, R >= 1, n >= 1, "
                "D >= 1; got R %d, n %d, D %d)", R, n, D);
  dsk::aam_shard_rows_bwd_kernel<<<(n + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(E, parts, R, n, D, gE);
  KERNEL_CHECK();
  return DSK_OK;
}

// ---- generalised end-to-end (GE2E) loss ---------------------------------------------------------------------------
// The handle's GE2E plan for (N, P, D, row0, rows).  A rebuild synchronises `s` (buffers in use are freed).
static int ge2e_plan(dsk_handle h, int N, int P, int D, int row0, int rows, cudaStream_t s, Ge2ePlan** out) {
  Ge2ePlan& G = h->ge2e;
  *out = &G;
  return plan_acquire(G, {N, P, D, row0, rows}, s, [&]() -> int {
    const int Np = (N + 127) / 128 * 128, Rp = (rows + 127) / 128 * 128, Cp = (P + 127) / 128 * 128;
    G.N = N;
    G.P = P;
    G.D = D;
    G.Np = Np;
    G.Rp = Rp;
    G.Cp = Cp;
    G.sc = (Cp + dsk::kAamSlice - 1) / dsk::kAamSlice;
    G.sn = (Np + dsk::kAamSlice - 1) / dsk::kAamSlice;
    const size_t d3 = 3ull * D, pd = static_cast<size_t>(P) * D * 4;
    const size_t whole = row0 == 0 && rows == N ? 1 : 0;
    // the arena's zeros: the rows [rows, Rp) of the dcos image, and (written by dsk_ge2e_bwd's path) the workspace rows
    // [N, Np), are never written again
    int rc = arena_alloc(&G.buf, {{&G.row_loss, whole * N * 4},       {&G.tdc, whole * N * 4},
                                  {&G.part, whole * 2 * N * 8},
                                  {&G.cent, pd},                      {&G.nr64, N * 8ull},
                                  {&G.nrm_e, N * 4ull},               {&G.nrm_c, P * 4ull},
                                  {&G.ea, Rp * d3 * 2},               {&G.cb, Cp * d3 * 2},
                                  {&G.et, Np * d3 * 2},               {&G.ct, Cp * d3 * 2},
                                  {&G.da, 3ull * Rp * Cp * 2},        {&G.dt, 3ull * Np * Cp * 2},
                                  {&G.gcos, 1ull * Rp * Cp * 4},      {&G.dcos, 1ull * Np * Cp * 4},
                                  {&G.rinv, Rp * 4ull},               {&G.cinv, Cp * 4ull},
                                  {&G.ge, 1ull * G.sc * Rp * D * 4},  {&G.gc, 1ull * G.sn * Cp * D * 4},
                                  {&G.gcent, pd},                     {&G.own, 1ull * Rp * D * 4},
                                  {&G.xg, 1ull * N * D * 4},          {&G.ones, Rp * 4ull}}, s);
    if (rc) return rc;
    const std::vector<float> ones(Rp, 1.f);
    CUDA_TRY(cudaMemcpyAsync(G.ones, ones.data(), Rp * 4ull, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    // cos = E^ C^T for the range (K = 3D); gE^ = dcos C^ for the range (K = 3Cp) and gC^ = dcos^T E^ over all N rows
    // (K = 3Np)
    rc = build_gemm(h, &G.fwd, G.ea, Rp, G.cb, Cp, 3 * D, G.gcos, true);
    if (!rc) rc = build_sliced_gemm(h, &G.ge_gemm, G.da, Rp, G.ct, D, Cp, G.ge);
    if (!rc) rc = build_sliced_gemm(h, &G.gc_gemm, G.dt, Cp, G.et, D, Np, G.gc);
    return rc;
  });
}

// The argument checks of the GE2E entry points, before any launch.  An op without a D, V or method passes 64, 1 and
// DSK_GE2E_SOFTMAX for them; the whole-batch ops pass the range (0, N).
static int ge2e_check(bool ptrs_ok, int N, int D, int P, int V, int method, int row0, int rows, const char* what) {
  if (!ptrs_ok || N < 2 || P < 2 || P > DSK_AAM_MAX_C || P > N || D < 64 || D % 64 || V < 1 || V > N ||
      (method != DSK_GE2E_SOFTMAX && method != DSK_GE2E_CONTRAST) || row0 < 0 || rows < 1 || row0 > N - rows)
    return fail(DSK_ERR_INVALID, "%s: bad arguments (need non-null pointers, 2 <= P <= min(N, %d), D a positive multiple "
                "of 64, 1 <= V <= N, method DSK_GE2E_SOFTMAX or DSK_GE2E_CONTRAST, 0 <= row0, 1 <= rows and "
                "row0 + rows <= N; got N %d, P %d, D %d, V %d, method %d, row0 %d, rows %d)", what, DSK_AAM_MAX_C, N,
                P, D, V, method, row0, rows);
  return DSK_OK;
}

// inclusive centroids, fp64 row norms and the centroids' fp32 norms: always over the whole batch
static int ge2e_centroids(const Ge2ePlan& G, const float* E, const int64_t* order, const int64_t* offsets,
                          cudaStream_t s) {
  dsk::class_centroids_kernel<<<dim3(G.P, (G.D + 255) / 256), 256, 0, s>>>(E, G.N, G.D, order, offsets, G.cent);
  KERNEL_CHECK();
  dsk::ge2e_norm64_kernel<<<(G.N + 7) / 8, 256, 0, s>>>(E, G.N, G.D, G.nr64);
  KERNEL_CHECK();
  const CosRows c{G.cent, G.P, G.Cp, G.nrm_c, true, nullptr, nullptr};
  return cos_prep(G.D, nullptr, &c, s);
}

// dsk_ge2e_rows after its checks
static int ge2e_rows_run(dsk_handle h, const float* E, int N, int D, const int64_t* order, const int64_t* offsets,
                         const int64_t* col, int P, const float* w, const float* b, int method, int row0, int rows,
                         float* cos, float* rec, float* row_loss, cudaStream_t s) {
  Ge2ePlan* G = nullptr;
  int rc = ge2e_plan(h, N, P, D, row0, rows, s, &G);
  if (rc || (rc = ge2e_centroids(*G, E, order, offsets, s))) return rc;
  const CosRows e{E + static_cast<size_t>(row0) * D, rows, G->Rp, G->nrm_e + row0, true, G->ea, nullptr};
  const CosRows c{G->cent, P, G->Cp, G->nrm_c, false, G->cb, nullptr};
  if ((rc = cos_prep(D, &e, &c, s))) return rc;
  for (const ConvLaunch& L : G->fwd)
    if ((rc = launch_conv(L, s))) return rc;
  dsk::ge2e_rows_kernel<<<rows, 256, 0, s>>>(G->gcos, G->Cp, E, D, G->nr64, order, offsets, col, P, w, b, method, row0,
                                             cos, rec, row_loss);
  KERNEL_CHECK();
  return DSK_OK;
}

// dsk_ge2e_dcos_rows after its checks; part: a [2][rows] fp64 workspace.  With G (the plan of the range (0, N), for
// dsk_ge2e_bwd) the rows go straight into G's zero-padded dcos workspace and gE^ image instead of `dcos`.
static int ge2e_dcos_run(const float* cos, const float* rec, const int64_t* offsets, const int64_t* col, int P, int V,
                         const float* w, const float* b, int method, const float* grad_loss, int row0, int rows,
                         float* dcos, float* tdc, float* gw, float* gb, double* part, Ge2ePlan* G, cudaStream_t s) {
  if (G)
    dsk::ge2e_dcos_rows_kernel<<<rows, 256, 0, s>>>(cos, rec, offsets, col, row0, P, V, w, b, method, grad_loss,
                                                    G->dcos, G->Cp, tdc, part, G->Cp, G->Rp, G->da, G->rinv);
  else
    dsk::ge2e_dcos_rows_kernel<<<rows, 256, 0, s>>>(cos, rec, offsets, col, row0, P, V, w, b, method, grad_loss, dcos,
                                                    P, tdc, part, P, 0, nullptr, nullptr);
  KERNEL_CHECK();
  dsk::ge2e_scalars_kernel<<<1, 256, 0, s>>>(part, rows, w, method, gw, gb);
  KERNEL_CHECK();
  return DSK_OK;
}

// dsk_ge2e_bwd_rows after its checks; dcos == NULL: the plan's dcos workspace and gE^ image are already built (by
// ge2e_dcos_run with the plan, in dsk_ge2e_bwd)
static int ge2e_bwd_rows_run(dsk_handle h, const float* E, int N, int D, const int64_t* order, const int64_t* offsets,
                             const int64_t* col, int P, const float* dcos, const float* tdc, int row0, int rows,
                             float* gE_rows, cudaStream_t s) {
  Ge2ePlan* G = nullptr;
  int rc = ge2e_plan(h, N, P, D, row0, rows, s, &G);
  if (rc || (rc = ge2e_centroids(*G, E, order, offsets, s))) return rc;
  const int Np = G->Np, Rp = G->Rp, Cp = G->Cp;
  const CosRows e{E, N, Np, G->nrm_e, true, nullptr, G->et};
  const CosRows c{G->cent, P, Cp, G->nrm_c, false, nullptr, G->ct};
  if ((rc = cos_prep(D, &e, &c, s))) return rc;
  if (dcos) {
    dsk::ge2e_dcos_img_kernel<<<Np, 256, 0, s>>>(dcos, N, P, Cp, row0, rows, Rp, G->dcos, G->da, G->rinv);
    KERNEL_CHECK();
  }
  dsk::aam_dcos_t_kernel<<<Cp / 32, 256, 0, s>>>(G->dcos, Np, Cp, G->dt, G->cinv);
  KERNEL_CHECK();
  for (const ConvLaunch& L : G->ge_gemm)  // dcos C^ for the range (target column zeroed)
    if ((rc = launch_conv(L, s))) return rc;
  for (const ConvLaunch& L : G->gc_gemm)  // dcos^T E^ over all N rows: the gradient w.r.t. the normalised centroids
    if ((rc = launch_conv(L, s))) return rc;
  dsk::aam_normalize_bwd_kernel<<<(P + 7) / 8, 256, 0, s>>>(G->cent, G->nrm_c, G->gc, G->sn, static_cast<long>(Cp) * D,
                                                            G->cinv, P, D, G->gcent);
  KERNEL_CHECK();
  dsk::ge2e_excl_bwd_kernel<<<N, 256, 0, s>>>(E, D, G->nr64, order, offsets, col, tdc, row0, rows, G->own, G->xg);
  KERNEL_CHECK();
  dsk::ge2e_gather_kernel<<<dim3(rows, (D + 255) / 256), 256, 0, s>>>(G->ge, G->sc, static_cast<long>(Rp) * D, G->rinv,
                                                                      G->gcent, order, offsets, col, G->xg, D, row0,
                                                                      G->own);
  KERNEL_CHECK();
  dsk::aam_normalize_bwd_kernel<<<(rows + 7) / 8, 256, 0, s>>>(E + static_cast<size_t>(row0) * D, G->nrm_e + row0,
                                                               G->own, 1, 0, G->ones, rows, D, gE_rows);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_ge2e_rows(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                      const int64_t* col, int32_t P, int32_t V, const float* w, const float* b, int32_t method,
                      int32_t row0, int32_t rows, float* cos, float* rec, float* row_loss, void* stream) {
  int rc = ge2e_check(E && order && offsets && col && w && b && cos && rec && row_loss, N, D, P, V, method, row0, rows,
                      "dsk_ge2e_rows");
  if (rc || (rc = check_handle(h))) return rc;
  return ge2e_rows_run(h, E, N, D, order, offsets, col, P, w, b, method, row0, rows, cos, rec, row_loss,
                       static_cast<cudaStream_t>(stream));
}

int32_t dsk_ge2e_mean(const float* row_loss, int32_t N, int32_t V, float* loss, void* stream) {
  if (!row_loss || !loss || N < 2 || V < 1 || V > N)
    return fail(DSK_ERR_INVALID, "dsk_ge2e_mean: bad arguments (need non-null pointers, N >= 2 and 1 <= V <= N; got N "
                "%d, V %d)", N, V);
  dsk::mean_rows_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(row_loss, N, V, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_ge2e_dcos_rows(const float* cos, const float* rec, int32_t N, const int64_t* offsets, const int64_t* col,
                           int32_t P, int32_t V, const float* w, const float* b, int32_t method, const float* grad_loss,
                           int32_t row0, int32_t rows, float* dcos, float* tdc, float* gw, float* gb, void* stream) {
  int rc = ge2e_check(cos && rec && offsets && col && w && b && grad_loss && dcos && tdc && gw && gb, N, 64, P, V,
                      method, row0, rows, "dsk_ge2e_dcos_rows");
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  double* part = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&part), 2ull * rows * sizeof(double), s));
  rc = ge2e_dcos_run(cos, rec, offsets, col, P, V, w, b, method, grad_loss, row0, rows, dcos, tdc, gw, gb, part,
                     nullptr, s);
  CUDA_TRY(cudaFreeAsync(part, s));
  return rc;
}

int32_t dsk_ge2e_bwd_rows(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order,
                          const int64_t* offsets, const int64_t* col, int32_t P, const float* dcos, const float* tdc,
                          int32_t row0, int32_t rows, float* gE_rows, void* stream) {
  int rc = ge2e_check(E && order && offsets && col && dcos && tdc && gE_rows, N, D, P, 1, DSK_GE2E_SOFTMAX, row0, rows,
                      "dsk_ge2e_bwd_rows");
  if (rc || (rc = check_handle(h))) return rc;
  return ge2e_bwd_rows_run(h, E, N, D, order, offsets, col, P, dcos, tdc, row0, rows, gE_rows,
                           static_cast<cudaStream_t>(stream));
}

int32_t dsk_ge2e(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                 const int64_t* col, int32_t P, int32_t V, const float* w, const float* b, int32_t method, float* loss,
                 float* cos, float* rec, void* stream) {
  int rc = ge2e_check(E && order && offsets && col && w && b && loss && cos && rec, N, D, P, V, method, 0, N, "dsk_ge2e");
  if (rc || (rc = check_handle(h))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Ge2ePlan* G = nullptr;
  if ((rc = ge2e_plan(h, N, P, D, 0, N, s, &G))) return rc;
  rc = ge2e_rows_run(h, E, N, D, order, offsets, col, P, w, b, method, 0, N, cos, rec, G->row_loss, s);
  return rc ? rc : dsk_ge2e_mean(G->row_loss, N, V, loss, stream);
}

int32_t dsk_ge2e_bwd(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                     const int64_t* col, int32_t P, int32_t V, const float* w, const float* b, int32_t method,
                     const float* cos, const float* rec, const float* grad_loss, float* gE, float* gw, float* gb,
                     void* stream) {
  int rc = ge2e_check(E && order && offsets && col && w && b && cos && rec && grad_loss && gE && gw && gb, N, D, P, V,
                      method, 0, N, "dsk_ge2e_bwd");
  if (rc || (rc = check_handle(h))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Ge2ePlan* G = nullptr;
  if ((rc = ge2e_plan(h, N, P, D, 0, N, s, &G))) return rc;
  // the dcos rows of all N go straight into the padded workspace and the gE^ image: no (N, P) round trip
  rc = ge2e_dcos_run(cos, rec, offsets, col, P, V, w, b, method, grad_loss, 0, N, nullptr, G->tdc, gw, gb, G->part, G,
                     s);
  return rc ? rc : ge2e_bwd_rows_run(h, E, N, D, order, offsets, col, P, nullptr, G->tdc, 0, N, gE, s);
}

// ---- supervised-contrastive loss ----------------------------------------------------------------------------------
static int supcon_check(dsk_handle h, bool ptrs_ok, int N, int D, int V, float tau, const char* what) {
  if (!ptrs_ok || N < 2 || N > DSK_SUPCON_MAX_N || D < 64 || D % 64 || V < 1 || V > N || !std::isfinite(tau) ||
      !(tau > 0.f))
    return fail(DSK_ERR_INVALID, "%s: bad arguments (need non-null pointers, 2 <= N <= %d, D a positive multiple of 64, "
                "1 <= V <= N and a finite tau > 0; got N %d, D %d, V %d, tau %g)", what, DSK_SUPCON_MAX_N, N, D, V, tau);
  return check_handle(h);
}

// The handle's supervised-contrastive plan (the AAM plan for (N, N, D) in its own slot) and E's norms and operand
// images, on both sides of its GEMMs (forward: row-major; backward: transposed)
static int supcon_prep(dsk_handle h, const float* E, int N, int D, bool backward, cudaStream_t s, AamPlan** out) {
  if (int rc = aam_plan(h, h->supcon, N, N, D, s, out)) return rc;
  AamPlan& P = **out;
  const CosRows a{E, N, P.Np, P.nrm_e, true, backward ? nullptr : P.ea, backward ? P.et : nullptr};
  const CosRows b{E, N, P.Cp, P.nrm_e, false, backward ? nullptr : P.wb, backward ? P.wt : nullptr};
  return cos_prep(D, &a, &b, s);
}

int32_t dsk_supcon(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D, int32_t V, float tau,
                   float* loss, float* cos, float* lse, void* stream) {
  int rc = supcon_check(h, E && labels && loss && cos && lse, N, D, V, tau, "dsk_supcon");
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AamPlan* P = nullptr;
  if ((rc = supcon_prep(h, E, N, D, false, s, &P))) return rc;
  for (const ConvLaunch& L : P->fwd)
    if ((rc = launch_conv(L, s))) return rc;
  dsk::supcon_rows_kernel<<<N, 256, 0, s>>>(P->gcos, P->Cp, E, D, labels, N, 1.0 / tau, cos, lse, P->row_loss);
  KERNEL_CHECK();
  dsk::mean_rows_kernel<<<1, 1024, 0, s>>>(P->row_loss, N, V, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_supcon_bwd(dsk_handle h, const float* E, const int64_t* labels, const float* cos, const float* lse,
                       int32_t N, int32_t D, int32_t V, float tau, const float* grad_loss, float* gE, void* stream) {
  int rc = supcon_check(h, E && labels && cos && lse && grad_loss && gE, N, D, V, tau, "dsk_supcon_bwd");
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AamPlan* P = nullptr;
  if ((rc = supcon_prep(h, E, N, D, true, s, &P))) return rc;
  dsk::supcon_dcos_kernel<<<P->Np, 256, 0, s>>>(cos, lse, labels, N, V, 1.0 / tau, grad_loss, P->Cp, P->dcos, P->da,
                                                P->rinv);
  KERNEL_CHECK();
  dsk::aam_dcos_t_kernel<<<P->Cp / 32, 256, 0, s>>>(P->dcos, P->Np, P->Cp, P->dt, P->cinv);
  KERNEL_CHECK();
  for (const ConvLaunch& L : P->ge_gemm)  // dC E^
    if ((rc = launch_conv(L, s))) return rc;
  for (const ConvLaunch& L : P->gw_gemm)  // dC^T E^
    if ((rc = launch_conv(L, s))) return rc;
  // the two products un-scaled into parts [2][N][D] (dC E^ first), added in that order by the Jacobian kernel
  const size_t nd = static_cast<size_t>(N) * D;
  float* parts = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&parts), 2 * nd * sizeof(float), s));
  const unsigned grid = static_cast<unsigned>((nd + 255) / 256);
  dsk::aam_shard_gpart_kernel<<<grid, 256, 0, s>>>(P->ge, P->sc, static_cast<size_t>(P->Np) * D, P->rinv, N, D, parts);
  KERNEL_CHECK();
  dsk::aam_shard_gpart_kernel<<<grid, 256, 0, s>>>(P->gw, P->sn, static_cast<size_t>(P->Cp) * D, P->cinv, N, D,
                                                   parts + nd);
  KERNEL_CHECK();
  dsk::aam_shard_rows_bwd_kernel<<<(N + 7) / 8, 256, 0, s>>>(E, parts, 2, N, D, gE);
  KERNEL_CHECK();
  CUDA_TRY(cudaFreeAsync(parts, s));
  return DSK_OK;
}

// ---- cosine scoring, cohort statistics (AS-norm) ------------------------------------------------------------------
// Rows of E per GEMM chunk: the largest multiple of 128 with chunk x Np x 4 B <= kScoreChunkBytes (at least 128), and no
// more than M rounded up to 128.
constexpr size_t kScoreChunkBytes = 256ull << 20;
static int score_chunk_rows(int M, int Np) {
  const long cap = static_cast<long>(kScoreChunkBytes / (static_cast<size_t>(Np) * 4)) / 128 * 128;
  const long m = (static_cast<long>(M) + 127) / 128 * 128;
  const long c = cap < 128 ? 128 : cap;
  return static_cast<int>(m < c ? m : c);
}

// The scoring plan in slot P of h (h->score or h->search) for (Nc, D, chunk).  A rebuild synchronises `s` (buffers in
// use are freed).
static int score_plan(dsk_handle h, ScorePlan& P, int M, int Nc, int D, cudaStream_t s, ScorePlan** out) {
  *out = &P;
  const int Np = (Nc + 127) / 128 * 128, chunk = score_chunk_rows(M, Np);
  return plan_acquire(P, {Nc, D, chunk}, s, [&]() -> int {
    P.D = D;
    P.chunk = chunk;
    P.Np = Np;
    const size_t d3 = 3ull * D;
    const int rc = arena_alloc(&P.buf, {{&P.ea, chunk * d3 * 2}, {&P.cb, Np * d3 * 2}, {&P.nrm_e, chunk * 4ull},
                                        {&P.nrm_c, Np * 4ull}, {&P.cos, 1ull * chunk * Np * 4}}, s);
    return rc ? rc : build_gemm(h, &P.gemm, P.ea, chunk, P.cb, Np, 3 * D, P.cos, true);  // cos = E^ C^T, K = 3D
  });
}

static int score_check(dsk_handle h, bool ptrs_ok, int M, int Nc, int D, int k, const char* what) {
  if (!ptrs_ok || M < 1 || Nc < 2 || Nc > DSK_SCORE_MAX_COHORT || D < 64 || D % 64 || k < 2 || k > Nc)
    return fail(DSK_ERR_INVALID, "%s: bad arguments (need non-null pointers, M >= 1, 2 <= Nc <= %d, D a positive multiple "
                "of 64, 2 <= k <= Nc; got M %d, Nc %d, D %d, k %d)", what, DSK_SCORE_MAX_COHORT, M, Nc, D, k);
  return check_handle(h);
}

// The norms and B-side operand image of the cohort's rows B (cols <= the plan's Nc of them; rows [cols, Np) are zero), rebuilt
// on every call
static int score_prep_cohort(const ScorePlan& P, const float* B, int cols, cudaStream_t s) {
  const CosRows c{B, cols, P.Np, P.nrm_c, true, P.cb, nullptr};
  return cos_prep(P.D, nullptr, &c, s);
}

// P.cos[0, rows) = cosines of rows [0, rows) of E (rows <= chunk) against the cohort; rows [rows, chunk) are zero
static int score_gemm_chunk(const ScorePlan& P, const float* E, int rows, cudaStream_t s) {
  const CosRows e{E, rows, P.chunk, P.nrm_e, true, P.ea, nullptr};
  if (int rc = cos_prep(P.D, &e, nullptr, s)) return rc;
  for (const ConvLaunch& L : P.gemm)
    if (int rc = launch_conv(L, s)) return rc;
  return DSK_OK;
}

static int launch_topk_stats(const float* S, int rows, int cols, long ld, int k, float* mean, float* std, cudaStream_t s) {
  if (cols <= dsk::kTopkStageCols) {
    const int smem = cols * 4;
    auto kern = dsk::topk_select_stats_kernel<true>;
    if (int rc = ensure_smem_optin(reinterpret_cast<const void*>(kern), smem)) return rc;
    kern<<<rows, dsk::kTopkThreads, smem, s>>>(S, cols, ld, k, mean, std);
  } else {
    dsk::topk_select_stats_kernel<false><<<rows, dsk::kTopkThreads, 0, s>>>(S, cols, ld, k, mean, std);
  }
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_cosine_matrix(dsk_handle h, const float* A, int32_t M, const float* B, int32_t Nc, int32_t D, float* cos,
                          void* stream) {
  int rc = score_check(h, A && B && cos, M, Nc, D, 2, "dsk_cosine_matrix");
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  ScorePlan* P = nullptr;
  if ((rc = score_plan(h, h->score, M, Nc, D, s, &P))) return rc;
  if ((rc = score_prep_cohort(*P, B, Nc, s))) return rc;
  for (int r0 = 0; r0 < M; r0 += P->chunk) {
    const int rows = M - r0 < P->chunk ? M - r0 : P->chunk;
    if ((rc = score_gemm_chunk(*P, A + static_cast<size_t>(r0) * D, rows, s))) return rc;
    CUDA_TRY(cudaMemcpy2DAsync(cos + static_cast<size_t>(r0) * Nc, Nc * 4ull, P->cos, P->Np * 4ull, Nc * 4ull, rows,
                               cudaMemcpyDeviceToDevice, s));
  }
  return DSK_OK;
}

int32_t dsk_topk_mean_std(const float* S, int32_t rows, int32_t cols, int64_t ld, int32_t k, float* mean, float* std,
                          void* stream) {
  if (!S || !mean || !std || rows < 1 || cols < 2 || cols > DSK_SCORE_MAX_COHORT || ld < cols || k < 2 || k > cols)
    return fail(DSK_ERR_INVALID, "dsk_topk_mean_std: bad arguments (need non-null pointers, rows >= 1, 2 <= cols <= %d, "
                "ld >= cols, 2 <= k <= cols; got rows %d, cols %d, ld %lld, k %d)", DSK_SCORE_MAX_COHORT, rows, cols,
                static_cast<long long>(ld), k);
  return launch_topk_stats(S, rows, cols, static_cast<long>(ld), k, mean, std, static_cast<cudaStream_t>(stream));
}

int32_t dsk_cohort_stats(dsk_handle h, const float* E, int32_t M, const float* cohort, int32_t Nc, int32_t D, int32_t k,
                         float* mean, float* std, void* stream) {
  int rc = score_check(h, E && cohort && mean && std, M, Nc, D, k, "dsk_cohort_stats");
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  ScorePlan* P = nullptr;
  if ((rc = score_plan(h, h->score, M, Nc, D, s, &P))) return rc;
  if ((rc = score_prep_cohort(*P, cohort, Nc, s))) return rc;
  for (int r0 = 0; r0 < M; r0 += P->chunk) {
    const int rows = M - r0 < P->chunk ? M - r0 : P->chunk;
    if ((rc = score_gemm_chunk(*P, E + static_cast<size_t>(r0) * D, rows, s))) return rc;
    if ((rc = launch_topk_stats(P->cos, rows, Nc, P->Np, k, mean + r0, std + r0, s))) return rc;
  }
  return DSK_OK;
}

int32_t dsk_score_trials(const float* X, int32_t U, int32_t D, const int64_t* trials, int64_t T, const float* mean,
                         const float* std, float* raw, float* normed, void* stream) {
  const bool stats = mean || std;
  if (!X || !trials || !raw || U < 1 || D < 1 || T < 1 || T > (1ll << 33) || (stats && (!mean || !std || !normed)))
    return fail(DSK_ERR_INVALID, "dsk_score_trials: bad arguments (need non-null X, trials and raw, U >= 1, D >= 1, "
                "1 <= T <= 2^33, and mean, std and normed all non-null or mean and std both NULL; got U %d, D %d, T %lld)",
                U, D, static_cast<long long>(T));
  const unsigned blocks = static_cast<unsigned>((T + dsk::kScoreWarps - 1) / dsk::kScoreWarps);
  dsk::score_trials_kernel<<<blocks, 32 * dsk::kScoreWarps, 0, static_cast<cudaStream_t>(stream)>>>(
      X, U, D, trials, static_cast<long long>(T), stats ? mean : nullptr, std, raw, normed);
  KERNEL_CHECK();
  return DSK_OK;
}

// ---- identification: gallery search, class centroids -------------------------------------------------------------
static int launch_topk_indices(const float* S, int rows, int cols, long ld, int k, long long col0, int64_t* idx,
                               float* val, long ldo, cudaStream_t s) {
  if (cols <= dsk::kTopkStageCols) {
    const int smem = cols * 4;
    auto kern = dsk::topk_indices_kernel<true>;
    if (int rc = ensure_smem_optin(reinterpret_cast<const void*>(kern), smem)) return rc;
    kern<<<rows, dsk::kTopkThreads, smem, s>>>(S, cols, ld, k, col0, idx, val, ldo);
  } else {
    dsk::topk_indices_kernel<false><<<rows, dsk::kTopkThreads, 0, s>>>(S, cols, ld, k, col0, idx, val, ldo);
  }
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_topk_indices(const float* S, int32_t rows, int32_t cols, int64_t ld, int32_t k, int64_t* idx, float* val,
                         void* stream) {
  if (!S || !idx || !val || rows < 1 || cols < 1 || cols > DSK_SCORE_MAX_COHORT || ld < cols || k < 1 || k > cols ||
      k > DSK_SEARCH_MAX_K)
    return fail(DSK_ERR_INVALID, "dsk_topk_indices: bad arguments (need non-null pointers, rows >= 1, 1 <= cols <= %d, "
                "ld >= cols, 1 <= k <= min(cols, %d); got rows %d, cols %d, ld %lld, k %d)", DSK_SCORE_MAX_COHORT,
                DSK_SEARCH_MAX_K, rows, cols, static_cast<long long>(ld), k);
  return launch_topk_indices(S, rows, cols, static_cast<long>(ld), k, 0, idx, val, k, static_cast<cudaStream_t>(stream));
}

// Gallery columns per search chunk: every selection runs on a row staged in shared memory
static_assert(dsk::kSearchMaxK <= dsk::kTopkStageCols,
              "the first gallery chunk holds at least k columns");

int32_t dsk_cosine_topk(dsk_handle h, const float* Q, int32_t M, const float* G, int32_t Ng, int32_t D, int32_t k,
                        int64_t* idx, float* val, void* stream) {
  if (!Q || !G || !idx || !val || M < 1 || k < 1 || k > DSK_SEARCH_MAX_K || Ng < k || D < 64 || D % 64)
    return fail(DSK_ERR_INVALID, "dsk_cosine_topk: bad arguments (need non-null pointers, M >= 1, 1 <= k <= %d, Ng >= k, "
                "D a positive multiple of 64; got M %d, Ng %d, D %d, k %d)", DSK_SEARCH_MAX_K, M, Ng, D, k);
  int rc = check_handle(h);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int width = Ng < dsk::kTopkStageCols ? Ng : dsk::kTopkStageCols;
  ScorePlan* P = nullptr;
  if ((rc = score_plan(h, h->search, M, width, D, s, &P))) return rc;
  // later chunks select into (wi, wv) [chunk][k] and are merged into the caller's running lists
  int64_t* wi = nullptr;
  float* wv = nullptr;
  if (Ng > width) {
    CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&wi), static_cast<size_t>(P->chunk) * k * 12, s));
    wv = reinterpret_cast<float*>(wi + static_cast<size_t>(P->chunk) * k);
  }
  for (long c0 = 0; c0 < Ng && !rc; c0 += width) {
    const int cols = Ng - c0 < width ? static_cast<int>(Ng - c0) : width, kc = cols < k ? cols : k;
    rc = score_prep_cohort(*P, G + static_cast<size_t>(c0) * D, cols, s);
    for (int r0 = 0; r0 < M && !rc; r0 += P->chunk) {
      const int rows = M - r0 < P->chunk ? M - r0 : P->chunk;
      int64_t* oi = idx + static_cast<size_t>(r0) * k;
      float* ov = val + static_cast<size_t>(r0) * k;
      if ((rc = score_gemm_chunk(*P, Q + static_cast<size_t>(r0) * D, rows, s))) break;
      if (c0 == 0) {
        rc = launch_topk_indices(P->cos, rows, cols, P->Np, k, 0, oi, ov, k, s);
      } else if (!(rc = launch_topk_indices(P->cos, rows, cols, P->Np, kc, c0, wi, wv, k, s))) {
        dsk::topk_merge_kernel<<<rows, dsk::kTopkThreads, 0, s>>>(oi, ov, wi, wv, k, kc);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) rc = fail(DSK_ERR_CUDA, "kernel launch failed: %s (topk_merge_kernel)", cudaGetErrorString(e));
      }
    }
  }
  if (wi) cudaFreeAsync(wi, s);
  return rc;
}

int32_t dsk_class_centroids(const float* X, int32_t U, int32_t D, const int64_t* order, const int64_t* offsets,
                            int32_t S, float* out, void* stream) {
  if (!X || !order || !offsets || !out || U < 1 || D < 1 || S < 1)
    return fail(DSK_ERR_INVALID, "dsk_class_centroids: bad arguments (need non-null pointers, U >= 1, D >= 1, S >= 1; got "
                "U %d, D %d, S %d)", U, D, S);
  dsk::class_centroids_kernel<<<dim3(S, (D + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(X, U, D, order,
                                                                                                       offsets, out);
  KERNEL_CHECK();
  return DSK_OK;
}

// ---- PLDA backend: fit statistics, transforms, LLR scoring --------------------------------------------------------
int32_t dsk_class_sums_f64(const float* X, int64_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                           int32_t C, const double* mu, double* out, void* stream) {
  if (!X || !order || !offsets || !out || N < 1 || D < 1 || C < 1)
    return fail(DSK_ERR_INVALID, "dsk_class_sums_f64: bad arguments (need non-null X, order, offsets and out, N >= 1, "
                "D >= 1, C >= 1; got N %lld, D %d, C %d)", static_cast<long long>(N), D, C);
  dsk::class_sums_f64_kernel<<<dim3(C, (D + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      X, static_cast<long long>(N), D, order, offsets, mu, out);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_gram_f64(const float* X, int64_t N, int32_t D, const double* mu, double* G, void* stream) {
  if (!X || !G || N < 1 || D < 1 || D > DSK_F64_MAX_DIM)
    return fail(DSK_ERR_INVALID, "dsk_gram_f64: bad arguments (need non-null X and G, N >= 1, 1 <= D <= %d; got N %lld, "
                "D %d)", DSK_F64_MAX_DIM, static_cast<long long>(N), D);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // split-K over rows: a function of (N, D) only, so the partials and their fixed-order sum are too
  const long long tiles = (D + dsk::kF64Tile - 1) / dsk::kF64Tile, nt = tiles * (tiles + 1) / 2;
  const long long kblocks = (N + dsk::kF64K - 1) / dsk::kF64K;
  long long splits = std::max(1ll, std::min((dsk::kF64GramCtas + nt - 1) / nt, kblocks));
  const long long rows_per = (kblocks + splits - 1) / splits * dsk::kF64K;
  splits = (N + rows_per - 1) / rows_per;
  double* ws = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&ws),
                           static_cast<size_t>(splits * nt) * dsk::kF64Tile * dsk::kF64Tile * sizeof(double), s));
  dsk::gram_f64_kernel<<<dim3(static_cast<unsigned>(nt), static_cast<unsigned>(splits)), dsk::kF64Threads, 0, s>>>(
      X, static_cast<long long>(N), D, mu, rows_per, ws);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) {
    dsk::gram_reduce_kernel<<<static_cast<unsigned>(nt), 256, 0, s>>>(ws, D, static_cast<int>(splits), G);
    e = cudaGetLastError();
  }
  const cudaError_t fe = cudaFreeAsync(ws, s);
  if (e != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_gram_f64: kernel launch failed: %s", cudaGetErrorString(e));
  if (fe != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_gram_f64: cudaFreeAsync failed: %s", cudaGetErrorString(fe));
  return DSK_OK;
}

int32_t dsk_affine_norm_f64(const float* X, int64_t N, int32_t D, const double* A, int32_t d, const double* c,
                            int32_t mode, const double* psi, const int32_t* counts, float* Y, void* stream) {
  if (!X || !A || !Y || N < 1 || D < 1 || D > DSK_F64_MAX_DIM || d < 1 || d > DSK_F64_MAX_DIM ||
      (mode != DSK_NORM_NONE && mode != DSK_NORM_LENGTH && mode != DSK_NORM_PLDA) || (mode == DSK_NORM_PLDA && !psi))
    return fail(DSK_ERR_INVALID, "dsk_affine_norm_f64: bad arguments (need non-null X, A and Y, N >= 1, 1 <= D, d <= %d, "
                "mode %d, %d or %d, psi non-null in mode %d; got N %lld, D %d, d %d, mode %d)", DSK_F64_MAX_DIM,
                DSK_NORM_NONE, DSK_NORM_LENGTH, DSK_NORM_PLDA, DSK_NORM_PLDA, static_cast<long long>(N), D, d, mode);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // the fp64 rows go through a workspace of at most 128 MiB, taken in row chunks in order
  const long long per = std::max<long long>(dsk::kF64Tile, (128ll << 20) / (8ll * d) / dsk::kF64Tile * dsk::kF64Tile);
  const long long chunk = std::min<long long>(per, (N + dsk::kF64Tile - 1) / dsk::kF64Tile * dsk::kF64Tile);
  double* Z = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&Z), static_cast<size_t>(chunk) * d * sizeof(double), s));
  cudaError_t e = cudaSuccess;
  for (long long r0 = 0; r0 < N && e == cudaSuccess; r0 += chunk) {
    const long long rows = std::min(chunk, static_cast<long long>(N) - r0);
    dsk::affine_f64_kernel<<<dim3((d + dsk::kF64Tile - 1) / dsk::kF64Tile,
                                  static_cast<unsigned>((rows + dsk::kF64Tile - 1) / dsk::kF64Tile)),
                             dsk::kF64Threads, 0, s>>>(X + r0 * D, rows, D, A, d, c, Z);
    e = cudaGetLastError();
    if (e != cudaSuccess) break;
    dsk::affine_scale_kernel<<<static_cast<unsigned>((rows + dsk::kPldaWarps - 1) / dsk::kPldaWarps), 256, 0, s>>>(
        Z, rows, d, mode, psi, counts ? counts + r0 : nullptr, Y + r0 * d);
    e = cudaGetLastError();
  }
  const cudaError_t fe = cudaFreeAsync(Z, s);
  if (e != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_affine_norm_f64: kernel launch failed: %s", cudaGetErrorString(e));
  if (fe != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_affine_norm_f64: cudaFreeAsync failed: %s", cudaGetErrorString(fe));
  return DSK_OK;
}

int32_t dsk_plda_score_trials(const float* Y, int32_t U, int32_t d, const double* psi, const int32_t* counts,
                              const int64_t* trials, int64_t T, float* llr, void* stream) {
  if (!Y || !psi || !trials || !llr || U < 1 || d < 1 || T < 1 || T > (1ll << 33))
    return fail(DSK_ERR_INVALID, "dsk_plda_score_trials: bad arguments (need non-null Y, psi, trials and llr, U >= 1, "
                "d >= 1, 1 <= T <= 2^33; got U %d, d %d, T %lld)", U, d, static_cast<long long>(T));
  const unsigned blocks = static_cast<unsigned>((T + dsk::kPldaWarps - 1) / dsk::kPldaWarps);
  dsk::plda_trials_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(Y, U, d, psi, counts, trials,
                                                                                 static_cast<long long>(T), llr);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_plda_score_matrix(const float* Ya, int32_t M, const float* Yb, int32_t N, int32_t d, const double* psi,
                              float* S, int64_t ld, void* stream) {
  if (!Ya || !Yb || !psi || !S || M < 1 || M > DSK_PLDA_MAX_ROWS || N < 1 || d < 1 || ld < N)
    return fail(DSK_ERR_INVALID, "dsk_plda_score_matrix: bad arguments (need non-null Ya, Yb, psi and S, 1 <= M <= %d, "
                "N >= 1, d >= 1, ld >= N; got M %d, N %d, d %d, ld %lld)", DSK_PLDA_MAX_ROWS, M, N, d,
                static_cast<long long>(ld));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long rows = static_cast<long long>(M) + N;
  double* ws = nullptr;  // [w (d), beta (d), k], then q of Ya's rows and Yb's rows
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&ws), static_cast<size_t>(2 * d + 1 + rows) * sizeof(double), s));
  double* q = ws + 2 * d + 1;
  dsk::plda_coef_kernel<<<1, 32, 0, s>>>(psi, d, ws);
  dsk::plda_q_kernel<<<static_cast<unsigned>((rows + dsk::kPldaWarps - 1) / dsk::kPldaWarps), 256, 0, s>>>(
      Ya, M, Yb, N, d, ws, q);
  dsk::plda_matrix_kernel<<<dim3((N + dsk::kF64Tile - 1) / dsk::kF64Tile, (M + dsk::kF64Tile - 1) / dsk::kF64Tile),
                            dsk::kF64Threads, 0, s>>>(Ya, M, Yb, N, d, ws, q, S, static_cast<long long>(ld));
  const cudaError_t e = cudaGetLastError();
  const cudaError_t fe = cudaFreeAsync(ws, s);
  if (e != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_plda_score_matrix: kernel launch failed: %s", cudaGetErrorString(e));
  if (fe != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_plda_score_matrix: cudaFreeAsync failed: %s", cudaGetErrorString(fe));
  return DSK_OK;
}

// ---- VBx: Bayesian HMM clustering of window embeddings ------------------------------------------------------------
constexpr int kVbxItersPerCheck = 8;  // iterations between reads of the device-side count of finished recordings

int32_t dsk_vbx(const float* X, int64_t W, int32_t d, const int64_t* offsets, int32_t R, const int32_t* init_labels,
                int32_t S, const double* phi, double Fa, double Fb, double loop_p, double init_smoothing,
                int32_t max_iters, double epsilon, double* gamma, double* pi, double* elbo, int32_t* iters,
                int32_t* labels, void* stream) {
  bool ok = X && offsets && init_labels && phi && gamma && pi && elbo && iters && labels && R >= 1 && d >= 1 &&
            d <= DSK_F64_MAX_DIM && S >= 1 && S <= DSK_VBX_MAX_SPEAKERS && !std::isnan(Fa) && !std::isnan(Fb) &&
            !std::isnan(loop_p) && !std::isnan(init_smoothing) && !std::isnan(epsilon) && Fa > 0 && Fb > 0 &&
            loop_p >= 0 && loop_p <= 1 && init_smoothing >= 0 && max_iters >= 1;
  if (ok) ok = offsets[0] == 0 && offsets[R] == W;
  for (int32_t r = 0; ok && r < R; ++r)
    ok = offsets[r + 1] > offsets[r] && offsets[r + 1] - offsets[r] <= DSK_AHC_MAX_N;
  if (!ok)
    return fail(DSK_ERR_INVALID, "dsk_vbx: bad arguments (need non-null pointers, R >= 1, 1 <= d <= %d, 1 <= S <= %d, "
                "offsets strictly increasing from 0 to W with at most %d rows per recording, Fa > 0, Fb > 0, loop_p in "
                "[0, 1], init_smoothing >= 0, max_iters >= 1, no NaN parameter; got W %lld, d %d, R %d, S %d, Fa %g, "
                "Fb %g, loop_p %g, init_smoothing %g, max_iters %d, epsilon %g)", DSK_F64_MAX_DIM,
                DSK_VBX_MAX_SPEAKERS, DSK_AHC_MAX_N, static_cast<long long>(W), d, R, S, Fa, Fb, loop_p,
                init_smoothing, max_iters, epsilon);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // work tables: (recording, split) for the statistics, (recording, row tile) for the log-likelihoods; every split
  // depends only on the recording's own length
  std::vector<int32_t> stat_tab, ll_tab, split_base(R + 1, 0);
  for (int32_t r = 0; r < R; ++r) {
    const int64_t n = offsets[r + 1] - offsets[r];
    const int splits = static_cast<int>((n + dsk::kVbxSplitRows - 1) / dsk::kVbxSplitRows);
    for (int k = 0; k < splits; ++k) stat_tab.insert(stat_tab.end(), {r, k});
    for (int k = 0; k < (n + dsk::kF64Tile - 1) / dsk::kF64Tile; ++k) ll_tab.insert(ll_tab.end(), {r, k});
    split_base[r + 1] = split_base[r] + splits;
  }
  const int n_stat = static_cast<int>(stat_tab.size() / 2), n_ll = static_cast<int>(ll_tab.size() / 2);
  const int tiles_s = (S + dsk::kF64Tile - 1) / dsk::kF64Tile, tiles_c = (d + 1 + dsk::kF64Tile - 1) / dsk::kF64Tile;
  // workspace: rho (W,d), G (W), lnp (W,S), ln C (W), the partials, alpha (R,S,d), cst and kl (R,S), then the tables,
  // offsets and per-recording ints
  const size_t Wd = static_cast<size_t>(W);
  size_t sizes[] = {Wd * d * 8, Wd * 8, Wd * S * 8, Wd * 8,
                    static_cast<size_t>(n_stat) * tiles_s * tiles_c * dsk::kF64Tile * dsk::kF64Tile * 8,
                    static_cast<size_t>(R) * S * d * 8, static_cast<size_t>(R) * S * 8, static_cast<size_t>(R) * S * 8,
                    static_cast<size_t>(R + 1) * 8, stat_tab.size() * 4, ll_tab.size() * 4,
                    static_cast<size_t>(R + 1) * 4, (3 * static_cast<size_t>(R) + 1) * 4};
  size_t total = 0;
  for (size_t& z : sizes) total += z = (z + 255) / 256 * 256;
  uint8_t* ws = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&ws), total, s));
  uint8_t* p = ws;
  auto take = [&](int i) {
    uint8_t* q = p;
    p += sizes[i];
    return q;
  };
  double* rho = reinterpret_cast<double*>(take(0));
  double* G = reinterpret_cast<double*>(take(1));
  double* lnp = reinterpret_cast<double*>(take(2));
  double* lnc = reinterpret_cast<double*>(take(3));
  double* part = reinterpret_cast<double*>(take(4));
  double* alpha = reinterpret_cast<double*>(take(5));
  double* cst = reinterpret_cast<double*>(take(6));
  double* kl = reinterpret_cast<double*>(take(7));
  int64_t* off_d = reinterpret_cast<int64_t*>(take(8));
  int32_t* stat_d = reinterpret_cast<int32_t*>(take(9));
  int32_t* ll_d = reinterpret_cast<int32_t*>(take(10));
  int32_t* base_d = reinterpret_cast<int32_t*>(take(11));
  int32_t* rec_S = reinterpret_cast<int32_t*>(take(12));
  int32_t* bad = rec_S + R;
  int32_t* done = bad + R;
  int32_t* n_done = done + R;
  const double ratio = Fa / Fb;
  int rc = DSK_OK;
  cudaError_t e = cudaSuccess;
  do {
    // pageable sources: each copy has read its host buffer when it returns
    e = cudaMemcpyAsync(off_d, offsets, (R + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(stat_d, stat_tab.data(), stat_tab.size() * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ll_d, ll_tab.data(), ll_tab.size() * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(base_d, split_base.data(), (R + 1) * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(rec_S, 0, (3 * static_cast<size_t>(R) + 1) * 4, s);
    if (e != cudaSuccess) break;
    dsk::vbx_prep_kernel<<<static_cast<unsigned>((W + dsk::kPldaWarps - 1) / dsk::kPldaWarps), 256, 0, s>>>(
        X, W, d, off_d, R, init_labels, S, phi, rho, G, rec_S, bad);
    dsk::vbx_rec_init_kernel<<<(R + 127) / 128, 128, 0, s>>>(R, S, max_iters, rec_S, bad, done, n_done, pi, elbo,
                                                             iters);
    dsk::vbx_gamma0_kernel<<<static_cast<unsigned>((W + 255) / 256), 256, 0, s>>>(W, off_d, R, init_labels, S,
                                                                                   init_smoothing, rec_S, bad, gamma);
    e = cudaGetLastError();
    for (int it = 0; it < max_iters && e == cudaSuccess; ++it) {
      dsk::vbx_stats_kernel<<<dim3(n_stat, tiles_s * tiles_c), dsk::kF64Threads, 0, s>>>(gamma, S, rho, d, off_d, stat_d,
                                                                                         rec_S, done, part);
      dsk::vbx_model_kernel<<<dim3(R, (S + dsk::kPldaWarps - 1) / dsk::kPldaWarps), 256, 0, s>>>(
          part, off_d, base_d, S, d, phi, ratio, rec_S, done, alpha, cst, kl);
      dsk::vbx_loglik_kernel<<<dim3(n_ll, tiles_s), dsk::kF64Threads, 0, s>>>(rho, d, alpha, cst, G, S, Fa, off_d, ll_d,
                                                                              rec_S, done, lnp);
      dsk::vbx_fb_kernel<<<R, 32, 0, s>>>(off_d, S, lnp, gamma, lnc, kl, loop_p, Fb, epsilon, it, max_iters, rec_S,
                                          done, n_done, pi, elbo, iters);
      e = cudaGetLastError();
      if (e == cudaSuccess && (it + 1) % kVbxItersPerCheck == 0 && it + 1 < max_iters) {
        int32_t nd = 0;
        e = cudaMemcpyAsync(&nd, n_done, sizeof(nd), cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e == cudaSuccess && nd == R) break;
      }
    }
    if (e != cudaSuccess) break;
    dsk::vbx_labels_kernel<<<static_cast<unsigned>((W + 255) / 256), 256, 0, s>>>(W, off_d, R, S, rec_S, bad, gamma,
                                                                                  labels);
    e = cudaGetLastError();
  } while (false);
  if (e != cudaSuccess) rc = fail(DSK_ERR_CUDA, "dsk_vbx: %s", cudaGetErrorString(e));
  const cudaError_t fe = cudaFreeAsync(ws, s);
  if (rc) return rc;
  if (fe != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_vbx: cudaFreeAsync failed: %s", cudaGetErrorString(fe));
  return DSK_OK;
}

// ---- classifier head, cross-entropy, fused optimizer step ---------------------------------------------------------
int32_t dsk_linear_forward(const float* x, const float* w, const float* b, int32_t M, int32_t N, int32_t K, float* y,
                           void* stream) {
  if (!x || !w || !y || M <= 0 || N <= 0 || K <= 0) return fail(DSK_ERR_INVALID, "dsk_linear_forward: bad arguments");
  dim3 g((N + dsk::kGemmTile - 1) / dsk::kGemmTile, (M + dsk::kGemmTile - 1) / dsk::kGemmTile);
  // y[i][j] = sum_k x[i][k] * w[j][k] + b[j]
  dsk::sgemm_strided_kernel<<<g, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, K, 1, w, 1, K, b, y, M, N, K);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_linear_backward(const float* x, const float* w, const float* gy, int32_t M, int32_t N, int32_t K, float* gx,
                            float* gw, float* gb, void* stream) {
  if (!x || !w || !gy || M <= 0 || N <= 0 || K <= 0) return fail(DSK_ERR_INVALID, "dsk_linear_backward: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int T = dsk::kGemmTile;
  if (gx) {  // gx[i][k] = sum_j gy[i][j] * w[j][k]
    dsk::sgemm_strided_kernel<<<dim3((K + T - 1) / T, (M + T - 1) / T), 256, 0, s>>>(gy, N, 1, w, K, 1, nullptr, gx, M, K, N);
    KERNEL_CHECK();
  }
  if (gw) {  // gw[j][k] = sum_i gy[i][j] * x[i][k]
    dsk::sgemm_strided_kernel<<<dim3((K + T - 1) / T, (N + T - 1) / T), 256, 0, s>>>(gy, 1, N, x, K, 1, nullptr, gw, N, K, M);
    KERNEL_CHECK();
  }
  if (gb) {
    dsk::colsum_kernel<<<(N + 127) / 128, 128, 0, s>>>(gy, M, N, gb);
    KERNEL_CHECK();
  }
  return DSK_OK;
}

int32_t dsk_cross_entropy(const float* logits, const int64_t* labels, int32_t M, int32_t C, float* loss, float* lse,
                          float* row_loss, void* stream) {
  if (!logits || !labels || !loss || !lse || !row_loss || M <= 0 || C <= 0)
    return fail(DSK_ERR_INVALID, "dsk_cross_entropy: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dsk::ce_rows_kernel<<<M, 256, 0, s>>>(logits, labels, C, lse, row_loss);
  KERNEL_CHECK();
  dsk::mean_rows_kernel<<<1, 1024, 0, s>>>(row_loss, M, M, loss);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_cross_entropy_bwd(const float* logits, const int64_t* labels, const float* lse, const float* grad_loss,
                              int32_t M, int32_t C, float* dlogits, void* stream) {
  if (!logits || !labels || !lse || !grad_loss || !dlogits || M <= 0 || C <= 0)
    return fail(DSK_ERR_INVALID, "dsk_cross_entropy_bwd: bad arguments");
  const long total = static_cast<long>(M) * C;
  const int blocks = static_cast<int>((total + 255) / 256 < 2368 ? (total + 255) / 256 : 2368);
  dsk::ce_bwd_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, labels, lse, grad_loss, M, C, dlogits);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_adagrad_step(float* param, const float* grad, float* state_sum, int64_t n, double lr, double lr_decay,
                         double weight_decay, double eps, int64_t step, float grad_div, const float* grad_denom,
                         void* stream) {
  if (!param || !grad || !state_sum || n <= 0 || step < 1 || !(grad_div > 0.f))
    return fail(DSK_ERR_INVALID, "dsk_adagrad_step: bad arguments (step counts from 1, grad_div > 0)");
  if ((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(state_sum)) & 15)
    return fail(DSK_ERR_INVALID, "dsk_adagrad_step: buffers must be 16-byte aligned");
  // clr as torch computes it (Python double arithmetic, then one rounding to float at the kernel boundary)
  const double minus_clr = -lr / (1.0 + static_cast<double>(step - 1) * lr_decay);
  const long n4 = n / 4 > 0 ? n / 4 : 1;
  const int blocks = static_cast<int>((n4 + 255) / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  dsk::adagrad_flat_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      param, grad, state_sum, n, grad_div, grad_denom, static_cast<float>(minus_clr), static_cast<float>(eps),
      static_cast<float>(weight_decay));
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_threshold_counts(const float* dist, const uint8_t* same, int32_t P, const double* thresholds, int32_t nT,
                             int32_t* tp, int32_t* fp, void* stream) {
  if (!dist || !same || !thresholds || !tp || !fp || P <= 0 || nT <= 0)
    return fail(DSK_ERR_INVALID, "dsk_threshold_counts: bad arguments");
  const int blocks = (nT + dsk::kSweepThreads - 1) / dsk::kSweepThreads;
  dsk::threshold_counts_kernel<<<blocks, dsk::kSweepThreads, 0, static_cast<cudaStream_t>(stream)>>>(dist, same, P, thresholds,
                                                                                                      nT, tp, fp);
  KERNEL_CHECK();
  return DSK_OK;
}

// ---- agglomerative clustering ------------------------------------------------------------------------------------
// Rounds between two reads of the device-side done flag: a finished run costs at most this many rounds of launches
// that return at once.
static constexpr int kAhcRoundsPerBatch = 64;

// The merge records, in round order, into scipy's linkage matrix: rows sorted by (height, round, representative of the
// lower cluster), of which the first `keep` are written, and the flat labels after those `keep` merges.  The height used
// for sorting is raised to the sorting height of the merged clusters, so a parent never sorts before a child whose
// rounded height came out 1 ulp above its own (with exact arithmetic a reducible linkage is monotone and this changes
// nothing).  The cut at k clusters is taken here, from the sorted tree, and not by stopping the rounds at k clusters: a
// round may merge a mutual pair far above heights that later rounds merge below it (two isolated points that are each
// other's nearest), so the rounds reach k clusters with a different partition than the tree's cut.
static void ahc_assemble(const std::vector<dsk::AhcRecord>& rec, int N, int keep, double* Z, int32_t* labels) {
  const int m = static_cast<int>(rec.size());
  std::vector<double> key(m), cl_key(N, -HUGE_VAL);
  for (int k = 0; k < m; ++k) {
    const double h = std::max(rec[k].height, std::max(cl_key[rec[k].rep_a], cl_key[rec[k].rep_b]));
    key[k] = h;
    cl_key[rec[k].rep_a] = h;  // the merged cluster keeps the lower representative
  }
  std::vector<int> order(m);
  for (int k = 0; k < m; ++k) order[k] = k;
  std::sort(order.begin(), order.end(), [&](int x, int y) {
    if (key[x] != key[y]) return key[x] < key[y];
    if (rec[x].round != rec[y].round) return rec[x].round < rec[y].round;
    return rec[x].rep_a < rec[y].rep_a;
  });
  std::vector<int> cur(N), parent(N);
  for (int i = 0; i < N; ++i) cur[i] = parent[i] = i;
  for (int r = 0; r < keep; ++r) {
    const dsk::AhcRecord& e = rec[order[r]];
    const int ia = cur[e.rep_a], ib = cur[e.rep_b];
    Z[4 * r + 0] = std::min(ia, ib);
    Z[4 * r + 1] = std::max(ia, ib);
    Z[4 * r + 2] = e.height;
    Z[4 * r + 3] = e.size;
    cur[e.rep_a] = N + r;
    parent[e.rep_b] = e.rep_a;  // representatives only ever point to lower representatives
  }
  int next = 0;
  std::vector<int> lab(N, -1);
  for (int i = 0; i < N; ++i) {
    int r = i;
    while (parent[r] != r) r = parent[r];
    for (int x = i; parent[x] != x;) {  // path compression
      const int nx = parent[x];
      parent[x] = r;
      x = nx;
    }
    if (lab[r] < 0) lab[r] = next++;
    labels[i] = lab[r];
  }
}

int32_t dsk_ahc(const float* S, int32_t N, int64_t ld, int32_t linkage, int32_t stop_k, double stop_height, double* Z,
                int32_t* n_merges, int32_t* labels, int32_t* n_rounds, void* stream) {
  if (!S || !Z || !n_merges || !labels || N < 2 || N > DSK_AHC_MAX_N || ld < N || stop_k < 1 || stop_k > N ||
      (linkage != DSK_LINKAGE_AVERAGE && linkage != DSK_LINKAGE_COMPLETE) || std::isnan(stop_height))
    return fail(DSK_ERR_INVALID, "dsk_ahc: bad arguments (need non-null S, Z, n_merges and labels, 2 <= N <= %d, "
                "ld >= N, 1 <= stop_k <= N, linkage %d or %d, stop_height not NaN; got N %d, ld %lld, linkage %d, "
                "stop_k %d)", DSK_AHC_MAX_N, DSK_LINKAGE_AVERAGE, DSK_LINKAGE_COMPLETE, N, static_cast<long long>(ld),
                linkage, stop_k);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int dev = 0, sms = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const size_t n2 = static_cast<size_t>(N) * N, h = (N + 1) / 2, q2 = h * h;
  // workspace: the matrix, the quarter-size repack target (the first repack leaves fewer than N / 2 slots, and every
  // later one fewer than half of the previous), then the state, the per-slot arrays and the records
  const size_t small = sizeof(dsk::AhcState) + 8 * static_cast<size_t>(N) * sizeof(double) +
                       static_cast<size_t>(N) * sizeof(dsk::AhcRecord);
  uint8_t* ws = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&ws), (n2 + q2) * sizeof(double) + small, s));
  double* mat0 = reinterpret_cast<double*>(ws);
  double* mat1 = mat0 + n2;
  uint8_t* p = reinterpret_cast<uint8_t*>(mat1 + q2);
  dsk::AhcState* st = reinterpret_cast<dsk::AhcState*>(p);
  p += (sizeof(dsk::AhcState) + 15) / 16 * 16;
  dsk::AhcBufs b;
  b.nnd = reinterpret_cast<double*>(p);
  p += N * sizeof(double);
  b.rec = reinterpret_cast<dsk::AhcRecord*>(p);
  p += N * sizeof(dsk::AhcRecord);
  int32_t* ip = reinterpret_cast<int32_t*>(p);
  int32_t** arrays[] = {&b.rep, &b.size, &b.active, &b.nn, &b.pair_of, &b.pa, &b.pb, &b.pna, &b.pnb, &b.map, &b.tmp};
  for (int32_t** a : arrays) {
    *a = ip;
    ip += N;
  }
  ip += N;  // tmp holds 2 N
  int rc = DSK_OK;
  dsk::AhcState hs{};
  std::vector<dsk::AhcRecord> rec;
  do {
    dsk::ahc_init_state_kernel<<<(N + 255) / 256, 256, 0, s>>>(st, b, N, mat0, mat1, linkage, stop_height);
    const int tiles = (N + dsk::kAhcTile - 1) / dsk::kAhcTile;
    dsk::ahc_init_matrix_kernel<<<dim3(tiles, tiles), dim3(dsk::kAhcTile, 8), 0, s>>>(S, ld, N, mat0, st);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(&hs, st, sizeof(hs), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
      rc = fail(DSK_ERR_CUDA, "dsk_ahc: %s", cudaGetErrorString(e));
      break;
    }
    if (hs.bad) {
      rc = fail(DSK_ERR_INVALID, "dsk_ahc: bad arguments (a non-finite similarity in the upper triangle of S)");
      break;
    }
    const int grid = 8 * sms;
    while (!hs.done) {
      for (int r = 0; r < kAhcRoundsPerBatch; ++r) {
        dsk::ahc_nn_kernel<<<grid, dsk::kAhcThreads, 0, s>>>(st, b);
        dsk::ahc_decide_kernel<<<1, dsk::kAhcDecideThreads, 0, s>>>(st, b);
        dsk::ahc_update_kernel<<<grid, dsk::kAhcThreads, 0, s>>>(st, b);
        dsk::ahc_compact_kernel<<<grid, dsk::kAhcThreads, 0, s>>>(st, b);
        dsk::ahc_finalize_kernel<<<1, dsk::kAhcDecideThreads, 0, s>>>(st, b);
      }
      e = cudaGetLastError();
      if (e == cudaSuccess) e = cudaMemcpyAsync(&hs, st, sizeof(hs), cudaMemcpyDeviceToHost, s);
      if (e == cudaSuccess) e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) {
        rc = fail(DSK_ERR_CUDA, "dsk_ahc: %s", cudaGetErrorString(e));
        break;
      }
      if (hs.round > N) {  // every round that is not the last merges at least one pair
        rc = fail(DSK_ERR_STATE, "dsk_ahc: %d rounds for %d points", hs.round, N);
        break;
      }
    }
    if (rc) break;
    rec.resize(hs.n_rec);
    if (hs.n_rec) e = cudaMemcpyAsync(rec.data(), b.rec, hs.n_rec * sizeof(dsk::AhcRecord), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(DSK_ERR_CUDA, "dsk_ahc: %s", cudaGetErrorString(e));
  } while (false);
  const cudaError_t fe = cudaFreeAsync(ws, s);
  if (rc) return rc;
  if (fe != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_ahc: cudaFreeAsync failed: %s", cudaGetErrorString(fe));
  const int keep = std::min(hs.n_rec, N - stop_k);
  ahc_assemble(rec, N, keep, Z, labels);
  *n_merges = keep;
  if (n_rounds) *n_rounds = hs.round;
  return DSK_OK;
}

// ---- spectral clustering -----------------------------------------------------------------------------------------
static_assert(dsk::kScMaxB >= DSK_SC_MAX_SPEAKERS + 1 + dsk::kScGuard && DSK_SC_MAX_P <= 64,
              "spectral: block and grid limits");

int32_t dsk_spectral_cluster(const float* S, int32_t N, int64_t ld, const int32_t* p_values, int32_t n_p,
                             int32_t max_speakers, int32_t num_speakers, int32_t kmeans_iters, int32_t* labels,
                             int32_t* k_out, int32_t* p_index_out, double* eigenvalues, double* lambda_max,
                             double* ratio, double* embedding, void* stream) {
  bool ok = S && p_values && labels && k_out && p_index_out && eigenvalues && lambda_max && ratio && N >= 2 &&
            N <= DSK_AHC_MAX_N && ld >= N && n_p >= 1 && n_p <= DSK_SC_MAX_P && max_speakers >= 1 &&
            max_speakers <= DSK_SC_MAX_SPEAKERS && num_speakers >= 0 &&
            num_speakers <= std::min<int32_t>(N - 1, DSK_SC_MAX_SPEAKERS) && kmeans_iters >= 1;
  for (int32_t t = 0; ok && t < n_p; ++t)
    ok = p_values[t] >= 1 && p_values[t] <= N - 1 && (t == 0 || p_values[t] > p_values[t - 1]);
  if (!ok)
    return fail(DSK_ERR_INVALID, "dsk_spectral_cluster: bad arguments (need non-null S, p_values and outputs, "
                "2 <= N <= %d, ld >= N, 1 <= n_p <= %d, p_values strictly increasing in [1, N - 1], 1 <= max_speakers "
                "<= %d, 0 <= num_speakers <= min(N - 1, %d), kmeans_iters >= 1; got N %d, ld %lld, n_p %d, "
                "max_speakers %d, num_speakers %d, kmeans_iters %d)", DSK_AHC_MAX_N, DSK_SC_MAX_P,
                DSK_SC_MAX_SPEAKERS, DSK_SC_MAX_SPEAKERS, N, static_cast<long long>(ld), n_p, max_speakers,
                num_speakers, kmeans_iters);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int m = num_speakers ? num_speakers + 1 : std::min(max_speakers + 1, static_cast<int>(N));
  const int B = std::min(std::max(m + dsk::kScGuard, dsk::kScMinB), static_cast<int>(N)), P = 2 * n_p;
  const int splits = (N + dsk::kScSplitRows - 1) / dsk::kScSplitRows, tiles = (N + dsk::kScRows - 1) / dsk::kScRows;
  const size_t n2 = static_cast<size_t>(N) * N, blk = static_cast<size_t>(P) * N * B;
  const size_t mb2 = dsk::kScMaxB * dsk::kScMaxB;
  // workspace: codes (N^2 bytes), W (N^2 uint16), deg (n_p N), four blocks (P N B), partials (P splits 48^2), the
  // small matrices (P 48^2), theta (P 48), the problems, the outputs of step 4 and the flags
  const size_t sizes[] = {n2, n2 * 2, static_cast<size_t>(n_p) * N * 8, blk * 8, blk * 8, blk * 8, blk * 8,
                          static_cast<size_t>(P) * splits * mb2 * 8, P * mb2 * 8, P * dsk::kScMaxB * 8,
                          P * sizeof(dsk::ScProb), static_cast<size_t>(n_p) * m * 8, static_cast<size_t>(n_p) * 8,
                          static_cast<size_t>(n_p) * 8, static_cast<size_t>(N) * 8, static_cast<size_t>(N) * 4,
                          static_cast<size_t>(n_p) * 4, 16};
  constexpr int n_buf = sizeof(sizes) / sizeof(sizes[0]);
  size_t total = 0, offs[n_buf];
  for (int i = 0; i < n_buf; ++i) {
    offs[i] = total;
    total += (sizes[i] + 255) / 256 * 256;
  }
  uint8_t* ws = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&ws), total, s));
  uint8_t* code = ws + offs[0];
  uint16_t* W = reinterpret_cast<uint16_t*>(ws + offs[1]);
  double* deg = reinterpret_cast<double*>(ws + offs[2]);
  double* buf[4];
  for (int i = 0; i < 4; ++i) buf[i] = reinterpret_cast<double*>(ws + offs[3 + i]);
  double* part = reinterpret_cast<double*>(ws + offs[7]);
  double* mat = reinterpret_cast<double*>(ws + offs[8]);
  double* theta = reinterpret_cast<double*>(ws + offs[9]);
  dsk::ScProb* probs = reinterpret_cast<dsk::ScProb*>(ws + offs[10]);
  double* d_eig = reinterpret_cast<double*>(ws + offs[11]);
  double* d_lmax = reinterpret_cast<double*>(ws + offs[12]);
  double* d_ratio = reinterpret_cast<double*>(ws + offs[13]);
  double* scratch = reinterpret_cast<double*>(ws + offs[14]);
  int32_t* d_labels = reinterpret_cast<int32_t*>(ws + offs[15]);
  int32_t* d_pv = reinterpret_cast<int32_t*>(ws + offs[16]);
  int32_t* flags = reinterpret_cast<int32_t*>(ws + offs[17]);  // [0] bad, [1..2] the selection (k, t)
  int rc = DSK_OK;
  std::vector<dsk::ScProb> hp(P);
  int32_t hsel[3] = {0, 0, 0};
  do {
    cudaError_t e = cudaMemcpyAsync(d_pv, p_values, n_p * sizeof(int32_t), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(flags, 0, 16, s);
    const size_t rank_smem = static_cast<size_t>(N) * 4;
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(dsk::sc_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               static_cast<int>(rank_smem));
    if (e == cudaSuccess) {
      dsk::sc_rank_kernel<<<N, dsk::kScThreads, rank_smem, s>>>(S, N, ld, d_pv, n_p, code, flags);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(hsel, flags, sizeof(int32_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
      rc = fail(DSK_ERR_CUDA, "dsk_spectral_cluster: %s", cudaGetErrorString(e));
      break;
    }
    if (hsel[0]) {
      rc = fail(DSK_ERR_INVALID, "dsk_spectral_cluster: bad arguments (a non-finite off-diagonal similarity in S)");
      break;
    }
    const int t32 = (N + 31) / 32;
    dsk::sc_pair_kernel<<<dim3(t32, t32), dim3(32, 8), 0, s>>>(code, N, W);
    dsk::sc_degree_kernel<<<N, dsk::kScThreads, 0, s>>>(W, N, n_p, deg);
    dsk::sc_setup_kernel<<<P, dsk::kScThreads, 0, s>>>(deg, N, n_p, m, B, probs);
    dsk::sc_init_kernel<<<dim3(static_cast<unsigned>((static_cast<size_t>(N) * B + 255) / 256), P), 256, 0, s>>>(
        buf[0], N, B, probs);
    int src = 0;  // the buffer holding every active problem's block
    bool done = false;
    for (int it = 0; it < dsk::kScMaxOuter && !done && rc == DSK_OK; ++it) {
      // orthonormalise by three CholeskyQR passes, src -> x -> y -> 0 (x, y the two other scratch buffers): the first
      // may need the shift, the others restore orthogonality to rounding (shifted CholeskyQR3)
      const int x = src == 1 ? 2 : 1, y = src == 0 ? 2 : 3;  // src 0: 1, 2; src 1: 2, 3; src 2: 1, 3
      const int from[3] = {src, x, y}, to[3] = {x, y, 0};
      for (int pass = 0; pass < 3; ++pass) {
        dsk::sc_gram_kernel<<<dim3(P, splits), dsk::kScThreads, 0, s>>>(buf[from[pass]], buf[from[pass]], N, B, probs,
                                                                        part);
        dsk::sc_small_kernel<<<P, dsk::kScThreads, 0, s>>>(part, splits, N, probs, dsk::kScModeChol, mat, theta);
        dsk::sc_apply_kernel<<<dim3(P, tiles), dsk::kScThreads, 0, s>>>(buf[from[pass]], buf[to[pass]], N, B, probs,
                                                                        mat);
      }
      // Rayleigh-Ritz: Z = Op X (buffer 1), H = X^T Z, X Q -> 2, Z Q -> 3, then the residuals
      dsk::sc_matvec_kernel<<<dim3(P, tiles), dsk::kScThreads, 0, s>>>(W, deg, probs, N, B, -1, buf[0], nullptr,
                                                                       buf[1]);
      dsk::sc_gram_kernel<<<dim3(P, splits), dsk::kScThreads, 0, s>>>(buf[0], buf[1], N, B, probs, part);
      dsk::sc_small_kernel<<<P, dsk::kScThreads, 0, s>>>(part, splits, N, probs, dsk::kScModeRR, mat, theta);
      dsk::sc_apply_kernel<<<dim3(P, tiles), dsk::kScThreads, 0, s>>>(buf[0], buf[2], N, B, probs, mat);
      dsk::sc_apply_kernel<<<dim3(P, tiles), dsk::kScThreads, 0, s>>>(buf[1], buf[3], N, B, probs, mat);
      dsk::sc_resid_kernel<<<dim3(P, splits), dsk::kScMaxB, 0, s>>>(buf[2], buf[3], N, B, probs, theta, part);
      dsk::sc_small_kernel<<<P, dsk::kScThreads, 0, s>>>(part, splits, N, probs, dsk::kScModeRes, mat, theta);
      e = cudaGetLastError();
      if (e == cudaSuccess) e = cudaMemcpyAsync(hp.data(), probs, P * sizeof(dsk::ScProb), cudaMemcpyDeviceToHost, s);
      if (e == cudaSuccess) e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) {
        rc = fail(DSK_ERR_CUDA, "dsk_spectral_cluster: %s", cudaGetErrorString(e));
        break;
      }
      int max_deg = 0;
      done = true;
      for (const dsk::ScProb& p : hp) {
        if (p.failed) {
          rc = fail(DSK_ERR_STATE, "dsk_spectral_cluster: the %s eigenpairs at p = %d did not converge in %d "
                    "iterations (residual %.3g of the spectrum bound)", p.top ? "largest" : "smallest",
                    p_values[p.t], dsk::kScMaxOuter, p.res);
          break;
        }
        if (!p.conv) {
          done = false;
          max_deg = std::max(max_deg, p.deg);
        }
      }
      if (rc || done) break;
      // Chebyshev filter from the Ritz vectors in 2, rotating through 2 -> 0 -> 1 -> 2 ...
      int cur = 2, prev = 2;
      for (int k = 0; k < max_deg; ++k) {
        const int nxt = (cur + 1) % 3;
        dsk::sc_matvec_kernel<<<dim3(P, tiles), dsk::kScThreads, 0, s>>>(W, deg, probs, N, B, k, buf[cur], buf[prev],
                                                                         buf[nxt]);
        prev = cur;
        cur = nxt;
      }
      src = cur;
    }
    if (rc) break;
    if (!done) {
      rc = fail(DSK_ERR_STATE, "dsk_spectral_cluster: no convergence in %d iterations", dsk::kScMaxOuter);
      break;
    }
    // the final Ritz vectors and values of every problem are in buffer 2 and theta
    dsk::sc_select_kernel<<<1, 1, 0, s>>>(probs, theta, n_p, m, N, d_pv, num_speakers, d_eig, d_lmax, d_ratio,
                                          flags + 1);
    dsk::sc_kmeans_kernel<<<1, dsk::kScKmThreads, 0, s>>>(buf[2], N, B, flags + 1, kmeans_iters, scratch, d_labels,
                                                          embedding, m - 1);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(hsel, flags, 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(labels, d_labels, N * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(eigenvalues, d_eig, n_p * m * sizeof(double), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(lambda_max, d_lmax, n_p * sizeof(double), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ratio, d_ratio, n_p * sizeof(double), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(DSK_ERR_CUDA, "dsk_spectral_cluster: %s", cudaGetErrorString(e));
  } while (false);
  const cudaError_t fe = cudaFreeAsync(ws, s);
  if (rc) return rc;
  if (fe != cudaSuccess) return fail(DSK_ERR_CUDA, "dsk_spectral_cluster: cudaFreeAsync failed: %s", cudaGetErrorString(fe));
  *k_out = hsel[1];
  *p_index_out = hsel[2];
  return DSK_OK;
}


// =================================================================================================
// Serving pipeline (dsk_pipeline_*): the reference's test() loop (train_triplet.py:337-350) moves a batch to the GPU,
// runs the model and pulls the result back, all on one stream and all driven from Python.  Here one call per batch
// queues: H2D copy of the pinned input into a device slot (copy stream) -> eval forward on the next compute lane
// (its own handle / activation workspace; lanes share one packed weight image) -> D2H copy of the embeddings (second
// copy stream).  Ordering is by CUDA events only; the host never blocks in submit, and the whole submit is ~12 CUDA
// runtime calls issued from C++ (the Python pipeline spent 0.12-0.18 ms per batch on the host against a 0.2 ms GPU step).
// =================================================================================================
struct dsk_pipeline_s {
  dsk_handle primary = nullptr;
  int device = 0;
  int lanes = 0, depth = 0;
  std::vector<dsk_handle> handle;          // [lanes], all owned: each borrows the primary's packed weights
  std::vector<cudaStream_t> lane_stream;   // [lanes]
  cudaStream_t h2d = nullptr, d2h = nullptr;
  struct Slot {
    float* x = nullptr;
    float* emb = nullptr;
    size_t x_bytes = 0, emb_bytes = 0;
    cudaEvent_t h2d_done = nullptr, fwd_done = nullptr, d2h_done = nullptr;
    long long ticket = -1;
  };
  std::vector<Slot> slot;                  // [lanes * depth]
  std::vector<cudaEvent_t> join_ev;        // [lanes]
  cudaEvent_t in_ev = nullptr;
  long long next = 0;
};

static int pipeline_slot_fit(dsk_pipeline_s* p, dsk_pipeline_s::Slot& s, size_t xb, size_t eb) {
  if (s.x_bytes < xb) {
    if (s.x) {
      CUDA_TRY(cudaEventSynchronize(s.fwd_done));  // the forward that read the old buffer
      CUDA_TRY(cudaFree(s.x));
    }
    s.x = nullptr;
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&s.x), xb));
    s.x_bytes = xb;
  }
  if (s.emb_bytes < eb) {
    if (s.emb) {
      CUDA_TRY(cudaEventSynchronize(s.d2h_done));
      CUDA_TRY(cudaFree(s.emb));
    }
    s.emb = nullptr;
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&s.emb), eb));
    s.emb_bytes = eb;
  }
  (void)p;
  return DSK_OK;
}

int32_t dsk_pipeline_create(dsk_pipeline* out, dsk_handle primary, int32_t lanes, int32_t depth) {
  if (!out) return fail(DSK_ERR_INVALID, "dsk_pipeline_create: out is null");
  int rc = check_handle(primary);
  if (rc) return rc;
  if (primary->src) return fail(DSK_ERR_INVALID, "dsk_pipeline_create: the primary handle must own its weights");
  if (lanes < 1 || lanes > 8 || depth < 1 || depth > 16) return fail(DSK_ERR_INVALID, "dsk_pipeline_create: lanes 1..8, depth 1..16");
  dsk_pipeline_s* p = new dsk_pipeline_s();
  p->primary = primary;
  p->device = primary->device;
  p->lanes = lanes;
  p->depth = depth;
  p->handle.assign(lanes, nullptr);
  p->lane_stream.assign(lanes, nullptr);
  p->join_ev.assign(lanes, nullptr);
  p->slot.resize(static_cast<size_t>(lanes) * depth);
  auto bail = [&](int code) {
    dsk_pipeline_destroy(p);
    return code;
  };
  for (int i = 0; i < lanes; ++i) {  // the primary itself stays free for the caller's own stream
    rc = dsk_create(&p->handle[i], primary->device, primary->bf16 ? DSK_BF16 : DSK_F16);
    if (rc) return bail(rc);
    rc = dsk_share_weights(p->handle[i], primary);
    if (rc) return bail(rc);
  }
  for (int i = 0; i < lanes; ++i) {
    if (cudaStreamCreateWithFlags(&p->lane_stream[i], cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&p->join_ev[i], cudaEventDisableTiming) != cudaSuccess)
      return bail(fail(DSK_ERR_CUDA, "dsk_pipeline_create: stream / event creation failed"));
  }
  if (cudaStreamCreateWithFlags(&p->h2d, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&p->d2h, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->in_ev, cudaEventDisableTiming) != cudaSuccess)
    return bail(fail(DSK_ERR_CUDA, "dsk_pipeline_create: stream creation failed"));
  for (auto& s : p->slot) {
    if (cudaEventCreateWithFlags(&s.h2d_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.fwd_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.d2h_done, cudaEventDisableTiming) != cudaSuccess)
      return bail(fail(DSK_ERR_CUDA, "dsk_pipeline_create: event creation failed"));
  }
  *out = p;
  return DSK_OK;
}

int32_t dsk_pipeline_destroy(dsk_pipeline p) {
  if (!p) return DSK_OK;
  cudaSetDevice(p->device);
  for (cudaStream_t s : p->lane_stream)
    if (s) cudaStreamSynchronize(s);
  if (p->h2d) cudaStreamSynchronize(p->h2d);
  if (p->d2h) cudaStreamSynchronize(p->d2h);
  for (dsk_handle h : p->handle)
    if (h) dsk_destroy(h);
  for (auto& s : p->slot) {
    cudaFree(s.x);
    cudaFree(s.emb);
    if (s.h2d_done) cudaEventDestroy(s.h2d_done);
    if (s.fwd_done) cudaEventDestroy(s.fwd_done);
    if (s.d2h_done) cudaEventDestroy(s.d2h_done);
  }
  for (cudaEvent_t e : p->join_ev)
    if (e) cudaEventDestroy(e);
  if (p->in_ev) cudaEventDestroy(p->in_ev);
  for (cudaStream_t s : p->lane_stream)
    if (s) cudaStreamDestroy(s);
  if (p->h2d) cudaStreamDestroy(p->h2d);
  if (p->d2h) cudaStreamDestroy(p->d2h);
  delete p;
  return DSK_OK;
}

int32_t dsk_pipeline_submit(dsk_pipeline p, const float* x_host, int32_t B, int32_t T, float* emb_host, int64_t* ticket) {
  if (!p || !x_host || !emb_host || B <= 0) return fail(DSK_ERR_INVALID, "dsk_pipeline_submit: bad arguments");
  if (T < 16 || T % 16) return fail(DSK_ERR_INVALID, "dsk_pipeline_submit: T must be a positive multiple of 16 (got %d)", T);
  CUDA_TRY(cudaSetDevice(p->device));
  const long long i = p->next;
  const int lane = static_cast<int>(i % p->lanes);
  dsk_pipeline_s::Slot& s = p->slot[static_cast<size_t>(i % (static_cast<long long>(p->lanes) * p->depth))];
  const size_t xb = static_cast<size_t>(B) * T * 64 * sizeof(float);
  const size_t eb = static_cast<size_t>(B) * p->primary->emb * sizeof(float);
  int rc = pipeline_slot_fit(p, s, xb, eb);
  if (rc) return rc;
  cudaStream_t ls = p->lane_stream[lane];
  if (s.ticket >= 0) CUDA_TRY(cudaStreamWaitEvent(p->h2d, s.fwd_done, 0));  // the forward that read this slot's input
  CUDA_TRY(cudaMemcpyAsync(s.x, x_host, xb, cudaMemcpyHostToDevice, p->h2d));
  CUDA_TRY(cudaEventRecord(s.h2d_done, p->h2d));
  CUDA_TRY(cudaStreamWaitEvent(ls, s.h2d_done, 0));
  if (s.ticket >= 0) CUDA_TRY(cudaStreamWaitEvent(ls, s.d2h_done, 0));       // the copy that read this slot's embeddings
  rc = dsk_rescnn_forward(p->handle[lane], s.x, B, T, s.emb, DSK_EVAL, ls);
  if (rc) return rc;
  CUDA_TRY(cudaEventRecord(s.fwd_done, ls));
  CUDA_TRY(cudaStreamWaitEvent(p->d2h, s.fwd_done, 0));
  CUDA_TRY(cudaMemcpyAsync(emb_host, s.emb, eb, cudaMemcpyDeviceToHost, p->d2h));
  CUDA_TRY(cudaEventRecord(s.d2h_done, p->d2h));
  s.ticket = i;
  p->next = i + 1;
  if (ticket) *ticket = i;
  return DSK_OK;
}

int32_t dsk_pipeline_submit_device(dsk_pipeline p, const float* x_dev, int32_t B, int32_t T, float* emb_dev, void* after_stream,
                                   int64_t* ticket) {
  if (!p || !x_dev || !emb_dev || B <= 0) return fail(DSK_ERR_INVALID, "dsk_pipeline_submit_device: bad arguments");
  CUDA_TRY(cudaSetDevice(p->device));
  const long long i = p->next;
  const int lane = static_cast<int>(i % p->lanes);
  cudaStream_t ls = p->lane_stream[lane];
  // the inputs (and the output buffer's previous use) are ordered on the caller's stream
  CUDA_TRY(cudaEventRecord(p->in_ev, static_cast<cudaStream_t>(after_stream)));
  CUDA_TRY(cudaStreamWaitEvent(ls, p->in_ev, 0));
  int rc = dsk_rescnn_forward(p->handle[lane], x_dev, B, T, emb_dev, DSK_EVAL, ls);
  if (rc) return rc;
  p->next = i + 1;
  if (ticket) *ticket = i;
  return DSK_OK;
}

int32_t dsk_pipeline_join(dsk_pipeline p, void* stream) {
  if (!p) return fail(DSK_ERR_INVALID, "dsk_pipeline_join: null pipeline");
  CUDA_TRY(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < p->lanes; ++i) {
    CUDA_TRY(cudaEventRecord(p->join_ev[i], p->lane_stream[i]));
    CUDA_TRY(cudaStreamWaitEvent(st, p->join_ev[i], 0));
  }
  return DSK_OK;
}

int32_t dsk_pipeline_wait(dsk_pipeline p, int64_t ticket) {
  if (!p || ticket < 0 || ticket >= p->next) return fail(DSK_ERR_INVALID, "dsk_pipeline_wait: unknown ticket");
  CUDA_TRY(cudaSetDevice(p->device));
  dsk_pipeline_s::Slot& s = p->slot[static_cast<size_t>(ticket % (static_cast<long long>(p->lanes) * p->depth))];
  if (s.ticket == ticket) CUDA_TRY(cudaEventSynchronize(s.d2h_done));
  // a ticket whose slot has been reused was completed before the reuse was allowed to start (or was a device submit)
  else if (s.ticket < ticket) {
    for (cudaStream_t ls : p->lane_stream) CUDA_TRY(cudaStreamSynchronize(ls));
  }
  return DSK_OK;
}

int32_t dsk_pipeline_sync(dsk_pipeline p) {
  if (!p) return fail(DSK_ERR_INVALID, "dsk_pipeline_sync: null pipeline");
  CUDA_TRY(cudaSetDevice(p->device));
  CUDA_TRY(cudaStreamSynchronize(p->h2d));
  for (cudaStream_t ls : p->lane_stream) CUDA_TRY(cudaStreamSynchronize(ls));
  CUDA_TRY(cudaStreamSynchronize(p->d2h));
  return DSK_OK;
}

int32_t dsk_pipeline_lane_stream(dsk_pipeline p, int32_t lane, void** stream_out) {
  if (!p || lane < -2 || lane >= p->lanes || !stream_out) return fail(DSK_ERR_INVALID, "dsk_pipeline_lane_stream: bad arguments");
  *stream_out = lane == -1 ? p->h2d : lane == -2 ? p->d2h : p->lane_stream[lane];
  return DSK_OK;
}


// ---- log-fbank front-end (audio_processing.py:9-36) ------------------------------------------------------------------
static long fbank_round_half_up(double v) { return static_cast<long>(std::floor(v + 0.5)); }

// A rate the front-end can frame: a 10 ms step of at least one sample (a zero step has no frame count) and a 25 ms
// frame within NFFT = 512, that is DSK_FBANK_MIN_RATE <= sample_rate <= DSK_FBANK_MAX_RATE.
static bool fbank_rate_ok(int32_t sample_rate) {
  return sample_rate > 0 && fbank_round_half_up(0.01 * sample_rate) >= 1 &&
         fbank_round_half_up(0.025 * sample_rate) <= dsk::kFbNfft;
}

#define FBANK_RATE_MSG "sample_rate must lie in [50, 20499] Hz"

int64_t dsk_fbank_num_frames(int64_t n_samples, int32_t sample_rate) {
  if (n_samples <= 0 || !fbank_rate_ok(sample_rate)) return 0;
  const long flen = fbank_round_half_up(0.025 * sample_rate), step = fbank_round_half_up(0.01 * sample_rate);
  if (n_samples <= flen) return 1;
  return 1 + static_cast<int64_t>(std::ceil((static_cast<double>(n_samples) - flen) / step));
}

int32_t dsk_fbank_frame_offsets(const int64_t* sample_off, int32_t U, int32_t sample_rate, int64_t* frame_off) {
  if (!sample_off || !frame_off || U < 1 || sample_off[0] < 0)
    return fail(DSK_ERR_INVALID, "dsk_fbank_frame_offsets: bad arguments (need non-null offsets, U >= 1, "
                "sample_off[0] >= 0; got U %d)", U);
  if (!fbank_rate_ok(sample_rate))
    return fail(DSK_ERR_INVALID, "dsk_fbank_frame_offsets: " FBANK_RATE_MSG ", got %d", sample_rate);
  frame_off[0] = 0;
  for (int32_t u = 0; u < U; ++u) {
    const int64_t len = sample_off[u + 1] - sample_off[u];
    if (len <= 0 || len >= (1ll << 31))
      return fail(DSK_ERR_INVALID, "dsk_fbank_frame_offsets: utterance %d has %lld samples (need 1 <= n < 2^31)", u,
                  static_cast<long long>(len));
    frame_off[u + 1] = frame_off[u] + dsk_fbank_num_frames(len, sample_rate);
  }
  return DSK_OK;
}

int32_t dsk_fbank_filterbank(int32_t sample_rate, float* fb) {
  if (!fb) return fail(DSK_ERR_INVALID, "dsk_fbank_filterbank: fb is null");
  if (!fbank_rate_ok(sample_rate))
    return fail(DSK_ERR_INVALID, "dsk_fbank_filterbank: " FBANK_RATE_MSG ", got %d", sample_rate);
  // python_speech_features.get_filterbanks(nfilt=64, nfft=512, samplerate, lowfreq=0, highfreq=samplerate/2)
  std::fill(fb, fb + static_cast<size_t>(dsk::kFbFilters) * dsk::kFbBins, 0.f);
  auto hz2mel = [](double hz) { return 2595.0 * std::log10(1.0 + hz / 700.0); };
  auto mel2hz = [](double mel) { return 700.0 * (std::pow(10.0, mel / 2595.0) - 1.0); };
  const double lowmel = hz2mel(0.0), highmel = hz2mel(sample_rate / 2.0);
  double bin[dsk::kFbFilters + 2];
  for (int i = 0; i < dsk::kFbFilters + 2; ++i) {
    const double mel = lowmel + (highmel - lowmel) * i / (dsk::kFbFilters + 1);
    bin[i] = std::floor((dsk::kFbNfft + 1) * mel2hz(mel) / sample_rate);
  }
  for (int j = 0; j < dsk::kFbFilters; ++j) {
    for (int i = static_cast<int>(bin[j]); i < static_cast<int>(bin[j + 1]); ++i)
      fb[j * dsk::kFbBins + i] = static_cast<float>((i - bin[j]) / (bin[j + 1] - bin[j]));
    for (int i = static_cast<int>(bin[j + 1]); i < static_cast<int>(bin[j + 2]); ++i)
      fb[j * dsk::kFbBins + i] = static_cast<float>((bin[j + 2] - i) / (bin[j + 2] - bin[j + 1]));
  }
  return DSK_OK;
}

struct FbankVad {
  double energy_threshold, mean_scale, proportion;
  int32_t context;
  float* energy;      // may be null
  uint8_t* speech;
};

// dsk_fbank_batch, and with vad the energies and speech decisions of the same frames (the features do not depend on it)
static int32_t fbank_batch(const float* audio, const int64_t* sample_off, int32_t U, int32_t sample_rate, int32_t log_scale,
                           int32_t subtract_mean, float* feat, const FbankVad* vad, void* stream) {
  if (!audio || !feat || !sample_off || U < 1)
    return fail(DSK_ERR_INVALID, "dsk_fbank_batch: bad arguments (need non-null pointers and U >= 1; got U %d)", U);
  if (!fbank_rate_ok(sample_rate)) return fail(DSK_ERR_INVALID, "dsk_fbank_batch: " FBANK_RATE_MSG ", got %d", sample_rate);
  const long flen = fbank_round_half_up(0.025 * sample_rate), step = fbank_round_half_up(0.01 * sample_rate);
  std::vector<int64_t> off(3 * (static_cast<size_t>(U) + 1));   // soff | foff | boff
  std::copy(sample_off, sample_off + U + 1, off.begin());
  int64_t* foff = off.data() + (U + 1);
  int64_t* boff = foff + (U + 1);
  if (int32_t rc = dsk_fbank_frame_offsets(sample_off, U, sample_rate, foff)) return rc;
  boff[0] = 0;
  for (int32_t u = 0; u < U; ++u)
    boff[u + 1] = boff[u] + (foff[u + 1] - foff[u] + dsk::kFbFramesPerBlock - 1) / dsk::kFbFramesPerBlock;
  const int64_t nblk = boff[U];
  if (nblk >= (1ll << 31)) return fail(DSK_ERR_INVALID, "dsk_fbank_batch: %lld frames exceed one launch", static_cast<long long>(foff[U]));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // built once per call for all U utterances
  std::vector<float> fb(static_cast<size_t>(dsk::kFbFilters) * dsk::kFbBins);
  if (int32_t rc = dsk_fbank_filterbank(sample_rate, fb.data())) return rc;
  // scratch: the three offset tables (int64) | [64][257] filterbank | [nblk][64] column-sum partials | [U][64] means,
  // then with vad: ln E [F] | block partials [nblk] | thresholds [U] (fp64) | energies [F] fp32 when vad->energy is null
  const size_t off_bytes = off.size() * sizeof(int64_t), fb_bytes = fb.size() * sizeof(float);
  const size_t fbank_bytes = off_bytes + fb_bytes + (static_cast<size_t>(nblk) + U) * dsk::kFbFilters * sizeof(float);
  const int64_t F = foff[U];
  const size_t vad_bytes = !vad ? 0 : (static_cast<size_t>(F) + nblk + U) * sizeof(double) +
                                          (vad->energy ? 0 : static_cast<size_t>(F) * sizeof(float));
  const size_t bytes = fbank_bytes + vad_bytes;
  char* scratch = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&scratch), bytes, s));
  CUDA_TRY(cudaMemcpyAsync(scratch, off.data(), off_bytes, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(scratch + off_bytes, fb.data(), fb_bytes, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaStreamSynchronize(s));  // off / fb are call-lifetime host vectors (pageable copies): the call's one sync
  const int64_t* d_soff = reinterpret_cast<const int64_t*>(scratch);
  const int64_t* d_foff = d_soff + (U + 1);
  const int64_t* d_boff = d_foff + (U + 1);
  const float* d_fb = reinterpret_cast<const float*>(scratch + off_bytes);
  float* partial = reinterpret_cast<float*>(scratch + off_bytes + fb_bytes);
  float* mean = partial + nblk * dsk::kFbFilters;
  double* loge = reinterpret_cast<double*>(scratch + fbank_bytes);
  double* lpartial = loge + F;
  double* thr = lpartial + nblk;
  float* energy = vad ? (vad->energy ? vad->energy : reinterpret_cast<float*>(thr + U)) : nullptr;
  dsk::fbank_kernel<<<static_cast<unsigned>(nblk), dsk::kFbThreads, 0, s>>>(audio, d_soff, d_foff, d_boff, U, static_cast<int>(flen),
                                                                            static_cast<int>(step), 0.97f, d_fb, log_scale, 1e-5f,
                                                                            feat, partial, energy);
  KERNEL_CHECK();
  if (subtract_mean) {
    dsk::fbank_mean_kernel<<<static_cast<unsigned>((static_cast<long>(U) * dsk::kFbFilters + 255) / 256), 256, 0, s>>>(partial, d_foff, d_boff, U, mean);
    KERNEL_CHECK();
    dsk::fbank_mean_sub_kernel<<<static_cast<unsigned>(nblk), dsk::kFbThreads, 0, s>>>(feat, d_foff, d_boff, U, mean);
    KERNEL_CHECK();
  }
  if (vad) {
    dsk::vad_log_energy_kernel<<<static_cast<unsigned>((nblk + 255) / 256), 256, 0, s>>>(energy, d_foff, d_boff, U, nblk, loge,
                                                                                        lpartial);
    KERNEL_CHECK();
    dsk::vad_threshold_kernel<<<(U + 255) / 256, 256, 0, s>>>(lpartial, d_foff, d_boff, U, vad->energy_threshold,
                                                              vad->mean_scale, thr);
    KERNEL_CHECK();
    dsk::vad_decide_kernel<<<static_cast<unsigned>((F + 255) / 256), 256, 0, s>>>(loge, d_foff, U, thr, F, vad->context,
                                                                                 vad->proportion, vad->speech);
    KERNEL_CHECK();
  }
  CUDA_TRY(cudaFreeAsync(scratch, s));
  return DSK_OK;
}

int32_t dsk_fbank_batch(const float* audio, const int64_t* sample_off, int32_t U, int32_t sample_rate, int32_t log_scale,
                        int32_t subtract_mean, float* feat, void* stream) {
  return fbank_batch(audio, sample_off, U, sample_rate, log_scale, subtract_mean, feat, nullptr, stream);
}

int32_t dsk_fbank_batch_vad(const float* audio, const int64_t* sample_off, int32_t U, int32_t sample_rate,
                            int32_t log_scale, int32_t subtract_mean, double energy_threshold, double mean_scale,
                            int32_t context, double proportion, float* feat, float* energy, uint8_t* speech,
                            void* stream) {
  if (!speech || !std::isfinite(energy_threshold) || !std::isfinite(mean_scale) || !std::isfinite(proportion) ||
      context < 0 || proportion < 0)
    return fail(DSK_ERR_INVALID, "dsk_fbank_batch_vad: bad VAD arguments (need non-null speech, finite energy_threshold, "
                "mean_scale and proportion, context >= 0, proportion >= 0; got %g, %g, %d, %g)", energy_threshold,
                mean_scale, context, proportion);
  const FbankVad vad{energy_threshold, mean_scale, proportion, context, energy, speech};
  return fbank_batch(audio, sample_off, U, sample_rate, log_scale, subtract_mean, feat, &vad, stream);
}

int32_t dsk_frame_runs(const uint8_t* mask, const int64_t* frame_off, int32_t U, const int64_t* utt,
                       const int64_t* list_off, int32_t K, int64_t P, int64_t capacity, int64_t* runs, int64_t* run_off,
                       int64_t* counts, void* stream) {
  if (!mask || !frame_off || !utt || !list_off || !runs || !run_off || !counts || U < 1 || K < 1 || P < K ||
      capacity < 0)
    return fail(DSK_ERR_INVALID, "dsk_frame_runs: bad arguments (need non-null pointers, U, K >= 1, P >= K, capacity >= 0; "
                "got U %d, K %d, P %lld, capacity %lld)", U, K, static_cast<long long>(P), static_cast<long long>(capacity));
  const int64_t ntiles = (P + dsk::kRunTile - 1) / dsk::kRunTile;
  if (ntiles >= (1ll << 31)) return fail(DSK_ERR_INVALID, "dsk_frame_runs: %lld frames exceed one launch", static_cast<long long>(P));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // scratch: tile run starts [ntiles] | tile kept frames [ntiles] | totals [2]
  int64_t* scratch = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&scratch), (2 * ntiles + 2) * sizeof(int64_t), s));
  int64_t* tile_starts = scratch;
  int64_t* tile_kept = scratch + ntiles;
  int64_t* totals = tile_kept + ntiles;
  dsk::run_count_kernel<<<static_cast<unsigned>(ntiles), dsk::kRunThreads, 0, s>>>(mask, frame_off, utt, list_off, K, P,
                                                                                  tile_starts, tile_kept);
  KERNEL_CHECK();
  dsk::run_scan_kernel<<<1, dsk::kRunThreads, 0, s>>>(tile_starts, tile_kept, ntiles, capacity, run_off, totals);
  KERNEL_CHECK();
  dsk::run_write_kernel<<<static_cast<unsigned>(ntiles), dsk::kRunThreads, 0, s>>>(mask, frame_off, utt, list_off, K, P,
                                                                                  tile_starts, tile_kept, capacity, runs,
                                                                                  run_off);
  KERNEL_CHECK();
  CUDA_TRY(cudaMemcpyAsync(counts, totals, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaFreeAsync(scratch, s));
  CUDA_TRY(cudaStreamSynchronize(s));   // the call's one host read: the run count sizes the caller's next step
  if (counts[0] > capacity)
    return fail(DSK_ERR_INVALID, "dsk_frame_runs: %lld runs exceed the capacity %lld", static_cast<long long>(counts[0]),
                static_cast<long long>(capacity));
  return DSK_OK;
}

int32_t dsk_gather_runs(const float* feat, const int64_t* frame_off, int32_t U, const int64_t* utt, const int64_t* runs,
                        const int64_t* run_off, int64_t n_runs, int64_t rows, float* out, void* stream) {
  if (!feat || !frame_off || !utt || !runs || !run_off || !out || U < 1 || n_runs < 1 || rows < n_runs)
    return fail(DSK_ERR_INVALID, "dsk_gather_runs: bad arguments (need non-null pointers, U, n_runs >= 1, rows >= n_runs; "
                "got U %d, n_runs %lld, rows %lld)", U, static_cast<long long>(n_runs), static_cast<long long>(rows));
  if ((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(out)) & 15)
    return fail(DSK_ERR_INVALID, "dsk_gather_runs: feat and out must be 16-byte aligned");
  const int64_t grid = (rows + dsk::kRunGatherRows - 1) / dsk::kRunGatherRows;
  if (grid >= (1ll << 31)) return fail(DSK_ERR_INVALID, "dsk_gather_runs: %lld rows exceed one launch", static_cast<long long>(rows));
  dsk::run_gather_kernel<<<static_cast<unsigned>(grid), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      feat, frame_off, utt, runs, run_off, n_runs, rows, out);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_fbank(const float* audio, int64_t n_samples, int32_t sample_rate, int32_t log_scale, int32_t subtract_mean,
                  float* feat, void* stream) {
  if (!audio || !feat || n_samples <= 0 || n_samples >= (1ll << 31))
    return fail(DSK_ERR_INVALID, "dsk_fbank: bad arguments");
  if (!fbank_rate_ok(sample_rate)) return fail(DSK_ERR_INVALID, "dsk_fbank: " FBANK_RATE_MSG ", got %d", sample_rate);
  const int64_t sample_off[2] = {0, n_samples};
  return dsk_fbank_batch(audio, sample_off, 1, sample_rate, log_scale, subtract_mean, feat, stream);
}

int32_t dsk_fbank_crops(const float* feat, const int64_t* frame_off, int32_t U, const int64_t* utt, const int64_t* start,
                        int32_t B, int32_t T, const int32_t* time_masks, int32_t n_time, const int32_t* freq_masks,
                        int32_t n_freq, float* out, void* stream) {
  if (!feat || !frame_off || !utt || !start || !out || U < 1 || B < 1 || T < 1 || n_time < 0 || n_freq < 0 ||
      (n_time > 0 && !time_masks) || (n_freq > 0 && !freq_masks))
    return fail(DSK_ERR_INVALID, "dsk_fbank_crops: bad arguments (need non-null pointers, U, B, T >= 1, n_time, n_freq >= 0 "
                "with their masks; got U %d, B %d, T %d, n_time %d, n_freq %d)", U, B, T, n_time, n_freq);
  if ((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(out)) & 15)
    return fail(DSK_ERR_INVALID, "dsk_fbank_crops: feat and out must be 16-byte aligned");
  const int64_t grid = static_cast<int64_t>(B) * ((T + dsk::kCropRows - 1) / dsk::kCropRows);
  if (grid >= (1ll << 31)) return fail(DSK_ERR_INVALID, "dsk_fbank_crops: %d crops of %d frames exceed one launch", B, T);
  dsk::fbank_crop_kernel<<<static_cast<unsigned>(grid), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      feat, frame_off, U, utt, start, T, time_masks, n_time, freq_masks, n_freq, out);
  KERNEL_CHECK();
  return DSK_OK;
}

int32_t dsk_fbank_segments(const float* audio, int32_t B, int32_t L, int32_t sample_rate, int32_t log_scale,
                           int32_t subtract_mean, const float* fb, const int32_t* time_masks, int32_t n_time,
                           const int32_t* freq_masks, int32_t n_freq, float* out, void* stream) {
  if (!audio || !fb || !out || B < 1 || L < 1 || n_time < 0 || n_freq < 0 || (n_time > 0 && !time_masks) ||
      (n_freq > 0 && !freq_masks))
    return fail(DSK_ERR_INVALID, "dsk_fbank_segments: bad arguments (need non-null pointers, B, L >= 1, "
                "n_time, n_freq >= 0 with their masks; got B %d, L %d, n_time %d, n_freq %d)", B, L, n_time, n_freq);
  if (!fbank_rate_ok(sample_rate)) return fail(DSK_ERR_INVALID, "dsk_fbank_segments: " FBANK_RATE_MSG ", got %d", sample_rate);
  if (reinterpret_cast<uintptr_t>(out) & 15) return fail(DSK_ERR_INVALID, "dsk_fbank_segments: out must be 16-byte aligned");
  const long flen = fbank_round_half_up(0.025 * sample_rate), step = fbank_round_half_up(0.01 * sample_rate);
  const int64_t T = dsk_fbank_num_frames(L, sample_rate);
  const int64_t blocks_per = (T + dsk::kFbFramesPerBlock - 1) / dsk::kFbFramesPerBlock, nblk = blocks_per * B;
  const int64_t mask_grid = static_cast<int64_t>(B) * ((T + dsk::kCropRows - 1) / dsk::kCropRows);
  if (nblk >= (1ll << 31) || mask_grid >= (1ll << 31))
    return fail(DSK_ERR_INVALID, "dsk_fbank_segments: %d segments of %lld frames exceed one launch", B, static_cast<long long>(T));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // scratch: soff | foff | boff (B + 1 each, int64) | [nblk][64] column-sum partials | [B][64] means
  const size_t off_bytes = 3 * (static_cast<size_t>(B) + 1) * sizeof(int64_t);
  const size_t bytes = off_bytes + (static_cast<size_t>(nblk) + B) * dsk::kFbFilters * sizeof(float);
  char* scratch = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&scratch), bytes, s));
  int64_t* d_soff = reinterpret_cast<int64_t*>(scratch);
  int64_t* d_foff = d_soff + (B + 1);
  int64_t* d_boff = d_foff + (B + 1);
  float* partial = reinterpret_cast<float*>(scratch + off_bytes);
  float* mean = partial + nblk * dsk::kFbFilters;
  dsk::fbank_regular_offsets_kernel<<<(B + 1 + 255) / 256, 256, 0, s>>>(B, L, static_cast<int>(T), d_soff, d_foff, d_boff);
  KERNEL_CHECK();
  // (B, 1, T, 64) is the (B T, 64) layout of the B segments' frames: the features are written straight into out
  dsk::fbank_kernel<<<static_cast<unsigned>(nblk), dsk::kFbThreads, 0, s>>>(audio, d_soff, d_foff, d_boff, B, static_cast<int>(flen),
                                                                            static_cast<int>(step), 0.97f, fb, log_scale, 1e-5f,
                                                                            out, partial);
  KERNEL_CHECK();
  if (subtract_mean) {
    dsk::fbank_mean_kernel<<<static_cast<unsigned>((static_cast<long>(B) * dsk::kFbFilters + 255) / 256), 256, 0, s>>>(partial, d_foff, d_boff, B, mean);
    KERNEL_CHECK();
    dsk::fbank_mean_sub_kernel<<<static_cast<unsigned>(nblk), dsk::kFbThreads, 0, s>>>(out, d_foff, d_boff, B, mean);
    KERNEL_CHECK();
  }
  if (n_time > 0 || n_freq > 0) {
    dsk::fbank_mask_kernel<<<static_cast<unsigned>(mask_grid), 256, 0, s>>>(out, static_cast<int>(T), time_masks, n_time,
                                                                            freq_masks, n_freq);
    KERNEL_CHECK();
  }
  CUDA_TRY(cudaFreeAsync(scratch, s));
  return DSK_OK;
}

// A bank pointer as the kernels read it: device (or managed) memory as is, page-locked host memory through its mapped
// device address.  Pageable host memory is rejected: the kernels could not read it, and a copy would synchronise.
static int32_t aug_resolve(const void* p, const void** dev, const char* what) {
  cudaPointerAttributes a{};
  CUDA_TRY(cudaPointerGetAttributes(&a, p));
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
    *dev = p;
    return DSK_OK;
  }
  if (a.type == cudaMemoryTypeHost) {
    void* d = nullptr;
    CUDA_TRY(cudaHostGetDevicePointer(&d, const_cast<void*>(p), 0));
    *dev = d;
    return DSK_OK;
  }
  return fail(DSK_ERR_INVALID, "dsk_wave_augment: %s is pageable host memory (use device or page-locked memory)", what);
}

int32_t dsk_speed_filter(int32_t p, int32_t q, float* taps) {
  if (!taps || p < 1 || q < 1 || q > dsk::kSpeedMaxDen || 2 * p < q || p > 2 * q || std::gcd(p, q) != 1)
    return fail(DSK_ERR_INVALID, "dsk_speed_filter: bad arguments (need non-null taps and p / q in lowest terms with "
                "1/2 <= p / q <= 2, q <= %d; got %d / %d)", dsk::kSpeedMaxDen, p, q);
  const double pi = 3.141592653589793;
  const double fc = 0.5 * 0.99 * std::min(1.0, static_cast<double>(q) / static_cast<double>(p));
  const double zs = 12.0 / (2.0 * fc);
  for (int32_t r = 0; r < q; ++r) {
    for (int32_t j = 0; j < dsk::kSpeedTaps; ++j) {
      const double tau = static_cast<double>(r) / static_cast<double>(q) - static_cast<double>(j - (dsk::kSpeedTaps / 2 - 1));
      double h = 0.0;
      if (std::fabs(tau) <= zs) {
        const double x = 2.0 * fc * tau;
        const double sinc = x == 0.0 ? 1.0 : std::sin(pi * x) / (pi * x);
        const double w = std::cos(pi * tau / (2.0 * zs));
        h = 2.0 * fc * sinc * (w * w);
      }
      taps[r * dsk::kSpeedTaps + j] = static_cast<float>(h);
    }
  }
  return DSK_OK;
}

int32_t dsk_wave_augment(const int16_t* speech, const int64_t* speech_off, int32_t U, const int64_t* utt,
                         const int64_t* start, int32_t B, int32_t L, const float* rir, const int64_t* rir_off, int32_t R,
                         int32_t max_rir_len, const int64_t* rir_idx, const int16_t* noise, const int64_t* noise_off,
                         int32_t N, int32_t M, const int64_t* noise_idx, const int64_t* noise_start, const double* snr_db,
                         float* out, void* stream) {
  return dsk_wave_augment_speed(speech, speech_off, U, utt, start, B, L, rir, rir_off, R, max_rir_len, rir_idx, noise,
                                noise_off, N, M, noise_idx, noise_start, snr_db, nullptr, nullptr, 0, nullptr, out, stream);
}

int32_t dsk_wave_augment_speed(const int16_t* speech, const int64_t* speech_off, int32_t U, const int64_t* utt,
                               const int64_t* start, int32_t B, int32_t L, const float* rir, const int64_t* rir_off,
                               int32_t R, int32_t max_rir_len, const int64_t* rir_idx, const int16_t* noise,
                               const int64_t* noise_off, int32_t N, int32_t M, const int64_t* noise_idx,
                               const int64_t* noise_start, const double* snr_db, const int32_t* speed_ratio,
                               const float* speed_taps, int32_t K, const int64_t* speed_idx, float* out, void* stream) {
  if (!speech || !speech_off || !utt || !start || !out || U < 1 || B < 1 || L < 1 || L > (1 << 24) || M < 0 ||
      M > dsk::kAugMaxSources || max_rir_len < 1 || max_rir_len > dsk::kAugMaxRir)
    return fail(DSK_ERR_INVALID, "dsk_wave_augment: bad arguments (need non-null speech, offsets, utt, start, out; U, B >= 1; "
                "1 <= L <= 2^24; 0 <= M <= %d; 1 <= max_rir_len <= %d; got U %d, B %d, L %d, M %d, max_rir_len %d)",
                dsk::kAugMaxSources, dsk::kAugMaxRir, U, B, L, M, max_rir_len);
  if (rir_idx && (!rir || !rir_off || R < 1))
    return fail(DSK_ERR_INVALID, "dsk_wave_augment: rir_idx needs a RIR bank (non-null rir, rir_off and R >= 1; got R %d)", R);
  if (M > 0 && (!noise || !noise_off || N < 1 || !noise_idx || !noise_start || !snr_db))
    return fail(DSK_ERR_INVALID, "dsk_wave_augment: M = %d sources need a noise bank (N >= 1; got %d) and non-null "
                "noise_idx, noise_start, snr_db", M, N);
  if (K < 0 || K > dsk::kSpeedMaxFactors || (K > 0 && (!speed_ratio || !speed_taps || !speed_idx)))
    return fail(DSK_ERR_INVALID, "dsk_wave_augment: need 0 <= K <= %d speed factors, with non-null speed_ratio, "
                "speed_taps and speed_idx when K > 0; got K %d", dsk::kSpeedMaxFactors, K);
  const int64_t tiles = (L + dsk::kAugGatherPerBlock - 1) / dsk::kAugGatherPerBlock;
  const int64_t nb = (L + dsk::kAugPart - 1) / dsk::kAugPart, kp = (max_rir_len + dsk::kAugPart - 1) / dsk::kAugPart;
  if (B * tiles >= (1ll << 31) || B * nb >= (1ll << 31) || B * kp >= (1ll << 31))
    return fail(DSK_ERR_INVALID, "dsk_wave_augment: %d segments of %d samples exceed one launch", B, L);
  const void *sp = nullptr, *sop = nullptr, *rp = nullptr, *rop = nullptr, *np_ = nullptr, *nop = nullptr;
  if (int32_t rc = aug_resolve(speech, &sp, "the speech bank")) return rc;
  if (int32_t rc = aug_resolve(speech_off, &sop, "the speech offsets")) return rc;
  if (rir_idx) {
    if (int32_t rc = aug_resolve(rir, &rp, "the RIR bank")) return rc;
    if (int32_t rc = aug_resolve(rir_off, &rop, "the RIR offsets")) return rc;
  }
  if (M > 0) {
    if (int32_t rc = aug_resolve(noise, &np_, "the noise bank")) return rc;
    if (int32_t rc = aug_resolve(noise_off, &nop, "the noise offsets")) return rc;
  }
  const int16_t* d_speech = static_cast<const int16_t*>(sp);
  const int64_t* d_soff = static_cast<const int64_t*>(sop);
  const float* d_rir = static_cast<const float*>(rp);
  const int64_t* d_roff = static_cast<const int64_t*>(rop);
  const int16_t* d_noise = static_cast<const int16_t*>(np_);
  const int64_t* d_noff = static_cast<const int64_t*>(nop);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // scratch: ok (B int32, padded to 256 bytes) | X [B][nb][P + 1] | H [B][kp][P + 1] (complex fp32, reverb only)
  const size_t ok_bytes = (static_cast<size_t>(B) * sizeof(int) + 255) / 256 * 256;
  const size_t x_elems = rir_idx ? static_cast<size_t>(B) * nb * dsk::kAugBins : 0;
  const size_t h_elems = rir_idx ? static_cast<size_t>(B) * kp * dsk::kAugBins : 0;
  char* scratch = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&scratch), ok_bytes + (x_elems + h_elems) * sizeof(float2), s));
  int* ok = reinterpret_cast<int*>(scratch);
  float2* X = reinterpret_cast<float2*>(scratch + ok_bytes);
  float2* H = X + x_elems;
  dsk::aug_check_kernel<<<(B + 255) / 256, 256, 0, s>>>(d_soff, U, utt, start, B, d_roff, R, rir_idx, max_rir_len, d_noff, N, M,
                                                        noise_idx, noise_start, snr_db, speed_ratio, K, speed_idx, ok);
  KERNEL_CHECK();
  if (K > 0) {
    dsk::aug_speed_kernel<<<static_cast<unsigned>(B * tiles), dsk::kAugGatherThreads, 0, s>>>(
        d_speech, d_soff, utt, start, ok, speed_ratio, speed_taps, speed_idx, L, out);
    KERNEL_CHECK();
  }
  dsk::aug_gather_kernel<<<static_cast<unsigned>(B * tiles), dsk::kAugGatherThreads, 0, s>>>(d_speech, d_soff, utt, start, ok, L, out);
  KERNEL_CHECK();
  if (rir_idx) {
    dsk::aug_fft_in_kernel<<<static_cast<unsigned>(B * nb), dsk::kAugFftThreads, 0, s>>>(out, L, static_cast<int>(nb), ok, rir_idx,
                                                                                       d_roff, X);
    KERNEL_CHECK();
    dsk::aug_fft_rir_kernel<<<static_cast<unsigned>(B * kp), dsk::kAugFftThreads, 0, s>>>(d_rir, d_roff, ok, rir_idx,
                                                                                        static_cast<int>(kp), H);
    KERNEL_CHECK();
    dsk::aug_conv_out_kernel<<<static_cast<unsigned>(B * nb), dsk::kAugFftThreads, 0, s>>>(X, H, static_cast<int>(nb),
                                                                                         static_cast<int>(kp), ok, rir_idx,
                                                                                         d_roff, L, out);
    KERNEL_CHECK();
  }
  if (M > 0) {
    dsk::aug_mix_kernel<<<B, dsk::kAugMixThreads, 0, s>>>(d_noise, d_noff, M, noise_idx, noise_start, snr_db, ok, L, out);
    KERNEL_CHECK();
  }
  CUDA_TRY(cudaFreeAsync(scratch, s));
  return DSK_OK;
}

}  // extern "C"
