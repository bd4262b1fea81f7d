// engine.cu -- the DorPatch hot-path engine behind include/dorpatch.h.
//
// One engine per GPU.  It owns: the standardised classifier weights (ResNetV2-50x1-BiT,
// NHWC/KRSC), a workspace arena sized for `chunk` EOT samples, cuDNN + cublasLt handles.
// The classifier's 3x3 / 7x7 convolutions run on tensor cores through cuDNN, the 1x1
// convolutions (36 of 53) are plain NHWC GEMMs through cublasLt (the residual add is fused
// as the GEMM's C operand); everything else is the hand-written kernels of kernels_*.cu.
// The attack's backward is data-gradient only (the weights are frozen; the reference's unused weight gradient, SURVEY
// quirk Q7, is not computed there).  dp_eot_backward_params adds an opt-in weight-gradient pass (fine-tuning).
#include <cublasLt.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cudnn.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <map>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: no-ops unless a profiler injects itself (ncu --nvtx, nsys)

#include "../../include/dorpatch.h"
#include "kernels.h"

namespace {

thread_local std::string g_last_error;

[[noreturn]] void fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw std::runtime_error(buf);
}

#define CUDA_OK(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) fail("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
  } while (0)
#define CUDNN_OK(expr)                                                                             \
  do {                                                                                             \
    cudnnStatus_t _s = (expr);                                                                     \
    if (_s != CUDNN_STATUS_SUCCESS) fail("cuDNN error %d (%s) at %s:%d [%s]", (int)_s, cudnnGetErrorString(_s), __FILE__, __LINE__, #expr); \
  } while (0)
#define CUBLAS_OK(expr)                                                                            \
  do {                                                                                             \
    cublasStatus_t _s = (expr);                                                                    \
    if (_s != CUBLAS_STATUS_SUCCESS) fail("cuBLASLt error %d at %s:%d [%s]", (int)_s, __FILE__, __LINE__, #expr); \
  } while (0)

constexpr int DEPTHS[4] = {3, 4, 6, 3};
constexpr int WIDTHS[4] = {256, 512, 1024, 2048};
constexpr int STEM_CH = 64;
// NVTX range around the phases of the hot loop (host side; inside a graph capture they mark the capture, not the replay)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

struct ConvW {            // one convolution's weights (device, KRSC, activation dtype)
  int cin = 0, cin_pad = 0, cout = 0, k = 1, stride = 1, pad = 0;
  void* w = nullptr;
  float* raw = nullptr;     // the fp32 OIHW weights as loaded (the weight-standardisation adjoint reads them)
  int pid = -1;             // index into dp_engine::wparams
  cudnnFilterDescriptor_t wdesc = nullptr;
  cudnnConvolutionDescriptor_t cdesc = nullptr;
};
// pos: every gamma > 0 (packed bf16 ReLU gate allowed).  pid: gamma's wparams index (beta's is pid + 1).
struct GNW { int C = 0; float* gamma = nullptr; float* beta = nullptr; bool pos = false; int pid = -1; };
struct Block {
  int cin, mid, cout, stride, hin, hout;
  bool has_ds;
  GNW n1, n2, n3;
  ConvW ds, c1, c2, c3;
  void* c1p = nullptr; void* c3p = nullptr;   // conv1 / conv3 weights as wgmma operand tiles (DORPATCH_FUSED_GEMM=1)
};

struct CudnnPlan {
  cudnnTensorDescriptor_t xdesc = nullptr, ydesc = nullptr;
  cudnnConvolutionFwdAlgo_t fwd_algo; cudnnMathType_t fwd_math; size_t fwd_ws = 0; bool fwd_ready = false;
  cudnnConvolutionBwdDataAlgo_t bwd_algo; cudnnMathType_t bwd_math; size_t bwd_ws = 0; bool bwd_ready = false;
  cudnnConvolutionBwdFilterAlgo_t wgd_algo; cudnnMathType_t wgd_math; size_t wgd_ws = 0; bool wgd_ready = false;
};
struct GemmPlan {
  cublasLtMatmulDesc_t op = nullptr;
  cublasLtMatrixLayout_t a = nullptr, b = nullptr, c = nullptr;
  cublasLtMatmulAlgo_t algo;
  std::vector<cublasLtMatmulAlgo_t> candidates;   // heuristic top-k, timed on first use when autotune is on
  bool tuned = false;
};

}  // namespace

struct dp_engine {
  dp_config cfg;
  bool bf16 = false;
  size_t es = 4;            // activation element size
  bool fused_gemm = false;  // opt-in (DORPATCH_FUSED_GEMM=1, bf16): GN+ReLU applied inside the wgmma 1x1-conv GEMM of kernels_gemm.cu
  int H = 224, K = 1000, chunk = 64;
  int num_sms = 132;
  cublasLtHandle_t lt = nullptr;
  cudnnDataType_t cudnn_dt = CUDNN_DATA_FLOAT;
  cudaDataType_t cuda_dt = CUDA_R_32F;
  cublasComputeType_t lt_compute = CUBLAS_COMPUTE_32F;
  int64_t device_bytes = 0, launches = 0;
  std::vector<void*> allocs;
  bool weights_loaded = false;

  std::vector<Block> blocks;
  GNW head_gn;
  float* fc_w = nullptr; float* fc_b = nullptr;

  size_t lib_ws_bytes = 0;         // each lane's cuDNN / cublasLt workspace

  // ---- lanes: complete per-chunk workspaces (sized for `chunk` samples).  A chunk loop runs every chunk on lane 0
  // and the caller's stream, or alternates its chunks between two lanes on two internal streams (LaneWalk) so that one
  // chunk's kernel tails / memory-bound GroupNorm passes overlap the other chunk's tensor-core convolutions.  Every
  // classifier pass is given the lane whose buffers, cuDNN handle and weight-gradient accumulators it uses.
  struct Lane {
    void* net_in = nullptr;          // [chunk,H,H,stem.in_ch]
    void* act = nullptr;             // scratch activation (stem out / GN outputs)
    void* act2 = nullptr;            // scratch (subsampled shortcut input)
    void* x0 = nullptr;              // pooled stem output (saved)
    int8_t* pool_amax = nullptr;
    void* g[4] = {nullptr, nullptr, nullptr, nullptr};   // gradient scratch
    float *gn_partial = nullptr, *head_stats = nullptr, *pooled = nullptr, *dpooled = nullptr, *logits = nullptr, *dlogits = nullptr;
    void* lib_ws = nullptr;
    struct Saved { void *h1, *h2, *out; float *st1, *st2, *st3; };   // per block: saved tensors / stats for backward
    std::vector<Saved> saved;
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    cudnnHandle_t cudnn = nullptr;
    // weight gradients (dp_eot_backward_params; allocated on first use): fp32 accumulators, GroupNorm / stem partial
    // sums, bf16 cuDNN filter gradient before it is added in fp32
    float* wacc = nullptr; float* wg_partial = nullptr; void* wg_half = nullptr;
    int held = -1;                   // the dp_eot_forward chunk whose saved activations this lane holds, -1 none
  };
  std::vector<Lane> lanes;
  cudaEvent_t ev_prep = nullptr;

  // per-image buffers (max_images)
  float* adv_x = nullptr; float* dLs = nullptr; float* scale = nullptr; float* l2 = nullptr;
  float* loss_struc = nullptr; float* loss_density = nullptr; float* group_lasso = nullptr;
  float* win_dev = nullptr; float* grp_ss = nullptr;   // grp_ss: B*H*H floats, one per group at basic_unit 1
  int unit = 7;   // basic_unit of the last dp_attack_grad (attack.py:52); dp_attack_update's group-lasso term uses it
  // failed-mask sets (N2): one bitmap of failed_words words per image over failed_masks indices, its popcounts, staging
  // for one step's indices.  4096 masks until dp_failed_set_reset sizes the sets by the universe (the reference's
  // one-patch universe has 2520; the two-patch dropout-2 universe 90 720, 2835 words per image)
  int failed_masks = 4096, failed_words = 128, failed_words_alloc = 128;
  uint32_t* failed_bits = nullptr; int32_t* failed_count = nullptr; int32_t* failed_idx = nullptr; int32_t* failed_nff = nullptr;
  uint8_t* failed_active = nullptr; float* failed_loss = nullptr; int failed_cap = 0;
  // on-device EOT draw (dp_eot_universe_upload / dp_eot_draw): the universe's rectangle table [uni_n][uni_k][4], the
  // last draw's indices idx [B][S] | idx2 [B][S], nff [max_images], its local rectangles [B][S_loc][4][4] (what
  // dp_attack_grad_drawn's K1 reads) and the kernel's scratch.  The draw's parameters go through draw_pin ->
  // draw_par_d: seeds [max_images] uint64 | {stage, iter} int32 | active [max_images]; draw_ev marks the copy's end.
  int16_t* uni_d = nullptr; int uni_n = 0, uni_k = 0, uni_cap = 0;
  int32_t* draw_idx_d = nullptr; int32_t* draw_tmp_d = nullptr; int draw_cap = 0;
  int16_t* draw_rects_d = nullptr; int draw_rects_cap = 0;
  int32_t* draw_nff_d = nullptr; unsigned char* draw_par_d = nullptr; unsigned char* draw_pin = nullptr;
  cudaEvent_t draw_ev = nullptr;
  // the last draw's shape; `fresh` until dp_failed_set_update_drawn consumes it or a universe upload / set reset
  // invalidates it
  struct DrawSig { bool fresh = false; int B = 0, S = 0, S_loc = 0; bool dual = false; };
  DrawSig draw;
  size_t draw_par_bytes() const { return (size_t)cfg.max_images * 9 + 16; }
  float* helper_scale = nullptr; float* helper_l2 = nullptr; float* helper_ws = nullptr;   // scratch of dp_paste(out) / dp_window_sum
  float* lr_d = nullptr; float* structured_d = nullptr; float* coeff_d = nullptr;
  float* host_x = nullptr; float* host_mask = nullptr; float* host_pattern = nullptr; float* host_G = nullptr;  // dp_attack_step_host

  // per-sample buffers (grown on demand)
  int cap_samples = 0;
  int16_t* rects_d = nullptr; int32_t* y_d = nullptr; uint8_t* tg_d = nullptr;
  float* loss_d = nullptr; int32_t* preds_d = nullptr; float* xf_d = nullptr;
  // pinned staging
  unsigned char* pin = nullptr; size_t pin_bytes = 0;

  // ---- dp_eot_forward / dp_eot_backward: what the backward needs of the last forward.  fwd_gen is bumped by every
  // call that overwrites the lane arenas (dp_predict, dp_attack_grad, dp_net_forward_backward, dp_eot_forward, new
  // weights); a backward whose forward recorded an older generation is refused.  Lane::held is the chunk whose saved
  // activations (pre-norm outputs, GroupNorm statistics, max-pool argmax) the lane still holds.
  // xf: the forward warped its samples (dp_eot_forward_xform) with the transforms in eot_xf_d.
  // whole: the forward's K1 wrote every sample to net_in_all (a held chunk's input is its slice there).
  // bank: the forward occluded from this caller-owned mask bank with the indices in eot_bank_idx_d (dp_eot_forward_bank).
  struct EotSig { int64_t gen = -1; const float* img = nullptr; int B = 0, S = 0; bool rects = false, xf = false, whole = false;
                  const uint32_t* bank = nullptr; };
  int64_t fwd_gen = 0;
  EotSig eot;
  int16_t* eot_rects_d = nullptr; int eot_rects_cap = 0;   // the forward's rectangles (rects_d is shared scratch)
  int32_t* eot_bank_idx_d = nullptr; int eot_bank_idx_cap = 0;   // the forward's mask indices [N][2]
  int32_t* bank_idx_d = nullptr; int bank_idx_cap = 0;     // scratch: the mask indices of dp_predict_bank / dp_expand_bank
  float* eot_xf_d = nullptr; int eot_xf_cap = 0;           // the forward's transforms (xf_d is dp_attack_grad's)
  void forward_clobbered() {
    ++fwd_gen;
    for (auto& L : lanes) L.held = -1;
  }

  // ---- optional per-category profiler (CUDA events around every launch) --------------
  bool prof_on = false;
  struct ProfRec { int cat; cudaEvent_t a, b; double bytes, flops; };
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> prof_pool;
  std::vector<std::string> prof_names;
  std::vector<double> prof_ms, prof_bytes, prof_flops;
  std::vector<int64_t> prof_count;
  int prof_cat(const char* name) {
    for (size_t i = 0; i < prof_names.size(); ++i) if (prof_names[i] == name) return (int)i;
    prof_names.push_back(name); prof_ms.push_back(0); prof_bytes.push_back(0); prof_flops.push_back(0); prof_count.push_back(0);
    return (int)prof_names.size() - 1;
  }
  cudaEvent_t prof_event() {
    if (!prof_pool.empty()) { cudaEvent_t e = prof_pool.back(); prof_pool.pop_back(); return e; }
    cudaEvent_t e; CUDA_OK(cudaEventCreate(&e)); return e;
  }
  void prof_begin(const char* name, double bytes, double flops, cudaStream_t st) {
    if (!prof_on) return;
    ProfRec r; r.cat = prof_cat(name); r.bytes = bytes; r.flops = flops; r.a = prof_event(); r.b = prof_event();
    CUDA_OK(cudaEventRecord(r.a, st));
    prof_recs.push_back(r);
  }
  void prof_end(cudaStream_t st) {
    if (!prof_on) return;
    CUDA_OK(cudaEventRecord(prof_recs.back().b, st));
  }
  void prof_collect() {
    for (auto& r : prof_recs) {
      CUDA_OK(cudaEventSynchronize(r.b));
      float ms = 0.f; CUDA_OK(cudaEventElapsedTime(&ms, r.a, r.b));
      prof_ms[r.cat] += ms; prof_bytes[r.cat] += r.bytes; prof_flops[r.cat] += r.flops; prof_count[r.cat] += 1;
      prof_pool.push_back(r.a); prof_pool.push_back(r.b);
    }
    prof_recs.clear();
  }
  // Every launch of the engine: f() enqueues on st and returns the number of kernels it enqueued (a dp::launch_*'s
  // return value; 1 for a cuDNN / cublasLt call, whatever the library enqueues inside it).  The sum is `launches`
  // (dp_engine_launch_count); cuDNN Find* and cublasLt autotune trials run outside run() and are not counted.
  // cat: the profiler region's category and its algorithmic bytes / flops; run(st, f) is a launch outside the profile.
  template <class F>
  void run(const char* cat, double bytes, double flops, cudaStream_t st, F&& f) {
    if (cat) prof_begin(cat, bytes, flops, st);
    const int n = f();
    if (cat) prof_end(st);
    CUDA_OK(cudaGetLastError());
    launches += n;
  }
  template <class F>
  void run(cudaStream_t st, F&& f) { run(nullptr, 0, 0, st, std::forward<F>(f)); }

  // ---- whole-step CUDA graphs (SURVEY 8f N4): dp_attack_grad's launch sequence (staging copies, paste, regularisers,
  // every chunk's K1 -> forward -> CW -> backward -> K1^T on both lanes, result copies) captured once per call
  // signature and replayed; the first call of a signature runs eagerly (it picks cuDNN / cublasLt algorithms, which
  // synchronises and cannot be captured).  DORPATCH_GRAPH=0 disables.
  struct GraphEnt { int calls = 0; bool failed = false; cudaGraphExec_t exec = nullptr; int64_t launches = 0; };
  typedef std::tuple<int, int, int, int, const void*, const void*, const void*, const void*, float, float, int, int> GraphKey;
  std::map<GraphKey, GraphEnt> graphs;
  bool graphs_on = true;
  cudaStream_t cap_stream = nullptr;   // capture happens here when the caller's stream is the legacy / per-thread default stream (not capturable)
  int64_t graph_replays = 0;
  std::string graph_msg;               // why the last capture attempt was abandoned (diagnostics)
  void drop_graphs() {
    for (auto& kv : graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    graphs.clear();
  }

  std::map<std::pair<int, int>, CudnnPlan> cudnn_plans;                 // (layer id, N)
  std::map<std::tuple<int, int, int, int>, GemmPlan> gemm_plans;        // (rows, n_out, k, mode)

  // ---------------------------------------------------------------------------------
  void* dmalloc(size_t bytes) {
    void* p = nullptr;
    bytes = (bytes + 255) / 256 * 256;
    if (bytes == 0) bytes = 256;
    CUDA_OK(cudaMalloc(&p, bytes));
    allocs.push_back(p);
    device_bytes += (int64_t)bytes;
    return p;
  }
  void ensure_pin(size_t bytes) {
    if (bytes <= pin_bytes) return;
    drop_graphs();                       // captured copies hold the old staging address
    if (pin) cudaFreeHost(pin);
    pin_bytes = std::max(bytes, (size_t)1 << 20);
    CUDA_OK(cudaMallocHost((void**)&pin, pin_bytes));
  }
  // K1 for the WHOLE step in one launch (all B*S samples into one buffer, the chunks then read their slices): the launch
  // shape of one classifier chunk (16 images x 28 row tiles) is too small to fill 132 SMs for more than one ragged wave
  // (a 512-sample launch reaches a larger share of the HBM peak).  Bounded by
  // DORPATCH_K1_WHOLE_MB (default 4096; 0 = one launch per chunk as in round 1).
  void* net_in_all = nullptr;
  size_t net_in_all_cap = 0, k1_whole_max = (size_t)4096 << 20;
  size_t sample_in_bytes() const { return (size_t)H * H * stem.in_ch * es; }
  const void* whole_slice(int n0) const { return (const char*)net_in_all + (size_t)n0 * sample_in_bytes(); }
  bool k1_whole_ok(int n) const { return k1_whole_max > 0 && n > chunk && (size_t)n * sample_in_bytes() <= k1_whole_max; }
  bool ensure_net_in_all(int n) {
    if (!k1_whole_ok(n)) return false;
    const size_t bytes = (size_t)n * sample_in_bytes();
    if (bytes > net_in_all_cap) {
      drop_graphs();
      if (net_in_all) { CUDA_OK(cudaFree(net_in_all)); device_bytes -= (int64_t)net_in_all_cap; net_in_all = nullptr; net_in_all_cap = 0; }
      CUDA_OK(cudaMalloc(&net_in_all, bytes));
      net_in_all_cap = bytes;
      device_bytes += (int64_t)bytes;
    }
    return true;
  }
  void ensure_samples(int n) {
    if (n <= cap_samples) return;
    drop_graphs();                       // captured launches hold the old per-sample buffers
    // (old buffers stay in `allocs` and are released at destroy)
    cap_samples = std::max(n, cap_samples * 2);
    rects_d = (int16_t*)dmalloc((size_t)cap_samples * dp::RECT_SHORTS * sizeof(int16_t));
    y_d = (int32_t*)dmalloc((size_t)cap_samples * sizeof(int32_t));
    tg_d = (uint8_t*)dmalloc((size_t)cap_samples);
    loss_d = (float*)dmalloc((size_t)cap_samples * sizeof(float));
    preds_d = (int32_t*)dmalloc((size_t)cap_samples * sizeof(int32_t));
    xf_d = (float*)dmalloc((size_t)cap_samples * 8 * sizeof(float));
  }

  // ---- geometry -----------------------------------------------------------------------
  int Hs() const { return H / 2; }
  int Hp() const { return H / 4; }
  size_t max_act_elems() const {   // per sample
    size_t m = (size_t)Hs() * Hs() * STEM_CH;
    for (auto& b : blocks) {
      m = std::max(m, (size_t)b.hin * b.hin * std::max(b.cin, b.mid));
      m = std::max(m, (size_t)b.hout * b.hout * b.cout);
    }
    m = std::max(m, (size_t)H * H * std::max(stem.in_ch, stem.dx_ch));
    return m;
  }

  void build_arch() {
    int cin = STEM_CH, h = Hp();
    for (int s = 0; s < 4; ++s) {
      for (int bi = 0; bi < DEPTHS[s]; ++bi) {
        Block b{};
        b.cin = cin; b.cout = WIDTHS[s]; b.mid = b.cout / 4;
        b.stride = (bi == 0 && s > 0) ? 2 : 1;
        b.hin = h; b.hout = (h + b.stride - 1) / b.stride;
        b.has_ds = (bi == 0);
        blocks.push_back(b);
        cin = b.cout; h = b.hout;
      }
    }
  }

  void make_conv(ConvW& c, int cin, int cout, int k, int stride, int pad, int cin_pad) {
    c.cin = cin; c.cin_pad = cin_pad; c.cout = cout; c.k = k; c.stride = stride; c.pad = pad;
    c.w = dmalloc((size_t)cout * k * k * cin_pad * es);
    c.raw = (float*)dmalloc((size_t)cout * k * k * cin * 4);
    if (k > 1) {   // cuDNN path
      CUDNN_OK(cudnnCreateFilterDescriptor(&c.wdesc));
      CUDNN_OK(cudnnSetFilter4dDescriptor(c.wdesc, cudnn_dt, CUDNN_TENSOR_NHWC, cout, cin_pad, k, k));
      CUDNN_OK(cudnnCreateConvolutionDescriptor(&c.cdesc));
      CUDNN_OK(cudnnSetConvolution2dDescriptor(c.cdesc, pad, pad, stride, stride, 1, 1, CUDNN_CROSS_CORRELATION, CUDNN_DATA_FLOAT));
      CUDNN_OK(cudnnSetConvolutionMathType(c.cdesc, default_math()));
    }
  }
  cudnnMathType_t default_math() const {
    if (cfg.precision == DP_PREC_FP32) return CUDNN_FMA_MATH;
    if (cfg.precision == DP_PREC_TF32) return CUDNN_DEFAULT_MATH;   // fp32 data -> TF32 tensor cores
    return CUDNN_TENSOR_OP_MATH;
  }
  void make_gn(GNW& g_, int C) {
    g_.C = C;
    g_.gamma = (float*)dmalloc((size_t)C * 4);
    g_.beta = (float*)dmalloc((size_t)C * 4);
  }

  void allocate() {
    const size_t n = (size_t)chunk;
    stem.allocate();
    for (auto& b : blocks) {
      make_gn(b.n1, b.cin); make_gn(b.n2, b.mid); make_gn(b.n3, b.mid);
      if (b.has_ds) make_conv(b.ds, b.cin, b.cout, 1, b.stride, 0, b.cin);
      make_conv(b.c1, b.cin, b.mid, 1, 1, 0, b.cin);
      make_conv(b.c2, b.mid, b.mid, 3, b.stride, 1, b.mid);
      make_conv(b.c3, b.mid, b.cout, 1, 1, 0, b.mid);
      if (fused_gemm) {
        b.c1p = dmalloc((size_t)b.mid * b.cin * 2);
        b.c3p = dmalloc((size_t)b.cout * b.mid * 2);
      }
    }
    make_gn(head_gn, WIDTHS[3]);
    fc_w = (float*)dmalloc((size_t)K * WIDTHS[3] * 4);
    fc_b = (float*)dmalloc((size_t)K * 4);
    const size_t ma = max_act_elems();
    lib_ws_bytes = (size_t)512 << 20;
    int n_lanes = 2;
    if (const char* le = getenv("DORPATCH_LANES")) n_lanes = atoi(le);
    if (n_lanes < 1) n_lanes = 1;
    if (n_lanes > 2) n_lanes = 2;
    lanes.resize(n_lanes);
    CUDA_OK(cudaEventCreateWithFlags(&ev_prep, cudaEventDisableTiming));
    CUDA_OK(cudaStreamCreateWithFlags(&cap_stream, cudaStreamNonBlocking));
    for (int l = 0; l < n_lanes; ++l) {
      Lane& L = lanes[l];
      for (auto& b : blocks)
        L.saved.push_back(Lane::Saved{dmalloc(n * b.hin * b.hin * b.mid * es), dmalloc(n * b.hout * b.hout * b.mid * es),
                                      dmalloc(n * b.hout * b.hout * b.cout * es), (float*)dmalloc(n * dp::GN_GROUPS * 2 * 4),
                                      (float*)dmalloc(n * dp::GN_GROUPS * 2 * 4), (float*)dmalloc(n * dp::GN_GROUPS * 2 * 4)});
      L.net_in = dmalloc(n * H * H * stem.in_ch * es);
      L.act = dmalloc(n * ma * es);
      L.act2 = dmalloc(n * ma * es / 4 + 256);
      L.x0 = dmalloc(n * Hp() * Hp() * STEM_CH * es);
      L.pool_amax = (int8_t*)dmalloc(n * Hp() * Hp() * STEM_CH);
      for (int i = 0; i < 4; ++i) L.g[i] = dmalloc(n * ma * es);
      L.gn_partial = (float*)dmalloc((n * dp::GN_WS_FLOATS_PER_SAMPLE + dp::GN_WS_FLOATS_EXTRA) * 4);
      L.head_stats = (float*)dmalloc(n * dp::GN_GROUPS * 2 * 4);
      L.pooled = (float*)dmalloc(n * WIDTHS[3] * 4);
      L.dpooled = (float*)dmalloc(n * WIDTHS[3] * 4);
      L.logits = (float*)dmalloc(n * K * 4);
      L.dlogits = (float*)dmalloc(n * K * 4);
      L.lib_ws = dmalloc(lib_ws_bytes);
      CUDA_OK(cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
      CUDA_OK(cudaEventCreateWithFlags(&L.done, cudaEventDisableTiming));
      CUDNN_OK(cudnnCreate(&L.cudnn));
    }
    const size_t B = (size_t)cfg.max_images, HW = (size_t)H * H;
    adv_x = (float*)dmalloc(B * 3 * HW * 4);
    dLs = (float*)dmalloc(B * 3 * HW * 4);
    host_x = (float*)dmalloc(B * 3 * HW * 4);
    host_pattern = (float*)dmalloc(B * 3 * HW * 4);
    host_mask = (float*)dmalloc(B * HW * 4);
    host_G = (float*)dmalloc(B * 3 * HW * 4);
    for (float** p : {&scale, &l2, &loss_struc, &loss_density, &group_lasso, &lr_d, &structured_d, &coeff_d, &helper_scale, &helper_l2})
      *p = (float*)dmalloc(B * 4);
    helper_ws = (float*)dmalloc(B * HW * 4);
    failed_bits = (uint32_t*)dmalloc(B * failed_words_alloc * 4);
    CUDA_OK(cudaMemset(failed_bits, 0, B * failed_words_alloc * 4));
    failed_count = (int32_t*)dmalloc(B * 4); failed_nff = (int32_t*)dmalloc(B * 4); failed_active = (uint8_t*)dmalloc(B);
    draw_nff_d = (int32_t*)dmalloc(B * 4);
    draw_par_d = (unsigned char*)dmalloc(draw_par_bytes());
    CUDA_OK(cudaMallocHost((void**)&draw_pin, draw_par_bytes()));
    CUDA_OK(cudaEventCreateWithFlags(&draw_ev, cudaEventDisableTiming));
    win_dev = (float*)dmalloc(B * 64 * 4);
    grp_ss = (float*)dmalloc(B * HW * 4);
    ensure_samples(chunk);
    ensure_pin((size_t)4 << 20);
    build_wparams();
  }

  // ---- named parameters and the weight-gradient accumulators (dp_eot_backward_params) -------------------------
  // One entry per timm state-dict tensor.  Each has a slot in the fp32 accumulators: conv weights as d/d(standardised
  // weight) in the engine's KRSC, channel-padded layout (the standardisation adjoint runs once per call at the end),
  // GroupNorm gamma | beta adjacent, the fc weight [K][2048] and bias.  The head's four tensors come last.
  enum WKind { W_CONV = 0, W_GAMMA, W_BETA, W_FCW, W_FCB };
  struct WParam { std::string name; int kind; ConvW* conv; GNW* gn; int64_t numel; size_t off; };
  std::vector<WParam> wparams;
  std::map<std::string, int> wparam_idx;
  size_t wacc_floats = 0, wacc_trunk_end = 0;    // [0, wacc_trunk_end): stem + blocks; the rest: head
  std::vector<char> want;                        // per wparam: requested by the current call
  // acc_floats: the slot's size (0: the entry lives inside the slot just reserved, at `inner` floats from its start)
  void add_wparam(const std::string& name, int kind, ConvW* c, GNW* g, int64_t numel, size_t acc_floats, size_t inner = 0) {
    wparam_idx[name] = (int)wparams.size();
    if (c) c->pid = (int)wparams.size();
    if (g && kind == W_GAMMA) g->pid = (int)wparams.size();
    if (acc_floats == 0) {
      wparams.push_back(WParam{name, kind, c, g, numel, wparams.back().off + inner});
      return;
    }
    wparams.push_back(WParam{name, kind, c, g, numel, wacc_floats});
    wacc_floats += (acc_floats + 63) / 64 * 64;
  }
  void add_conv_param(const std::string& name, ConvW& c) {
    add_wparam(name, W_CONV, &c, nullptr, (int64_t)c.cout * c.cin * c.k * c.k, (size_t)c.cout * c.k * c.k * c.cin_pad);
  }
  void add_gn_params(const std::string& pre, GNW& g) {   // one slot [gamma | beta]: gn_wgrad adds both halves at once
    add_wparam(pre + ".weight", W_GAMMA, nullptr, &g, g.C, 2 * (size_t)g.C);
    add_wparam(pre + ".bias", W_BETA, nullptr, &g, g.C, 0, g.C);
  }
  void build_wparams() {
    add_conv_param("stem.conv.weight", stem.conv);
    int s = 0, bi = 0;
    for (auto& b : blocks) {
      char pre[64];
      snprintf(pre, sizeof(pre), "stages.%d.blocks.%d.", s, bi);
      const std::string P(pre);
      if (b.has_ds) add_conv_param(P + "downsample.conv.weight", b.ds);
      add_conv_param(P + "conv1.weight", b.c1);
      add_conv_param(P + "conv2.weight", b.c2);
      add_conv_param(P + "conv3.weight", b.c3);
      add_gn_params(P + "norm1", b.n1);
      add_gn_params(P + "norm2", b.n2);
      add_gn_params(P + "norm3", b.n3);
      if (++bi == DEPTHS[s]) { bi = 0; ++s; }
    }
    wacc_trunk_end = wacc_floats;
    add_gn_params("norm", head_gn);
    add_wparam("head.fc.weight", W_FCW, nullptr, nullptr, (int64_t)K * WIDTHS[3], (size_t)K * WIDTHS[3]);
    add_wparam("head.fc.bias", W_FCB, nullptr, nullptr, K, K);
    want.assign(wparams.size(), 0);
  }
  const WParam& wparam(const char* name) const {
    auto it = wparam_idx.find(name);
    if (it == wparam_idx.end()) fail("unknown parameter name '%s' (timm resnetv2_50x1_bit state-dict names)", name);
    return wparams[it->second];
  }
  void ensure_wgrad_buffers() {
    if (lanes[0].wacc) return;
    size_t part = std::max((size_t)chunk * 2 * WIDTHS[3], dp::stem_wgrad_partial_floats());
    part = std::max(part, (size_t)chunk * 2 * 2048);
    size_t half = 0;
    for (auto& b : blocks) half = std::max(half, (size_t)b.c2.cout * 9 * b.c2.cin_pad);
    half = std::max(half, (size_t)STEM_CH * 49 * stem.conv.cin_pad);
    for (auto& L : lanes) {
      L.wacc = (float*)dmalloc(wacc_floats * 4);
      L.wg_partial = (float*)dmalloc(part * 4);
      L.wg_half = dmalloc(half * 2);
    }
  }
  bool want_conv(const ConvW& c) const { return c.pid >= 0 && want[c.pid]; }
  bool want_gn(const GNW& g) const { return g.pid >= 0 && (want[g.pid] || want[g.pid + 1]); }
  // accumulator span of wparam i: [off, end); a GroupNorm's gamma and beta share one slot, zeroed and filled together
  std::pair<size_t, size_t> wspan(size_t i) const {
    const WParam& w = wparams[i];
    if (w.kind == W_GAMMA || w.kind == W_BETA) {
      const size_t g0 = wparams[w.gn->pid].off;
      return {g0, g0 + 2 * (size_t)w.gn->C};
    }
    size_t end = wacc_floats;
    for (size_t j = i + 1; j < wparams.size(); ++j) if (wparams[j].off > w.off) { end = wparams[j].off; break; }
    return {w.off, end};
  }
  float* acc_of(const Lane& L, int pid) const { return L.wacc + wparams[pid].off; }

  // ---- weights (their launches are counted, not profiled) --------------------------------------------------------
  void standardize(const ConvW& c, cudaStream_t st) {
    run(st, [&] { return dp::launch_weight_standardize(c.raw, c.w, c.cout, c.cin, c.k, c.k, c.cin_pad, bf16, true, st); });
  }
  // One timm tensor from `src` (kind: H2D or D2D, on st), then what that kind needs: a convolution is re-standardised
  // and its packed copies rebuilt (the stem's tile, or the fused GEMM's), a GroupNorm's "every gamma > 0" flag (the
  // packed bf16 ReLU gate) is recomputed from the new values.
  void load_param(const WParam& w, const float* src, cudaMemcpyKind kind, cudaStream_t st) {
    const size_t bytes = (size_t)w.numel * 4;
    switch (w.kind) {
      case W_CONV: {
        const ConvW& c = *w.conv;
        CUDA_OK(cudaMemcpyAsync(c.raw, src, bytes, kind, st));
        if (&c == &stem.conv) { stem.load(st); break; }
        standardize(c, st);
        if (fused_gemm)
          for (auto& b : blocks) {
            if (&c == &b.c1) run(st, [&] { return dp::launch_gn_gemm_pack(b.c1.w, b.c1p, b.mid, b.cin, st); });
            if (&c == &b.c3) run(st, [&] { return dp::launch_gn_gemm_pack(b.c3.w, b.c3p, b.cout, b.mid, st); });
          }
        break;
      }
      case W_GAMMA: {
        GNW& g_ = *w.gn;
        CUDA_OK(cudaMemcpyAsync(g_.gamma, src, bytes, kind, st));
        std::vector<float> h(g_.C);
        CUDA_OK(cudaMemcpyAsync(h.data(), g_.gamma, bytes, cudaMemcpyDeviceToHost, st));   // pageable: returns when done
        g_.pos = std::all_of(h.begin(), h.end(), [](float v) { return v > 0.f; });
        break;
      }
      case W_BETA: CUDA_OK(cudaMemcpyAsync(w.gn->beta, src, bytes, kind, st)); break;
      case W_FCW: CUDA_OK(cudaMemcpyAsync(fc_w, src, bytes, kind, st)); break;
      default: CUDA_OK(cudaMemcpyAsync(fc_b, src, bytes, kind, st)); break;
    }
  }
  // The full set from host memory, on the default stream: every name of the table is required, other names are ignored.
  void load_weights(int n, const char* const* names, const float* const* ptrs, const int64_t* numels) {
    std::map<std::string, int> idx;
    for (int i = 0; i < n; ++i) idx[names[i]] = i;
    for (const WParam& w : wparams) {
      auto it = idx.find(w.name);
      if (it == idx.end()) fail("missing weight tensor '%s'", w.name.c_str());
      const int i = it->second;
      if (numels[i] != w.numel) fail("weight tensor '%s' has %lld elements, expected %lld", names[i], (long long)numels[i], (long long)w.numel);
      load_param(w, ptrs[i], cudaMemcpyHostToDevice, 0);
    }
    CUDA_OK(cudaStreamSynchronize(0));
    weights_loaded = true;
    forward_clobbered();
  }

  // Reload named tensors from fp32 device buffers (after an optimizer step), on the caller's stream: no host copy of
  // the weights.  Any subset; everything is checked before anything changes.
  void load_weights_dev(int n, const char* const* names, const float* const* ptrs, const int64_t* numels, cudaStream_t st) {
    if (!weights_loaded) fail("dp_engine_load_weights_dev: load the full set with dp_engine_load_weights first");
    if (n < 0 || (n > 0 && (!names || !ptrs || !numels))) fail("dp_engine_load_weights_dev: null argument");
    std::vector<char> seen(wparams.size(), 0);
    for (int i = 0; i < n; ++i) {
      if (!names[i]) fail("dp_engine_load_weights_dev: null name at position %d", i);
      const WParam& w = wparam(names[i]);
      if (seen[&w - wparams.data()]++) fail("dp_engine_load_weights_dev: '%s' is named twice", names[i]);
      if (!ptrs[i]) fail("dp_engine_load_weights_dev: null pointer for '%s'", names[i]);
      if (numels[i] != w.numel) fail("dp_engine_load_weights_dev: '%s' has %lld elements, expected %lld", names[i], (long long)numels[i], (long long)w.numel);
    }
    drop_graphs();
    forward_clobbered();
    for (int i = 0; i < n; ++i) load_param(wparam(names[i]), ptrs[i], cudaMemcpyDeviceToDevice, st);
    CUDA_OK(cudaStreamSynchronize(st));
  }

  // ---- cuDNN convolution -------------------------------------------------------------
  CudnnPlan& conv_plan(int layer_id, const ConvW& c, int N, int hin, int hout) {
    auto key = std::make_pair(layer_id, N);
    auto it = cudnn_plans.find(key);
    if (it != cudnn_plans.end()) return it->second;
    CudnnPlan p;
    CUDNN_OK(cudnnCreateTensorDescriptor(&p.xdesc));
    CUDNN_OK(cudnnCreateTensorDescriptor(&p.ydesc));
    CUDNN_OK(cudnnSetTensor4dDescriptor(p.xdesc, CUDNN_TENSOR_NHWC, cudnn_dt, N, c.cin_pad, hin, hin));
    CUDNN_OK(cudnnSetTensor4dDescriptor(p.ydesc, CUDNN_TENSOR_NHWC, cudnn_dt, N, c.cout, hout, hout));
    int on, oc, oh, ow;
    CUDNN_OK(cudnnGetConvolution2dForwardOutputDim(c.cdesc, p.xdesc, c.wdesc, &on, &oc, &oh, &ow));
    if (on != N || oc != c.cout || oh != hout || ow != hout)
      fail("conv layer %d: cuDNN output dims (%d,%d,%d,%d) != expected (%d,%d,%d,%d)", layer_id, on, oc, oh, ow, N, c.cout, hout, hout);
    return cudnn_plans.emplace(key, p).first->second;
  }
  bool math_ok(cudnnMathType_t m) const {
    if (cfg.precision == DP_PREC_FP32) return m == CUDNN_FMA_MATH;   // parity mode: no TF32 down-conversion
    return true;
  }
  void pick_fwd(const Lane& L, CudnnPlan& p, const ConvW& c, const void* x, void* y) {
    cudnnConvolutionFwdAlgoPerf_t perf[16];
    int got = 0;
    if (cfg.autotune)
      CUDNN_OK(cudnnFindConvolutionForwardAlgorithmEx(L.cudnn, p.xdesc, x, c.wdesc, c.w, c.cdesc, p.ydesc, y, 16, &got, perf, L.lib_ws, lib_ws_bytes));
    else
      CUDNN_OK(cudnnGetConvolutionForwardAlgorithm_v7(L.cudnn, p.xdesc, c.wdesc, c.cdesc, p.ydesc, 16, &got, perf));
    for (int i = 0; i < got; ++i) {
      if (perf[i].status != CUDNN_STATUS_SUCCESS || perf[i].memory > lib_ws_bytes || !math_ok(perf[i].mathType)) continue;
      p.fwd_algo = perf[i].algo; p.fwd_math = perf[i].mathType; p.fwd_ws = perf[i].memory; p.fwd_ready = true;
      return;
    }
    fail("no usable cuDNN forward algorithm (cin=%d cout=%d k=%d stride=%d, %d candidates)", c.cin_pad, c.cout, c.k, c.stride, got);
  }
  void pick_bwd(const Lane& L, CudnnPlan& p, const ConvW& c, const void* dy, void* dx) {
    cudnnConvolutionBwdDataAlgoPerf_t perf[16];
    int got = 0;
    if (cfg.autotune)
      CUDNN_OK(cudnnFindConvolutionBackwardDataAlgorithmEx(L.cudnn, c.wdesc, c.w, p.ydesc, dy, c.cdesc, p.xdesc, dx, 16, &got, perf, L.lib_ws, lib_ws_bytes));
    else
      CUDNN_OK(cudnnGetConvolutionBackwardDataAlgorithm_v7(L.cudnn, c.wdesc, p.ydesc, c.cdesc, p.xdesc, 16, &got, perf));
    // results are sorted by time: take the fastest usable one, but prefer a deterministic algorithm
    // when it is within 25 % of it (a slow "deterministic" dgrad once cost 688 ms on the stem).
    int fastest = -1, det = -1;
    for (int i = 0; i < got; ++i) {
      if (perf[i].status != CUDNN_STATUS_SUCCESS || perf[i].memory > lib_ws_bytes || !math_ok(perf[i].mathType)) continue;
      if (fastest < 0) fastest = i;
      if (det < 0 && perf[i].determinism == CUDNN_DETERMINISTIC) det = i;
    }
    if (fastest >= 0) {
      int pick = fastest;
      if (det >= 0 && (!cfg.autotune || perf[det].time <= 1.25f * perf[fastest].time)) pick = det;
      p.bwd_algo = perf[pick].algo; p.bwd_math = perf[pick].mathType; p.bwd_ws = perf[pick].memory; p.bwd_ready = true;
      return;
    }
    fail("no usable cuDNN backward-data algorithm (cin=%d cout=%d k=%d stride=%d, %d candidates)", c.cin_pad, c.cout, c.k, c.stride, got);
  }
  void conv_fwd(const Lane& L, int layer_id, const ConvW& c, int N, int hin, int hout, const void* x, void* y, cudaStream_t st) {
    CudnnPlan& p = conv_plan(layer_id, c, N, hin, hout);
    if (!p.fwd_ready) pick_fwd(L, p, c, x, y);
    CUDNN_OK(cudnnSetConvolutionMathType(c.cdesc, p.fwd_math));
    const float one = 1.f, zero = 0.f;
    const double fl = 2.0 * N * hout * hout * c.cout * c.k * c.k * c.cin;
    const double by = ((double)N * hin * hin * c.cin_pad + (double)N * hout * hout * c.cout + (double)c.cout * c.k * c.k * c.cin_pad) * es;
    run(c.k == 7 ? "stem_conv_fwd" : "conv3x3_fwd", by, fl, st, [&] {
      CUDNN_OK(cudnnConvolutionForward(L.cudnn, &one, p.xdesc, x, c.wdesc, c.w, c.cdesc, p.fwd_algo, L.lib_ws, lib_ws_bytes, &zero, p.ydesc, y));
      return 1;
    });
  }
  void conv_bwd(const Lane& L, int layer_id, const ConvW& c, int N, int hin, int hout, const void* dy, void* dx, cudaStream_t st) {
    CudnnPlan& p = conv_plan(layer_id, c, N, hin, hout);
    if (!p.bwd_ready) pick_bwd(L, p, c, dy, dx);
    CUDNN_OK(cudnnSetConvolutionMathType(c.cdesc, p.bwd_math));
    const float one = 1.f, zero = 0.f;
    const double fl = 2.0 * N * hout * hout * c.cout * c.k * c.k * c.cin;
    const double by = ((double)N * hin * hin * c.cin_pad + (double)N * hout * hout * c.cout + (double)c.cout * c.k * c.k * c.cin_pad) * es;
    run(c.k == 7 ? "stem_conv_bwd" : "conv3x3_bwd", by, fl, st, [&] {
      CUDNN_OK(cudnnConvolutionBackwardData(L.cudnn, &one, c.wdesc, c.w, p.ydesc, dy, c.cdesc, p.bwd_algo, L.lib_ws, lib_ws_bytes, &zero, p.xdesc, dx));
      return 1;
    });
  }

  // ---- cublasLt GEMM (1x1 convolutions, NHWC) ---------------------------------------------
  // mode 0: Y[rows,nout] = X[rows,k] * W[nout,k]^T (+ Cres)      (forward)
  // mode 1: dX[rows,nout] = dY[rows,k] * W[k,nout] (+ dX if beta) (backward data)
  GemmPlan& gemm_plan(int rows, int nout, int k, int mode) {
    auto key = std::make_tuple(rows, nout, k, mode);
    auto it = gemm_plans.find(key);
    if (it != gemm_plans.end()) return it->second;
    GemmPlan p;
    // modes 2 / 3: the fp32 classifier head (fc forward with fused bias / fc backward), always fp32 math
    const bool head = mode >= 2;
    const cudaDataType_t cuda_dt = head ? CUDA_R_32F : this->cuda_dt;
    CUBLAS_OK(cublasLtMatmulDescCreate(&p.op, head ? CUBLAS_COMPUTE_32F : lt_compute, CUDA_R_32F));
    const cublasOperation_t ta = (mode == 0 || mode == 2) ? CUBLAS_OP_T : CUBLAS_OP_N, tb = CUBLAS_OP_N;
    if (mode == 2) {
      const cublasLtEpilogue_t epi = CUBLASLT_EPILOGUE_BIAS;
      const void* bias = fc_b;
      CUBLAS_OK(cublasLtMatmulDescSetAttribute(p.op, CUBLASLT_MATMUL_DESC_EPILOGUE, &epi, sizeof(epi)));
      CUBLAS_OK(cublasLtMatmulDescSetAttribute(p.op, CUBLASLT_MATMUL_DESC_BIAS_POINTER, &bias, sizeof(bias)));
    }
    CUBLAS_OK(cublasLtMatmulDescSetAttribute(p.op, CUBLASLT_MATMUL_DESC_TRANSA, &ta, sizeof(ta)));
    CUBLAS_OK(cublasLtMatmulDescSetAttribute(p.op, CUBLASLT_MATMUL_DESC_TRANSB, &tb, sizeof(tb)));
    // column-major view: D[nout x rows] = op(A) * B
    if (mode == 0 || mode == 2) CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.a, cuda_dt, k, nout, k));   // W as col-major [k x nout], ld k
    else CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.a, cuda_dt, nout, k, nout));              // W[k rows][nout] as col-major [nout x k], ld nout
    CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.b, cuda_dt, k, rows, k));                      // X / dY as col-major [k x rows]
    CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.c, cuda_dt, nout, rows, nout));
    cublasLtMatmulPreference_t pref;
    CUBLAS_OK(cublasLtMatmulPreferenceCreate(&pref));
    CUBLAS_OK(cublasLtMatmulPreferenceSetAttribute(pref, CUBLASLT_MATMUL_PREF_MAX_WORKSPACE_BYTES, &lib_ws_bytes, sizeof(lib_ws_bytes)));
    cublasLtMatmulHeuristicResult_t res[8];
    int got = 0;
    cublasStatus_t s = cublasLtMatmulAlgoGetHeuristic(lt, p.op, p.a, p.b, p.c, p.c, pref, 8, res, &got);
    cublasLtMatmulPreferenceDestroy(pref);
    if (s != CUBLAS_STATUS_SUCCESS || got == 0) fail("cublasLt: no algorithm for GEMM rows=%d nout=%d k=%d mode=%d (status %d)", rows, nout, k, mode, (int)s);
    p.algo = res[0].algo;
    for (int i = 0; i < got; ++i)
      if (res[i].state == CUBLAS_STATUS_SUCCESS) p.candidates.push_back(res[i].algo);
    return gemm_plans.emplace(key, p).first->second;
  }
  void gemm(const Lane& L, int rows, int nout, int k, int mode, const void* W, const void* X, const void* Cres, float beta, void* D, cudaStream_t st) {
    GemmPlan& p = gemm_plan(rows, nout, k, mode);
    const float one = 1.f;
    // Autotune (once per shape): time the heuristic's top candidates on the real operands.  Skipped
    // for in-place accumulation (C == D), where repeated trial runs would corrupt the addend.
    const bool in_place_acc = (beta != 0.f) && (Cres == nullptr || Cres == D);
    if (!p.tuned && cfg.autotune && !in_place_acc && p.candidates.size() > 1 && !prof_on) {
      cudaEvent_t e0, e1;
      CUDA_OK(cudaEventCreate(&e0)); CUDA_OK(cudaEventCreate(&e1));
      float best = 1e30f;
      for (auto& cand : p.candidates) {
        bool ok = true;
        for (int rep = 0; rep < 3 && ok; ++rep) {
          if (rep == 1) CUDA_OK(cudaEventRecord(e0, st));
          ok = cublasLtMatmul(lt, p.op, &one, W, p.a, X, p.b, &beta, Cres ? Cres : D, p.c, D, p.c, &cand, L.lib_ws, lib_ws_bytes, st) == CUBLAS_STATUS_SUCCESS;
        }
        if (!ok) continue;
        CUDA_OK(cudaEventRecord(e1, st));
        CUDA_OK(cudaEventSynchronize(e1));
        float ms = 0.f; CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) { best = ms; p.algo = cand; }
      }
      cudaEventDestroy(e0); cudaEventDestroy(e1);
      p.tuned = true;
    }
    const double by = ((double)rows * k + (double)rows * nout * (beta != 0.f ? 2 : 1) + (double)nout * k) * (mode >= 2 ? 4 : es);
    run(mode == 0 ? "gemm1x1_fwd" : (mode == 1 ? "gemm1x1_bwd" : (mode == 2 ? "fc_fwd" : "fc_bwd")), by, 2.0 * rows * nout * k, st, [&] {
      CUBLAS_OK(cublasLtMatmul(lt, p.op, &one, W, p.a, X, p.b, &beta, Cres ? Cres : D, p.c, D, p.c, &p.algo, L.lib_ws, lib_ws_bytes, st));
      return 1;
    });
  }

  // ---- weight gradients ----------------------------------------------------------------------
  // 3x3 / stem: acc (KRSC, fp32) += dW through cuDNN, deterministic algorithms only, the engine's precision rules.
  // cuDNN's filter gradient has the filter's data type: at bf16 it goes through the lane's bf16 scratch.
  void conv_wgrad(const Lane& L, int layer_id, const ConvW& c, int N, int hin, int hout, const void* x, const void* dy, float* acc, cudaStream_t st) {
    CudnnPlan& p = conv_plan(layer_id, c, N, hin, hout);
    if (!p.wgd_ready) {
      cudnnConvolutionBwdFilterAlgoPerf_t perf[16];
      int got = 0;
      CUDNN_OK(cudnnGetConvolutionBackwardFilterAlgorithm_v7(L.cudnn, p.xdesc, p.ydesc, c.cdesc, c.wdesc, 16, &got, perf));
      for (int i = 0; i < got && !p.wgd_ready; ++i) {
        if (perf[i].status != CUDNN_STATUS_SUCCESS || perf[i].memory > lib_ws_bytes || !math_ok(perf[i].mathType) ||
            perf[i].determinism != CUDNN_DETERMINISTIC) continue;
        p.wgd_algo = perf[i].algo; p.wgd_math = perf[i].mathType; p.wgd_ws = perf[i].memory; p.wgd_ready = true;
      }
      if (!p.wgd_ready) fail("no usable deterministic cuDNN backward-filter algorithm (cin=%d cout=%d k=%d stride=%d, %d candidates)",
                             c.cin_pad, c.cout, c.k, c.stride, got);
    }
    CUDNN_OK(cudnnSetConvolutionMathType(c.cdesc, p.wgd_math));
    const float one = 1.f, zero = 0.f;
    const size_t wn = (size_t)c.cout * c.k * c.k * c.cin_pad;
    const double fl = 2.0 * N * hout * hout * c.cout * c.k * c.k * c.cin;
    const double by = ((double)N * hin * hin * c.cin_pad + (double)N * hout * hout * c.cout) * es + (double)wn * 8;
    run(c.k == 7 ? "stem_wgrad" : "conv3x3_wgrad", by, fl, st, [&] {
      CUDNN_OK(cudnnConvolutionBackwardFilter(L.cudnn, &one, p.xdesc, x, p.ydesc, dy, c.cdesc, p.wgd_algo, L.lib_ws, lib_ws_bytes,
                                              bf16 ? &zero : &one, c.wdesc, bf16 ? L.wg_half : (void*)acc));
      return 1;
    });
    if (bf16) run(st, [&] { return dp::launch_add_bf16(L.wg_half, acc, wn, st); });
  }
  // 1x1 convolutions and the fc layer: D[cout][cin] (fp32) += dY^T X over `rows` pixels.  Column-major view:
  // D [cin x cout] = X [cin x rows] * (dY [cout x rows])^T.  head: fp32 operands and math (the fc layer is fp32).
  std::map<std::tuple<int, int, int, int>, GemmPlan> wgrad_plans;
  void wgrad_gemm(const Lane& L, int rows, int cout, int cin, const void* X, const void* dY, float* D, bool head, cudaStream_t st) {
    auto key = std::make_tuple(rows, cout, cin, head ? 1 : 0);
    auto it = wgrad_plans.find(key);
    if (it == wgrad_plans.end()) {
      GemmPlan p;
      const cudaDataType_t ab = head ? CUDA_R_32F : cuda_dt;
      CUBLAS_OK(cublasLtMatmulDescCreate(&p.op, head ? CUBLAS_COMPUTE_32F : lt_compute, CUDA_R_32F));
      const cublasOperation_t ta = CUBLAS_OP_N, tb = CUBLAS_OP_T;
      CUBLAS_OK(cublasLtMatmulDescSetAttribute(p.op, CUBLASLT_MATMUL_DESC_TRANSA, &ta, sizeof(ta)));
      CUBLAS_OK(cublasLtMatmulDescSetAttribute(p.op, CUBLASLT_MATMUL_DESC_TRANSB, &tb, sizeof(tb)));
      CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.a, ab, cin, rows, cin));
      CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.b, ab, cout, rows, cout));
      CUBLAS_OK(cublasLtMatrixLayoutCreate(&p.c, CUDA_R_32F, cin, cout, cin));
      cublasLtMatmulPreference_t pref;
      CUBLAS_OK(cublasLtMatmulPreferenceCreate(&pref));
      CUBLAS_OK(cublasLtMatmulPreferenceSetAttribute(pref, CUBLASLT_MATMUL_PREF_MAX_WORKSPACE_BYTES, &lib_ws_bytes, sizeof(lib_ws_bytes)));
      cublasLtMatmulHeuristicResult_t res[1];
      int got = 0;
      cublasStatus_t s = cublasLtMatmulAlgoGetHeuristic(lt, p.op, p.a, p.b, p.c, p.c, pref, 1, res, &got);
      cublasLtMatmulPreferenceDestroy(pref);
      if (s != CUBLAS_STATUS_SUCCESS || got == 0) fail("cublasLt: no algorithm for the weight-gradient GEMM rows=%d cout=%d cin=%d (status %d)", rows, cout, cin, (int)s);
      p.algo = res[0].algo;
      it = wgrad_plans.emplace(key, p).first;
    }
    GemmPlan& p = it->second;
    const float one = 1.f;
    const double by = ((double)rows * (cin + cout)) * (head ? 4 : es) + (double)cin * cout * 8;
    run(head ? "fc_wgrad" : "gemm1x1_wgrad", by, 2.0 * rows * cout * cin, st, [&] {
      CUBLAS_OK(cublasLtMatmul(lt, p.op, &one, X, p.a, dY, p.b, &one, D, p.c, D, p.c, &p.algo, L.lib_ws, lib_ws_bytes, st));
      return 1;
    });
  }
  // GroupNorm affine gradients of one norm: dy at its (ReLU) output, x its input, stats the forward's
  void gn_wgrad(const Lane& L, const GNW& g, const void* dy, const void* x, const float* stats, int N, int P, cudaStream_t st) {
    run("gn_affine_wgrad", 2.0 * N * P * g.C * es + (double)N * 2 * g.C * 8, 0, st, [&] {
      const int n = dp::launch_gn_affine_partial(dy, x, g.gamma, g.beta, stats, L.wg_partial, N, P, g.C, bf16, st);
      return n + dp::launch_colsum_add(L.wg_partial, acc_of(L, g.pid), N, 2 * g.C, st);
    });
  }
  void gn_apply(const GNW& g, const void* x, const float* stats, void* y, int N, int P, cudaStream_t st) {
    run("gn_apply_wgrad", 2.0 * N * P * g.C * es, 0, st, [&] { return dp::launch_gn_apply(x, y, g.gamma, g.beta, stats, N, P, g.C, bf16, st); });
  }

  // FusedReduce: the stem dgrad fused with the masked EOT reduce (K1^T) of samples [n0, n0 + N) into G.
  // Wgrad: the weight-gradient pass of one chunk (dp_eot_backward_params): accumulates d/d(parameter) of the requested
  // parameters (`want`) into the lane's accumulators.  input: the chunk's network input.  need_dx: the input gradient
  // is wanted too (else the backward stops at block `lo`, the lowest block whose gradients are wanted).
  struct FusedReduce {
    const int16_t* rects; float* G; int B, S, n0;
    dp::MaskBank bank;                                   // bank.idx null: occluded by rects
    const dp::MaskBank* bank_or_null() const { return bank.idx ? &bank : nullptr; }
  };
  struct Wgrad { const void* input; bool need_dx; int lo; };
  struct EotIn;

  // ---- the stem: timm's stem.conv (7x7/2, 3 -> 64), ConstantPad2d(1, 0), MaxPool2d(3, 2) -------------------------
  // Every choice about the stem is made here, once at create: the network-input layout, the forward, how the backward
  // ends and the weight gradient.  A variant is an enum value plus its launches in forward / backward.
  struct Stem {
    enum Fwd { FWD_OWN, FWD_CUDNN };   // own: bf16 mma.sync kernel on the tight C = 3 input
    // the backward ends in the library dgrad (K1^T separate), the dgrad fused with K1^T, or that plus the max-pool adjoint
    enum BwdEnd { END_CUDNN, END_FUSED_REDUCE, END_FUSED_POOL_REDUCE };
    enum WgradImpl { WG_OWN, WG_CUDNN };   // own: bf16 mma.sync kernel on the tight input
    static constexpr int SUB = 128;      // samples per cuDNN stem call
    dp_engine* e = nullptr;
    ConvW conv;
    void* w_kn = nullptr;   // FWD_OWN: the standardised weights as the kernel's packed tile
    int in_ch = 4;          // channels per pixel of the network input (3 = tight, FWD_OWN)
    int dx_ch = 4;          // channels per pixel of d(input) from the library dgrad, and of the stem filter (4 / 8)
    Fwd fwd = FWD_CUDNN; BwdEnd bwd = END_CUDNN; WgradImpl wgrad = WG_CUDNN;

    void configure(dp_engine* eng) {
      e = eng;
      auto is = [](const char* var, const char* val) { const char* s = getenv(var); return s && strcmp(s, val) == 0; };
      dx_ch = e->bf16 ? 8 : 4;
      if (const char* s = getenv("DORPATCH_CPAD")) dx_ch = atoi(s);
      if (dx_ch != 4 && dx_ch != 8) fail("DORPATCH_CPAD must be 4 or 8");
      const bool own = e->bf16 && !is("DORPATCH_STEM", "cudnn");
      fwd = own ? FWD_OWN : FWD_CUDNN;
      wgrad = own ? WG_OWN : WG_CUDNN;
      in_ch = own ? 3 : dx_ch;
      // measured: rebuilding the d_stem patch in shared memory costs more than the saved HBM round trip
      // (2.25 ms vs 1.33 + 0.71 ms per 512-sample step) -> off unless DORPATCH_POOL_BWD=fused
      if (!own || is("DORPATCH_STEM_BWD", "cudnn")) bwd = END_CUDNN;
      else bwd = is("DORPATCH_POOL_BWD", "fused") ? END_FUSED_POOL_REDUCE : END_FUSED_REDUCE;
    }
    void allocate() {
      e->make_conv(conv, 3, STEM_CH, 7, 2, 3, dx_ch);
      if (fwd == FWD_OWN) w_kn = e->dmalloc((size_t)160 * 64 * 2);
    }
    void load(cudaStream_t st) {   // after new raw weights
      e->standardize(conv, st);
      if (fwd == FWD_OWN) e->run(st, [&] { return dp::launch_stem_pack(conv.w, w_kn, conv.cin_pad, st); });
    }
    // Does the backward of a chunk expanded from `in` end in the fused K1^T (backward() given a FusedReduce)?  The fused
    // kernels have no affine (warped) variant.
    bool folds_k1t(const EotIn& in) const { return !in.xf && bwd != END_CUDNN; }
    // cuDNN's stem kernels degrade badly beyond ~128 samples of 224x224: the library forward, dgrad and filter gradient
    // run in slices of SUB samples.  f(n, x, y): a slice of x ([N,H,H,x_ch], input side) and of y ([N,H/2,H/2,64]).
    template <class F>
    void cudnn_slices(int N, const void* x, int x_ch, const void* y, F f) const {
      const int H = e->H, hs = e->Hs();
      for (int n0 = 0; n0 < N; n0 += SUB)
        f(std::min(SUB, N - n0), (char*)x + (size_t)n0 * H * H * x_ch * e->es, (char*)y + (size_t)n0 * hs * hs * STEM_CH * e->es);
    }
    // the own kernels and the max-pool, also behind the op-level test hooks; each returns its launch count (run())
    int own_forward(const void* input, void* out, int N, cudaStream_t st) const {
      return dp::launch_stem_forward(input, w_kn, out, N, e->H, e->H, st);
    }
    // ConstantPad2d(1, 0) + MaxPool2d(3, 2) of x [N,hs,hs,C] into y [N,hs/2,hs/2,C] (argmax: null or [N,hs/2,hs/2,C])
    int pool_forward(const void* x, void* y, int8_t* amax, int N, int hs, int C, cudaStream_t st) const {
      return dp::launch_maxpool_forward(x, y, amax, N, hs, hs, C, e->bf16, st);
    }
    int pool_backward(const void* dy, const int8_t* amax, void* dx, int N, int hs, int C, cudaStream_t st) const {
      return dp::launch_maxpool_backward(dy, amax, dx, N, hs, hs, C, e->bf16, st);
    }
    int own_wgrad(const void* input, const void* dY, float* partial, float* acc, int N, int cin_pad, cudaStream_t st) const {
      return dp::launch_stem_wgrad(input, dY, partial, acc, N, e->H, e->H, cin_pad, st);
    }
    int fused_reduce(const void* dY, const FusedReduce& fr, int N, cudaStream_t st) const {
      return dp::launch_stem_bwd_reduce(dY, conv.w, conv.cin_pad, fr.rects, fr.G, fr.B, fr.S, fr.n0, N, e->H, e->H, st, fr.bank_or_null());
    }
    int fused_pool_reduce(const void* dpool, const int8_t* amax, const FusedReduce& fr, int N, cudaStream_t st) const {
      return dp::launch_stem_bwd_pool_reduce(dpool, amax, conv.w, conv.cin_pad, fr.rects, fr.G, fr.B, fr.S, fr.n0, N, e->H, e->H, st,
                                             fr.bank_or_null());
    }
    // input [N,H,H,in_ch] -> conv -> max-pool into L.x0 (train: keep the argmax for the backward)
    void forward(const Lane& L, int N, const void* input, bool train, cudaStream_t st) const {
      const int H = e->H, hs = e->Hs(), hp = e->Hp();
      if (fwd == FWD_OWN) {
        e->run("stem_conv_fwd", ((double)N * H * H * 3 + (double)N * hs * hs * STEM_CH) * e->es, 2.0 * N * hs * hs * STEM_CH * 147, st,
               [&] { return own_forward(input, L.act, N, st); });
      } else {
        cudnn_slices(N, input, in_ch, L.act, [&](int n, char* x, char* y) { e->conv_fwd(L, 0, conv, n, H, hs, x, y, st); });
      }
      e->run("maxpool_fwd", (double)N * (hs * hs + hp * hp) * STEM_CH * e->es, 0, st,
             [&] { return pool_forward(L.act, L.x0, train ? L.pool_amax : nullptr, N, hs, STEM_CH, st); });
    }
    // d_x0: the gradient at the max-pool output.  Max-pool backward, the stem's weight gradient when wg wants it, then
    // the dgrad, or the fused reduce when fr is given.  Returns d/d(input) ([N,H,H,dx_ch] in L.g[2]), or null when
    // nothing of it was produced.
    void* backward(const Lane& L, int N, const void* d_x0, const FusedReduce* fr, const Wgrad* wg, cudaStream_t st) const {
      const int H = e->H, hs = e->Hs();
      void *const GB = L.g[1], *const GC = L.g[2];
      const bool want_w = wg && e->want_conv(conv);
      if (wg && !wg->need_dx && !want_w) return nullptr;
      if (fr && bwd == END_FUSED_POOL_REDUCE && !wg) {
        // max-pool backward + stem dgrad + masked EOT reduce in one kernel: neither d_stem nor d/d(input) is written
        e->run("stem_bwd_reduce", (double)N * (hs / 2) * (hs / 2) * STEM_CH * (e->es + 1) + 3.0 * H * H * 4 * (double)N / fr->S,
               2.0 * N * hs * hs * STEM_CH * 147, st, [&] { return fused_pool_reduce(d_x0, L.pool_amax, *fr, N, st); });
        return nullptr;
      }
      e->run("maxpool_bwd", (double)N * (hs * hs + (hs / 2) * (hs / 2)) * STEM_CH * e->es, 0, st,
             [&] { return pool_backward(d_x0, L.pool_amax, GB, N, hs, STEM_CH, st); });
      if (want_w) {                                                                // dY = the max-pool adjoint (GB)
        float* const acc = e->acc_of(L, conv.pid);
        if (wgrad == WG_OWN)
          e->run("stem_wgrad", (double)N * (H * H * 3 + hs * hs * STEM_CH) * e->es, 2.0 * N * hs * hs * STEM_CH * 147, st,
                 [&] { return own_wgrad(wg->input, GB, L.wg_partial, acc, N, conv.cin_pad, st); });
        else
          cudnn_slices(N, wg->input, in_ch, GB, [&](int n, char* x, char* y) { e->conv_wgrad(L, 0, conv, n, H, hs, x, y, acc, st); });
        if (!wg->need_dx) return nullptr;
      }
      if (fr) {
        e->run("stem_bwd_reduce", (double)N * hs * hs * STEM_CH * e->es + 3.0 * H * H * 4 * (double)N / fr->S,
               2.0 * N * hs * hs * STEM_CH * 147, st, [&] { return fused_reduce(GB, *fr, N, st); });
        return nullptr;
      }
      cudnn_slices(N, GC, dx_ch, GB, [&](int n, char* x, char* y) { e->conv_bwd(L, 0, conv, n, H, hs, y, x, st); });
      return GC;
    }
  };
  Stem stem;

  // ---- classifier forward ------------------------------------------------------------------
  // input: [N,H,H,stem.in_ch] T.  train: keep what backward needs.  Leaves logits in L.logits.
  void forward(const Lane& L, int N, const void* input, bool train, cudaStream_t st) {
    NvtxRange nvtx_("dorpatch.classifier_forward");
    if (!weights_loaded) fail("dp_engine_load_weights has not been called");
    if (N > chunk) fail("forward: N=%d exceeds chunk=%d", N, chunk);
    CUDNN_OK(cudnnSetStream(L.cudnn, st));
    void* const act = L.act;
    stem.forward(L, N, input, train, st);
    const void* cur = L.x0;
    for (size_t bi = 0; bi < blocks.size(); ++bi) {
      const Block& b = blocks[bi];
      const Lane::Saved& s = L.saved[bi];
      const int lid = (int)bi + 1;
      const int pin_ = b.hin * b.hin, pout = b.hout * b.hout;
      // opt-in: statistics pass + wgmma GEMM that normalises its A operand on the way into shared memory
      // (the relu(gn(.)) tensors of norm1 / norm3 are never written); blocks with a downsample branch keep norm1.
      const bool fuse1 = fused_gemm && !b.has_ds && dp::gn_gemm_supported(pin_, b.cin, b.mid);
      const bool fuse3 = fused_gemm && dp::gn_gemm_supported(pout, b.mid, b.cout);
      // xp = relu(gn1(cur))
      if (fuse1)
        run("gn_stats", 1.0 * N * pin_ * b.cin * es, 0, st, [&] { return dp::launch_gn_stats(cur, L.gn_partial, s.st1, N, pin_, b.cin, bf16, st); });
      else
        run("gn_relu_fwd", 2.0 * N * pin_ * b.cin * es, 0, st,
            [&] { return dp::launch_gn_relu_forward(cur, act, b.n1.gamma, b.n1.beta, L.gn_partial, s.st1, N, pin_, b.cin, bf16, st); });
      const void* shortcut = cur;
      if (b.has_ds) {
        const void* src = act;
        if (b.stride == 2) {
          run("subsample", 2.0 * N * pout * b.cin * es, 0, st, [&] { return dp::launch_subsample2(act, L.act2, N, b.hin, b.hin, b.cin, bf16, st); });
          src = L.act2;
        }
        gemm(L, N * pout, b.cout, b.cin, 0, b.ds.w, src, nullptr, 0.f, s.out, st);
        shortcut = s.out;
      }
      if (fuse1)
        run("gn_gemm1x1_fwd", ((double)N * pin_ * (b.cin + b.mid) + (double)b.mid * b.cin) * es, 2.0 * N * pin_ * b.mid * b.cin, st,
            [&] { return dp::launch_gn_gemm_forward(cur, b.c1p, s.st1, b.n1.gamma, b.n1.beta, nullptr, s.h1, N, pin_, b.cin, b.mid, st); });
      else
        gemm(L, N * pin_, b.mid, b.cin, 0, b.c1.w, act, nullptr, 0.f, s.h1, st);
      run("gn_relu_fwd", 2.0 * N * pin_ * b.mid * es, 0, st,
          [&] { return dp::launch_gn_relu_forward(s.h1, act, b.n2.gamma, b.n2.beta, L.gn_partial, s.st2, N, pin_, b.mid, bf16, st); });
      conv_fwd(L, lid, b.c2, N, b.hin, b.hout, act, s.h2, st);
      if (fuse3) {
        run("gn_stats", 1.0 * N * pout * b.mid * es, 0, st, [&] { return dp::launch_gn_stats(s.h2, L.gn_partial, s.st3, N, pout, b.mid, bf16, st); });
        run("gn_gemm1x1_fwd", ((double)N * pout * (b.mid + 2.0 * b.cout) + (double)b.cout * b.mid) * es, 2.0 * N * pout * b.cout * b.mid, st,
            [&] { return dp::launch_gn_gemm_forward(s.h2, b.c3p, s.st3, b.n3.gamma, b.n3.beta, shortcut, s.out, N, pout, b.mid, b.cout, st); });
      } else {
        run("gn_relu_fwd", 2.0 * N * pout * b.mid * es, 0, st,
            [&] { return dp::launch_gn_relu_forward(s.h2, act, b.n3.gamma, b.n3.beta, L.gn_partial, s.st3, N, pout, b.mid, bf16, st); });
        gemm(L, N * pout, b.cout, b.mid, 0, b.c3.w, act, shortcut, 1.f, s.out, st);   // + shortcut fused as C operand
      }
      cur = s.out;
    }
    const Block& last = blocks.back();
    const int pl = last.hout * last.hout;
    run("head_fwd", (double)N * pl * last.cout * es, 2.0 * N * last.cout * K, st, [&] {
      const int n = dp::launch_gn_stats(cur, L.gn_partial, L.head_stats, N, pl, last.cout, bf16, st);
      return n + dp::launch_head_pool(cur, head_gn.gamma, head_gn.beta, L.head_stats, L.pooled, N, pl, last.cout, bf16, st);
    });
    gemm(L, N, K, last.cout, 2, fc_w, L.pooled, nullptr, 0.f, L.logits, st);   // logits = pooled * Wfc^T + b (fp32)
  }

  // ---- classifier backward (to the input) -----------------------------------------------------
  // dlog: [N,K] fp32 dev.  Returns d/d(input) ([N,H,H,stem.dx_ch] T, in one of the lane's gradient buffers), or null
  // when nothing of it was produced.
  // `fused`: non-null -> finish with the stem's fused K1^T into fused->G instead (only where stem.folds_k1t).
  void* backward(const Lane& L, int N, const float* dlog, cudaStream_t st, const FusedReduce* fused = nullptr, const Wgrad* wg = nullptr) {
    NvtxRange nvtx_("dorpatch.classifier_backward");
    CUDNN_OK(cudnnSetStream(L.cudnn, st));
    void* const act = L.act;
    float* const gn_partial = L.gn_partial;
    const Block& last = blocks.back();
    const void* const last_out = L.saved.back().out;
    const int pl = last.hout * last.hout;
    void *GA = L.g[0], *GB = L.g[1], *GC = L.g[2], *GD = L.g[3];
    const bool W = wg != nullptr;
    if (W) {                                                                     // fc: dW += dlogits^T pooled, db += sum dlogits
      const int fw = wparam_idx.at("head.fc.weight"), fb = wparam_idx.at("head.fc.bias");
      if (want[fw]) wgrad_gemm(L, N, K, last.cout, L.pooled, dlog, acc_of(L, fw), true, st);
      if (want[fb]) run("fc_wgrad", (double)N * K * 4, 0, st, [&] { return dp::launch_colsum_add(dlog, acc_of(L, fb), N, K, st); });
      if (!wg->need_dx && wg->lo >= (int)blocks.size() && !want_gn(head_gn)) return nullptr;
    }
    gemm(L, N, last.cout, K, 3, fc_w, dlog, nullptr, 0.f, L.dpooled, st);      // dpooled = dlogits * Wfc (fp32)
    run("head_bwd", 2.0 * N * pl * last.cout * es, 0, st, [&] {
      const int n = dp::launch_pool_grad_bcast(L.dpooled, GB, N, pl, last.cout, bf16, st);
      return n + dp::launch_gn_relu_backward(GB, last_out, nullptr, GA, head_gn.gamma, head_gn.beta, L.head_stats, gn_partial, N, pl, last.cout, bf16, st, head_gn.pos);
    });
    if (W && want_gn(head_gn)) gn_wgrad(L, head_gn, GB, last_out, L.head_stats, N, pl, st);
    const int lo = W && !wg->need_dx ? wg->lo : 0;
    for (int bi = (int)blocks.size() - 1; bi >= lo; --bi) {
      const Block& b = blocks[bi];
      const Lane::Saved& s = L.saved[bi];
      const int lid = bi + 1;
      const int pin_ = b.hin * b.hin, pout = b.hout * b.hout;
      const void* xin = (bi == 0) ? L.x0 : L.saved[bi - 1].out;
      // conv3: dY = d_out (GA), X = relu(gn3(h2)) recomputed into act
      if (W && want_conv(b.c3)) {
        gn_apply(b.n3, s.h2, s.st3, act, N, pout, st);
        wgrad_gemm(L, N * pout, b.cout, b.mid, act, GA, acc_of(L, b.c3.pid), false, st);
      }
      // d_a3 = d_out * W3
      gemm(L, N * pout, b.mid, b.cout, 1, b.c3.w, GA, nullptr, 0.f, GB, st);
      run("gn_relu_bwd", 3.0 * N * pout * b.mid * es, 0, st,
          [&] { return dp::launch_gn_relu_backward(GB, s.h2, nullptr, GC, b.n3.gamma, b.n3.beta, s.st3, gn_partial, N, pout, b.mid, bf16, st, b.n3.pos); });
      if (W && want_gn(b.n3)) gn_wgrad(L, b.n3, GB, s.h2, s.st3, N, pout, st);
      if (W && want_conv(b.c2)) {                                                // conv2: dY = GC, X = relu(gn2(h1))
        gn_apply(b.n2, s.h1, s.st2, act, N, pin_, st);
        conv_wgrad(L, lid, b.c2, N, b.hin, b.hout, act, GC, acc_of(L, b.c2.pid), st);
      }
      conv_bwd(L, lid, b.c2, N, b.hin, b.hout, GC, GB, st);
      run("gn_relu_bwd", 3.0 * N * pin_ * b.mid * es, 0, st,
          [&] { return dp::launch_gn_relu_backward(GB, s.h1, nullptr, GC, b.n2.gamma, b.n2.beta, s.st2, gn_partial, N, pin_, b.mid, bf16, st, b.n2.pos); });
      if (W && want_gn(b.n2)) gn_wgrad(L, b.n2, GB, s.h1, s.st2, N, pin_, st);
      if (W && (want_conv(b.c1) || (b.has_ds && want_conv(b.ds)))) gn_apply(b.n1, xin, s.st1, act, N, pin_, st);   // relu(gn1(xin))
      if (W && want_conv(b.c1)) wgrad_gemm(L, N * pin_, b.mid, b.cin, act, GC, acc_of(L, b.c1.pid), false, st);   // conv1: dY = GC
      if (W && b.has_ds && want_conv(b.ds)) {                                    // downsample: dY = GA, X = (subsampled) act
        const void* src = act;
        if (b.stride == 2) {
          run("subsample", 2.0 * N * pout * b.cin * es, 0, st, [&] { return dp::launch_subsample2(act, L.act2, N, b.hin, b.hin, b.cin, bf16, st); });
          src = L.act2;
        }
        wgrad_gemm(L, N * pout, b.cout, b.cin, src, GA, acc_of(L, b.ds.pid), false, st);
      }
      gemm(L, N * pin_, b.cin, b.mid, 1, b.c1.w, GC, nullptr, 0.f, GB, st);       // d_xp (conv1 path)
      if (b.has_ds) {
        if (b.stride == 2) {
          gemm(L, N * pout, b.cin, b.cout, 1, b.ds.w, GA, nullptr, 0.f, GC, st);
          run("subsample", 3.0 * N * pout * b.cin * es, 0, st, [&] { return dp::launch_subsample2_adjoint_add(GC, GB, N, b.hin, b.hin, b.cin, bf16, st); });
        } else {
          gemm(L, N * pout, b.cin, b.cout, 1, b.ds.w, GA, nullptr, 1.f, GB, st); // accumulate
        }
        run("gn_relu_bwd", 3.0 * N * pin_ * b.cin * es, 0, st,
            [&] { return dp::launch_gn_relu_backward(GB, xin, nullptr, GD, b.n1.gamma, b.n1.beta, s.st1, gn_partial, N, pin_, b.cin, bf16, st, b.n1.pos); });
      } else {
        run("gn_relu_bwd", 4.0 * N * pin_ * b.cin * es, 0, st,
            [&] { return dp::launch_gn_relu_backward(GB, xin, GA, GD, b.n1.gamma, b.n1.beta, s.st1, gn_partial, N, pin_, b.cin, bf16, st, b.n1.pos); });
      }
      if (W && want_gn(b.n1)) gn_wgrad(L, b.n1, GB, xin, s.st1, N, pin_, st);
      std::swap(GA, GD);
    }
    if (W && lo > 0) return nullptr;                                             // nothing below block lo is wanted
    return stem.backward(L, N, GA, fused, wg, st);
  }

  // ---- EOT input: K1 and its adjoint K1^T for the chunk loops and the dp_expand* entry points ------------------------
  // What K1 expands into network input: `img` (plain, or warped per sample by the transforms `xf` [B*S][8]) or the
  // attack's paste of x / mask / pattern with the clip scale (fused), repeated S times per image and occluded by
  // `rects` [B*S][4][4] (null: none), or by the mask bank `bank` when bank.idx is set (img only, not warped).
  struct EotIn {
    const float* img;
    const float *x, *mask, *pattern, *scale;
    const float* xf;
    const int16_t* rects;
    int B, S;
    dp::MaskBank bank;
    static EotIn image(const float* img, const float* xf, const int16_t* rects, int B, int S) {
      return EotIn{img, nullptr, nullptr, nullptr, nullptr, xf, rects, B, S, dp::MaskBank{}};
    }
    static EotIn paste(const float* x, const float* mask, const float* pattern, const float* scale, const int16_t* rects, int B, int S) {
      return EotIn{nullptr, x, mask, pattern, scale, nullptr, rects, B, S, dp::MaskBank{}};
    }
    static EotIn banked(const float* img, const dp::MaskBank& bank, int B, int S) {
      return EotIn{img, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, B, S, bank};
    }
  };
  // K1 for samples [n0, n0 + n) into dst.  Algorithmic bytes: the samples written, plus the fp32 planes read once per
  // image (x, mask and pattern: 7 fused; the image's 3 otherwise).
  void launch_k1(const EotIn& in, int n0, int n, void* dst, cudaStream_t st) {
    const bool fused = in.x != nullptr;
    const double bytes = (double)n * H * H * 3 * es + (fused ? 7.0 : 3.0) * H * H * 4 * (double)n / in.S;
    if (in.bank.idx) {                                   // + each sample's bank rows (one mask) and indices
      if (in.xf || fused) fail("K1: a mask bank occludes an unwarped image only");
      const double bank_bytes = (double)n * (H * dp::bank_words(H) * 4.0 + 8.0);
      run("expand_k1_bank", bytes + bank_bytes, 0, st, [&] {
        return dp::launch_expand(in.img, nullptr, nullptr, nullptr, nullptr, nullptr, dst, in.B, in.S, n0, n, H, H, stem.in_ch, bf16, false, num_sms, st, &in.bank);
      });
    } else if (in.xf)
      run("expand_affine", bytes, 0, st, [&] { return dp::launch_expand_affine(in.img, in.xf, in.rects, dst, in.S, n0, n, H, H, stem.in_ch, bf16, st); });
    else
      run("expand_k1", bytes, 0, st, [&] {
        return dp::launch_expand(in.img, in.x, in.mask, in.pattern, in.scale, in.rects, dst, in.B, in.S, n0, n, H, H, stem.in_ch, bf16, fused, num_sms, st);
      });
  }
  // The network input of samples [n0, n0 + n): their slice of net_in_all when K1 ran once for the whole call, otherwise
  // K1 into the lane's net_in.
  const void* chunk_input(const Lane& L, const EotIn& in, int n0, int n, bool whole, cudaStream_t st) {
    if (whole) return whole_slice(n0);
    launch_k1(in, n0, n, L.net_in, st);
    return L.net_in;
  }
  // Backward of one chunk from the lane's dlogits, then K1^T into G: the fused bf16 stem dgrad + masked reduce when the
  // input is not warped, otherwise the library stem dgrad and then reduce_affine (warped) or reduce.  G null: no input
  // gradient (weight gradients only).
  void backward_reduce(const Lane& L, const EotIn& in, int n0, int n, float* G, cudaStream_t st, const Wgrad* wg = nullptr) {
    const bool fuse = G && stem.folds_k1t(in);
    const FusedReduce fr{in.rects, G, in.B, in.S, n0, in.bank};
    const void* dx = backward(L, n, L.dlogits, st, fuse ? &fr : nullptr, wg);
    if (!G || fuse) return;
    const double bytes = (double)n * H * H * 3 * es + 3.0 * H * H * 4 * (double)n / in.S;
    if (in.bank.idx)
      run("reduce_k1t_bank", bytes + (double)n * (H * dp::bank_words(H) * 4.0 + 8.0), 0, st,
          [&] { return dp::launch_reduce(dx, nullptr, G, in.B, in.S, n0, n, H, H, stem.dx_ch, bf16, st, &in.bank); });
    else if (in.xf)
      run("reduce_affine", bytes, 0, st, [&] { return dp::launch_reduce_affine(dx, in.img, in.xf, in.rects, G, in.S, n0, n, H, H, stem.dx_ch, bf16, st); });
    else
      run("reduce_k1t", bytes, 0, st, [&] { return dp::launch_reduce(dx, in.rects, G, in.B, in.S, n0, n, H, H, stem.dx_ch, bf16, st); });
  }

  // ---- helpers for the attack entry points --------------------------------------------------
  // Host table of n rows -> device `table`, first grown to at least n rows (the old one stays in `allocs` until
  // destroy).  The copy goes through `pin` and is synchronised, since `pin` is reused right after.
  template <class T>
  void stage(T*& table, int& cap, const void* host, int n, size_t row_bytes, cudaStream_t st) {
    if (n > cap) {
      cap = std::max(n, cap * 2);
      table = (T*)dmalloc((size_t)cap * row_bytes);
    }
    const size_t bytes = (size_t)n * row_bytes;
    ensure_pin(bytes);
    memcpy(pin, host, bytes);
    CUDA_OK(cudaMemcpyAsync(table, pin, bytes, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
  }
  void h2d_samples(const int16_t* rects_host, int N, cudaStream_t st) {
    ensure_samples(N);                   // every per-sample buffer holds N rows: rects_d does not grow on its own
    if (rects_host != nullptr) stage(rects_d, cap_samples, rects_host, N, dp::RECT_SHORTS * sizeof(int16_t), st);
  }
  // The mask-bank occlusion of N samples: checks the indices idx_host [N][2] against n_bank masks, stages them into
  // `table` and returns the MaskBank the kernels read.
  dp::MaskBank stage_bank(int32_t*& table, int& cap, const uint32_t* bank, int n_bank, const int32_t* idx_host, int N,
                          const char* fn, cudaStream_t st) {
    if (n_bank < 1) fail("%s: n_bank=%d < 1", fn, n_bank);
    if (!idx_host) fail("%s: null index array", fn);
    if (dp::bank_words(H) > 32) fail("%s: a mask bank needs img <= 1024 (img=%d)", fn, H);
    for (size_t i = 0; i < (size_t)N * 2; ++i) {
      const int32_t k = idx_host[i];
      if (k < -1 || k >= n_bank) fail("%s: mask index %d of sample %d outside [-1, %d)", fn, k, (int)(i / 2), n_bank);
      if (k >= 0 && !bank) fail("%s: sample %d selects mask %d of a null bank", fn, (int)(i / 2), k);
    }
    stage(table, cap, idx_host, N, 2 * sizeof(int32_t), st);
    return dp::MaskBank{bank, table, H, H};
  }
  // A dp_eot_draw of B images x S samples that no dp_failed_set_update_drawn, universe upload or set reset has used up.
  void check_drawn(const char* fn, int B, int S) const {
    if (!draw.fresh) fail("%s: no fresh dp_eot_draw (each draw serves one step: dp_attack_grad_drawn, then dp_failed_set_update_drawn)", fn);
    if (B != draw.B || S != draw.S) fail("%s: B=%d x S=%d, the last draw is %d x %d", fn, B, S, draw.B, draw.S);
  }
  void check_B(int B) const {
    if (B < 1 || B > cfg.max_images) fail("B=%d outside [1, max_images=%d]", B, cfg.max_images);
  }
};

namespace {
// The lanes of one chunk loop.  Two lanes run when the engine has them, the call asks for them (more than one chunk,
// and whatever else the call needs) and the profiler is off (it serialises on one lane so that category times do not
// overlap).  Then both lane streams first wait for everything enqueued so far on the caller's stream, lane l's chunks
// run on lane l's stream, and join() makes the caller's stream wait for both.  Otherwise every chunk runs on the
// caller's stream.
struct LaneWalk {
  dp_engine* e;
  cudaStream_t user;
  bool dual;
  LaneWalk(dp_engine* e_, cudaStream_t user_, bool want_dual) : e(e_), user(user_) {
    dual = want_dual && e->lanes.size() == 2 && !e->prof_on;
    if (!dual) return;
    CUDA_OK(cudaEventRecord(e->ev_prep, user));
    for (auto& L : e->lanes) CUDA_OK(cudaStreamWaitEvent(L.stream, e->ev_prep, 0));
  }
  int lane_of(int chunk_id) const { return dual ? chunk_id & 1 : 0; }   // chunks alternating between the lanes
  cudaStream_t stream(int l) const { return dual ? e->lanes[l].stream : user; }
  void join() const {
    if (!dual) return;
    for (auto& L : e->lanes) {
      CUDA_OK(cudaEventRecord(L.done, L.stream));
      CUDA_OK(cudaStreamWaitEvent(user, L.done, 0));
    }
  }
};
}  // namespace

// =========================================================================================
// C ABI
// =========================================================================================
// Every entry point returns 0, or 1 with the message of what f() threw in dp_last_error.
template <class F>
static int32_t guarded(F&& f) {
  try {
    f();
  } catch (const std::exception& ex) {
    g_last_error = ex.what();
    return 1;
  } catch (...) {
    g_last_error = "unknown C++ exception";
    return 1;
  }
  return 0;
}
// The same for an entry point on engine e: e is not null and its device is current when f(stream) runs.
template <class F>
static int32_t on_engine(dp_engine* e, void* stream, F&& f) {
  return guarded([&] {
    if (!e) fail("null engine");
    CUDA_OK(cudaSetDevice(e->cfg.device));
    f((cudaStream_t)stream);
  });
}

extern "C" {

int32_t dp_abi_version(void) { return DP_ABI_VERSION; }
const char* dp_last_error(void) { return g_last_error.c_str(); }

int32_t dp_engine_create(const dp_config* cfg, dp_engine** out) {
  return guarded([&] {
    if (!cfg || !out) fail("null argument");
    if (cfg->img % 56 != 0 || cfg->img < 56) fail("img=%d must be a positive multiple of 56", cfg->img);
    if (cfg->chunk < 1) fail("chunk must be >= 1");
    if (cfg->max_images < 1) fail("max_images must be >= 1");
    if (cfg->precision < 0 || cfg->precision > 2) fail("unknown precision %d", cfg->precision);
    int ndev = 0;
    CUDA_OK(cudaGetDeviceCount(&ndev));
    if (cfg->device < 0 || cfg->device >= ndev) fail("device %d not present (%d CUDA devices)", cfg->device, ndev);
    CUDA_OK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CUDA_OK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0) fail("device %d is sm_%d%d; this engine is built for sm_90a (H100) only", cfg->device, prop.major, prop.minor);
    dp_engine* e = new dp_engine();
    try {
      e->cfg = *cfg;
      e->num_sms = prop.multiProcessorCount;
      e->bf16 = (cfg->precision == DP_PREC_BF16);
      e->es = e->bf16 ? 2 : 4;
      e->stem.configure(e);
      const char* fg_env = getenv("DORPATCH_FUSED_GEMM");
      e->fused_gemm = e->bf16 && fg_env && atoi(fg_env) != 0;   // validated (tests/test_gpu_ops.py, test_gpu_fused_gemm.py) but slower than cublasLt + GroupNorm: off unless asked for
      if (const char* g_env = getenv("DORPATCH_GRAPH")) e->graphs_on = atoi(g_env) != 0;
      if (const char* k_env = getenv("DORPATCH_K1_WHOLE_MB")) e->k1_whole_max = (size_t)std::max(0, atoi(k_env)) << 20;
      e->H = cfg->img; e->K = cfg->n_classes; e->chunk = cfg->chunk;
      e->cudnn_dt = e->bf16 ? CUDNN_DATA_BFLOAT16 : CUDNN_DATA_FLOAT;
      e->cuda_dt = e->bf16 ? CUDA_R_16BF : CUDA_R_32F;
      e->lt_compute = (cfg->precision == DP_PREC_TF32) ? CUBLAS_COMPUTE_32F_FAST_TF32 : CUBLAS_COMPUTE_32F;
      CUBLAS_OK(cublasLtCreate(&e->lt));
      e->build_arch();
      e->allocate();
    } catch (...) {
      dp_engine_destroy(e);
      throw;
    }
    *out = e;
  });
}

void dp_engine_destroy(dp_engine* e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
  cudaDeviceSynchronize();
  for (auto& kv : e->cudnn_plans) {
    if (kv.second.xdesc) cudnnDestroyTensorDescriptor(kv.second.xdesc);
    if (kv.second.ydesc) cudnnDestroyTensorDescriptor(kv.second.ydesc);
  }
  for (auto& kv : e->wgrad_plans) {
    cublasLtMatmulDescDestroy(kv.second.op);
    cublasLtMatrixLayoutDestroy(kv.second.a);
    cublasLtMatrixLayoutDestroy(kv.second.b);
    cublasLtMatrixLayoutDestroy(kv.second.c);
  }
  for (auto& kv : e->gemm_plans) {
    cublasLtMatmulDescDestroy(kv.second.op);
    cublasLtMatrixLayoutDestroy(kv.second.a);
    cublasLtMatrixLayoutDestroy(kv.second.b);
    cublasLtMatrixLayoutDestroy(kv.second.c);
  }
  auto kill = [](ConvW& c) {
    if (c.wdesc) cudnnDestroyFilterDescriptor(c.wdesc);
    if (c.cdesc) cudnnDestroyConvolutionDescriptor(c.cdesc);
  };
  kill(e->stem.conv);
  for (auto& b : e->blocks) { kill(b.ds); kill(b.c1); kill(b.c2); kill(b.c3); }
  e->drop_graphs();
  for (auto& r : e->prof_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto ev : e->prof_pool) cudaEventDestroy(ev);
  for (auto& L : e->lanes) {
    if (L.stream) cudaStreamDestroy(L.stream);
    if (L.done) cudaEventDestroy(L.done);
    if (L.cudnn) cudnnDestroy(L.cudnn);
  }
  if (e->ev_prep) cudaEventDestroy(e->ev_prep);
  if (e->cap_stream) cudaStreamDestroy(e->cap_stream);
  if (e->net_in_all) cudaFree(e->net_in_all);
  for (void* p : e->allocs) cudaFree(p);
  if (e->pin) cudaFreeHost(e->pin);
  if (e->draw_pin) cudaFreeHost(e->draw_pin);
  if (e->draw_ev) cudaEventDestroy(e->draw_ev);
  if (e->lt) cublasLtDestroy(e->lt);
  delete e;
}

int32_t dp_engine_load_weights(dp_engine* e, int32_t n, const char* const* names, const float* const* ptrs, const int64_t* numels) {
  return on_engine(e, nullptr, [&](cudaStream_t) {
    e->load_weights(n, names, ptrs, numels);
  });
}

int32_t dp_engine_load_weights_dev(dp_engine* e, int32_t n, const char* const* names, const float* const* dev_ptrs,
                                   const int64_t* numels, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    e->load_weights_dev(n, names, dev_ptrs, numels, st);
  });
}

int64_t dp_engine_device_bytes(const dp_engine* e) { return e ? e->device_bytes : 0; }
int64_t dp_engine_launch_count(const dp_engine* e) { return e ? e->launches : 0; }
int64_t dp_engine_graph_replays(const dp_engine* e) { return e ? e->graph_replays : 0; }
const char* dp_engine_graph_status(const dp_engine* e) { return e ? e->graph_msg.c_str() : ""; }

int32_t dp_engine_profile(dp_engine* e, int32_t enable) {
  return on_engine(e, nullptr, [&](cudaStream_t) {
    e->prof_collect();
    e->prof_on = enable != 0;
    if (enable == 2) {   // reset
      for (size_t i = 0; i < e->prof_ms.size(); ++i) { e->prof_ms[i] = 0; e->prof_bytes[i] = 0; e->prof_flops[i] = 0; e->prof_count[i] = 0; }
    }
  });
}

int32_t dp_engine_profile_read(dp_engine* e, int32_t max_n, char* names, int32_t name_stride, double* ms, double* bytes,
                               double* flops, int64_t* counts, int32_t* n_out) {
  return on_engine(e, nullptr, [&](cudaStream_t) {
    e->prof_collect();
    int n = (int)e->prof_names.size();
    if (n > max_n) n = max_n;
    for (int i = 0; i < n; ++i) {
      snprintf(names + (size_t)i * name_stride, name_stride, "%s", e->prof_names[i].c_str());
      ms[i] = e->prof_ms[i]; bytes[i] = e->prof_bytes[i]; flops[i] = e->prof_flops[i]; counts[i] = e->prof_count[i];
    }
    *n_out = n;
  });
}

int32_t dp_input_layout(const dp_engine* e, int32_t* c_pad, int32_t* elem_bytes) {
  return guarded([&] {
    if (!e) fail("null engine");
    if (c_pad) *c_pad = e->stem.in_ch;
    if (elem_bytes) *elem_bytes = (int32_t)e->es;
  });
}

int32_t dp_paste(dp_engine* e, const float* x, const float* mask, const float* pattern, int32_t B, float eps,
                 float* adv_x_out, float* l2_host, float* scale_host, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    e->check_B(B);
    // with an output buffer this is the stand-alone helper (utils.clip, main.py:140): it must not disturb the per-step
    // state (adv_x, clip scale) a dp_attack_grad left behind for dp_attack_update; without one it IS the step's paste
    float* l2d = adv_x_out ? e->helper_l2 : e->l2;
    float* scd = adv_x_out ? e->helper_scale : e->scale;
    e->run(st, [&] { return dp::launch_paste(x, mask, pattern, adv_x_out ? adv_x_out : e->adv_x, l2d, scd, B, e->H, e->H, eps, st); });
    if (l2_host) CUDA_OK(cudaMemcpyAsync(l2_host, l2d, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    if (scale_host) CUDA_OK(cudaMemcpyAsync(scale_host, scd, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    if (l2_host || scale_host) CUDA_OK(cudaStreamSynchronize(st));
  });
}

int32_t dp_window_sum(dp_engine* e, const float* t, int32_t B, int32_t k, int32_t square, float* out_host, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    e->check_B(B);
    if (k < 1 || e->H % k != 0) fail("window %d does not divide img %d", k, e->H);
    const size_t n = (size_t)B * (e->H / k) * (e->H / k);
    float* tmp = e->helper_ws;   // own scratch (never the structural-loss gradient the sign step reads)
    e->run(st, [&] { return dp::launch_window_sum(t, tmp, B, e->H, e->H, k, square != 0, st); });
    CUDA_OK(cudaMemcpyAsync(out_host, tmp, n * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
  });
}

int32_t dp_expand(dp_engine* e, const float* img, int32_t B, int32_t S, const int16_t* rects_host, void* out, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    const int N = B * S;
    if (out == nullptr && N > e->chunk) fail("dp_expand: B*S=%d exceeds chunk=%d and no output buffer was given", N, e->chunk);
    e->h2d_samples(rects_host, N, st);
    e->launch_k1(dp_engine::EotIn::image(img, nullptr, rects_host ? e->rects_d : nullptr, B, S), 0, N, out ? out : e->lanes[0].net_in, st);
  });
}

int32_t dp_expand_bank(dp_engine* e, const float* img, int32_t B, int32_t S, const uint32_t* bank_dev, int32_t n_bank,
                       const int32_t* idx_host, void* out, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    const int N = B * S;
    if (!img || N < 1) fail("dp_expand_bank: bad arguments");
    if (out == nullptr && N > e->chunk) fail("dp_expand_bank: B*S=%d exceeds chunk=%d and no output buffer was given", N, e->chunk);
    const dp::MaskBank bank = e->stage_bank(e->bank_idx_d, e->bank_idx_cap, bank_dev, n_bank, idx_host, N, "dp_expand_bank", st);
    e->launch_k1(dp_engine::EotIn::banked(img, bank, B, S), 0, N, out ? out : e->lanes[0].net_in, st);
  });
}

int32_t dp_expand_dev(dp_engine* e, const float* img, int32_t B, int32_t S, const int16_t* rects_dev, void* out, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!out) fail("dp_expand_dev needs an output buffer");
    e->launch_k1(dp_engine::EotIn::image(img, nullptr, rects_dev, B, S), 0, B * S, out, st);
  });
}

int32_t dp_expand_step_dev(dp_engine* e, const float* x, const float* mask, const float* pattern, int32_t B, int32_t S,
                           const int16_t* rects_dev, int32_t n0, int32_t n, void* out, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!out || !x || !mask || !pattern) fail("dp_expand_step_dev: null pointer");
    if (n0 < 0 || n < 1 || n0 + n > B * S) fail("dp_expand_step_dev: samples [%d, %d) outside [0, %d)", n0, n0 + n, B * S);
    e->check_B(B);
    e->launch_k1(dp_engine::EotIn::paste(x, mask, pattern, e->scale, rects_dev, B, S), n0, n, out, st);
  });
}

int32_t dp_k1_samples_per_launch(const dp_engine* e, int32_t n_samples) {
  if (!e || n_samples < 1) return 0;
  return e->k1_whole_ok(n_samples) ? n_samples : std::min(n_samples, e->chunk);
}

// forward-only scan (collect_failure, PatchCleanser) of N samples expanded from `in`: chunks alternate between the two
// lanes like dp_attack_grad
static void predict_chunks(dp_engine* e, const dp_engine::EotIn& in, int N, int32_t* preds_host, float* logits_host, cudaStream_t st) {
  LaneWalk walk(e, st, N > e->chunk);
  for (int n0 = 0, c = 0; n0 < N; n0 += e->chunk, ++c) {
    const int n = std::min(e->chunk, N - n0);
    const dp_engine::Lane& L = e->lanes[walk.lane_of(c)];
    cudaStream_t const ls = walk.stream(walk.lane_of(c));
    e->forward(L, n, e->chunk_input(L, in, n0, n, false, ls), false, ls);
    e->run(ls, [&] { return dp::launch_argmax(L.logits, e->preds_d + n0, n, e->K, ls); });
    if (logits_host) CUDA_OK(cudaMemcpyAsync(logits_host + (size_t)n0 * e->K, L.logits, (size_t)n * e->K * 4, cudaMemcpyDeviceToHost, ls));
  }
  walk.join();
  CUDA_OK(cudaMemcpyAsync(preds_host, e->preds_d, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
}

int32_t dp_predict(dp_engine* e, const float* img, int32_t B, int32_t S, const int16_t* rects_host, int32_t* preds_host,
                   float* logits_host, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    NvtxRange nvtx_("dorpatch.predict");
    const int N = B * S;
    if (N < 1) fail("dp_predict: empty batch");
    e->forward_clobbered();
    e->h2d_samples(rects_host, N, st);
    predict_chunks(e, dp_engine::EotIn::image(img, nullptr, rects_host ? e->rects_d : nullptr, B, S), N, preds_host, logits_host, st);
  });
}

int32_t dp_predict_bank(dp_engine* e, const float* img, int32_t B, int32_t S, const uint32_t* bank_dev, int32_t n_bank,
                        const int32_t* idx_host, int32_t* preds_host, float* logits_host, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    NvtxRange nvtx_("dorpatch.predict_bank");
    const int N = B * S;
    if (N < 1) fail("dp_predict_bank: empty batch");
    const dp::MaskBank bank = e->stage_bank(e->bank_idx_d, e->bank_idx_cap, bank_dev, n_bank, idx_host, N, "dp_predict_bank", st);
    e->forward_clobbered();
    e->ensure_samples(N);
    predict_chunks(e, dp_engine::EotIn::banked(img, bank, B, S), N, preds_host, logits_host, st);
  });
}

// Everything dp_attack_grad puts on the stream: staging H2D copies, per-image kernels, the chunk loop on one or two
// lanes, result D2H copies into the pinned staging area.  No host synchronisation inside (capturable).
// rects_dev: the occlusions are already on the device (dp_attack_grad_drawn: the last dp_eot_draw's rectangles).
struct GradLayout { size_t rect_bytes, xf_bytes, d2h_off; int32_t* ys; uint8_t* tg; unsigned char* rp; const int16_t* rects_dev; };
static void attack_grad_enqueue(dp_engine* e, const dp_attack_args* a, const GradLayout& L_, cudaStream_t st) {
  const int B = a->B, S = a->S, N = B * S, H = e->H;
  const size_t rect_bytes = L_.rect_bytes, xf_bytes = L_.xf_bytes;
  CUDA_OK(cudaMemcpyAsync(e->y_d, L_.ys, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->tg_d, L_.tg, (size_t)N, cudaMemcpyHostToDevice, st));
  if (rect_bytes) CUDA_OK(cudaMemcpyAsync(e->rects_d, L_.rp, rect_bytes, cudaMemcpyHostToDevice, st));
  if (xf_bytes) {
    CUDA_OK(cudaMemcpyAsync(e->xf_d, L_.rp + rect_bytes, xf_bytes, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemsetAsync(a->grad_adv, 0, (size_t)B * 3 * H * H * sizeof(float), st));   // the adjoint scatters with atomics
  }
  const int16_t* rects = rect_bytes ? e->rects_d : L_.rects_dev;

  const double img_bytes = (double)B * H * H * 4;
  e->run("paste", 10.0 * img_bytes, 0, st, [&] { return dp::launch_paste(a->x, a->mask, a->pattern, e->adv_x, e->l2, e->scale, B, H, H, a->eps, st); });
  e->run("struct", 9.0 * img_bytes, 0, st, [&] { return dp::launch_struct(e->adv_x, a->x, e->loss_struc, e->dLs, B, H, H, st); });
  if (a->stage == 0)
    e->run("maskreg", img_bytes, 0, st,
           [&] { return dp::launch_maskreg(a->mask, e->loss_density, e->group_lasso, e->win_dev, e->grp_ss, B, H, H, e->unit, st); });
  const float inv_s = 1.0f / (float)a->S_total;
  // with transforms each chunk's input is the pasted image adv_x warped; otherwise K1 pastes as it expands
  const dp_engine::EotIn in = xf_bytes ? dp_engine::EotIn::image(e->adv_x, e->xf_d, rects, B, S)
                                       : dp_engine::EotIn::paste(a->x, a->mask, a->pattern, e->scale, rects, B, S);
  // K1 once for the whole step when its output fits the budget (see ensure_net_in_all); the chunks read their slices
  const bool k1_whole = !xf_bytes && e->net_in_all != nullptr && e->k1_whole_ok(N) && (size_t)N * e->sample_in_bytes() <= e->net_in_all_cap;
  if (k1_whole) e->launch_k1(in, 0, N, e->net_in_all, st);
  // Two lanes only when every chunk holds whole images, so no two chunks accumulate into the same G[b]
  LaneWalk walk(e, st, N > e->chunk && e->chunk % S == 0);
  for (int n0 = 0, c = 0; n0 < N; n0 += e->chunk, ++c) {
    const int n = std::min(e->chunk, N - n0);
    const dp_engine::Lane& L = e->lanes[walk.lane_of(c)];
    cudaStream_t const ls = walk.stream(walk.lane_of(c));
    e->forward(L, n, e->chunk_input(L, in, n0, n, k1_whole, ls), true, ls);
    e->run("cw_k4", 2.0 * n * e->K * 4, 0, ls, [&] {
      return dp::launch_cw(L.logits, e->y_d + n0, e->tg_d + n0, a->confidence, inv_s, e->loss_d + n0, e->preds_d + n0, L.dlogits, n, e->K, ls);
    });
    e->backward_reduce(L, in, n0, n, a->grad_adv, ls);
  }
  walk.join();
  // results -> host (pinned staging; the caller synchronises once)
  unsigned char* out = e->pin + L_.d2h_off;
  size_t off = 0;
  auto d2h = [&](const void* src, size_t bytes) { CUDA_OK(cudaMemcpyAsync(out + off, src, bytes, cudaMemcpyDeviceToHost, st)); off += (bytes + 15) / 16 * 16; };
  d2h(e->loss_d, (size_t)N * 4);
  d2h(e->preds_d, (size_t)N * 4);
  d2h(e->loss_struc, (size_t)B * 4);
  d2h(e->loss_density, (size_t)B * 4);
  d2h(e->group_lasso, (size_t)B * 4);
  d2h(e->l2, (size_t)B * 4);
}

static void attack_grad_impl(dp_engine* e, const dp_attack_args* a, cudaStream_t st, const int16_t* rects_dev = nullptr) {
  NvtxRange nvtx_("dorpatch.attack_grad");
  if (!a) fail("null args");
  e->check_B(a->B);
  if (a->S < 1 || a->S_total < a->S) fail("bad S=%d / S_total=%d", a->S, a->S_total);
  if (!a->x || !a->mask || !a->pattern || !a->grad_adv || !a->y_host || !a->targeted_host) fail("null pointer in dp_attack_args");
  const int B = a->B, S = a->S, N = B * S;
  const int unit = a->basic_unit == 0 ? 7 : a->basic_unit;
  if (unit < 1 || e->H % unit != 0) fail("basic_unit=%d does not divide the image size %d", unit, e->H);
  e->unit = unit;
  e->forward_clobbered();
  e->ensure_samples(N);
  if (!a->xform_host) e->ensure_net_in_all(N);
  // per-sample labels / criterion flags / rectangles -> pinned staging.  Layout:
  // [H2D region: ys | tg | rects | xforms][D2H region: results]; the regions never overlap.
  GradLayout L_;
  L_.rect_bytes = a->rects_host ? (size_t)N * dp::RECT_SHORTS * sizeof(int16_t) : 0;
  L_.rects_dev = rects_dev;
  L_.xf_bytes = a->xform_host ? (size_t)N * 8 * sizeof(float) : 0;
  const size_t h2d_bytes = (((size_t)N * 5 + 15) / 16) * 16 + L_.rect_bytes + L_.xf_bytes;
  L_.d2h_off = (h2d_bytes + 255) / 256 * 256;
  e->ensure_pin(L_.d2h_off + (size_t)N * 8 + (size_t)B * 16 + 512);
  L_.ys = (int32_t*)e->pin;
  L_.tg = (uint8_t*)(L_.ys + N);
  L_.rp = (unsigned char*)e->pin + (((size_t)N * 5 + 15) / 16) * 16;
  for (int b = 0; b < B; ++b)
    if (a->y_host[b] < 0 || a->y_host[b] >= e->K) fail("label %lld of image %d outside [0,%d)", (long long)a->y_host[b], b, e->K);
  for (int b = 0; b < B; ++b)
    for (int s = 0; s < S; ++s) { L_.ys[b * S + s] = (int32_t)a->y_host[b]; L_.tg[b * S + s] = a->targeted_host[b]; }
  if (L_.rect_bytes) memcpy(L_.rp, a->rects_host, L_.rect_bytes);
  if (L_.xf_bytes) memcpy(L_.rp + L_.rect_bytes, a->xform_host, L_.xf_bytes);

  bool done = false;
  if (e->graphs_on && !e->prof_on && !L_.xf_bytes) {
    dp_engine::GraphKey key{B, S, a->S_total, a->stage, a->x, a->mask, a->pattern, a->grad_adv, a->eps, a->confidence, L_.rect_bytes ? 1 : (rects_dev ? 2 : 0), unit};
    dp_engine::GraphEnt& ent = e->graphs[key];
    ++ent.calls;
    if (ent.exec != nullptr) {
      CUDA_OK(cudaGraphLaunch(ent.exec, st));
      e->launches += ent.launches; ++e->graph_replays;
      done = true;
    } else if (!ent.failed && ent.calls >= 2) {          // call 1 ran eagerly: every plan / algorithm choice exists now
      const int64_t l0 = e->launches;
      cudaGraph_t graph = nullptr;
      // the legacy / per-thread default streams (PyTorch's default current stream) cannot be captured: record the
      // sequence on an engine-owned stream instead; the instantiated graph launches on the caller's stream either way
      cudaStream_t cs = (st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread) ? e->cap_stream : st;
      const cudaError_t cb = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
      bool ok = cb == cudaSuccess;
      if (ok) {
        try { attack_grad_enqueue(e, a, L_, cs); } catch (const std::exception& ex) { ok = false; e->graph_msg = std::string("enqueue: ") + ex.what(); }
        const cudaError_t ce = cudaStreamEndCapture(cs, &graph);
        if (ce != cudaSuccess || graph == nullptr) { if (ok) e->graph_msg = std::string("end capture: ") + cudaGetErrorString(ce); ok = false; }
      } else e->graph_msg = std::string("begin capture: ") + cudaGetErrorString(cb);
      if (ok) {
        const cudaError_t ci = cudaGraphInstantiate(&ent.exec, graph, 0);
        if (ci != cudaSuccess) { ok = false; ent.exec = nullptr; e->graph_msg = std::string("instantiate: ") + cudaGetErrorString(ci); }
      }
      if (graph) cudaGraphDestroy(graph);
      if (ok) {
        ent.launches = e->launches - l0;
        CUDA_OK(cudaGraphLaunch(ent.exec, st));
        ++e->graph_replays;
        done = true;
      } else {
        cudaGetLastError();                                // clear the capture error; fall back to eager launches for this signature
        e->launches = l0;
        ent.failed = true;
      }
    }
  }
  if (!done) attack_grad_enqueue(e, a, L_, st);
  CUDA_OK(cudaStreamSynchronize(st));
  unsigned char* out = e->pin + L_.d2h_off;
  size_t off = 0;
  auto take = [&](void* dst, size_t bytes, bool want) { if (want && dst) memcpy(dst, out + off, bytes); off += (bytes + 15) / 16 * 16; };
  take(a->loss_adv_host, (size_t)N * 4, true);
  take(a->preds_host, (size_t)N * 4, true);
  take(a->loss_struc_host, (size_t)B * 4, true);
  take(a->loss_density_host, (size_t)B * 4, a->stage == 0);
  take(a->group_lasso_host, (size_t)B * 4, a->stage == 0);
  take(a->l2_host, (size_t)B * 4, true);
}

static void attack_update_impl(dp_engine* e, const dp_update_args* u, cudaStream_t st) {
  NvtxRange nvtx_("dorpatch.attack_update");
  if (!u) fail("null args");
  e->check_B(u->B);
  if (!u->x || !u->mask || !u->pattern || !u->grad_adv || !u->lr_host || !u->structured_host) fail("null pointer in dp_update_args");
  if (u->stage == 0 && !u->coeff_gl_host) fail("coeff_gl_host is required in stage 0");
  const int B = u->B;
  e->ensure_pin((size_t)B * 12 + 64);
  float* h = (float*)e->pin;
  for (int b = 0; b < B; ++b) { h[b] = u->lr_host[b]; h[B + b] = u->structured_host[b]; h[2 * B + b] = u->coeff_gl_host ? u->coeff_gl_host[b] : 0.f; }
  CUDA_OK(cudaMemcpyAsync(e->lr_d, h, (size_t)B * 4, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->structured_d, h + B, (size_t)B * 4, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->coeff_d, h + 2 * B, (size_t)B * 4, cudaMemcpyHostToDevice, st));
  e->run("update_k3", (double)B * e->H * e->H * 4 * (u->stage == 0 ? 15.0 : 13.0), 0, st, [&] {
    return dp::launch_update(u->x, u->mask, u->pattern, u->grad_adv, e->dLs, e->scale, e->win_dev, e->grp_ss, e->lr_d, e->structured_d,
                             e->coeff_d, u->density, u->clip_min, u->clip_max, u->stage, u->grad_pattern_out, u->grad_mask_out, u->grad_pattern_bias, B, e->H, e->H, e->unit, st);
  });
  CUDA_OK(cudaStreamSynchronize(st));   // `pin` may be reused by the next call
}

int32_t dp_attack_grad(dp_engine* e, const dp_attack_args* a, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    attack_grad_impl(e, a, st);
  });
}

int32_t dp_attack_grad_drawn(dp_engine* e, const dp_attack_args* a, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!a) fail("null args");
    if (a->rects_host) fail("dp_attack_grad_drawn: rects_host must be NULL: the occlusions are the last dp_eot_draw's");
    e->check_drawn("dp_attack_grad_drawn", a->B, a->S_total);
    if (a->S != e->draw.S_loc) fail("dp_attack_grad_drawn: S=%d, the draw's local slice has %d samples", a->S, e->draw.S_loc);
    attack_grad_impl(e, a, st, e->draw_rects_d);
  });
}

int32_t dp_attack_update(dp_engine* e, const dp_update_args* u, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    attack_update_impl(e, u, st);
  });
}

int32_t dp_attack_step_host(dp_engine* e, const dp_attack_args* g, const dp_update_args* u, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!g || !u) fail("null args");
    e->check_B(g->B);
    const size_t B = (size_t)g->B, HW = (size_t)e->H * e->H;
    CUDA_OK(cudaMemcpyAsync(e->host_x, g->x, B * 3 * HW * 4, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->host_mask, g->mask, B * HW * 4, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->host_pattern, g->pattern, B * 3 * HW * 4, cudaMemcpyHostToDevice, st));
    dp_attack_args ga = *g;
    ga.x = e->host_x; ga.mask = e->host_mask; ga.pattern = e->host_pattern; ga.grad_adv = e->host_G;
    attack_grad_impl(e, &ga, st);
    dp_update_args ua = *u;
    ua.x = e->host_x; ua.mask = e->host_mask; ua.pattern = e->host_pattern; ua.grad_adv = e->host_G;
    ua.grad_pattern_out = nullptr; ua.grad_mask_out = nullptr; ua.grad_pattern_bias = nullptr;
    attack_update_impl(e, &ua, st);
    CUDA_OK(cudaMemcpyAsync(u->mask, e->host_mask, B * HW * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(u->pattern, e->host_pattern, B * 3 * HW * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
  });
}

/* ---- differentiable classifier: model(occlude(img)) and its input gradient as two calls ------------------------- */
// Forward: dp_predict's chunk loop with the activations kept (train=true); K1 once for the whole call when its output
// fits net_in_all, as dp_attack_grad does.  Lane l ends up holding its last chunk.
// With transforms (xf_host, [N][8]) each chunk's input is dp_attack_grad's affine expansion instead, read from img.
// With a mask bank (bank_idx_host, [N][2] indices into bank_dev's n_bank masks) each sample is occluded from the bank
// instead; the backward reads the bank again, so it must stay unchanged until then.
static void eot_forward_impl(dp_engine* e, const float* img, int B, int S, const int16_t* rects_host, const float* xf_host,
                             float* logits, cudaStream_t st, const uint32_t* bank_dev = nullptr, int n_bank = 0,
                             const int32_t* bank_idx_host = nullptr) {
  NvtxRange nvtx_(xf_host ? "dorpatch.eot_forward_xform" : (bank_idx_host ? "dorpatch.eot_forward_bank" : "dorpatch.eot_forward"));
  const char* fn = xf_host ? "dp_eot_forward_xform" : (bank_idx_host ? "dp_eot_forward_bank" : "dp_eot_forward");
  if (!img || !logits) fail("%s: null pointer", fn);
  e->check_B(B);
  if (S < 1) fail("%s: S=%d < 1", fn, S);
  if (!rects_host && !xf_host && !bank_idx_host && S != 1) fail("dp_eot_forward: S=%d without rectangles (plain classification needs S=1)", S);
  const int N = B * S;
  dp::MaskBank bank{};
  if (bank_idx_host) bank = e->stage_bank(e->eot_bank_idx_d, e->eot_bank_idx_cap, bank_dev, n_bank, bank_idx_host, N, fn, st);
  if (xf_host)
    for (size_t i = 0; i < (size_t)N * 8; ++i)
      if (!std::isfinite(xf_host[i]))
        fail("dp_eot_forward_xform: transform of sample %d has a non-finite value %g at position %d", (int)(i / 8),
             (double)xf_host[i], (int)(i % 8));
  e->forward_clobbered();
  e->eot = dp_engine::EotSig{};
  if (rects_host) e->stage(e->eot_rects_d, e->eot_rects_cap, rects_host, N, dp::RECT_SHORTS * sizeof(int16_t), st);
  if (xf_host) e->stage(e->eot_xf_d, e->eot_xf_cap, xf_host, N, 8 * sizeof(float), st);
  const dp_engine::EotIn in = bank_idx_host ? dp_engine::EotIn::banked(img, bank, B, S)
                                             : dp_engine::EotIn::image(img, xf_host ? e->eot_xf_d : nullptr, rects_host ? e->eot_rects_d : nullptr, B, S);
  const bool whole = !xf_host && e->ensure_net_in_all(N);
  if (whole) e->launch_k1(in, 0, N, e->net_in_all, st);
  LaneWalk walk(e, st, N > e->chunk);
  for (int n0 = 0, c = 0; n0 < N; n0 += e->chunk, ++c) {
    const int n = std::min(e->chunk, N - n0);
    dp_engine::Lane& L = e->lanes[walk.lane_of(c)];
    cudaStream_t const ls = walk.stream(walk.lane_of(c));
    e->forward(L, n, e->chunk_input(L, in, n0, n, whole, ls), true, ls);
    CUDA_OK(cudaMemcpyAsync(logits + (size_t)n0 * e->K, L.logits, (size_t)n * e->K * 4, cudaMemcpyDeviceToDevice, ls));
    L.held = c;
  }
  walk.join();
  e->eot.gen = e->fwd_gen; e->eot.img = img; e->eot.B = B; e->eot.S = S; e->eot.rects = rects_host != nullptr;
  e->eot.xf = xf_host != nullptr;
  e->eot.whole = whole;
  e->eot.bank = bank_idx_host ? bank_dev : nullptr;
}

// Backward: every chunk through dp_engine::backward and K1^T.  A chunk no lane holds any more is recomputed first (its
// K1 slice, then the forward) in the lane whose held chunk is needed latest.  With whole images per chunk the lanes run
// on their own streams, resident chunks first (each G[b] is written by one chunk); otherwise the chunks run in order on
// the caller's stream, since an image's gradient is accumulated across its chunks and the first one overwrites it.
// After a dp_eot_forward_xform, K1^T is the warp adjoint reduce_affine (after the unfused stem dgrad: the fused bf16
// stem_bwd_reduce has no affine variant), which adds into G with atomics: G is zeroed first, and the same lane rule
// keeps two streams from adding into one image.
//
// With parameter gradients (pc, dp_eot_backward_params) every chunk also runs the weight-gradient pass into the
// accumulators of lane c % lanes, in an order fixed by the shapes (descending chunks per lane with two streams,
// ascending on one), so that repeated backwards give the same bits whichever chunks the lanes still hold; the lanes'
// accumulators are added in lane order at the end, by the weight-standardisation adjoint for the convolutions.
// G may then be null: no input gradient, and the backward stops at the lowest block whose parameters are wanted.
struct ParamCall { int n; const char* const* names; float* const* grads; int accumulate; };
static void eot_backward_impl(dp_engine* e, const float* dlogits, float* G, cudaStream_t st, const ParamCall* pc = nullptr) {
  NvtxRange nvtx_(pc ? "dorpatch.eot_backward_params" : "dorpatch.eot_backward");
  const char* fn = pc ? "dp_eot_backward_params" : "dp_eot_backward";
  if (!dlogits || (!G && !pc)) fail("%s: null pointer", fn);
  if (e->eot.gen < 0) fail("%s: no dp_eot_forward has run on this engine", fn);
  if (e->eot.gen != e->fwd_gen)
    fail("%s: stale forward: another forward-type call (dp_predict, dp_attack_grad, dp_net_forward_backward, "
         "dp_eot_forward or new weights) ran on this engine since the dp_eot_forward it would differentiate", fn);
  e->check_B(e->eot.B);
  const int B = e->eot.B, S = e->eot.S, N = B * S, H = e->H, K = e->K;
  const int n_chunks = (N + e->chunk - 1) / e->chunk, nl = (int)e->lanes.size();
  const dp_engine::EotIn in = e->eot.bank ? dp_engine::EotIn::banked(e->eot.img, dp::MaskBank{e->eot.bank, e->eot_bank_idx_d, H, H}, B, S)
                                          : dp_engine::EotIn::image(e->eot.img, e->eot.xf ? e->eot_xf_d : nullptr,
                                                                    e->eot.rects ? e->eot_rects_d : nullptr, B, S);
  dp_engine::Wgrad wg{nullptr, G != nullptr, (int)e->blocks.size()};
  if (pc) {
    if (pc->n < 0 || (pc->n > 0 && (!pc->names || !pc->grads))) fail("%s: null name / gradient list", fn);
    std::vector<char> want(e->wparams.size(), 0);
    for (int i = 0; i < pc->n; ++i) {
      if (!pc->names[i]) fail("%s: null name at position %d", fn, i);
      const int pid = (int)(&e->wparam(pc->names[i]) - e->wparams.data());
      if (!pc->grads[i]) fail("%s: null gradient pointer for '%s'", fn, pc->names[i]);
      if (want[pid]) fail("%s: '%s' is named twice", fn, pc->names[i]);
      want[pid] = 1;
    }
    e->ensure_wgrad_buffers();
    e->want = want;
    size_t lo_off = e->wacc_floats, hi_off = 0;
    for (size_t i = 0; i < want.size(); ++i) {
      if (!want[i]) continue;
      const auto sp = e->wspan(i);
      lo_off = std::min(lo_off, sp.first); hi_off = std::max(hi_off, sp.second);
    }
    if (want[e->stem.conv.pid]) wg.lo = 0;
    for (int bi = (int)e->blocks.size() - 1; bi >= 0; --bi) {
      const Block& b = e->blocks[bi];
      if (e->want_conv(b.c1) || e->want_conv(b.c2) || e->want_conv(b.c3) || (b.has_ds && e->want_conv(b.ds)) ||
          e->want_gn(b.n1) || e->want_gn(b.n2) || e->want_gn(b.n3)) wg.lo = std::min(wg.lo, bi);
    }
    if (hi_off > lo_off)
      for (auto& L : e->lanes) CUDA_OK(cudaMemsetAsync(L.wacc + lo_off, 0, (hi_off - lo_off) * 4, st));
  }
  if (in.xf && G) CUDA_OK(cudaMemsetAsync(G, 0, (size_t)B * 3 * H * H * sizeof(float), st));
  LaneWalk walk(e, st, N > e->chunk && e->chunk % S == 0);
  std::vector<int> order;
  if (pc) {
    for (int c = 0; c < n_chunks; ++c) order.push_back(walk.dual ? n_chunks - 1 - c : c);
  } else if (walk.dual) {
    for (auto& L : e->lanes) if (L.held >= 0) order.push_back(L.held);
    for (int c = 0; c < n_chunks; ++c) if (c != e->lanes[0].held && c != e->lanes[1].held) order.push_back(c);
  } else {
    for (int c = 0; c < n_chunks; ++c) order.push_back(c);
  }
  int last_lane = nl - 1;
  for (size_t i = 0; i < order.size(); ++i) {
    const int c = order[i], n0 = c * e->chunk, n = std::min(e->chunk, N - n0);
    int lane = -1;
    for (int l = 0; l < nl; ++l) if (e->lanes[l].held == c) lane = l;
    if (pc) lane = e->lanes[c % nl].held == c ? c % nl : -(1 + c % nl);   // the accumulators of lane c % nl
    const bool recompute = lane < 0;
    if (pc && recompute) lane = -lane - 1;
    else if (recompute) {                                // evict the held chunk needed latest (never again: latest)
      size_t best_next = 0;
      for (int k = 1; k <= nl; ++k) {
        const int l = (last_lane + k) % nl;              // ties go round-robin, so recomputed chunks alternate lanes
        size_t next = order.size();
        for (size_t j = i + 1; j < order.size(); ++j) if (order[j] == e->lanes[l].held) { next = j; break; }
        if (lane < 0 || next > best_next) { lane = l; best_next = next; }
      }
    }
    last_lane = lane;
    dp_engine::Lane& L = e->lanes[lane];
    cudaStream_t const ls = walk.stream(lane);
    const void* input = e->eot.whole ? e->whole_slice(n0) : L.net_in;   // what the forward left
    if (recompute) {
      L.held = -1;
      input = e->chunk_input(L, in, n0, n, false, ls);
      e->forward(L, n, input, true, ls);
      L.held = c;
    }
    // the caller's rows go to the lane's dlogits buffer: the head GEMM then reads what it reads in dp_attack_grad
    CUDA_OK(cudaMemcpyAsync(L.dlogits, dlogits + (size_t)n0 * K, (size_t)n * K * 4, cudaMemcpyDeviceToDevice, ls));
    wg.input = input;
    e->backward_reduce(L, in, n0, n, G, ls, pc ? &wg : nullptr);
  }
  walk.join();
  if (pc) {                                            // lanes added in order; conv weights through the WS adjoint
    for (int i = 0; i < pc->n; ++i) {
      const dp_engine::WParam& w = e->wparam(pc->names[i]);
      const float* a = e->lanes[0].wacc + w.off;
      const float* b = nl > 1 ? e->lanes[1].wacc + w.off : nullptr;
      if (w.kind == dp_engine::W_CONV) {
        const ConvW& c = *w.conv;
        e->run("ws_wgrad", (double)w.numel * 8 + (double)c.cout * c.k * c.k * c.cin_pad * 4 * nl, 0, st,
               [&] { return dp::launch_ws_backward(c.raw, a, b, pc->grads[i], c.cout, c.cin, c.k, c.k, c.cin_pad, pc->accumulate != 0, st); });
      } else {
        e->run("vec_wgrad", (double)w.numel * 4 * (nl + 2), 0, st,
               [&] { return dp::launch_vec_finish(a, b, pc->grads[i], (size_t)w.numel, pc->accumulate != 0, st); });
      }
    }
  }
}

int32_t dp_eot_forward(dp_engine* e, const float* img, int32_t B, int32_t S, const int16_t* rects_host, float* logits_dev,
                       void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    eot_forward_impl(e, img, B, S, rects_host, nullptr, logits_dev, st);
  });
}

int32_t dp_eot_forward_xform(dp_engine* e, const float* img, int32_t B, int32_t S, const int16_t* rects_host,
                             const float* xform_host, float* logits_dev, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    eot_forward_impl(e, img, B, S, rects_host, xform_host, logits_dev, st);
  });
}

int32_t dp_eot_forward_bank(dp_engine* e, const float* img, int32_t B, int32_t S, const uint32_t* bank_dev, int32_t n_bank,
                            const int32_t* idx_host, float* logits_dev, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!idx_host) fail("dp_eot_forward_bank: null index array");
    eot_forward_impl(e, img, B, S, nullptr, nullptr, logits_dev, st, bank_dev, n_bank, idx_host);
  });
}

int32_t dp_eot_backward(dp_engine* e, const float* dlogits_dev, float* grad_img_dev, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    eot_backward_impl(e, dlogits_dev, grad_img_dev, st);
  });
}

int32_t dp_eot_backward_params(dp_engine* e, const float* dlogits_dev, float* grad_img_dev, int32_t n, const char* const* names,
                               float* const* grad_dev_ptrs, int32_t accumulate, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    ParamCall pc{n, names, grad_dev_ptrs, accumulate};
    eot_backward_impl(e, dlogits_dev, grad_img_dev, st, &pc);
  });
}

int32_t dp_net_forward_backward(dp_engine* e, const float* z, int32_t N, float* logits_dev, const float* dlogits_dev,
                                float* dz_dev, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (N < 1 || N > e->chunk) fail("N=%d outside [1, chunk=%d]", N, e->chunk);
    e->forward_clobbered();
    const dp_engine::Lane& L = e->lanes[0];
    e->run(st, [&] { return dp::launch_pack_nchw(z, L.net_in, N, e->H, e->H, e->stem.in_ch, e->bf16, st); });
    e->forward(L, N, L.net_in, dlogits_dev != nullptr, st);
    if (logits_dev) CUDA_OK(cudaMemcpyAsync(logits_dev, L.logits, (size_t)N * e->K * 4, cudaMemcpyDeviceToDevice, st));
    if (dlogits_dev) {
      if (!dz_dev) fail("dz_dev is required when dlogits_dev is given");
      const void* dx = e->backward(L, N, dlogits_dev, st);
      e->run(st, [&] { return dp::launch_unpack_nhwc(dx, dz_dev, N, e->H, e->H, e->stem.dx_ch, e->bf16, st); });
    }
  });
}

/* ---- failed-mask sets on the device (attack.py:96,187-190,259-267) ------------------------------------- */
int32_t dp_failed_set_reset(dp_engine* e, int32_t n_mask, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (n_mask < 1) fail("dp_failed_set_reset: n_mask %d < 1", n_mask);
    const int words = (int)(((int64_t)n_mask + 31) / 32);
    const size_t B = (size_t)e->cfg.max_images;
    if (words > e->failed_words_alloc) {                 // the old bitmaps stay in `allocs` until destroy
      CUDA_OK(cudaStreamSynchronize(st));
      e->failed_bits = (uint32_t*)e->dmalloc(B * words * 4);
      e->failed_words_alloc = words;
    }
    e->failed_masks = n_mask;
    e->failed_words = words;
    e->draw.fresh = false;
    CUDA_OK(cudaMemsetAsync(e->failed_bits, 0, B * words * 4, st));
    CUDA_OK(cudaStreamSynchronize(st));
  });
}

int32_t dp_failed_set_write(dp_engine* e, int32_t b, const int32_t* idx_host, int32_t n, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (b < 0 || b >= e->cfg.max_images) fail("image %d outside [0, max_images=%d)", b, e->cfg.max_images);
    std::vector<uint32_t> w(e->failed_words, 0u);
    for (int i = 0; i < n; ++i) {
      if (idx_host[i] < 0 || idx_host[i] >= e->failed_masks) fail("mask index %d outside [0, %d)", idx_host[i], e->failed_masks);
      w[idx_host[i] >> 5] |= 1u << (idx_host[i] & 31);
    }
    CUDA_OK(cudaMemcpyAsync(e->failed_bits + (size_t)b * e->failed_words, w.data(), w.size() * 4, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
  });
}

// One step of the failed-set update from the sampled indices idx_dev [B*S] and nff_dev [B] already on the device.
static void failed_update_impl(dp_engine* e, int B, int S, const int32_t* idx_dev, const int32_t* nff_dev, const uint8_t* active_host,
                               const float* loss_host, float thresh, int32_t* count_host, cudaStream_t st) {
  const int N = B * S;
  CUDA_OK(cudaMemcpyAsync(e->failed_active, active_host, (size_t)B, cudaMemcpyHostToDevice, st));
  const float* loss = e->loss_d;                       // default: the per-sample CW losses the last dp_attack_grad left on the device
  if (loss_host != nullptr) {                          // EOT-sharded runs pass the all-gathered losses
    CUDA_OK(cudaMemcpyAsync(e->failed_loss, loss_host, (size_t)N * 4, cudaMemcpyHostToDevice, st));
    loss = e->failed_loss;
  } else if (N > e->cap_samples) fail("dp_failed_set_update: no device losses for %d samples", N);
  e->run(st, [&] {
    return dp::launch_failed_update(e->failed_bits, e->failed_words, idx_dev, loss, nff_dev, e->failed_active, B, S, thresh,
                                    e->failed_count, st);
  });
  CUDA_OK(cudaMemcpyAsync(count_host, e->failed_count, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
}
static void ensure_failed_cap(dp_engine* e, int N) {
  if (N <= e->failed_cap) return;
  e->failed_cap = std::max(N, e->failed_cap * 2);
  e->failed_idx = (int32_t*)e->dmalloc((size_t)e->failed_cap * 4);
  e->failed_loss = (float*)e->dmalloc((size_t)e->failed_cap * 4);
}

int32_t dp_failed_set_update(dp_engine* e, int32_t B, int32_t S, const int32_t* idx_host, const int32_t* nff_host, const uint8_t* active_host,
                             const float* loss_host, float thresh, int32_t* count_host, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    e->check_B(B);
    if (S < 1 || !idx_host || !nff_host || !active_host || !count_host) fail("dp_failed_set_update: bad arguments");
    const int N = B * S;
    ensure_failed_cap(e, N);
    for (int i = 0; i < N; ++i)
      if (idx_host[i] < 0 || idx_host[i] >= e->failed_masks) fail("mask index %d outside [0, %d)", idx_host[i], e->failed_masks);
    CUDA_OK(cudaMemcpyAsync(e->failed_idx, idx_host, (size_t)N * 4, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(e->failed_nff, nff_host, (size_t)B * 4, cudaMemcpyHostToDevice, st));
    failed_update_impl(e, B, S, e->failed_idx, e->failed_nff, active_host, loss_host, thresh, count_host, st);
  });
}

int32_t dp_failed_set_update_drawn(dp_engine* e, int32_t B, int32_t S, const uint8_t* active_host, const float* loss_host, float thresh,
                                   int32_t* count_host, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    e->check_B(B);
    if (!active_host || !count_host) fail("dp_failed_set_update_drawn: bad arguments");
    e->check_drawn("dp_failed_set_update_drawn", B, S);
    ensure_failed_cap(e, B * S);
    e->draw.fresh = false;                             // one update per draw: the next step draws again
    failed_update_impl(e, B, S, e->draw_idx_d, e->draw_nff_d, active_host, loss_host, thresh, count_host, st);
  });
}

/* ---- on-device EOT draw (DorPatch.generate(eot_sampler="device")) ------------------------------------------- */
int32_t dp_eot_universe_upload(dp_engine* e, const int16_t* table_host, int32_t n_mask, int32_t k, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!table_host || n_mask < 1 || k < 1 || k > 4) fail("dp_eot_universe_upload: bad arguments (n_mask=%d, k=%d)", n_mask, k);
    if (dp::eot_draw_smem_bytes(n_mask) > (size_t)227 << 10) fail("dp_eot_universe_upload: %d masks exceed the draw kernel's shared memory", n_mask);
    e->draw.fresh = false;
    e->stage(e->uni_d, e->uni_cap, table_host, n_mask * k * 4, sizeof(int16_t), st);
    e->uni_n = n_mask;
    e->uni_k = k;
  });
}

int32_t dp_eot_draw(dp_engine* e, int32_t B, int32_t S, const uint64_t* seeds_host, int32_t stage, int32_t iter, const uint8_t* active_host,
                    int32_t dual, int32_t rank, int32_t world, int32_t* idx_host_out, int32_t* idx2_host_out, int32_t* nff_host_out,
                    void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    NvtxRange nvtx_("dorpatch.eot_draw");
    e->check_B(B);
    if (!seeds_host || !active_host) fail("dp_eot_draw: null seeds or active flags");
    if (e->uni_n == 0) fail("dp_eot_draw: no universe uploaded (dp_eot_universe_upload)");
    if (S < 1 || S > e->uni_n) fail("dp_eot_draw: S=%d outside [1, n_mask=%d]", S, e->uni_n);
    if (e->uni_n > e->failed_masks)
      fail("dp_eot_draw: the universe's %d masks exceed the failed-set bitmaps of %d (dp_failed_set_reset)", e->uni_n, e->failed_masks);
    if (world < 1 || rank < 0 || rank >= world || S % world != 0) fail("dp_eot_draw: rank %d of world %d does not slice S=%d", rank, world, S);
    if (dual && e->uni_k > 2) fail("dp_eot_draw: dual needs <= 2 rectangles per universe mask, the universe has %d", e->uni_k);
    if (idx2_host_out && !dual) fail("dp_eot_draw: idx2_host_out without dual");
    if (stage < 0 || stage > 255 || iter < 0) fail("dp_eot_draw: bad step (stage %d, iteration %d)", stage, iter);
    const int N = B * S, S_loc = S / world;
    if (2 * N > e->draw_cap) {                           // the old buffers stay in `allocs` until destroy
      e->draw_cap = std::max(2 * N, 2 * e->draw_cap);
      e->draw_idx_d = (int32_t*)e->dmalloc((size_t)e->draw_cap * 4);
      e->draw_tmp_d = (int32_t*)e->dmalloc((size_t)e->draw_cap * 4);
    }
    if (B * S_loc > e->draw_rects_cap) {
      e->drop_graphs();                                  // captured dp_attack_grad_drawn launches hold the old rectangles
      e->draw_rects_cap = std::max(B * S_loc, 2 * e->draw_rects_cap);
      e->draw_rects_d = (int16_t*)e->dmalloc((size_t)e->draw_rects_cap * dp::RECT_SHORTS * sizeof(int16_t));
    }
    // staged parameters: seeds [B] | {stage, iter} | active [B]
    CUDA_OK(cudaEventSynchronize(e->draw_ev));           // the previous draw's copy has left draw_pin
    const size_t o_step = (size_t)B * 8, o_act = o_step + 8;
    memcpy(e->draw_pin, seeds_host, (size_t)B * 8);
    const int32_t step[2] = {stage, iter};
    memcpy(e->draw_pin + o_step, step, sizeof(step));
    memcpy(e->draw_pin + o_act, active_host, (size_t)B);
    CUDA_OK(cudaMemcpyAsync(e->draw_par_d, e->draw_pin, o_act + B, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaEventRecord(e->draw_ev, st));
    int32_t* idx2 = dual ? e->draw_idx_d + N : nullptr;
    const double words = (e->uni_n + 31) / 32;
    e->run("eot_draw", (double)B * (words * 4 + (double)N / B * 4 * (dual ? 2 : 1) + (double)S_loc * dp::RECT_SHORTS * 2), 0, st, [&] {
      return dp::launch_eot_draw(e->failed_bits, e->failed_words, e->uni_d, e->uni_n, e->uni_k, (const uint64_t*)e->draw_par_d,
                                 (const int32_t*)(e->draw_par_d + o_step), e->draw_par_d + o_act, B, S, dual ? 1 : 0, S_loc,
                                 rank * S_loc, e->draw_idx_d, idx2, e->draw_nff_d, e->draw_rects_d, e->draw_tmp_d, st);
    });
    e->draw.fresh = true; e->draw.B = B; e->draw.S = S; e->draw.S_loc = S_loc; e->draw.dual = dual != 0;
    if (idx_host_out || idx2_host_out || nff_host_out) {
      if (idx_host_out) CUDA_OK(cudaMemcpyAsync(idx_host_out, e->draw_idx_d, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
      if (idx2_host_out) CUDA_OK(cudaMemcpyAsync(idx2_host_out, idx2, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
      if (nff_host_out) CUDA_OK(cudaMemcpyAsync(nff_host_out, e->draw_nff_d, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
      CUDA_OK(cudaStreamSynchronize(st));
    }
  });
}

int32_t dp_eot_draw_rects(dp_engine* e, int16_t* rects_host_out, int32_t n, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!e->draw.fresh) fail("dp_eot_draw_rects: no fresh dp_eot_draw");
    if (!rects_host_out || n != e->draw.B * e->draw.S_loc) fail("dp_eot_draw_rects: the last draw has %d samples, buffer holds %d", e->draw.B * e->draw.S_loc, n);
    CUDA_OK(cudaMemcpyAsync(rects_host_out, e->draw_rects_d, (size_t)n * dp::RECT_SHORTS * sizeof(int16_t), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
  });
}

int32_t dp_failed_set_read(dp_engine* e, int32_t b, int32_t* idx_host_out, int32_t cap, int32_t* n_out, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (b < 0 || b >= e->cfg.max_images) fail("image %d outside [0, max_images=%d)", b, e->cfg.max_images);
    std::vector<uint32_t> w(e->failed_words);
    CUDA_OK(cudaMemcpyAsync(w.data(), e->failed_bits + (size_t)b * e->failed_words, w.size() * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    int n = 0;
    for (int j = 0; j < e->failed_words; ++j)            // set bits only: the 90 720-mask universe is 2835 words
      for (uint32_t v = w[j]; v; v &= v - 1) {
        const int i = j * 32 + __builtin_ctz(v);
        if (n < cap && idx_host_out) idx_host_out[n] = i;
        ++n;
      }
    if (n_out) *n_out = n;
    if (n > cap && idx_host_out) fail("dp_failed_set_read: %d indices, buffer holds %d", n, cap);
  });
}

/* ---- op-level test hooks (tests/test_gpu_ops.py, tests/test_gpu_stem_ops.py) --------------------------- */
// G is left to the kernel (no memset), which writes every element of every image: a gap would show as the caller's fill.
int32_t dp_debug_stem_bwd_reduce(dp_engine* e, const void* dY, const int16_t* rects_host, int32_t B, int32_t S, float* G,
                                 void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (e->stem.fwd != dp_engine::Stem::FWD_OWN) fail("dp_debug_stem_bwd_reduce: the fused stem backward exists for the bf16 engine only");
    if (!dY || !G || B < 1 || S < 1) fail("dp_debug_stem_bwd_reduce: bad arguments");
    const int N = B * S;
    e->h2d_samples(rects_host, N, st);
    const dp_engine::FusedReduce fr{rects_host ? e->rects_d : nullptr, G, B, S, 0};
    e->run(st, [&] { return e->stem.fused_reduce(dY, fr, N, st); });
  });
}

int32_t dp_debug_stem_bwd_reduce_bank(dp_engine* e, const void* dY, const uint32_t* bank_dev, int32_t n_bank, const int32_t* idx_host,
                                      int32_t B, int32_t S, float* G, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (e->stem.fwd != dp_engine::Stem::FWD_OWN) fail("dp_debug_stem_bwd_reduce_bank: the fused stem backward exists for the bf16 engine only");
    if (!dY || !G || B < 1 || S < 1) fail("dp_debug_stem_bwd_reduce_bank: bad arguments");
    const int N = B * S;
    const dp::MaskBank bank = e->stage_bank(e->bank_idx_d, e->bank_idx_cap, bank_dev, n_bank, idx_host, N, "dp_debug_stem_bwd_reduce_bank", st);
    const dp_engine::FusedReduce fr{nullptr, G, B, S, 0, bank};
    e->run(st, [&] { return e->stem.fused_reduce(dY, fr, N, st); });
  });
}

int32_t dp_debug_cw(dp_engine* e, const float* logits, const int32_t* y, const uint8_t* targeted, float confidence, float inv_s,
                    float* loss, int32_t* preds, float* dlogits, int32_t N, int32_t K, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!logits || N < 1 || K < 1) fail("dp_debug_cw: bad arguments");
    if (!y) {
      if (!preds) fail("dp_debug_cw: the argmax needs preds");
      e->run(st, [&] { return dp::launch_argmax(logits, preds, N, K, st); });
      return;
    }
    if (!targeted || !loss) fail("dp_debug_cw: the CW loss needs targeted and loss");
    std::vector<int32_t> ys(N);                          // the kernel reads logits[n][y[n]]: check the labels first
    CUDA_OK(cudaMemcpyAsync(ys.data(), y, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    for (int i = 0; i < N; ++i)
      if (ys[i] < 0 || ys[i] >= K) fail("dp_debug_cw: label %d of sample %d outside [0, %d)", ys[i], i, K);
    e->run(st, [&] { return dp::launch_cw(logits, y, targeted, confidence, inv_s, loss, preds, dlogits, N, K, st); });
  });
}

// G images b of the samples [n0, n0 + n) are written where the launch holds b's first sample, otherwise added to.
int32_t dp_debug_reduce(dp_engine* e, const void* dz, const int16_t* rects_host, const uint32_t* bank_dev, int32_t n_bank,
                        const int32_t* idx_host, int32_t B, int32_t S, int32_t n0, int32_t n, float* G, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!dz || !G || B < 1 || S < 1 || n0 < 0 || n < 1 || (int64_t)n0 + n > (int64_t)B * S)
      fail("dp_debug_reduce: bad arguments (B=%d S=%d samples [%d, %d))", B, S, n0, n0 + n);
    const bool banked = bank_dev || idx_host;
    if (banked && rects_host) fail("dp_debug_reduce: rectangles or a mask bank, not both");
    const int N = B * S, H = e->H;
    if (banked) {
      const dp::MaskBank bank = e->stage_bank(e->bank_idx_d, e->bank_idx_cap, bank_dev, n_bank, idx_host, N, "dp_debug_reduce", st);
      e->run(st, [&] { return dp::launch_reduce(dz, nullptr, G, B, S, n0, n, H, H, e->stem.dx_ch, e->bf16, st, &bank); });
    } else {
      e->h2d_samples(rects_host, N, st);
      const int16_t* rects = rects_host ? e->rects_d : nullptr;
      e->run(st, [&] { return dp::launch_reduce(dz, rects, G, B, S, n0, n, H, H, e->stem.dx_ch, e->bf16, st); });
    }
  });
}

int32_t dp_debug_stem_bwd_pool_reduce(dp_engine* e, const void* dpool, const int8_t* amax, const int16_t* rects_host, int32_t B,
                                      int32_t S, float* G, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (e->stem.fwd != dp_engine::Stem::FWD_OWN) fail("dp_debug_stem_bwd_pool_reduce: the fused stem backward exists for the bf16 engine only");
    if (!dpool || !amax || !G || B < 1 || S < 1) fail("dp_debug_stem_bwd_pool_reduce: bad arguments");
    const int N = B * S;
    e->h2d_samples(rects_host, N, st);
    const dp_engine::FusedReduce fr{rects_host ? e->rects_d : nullptr, G, B, S, 0};
    e->run(st, [&] { return e->stem.fused_pool_reduce(dpool, amax, fr, N, st); });
  });
}

int32_t dp_debug_stem_forward(dp_engine* e, const void* in, void* out, void* w_out, int32_t N, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (e->stem.fwd != dp_engine::Stem::FWD_OWN) fail("dp_debug_stem_forward: this engine's stem is not the own bf16 kernel");
    if (!in || !out || N < 1 || N > 65535) fail("dp_debug_stem_forward: bad arguments");
    const ConvW& c = e->stem.conv;
    if (w_out) CUDA_OK(cudaMemcpyAsync(w_out, c.w, (size_t)c.cout * c.k * c.k * c.cin_pad * 2, cudaMemcpyDeviceToDevice, st));
    e->run(st, [&] { return e->stem.own_forward(in, out, N, st); });
  });
}

int32_t dp_debug_maxpool(dp_engine* e, const void* x, void* y, int8_t* amax, const void* dy, void* dx, int32_t N, int32_t Hs,
                         int32_t C, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!x || !y || N < 1 || Hs < 2 || Hs % 2 != 0 || C < 1 || C % (e->bf16 ? 8 : 4) != 0 || (dy && (!amax || !dx)))
      fail("dp_debug_maxpool: bad arguments");
    e->run(st, [&] { return e->stem.pool_forward(x, y, amax, N, Hs, C, st); });
    if (dy) e->run(st, [&] { return e->stem.pool_backward(dy, amax, dx, N, Hs, C, st); });
  });
}

int32_t dp_debug_stem_wgrad(dp_engine* e, const void* in, const void* dY, int32_t N, float* dW, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!in || !dY || !dW || N < 1) fail("dp_debug_stem_wgrad: bad arguments");
    e->ensure_wgrad_buffers();
    CUDA_OK(cudaMemsetAsync(dW, 0, (size_t)STEM_CH * 49 * 3 * 4, st));
    e->run(st, [&] { return e->stem.own_wgrad(in, dY, e->lanes[0].wg_partial, dW, N, 3, st); });
  });
}

int32_t dp_debug_gn_wgrad(dp_engine* e, const void* x, const void* dy, const float* gamma, const float* beta, const float* stats,
                          int32_t N, int32_t P, int32_t C, float* dgb, void* y, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!x || !dy || !gamma || !beta || !stats || !dgb || N < 1 || N > e->chunk || P < 1 || C % dp::GN_GROUPS != 0 || C > 2048)
      fail("dp_debug_gn_wgrad: bad arguments");
    e->ensure_wgrad_buffers();
    CUDA_OK(cudaMemsetAsync(dgb, 0, (size_t)2 * C * 4, st));
    float* const partial = e->lanes[0].wg_partial;
    e->run(st, [&] { return dp::launch_gn_affine_partial(dy, x, gamma, beta, stats, partial, N, P, C, e->bf16, st); });
    e->run(st, [&] { return dp::launch_colsum_add(partial, dgb, N, 2 * C, st); });
    if (y) e->run(st, [&] { return dp::launch_gn_apply(x, y, gamma, beta, stats, N, P, C, e->bf16, st); });
  });
}

int32_t dp_debug_ws_backward(dp_engine* e, const float* w_raw, const float* g_a, const float* g_b, int32_t O, int32_t I, int32_t k,
                             int32_t Ipad, float* out, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!w_raw || !g_a || !out || O < 1 || I < 1 || k < 1 || Ipad < I) fail("dp_debug_ws_backward: bad arguments");
    e->run(st, [&] { return dp::launch_ws_backward(w_raw, g_a, g_b, out, O, I, k, k, Ipad, false, st); });
  });
}

int32_t dp_debug_k1_tuning(int32_t rows, int32_t sg, int32_t mode) {
  dp::set_expand_tuning(rows, sg, mode);
  return 0;
}

int32_t dp_debug_k1_last(int32_t* out4) {
  if (!out4) return 1;
  int v[4]; dp::get_expand_last(v);
  for (int i = 0; i < 4; ++i) out4[i] = v[i];
  return 0;
}

int32_t dp_debug_gn_gemm(dp_engine* e, const void* x, const void* w_nk, const float* stats, const float* gamma, const float* beta,
                         const void* shortcut, void* out, int32_t N, int32_t P, int32_t K, int32_t Nout, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (!dp::gn_gemm_supported(P, K, Nout)) fail("dp_debug_gn_gemm: shape P=%d K=%d Nout=%d not supported by the wgmma kernel", P, K, Nout);
    void* packed = nullptr;
    CUDA_OK(cudaMalloc(&packed, (size_t)Nout * K * 2));
    int fwd = 0;
    try {
      e->run(st, [&] {
        const int n = dp::launch_gn_gemm_pack(w_nk, packed, Nout, K, st);
        return n + (fwd = dp::launch_gn_gemm_forward(x, packed, stats, gamma, beta, shortcut, out, N, P, K, Nout, st));
      });
    } catch (...) {
      cudaFree(packed);
      throw;
    }
    const cudaError_t err = cudaStreamSynchronize(st);
    cudaFree(packed);
    if (!fwd) fail("dp_debug_gn_gemm: launch refused");
    CUDA_OK(err);
  });
}

int32_t dp_debug_gn(dp_engine* e, const void* x, const void* dy, const void* addend, const float* gamma, const float* beta,
                    int32_t gamma_positive, void* y, void* dx, float* stats, int32_t N, int32_t P, int32_t C, void* stream) {
  return on_engine(e, stream, [&](cudaStream_t st) {
    if (N > e->chunk) fail("dp_debug_gn: N=%d exceeds chunk=%d (statistics scratch)", N, e->chunk);
    float* const partial = e->lanes[0].gn_partial;
    if (y == nullptr) {   // statistics only: the pass in front of the wgmma GEMM / the classifier head
      e->run(st, [&] { return dp::launch_gn_stats(x, partial, stats, N, P, C, e->bf16, st); });
      return;
    }
    e->run(st, [&] { return dp::launch_gn_relu_forward(x, y, gamma, beta, partial, stats, N, P, C, e->bf16, st); });
    if (dy != nullptr)
      e->run(st, [&] { return dp::launch_gn_relu_backward(dy, x, addend, dx, gamma, beta, stats, partial, N, P, C, e->bf16, st, gamma_positive != 0); });
  });
}

}  // extern "C"
