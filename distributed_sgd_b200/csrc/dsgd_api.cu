// dsgd_api.cu -- the C ABI declared in include/dsgd.h over the sm_90a kernels in dsgd_kernels.cuh.
// There is no CPU path in this library: without a usable GPU dsgd_create fails with DSGD_ERR_CUDA.
#include "../../include/dsgd.h"

#include <cuda.h>  // driver types only: entry points are looked up through the runtime (load_all_kernels)
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types only: the library itself is bound at run time (see nccl_api)

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "dsgd_kernels.cuh"
#include "dsgd_persistent.cuh"
#include "dsgd_stream.cuh"
#include "dsgd_async.cuh"
#include "dsgd_metrics.cuh"
#include "dsgd_calibrate.cuh"
#include "dsgd_isotonic.cuh"
#include "dsgd_bootstrap.cuh"
#include "dsgd_topics.cuh"
#include <cstdlib>

#include <cub/device/device_radix_sort.cuh>  // header-only: its sort kernels are compiled into this library, for sm_90a
#include <cub/device/device_merge.cuh>       // the curve pass's merge and scan, likewise
#include <cub/device/device_segmented_radix_sort.cuh>   // the threshold tuning's per-topic sort, likewise
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

using namespace dsgd;

struct dsgd_ctx;

namespace {  // internal linkage: none of these types or their instantiations is exported from the library

// Device memory owned by a ctx (or, for a temporary, by one call). The destructor frees it; it runs with the ctx's device
// current (dsgd_destroy and the failure path of dsgd_create set it, and a call sets it before it allocates).
template <class T>
struct dev_buf {
  T *p = nullptr;
  int64_t cap = 0;  // elements
  dev_buf() = default;
  dev_buf(const dev_buf &) = delete;
  dev_buf &operator=(const dev_buf &) = delete;
  ~dev_buf() { release(); }
  operator T *() const { return p; }
  cudaError_t release() {
    if (!p) return cudaSuccess;
    const cudaError_t e = cudaFree(p);
    if (e == cudaSuccess) { p = nullptr; cap = 0; }
    return e;
  }
  // replaces the allocation with one of n elements (contents undefined)
  cudaError_t alloc(int64_t n) {
    cudaError_t e = release();
    if (e != cudaSuccess) return e;
    T *q = nullptr;
    if ((e = cudaMalloc(&q, sizeof(T) * (size_t)n)) == cudaSuccess) { p = q; cap = n; }
    return e;
  }
  // at least n elements: a smaller buffer is replaced by one of max(n, min_cap), zero-filled on ctx->stream if `zero`
  int grow(dsgd_ctx *ctx, int64_t n, int64_t min_cap, bool zero = false);
};

// A stream or event owned by a ctx, destroyed with it.
template <class H, cudaError_t (*Destroy)(H)>
struct cuda_handle {
  H h = nullptr;
  cuda_handle() = default;
  cuda_handle(cuda_handle &&o) noexcept : h(o.h) { o.h = nullptr; }
  cuda_handle(const cuda_handle &) = delete;
  cuda_handle &operator=(const cuda_handle &) = delete;
  ~cuda_handle() { if (h) Destroy(h); }
  operator H() const { return h; }
};
using owned_stream = cuda_handle<cudaStream_t, cudaStreamDestroy>;
using owned_event = cuda_handle<cudaEvent_t, cudaEventDestroy>;

// A peer's buffer as this ctx addresses it: mapped from another process with cudaIpcOpenMemHandle (the mapping is closed
// when it is replaced or destroyed), or a pointer into another ctx of this process (not owned).
struct peer_ptr {
  double *p = nullptr;
  bool via_ipc = false;
  peer_ptr() = default;
  peer_ptr(const peer_ptr &) = delete;
  peer_ptr &operator=(const peer_ptr &) = delete;
  ~peer_ptr() { set(nullptr, false); }
  operator double *() const { return p; }
  void set(double *q, bool ipc) {
    if (p && via_ipc) cudaIpcCloseMemHandle(p);
    p = q;
    via_ipc = ipc;
  }
};

}  // namespace

struct dsgd_ctx {
  int device = 0;
  int32_t dim = 0;
  double lambda = 0.0;
  double lambda1 = 0.0;   // dsgd_set_l1: the L1 penalty of the sync steps (0: off)
  double cw_pos = 1.0, cw_neg = 1.0;   // dsgd_set_class_weights: the weights of the y = +1 and y = -1 rows
  bool sw_on = false;   // dsgd_set_sample_weights: sw holds one weight per loaded row, and the sample-weighted forms run
  int rank = 0, world = 1;
  uint32_t flags = 0;
  int sm_count = 0;
  std::string dev_name;

  owned_stream own_stream;
  cudaStream_t stream = nullptr;
  owned_event ev0, ev1;
  int64_t launches = 0;

  // rows
  int64_t n_rows = 0, nnz = 0, n_pairs = 0;
  dev_buf<uint32_t> rp16;
  dev_buf<uint2> pairs;
  dev_buf<int8_t> label;
  dev_buf<float> yabs;   // label * sum_j |x_j| per row (dsgd_kernels.cuh: k_repack)
  dev_buf<double> sw;    // dsgd_set_sample_weights: one fp64 weight per row (allocated on first use, freed with the rows)
  // dsgd_load_topics: each row's topic ids (a CSR over the rows, ids ascending within a row), the labels dsgd_load_csr
  // loaded (dsgd_select_topic(-1) restores them), and the topic count (0: no topics); freed with the rows
  dev_buf<int64_t> t_ptr;
  dev_buf<int32_t> t_ids;
  dev_buf<int8_t> label0;
  int32_t n_topics = 0;
  // a topic evaluation (dsgd_eval_*topics): the T weight vectors and the DSGD_TOPIC_WORDS(T) counter words
  dev_buf<double> t_w;
  dev_buf<unsigned long long> t_cnt;
  // a topic ranking (dsgd_eval_*topic_ranking): its words and limb words; dsgd_topics_topk: the n k ids and margins
  dev_buf<unsigned long long> t_rank;
  dev_buf<int32_t> t_top_ids;
  dev_buf<double> t_top_m;
  // a threshold tuning (dsgd_tune_topic_thresholds*): a group's [G][n] margin keys and has-topic bytes and their sort
  // alternates, the T thresholds and the 8 T words; a thresholded evaluation (dsgd_eval*_thresholded_topics): the T thresholds
  dev_buf<unsigned long long> u_keys, u_alt;
  dev_buf<uint8_t> u_has, u_hasalt;
  dev_buf<double> u_thr;
  dev_buf<long long> u_words;

  // state (fp64, L2 resident) -- g has dim + 2 slots (hinge sum and batch size ride in the allreduce)
  dev_buf<double> w, g, d, w_req;
  dev_buf<float> w32, w32_req;
  dev_buf<unsigned long long> n_exact;  // rows that took the exact fallback in streaming passes (diagnostic)
  bool stream_ready = false;
  dev_buf<double> scal;
  dev_buf<unsigned long long> cnt;
  dev_buf<double> partial;  // 2 doubles per k_update block
  dev_buf<double> out2;     // loss, acc, hinge sum, correct count, ||w||^2
  dev_buf<double> cls_out;  // dsgd_eval*_class: ||w||^2, the two loss sums, correct and rows per class (k_class_fold);
                            // dsgd_eval*_weighted: ||w||^2, the three weighted sums and the correct count (k_sw_fold)
  dev_buf<double> gsum;     // master-side running sum of worker replies (dim + 2)
  std::vector<int32_t> worker_counts;  // logical workers on this ctx (empty: one worker, whole slice)
  int32_t n_local = 1, k_total = 0;    // k_total == 0: world
  bool have_d = false;

  // staged sample indices / per-step losses
  dev_buf<int32_t> samples;
  int64_t samples_n = 0;
  dev_buf<double> losses;
  dev_buf<double> lrs;      // per-step learning rates of a dsgd_sync_steps_lr call that runs the persistent kernel
  dev_buf<double> preds;
  // row ids of a request (forward, gradient, a sampled evaluation; drawn on the device or copied from the host): never the
  // staged stream above
  dev_buf<int32_t> eval_ids;
  // a metrics pass (dsgd_eval_*metrics, dsgd_metrics.cuh): the score keys (positives from the front, negatives from the back),
  // the radix sort's alternate keys and temporary storage, and the counter words (MetricWord)
  dev_buf<unsigned long long> m_keys, m_alt, m_cnt;
  dev_buf<unsigned char> m_tmp;
  // a weighted curve pass (dsgd_eval_*weighted_curve): each key's weight c in the key's slot and its sort alternate, and the
  // runs' inclusive prefix sums of R(c) (never grown by an async ctx, which these calls refuse)
  dev_buf<double> m_val, m_valt;
  dev_buf<limb_sum> c_pre;
  // a curve pass (dsgd_eval_*curve): its counter words (CurveWord), the merged key runs, the exclusive scan of their tie
  // ends, and the points (sort, merge and scan share m_tmp)
  dev_buf<unsigned long long> c_cnt, c_merged;
  dev_buf<int> c_excl;
  dev_buf<double> c_thr;
  dev_buf<long long> c_tp, c_fp;
  // a calibration fit (dsgd_calibrate*, dsgd_calibrate.cuh): one score and one label per position; the control words (the
  // counts, the three accumulator lines, the barrier counter and abort flag, the result); and the quality pass's block
  // (a weighted fit also keeps each position's weight c in k_cw)
  dev_buf<double> k_score, k_cw;
  dev_buf<int8_t> k_lab;
  dev_buf<unsigned long long> k_ctl, k_eval;
  int k_fit_occ = 0;     // CTAs of k_calib_fit<false> per SM at its full shared-memory budget (0: not asked yet)
  int k_fit_occ_w = 0;   // likewise for k_calib_fit<true>
  // an isotonic fit (dsgd_calibrate_isotonic*, dsgd_isotonic.cuh): the hull's two ping-pong vertex buffers, their two
  // count buffers and the scan of the blocks' X counts; X and Y; the block rows and positives; the X count.  A map applied
  // to rows (dsgd_isotonic_probabilities, dsgd_eval_isotonic_calibration*): its X and Y
  dev_buf<int> i_hull;
  // a weighted isotonic fit: the points' exact coordinates (all m, then the kept ones), their keep flags and its scan, the
  // kept points' scores, and the blocks' weights and positive weights
  dev_buf<u256> i_wpt;
  dev_buf<int> i_wkeep;
  dev_buf<double> i_wthr, i_wblk;
  dev_buf<double> i_out, i_map;
  dev_buf<long long> i_blk;
  dev_buf<unsigned long long> i_ctl;
  // a bootstrap pass (dsgd_eval_*bootstrap, dsgd_bootstrap.cuh; keys in m_keys / m_alt): each position's tag and its sort
  // alternate, the group starts and (every model but the SVM) the losses by position and in sorted order, and a chunk's
  // replicate words
  dev_buf<uint32_t> b_tag, b_tagt;
  dev_buf<int> b_gs;
  dev_buf<double> b_loss, b_eloss;
  dev_buf<unsigned long long> b_out;
  // a weighted bootstrap pass (dsgd_eval_*weighted_bootstrap) also keeps, in sorted order, the last index of every element's
  // tie group (the first in b_gs) and its weight c (fl(c L) in b_eloss)
  dev_buf<int> b_gl;
  dev_buf<double> b_c;

  ncclComm_t comm = nullptr;

  // persistent sync kernel resources (allocated on first use)
  dev_buf<double> p_wbuf[2];   // K GPUs
  dev_buf<double> p_gbuf[3];   // K GPUs
  dev_buf<double2> p_rec[3];   // one GPU: rotating {W, g} records
  dev_buf<unsigned long long> p_acc;   // fixed-point accumulators of the per-CTA partials [3][kAccStride]
  dev_buf<unsigned> p_hinge;   // one GPU: hinge count of every step and CTA [n_steps][CTAs]
  dev_buf<unsigned long long> p_hcode;   // one GPU with sample weights: the rows' 2-bit hinge codes [n_steps][CTAs]
  dev_buf<double> p_loss_nrm;  // one GPU: the norms of every step's loss [2][n_steps]
  dev_buf<unsigned> p_bar;   // [0]: grid barrier counter, [1]: abort flag
  bool p_ready = false;
  dev_buf<long long> p_tl;   // debug timeline (DSGD_PERSIST_TIMELINE)

  // averaged SGD: per-column fp64 sum of the weights after every sync step since dsgd_average_begin (which allocates it),
  // and the count
  dev_buf<double> avg;
  bool avg_on = false;        // the sync steps add to avg
  int64_t avg_n = 0;

  // async (Hogwild) mode
  owned_stream astream;   // the worker loop
  owned_stream stream2;   // service calls that must not queue behind anything
  dev_buf<double> m_w;      // master replica hosted by this ctx (dsgd_async_host_master)
  dev_buf<double> outbox;   // dsgd_async_outbox_enable: running sum of -delta of THIS worker (a replica-shaped block)
  peer_ptr peer_w[kMaxReplicas];  // [r] = replica of rank r, [world] = master replica; nullptr: not attached
  dev_buf<int> a_stop;
  dev_buf<unsigned long long> a_cnt;   // [0] claimed, [1] done
  dev_buf<double> a_scratch;           // [lanes][dim]
  dev_buf<int32_t> a_rows, a_assigned, a_replay;
  dev_buf<int32_t> u_idx; dev_buf<double> u_val;  // update_grad staging
  std::mutex u_mu;                  // dsgd_update_grad: one call at a time stages, launches and waits
  bool a_running = false;
  owned_event a_ev0, a_ev1;

  // sync-mode receive area shared with peers over NVLink: value words [sender][parity][dim + 8] x 16 B, then bitmap
  // words [sender][parity][ceil((dim + 1) / 32)] x 8 B (dsgd_persistent.cuh)
  dev_buf<double> xblk;
  peer_ptr peer_x[kMaxWorld];
  int grid_limit = 0;   // dsgd_set_grid_limit: CTAs of the persistent sync kernel (0: one per SM)
  int64_t x_step = 0;   // global step counter of the fused multi-GPU kernel (identical on every rank)
  int64_t x_steps_run = 0;  // SGD steps run by the fused kernel so far (dsgd_xchg_stats)
  dev_buf<unsigned long long> x_llw;  // this rank's weights in LL form, two parities
  dev_buf<unsigned long long> x_stats;  // [0] value words, [1] bitmap words pushed to each peer so far; [2] SGD steps of those launches

  // sampled per-launch timing of the gradient kernel
  int32_t prof_every = 0;
  int64_t prof_seen = 0;
  std::vector<std::pair<owned_event, owned_event>> prof_events;
  size_t prof_used = 0;

  mutable std::string err;
  mutable std::string info;
};

static thread_local std::string g_create_err;

// NCCL is bound lazily with dlopen instead of at link time: a host process may already carry its own libnccl.so.2
// (PyTorch bundles a newer one than the system's), and two different libraries under one SONAME cannot coexist.
// Order: a copy already loaded in the process, then $DSGD_NCCL_PATH, then the default search path.
struct nccl_api {
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
  std::string why;
};
static nccl_api &nccl() {
  static nccl_api api = [] {
    nccl_api a;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h)
      if (const char *p = getenv("DSGD_NCCL_PATH")) h = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { a.why = std::string("cannot load libnccl.so.2: ") + dlerror(); return a; }
    a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    a.CommInitRank = (decltype(a.CommInitRank))dlsym(h, "ncclCommInitRank");
    a.AllReduce = (decltype(a.AllReduce))dlsym(h, "ncclAllReduce");
    a.CommDestroy = (decltype(a.CommDestroy))dlsym(h, "ncclCommDestroy");
    a.GetErrorString = (decltype(a.GetErrorString))dlsym(h, "ncclGetErrorString");
    a.ok = a.GetUniqueId && a.CommInitRank && a.AllReduce && a.CommDestroy && a.GetErrorString;
    if (!a.ok) a.why = "libnccl.so.2 lacks a required symbol";
    return a;
  }();
  return api;
}

static int fail(const dsgd_ctx *ctx, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf; else g_create_err = buf;
  return code;
}

#define CU(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess)                                                                              \
      return fail(ctx, DSGD_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, \
                  __LINE__);                                                                            \
  } while (0)
#define NC(call)                                                                                         \
  do {                                                                                                   \
    ncclResult_t r_ = (call);                                                                            \
    if (r_ != ncclSuccess)                                                                               \
      return fail(ctx, DSGD_ERR_NCCL, "%s failed: %s (%s:%d)", #call, nccl().GetErrorString(r_), __FILE__, \
                  __LINE__);                                                                             \
  } while (0)
#define NEED(cond, code, ...) \
  do {                        \
    if (!(cond)) return fail(ctx, code, __VA_ARGS__); \
  } while (0)
#define LAUNCHED() (++ctx->launches)

template <class T>
int dev_buf<T>::grow(dsgd_ctx *ctx, int64_t n, int64_t min_cap, bool zero) {
  if (cap >= n) return DSGD_OK;
  CU(alloc(std::max(n, min_cap)));
  if (zero) CU(cudaMemsetAsync(p, 0, sizeof(T) * (size_t)cap, ctx->stream));
  return DSGD_OK;
}

// returns the event pair to bracket this gradient launch with, or nullptr
static std::pair<owned_event, owned_event> *prof_slot(dsgd_ctx *ctx) {
  if (ctx->prof_every <= 0) return nullptr;
  if ((ctx->prof_seen++ % ctx->prof_every) != 0) return nullptr;
  if (ctx->prof_used == ctx->prof_events.size()) {
    if (ctx->prof_events.size() >= 16384) return nullptr;
    std::pair<owned_event, owned_event> pe;
    if (cudaEventCreate(&pe.first.h) != cudaSuccess || cudaEventCreate(&pe.second.h) != cudaSuccess) return nullptr;
    ctx->prof_events.push_back(std::move(pe));
  }
  return &ctx->prof_events[ctx->prof_used++];
}

// runs `launch` (one gradient kernel launch on ctx->stream) between the events of prof_slot when this launch is sampled
template <class F>
static void profiled(dsgd_ctx *ctx, F &&launch) {
  auto *pe = prof_slot(ctx);
  if (pe) cudaEventRecord(pe->first, ctx->stream);
  launch();
  if (pe) cudaEventRecord(pe->second, ctx->stream);
}

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// The model of a ctx from its flag (dsgd_create admits at most one model flag), and its name in dsgd_info and messages
static constexpr uint32_t kModelFlags = DSGD_FLAG_LOGISTIC | DSGD_FLAG_SQUARED_HINGE | DSGD_FLAG_MODIFIED_HUBER;
static inline int model_of(const dsgd_ctx *ctx) {
  return (ctx->flags & DSGD_FLAG_LOGISTIC)         ? kLogistic
         : (ctx->flags & DSGD_FLAG_SQUARED_HINGE)  ? kSquaredHinge
         : (ctx->flags & DSGD_FLAG_MODIFIED_HUBER) ? kModifiedHuber
                                                   : kSvm;
}
static const char *const kModelNames[] = {"svm", "logistic", "squared_hinge", "modified_huber"};
// class weights other than (1, 1) are set
static inline bool has_class_weights(const dsgd_ctx *ctx) { return !(ctx->cw_pos == 1.0 && ctx->cw_neg == 1.0); }
// The weighting of a ctx's training passes: sample-weighted whenever sample weights are loaded, all ones included (their
// combined weights include the class weights), else class-weighted with class weights other than (1, 1)
static inline int weighting(const dsgd_ctx *ctx) {
  return ctx->sw_on ? kSampleWeighted : has_class_weights(ctx) ? kClassWeighted : kUnweighted;
}
// an intercept ctx (DSGD_FLAG_INTERCEPT): every weight vector is dim + 1 long, the intercept last (w[dim] on the device too)
static inline bool has_icpt(const dsgd_ctx *ctx) { return (ctx->flags & DSGD_FLAG_INTERCEPT) != 0; }
static inline int64_t wlen(const dsgd_ctx *ctx) { return (int64_t)ctx->dim + (has_icpt(ctx) ? 1 : 0); }
// The intercept of the device weight vector wd (its entry [dim]) on an intercept ctx, else nullptr: the icpt argument of
// every kernel that forms a score
static inline const double *icpt_of(const dsgd_ctx *ctx, const double *wd) { return has_icpt(ctx) ? wd + ctx->dim : nullptr; }
// The one step from a ctx's intercept to a template argument: f(std::true_type{}) on an intercept ctx, else
// f(std::false_type{})
template <class F>
static auto with_icpt(const dsgd_ctx *ctx, F &&f) {
  return has_icpt(ctx) ? f(std::true_type{}) : f(std::false_type{});
}
// The one step from a ctx's run-time model, intercept and a weighting to template arguments: f(model, weighting,
// intercept), all three as std::integral_constant.  with_model fixes the weighting (an evaluation of one tally); with_forms
// takes it at run time.
template <int kWeight, class F>
static int with_model(const dsgd_ctx *ctx, F &&f) {
  constexpr std::integral_constant<int, kWeight> weight{};
  return with_icpt(ctx, [&](auto icpt) {
    switch (model_of(ctx)) {
      case kLogistic: return f(std::integral_constant<int, kLogistic>{}, weight, icpt);
      case kSquaredHinge: return f(std::integral_constant<int, kSquaredHinge>{}, weight, icpt);
      case kModifiedHuber: return f(std::integral_constant<int, kModifiedHuber>{}, weight, icpt);
      default: return f(std::integral_constant<int, kSvm>{}, weight, icpt);
    }
  });
}
template <class F>
static int with_forms(const dsgd_ctx *ctx, int weight, F &&f) {
  return weight == kSampleWeighted ? with_model<kSampleWeighted>(ctx, f)
         : weight == kClassWeighted ? with_model<kClassWeighted>(ctx, f) : with_model<kUnweighted>(ctx, f);
}

// every id names a loaded row (the reference indexes its data array with it); fn is the entry point
static int check_ids(dsgd_ctx *ctx, const int32_t *ids, int64_t n, const char *fn, const char *what) {
  for (int64_t i = 0; i < n; ++i)
    NEED(ids[i] >= 0 && ids[i] < ctx->n_rows, DSGD_ERR_RANGE, "%s: %s %d at position %lld outside [0,%lld)", fn, what,
         ids[i], (long long)i, (long long)ctx->n_rows);
  return DSGD_OK;
}

// ---- lifecycle ---------------------------------------------------------------------------------------

extern "C" int dsgd_create(dsgd_ctx **out, int device, int32_t dim, double lambda, int rank, int world, uint32_t flags) {
  dsgd_ctx *ctx = nullptr;
  if (!out) return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: out is NULL");
  *out = nullptr;
  if (dim <= 0) return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: dim must be positive (got %d)", dim);
  if (world <= 0 || rank < 0 || rank >= world)
    return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: bad rank/world %d/%d", rank, world);
  if ((flags & kModelFlags) & ((flags & kModelFlags) - 1))
    return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: more than one model flag (0x%x)", flags & kModelFlags);
  if ((flags & kModelFlags) && (flags & DSGD_FLAG_ASYNC))
    return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: async mode supports the SVM model only");
  if ((flags & DSGD_FLAG_INTERCEPT) && (flags & DSGD_FLAG_ASYNC))
    return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: async mode has no intercept (DSGD_FLAG_INTERCEPT is sync-mode only)");
  // every async worker pushes each delta into all `world` replicas and the master's, through one table of kMaxReplicas slots
  if ((flags & DSGD_FLAG_ASYNC) && world > kMaxReplicas - 1)
    return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: async mode supports at most %d workers (got world %d)",
                kMaxReplicas - 1, world);
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return fail(nullptr, DSGD_ERR_CUDA, "dsgd_create: no usable CUDA device (%s); this library has no CPU path",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  if (device < 0 || device >= n_dev)
    return fail(nullptr, DSGD_ERR_INVALID, "dsgd_create: device %d out of range [0,%d)", device, n_dev);
  ctx = new dsgd_ctx();
  ctx->device = device; ctx->dim = dim; ctx->lambda = lambda; ctx->rank = rank; ctx->world = world; ctx->flags = flags;
  auto bail = [&](const char *what, cudaError_t err) {
    int rc = fail(nullptr, DSGD_ERR_CUDA, "dsgd_create: %s: %s", what, cudaGetErrorString(err));
    delete ctx;   // releases what was made so far
    return rc;
  };
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bail("cudaGetDeviceProperties", e);
  ctx->sm_count = prop.multiProcessorCount;
  ctx->dev_name = prop.name;
  if (prop.major != 9 || prop.minor != 0)   // sm_90a code loads on compute capability 9.0 only
    { int rc = fail(nullptr, DSGD_ERR_CUDA, "dsgd_create: device %d is sm_%d%d; this library is built for sm_90a only",
                    device, prop.major, prop.minor); delete ctx; return rc; }
  if ((e = cudaStreamCreateWithFlags(&ctx->own_stream.h, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  ctx->stream = ctx->own_stream;
  if (flags & DSGD_FLAG_ASYNC) {   // the worker loop's stream and the service stream exist in async mode only: streams
                                   // beyond the device's hardware queues (8 by default) alias and serialise each other
    if ((e = cudaStreamCreateWithFlags(&ctx->astream.h, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
    if ((e = cudaStreamCreateWithFlags(&ctx->stream2.h, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  }
  if ((e = cudaEventCreate(&ctx->ev0.h)) != cudaSuccess) return bail("event", e);
  if ((e = cudaEventCreate(&ctx->ev1.h)) != cudaSuccess) return bail("event", e);
  // a device buffer of n elements, all of it zeroed on the ctx's stream
  auto zeroed = [&](auto &buf, int64_t n, const char *what) {
    if ((e = buf.alloc(n)) == cudaSuccess) e = cudaMemsetAsync(buf.p, 0, sizeof *buf.p * (size_t)n, ctx->stream);
    return e == cudaSuccess ? DSGD_OK : bail(what, e);
  };
  const int64_t nv = (int64_t)dim + kReplicaPad;
  int rc;
  if ((rc = zeroed(ctx->a_stop, 1, "a_stop")) || (rc = zeroed(ctx->a_cnt, 2, "a_cnt")) || (rc = zeroed(ctx->w, nv, "w")) ||
      (rc = zeroed(ctx->g, nv, "g")) || (rc = zeroed(ctx->d, nv, "d")) || (rc = zeroed(ctx->w_req, nv, "w_req")) ||
      (rc = zeroed(ctx->w32, (int64_t)dim + 4, "w32")) || (rc = zeroed(ctx->w32_req, (int64_t)dim + 4, "w32_req")) ||
      (rc = zeroed(ctx->n_exact, 2, "n_exact")) || (rc = zeroed(ctx->scal, kNumScal, "scal")) ||
      (rc = zeroed(ctx->cnt, kNumCnt, "cnt")) || (rc = zeroed(ctx->partial, 2 * (int64_t)cdiv(dim, 256), "partial")) ||
      (rc = zeroed(ctx->out2, 8, "out2")) || (rc = zeroed(ctx->cls_out, 8, "cls_out")) || (rc = zeroed(ctx->gsum, nv, "gsum")))
    return rc;
  if ((e = cudaStreamSynchronize(ctx->stream)) != cudaSuccess) return bail("init memset", e);
  *out = ctx;
  return DSGD_OK;
}

extern "C" int dsgd_destroy(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (ctx->comm) nccl().CommDestroy(ctx->comm);
  delete ctx;   // its members free the device buffers, streams, events and peer mappings
  return DSGD_OK;
}

extern "C" const char *dsgd_last_error(const dsgd_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

extern "C" const char *dsgd_info(const dsgd_ctx *ctx) {
  if (!ctx) return "{}";
  char buf[640];
  snprintf(buf, sizeof buf,
           "{\"device\": %d, \"name\": \"%s\", \"sm_count\": %d, \"arch\": \"sm_90a\", \"dim\": %d, \"rank\": %d, "
           "\"world\": %d, \"n_rows\": %lld, \"nnz\": %lld, \"state_dtype\": \"f64\", \"value_dtype\": \"f32\", "
           "\"model\": \"%s\", \"lambda1\": %.17g, \"class_weights\": [%.17g, %.17g], \"sample_weights\": %s, "
           "\"intercept\": %s}",
           ctx->device, ctx->dev_name.c_str(), ctx->sm_count, ctx->dim, ctx->rank, ctx->world, (long long)ctx->n_rows,
           (long long)ctx->nnz, kModelNames[model_of(ctx)], ctx->lambda1, ctx->cw_pos, ctx->cw_neg,
           ctx->sw_on ? "true" : "false", has_icpt(ctx) ? "true" : "false");
  ctx->info = buf;
  return ctx->info.c_str();
}

extern "C" int dsgd_set_stream(dsgd_ctx *ctx, void *cuda_stream) {
  if (!ctx) return DSGD_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->stream = cuda_stream ? (cudaStream_t)cuda_stream : ctx->own_stream;
  return DSGD_OK;
}

extern "C" int dsgd_synchronize(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_timer_start(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  CU(cudaEventRecord(ctx->ev0, ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_timer_stop(dsgd_ctx *ctx, float *elapsed_ms) {
  if (!ctx || !elapsed_ms) return DSGD_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  CU(cudaEventRecord(ctx->ev1, ctx->stream));
  CU(cudaEventSynchronize(ctx->ev1));
  CU(cudaEventElapsedTime(elapsed_ms, ctx->ev0, ctx->ev1));
  return DSGD_OK;
}

extern "C" int dsgd_launch_count(const dsgd_ctx *ctx, int64_t *count) {
  if (!ctx || !count) return DSGD_ERR_INVALID;
  *count = ctx->launches;
  return DSGD_OK;
}

extern "C" int dsgd_profile_begin(dsgd_ctx *ctx, int32_t sample_every) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(sample_every > 0, DSGD_ERR_INVALID, "dsgd_profile_begin: sample_every must be positive");
  ctx->prof_every = sample_every;
  ctx->prof_seen = 0;
  ctx->prof_used = 0;
  return DSGD_OK;
}

extern "C" int dsgd_profile_end(dsgd_ctx *ctx, float *mean_ms, int64_t *n_sampled) {
  if (!ctx) return DSGD_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  double tot = 0.0;
  for (size_t i = 0; i < ctx->prof_used; ++i) {
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, ctx->prof_events[i].first, ctx->prof_events[i].second));
    tot += ms;
  }
  if (mean_ms) *mean_ms = ctx->prof_used ? (float)(tot / (double)ctx->prof_used) : 0.f;
  if (n_sampled) *n_sampled = (int64_t)ctx->prof_used;
  ctx->prof_every = 0;
  ctx->prof_used = 0;
  return DSGD_OK;
}

// ---- data --------------------------------------------------------------------------------------------

extern "C" int dsgd_load_csr(dsgd_ctx *ctx, int64_t n_rows, int64_t nnz, const int64_t *row_ptr, const int32_t *col,
                             const float *val, const int8_t *label) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n_rows > 0 && nnz >= 0 && row_ptr && label && (nnz == 0 || (col && val)), DSGD_ERR_INVALID,
       "dsgd_load_csr: bad arguments (n_rows=%lld nnz=%lld)", (long long)n_rows, (long long)nnz);
  NEED(n_rows < (int64_t)INT32_MAX, DSGD_ERR_INVALID, "dsgd_load_csr: sample ids are int32; n_rows too large");
  NEED(row_ptr[0] == 0 && row_ptr[n_rows] == nnz, DSGD_ERR_INVALID, "dsgd_load_csr: row_ptr[0] != 0 or row_ptr[n] != nnz");
  // validate + build 16-byte window offsets (host side of the data load, like Dataset.rcv1 building the Map per row)
  std::vector<uint32_t> rp16((size_t)n_rows + 1);
  uint64_t acc = 0;
  for (int64_t r = 0; r < n_rows; ++r) {
    const int64_t len = row_ptr[r + 1] - row_ptr[r];
    NEED(len >= 0, DSGD_ERR_INVALID, "dsgd_load_csr: row_ptr not monotone at row %lld", (long long)r);
    NEED(label[r] == 1 || label[r] == -1, DSGD_ERR_INVALID, "dsgd_load_csr: label of row %lld is %d, expected +1/-1",
         (long long)r, (int)label[r]);
    rp16[(size_t)r] = (uint32_t)acc;
    acc += (uint64_t)((len + 1) / 2);
    NEED(acc < (1ull << 32), DSGD_ERR_INVALID, "dsgd_load_csr: too many non-zeros for 32-bit window offsets");
  }
  rp16[(size_t)n_rows] = (uint32_t)acc;
  for (int64_t k = 0; k < nnz; ++k)
    NEED(col[k] >= 0 && col[k] < ctx->dim, DSGD_ERR_RANGE, "dsgd_load_csr: column %d at position %lld outside [0,%d)",
         col[k], (long long)k, ctx->dim);
  {  // the reference's rows are Maps: a key occurs once per row (any order); per-column stamp of the last row that held it
    std::vector<int64_t> seen((size_t)ctx->dim, -1);
    for (int64_t r = 0; r < n_rows; ++r)
      for (int64_t k = row_ptr[r]; k < row_ptr[r + 1]; ++k) {
        NEED(seen[(size_t)col[k]] != r, DSGD_ERR_INVALID, "dsgd_load_csr: row %lld repeats column %d (position %lld)",
             (long long)r, col[k], (long long)k);
        seen[(size_t)col[k]] = r;
      }
  }
  CU(cudaSetDevice(ctx->device));
  // the staged stream was checked against the previous rows: a shorter set would leave ids past its end in it
  ctx->samples_n = 0;
  // the sample weights named the previous rows: the ctx is unweighted again
  ctx->sw_on = false;
  // the topics named the previous rows too
  ctx->n_topics = 0;
  // all of the previous rows go before any of the new ones is allocated
  CU(ctx->rp16.release()); CU(ctx->pairs.release()); CU(ctx->label.release()); CU(ctx->yabs.release()); CU(ctx->sw.release());
  CU(ctx->t_ptr.release()); CU(ctx->t_ids.release()); CU(ctx->label0.release());
  const int64_t n_pairs = (int64_t)acc * 2;
  CU(ctx->rp16.alloc(n_rows + 1));
  CU(ctx->pairs.alloc(std::max<int64_t>(n_pairs, 1)));
  CU(ctx->label.alloc(n_rows));
  CU(ctx->yabs.alloc(n_rows));
  dev_buf<int64_t> d_rp; dev_buf<int32_t> d_col; dev_buf<float> d_val;
  CU(d_rp.alloc(n_rows + 1));
  CU(d_col.alloc(std::max<int64_t>(nnz, 1)));
  CU(d_val.alloc(std::max<int64_t>(nnz, 1)));
  CU(cudaMemcpyAsync(d_rp, row_ptr, sizeof(int64_t) * ((size_t)n_rows + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (nnz) {
    CU(cudaMemcpyAsync(d_col, col, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(d_val, val, sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice, ctx->stream));
  }
  CU(cudaMemcpyAsync(ctx->rp16, rp16.data(), sizeof(uint32_t) * ((size_t)n_rows + 1), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->label, label, (size_t)n_rows, cudaMemcpyHostToDevice, ctx->stream));
  const int blocks = std::min<int64_t>(cdiv(n_rows, 8), (int64_t)ctx->sm_count * 16);
  k_repack<<<blocks, 256, 0, ctx->stream>>>(d_rp, d_col, d_val, ctx->rp16, ctx->label, n_rows, ctx->pairs, ctx->yabs);
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  CU(d_rp.release()); CU(d_col.release()); CU(d_val.release());
  ctx->n_rows = n_rows; ctx->nnz = nnz; ctx->n_pairs = n_pairs;
  return DSGD_OK;
}

// c and ||w||^2 of the weights `w` into scal[c_slot] and scal[nrm_slot], and their fp32 shadow into w32
static void launch_prepare(dsgd_ctx *ctx, const double *w, float *w32, int c_slot, int nrm_slot) {
  k_prepare<1024><<<1, 1024, 0, ctx->stream>>>(w, ctx->d, ctx->dim, ctx->lambda, ctx->scal + c_slot, ctx->scal + nrm_slot);
  LAUNCHED();
  k_to_f32<<<cdiv(ctx->dim, 256), 256, 0, ctx->stream>>>(w, w32, ctx->dim);
  LAUNCHED();
}

// ||w||_1 of the resident weights into scal[kScalL1], which the per-step L1 update reads for the loss of its step
static void launch_l1_refresh(dsgd_ctx *ctx) {
  k_l1_norm<<<cdiv(ctx->dim, 256), 256, 0, ctx->stream>>>(ctx->w, ctx->dim, ctx->cnt);
  LAUNCHED();
  k_l1_finish<<<1, 1, 0, ctx->stream>>>(ctx->cnt, ctx->scal + kScalL1, nullptr);
  LAUNCHED();
}

// recompute c and ||w||^2 (and, with an L1 penalty, ||w||_1) of the resident weights, refresh the fp32 shadow
static int refresh_resident(dsgd_ctx *ctx) {
  launch_prepare(ctx, ctx->w, ctx->w32, kScalC, kScalNrm2);
  if (ctx->lambda1 > 0.0) launch_l1_refresh(ctx);
  if (ctx->flags & DSGD_FLAG_ASYNC) {
    k_async_init_ctl<1024><<<1, 1024, 0, ctx->stream>>>(ctx->w, ctx->d, ctx->dim);
    LAUNCHED();
  }
  CU(cudaGetLastError());
  return DSGD_OK;
}

extern "C" int dsgd_set_dim_sparsity(dsgd_ctx *ctx, const double *d) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(d, DSGD_ERR_INVALID, "dsgd_set_dim_sparsity: d is NULL");
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(ctx->d, d, sizeof(double) * (size_t)ctx->dim, cudaMemcpyHostToDevice, ctx->stream));
  ctx->have_d = true;
  int rc = refresh_resident(ctx);
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_compute_dim_sparsity(dsgd_ctx *ctx, int64_t n_train, double *d_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->pairs, DSGD_ERR_STATE, "dsgd_compute_dim_sparsity: no rows loaded");
  NEED(n_train >= 0 && n_train <= ctx->n_rows, DSGD_ERR_RANGE, "dsgd_compute_dim_sparsity: n_train %lld outside [0,%lld]",
       (long long)n_train, (long long)ctx->n_rows);
  CU(cudaSetDevice(ctx->device));
  dev_buf<unsigned> df;
  CU(df.alloc(ctx->dim));
  CU(cudaMemsetAsync(df, 0, sizeof(unsigned) * (size_t)ctx->dim, ctx->stream));
  uint32_t end16 = 0;
  CU(cudaMemcpyAsync(&end16, ctx->rp16 + n_train, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int64_t n_pairs = (int64_t)end16 * 2;
  if (n_pairs > 0) {
    const int blocks = std::min<int64_t>(cdiv(n_pairs, 256), (int64_t)ctx->sm_count * 16);
    k_col_hist<<<blocks, 256, 0, ctx->stream>>>(ctx->pairs, n_pairs, df);
    LAUNCHED();
  }
  k_dim_sparsity<<<cdiv(ctx->dim, 256), 256, 0, ctx->stream>>>(df, ctx->dim, ctx->d);
  LAUNCHED();
  CU(cudaGetLastError());
  ctx->have_d = true;
  int rc = refresh_resident(ctx);
  if (rc) return rc;
  if (d_out) CU(cudaMemcpyAsync(d_out, ctx->d, sizeof(double) * (size_t)ctx->dim, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  CU(df.release());
  return DSGD_OK;
}

extern "C" int dsgd_set_weights(dsgd_ctx *ctx, const double *w) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(w, DSGD_ERR_INVALID, "dsgd_set_weights: w is NULL");
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(ctx->w, w, sizeof(double) * (size_t)wlen(ctx), cudaMemcpyHostToDevice, ctx->stream));
  int rc = refresh_resident(ctx);
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_get_weights(dsgd_ctx *ctx, double *w) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(w, DSGD_ERR_INVALID, "dsgd_get_weights: w is NULL");
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(w, ctx->w, sizeof(double) * (size_t)wlen(ctx), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

// ---- sample staging ----------------------------------------------------------------------------------

extern "C" int dsgd_stage_samples(dsgd_ctx *ctx, const int32_t *samples, int64_t n) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->pairs, DSGD_ERR_STATE, "dsgd_stage_samples: no rows loaded");
  NEED(n >= 0 && (n == 0 || samples), DSGD_ERR_INVALID, "dsgd_stage_samples: bad arguments");
  int rc = check_ids(ctx, samples, n, __func__, "sample index");
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  if ((rc = ctx->samples.grow(ctx, n, 1024))) return rc;
  if (n) CU(cudaMemcpyAsync(ctx->samples, samples, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  ctx->samples_n = n;
  return DSGD_OK;
}

// weights to use for a request: NULL -> resident; else copy into w_req and compute its scalars.  On an async ctx NULL is a
// snapshot of the replica taken now, with its scalars computed like those of explicit weights: dsgd_update_grad, a peer's
// pushes and a loop that ended by itself change the replica without refreshing c, ||w||^2 or the fp32 shadow.
static int request_weights(dsgd_ctx *ctx, const double *w, const double **w_dev, const double **c_dev,
                           const double **nrm_dev, const float **w32_dev = nullptr) {
  CU(cudaSetDevice(ctx->device));  // every request path passes here: a caller thread may have another device current
  const bool snapshot = !w && (ctx->flags & DSGD_FLAG_ASYNC);
  if (!w && !snapshot) {
    *w_dev = ctx->w; *c_dev = ctx->scal + kScalC; *nrm_dev = ctx->scal + kScalNrm2;
    if (w32_dev) *w32_dev = ctx->w32;
    return DSGD_OK;
  }
  if (w32_dev) *w32_dev = ctx->w32_req;
  if (snapshot)
    CU(cudaMemcpyAsync(ctx->w_req, ctx->w, sizeof(double) * (size_t)ctx->dim, cudaMemcpyDeviceToDevice, ctx->stream));
  else
    CU(cudaMemcpyAsync(ctx->w_req, w, sizeof(double) * (size_t)wlen(ctx), cudaMemcpyHostToDevice, ctx->stream));
  launch_prepare(ctx, ctx->w_req, ctx->w32_req, kScalReqC, kScalReqNrm2);
  CU(cudaGetLastError());
  *w_dev = ctx->w_req; *c_dev = ctx->scal + kScalReqC; *nrm_dev = ctx->scal + kScalReqNrm2;
  return DSGD_OK;
}

static inline int rows_grid(const dsgd_ctx *ctx, int64_t n) {
  return (int)std::min<int64_t>(std::max<int64_t>(cdiv(n, 8), 1), (int64_t)ctx->sm_count * 8);
}

// ---- streaming pass (large n): fp32 weights staged in shared memory, one persistent CTA per SM (dsgd_stream.cuh) ----
constexpr int64_t kStreamMinRows = 2048;

constexpr size_t kStreamMaxSmem = 227u * 1024u - 1024u;   // the weights' staging of the largest eligible dim
static bool stream_eligible(const dsgd_ctx *ctx, int64_t n) {
  return n >= kStreamMinRows && stream_smem_bytes(ctx->dim) <= kStreamMaxSmem;
}

template <bool kScatter, bool kPreds, bool kContig, bool kCls = false>
static int stream_launch(dsgd_ctx *ctx, const int32_t *samples_dev, int64_t row_begin, int64_t n, const double *w_dev,
                         const float *w32_dev, double *g, double *preds) {
  const size_t smem = stream_smem_bytes(ctx->dim);
  // The attribute belongs to the kernel, not to the ctx: every ctx sets the bound of every eligible dim, so that a ctx of a
  // smaller dim set up later does not lower it under the launches of one of a larger dim.
  const int max_smem = (int)kStreamMaxSmem;
  if (!ctx->stream_ready) {
    CU(cudaFuncSetAttribute(k_stream_rows<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CU(cudaFuncSetAttribute(k_stream_rows<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CU(cudaFuncSetAttribute(k_stream_rows<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CU(cudaFuncSetAttribute(k_stream_rows<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CU(cudaFuncSetAttribute(k_stream_rows<false, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CU(cudaFuncSetAttribute(k_stream_rows<true, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CU(cudaFuncSetAttribute(k_stream_rows<false, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    ctx->stream_ready = true;
  }
  NEED(kContig == (samples_dev == nullptr), DSGD_ERR_INVALID, "stream_launch: sample list / row range mismatch");
  StreamParams sp;
  memset(&sp, 0, sizeof sp);
  sp.rp16 = ctx->rp16; sp.units = reinterpret_cast<const uint4 *>(ctx->pairs.p); sp.yabs = ctx->yabs;
  sp.samples = samples_dev; sp.row_begin = row_begin; sp.n = n;
  sp.w = w_dev; sp.w32 = w32_dev; sp.dim = ctx->dim;
  sp.w_pos = ctx->cw_pos; sp.w_neg = ctx->cw_neg;
  sp.g = g; sp.preds = preds; sp.cnt = ctx->cnt; sp.n_exact = ctx->n_exact; sp.next_block = ctx->n_exact + 1;
  CU(cudaMemsetAsync(ctx->n_exact + 1, 0, sizeof(unsigned long long), ctx->stream));
  // rows per block (the unit of the dynamic work distribution): 32, or fewer when that leaves a warp fewer than ~6 blocks
  const int64_t n_warps_all = (int64_t)ctx->sm_count * (kStreamThreads / 32);
  sp.rows_log2 = 5;
  while (sp.rows_log2 > 3 && ((n + (1 << sp.rows_log2) - 1) >> sp.rows_log2) < 6 * n_warps_all) --sp.rows_log2;
  // the last fifth of the pass goes out in blocks of half the size (not below 8 rows): warps end closer together.
  sp.tail_log2 = std::max(3, sp.rows_log2 - 1);
  sp.n_big = sp.tail_log2 < sp.rows_log2 ? ((n - n / 5) >> sp.rows_log2) : ((n + (1 << sp.rows_log2) - 1) >> sp.rows_log2);
  const int64_t n_blk = sp.n_big + cdiv(std::max<int64_t>(0, n - (sp.n_big << sp.rows_log2)), (int64_t)1 << sp.tail_log2);
  const int grid = (int)std::min<int64_t>(ctx->sm_count, std::max<int64_t>(1, cdiv(n_blk, kStreamThreads / 32)));
  profiled(ctx, [&] { k_stream_rows<kScatter, kPreds, kContig, kCls><<<grid, kStreamThreads, smem, ctx->stream>>>(sp); });
  LAUNCHED();
  CU(cudaGetLastError());
  return DSGD_OK;
}

// ---- forward / gradient / eval -------------------------------------------------------------------------

// The rows of a request: rows [row_begin, row_begin + n) when ids == nullptr, else the n row ids at the device address ids
// (in eval_ids: the staged stream stays as it was for the next dsgd_sync_steps_staged).  rows_range, rows_drawn and
// rows_list check the rows a request names and build its row_set (an evaluation reaches them through resolve_rows); fn is
// the entry point, and every message names it.
struct row_set {
  const int32_t *ids;
  int64_t row_begin, n;
};

static int rows_range(dsgd_ctx *ctx, int64_t row_begin, int64_t row_end, const char *fn, row_set *rows) {
  NEED(ctx->pairs, DSGD_ERR_STATE, "%s: no rows loaded", fn);
  NEED(row_begin >= 0 && row_end <= ctx->n_rows && row_begin <= row_end, DSGD_ERR_RANGE,
       "%s: rows [%lld,%lld) outside [0,%lld)", fn, (long long)row_begin, (long long)row_end, (long long)ctx->n_rows);
  NEED(row_end > row_begin, DSGD_ERR_EMPTY, "%s: empty range (reduce on an empty collection throws in the reference)", fn);
  *rows = {nullptr, row_begin, row_end - row_begin};
  return DSGD_OK;
}

// positions [pos_begin, pos_end) of the sample drawn from rows [row_begin, row_end) with `key`, as row ids into eval_ids
static int rows_drawn(dsgd_ctx *ctx, int64_t row_begin, int64_t row_end, uint64_t key, int64_t pos_begin, int64_t pos_end,
                      const char *fn, row_set *rows) {
  int rc = rows_range(ctx, row_begin, row_end, fn, rows);
  if (rc) return rc;
  const int64_t n = row_end - row_begin;
  NEED(n <= (int64_t)UINT32_MAX, DSGD_ERR_INVALID, "%s: %lld rows; the draw permutes 32-bit positions", fn, (long long)n);
  NEED(pos_begin >= 0 && pos_end <= n, DSGD_ERR_INVALID, "%s: positions [%lld,%lld) outside [0,%lld)", fn,
       (long long)pos_begin, (long long)pos_end, (long long)n);
  NEED(pos_end > pos_begin, DSGD_ERR_EMPTY, "%s: no positions (reduce on an empty collection throws)", fn);
  CU(cudaSetDevice(ctx->device));
  const int64_t k = pos_end - pos_begin;
  if ((rc = ctx->eval_ids.grow(ctx, k, 1024))) return rc;
  k_draw_rows<<<cdiv(k, 256), 256, 0, ctx->stream>>>(ctx->eval_ids, k, (uint32_t)pos_begin,
                                                      dsgd_feistel_half_bits((uint64_t)n), key, (uint32_t)n, row_begin);
  LAUNCHED();
  CU(cudaGetLastError());
  *rows = {ctx->eval_ids, 0, k};
  return DSGD_OK;
}

// Growing a device buffer (cudaMalloc, and cudaFree of the smaller one) waits for the kernels running on the device, so it
// would wait forever for an async loop that runs until stopped.  The start of an async loop therefore sizes the buffers of
// the request calls for n_rows rows (and the sort's storage for them), and a call that would have to grow one while the
// loop runs -- a list of more ids than rows -- is refused.
// The curve pass's merge of the two sorted key runs into c_merged, and the exclusive scan of tie_end over the merged keys
// into c_excl (tmp == nullptr: the storage they need, into bytes).  reserve_requests sizes with these same instantiations.
static cudaError_t merge_runs(dsgd_ctx *ctx, void *tmp, size_t &bytes, const unsigned long long *pos, int64_t n_pos,
                              const unsigned long long *neg, int64_t n_neg) {
  return cub::DeviceMerge::MergeKeys(tmp, bytes, pos, (int)n_pos, neg, (int)n_neg, ctx->c_merged.p, ::cuda::std::less<>{},
                                     ctx->stream);
}
static cudaError_t scan_tie_ends(dsgd_ctx *ctx, void *tmp, size_t &bytes, int64_t n_all) {
  auto flags = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), tie_end{ctx->c_merged.p, (int)n_all});
  return cub::DeviceScan::ExclusiveSum(tmp, bytes, flags, ctx->c_excl.p, (int)n_all, ctx->stream);
}

// The isotonic fit's exclusive scan of the X counts of the B blocks of the hull h into excl (tmp == nullptr: the storage it
// needs, into bytes).
static cudaError_t scan_x_counts(dsgd_ctx *ctx, void *tmp, size_t &bytes, const int *h, int B, int *excl) {
  auto counts = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), iso_x_count{h, B});
  return cub::DeviceScan::ExclusiveSum(tmp, bytes, counts, excl, B, ctx->stream);
}

static int reserve_requests(dsgd_ctx *ctx) {
  const int64_t n = ctx->n_rows;
  int rc;
  if ((rc = ctx->eval_ids.grow(ctx, n, 1024)) || (rc = ctx->preds.grow(ctx, n, 1024)) || (rc = ctx->m_keys.grow(ctx, n, 1024)) ||
      (rc = ctx->m_alt.grow(ctx, n, 1024)) || (rc = ctx->m_cnt.grow(ctx, kMetWords, kMetWords)) ||
      (rc = ctx->c_cnt.grow(ctx, kCurWords, kCurWords)) || (rc = ctx->c_merged.grow(ctx, n, 1024)) ||
      (rc = ctx->c_excl.grow(ctx, n, 1024)) || (rc = ctx->c_thr.grow(ctx, n, 1024)) || (rc = ctx->c_tp.grow(ctx, n, 1024)) ||
      (rc = ctx->c_fp.grow(ctx, n, 1024)) || (rc = ctx->k_eval.grow(ctx, kCevWords, kCevWords)) ||
      (rc = ctx->i_hull.grow(ctx, 5 * (n + 1), 1024)) || (rc = ctx->i_out.grow(ctx, 2 * n, 1024)) ||
      (rc = ctx->i_blk.grow(ctx, 2 * n, 1024)) || (rc = ctx->i_ctl.grow(ctx, 1, 1)))
    return rc;
  size_t tmp = 0, tmp_merge = 0, tmp_scan = 0, tmp_iso = 0;
  cub::DoubleBuffer<unsigned long long> kb(ctx->m_keys.p, ctx->m_alt.p);
  CU(cub::DeviceRadixSort::SortKeys(nullptr, tmp, kb, (int)n, 0, 64, ctx->stream));
  CU(merge_runs(ctx, nullptr, tmp_merge, ctx->m_keys.p, n - n / 2, ctx->m_alt.p, n / 2));   // sized by the total
  CU(scan_tie_ends(ctx, nullptr, tmp_scan, n));
  CU(scan_x_counts(ctx, nullptr, tmp_iso, ctx->i_hull.p, (int)n, ctx->i_hull.p));
  return ctx->m_tmp.grow(ctx, (int64_t)std::max({tmp, tmp_merge, tmp_scan, tmp_iso}), 1 << 16);
}

static int fits_while_running(dsgd_ctx *ctx, bool fits, const char *fn) {
  NEED(fits || !ctx->a_running, DSGD_ERR_STATE,
       "%s: more ids than rows while the async loop runs (the buffers cannot grow until it is stopped)", fn);
  return DSGD_OK;
}

// the n row ids at the host address ids, into eval_ids; `preds`: the call also writes one value per id into preds
static int rows_list(dsgd_ctx *ctx, const int32_t *ids, int64_t n, bool preds, const char *fn, row_set *rows) {
  NEED(ctx->pairs, DSGD_ERR_STATE, "%s: no rows loaded", fn);
  NEED(n >= 0 && (n == 0 || ids), DSGD_ERR_INVALID, "%s: bad arguments", fn);
  NEED(n > 0, DSGD_ERR_EMPTY, "%s: empty sample (reduce on an empty collection throws)", fn);
  int rc = fits_while_running(ctx, ctx->eval_ids.cap >= n && (!preds || ctx->preds.cap >= n), fn);
  if (rc || (rc = check_ids(ctx, ids, n, fn, "sample index"))) return rc;
  CU(cudaSetDevice(ctx->device));
  if ((rc = ctx->eval_ids.grow(ctx, n, 1024))) return rc;
  CU(cudaMemcpyAsync(ctx->eval_ids, ids, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if (preds && (rc = ctx->preds.grow(ctx, n, 1024))) return rc;
  *rows = {ctx->eval_ids, 0, n};
  return DSGD_OK;
}

// The rows an evaluation's caller named, in one of its three forms: a range, a sample drawn from a range, or a host list of
// ids.  Each family's request function makes its checks once, then resolve_rows builds the row_set.
struct row_request {
  enum { kRange, kDrawn, kList } form;
  int64_t row_begin, row_end;
  uint64_t key;
  int64_t pos_begin, pos_end;
  const int32_t *ids;
  int64_t n;
};
static row_request range_rows(int64_t row_begin, int64_t row_end) {
  return {row_request::kRange, row_begin, row_end, 0, 0, 0, nullptr, 0};
}
static row_request drawn_rows(int64_t row_begin, int64_t row_end, uint64_t key, int64_t pos_begin, int64_t pos_end) {
  return {row_request::kDrawn, row_begin, row_end, key, pos_begin, pos_end, nullptr, 0};
}
static row_request listed_rows(const int32_t *ids, int64_t n) { return {row_request::kList, 0, 0, 0, 0, 0, ids, n}; }

static int resolve_rows(dsgd_ctx *ctx, const row_request &req, const char *fn, row_set *rows) {
  switch (req.form) {
    case row_request::kRange: return rows_range(ctx, req.row_begin, req.row_end, fn, rows);
    case row_request::kDrawn: return rows_drawn(ctx, req.row_begin, req.row_end, req.key, req.pos_begin, req.pos_end, fn, rows);
    default: return rows_list(ctx, req.ids, req.n, false, fn, rows);
  }
}

// the metrics, curve and calibration calls take a list of at most 2^31 - 1 ids; a range or a drawn sample passes
static int ids_capped(dsgd_ctx *ctx, const row_request &req, const char *fn) {
  NEED(req.form != row_request::kList || req.n <= (int64_t)INT32_MAX, DSGD_ERR_INVALID, "%s: %lld ids; at most 2^31 - 1", fn,
       (long long)req.n);
  return DSGD_OK;
}

// The row pass of model kModel and weighting kWeight over `rows` with the weights w: counters into cnt; kScatter: the
// gradient into g; kPreds: the SVM's sign predictions into preds.  w32 != nullptr (a request): an unweighted or
// class-weighted SVM pass over kStreamMinRows rows or more is the fp32 streaming pass, or its per-class form (SVM only: it
// decides signs, and the logistic loss needs the dot's value); every other pass is the fp64 k_rows of its model and
// weighting.  Only an evaluation names a range of rows; a gradient or a forward pass always lists them.  A weighted pass
// ends with its fold, k_class_fold or k_sw_fold: with out == nullptr the batch's weighted loss sum is left in cnt for a
// weighted tail (kCw), else the evaluation's totals and *nrm go to out.  kIcpt (an intercept ctx): never the streaming
// pass, which has no intercept form; k_rows reads the intercept at w[dim].
template <int kModel, int kWeight, bool kScatter, bool kPreds = false, bool kIcpt = false>
static int launch_rows(dsgd_ctx *ctx, const row_set &rows, const double *w, const float *w32, double *g,
                       double *preds = nullptr, const double *nrm = nullptr, double *out = nullptr) {
  bool streamed = false;
  if constexpr (kModel == kSvm && kWeight != kSampleWeighted && !kIcpt) {
    constexpr bool kCls = kWeight == kClassWeighted;
    if ((streamed = w32 && stream_eligible(ctx, rows.n))) {
      int rc = rows.ids ? stream_launch<kScatter, kPreds, false, kCls>(ctx, rows.ids, 0, rows.n, w, w32, g, preds)
                        : stream_launch<false, false, true, kCls>(ctx, nullptr, rows.row_begin, rows.n, w, w32, nullptr, nullptr);
      if (rc) return rc;
    }
  }
  if (!streamed) {
    // sw == nullptr without sample weights (an evaluation): every s_i is 1
    k_rows<kModel, kWeight, kScatter, kPreds, kIcpt><<<rows_grid(ctx, rows.n), 256, 0, ctx->stream>>>(
        ctx->rp16, ctx->pairs, ctx->label, rows.ids, rows.row_begin, rows.n, w, g, preds, ctx->cnt, ctx->cw_pos, ctx->cw_neg,
        ctx->sw_on ? ctx->sw.p : nullptr, icpt_of(ctx, w));
    LAUNCHED();
  }
  if constexpr (kWeight == kClassWeighted) {
    k_class_fold<kModel><<<1, 1, 0, ctx->stream>>>(ctx->cnt, ctx->cw_pos, ctx->cw_neg, nrm, out);
    LAUNCHED();
  } else if constexpr (kWeight == kSampleWeighted) {
    k_sw_fold<<<1, 1, 0, ctx->stream>>>(ctx->cnt, nrm, out);
    LAUNCHED();
  }
  return DSGD_OK;
}

// The pass of a gradient (kScatter: the gradient into g, then k_finish) or of an evaluation over `rows` with the weights of
// request_weights, then the shared tail: out2 = {loss, accuracy, loss sum, correct count, ||w||^2}, and the counters
// cleared for the next pass (k_loss_scalar).  A weighted gradient's tails read its weighted loss sum.
template <int kModel, int kWeight, bool kScatter, bool kIcpt>
static int loss_pass(dsgd_ctx *ctx, const double *w_host, const row_set &rows) {
  const double *w = nullptr, *c = nullptr, *nrm = nullptr;
  const float *w32 = nullptr;
  int rc = request_weights(ctx, w_host, &w, &c, &nrm, &w32);
  if (rc || (rc = launch_rows<kModel, kWeight, kScatter, false, kIcpt>(ctx, rows, w, w32, kScatter ? ctx->g.p : nullptr)))
    return rc;
  const double n = (double)rows.n;
  constexpr bool kCw = kWeight != kUnweighted;
  if constexpr (kScatter) {
    k_finish<kModel, kCw, kIcpt><<<cdiv(ctx->dim + 1, 256), 256, 0, ctx->stream>>>(ctx->g, ctx->dim, c, ctx->cnt, n);
    LAUNCHED();
  }
  k_loss_scalar<kModel, kCw><<<1, 1, 0, ctx->stream>>>(nrm, ctx->cnt, ctx->lambda, n, ctx->out2);
  LAUNCHED();
  CU(cudaGetLastError());
  return DSGD_OK;
}

extern "C" int dsgd_forward(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *preds_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n >= 0 && (n == 0 || (samples && preds_out)), DSGD_ERR_INVALID, "dsgd_forward: bad arguments");
  if (n == 0) return DSGD_OK;
  row_set rows;
  const double *wd, *cd, *nd;
  const float *w32d;
  int rc = rows_list(ctx, samples, n, true, __func__, &rows);
  if (rc || (rc = request_weights(ctx, w, &wd, &cd, &nd, &w32d))) return rc;
  // a prediction is the sign of the score under every model: the SVM's row kernels
  if ((rc = with_model<kUnweighted>(ctx, [&](auto, auto, auto ic) {
         return launch_rows<kSvm, kUnweighted, false, true, ic>(ctx, rows, wd, w32d, nullptr, ctx->preds);
       })))
    return rc;
  CU(cudaGetLastError());
  CU(cudaMemsetAsync(ctx->cnt, 0, sizeof(unsigned long long) * 2, ctx->stream));
  CU(cudaMemcpyAsync(preds_out, ctx->preds, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_gradient(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *grad_out,
                             double *loss_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n >= 0 && grad_out, DSGD_ERR_INVALID, "dsgd_gradient: bad arguments");
  NEED(n > 0, DSGD_ERR_EMPTY, "dsgd_gradient: empty batch (Vec.sum of an empty list throws in the reference)");
  NEED(samples, DSGD_ERR_INVALID, "dsgd_gradient: samples is NULL");
  NEED(ctx->have_d, DSGD_ERR_STATE, "dsgd_gradient: dimSparsity not set");
  row_set rows;
  int rc = rows_list(ctx, samples, n, false, __func__, &rows);
  if (rc || (rc = with_forms(ctx, weighting(ctx), [&](auto m, auto wt, auto ic) {
               return loss_pass<m, wt, true, ic>(ctx, w, rows);
             })))
    return rc;
  CU(cudaMemcpyAsync(grad_out, ctx->g, sizeof(double) * (size_t)ctx->dim, cudaMemcpyDeviceToHost, ctx->stream));
  if (has_icpt(ctx)) {   // the intercept's gradient, and its two sums cleared for the next pass
    CU(cudaMemcpyAsync(grad_out + ctx->dim, ctx->g + ctx->dim + kIcptSlot, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemsetAsync(ctx->g + ctx->dim + kIcptSlot, 0, sizeof(double), ctx->stream));
    CU(cudaMemsetAsync(ctx->cnt + kCntIcpt, 0, sizeof(unsigned long long) * 2 * kLossAccWords, ctx->stream));
  }
  double out2[2];
  CU(cudaMemcpyAsync(out2, ctx->out2, sizeof out2, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemsetAsync(ctx->g, 0, sizeof(double) * (size_t)(ctx->dim + 2), ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (loss_out) *loss_out = out2[0];
  return DSGD_OK;
}

// One evaluation pass over `rows`: out = {loss, accuracy, loss sum, correct count, ||w||^2}.  The SVM's loss sum is the
// hinge sum, an integer.
static int eval_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, double out[5]) {
  int rc = with_model<kUnweighted>(ctx, [&](auto m, auto wt, auto ic) { return loss_pass<m, wt, false, ic>(ctx, w, rows); });
  if (rc) return rc;
  CU(cudaMemcpyAsync(out, ctx->out2, sizeof(double) * 5, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

// The evaluation behind the *_counts and *_sums calls, and their outputs (NULL: not wanted): the loss sum as hinge_sum
// (*_counts) or as loss_sum (*_sums), the correct count and ||w||^2.
static int eval_sums(dsgd_ctx *ctx, const double *w, const row_set &rows, double *loss_sum, int64_t *hinge_sum,
                     int64_t *correct, double *norm_squared) {
  double out[5];
  int rc = eval_pass(ctx, w, rows, out);
  if (rc) return rc;
  if (loss_sum) *loss_sum = out[2];
  if (hinge_sum) *hinge_sum = (int64_t)out[2];
  if (correct) *correct = (int64_t)out[3];
  if (norm_squared) *norm_squared = out[4];
  return DSGD_OK;
}

// the *_counts calls report integer hinge sums, which only the SVM has
static const char kCountsNeedSvm[] = "%s: the %s model's loss sum is not an integer; use the *_sums call";

// dsgd_eval: the loss and the accuracy (NULL: not wanted)
static int eval_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, double *loss_out,
                        double *acc_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  row_set rows;
  double out[5];
  int rc = resolve_rows(ctx, req, fn, &rows);
  if (rc || (rc = eval_pass(ctx, w, rows, out))) return rc;
  if (loss_out) *loss_out = out[0];
  if (acc_out) *acc_out = out[1];
  return DSGD_OK;
}

// the *_counts (kCounts: the SVM's integer hinge sum) and *_sums calls
template <bool kCounts>
static int sums_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, double *loss_sum,
                        int64_t *hinge_sum, int64_t *correct, double *norm_squared) {
  if (!ctx) return DSGD_ERR_INVALID;
  if constexpr (kCounts) NEED(model_of(ctx) == kSvm, DSGD_ERR_STATE, kCountsNeedSvm, fn, kModelNames[model_of(ctx)]);
  row_set rows;
  int rc = resolve_rows(ctx, req, fn, &rows);
  return rc ? rc : eval_sums(ctx, w, rows, loss_sum, hinge_sum, correct, norm_squared);
}

extern "C" int dsgd_eval(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *loss_out,
                         double *acc_out) {
  return eval_request(ctx, w, range_rows(row_begin, row_end), __func__, loss_out, acc_out);
}

extern "C" int dsgd_eval_counts(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *hinge_sum,
                                int64_t *correct, double *norm_squared) {
  return sums_request<true>(ctx, w, range_rows(row_begin, row_end), __func__, nullptr, hinge_sum, correct, norm_squared);
}

extern "C" int dsgd_eval_sums(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *loss_sum,
                              int64_t *correct, double *norm_squared) {
  return sums_request<false>(ctx, w, range_rows(row_begin, row_end), __func__, loss_sum, nullptr, correct, norm_squared);
}

extern "C" int dsgd_eval_sampled_counts(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                        int64_t pos_begin, int64_t pos_end, int64_t *hinge_sum, int64_t *correct,
                                        double *norm_squared) {
  return sums_request<true>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, nullptr, hinge_sum,
                            correct, norm_squared);
}

extern "C" int dsgd_eval_sampled_sums(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                      int64_t pos_begin, int64_t pos_end, double *loss_sum, int64_t *correct,
                                      double *norm_squared) {
  return sums_request<false>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, loss_sum, nullptr,
                             correct, norm_squared);
}

extern "C" int dsgd_eval_samples_counts(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                        int64_t *hinge_sum, int64_t *correct, double *norm_squared) {
  return sums_request<true>(ctx, w, listed_rows(samples, n), __func__, nullptr, hinge_sum, correct, norm_squared);
}

extern "C" int dsgd_eval_samples_sums(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *loss_sum,
                                      int64_t *correct, double *norm_squared) {
  return sums_request<false>(ctx, w, listed_rows(samples, n), __func__, loss_sum, nullptr, correct, norm_squared);
}

// One evaluation pass of a weighted tally over `rows`: the row kernel without the scatter, then its fold into cls_out.
// dsgd_eval*_class (kClassWeighted): ||w||^2, the two loss sums, correct and rows per class.  dsgd_eval*_weighted
// (kSampleWeighted): ||w||^2, the three weighted sums and the correct count; without sample weights the pass reads no
// weights: every s_i is 1 and c_i = w_y.
template <int kWeight>
static int tally_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, double *norm_squared, double *sums,
                      int64_t *counts) {
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  const float *w32 = nullptr;
  int rc = request_weights(ctx, w, &wd, &cd, &nd, &w32);
  if (rc || (rc = with_model<kWeight>(ctx, [&](auto m, auto wt, auto ic) {
               return launch_rows<m, wt, false, false, ic>(ctx, rows, wd, w32, nullptr, nullptr, nd, ctx->cls_out);
             })))
    return rc;
  CU(cudaGetLastError());
  constexpr bool kCls = kWeight == kClassWeighted;
  double out[kCls ? 7 : 5];
  CU(cudaMemcpyAsync(out, ctx->cls_out, sizeof out, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (norm_squared) *norm_squared = out[0];
  if constexpr (kCls) {
    if (sums) { sums[0] = out[1]; sums[1] = out[2]; }
    if (counts)
      for (int k = 0; k < 4; ++k) counts[k] = (int64_t)out[3 + k];
  } else {
    if (sums)
      for (int k = 0; k < 3; ++k) sums[k] = out[1 + k];
    if (counts) { counts[0] = rows.n; counts[1] = (int64_t)out[4]; }
  }
  return DSGD_OK;
}

// dsgd_eval*_class (kClassWeighted) and dsgd_eval*_weighted (kSampleWeighted)
template <int kWeight>
static int tally_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, double *norm_squared,
                         double *sums_out, int64_t *counts_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  row_set rows;
  int rc = resolve_rows(ctx, req, fn, &rows);
  return rc ? rc : tally_pass<kWeight>(ctx, w, rows, norm_squared, sums_out, counts_out);
}

extern "C" int dsgd_eval_class(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *norm_squared,
                               double *loss_sums_out, int64_t *counts_out) {
  return tally_request<kClassWeighted>(ctx, w, range_rows(row_begin, row_end), __func__, norm_squared, loss_sums_out,
                                       counts_out);
}

extern "C" int dsgd_eval_sampled_class(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                       int64_t pos_begin, int64_t pos_end, double *norm_squared, double *loss_sums_out,
                                       int64_t *counts_out) {
  return tally_request<kClassWeighted>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__,
                                       norm_squared, loss_sums_out, counts_out);
}

extern "C" int dsgd_eval_samples_class(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                       double *norm_squared, double *loss_sums_out, int64_t *counts_out) {
  return tally_request<kClassWeighted>(ctx, w, listed_rows(samples, n), __func__, norm_squared, loss_sums_out, counts_out);
}

extern "C" int dsgd_eval_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *norm_squared,
                                  double *sums_out, int64_t *counts_out) {
  return tally_request<kSampleWeighted>(ctx, w, range_rows(row_begin, row_end), __func__, norm_squared, sums_out, counts_out);
}

extern "C" int dsgd_eval_sampled_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                          int64_t pos_begin, int64_t pos_end, double *norm_squared, double *sums_out,
                                          int64_t *counts_out) {
  return tally_request<kSampleWeighted>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__,
                                        norm_squared, sums_out, counts_out);
}

extern "C" int dsgd_eval_samples_weighted(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                          double *norm_squared, double *sums_out, int64_t *counts_out) {
  return tally_request<kSampleWeighted>(ctx, w, listed_rows(samples, n), __func__, norm_squared, sums_out, counts_out);
}

// ---- scores and ranking metrics (dsgd_metrics.cuh) ------------------------------------------------------------------

// out[i] = x . w (prob: the model's P(y = +1 | x), k_margins) of the listed rows; the values go through `preds`, the per-row
// request buffer.  On an intercept ctx the score is x . w + beta (k_margins<..., true>)
static int scores_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, double *out, bool prob) {
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = request_weights(ctx, w, &wd, &cd, &nd);
  if (rc) return rc;
  const bool huber = model_of(ctx) == kModifiedHuber;
  with_icpt(ctx, [&](auto ic) {
    auto kernel = !prob ? k_margins<false, false, ic> : huber ? k_margins<true, true, ic> : k_margins<true, false, ic>;
    kernel<<<rows_grid(ctx, rows.n), 256, 0, ctx->stream>>>(ctx->rp16, ctx->pairs, rows.ids, rows.n, wd, ctx->preds,
                                                           icpt_of(ctx, wd));
  });
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, ctx->preds, sizeof(double) * (size_t)rows.n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_margins(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *margins_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(margins_out, DSGD_ERR_INVALID, "%s: output is NULL", __func__);
  row_set rows;
  int rc = rows_list(ctx, samples, n, true, __func__, &rows);
  return rc ? rc : scores_pass(ctx, w, rows, margins_out, false);
}

extern "C" int dsgd_probabilities(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *probs_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(probs_out, DSGD_ERR_INVALID, "%s: output is NULL", __func__);
  const int m = model_of(ctx);
  NEED(m == kLogistic || m == kModifiedHuber, DSGD_ERR_STATE,
       m == kSvm ? "%s: probabilities need the SparseLogistic model (DSGD_FLAG_LOGISTIC)"
                 : "%s: the squared_hinge model has no probabilities; they need SparseLogistic (DSGD_FLAG_LOGISTIC) or "
                   "SparseModifiedHuber (DSGD_FLAG_MODIFIED_HUBER)",
       __func__);
  row_set rows;
  int rc = rows_list(ctx, samples, n, true, __func__, &rows);
  return rc ? rc : scores_pass(ctx, w, rows, probs_out, true);
}

// The first half of a metrics or a curve pass over `rows`: scores and counts (k_metrics_score), the words and the run
// lengths read by the host (the sort takes its lengths from the host), and the key runs sorted.  A metrics pass
// (`each_run` false) sorts only when both runs have keys, since otherwise there is no pair to count; a curve pass sorts
// every run that has keys.  Launches of the sort's own kernels are not counted in dsgd_launch_count.
// kSampleWeighted (a weighted curve pass): every key carries its row's c_i, the runs are sorted as (key, c) pairs, and
// pos_c / neg_c are the sorted weights.
struct sorted_runs {
  unsigned long long h[kMetWords];   // the counter words as k_metrics_score left them
  int64_t n_pos, n_neg;
  const unsigned long long *pos, *neg;   // each run ascending, if it was sorted
  const double *pos_c, *neg_c;           // kSampleWeighted: the weights in the order of pos and neg
};
template <int kWeight>
static int score_and_sort(dsgd_ctx *ctx, const double *w, const row_set &rows, bool each_run, const char *fn,
                          sorted_runs *s) {
  constexpr bool kW = kWeight == kSampleWeighted;
  constexpr int kWords = kW ? kMetWWords : kMetWords;
  const int64_t n = rows.n;
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = fits_while_running(ctx, ctx->m_keys.cap >= n && ctx->m_alt.cap >= n && ctx->m_cnt, fn);
  if (rc || (rc = request_weights(ctx, w, &wd, &cd, &nd))) return rc;
  if ((rc = ctx->m_keys.grow(ctx, n, 1024)) || (rc = ctx->m_alt.grow(ctx, n, 1024)) ||
      (rc = ctx->m_cnt.grow(ctx, kWords, kWords)))
    return rc;
  if (kW && ((rc = ctx->m_val.grow(ctx, n, 1024)) || (rc = ctx->m_valt.grow(ctx, n, 1024)))) return rc;
  CU(cudaMemsetAsync(ctx->m_cnt, 0, sizeof(unsigned long long) * kWords, ctx->stream));
  const int grid = (int)std::min<int64_t>(cdiv(n, 256), (int64_t)ctx->sm_count * 8);   // >= 32 rows per warp
  with_icpt(ctx, [&](auto ic) {
    k_metrics_score<kWeight, ic><<<grid, 256, 0, ctx->stream>>>(ctx->rp16, ctx->pairs, ctx->label, rows.ids, rows.row_begin, n,
                                                                wd, ctx->m_keys, ctx->m_cnt, ctx->cw_pos, ctx->cw_neg,
                                                                ctx->sw_on ? ctx->sw.p : nullptr, kW ? ctx->m_val.p : nullptr,
                                                                icpt_of(ctx, wd));
  });
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(s->h, ctx->m_cnt, sizeof s->h, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int64_t n_pos = (int64_t)s->h[kMetPosSlots], n_neg = (int64_t)s->h[kMetNegSlots];
  // the positives sit in keys[0, n_pos), the negatives in keys[n - n_neg, n); each run sorts within its own slice of the
  // two buffers, and Current() is the buffer that holds it sorted
  cub::DoubleBuffer<unsigned long long> kp(ctx->m_keys.p, ctx->m_alt.p);
  cub::DoubleBuffer<unsigned long long> kn(ctx->m_keys.p + (n - n_neg), ctx->m_alt.p + (n - n_neg));
  cub::DoubleBuffer<double> vp(ctx->m_val.p, ctx->m_valt.p);
  cub::DoubleBuffer<double> vn(kW ? ctx->m_val.p + (n - n_neg) : nullptr, kW ? ctx->m_valt.p + (n - n_neg) : nullptr);
  // one run sorted: its keys alone, or (kW) its (key, c) pairs
  auto sort = [&](void *tmp, size_t &bytes, cub::DoubleBuffer<unsigned long long> &k, cub::DoubleBuffer<double> &v, int64_t m) {
    if constexpr (kW) return cub::DeviceRadixSort::SortPairs(tmp, bytes, k, v, (int)m, 0, 64, ctx->stream);
    else return cub::DeviceRadixSort::SortKeys(tmp, bytes, k, (int)m, 0, 64, ctx->stream);
  };
  const bool sort_pos = n_pos > 0 && (each_run || n_neg > 0), sort_neg = n_neg > 0 && (each_run || n_pos > 0);
  if (sort_pos || sort_neg) {
    size_t tmp_p = 0, tmp_n = 0;
    if (sort_pos) CU(sort(nullptr, tmp_p, kp, vp, n_pos));
    if (sort_neg) CU(sort(nullptr, tmp_n, kn, vn, n_neg));
    size_t tmp = std::max(tmp_p, tmp_n);
    if ((rc = fits_while_running(ctx, ctx->m_tmp.cap >= (int64_t)tmp, fn)) || (rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16)))
      return rc;
    if (sort_pos) CU(sort(ctx->m_tmp.p, tmp, kp, vp, n_pos));
    if (sort_neg) CU(sort(ctx->m_tmp.p, tmp, kn, vn, n_neg));
  }
  s->n_pos = n_pos;
  s->n_neg = n_neg;
  s->pos = kp.Current();
  s->neg = kn.Current();
  s->pos_c = vp.Current();
  s->neg_c = vn.Current();
  return DSGD_OK;
}

// One metrics pass over `rows`: score_and_sort, then U2 counted (k_auc_count).
static int metrics_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, int64_t *out, const char *fn) {
  sorted_runs s;
  int rc = score_and_sort<kUnweighted>(ctx, w, rows, false, fn, &s);
  if (rc) return rc;
  unsigned long long *h = s.h;
  const int64_t n_pos = s.n_pos, n_neg = s.n_neg;
  if (n_pos > 0 && n_neg > 0) {   // else no pair: U2 = 0
    // Sorted positives let the threads of a warp walk nearly the same search path through the negatives.
    const int cgrid = (int)std::min<int64_t>(cdiv(n_pos, 256), (int64_t)ctx->sm_count * 8);
    k_auc_count<<<cgrid, 256, 0, ctx->stream>>>(s.pos, n_pos, s.neg, n_neg, ctx->m_cnt + kMetU2);
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&h[kMetU2], ctx->m_cnt + kMetU2, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  for (int k = 0; k < DSGD_METRICS_WORDS; ++k) out[k] = (int64_t)h[k];
  return DSGD_OK;
}

// The inclusive scan of R(c) over one sorted run's weights into pre (tmp == nullptr: the storage it needs, into bytes).
static cudaError_t scan_weights(dsgd_ctx *ctx, void *tmp, size_t &bytes, const double *c, limb_sum *pre, int64_t n) {
  return cub::DeviceScan::InclusiveScan(tmp, bytes, thrust::make_transform_iterator(c, limb_of{}), pre, limb_plus{}, (int)n,
                                        ctx->stream);
}

// One curve pass over `rows` (DESIGN.md §4.9): score_and_sort with every run sorted, then k_curve_count (U2, the limbs of
// S = sum of v_i, the number of points m) and k_curve_sum.  With thr != nullptr also the points: the runs merged, the
// exclusive scan of the merged keys' tie ends, k_curve_emit, and the m points copied back at once; `device_points` (an
// isotonic fit): the points are emitted into c_thr / c_tp / c_fp and stay there.  AP = S / P, NaN when a
// score is NaN or there is no positive row.
// runs_out: the sorted runs, for a caller that reads them after the pass.
// kSampleWeighted (§4.14): the same steps in their weighted forms, each run's prefix sums of R(c) scanned into c_pre before
// k_curve_count (positives at c_pre[0, n_pos), negatives after them); out receives the DSGD_WCURVE_WORDS words instead of
// AP, and tp / fp the point weights as doubles (k_curve_emit writes their bits into c_tp / c_fp).
template <int kWeight>
static int curve_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, int64_t *words, double *out, int64_t *n_points,
                      double *thr, void *tp, void *fp, const char *fn, bool device_points = false,
                      sorted_runs *runs_out = nullptr) {
  constexpr bool kW = kWeight == kSampleWeighted;
  constexpr int kWords = kW ? kCurWWords : kCurWords;
  const int64_t n = rows.n;
  const bool curve = thr != nullptr || device_points;
  int rc = fits_while_running(ctx, ctx->c_cnt && (!curve || (ctx->c_merged.cap >= n && ctx->c_excl.cap >= n &&
                                                              ctx->c_thr.cap >= n && ctx->c_tp.cap >= n && ctx->c_fp.cap >= n)),
                              fn);
  sorted_runs s;
  if (rc || (rc = score_and_sort<kWeight>(ctx, w, rows, true, fn, &s)) || (rc = ctx->c_cnt.grow(ctx, kWords, kWords))) return rc;
  CU(cudaMemsetAsync(ctx->c_cnt, 0, sizeof(unsigned long long) * kWords, ctx->stream));
  const int64_t n_all = s.n_pos + s.n_neg;
  const int grid = (int)std::min<int64_t>(std::max(cdiv(n_all, 256), 1), (int64_t)ctx->sm_count * 8);
  const limb_sum *pre_pos = nullptr, *pre_neg = nullptr;
  if constexpr (kW) {
    if ((rc = ctx->c_pre.grow(ctx, n, 1024))) return rc;
    pre_pos = ctx->c_pre.p;
    pre_neg = ctx->c_pre.p + s.n_pos;
    size_t tmp_p = 0, tmp_n = 0;
    if (s.n_pos) CU(scan_weights(ctx, nullptr, tmp_p, s.pos_c, ctx->c_pre.p, s.n_pos));
    if (s.n_neg) CU(scan_weights(ctx, nullptr, tmp_n, s.neg_c, ctx->c_pre.p + s.n_pos, s.n_neg));
    size_t tmp = std::max(tmp_p, tmp_n);
    if ((rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16))) return rc;
    if (s.n_pos) CU(scan_weights(ctx, ctx->m_tmp.p, tmp, s.pos_c, ctx->c_pre.p, s.n_pos));
    if (s.n_neg) CU(scan_weights(ctx, ctx->m_tmp.p, tmp, s.neg_c, ctx->c_pre.p + s.n_pos, s.n_neg));
    k_curve_count<kWeight><<<grid, 256, 0, ctx->stream>>>(s.pos, s.n_pos, s.neg, s.n_neg, ctx->m_cnt + kMetU2, ctx->c_cnt,
                                                          s.pos_c, pre_pos, pre_neg);
    LAUNCHED();
    k_curve_sum<kWeight><<<1, 1, 0, ctx->stream>>>(ctx->c_cnt, s.pos, s.n_pos, s.neg, s.n_neg, pre_pos, pre_neg, ctx->m_cnt);
    LAUNCHED();
  } else {
    k_curve_count<kWeight><<<grid, 256, 0, ctx->stream>>>(s.pos, s.n_pos, s.neg, s.n_neg, ctx->m_cnt + kMetU2, ctx->c_cnt);
    LAUNCHED();
    k_curve_sum<kWeight><<<1, 1, 0, ctx->stream>>>(ctx->c_cnt);
    LAUNCHED();
  }
  CU(cudaGetLastError());
  if (curve && n_all > 0) {
    if ((rc = ctx->c_merged.grow(ctx, n, 1024)) || (rc = ctx->c_excl.grow(ctx, n, 1024)) || (rc = ctx->c_thr.grow(ctx, n, 1024)) ||
        (rc = ctx->c_tp.grow(ctx, n, 1024)) || (rc = ctx->c_fp.grow(ctx, n, 1024)))
      return rc;
    size_t tmp_merge = 0, tmp_scan = 0;
    CU(merge_runs(ctx, nullptr, tmp_merge, s.pos, s.n_pos, s.neg, s.n_neg));
    CU(scan_tie_ends(ctx, nullptr, tmp_scan, n_all));
    size_t tmp = std::max(tmp_merge, tmp_scan);
    if ((rc = fits_while_running(ctx, ctx->m_tmp.cap >= (int64_t)tmp, fn)) || (rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16)))
      return rc;
    CU(merge_runs(ctx, ctx->m_tmp.p, tmp, s.pos, s.n_pos, s.neg, s.n_neg));
    tmp = std::max(tmp_merge, tmp_scan);
    CU(scan_tie_ends(ctx, ctx->m_tmp.p, tmp, n_all));
    if constexpr (kW)
      k_curve_emit<kWeight><<<grid, 256, 0, ctx->stream>>>(ctx->c_merged, n_all, ctx->c_excl, s.pos, s.n_pos, s.neg, s.n_neg,
                                                           ctx->c_cnt, ctx->c_thr, ctx->c_tp, ctx->c_fp, pre_pos, pre_neg);
    else
      k_curve_emit<kWeight><<<grid, 256, 0, ctx->stream>>>(ctx->c_merged, n_all, ctx->c_excl, s.pos, s.n_pos, s.neg, s.n_neg,
                                                           ctx->c_cnt, ctx->c_thr, ctx->c_tp, ctx->c_fp);
    LAUNCHED();
    CU(cudaGetLastError());
  }
  unsigned long long c[kWords];
  CU(cudaMemcpyAsync(c, ctx->c_cnt, sizeof c, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(&s.h[kMetU2], ctx->m_cnt + kMetU2, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int64_t m = (int64_t)c[kCurPoints];
  if (thr && m > 0) {   // a weighted pass's c_tp / c_fp hold the bits of doubles: copied as bytes
    CU(cudaMemcpyAsync(thr, ctx->c_thr, sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(tp, ctx->c_tp, sizeof(int64_t) * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(fp, ctx->c_fp, sizeof(int64_t) * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  for (int k = 0; k < DSGD_METRICS_WORDS; ++k) words[k] = (int64_t)s.h[k];
  if constexpr (kW) {
    memcpy(out, &c[kCurOut], sizeof(double) * DSGD_WCURVE_WORDS);
  } else {
    const int64_t P = words[kMetTp] + words[kMetFn] + words[kMetPosNone];
    double S;
    memcpy(&S, &c[kCurSum], sizeof S);
    *out = (words[kMetNan] > 0 || P == 0) ? std::numeric_limits<double>::quiet_NaN() : S / (double)P;
  }
  if (runs_out) *runs_out = s;   // a weighted isotonic fit reads the sorted runs and their prefix sums
  *n_points = m;
  return DSGD_OK;
}

// the outputs of a curve call: words, ap and the point count always; the three point arrays all or none
static int curve_outputs(dsgd_ctx *ctx, const int64_t *words, const double *ap, const int64_t *n_points, const double *thr,
                         const int64_t *tp, const int64_t *fp, const char *fn) {
  NEED(words && ap && n_points, DSGD_ERR_INVALID, "%s: words_out, ap_out or n_points_out is NULL", fn);
  NEED(!thr == !tp && !tp == !fp, DSGD_ERR_INVALID,
       "%s: thr_out, tp_out and fp_out are all NULL (average precision only) or all set", fn);
  return DSGD_OK;
}

// A weighted curve call: the outputs as curve_outputs checks them (wsums_out in ap_out's place, tpw / fpw in tp / fp's), then
// an async ctx is refused before anything is launched -- its weights are always 1, and growing the pass's buffers would wait
// for the loop, which runs until stopped.
static int weighted_curve_args(dsgd_ctx *ctx, const int64_t *words, const double *wsums, const int64_t *n_points,
                               const double *thr, const double *tpw, const double *fpw, const char *fn) {
  NEED(words && wsums && n_points, DSGD_ERR_INVALID, "%s: words_out, wsums_out or n_points_out is NULL", fn);
  NEED(!thr == !tpw && !tpw == !fpw, DSGD_ERR_INVALID,
       "%s: thr_out, tpw_out and fpw_out are all NULL (the words only) or all set", fn);
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (row weights belong to the sync paths)",
       fn);
  return DSGD_OK;
}

// dsgd_eval*_curve (kUnweighted: AP into out, the point counts into tp / fp) and dsgd_eval*_weighted_curve (kSampleWeighted:
// the DSGD_WCURVE_WORDS sums into out, the point weights into tp / fp)
template <int kWeight, class P>
static int curve_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, int64_t *words, double *out,
                         int64_t *n_points, double *thr, P *tp, P *fp) {
  if (!ctx) return DSGD_ERR_INVALID;
  int rc;
  if constexpr (kWeight == kSampleWeighted) rc = weighted_curve_args(ctx, words, out, n_points, thr, tp, fp, fn);
  else rc = curve_outputs(ctx, words, out, n_points, thr, tp, fp, fn);
  row_set rows;
  if (rc || (rc = ids_capped(ctx, req, fn)) || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  return curve_pass<kWeight>(ctx, w, rows, words, out, n_points, thr, tp, fp, fn);
}

extern "C" int dsgd_eval_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *words_out,
                               double *ap_out, int64_t *n_points_out, double *thr_out, int64_t *tp_out, int64_t *fp_out) {
  return curve_request<kUnweighted>(ctx, w, range_rows(row_begin, row_end), __func__, words_out, ap_out, n_points_out, thr_out,
                                    tp_out, fp_out);
}

extern "C" int dsgd_eval_sampled_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                       int64_t pos_begin, int64_t pos_end, int64_t *words_out, double *ap_out,
                                       int64_t *n_points_out, double *thr_out, int64_t *tp_out, int64_t *fp_out) {
  return curve_request<kUnweighted>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, words_out,
                                    ap_out, n_points_out, thr_out, tp_out, fp_out);
}

extern "C" int dsgd_eval_samples_curve(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *words_out,
                                       double *ap_out, int64_t *n_points_out, double *thr_out, int64_t *tp_out,
                                       int64_t *fp_out) {
  return curve_request<kUnweighted>(ctx, w, listed_rows(samples, n), __func__, words_out, ap_out, n_points_out, thr_out,
                                    tp_out, fp_out);
}

extern "C" int dsgd_eval_weighted_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                        int64_t *words_out, double *wsums_out, int64_t *n_points_out, double *thr_out,
                                        double *tpw_out, double *fpw_out) {
  return curve_request<kSampleWeighted>(ctx, w, range_rows(row_begin, row_end), __func__, words_out, wsums_out, n_points_out,
                                        thr_out, tpw_out, fpw_out);
}

extern "C" int dsgd_eval_sampled_weighted_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                uint64_t key, int64_t pos_begin, int64_t pos_end, int64_t *words_out,
                                                double *wsums_out, int64_t *n_points_out, double *thr_out, double *tpw_out,
                                                double *fpw_out) {
  return curve_request<kSampleWeighted>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, words_out,
                                        wsums_out, n_points_out, thr_out, tpw_out, fpw_out);
}

extern "C" int dsgd_eval_samples_weighted_curve(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                                int64_t *words_out, double *wsums_out, int64_t *n_points_out,
                                                double *thr_out, double *tpw_out, double *fpw_out) {
  return curve_request<kSampleWeighted>(ctx, w, listed_rows(samples, n), __func__, words_out, wsums_out, n_points_out,
                                        thr_out, tpw_out, fpw_out);
}

static int metrics_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, int64_t *out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(out, DSGD_ERR_INVALID, "%s: out is NULL", fn);
  row_set rows;
  int rc = ids_capped(ctx, req, fn);
  if (rc || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  return metrics_pass(ctx, w, rows, out, fn);
}

extern "C" int dsgd_eval_metrics(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *out) {
  return metrics_request(ctx, w, range_rows(row_begin, row_end), __func__, out);
}

extern "C" int dsgd_eval_sampled_metrics(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                         int64_t pos_begin, int64_t pos_end, int64_t *out) {
  return metrics_request(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, out);
}

extern "C" int dsgd_eval_samples_metrics(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *out) {
  return metrics_request(ctx, w, listed_rows(samples, n), __func__, out);
}

// ---- topics (dsgd_topics.cuh; DESIGN.md §4.21) --------------------------------------------------------------------------

// the loaded labels back in ctx->label, and yabs's signs with them
static int restore_labels(dsgd_ctx *ctx) {
  k_topic_select<<<cdiv(ctx->n_rows, 256), 256, 0, ctx->stream>>>(ctx->t_ptr, ctx->t_ids, ctx->label0, ctx->n_rows, -1,
                                                                   ctx->label, ctx->yabs);
  LAUNCHED();
  CU(cudaGetLastError());
  return DSGD_OK;
}

extern "C" int dsgd_load_topics(dsgd_ctx *ctx, int32_t n_topics, const int64_t *topic_ptr, const int32_t *topic_id) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "dsgd_load_topics: ctx is in async mode (topics belong to the sync paths)");
  NEED(ctx->pairs, DSGD_ERR_STATE, "dsgd_load_topics: no rows loaded");
  NEED(n_topics >= 1 && n_topics <= DSGD_MAX_TOPICS, DSGD_ERR_INVALID, "dsgd_load_topics: %d topics; 1 .. %d", n_topics,
       DSGD_MAX_TOPICS);
  NEED(topic_ptr, DSGD_ERR_INVALID, "dsgd_load_topics: topic_ptr is NULL");
  const int64_t n = ctx->n_rows;
  NEED(topic_ptr[0] == 0, DSGD_ERR_INVALID, "dsgd_load_topics: topic_ptr[0] is %lld, not 0", (long long)topic_ptr[0]);
  for (int64_t r = 0; r < n; ++r)
    NEED(topic_ptr[r + 1] >= topic_ptr[r], DSGD_ERR_INVALID, "dsgd_load_topics: topic_ptr not monotone at row %lld",
         (long long)r);
  const int64_t nnz = topic_ptr[n];   // the id count
  NEED(nnz == 0 || topic_id, DSGD_ERR_INVALID, "dsgd_load_topics: topic_id is NULL with %lld ids", (long long)nnz);
  for (int64_t r = 0; r < n; ++r)
    for (int64_t k = topic_ptr[r]; k < topic_ptr[r + 1]; ++k) {
      NEED(topic_id[k] >= 0 && topic_id[k] < n_topics, DSGD_ERR_INVALID,
           "dsgd_load_topics: topic %d of row %lld outside [0,%d)", topic_id[k], (long long)r, n_topics);
      NEED(k == topic_ptr[r] || topic_id[k] > topic_id[k - 1], DSGD_ERR_INVALID,
           "dsgd_load_topics: the topics of row %lld are not strictly ascending at position %lld", (long long)r, (long long)k);
    }
  CU(cudaSetDevice(ctx->device));
  int rc;
  if (ctx->n_topics > 0) {   // a topic may be selected: the loaded labels go back first, and label0 keeps them
    if ((rc = restore_labels(ctx))) return rc;
  } else {
    CU(ctx->label0.alloc(n));
    CU(cudaMemcpyAsync(ctx->label0, ctx->label, (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  ctx->n_topics = 0;
  CU(ctx->t_ptr.alloc(n + 1));
  CU(ctx->t_ids.alloc(std::max<int64_t>(nnz, 1)));
  CU(cudaMemcpyAsync(ctx->t_ptr, topic_ptr, sizeof(int64_t) * (size_t)(n + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (nnz) CU(cudaMemcpyAsync(ctx->t_ids, topic_id, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->n_topics = n_topics;
  return DSGD_OK;
}

extern "C" int dsgd_select_topic(dsgd_ctx *ctx, int32_t topic) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE,
       "dsgd_select_topic: ctx is in async mode (the labels would change under the Hogwild loop)");
  NEED(ctx->n_topics > 0, DSGD_ERR_STATE, "dsgd_select_topic: no topics loaded");
  NEED(topic >= -1 && topic < ctx->n_topics, DSGD_ERR_INVALID, "dsgd_select_topic: topic %d outside [-1,%d)", topic,
       ctx->n_topics);
  CU(cudaSetDevice(ctx->device));
  k_topic_select<<<cdiv(ctx->n_rows, 256), 256, 0, ctx->stream>>>(ctx->t_ptr, ctx->t_ids, ctx->label0, ctx->n_rows, topic,
                                                                   ctx->label, ctx->yabs);
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

// the T weight vectors W on the device (ctx->t_w)
static int topic_weights_in(dsgd_ctx *ctx, const double *W, int32_t n_topics) {
  const int64_t nw = (int64_t)n_topics * wlen(ctx);
  int rc = ctx->t_w.grow(ctx, nw, 1024);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->t_w, W, sizeof(double) * (size_t)nw, cudaMemcpyHostToDevice, ctx->stream));
  return DSGD_OK;
}

// dsgd_eval*_topics (thresholded false) and dsgd_eval*_thresholded_topics (thresholded: the caller's T thresholds thr): the
// DSGD_TOPIC_WORDS(T) words into out.  Every refusal comes before anything is launched.
static int topics_request(dsgd_ctx *ctx, const double *W, int32_t n_topics, bool thresholded, const double *thr,
                          const row_request &req, const char *fn, int64_t *out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(out, DSGD_ERR_INVALID, "%s: out is NULL", fn);
  NEED(W, DSGD_ERR_INVALID, "%s: W is NULL (the call scores T weight vectors of the caller's)", fn);
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (topics belong to the sync paths)", fn);
  NEED(ctx->n_topics > 0, DSGD_ERR_STATE, "%s: no topics loaded", fn);
  NEED(n_topics == ctx->n_topics, DSGD_ERR_INVALID, "%s: %d weight vectors for %d loaded topics", fn, n_topics,
       ctx->n_topics);
  if (thresholded) {
    NEED(thr, DSGD_ERR_INVALID, "%s: thresholds is NULL", fn);
    for (int32_t t = 0; t < n_topics; ++t)
      NEED(!std::isnan(thr[t]), DSGD_ERR_INVALID, "%s: the threshold of topic %d is NaN", fn, t);
  }
  row_set rows;
  int rc = ids_capped(ctx, req, fn);
  if (rc || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  const int64_t T = n_topics, words = DSGD_TOPIC_WORDS(T);
  if ((rc = topic_weights_in(ctx, W, n_topics)) || (rc = ctx->t_cnt.grow(ctx, words, 1024)) ||
      (thresholded && (rc = ctx->u_thr.grow(ctx, T, 1024))))
    return rc;
  CU(cudaMemsetAsync(ctx->t_cnt, 0, sizeof(unsigned long long) * (size_t)words, ctx->stream));
  if (thresholded) CU(cudaMemcpyAsync(ctx->u_thr, thr, sizeof(double) * (size_t)T, cudaMemcpyHostToDevice, ctx->stream));
  const int grid = (int)std::min<int64_t>(cdiv(rows.n, 256), (int64_t)ctx->sm_count * 8);   // >= 32 rows per warp
  const size_t smem = sizeof(unsigned) * (size_t)(T * kTopicWords);
  with_icpt(ctx, [&](auto ic) {
    if (thresholded)
      k_topic_eval<ic, true><<<grid, 256, smem, ctx->stream>>>(ctx->rp16, ctx->pairs, ctx->t_ptr, ctx->t_ids, rows.ids,
                                                               rows.row_begin, rows.n, ctx->t_w, n_topics, ctx->dim,
                                                               ctx->t_cnt, ctx->u_thr);
    else
      k_topic_eval<ic><<<grid, 256, smem, ctx->stream>>>(ctx->rp16, ctx->pairs, ctx->t_ptr, ctx->t_ids, rows.ids,
                                                         rows.row_begin, rows.n, ctx->t_w, n_topics, ctx->dim, ctx->t_cnt);
  });
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, ctx->t_cnt, sizeof(int64_t) * (size_t)words, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_eval_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, int64_t row_begin, int64_t row_end,
                                int64_t *out) {
  return topics_request(ctx, W, n_topics, false, nullptr, range_rows(row_begin, row_end), __func__, out);
}

extern "C" int dsgd_eval_sampled_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, int64_t row_begin, int64_t row_end,
                                        uint64_t key, int64_t pos_begin, int64_t pos_end, int64_t *out) {
  return topics_request(ctx, W, n_topics, false, nullptr, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__,
                        out);
}

extern "C" int dsgd_eval_samples_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, const int32_t *samples, int64_t n,
                                        int64_t *out) {
  return topics_request(ctx, W, n_topics, false, nullptr, listed_rows(samples, n), __func__, out);
}

extern "C" int dsgd_eval_thresholded_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, const double *thresholds,
                                            int64_t row_begin, int64_t row_end, int64_t *out) {
  return topics_request(ctx, W, n_topics, true, thresholds, range_rows(row_begin, row_end), __func__, out);
}

extern "C" int dsgd_eval_sampled_thresholded_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics,
                                                    const double *thresholds, int64_t row_begin, int64_t row_end,
                                                    uint64_t key, int64_t pos_begin, int64_t pos_end, int64_t *out) {
  return topics_request(ctx, W, n_topics, true, thresholds, drawn_rows(row_begin, row_end, key, pos_begin, pos_end),
                        __func__, out);
}

extern "C" int dsgd_eval_samples_thresholded_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics,
                                                    const double *thresholds, const int32_t *samples, int64_t n,
                                                    int64_t *out) {
  return topics_request(ctx, W, n_topics, true, thresholds, listed_rows(samples, n), __func__, out);
}

// ---- topic threshold tuning (dsgd_topics.cuh: k_topic_keys, k_topic_tune; DESIGN.md §4.23) -------------------------------

static_assert(kTopicWords == 8 && kTuCand == 7, "DSGD_TOPIC_TUNE_WORDS layout");

constexpr int64_t kTuneKeys = 1ll << 27;   // keys per group: G = max(1, min(T, kTuneKeys / n)) topics of n positions

// the start of sorted segment s: segments of n keys each
struct tune_segment {
  int64_t n;
  __host__ __device__ int operator()(int s) const { return (int)(s * n); }
};

// dsgd_tune_topic_thresholds*: the T thresholds into thr_out and the DSGD_TOPIC_TUNE_WORDS(T) words into words_out, the
// topics scored, sorted and scanned in groups of G.  Every refusal comes before anything is launched or grown.
static int tune_request(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr, const row_request &req,
                        const char *fn, double *thr_out, int64_t *words_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(thr_out && words_out, DSGD_ERR_INVALID, "%s: an output is NULL", fn);
  NEED(W, DSGD_ERR_INVALID, "%s: W is NULL (the call tunes T weight vectors of the caller's)", fn);
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (topics belong to the sync paths)", fn);
  NEED(ctx->n_topics > 0, DSGD_ERR_STATE, "%s: no topics loaded", fn);
  NEED(n_topics == ctx->n_topics, DSGD_ERR_INVALID, "%s: %d weight vectors for %d loaded topics", fn, n_topics,
       ctx->n_topics);
  NEED(fbr >= 0.0 && fbr <= 1.0, DSGD_ERR_INVALID, "%s: fbr = %g; 0 .. 1", fn, fbr);
  row_set rows;
  int rc = ids_capped(ctx, req, fn);
  if (rc || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  const int64_t n = rows.n, T = n_topics, G = std::max<int64_t>(1, std::min<int64_t>(T, kTuneKeys / n));
  if ((rc = topic_weights_in(ctx, W, n_topics)) || (rc = ctx->u_keys.grow(ctx, G * n, 1024)) ||
      (rc = ctx->u_alt.grow(ctx, G * n, 1024)) || (rc = ctx->u_has.grow(ctx, G * n, 1024)) ||
      (rc = ctx->u_hasalt.grow(ctx, G * n, 1024)) || (rc = ctx->u_thr.grow(ctx, T, 1024)) ||
      (rc = ctx->u_words.grow(ctx, 8 * T, 1024)))
    return rc;
  const int grid = (int)std::min<int64_t>(cdiv(n, 256), (int64_t)ctx->sm_count * 8);   // >= 32 rows per warp
  const auto seg = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), tune_segment{n});
  for (int64_t t0 = 0; t0 < T; t0 += G) {
    const int64_t g = std::min(G, T - t0);
    with_icpt(ctx, [&](auto ic) {
      k_topic_keys<ic><<<grid, 256, 0, ctx->stream>>>(ctx->rp16, ctx->pairs, ctx->t_ptr, ctx->t_ids, rows.ids,
                                                      rows.row_begin, n, ctx->t_w, (int32_t)t0, (int32_t)g, ctx->dim,
                                                      ctx->u_keys, ctx->u_has);
    });
    LAUNCHED();
    CU(cudaGetLastError());
    cub::DoubleBuffer<unsigned long long> kb(ctx->u_keys.p, ctx->u_alt.p);
    cub::DoubleBuffer<uint8_t> hb(ctx->u_has.p, ctx->u_hasalt.p);
    size_t tmp = 0;
    CU(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, tmp, kb, hb, (int)(g * n), (int)g, seg, seg + 1, 0, 64,
                                                ctx->stream));
    if ((rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16))) return rc;
    CU(cub::DeviceSegmentedRadixSort::SortPairs(ctx->m_tmp.p, tmp, kb, hb, (int)(g * n), (int)g, seg, seg + 1, 0, 64,
                                                ctx->stream));
    LAUNCHED();
    k_topic_tune<<<(int)g, kTuneThreads, 0, ctx->stream>>>(kb.Current(), hb.Current(), n, (int32_t)t0, fbr, ctx->u_thr,
                                                          ctx->u_words);
    LAUNCHED();
    CU(cudaGetLastError());
  }
  CU(cudaMemcpyAsync(thr_out, ctx->u_thr, sizeof(double) * (size_t)T, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(words_out, ctx->u_words, sizeof(int64_t) * (size_t)(8 * T), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_tune_topic_thresholds(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr, int64_t row_begin,
                                          int64_t row_end, double *thresholds_out, int64_t *words_out) {
  return tune_request(ctx, W, n_topics, fbr, range_rows(row_begin, row_end), __func__, thresholds_out, words_out);
}

extern "C" int dsgd_tune_topic_thresholds_sampled(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr,
                                                  int64_t row_begin, int64_t row_end, uint64_t key, int64_t pos_begin,
                                                  int64_t pos_end, double *thresholds_out, int64_t *words_out) {
  return tune_request(ctx, W, n_topics, fbr, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__,
                      thresholds_out, words_out);
}

extern "C" int dsgd_tune_topic_thresholds_samples(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr,
                                                  const int32_t *samples, int64_t n, double *thresholds_out,
                                                  int64_t *words_out) {
  return tune_request(ctx, W, n_topics, fbr, listed_rows(samples, n), __func__, thresholds_out, words_out);
}

// ---- topic ranking (dsgd_topics.cuh: k_topic_rank; DESIGN.md §4.22) ----------------------------------------------------

static double fixed_read(const unsigned long long *limbs, unsigned long long ovf);   // with the calibration calls, below

static_assert(kRankMaxK == DSGD_TOPIC_RANK_MAX_K && kRankWords == 8 && kLossAccWords == 7, "DSGD_TOPIC_RANK_WORDS layout");

// k_topic_rank's grid for n rows: at least 32 rows per warp
static int rank_grid(const dsgd_ctx *ctx, int64_t n) {
  return (int)std::min<int64_t>(cdiv(n, 32 * kRankWarps), (int64_t)ctx->sm_count * 16);
}

// dsgd_eval*_topic_ranking: the DSGD_TOPIC_RANK_WORDS(k) words into words_out and the 2 + k sums into sums_out.  The limb
// words leave with their carries propagated (limbs 0..4 in [0, 2^40)) and each sum is fixed_read of its block, acc_value's
// conversion.  Every refusal comes before anything is launched.
static int topic_ranking_request(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, const row_request &req,
                                 const char *fn, int64_t *words_out, double *sums_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(words_out && sums_out, DSGD_ERR_INVALID, "%s: an output is NULL", fn);
  NEED(W, DSGD_ERR_INVALID, "%s: W is NULL (the call ranks by T weight vectors of the caller's)", fn);
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (topics belong to the sync paths)", fn);
  NEED(ctx->n_topics > 0, DSGD_ERR_STATE, "%s: no topics loaded", fn);
  NEED(n_topics == ctx->n_topics, DSGD_ERR_INVALID, "%s: %d weight vectors for %d loaded topics", fn, n_topics,
       ctx->n_topics);
  NEED(k >= 1 && k <= std::min(n_topics, (int32_t)DSGD_TOPIC_RANK_MAX_K), DSGD_ERR_INVALID, "%s: k = %d; 1 .. min(T, %d)",
       fn, k, DSGD_TOPIC_RANK_MAX_K);
  row_set rows;
  int rc = ids_capped(ctx, req, fn);
  if (rc || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  const int64_t words = DSGD_TOPIC_RANK_WORDS(k);
  if ((rc = topic_weights_in(ctx, W, n_topics)) || (rc = ctx->t_rank.grow(ctx, words, 1024))) return rc;
  CU(cudaMemsetAsync(ctx->t_rank, 0, sizeof(unsigned long long) * (size_t)words, ctx->stream));
  const size_t smem = sizeof(double) * (size_t)kRankWarps * (size_t)n_topics;
  with_icpt(ctx, [&](auto ic) {
    k_topic_rank<ic, false><<<rank_grid(ctx, rows.n), 32 * kRankWarps, smem, ctx->stream>>>(
        ctx->rp16, ctx->pairs, ctx->t_ptr, ctx->t_ids, rows.ids, rows.row_begin, rows.n, ctx->t_w, n_topics, ctx->dim, k,
        ctx->t_rank, nullptr, nullptr);
  });
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(words_out, ctx->t_rank, sizeof(int64_t) * (size_t)words, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < 2 + k; ++s) {
    unsigned long long *q = (unsigned long long *)words_out + kRankWords + k + (int64_t)s * kLossAccWords;
    for (int i = 0; i < kLossLimbs - 1; ++i) {
      q[i + 1] += q[i] >> 40;
      q[i] &= kLimbMask;
    }
    sums_out[s] = fixed_read(q, q[kLossLimbs]);
  }
  return DSGD_OK;
}

extern "C" int dsgd_eval_topic_ranking(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, int64_t row_begin,
                                       int64_t row_end, int64_t *words_out, double *sums_out) {
  return topic_ranking_request(ctx, W, n_topics, k, range_rows(row_begin, row_end), __func__, words_out, sums_out);
}

extern "C" int dsgd_eval_sampled_topic_ranking(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, int64_t row_begin,
                                               int64_t row_end, uint64_t key, int64_t pos_begin, int64_t pos_end,
                                               int64_t *words_out, double *sums_out) {
  return topic_ranking_request(ctx, W, n_topics, k, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__,
                               words_out, sums_out);
}

extern "C" int dsgd_eval_samples_topic_ranking(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k,
                                               const int32_t *samples, int64_t n, int64_t *words_out, double *sums_out) {
  return topic_ranking_request(ctx, W, n_topics, k, listed_rows(samples, n), __func__, words_out, sums_out);
}

extern "C" int dsgd_topics_topk(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, const int32_t *samples, int64_t n,
                                int32_t *ids_out, double *margins_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(W && ids_out && margins_out, DSGD_ERR_INVALID, "%s: W or an output is NULL", __func__);
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (topics belong to the sync paths)",
       __func__);
  NEED(n_topics >= 1 && n_topics <= DSGD_MAX_TOPICS, DSGD_ERR_INVALID, "%s: %d topics; 1 .. %d", __func__, n_topics,
       DSGD_MAX_TOPICS);
  NEED(k >= 1 && k <= std::min(n_topics, (int32_t)DSGD_TOPIC_RANK_MAX_K), DSGD_ERR_INVALID, "%s: k = %d; 1 .. min(T, %d)",
       __func__, k, DSGD_TOPIC_RANK_MAX_K);
  NEED(n <= (int64_t)INT32_MAX, DSGD_ERR_INVALID, "%s: %lld ids; at most 2^31 - 1", __func__, (long long)n);
  row_set rows;
  int rc = rows_list(ctx, samples, n, false, __func__, &rows);
  if (rc) return rc;
  const int64_t nk = n * k;
  if ((rc = topic_weights_in(ctx, W, n_topics)) || (rc = ctx->t_top_ids.grow(ctx, nk, 1024)) ||
      (rc = ctx->t_top_m.grow(ctx, nk, 1024)))
    return rc;
  const size_t smem = sizeof(double) * (size_t)kRankWarps * (size_t)n_topics;
  with_icpt(ctx, [&](auto ic) {
    k_topic_rank<ic, true><<<rank_grid(ctx, rows.n), 32 * kRankWarps, smem, ctx->stream>>>(
        ctx->rp16, ctx->pairs, nullptr, nullptr, rows.ids, rows.row_begin, rows.n, ctx->t_w, n_topics, ctx->dim, k, nullptr,
        ctx->t_top_ids, ctx->t_top_m);
  });
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(ids_out, ctx->t_top_ids, sizeof(int32_t) * (size_t)nk, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(margins_out, ctx->t_top_m, sizeof(double) * (size_t)nk, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

// ---- bootstrap (dsgd_bootstrap.cuh; DESIGN.md §4.19) --------------------------------------------------------------------

constexpr int64_t kBootChunk = 4096;   // replicates per k_boot_rep launch: its output block stays small whatever n_boot is

// The part of a bootstrap pass that does not depend on the replicate: every position of `rows` scored (k_boot_score, with
// the losses by position in b_loss for every model but the SVM) and the (key, tag) pairs sorted; *kb / *tb hold the sorted
// keys and tags.  The keys, tags and losses' buffers are grown here.
static int boot_sorted(dsgd_ctx *ctx, const double *w, const row_set &rows, cub::DoubleBuffer<unsigned long long> *kb,
                       cub::DoubleBuffer<uint32_t> *tb) {
  const int64_t n = rows.n;
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = request_weights(ctx, w, &wd, &cd, &nd);
  if (rc) return rc;
  const bool kl = model_of(ctx) != kSvm;
  if ((rc = ctx->m_keys.grow(ctx, n, 1024)) || (rc = ctx->m_alt.grow(ctx, n, 1024)) || (rc = ctx->b_tag.grow(ctx, n, 1024)) ||
      (rc = ctx->b_tagt.grow(ctx, n, 1024)) || (kl && (rc = ctx->b_loss.grow(ctx, n, 1024))))
    return rc;
  const int grid = (int)std::min<int64_t>(cdiv(n, 256), (int64_t)ctx->sm_count * 8);   // >= 32 positions per warp
  rc = with_model<kUnweighted>(ctx, [&](auto m, auto, auto ic) {
    k_boot_score<m, ic><<<grid, 256, 0, ctx->stream>>>(ctx->rp16, ctx->pairs, ctx->label, rows.ids, rows.row_begin, n, wd,
                                                      ctx->m_keys, ctx->b_tag, ctx->b_loss, icpt_of(ctx, wd));
    LAUNCHED();
    return DSGD_OK;
  });
  if (rc) return rc;
  CU(cudaGetLastError());
  *kb = cub::DoubleBuffer<unsigned long long>(ctx->m_keys.p, ctx->m_alt.p);
  *tb = cub::DoubleBuffer<uint32_t>(ctx->b_tag.p, ctx->b_tagt.p);
  size_t tmp = 0;
  CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp, *kb, *tb, (int)n, 0, 64, ctx->stream));
  if ((rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16))) return rc;
  CU(cub::DeviceRadixSort::SortPairs(ctx->m_tmp.p, tmp, *kb, *tb, (int)n, 0, 64, ctx->stream));
  return DSGD_OK;
}

// One bootstrap pass over `rows`: positions scored, sorted and arranged once, then replicates [b_begin, b_end) in chunks.
// Per replicate b (index b - b_begin of the outputs): the DSGD_BOOTSTRAP_WORDS words, AP = S / P under the curve pass's NaN
// rule, and the loss sum.  Launches of the sort's own kernels are not counted in dsgd_launch_count.
static int bootstrap_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, uint64_t bkey, int64_t b_begin, int64_t b_end,
                          int64_t *words, double *ap, double *loss) {
  const int64_t n = rows.n;
  const bool kl = model_of(ctx) != kSvm;
  cub::DoubleBuffer<unsigned long long> kb;
  cub::DoubleBuffer<uint32_t> tb;
  int rc;
  if ((rc = ctx->b_gs.grow(ctx, n, 1024)) || (kl && (rc = ctx->b_eloss.grow(ctx, n, 1024))) ||
      (rc = ctx->b_out.grow(ctx, kBootChunk * kBootOutWords, kBootChunk * kBootOutWords)) ||
      (rc = boot_sorted(ctx, w, rows, &kb, &tb)))
    return rc;
  const int agrid = (int)std::min<int64_t>(cdiv(n, 256), (int64_t)ctx->sm_count * 8);
  if (kl)
    k_boot_arrange<true><<<agrid, 256, 0, ctx->stream>>>(kb.Current(), tb.Current(), n, ctx->b_loss, ctx->b_gs, ctx->b_eloss);
  else
    k_boot_arrange<false><<<agrid, 256, 0, ctx->stream>>>(kb.Current(), tb.Current(), n, nullptr, ctx->b_gs, nullptr);
  LAUNCHED();
  CU(cudaGetLastError());
  std::vector<unsigned long long> h((size_t)(kBootChunk * kBootOutWords));
  for (int64_t b0 = b_begin; b0 < b_end; b0 += kBootChunk) {
    const int64_t k = std::min(kBootChunk, b_end - b0);
    if (kl)
      k_boot_rep<true><<<(int)k, kBootThreads, 0, ctx->stream>>>(tb.Current(), ctx->b_gs, ctx->b_eloss, n, bkey, b0, ctx->b_out);
    else
      k_boot_rep<false><<<(int)k, kBootThreads, 0, ctx->stream>>>(tb.Current(), ctx->b_gs, nullptr, n, bkey, b0, ctx->b_out);
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(h.data(), ctx->b_out, sizeof(unsigned long long) * (size_t)(k * kBootOutWords), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (int64_t r = 0; r < k; ++r) {
      const unsigned long long *o = &h[(size_t)(r * kBootOutWords)];
      int64_t *wr = words + (b0 - b_begin + r) * DSGD_BOOTSTRAP_WORDS;
      for (int q = 0; q < DSGD_BOOTSTRAP_WORDS; ++q) wr[q] = (int64_t)o[q];
      const int64_t P = wr[kMetTp] + wr[kMetFn] + wr[kMetPosNone];
      double S, L;
      memcpy(&S, &o[kBootS], sizeof S);
      memcpy(&L, &o[kBootLoss], sizeof L);
      ap[b0 - b_begin + r] = (wr[kMetNan] > 0 || P == 0) ? std::numeric_limits<double>::quiet_NaN() : S / (double)P;
      loss[b0 - b_begin + r] = L;
    }
  }
  return DSGD_OK;
}

// One weighted bootstrap pass over `rows` (DESIGN.md §4.20): scored and sorted as bootstrap_pass does, each sorted element's
// tie group, c and fl(c L) arranged once, then replicates [b_begin, b_end) in chunks.  Per replicate b (index j = b - b_begin):
// words[2 j] = sum m, words[2 j + 1] = the NaN-score rows, wsums[13 j ..] the DSGD_WCURVE_WORDS and loss[j] the weighted loss
// sum S of the expanded list.  Launches of the sort's own kernels are not counted in dsgd_launch_count.
static int weighted_bootstrap_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, uint64_t bkey, int64_t b_begin,
                                   int64_t b_end, int64_t *words, double *wsums, double *loss) {
  const int64_t n = rows.n;
  const bool kl = model_of(ctx) != kSvm;
  cub::DoubleBuffer<unsigned long long> kb;
  cub::DoubleBuffer<uint32_t> tb;
  int rc;
  if ((rc = ctx->b_gs.grow(ctx, n, 1024)) || (rc = ctx->b_gl.grow(ctx, n, 1024)) || (rc = ctx->b_c.grow(ctx, n, 1024)) ||
      (rc = ctx->b_eloss.grow(ctx, n, 1024)) ||
      (rc = ctx->b_out.grow(ctx, kBootChunk * kWbOutWords, kBootChunk * kWbOutWords)) ||
      (rc = boot_sorted(ctx, w, rows, &kb, &tb)))
    return rc;
  const int agrid = (int)std::min<int64_t>(cdiv(n, 256), (int64_t)ctx->sm_count * 8);
  const double *sw = ctx->sw_on ? ctx->sw.p : nullptr;
  if (kl)
    k_wboot_arrange<true><<<agrid, 256, 0, ctx->stream>>>(kb.Current(), tb.Current(), n, rows.ids, rows.row_begin, ctx->cw_pos,
                                                          ctx->cw_neg, sw, ctx->b_loss, ctx->b_gs, ctx->b_gl, ctx->b_c,
                                                          ctx->b_eloss);
  else
    k_wboot_arrange<false><<<agrid, 256, 0, ctx->stream>>>(kb.Current(), tb.Current(), n, rows.ids, rows.row_begin,
                                                           ctx->cw_pos, ctx->cw_neg, sw, nullptr, ctx->b_gs, ctx->b_gl,
                                                           ctx->b_c, ctx->b_eloss);
  LAUNCHED();
  CU(cudaGetLastError());
  std::vector<unsigned long long> h((size_t)(kBootChunk * kWbOutWords));
  for (int64_t b0 = b_begin; b0 < b_end; b0 += kBootChunk) {
    const int64_t k = std::min(kBootChunk, b_end - b0);
    k_wboot_rep<<<(int)k, kWbThreads, 0, ctx->stream>>>(kb.Current(), tb.Current(), ctx->b_gs, ctx->b_gl, ctx->b_c,
                                                         ctx->b_eloss, n, bkey, b0, ctx->b_out);
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(h.data(), ctx->b_out, sizeof(unsigned long long) * (size_t)(k * kWbOutWords), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (int64_t r = 0; r < k; ++r) {
      const unsigned long long *o = &h[(size_t)(r * kWbOutWords)];
      const int64_t j = b0 - b_begin + r;
      words[2 * j] = (int64_t)o[kWbSize];
      words[2 * j + 1] = (int64_t)o[kWbNan];
      memcpy(&wsums[DSGD_WCURVE_WORDS * j], &o[kWbSums], sizeof(double) * DSGD_WCURVE_WORDS);
      memcpy(&loss[j], &o[kWbLoss], sizeof(double));
    }
  }
  return DSGD_OK;
}

// dsgd_eval*_bootstrap: the outputs and the replicate range, an async ctx while its loop runs (the pass grows its own
// buffers), then the request's size -- all before anything is launched, the sampled form's draw included
static int bootstrap_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, uint64_t bkey,
                             int64_t b_begin, int64_t b_end, int64_t *words, double *ap, double *loss) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(words && ap && loss, DSGD_ERR_INVALID, "%s: words_out, ap_out or loss_out is NULL", fn);
  NEED(b_begin >= 0, DSGD_ERR_INVALID, "%s: replicates [%lld,%lld) start below 0", fn, (long long)b_begin, (long long)b_end);
  NEED(b_end > b_begin, DSGD_ERR_EMPTY, "%s: no replicates [%lld,%lld)", fn, (long long)b_begin, (long long)b_end);
  NEED(!ctx->a_running, DSGD_ERR_STATE, "%s: the async loop runs (the pass's buffers cannot grow until it is stopped)", fn);
  const int64_t n = req.form == row_request::kRange ? req.row_end - req.row_begin
                    : req.form == row_request::kDrawn ? req.pos_end - req.pos_begin : req.n;
  NEED(n <= kBootMaxRows, DSGD_ERR_INVALID, "%s: %lld rows; a bootstrap takes at most 2^26", fn, (long long)n);
  row_set rows;
  int rc = resolve_rows(ctx, req, fn, &rows);
  return rc ? rc : bootstrap_pass(ctx, w, rows, bkey, b_begin, b_end, words, ap, loss);
}

extern "C" int dsgd_eval_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t bkey,
                                   int64_t b_begin, int64_t b_end, int64_t *words_out, double *ap_out, double *loss_out) {
  return bootstrap_request(ctx, w, range_rows(row_begin, row_end), __func__, bkey, b_begin, b_end, words_out, ap_out,
                           loss_out);
}

extern "C" int dsgd_eval_sampled_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                           int64_t pos_begin, int64_t pos_end, uint64_t bkey, int64_t b_begin, int64_t b_end,
                                           int64_t *words_out, double *ap_out, double *loss_out) {
  return bootstrap_request(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, bkey, b_begin, b_end,
                           words_out, ap_out, loss_out);
}

extern "C" int dsgd_eval_samples_bootstrap(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, uint64_t bkey,
                                           int64_t b_begin, int64_t b_end, int64_t *words_out, double *ap_out,
                                           double *loss_out) {
  return bootstrap_request(ctx, w, listed_rows(samples, n), __func__, bkey, b_begin, b_end, words_out, ap_out, loss_out);
}

// dsgd_eval*_weighted_bootstrap: the outputs and the replicate range, an async ctx (its weights are always 1, and the pass
// grows its own buffers), then the request's size -- all before anything is launched, the sampled form's draw included
static int weighted_bootstrap_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, uint64_t bkey,
                                      int64_t b_begin, int64_t b_end, int64_t *words, double *wsums, double *loss) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(words && wsums && loss, DSGD_ERR_INVALID, "%s: words_out, wsums_out or loss_out is NULL", fn);
  NEED(b_begin >= 0, DSGD_ERR_INVALID, "%s: replicates [%lld,%lld) start below 0", fn, (long long)b_begin, (long long)b_end);
  NEED(b_end > b_begin, DSGD_ERR_EMPTY, "%s: no replicates [%lld,%lld)", fn, (long long)b_begin, (long long)b_end);
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (row weights belong to the sync paths)",
       fn);
  const int64_t n = req.form == row_request::kRange ? req.row_end - req.row_begin
                    : req.form == row_request::kDrawn ? req.pos_end - req.pos_begin : req.n;
  NEED(n <= kBootMaxRows, DSGD_ERR_INVALID, "%s: %lld rows; a bootstrap takes at most 2^26", fn, (long long)n);
  row_set rows;
  int rc = resolve_rows(ctx, req, fn, &rows);
  return rc ? rc : weighted_bootstrap_pass(ctx, w, rows, bkey, b_begin, b_end, words, wsums, loss);
}

extern "C" int dsgd_eval_weighted_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t bkey,
                                            int64_t b_begin, int64_t b_end, int64_t *words_out, double *wsums_out,
                                            double *loss_out) {
  return weighted_bootstrap_request(ctx, w, range_rows(row_begin, row_end), __func__, bkey, b_begin, b_end, words_out,
                                    wsums_out, loss_out);
}

extern "C" int dsgd_eval_sampled_weighted_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                    uint64_t key, int64_t pos_begin, int64_t pos_end, uint64_t bkey,
                                                    int64_t b_begin, int64_t b_end, int64_t *words_out, double *wsums_out,
                                                    double *loss_out) {
  return weighted_bootstrap_request(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, bkey, b_begin,
                                    b_end, words_out, wsums_out, loss_out);
}

extern "C" int dsgd_eval_samples_weighted_bootstrap(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                                    uint64_t bkey, int64_t b_begin, int64_t b_end, int64_t *words_out,
                                                    double *wsums_out, double *loss_out) {
  return weighted_bootstrap_request(ctx, w, listed_rows(samples, n), __func__, bkey, b_begin, b_end, words_out, wsums_out,
                                    loss_out);
}

// ---- calibration (dsgd_calibrate.cuh; DESIGN.md §4.11) ---------------------------------------------------------------

// Words of k_ctl: the counts of k_calib_score, the result of k_calib_fit, {barrier counter, abort flag}, the three lines
constexpr int kCtlCnt = 0, kCtlOut = kCalCntWords, kCtlBar = kCtlOut + kCalOutWords, kCtlAcc = 16;
constexpr int kCtlWords = kCtlAcc + 3 * kCalLineStride;
constexpr int kCtlW = kCtlWords, kCtlWWords = kCtlW + kCalWWords;   // a weighted fit's sums of R(c) (CalibWeightWord)
static_assert(kCtlBar + 1 <= kCtlAcc, "k_ctl layout");
static_assert(kCalMaxBins == DSGD_CALIBRATION_MAX_BINS && kCalOutEvals < kCalOutWords, "calibration layout");
constexpr int kCalSmemScores = 14336;   // scores (8 bytes) and labels (1 byte) a CTA of k_calib_fit keeps in shared memory: 126 KB
constexpr int kCalSmemScoresW = 7552;   // k_calib_fit<true>: score, weight (8 bytes each) and label, within the same 126 KB

// A cooperative grid cannot be assumed resident beside a kernel that runs until it is stopped.
static int calibrate_allowed(dsgd_ctx *ctx, const char *fn) {
  if (!ctx->a_running) return DSGD_OK;
  CU(cudaSetDevice(ctx->device));
  const cudaError_t e = cudaStreamQuery(ctx->astream);
  NEED(e != cudaErrorNotReady, DSGD_ERR_STATE, "%s: the async loop is running (stop it first: the fit is one cooperative launch)", fn);
  CU(e);
  return DSGD_OK;
}

// read() on the host: the value of six limb words and an overflow count, converted as acc_value converts them (the same
// operations in the same order, so the same bits): carries, then the limbs from the top down.
static double fixed_read(const unsigned long long *limbs, unsigned long long ovf) {
  if (ovf) return std::numeric_limits<double>::quiet_NaN();
  unsigned long long q[kLossLimbs];
  for (int i = 0; i < kLossLimbs; ++i) q[i] = limbs[i];
  for (int i = 0; i < kLossLimbs - 1; ++i) {
    q[i + 1] += q[i] >> 40;
    q[i] &= kLimbMask;
  }
  double s = (double)q[kLossLimbs - 1] * 0x1p40;
  for (int i = kLossLimbs - 2; i >= 0; --i) s += (double)q[i] * std::ldexp(1.0, 40 * i - 160);
  return s;
}

// One fit over `rows`: k_calib_score, the counts read by the host, k_calib_fit, the result read back.
// kW: the weighted fit (DESIGN.md §4.17): the targets and start point from W+ and W-, each read() of an exact sum of R(c_i);
// wsums_out = {W+, W-, the NaN rows' weight}.
template <bool kW>
static int calibrate_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, double *ab_out, double *objective_out,
                          int64_t *info_out, double *wsums_out, const char *fn) {
  const int64_t n = rows.n;
  const int ctl_words = kW ? kCtlWWords : kCtlWords;
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = request_weights(ctx, w, &wd, &cd, &nd);
  if (rc || (rc = ctx->k_score.grow(ctx, n, 1024)) || (rc = ctx->k_lab.grow(ctx, n, 1024)) ||
      (rc = ctx->k_ctl.grow(ctx, ctl_words, ctl_words)) || (kW && (rc = ctx->k_cw.grow(ctx, n, 1024))))
    return rc;
  CU(cudaMemsetAsync(ctx->k_ctl, 0, sizeof(unsigned long long) * ctl_words, ctx->stream));
  const int sgrid = (int)std::min<int64_t>(cdiv(n, 256), (int64_t)ctx->sm_count * 8);
  with_icpt(ctx, [&](auto ic) {
    k_calib_score<kW, ic><<<sgrid, 256, 0, ctx->stream>>>(ctx->rp16, ctx->pairs, ctx->label, rows.ids, rows.row_begin, n, wd,
                                                          ctx->k_score, ctx->k_lab, ctx->k_ctl + kCtlCnt, ctx->cw_pos,
                                                          ctx->cw_neg, ctx->sw_on ? ctx->sw.p : nullptr,
                                                          kW ? ctx->k_cw.p : nullptr, kW ? ctx->k_ctl + kCtlW : nullptr,
                                                          icpt_of(ctx, wd));
  });
  LAUNCHED();
  CU(cudaGetLastError());
  unsigned long long cnt[kCalCntWords], wacc[kCalWWords];
  CU(cudaMemcpyAsync(cnt, ctx->k_ctl + kCtlCnt, sizeof cnt, cudaMemcpyDeviceToHost, ctx->stream));
  if (kW) CU(cudaMemcpyAsync(wacc, ctx->k_ctl + kCtlW, sizeof wacc, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int64_t n_pos = (int64_t)cnt[kCalPos], n_neg = (int64_t)cnt[kCalNeg];
  double t_pos, t_neg, b0;
  if constexpr (kW) {
    const double w_p = fixed_read(wacc + kCalWPos, wacc[kCalWPos + kLossLimbs]);
    const double w_n = fixed_read(wacc + kCalWNeg, wacc[kCalWNeg + kLossLimbs]);
    wsums_out[0] = w_p;
    wsums_out[1] = w_n;
    wsums_out[2] = fixed_read(wacc + kCalWNan, wacc[kCalWNan + kLossLimbs]);
    NEED(w_p != 0.0 && w_n != 0.0, DSGD_ERR_EMPTY,
         "%s: positive weight %g and negative weight %g among the rows with a score: a sigmoid needs both classes", fn, w_p,
         w_n);
    t_pos = (w_p + 1.0) / (w_p + 2.0);
    t_neg = 1.0 / (w_n + 2.0);
    b0 = std::log((w_n + 1.0) / (w_p + 1.0));
  } else {
    NEED(n_pos > 0 && n_neg > 0, DSGD_ERR_EMPTY, "%s: %lld positive and %lld negative rows with a score (%lld NaN): a sigmoid needs both classes",
         fn, (long long)n_pos, (long long)n_neg, (long long)cnt[kCalNan]);
    t_pos = ((double)n_pos + 1.0) / ((double)n_pos + 2.0);
    t_neg = 1.0 / ((double)n_neg + 2.0);
    b0 = std::log(((double)n_neg + 1.0) / ((double)n_pos + 1.0));
  }

  constexpr int cap_max = kW ? kCalSmemScoresW : kCalSmemScores, per_score = kW ? 17 : 9;
  int &occ = kW ? ctx->k_fit_occ_w : ctx->k_fit_occ;
  if (!occ) {
    const int full = cap_max * per_score;
    CU(cudaFuncSetAttribute(k_calib_fit<kW>, cudaFuncAttributeMaxDynamicSharedMemorySize, full));
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_calib_fit<kW>, kCalThreads, (size_t)full));
    NEED(occ > 0, DSGD_ERR_CUDA, "%s: k_calib_fit does not fit on an SM", fn);
  }
  int G = ctx->sm_count * occ;   // resident at the full shared-memory budget, so at any smaller one
  if (ctx->grid_limit > 0) G = std::min(G, ctx->grid_limit);
  G = (int)std::min<int64_t>(G, cdiv(n, kCalThreads));
  CalibFitParams fp;
  memset(&fp, 0, sizeof fp);
  fp.score = ctx->k_score; fp.lab = ctx->k_lab; fp.n = n;
  fp.t_pos = t_pos;
  fp.t_neg = t_neg;
  fp.b0 = b0;
  fp.acc = ctx->k_ctl + kCtlAcc;
  fp.bar = reinterpret_cast<unsigned *>(ctx->k_ctl + kCtlBar);
  fp.abort_flag = reinterpret_cast<int *>(ctx->k_ctl + kCtlBar) + 1;
  fp.timeout_cycles = 4000000000ll;   // ~2 s, as the sync step's barrier
  fp.out = ctx->k_ctl + kCtlOut;
  fp.smem_cap = (int)std::min<int64_t>(cdiv(n, G), cap_max);
  if (kW) fp.cw = ctx->k_cw;
  void *args[] = {&fp};
  CU(cudaLaunchCooperativeKernel((void *)k_calib_fit<kW>, dim3(G), dim3(kCalThreads), args, (size_t)fp.smem_cap * per_score,
                                 ctx->stream));
  LAUNCHED();
  unsigned long long out[kCalOutWords + 1];
  CU(cudaMemcpyAsync(out, ctx->k_ctl + kCtlOut, sizeof out, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  NEED((out[kCalOutWords] >> 32) == 0, DSGD_ERR_TIMEOUT, "%s: the fit's grid barrier hit its watchdog", fn);
  memcpy(&ab_out[0], &out[kCalOutA], sizeof(double));
  memcpy(&ab_out[1], &out[kCalOutB], sizeof(double));
  memcpy(objective_out, &out[kCalOutF], sizeof(double));
  info_out[0] = (int64_t)out[kCalOutIter];
  info_out[1] = (int64_t)out[kCalOutStatus];
  info_out[2] = n_pos + n_neg;
  info_out[3] = (int64_t)cnt[kCalNan];
  info_out[4] = (int64_t)out[kCalOutEvals];
  return DSGD_OK;
}

// A weighted calibration call: an async ctx is refused before anything is launched (its weights are always 1), as the
// weighted curves refuse it.
static int weighted_calibration_allowed(dsgd_ctx *ctx, const char *fn) {
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "%s: ctx is in async mode (row weights belong to the sync paths)",
       fn);
  return DSGD_OK;
}

// dsgd_calibrate* and (kW) dsgd_calibrate_weighted*, which also write wsums_out
template <bool kW>
static int calibrate_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, double *ab_out,
                             double *objective_out, int64_t *info_out, double *wsums_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ab_out && objective_out && info_out && (!kW || wsums_out), DSGD_ERR_INVALID, "%s: an output is NULL", fn);
  int rc = kW ? weighted_calibration_allowed(ctx, fn) : DSGD_OK;
  if (rc || (rc = ids_capped(ctx, req, fn))) return rc;
  if (!kW && (rc = calibrate_allowed(ctx, fn))) return rc;
  row_set rows;
  if ((rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  return calibrate_pass<kW>(ctx, w, rows, ab_out, objective_out, info_out, wsums_out, fn);
}

extern "C" int dsgd_calibrate(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *ab_out,
                              double *objective_out, int64_t *info_out) {
  return calibrate_request<false>(ctx, w, range_rows(row_begin, row_end), __func__, ab_out, objective_out, info_out, nullptr);
}

extern "C" int dsgd_calibrate_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                      int64_t pos_begin, int64_t pos_end, double *ab_out, double *objective_out,
                                      int64_t *info_out) {
  return calibrate_request<false>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, ab_out,
                                  objective_out, info_out, nullptr);
}

extern "C" int dsgd_calibrate_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *ab_out,
                                      double *objective_out, int64_t *info_out) {
  return calibrate_request<false>(ctx, w, listed_rows(samples, n), __func__, ab_out, objective_out, info_out, nullptr);
}

extern "C" int dsgd_calibrate_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *ab_out,
                                       double *objective_out, int64_t *info_out, double *wsums_out) {
  return calibrate_request<true>(ctx, w, range_rows(row_begin, row_end), __func__, ab_out, objective_out, info_out,
                                 wsums_out);
}

extern "C" int dsgd_calibrate_weighted_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                               uint64_t key, int64_t pos_begin, int64_t pos_end, double *ab_out,
                                               double *objective_out, int64_t *info_out, double *wsums_out) {
  return calibrate_request<true>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, ab_out,
                                 objective_out, info_out, wsums_out);
}

extern "C" int dsgd_calibrate_weighted_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                               double *ab_out, double *objective_out, int64_t *info_out, double *wsums_out) {
  return calibrate_request<true>(ctx, w, listed_rows(samples, n), __func__, ab_out, objective_out, info_out, wsums_out);
}

extern "C" int dsgd_calibrated_probabilities(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double a,
                                             double b, double *probs_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(probs_out, DSGD_ERR_INVALID, "%s: output is NULL", __func__);
  NEED(std::isfinite(a) && std::isfinite(b), DSGD_ERR_INVALID, "%s: (a, b) = (%g, %g) is not finite", __func__, a, b);
  row_set rows;
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = rows_list(ctx, samples, n, true, __func__, &rows);
  if (rc || (rc = request_weights(ctx, w, &wd, &cd, &nd))) return rc;
  with_icpt(ctx, [&](auto ic) {
    k_calib_prob<ic><<<rows_grid(ctx, rows.n), 256, 0, ctx->stream>>>(ctx->rp16, ctx->pairs, rows.ids, rows.n, wd, a, b,
                                                                      ctx->preds, icpt_of(ctx, wd));
  });
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(probs_out, ctx->preds, sizeof(double) * (size_t)rows.n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

static int isotonic_map(dsgd_ctx *ctx, const double *X, const double *Y, int64_t k, const char *fn);
// The dynamic shared memory of a kernel that reads a map of k >= 1 points: the map when it fits (the kernel's kSmem form),
// else none (its kSmem = false form, which reads the map through L2)
static size_t map_smem(int64_t k) { return k <= kIsoSmemPoints ? (size_t)k * 16 : 0; }
// Launches kernel on 256-thread CTAs with smem bytes of dynamic shared memory, its limit raised to them first
static cudaError_t launch_smem(const void *kernel, int grid, size_t smem, cudaStream_t stream, void **args) {
  if (smem) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  return cudaLaunchKernel(kernel, dim3(grid), dim3(256), args, smem, stream);
}
// One quality pass over `rows`, at (a, b) or (kIso) at the map (X, Y): k_calib_eval, k_calib_eval_finish, the block read
// back.  words_out = {rows used, NaN rows} and (kIso) the rows whose log-loss term is infinite.
template <bool kIso>
static int calibration_quality_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, double a, double b, const double *X,
                                    const double *Y, int64_t k, int32_t n_bins, double *sums_out, int64_t *bin_rows,
                                    int64_t *bin_pos, double *bin_psum, int64_t *words_out, const char *fn) {
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = fits_while_running(ctx, ctx->k_eval, fn);
  if (rc || (rc = request_weights(ctx, w, &wd, &cd, &nd)) || (kIso && (rc = isotonic_map(ctx, X, Y, k, fn))) ||
      (rc = ctx->k_eval.grow(ctx, kCevWords, kCevWords)))
    return rc;
  CU(cudaMemsetAsync(ctx->k_eval, 0, sizeof(unsigned long long) * kCevWords, ctx->stream));
  const int grid = (int)std::min<int64_t>(cdiv(rows.n, 256), (int64_t)ctx->sm_count * 8);
  const double *mx = kIso ? ctx->i_map.p : nullptr, *my = kIso ? ctx->i_map.p + k : nullptr;
  int ki = (int)k, nb = n_bins;
  unsigned long long *blk = ctx->k_eval.p;
  const uint32_t *rp16 = ctx->rp16.p;
  const uint2 *pairs = ctx->pairs.p;
  const int8_t *label = ctx->label.p;
  const int32_t *ids = rows.ids;
  int64_t rb = rows.row_begin, rn = rows.n;
  const double *icpt = icpt_of(ctx, wd);
  void *args[] = {&rp16, &pairs, &label, &ids, &rb, &rn, &wd, &a, &b, &mx, &my, &ki, &nb, &blk, &icpt};
  const size_t smem = kIso ? map_smem(k) : 0;   // the kSmem form only at a map that fits
  CU(with_icpt(ctx, [&](auto ic) {
    auto kernel = smem ? k_calib_eval<kIso, kIso, ic> : k_calib_eval<kIso, false, ic>;
    return launch_smem((const void *)kernel, grid, smem, ctx->stream, args);
  }));
  LAUNCHED();
  k_calib_eval_finish<<<1, kCalMaxBins, 0, ctx->stream>>>(ctx->k_eval, n_bins);
  LAUNCHED();
  CU(cudaGetLastError());
  unsigned long long h[kCevWords];
  CU(cudaMemcpyAsync(h, ctx->k_eval, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  memcpy(sums_out, &h[kCevOutSums], 2 * sizeof(double));
  for (int i = 0; i < n_bins; ++i) {
    bin_rows[i] = (int64_t)h[kCevBinRows + i];
    bin_pos[i] = (int64_t)h[kCevBinPos + i];
  }
  memcpy(bin_psum, &h[kCevOutPsum], (size_t)n_bins * sizeof(double));
  words_out[0] = (int64_t)h[kCevRows];
  words_out[1] = (int64_t)h[kCevNan];
  if (kIso) words_out[2] = (int64_t)h[kCevInf];
  return DSGD_OK;
}

// One weighted quality pass over `rows`, at (a, b) or (kIso) at the map (X, Y): k_weval, the block read back, every sum
// read() on the host.
template <bool kIso>
static int weighted_quality_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, double a, double b, const double *X,
                                 const double *Y, int64_t k, int32_t n_bins, double *sums_out, double *bin_weight,
                                 double *bin_pos_weight, double *bin_psum, int64_t *words_out, const char *fn) {
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = request_weights(ctx, w, &wd, &cd, &nd);
  if (rc || (kIso && (rc = isotonic_map(ctx, X, Y, k, fn))) || (rc = ctx->k_eval.grow(ctx, kCwvWords, kCwvWords))) return rc;
  CU(cudaMemsetAsync(ctx->k_eval, 0, sizeof(unsigned long long) * kCwvWords, ctx->stream));
  const int grid = (int)std::min<int64_t>(cdiv(rows.n, 256), (int64_t)ctx->sm_count * 8);
  const double *mx = kIso ? ctx->i_map.p : nullptr, *my = kIso ? ctx->i_map.p + k : nullptr;
  int ki = (int)k, nb = n_bins;
  unsigned long long *blk = ctx->k_eval.p;
  const uint32_t *rp16 = ctx->rp16.p;
  const uint2 *pairs = ctx->pairs.p;
  const int8_t *label = ctx->label.p;
  const int32_t *ids = rows.ids;
  int64_t rb = rows.row_begin, rn = rows.n;
  double cwp = ctx->cw_pos, cwn = ctx->cw_neg;
  const double *swp = ctx->sw_on ? ctx->sw.p : nullptr;
  const double *icpt = icpt_of(ctx, wd);
  void *args[] = {&rp16, &pairs, &label, &ids, &rb, &rn, &wd, &a, &b, &mx, &my, &ki, &nb, &blk, &cwp, &cwn, &swp, &icpt};
  const size_t smem = kIso ? map_smem(k) : 0;   // the kSmem form only at a map that fits
  CU(with_icpt(ctx, [&](auto ic) {
    auto kernel = smem ? k_weval<kIso, kIso, ic> : k_weval<kIso, false, ic>;
    return launch_smem((const void *)kernel, grid, smem, ctx->stream, args);
  }));
  LAUNCHED();
  CU(cudaGetLastError());
  std::vector<unsigned long long> h(kCwvWords);
  CU(cudaMemcpyAsync(h.data(), ctx->k_eval, sizeof(unsigned long long) * kCwvWords, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  sums_out[0] = fixed_read(&h[kCwvBrier], h[kCwvBrier + kLossLimbs]);
  sums_out[1] = fixed_read(&h[kCwvLog], h[kCwvLog + kLossLimbs]);
  sums_out[2] = fixed_read(&h[kCwvW], h[kCwvW + kLossLimbs]);
  sums_out[3] = fixed_read(&h[kCwvInfW], h[kCwvInfW + kLossLimbs]);   // always 0 at a sigmoid: its term is finite
  for (int i = 0; i < n_bins; ++i) {
    const unsigned long long *q = &h[kCwvBins + i * kCwvBinStride], ovf = q[3 * kLossLimbs];
    bin_weight[i] = fixed_read(q, ovf);
    bin_pos_weight[i] = fixed_read(q + kLossLimbs, ovf);
    bin_psum[i] = fixed_read(q + 2 * kLossLimbs, ovf);
  }
  words_out[0] = (int64_t)h[kCwvRows];
  words_out[1] = (int64_t)h[kCwvNan];
  if (kIso) words_out[2] = (int64_t)h[kCwvInf];
  return DSGD_OK;
}

// The quality calls: dsgd_eval*_calibration at the sigmoid (a, b), or (kIso) dsgd_eval*_isotonic_calibration at the map
// (X, Y); counted (B = int64_t: the rows and the positives of each bin), or (kW) weighted (B = double: their weights)
template <bool kIso, bool kW, class B>
static int quality_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, double a, double b,
                           const double *X, const double *Y, int64_t k, int32_t n_bins, double *sums_out, B *bin_rows,
                           B *bin_pos, double *bin_psum, int64_t *words_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(sums_out && bin_rows && bin_pos && bin_psum && words_out, DSGD_ERR_INVALID, "%s: an output is NULL", fn);
  if constexpr (!kIso)
    NEED(std::isfinite(a) && std::isfinite(b), DSGD_ERR_INVALID, "%s: (a, b) = (%g, %g) is not finite", fn, a, b);
  NEED(n_bins >= 1 && n_bins <= kCalMaxBins, DSGD_ERR_INVALID, "%s: %d bins; 1 to %d", fn, (int)n_bins, kCalMaxBins);
  int rc = kW ? weighted_calibration_allowed(ctx, fn) : DSGD_OK;
  row_set rows;
  if (rc || (rc = ids_capped(ctx, req, fn)) || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  if constexpr (kW)
    return weighted_quality_pass<kIso>(ctx, w, rows, a, b, X, Y, k, n_bins, sums_out, bin_rows, bin_pos, bin_psum,
                                       words_out, fn);
  else
    return calibration_quality_pass<kIso>(ctx, w, rows, a, b, X, Y, k, n_bins, sums_out, bin_rows, bin_pos, bin_psum,
                                          words_out, fn);
}

extern "C" int dsgd_eval_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double a, double b,
                                     int32_t n_bins, double *sums_out, int64_t *bin_rows, int64_t *bin_pos, double *bin_psum,
                                     int64_t *words_out) {
  return quality_request<false, false>(ctx, w, range_rows(row_begin, row_end), __func__, a, b, nullptr, nullptr, 0, n_bins,
                                       sums_out, bin_rows, bin_pos, bin_psum, words_out);
}

extern "C" int dsgd_eval_sampled_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                             int64_t pos_begin, int64_t pos_end, double a, double b, int32_t n_bins,
                                             double *sums_out, int64_t *bin_rows, int64_t *bin_pos, double *bin_psum,
                                             int64_t *words_out) {
  return quality_request<false, false>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, a, b,
                                       nullptr, nullptr, 0, n_bins, sums_out, bin_rows, bin_pos, bin_psum, words_out);
}

extern "C" int dsgd_eval_samples_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double a,
                                             double b, int32_t n_bins, double *sums_out, int64_t *bin_rows, int64_t *bin_pos,
                                             double *bin_psum, int64_t *words_out) {
  return quality_request<false, false>(ctx, w, listed_rows(samples, n), __func__, a, b, nullptr, nullptr, 0, n_bins, sums_out,
                                       bin_rows, bin_pos, bin_psum, words_out);
}

extern "C" int dsgd_eval_weighted_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double a,
                                              double b, int32_t n_bins, double *sums_out, double *bin_weight,
                                              double *bin_pos_weight, double *bin_psum, int64_t *words_out) {
  return quality_request<false, true>(ctx, w, range_rows(row_begin, row_end), __func__, a, b, nullptr, nullptr, 0, n_bins,
                                      sums_out, bin_weight, bin_pos_weight, bin_psum, words_out);
}

extern "C" int dsgd_eval_sampled_weighted_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                      uint64_t key, int64_t pos_begin, int64_t pos_end, double a, double b,
                                                      int32_t n_bins, double *sums_out, double *bin_weight,
                                                      double *bin_pos_weight, double *bin_psum, int64_t *words_out) {
  return quality_request<false, true>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, a, b,
                                      nullptr, nullptr, 0, n_bins, sums_out, bin_weight, bin_pos_weight, bin_psum, words_out);
}

extern "C" int dsgd_eval_samples_weighted_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                                      double a, double b, int32_t n_bins, double *sums_out,
                                                      double *bin_weight, double *bin_pos_weight, double *bin_psum,
                                                      int64_t *words_out) {
  return quality_request<false, true>(ctx, w, listed_rows(samples, n), __func__, a, b, nullptr, nullptr, 0, n_bins, sums_out,
                                      bin_weight, bin_pos_weight, bin_psum, words_out);
}

// ---- isotonic calibration (dsgd_isotonic.cuh; DESIGN.md §4.16) ------------------------------------------------------

// Points of a hull tile: DSGD_ISOTONIC_TILE (1 .. kIsoTileMax) if set, else kIsoTileMax.  The fit has the same bits at every
// tile size; the variable lets a test see that.
static int isotonic_tile() {
  const char *v = getenv("DSGD_ISOTONIC_TILE");
  const long t = v ? strtol(v, nullptr, 10) : 0;
  return t >= 1 && t <= kIsoTileMax ? (int)t : kIsoTileMax;
}

// CTAs of a hull or emit launch of `items` work items: the grid limit if one is set (dsgd_set_grid_limit), else 8 per SM
static int isotonic_grid(const dsgd_ctx *ctx, int64_t items) {
  const int64_t cap = ctx->grid_limit > 0 ? ctx->grid_limit : (int64_t)ctx->sm_count * 8;
  return (int)std::max<int64_t>(1, std::min<int64_t>(items, cap));
}

// The hull and the emit of a fit over `points` points of the point set P (its arrays c0, c1; their scores thr): k_iso_tile,
// k_iso_merge rounds until one hull is left, the hull's vertex count read back, the scan of the blocks' X counts,
// k_iso_emit (X and Y into i_out, the blocks' two values into blk and blk + n), and the outputs copied back.  *n_blocks and
// *n_x: the blocks and the X entries.
template <class P>
static int isotonic_hull(dsgd_ctx *ctx, const typename P::Coord *c0, const typename P::Coord *c1, const double *thr,
                         int64_t points, int64_t n, typename P::Block *blk, double *x_out, double *y_out, void *rows_out,
                         void *pos_out, int *n_blocks, int64_t *n_x, const char *fn) {
  const int M = (int)points + 1, S = isotonic_tile(), T = (M + S - 1) / S;
  int *hv[2] = {ctx->i_hull.p, ctx->i_hull.p + M};
  int *hc[2] = {ctx->i_hull.p + 2 * (int64_t)M, ctx->i_hull.p + 2 * (int64_t)M + T};
  int *excl = ctx->i_hull.p + 2 * (int64_t)M + 2 * (int64_t)T;
  const size_t tile_bytes = (size_t)S * (2 * sizeof(typename P::Coord) + sizeof(int));
  CU(cudaFuncSetAttribute(k_iso_tile<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tile_bytes));
  k_iso_tile<P><<<isotonic_grid(ctx, T), kIsoThreads, tile_bytes, ctx->stream>>>(c0, c1, M, S, hv[0], hc[0]);
  LAUNCHED();
  int cur = 0;
  for (int64_t W = S, h = T; h > 1; W *= 2, h = (h + 1) / 2, cur ^= 1) {
    k_iso_merge<P><<<isotonic_grid(ctx, (h + 1) / 2), kIsoThreads, 0, ctx->stream>>>(c0, c1, (int)h, (int)W, hv[cur], hc[cur],
                                                                                     hv[cur ^ 1], hc[cur ^ 1]);
    LAUNCHED();
  }
  CU(cudaGetLastError());
  int V = 0;
  CU(cudaMemcpyAsync(&V, hc[cur], sizeof V, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int B = V - 1;   // the origin and the last point are always vertices: B >= 1
  NEED(B >= 1 && B <= points, DSGD_ERR_CUDA, "%s: a hull of %d vertices over %lld points", fn, V, (long long)points);
  size_t tmp = 0;
  CU(scan_x_counts(ctx, nullptr, tmp, hv[cur], B, excl));
  int rc = fits_while_running(ctx, ctx->m_tmp.cap >= (int64_t)tmp, fn);
  if (rc || (rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16))) return rc;
  CU(scan_x_counts(ctx, ctx->m_tmp.p, tmp, hv[cur], B, excl));
  double *X = ctx->i_out.p, *Y = ctx->i_out.p + n;
  k_iso_emit<P><<<isotonic_grid(ctx, cdiv(B, 256)), 256, 0, ctx->stream>>>(hv[cur], B, excl, thr, c0, c1, X, Y, blk, blk + n,
                                                                           ctx->i_ctl);
  LAUNCHED();
  CU(cudaGetLastError());
  unsigned long long nx = 0;
  CU(cudaMemcpyAsync(&nx, ctx->i_ctl, sizeof nx, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(rows_out, blk, sizeof(typename P::Block) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(pos_out, blk + n, sizeof(typename P::Block) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaMemcpyAsync(x_out, X, sizeof(double) * (size_t)nx, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(y_out, Y, sizeof(double) * (size_t)nx, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  *n_blocks = B;
  *n_x = (int64_t)nx;
  return DSGD_OK;
}

// One isotonic fit over `rows`: the curve pass with its points left on the device, then the hull and the emit over its
// counts (IsoCounts).
static int isotonic_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, int64_t *n_points_out, double *x_out,
                         double *y_out, int64_t *rows_out, int64_t *pos_out, int64_t *info_out, const char *fn) {
  const int64_t n = rows.n;
  int rc = fits_while_running(ctx, ctx->i_hull.cap >= 5 * (n + 1) && ctx->i_out.cap >= 2 * n && ctx->i_blk.cap >= 2 * n &&
                                       ctx->i_ctl,
                              fn);
  int64_t words[DSGD_METRICS_WORDS], m = 0;
  double ap = 0.0;
  if (rc || (rc = curve_pass<kUnweighted>(ctx, w, rows, words, &ap, &m, nullptr, nullptr, nullptr, fn, true))) return rc;
  const int64_t nan = words[kMetNan];
  NEED(m > 0, DSGD_ERR_EMPTY, "%s: all %lld rows have a NaN score", fn, (long long)n);
  if ((rc = ctx->i_hull.grow(ctx, 5 * (n + 1), 1024)) || (rc = ctx->i_out.grow(ctx, 2 * n, 1024)) ||
      (rc = ctx->i_blk.grow(ctx, 2 * n, 1024)) || (rc = ctx->i_ctl.grow(ctx, 1, 1)))
    return rc;
  int B = 0;
  if ((rc = isotonic_hull<IsoCounts>(ctx, ctx->c_tp, ctx->c_fp, ctx->c_thr, m, n, ctx->i_blk.p, x_out, y_out, rows_out,
                                     pos_out, &B, n_points_out, fn)))
    return rc;
  info_out[0] = B;
  info_out[1] = *n_points_out;
  info_out[2] = n - nan;
  info_out[3] = nan;
  info_out[4] = m;
  return DSGD_OK;
}

static int isotonic_weighted_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, int64_t *n_points_out, double *x_out,
                                  double *y_out, double *wrows_out, double *wpos_out, int64_t *info_out, double *wsums_out,
                                  const char *fn);

// dsgd_calibrate_isotonic* (B = int64_t: the blocks' rows and positives) and (kW) dsgd_calibrate_isotonic_weighted*
// (B = double: their weights; wsums_out too)
template <bool kW, class B>
static int isotonic_request(dsgd_ctx *ctx, const double *w, const row_request &req, const char *fn, int64_t *n_points_out,
                            double *x_out, double *y_out, B *rows_out, B *pos_out, int64_t *info_out, double *wsums_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n_points_out && x_out && y_out && rows_out && pos_out && info_out && (!kW || wsums_out), DSGD_ERR_INVALID,
       "%s: an output is NULL", fn);
  int rc = kW ? weighted_calibration_allowed(ctx, fn) : DSGD_OK;
  row_set rows;
  if (rc || (rc = ids_capped(ctx, req, fn)) || (rc = resolve_rows(ctx, req, fn, &rows))) return rc;
  if constexpr (kW)
    return isotonic_weighted_pass(ctx, w, rows, n_points_out, x_out, y_out, rows_out, pos_out, info_out, wsums_out, fn);
  else
    return isotonic_pass(ctx, w, rows, n_points_out, x_out, y_out, rows_out, pos_out, info_out, fn);
}

extern "C" int dsgd_calibrate_isotonic(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                       int64_t *n_points_out, double *x_out, double *y_out, int64_t *rows_out,
                                       int64_t *pos_out, int64_t *info_out) {
  return isotonic_request<false>(ctx, w, range_rows(row_begin, row_end), __func__, n_points_out, x_out, y_out, rows_out,
                                 pos_out, info_out, nullptr);
}

extern "C" int dsgd_calibrate_isotonic_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                               uint64_t key, int64_t pos_begin, int64_t pos_end, int64_t *n_points_out,
                                               double *x_out, double *y_out, int64_t *rows_out, int64_t *pos_out,
                                               int64_t *info_out) {
  return isotonic_request<false>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, n_points_out,
                                 x_out, y_out, rows_out, pos_out, info_out, nullptr);
}

extern "C" int dsgd_calibrate_isotonic_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                               int64_t *n_points_out, double *x_out, double *y_out, int64_t *rows_out,
                                               int64_t *pos_out, int64_t *info_out) {
  return isotonic_request<false>(ctx, w, listed_rows(samples, n), __func__, n_points_out, x_out, y_out, rows_out, pos_out,
                                 info_out, nullptr);
}

// A map (X, Y) of k points: X finite and strictly increasing, Y in [0, 1]; copied into i_map (X, then Y)
static int isotonic_map(dsgd_ctx *ctx, const double *X, const double *Y, int64_t k, const char *fn) {
  NEED(X && Y && k >= 1 && k <= (int64_t)INT32_MAX, DSGD_ERR_INVALID, "%s: the map needs X and Y of 1 to 2^31 - 1 points", fn);
  for (int64_t i = 0; i < k; ++i) {
    NEED(std::isfinite(X[i]) && (i == 0 || X[i] > X[i - 1]), DSGD_ERR_INVALID,
         "%s: X[%lld] = %g: X must be finite and strictly increasing", fn, (long long)i, X[i]);
    NEED(Y[i] >= 0.0 && Y[i] <= 1.0, DSGD_ERR_INVALID, "%s: Y[%lld] = %g is not in [0, 1]", fn, (long long)i, Y[i]);
  }
  int rc = fits_while_running(ctx, ctx->i_map.cap >= 2 * k, fn);
  if (rc || (rc = ctx->i_map.grow(ctx, 2 * k, 1024))) return rc;
  CU(cudaMemcpyAsync(ctx->i_map.p, X, sizeof(double) * (size_t)k, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->i_map.p + k, Y, sizeof(double) * (size_t)k, cudaMemcpyHostToDevice, ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_isotonic_probabilities(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, const double *X,
                                           const double *Y, int64_t k, double *probs_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(probs_out, DSGD_ERR_INVALID, "%s: output is NULL", __func__);
  row_set rows{};   // set whenever rows_list succeeds; initialised because GCC's -Wmaybe-uninitialized cannot see that
  const double *wd = nullptr, *cd = nullptr, *nd = nullptr;
  int rc = rows_list(ctx, samples, n, true, __func__, &rows);
  if (rc || (rc = request_weights(ctx, w, &wd, &cd, &nd)) || (rc = isotonic_map(ctx, X, Y, k, __func__))) return rc;
  const double *mx = ctx->i_map.p, *my = ctx->i_map.p + k;
  int ki = (int)k;
  double *out = ctx->preds.p;
  const uint32_t *rp16 = ctx->rp16.p;
  const uint2 *pairs = ctx->pairs.p;
  const int32_t *ids = rows.ids;
  int64_t rn = rows.n;
  const double *icpt = icpt_of(ctx, wd);
  void *args[] = {&rp16, &pairs, &ids, &rn, &wd, &mx, &my, &ki, &out, &icpt};
  const size_t smem = map_smem(k);
  CU(with_icpt(ctx, [&](auto ic) {
    auto kernel = smem ? k_iso_prob<true, ic> : k_iso_prob<false, ic>;
    return launch_smem((const void *)kernel, rows_grid(ctx, rows.n), smem, ctx->stream, args);
  }));
  LAUNCHED();
  CU(cudaMemcpyAsync(probs_out, ctx->preds, sizeof(double) * (size_t)rows.n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_eval_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                              const double *X, const double *Y, int64_t k, int32_t n_bins, double *sums_out,
                                              int64_t *bin_rows, int64_t *bin_pos, double *bin_psum, int64_t *words_out) {
  return quality_request<true, false>(ctx, w, range_rows(row_begin, row_end), __func__, 0.0, 0.0, X, Y, k, n_bins, sums_out,
                                      bin_rows, bin_pos, bin_psum, words_out);
}

extern "C" int dsgd_eval_sampled_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                      uint64_t key, int64_t pos_begin, int64_t pos_end, const double *X,
                                                      const double *Y, int64_t k, int32_t n_bins, double *sums_out,
                                                      int64_t *bin_rows, int64_t *bin_pos, double *bin_psum,
                                                      int64_t *words_out) {
  return quality_request<true, false>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, 0.0, 0.0, X,
                                      Y, k, n_bins, sums_out, bin_rows, bin_pos, bin_psum, words_out);
}

extern "C" int dsgd_eval_samples_isotonic_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                                      const double *X, const double *Y, int64_t k, int32_t n_bins,
                                                      double *sums_out, int64_t *bin_rows, int64_t *bin_pos,
                                                      double *bin_psum, int64_t *words_out) {
  return quality_request<true, false>(ctx, w, listed_rows(samples, n), __func__, 0.0, 0.0, X, Y, k, n_bins, sums_out,
                                      bin_rows, bin_pos, bin_psum, words_out);
}

// ---- weighted isotonic calibration (dsgd_isotonic.cuh; DESIGN.md §4.17) -----------------------------------------------

// One weighted isotonic fit over `rows`: the weighted curve pass with its points left on the device; the total weight of
// its non-NaN rows checked against the turn test's bound; every point's exact coordinates and the zero-weight points
// dropped (k_iso_wpoint, a scan of the keep flags, k_iso_wpack); then the hull and the emit over the kept points
// (IsoWeights).
static int isotonic_weighted_pass(dsgd_ctx *ctx, const double *w, const row_set &rows, int64_t *n_points_out, double *x_out,
                                  double *y_out, double *wrows_out, double *wpos_out, int64_t *info_out, double *wsums_out,
                                  const char *fn) {
  const int64_t n = rows.n;
  int64_t words[DSGD_METRICS_WORDS], m = 0;
  double wc[DSGD_WCURVE_WORDS];
  sorted_runs s;
  int rc = curve_pass<kSampleWeighted>(ctx, w, rows, words, wc, &m, nullptr, nullptr, nullptr, fn, true, &s);
  if (rc) return rc;
  // the totals of the two runs, exact: W+ and W- of the non-NaN rows
  limb_sum tot[2] = {{{0, 0, 0, 0, 0, 0}, 0}, {{0, 0, 0, 0, 0, 0}, 0}};
  if (s.n_pos) CU(cudaMemcpyAsync(&tot[0], ctx->c_pre.p + s.n_pos - 1, sizeof(limb_sum), cudaMemcpyDeviceToHost, ctx->stream));
  if (s.n_neg)
    CU(cudaMemcpyAsync(&tot[1], ctx->c_pre.p + s.n_pos + s.n_neg - 1, sizeof(limb_sum), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  unsigned long long q[kLossLimbs];
  for (int k = 0; k < kLossLimbs; ++k) q[k] = tot[0].l[k] + tot[1].l[k];
  for (int k = 0; k < kLossLimbs - 1; ++k) {
    q[k + 1] += q[k] >> 40;
    q[k] &= kLimbMask;
  }
  NEED(tot[0].ovf == 0 && tot[1].ovf == 0 && q[kLossLimbs - 1] < (1ull << 56), DSGD_ERR_RANGE,
       "%s: the rows' total weight is 2^96 or more (or a weight is 2^52 or more): the hull's turn test is exact below that",
       fn);
  wsums_out[0] = fixed_read(tot[0].l, 0);
  wsums_out[1] = fixed_read(tot[1].l, 0);
  bool any = false;
  for (int k = 0; k < kLossLimbs; ++k) any |= q[k] != 0;
  NEED(any, DSGD_ERR_EMPTY, "%s: no row with a non-NaN score has a positive weight (%lld rows, %lld NaN)", fn,
       (long long)n, (long long)words[kMetNan]);
  if ((rc = ctx->i_hull.grow(ctx, 5 * (n + 1), 1024)) || (rc = ctx->i_out.grow(ctx, 2 * n, 1024)) ||
      (rc = ctx->i_wblk.grow(ctx, 2 * n, 1024)) || (rc = ctx->i_ctl.grow(ctx, 4, 4)) || (rc = ctx->i_wpt.grow(ctx, 4 * n, 1024)) ||
      (rc = ctx->i_wkeep.grow(ctx, 2 * n, 1024)) || (rc = ctx->i_wthr.grow(ctx, n, 1024)))
    return rc;
  CU(cudaMemsetAsync(ctx->i_ctl, 0, sizeof(unsigned long long) * 4, ctx->stream));
  u256 *px = ctx->i_wpt.p, *py = px + n, *qx = px + 2 * n, *qy = px + 3 * n;
  int *keep = ctx->i_wkeep.p, *kexcl = keep + n;
  k_iso_wpoint<<<isotonic_grid(ctx, cdiv(std::max<int64_t>(m, s.n_pos + s.n_neg), 256)), 256, 0, ctx->stream>>>(
      ctx->c_thr, m, s.pos, s.n_pos, s.neg, s.n_neg, ctx->c_pre.p, ctx->c_pre.p + s.n_pos, s.pos_c, s.neg_c, px, py, keep,
      ctx->i_ctl + 1);
  LAUNCHED();
  size_t tmp = 0;
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp, keep, kexcl, (int)m, ctx->stream));
  if ((rc = ctx->m_tmp.grow(ctx, (int64_t)tmp, 1 << 16))) return rc;
  CU(cub::DeviceScan::ExclusiveSum(ctx->m_tmp.p, tmp, keep, kexcl, (int)m, ctx->stream));
  k_iso_wpack<<<isotonic_grid(ctx, cdiv(m, 256)), 256, 0, ctx->stream>>>(m, keep, kexcl, px, py, ctx->c_thr, qx, qy,
                                                                        ctx->i_wthr, ctx->i_ctl + 2);
  LAUNCHED();
  CU(cudaGetLastError());
  unsigned long long ctl[4];
  CU(cudaMemcpyAsync(ctl, ctx->i_ctl, sizeof ctl, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int64_t kept = (int64_t)ctl[2];
  NEED(kept >= 1 && kept <= m, DSGD_ERR_CUDA, "%s: %lld points kept of %lld", fn, (long long)kept, (long long)m);
  int B = 0;
  if ((rc = isotonic_hull<IsoWeights>(ctx, qx, qy, ctx->i_wthr, kept, n, ctx->i_wblk.p, x_out, y_out, wrows_out, wpos_out,
                                      &B, n_points_out, fn)))
    return rc;
  info_out[0] = B;
  info_out[1] = *n_points_out;
  info_out[2] = (int64_t)ctl[1];
  info_out[3] = words[kMetNan];
  info_out[4] = kept;
  return DSGD_OK;
}

extern "C" int dsgd_calibrate_isotonic_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                int64_t *n_points_out, double *x_out, double *y_out, double *wrows_out,
                                                double *wpos_out, int64_t *info_out, double *wsums_out) {
  return isotonic_request<true>(ctx, w, range_rows(row_begin, row_end), __func__, n_points_out, x_out, y_out, wrows_out,
                                wpos_out, info_out, wsums_out);
}

extern "C" int dsgd_calibrate_isotonic_weighted_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                        uint64_t key, int64_t pos_begin, int64_t pos_end,
                                                        int64_t *n_points_out, double *x_out, double *y_out,
                                                        double *wrows_out, double *wpos_out, int64_t *info_out,
                                                        double *wsums_out) {
  return isotonic_request<true>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, n_points_out,
                                x_out, y_out, wrows_out, wpos_out, info_out, wsums_out);
}

extern "C" int dsgd_calibrate_isotonic_weighted_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                                        int64_t *n_points_out, double *x_out, double *y_out,
                                                        double *wrows_out, double *wpos_out, int64_t *info_out,
                                                        double *wsums_out) {
  return isotonic_request<true>(ctx, w, listed_rows(samples, n), __func__, n_points_out, x_out, y_out, wrows_out, wpos_out,
                                info_out, wsums_out);
}

extern "C" int dsgd_eval_weighted_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                       const double *X, const double *Y, int64_t k, int32_t n_bins,
                                                       double *sums_out, double *bin_weight, double *bin_pos_weight,
                                                       double *bin_psum, int64_t *words_out) {
  return quality_request<true, true>(ctx, w, range_rows(row_begin, row_end), __func__, 0.0, 0.0, X, Y, k, n_bins, sums_out,
                                     bin_weight, bin_pos_weight, bin_psum, words_out);
}

extern "C" int dsgd_eval_sampled_weighted_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin,
                                                               int64_t row_end, uint64_t key, int64_t pos_begin,
                                                               int64_t pos_end, const double *X, const double *Y, int64_t k,
                                                               int32_t n_bins, double *sums_out, double *bin_weight,
                                                               double *bin_pos_weight, double *bin_psum,
                                                               int64_t *words_out) {
  return quality_request<true, true>(ctx, w, drawn_rows(row_begin, row_end, key, pos_begin, pos_end), __func__, 0.0, 0.0, X,
                                     Y, k, n_bins, sums_out, bin_weight, bin_pos_weight, bin_psum, words_out);
}

extern "C" int dsgd_eval_samples_weighted_isotonic_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples,
                                                               int64_t n, const double *X, const double *Y, int64_t k,
                                                               int32_t n_bins, double *sums_out, double *bin_weight,
                                                               double *bin_pos_weight, double *bin_psum,
                                                               int64_t *words_out) {
  return quality_request<true, true>(ctx, w, listed_rows(samples, n), __func__, 0.0, 0.0, X, Y, k, n_bins, sums_out,
                                     bin_weight, bin_pos_weight, bin_psum, words_out);
}

// Diagnostic: rows the streaming pass recomputed in fp64 because their fp32 dot was inside the rounding band (all
// streaming passes of this ctx so far: forward, gradient, and the full and sampled evaluations).
extern "C" int dsgd_stream_exact_rows(dsgd_ctx *ctx, int64_t *rows) {
  if (!ctx || !rows) return DSGD_ERR_INVALID;
  unsigned long long host = 0;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaMemcpy(&host, ctx->n_exact, sizeof host, cudaMemcpyDeviceToHost));
  *rows = (int64_t)host;
  return DSGD_OK;
}

// ---- sync mode -------------------------------------------------------------------------------------------

extern "C" int dsgd_comm_unique_id(uint8_t id[DSGD_UNIQUE_ID_BYTES]) {
  static_assert(sizeof(ncclUniqueId) == DSGD_UNIQUE_ID_BYTES, "ncclUniqueId size");
  if (!id) return DSGD_ERR_INVALID;
  if (!nccl().ok) return fail(nullptr, DSGD_ERR_NCCL, "%s", nccl().why.c_str());
  ncclUniqueId u;
  ncclResult_t r = nccl().GetUniqueId(&u);
  if (r != ncclSuccess) return fail(nullptr, DSGD_ERR_NCCL, "ncclGetUniqueId: %s", nccl().GetErrorString(r));
  memcpy(id, &u, sizeof u);
  return DSGD_OK;
}

extern "C" int dsgd_comm_init(dsgd_ctx *ctx, const uint8_t id[DSGD_UNIQUE_ID_BYTES]) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(id, DSGD_ERR_INVALID, "dsgd_comm_init: id is NULL");
  NEED(!ctx->comm, DSGD_ERR_STATE, "dsgd_comm_init: communicator already initialised");
  CU(cudaSetDevice(ctx->device));
  ncclUniqueId u;
  memcpy(&u, id, sizeof u);
  NEED(nccl().ok, DSGD_ERR_NCCL, "%s", nccl().why.c_str());
  NC(nccl().CommInitRank(&ctx->comm, ctx->world, u, ctx->rank));
  return DSGD_OK;
}

// ---- persistent sync loop (dsgd_persistent.cuh) ----------------------------------------------------------------
constexpr int kPCons = 8, kPUpd = 6, kPStages = 8, kPStagePairs = 2560, kPMaxChunks = 128;
using PSmem = PersistSmem<kPCons, kPUpd, kPStages, kPStagePairs, kPMaxChunks>;
// Every instantiation of k_sync_persistent: the one-GPU forms f = 8 weighting + 4 l1 + 2 avg + lr_table (0..23), and the
// fused K-GPU kernel (multi), which has no L1 or weighted form, f = 24 + 2 avg + lr_table: exactly 28 forms.
constexpr int kPersistForms = 28, kPersistFused = 24;
constexpr bool pf_multi(int f) { return f >= kPersistFused; }
constexpr int pf_weight(int f) { return pf_multi(f) ? kUnweighted : f / 8; }
constexpr bool pf_l1(int f) { return (f & 4) != 0; }   // never set in a fused form
template <int... F>
static void *const *persist_forms(std::integer_sequence<int, F...>) {
  static void *const k[] = {(void *)k_sync_persistent<kPCons, kPUpd, kPStages, kPStagePairs, kPMaxChunks, pf_multi(F),
                                                      (F & 2) != 0, (F & 1) != 0, pf_l1(F), pf_weight(F)>...};
  return k;
}
static void *const *const kPersistKernels = persist_forms(std::make_integer_sequence<int, kPersistForms>{});
// The form that runs a launch with these options; l1 and weight are not read for the fused kernel.
static int persist_form(bool multi, bool avg, bool lr_table, bool l1, int weight) {
  if (multi) return kPersistFused + 2 * avg + lr_table;
  return 8 * weight + 4 * l1 + 2 * avg + lr_table;
}
// Dynamic shared memory of form f: the sample-weighted forms keep their combined weights and hinge codes past PSmem
static size_t persist_smem(int f) {
  return sizeof(PSmem) + (pf_weight(f) == kSampleWeighted ? sizeof(PersistSwSmem<kPStages>) : 0);
}
static bool persist_timeline() { static const bool v = getenv("DSGD_PERSIST_TIMELINE") != nullptr; return v; }

static int persist_prepare(dsgd_ctx *ctx, int64_t n_steps) {
  if (!ctx->p_ready) {
    const int64_t nv = (int64_t)ctx->dim + 2;
    const size_t vd = sizeof(double) * (size_t)nv;
    for (int i = 0; i < 2; ++i) CU(ctx->p_wbuf[i].alloc(nv));
    for (int i = 0; i < 3; ++i) {
      CU(ctx->p_gbuf[i].alloc(nv));
      CU(cudaMemsetAsync(ctx->p_gbuf[i], 0, vd, ctx->stream));
      CU(ctx->p_rec[i].alloc(nv));
      CU(cudaMemsetAsync(ctx->p_rec[i], 0, 2 * vd, ctx->stream));
    }
    CU(ctx->p_acc.alloc(3 * kAccStride));
    CU(ctx->p_bar.alloc(4));
    for (int f = 0; f < kPersistForms; ++f)
      CU(cudaFuncSetAttribute(kPersistKernels[f], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)persist_smem(f)));
    ctx->p_ready = true;
  }
  // sized for the largest grid (persist_grid), which dsgd_reserve does not know yet
  int rc = ctx->p_hinge.grow(ctx, (int64_t)ctx->sm_count * n_steps, 4096 * (int64_t)ctx->sm_count);
  if (rc) return rc;
  // the hinge codes of the sample-weighted forms, only while sample weights are loaded
  if (weighting(ctx) == kSampleWeighted &&
      (rc = ctx->p_hcode.grow(ctx, (int64_t)ctx->sm_count * n_steps, 4096 * (int64_t)ctx->sm_count)))
    return rc;
  return ctx->p_loss_nrm.grow(ctx, 2 * n_steps, 2 * 4096);
}

// CTAs of the persistent kernel: one per SM (fastest at batch 64, 256 and 1024 when it was
// measured); every CTA owns at most kMaxRowsPerCta rows of a step.  0: the batch is too large for this kernel.
static int persist_grid(const dsgd_ctx *ctx, int64_t batch) {
  const int g = ctx->grid_limit > 0 ? std::min(ctx->grid_limit, ctx->sm_count) : ctx->sm_count;
  if (cdiv(batch, kMaxRowsPerCta) > g) return 0;
  if (ctx->n_pairs >= (1ll << 31)) return 0;  // chunk descriptors carry a 31-bit global pair index
  return g;
}
// K GPUs: one column of the CTA's slice per barrier-synchronised thread
static bool persist_multi_fits(const dsgd_ctx *ctx, int G) {
  const int slice = (cdiv(ctx->dim + 1, G) + 31) & ~31;
  return slice <= (kPCons + kPUpd) * 32;
}

// The kernel synchronises its CTAs itself, so all of them must be resident: a cooperative launch guarantees that.  With a
// grid limit (several contexts sharing one GPU: the K-rank tests on one device) the kernels of the ranks must also run
// CONCURRENTLY, which cooperative launches of different contexts do not (measured: they serialise and the ranks time
// out waiting for each other); a plain launch of at most one CTA per SM on an otherwise idle GPU is resident in full too.
static cudaError_t persist_launch(dsgd_ctx *ctx, int form, int G, void **args) {
  void *fn = kPersistKernels[form];
  const size_t smem = persist_smem(form);
  if (ctx->grid_limit > 0) return cudaLaunchKernel(fn, dim3(G), dim3((kPCons + kPUpd + 1) * 32), args, smem, ctx->stream);
  return cudaLaunchCooperativeKernel(fn, dim3(G), dim3((kPCons + kPUpd + 1) * 32), args, smem, ctx->stream);
}

// ---- fused K-GPU loop: all ranks run the persistent kernel and exchange gradients through peer memory ----
// exported block of a rank (in 8-byte words): value words [sender][parity][dim + 8] x 2, then bitmap words
// [sender][parity][ceil((dim + 1) / 32)]
static size_t xblk_stride(const dsgd_ctx *ctx) { return (size_t)(ctx->dim + kReplicaPad); }
static size_t xblk_words(const dsgd_ctx *ctx) { return ((size_t)ctx->dim + 1 + 31) / 32; }
static size_t xblk_bm_offset(const dsgd_ctx *ctx) { return 2 * (size_t)kMaxWorld * 2 * xblk_stride(ctx); }
static size_t xblk_doubles(const dsgd_ctx *ctx) { return xblk_bm_offset(ctx) + (size_t)kMaxWorld * 2 * xblk_words(ctx); }

static int xblk_ensure(dsgd_ctx *ctx) {
  if (ctx->xblk) return DSGD_OK;
  CU(cudaSetDevice(ctx->device));
  CU(ctx->xblk.alloc((int64_t)xblk_doubles(ctx)));
  CU(cudaMemset(ctx->xblk, 0, sizeof(double) * xblk_doubles(ctx)));
  CU(ctx->x_stats.alloc(4));
  CU(cudaMemset(ctx->x_stats, 0, sizeof(unsigned long long) * 4));
  return DSGD_OK;
}

static int xllw_ensure(dsgd_ctx *ctx) {
  if (ctx->x_llw) return DSGD_OK;
  CU(ctx->x_llw.alloc(2 * 2 * (int64_t)xblk_stride(ctx)));
  CU(cudaMemsetAsync(ctx->x_llw, 0, 2 * 2 * sizeof(unsigned long long) * xblk_stride(ctx), ctx->stream));
  return DSGD_OK;
}

static bool xchg_complete(const dsgd_ctx *ctx) {
  if (ctx->world <= 1 || ctx->world > kMaxWorld || !ctx->xblk) return false;
  for (int r = 0; r < ctx->world; ++r)
    if (r != ctx->rank && !ctx->peer_x[r]) return false;
  return true;
}

// One launch of the persistent kernel for n_steps SGD steps: on one GPU, or (multi) the fused K-GPU kernel in which every
// rank aggregates the gradients through the exchange blocks of its peers.  lrs_host (n_steps host values) or nullptr: the
// per-step rates of dsgd_sync_steps_lr, or the scalar lr for every step.
static int persist_run(dsgd_ctx *ctx, bool multi, const int32_t *samples_dev, int64_t n_per_step, int64_t n_steps,
                       double lr, const double *lrs_host, double *losses_dev) {
  int rc = persist_prepare(ctx, n_steps);
  if (rc) return rc;
  const int G = persist_grid(ctx, n_per_step);
  NEED((uint64_t)G * (uint64_t)(n_steps + 2) < (1ull << 32), DSGD_ERR_INVALID, "dsgd_sync_steps: too many steps for one launch");
  PersistParams pp;
  memset(&pp, 0, sizeof pp);
  pp.rp16 = ctx->rp16; pp.pairs = ctx->pairs; pp.label = ctx->label; pp.samples = samples_dev;
  pp.n_steps = n_steps; pp.batch = (int32_t)n_per_step; pp.dim = ctx->dim;
  pp.wbuf[0] = ctx->p_wbuf[0]; pp.wbuf[1] = ctx->p_wbuf[1];
  for (int i = 0; i < 3; ++i) { pp.gbuf[i] = ctx->p_gbuf[i]; pp.rec[i] = ctx->p_rec[i]; }
  pp.d = ctx->d; pp.acc = ctx->p_acc; pp.bar = ctx->p_bar; pp.hinge = ctx->p_hinge; pp.losses = losses_dev;
  pp.loss_nrm = ctx->p_loss_nrm;
  pp.w_out = ctx->w; pp.w32_out = ctx->w32; pp.scal = ctx->scal;
  pp.abort_flag = reinterpret_cast<int *>(ctx->p_bar + 1);
  CU(cudaMemsetAsync(ctx->p_acc, 0, sizeof(unsigned long long) * 3 * kAccStride, ctx->stream));
  pp.lambda = ctx->lambda; pp.lr = lr; pp.world = 1;
  CU(cudaMemsetAsync(ctx->p_bar, 0, sizeof(unsigned) * 4, ctx->stream));
  if (persist_timeline()) {
    if (!ctx->p_tl) CU(ctx->p_tl.alloc(kTlWords));
    CU(cudaMemsetAsync(ctx->p_tl, 0, sizeof(long long) * kTlWords, ctx->stream));
    pp.tl = ctx->p_tl;
  }
  if (!multi) {
    k_rec_init<<<cdiv(ctx->dim, 256), 256, 0, ctx->stream>>>(ctx->w, ctx->dim, ctx->p_rec[0], ctx->p_rec[1], ctx->p_rec[2]);
    LAUNCHED();
    pp.k_den = 1.0;
    pp.timeout_cycles = 4000000000ll;  // ~2 s at 1.9 GHz: a healthy barrier takes well under a microsecond
  } else {
    // the kernel's first interval reads the host-provided weights from wbuf[0] and publishes them in LL form
    CU(cudaMemcpyAsync(ctx->p_wbuf[0], ctx->w, sizeof(double) * (size_t)ctx->dim, cudaMemcpyDeviceToDevice, ctx->stream));
    pp.k_den = (double)ctx->world;
    pp.timeout_cycles = 20000000000ll;  // ~10 s: covers a peer that launches late
    pp.world = ctx->world; pp.rank = ctx->rank; pp.step_base = ctx->x_step;
    pp.xstride = (int)xblk_stride(ctx);
    pp.xwords = (int)xblk_words(ctx);
    for (int r = 0; r < ctx->world; ++r) {
      unsigned long long *blk = reinterpret_cast<unsigned long long *>((r == ctx->rank) ? ctx->xblk.p : ctx->peer_x[r].p);
      pp.xval[r] = blk;
      pp.xbm[r] = blk + xblk_bm_offset(ctx);
    }
    if ((rc = xllw_ensure(ctx))) return rc;
    pp.llw[0] = ctx->x_llw;
    pp.llw[1] = ctx->x_llw + 2 * xblk_stride(ctx);
    pp.xstats = ctx->x_stats;
  }
  // The averaging instantiations only while averaging is on, the table ones only for a table: otherwise the kernels of
  // before run.
  if (ctx->avg_on) pp.avg = ctx->avg;
  if (lrs_host) {
    if ((rc = ctx->lrs.grow(ctx, n_steps, 1024))) return rc;
    CU(cudaMemcpyAsync(ctx->lrs, lrs_host, sizeof(double) * (size_t)n_steps, cudaMemcpyHostToDevice, ctx->stream));
    pp.lrs = ctx->lrs;
    pp.lr = 0.0;   // not read: interval 0, the only one before lrs[0] is loaded, applies no update
  }
  void *args[] = {&pp};
  // the L1 forms only with a penalty, the weighted forms only in the ctx's weighting (none fused: sync_staged keeps such a
  // ctx off the fused path)
  const bool l1 = !multi && ctx->lambda1 > 0.0;
  pp.lambda1 = l1 ? ctx->lambda1 : 0.0;
  pp.w_pos = ctx->cw_pos; pp.w_neg = ctx->cw_neg;
  const int weight = multi ? kUnweighted : weighting(ctx);
  if (weight == kSampleWeighted) { pp.sw = ctx->sw; pp.hcode = ctx->p_hcode; }
  const int form = persist_form(multi, ctx->avg_on, lrs_host != nullptr, l1, weight);
  cudaError_t launch_err = cudaSuccess;
  profiled(ctx, [&] { launch_err = persist_launch(ctx, form, G, args); });
  CU(launch_err);
  LAUNCHED();
  if (ctx->avg_on) ctx->avg_n += n_steps;
  if (multi) {
    // The next launch must not meet LL words carrying tags this one used (the host may install new weights in between): the
    // step counter jumps.  By 6: a multiple of 3 keeps the rotation of the three gradient buffers (the dirty one is re-zeroed
    // before use), and an EVEN jump makes the first push of launch n+1 (its second interval) land in the receive parity that
    // a slow peer is NOT reading in launch n's last interval (+3 put them on the same one: ADVICE.md round 1).
    ctx->x_step += n_steps + 6;
    ctx->x_steps_run += n_steps;
  }
  return DSGD_OK;
}

extern "C" int dsgd_reserve(dsgd_ctx *ctx, int64_t n_samples, int64_t n_steps) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n_samples >= 0 && n_steps >= 0, DSGD_ERR_INVALID, "dsgd_reserve: negative size");
  CU(cudaSetDevice(ctx->device));
  int rc = ctx->samples.grow(ctx, n_samples, 1024);
  if (rc) return rc;
  if ((rc = ctx->losses.grow(ctx, n_steps, 1024))) return rc;
  if ((rc = ctx->lrs.grow(ctx, n_steps, 1024))) return rc;
  if ((rc = persist_prepare(ctx, n_steps))) return rc;
  if (persist_timeline() && !ctx->p_tl) CU(ctx->p_tl.alloc(kTlWords));
  if (ctx->world > 1 && !(ctx->flags & DSGD_FLAG_ASYNC)) {
    if ((rc = xblk_ensure(ctx))) return rc;
    if ((rc = xllw_ensure(ctx))) return rc;
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_set_grid_limit(dsgd_ctx *ctx, int32_t n_ctas) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n_ctas >= 0, DSGD_ERR_INVALID, "dsgd_set_grid_limit: negative");
  ctx->grid_limit = n_ctas;
  return DSGD_OK;
}

// Diagnostic for the bandwidth figures of the fused K-GPU step: words this rank has pushed to EACH peer so far (a value word
// is 16 bytes on the wire, a bitmap word 8) and the SGD steps of those launches.
extern "C" int dsgd_xchg_stats(dsgd_ctx *ctx, int64_t *value_words, int64_t *bitmap_words, int64_t *steps) {
  if (!ctx) return DSGD_ERR_INVALID;
  unsigned long long host[2] = {0, 0};
  if (ctx->x_stats) {
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(host, ctx->x_stats, sizeof host, cudaMemcpyDeviceToHost, ctx->stream));   // see persist_check
    CU(cudaStreamSynchronize(ctx->stream));
  }
  if (value_words) *value_words = (int64_t)host[0];
  if (bitmap_words) *bitmap_words = (int64_t)host[1];
  if (steps) *steps = ctx->x_steps_run;
  return DSGD_OK;
}

// ---- peer memory: buffers of other ranks, mapped from another process or attached from this one ----

static int open_ipc(dsgd_ctx *ctx, peer_ptr &slot, const uint8_t handle[DSGD_IPC_HANDLE_BYTES]) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof h);
  void *ptr = nullptr;
  CU(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
  slot.set(static_cast<double *>(ptr), true);
  return DSGD_OK;
}

// makes ctx's device current and lets it address the memory of peer's device
static int enable_peer_access(dsgd_ctx *ctx, const dsgd_ctx *peer, const char *who) {
  CU(cudaSetDevice(ctx->device));
  if (peer->device == ctx->device) return DSGD_OK;
  int can = 0;
  CU(cudaDeviceCanAccessPeer(&can, ctx->device, peer->device));
  NEED(can, DSGD_ERR_CUDA, "%s: device %d cannot access device %d", who, ctx->device, peer->device);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer->device, 0);
  if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU(e);
  (void)cudaGetLastError();
  return DSGD_OK;
}

extern "C" int dsgd_xchg_export(dsgd_ctx *ctx, uint8_t handle[DSGD_IPC_HANDLE_BYTES]) {
  if (!ctx || !handle) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "dsgd_xchg_export: ctx is in async mode");
  int rc = xblk_ensure(ctx);
  if (rc) return rc;
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, ctx->xblk));
  memcpy(handle, &h, sizeof h);
  return DSGD_OK;
}

extern "C" int dsgd_xchg_import(dsgd_ctx *ctx, int peer_rank, const uint8_t handle[DSGD_IPC_HANDLE_BYTES]) {
  if (!ctx || !handle) return DSGD_ERR_INVALID;
  NEED(peer_rank >= 0 && peer_rank < ctx->world && peer_rank < kMaxWorld && peer_rank != ctx->rank, DSGD_ERR_INVALID,
       "dsgd_xchg_import: bad peer rank %d", peer_rank);
  int rc = xblk_ensure(ctx);
  if (rc) return rc;
  return open_ipc(ctx, ctx->peer_x[peer_rank], handle);
}

extern "C" int dsgd_xchg_attach(dsgd_ctx *ctx, int peer_rank, dsgd_ctx *peer) {
  if (!ctx || !peer) return DSGD_ERR_INVALID;
  NEED(peer_rank >= 0 && peer_rank < ctx->world && peer_rank < kMaxWorld && peer_rank != ctx->rank, DSGD_ERR_INVALID,
       "dsgd_xchg_attach: bad peer rank %d", peer_rank);
  NEED(peer->dim == ctx->dim, DSGD_ERR_INVALID, "dsgd_xchg_attach: dimension mismatch");
  int rc = xblk_ensure(ctx);
  if (rc) return rc;
  if ((rc = xblk_ensure(peer))) { ctx->err = peer->err; return rc; }
  if ((rc = enable_peer_access(ctx, peer, "dsgd_xchg_attach"))) return rc;
  ctx->peer_x[peer_rank].set(peer->xblk, false);
  return DSGD_OK;
}

static int persist_check(dsgd_ctx *ctx) {  // after a stream sync: did a device-side wait hit its watchdog?
  if (!ctx->p_ready) return DSGD_OK;
  unsigned host[2] = {0, 0};
  // On this ctx's stream, not the legacy default stream: ranks sharing one GPU each run on their own stream, and a rank
  // reads this between two launches while a peer's next launch already spins waiting for it.  The legacy stream can share a
  // hardware queue with that peer's stream; a copy queued behind the spinning kernel holds this rank back until the peer's
  // watchdog ends it, and both launches fail with DSGD_ERR_TIMEOUT.
  CU(cudaMemcpyAsync(host, ctx->p_bar, sizeof host, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  NEED(host[1] == 0, DSGD_ERR_TIMEOUT, "persistent sync kernel: a device-side wait (grid barrier, peer word) hit its watchdog");
  return DSGD_OK;
}

// Debug: copies the last persistent run's timeline out (include/dsgd.h); needs DSGD_PERSIST_TIMELINE.
static_assert(kTlWords == DSGD_TIMELINE_WORDS, "timeline layout");
extern "C" int dsgd_debug_timeline(dsgd_ctx *ctx, long long *out) {
  if (!ctx || !out) return DSGD_ERR_INVALID;
  NEED(ctx->p_tl, DSGD_ERR_STATE, "no timeline recorded (set DSGD_PERSIST_TIMELINE=1)");
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaMemcpy(out, ctx->p_tl, sizeof(long long) * kTlWords, cudaMemcpyDeviceToHost));
  return DSGD_OK;
}

extern "C" int dsgd_set_workers(dsgd_ctx *ctx, int32_t n_local, const int32_t *counts, int32_t k_total) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(n_local >= 0 && k_total >= 0, DSGD_ERR_INVALID, "dsgd_set_workers: negative count");
  NEED(n_local <= 1 || counts, DSGD_ERR_INVALID, "dsgd_set_workers: counts is NULL");
  std::vector<int32_t> c;
  if (counts)
    for (int32_t v = 0; v < n_local; ++v) {
      NEED(counts[v] > 0, DSGD_ERR_EMPTY, "dsgd_set_workers: worker %d has an empty batch (Vec.sum of an empty list throws)", v);
      c.push_back(counts[v]);
    }
  ctx->worker_counts = c;
  ctx->n_local = n_local;
  ctx->k_total = k_total;
  return DSGD_OK;
}

// The per-step path of sync_staged for model kModel: n_steps steps of n_per_step staged ids from smp, step s at the rate
// lrs[s] (lrs == nullptr: lr), its loss into losses[s] (losses == nullptr: none)
// kWeight: every worker's pass is k_rows in that weighting (a weighted one followed by its fold, k_class_fold or
// k_sw_fold), and the tails of a weighted pass (kCw) read its weighted loss sum
// kIcpt: an intercept ctx; its gradient slot g[dim + kIcptSlot] widens the workers' sum and the allreduce by one entry
template <int kModel, int kWeight, bool kIcpt>
static int sync_per_step(dsgd_ctx *ctx, const int32_t *smp, int64_t n_per_step, int64_t n_steps, double lr,
                         const double *lrs, double *losses, bool single, int32_t k_total) {
  const int upd_blocks = cdiv(ctx->dim, 256);
  const int fin_blocks = cdiv(ctx->dim + 1, 256);
  constexpr bool kCw = kWeight != kUnweighted;
  double lr_s = lr;   // the rate of step s
  // The update of every step, in the form of this call [single][avg][l1]: one worker regularizes its raw gradient in the
  // update; while averaging the update also adds the new weights to avg; with an L1 penalty it soft-thresholds every column.
  using Update = decltype(&k_update<true, kModel, false, false, kCw, kIcpt>);
  static const Update kUpdate[2][2][2] = {
      {{k_update<false, kModel, false, false, kCw, kIcpt>, k_update<false, kModel, false, true, kCw, kIcpt>},
       {k_update<false, kModel, true, false, kCw, kIcpt>, k_update<false, kModel, true, true, kCw, kIcpt>}},
      {{k_update<true, kModel, false, false, kCw, kIcpt>, k_update<true, kModel, false, true, kCw, kIcpt>},
       {k_update<true, kModel, true, false, kCw, kIcpt>, k_update<true, kModel, true, true, kCw, kIcpt>}}};
  const size_t g_words = (size_t)ctx->dim + (kIcpt ? kIcptSlot + 1 : 2);
  const Update update = kUpdate[single][ctx->avg_on][ctx->lambda1 > 0.0];
  double *const avg = ctx->avg_on ? ctx->avg.p : nullptr;

  for (int64_t s = 0; s < n_steps; ++s, smp += n_per_step) {
    if (lrs) lr_s = lrs[s];
    double *loss_dev = losses ? losses + s : nullptr;
    double *gbuf = ctx->g;
    double k_den = 1.0, n_local = (double)n_per_step;
    if (single) {
      // one worker, one GPU: gradient -> (regularize + update) fused, two launches per step
      int rc = DSGD_OK;
      profiled(ctx, [&] {
        rc = launch_rows<kModel, kWeight, true, false, kIcpt>(ctx, {smp, 0, n_per_step}, ctx->w, nullptr, ctx->g);
      });
      if (rc) return rc;
    } else {
      // several workers or ranks: each worker's gradient, regularized and folded into gsum, then the allreduce and the update
      int64_t off = 0;
      for (int32_t v = 0; v < ctx->n_local; ++v) {
        const int64_t nv = ctx->worker_counts.empty() ? n_per_step : ctx->worker_counts[(size_t)v];
        int rc = DSGD_OK;
        profiled(ctx, [&] {
          rc = launch_rows<kModel, kWeight, true, false, kIcpt>(ctx, {smp + off, 0, nv}, ctx->w, nullptr, ctx->g);
        });
        if (rc) return rc;
        k_finish_acc<kModel, kCw, kIcpt><<<fin_blocks, 256, 0, ctx->stream>>>(ctx->g, ctx->gsum, ctx->dim, ctx->scal + kScalC,
                                                                       ctx->cnt, (double)nv, v == 0 ? 1 : 0);
        LAUNCHED();
        off += nv;
      }
      if (ctx->n_local == 0) CU(cudaMemsetAsync(ctx->gsum, 0, sizeof(double) * g_words, ctx->stream));
      if (ctx->world > 1) NC(nccl().AllReduce(ctx->gsum, ctx->gsum, g_words, ncclDouble, ncclSum, ctx->comm, ctx->stream));
      gbuf = ctx->gsum;
      k_den = (double)k_total;
      n_local = 0.0;
    }
    update<<<upd_blocks, 256, 0, ctx->stream>>>(ctx->w, ctx->w32, gbuf, ctx->d, ctx->dim, ctx->lambda, lr_s, k_den, ctx->scal,
                                                ctx->cnt, ctx->partial, n_local, loss_dev, avg, ctx->lambda1);
    LAUNCHED();
    if (ctx->avg_on) ++ctx->avg_n;
  }
  CU(cudaGetLastError());
  return DSGD_OK;
}

// The sync steps of dsgd_sync_steps_staged, and of dsgd_sync_steps_lr with lrs (n_steps host values, step s takes lrs[s])
// instead of the scalar lr.  The per-step paths pass each step's rate as the kernel argument they always take; the
// persistent and fused kernels read the table on the device (persist_run).
static int sync_staged(dsgd_ctx *ctx, int64_t first, int64_t n_per_step, int64_t n_steps, double lr, const double *lrs,
                       int want_losses) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "sync step on a ctx created in async mode");
  NEED(ctx->have_d, DSGD_ERR_STATE, "dsgd_sync_steps: dimSparsity not set");
  NEED(n_steps >= 0 && first >= 0, DSGD_ERR_INVALID, "dsgd_sync_steps: bad arguments");
  NEED(n_per_step >= 0, DSGD_ERR_INVALID, "dsgd_sync_steps: bad arguments");
  NEED(first + n_per_step * n_steps <= ctx->samples_n, DSGD_ERR_RANGE, "dsgd_sync_steps: staged samples exhausted");
  NEED(ctx->world == 1 || ctx->comm || xchg_complete(ctx), DSGD_ERR_STATE,
       "dsgd_sync_steps: world > 1 but neither dsgd_comm_init nor the peer exchange (dsgd_xchg_*) was set up");
  if (ctx->n_local == 0) {
    NEED(n_per_step == 0, DSGD_ERR_INVALID, "dsgd_sync_steps: a bystander rank (n_local == 0) takes no samples");
  } else {
    NEED(n_per_step > 0, DSGD_ERR_EMPTY, "dsgd_sync_steps: empty batch (Vec.sum of an empty list throws in the reference)");
    if (!ctx->worker_counts.empty()) {
      int64_t tot = 0;
      for (int32_t c : ctx->worker_counts) tot += c;
      NEED(tot == n_per_step, DSGD_ERR_INVALID, "dsgd_sync_steps: n_per_step %lld != sum of worker counts %lld",
           (long long)n_per_step, (long long)tot);
    }
  }
  const int32_t k_total = ctx->k_total > 0 ? ctx->k_total : ctx->world;
  const bool single = (ctx->world == 1 && ctx->n_local == 1 && k_total == 1);
  // The options the fused kernel has no form of, which with world > 1 take the per-step path over NCCL: the persistent and
  // fused kernels are SVM-only (a ctx of any other model always takes the per-step path below), and an L1 penalty, class
  // weights or sample weights have only one-GPU persistent forms.  An intercept has no persistent form at all: an intercept
  // ctx always takes the per-step path.  unfused names the first of them that is on.
  static const char *const kModelTakes[] = {nullptr, "the logistic model takes", "the squared_hinge model takes",
                                            "the modified_huber model takes"};
  const int model = model_of(ctx);
  const int weight = weighting(ctx);
  const char *unfused = model != kSvm ? kModelTakes[model]
                        : has_icpt(ctx) ? "the intercept takes"
                        : ctx->lambda1 > 0.0 ? "the L1 penalty takes"
                        : has_class_weights(ctx) ? "class weights take"
                        : weight == kSampleWeighted ? "sample weights take" : nullptr;
  NEED(!unfused || ctx->world == 1 || ctx->comm || n_steps == 0, DSGD_ERR_STATE,
       "dsgd_sync_steps: %s the NCCL allreduce path for world > 1, which needs dsgd_comm_init", unfused);
  const bool fused = !unfused && ctx->world > 1 && ctx->n_local == 1 && k_total == ctx->world && n_steps > 0 && xchg_complete(ctx) &&
                     persist_grid(ctx, n_per_step) > 0 && persist_multi_fits(ctx, persist_grid(ctx, n_per_step));
  // Ranks wired with the peer exchange only have no communicator for the step-by-step path below: refuse before anything
  // is launched instead of reaching the allreduce without one.
  NEED(ctx->world == 1 || ctx->comm || n_steps == 0 || fused, DSGD_ERR_STATE,
       "dsgd_sync_steps: world > 1 without dsgd_comm_init, and the fused peer-exchange kernel cannot take this step "
       "(it needs one worker per rank, batch <= %d x %d CTAs and dim + 1 <= %d x CTAs; batch %lld, dim %d)",
       kMaxRowsPerCta, ctx->grid_limit > 0 ? std::min(ctx->grid_limit, ctx->sm_count) : ctx->sm_count,
       (kPCons + kPUpd) * 32, (long long)n_per_step, ctx->dim);
  CU(cudaSetDevice(ctx->device));
  if (want_losses) {
    int rc = ctx->losses.grow(ctx, n_steps, 1024);
    if (rc) return rc;
  }
  if ((single && model == kSvm && !has_icpt(ctx) && n_steps > 0 && persist_grid(ctx, n_per_step) > 0) || fused) {
    // one worker on one GPU: the whole run of steps is one persistent cooperative kernel; one worker per GPU, every peer's
    // exchange block mapped (fused): the same kernel aggregates over NVLink
    return persist_run(ctx, fused, ctx->samples + first, n_per_step, n_steps, lr, lrs,
                       want_losses ? ctx->losses.p : nullptr);
  }
  const int32_t *smp = ctx->samples + first;
  double *loss_dev = want_losses ? ctx->losses.p : nullptr;
  return with_forms(ctx, weight, [&](auto m, auto wt, auto ic) {
    return sync_per_step<m, wt, ic>(ctx, smp, n_per_step, n_steps, lr, lrs, loss_dev, single, k_total);
  });
}

extern "C" int dsgd_sync_steps_staged(dsgd_ctx *ctx, int64_t first, int64_t n_per_step, int64_t n_steps, double lr,
                                      int want_losses) {
  return sync_staged(ctx, first, n_per_step, n_steps, lr, nullptr, want_losses);
}

extern "C" int dsgd_read_losses(dsgd_ctx *ctx, double *losses_out, int64_t n_steps) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(losses_out && n_steps >= 0 && n_steps <= ctx->losses.cap, DSGD_ERR_INVALID, "dsgd_read_losses: bad arguments");
  CU(cudaSetDevice(ctx->device));
  if (n_steps)
    CU(cudaMemcpyAsync(losses_out, ctx->losses, sizeof(double) * (size_t)n_steps, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return persist_check(ctx);
}

// dsgd_sync_steps, and dsgd_sync_steps_lr with lrs != nullptr
static int sync_steps(dsgd_ctx *ctx, const int32_t *samples, int64_t n_per_step, int64_t n_steps, double lr,
                      const double *lrs, double *losses_out) {
  NEED(n_steps >= 0 && n_per_step >= 0, DSGD_ERR_INVALID, "dsgd_sync_steps: bad arguments");
  NEED(n_per_step > 0 || ctx->n_local == 0, DSGD_ERR_EMPTY,
       "dsgd_sync_steps: empty batch (Vec.sum of an empty list throws in the reference)");
  int rc = dsgd_stage_samples(ctx, samples, n_per_step * n_steps);
  if (rc) return rc;
  if ((rc = sync_staged(ctx, 0, n_per_step, n_steps, lr, lrs, losses_out != nullptr))) return rc;
  if (losses_out) return dsgd_read_losses(ctx, losses_out, n_steps);
  CU(cudaStreamSynchronize(ctx->stream));
  return persist_check(ctx);
}

extern "C" int dsgd_sync_steps(dsgd_ctx *ctx, const int32_t *samples, int64_t n_per_step, int64_t n_steps, double lr,
                               double *losses_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  return sync_steps(ctx, samples, n_per_step, n_steps, lr, nullptr, losses_out);
}

extern "C" int dsgd_sync_steps_lr(dsgd_ctx *ctx, const int32_t *samples, int64_t n_per_step, int64_t n_steps,
                                  const double *lrs, double *losses_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "dsgd_sync_steps_lr: ctx is in async mode (Hogwild keeps its constant rate)");
  NEED(lrs || n_steps <= 0, DSGD_ERR_INVALID, "dsgd_sync_steps_lr: lrs is NULL");
  return sync_steps(ctx, samples, n_per_step, n_steps, 0.0, lrs, losses_out);
}

extern "C" int dsgd_sync_step(dsgd_ctx *ctx, const int32_t *samples, int64_t n, double lr, double *loss_out) {
  return dsgd_sync_steps(ctx, samples, n, 1, lr, loss_out);
}

// ---- the L1 penalty of the sync steps (dsgd_set_l1) and the L1 norm of a weight vector ----------------------------------

extern "C" int dsgd_set_l1(dsgd_ctx *ctx, double lambda1) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE,
       "dsgd_set_l1: ctx is in async mode (the L1 penalty is a step of the sync paths; Hogwild has no step order)");
  NEED(std::isfinite(lambda1) && lambda1 >= 0.0, DSGD_ERR_INVALID, "dsgd_set_l1: lambda1 must be finite and >= 0 (got %g)",
       lambda1);
  // scal[kScalL1] is kept only while the penalty is on: every step of an L1 ctx and dsgd_set_weights keep it from here on
  if (lambda1 > 0.0 && !(ctx->lambda1 > 0.0)) {
    CU(cudaSetDevice(ctx->device));
    launch_l1_refresh(ctx);
    CU(cudaGetLastError());
  }
  ctx->lambda1 = lambda1;
  return DSGD_OK;
}

// ---- class weights of the sync steps and of dsgd_gradient ------------------------------------------------------------------

extern "C" int dsgd_set_class_weights(dsgd_ctx *ctx, double w_pos, double w_neg) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE,
       "dsgd_set_class_weights: ctx is in async mode (class weights belong to the sync paths)");
  NEED(std::isfinite(w_pos) && w_pos >= 0.0 && std::isfinite(w_neg) && w_neg >= 0.0, DSGD_ERR_INVALID,
       "dsgd_set_class_weights: weights must be finite and >= 0 (got %g, %g)", w_pos, w_neg);
  ctx->cw_pos = w_pos;
  ctx->cw_neg = w_neg;
  return DSGD_OK;
}

extern "C" int dsgd_get_class_weights(const dsgd_ctx *ctx, double *w_pos_out, double *w_neg_out) {
  if (!ctx || !w_pos_out || !w_neg_out) return DSGD_ERR_INVALID;
  *w_pos_out = ctx->cw_pos;
  *w_neg_out = ctx->cw_neg;
  return DSGD_OK;
}

// ---- sample weights of the sync steps, of dsgd_gradient and of dsgd_eval*_weighted -------------------------------------

extern "C" int dsgd_set_sample_weights(dsgd_ctx *ctx, const double *sw, int64_t n) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE,
       "dsgd_set_sample_weights: ctx is in async mode (sample weights belong to the sync paths)");
  NEED(ctx->pairs, DSGD_ERR_STATE, "dsgd_set_sample_weights: no rows loaded");
  if (!sw && n == 0) {
    ctx->sw_on = false;
    return DSGD_OK;
  }
  NEED(sw && n == ctx->n_rows, DSGD_ERR_INVALID, "dsgd_set_sample_weights: %lld weights for %lld loaded rows", (long long)n,
       (long long)ctx->n_rows);
  for (int64_t i = 0; i < n; ++i)
    NEED(std::isfinite(sw[i]) && sw[i] >= 0.0, DSGD_ERR_INVALID,
         "dsgd_set_sample_weights: weight %g of row %lld is not finite and >= 0", sw[i], (long long)i);
  CU(cudaSetDevice(ctx->device));
  int rc = ctx->sw.grow(ctx, n, n);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->sw, sw, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->sw_on = true;
  return DSGD_OK;
}

extern "C" int dsgd_dim(const dsgd_ctx *ctx, int32_t *dim_out) {
  if (!ctx || !dim_out) return DSGD_ERR_INVALID;
  *dim_out = ctx->dim;
  return DSGD_OK;
}

extern "C" int dsgd_weights_l1(dsgd_ctx *ctx, const double *w, double *l1_out, int64_t *nnz_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE,
       "dsgd_weights_l1: ctx is in async mode (the L1 penalty is a step of the sync paths; Hogwild has no step order)");
  CU(cudaSetDevice(ctx->device));
  const double *src = ctx->w;
  if (w) {
    CU(cudaMemcpyAsync(ctx->w_req, w, sizeof(double) * (size_t)ctx->dim, cudaMemcpyHostToDevice, ctx->stream));
    src = ctx->w_req;
  }
  // out2[5] = ||w||_1, out2[6] = the count as an int64
  long long *nnz_dev = reinterpret_cast<long long *>(ctx->out2.p + 6);
  k_l1_norm<<<cdiv(ctx->dim, 256), 256, 0, ctx->stream>>>(src, ctx->dim, ctx->cnt);
  LAUNCHED();
  k_l1_finish<<<1, 1, 0, ctx->stream>>>(ctx->cnt, ctx->out2 + 5, nnz_dev);
  LAUNCHED();
  CU(cudaGetLastError());
  double l1 = 0.0;
  long long nnz = 0;
  CU(cudaMemcpyAsync(&l1, ctx->out2 + 5, sizeof l1, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(&nnz, nnz_dev, sizeof nnz, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (l1_out) *l1_out = l1;
  if (nnz_out) *nnz_out = nnz;
  return DSGD_OK;
}

// ---- averaged SGD: the sync step kernels add the new weights of every step to ctx->avg while ctx->avg_on ----------------

extern "C" int dsgd_average_begin(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "dsgd_average_begin: ctx is in async mode (averaging is sync-mode only)");
  ctx->avg_on = false;   // a failure below leaves averaging off and nothing to read
  ctx->avg_n = 0;
  CU(cudaSetDevice(ctx->device));
  if (!ctx->avg) CU(ctx->avg.alloc(wlen(ctx)));
  CU(cudaMemsetAsync(ctx->avg, 0, sizeof(double) * (size_t)wlen(ctx), ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->avg_on = true;
  return DSGD_OK;
}

extern "C" int dsgd_average_end(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "dsgd_average_end: ctx is in async mode (averaging is sync-mode only)");
  ctx->avg_on = false;
  return DSGD_OK;
}

extern "C" int dsgd_average_weights(dsgd_ctx *ctx, double *avg_out, int64_t *n_steps_out) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(!(ctx->flags & DSGD_FLAG_ASYNC), DSGD_ERR_STATE, "dsgd_average_weights: ctx is in async mode (averaging is sync-mode only)");
  NEED(ctx->avg, DSGD_ERR_STATE, "dsgd_average_weights: dsgd_average_begin was never called");
  NEED(ctx->avg_n > 0, DSGD_ERR_EMPTY, "dsgd_average_weights: no sync step since dsgd_average_begin (the mean of an empty list)");
  if (avg_out) {
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(avg_out, ctx->avg, sizeof(double) * (size_t)wlen(ctx), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    int rc = persist_check(ctx);   // the sums of a launch that hit its watchdog are garbage
    if (rc) return rc;
    // one IEEE division per column, then the constructor filter of a new Sparse (Sparse.scala:108-118)
    const double n = (double)ctx->avg_n;
    for (int64_t j = 0; j < wlen(ctx); ++j) {
      const double v = avg_out[j] / n;
      avg_out[j] = std::fabs(v) > kEps ? v : 0.0;
    }
  }
  if (n_steps_out) *n_steps_out = ctx->avg_n;
  return DSGD_OK;
}

// ---- async (Hogwild) mode -------------------------------------------------------------------------------------

extern "C" int dsgd_async_host_master(dsgd_ctx *ctx, const double *w0) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "Cannot host the async master replica: ctx is in synchronous mode.");
  NEED(w0, DSGD_ERR_INVALID, "dsgd_async_host_master: w0 is NULL");
  NEED(ctx->have_d, DSGD_ERR_STATE, "dsgd_async_host_master: dimSparsity not set");
  CU(cudaSetDevice(ctx->device));
  if (!ctx->m_w) CU(ctx->m_w.alloc((int64_t)ctx->dim + kReplicaPad));
  CU(cudaMemsetAsync(ctx->m_w, 0, sizeof(double) * (size_t)(ctx->dim + kReplicaPad), ctx->stream));
  CU(cudaMemcpyAsync(ctx->m_w, w0, sizeof(double) * (size_t)ctx->dim, cudaMemcpyHostToDevice, ctx->stream));
  k_async_init_ctl<1024><<<1, 1024, 0, ctx->stream>>>(ctx->m_w, ctx->d, ctx->dim);
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_ipc_export(dsgd_ctx *ctx, int which, uint8_t handle[DSGD_IPC_HANDLE_BYTES]) {
  if (!ctx || !handle) return DSGD_ERR_INVALID;
  static_assert(sizeof(cudaIpcMemHandle_t) == DSGD_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t size");
  NEED(which == DSGD_REPLICA_SELF || which == DSGD_REPLICA_MASTER, DSGD_ERR_INVALID, "dsgd_ipc_export: bad `which`");
  NEED(which == DSGD_REPLICA_SELF || ctx->m_w, DSGD_ERR_STATE, "dsgd_ipc_export: this ctx does not host the master replica");
  CU(cudaSetDevice(ctx->device));
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, which == DSGD_REPLICA_SELF ? ctx->w.p : ctx->m_w.p));
  memcpy(handle, &h, sizeof h);
  return DSGD_OK;
}

extern "C" int dsgd_ipc_import(dsgd_ctx *ctx, int peer_rank, const uint8_t handle[DSGD_IPC_HANDLE_BYTES]) {
  if (!ctx || !handle) return DSGD_ERR_INVALID;
  NEED(peer_rank >= 0 && peer_rank <= ctx->world && peer_rank < kMaxReplicas, DSGD_ERR_INVALID,
       "dsgd_ipc_import: peer_rank %d outside [0,%d]", peer_rank, ctx->world);
  NEED(peer_rank != ctx->rank, DSGD_ERR_INVALID, "dsgd_ipc_import: a worker does not import its own replica");
  NEED(!ctx->a_running, DSGD_ERR_STATE, "dsgd_ipc_import: async computation is running");
  CU(cudaSetDevice(ctx->device));
  return open_ipc(ctx, ctx->peer_w[peer_rank], handle);
}

extern "C" int dsgd_peer_attach(dsgd_ctx *ctx, int peer_rank, dsgd_ctx *peer, int which) {
  if (!ctx || !peer) return DSGD_ERR_INVALID;
  NEED(peer_rank >= 0 && peer_rank <= ctx->world && peer_rank < kMaxReplicas, DSGD_ERR_INVALID,
       "dsgd_peer_attach: peer_rank %d outside [0,%d]", peer_rank, ctx->world);
  NEED(which == DSGD_REPLICA_SELF || peer->m_w, DSGD_ERR_STATE, "dsgd_peer_attach: peer does not host the master replica");
  NEED(peer->dim == ctx->dim, DSGD_ERR_INVALID, "dsgd_peer_attach: dimension mismatch");
  // the running loop copied the replica table when it started: a replica attached now would never receive a delta
  NEED(!ctx->a_running, DSGD_ERR_STATE, "dsgd_peer_attach: async computation is running");
  int rc = enable_peer_access(ctx, peer, "dsgd_peer_attach");
  if (rc) return rc;
  ctx->peer_w[peer_rank].set(which == DSGD_REPLICA_SELF ? peer->w.p : peer->m_w.p, false);
  return DSGD_OK;
}

static double *master_replica(dsgd_ctx *ctx) {
  return ctx->m_w ? ctx->m_w.p : (ctx->world < kMaxReplicas ? ctx->peer_w[ctx->world].p : nullptr);
}

// CUDA loads a kernel when it is first launched (lazy loading, the default since CUDA 12.2), and loading may wait for every
// kernel running on the device.  An async loop started by dsgd_start_async runs until it is stopped, so the first launch of
// any other kernel while it runs -- an evaluation of the master's weights in MasterAsync.fit, a request, another context's
// loop -- would wait for it forever.  Before the first async loop on a device, every kernel of the library is loaded.
static int load_all_kernels(dsgd_ctx *ctx) {
  static std::mutex mu;
  static std::vector<int> done;   // devices whose kernels are loaded in this process
  std::lock_guard<std::mutex> lock(mu);
  if (std::find(done.begin(), done.end(), ctx->device) != done.end()) return DSGD_OK;
  void *get_module = nullptr, *count = nullptr, *enumerate = nullptr, *load = nullptr;
  cudaDriverEntryPointQueryResult q[4];
  CU(cudaGetDriverEntryPointByVersion("cuFuncGetModule", &get_module, 12040, cudaEnableDefault, &q[0]));
  CU(cudaGetDriverEntryPointByVersion("cuModuleGetFunctionCount", &count, 12040, cudaEnableDefault, &q[1]));
  CU(cudaGetDriverEntryPointByVersion("cuModuleEnumerateFunctions", &enumerate, 12040, cudaEnableDefault, &q[2]));
  CU(cudaGetDriverEntryPointByVersion("cuFuncLoad", &load, 12040, cudaEnableDefault, &q[3]));
  for (int i = 0; i < 4; ++i)
    NEED(q[i] == cudaDriverEntryPointSuccess, DSGD_ERR_CUDA, "async loop: the CUDA driver cannot preload kernels (needs 12.4)");
  cudaFunction_t any = nullptr;
  CU(cudaGetFuncBySymbol(&any, reinterpret_cast<const void *>(k_async_worker_b1)));
  CUmodule mod = nullptr;
  unsigned n = 0;
  CUresult r = reinterpret_cast<CUresult (*)(CUmodule *, CUfunction)>(get_module)(&mod, any);
  if (r == CUDA_SUCCESS) r = reinterpret_cast<CUresult (*)(unsigned *, CUmodule)>(count)(&n, mod);
  std::vector<CUfunction> fns(n);
  if (r == CUDA_SUCCESS && n)
    r = reinterpret_cast<CUresult (*)(CUfunction *, unsigned, CUmodule)>(enumerate)(fns.data(), n, mod);
  for (unsigned i = 0; i < n && r == CUDA_SUCCESS; ++i) r = reinterpret_cast<CUresult (*)(CUfunction)>(load)(fns[i]);
  NEED(r == CUDA_SUCCESS, DSGD_ERR_CUDA, "async loop: loading the library's kernels failed (CUresult %d)", (int)r);
  done.push_back(ctx->device);
  return DSGD_OK;
}

static int async_launch(dsgd_ctx *ctx, const double *w0, const int32_t *assigned, int64_t n_assigned, const int32_t *replay,
                        int32_t batch, double lr, int32_t lanes, int64_t max_updates, uint64_t seed, cudaStream_t st) {
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "Cannot initialize async computation: slave is in synchronous mode.");
  NEED(!ctx->a_running, DSGD_ERR_STATE,
       "Async computation already running, can't be initialized unless stopped first");
  NEED(ctx->pairs && ctx->have_d, DSGD_ERR_STATE, "dsgd_start_async: rows or dimSparsity missing");
  NEED(batch >= 1 && lanes >= 1 && lanes <= 4096, DSGD_ERR_INVALID, "dsgd_start_async: bad arguments");
  CU(cudaSetDevice(ctx->device));
  int rc = load_all_kernels(ctx);
  if (rc || (rc = reserve_requests(ctx))) return rc;
  if (w0) {  // weights() = request.weights
    CU(cudaMemcpyAsync(ctx->w, w0, sizeof(double) * (size_t)ctx->dim, cudaMemcpyHostToDevice, ctx->stream));
    rc = refresh_resident(ctx);  // also S = w . d and the control slots of the replica
    if (rc) return rc;
  }  // else: keep the resident replica (already initialised; deltas peers pushed since then must survive)
  if ((rc = ctx->a_scratch.grow(ctx, (int64_t)lanes * ctx->dim, 1, true))) return rc;
  if ((rc = ctx->a_rows.grow(ctx, (int64_t)lanes * batch, 1024))) return rc;
  CU(cudaMemsetAsync(ctx->a_stop, 0, sizeof(int), ctx->stream));
  CU(cudaMemsetAsync(ctx->a_cnt, 0, sizeof(unsigned long long) * 2, ctx->stream));
  AsyncParams ap;
  ap.rp16 = ctx->rp16; ap.pairs = ctx->pairs; ap.label = ctx->label; ap.d = ctx->d; ap.dim = ctx->dim;
  ap.assigned = assigned; ap.n_assigned = n_assigned; ap.replay = replay; ap.batch = batch; ap.lr = lr; ap.lambda = ctx->lambda;
  int nr = 0;
  ap.replica[nr++] = ctx->w;
  for (int r = 0; r < ctx->world && r < kMaxReplicas - 1; ++r)
    if (r != ctx->rank && ctx->peer_w[r]) ap.replica[nr++] = ctx->peer_w[r];
  ap.master_slot = -1;
  if (double *master = master_replica(ctx)) { ap.master_slot = nr; ap.replica[nr++] = master; }
  if (ctx->outbox) {   // colleagues reached over the host: one more target of every delta, relayed by the host in batches
    NEED(nr < kMaxReplicas, DSGD_ERR_INVALID, "dsgd_start_async: no replica slot left for the outbox");
    ap.replica[nr++] = ctx->outbox;
  }
  for (int q = nr; q < kMaxReplicas; ++q) ap.replica[q] = nullptr;
  ap.n_replicas = nr;
  ap.scratch = ctx->a_scratch; ap.batch_rows = ctx->a_rows; ap.n_lanes = lanes; ap.max_updates = max_updates; ap.seed = seed;
  ap.stop = ctx->a_stop; ap.claimed = ctx->a_cnt; ap.done = ctx->a_cnt + 1;
  CU(cudaStreamSynchronize(ctx->stream));  // inputs in place before the loop's own stream starts
  if (!ctx->a_ev0) { CU(cudaEventCreate(&ctx->a_ev0.h)); CU(cudaEventCreate(&ctx->a_ev1.h)); }
  CU(cudaEventRecord(ctx->a_ev0, st));
  // batch 1: the delta of every non-zero is formed straight from the pair, without the per-lane scratch vector
  if (batch == 1) k_async_worker_b1<<<cdiv(lanes, 4), 128, 0, st>>>(ap);
  else k_async_worker<<<cdiv(lanes, 4), 128, 0, st>>>(ap);
  CU(cudaEventRecord(ctx->a_ev1, st));
  LAUNCHED();
  CU(cudaGetLastError());
  return DSGD_OK;
}

extern "C" int dsgd_start_async(dsgd_ctx *ctx, const double *w0, const int32_t *assigned, int64_t n_assigned, int32_t batch,
                                double lr, int32_t concurrency, int64_t max_updates, uint64_t seed) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "Cannot initialize async computation: slave is in synchronous mode.");
  NEED(assigned && n_assigned >= 1, DSGD_ERR_EMPTY, "dsgd_start_async: no samples assigned (Random.nextInt(0) throws)");
  NEED(n_assigned <= ctx->n_rows, DSGD_ERR_RANGE, "dsgd_start_async: more assigned samples than rows");
  int rc = check_ids(ctx, assigned, n_assigned, __func__, "assigned sample");
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  if ((rc = ctx->a_assigned.grow(ctx, n_assigned, 1024))) return rc;
  CU(cudaMemcpyAsync(ctx->a_assigned, assigned, sizeof(int32_t) * (size_t)n_assigned, cudaMemcpyHostToDevice, ctx->stream));
  if (batch > n_assigned) batch = (int32_t)n_assigned;  // `take batchSize` of a shorter shuffle
  rc = async_launch(ctx, w0, ctx->a_assigned, n_assigned, nullptr, batch, lr, concurrency, max_updates, seed, ctx->astream);
  if (rc) return rc;
  ctx->a_running = true;
  return DSGD_OK;
}

extern "C" int dsgd_async_replay(dsgd_ctx *ctx, const double *w0, const int32_t *samples, int32_t batch, int64_t n_updates,
                                 double lr) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "Cannot initialize async computation: slave is in synchronous mode.");
  NEED(samples && batch >= 1 && n_updates >= 1, DSGD_ERR_EMPTY, "dsgd_async_replay: empty sequence");
  const int64_t n = (int64_t)batch * n_updates;
  int rc = check_ids(ctx, samples, n, __func__, "sample index");
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  if ((rc = ctx->a_replay.grow(ctx, n, 1024))) return rc;
  CU(cudaMemcpyAsync(ctx->a_replay, samples, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  rc = async_launch(ctx, w0, nullptr, 1, ctx->a_replay, batch, lr, 1, n_updates, 0, ctx->stream);
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  rc = refresh_resident(ctx);
  // refresh_resident re-derives S from the weights; the loop's running S is what the NEXT replay would start from anyway
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_async_running(dsgd_ctx *ctx, int *running) {
  if (!ctx || !running) return DSGD_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  *running = 0;
  if (ctx->a_running) {
    cudaError_t e = cudaStreamQuery(ctx->astream);
    if (e == cudaErrorNotReady) *running = 1;
    else if (e != cudaSuccess) CU(e);
  }
  return DSGD_OK;
}

extern "C" int dsgd_stop_async(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "Cannot stop async computation: slave is in synchronous mode.");
  CU(cudaSetDevice(ctx->device));
  if (!ctx->a_running) return DSGD_OK;  // runningAsync() = false on an idle slave is a no-op in the reference too
  static const int one = 1;
  CU(cudaMemcpyAsync(ctx->a_stop, &one, sizeof(int), cudaMemcpyHostToDevice, ctx->stream2));
  CU(cudaStreamSynchronize(ctx->stream2));
  CU(cudaStreamSynchronize(ctx->astream));
  ctx->a_running = false;
  // not refresh_resident: its k_async_init_ctl would zero the update counter the loop just advanced
  launch_prepare(ctx, ctx->w, ctx->w32, kScalC, kScalNrm2);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_async_elapsed_ms(dsgd_ctx *ctx, float *elapsed_ms) {
  if (!ctx || !elapsed_ms) return DSGD_ERR_INVALID;
  NEED(ctx->a_ev0 && !ctx->a_running, DSGD_ERR_STATE, "dsgd_async_elapsed_ms: no finished async loop (stop it first)");
  CU(cudaSetDevice(ctx->device));
  CU(cudaEventSynchronize(ctx->a_ev1));
  CU(cudaEventElapsedTime(elapsed_ms, ctx->a_ev0, ctx->a_ev1));
  return DSGD_OK;
}

extern "C" int dsgd_update_grad(dsgd_ctx *ctx, const int32_t *idx, const double *val, int64_t nnz) {
  if (!ctx) return DSGD_ERR_INVALID;
  // concurrent callers (a gRPC server's thread pool) share the staging buffers: the next call may refill or regrow them only
  // after this call's kernel has finished reading them
  std::lock_guard<std::mutex> lock(ctx->u_mu);
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "Cannot update gradient: slave is in synchronous mode.");
  NEED(nnz >= 0 && (nnz == 0 || (idx && val)), DSGD_ERR_INVALID, "dsgd_update_grad: bad arguments");
  for (int64_t k = 0; k < nnz; ++k)
    NEED(idx[k] >= 0 && idx[k] < ctx->dim, DSGD_ERR_RANGE, "dsgd_update_grad: key %d outside [0,%d)", idx[k], ctx->dim);
  if (nnz == 0) return DSGD_OK;
  CU(cudaSetDevice(ctx->device));
  int rc = ctx->u_idx.grow(ctx, nnz, 4096);
  if (rc) return rc;
  if ((rc = ctx->u_val.grow(ctx, nnz, 4096))) return rc;
  CU(cudaMemcpyAsync(ctx->u_idx, idx, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, ctx->stream2));
  CU(cudaMemcpyAsync(ctx->u_val, val, sizeof(double) * (size_t)nnz, cudaMemcpyHostToDevice, ctx->stream2));
  k_async_apply_delta<<<std::min(cdiv(nnz, 256), 64), 256, 0, ctx->stream2>>>(ctx->w, ctx->dim, ctx->d, ctx->u_idx, ctx->u_val, nnz, 0);
  LAUNCHED();
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream2));
  return DSGD_OK;
}

extern "C" int dsgd_async_updates(dsgd_ctx *ctx, int64_t *count) {
  if (!ctx || !count) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "dsgd_async_updates: ctx is in synchronous mode");
  CU(cudaSetDevice(ctx->device));
  unsigned long long v = 0;
  double *m = master_replica(ctx);
  const void *src = m ? (const void *)(reinterpret_cast<unsigned long long *>(m) + ctx->dim + kCtlUpdates) : (const void *)(ctx->a_cnt + 1);
  CU(cudaMemcpyAsync(&v, src, sizeof v, cudaMemcpyDeviceToHost, ctx->stream2));
  CU(cudaStreamSynchronize(ctx->stream2));
  *count = (int64_t)v;
  return DSGD_OK;
}

extern "C" int dsgd_async_outbox_enable(dsgd_ctx *ctx) {
  if (!ctx) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "dsgd_async_outbox_enable: ctx is in synchronous mode");
  NEED(!ctx->a_running, DSGD_ERR_STATE, "dsgd_async_outbox_enable: async computation is running");
  CU(cudaSetDevice(ctx->device));
  if (!ctx->outbox) CU(ctx->outbox.alloc((int64_t)ctx->dim + kReplicaPad));
  CU(cudaMemsetAsync(ctx->outbox, 0, sizeof(double) * (size_t)(ctx->dim + kReplicaPad), ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return DSGD_OK;
}

extern "C" int dsgd_async_outbox_read(dsgd_ctx *ctx, double *acc_out) {
  if (!ctx || !acc_out) return DSGD_ERR_INVALID;
  NEED(ctx->outbox, DSGD_ERR_STATE, "dsgd_async_outbox_read: the outbox is not enabled");
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(acc_out, ctx->outbox, sizeof(double) * (size_t)ctx->dim, cudaMemcpyDeviceToHost, ctx->stream2));
  CU(cudaStreamSynchronize(ctx->stream2));
  return DSGD_OK;
}

extern "C" int dsgd_async_master_weights(dsgd_ctx *ctx, double *w_out) {
  if (!ctx || !w_out) return DSGD_ERR_INVALID;
  NEED(ctx->flags & DSGD_FLAG_ASYNC, DSGD_ERR_STATE, "dsgd_async_master_weights: ctx is in synchronous mode");
  double *m = master_replica(ctx);
  NEED(m, DSGD_ERR_STATE, "dsgd_async_master_weights: no master replica hosted or imported");
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(w_out, m, sizeof(double) * (size_t)ctx->dim, cudaMemcpyDeviceToHost, ctx->stream2));
  CU(cudaStreamSynchronize(ctx->stream2));
  return DSGD_OK;
}
