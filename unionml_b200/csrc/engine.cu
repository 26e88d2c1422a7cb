// C ABI of the uml_b200 engine (see include/uml_b200.h): device binding, model/batch residency, predict calls.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <nvtx3/nvToolsExt.h>
#include <sched.h>

#include "uml_common.cuh"
#include "mlp_rescore.cuh"
#include "mlp_topk.cuh"

// NVTX ranges around the phases of a call (stage / score / re-score / exchange); free when no tool is attached
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

namespace uml {
cudaError_t launch_finite_scan(const float* x, int64_t ld, int64_t rows, int n_features, StageResult* result,
                               cudaStream_t stream);
cudaError_t launch_push_bytes(const void* src, void* const* dst, int n_dst, int64_t bytes, int sm_count,
                              cudaStream_t stream);
cudaError_t launch_labels_take(const void* labels, int label_bytes, int64_t n, const double* classes, int n_classes,
                               double* out, cudaStream_t stream);
cudaError_t launch_labels_count_equal(const void* labels, int label_bytes, int64_t n, const double* classes,
                                      int n_classes, const double* targets, unsigned long long* count,
                                      cudaStream_t stream);
}

using uml::FlagList;
using uml::LinearDeviceModel;
using uml::LinearLaunch;
using uml::StageResult;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static thread_local std::string g_create_error;

constexpr int kSmallRows = 64;              // online path: batches up to this many rows take the one-kernel fp64 route
constexpr int64_t kSmallBytes = 256 << 10;   // ... when their raw feature block fits the pinned request buffer

struct HostMirror {  // pinned; device counters are copied here
  int flag_count;
  int pad;
  unsigned long long counters[uml::kCounterTileClaim];  // the slots a synchronous call zeroes and reads back
  StageResult stage;
  uml::SmallResult small[kSmallRows];
};

// Host threads that gather a pageable source chunk into a pinned bounce buffer: cudaMemcpy from pageable memory is
// staged by the driver on one thread; a few threads doing plain memcpy into page-locked memory keep the link busy.
namespace uml {
int narrow_f64_to_f32(const double* src, float* dst, size_t n);  // host_narrow.cpp
}

class CopyPool {
 public:
  struct Task {  // `rows` runs of n bytes (rows == 1: one contiguous run)
    char* dst;
    const char* src;
    size_t n;
    size_t rows = 1, dpitch = 0, spitch = 0;
    // narrow != nullptr: the run is float64 and is written as float32 (n = source bytes, dst advances half as fast);
    // *narrow is set when a value does not survive the round trip (the caller then re-sends the chunk as float64)
    std::atomic<int>* narrow = nullptr;
  };
  explicit CopyPool(int n_threads) {
    for (int i = 0; i < n_threads; ++i) workers_.emplace_back([this] { loop(); });
  }
  ~CopyPool() {
    {
      std::lock_guard<std::mutex> g(mu_);
      stop_ = true;
    }
    cv_work_.notify_all();
    for (auto& t : workers_) t.join();
  }
  // copy every task; the calling thread works too and returns when all are done
  void run(const std::vector<Task>& tasks) {
    if (tasks.empty()) return;
    auto job = std::make_shared<Job>();
    job->tasks = tasks.data();
    job->n = tasks.size();
    {
      std::lock_guard<std::mutex> g(mu_);
      job_ = job;
      ++generation_;
    }
    cv_work_.notify_all();
    work(*job);
    std::unique_lock<std::mutex> g(mu_);
    cv_done_.wait(g, [&] { return job->done.load() == job->n; });
    job_.reset();
  }

 private:
  // a job owns its counters, so a worker that wakes up late only ever sees an exhausted index range of an old job
  struct Job {
    const Task* tasks = nullptr;
    size_t n = 0;
    std::atomic<size_t> next{0}, done{0};
  };
  void work(Job& job) {
    for (;;) {
      const size_t i = job.next.fetch_add(1);
      if (i >= job.n) return;
      const Task& t = job.tasks[i];
      if (t.narrow) {
        // (also "lossy" for NaN: such chunks travel as float64 and the staging kernel reports them)
        if (uml::narrow_f64_to_f32(reinterpret_cast<const double*>(t.src), reinterpret_cast<float*>(t.dst), t.n / 8))
          t.narrow->store(1, std::memory_order_relaxed);
      } else {
        for (size_t r = 0; r < t.rows; ++r) memcpy(t.dst + r * t.dpitch, t.src + r * t.spitch, t.n);
      }
      if (job.done.fetch_add(1) + 1 == job.n) {
        std::lock_guard<std::mutex> g(mu_);
        cv_done_.notify_all();
      }
    }
  }
  void loop() {
    uint64_t seen = 0;
    for (;;) {
      std::shared_ptr<Job> job;
      {
        std::unique_lock<std::mutex> g(mu_);
        cv_work_.wait(g, [&] { return stop_ || generation_ != seen; });
        if (stop_) return;
        seen = generation_;
        job = job_;
      }
      if (job) work(*job);
    }
  }
  std::vector<std::thread> workers_;
  std::mutex mu_;
  std::condition_variable cv_work_, cv_done_;
  std::shared_ptr<Job> job_;
  uint64_t generation_ = 0;
  bool stop_ = false;
};

struct SmallGraph {  // one captured small-batch kernel (linear or MLP) per (model, rows, features, dtype, output, k)
  uint64_t model_uid = 0;
  int n_rows = 0, n_features = 0, dtype = 0;
  int kind = 0, k = 0;  // uml::SmallOutput and the top-k width: a model's labels, probabilities and top-k differ
  cudaGraphExec_t exec = nullptr;
  uint64_t last_use = 0;
};

// engine scratch that only grows (see grow): N buffers of `cap` elements each, in device memory or, Pinned, in
// page-locked host memory
template <class T, int N = 1, bool Pinned = false>
struct Scratch {
  T* p[N] = {};
  int64_t cap = 0;
  void release() {
    for (auto& q : p) {
      if (q) Pinned ? cudaFreeHost(q) : cudaFree(q);
      q = nullptr;
    }
    cap = 0;
  }
};

struct uml_engine {
  int device = 0;
  cudaStream_t own_stream = nullptr, stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev[6] = {};
  cudaEvent_t chunk_ev[8] = {};
  uml_device_info info{};
  PFN_encodeTiled encode = nullptr;
  std::string last_error;
  // device scratch
  int* d_flag_count = nullptr;
  unsigned long long* d_counters = nullptr;
  StageResult* d_stage = nullptr;
  Scratch<int32_t> d_flag_rows;
  Scratch<int32_t> d_labels;             // labels on their way to another output (peer scatter, class values)
  Scratch<char> d_result;                // outputs of a resident-batch call bound for host memory (predict_resident)
  Scratch<char, 3> d_chunk;              // raw source chunks (staging / predict_host)
  Scratch<float, 3> d_xchunk;            // converted fp32 chunks (predict_host)
  Scratch<char, 3> d_ochunk;             // the output of a chunk (predict_host)
  Scratch<double> d_classes;
  Scratch<double> d_targets;             // uml_topk_count_hits: targets and first-hit counters
  Scratch<unsigned long long> d_hits;
  Scratch<char, 3, true> h_bounce;       // pinned bounce buffers for pageable sources
  Scratch<char, 3, true> h_result;       // pinned landing slots for chunk outputs bound for pageable memory
  CopyPool* pool = nullptr;
  // online path (B <= kSmallRows): pinned request buffer, its device twin, result slots, cached graphs
  void* h_req = nullptr;
  void* d_req = nullptr;
  uml::SmallResult* d_small = nullptr;
  std::vector<SmallGraph> small_graphs;
  uint64_t small_tick = 0;
  // asynchronous host call (uml_linear_predict_host_values_begin / _poll / _finish): one in flight per engine
  std::thread async_thread;
  std::atomic<int64_t> async_rows_done{0};
  std::atomic<int> async_finished{1};
  int async_status = UML_OK;
  uml_stats async_stats{};

  bool small_graph_ok = true;
  HostMirror* h = nullptr;
};

static std::atomic<uint64_t> g_model_uid{1};

struct uml_model {
  uml_engine* e = nullptr;
  uint64_t uid = 0;  // changes whenever the device operands are re-uploaded (keys the cached small-batch graphs)
  LinearDeviceModel dm{};
  int n_features_in = 0;
  int n_classes_in = 0;  // as passed by the caller (1 for sklearn's binary layout)
  std::vector<double> coef64, intercept64;  // caller's values (expanded), before any affine fold
  float* d_wt = nullptr;
  float* d_bias = nullptr;
  double* d_w64 = nullptr;
  double* d_b64 = nullptr;
  void* d_tc = nullptr;  // dm.tc_ops
};

struct uml_batch {
  uml_engine* e = nullptr;
  float* x = nullptr;
  double* x64 = nullptr;
  int64_t n_rows = 0, ld = 0, ld64 = 0;
  int n_features = 0;
  bool owns = false;
  bool lossless = true;
  int tf32_exact = -1;  // every fp32 feature is a tf32 value: 1 yes, 0 no, -1 not scanned yet (wrapped device rows)
  bool has_map = false;
  CUtensorMap map{};      // boxes of 128 rows x 32 features (MLP kernels)
  CUtensorMap lin_map{};  // boxes of uml::linear_box_rows(f_pad) rows x 32 features (linear tile kernel)
  // compact fp16 copy of the rows (staged batches with F <= 64 whose every value is an fp16 value): what the linear
  // tile kernel reads instead of x, through half_map's {64 features, 128 rows} boxes.  ldh = uml::linear_half_ld(F).
  void* xh = nullptr;
  int64_t ldh = 0;
  bool has_half = false;
  bool half_nonneg = false;  // the fp16 copy holds no value < 0 (the linear tile kernel's tensor-core schedule needs that)
  CUtensorMap half_map{};
};

struct uml_mlp {
  uml_engine* e = nullptr;
  uint64_t uid = 0;  // keys the cached small-batch graphs (from the same counter as uml_model::uid)
  size_t small_smem = 0;  // dynamic shared memory of mlp_small_kernel; 0: too large, batches keep the chunk pipeline
  size_t small_rec_smem = 0;  // ... of its probability / top-k forms (a logits strip more); 0: those keep the pipeline
  // where those forms write their records: mapped pinned memory for kSmallRows x C x 8 bytes, allocated at the model's
  // first such request and kept, so that the graphs captured with it stay valid
  void* h_rec = nullptr;
  void* d_rec = nullptr;
  uml::MlpDeviceModel dm{};
  float* d_w1t = nullptr;
  float* d_b1 = nullptr;
  float* d_w2t = nullptr;
  float* d_b2 = nullptr;
  double* d_w64 = nullptr;  // w1 | b1 | w2 | b2 packed
  float* d_w1_tiles = nullptr;  // tensor-core B operand: tf32 hi | lo rows, pre-swizzled
  uml::MlpHostModel host;
};

#define UML_FAIL(E, CODE, ...)                              \
  do {                                                      \
    char _buf[512];                                         \
    snprintf(_buf, sizeof(_buf), __VA_ARGS__);              \
    if (E) (E)->last_error = _buf; else g_create_error = _buf; \
    return (CODE);                                          \
  } while (0)

#define UML_CUDA(E, CALL)                                                                              \
  do {                                                                                                 \
    cudaError_t _err = (CALL);                                                                         \
    if (_err != cudaSuccess) {                                                                         \
      UML_FAIL(E, _err == cudaErrorMemoryAllocation ? UML_ERR_NOMEM : UML_ERR_CUDA, "%s failed: %s", #CALL, \
               cudaGetErrorString(_err));                                                              \
    }                                                                                                  \
  } while (0)

// UML_CUDA inside a pipeline (uml_stage_rows, predict_host_impl): both streams are drained before the call returns,
// because their queued copies still reference the caller's host memory
#define UML_CUDA_DRAIN(E, CALL)                                                                          \
  do {                                                                                                   \
    cudaError_t _ce = (CALL);                                                                            \
    if (_ce != cudaSuccess) {                                                                            \
      cudaStreamSynchronize((E)->stream);                                                                \
      cudaStreamSynchronize((E)->copy_stream);                                                           \
      UML_FAIL(E, _ce == cudaErrorMemoryAllocation ? UML_ERR_NOMEM : UML_ERR_CUDA, "%s failed: %s", #CALL, \
               cudaGetErrorString(_ce));                                                                 \
    }                                                                                                    \
  } while (0)

// make `s` hold at least n elements per buffer; it never shrinks, and reallocates only when n exceeds its capacity
template <class T, int N, bool Pinned>
static int grow(uml_engine* e, Scratch<T, N, Pinned>& s, int64_t n) {
  if (s.cap >= n) return UML_OK;
  s.release();
  for (auto& q : s.p) {
    void** v = (void**)&q;
    const size_t bytes = (size_t)n * sizeof(T);
    if (Pinned) UML_CUDA(e, cudaHostAlloc(v, bytes, cudaHostAllocDefault));
    else UML_CUDA(e, cudaMalloc(v, bytes));
  }
  s.cap = n;
  return UML_OK;
}

static FlagList flag_list(const uml_engine* e) {
  return FlagList{e->d_flag_count, e->d_flag_rows.p[0], (int)std::min<int64_t>(e->d_flag_rows.cap, INT32_MAX),
                  e->d_counters};
}

// a synchronous call reads its counters back at the end, so it starts them from zero
static cudaError_t reset_counters(uml_engine* e, cudaStream_t s) {
  const cudaError_t ce = cudaMemsetAsync(e->d_counters, 0, sizeof(e->h->counters), s);
  return ce != cudaSuccess ? ce : cudaMemsetAsync(e->d_flag_count, 0, sizeof(int), s);
}

// which MLP kernel scores the rows (the stats' path): 5 tensor cores, 3 CUDA cores, 2 the generic fp64 scorer.  Tensor
// cores when every feature is a tf32 value (integer / pixel domains), CUDA cores otherwise; both read the rows through
// a tensor map.  UML_B200_MLP_TC=0 / 1 forces the choice; 1 does not apply to class probabilities (labels: rows that
// are not tf32 values are caught in the kernel and re-scored; the probability kernels have no fp64 re-score behind
// them).  tf32() is asked only when its answer decides: it may cost a pass over the rows.
// topk: the tile kernels' top-k form, routed as the labels are (it has the same fp64 re-score behind it)
template <class Tf32>
static int mlp_route(const uml::MlpDeviceModel& m, bool has_map, bool proba, Tf32&& tf32, bool topk = false) {
  if (!has_map) return 2;
  std::string why;
  if (uml::mlp_tc_supported(m, &why, topk)) {
    const char* env = getenv("UML_B200_MLP_TC");
    const bool off = env && env[0] == '0', on = env && env[0] == '1' && !proba;
    if (!off && (on || tf32())) return 5;
  }
  return uml::mlp_tma_supported(m, &why, proba, topk) ? 3 : 2;
}

static int dtype_size(int dt) {
  switch (dt) {
    case UML_F32: return 4;
    case UML_F64: return 8;
    case UML_I64: return 8;
    case UML_I32: return 4;
    case UML_U8: return 1;
    default: return 0;
  }
}

extern "C" {

int uml_abi_version(void) { return UML_B200_ABI_VERSION; }

const char* uml_last_error(const uml_engine* e) { return e ? e->last_error.c_str() : g_create_error.c_str(); }

int uml_engine_create(uml_engine** out, int device_id) {
  if (!out) UML_FAIL((uml_engine*)nullptr, UML_ERR_INVALID, "uml_engine_create: out is NULL");
  *out = nullptr;
  int n = 0;
  cudaError_t err = cudaGetDeviceCount(&n);
  if (err != cudaSuccess || n == 0)
    UML_FAIL((uml_engine*)nullptr, UML_ERR_NO_DEVICE, "no CUDA device visible (%s); uml_b200 has no CPU fallback",
             err != cudaSuccess ? cudaGetErrorString(err) : "device count 0");
  if (device_id < 0 || device_id >= n)
    UML_FAIL((uml_engine*)nullptr, UML_ERR_INVALID, "device_id %d out of range [0,%d)", device_id, n);
  uml_engine* e = new uml_engine();
  e->device = device_id;
  auto fail = [&](const char* what, cudaError_t ce) {
    char buf[256];
    snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(ce));
    g_create_error = buf;
    delete e;
    return (int)UML_ERR_CUDA;
  };
  if ((err = cudaSetDevice(device_id)) != cudaSuccess) return fail("cudaSetDevice", err);
  cudaDeviceProp prop;
  if ((err = cudaGetDeviceProperties(&prop, device_id)) != cudaSuccess) return fail("cudaGetDeviceProperties", err);
  e->info.device_id = device_id;
  e->info.sm_count = prop.multiProcessorCount;
  e->info.cc_major = prop.major;
  e->info.cc_minor = prop.minor;
  e->info.total_mem_bytes = (int64_t)prop.totalGlobalMem;
  e->info.l2_bytes = prop.l2CacheSize;
  cudaDeviceGetAttribute(&e->info.sm_clock_khz, cudaDevAttrClockRate, device_id);
  cudaDeviceGetAttribute(&e->info.mem_clock_khz, cudaDevAttrMemoryClockRate, device_id);
  strncpy(e->info.name, prop.name, sizeof(e->info.name) - 1);
  if (prop.major != 9 || prop.minor != 0) {
    char buf[256];
    snprintf(buf, sizeof(buf), "device %d (%s) is compute capability %d.%d; this library is built for sm_90a only",
             device_id, prop.name, prop.major, prop.minor);
    g_create_error = buf;
    delete e;
    return UML_ERR_NO_DEVICE;
  }
  if ((err = cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking)) != cudaSuccess)
    return fail("cudaStreamCreate", err);
  if ((err = cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking)) != cudaSuccess)
    return fail("cudaStreamCreate", err);
  e->stream = e->own_stream;
  for (auto& ev : e->ev)
    if ((err = cudaEventCreate(&ev)) != cudaSuccess) return fail("cudaEventCreate", err);
  for (auto& ev : e->chunk_ev)
    if ((err = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", err);
  if ((err = cudaMalloc(&e->d_flag_count, sizeof(int))) != cudaSuccess) return fail("cudaMalloc", err);
  if ((err = cudaMalloc(&e->d_counters, uml::kCounterSlots * sizeof(unsigned long long))) != cudaSuccess)
    return fail("cudaMalloc", err);
  if ((err = cudaMalloc(&e->d_stage, sizeof(StageResult))) != cudaSuccess) return fail("cudaMalloc", err);
  if ((err = cudaHostAlloc((void**)&e->h, sizeof(HostMirror), cudaHostAllocMapped)) != cudaSuccess)
    return fail("cudaHostAlloc", err);
  memset(e->h, 0, sizeof(HostMirror));
  // the scoring steps do not memset these: the re-score kernel hands the flag list back empty (label_store.cuh)
  if ((err = cudaMemset(e->d_flag_count, 0, sizeof(int))) != cudaSuccess) return fail("cudaMemset", err);
  if ((err = cudaMemset(e->d_counters, 0, uml::kCounterSlots * sizeof(unsigned long long))) != cudaSuccess)
    return fail("cudaMemset", err);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (err != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) return fail("cuTensorMapEncodeTiled lookup", err);
  e->encode = (PFN_encodeTiled)fn;
  *out = e;
  return UML_OK;
}

void uml_engine_destroy(uml_engine* e) {
  if (!e) return;
  if (e->async_thread.joinable()) e->async_thread.join();
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  cudaFree(e->d_flag_count);
  cudaFree(e->d_counters);
  cudaFree(e->d_stage);
  e->d_flag_rows.release();
  e->d_labels.release();
  e->d_result.release();
  e->d_chunk.release();
  e->d_xchunk.release();
  e->d_ochunk.release();
  e->d_classes.release();
  e->d_targets.release();
  e->d_hits.release();
  e->h_bounce.release();
  e->h_result.release();
  delete e->pool;
  for (auto& g : e->small_graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  if (e->h_req) cudaFreeHost(e->h_req);  // d_req / d_small are device aliases of pinned host memory
  if (e->h) cudaFreeHost(e->h);
  for (auto ev : e->ev)
    if (ev) cudaEventDestroy(ev);
  for (auto ev : e->chunk_ev)
    if (ev) cudaEventDestroy(ev);
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  delete e;
}

int uml_engine_info(const uml_engine* e, uml_device_info* out) {
  if (!e || !out) return UML_ERR_INVALID;
  *out = e->info;
  return UML_OK;
}

int uml_engine_set_stream(uml_engine* e, void* cuda_stream) {
  if (!e) return UML_ERR_INVALID;
  e->stream = cuda_stream ? (cudaStream_t)cuda_stream : e->own_stream;
  return UML_OK;
}

int uml_engine_synchronize(uml_engine* e) {
  if (!e) return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  UML_CUDA(e, cudaStreamSynchronize(e->stream));
  UML_CUDA(e, cudaStreamSynchronize(e->copy_stream));
  return UML_OK;
}

int uml_host_alloc(uml_engine* e, void** out, int64_t bytes) {
  if (!e || !out || bytes < 0) return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  UML_CUDA(e, cudaHostAlloc(out, (size_t)(bytes > 0 ? bytes : 1), cudaHostAllocDefault));
  return UML_OK;
}

int uml_device_alloc(uml_engine* e, void** out, int64_t bytes) {
  if (!e || !out || bytes < 0) return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  UML_CUDA(e, cudaMalloc(out, (size_t)(bytes > 0 ? bytes : 1)));
  return UML_OK;
}

int uml_device_free(uml_engine* e, void* p) {
  if (!e) return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  if (p) UML_CUDA(e, cudaFree(p));
  return UML_OK;
}

int uml_host_free(uml_engine* e, void* p) {
  if (!e) return UML_ERR_INVALID;
  if (p) UML_CUDA(e, cudaFreeHost(p));
  return UML_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// model
// ---------------------------------------------------------------------------------------------------------------
// ---- tensor-core operands of the linear tile kernel (DESIGN.md 3.1, 3.2) ----
// the fp16 value nearest to v (ties to even; up: the smallest fp16 value >= v), for |v| below 2^16
static double f16_round(double v, bool up = false) {
  if (v == 0.0) return v;
  int e = 0;
  std::frexp(std::fabs(v), &e);  // |v| in [2^(e-1), 2^e): 11 significant bits, or the subnormal spacing 2^-24
  const int q = std::max(e - 11, -24);
  const double m = std::ldexp(v, -q);
  return std::ldexp(up ? std::ceil(m) : std::nearbyint(m), q);
}
// bit pattern of an fp16 value held exactly in v
static uint16_t f16_bits(double v) {
  const uint16_t sign = std::signbit(v) ? 0x8000u : 0u;
  const double a = std::fabs(v);
  if (a < 0x1p-14) return sign | (uint16_t)std::ldexp(a, 24);
  int e = 0;
  const double m = std::frexp(a, &e);  // a = m 2^e, m in [0.5, 1)
  return sign | (uint16_t)((e + 14) << 10) | (uint16_t)std::ldexp(m * 2.0 - 1.0, 10);
}
// per-k16-step budget of the f16 wgmma accumulation, in u = 2^-24 of the running |.| sum (DESIGN.md 3.2): above the
// 36u of a truncating aligner without guard bits over 16 products and the accumulator ((2 x 17 + 2) u, the model of
// 3.3), and at least 4x the worst that tests/test_gpu_wgmma_f16_accum.py measures on the hardware
constexpr double kTcStepBudget = 64.0;
// The B operand image of LinearDeviceModel::tc_ops and the certification factor, or false when the model does not take
// the tensor-core schedule: a folded affine map (its score error is bounded in the fp64 terms only), non-finite weights,
// or magnitudes at which the scaled A of DESIGN.md 3.2 could leave the normal fp32 range.  wt / bias are the fp32
// route's operands (its bound column and bias bound are what tier 1 must dominate).
static bool build_tc_operands(const std::vector<double>& w, const std::vector<double>& b, const std::vector<float>& wt,
                              const std::vector<float>& bias, int C, int F, int f_pad, int cp, double fold_rel,
                              std::vector<uint8_t>* image, float* kappa) {
  if (f_pad > uml::kHalfBoxF || fold_rel != 0.0) return false;
  double wabs = 0.0;
  for (double v : w) {
    if (!std::isfinite(v)) return false;
    wabs = std::max(wabs, std::fabs(v));
  }
  for (int c = 0; c < C; ++c)
    if (!std::isfinite(b[c])) return false;
  int ex = 0;
  if (wabs > 0.0) std::frexp(wabs, &ex);  // wabs < 2^ex
  const int sigma = 15 - ex;               // max |w| 2^sigma in [2^14, 2^15): every hi piece is a normal fp16 value
  double wsum = 0.0;
  for (int f = 0; f < F; ++f) wsum += wt[(size_t)f * cp + C];
  const double a32 = (double)bias[C] + 65504.0 * wsum;  // the fp32 route's A of the largest fp16 row
  if (!(std::ldexp(a32, std::max(sigma, 0)) < 0x1p100) || !(std::ldexp((double)bias[C], sigma) > 0x1p-100)) return false;
  const int NH = uml::linear_tc_hi_cols(C), N = uml::linear_tc_cols(C);
  std::vector<uint16_t> bt((size_t)N * uml::kHalfBoxF, 0);
  // column n's 128-byte row, its 16-byte chunks XOR-swizzled by (n & 7): the SWIZZLE_128B K-major layout
  auto put = [&](int n, int f, double v) { bt[(size_t)n * 64 + (((f / 8) ^ (n & 7)) * 8) + f % 8] = f16_bits(v); };
  for (int f = 0; f < F; ++f) {
    double wmax = std::ldexp((double)wt[(size_t)f * cp + C], sigma);
    for (int c = 0; c < C; ++c) {
      const double v = std::ldexp(w[(size_t)c * F + f], sigma);
      const double hi = f16_round(v);
      put(c, f, hi);
      put(NH + c, f, f16_round(v - hi));
      wmax = std::max(wmax, std::fabs(v));
    }
    // floored at 2^-3 so that 2^-22 of it covers the 2^-25 a subnormal piece errs by (hi + lo errs by <= 2^-21 of it).
    // The fp32 route's FLT_MIN floor can scale past fp16 when every weight is below 2^-127: no route then.
    const double wb = f16_round(std::max(wmax, 0.125), true);
    if (!(wb <= 65504.0)) return false;
    put(C, f, wb);
  }
  std::vector<float> tb(NH, 0.f);
  for (int c = 0; c < C; ++c) tb[c] = (float)std::ldexp(b[c], sigma);
  tb[C] = (float)std::ldexp((double)bias[C], sigma);  // exact: a power-of-two multiple of an fp32 value in range
  image->assign((size_t)N * 128 + tb.size() * 4, 0);
  std::memcpy(image->data(), bt.data(), (size_t)N * 128);
  std::memcpy(image->data() + (size_t)N * 128, tb.data(), tb.size() * 4);
  // tier 1 certifies iff margin > 2 Etc + 2.5 thr A32+ (DESIGN.md 3.2): Etc <= e_rel A, A <= Ahat / (1 - step)
  const double u = uml::kU;
  const double step = kTcStepBudget * u * (f_pad / 16);
  const double e_rel = (0x1p-21 + step * (1.0 + 0x1p-10) + 4.0 * u) * (1.0 + 0x1p-10);
  const double thr = uml::linear_margin_thr(F);
  *kappa = (float)((2.0 * e_rel + 2.5 * thr * (1.0 + (F + 2.0) * u)) / (1.0 - step) * (1.0 + 0x1p-10));
  return true;
}

// bmag[c] >= |b_c| is the bias magnitude both bounds use (|b_c| + sum_f |shift_f w'_cf| for a folded affine map) and
// fold_rel the fp64 bound's extra relative term of such a map (DESIGN.md 3.2)
static int upload_model(uml_engine* e, uml_model* m, const std::vector<double>& w, const std::vector<double>& b,
                        const std::vector<double>& bmag, double fold_rel) {
  const int C = m->dm.n_classes, F = m->dm.n_features;
  const int cp = (C + 1 + 3) / 4 * 4;
  const int f_pad = (F + uml::kChunkF - 1) / uml::kChunkF * uml::kChunkF;
  std::vector<float> wt((size_t)f_pad * cp, 0.f), bias(cp, 0.f);
  float bmax = 0.f;
  for (int c = 0; c < C; ++c) {
    bias[c] = (float)b[c];
    bmax = fmaxf(bmax, fmaxf(fabsf(bias[c]), (float)bmag[c]));
  }
  // bound column (DESIGN.md 3.2).  A weight that rounds into the subnormals errs by up to 2^-150 = u FLT_MIN, so
  // wmax_f is floored at FLT_MIN.  Every FMA of a class chain, the bias rounding and every float64 -> fp32 feature
  // cast add up to 2^-150 |w| absolute: (F + 2 + sum_f wmax_f) 2^-150 per score.  The guard compares the margin of
  // two scores, each of which may carry that error with opposite signs, so the constant added to max|b| makes
  // thr * K cover twice it; its FLT_MIN / thr part keeps thr * A a normal number.
  double wsum = 0.0;
  for (int f = 0; f < F; ++f) {
    float wmax = 0.f;
    for (int c = 0; c < C; ++c) {
      const float v = (float)w[(size_t)c * F + f];
      wt[(size_t)f * cp + c] = v;
      wmax = fmaxf(wmax, fabsf(v));
    }
    wmax = fmaxf(wmax, (float)uml::kFltMin);
    wt[(size_t)f * cp + C] = wmax;
    wsum += wmax;
  }
  const double abs_err = (F + 2.0 + wsum) * uml::kHalfSubnormal;
  bias[C] = (float)(bmax + (uml::kFltMin + 2.0 * abs_err) / uml::linear_margin_thr(F) * (1.0 + 1.0 / 1024));
  auto ensure = [&](void** p, size_t bytes) -> cudaError_t {
    if (*p) cudaFree(*p);
    *p = nullptr;
    return cudaMalloc(p, bytes);
  };
  UML_CUDA(e, ensure((void**)&m->d_wt, wt.size() * 4));
  UML_CUDA(e, ensure((void**)&m->d_bias, bias.size() * 4));
  // fp64 weights feature-major: w64t[f][stride], the classes of one feature contiguous (zero padded)
  const int stride = uml::linear_w64_stride(C);
  std::vector<double> w64t((size_t)F * stride, 0.0);
  for (int c = 0; c < C; ++c)
    for (int f = 0; f < F; ++f) w64t[(size_t)f * stride + c] = w[(size_t)c * F + f];
  UML_CUDA(e, ensure((void**)&m->d_w64, w64t.size() * 8));
  std::vector<double> b64(b);
  b64.insert(b64.end(), bmag.begin(), bmag.end());
  UML_CUDA(e, ensure((void**)&m->d_b64, b64.size() * 8));
  UML_CUDA(e, cudaMemcpy(m->d_wt, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice));
  UML_CUDA(e, cudaMemcpy(m->d_bias, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
  UML_CUDA(e, cudaMemcpy(m->d_w64, w64t.data(), w64t.size() * 8, cudaMemcpyHostToDevice));
  UML_CUDA(e, cudaMemcpy(m->d_b64, b64.data(), b64.size() * 8, cudaMemcpyHostToDevice));
  std::vector<uint8_t> tc;
  float kappa = 0.f;
  if (m->d_tc) cudaFree(m->d_tc);
  m->d_tc = nullptr;
  if (build_tc_operands(w, b, wt, bias, C, F, f_pad, cp, fold_rel, &tc, &kappa)) {
    UML_CUDA(e, cudaMalloc(&m->d_tc, tc.size()));
    UML_CUDA(e, cudaMemcpy(m->d_tc, tc.data(), tc.size(), cudaMemcpyHostToDevice));
  }
  m->dm.tc_ops = m->d_tc;
  m->dm.tc_kappa = kappa;
  m->dm.wt = m->d_wt;
  m->dm.bias = m->d_bias;
  m->dm.w64 = m->d_w64;
  m->dm.b64 = m->d_b64;
  m->dm.w64_stride = stride;
  m->dm.fold_rel = fold_rel;
  m->dm.binary = m->n_classes_in == 1 ? 1 : 0;
  m->dm.cp = cp;
  m->dm.f_pad = f_pad;
  m->uid = g_model_uid.fetch_add(1);
  return UML_OK;
}

int uml_linear_load(uml_engine* e, uml_model** out, const void* coef, const void* intercept, int n_classes,
                    int n_features, int dtype) {
  if (!e || !out || !coef || !intercept) return UML_ERR_INVALID;
  *out = nullptr;
  if (n_classes < 1 || n_features < 1) UML_FAIL(e, UML_ERR_INVALID, "n_classes=%d n_features=%d", n_classes, n_features);
  if (dtype != UML_F32 && dtype != UML_F64) UML_FAIL(e, UML_ERR_INVALID, "coef dtype must be F32 or F64");
  UML_CUDA(e, cudaSetDevice(e->device));
  auto get = [&](const void* p, size_t i) -> double {
    return dtype == UML_F64 ? ((const double*)p)[i] : (double)((const float*)p)[i];
  };
  uml_model* m = new uml_model();
  m->e = e;
  m->n_features_in = n_features;
  m->n_classes_in = n_classes;
  const int C = n_classes == 1 ? 2 : n_classes;  // binary: scores > 0  <=>  argmax([0, s]) with first-max ties
  const int F = n_features;
  m->coef64.assign((size_t)C * F, 0.0);
  m->intercept64.assign(C, 0.0);
  const int c0 = n_classes == 1 ? 1 : 0;
  for (int c = 0; c < n_classes; ++c) {
    for (int f = 0; f < F; ++f) m->coef64[(size_t)(c + c0) * F + f] = get(coef, (size_t)c * F + f);
    m->intercept64[c + c0] = get(intercept, c);
  }
  m->dm.n_classes = C;
  m->dm.n_features = F;
  std::vector<double> bmag(C);
  for (int c = 0; c < C; ++c) bmag[c] = fabs(m->intercept64[c]);
  int rc = upload_model(e, m, m->coef64, m->intercept64, bmag, 0.0);
  if (rc != UML_OK) {
    uml_model_free(m);
    return rc;
  }
  *out = m;
  return UML_OK;
}

int uml_linear_set_affine(uml_engine* e, uml_model* m, const double* shift, const double* scale) {
  if (!e || !m) return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  const int C = m->dm.n_classes, F = m->dm.n_features;
  std::vector<double> w = m->coef64, b = m->intercept64, bmag(C);
  // s_c = sum_f ((x_f - shift_f) * scale_f) w_cf + b_c = sum_f x_f w'_cf + b'_c,  w'_cf = scale_f w_cf,
  // b'_c = b_c - sum_f shift_f w'_cf.  With shift >> the spread of x (a StandardScaler's mean_), the terms of b'_c are
  // large, of one sign, and cancel against sum_f x_f w'_cf: a plain running sum would round every step the same way
  // and move the score by up to (F/2) u sum_f |shift_f w'_cf|, outside both bounds.  So b'_c is summed exactly up to
  // one final rounding plus O(F u^2): each product is split by fma into p + pe (TwoProduct) and the sum carries its
  // rounding errors in a Neumaier compensation term.  bmag_c = |b_c| + sum_f |shift_f w'_cf| bounds every term.
  for (int c = 0; c < C; ++c) {
    double s = b[c], comp = 0.0, mag = fabs(b[c]);
    for (int f = 0; f < F; ++f) {
      const double sc = scale ? scale[f] : 1.0;
      const double sh = shift ? shift[f] : 0.0;
      const double wf = w[(size_t)c * F + f] * sc;
      w[(size_t)c * F + f] = wf;
      const double p = -(sh * wf);
      const double pe = -std::fma(sh, wf, p);  // sh * wf + p exactly, negated: p + pe = -sh * wf
      const double t = s + p;
      comp += fabs(s) >= fabs(p) ? (s - t) + p : (p - t) + s;
      comp += pe;
      s = t;
      mag += fabs(p);
    }
    b[c] = s + comp;
    bmag[c] = mag;
  }
  // the fold's own rounding (DESIGN.md 3.2): w'_cf and scikit-learn's z_f = (x_f - mean_f) / scale_f each round
  // relatively (2u both), which moves a score by <= 4.01 u sum_f |z_f w_cf| <= 4.01 u (a + bmag); b'_c errs by <= u |b'_c|
  // + O(F u^2) bmag.  fold_rel = 8u covers both against the bound's a = max_c (sum_f |x_f w'_cf| + bmag_c).
  const double fold_rel = (shift || scale) ? 8.0 * 1.1102230246251565e-16 : 0.0;
  return upload_model(e, m, w, b, bmag, fold_rel);
}

void uml_model_free(uml_model* m) {
  if (!m) return;
  if (m->e) cudaSetDevice(m->e->device);
  cudaFree(m->d_wt);
  cudaFree(m->d_bias);
  cudaFree(m->d_tc);
  cudaFree(m->d_w64);
  cudaFree(m->d_b64);
  delete m;
}

// ---------------------------------------------------------------------------------------------------------------
// batch
// ---------------------------------------------------------------------------------------------------------------
static int encode_map(uml_engine* e, CUtensorMap* map, const float* x, int64_t n_rows, int F, int64_t ld,
                      int box_rows = uml::kTileRows) {
  if (((uintptr_t)x & 15) != 0 || (ld % 4) != 0) UML_FAIL(e, UML_ERR_UNSUPPORTED, "rows must be 16-byte aligned with ld %% 4 == 0");
  if (n_rows >= (1ll << 31) - uml::kTileRows) UML_FAIL(e, UML_ERR_UNSUPPORTED, "more than 2^31 rows in one batch");
  cuuint64_t gdim[2] = {(cuuint64_t)F, (cuuint64_t)n_rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)uml::kChunkF, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = e->encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)x, gdim, gstride, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) UML_FAIL(e, UML_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) for %lld x %d ld %lld", (int)r,
                                  (long long)n_rows, F, (long long)ld);
  return UML_OK;
}

static int linear_box_rows_for(int F) { return uml::linear_box_rows((F + uml::kChunkF - 1) / uml::kChunkF * uml::kChunkF); }

// both tensor maps of a batch: the MLP kernels' 128-row boxes and the linear tile kernel's
static int encode_batch_maps(uml_engine* e, uml_batch* b) {
  int rc = encode_map(e, &b->map, b->x, b->n_rows, b->n_features, b->ld);
  if (rc == UML_OK) rc = encode_map(e, &b->lin_map, b->x, b->n_rows, b->n_features, b->ld, linear_box_rows_for(b->n_features));
  b->has_map = rc == UML_OK;
  return rc;
}

// the compact fp16 copy of a staged batch whose staging pass found every value to be an fp16 value (stage.not_f16 == 0):
// one pack kernel from the fp32 rows and its tensor map.  The copy is an optimisation: when there is no room for it the
// batch keeps the fp32 route, and the call still succeeds.
static int build_half_copy(uml_engine* e, uml_batch* b) {
  const int F = b->n_features;
  const int64_t ldh = uml::linear_half_ld(F);
  if (cudaMalloc(&b->xh, (size_t)b->n_rows * ldh * 2) != cudaSuccess) {
    (void)cudaGetLastError();
    b->xh = nullptr;
    return UML_OK;
  }
  b->ldh = ldh;
  UML_CUDA(e, cudaMemsetAsync(&e->d_stage->negative, 0, sizeof(unsigned long long), e->stream));
  UML_CUDA(e, uml::launch_pack_half(b->x, b->ld, b->n_rows, F, b->xh, ldh, &e->d_stage->negative, e->stream));
  UML_CUDA(e, cudaMemcpyAsync(&e->h->stage.negative, &e->d_stage->negative, sizeof(unsigned long long),
                              cudaMemcpyDeviceToHost, e->stream));
  cuuint64_t gdim[2] = {(cuuint64_t)F, (cuuint64_t)b->n_rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ldh * 2};
  cuuint32_t box[2] = {(cuuint32_t)uml::kHalfBoxF, (cuuint32_t)uml::kTileRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = e->encode(&b->half_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, b->xh, gdim, gstride, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) UML_FAIL(e, UML_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) for the fp16 copy, %lld x %d", (int)r,
                                  (long long)b->n_rows, F);
  UML_CUDA(e, cudaStreamSynchronize(e->stream));  // later calls may run on another stream (uml_engine_set_stream)
  b->has_half = true;
  b->half_nonneg = e->h->stage.negative == 0;
  return UML_OK;
}

// UML_B200_COMPACT_ROWS=0 makes the linear tile kernel read the fp32 rows of a batch that has an fp16 copy (test and A/B
// hook, read per call)
static bool compact_rows_enabled() {
  const char* env = getenv("UML_B200_COMPACT_ROWS");
  return !(env && env[0] == '0');
}

int uml_batch_from_device(uml_engine* e, uml_batch** out, const void* dev_ptr, int64_t n_rows, int n_features,
                          int64_t ld) {
  if (!e || !out || (!dev_ptr && n_rows > 0) || n_rows < 0 || n_features < 1 || ld < n_features) return UML_ERR_INVALID;
  *out = nullptr;
  UML_CUDA(e, cudaSetDevice(e->device));
  uml_batch* b = new uml_batch();
  b->e = e;
  b->x = (float*)dev_ptr;
  b->n_rows = n_rows;
  b->n_features = n_features;
  b->ld = ld;
  b->owns = false;
  if (n_rows > 0) {
    int rc = encode_batch_maps(e, b);
    if (rc != UML_OK && rc != UML_ERR_UNSUPPORTED) {
      delete b;
      return rc;
    }
  }
  *out = b;
  return UML_OK;
}

struct SrcLayout {
  bool feature_major;
  int64_t pitch_elems;
  int elem;
};

static int classify_layout(uml_engine* e, int64_t n_rows, int F, int64_t rs, int64_t cs, int dtype, SrcLayout* L) {
  const int elem = dtype_size(dtype);
  if (!elem) UML_FAIL(e, UML_ERR_INVALID, "unknown dtype %d", dtype);
  L->elem = elem;
  if (cs == elem || F == 1) {
    if (rs % elem != 0 || rs < (int64_t)F * elem) {
      if (n_rows > 1) UML_FAIL(e, UML_ERR_UNSUPPORTED, "row stride %lld not a multiple of the element size / overlaps", (long long)rs);
      rs = (int64_t)F * elem;
    }
    L->feature_major = false;
    L->pitch_elems = rs / elem;
    return UML_OK;
  }
  if (rs == elem || n_rows == 1) {
    if (cs % elem != 0 || cs < n_rows * elem) UML_FAIL(e, UML_ERR_UNSUPPORTED, "column stride %lld unsupported", (long long)cs);
    L->feature_major = true;
    L->pitch_elems = cs / elem;
    return UML_OK;
  }
  UML_FAIL(e, UML_ERR_UNSUPPORTED, "features must be contiguous along rows or along columns (strides %lld, %lld bytes)",
           (long long)rs, (long long)cs);
}

// copy rows [r0, r0+rows) of the host source into device chunk buffer `dst` (compact: pitch = F or rows elements)
static cudaError_t copy_chunk_h2d(void* dst, const void* host, const SrcLayout& L, int64_t r0, int64_t rows, int F,
                                  cudaStream_t s) {
  const char* src = (const char*)host;
  if (!L.feature_major) {
    const size_t width = (size_t)F * L.elem;
    const size_t spitch = (size_t)L.pitch_elems * L.elem;
    if (spitch == width) return cudaMemcpyAsync(dst, src + (size_t)r0 * spitch, width * rows, cudaMemcpyHostToDevice, s);
    return cudaMemcpy2DAsync(dst, width, src + (size_t)r0 * spitch, spitch, width, (size_t)rows, cudaMemcpyHostToDevice, s);
  }
  const size_t width = (size_t)rows * L.elem;
  const size_t spitch = (size_t)L.pitch_elems * L.elem;
  return cudaMemcpy2DAsync(dst, width, src + (size_t)r0 * L.elem, spitch, width, (size_t)F, cudaMemcpyHostToDevice, s);
}

static bool host_ptr_is_pinned(const void* p) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

static bool lossy_capable(int dtype) { return dtype == UML_F64 || dtype == UML_I64 || dtype == UML_I32; }

// gather tasks for rows [r0, r0+rows) of the host source into a compact chunk (row-major [rows][F] or feature-major
// [F][rows]) at `dst`; contiguous runs are cut into <= 1 MiB pieces so the pool's threads share them
static void build_gather_tasks(std::vector<CopyPool::Task>& tasks, char* dst, const void* host, const SrcLayout& L,
                               int64_t r0, int64_t rows, int F, std::atomic<int>* narrow = nullptr) {
  tasks.clear();
  const char* src = (const char*)host;
  const size_t piece = 1u << 20;
  // narrow (float64 source only, contiguous runs): the destination holds float32, so it advances half as fast
  auto add_run = [&](char* d, const char* s_, size_t n) {
    for (size_t o = 0; o < n; o += piece) {
      CopyPool::Task t{d + (narrow ? o / 2 : o), s_ + o, std::min(piece, n - o)};
      t.narrow = narrow;
      tasks.push_back(t);
    }
  };
  if (!L.feature_major) {
    const size_t width = (size_t)F * L.elem, spitch = (size_t)L.pitch_elems * L.elem;
    if (spitch == width) {
      add_run(dst, src + (size_t)r0 * spitch, width * (size_t)rows);
    } else {
      // strided rows (a column slice of a wider C-order array): blocks of rows, each row its own run
      const int64_t rows_per_task = std::max<int64_t>(1, (int64_t)(piece / width));
      for (int64_t r = 0; r < rows; r += rows_per_task) {
        const int64_t n = std::min(rows_per_task, rows - r);
        tasks.push_back({dst + (size_t)r * width, src + (size_t)(r0 + r) * spitch, width, (size_t)n, width, spitch});
      }
    }
  } else {
    const size_t run = (size_t)rows * L.elem, spitch = (size_t)L.pitch_elems * L.elem;
    for (int f = 0; f < F; ++f)
      add_run(dst + (size_t)f * (narrow ? run / 2 : run), src + (size_t)f * spitch + (size_t)r0 * L.elem, run);
  }
}

// CPUs this process can use: scheduler affinity, capped by the cgroup CPU quota (v2 cpu.max, v1 cfs_quota_us)
static int usable_cpus(int* logical = nullptr) {
  int n = (int)std::thread::hardware_concurrency();
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof(set), &set) == 0) n = CPU_COUNT(&set);
  if (n <= 0) n = 4;
  if (logical) *logical = n;  // CPUs the scheduler may place threads on (before the quota)
  auto read_two = [](const char* path, long long* a, long long* b) -> bool {
    FILE* f = fopen(path, "r");
    if (!f) return false;
    char first[64] = {0};
    const int got = fscanf(f, "%63s %lld", first, b);
    fclose(f);
    if (got < 1 || strcmp(first, "max") == 0) return false;
    *a = atoll(first);
    return got == 2;
  };
  long long quota = 0, period = 0;
  if (read_two("/sys/fs/cgroup/cpu.max", &quota, &period) && quota > 0 && period > 0) {
    n = std::min<long long>(n, std::max<long long>(1, quota / period));
  } else {
    FILE* fq = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r");
    FILE* fp = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
    if (fq && fp && fscanf(fq, "%lld", &quota) == 1 && fscanf(fp, "%lld", &period) == 1 && quota > 0 && period > 0)
      n = std::min<long long>(n, std::max<long long>(1, quota / period));
    if (fq) fclose(fq);
    if (fp) fclose(fp);
  }
  return n;
}

// pinned bounce buffers (3 slots) + the copy pool, created on first use
static int grow_bounce(uml_engine* e, int64_t bytes) {
  const int rc = grow(e, e->h_bounce, bytes);
  if (rc != UML_OK) return rc;
  if (!e->pool) {
    int n = 0;
    if (const char* env = getenv("UML_B200_COPY_THREADS")) n = atoi(env);
    // default: sized from the CPU time this process may really use (affinity and cgroup quota - the GPU boxes give a
    // container a 16-CPU quota on 128 logical CPUs).  The gather threads are stalled on host memory most of the time
    // and idle between chunks, so 1.5 x the quota is where the 10M x 64 float64 frame gathers fastest on those boxes
    // (threads: pipeline ms  10: 98, 14: 99, 20: 77-89, 24: 70, 28: 74, 32: 70, 40: 77-116, 56: 133 - past ~2 x the
    // quota CFS throttles every thread for the rest of the period).  Never more than the logical CPUs minus two (the
    // caller's thread fills the result list meanwhile), at most 32, and the CPUs are shared by the ranks of this node
    // (torchrun exports LOCAL_WORLD_SIZE).
    if (n <= 0) {
      int ranks = 1;
      if (const char* lw = getenv("LOCAL_WORLD_SIZE")) ranks = std::max(1, atoi(lw));
      int logical = 0;
      const int quota = usable_cpus(&logical);
      n = std::min(32, std::max(1, std::min(logical - 2, quota * 3 / 2) / ranks));
    }
    e->pool = new CopyPool(n - 1);  // the calling thread is the n-th worker
  }
  return UML_OK;
}

static bool want_bounce(const void* host_ptr, int64_t bytes) {
  return bytes >= (8ll << 20) && !host_ptr_is_pinned(host_ptr) && !getenv("UML_B200_NO_BOUNCE");
}

int uml_stage_rows(uml_engine* e, uml_batch** out, const void* host_ptr, int64_t n_rows, int n_features,
                   int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, uint32_t flags) {
  if (!e || !out || (!host_ptr && n_rows > 0) || n_rows < 0 || n_features < 1) return UML_ERR_INVALID;
  *out = nullptr;
  UML_CUDA(e, cudaSetDevice(e->device));
  (void)cudaGetLastError();
  SrcLayout L{};
  int rc = UML_OK;
  if (n_rows > 0 && (rc = classify_layout(e, n_rows, n_features, row_stride_bytes, col_stride_bytes, src_dtype, &L)) != UML_OK)
    return rc;
  const int F = n_features;
  const int64_t ld = (F + 3) / 4 * 4;
  const bool check = !(flags & UML_STAGE_SKIP_FINITE_CHECK);
  // float64 / int64 / int32 values may not survive the fp32 down-cast (|int32| > 2^24 does not)
  const bool want64 = (flags & UML_STAGE_KEEP_F64) && (src_dtype == UML_F64 || src_dtype == UML_I64 || src_dtype == UML_I32);

  // the half-built batch is freed on every early return
  std::unique_ptr<uml_batch, decltype(&uml_batch_free)> b(new uml_batch(), uml_batch_free);
  b->e = e;
  b->n_rows = n_rows;
  b->n_features = F;
  b->ld = ld;
  b->owns = true;
  if (n_rows == 0) {
    *out = b.release();
    return UML_OK;
  }
  cudaError_t ce;
  if ((ce = cudaMalloc((void**)&b->x, (size_t)n_rows * ld * 4)) != cudaSuccess) {
    e->last_error = std::string("cudaMalloc(batch): ") + cudaGetErrorString(ce);
    return ce == cudaErrorMemoryAllocation ? UML_ERR_NOMEM : UML_ERR_CUDA;
  }
  if (want64) {
    b->ld64 = F;
    if ((ce = cudaMalloc((void**)&b->x64, (size_t)n_rows * F * 8)) != cudaSuccess) {
      e->last_error = std::string("cudaMalloc(batch f64): ") + cudaGetErrorString(ce);
      return ce == cudaErrorMemoryAllocation ? UML_ERR_NOMEM : UML_ERR_CUDA;
    }
  }
  cudaStream_t cs = e->stream;
  UML_CUDA_DRAIN(e, cudaMemsetAsync(e->d_stage, 0, sizeof(StageResult), cs));

  // already the resident layout and page-locked: one straight H2D, then the finiteness scan (a large pageable source
  // goes through the chunked path instead, where host threads feed pinned bounce buffers)
  const bool direct = !L.feature_major && src_dtype == UML_F32 && L.pitch_elems == ld &&
                      !want_bounce(host_ptr, n_rows * (int64_t)F * L.elem);
  if (direct) {
    UML_CUDA_DRAIN(e, cudaMemcpyAsync(b->x, host_ptr, (size_t)n_rows * ld * 4, cudaMemcpyHostToDevice, cs));
    if (check) UML_CUDA_DRAIN(e, uml::launch_finite_scan(b->x, ld, n_rows, F, e->d_stage, cs));
  } else {
    // chunked: H2D of raw source bytes on the copy stream, transpose/convert kernel on the compute stream
    const int64_t row_bytes = (int64_t)F * L.elem;
    int64_t chunk_rows = std::max<int64_t>(1024, (64ll << 20) / row_bytes);
    chunk_rows = std::min<int64_t>((chunk_rows + 31) / 32 * 32, std::max<int64_t>(n_rows, 1));
    if ((rc = grow(e, e->d_chunk, chunk_rows * row_bytes)) != UML_OK) return rc;
    // pageable frames: a few host threads gather each chunk into a pinned bounce buffer (see CopyPool)
    const bool bounce = want_bounce(host_ptr, n_rows * row_bytes);
    if (bounce && (rc = grow_bounce(e, chunk_rows * row_bytes)) != UML_OK) return rc;
    std::vector<CopyPool::Task> tasks;
    int slot = 0;
    bool used[3] = {false, false, false};
    for (int64_t r0 = 0; r0 < n_rows; r0 += chunk_rows, slot = (slot + 1) % 3) {
      const int64_t rows = std::min(chunk_rows, n_rows - r0);
      char* raw = e->d_chunk.p[slot];
      if (used[slot]) UML_CUDA_DRAIN(e, cudaStreamWaitEvent(e->copy_stream, e->chunk_ev[3 + slot], 0));  // convert done
      if (bounce) {
        // previous H2D has left the bounce buffer
        if (used[slot]) UML_CUDA_DRAIN(e, cudaEventSynchronize(e->chunk_ev[slot]));
        build_gather_tasks(tasks, e->h_bounce.p[slot], host_ptr, L, r0, rows, F);
        e->pool->run(tasks);
        UML_CUDA_DRAIN(e, cudaMemcpyAsync(raw, e->h_bounce.p[slot], (size_t)(rows * row_bytes), cudaMemcpyHostToDevice,
                                          e->copy_stream));
      } else {
        UML_CUDA_DRAIN(e, copy_chunk_h2d(raw, host_ptr, L, r0, rows, F, e->copy_stream));
      }
      UML_CUDA_DRAIN(e, cudaEventRecord(e->chunk_ev[slot], e->copy_stream));
      UML_CUDA_DRAIN(e, cudaStreamWaitEvent(cs, e->chunk_ev[slot], 0));
      UML_CUDA_DRAIN(e, uml::launch_stage_convert(raw, src_dtype, L.feature_major, L.feature_major ? rows : F, rows, F,
                                                  b->x + r0 * ld, ld, b->x64 ? b->x64 + r0 * b->ld64 : nullptr, b->ld64,
                                                  e->d_stage, check, cs));
      UML_CUDA_DRAIN(e, cudaEventRecord(e->chunk_ev[3 + slot], cs));
      used[slot] = true;
    }
  }
  UML_CUDA_DRAIN(e, cudaMemcpyAsync(&e->h->stage, e->d_stage, sizeof(StageResult), cudaMemcpyDeviceToHost, cs));
  UML_CUDA_DRAIN(e, cudaStreamSynchronize(cs));
  if (check && e->h->stage.nonfinite) UML_FAIL(e, UML_ERR_NONFINITE, "Input X contains NaN or infinity.");
  b->lossless = direct ? true : e->h->stage.lossy == 0;
  if (check || !direct) b->tf32_exact = e->h->stage.not_tf32 == 0 ? 1 : 0;  // the scan / conversion pass saw every value
  if (b->x64 && b->lossless) {
    cudaFree(b->x64);
    b->x64 = nullptr;
  }
  rc = encode_batch_maps(e, b.get());
  if (rc != UML_OK && rc != UML_ERR_UNSUPPORTED) return rc;
  if (rc == UML_OK && (check || !direct) && e->h->stage.not_f16 == 0 && F <= uml::kHalfBoxF &&
      (rc = build_half_copy(e, b.get())) != UML_OK)
    return rc;
  *out = b.release();
  return UML_OK;
}

int uml_batch_info(const uml_batch* b, int64_t* n_rows, int* n_features, int64_t* ld, const void** dev_ptr,
                   int* lossless) {
  if (!b) return UML_ERR_INVALID;
  if (n_rows) *n_rows = b->n_rows;
  if (n_features) *n_features = b->n_features;
  if (ld) *ld = b->ld;
  if (dev_ptr) *dev_ptr = b->x;
  if (lossless) *lossless = b->lossless ? 1 : 0;
  return UML_OK;
}

void uml_batch_free(uml_batch* b) {
  if (!b) return;
  if (b->e) cudaSetDevice(b->e->device);
  if (b->owns) cudaFree(b->x);
  cudaFree(b->x64);
  cudaFree(b->xh);
  delete b;
}

// ---------------------------------------------------------------------------------------------------------------
// predict
// ---------------------------------------------------------------------------------------------------------------
// enqueue the scoring of one resident block of rows on e->stream; no host synchronisation.  timed: ev[2] ends the
// scoring kernel (the caller brackets the step with ev[1] / ev[3]).  half_map (optional): the rows' compact fp16
// copy, which the tile kernel then reads; *x_elem_bytes (optional) gets the bytes per feature it read (2 or 4).
static int enqueue_predict(uml_engine* e, const uml_model* m, const LinearLaunch& l, const CUtensorMap* map,
                           const CUtensorMap* half_map, int mode, bool timed, int* launches, int* path,
                           int* x_elem_bytes = nullptr, bool half_nonneg = false) {
  const FlagList fl = flag_list(e);
  const bool exact = mode == UML_PREDICT_EXACT;
  std::string why;
  const bool tma = map != nullptr && uml::linear_tma_supported(m->dm, &why);
  if (tma) {
    NvtxRange r_score("uml:score");
    std::string err;
    bool need_rescore = false;
    if (half_map && !uml::linear_half_rows_ok(m->dm.f_pad)) half_map = nullptr;
    cudaError_t ce = uml::launch_linear_tma(*map, half_map, m->dm, l, exact, fl, e->info.sm_count, e->stream, &err,
                                            &need_rescore, half_nonneg);
    if (ce != cudaSuccess) UML_FAIL(e, UML_ERR_CUDA, "linear_argmax_tma launch: %s %s", cudaGetErrorString(ce), err.c_str());
    *launches += 1;
    *path = 1;
    if (x_elem_bytes) *x_elem_bytes = half_map ? 2 : 4;
    if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], e->stream));
    if (need_rescore) {  // UML_B200_RESCORE_MODE=kernel; in queue mode flagged rows are re-scored by a warp of the tile kernel
      NvtxRange r_rescore("uml:rescore_f64");
      UML_CUDA(e, uml::launch_rescore_f64(m->dm, l, fl, false, e->info.sm_count, e->stream));
      *launches += 1;
    }
  } else {
    NvtxRange r_score("uml:score_f64_generic");
    UML_CUDA(e, uml::launch_rescore_f64(m->dm, l, fl, true, e->info.sm_count, e->stream));
    *launches += 1;
    *path = 2;
    if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], e->stream));
  }
  return UML_OK;
}

// the MLP counterpart of enqueue_predict: the scoring kernel of `route` (mlp_route), the fp64 re-score of its flagged
// rows when exact, and for the CUDA-core kernel with peers, the scatter of its labels.  `out` holds the row count and
// where the labels go.  No host synchronisation; timed: ev[2] ends the scoring kernel, as in enqueue_predict.
static int enqueue_mlp(uml_engine* e, const uml::MlpDeviceModel& m, const CUtensorMap& map, const float* x, int64_t ld,
                       const uml::MlpTcLaunch& out, bool exact, int route, bool timed, int* launches, int* path) {
  const FlagList fl = flag_list(e);
  const int sm = e->info.sm_count;
  cudaStream_t s = e->stream;
  *path = route;
  if (route == 2) {
    NvtxRange r_score("uml:mlp_score_f64_generic");
    UML_CUDA(e, uml::launch_mlp_rescore_f64(m, x, ld, out.n_rows, out, fl, true, sm, s));
    *launches += 1;
    if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], s));
  } else {
    // the CUDA-core kernel has no peer stores: it writes int32 labels to scratch (the caller grew e->d_labels to
    // n_rows) and a thin kernel scatters them
    const bool scatter = route == 3 && out.targets.n_peers > 0;
    uml::MlpTcLaunch own = out;
    if (scatter) own.targets.labels = e->d_labels.p[0];
    {
      NvtxRange r_score(route == 5 ? "uml:mlp_score_tc" : "uml:mlp_score_ffma");
      if (route == 5) UML_CUDA(e, uml::launch_mlp_tc(map, m, out, exact, fl, sm, s));
      else UML_CUDA(e, uml::launch_mlp_tma(map, m, x, out.n_rows, own.targets.labels, exact, fl, sm, s));
      *launches += 1;
      if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], s));
    }
    if (exact) {
      NvtxRange r_rescore("uml:mlp_rescore_f64");
      UML_CUDA(e, uml::launch_mlp_rescore_f64(m, x, ld, out.n_rows, own, fl, false, sm, s));
      *launches += 1;
    }
    if (scatter) {
      UML_CUDA(e, uml::launch_labels_scatter(own.targets.labels, out.n_rows, out.targets, sm, s));
      *launches += 1;
    }
  }
  return UML_OK;
}

// uml_stats.path of the float64 scores kernel: 6 for decision_function scores, 7 for probabilities or their logs
static int f64_path(int kind) { return kind == uml::kF64Scores ? 6 : 7; }

static int finish_stats(uml_engine* e, uml_stats* stats, int64_t n_rows, int launches, int path, bool timed,
                        bool kernel_events = true) {
  // counters -> pinned mirror, then synchronise and report
  UML_CUDA(e, cudaMemcpyAsync(&e->h->flag_count, e->d_flag_count, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  UML_CUDA(e, cudaMemcpyAsync(e->h->counters, e->d_counters, sizeof(e->h->counters), cudaMemcpyDeviceToHost, e->stream));
  if (timed) UML_CUDA(e, cudaEventRecord(e->ev[4], e->stream));
  UML_CUDA(e, cudaStreamSynchronize(e->stream));
  if (stats) {
    stats->n_rows = n_rows;
    stats->n_ambiguous = (int64_t)e->h->counters[uml::kCounterAmbiguous];
    stats->n_nonfinite = (int64_t)e->h->counters[uml::kCounterNonfinite];
    stats->n_flagged = (int64_t)e->h->counters[uml::kCounterFlagged];
    stats->kernel_launches = launches;
    stats->path = path;
    if (timed) {
      float ms = 0.f;
      if (kernel_events) {
        if (cudaEventElapsedTime(&ms, e->ev[1], e->ev[2]) == cudaSuccess) stats->kernel_ms = ms;
        if (cudaEventElapsedTime(&ms, e->ev[2], e->ev[3]) == cudaSuccess) stats->recheck_ms = ms;
      }
      if (cudaEventElapsedTime(&ms, e->ev[0], e->ev[4]) == cudaSuccess) stats->total_ms = ms;
      (void)cudaGetLastError();  // never leave a stale error behind for the next launch check
    }
  }
  if (e->h->counters[uml::kCounterNonfinite] > 0) UML_FAIL(e, UML_ERR_NONFINITE, "Input X contains NaN or infinity.");
  return UML_OK;
}

// the checks every predict call makes of its mode and of the rows' feature count.  `model` names the model as the
// message does: "estimator" as scikit-learn words it, "module" as the torch app does.  A call without a mode passes FAST.
static int check_mode_features(uml_engine* e, int mode, int n_features, int want, const char* model) {
  if (mode != UML_PREDICT_FAST && mode != UML_PREDICT_EXACT) UML_FAIL(e, UML_ERR_INVALID, "mode %d", mode);
  if (n_features != want)
    UML_FAIL(e, UML_ERR_SHAPE, "X has %d features, but the %s is expecting %d features as input.", n_features, model,
             want);
  return UML_OK;
}

// What a predict call on a resident batch hands predict_resident besides its steps: its model's shape, its outputs
// (out[1] is optional: top-k's probabilities) with their bytes per row, in host or device memory, its mode and stats.
// always_sync: synchronous even with device outputs and no stats, so that NaN / Inf are reported on return.
// n_peers / label_bytes: the labels' fused exchange (with peers, out[0] is NULL and each model's labels step serves them).
struct ResidentCall {
  int n_classes, n_features;
  const char* model;
  void* out[2];
  int64_t row_bytes[2];
  int on_device, mode;
  uml_stats* stats;
  bool always_sync = false;
  int n_peers = 0, label_bytes = 4;
};

// One predict call on a resident batch: the checks, device setup, output scratch, events, counters, D2H and stats
// that every such call shares.  prepare() makes the call's host-side checks and choices before the first timed stream
// operation; score(out, timed, &launches, &path, &x_elem_bytes) enqueues its own step between ev[1] and ev[3], writing
// output i to out[i] (the caller's device memory, or scratch bound for host memory) and recording ev[2] after its
// scoring kernel when timed.  An asynchronous call (device outputs, no stats) returns once the step is enqueued.
extern "C++" {  // a template cannot have the C linkage of the ABI section around it
template <class Prepare, class Score>
static int predict_resident(uml_engine* e, const uml_batch* b, const ResidentCall& c, Prepare&& prepare, Score&& score) {
  if (!e || !b) return UML_ERR_INVALID;
  if (!c.out[0] && b->n_rows > 0 && c.n_peers == 0) return UML_ERR_INVALID;
  if (c.n_peers < 0 || c.n_peers > 8) UML_FAIL(e, UML_ERR_INVALID, "n_peers %d (max 8)", c.n_peers);
  if (c.n_peers > 0 && c.label_bytes != 1 && c.label_bytes != 4)
    UML_FAIL(e, UML_ERR_INVALID, "label_bytes %d", c.label_bytes);
  if (c.n_peers > 0 && c.label_bytes == 1 && c.n_classes > 256)
    UML_FAIL(e, UML_ERR_UNSUPPORTED, "byte labels need n_classes <= 256 (model has %d)", c.n_classes);
  int rc;
  if ((rc = check_mode_features(e, c.mode, b->n_features, c.n_features, c.model)) != UML_OK) return rc;
  UML_CUDA(e, cudaSetDevice(e->device));
  (void)cudaGetLastError();
  uml_stats* stats = c.stats;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (b->n_rows == 0) return UML_OK;
  const bool timed = stats != nullptr;
  const bool sync_call = stats || !c.on_device || c.always_sync;
  if (c.mode == UML_PREDICT_EXACT && (rc = grow(e, e->d_flag_rows, b->n_rows)) != UML_OK) return rc;
  if ((rc = prepare()) != UML_OK) return rc;
  void* out[2] = {c.out[0], c.out[1]};
  int64_t d2h = 0;
  if (!c.on_device) {  // back to back in scratch
    for (int i = 0; i < 2; ++i) d2h += c.out[i] ? b->n_rows * c.row_bytes[i] : 0;
    if ((rc = grow(e, e->d_result, d2h)) != UML_OK) return rc;
    out[0] = e->d_result.p[0];
    if (c.out[1]) out[1] = e->d_result.p[0] + b->n_rows * c.row_bytes[0];
  }
  if (timed) UML_CUDA(e, cudaEventRecord(e->ev[0], e->stream));
  // The asynchronous step needs no memset at all: the flag list is handed back empty by the previous re-score kernel.
  if (sync_call) UML_CUDA(e, reset_counters(e, e->stream));
  if (timed) UML_CUDA(e, cudaEventRecord(e->ev[1], e->stream));
  int launches = 0, path = 0, x_elem_bytes = 0;
  if ((rc = score(out, timed, &launches, &path, &x_elem_bytes)) != UML_OK) return rc;
  if (timed) UML_CUDA(e, cudaEventRecord(e->ev[3], e->stream));
  if (!sync_call) return UML_OK;
  for (int i = 0; i < 2; ++i)
    if (!c.on_device && c.out[i])
      UML_CUDA(e, cudaMemcpyAsync(c.out[i], out[i], (size_t)(b->n_rows * c.row_bytes[i]), cudaMemcpyDeviceToHost,
                                  e->stream));
  rc = finish_stats(e, stats, b->n_rows, launches, path, timed);
  if (stats) {
    stats->d2h_bytes = d2h;
    stats->x_elem_bytes = x_elem_bytes;
  }
  return rc;
}
}  // extern "C++"

static int no_prepare() { return UML_OK; }

static int linear_predict_resident(uml_engine* e, const uml_model* m, const uml_batch* b, int32_t* labels_out,
                                   int labels_on_device, void* const* peers, int n_peers, int64_t row_offset,
                                   int label_bytes, int mode, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  auto score = [&](void* const* out, bool timed, int* launches, int* path, int* elem_bytes) {
    LinearLaunch l{};
    l.x = b->x;
    l.x64 = b->x64;
    l.ld = b->ld;
    l.ld64 = b->ld64;
    l.n_rows = b->n_rows;
    uml::LabelTargets& t = l.targets;
    t.labels = static_cast<int32_t*>(out[0]);
    t.wire_u8 = n_peers > 0 && label_bytes == 1 ? 1 : 0;
    t.row_offset = row_offset;
    // fused int32 exchange: entry 0 is this rank's own full-length vector, the local label target.  Byte vectors are
    // all peers (own vector included); no int32 copy is kept.
    const int own = n_peers > 0 && !t.wire_u8 ? 1 : 0;
    if (own) t.labels = static_cast<int32_t*>(peers[0]) + row_offset;
    t.n_peers = n_peers - own;
    for (int i = 0; i < t.n_peers; ++i) t.peers[i] = peers[own + i];
    const CUtensorMap* half = b->has_half && compact_rows_enabled() ? &b->half_map : nullptr;
    *elem_bytes = 4;
    return enqueue_predict(e, m, l, b->has_map ? &b->lin_map : nullptr, half, mode, timed, launches, path, elem_bytes,
                           b->half_nonneg);
  };
  ResidentCall c{m->dm.n_classes, m->n_features_in, "estimator", {labels_out, nullptr}, {4, 0}, labels_on_device, mode,
                 stats};
  c.n_peers = n_peers;
  c.label_bytes = label_bytes;
  return predict_resident(e, b, c, no_prepare, score);
}

int uml_linear_predict(uml_engine* e, const uml_model* m, const uml_batch* b, int32_t* labels_out,
                       int labels_on_device, int mode, uml_stats* stats) {
  return linear_predict_resident(e, m, b, labels_out, labels_on_device, nullptr, 0, 0, 4, mode, stats);
}

int uml_linear_predict_peers(uml_engine* e, const uml_model* m, const uml_batch* b, void* const* peer_labels,
                             int n_peers, int64_t row_offset, int label_bytes, int mode, uml_stats* stats) {
  if (!peer_labels || n_peers < 1) return UML_ERR_INVALID;
  // peer_labels[0] must be this rank's own vector (local target); labels land at peer_labels[i] + row_offset for all i
  return linear_predict_resident(e, m, b, nullptr, 1, peer_labels, n_peers, row_offset, label_bytes, mode, stats);
}

// labels (device, int32 or uint8 indices) -> classes_[idx] as float64 in HOST memory: the device-side classes_.take of
// sklearn/linear_model/_base.py:423 followed by the float conversion of the canonical predictor (README.md:92)
int uml_labels_take(uml_engine* e, const void* labels_dev, int label_bytes, int64_t n, const double* classes_host,
                    int n_classes, double* out_host) {
  if (!e || (!labels_dev && n > 0) || !classes_host || n_classes < 1 || (!out_host && n > 0) || n < 0) return UML_ERR_INVALID;
  if (label_bytes != 1 && label_bytes != 4) UML_FAIL(e, UML_ERR_INVALID, "label_bytes %d", label_bytes);
  UML_CUDA(e, cudaSetDevice(e->device));
  if (n == 0) return UML_OK;
  int rc;
  if ((rc = grow(e, e->d_classes, n_classes)) != UML_OK || (rc = grow(e, e->d_result, n * 8)) != UML_OK) return rc;
  double* d_out = reinterpret_cast<double*>(e->d_result.p[0]);
  cudaError_t ce;
  if ((ce = cudaMemcpyAsync(e->d_classes.p[0], classes_host, (size_t)n_classes * 8, cudaMemcpyHostToDevice, e->stream)) != cudaSuccess ||
      (ce = uml::launch_labels_take(labels_dev, label_bytes, n, e->d_classes.p[0], n_classes, d_out, e->stream)) != cudaSuccess ||
      (ce = cudaMemcpyAsync(out_host, d_out, (size_t)n * 8, cudaMemcpyDeviceToHost, e->stream)) != cudaSuccess ||
      (ce = cudaStreamSynchronize(e->stream)) != cudaSuccess) {
    cudaStreamSynchronize(e->stream);
    UML_FAIL(e, UML_ERR_CUDA, "uml_labels_take: %s", cudaGetErrorString(ce));
  }
  return UML_OK;
}

// number of rows whose predicted class value equals the target (the numerator of accuracy_score in the reference's
// evaluator, README.md:94-100); targets are float64 in HOST memory
int uml_labels_count_equal(uml_engine* e, const void* labels_dev, int label_bytes, int64_t n, const double* classes_host,
                           int n_classes, const double* targets_host, int64_t* count_out) {
  if (!e || (!labels_dev && n > 0) || !classes_host || n_classes < 1 || (!targets_host && n > 0) || !count_out || n < 0)
    return UML_ERR_INVALID;
  if (label_bytes != 1 && label_bytes != 4) UML_FAIL(e, UML_ERR_INVALID, "label_bytes %d", label_bytes);
  UML_CUDA(e, cudaSetDevice(e->device));
  *count_out = 0;
  if (n == 0) return UML_OK;
  int rc;
  if ((rc = grow(e, e->d_classes, n_classes)) != UML_OK || (rc = grow(e, e->d_targets, n)) != UML_OK) return rc;
  cudaError_t ce;
  if ((ce = cudaMemcpyAsync(e->d_classes.p[0], classes_host, (size_t)n_classes * 8, cudaMemcpyHostToDevice, e->stream)) != cudaSuccess ||
      (ce = cudaMemcpyAsync(e->d_targets.p[0], targets_host, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream)) != cudaSuccess ||
      (ce = cudaMemsetAsync(e->d_counters, 0, sizeof(e->h->counters), e->stream)) != cudaSuccess ||
      (ce = uml::launch_labels_count_equal(labels_dev, label_bytes, n, e->d_classes.p[0], n_classes, e->d_targets.p[0],
                                           e->d_counters, e->stream)) != cudaSuccess ||
      (ce = cudaMemcpyAsync(e->h->counters, e->d_counters, sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream)) != cudaSuccess ||
      (ce = cudaStreamSynchronize(e->stream)) != cudaSuccess) {
    cudaStreamSynchronize(e->stream);
    UML_FAIL(e, UML_ERR_CUDA, "uml_labels_count_equal: %s", cudaGetErrorString(ce));
  }
  *count_out = (int64_t)e->h->counters[0];
  return UML_OK;
}

// top-k hit counts of the quickdraw template's accuracy(output, target, topk) (quickdraw/model.py:20-27):
// hits_out[j] = rows whose target is among their first j + 1 classes, for every j < k, in one pass
int uml_topk_count_hits(uml_engine* e, const int32_t* idx_dev, int k, int64_t n, const double* classes_host,
                        int n_classes, const double* targets_host, int64_t* hits_out) {
  if (!e || (!idx_dev && n > 0) || k < 1 || n < 0 || !classes_host || n_classes < 1 || (!targets_host && n > 0) || !hits_out)
    return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  for (int j = 0; j < k; ++j) hits_out[j] = 0;
  if (n == 0) return UML_OK;
  int rc;
  if ((rc = grow(e, e->d_classes, n_classes)) != UML_OK || (rc = grow(e, e->d_targets, n)) != UML_OK ||
      (rc = grow(e, e->d_hits, k)) != UML_OK)
    return rc;
  std::vector<unsigned long long> first(k);
  cudaStream_t s = e->stream;
  UML_CUDA(e, cudaMemcpyAsync(e->d_classes.p[0], classes_host, (size_t)n_classes * 8, cudaMemcpyHostToDevice, s));
  UML_CUDA(e, cudaMemcpyAsync(e->d_targets.p[0], targets_host, (size_t)n * 8, cudaMemcpyHostToDevice, s));
  UML_CUDA(e, cudaMemsetAsync(e->d_hits.p[0], 0, (size_t)k * 8, s));
  UML_CUDA(e, uml::launch_topk_first_hits(idx_dev, k, n, e->d_classes.p[0], n_classes, e->d_targets.p[0],
                                          e->d_hits.p[0], s));
  UML_CUDA(e, cudaMemcpyAsync(first.data(), e->d_hits.p[0], (size_t)k * 8, cudaMemcpyDeviceToHost, s));
  UML_CUDA(e, cudaStreamSynchronize(s));
  int64_t run = 0;
  for (int j = 0; j < k; ++j) hits_out[j] = run += (int64_t)first[j];
  return UML_OK;
}

int uml_labels_push(uml_engine* e, const void* src, void* const* dst, int n_dst, int64_t bytes) {
  if (!e || (!src && bytes > 0) || !dst || n_dst < 1 || n_dst > 8 || bytes < 0) return UML_ERR_INVALID;
  UML_CUDA(e, cudaSetDevice(e->device));
  UML_CUDA(e, uml::launch_push_bytes(src, dst, n_dst, bytes, e->info.sm_count, e->stream));
  return UML_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// host rows -> host labels
// ---------------------------------------------------------------------------------------------------------------
// are the first rows of a host source tf32 values once cast to fp32 (low 13 mantissa bits zero)?  A cheap guess used
// to pick the MLP kernel for the chunk pipeline; correctness never depends on it
static bool host_sample_is_tf32(const void* host, const SrcLayout& L, int64_t n_rows, int F, int dtype) {
  const int64_t rows = std::min<int64_t>(n_rows, 2048);
  const char* base = (const char*)host;
  for (int64_t r = 0; r < rows; ++r)
    for (int f = 0; f < F; ++f) {
      const size_t i = L.feature_major ? (size_t)f * L.pitch_elems + r : (size_t)r * L.pitch_elems + f;
      float v;
      switch (dtype) {
        case UML_F64: v = (float)((const double*)base)[i]; break;
        case UML_I64: v = (float)((const long long*)base)[i]; break;
        case UML_I32: v = (float)((const int*)base)[i]; break;
        case UML_U8: v = (float)((const unsigned char*)base)[i]; break;
        default: v = ((const float*)base)[i]; break;
      }
      uint32_t bits;
      memcpy(&bits, &v, 4);
      if (bits & 0x1fffu) return false;
    }
  return true;
}

using SmallLaunch = std::function<cudaError_t(const uml::SrcView&, int, cudaStream_t)>;

// One chunk of host rows as the pipeline hands it to a score step
struct Chunk {
  float* x;          // the fp32 rows (staged and checked, unless the step reads the raw chunk)
  int64_t ld, rows;
  uml::SrcView src;  // the caller's own values as they crossed PCIe (a float64 chunk that travelled as fp32 was checked
                     // lossless by the gather threads); rows already in the resident layout: x itself
  std::function<bool()> tf32;  // a host-side guess at whether the rows are tf32 values (MLP kernel choice)
};

// What a call through the chunk pipeline computes: score(chunk, out, &launches, &path) enqueues it on e->stream and
// writes chunk.rows x row_bytes to the device buffer `out`.  n_features / model: as for check_mode_features.
struct ChunkStep {
  int n_features;
  const char* model;
  int64_t row_bytes;
  bool raw;  // reads chunk.src only: no staging kernel or finite scan (the float64 outputs check finiteness themselves)
  std::function<int(const Chunk&, void*, int*, int*)> score;
  std::function<int(int64_t)> prepare;  // optional, given chunk_rows once the pipeline's scratch exists
  // the <= kSmallRows route, none without a kernel: the model uid that keys its graphs, and the classes it writes
  // as float64 in place of the label (class values).  small_rec: the host view of the records the kernel writes in
  // place of labels (row_bytes each; kind / k key its graphs), nullptr for labels
  SmallLaunch small;
  uint64_t small_uid = 0;
  const double* classes = nullptr;
  int n_classes = 0;
  const void* small_rec = nullptr;
  int small_kind = uml::kSmallLabels, small_k = 0;
};

// B <= kSmallRows: request block -> pinned (device-mapped) buffer -> one small-batch kernel (replayed as a CUDA graph)
// -> labels written straight into pinned host memory.  The kernel scores in fp64 (linear_small_kernel from the
// caller's own values, mlp_small_kernel from their fp32 cast), so the result is the exact-mode result for either mode.
// step.small(view, rows, stream) enqueues that kernel on the request block; step.small_uid keys its cached graphs.
// out: the int32 labels, with step.classes classes[label] as float64, or with step.small_rec the kernel's records.
static int predict_host_small(uml_engine* e, const ChunkStep& step, const void* host_ptr, int n_rows, int F,
                              const SrcLayout& L, int src_dtype, void* out, uml_stats* stats) {
  NvtxRange r_all("uml:predict_host_small");
  const size_t width = (size_t)F * L.elem;
  const size_t bytes = width * (size_t)n_rows;
  if (!e->h_req) {
    // zero-copy: the kernel reads the request straight from page-locked host memory over PCIe (16 KiB for 32 x 64
    // float64) and writes the labels straight back - no H2D / D2H copy nodes on the latency path
    UML_CUDA(e, cudaHostAlloc(&e->h_req, (size_t)kSmallBytes, cudaHostAllocMapped));
    UML_CUDA(e, cudaHostGetDevicePointer(&e->d_req, e->h_req, 0));
    void* d_small = nullptr;
    UML_CUDA(e, cudaHostGetDevicePointer(&d_small, e->h->small, 0));
    e->d_small = (uml::SmallResult*)d_small;
  }
  // gather into the pinned request buffer as compact row-major rows (the kernel reads any order, but a compact
  // block keeps the H2D copy one contiguous piece)
  {
    const char* src = (const char*)host_ptr;
    char* dst = (char*)e->h_req;
    if (!L.feature_major) {
      const size_t spitch = (size_t)L.pitch_elems * L.elem;
      if (spitch == width) memcpy(dst, src, bytes);
      else for (int r = 0; r < n_rows; ++r) memcpy(dst + (size_t)r * width, src + (size_t)r * spitch, width);
    } else {
      // feature-major request (a pandas block): typed transpose into rows
      const size_t pitch = (size_t)L.pitch_elems;
      auto transpose = [&](auto* d, const auto* s_) {
        for (int f = 0; f < F; ++f)
          for (int r = 0; r < n_rows; ++r) d[(size_t)r * F + f] = s_[(size_t)f * pitch + r];
      };
      switch (L.elem) {
        case 8: transpose((uint64_t*)dst, (const uint64_t*)src); break;
        case 4: transpose((uint32_t*)dst, (const uint32_t*)src); break;
        default: transpose((uint8_t*)dst, (const uint8_t*)src); break;
      }
    }
  }
  uml::SrcView view{e->d_req, src_dtype, (long long)F, 1};
  auto enqueue = [&](cudaStream_t s) -> cudaError_t { return step.small(view, n_rows, s); };
  const uint64_t model_uid = step.small_uid;
  static const bool no_graph = getenv("UML_B200_NO_GRAPH") != nullptr;
  bool launched = false;
  if (e->small_graph_ok && !no_graph) {
    SmallGraph* hit = nullptr;
    for (auto& g : e->small_graphs)
      if (g.model_uid == model_uid && g.n_rows == n_rows && g.n_features == F && g.dtype == src_dtype &&
          g.kind == step.small_kind && g.k == step.small_k)
        hit = &g;
    if (!hit) {
      cudaGraph_t graph = nullptr;
      cudaGraphExec_t exec = nullptr;
      cudaError_t ce = cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal);
      if (ce == cudaSuccess) {
        cudaError_t body = enqueue(e->stream);
        ce = cudaStreamEndCapture(e->stream, &graph);
        if (body != cudaSuccess) ce = body;
      }
      if (ce == cudaSuccess) ce = cudaGraphInstantiate(&exec, graph, 0);
      if (graph) cudaGraphDestroy(graph);
      if (ce != cudaSuccess) {
        (void)cudaGetLastError();
        e->small_graph_ok = false;  // capture is not available here (e.g. the caller's stream is itself capturing)
      } else {
        if (e->small_graphs.size() >= 16) {  // evict the least recently used
          size_t lru = 0;
          for (size_t i = 1; i < e->small_graphs.size(); ++i)
            if (e->small_graphs[i].last_use < e->small_graphs[lru].last_use) lru = i;
          cudaGraphExecDestroy(e->small_graphs[lru].exec);
          e->small_graphs.erase(e->small_graphs.begin() + (long)lru);
        }
        e->small_graphs.push_back({model_uid, n_rows, F, src_dtype, step.small_kind, step.small_k, exec, 0});
        hit = &e->small_graphs.back();
      }
    }
    if (hit) {
      hit->last_use = ++e->small_tick;
      UML_CUDA(e, cudaGraphLaunch(hit->exec, e->stream));
      launched = true;
    }
  }
  if (!launched) UML_CUDA(e, enqueue(e->stream));
  UML_CUDA(e, cudaStreamSynchronize(e->stream));
  int64_t n_bad = 0, n_amb = 0;
  const double* classes = step.classes;
  if (step.small_rec) memcpy(out, step.small_rec, (size_t)(n_rows * step.row_bytes));
  for (int r = 0; r < n_rows; ++r) {
    const uml::SmallResult& q = e->h->small[r];
    if (!step.small_rec && classes)
      static_cast<double*>(out)[r] = (q.label >= 0 && q.label < step.n_classes) ? classes[q.label] : NAN;
    else if (!step.small_rec)
      static_cast<int32_t*>(out)[r] = q.label;
    n_bad += q.status & 1;
    n_amb += (q.status >> 1) & 1;
  }
  if (stats) {
    stats->n_rows = n_rows;
    stats->n_nonfinite = n_bad;
    stats->n_ambiguous = n_amb;
    stats->kernel_launches = 1;
    stats->path = 4;
    stats->h2d_bytes = (int64_t)bytes;  // read by the kernel over PCIe (zero-copy), not by a copy engine
    stats->d2h_bytes = (int64_t)sizeof(uml::SmallResult) * n_rows + (step.small_rec ? n_rows * step.row_bytes : 0);
  }
  if (n_bad > 0) UML_FAIL(e, UML_ERR_NONFINITE, "Input X contains NaN or infinity.");
  return UML_OK;
}

// host rows -> `out` (host memory, n_rows x step.row_bytes) in chunks: gather / H2D on the copy stream, staging, the
// step and the D2H on e->stream, three chunks in flight.  progress: the asynchronous call's published row count
static int predict_host_impl(uml_engine* e, const ChunkStep& step, const void* host_ptr, int64_t n_rows, int n_features,
                             int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, void* out, int mode,
                             int64_t chunk_rows, uml_stats* stats, std::atomic<int64_t>* progress = nullptr) {
  if (!e || (!host_ptr && n_rows > 0) || (!out && n_rows > 0) || n_rows < 0 || n_features < 1) return UML_ERR_INVALID;
  int rc;
  if ((rc = check_mode_features(e, mode, n_features, step.n_features, step.model)) != UML_OK) return rc;
  UML_CUDA(e, cudaSetDevice(e->device));
  (void)cudaGetLastError();
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n_rows == 0) return UML_OK;
  SrcLayout L{};
  if ((rc = classify_layout(e, n_rows, n_features, row_stride_bytes, col_stride_bytes, src_dtype, &L)) != UML_OK) return rc;
  const int F = n_features;
  if (step.small && n_rows <= kSmallRows && (int64_t)F * L.elem * n_rows <= kSmallBytes) {
    rc = predict_host_small(e, step, host_ptr, (int)n_rows, F, L, src_dtype, out, stats);
    if (progress && rc == UML_OK) progress->store(n_rows);
    return rc;
  }

  NvtxRange r_all("uml:predict_host");
  const int64_t ld = (F + 3) / 4 * 4;
  const bool exact = mode == UML_PREDICT_EXACT;
  const int64_t row_bytes = (int64_t)F * L.elem;
  const int64_t out_bytes = step.row_bytes;
  if (chunk_rows <= 0)
    chunk_rows = std::max<int64_t>(4096, (32ll << 20) / std::max<int64_t>({ld * 4, row_bytes, out_bytes}));
  chunk_rows = std::min<int64_t>((chunk_rows + 127) / 128 * 128, (n_rows + 127) / 128 * 128);
  const bool direct = !L.feature_major && src_dtype == UML_F32 && L.pitch_elems == ld;
  // pageable sources of any size worth the trouble go through pinned bounce buffers filled by the copy pool
  const bool bounce = want_bounce(host_ptr, n_rows * row_bytes);

  if (!direct && (rc = grow(e, e->d_chunk, chunk_rows * row_bytes)) != UML_OK) return rc;
  if ((rc = grow(e, e->d_xchunk, chunk_rows * ld)) != UML_OK) return rc;
  // bytes of one row as it travels: `direct` rows keep their padding up to ld
  const int64_t wire_row_bytes = direct ? ld * 4 : row_bytes;
  if (bounce && (rc = grow_bounce(e, chunk_rows * wire_row_bytes)) != UML_OK) return rc;
  if ((rc = grow(e, e->d_ochunk, chunk_rows * out_bytes)) != UML_OK) return rc;
  if (exact && (rc = grow(e, e->d_flag_rows, chunk_rows)) != UML_OK) return rc;
  // A device-to-host copy into PAGEABLE memory blocks the calling thread until the chunk's whole pipeline has drained,
  // which would serialise gather / H2D / scoring.  Pageable outputs therefore land in pinned slots first and are
  // copied out by the host when the slot comes round again (three chunks later) or at the end.
  // (the asynchronous variant always does: the flush is also where a finished prefix is published to the poller)
  const bool result_bounce = progress != nullptr || !host_ptr_is_pinned(out);
  if (result_bounce && (rc = grow(e, e->h_result, chunk_rows * out_bytes)) != UML_OK) return rc;
  struct Pending {
    int64_t r0 = 0, rows = 0;
    bool live = false;
  } pending[3];
  auto flush_slot = [&](int sl) -> cudaError_t {
    if (!pending[sl].live) return cudaSuccess;
    cudaError_t fe = cudaEventSynchronize(e->chunk_ev[3 + sl]);  // recorded after the slot's D2H copies
    if (fe != cudaSuccess) return fe;
    memcpy(static_cast<char*>(out) + pending[sl].r0 * out_bytes, e->h_result.p[sl], (size_t)(pending[sl].rows * out_bytes));
    pending[sl].live = false;
    if (progress) progress->store(pending[sl].r0 + pending[sl].rows, std::memory_order_release);  // slots flush in row order
    return cudaSuccess;
  };

  // MLP: the tensor cores' tf32 question is answered by a host-side sample of the first rows (rows that are not tf32
  // values are caught in the kernel and re-scored, so a wrong guess costs time, never labels); taken once
  int sample_tf32 = -1;
  Chunk c{};
  c.ld = ld;
  c.tf32 = [&] {
    if (sample_tf32 < 0) sample_tf32 = host_sample_is_tf32(host_ptr, L, n_rows, F, src_dtype) ? 1 : 0;
    return sample_tf32 == 1;
  };

  const bool timed = stats != nullptr;
  cudaStream_t cs = e->stream;
  if (timed) UML_CUDA_DRAIN(e, cudaEventRecord(e->ev[0], cs));
  UML_CUDA_DRAIN(e, reset_counters(e, cs));
  UML_CUDA_DRAIN(e, cudaMemsetAsync(e->d_stage, 0, sizeof(StageResult), cs));
  if (step.prepare && (rc = step.prepare(chunk_rows)) != UML_OK) return rc;
  UML_CUDA_DRAIN(e, cudaEventRecord(e->chunk_ev[6], cs));
  UML_CUDA_DRAIN(e, cudaStreamWaitEvent(e->copy_stream, e->chunk_ev[6], 0));
  int launches = 0, path = 0;
  int64_t h2d = 0, d2h = 0;
  bool used[3] = {false, false, false};
  int slot = 0;
  std::vector<CopyPool::Task> tasks;
  bool wire_f32 = bounce && !direct && src_dtype == UML_F64 && (L.feature_major || L.pitch_elems == F) &&
                  !getenv("UML_B200_NO_NARROW");
  // UML_B200_PROFILE_HOST=1: host-side seconds per phase of this call on stderr (diagnostics, not a product feature)
  static const bool prof = getenv("UML_B200_PROFILE_HOST") != nullptr;
  double t_wait = 0, t_gather = 0, t_enqueue = 0;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto secs = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double>(b - a).count();
  };
  // ... and, for the first chunks, a device timeline from CUDA events on both streams (H2D / convert+score+D2H), which
  // is what shows the overlap of the pipeline without nsys
  constexpr int kTl = 12;
  cudaEvent_t tl[kTl][4] = {};
  int tl_n = 0;
  if (prof)
    for (auto& row : tl)
      for (auto& ev : row) cudaEventCreate(&ev);
  for (int64_t r0 = 0; r0 < n_rows; r0 += chunk_rows, slot = (slot + 1) % 3) {
    const int64_t rows = std::min(chunk_rows, n_rows - r0);
    float* xc = e->d_xchunk.p[slot];
    void* raw = direct ? (void*)xc : e->d_chunk.p[slot];
    const int tli = (prof && tl_n < kTl) ? tl_n++ : -1;
    bool chunk_narrow = false;  // this chunk crossed PCIe as fp32 (lossless float64 source)
    // (1) H2D on the copy stream, once the previous user of this slot has finished scoring (the re-score reads the
    //     raw chunk, so that includes it)
    if (used[slot]) UML_CUDA_DRAIN(e, cudaStreamWaitEvent(e->copy_stream, e->chunk_ev[3 + slot], 0));
    if (result_bounce) UML_CUDA_DRAIN(e, flush_slot(slot));
    if (tli >= 0) cudaEventRecord(tl[tli][0], e->copy_stream);
    {
      NvtxRange r_h2d("uml:h2d");
      if (bounce) {
        auto t0 = now();
        // the slot's previous H2D has left the bounce buffer
        if (used[slot]) UML_CUDA_DRAIN(e, cudaEventSynchronize(e->chunk_ev[slot]));
        auto t1 = now();
        t_wait += secs(t0, t1);
        if (direct) {  // already the resident layout (padding included): one contiguous run
          tasks.clear();
          const char* src0 = (const char*)host_ptr + (size_t)r0 * ld * 4;
          const size_t total = (size_t)rows * ld * 4, piece = 1u << 20;
          for (size_t o = 0; o < total; o += piece)
            tasks.push_back({e->h_bounce.p[slot] + o, src0 + o, std::min(piece, total - o)});
        }
        auto t2 = now();
        if (direct) {
          e->pool->run(tasks);
        } else {
          // float64 frames whose values are exactly representable in fp32 (integer / pixel domains) cross PCIe as fp32:
          // the gather threads convert while they copy and check every value; the first chunk that is not lossless
          // (and every chunk after it) travels as float64, as before
          chunk_narrow = wire_f32;
          if (chunk_narrow) {
            std::atomic<int> lossy{0};
            build_gather_tasks(tasks, e->h_bounce.p[slot], host_ptr, L, r0, rows, F, &lossy);
            e->pool->run(tasks);
            if (lossy.load()) {
              wire_f32 = false;
              chunk_narrow = false;
            }
          }
          if (!chunk_narrow) {
            build_gather_tasks(tasks, e->h_bounce.p[slot], host_ptr, L, r0, rows, F);
            e->pool->run(tasks);
          }
        }
        auto t3 = now();
        t_gather += secs(t2, t3);
        UML_CUDA_DRAIN(e, cudaMemcpyAsync(raw, e->h_bounce.p[slot],
                                          (size_t)(rows * (chunk_narrow ? wire_row_bytes / 2 : wire_row_bytes)),
                                          cudaMemcpyHostToDevice, e->copy_stream));
        t_enqueue += secs(t3, now());
      } else if (direct) {
        UML_CUDA_DRAIN(e, cudaMemcpyAsync(xc, (const char*)host_ptr + (size_t)r0 * ld * 4, (size_t)rows * ld * 4,
                                          cudaMemcpyHostToDevice, e->copy_stream));
      } else {
        UML_CUDA_DRAIN(e, copy_chunk_h2d(raw, host_ptr, L, r0, rows, F, e->copy_stream));
      }
    }
    h2d += rows * (chunk_narrow ? wire_row_bytes / 2 : wire_row_bytes);
    if (tli >= 0) cudaEventRecord(tl[tli][1], e->copy_stream);
    UML_CUDA_DRAIN(e, cudaEventRecord(e->chunk_ev[slot], e->copy_stream));
    UML_CUDA_DRAIN(e, cudaStreamWaitEvent(cs, e->chunk_ev[slot], 0));
    if (tli >= 0) cudaEventRecord(tl[tli][2], cs);
    // (2) transpose / down-cast (+ finiteness) on the compute stream; not for a step that reads the chunk as it arrived
    if (!direct && !step.raw) {
      NvtxRange r_stage("uml:stage_convert");
      UML_CUDA_DRAIN(e, uml::launch_stage_convert(raw, chunk_narrow ? (int)UML_F32 : src_dtype, L.feature_major,
                                                  L.feature_major ? rows : F, rows, F, xc, ld, nullptr, 0, e->d_stage,
                                                  true, cs));
      launches += 1;
    } else if (!exact && !step.raw) {
      UML_CUDA_DRAIN(e, uml::launch_finite_scan(xc, ld, rows, F, e->d_stage, cs));
      launches += 1;
    }
    // (3) score
    c.x = xc;
    c.rows = rows;
    c.src = direct ? uml::SrcView{xc, UML_F32, ld, 1}
                   : uml::SrcView{raw, chunk_narrow ? (int)UML_F32 : src_dtype, L.feature_major ? 1 : F,
                                  L.feature_major ? rows : 1};
    if ((rc = step.score(c, e->d_ochunk.p[slot], &launches, &path)) != UML_OK) {
      cudaStreamSynchronize(cs);
      cudaStreamSynchronize(e->copy_stream);
      return rc;
    }
    // (4) the output back
    const int64_t bytes = rows * out_bytes;
    UML_CUDA_DRAIN(e, cudaMemcpyAsync(result_bounce ? (void*)e->h_result.p[slot] : static_cast<char*>(out) + r0 * out_bytes,
                                      e->d_ochunk.p[slot], (size_t)bytes, cudaMemcpyDeviceToHost, cs));
    d2h += bytes;
    if (result_bounce) {
      pending[slot].r0 = r0;
      pending[slot].rows = rows;
      pending[slot].live = true;
    }
    if (tli >= 0) cudaEventRecord(tl[tli][3], cs);
    UML_CUDA_DRAIN(e, cudaEventRecord(e->chunk_ev[3 + slot], cs));
    used[slot] = true;
  }
  UML_CUDA_DRAIN(e, cudaMemcpyAsync(&e->h->stage, e->d_stage, sizeof(StageResult), cudaMemcpyDeviceToHost, cs));
  if (prof && tl_n > 0) {
    cudaStreamSynchronize(cs);
    cudaStreamSynchronize(e->copy_stream);
    fprintf(stderr, "uml predict_host timeline (ms since the first H2D began; chunk: h2d [begin,end]  convert+score+d2h [begin,end])\n");
    for (int i = 0; i < tl_n; ++i) {
      float a = 0, b2 = 0, c = 0, d = 0;
      cudaEventElapsedTime(&a, tl[0][0], tl[i][0]);
      cudaEventElapsedTime(&b2, tl[0][0], tl[i][1]);
      cudaEventElapsedTime(&c, tl[0][0], tl[i][2]);
      cudaEventElapsedTime(&d, tl[0][0], tl[i][3]);
      fprintf(stderr, "  chunk %2d: h2d [%7.3f, %7.3f]  compute [%7.3f, %7.3f]\n", i, a, b2, c, d);
    }
    (void)cudaGetLastError();
  }
  if (prof)
    for (auto& row : tl)
      for (auto& ev : row)
        if (ev) cudaEventDestroy(ev);
  if (prof)
    fprintf(stderr, "uml predict_host: rows %lld chunk_rows %lld bounce %d direct %d | wait-for-slot %.4f s, gather %.4f s, "
                    "memcpyAsync enqueue %.4f s\n", (long long)n_rows, (long long)chunk_rows, (int)bounce, (int)direct, t_wait,
            t_gather, t_enqueue);
  rc = finish_stats(e, stats, n_rows, launches, path, timed, false);
  cudaStreamSynchronize(e->copy_stream);
  for (int sl = 0; sl < 3; ++sl)
    if (flush_slot(sl) != cudaSuccess && rc == UML_OK) rc = UML_ERR_CUDA;
  if (stats) {
    stats->h2d_bytes = h2d;
    stats->d2h_bytes = d2h;
  }
  // NaN/Inf in the caller's values (the staging kernel checks the source dtype, so a finite float64 that overflows
  // fp32 is not an error here - exact mode re-scores such rows from the float64 source)
  if (rc == UML_OK && e->h->stage.nonfinite) UML_FAIL(e, UML_ERR_NONFINITE, "Input X contains NaN or infinity.");
  return rc;
}

// The chunk pipeline's steps.  They capture by value: an asynchronous call runs its step on the library thread after
// the entry point has returned.
static ChunkStep linear_labels_step(uml_engine* e, const uml_model* m, int mode) {
  ChunkStep s{m->n_features_in, "estimator", 4, false};
  s.score = [=](const Chunk& c, void* out, int* launches, int* path) {
    LinearLaunch l{};
    l.x = c.x;
    l.ld = c.ld;
    l.n_rows = c.rows;
    l.targets.labels = static_cast<int32_t*>(out);
    // (the reference MLP predictor casts to float32; a chunk that travelled as fp32 was checked lossless on the host: its
    // fp32 rows ARE the caller's values) flagged rows are re-scored from the caller's own values (the raw chunk is still
    // resident): float64 / int features that do not survive the fp32 down-cast still get sklearn's float64 labels
    // (_base.py:366-396)
    if (mode == UML_PREDICT_EXACT && lossy_capable(c.src.dtype)) l.src = c.src;
    CUtensorMap map;
    const bool has_map = encode_map(e, &map, c.x, c.rows, m->n_features_in, c.ld, linear_box_rows_for(m->n_features_in)) == UML_OK;
    return enqueue_predict(e, m, l, has_map ? &map : nullptr, nullptr, mode, false, launches, path);
  };
  s.small = [=](const uml::SrcView& v, int rows, cudaStream_t st) {
    return uml::launch_linear_small(m->dm, v, rows, e->d_small, st);
  };
  s.small_uid = m->uid;
  return s;
}

// the labels, then classes[label] as float64 on the device
static ChunkStep linear_values_step(uml_engine* e, const uml_model* m, int mode, const double* classes, int n_classes) {
  ChunkStep s = linear_labels_step(e, m, mode);
  s.row_bytes = 8;
  s.classes = classes;
  s.n_classes = n_classes;
  s.prepare = [=](int64_t chunk_rows) -> int {
    int rc;
    if ((rc = grow(e, e->d_labels, chunk_rows)) != UML_OK || (rc = grow(e, e->d_classes, n_classes)) != UML_OK) return rc;
    UML_CUDA(e, cudaMemcpyAsync(e->d_classes.p[0], classes, (size_t)n_classes * 8, cudaMemcpyHostToDevice, e->stream));
    return UML_OK;
  };
  s.score = [=, labels = s.score](const Chunk& c, void* out, int* launches, int* path) -> int {
    const int rc = labels(c, e->d_labels.p[0], launches, path);
    if (rc != UML_OK) return rc;
    UML_CUDA(e, uml::launch_labels_take(e->d_labels.p[0], 4, c.rows, e->d_classes.p[0], n_classes,
                                        static_cast<double*>(out), e->stream));
    *launches += 1;
    return UML_OK;
  };
  return s;
}

// float64 scores, probabilities or log-probabilities (kind) from the chunk as it crossed PCIe
static ChunkStep linear_f64_step(uml_engine* e, const uml_model* m, int kind) {
  ChunkStep s{m->n_features_in, "estimator", 8ll * uml::linear_f64_width(m->dm, kind), true};
  s.score = [=](const Chunk& c, void* out, int* launches, int* path) -> int {
    NvtxRange r_score("uml:scores_f64");
    UML_CUDA(e, uml::launch_linear_scores_f64(m->dm, c.src, c.rows, static_cast<double*>(out),
                                              e->d_counters + uml::kCounterNonfinite, e->info.sm_count, e->stream, kind));
    *launches += 1;
    *path = f64_path(kind);
    return UML_OK;
  };
  return s;
}

// an MLP whose weights and strips do not fit one SM's shared memory has no small-batch kernel
static ChunkStep mlp_labels_step(uml_engine* e, const uml_mlp* m, int mode) {
  ChunkStep s{m->dm.n_in, "module", 4, false};
  s.score = [=](const Chunk& c, void* out, int* launches, int* path) {
    CUtensorMap map;
    const bool has_map = encode_map(e, &map, c.x, c.rows, m->dm.n_in, c.ld) == UML_OK;
    uml::MlpTcLaunch o{};
    o.n_rows = c.rows;
    o.targets.labels = static_cast<int32_t*>(out);
    return enqueue_mlp(e, m->dm, map, c.x, c.ld, o, mode == UML_PREDICT_EXACT, mlp_route(m->dm, has_map, false, c.tf32),
                       false, launches, path);
  };
  if (m->small_smem > 0) {
    s.small = [=](const uml::SrcView& v, int rows, cudaStream_t st) {
      return uml::launch_mlp_small(m->dm, v, rows, e->d_small, m->small_smem, st);
    };
    s.small_uid = m->uid;
  }
  return s;
}

// The probability and top-k steps have no re-score that would find a finite float64 beyond the fp32 range (the staging
// kernel checks the caller's values, and the fp32 cast of such a value is inf): a chunk that crossed PCIe as float64
// has its fp32 rows scanned for NaN / Inf, as the reference's cast makes them.
static int mlp_scan_f64_chunk(uml_engine* e, const uml_mlp* m, const Chunk& c, int* launches) {
  if (c.src.dtype != UML_F64) return UML_OK;
  UML_CUDA(e, uml::launch_finite_scan(c.x, c.ld, c.rows, m->dm.n_in, e->d_stage, e->stream));
  *launches += 1;
  return UML_OK;
}

// the <= kSmallRows form of a probability / top-k step: mlp_small_kernel's record form into the model's mapped buffer
static void mlp_small_records(uml_engine* e, const uml_mlp* m, ChunkStep& s, int kind, int k) {
  if (m->small_rec_smem == 0 || !m->h_rec) return;
  s.small = [=](const uml::SrcView& v, int rows, cudaStream_t st) {
    return uml::launch_mlp_small(m->dm, v, rows, e->d_small, m->small_rec_smem, st, kind, k, m->d_rec);
  };
  s.small_uid = m->uid;
  s.small_rec = m->h_rec;
  s.small_kind = kind;
  s.small_k = k;
}

// class probabilities: the kernel mlp_route picks from the chunk's tf32 guess.  Behind the tensor cores, the float64
// probabilities of the rows they flagged (not tf32 values) overwrite theirs.
static ChunkStep mlp_proba_step(uml_engine* e, const uml_mlp* m) {
  ChunkStep s{m->dm.n_in, "module", 4ll * m->dm.n_classes, false};
  s.prepare = [=](int64_t chunk_rows) { return grow(e, e->d_flag_rows, chunk_rows); };
  s.score = [=](const Chunk& c, void* out, int* launches, int* path) -> int {
    int rc;
    if ((rc = mlp_scan_f64_chunk(e, m, c, launches)) != UML_OK) return rc;
    CUtensorMap map;
    const bool has_map = encode_map(e, &map, c.x, c.rows, m->dm.n_in, c.ld) == UML_OK;
    const int route = mlp_route(m->dm, has_map, true, c.tf32);
    float* proba = static_cast<float*>(out);
    const int sm = e->info.sm_count;
    if (route == 5) {
      uml::MlpTcLaunch o{};
      o.n_rows = c.rows;
      o.proba = proba;
      UML_CUDA(e, uml::launch_mlp_tc_proba(map, m->dm, o, flag_list(e), sm, e->stream));
      UML_CUDA(e, uml::launch_mlp_proba_f64(m->dm, c.x, c.ld, c.rows, proba, flag_list(e), false, sm, e->stream));
      *launches += 2;
    } else if (route == 3) {
      UML_CUDA(e, uml::launch_mlp_tma(map, m->dm, c.x, c.rows, nullptr, false, {}, sm, e->stream, proba));
      *launches += 1;
    } else {
      UML_CUDA(e, uml::launch_mlp_proba_f64(m->dm, c.x, c.ld, c.rows, proba, {}, true, sm, e->stream));
      *launches += 1;
    }
    *path = route;
    return UML_OK;
  };
  mlp_small_records(e, m, s, uml::kSmallProba, 0);
  return s;
}

// top-k: routed as uml_mlp_predict_topk, with the chunk's tf32 guess.  Behind a tensor-core or EXACT launch, the float64
// top-k of the flagged rows.  The kernels write [rows][k] index and probability planes to scratch; two strided copies
// lay them into the pipeline's one output, a record of k int32 indices then k fp32 probabilities per row.
static ChunkStep mlp_topk_step(uml_engine* e, const uml_mlp* m, int k, int mode) {
  ChunkStep s{m->dm.n_in, "module", 8ll * k, false};
  s.prepare = [=](int64_t chunk_rows) {
    int rc;
    if ((rc = grow(e, e->d_flag_rows, chunk_rows)) != UML_OK) return rc;
    return grow(e, e->d_labels, 2 * k * chunk_rows);
  };
  s.score = [=](const Chunk& c, void* out, int* launches, int* path) -> int {
    int rc;
    if ((rc = mlp_scan_f64_chunk(e, m, c, launches)) != UML_OK) return rc;
    const bool exact = mode == UML_PREDICT_EXACT;
    CUtensorMap map;
    int route = 2;
    if (k <= uml::kMlpTopkMax) {
      const bool has_map = encode_map(e, &map, c.x, c.rows, m->dm.n_in, c.ld) == UML_OK;
      route = mlp_route(m->dm, has_map, false, c.tf32, true);
    }
    int32_t* idx = e->d_labels.p[0];
    float* proba = reinterpret_cast<float*>(idx + k * c.rows);
    const FlagList fl = flag_list(e);
    const int sm = e->info.sm_count;
    cudaStream_t st = e->stream;
    if (route == 2) {
      UML_CUDA(e, uml::launch_mlp_topk_f64(m->dm, c.x, c.ld, c.rows, k, idx, proba, fl, true, sm, st));
      *launches += 1;
    } else {
      if (route == 5) {
        uml::MlpTcLaunch o{};
        o.n_rows = c.rows;
        o.topk_idx = idx;
        o.topk_proba = proba;
        o.topk_k = k;
        UML_CUDA(e, uml::launch_mlp_tc_topk(map, m->dm, o, exact, fl, sm, st));
      } else {
        UML_CUDA(e, uml::launch_mlp_tma_topk(map, m->dm, c.rows, k, idx, proba, exact, fl, sm, st));
      }
      *launches += 1;
      if (exact || route == 5) {
        UML_CUDA(e, uml::launch_mlp_topk_f64(m->dm, c.x, c.ld, c.rows, k, idx, proba, fl, false, sm, st));
        *launches += 1;
      }
    }
    const size_t plane = 4ull * k;
    UML_CUDA(e, cudaMemcpy2DAsync(out, 2 * plane, idx, plane, plane, (size_t)c.rows, cudaMemcpyDeviceToDevice, st));
    UML_CUDA(e, cudaMemcpy2DAsync(static_cast<char*>(out) + plane, 2 * plane, proba, plane, plane, (size_t)c.rows,
                                  cudaMemcpyDeviceToDevice, st));
    *path = route;
    return UML_OK;
  };
  mlp_small_records(e, m, s, uml::kSmallTopk, k);
  return s;
}

int uml_linear_predict_host(uml_engine* e, const uml_model* m, const void* host_ptr, int64_t n_rows, int n_features,
                            int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, int32_t* labels_out,
                            int mode, int64_t chunk_rows, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  return predict_host_impl(e, linear_labels_step(e, m, mode), host_ptr, n_rows, n_features, row_stride_bytes,
                           col_stride_bytes, src_dtype, labels_out, mode, chunk_rows, stats);
}

int uml_linear_predict_host_values(uml_engine* e, const uml_model* m, const void* host_ptr, int64_t n_rows,
                                   int n_features, int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype,
                                   const double* classes_host, int n_classes, double* values_out, int mode,
                                   int64_t chunk_rows, uml_stats* stats) {
  if (!m || (!values_out && n_rows > 0) || !classes_host || n_classes < 1) return UML_ERR_INVALID;
  if (n_classes < m->dm.n_classes) UML_FAIL(e, UML_ERR_INVALID, "classes_ has %d entries, the model scores %d classes", n_classes, m->dm.n_classes);
  return predict_host_impl(e, linear_values_step(e, m, mode, classes_host, n_classes), host_ptr, n_rows, n_features,
                           row_stride_bytes, col_stride_bytes, src_dtype, values_out, mode, chunk_rows, stats);
}

// asynchronous variant: the whole pipeline runs on a library thread so that the caller (Python building the
// List[float] of the predictor contract) can consume labels_out[0, rows_done) while the rest of the batch is still
// crossing PCIe.  One call in flight per engine; no other call on the engine until _finish.
static int async_begin(uml_engine* e, const ChunkStep& step, const void* host_ptr, int64_t n_rows, int n_features,
                       int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, int32_t* labels_out, int mode,
                       int64_t chunk_rows) {
  if (!e || (!labels_out && n_rows > 0)) return UML_ERR_INVALID;
  if (!e->async_finished.load() || e->async_thread.joinable())
    UML_FAIL(e, UML_ERR_INVALID, "an asynchronous call is already in flight on this engine (call uml_async_finish first)");
  e->async_rows_done.store(0);
  e->async_finished.store(0);
  e->async_status = UML_OK;
  memset(&e->async_stats, 0, sizeof(e->async_stats));
  e->async_thread = std::thread([=]() {
    e->async_status = predict_host_impl(e, step, host_ptr, n_rows, n_features, row_stride_bytes, col_stride_bytes,
                                        src_dtype, labels_out, mode, chunk_rows, &e->async_stats, &e->async_rows_done);
    e->async_finished.store(1, std::memory_order_release);
  });
  return UML_OK;
}

int uml_linear_predict_host_begin(uml_engine* e, const uml_model* m, const void* host_ptr, int64_t n_rows, int n_features,
                                  int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, int32_t* labels_out,
                                  int mode, int64_t chunk_rows) {
  if (!m) return UML_ERR_INVALID;
  return async_begin(e, linear_labels_step(e, m, mode), host_ptr, n_rows, n_features, row_stride_bytes,
                     col_stride_bytes, src_dtype, labels_out, mode, chunk_rows);
}

// the MLP predictor through the same chunk pipeline, or for B <= kSmallRows the same online route (mlp_small_kernel):
// labels_out[i] = argmax class index of row i, i.e. what `module(features).argmax(1)` yields
// (tests/integration/pytorch_app/quickstart.py:68-70)
int uml_mlp_predict_host(uml_engine* e, const uml_mlp* m, const void* host_ptr, int64_t n_rows, int n_features,
                         int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, int32_t* labels_out, int mode,
                         int64_t chunk_rows, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  return predict_host_impl(e, mlp_labels_step(e, m, mode), host_ptr, n_rows, n_features, row_stride_bytes,
                           col_stride_bytes, src_dtype, labels_out, mode, chunk_rows, stats);
}

int uml_mlp_predict_host_begin(uml_engine* e, const uml_mlp* m, const void* host_ptr, int64_t n_rows, int n_features,
                               int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, int32_t* labels_out,
                               int mode, int64_t chunk_rows) {
  if (!m) return UML_ERR_INVALID;
  return async_begin(e, mlp_labels_step(e, m, mode), host_ptr, n_rows, n_features, row_stride_bytes, col_stride_bytes,
                     src_dtype, labels_out, mode, chunk_rows);
}

// the online route's record buffer of a model (uml_mlp::h_rec), made at its first request that can take the route
static int mlp_reserve_records(uml_engine* e, const uml_mlp* m, int64_t n_rows) {
  if (n_rows > kSmallRows || m->small_rec_smem == 0 || m->h_rec) return UML_OK;
  uml_mlp* mm = const_cast<uml_mlp*>(m);  // the handle is logically const for the caller
  UML_CUDA(e, cudaSetDevice(e->device));
  UML_CUDA(e, cudaHostAlloc(&mm->h_rec, (size_t)kSmallRows * m->dm.n_classes * 8, cudaHostAllocMapped));
  UML_CUDA(e, cudaHostGetDevicePointer(&mm->d_rec, mm->h_rec, 0));
  return UML_OK;
}

int uml_mlp_predict_proba_host(uml_engine* e, const uml_mlp* m, const void* host_ptr, int64_t n_rows, int n_features,
                               int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, float* proba_out,
                               int64_t chunk_rows, uml_stats* stats) {
  if (!e || !m) return UML_ERR_INVALID;
  int rc;
  if ((rc = mlp_reserve_records(e, m, n_rows)) != UML_OK) return rc;
  return predict_host_impl(e, mlp_proba_step(e, m), host_ptr, n_rows, n_features, row_stride_bytes, col_stride_bytes,
                           src_dtype, proba_out, UML_PREDICT_FAST, chunk_rows, stats);
}

int uml_mlp_predict_topk_host(uml_engine* e, const uml_mlp* m, const void* host_ptr, int64_t n_rows, int n_features,
                              int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype, int k, int32_t* out,
                              int mode, int64_t chunk_rows, uml_stats* stats) {
  if (!e || !m) return UML_ERR_INVALID;
  const int C = m->dm.n_classes;
  if (k < 1 || k > C) UML_FAIL(e, UML_ERR_INVALID, "k = %d: the module has %d classes (need 1 <= k <= %d)", k, C, C);
  int rc;
  if ((rc = mlp_reserve_records(e, m, n_rows)) != UML_OK) return rc;
  return predict_host_impl(e, mlp_topk_step(e, m, k, mode), host_ptr, n_rows, n_features, row_stride_bytes,
                           col_stride_bytes, src_dtype, out, mode, chunk_rows, stats);
}

int uml_async_poll(uml_engine* e, int64_t* rows_done, int* finished) {
  if (!e) return UML_ERR_INVALID;
  const int fin = e->async_finished.load(std::memory_order_acquire);  // read first: rows_done is final once it is set
  if (rows_done) *rows_done = e->async_rows_done.load(std::memory_order_acquire);
  if (finished) *finished = fin;
  return UML_OK;
}

int uml_async_finish(uml_engine* e, uml_stats* stats) {
  if (!e) return UML_ERR_INVALID;
  if (e->async_thread.joinable()) e->async_thread.join();
  if (stats) *stats = e->async_stats;
  return e->async_status;
}

int uml_linear_predict_proba(uml_engine* e, const uml_model* m, const uml_batch* b, float* proba_out, int proba_on_device) {
  if (!m) return UML_ERR_INVALID;
  NvtxRange r_all("uml:predict_proba");
  auto score = [&](void* const* out, bool, int* launches, int*, int*) -> int {
    UML_CUDA(e, uml::launch_linear_proba(m->dm, b->x, b->ld, b->n_rows, static_cast<float*>(out[0]), e->info.sm_count,
                                         e->stream));
    *launches = 1;
    return UML_OK;
  };
  return predict_resident(e, b, {m->dm.n_classes, m->n_features_in, "estimator", {proba_out, nullptr},
                                 {4ll * m->dm.n_classes, 0}, proba_on_device, UML_PREDICT_FAST, nullptr},
                          no_prepare, score);
}

// float64 decision_function scores of a resident batch (sklearn/linear_model/_base.py:366-396), or their probabilities /
// log-probabilities (kind), from the caller's own values: the batch's float64 copy when it has one, else its fp32 rows,
// which are then the caller's values (lossless staging, or rows wrapped in place).  Synchronous: the output is written,
// and NaN / Inf reported, when it returns.
static int linear_f64_resident(uml_engine* e, const uml_model* m, const uml_batch* b, double* out, int on_device,
                               int kind, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  auto prepare = [&]() -> int {
    if (!b->x64 && !b->lossless)
      UML_FAIL(e, UML_ERR_UNSUPPORTED, "the batch's fp32 rows are a lossy cast of the caller's values and it kept no "
                                       "float64 copy: stage it with UML_STAGE_KEEP_F64 for its float64 %s",
               kind == uml::kF64Scores ? "scores" : "probabilities");
    return UML_OK;
  };
  auto score = [&](void* const* o, bool timed, int* launches, int* path, int*) -> int {
    const uml::SrcView src = b->x64 ? uml::SrcView{b->x64, UML_F64, b->ld64, 1} : uml::SrcView{b->x, UML_F32, b->ld, 1};
    UML_CUDA(e, uml::launch_linear_scores_f64(m->dm, src, b->n_rows, static_cast<double*>(o[0]),
                                              e->d_counters + uml::kCounterNonfinite, e->info.sm_count, e->stream, kind));
    if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], e->stream));
    *launches = 1;
    *path = f64_path(kind);
    return UML_OK;
  };
  ResidentCall c{m->dm.n_classes, m->n_features_in, "estimator", {out, nullptr},
                 {8ll * uml::linear_f64_width(m->dm, kind), 0}, on_device, UML_PREDICT_FAST, stats};
  c.always_sync = true;
  return predict_resident(e, b, c, prepare, score);
}

int uml_linear_decision_function(uml_engine* e, const uml_model* m, const uml_batch* b, double* scores_out,
                                 int scores_on_device, uml_stats* stats) {
  NvtxRange r_all("uml:decision_function");
  return linear_f64_resident(e, m, b, scores_out, scores_on_device, uml::kF64Scores, stats);
}

// the same scores from HOST rows through the chunk pipeline of uml_linear_predict_host (any layout and dtype it takes)
int uml_linear_decision_function_host(uml_engine* e, const uml_model* m, const void* host_ptr, int64_t n_rows,
                                      int n_features, int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype,
                                      double* scores_out, int64_t chunk_rows, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  NvtxRange r_all("uml:decision_function");
  return predict_host_impl(e, linear_f64_step(e, m, uml::kF64Scores), host_ptr, n_rows, n_features, row_stride_bytes,
                           col_stride_bytes, src_dtype, scores_out, UML_PREDICT_FAST, chunk_rows, stats);
}

// float64 probabilities (LogisticRegression.predict_proba) or their logs (predict_log_proba) of a resident batch, from
// the caller's own values as uml_linear_decision_function reads them
int uml_linear_predict_proba_f64(uml_engine* e, const uml_model* m, const uml_batch* b, double* proba_out,
                                 int proba_on_device, int log_proba, uml_stats* stats) {
  NvtxRange r_all("uml:predict_proba_f64");
  return linear_f64_resident(e, m, b, proba_out, proba_on_device, log_proba ? uml::kF64LogProba : uml::kF64Proba, stats);
}

// the same from HOST rows through the chunk pipeline of uml_linear_predict_host (any layout and dtype it takes)
int uml_linear_predict_proba_f64_host(uml_engine* e, const uml_model* m, const void* host_ptr, int64_t n_rows,
                                      int n_features, int64_t row_stride_bytes, int64_t col_stride_bytes, int src_dtype,
                                      double* proba_out, int log_proba, int64_t chunk_rows, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  NvtxRange r_all("uml:predict_proba_f64");
  return predict_host_impl(e, linear_f64_step(e, m, log_proba ? uml::kF64LogProba : uml::kF64Proba), host_ptr, n_rows,
                           n_features, row_stride_bytes, col_stride_bytes, src_dtype, proba_out, UML_PREDICT_FAST,
                           chunk_rows, stats);
}

// ---------------------------------------------------------------------------------------------------------------
// MLP: PytorchModel(in, hidden, out) of tests/integration/pytorch_app/quickstart.py
// ---------------------------------------------------------------------------------------------------------------
int uml_mlp_load(uml_engine* e, uml_mlp** out, const float* w1, const float* b1, const float* w2, const float* b2,
                 int n_in, int n_hidden, int n_out) {
  if (!e || !out || !w1 || !b1 || !w2 || !b2) return UML_ERR_INVALID;
  *out = nullptr;
  if (n_in < 1 || n_hidden < 1 || n_out < 2 || n_hidden > 256)
    UML_FAIL(e, UML_ERR_UNSUPPORTED, "MLP shape %d -> %d -> %d (need hidden <= 256, out >= 2)", n_in, n_hidden, n_out);
  {  // the fp64 re-score kernel keeps W1, W2 and eight row strips in shared memory
    const size_t need = ((size_t)n_in * n_hidden + (size_t)n_out * (n_hidden + 1) + 2 * (size_t)n_hidden + n_out + n_in +
                         8 * ((size_t)n_in + n_hidden)) * 8;
    if (need > (size_t)uml::kMaxSmemBytes)
      UML_FAIL(e, UML_ERR_UNSUPPORTED, "MLP shape %d -> %d -> %d: fp64 weights (%zu B) exceed the shared memory of one SM", n_in,
               n_hidden, n_out, need);
  }
  UML_CUDA(e, cudaSetDevice(e->device));
  const int F = n_in, H = n_hidden, C = n_out;
  const int HP = H + 4, cp = (C + 1 + 3) / 4 * 4;
  const int f_pad = (F + uml::kChunkF - 1) / uml::kChunkF * uml::kChunkF;
  std::vector<float> w1t((size_t)f_pad * HP, 0.f), b1p(HP, 0.f), w2t((size_t)H * cp, 0.f), b2p(cp, 0.f);
  for (int f = 0; f < F; ++f) {
    float wmax = 0.f;
    for (int n = 0; n < H; ++n) {
      const float v = w1[(size_t)n * F + f];  // torch Linear weight: (out, in)
      w1t[(size_t)f * HP + n] = v;
      wmax = fmaxf(wmax, fabsf(v));
    }
    w1t[(size_t)f * HP + H] = wmax;
  }
  float bmax = 0.f;
  for (int n = 0; n < H; ++n) {
    b1p[n] = b1[n];
    bmax = fmaxf(bmax, fabsf(b1[n]));
  }
  b1p[H] = bmax;
  double row_sum_max = 0.0;
  for (int c = 0; c < C; ++c) {
    double rs = 0.0;
    for (int n = 0; n < H; ++n) rs += fabs((double)w2[(size_t)c * H + n]);
    row_sum_max = std::max(row_sum_max, rs);
  }
  for (int n = 0; n < H; ++n) {
    float wmax = 0.f;
    for (int c = 0; c < C; ++c) {
      const float v = w2[(size_t)c * H + n];
      w2t[(size_t)n * cp + c] = v;
      wmax = fmaxf(wmax, fabsf(v));
    }
    w2t[(size_t)n * cp + C] = wmax;
  }
  bmax = 0.f;
  for (int c = 0; c < C; ++c) {
    b2p[c] = b2[c];
    bmax = fmaxf(bmax, fabsf(b2[c]));
  }
  // CUDA-core kernel (DESIGN.md 3.4): the weights and features are the caller's fp32 values, so a hidden unit's only
  // absolute error is its F FMAs' roundings into the subnormals, plus one for the fp32 A1 chain it is bounded with
  b2p[C] = uml::mlp_a2_bias_entry(bmax, (F + 2.0) * uml::kHalfSubnormal, row_sum_max, H);
  // fp64 operands of the re-score, laid out as the kernels keep them in shared memory
  const std::vector<double> w64 = uml::mlp_rs_build_pack(w1, b1, w2, b2, F, H, C);

  uml_mlp* m = new uml_mlp();
  m->e = e;
  m->host.w1.assign(w1, w1 + (size_t)H * F);
  m->host.b1.assign(b1, b1 + H);
  m->host.w2.assign(w2, w2 + (size_t)C * H);
  m->host.b2.assign(b2, b2 + C);
  std::vector<float> tiles;
  if (f_pad <= 128 && (H == 16 || H == 32)) tiles = uml::mlp_tc_build_w1_tiles(w1, H, F, f_pad);
  auto up = [&](void** dst, const void* src, size_t bytes) -> cudaError_t {
    cudaError_t ce = cudaMalloc(dst, bytes);
    if (ce != cudaSuccess) return ce;
    return cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
  };
  cudaError_t ce;
  if ((ce = up((void**)&m->d_w1t, w1t.data(), w1t.size() * 4)) != cudaSuccess ||
      (ce = up((void**)&m->d_b1, b1p.data(), b1p.size() * 4)) != cudaSuccess ||
      (ce = up((void**)&m->d_w2t, w2t.data(), w2t.size() * 4)) != cudaSuccess ||
      (ce = up((void**)&m->d_b2, b2p.data(), b2p.size() * 4)) != cudaSuccess ||
      (ce = up((void**)&m->d_w64, w64.data(), w64.size() * 8)) != cudaSuccess ||
      (!tiles.empty() && (ce = up((void**)&m->d_w1_tiles, tiles.data(), tiles.size() * 4)) != cudaSuccess)) {
    e->last_error = std::string("uml_mlp_load: ") + cudaGetErrorString(ce);
    uml_mlp_free(m);
    return ce == cudaErrorMemoryAllocation ? UML_ERR_NOMEM : UML_ERR_CUDA;
  }
  m->dm.w1t = m->d_w1t;
  m->dm.b1 = m->d_b1;
  m->dm.w2t = m->d_w2t;
  m->dm.b2 = m->d_b2;
  m->dm.rs_pack = m->d_w64;
  m->dm.n_in = F;
  m->dm.n_hidden = H;
  m->dm.n_classes = C;
  m->dm.cp = cp;
  m->dm.f_pad = f_pad;
  m->dm.w2_abs_row_sum_max = row_sum_max;
  m->dm.w1_tiles = m->d_w1_tiles;
  m->dm.host = &m->host;
  m->uid = g_model_uid.fetch_add(1);
  // the online kernel's shared-memory limit is set here, not where its launch is captured into a graph
  m->small_smem = uml::mlp_small_smem_bytes(F, H, C);
  m->small_rec_smem = uml::mlp_small_smem_bytes(F, H, C, true);
  if ((m->small_smem > 0 && (ce = uml::mlp_small_reserve(m->small_smem)) != cudaSuccess) ||
      (m->small_rec_smem > 0 && (ce = uml::mlp_small_reserve(m->small_rec_smem, true)) != cudaSuccess)) {
    e->last_error = std::string("uml_mlp_load: ") + cudaGetErrorString(ce);
    uml_mlp_free(m);
    return UML_ERR_CUDA;
  }
  *out = m;
  return UML_OK;
}

void uml_mlp_free(uml_mlp* m) {
  if (!m) return;
  if (m->e) cudaSetDevice(m->e->device);
  cudaFree(m->d_w1t);
  cudaFree(m->d_b1);
  cudaFree(m->d_w2t);
  cudaFree(m->d_b2);
  cudaFree(m->d_w64);
  cudaFree(m->d_w1_tiles);
  if (m->h_rec) cudaFreeHost(m->h_rec);  // no graph replays it: the graphs are keyed by this model's uid
  delete m;
}

// is every fp32 feature of the batch a tf32 value?  Known from staging; wrapped device rows are scanned once (one
// HBM pass, cached in the batch handle - the handle is logically const for the caller)
static int batch_tf32_exact(uml_engine* e, const uml_batch* b) {
  if (b->tf32_exact >= 0) return b->tf32_exact;
  cudaError_t ce;
  if ((ce = cudaMemsetAsync(e->d_stage, 0, sizeof(StageResult), e->stream)) != cudaSuccess ||
      (ce = uml::launch_finite_scan(b->x, b->ld, b->n_rows, b->n_features, e->d_stage, e->stream)) != cudaSuccess ||
      (ce = cudaMemcpyAsync(&e->h->stage, e->d_stage, sizeof(StageResult), cudaMemcpyDeviceToHost, e->stream)) != cudaSuccess ||
      (ce = cudaStreamSynchronize(e->stream)) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  const_cast<uml_batch*>(b)->tf32_exact = e->h->stage.not_tf32 == 0 ? 1 : 0;
  return b->tf32_exact;
}

static int mlp_predict_resident(uml_engine* e, const uml_mlp* m, const uml_batch* b, int32_t* labels_out,
                                int labels_on_device, void* const* peers, int n_peers, int64_t row_offset,
                                int label_bytes, int mode, uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  int route = 2;
  auto prepare = [&] {
    route = mlp_route(m->dm, b->has_map, false, [&] { return batch_tf32_exact(e, b) == 1; });
    // scratch for the CUDA-core kernel's labels on their way to the peers (enqueue_mlp)
    return route == 3 && n_peers > 0 ? grow(e, e->d_labels, b->n_rows) : (int)UML_OK;
  };
  auto score = [&](void* const* out, bool timed, int* launches, int* path, int* elem_bytes) {
    uml::MlpTcLaunch o{};
    o.n_rows = b->n_rows;
    uml::LabelTargets& t = o.targets;
    t.labels = static_cast<int32_t*>(out[0]);
    t.row_offset = row_offset;
    t.wire_u8 = n_peers > 0 && label_bytes == 1 ? 1 : 0;
    t.n_peers = n_peers;  // every peer vector, this rank's own included
    for (int i = 0; i < n_peers; ++i) t.peers[i] = peers[i];
    *elem_bytes = 4;  // the MLP kernels read fp32 rows
    return enqueue_mlp(e, m->dm, b->map, b->x, b->ld, o, mode == UML_PREDICT_EXACT, route, timed, launches, path);
  };
  ResidentCall c{m->dm.n_classes, m->dm.n_in, "module", {labels_out, nullptr}, {4, 0}, labels_on_device, mode, stats};
  c.n_peers = n_peers;
  c.label_bytes = label_bytes;
  return predict_resident(e, b, c, prepare, score);
}

int uml_mlp_predict(uml_engine* e, const uml_mlp* m, const uml_batch* b, int32_t* labels_out, int labels_on_device,
                    int mode, uml_stats* stats) {
  return mlp_predict_resident(e, m, b, labels_out, labels_on_device, nullptr, 0, 0, 4, mode, stats);
}

int uml_mlp_predict_peers(uml_engine* e, const uml_mlp* m, const uml_batch* b, void* const* peer_labels, int n_peers,
                          int64_t row_offset, int label_bytes, int mode, uml_stats* stats) {
  if (!peer_labels || n_peers < 1) return UML_ERR_INVALID;
  return mlp_predict_resident(e, m, b, nullptr, 1, peer_labels, n_peers, row_offset, label_bytes, mode, stats);
}

int uml_mlp_predict_proba(uml_engine* e, const uml_mlp* m, const uml_batch* b, float* proba_out, int proba_on_device,
                          uml_stats* stats) {
  if (!m) return UML_ERR_INVALID;
  NvtxRange r_all("uml:mlp_proba");
  int route = 2;
  auto prepare = [&] {
    route = mlp_route(m->dm, b->has_map, true, [&] { return batch_tf32_exact(e, b) == 1; });
    return (int)UML_OK;
  };
  auto score = [&](void* const* out, bool timed, int* launches, int* path, int*) -> int {
    float* proba = static_cast<float*>(out[0]);
    if (route == 5) {
      uml::MlpTcLaunch o{};
      o.n_rows = b->n_rows;
      o.proba = proba;
      // (every row is a tf32 value, or mlp_route would not have picked the tensor cores: no flag list)
      UML_CUDA(e, uml::launch_mlp_tc_proba(b->map, m->dm, o, {}, e->info.sm_count, e->stream));
    } else if (route == 3) {  // (no labels, so no flag list)
      UML_CUDA(e, uml::launch_mlp_tma(b->map, m->dm, b->x, b->n_rows, nullptr, false, {}, e->info.sm_count, e->stream,
                                      proba));
    } else {
      UML_CUDA(e, uml::launch_mlp_proba_f64(m->dm, b->x, b->ld, b->n_rows, proba, {}, true, e->info.sm_count, e->stream));
    }
    if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], e->stream));
    *launches = 1;
    *path = route;
    return UML_OK;
  };
  return predict_resident(e, b, {m->dm.n_classes, m->dm.n_in, "module", {proba_out, nullptr}, {4ll * m->dm.n_classes, 0},
                                 proba_on_device, UML_PREDICT_FAST, stats},
                          prepare, score);
}

int uml_mlp_predict_topk(uml_engine* e, const uml_mlp* m, const uml_batch* b, int k, int32_t* idx_out, float* proba_out,
                         int out_on_device, int mode, uml_stats* stats) {
  if (!e || !m) return UML_ERR_INVALID;
  const int C = m->dm.n_classes;
  if (k < 1 || k > C) UML_FAIL(e, UML_ERR_INVALID, "k = %d: the module has %d classes (need 1 <= k <= %d)", k, C, C);
  NvtxRange r_all("uml:mlp_topk");
  int route = 2;
  auto prepare = [&] {
    // k beyond what the tile kernels select in registers: the float64 kernel serves every row
    if (k <= uml::kMlpTopkMax) route = mlp_route(m->dm, b->has_map, false, [&] { return batch_tf32_exact(e, b) == 1; }, true);
    return (int)UML_OK;
  };
  auto score = [&](void* const* out, bool timed, int* launches, int* path, int*) -> int {
    int32_t* idx = static_cast<int32_t*>(out[0]);
    float* proba = static_cast<float*>(out[1]);
    const bool exact = mode == UML_PREDICT_EXACT;
    const FlagList fl = flag_list(e);
    const int sm = e->info.sm_count;
    cudaStream_t s = e->stream;
    *launches = 1;
    *path = route;
    if (route == 2) {
      UML_CUDA(e, uml::launch_mlp_topk_f64(m->dm, b->x, b->ld, b->n_rows, k, idx, proba, fl, true, sm, s));
      if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], s));
      return UML_OK;
    }
    if (route == 5) {
      uml::MlpTcLaunch o{};
      o.n_rows = b->n_rows;
      o.topk_idx = idx;
      o.topk_proba = proba;
      o.topk_k = k;
      // FAST: no flag list, so that no row waits for a float64 pass this call does not make (a batch routed here is
      // all tf32 values, unless UML_B200_MLP_TC=1 forces the route)
      UML_CUDA(e, uml::launch_mlp_tc_topk(b->map, m->dm, o, exact, exact ? fl : FlagList{}, sm, s));
    } else {
      UML_CUDA(e, uml::launch_mlp_tma_topk(b->map, m->dm, b->n_rows, k, idx, proba, exact, fl, sm, s));
    }
    if (timed) UML_CUDA(e, cudaEventRecord(e->ev[2], s));
    if (exact) {
      NvtxRange r_rescore("uml:mlp_topk_f64");
      UML_CUDA(e, uml::launch_mlp_topk_f64(m->dm, b->x, b->ld, b->n_rows, k, idx, proba, fl, false, sm, s));
      ++*launches;
    }
    return UML_OK;
  };
  return predict_resident(e, b, {C, m->dm.n_in, "module", {idx_out, proba_out}, {4ll * k, 4ll * k}, out_on_device, mode,
                                 stats},
                          prepare, score);
}

}  // extern "C"
