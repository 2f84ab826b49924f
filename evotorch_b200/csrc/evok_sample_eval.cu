// K1 / K2: fused Philox sampling -> perturbation write -> objective row-reduction, and the stand-alone
// evaluation kernel: the host side of the kernels in evok_sampler.cuh, for the built-in objectives and for the objectives
// registered at run time (evok_objective_register: NVRTC-compiled instantiations of the same kernels).
#include <cuda.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "evok_common.cuh"

namespace evok {

static int g_sm_count = 0;
static int sm_count() {
  if (g_sm_count == 0) {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kNumSMs;
    g_sm_count = n;
  }
  return g_sm_count;
}

// Batched searches (functional ask/tell API with leading batch dimensions, funcpgpe.py:301-327): blockIdx.y = batch item, every
// item has its own centre / stdev row (item stride 0 = shared) and its own Philox stream (stream word + item), so one launch
// draws the populations of all items -- bit-identical to one evok_sample_eval call per item with stream_id = item.
template <bool SYM, bool VEC>
__global__ void __launch_bounds__(kSampleThreads, SampleTune<ObjAcc<EVOK_OBJ_NONE>>::kMinBlocks)
    sample_batched_kernel(float* __restrict__ X, int64_t item_stride_x, int64_t ldx, const float* __restrict__ mu, int64_t item_stride_mu,
                          const float* __restrict__ sigma, int64_t item_stride_sigma, int64_t n_units, int64_t D, const __grid_constant__ PhiloxKey key) {
  const int lane = threadIdx.x & 31;
  const int64_t item = blockIdx.y;
  X += item * item_stride_x;
  mu += item * item_stride_mu;
  sigma += item * item_stride_sigma;
  const uint32_t sw = key.stream_lo + (uint32_t)item;
  const int64_t warps_total = (int64_t)gridDim.x * (kSampleThreads / 32);
  const int64_t gw = (int64_t)blockIdx.x * (kSampleThreads / 32) + (threadIdx.x >> 5);
  const uint32_t nq = (uint32_t)((D + 3) >> 2);
  for (int64_t u = gw; u < n_units; u += warps_total) {
    ObjAcc<EVOK_OBJ_NONE> accp(D), accm(D);
    float* xp = X + (SYM ? 2 * u : u) * ldx;
    float* xm = xp + ldx;
    for (uint32_t q = lane; q < nq; q += 32) sample_group<ObjAcc<EVOK_OBJ_NONE>, SYM, true, VEC>(key, sw, (uint64_t)u, q, D, mu, sigma, xp, xm, accp, accm);
  }
}

template <typename K>
static int resident_grid(K kernel, int threads, int64_t units_per_cta_needed) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm <= 0) per_sm = 4;
  int64_t g = (int64_t)per_sm * sm_count();
  if (g > units_per_cta_needed) g = units_per_cta_needed;
  if (g < 1) g = 1;
  return (int)g;
}

struct PushArgs {
  PeerSink sink;
  const unsigned long long* epoch;
  unsigned int* done;
};

template <int OBJ, bool SYM, bool STORE, bool PUSH = false, bool SQ = false>
static int launch_sample(float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D,
                         uint64_t seed, uint64_t stream_id, const uint32_t* stream_off, float* f, cudaStream_t st,
                         const PushArgs* push = nullptr, float* q = nullptr) {
  const int64_t n_units = SYM ? n_rows / 2 : n_rows;
  const bool vec = (D % 4 == 0) && aligned16(mu) && aligned16(sigma) && (!STORE || (aligned16(X) && ldx % 4 == 0));
  const int64_t ctas_needed = (n_units + (kSampleThreads / 32) - 1) / (kSampleThreads / 32);
  const PhiloxKey key = make_philox_key(seed, stream_id);
  PushArgs none{};
  const PushArgs& pa = PUSH ? *push : none;
  if (vec) {
    auto k = sample_eval_kernel<ObjAcc<OBJ>, SYM, STORE, true, PUSH, SQ>;
    k<<<resident_grid(k, kSampleThreads, ctas_needed), kSampleThreads, 0, st>>>(X, ldx, mu, sigma, row0, n_units, D, key, stream_off, f, pa.sink,
                                                                                pa.epoch, pa.done, q);
  } else {
    auto k = sample_eval_kernel<ObjAcc<OBJ>, SYM, STORE, false, PUSH, SQ>;
    k<<<resident_grid(k, kSampleThreads, ctas_needed), kSampleThreads, 0, st>>>(X, ldx, mu, sigma, row0, n_units, D, key, stream_off, f, pa.sink,
                                                                                pa.epoch, pa.done, q);
  }
  EVOK_CHECK_LAUNCH();
  return 0;
}

template <int OBJ>
static int dispatch_sample(float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D,
                           int symmetric, uint64_t seed, uint64_t stream_id, const uint32_t* stream_off, float* f, cudaStream_t st) {
  if (symmetric) {
    return X ? launch_sample<OBJ, true, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, f, st)
             : launch_sample<OBJ, true, false>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, f, st);
  }
  return X ? launch_sample<OBJ, false, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, f, st)
           : launch_sample<OBJ, false, false>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, f, st);
}

template <int OBJ>
static int dispatch_sample_sq(float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D, uint64_t seed,
                              uint64_t stream_id, const uint32_t* stream_off, float* f, float* q, cudaStream_t st) {
  if (X) return launch_sample<OBJ, false, true, false, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, f, st, nullptr, q);
  if constexpr (OBJ == EVOK_OBJ_NONE) return EVOK_E_NULLPTR;  // rejected by the entry point: no kernel for "q only"
  else return launch_sample<OBJ, false, false, false, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, f, st, nullptr, q);
}

template <int OBJ>
static int dispatch_sample_push(float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D,
                                int symmetric, uint64_t seed, uint64_t stream_id, const uint32_t* stream_off, const PushArgs& push, cudaStream_t st) {
  if (symmetric) {
    return X ? launch_sample<OBJ, true, true, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, nullptr, st, &push)
             : launch_sample<OBJ, true, false, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, nullptr, st, &push);
  }
  return X ? launch_sample<OBJ, false, true, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, nullptr, st, &push)
           : launch_sample<OBJ, false, false, true>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_off, nullptr, st, &push);
}

template <int OBJ>
static int launch_eval(const float* X, int64_t ldx, int64_t n_rows, int64_t D, float* f, cudaStream_t st) {
  const bool vec = (D % 4 == 0) && aligned16(X) && (ldx % 4 == 0);
  const int64_t ctas_needed = (n_rows + (kEvalThreads / 32) - 1) / (kEvalThreads / 32);
  if (vec) {
    auto k = eval_kernel<ObjAcc<OBJ>, true>;
    k<<<resident_grid(k, kEvalThreads, ctas_needed), kEvalThreads, 0, st>>>(X, ldx, n_rows, D, f);
  } else {
    auto k = eval_kernel<ObjAcc<OBJ>, false>;
    k<<<resident_grid(k, kEvalThreads, ctas_needed), kEvalThreads, 0, st>>>(X, ldx, n_rows, D, f);
  }
  EVOK_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Objectives registered at run time.  A registration keeps a copy of the cubin and the lowered names of its kernels (in the
// EVOK_OBJ_KERNEL_* order); the module is loaded into the current device's primary context on the first use on that device
// (each device has its own module, functions, occupancy and SM count).  Loaded modules stay until the process ends.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxDevices = 64;

struct UserDevice {
  int state = 0;  // 0: not loaded; 1: loaded; EVOK_E_NOKERNEL: the cubin lacks a kernel (a permanent failure)
  CUmodule module = nullptr;
  CUfunction fn[EVOK_OBJ_KERNELS] = {};
  int per_sm[EVOK_OBJ_KERNELS] = {};
  int sms = 0;
};

struct UserObjective {
  std::vector<char> image;
  std::vector<std::string> names;
  UserDevice dev[kMaxDevices];
};

// the driver API through the runtime's entry points (the library does not link libcuda)
struct DriverApi {
  decltype(&cuDeviceGet) device_get = nullptr;
  decltype(&cuDeviceGetAttribute) device_attribute = nullptr;
  decltype(&cuModuleLoadData) module_load = nullptr;
  decltype(&cuModuleGetFunction) module_function = nullptr;
  decltype(&cuModuleUnload) module_unload = nullptr;
  decltype(&cuOccupancyMaxActiveBlocksPerMultiprocessor) occupancy = nullptr;
  decltype(&cuLaunchKernel) launch = nullptr;
};
static DriverApi g_driver;

template <typename F>
static bool driver_symbol(const char* name, F& fn) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return false;
  fn = reinterpret_cast<F>(p);
  return true;
}

static bool driver_api() {
  DriverApi& d = g_driver;
  if (d.launch) return true;
  return driver_symbol("cuDeviceGet", d.device_get) && driver_symbol("cuDeviceGetAttribute", d.device_attribute) &&
         driver_symbol("cuModuleLoadData", d.module_load) && driver_symbol("cuModuleGetFunction", d.module_function) &&
         driver_symbol("cuModuleUnload", d.module_unload) && driver_symbol("cuOccupancyMaxActiveBlocksPerMultiprocessor", d.occupancy) &&
         driver_symbol("cuLaunchKernel", d.launch);
}

static std::mutex g_user_mutex;
static UserObjective* g_user[EVOK_OBJ_USER_CAPACITY];
static std::atomic<int> g_user_count{0};

static bool is_user(int objective) {
  return objective >= EVOK_OBJ_USER_BASE && objective - EVOK_OBJ_USER_BASE < g_user_count.load(std::memory_order_acquire);
}

static int kernel_threads(int k) { return k >= EVOK_OBJ_KERNEL_EVAL ? kEvalThreads : kSampleThreads; }

// The loaded module of a registered objective on the current device (loaded here on the first call for that device).
static int user_device(int objective, const UserDevice** out) {
  int dev = 0;
  cudaError_t ce = cudaGetDevice(&dev);
  if (ce != cudaSuccess) return (int)ce;
  if (dev < 0 || dev >= kMaxDevices) return EVOK_E_BADSIZE;
  std::lock_guard<std::mutex> lock(g_user_mutex);
  UserObjective& obj = *g_user[objective - EVOK_OBJ_USER_BASE];
  UserDevice& d = obj.dev[dev];
  if (d.state == 0) {
    ce = cudaSetDevice(dev);  // makes the device's primary context (the runtime's) current, creating it if needed
    if (ce != cudaSuccess) return (int)ce;
    if (!driver_api()) return (int)cudaErrorNotSupported;
    const DriverApi& api = g_driver;
    CUdevice cu_dev;
    CUresult r = api.device_get(&cu_dev, dev);
    if (r == CUDA_SUCCESS) r = api.device_attribute(&d.sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, cu_dev);
    if (r == CUDA_SUCCESS) r = api.module_load(&d.module, obj.image.data());
    if (r != CUDA_SUCCESS) return (int)r;  // CUresult and cudaError_t share their codes
    for (int k = 0; k < EVOK_OBJ_KERNELS; ++k) {
      if (api.module_function(&d.fn[k], d.module, obj.names[k].c_str()) != CUDA_SUCCESS) {
        api.module_unload(d.module);
        d.module = nullptr;
        d.state = EVOK_E_NOKERNEL;
        return d.state;
      }
      if (api.occupancy(&d.per_sm[k], d.fn[k], kernel_threads(k), 0) != CUDA_SUCCESS || d.per_sm[k] <= 0) d.per_sm[k] = 4;
    }
    if (d.sms <= 0) d.sms = kNumSMs;
    d.state = 1;
  }
  if (d.state != 1) return d.state;
  *out = &d;
  return 0;
}

// the launch of kernel k with the grid rule of resident_grid (the driver API is resolved: user_device succeeded)
static int user_launch(const UserDevice& d, int k, int64_t ctas_needed, void** args, cudaStream_t st) {
  int64_t g = (int64_t)d.per_sm[k] * d.sms;
  if (g > ctas_needed) g = ctas_needed;
  if (g < 1) g = 1;
  const CUresult r = g_driver.launch(d.fn[k], (unsigned)g, 1, 1, kernel_threads(k), 1, 1, 0, (CUstream)st, args, nullptr);
  if (r != CUDA_SUCCESS) return (int)r;
  count_launches(1);
  return 0;
}

// launch_sample for a registered objective: the same kernel choice (symmetric, store, VEC, PUSH, SQ) and grid
static int user_sample(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D,
                       bool sym, uint64_t seed, uint64_t stream_id, const uint32_t* stream_off, float* f, cudaStream_t st,
                       const PushArgs* push = nullptr, float* q = nullptr) {
  const UserDevice* d = nullptr;
  const int rc = user_device(objective, &d);
  if (rc != 0) return rc;
  const bool store = X != nullptr;
  int64_t n_units = sym ? n_rows / 2 : n_rows;
  const bool vec = (D % 4 == 0) && aligned16(mu) && aligned16(sigma) && (!store || (aligned16(X) && ldx % 4 == 0));
  const int64_t ctas_needed = (n_units + (kSampleThreads / 32) - 1) / (kSampleThreads / 32);
  PhiloxKey key = make_philox_key(seed, stream_id);
  PushArgs pa{};
  if (push) pa = *push;
  const int variant = (store ? 2 : 0) + (vec ? 1 : 0);
  const int k = q ? EVOK_OBJ_KERNEL_SQ + variant : (push ? EVOK_OBJ_KERNEL_PUSH : EVOK_OBJ_KERNEL_SAMPLE) + (sym ? 4 : 0) + variant;
  void* args[] = {&X, &ldx, &mu, &sigma, &row0, &n_units, &D, &key, &stream_off, &f, &pa.sink, &pa.epoch, &pa.done, &q};
  return user_launch(*d, k, ctas_needed, args, st);
}

static int user_eval(int objective, const float* X, int64_t ldx, int64_t n_rows, int64_t D, float* f, cudaStream_t st) {
  const UserDevice* d = nullptr;
  const int rc = user_device(objective, &d);
  if (rc != 0) return rc;
  const bool vec = (D % 4 == 0) && aligned16(X) && (ldx % 4 == 0);
  const int64_t ctas_needed = (n_rows + (kEvalThreads / 32) - 1) / (kEvalThreads / 32);
  void* args[] = {&X, &ldx, &n_rows, &D, &f};
  return user_launch(*d, EVOK_OBJ_KERNEL_EVAL + (vec ? 1 : 0), ctas_needed, args, st);
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API int evok_objective_register(const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels,
                                                int* id_out_host) {
  if (!cubin || !kernel_names_host || !id_out_host) return EVOK_E_NULLPTR;
  if (bytes == 0 || n_kernels != EVOK_OBJ_KERNELS) return EVOK_E_BADSIZE;
  for (int k = 0; k < n_kernels; ++k)
    if (!kernel_names_host[k]) return EVOK_E_NULLPTR;
  std::lock_guard<std::mutex> lock(g_user_mutex);
  const int n = g_user_count.load(std::memory_order_relaxed);
  if (n >= EVOK_OBJ_USER_CAPACITY) return EVOK_E_BADSIZE;
  UserObjective* obj = new UserObjective;
  obj->image.assign(static_cast<const char*>(cubin), static_cast<const char*>(cubin) + bytes);
  for (int k = 0; k < n_kernels; ++k) obj->names.emplace_back(kernel_names_host[k]);
  g_user[n] = obj;
  g_user_count.store(n + 1, std::memory_order_release);
  *id_out_host = EVOK_OBJ_USER_BASE + n;
  return 0;
}

extern "C" EVOK_API int evok_objective_load(int objective) {
  if (!is_user(objective)) return EVOK_E_BADENUM;
  const UserDevice* d = nullptr;
  return user_device(objective, &d);
}

extern "C" EVOK_API int evok_sample_eval(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0,
                                int64_t n_rows, int64_t D, int symmetric, uint64_t seed, uint64_t stream_id,
                                const uint32_t* stream_offset_dev, float* f, void* stream) {
  const uint32_t* stream_off = stream_offset_dev;
  if (!mu || !sigma) return EVOK_E_NULLPTR;
  const bool user = is_user(objective);
  if ((objective < 0 || objective >= EVOK_OBJ_COUNT) && !user) return EVOK_E_BADENUM;
  if (objective == EVOK_OBJ_NONE && !X) return EVOK_E_NULLPTR;
  if (objective != EVOK_OBJ_NONE && !f) return EVOK_E_NULLPTR;
  if (n_rows < 0 || D <= 0 || row0 < 0 || (X && ldx < D)) return EVOK_E_BADSIZE;
  if (symmetric && ((n_rows & 1) || (row0 & 1))) return EVOK_E_ODDROWS;
  if (n_rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (user) return user_sample(objective, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, seed, stream_id, stream_off, f, st);
  switch (objective) {
    case EVOK_OBJ_NONE: return dispatch_sample<EVOK_OBJ_NONE>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_off, f, st);
    case EVOK_OBJ_SPHERE: return dispatch_sample<EVOK_OBJ_SPHERE>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_off, f, st);
    case EVOK_OBJ_RASTRIGIN: return dispatch_sample<EVOK_OBJ_RASTRIGIN>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_off, f, st);
    case EVOK_OBJ_ACKLEY: return dispatch_sample<EVOK_OBJ_ACKLEY>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_off, f, st);
  }
  return EVOK_E_BADENUM;
}

extern "C" EVOK_API int evok_sample_eval_sq(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                                            int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float* f, float* q,
                                            void* stream) {
  if (!mu || !sigma || !q) return EVOK_E_NULLPTR;
  const bool user = is_user(objective);
  if ((objective < 0 || objective >= EVOK_OBJ_COUNT) && !user) return EVOK_E_BADENUM;
  if (objective == EVOK_OBJ_NONE && !X) return EVOK_E_NULLPTR;
  if (objective != EVOK_OBJ_NONE && !f) return EVOK_E_NULLPTR;
  if (n_rows < 0 || D <= 0 || row0 < 0 || (X && ldx < D)) return EVOK_E_BADSIZE;
  if (n_rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (user) return user_sample(objective, X, ldx, mu, sigma, row0, n_rows, D, false, seed, stream_id, stream_offset_dev, f, st, nullptr, q);
  switch (objective) {
    case EVOK_OBJ_NONE: return dispatch_sample_sq<EVOK_OBJ_NONE>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_offset_dev, f, q, st);
    case EVOK_OBJ_SPHERE: return dispatch_sample_sq<EVOK_OBJ_SPHERE>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_offset_dev, f, q, st);
    case EVOK_OBJ_RASTRIGIN: return dispatch_sample_sq<EVOK_OBJ_RASTRIGIN>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_offset_dev, f, q, st);
    case EVOK_OBJ_ACKLEY: return dispatch_sample_sq<EVOK_OBJ_ACKLEY>(X, ldx, mu, sigma, row0, n_rows, D, seed, stream_id, stream_offset_dev, f, q, st);
  }
  return EVOK_E_BADENUM;
}

extern "C" EVOK_API int evok_sample_eval_push(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                                              int64_t D, int symmetric, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev,
                                              int world, int rank, void* const* peer_f, void* const* peer_flags, const uint64_t* epoch_dev,
                                              uint32_t* done_dev, void* stream) {
  if (!mu || !sigma || !peer_f || !peer_flags || !epoch_dev || !done_dev) return EVOK_E_NULLPTR;
  const bool user = is_user(objective);
  if ((objective <= EVOK_OBJ_NONE || objective >= EVOK_OBJ_COUNT) && !user) return EVOK_E_BADENUM;
  if (world < 1 || world > EVOK_MAX_PEERS || rank < 0 || rank >= world) return EVOK_E_BADSIZE;
  if (n_rows < 0 || D <= 0 || row0 < 0 || (X && ldx < D)) return EVOK_E_BADSIZE;
  if (symmetric && ((n_rows & 1) || (row0 & 1))) return EVOK_E_ODDROWS;
  PushArgs push{};
  push.sink.world = world;
  push.sink.rank = rank;
  for (int p = 0; p < world; ++p) {
    if (!peer_f[p] || !peer_flags[p]) return EVOK_E_NULLPTR;
    push.sink.data[p] = peer_f[p];
    push.sink.flags[p] = static_cast<unsigned long long*>(peer_flags[p]);
  }
  push.epoch = reinterpret_cast<const unsigned long long*>(epoch_dev);
  push.done = done_dev;
  // n_rows == 0 still launches one CTA: the peers wait for this rank's flag
  cudaStream_t st = (cudaStream_t)stream;
  if (user) return user_sample(objective, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, seed, stream_id, stream_offset_dev, nullptr, st, &push);
  switch (objective) {
    case EVOK_OBJ_SPHERE: return dispatch_sample_push<EVOK_OBJ_SPHERE>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_offset_dev, push, st);
    case EVOK_OBJ_RASTRIGIN: return dispatch_sample_push<EVOK_OBJ_RASTRIGIN>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_offset_dev, push, st);
    case EVOK_OBJ_ACKLEY: return dispatch_sample_push<EVOK_OBJ_ACKLEY>(X, ldx, mu, sigma, row0, n_rows, D, symmetric, seed, stream_id, stream_offset_dev, push, st);
  }
  return EVOK_E_BADENUM;
}

extern "C" EVOK_API int evok_eval(int objective, const float* X, int64_t ldx, int64_t n_rows, int64_t D, float* f, void* stream) {
  if (!X || !f) return EVOK_E_NULLPTR;
  const bool user = is_user(objective);
  if ((objective <= EVOK_OBJ_NONE || objective >= EVOK_OBJ_COUNT) && !user) return EVOK_E_BADENUM;
  if (n_rows < 0 || D <= 0 || ldx < D) return EVOK_E_BADSIZE;
  if (n_rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (user) return user_eval(objective, X, ldx, n_rows, D, f, st);
  switch (objective) {
    case EVOK_OBJ_SPHERE: return launch_eval<EVOK_OBJ_SPHERE>(X, ldx, n_rows, D, f, st);
    case EVOK_OBJ_RASTRIGIN: return launch_eval<EVOK_OBJ_RASTRIGIN>(X, ldx, n_rows, D, f, st);
    case EVOK_OBJ_ACKLEY: return launch_eval<EVOK_OBJ_ACKLEY>(X, ldx, n_rows, D, f, st);
  }
  return EVOK_E_BADENUM;
}

extern "C" EVOK_API int evok_sample_batched(float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu, const float* sigma,
                                            int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, int symmetric, uint64_t seed,
                                            uint64_t stream_id0, void* stream) {
  if (!X || !mu || !sigma) return EVOK_E_NULLPTR;
  if (n_items < 0 || n_rows < 0 || D <= 0 || ldx < D || item_stride_x < 0 || item_stride_mu < 0 || item_stride_sigma < 0)
    return EVOK_E_BADSIZE;
  if (symmetric && (n_rows & 1)) return EVOK_E_ODDROWS;
  if (n_items == 0 || n_rows == 0) return 0;
  const int64_t n_units = symmetric ? n_rows / 2 : n_rows;
  const bool vec = (D % 4 == 0) && aligned16(mu) && aligned16(sigma) && aligned16(X) && ldx % 4 == 0 && item_stride_x % 4 == 0 &&
                   item_stride_mu % 4 == 0 && item_stride_sigma % 4 == 0;
  int64_t ctas = (n_units + (kSampleThreads / 32) - 1) / (kSampleThreads / 32);
  const int64_t cap = ((int64_t)sm_count() * 8 + n_items - 1) / n_items;  // about 8 CTAs per SM over all items
  if (ctas > cap) ctas = cap < 1 ? 1 : cap;
  const PhiloxKey key = make_philox_key(seed, stream_id0);
  cudaStream_t st = (cudaStream_t)stream;
  // grid y is at most kMaxGridY items: larger batches go in item chunks, chunk b0 starting at stream word stream_lo + b0, so item b
  // keeps its Philox stream stream_id0 + b
  for (int64_t b0 = 0; b0 < n_items; b0 += kMaxGridY) {
    const int64_t nb = n_items - b0 < kMaxGridY ? n_items - b0 : kMaxGridY;
    PhiloxKey kc = key;
    kc.stream_lo += (uint32_t)b0;
    const dim3 grid((unsigned)ctas, (unsigned)nb);
    float* Xc = X + b0 * item_stride_x;
    const float* muc = mu + b0 * item_stride_mu;
    const float* sgc = sigma + b0 * item_stride_sigma;
#define EVOK_LAUNCH_SB(SYMV, VECV) \
  sample_batched_kernel<SYMV, VECV><<<grid, kSampleThreads, 0, st>>>(Xc, item_stride_x, ldx, muc, item_stride_mu, sgc, item_stride_sigma, n_units, D, kc)
    if (symmetric) {
      if (vec) EVOK_LAUNCH_SB(true, true);
      else EVOK_LAUNCH_SB(true, false);
    } else {
      if (vec) EVOK_LAUNCH_SB(false, true);
      else EVOK_LAUNCH_SB(false, false);
    }
#undef EVOK_LAUNCH_SB
    EVOK_CHECK_LAUNCH();
  }
  return 0;
}
