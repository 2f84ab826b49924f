// K1 / K2: fused Philox sampling -> perturbation write -> objective row-reduction, and the stand-alone
// evaluation kernel: the host side of the kernels in evok_sampler.cuh, for the built-in objectives and for the objectives
// registered at run time (evok_objective_register: NVRTC-compiled instantiations of the same kernels).
#include <cuda.h>

#include <atomic>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "evok_common.cuh"

namespace evok {

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

struct PushArgs {
  PeerSink sink;
  const unsigned long long* epoch;
  unsigned int* done;
};

// ------------------------------------------------------------------------------------------------
// The kernel table.  Every objective, built-in or registered at run time (evok_objective_register: NVRTC-compiled
// instantiations of the same kernels), has the EVOK_OBJ_KERNELS kernels of include/evok.h on each device.  One rule picks the
// kernel of a call (choose_kernel) and one function launches it (launch).
// ------------------------------------------------------------------------------------------------

// The position of a kernel in the EVOK_OBJ_KERNEL_* order: its family (EVOK_OBJ_KERNEL_SAMPLE, _PUSH, _SQ or _EVAL), then
// + 4 sym (SAMPLE and PUSH), + 2 store (all but EVAL), + vec.  jit.kernel_expressions() lists a registered objective's kernels
// in the same order.
constexpr int kernel_index(int family, bool sym, bool store, bool vec) {
  return family + (sym && family < EVOK_OBJ_KERNEL_SQ ? 4 : 0) + (store && family < EVOK_OBJ_KERNEL_EVAL ? 2 : 0) + (vec ? 1 : 0);
}

static int kernel_threads(int k) { return k >= EVOK_OBJ_KERNEL_EVAL ? kEvalThreads : kSampleThreads; }

// The sampler of built-in objective OBJ with the variant bits V = sym | store << 1 | vec << 2 | push << 3 | sq << 4, if it
// exists (the SQ sampler is plain and non-symmetric) and can be reached: EVOK_OBJ_NONE only stores samples, since
// evok_sample_eval and _sq refuse it without X, and _push refuses it always.
template <int OBJ, int V>
static void put_builtin_sampler(void** fn) {
  constexpr bool sym = V & 1, store = V & 2, vec = V & 4, push = V & 8, sq = V & 16;
  if constexpr (!(sq && (sym || push)) && (OBJ != EVOK_OBJ_NONE || (store && !push)))
    fn[kernel_index(sq ? EVOK_OBJ_KERNEL_SQ : push ? EVOK_OBJ_KERNEL_PUSH : EVOK_OBJ_KERNEL_SAMPLE, sym, store, vec)] =
        reinterpret_cast<void*>(sample_eval_kernel<ObjAcc<OBJ>, sym, store, vec, push, sq>);
}

template <int OBJ, int... V>
static void put_builtin_kernels(void** fn, std::integer_sequence<int, V...>) {
  (put_builtin_sampler<OBJ, V>(fn), ...);
  if constexpr (OBJ != EVOK_OBJ_NONE) {  // evok_eval refuses EVOK_OBJ_NONE
    fn[kernel_index(EVOK_OBJ_KERNEL_EVAL, false, true, false)] = reinterpret_cast<void*>(eval_kernel<ObjAcc<OBJ>, false>);
    fn[kernel_index(EVOK_OBJ_KERNEL_EVAL, false, true, true)] = reinterpret_cast<void*>(eval_kernel<ObjAcc<OBJ>, true>);
  }
}

template <int OBJ>
static void builtin_kernels(void** fn) {
  put_builtin_kernels<OBJ>(fn, std::make_integer_sequence<int, 32>());
}

static void (*const kBuiltinKernels[EVOK_OBJ_COUNT])(void**) = {builtin_kernels<EVOK_OBJ_NONE>, builtin_kernels<EVOK_OBJ_SPHERE>,
                                                                 builtin_kernels<EVOK_OBJ_RASTRIGIN>, builtin_kernels<EVOK_OBJ_ACKLEY>};

constexpr int kMaxDevices = 64;

// The kernels of one objective on one device, filled on the first use there and kept until the process ends.  A built-in
// objective's entries are its nvcc-compiled kernels (null where no entry point reaches them); a registered objective's are the
// functions of its module, loaded into the device's primary context.
struct DeviceKernels {
  int state = 0;              // 0: not filled; 1: filled; EVOK_E_NOKERNEL: the cubin lacks a kernel (a permanent failure)
  CUmodule module = nullptr;  // set for a registered objective: fn holds CUfunctions, launched through the driver
  void* fn[EVOK_OBJ_KERNELS] = {};
  int per_sm[EVOK_OBJ_KERNELS] = {};  // resident CTAs per SM
  int sms = 0;
};

struct Objective {
  std::vector<char> image;  // a registered objective's cubin and the lowered names of its kernels (in the EVOK_OBJ_KERNEL_* order)
  std::vector<std::string> names;
  DeviceKernels dev[kMaxDevices];
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

static std::mutex g_objective_mutex;
static Objective g_builtin[EVOK_OBJ_COUNT];
static Objective* g_user[EVOK_OBJ_USER_CAPACITY];
static std::atomic<int> g_user_count{0};

static bool is_user(int objective) {
  return objective >= EVOK_OBJ_USER_BASE && objective - EVOK_OBJ_USER_BASE < g_user_count.load(std::memory_order_acquire);
}

static void fill_builtin(int objective, int dev, DeviceKernels& d) {
  kBuiltinKernels[objective](d.fn);
  for (int k = 0; k < EVOK_OBJ_KERNELS; ++k)
    if (d.fn[k] && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.per_sm[k], d.fn[k], kernel_threads(k), 0) != cudaSuccess || d.per_sm[k] <= 0))
      d.per_sm[k] = 4;
  if (cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.sms <= 0) d.sms = kNumSMs;
  d.state = 1;
}

static int load_module(const Objective& obj, int dev, DeviceKernels& d) {
  cudaError_t ce = cudaSetDevice(dev);  // makes the device's primary context (the runtime's) current, creating it if needed
  if (ce != cudaSuccess) return (int)ce;
  if (!driver_api()) return (int)cudaErrorNotSupported;
  const DriverApi& api = g_driver;
  CUdevice cu_dev;
  CUresult r = api.device_get(&cu_dev, dev);
  if (r == CUDA_SUCCESS) r = api.device_attribute(&d.sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, cu_dev);
  if (r == CUDA_SUCCESS) r = api.module_load(&d.module, obj.image.data());
  if (r != CUDA_SUCCESS) return (int)r;  // CUresult and cudaError_t share their codes
  for (int k = 0; k < EVOK_OBJ_KERNELS; ++k) {
    CUfunction fn = nullptr;
    if (api.module_function(&fn, d.module, obj.names[k].c_str()) != CUDA_SUCCESS) {
      api.module_unload(d.module);
      d.module = nullptr;
      d.state = EVOK_E_NOKERNEL;
      return d.state;
    }
    d.fn[k] = fn;
    if (api.occupancy(&d.per_sm[k], fn, kernel_threads(k), 0) != CUDA_SUCCESS || d.per_sm[k] <= 0) d.per_sm[k] = 4;
  }
  if (d.sms <= 0) d.sms = kNumSMs;
  d.state = 1;
  return 0;
}

// The kernel table of an objective (a built-in id or a registered one) on the current device, filled here on the first call
// for that device.
static int device_kernels(int objective, const DeviceKernels** out) {
  int dev = 0;
  const cudaError_t ce = cudaGetDevice(&dev);
  if (ce != cudaSuccess) return (int)ce;
  if (dev < 0 || dev >= kMaxDevices) return EVOK_E_BADSIZE;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const bool user = objective >= EVOK_OBJ_USER_BASE;
  Objective& obj = user ? *g_user[objective - EVOK_OBJ_USER_BASE] : g_builtin[objective];
  DeviceKernels& d = obj.dev[dev];
  if (d.state == 0) {
    if (!user) fill_builtin(objective, dev, d);
    else if (const int rc = load_module(obj, dev, d)) return rc;
  }
  if (d.state != 1) return d.state;
  *out = &d;
  return 0;
}

struct KernelChoice {
  int k;                // index in the EVOK_OBJ_KERNEL_* order
  int64_t n_units;      // rows, or antithetic row pairs for symmetric sampling; one warp each
  int64_t ctas_needed;  // CTAs that give every unit its own warp
};

// The kernel of a call: family (EVOK_OBJ_KERNEL_*) and sym; stored samples when X is given; the vectorised variant when
// D % 4 == 0 and every operand read or written with float4 loads / stores is 16-byte aligned with 16-byte aligned rows (mu and
// sigma are null for the evaluation kernel, which reads X only).
static KernelChoice choose_kernel(int family, bool sym, const float* X, int64_t ldx, const float* mu, const float* sigma, int64_t n_rows,
                                  int64_t D) {
  const bool store = X != nullptr;
  const bool vec = (D % 4 == 0) && aligned16(mu) && aligned16(sigma) && (!store || (aligned16(X) && ldx % 4 == 0));
  KernelChoice c;
  c.k = kernel_index(family, sym, store, vec);
  c.n_units = sym ? n_rows / 2 : n_rows;
  const int warps = kernel_threads(c.k) / 32;
  c.ctas_needed = (c.n_units + warps - 1) / warps;
  return c;
}

// Launches kernel c.k of an objective on the current device with `args` in the kernel's parameter order, on as many CTAs as
// stay resident but no more than the units need, and at least one (the push sampler with no rows still raises this rank's
// flag).  A built-in kernel goes through the runtime, a registered one through the driver.
static int launch(int objective, const KernelChoice& c, void** args, cudaStream_t st) {
  const DeviceKernels* d = nullptr;
  const int rc = device_kernels(objective, &d);
  if (rc != 0) return rc;
  int64_t g = (int64_t)d->per_sm[c.k] * d->sms;
  if (g > c.ctas_needed) g = c.ctas_needed;
  if (g < 1) g = 1;
  const int threads = kernel_threads(c.k);
  if (d->module) {
    const CUresult r = g_driver.launch(static_cast<CUfunction>(d->fn[c.k]), (unsigned)g, 1, 1, threads, 1, 1, 0, (CUstream)st, args, nullptr);
    if (r != CUDA_SUCCESS) return (int)r;
    count_launches(1);
    return 0;
  }
  cudaLaunchKernel(d->fn[c.k], dim3((unsigned)g), dim3(threads), args, 0, st);
  EVOK_CHECK_LAUNCH();
  return 0;
}

// The argument checks of evok_sample_eval, _sq and _push, in the order of include/evok.h's error codes for them: the first
// check that fails gives the code (the pointers only one entry point takes are checked there first, with mu and sigma).
// push: the peer-exchange sampler, which takes no f, has no kernels for EVOK_OBJ_NONE and checks its world and rank.
static int check_sample(int objective, const float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                        int64_t D, bool sym, const float* f, const PushArgs* push) {
  if (!mu || !sigma) return EVOK_E_NULLPTR;
  const int first = push ? EVOK_OBJ_NONE + 1 : EVOK_OBJ_NONE;
  if ((objective < first || objective >= EVOK_OBJ_COUNT) && !is_user(objective)) return EVOK_E_BADENUM;
  if (push) {
    if (push->sink.world < 1 || push->sink.world > EVOK_MAX_PEERS || push->sink.rank < 0 || push->sink.rank >= push->sink.world)
      return EVOK_E_BADSIZE;
  } else {
    if (objective == EVOK_OBJ_NONE && !X) return EVOK_E_NULLPTR;
    if (objective != EVOK_OBJ_NONE && !f) return EVOK_E_NULLPTR;
  }
  if (n_rows < 0 || D <= 0 || row0 < 0 || (X && ldx < D)) return EVOK_E_BADSIZE;
  if (sym && ((n_rows & 1) || (row0 & 1))) return EVOK_E_ODDROWS;
  return 0;
}

// One launch of a sampler of family EVOK_OBJ_KERNEL_SAMPLE, _PUSH (push set) or _SQ (q set).
static int sample(int objective, int family, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                  int64_t D, bool sym, uint64_t seed, uint64_t stream_id, const uint32_t* stream_off, float* f, float* q, PushArgs push,
                  cudaStream_t st) {
  KernelChoice c = choose_kernel(family, sym, X, ldx, mu, sigma, n_rows, D);
  PhiloxKey key = make_philox_key(seed, stream_id);
  void* args[] = {&X, &ldx, &mu, &sigma, &row0, &c.n_units, &D, &key, &stream_off, &f, &push.sink, &push.epoch, &push.done, &q};
  return launch(objective, c, args, st);
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API int evok_objective_register(const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels,
                                                int* id_out_host) {
  if (!cubin || !kernel_names_host || !id_out_host) return EVOK_E_NULLPTR;
  if (bytes == 0 || n_kernels != EVOK_OBJ_KERNELS) return EVOK_E_BADSIZE;
  for (int k = 0; k < n_kernels; ++k)
    if (!kernel_names_host[k]) return EVOK_E_NULLPTR;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const int n = g_user_count.load(std::memory_order_relaxed);
  if (n >= EVOK_OBJ_USER_CAPACITY) return EVOK_E_BADSIZE;
  Objective* obj = new Objective;
  obj->image.assign(static_cast<const char*>(cubin), static_cast<const char*>(cubin) + bytes);
  for (int k = 0; k < n_kernels; ++k) obj->names.emplace_back(kernel_names_host[k]);
  g_user[n] = obj;
  g_user_count.store(n + 1, std::memory_order_release);
  *id_out_host = EVOK_OBJ_USER_BASE + n;
  return 0;
}

extern "C" EVOK_API int evok_objective_load(int objective) {
  if (!is_user(objective)) return EVOK_E_BADENUM;
  const DeviceKernels* d = nullptr;
  return device_kernels(objective, &d);
}

extern "C" EVOK_API int evok_sample_eval(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0,
                                int64_t n_rows, int64_t D, int symmetric, uint64_t seed, uint64_t stream_id,
                                const uint32_t* stream_offset_dev, float* f, void* stream) {
  const int rc = check_sample(objective, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, f, nullptr);
  if (rc != 0 || n_rows == 0) return rc;
  return sample(objective, EVOK_OBJ_KERNEL_SAMPLE, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, seed, stream_id, stream_offset_dev, f,
                nullptr, PushArgs{}, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_sample_eval_sq(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                                            int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float* f, float* q,
                                            void* stream) {
  if (!q) return EVOK_E_NULLPTR;
  const int rc = check_sample(objective, X, ldx, mu, sigma, row0, n_rows, D, false, f, nullptr);
  if (rc != 0 || n_rows == 0) return rc;
  return sample(objective, EVOK_OBJ_KERNEL_SQ, X, ldx, mu, sigma, row0, n_rows, D, false, seed, stream_id, stream_offset_dev, f, q, PushArgs{},
                (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_sample_eval_push(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                                              int64_t D, int symmetric, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev,
                                              int world, int rank, void* const* peer_f, void* const* peer_flags, const uint64_t* epoch_dev,
                                              uint32_t* done_dev, void* stream) {
  if (!peer_f || !peer_flags || !epoch_dev || !done_dev) return EVOK_E_NULLPTR;
  PushArgs push{};
  push.sink.world = world;
  push.sink.rank = rank;
  push.epoch = reinterpret_cast<const unsigned long long*>(epoch_dev);
  push.done = done_dev;
  const int rc = check_sample(objective, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, nullptr, &push);
  if (rc != 0) return rc;
  for (int p = 0; p < world; ++p) {
    if (!peer_f[p] || !peer_flags[p]) return EVOK_E_NULLPTR;
    push.sink.data[p] = peer_f[p];
    push.sink.flags[p] = static_cast<unsigned long long*>(peer_flags[p]);
  }
  // n_rows == 0 still launches one CTA: the peers wait for this rank's flag
  return sample(objective, EVOK_OBJ_KERNEL_PUSH, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, seed, stream_id, stream_offset_dev,
                nullptr, nullptr, push, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_eval(int objective, const float* X, int64_t ldx, int64_t n_rows, int64_t D, float* f, void* stream) {
  if (!X || !f) return EVOK_E_NULLPTR;
  if ((objective <= EVOK_OBJ_NONE || objective >= EVOK_OBJ_COUNT) && !is_user(objective)) return EVOK_E_BADENUM;
  if (n_rows < 0 || D <= 0 || ldx < D) return EVOK_E_BADSIZE;
  if (n_rows == 0) return 0;
  const KernelChoice c = choose_kernel(EVOK_OBJ_KERNEL_EVAL, false, X, ldx, nullptr, nullptr, n_rows, D);
  void* args[] = {&X, &ldx, &n_rows, &D, &f};
  return launch(objective, c, args, (cudaStream_t)stream);
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
  const DeviceKernels* d = nullptr;
  const int rc = device_kernels(EVOK_OBJ_NONE, &d);
  if (rc != 0) return rc;
  const int64_t cap = ((int64_t)d->sms * 8 + n_items - 1) / n_items;  // about 8 CTAs per SM over all items
  if (ctas > cap) ctas = cap < 1 ? 1 : cap;
  const PhiloxKey key = make_philox_key(seed, stream_id0);
  cudaStream_t st = (cudaStream_t)stream;
  // grid y is at most kMaxGridY items: larger batches go in item chunks, chunk b0 starting at stream word stream_lo + b0, so item b
  // keeps its Philox stream stream_id0 + b
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
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
    return 0;
  });
}
