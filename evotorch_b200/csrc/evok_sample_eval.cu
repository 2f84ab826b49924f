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

// The position of a kernel in the EVOK_OBJ_KERNEL_* order: its family (EVOK_OBJ_KERNEL_SAMPLE, _PUSH, _SQ, _EVAL, _BATCHED or
// _EVAL_BATCHED), then + 4 sym (SAMPLE, PUSH and BATCHED), + 2 store (all but the evaluation families), + vec.
// jit.kernel_expressions() lists a registered objective's first EVOK_OBJ_KERNELS kernels in the same order,
// jit.batched_kernel_expressions() its batched samplers and jit.eval_batched_kernel_expressions() its batched evaluation.
constexpr bool is_eval_family(int family) { return family == EVOK_OBJ_KERNEL_EVAL || family == EVOK_OBJ_KERNEL_EVAL_BATCHED; }
constexpr int kernel_index(int family, bool sym, bool store, bool vec) {
  return family + (sym && (family < EVOK_OBJ_KERNEL_SQ || family == EVOK_OBJ_KERNEL_BATCHED) ? 4 : 0) +
         (store && !is_eval_family(family) ? 2 : 0) + (vec ? 1 : 0);
}

// every kernel of an objective's table: the EVOK_OBJ_KERNELS of its first image, the batched samplers of its second, the
// batched evaluation of its third, the transformed evaluation of its fourth
constexpr int kImages = 4;
constexpr int kTableKernels = EVOK_OBJ_KERNEL_TRANSFORM + EVOK_OBJ_TRANSFORM_KERNELS;
static_assert(EVOK_OBJ_KERNEL_BATCHED == EVOK_OBJ_KERNELS, "the batched family follows the first image's kernels");
static_assert(EVOK_OBJ_KERNEL_EVAL_BATCHED == EVOK_OBJ_KERNEL_BATCHED + EVOK_OBJ_BATCHED_KERNELS, "the batched evaluation follows the batched samplers");
static_assert(EVOK_OBJ_KERNEL_TRANSFORM == EVOK_OBJ_KERNEL_EVAL_BATCHED + EVOK_OBJ_EVAL_BATCHED_KERNELS, "the transformed evaluation comes last");

// the first table position and the number of kernels of each image
constexpr int kImageFirst[kImages] = {0, EVOK_OBJ_KERNEL_BATCHED, EVOK_OBJ_KERNEL_EVAL_BATCHED, EVOK_OBJ_KERNEL_TRANSFORM};
constexpr int kImageKernels[kImages] = {EVOK_OBJ_KERNELS, EVOK_OBJ_BATCHED_KERNELS, EVOK_OBJ_EVAL_BATCHED_KERNELS, EVOK_OBJ_TRANSFORM_KERNELS};

static int kernel_threads(int k) {
  return (k >= EVOK_OBJ_KERNEL_EVAL && k < EVOK_OBJ_KERNEL_BATCHED) || k >= EVOK_OBJ_KERNEL_EVAL_BATCHED ? kEvalThreads : kSampleThreads;
}

// the image of a registered objective that holds kernel k: 0 = the one of evok_objective_register, 1 = the batched samplers,
// 2 = the batched evaluation, 3 = the transformed evaluation
static int image_of(int k) {
  return k >= EVOK_OBJ_KERNEL_TRANSFORM ? 3 : k >= EVOK_OBJ_KERNEL_EVAL_BATCHED ? 2 : k >= EVOK_OBJ_KERNEL_BATCHED ? 1 : 0;
}

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

// The batched sampler of built-in objective OBJ with V = sym | store << 1 | vec << 2 (V < 8); EVOK_OBJ_NONE only stores samples.
template <int OBJ, int V>
static void put_builtin_batched(void** fn) {
  constexpr bool sym = V & 1, store = V & 2, vec = V & 4;
  if constexpr (V < EVOK_OBJ_BATCHED_KERNELS && (OBJ != EVOK_OBJ_NONE || store))
    fn[kernel_index(EVOK_OBJ_KERNEL_BATCHED, sym, store, vec)] = reinterpret_cast<void*>(sample_eval_batched_kernel<ObjAcc<OBJ>, sym, store, vec>);
}

template <int OBJ, int... V>
static void put_builtin_kernels(void** fn, std::integer_sequence<int, V...>) {
  (put_builtin_sampler<OBJ, V>(fn), ...);
  (put_builtin_batched<OBJ, V>(fn), ...);
  if constexpr (OBJ != EVOK_OBJ_NONE) {  // evok_eval and evok_eval_batched refuse EVOK_OBJ_NONE
    fn[kernel_index(EVOK_OBJ_KERNEL_EVAL, false, true, false)] = reinterpret_cast<void*>(eval_kernel<ObjAcc<OBJ>, false>);
    fn[kernel_index(EVOK_OBJ_KERNEL_EVAL, false, true, true)] = reinterpret_cast<void*>(eval_kernel<ObjAcc<OBJ>, true>);
    fn[kernel_index(EVOK_OBJ_KERNEL_EVAL_BATCHED, false, true, false)] = reinterpret_cast<void*>(eval_batched_kernel<ObjAcc<OBJ>, false>);
    fn[kernel_index(EVOK_OBJ_KERNEL_EVAL_BATCHED, false, true, true)] = reinterpret_cast<void*>(eval_batched_kernel<ObjAcc<OBJ>, true>);
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
// functions of its modules, loaded into the device's primary context: the first image's on the first use of the id, the
// batched samplers' on the first batched sampling, the batched evaluation's on the first batched evaluation.
struct DeviceKernels {
  int state[kImages] = {};        // per image: 0: not filled; 1: filled; EVOK_E_NOKERNEL: the cubin lacks a kernel (a permanent failure)
  CUmodule module[kImages] = {};  // set for a registered objective: fn holds CUfunctions, launched through the driver
  void* fn[kTableKernels] = {};
  int per_sm[kTableKernels] = {};  // resident CTAs per SM
  int sms = 0;
  int smem_optin = 0;  // shared memory per CTA the fused transformed kernels may take (set with image 3)
};

struct Objective {
  // a registered objective's cubins and the lowered names of their kernels (in the EVOK_OBJ_KERNEL_* order): [0] from
  // evok_objective_register, [1] (the batched samplers, empty until attached) from evok_objective_register_batched, [2] (the
  // batched evaluation, empty until attached) from evok_objective_register_eval_batched; a transformed objective
  // (evok_objective_register_transform) has [3] only
  std::vector<char> image[kImages];
  std::vector<std::string> names[kImages];
  // evok_objective_declare_data: the data names of its accumulator (0: none) and which of them are vectors of the row length
  int n_data = 0;
  bool is_vector[EVOK_MAX_DATA] = {};
  // evok_objective_declare_noise: its accumulator draws noise, and its EVOK_OBJ_KERNEL_EVAL entries take the key
  bool noisy = false;
  DeviceKernels dev[kMaxDevices];
};

// An instance of a registered objective with data (evok_objective_instance): the kernels of `base`, its own binding.
struct Instance {
  int base = -1;  // -1: the slot is free
  const float* p[EVOK_MAX_DATA] = {};
  int64_t len[EVOK_MAX_DATA] = {}, stride[EVOK_MAX_DATA] = {};
  int64_t n_items = 1;
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
  decltype(&cuFuncSetAttribute) func_attribute = nullptr;
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
         driver_symbol("cuLaunchKernel", d.launch) && driver_symbol("cuFuncSetAttribute", d.func_attribute);
}

static std::mutex g_objective_mutex;
static Objective g_builtin[EVOK_OBJ_COUNT];
static Objective* g_user[EVOK_OBJ_USER_CAPACITY];
static std::atomic<int> g_user_count{0};

static std::vector<Instance> g_instances;  // slot i is the id EVOK_OBJ_INSTANCE_BASE + i; guarded by g_objective_mutex
static std::vector<int> g_free_instances;

static bool is_user(int objective) {
  return objective >= EVOK_OBJ_USER_BASE && objective - EVOK_OBJ_USER_BASE < g_user_count.load(std::memory_order_acquire);
}

// the live instance of an id, else null; call with g_objective_mutex held
static const Instance* instance_of(int objective) {
  const int64_t slot = (int64_t)objective - EVOK_OBJ_INSTANCE_BASE;
  return slot >= 0 && slot < (int64_t)g_instances.size() && g_instances[slot].base >= 0 ? &g_instances[slot] : nullptr;
}

// The id whose kernels `objective` launches: the base of a live instance, else `objective` itself (an id that is neither an
// instance nor an objective then fails the enum check of its entry point).
static int base_of(int objective) {
  if (objective < EVOK_OBJ_INSTANCE_BASE) return objective;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const Instance* inst = instance_of(objective);
  return inst ? inst->base : objective;
}

// The data of one call: the kernels' last argument, the id that holds the kernels, and whether every vector allows the 16-byte
// loads of the vectorised kernels (its base 16-byte aligned, its item stride a multiple of 4).
struct LaunchData {
  DataBinding binding{};
  int base = 0;
  bool vec_ok = true;
};

// The data checks of a call with row length D on `items` items (0: an entry point that is not batched), after the entry point's
// own checks: EVOK_E_NODATA for an objective that declares data and is not launched through an instance; EVOK_E_BADSIZE for a
// vector whose length is not D, and for a per-item binding on a non-batched entry or on another number of items.
static int bind_data(int objective, int64_t D, int64_t items, LaunchData* out) {
  out->base = objective;
  if (objective < EVOK_OBJ_USER_BASE) return 0;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const Instance* inst = instance_of(objective);
  if (!inst) return is_user(objective) && g_user[objective - EVOK_OBJ_USER_BASE]->n_data > 0 ? EVOK_E_NODATA : 0;
  const Objective& obj = *g_user[inst->base - EVOK_OBJ_USER_BASE];
  out->base = inst->base;
  if (inst->n_items > 1 && items != inst->n_items) return EVOK_E_BADSIZE;
  for (int i = 0; i < obj.n_data; ++i) {
    const int64_t stride = inst->n_items > 1 ? inst->stride[i] : 0;
    if (obj.is_vector[i]) {
      if (inst->len[i] != D) return EVOK_E_BADSIZE;
      if (!aligned16(inst->p[i]) || stride % 4 != 0) out->vec_ok = false;
    }
    out->binding.p[i] = inst->p[i];
    out->binding.item_stride[i] = stride;
  }
  return 0;
}

// true for a registered id (a base, not an instance) that declares noise
static bool is_noisy(int base) {
  if (!is_user(base)) return false;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  return g_user[base - EVOK_OBJ_USER_BASE]->noisy;
}

static void fill_builtin(int objective, int dev, DeviceKernels& d) {
  kBuiltinKernels[objective](d.fn);
  for (int k = 0; k < kTableKernels; ++k)
    if (d.fn[k] && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.per_sm[k], d.fn[k], kernel_threads(k), 0) != cudaSuccess || d.per_sm[k] <= 0))
      d.per_sm[k] = 4;
  if (cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.sms <= 0) d.sms = kNumSMs;
  for (int part = 0; part < kImages; ++part) d.state[part] = 1;
}

// Loads image `part` of a registered objective on device `dev` into its table positions (kImageKernels[part] kernels from
// kImageFirst[part]).
static int load_module(const Objective& obj, int part, int dev, DeviceKernels& d) {
  cudaError_t ce = cudaSetDevice(dev);  // makes the device's primary context (the runtime's) current, creating it if needed
  if (ce != cudaSuccess) return (int)ce;
  if (!driver_api()) return (int)cudaErrorNotSupported;
  const DriverApi& api = g_driver;
  CUdevice cu_dev;
  CUresult r = api.device_get(&cu_dev, dev);
  if (r == CUDA_SUCCESS) r = api.device_attribute(&d.sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, cu_dev);
  if (r == CUDA_SUCCESS) r = api.module_load(&d.module[part], obj.image[part].data());
  if (r != CUDA_SUCCESS) return (int)r;  // CUresult and cudaError_t share their codes
  const int k0 = kImageFirst[part];
  const int n = kImageKernels[part];
  for (int i = 0; i < n; ++i) {
    const int k = k0 + i;
    CUfunction fn = nullptr;
    if (api.module_function(&fn, d.module[part], obj.names[part][i].c_str()) != CUDA_SUCCESS) {
      api.module_unload(d.module[part]);
      d.module[part] = nullptr;
      d.state[part] = EVOK_E_NOKERNEL;
      return d.state[part];
    }
    d.fn[k] = fn;
    if (api.occupancy(&d.per_sm[k], fn, kernel_threads(k), 0) != CUDA_SUCCESS || d.per_sm[k] <= 0) d.per_sm[k] = 4;
  }
  if (part == 3) {  // the fused transformed kernels may take the device's opt-in shared memory per CTA
    if (api.device_attribute(&d.smem_optin, CU_DEVICE_ATTRIBUTE_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN, cu_dev) != CUDA_SUCCESS) d.smem_optin = 48 * 1024;
    for (int v = 0; v < 2; ++v)
      api.func_attribute(static_cast<CUfunction>(d.fn[EVOK_OBJ_KERNEL_TRANSFORM + v]), CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, d.smem_optin);
  }
  if (d.sms <= 0) d.sms = kNumSMs;
  d.state[part] = 1;
  return 0;
}

// The kernel table of an objective (a built-in id or a registered one) on the current device, with the kernels of image `part`
// (image_of) filled here on the first call that needs them on that device.  A registered id without image `part` (1 or 2) gives
// EVOK_E_NOKERNEL (not kept: the image may be attached later).
static int device_kernels(int objective, int part, const DeviceKernels** out) {
  int dev = 0;
  const cudaError_t ce = cudaGetDevice(&dev);
  if (ce != cudaSuccess) return (int)ce;
  if (dev < 0 || dev >= kMaxDevices) return EVOK_E_BADSIZE;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const bool user = objective >= EVOK_OBJ_USER_BASE;
  Objective& obj = user ? *g_user[objective - EVOK_OBJ_USER_BASE] : g_builtin[objective];
  DeviceKernels& d = obj.dev[dev];
  if (d.state[part] == 0) {
    if (!user) fill_builtin(objective, dev, d);
    else if (obj.image[part].empty()) return EVOK_E_NOKERNEL;
    else if (const int rc = load_module(obj, part, dev, d)) return rc;
  }
  if (d.state[part] != 1) return d.state[part];
  *out = &d;
  return 0;
}

struct KernelChoice {
  int k;                // index in the EVOK_OBJ_KERNEL_* order
  int64_t n_units;      // rows, or antithetic row pairs for symmetric sampling; one warp each (per item)
  int64_t ctas_needed;  // CTAs that give every unit of an item its own warp
};

// The kernel of a call: family (EVOK_OBJ_KERNEL_*) and sym; stored samples when X is given; the vectorised variant when
// D % 4 == 0 and every operand read or written with float4 loads / stores is 16-byte aligned with 16-byte aligned rows (mu and
// sigma are null for the evaluation kernel, which reads X only) in every item: `item_strides` is the bitwise OR of the item
// strides of the batched family (0 for one item), a multiple of 4 when each of them is.  The data vectors of an objective are
// such operands too (data.vec_ok): one that is not aligned sends the whole call to the scalar-column kernels.
static KernelChoice choose_kernel(int family, bool sym, const float* X, int64_t ldx, const float* mu, const float* sigma, int64_t n_rows,
                                  int64_t D, const LaunchData& data, int64_t item_strides = 0) {
  const bool store = X != nullptr;
  const bool vec = (D % 4 == 0) && aligned16(mu) && aligned16(sigma) && (!store || (aligned16(X) && ldx % 4 == 0)) && item_strides % 4 == 0 &&
                   data.vec_ok;
  KernelChoice c;
  c.k = kernel_index(family, sym, store, vec);
  c.n_units = sym ? n_rows / 2 : n_rows;
  const int warps = kernel_threads(c.k) / 32;
  c.ctas_needed = (c.n_units + warps - 1) / warps;
  return c;
}

// Launches kernel c.k of an objective on the current device with `args` in the kernel's parameter order (the last one is the
// data binding, which a kernel without data terms takes as an empty struct), for `items` items
// (grid y, at most kMaxGridY), on as many CTAs per item as stay resident when the items share the device, but no more than the
// units need, and at least one (the push sampler with no rows still raises this rank's flag).  A built-in kernel goes through
// the runtime, a registered one through the driver.
static int launch(int objective, const KernelChoice& c, void** args, cudaStream_t st, int64_t items = 1) {
  const DeviceKernels* d = nullptr;
  const int rc = device_kernels(objective, image_of(c.k), &d);
  if (rc != 0) return rc;
  int64_t g = (int64_t)d->per_sm[c.k] * d->sms / items;
  if (g > c.ctas_needed) g = c.ctas_needed;
  if (g < 1) g = 1;
  const int threads = kernel_threads(c.k);
  if (d->module[image_of(c.k)]) {
    const CUresult r = g_driver.launch(static_cast<CUfunction>(d->fn[c.k]), (unsigned)g, (unsigned)items, 1, threads, 1, 1, 0, (CUstream)st, args,
                                       nullptr);
    if (r != CUDA_SUCCESS) return (int)r;
    count_launches(1);
    return 0;
  }
  cudaLaunchKernel(d->fn[c.k], dim3((unsigned)g, (unsigned)items), dim3(threads), args, 0, st);
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
  LaunchData data;
  if (const int rc = bind_data(objective, D, 0, &data)) return rc;
  KernelChoice c = choose_kernel(family, sym, X, ldx, mu, sigma, n_rows, D, data);
  PhiloxKey key = make_philox_key(seed, stream_id);
  void* args[] = {&X, &ldx, &mu, &sigma, &row0, &c.n_units, &D, &key, &stream_off, &f, &push.sink, &push.epoch, &push.done, &q, &data.binding};
  return launch(data.base, c, args, st);
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
  obj->image[0].assign(static_cast<const char*>(cubin), static_cast<const char*>(cubin) + bytes);
  for (int k = 0; k < n_kernels; ++k) obj->names[0].emplace_back(kernel_names_host[k]);
  g_user[n] = obj;
  g_user_count.store(n + 1, std::memory_order_release);
  *id_out_host = EVOK_OBJ_USER_BASE + n;
  return 0;
}

extern "C" EVOK_API int evok_objective_load(int objective) {
  objective = base_of(objective);
  if (!is_user(objective)) return EVOK_E_BADENUM;
  const DeviceKernels* d = nullptr;
  return device_kernels(objective, 0, &d);
}

// evok_objective_register_batched (part 1) and evok_objective_register_eval_batched (part 2): attach image `part` of a registered id
static int attach_image(int objective, int part, const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels) {
  if (!cubin || !kernel_names_host) return EVOK_E_NULLPTR;
  if (bytes == 0 || n_kernels != kImageKernels[part]) return EVOK_E_BADSIZE;
  for (int k = 0; k < n_kernels; ++k)
    if (!kernel_names_host[k]) return EVOK_E_NULLPTR;
  if (!is_user(objective)) return EVOK_E_BADENUM;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  Objective& obj = *g_user[objective - EVOK_OBJ_USER_BASE];
  obj.image[part].assign(static_cast<const char*>(cubin), static_cast<const char*>(cubin) + bytes);
  obj.names[part].assign(kernel_names_host, kernel_names_host + n_kernels);
  return 0;
}

extern "C" EVOK_API int evok_objective_register_batched(int objective, const void* cubin, size_t bytes, const char* const* kernel_names_host,
                                                        int n_kernels) {
  return attach_image(objective, 1, cubin, bytes, kernel_names_host, n_kernels);
}

extern "C" EVOK_API int evok_objective_register_eval_batched(int objective, const void* cubin, size_t bytes, const char* const* kernel_names_host,
                                                             int n_kernels) {
  return attach_image(objective, 2, cubin, bytes, kernel_names_host, n_kernels);
}

extern "C" EVOK_API int evok_objective_declare_data(int objective, int n_data, const int* is_vector_host) {
  if (!is_vector_host) return EVOK_E_NULLPTR;
  if (!is_user(objective)) return EVOK_E_BADENUM;
  if (n_data < 1 || n_data > EVOK_MAX_DATA) return EVOK_E_BADSIZE;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  Objective& obj = *g_user[objective - EVOK_OBJ_USER_BASE];
  if (obj.n_data != 0) return EVOK_E_BADSIZE;
  obj.n_data = n_data;
  for (int i = 0; i < n_data; ++i) obj.is_vector[i] = is_vector_host[i] != 0;
  return 0;
}

extern "C" EVOK_API int evok_objective_declare_noise(int objective) {
  if (!is_user(objective)) return EVOK_E_BADENUM;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  g_user[objective - EVOK_OBJ_USER_BASE]->noisy = true;
  return 0;
}

extern "C" EVOK_API int evok_objective_instance(int base, const float* const* ptrs_host, const int64_t* lens_host, const int64_t* item_strides_host,
                                                int64_t n_items, int n_data, int* id_out_host) {
  if (!ptrs_host || !lens_host || !item_strides_host || !id_out_host) return EVOK_E_NULLPTR;
  if (!is_user(base)) return EVOK_E_BADENUM;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const Objective& obj = *g_user[base - EVOK_OBJ_USER_BASE];
  if (obj.n_data == 0) return EVOK_E_NODATA;
  if (n_data != obj.n_data || n_items < 1) return EVOK_E_BADSIZE;
  Instance inst;
  for (int i = 0; i < n_data; ++i) {
    if (!ptrs_host[i]) return EVOK_E_NULLPTR;
    if (lens_host[i] < 1 || (lens_host[i] == 1) == obj.is_vector[i] || item_strides_host[i] < 0) return EVOK_E_BADSIZE;
    inst.p[i] = ptrs_host[i];
    inst.len[i] = lens_host[i];
    inst.stride[i] = item_strides_host[i];
  }
  inst.base = base;
  inst.n_items = n_items;
  int slot;
  if (!g_free_instances.empty()) {
    slot = g_free_instances.back();
    g_free_instances.pop_back();
  } else {
    if (g_instances.size() >= EVOK_OBJ_INSTANCE_CAPACITY) return EVOK_E_BADSIZE;
    slot = (int)g_instances.size();
    g_instances.emplace_back();
  }
  g_instances[slot] = inst;
  *id_out_host = EVOK_OBJ_INSTANCE_BASE + slot;
  return 0;
}

extern "C" EVOK_API int evok_objective_release(int id) {
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  if (!instance_of(id)) return EVOK_E_BADENUM;
  g_instances[id - EVOK_OBJ_INSTANCE_BASE] = Instance{};
  g_free_instances.push_back(id - EVOK_OBJ_INSTANCE_BASE);
  return 0;
}

extern "C" EVOK_API int evok_sample_eval(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0,
                                int64_t n_rows, int64_t D, int symmetric, uint64_t seed, uint64_t stream_id,
                                const uint32_t* stream_offset_dev, float* f, void* stream) {
  const int rc = check_sample(base_of(objective), X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, f, nullptr);
  if (rc != 0 || n_rows == 0) return rc;
  return sample(objective, EVOK_OBJ_KERNEL_SAMPLE, X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, seed, stream_id, stream_offset_dev, f,
                nullptr, PushArgs{}, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_sample_eval_sq(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                                            int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float* f, float* q,
                                            void* stream) {
  if (!q) return EVOK_E_NULLPTR;
  const int rc = check_sample(base_of(objective), X, ldx, mu, sigma, row0, n_rows, D, false, f, nullptr);
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
  const int rc = check_sample(base_of(objective), X, ldx, mu, sigma, row0, n_rows, D, symmetric != 0, nullptr, &push);
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

// evok_eval (keyed = false) and evok_eval_keyed.  The evaluation kernel's last argument is the draw of the rows (EvalKey) for
// an objective with noise, an empty struct (which takes its one byte from `noise`) for every other.
static int eval_call(int objective, const float* X, int64_t ldx, int64_t row0, int64_t n_rows, int64_t D, bool keyed, uint64_t seed,
                     uint64_t stream_id, const uint32_t* stream_off, float* f, cudaStream_t st) {
  if (!X || !f) return EVOK_E_NULLPTR;
  const int base = base_of(objective);
  if ((base <= EVOK_OBJ_NONE || base >= EVOK_OBJ_COUNT) && !is_user(base)) return EVOK_E_BADENUM;
  if (n_rows < 0 || D <= 0 || ldx < D || row0 < 0) return EVOK_E_BADSIZE;
  const bool noisy = is_noisy(base);
  if (noisy && !keyed) return EVOK_E_NOISEKEY;
  if (n_rows == 0) return 0;
  LaunchData data;
  if (const int rc = bind_data(objective, D, 0, &data)) return rc;
  const KernelChoice c = choose_kernel(EVOK_OBJ_KERNEL_EVAL, false, X, ldx, nullptr, nullptr, n_rows, D, data);
  EvalKey noise{noisy ? make_philox_key(seed, stream_id) : PhiloxKey{}, stream_off, row0};
  void* args[] = {&X, &ldx, &n_rows, &D, &f, &data.binding, &noise};
  return launch(data.base, c, args, st);
}

extern "C" EVOK_API int evok_eval(int objective, const float* X, int64_t ldx, int64_t n_rows, int64_t D, float* f, void* stream) {
  return eval_call(objective, X, ldx, 0, n_rows, D, false, 0, 0, nullptr, f, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_eval_keyed(int objective, const float* X, int64_t ldx, int64_t row0, int64_t n_rows, int64_t D, uint64_t seed,
                                        uint64_t stream_id, const uint32_t* stream_offset_dev, float* f, void* stream) {
  return eval_call(objective, X, ldx, row0, n_rows, D, true, seed, stream_id, stream_offset_dev, f, (cudaStream_t)stream);
}

// One launch per item chunk of the batched family: item b of the batch samples with stream word (stream_id0 + b), chunk b0 of
// at most kMaxGridY items (grid y) starting at stream word stream_lo + b0 and at item b0 of X, mu, sigma and the objective's
// data; f (null for EVOK_OBJ_NONE) is [items][n_rows].
static int sample_items(int objective, float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu, const float* sigma,
                        int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, bool sym, uint64_t seed, uint64_t stream_id0, float* f,
                        cudaStream_t st) {
  LaunchData data;
  if (const int rc = bind_data(objective, D, n_items, &data)) return rc;
  KernelChoice c = choose_kernel(EVOK_OBJ_KERNEL_BATCHED, sym, X, ldx, mu, sigma, n_rows, D, data,
                                 (X ? item_stride_x : 0) | item_stride_mu | item_stride_sigma);
  const PhiloxKey key = make_philox_key(seed, stream_id0);
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    PhiloxKey kc = key;
    kc.stream_lo += (uint32_t)b0;
    float* Xc = X ? X + b0 * item_stride_x : nullptr;
    const float* muc = mu + b0 * item_stride_mu;
    const float* sgc = sigma + b0 * item_stride_sigma;
    float* fc = f ? f + b0 * n_rows : nullptr;
    DataBinding dc = data.binding;
    for (int i = 0; i < EVOK_MAX_DATA; ++i) dc.p[i] += b0 * dc.item_stride[i];
    void* args[] = {&Xc, &item_stride_x, &ldx, &muc, &item_stride_mu, &sgc, &item_stride_sigma, &c.n_units, &D, &kc, &fc, &dc};
    return launch(data.base, c, args, st, nb);
  });
}

extern "C" EVOK_API int evok_sample_batched(float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu, const float* sigma,
                                            int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, int symmetric, uint64_t seed,
                                            uint64_t stream_id0, void* stream) {
  if (!X || !mu || !sigma) return EVOK_E_NULLPTR;
  if (n_items < 0 || n_rows < 0 || D <= 0 || ldx < D || item_stride_x < 0 || item_stride_mu < 0 || item_stride_sigma < 0)
    return EVOK_E_BADSIZE;
  if (symmetric && (n_rows & 1)) return EVOK_E_ODDROWS;
  if (n_items == 0 || n_rows == 0) return 0;
  return sample_items(EVOK_OBJ_NONE, X, item_stride_x, ldx, mu, item_stride_mu, sigma, item_stride_sigma, n_items, n_rows, D, symmetric != 0, seed,
                      stream_id0, nullptr, (cudaStream_t)stream);
}

// The argument checks of evok_sample_eval_batched, in the order of include/evok.h.
static int check_sample_batched(int objective, const float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu,
                                const float* sigma, int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, bool sym, const float* f) {
  if (!mu || !sigma || !f) return EVOK_E_NULLPTR;
  if ((objective <= EVOK_OBJ_NONE || objective >= EVOK_OBJ_COUNT) && !is_user(objective)) return EVOK_E_BADENUM;
  if (n_items < 0 || n_rows < 0 || D <= 0 || (X && (ldx < D || item_stride_x < 0)) || item_stride_mu < 0 || item_stride_sigma < 0)
    return EVOK_E_BADSIZE;
  if (sym && (n_rows & 1)) return EVOK_E_ODDROWS;
  if (is_user(objective)) {  // a registered id samples batched only with its batched image: nothing is launched without it
    std::lock_guard<std::mutex> lock(g_objective_mutex);
    if (g_user[objective - EVOK_OBJ_USER_BASE]->image[1].empty()) return EVOK_E_NOKERNEL;
  }
  return 0;
}

extern "C" EVOK_API int evok_sample_eval_batched(int objective, float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu,
                                                 const float* sigma, int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D,
                                                 int symmetric, uint64_t seed, uint64_t stream_id0, float* f, void* stream) {
  const int rc = check_sample_batched(base_of(objective), X, item_stride_x, ldx, mu, item_stride_mu, sigma, item_stride_sigma, n_items, n_rows, D,
                                      symmetric != 0, f);
  if (rc != 0 || n_items == 0 || n_rows == 0) return rc;
  return sample_items(objective, X, item_stride_x, ldx, mu, item_stride_mu, sigma, item_stride_sigma, n_items, n_rows, D, symmetric != 0, seed,
                      stream_id0, f, (cudaStream_t)stream);
}

// true for a registered id (a base) without image `part`: its calls of that family launch nothing (EVOK_E_NOKERNEL)
static bool lacks_image(int base, int part) {
  if (!is_user(base)) return false;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  return g_user[base - EVOK_OBJ_USER_BASE]->image[part].empty();
}

// true for an instance id whose binding has per-item data for another number of items than n_items
static bool items_differ(int objective, int64_t n_items) {
  if (objective < EVOK_OBJ_INSTANCE_BASE) return false;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const Instance* inst = instance_of(objective);
  return inst && inst->n_items > 1 && inst->n_items != n_items;
}

extern "C" EVOK_API int evok_eval_batched(int objective, const float* X, int64_t item_stride_x, int64_t ldx, int64_t n_items, int64_t n_rows,
                                          int64_t D, uint64_t seed, uint64_t stream_id0, float* f, void* stream) {
  if (!X || !f) return EVOK_E_NULLPTR;
  const int base = base_of(objective);
  if ((base <= EVOK_OBJ_NONE || base >= EVOK_OBJ_COUNT) && !is_user(base)) return EVOK_E_BADENUM;
  if (n_items < 0 || n_rows < 0 || item_stride_x < 0 || D <= 0 || ldx < D || items_differ(objective, n_items)) return EVOK_E_BADSIZE;
  if (lacks_image(base, 2)) return EVOK_E_NOKERNEL;
  LaunchData data;
  if (const int rc = bind_data(objective, D, n_items, &data)) return rc;
  if (n_items == 0 || n_rows == 0) return 0;
  const KernelChoice c = choose_kernel(EVOK_OBJ_KERNEL_EVAL_BATCHED, false, X, ldx, nullptr, nullptr, n_rows, D, data, item_stride_x);
  // one key for all items: item b draws its noise on stream word (stream_id0 + b), chunk b0 from stream_lo + b0
  const EvalKey noise{is_noisy(base) ? make_philox_key(seed, stream_id0) : PhiloxKey{}, nullptr, 0};
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    EvalKey kc = noise;
    kc.key.stream_lo += (uint32_t)b0;
    const float* Xc = X + b0 * item_stride_x;
    float* fc = f + b0 * n_rows;
    DataBinding dc = data.binding;
    for (int i = 0; i < EVOK_MAX_DATA; ++i) dc.p[i] += b0 * dc.item_stride[i];
    void* args[] = {&Xc, &item_stride_x, &ldx, &n_rows, &D, &fc, &dc, &kc};
    return launch(data.base, c, args, (cudaStream_t)stream, nb);
  });
}

// ------------------------------------------------------------------------------------------------
// Transformed evaluation (evok_eval_transform_batched): the terms read y = M (x - o) per item.  Up to EVOK_TRANSFORM_FUSED_MAX_D
// columns one fused launch per 65535 items computes y on the CUDA cores in shared memory (eval_transform_fused_kernel); above it
// each item chunk is a fixed number of launches: x - o into the workspace (transform_center_kernel), the batched 3xTF32 GEMM
// (evok_gemm_nt_batched) writes y next to it, and eval_transform_kernel folds the x and y rows.
// ------------------------------------------------------------------------------------------------
// The cutoff: both paths timed at the same D on the H100 (scripts/transformed_cutoff_sweep.py, DESIGN.md) cross between D = 96
// and 112 at 1024 items.  Its upper end is the shared memory of one CTA (M and two rows), D = 236; the sweep builds 0 and 236.
#ifndef EVOK_TRANSFORM_FUSED_MAX_D
#define EVOK_TRANSFORM_FUSED_MAX_D 96
#endif
static_assert(EVOK_TRANSFORM_FUSED_MAX_D >= 0 && evok::transform_smem_floats(EVOK_TRANSFORM_FUSED_MAX_D, 2) * 4 <= 227 * 1024,
              "the fused transformed kernel stages M in the 227 KB of shared memory a CTA can take on sm_90");

namespace evok {

constexpr int64_t kTransformTileRows = 32;                  // rows of one fused tile at most (even)
constexpr size_t kTransformChunkBytes = size_t(256) << 20;  // x - o and y of one item chunk on the GEMM path, at most (>= one item)

// out[b][r][k] = X[b][r][k] - o[b][k] for the n_rows x D rows of item b = blockIdx.y (out: item pitch n_rows * ld, row pitch ld)
__global__ void transform_center_kernel(const float* __restrict__ X, int64_t item_stride_x, int64_t ldx, const float* __restrict__ o,
                                        int64_t item_stride_o, int64_t n_rows, int64_t D, float* __restrict__ out, int64_t ld) {
  const int64_t item = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows * D) return;
  const int64_t r = i / D, k = i - r * D;
  out[(item * n_rows + r) * ld + k] = X[item * item_stride_x + r * ldx + k] - __ldg(o + item * item_stride_o + k);
}

static bool transform_fused(int64_t D) { return D <= EVOK_TRANSFORM_FUSED_MAX_D; }

// the items of one chunk of the GEMM path: as many as keep x - o and y within kTransformChunkBytes, at least 1, at most kMaxGridY
static int64_t transform_chunk(int64_t n_items, int64_t n_rows, int64_t D) {
  const int64_t per_item = 2 * n_rows * round4(D) * (int64_t)sizeof(float);
  int64_t c = (int64_t)kTransformChunkBytes / per_item;
  if (c > n_items) c = n_items;
  if (c > kMaxGridY) c = kMaxGridY;
  return c < 1 ? 1 : c;
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// the workspace of a call: none on the fused path; x - o and y of one chunk, then the GEMM's own workspace, on the GEMM path
static size_t transform_ws(const float* M, int64_t item_stride_m, int64_t n_items, int64_t n_rows, int64_t D) {
  if (transform_fused(D) || n_items <= 0 || n_rows <= 0 || D <= 0) return 0;
  const int64_t chunk = transform_chunk(n_items, n_rows, D), ld = round4(D);
  const size_t half = align256((size_t)(chunk * n_rows * ld) * sizeof(float));
  const float* xo = reinterpret_cast<const float*>(uintptr_t(256));  // where x - o goes: 256-byte aligned, row pitch ld
  return 256 + 2 * half + evok_gemm_nt_batched_workspace_bytes(xo, ld, n_rows * ld, M, D, item_stride_m, chunk, n_rows, D, D);
}

}  // namespace evok

extern "C" EVOK_API int evok_objective_register_transform(const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels,
                                                          int* id_out_host) {
  if (!cubin || !kernel_names_host || !id_out_host) return EVOK_E_NULLPTR;
  if (bytes == 0 || n_kernels != EVOK_OBJ_TRANSFORM_KERNELS) return EVOK_E_BADSIZE;
  for (int k = 0; k < n_kernels; ++k)
    if (!kernel_names_host[k]) return EVOK_E_NULLPTR;
  std::lock_guard<std::mutex> lock(g_objective_mutex);
  const int n = g_user_count.load(std::memory_order_relaxed);
  if (n >= EVOK_OBJ_USER_CAPACITY) return EVOK_E_BADSIZE;
  Objective* obj = new Objective;
  obj->image[3].assign(static_cast<const char*>(cubin), static_cast<const char*>(cubin) + bytes);
  obj->names[3].assign(kernel_names_host, kernel_names_host + n_kernels);
  g_user[n] = obj;
  g_user_count.store(n + 1, std::memory_order_release);
  *id_out_host = EVOK_OBJ_USER_BASE + n;
  return 0;
}

extern "C" EVOK_API size_t evok_eval_transform_workspace_bytes(const float* M, int64_t item_stride_m, int64_t n_items, int64_t n_rows, int64_t D) {
  return transform_ws(M, item_stride_m, n_items, n_rows, D);
}

extern "C" EVOK_API int evok_eval_transform_batched(int objective, const float* X, int64_t item_stride_x, int64_t ldx, const float* M,
                                                    int64_t item_stride_m, const float* o, int64_t item_stride_o, int64_t n_items, int64_t n_rows,
                                                    int64_t D, uint64_t seed, uint64_t stream_id0, void* ws, size_t ws_bytes, float* f,
                                                    void* stream) {
  if (!X || !M || !o || !f) return EVOK_E_NULLPTR;
  const int base = base_of(objective);
  if ((base <= EVOK_OBJ_NONE || base >= EVOK_OBJ_COUNT) && !is_user(base)) return EVOK_E_BADENUM;
  if (n_items < 0 || n_rows < 0 || item_stride_x < 0 || item_stride_m < 0 || item_stride_o < 0 || D <= 0 || ldx < D ||
      items_differ(objective, n_items))
    return EVOK_E_BADSIZE;
  if (!is_user(base) || lacks_image(base, 3)) return EVOK_E_NOKERNEL;
  LaunchData data;
  if (const int rc = bind_data(objective, D, n_items, &data)) return rc;
  if (n_items == 0 || n_rows == 0) return 0;
  const size_t need = transform_ws(M, item_stride_m, n_items, n_rows, D);
  if (need > 0 && !ws) return EVOK_E_NULLPTR;
  if (ws_bytes < need) return EVOK_E_BADSIZE;
  const DeviceKernels* d = nullptr;
  if (const int rc = device_kernels(data.base, 3, &d)) return rc;
  const bool vec = D % 4 == 0 && aligned16(X) && ldx % 4 == 0 && item_stride_x % 4 == 0 && data.vec_ok;
  // one key for all items: item b draws its noise on stream word (stream_id0 + b), chunk b0 from stream_lo + b0
  const EvalKey noise{is_noisy(base) ? make_philox_key(seed, stream_id0) : PhiloxKey{}, nullptr, 0};
  const cudaStream_t st = (cudaStream_t)stream;
  auto chunk_args = [&](int64_t b0, EvalKey& kc, const float*& Xc, float*& fc, DataBinding& dc) {
    kc = noise;
    kc.key.stream_lo += (uint32_t)b0;
    Xc = X + b0 * item_stride_x;
    fc = f + b0 * n_rows;
    dc = data.binding;
    for (int i = 0; i < EVOK_MAX_DATA; ++i) dc.p[i] += b0 * dc.item_stride[i];
  };
  if (transform_fused(D)) {
    const CUfunction fn = static_cast<CUfunction>(d->fn[EVOK_OBJ_KERNEL_TRANSFORM + (vec ? 1 : 0)]);
    int64_t tile = n_rows + (n_rows & 1) < kTransformTileRows ? n_rows + (n_rows & 1) : kTransformTileRows;
    while (tile > 2 && transform_smem_floats(D, tile) * (int64_t)sizeof(float) > d->smem_optin) tile -= 2;
    const size_t smem = (size_t)transform_smem_floats(D, tile) * sizeof(float);
    if (smem > (size_t)d->smem_optin) return EVOK_E_BADSIZE;
    int per_sm = 0;
    if (g_driver.occupancy(&per_sm, fn, kEvalThreads, smem) != CUDA_SUCCESS || per_sm <= 0) per_sm = 1;
    const int64_t tiles = (n_rows + tile - 1) / tile;
    return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
      EvalKey kc;
      const float* Xc;
      float* fc;
      DataBinding dc;
      chunk_args(b0, kc, Xc, fc, dc);
      const float* Mc = M + b0 * item_stride_m;
      const float* oc = o + b0 * item_stride_o;
      int64_t g = (int64_t)per_sm * d->sms / nb;
      if (g > tiles) g = tiles;
      if (g < 1) g = 1;
      void* args[] = {&Xc, &item_stride_x, &ldx, &Mc, &item_stride_m, &oc, &item_stride_o, &n_rows, &D, &tile, &fc, &dc, &kc};
      const CUresult r = g_driver.launch(fn, (unsigned)g, (unsigned)nb, 1, kEvalThreads, 1, 1, (unsigned)smem, (CUstream)st, args, nullptr);
      if (r != CUDA_SUCCESS) return (int)r;
      count_launches(1);
      return 0;
    });
  }
  const int k = EVOK_OBJ_KERNEL_TRANSFORM + 2 + (vec ? 1 : 0);
  const CUfunction fn = static_cast<CUfunction>(d->fn[k]);
  int64_t ld = round4(D), item_stride_y = n_rows * ld;
  const int64_t chunk = transform_chunk(n_items, n_rows, D);
  char* w = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  const size_t half = align256((size_t)(chunk * n_rows * ld) * sizeof(float));
  float* xo = reinterpret_cast<float*>(w);
  const float* Y = reinterpret_cast<const float*>(w + half);
  void* gws = w + 2 * half;
  const size_t gws_bytes = ws_bytes - (size_t)(static_cast<char*>(gws) - static_cast<char*>(ws));
  const int64_t ctas_needed = (n_rows + kEvalThreads / 32 - 1) / (kEvalThreads / 32);
  return for_item_chunks(n_items, chunk, [&](int64_t b0, int64_t nb) {
    EvalKey kc;
    const float* Xc;
    float* fc;
    DataBinding dc;
    chunk_args(b0, kc, Xc, fc, dc);
    transform_center_kernel<<<dim3((unsigned)((n_rows * D + 255) / 256), (unsigned)nb), 256, 0, st>>>(Xc, item_stride_x, ldx, o + b0 * item_stride_o,
                                                                                                        item_stride_o, n_rows, D, xo, ld);
    EVOK_CHECK_LAUNCH();
    if (const int rc = evok_gemm_nt_batched(xo, ld, item_stride_y, M + b0 * item_stride_m, D, item_stride_m, nb, n_rows, D, D, const_cast<float*>(Y), ld,
                                            item_stride_y, nullptr, 0, 0, nullptr, 0, nullptr, 0, gws, gws_bytes, st))
      return rc;
    int64_t g = (int64_t)d->per_sm[k] * d->sms / nb;
    if (g > ctas_needed) g = ctas_needed;
    if (g < 1) g = 1;
    void* args[] = {&Xc, &item_stride_x, &ldx, &Y, &item_stride_y, &ld, &n_rows, &D, &fc, &dc, &kc};
    const CUresult r = g_driver.launch(fn, (unsigned)g, (unsigned)nb, 1, kEvalThreads, 1, 1, 0, (CUstream)st, args, nullptr);
    if (r != CUDA_SUCCESS) return (int)r;
    count_launches(1);
    return 0;
  });
}
