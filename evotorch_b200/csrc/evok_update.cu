// K5: D-vector parameter updates.  These are launch-latency bound (D floats); each is ONE single-CTA kernel that
// reduces the norms it needs on the device (no host synchronisation, unlike optimizers.py:313 in the reference) so
// a whole generation stays CUDA-graph capturable.
#include "evok_common.cuh"

namespace evok {

unsigned long long g_launch_count = 0;

constexpr int kUpdThreads = 1024;

// ClipUp on one D-vector, by one CTA of kUpdThreads; store(i, step) writes step i where the caller wants it
template <typename Store>
__device__ __forceinline__ void clipup(const float* __restrict__ g, int64_t D, float* __restrict__ velocity, float stepsize, float momentum,
                                       float max_speed, Store store) {
  __shared__ double sm[33];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < D; i += kUpdThreads) {
    const double v = (double)g[i];
    acc += v * v;
  }
  const float gnorm = (float)sqrt(block_sum<double>(acc, sm));
  // v' = momentum * v + (g / ||g||) * stepsize      (optimizers.py:348-350)
  acc = 0.0;
  for (int64_t i = threadIdx.x; i < D; i += kUpdThreads) {
    const float nv = momentum * velocity[i] + __fdiv_rn(g[i], gnorm) * stepsize;
    velocity[i] = nv;
    acc += (double)nv * (double)nv;
  }
  const float vnorm = (float)sqrt(block_sum<double>(acc, sm));
  const bool clip = vnorm > max_speed;  // optimizers.py:313
  const float ratio = clip ? __fdiv_rn(max_speed, vnorm) : 1.0f;
  for (int64_t i = threadIdx.x; i < D; i += kUpdThreads) {
    float nv = velocity[i];
    if (clip) {
      nv *= ratio;
      velocity[i] = nv;
    }
    store(i, nv);
  }
}

__global__ void __launch_bounds__(kUpdThreads) clipup_kernel(const float* __restrict__ g, int64_t D, float* __restrict__ velocity,
                                                             float stepsize, float momentum, float max_speed, float* __restrict__ step_out,
                                                             float* __restrict__ mu) {
  clipup(g, D, velocity, stepsize, momentum, max_speed, [&](int64_t i, float nv) {
    if (step_out) step_out[i] = nv;
    if (mu) mu[i] += nv;
  });
}

__global__ void __launch_bounds__(256) adam_kernel(const float* __restrict__ g, int64_t D, float* __restrict__ m, float* __restrict__ v,
                                                   float b1, float b2, float step_size, float inv_sqrt_bc2, float eps,
                                                   float* __restrict__ step_out, float* __restrict__ mu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  const float gi = g[i];
  const float mi = b1 * m[i] + (1.0f - b1) * gi;
  const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) * inv_sqrt_bc2 + eps;
  const float s = step_size * __fdiv_rn(mi, denom);
  if (step_out) step_out[i] = s;
  if (mu) mu[i] += s;
}

__global__ void __launch_bounds__(256) sgd_kernel(const float* __restrict__ g, int64_t D, float* __restrict__ buf, int first_step, float lr,
                                                  float momentum, float* __restrict__ step_out, float* __restrict__ mu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  float d = g[i];
  if (momentum != 0.0f && buf) {
    d = first_step ? d : momentum * buf[i] + d;
    buf[i] = d;
  }
  const float s = lr * d;
  if (step_out) step_out[i] = s;
  if (mu) mu[i] += s;
}

__global__ void __launch_bounds__(256) axpy_kernel(const float* __restrict__ g, int64_t D, float lr, float* __restrict__ mu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D) mu[i] += lr * g[i];
}

// torch.max / torch.min: NaN if either operand is NaN (fmaxf / fminf would return the other one)
__device__ __forceinline__ float torch_max(float a, float b) { return (a != a || b != b) ? NAN : fmaxf(a, b); }
__device__ __forceinline__ float torch_min(float a, float b) { return (a != a || b != b) ? NAN : fminf(a, b); }

// modify_tensor (tools/misc.py) on one element: every operand the caller supplied takes part in torch.max / torch.min, so a NaN
// target, a NaN bound or a NaN allowed change (|0| * inf) gives NaN; an absent bound is -inf / +inf, an absent max_change no limit
__device__ __forceinline__ float clamp_sigma(float s, float target, float lo, float hi, bool has_mc, float c) {
  if (has_mc) {
    const float allowed = fabsf(s) * c;
    lo = torch_max(lo, s - allowed);
    hi = torch_min(hi, s + allowed);
  }
  return torch_min(torch_max(target, lo), hi);
}

// sigma[i] after the step lr * g[i]: the target sigma + step (or sigma * exp(step / 2)), then clamp_sigma
__device__ __forceinline__ void sigma_step(float* __restrict__ sigma, const float* __restrict__ g, int64_t i, float lr, int exp_form,
                                           const float* __restrict__ lb_vec, float lb, const float* __restrict__ ub_vec, float ub,
                                           const float* __restrict__ mc_vec, float mc) {
  const float s = sigma[i];
  const float step = lr * g[i];
  const float target = exp_form ? s * expf(0.5f * step) : s + step;
  // a NaN scalar means "not set"; vector entries are user data and keep their NaNs
  const float lo = lb_vec ? lb_vec[i] : (lb != lb ? -INFINITY : lb);
  const float hi = ub_vec ? ub_vec[i] : (ub != ub ? INFINITY : ub);
  const bool has_mc = mc_vec != nullptr || mc == mc;
  sigma[i] = clamp_sigma(s, target, lo, hi, has_mc, mc_vec ? mc_vec[i] : mc);
}

__global__ void __launch_bounds__(256) sigma_update_kernel(float* __restrict__ sigma, const float* __restrict__ g, int64_t D, float lr,
                                                           int exp_form, const float* __restrict__ lb_vec, float lb,
                                                           const float* __restrict__ ub_vec, float ub, const float* __restrict__ mc_vec,
                                                           float mc) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  sigma_step(sigma, g, i, lr, exp_form, lb_vec, lb, ub_vec, ub, mc_vec, mc);
}

// Batched searches: per-item scalar hyper-parameters travel BY VALUE in the launch parameters (no device copy, no sync)
constexpr int kItemsPerLaunch = 256;
struct ItemScalars {
  float a[kItemsPerLaunch], b[kItemsPerLaunch], c[kItemsPerLaunch];
};

// one CTA per item: clipup on row blockIdx.x of [items][D] tensors, with that item's (lr, momentum, max_speed)
__global__ void __launch_bounds__(kUpdThreads) clipup_batched_kernel(const float* __restrict__ g, int64_t D, float* __restrict__ velocity,
                                                                     float* __restrict__ center, const __grid_constant__ ItemScalars sc) {
  const int item = blockIdx.x;
  const int64_t off = (int64_t)item * D;
  clipup(g + off, D, velocity + off, sc.a[item], sc.b[item], sc.c[item], [&](int64_t i, float nv) { center[off + i] += nv; });
}

// sigma_update_kernel on [items][D] tensors with a per-item learning rate (blockIdx.y = item)
__global__ void __launch_bounds__(256) sigma_update_batched_kernel(float* __restrict__ sigma, const float* __restrict__ g, int64_t D, int exp_form,
                                                                   const float* __restrict__ lb_vec, const float* __restrict__ ub_vec,
                                                                   const float* __restrict__ mc_vec, const __grid_constant__ ItemScalars sc) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  // absent bounds and max_change: the NaN scalars
  sigma_step(sigma, g, (int64_t)blockIdx.y * D + j, sc.a[blockIdx.y], exp_form, lb_vec, NAN, ub_vec, NAN, mc_vec, NAN);
}

// E elites: grad_mu = S1 / E, grad_sigma = unbiased std - sigma.  As torch.std: E = 1 (a zero divisor) and E = 0 give NaN, and a NaN
// variance stays NaN through the clamp at 0 (torch.clamp_min); without the E = 1 case the fp32 rounding error of S2 over 0 gave +-inf.
__global__ void __launch_bounds__(256) cem_finalize_kernel(const float* __restrict__ s1, const float* __restrict__ s2,
                                                           const float* __restrict__ sigma, int64_t D, float E, float* __restrict__ grad_mu,
                                                           float* __restrict__ grad_sigma) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  const double a = (double)s1[i], b = (double)s2[i], e = (double)E;
  const double var = e > 1.0 ? (b - a * a / e) / (e - 1.0) : (double)NAN;
  grad_mu[i] = (float)(a / e);
  grad_sigma[i] = (float)sqrt(var > 0.0 || var != var ? var : 0.0) - sigma[i];
}

}  // namespace evok

using namespace evok;

static inline unsigned nblk(int64_t D) { return (unsigned)((D + 255) / 256); }

extern "C" EVOK_API int evok_clipup_step(const float* g, int64_t D, float* velocity, float stepsize, float momentum, float max_speed,
                                float* step_out, float* mu, void* stream) {
  if (!g || !velocity) return EVOK_E_NULLPTR;
  if (D <= 0) return EVOK_E_BADSIZE;
  clipup_kernel<<<1, kUpdThreads, 0, (cudaStream_t)stream>>>(g, D, velocity, stepsize, momentum, max_speed, step_out, mu);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_adam_step(const float* g, int64_t D, float* m, float* v, int64_t t, float lr, float beta1, float beta2, float eps,
                              float* step_out, float* mu, void* stream) {
  if (!g || !m || !v) return EVOK_E_NULLPTR;
  if (D <= 0 || t < 1) return EVOK_E_BADSIZE;
  const double bc1 = 1.0 - pow((double)beta1, (double)t), bc2 = 1.0 - pow((double)beta2, (double)t);
  adam_kernel<<<nblk(D), 256, 0, (cudaStream_t)stream>>>(g, D, m, v, beta1, beta2, (float)((double)lr / bc1), (float)(1.0 / sqrt(bc2)), eps,
                                                         step_out, mu);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_sgd_step(const float* g, int64_t D, float* buf, int first_step, float lr, float momentum, float* step_out, float* mu,
                             void* stream) {
  if (!g) return EVOK_E_NULLPTR;
  if (momentum != 0.0f && !buf) return EVOK_E_NULLPTR;
  if (D <= 0) return EVOK_E_BADSIZE;
  sgd_kernel<<<nblk(D), 256, 0, (cudaStream_t)stream>>>(g, D, buf, first_step, lr, momentum, step_out, mu);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_axpy(const float* g, int64_t D, float lr, float* mu, void* stream) {
  if (!g || !mu) return EVOK_E_NULLPTR;
  if (D <= 0) return EVOK_E_BADSIZE;
  axpy_kernel<<<nblk(D), 256, 0, (cudaStream_t)stream>>>(g, D, lr, mu);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_sigma_update(float* sigma, const float* g, int64_t D, float lr, int exp_form, const float* lb_vec, float lb,
                                 const float* ub_vec, float ub, const float* mc_vec, float mc, void* stream) {
  if (!sigma || !g) return EVOK_E_NULLPTR;
  if (D <= 0) return EVOK_E_BADSIZE;
  sigma_update_kernel<<<nblk(D), 256, 0, (cudaStream_t)stream>>>(sigma, g, D, lr, exp_form, lb_vec, lb, ub_vec, ub, mc_vec, mc);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_cem_finalize(const float* s1, const float* s2, const float* sigma, int64_t D, int64_t num_elites, float* grad_mu,
                                 float* grad_sigma, void* stream) {
  if (!s1 || !s2 || !sigma || !grad_mu || !grad_sigma) return EVOK_E_NULLPTR;
  if (D <= 0 || num_elites < 0) return EVOK_E_BADSIZE;
  cem_finalize_kernel<<<nblk(D), 256, 0, (cudaStream_t)stream>>>(s1, s2, sigma, D, (float)num_elites, grad_mu, grad_sigma);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_clipup_batched(const float* g, int64_t n_items, int64_t D, float* velocity, float* center, const float* stepsize_host,
                                            const float* momentum_host, const float* max_speed_host, void* stream) {
  if (!g || !velocity || !center || !stepsize_host || !momentum_host || !max_speed_host) return EVOK_E_NULLPTR;
  if (D <= 0 || n_items < 0) return EVOK_E_BADSIZE;
  return for_item_chunks(n_items, kItemsPerLaunch, [&](int64_t b0, int64_t n) {
    ItemScalars sc;
    for (int i = 0; i < n; ++i) {
      sc.a[i] = stepsize_host[b0 + i];
      sc.b[i] = momentum_host[b0 + i];
      sc.c[i] = max_speed_host[b0 + i];
    }
    clipup_batched_kernel<<<(unsigned)n, kUpdThreads, 0, (cudaStream_t)stream>>>(g + b0 * D, D, velocity + b0 * D, center + b0 * D, sc);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_sigma_update_batched(float* sigma, const float* g, int64_t n_items, int64_t D, const float* lr_host, int exp_form,
                                                  const float* lb_vec, const float* ub_vec, const float* mc_vec, void* stream) {
  if (!sigma || !g || !lr_host) return EVOK_E_NULLPTR;
  if (D <= 0 || n_items < 0) return EVOK_E_BADSIZE;
  return for_item_chunks(n_items, kItemsPerLaunch, [&](int64_t b0, int64_t n) {
    ItemScalars sc;
    for (int i = 0; i < n; ++i) sc.a[i] = lr_host[b0 + i];
    const int64_t off = b0 * D;
    sigma_update_batched_kernel<<<dim3(nblk(D), (unsigned)n), 256, 0, (cudaStream_t)stream>>>(
        sigma + off, g + off, D, exp_form, lb_vec ? lb_vec + off : nullptr, ub_vec ? ub_vec + off : nullptr, mc_vec ? mc_vec + off : nullptr, sc);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_abi_version(void) { return EVOK_ABI_VERSION; }

extern "C" EVOK_API uint64_t evok_launch_count(void) { return (uint64_t)__atomic_load_n(&g_launch_count, __ATOMIC_RELAXED); }

extern "C" EVOK_API const char* evok_error_string(int code) {
  switch (code) {
    case 0: return "ok";
    case EVOK_E_NULLPTR: return "null pointer argument";
    case EVOK_E_BADSIZE: return "invalid size argument";
    case EVOK_E_BADENUM: return "invalid enum argument";
    case EVOK_E_WORKSPACE: return "workspace too small";
    case EVOK_E_ODDROWS: return "symmetric sampling needs an even number of rows";
    case EVOK_E_ALIGN: return "misaligned pointer";
    case EVOK_E_NOKERNEL: return "the cubin of the registered objective lacks one of its kernels";
    case EVOK_E_NODATA: return "the objective declares data: launch an instance of it (evok_objective_instance)";
    case EVOK_E_NOISEKEY: return "the objective draws noise: evaluate it with the key of its rows (evok_eval_keyed)";
    default: return code > 0 ? cudaGetErrorString((cudaError_t)code) : "unknown error";
  }
}
