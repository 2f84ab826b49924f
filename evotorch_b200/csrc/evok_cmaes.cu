// CMA-ES generation glue (cmaes.py:432-553 of the reference): the D-vector / N-vector arithmetic between the dense
// contractions, fused so that a whole generation is a short chain of kernels without host reads and is CUDA-graph
// capturable.  The reference runs these as ~35 eager torch ops per generation.
//
//   evok_cmaes_row_weights   N-vector: positive part of the assigned weights (recombination) and the active-CMA
//                            reweighting  w_i > 0 ? w_i : d * w_i / ||z_i||^2   (cmaes.py:468-475, :531-535); one pass over Z
//   evok_cmaes_vector_update D-vectors + scalars, one CTA: m, p_sigma, sigma, h_sig, p_c and the three coefficients of the
//                            covariance update consumed by evok_gemm_nt_affine (cmaes.py:454-517, :31-46, :537-545)
// The *_batched entry points run the same kernels for a batch of independent searches: grid y (row weights) or grid x (vector
// update) is the item, so every item gets the bits of the single call on its operands.
#include "evok_common.cuh"

namespace evok {

// one warp per row: ||z_i||^2, then the two weight vectors.  grid y = item: Z at item stride item_stride_z, aw / w_pos / w_act at N
// TIERED (padded populations): item b uses its first counts[tier[b]] rows; w_pos = w_act = 0 on the others, whatever Z holds there
template <bool TIERED>
__global__ void __launch_bounds__(256) cmaes_row_weights_kernel(const float* __restrict__ aw, const float* __restrict__ Z, int64_t ldz, int64_t N,
                                                                int64_t D, int active, float* __restrict__ w_pos, float* __restrict__ w_act,
                                                                int64_t item_stride_z, const int* __restrict__ tier, const int* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= N) return;
  Z += blockIdx.y * item_stride_z;
  aw += blockIdx.y * N;
  w_pos += blockIdx.y * N;
  w_act += blockIdx.y * N;
  if (TIERED && row >= counts[tier[blockIdx.y]]) {
    if (lane == 0) w_pos[row] = w_act[row] = 0.0f;
    return;
  }
  const float a = aw[row];
  float out_act = a;
  if (active && !(a > 0.0f)) {  // only the non-positive weights need the row norm (cmaes.py:532)
    const float* z = Z + row * ldz;
    float s = 0.0f;
    if ((D & 3) == 0 && (ldz & 3) == 0 && aligned16_dev(Z)) {
      for (int64_t q = lane; q < (D >> 2); q += 32) {
        const float4 v = ld_stream4(z + 4 * q);
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
      }
    } else {
      for (int64_t j = lane; j < D; j += 32) {
        const float v = z[j];
        s = fmaf(v, v, s);
      }
    }
    s = warp_sum(s);
    out_act = __fdiv_rn((float)D * a, s);
  }
  if (lane == 0) {
    w_pos[row] = fmaxf(a, 0.0f);
    w_act[row] = out_act;
  }
}

struct CmaesConsts {
  float c_m, c_sigma, damp_sigma, c_c, c_1, c_mu, vd_sigma, vd_c, unbiased_expectation, weights_sum;
  int csa_squared;
};

constexpr int kCmaThreads = 1024;

// padded populations (the *_tiered entries): the constants of tier k, row k of a device table [tiers][10] in the order of
// cmaes_consts; csa_squared stays the shared one
__device__ __forceinline__ CmaesConsts tier_consts(const CmaesConsts& shared, const float* __restrict__ tab, int k) {
  const float* r = tab + (int64_t)k * 10;
  CmaesConsts c;
  c.c_m = r[0]; c.c_sigma = r[1]; c.damp_sigma = r[2]; c.c_c = r[3]; c.c_1 = r[4]; c.c_mu = r[5]; c.vd_sigma = r[6]; c.vd_c = r[7];
  c.unbiased_expectation = r[8]; c.weights_sum = r[9];
  c.csa_squared = shared.csa_squared;
  return c;
}

struct CmaVectorStep {
  float new_sigma, h;
  long long steps;  // generation counter before this generation's increment
};

// update_m, update_p_sigma, update_sigma, _h_sig, update_p_c (cmaes.py:454-517, :31-46) on one CTA, in place; element i belongs
// to thread i % kCmaThreads.  The shaped displacement sum_i w_i y_i is `shaped_disp` or, separable (SEP), A * local_disp (y = A z
// elementwise).  m_prev (SEP, nullable) receives m before the update.  *sigma is left to the caller (read by every thread first).
template <bool SEP>
__device__ __forceinline__ CmaVectorStep cma_vector_step(const float* __restrict__ local_disp, const float* __restrict__ shaped_disp,
                                                         const float* __restrict__ A, int64_t D, float* __restrict__ m, float* __restrict__ p_sigma,
                                                         float* __restrict__ p_c, const float* sigma, const long long* steps_dev, long long steps_host,
                                                         const CmaesConsts& c, double* sm, float* __restrict__ m_prev) {
  const float sig = *sigma;
  const long long steps = steps_dev ? *steps_dev : steps_host;
  // update_m (cmaes.py:477-479, uses the OLD sigma) and update_p_sigma (:483-490)
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < D; i += kCmaThreads) {
    const float mi = m[i];
    if (SEP && m_prev) m_prev[i] = mi;
    m[i] = mi + c.c_m * sig * (SEP ? A[i] * local_disp[i] : shaped_disp[i]);
    const float ps = (1.0f - c.c_sigma) * p_sigma[i] + c.vd_sigma * local_disp[i];
    p_sigma[i] = ps;
    acc += (double)ps * (double)ps;
  }
  const float pnorm = (float)sqrt(block_sum<double>(acc, sm));
  // update_sigma (:492-507)
  const float dn = (float)D;
  const float expo = c.csa_squared ? (pnorm * pnorm / dn - 1.0f) * 0.5f : pnorm / c.unbiased_expectation - 1.0f;
  const float new_sigma = sig * expf((c.c_sigma / c.damp_sigma) * expo);
  // _h_sig (:31-46): generation counter BEFORE the increment
  const double decay = 1.0 - pow(1.0 - (double)c.c_sigma, (double)(2 * steps + 1));
  const float squared_sum = (float)((double)(pnorm * pnorm) / decay);
  const float h = ((squared_sum / dn) - 1.0f < 1.0f + 4.0f / (dn + 1.0f)) ? 1.0f : 0.0f;
  // update_p_c (:509-517)
  for (int64_t i = threadIdx.x; i < D; i += kCmaThreads)
    p_c[i] = (1.0f - c.c_c) * p_c[i] + h * c.vd_c * (SEP ? A[i] * local_disp[i] : shaped_disp[i]);
  return CmaVectorStep{new_sigma, h, steps};
}

// one CTA per item (grid x): the D-vectors of item b at b * D, its sigma at b, its k_out at 3 b, its step counter (nullable) at
// steps_dev[b] (h_sig_out: single call only).  TIERED: item b's constants are row tier[b] of consts_tab.
template <bool TIERED>
__global__ void __launch_bounds__(kCmaThreads)
    cmaes_vector_update_kernel(const float* __restrict__ local_disp, const float* __restrict__ shaped_disp, int64_t D, float* __restrict__ m,
                               float* __restrict__ p_sigma, float* __restrict__ p_c, float* __restrict__ sigma, long long* steps_dev,
                               long long steps_host, const __grid_constant__ CmaesConsts shared, float* __restrict__ k_out, float* __restrict__ h_sig_out,
                               const int* __restrict__ tier, const float* __restrict__ consts_tab) {
  __shared__ double sm[33];
  const CmaesConsts c = TIERED ? tier_consts(shared, consts_tab, tier[blockIdx.x]) : shared;
  const int64_t off = (int64_t)blockIdx.x * D;
  local_disp += off;
  shaped_disp += off;
  m += off;
  p_sigma += off;
  p_c += off;
  sigma += blockIdx.x;
  k_out += 3 * (int64_t)blockIdx.x;
  if (steps_dev) steps_dev += blockIdx.x;
  const CmaVectorStep v = cma_vector_step<false>(local_disp, shaped_disp, nullptr, D, m, p_sigma, p_c, sigma, steps_dev, steps_host, c, sm, nullptr);
  const float new_sigma = v.new_sigma, h = v.h;
  const long long steps = v.steps;
  if (threadIdx.x == 0) {
    *sigma = new_sigma;
    if (steps_dev) *steps_dev = steps + 1;
    // covariance update C <- C + c1a (pc pc^T - C) + c_mu (S - sum(w) C), pc = weighted_pc * p_c   (:537-549)
    const float c1a = c.c_1 * (1.0f - (1.0f - h * h) * c.c_c * (2.0f - c.c_c));
    const float wpc2 = c.c_1 / (c1a + 1e-23f);  // weighted_pc squared
    k_out[0] = c.c_mu;
    k_out[1] = 1.0f - c1a - c.c_mu * c.weights_sum;
    k_out[2] = c1a * wpc2;
    if (h_sig_out) *h_sig_out = h;
  }
}

// Separable CMA-ES, everything after the moments in one CTA: cma_vector_step, then per element (cmaes.py:536-545, separable
// branch, and :49-79, :555-565 of the reference)
//   C <- C + c1a (p_c^2 - C) + c_mu (A^2 S2 - wsum C)              (S2 = sum_i b_i z_i^2, so A^2 S2 = sum_i b_i y_i^2)
//   stdev bounds with the new sigma: C <- (clamp(sigma' sqrt(C), lo, hi) / sigma')^2
//   A <- sqrt(C) on the generations where (steps + 1) % decompose_freq == 0;   s <- sigma' A  (the sampler's per-column stdev)
// s_prev (nullable) receives s before the update.  lo / hi: NaN = no bound.  Grid x = item: the D-vectors of item b at b * D, its sigma
// and wsum at b, its step counter (nullable) at steps_dev[b] (m_prev / s_prev / h_sig_out: single call only).  TIERED: item b's
// constants are row tier[b] of consts_tab and its decomposition period freq_tab[tier[b]].
template <bool TIERED>
__global__ void __launch_bounds__(kCmaThreads)
    sepcma_update_kernel(const float* __restrict__ local_disp, const float* __restrict__ S2, const float* __restrict__ wsum, int64_t D,
                         float* __restrict__ m, float* __restrict__ p_sigma, float* __restrict__ p_c, float* __restrict__ sigma, float* __restrict__ C,
                         float* __restrict__ A, float* __restrict__ s, float* __restrict__ m_prev, float* __restrict__ s_prev, long long* steps_dev,
                         long long steps_host, const __grid_constant__ CmaesConsts shared, long long decompose_freq_shared, float lo, float hi,
                         float* __restrict__ h_sig_out, const int* __restrict__ tier, const float* __restrict__ consts_tab,
                         const long long* __restrict__ freq_tab) {
  __shared__ double sm[33];
  const CmaesConsts c = TIERED ? tier_consts(shared, consts_tab, tier[blockIdx.x]) : shared;
  const long long decompose_freq = TIERED ? freq_tab[tier[blockIdx.x]] : decompose_freq_shared;
  const int64_t off = (int64_t)blockIdx.x * D;
  local_disp += off;
  S2 += off;
  m += off;
  p_sigma += off;
  p_c += off;
  C += off;
  A += off;
  s += off;
  sigma += blockIdx.x;
  wsum += blockIdx.x;
  if (steps_dev) steps_dev += blockIdx.x;
  const CmaVectorStep v = cma_vector_step<true>(local_disp, nullptr, A, D, m, p_sigma, p_c, sigma, steps_dev, steps_host, c, sm, m_prev);
  const float sg = v.new_sigma, h = v.h;
  const float c1a = c.c_1 * (1.0f - (1.0f - h * h) * c.c_c * (2.0f - c.c_c));
  const float ws = *wsum;
  const bool has_lo = !isnan(lo), has_hi = !isnan(hi);
  const bool decompose = (v.steps + 1) % decompose_freq == 0;
  for (int64_t i = threadIdx.x; i < D; i += kCmaThreads) {
    const float Ci = C[i], Ai = A[i], pc = p_c[i];  // p_c[i] was just written by this thread
    float Cn = Ci + c1a * (pc * pc - Ci) + c.c_mu * (Ai * Ai * S2[i] - ws * Ci);
    if (has_lo || has_hi) {
      float sd = sg * sqrtf(Cn);
      if (has_lo && sd < lo) sd = lo;  // NaN stays NaN, like torch.clamp
      if (has_hi && sd > hi) sd = hi;
      const float u = __fdiv_rn(sd, sg);
      Cn = u * u;
    }
    C[i] = Cn;
    const float An = decompose ? sqrtf(Cn) : Ai;
    A[i] = An;
    if (s_prev) s_prev[i] = s[i];
    s[i] = sg * An;
  }
  if (threadIdx.x == 0) {
    *sigma = sg;
    if (steps_dev) *steps_dev = v.steps + 1;
    if (h_sig_out) *h_sig_out = h;
  }
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API int evok_cmaes_row_weights(const float* assigned_weights, const float* Z, int64_t ldz, int64_t N, int64_t D, int active,
                                               float* w_positive, float* w_active, void* stream) {
  if (!assigned_weights || !Z || !w_positive || !w_active) return EVOK_E_NULLPTR;
  if (N <= 0 || D <= 0 || ldz < D) return EVOK_E_BADSIZE;
  cmaes_row_weights_kernel<false><<<(unsigned)((N + 7) / 8), 256, 0, (cudaStream_t)stream>>>(assigned_weights, Z, ldz, N, D, active, w_positive,
                                                                                       w_active, 0, nullptr, nullptr);
  EVOK_CHECK_LAUNCH();
  return 0;
}

// the batched row weights, every row of every item (tier == NULL) or the first counts[tier[b]] rows of item b
template <bool TIERED>
static int cmaes_row_weights_items(const float* assigned_weights, const float* Z, int64_t item_stride_z, int64_t ldz, int64_t n_items, int64_t N,
                                   int64_t D, int active, const int32_t* tier, const int32_t* counts, float* w_positive, float* w_active,
                                   void* stream) {
  if (!assigned_weights || !Z || !w_positive || !w_active) return EVOK_E_NULLPTR;
  if (n_items < 0 || N <= 0 || D <= 0 || ldz < D || item_stride_z < 0) return EVOK_E_BADSIZE;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    cmaes_row_weights_kernel<TIERED><<<dim3((unsigned)((N + 7) / 8), (unsigned)nb), 256, 0, (cudaStream_t)stream>>>(
        assigned_weights + b0 * N, Z + b0 * item_stride_z, ldz, N, D, active, w_positive + b0 * N, w_active + b0 * N, item_stride_z,
        TIERED ? tier + b0 : nullptr, counts);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_cmaes_row_weights_batched(const float* assigned_weights, const float* Z, int64_t item_stride_z, int64_t ldz, int64_t n_items,
                                                       int64_t N, int64_t D, int active, float* w_positive, float* w_active, void* stream) {
  return cmaes_row_weights_items<false>(assigned_weights, Z, item_stride_z, ldz, n_items, N, D, active, nullptr, nullptr, w_positive, w_active, stream);
}

extern "C" EVOK_API int evok_cmaes_row_weights_batched_tiered(const float* assigned_weights, const float* Z, int64_t item_stride_z, int64_t ldz,
                                                              int64_t n_items, int64_t N, int64_t D, int active, const int32_t* tier,
                                                              const int32_t* counts, float* w_positive, float* w_active, void* stream) {
  if (!tier || !counts) return EVOK_E_NULLPTR;
  return cmaes_row_weights_items<true>(assigned_weights, Z, item_stride_z, ldz, n_items, N, D, active, tier, counts, w_positive, w_active, stream);
}

static CmaesConsts cmaes_consts(const float* consts_host, int csa_squared) {
  CmaesConsts c;
  c.c_m = consts_host[0]; c.c_sigma = consts_host[1]; c.damp_sigma = consts_host[2]; c.c_c = consts_host[3]; c.c_1 = consts_host[4];
  c.c_mu = consts_host[5]; c.vd_sigma = consts_host[6]; c.vd_c = consts_host[7]; c.unbiased_expectation = consts_host[8];
  c.weights_sum = consts_host[9];
  c.csa_squared = csa_squared;
  return c;
}

extern "C" EVOK_API int evok_cmaes_vector_update(const float* local_disp, const float* shaped_disp, int64_t D, float* m, float* p_sigma, float* p_c,
                                                 float* sigma_dev, int64_t* steps_dev, int64_t steps_host, const float* consts_host, int csa_squared,
                                                 float* k_out, float* h_sig_out, void* stream) {
  if (!local_disp || !shaped_disp || !m || !p_sigma || !p_c || !sigma_dev || !consts_host || !k_out) return EVOK_E_NULLPTR;
  if (D <= 0) return EVOK_E_BADSIZE;
  const CmaesConsts c = cmaes_consts(consts_host, csa_squared);
  cmaes_vector_update_kernel<false><<<1, kCmaThreads, 0, (cudaStream_t)stream>>>(local_disp, shaped_disp, D, m, p_sigma, p_c, sigma_dev,
                                                                                reinterpret_cast<long long*>(steps_dev), (long long)steps_host, c, k_out,
                                                                                h_sig_out, nullptr, nullptr);
  EVOK_CHECK_LAUNCH();
  return 0;
}

// the batched vector update with a shared step counter (steps_dev == NULL) or one per item (steps_dev[b]), with the shared
// constants of consts_host or (TIERED) item b's row tier[b] of the device table consts_dev
template <bool TIERED>
static int cmaes_vector_update_items(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D, float* m, float* p_sigma,
                                     float* p_c, float* sigma_dev, int64_t* steps_dev, int64_t steps_host, const float* consts_host, int csa_squared,
                                     float* k_out, const int32_t* tier, const float* consts_dev, void* stream) {
  if (!local_disp || !shaped_disp || !m || !p_sigma || !p_c || !sigma_dev || !(TIERED ? consts_dev : consts_host) || !k_out) return EVOK_E_NULLPTR;
  if (n_items < 0 || D <= 0) return EVOK_E_BADSIZE;
  const float zeros[10] = {};
  const CmaesConsts c = cmaes_consts(TIERED ? zeros : consts_host, csa_squared);
  return for_item_chunks(n_items, (int64_t)INT32_MAX, [&](int64_t b0, int64_t nb) {
    const int64_t off = b0 * D;
    cmaes_vector_update_kernel<TIERED><<<(unsigned)nb, kCmaThreads, 0, (cudaStream_t)stream>>>(
        local_disp + off, shaped_disp + off, D, m + off, p_sigma + off, p_c + off, sigma_dev + b0,
        steps_dev ? reinterpret_cast<long long*>(steps_dev + b0) : nullptr, (long long)steps_host, c, k_out + 3 * b0, nullptr,
        TIERED ? tier + b0 : nullptr, consts_dev);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_cmaes_vector_update_batched(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D, float* m,
                                                         float* p_sigma, float* p_c, float* sigma_dev, int64_t steps_host, const float* consts_host,
                                                         int csa_squared, float* k_out, void* stream) {
  return cmaes_vector_update_items<false>(local_disp, shaped_disp, n_items, D, m, p_sigma, p_c, sigma_dev, nullptr, steps_host, consts_host,
                                          csa_squared, k_out, nullptr, nullptr, stream);
}

extern "C" EVOK_API int evok_cmaes_vector_update_batched_steps(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D,
                                                               float* m, float* p_sigma, float* p_c, float* sigma_dev, int64_t* steps_dev,
                                                               const float* consts_host, int csa_squared, float* k_out, void* stream) {
  if (!steps_dev) return EVOK_E_NULLPTR;
  return cmaes_vector_update_items<false>(local_disp, shaped_disp, n_items, D, m, p_sigma, p_c, sigma_dev, steps_dev, 0, consts_host, csa_squared,
                                          k_out, nullptr, nullptr, stream);
}

extern "C" EVOK_API int evok_cmaes_vector_update_batched_tiered(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D,
                                                                float* m, float* p_sigma, float* p_c, float* sigma_dev, int64_t* steps_dev,
                                                                const int32_t* tier, const float* consts_dev, int csa_squared, float* k_out,
                                                                void* stream) {
  if (!steps_dev || !tier) return EVOK_E_NULLPTR;
  return cmaes_vector_update_items<true>(local_disp, shaped_disp, n_items, D, m, p_sigma, p_c, sigma_dev, steps_dev, 0, nullptr, csa_squared, k_out,
                                         tier, consts_dev, stream);
}

extern "C" EVOK_API int evok_sepcma_update(const float* local_disp, const float* S2, const float* wsum, int64_t D, float* m, float* p_sigma, float* p_c,
                                           float* sigma_dev, float* C, float* A, float* s, float* m_prev, float* s_prev, int64_t* steps_dev,
                                           int64_t steps_host, const float* consts_host, int csa_squared, int64_t decompose_C_freq, float stdev_min,
                                           float stdev_max, float* h_sig_out, void* stream) {
  if (!local_disp || !S2 || !wsum || !m || !p_sigma || !p_c || !sigma_dev || !C || !A || !s || !consts_host) return EVOK_E_NULLPTR;
  if (D <= 0 || decompose_C_freq < 1) return EVOK_E_BADSIZE;
  const CmaesConsts c = cmaes_consts(consts_host, csa_squared);
  sepcma_update_kernel<false><<<1, kCmaThreads, 0, (cudaStream_t)stream>>>(local_disp, S2, wsum, D, m, p_sigma, p_c, sigma_dev, C, A, s, m_prev,
                                                                          s_prev, reinterpret_cast<long long*>(steps_dev), (long long)steps_host, c,
                                                                          (long long)decompose_C_freq, stdev_min, stdev_max, h_sig_out, nullptr, nullptr,
                                                                          nullptr);
  EVOK_CHECK_LAUNCH();
  return 0;
}

// the batched separable update with a shared step counter (steps_dev == NULL) or one per item (steps_dev[b]), with the shared
// constants and decomposition period or (TIERED) item b's row tier[b] of the device tables consts_dev and freq_dev
template <bool TIERED>
static int sepcma_update_items(const float* local_disp, const float* S2, const float* wsum, int64_t n_items, int64_t D, float* m, float* p_sigma,
                               float* p_c, float* sigma_dev, float* C, float* A, float* s, int64_t* steps_dev, int64_t steps_host,
                               const float* consts_host, int csa_squared, int64_t decompose_C_freq, float stdev_min, float stdev_max,
                               const int32_t* tier, const float* consts_dev, const int64_t* freq_dev, void* stream) {
  if (!local_disp || !S2 || !wsum || !m || !p_sigma || !p_c || !sigma_dev || !C || !A || !s || !(TIERED ? consts_dev && freq_dev : consts_host != nullptr))
    return EVOK_E_NULLPTR;
  if (n_items < 0 || D <= 0 || decompose_C_freq < 1) return EVOK_E_BADSIZE;
  const float zeros[10] = {};
  const CmaesConsts c = cmaes_consts(TIERED ? zeros : consts_host, csa_squared);
  return for_item_chunks(n_items, (int64_t)INT32_MAX, [&](int64_t b0, int64_t nb) {
    const int64_t off = b0 * D;
    sepcma_update_kernel<TIERED><<<(unsigned)nb, kCmaThreads, 0, (cudaStream_t)stream>>>(
        local_disp + off, S2 + off, wsum + b0, D, m + off, p_sigma + off, p_c + off, sigma_dev + b0, C + off, A + off, s + off, nullptr, nullptr,
        steps_dev ? reinterpret_cast<long long*>(steps_dev + b0) : nullptr, (long long)steps_host, c, (long long)decompose_C_freq, stdev_min,
        stdev_max, nullptr, TIERED ? tier + b0 : nullptr, consts_dev, reinterpret_cast<const long long*>(freq_dev));
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_sepcma_update_batched(const float* local_disp, const float* S2, const float* wsum, int64_t n_items, int64_t D, float* m,
                                                   float* p_sigma, float* p_c, float* sigma_dev, float* C, float* A, float* s, int64_t steps_host,
                                                   const float* consts_host, int csa_squared, int64_t decompose_C_freq, float stdev_min, float stdev_max,
                                                   void* stream) {
  return sepcma_update_items<false>(local_disp, S2, wsum, n_items, D, m, p_sigma, p_c, sigma_dev, C, A, s, nullptr, steps_host, consts_host, csa_squared,
                                    decompose_C_freq, stdev_min, stdev_max, nullptr, nullptr, nullptr, stream);
}

extern "C" EVOK_API int evok_sepcma_update_batched_steps(const float* local_disp, const float* S2, const float* wsum, int64_t n_items, int64_t D,
                                                         float* m, float* p_sigma, float* p_c, float* sigma_dev, float* C, float* A, float* s,
                                                         int64_t* steps_dev, const float* consts_host, int csa_squared, int64_t decompose_C_freq,
                                                         float stdev_min, float stdev_max, void* stream) {
  if (!steps_dev) return EVOK_E_NULLPTR;
  return sepcma_update_items<false>(local_disp, S2, wsum, n_items, D, m, p_sigma, p_c, sigma_dev, C, A, s, steps_dev, 0, consts_host, csa_squared,
                                    decompose_C_freq, stdev_min, stdev_max, nullptr, nullptr, nullptr, stream);
}

extern "C" EVOK_API int evok_sepcma_update_batched_tiered(const float* local_disp, const float* S2, const float* wsum, int64_t n_items, int64_t D,
                                                          float* m, float* p_sigma, float* p_c, float* sigma_dev, float* C, float* A, float* s,
                                                          int64_t* steps_dev, const int32_t* tier, const float* consts_dev,
                                                          const int64_t* decompose_C_freq_dev, int csa_squared, float stdev_min, float stdev_max,
                                                          void* stream) {
  if (!steps_dev || !tier) return EVOK_E_NULLPTR;
  return sepcma_update_items<true>(local_disp, S2, wsum, n_items, D, m, p_sigma, p_c, sigma_dev, C, A, s, steps_dev, 0, nullptr, csa_squared, 1,
                                   stdev_min, stdev_max, tier, consts_dev, decompose_C_freq_dev, stream);
}
