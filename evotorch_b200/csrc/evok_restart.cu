// The restart stage of the functional CMA-ES families (full and separable): per item, after the family's update, the best-ever
// solution, the tol_fun history, the termination criteria and the re-initialisation of the items that met one, without host reads.
//
//   cma_restart_kernel     one CTA per item: best of this generation, best ever, history, criteria, stop flags; for a restarted
//                          item a uniform centre in [lb, ub], sigma0, zero paths, counter 0, empty history (separable: C = A = 1, s)
//   cma_restart_eye_kernel full family only: C = A = I for the restarted items, grid-wide, masked by the flags
// The tiered form (IPOP, padded populations) reads N and H of item b from its tier, moves a restarted item one tier up and
// counts the evaluations of each item.  The BIPOP form is the tiered one with a per-item policy at restart time instead of the
// tier advance: a large run one rung up the ladder or a small run of random population size and step size, whichever regime has
// used fewer evaluations, and a budget stop (bit 7) for small runs.
#include "evok_common.cuh"

namespace evok {

constexpr int kRestartThreads = 256;
constexpr int kRestartWarps = kRestartThreads / kWarp;
constexpr int kEyeThreads = 256;
constexpr int64_t kEyeMaxBlocksPerItem = 64;

// the forms of the stage: plain, tiered (IPOP) and BIPOP (tiered, with the regime policy at restart time)
enum RestartMode : int { kRestartPlain = 0, kRestartTiered = 1, kRestartBipop = 2 };

struct RestartArgs {
  const float* f;       // [items][n_rows]
  const float* X;       // [items][n_rows][D] at item_stride_x / ldx; NULL (separable): rows rebuilt from the draw
  int64_t item_stride_x, ldx;
  const float* m_draw;  // the centre and stdev the population was drawn from (rebuilt rows only) [items][D]
  const float* s_draw;
  PhiloxKey draw_key;   // (seed of the draw, stream 0): item b on stream word draw_key.stream_lo + b
  PhiloxKey reset_key;  // (seed of this stage, stream 0): item b on stream word reset_key.stream_lo + b
  int64_t n_rows, D, H;
  int separable, maximize;
  long long* item_steps;  // generations since the item's (re)start, after this generation's update
  float *m, *sigma, *p_sigma, *p_c, *C, *A, *s;  // full: C, A [items][D][D] (diagonals read); separable: C, A, s [items][D]
  float* history;                                // [items][H]
  float *best_x, *best_f;
  long long* num_restarts;
  int* stop_flags;
  const float *sigma0, *lb, *ub;
  int64_t item_stride_bounds;
  float tol_fun, tol_x, tol_x_up, max_condition, min_fitness_stdev, max_generations;  // NaN = off
  // tiered only: item b uses the first tier_counts[tier[b]] of its n_rows rows and the first tier_history[tier[b]] of its H slots
  int* tier;
  const int* tier_counts;
  const long long* tier_history;
  int n_tiers;
  long long* num_evaluations;
  // BIPOP only: the regime (0 first run, 1 large, 2 small), the ladder rung of the latest large run, the evaluations of each regime
  // and of the latest large run, the step size the current run started with; tiers 0..n_large-1 are the ladder, tier
  // n_large + (lambda - popsize0) the small run of population size lambda; sigma0 is the default step size
  int *regime, *large_tier;
  long long *large_evaluations, *small_evaluations, *last_large_evaluations;
  float* run_stdev;
  int n_large, popsize0;
};

// the row that wins: finite, better under the sense, the lower index on ties; index -1 = none
__device__ __forceinline__ bool wins(float a, long long ia, float b, long long ib, bool maximize) {
  if (ia < 0) return false;
  if (ib < 0) return true;
  if (a != b) return maximize ? a > b : a < b;
  return ia < ib;
}

template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* sm /* kRestartWarps + 1 */) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    T t = sm[0];
    for (int w = 1; w < kRestartWarps; ++w) t = op(t, sm[w]);
    sm[kRestartWarps] = t;
  }
  __syncthreads();
  return sm[kRestartWarps];
}

struct FMax { __device__ float operator()(float a, float b) const { return fmaxf(a, b); } };
struct FMin { __device__ float operator()(float a, float b) const { return fminf(a, b); } };
struct DSum { __device__ double operator()(double a, double b) const { return a + b; } };

// BIPOP, thread 0 of a restarting item's CTA, after its run was accounted: the next run.  Large (one rung up the ladder, the default
// step size) unless the large runs used more evaluations than the small ones.  Small: lambda_s = max(lambda_0, floor(lambda_0
// (lambda_l / (2 lambda_0))^(u1^2))), step size sigma_def 10^(-2 u2), in float64, with u1, u2 = uniform24 of words x, y of Philox
// counter (0, 1, 0xFF000000, item) under the reset key: the reset centres use (j >> 2, 0, 0xFF000000, item), so no other draw
// has this counter.
__device__ __forceinline__ void bipop_next_run(const RestartArgs& a, int64_t b, int regime, long long gen, int64_t N, float* s_run_stdev) {
  if (regime == 1) a.last_large_evaluations[b] = gen * N;
  int lt = a.large_tier[b], next;
  float stdev = a.sigma0[b];
  if (a.large_evaluations[b] <= a.small_evaluations[b]) {
    lt = min(lt + 1, a.n_large - 1);
    a.large_tier[b] = lt;
    a.regime[b] = 1;
    next = lt;
  } else {
    const U4 r = philox4x32_10(U4{0u, 1u, 0xFF000000u, a.reset_key.stream_lo + (uint32_t)b}, a.reset_key);
    const double u1 = (double)uniform24(r.x), u2 = (double)uniform24(r.y);
    const double lam0 = (double)a.popsize0;
    const double lam = floor(lam0 * exp(u1 * u1 * log(0.5 * (double)a.tier_counts[lt] / lam0)));
    const int small = lam > lam0 ? (int)lam - a.popsize0 : 0;
    next = min(a.n_large + small, a.n_tiers - 1);
    stdev = (float)((double)a.sigma0[b] * exp10(-2.0 * u2));
    a.regime[b] = 2;
  }
  a.tier[b] = next;
  a.run_stdev[b] = stdev;
  *s_run_stdev = stdev;
}

template <int MODE>
__global__ void __launch_bounds__(kRestartThreads) cma_restart_kernel(const __grid_constant__ RestartArgs a) {
  constexpr bool TIERED = MODE != kRestartPlain;
  constexpr bool BIPOP = MODE == kRestartBipop;
  __shared__ float smf[kRestartWarps + 1];
  __shared__ double smd[kRestartWarps + 1];
  __shared__ float s_best_v[kRestartWarps];
  __shared__ long long s_best_i[kRestartWarps];
  __shared__ int s_flags;
  __shared__ float s_run_stdev;
  const int64_t b = blockIdx.x, D = a.D;
  const int tk = TIERED ? a.tier[b] : 0;
  const int64_t N = TIERED ? min((int64_t)a.tier_counts[tk], a.n_rows) : a.n_rows;
  const int64_t H = TIERED ? min((int64_t)a.tier_history[tk], a.H) : a.H;
  const bool maximize = a.maximize != 0;
  const float* f = a.f + b * a.n_rows;
  const float old_best = a.best_f[b];  // read before the barriers below: thread 0 overwrites it

  // this generation's fitnesses: the best finite row, min, max, a non-finite one, the sum
  float bv = 0.0f, fmn = INFINITY, fmx = -INFINITY;
  long long bi = -1;
  int bad = 0;
  double sum = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += kRestartThreads) {
    const float v = f[i];
    if (isfinite(v)) {
      if (wins(v, i, bv, bi, maximize)) { bv = v; bi = i; }
    } else {
      bad = 1;
    }
    fmn = fminf(fmn, v);
    fmx = fmaxf(fmx, v);
    sum += (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (wins(ov, oi, bv, bi, maximize)) { bv = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { s_best_v[threadIdx.x >> 5] = bv; s_best_i[threadIdx.x >> 5] = bi; }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) {
    for (int w = 1; w < kRestartWarps; ++w)
      if (wins(s_best_v[w], s_best_i[w], bv, bi, maximize)) { bv = s_best_v[w]; bi = s_best_i[w]; }
    s_best_v[0] = bv;
    s_best_i[0] = bi;
  }
  fmn = block_reduce(fmn, FMin(), smf);
  fmx = block_reduce(fmx, FMax(), smf);
  sum = block_reduce(sum, DSum(), smd);
  bv = s_best_v[0];
  bi = s_best_i[0];
  const double mean = sum / (double)N;
  double dev = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += kRestartThreads) {
    const double e = (double)f[i] - mean;
    dev += e * e;
  }
  dev = block_reduce(dev, DSum(), smd);

  // best ever: copy the winning row (as told, or rebuilt bit for bit from the draw) when it is strictly better
  if (bi >= 0 && (maximize ? bv > old_best : bv < old_best)) {
    float* bx = a.best_x + b * D;
    if (a.X) {
      const float* x = a.X + b * a.item_stride_x + bi * a.ldx;
      for (int64_t j = threadIdx.x; j < D; j += kRestartThreads) bx[j] = x[j];
    } else {
      const float* md = a.m_draw + b * D;
      const float* sd = a.s_draw + b * D;
      const uint32_t sw = a.draw_key.stream_lo + (uint32_t)b;
      for (int64_t g = threadIdx.x; 4 * g < D; g += kRestartThreads) {
        float z[4];
        normals4(a.draw_key, sw, (uint64_t)bi, (uint32_t)g, z);
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (4 * g + c < D) bx[4 * g + c] = fmaf(sd[4 * g + c], z[c], md[4 * g + c]);
      }
    }
    if (threadIdx.x == 0) a.best_f[b] = bv;
  }

  // history: slot (g - 1) % H holds the best eval of the item's generation g (NaN: none was finite)
  const long long gen = a.item_steps[b];
  float* hist = a.history + b * a.H;
  if (threadIdx.x == 0 && gen >= 1) hist[(gen - 1) % H] = bi >= 0 ? bv : NAN;
  __syncthreads();
  float hmn = INFINITY, hmx = -INFINITY;
  int hbad = 0;
  if (gen >= H) {
    for (int64_t k = threadIdx.x; k < H; k += kRestartThreads) {
      const float v = hist[k];
      hbad |= !isfinite(v);
      hmn = fminf(hmn, v);
      hmx = fmaxf(hmx, v);
    }
  }
  hbad = __syncthreads_or(hbad);
  hmn = block_reduce(hmn, FMin(), smf);
  hmx = block_reduce(hmx, FMax(), smf);

  // the state after the update: sigma, max |p_c|, max sqrt(diag C), the range of diag A (full) or diag C (separable), finiteness
  const float sig = a.sigma[b];
  const float* m = a.m + b * D;
  const float* ps = a.p_sigma + b * D;
  const float* pc = a.p_c + b * D;
  const int64_t dstride = a.separable ? 1 : D + 1;
  const float* Cd = a.C + b * (a.separable ? D : D * D);
  const float* Ad = a.A + b * (a.separable ? D : D * D);
  float mpc = 0.0f, msd = 0.0f, rmx = -INFINITY, rmn = INFINITY;
  int nonfinite = !(sig > 0.0f) || !isfinite(sig);
  for (int64_t j = threadIdx.x; j < D; j += kRestartThreads) {
    const float cj = Cd[j * dstride], r = a.separable ? cj : Ad[j * dstride];
    nonfinite |= !isfinite(m[j]) || !isfinite(ps[j]) || !isfinite(pc[j]) || !isfinite(cj);
    mpc = fmaxf(mpc, fabsf(pc[j]));
    msd = fmaxf(msd, sqrtf(cj));
    rmx = fmaxf(rmx, r);
    rmn = fminf(rmn, r);
  }
  nonfinite = __syncthreads_or(nonfinite);
  mpc = block_reduce(mpc, FMax(), smf);
  msd = block_reduce(msd, FMax(), smf);
  rmx = block_reduce(rmx, FMax(), smf);
  rmn = block_reduce(rmn, FMin(), smf);

  if (threadIdx.x == 0) {
    const double s0 = (double)(BIPOP ? a.run_stdev[b] : a.sigma0[b]);
    int flags = 0;
    if (!isnan(a.tol_fun) && gen >= H && !bad && !hbad && (double)fmaxf(fmx, hmx) - (double)fminf(fmn, hmn) < (double)a.tol_fun) flags |= 1;
    if (!isnan(a.tol_x) && (double)sig * (double)fmaxf(mpc, msd) < (double)a.tol_x * s0) flags |= 2;
    if (!isnan(a.tol_x_up) && (double)sig * (double)msd > (double)a.tol_x_up * s0) flags |= 4;
    if (!isnan(a.max_condition)) {
      const double q = (double)rmx / (double)rmn;
      if ((a.separable ? q : q * q) > (double)a.max_condition) flags |= 8;
    }
    if (!isnan(a.min_fitness_stdev) && N > 1 && sqrt(dev / (double)(N - 1)) < (double)a.min_fitness_stdev) flags |= 16;
    if (!isnan(a.max_generations) && (double)gen >= (double)a.max_generations) flags |= 32;
    if (nonfinite) flags |= 64;
    if constexpr (BIPOP) {
      const int regime = a.regime[b];
      if (regime == 1) a.large_evaluations[b] += N;
      if (regime == 2) a.small_evaluations[b] += N;
      if (regime == 2 && 2 * gen * N >= a.last_large_evaluations[b]) flags |= 128;  // the run used half the latest large run
      if (flags) bipop_next_run(a, b, regime, gen, N, &s_run_stdev);
    }
    a.stop_flags[b] = flags;
    s_flags = flags;
    if (TIERED) a.num_evaluations[b] += N;
  }
  __syncthreads();
  if (s_flags == 0) return;


  // re-initialisation: x_j = lb_j + (ub_j - lb_j) u_j, u_j = uniform24 of word j & 3 of Philox counter (j >> 2, 0, 0xFF000000, item)
  const float* lb = a.lb + b * a.item_stride_bounds;
  const float* ub = a.ub + b * a.item_stride_bounds;
  const float s0 = BIPOP ? s_run_stdev : a.sigma0[b];
  float* mw = a.m + b * D;
  float* psw = a.p_sigma + b * D;
  float* pcw = a.p_c + b * D;
  const uint32_t sw = a.reset_key.stream_lo + (uint32_t)b;
  for (int64_t g = threadIdx.x; 4 * g < D; g += kRestartThreads) {
    const U4 r = philox4x32_10(U4{(uint32_t)g, 0u, 0xFF000000u, sw}, a.reset_key);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int64_t j = 4 * g + c;
      if (j < D) mw[j] = __fadd_rn(lb[j], __fmul_rn(__fsub_rn(ub[j], lb[j]), uniform24(w[c])));
    }
  }
  for (int64_t j = threadIdx.x; j < D; j += kRestartThreads) {
    psw[j] = 0.0f;
    pcw[j] = 0.0f;
    if (a.separable) {
      a.C[b * D + j] = 1.0f;
      a.A[b * D + j] = 1.0f;
      a.s[b * D + j] = s0;
    }
  }
  for (int64_t k = threadIdx.x; k < a.H; k += kRestartThreads) hist[k] = NAN;
  if (threadIdx.x == 0) {
    if (MODE == kRestartTiered) a.tier[b] = min(tk + 1, a.n_tiers - 1);
    a.sigma[b] = s0;
    a.item_steps[b] = 0;
    a.num_restarts[b] += 1;
  }
}

// C = A = I for the items with a stop flag; grid y = item (chunks of kMaxGridY), grid x strides over the D x D entries
__global__ void __launch_bounds__(kEyeThreads) cma_restart_eye_kernel(const int* __restrict__ stop_flags, int64_t D, float* __restrict__ C,
                                                                      float* __restrict__ A) {
  const int64_t b = blockIdx.y;
  if (stop_flags[b] == 0) return;
  C += b * D * D;
  A += b * D * D;
  for (int64_t e = (int64_t)blockIdx.x * kEyeThreads + threadIdx.x; e < D * D; e += (int64_t)gridDim.x * kEyeThreads) {
    const float v = e / D == e % D ? 1.0f : 0.0f;
    C[e] = v;
    A[e] = v;
  }
}

}  // namespace evok

using namespace evok;

// BIPOP's per-item policy arrays (evok_cma_restart_batched_bipop); unused by the other forms
struct BipopArrays {
  int32_t *regime, *large_tier;
  int64_t *large_evaluations, *small_evaluations, *last_large_evaluations;
  float* run_stdev;
  int64_t n_large, popsize0;
};

// the restart stage of evok_cma_restart_batched, of evok_cma_restart_batched_tiered with the tier arrays (kRestartTiered), or of
// evok_cma_restart_batched_bipop with the tier and policy arrays (kRestartBipop)
template <int MODE>
static int cma_restart_items(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx, const float* m_draw, const float* s_draw,
                             uint64_t draw_seed, int64_t n_items, int64_t n_rows, int64_t D, int maximize, int64_t* item_steps, float* m, float* sigma,
                             float* p_sigma, float* p_c, float* C, float* A, float* s, float* history, int64_t H, float* best_x, float* best_f,
                             int64_t* num_restarts, int32_t* stop_flags, const float* sigma0, const float* lb, const float* ub,
                             int64_t item_stride_bounds, const float* thresholds_host, uint64_t seed, int32_t* tier, const int32_t* tier_counts,
                             const int64_t* tier_history, int64_t n_tiers, int64_t* num_evaluations, const BipopArrays& bp, void* stream) {
  constexpr bool TIERED = MODE != kRestartPlain;
  constexpr bool BIPOP = MODE == kRestartBipop;
  if (!f || !item_steps || !m || !sigma || !p_sigma || !p_c || !C || !A || !history || !best_x || !best_f || !num_restarts || !stop_flags || !sigma0 ||
      !lb || !ub || !thresholds_host)
    return EVOK_E_NULLPTR;
  if (separable ? (!s || (!X && (!m_draw || !s_draw))) : !X) return EVOK_E_NULLPTR;
  if (TIERED && (!tier || !tier_counts || !tier_history || !num_evaluations)) return EVOK_E_NULLPTR;
  if (BIPOP && (!bp.regime || !bp.large_tier || !bp.large_evaluations || !bp.small_evaluations || !bp.last_large_evaluations || !bp.run_stdev))
    return EVOK_E_NULLPTR;
  if (n_items < 0 || n_rows <= 0 || D <= 0 || H <= 0 || (X && (ldx < D || item_stride_x < 0)) || (item_stride_bounds != 0 && item_stride_bounds != D))
    return EVOK_E_BADSIZE;
  if (TIERED && (n_tiers < 1 || n_tiers > INT32_MAX)) return EVOK_E_BADSIZE;
  if (BIPOP && (bp.n_large < 1 || bp.n_large >= n_tiers || bp.popsize0 < 1 || bp.popsize0 > INT32_MAX)) return EVOK_E_BADSIZE;
  if (n_items == 0) return 0;
  RestartArgs a;
  a.f = f; a.X = X; a.item_stride_x = item_stride_x; a.ldx = ldx; a.m_draw = m_draw; a.s_draw = s_draw;
  a.draw_key = make_philox_key(draw_seed, 0);
  a.reset_key = make_philox_key(seed, 0);
  a.n_rows = n_rows; a.D = D; a.H = H; a.separable = separable != 0; a.maximize = maximize != 0;
  a.item_steps = reinterpret_cast<long long*>(item_steps);
  a.m = m; a.sigma = sigma; a.p_sigma = p_sigma; a.p_c = p_c; a.C = C; a.A = A; a.s = s; a.history = history; a.best_x = best_x; a.best_f = best_f;
  a.num_restarts = reinterpret_cast<long long*>(num_restarts);
  a.stop_flags = stop_flags;
  a.sigma0 = sigma0; a.lb = lb; a.ub = ub; a.item_stride_bounds = item_stride_bounds;
  a.tol_fun = thresholds_host[0]; a.tol_x = thresholds_host[1]; a.tol_x_up = thresholds_host[2]; a.max_condition = thresholds_host[3];
  a.min_fitness_stdev = thresholds_host[4]; a.max_generations = thresholds_host[5];
  a.tier = tier; a.tier_counts = tier_counts; a.tier_history = reinterpret_cast<const long long*>(tier_history); a.n_tiers = (int)n_tiers;
  a.num_evaluations = reinterpret_cast<long long*>(num_evaluations);
  a.regime = bp.regime; a.large_tier = bp.large_tier;
  a.large_evaluations = reinterpret_cast<long long*>(bp.large_evaluations);
  a.small_evaluations = reinterpret_cast<long long*>(bp.small_evaluations);
  a.last_large_evaluations = reinterpret_cast<long long*>(bp.last_large_evaluations);
  a.run_stdev = bp.run_stdev; a.n_large = (int)bp.n_large; a.popsize0 = (int)bp.popsize0;
  const int rc = for_item_chunks(n_items, (int64_t)INT32_MAX, [&](int64_t b0, int64_t nb) {
    RestartArgs c = a;
    const int64_t mat = separable ? D : D * D;
    c.f += b0 * n_rows;
    if (c.X) c.X += b0 * item_stride_x;
    if (c.m_draw) { c.m_draw += b0 * D; c.s_draw += b0 * D; }
    c.draw_key.stream_lo += (uint32_t)b0;
    c.reset_key.stream_lo += (uint32_t)b0;
    c.item_steps += b0; c.m += b0 * D; c.sigma += b0; c.p_sigma += b0 * D; c.p_c += b0 * D; c.C += b0 * mat; c.A += b0 * mat;
    if (c.s) c.s += b0 * D;
    c.history += b0 * H; c.best_x += b0 * D; c.best_f += b0; c.num_restarts += b0; c.stop_flags += b0; c.sigma0 += b0;
    c.lb += b0 * item_stride_bounds; c.ub += b0 * item_stride_bounds;
    if (TIERED) { c.tier += b0; c.num_evaluations += b0; }
    if (BIPOP) {
      c.regime += b0; c.large_tier += b0; c.large_evaluations += b0; c.small_evaluations += b0; c.last_large_evaluations += b0;
      c.run_stdev += b0;
    }
    cma_restart_kernel<MODE><<<(unsigned)nb, kRestartThreads, 0, (cudaStream_t)stream>>>(c);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
  if (rc || separable) return rc;
  const int64_t per_item = (D * D + kEyeThreads - 1) / kEyeThreads;
  const unsigned gx = (unsigned)(per_item < kEyeMaxBlocksPerItem ? per_item : kEyeMaxBlocksPerItem);
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    cma_restart_eye_kernel<<<dim3(gx, (unsigned)nb), kEyeThreads, 0, (cudaStream_t)stream>>>(stop_flags + b0, D, C + b0 * D * D, A + b0 * D * D);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_cma_restart_batched(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx, const float* m_draw,
                                                 const float* s_draw, uint64_t draw_seed, int64_t n_items, int64_t n_rows, int64_t D, int maximize,
                                                 int64_t* item_steps, float* m, float* sigma, float* p_sigma, float* p_c, float* C, float* A, float* s,
                                                 float* history, int64_t H, float* best_x, float* best_f, int64_t* num_restarts, int32_t* stop_flags,
                                                 const float* sigma0, const float* lb, const float* ub, int64_t item_stride_bounds,
                                                 const float* thresholds_host, uint64_t seed, void* stream) {
  return cma_restart_items<kRestartPlain>(separable, f, X, item_stride_x, ldx, m_draw, s_draw, draw_seed, n_items, n_rows, D, maximize, item_steps, m,
                                          sigma, p_sigma, p_c, C, A, s, history, H, best_x, best_f, num_restarts, stop_flags, sigma0, lb, ub,
                                          item_stride_bounds, thresholds_host, seed, nullptr, nullptr, nullptr, 0, nullptr, BipopArrays{}, stream);
}

extern "C" EVOK_API int evok_cma_restart_batched_tiered(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx,
                                                        const float* m_draw, const float* s_draw, uint64_t draw_seed, int64_t n_items, int64_t n_rows,
                                                        int64_t D, int maximize, int64_t* item_steps, float* m, float* sigma, float* p_sigma, float* p_c,
                                                        float* C, float* A, float* s, float* history, int64_t H, float* best_x, float* best_f,
                                                        int64_t* num_restarts, int32_t* stop_flags, const float* sigma0, const float* lb, const float* ub,
                                                        int64_t item_stride_bounds, const float* thresholds_host, uint64_t seed, int32_t* tier,
                                                        const int32_t* tier_counts, const int64_t* tier_history, int64_t n_tiers,
                                                        int64_t* num_evaluations, void* stream) {
  return cma_restart_items<kRestartTiered>(separable, f, X, item_stride_x, ldx, m_draw, s_draw, draw_seed, n_items, n_rows, D, maximize, item_steps, m,
                                           sigma, p_sigma, p_c, C, A, s, history, H, best_x, best_f, num_restarts, stop_flags, sigma0, lb, ub,
                                           item_stride_bounds, thresholds_host, seed, tier, tier_counts, tier_history, n_tiers, num_evaluations,
                                           BipopArrays{}, stream);
}

extern "C" EVOK_API int evok_cma_restart_batched_bipop(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx,
                                                       const float* m_draw, const float* s_draw, uint64_t draw_seed, int64_t n_items, int64_t n_rows,
                                                       int64_t D, int maximize, int64_t* item_steps, float* m, float* sigma, float* p_sigma, float* p_c,
                                                       float* C, float* A, float* s, float* history, int64_t H, float* best_x, float* best_f,
                                                       int64_t* num_restarts, int32_t* stop_flags, const float* sigma_def, const float* lb, const float* ub,
                                                       int64_t item_stride_bounds, const float* thresholds_host, uint64_t seed, int32_t* tier,
                                                       const int32_t* tier_counts, const int64_t* tier_history, int64_t n_tiers,
                                                       int64_t* num_evaluations, int32_t* regime, int32_t* large_tier, int64_t* large_evaluations,
                                                       int64_t* small_evaluations, int64_t* last_large_evaluations, float* run_stdev, int64_t n_large,
                                                       int64_t popsize0, void* stream) {
  const BipopArrays bp{regime, large_tier, large_evaluations, small_evaluations, last_large_evaluations, run_stdev, n_large, popsize0};
  return cma_restart_items<kRestartBipop>(separable, f, X, item_stride_x, ldx, m_draw, s_draw, draw_seed, n_items, n_rows, D, maximize, item_steps, m,
                                          sigma, p_sigma, p_c, C, A, s, history, H, best_x, best_f, num_restarts, stop_flags, sigma_def, lb, ub,
                                          item_stride_bounds, thresholds_host, seed, tier, tier_counts, tier_history, n_tiers, num_evaluations, bp,
                                          stream);
}
