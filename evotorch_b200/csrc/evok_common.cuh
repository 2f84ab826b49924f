// Shared helpers for libevok (sm_90a).  See include/evok.h for the ABI.  The device-only sampler helpers (Philox, warp sums,
// streaming accesses, the peer sink) are in evok_sampler.cuh, which NVRTC compiles too.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/evok.h"
#include "evok_sampler.cuh"

#define EVOK_CHECK_LAUNCH_N(n)                       \
  do {                                               \
    cudaError_t e__ = cudaPeekAtLastError();         \
    if (e__ != cudaSuccess) return (int)e__;         \
    evok::count_launches(n);                         \
  } while (0)
#define EVOK_CHECK_LAUNCH() EVOK_CHECK_LAUNCH_N(1)

namespace evok {

// number of kernels this library has launched (exposed as evok_launch_count(); bench.py reports it)
extern unsigned long long g_launch_count;
inline void count_launches(int n) { __atomic_fetch_add(&g_launch_count, (unsigned long long)n, __ATOMIC_RELAXED); }

constexpr int kWarp = 32;
constexpr int kNumSMs = 132;  // H100 SXM
// largest grid y / z: the batched entry points launch item chunks of at most this many items, one after another on the stream
constexpr int64_t kMaxGridY = 65535;

// fn(b0, nb) for the item chunks [b0, b0 + nb) of a batch, nb <= max_items, in order; returns the first non-zero code of fn
template <typename Fn>
inline int for_item_chunks(int64_t n_items, int64_t max_items, Fn&& fn) {
  for (int64_t b0 = 0; b0 < n_items; b0 += max_items) {
    const int rc = fn(b0, n_items - b0 < max_items ? n_items - b0 : max_items);
    if (rc) return rc;
  }
  return 0;
}

inline PhiloxKey make_philox_key(uint64_t seed, uint64_t stream_id) {
  PhiloxKey k;
  uint32_t a = (uint32_t)seed, b = (uint32_t)(seed >> 32) ^ (uint32_t)(stream_id >> 32);
  for (int r = 0; r < 10; ++r) {
    k.k0[r] = a;
    k.k1[r] = b;
    a += 0x9E3779B9u;
    b += 0xBB67AE85u;
  }
  k.stream_lo = (uint32_t)stream_id;
  return k;
}

// Sum over a whole CTA (blockDim.x multiple of 32, <= 1024).  Result valid in every thread.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem /* >= 33 entries */) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect smem reuse across consecutive calls
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  if (wid == 0) {
    T t = lane < nw ? smem[lane] : T(0);
    t = warp_sum(t);
    if (lane == 0) smem[32] = t;
  }
  __syncthreads();
  return smem[32];
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
__device__ __forceinline__ bool aligned16_dev(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// activations of the policy-forward kernels (tanh to ~1e-6 absolute: a 4-term odd polynomial below 0.25, (1 - e) / (1 + e) above)
__device__ __forceinline__ float tanh_1e6(float x) {
  const float ax = fabsf(x);
  float r;
  if (ax < 0.25f) {
    const float t = ax * ax;
    r = ax * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 0.021869488f, -0.053968254f), 0.13333334f), -0.33333334f), 1.0f);
  } else {
    const float e = __expf(-2.0f * ax);
    r = __fdividef(1.0f - e, 1.0f + e);
  }
  return copysignf(r, x);
}
// branch-free tanh = (1 - e) / (1 + e), e = exp(-2 |x|), with the hardware ex2 / rcp: 7 instructions, absolute error ~1e-7 (the RELATIVE
// error grows towards x = 0, where 1 - e cancels: use tanh_1e6 where that matters).  For the GEMM epilogue of the policy forward, where
// 128 activations per thread sit on the critical path of every tile.
__device__ __forceinline__ float tanh_abs1e7(float x) {
  const float e = __expf(-2.0f * fabsf(x));
  return copysignf(__fdividef(1.0f - e, 1.0f + e), x);
}
__device__ __forceinline__ float activate_fast(float v, int act) {
  switch (act) {
    case EVOK_ACT_TANH: return tanh_1e6(v);
    case EVOK_ACT_RELU: return fmaxf(v, 0.0f);
    case EVOK_ACT_SIGMOID: return __fdividef(1.0f, 1.0f + __expf(-v));
    default: return v;
  }
}

}  // namespace evok
