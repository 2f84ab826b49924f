// The device-only half of K1 / K2: Philox normals, the streaming stores, the peer-exchange sink, the objective accumulators
// and the sampling / evaluation kernels.  nvcc compiles it into libevok.so (evok_sample_eval.cu, with the built-in
// objectives) and NVRTC compiles it at run time with a user-defined accumulator (evotorch_b200/jit.py), so it has no host
// includes and no host code: under NVRTC the integer types come from the typedefs below.
#pragma once

#ifdef __CUDACC_RTC__
typedef signed char int8_t;
typedef unsigned char uint8_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
#endif

#include "../../include/evok.h"

namespace evok {

// ------------------------------------------------------------------------------------------------
// Peer exchange over NVLink (evok_peer.cu): where a producing kernel's result is needed by every GPU, the kernel itself
// stores it into every peer's buffer and the LAST CTA to finish raises this rank's flag in every peer's flag array.
// ------------------------------------------------------------------------------------------------
struct PeerSink {
  void* data[EVOK_MAX_PEERS];                 // peer p's destination buffer (this rank's own buffer at p == rank)
  unsigned long long* flags[EVOK_MAX_PEERS];  // peer p's flag array (one 64-bit epoch per source rank)
  int world, rank;
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// Call from ALL threads of EVERY CTA of a 1-D grid after the CTA's last peer store.  `epoch` (local) holds the number of
// completed exchanges; the flag value raised is epoch + 1 (the waiting kernel advances `epoch`).  `done` is a local counter
// that returns to 0 for the next launch.
static __device__ __noinline__ void peer_signal_tail(const PeerSink& s, const unsigned long long* epoch, unsigned int* done) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();  // this CTA's peer stores are visible system-wide before the counter moves
    const unsigned int prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {
      *done = 0;
      __threadfence_system();
      const unsigned long long e = *epoch + 1ull;
      for (int p = 0; p < s.world; ++p) st_release_sys(s.flags[p] + s.rank, e);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11).  One call -> 4 x 32 random bits.
// ------------------------------------------------------------------------------------------------
struct U4 {
  uint32_t x, y, z, w;
};

// The 10 round keys of one (seed, stream) pair, precomputed on the host and passed to the kernels BY VALUE: they live in
// the constant bank, so each round's key XOR takes its operand straight from c[][] (no per-thread key-schedule adds).
struct PhiloxKey {
  uint32_t k0[10], k1[10];
  uint32_t stream_lo;
};

// EVOK_PHILOX_ROUNDS exists for MEASUREMENT builds only (scripts/build_variants.py: what would fewer rounds buy?); the
// product is Philox4x32-10, the variant cuRAND / torch use, and the oracle restates exactly that.
#ifndef EVOK_PHILOX_ROUNDS
#define EVOK_PHILOX_ROUNDS 10
#endif
__device__ __forceinline__ U4 philox4x32_10(U4 c, const PhiloxKey& key) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#pragma unroll
  for (int r = 0; r < EVOK_PHILOX_ROUNDS; ++r) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    U4 n;
    n.x = hi1 ^ c.y ^ key.k0[r];
    n.y = lo1;
    n.z = hi0 ^ c.w ^ key.k1[r];
    n.w = lo0;
    c = n;
  }
  return c;
}

__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ float lg2_approx(float x) {
  float r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// Box-Muller on 32+32 random bits -> two standard normals.
//   u1 = 2^-33 + a * 2^-32 in (0, 1]  (never 0, so the log is finite);  r = sqrt(-2 ln u1) = sqrt(lg2(u1) * (-2 ln 2))
//   theta = 2 pi (2^-33 + b * 2^-32): the 2 pi is folded into the conversion constants.
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float u1 = fmaf((float)a, 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  const float th = fmaf((float)b, 1.4629180792671596e-09f, 7.314590396335798e-10f);
  const float r = sqrt_approx(lg2_approx(u1) * -1.3862943611198906f);
  float s, c;
  __sincosf(th, &s, &c);
  z0 = r * c;
  z1 = r * s;
}

// The four standard normals of (unit, column group q): `unit` is the GLOBAL direction index (symmetric
// sampling: rows 2*unit and 2*unit+1) or the global row index (non-symmetric); columns 4q .. 4q+3.
// `stream_word` = low 32 bits of the stream id (key.stream_lo plus an optional device-side generation offset, which lets a
// CUDA graph that was captured once draw a fresh population on every replay)
__device__ __forceinline__ void normals4(const PhiloxKey& key, uint32_t stream_word, uint64_t unit, uint32_t q, float z[4]) {
  U4 c;
  c.x = q;
  c.y = (uint32_t)unit;
  c.z = (uint32_t)(unit >> 32);
  c.w = stream_word;
  const U4 r = philox4x32_10(c, key);
  box_muller(r.x, r.y, z[0], z[1]);
  box_muller(r.z, r.w, z[2], z[3]);
}

// ------------------------------------------------------------------------------------------------
// Noise: the draws of rand() / randn() in a generated accumulator, on the key and stream word of the population's own draw.
// Occurrence k of the source (0 .. 3 in the element terms, 4 .. 7 in `value`) at global row `row` takes Philox counter
//   c = (x, (uint32)row, 0x80000000 | k << 24 | (row >> 32) & 0xFFFFFF, stream word),
// x = the column group q = j >> 2 of an element occurrence at column j, 0xFFFFFFFF for one in `value`.  A sample counter
// (normals4) has c.z = unit >> 32 < 2^31, so no noise counter equals a sample counter, on any path.
// rand() is (word >> 8) * 2^-24 in [0, 1), exact in float32; randn() is box_muller of the sampler.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ U4 noise_bits(const PhiloxKey& key, uint32_t stream_word, uint64_t row, uint32_t x, int k) {
  U4 c;
  c.x = x;
  c.y = (uint32_t)row;
  c.z = 0x80000000u | ((uint32_t)k << 24) | ((uint32_t)(row >> 32) & 0xFFFFFFu);
  c.w = stream_word;
  return philox4x32_10(c, key);
}
__device__ __forceinline__ float uniform24(uint32_t w) { return (float)(w >> 8) * 5.9604644775390625e-08f; }

// element occurrence k at the 4 columns of group q: rand() takes word c for column 4q + c; randn() the normals4 layout
// (columns 4q, 4q + 1 from (x, y), 4q + 2, 4q + 3 from (z, w))
__device__ __forceinline__ void noise4(const PhiloxKey& key, uint32_t stream_word, uint64_t row, uint32_t q, int k, bool normal, float u[4]) {
  const U4 r = noise_bits(key, stream_word, row, q, k);
  if (normal) {
    box_muller(r.x, r.y, u[0], u[1]);
    box_muller(r.z, r.w, u[2], u[3]);
  } else {
    u[0] = uniform24(r.x); u[1] = uniform24(r.y); u[2] = uniform24(r.z); u[3] = uniform24(r.w);
  }
}
// the same draw for column j alone (one call, one word or one word pair): entry j & 3 of noise4 for group j >> 2
__device__ __forceinline__ float noise1(const PhiloxKey& key, uint32_t stream_word, uint64_t row, int64_t j, int k, bool normal) {
  const U4 r = noise_bits(key, stream_word, row, (uint32_t)(j >> 2), k);
  const int c = (int)(j & 3);
  if (normal) {
    float z0, z1;
    box_muller(c < 2 ? r.x : r.z, c < 2 ? r.y : r.w, z0, z1);
    return (c & 1) ? z1 : z0;
  }
  return uniform24(c == 0 ? r.x : c == 1 ? r.y : c == 2 ? r.z : r.w);
}
// occurrence k of `value`: rand() takes word x, randn() z0 of box_muller(x, y)
__device__ __forceinline__ float value_rand(const PhiloxKey& key, uint32_t stream_word, uint64_t row, int k) {
  return uniform24(noise_bits(key, stream_word, row, 0xFFFFFFFFu, k).x);
}
__device__ __forceinline__ float value_randn(const PhiloxKey& key, uint32_t stream_word, uint64_t row, int k) {
  const U4 r = noise_bits(key, stream_word, row, 0xFFFFFFFFu, k);
  float z0, z1;
  box_muller(r.x, r.y, z0, z1);
  return z0;
}

// ------------------------------------------------------------------------------------------------
// Warp reductions
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The other reductions of a generated accumulator (products, maxima, minima): the butterfly of warp_sum with another combine,
// in the same xor order, so every lane ends with the same, reproducible bits.  max / min propagate NaN (max.NaN / min.NaN: a
// NaN operand gives NaN, as torch.amax / amin do; fmaxf / fminf would drop it).
__device__ __forceinline__ float inf() { return __int_as_float(0x7f800000); }
__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float min_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float warp_prod(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v *= __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// streaming 128-bit accesses: the population is touched once per kernel, keep it out of L1
__device__ __forceinline__ float4 ld_stream4(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_stream1(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream4(float* p, float a, float b, float c, float d) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void st_stream1(float* p, float a) {
  asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory");
}

// ------------------------------------------------------------------------------------------------
// Objective accumulators.  An accumulator is a type with
//   Acc(D)      : a fresh accumulator for one row of D columns (one per row and lane);
//   add(x, j)   : fold element x of column j (0-based, global) into this lane's partial sums;
//   finish(D)   : warp-reduce the partials and return the fitness of the row (every lane gets it; lane 0 stores it).
// A row's elements reach add() in no fixed column order (strided over the lanes of a warp), so an accumulator holds
// reductions with an associative combine: sums, and in a generated one also products, maxima and minima (warp_prod / _max /
// _min), each slot starting from its combine's identity.
// The built-in ones are ObjAcc<EVOK_OBJ_*>; a user-defined one is generated by evotorch_b200/jit.py and may declare optional
// markers, each of which adds calls or arguments:
//   kPairs = true (pair terms):
//     add_pair(x, xn, j)  : fold the neighbour pair (x_j, x_{j+1}); it is called exactly once for every j in [0, D-2] of a
//                           row, by the lane that holds column j+1, also in no fixed order across lanes (fold_pairs).
//   kRunning = true, kRunningSums = R <= 2 (running sums c_j = sum_{k<=j} h(x_k, k)):
//     running(x, j, h)    : h[i] = the increment of running sum i at column j;
//     add(x, j, r)        : the element fold takes r last, r[i] = c_j of running sum i (fold_running computes it).
//   kData = true, kVectors (data: float32 vectors of the row length and scalars, bound per launch):
//     Acc(D, binding)     : the constructor takes the DataBinding of the launch's item, keeps `const float* vec[]` (the vectors)
//                           and loads the scalars.
//   kNoise = true, kDraws <= 4, kNormalDraws (rand() / randn(): kDraws occurrences in the element terms, bit k of kNormalDraws
//   set where occurrence k is randn(), and up to 4 in `value`):
//     finish(D, key, stream_word, row) : row = the global row index; `value` draws with value_rand / value_randn.
//   kTransform = true (terms of the transformed row y = M (x - o)): every fold takes the entry of y at the same column after
//   that of x, add(x, y, j, ...), add_pair(x, xn, y, yn, j, ...), running(x, y, j, ...).  The kernels carry a column as XY (ColVal)
//   and only the transformed evaluation kernels below instantiate such an accumulator.
// An accumulator with data vectors or element draws takes the column entries of a fold after j (DataCols: d[i] = vec[i][j],
// then d[kVectors + k] = element draw k at column j), in every fold, whether its terms use them or not:
//   add(x, j, d[, r]),  running(x, j, d, h),  add_pair(x, xn, j, d, dn)  with dn the entries at column j + 1.
// AccTraits reads the markers, and the acc_* functions below are the only calls into an accumulator: the kernels hand every
// fold the column entries, every finish the row's draw, and never depend on which of these signatures an accumulator has.
// ------------------------------------------------------------------------------------------------
template <int OBJ>
struct ObjAcc;

template <>
struct ObjAcc<EVOK_OBJ_NONE> {
  __device__ __forceinline__ explicit ObjAcc(int64_t) {}
  __device__ __forceinline__ void add(float, int64_t) {}
  __device__ __forceinline__ float finish(int64_t) { return 0.f; }
};
template <>
struct ObjAcc<EVOK_OBJ_SPHERE> {
  __device__ __forceinline__ explicit ObjAcc(int64_t) {}
  float s2 = 0.f;
  __device__ __forceinline__ void add(float x, int64_t) { s2 = fmaf(x, x, s2); }
  __device__ __forceinline__ float finish(int64_t) { return warp_sum(s2); }
};
template <>
struct ObjAcc<EVOK_OBJ_RASTRIGIN> {
  __device__ __forceinline__ explicit ObjAcc(int64_t) {}
  float s2 = 0.f, sc = 0.f;
  __device__ __forceinline__ void add(float x, int64_t) {
    s2 = fmaf(x, x, s2);
    sc += __cosf(6.2831853071795865f * x);
  }
  __device__ __forceinline__ float finish(int64_t D) {
    const float a = warp_sum(s2), c = warp_sum(sc);
    return fmaf(-10.f, c, a) + 10.f * (float)D;
  }
};
template <>
struct ObjAcc<EVOK_OBJ_ACKLEY> {
  __device__ __forceinline__ explicit ObjAcc(int64_t) {}
  float s2 = 0.f, sc = 0.f;
  __device__ __forceinline__ void add(float x, int64_t) {
    s2 = fmaf(x, x, s2);
    sc += __cosf(6.2831853071795865f * x);
  }
  __device__ __forceinline__ float finish(int64_t D) {
    const float a = warp_sum(s2), c = warp_sum(sc);
    const float invD = 1.0f / (float)D;
    return -20.f * expf(-0.2f * sqrtf(a * invD)) - expf(c * invD) + 20.f + 2.718281828459045f;
  }
};

// The data of one launch of an objective with data terms: p[i] is data name i of the launch's first item and item_stride[i]
// the distance in floats to the next item's (0: shared by all items; only the batched sampler has more than one item).  It is
// a kernel argument, so two objectives of one source in flight on two streams, or captured in two graphs, never share it.
struct DataBinding {
  const float* p[EVOK_MAX_DATA];
  int64_t item_stride[EVOK_MAX_DATA];
};
struct NoData {};

// The draw of the rows that eval_kernel evaluates, its last argument for an accumulator with noise: row r of X is global row
// row0 + r, on stream word key.stream_lo + *stream_off (stream_off may be null)
struct EvalKey {
  PhiloxKey key;
  const uint32_t* stream_off;
  int64_t row0;
};

// tunables (build-time, for measurement builds: scripts/build_variants.py, scripts/kbench.py)
#ifndef EVOK_SAMPLE_THREADS
#define EVOK_SAMPLE_THREADS 256
#endif
#ifndef EVOK_SAMPLE_MINB
#define EVOK_SAMPLE_MINB 3
#endif
#ifndef EVOK_SAMPLE_UNR
#define EVOK_SAMPLE_UNR 2
#endif
#ifndef EVOK_SAMPLEONLY_MINB
#define EVOK_SAMPLEONLY_MINB 5
#endif
#ifndef EVOK_SAMPLEONLY_UNR
#define EVOK_SAMPLEONLY_UNR 1
#endif

// One optional marker of an accumulator: whether it is declared (and true), and the counts declared with it.  Every marker is
// read with one idiom: the first overload exists only when Acc declares the marker, and the argument 0 prefers its int
// parameter to the second overload's long.
struct Marker {
  bool on = false;
  int n = 0;
  unsigned mask = 0u;
};
template <typename A> constexpr auto pairs_marker(int) -> decltype(Marker{A::kPairs}) { return {A::kPairs}; }
template <typename A> constexpr Marker pairs_marker(long) { return {}; }
template <typename A> constexpr auto running_marker(int) -> decltype(Marker{A::kRunning}) { return {A::kRunning, A::kRunningSums}; }
template <typename A> constexpr Marker running_marker(long) { return {}; }
template <typename A> constexpr auto data_marker(int) -> decltype(Marker{A::kData}) { return {A::kData, A::kVectors}; }
template <typename A> constexpr Marker data_marker(long) { return {}; }
template <typename A> constexpr auto noise_marker(int) -> decltype(Marker{A::kNoise}) { return {A::kNoise, A::kDraws, A::kNormalDraws}; }
template <typename A> constexpr Marker noise_marker(long) { return {}; }
template <typename A> constexpr auto transform_marker(int) -> decltype(Marker{A::kTransform}) { return {A::kTransform}; }
template <typename A> constexpr Marker transform_marker(long) { return {}; }
// ObjAcc<EVOK_OBJ_NONE> samples without evaluating
template <typename A> constexpr bool sample_only(const A*) { return false; }
constexpr bool sample_only(const ObjAcc<EVOK_OBJ_NONE>*) { return true; }

template <bool B, typename T, typename F>
struct Pick {
  using type = F;
};
template <typename T, typename F>
struct Pick<true, T, F> {
  using type = T;
};

// one column of a row and of its transformed row y = M (x - o), for an accumulator with kTransform
struct XY {
  float x, y;
};
__device__ __forceinline__ float shfl_col(float v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ XY shfl_col(XY v, int src) { return {__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src)}; }

// Every compile-time fact about an accumulator that the kernels use.  Each feature's code is under `if constexpr` on its
// fact, so the kernels of an accumulator without it are those of one written without the feature.
template <typename Acc>
struct AccTraits {
  static constexpr Marker kPairMark = pairs_marker<Acc>(0), kRunMark = running_marker<Acc>(0), kDataMark = data_marker<Acc>(0),
                          kNoiseMark = noise_marker<Acc>(0);
  static constexpr bool kSampleOnly = sample_only(static_cast<const Acc*>(nullptr));
  static constexpr bool kPairs = kPairMark.on;
  static constexpr bool kRunning = kRunMark.on;
  static constexpr int kRunningSums = kRunning ? kRunMark.n : 0;
  static constexpr bool kData = kDataMark.on;
  static constexpr int kVectors = kData ? kDataMark.n : 0;
  static constexpr bool kNoise = kNoiseMark.on;
  static constexpr int kDraws = kNoise ? kNoiseMark.n : 0;  // element draws (those of `value` are the accumulator's own)
  static constexpr unsigned kNormal = kNoise ? kNoiseMark.mask : 0u;
  static constexpr bool kTransform = transform_marker<Acc>(0).on;
  // what a fold takes for one column: its x, or (x, y) with a transform
  using ColVal = typename Pick<kTransform, XY, float>::type;
  // element draws: the + and - rows of a direction fold with their own column entries
  static constexpr bool kElementDraws = kDraws > 0;
  // the folds take column entries (data vectors, then element draws), kSlots of them per column
  static constexpr bool kCols = kData || kElementDraws;
  static constexpr int kSlots = kVectors + kDraws > 0 ? kVectors + kDraws : 1;
  // the kernels take warp-uniform steps of 32 lanes (pair folds and running sums shuffle across lanes)
  static constexpr bool kWarpSteps = kPairs || kRunning;
  // Launch bounds.  The fused samplers are issue/XU bound (two independent Philox chains per lane help); the sample-only kernel
  // is store bound and prefers occupancy.  Running sums, and more than one element draw per column, run one Philox chain per
  // lane, the latter at 2 CTAs per SM, so that no kernel spills.  eval_kernel of an accumulator with noise has 2 CTAs per SM:
  // without a bound ptxas fits the kernel of a `value` draw with few element terms into 32 registers and spills.
  static constexpr int kSampleUnroll = kSampleOnly ? EVOK_SAMPLEONLY_UNR : kRunning || kDraws > 1 ? 1 : EVOK_SAMPLE_UNR;
  static constexpr int kSampleMinBlocks = kSampleOnly ? EVOK_SAMPLEONLY_MINB : kDraws > 1 ? 2 : EVOK_SAMPLE_MINB;
  static constexpr int kEvalMinBlocks = kNoise ? 2 : 0;
  // the last argument of the sampling kernels, and of eval_kernel (empty structs for an accumulator without data / noise)
  using DataArg = typename Pick<kData, DataBinding, NoData>::type;
  using EvalArg = typename Pick<kNoise, EvalKey, NoData>::type;
};

// The accumulator calls.  d / dn are the column entries of a fold (a row of DataCols), r / h the running sums and their
// increments, (key, sw, row) the draw of the row; each function passes on what the accumulator's signature takes.
template <typename Acc, typename Arg>
__device__ __forceinline__ Acc acc_make(int64_t D, const Arg& data) {
  if constexpr (AccTraits<Acc>::kData) return Acc(D, data);
  else return Acc(D);
}
// x: the column's ColVal, (x, y) with a transform.
template <typename Acc, typename... Run>
__device__ __forceinline__ void acc_add(Acc& acc, typename AccTraits<Acc>::ColVal x, int64_t j, const float (&d)[AccTraits<Acc>::kSlots],
                                        const Run&... r) {
  if constexpr (AccTraits<Acc>::kTransform) {
    if constexpr (AccTraits<Acc>::kCols) acc.add(x.x, x.y, j, d, r...);
    else acc.add(x.x, x.y, j, r...);
  } else if constexpr (AccTraits<Acc>::kCols) acc.add(x, j, d, r...);
  else acc.add(x, j, r...);
}
template <typename Acc>
__device__ __forceinline__ void acc_pair(Acc& acc, typename AccTraits<Acc>::ColVal x, typename AccTraits<Acc>::ColVal xn, int64_t j,
                                         const float (&d)[AccTraits<Acc>::kSlots], const float (&dn)[AccTraits<Acc>::kSlots]) {
  if constexpr (AccTraits<Acc>::kTransform) {
    if constexpr (AccTraits<Acc>::kCols) acc.add_pair(x.x, xn.x, x.y, xn.y, j, d, dn);
    else acc.add_pair(x.x, xn.x, x.y, xn.y, j);
  } else if constexpr (AccTraits<Acc>::kCols) acc.add_pair(x, xn, j, d, dn);
  else acc.add_pair(x, xn, j);
}
template <typename Acc, int R>
__device__ __forceinline__ void acc_running(Acc& acc, typename AccTraits<Acc>::ColVal x, int64_t j, const float (&d)[AccTraits<Acc>::kSlots],
                                            float (&h)[R]) {
  if constexpr (AccTraits<Acc>::kTransform) {
    if constexpr (AccTraits<Acc>::kCols) acc.running(x.x, x.y, j, d, h);
    else acc.running(x.x, x.y, j, h);
  } else if constexpr (AccTraits<Acc>::kCols) acc.running(x, j, d, h);
  else acc.running(x, j, h);
}
// key: null for an accumulator without noise (eval_kernel has no draw then)
template <typename Acc>
__device__ __forceinline__ float acc_finish(Acc& acc, int64_t D, const PhiloxKey* key, uint32_t sw, uint64_t row) {
  if constexpr (AccTraits<Acc>::kNoise) return acc.finish(D, *key, sw, row);
  else return acc.finish(D);
}

// the carries of one row along warp-uniform steps: the last column of the previous step (pair terms) and the running sums of
// all columns of the previous steps
template <typename Acc>
struct StepCarry {
  typename AccTraits<Acc>::ColVal pair{};
  float run[AccTraits<Acc>::kRunningSums > 0 ? AccTraits<Acc>::kRunningSums : 1] = {};
};

__device__ __forceinline__ NoData item_data(const NoData& d, int64_t) { return d; }
__device__ __forceinline__ DataBinding item_data(DataBinding d, int64_t item) {
#pragma unroll
  for (int i = 0; i < EVOK_MAX_DATA; ++i) d.p[i] += item * d.item_stride[i];
  return d;
}

// The column entries of the N columns a lane holds in one step: v[c] = the entries of column c of the step, the data vectors'
// vec[i][column] read through the read-only cache (a D-vector is re-read by every row, so it stays in L1 / L2), then the element
// draws.  One load serves the + and the - row of a symmetric pair.  `left` holds the data entries at the column before the
// first (the left neighbour of a pair fold across lanes).  Without data vectors and element draws nothing is loaded or drawn.
template <typename Acc, int N>
struct DataCols {
  static constexpr int kVectors = AccTraits<Acc>::kVectors, kDraws = AccTraits<Acc>::kDraws;
  float v[N][AccTraits<Acc>::kSlots], left[AccTraits<Acc>::kSlots];
  // columns j .. j + 3 with one 16-byte load per vector: the vectorised kernels, which the host picks only when every vector is
  // 16-byte aligned (choose_kernel)
  __device__ __forceinline__ void load4(const Acc& acc, int64_t j) {
    static_assert(N == 4, "a column group is 4 columns");
    if constexpr (kVectors > 0)  // an accumulator without data vectors has no `vec`
#pragma unroll
    for (int i = 0; i < kVectors; ++i) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(acc.vec[i] + j));
      v[0][i] = t.x; v[1][i] = t.y; v[2][i] = t.z; v[3][i] = t.w;
    }
  }
  __device__ __forceinline__ void load1(const Acc& acc, int64_t j, int c) {  // column j into slot c
    if constexpr (kVectors > 0)
#pragma unroll
    for (int i = 0; i < kVectors; ++i) v[c][i] = __ldg(acc.vec[i] + j);
  }
  __device__ __forceinline__ void load_left(const Acc& acc, int64_t j) {  // column j - 1, j > 0
    if constexpr (kVectors > 0)
#pragma unroll
    for (int i = 0; i < kVectors; ++i) left[i] = __ldg(acc.vec[i] + j - 1);
  }
  // the element draws of global row `row` at the columns of group q (one Philox call per occurrence), after the data entries
  __device__ __forceinline__ void draw4(const PhiloxKey& key, uint32_t sw, uint64_t row, uint32_t q) {
    static_assert(N == 4, "a column group is 4 columns");
#pragma unroll
    for (int k = 0; k < kDraws; ++k) {
      float u[4];
      noise4(key, sw, row, q, k, (AccTraits<Acc>::kNormal >> k) & 1u, u);
      v[0][kVectors + k] = u[0]; v[1][kVectors + k] = u[1]; v[2][kVectors + k] = u[2]; v[3][kVectors + k] = u[3];
    }
  }
  __device__ __forceinline__ void draw1(const PhiloxKey& key, uint32_t sw, uint64_t row, int64_t j, int c) {  // column j into slot c
#pragma unroll
    for (int k = 0; k < kDraws; ++k) v[c][kVectors + k] = noise1(key, sw, row, j, k, (AccTraits<Acc>::kNormal >> k) & 1u);
  }
};

// One warp step of pair folds: this lane holds the N consecutive columns j .. j+N-1 of a row (v[]), of which the first
// n_valid exist (0 for a lane past the row's end).  The lane holding column c + 1 folds (x_c, x_{c+1}): inside v[] from
// registers, and for its first column with x_{j-1} = the last column of lane - 1, or for lane 0 the last column lane 31
// held in the previous step of the same row (`carry`, zero-initialised per row and advanced here).  Every lane of the warp
// must call it on every step, in the same order (it shuffles); a column's left neighbour is always in the previous lane
// or the previous step because each step covers 32 * N consecutive columns.
// dc: the column entries of the same columns (with `left` loaded when j > 0).
template <int N, typename Acc, typename V>
__device__ __forceinline__ void fold_pairs(Acc& acc, const V (&v)[N], int64_t j, int n_valid, V& carry, const DataCols<Acc, N>& dc) {
  const int lane = threadIdx.x & 31;
  const V rot = shfl_col(v[N - 1], (lane + 31) & 31);  // lane 0 receives lane 31's: next step's carry
  const V left = lane == 0 ? carry : rot;
  carry = rot;
  if (n_valid > 0 && j > 0) acc_pair(acc, left, v[0], j - 1, dc.left, dc.v[0]);
#pragma unroll
  for (int c = 1; c < N; ++c)
    if (c < n_valid) acc_pair(acc, v[c - 1], v[c], j + c - 1, dc.v[c - 1], dc.v[c]);
}

// One warp step of the element folds of an accumulator with running sums, in the layout of fold_pairs (this lane holds the
// columns j .. j+N-1, of which the first n_valid exist; every lane calls it on every step, in increasing column order).  For
// each running sum: the lane evaluates the increments h of its columns (0 past the row's end), forms their inclusive prefix
// p_c, and takes the exclusive scan e of the lane totals p_{N-1} across the warp (a Kogge-Stone scan with __shfl_up_sync, five
// rounds, then one shift); then c_{j+c} = p_c + (e + carry), where carry is the sum of all earlier steps of the row, and the
// carry advances by the step total, the inclusive scan of lane 31.  Then each column's element terms are folded with its c.
template <int N, typename Acc, typename V, int R>
__device__ __forceinline__ void fold_running(Acc& acc, const V (&v)[N], int64_t j, int n_valid, float (&carry)[R], const DataCols<Acc, N>& dc) {
  const int lane = threadIdx.x & 31;
  float p[N][R];
#pragma unroll
  for (int c = 0; c < N; ++c) {
    float h[R];
#pragma unroll
    for (int i = 0; i < R; ++i) h[i] = 0.f;
    if (c < n_valid) acc_running(acc, v[c], j + c, dc.v[c], h);
#pragma unroll
    for (int i = 0; i < R; ++i) p[c][i] = c == 0 ? h[i] : p[c - 1][i] + h[i];
  }
#pragma unroll
  for (int i = 0; i < R; ++i) {
    float incl = p[N - 1][i];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    const float total = __shfl_sync(0xffffffffu, incl, 31);
    const float base = lane == 0 ? carry[i] : excl + carry[i];
#pragma unroll
    for (int c = 0; c < N; ++c) p[c][i] += base;
    carry[i] += total;
  }
#pragma unroll
  for (int c = 0; c < N; ++c)
    if (c < n_valid) acc_add(acc, v[c], j + c, dc.v[c], p[c]);
}

// the element folds and pair folds of one warp step (see fold_pairs and fold_running): the element folds of an accumulator
// without running sums have been made by the caller already
template <int N, typename Acc, typename V>
__device__ __forceinline__ void fold_step(Acc& acc, const V (&v)[N], int64_t j, int n_valid, StepCarry<Acc>& carry, const DataCols<Acc, N>& dc) {
  if constexpr (AccTraits<Acc>::kRunning) fold_running<N>(acc, v, j, n_valid, carry.run, dc);
  if constexpr (AccTraits<Acc>::kPairs) fold_pairs<N>(acc, v, j, n_valid, carry.pair, dc);
}

// ------------------------------------------------------------------------------------------------
// K1 / K2 kernels.  HBM-bound design: one warp owns one direction (a +/- row pair) or one row; every lane produces 4
// consecutive columns per step from ONE Philox4x32-10 call, writes them with 128-bit streaming stores (512 contiguous bytes
// per warp-row) and folds them into the objective accumulators while they are still in registers, so the population is
// written once and never re-read for evaluation.
// ------------------------------------------------------------------------------------------------
constexpr int kSampleThreads = EVOK_SAMPLE_THREADS;

// the column entries the - row of a direction folds with: its own (dm) when the element terms draw noise, else the + row's
template <typename Acc, typename Cols>
__device__ __forceinline__ const Cols& minus_cols(const Cols& dp, const Cols& dm) {
  if constexpr (AccTraits<Acc>::kElementDraws) return dm;
  else return dp;
}

// the element draws of unit `unit` at column group q: its row (the + row, global row 2 unit, of a direction) into dp, and the
// - row's (2 unit + 1) into dm, which takes dp's data entries first
template <typename Acc, bool SYM, typename Cols>
__device__ __forceinline__ void draw_rows(Cols& dp, Cols& dm, const PhiloxKey& key, uint32_t sw, uint64_t unit, uint32_t q) {
  if constexpr (AccTraits<Acc>::kElementDraws) {
    const uint64_t row = SYM ? 2 * unit : unit;
    if (SYM) {
      dm = dp;
      dm.draw4(key, sw, row + 1, q);
    }
    dp.draw4(key, sw, row, q);
  }
}

// One column group (4 columns) of one unit: sample, store, fold.  SQ: also *zsq += z^2 (the unscaled normals; the squared norm
// that separable CMA-ES's active reweighting needs), in column order.
// An accumulator without warp steps folds each element as it is sampled; `active` and the carries are not used.  One with warp
// steps is called by EVERY lane of the warp on every step (fold_step shuffles): a lane whose group lies past the row's end
// (!active) draws, loads and stores nothing and folds nothing.  Its samples and element folds are the same, in the same order
// (with running sums the element folds come after the scan, in fold_running); the + and - rows have their own neighbours and
// carries.
template <typename Acc, bool SYM, bool STORE, bool VEC, bool SQ>
__device__ __forceinline__ void sample_group(const PhiloxKey& key, uint32_t sw, uint64_t unit, uint32_t q, int64_t D,
                                             const float* __restrict__ mu, const float* __restrict__ sigma, float* xp, float* xm,
                                             Acc& accp, Acc& accm, float* zsq, bool active, StepCarry<Acc>& carry_p,
                                             StepCarry<Acc>& carry_m) {
  using T = AccTraits<Acc>;
  constexpr bool kFoldNow = !T::kRunning;  // element terms without running sums fold as they are sampled
  float p[4] = {0.f, 0.f, 0.f, 0.f}, n[4] = {0.f, 0.f, 0.f, 0.f};
  const int64_t j = (int64_t)q << 2;
  int n_valid = 0;
  DataCols<Acc, 4> dc, dm;  // dm: the - row's entries, with its own draws (element noise only)
  const auto& dcm = minus_cols<Acc>(dc, dm);
  if (!T::kWarpSteps || active) {  // a compile-time true without warp steps
    float z[4];
    normals4(key, sw, unit, q, z);
    if (VEC) {
      if (SQ) {
        *zsq = fmaf(z[0], z[0], *zsq); *zsq = fmaf(z[1], z[1], *zsq); *zsq = fmaf(z[2], z[2], *zsq); *zsq = fmaf(z[3], z[3], *zsq);
      }
      const float4 m = __ldg(reinterpret_cast<const float4*>(mu + j));
      const float4 s = __ldg(reinterpret_cast<const float4*>(sigma + j));
      p[0] = fmaf(s.x, z[0], m.x); p[1] = fmaf(s.y, z[1], m.y); p[2] = fmaf(s.z, z[2], m.z); p[3] = fmaf(s.w, z[3], m.w);
      if (STORE) st_stream4(xp + j, p[0], p[1], p[2], p[3]);
      dc.load4(accp, j);
      draw_rows<Acc, SYM>(dc, dm, key, sw, unit, q);
      if constexpr (kFoldNow) {
        acc_add(accp, p[0], j, dc.v[0]); acc_add(accp, p[1], j + 1, dc.v[1]); acc_add(accp, p[2], j + 2, dc.v[2]); acc_add(accp, p[3], j + 3, dc.v[3]);
      }
      if (SYM) {
        n[0] = fmaf(-s.x, z[0], m.x); n[1] = fmaf(-s.y, z[1], m.y); n[2] = fmaf(-s.z, z[2], m.z); n[3] = fmaf(-s.w, z[3], m.w);
        if (STORE) st_stream4(xm + j, n[0], n[1], n[2], n[3]);
        if constexpr (kFoldNow) {
          acc_add(accm, n[0], j, dcm.v[0]); acc_add(accm, n[1], j + 1, dcm.v[1]); acc_add(accm, n[2], j + 2, dcm.v[2]); acc_add(accm, n[3], j + 3, dcm.v[3]);
        }
      }
      n_valid = 4;
    } else {
      draw_rows<Acc, SYM>(dc, dm, key, sw, unit, q);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (j + c < D) {
          if (SQ) *zsq = fmaf(z[c], z[c], *zsq);
          const float m = __ldg(mu + j + c), s = __ldg(sigma + j + c);
          p[c] = fmaf(s, z[c], m);
          if (STORE) st_stream1(xp + j + c, p[c]);
          dc.load1(accp, j + c, c);
          if constexpr (kFoldNow) acc_add(accp, p[c], j + c, dc.v[c]);
          if (SYM) {
            n[c] = fmaf(-s, z[c], m);
            if (STORE) st_stream1(xm + j + c, n[c]);
            if constexpr (T::kElementDraws) dm.load1(accp, j + c, c);
            if constexpr (kFoldNow) acc_add(accm, n[c], j + c, dcm.v[c]);
          }
        }
      }
      n_valid = D - j < 4 ? (int)(D - j) : 4;  // the partial last group: a pair is folded only where column j + 1 < D
    }
  }
  if constexpr (T::kWarpSteps) {
    if constexpr (T::kPairs)
      if (n_valid > 0 && j > 0) {
        dc.load_left(accp, j);
        if constexpr (T::kElementDraws) dm.load_left(accp, j);
      }
    fold_step<4>(accp, p, j, n_valid, carry_p, dc);
    if (SYM) fold_step<4>(accm, n, j, n_valid, carry_m, dcm);
  }
}

// One unit u (a direction of symmetric sampling, else a row) of the warp of lane `lane`: sample its row(s) from (key, stream word sw, unit
// unit0 + u), store them at row r = (SYM ? 2u : u) of X when STORE, fold them into the objective and store the fitness at f[r]
// (or, PUSH, at row0 + r of every peer's vector); SQ: q_out[r] = sum of z^2; data: the binding of an accumulator with data terms.  The body of sample_eval_kernel and of
// sample_eval_batched_kernel, so both give the same bits for the same operands and counters.
template <typename Acc, bool SYM, bool STORE, bool VEC, bool PUSH, bool SQ>
__device__ __forceinline__ void sample_eval_unit(int lane, float* __restrict__ X, int64_t ldx, const float* __restrict__ mu,
                                                 const float* __restrict__ sigma, int64_t row0, int64_t u, int64_t D, const PhiloxKey& key, uint32_t sw,
                                                 uint32_t nq, uint64_t unit0, float* __restrict__ f, const PeerSink& sink, float* __restrict__ q_out,
                                                 const typename AccTraits<Acc>::DataArg& data) {
  Acc accp = acc_make<Acc>(D, data), accm = acc_make<Acc>(D, data);
  const int64_t r = SYM ? 2 * u : u;
  float* xp = STORE ? X + r * ldx : nullptr;
  float* xm = STORE ? xp + ldx : nullptr;
  const uint64_t unit = unit0 + (uint64_t)u;
  constexpr int kSampleUnroll = AccTraits<Acc>::kSampleUnroll;
  float zsq = 0.f;
  StepCarry<Acc> carry_p, carry_m;
  if constexpr (AccTraits<Acc>::kWarpSteps) {
    // warp-uniform steps of 32 groups in increasing column order (fold_step shuffles and carries from step to step); each lane
    // still visits its groups lane, lane + 32, ... in increasing order, the order of the loops below and of eval_kernel
    uint32_t b = 0;
    for (; b + 32u * kSampleUnroll <= nq; b += 32u * kSampleUnroll) {
#pragma unroll
      for (int uu = 0; uu < kSampleUnroll; ++uu)
        sample_group<Acc, SYM, STORE, VEC, SQ>(key, sw, unit, b + 32u * uu + lane, D, mu, sigma, xp, xm, accp, accm, &zsq, true,
                                               carry_p, carry_m);
    }
    for (; b < nq; b += 32)
      sample_group<Acc, SYM, STORE, VEC, SQ>(key, sw, unit, b + lane, D, mu, sigma, xp, xm, accp, accm, &zsq, b + lane < nq,
                                             carry_p, carry_m);
  } else {
    uint32_t q = lane;
    if (kSampleUnroll > 1) {
      // independent Philox chains in flight per lane
      for (; q + 32u * (kSampleUnroll - 1) < nq; q += 32u * kSampleUnroll) {
#pragma unroll
        for (int uu = 0; uu < kSampleUnroll; ++uu)
          sample_group<Acc, SYM, STORE, VEC, SQ>(key, sw, unit, q + 32u * uu, D, mu, sigma, xp, xm, accp, accm, &zsq, true, carry_p,
                                                 carry_m);
      }
    }
    for (; q < nq; q += 32)
      sample_group<Acc, SYM, STORE, VEC, SQ>(key, sw, unit, q, D, mu, sigma, xp, xm, accp, accm, &zsq, true, carry_p, carry_m);
  }
  if (SQ) {
    zsq = warp_sum(zsq);
    if (lane == 0) q_out[r] = zsq;
  }
  if (!AccTraits<Acc>::kSampleOnly) {
    const uint64_t row = SYM ? 2 * unit : unit;  // the global row of the + row (or the row)
    const float fp = acc_finish(accp, D, &key, sw, row);
    float fm = 0.f;
    if (SYM) fm = acc_finish(accm, D, &key, sw, row + 1);
    if (lane == 0) {
      if (PUSH) {
        for (int p = 0; p < sink.world; ++p) {
          float* fr = static_cast<float*>(sink.data[p]) + row0 + r;
          fr[0] = fp;
          if (SYM) fr[1] = fm;
        }
      } else {
        f[r] = fp;
        if (SYM) f[r + 1] = fm;
      }
    }
  }
}

// PUSH: the fitness of row i goes to row (row0 + i) of EVERY peer's fitness vector (the all-gather of the sharded
// generation, fused into the producer) and the last CTA raises this rank's flag on every peer.
// SQ (non-symmetric only): q[r] = sum_j z_rj^2 of the unscaled normals, accumulated in registers next to the objective.
template <typename Acc, bool SYM, bool STORE, bool VEC, bool PUSH, bool SQ = false>
__global__ void __launch_bounds__(kSampleThreads, AccTraits<Acc>::kSampleMinBlocks)
    sample_eval_kernel(float* __restrict__ X, int64_t ldx, const float* __restrict__ mu, const float* __restrict__ sigma,
                       int64_t row0, int64_t n_units, int64_t D, const __grid_constant__ PhiloxKey key, const uint32_t* __restrict__ stream_off,
                       float* __restrict__ f, const __grid_constant__ PeerSink sink, const unsigned long long* epoch, unsigned int* done,
                       float* __restrict__ q_out, const typename AccTraits<Acc>::DataArg data) {
  static_assert(!(SQ && (SYM || PUSH)), "the squared norms are produced by the plain non-symmetric sampler only");
  const int lane = threadIdx.x & 31;
  const uint32_t sw = key.stream_lo + (stream_off ? __ldg(stream_off) : 0u);
  const int64_t warps_total = (int64_t)gridDim.x * (kSampleThreads / 32);
  const int64_t gw = (int64_t)blockIdx.x * (kSampleThreads / 32) + (threadIdx.x >> 5);
  const uint32_t nq = (uint32_t)((D + 3) >> 2);
  const uint64_t unit0 = (uint64_t)(SYM ? (row0 >> 1) : row0);

  for (int64_t u = gw; u < n_units; u += warps_total)
    sample_eval_unit<Acc, SYM, STORE, VEC, PUSH, SQ>(lane, X, ldx, mu, sigma, row0, u, D, key, sw, nq, unit0, f, sink, q_out, data);
  if (PUSH) peer_signal_tail(sink, epoch, done);
}

// Batched searches (the functional ask / tell API with leading batch dimensions): blockIdx.y = item b of the launch.  Every
// item has its own X, mu and sigma at an item stride (0 = the operand is shared by all items), its fitnesses at row b of
// f [items][n_rows], and its own Philox stream word key.stream_lo + b, so one launch samples and evaluates the populations of
// all items, bit-identical to one sample_eval_kernel launch per item with stream id (stream id of the key) + b.  The data of
// an accumulator with data terms is per item too, at the item strides of its binding.
template <typename Acc, bool SYM, bool STORE, bool VEC>
__global__ void __launch_bounds__(kSampleThreads, AccTraits<Acc>::kSampleMinBlocks)
    sample_eval_batched_kernel(float* __restrict__ X, int64_t item_stride_x, int64_t ldx, const float* __restrict__ mu, int64_t item_stride_mu,
                               const float* __restrict__ sigma, int64_t item_stride_sigma, int64_t n_units, int64_t D,
                               const __grid_constant__ PhiloxKey key, float* __restrict__ f, const typename AccTraits<Acc>::DataArg data) {
  const int lane = threadIdx.x & 31;
  const int64_t item = blockIdx.y;
  if (STORE) X += item * item_stride_x;
  mu += item * item_stride_mu;
  sigma += item * item_stride_sigma;
  if (!AccTraits<Acc>::kSampleOnly) f += item * (SYM ? 2 * n_units : n_units);
  const uint32_t sw = key.stream_lo + (uint32_t)item;
  const int64_t warps_total = (int64_t)gridDim.x * (kSampleThreads / 32);
  const int64_t gw = (int64_t)blockIdx.x * (kSampleThreads / 32) + (threadIdx.x >> 5);
  const uint32_t nq = (uint32_t)((D + 3) >> 2);
  const PeerSink no_sink{};
  const typename AccTraits<Acc>::DataArg my_data = item_data(data, item);
  for (int64_t u = gw; u < n_units; u += warps_total)
    sample_eval_unit<Acc, SYM, STORE, VEC, false, false>(lane, X, ldx, mu, sigma, 0, u, D, key, sw, nq, 0, f, no_sink, nullptr, my_data);
}

constexpr int kEvalThreads = 256;

// The columns of one row of an accumulator with kTransform as fold_row takes them: a row x of X (global memory, streaming loads)
// and its transformed row y (shared memory or a workspace, 16-byte aligned where load4 reads it)
struct RowColsXY {
  const float* x;
  const float* y;
  __device__ __forceinline__ void load4(int64_t j, XY (&v)[4]) const {
    const float4 a = ld_stream4(x + j);
    const float4 b = *reinterpret_cast<const float4*>(y + j);
    v[0] = {a.x, b.x}; v[1] = {a.y, b.y}; v[2] = {a.z, b.z}; v[3] = {a.w, b.w};
  }
  __device__ __forceinline__ XY load1(int64_t j) const { return {ld_stream1(x + j), y[j]}; }
};

// The fitness of row r (D columns, read through the loader make_row() returns; every lane gets it), with the data binding `data`
// and, for an accumulator with noise, global row row0 + r of the draw (key, stream word sw); key is null for every other
// accumulator.  eval_row below, with the columns of a loader, in its order on every path: the body of the transformed evaluation
// kernels, which therefore give the bits eval_row gives the same (x, y) columns.  (eval_row keeps its own body: the built-in
// kernels of libevok are compiled from it as they were.)  A change to the fold order of one must be made in the other; the GPU
// test of permutation transforms (tests/test_transformed_objective_gpu.py) compares their bits.
template <typename Acc, bool VEC, typename MakeRow>
__device__ __forceinline__ float fold_row(int lane, const MakeRow& make_row, int64_t r, int64_t D, const typename AccTraits<Acc>::DataArg& data,
                                          const PhiloxKey* key, uint32_t sw, int64_t row0) {
  using T = AccTraits<Acc>;
  using V = typename T::ColVal;
  Acc acc = acc_make<Acc>(D, data);
  const auto row = make_row();
  if constexpr (T::kWarpSteps) {
    // warp-uniform steps (fold_step shuffles); per lane the groups, element adds, running sums and pair folds of
    // sample_eval_kernel's VEC path in the same order, so both kernels give the same fitness bit for bit on the same X
    constexpr bool kFoldNow = !T::kRunning;
    StepCarry<Acc> carry;
    if (VEC) {
      const int64_t nq = D >> 2;
      int64_t b = 0;
      for (; b + 128 <= nq; b += 128) {
        const int64_t q = b + lane;
        V g[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) row.load4(4 * (q + 32 * k), g[k]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int64_t jk = 4 * (q + 32 * k);
          const V (&v)[4] = g[k];
          DataCols<Acc, 4> dc;
          dc.load4(acc, jk);
          if constexpr (T::kElementDraws) dc.draw4(*key, sw, row0 + r, (uint32_t)(q + 32 * k));
          if constexpr (T::kPairs)
            if (jk > 0) dc.load_left(acc, jk);
          if constexpr (kFoldNow) {
            acc_add(acc, v[0], jk, dc.v[0]); acc_add(acc, v[1], jk + 1, dc.v[1]); acc_add(acc, v[2], jk + 2, dc.v[2]); acc_add(acc, v[3], jk + 3, dc.v[3]);
          }
          fold_step<4>(acc, v, jk, 4, carry, dc);
        }
      }
      for (; b < nq; b += 32) {
        const int64_t q = b + lane;
        const bool active = q < nq;
        V v[4] = {};
        if (active) row.load4(4 * q, v);
        const int64_t ja = 4 * q;
        DataCols<Acc, 4> dc;
        if (active) {
          dc.load4(acc, ja);
          if constexpr (T::kElementDraws) dc.draw4(*key, sw, row0 + r, (uint32_t)q);
          if constexpr (T::kPairs)
            if (ja > 0) dc.load_left(acc, ja);
          if constexpr (kFoldNow) {
            acc_add(acc, v[0], ja, dc.v[0]); acc_add(acc, v[1], ja + 1, dc.v[1]); acc_add(acc, v[2], ja + 2, dc.v[2]); acc_add(acc, v[3], ja + 3, dc.v[3]);
          }
        }
        fold_step<4>(acc, v, ja, active ? 4 : 0, carry, dc);
      }
    } else {
      for (int64_t b = 0; b < D; b += 32) {
        const int64_t j = b + lane;
        const bool active = j < D;
        V v[1] = {};
        if (active) v[0] = row.load1(j);
        DataCols<Acc, 1> dc;
        if (active) {
          dc.load1(acc, j, 0);
          if constexpr (T::kElementDraws) dc.draw1(*key, sw, row0 + r, j, 0);
          if constexpr (T::kPairs)
            if (j > 0) dc.load_left(acc, j);
          if constexpr (kFoldNow) acc_add(acc, v[0], j, dc.v[0]);
        }
        fold_step<1>(acc, v, j, active ? 1 : 0, carry, dc);
      }
    }
  } else if (VEC) {
    const int64_t nq = D >> 2;
    int64_t q = lane;
    // 4 independent 128-bit loads in flight per lane
    for (; q + 96 < nq; q += 128) {
      V a[4], b[4], c[4], d[4];
      row.load4(4 * q, a); row.load4(4 * (q + 32), b); row.load4(4 * (q + 64), c); row.load4(4 * (q + 96), d);
      const int64_t ja = 4 * q, jb = 4 * (q + 32), jc = 4 * (q + 64), jd = 4 * (q + 96);
      DataCols<Acc, 4> da, db, dc, dd;
      da.load4(acc, ja); db.load4(acc, jb); dc.load4(acc, jc); dd.load4(acc, jd);
      if constexpr (T::kElementDraws) {
        const uint64_t row = row0 + r;
        da.draw4(*key, sw, row, (uint32_t)q); db.draw4(*key, sw, row, (uint32_t)(q + 32));
        dc.draw4(*key, sw, row, (uint32_t)(q + 64)); dd.draw4(*key, sw, row, (uint32_t)(q + 96));
      }
      acc_add(acc, a[0], ja, da.v[0]); acc_add(acc, a[1], ja + 1, da.v[1]); acc_add(acc, a[2], ja + 2, da.v[2]); acc_add(acc, a[3], ja + 3, da.v[3]);
      acc_add(acc, b[0], jb, db.v[0]); acc_add(acc, b[1], jb + 1, db.v[1]); acc_add(acc, b[2], jb + 2, db.v[2]); acc_add(acc, b[3], jb + 3, db.v[3]);
      acc_add(acc, c[0], jc, dc.v[0]); acc_add(acc, c[1], jc + 1, dc.v[1]); acc_add(acc, c[2], jc + 2, dc.v[2]); acc_add(acc, c[3], jc + 3, dc.v[3]);
      acc_add(acc, d[0], jd, dd.v[0]); acc_add(acc, d[1], jd + 1, dd.v[1]); acc_add(acc, d[2], jd + 2, dd.v[2]); acc_add(acc, d[3], jd + 3, dd.v[3]);
    }
    for (; q < nq; q += 32) {
      V a[4];
      row.load4(4 * q, a);
      const int64_t ja = 4 * q;
      DataCols<Acc, 4> da;
      da.load4(acc, ja);
      if constexpr (T::kElementDraws) da.draw4(*key, sw, row0 + r, (uint32_t)q);
      acc_add(acc, a[0], ja, da.v[0]); acc_add(acc, a[1], ja + 1, da.v[1]); acc_add(acc, a[2], ja + 2, da.v[2]); acc_add(acc, a[3], ja + 3, da.v[3]);
    }
  } else {
    for (int64_t j = lane; j < D; j += 32) {
      DataCols<Acc, 1> dc;
      dc.load1(acc, j, 0);
      if constexpr (T::kElementDraws) dc.draw1(*key, sw, row0 + r, j, 0);
      acc_add(acc, row.load1(j), j, dc.v[0]);
    }
  }
  return acc_finish(acc, D, key, sw, (uint64_t)(row0 + r));
}

// eval_row's fold order is also that of fold_row above (the transformed kernels): change both together.
// One row of the evaluation kernels: the fitness of row r of X (row pitch ldx, D columns; every lane gets it), with the data
// binding `data` and, for an accumulator with noise, global row row0 + r of the draw (key, stream word sw); key is null for every
// other accumulator.  The body of eval_kernel and of eval_batched_kernel, so both give the same bits for the same row, draw and
// path.
template <typename Acc, bool VEC>
__device__ __forceinline__ float eval_row(int lane, const float* __restrict__ X, int64_t ldx, int64_t r, int64_t D,
                                          const typename AccTraits<Acc>::DataArg& data, const PhiloxKey* key, uint32_t sw, int64_t row0) {
  using T = AccTraits<Acc>;
  Acc acc = acc_make<Acc>(D, data);
  const float* x = X + r * ldx;
  if constexpr (T::kWarpSteps) {
    // warp-uniform steps (fold_step shuffles); per lane the groups, element adds, running sums and pair folds of
    // sample_eval_kernel's VEC path in the same order, so both kernels give the same fitness bit for bit on the same X
    constexpr bool kFoldNow = !T::kRunning;
    StepCarry<Acc> carry;
    if (VEC) {
      const int64_t nq = D >> 2;
      int64_t b = 0;
      for (; b + 128 <= nq; b += 128) {
        const int64_t q = b + lane;
        float4 g[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) g[k] = ld_stream4(x + 4 * (q + 32 * k));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int64_t jk = 4 * (q + 32 * k);
          const float v[4] = {g[k].x, g[k].y, g[k].z, g[k].w};
          DataCols<Acc, 4> dc;
          dc.load4(acc, jk);
          if constexpr (T::kElementDraws) dc.draw4(*key, sw, row0 + r, (uint32_t)(q + 32 * k));
          if constexpr (T::kPairs)
            if (jk > 0) dc.load_left(acc, jk);
          if constexpr (kFoldNow) {
            acc_add(acc, v[0], jk, dc.v[0]); acc_add(acc, v[1], jk + 1, dc.v[1]); acc_add(acc, v[2], jk + 2, dc.v[2]); acc_add(acc, v[3], jk + 3, dc.v[3]);
          }
          fold_step<4>(acc, v, jk, 4, carry, dc);
        }
      }
      for (; b < nq; b += 32) {
        const int64_t q = b + lane;
        const bool active = q < nq;
        const float4 a = active ? ld_stream4(x + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float v[4] = {a.x, a.y, a.z, a.w};
        const int64_t ja = 4 * q;
        DataCols<Acc, 4> dc;
        if (active) {
          dc.load4(acc, ja);
          if constexpr (T::kElementDraws) dc.draw4(*key, sw, row0 + r, (uint32_t)q);
          if constexpr (T::kPairs)
            if (ja > 0) dc.load_left(acc, ja);
          if constexpr (kFoldNow) {
            acc_add(acc, v[0], ja, dc.v[0]); acc_add(acc, v[1], ja + 1, dc.v[1]); acc_add(acc, v[2], ja + 2, dc.v[2]); acc_add(acc, v[3], ja + 3, dc.v[3]);
          }
        }
        fold_step<4>(acc, v, ja, active ? 4 : 0, carry, dc);
      }
    } else {
      for (int64_t b = 0; b < D; b += 32) {
        const int64_t j = b + lane;
        const bool active = j < D;
        const float v[1] = {active ? ld_stream1(x + j) : 0.f};
        DataCols<Acc, 1> dc;
        if (active) {
          dc.load1(acc, j, 0);
          if constexpr (T::kElementDraws) dc.draw1(*key, sw, row0 + r, j, 0);
          if constexpr (T::kPairs)
            if (j > 0) dc.load_left(acc, j);
          if constexpr (kFoldNow) acc_add(acc, v[0], j, dc.v[0]);
        }
        fold_step<1>(acc, v, j, active ? 1 : 0, carry, dc);
      }
    }
  } else if (VEC) {
    const int64_t nq = D >> 2;
    int64_t q = lane;
    // 4 independent 128-bit loads in flight per lane
    for (; q + 96 < nq; q += 128) {
      const float4 a = ld_stream4(x + 4 * q), b = ld_stream4(x + 4 * (q + 32)), c = ld_stream4(x + 4 * (q + 64)),
                   d = ld_stream4(x + 4 * (q + 96));
      const int64_t ja = 4 * q, jb = 4 * (q + 32), jc = 4 * (q + 64), jd = 4 * (q + 96);
      DataCols<Acc, 4> da, db, dc, dd;
      da.load4(acc, ja); db.load4(acc, jb); dc.load4(acc, jc); dd.load4(acc, jd);
      if constexpr (T::kElementDraws) {
        const uint64_t row = row0 + r;
        da.draw4(*key, sw, row, (uint32_t)q); db.draw4(*key, sw, row, (uint32_t)(q + 32));
        dc.draw4(*key, sw, row, (uint32_t)(q + 64)); dd.draw4(*key, sw, row, (uint32_t)(q + 96));
      }
      acc_add(acc, a.x, ja, da.v[0]); acc_add(acc, a.y, ja + 1, da.v[1]); acc_add(acc, a.z, ja + 2, da.v[2]); acc_add(acc, a.w, ja + 3, da.v[3]);
      acc_add(acc, b.x, jb, db.v[0]); acc_add(acc, b.y, jb + 1, db.v[1]); acc_add(acc, b.z, jb + 2, db.v[2]); acc_add(acc, b.w, jb + 3, db.v[3]);
      acc_add(acc, c.x, jc, dc.v[0]); acc_add(acc, c.y, jc + 1, dc.v[1]); acc_add(acc, c.z, jc + 2, dc.v[2]); acc_add(acc, c.w, jc + 3, dc.v[3]);
      acc_add(acc, d.x, jd, dd.v[0]); acc_add(acc, d.y, jd + 1, dd.v[1]); acc_add(acc, d.z, jd + 2, dd.v[2]); acc_add(acc, d.w, jd + 3, dd.v[3]);
    }
    for (; q < nq; q += 32) {
      const float4 a = ld_stream4(x + 4 * q);
      const int64_t ja = 4 * q;
      DataCols<Acc, 4> da;
      da.load4(acc, ja);
      if constexpr (T::kElementDraws) da.draw4(*key, sw, row0 + r, (uint32_t)q);
      acc_add(acc, a.x, ja, da.v[0]); acc_add(acc, a.y, ja + 1, da.v[1]); acc_add(acc, a.z, ja + 2, da.v[2]); acc_add(acc, a.w, ja + 3, da.v[3]);
    }
  } else {
    for (int64_t j = lane; j < D; j += 32) {
      DataCols<Acc, 1> dc;
      dc.load1(acc, j, 0);
      if constexpr (T::kElementDraws) dc.draw1(*key, sw, row0 + r, j, 0);
      acc_add(acc, ld_stream1(x + j), j, dc.v[0]);
    }
  }
  return acc_finish(acc, D, key, sw, (uint64_t)(row0 + r));
}

// The evaluation kernel.  Row r of X is global row noise.row0 + r of the draw (noise.key, stream word noise.key.stream_lo +
// *noise.stream_off) for an accumulator with noise (evok_eval_keyed), which then gets the noise the sampler gave the row;
// `noise` is an empty struct for every other accumulator.
template <typename Acc, bool VEC>
__global__ void __launch_bounds__(kEvalThreads, AccTraits<Acc>::kEvalMinBlocks)
    eval_kernel(const float* __restrict__ X, int64_t ldx, int64_t n_rows, int64_t D, float* __restrict__ f,
                const typename AccTraits<Acc>::DataArg data, const typename AccTraits<Acc>::EvalArg noise) {
  using T = AccTraits<Acc>;
  const int lane = threadIdx.x & 31;
  const PhiloxKey* key = nullptr;  // the rows' draw: none without noise
  uint32_t sw = 0u;
  int64_t row0 = 0;
  if constexpr (T::kNoise) {
    key = &noise.key;
    sw = noise.key.stream_lo + (noise.stream_off ? __ldg(noise.stream_off) : 0u);
    row0 = noise.row0;
  }
  const int64_t warps_total = (int64_t)gridDim.x * (kEvalThreads / 32);
  const int64_t gw = (int64_t)blockIdx.x * (kEvalThreads / 32) + (threadIdx.x >> 5);
  for (int64_t r = gw; r < n_rows; r += warps_total) {
    const float v = eval_row<Acc, VEC>(lane, X, ldx, r, D, data, key, sw, row0);
    if (lane == 0) f[r] = v;
  }
}

// The evaluation of a batch of populations (evok_eval_batched): blockIdx.y = item b of the launch, whose rows are those of
// X + b * item_stride_x (row pitch ldx; item stride 0 = every item evaluates the same rows), whose data is item b of the binding
// (item_data) and whose fitnesses go to f[b * n_rows + r].  For an accumulator with noise, row r of item b is row r of the draw
// (noise.key, stream word noise.key.stream_lo + b): the noise the batched sampler gives row r of item b with that key, so a
// population it stored gets its fitnesses again.  noise.stream_off and noise.row0 are not read (null and 0).  Every item gets
// the bits of one eval_kernel launch on its rows with stream id (stream id of the key) + b, on the same path.
template <typename Acc, bool VEC>
__global__ void __launch_bounds__(kEvalThreads, AccTraits<Acc>::kEvalMinBlocks)
    eval_batched_kernel(const float* __restrict__ X, int64_t item_stride_x, int64_t ldx, int64_t n_rows, int64_t D, float* __restrict__ f,
                        const typename AccTraits<Acc>::DataArg data, const typename AccTraits<Acc>::EvalArg noise) {
  const int lane = threadIdx.x & 31;
  const int64_t item = blockIdx.y;
  X += item * item_stride_x;
  f += item * n_rows;
  const PhiloxKey* key = nullptr;
  uint32_t sw = 0u;
  if constexpr (AccTraits<Acc>::kNoise) {
    key = &noise.key;
    sw = noise.key.stream_lo + (uint32_t)item;
  }
  const typename AccTraits<Acc>::DataArg my_data = item_data(data, item);
  const int64_t warps_total = (int64_t)gridDim.x * (kEvalThreads / 32);
  const int64_t gw = (int64_t)blockIdx.x * (kEvalThreads / 32) + (threadIdx.x >> 5);
  for (int64_t r = gw; r < n_rows; r += warps_total) {
    const float v = eval_row<Acc, VEC>(lane, X, ldx, r, D, my_data, key, sw, 0);
    if (lane == 0) f[r] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Transformed evaluation (evok_eval_transform_batched): the terms of an accumulator with kTransform read y = M (x - o) of each row,
// with M (D x D, row-major, row pitch D) and o (D) of the row's item at their item strides (0: shared by all items).  Each x_k - o_k
// is rounded to float32 first, so a row equal to o has y = 0 exactly whatever M is.  Item b of a launch is blockIdx.y and draws
// its noise as eval_batched_kernel's item b does (stream word key.stream_lo + b, global row = its row).
// ------------------------------------------------------------------------------------------------
// The shared-memory layout of the fused kernel: M with an odd row pitch (column reads of 32 rows hit 32 banks), o, then the tile's
// x - o and y, rows at a pitch of round4(D) floats (16-byte aligned rows for fold_row's 16-byte loads).
__host__ __device__ constexpr int64_t transform_pitch_m(int64_t D) { return D | 1; }
__host__ __device__ constexpr int64_t round4(int64_t n) { return (n + 3) & ~int64_t(3); }
__host__ __device__ constexpr int64_t transform_smem_floats(int64_t D, int64_t tile_rows) {
  return round4(D * transform_pitch_m(D)) + round4(D) + 2 * tile_rows * round4(D);
}

// The small-D path, one launch: CTA (x, b) stages item b's M and o, then for each tile of `tile_rows` rows (tiles strided over
// grid x) stages x - o, computes y_j = sum_{k=0}^{D-1} M[j][k] (x_k - o_k) as one FP32 FMA chain in increasing k from 0 (a thread
// per column and pair of rows), and folds each row's (x, y) with one warp (fold_row: the order of eval_row).  With M a permutation
// and o = 0 the y of a finite row are its permuted entries exactly, so the fitness is the bits of eval_batched_kernel on the
// permuted rows, on the same path.  Dynamic shared memory: transform_smem_floats(D, tile_rows) floats, tile_rows even.
template <typename Acc, bool VEC>
__global__ void __launch_bounds__(kEvalThreads, 1)
    eval_transform_fused_kernel(const float* __restrict__ X, int64_t item_stride_x, int64_t ldx, const float* __restrict__ M,
                                int64_t item_stride_m, const float* __restrict__ o, int64_t item_stride_o, int64_t n_rows, int64_t D,
                                int64_t tile_rows, float* __restrict__ f, const typename AccTraits<Acc>::DataArg data,
                                const typename AccTraits<Acc>::EvalArg noise) {
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t item = blockIdx.y;
  X += item * item_stride_x;
  M += item * item_stride_m;
  o += item * item_stride_o;
  f += item * n_rows;
  const PhiloxKey* key = nullptr;
  uint32_t sw = 0u;
  if constexpr (AccTraits<Acc>::kNoise) {
    key = &noise.key;
    sw = noise.key.stream_lo + (uint32_t)item;
  }
  const typename AccTraits<Acc>::DataArg my_data = item_data(data, item);
  const int64_t pm = transform_pitch_m(D), p4 = round4(D);
  float* sM = smem;
  float* so = smem + round4(D * pm);
  float* sxo = so + p4;
  float* sy = sxo + tile_rows * p4;
  for (int64_t i = tid; i < D * D; i += kEvalThreads) {
    const int64_t r = i / D;
    sM[r * pm + (i - r * D)] = __ldg(M + i);
  }
  for (int64_t i = tid; i < D; i += kEvalThreads) so[i] = __ldg(o + i);
  for (int64_t t0 = (int64_t)blockIdx.x * tile_rows; t0 < n_rows; t0 += (int64_t)gridDim.x * tile_rows) {
    const int64_t rows = n_rows - t0 < tile_rows ? n_rows - t0 : tile_rows;
    __syncthreads();  // M and o are staged, and the previous tile's folds have read their y
    for (int64_t i = tid; i < rows * D; i += kEvalThreads) {
      const int64_t r = i / D, k = i - r * D;
      sxo[r * p4 + k] = X[(t0 + r) * ldx + k] - so[k];
    }
    __syncthreads();
    const int64_t pairs = (rows + 1) >> 1;
    for (int64_t i = tid; i < pairs * D; i += kEvalThreads) {
      const int64_t r = 2 * (i / D), j = i - (r >> 1) * D;
      const bool two = r + 1 < rows;
      const float* m = sM + j * pm;
      const float* a = sxo + r * p4;
      const float* b = two ? a + p4 : a;
      float ya = 0.f, yb = 0.f;
#pragma unroll 4
      for (int64_t k = 0; k < D; ++k) {
        const float mk = m[k];
        ya = fmaf(mk, a[k], ya);
        yb = fmaf(mk, b[k], yb);
      }
      sy[r * p4 + j] = ya;
      if (two) sy[(r + 1) * p4 + j] = yb;
    }
    __syncthreads();
    for (int64_t r = warp; r < rows; r += kEvalThreads / 32) {
      const float v = fold_row<Acc, VEC>(lane, [&] { return RowColsXY{X + (t0 + r) * ldx, sy + r * p4}; }, r, D, my_data, key, sw, t0);
      if (lane == 0) f[t0 + r] = v;
    }
  }
}

// The large-D path's evaluation: the y of every row are in Y (written by the batched 3xTF32 GEMM of x - o and M), item b's row r
// at Y + b * item_stride_y + r * ldy; one warp per row folds (x, y) as eval_batched_kernel folds x.
// (at least one CTA per SM in the launch bounds: with none ptxas caps some accumulators at 64 registers and spills)
template <typename Acc, bool VEC>
__global__ void __launch_bounds__(kEvalThreads, AccTraits<Acc>::kNoise ? 2 : 1)
    eval_transform_kernel(const float* __restrict__ X, int64_t item_stride_x, int64_t ldx, const float* __restrict__ Y, int64_t item_stride_y,
                          int64_t ldy, int64_t n_rows, int64_t D, float* __restrict__ f, const typename AccTraits<Acc>::DataArg data,
                          const typename AccTraits<Acc>::EvalArg noise) {
  const int lane = threadIdx.x & 31;
  const int64_t item = blockIdx.y;
  X += item * item_stride_x;
  Y += item * item_stride_y;
  f += item * n_rows;
  const PhiloxKey* key = nullptr;
  uint32_t sw = 0u;
  if constexpr (AccTraits<Acc>::kNoise) {
    key = &noise.key;
    sw = noise.key.stream_lo + (uint32_t)item;
  }
  const typename AccTraits<Acc>::DataArg my_data = item_data(data, item);
  const int64_t warps_total = (int64_t)gridDim.x * (kEvalThreads / 32);
  const int64_t gw = (int64_t)blockIdx.x * (kEvalThreads / 32) + (threadIdx.x >> 5);
  for (int64_t r = gw; r < n_rows; r += warps_total) {
    const float v = fold_row<Acc, VEC>(lane, [&] { return RowColsXY{X + r * ldx, Y + r * ldy}; }, r, D, my_data, key, sw, 0);
    if (lane == 0) f[r] = v;
  }
}

}  // namespace evok
