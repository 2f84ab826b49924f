// K4: utility-weighted column reductions over the population (one fused pass, two accumulators per column).
//   S1_j = sum_r a_r eps_rj          S2_j = sum_r b_r (eps_rj^2 * c1_j - c0_j)         eps = X - mu
// with (c1, c0) = (1/sigma, sigma) for the PGPE forms, (1/sigma^2, 1) for SNES, (1, 0) for raw moments.
// HBM-bound: each CTA owns a column tile (128-bit loads, 4 rows in flight per thread) and a contiguous chunk of
// rows; partial sums go to a [chunk][2][D] workspace and a second tiny kernel adds the chunks in a fixed order
// (deterministic, no atomics).  In the symmetric form only the even ("+") rows are read.
#include <dlfcn.h>

#include <atomic>
#include <cstdlib>

#include "evok_common.cuh"

#ifndef EVOK_GRAD_TMA_DEFAULT
#define EVOK_GRAD_TMA_DEFAULT 1
#endif

namespace evok {

constexpr int kGradThreads = 256;
constexpr int kGradUnroll = 4;
constexpr int kGradMinBlocks = 4;  // __launch_bounds__ of grad_partial_kernel
constexpr int kGradCtasPerSm = 4;  // the LDG plan's wave of resident CTAs
constexpr int kMaxResidentCtas = kNumSMs * 8;

template <int VEC>
struct VecF;
template <>
struct VecF<4> {
  float v[4];
};
template <>
struct VecF<1> {
  float v[1];
};

template <int VEC>
__device__ __forceinline__ VecF<VEC> load_row(const float* p) {
  VecF<VEC> r;
  if (VEC == 4) {
    const float4 t = ld_stream4(p);
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  } else {
    r.v[0] = ld_stream1(p);
  }
  return r;
}

// Batched searches (functional API): blockIdx.z = batch item; element strides between the items' operands (0 = shared)
struct GradItems {
  int64_t x, w, mu, sigma, partial;
};

// Separable CMA-ES row weights (SEPW mode): w holds the rank-assigned weights aw; row r contributes a = max(aw, 0) to S1
// (recombination) and b = aw, or with active weights b = aw > 0 ? aw : D * aw / q[r] (q = ||z_r||^2, cmaes.py:531-535 of the
// reference), to S2; the CTAs of column tile 0 also add up b per row chunk into wsum_partial[chunk].  In a batch q is [items][n_rows]
// (the layout of w) and wsum_partial [items][n_chunks].
struct SepWeights {
  const float* q;
  int active;
  float* wsum_partial;
};

// Where eps comes from (EPS): kEpsRead: eps = X - mu from the stored rows; kEpsRegen: eps = sigma * z regenerated from Philox
// (the lazy population of evok_sample_eval); kEpsRebuild: the row rebuilt as the sampler stored it, x = fmaf(sigma, z, mu), then
// eps = x - mu, bit-identical to kEpsRead over the stored rows, with item b of a batch (blockIdx.z) on stream word stream_lo + b.
constexpr int kEpsRead = 0, kEpsRegen = 1, kEpsRebuild = 2;

// The arithmetic both partial kernels share.  (c1, c0) of column sigma s for `form`:
__device__ __forceinline__ void grad_coeffs(int form, float s, float& c1, float& c0) {
  if (form == EVOK_GRAD_EXP) {
    c1 = __fdiv_rn(1.0f, s * s);
    c0 = 1.0f;
  } else if (form == EVOK_GRAD_MOMENTS) {
    c1 = 1.0f;
    c0 = 0.0f;
  } else {
    c1 = __fdiv_rn(1.0f, s);
    c0 = s;
  }
}

// (a, b) of unit r: the SEPW weights above, the half difference and half sum of a direction's two rows, or w[r] twice
template <bool SYM, bool SEPW = false>
__device__ __forceinline__ void row_weights(const float* __restrict__ w, int64_t r, float& a, float& b, int64_t D = 0,
                                            const float* __restrict__ q = nullptr, int active = 0) {
  if (SEPW) {
    const float aw = __ldg(w + r);
    a = fmaxf(aw, 0.0f);
    // q is read only for the negative weights: a zero-weight row is never regenerated and never looks at its norm
    b = (active && aw < 0.0f) ? __fdiv_rn((float)D * aw, __ldg(q + r)) : aw;
  } else if (SYM) {
    const float wp = __ldg(w + 2 * r), wm = __ldg(w + 2 * r + 1);
    a = 0.5f * (wp - wm);
    b = 0.5f * (wp + wm);
  } else {
    a = b = __ldg(w + r);
  }
}

__device__ __forceinline__ void accumulate(float a, float b, float e, float c1, float c0, float& s1, float& s2) {
  s1 = fmaf(a, e, s1);
  s2 = fmaf(b, fmaf(e * e, c1, -c0), s2);
}

// (S1, S2) of this thread's VEC columns into row chunk `chunk` of the [chunk][2][D] workspace; TAIL: a column may lie past D
template <int VEC, bool TAIL = true>
__device__ __forceinline__ void store_partial(float* partial, int64_t chunk, int64_t D, int64_t col, const float* s1, const float* s2) {
  float* p1 = partial + (chunk * 2 + 0) * D + col;
  float* p2 = partial + (chunk * 2 + 1) * D + col;
#pragma unroll
  for (int c = 0; c < VEC; ++c) {
    if (!TAIL || col + c < D) {
      p1[c] = s1[c];
      p2[c] = s2[c];
    }
  }
}

// SYM: unit r = direction (rows 2r, 2r+1), else unit r = row r.
// SEPW (non-symmetric, form MOMENTS): the weights above, over the steps z.  With kEpsRegen (mu = sigma = NULL) z is the Philox
// normal itself; with kEpsRead / kEpsRebuild it is the step recovered from the row as the functional tell recovers it,
// z = (x - m) / s correctly rounded, with (mu, sigma) = (m, s), the centre and per-column stdev the rows were drawn from.
template <int VEC, int TX, bool SYM, int EPS, bool SEPW = false>
__global__ void __launch_bounds__(kGradThreads, kGradMinBlocks)
    grad_partial_kernel(int form, const float* __restrict__ X, int64_t ldx, const float* __restrict__ w, const float* __restrict__ mu,
                        const float* __restrict__ sigma, int64_t n_units, int64_t D, int64_t units_per_chunk, uint64_t unit0,
                        const __grid_constant__ PhiloxKey key, const uint32_t* __restrict__ stream_off, float* __restrict__ partial,
                        const __grid_constant__ GradItems items, const __grid_constant__ SepWeights sepw) {
  static_assert(!SEPW || !SYM, "the CMA-ES weight mode reduces non-symmetric rows");
  constexpr int TY = kGradThreads / TX;
  const float* q = sepw.q;
  float* wsum_partial = sepw.wsum_partial;
  if (gridDim.z > 1) {
    const int64_t item = blockIdx.z;
    X += item * items.x;
    w += item * items.w;
    mu += item * items.mu;
    sigma += item * items.sigma;
    partial += item * items.partial;
    if (SEPW) {
      q += item * items.w;
      wsum_partial += item * gridDim.y;
    }
  }
  const uint32_t sw = key.stream_lo + ((EPS != kEpsRead && stream_off) ? __ldg(stream_off) : 0u) + (EPS == kEpsRebuild ? (uint32_t)blockIdx.z : 0u);
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
  const int64_t col = ((int64_t)blockIdx.x * TX + tx) * VEC;
  const bool active = col < D;

  float m[VEC], c1[VEC], c0[VEC], sg[VEC];
#pragma unroll
  for (int c = 0; c < VEC; ++c) {
    const bool ok = active && (col + c < D) && !(SEPW && EPS == kEpsRegen);
    const float s = ok ? __ldg(sigma + col + c) : 1.0f;
    m[c] = ok ? __ldg(mu + col + c) : 0.0f;
    sg[c] = s;
    grad_coeffs(form, s, c1[c], c0[c]);
  }

  float s1[VEC], s2[VEC];
#pragma unroll
  for (int c = 0; c < VEC; ++c) s1[c] = s2[c] = 0.0f;

  const int64_t r_begin = (int64_t)blockIdx.y * units_per_chunk;
  const int64_t r_end = min(n_units, r_begin + units_per_chunk);
  float wb = 0.0f;  // SEPW: sum of this thread's b (rows in a fixed order)

  for (int64_t r0 = r_begin + ty; r0 < r_end; r0 += (int64_t)TY * kGradUnroll) {
    float a[kGradUnroll], b[kGradUnroll];
    bool need[kGradUnroll];
    VecF<VEC> x[kGradUnroll];
#pragma unroll
    for (int u = 0; u < kGradUnroll; ++u) {
      const int64_t r = r0 + (int64_t)u * TY;
      a[u] = b[u] = 0.0f;
      if (r < r_end) {
        row_weights<SYM, SEPW>(w, r, a[u], b[u], D, q, sepw.active);
        if (SEPW) wb += b[u];
      }
      need[u] = active && (a[u] != 0.0f || b[u] != 0.0f);
    }
#pragma unroll
    for (int u = 0; u < kGradUnroll; ++u) {
      const int64_t r = r0 + (int64_t)u * TY;
      if (need[u]) {
        if (EPS != kEpsRead) {
          if (VEC == 4) {
            normals4(key, sw, unit0 + (uint64_t)r, (uint32_t)(col >> 2), x[u].v);
          } else {
            float z[4];
            normals4(key, sw, unit0 + (uint64_t)r, (uint32_t)(col >> 2), z);
            x[u].v[0] = z[col & 3];
          }
        } else {
          x[u] = load_row<VEC>(X + (SYM ? 2 * r : r) * ldx + col);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kGradUnroll; ++u) {
      if (need[u]) {
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
          float e = EPS == kEpsRegen ? sg[c] * x[u].v[c] : EPS == kEpsRebuild ? fmaf(sg[c], x[u].v[c], m[c]) - m[c] : x[u].v[c] - m[c];
          if (SEPW && EPS != kEpsRegen) e = __fdiv_rn(e, sg[c]);  // the recovered step
          accumulate(a[u], b[u], e, c1[c], c0[c], s1[c], s2[c]);
        }
      }
    }
  }

  // combine the TY row-threads of each column in a fixed order
  __shared__ float red[TY > 1 ? TY : 1][TX][2 * VEC];
  if (TY > 1) {
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
      red[ty][tx][c] = s1[c];
      red[ty][tx][VEC + c] = s2[c];
    }
    __syncthreads();
    if (ty == 0) {
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        float t1 = red[0][tx][c], t2 = red[0][tx][VEC + c];
        for (int y = 1; y < TY; ++y) {
          t1 += red[y][tx][c];
          t2 += red[y][tx][VEC + c];
        }
        s1[c] = t1;
        s2[c] = t2;
      }
    }
  }
  if (ty == 0 && active) store_partial<VEC>(partial, blockIdx.y, D, col, s1, s2);
  if (SEPW && blockIdx.x == 0) {  // uniform per CTA: every tile's row threads see the same rows, tile 0 reports their b sum
    __shared__ float wred[TY];
    if (tx == 0) wred[ty] = wb;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = wred[0];
      for (int y = 1; y < TY; ++y) t += wred[y];
      wsum_partial[blockIdx.y] = t;
    }
  }
}

// (S1, S2) of column j over the n_chunks row chunks, in chunk order: the fixed order that makes the result deterministic
__device__ __forceinline__ void sum_chunks(const float* __restrict__ partial, int n_chunks, int64_t D, int64_t j, float& t1, float& t2) {
  t1 = 0.0f;
  t2 = 0.0f;
  for (int c = 0; c < n_chunks; ++c) {
    t1 += partial[((int64_t)c * 2 + 0) * D + j];
    t2 += partial[((int64_t)c * 2 + 1) * D + j];
  }
}

// WSUM: block x 0 of item y also adds the item's per-chunk sums of the separable CMA-ES weight mode, in chunk order, into wsum_out[y]
template <bool WSUM = false>
__global__ void __launch_bounds__(256) grad_finalize_kernel(const float* __restrict__ partial, int n_chunks, int64_t D, float scale_mu,
                                                            float scale_sigma, float* __restrict__ out_mu, float* __restrict__ out_sigma,
                                                            int64_t item_stride_partial = 0, const float* __restrict__ wsum_partial = nullptr,
                                                            float* __restrict__ wsum_out = nullptr) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (WSUM && j == 0) {
    wsum_partial += (int64_t)blockIdx.y * n_chunks;
    float t = 0.0f;
    for (int c = 0; c < n_chunks; ++c) t += wsum_partial[c];
    wsum_out[blockIdx.y] = t;
  }
  if (j >= D) return;
  partial += (int64_t)blockIdx.y * item_stride_partial;  // batched: blockIdx.y = item, outputs contiguous [items][D]
  out_mu += (int64_t)blockIdx.y * D;
  out_sigma += (int64_t)blockIdx.y * D;
  float t1, t2;
  sum_chunks(partial, n_chunks, D, j, t1, t2);
  out_mu[j] = t1 * scale_mu;
  out_sigma[j] = t2 * scale_sigma;
}

// The row pass of the separable CMA-ES moments over recovered steps: q_i = ||z_i||^2 with z_ij = (x_ij - m_j) / s_j correctly
// rounded, the z of the column pass.  One warp per row, only for the rows whose norm the column pass reads (aw_i < 0).  Lane l
// takes the column groups l, l + 32, ... of 4 columns in order and the warp adds the lanes in a fixed order.  x is the stored row
// (kEpsRead) or the row rebuilt as the batched sampler stored it (kEpsRebuild: x = fmaf(s, z, m), item b on stream word
// key.stream_lo + b); both give the same bits.  grid y = item: X at item_stride_x, m / s [items][D], aw / q [items][n_rows].
template <int EPS>
__global__ void __launch_bounds__(256) sepcma_sqnorm_kernel(const float* __restrict__ X, int64_t item_stride_x, int64_t ldx, const float* __restrict__ m,
                                                            const float* __restrict__ s, const float* __restrict__ aw, int64_t n_rows, int64_t D,
                                                            const __grid_constant__ PhiloxKey key, float* __restrict__ q) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int64_t item = blockIdx.y;
  aw += item * n_rows;
  q += item * n_rows;
  if (!(__ldg(aw + row) < 0.0f)) return;  // warp-uniform
  m += item * D;
  s += item * D;
  const float* x_row = EPS == kEpsRead ? X + item * item_stride_x + row * ldx : nullptr;
  const bool vec = EPS == kEpsRead && (D & 3) == 0 && aligned16_dev(x_row);
  const uint32_t sw = key.stream_lo + (uint32_t)item;
  float acc = 0.0f;
  for (int64_t g = lane; 4 * g < D; g += 32) {
    const int64_t col = 4 * g;
    float x[4];
    if (EPS == kEpsRebuild) {
      float z[4];
      normals4(key, sw, (uint64_t)row, (uint32_t)g, z);
#pragma unroll
      for (int c = 0; c < 4; ++c) x[c] = col + c < D ? fmaf(__ldg(s + col + c), z[c], __ldg(m + col + c)) : 0.0f;
    } else if (vec) {
      const float4 v = ld_stream4(x_row + col);
      x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c) x[c] = col + c < D ? ld_stream1(x_row + col + c) : 0.0f;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (col + c < D) {
        const float z = __fdiv_rn(x[c] - __ldg(m + col + c), __ldg(s + col + c));
        acc = fmaf(z, z, acc);
      }
    }
  }
  acc = warp_sum(acc);
  if (lane == 0) q[row] = acc;
}

// The same finalisation for the sharded generation: this rank's (grad_mu | grad_sigma) goes into slot `rank` of EVERY peer's
// slot array (world x 2D floats) and the last CTA raises this rank's flag on every peer -- the send half of the all-reduce,
// fused into the kernel that produces the data (the receive half is peer_reduce_kernel, evok_peer.cu).
struct GradPush {
  PeerSink sink;
  const unsigned long long* epoch;
  unsigned int* done;
};

__global__ void __launch_bounds__(256) grad_finalize_push_kernel(const float* __restrict__ partial, int n_chunks, int64_t D, float scale_mu,
                                                                 float scale_sigma, const __grid_constant__ PeerSink sink,
                                                                 const unsigned long long* epoch, unsigned int* done) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < D) {
    float t1, t2;
    sum_chunks(partial, n_chunks, D, j, t1, t2);
    t1 *= scale_mu;
    t2 *= scale_sigma;
    for (int p = 0; p < sink.world; ++p) {
      float* slot = static_cast<float*>(sink.data[p]) + (int64_t)sink.rank * 2 * D;
      slot[j] = t1;
      slot[D + j] = t2;
    }
  }
  peer_signal_tail(sink, epoch, done);
}

// ------------------------------------------------------------------------------------------------------------
// TMA-staged variant of the partial kernel: a producer warp streams row segments global -> shared with 1-D bulk async
// copies (cp.async.bulk, completion counted on an mbarrier), S stages of R rows x 4 KB deep, so each SM keeps
// 2 CTAs x S x R x 4 KB in flight without spending registers or issue slots on loads; 8 consumer warps read the staged
// rows from shared memory (128-bit, conflict free) and accumulate.  Column tile = 1024 columns, one float4 per thread.
// ------------------------------------------------------------------------------------------------------------
#ifndef EVOK_GRAD_TMA_ROWS
#define EVOK_GRAD_TMA_ROWS 4
#endif
#ifndef EVOK_GRAD_TMA_STAGES
#define EVOK_GRAD_TMA_STAGES 4
#endif
#ifndef EVOK_GRAD_TMA_CTAS_PER_SM
#define EVOK_GRAD_TMA_CTAS_PER_SM 3
#endif
constexpr int kTmaRows = EVOK_GRAD_TMA_ROWS;
constexpr int kTmaStages = EVOK_GRAD_TMA_STAGES;
constexpr int kTmaCols = 1024;
constexpr int kTmaConsumers = 256;
constexpr int kTmaThreads = kTmaConsumers + 32;
constexpr size_t kTmaSmemBytes = (size_t)kTmaStages * kTmaRows * kTmaCols * sizeof(float) + 2 * kTmaStages * sizeof(uint64_t) + 128;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Hybrid schedule: streaming leaves the SMs' issue slots nearly idle, so part of the row groups (kTmaRows rows each) are
// rebuilt on the SMs from the Philox counters that produced them instead of being streamed (see kAutoSplitFull for how much).  `split` of every kSplitPeriod
// consecutive groups of a chunk are rebuilt, spread evenly over the period (the same mix in every CTA); split 0 streams every
// group, kSplitPeriod rebuilds every group.  A rebuilt row is bit-identical to the stored one (same normals4 call, same
// fmaf(sigma, z, mu) as sample_group) and the accumulation order does not depend on the schedule, so neither does the result.
// The schedule is one kSplitPeriod-bit mask, built once per thread: bit k set = group k of every period is rebuilt.
constexpr int kSplitPeriod = 16;
__device__ __forceinline__ uint32_t rebuilt_mask(int split) {
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < kSplitPeriod; ++k)
    if ((k + 1) * split / kSplitPeriod > k * split / kSplitPeriod) m |= 1u << k;
  return m;
}
__device__ __forceinline__ bool group_rebuilt(uint32_t mask, int64_t g) { return (mask >> ((int)g & (kSplitPeriod - 1))) & 1u; }

template <bool SYM>
__global__ void __launch_bounds__(kTmaThreads, EVOK_GRAD_TMA_CTAS_PER_SM)
    grad_partial_tma_kernel(int form, const float* __restrict__ X, int64_t ldx, const float* __restrict__ w, const float* __restrict__ mu,
                            const float* __restrict__ sigma, int64_t n_units, int64_t D, int64_t units_per_chunk, int split, uint64_t unit0,
                            const __grid_constant__ PhiloxKey key, const uint32_t* __restrict__ stream_off, float* __restrict__ partial) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tiles = reinterpret_cast<float*>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)kTmaStages * kTmaRows * kTmaCols * sizeof(float));
  uint64_t* empty = full + kTmaStages;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t col0 = (int64_t)blockIdx.x * kTmaCols;
  const int64_t width = min((int64_t)kTmaCols, D - col0);  // columns of this tile (multiple of 4)
  const int64_t r_begin = (int64_t)blockIdx.y * units_per_chunk;
  const int64_t r_end = min(n_units, r_begin + units_per_chunk);
  const int64_t n_rows = r_end - r_begin;
  const int64_t n_groups = (n_rows + kTmaRows - 1) / kTmaRows;
  const int64_t row_stride = (SYM ? 2 : 1) * ldx;
  const uint32_t mask = rebuilt_mask(split);

  if (tid == 0) {
    for (int s = 0; s < kTmaStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kTmaConsumers / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kTmaConsumers / 32) {
    // ===== producer warp: one elected lane issues the bulk copies =====
    if (lane == 0) {
      const uint32_t row_bytes = (uint32_t)(width * sizeof(float));
      int64_t t = 0;  // streamed groups so far: the ring advances only on these
      for (int64_t g = 0; g < n_groups; ++g) {
        if (group_rebuilt(mask, g)) continue;
        const int s = (int)(t % kTmaStages);
        const uint32_t use = (uint32_t)(t / kTmaStages);
        ++t;
        if (use > 0) mbar_wait(&empty[s], (use - 1) & 1);
        const int64_t r0 = r_begin + g * kTmaRows;
        const int rows = (int)min((int64_t)kTmaRows, r_end - r0);
        mbar_expect_tx(&full[s], rows * row_bytes);
        float* dst = tiles + (size_t)s * kTmaRows * kTmaCols;
        for (int i = 0; i < rows; ++i) bulk_load(dst + (size_t)i * kTmaCols, X + (r0 + i) * row_stride + col0, row_bytes, &full[s]);
      }
    }
    return;
  }

  // ===== consumer warps =====
  const int64_t col = col0 + (int64_t)tid * 4;
  const bool active = col < D;
  const uint32_t sw = key.stream_lo + (stream_off ? __ldg(stream_off) : 0u);
  // the symmetric instantiation only ever runs the symmetric form: saying so lets c0 share sg's registers
  const int frm = SYM ? EVOK_GRAD_SYMMETRIC : form;
  float m[4], sg[4], c1[4], c0[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    sg[c] = active ? __ldg(sigma + col + c) : 1.0f;
    m[c] = active ? __ldg(mu + col + c) : 0.0f;
    grad_coeffs(frm, sg[c], c1[c], c0[c]);
  }
  float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};

  int64_t t = 0;  // streamed groups consumed so far (the producer's ring position)
  for (int64_t g = 0; g < n_groups; ++g) {
    const int64_t r0 = r_begin + g * kTmaRows;
    const int rows = (int)min((int64_t)kTmaRows, r_end - r0);
    float a[kTmaRows], b[kTmaRows];
    bool need[kTmaRows];  // rows whose weights are both zero are skipped, as in grad_partial_kernel: their values never matter
#pragma unroll
    for (int i = 0; i < kTmaRows; ++i) {
      a[i] = b[i] = 0.0f;
      if (i < rows) row_weights<SYM>(w, r0 + i, a[i], b[i]);
      need[i] = a[i] != 0.0f || b[i] != 0.0f;
    }
    if (group_rebuilt(mask, g)) {
      if (active) {
        // every row's Philox chain, unconditionally: one straight-line block keeps kTmaRows independent chains in flight per
        // thread (their latencies overlap) and none of them waits for the weights; `need` gates only the FMA chain, the same as below
        float x[kTmaRows][4];
#pragma unroll
        for (int i = 0; i < kTmaRows; ++i) {
          float z[4];
          normals4(key, sw, unit0 + (uint64_t)(r0 + i), (uint32_t)(col >> 2), z);
#pragma unroll
          for (int c = 0; c < 4; ++c) x[i][c] = fmaf(sg[c], z[c], m[c]);
        }
#pragma unroll
        for (int i = 0; i < kTmaRows; ++i) {
          if (need[i]) {
#pragma unroll
            for (int c = 0; c < 4; ++c) accumulate(a[i], b[i], x[i][c] - m[c], c1[c], c0[c], s1[c], s2[c]);
          }
        }
      }
      continue;
    }
    const int s = (int)(t % kTmaStages);
    const uint32_t use = (uint32_t)(t / kTmaStages);
    ++t;
    mbar_wait(&full[s], use & 1);
    const float4* tile = reinterpret_cast<const float4*>(tiles + (size_t)s * kTmaRows * kTmaCols) + tid;
    if (active) {
      float4 v4[kTmaRows];  // every slot of the stage is loaded (a slot past `rows` holds stale data that is never used)
#pragma unroll
      for (int i = 0; i < kTmaRows; ++i) v4[i] = tile[(size_t)i * (kTmaCols / 4)];
#pragma unroll
      for (int i = 0; i < kTmaRows; ++i) {
        if (need[i]) {
          const float4 v = v4[i];
          const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int c = 0; c < 4; ++c) accumulate(a[i], b[i], x[c] - m[c], c1[c], c0[c], s1[c], s2[c]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  if (active) store_partial<4, false>(partial, blockIdx.y, D, col, s1, s2);
}

// Rebuilt groups per kSplitPeriod when the caller leaves the choice to the library, by the card's enforced power limit
// (scripts/grad_hybrid_bench.py, 1 M x 10 k symmetric).
// - H100 SXM capped at 400 W (kAutoSplitCapped): the pass is bound by power, not by bandwidth or issue.  Streaming alone
//   already draws the cap (the SM clock drops to ~1.1 GHz), rebuilding alone draws it at ~1.9 GHz, and both cost about the
//   same energy per element.  A small rebuilt share fills the idle issue slots of the streaming pass; more shifts the pass
//   towards the slower all-rebuild end (split 0 7.31-7.39 ms, 2 6.72 ms, 4 6.80-6.87 ms, 8 7.30 ms, 16 7.78-7.82 ms; measured
//   before the straight-line rebuild, not re-measured since).
// - H100 80 GB HBM3 at 700 W, 1980 MHz (kAutoSplitFull): the clock holds and the two ends overlap (two sweeps: split 0
//   6.34-6.35 ms, 2 5.63 ms, 4 4.96-4.97 ms, 5 4.65-4.67 ms, 6 4.81-5.00 ms, 8 5.25-5.31 ms, 16 7.00-7.02 ms).
// The limit is read once per device through NVML (read-only); when it cannot be read the capped value is used.
constexpr int kAutoSplitCapped = 2;
constexpr int kAutoSplitFull = 5;
constexpr int64_t kFullPowerMilliwatts = 550000;  // at or above: the full-power sweep applies

static int auto_split_for_power(int64_t milliwatts) { return milliwatts >= kFullPowerMilliwatts ? kAutoSplitFull : kAutoSplitCapped; }

// The enforced power limit of CUDA device `device` in mW, or -1 when NVML or the device is not available.  NVML is opened
// at run time (the library does not link it) and only read.
static int64_t enforced_power_limit_mw(int device) {
  char bus_id[32];
  if (cudaDeviceGetPCIBusId(bus_id, (int)sizeof(bus_id), device) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  void* nvml = dlopen("libnvidia-ml.so.1", RTLD_NOW | RTLD_LOCAL);
  if (!nvml) return -1;
  using init_t = int (*)();
  using by_bus_t = int (*)(const char*, void**);
  using limit_t = int (*)(void*, unsigned int*);
  const auto init = reinterpret_cast<init_t>(dlsym(nvml, "nvmlInit_v2"));
  const auto shutdown = reinterpret_cast<init_t>(dlsym(nvml, "nvmlShutdown"));
  const auto by_bus = reinterpret_cast<by_bus_t>(dlsym(nvml, "nvmlDeviceGetHandleByPciBusId_v2"));
  const auto limit = reinterpret_cast<limit_t>(dlsym(nvml, "nvmlDeviceGetEnforcedPowerLimit"));
  int64_t mw = -1;
  if (init && shutdown && by_bus && limit && init() == 0) {
    void* handle = nullptr;
    unsigned int v = 0;
    if (by_bus(bus_id, &handle) == 0 && limit(handle, &v) == 0) mw = v;
    shutdown();
  }
  dlclose(nvml);
  return mw;
}

// split -1 on the current device: resolved on the first call and kept for the life of the process
static int device_auto_split() {
  constexpr int kMaxDevices = 64;
  static std::atomic<int> resolved[kMaxDevices];  // 0 = not yet, else split + 1
  int device = 0;
  if (cudaGetDevice(&device) != cudaSuccess || device < 0 || device >= kMaxDevices) {
    cudaGetLastError();
    return kAutoSplitCapped;
  }
  int s = resolved[device].load(std::memory_order_relaxed);
  if (s == 0) {
    s = auto_split_for_power(enforced_power_limit_mw(device)) + 1;
    resolved[device].store(s, std::memory_order_relaxed);
  }
  return s - 1;
}

// ------------------------------------------------------------------------------------------------------------
// Host side.  Every entry point describes its call as one GradCall and hands it to run_grad: one plan (plan_grad), one
// partial launch per item chunk (launch_partial) and one finalisation (launch_finalize).  A single search runs as a batch of
// one item: with zero item strides and grid z = 1 it takes the LDG plan a one-item batch takes, unless it qualifies for the
// TMA kernel, which only single searches use.
// ------------------------------------------------------------------------------------------------------------

// One call of the gradient pass.  The constructor takes what every entry point gives; the other fields keep the defaults of a
// single search without Philox counters, peers or separable CMA-ES weights.
struct GradCall {
  GradCall(int form, int eps, const float* w, const float* mu, const float* sigma, int64_t n_rows, int64_t D, float scale_mu, float scale_sigma,
           float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream)
      : form(form), eps(eps), w(w), mu(mu), sigma(sigma), n_rows(n_rows), D(D), scale_mu(scale_mu), scale_sigma(scale_sigma), out_mu(out_mu),
        out_sigma(out_sigma), ws(ws), ws_bytes(ws_bytes), st((cudaStream_t)stream) {}
  int form;
  int eps;                            // where eps comes from: X, or the Philox counters (kEpsRegen / kEpsRebuild)
  const float* w;                     // [items][n_rows]
  const float* mu;                    // NULL with sepw
  const float* sigma;
  int64_t n_rows, D;                  // rows per item, as the caller counts them (the symmetric form pairs them)
  float scale_mu, scale_sigma;
  float* out_mu;                      // [items][D]
  float* out_sigma;
  void* ws;
  size_t ws_bytes;
  cudaStream_t st;
  const float* X = nullptr;           // kEpsRead: [items][n_rows][ldx]
  int64_t ldx = 0;
  int64_t row0 = 0;
  PhiloxKey key{};                    // item b draws on stream word key.stream_lo + b
  const uint32_t* stream_off = nullptr;
  bool batched = false;               // evok_grad_batched / _batched_regen: the LDG plan of a batch, whatever the item count
  int64_t n_items = 1;
  GradItems items{0, 0, 0, 0, 0};     // element strides between the items' operands; run_grad sets .partial from the plan
  int split = 0;                      // rebuilt groups per kSplitPeriod of the TMA kernel (-1 = device_auto_split())
  SepWeights sepw{nullptr, 0, nullptr};  // the separable CMA-ES weight mode, with its weight sums into wsum [items]
  float* wsum = nullptr;
  const GradPush* push = nullptr;     // instead of out_mu / out_sigma: into every peer's slot
};

static bool is_sym(const GradCall& c) { return c.form == EVOK_GRAD_SYMMETRIC; }

// The plan fixes the summation order, and with it the bits: the kernel, the column tiles, and the row chunks of every item.
struct GradPlan {
  bool tma;
  int vec, tx, n_coltiles, n_chunks;  // vec, tx: the LDG kernel's columns per thread and column threads per CTA
  int64_t n_units, units_per_chunk;
};

static void set_chunks(GradPlan& p, int64_t chunks) {
  if (chunks < 1) chunks = 1;
  if (chunks > 65535) chunks = 65535;
  p.units_per_chunk = (p.n_units + chunks - 1) / chunks;
  p.n_chunks = (int)((p.n_units + p.units_per_chunk - 1) / p.units_per_chunk);
}

// EVOK_GRAD_TMA=0 / 1 picks the LDG or TMA kernel, read per call (a getenv is ~100 ns): the parity tests run both in one process
static bool tma_enabled() {
  const char* env = getenv("EVOK_GRAD_TMA");
  return env ? atoi(env) != 0 : EVOK_GRAD_TMA_DEFAULT != 0;
}

// For n_units > 0.
static GradPlan plan_grad(const GradCall& c) {
  GradPlan p{};
  p.n_units = is_sym(c) ? c.n_rows / 2 : c.n_rows;
  // 16-byte columns: always for regenerated rows, else when every item's X, mu and sigma allow them
  const bool vec_ok = c.eps == kEpsRegen || (c.D % 4 == 0 && (c.eps == kEpsRebuild || (c.ldx % 4 == 0 && aligned16(c.X) && c.items.x % 4 == 0)) &&
                                             c.items.mu % 4 == 0 && c.items.sigma % 4 == 0);
  p.vec = vec_ok ? 4 : 1;
  // the TMA kernel: a single search (not a batch, even of one item) over wide stored rows with enough of them to fill its ring
  p.tma = !c.batched && c.eps == kEpsRead && vec_ok && c.form != EVOK_GRAD_MOMENTS && c.D >= 512 && p.n_units >= 4096 && tma_enabled();
  if (p.tma) {
    p.n_coltiles = (int)((c.D + kTmaCols - 1) / kTmaCols);
    set_chunks(p, (int64_t)kNumSMs * EVOK_GRAD_TMA_CTAS_PER_SM / p.n_coltiles);
    return p;
  }
  const int64_t col_threads = (c.D + p.vec - 1) / p.vec;
  p.tx = 32;
  while (p.tx < kGradThreads && p.tx < col_threads) p.tx <<= 1;
  p.n_coltiles = (int)((col_threads + p.tx - 1) / p.tx);
  const int ty = kGradThreads / p.tx;
  int64_t chunks = (int64_t)kNumSMs * kGradCtasPerSm / p.n_coltiles;  // one wave of resident CTAs
  // at least 16 unrolled iterations per CTA: fewer, fatter chunks keep the fixed-order finalisation short for small populations
  const int64_t max_useful = (p.n_units + (int64_t)ty * kGradUnroll * 16 - 1) / ((int64_t)ty * kGradUnroll * 16);
  set_chunks(p, chunks < max_useful ? chunks : max_useful);
  // a batch fills the GPU: fewer row chunks per item keep the fixed-order finalisation short (one item never gets fewer).  The
  // separable CMA-ES moments keep the plan of one item for every item, so that item b has the bits of a one-item call.
  chunks = ((int64_t)kNumSMs * kGradCtasPerSm + (int64_t)p.n_coltiles * c.n_items - 1) / ((int64_t)p.n_coltiles * c.n_items);
  if (chunks < p.n_chunks && !c.wsum) set_chunks(p, chunks);
  // The rebuild always runs 4 columns per thread: one Philox group gives all 4 (a thread per column would draw each group 4
  // times).  A column's sum depends only on the row threads per CTA (kGradThreads / tx) and the row chunks, so for the scalar
  // plan it keeps that plan's tx and chunks, with a quarter of its column tiles, and gives the scalar read path's bits.
  if (c.eps == kEpsRebuild && !vec_ok) {
    p.vec = 4;
    p.n_coltiles = (int)(((c.D + 3) / 4 + p.tx - 1) / p.tx);
  }
  return p;
}

// Every instantiation of grad_partial_kernel, by [row][tx]: row partial_row(...), tx 32, 64, 128, 256
using PartialKernel = void (*)(int, const float*, int64_t, const float*, const float*, const float*, int64_t, int64_t, int64_t, uint64_t,
                               PhiloxKey, const uint32_t*, float*, GradItems, SepWeights);
#define EVOK_GRAD_TXS(VEC, SYM, EPS, SEPW)                                                                             \
  {                                                                                                                    \
    grad_partial_kernel<VEC, 32, SYM, EPS, SEPW>, grad_partial_kernel<VEC, 64, SYM, EPS, SEPW>,                        \
        grad_partial_kernel<VEC, 128, SYM, EPS, SEPW>, grad_partial_kernel<VEC, 256, SYM, EPS, SEPW>                   \
  }
static const PartialKernel kPartialKernels[12][4] = {
    EVOK_GRAD_TXS(1, false, kEpsRead, false),    EVOK_GRAD_TXS(1, true, kEpsRead, false),  EVOK_GRAD_TXS(4, false, kEpsRead, false),
    EVOK_GRAD_TXS(4, true, kEpsRead, false),     EVOK_GRAD_TXS(4, false, kEpsRegen, false), EVOK_GRAD_TXS(4, true, kEpsRegen, false),
    EVOK_GRAD_TXS(4, false, kEpsRebuild, false), EVOK_GRAD_TXS(4, true, kEpsRebuild, false), EVOK_GRAD_TXS(4, false, kEpsRegen, true),
    EVOK_GRAD_TXS(1, false, kEpsRead, true),     EVOK_GRAD_TXS(4, false, kEpsRead, true),  EVOK_GRAD_TXS(4, false, kEpsRebuild, true)};
#undef EVOK_GRAD_TXS

// (eps, vec, sym): the read kernels by vec, then one pair of rows per Philox mode; the SEPW mode: regenerated, read by vec, rebuilt
static int partial_row(int eps, int vec, bool sym, bool sepw) {
  if (sepw) return eps == kEpsRegen ? 8 : eps == kEpsRead ? 9 + vec / 4 : 11;
  return 2 * (eps == kEpsRead ? vec / 4 : 1 + eps) + (sym ? 1 : 0);
}
static int tx_index(int tx) { return tx == 32 ? 0 : tx == 64 ? 1 : tx == 128 ? 2 : 3; }

// The partial sums of item chunk [b0, b0 + nb) into partial[item - b0][chunk][2][D]
static void launch_partial(const GradCall& c, const GradPlan& p, int64_t b0, int64_t nb, float* partial) {
  PhiloxKey key = c.key;
  key.stream_lo += (uint32_t)b0;  // item b0 + z on stream word stream_lo + b0 + z, as the batched sampler draws it
  const float* X = c.X + b0 * c.items.x;
  const float* w = c.w + b0 * c.items.w;
  const float* mu = c.mu + b0 * c.items.mu;
  const float* sigma = c.sigma + b0 * c.items.sigma;
  // symmetric sampling keys its counters by direction; the regenerating kernel must use the same unit index
  const uint64_t unit0 = (uint64_t)(is_sym(c) ? c.row0 / 2 : c.row0);
  if (p.tma) {
    const int rebuilt = c.split < 0 ? device_auto_split() : c.split;
    auto kernel = is_sym(c) ? grad_partial_tma_kernel<true> : grad_partial_tma_kernel<false>;
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmemBytes);
    kernel<<<dim3(p.n_coltiles, p.n_chunks), kTmaThreads, kTmaSmemBytes, c.st>>>(c.form, X, c.ldx, w, mu, sigma, p.n_units, c.D, p.units_per_chunk,
                                                                                  rebuilt, unit0, key, c.stream_off, partial);
    return;
  }
  SepWeights sepw = c.sepw;
  if (sepw.q) sepw.q += b0 * c.items.w;  // the squared norms have the layout of w
  const PartialKernel kernel = kPartialKernels[partial_row(c.eps, p.vec, is_sym(c), c.wsum != nullptr)][tx_index(p.tx)];
  kernel<<<dim3(p.n_coltiles, p.n_chunks, (unsigned)nb), kGradThreads, 0, c.st>>>(c.form, X, c.ldx, w, mu, sigma, p.n_units, c.D,
                                                                                    p.units_per_chunk, unit0, key, c.stream_off, partial, c.items, sepw);
}

// Adds the n_chunks row chunks of item chunk [b0, b0 + nb) in order into the outputs: out_mu / out_sigma (with the SEPW weight
// sum into *wsum), or this rank's slot of every peer (push)
static int launch_finalize(const GradCall& c, int n_chunks, int64_t b0, int64_t nb, const float* partial) {
  const unsigned grid = (unsigned)((c.D + 255) / 256);
  if (c.push) {
    grad_finalize_push_kernel<<<grid, 256, 0, c.st>>>(partial, n_chunks, c.D, c.scale_mu, c.scale_sigma, c.push->sink, c.push->epoch, c.push->done);
  } else if (c.wsum) {
    grad_finalize_kernel<true><<<dim3(grid, (unsigned)nb), 256, 0, c.st>>>(partial, n_chunks, c.D, c.scale_mu, c.scale_sigma, c.out_mu + b0 * c.D,
                                                                           c.out_sigma + b0 * c.D, c.items.partial, c.sepw.wsum_partial, c.wsum + b0);
  } else {
    grad_finalize_kernel<<<dim3(grid, (unsigned)nb), 256, 0, c.st>>>(partial, n_chunks, c.D, c.scale_mu, c.scale_sigma, c.out_mu + b0 * c.D,
                                                                     c.out_sigma + b0 * c.D, c.items.partial);
  }
  EVOK_CHECK_LAUNCH();
  return 0;
}

// A checked call: the empty case, the plan, then the partial and final kernels of every item chunk
static int run_grad(GradCall c) {
  if (c.n_items == 0) return 0;
  float* partial = (float*)c.ws;
  if ((is_sym(c) ? c.n_rows / 2 : c.n_rows) == 0) {
    if (c.push) return launch_finalize(c, 0, 0, 1, partial);  // zeros + this rank's flag
    cudaMemsetAsync(c.out_mu, 0, (size_t)c.n_items * c.D * 4, c.st);
    cudaMemsetAsync(c.out_sigma, 0, (size_t)c.n_items * c.D * 4, c.st);
    return 0;
  }
  const GradPlan p = plan_grad(c);  // after the empty case: the plan divides by the units per chunk
  c.items.partial = (int64_t)p.n_chunks * 2 * c.D;
  // grid z / y hold at most kMaxGridY items: larger batches run as item chunks with the plan above, in order on the stream, each
  // reusing the partial sums of the previous one
  const int64_t chunk = c.n_items < kMaxGridY ? c.n_items : kMaxGridY;
  if (c.ws_bytes < (size_t)chunk * c.items.partial * sizeof(float)) return EVOK_E_WORKSPACE;
  return for_item_chunks(c.n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    launch_partial(c, p, b0, nb, partial);
    EVOK_CHECK_LAUNCH();
    return launch_finalize(c, p.n_chunks, b0, nb, partial);
  });
}

static bool bad_form(int form) { return form < EVOK_GRAD_SEPARABLE || form > EVOK_GRAD_MOMENTS; }

// The checks of evok_grad, _regen, _hybrid and _push (after the push's own), in this order, then the pass
static int grad_single(const GradCall& c) {
  const bool read = c.eps == kEpsRead;
  // an empty shard has no weights to point at (an empty CUDA tensor's data pointer is NULL)
  if ((!c.w && c.n_rows != 0) || !c.mu || !c.sigma || !c.ws || (read && !c.X) || (!c.push && (!c.out_mu || !c.out_sigma))) return EVOK_E_NULLPTR;
  if (bad_form(c.form)) return EVOK_E_BADENUM;
  if (c.n_rows < 0 || c.D <= 0 || c.row0 < 0 || (read && c.ldx < c.D) || c.split < -1 || c.split > kSplitPeriod) return EVOK_E_BADSIZE;
  if (is_sym(c) && ((c.n_rows & 1) || (c.row0 & 1))) return EVOK_E_ODDROWS;
  if (c.ws_bytes < evok_grad_workspace_bytes(c.n_rows, c.D)) return EVOK_E_WORKSPACE;
  return run_grad(c);
}

// The checks of evok_grad_batched and evok_grad_batched_regen, in this order, then the pass
static int grad_batched(const GradCall& c) {
  const bool read = c.eps == kEpsRead;
  if ((read && !c.X) || !c.w || !c.mu || !c.sigma || !c.out_mu || !c.out_sigma || !c.ws) return EVOK_E_NULLPTR;
  if (bad_form(c.form)) return EVOK_E_BADENUM;
  if (c.n_items < 0 || c.n_rows < 0 || c.D <= 0 || (read && c.ldx < c.D) || c.items.x < 0 || c.items.mu < 0 || c.items.sigma < 0)
    return EVOK_E_BADSIZE;
  if (is_sym(c) && (c.n_rows & 1)) return EVOK_E_ODDROWS;
  return run_grad(c);
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API size_t evok_grad_workspace_bytes(int64_t n_rows, int64_t D) {
  (void)n_rows;
  if (D <= 0) return 256;
  // n_chunks * n_coltiles <= kMaxResidentCtas/2 + n_coltiles and every column tile spans <= 1024 columns
  return ((size_t)kMaxResidentCtas * 1024 + 2 * (size_t)D + 64) * sizeof(float);
}

extern "C" EVOK_API int evok_grad(int form, const float* X, int64_t ldx, const float* w, const float* mu, const float* sigma, int64_t n_rows,
                         int64_t D, float scale_mu, float scale_sigma, float* out_mu, float* out_sigma, void* ws, size_t ws_bytes,
                         void* stream) {
  GradCall c(form, kEpsRead, w, mu, sigma, n_rows, D, scale_mu, scale_sigma, out_mu, out_sigma, ws, ws_bytes, stream);
  c.X = X;
  c.ldx = ldx;
  return grad_single(c);
}

extern "C" EVOK_API int evok_grad_regen(int form, const float* w, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D,
                               uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float scale_mu, float scale_sigma,
                               float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream) {
  GradCall c(form, kEpsRegen, w, mu, sigma, n_rows, D, scale_mu, scale_sigma, out_mu, out_sigma, ws, ws_bytes, stream);
  c.row0 = row0;
  c.key = make_philox_key(seed, stream_id);
  c.stream_off = stream_offset_dev;
  return grad_single(c);
}

// split: rebuilt groups per kSplitPeriod in the TMA kernel (0 = stream every row, -1 = device_auto_split()); rows are rebuilt from
// (seed, stream_id, *stream_off, row0), which must be the counters that sampled X from this mu and sigma.
extern "C" EVOK_API int evok_grad_hybrid(int form, const float* X, int64_t ldx, const float* w, const float* mu, const float* sigma, int64_t row0,
                                         int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, int split,
                                         float scale_mu, float scale_sigma, float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream) {
  GradCall c(form, kEpsRead, w, mu, sigma, n_rows, D, scale_mu, scale_sigma, out_mu, out_sigma, ws, ws_bytes, stream);
  c.X = X;
  c.ldx = ldx;
  c.row0 = row0;
  c.key = make_philox_key(seed, stream_id);
  c.stream_off = stream_offset_dev;
  c.split = split;
  return grad_single(c);
}

extern "C" EVOK_API int evok_grad_auto_split(int64_t power_limit_mw) { return auto_split_for_power(power_limit_mw); }

extern "C" EVOK_API int64_t evok_grad_power_limit_mw(int device) { return enforced_power_limit_mw(device); }

extern "C" EVOK_API size_t evok_sepcma_workspace_bytes(int64_t n_rows, int64_t D) {
  // the gradient partials, then one float per row chunk (plan_grad: at most kNumSMs * kGradCtasPerSm chunks)
  return evok_grad_workspace_bytes(n_rows, D) + (size_t)kMaxResidentCtas * sizeof(float);
}

extern "C" EVOK_API int evok_sepcma_moments(const float* aw, const float* q, int active, int64_t row0, int64_t n_rows, int64_t D, uint64_t seed,
                                            uint64_t stream_id, const uint32_t* stream_offset_dev, float* local, float* S2, float* wsum, void* ws,
                                            size_t ws_bytes, void* stream) {
  if (!aw || (active && !q) || !local || !S2 || !wsum || !ws) return EVOK_E_NULLPTR;
  if (n_rows <= 0 || D <= 0 || row0 < 0) return EVOK_E_BADSIZE;
  if (ws_bytes < evok_sepcma_workspace_bytes(n_rows, D)) return EVOK_E_WORKSPACE;
  GradCall c(EVOK_GRAD_MOMENTS, kEpsRegen, aw, nullptr, nullptr, n_rows, D, 1.0f, 1.0f, local, S2, ws, ws_bytes, stream);
  c.row0 = row0;
  c.key = make_philox_key(seed, stream_id);
  c.stream_off = stream_offset_dev;
  c.sepw = SepWeights{q, active, (float*)ws + evok_grad_workspace_bytes(n_rows, D) / sizeof(float)};
  c.wsum = wsum;
  return run_grad(c);
}

extern "C" EVOK_API int evok_grad_push(int form, const float* X, int64_t ldx, const float* w, const float* mu, const float* sigma, int64_t row0,
                                       int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev,
                                       float scale_mu, float scale_sigma, int world, int rank, void* const* peer_slots, void* const* peer_flags,
                                       const uint64_t* epoch_dev, uint32_t* done_dev, void* ws, size_t ws_bytes, void* stream) {
  if (!peer_slots || !peer_flags || !epoch_dev || !done_dev) return EVOK_E_NULLPTR;
  if (world < 1 || world > EVOK_MAX_PEERS || rank < 0 || rank >= world) return EVOK_E_BADSIZE;
  GradPush push{};
  push.sink.world = world;
  push.sink.rank = rank;
  for (int p = 0; p < world; ++p) {
    if (!peer_slots[p] || !peer_flags[p]) return EVOK_E_NULLPTR;
    push.sink.data[p] = peer_slots[p];
    push.sink.flags[p] = static_cast<unsigned long long*>(peer_flags[p]);
  }
  push.epoch = reinterpret_cast<const unsigned long long*>(epoch_dev);
  push.done = done_dev;
  GradCall c(form, X ? kEpsRead : kEpsRegen, w, mu, sigma, n_rows, D, scale_mu, scale_sigma, nullptr, nullptr, ws, ws_bytes, stream);
  c.X = X;
  c.ldx = X ? ldx : 0;
  c.row0 = row0;
  c.key = make_philox_key(seed, stream_id);
  c.stream_off = stream_offset_dev;
  c.push = &push;
  return grad_single(c);
}

// Batched searches: n_items independent weighted column reductions in ONE launch chain (blockIdx.z = item).  X: [items][n_rows][D]
// (item stride item_stride_x elements), w: [items][n_rows] contiguous, mu / sigma: item strides (0 = shared by all items),
// outputs contiguous [items][D].  Same arithmetic as evok_grad per item (LDG kernel, fixed-order two-stage reduction).
extern "C" EVOK_API size_t evok_grad_batched_workspace_bytes(int64_t n_items, int64_t n_rows, int64_t D) {
  if (n_items <= 0 || D <= 0) return 256;
  (void)n_rows;
  // all items together use about one wave of CTAs: sum over items of n_chunks * 2 * D <= (592 / coltiles) * 2 * D + (2 per item of slack) * 2 * D
  return ((size_t)kMaxResidentCtas * 1024 + 4 * (size_t)n_items * (size_t)D + 64) * sizeof(float);
}

extern "C" EVOK_API int evok_grad_batched(int form, const float* X, int64_t item_stride_x, int64_t ldx, const float* w, const float* mu,
                                          int64_t item_stride_mu, const float* sigma, int64_t item_stride_sigma, int64_t n_items, int64_t n_rows,
                                          int64_t D, float scale_mu, float scale_sigma, float* out_mu, float* out_sigma, void* ws, size_t ws_bytes,
                                          void* stream) {
  GradCall c(form, kEpsRead, w, mu, sigma, n_rows, D, scale_mu, scale_sigma, out_mu, out_sigma, ws, ws_bytes, stream);
  c.X = X;
  c.ldx = ldx;
  c.batched = true;
  c.n_items = n_items;
  c.items = GradItems{item_stride_x, n_rows, item_stride_mu, item_stride_sigma, 0};
  return grad_batched(c);
}

// Every needed row rebuilt from (seed, stream_id0 + item) as the batched sampler stored it.  The rebuilt rows take the plan of a
// contiguous, 16-byte aligned X [items][n_rows][D], so both entry points give the same bits.
extern "C" EVOK_API int evok_grad_batched_regen(int form, const float* w, const float* mu, int64_t item_stride_mu, const float* sigma,
                                                int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, uint64_t seed,
                                                uint64_t stream_id0, float scale_mu, float scale_sigma, float* out_mu, float* out_sigma, void* ws,
                                                size_t ws_bytes, void* stream) {
  GradCall c(form, kEpsRebuild, w, mu, sigma, n_rows, D, scale_mu, scale_sigma, out_mu, out_sigma, ws, ws_bytes, stream);
  c.key = make_philox_key(seed, stream_id0);
  c.batched = true;
  c.n_items = n_items;
  c.items = GradItems{0, n_rows, item_stride_mu, item_stride_sigma, 0};
  return grad_batched(c);
}

// Separable CMA-ES moments of a batch of searches over the steps recovered from their rows.  Every item has the plan of one item,
// whose row chunks depend only on the columns per thread: the most chunks of either width (16-byte rows, or the scalar plan that
// unaligned stored rows and rebuilt rows with D % 4 != 0 take).  The workspace holds the partial sums of the column pass and the
// per-chunk weight sums of at most kMaxGridY items, then q [items][n_rows].
static size_t round256(size_t b) { return (b + 255) / 256 * 256; }
static int64_t sepcma_max_chunks(int64_t n_rows, int64_t D) {
  int64_t most = 1;
  for (int scalar = 0; scalar < 2; ++scalar) {
    GradCall c(EVOK_GRAD_MOMENTS, scalar ? kEpsRead : kEpsRebuild, nullptr, nullptr, nullptr, n_rows, D, 1.0f, 1.0f, nullptr, nullptr, nullptr, 0,
               nullptr);
    c.ldx = D + 1;  // rows whose pitch rules out 16-byte loads
    c.batched = true;
    const GradPlan p = plan_grad(c);
    if (p.n_chunks > most) most = p.n_chunks;
  }
  return most;
}
static int64_t item_chunk(int64_t n_items) { return n_items < kMaxGridY ? n_items : kMaxGridY; }
static size_t sepcma_batched_grad_bytes(int64_t n_items, int64_t n_rows, int64_t D) {
  return round256((size_t)item_chunk(n_items) * (size_t)sepcma_max_chunks(n_rows, D) * 2 * (size_t)D * sizeof(float));
}
static size_t sepcma_batched_wsum_bytes(int64_t n_items, int64_t n_rows, int64_t D) {
  return round256((size_t)item_chunk(n_items) * (size_t)sepcma_max_chunks(n_rows, D) * sizeof(float));
}

extern "C" EVOK_API size_t evok_sepcma_moments_batched_workspace_bytes(int64_t n_items, int64_t n_rows, int64_t D) {
  if (n_items <= 0 || n_rows <= 0 || D <= 0) return 256;
  return sepcma_batched_grad_bytes(n_items, n_rows, D) + sepcma_batched_wsum_bytes(n_items, n_rows, D) + (size_t)n_items * (size_t)n_rows * sizeof(float);
}

extern "C" EVOK_API int evok_sepcma_moments_batched(const float* X, int64_t item_stride_x, int64_t ldx, const float* m, const float* s, const float* aw,
                                                    int active, int64_t n_items, int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id0,
                                                    float* local, float* S2, float* wsum, void* ws, size_t ws_bytes, void* stream) {
  if (!m || !s || !aw || !local || !S2 || !wsum || !ws) return EVOK_E_NULLPTR;
  if (n_items < 0 || n_rows <= 0 || D <= 0 || (X && (ldx < D || item_stride_x < 0))) return EVOK_E_BADSIZE;
  if (n_items == 0) return 0;
  if (ws_bytes < evok_sepcma_moments_batched_workspace_bytes(n_items, n_rows, D)) return EVOK_E_WORKSPACE;
  const size_t grad_bytes = sepcma_batched_grad_bytes(n_items, n_rows, D);
  float* wsum_partial = (float*)((char*)ws + grad_bytes);
  float* q = active ? (float*)((char*)ws + grad_bytes + sepcma_batched_wsum_bytes(n_items, n_rows, D)) : nullptr;
  const cudaStream_t st = (cudaStream_t)stream;
  const PhiloxKey key = make_philox_key(seed, stream_id0);
  if (active) {  // the row pass: q of the rows with a negative weight, before the column pass reads it
    const int rc = for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
      PhiloxKey kc = key;
      kc.stream_lo += (uint32_t)b0;
      const dim3 grid((unsigned)((n_rows + 7) / 8), (unsigned)nb);
      const float* Xc = X ? X + b0 * item_stride_x : nullptr;
      if (X)
        sepcma_sqnorm_kernel<kEpsRead><<<grid, 256, 0, st>>>(Xc, item_stride_x, ldx, m + b0 * D, s + b0 * D, aw + b0 * n_rows, n_rows, D, kc,
                                                             q + b0 * n_rows);
      else
        sepcma_sqnorm_kernel<kEpsRebuild><<<grid, 256, 0, st>>>(nullptr, 0, 0, m + b0 * D, s + b0 * D, aw + b0 * n_rows, n_rows, D, kc,
                                                                q + b0 * n_rows);
      EVOK_CHECK_LAUNCH();
      return 0;
    });
    if (rc) return rc;
  }
  GradCall c(EVOK_GRAD_MOMENTS, X ? kEpsRead : kEpsRebuild, aw, m, s, n_rows, D, 1.0f, 1.0f, local, S2, ws, grad_bytes, stream);
  c.X = X;
  c.ldx = X ? ldx : 0;
  c.key = key;
  c.batched = true;
  c.n_items = n_items;
  c.items = GradItems{X ? item_stride_x : 0, n_rows, D, D, 0};
  c.sepw = SepWeights{q, active, wsum_partial};
  c.wsum = wsum;
  return run_grad(c);
}
