// Functional XNES (Glasmachers et al., GECCO 2010) for a batch of independent searches at small D: the symmetric matrix
// exponential pair F+- = expm(+-S) - I, and the tell that uses it, one CTA per item, on the CUDA cores in shared memory.
//
// The exponential is kept in the expm1 form F = e^S - I, so that a tiny S keeps its relative precision instead of vanishing
// against I: the updates are A' = A + A F+ and A_inv' = A_inv + F- A_inv.  Scaling and squaring:
//   s = max(0, ceil(log2(|S|_1 / theta))) per item, on the device; X = S / 2^s (exact: a power of two);
//   Taylor core in Y = X^2: U = sum_{i=1..q} Y^i / (2i)!, V = X sum_{i=0..q} Y^i / (2i+1)!  (the even and odd parts of e^X - I);
//   F+ = U + V, F- = U - V: one set of powers serves both signs; then F <- 2F + F^2, s times for each sign.
// theta = 1 and q = 5 (degree 11): with |X|_2 <= |X|_1 <= 1 the first omitted terms are at most 1/12! = 2.1e-9 (U) and
// 1/13! = 1.6e-10 (V), while |e^X - I|_2 >= (1 - 1/e) |X|_2 for a symmetric X; so the truncation lies below
// 2.1e-9 / 0.63 = 3.3e-9 relative to F, under float32 rounding (2^-24 = 6.0e-8) at every |X|.
//
// Every product is one CTA-wide pass over matrices in shared memory at an odd row pitch (D + 1): thread (ti, tj) of 16 x 16
// owns entries (ti + 16 a, tj + 16 b), a, b < PER = ceil(D / 16) rounded up to 1, 2, 4 or 6, and sums over k in order, so an item
// gives the bits of a one-item call.  The
// working set is four D x (D + 1) float32 matrices: 145.5 KB at D = EVOK_XNES_MAX_D = 96, inside the 227 KB a CTA can take.
#include <cmath>
#include <type_traits>

#include "evok_common.cuh"

namespace evok {
namespace {

constexpr int kXnThreads = 256;
constexpr int kXnSide = 16;  // threads per side of the output grid
constexpr int kXnMaxD = EVOK_XNES_MAX_D;
static_assert(kXnSide * kXnSide == kXnThreads && kXnMaxD % kXnSide == 0, "the thread grid covers the largest matrix");

// Taylor coefficients of the core: U = Y (a0 + a1 Y + ... + a4 Y^4), a_i = 1 / (2i + 2)!; V = X (b0 + b1 Y + ... + b5 Y^5),
// b_i = 1 / (2i + 1)!.
__constant__ float kXnA[5] = {1.0f / 2.0f, 1.0f / 24.0f, 1.0f / 720.0f, 1.0f / 40320.0f, 1.0f / 3628800.0f};
__constant__ float kXnB[6] = {1.0f, 1.0f / 6.0f, 1.0f / 120.0f, 1.0f / 5040.0f, 1.0f / 362880.0f, 1.0f / 39916800.0f};

// C[i][j] = sum_{k < K} A[i][k] B[k][j] (k in order, from 0) + p E[i][j] + q [i == j], for i < M, j < N <= 16 PER.  A, B, E in
// shared memory at pitch ld; C at pitch ldc, in shared or global memory.  Every thread reads before any writes, so C may be A, B
// or E (in place).  PER, the outputs per thread and side, only sets how many registers a thread holds: an entry's sum is the
// same for every PER that covers D, so the kernels take the smallest (more CTAs fit on an SM at small D).
template <int PER>
__device__ __forceinline__ void xn_mm(const float* A, const float* B, int M, int N, int K, int ld, const float* E, float p, float q, float* C,
                                      int ldc) {
  const int ti = threadIdx.x / kXnSide, tj = threadIdx.x % kXnSide;
  float acc[PER][PER];
#pragma unroll
  for (int a = 0; a < PER; ++a)
#pragma unroll
    for (int b = 0; b < PER; ++b) acc[a][b] = 0.0f;
  for (int k = 0; k < K; ++k) {
    float av[PER], bv[PER];
#pragma unroll
    for (int a = 0; a < PER; ++a) {
      const int i = ti + kXnSide * a, j = tj + kXnSide * a;
      av[a] = i < M ? A[i * ld + k] : 0.0f;
      bv[a] = j < N ? B[k * ld + j] : 0.0f;
    }
#pragma unroll
    for (int a = 0; a < PER; ++a)
#pragma unroll
      for (int b = 0; b < PER; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
  }
  __syncthreads();
#pragma unroll
  for (int a = 0; a < PER; ++a) {
    const int i = ti + kXnSide * a;
#pragma unroll
    for (int b = 0; b < PER; ++b) {
      const int j = tj + kXnSide * b;
      if (i < M && j < N) {
        float v = acc[a][b];
        if (E) v = fmaf(p, E[i * ld + j], v);
        if (i == j) v += q;
        C[i * ldc + j] = v;
      }
    }
  }
  __syncthreads();
}

// The exponential pair of the D x D matrix in sX (pitch ld = D + 1): on return sX = F+ = e^S - I and sY = F- = e^-S - I.  sU and
// sV are work matrices; red holds >= 33 floats.  A non-finite S takes s = 0 and gives non-finite F.
template <int PER>
__device__ void xn_expm_pair(float* sX, float* sY, float* sU, float* sV, int D, float* red) {
  const int ld = D + 1, n = D * D;
  float col = 0.0f;  // |S|_1: the largest column sum of |S_ij|, rows in order
  if ((int)threadIdx.x < D)
    for (int i = 0; i < D; ++i) col += fabsf(sX[i * ld + threadIdx.x]);
  // the largest of non-negative floats (NaN kept): fmaxf drops a NaN, so non-finite sums are flagged apart
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  if (!(col <= 3.402823466e38f)) bad = 1;
  float nrm = col;
  for (int o = kWarp / 2; o > 0; o >>= 1) nrm = fmaxf(nrm, __shfl_xor_sync(0xffffffffu, nrm, o));
  if ((threadIdx.x & (kWarp - 1)) == 0) red[threadIdx.x / kWarp] = nrm;
  __syncthreads();
  nrm = 0.0f;
  for (int w = 0; w < kXnThreads / kWarp; ++w) nrm = fmaxf(nrm, red[w]);
  int s = 0;
  if (!bad && nrm > 1.0f) {  // theta = 1: s = ceil(log2 |S|_1), exactly from the bits of the (normal) float 1.f 2^e
    const unsigned bits = __float_as_uint(nrm);
    s = (int)((bits >> 23) & 0xffu) - 127 + ((bits & 0x7fffffu) != 0u);
  }
  for (int e = threadIdx.x; e < n; e += kXnThreads) {
    const int i = e / D, j = e % D;
    sX[i * ld + j] = ldexpf(sX[i * ld + j], -s);
  }
  __syncthreads();
  xn_mm<PER>(sX, sX, D, D, D, ld, nullptr, 0.0f, 0.0f, sY, ld);  // Y = X^2
  for (int e = threadIdx.x; e < n; e += kXnThreads) {
    const int i = e / D, j = e % D;
    const float y = sY[i * ld + j];
    sU[i * ld + j] = fmaf(kXnA[4], y, i == j ? kXnA[3] : 0.0f);
    sV[i * ld + j] = fmaf(kXnB[5], y, i == j ? kXnB[4] : 0.0f);
  }
  __syncthreads();
  for (int t = 2; t >= 0; --t) xn_mm<PER>(sY, sU, D, D, D, ld, nullptr, 0.0f, kXnA[t], sU, ld);
  for (int t = 3; t >= 0; --t) xn_mm<PER>(sY, sV, D, D, D, ld, nullptr, 0.0f, kXnB[t], sV, ld);
  xn_mm<PER>(sY, sU, D, D, D, ld, nullptr, 0.0f, 0.0f, sU, ld);  // U
  xn_mm<PER>(sX, sV, D, D, D, ld, nullptr, 0.0f, 0.0f, sV, ld);  // V
  for (int e = threadIdx.x; e < n; e += kXnThreads) {
    const int at = (e / D) * ld + e % D;
    const float u = sU[at], v = sV[at];
    sX[at] = u + v;
    sY[at] = u - v;
  }
  __syncthreads();
  for (int r = 0; r < s; ++r) {
    xn_mm<PER>(sX, sX, D, D, D, ld, sX, 2.0f, 0.0f, sX, ld);
    xn_mm<PER>(sY, sY, D, D, D, ld, sY, 2.0f, 0.0f, sY, ld);
  }
}

// CTAs per SM the register budget is set for: at small D more items run at once (their shared memory is small).
constexpr int xn_min_ctas(int per) { return per == 1 ? 5 : per == 2 ? 4 : 1; }

size_t xn_smem(int64_t D) { return (size_t)(4 * D * (D + 1) + 3 * D + 40) * sizeof(float); }

template <int PER>
__global__ void __launch_bounds__(kXnThreads, xn_min_ctas(PER)) sym_expm_pair_kernel(const float* __restrict__ S, int D, float* __restrict__ Fp,
                                                                   float* __restrict__ Fm) {
  extern __shared__ float xn_smem_f[];
  const int ld = D + 1, n = D * D;
  float* sX = xn_smem_f;
  float* sY = sX + D * ld;
  float* sU = sY + D * ld;
  float* sV = sU + D * ld;
  float* red = sV + D * ld;
  const int64_t item = blockIdx.x;
  S += item * n;
  for (int e = threadIdx.x; e < n; e += kXnThreads) sX[(e / D) * ld + e % D] = S[e];
  __syncthreads();
  xn_expm_pair<PER>(sX, sY, sU, sV, D, red);
  Fp += item * n;
  Fm += item * n;
  for (int e = threadIdx.x; e < n; e += kXnThreads) {
    const int at = (e / D) * ld + e % D;
    Fp[e] = sX[at];
    Fm[e] = sY[at];
  }
}

// The XNES tell of one item per CTA, from its rows X [n_rows][D] and their utilities w [n_rows] (ranked, and centred where the
// ranking needs it):
//   z_r = A_inv (x_r - mu) for the rows with a non-zero weight, in blocks of up to D rows (A_inv^T staged in shared memory);
//   d = sum_r w_r z_r and G = sum_r w_r z_r z_r^T (rows in order, G in registers), S = (lr_A / 2)(G - (sum_r w_r) I);
//   the exponential pair of S; mu' = mu + A (lr_mu d), A' = A + A F+, A_inv' = A_inv + F- A_inv.
template <int PER>
__global__ void __launch_bounds__(kXnThreads, xn_min_ctas(PER)) xnes_tell_kernel(const float* __restrict__ X, const float* __restrict__ w, const float* __restrict__ mu,
                                                               const float* __restrict__ A, const float* __restrict__ A_inv, int64_t n_rows, int D,
                                                               float lr_mu, float half_lr_A, float* __restrict__ mu_out, float* __restrict__ A_out,
                                                               float* __restrict__ A_inv_out) {
  extern __shared__ float xn_smem_f[];
  const int ld = D + 1, n = D * D;
  float* s0 = xn_smem_f;
  float* s1 = s0 + D * ld;
  float* s2 = s1 + D * ld;
  float* s3 = s2 + D * ld;
  float* red = s3 + D * ld;          // 40
  float* wblk = red + 40;            // [D]: weights of the block's rows
  float* vec = wblk + D;             // [D]: lr_mu d
  int* rows = (int*)(vec + D);       // [D]: the block's rows
  __shared__ int nb_s;
  __shared__ int64_t cursor_s;
  __shared__ float wsum_s;
  const int64_t item = blockIdx.x;
  X += item * n_rows * D;
  w += item * n_rows;
  mu += item * D;
  A += item * n;
  A_inv += item * n;
  const int ti = threadIdx.x / kXnSide, tj = threadIdx.x % kXnSide;
  for (int e = threadIdx.x; e < n; e += kXnThreads) s0[(e % D) * ld + e / D] = A_inv[e];  // A_inv^T
  if (threadIdx.x == 0) {
    cursor_s = 0;
    wsum_s = 0.0f;
  }
  float g[PER][PER];
#pragma unroll
  for (int a = 0; a < PER; ++a)
#pragma unroll
    for (int b = 0; b < PER; ++b) g[a][b] = 0.0f;
  float dacc = 0.0f;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) {  // the next (up to) D rows with a non-zero weight, in order
      int nb = 0;
      int64_t r = cursor_s;
      float ws = wsum_s;
      for (; r < n_rows && nb < D; ++r) {
        const float wr = w[r];
        if (wr != 0.0f) {
          rows[nb] = (int)r;
          wblk[nb] = wr;
          ws += wr;
          ++nb;
        }
      }
      cursor_s = r;
      wsum_s = ws;
      nb_s = nb;
    }
    __syncthreads();
    const int nb = nb_s;
    if (nb == 0) break;
    for (int e = threadIdx.x; e < nb * D; e += kXnThreads) {
      const int r = e / D, j = e % D;
      s1[r * ld + j] = X[(int64_t)rows[r] * D + j] - mu[j];
    }
    __syncthreads();
    xn_mm<PER>(s1, s0, nb, D, D, ld, nullptr, 0.0f, 0.0f, s2, ld);  // z rows: (x - mu) A_inv^T
    for (int r = 0; r < nb; ++r) {
      const float wr = wblk[r];
      float zi[PER], zj[PER];
#pragma unroll
      for (int a = 0; a < PER; ++a) {
        const int i = ti + kXnSide * a, j = tj + kXnSide * a;
        zi[a] = i < D ? wr * s2[r * ld + i] : 0.0f;
        zj[a] = j < D ? s2[r * ld + j] : 0.0f;
      }
#pragma unroll
      for (int a = 0; a < PER; ++a)
#pragma unroll
        for (int b = 0; b < PER; ++b) g[a][b] = fmaf(zi[a], zj[b], g[a][b]);
      if ((int)threadIdx.x < D) dacc = fmaf(wr, s2[r * ld + threadIdx.x], dacc);
    }
  }
  const float wsum = wsum_s;
#pragma unroll
  for (int a = 0; a < PER; ++a) {
    const int i = ti + kXnSide * a;
#pragma unroll
    for (int b = 0; b < PER; ++b) {
      const int j = tj + kXnSide * b;
      if (i < D && j < D) s0[i * ld + j] = half_lr_A * (i == j ? g[a][b] - wsum : g[a][b]);
    }
  }
  if ((int)threadIdx.x < D) vec[threadIdx.x] = lr_mu * dacc;
  __syncthreads();
  xn_expm_pair<PER>(s0, s1, s2, s3, D, red);
  for (int e = threadIdx.x; e < n; e += kXnThreads) {
    const int at = (e / D) * ld + e % D;
    s2[at] = A[e];
    s3[at] = A_inv[e];
  }
  __syncthreads();
  if ((int)threadIdx.x < D) {
    const int i = threadIdx.x;
    float v = 0.0f;
    for (int j = 0; j < D; ++j) v = fmaf(s2[i * ld + j], vec[j], v);
    mu_out[item * D + i] = mu[i] + v;
  }
  xn_mm<PER>(s2, s0, D, D, D, ld, s2, 1.0f, 0.0f, A_out + item * n, D);      // A + A F+
  xn_mm<PER>(s1, s3, D, D, D, ld, s3, 1.0f, 0.0f, A_inv_out + item * n, D);  // A_inv + F- A_inv
}

// fn<PER>(): the launch of the instantiation that covers D, after raising its shared-memory limit to the largest D it takes.
template <typename Fn>
int xn_dispatch(int64_t D, Fn&& fn) {
  if (D <= kXnSide) return fn(std::integral_constant<int, 1>{});
  if (D <= 2 * kXnSide) return fn(std::integral_constant<int, 2>{});
  if (D <= 4 * kXnSide) return fn(std::integral_constant<int, 4>{});
  return fn(std::integral_constant<int, kXnMaxD / kXnSide>{});
}

int xn_allow_smem(const void* fn, int per) {
  return (int)cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)xn_smem(kXnSide * per));
}

}  // namespace
}  // namespace evok

using namespace evok;

extern "C" EVOK_API int evok_sym_expm_pair_batched(const float* S, int64_t n_items, int64_t D, float* F_plus, float* F_minus, void* stream) {
  if (!S || !F_plus || !F_minus) return EVOK_E_NULLPTR;
  if (n_items < 0 || D < 1 || D > kXnMaxD) return EVOK_E_BADSIZE;
  if (n_items == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  return xn_dispatch(D, [&](auto per) {
    constexpr int PER = decltype(per)::value;
    if (const int rc = xn_allow_smem((const void*)sym_expm_pair_kernel<PER>, PER)) return rc;
    return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
      sym_expm_pair_kernel<PER><<<(unsigned)nb, kXnThreads, xn_smem(D), st>>>(S + b0 * D * D, (int)D, F_plus + b0 * D * D, F_minus + b0 * D * D);
      EVOK_CHECK_LAUNCH();
      return 0;
    });
  });
}

extern "C" EVOK_API int evok_xnes_tell_batched(const float* X, const float* w, const float* mu, const float* A, const float* A_inv, int64_t n_items,
                                               int64_t n_rows, int64_t D, float lr_mu, float lr_A, float* mu_out, float* A_out, float* A_inv_out,
                                               void* stream) {
  if (!X || !w || !mu || !A || !A_inv || !mu_out || !A_out || !A_inv_out) return EVOK_E_NULLPTR;
  if (n_items < 0 || n_rows < 2 || n_rows > INT32_MAX || D < 1 || D > kXnMaxD) return EVOK_E_BADSIZE;
  if (n_items == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  const float half_lr_A = 0.5f * lr_A;
  return xn_dispatch(D, [&](auto per) {
    constexpr int PER = decltype(per)::value;
    if (const int rc = xn_allow_smem((const void*)xnes_tell_kernel<PER>, PER)) return rc;
    return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
      xnes_tell_kernel<PER><<<(unsigned)nb, kXnThreads, xn_smem(D), st>>>(X + b0 * n_rows * D, w + b0 * n_rows, mu + b0 * D, A + b0 * D * D,
                                                                          A_inv + b0 * D * D, n_rows, (int)D, lr_mu, half_lr_A, mu_out + b0 * D,
                                                                          A_out + b0 * D * D, A_inv_out + b0 * D * D);
      EVOK_CHECK_LAUNCH();
      return 0;
    });
  });
}
