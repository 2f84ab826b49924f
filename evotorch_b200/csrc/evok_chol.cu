// Cholesky factorisation C = L L^T of the CMA-ES covariance matrix (cmaes.py:555-565 `decompose_C`; the reference calls
// torch.linalg.cholesky -> cuSOLVER potrf, the largest single piece of a fused generation).
//
// ONE persistent kernel, tile dataflow instead of a sequence of panel / trsm / syrk launches: the lower triangle is cut into
// 64 x 64 tiles, tile (I, J) belongs to one CTA (column-major order, round-robin), which
//     accumulates      T = A[I,J] - sum_{k<J} L[I,k] L[J,k]^T      as soon as each L[.,k] pair is published (left-looking),
//     diagonal tile:   factorises T (two 32 x 32 in-register warp factorisations + a 32^3 update), inverts the factor,
//                      publishes L[J,J] and its inverse;
//     off-diagonal:    waits for the diagonal tile of its column, L[I,J] = T * inv(L[J,J])^T, publishes it.
// Tiles are published with a release store on a per-tile flag and consumed with acquire loads, so the critical path is
// (factor -> flag -> solve -> flag -> last update) per block column -- 16 columns at D = 1024 -- with no grid-wide barrier and no
// kernel boundary; all other updates run ahead of it.  Every dependency of a tile has a smaller column-major index and every CTA
// handles its tiles in increasing index with all CTAs resident (grid <= number of SMs), so the schedule cannot deadlock.
// fp32 FMA arithmetic (the factorisation is 0.36 GFLOP at D = 1024: latency-, not throughput-bound; no tensor cores needed).
#include "evok_common.cuh"

namespace evok {

constexpr int kCholNB = 64;
constexpr int kCholThreads = 256;
constexpr int kCholPitch = kCholNB + 1;

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// lane i holds row i of a symmetric positive definite 32 x 32 block (entries k <= i are used); on return row i of its
// Cholesky factor (entries k <= i).  496 shuffle + FMA pairs, fully unrolled: everything stays in registers.
__device__ __forceinline__ void chol32_warp(float (&a)[32], int lane) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float ajj = __shfl_sync(0xffffffffu, a[j], j);
    const float d = sqrtf(ajj);
    const float lij = (lane == j) ? d : __fdiv_rn(a[j], d);
    a[j] = lij;
#pragma unroll
    for (int k = j + 1; k < 32; ++k) {
      const float lkj = __shfl_sync(0xffffffffu, lij, k);
      a[k] = fmaf(-lij, lkj, a[k]);
    }
  }
}

// lane i holds row i of a lower-triangular 32 x 32 matrix L (entries k <= i); on return lane j holds COLUMN j of inv(L)
// (entries m[i], i >= j; zeros above the diagonal).
__device__ __forceinline__ void trinv32_warp(const float (&l)[32], float (&m)[32], int lane) {
#pragma unroll
  for (int i = 0; i < 32; ++i) m[i] = 0.0f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    // row i of L, broadcast element by element: m_ij = -(sum_{k=j}^{i-1} l_ik m_kj) / l_ii for j < i, 1 / l_ii for j = i
    const float lii = __shfl_sync(0xffffffffu, l[i], i);
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < i; ++k) {
      const float lik = __shfl_sync(0xffffffffu, l[k], i);
      s = fmaf(lik, m[k], s);  // m[k] = m_kj of this lane's column j (zero for k < j)
    }
    m[i] = (lane == i) ? __fdiv_rn(1.0f, lii) : ((lane < i) ? __fdiv_rn(-s, lii) : 0.0f);
  }
}

// acc[r][c] -= sum_k As[(r*16+ty)][k] * Bs[(c*16+tx)][k]   over a 64 x 64 x kk tile pair in shared memory (pitch kCholPitch)
__device__ __forceinline__ void tile_mma_sub(float (&acc)[4][4], const float* As, const float* Bs, int tx, int ty, int kk) {
#pragma unroll 8
  for (int k = 0; k < kk; ++k) {
    float a[4], b[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) a[r] = As[(r * 16 + ty) * kCholPitch + k];
#pragma unroll
    for (int c = 0; c < 4; ++c) b[c] = Bs[(c * 16 + tx) * kCholPitch + k];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(-a[r], b[c], acc[r][c]);
  }
}

// 64 x 64 tile global -> shared (zero-padded outside the matrix)
__device__ __forceinline__ void load_tile(float* dst, const float* src, int64_t ld, int64_t row0, int64_t col0, int64_t n, bool volatile_l2) {
  for (int e = threadIdx.x; e < kCholNB * kCholNB; e += kCholThreads) {
    const int r = e >> 6, c = e & 63;
    const int64_t gr = row0 + r, gc = col0 + c;
    float v = 0.0f;
    if (gr < n && gc < n) v = volatile_l2 ? __ldcg(src + gr * ld + gc) : src[gr * ld + gc];
    dst[r * kCholPitch + c] = v;
  }
}

__global__ void __launch_bounds__(kCholThreads, 1)
    cholesky_tiles_kernel(const float* A, int64_t lda, int64_t n, float* L, int64_t ldl, float* Linv /* [T][64][64] */, int* flags /* [T][T] */,
                          int T) {
  __shared__ float sA[kCholNB * kCholPitch];
  __shared__ float sB[kCholNB * kCholPitch];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t n_tiles = (int64_t)T * (T + 1) / 2;

  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    // column-major enumeration of the lower triangle: column J holds T - J tiles
    int J = 0;
    int64_t rem = t;
    while (rem >= T - J) {
      rem -= T - J;
      ++J;
    }
    const int I = J + (int)rem;
    const int64_t r0 = (int64_t)I * kCholNB, c0 = (int64_t)J * kCholNB;

    // accumulator: this thread owns elements (r*16+ty, c*16+tx)
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int64_t gr = r0 + r * 16 + ty, gc = c0 + c * 16 + tx;
        // the diagonal tile reads only the lower triangle of A (mirrored), so a non-symmetric input cannot leak in
        float v = 0.0f;
        if (gr < n && gc < n) v = (I == J && gc > gr) ? A[gc * lda + gr] : A[gr * lda + gc];
        acc[r][c] = v;
      }
    // left-looking updates with the already factorised block columns k < J
    for (int k = 0; k < J; ++k) {
      if (tid == 0) {
        while (ld_acquire_gpu(flags + I * T + k) == 0) __nanosleep(32);
        if (I != J)
          while (ld_acquire_gpu(flags + J * T + k) == 0) __nanosleep(32);
      }
      __syncthreads();
      load_tile(sA, L, ldl, r0, (int64_t)k * kCholNB, n, true);
      if (I != J) load_tile(sB, L, ldl, c0, (int64_t)k * kCholNB, n, true);
      __syncthreads();
      tile_mma_sub(acc, sA, I != J ? sB : sA, tx, ty, kCholNB);
      __syncthreads();
    }

    if (I == J) {
      // ---- diagonal tile: T -> shared, factorise as [[L11, 0], [L21, L22]] with 32 x 32 warp factorisations
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) sA[(r * 16 + ty) * kCholPitch + c * 16 + tx] = acc[r][c];
      __syncthreads();
      const int64_t valid = n - r0 < kCholNB ? n - r0 : kCholNB;  // rows / columns of this tile inside the matrix
      if (warp == 0) {
        // pad the part outside the matrix with the identity so that the factorisation stays finite
        float a[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) a[k] = (lane < valid && k < valid) ? sA[lane * kCholPitch + k] : (lane == k ? 1.0f : 0.0f);
        chol32_warp(a, lane);
#pragma unroll
        for (int k = 0; k < 32; ++k) sA[lane * kCholPitch + k] = (k <= lane) ? a[k] : 0.0f;  // L11
        float m[32];
        trinv32_warp(a, m, lane);
#pragma unroll
        for (int i = 0; i < 32; ++i) sB[i * kCholPitch + lane] = m[i];  // inv(L11), stored row-major
      }
      __syncthreads();
      // L21 = S21 * inv(L11)^T : rows 32..63, one thread per (row, column) pair x 4
      for (int e = tid; e < 32 * 32; e += kCholThreads) {
        const int i = 32 + (e >> 5), j = e & 31;
        float s = 0.0f;
        for (int k = 0; k <= j; ++k) s = fmaf(sA[i * kCholPitch + k], sB[j * kCholPitch + k], s);  // inv(L11)[j][k], k <= j
        sB[i * kCholPitch + j] = s;  // stage L21 in the lower-left block of sB (rows 32..63 are free there)
      }
      __syncthreads();
      for (int e = tid; e < 32 * 32; e += kCholThreads) {
        const int i = 32 + (e >> 5), j = e & 31;
        sA[i * kCholPitch + j] = sB[i * kCholPitch + j];
      }
      __syncthreads();
      // S22 -= L21 L21^T (lower part), then factorise it
      for (int e = tid; e < 32 * 32; e += kCholThreads) {
        const int i = 32 + (e >> 5), j = 32 + (e & 31);
        if (j <= i) {
          float s = sA[i * kCholPitch + j];
          for (int k = 0; k < 32; ++k) s = fmaf(-sA[i * kCholPitch + k], sA[j * kCholPitch + k], s);
          sA[i * kCholPitch + j] = s;
        }
      }
      __syncthreads();
      if (warp == 0) {
        float a[32];
#pragma unroll
        for (int k = 0; k < 32; ++k)
          a[k] = (32 + lane < valid && 32 + k < valid) ? sA[(32 + lane) * kCholPitch + 32 + k] : (lane == k ? 1.0f : 0.0f);
        chol32_warp(a, lane);
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          sA[(32 + lane) * kCholPitch + 32 + k] = (k <= lane) ? a[k] : 0.0f;  // L22
          sA[lane * kCholPitch + 32 + k] = 0.0f;                               // upper-right block of the factor
        }
        float m[32];
        trinv32_warp(a, m, lane);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          sB[(32 + i) * kCholPitch + 32 + lane] = m[i];  // inv(L22)
          sB[i * kCholPitch + 32 + lane] = 0.0f;
        }
      }
      __syncthreads();
      // lower-left block of the inverse: -inv(L22) * L21 * inv(L11); first W = L21 * inv(L11) into registers, then the product
      float w4[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * kCholThreads;
        const int i = 32 + (e >> 5), j = e & 31;
        float s = 0.0f;
        for (int k = j; k < 32; ++k) s = fmaf(sA[i * kCholPitch + k], sB[k * kCholPitch + j], s);  // L21[i][k] * inv(L11)[k][j], k >= j
        w4[q] = s;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * kCholThreads;
        sB[(32 + (e >> 5)) * kCholPitch + (e & 31)] = w4[q];  // W staged in the lower-left block
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * kCholThreads;
        const int i = 32 + (e >> 5), j = e & 31;
        float s = 0.0f;
        for (int k = 32; k <= i; ++k) s = fmaf(sB[i * kCholPitch + k], sB[k * kCholPitch + j], s);  // inv(L22)[i][k] * W[k][j], k <= i
        w4[q] = -s;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * kCholThreads;
        sB[(32 + (e >> 5)) * kCholPitch + (e & 31)] = w4[q];
      }
      __syncthreads();
      // publish L[J,J] (zeros above the diagonal) and its inverse
      float* inv_out = Linv + (int64_t)J * kCholNB * kCholNB;
      for (int e = tid; e < kCholNB * kCholNB; e += kCholThreads) {
        const int r = e >> 6, c = e & 63;
        if (r0 + r < n && c0 + c < n) L[(r0 + r) * ldl + c0 + c] = sA[r * kCholPitch + c];
        inv_out[e] = sB[r * kCholPitch + c];
      }
    } else {
      // ---- off-diagonal tile: L[I,J] = T * inv(L[J,J])^T
      if (tid == 0)
        while (ld_acquire_gpu(flags + J * T + J) == 0) __nanosleep(32);
      __syncthreads();
      const float* inv_in = Linv + (int64_t)J * kCholNB * kCholNB;
      for (int e = tid; e < kCholNB * kCholNB; e += kCholThreads) sB[(e >> 6) * kCholPitch + (e & 63)] = __ldcg(inv_in + e);
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) sA[(r * 16 + ty) * kCholPitch + c * 16 + tx] = acc[r][c];
      __syncthreads();
      float out[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) out[r][c] = 0.0f;
      tile_mma_sub(out, sA, sB, tx, ty, kCholNB);  // out = -T * inv^T (inv[c][k] is zero for k > c)
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int64_t gr = r0 + r * 16 + ty, gc = c0 + c * 16 + tx;
          if (gr < n && gc < n) L[gr * ldl + gc] = -out[r][c];
        }
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) st_release_gpu(flags + I * T + J, 1);
  }

  // strictly upper tiles of the output are zero (torch.linalg.cholesky returns the full lower-triangular matrix)
  for (int64_t u = blockIdx.x; u < (int64_t)T * T; u += gridDim.x) {
    const int I = (int)(u / T), J = (int)(u % T);
    if (J <= I) continue;
    for (int e = tid; e < kCholNB * kCholNB; e += kCholThreads) {
      const int64_t gr = (int64_t)I * kCholNB + (e >> 6), gc = (int64_t)J * kCholNB + (e & 63);
      if (gr < n && gc < n) L[gr * ldl + gc] = 0.0f;
    }
  }
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API size_t evok_cholesky_workspace_bytes(int64_t n) {
  if (n <= 0) return 256;
  const int64_t T = (n + kCholNB - 1) / kCholNB;
  return (size_t)T * kCholNB * kCholNB * sizeof(float) + (size_t)T * T * sizeof(int) + 512;
}

extern "C" EVOK_API int evok_cholesky(const float* A, int64_t lda, int64_t n, float* L, int64_t ldl, void* ws, size_t ws_bytes, void* stream) {
  if (!A || !L || !ws) return EVOK_E_NULLPTR;
  if (n <= 0 || lda < n || ldl < n || n > 32768) return EVOK_E_BADSIZE;
  if (ws_bytes < evok_cholesky_workspace_bytes(n)) return EVOK_E_WORKSPACE;
  if (A == L) return EVOK_E_BADSIZE;  // the updates read A's lower triangle while other CTAs already write L
  const int T = (int)((n + kCholNB - 1) / kCholNB);
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  float* linv = reinterpret_cast<float*>(base);
  int* flags = reinterpret_cast<int*>(base + (size_t)T * kCholNB * kCholNB * sizeof(float));
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(flags, 0, (size_t)T * T * sizeof(int), st);
  if (e != cudaSuccess) return (int)e;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = kNumSMs;
  }
  const int64_t n_tiles = (int64_t)T * (T + 1) / 2;
  const int grid = (int)(n_tiles < sms ? n_tiles : sms);  // all CTAs resident: the dataflow schedule needs it
  cholesky_tiles_kernel<<<grid, kCholThreads, 0, st>>>(A, lda, n, L, ldl, linv, flags, T);
  EVOK_CHECK_LAUNCH();
  return 0;
}
