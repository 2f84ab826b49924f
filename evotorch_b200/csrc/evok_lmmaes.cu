// Functional LM-MA-ES (Loshchilov, Glasmachers & Beyer, IEEE TEVC 23(2), 2019) for a batch of independent searches: the ask and
// the tell of every item, with the m direction vectors M [items][m][D] and their Gram matrix G = M M^T [items][m][m] as state.
//
// Every stage works in the coefficient form: a row's step d_i = alpha z_i + sum_j beta_ij M_j lies in
// span{z_i, M_1..M_k}, so the k serial row reductions of the paper's ask become one Gram pass (P = M Z^T), an O(lambda k^2)
// recursion per item, and one pass that writes x.  The tell's recovery of z from the values works the same way on Q = M D^T.
//
// Column passes split D into tiles of kLmTile columns, one CTA per (tile, item).  The tile width is fixed, so the summation
// order of an item depends on D only: item b gives the bits of a one-item call on its own operands, whatever the batch.
// Partial sums go to the workspace and one CTA per item adds them in tile order; nothing uses atomics.
#include <cmath>

#include "evok_common.cuh"

namespace evok {
namespace {

constexpr int kLmThreads = 256;
constexpr int kLmTile = 512;    // columns per CTA of a column pass
constexpr int kLmChunk = 32;    // columns staged in shared memory per step of a Gram pass
constexpr int kLmWChunk = 64;   // columns per step of the write pass
constexpr int kLmBlock = 64;    // rows of either operand of one Gram block: 16 x 16 threads of 4 x 4 outputs
constexpr int kLmMaxM = EVOK_LMMAES_MAX_VECTORS;
constexpr int kLmMaxRows = EVOK_LMMAES_MAX_POPSIZE;
static_assert(kLmMaxM <= kLmBlock, "one Gram block covers every vector");
static_assert(kLmTile % kLmChunk == 0 && kLmTile % kLmWChunk == 0, "chunks tile a column tile");

int64_t lm_tiles(int64_t D) { return (D + kLmTile - 1) / kLmTile; }

// The constants in float, from the double table of the C ABI (c_sigma, mu_eff, c_d[m], c_c[m]).
struct LmConsts {
  float cd[kLmMaxM];    // c_d,j
  float fd[kLmMaxM];    // 1 - c_d,j
  float fc[kLmMaxM];    // 1 - c_c,j
  float sc[kLmMaxM];    // sqrt(mu_eff c_c,j (2 - c_c,j))
  float fs, ss, half_cs;  // 1 - c_sigma, sqrt(mu_eff c_sigma (2 - c_sigma)), c_sigma / 2
  float alpha;          // prod_{j < k} (1 - c_d,j) in double, rounded once
};

LmConsts lm_consts(const double* t, int64_t m, int64_t k) {
  LmConsts c{};
  const double cs = t[0], mu_eff = t[1];
  double alpha = 1.0;
  for (int64_t j = 0; j < m; ++j) {
    const double cd = t[2 + j], cc = t[2 + m + j];
    c.cd[j] = (float)cd;
    c.fd[j] = (float)(1.0 - cd);
    c.fc[j] = (float)(1.0 - cc);
    c.sc[j] = (float)std::sqrt(mu_eff * cc * (2.0 - cc));
    if (j < k) alpha *= 1.0 - cd;
  }
  c.fs = (float)(1.0 - cs);
  c.ss = (float)std::sqrt(mu_eff * cs * (2.0 - cs));
  c.half_cs = (float)(cs / 2.0);
  c.alpha = (float)alpha;
  return c;
}

// acc[q][p] += sum_c A[4 ta + q][c] B[4 tb + p][c] over one staged chunk, in column order.
__device__ __forceinline__ void gram_chunk(const float (*sA)[kLmChunk + 1], const float (*sB)[kLmChunk + 1], int ta, int tb, float acc[4][4]) {
#pragma unroll 4
  for (int c = 0; c < kLmChunk; ++c) {
    float a[4], b[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      a[q] = sA[4 * ta + q][c];
      b[q] = sB[4 * tb + q][c];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) acc[q][p] = fmaf(a[q], b[p], acc[q][p]);
  }
}

// The rows of a tell with a non-zero weight, in row order, and their weights (thread 0 scans: lambda <= 128).
__device__ __forceinline__ int selected_rows(const float* __restrict__ aw, int64_t n_rows, int* rows, float* wts, int* count) {
  if (threadIdx.x == 0) {
    int n = 0;
    for (int64_t i = 0; i < n_rows; ++i) {
      const float w = aw[i];
      if (w != 0.0f) {
        rows[n] = (int)i;
        wts[n] = w;
        ++n;
      }
    }
    *count = n;
  }
  __syncthreads();
  return *count;
}

// Gram pass of the ask (STORED = false) or the tell (STORED = true), one CTA per (column tile, item).
//   ask : P_ji = sum_c M_jc z_ic over the tile for j < k and every row, z rebuilt as the batched sampler draws it (row i of item b
//         on stream word key.stream_lo + b, column group c / 4).
//   tell: Q_jr = sum_c M_jc d_rc for the rows r with a non-zero weight, d = (x - y) / sigma correctly rounded; also
//         S_d = sum_r w_r d_r for the tile's columns, rows in order (complete per tile: the tile holds every row).
// part [items][tiles][k][n_rows]: the tile's sums, by row (ask) or by position in the selected-row list (tell).
template <bool STORED>
__global__ void __launch_bounds__(kLmThreads) lmmaes_project_kernel(const float* __restrict__ M, int64_t m, int64_t k, const float* __restrict__ X,
                                                                    const float* __restrict__ aw, const float* __restrict__ y,
                                                                    const float* __restrict__ sigma, int64_t n_rows, int64_t D,
                                                                    const __grid_constant__ PhiloxKey key, float* __restrict__ part,
                                                                    float* __restrict__ sd) {
  __shared__ float sA[kLmBlock][kLmChunk + 1], sB[kLmBlock][kLmChunk + 1];
  __shared__ int rows[kLmMaxRows];
  __shared__ float wts[kLmMaxRows];
  __shared__ int count;
  const int64_t item = blockIdx.y, tile = blockIdx.x, tiles = gridDim.x;
  const int64_t c0 = tile * kLmTile, c1 = min(D, c0 + kLmTile);
  const int tid = threadIdx.x, ta = tid >> 4, tb = tid & 15;
  M += item * m * D;
  const uint32_t sw = key.stream_lo + (uint32_t)item;
  float s = 0.0f;
  int n_use = (int)n_rows;
  if (STORED) {
    X += item * n_rows * D;
    y += item * D;
    s = sigma[item];
    n_use = selected_rows(aw + item * n_rows, n_rows, rows, wts, &count);
  }
  part += (item * tiles + tile) * k * n_rows;
  if (STORED && n_use == 0)
    for (int64_t col = c0 + tid; col < c1; col += kLmThreads) sd[item * D + col] = 0.0f;
  for (int rb = 0; rb < n_use; rb += kLmBlock) {
    const int nr = min(kLmBlock, n_use - rb);
    float acc[4][4] = {};
    for (int64_t cc = c0; cc < c1; cc += kLmChunk) {
      for (int e = tid; e < k * kLmChunk; e += kLmThreads) {
        const int j = e / kLmChunk, c = e % kLmChunk;
        sA[j][c] = cc + c < c1 ? M[j * D + cc + c] : 0.0f;
      }
      if (STORED) {
        for (int e = tid; e < nr * kLmChunk; e += kLmThreads) {
          const int r = e / kLmChunk, c = e % kLmChunk;
          const int64_t col = cc + c;
          sB[r][c] = col < c1 ? __fdiv_rn(X[rows[rb + r] * D + col] - y[col], s) : 0.0f;
        }
      } else {
        for (int e = tid; e < nr * (kLmChunk / 4); e += kLmThreads) {
          const int r = e / (kLmChunk / 4), g = e % (kLmChunk / 4);
          const int64_t col = cc + 4 * g;
          float z[4];
          normals4(key, sw, (uint64_t)(rb + r), (uint32_t)(col >> 2), z);
#pragma unroll
          for (int q = 0; q < 4; ++q) sB[r][4 * g + q] = col + q < c1 ? z[q] : 0.0f;
        }
      }
      __syncthreads();
      if (STORED && tid < kLmChunk && cc + tid < c1) {
        float v = 0.0f;
        for (int r = 0; r < nr; ++r) v = fmaf(wts[rb + r], sB[r][tid], v);
        float* out = sd + item * D + cc + tid;
        *out = rb == 0 ? v : *out + v;
      }
      gram_chunk(sA, sB, ta, tb, acc);
      __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int j = 4 * ta + q, r = 4 * tb + p;
        if (j < k && r < nr) part[j * n_rows + rb + r] = acc[q][p];
      }
  }
}

// Sum of the tiles' partials [tiles][k][ld] of entries (j, r), j < k, r < n, in tile order, into s_out[j * ld + r] by all threads.
__device__ __forceinline__ void reduce_tiles(const float* __restrict__ part, int64_t tiles, int64_t k, int64_t ld, int64_t n, float* s_out) {
  for (int64_t e = threadIdx.x; e < k * n; e += blockDim.x) {
    const int64_t at = (e / n) * ld + e % n;
    float v = 0.0f;
#pragma unroll 8
    for (int64_t t = 0; t < tiles; ++t) v += part[t * k * ld + at];
    s_out[at] = v;
  }
}

// The ask's coefficients, one CTA per item, thread i for row i: P_ji summed over the tiles in order (all threads), then for
// j = 0 .. k-1
//   s_i = alpha P_ji + sum_{l<j} beta_il G_lj;  alpha, beta_i *= (1 - c_d,j);  beta_ij += c_d,j s_i.
// beta [items][k][n_rows].  Shared memory: G (k x k), beta and P (k x n_rows each).
__global__ void __launch_bounds__(kLmMaxRows) lmmaes_coef_kernel(const float* __restrict__ part, int64_t tiles, const float* __restrict__ G, int64_t m,
                                                                 int64_t k, int64_t n_rows, const __grid_constant__ LmConsts cst,
                                                                 float* __restrict__ beta) {
  extern __shared__ float lm_smem[];
  float* sG = lm_smem;                     // [k][k]
  float* sb = lm_smem + k * k;             // [k][n_rows]
  float* sP = lm_smem + k * k + k * n_rows;  // [k][n_rows]
  const int64_t item = blockIdx.x;
  G += item * m * m;
  for (int64_t e = threadIdx.x; e < k * k; e += blockDim.x) sG[e] = G[(e / k) * m + e % k];
  reduce_tiles(part + item * tiles * k * n_rows, tiles, k, n_rows, n_rows, sP);
  __syncthreads();
  const int64_t i = threadIdx.x;
  if (i >= n_rows) return;
  float alpha = 1.0f;
  for (int64_t j = 0; j < k; ++j) {
    float s = alpha * sP[j * n_rows + i];
    for (int64_t l = 0; l < j; ++l) s = fmaf(sb[l * n_rows + i], sG[l * k + j], s);
    const float f = cst.fd[j];
    alpha *= f;
    for (int64_t l = 0; l < j; ++l) sb[l * n_rows + i] *= f;
    sb[j * n_rows + i] = cst.cd[j] * s;
  }
  beta += item * k * n_rows;
  for (int64_t l = 0; l < k; ++l) beta[l * n_rows + i] = sb[l * n_rows + i];
}

// x_ic = y_c + sigma (alpha z_ic + sum_j beta_ij M_jc), one CTA per (column tile, item): each 64-column chunk of M is staged once
// and shared by every row; thread (tr, tc) writes rows 4 tr .. 4 tr + 3 of a 64-row block, columns 4 tc .. 4 tc + 3 of the chunk.
// With k = 0, x = fmaf(sigma, z, y): the bits of the batched sampler with mean y and stdev sigma.
__global__ void __launch_bounds__(kLmThreads) lmmaes_write_kernel(float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ sigma,
                                                                  const float* __restrict__ M, int64_t m, int64_t k, const float* __restrict__ beta,
                                                                  int64_t n_rows, int64_t D, const __grid_constant__ PhiloxKey key, float alpha) {
  __shared__ float sbeta[kLmBlock][kLmMaxM + 1];
  __shared__ __align__(16) float sM[kLmMaxM][kLmWChunk + 4];
  const int64_t item = blockIdx.y, tile = blockIdx.x;
  const int64_t c0 = tile * kLmTile, c1 = min(D, c0 + kLmTile);
  const int tid = threadIdx.x, tr = tid >> 4, tc = tid & 15;
  const uint32_t sw = key.stream_lo + (uint32_t)item;
  X += item * n_rows * D;
  y += item * D;
  M += item * m * D;
  beta += item * k * n_rows;
  const float s = sigma[item];
  for (int64_t rb = 0; rb < n_rows; rb += kLmBlock) {
    const int nr = (int)min((int64_t)kLmBlock, n_rows - rb);
    __syncthreads();
    for (int e = tid; e < nr * k; e += kLmThreads) {
      const int l = e / nr, r = e % nr;
      sbeta[r][l] = beta[l * n_rows + rb + r];
    }
    for (int64_t cc = c0; cc < c1; cc += kLmWChunk) {
      __syncthreads();
      for (int e = tid; e < k * kLmWChunk; e += kLmThreads) {
        const int l = e / kLmWChunk, c = e % kLmWChunk;
        sM[l][c] = cc + c < c1 ? M[l * D + cc + c] : 0.0f;
      }
      __syncthreads();
      const int64_t col = cc + 4 * tc;
      if (col >= c1) continue;
      float acc[4][4] = {};
      for (int l = 0; l < k; ++l) {
        const float4 mv = *reinterpret_cast<const float4*>(&sM[l][4 * tc]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float b = sbeta[4 * tr + q][l];
          acc[q][0] = fmaf(b, mv.x, acc[q][0]);
          acc[q][1] = fmaf(b, mv.y, acc[q][1]);
          acc[q][2] = fmaf(b, mv.z, acc[q][2]);
          acc[q][3] = fmaf(b, mv.w, acc[q][3]);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t row = rb + 4 * tr + q;
        if (row >= n_rows) break;
        float z[4];
        normals4(key, sw, (uint64_t)row, (uint32_t)(col >> 2), z);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          if (col + p < c1) {
            const float d = k > 0 ? fmaf(alpha, z[p], acc[q][p]) : z[p];
            X[row * D + col + p] = fmaf(s, d, y[col + p]);
          }
        }
      }
    }
  }
}

// The tell's recovery, one CTA per item, thread r for the r-th row with a non-zero weight: Q_jr summed over the tiles in order
// (all threads), then for j = k-1 .. 0
//   u = a Q_jr + sum_{l>j} gamma_rl G_lj;  a, gamma_r /= (1 - c_d,j);  gamma_rj -= kappa_j u / (1 - c_d,j),
// kappa_j = c_d,j / ((1 - c_d,j) + c_d,j G_jj), and then c_j = sum_r w_r gamma_rj (rows in order).  coef [items][1 + m]:
// (a, c_0 .. c_{k-1}), so that S_z = a S_d + sum_j c_j M_j.
__global__ void __launch_bounds__(kLmMaxRows) lmmaes_recover_kernel(const float* __restrict__ part, int64_t tiles, const float* __restrict__ aw,
                                                                    const float* __restrict__ G, int64_t m, int64_t k, int64_t n_rows,
                                                                    const __grid_constant__ LmConsts cst, float* __restrict__ coef) {
  extern __shared__ float lm_smem[];
  float* sG = lm_smem;                       // [k][k]
  float* sg = lm_smem + k * k;               // [k][n_rows]: gamma
  float* sQ = lm_smem + k * k + k * n_rows;  // [k][n_rows]
  __shared__ int rows[kLmMaxRows];
  __shared__ float wts[kLmMaxRows];
  __shared__ int count;
  const int64_t item = blockIdx.x;
  G += item * m * m;
  for (int64_t e = threadIdx.x; e < k * k; e += blockDim.x) sG[e] = G[(e / k) * m + e % k];
  const int n_sel = selected_rows(aw + item * n_rows, n_rows, rows, wts, &count);
  reduce_tiles(part + item * tiles * k * n_rows, tiles, k, n_rows, n_sel, sQ);
  __syncthreads();
  const int r = threadIdx.x;
  float a = 1.0f;
  if (r < n_sel) {
    for (int64_t j = k - 1; j >= 0; --j) {
      float u = a * sQ[j * n_rows + r];
      for (int64_t l = j + 1; l < k; ++l) u = fmaf(sg[l * n_rows + r], sG[l * k + j], u);
      const float f = cst.fd[j], kappa = cst.cd[j] / (f + cst.cd[j] * sG[j * k + j]);
      a = a / f;
      for (int64_t l = j + 1; l < k; ++l) sg[l * n_rows + r] = sg[l * n_rows + r] / f;
      sg[j * n_rows + r] = -(kappa * u / f);
    }
  }
  __syncthreads();
  coef += item * (1 + m);
  if (r < k) {
    float c = 0.0f;
    for (int i = 0; i < n_sel; ++i) c = fmaf(wts[i], sg[r * n_rows + i], c);
    coef[1 + r] = c;
  }
  if (r == 0) {
    float a0 = 1.0f;  // the a of every row (a row-independent product), also with no selected row
    for (int64_t j = k - 1; j >= 0; --j) a0 = a0 / cst.fd[j];
    coef[0] = a0;
  }
}

// The update, one CTA per (column tile, item): per column S_z = a S_d + sum_{j<k} c_j M_j, then for every j < m
// M'_j = (1 - c_c,j) M_j + sqrt(mu_eff c_c,j (2 - c_c,j)) S_z, p_sigma' = (1 - c_sigma) p_sigma + sqrt(mu_eff c_sigma (2 - c_sigma)) S_z
// and y' = y + sigma S_d.  The tile's sums of |p_sigma'|^2 (columns in order) and of M' M'^T (a Gram pass over the M' it writes)
// go to pp [items][tiles] and pg [items][tiles][m][m].
__global__ void __launch_bounds__(kLmThreads) lmmaes_update_kernel(const float* __restrict__ M, int64_t m, int64_t k, const float* __restrict__ sd,
                                                                   const float* __restrict__ coef, const float* __restrict__ y,
                                                                   const float* __restrict__ sigma, const float* __restrict__ p_sigma, int64_t D,
                                                                   const __grid_constant__ LmConsts cst, float* __restrict__ M_out,
                                                                   float* __restrict__ y_out, float* __restrict__ p_out, float* __restrict__ pg,
                                                                   float* __restrict__ pp) {
  __shared__ float sA[kLmBlock][kLmChunk + 1];
  __shared__ float sz[kLmChunk];
  const int64_t item = blockIdx.y, tile = blockIdx.x, tiles = gridDim.x;
  const int64_t c0 = tile * kLmTile, c1 = min(D, c0 + kLmTile);
  const int tid = threadIdx.x, ta = tid >> 4, tb = tid & 15;
  M += item * m * D;
  M_out += item * m * D;
  sd += item * D;
  coef += item * (1 + m);
  y += item * D;
  y_out += item * D;
  p_sigma += item * D;
  p_out += item * D;
  const float s = sigma[item], a = coef[0];
  float acc[4][4] = {};
  float psq = 0.0f;
  for (int64_t cc = c0; cc < c1; cc += kLmChunk) {
    for (int e = tid; e < m * kLmChunk; e += kLmThreads) {
      const int j = e / kLmChunk, c = e % kLmChunk;
      sA[j][c] = cc + c < c1 ? M[j * D + cc + c] : 0.0f;
    }
    __syncthreads();
    if (tid < kLmChunk) {
      const int64_t col = cc + tid;
      float v = 0.0f;
      if (col < c1) {
        const float dsum = sd[col];
        v = a * dsum;
        for (int j = 0; j < k; ++j) v = fmaf(coef[1 + j], sA[j][tid], v);
        const float p = fmaf(cst.fs, p_sigma[col], cst.ss * v);
        p_out[col] = p;
        psq = fmaf(p, p, psq);
        y_out[col] = fmaf(s, dsum, y[col]);
      }
      sz[tid] = v;
    }
    __syncthreads();
    for (int e = tid; e < m * kLmChunk; e += kLmThreads) {
      const int j = e / kLmChunk, c = e % kLmChunk;
      const float v = cc + c < c1 ? fmaf(cst.fc[j], sA[j][c], cst.sc[j] * sz[c]) : 0.0f;
      sA[j][c] = v;
      if (cc + c < c1) M_out[j * D + cc + c] = v;
    }
    __syncthreads();
    gram_chunk(sA, sA, ta, tb, acc);
    __syncthreads();
  }
  pg += (item * tiles + tile) * m * m;
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int j = 4 * ta + q, l = 4 * tb + p;
      if (j < m && l < m) pg[j * m + l] = acc[q][p];
    }
  if (tid < kWarp) {
    psq = warp_sum(psq);
    if (tid == 0) pp[item * tiles + tile] = psq;
  }
}

// G' = the tiles' Gram sums added in order, sigma' = sigma exp((c_sigma / 2)(|p_sigma'|^2 / D - 1)); one CTA per item.
__global__ void __launch_bounds__(kLmThreads) lmmaes_finish_kernel(const float* __restrict__ pg, const float* __restrict__ pp, int64_t tiles, int64_t m,
                                                                   int64_t D, const float* __restrict__ sigma, const __grid_constant__ LmConsts cst,
                                                                   float* __restrict__ G_out, float* __restrict__ sigma_out) {
  const int64_t item = blockIdx.x;
  pg += item * tiles * m * m;
  for (int64_t e = threadIdx.x; e < m * m; e += blockDim.x) {
    float g = 0.0f;
#pragma unroll 8
    for (int64_t t = 0; t < tiles; ++t) g += pg[t * m * m + e];
    G_out[item * m * m + e] = g;
  }
  if (threadIdx.x == 0) {
    float p = 0.0f;
    for (int64_t t = 0; t < tiles; ++t) p += pp[item * tiles + t];
    sigma_out[item] = sigma[item] * expf(cst.half_cs * (p / (float)D - 1.0f));
  }
}

// Workspace of one item chunk (<= kMaxGridY items), in floats: the Gram partials (tiles x m x max(n_rows, m)), S_d (D), beta or the
// recovery coefficients (m x n_rows + 1 + m) and the |p_sigma|^2 partials (tiles).
int64_t lm_item_floats(int64_t n_rows, int64_t D, int64_t m) {
  const int64_t tiles = lm_tiles(D);
  return tiles * m * (n_rows > m ? n_rows : m) + D + m * n_rows + 1 + m + tiles;
}
int64_t lm_chunk_items(int64_t n_items) { return n_items < kMaxGridY ? n_items : kMaxGridY; }

int lm_check(int64_t n_items, int64_t n_rows, int64_t D, int64_t m, int64_t k) {
  if (n_items < 0 || n_rows < 2 || n_rows > kLmMaxRows || D <= 0 || m < 1 || m > kLmMaxM || k < 0 || k > m) return EVOK_E_BADSIZE;
  return 0;
}

struct LmWs {
  float *part, *sd, *coef, *pp;
};
LmWs lm_split(void* ws, int64_t nb, int64_t n_rows, int64_t D, int64_t m) {
  const int64_t tiles = lm_tiles(D);
  float* p = static_cast<float*>(ws);
  LmWs w;
  w.part = p;
  p += nb * tiles * m * (n_rows > m ? n_rows : m);
  w.sd = p;
  p += nb * D;
  w.coef = p;
  p += nb * (m * n_rows + 1 + m);
  w.pp = p;
  return w;
}

// G, beta (or gamma) and P (or Q) of the one-CTA-per-item kernels: up to 80 KB, above the default limit of 48 KB
size_t coef_smem(int64_t k, int64_t n_rows) { return (size_t)(k * k + 2 * k * n_rows) * sizeof(float); }
int allow_coef_smem(const void* fn) {
  const size_t most = coef_smem(kLmMaxM, kLmMaxRows);
  return (int)cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)most);
}

}  // namespace
}  // namespace evok

using namespace evok;

extern "C" EVOK_API size_t evok_lmmaes_workspace_bytes(int64_t n_items, int64_t n_rows, int64_t D, int64_t m) {
  if (lm_check(n_items, n_rows, D, m, 0) || n_items == 0) return 256;
  return (size_t)lm_chunk_items(n_items) * (size_t)lm_item_floats(n_rows, D, m) * sizeof(float);
}

extern "C" EVOK_API int evok_lmmaes_ask_batched(float* X, const float* y, const float* sigma, const float* M, const float* G, int64_t n_items,
                                                int64_t n_rows, int64_t D, int64_t m, int64_t k, const double* consts_host, uint64_t seed,
                                                uint64_t stream_id0, void* ws, size_t ws_bytes, void* stream) {
  if (!X || !y || !sigma || !M || !G || !consts_host || !ws) return EVOK_E_NULLPTR;
  if (const int rc = lm_check(n_items, n_rows, D, m, k)) return rc;
  if (n_items == 0) return 0;
  if (ws_bytes < evok_lmmaes_workspace_bytes(n_items, n_rows, D, m)) return EVOK_E_WORKSPACE;
  const cudaStream_t st = (cudaStream_t)stream;
  const LmConsts cst = lm_consts(consts_host, m, k);
  const PhiloxKey key = make_philox_key(seed, stream_id0);
  const int64_t tiles = lm_tiles(D);
  if (const int rc = allow_coef_smem((const void*)lmmaes_coef_kernel)) return rc;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    PhiloxKey kc = key;
    kc.stream_lo += (uint32_t)b0;
    const LmWs w = lm_split(ws, nb, n_rows, D, m);
    const dim3 grid((unsigned)tiles, (unsigned)nb);
    const float* Mc = M + b0 * m * D;
    if (k > 0) {
      lmmaes_project_kernel<false><<<grid, kLmThreads, 0, st>>>(Mc, m, k, nullptr, nullptr, nullptr, nullptr, n_rows, D, kc, w.part, nullptr);
      lmmaes_coef_kernel<<<(unsigned)nb, kLmMaxRows, coef_smem(k, n_rows), st>>>(w.part, tiles, G + b0 * m * m, m, k, n_rows, cst, w.coef);
      EVOK_CHECK_LAUNCH_N(2);
    }
    lmmaes_write_kernel<<<grid, kLmThreads, 0, st>>>(X + b0 * n_rows * D, y + b0 * D, sigma + b0, Mc, m, k, w.coef, n_rows, D, kc, cst.alpha);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_lmmaes_tell_batched(const float* X, const float* aw, const float* y, const float* sigma, const float* p_sigma,
                                                 const float* M, const float* G, int64_t n_items, int64_t n_rows, int64_t D, int64_t m, int64_t k,
                                                 const double* consts_host, float* y_out, float* sigma_out, float* p_sigma_out, float* M_out,
                                                 float* G_out, void* ws, size_t ws_bytes, void* stream) {
  if (!X || !aw || !y || !sigma || !p_sigma || !M || !G || !consts_host || !y_out || !sigma_out || !p_sigma_out || !M_out || !G_out || !ws)
    return EVOK_E_NULLPTR;
  if (const int rc = lm_check(n_items, n_rows, D, m, k)) return rc;
  if (n_items == 0) return 0;
  if (ws_bytes < evok_lmmaes_workspace_bytes(n_items, n_rows, D, m)) return EVOK_E_WORKSPACE;
  const cudaStream_t st = (cudaStream_t)stream;
  const LmConsts cst = lm_consts(consts_host, m, k);
  const int64_t tiles = lm_tiles(D);
  if (const int rc = allow_coef_smem((const void*)lmmaes_recover_kernel)) return rc;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    const LmWs w = lm_split(ws, nb, n_rows, D, m);
    const dim3 grid((unsigned)tiles, (unsigned)nb);
    const float* Mc = M + b0 * m * D;
    const float* awc = aw + b0 * n_rows;
    lmmaes_project_kernel<true><<<grid, kLmThreads, 0, st>>>(Mc, m, k, X + b0 * n_rows * D, awc, y + b0 * D, sigma + b0, n_rows, D, PhiloxKey{},
                                                             w.part, w.sd);
    lmmaes_recover_kernel<<<(unsigned)nb, kLmMaxRows, coef_smem(k, n_rows), st>>>(w.part, tiles, awc, G + b0 * m * m, m, k, n_rows, cst, w.coef);
    lmmaes_update_kernel<<<grid, kLmThreads, 0, st>>>(Mc, m, k, w.sd, w.coef, y + b0 * D, sigma + b0, p_sigma + b0 * D, D, cst, M_out + b0 * m * D,
                                                      y_out + b0 * D, p_sigma_out + b0 * D, w.part, w.pp);
    lmmaes_finish_kernel<<<(unsigned)nb, kLmThreads, 0, st>>>(w.part, w.pp, tiles, m, D, sigma + b0, cst, G_out + b0 * m * m, sigma_out + b0);
    EVOK_CHECK_LAUNCH_N(4);
    return 0;
  });
}
