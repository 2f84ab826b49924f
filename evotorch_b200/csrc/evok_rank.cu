// K3: fitness -> utilities.  A hand-written stable LSD radix sort of (orderable fp32 key, index) pairs
// (4 passes x 8 bits; per pass: per-tile digit histogram -> per-digit exclusive scan -> stable scatter using
// warp match/ballot ranking), followed by one scatter of what each sorted position writes (emit_at).  N is the population size
// (<= a few million): the whole working set lives in L2, the kernels are latency-, not bandwidth-bound.
#include "evok_common.cuh"

namespace evok {

constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;
constexpr int kSortThreads = 256;               // 8 warps; must equal kRadix (one thread per digit)
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kItemsPerThread = 8;
constexpr int kTile = kSortThreads * kItemsPerThread;  // 2048 keys per CTA per pass

// fp32 -> uint32 whose unsigned order is the float order; -0 -> +0 first; NaN (any sign) -> largest.
__device__ __forceinline__ uint32_t orderable(float v) {
  if (v != v) return 0xFFFFFFFFu;
  v += 0.0f;  // -0 -> +0
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// the sort key of fitness f: descending + stable == ascending on the complemented key
__device__ __forceinline__ uint32_t sort_key(float f, int descending) {
  const uint32_t k = orderable(f);
  return descending ? ~k : k;
}

__global__ void __launch_bounds__(256) make_keys_kernel(const float* __restrict__ f, int64_t N, int descending,
                                                        uint32_t* __restrict__ keys, uint32_t* __restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) {
    keys[i] = sort_key(f[i], descending);
    idx[i] = (uint32_t)i;
  }
}

// counts[d * n_tiles + tile]
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const uint32_t* __restrict__ keys, int64_t N, int shift,
                                                                  uint32_t* __restrict__ counts, int n_tiles) {
  __shared__ uint32_t h[kRadix];
  for (int i = threadIdx.x; i < kRadix; i += kSortThreads) h[i] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kTile;
#pragma unroll
  for (int it = 0; it < kItemsPerThread; ++it) {
    const int64_t i = base + it * kSortThreads + threadIdx.x;
    if (i < N) atomicAdd(&h[(keys[i] >> shift) & (kRadix - 1)], 1u);
  }
  __syncthreads();
  for (int d = threadIdx.x; d < kRadix; d += kSortThreads) counts[(int64_t)d * n_tiles + blockIdx.x] = h[d];
}

// Variant for moderate tile counts (n_tiles <= kSelfScanMaxTiles, i.e. up to 512 k keys -- every sharded ranking and most
// populations): the histogram kernel writes its counts TILE-major (counts_t[tile][digit]) and, on the first pass, also builds
// the orderable keys / indices from the fitnesses; the scatter kernel then derives its own offsets (thread d sums digit d over
// the tiles: n_tiles coalesced, independent loads), so a pass is 2 launches instead of 3 and make_keys disappears.
constexpr int kSelfScanMaxTiles = 256;

template <bool FIRST>
__global__ void __launch_bounds__(kSortThreads)
    radix_hist_t_kernel(const float* __restrict__ f, int descending, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx, int64_t N, int shift,
                        uint32_t* __restrict__ counts_t) {
  __shared__ uint32_t h[kRadix];
  for (int i = threadIdx.x; i < kRadix; i += kSortThreads) h[i] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kTile;
#pragma unroll
  for (int it = 0; it < kItemsPerThread; ++it) {
    const int64_t i = base + it * kSortThreads + threadIdx.x;
    if (i < N) {
      uint32_t k;
      if (FIRST) {
        k = sort_key(f[i], descending);
        keys[i] = k;
        idx[i] = (uint32_t)i;
      } else {
        k = keys[i];
      }
      atomicAdd(&h[(k >> shift) & (kRadix - 1)], 1u);
    }
  }
  __syncthreads();
  for (int d = threadIdx.x; d < kRadix; d += kSortThreads) counts_t[(int64_t)blockIdx.x * kRadix + d] = h[d];
}

// per digit d (one CTA each): exclusive scan in place of counts[d][0..n_tiles) and the digit total.
__global__ void __launch_bounds__(256) digit_scan_kernel(uint32_t* __restrict__ counts, int n_tiles, uint32_t* __restrict__ totals) {
  __shared__ uint32_t warp_tot[8];
  __shared__ uint32_t carry_s, chunk_s;
  uint32_t* row = counts + (int64_t)blockIdx.x * n_tiles;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < n_tiles; base += 256) {
    const int i = base + threadIdx.x;
    const uint32_t v = i < n_tiles ? row[i] : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      const uint32_t t = lane < 8 ? warp_tot[lane] : 0u;
      uint32_t ti = t;
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, ti, o);
        if (lane >= o) ti += u;
      }
      if (lane < 8) warp_tot[lane] = ti - t;  // exclusive warp offsets
      if (lane == 7) chunk_s = ti;
    }
    __syncthreads();
    const uint32_t carry = carry_s;
    if (i < n_tiles) row[i] = carry + warp_tot[wid] + incl - v;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + chunk_s;
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = carry_s;
}

// stable scatter of one tile.  Item order inside a tile: warp w owns the contiguous range
// [w*256, (w+1)*256); iteration `it` covers 32 consecutive items, lane = position.
// SELF_SCAN: `offsets` holds tile-major raw counts (radix_hist_t_kernel); thread d sums digit d over the tiles itself
template <bool SELF_SCAN>
__global__ void __launch_bounds__(kSortThreads)
    radix_scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ idx_in, uint32_t* __restrict__ keys_out,
                         uint32_t* __restrict__ idx_out, int64_t N, int shift, const uint32_t* __restrict__ offsets, int n_tiles,
                         const uint32_t* __restrict__ totals) {
  __shared__ uint32_t wcount[kSortWarps][kRadix];  // per-warp digit counts, then per-warp exclusive bases
  __shared__ uint32_t digit_base[kRadix];          // exclusive scan of the digit totals
  __shared__ uint32_t wtot[kSortWarps];
  __shared__ uint32_t tile_prefix[kRadix];         // SELF_SCAN: keys of digit d in the tiles before this one
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < kSortWarps * kRadix; i += kSortThreads) (&wcount[0][0])[i] = 0;
  {  // kSortThreads == kRadix: thread d owns digit d
    uint32_t t;
    if (SELF_SCAN) {
      uint32_t before = 0, all = 0;
      for (int tile = 0; tile < n_tiles; ++tile) {
        const uint32_t c = offsets[(int64_t)tile * kRadix + threadIdx.x];
        all += c;
        before += tile < (int)blockIdx.x ? c : 0u;
      }
      tile_prefix[threadIdx.x] = before;
      t = all;
    } else {
      t = totals[threadIdx.x];
    }
    uint32_t incl = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) wtot[wid] = incl;
    __syncthreads();
    uint32_t wb = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) wb += w < wid ? wtot[w] : 0u;
    digit_base[threadIdx.x] = wb + incl - t;
  }
  __syncthreads();

  const int64_t wbase = (int64_t)blockIdx.x * kTile + (int64_t)wid * (32 * kItemsPerThread);
  uint32_t key[kItemsPerThread], val[kItemsPerThread], rnk[kItemsPerThread];
#pragma unroll
  for (int it = 0; it < kItemsPerThread; ++it) {
    const int64_t i = wbase + it * 32 + lane;
    const bool ok = i < N;
    key[it] = ok ? keys_in[i] : 0xFFFFFFFFu;
    val[it] = ok ? idx_in[i] : 0u;
    const uint32_t d = (key[it] >> shift) & (kRadix - 1);
    // lanes holding the same digit (invalid lanes form their own group via the extra bit)
    const uint32_t peers = __match_any_sync(0xffffffffu, ok ? d : (kRadix + 1u));
    const uint32_t below = __popc(peers & ((1u << lane) - 1u));
    uint32_t base = 0;
    if (ok && below == 0) {  // group leader: lowest lane of the group
      base = wcount[wid][d];
      wcount[wid][d] = base + __popc(peers);
    }
    base = __shfl_sync(0xffffffffu, base, __ffs(peers) - 1);
    rnk[it] = base + below;
    __syncwarp();
  }
  __syncthreads();
  // per digit: exclusive scan over the warps (in warp order) + global tile offset
  for (int d = threadIdx.x; d < kRadix; d += kSortThreads) {
    uint32_t run = digit_base[d] + (SELF_SCAN ? tile_prefix[d] : offsets[(int64_t)d * n_tiles + blockIdx.x]);
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) {
      const uint32_t c = wcount[w][d];
      wcount[w][d] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kItemsPerThread; ++it) {
    const int64_t i = wbase + it * 32 + lane;
    if (i < N) {
      const uint32_t d = (key[it] >> shift) & (kRadix - 1);
      const uint32_t pos = wcount[wid][d] + rnk[it];
      keys_out[pos] = key[it];
      idx_out[pos] = val[it];
    }
  }
}

// ---- what a sorted position writes -----------------------------------------------------------------
// NES utility of sorted position p (0 = worst) of N before normalisation: max(0, top - ln(N-p)), Nf = N, top = ln(N/2+1)
__device__ __forceinline__ float nes_term(int64_t p, float Nf, float top) { return fmaxf(0.0f, top - logf(Nf - (float)p)); }

// this thread's share of the NES table sum: positions first, first + stride, ... (fp32 terms, double accumulation in that order)
__device__ __forceinline__ double nes_partial_sum(int64_t N, int64_t first, int stride) {
  const float Nf = (float)N, top = logf(Nf / 2.0f + 1.0f);
  double acc = 0.0;
  for (int64_t p = first; p < N; p += stride) acc += (double)nes_term(p, Nf, top);
  return acc;
}

// utility of sorted position p of N; *nes_sum (the table sum) is read for NES only
__device__ __forceinline__ float utility_at(int64_t p, int64_t N, int method, const float* nes_sum) {
  if (method == EVOK_RANK_CENTERED) return __fdiv_rn((float)p, (float)(N - 1)) - 0.5f;
  if (method == EVOK_RANK_LINEAR) return __fdiv_rn((float)p, (float)(N - 1));
  const float Nf = (float)N;
  return __fdiv_rn(nes_term(p, Nf, logf(Nf / 2.0f + 1.0f)), *nes_sum) - __fdiv_rn(1.0f, Nf);
}

enum { kUtilities = 0, kArgsort = 1, kEliteMask = 2, kTable = 3 };

// The outputs of a ranking, [items][N] like its keys; the table is shared by the items.
struct Emit {
  int mode;            // kUtilities / kArgsort / kEliteMask / kTable
  int method;          // kUtilities: the ranking method
  int64_t num_elites;  // kEliteMask
  float* out;          // utility / elite flag / table entry, in the solution's slot (unused by kArgsort)
  int64_t* perm;       // nullable: the solution at each sorted position
  const float* table;  // kTable: the value of each sorted position (CMA-ES: weight of a solution = weights[its rank], cmaes.py:445-451)
  __host__ __device__ Emit item(int64_t off) const {
    Emit e = *this;
    if (out) e.out += off;
    if (perm) e.perm += off;
    return e;
  }
};

// the four kinds of output (out / perm [items][N]; perm may be null for utilities)
static Emit utilities(int method, float* w, int64_t* perm) { return Emit{kUtilities, method, 0, w, perm, nullptr}; }
static Emit permutation(int64_t* perm) { return Emit{kArgsort, 0, 0, nullptr, perm, nullptr}; }
static Emit elite_flags(int64_t num_elites, float* mask) { return Emit{kEliteMask, 0, num_elites, mask, nullptr, nullptr}; }
static Emit table_entries(const float* table, float* out) { return Emit{kTable, 0, 0, out, nullptr, table}; }

// solution i sits at sorted position p (0 = first in the stable order): write what `mode` asks for
__device__ __forceinline__ void emit_at(int64_t p, uint32_t i, int64_t N, const Emit& e, const float* nes_sum) {
  if (e.perm) e.perm[p] = (int64_t)i;
  if (e.mode == kUtilities) e.out[i] = utility_at(p, N, e.method, nes_sum);
  else if (e.mode == kEliteMask) e.out[i] = p < e.num_elites ? 1.0f : 0.0f;
  else if (e.mode == kTable) e.out[i] = e.table[p];
}

// the NES table sum of N positions; single CTA
__global__ void __launch_bounds__(1024) nes_table_sum_kernel(int64_t N, float* __restrict__ out_sum) {
  __shared__ double sm[33];
  const double tot = block_sum<double>(nes_partial_sum(N, threadIdx.x, 1024), sm);
  if (threadIdx.x == 0) *out_sum = (float)tot;
}

// after the radix sort: emit_at for every position p of the sorted index array
__global__ void __launch_bounds__(256) scatter_sorted_kernel(const uint32_t* __restrict__ idx, int64_t N, const Emit e,
                                                             const float* __restrict__ nes_sum) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < N) emit_at(p, idx[p], N, e, nes_sum);
}

// normalized / raw: no sort.  stats[0] = mean, stats[1] = unbiased std of g = +-f (double accumulation).
__global__ void __launch_bounds__(1024) mean_std_kernel(const float* __restrict__ f, int64_t N, float sign, float* __restrict__ stats) {
  __shared__ double sm[33];
  f += (int64_t)blockIdx.x * N;  // batched: one CTA per item, stats[2 * item ..]
  stats += 2 * blockIdx.x;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += 1024) s += (double)(sign * f[i]);
  const double mean = block_sum<double>(s, sm) / (double)N;
  double q = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += 1024) {
    const double d = (double)(sign * f[i]) - mean;
    q += d * d;
  }
  const double var = block_sum<double>(q, sm) / (double)(N - 1);
  if (threadIdx.x == 0) {
    stats[0] = (float)mean;
    stats[1] = (float)sqrt(var);
  }
}
__global__ void __launch_bounds__(256) affine_kernel(const float* __restrict__ f, int64_t N, float sign, const float* __restrict__ stats,
                                                     int normalized, float* __restrict__ w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  f += (int64_t)blockIdx.y * N;  // batched: blockIdx.y = item
  w += (int64_t)blockIdx.y * N;
  stats += 2 * blockIdx.y;
  const float g = sign * f[i];
  w[i] = normalized ? __fdiv_rn(g - stats[0], stats[1]) : g;
}

// in-place weight adjustments
__global__ void __launch_bounds__(1024) weights_adjust_kernel(float* __restrict__ w, int64_t N, int mode) {
  __shared__ double sm[33];
  w += (int64_t)blockIdx.x * N;  // batched: one CTA per item
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += 1024) s += mode == 1 ? (double)w[i] : (double)fabsf(w[i]);
  const double tot = block_sum<double>(s, sm);
  if (mode == 1) {
    const float mean = (float)(tot / (double)N);
    for (int64_t i = threadIdx.x; i < N; i += 1024) w[i] -= mean;
  } else {
    const float d = (float)tot;
    for (int64_t i = threadIdx.x; i < N; i += 1024) w[i] = __fdiv_rn(w[i], d);
  }
}

// ---- small populations: rank by counting, ONE launch -------------------------------------------------
// For N <= kSmallRankMax the 14-launch radix pipeline is pure launch latency (even inside a CUDA graph), while the stable rank of element i is simply  #{j : key_j < key_i} + #{j < i : key_j == key_i}.  All N^2 comparisons
// (67 M at N = 8192) spread over the whole GPU take a few microseconds: 4 lanes share one element (interleaved quarters of
// the key tile staged in shared memory: conflict-free, broadcast reads; 8 or 16 lanes for larger N, so that the grid always
// covers the GPU), 256 / lanes elements per CTA.  The utility (or the elite flag,
// or the permutation entry) is written by the same kernel, so make_keys + 12 sort launches + the scatter collapse into one.
constexpr int kSmallRankMax = 8192;
constexpr int kSmallThreads = 256;
constexpr int kSmallTile = 2048;

// the stable position of key i among the first N keys of f (PARTS lanes per element, reduced over them)
template <int PARTS>
__device__ __forceinline__ uint32_t counting_rank(const float* __restrict__ f, int N, int i, int part, int descending, uint32_t* tile) {
  const uint32_t ki = i < N ? sort_key(f[i], descending) : 0u;
  uint32_t cnt = 0;
  for (int base = 0; base < N; base += kSmallTile) {
    __syncthreads();
    for (int t = threadIdx.x; t < kSmallTile; t += kSmallThreads) {
      const int j = base + t;
      tile[t] = j < N ? sort_key(f[j], descending) : 0xFFFFFFFFu;  // padding: never below a real key, never "equal with a lower index"
    }
    __syncthreads();
    const int lim = min(kSmallTile, N - base);
#pragma unroll 4
    for (int t = part; t < lim; t += PARTS) {
      const uint32_t k = tile[t];
      cnt += (uint32_t)(k < ki) + (uint32_t)((k == ki) & (base + t < i));
    }
  }
#pragma unroll
  for (int o = 1; o < PARTS; o <<= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  return cnt;
}

template <int PARTS>
__global__ void __launch_bounds__(kSmallThreads) rank_small_kernel(const float* __restrict__ f, int N, int descending, Emit e) {
  __shared__ uint32_t tile[kSmallTile];
  __shared__ double red[33];
  constexpr int kElems = kSmallThreads / PARTS;
  // batched searches: blockIdx.y = batch item, every item ranks its own N fitnesses
  f += (int64_t)blockIdx.y * N;
  e = e.item((int64_t)blockIdx.y * N);
  const int part = threadIdx.x % PARTS;
  const int i = blockIdx.x * kElems + threadIdx.x / PARTS;
  const uint32_t cnt = counting_rank<PARTS>(f, N, i, part, descending, tile);

  float nes_sum = 0.0f;
  if (e.mode == kUtilities && e.method == EVOK_RANK_NES)  // the table sum of nes_table_sum_kernel, once per CTA
    nes_sum = (float)block_sum<double>(nes_partial_sum(N, threadIdx.x, kSmallThreads), red);
  if (i < N && part == 0) emit_at(cnt, (uint32_t)i, N, e, &nes_sum);  // cnt: position in sorted order
}

// one launch for n_items rows of N <= kSmallRankMax keys
static int rank_small(const float* f, int64_t N, int64_t n_items, int descending, const Emit& e, cudaStream_t st) {
  // lanes per element grow with N: the work per thread stays <= 512 comparisons and the grid >= N / 64 CTAs
  if (N <= 1024) {
    rank_small_kernel<4><<<dim3((unsigned)((N + 63) / 64), (unsigned)n_items), kSmallThreads, 0, st>>>(f, (int)N, descending, e);
  } else if (N <= 4096) {
    rank_small_kernel<8><<<dim3((unsigned)((N + 31) / 32), (unsigned)n_items), kSmallThreads, 0, st>>>(f, (int)N, descending, e);
  } else {
    rank_small_kernel<16><<<dim3((unsigned)((N + 15) / 16), (unsigned)n_items), kSmallThreads, 0, st>>>(f, (int)N, descending, e);
  }
  EVOK_CHECK_LAUNCH();
  return 0;
}

// Tiered rank-table lookup (padded populations): item b (grid y) ranks its first n = counts[tier[b]] of N keys and writes
// tables[tier[b]][its position] to them, 0 to its pad rows n..N-1.  The table row is read only at positions < n.
template <int PARTS>
__global__ void __launch_bounds__(kSmallThreads)
    rank_table_tiered_kernel(const float* __restrict__ f, int N, int descending, const float* __restrict__ tables, const int* __restrict__ tier,
                             const int* __restrict__ counts, float* __restrict__ out) {
  __shared__ uint32_t tile[kSmallTile];
  constexpr int kElems = kSmallThreads / PARTS;
  f += (int64_t)blockIdx.y * N;
  out += (int64_t)blockIdx.y * N;
  const int k = tier[blockIdx.y];
  const int n = min(counts[k], N);
  const int part = threadIdx.x % PARTS;
  const int i = blockIdx.x * kElems + threadIdx.x / PARTS;
  const uint32_t cnt = counting_rank<PARTS>(f, n, i, part, descending, tile);
  if (i < N && part == 0) out[i] = i < n ? tables[(int64_t)k * N + cnt] : 0.0f;
}

// ---- host side ------------------------------------------------------------------------------------
struct SortPlan {
  int64_t N;
  int n_tiles;
  size_t off_keys0, off_keys1, off_idx0, off_idx1, off_counts, off_totals, off_scalar, total;
};

static SortPlan make_plan(int64_t N) {
  SortPlan p;
  p.N = N;
  p.n_tiles = (int)((N + kTile - 1) / kTile);
  if (p.n_tiles < 1) p.n_tiles = 1;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  size_t o = 0;
  p.off_keys0 = o; o += al((size_t)N * 4);
  p.off_keys1 = o; o += al((size_t)N * 4);
  p.off_idx0 = o; o += al((size_t)N * 4);
  p.off_idx1 = o; o += al((size_t)N * 4);
  p.off_counts = o; o += al((size_t)kRadix * p.n_tiles * 4);
  p.off_totals = o; o += al((size_t)kRadix * 4);
  p.off_scalar = o; o += 64 + 2 * kNumSMs * 8 + 192;  // scalar slot + per-CTA partial sums of the sharded ranking's push kernel
  p.total = o;
  return p;
}

// sorts; returns the device pointer (inside ws) of the sorted index array (and of the sorted keys).
// Up to kSelfScanMaxTiles tiles (512 k keys) the 13-launch pipeline (make_keys + 4 x (hist, scan, scatter)) shrinks to 8
// (4 x (hist [+ keys], self-scanning scatter)).
static int sort_pairs(const float* f, int64_t N, int descending, void* ws, const SortPlan& p, cudaStream_t st, uint32_t** sorted_idx,
                      uint32_t** sorted_keys = nullptr) {
  char* base = (char*)ws;
  uint32_t* keys[2] = {(uint32_t*)(base + p.off_keys0), (uint32_t*)(base + p.off_keys1)};
  uint32_t* idx[2] = {(uint32_t*)(base + p.off_idx0), (uint32_t*)(base + p.off_idx1)};
  uint32_t* counts = (uint32_t*)(base + p.off_counts);
  uint32_t* totals = (uint32_t*)(base + p.off_totals);
  const bool self_scan = p.n_tiles <= kSelfScanMaxTiles;
  if (!self_scan) {
    make_keys_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(f, N, descending, keys[0], idx[0]);
    EVOK_CHECK_LAUNCH();
  }
  int cur = 0;
  for (int pass = 0; pass < 32 / kRadixBits; ++pass) {
    const int shift = pass * kRadixBits;
    if (self_scan) {
      if (pass == 0) radix_hist_t_kernel<true><<<p.n_tiles, kSortThreads, 0, st>>>(f, descending, keys[0], idx[0], N, shift, counts);
      else radix_hist_t_kernel<false><<<p.n_tiles, kSortThreads, 0, st>>>(nullptr, 0, keys[cur], nullptr, N, shift, counts);
      radix_scatter_kernel<true><<<p.n_tiles, kSortThreads, 0, st>>>(keys[cur], idx[cur], keys[cur ^ 1], idx[cur ^ 1], N, shift, counts, p.n_tiles, totals);
      EVOK_CHECK_LAUNCH_N(2);
    } else {
      radix_hist_kernel<<<p.n_tiles, kSortThreads, 0, st>>>(keys[cur], N, shift, counts, p.n_tiles);
      digit_scan_kernel<<<kRadix, 256, 0, st>>>(counts, p.n_tiles, totals);
      radix_scatter_kernel<false><<<p.n_tiles, kSortThreads, 0, st>>>(keys[cur], idx[cur], keys[cur ^ 1], idx[cur ^ 1], N, shift, counts, p.n_tiles, totals);
      EVOK_CHECK_LAUNCH_N(3);
    }
    cur ^= 1;
  }
  *sorted_idx = idx[cur];
  if (sorted_keys) *sorted_keys = keys[cur];
  return 0;
}

// n_items rankings of N keys each ([items][N], like the outputs of e): for N <= kSmallRankMax the counting rank, one launch per item
// chunk; above, per item on the one workspace, the radix sort, the NES table sum if the utilities need it, and the scatter.  The
// single-search entry points check the workspace for every N; the batched ones need it, and check it, for the sort only.
static int rank_rows(const float* keys, int64_t N, int64_t n_items, int descending, const Emit& e, void* ws, size_t ws_bytes,
                     cudaStream_t st) {
  if (N <= kSmallRankMax)
    return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
      return rank_small(keys + b0 * N, N, nb, descending, e.item(b0 * N), st);
    });
  const SortPlan p = make_plan(N);
  if (ws_bytes < p.total) return EVOK_E_WORKSPACE;
  float* nes_sum = (float*)((char*)ws + p.off_scalar);
  const bool nes = e.mode == kUtilities && e.method == EVOK_RANK_NES;
  for (int64_t b = 0; b < n_items; ++b) {
    uint32_t* sidx = nullptr;
    const int rc = sort_pairs(keys + b * N, N, descending, ws, p, st, &sidx);
    if (rc) return rc;
    if (nes) nes_table_sum_kernel<<<1, 1024, 0, st>>>(N, nes_sum);
    scatter_sorted_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(sidx, N, e.item(b * N), nes_sum);
    EVOK_CHECK_LAUNCH_N(nes ? 2 : 1);
  }
  return 0;
}

// normalized / raw (no sort) for n_items rows of N: stats holds (mean, std) of +-f for each item of a chunk
static int affine_rows(int method, const float* f, int64_t N, int64_t n_items, int higher_is_better, float* w, float* stats, cudaStream_t st) {
  const float sign = higher_is_better ? 1.0f : -1.0f;
  const int normalized = method == EVOK_RANK_NORMALIZED;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    const float* fc = f + b0 * N;
    if (normalized) mean_std_kernel<<<(unsigned)nb, 1024, 0, st>>>(fc, N, sign, stats);
    affine_kernel<<<dim3((unsigned)((N + 255) / 256), (unsigned)nb), 256, 0, st>>>(fc, N, sign, stats, normalized, w + b0 * N);
    EVOK_CHECK_LAUNCH_N(normalized ? 2 : 1);
    return 0;
  });
}

// ---- sharded ranking over peer memory ----------------------------------------------------------------
// Every GPU sorts only ITS OWN n_local fitnesses, pushes the sorted keys into every peer's key table (NVLink) and then
// ranks its own rows against the world:  global position of a local element = its position in the local order
//   + sum over the other shards s of  #{keys of s that precede it}   (upper bound for s < rank: equal keys of a lower
//   shard have lower global indices and come first in the stable order; lower bound for s > rank).
// Per GPU that is a sort of N / world keys plus n_local x (world - 1) binary searches over an L2-resident table instead
// of a replicated sort of all N keys; the resulting positions (hence utilities) are bit-identical to the global sort.
struct ShardTable {
  long long off[EVOK_MAX_PEERS + 1];  // row offsets of the shards; off[world] = N
};

// One CTA per destination GPU (like evok_peer_push): CTA j copies ALL sorted keys of this rank into peer p's table with 16-byte
// stores, adds up the local fitnesses (every CTA computes the same deterministic sum: fixed strided order + fixed tree), stores it,
// fences ONCE and raises the flag on that peer.  No cross-CTA coordination, 8 system fences instead of one per CTA of a wide grid.
constexpr int kRankPushThreads = 1024;

__global__ void __launch_bounds__(kRankPushThreads)
    rank_push_kernel(const uint32_t* __restrict__ sorted_keys, const float* __restrict__ f, int64_t n_local, int64_t my_off,
                     const __grid_constant__ PeerSink keys_sink, const __grid_constant__ PeerSink fsum_sink, const unsigned long long* epoch) {
  __shared__ double red[33];
  const int p = (keys_sink.rank + 1 + blockIdx.x) % keys_sink.world;  // rotated start: spread the links
  uint32_t* dst = static_cast<uint32_t*>(keys_sink.data[p]) + my_off;
  if (((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(sorted_keys)) & 15u) == 0) {
    const int64_t nq = n_local >> 2;
    for (int64_t q = threadIdx.x; q < nq; q += kRankPushThreads) reinterpret_cast<uint4*>(dst)[q] = reinterpret_cast<const uint4*>(sorted_keys)[q];
    for (int64_t i = (nq << 2) + threadIdx.x; i < n_local; i += kRankPushThreads) dst[i] = sorted_keys[i];
  } else {
    for (int64_t i = threadIdx.x; i < n_local; i += kRankPushThreads) dst[i] = sorted_keys[i];
  }
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < n_local; i += kRankPushThreads) acc += (double)f[i];
  const double tot = block_sum<double>(acc, red);
  if (threadIdx.x == 0) {
    static_cast<double*>(fsum_sink.data[p])[keys_sink.rank] = tot;
    __threadfence_system();
    st_release_sys(keys_sink.flags[p] + keys_sink.rank, *epoch + 1ull);
  }
}

__device__ __forceinline__ unsigned long long rank_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__global__ void __launch_bounds__(256)
    rank_merge_kernel(const uint32_t* keys_all, const uint32_t* __restrict__ sorted_idx, const __grid_constant__ ShardTable tab, int world, int rank,
                      int method, const float* __restrict__ nes_sum, const double* fsum, const unsigned long long* flags,
                      unsigned long long* epoch, unsigned int* done, unsigned int* err, unsigned long long timeout_ns,
                      float* __restrict__ w_local, float* __restrict__ mean_out) {
  // wait until every rank's sorted keys have landed in the local table
  const unsigned long long want = *epoch + 1ull;
  if ((int)threadIdx.x < world) {
    const unsigned long long t0 = rank_timer_ns();
    while (ld_acquire_sys(flags + threadIdx.x) < want) {
      if (rank_timer_ns() - t0 > timeout_ns) {
        atomicExch(err, 1u);
        break;
      }
      __nanosleep(64);
    }
  }
  __syncthreads();
  const int64_t N = tab.off[world];
  const int64_t my_off = tab.off[rank], n_local = tab.off[rank + 1] - my_off;
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n_local) {
    const uint32_t key = __ldcg(keys_all + my_off + p);
    // (world - 1) independent binary searches, advanced in lock step so that their L2 loads overlap
    int64_t lo[EVOK_MAX_PEERS], hi[EVOK_MAX_PEERS];
    int steps = 0;
#pragma unroll
    for (int s = 0; s < EVOK_MAX_PEERS; ++s) {
      lo[s] = 0;
      hi[s] = (s < world && s != rank) ? tab.off[s + 1] - tab.off[s] : 0;
      int need = 0;
      for (int64_t n = hi[s]; n > 0; n >>= 1) ++need;
      steps = max(steps, need);
    }
    for (int it = 0; it < steps; ++it) {
#pragma unroll
      for (int s = 0; s < EVOK_MAX_PEERS; ++s) {
        if (s < world && lo[s] < hi[s]) {
          const int64_t mid = (lo[s] + hi[s]) >> 1;
          const uint32_t k = __ldcg(keys_all + tab.off[s] + mid);
          const bool before = s < rank ? (k <= key) : (k < key);  // does element `mid` of shard s precede ours?
          if (before) lo[s] = mid + 1;
          else hi[s] = mid;
        }
      }
    }
    int64_t pos = p;
#pragma unroll
    for (int s = 0; s < EVOK_MAX_PEERS; ++s)
      if (s < world && s != rank) pos += lo[s];
    w_local[sorted_idx[p]] = utility_at(pos, N, method, nes_sum);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && mean_out) {
    double tot = 0.0;
    for (int r = 0; r < world; ++r) tot += __ldcg(fsum + r);  // rank order: identical on every GPU
    *mean_out = (float)(tot / (double)N);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {  // every CTA has read `epoch` before arriving here
      *done = 0;
      *epoch = want;
    }
  }
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API size_t evok_rank_workspace_bytes(int64_t N) {
  if (N <= 0) return 256;
  return make_plan(N).total;
}

extern "C" EVOK_API int evok_rank(int method, const float* f, int64_t N, int higher_is_better, float* w, int64_t* perm, void* ws,
                         size_t ws_bytes, void* stream) {
  if (!f || !w || !ws) return EVOK_E_NULLPTR;
  if (method < EVOK_RANK_CENTERED || method > EVOK_RANK_RAW) return EVOK_E_BADENUM;
  if (N < 0 || N >= (int64_t)1 << 32) return EVOK_E_BADSIZE;
  if (N == 0) return 0;
  const SortPlan p = make_plan(N);
  if (ws_bytes < p.total) return EVOK_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  if (method == EVOK_RANK_NORMALIZED || method == EVOK_RANK_RAW) {
    const int rc = affine_rows(method, f, N, 1, higher_is_better, w, (float*)((char*)ws + p.off_scalar), st);
    if (rc || !perm) return rc;
    return rank_rows(f, N, 1, !higher_is_better, permutation(perm), ws, ws_bytes, st);
  }
  return rank_rows(f, N, 1, !higher_is_better, utilities(method, w, perm), ws, ws_bytes, st);
}

extern "C" EVOK_API int evok_argsort(const float* keys, int64_t N, int descending, int64_t* perm, void* ws, size_t ws_bytes, void* stream) {
  if (!keys || !perm || !ws) return EVOK_E_NULLPTR;
  if (N < 0 || N >= (int64_t)1 << 32) return EVOK_E_BADSIZE;
  if (N == 0) return 0;
  if (ws_bytes < make_plan(N).total) return EVOK_E_WORKSPACE;
  return rank_rows(keys, N, 1, descending, permutation(perm), ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_weights_adjust(float* w, int64_t N, int mode, void* stream) { return evok_weights_adjust_batched(w, N, 1, mode, stream); }

extern "C" EVOK_API int evok_elite_mask(const float* w, int64_t N, int64_t num_elites, float* mask, void* ws, size_t ws_bytes, void* stream) {
  if (!w || !mask || !ws) return EVOK_E_NULLPTR;
  if (N < 0 || N >= (int64_t)1 << 32 || num_elites < 0 || num_elites > N) return EVOK_E_BADSIZE;
  if (N == 0) return 0;
  if (ws_bytes < make_plan(N).total) return EVOK_E_WORKSPACE;
  return rank_rows(w, N, 1, /*descending=*/1, elite_flags(num_elites, mask), ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_rank_sharded(int method, const float* f_local, int64_t N, int higher_is_better, int world, int rank,
                                          const int64_t* row_offsets_host, void* const* peer_keys_host, void* const* peer_fsum_host,
                                          void* const* peer_flags_host, uint64_t* epoch_dev, uint32_t* done_dev, uint32_t* err_dev,
                                          uint64_t timeout_ns, float* w_local, float* mean_out, void* ws, size_t ws_bytes, void* stream) {
  if (!row_offsets_host || !peer_keys_host || !peer_fsum_host || !peer_flags_host || !epoch_dev || !done_dev || !err_dev || !ws)
    return EVOK_E_NULLPTR;
  if (method != EVOK_RANK_CENTERED && method != EVOK_RANK_LINEAR && method != EVOK_RANK_NES) return EVOK_E_BADENUM;
  if (world < 1 || world > EVOK_MAX_PEERS || rank < 0 || rank >= world) return EVOK_E_BADSIZE;
  if (N < 1 || N >= (int64_t)1 << 32 || row_offsets_host[0] != 0 || row_offsets_host[world] != N) return EVOK_E_BADSIZE;
  ShardTable tab{};
  for (int r = 0; r <= world; ++r) {
    if (r > 0 && row_offsets_host[r] < row_offsets_host[r - 1]) return EVOK_E_BADSIZE;
    tab.off[r] = row_offsets_host[r];
  }
  const int64_t my_off = tab.off[rank], n_local = tab.off[rank + 1] - my_off;
  // an empty shard has no fitnesses or utilities to point at (an empty CUDA tensor's data pointer is NULL)
  if (n_local > 0 && (!f_local || !w_local)) return EVOK_E_NULLPTR;
  const SortPlan p = make_plan(n_local > 0 ? n_local : 1);
  if (ws_bytes < p.total) return EVOK_E_WORKSPACE;
  PeerSink keys_sink{}, fsum_sink{};
  keys_sink.world = fsum_sink.world = world;
  keys_sink.rank = fsum_sink.rank = rank;
  for (int q = 0; q < world; ++q) {
    if (!peer_keys_host[q] || !peer_fsum_host[q] || !peer_flags_host[q]) return EVOK_E_NULLPTR;
    keys_sink.data[q] = peer_keys_host[q];
    fsum_sink.data[q] = peer_fsum_host[q];
    keys_sink.flags[q] = fsum_sink.flags[q] = static_cast<unsigned long long*>(peer_flags_host[q]);
  }
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned long long* epoch = reinterpret_cast<const unsigned long long*>(epoch_dev);
  uint32_t *sidx = nullptr, *skeys = nullptr;
  if (n_local > 0) {
    int rc = sort_pairs(f_local, n_local, !higher_is_better, ws, p, st, &sidx, &skeys);
    if (rc) return rc;
  }
  rank_push_kernel<<<world, kRankPushThreads, 0, st>>>(skeys, f_local, n_local, my_off, keys_sink, fsum_sink, epoch);
  EVOK_CHECK_LAUNCH();
  float* scalar = (float*)((char*)ws + p.off_scalar);
  if (method == EVOK_RANK_NES) {
    nes_table_sum_kernel<<<1, 1024, 0, st>>>(N, scalar);
    EVOK_CHECK_LAUNCH();
  }
  const unsigned merge_grid = (unsigned)((n_local + 255) / 256 > 0 ? (n_local + 255) / 256 : 1);
  rank_merge_kernel<<<merge_grid, 256, 0, st>>>(static_cast<const uint32_t*>(peer_keys_host[rank]), sidx, tab, world, rank, method, scalar,
                                               static_cast<const double*>(peer_fsum_host[rank]),
                                               static_cast<const unsigned long long*>(peer_flags_host[rank]),
                                               reinterpret_cast<unsigned long long*>(epoch_dev), done_dev + 2, err_dev, timeout_ns, w_local, mean_out);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_rank_table(const float* keys, int64_t N, int descending, const float* table, float* out, void* ws, size_t ws_bytes,
                                        void* stream) {
  if (!keys || !table || !out || !ws) return EVOK_E_NULLPTR;
  if (N < 0 || N >= (int64_t)1 << 32) return EVOK_E_BADSIZE;
  if (N == 0) return 0;
  if (ws_bytes < make_plan(N).total) return EVOK_E_WORKSPACE;
  return rank_rows(keys, N, 1, descending, table_entries(table, out), ws, ws_bytes, (cudaStream_t)stream);
}

// ---- batched searches (functional API with leading batch dimensions): n_items independent rankings of N fitnesses each, f and w
// contiguous [n_items][N], through the same path as the single searches (see rank_rows).
extern "C" EVOK_API int evok_rank_batched(int method, const float* f, int64_t N, int64_t n_items, int higher_is_better, float* w, void* ws,
                                          size_t ws_bytes, void* stream) {
  if (!f || !w || !ws) return EVOK_E_NULLPTR;
  if (method < EVOK_RANK_CENTERED || method > EVOK_RANK_RAW) return EVOK_E_BADENUM;
  if (N < 0 || N >= (int64_t)1 << 32 || n_items < 0) return EVOK_E_BADSIZE;
  if (N == 0 || n_items == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (method == EVOK_RANK_NORMALIZED || method == EVOK_RANK_RAW) {
    const int64_t chunk = n_items < kMaxGridY ? n_items : kMaxGridY;
    if (ws_bytes < (size_t)chunk * 8 + 256) return EVOK_E_WORKSPACE;
    return affine_rows(method, f, N, n_items, higher_is_better, w, (float*)ws, st);
  }
  return rank_rows(f, N, n_items, !higher_is_better, utilities(method, w, nullptr), ws, ws_bytes, st);
}

// n_items rank-table lookups (keys, out: [items][N]) with one shared table
extern "C" EVOK_API int evok_rank_table_batched(const float* keys, int64_t N, int64_t n_items, int descending, const float* table, float* out, void* ws,
                                                size_t ws_bytes, void* stream) {
  if (!keys || !table || !out || !ws) return EVOK_E_NULLPTR;
  if (N < 0 || N >= (int64_t)1 << 32 || n_items < 0) return EVOK_E_BADSIZE;
  if (N == 0 || n_items == 0) return 0;
  return rank_rows(keys, N, n_items, descending, table_entries(table, out), ws, ws_bytes, (cudaStream_t)stream);
}

// n_items tiered rank-table lookups (padded populations of N rows): the counting rank of rank_small, one launch per item chunk
extern "C" EVOK_API int evok_rank_table_batched_tiered(const float* keys, int64_t N, int64_t n_items, int descending, const float* tables,
                                                       const int32_t* tier, const int32_t* counts, float* out, void* stream) {
  if (!keys || !tables || !tier || !counts || !out) return EVOK_E_NULLPTR;
  if (N < 0 || N > kSmallRankMax || n_items < 0) return EVOK_E_BADSIZE;
  if (N == 0 || n_items == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    const float* f = keys + b0 * N;
    const int* t = tier + b0;
    float* o = out + b0 * N;
    if (N <= 1024) {
      rank_table_tiered_kernel<4><<<dim3((unsigned)((N + 63) / 64), (unsigned)nb), kSmallThreads, 0, st>>>(f, (int)N, descending, tables, t, counts, o);
    } else if (N <= 4096) {
      rank_table_tiered_kernel<8><<<dim3((unsigned)((N + 31) / 32), (unsigned)nb), kSmallThreads, 0, st>>>(f, (int)N, descending, tables, t, counts, o);
    } else {
      rank_table_tiered_kernel<16><<<dim3((unsigned)((N + 15) / 16), (unsigned)nb), kSmallThreads, 0, st>>>(f, (int)N, descending, tables, t, counts, o);
    }
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_elite_mask_batched(const float* w, int64_t N, int64_t n_items, int64_t num_elites, float* mask, void* ws,
                                                size_t ws_bytes, void* stream) {
  if (!w || !mask || !ws) return EVOK_E_NULLPTR;
  if (N < 0 || N >= (int64_t)1 << 32 || n_items < 0 || num_elites < 0 || num_elites > N) return EVOK_E_BADSIZE;
  if (N == 0 || n_items == 0) return 0;
  return rank_rows(w, N, n_items, /*descending=*/1, elite_flags(num_elites, mask), ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" EVOK_API int evok_weights_adjust_batched(float* w, int64_t N, int64_t n_items, int mode, void* stream) {
  if (!w) return EVOK_E_NULLPTR;
  if (mode != 1 && mode != 2) return EVOK_E_BADENUM;
  if (N < 0 || n_items < 0) return EVOK_E_BADSIZE;
  if (N == 0 || n_items == 0) return 0;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    weights_adjust_kernel<<<(unsigned)nb, 1024, 0, (cudaStream_t)stream>>>(w + b0 * N, N, mode);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}
