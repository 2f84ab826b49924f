// K6 / K7: fp32-accurate GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier), for the dense contractions of
// CMA-ES (cmaes.py:427 `Y = Z A^T`, :548 rank-mu update `Y^T diag(w) Y`) and XNES.
//
//   C[M x N] = A[M x K] * B[N x K]^T            (A, B row-major with K contiguous: "K-major"; fp32 in, fp32 out)
//
// Accuracy: every fp32 operand x is split as x = hi + lo with hi = x rounded down to TF32 (13 low mantissa bits cleared)
// and lo = x - hi (exact); the kernel accumulates hi*hi + hi*lo + lo*hi in fp32 with wgmma.mma_async...tf32 ("3xTF32"),
// which restores ~2^-21 relative accuracy per product -- plain single-pass TF32 (2^-10) would break the 1e-5 parity bar of
// the searchers' state.
//
// Structure (one CTA per 128 x 128 output tile, optional split-K over blockIdx.z; 384 threads = 3 warpgroups):
//   warp 0      TMA producer, 3-stage mbarrier ring.  CONVERT = true (operands 16-byte aligned, the normal case): TWO raw fp32
//               tile loads per K-block (A, B; 128-byte swizzle) -- the tensor core ignores the 13 low mantissa bits of a tf32
//               operand, so the raw tile IS the hi operand, and two converter warps derive the lo tiles (x - trunc(x), same
//               swizzled positions, element-wise) in shared memory while earlier MMAs run: the operands are read from HBM exactly
//               once and no split copies exist.  CONVERT = false (unaligned operands): 4 loads of tiles pre-split by a pre-pass
//   warp 1      idle (keeps the consumers on a warpgroup boundary)
//   warps 2-3   converters (CONVERT only, see warp 0)
//   warps 4-11  two consumer warpgroups, tile rows 0-63 and 64-127: each issues the 12 wgmma.m64n128k8 of a K-block (its half of
//               the A tile against the whole B tile) and accumulates in registers in chunks of 4 K-blocks; each finished chunk
//               is folded into a second register accumulator with round-to-nearest fp32 adds.  The final tile is written through
//               a shared-memory transpose; optional second output C2 = alpha * acc + bias[col]
#include <cuda.h>

#include <cstdlib>

#include "evok_common.cuh"

namespace evok {

constexpr int kGemmBM = 128;
constexpr int kGemmBN = 128;
constexpr int kGemmBK = 32;  // floats = 128 bytes = one swizzle span
constexpr int kGemmStages = 3;
constexpr int kGemmThreads = 384;  // producer warpgroup (TMA warp, idle warp, 2 converter warps) + 2 consumer warpgroups
constexpr int kWgmmaK = 8;         // tf32: 32 bytes of K per MMA
constexpr int kAcc = kGemmBN / 2;  // fp32 accumulator registers per consumer thread (m64 x n128 over 128 threads)
constexpr uint32_t kTileABytes = kGemmBM * kGemmBK * 4;  // 16 KB
constexpr uint32_t kTileBBytes = kGemmBN * kGemmBK * 4;  // 16 KB
constexpr uint32_t kHalfABytes = kTileABytes / 2;        // the 64 rows of one consumer warpgroup
constexpr uint32_t kStageBytes = 2 * kTileABytes + 2 * kTileBBytes;  // 64 KB
constexpr int kEpiPitch = kGemmBN + 8;  // floats per row of the epilogue tile (the fragment's 8-byte stores of 8 rows hit 32 distinct banks)
constexpr size_t kGemmSmemBytes = (size_t)kGemmStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert((size_t)kGemmBM * kEpiPitch * 4 <= (size_t)kGemmStages * kStageBytes, "epilogue tile reuses the stages");

// ---- PTX wrappers ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(uint64_t* b, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void bar_wait(uint64_t* b, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(s32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(s32(dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(s32(bar))
               : "memory");
}
// rank-3 map [items][rows][K] (batched GEMM): box depth 1, so a tile never reads the next item's rows
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(s32(dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(z), "r"(s32(bar))
               : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of the accumulator registers across a wgmma fence / wait
__device__ __forceinline__ void fence_acc(float (&d)[kAcc]) {
#pragma unroll
  for (int j = 0; j < kAcc; ++j) asm volatile("" : "+f"(d[j])::"memory");
}
// D (+)= A[smem desc, 64 x 8] * B[smem desc, 128 x 8]^T, tf32 inputs, fp32 accumulate in registers.  Fragment of thread t of the
// warpgroup: d[4 j + 2 h + c] = D[16 (t / 32) + (t % 32) / 4 + 8 h][8 j + 2 (t % 4) + c]
__device__ __forceinline__ void wgmma_tf32(float (&d)[kAcc], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, "
      "%28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, "
      "%54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
        "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
        "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
        "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// shared-memory matrix descriptor (wgmma) of a K-major tile stored as rows of 128 bytes with the 128-byte swizzle:
// start >> 4 | LBO (unused for swizzled K-major, canonical 1) << 16 | SBO (8 rows x 128 B between core-matrix groups) >> 4 << 32 |
// layout SWIZZLE_128B (1) << 62.  Tiles are 1024-byte aligned, so the base offset field stays 0.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// The 3xTF32 products of one K-block (32 floats = 4 wgmma K-steps) into the chunk accumulator d; small terms first, the dominant
// hi*hi product last.  `first`: the chunk starts here (the first MMA overwrites d).
__device__ __forceinline__ void mma_kblock(float (&d)[kAcc], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, bool first) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kGemmBK / kWgmmaK; ++k) {
    const uint64_t adv = (uint64_t)((k * kWgmmaK * 4) >> 4);  // advance the start address by 32 bytes per MMA along K
    wgmma_tf32(d, a_hi + adv, b_lo + adv, (first && k == 0) ? 0u : 1u);
    wgmma_tf32(d, a_lo + adv, b_hi + adv, 1u);
    wgmma_tf32(d, a_hi + adv, b_hi + adv, 1u);
  }
  wgmma_commit();
}

// lo = x - trunc_tf32(x) of a whole tile, by 64 threads: thread ct handles the float4 at byte ct * 16 + j * 1024 (addresses in the shared
// window); 16 loads are issued before the first use
template <uint32_t BYTES>
__device__ __forceinline__ void split_lo_tile(uint32_t src, uint32_t dst) {
#pragma unroll
  for (uint32_t b = 0; b < BYTES / 1024u; b += 16) {
    float4 v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j)
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[j].x), "=f"(v[j].y), "=f"(v[j].z), "=f"(v[j].w) : "r"(src + (b + j) * 1024u));
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float lx = v[j].x - __uint_as_float(__float_as_uint(v[j].x) & 0xFFFFE000u);
      const float ly = v[j].y - __uint_as_float(__float_as_uint(v[j].y) & 0xFFFFE000u);
      const float lz = v[j].z - __uint_as_float(__float_as_uint(v[j].z) & 0xFFFFE000u);
      const float lw = v[j].w - __uint_as_float(__float_as_uint(v[j].w) & 0xFFFFE000u);
      asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + (b + j) * 1024u), "f"(lx), "f"(ly), "f"(lz), "f"(lw) : "memory");
    }
  }
}

struct GemmParams {
  int M, N, K;
  int kblocks_per_split;
  float* C;
  int64_t ldc;
  int64_t split_stride;  // elements between the partial outputs of consecutive K splits
  float* C2;             // optional second output alpha * acc + bias[col]
  int64_t ldc2;
  const float* alpha_dev;
  const float* bias;
  // optional in-place style update  C = k[0] * acc + k[1] * E[i][j] + k[2] * u[i] * u[j]   (k: 3 device floats; CMA-ES covariance
  // update cmaes.py:519-553 with acc = Y^T diag(w) Y, E = old C, u = p_c).  Applied by the epilogue, or by the split-K reduction.
  const float* affine_k;
  const float* affine_E;
  int64_t lde;
  const float* affine_u;
  // GATHER (batched policy forward, stacked weight rows): row m of the A operand lives at
  //   gather_a + (m / ga_rows_per_batch) * ga_batch_stride + (m % ga_rows_per_batch) * ga_row_stride     (any 4-byte alignment)
  // and the epilogue applies  C = act(acc + row_bias[(m / rows_per_batch) * rb_batch_stride + m % rows_per_batch])
  const float* gather_a;
  int64_t ga_rows_per_batch, ga_batch_stride, ga_row_stride;
  const float* row_bias;
  int64_t rb_batch_stride;
  int row_act;
  int b_lo_tma;  // CONVERT: the lo tile of B comes from a pre-split copy (map_b_lo) instead of being derived by the converter warps
  int c_unit_fastest;  // persistent gather kernel: C[(batch * N + col) * rows_per_batch + row_in_batch]
  // BATCHED: grid z = item (never a K split); split_stride is then C's item stride.  map_item_a / _b: 1 = the operand's map has one
  // plane per item, 0 = one plane shared by all items.  The epilogue operands sit at these item strides (0 = shared).
  int map_item_a, map_item_b;
  int64_t c2_item_stride, alpha_item_stride, bias_item_stride, k_item_stride, e_item_stride, u_item_stride;
};

// The tensor core does not round its fp32 accumulation to nearest; over hundreds of MMAs that is a systematic drift of the
// result.  The accumulation is therefore CHUNKED: kGemmChunk K-blocks (48 MMAs) go into the wgmma accumulator, which the consumer
// threads then fold into a second register accumulator with ordinary round-to-nearest fp32 adds.
constexpr int kGemmChunk = 4;

__device__ __noinline__ float gemm_act(float v, int act) {
  switch (act) {
    case EVOK_ACT_TANH: return tanhf(v);
    case EVOK_ACT_RELU: return fmaxf(v, 0.0f);
    case EVOK_ACT_SIGMOID: return __fdiv_rn(1.0f, 1.0f + expf(-v));
    default: return v;
  }
}

// GATHER (implies CONVERT): the A operand is not TMA-addressable (rows only 4-byte aligned, non-uniform pitch: the stacked first-layer
// weights of a population of flat parameter vectors); the two converter warps fetch its tile with coalesced 128-byte row loads and
// write BOTH the raw and the lo tile in the 128-byte-swizzled layout the tensor core expects, so the weights are read from HBM once.
// BATCHED: independent products C_b = A_b B_b^T, item b = blockIdx.z, through rank-3 maps [items][rows][K] (rows past M / N zero-filled
// per item); each item walks the whole K range in the order of a one-split single call, so it gets that call's bits.
template <bool CONVERT, bool GATHER, bool BATCHED>
__device__ __forceinline__ void gemm_tf32x3_body(const CUtensorMap& map_a_hi, const CUtensorMap& map_a_lo, const CUtensorMap& map_b_hi,
                                                 const CUtensorMap& map_b_lo, const GemmParams p) {
  extern __shared__ unsigned char gemm_smem_raw[];
  // tiles need 1024-byte alignment (swizzle atom)
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(gemm_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)kGemmStages * kStageBytes);
  uint64_t* empty = full + kGemmStages;
  uint64_t* conv = empty + kGemmStages;  // [kGemmStages] lo tiles of the stage derived (CONVERT)

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // (uniform: keeps the wgmma path non-divergent)
  const int m0 = blockIdx.x * kGemmBM, n0 = blockIdx.y * kGemmBN;
  const int total_kb = (p.K + kGemmBK - 1) / kGemmBK;
  const int kb_begin = BATCHED ? 0 : blockIdx.z * p.kblocks_per_split;
  const int kb_end = min(total_kb, kb_begin + p.kblocks_per_split);
  const int num_kb = max(kb_end - kb_begin, 0);
  const int64_t item = BATCHED ? blockIdx.z : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kGemmStages; ++s) {
      bar_init(&full[s], 1);
      bar_init(&empty[s], 8);  // one arrival per consumer warp
      bar_init(&conv[s], 2);   // one arrival per converter warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % kGemmStages;
        const uint32_t use = i / kGemmStages;
        bar_wait(&empty[s], (use & 1) ^ 1);  // first use of a stage passes immediately
        unsigned char* st = base + (size_t)s * kStageBytes;
        bar_expect_tx(&full[s], (GATHER ? kTileBBytes : (CONVERT ? kTileABytes + kTileBBytes : kStageBytes)) + ((CONVERT && p.b_lo_tma) ? kTileBBytes : 0u));
        const int kx = (kb_begin + i) * kGemmBK;
        if (BATCHED) {
          const int za = (int)item * p.map_item_a, zb = (int)item * p.map_item_b;
          tma_load_3d(st, &map_a_hi, kx, m0, za, &full[s]);
          if (!CONVERT) tma_load_3d(st + kTileABytes, &map_a_lo, kx, m0, za, &full[s]);
          tma_load_3d(st + 2 * kTileABytes, &map_b_hi, kx, n0, zb, &full[s]);
          if (!CONVERT) tma_load_3d(st + 2 * kTileABytes + kTileBBytes, &map_b_lo, kx, n0, zb, &full[s]);
          continue;
        }
        if (!GATHER) tma_load_2d(st, &map_a_hi, kx, m0, &full[s]);
        if (!CONVERT) tma_load_2d(st + kTileABytes, &map_a_lo, kx, m0, &full[s]);
        tma_load_2d(st + 2 * kTileABytes, &map_b_hi, kx, n0, &full[s]);
        if (!CONVERT || p.b_lo_tma) tma_load_2d(st + 2 * kTileABytes + kTileBBytes, &map_b_lo, kx, n0, &full[s]);
      }
    }
  } else if (warp < 4) {
    // ===== 2 converter warps (CONVERT): per K-block wait for the raw tiles, derive lo = x - trunc_tf32(x) for both operands
    // (element-wise, so every element simply keeps its swizzled position: 2048 float4 per stage, 32 per thread), publish them to
    // the tensor core (async proxy) and signal the consumers.  Runs up to two K-blocks ahead of the MMAs.
    if (CONVERT && warp >= 2) {
      const int ct = threadIdx.x - 64;  // 0 .. 63
      // GATHER: the A tile of K-block i is fetched with 4-byte cp.async copies (global -> shared, no registers, zero fill outside
      // the matrix): one 128-byte row segment per warp instruction, 64 rows per warp, all in flight at once; element (r, k) of a
      // 128B-swizzled K-major tile sits at  r * 128 + ((k / 4) ^ (r % 8)) * 16 + (k % 4) * 4.  The copy of block i + 1 is issued
      // right after block i has been converted, so a 16 KB tile per SM is in flight while the tensor core works on block i.
      auto issue_gather = [&](int i) {
        const int s = i % kGemmStages;
        const uint32_t use = i / kGemmStages;
        bar_wait(&empty[s], (use & 1) ^ 1);  // the stage's previous MMAs are done
        const uint32_t st_a = s32(base + (size_t)s * kStageBytes);
        const int kcol = (kb_begin + i) * kGemmBK + lane;
        const bool k_ok = kcol < p.K;
        const int wrow0 = (warp - 2) * 64;
        const int m_first = m0 + wrow0;
        int hrow = m_first % (int)p.ga_rows_per_batch;
        const float* rowp = p.gather_a + (int64_t)(m_first / (int)p.ga_rows_per_batch) * p.ga_batch_stride + (int64_t)hrow * p.ga_row_stride + kcol;
        const int64_t wrap = p.ga_batch_stride - p.ga_rows_per_batch * p.ga_row_stride;
#pragma unroll 8
        for (int it = 0; it < 64; ++it) {
          const int r = wrow0 + it;
          const bool ok = k_ok && (m0 + r < p.M);
          const uint32_t off = (uint32_t)r * 128u + ((((uint32_t)lane >> 2) ^ ((uint32_t)r & 7u)) << 4) + (((uint32_t)lane & 3u) << 2);
          const float* src = ok ? rowp : p.gather_a;  // a valid address even when nothing is read (src-size 0 -> zero fill)
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(st_a + off), "l"(src), "r"(ok ? 4 : 0) : "memory");
          rowp += p.ga_row_stride;
          if (++hrow == (int)p.ga_rows_per_batch) {
            hrow = 0;
            rowp += wrap;
          }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
      };
      if (GATHER && num_kb > 0) issue_gather(0);
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % kGemmStages;
        const uint32_t use = i / kGemmStages;
        unsigned char* st = base + (size_t)s * kStageBytes;
        if (GATHER) {
          asm volatile("cp.async.wait_group 0;" ::: "memory");  // this thread's copies of block i have landed
          asm volatile("bar.sync 1, 64;" ::: "memory");         // ... and so have the other converter warp's
        }
        bar_wait(&full[s], use & 1);
        const float4* a_raw = reinterpret_cast<const float4*>(st);
        float4* a_lo = reinterpret_cast<float4*>(st + kTileABytes);
        const float4* b_raw = reinterpret_cast<const float4*>(st + 2 * kTileABytes);
        float4* b_lo = reinterpret_cast<float4*>(st + 2 * kTileABytes + kTileBBytes);
        // shared-space 16-byte loads / stores with immediate offsets, 16 loads in flight; B is skipped when its lo tile came by TMA
        split_lo_tile<kTileABytes>(s32(a_raw) + (uint32_t)ct * 16u, s32(a_lo) + (uint32_t)ct * 16u);
        if (!p.b_lo_tma) split_lo_tile<kTileBBytes>(s32(b_raw) + (uint32_t)ct * 16u, s32(b_lo) + (uint32_t)ct * 16u);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core's reads
        __syncwarp();
        if (lane == 0) bar_arrive(&conv[s]);
        // the next block's copy is issued AFTER this block has been handed to the tensor core
        if (GATHER && i + 1 < num_kb) issue_gather(i + 1);
      }
    }
  } else {
    // ===== 2 consumer warpgroups: warpgroup wg owns rows wg * 64 .. wg * 64 + 63 of the tile =====
    const int wg = (warp - 4) >> 2;
    float acc[kAcc], frag[kAcc];
#pragma unroll
    for (int j = 0; j < kAcc; ++j) acc[j] = 0.0f;
    int pending = -1;  // stage whose MMAs may still be in flight (released once the next K-block's wait proves them done)
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) bar_arrive(&empty[s]);
    };
    for (int i = 0; i < num_kb; ++i) {
      const int s = i % kGemmStages;
      const uint32_t use = i / kGemmStages;
      const int in_chunk = i % kGemmChunk;
      bar_wait(CONVERT ? &conv[s] : &full[s], use & 1);  // CONVERT: the converter warps have derived the lo tiles of this stage
      const uint32_t st = s32(base + (size_t)s * kStageBytes);
      mma_kblock(frag, make_sw128_desc(st + wg * kHalfABytes), make_sw128_desc(st + kTileABytes + wg * kHalfABytes),
                 make_sw128_desc(st + 2 * kTileABytes), make_sw128_desc(st + 2 * kTileABytes + kTileBBytes), in_chunk == 0);
      if (in_chunk == kGemmChunk - 1 || i == num_kb - 1) {  // chunk complete: fold it
        wgmma_wait<0>();
        fence_acc(frag);
        if (pending >= 0) release(pending);
        release(s);
        pending = -1;
#pragma unroll
        for (int j = 0; j < kAcc; ++j) acc[j] += frag[j];
      } else {
        wgmma_wait<1>();  // the previous K-block's MMAs are done
        if (pending >= 0) release(pending);
        pending = s;
      }
    }
    wgmma_wait<0>();  // (the last K-block always waited already; this makes it visible to the compiler, which would insert its own)
    // every MMA of both warpgroups has completed (and with them every load and conversion feeding them): the stages are free, use
    // them as a transpose tile so that a warp writes 512 contiguous bytes of one row per instruction
    asm volatile("bar.sync 2, 256;" ::: "memory");
    float* stile = reinterpret_cast<float*>(base);
    {
      const int t = threadIdx.x & 127;
      const int r = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
      for (int j = 0; j < kAcc / 4; ++j) {
        *reinterpret_cast<float2*>(stile + r * kEpiPitch + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(stile + (r + 8) * kEpiPitch + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    asm volatile("bar.sync 2, 256;" ::: "memory");
    const float alpha = (p.C2 && p.alpha_dev) ? p.alpha_dev[item * p.alpha_item_stride] : 1.0f;
    const bool affine = p.affine_k != nullptr && (BATCHED || gridDim.z == 1);
    const float* kk = p.affine_k + item * p.k_item_stride;
    const float k0 = affine ? kk[0] : 1.0f, k1 = affine ? kk[1] : 0.0f, k2 = affine ? kk[2] : 0.0f;
    const float* affine_E = p.affine_E ? p.affine_E + item * p.e_item_stride : nullptr;
    const float* affine_u = p.affine_u ? p.affine_u + item * p.u_item_stride : nullptr;
    const float* bias = p.bias ? p.bias + item * p.bias_item_stride : nullptr;
    float* c2base = p.C2 ? p.C2 + item * p.c2_item_stride : nullptr;
    float* cbase = p.C + (int64_t)blockIdx.z * p.split_stride;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(cbase) & 15) == 0) && (p.ldc % 4 == 0);
    const int col = n0 + lane * 4;
    for (int rr = warp - 4; rr < kGemmBM && m0 + rr < p.M; rr += 8) {
      const int row = m0 + rr;
      const float4 v = *reinterpret_cast<const float4*>(stile + rr * kEpiPitch + lane * 4);
      float e[4] = {v.x, v.y, v.z, v.w};
      if (GATHER && (p.row_bias || p.row_act != EVOK_ACT_NONE)) {  // C = act(acc + bias of this row), bias 0 without one
        float b = 0.0f;
        if (p.row_bias) {
          const int64_t bi = row / p.ga_rows_per_batch;
          b = __ldg(p.row_bias + bi * p.rb_batch_stride + (row - bi * p.ga_rows_per_batch));
        }
        for (int t = 0; t < 4; ++t) e[t] = p.row_act == EVOK_ACT_NONE ? e[t] + b : gemm_act(e[t] + b, p.row_act);
      }
      if (affine) {
        const float ur = affine_u ? __ldg(affine_u + row) : 0.0f;
        for (int t = 0; t < 4; ++t)
          if (col + t < p.N)
            e[t] = fmaf(k0, e[t], fmaf(k1, affine_E ? affine_E[(int64_t)row * p.lde + col + t] : 0.0f,
                                      k2 * ur * (affine_u ? __ldg(affine_u + col + t) : 0.0f)));
      }
      float* cp = cbase + (int64_t)row * p.ldc + col;
      if (vec_ok && col + 4 <= p.N) {
        *reinterpret_cast<float4*>(cp) = make_float4(e[0], e[1], e[2], e[3]);
      } else {
        for (int t = 0; t < 4; ++t)
          if (col + t < p.N) cp[t] = e[t];
      }
      if (c2base) {
        float* c2 = c2base + (int64_t)row * p.ldc2 + col;
        for (int t = 0; t < 4; ++t)
          if (col + t < p.N) c2[t] = fmaf(alpha, e[t], bias ? __ldg(bias + col + t) : 0.0f);
      }
    }
  }
}

template <bool CONVERT, bool GATHER = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
    gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                       const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo, const GemmParams p) {
  gemm_tf32x3_body<CONVERT, GATHER, false>(map_a_hi, map_a_lo, map_b_hi, map_b_lo, p);
}

template <bool CONVERT>
__global__ void __launch_bounds__(kGemmThreads, 1)
    gemm_tf32x3_batched_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                               const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo, const GemmParams p) {
  gemm_tf32x3_body<CONVERT, false, true>(map_a_hi, map_a_lo, map_b_hi, map_b_lo, p);
}

// ---- persistent gather GEMM (batched policy forward on ONE shared minibatch) ------------------------------------------------
// Same arithmetic as gemm_tf32x3_kernel<true, true>, restructured for the shape this path has -- millions of A rows (the stacked
// first-layer weights), a small B operand (the minibatch) that every tile re-reads:
//   * PERSISTENT: one CTA per SM walks the output tiles (tile = blockIdx.x + q * gridDim.x), so barrier set-up happens once and the
//     gather of the next tile's A operand is already in flight while the consumers store the previous tile;
//   * the minibatch is split into hi / lo ONCE by a pre-pass (it is a few hundred KB) and both tiles arrive by TMA: the converter
//     warps only derive the lo tile of the gathered A operand (a third of the element-wise work of the generic kernel);
//   * the gathered A tiles live in a 4-deep ring of raw tiles (three 16 KB gathers in flight per SM while one is converted) with only
//     two lo buffers behind it (a lo tile is derived right before its MMAs); the minibatch tiles (3 stages of hi + lo) come from L2;
//   * the consumers apply bias + activation to their accumulator fragments and store them straight from registers.
// the minibatch operand, pre-split into hi / lo and stored four times, copy s shifted right by s floats (xs[b][k'] = x[b][k' - s], zero
// outside): TMA needs 16-byte aligned box coordinates, so a tile whose rows sit sh floats past a 16-byte boundary reads copy sh at the
// aligned coordinate 32 i instead of the original at 32 i - sh
struct GatherMaps {
  CUtensorMap hi[4];
  CUtensorMap lo[4];
};

constexpr int kPersChunk = 4;  // K-blocks per accumulator chunk, as in the generic kernel
constexpr int kPersRawStages = 4, kPersLoStages = 2, kPersBStages = 3;
constexpr uint32_t kPersBStageBytes = 2 * kTileBBytes;
constexpr size_t kPersSmemBytes =
    (size_t)(kPersRawStages + kPersLoStages) * kTileABytes + (size_t)kPersBStages * kPersBStageBytes + 1024 /*align*/ + 256;

// bias + activation of one accumulator fragment, stored on the way out (one unrolled copy per activation: a per-element switch would
// not fit the instruction cache).  Rows r_first and r_first + 8 of the tile, columns n0 + 8 j + c and + 1.
template <int ACT>
__device__ __forceinline__ float pers_act(float v) {
  if (ACT == EVOK_ACT_RELU) return fmaxf(v, 0.0f);
  if (ACT == EVOK_ACT_TANH) return tanh_abs1e7(v);
  if (ACT == EVOK_ACT_SIGMOID) return activate_fast(v, EVOK_ACT_SIGMOID);
  return v;
}
template <int ACT>
__device__ __forceinline__ void pers_store(const GemmParams& p, const float (&acc)[kAcc], int m0, int r_first, int n0, int c, bool vec_ok) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t m = (int64_t)m0 + r_first + 8 * h;
    if (m >= p.M) continue;
    const int64_t bi = m / p.ga_rows_per_batch, hrow = m - bi * p.ga_rows_per_batch;
    const float b = p.row_bias ? __ldg(p.row_bias + bi * p.rb_batch_stride + hrow) : 0.0f;
    float* crow = p.C + m * p.ldc;
    // unit-fastest layout: the 8 rows a warp holds per register are consecutive units of one batch (32 contiguous bytes per column)
    float* ccol = p.C + (bi * p.N) * p.ga_rows_per_batch + hrow;
#pragma unroll
    for (int j = 0; j < kAcc / 4; ++j) {
      const int col = n0 + 8 * j + c;
      const float v0 = pers_act<ACT>(acc[4 * j + 2 * h] + b), v1 = pers_act<ACT>(acc[4 * j + 2 * h + 1] + b);
      if (p.c_unit_fastest) {
        if (col < p.N) ccol[(int64_t)col * p.ga_rows_per_batch] = v0;
        if (col + 1 < p.N) ccol[(int64_t)(col + 1) * p.ga_rows_per_batch] = v1;
      } else if (vec_ok && col + 2 <= p.N) {
        *reinterpret_cast<float2*>(crow + col) = make_float2(v0, v1);
      } else {
        if (col < p.N) crow[col] = v0;
        if (col + 1 < p.N) crow[col + 1] = v1;
      }
    }
  }
}

__global__ void __launch_bounds__(kGemmThreads, 1)
    gemm_gather_persistent_kernel(const __grid_constant__ GatherMaps maps, const GemmParams p) {
  extern __shared__ unsigned char gemm_smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(gemm_smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* raw_base = base;                                             // gathered A tiles (= the hi operand)
  unsigned char* lo_base = base + (size_t)kPersRawStages * kTileABytes;       // their lo tiles
  unsigned char* b_base = lo_base + (size_t)kPersLoStages * kTileABytes;
  uint64_t* full_b = reinterpret_cast<uint64_t*>(b_base + (size_t)kPersBStages * kPersBStageBytes);
  uint64_t* empty_b = full_b + kPersBStages;
  uint64_t* empty_raw = empty_b + kPersBStages;
  uint64_t* empty_lo = empty_raw + kPersRawStages;
  uint64_t* conv_a = empty_lo + kPersLoStages;

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // (uniform: keeps the wgmma path non-divergent)
  // VECTOR mode (rows of K % 4 == 0 floats at pitch K, a tile never straddles two batches): all rows of a tile share one misalignment
  // `sh` (0..3 floats past a 16-byte boundary), so the K axis of that tile is simply cut at 16-byte-aligned source addresses --
  // K-block i covers k = 32 i - sh .. 32 i - sh + 31 for BOTH operands (the minibatch tile comes from the copy shifted by sh floats,
  // GatherMaps; zeros for k < 0 and k >= K) -- and the gather moves 16 bytes per copy instead of 4.
  const bool vec_mode = (p.K % 4 == 0) && (p.ga_row_stride == p.K) && (p.ga_rows_per_batch % kGemmBM == 0);
  const int num_kb = (p.K + (vec_mode ? 3 : 0) + kGemmBK - 1) / kGemmBK;
  const int n_tiles = (p.N + kGemmBN - 1) / kGemmBN;
  const int64_t total_tiles = (int64_t)((p.M + kGemmBM - 1) / kGemmBM) * n_tiles;
  auto tile_rows = [&](int64_t t, int& m0, int& sh) -> const float* {  // first row of tile t (VECTOR mode) and its misalignment
    m0 = ((int)t / n_tiles) * kGemmBM;  // (fewer than 2^31 tiles: M < 2^31)
    const int rpb = (int)p.ga_rows_per_batch;
    const int bi = m0 / rpb;
    const float* tb = p.gather_a + (int64_t)bi * p.ga_batch_stride + (int64_t)(m0 - bi * rpb) * p.ga_row_stride;
    sh = vec_mode ? (int)((reinterpret_cast<uintptr_t>(tb) >> 2) & 3) : 0;
    return tb;
  };
  const int64_t my_tiles = total_tiles > blockIdx.x ? (total_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kPersBStages; ++s) {
      bar_init(&full_b[s], 1);
      bar_init(&empty_b[s], 8);  // one arrival per consumer warp
    }
    for (int s = 0; s < kPersRawStages; ++s) bar_init(&empty_raw[s], 8);
    for (int s = 0; s < kPersLoStages; ++s) {
      bar_init(&empty_lo[s], 8);
      bar_init(&conv_a[s], 2);  // one arrival per converter warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===== TMA producer of the minibatch tiles (hi, lo) =====
    if (lane == 0) {
      uint32_t g = 0;
      for (int64_t q = 0; q < my_tiles; ++q) {
        const int64_t t = blockIdx.x + q * gridDim.x;
        const int n0 = (int)(t % n_tiles) * kGemmBN;
        int m0_unused, sh;
        tile_rows(t, m0_unused, sh);
        for (int i = 0; i < num_kb; ++i, ++g) {
          const int s = g % kPersBStages;
          bar_wait(&empty_b[s], ((g / kPersBStages) & 1) ^ 1);
          unsigned char* st = b_base + (size_t)s * kPersBStageBytes;
          bar_expect_tx(&full_b[s], kPersBStageBytes);
          tma_load_2d(st, &maps.hi[sh], i * kGemmBK, n0, &full_b[s]);
          tma_load_2d(st + kTileBBytes, &maps.lo[sh], i * kGemmBK, n0, &full_b[s]);
        }
      }
    }
  } else if (warp == 1) {
    // idle
  } else if (warp < 4) {
    // ===== 2 converter warps: gather the A tile of K-block g (64 rows per warp), derive its lo tile =====
    // One warp executes a dependent instruction stream at low IPC, so what bounds this role is its instruction COUNT per K-block:
    // everything that does not change between K-blocks is hoisted (lane offsets, per-tile base / misalignment), shared memory is
    // addressed through 32-bit shared-space addresses (LDS / STS / LDGSTS with immediate offsets), and the rare cases (first chunk of a
    // misaligned row, partial tiles) live in their own branches.
    const int ct = threadIdx.x - 64;
    const uint32_t total_g = (uint32_t)(my_tiles * num_kb);
    const int wrow0 = (warp - 2) * 64;
    const uint32_t raw_s = s32(raw_base), lo_s = s32(lo_base);
    // the issue cursor (tile, K-block) with the per-tile constants of its tile
    int64_t is_t = blockIdx.x;
    int is_i = 0, is_m0 = 0, is_sh = 0;
    const float* is_base = p.gather_a;
    if (my_tiles > 0) is_base = tile_rows(is_t, is_m0, is_sh);
    // VECTOR mode: lane = (row within a group of 4, 16-byte chunk c of the 128-byte row segment); rows wrow0 + 8 j + rsub ("even") and
    // wrow0 + 8 j + 4 + rsub ("odd") for j = 0..7; chunk c of row r sits at r * 128 + ((c ^ (r % 8)) << 4)
    const int c = lane & 7, rsub = lane >> 3;
    const uint32_t off_even = (uint32_t)(wrow0 + rsub) * 128u + ((uint32_t)(c ^ rsub) << 4);
    const uint32_t off_odd = (uint32_t)(wrow0 + 4 + rsub) * 128u + ((uint32_t)(c ^ (4 + rsub)) << 4);
    // 4-byte mode: lane = column of the K-block; element (r, lane) sits at r * 128 + sw[r % 8]
    uint32_t sw[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) sw[j] = ((((uint32_t)lane >> 2) ^ (uint32_t)j) << 4) + (((uint32_t)lane & 3u) << 2);
    const bool rows_regular = (p.ga_rows_per_batch % 64) == 0;  // a warp's 64 rows never straddle two batches
    auto issue_gather = [&](uint32_t g) {
      const int s = g % kPersRawStages;
      bar_wait(&empty_raw[s], ((g / kPersRawStages) & 1) ^ 1);
      const uint32_t st_a = raw_s + (uint32_t)s * kTileABytes;
      const int i = is_i, m0 = is_m0;
      if (vec_mode) {
        const int k_first = i * kGemmBK + 4 * c - is_sh;  // first element of this lane's chunk (16-byte aligned in memory)
        if (k_first >= 0 && m0 + kGemmBM <= p.M) {
          const uint32_t sz = (uint32_t)min(max(p.K - k_first, 0), 4) * 4u;  // bytes read; the rest of the 16 is zero-filled
          const float* src = sz ? is_base + (int64_t)(wrow0 + rsub) * p.K + k_first : is_base - is_sh;  // (any aligned address if sz = 0)
          const int64_t pitch4 = sz ? 4 * (int64_t)p.K : 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(st_a + off_even + (uint32_t)j * 1024u), "l"(src + (2 * j) * pitch4),
                         "r"(sz)
                         : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(st_a + off_odd + (uint32_t)j * 1024u),
                         "l"(src + (2 * j + 1) * pitch4), "r"(sz)
                         : "memory");
          }
        } else {
          // the chunk in front of a misaligned row (K-block 0: its first sh floats are NOT this row's -- they are zeroed rather than
          // left to the minibatch's zero fill, a NaN there would leak into the row), and the rows of a partial last tile
#pragma unroll 1
          for (int it = 0; it < 16; ++it) {
            const int r = wrow0 + it * 4 + rsub;
            const bool row_ok = m0 + r < p.M;
            const uint32_t dst = st_a + (uint32_t)r * 128u + ((uint32_t)(c ^ (r & 7)) << 4);
            const float* src = is_base + (int64_t)r * p.K + k_first;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const bool ok = row_ok && (k_first + e >= 0) && (k_first + e < p.K);
              asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst + 4u * e), "l"(ok ? src + e : p.gather_a), "r"(ok ? 4 : 0)
                           : "memory");
            }
          }
        }
      } else {
        const int kcol = i * kGemmBK + lane;
        const bool k_ok = kcol < p.K;
        const int m_first = m0 + wrow0;
        const uint32_t dst0 = st_a + (uint32_t)wrow0 * 128u;
        const int rpb = (int)p.ga_rows_per_batch;
        int hrow = m_first % rpb;
        const float* rowp = p.gather_a + (int64_t)(m_first / rpb) * p.ga_batch_stride + (int64_t)hrow * p.ga_row_stride + kcol;
        if (rows_regular && m_first + 64 <= p.M) {
          const float* src = k_ok ? rowp : p.gather_a;
          const int64_t pitch = k_ok ? p.ga_row_stride : 0;
          const uint32_t sz = k_ok ? 4u : 0u;
#pragma unroll
          for (int it = 0; it < 64; ++it)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst0 + (uint32_t)it * 128u + sw[it & 7]), "l"(src + it * pitch), "r"(sz)
                         : "memory");
        } else {
          const int64_t wrap = p.ga_batch_stride - p.ga_rows_per_batch * p.ga_row_stride;
#pragma unroll 8
          for (int it = 0; it < 64; ++it) {
            const bool ok = k_ok && (m_first + it < p.M);
            const float* src = ok ? rowp : p.gather_a;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst0 + (uint32_t)it * 128u + sw[it & 7]), "l"(src), "r"(ok ? 4 : 0)
                         : "memory");
            rowp += p.ga_row_stride;
            if (++hrow == rpb) {
              hrow = 0;
              rowp += wrap;
            }
          }
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      if (++is_i == num_kb) {  // the cursor moves on to the next tile of this CTA
        is_i = 0;
        is_t += gridDim.x;
        if (is_t < total_tiles) is_base = tile_rows(is_t, is_m0, is_sh);
      }
    };
    if (total_g > 0) issue_gather(0);
    if (total_g > 1) issue_gather(1);
    if (total_g > 2) issue_gather(2);
    for (uint32_t g = 0; g < total_g; ++g) {
      const int sr = g % kPersRawStages, sl = g % kPersLoStages;
      // block g has landed (blocks g + 1, g + 2 may still be in flight)
      if (g + 2 < total_g) asm volatile("cp.async.wait_group 2;" ::: "memory");
      else if (g + 1 < total_g) asm volatile("cp.async.wait_group 1;" ::: "memory");
      else asm volatile("cp.async.wait_group 0;" ::: "memory");
      asm volatile("bar.sync 1, 64;" ::: "memory");  // ... and so have the other converter warp's rows
      bar_wait(&empty_lo[sl], ((g / kPersLoStages) & 1) ^ 1);  // the MMAs of block g - 2 are done with this lo buffer
      // lo = x - trunc_tf32(x), element-wise (every element keeps its swizzled position): 16 float4 per thread, all loads first
      const uint32_t ra = raw_s + (uint32_t)sr * kTileABytes + (uint32_t)ct * 16u, la = lo_s + (uint32_t)sl * kTileABytes + (uint32_t)ct * 16u;
      split_lo_tile<kTileABytes>(ra, la);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(&conv_a[sl])) : "memory");
      if (g + 3 < total_g) issue_gather(g + 3);
    }
  } else {
    // ===== 2 consumer warpgroups: warpgroup wg owns rows wg * 64 .. wg * 64 + 63 of every tile =====
    const int wg = (warp - 4) >> 2, t = threadIdx.x & 127;
    const int r_first = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2), c = 2 * (t & 3);  // accumulator fragment position (wgmma_tf32)
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && (p.ldc % 4 == 0);
    auto release = [&](uint32_t g) {  // the MMAs of block g are done with its raw, lo and minibatch stages
      __syncwarp();
      if (lane == 0) {
        bar_arrive(&empty_raw[g % kPersRawStages]);
        bar_arrive(&empty_lo[g % kPersLoStages]);
        bar_arrive(&empty_b[g % kPersBStages]);
      }
    };
    uint32_t g = 0;
    for (int64_t q = 0; q < my_tiles; ++q) {
      const int64_t tile = blockIdx.x + q * gridDim.x;
      const int m0 = (int)(tile / n_tiles) * kGemmBM, n0 = (int)(tile % n_tiles) * kGemmBN;
      float acc[kAcc], frag[kAcc];
#pragma unroll
      for (int j = 0; j < kAcc; ++j) acc[j] = 0.0f;
      bool pending = false;  // block g - 1 may still be in flight
      for (int i = 0; i < num_kb; ++i, ++g) {
        const int sr = g % kPersRawStages, sl = g % kPersLoStages, sb = g % kPersBStages;
        const int in_chunk = i % kPersChunk;
        bar_wait(&conv_a[sl], (g / kPersLoStages) & 1);
        bar_wait(&full_b[sb], (g / kPersBStages) & 1);
        const uint32_t stb = s32(b_base + (size_t)sb * kPersBStageBytes);
        mma_kblock(frag, make_sw128_desc(s32(raw_base + (size_t)sr * kTileABytes) + wg * kHalfABytes),
                   make_sw128_desc(s32(lo_base + (size_t)sl * kTileABytes) + wg * kHalfABytes), make_sw128_desc(stb),
                   make_sw128_desc(stb + kTileBBytes), in_chunk == 0);
        if (in_chunk == kPersChunk - 1 || i == num_kb - 1) {  // chunk complete: fold it
          wgmma_wait<0>();
          fence_acc(frag);
          if (pending) release(g - 1);
          release(g);
          pending = false;
#pragma unroll
          for (int j = 0; j < kAcc; ++j) acc[j] += frag[j];
        } else {
          wgmma_wait<1>();
          if (pending) release(g - 1);
          pending = true;
        }
      }
      wgmma_wait<0>();  // (as in gemm_tf32x3_kernel: already true, stated for the compiler)
      switch (p.row_act) {
        case EVOK_ACT_RELU: pers_store<EVOK_ACT_RELU>(p, acc, m0, r_first, n0, c, vec_ok); break;
        case EVOK_ACT_TANH: pers_store<EVOK_ACT_TANH>(p, acc, m0, r_first, n0, c, vec_ok); break;
        case EVOK_ACT_SIGMOID: pers_store<EVOK_ACT_SIGMOID>(p, acc, m0, r_first, n0, c, vec_ok); break;
        default: pers_store<EVOK_ACT_NONE>(p, acc, m0, r_first, n0, c, vec_ok); break;
      }
    }
  }
}

// ---- operand preparation -----------------------------------------------------------------------------------------
// hi = x with the 13 low mantissa bits cleared (exactly representable in TF32), lo = x - hi (exact in fp32)
__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, float* __restrict__ hi,
                                                         float* __restrict__ lo, int64_t ldo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int64_t r = i / cols, c = i % cols;
  const float v = x[r * ldx + c];
  const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  hi[r * ldo + c] = h;
  lo[r * ldo + c] = v - h;
}

// lo[r][c] = x[r][c] - trunc_tf32(x[r][c])   (the pre-split lo copy of the B operand, pitch ldo)
__global__ void __launch_bounds__(256) lo_tf32_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, float* __restrict__ lo,
                                                      int64_t ldo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * ldo) return;
  const int64_t r = i / ldo, c = i - r * ldo;
  const float v = c < cols ? x[r * ldx + c] : 0.0f;
  lo[i] = v - __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
}

// the four shifted hi / lo copies of the minibatch (GatherMaps): hi[s][r][c] / lo[s][r][c] of x[r][c - s], zero for c - s outside [0, cols)
__global__ void __launch_bounds__(256) split_shifted_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, float* __restrict__ hi,
                                                            float* __restrict__ lo, int64_t ldo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * rows * ldo) return;
  const int64_t s = i / (rows * ldo), rem = i - s * rows * ldo;
  const int64_t r = rem / ldo, c = rem - r * ldo - s;
  const float v = (c >= 0 && c < cols) ? x[r * ldx + c] : 0.0f;
  const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  hi[i] = h;
  lo[i] = v - h;
}

// out[c, r] = (w ? w[r] : 1) * in[r, c]   (32 x 32 tiles through shared memory)
__global__ void __launch_bounds__(256) transpose_scale_kernel(const float* __restrict__ in, int64_t ldi, int64_t rows, int64_t cols,
                                                              const float* __restrict__ w, float* __restrict__ out, int64_t ldo) {
  __shared__ float tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.y * 32, c0 = (int64_t)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int k = ty; k < 32; k += 8) {
    const int64_t r = r0 + k, c = c0 + tx;
    tile[k][tx] = (r < rows && c < cols) ? in[r * ldi + c] * (w ? w[r] : 1.0f) : 0.0f;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int64_t c = c0 + k, r = r0 + tx;
    if (c < cols && r < rows) out[c * ldo + r] = tile[tx][k];
  }
}

__global__ void __launch_bounds__(256) reduce_splits_kernel(const float* __restrict__ partial, int splits, int64_t split_stride, int64_t M,
                                                            int64_t N, int64_t ldp, float* C, int64_t ldc, const float* __restrict__ affine_k,
                                                            const float* affine_E, int64_t lde, const float* __restrict__ affine_u) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * N) return;
  const int64_t r = i / N, c = i % N;
  float acc = 0.0f;
  for (int s = 0; s < splits; ++s) acc += partial[(int64_t)s * split_stride + r * ldp + c];
  if (affine_k) {  // same update as the epilogue's (GemmParams::affine_*); E may alias C (element read before it is written)
    const float e = affine_E ? affine_E[r * lde + c] : 0.0f;
    const float uu = affine_u ? affine_u[r] * affine_u[c] : 0.0f;
    acc = fmaf(affine_k[0], acc, fmaf(affine_k[1], e, affine_k[2] * uu));
  }
  C[r * ldc + c] = acc;
}

// hi / lo split copies of a batch of operands: item b's rows x cols at x + b * item_stride (pitch ldx) -> [b][r][c] at pitch ldo
__global__ void __launch_bounds__(256) split_tf32_items_kernel(const float* __restrict__ x, int64_t item_stride, int64_t ldx, int64_t rows,
                                                               int64_t cols, float* __restrict__ hi, float* __restrict__ lo, int64_t ldo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t b = blockIdx.y;
  if (i >= rows * cols) return;
  const int64_t r = i / cols, c = i % cols;
  const float v = x[b * item_stride + r * ldx + c];
  const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  hi[(b * rows + r) * ldo + c] = h;
  lo[(b * rows + r) * ldo + c] = v - h;
}

// Operands of the weighted SYRK  S = Y^T diag(w) Y  as K-major matrices (K = the population axis), built in ONE pass over Y:
//   out_w[c, r] = w[r] * Y[r, c]      out_p[c, r] = Y[r, c]          (32 x 32 tiles through shared memory)
// grid z = item of a batch (strides in elements; 0 for a single operand)
__global__ void __launch_bounds__(256) transpose_pair_kernel(const float* __restrict__ in, int64_t ldi, int64_t rows, int64_t cols,
                                                             const float* __restrict__ w, float* __restrict__ out_w, float* __restrict__ out_p,
                                                             int64_t ldo, int64_t item_stride_in, int64_t item_stride_w, int64_t item_stride_out) {
  __shared__ float tile[32][33];
  __shared__ float wrow[32];
  in += blockIdx.z * item_stride_in;
  w += blockIdx.z * item_stride_w;
  out_w += blockIdx.z * item_stride_out;
  out_p += blockIdx.z * item_stride_out;
  const int64_t r0 = (int64_t)blockIdx.y * 32, c0 = (int64_t)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  if (ty == 0) wrow[tx] = (r0 + tx < rows) ? w[r0 + tx] : 0.0f;
  for (int k = ty; k < 32; k += 8) {
    const int64_t r = r0 + k, c = c0 + tx;
    tile[k][tx] = (r < rows && c < cols) ? in[r * ldi + c] : 0.0f;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int64_t c = c0 + k, r = r0 + tx;
    if (c < cols && r < rows) {
      const float v = tile[tx][k];
      out_p[c * ldo + r] = v;
      out_w[c * ldo + r] = v * wrow[tx];
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 2-D fp32 tensor [rows x K], K contiguous (pitch ld floats); box = 32 floats (128 B) x box_rows; 128-byte swizzle
static int make_map(CUtensorMap* map, const float* ptr, int64_t rows, int64_t K, int64_t ld, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return (int)cudaErrorNotSupported;
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)kGemmBK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

// 3-D fp32 tensor [items][rows][K] (row pitch ld, item pitch item_ld floats); box = 32 floats x box_rows x 1 item; 128-byte swizzle
static int make_map3(CUtensorMap* map, const float* ptr, int64_t items, int64_t rows, int64_t K, int64_t ld, int64_t item_ld, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return (int)cudaErrorNotSupported;
  const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)items};
  const cuuint64_t strides[2] = {(cuuint64_t)ld * sizeof(float), (cuuint64_t)item_ld * sizeof(float)};
  const cuuint32_t box[3] = {(cuuint32_t)kGemmBK, (cuuint32_t)box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

struct GemmPlan {
  int64_t ldk;  // pitch of the split operands (floats), multiple of 4
  int splits, kblocks_per_split;
  size_t off_a_hi, off_a_lo, off_b_hi, off_b_lo, off_partial, total;
};

static GemmPlan plan_gemm(int64_t M, int64_t N, int64_t K, bool allow_split = true) {
  GemmPlan g;
  g.ldk = round_up(K, 4);
  const int64_t tiles = ((M + kGemmBM - 1) / kGemmBM) * ((N + kGemmBN - 1) / kGemmBN);
  const int total_kb = (int)((K + kGemmBK - 1) / kGemmBK);
  int splits = 1;
  while (allow_split && tiles * splits * 2 <= kNumSMs && splits * 2 <= total_kb && splits < 16) splits *= 2;
  g.kblocks_per_split = (total_kb + splits - 1) / splits;
  g.splits = (total_kb + g.kblocks_per_split - 1) / g.kblocks_per_split;
  auto al = [](size_t x) { return (x + 1023) & ~(size_t)1023; };
  size_t o = 0;
  g.off_a_hi = o; o += al((size_t)M * g.ldk * 4);
  g.off_a_lo = o; o += al((size_t)M * g.ldk * 4);
  g.off_b_hi = o; o += al((size_t)N * g.ldk * 4);
  g.off_b_lo = o; o += al((size_t)N * g.ldk * 4);
  g.off_partial = o; o += g.splits > 1 ? al((size_t)g.splits * M * N * 4) : 0;
  g.total = o;
  return g;
}

}  // namespace evok

using namespace evok;

extern "C" EVOK_API size_t evok_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K) {
  if (M <= 0 || N <= 0 || K <= 0) return 1024;
  return plan_gemm(M, N, K).total + 1024;
}

struct GemmAffine {
  const float* k;
  const float* E;
  int64_t lde;
  const float* u;
};

static bool tma_ok(const float* p, int64_t ld) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0 && ld % 4 == 0; }

static int gemm_impl(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc, float* C2,
                     int64_t ldc2, const float* alpha_dev, const float* bias, const GemmAffine* aff, void* ws, size_t ws_bytes, void* stream) {
  if (!A || !B || !C || !ws) return EVOK_E_NULLPTR;
  if (M <= 0 || N <= 0 || K <= 0 || lda < K || ldb < K || ldc < N || (C2 && ldc2 < N)) return EVOK_E_BADSIZE;
  if (M >= (1ll << 31) || N >= (1ll << 31) || K >= (1ll << 31)) return EVOK_E_BADSIZE;
  if (aff && (!aff->k || (aff->u && M != N) || (aff->E && aff->lde < N))) return EVOK_E_BADSIZE;
  const GemmPlan g = plan_gemm(M, N, K, C2 == nullptr);  // the fused second output needs the whole K range in one CTA
  char* w8 = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~(uintptr_t)1023);
  if (ws_bytes < g.total + (size_t)(w8 - (char*)ws)) return EVOK_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  float* partial = (float*)(w8 + g.off_partial);
  // Operands that TMA can address directly (16-byte aligned base and pitch: every matrix this package allocates) are read from
  // HBM once, by the GEMM itself, which derives the lo halves in shared memory; otherwise a pre-pass writes aligned split copies.
  static const int allow_convert = [] {
    const char* e = getenv("EVOK_GEMM_CONVERT");
    return e ? atoi(e) : 1;
  }();
  const bool convert = allow_convert && tma_ok(A, lda) && tma_ok(B, ldb);
  static const int allow_b_lo = [] {
    // =1: B's lo tile by TMA from a pre-split copy instead of the converter warps: half the conversion work, but one more pre-pass
    // launch, which small (CMA-ES-sized) products feel -- off by default
    const char* e = getenv("EVOK_GEMM_B_LO_TMA");
    return e ? atoi(e) : 0;
  }();
  const bool b_lo_tma = convert && allow_b_lo;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  int rc;
  if (convert) {
    if ((rc = make_map(&ma_hi, A, M, K, lda, kGemmBM))) return rc;
    if ((rc = make_map(&mb_hi, B, N, K, ldb, kGemmBN))) return rc;
    ma_lo = ma_hi;
    mb_lo = mb_hi;
    if (b_lo_tma) {  // B's lo tile by TMA from a pre-split copy: the converter warps only derive A's (a third of the element-wise work)
      float* b_lo = (float*)(w8 + g.off_b_lo);
      lo_tf32_kernel<<<(unsigned)((N * g.ldk + 255) / 256), 256, 0, st>>>(B, ldb, N, K, b_lo, g.ldk);
      EVOK_CHECK_LAUNCH();
      if ((rc = make_map(&mb_lo, b_lo, N, K, g.ldk, kGemmBN))) return rc;
    }
  } else {
    float* a_hi = (float*)(w8 + g.off_a_hi);
    float* a_lo = (float*)(w8 + g.off_a_lo);
    float* b_hi = (float*)(w8 + g.off_b_hi);
    float* b_lo = (float*)(w8 + g.off_b_lo);
    split_tf32_kernel<<<(unsigned)((M * K + 255) / 256), 256, 0, st>>>(A, lda, M, K, a_hi, a_lo, g.ldk);
    split_tf32_kernel<<<(unsigned)((N * K + 255) / 256), 256, 0, st>>>(B, ldb, N, K, b_hi, b_lo, g.ldk);
    EVOK_CHECK_LAUNCH_N(2);
    if ((rc = make_map(&ma_hi, a_hi, M, K, g.ldk, kGemmBM))) return rc;
    if ((rc = make_map(&ma_lo, a_lo, M, K, g.ldk, kGemmBM))) return rc;
    if ((rc = make_map(&mb_hi, b_hi, N, K, g.ldk, kGemmBN))) return rc;
    if ((rc = make_map(&mb_lo, b_lo, N, K, g.ldk, kGemmBN))) return rc;
  }
  GemmParams p{};
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.kblocks_per_split = g.kblocks_per_split;
  const bool split = g.splits > 1;
  p.C = split ? partial : C;
  p.ldc = split ? N : ldc;
  p.split_stride = split ? M * N : 0;
  p.C2 = split ? nullptr : C2;
  p.ldc2 = ldc2;
  p.alpha_dev = alpha_dev;
  p.bias = bias;
  p.affine_k = (aff && !split) ? aff->k : nullptr;
  p.affine_E = aff ? aff->E : nullptr;
  p.lde = aff ? aff->lde : 0;
  p.affine_u = aff ? aff->u : nullptr;
  p.gather_a = nullptr;
  p.ga_rows_per_batch = p.ga_batch_stride = p.ga_row_stride = p.rb_batch_stride = 0;
  p.row_bias = nullptr;
  p.row_act = 0;
  p.b_lo_tma = b_lo_tma ? 1 : 0;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_tf32x3_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tf32x3_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tf32x3_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmemBytes) != cudaSuccess)
      return (int)cudaGetLastError();
    attr_set = true;
  }
  dim3 grid((unsigned)((M + kGemmBM - 1) / kGemmBM), (unsigned)((N + kGemmBN - 1) / kGemmBN), (unsigned)g.splits);
  if (convert) gemm_tf32x3_kernel<true, false><<<grid, kGemmThreads, kGemmSmemBytes, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, p);
  else gemm_tf32x3_kernel<false, false><<<grid, kGemmThreads, kGemmSmemBytes, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, p);
  EVOK_CHECK_LAUNCH();
  if (split) {
    reduce_splits_kernel<<<(unsigned)((M * N + 255) / 256), 256, 0, st>>>(partial, g.splits, M * N, M, N, N, C, ldc, aff ? aff->k : nullptr,
                                                                          aff ? aff->E : nullptr, aff ? aff->lde : 0, aff ? aff->u : nullptr);
    EVOK_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" EVOK_API int evok_gemm_nt(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N, int64_t K, float* C,
                                     int64_t ldc, float* C2, int64_t ldc2, const float* alpha_dev, const float* bias, void* ws, size_t ws_bytes,
                                     void* stream) {
  return gemm_impl(A, lda, B, ldb, M, N, K, C, ldc, C2, ldc2, alpha_dev, bias, nullptr, ws, ws_bytes, stream);
}

extern "C" EVOK_API int evok_gemm_nt_affine(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N, int64_t K, float* C,
                                            int64_t ldc, const float* k_dev, const float* E, int64_t lde, const float* u, void* ws, size_t ws_bytes,
                                            void* stream) {
  if (!k_dev) return EVOK_E_NULLPTR;
  const GemmAffine aff{k_dev, E, lde, u};
  return gemm_impl(A, lda, B, ldb, M, N, K, C, ldc, nullptr, 0, nullptr, nullptr, &aff, ws, ws_bytes, stream);
}

// ---- batched products: C_b = A_b B_b^T for n_items items, item b = grid z ------------------------------------------------
struct ItemOperand {
  const float* ptr;
  int64_t ld, item_stride;  // item_stride 0: one matrix shared by every item
};

// read by the GEMM itself through a rank-3 map (16-byte aligned base, row and item pitch, items that do not overlap), or not
static bool tma_ok_items(const ItemOperand& o, int64_t rows) {
  return tma_ok(o.ptr, o.ld) && (o.item_stride == 0 || (o.item_stride % 4 == 0 && o.item_stride >= rows * o.ld));
}

struct BatchedPlan {
  bool convert;  // both operands by TMA straight from their own memory; else both from split copies in the workspace
  int64_t ldk;
  size_t off_a_lo, off_b_hi, off_b_lo, total;
};

static BatchedPlan plan_batched(const ItemOperand& a, const ItemOperand& b, int64_t n_items, int64_t M, int64_t N, int64_t K) {
  BatchedPlan g{};
  g.convert = tma_ok_items(a, M) && tma_ok_items(b, N);
  g.ldk = round_up(K, 4);
  if (g.convert) return g;
  const int64_t chunk = n_items < kMaxGridY ? n_items : kMaxGridY;  // one chunk at a time reuses the copies
  auto al = [](size_t x) { return (x + 1023) & ~(size_t)1023; };
  const size_t a_bytes = al((size_t)(a.item_stride ? chunk : 1) * M * g.ldk * 4), b_bytes = al((size_t)(b.item_stride ? chunk : 1) * N * g.ldk * 4);
  g.off_a_lo = a_bytes;
  g.off_b_hi = 2 * a_bytes;
  g.off_b_lo = 2 * a_bytes + b_bytes;
  g.total = 2 * a_bytes + 2 * b_bytes;
  return g;
}

// per-item epilogue operands and their item strides (0 = shared)
struct ItemEpilogue {
  float* C2;
  int64_t ldc2, item_stride_c2;
  const float* alpha;
  int64_t item_stride_alpha;
  const float* bias;
  int64_t item_stride_bias;
  const GemmAffine* aff;
  int64_t item_stride_k, item_stride_e, item_stride_u;
};

static int gemm_batched_impl(const ItemOperand& a, const ItemOperand& b, int64_t n_items, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc,
                             int64_t item_stride_c, const ItemEpilogue& ep, void* ws, size_t ws_bytes, void* stream) {
  const GemmAffine* aff = ep.aff;
  if (!a.ptr || !b.ptr || !C || !ws) return EVOK_E_NULLPTR;
  if (n_items < 0 || M <= 0 || N <= 0 || K <= 0 || a.ld < K || b.ld < K || ldc < N || (ep.C2 && ep.ldc2 < N)) return EVOK_E_BADSIZE;
  if (M >= (1ll << 31) || N >= (1ll << 31) || K >= (1ll << 31)) return EVOK_E_BADSIZE;
  if (a.item_stride < 0 || b.item_stride < 0 || ep.item_stride_alpha < 0 || ep.item_stride_bias < 0 || ep.item_stride_k < 0 || ep.item_stride_e < 0 ||
      ep.item_stride_u < 0)
    return EVOK_E_BADSIZE;
  // the outputs belong to one item each
  if (n_items > 1 && (item_stride_c < (M - 1) * ldc + N || (ep.C2 && ep.item_stride_c2 < (M - 1) * ep.ldc2 + N))) return EVOK_E_BADSIZE;
  if (aff && (!aff->k || (aff->u && M != N) || (aff->E && aff->lde < N))) return EVOK_E_BADSIZE;
  if (n_items == 0) return 0;
  const BatchedPlan g = plan_batched(a, b, n_items, M, N, K);
  char* w8 = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~(uintptr_t)1023);
  if (ws_bytes < g.total + (size_t)(w8 - (char*)ws)) return EVOK_E_WORKSPACE;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_tf32x3_batched_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tf32x3_batched_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmemBytes) != cudaSuccess)
      return (int)cudaGetLastError();
    attr_set = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    const float* pa = a.ptr + b0 * a.item_stride;
    const float* pb = b.ptr + b0 * b.item_stride;
    const int64_t ia = a.item_stride ? nb : 1, ib = b.item_stride ? nb : 1;
    CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
    int rc;
    if (g.convert) {
      if ((rc = make_map3(&ma_hi, pa, ia, M, K, a.ld, a.item_stride ? a.item_stride : M * a.ld, kGemmBM))) return rc;
      if ((rc = make_map3(&mb_hi, pb, ib, N, K, b.ld, b.item_stride ? b.item_stride : N * b.ld, kGemmBN))) return rc;
      ma_lo = ma_hi;
      mb_lo = mb_hi;
    } else {
      float* a_hi = (float*)w8;
      float* a_lo = (float*)(w8 + g.off_a_lo);
      float* b_hi = (float*)(w8 + g.off_b_hi);
      float* b_lo = (float*)(w8 + g.off_b_lo);
      split_tf32_items_kernel<<<dim3((unsigned)((M * K + 255) / 256), (unsigned)ia), 256, 0, st>>>(pa, a.item_stride, a.ld, M, K, a_hi, a_lo, g.ldk);
      split_tf32_items_kernel<<<dim3((unsigned)((N * K + 255) / 256), (unsigned)ib), 256, 0, st>>>(pb, b.item_stride, b.ld, N, K, b_hi, b_lo, g.ldk);
      EVOK_CHECK_LAUNCH_N(2);
      if ((rc = make_map3(&ma_hi, a_hi, ia, M, K, g.ldk, M * g.ldk, kGemmBM))) return rc;
      if ((rc = make_map3(&ma_lo, a_lo, ia, M, K, g.ldk, M * g.ldk, kGemmBM))) return rc;
      if ((rc = make_map3(&mb_hi, b_hi, ib, N, K, g.ldk, N * g.ldk, kGemmBN))) return rc;
      if ((rc = make_map3(&mb_lo, b_lo, ib, N, K, g.ldk, N * g.ldk, kGemmBN))) return rc;
    }
    GemmParams p{};
    p.M = (int)M; p.N = (int)N; p.K = (int)K;
    p.kblocks_per_split = (int)((K + kGemmBK - 1) / kGemmBK);  // never split K: the items fill the grid
    p.C = C + b0 * item_stride_c;
    p.ldc = ldc;
    p.split_stride = item_stride_c;
    p.C2 = ep.C2 ? ep.C2 + b0 * ep.item_stride_c2 : nullptr;
    p.ldc2 = ep.ldc2;
    p.c2_item_stride = ep.item_stride_c2;
    p.alpha_dev = ep.alpha ? ep.alpha + b0 * ep.item_stride_alpha : nullptr;
    p.alpha_item_stride = ep.item_stride_alpha;
    p.bias = ep.bias ? ep.bias + b0 * ep.item_stride_bias : nullptr;
    p.bias_item_stride = ep.item_stride_bias;
    if (aff) {
      p.affine_k = aff->k + b0 * ep.item_stride_k;
      p.k_item_stride = ep.item_stride_k;
      p.affine_E = aff->E ? aff->E + b0 * ep.item_stride_e : nullptr;
      p.lde = aff->lde;
      p.e_item_stride = ep.item_stride_e;
      p.affine_u = aff->u ? aff->u + b0 * ep.item_stride_u : nullptr;
      p.u_item_stride = ep.item_stride_u;
    }
    p.map_item_a = a.item_stride ? 1 : 0;
    p.map_item_b = b.item_stride ? 1 : 0;
    const dim3 grid((unsigned)((M + kGemmBM - 1) / kGemmBM), (unsigned)((N + kGemmBN - 1) / kGemmBN), (unsigned)nb);
    if (g.convert) gemm_tf32x3_batched_kernel<true><<<grid, kGemmThreads, kGemmSmemBytes, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, p);
    else gemm_tf32x3_batched_kernel<false><<<grid, kGemmThreads, kGemmSmemBytes, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, p);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API size_t evok_gemm_nt_batched_workspace_bytes(const float* A, int64_t lda, int64_t item_stride_a, const float* B, int64_t ldb,
                                                                int64_t item_stride_b, int64_t n_items, int64_t M, int64_t N, int64_t K) {
  if (n_items <= 0 || M <= 0 || N <= 0 || K <= 0) return 1024;
  return plan_batched(ItemOperand{A, lda, item_stride_a}, ItemOperand{B, ldb, item_stride_b}, n_items, M, N, K).total + 1024;
}

extern "C" EVOK_API int evok_gemm_nt_batched(const float* A, int64_t lda, int64_t item_stride_a, const float* B, int64_t ldb, int64_t item_stride_b,
                                             int64_t n_items, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc, int64_t item_stride_c, float* C2,
                                             int64_t ldc2, int64_t item_stride_c2, const float* alpha_dev, int64_t item_stride_alpha, const float* bias,
                                             int64_t item_stride_bias, void* ws, size_t ws_bytes, void* stream) {
  const ItemEpilogue ep{C2, ldc2, item_stride_c2, alpha_dev, item_stride_alpha, bias, item_stride_bias, nullptr, 0, 0, 0};
  return gemm_batched_impl(ItemOperand{A, lda, item_stride_a}, ItemOperand{B, ldb, item_stride_b}, n_items, M, N, K, C, ldc, item_stride_c, ep, ws,
                           ws_bytes, stream);
}

extern "C" EVOK_API int evok_gemm_nt_affine_batched(const float* A, int64_t lda, int64_t item_stride_a, const float* B, int64_t ldb,
                                                    int64_t item_stride_b, int64_t n_items, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc,
                                                    int64_t item_stride_c, const float* k_dev, int64_t item_stride_k, const float* E, int64_t lde,
                                                    int64_t item_stride_e, const float* u, int64_t item_stride_u, void* ws, size_t ws_bytes,
                                                    void* stream) {
  if (!k_dev) return EVOK_E_NULLPTR;
  const GemmAffine aff{k_dev, E, lde, u};
  const ItemEpilogue ep{nullptr, 0, 0, nullptr, 0, nullptr, 0, &aff, item_stride_k, item_stride_e, item_stride_u};
  return gemm_batched_impl(ItemOperand{A, lda, item_stride_a}, ItemOperand{B, ldb, item_stride_b}, n_items, M, N, K, C, ldc, item_stride_c, ep, ws,
                           ws_bytes, stream);
}

// Stacked-rows GEMM of the batched policy forward:  C[(i, h), b] = act( sum_k W_i[h, k] * X[b, k] + bias_i[h] )
// A rows gathered from the population matrix (see GemmParams::gather_a), B = the shared input batch X (n_cols x K, TMA: 16-byte aligned).
extern "C" EVOK_API int evok_gemm_gather_rows(const float* params, int64_t batch_stride, int64_t w_offset, int64_t rows_per_batch, int64_t n_batches,
                                              const float* X, int64_t ldx, int64_t n_cols, int64_t K, int64_t bias_offset, int act, float* C,
                                              int64_t ldc, void* stream) {
  if (!params || !X || !C) return EVOK_E_NULLPTR;
  const int64_t M = rows_per_batch * n_batches;
  if (rows_per_batch <= 0 || n_batches <= 0 || n_cols <= 0 || K <= 0 || ldx < K || ldc < n_cols || M >= (1ll << 31)) return EVOK_E_BADSIZE;
  if (act < EVOK_ACT_NONE || act > EVOK_ACT_SIGMOID) return EVOK_E_BADENUM;
  if (!tma_ok(X, ldx)) return EVOK_E_ALIGN;
  CUtensorMap mb;
  int rc;
  if ((rc = make_map(&mb, X, n_cols, K, ldx, kGemmBN))) return rc;
  GemmParams p{};
  p.M = (int)M; p.N = (int)n_cols; p.K = (int)K;
  p.kblocks_per_split = (int)((K + kGemmBK - 1) / kGemmBK);
  p.C = C;
  p.ldc = ldc;
  p.gather_a = params + w_offset;
  p.ga_rows_per_batch = rows_per_batch;
  p.ga_batch_stride = batch_stride;
  p.ga_row_stride = K;
  p.row_bias = bias_offset >= 0 ? params + bias_offset : nullptr;
  p.rb_batch_stride = batch_stride;
  p.row_act = act;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_tf32x3_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmemBytes) != cudaSuccess)
      return (int)cudaGetLastError();
    attr_set = true;
  }
  dim3 grid((unsigned)((M + kGemmBM - 1) / kGemmBM), (unsigned)((n_cols + kGemmBN - 1) / kGemmBN), 1);
  gemm_tf32x3_kernel<true, true><<<grid, kGemmThreads, kGemmSmemBytes, (cudaStream_t)stream>>>(mb, mb, mb, mb, p);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API size_t evok_gemm_gather_rows_workspace_bytes(int64_t n_cols, int64_t K) {
  if (n_cols <= 0 || K <= 0) return 512;
  return (size_t)8 * n_cols * round_up(K + 3, 4) * sizeof(float) + 512;  // 4 shifted copies of the hi and of the lo part
}

// The same product on the persistent kernel (gemm_gather_persistent_kernel): X is split into hi / lo copies in `ws` first (any
// alignment / pitch of X is fine).  unit_fastest = 1 writes C[(batch * n_cols + col) * rows_per_batch + row] instead of the row-major
// C[(batch * rows_per_batch + row) * ldc + col]: the rows a warp stores per instruction are consecutive floats.
// EVOK_GATHER_PERSISTENT=0 routes the row-major case to the one-tile-per-CTA kernel instead (measurement only).
extern "C" EVOK_API int evok_gemm_gather_rows_ws(const float* params, int64_t batch_stride, int64_t w_offset, int64_t rows_per_batch,
                                                 int64_t n_batches, const float* X, int64_t ldx, int64_t n_cols, int64_t K, int64_t bias_offset,
                                                 int act, float* C, int64_t ldc, int unit_fastest, void* ws, size_t ws_bytes, void* stream) {
  if (!params || !X || !C || !ws) return EVOK_E_NULLPTR;
  const int64_t M = rows_per_batch * n_batches;
  if (rows_per_batch <= 0 || n_batches <= 0 || n_cols <= 0 || K <= 0 || ldx < K || (!unit_fastest && ldc < n_cols) || M >= (1ll << 31))
    return EVOK_E_BADSIZE;
  if (act < EVOK_ACT_NONE || act > EVOK_ACT_SIGMOID) return EVOK_E_BADENUM;
  {
    const char* e = getenv("EVOK_GATHER_PERSISTENT");
    if (!unit_fastest && e && atoi(e) == 0 && tma_ok(X, ldx))
      return evok_gemm_gather_rows(params, batch_stride, w_offset, rows_per_batch, n_batches, X, ldx, n_cols, K, bias_offset, act, C, ldc, stream);
  }
  const int64_t ldk = round_up(K + 3, 4);
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  if (ws_bytes < (size_t)(base - (char*)ws) + (size_t)8 * n_cols * ldk * sizeof(float)) return EVOK_E_WORKSPACE;
  float* x_hi = reinterpret_cast<float*>(base);
  float* x_lo = x_hi + 4 * n_cols * ldk;
  split_shifted_kernel<<<(unsigned)((4 * n_cols * ldk + 255) / 256), 256, 0, (cudaStream_t)stream>>>(X, ldx, n_cols, K, x_hi, x_lo, ldk);
  EVOK_CHECK_LAUNCH();
  GatherMaps maps;
  int rc;
  for (int s = 0; s < 4; ++s) {
    if ((rc = make_map(&maps.hi[s], x_hi + s * n_cols * ldk, n_cols, ldk, ldk, kGemmBN))) return rc;
    if ((rc = make_map(&maps.lo[s], x_lo + s * n_cols * ldk, n_cols, ldk, ldk, kGemmBN))) return rc;
  }
  GemmParams p{};
  p.M = (int)M; p.N = (int)n_cols; p.K = (int)K;
  p.kblocks_per_split = (int)((K + kGemmBK - 1) / kGemmBK);
  p.C = C;
  p.ldc = ldc;
  p.gather_a = params + w_offset;
  p.ga_rows_per_batch = rows_per_batch;
  p.ga_batch_stride = batch_stride;
  p.ga_row_stride = K;
  p.row_bias = bias_offset >= 0 ? params + bias_offset : nullptr;
  p.rb_batch_stride = batch_stride;
  p.row_act = act;
  p.c_unit_fastest = unit_fastest ? 1 : 0;
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sm_count <= 0) sm_count = kNumSMs;
    if (cudaFuncSetAttribute(gemm_gather_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPersSmemBytes) != cudaSuccess) {
      sm_count = 0;
      return (int)cudaGetLastError();
    }
  }
  const int64_t tiles = ((M + kGemmBM - 1) / kGemmBM) * ((n_cols + kGemmBN - 1) / kGemmBN);
  const unsigned grid = (unsigned)(tiles < sm_count ? tiles : sm_count);
  gemm_gather_persistent_kernel<<<grid, kGemmThreads, kPersSmemBytes, (cudaStream_t)stream>>>(maps, p);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_transpose_pair(const float* in, int64_t ldi, int64_t rows, int64_t cols, const float* w, float* out_w, float* out_p,
                                            int64_t ldo, void* stream) {
  if (!in || !w || !out_w || !out_p) return EVOK_E_NULLPTR;
  if (rows <= 0 || cols <= 0 || ldi < cols || ldo < rows) return EVOK_E_BADSIZE;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
  transpose_pair_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, ldi, rows, cols, w, out_w, out_p, ldo, 0, 0, 0);
  EVOK_CHECK_LAUNCH();
  return 0;
}

extern "C" EVOK_API int evok_transpose_pair_batched(const float* in, int64_t ldi, int64_t item_stride_in, int64_t rows, int64_t cols, const float* w,
                                                    int64_t item_stride_w, float* out_w, float* out_p, int64_t ldo, int64_t item_stride_out,
                                                    int64_t n_items, void* stream) {
  if (!in || !w || !out_w || !out_p) return EVOK_E_NULLPTR;
  if (rows <= 0 || cols <= 0 || n_items < 0 || ldi < cols || ldo < rows || item_stride_in < 0 || item_stride_w < 0) return EVOK_E_BADSIZE;
  if (n_items > 1 && item_stride_out < cols * ldo) return EVOK_E_BADSIZE;  // the outputs are per item
  if ((rows + 31) / 32 > kMaxGridY) return EVOK_E_BADSIZE;
  const dim3 tiles((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
  return for_item_chunks(n_items, kMaxGridY, [&](int64_t b0, int64_t nb) {
    transpose_pair_kernel<<<dim3(tiles.x, tiles.y, (unsigned)nb), 256, 0, (cudaStream_t)stream>>>(
        in + b0 * item_stride_in, ldi, rows, cols, w + b0 * item_stride_w, out_w + b0 * item_stride_out, out_p + b0 * item_stride_out, ldo,
        item_stride_in, item_stride_w, item_stride_out);
    EVOK_CHECK_LAUNCH();
    return 0;
  });
}

extern "C" EVOK_API int evok_transpose_scale(const float* in, int64_t ldi, int64_t rows, int64_t cols, const float* w, float* out, int64_t ldo,
                                             void* stream) {
  if (!in || !out) return EVOK_E_NULLPTR;
  if (rows <= 0 || cols <= 0 || ldi < cols || ldo < rows) return EVOK_E_BADSIZE;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
  transpose_scale_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, ldi, rows, cols, w, out, ldo);
  EVOK_CHECK_LAUNCH();
  return 0;
}
