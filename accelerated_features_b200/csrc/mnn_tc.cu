// Mutual-NN similarity scan on the Hopper tensor cores (wgmma + TMA), fp32-equivalent precision.
//
// fp32-equivalent via operand splitting: x*s = hi + lo with hi, lo in fp16 (s = power of two chosen from max|x| so that
// hi uses the fp16 range and lo stays normal), rows stored as [hi(64) | lo(64)] halves, and three K = 64 fp16 GEMM blocks
// with fp32 accumulation into the same register tile
//      S = hi1.hi2^T + hi1.lo2^T + lo1.hi2^T
// (the dropped lo.lo term is ~2^-22 relative, below fp32 accumulation noise).  The blocks are selected by the wgmma
// descriptor addresses (hi box / lo box of each operand), so nothing is stored twice.  The same two arrays serve both scan
// directions (rows of F1 against F2, rows of F2 against F1), which add the same three products in the same order.
//
// One work item = 256 rows (two 128-row slabs) x all 128-column tiles of the other set; TMA streams the B tiles through a
// ring of stages while the two consumer warpgroups reduce.  Nothing but the final (value, index) per row ever leaves the SM.
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

constexpr int TC_ROWS = 256, TC_BN = 128, TC_KP = 128, TC_BOX_BYTES = 128 * 128;  // operand row [hi(64) | lo(64)]; box = 128 rows x 128 B
constexpr size_t TC_SMEM = 1024 + 8 * (size_t)TC_BOX_BYTES + 256;

// max |x| over the first n rows of each set into *out.  kPairs: one word per pair instead -- out[p] = max |x| over the first n
// rows of both images of pairs[p] = (i, j) (blockIdx.z = side) of one table of images at `stride` floats each, exactly the
// maximum the single-pair launch measures over its two sets.  A template flag, so that the per-set build keeps its code.
template <bool kPairs = false>
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ f, const int* __restrict__ np, int n_max,
                                                     int64_t stride, unsigned* __restrict__ out,
                                                     const int2* __restrict__ pairs = nullptr) {
  const int pair = blockIdx.y;
  const int set = kPairs ? (blockIdx.z ? __ldg(pairs + pair).y : __ldg(pairs + pair).x) : pair;
  const int n = np ? min(np[set], n_max) : n_max;
  const float4* p = reinterpret_cast<const float4*>(f + (int64_t)set * stride);
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * 16; i += gridDim.x * blockDim.x) {
    const float4 v = __ldg(p + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out + (kPairs ? pair : 0), __float_as_uint(m));
}

// One warp per row: writes the 128-half split row [hi(64) | lo(64)]; zero rows past n.
// kPairs: pair p = pairs[p] = (i, j) of one table of images at `stride` floats each; side s = blockIdx.z splits the rows of
// image (s ? j : i) at the exponent of the pair's own maximum absmax[p] (absmax_kernel<true>) into block s * gridDim.y + p of
// `out` (side 0: the pairs' A rows, side 1: their B rows), and writes that image's count to cnt[s * gridDim.y + p].
template <bool kPairs = false>
__global__ void __launch_bounds__(256) split_kernel(const float* __restrict__ f, const int* __restrict__ np, int n_max,
                                                    int n_pad, int64_t stride, const unsigned* __restrict__ absmax,
                                                    float abs_bound, __half* __restrict__ out, float* __restrict__ inv_s2,
                                                    const int2* __restrict__ pairs = nullptr, int* __restrict__ cnt = nullptr) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int pair = blockIdx.y;
  if (wid >= n_pad) return;
  const int set = kPairs ? (blockIdx.z ? __ldg(pairs + pair).y : __ldg(pairs + pair).x) : pair;
  const int blk = kPairs ? (int)(blockIdx.z * gridDim.y) + pair : pair;
  const int n = np ? min(np[set], n_max) : n_max;
  const float mx = abs_bound > 0.f ? abs_bound : __uint_as_float(absmax[kPairs ? pair : 0]);   // caller's bound or the measured maximum
  int e = 0;
  if (mx > 0.f) frexpf(mx, &e);                 // mx = m * 2^e, m in [0.5, 1)  ->  mx < 2^e
  const float s = (mx > 0.f) ? ldexpf(1.f, 14 - e) : 1.f;   // mx * s in [2^13, 2^14)
  if (wid == 0 && lane == 0 && pair == 0 && inv_s2) *inv_s2 = (mx > 0.f) ? ldexpf(1.f, 2 * (e - 14)) : 1.f;
  if (kPairs && wid == 0 && lane == 0) cnt[blk] = np[set];
  __half2 hi = __floats2half2_rn(0.f, 0.f), lo = hi;
  if (wid < n) {
    const float2 v = __ldg(reinterpret_cast<const float2*>(f + (int64_t)set * stride + wid * 64) + lane);
    const float x0 = v.x * s, x1 = v.y * s;      // exact (power of two)
    hi = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(hi);
    lo = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  }
  __half2* o = reinterpret_cast<__half2*>(out + ((int64_t)blk * n_pad + wid) * TC_KP);
  o[lane] = hi;
  o[32 + lane] = lo;
}

struct TcMaps {
  CUtensorMap m1, m2;
};
// operand arrays per scan direction: direction d multiplies rows of a<d> (the scanned rows) with rows of b<d> (the columns).
// Full scan: a0 = b1 = set 1, b0 = a1 = set 2.  Re-scoring pass of mnn_fast.cu: a<d> = compact lists of ambiguous rows.
struct TcMaps4 {
  CUtensorMap a0, b0, a1, b1;
};

// ---------------------------------------------------------------------------------------------------------------------
// Hopper mapping (shared by the kernels below): 256 rows per work item = two 128-row slabs, one consumer warpgroup per slab
// (warps 0-3 / 4-7) issuing wgmma 64 x 128 x 16 for its two 64-row halves into registers; warp 8 = TMA producer.  A thread
// holds, per tile, rows 16w + l/4 + {0, 8, 64, 72} of its slab (w = warp in the group, l = lane) and columns 8j + 2(l%4) + {0,1}.
// The row arg-max is reduced in-thread, then across the four lanes of a row as packed (value, ~column) 64-bit maxima
// (pack_vi: larger value, then lower column -- torch's first-index rule).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int MT_THREADS = 288;           // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr uint32_t MT_HALF = (64 * 128) >> 4;   // descriptor offset of rows 64-127 of a slab

// three-term S tile of one slab: hi.hi + (dir ? lo.hi, hi.lo : hi.lo, lo.hi), both directions in the same order so that
// S12[i][j] and S21[j][i] come out of the same three products
__device__ __forceinline__ void mnn_tile_mma_issue(float (&acc0)[64], float (&acc1)[64], uint32_t a_slab, uint32_t b_stage, int dir) {
  const int a_sel[3] = {0, dir ? 1 : 0, dir ? 0 : 1};
  const int b_sel[3] = {0, dir ? 0 : 1, dir ? 1 : 0};
  tc::wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < 3; ++kb) {
    const uint64_t da = tc::make_desc_sw128(a_slab + a_sel[kb] * TC_BOX_BYTES, 1024);
    const uint64_t db = tc::make_desc_sw128(b_stage + b_sel[kb] * TC_BOX_BYTES, 1024);
#pragma unroll
    for (int k = 0; k < 4; ++k) {   // 16 halves = 32 B = 2 x 16-byte units along K inside the 128 B swizzle row
      tc::wgmma_f16<128>(acc0, da + 2 * k, db + 2 * k, (kb | k) ? 1u : 0u);
      tc::wgmma_f16<128>(acc1, da + MT_HALF + 2 * k, db + 2 * k, (kb | k) ? 1u : 0u);
    }
  }
  tc::wgmma_commit();
}
__device__ __forceinline__ void mnn_tile_mma(float (&acc0)[64], float (&acc1)[64], uint32_t a_slab, uint32_t b_stage, int dir) {
  mnn_tile_mma_issue(acc0, acc1, a_slab, b_stage, dir);
  tc::wgmma_wait<0>();
  tc::acc_fence(acc0);
  tc::acc_fence(acc1);
}

// running row arg-max of the thread's four rows over one tile (columns col0 .. col0+127, the first n_valid of them real)
__device__ __forceinline__ void mnn_row_argmax(const float (&acc0)[64], const float (&acc1)[64], int col0, int n_valid,
                                               int lane, unsigned long long (&best)[4]) {
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    float m = -INFINITY;
    int c = -1;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = tc::frag_val(acc0, acc1, h, j, e);
        const int cc = 8 * j + cq + e;
        if (cc < n_valid && v > m) { m = v; c = cc; }   // strict, columns ascending: first index wins ties
      }
    unsigned long long p = (c >= 0) ? pack_vi(m, (uint32_t)(col0 + c)) : 0ull;
    unsigned long long o = __shfl_xor_sync(0xffffffffu, p, 1);
    p = o > p ? o : p;
    o = __shfl_xor_sync(0xffffffffu, p, 2);
    p = o > p ? o : p;
    best[h] = p > best[h] ? p : best[h];
  }
}

// rows_cnt (optional): [pair][dir] number of rows of the A array to scan (the compact lists of mnn_fast.cu) instead of the
// set size; row_map (optional): [pair][dir][n_pad] output row of compact row r.
// pairs (optional): pair p = (image i, image j) of one image table of n_images * n_pad rows that every map covers; the counts are
// n1p[i] and n2p[j], the A rows of direction 0 start at i * n_pad and its B rows at j * n_pad (the other way round for direction 1).
// best12 / best21 stay per pair.  NULL: image p of each set is pair p.
__global__ void __launch_bounds__(MT_THREADS, 1) mnn_tc_kernel(const __grid_constant__ TcMaps4 maps,
                                                               const int* __restrict__ n1p, int n1_max,
                                                               const int* __restrict__ n2p, int n2_max, int n_pad,
                                                               unsigned long long* __restrict__ best12,
                                                               unsigned long long* __restrict__ best21,
                                                               const int* __restrict__ rows_cnt,
                                                               const int* __restrict__ row_map,
                                                               const int2* __restrict__ pairs) {
  const int pair = blockIdx.y, dir = blockIdx.z;
  const int2 ij = pairs ? __ldg(pairs + pair) : make_int2(pair, pair);
  const int n1 = n1p ? min(n1p[ij.x], n1_max) : n1_max;
  const int n2 = n2p ? min(n2p[ij.y], n2_max) : n2_max;
  const int n_rows = rows_cnt ? min(rows_cnt[pair * 2 + dir], n_pad) : (dir ? n2 : n1), n_cols = dir ? n1 : n2;
  const int out_stride = dir ? n2_max : n1_max;
  unsigned long long* out = dir ? best21 : best12;
  const CUtensorMap* mapA = dir ? &maps.a1 : &maps.a0;
  const CUtensorMap* mapB = dir ? &maps.b1 : &maps.b0;
  const int row0 = blockIdx.x * TC_ROWS;
  if (row0 >= n_rows) return;

  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sA = base;                       // [slab 2][hi, lo] boxes
  unsigned char* sB = base + 4 * TC_BOX_BYTES;    // [stage 2][hi, lo] boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + 8 * TC_BOX_BYTES);
  uint64_t* a_full = bars;
  uint64_t* b_full = bars + 1;     // [2]
  uint64_t* b_empty = bars + 3;    // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = (n_cols + TC_BN - 1) / TC_BN;

  if (warp == 8 && lane == 0) {
    tc::tma_prefetch_desc(mapA);
    tc::tma_prefetch_desc(mapB);
    tc::mbar_init(a_full, 1);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&b_full[i], 1);
      tc::mbar_init(&b_empty[i], 8);   // one arrival per consumer warp
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (T > 0 && tc::elect_one()) {
      // ---------------- TMA producer ----------------
      const int arow = (dir ? ij.y : ij.x) * n_pad + row0;
      tc::mbar_expect_tx(a_full, 4 * TC_BOX_BYTES);
      for (int slab = 0; slab < 2; ++slab)
        for (int kb = 0; kb < 2; ++kb)
          tc::tma_load_2d(sA + (slab * 2 + kb) * TC_BOX_BYTES, mapA, a_full, kb * 64, arow + slab * 128);
      const int brow = (dir ? ij.x : ij.y) * n_pad;
      for (int t = 0; t < T; ++t) {
        const int s = t & 1;
        tc::mbar_wait(&b_empty[s], ((t >> 1) & 1) ^ 1);
        tc::mbar_expect_tx(&b_full[s], 2 * TC_BOX_BYTES);
        for (int kb = 0; kb < 2; ++kb)
          tc::tma_load_2d(sB + (s * 2 + kb) * TC_BOX_BYTES, mapB, &b_full[s], kb * 64, brow + t * TC_BN);
      }
    }
    __syncwarp();
  } else {
    // ---------------- consumer warpgroup `slab`: wgmma + running row arg-max ----------------
    const int slab = warp >> 2, wt = threadIdx.x & 127;
    float acc0[64], acc1[64];
    unsigned long long best[4] = {0ull, 0ull, 0ull, 0ull};
    if (T > 0) tc::mbar_wait(a_full, 0);
    const uint32_t a_slab = tc::smem_u32(sA + slab * 2 * TC_BOX_BYTES);
    for (int t = 0; t < T; ++t) {
      const int s = t & 1;
      tc::mbar_wait(&b_full[s], (t >> 1) & 1);
      mnn_tile_mma(acc0, acc1, a_slab, tc::smem_u32(sB + s * 2 * TC_BOX_BYTES), dir);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&b_empty[s]);   // this warp's reads of the B stage are complete
      mnn_row_argmax(acc0, acc1, t * TC_BN, n_cols - t * TC_BN, lane, best);
    }
    if ((lane & 3) == 0) {
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int row = row0 + slab * 128 + tc::frag_row(wt, h);
        if (row < n_rows) {
          const int orow = row_map ? __ldg(row_map + (int64_t)(pair * 2 + dir) * n_pad + row) : row;
          out[(int64_t)pair * out_stride + orow] = best[h];
        }
      }
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Persistent form of mnn_tc_kernel (implementation 2, the reference of the single-GEMM kernel below): one CTA per SM walks
// work items (pair, direction, 256-row block) instead of one CTA per item, so barrier initialisation and -- above all -- the
// 64 KB A-slab load of the NEXT item overlap the tiles of the current one (A slabs double buffered, 3-stage ring of B tiles).
// Same arithmetic, same results.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int TCP_NSB = 3;
constexpr size_t TCP_SMEM = 1024 + (size_t)(8 + 2 * TCP_NSB) * TC_BOX_BYTES + 256;

__global__ void __launch_bounds__(MT_THREADS, 1) mnn_tc_persist2_kernel(const __grid_constant__ TcMaps maps,
                                                                       const int* __restrict__ n1p, int n1_max,
                                                                       const int* __restrict__ n2p, int n2_max, int n_pad, int batch,
                                                                       unsigned long long* __restrict__ best12,
                                                                       unsigned long long* __restrict__ best21,
                                                                       const int2* __restrict__ pairs) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sA = base;                       // [buffer 2][slab 2][hi, lo] boxes
  unsigned char* sB = base + 8 * TC_BOX_BYTES;    // [stage TCP_NSB][hi, lo] boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + (8 + 2 * TCP_NSB) * TC_BOX_BYTES);
  uint64_t* a_full = bars;                        // [2]
  uint64_t* a_empty = bars + 2;                   // [2]
  uint64_t* b_full = bars + 4;                    // [TCP_NSB]
  uint64_t* b_empty = b_full + TCP_NSB;           // [TCP_NSB]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RB = n_pad / TC_ROWS;
  const int n_items = batch * 2 * RB;

  if (warp == 8 && lane == 0) {
    tc::tma_prefetch_desc(&maps.m1);
    tc::tma_prefetch_desc(&maps.m2);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&a_full[i], 1);
      tc::mbar_init(&a_empty[i], 8);
    }
    for (int i = 0; i < TCP_NSB; ++i) {
      tc::mbar_init(&b_full[i], 1);
      tc::mbar_init(&b_empty[i], 8);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  // item -> (pair, dir, row block) and the images (ia, ib) of its A and B rows (pairs: see mnn_tc_kernel); every role walks the
  // same sequence and skips the same (empty) items
  auto decode = [&](int item, int& pair, int& dir, int& row0, int& n_rows, int& n_cols, int& ia, int& ib) {
    const int rb = item % RB, pd = item / RB;
    pair = pd >> 1;
    dir = pd & 1;
    row0 = rb * TC_ROWS;
    const int2 ij = pairs ? __ldg(pairs + pair) : make_int2(pair, pair);
    const int n1 = n1p ? min(__ldg(n1p + ij.x), n1_max) : n1_max;
    const int n2 = n2p ? min(__ldg(n2p + ij.y), n2_max) : n2_max;
    n_rows = dir ? n2 : n1;
    n_cols = dir ? n1 : n2;
    ia = dir ? ij.y : ij.x;
    ib = dir ? ij.x : ij.y;
    return row0 < n_rows && n_cols > 0;
  };

  if (warp == 8) {
    if (tc::elect_one()) {
      uint32_t ai = 0, bi = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        int pair, dir, row0, n_rows, n_cols, ia, ib;
        if (!decode(item, pair, dir, row0, n_rows, n_cols, ia, ib)) continue;
        const CUtensorMap* mapA = dir ? &maps.m2 : &maps.m1;
        const CUtensorMap* mapB = dir ? &maps.m1 : &maps.m2;
        const int T = (n_cols + TC_BN - 1) / TC_BN;
        const int ab = ai & 1;
        tc::mbar_wait(&a_empty[ab], ((ai >> 1) & 1) ^ 1);
        tc::mbar_expect_tx(&a_full[ab], 4 * TC_BOX_BYTES);
        const int arow = ia * n_pad + row0;
        for (int slab = 0; slab < 2; ++slab)
          for (int kb = 0; kb < 2; ++kb)
            tc::tma_load_2d(sA + ((ab * 2 + slab) * 2 + kb) * TC_BOX_BYTES, mapA, &a_full[ab], kb * 64, arow + slab * 128);
        ++ai;
        const int brow = ib * n_pad;
        for (int t = 0; t < T; ++t, ++bi) {
          const int s = bi % TCP_NSB;
          tc::mbar_wait(&b_empty[s], ((bi / TCP_NSB) & 1) ^ 1);
          tc::mbar_expect_tx(&b_full[s], 2 * TC_BOX_BYTES);
          for (int kb = 0; kb < 2; ++kb)
            tc::tma_load_2d(sB + (s * 2 + kb) * TC_BOX_BYTES, mapB, &b_full[s], kb * 64, brow + t * TC_BN);
        }
      }
    }
    __syncwarp();
  } else {
    const int slab = warp >> 2, wt = threadIdx.x & 127;
    float acc0[64], acc1[64];
    uint32_t ai = 0, bi = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      int pair, dir, row0, n_rows, n_cols, ia, ib;
      if (!decode(item, pair, dir, row0, n_rows, n_cols, ia, ib)) continue;
      const int T = (n_cols + TC_BN - 1) / TC_BN;
      const int ab = ai & 1;
      tc::mbar_wait(&a_full[ab], (ai >> 1) & 1);
      const uint32_t a_slab = tc::smem_u32(sA + (ab * 2 + slab) * 2 * TC_BOX_BYTES);
      unsigned long long best[4] = {0ull, 0ull, 0ull, 0ull};
      for (int t = 0; t < T; ++t, ++bi) {
        const int s = bi % TCP_NSB;
        tc::mbar_wait(&b_full[s], (bi / TCP_NSB) & 1);
        mnn_tile_mma(acc0, acc1, a_slab, tc::smem_u32(sB + s * 2 * TC_BOX_BYTES), dir);
        __syncwarp();
        if (lane == 0) {
          tc::mbar_arrive(&b_empty[s]);
          if (t == T - 1) tc::mbar_arrive(&a_empty[ab]);   // the A slabs may be overwritten
        }
        mnn_row_argmax(acc0, acc1, t * TC_BN, n_cols - t * TC_BN, lane, best);
      }
      ++ai;
      if ((lane & 3) == 0) {
        unsigned long long* out = dir ? best21 : best12;
        const int out_stride = dir ? n2_max : n1_max;
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int row = row0 + slab * 128 + tc::frag_row(wt, h);
          if (row < n_rows) out[(int64_t)pair * out_stride + row] = best[h];
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Default kernel (implementation 1): S = F1.F2^T is computed ONCE per pair, in the three-term order of mnn_tile_mma(dir = 0),
// and the same accumulator tile yields both arg-maxes.  Persistent CTAs walk items (pair, 256-column block of set 2), pair-major
// so that the CTAs in flight share one pair's set 1 in L2.  The item's two 128-column slabs of set 2 (the B operand) stay
// resident and TMA streams every 128-row A tile of set 1 past them; warpgroup w owns slab w for the whole item.
//
// Ping-pong: the two consumer warpgroups take turns issuing their MMAs on an A tile (named barriers 1 and 2 pass the turn), so
// warpgroup 0 reduces tile t while the tensor pipe runs warpgroup 1's MMAs on t, and warpgroup 1 reduces t while warpgroup 0's
// MMAs on t+1 run.  Each warpgroup commits a tile's MMAs as two groups (rows 0-63, rows 64-127) and starts the epilogue of the
// first half while the tensor cores still run the second.  An A stage is released once all eight consumer warps' MMAs on it
// retired.
//
// Epilogue of one tile, per thread 4 rows x 32 columns (mnn_half_epilogue, once per 64-row half):
//   rows:    maximum of each row over the slab's 128 columns (fp32 maximum over the thread's columns, then the quad of lanes
//            that shares the row) and the first column that holds it; one red.global.max.u64 per row, slab and item merges
//            the packed (value, ~column) into best12.  The packed max is associative and commutative, so the atomic order
//            does not matter and the lowest column wins ties (torch's first-index rule).
//   columns: a running (value, row) per column over all tiles of the item, strict > in ascending row order (tiles ascend,
//            and h = 0..3 is r, r+8, r+64, r+72), so each thread keeps its first row on ties.  Nothing crosses lanes.
// Once per item, the 8 row lanes (shuffles) and the 4 warps (shared memory) combine the column partials as packed (value,
// ~row) maxima.  A column lives in one slab of one item, so best21 is written once, without atomics, in the format and tie
// rule of a row arg-max of S21 that mnn_finalize_kernel reads.
// Rows past n1 (last tile) and columns past n2 (last item) are set to -inf before the reductions.
//
// Shared memory: the B slabs double buffered across items (2 x 64 KB), a 2-stage A ring (2 x 32 KB), the column partials
// [slab][item parity][warp][column] as packed u64 = 16 KB.  A third A stage does not fit beside them (227 KB per block).
// Registers: the accumulator (128) and the column state (64) need more than the 168 per thread that 384 threads leave, so the
// producer is a whole warpgroup (warps 8-11; one lane of warp 8 issues the loads) that hands its registers to the consumers
// with setmaxnreg (40 / 232).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int TCF_THREADS = 384;
constexpr int TCF_NSA = 2;
constexpr size_t TCF_COL_BYTES = 2 * 2 * 4 * 128 * sizeof(unsigned long long);
constexpr size_t TCF_SMEM = 1024 + (size_t)(8 + 2 * TCF_NSA) * TC_BOX_BYTES + 256 + TCF_COL_BYTES;

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// mnn_tile_mma_issue(dir = 0) as two commit groups, rows 0-63 of the A tile (acc0) and then rows 64-127 (acc1), so that
// wgmma_wait<1> hands acc0 to the epilogue while the tensor cores still run acc1.  Every accumulator adds the same products in
// the same order as mnn_tile_mma_issue.
__device__ __forceinline__ void mnn_tile_mma_issue_halves(float (&acc0)[64], float (&acc1)[64], uint32_t a_tile, uint32_t b_slab) {
  tc::wgmma_fence();
#pragma unroll
  for (int half = 0; half < 2; ++half) {
#pragma unroll
    for (int kb = 0; kb < 3; ++kb) {
      const uint64_t da = tc::make_desc_sw128(a_tile + (kb == 2 ? 1 : 0) * TC_BOX_BYTES, 1024) + half * MT_HALF;
      const uint64_t db = tc::make_desc_sw128(b_slab + (kb == 1 ? 1 : 0) * TC_BOX_BYTES, 1024);
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::wgmma_f16<128>(half ? acc1 : acc0, da + 2 * k, db + 2 * k, (kb | k) ? 1u : 0u);
    }
    tc::wgmma_commit();
  }
}

// Epilogue of one 64-row half d of a slab tile (d = acc0: fragment rows h = 0, 1; d = acc1: h = 2, 3, as tc::frag_val): element
// (h, j, e) of the half is d[4j + 2h + e], row row[H0 + h] of the pair, column col0 + 8j + 2(lane%4) + e of set 2.
//   Masking: columns from n_valid on and, in a tile that reaches past n1 (rows_partial), rows from n_rows on become -inf.
//   Rows: the maximum over the slab's 128 columns (thread, then the quad of lanes that shares the row) and the first column
//     that holds it, merged into best12 with red.global.max (a row that is all -inf writes nothing).  Both rows go through
//     each step together and the first-column search runs as four short select chains per row, which keeps independent work
//     in flight: while the tensor cores run MMAs, each scheduler has one warp in this epilogue.
//   Columns: the running (value, row) of column 8j + 2(lane%4) + e is (cv, cr)[2j + e], updated with strict > in ascending row
//     order (H0 = 0 before H0 = 2, tiles ascending), so each thread keeps its first row on ties.
template <int H0>
__device__ __forceinline__ void mnn_half_epilogue(float (&d)[64], const int (&row)[4], int col0, int n_valid, int n_rows,
                                                  bool rows_partial, int lane, unsigned long long* best12, float (&cv)[32], int (&cr)[32]) {
  const int cq = 2 * (lane & 3);
  if (n_valid < TC_BN) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (8 * j + cq + e >= n_valid) d[4 * j + e] = d[4 * j + 2 + e] = -INFINITY;
  }
  if (rows_partial)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (row[H0 + h] >= n_rows)
#pragma unroll
        for (int i = 0; i < 32; ++i) d[4 * (i >> 1) + 2 * h + (i & 1)] = -INFINITY;

  float mx[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float m[8];
#pragma unroll
    for (int q = 0; q < 8; ++q)
      m[q] = fmaxf(fmaxf(d[8 * q + 2 * h], d[8 * q + 2 * h + 1]), fmaxf(d[8 * q + 4 + 2 * h], d[8 * q + 5 + 2 * h]));
    mx[h] = fmaxf(fmaxf(fmaxf(m[0], m[1]), fmaxf(m[2], m[3])), fmaxf(fmaxf(m[4], m[5]), fmaxf(m[6], m[7])));
  }
#pragma unroll
  for (int o = 1; o < 4; o <<= 1)
#pragma unroll
    for (int h = 0; h < 2; ++h) mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], o));
  int c[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int cs[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {   // columns 32g .. 32g+31 of the tile, first equal one
      cs[g] = 1 << 30;
#pragma unroll
      for (int j = 4 * g + 3; j >= 4 * g; --j)
#pragma unroll
        for (int e = 1; e >= 0; --e) cs[g] = (d[4 * j + 2 * h + e] == mx[h]) ? 8 * j + e : cs[g];
    }
    c[h] = min(min(cs[0], cs[1]), min(cs[2], cs[3])) + cq;
  }
#pragma unroll
  for (int o = 1; o < 4; o <<= 1)
#pragma unroll
    for (int h = 0; h < 2; ++h) c[h] = min(c[h], __shfl_xor_sync(0xffffffffu, c[h], o));

#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float v0 = d[4 * j + e], v1 = d[4 * j + 2 + e];
      const float m = v1 > v0 ? v1 : v0;
      const int r = v1 > v0 ? row[H0 + 1] : row[H0];
      if (m > cv[2 * j + e]) { cv[2 * j + e] = m; cr[2 * j + e] = r; }
    }

  if ((lane & 3) == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (mx[h] != -INFINITY) atomicMax(best12 + row[H0 + h], pack_vi(mx[h], (uint32_t)(col0 + c[h])));
  }
}

__global__ void __launch_bounds__(TCF_THREADS, 1) mnn_tc_persist_kernel(const __grid_constant__ TcMaps maps,
                                                                       const int* __restrict__ n1p, int n1_max,
                                                                       const int* __restrict__ n2p, int n2_max, int n_pad, int batch,
                                                                       unsigned long long* __restrict__ best12,
                                                                       unsigned long long* __restrict__ best21,
                                                                       const int2* __restrict__ pairs) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sB = base;                       // [buffer 2][slab 2][hi, lo] boxes
  unsigned char* sA = base + 8 * TC_BOX_BYTES;    // [stage TCF_NSA][hi, lo] boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + (8 + 2 * TCF_NSA) * TC_BOX_BYTES);
  uint64_t* b_full = bars;                        // [2]
  uint64_t* b_empty = bars + 2;                   // [2]
  uint64_t* a_full = bars + 4;                    // [TCF_NSA]
  uint64_t* a_empty = a_full + TCF_NSA;           // [TCF_NSA]
  unsigned long long* sCol =
      reinterpret_cast<unsigned long long*>(base + (8 + 2 * TCF_NSA) * TC_BOX_BYTES + 256);   // [slab 2][parity 2][warp 4][128]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int CB = n_pad / TC_ROWS;   // 256-column blocks per pair
  const int n_items = batch * CB;

  if (warp == 8 && lane == 0) {
    tc::tma_prefetch_desc(&maps.m1);
    tc::tma_prefetch_desc(&maps.m2);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&b_full[i], 1);
      tc::mbar_init(&b_empty[i], 8);
    }
    for (int i = 0; i < TCF_NSA; ++i) {
      tc::mbar_init(&a_full[i], 1);
      tc::mbar_init(&a_empty[i], 8);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  // item -> (pair, column block) and the images (ia, ib) of its A and B rows (pairs: see mnn_tc_kernel); every role walks the
  // same sequence and skips the same (empty) items
  auto decode = [&](int item, int& pair, int& col0, int& n_rows, int& n_cols, int& ia, int& ib) {
    pair = item / CB;
    col0 = (item - pair * CB) * TC_ROWS;
    const int2 ij = pairs ? __ldg(pairs + pair) : make_int2(pair, pair);
    ia = ij.x;
    ib = ij.y;
    n_rows = n1p ? min(__ldg(n1p + ia), n1_max) : n1_max;
    n_cols = n2p ? min(__ldg(n2p + ib), n2_max) : n2_max;
    return col0 < n_cols && n_rows > 0;
  };

  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8 && tc::elect_one()) {
      uint32_t bi = 0, ai = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        int pair, col0, n_rows, n_cols, ia, ib;
        if (!decode(item, pair, col0, n_rows, n_cols, ia, ib)) continue;
        const int T = (n_rows + TC_BN - 1) / TC_BN;
        const int bb = bi & 1;
        tc::mbar_wait(&b_empty[bb], ((bi >> 1) & 1) ^ 1);
        tc::mbar_expect_tx(&b_full[bb], 4 * TC_BOX_BYTES);
        const int brow = ib * n_pad + col0;
        for (int slab = 0; slab < 2; ++slab)
          for (int kb = 0; kb < 2; ++kb)
            tc::tma_load_2d(sB + ((bb * 2 + slab) * 2 + kb) * TC_BOX_BYTES, &maps.m2, &b_full[bb], kb * 64, brow + slab * 128);
        ++bi;
        const int arow = ia * n_pad;
        for (int t = 0; t < T; ++t, ++ai) {
          const int s = ai % TCF_NSA;
          tc::mbar_wait(&a_empty[s], ((ai / TCF_NSA) & 1) ^ 1);
          tc::mbar_expect_tx(&a_full[s], 2 * TC_BOX_BYTES);
          for (int kb = 0; kb < 2; ++kb)
            tc::tma_load_2d(sA + (s * 2 + kb) * TC_BOX_BYTES, &maps.m1, &a_full[s], kb * 64, arow + t * TC_BN);
        }
      }
    }
    __syncwarp();
  } else {
    const int slab = warp >> 2, wt = threadIdx.x & 127, cq = 2 * (lane & 3);
    const int my_turn = 1 + slab, next_turn = 2 - slab;   // named barriers: warpgroup 0 issues on 1, warpgroup 1 on 2
    setmaxnreg_inc<232>();
    float acc0[64], acc1[64];
    float cv[32];
    int cr[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      cv[i] = -INFINITY;
      cr[i] = 0;
    }
    uint32_t bi = 0, ai = 0;
    if (slab == 1) named_arrive(1, 256);   // warpgroup 0 goes first
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      int pair, col0, n_rows, n_cols, ia, ib;
      if (!decode(item, pair, col0, n_rows, n_cols, ia, ib)) continue;
      const int T = (n_rows + TC_BN - 1) / TC_BN;
      const int bb = bi & 1;
      const int scol0 = col0 + slab * TC_BN, n_valid = n_cols - scol0;   // n_valid <= 0: the whole slab lies past n2
      unsigned long long* b12 = best12 + (int64_t)pair * n1_max;
      tc::mbar_wait(&b_full[bb], (bi >> 1) & 1);
      const uint32_t b_slab = tc::smem_u32(sB + (bb * 2 + slab) * 2 * TC_BOX_BYTES);
      for (int t = 0; t < T; ++t, ++ai) {
        const int s = ai % TCF_NSA;
        tc::mbar_wait(&a_full[s], (ai / TCF_NSA) & 1);
        named_sync(my_turn, 256);
        mnn_tile_mma_issue_halves(acc0, acc1, tc::smem_u32(sA + s * 2 * TC_BOX_BYTES), b_slab);
        named_arrive(next_turn, 256);
        int row[4];
#pragma unroll
        for (int h = 0; h < 4; ++h) row[h] = t * TC_BN + tc::frag_row(wt, h);
        const bool rows_partial = (t + 1) * TC_BN > n_rows;
        tc::wgmma_wait<1>();   // rows 0-63 of the tile are in acc0; rows 64-127 are still being computed
        tc::acc_fence(acc0);
        mnn_half_epilogue<0>(acc0, row, scol0, n_valid, n_rows, rows_partial, lane, b12, cv, cr);
        tc::wgmma_wait<0>();
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) {
          tc::mbar_arrive(&a_empty[s]);
          if (t == T - 1) tc::mbar_arrive(&b_empty[bb]);   // the B slabs may be overwritten
        }
        mnn_half_epilogue<2>(acc1, row, scol0, n_valid, n_rows, rows_partial, lane, b12, cv, cr);
      }
      // the item's column partials: the 8 row lanes of a column, then the 4 warps; parity bi & 1 is written again two items on
      unsigned long long* sc = sCol + (slab * 2 + bb) * 4 * 128;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          unsigned long long p = cv[2 * j + e] != -INFINITY ? pack_vi(cv[2 * j + e], (uint32_t)cr[2 * j + e]) : 0ull;
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            const unsigned long long q = __shfl_xor_sync(0xffffffffu, p, o);
            p = q > p ? q : p;
          }
          if (lane < 4) sc[(wt >> 5) * 128 + 8 * j + cq + e] = p;
          cv[2 * j + e] = -INFINITY;
        }
      ++bi;
      tc::wg_sync(3 + slab);
      if (wt < n_valid) {
        unsigned long long p = sc[wt];
#pragma unroll
        for (int w = 1; w < 4; ++w) {
          const unsigned long long q = sc[w * 128 + wt];
          p = q > p ? q : p;
        }
        best21[(int64_t)pair * n2_max + scol0 + wt] = p;
      }
    }
    if (slab == 0) named_sync(1, 256);   // warpgroup 1's last hand-over
  }
}

// The three-term scan of both directions over the full sets.  variant 0 (implementation 1, default): the single-GEMM persistent
// kernel; 1 (implementation 2): the persistent kernel with one GEMM per direction; 2 (implementation 3) or XFEAT_MNN_ONESHOT=1:
// one CTA per (row block, pair, direction).  pairs: optional (image i, image j) table (see mnn_tc_kernel).
static int launch_mnn_tc_main(const TcMaps& maps, const int* n1, int n1_max, const int* n2, int n2_max, int n_pad, int batch,
                              unsigned long long* best12, unsigned long long* best21, cudaStream_t st, int variant,
                              const int2* pairs = nullptr) {
  static const bool oneshot_env = getenv("XFEAT_MNN_ONESHOT") != nullptr;
  if (variant == 2 || oneshot_env) {
    XF_DYN_SMEM(mnn_tc_kernel, TC_SMEM);
    dim3 grid(n_pad / TC_ROWS, batch, 2);
    TcMaps4 m4;
    m4.a0 = maps.m1; m4.b0 = maps.m2; m4.a1 = maps.m2; m4.b1 = maps.m1;
    mnn_tc_kernel<<<grid, MT_THREADS, TC_SMEM, st>>>(m4, n1, n1_max, n2, n2_max, n_pad, best12, best21, nullptr, nullptr, pairs);
    XF_LAUNCH_CHECK();
    return XF_OK;
  }
  int dev = 0, sms = 148;
  XF_CUDA(cudaGetDevice(&dev));
  XF_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (variant == 1) {
    XF_DYN_SMEM(mnn_tc_persist2_kernel, TCP_SMEM);
    const int n_items = batch * 2 * (n_pad / TC_ROWS);
    mnn_tc_persist2_kernel<<<n_items < sms ? n_items : sms, MT_THREADS, TCP_SMEM, st>>>(maps, n1, n1_max, n2, n2_max, n_pad, batch,
                                                                                       best12, best21, pairs);
  } else {
    XF_DYN_SMEM(mnn_tc_persist_kernel, TCF_SMEM);
    const int n_items = batch * (n_pad / TC_ROWS);
    mnn_tc_persist_kernel<<<n_items < sms ? n_items : sms, TCF_THREADS, TCF_SMEM, st>>>(maps, n1, n1_max, n2, n2_max, n_pad, batch,
                                                                                      best12, best21, pairs);
  }
  XF_LAUNCH_CHECK();
  return XF_OK;
}

struct MnnTcWs {
  __half *f1s, *f2s;
  unsigned long long *best12, *best21;
  unsigned* absmax;
  float* inv_s2;
};
static inline int tc_pad(int n) { return (n + 2 * TC_ROWS - 1) / (2 * TC_ROWS) * (2 * TC_ROWS); }   // 512 rows (operand layout of the API)

void carve_mnn_tc(Bump& bump, int batch, int n1_max, int n2_max, MnnTcWs& ws) {
  const int n_pad = tc_pad(n1_max > n2_max ? n1_max : n2_max);
  ws.f1s = bump.take<__half>((size_t)batch * n_pad * TC_KP);
  ws.f2s = bump.take<__half>((size_t)batch * n_pad * TC_KP);
  ws.best12 = bump.take<unsigned long long>((size_t)batch * n1_max);
  ws.best21 = bump.take<unsigned long long>((size_t)batch * n2_max);
  ws.absmax = bump.take<unsigned>(1);
  ws.inv_s2 = bump.take<float>(1);
}

size_t mnn_tc_workspace_bytes(int batch, int n1_max, int n2_max) {
  Bump bump(nullptr, 0);
  MnnTcWs ws;
  carve_mnn_tc(bump, batch, n1_max, n2_max, ws);
  return bump.used();
}

static int make_map(CUtensorMap* m, const __half* ptr, uint64_t rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)TC_KP, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)TC_KP * sizeof(__half)};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return XF_E_CUDA;
  }
  return XF_OK;
}

// Fills best12 (rows of F1 -> arg-max column in F2) and best21 (rows of F2 -> arg-max in F1), packed (value*s^2, index).
int launch_mnn_tc(const float* f1, const int* n1, int n1_max, int64_t stride1, const float* f2, const int* n2, int n2_max,
                  int64_t stride2, int batch, void* d_ws, size_t ws_bytes, unsigned long long** best12,
                  unsigned long long** best21, float** inv_s2, cudaStream_t st, int variant, float abs_bound) {
  Bump bump(d_ws, ws_bytes);
  MnnTcWs ws;
  carve_mnn_tc(bump, batch, n1_max, n2_max, ws);
  if (!bump.ok) {
    set_error("mnn_match(tensor cores): workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  const int n_pad = tc_pad(n1_max > n2_max ? n1_max : n2_max);
  XF_REQUIRE((int64_t)batch * n_pad < (1ll << 31), "mnn_match(tensor cores): batch * n too large");
  if (!(abs_bound > 0.f)) {   // no bound from the caller: max |x| over both sets fixes the power-of-two operand scale
    XF_CUDA(cudaMemsetAsync(ws.absmax, 0, sizeof(unsigned), st));
    absmax_kernel<<<dim3(8, batch), 256, 0, st>>>(f1, n1, n1_max, stride1, ws.absmax);
    XF_LAUNCH_CHECK();
    absmax_kernel<<<dim3(8, batch), 256, 0, st>>>(f2, n2, n2_max, stride2, ws.absmax);
    XF_LAUNCH_CHECK();
  }
  const dim3 sgrid(cdiv(n_pad * 32, 256), batch);
  split_kernel<<<sgrid, 256, 0, st>>>(f1, n1, n1_max, n_pad, stride1, ws.absmax, abs_bound, ws.f1s, ws.inv_s2);
  XF_LAUNCH_CHECK();
  split_kernel<<<sgrid, 256, 0, st>>>(f2, n2, n2_max, n_pad, stride2, ws.absmax, abs_bound, ws.f2s, nullptr);
  XF_LAUNCH_CHECK();
  TcMaps maps;
  int rc;
  if ((rc = make_map(&maps.m1, ws.f1s, (uint64_t)batch * n_pad))) return rc;
  if ((rc = make_map(&maps.m2, ws.f2s, (uint64_t)batch * n_pad))) return rc;
  XF_CUDA(cudaMemsetAsync(ws.best12, 0, sizeof(unsigned long long) * (size_t)batch * n1_max, st));
  *inv_s2 = ws.inv_s2;
  *best12 = ws.best12;
  *best21 = ws.best21;
  XF_CUDA(cudaMemsetAsync(ws.best21, 0, sizeof(unsigned long long) * (size_t)batch * n2_max, st));
  return launch_mnn_tc_main(maps, n1, n1_max, n2, n2_max, n_pad, batch, ws.best12, ws.best21, st, variant);
}

int launch_mnn_tc_rows(const __half* a0, const __half* b0, const __half* a1, const __half* b1, const int* n1, int n1_max,
                       const int* n2, int n2_max, int n_pad, int batch, const int* rows_cnt, const int* row_map,
                       unsigned long long* best12, unsigned long long* best21, cudaStream_t st);
__global__ void set_scalar_kernel(float* p, float v) { *p = v; }

// Operands already split by the producer (xfeat_detect_sparse_split): (batch * n_pad) rows x 128 halves each, scaled by 2^scale_log2.
// pairs != NULL: f1s == f2s is one table of n_images images (n_images * n_pad rows) and pair p matches the images pairs[p] = (i, j)
// of it (the counts n1[i], n2[j]); batch is the number of pairs.
int launch_mnn_tc_presplit(const __half* f1s, const int* n1, int n1_max, const __half* f2s, const int* n2, int n2_max, int n_pad,
                           int batch, int scale_log2, void* d_ws, size_t ws_bytes, unsigned long long** best12,
                           unsigned long long** best21, float** inv_s2, cudaStream_t st, int variant,
                           const int2* pairs, int n_images) {
  XF_REQUIRE(n_pad % (2 * TC_ROWS) == 0 && n_pad >= n1_max && n_pad >= n2_max, "mnn_match_presplit: n_pad must be a multiple of %d covering both sets", 2 * TC_ROWS);
  const int64_t table_rows = (int64_t)(pairs ? n_images : batch) * n_pad;
  XF_REQUIRE(table_rows < (1ll << 31), "mnn_match_presplit: batch * n too large");
  Bump bump(d_ws, ws_bytes);
  unsigned long long* b12 = bump.take<unsigned long long>((size_t)batch * n1_max);
  unsigned long long* b21 = bump.take<unsigned long long>((size_t)batch * n2_max);
  float* scale = bump.take<float>(1);
  if (!bump.ok) {
    set_error("mnn_match_presplit: workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  XF_CUDA(cudaMemsetAsync(b12, 0, sizeof(unsigned long long) * (size_t)batch * n1_max, st));
  XF_CUDA(cudaMemsetAsync(b21, 0, sizeof(unsigned long long) * (size_t)batch * n2_max, st));
  set_scalar_kernel<<<1, 1, 0, st>>>(scale, ldexpf(1.f, -2 * scale_log2));
  XF_LAUNCH_CHECK();
  *best12 = b12; *best21 = b21; *inv_s2 = scale;
  TcMaps maps;
  int rc;
  if ((rc = make_map(&maps.m1, f1s, (uint64_t)table_rows))) return rc;
  if ((rc = make_map(&maps.m2, f2s, (uint64_t)table_rows))) return rc;
  return launch_mnn_tc_main(maps, n1, n1_max, n2, n2_max, n_pad, batch, b12, b21, st, variant, pairs);
}

// Pair lists over one fp32 image table (xfeat_mnn_match_pairs_f32): f (n_images, n_max, 64), n (n_images) counts.  Pair p is
// split at the exponent of its own maximum -- max |x| over its two images, the one launch_mnn_tc measures for that pair alone --
// into per-pair operand blocks (A rows at p * n_pad of one array, B rows at p * n_pad of the other, with per-pair counts) that
// the presplit kernels match as they stand.  One exponent per image or per table would change the lo terms (and the tiny hi
// terms) that round into fp16 subnormals, hence S in its last bits, hence near-tie arg-maxes.
struct MnnPairsWs {
  __half* ops;
  unsigned* absmax;
  int* cnt;
};
static void carve_mnn_pairs(Bump& bump, int n_pairs, int n_max, MnnPairsWs& ws) {
  ws.ops = bump.take<__half>((size_t)2 * n_pairs * tc_pad(n_max) * TC_KP);
  ws.absmax = bump.take<unsigned>(n_pairs);
  ws.cnt = bump.take<int>((size_t)2 * n_pairs);
  bump.take<unsigned long long>((size_t)n_pairs * n_max);   // the presplit launch's best12 / best21 / scale, carved by it
  bump.take<unsigned long long>((size_t)n_pairs * n_max);
  bump.take<float>(1);
}

size_t mnn_tc_pairs_workspace_bytes(int n_pairs, int n_max) {
  Bump bump(nullptr, 0);
  MnnPairsWs ws;
  carve_mnn_pairs(bump, n_pairs, n_max, ws);
  return bump.used();
}

int launch_mnn_tc_pairs_f32(const float* f, const int* n, int n_max, const int2* pairs, int n_pairs, void* d_ws, size_t ws_bytes,
                            unsigned long long** best12, unsigned long long** best21, float** inv_s2, const int** cnt1,
                            const int** cnt2, cudaStream_t st, int variant) {
  const int n_pad = tc_pad(n_max);
  XF_REQUIRE((int64_t)n_pairs * n_pad < (1ll << 31), "mnn_match_pairs_f32: n_pairs * n too large");
  Bump bump(d_ws, ws_bytes);
  MnnPairsWs ws;
  carve_mnn_pairs(bump, n_pairs, n_max, ws);
  if (!bump.ok) {
    set_error("mnn_match_pairs_f32: workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  const int64_t stride = (int64_t)n_max * 64;
  XF_CUDA(cudaMemsetAsync(ws.absmax, 0, sizeof(unsigned) * (size_t)n_pairs, st));
  absmax_kernel<true><<<dim3(8, n_pairs, 2), 256, 0, st>>>(f, n, n_max, stride, ws.absmax, pairs);
  XF_LAUNCH_CHECK();
  split_kernel<true><<<dim3(cdiv(n_pad * 32, 256), n_pairs, 2), 256, 0, st>>>(f, n, n_max, n_pad, stride, ws.absmax, 0.f, ws.ops,
                                                                              nullptr, pairs, ws.cnt);
  XF_LAUNCH_CHECK();
  *cnt1 = ws.cnt;
  *cnt2 = ws.cnt + n_pairs;
  const size_t head = (size_t)((char*)(ws.cnt + 2 * (size_t)n_pairs) - (char*)d_ws);
  const size_t off = (head + 255) / 256 * 256;   // the rest of the workspace: what carve_mnn_pairs reserved for this launch
  // scale_log2 only feeds the min_cossim test, which this path does not run
  return launch_mnn_tc_presplit(ws.ops, ws.cnt, n_max, ws.ops + (size_t)n_pairs * n_pad * TC_KP, ws.cnt + n_pairs, n_max, n_pad,
                                n_pairs, 0, (char*)d_ws + off, ws_bytes - off, best12, best21, inv_s2, st, variant, nullptr, 0);
}

int launch_absmax(const float* f, const int* np, int n_max, int64_t stride, int batch, unsigned* out, cudaStream_t st) {
  absmax_kernel<<<dim3(8, batch), 256, 0, st>>>(f, np, n_max, stride, out);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// The three-term kernel on explicit operand arrays (all (batch * n_pad) x 128 halves): direction d scans the first
// rows_cnt[pair][d] rows of a<d> against set (d ? 1 : 2) in b<d> and writes row r's result at row_map[pair][d][r].
int launch_mnn_tc_rows(const __half* a0, const __half* b0, const __half* a1, const __half* b1, const int* n1, int n1_max,
                       const int* n2, int n2_max, int n_pad, int batch, const int* rows_cnt, const int* row_map,
                       unsigned long long* best12, unsigned long long* best21, cudaStream_t st) {
  XF_REQUIRE(n_pad % (2 * TC_ROWS) == 0, "mnn_tc_rows: n_pad must be a multiple of %d", 2 * TC_ROWS);
  TcMaps4 m4;
  int rc;
  if ((rc = make_map(&m4.a0, a0, (uint64_t)batch * n_pad))) return rc;
  if ((rc = make_map(&m4.b0, b0, (uint64_t)batch * n_pad))) return rc;
  if ((rc = make_map(&m4.a1, a1, (uint64_t)batch * n_pad))) return rc;
  if ((rc = make_map(&m4.b1, b1, (uint64_t)batch * n_pad))) return rc;
  XF_DYN_SMEM(mnn_tc_kernel, TC_SMEM);
  dim3 grid(n_pad / TC_ROWS, batch, 2);
  mnn_tc_kernel<<<grid, MT_THREADS, TC_SMEM, st>>>(m4, n1, n1_max, n2, n2_max, n_pad, best12, best21, rows_cnt, row_map, nullptr);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf
