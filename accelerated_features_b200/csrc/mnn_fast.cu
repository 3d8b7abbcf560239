// Mutual-NN scan, "filter + exact re-score" formulation (xfeat_set_mnn_impl(4); see mnn.cu for why it is not the default).
//
// mnn_tc_kernel (mnn_tc.cu) computes every similarity in fp32-equivalent precision: three fp16 GEMM passes per direction,
// 6x the MACs of one similarity matrix.  Almost none of that precision decides anything: a row's arg-max only needs it when
// the runner-up is within rounding distance.  Here (SURVEY 7.2):
//   pass 1  mnn_fast_kernel: ONE fp16 pass per direction, S~ = hi1 . hi2^T (fp32 accumulate), tracking per row the maximum,
//           its column and the SECOND largest value.  |S~ - S| <= ||hi1|| ||lo2|| + ||lo1|| ||hi2|| (Cauchy-Schwarz on the two
//           dropped split terms), so with tau_i = 2 (||hi_i|| Lmax + ||lo_i|| Hmax) + accumulation slack, a row whose
//           top-1 / top-2 gap exceeds tau_i has the SAME arg-max in exact arithmetic: done.  Rows that fail the test (a few
//           per cent) are appended, with their split operand row, to a compact per-(pair, direction) list.
//   pass 2  mnn_tc_kernel on the compact lists only: the 3-term split against ALL columns, i.e. exactly the value order and
//           tie rule of the full kernel, scattered over the pass-1 result.
// The result is identical to implementation 1 (the test-suite runs both), at ~1/3 of the tensor work.
//
// Pass-1 kernel: persistent CTAs (one per SM) over work items (pair, direction, 256-row block); warp 8 = TMA producer (A
// slabs double buffered across items, 6-stage ring of 128-column B tiles, hi boxes only), warps 0-7 = two consumer warpgroups,
// one per 128-row slab: wgmma 64 x 128 x 16 into registers, then per row the maximum, its first column and the runner-up
// value, reduced in-thread and across the four lanes of a row (mnn_tc.cu describes the fragment layout).
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

constexpr int MF_ROWS = 256, MF_BN = 128, MF_KP = 128, MF_BOX = 128 * 128;   // hi box: 128 rows x 64 halves
constexpr int MF_NSB = 6;                                                      // B tile ring depth
constexpr int MF_THREADS = 288;                                              // warps 0-7: two consumer warpgroups, warp 8: TMA
constexpr size_t MF_SMEM = 1024 + (size_t)(4 + MF_NSB) * MF_BOX + 512;

// One warp per row: split row [hi(64) | lo(64)] (as split_kernel in mnn_tc.cu) plus the row's ||hi||, ||lo|| (in scaled
// units) and the per-(pair) maxima of both over the set, as float bits (non-negative floats order like unsigned ints).
__global__ void __launch_bounds__(256) split_norm_kernel(const float* __restrict__ f, const int* __restrict__ np, int n_max,
                                                         int n_pad, int64_t stride, const unsigned* __restrict__ absmax,
                                                         float abs_bound, __half* __restrict__ out, float2* __restrict__ norms,
                                                         unsigned* __restrict__ maxn /* [pair][2] */, float* __restrict__ inv_s2) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int pair = blockIdx.y;
  // grid.x * 8 warps == n_pad exactly (n_pad is a multiple of 512): no warp leaves before the block barrier below
  const int n = np ? min(np[pair], n_max) : n_max;
  const float mx = abs_bound > 0.f ? abs_bound : __uint_as_float(*absmax);
  int e = 0;
  if (mx > 0.f) frexpf(mx, &e);
  const float s = (mx > 0.f) ? ldexpf(1.f, 14 - e) : 1.f;   // mx * s in [2^13, 2^14)
  if (wid == 0 && lane == 0 && pair == 0 && inv_s2) *inv_s2 = (mx > 0.f) ? ldexpf(1.f, 2 * (e - 14)) : 1.f;
  __half2 hi = __floats2half2_rn(0.f, 0.f), lo = hi;
  float sh = 0.f, sl = 0.f;
  if (wid < n) {
    const float2 v = __ldg(reinterpret_cast<const float2*>(f + (int64_t)pair * stride + wid * 64) + lane);
    const float x0 = v.x * s, x1 = v.y * s;
    hi = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(hi);
    // what the exact kernel uses as "lo" is the fp16 rounding of the remainder; the bound needs the remainder pass 2 sees, plus
    // what pass 2 itself drops is irrelevant (pass 2 IS the reference arithmetic)
    lo = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    const float2 lf = __half22float2(lo);
    sh = hf.x * hf.x + hf.y * hf.y;
    sl = lf.x * lf.x + lf.y * lf.y;
  }
  __half2* o = reinterpret_cast<__half2*>(out + ((int64_t)pair * n_pad + wid) * MF_KP);
  o[lane] = hi;
  o[32 + lane] = lo;
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    sh += __shfl_xor_sync(0xffffffffu, sh, k);
    sl += __shfl_xor_sync(0xffffffffu, sl, k);
  }
  __shared__ float s_nh[8], s_nl[8];
  float nh = 0.f, nl = 0.f;
  if (lane == 0) {
    // round the norms UP a little: they bound an error, sqrt/add rounding must not shrink them
    nh = sqrtf(sh) * 1.0001f;
    nl = sqrtf(sl) * 1.0001f;
    norms[(int64_t)pair * n_pad + wid] = make_float2(nh, nl);
    s_nh[threadIdx.x >> 5] = (wid < n) ? nh : 0.f;
    s_nl[threadIdx.x >> 5] = (wid < n) ? nl : 0.f;
  }
  __syncthreads();     // every warp of the block reaches this point (rows past n_pad returned above only in the last block: see launch)
  if (threadIdx.x == 0) {
    float mh = 0.f, ml = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { mh = fmaxf(mh, s_nh[i]); ml = fmaxf(ml, s_nl[i]); }
    // one atomic per block, and only when it can raise the maximum (4k warps hammering two words per pair cost 300 us)
    if (__float_as_uint(mh) > *reinterpret_cast<volatile unsigned*>(&maxn[pair * 2 + 0])) atomicMax(&maxn[pair * 2 + 0], __float_as_uint(mh));
    if (__float_as_uint(ml) > *reinterpret_cast<volatile unsigned*>(&maxn[pair * 2 + 1])) atomicMax(&maxn[pair * 2 + 1], __float_as_uint(ml));
  }
}

struct MfParams {
  CUtensorMap m1, m2;                 // split operand arrays of set 1 / set 2: (batch * n_pad) rows x 128 halves
  const int *n1p, *n2p;
  int n1_max, n2_max, n_pad, batch;
  const __half *f1s, *f2s;            // the same arrays, for the compact copy of ambiguous rows
  const float2 *norms1, *norms2;      // (batch * n_pad) x (||hi||, ||lo||)
  const unsigned *maxn1, *maxn2;      // [pair][2] maxima of the above over the set
  unsigned long long *best12, *best21;
  int* amb_cnt;                       // [pair][dir]
  int* amb_idx;                       // [pair][dir][n_pad] source row of compact row r
  __half *amb_rows0, *amb_rows1;      // compact operand rows per direction: (batch * n_pad) x 128 halves
};

__global__ void __launch_bounds__(MF_THREADS, 1) mnn_fast_kernel(const __grid_constant__ MfParams P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sA = base;                       // [buffer 2][slab 2] hi boxes
  unsigned char* sB = base + 4 * MF_BOX;          // [MF_NSB] hi boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + (4 + MF_NSB) * MF_BOX);
  uint64_t* a_full = bars;                        // [2]
  uint64_t* a_empty = bars + 2;                   // [2]
  uint64_t* b_full = bars + 4;                    // [MF_NSB]
  uint64_t* b_empty = b_full + MF_NSB;            // [MF_NSB]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RB = P.n_pad / MF_ROWS;
  const int n_items = P.batch * 2 * RB;

  if (warp == 8 && lane == 0) {
    tc::tma_prefetch_desc(&P.m1);
    tc::tma_prefetch_desc(&P.m2);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&a_full[i], 1);
      tc::mbar_init(&a_empty[i], 8);
    }
    for (int i = 0; i < MF_NSB; ++i) {
      tc::mbar_init(&b_full[i], 1);
      tc::mbar_init(&b_empty[i], 8);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  // item -> (pair, dir, row block); every role walks the same sequence and skips the same (empty) items
  auto decode = [&](int item, int& pair, int& dir, int& row0, int& n_rows, int& n_cols) {
    const int rb = item % RB, pd = item / RB;
    pair = pd >> 1;
    dir = pd & 1;
    row0 = rb * MF_ROWS;
    const int n1 = P.n1p ? min(__ldg(P.n1p + pair), P.n1_max) : P.n1_max;
    const int n2 = P.n2p ? min(__ldg(P.n2p + pair), P.n2_max) : P.n2_max;
    n_rows = dir ? n2 : n1;
    n_cols = dir ? n1 : n2;
    return row0 < n_rows && n_cols > 0;
  };

  if (warp == 8) {
    if (tc::elect_one()) {
      // ---------------- TMA producer ----------------
      uint32_t ai = 0, bi = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        int pair, dir, row0, n_rows, n_cols;
        if (!decode(item, pair, dir, row0, n_rows, n_cols)) continue;
        const CUtensorMap* mapA = dir ? &P.m2 : &P.m1;
        const CUtensorMap* mapB = dir ? &P.m1 : &P.m2;
        const int T = (n_cols + MF_BN - 1) / MF_BN;
        const int ab = ai & 1;
        tc::mbar_wait(&a_empty[ab], ((ai >> 1) & 1) ^ 1);
        tc::mbar_expect_tx(&a_full[ab], 2 * MF_BOX);
        const int arow = pair * P.n_pad + row0;
        tc::tma_load_2d(sA + (ab * 2 + 0) * MF_BOX, mapA, &a_full[ab], 0, arow);
        tc::tma_load_2d(sA + (ab * 2 + 1) * MF_BOX, mapA, &a_full[ab], 0, arow + 128);
        ++ai;
        const int brow = pair * P.n_pad;
        for (int t = 0; t < T; ++t, ++bi) {
          const int s = bi % MF_NSB;
          tc::mbar_wait(&b_empty[s], ((bi / MF_NSB) & 1) ^ 1);
          tc::mbar_expect_tx(&b_full[s], MF_BOX);
          tc::tma_load_2d(sB + s * MF_BOX, mapB, &b_full[s], 0, brow + t * MF_BN);
        }
      }
    }
    __syncwarp();
  } else {
    // ---------------- consumer warpgroup `slab`: hi.hi^T tile + per-row top-1 (value, first column) and top-2 value ----------------
    const int slab = warp >> 2, wt = threadIdx.x & 127;
    const int cq = 2 * (lane & 3);
    constexpr uint32_t HALF = (64 * 128) >> 4;
    float acc0[64], acc1[64];
    uint32_t ai = 0, bi = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      int pair, dir, row0, n_rows, n_cols;
      if (!decode(item, pair, dir, row0, n_rows, n_cols)) continue;
      const int T = (n_cols + MF_BN - 1) / MF_BN;
      const int ab = ai & 1;
      tc::mbar_wait(&a_full[ab], (ai >> 1) & 1);
      const uint64_t da = tc::make_desc_sw128(tc::smem_u32(sA + (ab * 2 + slab) * MF_BOX), 1024);
      float best[4], sec[4];
      int col[4];
#pragma unroll
      for (int h = 0; h < 4; ++h) { best[h] = -INFINITY; sec[h] = -INFINITY; col[h] = 0; }
      for (int t = 0; t < T; ++t, ++bi) {
        const int s = bi % MF_NSB;
        tc::mbar_wait(&b_full[s], (bi / MF_NSB) & 1);
        const uint64_t db = tc::make_desc_sw128(tc::smem_u32(sB + s * MF_BOX), 1024);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<128>(acc0, da + 2 * k, db + 2 * k, k ? 1u : 0u);
          tc::wgmma_f16<128>(acc1, da + HALF + 2 * k, db + 2 * k, k ? 1u : 0u);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) {
          tc::mbar_arrive(&b_empty[s]);
          if (t == T - 1) tc::mbar_arrive(&a_empty[ab]);
        }
        const int cb = t * MF_BN, nv = n_cols - cb;
#pragma unroll
        for (int h = 0; h < 4; ++h)
#pragma unroll
          for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + cq + e;
              const float v = (c < nv) ? tc::frag_val(acc0, acc1, h, j, e) : -INFINITY;
              // columns ascending: a strictly larger value takes over (the old maximum becomes the runner-up), an equal one
              // leaves the first column and makes the runner-up equal to the maximum (an ambiguous row)
              sec[h] = fmaxf(sec[h], fminf(v, best[h]));
              if (v > best[h]) { best[h] = v; col[h] = cb + c; }
            }
      }
      ++ai;
      // merge the four lanes of every row: exact top-1 (lowest column on ties) and top-2 of the union
#pragma unroll
      for (int h = 0; h < 4; ++h)
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best[h], o), os = __shfl_xor_sync(0xffffffffu, sec[h], o);
          const int oc = __shfl_xor_sync(0xffffffffu, col[h], o);
          const float nsec = fmaxf(fmaxf(sec[h], os), fminf(best[h], ob));
          if (ob > best[h] || (ob == best[h] && oc < col[h])) { best[h] = ob; col[h] = oc; }
          sec[h] = nsec;
        }
      const float2* norms = dir ? P.norms2 : P.norms1;
      const unsigned* mo = (dir ? P.maxn1 : P.maxn2) + pair * 2;            // the OTHER set's maxima
      const float Hmax = __uint_as_float(__ldg(mo)), Lmax = __uint_as_float(__ldg(mo + 1));
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int row = row0 + slab * 128 + tc::frag_row(wt, h);
        const bool live = (lane & 3) == 0 && row < n_rows;
        bool amb = false;
        if (live) {
          const float2 nr = __ldg(norms + (int64_t)pair * P.n_pad + row);
          // |S~ - S| <= ||hi_i|| Lmax + ||lo_i|| Hmax for every column; both the best and a competitor may be off by that much;
          // 2^-14 ||hi_i|| Hmax covers the fp32 accumulation-order difference between the one-term and the three-term sums.
          const float tau = 2.1f * (nr.x * Lmax + nr.y * Hmax) + 6.2e-5f * nr.x * Hmax;
          amb = !(best[h] - sec[h] > tau);                                      // also true for NaN / -inf oddities
          unsigned long long* out = dir ? P.best21 : P.best12;
          out[(int64_t)pair * (dir ? P.n2_max : P.n1_max) + row] = pack_vi(best[h], (uint32_t)col[h]);
        }
        // ambiguous rows: append (row index + split operand row) to the compact list of this (pair, direction)
        unsigned mask = __ballot_sync(0xffffffffu, amb);
        if (mask) {
          const int pd = pair * 2 + dir;
          int slot = 0;
          if (lane == 0) slot = atomicAdd(P.amb_cnt + pd, __popc(mask));
          slot = __shfl_sync(0xffffffffu, slot, 0);
          const __half* src_set = dir ? P.f2s : P.f1s;
          __half* dst_set = dir ? P.amb_rows1 : P.amb_rows0;
          while (mask) {
            const int l = __ffs(mask) - 1;
            mask &= mask - 1;
            const int src_row = __shfl_sync(0xffffffffu, row, l);
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(src_set + ((int64_t)pair * P.n_pad + src_row) * MF_KP) + lane);
            reinterpret_cast<uint2*>(dst_set + ((int64_t)pair * P.n_pad + slot) * MF_KP)[lane] = v;
            if (lane == 0) P.amb_idx[(int64_t)pd * P.n_pad + slot] = src_row;
            ++slot;
          }
        }
      }
    }
  }
}

struct MnnFastWs {
  __half *f1s, *f2s, *amb0, *amb1;
  unsigned long long *best12, *best21;
  float2 *norms1, *norms2;
  unsigned *maxn1, *maxn2, *absmax;
  int *amb_cnt, *amb_idx;
  float* inv_s2;
};
static inline int mf_pad(int n) { return (n + 2 * MF_ROWS - 1) / (2 * MF_ROWS) * (2 * MF_ROWS); }

static void carve_mnn_fast(Bump& bump, int batch, int n1_max, int n2_max, MnnFastWs& ws) {
  const int n_pad = mf_pad(n1_max > n2_max ? n1_max : n2_max);
  const size_t rows = (size_t)batch * n_pad;
  ws.f1s = bump.take<__half>(rows * MF_KP);
  ws.f2s = bump.take<__half>(rows * MF_KP);
  ws.amb0 = bump.take<__half>(rows * MF_KP);
  ws.amb1 = bump.take<__half>(rows * MF_KP);
  ws.best12 = bump.take<unsigned long long>((size_t)batch * n1_max);
  ws.best21 = bump.take<unsigned long long>((size_t)batch * n2_max);
  ws.norms1 = bump.take<float2>(rows);
  ws.norms2 = bump.take<float2>(rows);
  // one zero-initialised block: maxn1 [batch][2], maxn2 [batch][2], amb_cnt [batch][2], absmax [1]
  ws.maxn1 = bump.take<unsigned>((size_t)batch * 6 + 1);
  ws.maxn2 = ws.maxn1 + (size_t)batch * 2;
  ws.amb_cnt = reinterpret_cast<int*>(ws.maxn2 + (size_t)batch * 2);
  ws.absmax = reinterpret_cast<unsigned*>(ws.amb_cnt + (size_t)batch * 2);
  ws.amb_idx = bump.take<int>(rows * 2);
  ws.inv_s2 = bump.take<float>(1);
}

size_t mnn_fast_workspace_bytes(int batch, int n1_max, int n2_max) {
  Bump bump(nullptr, 0);
  MnnFastWs ws;
  carve_mnn_fast(bump, batch, n1_max, n2_max, ws);
  return bump.used();
}

int launch_absmax(const float* f, const int* np, int n_max, int64_t stride, int batch, unsigned* out, cudaStream_t st);   // mnn_tc.cu
int launch_mnn_tc_rows(const __half* a0, const __half* b0, const __half* a1, const __half* b1, const int* n1, int n1_max,
                       const int* n2, int n2_max, int n_pad, int batch, const int* rows_cnt, const int* row_map,
                       unsigned long long* best12, unsigned long long* best21, cudaStream_t st);   // mnn_tc.cu

static int mf_make_map(CUtensorMap* m, const __half* ptr, uint64_t rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)MF_KP, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)MF_KP * sizeof(__half)};
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

// Fills best12 / best21 exactly as launch_mnn_tc does (packed (value * s^2, index); the VALUE of a row that was not re-scored
// is the one-term approximation: the finalize step of this implementation thresholds on an exact dot product instead).
int launch_mnn_fast(const float* f1, const int* n1, int n1_max, int64_t stride1, const float* f2, const int* n2, int n2_max,
                    int64_t stride2, int batch, void* d_ws, size_t ws_bytes, unsigned long long** best12,
                    unsigned long long** best21, float** inv_s2, cudaStream_t st, float abs_bound, int sm_count) {
  Bump bump(d_ws, ws_bytes);
  MnnFastWs ws;
  carve_mnn_fast(bump, batch, n1_max, n2_max, ws);
  if (!bump.ok) {
    set_error("mnn_match(fast): workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  const int n_pad = mf_pad(n1_max > n2_max ? n1_max : n2_max);
  XF_REQUIRE((int64_t)batch * n_pad < (1ll << 31), "mnn_match(fast): batch * n too large");
  XF_CUDA(cudaMemsetAsync(ws.maxn1, 0, sizeof(unsigned) * ((size_t)batch * 6 + 1), st));
  int rc0;
  if (!(abs_bound > 0.f)) {
    if ((rc0 = launch_absmax(f1, n1, n1_max, stride1, batch, ws.absmax, st))) return rc0;
    if ((rc0 = launch_absmax(f2, n2, n2_max, stride2, batch, ws.absmax, st))) return rc0;
  }
  const dim3 sgrid(cdiv(n_pad * 32, 256), batch);
  split_norm_kernel<<<sgrid, 256, 0, st>>>(f1, n1, n1_max, n_pad, stride1, ws.absmax, abs_bound, ws.f1s, ws.norms1, ws.maxn1,
                                           ws.inv_s2);
  XF_LAUNCH_CHECK();
  split_norm_kernel<<<sgrid, 256, 0, st>>>(f2, n2, n2_max, n_pad, stride2, ws.absmax, abs_bound, ws.f2s, ws.norms2, ws.maxn2,
                                           nullptr);
  XF_LAUNCH_CHECK();
  XF_CUDA(cudaMemsetAsync(ws.best12, 0, sizeof(unsigned long long) * (size_t)batch * n1_max, st));
  XF_CUDA(cudaMemsetAsync(ws.best21, 0, sizeof(unsigned long long) * (size_t)batch * n2_max, st));
  MfParams P;
  int rc;
  if ((rc = mf_make_map(&P.m1, ws.f1s, (uint64_t)batch * n_pad))) return rc;
  if ((rc = mf_make_map(&P.m2, ws.f2s, (uint64_t)batch * n_pad))) return rc;
  P.n1p = n1; P.n2p = n2;
  P.n1_max = n1_max; P.n2_max = n2_max; P.n_pad = n_pad; P.batch = batch;
  P.f1s = ws.f1s; P.f2s = ws.f2s;
  P.norms1 = ws.norms1; P.norms2 = ws.norms2;
  P.maxn1 = ws.maxn1; P.maxn2 = ws.maxn2;
  P.best12 = ws.best12; P.best21 = ws.best21;
  P.amb_cnt = ws.amb_cnt; P.amb_idx = ws.amb_idx;
  P.amb_rows0 = ws.amb0; P.amb_rows1 = ws.amb1;
  XF_DYN_SMEM(mnn_fast_kernel, MF_SMEM);
  const int n_items = batch * 2 * (n_pad / MF_ROWS);
  const int grid = n_items < sm_count ? n_items : sm_count;
  mnn_fast_kernel<<<grid, MF_THREADS, MF_SMEM, st>>>(P);
  XF_LAUNCH_CHECK();
  // pass 2: the exact three-term kernel on the compact lists: direction 0 = ambiguous rows of set 1 against all of set 2, ...
  if ((rc = launch_mnn_tc_rows(ws.amb0, ws.f2s, ws.amb1, ws.f1s, n1, n1_max, n2, n2_max, n_pad, batch, ws.amb_cnt, ws.amb_idx,
                               ws.best12, ws.best21, st)))
    return rc;
  *best12 = ws.best12;
  *best21 = ws.best21;
  *inv_s2 = ws.inv_s2;
  return XF_OK;
}

}  // namespace xf
