// Mutual-nearest-neighbour matching on 64-D descriptors (XFeat.match xfeat.py:327-348, XFeat.batch_match :265-290).
//
// The reference materialises S = F1 F2^T (and its transpose) in memory (2 x 67 MB at N=4096) and reduces it four times.
// Here S is never written: a CTA owns a 128-row slab of F1, walks all 128-column tiles of F2, and keeps
//   * a running row arg-max in registers (final result for its rows),
//   * per-tile column arg-maxima that are merged across CTAs with one 64-bit atomicMax per column per CTA,
// both carried as (order-preserving value bits << 32 | ~index) so that an unsigned max implements torch's
// "largest value, lowest index on ties" rule exactly.  A second tiny kernel applies the mutual test, the optional
// min_cossim threshold and an ordered compaction (idx0 ascending, as boolean-mask indexing gives in the reference).
//
// fp32 FFMA (exact fp32 products, fp32 accumulate) -- the precision the integer outputs are specified against.
#include <cuda_fp16.h>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace xf {

constexpr int MNN_BM = 128, MNN_BN = 128, MNN_D = 64, MNN_THREADS = 256;
constexpr size_t MNN_SMEM = (size_t)(2 * MNN_D * MNN_BM) * sizeof(float) + 8 * MNN_BN * sizeof(unsigned long long);

// dst[k][r] = src[(row0 + r)][k] for r < 128, zero rows past nrows.
__device__ __forceinline__ void load_tile_T(float* __restrict__ dst, const float* __restrict__ src, int row0, int nrows,
                                            int tid) {
  // lanes walk rows (conflict-free transposed stores); 16 float4 per row
  for (int idx = tid; idx < 128 * 16; idx += MNN_THREADS) {
    const int r = idx & 127, q = idx >> 7;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < nrows) v = __ldg(reinterpret_cast<const float4*>(src + (int64_t)(row0 + r) * MNN_D) + q);
    dst[(4 * q + 0) * 128 + r] = v.x;
    dst[(4 * q + 1) * 128 + r] = v.y;
    dst[(4 * q + 2) * 128 + r] = v.z;
    dst[(4 * q + 3) * 128 + r] = v.w;
  }
}

__global__ void __launch_bounds__(MNN_THREADS) mnn_scan_kernel(const float* __restrict__ f1, const int* __restrict__ n1p,
                                                               int n1_max, int64_t stride1, const float* __restrict__ f2,
                                                               const int* __restrict__ n2p, int n2_max, int64_t stride2,
                                                               unsigned long long* __restrict__ row_best,
                                                               unsigned long long* __restrict__ col_best) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sA = reinterpret_cast<float*>(smem_raw);                 // [64][128]
  float* sB = sA + MNN_D * MNN_BM;                                // [64][128]
  unsigned long long* sCol = reinterpret_cast<unsigned long long*>(sB + MNN_D * MNN_BN);  // [8][128]

  const int pair = blockIdx.y;
  const int n1 = n1p ? min(n1p[pair], n1_max) : n1_max;
  const int n2 = n2p ? min(n2p[pair], n2_max) : n2_max;
  const int row0 = blockIdx.x * MNN_BM;
  if (row0 >= n1) return;
  const float* A = f1 + (int64_t)pair * stride1;
  const float* Bm = f2 + (int64_t)pair * stride2;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, warp = tid >> 5, lane = tid & 31;

  load_tile_T(sA, A, row0, n1, tid);

  unsigned long long rbest[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) rbest[i] = 0ull;

  for (int col0 = 0; col0 < n2; col0 += MNN_BN) {
    __syncthreads();  // previous tile's sB / sCol consumers are done
    load_tile_T(sB, Bm, col0, n2, tid);
    __syncthreads();
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
#pragma unroll 8
    for (int k = 0; k < MNN_D; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(sA + k * 128 + 4 * ty);
      const float4 a1 = *reinterpret_cast<const float4*>(sA + k * 128 + 64 + 4 * ty);
      const float4 b0 = *reinterpret_cast<const float4*>(sB + k * 128 + 4 * tx);
      const float4 b1 = *reinterpret_cast<const float4*>(sB + k * 128 + 64 + 4 * tx);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    // ---- row arg-max over this tile's columns (ascending column order, strict > keeps the first) ----
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float bv = -INFINITY;
      int bc = -1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = col0 + ((j < 4) ? 4 * tx + j : 64 + 4 * tx + (j - 4));
        const float v = acc[i][j];
        if (c < n2 && (bc < 0 || v > bv)) { bv = v; bc = c; }
      }
      if (bc >= 0) {
        const unsigned long long p = pack_vi(bv, (uint32_t)bc);
        if (p > rbest[i]) rbest[i] = p;
      }
    }
    // ---- column arg-max over this CTA's rows ----
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float bv = -INFINITY;
      int br = -1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = row0 + ((i < 4) ? 4 * ty + i : 64 + 4 * ty + (i - 4));
        const float v = acc[i][j];
        if (r < n1 && (br < 0 || v > bv)) { bv = v; br = r; }
      }
      unsigned long long p = (br >= 0) ? pack_vi(bv, (uint32_t)br) : 0ull;
      // lanes l and l^16 hold the same columns for ty and ty^1
      const unsigned long long q = __shfl_xor_sync(0xffffffffu, p, 16);
      if (q > p) p = q;
      if (lane < 16) sCol[warp * 128 + ((j < 4) ? 4 * tx + j : 64 + 4 * tx + (j - 4))] = p;
    }
    __syncthreads();
    if (tid < 128 && col0 + tid < n2) {
      unsigned long long p = sCol[tid];
#pragma unroll
      for (int w = 1; w < 8; ++w) {
        const unsigned long long q = sCol[w * 128 + tid];
        if (q > p) p = q;
      }
      if (p) atomicMax(col_best + (int64_t)pair * n2_max + col0 + tid, p);
    }
  }
  // ---- finish rows: reduce across the 16 lanes (tx) that share them ----
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    unsigned long long p = rbest[i];
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      const unsigned long long q = __shfl_xor_sync(0xffffffffu, p, o);
      if (q > p) p = q;
    }
    const int r = row0 + ((i < 4) ? 4 * ty + i : 64 + 4 * ty + (i - 4));
    if (tx == 0 && r < n1) row_best[(int64_t)pair * n1_max + r] = p;
  }
}

// One CTA per pair: mutual test + threshold + ordered compaction.
// f1 / f2 (optional, with their per-pair strides in floats): when given, the min_cossim test uses the fp32 dot product of the
// matched rows instead of the packed value (implementation 4 carries approximate values for rows it did not re-score).
// kPairs: pair p = (image i, image j) of `pairs` reads its counts as n1p[i], n2p[j] (the pair table of mnn_tc_kernel); row_best,
// col_best and the outputs stay per pair.  A template flag, so that the per-pair instantiation keeps its code as it was.
template <bool kPairs = false>
__global__ void __launch_bounds__(1024) mnn_finalize_kernel(const unsigned long long* __restrict__ row_best,
                                                            const unsigned long long* __restrict__ col_best,
                                                            const int* __restrict__ n1p, const int* __restrict__ n2p,
                                                            int n1_max, int n2_max, float min_cossim,
                                                            const float* __restrict__ val_scale,
                                                            long long* __restrict__ idx0,
                                                            long long* __restrict__ idx1, int* __restrict__ n_matches,
                                                            const float* __restrict__ f1 = nullptr, int64_t stride1 = 0,
                                                            const float* __restrict__ f2 = nullptr, int64_t stride2 = 0,
                                                            const int2* __restrict__ pairs = nullptr) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_base;
  const int pair = blockIdx.x;
  const int2 ij = kPairs ? pairs[pair] : make_int2(pair, pair);
  const int n1 = n1p ? min(n1p[ij.x], n1_max) : n1_max;
  if (threadIdx.x == 0) s_base = 0;
  const float vs = val_scale ? __ldg(val_scale) : 1.0f;   // tensor-core path carries values scaled by a power of two
  __syncthreads();
  for (int i0 = 0; i0 < n1; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    int flag = 0;
    uint32_t j = 0;
    if (i < n1) {
      const unsigned long long rb = row_best[(int64_t)pair * n1_max + i];
      if (rb) {
        j = packed_idx(rb);
        const unsigned long long cb = col_best[(int64_t)pair * n2_max + j];
        flag = (cb != 0ull) && (packed_idx(cb) == (uint32_t)i);
        if (flag && min_cossim > 0.f) {
          float v = packed_val(rb) * vs;
          if (f1) {
            const float4* a = reinterpret_cast<const float4*>(f1 + (int64_t)pair * stride1 + (int64_t)i * 64);
            const float4* b = reinterpret_cast<const float4*>(f2 + (int64_t)pair * stride2 + (int64_t)j * 64);
            v = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
              const float4 x = __ldg(a + k), y = __ldg(b + k);
              v = fmaf(x.x, y.x, v); v = fmaf(x.y, y.y, v); v = fmaf(x.z, y.z, v); v = fmaf(x.w, y.w, v);
            }
          }
          flag = v > min_cossim;
        }
      }
    }
    int off, total;
    Scan(tmp).ExclusiveSum(flag, off, total);
    const int base = s_base;
    if (flag) {
      idx0[(int64_t)pair * n1_max + base + off] = i;
      idx1[(int64_t)pair * n1_max + base + off] = (long long)j;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_base = base + total;
    __syncthreads();
  }
  // a negative count is xfeat_detect_sparse's overflow indicator (XF_N_OVERFLOW): it propagates instead of reading as "no matches"
  const bool overflow = (n1p && n1p[ij.x] < 0) || (n2p && n2p[ij.y] < 0);
  if (threadIdx.x == 0) n_matches[pair] = overflow ? -1 : s_base;
}

// kPairs: pair p = (image i, image j) of `pairs` reads keypoints k0[i] and k1[j] (both usually the same image table)
template <bool kPairs = false>
__global__ void __launch_bounds__(256) gather_matches_kernel(const float* __restrict__ k0, const float* __restrict__ k1,
                                                             int n1_max, int n2_max, const long long* __restrict__ idx0,
                                                             const long long* __restrict__ idx1,
                                                             const int* __restrict__ n_matches, float* __restrict__ o0,
                                                             float* __restrict__ o1, const int2* __restrict__ pairs = nullptr) {
  const int pair = blockIdx.y;
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_matches[pair]) return;
  const int2 ij = kPairs ? __ldg(pairs + pair) : make_int2(pair, pair);
  const int64_t o = (int64_t)pair * n1_max + m;
  const long long a = idx0[o], b = idx1[o];
  reinterpret_cast<float2*>(o0)[o] = __ldg(reinterpret_cast<const float2*>(k0) + (int64_t)ij.x * n1_max + a);
  reinterpret_cast<float2*>(o1)[o] = __ldg(reinterpret_cast<const float2*>(k1) + (int64_t)ij.y * n2_max + b);
}

struct MnnWs {
  unsigned long long *row_best, *col_best;
};
static void carve_mnn(Bump& bump, int batch, int n1_max, int n2_max, MnnWs& ws) {
  ws.row_best = bump.take<unsigned long long>((size_t)batch * n1_max);
  ws.col_best = bump.take<unsigned long long>((size_t)batch * n2_max);
}

// tensor-core implementation (mnn_tc.cu)
size_t mnn_tc_workspace_bytes(int batch, int n1_max, int n2_max);
int launch_mnn_tc(const float* f1, const int* n1, int n1_max, int64_t stride1, const float* f2, const int* n2, int n2_max,
                  int64_t stride2, int batch, void* d_ws, size_t ws_bytes, unsigned long long** best12,
                  unsigned long long** best21, float** inv_s2, cudaStream_t st, int variant, float abs_bound);
// 0 = fp32 CUDA cores; 1 = wgmma split-fp16, persistent, ONE GEMM per pair whose accumulator tiles give both the row and the
// column arg-max, the two consumer warpgroups' epilogues overlapped with each other's MMAs (default); 2 = the persistent
// kernel with one GEMM per direction -- same results, kept as the reference implementation 1 is compared against;
// 3 = one CTA per (row block, pair, direction), one GEMM per direction
// 4 = filter + exact re-score (mnn_fast.cu): one fp16 pass per direction tracking top-1 / top-2, the three-term kernel only on
// the rows whose gap is within the rounding bound -- same results as 1.  Measured (profiles/r02/mnn_probe.json, 64 x 4096^2):
// the filter pass is bound by the ALU pipe (FMNMX at 16 lanes/clk: 370 us against 115 us of tensor time), and the descriptors of
// the bench images (strong common mode, median top-1/top-2 gap 1.6e-3 against a bound of 1.1e-3) send 40 % of the rows to the
// exact kernel: 0.57 ms vs 0.61 ms on well separated descriptors, 0.80 ms vs 0.61 ms on the bench workload.  Selectable, not
// default.
static int g_mnn_impl = 1;
size_t mnn_fast_workspace_bytes(int batch, int n1_max, int n2_max);
int launch_mnn_tc_presplit(const __half* f1s, const int* n1, int n1_max, const __half* f2s, const int* n2, int n2_max, int n_pad,
                           int batch, int scale_log2, void* d_ws, size_t ws_bytes, unsigned long long** best12,
                           unsigned long long** best21, float** inv_s2, cudaStream_t st, int variant,
                           const int2* pairs = nullptr, int n_images = 0);
int launch_mnn_fast(const float* f1, const int* n1, int n1_max, int64_t stride1, const float* f2, const int* n2, int n2_max,
                    int64_t stride2, int batch, void* d_ws, size_t ws_bytes, unsigned long long** best12,
                    unsigned long long** best21, float** inv_s2, cudaStream_t st, float abs_bound, int sm_count);
size_t mnn_tc_pairs_workspace_bytes(int n_pairs, int n_max);
int launch_mnn_tc_pairs_f32(const float* f, const int* n, int n_max, const int2* pairs, int n_pairs, void* d_ws, size_t ws_bytes,
                            unsigned long long** best12, unsigned long long** best21, float** inv_s2, const int** cnt1,
                            const int** cnt2, cudaStream_t st, int variant);

}  // namespace xf

extern "C" void xfeat_set_mnn_impl(int impl) { xf::g_mnn_impl = impl < 0 ? 0 : (impl > 4 ? 4 : impl); }
extern "C" int xfeat_get_mnn_impl(void) { return xf::g_mnn_impl; }

extern "C" size_t xfeat_mnn_workspace_bytes(int batch, int n1_max, int n2_max) {
  xf::Bump bump(nullptr, 0);
  xf::MnnWs ws;
  xf::carve_mnn(bump, batch, n1_max, n2_max, ws);
  const size_t a = bump.used(), b = xf::mnn_tc_workspace_bytes(batch, n1_max, n2_max);
  const size_t c = xf::mnn_fast_workspace_bytes(batch, n1_max, n2_max);
  return (a > b ? a : b) > c ? (a > b ? a : b) : c;
}

extern "C" int xfeat_mnn_match(const float* d_f1, const int32_t* d_n1, int n1_max, int64_t stride1, const float* d_f2,
                               const int32_t* d_n2, int n2_max, int64_t stride2, int batch, float min_cossim,
                               int64_t* d_idx0, int64_t* d_idx1, int32_t* d_n_matches, void* d_ws, size_t ws_bytes,
                               void* stream) {
  return xfeat_mnn_match_bounded(d_f1, d_n1, n1_max, stride1, d_f2, d_n2, n2_max, stride2, batch, min_cossim, 0.f, d_idx0, d_idx1,
                                 d_n_matches, d_ws, ws_bytes, stream);
}

extern "C" int xfeat_mnn_match_bounded(const float* d_f1, const int32_t* d_n1, int n1_max, int64_t stride1, const float* d_f2,
                                       const int32_t* d_n2, int n2_max, int64_t stride2, int batch, float min_cossim,
                                       float abs_bound, int64_t* d_idx0, int64_t* d_idx1, int32_t* d_n_matches, void* d_ws,
                                       size_t ws_bytes, void* stream) {
  XF_REQUIRE(d_f1 && d_f2 && d_idx0 && d_idx1 && d_n_matches && d_ws, "mnn_match: null pointer");
  XF_REQUIRE(batch > 0 && batch <= 65535 && n1_max > 0 && n2_max > 0, "mnn_match: bad sizes");
  XF_REQUIRE(((uintptr_t)d_f1 % 16) == 0 && ((uintptr_t)d_f2 % 16) == 0 && stride1 % 4 == 0 && stride2 % 4 == 0,
             "mnn_match: descriptors must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (!(abs_bound > 0.f) || !isfinite(abs_bound)) abs_bound = 0.f;   // no usable bound: measure max |x| on the device
  if (xf::g_mnn_impl == 4) {
    unsigned long long *b12 = nullptr, *b21 = nullptr;
    float* inv_s2 = nullptr;
    int dev = 0, sms = 148;
    XF_CUDA(cudaGetDevice(&dev));
    XF_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int rc = xf::launch_mnn_fast(d_f1, d_n1, n1_max, stride1, d_f2, d_n2, n2_max, stride2, batch, d_ws, ws_bytes, &b12, &b21,
                                 &inv_s2, st, abs_bound, sms);
    if (rc) return rc;
    xf::mnn_finalize_kernel<<<batch, 1024, 0, st>>>(b12, b21, d_n1, d_n2, n1_max, n2_max, min_cossim, inv_s2, (long long*)d_idx0,
                                                    (long long*)d_idx1, d_n_matches, d_f1, stride1, d_f2, stride2);
    XF_LAUNCH_CHECK();
    return XF_OK;
  }
  if (xf::g_mnn_impl >= 1) {
    unsigned long long *b12 = nullptr, *b21 = nullptr;
    float* inv_s2 = nullptr;
    int rc = xf::launch_mnn_tc(d_f1, d_n1, n1_max, stride1, d_f2, d_n2, n2_max, stride2, batch, d_ws, ws_bytes, &b12, &b21,
                               &inv_s2, st, xf::g_mnn_impl - 1, abs_bound);
    if (rc) return rc;
    xf::mnn_finalize_kernel<<<batch, 1024, 0, st>>>(b12, b21, d_n1, d_n2, n1_max, n2_max, min_cossim, inv_s2, (long long*)d_idx0,
                                                    (long long*)d_idx1, d_n_matches);
    XF_LAUNCH_CHECK();
    return XF_OK;
  }
  xf::Bump bump(d_ws, ws_bytes);
  xf::MnnWs ws;
  xf::carve_mnn(bump, batch, n1_max, n2_max, ws);
  if (!bump.ok) {
    xf::set_error("mnn_match: workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  XF_DYN_SMEM(xf::mnn_scan_kernel, xf::MNN_SMEM);
  XF_CUDA(cudaMemsetAsync(ws.row_best, 0, sizeof(unsigned long long) * (size_t)batch * n1_max, st));
  XF_CUDA(cudaMemsetAsync(ws.col_best, 0, sizeof(unsigned long long) * (size_t)batch * n2_max, st));
  dim3 grid(xf::cdiv(n1_max, xf::MNN_BM), batch);
  xf::mnn_scan_kernel<<<grid, xf::MNN_THREADS, xf::MNN_SMEM, st>>>(d_f1, d_n1, n1_max, stride1, d_f2, d_n2, n2_max, stride2,
                                                                  ws.row_best, ws.col_best);
  XF_LAUNCH_CHECK();
  xf::mnn_finalize_kernel<<<batch, 1024, 0, st>>>(ws.row_best, ws.col_best, d_n1, d_n2, n1_max, n2_max, min_cossim, nullptr,
                                                  (long long*)d_idx0, (long long*)d_idx1, d_n_matches);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" size_t xfeat_mnn_presplit_workspace_bytes(int batch, int n1_max, int n2_max) {
  xf::Bump bump(nullptr, 0);
  bump.take<unsigned long long>((size_t)batch * n1_max);
  bump.take<unsigned long long>((size_t)batch * n2_max);
  bump.take<float>(1);
  return bump.used();
}

extern "C" int xfeat_mnn_match_presplit(const void* d_f1s, const int32_t* d_n1, int n1_max, const void* d_f2s, const int32_t* d_n2,
                                        int n2_max, int n_pad, int batch, int scale_log2, float min_cossim, int64_t* d_idx0,
                                        int64_t* d_idx1, int32_t* d_n_matches, void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(d_f1s && d_f2s && d_idx0 && d_idx1 && d_n_matches && d_ws, "mnn_match_presplit: null pointer");
  XF_REQUIRE(batch > 0 && batch <= 65535 && n1_max > 0 && n2_max > 0, "mnn_match_presplit: bad sizes");
  XF_REQUIRE(((uintptr_t)d_f1s % 128) == 0 && ((uintptr_t)d_f2s % 128) == 0, "mnn_match_presplit: operands must be 128-byte aligned");
  if (xf::g_mnn_impl < 1 || xf::g_mnn_impl > 3) {
    xf::set_error("mnn_match_presplit: implementation %d does not take pre-split operands (1, 2 and 3 do)", xf::g_mnn_impl);
    return XF_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long *b12 = nullptr, *b21 = nullptr;
  float* inv_s2 = nullptr;
  int rc = xf::launch_mnn_tc_presplit((const __half*)d_f1s, d_n1, n1_max, (const __half*)d_f2s, d_n2, n2_max, n_pad, batch,
                                      scale_log2, d_ws, ws_bytes, &b12, &b21, &inv_s2, st, xf::g_mnn_impl - 1);
  if (rc) return rc;
  xf::mnn_finalize_kernel<<<batch, 1024, 0, st>>>(b12, b21, d_n1, d_n2, n1_max, n2_max, min_cossim, inv_s2, (long long*)d_idx0,
                                                  (long long*)d_idx1, d_n_matches);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" size_t xfeat_mnn_pairs_workspace_bytes(int n_pairs, int n_max) {
  return xfeat_mnn_presplit_workspace_bytes(n_pairs, n_max, n_max);
}

extern "C" int xfeat_mnn_match_pairs(const void* d_fs, const int32_t* d_n, int n_images, int n_max, int n_pad,
                                     const int32_t* d_pairs, int n_pairs, int scale_log2, float min_cossim, int64_t* d_idx0,
                                     int64_t* d_idx1, int32_t* d_n_matches, void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(d_fs && d_n && d_pairs && d_idx0 && d_idx1 && d_n_matches && d_ws, "mnn_match_pairs: null pointer");
  XF_REQUIRE(n_images > 0 && n_pairs > 0 && n_pairs <= 65535 && n_max > 0, "mnn_match_pairs: bad sizes");
  XF_REQUIRE(((uintptr_t)d_fs % 128) == 0, "mnn_match_pairs: operands must be 128-byte aligned");
  XF_REQUIRE(((uintptr_t)d_pairs % 8) == 0, "mnn_match_pairs: the pair table must be 8-byte aligned");
  if (xf::g_mnn_impl < 1 || xf::g_mnn_impl > 3) {
    xf::set_error("mnn_match_pairs: implementation %d does not take pre-split operands (1, 2 and 3 do)", xf::g_mnn_impl);
    return XF_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int2* pairs = reinterpret_cast<const int2*>(d_pairs);
  unsigned long long *b12 = nullptr, *b21 = nullptr;
  float* inv_s2 = nullptr;
  int rc = xf::launch_mnn_tc_presplit((const __half*)d_fs, d_n, n_max, (const __half*)d_fs, d_n, n_max, n_pad, n_pairs, scale_log2,
                                      d_ws, ws_bytes, &b12, &b21, &inv_s2, st, xf::g_mnn_impl - 1, pairs, n_images);
  if (rc) return rc;
  xf::mnn_finalize_kernel<true><<<n_pairs, 1024, 0, st>>>(b12, b21, d_n, d_n, n_max, n_max, min_cossim, inv_s2, (long long*)d_idx0,
                                                    (long long*)d_idx1, d_n_matches, nullptr, 0, nullptr, 0, pairs);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" size_t xfeat_mnn_pairs_f32_workspace_bytes(int n_pairs, int n_max) {
  return xf::mnn_tc_pairs_workspace_bytes(n_pairs, n_max);
}

extern "C" int xfeat_mnn_match_pairs_f32(const float* d_f, const int32_t* d_n, int n_images, int n_max, const int32_t* d_pairs,
                                         int n_pairs, int64_t* d_idx0, int64_t* d_idx1, int32_t* d_n_matches, void* d_ws,
                                         size_t ws_bytes, void* stream) {
  XF_REQUIRE(d_f && d_n && d_pairs && d_idx0 && d_idx1 && d_n_matches && d_ws, "mnn_match_pairs_f32: null pointer");
  XF_REQUIRE(n_images > 0 && n_pairs > 0 && n_pairs <= 65535 && n_max > 0, "mnn_match_pairs_f32: bad sizes");
  XF_REQUIRE(((uintptr_t)d_f % 16) == 0, "mnn_match_pairs_f32: descriptors must be 16-byte aligned");
  XF_REQUIRE(((uintptr_t)d_pairs % 8) == 0, "mnn_match_pairs_f32: the pair table must be 8-byte aligned");
  if (xf::g_mnn_impl < 1 || xf::g_mnn_impl > 3) {
    xf::set_error("mnn_match_pairs_f32: implementation %d does not take pre-split operands (1, 2 and 3 do)", xf::g_mnn_impl);
    return XF_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long *b12 = nullptr, *b21 = nullptr;
  float* inv_s2 = nullptr;
  const int *n1 = nullptr, *n2 = nullptr;
  int rc = xf::launch_mnn_tc_pairs_f32(d_f, d_n, n_max, reinterpret_cast<const int2*>(d_pairs), n_pairs, d_ws, ws_bytes, &b12,
                                       &b21, &inv_s2, &n1, &n2, st, xf::g_mnn_impl - 1);
  if (rc) return rc;
  xf::mnn_finalize_kernel<<<n_pairs, 1024, 0, st>>>(b12, b21, n1, n2, n_max, n_max, -1.f, inv_s2, (long long*)d_idx0,
                                                    (long long*)d_idx1, d_n_matches);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_gather_matches_pairs(const float* d_kpts, int n_max, const int32_t* d_pairs, const int64_t* d_idx0,
                                          const int64_t* d_idx1, const int32_t* d_n_matches, int n_pairs, float* d_out0,
                                          float* d_out1, void* stream) {
  XF_REQUIRE(d_kpts && d_pairs && d_idx0 && d_idx1 && d_n_matches && d_out0 && d_out1, "gather_matches_pairs: null pointer");
  XF_REQUIRE(n_pairs > 0 && n_pairs <= 65535 && n_max > 0, "gather_matches_pairs: bad sizes");
  XF_REQUIRE(((uintptr_t)d_pairs % 8) == 0, "gather_matches_pairs: the pair table must be 8-byte aligned");
  dim3 grid(xf::cdiv(n_max, 256), n_pairs);
  xf::gather_matches_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(d_kpts, d_kpts, n_max, n_max, (const long long*)d_idx0,
                                                                    (const long long*)d_idx1, d_n_matches, d_out0, d_out1,
                                                                    reinterpret_cast<const int2*>(d_pairs));
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_gather_matches(const float* d_kpts0, const float* d_kpts1, int n1_max, int n2_max,
                                    const int64_t* d_idx0, const int64_t* d_idx1, const int32_t* d_n_matches, int batch,
                                    float* d_out0, float* d_out1, void* stream) {
  XF_REQUIRE(d_kpts0 && d_kpts1 && d_idx0 && d_idx1 && d_n_matches && d_out0 && d_out1, "gather_matches: null pointer");
  dim3 grid(xf::cdiv(n1_max, 256), batch);
  xf::gather_matches_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_kpts0, d_kpts1, n1_max, n2_max,
                                                                    (const long long*)d_idx0, (const long long*)d_idx1,
                                                                    d_n_matches, d_out0, d_out1);
  XF_LAUNCH_CHECK();
  return XF_OK;
}
