// XFeat* match refinement for a whole batch of pairs at once (XFeat.refine_matches xfeat.py:306-325,
// subpix_softmax2d xfeat.py:292-304, fine_matcher model.py:97-111).
//   1. exclusive scan of the per-pair coarse match counts -> row offsets (device side, no host sync);
//   2. gather cat(desc0[idx0], desc1[idx1]) into a dense (rows,128) matrix;
//   3. the 5-layer MLP runs through the generic fp32 GEMM kernel in flattened-row mode; tiles past the live row count
//      exit immediately (count read from device memory);
//   4. per row: conf = max softmax(3 o), offset = E[(x-4, y-4)], kp0 += offset * scale0; conf > fine_conf kept;
//   5. ordered per-pair compaction (boolean-mask order of the reference).
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace xf {

__global__ void __launch_bounds__(1024) scan_counts_kernel(const int* __restrict__ counts, int n, int cap,
                                                           int* __restrict__ offsets /* n+1 */) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_base;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    const int c = (i < n) ? max(0, min(counts[i], cap)) : 0;
    int off, total;
    Scan(tmp).ExclusiveSum(c, off, total);
    const int base = s_base;
    if (i < n) offsets[i] = base + off;
    __syncthreads();
    if (threadIdx.x == 0) s_base = base + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[n] = s_base;
}

// warp per (pair, m): X[row] = [desc0[pair][idx0[m]], desc1[pair][idx1[m]]]
// kPairs: pair p = pairs[p] = (i, j) reads desc0[i] and desc1[j] of one table (both at stride n_max = n1_max) -- the image slots
// of xfeat_refine_pairs.  A template flag, so that the per-pair build keeps its code.
template <bool kPairs = false>
__global__ void __launch_bounds__(256) refine_gather_kernel(const float* __restrict__ d0, const float* __restrict__ d1,
                                                            const long long* __restrict__ idx0,
                                                            const long long* __restrict__ idx1,
                                                            const int* __restrict__ n_matches,
                                                            const int* __restrict__ offsets, int batch, int n_max,
                                                            int n1_max, float* __restrict__ X, __half* __restrict__ Xs,
                                                            const int2* __restrict__ pairs = nullptr) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (int64_t)batch * n_max) return;
  const int pair = (int)(wid / n_max), m = (int)(wid - (int64_t)pair * n_max);
  if (m >= min(n_matches[pair], n_max)) return;
  const int64_t row = offsets[pair] + m;
  const long long a = idx0[wid], b = idx1[wid];
  const int2 ij = kPairs ? __ldg(pairs + pair) : make_int2(pair, pair);
  const float2 u = __ldg(reinterpret_cast<const float2*>(d0 + ((int64_t)ij.x * n_max + a) * 64) + lane);
  const float2 v = __ldg(reinterpret_cast<const float2*>(d1 + ((int64_t)ij.y * n1_max + b) * 64) + lane);
  if (Xs) {   // tensor-core MLP: split fp16 row [hi(128) | lo(128)] (mlp_tc.cu)
    const __half2 uh = __floats2half2_rn(u.x, u.y), vh = __floats2half2_rn(v.x, v.y);
    const float2 uf = __half22float2(uh), vf = __half22float2(vh);
    __half2* o = reinterpret_cast<__half2*>(Xs + row * 256);
    o[lane] = uh;
    o[32 + lane] = vh;
    o[64 + lane] = __floats2half2_rn(u.x - uf.x, u.y - uf.y);
    o[96 + lane] = __floats2half2_rn(v.x - vf.x, v.y - vf.y);
    return;
  }
  reinterpret_cast<float2*>(X + row * 128)[lane] = u;
  reinterpret_cast<float2*>(X + row * 128 + 64)[lane] = v;
}

// warp per (pair, m): softmax(3*o) statistics -> tmp[wid] = (x0', y0', x1, y1, keep)
// kPairs: k0 / sc0 of image i and k1 of image j of pairs[p] = (i, j), as in refine_gather_kernel
template <bool kPairs = false>
__global__ void __launch_bounds__(256) refine_finish_kernel(const float* __restrict__ logits,
                                                            const float* __restrict__ k0, const float* __restrict__ k1,
                                                            const float* __restrict__ sc0,
                                                            const long long* __restrict__ idx0,
                                                            const long long* __restrict__ idx1,
                                                            const int* __restrict__ n_matches,
                                                            const int* __restrict__ offsets, int batch, int n_max,
                                                            int n1_max, float fine_conf, float* __restrict__ tmp,
                                                            int* __restrict__ keep, const int2* __restrict__ pairs = nullptr) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (int64_t)batch * n_max) return;
  const int pair = (int)(wid / n_max), m = (int)(wid - (int64_t)pair * n_max);
  if (m >= min(n_matches[pair], n_max)) return;
  const int64_t row = offsets[pair] + m;
  const float2 o = __ldg(reinterpret_cast<const float2*>(logits + row * 64) + lane);
  const float z0 = o.x * 3.f, z1 = o.y * 3.f;
  float mx = fmaxf(z0, z1);
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
  const float e0 = expf(z0 - mx), e1 = expf(z1 - mx);
  // channel c = 2*lane (+1): x = c % 8 - 4, y = c / 8 - 4   (meshgrid 'xy', x fastest; xfeat.py:295-297)
  const int c0 = 2 * lane;
  const float x0 = (float)((c0 & 7) - 4), x1 = (float)(((c0 + 1) & 7) - 4), y = (float)((c0 >> 3) - 4);
  float s = e0 + e1, sx = e0 * x0 + e1 * x1, sy = (e0 + e1) * y;
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, k);
    sx += __shfl_xor_sync(0xffffffffu, sx, k);
    sy += __shfl_xor_sync(0xffffffffu, sy, k);
  }
  if (lane == 0) {
    const float conf = 1.0f / s;  // max of the softmax = exp(0)/sum
    const long long a = idx0[wid], b = idx1[wid];
    const int2 ij = kPairs ? __ldg(pairs + pair) : make_int2(pair, pair);
    const float scale = __ldg(sc0 + (int64_t)ij.x * n_max + a);
    const float2 p0 = __ldg(reinterpret_cast<const float2*>(k0) + (int64_t)ij.x * n_max + a);
    const float2 p1 = __ldg(reinterpret_cast<const float2*>(k1) + (int64_t)ij.y * n1_max + b);
    float* t = tmp + wid * 4;
    t[0] = p0.x + (sx / s) * scale;  // mkpts_0 += offsets * sc0 (xfeat.py:319)
    t[1] = p0.y + (sy / s) * scale;
    t[2] = p1.x;
    t[3] = p1.y;
    keep[wid] = conf > fine_conf;
  }
}

__global__ void __launch_bounds__(1024) refine_compact_kernel(const float* __restrict__ tmp, const int* __restrict__ keep,
                                                              const int* __restrict__ n_matches, int n_max,
                                                              float* __restrict__ out, int* __restrict__ n_refined) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmpst;
  __shared__ int s_base;
  const int pair = blockIdx.x;
  const int n = min(n_matches[pair], n_max);
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    const int64_t g = (int64_t)pair * n_max + i;
    const int flag = (i < n) ? keep[g] : 0;
    int off, total;
    Scan(tmpst).ExclusiveSum(flag, off, total);
    const int base = s_base;
    if (flag) reinterpret_cast<float4*>(out)[(int64_t)pair * n_max + base + off] = reinterpret_cast<const float4*>(tmp)[g];
    __syncthreads();
    if (threadIdx.x == 0) s_base = base + total;
    __syncthreads();
  }
  // a negative count (XF_N_OVERFLOW from the matcher) is a status, not "no matches": pass it through
  if (threadIdx.x == 0) n_refined[pair] = n_matches[pair] < 0 ? n_matches[pair] : s_base;
}

struct RefineWs {
  int* offsets;
  float *X, *actA, *actB, *logits, *tmp;
  int* keep;
};
static void carve_refine(Bump& bump, int batch, int n_max, RefineWs& ws) {
  const size_t cap = (size_t)batch * n_max;
  ws.offsets = bump.take<int>(batch + 1);
  ws.X = bump.take<float>(cap * 128);
  ws.actA = bump.take<float>(cap * 512);
  ws.actB = bump.take<float>(cap * 512);
  ws.logits = bump.take<float>(cap * 64);
  ws.tmp = bump.take<float>(cap * 4);
  ws.keep = bump.take<int>(cap);
}

// fine_matcher (model.py:97-111): 128 -> 512 -> 512 -> 512 -> 512 -> 64 on `rows_cap` rows of X (row-major, 128 floats);
// n_live (device, may be null) = number of live rows: tiles past it exit immediately.
int launch_fine_mlp(const xfeat_ctx* ctx, const float* X, int rows_cap, const int* n_live, float* actA, float* actB,
                    float* logits, cudaStream_t st) {
  int rc;
  if ((rc = launch_conv_layer(ctx, L_FM_0, X, IN_NHWC, 1, 1, rows_cap, actA, st, n_live))) return rc;
  if ((rc = launch_conv_layer(ctx, L_FM_1, actA, IN_NHWC, 1, 1, rows_cap, actB, st, n_live))) return rc;
  if ((rc = launch_conv_layer(ctx, L_FM_2, actB, IN_NHWC, 1, 1, rows_cap, actA, st, n_live))) return rc;
  if ((rc = launch_conv_layer(ctx, L_FM_3, actA, IN_NHWC, 1, 1, rows_cap, actB, st, n_live))) return rc;
  return launch_conv_layer(ctx, L_FM_4, actB, IN_NHWC, 1, 1, rows_cap, logits, st, n_live);
}

}  // namespace xf

extern "C" size_t xfeat_refine_workspace_bytes(int batch, int n_max) {
  xf::Bump bump(nullptr, 0);
  xf::RefineWs ws;
  xf::carve_refine(bump, batch, n_max, ws);
  return bump.used();
}

// xfeat_refine and xfeat_refine_pairs: pairs == NULL -> pair p reads slot p of desc0 / desc1 / kpts0 / kpts1 / scales0.
static int refine_impl(xfeat_ctx* ctx, const float* d_desc0, const float* d_desc1, const float* d_kpts0, const float* d_kpts1,
                       const float* d_scales0, const int64_t* d_idx0, const int64_t* d_idx1, const int32_t* d_n_matches, int batch,
                       int n_max, int n1_max, float fine_conf, float* d_matches, int32_t* d_n_refined, void* d_ws,
                       size_t ws_bytes, cudaStream_t st, const int2* pairs) {
  XF_CUDA(cudaSetDevice(ctx->device));
  xf::Bump bump(d_ws, ws_bytes);
  xf::RefineWs ws;
  xf::carve_refine(bump, batch, n_max, ws);
  if (!bump.ok) {
    xf::set_error("refine: workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  const int64_t cap = (int64_t)batch * n_max;
  const unsigned wblocks = (unsigned)((cap * 32 + 255) / 256);
  const bool tc = xf::g_conv_impl != 0;   // xfeat_set_conv_impl(0): everything on the fp32 CUDA-core kernels (A/B reference)
  xf::scan_counts_kernel<<<1, 1024, 0, st>>>(d_n_matches, batch, n_max, ws.offsets);
  XF_LAUNCH_CHECK();
  if (pairs)
    xf::refine_gather_kernel<true><<<wblocks, 256, 0, st>>>(d_desc0, d_desc1, (const long long*)d_idx0, (const long long*)d_idx1,
                                                            d_n_matches, ws.offsets, batch, n_max, n1_max, ws.X,
                                                            tc ? (__half*)ws.X : nullptr, pairs);
  else
    xf::refine_gather_kernel<<<wblocks, 256, 0, st>>>(d_desc0, d_desc1, (const long long*)d_idx0, (const long long*)d_idx1,
                                                      d_n_matches, ws.offsets, batch, n_max, n1_max, ws.X,
                                                      tc ? (__half*)ws.X : nullptr);
  XF_LAUNCH_CHECK();
  const int* n_live = ws.offsets + batch;
  int rc;
  if (tc) {   // X (cap x 128 floats) holds the split row (cap x 256 halves); actA / actB (cap x 512 floats) hold cap x 1024 halves
    if ((rc = xf::launch_fine_mlp_tc(ctx, (const __half*)ws.X, (int)cap, n_live, (__half*)ws.actA, (__half*)ws.actB, ws.logits, st)))
      return rc;
  } else if ((rc = xf::launch_fine_mlp(ctx, ws.X, (int)cap, n_live, ws.actA, ws.actB, ws.logits, st))) {
    return rc;
  }
  if (pairs)
    xf::refine_finish_kernel<true><<<wblocks, 256, 0, st>>>(ws.logits, d_kpts0, d_kpts1, d_scales0, (const long long*)d_idx0,
                                                            (const long long*)d_idx1, d_n_matches, ws.offsets, batch, n_max,
                                                            n1_max, fine_conf, ws.tmp, ws.keep, pairs);
  else
    xf::refine_finish_kernel<<<wblocks, 256, 0, st>>>(ws.logits, d_kpts0, d_kpts1, d_scales0, (const long long*)d_idx0,
                                                      (const long long*)d_idx1, d_n_matches, ws.offsets, batch, n_max, n1_max,
                                                      fine_conf, ws.tmp, ws.keep);
  XF_LAUNCH_CHECK();
  xf::refine_compact_kernel<<<batch, 1024, 0, st>>>(ws.tmp, ws.keep, d_n_matches, n_max, d_matches, d_n_refined);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_refine(xfeat_ctx* ctx, const float* d_desc0, const float* d_desc1, const float* d_kpts0,
                            const float* d_kpts1, const float* d_scales0, const int64_t* d_idx0, const int64_t* d_idx1,
                            const int32_t* d_n_matches, int batch, int n_max, int n1_max, float fine_conf, float* d_matches,
                            int32_t* d_n_refined, void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(ctx && d_desc0 && d_desc1 && d_kpts0 && d_kpts1 && d_scales0 && d_idx0 && d_idx1 && d_n_matches &&
                 d_matches && d_n_refined && d_ws,
             "refine: null pointer");
  XF_REQUIRE(batch > 0 && batch <= 65535 && n_max > 0 && n1_max > 0 && (int64_t)batch * n_max < (1ll << 31), "refine: bad sizes");
  return refine_impl(ctx, d_desc0, d_desc1, d_kpts0, d_kpts1, d_scales0, d_idx0, d_idx1, d_n_matches, batch, n_max, n1_max,
                     fine_conf, d_matches, d_n_refined, d_ws, ws_bytes, (cudaStream_t)stream, nullptr);
}

extern "C" size_t xfeat_refine_pairs_workspace_bytes(int n_pairs, int n_max) { return xfeat_refine_workspace_bytes(n_pairs, n_max); }

extern "C" int xfeat_refine_pairs(xfeat_ctx* ctx, const float* d_desc, const float* d_kpts, const float* d_scales, int n_max,
                                  const int32_t* d_pairs, const int64_t* d_idx0, const int64_t* d_idx1,
                                  const int32_t* d_n_matches, int n_pairs, float fine_conf, float* d_matches,
                                  int32_t* d_n_refined, void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(ctx && d_desc && d_kpts && d_scales && d_pairs && d_idx0 && d_idx1 && d_n_matches && d_matches && d_n_refined && d_ws,
             "refine_pairs: null pointer");
  XF_REQUIRE(n_pairs > 0 && n_pairs <= 65535 && n_max > 0 && (int64_t)n_pairs * n_max < (1ll << 31), "refine_pairs: bad sizes");
  XF_REQUIRE(((uintptr_t)d_pairs % 8) == 0, "refine_pairs: the pair table must be 8-byte aligned");
  return refine_impl(ctx, d_desc, d_desc, d_kpts, d_kpts, d_scales, d_idx0, d_idx1, d_n_matches, n_pairs, n_max, n_max, fine_conf,
                     d_matches, d_n_refined, d_ws, ws_bytes, (cudaStream_t)stream, reinterpret_cast<const int2*>(d_pairs));
}
