// Stand-alone forms of the reference's helper methods, for callers that use them directly (SURVEY 8b: the drop-in surface
// of modules/xfeat.py).  Inside detectAndCompute / match_xfeat_star the same arithmetic runs fused in the stage kernels
// (head_chain_tc.cu, sparse.cu, refine.cu); these entry points exist so that XFeat.get_kpts_heatmap, XFeat.NMS,
// XFeat.subpix_softmax2d and XFeat.net.fine_matcher are kernels of this library too, not PyTorch ops.
#include <cuda_fp16.h>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace xf {

// get_kpts_heatmap (xfeat.py:242-247): softmax over the 65 logits of a cell (x * temp), drop the dustbin, depth-to-space:
// heat[b, 8h+i, 8w+j] = p[b, 8i+j, h, w].  logits are NCHW (B,65,Hc,Wc); one thread per cell, channel loads coalesce across
// the warp (adjacent cells are adjacent in memory).
__global__ void __launch_bounds__(128) kpts_heatmap_kernel(const float* __restrict__ logits, int Hc, int Wc, float temp,
                                                           float* __restrict__ heat, int64_t ncell) {
  const int64_t cell = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= ncell) return;
  const int64_t plane = (int64_t)Hc * Wc;
  const int64_t b = cell / plane;
  const int rem = (int)(cell - b * plane);
  const int h = rem / Wc, w = rem - h * Wc;
  const float* lp = logits + b * 65 * plane + rem;
  float v[65];
  float mx = -INFINITY;
#pragma unroll
  for (int c = 0; c < 65; ++c) {
    v[c] = __fmul_rn(__ldg(lp + (int64_t)c * plane), temp);
    mx = fmaxf(mx, v[c]);
  }
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < 65; ++c) {
    v[c] = expf(v[c] - mx);
    sum += v[c];
  }
  const int W = Wc * 8;
  float* hp = heat + (b * Hc * 8 + (int64_t)h * 8) * W + (int64_t)w * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float4 a = make_float4(__fdiv_rn(v[8 * i], sum), __fdiv_rn(v[8 * i + 1], sum), __fdiv_rn(v[8 * i + 2], sum),
                           __fdiv_rn(v[8 * i + 3], sum));
    float4 c = make_float4(__fdiv_rn(v[8 * i + 4], sum), __fdiv_rn(v[8 * i + 5], sum), __fdiv_rn(v[8 * i + 6], sum),
                           __fdiv_rn(v[8 * i + 7], sum));
    reinterpret_cast<float4*>(hp + (int64_t)i * W)[0] = a;
    reinterpret_cast<float4*>(hp + (int64_t)i * W)[1] = c;
  }
}

// NMS (xfeat.py:249-263): pos = (x == maxpool_k(x)) & (x > thr), -inf padding.  Raster-ordered compaction in two passes over
// 1024-pixel chunks (one CTA each): pass 0 counts, the host-visible per-image totals size the output, pass 1 writes (x, y).
constexpr int NMSH_CHUNK = 1024;

__device__ __forceinline__ bool nms_is_max(const float* __restrict__ hb, int H, int W, int x, int y, int r, float thr) {
  const float v = __ldg(hb + (int64_t)y * W + x);
  if (!(v > thr)) return false;
  for (int dy = -r; dy <= r; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -r; dx <= r; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      // !(nb <= v), not nb > v: a NaN neighbour suppresses the pixel, as NaN propagates through the reference's max_pool2d
      if (!(__ldg(hb + (int64_t)yy * W + xx) <= v)) return false;
    }
  }
  return true;
}

// mode 0: chunk_counts[b][chunk] = maxima in the chunk.  mode 1: write positions at chunk_offsets[b][chunk] + rank.
__global__ void __launch_bounds__(NMSH_CHUNK) nms_helper_kernel(const float* __restrict__ heat, int H, int W, int r, float thr,
                                                               int mode, int* __restrict__ chunk_counts,
                                                               const int* __restrict__ chunk_offsets, long long* __restrict__ pos,
                                                               int pos_cap) {
  using Scan = cub::BlockScan<int, NMSH_CHUNK>;
  __shared__ typename Scan::TempStorage tmp;
  const int b = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int64_t p = (int64_t)chunk * NMSH_CHUNK + threadIdx.x;
  const float* hb = heat + (int64_t)b * H * W;
  int flag = 0, x = 0, y = 0;
  if (p < (int64_t)H * W) {
    y = (int)(p / W);
    x = (int)(p - (int64_t)y * W);
    flag = nms_is_max(hb, H, W, x, y, r, thr) ? 1 : 0;
  }
  if (mode == 0) {
    const int total = __syncthreads_count(flag);
    if (threadIdx.x == 0) chunk_counts[b * nchunk + chunk] = total;
    return;
  }
  int off, total;
  Scan(tmp).ExclusiveSum(flag, off, total);
  if (flag) {
    const int o = chunk_offsets[b * nchunk + chunk] + off;
    if (o < pos_cap) {
      pos[((int64_t)b * pos_cap + o) * 2] = x;
      pos[((int64_t)b * pos_cap + o) * 2 + 1] = y;
    }
  }
}

// per image: exclusive scan of the chunk counts; totals[b] = number of maxima
__global__ void __launch_bounds__(1024) nms_helper_scan_kernel(const int* __restrict__ counts, int nchunk, int* __restrict__ offsets,
                                                              int* __restrict__ totals) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_base;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  for (int i0 = 0; i0 < nchunk; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    const int c = (i < nchunk) ? counts[b * nchunk + i] : 0;
    int off, total;
    Scan(tmp).ExclusiveSum(c, off, total);
    const int base = s_base;
    if (i < nchunk) offsets[b * nchunk + i] = base + off;
    __syncthreads();
    if (threadIdx.x == 0) s_base = base + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[b] = s_base;
}

// subpix_softmax2d (xfeat.py:292-304): softmax(temp * h) over the 64 entries of an 8x8 map, expectation of (x - 4, y - 4),
// x the fast axis.  One warp per map, two entries per lane.
__global__ void __launch_bounds__(256) subpix_softmax2d_kernel(const float* __restrict__ maps, int64_t n, float temp,
                                                               float* __restrict__ out) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= n) return;
  const float2 o = __ldg(reinterpret_cast<const float2*>(maps + wid * 64) + lane);
  const float z0 = __fmul_rn(o.x, temp), z1 = __fmul_rn(o.y, temp);
  float mx = fmaxf(z0, z1);
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
  const float e0 = expf(z0 - mx), e1 = expf(z1 - mx);
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
    out[wid * 2] = sx / s;
    out[wid * 2 + 1] = sy / s;
  }
}


// InterpolateSparse2d.forward (interpolator.py:17-33): grid = 2 * pos / (W-1, H-1) - 1, F.grid_sample(align_corners=False,
// zeros padding) in mode nearest (0) / bilinear (1) / bicubic (2, A = -0.75).  x is NCHW (B,C,Hm,Wm), pos (B,N,2) fp32,
// out (B,N,C); one thread per output element, channel fastest (coalesced stores).
__device__ __forceinline__ float hl_cubic1(float x) { const float A = -0.75f; return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float hl_cubic2(float x) { const float A = -0.75f; return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
__device__ __forceinline__ float hl_src(float p, int size_pos, int size_map) {
  const float g = __fsub_rn(__fmul_rn(2.0f, __fdiv_rn(p, (float)(size_pos - 1))), 1.0f);
  return __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.0f), (float)size_map), 1.0f), 2.0f);
}
__global__ void __launch_bounds__(256) interpolate_sparse_kernel(const float* __restrict__ x, const float* __restrict__ pos, int C,
                                                                 int Hm, int Wm, int N, int H, int W, int mode,
                                                                 float* __restrict__ out, int64_t total) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int c = (int)(gid % C);
  const int64_t bn = gid / C;
  const int64_t b = bn / N;
  const float px = __ldg(pos + bn * 2), py = __ldg(pos + bn * 2 + 1);
  const float* xp = x + (b * C + c) * (int64_t)Hm * Wm;
  const float ix = hl_src(px, W, Wm), iy = hl_src(py, H, Hm);
  auto at = [&](int yy, int xx) -> float {
    return (yy >= 0 && yy < Hm && xx >= 0 && xx < Wm) ? __ldg(xp + (int64_t)yy * Wm + xx) : 0.f;
  };
  float o = 0.f;
  if (mode == 0) {
    o = at((int)rintf(iy), (int)rintf(ix));
  } else if (mode == 1) {
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float wx1 = __fsub_rn(ix, fx), wx0 = __fsub_rn(__fadd_rn(fx, 1.0f), ix);
    const float wy1 = __fsub_rn(iy, fy), wy0 = __fsub_rn(__fadd_rn(fy, 1.0f), iy);
    if (x0 >= 0 && x0 < Wm && y0 >= 0 && y0 < Hm) o = __fadd_rn(o, __fmul_rn(at(y0, x0), __fmul_rn(wx0, wy0)));
    if (x0 + 1 >= 0 && x0 + 1 < Wm && y0 >= 0 && y0 < Hm) o = __fadd_rn(o, __fmul_rn(at(y0, x0 + 1), __fmul_rn(wx1, wy0)));
    if (x0 >= 0 && x0 < Wm && y0 + 1 >= 0 && y0 + 1 < Hm) o = __fadd_rn(o, __fmul_rn(at(y0 + 1, x0), __fmul_rn(wx0, wy1)));
    if (x0 + 1 >= 0 && x0 + 1 < Wm && y0 + 1 >= 0 && y0 + 1 < Hm) o = __fadd_rn(o, __fmul_rn(at(y0 + 1, x0 + 1), __fmul_rn(wx1, wy1)));
  } else {
    const float fx = floorf(ix), fy = floorf(iy);
    const float tx = __fsub_rn(ix, fx), ty = __fsub_rn(iy, fy);
    const int x0 = (int)fx - 1, y0 = (int)fy - 1;
    const float cx[4] = {hl_cubic2(tx + 1.f), hl_cubic1(tx), hl_cubic1(1.f - tx), hl_cubic2((1.f - tx) + 1.f)};
    const float cy[4] = {hl_cubic2(ty + 1.f), hl_cubic1(ty), hl_cubic1(1.f - ty), hl_cubic2((1.f - ty) + 1.f)};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float rr = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) rr = fmaf(at(y0 + i, x0 + j), cx[j], rr);
      o = fmaf(rr, cy[i], o);
    }
  }
  out[gid] = o;
}

// fp32 rows (n, 128) -> split fp16 rows [hi(128) | lo(128)] for the tensor-core MLP; one warp per row
__global__ void __launch_bounds__(256) split_rows128_kernel(const float* __restrict__ x, int64_t n, __half* __restrict__ out) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= n) return;
  const float4 v = __ldg(reinterpret_cast<const float4*>(x + wid * 128) + lane);
  const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  __half2* o = reinterpret_cast<__half2*>(out + wid * 256);
  o[2 * lane] = h0;
  o[2 * lane + 1] = h1;
  o[64 + 2 * lane] = __floats2half2_rn(v.x - f0.x, v.y - f0.y);
  o[64 + 2 * lane + 1] = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
}

int launch_fine_mlp(const xfeat_ctx* ctx, const float* X, int rows_cap, const int* n_live, float* actA, float* actB,
                    float* logits, cudaStream_t st);

}  // namespace xf

extern "C" int xfeat_kpts_heatmap(const float* d_logits, int B, int Hc, int Wc, float softmax_temp, float* d_heat,
                                  void* stream) {
  XF_REQUIRE(d_logits && d_heat && B > 0 && Hc > 0 && Wc > 0, "kpts_heatmap: bad arguments");
  const int64_t ncell = (int64_t)B * Hc * Wc;
  xf::kpts_heatmap_kernel<<<(unsigned)((ncell + 127) / 128), 128, 0, (cudaStream_t)stream>>>(d_logits, Hc, Wc, softmax_temp,
                                                                                          d_heat, ncell);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" size_t xfeat_nms_workspace_bytes(int B, int H, int W) {
  const size_t nchunk = ((size_t)H * W + xf::NMSH_CHUNK - 1) / xf::NMSH_CHUNK;
  return 2 * xf::align_up((size_t)B * nchunk * sizeof(int), 256);
}

extern "C" int xfeat_nms_count(const float* d_heat, int B, int H, int W, int kernel_size, float threshold, int32_t* d_counts,
                               void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(d_heat && d_counts && d_ws && B > 0 && B <= 65535 && H > 0 && W > 0, "nms_count: bad arguments");
  XF_REQUIRE(kernel_size >= 1 && (kernel_size & 1), "nms: kernel_size must be odd (got %d)", kernel_size);
  XF_REQUIRE(ws_bytes >= xfeat_nms_workspace_bytes(B, H, W), "nms_count: workspace too small");
  const int nchunk = (int)(((size_t)H * W + xf::NMSH_CHUNK - 1) / xf::NMSH_CHUNK);
  int* counts = (int*)d_ws;
  int* offsets = (int*)((char*)d_ws + xf::align_up((size_t)B * nchunk * sizeof(int), 256));
  cudaStream_t st = (cudaStream_t)stream;
  xf::nms_helper_kernel<<<dim3(nchunk, B), xf::NMSH_CHUNK, 0, st>>>(d_heat, H, W, kernel_size / 2, threshold, 0, counts, nullptr,
                                                                    nullptr, 0);
  XF_LAUNCH_CHECK();
  xf::nms_helper_scan_kernel<<<B, 1024, 0, st>>>(counts, nchunk, offsets, d_counts);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_nms_write(const float* d_heat, int B, int H, int W, int kernel_size, float threshold, int64_t* d_pos,
                               int pos_cap, void* d_ws, size_t ws_bytes, void* stream) {
  // pos_cap 0 (every image empty) writes nothing: d_pos may then be the null pointer of an empty (B, 0, 2) tensor
  XF_REQUIRE(d_heat && (d_pos || pos_cap == 0) && d_ws && B > 0 && B <= 65535 && H > 0 && W > 0 && pos_cap >= 0,
             "nms_write: bad arguments");
  XF_REQUIRE(kernel_size >= 1 && (kernel_size & 1), "nms: kernel_size must be odd (got %d)", kernel_size);
  XF_REQUIRE(ws_bytes >= xfeat_nms_workspace_bytes(B, H, W), "nms_write: workspace too small");
  if (pos_cap == 0) return XF_OK;
  const int nchunk = (int)(((size_t)H * W + xf::NMSH_CHUNK - 1) / xf::NMSH_CHUNK);
  int* counts = (int*)d_ws;
  int* offsets = (int*)((char*)d_ws + xf::align_up((size_t)B * nchunk * sizeof(int), 256));
  xf::nms_helper_kernel<<<dim3(nchunk, B), xf::NMSH_CHUNK, 0, (cudaStream_t)stream>>>(
      d_heat, H, W, kernel_size / 2, threshold, 1, counts, offsets, (long long*)d_pos, pos_cap);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_subpix_softmax2d(const float* d_maps, int64_t n, float temp, float* d_out, void* stream) {
  XF_REQUIRE(n >= 0 && (n == 0 || (d_maps && d_out)), "subpix_softmax2d: bad arguments");   // n = 0: empty tensors, null
  if (n == 0) return XF_OK;
  xf::subpix_softmax2d_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_maps, n, temp, d_out);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" size_t xfeat_fine_matcher_workspace_bytes(int n) {
  const size_t rows = (size_t)(n > 0 ? n : 1);
  return 2 * xf::align_up(rows * 512 * sizeof(float), 256) + xf::align_up(rows * 256 * sizeof(__half), 256);
}

extern "C" int xfeat_fine_matcher(xfeat_ctx* ctx, const float* d_x, int n, float* d_out, void* d_ws, size_t ws_bytes,
                                  void* stream) {
  XF_REQUIRE(ctx && d_x && d_out && d_ws && n >= 0, "fine_matcher: bad arguments");
  XF_REQUIRE(ws_bytes >= xfeat_fine_matcher_workspace_bytes(n), "fine_matcher: workspace too small");
  if (n == 0) return XF_OK;
  XF_CUDA(cudaSetDevice(ctx->device));
  float* actA = (float*)d_ws;
  float* actB = (float*)((char*)d_ws + xf::align_up((size_t)n * 512 * sizeof(float), 256));
  if (xf::g_conv_impl != 0) {
    __half* xs = (__half*)((char*)d_ws + 2 * xf::align_up((size_t)n * 512 * sizeof(float), 256));
    xf::split_rows128_kernel<<<(unsigned)(((int64_t)n * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_x, n, xs);
    XF_LAUNCH_CHECK();
    return xf::launch_fine_mlp_tc(ctx, xs, n, nullptr, (__half*)actA, (__half*)actB, d_out, (cudaStream_t)stream);
  }
  return xf::launch_fine_mlp(ctx, d_x, n, nullptr, actA, actB, d_out, (cudaStream_t)stream);
}

extern "C" int xfeat_interpolate_sparse(const float* d_x, const float* d_pos, int B, int C, int Hm, int Wm, int N, int H, int W,
                                        int mode, float* d_out, void* stream) {
  XF_REQUIRE(d_x && (N == 0 || (d_pos && d_out)) && B > 0 && C > 0 && Hm > 0 && Wm > 0 && N >= 0 && mode >= 0 && mode <= 2,
             "interpolate_sparse: bad arguments");   // N = 0: pos and out are empty tensors, null
  const int64_t total = (int64_t)B * N * C;
  if (total == 0) return XF_OK;
  xf::interpolate_sparse_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_x, d_pos, C, Hm, Wm, N, H, W,
                                                                                                mode, d_out, total);
  XF_LAUNCH_CHECK();
  return XF_OK;
}
