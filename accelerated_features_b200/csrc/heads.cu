// Small fused kernels around the conv stack: pyramid fusion input (model.py:146-148), reliability head tail
// (heatmap_head.2 + sigmoid, model.py:82-83), keypoint head tail (keypoint_head.3 + softmax(65) + drop dustbin +
// 8x8 depth-to-space, model.py:91 + xfeat.py:242-247).
#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

// out = x3 + up2(x4) + up4(x5)   (NHWC, 64 channels; bilinear, align_corners=False; F.interpolate to x3's size)
__global__ void __launch_bounds__(256) fuse_pyramid_kernel(const float* __restrict__ x3, const float* __restrict__ x4,
                                                           const float* __restrict__ x5, float* __restrict__ out, int H3,
                                                           int W3, int H4, int W4, int H5, int W5, int64_t total4) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int c4 = (int)(i & 15);
  int64_t p = i >> 4;
  const int x = (int)(p % W3);
  p /= W3;
  const int y = (int)(p % H3);
  const int b = (int)(p / H3);
  float4 r = __ldg(reinterpret_cast<const float4*>(x3) + i);
  {
    const LinTap ty = lin_tap(y, (float)H4 / (float)H3, H4), tx = lin_tap(x, (float)W4 / (float)W3, W4);
    const float4* base = reinterpret_cast<const float4*>(x4) + (int64_t)b * H4 * W4 * 16 + c4;
    const float4 v00 = __ldg(base + ((int64_t)ty.i0 * W4 + tx.i0) * 16), v01 = __ldg(base + ((int64_t)ty.i0 * W4 + tx.i1) * 16);
    const float4 v10 = __ldg(base + ((int64_t)ty.i1 * W4 + tx.i0) * 16), v11 = __ldg(base + ((int64_t)ty.i1 * W4 + tx.i1) * 16);
#define XF_BIL(f) (ty.l0 * (tx.l0 * v00.f + tx.l1 * v01.f) + ty.l1 * (tx.l0 * v10.f + tx.l1 * v11.f))
    r.x += XF_BIL(x); r.y += XF_BIL(y); r.z += XF_BIL(z); r.w += XF_BIL(w);
  }
  {
    const LinTap ty = lin_tap(y, (float)H5 / (float)H3, H5), tx = lin_tap(x, (float)W5 / (float)W3, W5);
    const float4* base = reinterpret_cast<const float4*>(x5) + (int64_t)b * H5 * W5 * 16 + c4;
    const float4 v00 = __ldg(base + ((int64_t)ty.i0 * W5 + tx.i0) * 16), v01 = __ldg(base + ((int64_t)ty.i0 * W5 + tx.i1) * 16);
    const float4 v10 = __ldg(base + ((int64_t)ty.i1 * W5 + tx.i0) * 16), v11 = __ldg(base + ((int64_t)ty.i1 * W5 + tx.i1) * 16);
    r.x += XF_BIL(x); r.y += XF_BIL(y); r.z += XF_BIL(z); r.w += XF_BIL(w);
#undef XF_BIL
  }
  reinterpret_cast<float4*>(out)[i] = r;
}

// reliability = sigmoid(t . w + b), t: (npix,64) NHWC. 8 lanes per pixel, 8 channels per lane.
__global__ void __launch_bounds__(256) reliability_kernel(const float* __restrict__ t, const float* __restrict__ w,
                                                          const float* __restrict__ bias, float* __restrict__ out,
                                                          int64_t npix) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t pix = gid >> 3;
  const int sub = (int)(gid & 7);
  float s = 0.f;
  if (pix < npix) {
    const float4* tp = reinterpret_cast<const float4*>(t + pix * 64) + sub * 2;
    const float4* wp = reinterpret_cast<const float4*>(w) + sub * 2;
    const float4 a0 = __ldg(tp), a1 = __ldg(tp + 1), w0 = __ldg(wp), w1 = __ldg(wp + 1);
    s = a0.x * w0.x + a0.y * w0.y + a0.z * w0.z + a0.w * w0.w + a1.x * w1.x + a1.y * w1.y + a1.z * w1.z + a1.w * w1.w;
  }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (pix < npix && sub == 0) {
    const float z = s + __ldg(bias);
    out[pix] = 1.0f / (1.0f + expf(-z));
  }
}

// keypoint_head.3 (64->65, bias) + softmax over the 65 logits + heat[b, 8h+i, 8w+j] = p[8i+j].
// A warp handles KPT_CPW consecutive cells per pass: their 64-vectors are staged k-major in shared memory so one
// 128-bit broadcast load feeds 4 cells; weights [64][65] (stride 65: conflict-free along the output-channel axis)
// are shared by the 4 cells -> 4 LDS per 12 FFMA.
constexpr int KPT_WARPS = 8, KPT_CPW = 4;
__global__ void __launch_bounds__(KPT_WARPS * 32) kpt_softmax_kernel(const float* __restrict__ t,
                                                                     const float* __restrict__ w,
                                                                     const float* __restrict__ bias,
                                                                     float* __restrict__ heat,
                                                                     float* __restrict__ logits_out, int Hc, int Wc,
                                                                     int64_t ncell) {
  __shared__ float sW[64 * 65];
  __shared__ float sB[65];
  __shared__ __align__(16) float sT[KPT_WARPS][64][KPT_CPW];
  for (int i = threadIdx.x; i < 64 * 65; i += blockDim.x) sW[i] = __ldg(w + i);
  if (threadIdx.x < 65) sB[threadIdx.x] = __ldg(bias + threadIdx.x);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int W = Wc * 8;
  const int64_t ngroup = (ncell + KPT_CPW - 1) / KPT_CPW;
  for (int64_t grp = (int64_t)blockIdx.x * KPT_WARPS + warp; grp < ngroup; grp += (int64_t)gridDim.x * KPT_WARPS) {
    const int64_t cell0 = grp * KPT_CPW;
    __syncwarp();
#pragma unroll
    for (int c = 0; c < KPT_CPW; ++c) {
      float2 tv = make_float2(0.f, 0.f);
      if (cell0 + c < ncell) tv = __ldg(reinterpret_cast<const float2*>(t + (cell0 + c) * 64) + lane);
      sT[warp][2 * lane][c] = tv.x;
      sT[warp][2 * lane + 1][c] = tv.y;
    }
    __syncwarp();
    float l0[KPT_CPW], l1[KPT_CPW], l2[KPT_CPW];
#pragma unroll
    for (int c = 0; c < KPT_CPW; ++c) { l0[c] = sB[lane]; l1[c] = sB[lane + 32]; l2[c] = sB[64]; }
#pragma unroll 8
    for (int k = 0; k < 64; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&sT[warp][k][0]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
      const float w0 = sW[k * 65 + lane], w1 = sW[k * 65 + lane + 32], w2 = sW[k * 65 + 64];
#pragma unroll
      for (int c = 0; c < KPT_CPW; ++c) {
        l0[c] = fmaf(a[c], w0, l0[c]);
        l1[c] = fmaf(a[c], w1, l1[c]);
        l2[c] = fmaf(a[c], w2, l2[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < KPT_CPW; ++c) {
      const int64_t cell = cell0 + c;
      if (cell >= ncell) break;  // warp-uniform
      if (logits_out) {
        float* lo = logits_out + cell * 65;
        lo[lane] = l0[c];
        lo[lane + 32] = l1[c];
        if (lane == 0) lo[64] = l2[c];
      }
      float m = fmaxf(fmaxf(l0[c], l1[c]), l2[c]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const float e0 = expf(l0[c] - m), e1 = expf(l1[c] - m), e2 = expf(l2[c] - m);
      float s = e0 + e1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      s += e2;
      const int64_t b = cell / ((int64_t)Hc * Wc);
      const int rem = (int)(cell - b * Hc * Wc);
      const int h = rem / Wc, wc = rem - h * Wc;
      // channel c = 8i + j -> pixel (8h+i, 8wc+j): lane -> (i = lane>>3, j = lane&7), second half i += 4
      float* hp = heat + ((int64_t)b * Hc * 8 + h * 8 + (lane >> 3)) * W + wc * 8 + (lane & 7);
      hp[0] = e0 / s;
      hp[(int64_t)4 * W] = e1 / s;
    }
  }
}

// Same fusion, but x3 / x4 / x5 arrive as split fp16 [hi(64) | lo(64)] (x = hi + lo) straight from the tensor-core layers, so
// block3.2 / block4.2 / block5.3 need not write a second, fp32 copy of their output.
// 16 channels per thread: 32 bytes of the hi and of the lo halves per load call (two 128-bit read-only loads each).
struct F16v {
  float v[16];
};
__device__ __forceinline__ void ld_v8_nc(const void* p, uint32_t (&r)[8]) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ F16v ld_split16(const __half* __restrict__ base, int64_t pix, int c16) {
  uint32_t hw[8], lw[8];
  ld_v8_nc(base + pix * 128 + c16 * 16, hw);
  ld_v8_nc(base + pix * 128 + 64 + c16 * 16, lw);
  F16v r;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hw[i])), c = __half22float2(*reinterpret_cast<const __half2*>(&lw[i]));
    r.v[2 * i] = a.x + c.x;
    r.v[2 * i + 1] = a.y + c.y;
  }
  return r;
}
__global__ void __launch_bounds__(256) fuse_pyramid_split_kernel(const __half* __restrict__ x3, const __half* __restrict__ x4,
                                                                 const __half* __restrict__ x5, __half* __restrict__ out_split,
                                                                 int H3, int W3, int H4, int W4, int H5, int W5, int64_t total16) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total16) return;
  const int c16 = (int)(i & 3);
  int64_t p = i >> 2;
  const int x = (int)(p % W3);
  p /= W3;
  const int y = (int)(p % H3);
  const int b = (int)(p / H3);
  F16v r = ld_split16(x3, i >> 2, c16);
  {
    const LinTap ty = lin_tap(y, (float)H4 / (float)H3, H4), tx = lin_tap(x, (float)W4 / (float)W3, W4);
    const int64_t bb = (int64_t)b * H4 * W4;
    const F16v v00 = ld_split16(x4, bb + (int64_t)ty.i0 * W4 + tx.i0, c16), v01 = ld_split16(x4, bb + (int64_t)ty.i0 * W4 + tx.i1, c16);
    const F16v v10 = ld_split16(x4, bb + (int64_t)ty.i1 * W4 + tx.i0, c16), v11 = ld_split16(x4, bb + (int64_t)ty.i1 * W4 + tx.i1, c16);
#pragma unroll
    for (int k = 0; k < 16; ++k) r.v[k] += ty.l0 * (tx.l0 * v00.v[k] + tx.l1 * v01.v[k]) + ty.l1 * (tx.l0 * v10.v[k] + tx.l1 * v11.v[k]);
  }
  {
    const LinTap ty = lin_tap(y, (float)H5 / (float)H3, H5), tx = lin_tap(x, (float)W5 / (float)W3, W5);
    const int64_t bb = (int64_t)b * H5 * W5;
    const F16v v00 = ld_split16(x5, bb + (int64_t)ty.i0 * W5 + tx.i0, c16), v01 = ld_split16(x5, bb + (int64_t)ty.i0 * W5 + tx.i1, c16);
    const F16v v10 = ld_split16(x5, bb + (int64_t)ty.i1 * W5 + tx.i0, c16), v11 = ld_split16(x5, bb + (int64_t)ty.i1 * W5 + tx.i1, c16);
#pragma unroll
    for (int k = 0; k < 16; ++k) r.v[k] += ty.l0 * (tx.l0 * v00.v[k] + tx.l1 * v01.v[k]) + ty.l1 * (tx.l0 * v10.v[k] + tx.l1 * v11.v[k]);
  }
  __half* hp = out_split + (i >> 2) * 128 + c16 * 16;
  tc::store_split_row<16>(hp, hp + 64, r.v);
}

int launch_fuse_pyramid_split(const __half* x3, const __half* x4, const __half* x5, __half* out_split, int B, int H3, int W3,
                              cudaStream_t st) {
  const int64_t total16 = (int64_t)B * H3 * W3 * 4;
  fuse_pyramid_split_kernel<<<(unsigned)((total16 + 255) / 256), 256, 0, st>>>(x3, x4, x5, out_split, H3, W3, H3 / 2, W3 / 2, H3 / 4,
                                                                                W3 / 4, total16);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

int launch_fuse_pyramid(const float* x3, const float* x4, const float* x5, float* out, int B, int H3, int W3, cudaStream_t st) {
  const int64_t total4 = (int64_t)B * H3 * W3 * 16;
  fuse_pyramid_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, st>>>(x3, x4, x5, out, H3, W3, H3 / 2, W3 / 2, H3 / 4, W3 / 4,
                                                                         total4);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

int launch_reliability(const xfeat_ctx* ctx, const float* t, float* out, int64_t npix, cudaStream_t st) {
  const float* w = ctx->d_weights + ctx->table.w_off[L_HH_2];
  const float* b = ctx->d_weights + ctx->table.b_off[L_HH_2];
  reliability_kernel<<<(unsigned)((npix * 8 + 255) / 256), 256, 0, st>>>(t, w, b, out, npix);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

int launch_kpt_softmax(const xfeat_ctx* ctx, const float* t, float* heat, float* logits, int B, int Hc, int Wc,
                       cudaStream_t st) {
  const float* w = ctx->d_weights + ctx->table.w_off[L_KH_3];
  const float* b = ctx->d_weights + ctx->table.b_off[L_KH_3];
  const int64_t ncell = (int64_t)B * Hc * Wc;
  const int64_t ngroup = (ncell + KPT_CPW - 1) / KPT_CPW;
  const int blocks = (int)std::min<int64_t>((ngroup + KPT_WARPS - 1) / KPT_WARPS, (int64_t)ctx->sm_count * 8);
  kpt_softmax_kernel<<<blocks, KPT_WARPS * 32, 0, st>>>(t, w, b, heat, logits, Hc, Wc, ncell);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf
