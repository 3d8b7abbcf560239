// Image ingest: bilinear resize, channel mean, per-image instance normalisation.
// Reference: preprocess_tensor (xfeat.py:219-240), XFeatModel.forward normalisation (model.py:135-136),
// extract_dualscale's F.interpolate (xfeat.py:380-381).  All HBM-bound streaming kernels.
#include <atomic>

#include "common.cuh"

namespace xf {

template <int DTYPE>
__device__ __forceinline__ float load_px(const void* p, int64_t off, int div255) {
  float v;
  if (DTYPE == XF_DTYPE_U8) v = (float)((const unsigned char*)p)[off];
  else v = __ldg((const float*)p + off);
  if (div255) v = __fdiv_rn(v, 255.0f);
  return v;
}

// One thread per output pixel: bilinear sample of every channel (ATen upsample_bilinear2d arithmetic), mean over
// channels, write gray; block-reduce sum / sum-of-squares in double -> atomicAdd into stats[b] = {sum, sumsq}.
template <int DTYPE>
__global__ void __launch_bounds__(256) gray_resize_kernel(const void* __restrict__ img, int C, int Hi, int Wi,
                                                          int64_t sb, int64_t sc, int64_t sh, int64_t sw, int div255,
                                                          int H, int W, float scale_h, float scale_w,
                                                          float* __restrict__ gray, double* __restrict__ stats) {
  const int b = blockIdx.z;
  const int x = blockIdx.x * 64 + (threadIdx.x & 63);
  const int y = blockIdx.y * 4 + (threadIdx.x >> 6);
  float g = 0.f;
  const bool in = (x < W) && (y < H);
  if (in) {
    const LinTap ty = lin_tap(y, scale_h, Hi);
    const LinTap tx = lin_tap(x, scale_w, Wi);
    const int64_t base = (int64_t)b * sb;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) {
      const int64_t bc = base + (int64_t)c * sc;
      const float v00 = load_px<DTYPE>(img, bc + ty.i0 * sh + tx.i0 * sw, div255);
      const float v01 = load_px<DTYPE>(img, bc + ty.i0 * sh + tx.i1 * sw, div255);
      const float v10 = load_px<DTYPE>(img, bc + ty.i1 * sh + tx.i0 * sw, div255);
      const float v11 = load_px<DTYPE>(img, bc + ty.i1 * sh + tx.i1 * sw, div255);
      // ATen: l0h*(l0w*v00 + l1w*v01) + l1h*(l0w*v10 + l1w*v11)
      const float top = __fadd_rn(__fmul_rn(tx.l0, v00), __fmul_rn(tx.l1, v01));
      const float bot = __fadd_rn(__fmul_rn(tx.l0, v10), __fmul_rn(tx.l1, v11));
      const float v = __fadd_rn(__fmul_rn(ty.l0, top), __fmul_rn(ty.l1, bot));
      acc = __fadd_rn(acc, v);
    }
    g = (C == 1) ? acc : __fdiv_rn(acc, (float)C);
    gray[((int64_t)b * H + y) * W + x] = g;
  }
  double s = in ? (double)g : 0.0, ss = in ? (double)g * (double)g : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  __shared__ double sh_s[8], sh_ss[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sh_s[warp] = s; sh_ss[warp] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c2 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += sh_s[i]; c2 += sh_ss[i]; }
    atomicAdd(&stats[2 * b], a);
    atomicAdd(&stats[2 * b + 1], c2);
  }
}

// gray_resize_kernel for fp32 planes with unit pixel stride (the dual-scale star path resizes 64 x 3 x 960 x 1280 four times per
// step): one thread owns 4 consecutive output columns x GRX_ROWS rows, so the 4 column taps are computed once and reused for every
// row and channel, the 16 loads of a (row, channel) are issued together, offsets inside an image are 32-bit, the output is one
// 128-bit store per row and the fp64 statistics take one atomic pair per 64 x 16 pixel block.  Per-pixel arithmetic is the
// generic kernel's (ATen upsample_bilinear2d order), so the two produce identical bits.
constexpr int GRX_ROWS = 4;
__global__ void __launch_bounds__(256) gray_resize_f32x4_kernel(const float* __restrict__ img, int C, int Hi, int Wi, int64_t sb,
                                                                int sc, int sh, int div255, int H, int W4, float scale_h,
                                                                float scale_w, float* __restrict__ gray,
                                                                double* __restrict__ stats) {
  const int b = blockIdx.z;
  const int x4 = blockIdx.x * 64 + (threadIdx.x & 63);
  const bool in = x4 < W4;
  const float* pb = img + (int64_t)b * sb;
  LinTap tx[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) tx[j] = lin_tap(in ? 4 * x4 + j : 0, scale_w, Wi);
  double s = 0.0, ss = 0.0;
  const float fc = (float)C;
#pragma unroll 1
  for (int r = 0; r < GRX_ROWS; ++r) {
    const int y = (blockIdx.y * GRX_ROWS + r) * 4 + (threadIdx.x >> 6);
    if (!in || y >= H) continue;
    const LinTap ty = lin_tap(y, scale_h, Hi);
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < C; ++c) {
      const float* r0 = pb + (c * sc + ty.i0 * sh);
      const float* r1 = pb + (c * sc + ty.i1 * sh);
      float v00[4], v01[4], v10[4], v11[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v00[j] = __ldg(r0 + tx[j].i0); v01[j] = __ldg(r0 + tx[j].i1);
        v10[j] = __ldg(r1 + tx[j].i0); v11[j] = __ldg(r1 + tx[j].i1);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (div255) {
          v00[j] = __fdiv_rn(v00[j], 255.f); v01[j] = __fdiv_rn(v01[j], 255.f);
          v10[j] = __fdiv_rn(v10[j], 255.f); v11[j] = __fdiv_rn(v11[j], 255.f);
        }
        const float top = __fadd_rn(__fmul_rn(tx[j].l0, v00[j]), __fmul_rn(tx[j].l1, v01[j]));
        const float bot = __fadd_rn(__fmul_rn(tx[j].l0, v10[j]), __fmul_rn(tx[j].l1, v11[j]));
        g[j] = __fadd_rn(g[j], __fadd_rn(__fmul_rn(ty.l0, top), __fmul_rn(ty.l1, bot)));
      }
    }
    if (C != 1) {
#pragma unroll
      for (int j = 0; j < 4; ++j) g[j] = __fdiv_rn(g[j], fc);
    }
    reinterpret_cast<float4*>(gray + ((int64_t)b * H + y) * (4 * (int64_t)W4))[x4] = make_float4(g[0], g[1], g[2], g[3]);
    s += ((double)g[0] + (double)g[1]) + ((double)g[2] + (double)g[3]);
    ss += ((double)g[0] * g[0] + (double)g[1] * g[1]) + ((double)g[2] * g[2] + (double)g[3] * g[3]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  __shared__ double sh_s[8], sh_ss[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sh_s[warp] = s; sh_ss[warp] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c2 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += sh_s[i]; c2 += sh_ss[i]; }
    atomicAdd(&stats[2 * b], a);
    atomicAdd(&stats[2 * b + 1], c2);
  }
}

// Fast path of gray_resize_kernel for the common case (BASELINE configs): fp32 input already at network resolution
// (the bilinear resize is the identity: src == dst, lambda == 0), unit pixel stride, 16-byte aligned rows.
// The image is walked as a linear array of 4-pixel groups (a 2-D block tiling left 7/8 of every second block idle at W = 640),
// 4 groups per thread, and the loads of up to 4 channels x 4 groups are all issued before the first use; same per-pixel
// arithmetic as the generic kernel restricted to that case.
constexpr int GI_NPT = 4;
__global__ void __launch_bounds__(256) gray_identity_f32_kernel(const float* __restrict__ img, int C, int64_t sb, int64_t sc,
                                                                int64_t sh, int div255, int H, int W4,
                                                                float* __restrict__ gray, double* __restrict__ stats) {
  const int b = blockIdx.z;
  const unsigned n4 = (unsigned)H * (unsigned)W4;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  unsigned e[GI_NPT];
  bool in[GI_NPT];
  const float* p[GI_NPT];
  float4 g[GI_NPT];
#pragma unroll
  for (int k = 0; k < GI_NPT; ++k) {
    e[k] = ((unsigned)blockIdx.x * GI_NPT + k) * 256u + threadIdx.x;
    in[k] = e[k] < n4;
    const unsigned y = in[k] ? e[k] / (unsigned)W4 : 0u, x4 = in[k] ? e[k] - y * (unsigned)W4 : 0u;
    p[k] = img + (int64_t)b * sb + (int64_t)y * sh + 4 * x4;
    g[k] = zero4;
  }
  for (int c0 = 0; c0 < C; c0 += 4) {
    float4 l[4][GI_NPT];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int k = 0; k < GI_NPT; ++k)
        l[u][k] = (c0 + u < C && in[k]) ? __ldg(reinterpret_cast<const float4*>(p[k] + (int64_t)(c0 + u) * sc)) : zero4;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (c0 + u < C) {
#pragma unroll
        for (int k = 0; k < GI_NPT; ++k) {
          float4 v = l[u][k];
          if (div255) { v.x = __fdiv_rn(v.x, 255.f); v.y = __fdiv_rn(v.y, 255.f); v.z = __fdiv_rn(v.z, 255.f); v.w = __fdiv_rn(v.w, 255.f); }
          g[k].x = __fadd_rn(g[k].x, v.x); g[k].y = __fadd_rn(g[k].y, v.y); g[k].z = __fadd_rn(g[k].z, v.z); g[k].w = __fadd_rn(g[k].w, v.w);
        }
      }
    }
  }
  double s = 0.0, ss = 0.0;
  float4* out = reinterpret_cast<float4*>(gray + (int64_t)b * H * W4 * 4);
#pragma unroll
  for (int k = 0; k < GI_NPT; ++k) {
    if (C != 1) {
      const float fc = (float)C;
      g[k].x = __fdiv_rn(g[k].x, fc); g[k].y = __fdiv_rn(g[k].y, fc); g[k].z = __fdiv_rn(g[k].z, fc); g[k].w = __fdiv_rn(g[k].w, fc);
    }
    if (in[k]) out[e[k]] = g[k];     // out-of-range groups hold zeros and add nothing to the sums
    s += ((double)g[k].x + (double)g[k].y) + ((double)g[k].z + (double)g[k].w);
    ss += (double)g[k].x * g[k].x + (double)g[k].y * g[k].y + (double)g[k].z * g[k].z + (double)g[k].w * g[k].w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  __shared__ double sh_s[8], sh_ss[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sh_s[warp] = s; sh_ss[warp] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c2 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += sh_s[i]; c2 += sh_ss[i]; }
    atomicAdd(&stats[2 * b], a);
    atomicAdd(&stats[2 * b + 1], c2);
  }
}

// Fast path for camera-style input: uint8 HWC (3 interleaved channels, e.g. cv2 BGR), already at network resolution.
// 4 pixels (12 bytes = three aligned 32-bit words) per thread; same arithmetic as the generic kernel:
// per channel float(u8)/255 (parse_input, xfeat.py:400-401), channel sum, /3 (model.py:135).
__global__ void __launch_bounds__(256) gray_identity_u8hwc_kernel(const unsigned char* __restrict__ img, int64_t sb, int64_t sh,
                                                                  int div255, int H, int W4, float* __restrict__ gray,
                                                                  double* __restrict__ stats) {
  const int b = blockIdx.z;
  const int x4 = blockIdx.x * 64 + (threadIdx.x & 63);
  const int y = blockIdx.y * 4 + (threadIdx.x >> 6);
  const bool in = (x4 < W4) && (y < H);
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (in) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(img + (int64_t)b * sb + (int64_t)y * sh) + 3 * x4;
    const uint32_t w0 = __ldg(p), w1 = __ldg(p + 1), w2 = __ldg(p + 2);
    const unsigned char by[12] = {(unsigned char)(w0), (unsigned char)(w0 >> 8), (unsigned char)(w0 >> 16), (unsigned char)(w0 >> 24),
                                  (unsigned char)(w1), (unsigned char)(w1 >> 8), (unsigned char)(w1 >> 16), (unsigned char)(w1 >> 24),
                                  (unsigned char)(w2), (unsigned char)(w2 >> 8), (unsigned char)(w2 >> 16), (unsigned char)(w2 >> 24)};
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = (float)by[3 * i + c];
        if (div255) v = __fdiv_rn(v, 255.f);
        acc = __fadd_rn(acc, v);
      }
      o[i] = __fdiv_rn(acc, 3.f);
    }
    g = make_float4(o[0], o[1], o[2], o[3]);
    reinterpret_cast<float4*>(gray + ((int64_t)b * H + y) * (W4 * 4))[x4] = g;
  }
  double s = (double)g.x + (double)g.y + (double)g.z + (double)g.w;
  double ss = (double)g.x * g.x + (double)g.y * g.y + (double)g.z * g.z + (double)g.w * g.w;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  __shared__ double sh_s[8], sh_ss[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sh_s[warp] = s; sh_ss[warp] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c2 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += sh_s[i]; c2 += sh_ss[i]; }
    atomicAdd(&stats[2 * b], a);
    atomicAdd(&stats[2 * b + 1], c2);
  }
}

// InstanceNorm2d(1) parameters from the fp64 (sum, sum of squares) of n pixels: biased variance sum_sq / n - mean^2 (clamped at
// 0), then mean and 1 / sqrt(var + 1e-5) rounded to float.  Both forms below call this, and every double operation is rounded on
// its own: left to the compiler, sum_sq / n - mean * mean was contracted into an FMA in one kernel and not in the other, and for
// a low-contrast image (mean^2 close to sum_sq / n) the two forms disagreed in the last bit of invstd.
__device__ __forceinline__ void instnorm_params(double sum, double sum_sq, double n, float& meanf, float& invstd) {
  const double mean = sum / n;
  double var = __dsub_rn(sum_sq / n, __dmul_rn(mean, mean));
  if (var < 0) var = 0;
  meanf = (float)mean;
  invstd = (float)(1.0 / sqrt(var + 1e-5));
}

// Gray conversion + InstanceNorm in ONE pass for images at network resolution that fit the shared memory of a thread-block
// cluster (VGA: 1.2 MB of gray = 16 CTAs x 75 KB, two CTAs per SM so that clusters in different phases overlap).  A cluster owns an image: every CTA converts its share into shared memory
// and sums it (fp64), the partial sums are exchanged through distributed shared memory (read in rank order by every CTA:
// the statistics are deterministic, unlike the atomics of the two-kernel form), and the normalised values are written from
// shared memory.  The gray image is never written to / re-read from HBM: 16 B in + 4 B out per pixel instead of 16 + 4 + 4 + 4.
// Per-pixel arithmetic is that of gray_identity_f32_kernel and instnorm_kernel.  (The uint8 ingest keeps the two-kernel form:
// measured through the streaming pipeline it is 3-4 % faster there, bench.py e2e_u8.)
constexpr int GN_THREADS = 512;   // cluster of 16 (non-portable size, 2 CTAs per SM) when a sixteenth fits 100 KB, else 8
constexpr size_t GN_MAX_SMEM = 200 * 1024, GN_SMEM_2PER_SM = 100 * 1024;

__device__ __forceinline__ double ld_dsmem_f64(uint32_t cluster_addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(cluster_addr));
  return v;
}
__device__ __forceinline__ uint32_t gn_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void gn_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__global__ void __launch_bounds__(GN_THREADS, 2)
    gray_norm_cluster_kernel(const float* __restrict__ img, int C, int64_t sb, int64_t sc, int64_t sh, int div255, int H, int W4,
                             float* __restrict__ xn, double* __restrict__ stats) {
  extern __shared__ float4 sG[];            // this CTA's share of the gray image, 4-pixel groups
  __shared__ double sRed[2][GN_THREADS / 32];
  __shared__ double sPart[2];               // this CTA's (sum, sum of squares): read by the whole cluster
  __shared__ float sNorm[2];
  const int b = blockIdx.y, tid = threadIdx.x;
  const unsigned rank = gn_cluster_rank(), nranks = gridDim.x;        // the cluster spans grid.x
  const unsigned per = (unsigned)H * (unsigned)W4 / nranks, e0 = rank * per;
  constexpr int U = 2;   // 4-pixel groups per thread and trip: 96 B of loads in flight per thread at 3 channels
  double s = 0.0, ss = 0.0;
  for (unsigned i0 = 0; i0 < per; i0 += U * GN_THREADS) {
    float4 g[U];
    bool in[U];
    {
      const float* p[U];
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const unsigned i = i0 + k * GN_THREADS + tid;
        in[k] = i < per;
        const unsigned e = in[k] ? e0 + i : e0;
        const unsigned y = e / (unsigned)W4, x4 = e - y * (unsigned)W4;
        p[k] = img + (int64_t)b * sb + (int64_t)y * sh + 4 * x4;
        g[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      for (int c0 = 0; c0 < C; c0 += 4) {
        float4 l[4][U];
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int k = 0; k < U; ++k)
            l[u][k] = (c0 + u < C && in[k]) ? __ldg(reinterpret_cast<const float4*>(p[k] + (int64_t)(c0 + u) * sc))
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (c0 + u < C) {
#pragma unroll
            for (int k = 0; k < U; ++k) {
              float4 v = l[u][k];
              if (div255) { v.x = __fdiv_rn(v.x, 255.f); v.y = __fdiv_rn(v.y, 255.f); v.z = __fdiv_rn(v.z, 255.f); v.w = __fdiv_rn(v.w, 255.f); }
              g[k].x = __fadd_rn(g[k].x, v.x); g[k].y = __fadd_rn(g[k].y, v.y); g[k].z = __fadd_rn(g[k].z, v.z); g[k].w = __fadd_rn(g[k].w, v.w);
            }
          }
        }
      }
      if (C != 1) {
        const float fc = (float)C;
#pragma unroll
        for (int k = 0; k < U; ++k) {
          g[k].x = __fdiv_rn(g[k].x, fc); g[k].y = __fdiv_rn(g[k].y, fc); g[k].z = __fdiv_rn(g[k].z, fc); g[k].w = __fdiv_rn(g[k].w, fc);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (in[k]) {
        sG[i0 + k * GN_THREADS + tid] = g[k];
        s += ((double)g[k].x + (double)g[k].y) + ((double)g[k].z + (double)g[k].w);
        ss += (double)g[k].x * g[k].x + (double)g[k].y * g[k].y + (double)g[k].z * g[k].z + (double)g[k].w * g[k].w;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  const int warp = tid >> 5, lane = tid & 31;
  if (lane == 0) { sRed[0][warp] = s; sRed[1][warp] = ss; }
  __syncthreads();
  if (tid == 0) {
    double a = 0, c2 = 0;
    for (int i = 0; i < GN_THREADS / 32; ++i) { a += sRed[0][i]; c2 += sRed[1][i]; }
    sPart[0] = a; sPart[1] = c2;
  }
  gn_cluster_sync();                                   // every CTA's partial sums are visible cluster-wide
  if (tid == 0) {
    const uint32_t a0 = (uint32_t)__cvta_generic_to_shared(&sPart[0]), a1 = (uint32_t)__cvta_generic_to_shared(&sPart[1]);
    double sum = 0, sq = 0;
    for (unsigned r = 0; r < nranks; ++r) {             // rank order: the same value in every CTA, run to run
      uint32_t ra, rb;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a0), "r"(r));
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(a1), "r"(r));
      sum += ld_dsmem_f64(ra);
      sq += ld_dsmem_f64(rb);
    }
    instnorm_params(sum, sq, (double)H * (double)W4 * 4.0, sNorm[0], sNorm[1]);
    if (rank == 0) { stats[2 * b] = sum; stats[2 * b + 1] = sq; }
  }
  __syncthreads();
  const float meanf = sNorm[0], invstd = sNorm[1];
  float4* out = reinterpret_cast<float4*>(xn) + (int64_t)b * H * W4 + e0;
  for (unsigned i = tid; i < per; i += GN_THREADS) {
    float4 v = sG[i];
    v.x = __fmul_rn(__fsub_rn(v.x, meanf), invstd);
    v.y = __fmul_rn(__fsub_rn(v.y, meanf), invstd);
    v.z = __fmul_rn(__fsub_rn(v.z, meanf), invstd);
    v.w = __fmul_rn(__fsub_rn(v.w, meanf), invstd);
    out[i] = v;
  }
  gn_cluster_sync();                                   // no CTA leaves while its partial sums may still be read
}

// InstanceNorm2d(1): (g - mean) * rsqrt(var_biased + 1e-5), float4 vectorised, in place.
__global__ void __launch_bounds__(256) instnorm_kernel(float* __restrict__ gray, const double* __restrict__ stats,
                                                       int HW4) {
  const int b = blockIdx.y;
  float meanf, invstd;
  instnorm_params(stats[2 * b], stats[2 * b + 1], (double)HW4 * 4.0, meanf, invstd);
  float4* p = reinterpret_cast<float4*>(gray) + (int64_t)b * HW4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW4; i += gridDim.x * blockDim.x) {
    float4 v = p[i];
    v.x = __fmul_rn(__fsub_rn(v.x, meanf), invstd);
    v.y = __fmul_rn(__fsub_rn(v.y, meanf), invstd);
    v.z = __fmul_rn(__fsub_rn(v.z, meanf), invstd);
    v.w = __fmul_rn(__fsub_rn(v.w, meanf), invstd);
    p[i] = v;
  }
}

template <int DTYPE>
__global__ void __launch_bounds__(256) resize_bilinear_kernel(const void* __restrict__ in, int C, int Hi, int Wi,
                                                              int64_t sb, int64_t sc, int64_t sh, int64_t sw, int div255,
                                                              float* __restrict__ out, int Ho, int Wo, float scale_h,
                                                              float scale_w) {
  const int plane = blockIdx.z;  // b*C + c
  const int x = blockIdx.x * 64 + (threadIdx.x & 63);
  const int y = blockIdx.y * 4 + (threadIdx.x >> 6);
  if (x >= Wo || y >= Ho) return;
  const LinTap ty = lin_tap(y, scale_h, Hi);
  const LinTap tx = lin_tap(x, scale_w, Wi);
  const int64_t base = (int64_t)(plane / C) * sb + (int64_t)(plane % C) * sc;
  const float v00 = load_px<DTYPE>(in, base + ty.i0 * sh + tx.i0 * sw, div255);
  const float v01 = load_px<DTYPE>(in, base + ty.i0 * sh + tx.i1 * sw, div255);
  const float v10 = load_px<DTYPE>(in, base + ty.i1 * sh + tx.i0 * sw, div255);
  const float v11 = load_px<DTYPE>(in, base + ty.i1 * sh + tx.i1 * sw, div255);
  const float top = __fadd_rn(__fmul_rn(tx.l0, v00), __fmul_rn(tx.l1, v01));
  const float bot = __fadd_rn(__fmul_rn(tx.l0, v10), __fmul_rn(tx.l1, v11));
  out[((int64_t)plane * Ho + y) * Wo + x] = __fadd_rn(__fmul_rn(ty.l0, top), __fmul_rn(ty.l1, bot));
}

}  // namespace xf

extern "C" int xfeat_resize_bilinear(const void* d_in, int dtype, int B, int C, int Hi, int Wi, int64_t stride_b,
                                     int64_t stride_c, int64_t stride_h, int64_t stride_w, int div255, float* d_out,
                                     int Ho, int Wo, float scale_h, float scale_w, void* stream) {
  XF_REQUIRE(d_in && d_out && B > 0 && C > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0, "resize: bad arguments");
  XF_REQUIRE((int64_t)B * C <= 65535, "resize: B*C too large for grid.z");
  XF_REQUIRE(dtype == XF_DTYPE_F32 || dtype == XF_DTYPE_U8, "resize: unsupported dtype %d", dtype);
  // ATen copies along an axis whose size does not change, whatever the scale: scale 1 samples src == dst with weight 0 on i1
  if (Ho == Hi) scale_h = 1.0f;
  if (Wo == Wi) scale_w = 1.0f;
  dim3 grid(xf::cdiv(Wo, 64), xf::cdiv(Ho, 4), B * C);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == XF_DTYPE_F32)
    xf::resize_bilinear_kernel<XF_DTYPE_F32><<<grid, 256, 0, st>>>(d_in, C, Hi, Wi, stride_b, stride_c, stride_h, stride_w,
                                                                  div255, d_out, Ho, Wo, scale_h, scale_w);
  else
    xf::resize_bilinear_kernel<XF_DTYPE_U8><<<grid, 256, 0, st>>>(d_in, C, Hi, Wi, stride_b, stride_c, stride_h, stride_w,
                                                                 div255, d_out, Ho, Wo, scale_h, scale_w);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_preprocess(const void* d_img, int dtype, int B, int C, int Hi, int Wi, int64_t stride_b,
                                int64_t stride_c, int64_t stride_h, int64_t stride_w, int div255, int H, int W,
                                float* d_xn, double* d_stats, void* stream) {
  // ATen area_pixel_compute_scale (size given): scale = float(in) / out
  return xfeat_preprocess_scaled(d_img, dtype, B, C, Hi, Wi, stride_b, stride_c, stride_h, stride_w, div255, H, W,
                                 (float)Hi / (float)H, (float)Wi / (float)W, d_xn, d_stats, stream);
}

extern "C" int xfeat_preprocess_scaled(const void* d_img, int dtype, int B, int C, int Hi, int Wi, int64_t stride_b,
                                       int64_t stride_c, int64_t stride_h, int64_t stride_w, int div255, int H, int W,
                                       float sh, float sw, float* d_xn, double* d_stats, void* stream) {
  XF_REQUIRE(d_img && d_xn && d_stats, "preprocess: null pointer");
  XF_REQUIRE(B > 0 && B <= 65535 && C > 0 && Hi > 0 && Wi > 0, "preprocess: bad shape");
  XF_REQUIRE(H > 0 && W > 0 && (H % 32) == 0 && (W % 32) == 0, "preprocess: H, W must be positive multiples of 32");
  XF_REQUIRE(dtype == XF_DTYPE_F32 || dtype == XF_DTYPE_U8, "preprocess: unsupported dtype %d", dtype);
  // ATen copies along an axis whose size does not change, whatever the scale (compute_source_index_and_lambda): every form
  // below then samples src == dst there, as the same-size fast forms do
  if (Hi == H) sh = 1.0f;
  if (Wi == W) sw = 1.0f;
  cudaStream_t st = (cudaStream_t)stream;
  XF_CUDA(cudaMemsetAsync(d_stats, 0, sizeof(double) * 2 * B, st));
  dim3 grid(xf::cdiv(W, 64), xf::cdiv(H, 4), B);
  const bool fast = dtype == XF_DTYPE_F32 && Hi == H && Wi == W && stride_w == 1 && ((uintptr_t)d_img % 16) == 0 &&
                    stride_b % 4 == 0 && stride_c % 4 == 0 && stride_h % 4 == 0;
  const bool fast_u8 = dtype == XF_DTYPE_U8 && Hi == H && Wi == W && C == 3 && stride_c == 1 && stride_w == 3 &&
                       ((uintptr_t)d_img % 4) == 0 && stride_b % 4 == 0 && stride_h % 4 == 0;
  // one-pass cluster form: the image's gray fits the shared memory of a cluster (XFEAT_PREP_TWO_PASS=1 keeps the two-kernel form)
  static const bool two_pass = getenv("XFEAT_PREP_TWO_PASS") != nullptr;
  const size_t img_bytes = (size_t)H * W * sizeof(float);
  const int n4 = H * (W / 4);
  int cl = 0;
  if (n4 % 16 == 0 && img_bytes / 16 <= xf::GN_SMEM_2PER_SM) cl = 16;
  else if (n4 % 8 == 0 && img_bytes / 8 <= xf::GN_MAX_SMEM) cl = 8;
  // largest cluster size this process has not seen refused (16 is a non-portable size); XFEAT_PREP_CLUSTER_MAX=8|0 starts lower
  static std::atomic<int> cluster_cap_a{getenv("XFEAT_PREP_CLUSTER_MAX") ? atoi(getenv("XFEAT_PREP_CLUSTER_MAX")) : 16};
  int cluster_cap = cluster_cap_a.load(std::memory_order_relaxed);
  while (!two_pass && fast && cl) {
    if (cl > cluster_cap) {        // step down: 16 -> 8 -> two-kernel form
      cl = (cl == 16 && cluster_cap >= 8 && n4 % 8 == 0 && img_bytes / 8 <= xf::GN_MAX_SMEM) ? 8 : 0;
      continue;
    }
    const size_t gn_smem = img_bytes / cl;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cl, B);
    cfg.blockDim = dim3(xf::GN_THREADS);
    cfg.dynamicSmemBytes = gn_smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    const int W4 = W / 4;
    XF_DYN_SMEM(xf::gray_norm_cluster_kernel, gn_smem);
    cudaError_t e = cudaSuccess;
    if (cl > 8) e = cudaFuncSetAttribute(xf::gray_norm_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e == cudaSuccess)
      e = cudaLaunchKernelEx(&cfg, xf::gray_norm_cluster_kernel, (const float*)d_img, C, stride_b, stride_c, stride_h, div255, H, W4,
                             d_xn, d_stats);
    if (e == cudaSuccess) {
      XF_LAUNCH_CHECK();
      return XF_OK;
    }
    (void)cudaGetLastError();      // a refused cluster shape is a launch-configuration error: nothing ran, try the next form
    cluster_cap = cl == 16 ? 8 : 0;
    cluster_cap_a.store(cluster_cap, std::memory_order_relaxed);
    // Inside a stream capture the refused launch has already invalidated the capture, so a retry cannot rescue it: report the
    // refusal.  The step-down above is kept, so the same call made outside a capture takes the smaller form from then on.
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
      xf::set_error("preprocess: cluster launch of %d CTAs refused (%s) during a stream capture; run the call once before "
                    "capturing it", cl, cudaGetErrorString(e));
      return XF_E_CUDA;
    }
  }
  if (fast_u8) {
    dim3 g4(xf::cdiv(W / 4, 64), xf::cdiv(H, 4), B);
    xf::gray_identity_u8hwc_kernel<<<g4, 256, 0, st>>>((const unsigned char*)d_img, stride_b, stride_h, div255, H, W / 4, d_xn,
                                                       d_stats);
  } else if (fast) {
    dim3 g4(xf::cdiv(H * (W / 4), 256 * xf::GI_NPT), 1, B);
    xf::gray_identity_f32_kernel<<<g4, 256, 0, st>>>((const float*)d_img, C, stride_b, stride_c, stride_h, div255, H, W / 4,
                                                     d_xn, d_stats);
  } else if (dtype == XF_DTYPE_F32 && stride_w == 1 &&
             (int64_t)(C - 1) * stride_c + (int64_t)(Hi - 1) * stride_h + Wi < (int64_t)1 << 31 && stride_c >= 0 && stride_h >= 0) {
    dim3 gx(xf::cdiv(W / 4, 64), xf::cdiv(H, 4 * xf::GRX_ROWS), B);
    xf::gray_resize_f32x4_kernel<<<gx, 256, 0, st>>>((const float*)d_img, C, Hi, Wi, stride_b, (int)stride_c, (int)stride_h, div255,
                                                     H, W / 4, sh, sw, d_xn, d_stats);
  } else if (dtype == XF_DTYPE_F32)
    xf::gray_resize_kernel<XF_DTYPE_F32><<<grid, 256, 0, st>>>(d_img, C, Hi, Wi, stride_b, stride_c, stride_h, stride_w,
                                                              div255, H, W, sh, sw, d_xn, d_stats);
  else
    xf::gray_resize_kernel<XF_DTYPE_U8><<<grid, 256, 0, st>>>(d_img, C, Hi, Wi, stride_b, stride_c, stride_h, stride_w,
                                                             div255, H, W, sh, sw, d_xn, d_stats);
  XF_LAUNCH_CHECK();
  const int HW4 = H * W / 4;
  dim3 g2(std::min(xf::cdiv(HW4, 256), 1024), B);
  xf::instnorm_kernel<<<g2, 256, 0, st>>>(d_xn, d_stats, HW4);
  XF_LAUNCH_CHECK();
  return XF_OK;
}
