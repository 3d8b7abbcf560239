// Generic folded conv (3x3 / 1x1, stride 1 / 2) + bias + optional ReLU on NHWC fp32 activations -- the fp32-exact
// CUDA-core implicit-GEMM used for block2..block5, block_fusion, the heads and the fine-matcher MLP
// (model.py:50-111).  M = output pixels of a TH x TW tile, N = a CT-wide slice of output channels, K = taps x Cin.
//
// Work decomposition (register-tiled SGEMM shape):
//   * a CTA owns TH x TW output pixels x CT output channels; a thread owns PM consecutive pixels of one row x 8 channels;
//   * Cin is walked in chunks of KC: the (haloed) input patch chunk is staged in shared memory channel-planar
//     [kc][row][col] so a thread fetches its (PM-1)*S+KS row segment with 128-bit LDS once per (kc, ky) and reuses it for
//     the KS horizontal taps; the weight chunk [tap][kc][cout] is staged next to it;
//   * the 8 channels of a thread are {4g..4g+3} U {CT/2+4g..} (CT = 64) so that a quarter-warp's 128-bit weight loads
//     cover 128 contiguous bytes (conflict free), and lanes that share a pixel group broadcast the activation loads.
//   => per (kc, ky): ~9 LDS.128 for 192 FFMA.
#include "common.cuh"

namespace xf {

constexpr int cmax(int a, int b) { return a > b ? a : b; }
constexpr int roundup4(int a) { return (a + 3) / 4 * 4; }

template <int CIN_, int COUT_, int CT_, int KS_, int S_, int TH_, int TW_, int PM_, int KC_, int IN_MODE_, int RELU_>
struct ConvCfg {
  static constexpr int CIN = CIN_, COUT = COUT_, CT = CT_, KS = KS_, S = S_, TH = TH_, TW = TW_, PM = PM_, KC = KC_;
  static constexpr int IN_MODE = IN_MODE_, RELU = RELU_;
  static constexpr int NCG = CT / 8;
  static constexpr int NPGX = TW / PM;
  static constexpr int NPG = NPGX * TH;
  static constexpr int THREADS = NCG * NPG;
  static constexpr int PAD = KS / 2;
  static constexpr int PH = (TH - 1) * S + KS;
  static constexpr int PW = (TW - 1) * S + KS;
  static constexpr int NA = (PM - 1) * S + KS;
  static constexpr int NA4 = (NA + 3) / 4;
  static constexpr int PWP = roundup4(cmax(PW, (TW - PM) * S + NA4 * 4));
  static constexpr int SA = KC * PH * PWP;
  static constexpr int SW = KS * KS * KC * CT;
  static constexpr size_t SMEM = (size_t)(SA + SW) * sizeof(float);
  static_assert(CT % 8 == 0 && COUT % CT == 0, "cout tiling");
  static_assert(TW % PM == 0 && (PM == 4 || PM == 8), "pixel tiling");
  static_assert(CIN % KC == 0 && KC % 4 == 0, "cin chunking");
  static_assert(THREADS <= 1024 && THREADS >= 32, "block size");
};

template <int IN_MODE>
__device__ __forceinline__ float4 load_in4(const float* __restrict__ in, int b, int iy, int ix, int c, int Hi, int Wi,
                                           int CIN) {
  if constexpr (IN_MODE == IN_NHWC) {
    return __ldg(reinterpret_cast<const float4*>(in + (((int64_t)b * Hi + iy) * Wi + ix) * CIN + c));
  } else {
    // logical NHWC (B,Hi,Wi,64) view of the normalised gray image xn (B,8Hi,8Wi): channel 8i+j = pixel (8y+i, 8x+j)
    // == XFeatModel._unfold2d(x, ws=8) (model.py:113-120) without materialising it.
    const int i = c >> 3, j = c & 7;
    return __ldg(reinterpret_cast<const float4*>(in + ((int64_t)b * Hi * 8 + iy * 8 + i) * (Wi * 8) + ix * 8 + j));
  }
}

template <class C>
__global__ void __launch_bounds__(C::THREADS) conv_simt_kernel(const float* __restrict__ in,
                                                               const float* __restrict__ wgt,
                                                               const float* __restrict__ bias, float* __restrict__ out,
                                                               int Hi, int Wi, int Ho, int Wo,
                                                               const int* __restrict__ n_live_cols) {
  constexpr int CIN = C::CIN, COUT = C::COUT, CT = C::CT, KS = C::KS, S = C::S, TH = C::TH, TW = C::TW, PM = C::PM;
  constexpr int KC = C::KC, NCG = C::NCG, NPGX = C::NPGX, PH = C::PH, PW = C::PW, PWP = C::PWP, NA4 = C::NA4;
  extern __shared__ __align__(16) float smem[];
  float* sA = smem;
  float* sW = smem + C::SA;

  const int tid = threadIdx.x;
  const int cg = tid % NCG, pg = tid / NCG;
  const int prow = pg / NPGX, pcol = (pg % NPGX) * PM;
  const int tiles_x = (Wo + TW - 1) / TW;
  const int oy0 = (blockIdx.x / tiles_x) * TH, ox0 = (blockIdx.x % tiles_x) * TW;
  const int co_base = blockIdx.y * CT;
  const int b = blockIdx.z;
  const int iy0 = oy0 * S - C::PAD, ix0 = ox0 * S - C::PAD;
  // flattened row mode (fine-matcher MLP): the live row count is only known on the device; dead tiles exit at once
  if (n_live_cols != nullptr && ox0 >= __ldg(n_live_cols)) return;
  const int coA = (CT == 64) ? 4 * cg : 8 * cg;       // first 4 channels of this thread (within the CT slice)
  const int coB = (CT == 64) ? 32 + 4 * cg : 8 * cg + 4;  // second 4 channels

  float acc[PM][8];
#pragma unroll
  for (int m = 0; m < PM; ++m)
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[m][n] = 0.f;

#pragma unroll 1
  for (int c0 = 0; c0 < CIN; c0 += KC) {
    __syncthreads();
    // ---- stage the input patch chunk, channel-planar ----
    constexpr int NPIX = PH * PW;
    for (int idx = tid; idx < (KC / 4) * NPIX; idx += C::THREADS) {
      const int q = idx / NPIX, pix = idx - q * NPIX;
      const int r = pix / PW, c = pix - r * PW;
      const int iy = iy0 + r, ix = ix0 + c;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < Hi && ix >= 0 && ix < Wi) v = load_in4<C::IN_MODE>(in, b, iy, ix, c0 + 4 * q, Hi, Wi, CIN);
      float* d = sA + (4 * q) * (PH * PWP) + r * PWP + c;
      d[0] = v.x;
      d[PH * PWP] = v.y;
      d[2 * PH * PWP] = v.z;
      d[3 * PH * PWP] = v.w;
    }
    // ---- stage the weight chunk [tap][kc][CT] ----
    for (int idx = tid; idx < KS * KS * KC * (CT / 4); idx += C::THREADS) {
      const int co4 = idx % (CT / 4);
      const int rest = idx / (CT / 4);
      const int kc = rest % KC, t = rest / KC;
      const float4 v = __ldg(reinterpret_cast<const float4*>(wgt + ((int64_t)(t * CIN + c0 + kc)) * COUT + co_base) + co4);
      reinterpret_cast<float4*>(sW + (t * KC + kc) * CT)[co4] = v;
    }
    __syncthreads();
    // ---- FMA ----
#pragma unroll 1
    for (int kc = 0; kc < KC; ++kc) {
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
        float a[NA4 * 4];
        const float4* ap = reinterpret_cast<const float4*>(sA + kc * (PH * PWP) + (prow * S + ky) * PWP + pcol * S);
#pragma unroll
        for (int i = 0; i < NA4; ++i) {
          const float4 t = ap[i];
          a[4 * i] = t.x; a[4 * i + 1] = t.y; a[4 * i + 2] = t.z; a[4 * i + 3] = t.w;
        }
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const float* wp = sW + ((ky * KS + kx) * KC + kc) * CT;
          const float4 b0 = *reinterpret_cast<const float4*>(wp + coA);
          const float4 b1 = *reinterpret_cast<const float4*>(wp + coB);
          const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
          for (int m = 0; m < PM; ++m)
#pragma unroll
            for (int n = 0; n < 8; ++n) acc[m][n] = fmaf(a[m * S + kx], bb[n], acc[m][n]);
        }
      }
    }
  }
  // ---- epilogue: bias (+ReLU), NHWC store ----
  const float4 bi0 = __ldg(reinterpret_cast<const float4*>(bias + co_base + coA));
  const float4 bi1 = __ldg(reinterpret_cast<const float4*>(bias + co_base + coB));
  const float bv[8] = {bi0.x, bi0.y, bi0.z, bi0.w, bi1.x, bi1.y, bi1.z, bi1.w};
  const int oy = oy0 + prow;
  if (oy < Ho) {
#pragma unroll
    for (int m = 0; m < PM; ++m) {
      const int ox = ox0 + pcol + m;
      if (ox < Wo) {
        float r[8];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          float v = acc[m][n] + bv[n];
          if (C::RELU) v = fmaxf(v, 0.f);
          r[n] = v;
        }
        float* op = out + (((int64_t)b * Ho + oy) * Wo + ox) * COUT + co_base;
        *reinterpret_cast<float4*>(op + coA) = make_float4(r[0], r[1], r[2], r[3]);
        *reinterpret_cast<float4*>(op + coB) = make_float4(r[4], r[5], r[6], r[7]);
      }
    }
  }
}

template <class C>
static int launch_cfg(const float* in, const float* w, const float* bias, float* out, int B, int Hi, int Wi,
                      cudaStream_t st, const int* n_live = nullptr) {
  const int Ho = (C::KS == 3) ? (Hi + 2 - 3) / C::S + 1 : Hi / C::S;
  const int Wo = (C::KS == 3) ? (Wi + 2 - 3) / C::S + 1 : Wi / C::S;
  XF_DYN_SMEM(conv_simt_kernel<C>, C::SMEM);
  XF_REQUIRE(B <= 65535, "conv: batch too large for grid.z");
  dim3 grid(cdiv(Ho, C::TH) * cdiv(Wo, C::TW), C::COUT / C::CT, B);
  conv_simt_kernel<C><<<grid, C::THREADS, C::SMEM, st>>>(in, w, bias, out, Hi, Wi, Ho, Wo, n_live);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// Flattened 1x1 layer: geometry is irrelevant, treat the whole batch as one row of B*H*W pixels.
template <int CIN, int COUT, int RELU>
static int launch_pointwise(const float* in, const float* w, const float* bias, float* out, int64_t npix,
                            cudaStream_t st, const int* n_live = nullptr) {
  using C = ConvCfg<CIN, COUT, 64, 1, 1, 1, 256, 8, 8, IN_NHWC, RELU>;
  XF_REQUIRE(npix < (1ll << 31), "pointwise: too many pixels");
  return launch_cfg<C>(in, w, bias, out, 1, 1, (int)npix, st, n_live);
}

int launch_conv_layer(const xfeat_ctx* ctx, int layer, const float* in, int in_mode, int B, int Hi, int Wi, float* out,
                      cudaStream_t st, const int* n_live) {
  const float* w = ctx->d_weights + ctx->table.w_off[layer];
  const float* bi = ctx->d_weights + ctx->table.b_off[layer];
  const int64_t npix = (int64_t)B * Hi * Wi;
  switch (layer) {
    case L_B2_0:
    case L_B2_1:  // 24->24 3x3 s1 at 1/4 res
      return launch_cfg<ConvCfg<24, 24, 24, 3, 1, 16, 32, 8, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B3_0:  // 24->64 3x3 s2 -> 1/8 res
      return launch_cfg<ConvCfg<24, 64, 64, 3, 2, 10, 16, 8, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B3_1:
    case L_FU_0:
    case L_FU_1:  // 64->64 3x3 s1 at 1/8 res (40% of all FLOPs)
      return launch_cfg<ConvCfg<64, 64, 64, 3, 1, 12, 16, 8, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B4_0:  // 64->64 3x3 s2 -> 1/16 res
      return launch_cfg<ConvCfg<64, 64, 64, 3, 2, 5, 40, 8, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B4_1:
    case L_B4_2:  // 64->64 3x3 s1 at 1/16 res
      return launch_cfg<ConvCfg<64, 64, 64, 3, 1, 6, 40, 8, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B5_0:  // 64->128 3x3 s2 -> 1/32 res
      return launch_cfg<ConvCfg<64, 128, 64, 3, 2, 5, 20, 4, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B5_1:
    case L_B5_2:  // 128->128 3x3 s1 at 1/32 res
      return launch_cfg<ConvCfg<128, 128, 64, 3, 1, 5, 20, 4, 8, IN_NHWC, 1>>(in, w, bi, out, B, Hi, Wi, st);
    case L_B5_3:
      return launch_pointwise<128, 64, 1>(in, w, bi, out, npix, st);
    case L_B3_2:
    case L_HH_0:
    case L_HH_1:
    case L_KH_1:
    case L_KH_2:
      return launch_pointwise<64, 64, 1>(in, w, bi, out, npix, st);
    case L_FU_2:
      return launch_pointwise<64, 64, 0>(in, w, bi, out, npix, st);
    case L_KH_0:
      if (in_mode == IN_UNFOLD8)
        return launch_cfg<ConvCfg<64, 64, 64, 1, 1, 12, 16, 8, 8, IN_UNFOLD8, 1>>(in, w, bi, out, B, Hi, Wi, st);
      return launch_pointwise<64, 64, 1>(in, w, bi, out, npix, st);
    case L_FM_0:
      return launch_pointwise<128, 512, 1>(in, w, bi, out, npix, st, n_live);
    case L_FM_1:
    case L_FM_2:
    case L_FM_3:
      return launch_pointwise<512, 512, 1>(in, w, bi, out, npix, st, n_live);
    case L_FM_4:
      return launch_pointwise<512, 64, 0>(in, w, bi, out, npix, st, n_live);
    default:
      set_error("launch_conv_layer: layer %d has no generic-kernel configuration", layer);
      return XF_E_UNSUPPORTED;
  }
}

}  // namespace xf

extern "C" int xfeat_debug_conv_layer(xfeat_ctx* ctx, int layer, const float* d_in, int B, int Hi, int Wi, float* d_out,
                                      void* stream) {
  XF_REQUIRE(ctx && d_in && d_out && layer >= 0 && layer < xf::L_COUNT, "debug_conv_layer: bad arguments");
  XF_CUDA(cudaSetDevice(ctx->device));
  return xf::launch_conv_layer(ctx, layer, d_in, xf::IN_NHWC, B, Hi, Wi, d_out, (cudaStream_t)stream, nullptr);
}
