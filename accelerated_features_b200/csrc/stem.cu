// Stem: block1 (four thin 3x3 convs, 1->4->8->8->24 channels) and skip1 (AvgPool4 + 1x1), model.py:40-48,139-140.
// GEMM-K is 9/36/72/72: too thin for tensor-core tiles, and the layers are HBM-bound (4-18 FLOP/B, SURVEY 8a table),
// so these are direct convolutions on CUDA cores: one thread per output pixel, all output channels in registers,
// folded weights passed BY VALUE as a __grid_constant__ kernel parameter so every FFMA reads its weight straight
// from the constant bank (no shared-memory or register traffic for weights).
#include "common.cuh"

namespace xf {

template <int CIN, int COUT>
struct StemW {
  float w[9 * CIN * COUT];  // [tap][cin][cout]
  float b[COUT];
};
struct SkipW {
  float w[24];
  float b[24];
};

template <int CIN>
__device__ __forceinline__ void load_vec(const float* __restrict__ p, float (&v)[CIN]) {
  if constexpr (CIN == 1) {
    v[0] = __ldg(p);
  } else {
#pragma unroll
    for (int i = 0; i < CIN / 4; ++i) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p) + i);
      v[4 * i + 0] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
  }
}

// in: (B,Hi,Wi,CIN) NHWC, out: (B,Ho,Wo,COUT) NHWC, 3x3, pad 1, stride S; out = relu(conv + b) [+ skip].
template <int CIN, int COUT, int S, bool SKIP>
__global__ void __launch_bounds__(128) stem_conv_kernel(const __grid_constant__ StemW<CIN, COUT> P,
                                                        const __grid_constant__ SkipW K,
                                                        const float* __restrict__ in, const float* __restrict__ xn,
                                                        float* __restrict__ out, __half* __restrict__ out_split32, int Hi,
                                                        int Wi, int Ho, int Wo) {
  const int ox = blockIdx.x * 32 + (threadIdx.x & 31);
  const int oy = blockIdx.y * 4 + (threadIdx.x >> 5);
  const int b = blockIdx.z;
  if (ox >= Wo || oy >= Ho) return;
  float acc[COUT];
#pragma unroll
  for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
  const float* inb = in + (int64_t)b * Hi * Wi * CIN;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * S - 1 + ky;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * S - 1 + kx;
      float v[CIN];
      if (iy >= 0 && iy < Hi && ix >= 0 && ix < Wi) {
        load_vec<CIN>(inb + ((int64_t)iy * Wi + ix) * CIN, v);
      } else {
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) v[ci] = 0.f;
      }
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci)
#pragma unroll
        for (int co = 0; co < COUT; ++co)
          acc[co] = fmaf(v[ci], P.w[((ky * 3 + kx) * CIN + ci) * COUT + co], acc[co]);
    }
  }
  float skipv = 0.f;
  if constexpr (SKIP) {
    // AvgPool2d(4,4) of the normalised gray image (model.py:40), then 1x1 conv 1->24 with bias (model.py:41)
    const int W0 = Wo * 4;
    const float* xp = xn + ((int64_t)b * Ho * 4 + oy * 4) * W0 + ox * 4;
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(xp + (int64_t)r * W0));
      s += t.x; s += t.y; s += t.z; s += t.w;
    }
    skipv = s * (1.0f / 16.0f);
  }
  float res[COUT];
#pragma unroll
  for (int co = 0; co < COUT; ++co) {
    float v = fmaxf(acc[co] + P.b[co], 0.f);
    if constexpr (SKIP) v += fmaf(skipv, K.w[co], K.b[co]);
    res[co] = v;
  }
  if constexpr (COUT == 24) {
    if (out_split32 != nullptr) {
      // feed the tensor-core block2: [hi(32) | lo(32)] fp16 per pixel, channels 24..31 zero (conv_tc.cu)
      uint4* sp = reinterpret_cast<uint4*>(out_split32 + (((int64_t)b * Ho + oy) * Wo + ox) * 64);
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = 8 * g + 2 * j;
          const float x0 = (c < 24) ? res[c < 24 ? c : 0] : 0.f, x1 = (c + 1 < 24) ? res[c + 1 < 24 ? c + 1 : 0] : 0.f;
          const __half2 h = __floats2half2_rn(x0, x1);
          const float2 hf = __half22float2(h);
          const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
          hw[j] = *reinterpret_cast<const uint32_t*>(&h);
          lw[j] = *reinterpret_cast<const uint32_t*>(&l);
        }
        sp[g] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        sp[4 + g] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      }
      return;
    }
  }
  if constexpr (COUT == 8) {
    if (out_split32 != nullptr) {
      // feed the tensor-core block1.2: [hi(8) | lo(8)] fp16 per pixel = 32 bytes (conv_tc_halo.cu, 32-byte operand rows)
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __half2 h = __floats2half2_rn(res[2 * j], res[2 * j + 1]);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(res[2 * j] - hf.x, res[2 * j + 1] - hf.y);
        hw[j] = *reinterpret_cast<const uint32_t*>(&h);
        lw[j] = *reinterpret_cast<const uint32_t*>(&l);
      }
      uint4* sp = reinterpret_cast<uint4*>(out_split32 + (((int64_t)b * Ho + oy) * Wo + ox) * 16);
      sp[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      sp[1] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      return;
    }
  }
  float* op = out + (((int64_t)b * Ho + oy) * Wo + ox) * COUT;
#pragma unroll
  for (int c4 = 0; c4 < COUT / 4; ++c4)
    reinterpret_cast<float4*>(op)[c4] = make_float4(res[4 * c4], res[4 * c4 + 1], res[4 * c4 + 2], res[4 * c4 + 3]);
}

template <int CIN, int COUT, int S, bool SKIP>
static int launch_stem(const float* hw, const float* hb, const float* sw, const float* sb, const float* in,
                       const float* xn, float* out, __half* out_split32, int B, int Hi, int Wi, cudaStream_t st) {
  StemW<CIN, COUT> P;
  memcpy(P.w, hw, sizeof(P.w));
  memcpy(P.b, hb, sizeof(P.b));
  SkipW K;
  memset(&K, 0, sizeof(K));
  if (SKIP) { memcpy(K.w, sw, sizeof(K.w)); memcpy(K.b, sb, sizeof(K.b)); }
  const int Ho = Hi / S, Wo = Wi / S;
  dim3 grid(cdiv(Wo, 32), cdiv(Ho, 4), B);
  stem_conv_kernel<CIN, COUT, S, SKIP><<<grid, 128, 0, st>>>(P, K, in, xn, out, out_split32, Hi, Wi, Ho, Wo);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// block1.0 + block1.1 in one pass (tensor-core schedule): a thread produces a 2x2 patch of the half-resolution, 8-channel
// block1.1 output.  It needs the 5x5 full-resolution block1.0 pixels around it, which it recomputes from a 7x7 window of the
// gray image held in registers, so the (B,H,W,4) fp32 intermediate (630 MB written + read per 128 VGA images) never exists.
// FMA order per output equals stem_conv_kernel's (taps row-major, then input channel), so both schedules agree bit for bit.
struct Stem01W {
  float w0[9 * 4];      // block1.0 [tap][cout4]
  float b0[4];
  float w1[9 * 4 * 8];  // block1.1 [tap][cin4][cout8]
  float b1[8];
};

// d.xy = a * w.xy + c.xy, each half an IEEE fma (the weight pair comes from the constant bank)
__device__ __forceinline__ float2 fma2(float a, float2 w, float2 c) {
  return make_float2(__fmaf_rn(a, w.x, c.x), __fmaf_rn(a, w.y, c.y));
}

__global__ void __launch_bounds__(128) stem01_kernel(const __grid_constant__ Stem01W P, const float* __restrict__ xn,
                                                     __half* __restrict__ out_split8, int H, int W) {
  const int Ho = H >> 1, Wo = W >> 1;
  const int ox0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 2;
  const int oy0 = (blockIdx.y * 4 + (threadIdx.x >> 5)) * 2;
  const int b = blockIdx.z;
  if (ox0 >= Wo || oy0 >= Ho) return;
  const float* xb = xn + (int64_t)b * H * W;
  const int gy0 = 2 * oy0 - 2, gx0 = 2 * ox0 - 2;   // top-left of the 7x7 gray window
  float g[7][7];
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    const int y = gy0 + r;
    const bool yin = y >= 0 && y < H;
    const float* row = xb + (int64_t)(yin ? y : 0) * W;
#pragma unroll
    for (int c = 0; c < 7; ++c) {
      const int x = gx0 + c;
      g[r][c] = (yin && x >= 0 && x < W) ? __ldg(row + x) : 0.f;
    }
  }
  float2 acc[2][2][4];   // [dy][dx][channel pair]
#pragma unroll
  for (int i = 0; i < 16; ++i) (&acc[0][0][0])[i] = make_float2(0.f, 0.f);
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    const int ay = 2 * oy0 - 1 + r;
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      const int ax = 2 * ox0 - 1 + c;
      float2 a2[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float gv = g[r + ky][c + kx];
          const float* w = &P.w0[(ky * 3 + kx) * 4];
          a2[0] = fma2(gv, make_float2(w[0], w[1]), a2[0]);
          a2[1] = fma2(gv, make_float2(w[2], w[3]), a2[1]);
        }
      const bool ain = ay >= 0 && ay < H && ax >= 0 && ax < W;   // outside the image block1.1 sees zero padding
      float a[4] = {a2[0].x, a2[0].y, a2[1].x, a2[1].y};
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) a[ch] = ain ? fmaxf(a[ch] + P.b0[ch], 0.f) : 0.f;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
        const int ky = r - 2 * dy;
        if (ky < 0 || ky > 2) continue;
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const int kx = c - 2 * dx;
          if (kx < 0 || kx > 2) continue;
#pragma unroll
          for (int ci = 0; ci < 4; ++ci) {
            const float* w = &P.w1[((ky * 3 + kx) * 4 + ci) * 8];
#pragma unroll
            for (int cp = 0; cp < 4; ++cp) acc[dy][dx][cp] = fma2(a[ci], make_float2(w[2 * cp], w[2 * cp + 1]), acc[dy][dx][cp]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int dy = 0; dy < 2; ++dy) {
    uint4* sp = reinterpret_cast<uint4*>(out_split8 + (((int64_t)b * Ho + oy0 + dy) * Wo + ox0) * 16);
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v0 = fmaxf(acc[dy][dx][j].x + P.b1[2 * j], 0.f), v1 = fmaxf(acc[dy][dx][j].y + P.b1[2 * j + 1], 0.f);
        const __half2 h = __floats2half2_rn(v0, v1);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
        hw[j] = *reinterpret_cast<const uint32_t*>(&h);
        lw[j] = *reinterpret_cast<const uint32_t*>(&l);
      }
      sp[2 * dx] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      sp[2 * dx + 1] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
  }
}

static int g_stem_fused = 1;   // XFEAT_STEM_UNFUSED=1 in the environment selects the two-kernel path (A/B measurements)

// xn (B,H,W) -> a1 (B,H,W,4) -> a2 (B,H/2,W/2,8) -> a3 (same,8) -> x1s (B,H/4,W/4,24) = block1(x) + skip1(x)
// tc_tail != 0: only block1.0 and block1.1 run here (block1.1 writes split fp16 [hi8|lo8] into a2); block1.2 / block1.3 + skip
// continue on the tensor cores (api.cu).
int launch_stem_chain(const float* h_weights, const LayerTable& t, const float* xn, float* a1, float* a2, float* a3,
                      float* x1s, __half* x1s_split32, int B, int H, int W, cudaStream_t st, int tc_tail) {
  const float* hw = h_weights;
  int rc;
  static const bool unfused = getenv("XFEAT_STEM_UNFUSED") != nullptr;
  if (tc_tail && g_stem_fused && !unfused) {
    Stem01W P;
    memcpy(P.w0, hw + t.w_off[L_B1_0], sizeof(P.w0));
    memcpy(P.b0, hw + t.b_off[L_B1_0], sizeof(P.b0));
    memcpy(P.w1, hw + t.w_off[L_B1_1], sizeof(P.w1));
    memcpy(P.b1, hw + t.b_off[L_B1_1], sizeof(P.b1));
    dim3 grid(cdiv(W / 4, 32), cdiv(H / 4, 4), B);
    // (capping registers at 128 for 4 CTAs/SM measured the same 333 us as 158 registers / 3 CTAs: issue-bound, not latency-bound)
    stem01_kernel<<<grid, 128, 0, st>>>(P, xn, (__half*)a2, H, W);
    XF_LAUNCH_CHECK();
    return XF_OK;
  }
  rc = launch_stem<1, 4, 1, false>(hw + t.w_off[L_B1_0], hw + t.b_off[L_B1_0], nullptr, nullptr, xn, nullptr, a1, nullptr, B, H, W, st);
  if (rc) return rc;
  rc = launch_stem<4, 8, 2, false>(hw + t.w_off[L_B1_1], hw + t.b_off[L_B1_1], nullptr, nullptr, a1, nullptr, a2,
                                   tc_tail ? (__half*)a2 : nullptr, B, H, W, st);
  if (rc || tc_tail) return rc;
  rc = launch_stem<8, 8, 1, false>(hw + t.w_off[L_B1_2], hw + t.b_off[L_B1_2], nullptr, nullptr, a2, nullptr, a3, nullptr, B, H / 2, W / 2, st);
  if (rc) return rc;
  rc = launch_stem<8, 24, 2, true>(hw + t.w_off[L_B1_3], hw + t.b_off[L_B1_3], hw + t.w_off[L_SKIP1], hw + t.b_off[L_SKIP1],
                                   a3, xn, x1s, x1s_split32, B, H / 2, W / 2, st);
  return rc;
}

}  // namespace xf
