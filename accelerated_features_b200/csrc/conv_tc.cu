// 64->64 convolutions (3x3 pad 1 / 1x1, stride 1) as implicit GEMM on the Hopper tensor cores:
// TMA-fed shared-memory operands, wgmma with fp32 register accumulators, bias+ReLU epilogue.
// Used for block3.1/3.2, block4.1/4.2, block_fusion.0-2, heatmap_head.0-1, keypoint_head.0-2 (model.py:55-92) -- 48 % of
// the network's FLOPs.
//
// fp32-equivalent precision by operand splitting (SURVEY 7.2: single-pass TF32/BF16/FP16 moves keypoints and misses the
// 1e-3 descriptor tolerance; 3-term splits reproduce the fp32 result):  x = hi + lo in fp16, w*2^k = whi + wlo in fp16,
//      y = (hi.whi + hi.wlo + lo.whi) * 2^-k     (fp32 accumulation; the dropped lo.wlo term is ~2^-22 relative).
// Activations travel between tensor-core layers already split: NHWC with 128 halves per pixel, [hi(64) | lo(64)] -- the
// same 256 bytes per pixel as fp32, written by the producing epilogue.
//
// GEMM mapping: M = 128 output pixels (a TH x TW patch of one image), N = 64 output channels, K = taps x 64 x 3 terms.
//   * the A operand of tap (dy,dx) is the input patch shifted by (dy-1, dx-1): ONE 4-D TMA box {64 ch, TW, TH, 1} per
//     term, 128B-swizzled K-major, out-of-image coordinates zero-filled by the TMA unit (= the conv's zero padding);
//   * the folded, pre-split weights of all taps stay resident in shared memory for the life of the (persistent) CTA;
//   * warps 0-3 = one warpgroup that issues the wgmmas (two 64-row slabs per tile) and runs the epilogue, one pixel row per
//     thread (the accumulator fragments are handed over through a 16 KB staging buffer); warp 4 = TMA producer, which runs
//     up to NS taps ahead, so the operand loads of tile i+1 overlap the epilogue of tile i.
#include <cuda_fp16.h>

#include <vector>

#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

constexpr int CT_THREADS = 160;    // warps 0-3: wgmma + epilogue warpgroup, warp 4: TMA producer
constexpr int CT_ABOX = 128 * 128;   // bytes: 128 pixels x 128 B (64 halves)

// CINP = padded input channels per term (64: two boxes per tap, hi and lo; 32: ONE box per tap whose 128-byte rows are
// [hi(32) | lo(32)]).  NOUT = output channels of this CTA's N tile (32 or 64).  Weight rows are 64 halves (128 B):
//   CINP = 64: group 0 = whi, group 1 = wlo                          -> hi.whi, hi.wlo, lo.whi  (3 x 4 K-steps)
//   CINP = 32: group 0 = [whi | whi], group 1 = [wlo | 0]            -> [hi|lo].[whi|whi] (4 K-steps) + hi.wlo (2 K-steps)
template <int KS, int CINP, int NOUT>
struct ConvTcCfg {
  static constexpr int TAPS = KS * KS;
  static constexpr int ROWB = (CINP == 8) ? 32 : 128;                 // operand row bytes ([hi(8)|lo(8)] halves for the stem)
  static constexpr int KSTEPS = ROWB / 32;
  static constexpr int A_BOXES = (CINP == 64) ? 2 : 1;
  // CINP = 8: a tap is only 4 KB and one K-step, so a pipeline stage carries ALL taps of a tile (one barrier round trip per
  // tile instead of per tap); otherwise one tap per stage.
  static constexpr int TPS = (CINP == 8) ? TAPS : 1;
  static constexpr int A_TAP = A_BOXES * 128 * ROWB;
  static constexpr int A_STAGE = TPS * A_TAP;
  static constexpr int W_GROUP = NOUT * ROWB;                         // bytes
  static constexpr size_t W_BYTES = (size_t)TAPS * 2 * W_GROUP;
  static constexpr int NS_MAX = (int)((227 * 1024 - 2048 - W_BYTES - tc::STG_BYTES) / A_STAGE);
  static constexpr int NS_CAP = (CINP == 8) ? 4 : 6;
  static constexpr int NS = NS_MAX > NS_CAP ? NS_CAP : NS_MAX;        // A stages (one tap each)
  static constexpr size_t A_BYTES = (size_t)NS * A_STAGE;
  static constexpr size_t SMEM = 1024 + W_BYTES + A_BYTES + tc::STG_BYTES + 1536;
  // accumulator: columns [0,NOUT) = terms against weight group 0, [NOUT,2*NOUT) = against group 1: a single wgmma with
  // N = 2*NOUT reads the activation operand once for both groups (the layers are shared-memory-bandwidth bound).
  static_assert(NS >= 2, "need at least two A stages");
  static_assert(CINP == 8 || CINP == 32 || CINP == 64, "CINP");
  static_assert(NOUT == 32 || NOUT == 64, "NOUT");
};

struct ConvTcParams {
  CUtensorMap amap;   // input activations, split fp16 (B,Hin,Win,2*CINP); box {64, S*TW, S*TH, 1}, element strides {1,S,S,1}
  CUtensorMap wmap;   // weights of this N tile: rows [tap][group][NOUT] x 64 halves
  const float* bias;  // bias + co0
  float inv_wscale;
  int B, H, W;        // OUTPUT height / width
  int stride;         // 1 or 2
  int pad;            // KS / 2
  int tw_log2;        // TW = 1 << tw_log2, TH = 128 / TW
  __half* out_split;  // (B,H,W,2*split_c) [hi(split_c) | lo(split_c)] or null; split_c = 32 or 64
  int split_c;
  float* out_f32;     // (B,H,W,f32_c) or null; this CTA's channels start at f32_co0, n_real of them are real
  int f32_c, f32_co0, n_real;
  int relu;
  // optional skip branch of the stem (model.py:40-41,140): out += avgpool4(xn) * skip_w + skip_b, xn = (B, 4H, 4W) fp32
  const float* skip_xn;
  const float* skip_w;   // 24 weights then 24 biases
  FastDiv div_img, div_x; // tiles per image, tiles per row
};

template <int KS, int CINP, int NOUT>
__global__ void __launch_bounds__(CT_THREADS, 1) conv_tc_kernel(const __grid_constant__ ConvTcParams P) {
  using C = ConvTcCfg<KS, CINP, NOUT>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sW = base;
  unsigned char* sA = base + C::W_BYTES;
  float* sStg = reinterpret_cast<float*>(base + C::W_BYTES + C::A_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + C::W_BYTES + C::A_BYTES + tc::STG_BYTES);
  uint64_t* w_full = bars;
  uint64_t* a_full = bars + 1;                 // [NS]
  uint64_t* a_empty = bars + 1 + C::NS;        // [NS]
  float* sBias = reinterpret_cast<float*>(bars + 1 + 2 * C::NS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int TW = 1 << P.tw_log2, TH = 128 >> P.tw_log2;
  const int tiles_x = (P.W + TW - 1) / TW, tiles_y = (P.H + TH - 1) / TH;
  const int tiles_img = tiles_x * tiles_y;
  const int n_tiles = tiles_img * P.B;

  if (threadIdx.x < NOUT) sBias[threadIdx.x] = (threadIdx.x < P.n_real) ? __ldg(P.bias + threadIdx.x) : 0.f;
  float* sSkip = sBias + NOUT;   // [2][NOUT]: skip weights, skip biases (zero when unused / padded)
  if (threadIdx.x < 2 * NOUT) {
    const int c = threadIdx.x % NOUT, wb = threadIdx.x / NOUT;
    sSkip[threadIdx.x] = (P.skip_w != nullptr && c < 24) ? __ldg(P.skip_w + wb * 24 + c) : 0.f;
  }
  if (warp == 4 && lane == 0) {
    tc::tma_prefetch_desc(&P.amap);
    tc::tma_prefetch_desc(&P.wmap);
    tc::mbar_init(w_full, 1);
    for (int i = 0; i < C::NS; ++i) {
      tc::mbar_init(&a_full[i], 1);
      tc::mbar_init(&a_empty[i], 4);   // one arrival per consumer warp
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      // ---------------- TMA producer ----------------
      tc::mbar_expect_tx(w_full, (uint32_t)C::W_BYTES);
      for (int i = 0; i < C::TAPS * 2; ++i) tc::tma_load_2d(sW + (size_t)i * C::W_GROUP, &P.wmap, w_full, 0, i * NOUT);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
        const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
        const int y0 = ty_ * TH * P.stride - P.pad, x0 = tx_ * TW * P.stride - P.pad;
        for (int tap0 = 0; tap0 < C::TAPS; tap0 += C::TPS, ++it) {
          const int s = it % C::NS;
          const uint32_t ph = (it / C::NS) & 1;
          tc::mbar_wait(&a_empty[s], ph ^ 1);
          tc::mbar_expect_tx(&a_full[s], C::A_STAGE);
#pragma unroll
          for (int j = 0; j < C::TPS; ++j) {
            const int tap = tap0 + j;
            const int dy = (KS == 3) ? tap / 3 : 0, dx = (KS == 3) ? tap % 3 : 0;
            unsigned char* dst = sA + (size_t)s * C::A_STAGE + (size_t)j * C::A_TAP;
            tc::tma_load_4d(dst, &P.amap, &a_full[s], 0, x0 + dx, y0 + dy, b);                    // hi (CINP=64) or [hi|lo]
            if (C::A_BOXES == 2) tc::tma_load_4d(dst + CT_ABOX, &P.amap, &a_full[s], 64, x0 + dx, y0 + dy, b);  // lo
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ---------------- wgmma + epilogue warpgroup: thread r owns pixel r of the tile ----------------
    constexpr int N2 = 2 * NOUT;
    constexpr uint32_t HALF = (64 * C::ROWB) >> 4;   // descriptor offset of rows 64-127
    const int r = threadIdx.x;
    const int ph_ = r >> P.tw_log2, pw_ = r & (TW - 1);
    float acc0[NOUT], acc1[NOUT];                    // rows 0-63 / 64-127, N2 columns each
    tc::mbar_wait(w_full, 0);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      for (int tap0 = 0; tap0 < C::TAPS; tap0 += C::TPS, ++it) {
        const int s = it % C::NS;
        tc::mbar_wait(&a_full[s], (it / C::NS) & 1);
        tc::wgmma_fence();
#pragma unroll
        for (int j = 0; j < C::TPS; ++j) {
          const int tap = tap0 + j;
          const uint32_t a_addr = tc::smem_u32(sA + (size_t)s * C::A_STAGE + (size_t)j * C::A_TAP);
          const uint32_t w_addr = tc::smem_u32(sW + (size_t)tap * 2 * C::W_GROUP);
          const uint64_t a0 = tc::make_desc_rows<C::ROWB>(a_addr);
          const uint64_t w0 = tc::make_desc_rows<C::ROWB>(w_addr);   // group 0, and (N = 2*NOUT) groups [0 ; 1] stacked
          if (C::A_BOXES == 2) {
            const uint64_t a1 = tc::make_desc_sw128(a_addr + CT_ABOX, 1024);
#pragma unroll
            for (int k = 0; k < 4; ++k) {   // hi.whi | hi.wlo
              tc::wgmma_f16<N2>(acc0, a0 + 2 * k, w0 + 2 * k, (tap | k) ? 1u : 0u);
              tc::wgmma_f16<N2>(acc1, a0 + HALF + 2 * k, w0 + 2 * k, (tap | k) ? 1u : 0u);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {   // lo.whi
              tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc0), a1 + 2 * k, w0 + 2 * k, 1u);
              tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc1), a1 + HALF + 2 * k, w0 + 2 * k, 1u);
            }
          } else {
#pragma unroll
            for (int k = 0; k < C::KSTEPS; ++k) {   // [hi|lo].[[whi|whi];[wlo|0]]; the lo K-steps of 128-byte rows skip the zero block
              const bool lo_half = (C::ROWB == 128) && (k >= C::KSTEPS / 2);
              if (lo_half) {
                tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc0), a0 + 2 * k, w0 + 2 * k, 1u);
                tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc1), a0 + HALF + 2 * k, w0 + 2 * k, 1u);
              } else {
                tc::wgmma_f16<N2>(acc0, a0 + 2 * k, w0 + 2 * k, (tap | k) ? 1u : 0u);
                tc::wgmma_f16<N2>(acc1, a0 + HALF + 2 * k, w0 + 2 * k, (tap | k) ? 1u : 0u);
              }
            }
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&a_empty[s]);   // this warp's reads of the stage are complete
      }
      // ---------------- epilogue ----------------
      const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
      const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
      const int y = ty_ * TH + ph_, x = tx_ * TW + pw_;
      uint32_t v[N2];
#pragma unroll
      for (int c = 0; c < N2 / 32; ++c) {
        uint32_t t[32];
        tc::acc_rows<32>(sStg, acc0, acc1, c * 32, r, 1, t);
#pragma unroll
        for (int j = 0; j < 32; ++j) v[c * 32 + j] = t[j];
      }
      if (y < P.H && x < P.W) {
        const int64_t pix = ((int64_t)b * P.H + y) * P.W + x;
        float o[NOUT];
#pragma unroll
        for (int c = 0; c < NOUT; ++c) {
          float t0 = fmaf(__uint_as_float(v[c]) + __uint_as_float(v[NOUT + c]), P.inv_wscale, sBias[c]);
          if (P.relu) t0 = fmaxf(t0, 0.f);
          o[c] = t0;
        }
        if (P.skip_xn != nullptr) {
          // AvgPool2d(4,4) of the normalised gray image, then 1x1 conv 1 -> 24 with bias, added AFTER the ReLU (model.py:140)
          const int W0 = P.W * 4;
          const float* xp = P.skip_xn + ((int64_t)b * P.H * 4 + y * 4) * W0 + x * 4;
          float sacc = 0.f;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(xp + (int64_t)rr * W0));
            sacc += t.x; sacc += t.y; sacc += t.z; sacc += t.w;
          }
          const float skipv = sacc * (1.0f / 16.0f);
#pragma unroll
          for (int c = 0; c < NOUT; ++c) o[c] += fmaf(skipv, sSkip[c], sSkip[NOUT + c]);
        }
        if (P.out_f32) tc::store_f32_row<NOUT>(P.out_f32 + pix * P.f32_c + P.f32_co0, o, P.n_real);
        if (P.out_split) {
          // [hi(split_c) | lo(split_c)]; this N tile owns channels f32_co0 .. f32_co0+NOUT-1 (padded channels: exact zeros)
          __half* hp = P.out_split + pix * (2 * P.split_c) + P.f32_co0;
          tc::store_split_row<NOUT>(hp, hp + P.split_c, o);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 128-input-channel layers (block5.1, block5.2 3x3; block5.3 1x1): the weights of all taps no longer fit in shared memory,
// so each pipeline stage carries one tap of BOTH operands: A = {hi0, hi1, lo0, lo1} boxes (128 px x 64 halves each) and
// W = {whi0, wlo0, whi1, wlo1} (64 cout x 64 halves each) of this CTA's 64-channel N tile (blockIdx.y).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int C128_WBOX = 64 * 128;
constexpr int C128_STAGE = 4 * CT_ABOX + 4 * C128_WBOX;   // 96 KB
constexpr size_t C128_SMEM = 1024 + 2 * (size_t)C128_STAGE + tc::STG_BYTES + 768;

template <int KS>
__global__ void __launch_bounds__(CT_THREADS, 1) conv_tc128_kernel(const __grid_constant__ ConvTcParams P) {
  constexpr int TAPS = KS * KS, NOUT = 64, NS = 2;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sS = base;
  float* sStg = reinterpret_cast<float*>(base + NS * (size_t)C128_STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + NS * (size_t)C128_STAGE + tc::STG_BYTES);
  uint64_t* s_full = bars;           // [NS]
  uint64_t* s_empty = bars + NS;     // [NS]
  float* sBias = reinterpret_cast<float*>(bars + 2 * NS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int TW = 1 << P.tw_log2, TH = 128 >> P.tw_log2;
  const int tiles_x = (P.W + TW - 1) / TW, tiles_y = (P.H + TH - 1) / TH;
  const int tiles_img = tiles_x * tiles_y;
  const int n_tiles = tiles_img * P.B;
  const int nt = blockIdx.y;                     // N tile: output channels nt*64 .. nt*64+63
  const int co0 = nt * NOUT;

  if (threadIdx.x < NOUT) sBias[threadIdx.x] = __ldg(P.bias + co0 + threadIdx.x);
  if (warp == 4 && lane == 0) {
    tc::tma_prefetch_desc(&P.amap);
    tc::tma_prefetch_desc(&P.wmap);
    for (int i = 0; i < NS; ++i) {
      tc::mbar_init(&s_full[i], 1);
      tc::mbar_init(&s_empty[i], 4);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
        const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
        const int y0 = ty_ * TH - P.pad, x0 = tx_ * TW - P.pad;
        for (int tap = 0; tap < TAPS; ++tap, ++it) {
          const int s = it % NS;
          const int dy = (KS == 3) ? tap / 3 : 0, dx = (KS == 3) ? tap % 3 : 0;
          tc::mbar_wait(&s_empty[s], ((it / NS) & 1) ^ 1);
          tc::mbar_expect_tx(&s_full[s], C128_STAGE);
          unsigned char* dst = sS + (size_t)s * C128_STAGE;
#pragma unroll
          for (int j = 0; j < 4; ++j)   // channel blocks hi0, hi1, lo0, lo1 = halves [0,64) [64,128) [128,192) [192,256)
            tc::tma_load_4d(dst + j * CT_ABOX, &P.amap, &s_full[s], 64 * j, x0 + dx, y0 + dy, b);
          // weights: rows ((nt * TAPS + tap) * 4 + g) * 64, g = whi0, wlo0, whi1, wlo1 -> one 256-row box
          tc::tma_load_2d(dst + 4 * CT_ABOX, &P.wmap, &s_full[s], 0, ((nt * TAPS + tap) * 4) * 64);
        }
      }
    }
    __syncwarp();
  } else {
    constexpr uint32_t HALF = (64 * 128) >> 4;   // descriptor offset of rows 64-127
    const int r = threadIdx.x;
    const int ph_ = r >> P.tw_log2, pw_ = r & (TW - 1);
    float acc0[NOUT], acc1[NOUT];                 // rows 0-63 / 64-127, 2*NOUT columns each
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      for (int tap = 0; tap < TAPS; ++tap, ++it) {
        const int s = it % NS;
        tc::mbar_wait(&s_full[s], (it / NS) & 1);
        tc::wgmma_fence();
        const uint32_t sa = tc::smem_u32(sS + (size_t)s * C128_STAGE), sw = sa + 4 * CT_ABOX;
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint64_t ahi = tc::make_desc_sw128(sa + kb * CT_ABOX, 1024), alo = tc::make_desc_sw128(sa + (2 + kb) * CT_ABOX, 1024);
          const uint64_t whi = tc::make_desc_sw128(sw + (2 * kb) * C128_WBOX, 1024);   // also [whi_kb ; wlo_kb] with N = 128
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // hi.whi | hi.wlo
            tc::wgmma_f16<2 * NOUT>(acc0, ahi + 2 * k, whi + 2 * k, (tap | kb | k) ? 1u : 0u);
            tc::wgmma_f16<2 * NOUT>(acc1, ahi + HALF + 2 * k, whi + 2 * k, (tap | kb | k) ? 1u : 0u);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // lo.whi
            tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc0), alo + 2 * k, whi + 2 * k, 1u);
            tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc1), alo + HALF + 2 * k, whi + 2 * k, 1u);
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&s_empty[s]);
      }
      const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
      const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
      const int y = ty_ * TH + ph_, x = tx_ * TW + pw_;
      uint32_t v0[32], v1[32], v2[32], v3[32];
      tc::acc_rows<32>(sStg, acc0, acc1, 0, r, 1, v0);
      tc::acc_rows<32>(sStg, acc0, acc1, 32, r, 1, v1);
      tc::acc_rows<32>(sStg, acc0, acc1, 64, r, 1, v2);
      tc::acc_rows<32>(sStg, acc0, acc1, 96, r, 1, v3);
      if (y < P.H && x < P.W) {
        const int64_t pix = ((int64_t)b * P.H + y) * P.W + x;
        float o[NOUT];
#pragma unroll
        for (int c = 0; c < 32; ++c) {
          float t0 = fmaf(__uint_as_float(v0[c]) + __uint_as_float(v2[c]), P.inv_wscale, sBias[c]);
          float t1 = fmaf(__uint_as_float(v1[c]) + __uint_as_float(v3[c]), P.inv_wscale, sBias[32 + c]);
          if (P.relu) { t0 = fmaxf(t0, 0.f); t1 = fmaxf(t1, 0.f); }
          o[c] = t0; o[32 + c] = t1;
        }
        if (P.out_f32) tc::store_f32_row<NOUT>(P.out_f32 + pix * P.f32_c + co0, o, NOUT);
        if (P.out_split) {
          __half* hp = P.out_split + pix * (2 * P.split_c) + co0;
          tc::store_split_row<NOUT>(hp, hp + P.split_c, o);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// helpers: fp32 NHWC (64 ch) -> split fp16 NHWC (128 halves); unfold8 + split of the normalised gray image
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void split8(const float (&x)[8], uint4& hi, uint4& lo) {
  __half2 h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[j] = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
    const float2 hf = __half22float2(h[j]);
    l[j] = __floats2half2_rn(x[2 * j] - hf.x, x[2 * j + 1] - hf.y);
  }
  hi = make_uint4(*reinterpret_cast<uint32_t*>(&h[0]), *reinterpret_cast<uint32_t*>(&h[1]), *reinterpret_cast<uint32_t*>(&h[2]),
                  *reinterpret_cast<uint32_t*>(&h[3]));
  lo = make_uint4(*reinterpret_cast<uint32_t*>(&l[0]), *reinterpret_cast<uint32_t*>(&l[1]), *reinterpret_cast<uint32_t*>(&l[2]),
                  *reinterpret_cast<uint32_t*>(&l[3]));
}

// fp32 NHWC with C real channels (multiple of 8) -> split fp16 NHWC [hi(CP) | lo(CP)], channels C..CP-1 zero.
__global__ void __launch_bounds__(256) split_nhwc_kernel(const float* __restrict__ in, __half* __restrict__ out, int64_t npix,
                                                         int C, int CP) {
  const int G = CP / 8;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (pixel, 8-channel group)
  if (gid >= npix * G) return;
  const int64_t pix = gid / G;
  const int g = (int)(gid - pix * G);
  float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (8 * g < C) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(in + pix * C) + 2 * g);
    const float4 b = __ldg(reinterpret_cast<const float4*>(in + pix * C) + 2 * g + 1);
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  }
  uint4 hi, lo;
  split8(x, hi, lo);
  reinterpret_cast<uint4*>(out + pix * 2 * CP)[g] = hi;
  reinterpret_cast<uint4*>(out + pix * 2 * CP)[G + g] = lo;
}

// XFeatModel._unfold2d(x, 8) (model.py:113-120) fused with the split: channel 8i+j of cell (h,w) = xn[8h+i, 8w+j].
__global__ void __launch_bounds__(256) unfold8_split_kernel(const float* __restrict__ xn, __half* __restrict__ out, int Hc,
                                                            int Wc, int64_t ncell) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (cell, row i)
  if (gid >= ncell * 8) return;
  const int64_t cell = gid >> 3;
  const int i = (int)(gid & 7);
  const int64_t b = cell / ((int64_t)Hc * Wc);
  const int rem = (int)(cell - b * Hc * Wc);
  const int h = rem / Wc, w = rem - h * Wc;
  const float* p = xn + ((int64_t)b * Hc * 8 + h * 8 + i) * (Wc * 8) + w * 8;
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), c = __ldg(reinterpret_cast<const float4*>(p) + 1);
  const float x[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
  uint4 hi, lo;
  split8(x, hi, lo);
  reinterpret_cast<uint4*>(out + cell * 128)[i] = hi;
  reinterpret_cast<uint4*>(out + cell * 128)[8 + i] = lo;
}

int launch_split_nhwc(const float* in, __half* out, int64_t npix, int C, int CP, cudaStream_t st) {
  split_nhwc_kernel<<<(unsigned)((npix * (CP / 8) + 255) / 256), 256, 0, st>>>(in, out, npix, C, CP);
  XF_LAUNCH_CHECK();
  return XF_OK;
}
int launch_unfold8_split(const float* xn, __half* out, int B, int Hc, int Wc, cudaStream_t st) {
  const int64_t ncell = (int64_t)B * Hc * Wc;
  unfold8_split_kernel<<<(unsigned)((ncell * 8 + 255) / 256), 256, 0, st>>>(xn, out, Hc, Wc, ncell);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// host: weight preparation at context creation, per-launch tensor maps
// ---------------------------------------------------------------------------------------------------------------------
// Layers that run on the tensor-core kernel and their operand geometry.
struct TcLayer { int cinp, nout, ntiles; };
static bool tc_layer_cfg(int layer, TcLayer& c) {
  if (layer >= L_FM_0) return false;
  const LayerSpec& s = kLayers[layer];
  if (s.cin == 64 && s.cout == 64) { c = {64, 64, 1}; return true; }            // block3.1/2, block4.*, fusion, heads
  if (s.cin == 24 && s.cout == 24) { c = {32, 32, 1}; return true; }            // block2 (channels padded 24 -> 32)
  if (s.cin == 8 && s.cout == 8) { c = {8, 8, 1}; return true; }                // block1.2 (halo kernel only), 32-byte operand rows
  if (s.cin == 8 && s.cout == 24) { c = {8, 32, 1}; return true; }              // block1.3 (stride 2) + skip1
  if (s.cin == 24 && s.cout == 64) { c = {32, 64, 1}; return true; }            // block3.0 (stride 2)
  if (s.cin == 64 && s.cout == 128) { c = {64, 64, 2}; return true; }           // block5.0 (stride 2), two N tiles
  if (s.cin == 128 && s.stride == 1) { c = {128, 64, s.cout / 64}; return true; }   // block5.1/5.2 (3x3), block5.3 (1x1): streamed weights
  if (s.cin == 64 && s.cout == 65) { c = {64, 80, 1}; return true; }            // keypoint_head.3, N padded to 80 (head_chain_tc.cu only)
  if (s.cin == 64 && s.cout == 1) { c = {64, 16, 1}; return true; }             // heatmap_head.2, N padded to 16 (head_chain_tc.cu only)
  return false;
}
bool conv_tc_eligible(int layer) {
  TcLayer c;
  return tc_layer_cfg(layer, c);
}

int conv_tc_prepare(xfeat_ctx* ctx) {
  // split weights: W[tap][cin][cout] fp32 (BN folded) * 2^k -> per N tile rows [tap][group][NOUT] x 64 halves
  size_t total = 0;
  for (int l = 0; l < L_COUNT; ++l) {
    ctx->tc_off[l] = (size_t)-1;
    TcLayer c;
    if (tc_layer_cfg(l, c)) {
      ctx->tc_off[l] = total;
      total += (size_t)c.ntiles * kLayers[l].ks * kLayers[l].ks * 2 * c.nout * 64 * (c.cinp == 128 ? 2 : 1);   // (8-channel layers use 16 of the 64 halves per row slot: simpler indexing, 36 KB wasted)
    }
  }
  std::vector<__half> h(total, __float2half_rn(0.f));
  for (int l = 0; l < L_COUNT; ++l) {
    TcLayer c;
    if (!tc_layer_cfg(l, c)) continue;
    const LayerSpec& sp = kLayers[l];
    const int taps = sp.ks * sp.ks;
    const float* w = ctx->h_weights + ctx->table.w_off[l];
    float mx = 0.f;
    for (int i = 0; i < taps * sp.cin * sp.cout; ++i) mx = fmaxf(mx, fabsf(w[i]));
    int e = 0;
    if (mx > 0.f) frexpf(mx, &e);
    const float s = (mx > 0.f) ? ldexpf(1.f, 13 - e) : 1.f;          // max|w| * s in [2^12, 2^13)
    ctx->tc_inv_wscale[l] = (mx > 0.f) ? ldexpf(1.f, e - 13) : 1.f;
    if (c.cinp == 128) {
      for (int nt = 0; nt < c.ntiles; ++nt)
        for (int t = 0; t < taps; ++t)
          for (int n = 0; n < 64; ++n) {
            const int co = nt * 64 + n;
            for (int ci = 0; ci < 128; ++ci) {
              const float v = w[((size_t)t * sp.cin + ci) * sp.cout + co] * s;
              const __half hi = __float2half_rn(v);
              const __half lo = __float2half_rn(v - __half2float(hi));
              const int kb = ci >> 6, cc = ci & 63;
              __half* grp = h.data() + ctx->tc_off[l] + ((((size_t)nt * taps + t) * 4 + 2 * kb) * 64 + n) * 64;
              grp[cc] = hi;                 // group 2*kb   : whi of K block kb
              grp[64 * 64 + cc] = lo;       // group 2*kb+1 : wlo of K block kb
            }
          }
      continue;
    }
    const int rowh = (c.cinp == 8) ? 16 : 64;   // halves per weight row
    for (int nt = 0; nt < c.ntiles; ++nt) {
      __half* dst = h.data() + ctx->tc_off[l] + (size_t)nt * taps * 2 * c.nout * rowh;
      for (int t = 0; t < taps; ++t)
        for (int n = 0; n < c.nout; ++n) {
          const int co = nt * c.nout + n;
          __half* g0 = dst + (((size_t)t * 2 + 0) * c.nout + n) * rowh;
          __half* g1 = dst + (((size_t)t * 2 + 1) * c.nout + n) * rowh;
          if (co >= sp.cout) continue;                                 // padded output channel: zero row
          for (int ci = 0; ci < sp.cin; ++ci) {
            const float v = w[((size_t)t * sp.cin + ci) * sp.cout + co] * s;
            const __half hi = __float2half_rn(v);
            const __half lo = __float2half_rn(v - __half2float(hi));
            if (c.cinp == 64) { g0[ci] = hi; g1[ci] = lo; }
            else { g0[ci] = hi; g0[c.cinp + ci] = hi; g1[ci] = lo; }  // [whi|whi], [wlo|0]  (cinp = 32 or 8)
          }
        }
    }
  }
  XF_CUDA(cudaMalloc(&ctx->d_tcw, total * sizeof(__half)));
  XF_CUDA(cudaMemcpy(ctx->d_tcw, h.data(), total * sizeof(__half), cudaMemcpyHostToDevice));
  return XF_OK;
}

static void pick_tile(int H, int W, int& tw_log2) {
  // TH x TW = 128: choose the shape that wastes the fewest out-of-image pixels
  int best = -1;
  long best_cost = 0;
  for (int l = 2; l <= 6; ++l) {
    const int TW = 1 << l, TH = 128 >> l;
    const long cost = (long)cdiv(H, TH) * TH * cdiv(W, TW) * TW;
    if (best < 0 || cost < best_cost) { best = l; best_cost = cost; }
  }
  tw_log2 = best;
}

template <int KS, int CINP, int NOUT>
static int launch_tc_cfg(const ConvTcParams& P, int grid, cudaStream_t st) {
  using C = ConvTcCfg<KS, CINP, NOUT>;
  XF_DYN_SMEM((conv_tc_kernel<KS, CINP, NOUT>), C::SMEM);
  conv_tc_kernel<KS, CINP, NOUT><<<grid, CT_THREADS, C::SMEM, st>>>(P);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// in_split: (B,Hin,Win,2*CINP) halves [hi|lo].  out_split (optional): (B,Ho,Wo,2*NOUT); out_f32 (optional): (B,Ho,Wo,cout).
int launch_conv_tc(const xfeat_ctx* ctx, int layer, const __half* in_split, int B, int Hin, int Win, __half* out_split,
                   float* out_f32, cudaStream_t st, const float* skip_xn) {
  TcLayer c;
  XF_REQUIRE(tc_layer_cfg(layer, c) && ctx->d_tcw, "conv_tc: layer %d not prepared for the tensor-core path", layer);
  XF_REQUIRE(out_split || out_f32, "conv_tc: no output");
  XF_REQUIRE(!(c.cinp == 8 && c.nout == 8 && g_conv_impl != 2), "conv_tc: block1.2 runs on the halo kernel only (conv impl 2)");
  if (g_conv_impl == 2 && kLayers[layer].ks == 3 && kLayers[layer].stride == 1 && c.ntiles == 1 && c.cinp == c.nout)
    return launch_conv_tc_halo(ctx, layer, in_split, B, Hin, Win, out_split, out_f32, st);
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  const LayerSpec& sp = kLayers[layer];
  const int S = sp.stride, Ho = Hin / S, Wo = Win / S;
  ConvTcParams P;
  int tw_log2;
  pick_tile(Ho, Wo, tw_log2);
  const int TW = 1 << tw_log2, TH = 128 >> tw_log2;
  const int rowh = (c.cinp == 8) ? 16 : 64;
  const CUtensorMapSwizzle swz = (c.cinp == 8) ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_128B;
  const cuuint64_t row_bytes = (cuuint64_t)2 * c.cinp * sizeof(__half);
  const cuuint64_t dims[4] = {(cuuint64_t)2 * c.cinp, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)B};
  const cuuint64_t strides[3] = {row_bytes, (cuuint64_t)Win * row_bytes, (cuuint64_t)Hin * Win * row_bytes};
  const cuuint32_t box[4] = {(cuuint32_t)rowh, (cuuint32_t)(TW * S), (cuuint32_t)(TH * S), 1};
  const cuuint32_t estr[4] = {1, (cuuint32_t)S, (cuuint32_t)S, 1};
  CUresult r = enc(&P.amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)in_split, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(activations %dx%dx%d, stride %d) failed: %d", B, Hin, Win, S, (int)r);
    return XF_E_CUDA;
  }
  const int taps = sp.ks * sp.ks;
  P.inv_wscale = ctx->tc_inv_wscale[layer];
  P.B = B; P.H = Ho; P.W = Wo;
  P.stride = S;
  P.pad = sp.ks / 2;
  P.tw_log2 = tw_log2;
  P.out_split = out_split;
  P.out_f32 = out_f32;
  P.f32_c = sp.cout;
  P.relu = sp.relu;
  P.skip_xn = skip_xn;
  P.skip_w = skip_xn ? ctx->d_weights + ctx->table.w_off[L_SKIP1] : nullptr;   // 24 weights; the 24 biases follow (layers.h packing)
  const int n_tiles = cdiv(Ho, TH) * cdiv(Wo, TW) * B;
  XF_REQUIRE(n_tiles < (1 << 22), "conv_tc: too many tiles (%d)", n_tiles);
  P.div_img = make_fastdiv((unsigned)(cdiv(Ho, TH) * cdiv(Wo, TW)));
  P.div_x = make_fastdiv((unsigned)cdiv(Wo, TW));
  const int grid = n_tiles < ctx->sm_count ? n_tiles : ctx->sm_count;
  P.split_c = sp.cout <= 32 ? 32 : sp.cout;   // channel count of the split output tensor [hi(split_c) | lo(split_c)]
  if (c.cinp == 128) {
    const cuuint64_t wdims[2] = {64, (cuuint64_t)c.ntiles * taps * 4 * 64};
    const cuuint64_t wstrides[1] = {128};
    const cuuint32_t wbox[2] = {64, 256};
    const cuuint32_t westr[2] = {1, 1};
    r = enc(&P.wmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)((__half*)ctx->d_tcw + ctx->tc_off[layer]), wdims, wstrides, wbox,
            westr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(weights128, layer %d) failed: %d", layer, (int)r);
      return XF_E_CUDA;
    }
    P.bias = ctx->d_weights + ctx->table.b_off[layer];
    P.f32_co0 = 0;
    P.n_real = 64;
    const int gx = cdiv(ctx->sm_count, c.ntiles) < n_tiles ? cdiv(ctx->sm_count, c.ntiles) : n_tiles;
    dim3 g2(gx, c.ntiles);
    if (sp.ks == 3) {
      XF_DYN_SMEM(conv_tc128_kernel<3>, C128_SMEM);
      conv_tc128_kernel<3><<<g2, CT_THREADS, C128_SMEM, st>>>(P);
    } else {
      XF_DYN_SMEM(conv_tc128_kernel<1>, C128_SMEM);
      conv_tc128_kernel<1><<<g2, CT_THREADS, C128_SMEM, st>>>(P);
    }
    XF_LAUNCH_CHECK();
    return XF_OK;
  }
  for (int nt = 0; nt < c.ntiles; ++nt) {
    const cuuint64_t wdims[2] = {(cuuint64_t)rowh, (cuuint64_t)taps * 2 * c.nout};
    const cuuint64_t wstrides[1] = {(cuuint64_t)rowh * 2};
    const cuuint32_t wbox[2] = {(cuuint32_t)rowh, (cuuint32_t)c.nout};
    const cuuint32_t westr[2] = {1, 1};
    __half* wptr = (__half*)ctx->d_tcw + ctx->tc_off[layer] + (size_t)nt * taps * 2 * c.nout * rowh;
    r = enc(&P.wmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)wptr, wdims, wstrides, wbox, westr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(weights, layer %d) failed: %d", layer, (int)r);
      return XF_E_CUDA;
    }
    P.bias = ctx->d_weights + ctx->table.b_off[layer] + nt * c.nout;
    P.f32_co0 = nt * c.nout;
    P.n_real = sp.cout - nt * c.nout < c.nout ? sp.cout - nt * c.nout : c.nout;
    int rc;
    if (sp.ks == 3 && c.cinp == 64 && c.nout == 64) rc = launch_tc_cfg<3, 64, 64>(P, grid, st);
    else if (sp.ks == 1 && c.cinp == 64 && c.nout == 64) rc = launch_tc_cfg<1, 64, 64>(P, grid, st);
    else if (sp.ks == 3 && c.cinp == 32 && c.nout == 32) rc = launch_tc_cfg<3, 32, 32>(P, grid, st);
    else if (sp.ks == 3 && c.cinp == 32 && c.nout == 64) rc = launch_tc_cfg<3, 32, 64>(P, grid, st);
    else if (sp.ks == 3 && c.cinp == 8 && c.nout == 32) rc = launch_tc_cfg<3, 8, 32>(P, grid, st);
    else {
      set_error("conv_tc: no kernel instantiation for layer %d", layer);
      return XF_E_UNSUPPORTED;
    }
    if (rc) return rc;
  }
  return XF_OK;
}

}  // namespace xf

// Test hooks: one eligible layer through the tensor-core kernel from fp32 NHWC input (the split of the input runs first); the
// _ex form also writes the split output the next layer reads and takes block1.3's skip input.
extern "C" int xfeat_debug_conv_layer_tc_ex(xfeat_ctx* ctx, int layer, const float* d_in, int B, int H, int W,
                                            float* d_out_f32, void* d_out_split, const float* d_skip_xn, void* d_scratch,
                                            size_t scratch_bytes, void* stream) {
  XF_REQUIRE(ctx && d_in && (d_out_f32 || d_out_split) && d_scratch && layer >= 0 && layer < xf::L_COUNT && B > 0 && H > 0 &&
                 W > 0,
             "debug_conv_layer_tc: bad arguments");
  XF_REQUIRE(xf::conv_tc_eligible(layer), "debug_conv_layer_tc: layer %d has no tensor-core configuration", layer);
  XF_REQUIRE(!d_skip_xn || layer == xf::L_B1_3, "debug_conv_layer_tc: the skip input belongs to block1.3 only");
  const int cin = xf::kLayers[layer].cin, cinp = cin <= 8 ? 8 : (cin <= 32 ? 32 : (cin <= 64 ? 64 : 128));
  const int64_t npix = (int64_t)B * H * W;
  XF_REQUIRE(scratch_bytes >= (size_t)npix * 4 * cinp, "debug_conv_layer_tc: scratch must hold B*H*W*%d bytes", 4 * cinp);
  XF_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = xf::launch_split_nhwc(d_in, (__half*)d_scratch, npix, cin, cinp, st);
  if (rc) return rc;
  return xf::launch_conv_tc(ctx, layer, (const __half*)d_scratch, B, H, W, (__half*)d_out_split, d_out_f32, st, d_skip_xn);
}

extern "C" int xfeat_debug_conv_layer_tc(xfeat_ctx* ctx, int layer, const float* d_in, int B, int H, int W, float* d_out,
                                         void* d_scratch, size_t scratch_bytes, void* stream) {
  XF_REQUIRE(d_out, "debug_conv_layer_tc: bad arguments");
  return xfeat_debug_conv_layer_tc_ex(ctx, layer, d_in, B, H, W, d_out, nullptr, nullptr, d_scratch, scratch_bytes, stream);
}
