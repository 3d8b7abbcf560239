// Fused 1x1 head chains on the Hopper tensor cores (wgmma): the activations of a 128-pixel tile never leave the SM between layers.
//   keypoint head   (model.py:87-92 + xfeat.py:242-247): 3 x [64->64 + BN + ReLU] -> 64->65 -> soft-max(65) -> drop dustbin
//                                                         -> 8x8 depth-to-space into the full-resolution heat-map
//   reliability head (model.py:79-84)                   : 2 x [64->64 + BN + ReLU] -> 64->1 -> sigmoid
// Per tile: TMA loads the split-fp16 input rows [hi(64)|lo(64)] once; each hidden layer is 3 split terms x 4 K-steps of wgmma
// (N = 64) per 64-row slab into registers; the warpgroup applies bias + ReLU, re-splits to fp16 and writes the NEXT layer's
// A operand straight back into shared memory in the 128B-swizzled K-major layout the MMA expects (generic-proxy stores +
// fence.proxy.async); the last GEMM (N = 80 / 16, zero padded) is followed by the soft-max or sigmoid in registers (one
// pixel per thread) and the only global write of the chain.
// Replaces 3 (2) conv launches + the SIMT soft-max kernel and their 4 (3) HBM round trips of 157 MB each.
// head_chain_kernel below is the reference form; xfeat_net runs head_chain_rf_kernel (layers chained in registers, further down).
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

constexpr int HC_THREADS = 160;   // warps 0-3: wgmma + epilogue warpgroup, warp 4: TMA producer
constexpr int HC_ABOX = 128 * 128;
constexpr int HC_WBOX = 64 * 128;

struct HeadChainParams {
  CUtensorMap amap;       // (npix, 128 halves) 2-D view of the split input; box {64, 128}
  CUtensorMap wmap[3];    // hidden layers: rows [group][64] x 64 halves
  CUtensorMap wfin;       // final layer: rows [group][NF] x 64 halves
  const float* bias[3];
  const float* bias_fin;
  float inv_ws[3];
  float inv_ws_fin;
  int64_t npix;
  int Hc, Wc;             // cells per image (keypoint head: heat-map geometry)
  const float* xn;        // keypoint head: normalised gray image (B, 8Hc, 8Wc); the 8x8 unfold + split happens in the kernel
  float* out;             // heat (B, 8Hc, 8Wc) or reliability (npix)
  float* logits;          // optional (npix, 65) raw logits (tests)
  // head_chain_rf_kernel<1> only: block_fusion.2 in front of the reliability head (amap = its input, fusion.1's split output)
  CUtensorMap wfu;        // rows [group][64] x 64 halves
  CUtensorMap fmap;       // fp32 feats as (npix, 64): 4-D map {64, npix, 1, 1}, boxes {16, 128, 1, 1}, SWIZZLE_64B
  const float* bias_fu;
  float inv_ws_fu;
};

// MODE 0: keypoint head (NH = 3 hidden layers, NF = 80); MODE 1: reliability head (NH = 2, NF = 16)
template <int MODE>
__global__ void __launch_bounds__(HC_THREADS, 1) head_chain_kernel(const __grid_constant__ HeadChainParams P) {
  constexpr int NH = (MODE == 0) ? 3 : 2;
  constexpr int NF = (MODE == 0) ? 80 : 16;
  constexpr int WF_GROUP = NF * 128;
  constexpr size_t W_BYTES = (size_t)NH * 2 * HC_WBOX + 2 * WF_GROUP;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sW = base;                                   // hidden weights, then final weights
  unsigned char* sWf = base + (size_t)NH * 2 * HC_WBOX;
  unsigned char* sA = base + ((W_BYTES + 1023) & ~(size_t)1023);   // 2 buffers x {hi box, lo box}
  float* sStg = reinterpret_cast<float*>(sA + 4 * (size_t)HC_ABOX);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sA + 4 * (size_t)HC_ABOX + tc::STG_BYTES);
  uint64_t* w_full = bars;
  uint64_t* a_full = bars + 1;      // [2]  TMA -> MMA (layer-0 operand of a tile, MODE 1)
  uint64_t* a_free = bars + 3;      // [2]  MMA -> TMA (all GEMMs of the tile that used this buffer have retired)
  float* sBias = reinterpret_cast<float*>(bars + 5);          // [NH][64] + [NF]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (int)((P.npix + 127) / 128);

  for (int i = threadIdx.x; i < NH * 64; i += HC_THREADS) sBias[i] = __ldg(P.bias[i / 64] + (i & 63));
  for (int i = threadIdx.x; i < NF; i += HC_THREADS) sBias[NH * 64 + i] = (i < (MODE == 0 ? 65 : 1)) ? __ldg(P.bias_fin + i) : 0.f;
  if (warp == 4 && lane == 0) {
    if constexpr (MODE == 1) tc::tma_prefetch_desc(&P.amap);
    tc::mbar_init(w_full, 1);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&a_full[i], 1);
      tc::mbar_init(&a_free[i], 4);   // one arrival per consumer warp
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      tc::mbar_expect_tx(w_full, (uint32_t)W_BYTES);
      for (int l = 0; l < NH; ++l)
        for (int g = 0; g < 2; ++g) tc::tma_load_2d(sW + (size_t)(l * 2 + g) * HC_WBOX, &P.wmap[l], w_full, 0, g * 64);
      for (int g = 0; g < 2; ++g) tc::tma_load_2d(sWf + (size_t)g * WF_GROUP, &P.wfin, w_full, 0, g * NF);
      if constexpr (MODE == 1) {   // (MODE 0: the warpgroup builds the layer-0 operand from the gray image itself)
        uint32_t tcount = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tcount) {
          const int s = tcount & 1;
          tc::mbar_wait(&a_free[s], ((tcount >> 1) & 1) ^ 1);
          tc::mbar_expect_tx(&a_full[s], 2 * HC_ABOX);
          tc::tma_load_2d(sA + (size_t)s * 2 * HC_ABOX, &P.amap, &a_full[s], 0, tile * 128);              // hi
          tc::tma_load_2d(sA + (size_t)s * 2 * HC_ABOX + HC_ABOX, &P.amap, &a_full[s], 64, tile * 128);   // lo
        }
      }
    }
    __syncwarp();
  } else {
    constexpr uint32_t HALF = (64 * 128) >> 4;   // descriptor offset of rows 64-127
    const int r = threadIdx.x;                   // pixel row of the tile
    tc::mbar_wait(w_full, 0);
    uint32_t tcount = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tcount) {
      const int s = (MODE == 0) ? 0 : (int)(tcount & 1);
      unsigned char* a_hi = sA + (size_t)s * 2 * HC_ABOX;
      unsigned char* a_lo = a_hi + HC_ABOX;
      const int64_t pix = (int64_t)tile * 128 + r;
      if constexpr (MODE == 0) {
        // ---- layer-0 operand: XFeatModel._unfold2d(x, 8) (model.py:113-120) + split, straight from the normalised gray image:
        // channel 8i+j of cell (h, w) = xn[8h+i, 8w+j].  The previous tile's GEMMs have all retired (wgmma_wait below). ----
        if (pix < P.npix) {
          const int64_t b = pix / ((int64_t)P.Hc * P.Wc);
          const int rem = (int)(pix - b * P.Hc * P.Wc);
          const int h = rem / P.Wc, wc = rem - h * P.Wc;
          const float* xp = P.xn + ((int64_t)b * P.Hc * 8 + (int64_t)h * 8) * (P.Wc * 8) + wc * 8;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(xp + (int64_t)i * (P.Wc * 8)));
            const float4 c = __ldg(reinterpret_cast<const float4*>(xp + (int64_t)i * (P.Wc * 8)) + 1);
            const float x[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const __half2 hh = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
              const float2 hf = __half22float2(hh);
              const __half2 lo = __floats2half2_rn(x[2 * j] - hf.x, x[2 * j + 1] - hf.y);
              hw[j] = *reinterpret_cast<const uint32_t*>(&hh);
              lw[j] = *reinterpret_cast<const uint32_t*>(&lo);
            }
            const int off = r * 128 + ((i ^ (r & 7)) << 4);      // 16-byte chunk i (channels 8i..8i+7) of row r, 128B swizzle
            *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int off = r * 128 + ((i ^ (r & 7)) << 4);
            *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(0u, 0u, 0u, 0u);
          }
        }
        tc::fence_proxy_async();        // generic-proxy smem writes -> visible to the tensor core (async proxy)
        tc::wg_sync(1);
      } else {
        tc::mbar_wait(&a_full[s], (tcount >> 1) & 1);
      }
      const uint32_t a_addr = tc::smem_u32(a_hi);
      const uint64_t ahi = tc::make_desc_sw128(a_addr, 1024), alo = tc::make_desc_sw128(a_addr + HC_ABOX, 1024);
#pragma unroll 1
      for (int l = 0; l < NH; ++l) {
        // ---- hidden layer: 64 -> 64, bias + ReLU, re-split, written back as the next A operand (chunk j of row r at j ^ (r & 7)) ----
        float acc0[32], acc1[32];
        const uint32_t w_addr = tc::smem_u32(sW + (size_t)l * 2 * HC_WBOX);
        const uint64_t whi = tc::make_desc_sw128(w_addr, 1024), wlo = tc::make_desc_sw128(w_addr + HC_WBOX, 1024);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<64>(acc0, ahi + 2 * k, whi + 2 * k, k ? 1u : 0u);
          tc::wgmma_f16<64>(acc1, ahi + HALF + 2 * k, whi + 2 * k, k ? 1u : 0u);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<64>(acc0, ahi + 2 * k, wlo + 2 * k, 1u);
          tc::wgmma_f16<64>(acc1, ahi + HALF + 2 * k, wlo + 2 * k, 1u);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<64>(acc0, alo + 2 * k, whi + 2 * k, 1u);
          tc::wgmma_f16<64>(acc1, alo + HALF + 2 * k, whi + 2 * k, 1u);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        uint32_t v0[32], v1[32];
        tc::acc_rows<32>(sStg, acc0, acc1, 0, r, 1, v0);    // (its barriers also order every warp's wgmma reads of sA
        tc::acc_rows<32>(sStg, acc0, acc1, 32, r, 1, v1);   //  before the operand is overwritten below)
        const float inv = P.inv_ws[l];
        const float* bs = sBias + l * 64;
#pragma unroll
        for (int c8 = 0; c8 < 8; ++c8) {
          uint32_t hw[4], lw[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 8 * c8 + 2 * j;
            const float x0 = fmaxf(fmaf(__uint_as_float(c < 32 ? v0[c & 31] : v1[c & 31]), inv, bs[c]), 0.f);
            const float x1 = fmaxf(fmaf(__uint_as_float(c + 1 < 32 ? v0[(c + 1) & 31] : v1[(c + 1) & 31]), inv, bs[c + 1]), 0.f);
            const __half2 h = __floats2half2_rn(x0, x1);
            const float2 hf = __half22float2(h);
            const __half2 lo = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
            hw[j] = *reinterpret_cast<const uint32_t*>(&h);
            lw[j] = *reinterpret_cast<const uint32_t*>(&lo);
          }
          const int off = r * 128 + ((c8 ^ (r & 7)) << 4);
          *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
          *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
        tc::fence_proxy_async();
        tc::wg_sync(1);
      }
      // ---- final layer: 64 -> NF (zero padded) ----
      float acc0[NF / 2], acc1[NF / 2];
      {
        const uint32_t w_addr = tc::smem_u32(sWf);
        const uint64_t whi = tc::make_desc_sw128(w_addr, 1024), wlo = tc::make_desc_sw128(w_addr + WF_GROUP, 1024);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<NF>(acc0, ahi + 2 * k, whi + 2 * k, k ? 1u : 0u);
          tc::wgmma_f16<NF>(acc1, ahi + HALF + 2 * k, whi + 2 * k, k ? 1u : 0u);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<NF>(acc0, ahi + 2 * k, wlo + 2 * k, 1u);
          tc::wgmma_f16<NF>(acc1, ahi + HALF + 2 * k, wlo + 2 * k, 1u);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          tc::wgmma_f16<NF>(acc0, alo + 2 * k, whi + 2 * k, 1u);
          tc::wgmma_f16<NF>(acc1, alo + HALF + 2 * k, whi + 2 * k, 1u);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (MODE == 1 && lane == 0) tc::mbar_arrive(&a_free[s]);   // last reader of this A buffer
      }
      if constexpr (MODE == 0) {
        // ---- keypoint logits: soft-max over 65, drop the dustbin, 8x8 depth-to-space (xfeat.py:242-247) ----
        uint32_t v0[32], v1[32], v2[16];
        tc::acc_rows<32>(sStg, acc0, acc1, 0, r, 1, v0);
        tc::acc_rows<32>(sStg, acc0, acc1, 32, r, 1, v1);
        tc::acc_rows<16>(sStg, acc0, acc1, 64, r, 1, v2);   // columns 64..79: only 64 (the dustbin) is meaningful
        if (pix < P.npix) {
          const float inv = P.inv_ws_fin;
          const float* bs = sBias + NH * 64;
          float z[65];
#pragma unroll
          for (int c = 0; c < 32; ++c) {
            z[c] = fmaf(__uint_as_float(v0[c]), inv, bs[c]);
            z[32 + c] = fmaf(__uint_as_float(v1[c]), inv, bs[32 + c]);
          }
          z[64] = fmaf(__uint_as_float(v2[0]), inv, bs[64]);
          if (P.logits) {
            float* lo = P.logits + pix * 65;
#pragma unroll
            for (int c = 0; c < 65; ++c) lo[c] = z[c];
          }
          float m = z[0];
#pragma unroll
          for (int c = 1; c < 65; ++c) m = fmaxf(m, z[c]);
          float sum = 0.f;
#pragma unroll
          // __expf / reciprocal-multiply: 1e-7 relative on every heat value that can pass the 0.05 threshold, far inside the
          // 5e-5 this tensor-core path is specified to (the fp32 CUDA-core path keeps expf and IEEE division)
          for (int c = 0; c < 65; ++c) { z[c] = __expf(z[c] - m); sum += z[c]; }
          const float rs = __fdiv_rn(1.0f, sum);
          const int64_t b = pix / ((int64_t)P.Hc * P.Wc);
          const int rem = (int)(pix - b * P.Hc * P.Wc);
          const int h = rem / P.Wc, w = rem - h * P.Wc;
          const int Wf = P.Wc * 8;
          float* hp = P.out + ((int64_t)b * P.Hc * 8 + h * 8) * Wf + w * 8;
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // channel 8i+j -> pixel (8h+i, 8w+j): one 32-byte row piece per store
            uint32_t v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = __float_as_uint(z[8 * i + j] * rs);
            tc::st_global_v8(hp + (int64_t)i * Wf, v);
          }
        }
      } else {
        // ---- reliability: 64 -> 1 + sigmoid (model.py:82-83) ----
        uint32_t v0[16];
        tc::acc_rows<16>(sStg, acc0, acc1, 0, r, 1, v0);
        if (pix < P.npix) {
          const float zz = fmaf(__uint_as_float(v0[0]), P.inv_ws_fin, sBias[NH * 64]);
          P.out[pix] = 1.0f / (1.0f + expf(-zz));
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// head_chain_rf_kernel: the same chains with the activations handed from layer to layer in registers, two tiles in flight per SM.
// Each hidden layer's accumulator fragment, after bias + ReLU + split, is the A operand of the next layer as it stands
// (tc::wgmma_f16_ra), so no activation goes back to shared memory and no barrier or proxy fence separates the layers.  Every
// GEMM keeps head_chain_kernel's shapes, k order and split terms and every value its float operations, so the outputs are the
// same bits.  Two consumer warpgroups run independent tiles on one copy of the weights (two CTAs per SM would need two copies).
//   keypoint head: each thread copies the gray pixels of its own fragment rows for the NEXT tile with cp.async while the
//                  current tile's GEMMs run (no barrier: a thread reads only what it copied); the final layer's logits reach
//                  one-row-per-thread through the warpgroup's staging buffer for the channel-order soft-max.
//   block_fusion.2 + reliability head (MODE 1): one thread of each warpgroup TMA-loads fusion.1's split output into a two-slot
//                  ring; fusion.2 runs conv_tc_kernel<1,64,64>'s sequence on it (hi.[whi;wlo] at N = 128, then lo.whi at
//                  N = 64 into the first half), and a slot is reloaded as soon as that has retired.  Its epilogue is
//                  tc::conv_values (fmaf(g0 + g1, inv_ws, bias), no ReLU): the fp32 feats leave by TMA stores, and the split
//                  values are the first hidden layer's register A operand, so the split copy of feats is never written.  The
//                  sigmoid runs on the column-0 fragments (lanes with l % 4 == 0).
// 256 threads: ptxas caps a kernel of nine warps at 168 registers per thread (measured: three of the nine warps share one of
// the SM's four 16K-register scheduler partitions), and these kernels need up to 244.
constexpr int HR_THREADS = 256;
constexpr int HR_XBUF = 32 * 128 * 8;   // keypoint head: 32 float2 per thread of a warpgroup

__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// hi.whi, hi.wlo, lo.whi over 4 k-steps into one accumulator per slab, A from registers ([slab][k-step][4])
template <int N>
__device__ __forceinline__ void gemm_split_ra(float (&acc0)[N / 2], float (&acc1)[N / 2], const uint32_t (&ahi)[2][4][4],
                                              const uint32_t (&alo)[2][4][4], uint64_t whi, uint64_t wlo) {
  tc::wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    tc::wgmma_f16_ra<N>(acc0, ahi[0][k], whi + 2 * k, k ? 1u : 0u);
    tc::wgmma_f16_ra<N>(acc1, ahi[1][k], whi + 2 * k, k ? 1u : 0u);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    tc::wgmma_f16_ra<N>(acc0, ahi[0][k], wlo + 2 * k, 1u);
    tc::wgmma_f16_ra<N>(acc1, ahi[1][k], wlo + 2 * k, 1u);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    tc::wgmma_f16_ra<N>(acc0, alo[0][k], whi + 2 * k, 1u);
    tc::wgmma_f16_ra<N>(acc1, alo[1][k], whi + 2 * k, 1u);
  }
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::acc_fence(acc0);
  tc::acc_fence(acc1);
}

// hidden-layer epilogue on the fragment: bias + ReLU + split; element d[8k + 2m + e] (column 16k + 8(m/2) + 2q + e) goes to
// A register m of k-step k
__device__ __forceinline__ void hidden_to_frag(const float (&d)[32], float inv, const float* bs, int q, uint32_t (&hi)[4][4],
                                               uint32_t (&lo)[4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int n = 8 * k + 2 * m, c = 16 * k + 8 * (m >> 1) + 2 * q;
      const float x0 = fmaxf(fmaf(d[n], inv, bs[c]), 0.f);
      const float x1 = fmaxf(fmaf(d[n + 1], inv, bs[c + 1]), 0.f);
      split_pair(x0, x1, hi[k][m], lo[k][m]);
    }
}

// keypoint head: cp.async of the gray pixels this thread's layer-0 fragments need: for fragment row h (tile rows r, r+8, r+64,
// r+72) and patch row i, columns 2q, 2q+1 of the cell's 8x8 patch, into float2 slot (8h + i) * 128 + wt of the warpgroup's
// buffer (the thread's own slots, so no barrier orders the copy and the reads); cells past npix are zero-filled
__device__ __forceinline__ void kp_prefetch(const HeadChainParams& P, int tile, int wt, float2* xb) {
  const int q = wt & 3;
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    const int64_t pix = (int64_t)tile * 128 + tc::frag_row(wt, h);
    const float* src = P.xn;
    uint32_t bytes = 0;
    int64_t stride = 0;
    if (pix < P.npix) {
      const int64_t b = pix / ((int64_t)P.Hc * P.Wc);
      const int rem = (int)(pix - b * P.Hc * P.Wc);
      const int hh = rem / P.Wc, wc = rem - hh * P.Wc;
      src = P.xn + ((int64_t)b * P.Hc * 8 + (int64_t)hh * 8) * (P.Wc * 8) + wc * 8 + 2 * q;
      bytes = 8;
      stride = (int64_t)P.Wc * 8;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) tc::cp_async8(xb + (h * 8 + i) * 128 + wt, src + i * stride, bytes);
  }
  tc::cp_async_commit();
}

template <int MODE>
__global__ void __launch_bounds__(HR_THREADS, 1) head_chain_rf_kernel(const __grid_constant__ HeadChainParams P) {
  constexpr int NH = (MODE == 0) ? 3 : 2;
  constexpr int NF = (MODE == 0) ? 80 : 16;
  constexpr int WF_GROUP = NF * 128;
  constexpr size_t FU_BYTES = (MODE == 1) ? 2 * (size_t)HC_WBOX : 0;   // block_fusion.2 weights [whi; wlo]
  constexpr size_t W_BYTES = FU_BYTES + (size_t)NH * 2 * HC_WBOX + 2 * WF_GROUP;
  constexpr size_t IN_BYTES = (MODE == 0) ? (size_t)HR_XBUF : 4 * (size_t)HC_ABOX;   // per warpgroup: input, then staging
  constexpr size_t WG_BYTES = IN_BYTES + tc::STG_BYTES;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sFu = base;
  unsigned char* sW = base + FU_BYTES;
  unsigned char* sWf = sW + (size_t)NH * 2 * HC_WBOX;
  unsigned char* sG = base + ((W_BYTES + 1023) & ~(size_t)1023);   // [2] warpgroup regions
  uint64_t* bars = reinterpret_cast<uint64_t*>(sG + 2 * WG_BYTES);
  uint64_t* w_full = bars;
  uint64_t* a_full = bars + 1;      // [warpgroup][slot]  TMA -> MMA (reliability head)
  uint64_t* a_free = bars + 5;      // [warpgroup][slot]  layer 0 of the tile in this slot has retired
  float* sBias = reinterpret_cast<float*>(bars + 9);          // [NH][64] + [NF] (+ [64] block_fusion.2)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (int)((P.npix + 127) / 128);
  const int g = warp >> 2;                 // warpgroup
  const int wt = threadIdx.x & 127;        // thread of the warpgroup
  const int q = lane & 3;
  unsigned char* sGw = sG + g * WG_BYTES;
  const int tile0 = blockIdx.x + g * gridDim.x, tstride = 2 * gridDim.x;
  const bool issuer = (wt >> 5) == 0 && tc::elect_one();   // one thread of warp 0 of each warpgroup issues its TMA loads
  // reliability head: TMA of tile cc of this warpgroup (hi and lo boxes) into slot cc % 2
  auto load_tile = [&](uint32_t cc) {
    const int slot = g * 2 + (int)(cc & 1);
    unsigned char* dst = sGw + (cc & 1) * 2 * (size_t)HC_ABOX;
    const int t = tile0 + (int)cc * tstride;
    tc::mbar_expect_tx(&a_full[slot], 2 * HC_ABOX);
    tc::tma_load_2d(dst, &P.amap, &a_full[slot], 0, t * 128);              // hi
    tc::tma_load_2d(dst + HC_ABOX, &P.amap, &a_full[slot], 64, t * 128);   // lo
  };

  for (int i = threadIdx.x; i < NH * 64; i += HR_THREADS) sBias[i] = __ldg(P.bias[i / 64] + (i & 63));
  for (int i = threadIdx.x; i < NF; i += HR_THREADS) sBias[NH * 64 + i] = (i < (MODE == 0 ? 65 : 1)) ? __ldg(P.bias_fin + i) : 0.f;
  if constexpr (MODE == 1)
    for (int i = threadIdx.x; i < 64; i += HR_THREADS) sBias[NH * 64 + NF + i] = __ldg(P.bias_fu + i);
  if (threadIdx.x == 0) {
    if constexpr (MODE == 1) {
      tc::tma_prefetch_desc(&P.amap);
      tc::tma_prefetch_desc(&P.fmap);
    }
    tc::mbar_init(w_full, 1);
    for (int i = 0; i < 4; ++i) {
      tc::mbar_init(&a_full[i], 1);
      tc::mbar_init(&a_free[i], 4);   // one arrival per warp of the warpgroup
    }
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (g == 0 && issuer) {
    tc::mbar_expect_tx(w_full, (uint32_t)W_BYTES);
    if constexpr (MODE == 1)
      for (int k = 0; k < 2; ++k) tc::tma_load_2d(sFu + (size_t)k * HC_WBOX, &P.wfu, w_full, 0, k * 64);
    for (int l = 0; l < NH; ++l)
      for (int k = 0; k < 2; ++k) tc::tma_load_2d(sW + (size_t)(l * 2 + k) * HC_WBOX, &P.wmap[l], w_full, 0, k * 64);
    for (int k = 0; k < 2; ++k) tc::tma_load_2d(sWf + (size_t)k * WF_GROUP, &P.wfin, w_full, 0, k * NF);
  }
  float2* xb = reinterpret_cast<float2*>(sGw);                            // MODE 0
  unsigned char* sStg = sGw + IN_BYTES;
  if constexpr (MODE == 0) {
    if (tile0 < n_tiles) kp_prefetch(P, tile0, wt, xb);
  } else if (issuer) {
    for (uint32_t cc = 0; cc < 2; ++cc)
      if (tile0 + (int)cc * tstride < n_tiles) load_tile(cc);
  }
  tc::mbar_wait(w_full, 0);
  uint32_t c = 0, piece = 0;
  for (int tile = tile0; tile < n_tiles; tile += tstride, ++c) {
    uint32_t ahi[2][4][4], alo[2][4][4];
    if constexpr (MODE == 0) {
      // ---- layer-0 operand: channel 8i+j of cell (h, w) = xn[8h+i, 8w+j] (model.py:113-120), split ----
      tc::cp_async_wait_all();
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int m = 0; m < 4; ++m) {
            const float2 x = xb[((2 * s + (m & 1)) * 8 + 2 * k + (m >> 1)) * 128 + wt];
            split_pair(x.x, x.y, ahi[s][k][m], alo[s][k][m]);
          }
      if (tile + tstride < n_tiles) kp_prefetch(P, tile + tstride, wt, xb);
    } else {
      // ---- block_fusion.2 from the TMA-loaded split rows in shared memory, as conv_tc_kernel<1,64,64> ----
      constexpr uint32_t HALF = (64 * 128) >> 4;   // descriptor offset of rows 64-127
      const int slot = g * 2 + (int)(c & 1);
      tc::mbar_wait(&a_full[slot], (c >> 1) & 1);
      const uint32_t a_addr = tc::smem_u32(sGw + (c & 1) * 2 * (size_t)HC_ABOX);
      const uint64_t dhi = tc::make_desc_sw128(a_addr, 1024), dlo = tc::make_desc_sw128(a_addr + HC_ABOX, 1024);
      const uint64_t wfu = tc::make_desc_sw128(tc::smem_u32(sFu), 1024);   // [whi; wlo]: N = 128
      float g0[64], g1[64];   // rows 0-63 / 64-127; columns [0,64) hi.whi + lo.whi, [64,128) hi.wlo
      tc::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {   // hi.whi | hi.wlo
        tc::wgmma_f16<128>(g0, dhi + 2 * k, wfu + 2 * k, k ? 1u : 0u);
        tc::wgmma_f16<128>(g1, dhi + HALF + 2 * k, wfu + 2 * k, k ? 1u : 0u);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {   // lo.whi
        tc::wgmma_f16<64>(tc::acc_head<64>(g0), dlo + 2 * k, wfu + 2 * k, 1u);
        tc::wgmma_f16<64>(tc::acc_head<64>(g1), dlo + HALF + 2 * k, wfu + 2 * k, 1u);
      }
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      tc::acc_fence(g0);
      tc::acc_fence(g1);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&a_free[slot]);
      if (issuer && tile + 2 * tstride < n_tiles) {   // the slot is free once all four warps' fusion.2 GEMMs have retired
        tc::mbar_wait(&a_free[slot], (c >> 1) & 1);
        load_tile(c + 2);
      }
      // ---- epilogue: feats = fmaf(g0 + g1, inv_ws, bias) to HBM by TMA stores (rows past npix are clipped); its split
      // is the first hidden layer's A operand: value (fragment row h, column 8j + 2q + e) -> slab h/2, k-step j/2,
      // register 2(j%2) + h%2 ----
      tc::ConvEpi E;
      E.split = nullptr;
      E.f32 = &P.fmap;
      E.split_c = 64;
      E.co = 0;
      E.inv_wscale = P.inv_ws_fu;
      E.relu = 0;
      E.bias = sBias + NH * 64 + NF;
      E.skip_w = nullptr;
      E.skip_v = nullptr;
      E.x0 = tile * 128;
      E.y0 = 0;
      E.b = 0;
      E.wg = g;
      const float sv[4] = {0.f, 0.f, 0.f, 0.f};
      int srow[4];
#pragma unroll
      for (int h = 0; h < 4; ++h) srow[h] = tc::frag_row(wt, h);
#pragma unroll
      for (int cb = 0; cb < 2; ++cb) {
        float o[4][4][2];
        uint32_t hi[4][4], lo[4][4];
        tc::conv_values<64>(g0, g1, cb, sv, E, o, hi, lo);
#pragma unroll
        for (int h = 0; h < 4; ++h)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * cb + jj;
            ahi[h >> 1][j >> 1][2 * (j & 1) + (h & 1)] = hi[h][jj];
            alo[h >> 1][j >> 1][2 * (j & 1) + (h & 1)] = lo[h][jj];
          }
#pragma unroll
        for (int k = 0; k < 2; ++k)   // 16 channels (64-byte rows) per piece, as tc::conv_epilogue
          tc::conv_store_piece(sStg, piece, E.f32, 32 * cb + 16 * k, E, [&](unsigned char* buf) {
#pragma unroll
            for (int h = 0; h < 4; ++h)
#pragma unroll
              for (int jj = 0; jj < 2; ++jj)
                *reinterpret_cast<float2*>(buf + tc::piece_off<64>(srow[h], 32 * jj + 8 * q)) =
                    make_float2(o[h][2 * k + jj][0], o[h][2 * k + jj][1]);
          });
      }
    }
    float acc0[32], acc1[32];
#pragma unroll 1
    for (int l = 0; l < NH; ++l) {
      const uint32_t w_addr = tc::smem_u32(sW + (size_t)l * 2 * HC_WBOX);
      gemm_split_ra<64>(acc0, acc1, ahi, alo, tc::make_desc_sw128(w_addr, 1024), tc::make_desc_sw128(w_addr + HC_WBOX, 1024));
      hidden_to_frag(acc0, P.inv_ws[l], sBias + l * 64, q, ahi[0], alo[0]);
      hidden_to_frag(acc1, P.inv_ws[l], sBias + l * 64, q, ahi[1], alo[1]);
    }
    // ---- final layer: 64 -> NF (zero padded) ----
    float f0[NF / 2], f1[NF / 2];
    {
      const uint32_t w_addr = tc::smem_u32(sWf);
      gemm_split_ra<NF>(f0, f1, ahi, alo, tc::make_desc_sw128(w_addr, 1024), tc::make_desc_sw128(w_addr + WF_GROUP, 1024));
    }
    if constexpr (MODE == 0) {
      // ---- keypoint logits: soft-max over 65, drop the dustbin, 8x8 depth-to-space (xfeat.py:242-247), as head_chain_kernel ----
      const int64_t pix = (int64_t)tile * 128 + wt;
      uint32_t v0[32], v1[32], v2[16];
      tc::acc_rows<32>(reinterpret_cast<float*>(sStg), f0, f1, 0, wt, 1 + g, v0);
      tc::acc_rows<32>(reinterpret_cast<float*>(sStg), f0, f1, 32, wt, 1 + g, v1);
      tc::acc_rows<16>(reinterpret_cast<float*>(sStg), f0, f1, 64, wt, 1 + g, v2);
      if (pix < P.npix) {
        const float inv = P.inv_ws_fin;
        const float* bs = sBias + NH * 64;
        float z[65];
#pragma unroll
        for (int cc = 0; cc < 32; ++cc) {
          z[cc] = fmaf(__uint_as_float(v0[cc]), inv, bs[cc]);
          z[32 + cc] = fmaf(__uint_as_float(v1[cc]), inv, bs[32 + cc]);
        }
        z[64] = fmaf(__uint_as_float(v2[0]), inv, bs[64]);
        if (P.logits) {
          float* lo = P.logits + pix * 65;
#pragma unroll
          for (int cc = 0; cc < 65; ++cc) lo[cc] = z[cc];
        }
        float m = z[0];
#pragma unroll
        for (int cc = 1; cc < 65; ++cc) m = fmaxf(m, z[cc]);
        float sum = 0.f;
#pragma unroll
        for (int cc = 0; cc < 65; ++cc) { z[cc] = __expf(z[cc] - m); sum += z[cc]; }
        const float rs = __fdiv_rn(1.0f, sum);
        const int64_t b = pix / ((int64_t)P.Hc * P.Wc);
        const int rem = (int)(pix - b * P.Hc * P.Wc);
        const int h = rem / P.Wc, w = rem - h * P.Wc;
        const int Wf = P.Wc * 8;
        float* hp = P.out + ((int64_t)b * P.Hc * 8 + h * 8) * Wf + w * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          uint32_t v[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = __float_as_uint(z[8 * i + j] * rs);
          tc::st_global_v8(hp + (int64_t)i * Wf, v);
        }
      }
    } else {
      // ---- reliability: 64 -> 1 + sigmoid (model.py:82-83) on column 0: fragment rows r, r+8, r+64, r+72 ----
      if (q == 0) {
        const float vals[4] = {f0[0], f0[2], f1[0], f1[2]};
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int64_t pix = (int64_t)tile * 128 + tc::frag_row(wt, h);
          if (pix < P.npix) {
            const float zz = fmaf(vals[h], P.inv_ws_fin, sBias[NH * 64]);
            P.out[pix] = 1.0f / (1.0f + expf(-zz));
          }
        }
      }
    }
  }
  if constexpr (MODE == 1)
    if (wt == 0) tc::bulk_wait_all();   // the feats stores have completed
}

static int make_w_map(CUtensorMap* m, const __half* ptr, int rows_per_group) {
  PFN_encodeTiled enc = get_encode_tiled();
  const cuuint64_t dims[2] = {64, (cuuint64_t)2 * rows_per_group};
  const cuuint64_t strides[1] = {128};
  const cuuint32_t box[2] = {64, (cuuint32_t)rows_per_group};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(head chain weights) failed: %d", (int)r);
    return XF_E_CUDA;
  }
  return XF_OK;
}

// Input map, weights and outputs of a head chain.  mode 0: keypoint head, `in` = normalised gray image (B, 8Hc, 8Wc) fp32;
// mode 1: reliability head, `in` = split rows (npix, 128 halves): the features (head_chain_kernel<1>) or fusion.1's output
// (head_chain_rf_kernel<1>, which runs block_fusion.2 first).
static int make_head_params(const xfeat_ctx* ctx, int mode, const void* in, int B, int Hc, int Wc, float* out, float* logits,
                            HeadChainParams& P) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  memset(&P, 0, sizeof(P));
  const int64_t npix = (int64_t)B * Hc * Wc;
  if (mode == 1) {
    const cuuint64_t dims[2] = {128, (cuuint64_t)npix};
    const cuuint64_t strides[1] = {256};
    const cuuint32_t box[2] = {64, 128};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&P.amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(in), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(head chain input) failed: %d", (int)r);
      return XF_E_CUDA;
    }
  }
  P.xn = (mode == 0) ? (const float*)in : nullptr;
  const int hidden0 = (mode == 0) ? L_KH_0 : L_HH_0, nh = (mode == 0) ? 3 : 2, lfin = (mode == 0) ? L_KH_3 : L_HH_2;
  int rc;
  for (int l = 0; l < nh; ++l) {
    if ((rc = make_w_map(&P.wmap[l], (const __half*)ctx->d_tcw + ctx->tc_off[hidden0 + l], 64))) return rc;
    P.bias[l] = ctx->d_weights + ctx->table.b_off[hidden0 + l];
    P.inv_ws[l] = ctx->tc_inv_wscale[hidden0 + l];
  }
  if (nh == 2) { P.wmap[2] = P.wmap[1]; P.bias[2] = P.bias[1]; P.inv_ws[2] = 1.f; }
  if ((rc = make_w_map(&P.wfin, (const __half*)ctx->d_tcw + ctx->tc_off[lfin], mode == 0 ? 80 : 16))) return rc;
  P.bias_fin = ctx->d_weights + ctx->table.b_off[lfin];
  P.inv_ws_fin = ctx->tc_inv_wscale[lfin];
  P.npix = npix;
  P.Hc = Hc; P.Wc = Wc;
  P.out = out;
  P.logits = logits;
  return XF_OK;
}

// mode 0: keypoint head on the gray image -> heat (B,8Hc,8Wc) [+ logits]; head_chain_rf_kernel<0>, or with `reference`
// head_chain_kernel<0>.  mode 1: reliability head on the split features -> reliability (npix), head_chain_kernel<1>: the
// reference of launch_fusion_reliability.  The tests hold each pair to the same bits.
int launch_head_chain(const xfeat_ctx* ctx, int mode, const void* in, int B, int Hc, int Wc, float* out, float* logits,
                      cudaStream_t st, bool reference) {
  HeadChainParams P;
  int rc = make_head_params(ctx, mode, in, B, Hc, Wc, out, logits, P);
  if (rc) return rc;
  const int n_tiles = (int)((P.npix + 127) / 128);
  if (reference || mode == 1) {
    const int grid = n_tiles < ctx->sm_count ? n_tiles : ctx->sm_count;
    const size_t smem0 = 1024 + (((size_t)3 * 2 * HC_WBOX + 2 * 80 * 128 + 1023) & ~(size_t)1023) + 4 * (size_t)HC_ABOX + tc::STG_BYTES + 2048;
    const size_t smem1 = 1024 + (((size_t)2 * 2 * HC_WBOX + 2 * 16 * 128 + 1023) & ~(size_t)1023) + 4 * (size_t)HC_ABOX + tc::STG_BYTES + 2048;
    if (mode == 0) {
      XF_DYN_SMEM(head_chain_kernel<0>, smem0);
      head_chain_kernel<0><<<grid, HC_THREADS, smem0, st>>>(P);
    } else {
      XF_DYN_SMEM(head_chain_kernel<1>, smem1);
      head_chain_kernel<1><<<grid, HC_THREADS, smem1, st>>>(P);
    }
  } else {
    // two warpgroups per CTA, one CTA per SM (the shared memory allows no second)
    const int pairs = (n_tiles + 1) / 2;
    const int grid = pairs < ctx->sm_count ? pairs : ctx->sm_count;
    const size_t smem0 = 1024 + (((size_t)3 * 2 * HC_WBOX + 2 * 80 * 128 + 1023) & ~(size_t)1023) + 2 * ((size_t)HR_XBUF + tc::STG_BYTES) + 2048;
    XF_DYN_SMEM(head_chain_rf_kernel<0>, smem0);
    head_chain_rf_kernel<0><<<grid, HR_THREADS, smem0, st>>>(P);
  }
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// block_fusion.2 + reliability head in one kernel (head_chain_rf_kernel<1>): `f1_split` = fusion.1's split output
// (npix, [hi(64) | lo(64)]) -> feats (B,Hc,Wc,64) fp32 and reliability (npix).  Computes what launch_conv_tc(L_FU_2) followed
// by launch_head_chain(mode 1) computes, without writing the split copy of feats.
int launch_fusion_reliability(const xfeat_ctx* ctx, const __half* f1_split, int B, int Hc, int Wc, float* feats, float* rel,
                              cudaStream_t st) {
  XF_REQUIRE(conv_tc_eligible(L_FU_2), "fusion_reliability: block_fusion.2 is not prepared for the tensor cores");
  const int64_t npix = (int64_t)B * Hc * Wc;
  XF_REQUIRE(npix < (int64_t)1 << 31, "fusion_reliability: too many cells (%lld)", (long long)npix);
  HeadChainParams P;
  int rc = make_head_params(ctx, 1, f1_split, B, Hc, Wc, rel, nullptr, P);
  if (rc) return rc;
  if ((rc = make_w_map(&P.wfu, (const __half*)ctx->d_tcw + ctx->tc_off[L_FU_2], 64))) return rc;
  P.bias_fu = ctx->d_weights + ctx->table.b_off[L_FU_2];
  P.inv_ws_fu = ctx->tc_inv_wscale[L_FU_2];
  CUtensorMap unused;
  if ((rc = encode_conv_out_maps(get_encode_tiled(), &unused, nullptr, 64, &P.fmap, feats, 64, false, 1, 1, (int)npix, 128, 1)))
    return rc;
  const int n_tiles = (int)((npix + 127) / 128);
  const int pairs = (n_tiles + 1) / 2;
  const int grid = pairs < ctx->sm_count ? pairs : ctx->sm_count;
  const size_t smem = 1024 + (((size_t)3 * 2 * HC_WBOX + 2 * 16 * 128 + 1023) & ~(size_t)1023) +
                      2 * (4 * (size_t)HC_ABOX + tc::STG_BYTES) + 2048;
  XF_DYN_SMEM(head_chain_rf_kernel<1>, smem);
  head_chain_rf_kernel<1><<<grid, HR_THREADS, smem, st>>>(P);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf

// Test hook: block_fusion.1's fp32 output is split as xfeat_debug_conv_layer_tc_ex splits it, then
//   variant 0: block_fusion.2 on conv_tc_kernel<1,64,64> (feats + split copy), head_chain_kernel<1>, head_chain_kernel<0>;
//   variant 1: what xfeat_net runs, head_chain_rf_kernel<1> (block_fusion.2 + reliability head), head_chain_rf_kernel<0>.
extern "C" int xfeat_debug_heads(xfeat_ctx* ctx, int variant, const float* d_f1, const float* d_xn, int B, int Hc, int Wc,
                                 float* d_feats, float* d_heat, float* d_rel, float* d_logits, void* d_scratch, size_t scratch_bytes,
                                 void* stream) {
  XF_REQUIRE(ctx && d_f1 && d_xn && d_feats && d_heat && d_rel && d_scratch && (variant == 0 || variant == 1) && B > 0 && Hc > 0 &&
                 Wc > 0,
             "debug_heads: bad arguments");
  const int64_t npix = (int64_t)B * Hc * Wc;
  XF_REQUIRE(scratch_bytes >= (size_t)npix * 512, "debug_heads: scratch must hold B*Hc*Wc*512 bytes");
  XF_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  __half* s_in = (__half*)d_scratch;
  __half* s_out = s_in + npix * 128;
  int rc = xf::launch_split_nhwc(d_f1, s_in, npix, 64, 64, st);
  if (rc) return rc;
  if (variant == 0) {
    rc = xf::launch_conv_tc(ctx, xf::L_FU_2, s_in, B, Hc, Wc, s_out, d_feats, st);
    if (!rc) rc = xf::launch_head_chain(ctx, 1, s_out, B, Hc, Wc, d_rel, nullptr, st, true);
  } else {
    rc = xf::launch_fusion_reliability(ctx, s_in, B, Hc, Wc, d_feats, d_rel, st);
  }
  if (!rc) rc = xf::launch_head_chain(ctx, 0, d_xn, B, Hc, Wc, d_heat, d_logits, st, variant == 0);
  return rc;
}
