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

// mode 0: keypoint head on the unfolded split image (npix = B*Hc*Wc cells) -> heat (B,8Hc,8Wc) [+ logits];
// mode 1: reliability head on the split feature map -> reliability (npix)
int launch_head_chain(const xfeat_ctx* ctx, int mode, const void* in, int B, int Hc, int Wc, float* out, float* logits,
                      cudaStream_t st) {
  // mode 0: `in` = normalised gray image (B, 8Hc, 8Wc) fp32; mode 1: `in` = split feature map (npix, 128 halves)
  const __half* in_split = (mode == 1) ? (const __half*)in : nullptr;
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  HeadChainParams P;
  const int64_t npix = (int64_t)B * Hc * Wc;
  const cuuint64_t dims[2] = {128, (cuuint64_t)npix};
  const cuuint64_t strides[1] = {256};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  if (mode == 1) {
    CUresult r = enc(&P.amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)in_split, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(head chain input) failed: %d", (int)r);
      return XF_E_CUDA;
    }
  } else {
    memset(&P.amap, 0, sizeof(P.amap));
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
  const int n_tiles = (int)((npix + 127) / 128);
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
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf
