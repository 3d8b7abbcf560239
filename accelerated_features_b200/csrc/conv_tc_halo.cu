// 3x3 / stride-1 convolution on the Hopper tensor cores (wgmma) with HALO-PATCH operand reuse.
//
// conv_tc_kernel re-reads the input patch once per tap (9x the activation bytes through L2).  Here the haloed patch
// (TH+2) x (TW+2) pixels is loaded ONCE per tile by a single 4-D TMA box into a 128B-swizzled K-major array whose rows
// are the patch pixels in raster order (pitch PW = TW + 2).  If the GEMM rows are enumerated with the same pitch,
//      m = h * PW + w      (h < TH, w < PW; columns w >= TW are junk lanes that are never stored)
// then the A operand of tap (dy,dx) is the SAME array shifted by a constant number of rows:
//      row(m, tap) = m + dy * PW + dx
// i.e. the tap is selected by advancing the shared-memory matrix descriptor's start address by (dy*PW+dx)*128 bytes
// (not 1024-aligned in general; the 128B swizzle is applied on physical address bits, so the shifted descriptor keeps
// base_offset = 0 -- see tests/test_gpu_conv_halo.py, which checks both settings).
// TH * PW <= 128, so a tile yields TH*TW valid pixels out of 128 MMA rows (TW = 40: 120/128).
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

constexpr int CH_THREADS = 160;   // warps 0-3: wgmma + epilogue warpgroup, warp 4: TMA producer
constexpr int CH_PATCH_BYTES = 34816;   // CINP=32: >= (2*PW + 2 + 128) * 128 for PW <= 66, multiple of 1024
constexpr int CH_PATCH64_BYTES = 27648; // CINP=64: PW <= 42 (TW <= 40): 214 rows x 128 B

template <int CINP, int NOUT>
struct HaloCfg {
  static constexpr int ROWB = (CINP == 8) ? 32 : 128;     // bytes per operand row: [hi(8)|lo(8)] halves, or 64 halves
  static constexpr int KSTEPS = ROWB / 32;                // wgmma K = 16 halves = 32 B
  static constexpr int W_GROUP = NOUT * ROWB;
  static constexpr size_t W_BYTES = (size_t)9 * 2 * W_GROUP;
  // patch buffers: CINP=32 -> 4-deep ring over tiles; CINP=64 -> hi and lo buffer (the 144 KB of weights leave no room for more)
  static constexpr int NP = (CINP == 64) ? 2 : (CINP == 32 ? 4 : 16);
  static constexpr int PB = (CINP == 64) ? CH_PATCH64_BYTES : (CINP == 32 ? CH_PATCH_BYTES : CH_PATCH_BYTES / 4);
  static constexpr size_t SMEM = 1024 + W_BYTES + NP * (size_t)PB + tc::STG_BYTES + 1024;
};

struct HaloParams {
  CUtensorMap amap;   // (B,H,W,2*CINP) halves; box {64, PW, TH+2, 1}
  CUtensorMap wmap;
  const float* bias;
  float inv_wscale;
  int B, H, W;
  int TW, TH, PW;
  __half* out_split;
  float* out_f32;
  int f32_c, n_real;
  int relu;
  FastDiv div_img, div_x;
  int desc_mode;      // 0 (default): base_offset = 0; 1: base_offset = (addr >> 7) & 7 (bring-up experiment)
};

__device__ __forceinline__ uint64_t make_desc_sw128_at(uint32_t smem_addr, uint32_t sbo_bytes, int mode) {
  uint64_t d = tc::make_desc_sw128(smem_addr, sbo_bytes);
  if (mode) d |= (uint64_t)((smem_addr >> 7) & 7) << 49;
  return d;
}
template <int ROWB>
__device__ __forceinline__ uint64_t make_desc_rows_at(uint32_t smem_addr, int mode) {
  return ROWB == 128 ? make_desc_sw128_at(smem_addr, 1024, mode) : tc::make_desc_sw32(smem_addr, 256);
}

template <int CINP, int NOUT>
__global__ void __launch_bounds__(CH_THREADS, 1) conv_tc_halo_kernel(const __grid_constant__ HaloParams P) {
  using C = HaloCfg<CINP, NOUT>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sW = base;
  unsigned char* sP = base + C::W_BYTES;                     // patch buffers
  constexpr int NP = C::NP;
  constexpr int PB = C::PB;
  float* sStg = reinterpret_cast<float*>(base + C::W_BYTES + NP * PB);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + C::W_BYTES + NP * PB + tc::STG_BYTES);
  uint64_t* w_full = bars;
  uint64_t* p_full = bars + 1;            // [NP]
  uint64_t* p_empty = bars + 1 + NP;      // [NP]
  float* sBias = reinterpret_cast<float*>(bars + 1 + 2 * NP);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_x = (P.W + P.TW - 1) / P.TW, tiles_y = (P.H + P.TH - 1) / P.TH;
  const int tiles_img = tiles_x * tiles_y;
  const int n_tiles = tiles_img * P.B;
  constexpr int ROWB = C::ROWB, KSTEPS = C::KSTEPS;
  const uint32_t patch_tx = (uint32_t)(P.TH + 2) * P.PW * ROWB;

  if (threadIdx.x < NOUT) sBias[threadIdx.x] = (threadIdx.x < P.n_real) ? __ldg(P.bias + threadIdx.x) : 0.f;
  if (warp == 4 && lane == 0) {
    tc::tma_prefetch_desc(&P.amap);
    tc::tma_prefetch_desc(&P.wmap);
    tc::mbar_init(w_full, 1);
    for (int i = 0; i < NP; ++i) {
      tc::mbar_init(&p_full[i], 1);
      tc::mbar_init(&p_empty[i], 4);   // one arrival per consumer warp
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  // CINP = 64: buffer 0 = hi patch, buffer 1 = lo patch of the SAME tile (the hi MMAs of a tile run first, so the next tile's
  //            hi patch streams in while the lo MMAs and the epilogue run).
  // CINP = 32 / 8: a ring of NP buffers over tiles (rows are [hi|lo]): the producer runs up to NP-1 tiles ahead.
  if (warp == 4) {
    if (tc::elect_one()) {
      tc::mbar_expect_tx(w_full, (uint32_t)C::W_BYTES);
      for (int i = 0; i < 18; ++i) tc::tma_load_2d(sW + (size_t)i * C::W_GROUP, &P.wmap, w_full, 0, i * NOUT);
      uint32_t tcount = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tcount) {
        const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
        const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
        const int y0 = ty_ * P.TH - 1, x0 = tx_ * P.TW - 1;
        if (CINP == 64) {
#pragma unroll
          for (int term = 0; term < 2; ++term) {       // load index li = 2*tcount + term: hi then lo patch of this tile
            const uint32_t li = 2 * tcount + term;
            const int s = li % NP;
            tc::mbar_wait(&p_empty[s], ((li / NP) & 1) ^ 1);
            tc::mbar_expect_tx(&p_full[s], patch_tx);
            tc::tma_load_4d(sP + (size_t)s * PB, &P.amap, &p_full[s], 64 * term, x0, y0, b);
          }
        } else {
          const int s = tcount % NP;
          tc::mbar_wait(&p_empty[s], ((tcount / NP) & 1) ^ 1);
          tc::mbar_expect_tx(&p_full[s], patch_tx);
          tc::tma_load_4d(sP + (size_t)s * PB, &P.amap, &p_full[s], 0, x0, y0, b);
        }
      }
    }
    __syncwarp();
  } else {
    constexpr int N2 = 2 * NOUT;
    constexpr uint32_t HALF = 64u * ROWB;          // bytes: rows 64-127 of the GEMM
    const int m = threadIdx.x;                     // GEMM row of this thread = patch-pitch pixel
    const int mh = m / P.PW, mw = m - mh * P.PW;
    const bool lane_ok = (mh < P.TH) && (mw < P.TW);
    float acc0[NOUT], acc1[NOUT];
    const uint32_t w_base = tc::smem_u32(sW);
    tc::mbar_wait(w_full, 0);
    uint32_t tcount = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tcount) {
      if (CINP == 64) {
        const uint32_t li_hi = 2 * tcount, li_lo = 2 * tcount + 1;
        const int s_hi = li_hi % NP, s_lo = li_lo % NP;
        const uint32_t hi_base = tc::smem_u32(sP) + (uint32_t)s_hi * PB, lo_base = tc::smem_u32(sP) + (uint32_t)s_lo * PB;
        tc::mbar_wait(&p_full[s_hi], (li_hi / NP) & 1);
        tc::wgmma_fence();
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t shift = (uint32_t)((tap / 3) * P.PW + (tap % 3)) * 128u;
          const uint64_t ahi = make_desc_sw128_at(hi_base + shift, 1024, P.desc_mode);
          const uint64_t ahi1 = make_desc_sw128_at(hi_base + shift + HALF, 1024, P.desc_mode);
          const uint64_t wboth = tc::make_desc_sw128(w_base + (uint32_t)(tap * 2) * C::W_GROUP, 1024);   // [whi ; wlo], N = 128
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // hi.whi | hi.wlo
            tc::wgmma_f16<N2>(acc0, ahi + 2 * k, wboth + 2 * k, (tap | k) ? 1u : 0u);
            tc::wgmma_f16<N2>(acc1, ahi1 + 2 * k, wboth + 2 * k, (tap | k) ? 1u : 0u);
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&p_empty[s_hi]);   // hi patch buffer may be refilled
        tc::mbar_wait(&p_full[s_lo], (li_lo / NP) & 1);
        tc::wgmma_fence();
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t shift = (uint32_t)((tap / 3) * P.PW + (tap % 3)) * 128u;
          const uint64_t alo = make_desc_sw128_at(lo_base + shift, 1024, P.desc_mode);
          const uint64_t alo1 = make_desc_sw128_at(lo_base + shift + HALF, 1024, P.desc_mode);
          const uint64_t whi = tc::make_desc_sw128(w_base + (uint32_t)(tap * 2) * C::W_GROUP, 1024);
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // lo.whi
            tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc0), alo + 2 * k, whi + 2 * k, 1u);
            tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc1), alo1 + 2 * k, whi + 2 * k, 1u);
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&p_empty[s_lo]);
      } else {
        const int s = tcount % NP;
        const uint32_t p_base = tc::smem_u32(sP) + (uint32_t)s * PB;
        tc::mbar_wait(&p_full[s], (tcount / NP) & 1);
        tc::wgmma_fence();
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t shift = (uint32_t)((tap / 3) * P.PW + (tap % 3)) * (uint32_t)ROWB;
          const uint64_t a0 = make_desc_rows_at<ROWB>(p_base + shift, P.desc_mode);
          const uint64_t a1 = make_desc_rows_at<ROWB>(p_base + shift + HALF, P.desc_mode);
          const uint64_t wboth = tc::make_desc_rows<ROWB>(w_base + (uint32_t)(tap * 2) * C::W_GROUP);
#pragma unroll
          for (int k = 0; k < KSTEPS; ++k) {   // [hi|lo] . [[whi|whi] ; [wlo|0]]  ->  cols [0,N): hi.whi + lo.whi, cols [N,2N): hi.wlo
            // 128-byte rows: K-steps 0,1 are the hi channels, 2,3 the lo channels, whose [wlo|0] rows multiply by zero -- those
            // K-steps run at N = NOUT against the [whi|whi] rows only
            const bool lo_half = (ROWB == 128) && (k >= KSTEPS / 2);
            if (lo_half) {
              tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc0), a0 + 2 * k, wboth + 2 * k, 1u);
              tc::wgmma_f16<NOUT>(tc::acc_head<NOUT>(acc1), a1 + 2 * k, wboth + 2 * k, 1u);
            } else {
              tc::wgmma_f16<N2>(acc0, a0 + 2 * k, wboth + 2 * k, (tap | k) ? 1u : 0u);
              tc::wgmma_f16<N2>(acc1, a1 + 2 * k, wboth + 2 * k, (tap | k) ? 1u : 0u);
            }
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&p_empty[s]);
      }
      // ---------------- epilogue ----------------
      const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
      const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
      const int y = ty_ * P.TH + mh, x = tx_ * P.TW + mw;
      uint32_t v[N2];
      if constexpr (NOUT == 8) {
        tc::acc_rows<16>(sStg, acc0, acc1, 0, m, 1, v);
      } else {
#pragma unroll
        for (int c = 0; c < N2 / 32; ++c) {
          uint32_t t[32];
          tc::acc_rows<32>(sStg, acc0, acc1, c * 32, m, 1, t);
#pragma unroll
          for (int j = 0; j < 32; ++j) v[c * 32 + j] = t[j];
        }
      }
      if (lane_ok && y < P.H && x < P.W) {
        const int64_t pix = ((int64_t)b * P.H + y) * P.W + x;
        float o[NOUT];
#pragma unroll
        for (int c = 0; c < NOUT; ++c) {
          float t0 = fmaf(__uint_as_float(v[c]) + __uint_as_float(v[NOUT + c]), P.inv_wscale, sBias[c]);
          if (P.relu) t0 = fmaxf(t0, 0.f);
          o[c] = t0;
        }
        if (P.out_f32) tc::store_f32_row<NOUT>(P.out_f32 + pix * P.f32_c, o, P.n_real);
        if (P.out_split) {
          __half* hp = P.out_split + pix * (2 * NOUT);
          tc::store_split_row<NOUT>(hp, hp + NOUT, o);
        }
      }
    }
  }
}

// tile geometry: TW <= 64 (PW <= 66), TH = 128 / PW; minimise MMA rows spent per valid output pixel
static void pick_halo_tile(int H, int W, int tw_max, int& TW, int& TH) {
  double best = 1e30;
  TW = 16; TH = 7;
  for (int tw = 8; tw <= tw_max; ++tw) {
    const int pw = tw + 2, th = 128 / pw;
    if (th < 1) continue;
    const double tiles = (double)cdiv(W, tw) * cdiv(H, th);
    const double cost = tiles * (128.0 + 0.15 * (th + 2) * pw);   // MMA rows + a term for the patch bytes
    if (cost < best) { best = cost; TW = tw; TH = th; }
  }
}

int g_halo_desc_mode = 0;   // the wgmma swizzle is a function of the physical shared-memory address, so a start address
                            // shifted by whole 128-byte rows needs base_offset = 0 (mode 1 gives wrong results)

// same contract as launch_conv_tc, for 3x3 stride-1 layers with (CINP,NOUT) in {(64,64), (32,32)}
int launch_conv_tc_halo(const xfeat_ctx* ctx, int layer, const __half* in_split, int B, int H, int W, __half* out_split,
                        float* out_f32, cudaStream_t st) {
  const LayerSpec& sp = kLayers[layer];
  XF_REQUIRE(sp.ks == 3 && sp.stride == 1 && ctx->d_tcw && ctx->tc_off[layer] != (size_t)-1,
             "conv_tc_halo: layer %d is not a prepared 3x3 stride-1 layer", layer);
  const bool c64 = (sp.cin == 64 && sp.cout == 64), c32 = (sp.cin == 24 && sp.cout == 24), c8 = (sp.cin == 8 && sp.cout == 8);
  XF_REQUIRE(c64 || c32 || c8, "conv_tc_halo: unsupported channel configuration");
  const int cinp = c64 ? 64 : (c32 ? 32 : 8), nout = cinp;
  const int rowh = c8 ? 16 : 64;                       // halves per operand row
  const CUtensorMapSwizzle swz = c8 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_128B;
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  HaloParams P;
  pick_halo_tile(H, W, c64 ? 40 : 64, P.TW, P.TH);
  P.PW = P.TW + 2;
  const cuuint64_t row_bytes = (cuuint64_t)2 * cinp * sizeof(__half);
  const cuuint64_t dims[4] = {(cuuint64_t)2 * cinp, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {row_bytes, (cuuint64_t)W * row_bytes, (cuuint64_t)H * W * row_bytes};
  const cuuint32_t box[4] = {(cuuint32_t)rowh, (cuuint32_t)P.PW, (cuuint32_t)(P.TH + 2), 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(&P.amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)in_split, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(halo activations) failed: %d", (int)r);
    return XF_E_CUDA;
  }
  const cuuint64_t wdims[2] = {(cuuint64_t)rowh, (cuuint64_t)18 * nout};
  const cuuint64_t wstrides[1] = {(cuuint64_t)rowh * 2};
  const cuuint32_t wbox[2] = {(cuuint32_t)rowh, (cuuint32_t)nout};
  const cuuint32_t westr[2] = {1, 1};
  r = enc(&P.wmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)((__half*)ctx->d_tcw + ctx->tc_off[layer]), wdims, wstrides, wbox,
          westr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(halo weights) failed: %d", (int)r);
    return XF_E_CUDA;
  }
  P.bias = ctx->d_weights + ctx->table.b_off[layer];
  P.inv_wscale = ctx->tc_inv_wscale[layer];
  P.B = B; P.H = H; P.W = W;
  P.out_split = out_split;
  P.out_f32 = out_f32;
  P.f32_c = sp.cout;
  P.n_real = sp.cout;
  P.relu = sp.relu;
  P.desc_mode = g_halo_desc_mode;
  const int n_tiles = cdiv(H, P.TH) * cdiv(W, P.TW) * B;
  XF_REQUIRE(n_tiles < (1 << 22), "conv_tc_halo: too many tiles (%d)", n_tiles);
  P.div_img = make_fastdiv((unsigned)(cdiv(H, P.TH) * cdiv(W, P.TW)));
  P.div_x = make_fastdiv((unsigned)cdiv(W, P.TW));
  const int grid = n_tiles < ctx->sm_count ? n_tiles : ctx->sm_count;
  if (c64) {
    XF_DYN_SMEM((conv_tc_halo_kernel<64, 64>), (HaloCfg<64, 64>::SMEM));
    conv_tc_halo_kernel<64, 64><<<grid, CH_THREADS, HaloCfg<64, 64>::SMEM, st>>>(P);
  } else if (c32) {
    XF_DYN_SMEM((conv_tc_halo_kernel<32, 32>), (HaloCfg<32, 32>::SMEM));
    conv_tc_halo_kernel<32, 32><<<grid, CH_THREADS, HaloCfg<32, 32>::SMEM, st>>>(P);
  } else {
    XF_DYN_SMEM((conv_tc_halo_kernel<8, 8>), (HaloCfg<8, 8>::SMEM));
    conv_tc_halo_kernel<8, 8><<<grid, CH_THREADS, HaloCfg<8, 8>::SMEM, st>>>(P);
  }
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf

extern "C" void xfeat_set_halo_desc_mode(int mode) { xf::g_halo_desc_mode = mode; }
