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
  CUtensorMap smap;   // split output (B,H,W,2*NOUT); box {32, TW, TH, 1} (NOUT = 8: {16, TW, TH, 1})
  CUtensorMap fmap;   // fp32 output (B,H,W,cout); box {16, TW, TH, 1} (NOUT = 8: {8, TW, TH, 1})
  int has_split, has_f32;
  int n_real;
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
  unsigned char* sStg = base + C::W_BYTES + NP * PB;
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
    if (P.has_split) tc::tma_prefetch_desc(&P.smap);
    if (P.has_f32) tc::tma_prefetch_desc(&P.fmap);
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
    float acc0[NOUT], acc1[NOUT];
    int srow[4];   // GEMM row m = h * PW + w -> staging row h * TW + w; rows with w >= TW or h >= TH are junk
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = tc::frag_row(threadIdx.x, i), mh = m / P.PW, mw = m - mh * P.PW;
      srow[i] = (mh < P.TH && mw < P.TW) ? mh * P.TW + mw : -1;
    }
    tc::ConvEpi E;
    E.split = P.has_split ? &P.smap : nullptr;
    E.f32 = P.has_f32 ? &P.fmap : nullptr;
    E.split_c = NOUT;
    E.co = 0;
    E.inv_wscale = P.inv_wscale;
    E.relu = P.relu;
    E.bias = sBias;
    E.skip_w = nullptr;
    E.skip_v = nullptr;
    uint32_t piece = 0;
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
        tc::wgmma_commit();   // the hi group stays in flight while the lo patch is awaited and the lo MMAs are queued
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
        tc::wgmma_wait<1>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&p_empty[s_hi]);   // hi group retired: the hi patch buffer may be refilled
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
        // unrolled: the scale-d flags become constants.  Left as a loop, ptxas (C7520) serialises every wgmma of this path
        // behind a warpgroup.arrive + wait of its own.
#pragma unroll
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
      E.x0 = tx_ * P.TW;
      E.y0 = ty_ * P.TH;
      E.b = b;
      tc::conv_epilogue<NOUT>(acc0, acc1, sStg, piece, srow, E);
    }
    if (threadIdx.x == 0) tc::bulk_wait_all();
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
  P.has_split = out_split != nullptr;
  P.has_f32 = out_f32 != nullptr;
  P.n_real = sp.cout;
  P.relu = sp.relu;
  P.desc_mode = g_halo_desc_mode;
  const int rc = encode_conv_out_maps(enc, &P.smap, out_split, nout, &P.fmap, out_f32, sp.cout, c8, B, H, W, P.TW, P.TH);
  if (rc) return rc;
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

// ---------------------------------------------------------------------------------------------------------------------
// The stem tail: block1.2 (8 -> 8, 3x3, half resolution) and block1.3 (8 -> 24, 3x3, stride 2) + skip1 in one kernel, with
// block1.2's output a3 kept in shared memory.  Split in two, the layers move a3 through HBM twice (written once, gathered
// by nine strided boxes); here a tile reads one a2 patch and writes its x1s block, and nothing else leaves the SM.
//
// A tile is a THq x TWq block of block1.3 outputs (quarter resolution).  Its block1.3 GEMM rows are m = ly * PQ + lx
// (PQ = TWq + 1; lx == TWq is a junk lane), and output (ly, lx) reads a3 at region position (u, v) = (2ly + dy, 2lx + dx),
// where region (0, 0) is a3 pixel (2 Y0 - 1, 2 X0 - 1).
//  * block1.2 computes the (2THq+1) x (2TWq+1) region as conv_tc_halo_kernel<8,8> does -- rows n = u * PW + v of the a2
//    patch (2THq+3) x (2TWq+3), pitch PW = 2TWq + 3, tap (dy,dx) = the descriptor shifted by dy * PW + dx rows -- in chunks
//    of 128 rows.  Its epilogue writes a3 into four POLYPHASE planes, plane (u & 1, v & 1) row (u >> 1) * PQ + (v >> 1), in
//    the SWIZZLE_32B row layout the TMA would have written.
//  * block1.3's tap (dy,dx) is then plane (dy & 1, dx & 1) shifted by (dy >> 1) * PQ + (dx >> 1) rows: again a constant
//    descriptor shift, and a valid row m reads plane positions (ly + (dy >> 1), lx + (dx >> 1)), all inside the region.
// Both layers issue per pixel exactly the wgmma sequence of their per-layer kernels, and a3 is rounded by the same epilogue
// arithmetic (tc::conv_values), so x1s is bit-identical to conv_tc_halo_kernel<8,8> followed by conv_tc_kernel<3,8,32>.
// Region positions outside the half-resolution image are exact zeros (the per-layer path's TMA zero fill), not relu(bias).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int ST_TWQ = 15, ST_THQ = 8;                    // 120 of 128 block1.3 rows; one tile reads a 19 x 33 a2 patch
constexpr int ST_PQ = ST_TWQ + 1;
constexpr int ST_RW = 2 * ST_TWQ + 1, ST_RH = 2 * ST_THQ + 1;   // a3 region
constexpr int ST_PW = ST_RW + 2, ST_PH = ST_RH + 2;             // a2 patch
constexpr int ST_CHUNKS = (ST_RH * ST_PW + 127) / 128;          // block1.2 GEMM chunks of 128 rows
// the last chunk's taps read 2 * PW + 2 rows past it; a plane is read up to row 127 + PQ + 1
constexpr int ST_PATCH_BYTES = ((ST_CHUNKS * 128 + 2 * ST_PW + 2) * 32 + 1023) / 1024 * 1024;
constexpr int ST_PLANE_BYTES = ((128 + ST_PQ + 1) * 32 + 255) / 256 * 256;
constexpr int ST_NP = 2;                                        // patch ring; two CTAs per SM
constexpr int ST_W12_GROUP = 8 * 32, ST_W13_GROUP = 32 * 32;    // bytes: [whi|whi] or [wlo|0] rows of one tap
constexpr int ST_W12_BYTES = 18 * ST_W12_GROUP, ST_W13_BYTES = 18 * ST_W13_GROUP;
constexpr size_t ST_SMEM = 1024 + (size_t)ST_NP * ST_PATCH_BYTES + ST_W13_BYTES + tc::STG_BYTES + ST_W12_BYTES +
                           4 * ST_PLANE_BYTES + 1024;
static_assert(ST_THQ * ST_PQ <= 128, "stem tail: block1.3 tile exceeds 128 GEMM rows");

struct StemTailParams {
  CUtensorMap amap;     // a2 split (B,H2,W2,16) halves [hi(8)|lo(8)]; box {16, PW, PH, 1}
  CUtensorMap w12map;   // block1.2 weights: rows [tap][group][8] x 16 halves
  CUtensorMap w13map;   // block1.3 weights: rows [tap][group][32] x 16 halves
  CUtensorMap smap;     // x1s split (B,H4,W4,64) [hi(32)|lo(32)]; box {32, TWq, THq, 1}
  const float* bias12;
  const float* bias13;
  const float* skip_w;  // 24 weights then 24 biases
  const float* xn;      // normalised gray image (B, 4*H4, 4*W4)
  float inv_wscale12, inv_wscale13;
  int B, H2, W2, H4, W4;
  FastDiv div_img, div_x;
};

__global__ void __launch_bounds__(CH_THREADS, 2) stem_tail_halo_kernel(const __grid_constant__ StemTailParams P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sP = base;                                  // patch ring
  unsigned char* sW13 = sP + ST_NP * ST_PATCH_BYTES;
  unsigned char* sStg = sW13 + ST_W13_BYTES;
  unsigned char* sW12 = sStg + tc::STG_BYTES;
  unsigned char* sPl = sW12 + ST_W12_BYTES;                  // four a3 planes, 256-byte aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(sPl + 4 * ST_PLANE_BYTES);
  uint64_t* w_full = bars;
  uint64_t* p_full = bars + 1;            // [NP]
  uint64_t* p_empty = bars + 1 + ST_NP;   // [NP]
  float* sBias12 = reinterpret_cast<float*>(bars + 1 + 2 * ST_NP);
  float* sBias13 = sBias12 + 8;
  float* sSkip = sBias13 + 32;            // [2][32]: skip weights, skip biases (channels 24-31 zero)
  float* sSkipv = sSkip + 64;             // [128]: pooled skip input per staging row

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_x = (P.W4 + ST_TWQ - 1) / ST_TWQ, tiles_y = (P.H4 + ST_THQ - 1) / ST_THQ;
  const int tiles_img = tiles_x * tiles_y;
  const int n_tiles = tiles_img * P.B;

  if (threadIdx.x < 8) sBias12[threadIdx.x] = __ldg(P.bias12 + threadIdx.x);
  if (threadIdx.x < 32) sBias13[threadIdx.x] = threadIdx.x < 24 ? __ldg(P.bias13 + threadIdx.x) : 0.f;
  if (threadIdx.x < 64) {
    const int c = threadIdx.x % 32, wb = threadIdx.x / 32;
    sSkip[threadIdx.x] = c < 24 ? __ldg(P.skip_w + wb * 24 + c) : 0.f;
  }
  if (warp == 4 && lane == 0) {
    tc::tma_prefetch_desc(&P.amap);
    tc::tma_prefetch_desc(&P.w12map);
    tc::tma_prefetch_desc(&P.w13map);
    tc::tma_prefetch_desc(&P.smap);
    tc::mbar_init(w_full, 1);
    for (int i = 0; i < ST_NP; ++i) {
      tc::mbar_init(&p_full[i], 1);
      tc::mbar_init(&p_empty[i], 4);   // one arrival per consumer warp
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      tc::mbar_expect_tx(w_full, (uint32_t)(ST_W12_BYTES + ST_W13_BYTES));
      for (int i = 0; i < 18; ++i) tc::tma_load_2d(sW12 + i * ST_W12_GROUP, &P.w12map, w_full, 0, i * 8);
      for (int i = 0; i < 18; ++i) tc::tma_load_2d(sW13 + i * ST_W13_GROUP, &P.w13map, w_full, 0, i * 32);
      uint32_t tcount = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tcount) {
        const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
        const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
        const int s = tcount % ST_NP;
        tc::mbar_wait(&p_empty[s], ((tcount / ST_NP) & 1) ^ 1);
        tc::mbar_expect_tx(&p_full[s], (uint32_t)(ST_PW * ST_PH * 32));
        tc::tma_load_4d(sP + (size_t)s * ST_PATCH_BYTES, &P.amap, &p_full[s], 0, 2 * ST_TWQ * tx_ - 2, 2 * ST_THQ * ty_ - 2, b);
      }
    }
    __syncwarp();
  } else {
    constexpr uint32_t HALF = 64 * 32;   // bytes: rows 64-127 of the GEMM
    const int q = threadIdx.x & 3;
    int srow[4];   // block1.3 GEMM row m = ly * PQ + lx -> staging row ly * TWq + lx, or -1 for a junk row
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = tc::frag_row(threadIdx.x, i), ly = m / ST_PQ, lx = m - ly * ST_PQ;
      srow[i] = (ly < ST_THQ && lx < ST_TWQ) ? ly * ST_TWQ + lx : -1;
    }
    tc::ConvEpi E12;   // block1.2: values only, into the planes
    E12.split = nullptr;
    E12.f32 = nullptr;
    E12.inv_wscale = P.inv_wscale12;
    E12.relu = 1;
    E12.bias = sBias12;
    E12.skip_w = nullptr;
    E12.skip_v = nullptr;
    tc::ConvEpi E13;
    E13.split = &P.smap;
    E13.f32 = nullptr;
    E13.split_c = 32;
    E13.co = 0;
    E13.inv_wscale = P.inv_wscale13;
    E13.relu = 1;
    E13.bias = sBias13;
    E13.skip_w = sSkip;
    E13.skip_v = sSkipv;
    const float no_skip[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t piece = 0;
    const uint32_t w12 = tc::smem_u32(sW12), w13 = tc::smem_u32(sW13), planes = tc::smem_u32(sPl);
    tc::mbar_wait(w_full, 0);
    uint32_t tcount = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tcount) {
      const int b = (int)fdiv((unsigned)tile, P.div_img), rem = tile - b * tiles_img;
      const int ty_ = (int)fdiv((unsigned)rem, P.div_x), tx_ = rem - ty_ * tiles_x;
      const int Y0 = ty_ * ST_THQ, X0 = tx_ * ST_TWQ;
      const int gy0 = 2 * Y0 - 1, gx0 = 2 * X0 - 1;   // a3 pixel of region position (0, 0)
      // block1.2's epilogue for chunk ch: region rows only; out-of-image positions are zeros in both halves
      auto to_planes = [&](int ch, const float (&d0)[8], const float (&d1)[8]) {
        float o[4][1][2];
        uint32_t hi[4][1], lo[4][1];
        tc::conv_values<8>(d0, d1, 0, no_skip, E12, o, hi, lo);
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int n = ch * 128 + tc::frag_row(threadIdx.x, h), u = n / ST_PW, v = n - u * ST_PW;
          if (u < ST_RH && v < ST_RW) {
            const int gy = gy0 + u, gx = gx0 + v;
            const bool inside = gy >= 0 && gy < P.H2 && gx >= 0 && gx < P.W2;
            unsigned char* pl = sPl + ((u & 1) * 2 + (v & 1)) * ST_PLANE_BYTES;
            const int row = (u >> 1) * ST_PQ + (v >> 1);
            *reinterpret_cast<uint32_t*>(pl + tc::piece_off<32>(row, 4 * q)) = inside ? hi[h][0] : 0u;
            *reinterpret_cast<uint32_t*>(pl + tc::piece_off<32>(row, 16 + 4 * q)) = inside ? lo[h][0] : 0u;
          }
        }
      };

      // ---------------- block1.2: chunk ch's MMAs run while chunk ch-1's epilogue writes the planes ----------------
      const int s = tcount % ST_NP;
      const uint32_t p_base = tc::smem_u32(sP) + (uint32_t)s * ST_PATCH_BYTES;
      tc::mbar_wait(&p_full[s], (tcount / ST_NP) & 1);
      float c0[2][8], c1[2][8];
#pragma unroll
      for (int ch = 0; ch < ST_CHUNKS; ++ch) {
        tc::wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t a = p_base + (uint32_t)(ch * 128 + (tap / 3) * ST_PW + (tap % 3)) * 32u;
          const uint64_t w = tc::make_desc_sw32(w12 + (uint32_t)(tap * 2) * ST_W12_GROUP, 256);   // [whi|whi] ; [wlo|0], N = 16
          tc::wgmma_f16<16>(c0[ch & 1], tc::make_desc_sw32(a, 256), w, tap ? 1u : 0u);
          tc::wgmma_f16<16>(c1[ch & 1], tc::make_desc_sw32(a + HALF, 256), w, tap ? 1u : 0u);
        }
        tc::wgmma_commit();
        if (ch > 0) {
          tc::wgmma_wait<1>();
          tc::acc_fence(c0[(ch - 1) & 1]);
          tc::acc_fence(c1[(ch - 1) & 1]);
          to_planes(ch - 1, c0[(ch - 1) & 1], c1[(ch - 1) & 1]);
        }
      }
      tc::wgmma_wait<0>();
      tc::acc_fence(c0[(ST_CHUNKS - 1) & 1]);
      tc::acc_fence(c1[(ST_CHUNKS - 1) & 1]);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&p_empty[s]);   // the patch may be refilled
      to_planes(ST_CHUNKS - 1, c0[(ST_CHUNKS - 1) & 1], c1[(ST_CHUNKS - 1) & 1]);
      tc::fence_proxy_async();   // the planes' generic-proxy writes, before the wgmmas (async proxy) read them
      tc::wg_sync(2);

      // ---------------- block1.3 + skip1 ----------------
      float acc0[32], acc1[32];
      tc::wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int dy = tap / 3, dx = tap % 3;
        const uint32_t a = planes + (uint32_t)((dy & 1) * 2 + (dx & 1)) * ST_PLANE_BYTES + (uint32_t)((dy >> 1) * ST_PQ + (dx >> 1)) * 32u;
        const uint64_t w = tc::make_desc_sw32(w13 + (uint32_t)(tap * 2) * ST_W13_GROUP, 256);   // groups [0 ; 1], N = 64
        tc::wgmma_f16<64>(acc0, tc::make_desc_sw32(a, 256), w, tap ? 1u : 0u);
        tc::wgmma_f16<64>(acc1, tc::make_desc_sw32(a + HALF, 256), w, tap ? 1u : 0u);
      }
      tc::wgmma_commit();
      // AvgPool2d(4,4) of the gray image under the MMAs, one tile pixel per thread, summed as conv_tc_kernel sums it
      if (threadIdx.x < ST_THQ * ST_TWQ) {
        const int ly = threadIdx.x / ST_TWQ, y = Y0 + ly, x = X0 + threadIdx.x - ly * ST_TWQ;
        float skipv = 0.f;
        if (y < P.H4 && x < P.W4) {
          const int W0 = P.W4 * 4;
          const float* xp = P.xn + ((int64_t)b * P.H4 * 4 + y * 4) * W0 + x * 4;
          float sacc = 0.f;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(xp + (int64_t)rr * W0));
            sacc += t.x; sacc += t.y; sacc += t.z; sacc += t.w;
          }
          skipv = sacc * (1.0f / 16.0f);
        }
        sSkipv[threadIdx.x] = skipv;
      }
      tc::wgmma_wait<0>();
      tc::acc_fence(acc0);
      tc::acc_fence(acc1);
      tc::wg_sync(1);
      E13.x0 = X0;
      E13.y0 = Y0;
      E13.b = b;
      tc::conv_epilogue<32>(acc0, acc1, sStg, piece, srow, E13);
    }
    if (threadIdx.x == 0) tc::bulk_wait_all();
  }
}

// a2 (B,H2,W2,16) split fp16 [hi(8)|lo(8)] (block1.1's output) -> x1s (B,H2/2,W2/2,64) split fp16 [hi(32)|lo(32)], channels
// 24-31 zero: block1.2, block1.3 and skip1 (xn: the normalised gray image (B,2*H2,2*W2))
int launch_stem_tail_halo(const xfeat_ctx* ctx, const __half* a2_split, const float* xn, int B, int H2, int W2, __half* out_split,
                          cudaStream_t st) {
  XF_REQUIRE(ctx->d_tcw && ctx->tc_off[L_B1_2] != (size_t)-1 && ctx->tc_off[L_B1_3] != (size_t)-1,
             "stem_tail: block1.2 / block1.3 are not prepared for the tensor cores");
  XF_REQUIRE(a2_split && xn && out_split && B > 0 && H2 >= 2 && W2 >= 2 && H2 % 2 == 0 && W2 % 2 == 0,
             "stem_tail: bad arguments B=%d H2=%d W2=%d", B, H2, W2);
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  StemTailParams P;
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const cuuint64_t dims[4] = {16, (cuuint64_t)W2, (cuuint64_t)H2, (cuuint64_t)B};
  const cuuint64_t strides[3] = {32, (cuuint64_t)W2 * 32, (cuuint64_t)H2 * W2 * 32};
  const cuuint32_t box[4] = {16, (cuuint32_t)ST_PW, (cuuint32_t)ST_PH, 1};
  CUresult r = enc(&P.amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)a2_split, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(stem tail a2) failed: %d", (int)r);
    return XF_E_CUDA;
  }
  const struct { CUtensorMap* map; int layer, nout; } wm[2] = {{&P.w12map, L_B1_2, 8}, {&P.w13map, L_B1_3, 32}};
  for (const auto& m : wm) {
    const cuuint64_t wdims[2] = {16, (cuuint64_t)18 * m.nout};
    const cuuint64_t wstrides[1] = {32};
    const cuuint32_t wbox[2] = {16, (cuuint32_t)m.nout};
    r = enc(m.map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)((__half*)ctx->d_tcw + ctx->tc_off[m.layer]), wdims, wstrides, wbox, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(stem tail weights, layer %d) failed: %d", m.layer, (int)r);
      return XF_E_CUDA;
    }
  }
  P.B = B; P.H2 = H2; P.W2 = W2; P.H4 = H2 / 2; P.W4 = W2 / 2;
  const int rc = encode_conv_out_maps(enc, &P.smap, out_split, 32, nullptr, nullptr, 24, false, B, P.H4, P.W4, ST_TWQ, ST_THQ);
  if (rc) return rc;
  P.bias12 = ctx->d_weights + ctx->table.b_off[L_B1_2];
  P.bias13 = ctx->d_weights + ctx->table.b_off[L_B1_3];
  P.skip_w = ctx->d_weights + ctx->table.w_off[L_SKIP1];   // 24 weights; the 24 biases follow (layers.h packing)
  P.xn = xn;
  P.inv_wscale12 = ctx->tc_inv_wscale[L_B1_2];
  P.inv_wscale13 = ctx->tc_inv_wscale[L_B1_3];
  const int tiles_img = cdiv(P.H4, ST_THQ) * cdiv(P.W4, ST_TWQ);
  XF_REQUIRE((int64_t)tiles_img * B < (1 << 22), "stem_tail: too many tiles (%lld)", (long long)tiles_img * B);
  const int n_tiles = tiles_img * B;
  P.div_img = make_fastdiv((unsigned)tiles_img);
  P.div_x = make_fastdiv((unsigned)cdiv(P.W4, ST_TWQ));
  const int grid = n_tiles < 2 * ctx->sm_count ? n_tiles : 2 * ctx->sm_count;
  XF_DYN_SMEM(stem_tail_halo_kernel, ST_SMEM);
  stem_tail_halo_kernel<<<grid, CH_THREADS, ST_SMEM, st>>>(P);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf

extern "C" void xfeat_set_halo_desc_mode(int mode) { xf::g_halo_desc_mode = mode; }

// Test hook: block1.1's fp32 output (B,H2,W2,8) is split as xfeat_debug_conv_layer_tc_ex splits it, then the stem tail runs.
extern "C" int xfeat_debug_stem_tail(xfeat_ctx* ctx, const float* d_in, const float* d_xn, int B, int H2, int W2, void* d_out_split,
                                     void* d_scratch, size_t scratch_bytes, void* stream) {
  XF_REQUIRE(ctx && d_in && d_xn && d_out_split && d_scratch && B > 0 && H2 > 0 && W2 > 0, "debug_stem_tail: bad arguments");
  const int64_t npix = (int64_t)B * H2 * W2;
  XF_REQUIRE(scratch_bytes >= (size_t)npix * 32, "debug_stem_tail: scratch must hold B*H2*W2*32 bytes");
  XF_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = xf::launch_split_nhwc(d_in, (__half*)d_scratch, npix, 8, 8, st);
  if (rc) return rc;
  return xf::launch_stem_tail_halo(ctx, (const __half*)d_scratch, d_xn, B, H2, W2, (__half*)d_out_split, st);
}
