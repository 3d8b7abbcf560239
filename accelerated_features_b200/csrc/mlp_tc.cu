// fine_matcher MLP (model.py:97-111: 128 -> 512 -> 512 -> 512 -> 512 -> 64, BatchNorm1d folded, ReLU) on the tensor cores.
//
// Each layer is one launch of a persistent split-fp16 GEMM  Y[rows x N] = X[rows x K] . W[N x K]^T  over ALL coarse matches of
// the batch at once (rows = sum of the per-pair match counts, read from device memory: tiles past the live rows are never
// scheduled).  Operands are split as everywhere in this library: x = hi + lo (fp16), w * 2^k = whi + wlo,
//      y = (hi.whi + hi.wlo + lo.whi) * 2^-k + b          (fp32 accumulation in registers)
// so the result is fp32-equivalent (tests: 6e-4 absolute on the logits, at most 1/5 of the error with any one term dropped, and
// 5e-4 px on the sub-pixel offsets; tests/split_ref.py).  Activations travel between
// the layers already split, rows of [hi(K) | lo(K)] halves, written by the producing epilogue.
//   warp 4: TMA producer, one 64-channel K block per stage {A hi, A lo, W hi, W lo};  warps 0-3: one warpgroup that issues, per
//   K block and 64-row slab, 4 x wgmma(64 x 2NT x 16) hi.[whi ; wlo] + 4 x wgmma(64 x NT x 16) lo.whi, then runs the epilogue
//   (bias, ReLU, split, one row per thread).  NT = 64: the 2 x 128 accumulator columns of both slabs fill 128 registers per
//   thread.  Weights (1 MB per 512 x 512 layer) stream from L2; an n-fastest tile order keeps the A tile of a row block
//   L2-resident across its N tiles.
// Replaces the five fp32 CUDA-core launches of round 1 (refine.cu); the fp32 path stays as xfeat_set_conv_impl(0).
#include <cuda_fp16.h>

#include <vector>

#include "common.cuh"
#include "tc_common.cuh"

namespace xf {

constexpr int ML_THREADS = 160, ML_BOX = 128 * 128;   // 128 rows x 64 halves

template <int NT>
struct MlpCfg {
  static constexpr int W_BOX = NT * 128;                         // NT rows x 64 halves
  static constexpr int STAGE = 2 * ML_BOX + 2 * W_BOX;           // A hi, A lo, W hi, W lo
  static constexpr int NS = 4;
  static constexpr size_t SMEM = 1024 + (size_t)NS * STAGE + tc::STG_BYTES + 256;
};

struct MlpParams {
  CUtensorMap amap;     // X split: (rows_cap, 2K) halves, box {64, 128}
  CUtensorMap wmap;     // W split: (N_pad, 2K) halves, box {64, NT}
  const float* bias;    // N
  float inv_scale;
  int K, N, n_tiles;    // n_tiles = N_pad / NT
  const int* n_live;    // device: live rows (null: rows_cap)
  int rows_cap;
  int relu;
  __half* out_split;    // (rows_cap, 2N) halves [hi(N) | lo(N)] or null
  float* out_f32;       // (rows_cap, N) or null
};

template <int NT>
__global__ void __launch_bounds__(ML_THREADS, 1) mlp_gemm_kernel(const __grid_constant__ MlpParams P) {
  using C = MlpCfg<NT>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sS = base;
  float* sStg = reinterpret_cast<float*>(base + (size_t)C::NS * C::STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + (size_t)C::NS * C::STAGE + tc::STG_BYTES);
  uint64_t* s_full = bars;                 // [NS]
  uint64_t* s_empty = bars + C::NS;        // [NS]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = P.n_live ? min(__ldg(P.n_live), P.rows_cap) : P.rows_cap;
  const int m_tiles = (rows + 127) / 128;
  const int total = m_tiles * P.n_tiles;
  const int KB = P.K / 64;

  if (warp == 4 && lane == 0) {
    tc::tma_prefetch_desc(&P.amap);
    tc::tma_prefetch_desc(&P.wmap);
    for (int i = 0; i < C::NS; ++i) {
      tc::mbar_init(&s_full[i], 1);
      tc::mbar_init(&s_empty[i], 4);   // one arrival per consumer warp
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int m = tile / P.n_tiles, nt = tile - m * P.n_tiles;
        for (int kb = 0; kb < KB; ++kb, ++it) {
          const int s = it % C::NS;
          tc::mbar_wait(&s_empty[s], ((it / C::NS) & 1) ^ 1);
          tc::mbar_expect_tx(&s_full[s], C::STAGE);
          unsigned char* dst = sS + (size_t)s * C::STAGE;
          tc::tma_load_2d(dst, &P.amap, &s_full[s], kb * 64, m * 128);                          // A hi
          tc::tma_load_2d(dst + ML_BOX, &P.amap, &s_full[s], P.K + kb * 64, m * 128);           // A lo
          tc::tma_load_2d(dst + 2 * ML_BOX, &P.wmap, &s_full[s], kb * 64, nt * NT);             // W hi
          tc::tma_load_2d(dst + 2 * ML_BOX + C::W_BOX, &P.wmap, &s_full[s], P.K + kb * 64, nt * NT);   // W lo
        }
      }
    }
    __syncwarp();
  } else {
    constexpr uint32_t HALF = (64 * 128) >> 4;   // descriptor offset of rows 64-127
    const int r = threadIdx.x;
    float acc0[NT], acc1[NT];                     // rows 0-63 / 64-127, 2*NT columns each
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const int m = tile / P.n_tiles, nt = tile - m * P.n_tiles;
      for (int kb = 0; kb < KB; ++kb, ++it) {
        const int s = it % C::NS;
        tc::mbar_wait(&s_full[s], (it / C::NS) & 1);
        tc::wgmma_fence();
        const uint32_t sa = tc::smem_u32(sS + (size_t)s * C::STAGE);
        const uint64_t ahi = tc::make_desc_sw128(sa, 1024), alo = tc::make_desc_sw128(sa + ML_BOX, 1024);
        const uint64_t w = tc::make_desc_sw128(sa + 2 * ML_BOX, 1024);     // [whi ; wlo]: 2 NT rows, or whi alone: NT rows
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // hi.whi | hi.wlo
          tc::wgmma_f16<2 * NT>(acc0, ahi + 2 * k, w + 2 * k, (kb | k) ? 1u : 0u);
          tc::wgmma_f16<2 * NT>(acc1, ahi + HALF + 2 * k, w + 2 * k, (kb | k) ? 1u : 0u);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // lo.whi
          tc::wgmma_f16<NT>(tc::acc_head<NT>(acc0), alo + 2 * k, w + 2 * k, 1u);
          tc::wgmma_f16<NT>(tc::acc_head<NT>(acc1), alo + HALF + 2 * k, w + 2 * k, 1u);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc0);
        tc::acc_fence(acc1);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&s_empty[s]);
      }
      const int row = m * 128 + r;
      const bool live = row < rows;
#pragma unroll
      for (int c0 = 0; c0 < NT; c0 += 32) {
        uint32_t v0[32], v1[32];
        tc::acc_rows<32>(sStg, acc0, acc1, c0, r, 1, v0);
        tc::acc_rows<32>(sStg, acc0, acc1, NT + c0, r, 1, v1);
        const int n0 = nt * NT + c0;
        if (live && n0 < P.N) {
          float o[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            float t = fmaf(__uint_as_float(v0[j]) + __uint_as_float(v1[j]), P.inv_scale, __ldg(P.bias + n0 + j));
            if (P.relu) t = fmaxf(t, 0.f);
            o[j] = t;
          }
          if (P.out_f32) tc::store_f32_row<32>(P.out_f32 + (int64_t)row * P.N + n0, o, 32);
          if (P.out_split) {
            __half* hp = P.out_split + (int64_t)row * (2 * P.N) + n0;
            tc::store_split_row<32>(hp, hp + P.N, o);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
static const int kMlpLayers[5] = {L_FM_0, L_FM_1, L_FM_2, L_FM_3, L_FM_4};

// split weights of the five Linear layers: rows [N_pad][2K] halves = [whi(K) | wlo(K)], scaled by 2^k (max |w| 2^k in [2^12, 2^13))
int mlp_tc_prepare(xfeat_ctx* ctx) {
  size_t total = 0;
  for (int i = 0; i < 5; ++i) {
    const LayerSpec& sp = kLayers[kMlpLayers[i]];
    const int npad = (sp.cout + 63) / 64 * 64;
    ctx->mlp_off[i] = total;
    total += (size_t)npad * 2 * sp.cin;
  }
  std::vector<__half> h(total, __float2half_rn(0.f));
  for (int i = 0; i < 5; ++i) {
    const int l = kMlpLayers[i];
    const LayerSpec& sp = kLayers[l];
    const float* w = ctx->h_weights + ctx->table.w_off[l];     // [cin][cout], cout fastest (layers.h)
    float mx = 0.f;
    for (int j = 0; j < sp.cin * sp.cout; ++j) mx = fmaxf(mx, fabsf(w[j]));
    int e = 0;
    if (mx > 0.f) frexpf(mx, &e);
    const float s = (mx > 0.f) ? ldexpf(1.f, 13 - e) : 1.f;
    ctx->mlp_inv_scale[i] = (mx > 0.f) ? ldexpf(1.f, e - 13) : 1.f;
    __half* dst = h.data() + ctx->mlp_off[i];
    for (int n = 0; n < sp.cout; ++n)
      for (int k = 0; k < sp.cin; ++k) {
        const float v = w[(size_t)k * sp.cout + n] * s;
        const __half hi = __float2half_rn(v);
        dst[(size_t)n * 2 * sp.cin + k] = hi;
        dst[(size_t)n * 2 * sp.cin + sp.cin + k] = __float2half_rn(v - __half2float(hi));
      }
  }
  XF_CUDA(cudaMalloc(&ctx->d_mlpw, total * sizeof(__half)));
  XF_CUDA(cudaMemcpy(ctx->d_mlpw, h.data(), total * sizeof(__half), cudaMemcpyHostToDevice));
  return XF_OK;
}

static int mlp_map(CUtensorMap* m, const void* ptr, uint64_t row_halves, uint64_t rows, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return XF_E_CUDA;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)row_halves, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)row_halves * sizeof(__half)};
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(mlp) failed: %d", (int)r);
    return XF_E_CUDA;
  }
  return XF_OK;
}

// One layer: x_split (rows_cap, 2K) -> out_split (rows_cap, 2N) or out_f32 (rows_cap, N)
static int launch_mlp_layer(const xfeat_ctx* ctx, int i, const __half* x_split, int rows_cap, const int* n_live, __half* out_split,
                            float* out_f32, cudaStream_t st) {
  const LayerSpec& sp = kLayers[kMlpLayers[i]];
  constexpr int NT = 64;
  const int npad = (sp.cout + 63) / 64 * 64;
  MlpParams P;
  int rc;
  if ((rc = mlp_map(&P.amap, x_split, (uint64_t)2 * sp.cin, (uint64_t)rows_cap, 128))) return rc;
  if ((rc = mlp_map(&P.wmap, (const __half*)ctx->d_mlpw + ctx->mlp_off[i], (uint64_t)2 * sp.cin, (uint64_t)npad, (uint32_t)NT))) return rc;
  P.bias = ctx->d_weights + ctx->table.b_off[kMlpLayers[i]];
  P.inv_scale = ctx->mlp_inv_scale[i];
  P.K = sp.cin; P.N = sp.cout; P.n_tiles = npad / NT;
  P.n_live = n_live; P.rows_cap = rows_cap;
  P.relu = sp.relu;
  P.out_split = out_split; P.out_f32 = out_f32;
  const int max_tiles = cdiv(rows_cap, 128) * P.n_tiles;
  const int grid = max_tiles < ctx->sm_count ? max_tiles : ctx->sm_count;
  XF_DYN_SMEM(mlp_gemm_kernel<NT>, MlpCfg<NT>::SMEM);
  mlp_gemm_kernel<NT><<<grid, ML_THREADS, MlpCfg<NT>::SMEM, st>>>(P);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// X_split: (rows_cap, 256) halves [hi(128) | lo(128)]; act_a / act_b: (rows_cap, 1024) halves each; logits (rows_cap, 64) fp32
int launch_fine_mlp_tc(const xfeat_ctx* ctx, const __half* X_split, int rows_cap, const int* n_live, __half* act_a, __half* act_b,
                       float* logits, cudaStream_t st) {
  XF_REQUIRE(ctx->d_mlpw, "fine_mlp_tc: weights not prepared");
  int rc;
  if ((rc = launch_mlp_layer(ctx, 0, X_split, rows_cap, n_live, act_a, nullptr, st))) return rc;
  if ((rc = launch_mlp_layer(ctx, 1, act_a, rows_cap, n_live, act_b, nullptr, st))) return rc;
  if ((rc = launch_mlp_layer(ctx, 2, act_b, rows_cap, n_live, act_a, nullptr, st))) return rc;
  if ((rc = launch_mlp_layer(ctx, 3, act_a, rows_cap, n_live, act_b, nullptr, st))) return rc;
  return launch_mlp_layer(ctx, 4, act_b, rows_cap, n_live, nullptr, logits, st);
}

}  // namespace xf
