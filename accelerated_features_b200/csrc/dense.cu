// Semi-dense (XFeat*) coarse feature selection: top-k cells of the reliability map + gathers
// (XFeat.extractDense xfeat.py:366-375, extract_dualscale xfeat.py:388).
#include <cub/device/device_segmented_sort.cuh>

#include "common.cuh"

namespace xf {

__global__ void __launch_bounds__(256) dense_keys_kernel(const float* __restrict__ rel, int cells, int64_t total,
                                                         unsigned long long* __restrict__ keys) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const uint32_t cell = (uint32_t)(i % cells);
  keys[i] = ((unsigned long long)f2ord(__ldg(rel + i) + 0.0f) << 32) | (unsigned long long)(0xffffffffu - cell);
}

__global__ void uniform_offsets_kernel(int cells, int B, int* __restrict__ begin, int* __restrict__ end) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) { begin[b] = b * cells; end[b] = (b + 1) * cells; }
}

// One warp per (b, r < k): gather the un-normalised 64-D feature of the r-th most reliable cell and its coordinate.
__global__ void __launch_bounds__(256) dense_gather_kernel(const unsigned long long* __restrict__ sorted,
                                                           const float* __restrict__ feats, int B, int cells, int Wm,
                                                           int k, float rw, float rh, float div_scale, float scale_value,
                                                           int out_rows, int out_offset, float* __restrict__ kpts,
                                                           float* __restrict__ desc, float* __restrict__ scales,
                                                           int* __restrict__ topk_idx) {
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (int64_t)B * k) return;
  const int b = (int)(wid / k), r = (int)(wid - (int64_t)b * k);
  const unsigned long long key = sorted[(int64_t)b * cells + r];
  const int cell = (int)(0xffffffffu - (uint32_t)(key & 0xffffffffu));
  const float2 v = __ldg(reinterpret_cast<const float2*>(feats + ((int64_t)b * cells + cell) * 64) + lane);
  const int64_t orow = (int64_t)b * out_rows + out_offset + r;
  reinterpret_cast<float2*>(desc + orow * 64)[lane] = v;
  if (lane == 0) {
    const int x = cell % Wm, y = cell / Wm;
    // (xy * 8) * [rw, rh]  (xfeat.py:366,375) then / s (xfeat.py:388) -- fp32 multiply, fp32 true division
    kpts[orow * 2] = __fdiv_rn(__fmul_rn((float)(x * 8), rw), div_scale);
    kpts[orow * 2 + 1] = __fdiv_rn(__fmul_rn((float)(y * 8), rh), div_scale);
    if (scales) scales[orow] = scale_value;
    if (topk_idx) topk_idx[(int64_t)b * k + r] = cell;
  }
}

struct DenseWs {
  unsigned long long *keys, *sorted;
  int *seg_begin, *seg_end;
  void* cub_temp;
  size_t cub_bytes;
};
static int carve_dense(Bump& bump, int B, int cells, DenseWs& ws) {
  ws.keys = bump.take<unsigned long long>((size_t)B * cells);
  ws.sorted = bump.take<unsigned long long>((size_t)B * cells);
  ws.seg_begin = bump.take<int>(B);
  ws.seg_end = bump.take<int>(B);
  size_t tb = 0;
  cudaError_t e = cub::DeviceSegmentedSort::SortKeysDescending(nullptr, tb, (const unsigned long long*)nullptr,
                                                               (unsigned long long*)nullptr, B * cells, B, (const int*)nullptr,
                                                               (const int*)nullptr, (cudaStream_t)0);
  if (e != cudaSuccess) {
    set_error("cub temp-size query failed: %s", cudaGetErrorString(e));
    return XF_E_CUDA;
  }
  ws.cub_bytes = tb;
  ws.cub_temp = bump.take<char>(tb);
  return XF_OK;
}

}  // namespace xf

extern "C" size_t xfeat_dense_workspace_bytes(int B, int H, int W, int top_k) {
  (void)top_k;
  xf::Bump bump(nullptr, 0);
  xf::DenseWs ws;
  if (xf::carve_dense(bump, B, (H / 8) * (W / 8), ws) != XF_OK) return 0;
  return bump.used();
}

extern "C" int xfeat_detect_dense(xfeat_ctx* ctx, const float* d_feats, const float* d_reliability, int B, int H, int W,
                                  int top_k, float rw, float rh, float div_scale, float scale_value, int out_rows,
                                  int out_offset, float* d_kpts, float* d_desc, float* d_scales, int32_t* d_topk_idx,
                                  void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(ctx && d_feats && d_reliability && d_kpts && d_desc && d_ws, "detect_dense: null pointer");
  XF_REQUIRE(B > 0 && H > 0 && W > 0 && H % 32 == 0 && W % 32 == 0 && top_k > 0, "detect_dense: bad shape");
  const int Hm = H / 8, Wm = W / 8, cells = Hm * Wm;
  const int k = top_k < cells ? top_k : cells;  // torch.topk(k = min(len, top_k)), xfeat.py:371
  XF_REQUIRE(out_offset >= 0 && out_offset + k <= out_rows, "detect_dense: output rows [%d,%d) exceed %d", out_offset,
             out_offset + k, out_rows);
  XF_REQUIRE((int64_t)B * cells < (1ll << 31), "detect_dense: batch too large for 32-bit offsets");
  XF_REQUIRE(((uintptr_t)d_feats | (uintptr_t)d_desc) % 8 == 0,   // the gather moves feature rows as float2
             "detect_dense: d_feats and d_desc must be 8-byte aligned");
  XF_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  xf::Bump bump(d_ws, ws_bytes);
  xf::DenseWs ws;
  int rc = xf::carve_dense(bump, B, cells, ws);
  if (rc) return rc;
  if (!bump.ok) {
    xf::set_error("detect_dense: workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  const int64_t total = (int64_t)B * cells;
  xf::dense_keys_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_reliability, cells, total, ws.keys);
  XF_LAUNCH_CHECK();
  static const bool force_cub = getenv("XFEAT_TOPK_CUB") != nullptr;
  if (!force_cub && k <= 8192) {   // radix select + sort of the k survivors per image (sparse.cu) instead of sorting every cell
    if ((rc = xf::launch_topk_select_sort(ws.keys, nullptr, cells, cells, k, B, ws.sorted, st))) return rc;
  } else {
    xf::uniform_offsets_kernel<<<xf::cdiv(B, 128), 128, 0, st>>>(cells, B, ws.seg_begin, ws.seg_end);
    XF_LAUNCH_CHECK();
    size_t tb = ws.cub_bytes;
    XF_CUDA(cub::DeviceSegmentedSort::SortKeysDescending(ws.cub_temp, tb, ws.keys, ws.sorted, (int)total, B, ws.seg_begin,
                                                         ws.seg_end, st));
  }
  const int64_t warps = (int64_t)B * k;
  xf::dense_gather_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(
      ws.sorted, d_feats, B, cells, Wm, k, rw, rh, div_scale, scale_value, out_rows, out_offset, d_kpts, d_desc, d_scales,
      d_topk_idx);
  XF_LAUNCH_CHECK();
  return XF_OK;
}
