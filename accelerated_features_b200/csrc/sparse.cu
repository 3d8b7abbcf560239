// Sparse keypoint selection + description (xfeat.py:70-103):
//   nms_score_kernel   : 5x5 max-pool equality NMS + threshold (XFeat.NMS, xfeat.py:249-263) fused with the score
//                        nearest(K1h) * bilinear(H1) (xfeat.py:77-80) -> (score, pixel) keys appended per image;
//   cub segmented sort : argsort(-scores) (xfeat.py:83) with a deterministic tie rule (score desc, raster index asc);
//   sample_desc_kernel : top-k cut, bicubic sampling of the channel-normalised feature map (xfeat.py:70,90),
//                        L2 normalisation (xfeat.py:93), keypoint rescale (xfeat.py:96), valid count (xfeat.py:98).
// Everything stays on the device with fixed-capacity buffers; the only host-visible scalars are the per-image counts.
#include <cub/device/device_segmented_sort.cuh>

#include <stdlib.h>

#include <cuda_fp16.h>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace xf {

constexpr int NMS_TX = 64, NMS_TY = 16, NMS_R = 2;
constexpr int NMS_RW = NMS_TX / 8 + 4, NMS_RH = NMS_TY / 8 + 3;   // cached window of the 1/8-res reliability map

// Phase A: every pixel tests "is 5x5 maximum and > threshold" (separable max in shared memory) and the few hits are
// compacted into a CTA-local list.  Phase B: the list is scored densely (one candidate per thread) -- the score path
// (coordinate arithmetic, nearest + bilinear sampling) is ~10x longer than the test and would otherwise be executed by
// every warp under divergence.  Phase C: one global atomic per CTA reserves the output range.
__global__ void __launch_bounds__(256) nms_score_kernel(const float* __restrict__ heat, const float* __restrict__ rel,
                                                        int H, int W, int Hm, int Wm, float thr, int cap,
                                                        unsigned long long* __restrict__ keys,
                                                        int* __restrict__ n_keep, int* __restrict__ n_cand) {
  __shared__ float sIn[NMS_TY + 2 * NMS_R][NMS_TX + 2 * NMS_R];
  __shared__ float sRow[NMS_TY + 2 * NMS_R][NMS_TX];
  __shared__ unsigned long long sKeys[NMS_TX * NMS_TY];
  __shared__ unsigned short sCand[NMS_TX * NMS_TY];   // tile-local pixel index of each maximum
  __shared__ int sCnt[3];  // [0] maxima above threshold, [1] kept (score > 0), [2] global base
  __shared__ float sRel[NMS_RH][NMS_RW];
  const int b = blockIdx.z;
  const int ox0 = blockIdx.x * NMS_TX, oy0 = blockIdx.y * NMS_TY;
  const float* hb = heat + (int64_t)b * H * W;
  const float* rb = rel + (int64_t)b * Hm * Wm;
  const int rx0 = ox0 / 8 - 1, ry0 = oy0 / 8 - 1;   // window origin (cells); all bilinear taps of this tile fall inside
  constexpr int PW = NMS_TX + 2 * NMS_R, PH = NMS_TY + 2 * NMS_R;
  if (threadIdx.x < 3) sCnt[threadIdx.x] = 0;
  for (int idx = threadIdx.x; idx < NMS_RW * NMS_RH; idx += 256) {
    const int r = idx / NMS_RW, c = idx - r * NMS_RW;
    const int cy = ry0 + r, cx = rx0 + c;
    sRel[r][c] = (cy >= 0 && cy < Hm && cx >= 0 && cx < Wm) ? __ldg(rb + (int64_t)cy * Wm + cx) : 0.f;
  }
  for (int idx = threadIdx.x; idx < PW * PH; idx += 256) {
    const int r = idx / PW, c = idx - r * PW;
    const int y = oy0 - NMS_R + r, x = ox0 - NMS_R + c;
    sIn[r][c] = (y >= 0 && y < H && x >= 0 && x < W) ? __ldg(hb + (int64_t)y * W + x) : -INFINITY;  // MaxPool2d pads with -inf
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < PH * NMS_TX; idx += 256) {
    const int r = idx / NMS_TX, c = idx - r * NMS_TX;
    float m = sIn[r][c];
#pragma unroll
    for (int d = 1; d <= 2 * NMS_R; ++d) m = fmaxf(m, sIn[r][c + d]);
    sRow[r][c] = m;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  // ---- phase A: detect + compact ----
#pragma unroll
  for (int k = 0; k < (NMS_TX * NMS_TY) / 256; ++k) {
    const int idx = threadIdx.x + 256 * k;
    const int r = idx / NMS_TX, c = idx - r * NMS_TX;
    float m = sRow[r][c];
#pragma unroll
    for (int d = 1; d <= 2 * NMS_R; ++d) m = fmaxf(m, sRow[r + d][c]);
    const float v = sIn[r + NMS_R][c + NMS_R];
    const bool pos = (ox0 + c < W) && (oy0 + r < H) && (v == m) && (v > thr);
    const unsigned mpos = __ballot_sync(0xffffffffu, pos);
    if (mpos) {
      const int leader = __ffs(mpos) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(&sCnt[0], __popc(mpos));
      base = __shfl_sync(0xffffffffu, base, leader);
      if (pos) sCand[base + __popc(mpos & ((1u << lane) - 1u))] = (unsigned short)idx;
    }
  }
  __syncthreads();
  // ---- phase B: score the candidates densely ----
  const int nc = sCnt[0];
  for (int i0 = 0; i0 < nc; i0 += 256) {
    const int i = i0 + threadIdx.x;
    bool keep = false;
    unsigned long long key = 0;
    if (i < nc) {
      const int idx = sCand[i];
      const int r = idx / NMS_TX, c = idx - r * NMS_TX;
      const int x = ox0 + c, y = oy0 + r;
      const float v = sIn[r + NMS_R][c + NMS_R];
      // nearest sample of the heat-map at the keypoint itself: round-half-even of x*W/(W-1)-0.5 is x except on the
      // last row/column, where it falls out of bounds -> 0 (reference quirk, SURVEY 8a-7 A).
      const int xn = (int)rintf(sparse_src_coord(x, W, W));
      const int yn = (int)rintf(sparse_src_coord(y, H, H));
      float kv = 0.f;
      if (xn >= 0 && xn < W && yn >= 0 && yn < H) kv = (xn == x && yn == y) ? v : __ldg(hb + (int64_t)yn * W + xn);
      // bilinear sample of the 1/8-res reliability map, zeros padding (ATen grid_sampler_2d)
      const float ix = sparse_src_coord(x, W, Wm), iy = sparse_src_coord(y, H, Hm);
      const float fx = floorf(ix), fy = floorf(iy);
      const int x0 = (int)fx, y0 = (int)fy;
      const float wx1 = __fsub_rn(ix, fx), wx0 = __fsub_rn(__fadd_rn(fx, 1.0f), ix);
      const float wy1 = __fsub_rn(iy, fy), wy0 = __fsub_rn(__fadd_rn(fy, 1.0f), iy);
      float bil = 0.f;
      const bool xin0 = (x0 >= 0 && x0 < Wm), xin1 = (x0 + 1 >= 0 && x0 + 1 < Wm);
      const bool yin0 = (y0 >= 0 && y0 < Hm), yin1 = (y0 + 1 >= 0 && y0 + 1 < Hm);
      const int wx = x0 - rx0, wy = y0 - ry0;          // position inside the cached window
      const bool cached = (wx >= 0 && wx + 1 < NMS_RW && wy >= 0 && wy + 1 < NMS_RH);
      auto R = [&](int yy, int xx) -> float {
        return cached ? sRel[yy - ry0][xx - rx0] : __ldg(rb + (int64_t)yy * Wm + xx);
      };
      if (xin0 && yin0) bil = __fadd_rn(bil, __fmul_rn(R(y0, x0), __fmul_rn(wx0, wy0)));
      if (xin1 && yin0) bil = __fadd_rn(bil, __fmul_rn(R(y0, x0 + 1), __fmul_rn(wx1, wy0)));
      if (xin0 && yin1) bil = __fadd_rn(bil, __fmul_rn(R(y0 + 1, x0), __fmul_rn(wx0, wy1)));
      if (xin1 && yin1) bil = __fadd_rn(bil, __fmul_rn(R(y0 + 1, x0 + 1), __fmul_rn(wx1, wy1)));
      float score = __fmul_rn(kv, bil);
      if (x == 0 && y == 0) score = -1.f;  // indistinguishable from the zero padding rows (xfeat.py:80)
      keep = score > 0.f;                  // `valid = scores > 0` (xfeat.py:98) applied early: positives sort first anyway
      key = ((unsigned long long)f2ord(score) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)(y * W + x));
    }
    const unsigned mkeep = __ballot_sync(0xffffffffu, keep);
    if (mkeep) {
      const int leader = __ffs(mkeep) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(&sCnt[1], __popc(mkeep));
      base = __shfl_sync(0xffffffffu, base, leader);
      if (keep) sKeys[base + __popc(mkeep & ((1u << lane) - 1u))] = key;
    }
  }
  __syncthreads();
  // ---- phase C: reserve the output range, write ----
  const int nk = sCnt[1];
  if (threadIdx.x == 0) {
    if (nc) atomicAdd(&n_cand[b], nc);
    sCnt[2] = nk ? atomicAdd(&n_keep[b], nk) : 0;
  }
  __syncthreads();
  const int gbase = sCnt[2];
  for (int i = threadIdx.x; i < nk; i += 256)
    if (gbase + i < cap) keys[(int64_t)b * cap + gbase + i] = sKeys[i];
}

// Score of one NMS survivor, packed as a sort key: nearest(K1h) * bilinear(H1) with the reference's out-of-range quirks
// (xfeat.py:77-80); returns false when the score is not positive (`valid = scores > 0`, xfeat.py:98).
__device__ __forceinline__ bool nms_score_key(const float* __restrict__ hb, const float* __restrict__ rb, int x, int y, float v,
                                              int H, int W, int Hm, int Wm, unsigned long long& key) {
  const int xn = (int)rintf(sparse_src_coord(x, W, W));
  const int yn = (int)rintf(sparse_src_coord(y, H, H));
  float kv = 0.f;
  if (xn >= 0 && xn < W && yn >= 0 && yn < H) kv = (xn == x && yn == y) ? v : __ldg(hb + (int64_t)yn * W + xn);
  const float ix = sparse_src_coord(x, W, Wm), iy = sparse_src_coord(y, H, Hm);
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy;
  const float wx1 = __fsub_rn(ix, fx), wx0 = __fsub_rn(__fadd_rn(fx, 1.0f), ix);
  const float wy1 = __fsub_rn(iy, fy), wy0 = __fsub_rn(__fadd_rn(fy, 1.0f), iy);
  const bool xin0 = (x0 >= 0 && x0 < Wm), xin1 = (x0 + 1 >= 0 && x0 + 1 < Wm);
  const bool yin0 = (y0 >= 0 && y0 < Hm), yin1 = (y0 + 1 >= 0 && y0 + 1 < Hm);
  float bil = 0.f;
  if (xin0 && yin0) bil = __fadd_rn(bil, __fmul_rn(__ldg(rb + (int64_t)y0 * Wm + x0), __fmul_rn(wx0, wy0)));
  if (xin1 && yin0) bil = __fadd_rn(bil, __fmul_rn(__ldg(rb + (int64_t)y0 * Wm + x0 + 1), __fmul_rn(wx1, wy0)));
  if (xin0 && yin1) bil = __fadd_rn(bil, __fmul_rn(__ldg(rb + (int64_t)(y0 + 1) * Wm + x0), __fmul_rn(wx0, wy1)));
  if (xin1 && yin1) bil = __fadd_rn(bil, __fmul_rn(__ldg(rb + (int64_t)(y0 + 1) * Wm + x0 + 1), __fmul_rn(wx1, wy1)));
  float score = __fmul_rn(kv, bil);
  if (x == 0 && y == 0) score = -1.f;  // indistinguishable from the zero padding rows (xfeat.py:80)
  key = ((unsigned long long)f2ord(score) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)(y * W + x));
  return score > 0.f;
}

// Overflow path of nms_march_kernel (CTA-local list full): score and append one survivor directly.  Not inlined: it would be
// replicated into every unrolled row of the march and push the hot loop out of the instruction cache.
__device__ __noinline__ void nms_emit_direct(const float* __restrict__ hb, const float* __restrict__ rb, int px, int py, float v,
                                             int H, int W, int Hm, int Wm, unsigned long long* __restrict__ keys_b,
                                             int* __restrict__ n_keep_b, int cap) {
  unsigned long long key;
  if (nms_score_key(hb, rb, px, py, v, H, W, Hm, Wm, key)) {
    const int g = atomicAdd(n_keep_b, 1);
    if (g < cap) keys_b[g] = key;
  }
}

// Register-marching variant of the NMS test (default).  A warp owns a 128-pixel-wide column strip and walks down NM_RS + 4
// rows: one 128-bit load per lane and row, the two neighbours on either side come from the adjacent lanes by shuffle, the
// horizontal 5-max of the last five rows lives in a register ring, so the heat-map is read once (plus 4 halo rows per strip)
// and no shared-memory tile or block barrier sits on the streaming path.  Survivors (a few per cent of the pixels) go to a
// CTA-local list and are scored densely afterwards exactly as in nms_score_kernel; a full list degrades to direct emission.
constexpr int NM_WARPS = 4, NM_RS = 16, NM_TW = 128, NM_LIST = 1024;

__global__ void __launch_bounds__(NM_WARPS * 32, 5) nms_march_kernel(const float* __restrict__ heat, const float* __restrict__ rel,
                                                                  int H, int W, int Hm, int Wm, float thr, int cap,
                                                                  unsigned long long* __restrict__ keys,
                                                                  int* __restrict__ n_keep, int* __restrict__ n_cand) {
  __shared__ unsigned sPos[NM_LIST];
  __shared__ float sVal[NM_LIST];
  __shared__ unsigned long long sKeys[NM_LIST];
  __shared__ int sCnt[3];  // [0] maxima above threshold, [1] kept (score > 0), [2] global base
  const int b = blockIdx.z, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* hb = heat + (int64_t)b * H * W;
  const float* rb = rel + (int64_t)b * Hm * Wm;
  if (threadIdx.x < 3) sCnt[threadIdx.x] = 0;
  __syncthreads();
  const int x = blockIdx.x * NM_TW + lane * 4;
  const int y0 = (blockIdx.y * NM_WARPS + warp) * NM_RS;
  const bool xin = x < W;   // W % 4 == 0: a lane's four pixels are inside or outside together
  if (y0 < H) {
    float hr[5][4];   // horizontal 5-max of the last five rows
    float vc[5][4];   // centre values of the last five rows (same period as hr, so every batch of NB = 5 rows is the same code)
    constexpr int NB = 5;   // rows loaded per batch: all loads of a batch are issued before the first is consumed
    static_assert((NM_RS + 4) % NB == 0, "march length must be a multiple of the load batch");
#pragma unroll 1   // rolled: the fully unrolled march (20 rows) stalled on instruction fetch (ncu: no_instruction 3.0 per issue)
    for (int i0 = 0; i0 < NM_RS + 4; i0 += NB) {
    float4 vb[NB];
    float2 eb[NB];   // lane 0: pixels x-2, x-1; lane 31: pixels x+4, x+5 (the neighbours no other lane of the warp holds)
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      const int y = y0 - 2 + i0 + u;
      const bool yin = y >= 0 && y < H;
      const float* row = hb + (int64_t)(yin ? y : 0) * W;
      vb[u] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);   // MaxPool2d pads with -inf
      eb[u] = make_float2(-INFINITY, -INFINITY);
      if (yin && xin) vb[u] = __ldg(reinterpret_cast<const float4*>(row + x));
      if (yin && xin && lane == 0 && x > 0) eb[u] = __ldg(reinterpret_cast<const float2*>(row + x - 2));
      if (yin && lane == 31 && x + 4 < W) eb[u] = __ldg(reinterpret_cast<const float2*>(row + x + 4));
    }
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      const int i = i0 + u;
      const int y = y0 - 2 + i;
      const float4 v = vb[u];
      float l1 = __shfl_up_sync(0xffffffffu, v.w, 1);
      float l2 = __shfl_up_sync(0xffffffffu, v.z, 1);
      float r1 = __shfl_down_sync(0xffffffffu, v.x, 1);
      float r2 = __shfl_down_sync(0xffffffffu, v.y, 1);
      if (lane == 0) { l2 = eb[u].x; l1 = eb[u].y; }
      if (lane == 31) { r1 = eb[u].x; r2 = eb[u].y; }
      const float mxyz = fmaxf(fmaxf(v.x, v.y), v.z), myzw = fmaxf(fmaxf(v.y, v.z), v.w);
      hr[u][0] = fmaxf(fmaxf(l2, l1), mxyz);
      hr[u][1] = fmaxf(fmaxf(l1, v.w), mxyz);
      hr[u][2] = fmaxf(fmaxf(v.x, r1), myzw);
      hr[u][3] = fmaxf(fmaxf(r1, r2), myzw);
      vc[u][0] = v.x; vc[u][1] = v.y; vc[u][2] = v.z; vc[u][3] = v.w;
      if (i >= 4) {
        const int yo = y - 2;   // output row: window rows yo-2 .. yo+2 are in the ring
        unsigned mask = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float m = fmaxf(fmaxf(fmaxf(hr[0][k], hr[1][k]), fmaxf(hr[2][k], hr[3][k])), hr[4][k]);
          const float c = vc[(u + 3) % 5][k];
          if (c == m && c > thr) mask |= 1u << k;
        }
        if (!(xin && yo < H)) mask = 0;
        if (mask) {
          int e = atomicAdd(&sCnt[0], __popc(mask));
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (mask & (1u << k)) {
              const float c = vc[(u + 3) % 5][k];
              if (e < NM_LIST) {
                sPos[e] = (uint32_t)(yo * W + x + k);
                sVal[e] = c;
              } else {
                nms_emit_direct(hb, rb, x + k, yo, c, H, W, Hm, Wm, keys + (int64_t)b * cap, n_keep + b, cap);
              }
              ++e;
            }
        }
      }
    }
    }
  }
  __syncthreads();
  // ---- score the survivors densely, compact the positive scores ----
  const int nc_all = sCnt[0];
  const int nc = nc_all < NM_LIST ? nc_all : NM_LIST;
  for (int i0 = 0; i0 < nc; i0 += NM_WARPS * 32) {
    const int i = i0 + threadIdx.x;
    bool keep = false;
    unsigned long long key = 0;
    if (i < nc) {
      const int pix = (int)sPos[i];
      const int py = pix / W, px = pix - py * W;
      keep = nms_score_key(hb, rb, px, py, sVal[i], H, W, Hm, Wm, key);
    }
    const unsigned mkeep = __ballot_sync(0xffffffffu, keep);
    if (mkeep) {
      const int leader = __ffs(mkeep) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(&sCnt[1], __popc(mkeep));
      base = __shfl_sync(0xffffffffu, base, leader);
      if (keep) sKeys[base + __popc(mkeep & ((1u << lane) - 1u))] = key;
    }
  }
  __syncthreads();
  const int nk = sCnt[1];
  if (threadIdx.x == 0) {
    if (nc_all) atomicAdd(&n_cand[b], nc_all);
    sCnt[2] = nk ? atomicAdd(&n_keep[b], nk) : 0;
  }
  __syncthreads();
  const int gbase = sCnt[2];
  for (int i = threadIdx.x; i < nk; i += NM_WARPS * 32)
    if (gbase + i < cap) keys[(int64_t)b * cap + gbase + i] = sKeys[i];
}


// Per-image top-k of the NMS candidates, sorted (replaces the capacity-wide cub segmented sort for top_k <= 8192: the sort
// handled every candidate -- 20-30 k per noise image -- to keep 4096).  One CTA per image:
//   1. radix select (11-bit digits, most significant first) of the k-th largest 64-bit key; keys are unique (the pixel index sits
//      in the low word), so the k largest are exactly the keys >= that threshold;  2. compaction of those k keys into shared
//   memory;  3. bitonic sort, descending.  Same order as the cub sort: (score desc, raster index asc).
constexpr int TS_THREADS = 1024, TS_BITS = 11, TS_BINS = 1 << TS_BITS;

__global__ void __launch_bounds__(TS_THREADS) topk_select_sort_kernel(const unsigned long long* __restrict__ keys,
                                                                      const int* __restrict__ n_keep, int n_const, int cap, int top_k,
                                                                      int P, unsigned long long* __restrict__ sorted) {
  extern __shared__ unsigned long long sK[];   // [P], P = power of two >= top_k
  __shared__ int sHist[TS_BINS];
  __shared__ int sSel[2];                      // chosen digit, keys taken from the digits above it
  __shared__ int sCnt;
  using Scan = cub::BlockScan<int, TS_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int nk = n_keep ? n_keep[b] : n_const;
  if (nk > cap) return;                        // candidate overflow: the sampler reports XF_N_OVERFLOW and reads nothing
  const int n = nk, k = min(n, top_k);
  const unsigned long long* kb = keys + (int64_t)b * cap;
  for (int i = tid; i < P; i += TS_THREADS) sK[i] = 0ull;
  __syncthreads();
  if (n <= top_k) {
    for (int i = tid; i < n; i += TS_THREADS) sK[i] = kb[i];
  } else {
    unsigned long long prefix = 0ull;          // digits chosen so far (the high 64 - shift bits of the threshold)
    int remaining = k, shift = 64;
    unsigned long long sel_val = 0ull;
    int sel_shift = 0;
    while (true) {
      const int bits = (shift >= TS_BITS) ? TS_BITS : shift;
      const int hi_shift = shift;              // keys must agree with `prefix` above this bit
      shift -= bits;
      for (int i = tid; i < TS_BINS; i += TS_THREADS) sHist[i] = 0;
      __syncthreads();
      const unsigned mask = (1u << bits) - 1u;
      for (int i = tid; i < n; i += TS_THREADS) {
        const unsigned long long key = kb[i];
        if (hi_shift == 64 || (key >> hi_shift) == prefix) atomicAdd(&sHist[(unsigned)(key >> shift) & mask], 1);
      }
      __syncthreads();
      // from the largest digit down: first digit D whose cumulative count reaches `remaining`
      const int r0 = 2 * tid, r1 = 2 * tid + 1;                       // reversed bin indices (0 = largest digit)
      const int c0 = sHist[TS_BINS - 1 - r0], c1 = sHist[TS_BINS - 1 - r1];
      int excl, total;
      Scan(scan_tmp).ExclusiveSum(c0 + c1, excl, total);
      if (excl < remaining && excl + c0 >= remaining) { sSel[0] = TS_BINS - 1 - r0; sSel[1] = excl; }
      else if (excl + c0 < remaining && excl + c0 + c1 >= remaining) { sSel[0] = TS_BINS - 1 - r1; sSel[1] = excl + c0; }
      __syncthreads();
      const int D = sSel[0], need = remaining - sSel[1], have = sHist[D];
      prefix = (prefix << bits) | (unsigned long long)D;
      __syncthreads();                          // sHist / sSel are rewritten by the next round
      if (need == have || shift == 0) {         // the whole bucket is wanted: the threshold is settled at this digit
        sel_val = prefix;
        sel_shift = shift;
        break;
      }
      remaining = need;
    }
    if (tid == 0) sCnt = 0;
    __syncthreads();
    for (int i = tid; i < n; i += TS_THREADS) {
      const unsigned long long key = kb[i];
      if ((key >> sel_shift) >= sel_val) {
        const int pos = atomicAdd(&sCnt, 1);
        if (pos < P) sK[pos] = key;
      }
    }
  }
  // bitonic sort, descending
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = tid; t < (P >> 1); t += TS_THREADS) {
        const int i = 2 * t - (t & (stride - 1)), j = i + stride;
        const bool desc = ((i & size) == 0);
        const unsigned long long a = sK[i], c = sK[j];
        if ((a < c) == desc) { sK[i] = c; sK[j] = a; }
      }
    }
  __syncthreads();
  for (int r = tid; r < k; r += TS_THREADS) sorted[(int64_t)b * cap + r] = sK[r];
}

// keys: B segments of `cap` slots, the first n_keep[b] (or n_const when n_keep is null) valid; sorted[b * cap + r], r < min(n, top_k)
int launch_topk_select_sort(const unsigned long long* keys, const int* n_keep, int n_const, int cap, int top_k, int B,
                            unsigned long long* sorted, cudaStream_t st) {
  XF_REQUIRE(top_k > 0 && top_k <= 8192, "topk_select_sort: top_k %d out of range", top_k);
  int P = 1;
  while (P < top_k) P <<= 1;
  const size_t smem_ts = (size_t)P * sizeof(unsigned long long);
  XF_DYN_SMEM(topk_select_sort_kernel, smem_ts);
  topk_select_sort_kernel<<<B, TS_THREADS, smem_ts, st>>>(keys, n_keep, n_const, cap, top_k, P, sorted);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

__global__ void segment_offsets_kernel(const int* __restrict__ counts, int cap, int B, int* __restrict__ begin,
                                       int* __restrict__ end) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) {
    begin[b] = b * cap;
    end[b] = b * cap + min(counts[b], cap);
  }
}

__device__ __forceinline__ float cubic1(float x) {  // |x| <= 1, A = -0.75 (ATen cubic_convolution1)
  const float A = -0.75f;
  return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
}
__device__ __forceinline__ float cubic2(float x) {  // 1 < |x| < 2 (ATen cubic_convolution2)
  const float A = -0.75f;
  return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
}

// den[p] = 1 / max(||feats[p]||_2, 1e-12): reciprocal of the denominator of F.normalize(M1, dim=1) (xfeat.py:70), so that the
// sampler multiplies instead of dividing 64 times per keypoint (<= 1 ulp away from x / den). 8 lanes per pixel.
__global__ void __launch_bounds__(256) feat_norm_kernel(const float* __restrict__ feats, float* __restrict__ den,
                                                        int64_t npix) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t pix = gid >> 3;
  const int sub = (int)(gid & 7);
  float s = 0.f;
  if (pix < npix) {
    const float4* tp = reinterpret_cast<const float4*>(feats + pix * 64) + sub * 2;
    const float4 a0 = __ldg(tp), a1 = __ldg(tp + 1);
    s = a0.x * a0.x + a0.y * a0.y + a0.z * a0.z + a0.w * a0.w + a1.x * a1.x + a1.y * a1.y + a1.z * a1.z + a1.w * a1.w;
  }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (pix < npix && sub == 0) den[pix] = __fdiv_rn(1.0f, fmaxf(sqrtf(s), 1e-12f));
}

// Bicubic sample (ATen grid_sampler_2d, A = -0.75, zeros padding) of the channel-normalised map at pixel (x, y), for the 4
// channels owned by lane l16 of a 16-lane group; returns the un-normalised 4-vector and the group-wide sum of squares.
// UNIFORM: every lane of the warp calls (with valid coordinates), so the interior test can be made warp-wide and the two
// half-warps of a keypoint pair never run both paths one after the other.
template <bool UNIFORM>
__device__ __forceinline__ float4 bicubic4(const float* __restrict__ fb, const float* __restrict__ db, int x, int y, int H, int W,
                                           int Hm, int Wm, int l16) {
  const float ix = sparse_src_coord(x, W, Wm), iy = sparse_src_coord(y, H, Hm);
  const float fx = floorf(ix), fy = floorf(iy);
  const float tx = __fsub_rn(ix, fx), ty = __fsub_rn(iy, fy);
  const int x0 = (int)fx - 1, y0 = (int)fy - 1;
  const float cx[4] = {cubic2(tx + 1.f), cubic1(tx), cubic1(1.f - tx), cubic2((1.f - tx) + 1.f)};
  const float cy[4] = {cubic2(ty + 1.f), cubic1(ty), cubic1(1.f - ty), cubic2((1.f - ty) + 1.f)};
  bool interior = x0 >= 0 && x0 + 3 < Wm && y0 >= 0 && y0 + 3 < Hm;
  if (UNIFORM) interior = __all_sync(0xffffffffu, interior);
  const float4* f4 = reinterpret_cast<const float4*>(fb) + (uint32_t)l16;
  // per component: v*d, then fma(v*d, cx[j], row), then fma(row, cy[i], out)
  float2 oa = make_float2(0.f, 0.f), ob = make_float2(0.f, 0.f);
  if (interior) {
    // interior keypoint (almost all): no per-tap tests, 32-bit offsets from one base pointer
    const float4* p0 = f4 + (uint32_t)(y0 * Wm + x0) * 16u;
    const float* d0 = db + (uint32_t)(y0 * Wm + x0);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 ra = make_float2(0.f, 0.f), rb = make_float2(0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 v = __ldg(p0 + (uint32_t)(i * Wm + j) * 16u);
        const float d = __ldg(d0 + (uint32_t)(i * Wm + j));
        const float2 dd = make_float2(d, d), cc = make_float2(cx[j], cx[j]);
        ra = f2_fma(f2_mul(make_float2(v.x, v.y), dd), cc, ra);
        rb = f2_fma(f2_mul(make_float2(v.z, v.w), dd), cc, rb);
      }
      const float2 cyy = make_float2(cy[i], cy[i]);
      oa = f2_fma(ra, cyy, oa);
      ob = f2_fma(rb, cyy, ob);
    }
    return make_float4(oa.x, oa.y, ob.x, ob.y);
  }
  // border keypoint: taps outside the map add nothing (grid_sample zeros padding).  The address is clamped into the map and the
  // tap's normaliser d is replaced by 0, so the same instruction sequence runs (v*0 = +-0, and row + (+-0 * c) == row bit for
  // bit: the accumulators start at +0) -- 16 unconditional taps instead of 16 predicated ones with 64-bit addressing.
  uint32_t xo[4], yo[4];
  bool vx[4], vy[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int xx = x0 + k, yy = y0 + k;
    vx[k] = xx >= 0 && xx < Wm;
    vy[k] = yy >= 0 && yy < Hm;
    xo[k] = (uint32_t)min(max(xx, 0), Wm - 1);
    yo[k] = (uint32_t)min(max(yy, 0), Hm - 1) * (uint32_t)Wm;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 ra = make_float2(0.f, 0.f), rb = make_float2(0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t off = yo[i] + xo[j];
      const float4 v = __ldg(f4 + off * 16u);
      float d = __ldg(db + off);                 // 1 / F.normalize(M1, dim=1) denominator, xfeat.py:70
      if (!(vx[j] && vy[i])) d = 0.f;
      const float2 dd = make_float2(d, d), cc = make_float2(cx[j], cx[j]);
      ra = f2_fma(f2_mul(make_float2(v.x, v.y), dd), cc, ra);
      rb = f2_fma(f2_mul(make_float2(v.z, v.w), dd), cc, rb);
    }
    const float2 cyy = make_float2(cy[i], cy[i]);
    oa = f2_fma(ra, cyy, oa);
    ob = f2_fma(rb, cyy, ob);
  }
  return make_float4(oa.x, oa.y, ob.x, ob.y);
}

// Sum of squares of the lane's 4 channels with explicit rounding: both samplers must produce the same bits, which a
// compiler-chosen FMA contraction does not guarantee across kernels.
__device__ __forceinline__ float sumsq4(const float4& o) {
  return __fmaf_rn(o.w, o.w, __fmaf_rn(o.z, o.z, __fmaf_rn(o.y, o.y, __fmul_rn(o.x, o.x))));
}

// Half a warp per output slot (b, r): lane owns 4 channels. feats: (B,Hm,Wm,64) NHWC un-normalised, den: (B,Hm,Wm).
// The matcher's operand row of a unit-norm descriptor: x * 2^13 = hi + lo in fp16, [hi(64) | lo(64)] (mnn_tc.cu, abs_bound = 1).
// Written next to the fp32 descriptor so xfeat_mnn_match_presplit needs no max-reduction / split pass over the descriptors.
constexpr float kDescSplitScale = 8192.0f;
__device__ __forceinline__ void store_desc_split(__half* sp, const float4& d) {
  const float x0 = d.x * kDescSplitScale, x1 = d.y * kDescSplitScale, x2 = d.z * kDescSplitScale, x3 = d.w * kDescSplitScale;
  const __half2 h0 = __floats2half2_rn(x0, x1), h1 = __floats2half2_rn(x2, x3);
  const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  const __half2 l0 = __floats2half2_rn(x0 - f0.x, x1 - f0.y), l1 = __floats2half2_rn(x2 - f1.x, x3 - f1.y);
  *reinterpret_cast<uint2*>(sp) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
  *reinterpret_cast<uint2*>(sp + 64) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
}

// Generic kernel (any top_k): slots are visited in score order, so taps of neighbouring keypoints rarely share L1 lines.
__global__ void __launch_bounds__(256) sample_desc_kernel(const unsigned long long* __restrict__ sorted,
                                                          const int* __restrict__ n_keep, const float* __restrict__ feats,
                                                          const float* __restrict__ den, int B, int H, int W, int Hm, int Wm,
                                                          int cap, int top_k, float rw, float rh, float* __restrict__ kpts,
                                                          float* __restrict__ scores, float* __restrict__ desc,
                                                          int* __restrict__ n_valid, int* __restrict__ kpts_int,
                                                          __half* __restrict__ desc_split, int split_rows) {
  const int64_t slot = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
  const int l16 = threadIdx.x & 15;
  const int64_t total = (int64_t)B * top_k;
  const bool live = slot < total;
  const int64_t sl = live ? slot : total - 1;   // keep the whole warp converged for the shuffles below
  const int b = (int)(sl / top_k), r = (int)(sl - (int64_t)b * top_k);
  const int nk = n_keep[b];
  const int nv = nk > cap ? 0 : min(nk, top_k);   // candidate overflow: nothing is trusted, n_valid = XF_N_OVERFLOW (header)
  if (live && r == 0 && l16 == 0) n_valid[b] = nk > cap ? -1 : nv;
  const bool valid = r < nv;
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  int x = 0, y = 0;
  unsigned long long key = 0;
  if (valid) {
    key = sorted[(int64_t)b * cap + r];
    const uint32_t lin = 0xffffffffu - (uint32_t)(key & 0xffffffffu);
    x = (int)(lin % (uint32_t)W); y = (int)(lin / (uint32_t)W);
    o = bicubic4<false>(feats + (int64_t)b * Hm * Wm * 64, den + (int64_t)b * Hm * Wm, x, y, H, W, Hm, Wm, l16);
  }
  float ss = sumsq4(o);
#pragma unroll
  for (int s = 8; s > 0; s >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, s);
  if (!live) return;
  float4* dp = desc ? reinterpret_cast<float4*>(desc + slot * 64) + l16 : nullptr;   // desc == null: only the matcher's rows are wanted
  __half* sp = desc_split ? desc_split + ((int64_t)b * split_rows + r) * 128 + l16 * 4 : nullptr;
  if (!valid) {
    if (dp) *dp = make_float4(0.f, 0.f, 0.f, 0.f);
    if (sp) { *reinterpret_cast<uint2*>(sp) = make_uint2(0u, 0u); *reinterpret_cast<uint2*>(sp + 64) = make_uint2(0u, 0u); }
    if (l16 == 0) {
      kpts[slot * 2] = 0.f; kpts[slot * 2 + 1] = 0.f; scores[slot] = 0.f;
      if (kpts_int) { kpts_int[slot * 2] = 0; kpts_int[slot * 2 + 1] = 0; }
    }
    return;
  }
  const float dn = __fdiv_rn(1.0f, fmaxf(sqrtf(ss), 1e-12f));  // F.normalize(feats, dim=-1), xfeat.py:93
  const float4 dv = make_float4(o.x * dn, o.y * dn, o.z * dn, o.w * dn);
  if (dp) *dp = dv;
  if (sp) store_desc_split(sp, dv);
  if (l16 == 0) {
    kpts[slot * 2] = __fmul_rn((float)x, rw);  // mkpts * [rw, rh], xfeat.py:96
    kpts[slot * 2 + 1] = __fmul_rn((float)y, rh);
    scores[slot] = ord2f((uint32_t)(key >> 32));
    if (kpts_int) { kpts_int[slot * 2] = x; kpts_int[slot * 2 + 1] = y; }
  }
}

// One CTA per image (top_k <= SAMPLE_MAX_K): the image's top-k keys are bucketed by feature-map row in shared memory and
// the keypoints are then processed in that (spatial) order, so the 4x4x256 B tap blocks of neighbouring keypoints hit
// L1 instead of L2 (5x5 NMS puts keypoints >= 3 px apart while a feature cell covers 8 px).  Results go to the slot given
// by the score rank, exactly as in the generic kernel.
// (Sharing an image between 4 CTAs of 512 threads, each repeating the bucketing, measured 321 us vs 268 us: not kept.)
// 256-thread CTAs, SAMPLE_PARTS per image (each rebuilds the image's spatial order -- 4096 shared-memory atomics -- and samples its
// share of it): 4 CTAs per SM by registers, and the 128 x 8 CTAs of the BASELINE batch spread over all SMs, where one
// 1024-thread CTA per image left 20 SMs idle.
constexpr int SAMPLE_MAX_K = 8192, SAMPLE_THREADS = 256, SAMPLE_MAX_ROWS = 512, SAMPLE_PARTS = 8;
__global__ void __launch_bounds__(SAMPLE_THREADS, 4) sample_desc_sorted_kernel(
    const unsigned long long* __restrict__ sorted, const int* __restrict__ n_keep, const float* __restrict__ feats,
    const float* __restrict__ den, int H, int W, int Hm, int Wm, int cap, int top_k, float rw, float rh, float* __restrict__ kpts,
    float* __restrict__ scores, float* __restrict__ desc, int* __restrict__ n_valid, int* __restrict__ kpts_int,
    __half* __restrict__ desc_split, int split_rows, unsigned long long magic_w, unsigned long long magic_xw) {
  extern __shared__ unsigned char sm_raw[];
  unsigned long long* sKey = reinterpret_cast<unsigned long long*>(sm_raw);           // [top_k]
  unsigned short* sOrder = reinterpret_cast<unsigned short*>(sKey + top_k);            // [top_k]
  unsigned short* sBkt = sOrder + top_k;                                               // [top_k] bucket of key r
  __shared__ int sHist[SAMPLE_MAX_ROWS];
  const int b = blockIdx.x, tid = threadIdx.x, part = blockIdx.y, nparts = gridDim.y;
  const int nk = n_keep[b];
  const int nv = nk > cap ? 0 : min(nk, top_k);   // candidate overflow: nothing is trusted, n_valid = XF_N_OVERFLOW (header)
  if (tid == 0 && part == 0) n_valid[b] = nk > cap ? -1 : nv;
  // spatial buckets: one feature row (8 image rows) x nxb column strips, so that the 4 x (strip + 3) cells the taps of
  // consecutive keypoints touch (~20 KB at 16-cell strips) stay in L1 for all the CTAs resident on the SM
  const int nxb = max(1, min(8, SAMPLE_MAX_ROWS / Hm));
  const uint32_t xw = (uint32_t)((W + nxb - 1) / nxb);
  // divisions by W and by the strip width through 2^40 reciprocals (exact for lin * d < 2^40; the host checks H*W*W)
  auto bucket_of = [&](unsigned long long key) {
    const uint32_t lin = 0xffffffffu - (uint32_t)(key & 0xffffffffu);
    const uint32_t yy = (uint32_t)(((unsigned long long)lin * magic_w) >> 40), xx = lin - yy * (uint32_t)W;
    return min((int)((yy >> 3) * (uint32_t)nxb + (uint32_t)(((unsigned long long)xx * magic_xw) >> 40)), SAMPLE_MAX_ROWS - 1);
  };
  for (int i = tid; i < SAMPLE_MAX_ROWS; i += SAMPLE_THREADS) sHist[i] = 0;
  __syncthreads();
  for (int r = tid; r < nv; r += SAMPLE_THREADS) {
    const unsigned long long key = sorted[(int64_t)b * cap + r];
    sKey[r] = key;
    const int bk = bucket_of(key);
    sBkt[r] = (unsigned short)bk;
    atomicAdd(&sHist[bk], 1);
  }
  __syncthreads();
  if (tid < 32) {   // exclusive scan of the row histogram (<= 512 buckets) by one warp
    int carry = 0;
    for (int i0 = 0; i0 < SAMPLE_MAX_ROWS; i0 += 32) {
      const int v = sHist[i0 + tid];
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (tid >= o) inc += t;
      }
      sHist[i0 + tid] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  __syncthreads();
  for (int r = tid; r < nv; r += SAMPLE_THREADS) {
    const int pos = atomicAdd(&sHist[sBkt[r]], 1);
    sOrder[pos] = (unsigned short)r;
  }
  __syncthreads();
  // This CTA's share of the spatially ordered list.  The order INSIDE a row bucket depends on the atomics' arrival order and
  // differs between the CTAs of an image, so shares are cut at bucket ends (sHist[i] now holds the end offset of bucket i, a
  // function of the counts alone): share p = [first end >= p*nv/parts, first end >= (p+1)*nv/parts).
  __shared__ int sRange[2];
  if (tid < 32) {
    const int tl = (int)((int64_t)part * nv / nparts), th = (int)((int64_t)(part + 1) * nv / nparts);
    int ml = nv, mh = nv;
    for (int i = tid; i < SAMPLE_MAX_ROWS; i += 32) {
      const int e = sHist[i];
      if (e >= tl) ml = min(ml, e);
      if (e >= th) mh = min(mh, e);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ml = min(ml, __shfl_xor_sync(0xffffffffu, ml, o));
      mh = min(mh, __shfl_xor_sync(0xffffffffu, mh, o));
    }
    if (tid == 0) {
      sRange[0] = part == 0 ? 0 : ml;
      sRange[1] = part == nparts - 1 ? nv : mh;
    }
  }
  __syncthreads();
  const int lo = sRange[0], hi = sRange[1];
  const int l16 = tid & 15, grp = tid >> 4, ngrp = SAMPLE_THREADS / 16;
  const float* fb = feats + (int64_t)b * Hm * Wm * 64;
  const float* db = den + (int64_t)b * Hm * Wm;
  for (int i = lo + grp; i < lo + ((hi - lo + 1) & ~1); i += ngrp) {   // both half-warps of a warp iterate together (shuffles below)
    const bool valid = i < hi;
    const int r = valid ? (int)sOrder[i] : 0;
    const unsigned long long key = sKey[valid ? r : 0];
    const uint32_t lin = 0xffffffffu - (uint32_t)(key & 0xffffffffu);
    const int y = (int)(((unsigned long long)lin * magic_w) >> 40), x = (int)lin - y * W;
    float4 o = bicubic4<true>(fb, db, x, y, H, W, Hm, Wm, l16);   // (an odd tail's idle half-warp samples slot 0 again and drops it)
    if (!valid) o = make_float4(0.f, 0.f, 0.f, 0.f);
    float ss = sumsq4(o);
#pragma unroll
    for (int s = 8; s > 0; s >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, s);
    if (valid) {
      const int64_t slot = (int64_t)b * top_k + r;
      const float dn = __fdiv_rn(1.0f, fmaxf(sqrtf(ss), 1e-12f));  // F.normalize(feats, dim=-1), xfeat.py:93
      const float4 dv = make_float4(o.x * dn, o.y * dn, o.z * dn, o.w * dn);
      if (desc) reinterpret_cast<float4*>(desc + slot * 64)[l16] = dv;
      if (desc_split) store_desc_split(desc_split + ((int64_t)b * split_rows + r) * 128 + l16 * 4, dv);
      if (l16 == 0) {
        kpts[slot * 2] = __fmul_rn((float)x, rw);  // mkpts * [rw, rh], xfeat.py:96
        kpts[slot * 2 + 1] = __fmul_rn((float)y, rh);
        scores[slot] = ord2f((uint32_t)(key >> 32));
        if (kpts_int) { kpts_int[slot * 2] = x; kpts_int[slot * 2 + 1] = y; }
      }
    }
  }
  if (desc_split) {   // rows past n_valid up to the matcher's row padding are zero operands
    uint4* zp = reinterpret_cast<uint4*>(desc_split + ((int64_t)b * split_rows + nv) * 128);
    for (int64_t e = tid + (int64_t)part * SAMPLE_THREADS; e < (int64_t)(split_rows - nv) * 16; e += (int64_t)SAMPLE_THREADS * nparts)
      zp[e] = make_uint4(0u, 0u, 0u, 0u);
  }
  // zero-fill the slots past n_valid
  for (int64_t e = (int64_t)nv * 16 + tid + (int64_t)part * SAMPLE_THREADS; e < (int64_t)top_k * 16; e += (int64_t)SAMPLE_THREADS * nparts) {
    const int64_t slot = (int64_t)b * top_k + (e >> 4);
    if (desc) reinterpret_cast<float4*>(desc + slot * 64)[e & 15] = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((e & 15) == 0) {
      kpts[slot * 2] = 0.f; kpts[slot * 2 + 1] = 0.f; scores[slot] = 0.f;
      if (kpts_int) { kpts_int[slot * 2] = 0; kpts_int[slot * 2 + 1] = 0; }
    }
  }
}

static inline int sparse_cap(int H, int W) { return H * W / 4; }

struct SparseWs {
  unsigned long long *keys, *sorted;
  int *n_keep, *n_cand, *seg_begin, *seg_end;
  float* den;
  void* cub_temp;
  size_t cub_bytes;
};

static int carve_sparse(Bump& bump, int B, int H, int W, SparseWs& ws) {
  const int cap = sparse_cap(H, W);
  ws.keys = bump.take<unsigned long long>((size_t)B * cap);
  ws.sorted = bump.take<unsigned long long>((size_t)B * cap);
  ws.n_keep = bump.take<int>(B);
  ws.n_cand = bump.take<int>(B);
  ws.seg_begin = bump.take<int>(B);
  ws.seg_end = bump.take<int>(B);
  ws.den = bump.take<float>((size_t)B * (H / 8) * (W / 8));
  size_t tb = 0;
  cudaError_t e = cub::DeviceSegmentedSort::SortKeysDescending(nullptr, tb, (const unsigned long long*)nullptr,
                                                               (unsigned long long*)nullptr, B * cap, B, (const int*)nullptr,
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

extern "C" size_t xfeat_sparse_workspace_bytes(int B, int H, int W, int top_k) {
  (void)top_k;
  xf::Bump bump(nullptr, 0);
  xf::SparseWs ws;
  if (xf::carve_sparse(bump, B, H, W, ws) != XF_OK) return 0;
  return bump.used();
}

extern "C" int xfeat_detect_sparse(xfeat_ctx* ctx, const float* d_feats, const float* d_heat, const float* d_reliability,
                                   int B, int H, int W, int top_k, float threshold, float rw, float rh, float* d_kpts,
                                   float* d_scores, float* d_desc, int32_t* d_n_valid, int32_t* d_n_cand,
                                   int32_t* d_kpts_int, void* d_ws, size_t ws_bytes, void* stream) {
  return xfeat_detect_sparse_split(ctx, d_feats, d_heat, d_reliability, B, H, W, top_k, threshold, rw, rh, d_kpts, d_scores, d_desc,
                                   d_n_valid, d_n_cand, d_kpts_int, nullptr, 0, d_ws, ws_bytes, stream);
}

extern "C" int xfeat_detect_sparse_split(xfeat_ctx* ctx, const float* d_feats, const float* d_heat, const float* d_reliability,
                                         int B, int H, int W, int top_k, float threshold, float rw, float rh, float* d_kpts,
                                         float* d_scores, float* d_desc, int32_t* d_n_valid, int32_t* d_n_cand,
                                         int32_t* d_kpts_int, void* d_desc_split, int split_rows, void* d_ws, size_t ws_bytes,
                                         void* stream) {
  XF_REQUIRE(d_desc_split == nullptr || (split_rows >= top_k && split_rows % 512 == 0),
             "detect_sparse: split_rows must be a multiple of 512 and >= top_k (got %d)", split_rows);
  XF_REQUIRE(ctx && d_feats && d_heat && d_reliability && d_kpts && d_scores && (d_desc || d_desc_split) && d_n_valid && d_ws,
             "detect_sparse: null pointer");
  XF_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0 && H % 32 == 0 && W % 32 == 0 && top_k > 0,
             "detect_sparse: bad shape B=%d H=%d W=%d top_k=%d", B, H, W, top_k);
  XF_REQUIRE((int64_t)B * xf::sparse_cap(H, W) < (1ll << 31), "detect_sparse: batch too large for 32-bit offsets");
  // the NMS reads d_heat and the samplers read d_feats as float4, and store d_desc as float4 and d_desc_split as uint4
  XF_REQUIRE(((uintptr_t)d_heat | (uintptr_t)d_feats | (uintptr_t)d_desc | (uintptr_t)d_desc_split) % 16 == 0,
             "detect_sparse: d_heat, d_feats, d_desc and d_desc_split must be 16-byte aligned");
  XF_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  xf::Bump bump(d_ws, ws_bytes);
  xf::SparseWs ws;
  int rc = xf::carve_sparse(bump, B, H, W, ws);
  if (rc) return rc;
  if (!bump.ok) {
    xf::set_error("detect_sparse: workspace too small (%zu < %zu)", ws_bytes, bump.used());
    return XF_E_WORKSPACE;
  }
  const int cap = xf::sparse_cap(H, W), Hm = H / 8, Wm = W / 8;
  XF_CUDA(cudaMemsetAsync(ws.n_keep, 0, sizeof(int) * B, st));
  XF_CUDA(cudaMemsetAsync(ws.n_cand, 0, sizeof(int) * B, st));
  static const bool nms_tiled = getenv("XFEAT_NMS_TILED") != nullptr;   // A/B switch: the shared-memory tile kernel
  if (nms_tiled || (W & 3)) {
    dim3 grid(xf::cdiv(W, xf::NMS_TX), xf::cdiv(H, xf::NMS_TY), B);
    xf::nms_score_kernel<<<grid, 256, 0, st>>>(d_heat, d_reliability, H, W, Hm, Wm, threshold, cap, ws.keys, ws.n_keep,
                                               ws.n_cand);
  } else {
    dim3 grid(xf::cdiv(W, xf::NM_TW), xf::cdiv(H, xf::NM_WARPS * xf::NM_RS), B);
    xf::nms_march_kernel<<<grid, xf::NM_WARPS * 32, 0, st>>>(d_heat, d_reliability, H, W, Hm, Wm, threshold, cap, ws.keys,
                                                             ws.n_keep, ws.n_cand);
  }
  XF_LAUNCH_CHECK();
  static const bool force_cub = getenv("XFEAT_TOPK_CUB") != nullptr;   // A/B switch: the capacity-wide segmented sort
  if (!force_cub && top_k <= 8192) {
    if ((rc = xf::launch_topk_select_sort(ws.keys, ws.n_keep, 0, cap, top_k, B, ws.sorted, st))) return rc;
  } else {
    xf::segment_offsets_kernel<<<xf::cdiv(B, 128), 128, 0, st>>>(ws.n_keep, cap, B, ws.seg_begin, ws.seg_end);
    XF_LAUNCH_CHECK();
    size_t tb = ws.cub_bytes;
    XF_CUDA(cub::DeviceSegmentedSort::SortKeysDescending(ws.cub_temp, tb, ws.keys, ws.sorted, B * cap, B, ws.seg_begin,
                                                         ws.seg_end, st));
  }
  const int64_t npix = (int64_t)B * Hm * Wm;
  xf::feat_norm_kernel<<<(unsigned)((npix * 8 + 255) / 256), 256, 0, st>>>(d_feats, ws.den, npix);
  XF_LAUNCH_CHECK();
  // one-CTA-per-image spatially ordered variant: L1-friendly, measured 268 vs 330 us at B = 128 x 4096 keypoints; it
  // needs enough images to fill the GPU (XFEAT_SAMPLE_GENERIC=1 forces the generic kernel)
  static const bool force_generic = getenv("XFEAT_SAMPLE_GENERIC") != nullptr;
  if (!force_generic && B >= 32 && top_k <= xf::SAMPLE_MAX_K && Hm <= xf::SAMPLE_MAX_ROWS && (int64_t)H * W * W < (1ll << 40)) {
    const size_t smem = (size_t)top_k * (sizeof(unsigned long long) + 2 * sizeof(unsigned short));
    const int nxb = std::max(1, std::min(8, xf::SAMPLE_MAX_ROWS / Hm));
    const unsigned xw = (unsigned)((W + nxb - 1) / nxb);
    const unsigned long long magic_w = (1ull << 40) / (unsigned)W + 1, magic_xw = (1ull << 40) / xw + 1;
    XF_DYN_SMEM(xf::sample_desc_sorted_kernel, smem);
    const int parts = std::max(1, std::min(xf::SAMPLE_PARTS, top_k / 512));
    xf::sample_desc_sorted_kernel<<<dim3(B, parts), xf::SAMPLE_THREADS, smem, st>>>(ws.sorted, ws.n_keep, d_feats, ws.den, H, W, Hm, Wm, cap,
                                                                      top_k, rw, rh, d_kpts, d_scores, d_desc, d_n_valid,
                                                                      d_kpts_int, (__half*)d_desc_split, split_rows, magic_w, magic_xw);
  } else {
    const int64_t slots = (int64_t)B * top_k;
    if (d_desc_split && split_rows > top_k)   // this kernel only visits the top_k slots: the matcher's padding rows are cleared here
      XF_CUDA(cudaMemsetAsync(d_desc_split, 0, (size_t)B * split_rows * 128 * sizeof(__half), st));
    xf::sample_desc_kernel<<<(unsigned)((slots * 16 + 255) / 256), 256, 0, st>>>(
        ws.sorted, ws.n_keep, d_feats, ws.den, B, H, W, Hm, Wm, cap, top_k, rw, rh, d_kpts, d_scores, d_desc, d_n_valid,
        d_kpts_int, (__half*)d_desc_split, split_rows);
  }
  XF_LAUNCH_CHECK();
  if (d_n_cand) XF_CUDA(cudaMemcpyAsync(d_n_cand, ws.n_cand, sizeof(int) * B, cudaMemcpyDeviceToDevice, st));
  return XF_OK;
}
