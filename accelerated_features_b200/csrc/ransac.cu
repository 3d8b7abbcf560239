// Geometric verification of the matches, on the GPU, for a whole batch of pairs at once (SURVEY 8f-3).  Every caller of the
// reference runs a robust estimator right after the path: cv2.findHomography(pts1, pts2, cv2.USAC_MAGSAC, thr, maxIters=700,
// confidence=0.995) in realtime_demo.py:225 and the notebooks, poselib.estimate_relative_pose in the 1500-pair benchmarks
// (modules/eval/megadepth1500.py:98-113).  Both algorithms live in un-vendored third-party packages (opencv-contrib 4.10.0.84
// is pinned in requirements.txt; poselib is not pinned), so what is restated here is the published scheme they share:
//   hypothesise from minimal samples -> score every hypothesis on all correspondences -> keep the best -> re-fit on its
//   inliers (local optimisation) -> classify with the threshold,
// with MSAC scoring (truncated squared error).  Parity is anchored on the call sites: same inputs, same threshold meaning
// (pixels of the second image for the homography, Sampson distance in normalised image coordinates for the essential matrix,
// Sampson distance in pixels for the fundamental matrix as in OpenCV's USAC methods);
// tests compare inlier sets and model error with cv2 on the same correspondences (stochastic: agreement, not bit equality).
//
// The three estimators share one set of device steps: a block caches its pair's correspondences in shared memory, draws
// minimal samples from a hash of (seed, pair id, hypothesis id) (rs_draw), scores hypotheses with MSAC by warp and writes its
// best record (rs_block_best); a later launch picks the pair's best record (rs_pair_best) and classifies.  The homography runs
// in two launches: a warp owns one 4-point hypothesis (lane 0 solves, fp64), and the final launch re-fits the pair's winner by
// least squares on its inliers twice (normal equations in fp64, smallest eigenvector by cyclic Jacobi) before it classifies.
// The essential and fundamental matrices run in three launches from one set of kernel templates over a model struct
// (RsEssential, RsFundamental): every lane solves a sample, every block's winner is locally optimised (rs_local_opt), and the
// final launch classifies.  Nothing returns to the host.
#include "common.cuh"

namespace xf {

constexpr int RS_THREADS = 256, RS_WARPS = RS_THREADS / 32;
constexpr int RS_E_REFITS = 8;         // local-optimisation rounds of every block's epipolar winner (rs_local_opt)
constexpr int RS_MAX_PTS = 8192;       // correspondences per pair cached in shared memory (4 floats each)
constexpr float RS_NO_COST = 3.0e38f;  // cost of a record that holds no hypothesis

__device__ __forceinline__ uint32_t rs_hash(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// Hartley normalisation of one point set: centroid to the origin, mean distance sqrt(2).  Returns (cx, cy, s).
struct RsNorm { float cx, cy, s; };

__device__ RsNorm rs_normaliser(const float* __restrict__ p, int n) {
  __shared__ float red[3 * RS_WARPS];
  float sx = 0.f, sy = 0.f;
  for (int i = threadIdx.x; i < n; i += RS_THREADS) { sx += p[2 * i]; sy += p[2 * i + 1]; }
  for (int o = 16; o > 0; o >>= 1) { sx += __shfl_xor_sync(0xffffffffu, sx, o); sy += __shfl_xor_sync(0xffffffffu, sy, o); }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[w] = sx; red[RS_WARPS + w] = sy; }
  __syncthreads();
  float cx = 0.f, cy = 0.f;
  for (int i = 0; i < RS_WARPS; ++i) { cx += red[i]; cy += red[RS_WARPS + i]; }
  cx /= (float)max(n, 1); cy /= (float)max(n, 1);
  __syncthreads();
  float sd = 0.f;
  for (int i = threadIdx.x; i < n; i += RS_THREADS) { const float dx = p[2 * i] - cx, dy = p[2 * i + 1] - cy; sd += sqrtf(dx * dx + dy * dy); }
  for (int o = 16; o > 0; o >>= 1) sd += __shfl_xor_sync(0xffffffffu, sd, o);
  if (l == 0) red[2 * RS_WARPS + w] = sd;
  __syncthreads();
  float md = 0.f;
  for (int i = 0; i < RS_WARPS; ++i) md += red[2 * RS_WARPS + i];
  md /= (float)max(n, 1);
  __syncthreads();
  RsNorm r;
  r.cx = cx; r.cy = cy; r.s = (md > 1e-12f) ? 1.41421356f / md : 1.f;
  return r;
}

// Solve the 8x8 system of a 4-point homography (h22 = 1) by Gaussian elimination with partial pivoting (fp64).
__device__ bool rs_solve_h4(const float (&x)[4], const float (&y)[4], const float (&u)[4], const float (&v)[4], double (&h)[9]) {
  double A[8][9];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double X = x[i], Y = y[i], U = u[i], V = v[i];
    double* r0 = A[2 * i]; double* r1 = A[2 * i + 1];
    r0[0] = X; r0[1] = Y; r0[2] = 1; r0[3] = 0; r0[4] = 0; r0[5] = 0; r0[6] = -U * X; r0[7] = -U * Y; r0[8] = U;
    r1[0] = 0; r1[1] = 0; r1[2] = 0; r1[3] = X; r1[4] = Y; r1[5] = 1; r1[6] = -V * X; r1[7] = -V * Y; r1[8] = V;
  }
  for (int c = 0; c < 8; ++c) {
    int piv = c;
    double best = fabs(A[c][c]);
    for (int r = c + 1; r < 8; ++r)
      if (fabs(A[r][c]) > best) { best = fabs(A[r][c]); piv = r; }
    if (best < 1e-10) return false;                       // degenerate sample (three points on a line, repeated point)
    if (piv != c)
      for (int k = c; k < 9; ++k) { const double t = A[c][k]; A[c][k] = A[piv][k]; A[piv][k] = t; }
    const double inv = 1.0 / A[c][c];
    for (int r = c + 1; r < 8; ++r) {
      const double f = A[r][c] * inv;
      for (int k = c; k < 9; ++k) A[r][k] -= f * A[c][k];
    }
  }
  for (int c = 7; c >= 0; --c) {
    double s = A[c][8];
    for (int k = c + 1; k < 8; ++k) s -= A[c][k] * h[k];
    h[c] = s / A[c][c];
  }
  h[8] = 1.0;
  return true;
}

// Eigen-decomposition of a symmetric N x N matrix (cyclic Jacobi, fp64): M is diagonalised in place (eigenvalue i on M[i][i]),
// the eigenvectors are the columns of V.
template <int N>
__device__ __forceinline__ void rs_jacobi(double (&M)[N][N], double (&V)[N][N]) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int i = 0; i < N; ++i)
      for (int j = i + 1; j < N; ++j) off += M[i][j] * M[i][j];
    if (off < 1e-30) break;
    for (int p = 0; p < N; ++p)
      for (int q = p + 1; q < N; ++q) {
        if (fabs(M[p][q]) < 1e-300) continue;
        const double theta = (M[q][q] - M[p][p]) / (2.0 * M[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {
          const double mkp = M[k][p], mkq = M[k][q];
          M[k][p] = c * mkp - s * mkq;
          M[k][q] = s * mkp + c * mkq;
        }
        for (int k = 0; k < N; ++k) {
          const double mpk = M[p][k], mqk = M[q][k];
          M[p][k] = c * mpk - s * mqk;
          M[q][k] = s * mpk + c * mqk;
        }
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
}

// Smallest-eigenvalue eigenvector of a symmetric N x N matrix (cyclic Jacobi, fp64); M is destroyed.
template <int N>
__device__ void rs_smallest_eigvec(double (&M)[N][N], double (&vec)[N]) {
  double V[N][N];
  rs_jacobi<N>(M, V);
  int best = 0;
  for (int i = 1; i < N; ++i)
    if (M[i][i] < M[best][best]) best = i;
  for (int k = 0; k < N; ++k) vec[k] = V[k][best];
}

// ---------------------------------------------------------------------------------------------------------------------
// Steps shared by the estimators.  Hypotheses go to per-block records in the workspace: [batch][blocks_per_pair] of
// (MSAC cost, 9 model floats); a block that found no hypothesis leaves cost RS_NO_COST.
// ---------------------------------------------------------------------------------------------------------------------
struct RsRecord {
  float cost;
  float m[9];
};

// K distinct indices in [0, n) for hypothesis `hid` of pair `pid`: a hash of (seed, pid, hid), redrawn on a repeat.
template <int K>
__device__ __forceinline__ void rs_draw(uint32_t seed, uint32_t pid, uint32_t hid, int n, int (&idx)[K]) {
  uint32_t s = rs_hash(seed ^ (0x9e3779b9u * (pid + 1)) ^ (0x85ebca6bu * (hid + 1)));
  for (int k = 0; k < K; ++k) {
    bool dup;
    do {
      s = rs_hash(s + 0x6d2b79f5u);
      idx[k] = (int)(((uint64_t)s * (uint64_t)n) >> 32);
      dup = false;
      for (int j = 0; j < k; ++j) dup |= (idx[j] == idx[k]);
    } while (dup);
  }
}

// Every warp's best record (warp-uniform `mine`) to the block's best, lowest warp on ties, written by thread 0 to the block's
// record of a (blocks_per_pair, batch) grid.
__device__ __forceinline__ void rs_block_best(const RsRecord& mine, RsRecord* __restrict__ best) {
  __shared__ RsRecord sBest[RS_WARPS];
  if ((threadIdx.x & 31) == 0) sBest[threadIdx.x >> 5] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    RsRecord b = sBest[0];
    for (int w = 1; w < RS_WARPS; ++w)
      if (sBest[w].cost < b.cost) b = sBest[w];
    best[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = b;
  }
}

// The pair's best record over its blocks, lowest block on ties.
__device__ __forceinline__ RsRecord rs_pair_best(const RsRecord* __restrict__ best, int pair, int blocks_per_pair) {
  RsRecord b = best[(int64_t)pair * blocks_per_pair];
  for (int k = 1; k < blocks_per_pair; ++k) {
    const RsRecord c = best[(int64_t)pair * blocks_per_pair + k];
    if (c.cost < b.cost) b = c;
  }
  return b;
}

// A pair without a model (its mask already cleared): `diag` on the model's diagonal (1: identity H, 0: zero E / F) and no
// inliers; a negative count (XF_N_OVERFLOW) passes through.
__device__ __forceinline__ void rs_write_none(int n_all, float diag, float* __restrict__ m_out, int* __restrict__ n_inl) {
  *n_inl = n_all < 0 ? n_all : 0;
  for (int k = 0; k < 9; ++k) m_out[k] = (k % 4 == 0) ? diag : 0.f;
}

// Block-wide sum of one count per thread, returned to every thread.  Two calls need a barrier between them.
__device__ __forceinline__ int rs_block_count(int cnt) {
  __shared__ int sCnt;
  if (threadIdx.x == 0) sCnt = 0;
  __syncthreads();
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&sCnt, cnt);
  __syncthreads();
  return sCnt;
}

// The block's 9 x 9 normal matrix from every thread's upper-triangle terms acc (45, row-major) and row count cnt: each warp's
// sum, then the warps in order.  Returns the block's row count to every thread; thread 0 gets M when it is >= min_rows.
__device__ __forceinline__ int rs_block_normal_matrix(const double (&acc)[45], int cnt, int min_rows, double (&M)[9][9]) {
  __shared__ double sAcc[RS_WARPS][45];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 45; ++k) {
    double v = acc[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sAcc[warp][k] = v;
  }
  const int total = rs_block_count(cnt);
  if (threadIdx.x == 0 && total >= min_rows) {
    int e = 0;
    for (int a = 0; a < 9; ++a)
      for (int b2 = a; b2 < 9; ++b2) {
        double v = 0.0;
        for (int w = 0; w < RS_WARPS; ++w) v += sAcc[w][e];
        M[a][b2] = v; M[b2][a] = v;
        ++e;
      }
  }
  return total;
}

// ---------------------------------------------------------------------------------------------------------------------
// Homography.  Both launches Hartley-normalise each image of the pair; the threshold is image 1's pixel threshold in its
// normalised frame.
// ---------------------------------------------------------------------------------------------------------------------

// squared forward transfer error of a homography (normalised coordinates); invalid (point at infinity) -> huge
__device__ __forceinline__ float rs_h_err2(const float (&h)[9], float x, float y, float u, float v) {
  const float w = h[6] * x + h[7] * y + h[8];
  if (fabsf(w) < 1e-8f) return 1e30f;
  const float iw = 1.0f / w;
  const float du = (h[0] * x + h[1] * y + h[2]) * iw - u, dv = (h[3] * x + h[4] * y + h[5]) * iw - v;
  return du * du + dv * dv;
}

// The pair's normalised (x, y, u, v) into sPts, visible to the block on return, and the two normalisers.
__device__ __forceinline__ void rs_h_load(const float* __restrict__ q0, const float* __restrict__ q1, int n, float4* sPts,
                                          RsNorm& n0, RsNorm& n1) {
  n0 = rs_normaliser(q0, n);
  n1 = rs_normaliser(q1, n);
  for (int i = threadIdx.x; i < n; i += RS_THREADS)
    sPts[i] = make_float4((q0[2 * i] - n0.cx) * n0.s, (q0[2 * i + 1] - n0.cy) * n0.s, (q1[2 * i] - n1.cx) * n1.s,
                          (q1[2 * i + 1] - n1.cy) * n1.s);
  __syncthreads();
}

// stage 1: grid (blocks_per_pair, batch); every warp scores `hyp_per_warp` hypotheses and keeps its best.
__global__ void __launch_bounds__(RS_THREADS) ransac_h_hyp_kernel(const float* __restrict__ p0, const float* __restrict__ p1,
                                                                  const int* __restrict__ np, int n_max, float thr,
                                                                  int hyp_per_warp, uint32_t seed, RsRecord* __restrict__ best) {
  extern __shared__ float4 sPts[];                 // (x, y, u, v) normalised
  const int pair = blockIdx.y;
  const int n = min(np ? np[pair] : n_max, min(n_max, RS_MAX_PTS));
  RsRecord mine;
  mine.cost = RS_NO_COST;
#pragma unroll
  for (int k = 0; k < 9; ++k) mine.m[k] = (k % 4 == 0) ? 1.f : 0.f;
  if (n >= 4) {
    RsNorm n0, n1;
    rs_h_load(p0 + (int64_t)pair * n_max * 2, p1 + (int64_t)pair * n_max * 2, n, sPts, n0, n1);
    const float t2 = (thr * n1.s) * (thr * n1.s);  // pixel threshold of image 1 in its normalised frame
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int it = 0; it < hyp_per_warp; ++it) {
      const uint32_t hid = (uint32_t)((blockIdx.x * RS_WARPS + warp) * hyp_per_warp + it);
      float h[9];
      int ok = 0;
      if (lane == 0) {
        int idx[4];
        rs_draw<4>(seed, (uint32_t)pair, hid, n, idx);
        float x[4], y[4], u[4], v[4];
        for (int k = 0; k < 4; ++k) { const float4 c = sPts[idx[k]]; x[k] = c.x; y[k] = c.y; u[k] = c.z; v[k] = c.w; }
        double hd[9];
        ok = rs_solve_h4(x, y, u, v, hd) ? 1 : 0;
        if (ok)
          for (int k = 0; k < 9; ++k) h[k] = (float)hd[k];
      }
      ok = __shfl_sync(0xffffffffu, ok, 0);
      if (!ok) continue;
#pragma unroll
      for (int k = 0; k < 9; ++k) h[k] = __shfl_sync(0xffffffffu, h[k], 0);
      float cost = 0.f;
      for (int i = lane; i < n; i += 32) {
        const float4 c = sPts[i];
        cost += fminf(rs_h_err2(h, c.x, c.y, c.z, c.w), t2);      // MSAC
      }
      for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
      if (cost < mine.cost) {
        mine.cost = cost;
#pragma unroll
        for (int k = 0; k < 9; ++k) mine.m[k] = h[k];
      }
    }
    rs_block_best(mine, best);
  } else if (threadIdx.x == 0) {   // the empty record; calling rs_block_best on this path too costs the kernel 16 spill bytes
    best[(int64_t)pair * gridDim.x + blockIdx.x] = mine;
  }
}

// stage 2: one block per pair: best hypothesis -> two rounds of least-squares re-fit on its inliers -> model, mask, count
__global__ void __launch_bounds__(RS_THREADS) ransac_h_final_kernel(const float* __restrict__ p0, const float* __restrict__ p1,
                                                                    const int* __restrict__ np, int n_max, float thr,
                                                                    const RsRecord* __restrict__ best, int blocks_per_pair,
                                                                    float* __restrict__ H_out, unsigned char* __restrict__ mask,
                                                                    int* __restrict__ n_inl) {
  extern __shared__ float4 sPts[];
  __shared__ float sH[9];
  __shared__ int sFound;
  const int pair = blockIdx.x;
  const int n_all = np ? np[pair] : n_max;
  const int n = min(n_all, min(n_max, RS_MAX_PTS));
  unsigned char* mk = mask + (int64_t)pair * n_max;
  for (int i = threadIdx.x; i < n_max; i += RS_THREADS) mk[i] = 0;
  if (n < 4) {
    if (threadIdx.x == 0) rs_write_none(n_all, 1.f, H_out + pair * 9, n_inl + pair);
    return;
  }
  RsNorm n0, n1;
  rs_h_load(p0 + (int64_t)pair * n_max * 2, p1 + (int64_t)pair * n_max * 2, n, sPts, n0, n1);
  if (threadIdx.x == 0) {
    const RsRecord b = rs_pair_best(best, pair, blocks_per_pair);
    for (int k = 0; k < 9; ++k) sH[k] = b.m[k];
    sFound = b.cost < RS_NO_COST;
  }
  __syncthreads();
  if (!sFound) {          // every 4-point sample was degenerate (identical or collinear points): no model, as for n < 4
    if (threadIdx.x == 0) rs_write_none(n_all, 1.f, H_out + pair * 9, n_inl + pair);
    return;
  }
  const float t2 = (thr * n1.s) * (thr * n1.s);
  for (int round = 0; round < 2; ++round) {
    // normal equations of the DLT rows of the current inliers: A^T A (9 x 9 symmetric, 45 entries)
    float h[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) h[k] = sH[k];
    double acc[45];
#pragma unroll
    for (int k = 0; k < 45; ++k) acc[k] = 0.0;
    int cnt = 0;
    for (int i = threadIdx.x; i < n; i += RS_THREADS) {
      const float4 c = sPts[i];
      if (rs_h_err2(h, c.x, c.y, c.z, c.w) < t2) {
        ++cnt;
        const double r0[9] = {c.x, c.y, 1.0, 0, 0, 0, -(double)c.z * c.x, -(double)c.z * c.y, -(double)c.z};
        const double r1[9] = {0, 0, 0, c.x, c.y, 1.0, -(double)c.w * c.x, -(double)c.w * c.y, -(double)c.w};
        int e = 0;
#pragma unroll
        for (int a = 0; a < 9; ++a)
#pragma unroll
          for (int b2 = a; b2 < 9; ++b2) acc[e++] += r0[a] * r0[b2] + r1[a] * r1[b2];
      }
    }
    double M[9][9], vec[9];
    if (rs_block_normal_matrix(acc, cnt, 4, M) >= 4 && threadIdx.x == 0) {
      rs_smallest_eigvec<9>(M, vec);
      if (fabs(vec[8]) > 1e-12)
        for (int k = 0; k < 9; ++k) sH[k] = (float)(vec[k] / vec[8]);
    }
    __syncthreads();
  }
  // final classification + de-normalisation  H = T1^-1 Hn T0
  float h[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) h[k] = sH[k];
  int cnt = 0;
  for (int i = threadIdx.x; i < n; i += RS_THREADS) {
    const float4 c = sPts[i];
    const bool in = rs_h_err2(h, c.x, c.y, c.z, c.w) < t2;
    mk[i] = in ? 1 : 0;
    cnt += in ? 1 : 0;
  }
  cnt = rs_block_count(cnt);
  if (threadIdx.x == 0) {
    n_inl[pair] = cnt;
    // T0 = [s0 0 -s0 cx0; 0 s0 -s0 cy0; 0 0 1],  T1^-1 = [1/s1 0 cx1; 0 1/s1 cy1; 0 0 1]
    double Hn[3][3], T0[3][3] = {{n0.s, 0, -n0.s * n0.cx}, {0, n0.s, -n0.s * n0.cy}, {0, 0, 1}};
    double T1i[3][3] = {{1.0 / n1.s, 0, n1.cx}, {0, 1.0 / n1.s, n1.cy}, {0, 0, 1}};
    for (int a = 0; a < 3; ++a)
      for (int b2 = 0; b2 < 3; ++b2) Hn[a][b2] = h[3 * a + b2];
    double tmp[3][3], Hf[3][3];
    for (int a = 0; a < 3; ++a)
      for (int b2 = 0; b2 < 3; ++b2) { double s = 0; for (int k = 0; k < 3; ++k) s += Hn[a][k] * T0[k][b2]; tmp[a][b2] = s; }
    for (int a = 0; a < 3; ++a)
      for (int b2 = 0; b2 < 3; ++b2) { double s = 0; for (int k = 0; k < 3; ++k) s += T1i[a][k] * tmp[k][b2]; Hf[a][b2] = s; }
    const double sc = fabs(Hf[2][2]) > 1e-12 ? 1.0 / Hf[2][2] : 1.0;
    for (int a = 0; a < 3; ++a)
      for (int b2 = 0; b2 < 3; ++b2) H_out[pair * 9 + 3 * a + b2] = (float)(Hf[a][b2] * sc);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Epipolar models: x1^T E x0 = 0, scored with the Sampson distance.
//
// Essential matrix (calibrated relative pose; the estimator the 1500-pair benchmarks call through poselib,
// modules/eval/megadepth1500.py:98-113).  Inputs are NORMALISED image coordinates (K^-1 applied by the caller); the minimal
// solver is the normalised 8-point algorithm projected onto the essential manifold (singular values (1,1,0)).  (poselib uses
// the 5-point solver, which also handles planar scenes; the 8-point form does not -- see DESIGN.md.)
//
// Fundamental matrix (uncalibrated two-view geometry; what cv2.findFundamentalMat(p0, p1, cv2.USAC_*, thr) computes).  Inputs
// are PIXELS, normalised per pair (rs_pair_normalise); the minimal solver is the 7-point algorithm (1-3 candidates).  thr is the
// USAC meaning: Sampson distance in pixels (OpenCV 4.13's USAC_DEFAULT / USAC_ACCURATE / USAC_MAGSAC masks are exactly
// `Sampson < thr`), and the final classification evaluates it in fp64 under the returned pixel F.
// ---------------------------------------------------------------------------------------------------------------------

// E = U diag(s) V^T projected onto s = (1,1,0): E' = u1 v1^T + u2 v2^T, with (v1, v2) the two leading right singular vectors
// (eigenvectors of E^T E) and u_i = E v_i / |E v_i|.
__device__ void rs_project_essential(double (&E)[9]) {
  double M[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i][j] = E[0 + i] * E[0 + j] + E[3 + i] * E[3 + j] + E[6 + i] * E[6 + j];
  rs_jacobi<3>(M, V);
  int lo = 0;                                   // column of the smallest eigenvalue: dropped
  for (int i = 1; i < 3; ++i)
    if (M[i][i] < M[lo][lo]) lo = i;
  double out[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int c = 0; c < 3; ++c) {
    if (c == lo) continue;
    double u[3];
    for (int r = 0; r < 3; ++r) u[r] = E[3 * r] * V[0][c] + E[3 * r + 1] * V[1][c] + E[3 * r + 2] * V[2][c];
    const double nrm = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
    if (nrm < 1e-300) continue;
    for (int r = 0; r < 3; ++r)
      for (int k = 0; k < 3; ++k) out[3 * r + k] += (u[r] / nrm) * V[k][c];
  }
  for (int k = 0; k < 9; ++k) E[k] = out[k];
}

// Nearest rank-2 matrix in the Frobenius norm: F - (F v) v^T with v the right singular vector of the smallest singular value
// (the eigenvector of F^T F of its smallest eigenvalue).
__device__ void rs_project_rank2(double (&F)[9]) {
  double M[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i][j] = F[0 + i] * F[0 + j] + F[3 + i] * F[3 + j] + F[6 + i] * F[6 + j];
  rs_jacobi<3>(M, V);
  int lo = 0;
  for (int i = 1; i < 3; ++i)
    if (M[i][i] < M[lo][lo]) lo = i;
  for (int r = 0; r < 3; ++r) {
    const double w = F[3 * r] * V[0][lo] + F[3 * r + 1] * V[1][lo] + F[3 * r + 2] * V[2][lo];
    for (int k = 0; k < 3; ++k) F[3 * r + k] -= w * V[k][lo];
  }
}

// squared Sampson distance of (x,y) <-> (u,v) under x1^T E x0 = 0
__device__ __forceinline__ float rs_sampson2(const float (&E)[9], float x, float y, float u, float v) {
  const float a = E[0] * x + E[1] * y + E[2], b = E[3] * x + E[4] * y + E[5], c = E[6] * x + E[7] * y + E[8];
  const float d = E[0] * u + E[3] * v + E[6], f = E[1] * u + E[4] * v + E[7];
  const float e = u * a + v * b + c;
  const float den = a * a + b * b + d * d + f * f;
  return den > 1e-20f ? e * e / den : 1e30f;
}

// Squared Sampson distance in pixels under the float32 pixel F, evaluated in fp64.  Far from the origin x1^T F x0 is the
// cancellation of terms many orders larger than itself: at coordinates near (7000, 5000), rs_sampson2's float32 evaluation is
// off by up to 0.17 px, so the mask would not be `Sampson < thr` under the returned F.
__device__ __forceinline__ double rs_sampson2_px(const float (&F)[9], double x, double y, double u, double v) {
  const double a = F[0] * x + F[1] * y + F[2], b = F[3] * x + F[4] * y + F[5], c = F[6] * x + F[7] * y + F[8];
  const double d = F[0] * u + F[3] * v + F[6], f = F[1] * u + F[4] * v + F[7];
  const double e = u * a + v * b + c;
  const double den = a * a + b * b + d * d + f * f;
  return den > 1e-300 ? e * e / den : 1e300;
}

__device__ __forceinline__ void rs_epi_row(float x, float y, float u, float v, double (&r)[9]) {
  r[0] = (double)u * x; r[1] = (double)u * y; r[2] = u; r[3] = (double)v * x; r[4] = (double)v * y; r[5] = v; r[6] = x; r[7] = y; r[8] = 1.0;
}

// 9 x 9 normal matrix of the K epipolar rows of pts[idx[0..K-1]] (normalised (x, y, u, v)), fp64.
template <int K>
__device__ __forceinline__ void rs_epi_normal(const float4* pts, const int (&idx)[K], double (&M)[9][9]) {
  for (int a = 0; a < 9; ++a)
    for (int b2 = 0; b2 < 9; ++b2) M[a][b2] = 0.0;
  for (int k = 0; k < K; ++k) {
    const float4 c = pts[idx[k]];
    double r[9];
    rs_epi_row(c.x, c.y, c.z, c.w, r);
    for (int a = 0; a < 9; ++a)
      for (int b2 = a; b2 < 9; ++b2) M[a][b2] += r[a] * r[b2];
  }
  for (int a = 0; a < 9; ++a)
    for (int b2 = 0; b2 < a; ++b2) M[a][b2] = M[b2][a];
}

// Normalisation of one pair: each image's centroid to the origin and ONE scale s for both images (mean distance sqrt(2) over
// all 2n points).  With one scale, the Sampson distance of the normalised points is exactly s times the pixel one, so the pixel
// threshold thr is thr * s in the normalised frame.  Writes the normalised (x, y, u, v) to sPts, visible to the block on return.
struct RsPairNorm { float cx0, cy0, cx1, cy1, s; };

__device__ RsPairNorm rs_pair_normalise(const float* __restrict__ q0, const float* __restrict__ q1, int n, float4* sPts) {
  __shared__ float red[4 * RS_WARPS];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  float a[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = threadIdx.x; i < n; i += RS_THREADS) { a[0] += q0[2 * i]; a[1] += q0[2 * i + 1]; a[2] += q1[2 * i]; a[3] += q1[2 * i + 1]; }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    if (l == 0) red[k * RS_WARPS + w] = a[k];
  }
  __syncthreads();
  float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    for (int i = 0; i < RS_WARPS; ++i) c[k] += red[k * RS_WARPS + i];
    c[k] /= (float)n;
  }
  __syncthreads();
  float sd = 0.f;
  for (int i = threadIdx.x; i < n; i += RS_THREADS) {
    const float dx0 = q0[2 * i] - c[0], dy0 = q0[2 * i + 1] - c[1], dx1 = q1[2 * i] - c[2], dy1 = q1[2 * i + 1] - c[3];
    sd += sqrtf(dx0 * dx0 + dy0 * dy0) + sqrtf(dx1 * dx1 + dy1 * dy1);
  }
  for (int o = 16; o > 0; o >>= 1) sd += __shfl_xor_sync(0xffffffffu, sd, o);
  if (l == 0) red[w] = sd;
  __syncthreads();
  float md = 0.f;
  for (int i = 0; i < RS_WARPS; ++i) md += red[i];
  md /= (float)(2 * n);
  const float s = (md > 1e-12f) ? 1.41421356f / md : 1.f;
  for (int i = threadIdx.x; i < n; i += RS_THREADS)
    sPts[i] = make_float4((q0[2 * i] - c[0]) * s, (q0[2 * i + 1] - c[1]) * s, (q1[2 * i] - c[2]) * s, (q1[2 * i + 1] - c[3]) * s);
  __syncthreads();
  return RsPairNorm{c[0], c[1], c[2], c[3], s};
}

__device__ __forceinline__ double rs_det3(const double (&F)[9]) {
  return F[0] * (F[4] * F[8] - F[5] * F[7]) - F[1] * (F[3] * F[8] - F[5] * F[6]) + F[2] * (F[3] * F[7] - F[4] * F[6]);
}

// The 7-point solver.  (F1, F2) span the null space of the sample's seven epipolar rows; F = l F1 + (1 - l) F2 with det F = 0 is
// a cubic in l, whose coefficients come from det F at l = 0, 1, -1, 2.  Each real root (Newton-polished) gives one candidate,
// scaled to unit Frobenius norm.  Returns the number of candidates (0 for a degenerate sample) written to Fc.
__device__ int rs_seven_point(const double (&F1)[9], const double (&F2)[9], float (&Fc)[3][9]) {
  double G[9], p[4];
  const double at[4] = {0.0, 1.0, -1.0, 2.0};
  for (int j = 0; j < 4; ++j) {
    for (int k = 0; k < 9; ++k) G[k] = at[j] * F1[k] + (1.0 - at[j]) * F2[k];
    p[j] = rs_det3(G);
  }
  const double c0 = p[0], c2 = 0.5 * (p[1] + p[2]) - p[0], odd = 0.5 * (p[1] - p[2]);
  const double c3 = (p[3] - 4.0 * c2 - c0 - 2.0 * odd) / 6.0, c1 = odd - c3;
  const double cm = fmax(fmax(fabs(c0), fabs(c1)), fmax(fabs(c2), fabs(c3)));
  if (!(cm > 1e-300)) return 0;
  double r[3];
  int nr = 0;
  if (fabs(c3) > 1e-10 * cm) {                      // l^3 + A l^2 + B l + C; l = t - A/3: t^3 + pp t + qq = 0
    const double A = c2 / c3, B = c1 / c3, C = c0 / c3;
    const double pp = B - A * A / 3.0, qq = 2.0 * A * A * A / 27.0 - A * B / 3.0 + C;
    const double D = 0.25 * qq * qq + pp * pp * pp / 27.0;
    if (D > 0.0) {
      const double sD = sqrt(D);
      r[nr++] = cbrt(-0.5 * qq + sD) + cbrt(-0.5 * qq - sD) - A / 3.0;
    } else if (pp < 0.0) {
      const double m = 2.0 * sqrt(-pp / 3.0);
      const double th = acos(fmin(1.0, fmax(-1.0, 3.0 * qq / (pp * m)))) / 3.0;
      for (int k = 0; k < 3; ++k) r[nr++] = m * cos(th - 2.0943951023931957 * k) - A / 3.0;
    } else {
      r[nr++] = -A / 3.0;
    }
  } else if (fabs(c2) > 1e-10 * cm) {               // the cubic term vanishes: the third root is at infinity (F1 - F2)
    const double disc = c1 * c1 - 4.0 * c2 * c0;
    if (disc >= 0.0) {
      const double qd = -0.5 * (c1 + (c1 >= 0.0 ? sqrt(disc) : -sqrt(disc)));
      r[nr++] = qd / c2;
      if (qd != 0.0) r[nr++] = c0 / qd;
    }
  } else if (fabs(c1) > 1e-10 * cm) {
    r[nr++] = -c0 / c1;
  }
  int nc = 0;
  for (int j = 0; j < nr; ++j) {
    double l = r[j];
    for (int it = 0; it < 2; ++it) {
      const double f = ((c3 * l + c2) * l + c1) * l + c0, df = (3.0 * c3 * l + 2.0 * c2) * l + c1;
      if (fabs(df) > 1e-300) l -= f / df;
    }
    double nrm = 0.0;
    for (int k = 0; k < 9; ++k) { G[k] = l * F1[k] + (1.0 - l) * F2[k]; nrm += G[k] * G[k]; }
    if (!(nrm > 1e-300) || !isfinite(nrm)) continue;
    const double inv = 1.0 / sqrt(nrm);
    for (int k = 0; k < 9; ++k) Fc[nc][k] = (float)(G[k] * inv);
    ++nc;
  }
  return nc;
}

// One 7-point sample, the body of a fundamental-matrix hypothesis lane: the 9 x 9 normal matrix of the seven epipolar rows of
// pts[idx[0..6]] (normalised (x, y, u, v)), its two smallest eigenvectors (cyclic Jacobi) as the null space, and the 1-3
// candidates of rs_seven_point.  Also run on its own by xfeat_debug_seven_point.
__device__ __forceinline__ int rs_f_sample(const float4* pts, const int (&idx)[7], float (&Fc)[3][9]) {
  double M[9][9];
  rs_epi_normal<7>(pts, idx, M);
  double V[9][9];
  rs_jacobi<9>(M, V);
  int i1 = 0, i2 = 1;                           // the two smallest eigenvalues: the null space of the 7 x 9 system
  if (M[i2][i2] < M[i1][i1]) { i1 = 1; i2 = 0; }
  for (int i = 2; i < 9; ++i) {
    if (M[i][i] < M[i1][i1]) { i2 = i1; i1 = i; }
    else if (M[i][i] < M[i2][i2]) i2 = i;
  }
  double F1[9], F2[9];
  for (int k = 0; k < 9; ++k) { F1[k] = V[k][i1]; F2[k] = V[k][i2]; }
  return rs_seven_point(F1, F2, Fc);
}

// ---------------------------------------------------------------------------------------------------------------------
// The five-point solver (Nistér 2004, "An efficient solution to the five-point relative pose problem"), fp64, no dynamic
// allocation and a fixed iteration cap.  E = x N0 + y N1 + z N2 + N3 over the null space of the sample's five epipolar rows;
// det(E) = 0 and 2 E E^T E - tr(E E^T) E = 0 are ten cubics in (x, y, z), stored over Nistér's order of the 20 monomials
//   x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2 xyz xy | xz^2 xz x yz^2 yz y z^3 z^2 z 1,
// Gauss-Jordan eliminated on the first ten.  Rows (4, 5), (6, 7), (8, 9) then differ by a factor z in their leading monomials,
// so row(2m+4) - z row(2m+5) is linear in (x, y, 1) with polynomial coefficients in z; the determinant of those three rows is a
// degree-10 polynomial whose real roots (Sturm sequence + bisection, then safeguarded Newton) give z, and the null vector of
// the 3 x 3 system gives (x, y).  __host__ so that the host build can run the same arithmetic.
// ---------------------------------------------------------------------------------------------------------------------

// q += s * a * b: two linear forms over (x, y, z, 1) into a quadratic over (x^2, y^2, z^2, xy, xz, yz, x, y, z, 1)
__host__ __device__ __forceinline__ void rs_mul11(const double (&a)[4], const double (&b)[4], double s, double (&q)[10]) {
  const int Q[4][4] = {{0, 3, 4, 6}, {3, 1, 5, 7}, {4, 5, 2, 8}, {6, 7, 8, 9}};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) q[Q[i][j]] += s * a[i] * b[j];
}

// c += s * q * a: a quadratic times a linear form into a cubic over the 20 monomials above
__host__ __device__ __forceinline__ void rs_mul21(const double (&q)[10], const double (&a)[4], double s, double (&c)[20]) {
  const int C[10][4] = {{0, 2, 4, 5},    {3, 1, 6, 7},     {10, 13, 16, 17}, {2, 3, 8, 9},     {4, 8, 10, 11},
                        {8, 6, 13, 14},  {5, 9, 11, 12},   {9, 7, 14, 15},   {11, 14, 17, 18}, {12, 15, 18, 19}};
#pragma unroll
  for (int i = 0; i < 10; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[C[i][j]] += s * q[i] * a[j];
}

// c = a * b (ascending powers of z)
template <int NA, int NB>
__host__ __device__ __forceinline__ void rs_pmul(const double (&a)[NA], const double (&b)[NB], double (&c)[NA + NB - 1]) {
  for (int k = 0; k < NA + NB - 1; ++k) c[k] = 0.0;
  for (int i = 0; i < NA; ++i)
    for (int j = 0; j < NB; ++j) c[i + j] += a[i] * b[j];
}

__host__ __device__ __forceinline__ double rs_horner(const double* c, int deg, double x) {
  double v = c[deg];
  for (int k = deg - 1; k >= 0; --k) v = v * x + c[k];
  return v;
}

constexpr int RS_ROOT_BISECT = 80;     // Sturm bisection steps per root (isolates roots 2e7 / 2^80 apart)
constexpr int RS_ROOT_POLISH = 100;    // bisection + safeguarded Newton steps per isolated root
constexpr double RS_ROOT_BOUND = 1e7;  // |z| beyond this (E nearly without an N3 component) is not searched
constexpr int RS_ROOT_DET_NEWTON = 3;  // Newton steps per root on the unexpanded determinant

__host__ __device__ __forceinline__ double rs_det3(const double* r0, const double* r1, const double* r2) {
  return r0[0] * (r1[1] * r2[2] - r1[2] * r2[1]) - r0[1] * (r1[0] * r2[2] - r1[2] * r2[0]) + r0[2] * (r1[0] * r2[1] - r1[1] * r2[0]);
}

// Sign changes of the Sturm sequence S[0..ns-1] (degrees dg) at x.
__host__ __device__ __forceinline__ int rs_sturm_changes(const double (&S)[11][11], const int (&dg)[11], int ns, double x) {
  int changes = 0, last = 0;
  for (int i = 0; i < ns; ++i) {
    const double v = rs_horner(S[i], dg[i], x);
    const int s = v > 0.0 ? 1 : (v < 0.0 ? -1 : 0);
    if (s != 0) {
      if (last != 0 && s != last) ++changes;
      last = s;
    }
  }
  return changes;
}

// The distinct real roots in (-RS_ROOT_BOUND, RS_ROOT_BOUND) of the polynomial c (ascending, degree <= 10), ascending.
__host__ __device__ int rs_real_roots(const double (&c)[11], double (&roots)[10]) {
  double amax = 0.0;
  for (int k = 0; k <= 10; ++k) amax = fmax(amax, fabs(c[k]));
  if (!(amax > 1e-300) || !isfinite(amax)) return 0;
  int d = 10;
  while (d > 0 && fabs(c[d]) <= 1e-14 * amax) --d;   // leading terms at rounding level: those roots are at infinity
  if (d == 0) return 0;
  double S[11][11];
  int dg[11];
  for (int k = 0; k <= d; ++k) S[0][k] = c[k] / amax;
  dg[0] = d;
  double dmax = 0.0;
  for (int k = 1; k <= d; ++k) dmax = fmax(dmax, fabs(k * S[0][k]));
  for (int k = 1; k <= d; ++k) S[1][k - 1] = k * S[0][k] / dmax;
  dg[1] = d - 1;
  int ns = 2;
  while (ns < 11 && dg[ns - 1] > 0) {                  // S[i+1] = -(S[i-1] mod S[i]), each scaled to max |coefficient| 1
    double r[11];
    const int da = dg[ns - 2], db = dg[ns - 1];
    for (int k = 0; k <= da; ++k) r[k] = S[ns - 2][k];
    for (int k = da; k >= db; --k) {
      const double q = r[k] / S[ns - 1][db];
      for (int j = 0; j <= db; ++j) r[k - db + j] -= q * S[ns - 1][j];
    }
    int dr = db - 1;
    double rmax = 0.0;
    for (int k = 0; k <= dr; ++k) rmax = fmax(rmax, fabs(r[k]));
    if (!(rmax > 1e-12)) break;                        // S[ns-1] divides S[ns-2]: a repeated root; the count stays exact
    while (dr > 0 && fabs(r[dr]) <= 1e-14 * rmax) --dr;
    for (int k = 0; k <= dr; ++k) S[ns][k] = -r[k] / rmax;
    dg[ns] = dr;
    ++ns;
  }
  double bound = 0.0;                                  // Cauchy bound of the roots
  for (int k = 0; k < d; ++k) bound = fmax(bound, fabs(S[0][k] / S[0][d]));
  bound = fmin(1.0 + bound, RS_ROOT_BOUND);
  const int v_lo = rs_sturm_changes(S, dg, ns, -bound);
  const int total = min(max(v_lo - rs_sturm_changes(S, dg, ns, bound), 0), 10);
  double lo = -bound;
  int c_lo = 0;                                        // roots <= lo
  int nr = 0;
  for (int k = 0; k < total; ++k) {
    double hi = bound;
    int c_hi = total;
    for (int it = 0; it < RS_ROOT_BISECT && (c_hi - c_lo > 1 || c_lo != k); ++it) {
      const double mid = 0.5 * (lo + hi);
      const int cm = v_lo - rs_sturm_changes(S, dg, ns, mid);
      if (cm > k) { hi = mid; c_hi = cm; }
      else { lo = mid; c_lo = cm; }
    }
    // the k-th root is alone in (lo, hi]: bisection on the sign of S[0] down to a narrow bracket (an isolating interval can
    // be as wide as the search range), then Newton steps kept inside the bracket
    double a = lo, b = hi, fa = rs_horner(S[0], d, a);
    double x = 0.5 * (a + b);
    for (int it = 0; it < RS_ROOT_POLISH; ++it) {
      const double f = rs_horner(S[0], d, x);
      if (f == 0.0) break;
      if ((f > 0.0) == (fa > 0.0)) { a = x; fa = f; } else { b = x; }
      double xn = 0.5 * (a + b);
      if (b - a < 1e-3 * fmax(1.0, fabs(x))) {
        double df = 0.0;
        for (int j = d; j >= 1; --j) df = df * x + j * S[0][j];
        const double xt = x - f / df;
        if (xt > a && xt < b) xn = xt;
      }
      if (fabs(xn - x) <= 1e-15 * fmax(1.0, fabs(x))) { x = xn; break; }
      x = xn;
    }
    roots[nr++] = x;
    lo = hi;
    c_lo = c_hi;
  }
  return nr;
}

// The five-point step on a null-space basis N (four 3 x 3 matrices, row-major): 0-10 candidates, unit Frobenius norm.
__host__ __device__ int rs_five_point(const double (&N)[4][9], float (&Ec)[10][9]) {
  double L[9][4];                                      // entry k of E as a linear form over (x, y, z, 1)
  for (int k = 0; k < 9; ++k)
    for (int j = 0; j < 4; ++j) L[k][j] = N[j][k];
  double A[10][20];
  for (int r = 0; r < 10; ++r)
    for (int k = 0; k < 20; ++k) A[r][k] = 0.0;
  {                                                    // det(E), along the first row
    const int cof[3][4] = {{4, 8, 5, 7}, {5, 6, 3, 8}, {3, 7, 4, 6}};
    for (int c = 0; c < 3; ++c) {
      double q[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
      rs_mul11(L[cof[c][0]], L[cof[c][1]], 1.0, q);
      rs_mul11(L[cof[c][2]], L[cof[c][3]], -1.0, q);
      rs_mul21(q, L[c], 1.0, A[0]);
    }
  }
  double P[3][3][10];                                  // E E^T
  double tr[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      for (int k = 0; k < 10; ++k) P[i][j][k] = 0.0;
      for (int k = 0; k < 3; ++k) rs_mul11(L[3 * i + k], L[3 * j + k], 1.0, P[i][j]);
    }
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 10; ++k) tr[k] += P[i][i][k];
  for (int i = 0; i < 3; ++i)                          // 2 E E^T E - tr(E E^T) E
    for (int j = 0; j < 3; ++j) {
      for (int k = 0; k < 3; ++k) rs_mul21(P[i][k], L[3 * k + j], 2.0, A[1 + 3 * i + j]);
      rs_mul21(tr, L[3 * i + j], -1.0, A[1 + 3 * i + j]);
    }
  double amax = 0.0;
  for (int r = 0; r < 10; ++r)
    for (int k = 0; k < 20; ++k) amax = fmax(amax, fabs(A[r][k]));
  if (!(amax > 1e-300) || !isfinite(amax)) return 0;
  for (int c = 0; c < 10; ++c) {                       // Gauss-Jordan with partial pivoting on the ten leading monomials
    int piv = c;
    for (int r = c + 1; r < 10; ++r)
      if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
    if (!(fabs(A[piv][c]) > 1e-11 * amax)) return 0;  // rank-deficient: repeated or degenerate points
    if (piv != c)
      for (int k = c; k < 20; ++k) { const double t = A[c][k]; A[c][k] = A[piv][k]; A[piv][k] = t; }
    const double inv = 1.0 / A[c][c];
    for (int k = c; k < 20; ++k) A[c][k] *= inv;
    for (int r = 0; r < 10; ++r) {
      if (r == c) continue;
      const double f = A[r][c];
      for (int k = c; k < 20; ++k) A[r][k] -= f * A[c][k];
    }
  }
  double bx[3][4], by[3][4], b1[3][5];                 // rows (2m+4) - z (2m+5): coefficients of x, y and 1 in z
  for (int m = 0; m < 3; ++m) {
    const double* e = A[4 + 2 * m];
    const double* f = A[5 + 2 * m];
    bx[m][0] = e[12]; bx[m][1] = e[11] - f[12]; bx[m][2] = e[10] - f[11]; bx[m][3] = -f[10];
    by[m][0] = e[15]; by[m][1] = e[14] - f[15]; by[m][2] = e[13] - f[14]; by[m][3] = -f[13];
    b1[m][0] = e[19]; b1[m][1] = e[18] - f[19]; b1[m][2] = e[17] - f[18]; b1[m][3] = e[16] - f[17]; b1[m][4] = -f[16];
  }
  double p[11];
  {
    double u[8], v[8], w[7], t[11];
    rs_pmul(by[1], b1[2], u); rs_pmul(b1[1], by[2], v);
    for (int k = 0; k < 8; ++k) u[k] -= v[k];
    rs_pmul(bx[0], u, p);
    rs_pmul(bx[1], b1[2], u); rs_pmul(b1[1], bx[2], v);
    for (int k = 0; k < 8; ++k) u[k] -= v[k];
    rs_pmul(by[0], u, t);
    for (int k = 0; k < 11; ++k) p[k] -= t[k];
    double w2[7];
    rs_pmul(bx[1], by[2], w); rs_pmul(by[1], bx[2], w2);
    for (int k = 0; k < 7; ++k) w[k] -= w2[k];
    rs_pmul(b1[0], w, t);
    for (int k = 0; k < 11; ++k) p[k] += t[k];
  }
  double z[10];
  const int nz = rs_real_roots(p, z);
  int nc = 0;
  for (int j = 0; j < nz; ++j) {
    double B[3][3];
    // Newton on det B(z) evaluated from B's entries: the expanded degree-10 coefficients cancel badly when roots cluster
    for (int it = 0; it < RS_ROOT_DET_NEWTON; ++it) {
      double D[3][3];
      for (int m = 0; m < 3; ++m) {
        B[m][0] = rs_horner(bx[m], 3, z[j]); B[m][1] = rs_horner(by[m], 3, z[j]); B[m][2] = rs_horner(b1[m], 4, z[j]);
        D[m][0] = (3.0 * bx[m][3] * z[j] + 2.0 * bx[m][2]) * z[j] + bx[m][1];
        D[m][1] = (3.0 * by[m][3] * z[j] + 2.0 * by[m][2]) * z[j] + by[m][1];
        D[m][2] = ((4.0 * b1[m][4] * z[j] + 3.0 * b1[m][3]) * z[j] + 2.0 * b1[m][2]) * z[j] + b1[m][1];
      }
      const double f = rs_det3(B[0], B[1], B[2]);
      const double df = rs_det3(D[0], B[1], B[2]) + rs_det3(B[0], D[1], B[2]) + rs_det3(B[0], B[1], D[2]);
      const double step = f / df;
      if (!(fabs(step) < 1e-3 * fmax(1.0, fabs(z[j])))) break;   // not converging here: keep the polynomial's root
      z[j] -= step;
    }
    for (int m = 0; m < 3; ++m) {
      B[m][0] = rs_horner(bx[m], 3, z[j]); B[m][1] = rs_horner(by[m], 3, z[j]); B[m][2] = rs_horner(b1[m], 4, z[j]);
    }
    double v[3] = {0.0, 0.0, 0.0}, vn = -1.0;          // (x, y, 1): the largest cross product of two rows
    for (int a = 0; a < 3; ++a) {
      const double* r0 = B[a];
      const double* r1 = B[(a + 1) % 3];
      const double cr[3] = {r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2], r0[0] * r1[1] - r0[1] * r1[0]};
      const double n2 = cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2];
      if (n2 > vn) { vn = n2; v[0] = cr[0]; v[1] = cr[1]; v[2] = cr[2]; }
    }
    if (!(fabs(v[2]) > 1e-12 * sqrt(vn))) continue;
    const double x = v[0] / v[2], y = v[1] / v[2];
    double E[9], nrm = 0.0;
    for (int k = 0; k < 9; ++k) { E[k] = x * N[0][k] + y * N[1][k] + z[j] * N[2][k] + N[3][k]; nrm += E[k] * E[k]; }
    if (!(nrm > 1e-300) || !isfinite(nrm)) continue;
    const double inv = 1.0 / sqrt(nrm);
    for (int k = 0; k < 9; ++k) Ec[nc][k] = (float)(E[k] * inv);
    ++nc;
  }
  return nc;
}

// One 5-point sample, the body of a relative-pose hypothesis lane: the 9 x 9 normal matrix of the five epipolar rows of
// pts[idx[0..4]] (calibrated (x, y, u, v)), its four smallest eigenvectors (cyclic Jacobi) as the null space, and the 0-10
// candidates of rs_five_point.  Also run on its own by xfeat_debug_five_point.
__device__ __forceinline__ int rs_e5_sample(const float4* pts, const int (&idx)[5], float (&Ec)[10][9]) {
  double M[9][9];
  rs_epi_normal<5>(pts, idx, M);
  double V[9][9];
  rs_jacobi<9>(M, V);
  bool used[9] = {false, false, false, false, false, false, false, false, false};
  double N[4][9];
  for (int j = 0; j < 4; ++j) {                        // the four smallest eigenvalues, ascending
    int lo = -1;
    for (int i = 0; i < 9; ++i)
      if (!used[i] && (lo < 0 || M[i][i] < M[lo][lo])) lo = i;
    used[lo] = true;
    for (int k = 0; k < 9; ++k) N[j][k] = V[k][lo];
  }
  double l5 = 3.0e300, lmax = 0.0;                     // five independent rows, or the null space is not 4-D
  for (int i = 0; i < 9; ++i) {
    lmax = fmax(lmax, M[i][i]);
    if (!used[i]) l5 = fmin(l5, M[i][i]);
  }
  if (!(l5 > 1e-13 * lmax)) return 0;                   // repeated points
  return rs_five_point(N, Ec);
}

// Per-pair intrinsics of the calibrated model: K0, K1 (batch, 4) as (fx, fy, cx, cy); null for the other models.
struct RsCams {
  const float* K0;
  const float* K1;
};

// What the epipolar kernels need to know about a model:
//   kSample, kCands     minimal sample size, candidates per sample
//   kMinPts             fewest correspondences a pair needs for a model (below it: no model)
//   kLoMinBlocks        minimum blocks per SM in the local-optimisation kernel's launch bound (0: none)
//   Norm, camera()      what the model keeps per pair; camera() loads the pair's intrinsics into it (a no-op without)
//   prepare()           caches the pair's correspondences in sPts (visible to the block on return) and returns the squared
//                       threshold in the cached frame
//   solve()             one lane's sample -> candidates (unit-scale float models in the cached frame)
//   project()           the constraint every local-optimisation refit is projected onto
//   to_output()         a model of the cached frame -> the record's output model
//   inlier()            the final classification on the caller's coordinates
struct RsEssential {
  static constexpr int kSample = 8, kCands = 1, kMinPts = 8, kLoMinBlocks = 0;
  struct Norm {};
  static __device__ __forceinline__ void camera(const RsCams&, int, Norm&) {}
  static __device__ __forceinline__ float prepare(const float* __restrict__ q0, const float* __restrict__ q1, int n, float thr,
                                                  float4* sPts, Norm&) {
    for (int i = threadIdx.x; i < n; i += RS_THREADS) sPts[i] = make_float4(q0[2 * i], q0[2 * i + 1], q1[2 * i], q1[2 * i + 1]);
    __syncthreads();
    return thr * thr;
  }
  static __device__ __forceinline__ int solve(const float4* pts, const int (&idx)[kSample], float (&Ec)[kCands][9]) {
    double M[9][9], e[9];
    rs_epi_normal<8>(pts, idx, M);
    rs_smallest_eigvec<9>(M, e);
    rs_project_essential(e);
    for (int k = 0; k < 9; ++k) Ec[0][k] = (float)e[k];
    return 1;
  }
  static __device__ __forceinline__ void project(double (&E)[9]) { rs_project_essential(E); }
  static __device__ __forceinline__ void to_output(const Norm&, const float* sE, float* out) {
    for (int k = 0; k < 9; ++k) out[k] = sE[k];
  }
  static __device__ __forceinline__ bool inlier(const Norm&, const float (&E)[9], float x, float y, float u, float v, float thr) {
    return rs_sampson2(E, x, y, u, v) < thr * thr;
  }
};

struct RsFundamental {
  // One block per SM in the local optimisation's launch bound: under the default, ptxas caps that kernel at 128 registers and
  // spills.
  static constexpr int kSample = 7, kCands = 3, kMinPts = 8, kLoMinBlocks = 1;
  using Norm = RsPairNorm;
  static __device__ __forceinline__ void camera(const RsCams&, int, Norm&) {}
  static __device__ __forceinline__ float prepare(const float* __restrict__ q0, const float* __restrict__ q1, int n, float thr,
                                                  float4* sPts, Norm& nz) {
    nz = rs_pair_normalise(q0, q1, n, sPts);
    return (thr * nz.s) * (thr * nz.s);
  }
  static __device__ __forceinline__ int solve(const float4* pts, const int (&idx)[kSample], float (&Fc)[kCands][9]) {
    return rs_f_sample(pts, idx, Fc);
  }
  static __device__ __forceinline__ void project(double (&F)[9]) { rs_project_rank2(F); }
  // F = T1^T Fn T0 with T_i = [s 0 -s cx_i; 0 s -s cy_i; 0 0 1], unit Frobenius norm
  static __device__ __forceinline__ void to_output(const Norm& nz, const float* sF, float* out) {
    const double s = nz.s, t0[2] = {-s * nz.cx0, -s * nz.cy0}, t1[2] = {-s * nz.cx1, -s * nz.cy1};
    double A[9], F[9];                               // A = Fn T0
    for (int r = 0; r < 3; ++r) {
      const double f0 = sF[3 * r], f1 = sF[3 * r + 1], f2 = sF[3 * r + 2];
      A[3 * r] = f0 * s; A[3 * r + 1] = f1 * s; A[3 * r + 2] = f0 * t0[0] + f1 * t0[1] + f2;
    }
    for (int c = 0; c < 3; ++c) {                    // F = T1^T A
      F[c] = s * A[c]; F[3 + c] = s * A[3 + c]; F[6 + c] = t1[0] * A[c] + t1[1] * A[3 + c] + A[6 + c];
    }
    double nrm = 0.0;
    for (int k = 0; k < 9; ++k) nrm += F[k] * F[k];
    const double inv = nrm > 1e-300 ? 1.0 / sqrt(nrm) : 0.0;
    for (int k = 0; k < 9; ++k) out[k] = (float)(F[k] * inv);
  }
  static __device__ __forceinline__ bool inlier(const Norm&, const float (&F)[9], float x, float y, float u, float v, float thr) {
    return rs_sampson2_px(F, x, y, u, v) < (double)thr * (double)thr;
  }
};

// Calibrated relative pose (what poselib.estimate_relative_pose runs in the 1500-pair benchmarks, modules/eval/megadepth1500.py:
// 98-113, minus its non-linear refinement).  Inputs are PIXELS with per-pair intrinsics; prepare() caches K^-1-normalised
// coordinates, the minimal solver is the five-point algorithm (0-10 candidates, planar scenes included), and thr (pixels)
// becomes thr / f with f = (fx0 + fy0 + fx1 + fy1) / 4, the rule of evalharness.estimate_pose_opencv.  Inliers: Sampson
// distance in normalised coordinates, as RsEssential.
struct RsEssential5 {
  static constexpr int kSample = 5, kCands = 10, kMinPts = 5, kLoMinBlocks = 0;
  struct Norm { float fx0, fy0, cx0, cy0, fx1, fy1, cx1, cy1; };
  static __device__ __forceinline__ void camera(const RsCams& c, int pair, Norm& nz) {
    const float* a = c.K0 + 4 * pair;
    const float* b = c.K1 + 4 * pair;
    nz = Norm{a[0], a[1], a[2], a[3], b[0], b[1], b[2], b[3]};
  }
  static __device__ __forceinline__ float threshold(const Norm& nz, float thr) {
    return thr / (0.25f * (nz.fx0 + nz.fy0 + nz.fx1 + nz.fy1));
  }
  static __device__ __forceinline__ float4 normalise(const Norm& nz, float x, float y, float u, float v) {
    return make_float4((x - nz.cx0) / nz.fx0, (y - nz.cy0) / nz.fy0, (u - nz.cx1) / nz.fx1, (v - nz.cy1) / nz.fy1);
  }
  static __device__ __forceinline__ float prepare(const float* __restrict__ q0, const float* __restrict__ q1, int n, float thr,
                                                  float4* sPts, Norm& nz) {
    for (int i = threadIdx.x; i < n; i += RS_THREADS) sPts[i] = normalise(nz, q0[2 * i], q0[2 * i + 1], q1[2 * i], q1[2 * i + 1]);
    __syncthreads();
    const float t = threshold(nz, thr);
    return t * t;
  }
  static __device__ __forceinline__ int solve(const float4* pts, const int (&idx)[kSample], float (&Ec)[kCands][9]) {
    return rs_e5_sample(pts, idx, Ec);
  }
  static __device__ __forceinline__ void project(double (&E)[9]) { rs_project_essential(E); }
  static __device__ __forceinline__ void to_output(const Norm&, const float* sE, float* out) {
    for (int k = 0; k < 9; ++k) out[k] = sE[k];
  }
  static __device__ __forceinline__ bool inlier(const Norm& nz, const float (&E)[9], float x, float y, float u, float v, float thr) {
    const float4 c = normalise(nz, x, y, u, v);
    const float t = threshold(nz, thr);
    return rs_sampson2(E, c.x, c.y, c.z, c.w) < t * t;
  }
};

// Local optimisation of one candidate, by the whole block.  The fit of a minimal sample is noisy, so its consensus set is only
// part of the true one: RS_E_REFITS rounds of a Sampson-weighted 8-point refit (rows scaled by 1/|grad|, one IRLS step towards
// the Sampson error) over the points within mult*thr of the current model, mult shrinking 3 -> 1, each refit projected by
// Model::project.  The model kept is the one with the lowest MSAC cost at the true threshold, so the result is never worse
// than the candidate.  sE (shared, 9 floats): candidate in, optimised model out (visible to all threads on return).  Returns
// its MSAC cost.
template <class Model>
__device__ __forceinline__ float rs_local_opt(const float4* __restrict__ sPts, int n, float t2, float* sE) {
  __shared__ float sCost[RS_WARPS];
  __shared__ float sBestE[9];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float best_cost = RS_NO_COST;                      // block-uniform
  __syncthreads();
  for (int round = 0; round <= RS_E_REFITS; ++round) {
    float E[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) E[k] = sE[k];
    float cost = 0.f;                                // MSAC cost of the current model at the true threshold
    for (int i = threadIdx.x; i < n; i += RS_THREADS) {
      const float4 c = sPts[i];
      cost += fminf(rs_sampson2(E, c.x, c.y, c.z, c.w), t2);
    }
    for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
    if (lane == 0) sCost[warp] = cost;
    __syncthreads();
    float total = 0.f;
    for (int w = 0; w < RS_WARPS; ++w) total += sCost[w];      // same order in every thread
    if (total < best_cost) {
      best_cost = total;
      if (threadIdx.x < 9) sBestE[threadIdx.x] = E[threadIdx.x];
    }
    if (round == RS_E_REFITS) break;
    const float mult = round < 2 ? 3.0f : (round < 4 ? 2.0f : (round < 5 ? 1.5f : 1.0f));
    const float t2r = t2 * mult * mult;
    double acc[45];
#pragma unroll
    for (int k = 0; k < 45; ++k) acc[k] = 0.0;
    int cnt = 0;
    for (int i = threadIdx.x; i < n; i += RS_THREADS) {
      const float4 c = sPts[i];
      const float ea = E[0] * c.x + E[1] * c.y + E[2], eb = E[3] * c.x + E[4] * c.y + E[5];
      const float ed = E[0] * c.z + E[3] * c.w + E[6], ef = E[1] * c.z + E[4] * c.w + E[7];
      const float den = ea * ea + eb * eb + ed * ed + ef * ef;
      if (rs_sampson2(E, c.x, c.y, c.z, c.w) < t2r && den > 1e-20f) {
        ++cnt;
        double r[9];
        rs_epi_row(c.x, c.y, c.z, c.w, r);
        const double wgt = 1.0 / (double)den;
        int e = 0;
#pragma unroll
        for (int a = 0; a < 9; ++a) {
          const double ra = r[a] * wgt;
#pragma unroll
          for (int b2 = a; b2 < 9; ++b2) acc[e++] += ra * r[b2];
        }
      }
    }
    double M[9][9], vec[9];
    if (rs_block_normal_matrix(acc, cnt, 8, M) < 8) break;     // block-uniform
    if (threadIdx.x == 0) {
      rs_smallest_eigvec<9>(M, vec);
      Model::project(vec);
      for (int k = 0; k < 9; ++k) sE[k] = (float)vec[k];
    }
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x < 9) sE[threadIdx.x] = sBestE[threadIdx.x];
  __syncthreads();
  return best_cost;
}

// stage 1: grid (blocks_per_pair, batch).  Every lane solves one sample per round and the warp scores the lanes' candidates one
// after the other.  Samples come from a hash of (seed, pair id, hypothesis id): with the id fixed (pair_ids; NULL: the batch
// position), a pair's result does not depend on the batch it is in.
template <class Model>
__global__ void __launch_bounds__(RS_THREADS) ransac_hyp_kernel(const float* __restrict__ p0, const float* __restrict__ p1,
                                                                const int* __restrict__ np, const int* __restrict__ pair_ids,
                                                                RsCams cams, int n_max, float thr, int rounds_per_warp,
                                                                uint32_t seed, RsRecord* __restrict__ best) {
  extern __shared__ float4 sPts[];                 // (x, y, u, v) in the model's frame
  const int pair = blockIdx.y;
  const int n = min(np ? np[pair] : n_max, min(n_max, RS_MAX_PTS));
  RsRecord mine;
  mine.cost = RS_NO_COST;
#pragma unroll
  for (int k = 0; k < 9; ++k) mine.m[k] = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (n >= Model::kMinPts) {
    typename Model::Norm nz;
    Model::camera(cams, pair, nz);
    const float t2 = Model::prepare(p0 + (int64_t)pair * n_max * 2, p1 + (int64_t)pair * n_max * 2, n, thr, sPts, nz);
    const uint32_t pid = pair_ids ? (uint32_t)pair_ids[pair] : (uint32_t)pair;
    for (int rd = 0; rd < rounds_per_warp; ++rd) {
      const uint32_t hid = (uint32_t)(((blockIdx.x * RS_WARPS + warp) * rounds_per_warp + rd) * 32 + lane);
      int idx[Model::kSample];
      rs_draw<Model::kSample>(seed, pid, hid, n, idx);
      float Fc[Model::kCands][9];
      const int nc = Model::solve(sPts, idx, Fc);
      for (int src = 0; src < 32; ++src) {
        const int ncs = __shfl_sync(0xffffffffu, nc, src);
#pragma unroll
        for (int j = 0; j < Model::kCands; ++j) {
          if (j >= ncs) break;
          float F[9];
#pragma unroll
          for (int k = 0; k < 9; ++k) F[k] = __shfl_sync(0xffffffffu, Fc[j][k], src);
          float cost = 0.f;
          for (int i = lane; i < n; i += 32) {
            const float4 c = sPts[i];
            cost += fminf(rs_sampson2(F, c.x, c.y, c.z, c.w), t2);
          }
          for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
          if (cost < mine.cost) {
            mine.cost = cost;
#pragma unroll
            for (int k = 0; k < 9; ++k) mine.m[k] = F[k];
          }
        }
      }
    }
  }
  rs_block_best(mine, best);
}

// stage 2: every block's winner is optimised on its own (grid (blocks_per_pair, batch)) -- with w^7 or w^8 all-inlier samples
// the raw winners are few and noisy, and which of them converges to the full consensus set is not predictable from their raw
// cost.  The record then holds Model::to_output of the result; its cost stays in the cached frame, which all blocks of a pair
// share, so the final launch compares like with like.
template <class Model>
__global__ void __launch_bounds__(RS_THREADS, Model::kLoMinBlocks) ransac_lo_kernel(const float* __restrict__ p0,
                                                                                    const float* __restrict__ p1,
                                                                                    const int* __restrict__ np, RsCams cams,
                                                                                    int n_max, float thr,
                                                                                    RsRecord* __restrict__ best) {
  extern __shared__ float4 sPts[];
  __shared__ float sE[9];
  const int pair = blockIdx.y;
  const int n = min(np ? np[pair] : n_max, min(n_max, RS_MAX_PTS));
  if (n < Model::kMinPts) return;
  RsRecord* rec = best + (int64_t)pair * gridDim.x + blockIdx.x;
  if (!(rec->cost < RS_NO_COST)) return;             // this block found no hypothesis (block-uniform)
  typename Model::Norm nz;
  Model::camera(cams, pair, nz);
  const float t2 = Model::prepare(p0 + (int64_t)pair * n_max * 2, p1 + (int64_t)pair * n_max * 2, n, thr, sPts, nz);
  if (threadIdx.x < 9) sE[threadIdx.x] = rec->m[threadIdx.x];
  const float cost = rs_local_opt<Model>(sPts, n, t2, sE);
  if (threadIdx.x == 0) {
    Model::to_output(nz, sE, rec->m);
    rec->cost = cost;
  }
}

// stage 3: one block per pair: the best optimised candidate classifies the correspondences (Model::inlier) -> model, mask, count.
template <class Model>
__global__ void __launch_bounds__(RS_THREADS) ransac_final_kernel(const float* __restrict__ p0, const float* __restrict__ p1,
                                                                  const int* __restrict__ np, RsCams cams, int n_max,
                                                                  float thr, const RsRecord* __restrict__ best,
                                                                  int blocks_per_pair, float* __restrict__ M_out,
                                                                  unsigned char* __restrict__ mask, int* __restrict__ n_inl) {
  __shared__ float sM[9];
  const int pair = blockIdx.x;
  const int n_all = np ? np[pair] : n_max;
  const int n = min(n_all, min(n_max, RS_MAX_PTS));
  unsigned char* mk = mask + (int64_t)pair * n_max;
  for (int i = threadIdx.x; i < n_max; i += RS_THREADS) mk[i] = 0;
  if (n < Model::kMinPts) {
    if (threadIdx.x == 0) rs_write_none(n_all, 0.f, M_out + pair * 9, n_inl + pair);
    return;
  }
  typename Model::Norm nz;
  Model::camera(cams, pair, nz);
  const float* q0 = p0 + (int64_t)pair * n_max * 2;
  const float* q1 = p1 + (int64_t)pair * n_max * 2;
  if (threadIdx.x == 0) {
    const RsRecord b = rs_pair_best(best, pair, blocks_per_pair);
    for (int k = 0; k < 9; ++k) sM[k] = b.m[k];
  }
  __syncthreads();
  float m[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) m[k] = sM[k];
  int cnt = 0;
  for (int i = threadIdx.x; i < n; i += RS_THREADS) {
    const bool in = Model::inlier(nz, m, q0[2 * i], q0[2 * i + 1], q1[2 * i], q1[2 * i + 1], thr);
    mk[i] = in ? 1 : 0;
    cnt += in ? 1 : 0;
  }
  cnt = rs_block_count(cnt);
  if (threadIdx.x == 0) {
    n_inl[pair] = cnt;
    for (int k = 0; k < 9; ++k) M_out[pair * 9 + k] = m[k];
  }
}

// stage 4 of the relative pose: one block per pair.  The four (R, t) decompositions of the pair's E in geometry.recover_pose's
// order -- (R1, t), (R1, -t), (R2, t), (R2, -t) with E = U diag(1, 1, 0) V^T, det U = det V = +1, R1 = U W V^T,
// R2 = U W^T V^T, t = U[:, 2] -- and for each, the RANSAC inliers triangulated by the same 2 x 2 least-squares depth solve
// (z0 R x0 - z1 x1 = -t, normal equations + 1e-12 I), in fp64; the candidate with the most points in front of both cameras wins,
// the first in that order on a tie.  A pair without a model (no inliers) gets R = I, t = 0, n_front = 0.
__global__ void __launch_bounds__(RS_THREADS) ransac_pose_kernel(const float* __restrict__ p0, const float* __restrict__ p1,
                                                                 const int* __restrict__ np, RsCams cams, int n_max,
                                                                 const float* __restrict__ E_in,
                                                                 const unsigned char* __restrict__ mask,
                                                                 const int* __restrict__ n_inl, float* __restrict__ R_out,
                                                                 float* __restrict__ t_out, int* __restrict__ n_front) {
  __shared__ double sR[2][9], sT[3];
  __shared__ int sOk;
  const int pair = blockIdx.x;
  const int n = min(np ? np[pair] : n_max, min(n_max, RS_MAX_PTS));
  if (threadIdx.x == 0) {
    double E[9], M[3][3], V[3][3];
    for (int k = 0; k < 9; ++k) E[k] = E_in[pair * 9 + k];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) M[i][j] = E[i] * E[j] + E[3 + i] * E[3 + j] + E[6 + i] * E[6 + j];
    rs_jacobi<3>(M, V);
    int o[3] = {0, 1, 2};                              // singular values descending
    for (int a = 0; a < 3; ++a)
      for (int b = a + 1; b < 3; ++b)
        if (M[o[b]][o[b]] > M[o[a]][o[a]]) { const int t = o[a]; o[a] = o[b]; o[b] = t; }
    double v[3][3], u[3][3];                           // v[c], u[c]: column c of V, U
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r) v[c][r] = V[r][o[c]];
    const double dv = v[0][0] * (v[1][1] * v[2][2] - v[1][2] * v[2][1]) - v[0][1] * (v[1][0] * v[2][2] - v[1][2] * v[2][0]) +
                      v[0][2] * (v[1][0] * v[2][1] - v[1][1] * v[2][0]);
    if (dv < 0.0)
      for (int r = 0; r < 3; ++r) v[2][r] = -v[2][r];
    double s[2];
    for (int c = 0; c < 2; ++c) {                      // u_c = E v_c, u_1 orthogonalised against u_0
      for (int r = 0; r < 3; ++r) u[c][r] = E[3 * r] * v[c][0] + E[3 * r + 1] * v[c][1] + E[3 * r + 2] * v[c][2];
      if (c == 1) {
        const double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
        for (int r = 0; r < 3; ++r) u[1][r] -= d * u[0][r];
      }
      s[c] = sqrt(u[c][0] * u[c][0] + u[c][1] * u[c][1] + u[c][2] * u[c][2]);
      if (s[c] > 1e-300)
        for (int r = 0; r < 3; ++r) u[c][r] /= s[c];
    }
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];   // det U = +1
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    sOk = n_inl[pair] > 0 && s[0] > 1e-300 && s[1] > 1e-300;
    // R = U W V^T = u0 (W^T row 0) ... : W = [[0,-1,0],[1,0,0],[0,0,1]] maps columns: U W = [u1, -u0, u2], U W^T = [-u1, u0, u2]
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        sR[0][3 * i + j] = u[1][i] * v[0][j] - u[0][i] * v[1][j] + u[2][i] * v[2][j];
        sR[1][3 * i + j] = -u[1][i] * v[0][j] + u[0][i] * v[1][j] + u[2][i] * v[2][j];
      }
    for (int r = 0; r < 3; ++r) sT[r] = u[2][r];
  }
  __syncthreads();
  if (!sOk) {
    if (threadIdx.x < 9) R_out[pair * 9 + threadIdx.x] = (threadIdx.x % 4 == 0) ? 1.f : 0.f;
    if (threadIdx.x < 3) t_out[pair * 3 + threadIdx.x] = 0.f;
    if (threadIdx.x == 0) n_front[pair] = 0;
    return;
  }
  RsEssential5::Norm nz;
  RsEssential5::camera(cams, pair, nz);
  const float* q0 = p0 + (int64_t)pair * n_max * 2;
  const float* q1 = p1 + (int64_t)pair * n_max * 2;
  const unsigned char* mk = mask + (int64_t)pair * n_max;
  int cnt[4] = {0, 0, 0, 0};
  for (int i = threadIdx.x; i < n; i += RS_THREADS) {
    if (!mk[i]) continue;
    const double h0[3] = {((double)q0[2 * i] - nz.cx0) / nz.fx0, ((double)q0[2 * i + 1] - nz.cy0) / nz.fy0, 1.0};
    const double h1[3] = {((double)q1[2 * i] - nz.cx1) / nz.fx1, ((double)q1[2 * i + 1] - nz.cy1) / nz.fy1, 1.0};
    const double h11 = h1[0] * h1[0] + h1[1] * h1[1] + 1.0 + 1e-12;
    const double h1t = h1[0] * sT[0] + h1[1] * sT[1] + h1[2] * sT[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const double* R = sR[r];
      double a[3];
      for (int k = 0; k < 3; ++k) a[k] = R[3 * k] * h0[0] + R[3 * k + 1] * h0[1] + R[3 * k + 2];
      const double aa = a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + 1e-12, ah = -(a[0] * h1[0] + a[1] * h1[1] + a[2]);
      const double at = a[0] * sT[0] + a[1] * sT[1] + a[2] * sT[2];
      const double det = aa * h11 - ah * ah;
#pragma unroll
      for (int sg = 0; sg < 2; ++sg) {               // A = [a, -h1], b = -(+-t): A^T b = (-+ a.t, +- h1.t)
        const double b0 = sg == 0 ? -at : at, b1 = sg == 0 ? h1t : -h1t;
        const double z0 = (h11 * b0 - ah * b1) / det, z1 = (aa * b1 - ah * b0) / det;
        cnt[2 * r + sg] += (z0 > 0.0 && z1 > 0.0) ? 1 : 0;
      }
    }
  }
  int tot[4];
  for (int c = 0; c < 4; ++c) {
    tot[c] = rs_block_count(cnt[c]);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int best = 0;
    for (int c = 1; c < 4; ++c)
      if (tot[c] > tot[best]) best = c;
    const double sg = (best & 1) ? -1.0 : 1.0;
    for (int k = 0; k < 9; ++k) R_out[pair * 9 + k] = (float)sR[best >> 1][k];
    for (int k = 0; k < 3; ++k) t_out[pair * 3 + k] = (float)(sg * sT[k]);
    n_front[pair] = tot[best];
  }
}

// Test hook: one thread per 5-point sample (5 calibrated (x, y, u, v) rows), candidates zero-padded to 10.
__global__ void __launch_bounds__(RS_THREADS) ransac_debug_five_point_kernel(const float4* __restrict__ samples, int n_samples,
                                                                             float* __restrict__ E_out, int* __restrict__ count) {
  const int i = blockIdx.x * RS_THREADS + threadIdx.x;
  if (i >= n_samples) return;
  const int idx[5] = {0, 1, 2, 3, 4};
  float Ec[10][9];
  const int nc = rs_e5_sample(samples + (int64_t)i * 5, idx, Ec);
  for (int j = 0; j < 10; ++j)
    for (int k = 0; k < 9; ++k) E_out[((int64_t)i * 10 + j) * 9 + k] = j < nc ? Ec[j][k] : 0.f;
  count[i] = nc;
}

// Test hook: one thread per 7-point sample (7 normalised (x, y, u, v) rows), candidates zero-padded to 3.
__global__ void __launch_bounds__(RS_THREADS) ransac_f_debug_seven_point_kernel(const float4* __restrict__ samples, int n_samples,
                                                                                float* __restrict__ F_out, int* __restrict__ count) {
  const int i = blockIdx.x * RS_THREADS + threadIdx.x;
  if (i >= n_samples) return;
  const int idx[7] = {0, 1, 2, 3, 4, 5, 6};
  float Fc[3][9];
  const int nc = rs_f_sample(samples + (int64_t)i * 7, idx, Fc);
  for (int j = 0; j < 3; ++j)
    for (int k = 0; k < 9; ++k) F_out[((int64_t)i * 3 + j) * 9 + k] = j < nc ? Fc[j][k] : 0.f;
  count[i] = nc;
}

// The argument checks of every estimator entry point.
static int rs_check(const char* what, bool pointers, int n_max, int batch, float thr, int iters, size_t ws_bytes) {
  XF_REQUIRE(pointers, "%s: null pointer", what);
  XF_REQUIRE(batch > 0 && batch <= 65535 && n_max > 0 && n_max <= RS_MAX_PTS && iters > 0 && thr > 0.f,
             "%s: bad arguments (n_max <= %d)", what, RS_MAX_PTS);
  XF_REQUIRE(ws_bytes >= xfeat_ransac_workspace_bytes(batch, iters), "%s: workspace too small", what);
  return XF_OK;
}

// hyp -> lo -> final for an epipolar model: one round = one sample per lane, so a block draws RS_THREADS samples per round.
template <class Model>
static int rs_launch_epipolar(const char* what, const float* d_p0, const float* d_p1, const int32_t* d_n, const int32_t* d_pair_ids,
                              RsCams cams, int n_max, int batch, float thr, int iters, uint32_t seed, float* d_out,
                              uint8_t* d_inliers, int32_t* d_n_inliers, void* d_ws, size_t ws_bytes, void* stream) {
  const int rc = rs_check(what, d_p0 && d_p1 && d_out && d_inliers && d_n_inliers && d_ws, n_max, batch, thr, iters, ws_bytes);
  if (rc != XF_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int bpp = cdiv(iters, RS_WARPS * 32);
  const int rounds = cdiv(iters, bpp * RS_WARPS * 32);
  const size_t smem = (size_t)n_max * sizeof(float4);
  XF_DYN_SMEM(ransac_hyp_kernel<Model>, smem);
  XF_DYN_SMEM(ransac_lo_kernel<Model>, smem);
  ransac_hyp_kernel<Model><<<dim3(bpp, batch), RS_THREADS, smem, st>>>(d_p0, d_p1, d_n, d_pair_ids, cams, n_max, thr, rounds,
                                                                       seed, (RsRecord*)d_ws);
  XF_LAUNCH_CHECK();
  ransac_lo_kernel<Model><<<dim3(bpp, batch), RS_THREADS, smem, st>>>(d_p0, d_p1, d_n, cams, n_max, thr, (RsRecord*)d_ws);
  XF_LAUNCH_CHECK();
  ransac_final_kernel<Model><<<batch, RS_THREADS, 0, st>>>(d_p0, d_p1, d_n, cams, n_max, thr, (const RsRecord*)d_ws, bpp,
                                                           d_out, d_inliers, d_n_inliers);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

}  // namespace xf

extern "C" size_t xfeat_ransac_workspace_bytes(int batch, int iters) {
  const int bpp = (iters + xf::RS_WARPS * 32 - 1) / (xf::RS_WARPS * 32);   // 32 hypotheses per warp
  return xf::align_up((size_t)batch * (bpp > 0 ? bpp : 1) * sizeof(xf::RsRecord), 256);
}

extern "C" int xfeat_ransac_homography(const float* d_pts0, const float* d_pts1, const int32_t* d_n, int n_max, int batch,
                                       float thr_px, int iters, uint32_t seed, float* d_H, uint8_t* d_inliers,
                                       int32_t* d_n_inliers, void* d_ws, size_t ws_bytes, void* stream) {
  const int rc = xf::rs_check("ransac_homography", d_pts0 && d_pts1 && d_H && d_inliers && d_n_inliers && d_ws, n_max, batch,
                              thr_px, iters, ws_bytes);
  if (rc != XF_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int bpp = xf::cdiv(iters, xf::RS_WARPS * 32);
  const int hyp_per_warp = xf::cdiv(iters, bpp * xf::RS_WARPS);
  const size_t smem = (size_t)n_max * sizeof(float4);
  XF_DYN_SMEM(xf::ransac_h_hyp_kernel, smem);
  XF_DYN_SMEM(xf::ransac_h_final_kernel, smem);
  xf::ransac_h_hyp_kernel<<<dim3(bpp, batch), xf::RS_THREADS, smem, st>>>(d_pts0, d_pts1, d_n, n_max, thr_px, hyp_per_warp, seed,
                                                                          (xf::RsRecord*)d_ws);
  XF_LAUNCH_CHECK();
  xf::ransac_h_final_kernel<<<batch, xf::RS_THREADS, smem, st>>>(d_pts0, d_pts1, d_n, n_max, thr_px, (const xf::RsRecord*)d_ws, bpp,
                                                                 d_H, d_inliers, d_n_inliers);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_ransac_essential(const float* d_x0, const float* d_x1, const int32_t* d_n, int n_max, int batch, float thr,
                                      int iters, uint32_t seed, float* d_E, uint8_t* d_inliers, int32_t* d_n_inliers, void* d_ws,
                                      size_t ws_bytes, void* stream) {
  return xf::rs_launch_epipolar<xf::RsEssential>("ransac_essential", d_x0, d_x1, d_n, nullptr, xf::RsCams{nullptr, nullptr}, n_max,
                                                 batch, thr, iters, seed, d_E, d_inliers, d_n_inliers, d_ws, ws_bytes, stream);
}

extern "C" int xfeat_ransac_fundamental(const float* d_pts0, const float* d_pts1, const int32_t* d_n, const int32_t* d_pair_ids,
                                        int n_max, int batch, float thr_px, int iters, uint32_t seed, float* d_F,
                                        uint8_t* d_inliers, int32_t* d_n_inliers, void* d_ws, size_t ws_bytes, void* stream) {
  // the records hold pixel F after the lo launch: the final launch classifies with `Sampson < thr_px` in pixels
  return xf::rs_launch_epipolar<xf::RsFundamental>("ransac_fundamental", d_pts0, d_pts1, d_n, d_pair_ids, xf::RsCams{nullptr, nullptr},
                                                   n_max, batch, thr_px, iters, seed, d_F, d_inliers, d_n_inliers, d_ws, ws_bytes,
                                                   stream);
}

extern "C" int xfeat_relative_pose(const float* d_pts0, const float* d_pts1, const int32_t* d_n, const float* d_K0,
                                   const float* d_K1, const int32_t* d_pair_ids, int n_max, int batch, float thr_px, int iters,
                                   uint32_t seed, float* d_E, float* d_R, float* d_t, uint8_t* d_inliers, int32_t* d_n_inliers,
                                   int32_t* d_n_front, void* d_ws, size_t ws_bytes, void* stream) {
  XF_REQUIRE(d_K0 && d_K1 && d_R && d_t && d_n_front, "relative_pose: null pointer");
  const xf::RsCams cams{d_K0, d_K1};
  const int rc = xf::rs_launch_epipolar<xf::RsEssential5>("relative_pose", d_pts0, d_pts1, d_n, d_pair_ids, cams, n_max, batch,
                                                          thr_px, iters, seed, d_E, d_inliers, d_n_inliers, d_ws, ws_bytes,
                                                          stream);
  if (rc != XF_OK) return rc;
  xf::ransac_pose_kernel<<<batch, xf::RS_THREADS, 0, (cudaStream_t)stream>>>(d_pts0, d_pts1, d_n, cams, n_max, d_E, d_inliers,
                                                                              d_n_inliers, d_R, d_t, d_n_front);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_debug_five_point(const float* d_samples, int n_samples, float* d_E, int32_t* d_count, void* stream) {
  XF_REQUIRE(d_samples && d_E && d_count, "debug_five_point: null pointer");
  XF_REQUIRE(n_samples > 0 && ((uintptr_t)d_samples & 15) == 0, "debug_five_point: bad arguments (16-byte aligned samples)");
  xf::ransac_debug_five_point_kernel<<<xf::cdiv(n_samples, xf::RS_THREADS), xf::RS_THREADS, 0, (cudaStream_t)stream>>>(
      (const float4*)d_samples, n_samples, d_E, d_count);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_debug_seven_point(const float* d_samples, int n_samples, float* d_F, int32_t* d_count, void* stream) {
  XF_REQUIRE(d_samples && d_F && d_count, "debug_seven_point: null pointer");
  XF_REQUIRE(n_samples > 0 && ((uintptr_t)d_samples & 15) == 0, "debug_seven_point: bad arguments (16-byte aligned samples)");
  xf::ransac_f_debug_seven_point_kernel<<<xf::cdiv(n_samples, xf::RS_THREADS), xf::RS_THREADS, 0, (cudaStream_t)stream>>>(
      (const float4*)d_samples, n_samples, d_F, d_count);
  XF_LAUNCH_CHECK();
  return XF_OK;
}
