// LighterGlue matcher (modules/lighterglue.py:12-27, LightGlue with 96-d descriptors, 6 layers, 1 head; xfeat.py:131-162) for a
// batch of pairs with fixed capacity n_max and device-side point counts.  All arithmetic is fp32 on the CUDA cores:
//   - lg_linear_kernel: token-wise linears over every point of the batch (64-row tiles, weights streamed in 32-deep K chunks),
//     with the epilogues the model needs: rotary encoding of q and k, LayerNorm + GELU of the ffn's hidden layer, residual add;
//   - lg_attention_kernel: flash-style attention (online softmax in fp32), one kernel for self and cross attention -- only the
//     image the keys and values come from changes.  Key tiles are visited in order 0..ceil(n_keys/64), so a pair's result does
//     not depend on n_max or on the other pairs of the batch;
//   - lg_assign_kernel: the assignment in two passes over S = md0 md1^T (never stored): row / column log-sum-exp, then row /
//     column arg-max (first index on ties) of (S - lse0) + (S - lse1) + (logsigmoid(z0) + logsigmoid(z1));
//   - pruning: keep flags from the matchability, a per-image stable scan and a copy, all driven by device counts.
// No host synchronisation anywhere: counts after pruning stay on the device.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

struct xfeat_lg_ctx {
  int device;
  float* d_weights;
};

namespace xf {
namespace lg {

constexpr int D = 96;          // descriptor_dim
constexpr int DIN = 64;        // input_dim
constexpr int NPE = 48;        // positional-encoding frequencies (head_dim / 2)
constexpr int NL = 6;          // layers
constexpr int BM = 64;         // token rows per linear / attention CTA
constexpr int KC = 32;         // K chunk of the streamed weights
constexpr float KEEP_MIN = 0.05f;   // width_confidence 0.95: keep sigmoid(z) > 1 - 0.95

struct BlockW {                // one self or cross block: [qkv | out | ffn] as packed by weights.pack_lighterglue
  const float *qkv_w, *qkv_b, *out_w, *out_b, *f0_w, *f0_b, *ln_w, *ln_b, *f3_w, *f3_b;
};
struct Weights {
  const float *in_w, *in_b, *wr;
  BlockW blk[NL][2];
  const float *fp_w[NL], *fp_b[NL], *mz_w[NL], *mz_b[NL];
  size_t total;
};

static size_t pad4(size_t n) { return (n + 3) / 4 * 4; }

static Weights layout(const float* base) {
  Weights w;
  size_t o = 0;
  auto take = [&](size_t n) { const float* p = base ? base + o : nullptr; o += pad4(n); return p; };
  w.in_w = take(DIN * D); w.in_b = take(D); w.wr = take(2 * NPE);
  for (int l = 0; l < NL; ++l)
    for (int s = 0; s < 2; ++s) {
      BlockW& b = w.blk[l][s];
      const int nqkv = s == 0 ? 3 * D : 2 * D;
      b.qkv_w = take(D * nqkv); b.qkv_b = take(nqkv); b.out_w = take(D * D); b.out_b = take(D);
      b.f0_w = take(4 * D * D); b.f0_b = take(2 * D); b.ln_w = take(2 * D); b.ln_b = take(2 * D);
      b.f3_w = take(2 * D * D); b.f3_b = take(D);
    }
  for (int l = 0; l < NL; ++l) { w.fp_w[l] = take(D * D); w.fp_b[l] = take(D); w.mz_w[l] = take(D); w.mz_b[l] = take(1); }
  w.total = o;
  return w;
}

// ------------------------------------------------------------------------------------------------------------------------------
// token-wise linear: out[r] = epilogue(A[r] . W + b) for rows r < rows whose in-image index is below the image's count
// ------------------------------------------------------------------------------------------------------------------------------
enum Epi { EPI_PLAIN = 0, EPI_ROPE = 1, EPI_LN_GELU = 2, EPI_RESID = 3 };

struct LinArgs {
  const float* a; int lda;        // columns [0, k1) of the input row
  const float* a2; int lda2;      // columns [k1, K) (the [x | m] concatenation of the ffn), or null
  int k1, K, N;
  const float *w, *b;             // W[K][N], b[N]
  float* out; int ldo;            // EPI_RESID: out += ...
  const float* enc;               // EPI_ROPE: (rows, 96) [cos 48 | sin 48]
  const float *ln_w, *ln_b;       // EPI_LN_GELU
  float post_div;                 // EPI_PLAIN: (acc + b) / post_div
  const int32_t* cnt; int n_max, rows;
};

__device__ __forceinline__ bool row_valid(const int32_t* cnt, int n_max, int rows, int r) {
  return r < rows && (r % n_max) < cnt[r / n_max];
}

template <int NJ, int EPI>
__global__ void __launch_bounds__(256) lg_linear_kernel(LinArgs p) {
  extern __shared__ float sm[];
  const int K = p.K, N = NJ * 16, lds = K + 1;
  float* As = sm;                     // [BM][K+1]
  float* Ws = sm + BM * lds;          // [KC][N]
  float* Os = sm;                     // [BM][N+1], after the main loop
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int r0 = blockIdx.x * BM;
  int any = 0;
  if (tid < BM) any = row_valid(p.cnt, p.n_max, p.rows, r0 + tid);
  if (!__syncthreads_or(any)) return;
  for (int e = tid; e < BM * K; e += 256) {
    const int r = e / K, c = e % K, gr = r0 + r;
    float v = 0.f;
    if (row_valid(p.cnt, p.n_max, p.rows, gr)) v = c < p.k1 ? p.a[(size_t)gr * p.lda + c] : p.a2[(size_t)gr * p.lda2 + c - p.k1];
    As[r * lds + c] = v;
  }
  float acc[4][NJ];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += KC) {
    __syncthreads();
    for (int e = tid; e < KC * N; e += 256) Ws[e] = p.w[(size_t)k0 * N + e];
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < KC; ++kk) {
      float av[4], wv[NJ];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[(ty + 16 * i) * lds + k0 + kk];
#pragma unroll
      for (int j = 0; j < NJ; ++j) wv[j] = Ws[kk * N + tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
  }
  __syncthreads();
  const int ldo_s = N + 1;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) Os[(ty + 16 * i) * ldo_s + tx + 16 * j] = acc[i][j] + p.b[tx + 16 * j];
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp; r < BM; r += 8) {
    const int gr = r0 + r;
    if (!row_valid(p.cnt, p.n_max, p.rows, gr)) continue;
    const float* o = Os + r * ldo_s;
    float* dst = p.out + (size_t)gr * p.ldo;
    if (EPI == EPI_PLAIN) {
      for (int c = lane; c < N; c += 32) dst[c] = o[c] / p.post_div;
    } else if (EPI == EPI_RESID) {
      for (int c = lane; c < N; c += 32) dst[c] = dst[c] + o[c];
    } else if (EPI == EPI_ROPE) {     // [q | k | v]: q, k rotated pairwise (2j, 2j+1) -> (t cos - t' sin, t' cos + t sin)
      const float* en = p.enc + (size_t)gr * D;
      for (int c = lane; c < N; c += 32) {
        float v = o[c];
        if (c < 2 * D) {
          const int cc = c % D, jj = cc >> 1;
          const float rot = (cc & 1) ? o[c - 1] : -o[c + 1];
          v = v * en[jj] + rot * en[NPE + jj];
        }
        dst[c] = v;
      }
    } else {                          // EPI_LN_GELU, N = 192: LayerNorm(eps 1e-5, affine) then GELU(erf)
      constexpr int PER = NJ * 16 / 32;
      float h[PER];
      float s = 0.f;
#pragma unroll
      for (int t = 0; t < PER; ++t) { h[t] = o[lane + 32 * t]; s += h[t]; }
#pragma unroll
      for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
      const float mu = s / (float)N;
      float q = 0.f;
#pragma unroll
      for (int t = 0; t < PER; ++t) { const float d = h[t] - mu; q += d * d; }
#pragma unroll
      for (int m = 16; m; m >>= 1) q += __shfl_xor_sync(0xffffffffu, q, m);
      const float rstd = 1.f / sqrtf(q / (float)N + 1e-5f);
#pragma unroll
      for (int t = 0; t < PER; ++t) {
        const int c = lane + 32 * t;
        const float y = (h[t] - mu) * rstd * p.ln_w[c] + p.ln_b[c];
        dst[c] = y * 0.5f * (1.f + erff(y * 0.70710678118654752f));
      }
    }
  }
}

template <int NJ, int EPI>
static int launch_linear(const LinArgs& p, cudaStream_t st) {
  const size_t main_f = (size_t)BM * (p.K + 1) + (size_t)KC * NJ * 16, epi_f = (size_t)BM * (NJ * 16 + 1);
  const size_t smem = sizeof(float) * (main_f > epi_f ? main_f : epi_f);
  XF_DYN_SMEM((lg_linear_kernel<NJ, EPI>), smem);
  lg_linear_kernel<NJ, EPI><<<cdiv(p.rows, BM), 256, smem, st>>>(p);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

static int linear(LinArgs p, int epi, cudaStream_t st) {
  if (p.rows == 0) return XF_OK;
  if (!p.a2) { p.a2 = p.a; p.lda2 = p.lda; p.k1 = p.K; }
  if (p.N == 96 && epi == EPI_PLAIN) return launch_linear<6, EPI_PLAIN>(p, st);
  if (p.N == 96 && epi == EPI_RESID) return launch_linear<6, EPI_RESID>(p, st);
  if (p.N == 192 && epi == EPI_PLAIN) return launch_linear<12, EPI_PLAIN>(p, st);
  if (p.N == 192 && epi == EPI_LN_GELU) return launch_linear<12, EPI_LN_GELU>(p, st);
  if (p.N == 288 && epi == EPI_ROPE) return launch_linear<18, EPI_ROPE>(p, st);
  set_error("lighterglue: no linear kernel for N=%d epilogue %d", p.N, epi);
  return XF_E_INVALID;
}

// ------------------------------------------------------------------------------------------------------------------------------
// attention: out[g][i] = softmax_j(q_i . k_j / sqrt(96)) v_j over the keys j < n[kv(g)] of image kv(g)
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int LDA = D + 4;     // smem row stride of the 96-wide tiles (float4 rows, conflict-free 128-bit phases)

struct AttnArgs {
  const float *q, *k, *v; int ld;    // (G, n_max, ld) rows, the 96 columns start at the pointer
  const int32_t* cnt; int n_max, G;
  int cross;                         // 0: keys of the same image; 1: keys of the pair's other image (g +- G/2)
  float* out;                        // (G, n_max, 96)
};

__global__ void __launch_bounds__(256) lg_attention_kernel(AttnArgs p) {
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;                    // [64][LDA]
  float* Ks = Qs + BM * LDA;         // [64][LDA]
  float* Vs = Ks + BM * LDA;         // [64][LDA]
  float* Ps = Vs + BM * LDA;         // [64][68]
  const int g = blockIdx.y, half = p.G / 2;
  const int gk = p.cross ? (g < half ? g + half : g - half) : g;
  const int nq = p.cnt[g], nk = p.cnt[gk];
  const int q0 = blockIdx.x * BM;
  if (q0 >= nq) return;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const float scale = 1.f / sqrtf((float)D);
  for (int e = tid; e < BM * D / 4; e += 256) {
    const int r = e / (D / 4), c = (e % (D / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < nq) {
      const float* s = p.q + ((size_t)g * p.n_max + q0 + r) * p.ld + c;
      v = make_float4(s[0], s[1], s[2], s[3]);
    }
    *(float4*)(Qs + r * LDA + c) = v;
  }
  float o[4][6], mrow[4], lrow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    mrow[i] = -INFINITY; lrow[i] = 0.f;
#pragma unroll
    for (int c = 0; c < 6; ++c) o[i][c] = 0.f;
  }
  for (int k0 = 0; k0 < nk; k0 += BM) {
    __syncthreads();
    for (int e = tid; e < BM * D / 4; e += 256) {
      const int r = e / (D / 4), c = (e % (D / 4)) * 4;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + r < nk) {
        const size_t row = ((size_t)gk * p.n_max + k0 + r) * p.ld + c;
        kv = make_float4(p.k[row], p.k[row + 1], p.k[row + 2], p.k[row + 3]);
        vv = make_float4(p.v[row], p.v[row + 1], p.v[row + 2], p.v[row + 3]);
      }
      *(float4*)(Ks + r * LDA + c) = kv;
      *(float4*)(Vs + r * LDA + c) = vv;
    }
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 2
    for (int d = 0; d < D; d += 4) {
      float4 qa[4], kb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qa[i] = *(const float4*)(Qs + (ty + 16 * i) * LDA + d);
#pragma unroll
      for (int j = 0; j < 4; ++j) kb[j] = *(const float4*)(Ks + (tx + 16 * j) * LDA + d);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[i][j] = fmaf(qa[i].x, kb[j].x, s[i][j]);
          s[i][j] = fmaf(qa[i].y, kb[j].y, s[i][j]);
          s[i][j] = fmaf(qa[i].z, kb[j].z, s[i][j]);
          s[i][j] = fmaf(qa[i].w, kb[j].w, s[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float tmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = (k0 + tx + 16 * j < nk) ? s[i][j] * scale : -INFINITY;
        tmax = fmaxf(tmax, s[i][j]);
      }
#pragma unroll
      for (int m = 8; m; m >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, m));
      const float mnew = fmaxf(mrow[i], tmax);          // finite: key k0 < nk is in this tile
      const float corr = expf(mrow[i] - mnew);
      float ls = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float e = expf(s[i][j] - mnew);
        Ps[(ty + 16 * i) * 68 + tx + 16 * j] = e;
        ls += e;
      }
#pragma unroll
      for (int m = 8; m; m >>= 1) ls += __shfl_xor_sync(0xffffffffu, ls, m);
      lrow[i] = lrow[i] * corr + ls;
      mrow[i] = mnew;
#pragma unroll
      for (int c = 0; c < 6; ++c) o[i][c] *= corr;
    }
    __syncthreads();
#pragma unroll 2
    for (int kk = 0; kk < BM; kk += 4) {
      float4 pa[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pa[i] = *(const float4*)(Ps + (ty + 16 * i) * 68 + kk);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float vv[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) vv[c] = Vs[(kk + u) * LDA + tx + 16 * c];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float pv = u == 0 ? pa[i].x : u == 1 ? pa[i].y : u == 2 ? pa[i].z : pa[i].w;
#pragma unroll
          for (int c = 0; c < 6; ++c) o[i][c] = fmaf(pv, vv[c], o[i][c]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = q0 + ty + 16 * i;
    if (r >= nq) continue;
    const float inv = lrow[i] > 0.f ? 1.f / lrow[i] : 0.f;      // no keys: zero message
    float* dst = p.out + ((size_t)g * p.n_max + r) * D;
#pragma unroll
    for (int c = 0; c < 6; ++c) dst[tx + 16 * c] = o[i][c] * inv;
  }
}

static size_t attention_smem() { return sizeof(float) * (3 * BM * LDA + BM * 68); }

static int attention(const AttnArgs& p, cudaStream_t st) {
  if (p.n_max == 0 || p.G == 0) return XF_OK;
  XF_DYN_SMEM(lg_attention_kernel, attention_smem());
  lg_attention_kernel<<<dim3(cdiv(p.n_max, BM), p.G), 256, attention_smem(), st>>>(p);
  XF_LAUNCH_CHECK();
  return XF_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// input projection's companions: positional encoding, index maps, counts
// ------------------------------------------------------------------------------------------------------------------------------
__global__ void lg_encode_kernel(const float* __restrict__ kpts, const float* __restrict__ size, const int32_t* __restrict__ n_in,
                                 const float* __restrict__ wr, int B, int n_max, int side, float* __restrict__ enc,
                                 int32_t* __restrict__ ind, int32_t* __restrict__ cnt) {
  const int b = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = side * B + b;
  if (t == 0) cnt[g] = min(max(n_in[b], 0), n_max);     // XF_N_OVERFLOW -> 0 (reported by finalize)
  if (t >= n_max) return;
  ind[(size_t)g * n_max + t] = t;
  if (t >= n_in[b]) return;      // (n_in > n_max is clamped above: t < n_max here)
  const float W = size[2 * b], H = size[2 * b + 1];
  const float sc = fmaxf(W, H) / 2.f;
  const float kx = (kpts[((size_t)b * n_max + t) * 2] - W / 2.f) / sc;
  const float ky = (kpts[((size_t)b * n_max + t) * 2 + 1] - H / 2.f) / sc;
  float* e = enc + ((size_t)g * n_max + t) * D;
  for (int j = 0; j < NPE; ++j) {
    const float pj = kx * wr[j] + ky * wr[NPE + j];
    e[j] = cosf(pj);
    e[NPE + j] = sinf(pj);
  }
}

// z = matchability(x) (warp per token).  mode 0: keep flag for pruning (images with count <= T keep everything);
// mode 1: logsigmoid(z) for the assignment.
__global__ void lg_matchability_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                       const int32_t* __restrict__ cnt, int n_max, int rows, int mode, int T,
                                       int32_t* __restrict__ keep, float* __restrict__ lz) {
  const int r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (r >= rows) return;
  const int g = r / n_max, c = cnt[g];
  if (r % n_max >= c) return;
  const float* xr = x + (size_t)r * D;
  float s = 0.f;
  for (int k = lane; k < D; k += 32) s = fmaf(xr[k], w[k], s);
#pragma unroll
  for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  if (lane) return;
  const float z = s + bias[0];
  if (mode == 0) keep[r] = (c <= T) || (1.f / (1.f + expf(-z)) > KEEP_MIN);
  else lz[r] = fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
}

// per image: stable positions of the kept points, new count (one CTA of 1024 threads per image)
__global__ void __launch_bounds__(1024) lg_prune_scan_kernel(const int32_t* __restrict__ keep, const int32_t* __restrict__ cnt,
                                                             int n_max, int32_t* __restrict__ pos, int32_t* __restrict__ cnt_new) {
  __shared__ int wsum[32];
  __shared__ int base;
  const int g = blockIdx.x, n = cnt[g], tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) base = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int t = c0 + tid;
    const int k = t < n ? keep[(size_t)g * n_max + t] : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, k);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int off = 0;
    for (int w = 0; w < warp; ++w) off += wsum[w];
    if (t < n) pos[(size_t)g * n_max + t] = k ? base + off + __popc(bal & ((1u << lane) - 1u)) : -1;
    __syncthreads();
    if (tid == 0) { int s = 0; for (int w = 0; w < 32; ++w) s += wsum[w]; base += s; }
    __syncthreads();
  }
  if (tid == 0) cnt_new[g] = base;
}

__global__ void lg_prune_copy_kernel(const float* __restrict__ x, const float* __restrict__ enc, const int32_t* __restrict__ ind,
                                     const int32_t* __restrict__ pos, const int32_t* __restrict__ cnt, int n_max, int rows,
                                     float* __restrict__ x2, float* __restrict__ enc2, int32_t* __restrict__ ind2) {
  const int r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (r >= rows) return;
  const int g = r / n_max;
  if (r % n_max >= cnt[g]) return;
  const int p = pos[r];
  if (p < 0) return;
  const size_t src = (size_t)r * D, dst = ((size_t)g * n_max + p) * D;
  for (int k = lane; k < D; k += 32) { x2[dst + k] = x[src + k]; enc2[dst + k] = enc[src + k]; }
  if (lane == 0) ind2[(size_t)g * n_max + p] = ind[r];
}

// ------------------------------------------------------------------------------------------------------------------------------
// assignment.  blockIdx.z = direction: 0 = rows (queries of image 0 of pair b, keys of image 1), 1 = columns.
//   pass 0: lse[q] = log sum_k exp(S)   pass 1: best[q], arg[q] = max / first arg-max over k of (S - L0) + (S - L1) + (Z0 + Z1)
// ------------------------------------------------------------------------------------------------------------------------------
struct AssignArgs {
  const float* md;                   // (G, n_max, 96): final_proj(x) / 96^0.25
  const float* lz;                   // (G, n_max) logsigmoid(matchability)
  const int32_t* cnt; int n_max, B;
  float* lse;                        // (G, n_max)
  float* best; int32_t* arg;         // (G, n_max)
  int pass;
};

__global__ void __launch_bounds__(256) lg_assign_kernel(AssignArgs p) {
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;
  float* Ks = Qs + BM * LDA;
  float* Kl = Ks + BM * LDA;         // per key: lse, lz
  float* Kz = Kl + BM;
  const int b = blockIdx.y, dir = blockIdx.z;
  const int gq = dir * p.B + b, gk = (1 - dir) * p.B + b;
  const int nq = p.cnt[gq], nk = p.cnt[gk];
  const int q0 = blockIdx.x * BM;
  if (q0 >= nq || nk == 0) return;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int e = tid; e < BM * D / 4; e += 256) {
    const int r = e / (D / 4), c = (e % (D / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < nq) v = *(const float4*)(p.md + ((size_t)gq * p.n_max + q0 + r) * D + c);
    *(float4*)(Qs + r * LDA + c) = v;
  }
  float ql[4], qz[4], m[4], l[4];
  unsigned long long bv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = q0 + ty + 16 * i;
    const size_t qi = (size_t)gq * p.n_max + (r < nq ? r : 0);
    ql[i] = p.pass ? p.lse[qi] : 0.f;
    qz[i] = p.pass ? p.lz[qi] : 0.f;
    m[i] = -INFINITY; l[i] = 0.f; bv[i] = 0ull;
  }
  for (int k0 = 0; k0 < nk; k0 += BM) {
    __syncthreads();
    for (int e = tid; e < BM * D / 4; e += 256) {
      const int r = e / (D / 4), c = (e % (D / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + r < nk) v = *(const float4*)(p.md + ((size_t)gk * p.n_max + k0 + r) * D + c);
      *(float4*)(Ks + r * LDA + c) = v;
    }
    if (p.pass && tid < BM) {
      const size_t ki = (size_t)gk * p.n_max + (k0 + tid < nk ? k0 + tid : 0);
      Kl[tid] = p.lse[ki];
      Kz[tid] = p.lz[ki];
    }
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 2
    for (int d = 0; d < D; d += 4) {
      float4 qa[4], kb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qa[i] = *(const float4*)(Qs + (ty + 16 * i) * LDA + d);
#pragma unroll
      for (int j = 0; j < 4; ++j) kb[j] = *(const float4*)(Ks + (tx + 16 * j) * LDA + d);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[i][j] = fmaf(qa[i].x, kb[j].x, s[i][j]);
          s[i][j] = fmaf(qa[i].y, kb[j].y, s[i][j]);
          s[i][j] = fmaf(qa[i].z, kb[j].z, s[i][j]);
          s[i][j] = fmaf(qa[i].w, kb[j].w, s[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (p.pass == 0) {
        float tmax = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (k0 + tx + 16 * j >= nk) s[i][j] = -INFINITY;
          tmax = fmaxf(tmax, s[i][j]);
        }
#pragma unroll
        for (int mm = 8; mm; mm >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, mm));
        const float mnew = fmaxf(m[i], tmax);
        float ls = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) ls += expf(s[i][j] - mnew);
#pragma unroll
        for (int mm = 8; mm; mm >>= 1) ls += __shfl_xor_sync(0xffffffffu, ls, mm);
        l[i] = l[i] * expf(m[i] - mnew) + ls;
        m[i] = mnew;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int kj = k0 + tx + 16 * j;
          if (kj >= nk) continue;
          const float kl = Kl[tx + 16 * j], kz = Kz[tx + 16 * j];
          const float v = dir == 0 ? (s[i][j] - ql[i]) + (s[i][j] - kl) + (qz[i] + kz)
                                   : (s[i][j] - kl) + (s[i][j] - ql[i]) + (kz + qz[i]);
          const unsigned long long pk = pack_vi(v, (uint32_t)kj);
          bv[i] = pk > bv[i] ? pk : bv[i];
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (p.pass) {
#pragma unroll
      for (int mm = 8; mm; mm >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, bv[i], mm);
        bv[i] = o > bv[i] ? o : bv[i];
      }
    }
    const int r = q0 + ty + 16 * i;
    if (tx != 0 || r >= nq) continue;
    const size_t qi = (size_t)gq * p.n_max + r;
    if (p.pass == 0) {
      p.lse[qi] = m[i] + logf(l[i]);
    } else {
      p.best[qi] = ord2f((uint32_t)(bv[i] >> 32));
      p.arg[qi] = (int32_t)(0xffffffffu - (uint32_t)(bv[i] & 0xffffffffu));
    }
  }
}

static size_t assign_smem() { return sizeof(float) * (2 * BM * LDA + 2 * BM); }

// mutual check, threshold, compaction in idx0 order, mapping through the pruning index maps (one CTA per pair)
__global__ void __launch_bounds__(1024) lg_finalize_kernel(const float* __restrict__ best, const int32_t* __restrict__ arg,
                                                           const int32_t* __restrict__ ind, const int32_t* __restrict__ cnt,
                                                           const int32_t* __restrict__ n0_in, const int32_t* __restrict__ n1_in,
                                                           int n_max, int B, float min_conf, int64_t* __restrict__ idx0,
                                                           int64_t* __restrict__ idx1, float* __restrict__ scores,
                                                           int32_t* __restrict__ n_matches) {
  __shared__ int wsum[32];
  __shared__ int base;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t r0 = (size_t)b * n_max, r1 = (size_t)(B + b) * n_max;
  const int n0 = min(cnt[b], n_max), n1 = min(cnt[B + b], n_max);
  const bool overflow = n0_in[b] < 0 || n1_in[b] < 0;
  if (tid == 0) base = 0;
  __syncthreads();
  const int n = (overflow || n1 == 0) ? 0 : n0;
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + tid;
    int ok = 0, j = 0;
    float sc = 0.f;
    if (i < n) {
      j = arg[r0 + i];
      sc = expf(best[r0 + i]);
      ok = arg[r1 + j] == i && sc > min_conf;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += wsum[w];
    if (ok) {
      const int o = off + __popc(bal & ((1u << lane) - 1u));
      idx0[r0 + o] = ind[r0 + i];
      idx1[r0 + o] = ind[r1 + j];
      scores[r0 + o] = sc;
    }
    __syncthreads();
    if (tid == 0) { int s = 0; for (int w = 0; w < 32; ++w) s += wsum[w]; base += s; }
    __syncthreads();
  }
  if (tid == 0) n_matches[b] = overflow ? XF_N_OVERFLOW : base;
}

// ------------------------------------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------------------------------------
struct Inputs {
  int B, n_max;
  const float *kpts[2], *desc[2], *size[2];
  const int32_t* n[2];
  int prune_min_points;
};

struct Work {
  float *x[2], *enc[2], *qkv, *msg, *msg2, *hid, *lz, *lse, *best;
  int32_t *ind[2], *cnt[2], *keep, *pos, *arg;
};

static size_t carve(Bump& bm, Work& w, int B, int n_max) {
  const size_t T = (size_t)2 * B * n_max;
  for (int s = 0; s < 2; ++s) {
    w.x[s] = bm.take<float>(T * D);
    w.enc[s] = bm.take<float>(T * D);
    w.ind[s] = bm.take<int32_t>(T);
    w.cnt[s] = bm.take<int32_t>(2 * B);
  }
  w.qkv = bm.take<float>(T * 3 * D);
  w.msg = bm.take<float>(T * D);
  w.msg2 = bm.take<float>(T * D);
  w.hid = bm.take<float>(T * 2 * D);
  w.lz = bm.take<float>(T);
  w.lse = bm.take<float>(T);
  w.best = bm.take<float>(T);
  w.keep = bm.take<int32_t>(T);
  w.pos = bm.take<int32_t>(T);
  w.arg = bm.take<int32_t>(T);
  return bm.used();
}

static int block(const BlockW& bw, int cross, Work& w, int cur, int G, int n_max, cudaStream_t st) {
  const int rows = G * n_max;
  float* x = w.x[cur];
  const int32_t* cnt = w.cnt[cur];
  LinArgs a{};
  a.cnt = cnt; a.n_max = n_max; a.rows = rows; a.post_div = 1.f;
  // q, k, v (self, rotary applied) or [qk | v] (cross)
  a.a = x; a.lda = D; a.K = D; a.N = cross ? 2 * D : 3 * D; a.w = bw.qkv_w; a.b = bw.qkv_b; a.out = w.qkv; a.ldo = a.N;
  a.enc = w.enc[cur];
  int rc = linear(a, cross ? EPI_PLAIN : EPI_ROPE, st);
  if (rc) return rc;
  AttnArgs at{};
  at.q = w.qkv; at.k = w.qkv + (cross ? 0 : D); at.v = w.qkv + (cross ? D : 2 * D); at.ld = a.N;
  at.cnt = cnt; at.n_max = n_max; at.G = G; at.cross = cross; at.out = w.msg;
  if ((rc = attention(at, st))) return rc;
  LinArgs o{};
  o.cnt = cnt; o.n_max = n_max; o.rows = rows; o.post_div = 1.f;
  o.a = w.msg; o.lda = D; o.K = D; o.N = D; o.w = bw.out_w; o.b = bw.out_b; o.out = w.msg2; o.ldo = D;
  if ((rc = linear(o, EPI_PLAIN, st))) return rc;
  LinArgs f{};
  f.cnt = cnt; f.n_max = n_max; f.rows = rows; f.post_div = 1.f;
  f.a = x; f.lda = D; f.a2 = w.msg2; f.lda2 = D; f.k1 = D; f.K = 2 * D; f.N = 2 * D;
  f.w = bw.f0_w; f.b = bw.f0_b; f.ln_w = bw.ln_w; f.ln_b = bw.ln_b; f.out = w.hid; f.ldo = 2 * D;
  if ((rc = linear(f, EPI_LN_GELU, st))) return rc;
  LinArgs r{};
  r.cnt = cnt; r.n_max = n_max; r.rows = rows; r.post_div = 1.f;
  r.a = w.hid; r.lda = 2 * D; r.K = 2 * D; r.N = D; r.w = bw.f3_w; r.b = bw.f3_b; r.out = x; r.ldo = D;
  return linear(r, EPI_RESID, st);
}

// Runs the input stage and `n_layers` layers (pruning after layers 0..4 when prune_min_points >= 0); with n_layers == NL also
// the assignment into w.best / w.arg.  Returns the index of the live buffer set in *cur_out.
static int run(const Weights& W, const Inputs& in, Work& w, int n_layers, int* cur_out, cudaStream_t st) {
  const int B = in.B, n_max = in.n_max, G = 2 * B, rows = G * n_max;
  int cur = 0, rc;
  for (int s = 0; s < 2; ++s) {
    lg_encode_kernel<<<dim3(cdiv(n_max, 128), B), 128, 0, st>>>(in.kpts[s], in.size[s], in.n[s], W.wr, B, n_max, s, w.enc[0],
                                                                w.ind[0], w.cnt[0]);
    XF_LAUNCH_CHECK();
  }
  for (int s = 0; s < 2; ++s) {
    LinArgs a{};
    a.a = in.desc[s]; a.lda = DIN; a.K = DIN; a.N = D; a.w = W.in_w; a.b = W.in_b;
    a.out = w.x[0] + (size_t)s * B * n_max * D; a.ldo = D; a.post_div = 1.f;
    a.cnt = w.cnt[0] + s * B; a.n_max = n_max; a.rows = B * n_max;
    if ((rc = linear(a, EPI_PLAIN, st))) return rc;
  }
  for (int l = 0; l < n_layers; ++l) {
    if ((rc = block(W.blk[l][0], 0, w, cur, G, n_max, st))) return rc;
    if ((rc = block(W.blk[l][1], 1, w, cur, G, n_max, st))) return rc;
    if (l == NL - 1 || in.prune_min_points < 0) continue;
    lg_matchability_kernel<<<cdiv(rows, 8), 256, 0, st>>>(w.x[cur], W.mz_w[l], W.mz_b[l], w.cnt[cur], n_max, rows, 0,
                                                          in.prune_min_points, w.keep, nullptr);
    XF_LAUNCH_CHECK();
    lg_prune_scan_kernel<<<G, 1024, 0, st>>>(w.keep, w.cnt[cur], n_max, w.pos, w.cnt[cur ^ 1]);
    XF_LAUNCH_CHECK();
    lg_prune_copy_kernel<<<cdiv(rows, 8), 256, 0, st>>>(w.x[cur], w.enc[cur], w.ind[cur], w.pos, w.cnt[cur], n_max, rows,
                                                        w.x[cur ^ 1], w.enc[cur ^ 1], w.ind[cur ^ 1]);
    XF_LAUNCH_CHECK();
    cur ^= 1;
  }
  *cur_out = cur;
  if (n_layers < NL) return XF_OK;
  LinArgs f{};
  f.a = w.x[cur]; f.lda = D; f.K = D; f.N = D; f.w = W.fp_w[NL - 1]; f.b = W.fp_b[NL - 1]; f.out = w.msg; f.ldo = D;
  f.post_div = powf(96.f, 0.25f); f.cnt = w.cnt[cur]; f.n_max = n_max; f.rows = rows;
  if ((rc = linear(f, EPI_PLAIN, st))) return rc;
  lg_matchability_kernel<<<cdiv(rows, 8), 256, 0, st>>>(w.x[cur], W.mz_w[NL - 1], W.mz_b[NL - 1], w.cnt[cur], n_max, rows, 1, 0,
                                                        nullptr, w.lz);
  XF_LAUNCH_CHECK();
  XF_DYN_SMEM(lg_assign_kernel, assign_smem());
  for (int pass = 0; pass < 2; ++pass) {
    AssignArgs a{w.msg, w.lz, w.cnt[cur], n_max, B, w.lse, w.best, w.arg, pass};
    lg_assign_kernel<<<dim3(cdiv(n_max, BM), B, 2), 256, assign_smem(), st>>>(a);
    XF_LAUNCH_CHECK();
  }
  return XF_OK;
}

}  // namespace lg
}  // namespace xf

using namespace xf;

extern "C" size_t xfeat_lg_packed_weight_floats(void) { return lg::layout(nullptr).total; }

extern "C" int xfeat_lg_create(xfeat_lg_ctx** out, int device, const float* packed_host, size_t n_floats) {
  XF_REQUIRE(out && packed_host, "lg_create: null pointer");
  XF_REQUIRE(n_floats == lg::layout(nullptr).total, "lg_create: packed blob has %zu floats, expected %zu", n_floats,
             lg::layout(nullptr).total);
  DeviceGuard guard(device);
  XF_REQUIRE(guard.ok, "lg_create: cudaSetDevice(%d) failed", device);
  cudaDeviceProp prop;
  XF_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("lg_create: device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
    return XF_E_UNSUPPORTED;
  }
  float* d = nullptr;
  cudaError_t e = cudaMalloc(&d, sizeof(float) * n_floats);
  if (e == cudaSuccess) e = cudaMemcpy(d, packed_host, sizeof(float) * n_floats, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error("lg_create: weight upload failed: %s", cudaGetErrorString(e));
    if (d) cudaFree(d);
    return XF_E_CUDA;
  }
  *out = new xfeat_lg_ctx{device, d};
  return XF_OK;
}

extern "C" void xfeat_lg_destroy(xfeat_lg_ctx* ctx) {
  if (!ctx) return;
  DeviceGuard guard(ctx->device);
  cudaFree(ctx->d_weights);
  delete ctx;
}

extern "C" size_t xfeat_lg_workspace_bytes(int batch, int n_max) {
  if (batch < 0 || n_max < 0) return 0;
  Bump bm(nullptr, 0);
  lg::Work w;
  return lg::carve(bm, w, batch, n_max);
}

static int lg_prepare(xfeat_lg_ctx* ctx, int batch, int n_max, const float* d_kpts0, const float* d_desc0, const int32_t* d_n0,
                      const float* d_size0, const float* d_kpts1, const float* d_desc1, const int32_t* d_n1, const float* d_size1,
                      int prune_min_points, void* d_ws, size_t ws_bytes, lg::Inputs& in, lg::Work& w, lg::Weights& W) {
  XF_REQUIRE(ctx, "lighterglue: null context");
  XF_REQUIRE(batch >= 0 && n_max >= 0, "lighterglue: negative batch / n_max");
  XF_REQUIRE((size_t)2 * batch * n_max <= 0x7fffffffu, "lighterglue: 2 * batch * n_max exceeds 2^31");
  XF_REQUIRE(d_kpts0 && d_desc0 && d_n0 && d_size0 && d_kpts1 && d_desc1 && d_n1 && d_size1, "lighterglue: null input");
  in = lg::Inputs{batch, n_max, {d_kpts0, d_kpts1}, {d_desc0, d_desc1}, {d_size0, d_size1}, {d_n0, d_n1}, prune_min_points};
  Bump bm(d_ws, ws_bytes);
  lg::carve(bm, w, batch, n_max);
  if (!bm.ok) {
    set_error("lighterglue: workspace too small (%zu < %zu)", ws_bytes, bm.used());
    return XF_E_WORKSPACE;
  }
  W = lg::layout(ctx->d_weights);
  return XF_OK;
}

extern "C" int xfeat_lg_match(xfeat_lg_ctx* ctx, int batch, int n_max, const float* d_kpts0, const float* d_desc0,
                              const int32_t* d_n0, const float* d_size0, const float* d_kpts1, const float* d_desc1,
                              const int32_t* d_n1, const float* d_size1, float min_conf, int prune_min_points, int64_t* d_idx0,
                              int64_t* d_idx1, float* d_scores, int32_t* d_n_matches, void* d_ws, size_t ws_bytes, void* stream) {
  lg::Inputs in;
  lg::Work w;
  lg::Weights W;
  int rc = lg_prepare(ctx, batch, n_max, d_kpts0, d_desc0, d_n0, d_size0, d_kpts1, d_desc1, d_n1, d_size1, prune_min_points, d_ws,
                      ws_bytes, in, w, W);
  if (rc) return rc;
  XF_REQUIRE(d_idx0 && d_idx1 && d_scores && d_n_matches, "lg_match: null output");
  if (batch == 0) return XF_OK;
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int cur = 0;
  if (n_max > 0 && (rc = lg::run(W, in, w, lg::NL, &cur, st))) return rc;
  const int32_t* cnt = n_max > 0 ? w.cnt[cur] : d_n0;
  const int32_t* ind = w.ind[cur];
  if (n_max == 0) {      // nothing to match; counts still report overflow
    lg::lg_finalize_kernel<<<batch, 1024, 0, st>>>(w.best, w.arg, ind, d_n0, d_n0, d_n1, 0, batch, min_conf, d_idx0, d_idx1,
                                                   d_scores, d_n_matches);
  } else {
    lg::lg_finalize_kernel<<<batch, 1024, 0, st>>>(w.best, w.arg, ind, cnt, d_n0, d_n1, n_max, batch, min_conf, d_idx0, d_idx1,
                                                   d_scores, d_n_matches);
  }
  XF_LAUNCH_CHECK();
  return XF_OK;
}

extern "C" int xfeat_lg_debug(xfeat_lg_ctx* ctx, int batch, int n_max, const float* d_kpts0, const float* d_desc0,
                              const int32_t* d_n0, const float* d_size0, const float* d_kpts1, const float* d_desc1,
                              const int32_t* d_n1, const float* d_size1, int prune_min_points, int n_layers, float* d_x,
                              int32_t* d_ind, int32_t* d_cnt, float* d_best, int32_t* d_arg, void* d_ws, size_t ws_bytes,
                              void* stream) {
  lg::Inputs in;
  lg::Work w;
  lg::Weights W;
  int rc = lg_prepare(ctx, batch, n_max, d_kpts0, d_desc0, d_n0, d_size0, d_kpts1, d_desc1, d_n1, d_size1, prune_min_points, d_ws,
                      ws_bytes, in, w, W);
  if (rc) return rc;
  XF_REQUIRE(n_layers >= 0 && n_layers <= lg::NL, "lg_debug: n_layers must be in 0..6");
  XF_REQUIRE(batch > 0 && n_max > 0 && d_x && d_ind && d_cnt, "lg_debug: empty batch or null output");
  XF_REQUIRE(!(d_best || d_arg) || (n_layers == lg::NL && d_best && d_arg), "lg_debug: assignment outputs need n_layers == 6");
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int cur = 0;
  if ((rc = lg::run(W, in, w, n_layers, &cur, st))) return rc;
  const size_t T = (size_t)2 * batch * n_max;
  XF_CUDA(cudaMemcpyAsync(d_x, w.x[cur], T * lg::D * sizeof(float), cudaMemcpyDeviceToDevice, st));
  XF_CUDA(cudaMemcpyAsync(d_ind, w.ind[cur], T * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  XF_CUDA(cudaMemcpyAsync(d_cnt, w.cnt[cur], 2 * batch * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  if (d_best) {
    XF_CUDA(cudaMemcpyAsync(d_best, w.best, T * sizeof(float), cudaMemcpyDeviceToDevice, st));
    XF_CUDA(cudaMemcpyAsync(d_arg, w.arg, T * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  return XF_OK;
}

extern "C" int xfeat_lg_debug_attention(const float* d_q, const float* d_k, const float* d_v, int ld, const int32_t* d_n, int groups,
                                        int n_max, int cross, float* d_out, void* stream) {
  XF_REQUIRE(d_q && d_k && d_v && d_n && d_out, "lg_debug_attention: null pointer");
  XF_REQUIRE(groups > 0 && n_max > 0 && ld >= lg::D && ld % 4 == 0 && (!cross || groups % 2 == 0),
             "lg_debug_attention: bad shape");
  lg::AttnArgs a{d_q, d_k, d_v, ld, d_n, n_max, groups, cross, d_out};
  return lg::attention(a, (cudaStream_t)stream);
}

extern "C" int xfeat_lg_debug_assign(const float* d_md, const float* d_lz, const int32_t* d_cnt, int batch, int n_max, float* d_lse,
                                     float* d_best, int32_t* d_arg, void* stream) {
  XF_REQUIRE(d_md && d_lz && d_cnt && d_lse && d_best && d_arg, "lg_debug_assign: null pointer");
  XF_REQUIRE(batch > 0 && n_max > 0 && (size_t)2 * batch * n_max <= 0x7fffffffu, "lg_debug_assign: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  XF_DYN_SMEM(lg::lg_assign_kernel, lg::assign_smem());
  for (int pass = 0; pass < 2; ++pass) {
    lg::AssignArgs a{d_md, d_lz, d_cnt, n_max, batch, d_lse, d_best, d_arg, pass};
    lg::lg_assign_kernel<<<dim3(cdiv(n_max, lg::BM), batch, 2), 256, lg::assign_smem(), st>>>(a);
    XF_LAUNCH_CHECK();
  }
  return XF_OK;
}
