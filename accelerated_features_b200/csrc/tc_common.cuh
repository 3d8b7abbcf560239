// Hand-written sm_90a primitives: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma.mma_async with fp32 register
// accumulators) and its shared-memory matrix descriptors.  Bit layouts follow the PTX ISA "wgmma" chapter.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace xf {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One elected lane of a converged warp.  Unlike `lane == 0`, ptxas knows the guarded region runs on a single thread, so
// per-thread values feeding uniform-datapath instructions (UTMALDG operands) need no "waterfall" loop.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (sm_90a)
// D[registers] (+)= A[smem] * B[smem] for a 64-row slab, issued collectively by the four warps of one warpgroup.  Thread
// (warp w of the group, lane l) holds rows 16w + l/4 and 16w + l/4 + 8, columns 8j + 2(l%4) + {0,1}:
//   d[4j + 0..1] = row 16w + l/4, d[4j + 2..3] = row 16w + l/4 + 8.
// Both operands K-major (no transpose), descriptors as make_desc_* below.  `accumulate` = 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<8>(float (&d)[4], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
      "{%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<80>(float (&d)[40], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}

// The first N columns of a wider accumulator (the split-term GEMMs add lo.whi into the whi columns only).
template <int N, int NW>
__device__ __forceinline__ float (&acc_head(float (&d)[NW]))[N / 2] {
  static_assert(N / 2 <= NW, "acc_head");
  return *reinterpret_cast<float(*)[N / 2]>(&d[0]);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over the 128 threads of one warpgroup (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Fragment of a 128 x 128 tile held as two 64-row slabs (d0: rows 0-63, d1: rows 64-127): element (h, j, e) of thread wt is
// row frag_row(wt, h) (h = 0..3: r, r+8, r+64, r+72), column 8j + 2(lane%4) + e.
__device__ __forceinline__ float frag_val(const float (&d0)[64], const float (&d1)[64], int h, int j, int e) {
  return (h < 2) ? d0[4 * j + 2 * h + e] : d1[4 * j + 2 * (h - 2) + e];
}
__device__ __forceinline__ int frag_row(int wt, int h) { return 16 * (wt >> 5) + ((wt & 31) >> 2) + 8 * (h & 1) + 64 * (h >> 1); }

// ---------------------------------------------------------------- accumulator -> one row per thread
// The epilogues work on one output row per thread (rows of the 128-row tile = threads of the warpgroup).  An accumulator tile of
// two 64-row slabs (d0: rows 0-63, d1: rows 64-127) is handed over CW columns at a time through a 16 KB shared-memory buffer:
// 128 rows x 32 floats, 16-byte chunks XOR-swizzled by row so that both the fragment writes and the row reads are conflict-free.
constexpr int STG_BYTES = 128 * 32 * 4;
__device__ __forceinline__ int stg_off(int row, int col) { return row * 32 + ((((col >> 2) ^ row) & 7) << 2) + (col & 3); }
template <int CW, int R>
__device__ __forceinline__ void stage_write(float* stg, const float (&d0)[R], const float (&d1)[R], int c0, int wt) {
  static_assert(CW == 16 || CW == 32, "stage_write: CW");
  const int w = wt >> 5, l = wt & 31;
  const int r = 16 * w + (l >> 2), cq = 2 * (l & 3);
#pragma unroll
  for (int jj = 0; jj < CW / 8; ++jj) {
    const int j = c0 / 8 + jj;
    if (4 * j + 3 < R) {
      const int c = 8 * jj + cq;
      *reinterpret_cast<float2*>(stg + stg_off(r, c)) = make_float2(d0[4 * j], d0[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + stg_off(r + 8, c)) = make_float2(d0[4 * j + 2], d0[4 * j + 3]);
      *reinterpret_cast<float2*>(stg + stg_off(r + 64, c)) = make_float2(d1[4 * j], d1[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + stg_off(r + 72, c)) = make_float2(d1[4 * j + 2], d1[4 * j + 3]);
    }
  }
}
template <int CW>
__device__ __forceinline__ void stage_read(const float* stg, int row, uint32_t (&v)[CW]) {
#pragma unroll
  for (int k = 0; k < CW / 4; ++k) {
    const float4 t = *reinterpret_cast<const float4*>(stg + stg_off(row, 4 * k));
    v[4 * k] = __float_as_uint(t.x); v[4 * k + 1] = __float_as_uint(t.y);
    v[4 * k + 2] = __float_as_uint(t.z); v[4 * k + 3] = __float_as_uint(t.w);
  }
}
// columns [c0, c0 + CW) of the tile into v[] of thread `wt` (= its row); `bar` = this warpgroup's named barrier
template <int CW, int R>
__device__ __forceinline__ void acc_rows(float* stg, const float (&d0)[R], const float (&d1)[R], int c0, int wt, int bar,
                                         uint32_t (&v)[CW]) {
  stage_write<CW>(stg, d0, d1, c0, wt);
  wg_sync(bar);
  stage_read<CW>(stg, wt, v);
  wg_sync(bar);
}

// ---------------------------------------------------------------- epilogue stores
// 32 bytes per thread and call as two 16-byte stores: the conv epilogues write one pixel row per thread, so a warp-wide store
// touches 32 different rows and every 32-byte sector is written by the same thread.
__device__ __forceinline__ void st_global_v8(void* p, const uint32_t (&v)[8]) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(v[4], v[5], v[6], v[7]);
}
// N fp32 values -> split fp16 row pieces: hi block at hp, lo block at lp (N halves each), x = hi + lo.  hp / lp 32-byte aligned
// for N >= 16; N == 8: lp == hp + 8 and the 32-byte row [hi(8) | lo(8)] goes out as one store.
template <int N>
__device__ __forceinline__ void store_split_row(__half* hp, __half* lp, const float (&o)[N]) {
  static_assert(N == 8 || N % 16 == 0, "store_split_row: N");
  if constexpr (N == 8) {
    uint32_t v[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 h = __floats2half2_rn(o[2 * j], o[2 * j + 1]);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(o[2 * j] - hf.x, o[2 * j + 1] - hf.y);
      v[j] = *reinterpret_cast<const uint32_t*>(&h);
      v[4 + j] = *reinterpret_cast<const uint32_t*>(&l);
    }
    st_global_v8(hp, v);
  } else {
#pragma unroll
    for (int c = 0; c < N / 16; ++c) {
      uint32_t vh[8], vl[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float x0 = o[16 * c + 2 * j], x1 = o[16 * c + 2 * j + 1];
        const __half2 h = __floats2half2_rn(x0, x1);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
        vh[j] = *reinterpret_cast<const uint32_t*>(&h);
        vl[j] = *reinterpret_cast<const uint32_t*>(&l);
      }
      st_global_v8(hp + 16 * c, vh);
      st_global_v8(lp + 16 * c, vl);
    }
  }
}
// N fp32 values to a 32-byte aligned fp32 row, the first n_real of them (a multiple of 4)
template <int N>
__device__ __forceinline__ void store_f32_row(float* op, const float (&o)[N], int n_real) {
#pragma unroll
  for (int c = 0; c < N / 8; ++c) {
    if (8 * c + 8 <= n_real) {
      uint32_t v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __float_as_uint(o[8 * c + j]);
      st_global_v8(op + 8 * c, v);
    } else if (8 * c < n_real) {
      reinterpret_cast<float4*>(op + 8 * c)[0] = make_float4(o[8 * c], o[8 * c + 1], o[8 * c + 2], o[8 * c + 3]);
    }
  }
}

// ---------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle: rows are 128 B apart inside an 8-row atom
// (1024 B), atoms SBO apart.  Fields (wgmma matrix descriptor): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) |
// base_offset [49,52) | layout_type [62,64) (1 = SWIZZLE_128B, 3 = SWIZZLE_32B).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
  d |= (uint64_t)1 << 16;                               // LBO (ignored for swizzled K-major; canonical value 1)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
  d |= (uint64_t)1 << 62;                               // SWIZZLE_128B
  return d;
}
// Same for 32-byte rows (SWIZZLE_32B): 8-row atoms of 256 B.
__device__ __forceinline__ uint64_t make_desc_sw32(uint32_t smem_addr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
  d |= (uint64_t)3 << 62;                               // SWIZZLE_32B
  return d;
}
template <int ROWB>
__device__ __forceinline__ uint64_t make_desc_rows(uint32_t smem_addr) {
  return ROWB == 128 ? make_desc_sw128(smem_addr, 1024) : make_desc_sw32(smem_addr, 256);
}
}  // namespace tc

// Exact n / d for n < 2^22 by multiply-shift (the persistent tile loops decode tile -> (image, row, col) once per tile in
// three warp roles; ptxas' generic 32-bit division is ~40 instructions with MUFU latency, 25 % of the stall samples of the
// thin conv kernels).
struct FastDiv {
  unsigned long long magic;
  unsigned d;
};
static inline FastDiv make_fastdiv(unsigned d) {
  FastDiv f;
  f.d = d;
  f.magic = (1ull << 40) / d + 1;
  return f;
}
__device__ __forceinline__ unsigned fdiv(unsigned n, const FastDiv& f) { return (unsigned)(((unsigned long long)n * f.magic) >> 40); }

// Host: cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda link dependency).
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

}  // namespace xf
