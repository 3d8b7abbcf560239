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
// shared -> global box store; the TMA clips the elements that fall outside the tensor
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the stores of all but the newest N committed groups have finished READING shared memory (their source may be rewritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// every committed store has completed
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- per-thread asynchronous copies (cp.async)
// 8 bytes global -> shared; src_bytes = 0 zero-fills the destination without reading src
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(smem_dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// this thread's committed copies have all landed
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

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

// The same with the A operand in registers: a[0..3] = f16x2 pairs of thread (warp w, lane l), rows 16w + l/4 (a[0], a[2]) and
// 16w + l/4 + 8 (a[1], a[3]), columns 2(l%4) + {0,1} (a[0], a[1]) and 8 + 2(l%4) + {0,1} (a[2], a[3]) of the 16-column k-step.
// That is the accumulator layout above, so accumulator elements d[8k .. 8k+7] of one layer, converted pairwise, are the A
// operand of k-step k of the next layer (FlashAttention-3's P.V).
template <int N>
__device__ __forceinline__ void wgmma_f16_ra(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16_ra<16>(float (&d)[8], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_ra<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_ra<80>(float (&d)[40], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %45, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, {%40, %41, %42, %43}, %44, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
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
// N fp32 values -> split fp16 row pieces: hi block at hp, lo block at lp (N halves each, 32-byte aligned), x = hi + lo
template <int N>
__device__ __forceinline__ void store_split_row(__half* hp, __half* lp, const float (&o)[N]) {
  static_assert(N % 16 == 0, "store_split_row: N");
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

// ---------------------------------------------------------------- conv epilogue: fragments -> TMA tensor stores
// The convolution kernels write a tile's outputs straight from the wgmma fragments: thread (warp w, lane l) holds the group-0
// column c and the group-1 column NOUT + c of every channel c = 8j + 2(l%4) + e it owns, for rows r, r+8, r+64, r+72
// (r = 16w + l/4), so the split-term sum needs no transpose.  The values go into a staging PIECE -- 128 pixel rows of RB
// bytes, pixel-major as the NHWC output, swizzled as the tensor map's SWIZZLE_<RB>B -- that one thread hands to the TMA as a
// box {channels, TW, TH, 1}.  Pieces alternate between the two halves of the staging region, so piece k+1 is written while the
// TMA still reads piece k; the TMA clips the box at the image's right and bottom edges.
constexpr int STG_PIECE = STG_BYTES / 2;
template <int RB>
__device__ __forceinline__ uint32_t piece_off(int row, int byte) {   // 16-byte chunk index ^= (byte offset >> 7) % (RB / 16)
  const uint32_t o = (uint32_t)(row * RB + byte);
  return o ^ (((o >> 7) & (RB / 16 - 1)) << 4);
}

struct ConvEpi {
  const CUtensorMap* split;   // split fp16 output [hi(split_c) | lo(split_c)] or null; boxes of 32 halves (8-ch: 16, a whole row)
  const CUtensorMap* f32;     // fp32 output or null; boxes of 16 floats (8-ch: 8)
  int split_c;                // channels per half of a split pixel row
  int co;                     // output channel of the tile's first accumulator channel
  float inv_wscale;
  int relu;
  const float* bias;          // shared memory [NOUT]
  const float* skip_w;        // block1.3's skip branch: shared memory [2][NOUT] weights, biases; or null
  const float* skip_v;        // ... and the pooled input per staging row
  int x0, y0, b;              // box origin: the tile's first output pixel
  int wg = 0;                 // warpgroup of a CTA with several: its thread 0 issues the stores, its named barrier is 1 + wg
};

// one piece: every thread writes its part, one thread stores it.  `piece` counts the CTA's pieces: before the barrier that
// publishes piece k, the issuing thread waits until the TMA has read piece k-1, whose half piece k+1 is written into.
template <class Write>
__device__ __forceinline__ void conv_store_piece(unsigned char* stg, uint32_t& piece, const CUtensorMap* map, int c, const ConvEpi& E,
                                                 Write&& write) {
  unsigned char* buf = stg + (piece & 1) * STG_PIECE;
  write(buf);
  fence_proxy_async();   // this thread's generic-proxy writes, before the TMA (async proxy) reads them
  const bool lead = threadIdx.x == 128 * E.wg;
  if (lead) bulk_wait_read<0>();
  wg_sync(1 + E.wg);
  if (lead) {
    tma_store_4d(map, buf, c, E.x0, E.y0, E.b);
    bulk_commit();
  }
  ++piece;
}

// Channels per epilogue block (CB) and 8-column fragment groups per block (JB).
template <int NOUT>
struct EpiBlock {
  static constexpr int CB = NOUT < 32 ? NOUT : 32;
  static constexpr int JB = CB / 8;
};

// The values of channel block cb: bias, ReLU, block1.3's skip term (sv[h], the pooled input of fragment row h), then the split
// x = hi + lo -- per value in the order the model defines.  Thread q = lane % 4 gets channels 8j + 2q + e of fragment rows
// r, r+8, r+64, r+72 as o[h][jj][e], and the packed half2 pairs hi[h][jj], lo[h][jj].
template <int NOUT>
__device__ __forceinline__ void conv_values(const float (&d0)[NOUT], const float (&d1)[NOUT], int cb, const float (&sv)[4],
                                            const ConvEpi& E, float (&o)[4][EpiBlock<NOUT>::JB][2],
                                            uint32_t (&hi)[4][EpiBlock<NOUT>::JB], uint32_t (&lo)[4][EpiBlock<NOUT>::JB]) {
  constexpr int JB = EpiBlock<NOUT>::JB;
  constexpr int G1 = NOUT / 8;                // fragment group of the group-1 column of channel 0
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int h = 0; h < 4; ++h) {
#pragma unroll
    for (int jj = 0; jj < JB; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = cb * JB + jj, c = 8 * j + 2 * q + e, i = 2 * (h & 1) + e;
        const float g0 = (h < 2) ? d0[4 * j + i] : d1[4 * j + i];
        const float g1 = (h < 2) ? d0[4 * (j + G1) + i] : d1[4 * (j + G1) + i];
        float t = fmaf(g0 + g1, E.inv_wscale, E.bias[c]);
        if (E.relu) t = fmaxf(t, 0.f);
        if (E.skip_w != nullptr) t += fmaf(sv[h], E.skip_w[c], E.skip_w[NOUT + c]);
        o[h][jj][e] = t;
      }
      const __half2 hh = __floats2half2_rn(o[h][jj][0], o[h][jj][1]);
      const float2 hf = __half22float2(hh);
      const __half2 ll = __floats2half2_rn(o[h][jj][0] - hf.x, o[h][jj][1] - hf.y);
      hi[h][jj] = *reinterpret_cast<const uint32_t*>(&hh);
      lo[h][jj] = *reinterpret_cast<const uint32_t*>(&ll);
    }
  }
}

// conv_values, then the TMA stores.  srow[h] is the staging row of fragment row h (r, r+8, r+64, r+72), or -1 for a GEMM row
// that is no output pixel (halo junk lanes).
template <int NOUT>
__device__ __forceinline__ void conv_epilogue(const float (&d0)[NOUT], const float (&d1)[NOUT], unsigned char* stg, uint32_t& piece,
                                              const int (&srow)[4], const ConvEpi& E) {
  static_assert(NOUT == 8 || NOUT == 32 || NOUT == 64, "conv_epilogue: NOUT");
  constexpr int CB = EpiBlock<NOUT>::CB;      // channels per block
  constexpr int JB = EpiBlock<NOUT>::JB;      // 8-column fragment groups per block
  constexpr int RB = NOUT < 32 ? 32 : 64;     // staging row bytes
  const int q = threadIdx.x & 3;
  float sv[4];
#pragma unroll
  for (int h = 0; h < 4; ++h) sv[h] = (E.skip_w != nullptr && srow[h] >= 0) ? E.skip_v[srow[h]] : 0.f;
#pragma unroll
  for (int cb = 0; cb < NOUT / CB; ++cb) {
    float o[4][JB][2];
    uint32_t hi[4][JB], lo[4][JB];
    conv_values<NOUT>(d0, d1, cb, sv, E, o, hi, lo);
    if (E.split != nullptr) {
      if constexpr (NOUT == 8) {   // one piece of whole [hi(8) | lo(8)] rows
        conv_store_piece(stg, piece, E.split, 0, E, [&](unsigned char* buf) {
#pragma unroll
          for (int h = 0; h < 4; ++h)
            if (srow[h] >= 0) {
              *reinterpret_cast<uint32_t*>(buf + piece_off<RB>(srow[h], 4 * q)) = hi[h][0];
              *reinterpret_cast<uint32_t*>(buf + piece_off<RB>(srow[h], 16 + 4 * q)) = lo[h][0];
            }
        });
      } else {
#pragma unroll
        for (int half = 0; half < 2; ++half) {   // the hi piece of channels co + 32cb.., then the lo piece
          conv_store_piece(stg, piece, E.split, half * E.split_c + E.co + CB * cb, E, [&](unsigned char* buf) {
#pragma unroll
            for (int h = 0; h < 4; ++h)
              if (srow[h] >= 0) {
#pragma unroll
                for (int jj = 0; jj < JB; ++jj)
                  *reinterpret_cast<uint32_t*>(buf + piece_off<RB>(srow[h], 16 * jj + 4 * q)) = half ? lo[h][jj] : hi[h][jj];
              }
          });
        }
      }
    }
    if (E.f32 != nullptr) {
      constexpr int FJ = RB / 32;   // fragment groups per fp32 piece (8 floats = 32 bytes each)
#pragma unroll
      for (int k = 0; k < JB / FJ; ++k) {
        conv_store_piece(stg, piece, E.f32, E.co + CB * cb + 8 * FJ * k, E, [&](unsigned char* buf) {
#pragma unroll
          for (int h = 0; h < 4; ++h)
            if (srow[h] >= 0) {
#pragma unroll
              for (int jj = 0; jj < FJ; ++jj)
                *reinterpret_cast<float2*>(buf + piece_off<RB>(srow[h], 32 * jj + 8 * q)) =
                    make_float2(o[h][FJ * k + jj][0], o[h][FJ * k + jj][1]);
            }
        });
      }
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
// Tensor maps of a convolution's NHWC outputs as tc::conv_epilogue stores them: the split fp16 tensor (B,H,W,2*split_c) in
// boxes {32 halves, TW, TH, 1} and the fp32 tensor (B,H,W,f32_c) in boxes {16 floats, TW, TH, 1}, SWIZZLE_64B; 8-channel
// layers (c8) use {16 halves} (a whole [hi(8)|lo(8)] row) and {8 floats}, SWIZZLE_32B.  A null output gets no map; an output
// base or row that is not 16-byte aligned is an error.
int encode_conv_out_maps(PFN_encodeTiled enc, CUtensorMap* smap, __half* out_split, int split_c, CUtensorMap* fmap, float* out_f32,
                         int f32_c, bool c8, int B, int H, int W, int TW, int TH);

}  // namespace xf
