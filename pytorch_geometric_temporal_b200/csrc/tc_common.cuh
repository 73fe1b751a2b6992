// tc_common.cuh -- Hopper warpgroup MMA (wgmma) building blocks shared by the fused graph-GRU kernel, the split-fp16 GEMMs and the
// weight-gradient contraction: GMMA shared-memory descriptors, wgmma issue / commit / wait, the accumulator fragment layout, the
// hand-written SWIZZLE_128B K-major operand layout and the fp32 -> fp16 (hi, lo) operand split.
//
// A wgmma is issued by a whole warpgroup (4 consecutive warps, 128 threads) and accumulates an M = 64 row tile in the registers of that
// warpgroup.  Fragment of an m64nN fp32 accumulator d[N/2]: thread (warp w of the group, lane l) holds, for every 8-column group j,
//   d[4j + 0, 1] = D[16w + l/4    ][8j + 2(l%4) + 0, 1]
//   d[4j + 2, 3] = D[16w + l/4 + 8][8j + 2(l%4) + 0, 1]
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace stmp {

// GmmaDescriptor (sm_90): start>>4 [0,14) | LBO>>4 [16,30) (unused by swizzled K-major layouts: 1) | SBO>>4 [32,46) = bytes between
// 8-row groups | layout_type [62,64) (1 = SWIZZLE_128B, 2 = SWIZZLE_64B).  Operand tiles start on a swizzle-atom boundary; a k-step
// inside the atom advances the start address (the hardware applies the XOR pattern to the absolute address bits).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t sbo, uint32_t layout) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo >> 4) << 32) | ((uint64_t)layout << 62);
}
// K-major, SWIZZLE_128B, 128-byte rows (64 fp16): 8-row atoms of 1024 B
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) { return gmma_desc(saddr, 1024, 1); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 operands (K-major in shared memory), fp32 accumulator; scale_d == 0 overwrites D
__device__ __forceinline__ void wgmma_f16_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <int N> __device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t s) { wgmma_f16_n16(d, da, db, s); }
template <> __device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t s) { wgmma_f16_n32(d, da, db, s); }
template <> __device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t s) { wgmma_f16_n64(d, da, db, s); }

// The same with A from registers: a[4] = the m64k16 fragment of thread (warp w of the group, lane l), fp16 pairs
//   a[0] = A[16w + l/4][2(l%4) + 0, 1]   a[1] = A[16w + l/4 + 8][2(l%4) + 0, 1]   a[2], a[3] = the same rows at k + 8
// The registers must keep their values until a wgmma.wait_group has retired the instruction.
__device__ __forceinline__ void wgmma_f16_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// D = A * B (scale-d 0) with D write-only: the accumulator is not live before the first MMA of a chain, which frees its registers
// between the chains
__device__ __forceinline__ void wgmma_f16_rs_n32_first(float (&d)[16], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, 0, 1, 1, 0;"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]),
        "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
__device__ __forceinline__ void wgmma_f16_rs_n64_first(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 0, 1, 1, 0;"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]),
        "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]),
        "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]),
        "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

// D[64 x 32] += A[64 x 8] * B[32 x 8]^T, TF32 operands (K-major), fp32 accumulator
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db));
}

// Writes an m64nN accumulator fragment (N = 2 R) of warpgroup-thread `wt` (0..127) into a row-major fp32 tile:
// rows row0 .. row0 + 63, columns col0 .. col0 + N - 1, `pitch` floats per row.
template <int R>
__device__ __forceinline__ void acc_store(float* tile, int pitch, int row0, int col0, int wt, const float (&d)[R]) {
  const int r = row0 + 16 * (wt >> 5) + ((wt & 31) >> 2), c = col0 + 2 * (wt & 3);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(tile + (size_t)r * pitch + c + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(tile + (size_t)(r + 8) * pitch + c + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// CW consecutive accumulator values of one row of such a tile (col % 4 == 0, pitch % 4 == 0)
template <int CW>
__device__ __forceinline__ void acc_ld(const float* tile, int pitch, int row, int col, uint32_t (&v)[CW]) {
  const float4* src = reinterpret_cast<const float4*>(tile + (size_t)row * pitch + col);
#pragma unroll
  for (int j = 0; j < CW / 4; ++j) {
    const float4 q = src[j];
    v[4 * j] = __float_as_uint(q.x); v[4 * j + 1] = __float_as_uint(q.y); v[4 * j + 2] = __float_as_uint(q.z); v[4 * j + 3] = __float_as_uint(q.w);
  }
}

// byte offset of element (row, kin) inside a K-panel (kin in [0,64))
__device__ __forceinline__ int sw128(int row, int kin) { return row * 128 + ((((kin >> 3) ^ (row & 7))) << 4) + ((kin & 7) << 1); }

__device__ __forceinline__ uint32_t pack_h2(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// split 4 floats into fp16 hi/lo and store them (8 B each) at k offset `kin` (multiple of 4) of `row`
__device__ __forceinline__ void store_split4(unsigned char* a_hi, unsigned char* a_lo, int row, int kin, float4 v) {
  const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
  const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
  const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
  const int off = sw128(row, kin);
  *reinterpret_cast<uint2*>(a_hi + off) = make_uint2(pack_h2(h01), pack_h2(h23));
  *reinterpret_cast<uint2*>(a_lo + off) = make_uint2(pack_h2(l01), pack_h2(l23));
}

}  // namespace stmp
