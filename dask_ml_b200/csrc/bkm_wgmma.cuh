// bkm_wgmma.cuh — Hopper (sm_90a) warpgroup MMA wrappers and the arg-min epilogue shared by the tensor-core kernels
// (bkm_tc.cu: fp16 split products, A from registers; bkm_tc2.cu: bf16 rows, A and B from shared memory).
//
// One warpgroup (128 threads) computes a 64-row x N-column fp32 tile.  Accumulator fragment of thread t
// (warp w = t / 32, g = lane / 4, c = lane % 4): d[4i + 0, 1] = row 16w + g, columns 8i + 2c, 8i + 2c + 1;
// d[4i + 2, 3] = row 16w + g + 8, same columns.  The fp16 A fragment of one K-step (16 columns) is
// a[0] = (row 16w+g, cols 2c, 2c+1), a[1] = (row +8, same), a[2] = (row 16w+g, cols 2c+8, 2c+9), a[3] = (row +8, same),
// the lower column in the low half of each register.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math_constants.h>
#include "bkm_ptx.cuh"

namespace bkm {
namespace wg {

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recently committed group have completed
__device__ __forceinline__ void wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void pin(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90): 8-row x 128-byte swizzle atoms, SBO = 1024 B between
// atoms along M/N, LBO unused for swizzled K-major layouts.  A K-step of 16 16-bit values (32 bytes inside the atom)
// advances the start address field by 2.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// byte offset of 16-byte chunk q (0..7) of row r inside one SWIZZLE_128B block ([rows][128 B])
__device__ __forceinline__ uint32_t sw128_chunk(int r, int q) { return (uint32_t)(r * 128 + ((q ^ (r & 7)) << 4)); }

// wgmma.m64nNk16 with fp32 accumulators: rs_f16 (A fp16 from registers, B fp16 from shared memory) and ss_bf16 (both
// bf16 from shared memory).  acc == 0 overwrites the accumulators.  N is the padded column count of the caller.
template <int N> struct Mma;
template <> struct Mma<16> {
  static __device__ __forceinline__ void rs_f16(float (&d)[8], const uint32_t (&a)[4], uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void ss_bf16(float (&d)[8], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Mma<32> {
  static __device__ __forceinline__ void rs_f16(float (&d)[16], const uint32_t (&a)[4], uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void ss_bf16(float (&d)[16], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Mma<64> {
  static __device__ __forceinline__ void rs_f16(float (&d)[32], const uint32_t (&a)[4], uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void ss_bf16(float (&d)[32], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Mma<128> {
  static __device__ __forceinline__ void rs_f16(float (&d)[64], const uint32_t (&a)[4], uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void ss_bf16(float (&d)[64], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Mma<256> {
  static __device__ __forceinline__ void rs_f16(float (&d)[128], const uint32_t (&a)[4], uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void ss_bf16(float (&d)[128], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(acc));
  }
};

// Column count of the MMA for `cols` valid columns (a multiple of 16, <= 256).
__host__ __device__ constexpr int mma_n(int cols) { return cols <= 16 ? 16 : cols <= 32 ? 32 : cols <= 64 ? 64 : cols <= 128 ? 128 : 256; }

// (best, its column, second best) of one row
struct Best2 { float m1, m2; int j; };
__device__ __forceinline__ void best2_add(Best2& b, float v, int j) {     // columns arrive in increasing order
  if (v < b.m1) { b.m2 = b.m1; b.m1 = v; b.j = j; }
  else b.m2 = fminf(b.m2, v);
}
// (best, column, second best) over the columns of b and o together, lowest column on exact ties
__device__ __forceinline__ void best2_join(Best2& b, const Best2& o) {
  if (o.m1 < b.m1 || (o.m1 == b.m1 && o.j < b.j)) { b.m2 = fminf(b.m1, o.m2); b.m1 = o.m1; b.j = o.j; }
  else b.m2 = fminf(b.m2, o.m1);
}
// merge with the lane `mask` away; both lanes end with the same result, lowest column on exact ties
__device__ __forceinline__ void best2_merge(Best2& b, int mask) {
  Best2 o;
  o.m1 = __shfl_xor_sync(0xffffffffu, b.m1, mask);
  o.m2 = __shfl_xor_sync(0xffffffffu, b.m2, mask);
  o.j = __shfl_xor_sync(0xffffffffu, b.j, mask);
  best2_join(b, o);
}
__device__ __forceinline__ Best2 best2_init() { return Best2{CUDART_INF_F, CUDART_INF_F, 0x7fffffff}; }
// Adds columns j0 .. j0 + N - 1 of the thread's two rows (g and g + 8) to (r0, r1): d is the 64 x N accumulator tile of
// those columns, value of column j = d[..] + cn[j] (cn: shared memory, padded columns hold a huge value).
template <int N>
__device__ __forceinline__ void best2_cols(const float (&d)[N / 2], const float* cn, int j0, int lane, Best2& r0, Best2& r1) {
  // two independent chains per row (the thread's even and its odd columns), joined at the end
  const int c2 = j0 + (lane & 3) * 2;
  Best2 o0 = best2_init(), o1 = o0;
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    const float2 cv = *reinterpret_cast<const float2*>(cn + 8 * i + c2);
    best2_add(r0, d[4 * i + 0] + cv.x, 8 * i + c2);
    best2_add(o0, d[4 * i + 1] + cv.y, 8 * i + c2 + 1);
    best2_add(r1, d[4 * i + 2] + cv.x, 8 * i + c2);
    best2_add(o1, d[4 * i + 3] + cv.y, 8 * i + c2 + 1);
  }
  best2_join(r0, o0);
  best2_join(r1, o1);
}
// merge over the four lanes of the quad: every lane ends with its rows' result over all the columns
__device__ __forceinline__ void best2_quad_merge(Best2& r0, Best2& r1) {
  best2_merge(r0, 1); best2_merge(r0, 2);
  best2_merge(r1, 1); best2_merge(r1, 2);
}
// Arg-min epilogue of a 64 x N accumulator tile.  Returns the (best, column, second best) of the thread's two rows,
// complete over all N columns.
template <int N>
__device__ __forceinline__ void tile_best2(const float (&d)[N / 2], const float* cn, int lane, Best2& r0, Best2& r1) {
  r0 = best2_init();
  r1 = r0;
  best2_cols<N>(d, cn, 0, lane, r0, r1);
  best2_quad_merge(r0, r1);
}

// Arg-min epilogue in two passes, for a caller that needs the best column and whether another column lies within a
// bound of it, but not the second-best value itself.  Pass 1 (min_cols, min_quad_merge) gives the row minimum m; the
// caller forms thr = m + bound; pass 2 (hit_cols, hit_quad_merge) counts the columns with value <= thr and sums their
// indices.  When thr is finite and the bound is >= 0, exactly one column qualifies iff the second best of the row is
// > thr, and that column is the arg-min.  NaN values are skipped by both passes, as best2_add skips them.
//
// Pass 1: forms the value d[..] + cn[j] of columns j0 .. j0 + N - 1 of the thread's two rows IN PLACE and folds their
// minima into m[0], m[1], in four independent chains per row (fminf returns the other operand of a NaN).
template <int N>
__device__ __forceinline__ void min_cols(float (&d)[N / 2], const float* cn, int j0, int lane, float (&m)[2]) {
  static_assert(N >= 16, "the chains start from columns i = 0, 1");
  const int c2 = j0 + (lane & 3) * 2;
  float p[2][4];                                     // [row][column parity + 2 (i parity)]
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    const float2 cv = *reinterpret_cast<const float2*>(cn + 8 * i + c2);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      d[4 * i + e] += (e & 1) ? cv.y : cv.x;
      float& c = p[e >> 1][2 * (i & 1) + (e & 1)];
      c = i < 2 ? d[4 * i + e] : fminf(c, d[4 * i + e]);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) m[h] = fminf(m[h], fminf(fminf(p[h][0], p[h][1]), fminf(p[h][2], p[h][3])));
}
// minimum over the four lanes of the quad: every lane ends with its rows' minima over all the columns
__device__ __forceinline__ void min_quad_merge(float (&m)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = fminf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
    m[h] = fminf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
  }
}
// Pass 2 over the values of columns j0 .. j0 + N - 1 (formed by min_cols) of the thread's two rows: hits[h] = the sum
// over those columns j with value <= t[h] of 1 + j / 1024, without the lane's column offset 2 (lane % 4) in j, which
// hit_quad_merge adds: each column then costs one FSET (0 for NaN) and one FFMA with an immediate (j0 is a constant of
// the unrolled caller).  Every partial sum is a multiple of 2^-10 below 2^9, so it is exact in any order.  Two chains
// per row.
template <int N>
__device__ __forceinline__ void hit_cols(const float (&d)[N / 2], int j0, const float (&t)[2], float (&hits)[2]) {
  float c[2][2] = {{0.f, 0.f}, {0.f, 0.f}};         // [row][column parity]
#pragma unroll
  for (int i = 0; i < N / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e)
      c[e >> 1][e & 1] = fmaf(ptx::fset_le(d[4 * i + e], t[e >> 1]), 1.f + (float)(j0 + 8 * i + (e & 1)) * 0.0009765625f, c[e >> 1][e & 1]);
#pragma unroll
  for (int h = 0; h < 2; ++h) hits[h] = c[h][0] + c[h][1];
}
// Both passes over one group of N columns (starting at j0) of a row whose columns are visited a group at a time, so
// that only one group's accumulators are live.  Before the first group m = +inf and hits = 0; after the last, m is the
// row minimum, thr = fma(tau, xb, m) (the near-tie bound tau xb does not depend on m) and hits is what hit_cols would
// count at thr over all the columns, or, for a row with two or more columns <= thr, some value >= 2 per quad.  At each
// group the running minimum mn = min(m, group minimum) gives thr; the earlier groups' hits were counted at the thr of
// their own running minimum m >= mn:
//   m == mn: thr is unchanged and they are exact;
//   m > thr: every earlier column is > thr, so they are dropped (0 hits);
//   mn < m <= thr: the earlier column at m and this group's column at mn are both <= thr: a near-tie either way, and the
//   earlier hits, which include the column at m (m <= fma(tau, xb, m), tau xb >= 0), keep the total >= 2.
// NaN values are skipped, and a NaN or infinite thr leaves the row a near-tie, as in the one-pass form.
template <int N>
__device__ __forceinline__ void near_tie_cols(float (&d)[N / 2], const float* cn, int j0, int lane, float tau,
                                              const float (&xb)[2], float (&m)[2], float (&thr)[2], float (&hits)[2]) {
  float mg[2] = {CUDART_INF_F, CUDART_INF_F};
  min_cols<N>(d, cn, j0, lane, mg);
  min_quad_merge(mg);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float mn = fminf(m[h], mg[h]);
    thr[h] = fmaf(tau, xb[h], mn);
    if (m[h] > thr[h]) hits[h] = 0.f;
    m[h] = mn;
  }
  float hg[2];
  hit_cols<N>(d, j0, thr, hg);
#pragma unroll
  for (int h = 0; h < 2; ++h) hits[h] += hg[h];
}
// Adds the lane's column offset, then sums over the quad: every lane ends with its rows' totals.  A lane with one hit
// holds a value in [1, 1.25) (its index part is < 256 / 1024), so floor() is its hit count; a lane with more hits
// gets some offset >= 0 and stays >= 2.  So the total lies in [1, 2) iff exactly one column of the row is <= t, and then
// it is 1 + (that column) / 1024.
__device__ __forceinline__ void hit_quad_merge(float (&hits)[2], int lane) {
  const float c2 = (float)((lane & 3) * 2) * 0.0009765625f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    hits[h] = fmaf(c2, floorf(hits[h]), hits[h]);
    hits[h] += __shfl_xor_sync(0xffffffffu, hits[h], 1);
    hits[h] += __shfl_xor_sync(0xffffffffu, hits[h], 2);
  }
}

// named barrier of one warpgroup (ids 1.. : id 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// 16-byte global -> shared copy; bytes beyond `src_bytes` (0..16) are zero-filled
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace wg
}  // namespace bkm
