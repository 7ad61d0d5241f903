// bkm_ptx.cuh — inline-PTX wrappers shared by the CUDA-core kernels (bkm_stream.cu, bkm_rowpass.cu, bkm_p2p.cu) and the
// float64 tensor-core passes (bkm_pca.cu, bkm_nb.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bkm {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n.reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n}"
      : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  return done != 0;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Wait with a WALL-CLOCK limit (2 s: profilers / sanitizers / time-slicing stretch spin counts, not the clock).
// Returns false on timeout; the caller records the failure in its abort word and drains.
__device__ __forceinline__ bool mbar_wait_timed(uint32_t bar, uint32_t parity, const volatile unsigned int* abort_word) {
  if (mbar_try(bar, parity)) return true;
  const unsigned long long t0 = globaltimer_ns();
  for (uint32_t spin = 0;; ++spin) {
    if (mbar_try(bar, parity)) return true;
    if ((spin & 63) == 63) {
      if (abort_word && *abort_word) return false;
      if (globaltimer_ns() - t0 > 2000000000ull) return false;
    }
  }
}
// plain wait (copies issued by the waiting warp itself: cannot dead-lock)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try(bar, parity)) { }
}
// 1-D bulk async copy global -> shared (16-byte aligned src/dst, size a multiple of 16), completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// packed fp32 pairs: two fused multiply-adds on the halves of a 64-bit register pair (sm_90 has no paired FFMA, so this
// is two FFMA; keeping the pair form lets the callers load / store operands as 64-bit pairs)
__device__ __forceinline__ unsigned long long pack2(float lo, float hi) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(unsigned long long v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ unsigned long long ffma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ float fmin3(float a, float b, float c) { return fminf(fminf(a, b), c); }
// 1.0f if a <= b else 0.0f (FSET: no predicate / select pair)
__device__ __forceinline__ float fset_le(float a, float b) {
  float r;
  asm("set.le.f32.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// D = A B + D, A 16x16 (row), B 16x8 (col), float64.  Fragments (g = lane / 4, t = lane % 4):
//   a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)],  b[i] = B[t + 4 i][g],  c = {(g, 2t), (g, 2t+1), (g+8, 2t), (g+8, 2t+1)}
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
        "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

}  // namespace ptx
}  // namespace bkm
