// ds_common.cuh — sm_90a device primitives shared by every kernel in libdsengine.
//
// Thin inline-PTX wrappers for the Hopper execution model: mbarrier and TMA (cp.async.bulk.tensor); the warpgroup
// MMA wrappers live in wgmma.cuh.  Nothing here is derived from the reference (it ships no native code, SURVEY.md
// §2.1); bit layouts follow the PTX ISA for sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ds {

// ----------------------------------------------------------------------------------------------
// small helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// bf16 pack on the INTEGER pipe: round-half-up on the 16 dropped mantissa bits (differs from RNE only on exact
// ties, no bias that matters) + one PRMT, instead of cvt.rn.bf16x2.f32, which issues at the lower XU rate.
// Inf stays Inf, NaN stays NaN; finite inputs only lose <= 0.5 ulp(bf16).
__device__ __forceinline__ uint32_t pack_bf16_alu(float lo, float hi) {
  const uint32_t a = __float_as_uint(lo) + 0x8000u;
  const uint32_t b = __float_as_uint(hi) + 0x8000u;
  return __byte_perm(a, b, 0x7632);  // {b.hi16, a.hi16}
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  A kernel launched with programmaticStreamSerializationAllowed may start
// (and run its prologue: barrier init, tensor-map prefetch) while its predecessor in the stream / graph
// is still draining; pdl_wait() blocks until the predecessor grid has completed and its memory is visible, and must
// precede the first global-memory access.  pdl_launch_dependents() lets OUR successor start early likewise.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy writes (st.shared) -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (launch error) instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 2000000000LL) __trap();  // ~1 s at 2 GHz: far beyond any legitimate wait
  }
}

// ----------------------------------------------------------------------------------------------
// TMA (tile mode). Coordinates are innermost-first and signed; out-of-bounds elements are zero-filled,
// which is what gives conv3x3 its zero padding and GEMM its M/N/K tails.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// math
// ----------------------------------------------------------------------------------------------
// x * sigmoid(x) with two MUFU ops (ex2 + rcp) instead of a full-precision divide
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// x * sigmoid(x) = 0.5 x (1 + tanh(x/2)) with ONE MUFU op (tanh.approx, abs err ~5e-4 on tanh => |err| <= 2.5e-4 |x|,
// below the bf16 rounding of the result for |x| < 16).  Used where the op is otherwise XU-bound (GroupNorm apply).
__device__ __forceinline__ float silu_tanh_f(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  const float hx = 0.5f * x;
  return fmaf(hx, t, hx);
}
// exact (erf) GELU, as nn.GELU() / diffusers GEGLU use
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// erf-GELU with the Abramowitz-Stegun 7.1.26 erf (|abs err| <= 1.5e-7, far below the bf16 output rounding):
//   erf(z) = 1 - (a1 t + ... + a5 t^5) exp(-z^2),  t = 1/(1 + 0.3275911 z),  z >= 0;  two MUFU ops + 8 FMAs
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-poly, e, 1.0f);           // erf(|x|/sqrt2)
  const float erf_v = copysignf(erf_abs, x);
  return 0.5f * x * (1.0f + erf_v);
}

// erf-GELU as x * sigmoid(2 k (x + a x^3 + b x^5)) with (k, a, b) fitted to x * Phi(x): |abs err| <= 2.6e-5 for every
// x (the classic tanh form with b = 0 is 4.7e-4), i.e. >= 10x below the bf16 rounding of the GEGLU product it feeds.
// 7 FP + 2 MUFU instead of the 15 FP + 2 MUFU of gelu_erf_fast, which keeps the GEGLU epilogue of the FF1 GEMM
// short.  The quintic changes sign beyond |x| ~ 11: clamp to +-10
// (sigmoid is saturated to 1 - 3e-9 there).
__device__ __forceinline__ float gelu_sig5(float x) {
  const float xc = fminf(fmaxf(x, -10.0f), 10.0f);
  const float x2 = xc * xc;
  float p = fmaf(-4.40769046e-4f, x2, 4.64016052e-2f);
  p = fmaf(p, x2, 1.0f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(xc * p * -2.301121339f));  // exp(-2 k u)
  return __fdividef(x, 1.0f + e);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace ds
