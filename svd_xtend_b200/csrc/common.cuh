// Common sm_90a device helpers: mbarrier, TMA and wgmma inline PTX wrappers.
// Hand-written for H100 (compile with -gencode arch=compute_90a,code=sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace svdx {

typedef __nv_bfloat16 bf16;

#define SVDX_DEVINL __device__ __forceinline__

// Spin budget before a barrier wait is declared dead (a hung kernel on a shared GPU is far more
// expensive than a trap).
#ifndef SVDX_WAIT_TIMEOUT_CYCLES
#define SVDX_WAIT_TIMEOUT_CYCLES (4000000000ll)
#endif

SVDX_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

SVDX_DEVINL uint32_t lane_id() { return threadIdx.x & 31; }

SVDX_DEVINL bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
SVDX_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
SVDX_DEVINL void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
SVDX_DEVINL void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
SVDX_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
SVDX_DEVINL void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
SVDX_DEVINL bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
SVDX_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > SVDX_WAIT_TIMEOUT_CYCLES) {
      printf("svdx: mbarrier wait timeout block %d thread %d bar %u parity %u\n", blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
}

// the same wait without the report: inside a wgmma main loop a call (printf) would make ptxas serialise the wgmma pipeline
SVDX_DEVINL void mbar_wait_mma(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > SVDX_WAIT_TIMEOUT_CYCLES) __trap();
}

// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor)
SVDX_DEVINL void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
SVDX_DEVINL void tma_load_2d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
SVDX_DEVINL void tma_load_3d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
SVDX_DEVINL void tma_load_4d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col mode: c0 = first channel, (c1, c2, c3) = (w, h, n) of the first pixel in the map's start-pixel box; the pixels
// walk that box (w, then h, then n) and each is read at (w + ow, h + oh, n)
SVDX_DEVINL void tma_load_4d_im2col(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1, int c2, int c3, uint16_t ow,
                                    uint16_t oh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"(ow), "h"(oh)
      : "memory");
}

// ---- TMA stores (shared -> global through a tensor map, bulk-group completion)
SVDX_DEVINL void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
SVDX_DEVINL void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
SVDX_DEVINL void tma_reduce_add_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
SVDX_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
SVDX_DEVINL void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
SVDX_DEVINL void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
SVDX_DEVINL void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
SVDX_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SVDX_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
SVDX_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
SVDX_DEVINL void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

SVDX_DEVINL void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// Shared-memory matrix descriptor (wgmma), 128-byte swizzle.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type: 1 = SWIZZLE_128B
// K-major operand, rows of 64 bf16 (128 B): 8-row atom = 1024 B -> SBO = 1024, LBO unused; a 16-deep k-step adds 32 B.
// MN-major operand, 64 contiguous MN elements per 128 B line, 8 k-lines per atom:
//   SBO = 1024 (next 8 k), LBO = byte distance between 64-wide MN blocks; a 16-deep k-step adds 2048 B.
SVDX_DEVINL uint64_t make_smem_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// ---------------------------------------------------------------- misc math
// sigmoid through ex2.approx + rcp.approx (2 ulp): the IEEE division would cost ~10 instructions per element
SVDX_DEVINL float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
SVDX_DEVINL float silu_grad_f(float x) {
  const float s = __fdividef(1.0f, 1.0f + __expf(-x));
  return s * fmaf(x, 1.0f - s, 1.0f);
}
// GELU(erf) through the normal tail  Phi(-|x|) = 0.5 erfc(|x| / sqrt 2) = 2^P(|x|):  P is the degree-7 least-squares fit
// of log2(0.5 erfc(t / sqrt 2)) on [0, 5.5] (Chebyshev nodes). In fp32 Horner form the tail has a RELATIVE error
// <= 4.4e-6 everywhere, so gelu(x) = x * Phi(x) keeps that relative accuracy on the negative side too (the previous
// Abramowitz-Stegun 7.1.26 form had 1.5e-7 ABSOLUTE error, i.e. several per cent of gelu(x) for x < -4), with one
// MUFU (ex2) instead of two (rcp + ex2) and ~14 instead of ~22 instructions. |x| is clamped at 5.5 (tail 1.9e-8).
// tests/test_gelu_host.py compiles this header for the host and sweeps it against erf() in double precision.
#define SVDX_HDINL __host__ __device__ __forceinline__
SVDX_HDINL float gelu_tail_log2(float ax) {
  float p = -1.92123457e-06f;
  p = fmaf(p, ax, 6.32884985e-05f);
  p = fmaf(p, ax, -0.000943420862f);
  p = fmaf(p, ax, 0.0085562719f);
  p = fmaf(p, ax, -0.0540522821f);
  p = fmaf(p, ax, -0.458381772f);
  p = fmaf(p, ax, -1.15127838f);
  p = fmaf(p, ax, -0.999993861f);
  return p;
}
SVDX_HDINL float exp2_fast(float x) {
#ifdef __CUDA_ARCH__
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
#else
  return exp2f(x);
#endif
}
// Phi(x), the standard normal CDF
SVDX_HDINL float normal_cdf_f(float x) {
  const float q = exp2_fast(gelu_tail_log2(fminf(fabsf(x), 5.5f)));   // Phi(-|x|)
  return x < 0.f ? q : 1.0f - q;
}
SVDX_HDINL float gelu_erf_f(float x) { return x * normal_cdf_f(x); }
SVDX_HDINL float gelu_erf_grad_f(float x) {
  // Phi(x) + x * phi(x),  phi(x) = exp(-x^2 / 2) / sqrt(2 pi) = 2^(-x^2 * log2(e) / 2) / sqrt(2 pi)
  const float pdf = 0.3989422804014327f * exp2_fast(-0.72134752044448170f * x * x);
  return fmaf(x, pdf, normal_cdf_f(x));
}

SVDX_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
SVDX_DEVINL float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

SVDX_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SVDX_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace svdx
