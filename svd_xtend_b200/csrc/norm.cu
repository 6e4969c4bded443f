// GroupNorm(32)(+SiLU) and LayerNorm, forward and backward, over channels-last bf16 activations.
// HBM-bound CUDA-core kernels: 16-byte vector accesses, fp32 statistics, warp-shuffle / shared-memory reductions, fp32
// atomics for the cross-CTA partial sums. The row-streaming kernels (GroupNorm apply / backward, LayerNorm forward /
// backward) keep their loads in flight through cp.async rings in shared memory instead of registers (DESIGN.md 3.3).
//
// Replaces F.group_norm + F.silu of ResnetBlock2D / TemporalResnetBlock / TransformerSpatioTemporalModel
// [D: diffusers models/resnet.py, transformer_temporal.py] and conv_norm_out
// (/root/reference/src/unet_spatio_temporal_condition.py:238-239,480-481), and F.layer_norm of
// BasicTransformerBlock / TemporalBasicTransformerBlock [D: models/attention.py].
#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"
#include <stdio.h>
#include <stdlib.h>

namespace svdx {

struct GnSrc {
  const bf16* x;
  long long ldx;
  int C1;
  const bf16* x2;
  long long ldx2;
  int C2;
};

constexpr int GNV_MAX_THREADS = 512;
constexpr int GN_RIF = 4;            // independent row loads per thread of the channel-sum kernel
#ifndef SVDX_LN_MINB
#define SVDX_LN_MINB 1               // register-array LayerNorm kernels (C > 1280 only): minimum resident CTAs per SM
#endif
extern __shared__ uint4 gn_ring_smem[];

// ------------------------------------------------------------------ GroupNorm channel sums
// Every GroupNorm consumer reads its statistics as per-(slab, channel) sums, [outer][2][ld] fp32 and zero on entry: the
// gn_sum / gnb_sum that svdx_tapgemm's epilogues accumulate (include/svd_xtend_b200.h). The two kernels below write the SAME
// sums for a tensor no epilogue covered. Both end the same way: each active thread leaves its 8 channels' partials in
// shared memory at part[(rl * 2 + moment) * C + c], and the block sums its RL row lanes there before one
// red.global.add.v4.f32 per 4 channels and moment.
SVDX_DEVINL void gn_csum_put(float* part, int C, int rl, int c0, const float (&a)[8], const float (&b)[8]) {
  float* p = part + (2LL * rl) * C + c0;
  *reinterpret_cast<float4*>(p) = make_float4(a[0], a[1], a[2], a[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(a[4], a[5], a[6], a[7]);
  *reinterpret_cast<float4*>(p + C) = make_float4(b[0], b[1], b[2], b[3]);
  *reinterpret_cast<float4*>(p + C + 4) = make_float4(b[4], b[5], b[6], b[7]);
}

SVDX_DEVINL void gn_csum_flush(const float* part, int C, int RL, float* out, long long ld) {
  const int C4 = C / 4;
  for (int i = threadIdx.x; i < 2 * C4; i += blockDim.x) {
    const int m = i / C4, c = (i - m * C4) * 4;
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1                                     // unrolled, this tail would set the kernels' register count
    for (int r = 0; r < RL; ++r) {
      const float4 v = *reinterpret_cast<const float4*>(part + (2LL * r + m) * C + c);
      t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
    }
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(out + m * ld + c), "f"(t.x), "f"(t.y), "f"(t.z), "f"(t.w) : "memory");
  }
}

SVDX_DEVINL uint4 load_vec8(const GnSrc& s, long long row, int c0) {
  const bf16* p = (c0 < s.C1) ? (s.x + row * s.ldx + c0) : (s.x2 + row * s.ldx2 + (c0 - s.C1));
  return *reinterpret_cast<const uint4*>(p);
}

// forward: sum x, sum x^2 per (slab, channel) into sum[outer][2][ld] (the gn_sum layout). A thread owns ONE 8-channel vector
// (16 B) and walks rows, keeping 4 loads in flight; the block is (C/8 channel vectors) x (row lanes), grid (row_chunks, outer),
// dynamic shared memory 2 * C * RL floats for the row-lane reduction.
__global__ void __launch_bounds__(GNV_MAX_THREADS, 1) gn_sums(GnSrc s, int rows, int rows_per_cta, float* sum, long long ld) {
  const int C = s.C1 + s.C2;
  const int CV = C / 8;
  const int n = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(r0 + rows_per_cta, rows);
  const int RL = blockDim.x / CV;          // row lanes
  const int cv = threadIdx.x % CV, rl = threadIdx.x / CV;
  float* part = reinterpret_cast<float*>(gn_ring_smem);
  if (rl < RL) {
    const int c0 = cv * 8;
    float a[8], b[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { a[k] = 0.f; b[k] = 0.f; }
    const long long base = (long long)n * rows;
    int r = r0 + rl;
    for (; r + 3 * RL < r1; r += 4 * RL) {
      uint4 u[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) u[q] = load_vec8(s, base + r + q * RL, c0);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t w[4] = {u[q].x, u[q].y, u[q].z, u[q].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 v = unpack_bf16x2(w[k]);
          a[2 * k] += v.x; a[2 * k + 1] += v.y;
          b[2 * k] += v.x * v.x; b[2 * k + 1] += v.y * v.y;
        }
      }
    }
    for (; r < r1; r += RL) {
      const uint4 u = load_vec8(s, base + r, c0);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 v = unpack_bf16x2(w[k]);
        a[2 * k] += v.x; a[2 * k + 1] += v.y;
        b[2 * k] += v.x * v.x; b[2 * k + 1] += v.y * v.y;
      }
    }
    gn_csum_put(part, C, rl, c0, a, b);
  }
  __syncthreads();
  gn_csum_flush(part, C, RL, sum + (2LL * n) * ld, ld);
}

// ------------------------------------------------------------------ GroupNorm, cp.async ring variants
// GroupNorm apply (+SiLU) and backward. Round 1-2's first versions kept 4 x 16-byte loads per tensor in flight per thread in
// REGISTERS and then stalled on them; with 84-128 registers a thread only 15-30 warps were resident, so an SM had a load burst
// in flight a fraction of the time (1-2.6 TB/s). Here every thread streams its rows through a private GN_RING-deep ring of 16-byte shared-memory slots filled by
// cp.async (LDGSTS): GN_RING rows per tensor stay in flight per thread continuously, no registers are tied up by loads in
// flight, and the first GN_RING rows are requested BEFORE the statistics prologue so its L2 round trips overlap the first
// HBM round trip. A thread only ever reads slots it filled itself: cp.async.wait_group is the only synchronisation.
constexpr int GN_RING = 8;

SVDX_DEVINL void cp_async16(const void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
SVDX_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
SVDX_DEVINL void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// fold per-channel sums (gn_sum of the producing epilogue) into G group mean / rstd in shared memory; all threads of the
// block take part (block = whole warps). The channel loads are issued together, then reduced.
SVDX_DEVINL void gn_fold_csum(const GnSrc& s, int n, int C, int cpg, int G, float inv_count, float eps, const float* __restrict__ csum1,
                              long long ldc1, const float* __restrict__ csum2, long long ldc2, float* sh_sum, float* sh_sq,
                              float* sh_mean, float* sh_rstd) {
  if (threadIdx.x < 32) { sh_sum[threadIdx.x] = 0.f; sh_sq[threadIdx.x] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  constexpr int NI = 4;                            // channel loads in flight per thread per round
  for (int cb = (threadIdx.x & ~31); cb < C; cb += NI * blockDim.x) {
    float a[NI], b[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int c = cb + i * blockDim.x + lane;
      a[i] = 0.f; b[i] = 0.f;
      if (c < C) {
        const float* base = (c < s.C1) ? (csum1 + (2LL * n) * ldc1 + c) : (csum2 + (2LL * n) * ldc2 + (c - s.C1));
        a[i] = base[0];
        b[i] = base[(c < s.C1) ? ldc1 : ldc2];
      }
    }
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int c = cb + i * blockDim.x + lane;
      if (cb + i * blockDim.x >= C) break;         // warp-uniform
      const int g = (c < C) ? c / cpg : -1;
      float av = a[i], bv = b[i];
      // segmented suffix sum over runs of equal group (non-decreasing across lanes), one shared atomic per run
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float a2 = __shfl_down_sync(0xffffffffu, av, o), b2 = __shfl_down_sync(0xffffffffu, bv, o);
        const int g2 = __shfl_down_sync(0xffffffffu, g, o);
        if (lane + o < 32 && g2 == g) { av += a2; bv += b2; }
      }
      const int gprev = __shfl_up_sync(0xffffffffu, g, 1);
      if (g >= 0 && (lane == 0 || gprev != g)) { atomicAdd(&sh_sum[g], av); atomicAdd(&sh_sq[g], bv); }
    }
  }
  __syncthreads();
  if (threadIdx.x < G) {
    const float m = sh_sum[threadIdx.x] * inv_count;
    const float var = fmaxf(sh_sq[threadIdx.x] * inv_count - m * m, 0.f);
    sh_mean[threadIdx.x] = m;
    sh_rstd[threadIdx.x] = rsqrtf(var + eps);
  }
  __syncthreads();
}

// y = [silu](x * scale + shift), statistics folded from the per-channel sums (mean / rstd are OUTPUTS, published by CTA
// x == 0 of the slab). block = RL row lanes x CV channel vectors, padded to warps.
__global__ void __launch_bounds__(GNV_MAX_THREADS, 2) gn_apply_ring(GnSrc s, int rows, int rows_per_cta, int RL, int G, float eps, float inv_count,
                                                                     const float* __restrict__ csum1, long long ldc1,
                                                                     const float* __restrict__ csum2, long long ldc2, float* mean, float* rstd,
                                                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                     int fuse_silu, bf16* __restrict__ y, long long ldy, float* __restrict__ ab_out) {
  __shared__ float sh_sum[32], sh_sq[32], sh_mean[32], sh_rstd[32];
  const int C = s.C1 + s.C2;
  const int CV = C / 8;
  const int cpg = C / G;
  const int n = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(r0 + rows_per_cta, rows);
  const int cv = threadIdx.x % CV, rl = threadIdx.x / CV;
  const bool active = rl < RL;
  const int c0 = cv * 8;
  const int bd = blockDim.x;
  uint4* ring = gn_ring_smem + threadIdx.x;
  const long long base = (long long)n * rows;
  const int rr = r0 + rl;
  const int nit = (active && rr < r1) ? (r1 - rr + RL - 1) / RL : 0;
  const bool first = c0 < s.C1;
  const long long ld = first ? s.ldx : s.ldx2;
  const bf16* px = (first ? (s.x + c0) : (s.x2 + (c0 - s.C1))) + (base + rr) * ld;
  const long long step = (long long)RL * ld;
#pragma unroll
  for (int d = 0; d < GN_RING; ++d) {
    if (d < nit) cp_async16(&ring[d * bd], px + d * step);
    cp_async_commit();
  }
  float gm[8], bt[8];
  if (active) {
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + c0), g1 = *reinterpret_cast<const float4*>(gamma + c0 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(beta + c0), b1 = *reinterpret_cast<const float4*>(beta + c0 + 4);
    gm[0] = g0.x; gm[1] = g0.y; gm[2] = g0.z; gm[3] = g0.w; gm[4] = g1.x; gm[5] = g1.y; gm[6] = g1.z; gm[7] = g1.w;
    bt[0] = b0.x; bt[1] = b0.y; bt[2] = b0.z; bt[3] = b0.w; bt[4] = b1.x; bt[5] = b1.y; bt[6] = b1.z; bt[7] = b1.w;
  }
  gn_fold_csum(s, n, C, cpg, G, inv_count, eps, csum1, ldc1, csum2, ldc2, sh_sum, sh_sq, sh_mean, sh_rstd);
  if (blockIdx.x == 0 && threadIdx.x < G) { mean[n * G + threadIdx.x] = sh_mean[threadIdx.x]; rstd[n * G + threadIdx.x] = sh_rstd[threadIdx.x]; }
  if (nit == 0) return;
  float sc[8], sh[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int g = (c0 + k) / cpg;
    sc[k] = sh_rstd[g] * gm[k];
    sh[k] = bt[k] - sh_mean[g] * sc[k];
  }
  if (ab_out && blockIdx.x == 0 && rl == 0) {
    // the per-channel scale / shift of this slab, for the backward sums fused into the consumer's dgrad epilogue (gnb_ab)
    float* a = ab_out + (2LL * n) * C + c0;
    *reinterpret_cast<float4*>(a) = make_float4(sc[0], sc[1], sc[2], sc[3]);
    *reinterpret_cast<float4*>(a + 4) = make_float4(sc[4], sc[5], sc[6], sc[7]);
    *reinterpret_cast<float4*>(a + C) = make_float4(sh[0], sh[1], sh[2], sh[3]);
    *reinterpret_cast<float4*>(a + C + 4) = make_float4(sh[4], sh[5], sh[6], sh[7]);
  }
  bf16* py = y + (base + rr) * ldy + c0;
  const long long ystep = (long long)RL * ldy;
  for (int i = 0; i < nit; ++i) {
    cp_async_wait<GN_RING - 1>();
    const int slot = (i & (GN_RING - 1)) * bd;
    const uint4 u = ring[slot];
    const uint32_t in[4] = {u.x, u.y, u.z, u.w};
    uint32_t out[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 v = unpack_bf16x2(in[k]);
      float a = fmaf(v.x, sc[2 * k], sh[2 * k]), b = fmaf(v.y, sc[2 * k + 1], sh[2 * k + 1]);
      if (fuse_silu) { a = silu_f(a); b = silu_f(b); }
      out[k] = pack_bf16x2(a, b);
    }
    *reinterpret_cast<uint4*>(py + i * ystep) = make_uint4(out[0], out[1], out[2], out[3]);
    if (i + GN_RING < nit) cp_async16(&ring[slot], px + (i + GN_RING) * step);
    cp_async_commit();
  }
}

// backward pass 1 on raw moments: sum e, sum e*x per (slab, channel) into sum[outer][2][C] (the gnb_sum layout),
// e = dy * silu'(x * scale + shift) with scale / shift read from the ab table the apply kernel wrote (only when fuse_silu).
// gn_bwd_fused_ring folds them into the group sums and derives dgamma / dbeta from them. The row-lane reduction reuses
// the ring memory, free once every thread has left its loop.
__global__ void __launch_bounds__(GNV_MAX_THREADS, 1) gn_bwd_sums_ring(GnSrc s, const bf16* __restrict__ dy, long long lddy, int rows, int rows_per_cta,
                                                                        int RL, const float* __restrict__ ab, int fuse_silu, float* sum) {
  const int C = s.C1 + s.C2;
  const int CV = C / 8;
  const int n = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(r0 + rows_per_cta, rows);
  const int cv = threadIdx.x % CV, rl = threadIdx.x / CV;
  const bool active = rl < RL;
  const int c0 = cv * 8;
  const int bd = blockDim.x;
  uint4* ringx = gn_ring_smem + threadIdx.x;
  uint4* ringd = ringx + GN_RING * bd;
  const long long base = (long long)n * rows;
  const int rr = r0 + rl;
  const int nit = (active && rr < r1) ? (r1 - rr + RL - 1) / RL : 0;
  const bool first = c0 < s.C1;
  const long long ld = first ? s.ldx : s.ldx2;
  const bf16* px = (first ? (s.x + c0) : (s.x2 + (c0 - s.C1))) + (base + rr) * ld;
  const bf16* pd = dy + (base + rr) * lddy + c0;
  const long long step = (long long)RL * ld, dstep = (long long)RL * lddy;
#pragma unroll
  for (int d = 0; d < GN_RING; ++d) {
    if (d < nit) { cp_async16(&ringx[d * bd], px + d * step); cp_async16(&ringd[d * bd], pd + d * dstep); }
    cp_async_commit();
  }
  float S[8], SX[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { S[k] = SX[k] = 0.f; }
  if (nit > 0) {
    float A[8], B[8];
    if (fuse_silu) {
      const float* a = ab + (2LL * n) * C + c0;
#pragma unroll
      for (int k = 0; k < 8; ++k) { A[k] = a[k]; B[k] = a[C + k]; }
    }
    for (int i = 0; i < nit; ++i) {
      cp_async_wait<GN_RING - 1>();
      const int slot = (i & (GN_RING - 1)) * bd;
      const uint4 ux = ringx[slot], ud = ringd[slot];
      const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 v = unpack_bf16x2(wx[k]), d = unpack_bf16x2(wd[k]);
        float e0 = d.x, e1 = d.y;
        if (fuse_silu) {
          e0 *= silu_grad_f(fmaf(v.x, A[2 * k], B[2 * k]));
          e1 *= silu_grad_f(fmaf(v.y, A[2 * k + 1], B[2 * k + 1]));
        }
        S[2 * k] += e0; S[2 * k + 1] += e1;
        SX[2 * k] = fmaf(e0, v.x, SX[2 * k]); SX[2 * k + 1] = fmaf(e1, v.y, SX[2 * k + 1]);
      }
      if (i + GN_RING < nit) { cp_async16(&ringx[slot], px + (i + GN_RING) * step); cp_async16(&ringd[slot], pd + (i + GN_RING) * dstep); }
      cp_async_commit();
    }
  }
  __syncthreads();
  float* part = reinterpret_cast<float*>(gn_ring_smem);
  if (active) gn_csum_put(part, C, rl, c0, S, SX);
  __syncthreads();
  gn_csum_flush(part, C, RL, sum + (2LL * n) * C, C);
}

// ------------------------------------------------------------------ LayerNorm

// forward: a warp takes RPW rows at a time (grid-stride), lane l owns the 8-channel vectors l, l + 32, ... of each (16-byte loads
// and stores; all RPW rows' loads are issued before any arithmetic so that a warp keeps RPW * C * 2 bytes in flight); the
// rows stay in registers between the two statistics passes and the normalisation
template <int NJ, int RPW>
__global__ void __launch_bounds__(256, SVDX_LN_MINB) ln_fwd_kernel(const bf16* __restrict__ x, long long ldx, int rows, int C,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                     bf16* __restrict__ y, long long ldy, float* __restrict__ mean, float* __restrict__ rstd,
                                                     const float* __restrict__ addvec, int add_div, bf16* __restrict__ xsum, long long ldxs) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int CV = C / 8;
  const float invC = 1.0f / C;
  for (int row0 = warp0 * RPW; row0 < rows; row0 += nwarps * RPW) {
    uint4 u[RPW][NJ];
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      if (row0 + r < rows) {
        const bf16* xr = x + (long long)(row0 + r) * ldx;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int v = lane + 32 * j;
          if (v < CV) u[r][j] = *reinterpret_cast<const uint4*>(xr + v * 8);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      const int row = row0 + r;
      if (row >= rows) break;                     // warp-uniform
      const float* av = addvec ? addvec + (long long)(row / add_div) * C : nullptr;
      float f[NJ][8];
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) {
          const uint32_t w[4] = {u[r][j].x, u[r][j].y, u[r][j].z, u[r][j].w};
#pragma unroll
          for (int k = 0; k < 4; ++k) { const float2 a = unpack_bf16x2(w[k]); f[j][2 * k] = a.x; f[j][2 * k + 1] = a.y; }
          if (av) {
            // x + addvec is rounded to bf16 (it is the residual stream value the reference materialises)
            const float4 a0 = *reinterpret_cast<const float4*>(av + v * 8), a1 = *reinterpret_cast<const float4*>(av + v * 8 + 4);
            const float ad[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            uint32_t pk[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              pk[k] = pack_bf16x2(f[j][2 * k] + ad[2 * k], f[j][2 * k + 1] + ad[2 * k + 1]);
              const float2 r2 = unpack_bf16x2(pk[k]);
              f[j][2 * k] = r2.x; f[j][2 * k + 1] = r2.y;
            }
            *reinterpret_cast<uint4*>(xsum + (long long)row * ldxs + v * 8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) sum += f[j][k];
        }
      }
      sum = warp_sum(sum);
      const float m = sum * invC;
      float sq = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) {
#pragma unroll
          for (int k = 0; k < 8; ++k) { const float d = f[j][k] - m; sq = fmaf(d, d, sq); }
        }
      }
      sq = warp_sum(sq);
      const float rs = rsqrtf(sq * invC + eps);
      if (lane == 0) { mean[row] = m; rstd[row] = rs; }
      bf16* yr = y + (long long)row * ldy;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + v * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
          const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, bt[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
          uint32_t pk[4];
#pragma unroll
          for (int k = 0; k < 4; ++k)
            pk[k] = pack_bf16x2(fmaf((f[j][2 * k] - m) * rs, gm[2 * k], bt[2 * k]), fmaf((f[j][2 * k + 1] - m) * rs, gm[2 * k + 1], bt[2 * k + 1]));
          *reinterpret_cast<uint4*>(yr + v * 8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        }
      }
    }
  }
}

// backward: each warp walks rows (grid-stride); a lane owns the 8-channel vectors lane, lane+32, ... (16-byte loads of x,
// dy and the residual gradient in flight together), keeps its dgamma/dbeta partials in registers, and the block reduces
// them through shared memory before one atomic per channel.
// dx = rstd*(gamma*dy - mean(gamma*dy) - xhat*mean(gamma*dy*xhat)) [+ dres]
template <int NJ, bool DG>
__global__ void __launch_bounds__(256, SVDX_LN_MINB) ln_bwd_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ dy, long long lddy,
                                                     int rows, int C, const float* __restrict__ gamma, const float* __restrict__ mean,
                                                     const float* __restrict__ rstd, bf16* __restrict__ dx, long long lddx,
                                                     const bf16* __restrict__ dres, long long lddres, float* dgamma, float* dbeta) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int CV = C / 8;
  float gm[NJ][8], dg[NJ][8], db[NJ][8];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int v = lane + 32 * j;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      gm[j][k] = (v < CV) ? gamma[v * 8 + k] : 0.f;
      dg[j][k] = 0.f;
      db[j][k] = 0.f;
    }
  }
  const float invC = 1.0f / C;
  for (int row = warp0; row < rows; row += nwarps) {
    const bf16* xr = x + (long long)row * ldx;
    const bf16* dr = dy + (long long)row * lddy;
    uint4 ux[NJ], ud[NJ], ur[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        ux[j] = *reinterpret_cast<const uint4*>(xr + v * 8);
        ud[j] = *reinterpret_cast<const uint4*>(dr + v * 8);
        if (dres) ur[j] = *reinterpret_cast<const uint4*>(dres + (long long)row * lddres + v * 8);
      }
    }
    const float m = mean[row], rs = rstd[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        const uint32_t wx[4] = {ux[j].x, ux[j].y, ux[j].z, ux[j].w}, wd[4] = {ud[j].x, ud[j].y, ud[j].z, ud[j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(wx[k]), d = unpack_bf16x2(wd[k]);
          const float x0 = (a.x - m) * rs, x1 = (a.y - m) * rs;
          const float g0 = d.x * gm[j][2 * k], g1 = d.y * gm[j][2 * k + 1];
          s1 += g0 + g1;
          s2 += g0 * x0 + g1 * x1;
          if (DG) {
            dg[j][2 * k] += d.x * x0; dg[j][2 * k + 1] += d.y * x1;
            db[j][2 * k] += d.x; db[j][2 * k + 1] += d.y;
          }
        }
      }
    }
    s1 = warp_sum(s1) * invC;
    s2 = warp_sum(s2) * invC;
    bf16* oxr = dx + (long long)row * lddx;
    // second pass recomputes xhat / g*gamma from the raw vectors still in registers (cheaper than keeping them live)
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        const uint32_t wx[4] = {ux[j].x, ux[j].y, ux[j].z, ux[j].w}, wd[4] = {ud[j].x, ud[j].y, ud[j].z, ud[j].w};
        float o[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(wx[k]), d = unpack_bf16x2(wd[k]);
          const float x0 = (a.x - m) * rs, x1 = (a.y - m) * rs;
          o[2 * k] = rs * (d.x * gm[j][2 * k] - s1 - x0 * s2);
          o[2 * k + 1] = rs * (d.y * gm[j][2 * k + 1] - s1 - x1 * s2);
        }
        if (dres) {
          const uint32_t wr[4] = {ur[j].x, ur[j].y, ur[j].z, ur[j].w};
#pragma unroll
          for (int k = 0; k < 4; ++k) { const float2 r2 = unpack_bf16x2(wr[k]); o[2 * k] += r2.x; o[2 * k + 1] += r2.y; }
        }
        *reinterpret_cast<uint4*>(oxr + v * 8) =
            make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
      }
    }
  }
  if (DG) {
    __shared__ float sh_g[256 * NJ], sh_b[256 * NJ];
    for (int i = threadIdx.x; i < 256 * NJ; i += blockDim.x) { sh_g[i] = 0.f; sh_b[i] = 0.f; }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { atomicAdd(&sh_g[v * 8 + k], dg[j][k]); atomicAdd(&sh_b[v * 8 + k], db[j][k]); }
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      atomicAdd(&dgamma[i], sh_g[i]);
      atomicAdd(&dbeta[i], sh_b[i]);
    }
  }
}

// backward pass 2, from the per-channel sums of pass 1 (svdx_tapgemm's gnb_sum, or gn_bwd_sums_ring): every CTA folds
// S_c = sum e, SX_c = sum e*x of its slab into s1_g = sum_c gamma_c S_c and sx_g = sum_c gamma_c SX_c (C values from L2), then
// streams rows: dx = rstd*(e*gamma - t1 - xhat*t2) [+ dres] = e*A - x*P + Q [+ dres], A = rstd*gamma, P = rstd^2 * t2,
// Q = mean*P - rstd*t1 (t1 = s1 / count, t2 = rstd * (sx - mean * s1) / count). CTA x == 0 of a slab also emits
// dgamma_c += rstd (SX_c - mean S_c), dbeta_c += S_c.
template <bool DRES>
__global__ void __launch_bounds__(GNV_MAX_THREADS, 1) gn_bwd_fused_ring(GnSrc s, const bf16* __restrict__ dy, long long lddy, int rows, int rows_per_cta,
                                                                         int RL, int G, const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                         const float* __restrict__ gamma, const float* __restrict__ beta, int fuse_silu,
                                                                         const float* __restrict__ csum, float inv_count, bf16* __restrict__ dx,
                                                                         long long lddx, bf16* __restrict__ dx2, long long lddx2,
                                                                         const bf16* __restrict__ dres, long long lddres, float* dgamma, float* dbeta) {
  __shared__ float sh_s1[32], sh_sx[32];
  const int C = s.C1 + s.C2;
  const int CV = C / 8;
  const int cpg = C / G;
  const int n = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(r0 + rows_per_cta, rows);
  const int cv = threadIdx.x % CV, rl = threadIdx.x / CV;
  const int c0 = cv * 8;
  const int bd = blockDim.x;
  const int rr = r0 + rl;
  const int nit = (rl < RL && rr < r1) ? (r1 - rr + RL - 1) / RL : 0;
  uint4* ringx = gn_ring_smem + threadIdx.x;
  uint4* ringd = ringx + GN_RING * bd;
  uint4* ringr = ringd + GN_RING * bd;
  const long long base = (long long)n * rows;
  const bool first = c0 < s.C1;
  const long long ld = first ? s.ldx : s.ldx2;
  const bf16* px = (first ? (s.x + c0) : (s.x2 + (c0 - s.C1))) + (base + rr) * ld;
  const bf16* pd = dy + (base + rr) * lddy + c0;
  const bf16* pr = DRES ? dres + (base + rr) * lddres + c0 : nullptr;
  const long long step = (long long)RL * ld, dstep = (long long)RL * lddy, rstep = (long long)RL * lddres;
#pragma unroll
  for (int d = 0; d < GN_RING; ++d) {
    if (d < nit) {
      cp_async16(&ringx[d * bd], px + d * step);
      cp_async16(&ringd[d * bd], pd + d * dstep);
      if (DRES) cp_async16(&ringr[d * bd], pr + d * rstep);
    }
    cp_async_commit();
  }
  // ---- fold the channel sums of this slab (weighted by gamma) into the G groups
  if (threadIdx.x < 32) { sh_s1[threadIdx.x] = 0.f; sh_sx[threadIdx.x] = 0.f; }
  __syncthreads();
  {
    const int lane = threadIdx.x & 31;
    const float* cs = csum + (2LL * n) * C;
    constexpr int NI = 4;
    for (int cb = (threadIdx.x & ~31); cb < C; cb += NI * bd) {
      float a[NI], b[NI], w[NI];
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        const int c = cb + i * bd + lane;
        a[i] = 0.f; b[i] = 0.f; w[i] = 0.f;
        if (c < C) { a[i] = cs[c]; b[i] = cs[C + c]; w[i] = gamma[c]; }
      }
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        const int c = cb + i * bd + lane;
        if (cb + i * bd >= C) break;               // warp-uniform
        const int g = (c < C) ? c / cpg : -1;
        if (dgamma && blockIdx.x == 0 && c < C) {
          const float mu = mean[n * G + g], rs = rstd[n * G + g];
          atomicAdd(&dgamma[c], rs * (b[i] - mu * a[i]));
          atomicAdd(&dbeta[c], a[i]);
        }
        float av = a[i] * w[i], bv = b[i] * w[i];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float a2 = __shfl_down_sync(0xffffffffu, av, o), b2 = __shfl_down_sync(0xffffffffu, bv, o);
          const int g2 = __shfl_down_sync(0xffffffffu, g, o);
          if (lane + o < 32 && g2 == g) { av += a2; bv += b2; }
        }
        const int gprev = __shfl_up_sync(0xffffffffu, g, 1);
        if (g >= 0 && (lane == 0 || gprev != g)) { atomicAdd(&sh_s1[g], av); atomicAdd(&sh_sx[g], bv); }
      }
    }
  }
  __syncthreads();
  if (nit == 0) return;
  float A[8], B[8], P[8], Q[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int g = (c0 + k) / cpg;
    const float mu = mean[n * G + g], rs = rstd[n * G + g];
    const float t1 = sh_s1[g] * inv_count, t2 = rs * (sh_sx[g] - mu * sh_s1[g]) * inv_count;
    A[k] = rs * gamma[c0 + k];
    B[k] = beta[c0 + k] - mu * A[k];
    P[k] = rs * rs * t2;
    Q[k] = mu * P[k] - rs * t1;
  }
  const long long ols = first ? lddx : lddx2;
  bf16* po = (first ? (dx + c0) : (dx2 + (c0 - s.C1))) + (base + rr) * ols;
  const long long ostep = (long long)RL * ols;
  for (int i = 0; i < nit; ++i) {
    cp_async_wait<GN_RING - 1>();
    const int slot = (i & (GN_RING - 1)) * bd;
    const uint4 ux = ringx[slot], ud = ringd[slot];
    uint4 ur = make_uint4(0u, 0u, 0u, 0u);
    if (DRES) ur = ringr[slot];
    const uint32_t in[4] = {ux.x, ux.y, ux.z, ux.w}, din[4] = {ud.x, ud.y, ud.z, ud.w}, rin[4] = {ur.x, ur.y, ur.z, ur.w};
    uint32_t out[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 v = unpack_bf16x2(in[k]), d = unpack_bf16x2(din[k]);
      float e0 = d.x, e1 = d.y;
      if (fuse_silu) {
        e0 *= silu_grad_f(fmaf(v.x, A[2 * k], B[2 * k]));
        e1 *= silu_grad_f(fmaf(v.y, A[2 * k + 1], B[2 * k + 1]));
      }
      float o0 = fmaf(e0, A[2 * k], fmaf(-v.x, P[2 * k], Q[2 * k]));
      float o1 = fmaf(e1, A[2 * k + 1], fmaf(-v.y, P[2 * k + 1], Q[2 * k + 1]));
      if (DRES) { const float2 r2 = unpack_bf16x2(rin[k]); o0 += r2.x; o1 += r2.y; }
      out[k] = pack_bf16x2(o0, o1);
    }
    *reinterpret_cast<uint4*>(po + i * ostep) = make_uint4(out[0], out[1], out[2], out[3]);
    if (i + GN_RING < nit) {
      cp_async16(&ringx[slot], px + (i + GN_RING) * step);
      cp_async16(&ringd[slot], pd + (i + GN_RING) * dstep);
      if (DRES) cp_async16(&ringr[slot], pr + (i + GN_RING) * rstep);
    }
    cp_async_commit();
  }
}

// ------------------------------------------------------------------ LayerNorm, cp.async ring variants
// A warp streams its rows (grid-stride) through a private ring of D row slots per tensor in shared memory, filled by
// cp.async; lane l copies and later reads the 16-byte vectors l, l + 32, ... of a row, so the x / dy / dres rings need no
// cross-lane synchronisation. Rows are re-read from shared memory in each pass instead of being held in registers, which
// keeps the register count independent of C, and D rows per tensor per warp are in flight at all times.
template <int NJ> struct LnRing {
  static constexpr int D_FWD = NJ <= 2 ? 8 : (NJ == 3 ? 4 : 2);
  static constexpr int W_BWD = NJ <= 3 ? 16 : 8;
  static constexpr int D_BWD = NJ <= 2 ? 4 : 2;
};

template <int NJ>
__global__ void __launch_bounds__(256, 2) ln_fwd_ring(const bf16* __restrict__ x, long long ldx, int rows, int C, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, bf16* __restrict__ y, long long ldy,
                                                       float* __restrict__ mean, float* __restrict__ rstd, const float* __restrict__ addvec,
                                                       int add_div, bf16* __restrict__ xsum, long long ldxs) {
  constexpr int D = LnRing<NJ>::D_FWD;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int gw = blockIdx.x * (blockDim.x >> 5) + wib;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int CV = C / 8;
  const float invC = 1.0f / C;
  uint4* ring = gn_ring_smem + (size_t)wib * D * CV;
  const int nit = gw < rows ? (rows - gw + nwarps - 1) / nwarps : 0;
  const bf16* px = x + (long long)gw * ldx;
  const long long step = (long long)nwarps * ldx;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (d < nit) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) cp_async16(&ring[d * CV + v], px + d * step + v * 8);
      }
    }
    cp_async_commit();
  }
  float gm[NJ][8], bt[NJ][8];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int v = lane + 32 * j;
    if (v < CV) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + v * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
      gm[j][0] = g0.x; gm[j][1] = g0.y; gm[j][2] = g0.z; gm[j][3] = g0.w; gm[j][4] = g1.x; gm[j][5] = g1.y; gm[j][6] = g1.z; gm[j][7] = g1.w;
      bt[j][0] = b0.x; bt[j][1] = b0.y; bt[j][2] = b0.z; bt[j][3] = b0.w; bt[j][4] = b1.x; bt[j][5] = b1.y; bt[j][6] = b1.z; bt[j][7] = b1.w;
    }
  }
  for (int i = 0; i < nit; ++i) {
    cp_async_wait<D - 1>();
    const int row = gw + i * nwarps;
    uint4* slot = ring + (i & (D - 1)) * CV;
    float sum = 0.f;
    if (addvec) {
      // x + addvec rounded to bf16 is the residual-stream value the reference materialises: written out and back into the slot
      const float* av = addvec + (long long)(row / add_div) * C;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) {
          const uint4 u = slot[v];
          const uint32_t w[4] = {u.x, u.y, u.z, u.w};
          const float4 a0 = *reinterpret_cast<const float4*>(av + v * 8), a1 = *reinterpret_cast<const float4*>(av + v * 8 + 4);
          const float ad[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
          uint32_t pk[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 a = unpack_bf16x2(w[k]);
            pk[k] = pack_bf16x2(a.x + ad[2 * k], a.y + ad[2 * k + 1]);
            const float2 r2 = unpack_bf16x2(pk[k]);
            sum += r2.x + r2.y;
          }
          const uint4 o = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          slot[v] = o;
          *reinterpret_cast<uint4*>(xsum + (long long)row * ldxs + v * 8) = o;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) {
          const uint4 u = slot[v];
          const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) { const float2 a = unpack_bf16x2(w[k]); sum += a.x + a.y; }
        }
      }
    }
    const float m = warp_sum(sum) * invC;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        const uint4 u = slot[v];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(w[k]);
          const float d0 = a.x - m, d1 = a.y - m;
          sq = fmaf(d0, d0, sq); sq = fmaf(d1, d1, sq);
        }
      }
    }
    const float rs = rsqrtf(warp_sum(sq) * invC + eps);
    if (lane == 0) { mean[row] = m; rstd[row] = rs; }
    bf16* yr = y + (long long)row * ldy;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        const uint4 u = slot[v];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
        uint32_t pk[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(w[k]);
          pk[k] = pack_bf16x2(fmaf((a.x - m) * rs, gm[j][2 * k], bt[j][2 * k]), fmaf((a.y - m) * rs, gm[j][2 * k + 1], bt[j][2 * k + 1]));
        }
        *reinterpret_cast<uint4*>(yr + v * 8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
      }
    }
    if (i + D < nit) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int v = lane + 32 * j;
        if (v < CV) cp_async16(&slot[v], px + (i + D) * step + v * 8);
      }
    }
    cp_async_commit();
  }
}

template <int NJ, bool DG, bool DRES>
__global__ void __launch_bounds__(LnRing<NJ>::W_BWD * 32, 1) ln_bwd_ring(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ dy, long long lddy,
                                                                          int rows, int C, const float* __restrict__ gamma, const float* __restrict__ mean,
                                                                          const float* __restrict__ rstd, bf16* __restrict__ dx, long long lddx,
                                                                          const bf16* __restrict__ dres, long long lddres, float* dgamma, float* dbeta) {
  constexpr int D = LnRing<NJ>::D_BWD;
  constexpr int W = LnRing<NJ>::W_BWD;
  __shared__ float sh_stat[W * D * 2];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int gw = blockIdx.x * W + wib;
  const int nwarps = gridDim.x * W;
  const int CV = C / 8;
  const float invC = 1.0f / C;
  uint4* ringx = gn_ring_smem + (size_t)wib * D * CV;
  uint4* ringd = ringx + (size_t)W * D * CV;
  uint4* ringr = ringd + (size_t)W * D * CV;
  float* stat = sh_stat + wib * D * 2;
  const int nit = gw < rows ? (rows - gw + nwarps - 1) / nwarps : 0;
  const bf16* px = x + (long long)gw * ldx;
  const bf16* pd = dy + (long long)gw * lddy;
  const bf16* pr = DRES ? dres + (long long)gw * lddres : nullptr;
  const long long step = (long long)nwarps * ldx, dstep = (long long)nwarps * lddy, rstep = (long long)nwarps * lddres;
  auto fill = [&](int it, int d) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        cp_async16(&ringx[d * CV + v], px + it * step + v * 8);
        cp_async16(&ringd[d * CV + v], pd + it * dstep + v * 8);
        if (DRES) cp_async16(&ringr[d * CV + v], pr + it * rstep + v * 8);
      }
    }
    if (lane < 2) {
      const float* src = (lane == 0 ? mean : rstd) + gw + (long long)it * nwarps;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(&stat[d * 2 + lane])), "l"(src) : "memory");
    }
  };
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (d < nit) fill(d, d);
    cp_async_commit();
  }
  float gm[NJ][8], dg[NJ][8], db[NJ][8];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int v = lane + 32 * j;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      gm[j][k] = (v < CV) ? gamma[v * 8 + k] : 0.f;
      dg[j][k] = 0.f;
      db[j][k] = 0.f;
    }
  }
  for (int i = 0; i < nit; ++i) {
    cp_async_wait<D - 1>();
    __syncwarp();                                   // the row statistics were copied by lanes 0 / 1
    const int row = gw + i * nwarps;
    const int d = i & (D - 1);
    const float m = stat[d * 2], rs = stat[d * 2 + 1];
    const uint4* sx = ringx + d * CV;
    const uint4* sd = ringd + d * CV;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        const uint4 ux = sx[v], ud = sd[v];
        const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(wx[k]), g = unpack_bf16x2(wd[k]);
          const float x0 = (a.x - m) * rs, x1 = (a.y - m) * rs;
          const float g0 = g.x * gm[j][2 * k], g1 = g.y * gm[j][2 * k + 1];
          s1 += g0 + g1;
          s2 += g0 * x0 + g1 * x1;
          if (DG) {
            dg[j][2 * k] += g.x * x0; dg[j][2 * k + 1] += g.y * x1;
            db[j][2 * k] += g.x; db[j][2 * k + 1] += g.y;
          }
        }
      }
    }
    s1 = warp_sum(s1) * invC;
    s2 = warp_sum(s2) * invC;
    bf16* oxr = dx + (long long)row * lddx;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
        const uint4 ux = sx[v], ud = sd[v];
        const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
        float o[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(wx[k]), g = unpack_bf16x2(wd[k]);
          const float x0 = (a.x - m) * rs, x1 = (a.y - m) * rs;
          o[2 * k] = rs * (g.x * gm[j][2 * k] - s1 - x0 * s2);
          o[2 * k + 1] = rs * (g.y * gm[j][2 * k + 1] - s1 - x1 * s2);
        }
        if (DRES) {
          const uint4 ur = (ringr + d * CV)[v];
          const uint32_t wr[4] = {ur.x, ur.y, ur.z, ur.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) { const float2 r2 = unpack_bf16x2(wr[k]); o[2 * k] += r2.x; o[2 * k + 1] += r2.y; }
        }
        *reinterpret_cast<uint4*>(oxr + v * 8) =
            make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
      }
    }
    __syncwarp();                                   // every lane has read the statistics slot before it is refilled
    if (i + D < nit) fill(i + D, d);
    cp_async_commit();
  }
  if (DG) {
    // block reduction through the (now idle) ring memory: 2 * C floats <= W * D * CV * 16 bytes
    __syncthreads();
    float* sh_g = reinterpret_cast<float*>(gn_ring_smem);
    float* sh_b = sh_g + C;
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sh_g[i] = 0.f;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int v = lane + 32 * j;
      if (v < CV) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { atomicAdd(&sh_g[v * 8 + k], dg[j][k]); atomicAdd(&sh_b[v * 8 + k], db[j][k]); }
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      atomicAdd(&dgamma[i], sh_g[i]);
      atomicAdd(&dbeta[i], sh_b[i]);
    }
  }
}

}  // namespace svdx

using namespace svdx;

// block = (C/8 channel vectors) x (row lanes) threads, ~8 CTAs per SM; each thread streams a multiple of 4 rows (4
// independent 16-byte loads in flight), and at least 16: a CTA's 2 * C channel-sum reds then stay small next to the rows it
// read (fewer rows made the reds the bottleneck at C = 640 / 1280)
static void gn_vec_config(int C, int outer, int rows, int& threads, int& rows_per_cta) {
  const int CV = C / 8;
  int RL = 256 / CV;
  if (RL < 1) RL = 1;
  threads = CV * RL;
  const long long want_ctas = 8LL * svdx_num_sms();
  long long chunks = (want_ctas + outer - 1) / outer;
  if (chunks < 1) chunks = 1;
  rows_per_cta = (int)((rows + chunks - 1) / chunks);
  const int quantum = GN_RIF * RL;
  rows_per_cta = ((rows_per_cta + quantum - 1) / quantum) * quantum;
  if (rows_per_cta < 4 * quantum) rows_per_cta = 4 * quantum;
}

// ring kernels: block = RL x CV threads padded to whole warps, ~2 CTAs per SM (each thread then walks enough rows to amortise
// the ring fill; in-step A/B on one box: 2 <= 3 < 1 < 4 < 6), dynamic shared memory GN_RING slots x 16 B x threads per
// streamed tensor
static void gn_ring_config(int C, int outer, int rows, int& threads, int& RL, int& rows_per_cta) {
  const int CV = C / 8;
  RL = 256 / CV;
  if (RL < 1) RL = 1;
  threads = (CV * RL + 31) & ~31;
  const long long want_ctas = 2LL * svdx_num_sms();
  long long chunks = (want_ctas + outer - 1) / outer;
  if (chunks < 1) chunks = 1;
  rows_per_cta = (int)((rows + chunks - 1) / chunks);
  rows_per_cta = ((rows_per_cta + RL - 1) / RL) * RL;
  if (rows_per_cta < RL) rows_per_cta = RL;
}
constexpr int GN_RING_SMEM_MAX = 3 * GN_RING * GNV_MAX_THREADS * 16;   // 196608 B
template <typename K>
static void gn_ring_attr(K kernel, bool* done) {
  const int slot = svdx_device_slot();
  if (!done[slot]) { cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GN_RING_SMEM_MAX); done[slot] = true; }
}

// the one or two bf16 sources: whole 8-channel vectors, at most GNV_MAX_THREADS of them per row, 16-byte aligned rows
static int gn_check(int C1, int C2, int64_t ldx, int64_t ldx2, const void* x, const void* x2) {
  const int C = C1 + C2;
  if (!x || C <= 0 || C % 8 || C1 % 8 || C2 % 8 || C / 8 > GNV_MAX_THREADS) return 1;
  if (C2 > 0 && !x2) return 1;
  if (ldx % 8 || (C2 > 0 && ldx2 % 8)) return 1;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (x2 && (reinterpret_cast<uintptr_t>(x2) & 15))) return 1;
  return 0;
}

// a row stride shorter than the row overlaps the next row; one row has no stride to check (torch gives a size-1 dim any stride)
static bool short_ld(long long ld, long long width, long long nrows) { return nrows > 1 && ld < width; }

// the row strides of the one or two sources (the kernels address row r of slab n at (n * rows + r) * ld): the violated
// constraint, or nullptr
static const char* gn_ld_error(int C1, int C2, int64_t ldx, int64_t ldx2, long long nrows) {
  if (short_ld(ldx, C1, nrows)) return "ldx < C1";
  if (C2 > 0 && short_ld(ldx2, C2, nrows)) return "ldx2 < C2";
  return nullptr;
}

static int norm_fail(const char* entry, const char* what) {
  char msg[96];
  snprintf(msg, sizeof(msg), "%s: %s", entry, what);
  return svdx_fail(SVDX_E_BADARG, msg);
}

// at most 32 groups (the consumers' shared-memory group tables) of an even number of channels
static int gn_groups_bad(int C, int G) { return G <= 0 || G > 32 || C % G || (C / G) % 2; }

extern "C" int svdx_groupnorm_sums(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2, int32_t outer,
                                   int32_t rows, float* sums, int64_t ld, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (gn_check(C1, C2, ldx, ldx2, x, x2) || outer <= 0 || rows <= 0 || !sums || (reinterpret_cast<uintptr_t>(sums) & 15) || ld < C1 + C2 || ld % 4)
    return svdx_fail(SVDX_E_BADARG, "groupnorm_sums: bad arguments");
  if (const char* e = gn_ld_error(C1, C2, ldx, ldx2, (long long)outer * rows)) return norm_fail("groupnorm_sums", e);
  GnSrc s{reinterpret_cast<const bf16*>(x), ldx, C1, reinterpret_cast<const bf16*>(x2), ldx2, C2};
  int threads, rpc;
  gn_vec_config(C1 + C2, outer, rows, threads, rpc);
  // row-lane partials: 2 moments x 8 channels per thread
  gn_sums<<<dim3((rows + rpc - 1) / rpc, outer), threads, (size_t)threads * 16 * sizeof(float), st>>>(s, rows, rpc, sums, ld);
  SVDX_CHECK_LAUNCH("groupnorm_sums");
  return SVDX_OK;
}

extern "C" int svdx_groupnorm_apply_fused(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2, int32_t outer,
                                          int32_t rows, int32_t num_groups, float eps, const float* csum1, int64_t ldc1,
                                          const float* csum2, int64_t ldc2, float* mean, float* rstd, const float* gamma,
                                          const float* beta, int32_t fuse_silu, void* y, int64_t ldy, float* ab_out, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (gn_check(C1, C2, ldx, ldx2, x, x2) || gn_groups_bad(C1 + C2, num_groups) || !y || ldy % 8 || (reinterpret_cast<uintptr_t>(y) & 15) || !mean ||
      !rstd || !gamma || !beta || (reinterpret_cast<uintptr_t>(gamma) & 15) || (reinterpret_cast<uintptr_t>(beta) & 15) ||
      (ab_out && ((reinterpret_cast<uintptr_t>(ab_out) & 15))) || !csum1 || ldc1 < C1 || (C2 > 0 && (!csum2 || ldc2 < C2)) || outer <= 0 || rows <= 0)
    return svdx_fail(SVDX_E_BADARG, "groupnorm_apply_fused: bad arguments");
  const long long M = (long long)outer * rows;
  if (const char* e = gn_ld_error(C1, C2, ldx, ldx2, M)) return norm_fail("groupnorm_apply_fused", e);
  if (short_ld(ldy, C1 + C2, M)) return norm_fail("groupnorm_apply_fused", "ldy < C1 + C2");
  GnSrc s{reinterpret_cast<const bf16*>(x), ldx, C1, reinterpret_cast<const bf16*>(x2), ldx2, C2};
  static bool attr[SVDX_MAX_DEVICES] = {false};
  gn_ring_attr(gn_apply_ring, attr);
  int threads, RL, rpc;
  gn_ring_config(C1 + C2, outer, rows, threads, RL, rpc);
  const float inv = 1.0f / ((float)rows * (float)((C1 + C2) / num_groups));
  gn_apply_ring<<<dim3((rows + rpc - 1) / rpc, outer), threads, (size_t)GN_RING * threads * 16, st>>>(
      s, rows, rpc, RL, num_groups, eps, inv, csum1, ldc1, csum2, ldc2, mean, rstd, gamma, beta, fuse_silu, reinterpret_cast<bf16*>(y), ldy, ab_out);
  SVDX_CHECK_LAUNCH("groupnorm_apply_fused");
  return SVDX_OK;
}

extern "C" int svdx_groupnorm_bwd_sums(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2, const void* dy,
                                       int64_t lddy, int32_t outer, int32_t rows, const float* ab, int32_t fuse_silu, float* sums, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (gn_check(C1, C2, ldx, ldx2, x, x2) || !dy || lddy % 8 || (reinterpret_cast<uintptr_t>(dy) & 15) || (fuse_silu && !ab) || !sums ||
      (reinterpret_cast<uintptr_t>(sums) & 15) || outer <= 0 || rows <= 0)
    return svdx_fail(SVDX_E_BADARG, "groupnorm_bwd_sums: bad arguments");
  const long long M = (long long)outer * rows;
  if (const char* e = gn_ld_error(C1, C2, ldx, ldx2, M)) return norm_fail("groupnorm_bwd_sums", e);
  if (short_ld(lddy, C1 + C2, M)) return norm_fail("groupnorm_bwd_sums", "lddy < C");
  GnSrc s{reinterpret_cast<const bf16*>(x), ldx, C1, reinterpret_cast<const bf16*>(x2), ldx2, C2};
  static bool attr[SVDX_MAX_DEVICES] = {false};
  gn_ring_attr(gn_bwd_sums_ring, attr);
  int threads, RL, rpc;
  gn_ring_config(C1 + C2, outer, rows, threads, RL, rpc);
  gn_bwd_sums_ring<<<dim3((rows + rpc - 1) / rpc, outer), threads, (size_t)2 * GN_RING * threads * 16, st>>>(
      s, reinterpret_cast<const bf16*>(dy), lddy, rows, rpc, RL, ab, fuse_silu, sums);
  SVDX_CHECK_LAUNCH("groupnorm_bwd_sums");
  return SVDX_OK;
}

extern "C" int svdx_groupnorm_bwd_fused(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2, const void* dy,
                                        int64_t lddy, int32_t outer, int32_t rows, int32_t num_groups, const float* mean, const float* rstd,
                                        const float* gamma, const float* beta, int32_t fuse_silu, const float* csum, void* dx, int64_t lddx,
                                        void* dx2, int64_t lddx2, float* dgamma, float* dbeta, const void* dres, int64_t lddres,
                                        void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (gn_check(C1, C2, ldx, ldx2, x, x2) || gn_groups_bad(C1 + C2, num_groups) || !dy || lddy % 8 || (reinterpret_cast<uintptr_t>(dy) & 15) || !dx ||
      lddx % 8 ||
      (reinterpret_cast<uintptr_t>(dx) & 15) || (C2 > 0 && (!dx2 || lddx2 % 8 || (reinterpret_cast<uintptr_t>(dx2) & 15))) || !csum || !mean || !rstd ||
      !gamma || !beta || (dgamma && !dbeta) || (dres && (C2 > 0 || lddres % 8 || (reinterpret_cast<uintptr_t>(dres) & 15))) || outer <= 0 || rows <= 0)
    return svdx_fail(SVDX_E_BADARG, "groupnorm_bwd_fused: bad arguments");
  const long long M = (long long)outer * rows;
  if (const char* e = gn_ld_error(C1, C2, ldx, ldx2, M)) return norm_fail("groupnorm_bwd_fused", e);
  if (short_ld(lddy, C1 + C2, M)) return norm_fail("groupnorm_bwd_fused", "lddy < C");
  if (short_ld(lddx, C1, M)) return norm_fail("groupnorm_bwd_fused", "lddx < C1");
  if (C2 > 0 && short_ld(lddx2, C2, M)) return norm_fail("groupnorm_bwd_fused", "lddx2 < C2");
  if (dres && short_ld(lddres, C1 + C2, M)) return norm_fail("groupnorm_bwd_fused", "lddres < C");
  GnSrc s{reinterpret_cast<const bf16*>(x), ldx, C1, reinterpret_cast<const bf16*>(x2), ldx2, C2};
  static bool a1[SVDX_MAX_DEVICES] = {false}, a2[SVDX_MAX_DEVICES] = {false};
  gn_ring_attr(gn_bwd_fused_ring<true>, a1);
  gn_ring_attr(gn_bwd_fused_ring<false>, a2);
  int threads, RL, rpc;
  gn_ring_config(C1 + C2, outer, rows, threads, RL, rpc);
  dim3 grid((rows + rpc - 1) / rpc, outer);
  const size_t slab = (size_t)GN_RING * threads * 16;
  const float inv = 1.0f / ((float)rows * (float)((C1 + C2) / num_groups));
  const bf16* dyb = reinterpret_cast<const bf16*>(dy);
  if (dres)
    gn_bwd_fused_ring<true><<<grid, threads, 3 * slab, st>>>(s, dyb, lddy, rows, rpc, RL, num_groups, mean, rstd, gamma, beta, fuse_silu, csum, inv,
                                                             reinterpret_cast<bf16*>(dx), lddx, reinterpret_cast<bf16*>(dx2), lddx2,
                                                             reinterpret_cast<const bf16*>(dres), lddres, dgamma, dbeta);
  else
    gn_bwd_fused_ring<false><<<grid, threads, 2 * slab, st>>>(s, dyb, lddy, rows, rpc, RL, num_groups, mean, rstd, gamma, beta, fuse_silu, csum, inv,
                                                              reinterpret_cast<bf16*>(dx), lddx, reinterpret_cast<bf16*>(dx2), lddx2, nullptr, 0, dgamma,
                                                              dbeta);
  SVDX_CHECK_LAUNCH("groupnorm_bwd_fused");
  return SVDX_OK;
}

template <int NJ, int RPW>
static void ln_fwd_launch(const void* x, int64_t ldx, int rows, int C, const float* g, const float* b, float eps, void* y, int64_t ldy,
                          float* mean, float* rstd, const float* addvec, int add_div, void* xsum, int64_t ldxs, cudaStream_t st) {
  int ctas = (rows + 8 * RPW - 1) / (8 * RPW);     // 8 warps per CTA, RPW rows in flight per warp, grid-stride over rows
  const int cap = svdx_num_sms() * 8;
  if (ctas > cap) ctas = cap;
  ln_fwd_kernel<NJ, RPW><<<ctas, 256, 0, st>>>(reinterpret_cast<const bf16*>(x), ldx, rows, C, g, b, eps, reinterpret_cast<bf16*>(y), ldy, mean, rstd,
                                          addvec, add_div, reinterpret_cast<bf16*>(xsum), ldxs);
}

static int ln_ring_cps(const char* name, int dflt) {
  const char* e = getenv(name);
  return (e && atoi(e) > 0) ? atoi(e) : dflt;
}

template <int NJ>
static void ln_fwd_ring_launch(const void* x, int64_t ldx, int rows, int C, const float* g, const float* b, float eps, void* y, int64_t ldy,
                               float* mean, float* rstd, const float* addvec, int add_div, void* xsum, int64_t ldxs, cudaStream_t st) {
  static bool attr[SVDX_MAX_DEVICES] = {false};
  gn_ring_attr(ln_fwd_ring<NJ>, attr);
  static int cps = ln_ring_cps("SVDX_LN_RING_CPS", 3);
  int ctas = (rows + 7) / 8;
  const int cap = svdx_num_sms() * cps;
  if (ctas > cap) ctas = cap;
  const size_t smem = (size_t)8 * LnRing<NJ>::D_FWD * (C / 8) * 16;
  ln_fwd_ring<NJ><<<ctas, 256, smem, st>>>(reinterpret_cast<const bf16*>(x), ldx, rows, C, g, b, eps, reinterpret_cast<bf16*>(y), ldy, mean, rstd,
                                           addvec, add_div, reinterpret_cast<bf16*>(xsum), ldxs);
}

template <int NJ, bool DG, bool DRES>
static void ln_bwd_ring_launch2(const void* x, int64_t ldx, const void* dy, int64_t lddy, int rows, int C, const float* g, const float* mean,
                                const float* rstd, void* dx, int64_t lddx, const void* dres, int64_t lddres, float* dgamma, float* dbeta,
                                cudaStream_t st) {
  static bool attr[SVDX_MAX_DEVICES] = {false};
  gn_ring_attr(ln_bwd_ring<NJ, DG, DRES>, attr);
  constexpr int W = LnRing<NJ>::W_BWD;
  int ctas = (rows + W - 1) / W;
  const int cap = svdx_num_sms();
  if (ctas > cap) ctas = cap;
  const size_t smem = (size_t)(DRES ? 3 : 2) * W * LnRing<NJ>::D_BWD * (C / 8) * 16;
  ln_bwd_ring<NJ, DG, DRES><<<ctas, W * 32, smem, st>>>(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(dy), lddy, rows, C, g, mean,
                                                        rstd, reinterpret_cast<bf16*>(dx), lddx, reinterpret_cast<const bf16*>(dres), lddres, dgamma,
                                                        dbeta);
}
template <int NJ>
static void ln_bwd_ring_launch(const void* x, int64_t ldx, const void* dy, int64_t lddy, int rows, int C, const float* g, const float* mean,
                               const float* rstd, void* dx, int64_t lddx, const void* dres, int64_t lddres, float* dgamma, float* dbeta,
                               cudaStream_t st) {
  if (dgamma) {
    if (dres) ln_bwd_ring_launch2<NJ, true, true>(x, ldx, dy, lddy, rows, C, g, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
    else ln_bwd_ring_launch2<NJ, true, false>(x, ldx, dy, lddy, rows, C, g, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
  } else {
    if (dres) ln_bwd_ring_launch2<NJ, false, true>(x, ldx, dy, lddy, rows, C, g, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
    else ln_bwd_ring_launch2<NJ, false, false>(x, ldx, dy, lddy, rows, C, g, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
  }
}

extern "C" int svdx_layernorm_fwd(const void* x, int64_t ldx, int32_t rows, int32_t C, const float* gamma, const float* beta, float eps,
                                  void* y, int64_t ldy, float* mean, float* rstd, const float* addvec, int32_t add_div, void* xsum,
                                  int64_t ldxs, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (!x || !y || !gamma || !beta || !mean || !rstd || rows <= 0 || C <= 0 || C % 8 || C > 2560 || ldx % 8 || ldy % 8 ||
      (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(gamma) & 15) ||
      (reinterpret_cast<uintptr_t>(beta) & 15) ||
      (addvec && (!xsum || add_div <= 0 || ldxs % 8 || (reinterpret_cast<uintptr_t>(addvec) & 15) || (reinterpret_cast<uintptr_t>(xsum) & 15))))
    return svdx_fail(SVDX_E_BADARG, "layernorm_fwd: bad arguments (C %% 8, C <= 2560, 16-byte aligned rows and vectors)");
  if (short_ld(ldx, C, rows)) return norm_fail("layernorm_fwd", "ldx < C");
  if (short_ld(ldy, C, rows)) return norm_fail("layernorm_fwd", "ldy < C");
  if (addvec && short_ld(ldxs, C, rows)) return norm_fail("layernorm_fwd", "ldxs < C");
  const int nj = (C / 8 + 31) / 32;
  if (nj <= 5) {
    if (nj <= 1) ln_fwd_ring_launch<1>(x, ldx, rows, C, gamma, beta, eps, y, ldy, mean, rstd, addvec, add_div, xsum, ldxs, st);
    else if (nj <= 2) ln_fwd_ring_launch<2>(x, ldx, rows, C, gamma, beta, eps, y, ldy, mean, rstd, addvec, add_div, xsum, ldxs, st);
    else if (nj <= 3) ln_fwd_ring_launch<3>(x, ldx, rows, C, gamma, beta, eps, y, ldy, mean, rstd, addvec, add_div, xsum, ldxs, st);
    else ln_fwd_ring_launch<5>(x, ldx, rows, C, gamma, beta, eps, y, ldy, mean, rstd, addvec, add_div, xsum, ldxs, st);
    SVDX_CHECK_LAUNCH("layernorm_fwd");
    return SVDX_OK;
  }
  ln_fwd_launch<10, 1>(x, ldx, rows, C, gamma, beta, eps, y, ldy, mean, rstd, addvec, add_div, xsum, ldxs, st);   // 1280 < C <= 2560: rows in registers
  SVDX_CHECK_LAUNCH("layernorm_fwd");
  return SVDX_OK;
}

template <int NJ>
static void ln_bwd_launch(const void* x, int64_t ldx, const void* dy, int64_t lddy, int rows, int C, const float* g, const float* mean,
                          const float* rstd, void* dx, int64_t lddx, const void* dres, int64_t lddres, float* dgamma, float* dbeta,
                          cudaStream_t st) {
  int ctas = (rows + 7) / 8;
  // with parameter gradients: few CTAs (the dgamma/dbeta atomics contend per address); without: fill the SMs with
  // resident warps, one row in flight per warp
  const int cap = svdx_num_sms() * (dgamma ? 2 : 8);
  if (ctas > cap) ctas = cap;
  if (dgamma)
    ln_bwd_kernel<NJ, true><<<ctas, 256, 0, st>>>(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(dy), lddy, rows, C, g, mean,
                                                  rstd, reinterpret_cast<bf16*>(dx), lddx, reinterpret_cast<const bf16*>(dres), lddres, dgamma, dbeta);
  else
    ln_bwd_kernel<NJ, false><<<ctas, 256, 0, st>>>(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(dy), lddy, rows, C, g, mean,
                                                   rstd, reinterpret_cast<bf16*>(dx), lddx, reinterpret_cast<const bf16*>(dres), lddres, dgamma, dbeta);
}

extern "C" int svdx_layernorm_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, int32_t rows, int32_t C, const float* gamma,
                                  const float* mean, const float* rstd, void* dx, int64_t lddx, const void* dres, int64_t lddres,
                                  float* dgamma, float* dbeta, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (!x || !dy || !dx || !gamma || !mean || !rstd || rows <= 0 || C <= 0 || C % 8 || C > 2560 || ldx % 8 || lddy % 8 || lddx % 8 ||
      (dgamma && !dbeta) || (dres && lddres % 8))
    return svdx_fail(SVDX_E_BADARG, "layernorm_bwd: bad arguments (C %% 8, C <= 2560, 16-byte aligned rows)");
  const int nj = (C / 8 + 31) / 32;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(dy) & 15) || (reinterpret_cast<uintptr_t>(dx) & 15) ||
      (dres && (reinterpret_cast<uintptr_t>(dres) & 15)))
    return svdx_fail(SVDX_E_BADARG, "layernorm_bwd: x / dy / dx / dres must be 16-byte aligned");
  if (short_ld(ldx, C, rows)) return norm_fail("layernorm_bwd", "ldx < C");
  if (short_ld(lddy, C, rows)) return norm_fail("layernorm_bwd", "lddy < C");
  if (short_ld(lddx, C, rows)) return norm_fail("layernorm_bwd", "lddx < C");
  if (dres && short_ld(lddres, C, rows)) return norm_fail("layernorm_bwd", "lddres < C");
  if (nj <= 5) {
    if (nj <= 1) ln_bwd_ring_launch<1>(x, ldx, dy, lddy, rows, C, gamma, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
    else if (nj <= 2) ln_bwd_ring_launch<2>(x, ldx, dy, lddy, rows, C, gamma, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
    else if (nj <= 3) ln_bwd_ring_launch<3>(x, ldx, dy, lddy, rows, C, gamma, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
    else ln_bwd_ring_launch<5>(x, ldx, dy, lddy, rows, C, gamma, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);
    SVDX_CHECK_LAUNCH("layernorm_bwd");
    return SVDX_OK;
  }
  ln_bwd_launch<10>(x, ldx, dy, lddy, rows, C, gamma, mean, rstd, dx, lddx, dres, lddres, dgamma, dbeta, st);   // 1280 < C <= 2560
  SVDX_CHECK_LAUNCH("layernorm_bwd");
  return SVDX_OK;
}
