// Short-sequence attention (S <= 32 tokens, head_dim 64): the temporal self-attention of the SVD UNet
// (TemporalBasicTransformerBlock.attn1 [D], one sequence of T = 14 / 25 frames per pixel and head), forward and backward.
//
// Why a second kernel family: this op is HBM-bound, not tensor-bound — per (pixel, head) it does 2 x 14 x 14 x 64 MACs on
// 3 x 14 x 128 bytes of input (0.64 GFLOP over 92 MB at the 40x64 level: 7 FLOP/byte). The wgmma kernel of attention.cu
// packs 8 pixel sequences into one 128-row tile and masks 7/8 of the 128 x 128 scores; every CTA pays barrier set-up and
// three TMA round trips for 6 KB of useful data. A CUDA-core version (one lane per query, K / V rows broadcast from shared
// memory) is shared-memory-bound.
// This version gives each WARP one (sequence, head) and uses warp-level tensor-core MMAs (mma.sync m16n8k16, bf16 x bf16 ->
// fp32) on 16-row tiles: the scores of a 14-token sequence are ONE 16 x 16 tile, the whole forward is 16 MMAs, the backward 56.
// The tiny MMA work leaves the kernel bound by its loads: Q / K / V (/ dO) head slices are staged with coalesced 16-byte loads
// into padded bf16 shared-memory tiles, fragments come from conflict-free 32-bit loads (K-major operands) or ldmatrix.trans
// (key-major V / K / dO / Q as the k x n operand), results go back through shared memory as full 128-byte rows.
// Token addressing follows the SvdxAttn descriptor (outer / inner / token strides): the strided "frames of one pixel" gather
// needs no permute. (the wgmma kernels work on 64-row warpgroup tiles of 128-row CTAs and need mbarrier plumbing per CTA; for 16-row problems the
// warp-level MMA is the tensor-core path that fits, and the op's roofline is HBM either way.)
//
// forward : S = Q K^T * scale -> softmax over the S keys -> O = P V,  lse = log sum exp (natural log, as attention.cu)
// backward: P recomputed; dP = dO V^T; delta = sum_s P dP; dS = P (dP - delta) * scale; dQ = dS K;
//           transposed tiles S^T = K Q^T, dP^T = V dO^T recomputed with the row statistics read back from shared memory:
//           dV = P^T dO, dK = dS^T Q. No atomics.
#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"
#include <stdlib.h>

namespace svdx {

constexpr float AS_LOG2E = 1.4426950408889634f;
constexpr int AS_ROW = 72;            // bf16 elements per staged row (64 + 8 pad: conflict-free fragment loads, 16 B aligned rows)
constexpr int AS_WARPS = 4;

struct SmallAttnP {
  const bf16 *q, *k, *v, *dout;
  bf16 *out, *dq, *dk, *dv;
  long long ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv;
  long long nseq;
  int heads, S, inner;
  long long outer_stride, inner_stride, tok_stride;
  float scale;
  float* lse;
};

SVDX_DEVINL void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// two transposed 8x8 b16 matrices: the (k x n) operand fragment of a [k rows][n cols] row-major shared-memory tile
SVDX_DEVINL void ldmatrix_x2_trans(uint32_t& b0, uint32_t& b1, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(addr));
}
SVDX_DEVINL uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// stage one [S][64] bf16 head slice (rows = tokens of one sequence) into a [16 * NT][AS_ROW] tile; rows >= S are zero
template <int NT>
SVDX_DEVINL void as_stage(const bf16* __restrict__ src, long long ld, long long tok0, long long tok_stride, int S, int lane, uint32_t tile) {
#pragma unroll
  for (int it = 0; it < 4 * NT; ++it) {
    const int r = it * 4 + (lane >> 3), c = lane & 7;
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (r < S) u = __ldg(reinterpret_cast<const uint4*>(src + (tok0 + (long long)r * tok_stride) * ld + c * 8));
    st_shared_v4(tile + (uint32_t)(r * AS_ROW + c * 8) * 2u, u.x, u.y, u.z, u.w);
  }
}
// write a [16 * NT][64] bf16 result tile (staged in shared memory) back as full 128-byte rows, rows < S only
template <int NT>
SVDX_DEVINL void as_unstage(bf16* __restrict__ dst, long long ld, long long tok0, long long tok_stride, int S, int lane, uint32_t tile) {
#pragma unroll
  for (int it = 0; it < 4 * NT; ++it) {
    const int r = it * 4 + (lane >> 3), c = lane & 7;
    if (r < S) {
      uint4 u;
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "r"(tile + (uint32_t)(r * AS_ROW + c * 8) * 2u));
      *reinterpret_cast<uint4*>(dst + (tok0 + (long long)r * tok_stride) * ld + c * 8) = u;
    }
  }
}

// acc[mt][nt] (16 x 8 tiles) = A[rows][64] * B[cols][64]^T for two K-major tiles (QK^T, dO V^T, K Q^T, V dO^T)
template <int NT>
SVDX_DEVINL void as_kmajor_product(float (&acc)[NT][2 * NT][4], uint32_t tA, uint32_t tB, int g, int tq) {
#pragma unroll
  for (int mt = 0; mt < NT; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t b[2 * NT][2];
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt) {
      const uint32_t base = tB + (uint32_t)((nt * 8 + g) * AS_ROW + ks * 16 + 2 * tq) * 2u;
      b[nt][0] = lds32(base);
      b[nt][1] = lds32(base + 16);
    }
#pragma unroll
    for (int mt = 0; mt < NT; ++mt) {
      uint32_t a[4];
      const uint32_t base = tA + (uint32_t)((mt * 16 + g) * AS_ROW + ks * 16 + 2 * tq) * 2u;
      a[0] = lds32(base);
      a[1] = lds32(base + 8 * AS_ROW * 2);
      a[2] = lds32(base + 16);
      a[3] = lds32(base + 8 * AS_ROW * 2 + 16);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt) mma_bf16_16816(acc[mt][nt], a, b[nt][0], b[nt][1]);
    }
  }
}

// out[mt][dn] (16 x 8 tiles over the 64 head dims) = P[rows][16 * NT] (fp32 accumulator layout, rounded to bf16) * B[16 * NT][64]
// with B a row-major [k][64] tile read through ldmatrix.trans (P V, dS K, P^T dO, dS^T Q)
template <int NT>
SVDX_DEVINL void as_pv_product(float (&out)[NT][8][4], const float (&p)[NT][2 * NT][4], uint32_t tB, int lane) {
#pragma unroll
  for (int mt = 0; mt < NT; ++mt)
#pragma unroll
    for (int dn = 0; dn < 8; ++dn)
#pragma unroll
      for (int i = 0; i < 4; ++i) out[mt][dn][i] = 0.f;
#pragma unroll
  for (int kk = 0; kk < NT; ++kk) {
    uint32_t a[NT][4];
#pragma unroll
    for (int mt = 0; mt < NT; ++mt) {
      a[mt][0] = pack_bf16x2(p[mt][2 * kk][0], p[mt][2 * kk][1]);
      a[mt][1] = pack_bf16x2(p[mt][2 * kk][2], p[mt][2 * kk][3]);
      a[mt][2] = pack_bf16x2(p[mt][2 * kk + 1][0], p[mt][2 * kk + 1][1]);
      a[mt][3] = pack_bf16x2(p[mt][2 * kk + 1][2], p[mt][2 * kk + 1][3]);
    }
#pragma unroll
    for (int dn = 0; dn < 8; ++dn) {
      uint32_t b0, b1;
      // lanes 0-7: rows 16kk + 0..7 of column block dn; lanes 8-15: rows 16kk + 8..15 (the other lanes' addresses are ignored)
      ldmatrix_x2_trans(b0, b1, tB + (uint32_t)((kk * 16 + (lane & 15)) * AS_ROW + dn * 8) * 2u);
#pragma unroll
      for (int mt = 0; mt < NT; ++mt) mma_bf16_16816(out[mt][dn], a[mt], b0, b1);
    }
  }
}

// accumulator tiles -> bf16 [rows][64] shared-memory tile (rows g / g + 8 of each 16-row block, column pairs 2 tq)
template <int NT>
SVDX_DEVINL void as_store_tile(uint32_t tile, const float (&o)[NT][8][4], const float (&s)[NT][2], int g, int tq) {
#pragma unroll
  for (int mt = 0; mt < NT; ++mt)
#pragma unroll
    for (int dn = 0; dn < 8; ++dn) {
      const uint32_t base = tile + (uint32_t)((mt * 16 + g) * AS_ROW + dn * 8 + 2 * tq) * 2u;
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(base), "r"(pack_bf16x2(o[mt][dn][0] * s[mt][0], o[mt][dn][1] * s[mt][0])) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(base + 8 * AS_ROW * 2), "r"(pack_bf16x2(o[mt][dn][2] * s[mt][1], o[mt][dn][3] * s[mt][1])) : "memory");
    }
}

SVDX_DEVINL float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
SVDX_DEVINL float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// row softmax of score tiles in the accumulator layout: s[mt][nt][0..1] = row g, [2..3] = row g + 8; key = nt * 8 + 2 tq + {0, 1}.
// On return s holds the NORMALISED probabilities; m2 (log2-domain row maximum) and l (row sum) are returned per (mt, row half).
template <int NT>
SVDX_DEVINL void as_softmax(float (&s)[NT][2 * NT][4], float qs, int S, int tq, float (&m2)[NT][2], float (&l)[NT][2]) {
#pragma unroll
  for (int mt = 0; mt < NT; ++mt) {
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const bool ok = nt * 8 + 2 * tq + i < S;
        s[mt][nt][i] = ok ? s[mt][nt][i] * qs : -INFINITY;
        s[mt][nt][2 + i] = ok ? s[mt][nt][2 + i] * qs : -INFINITY;
        mx0 = fmaxf(mx0, s[mt][nt][i]);
        mx1 = fmaxf(mx1, s[mt][nt][2 + i]);
      }
    mx0 = quad_max(mx0);
    mx1 = quad_max(mx1);
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        s[mt][nt][i] = exp2_fast(s[mt][nt][i] - mx0);
        s[mt][nt][2 + i] = exp2_fast(s[mt][nt][2 + i] - mx1);
        l0 += s[mt][nt][i];
        l1 += s[mt][nt][2 + i];
      }
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int i = 0; i < 2; ++i) { s[mt][nt][i] *= i0; s[mt][nt][2 + i] *= i1; }
    m2[mt][0] = mx0; m2[mt][1] = mx1; l[mt][0] = l0; l[mt][1] = l1;
  }
}

template <int NT>
__global__ void __launch_bounds__(AS_WARPS * 32) attn_small_fwd_kernel(const SmallAttnP p) {
  extern __shared__ __align__(16) uint8_t as_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;
  constexpr uint32_t TILE = 16 * NT * AS_ROW * 2;
  const uint32_t tQ = smem_u32(as_smem) + warp * 3 * TILE, tK = tQ + TILE, tV = tK + TILE;
  const int S = p.S;
  const long long total = p.nseq * p.heads;
  const float qs = p.scale * AS_LOG2E;
  for (long long pi = (long long)blockIdx.x * AS_WARPS + warp; pi < total; pi += (long long)gridDim.x * AS_WARPS) {
    const long long seq = pi / p.heads;
    const int h = (int)(pi - seq * p.heads);
    const long long outer = seq / p.inner;
    const long long tok0 = outer * p.outer_stride + (seq - outer * p.inner) * p.inner_stride;
    as_stage<NT>(p.q + h * 64, p.ldq, tok0, p.tok_stride, S, lane, tQ);
    as_stage<NT>(p.k + h * 64, p.ldk, tok0, p.tok_stride, S, lane, tK);
    as_stage<NT>(p.v + h * 64, p.ldv, tok0, p.tok_stride, S, lane, tV);
    __syncwarp();
    float s[NT][2 * NT][4];
    as_kmajor_product<NT>(s, tQ, tK, g, tq);
    float m2[NT][2], l[NT][2];
    as_softmax<NT>(s, qs, S, tq, m2, l);
    float o[NT][8][4];
    as_pv_product<NT>(o, s, tV, lane);
    __syncwarp();                                   // all fragment reads of tQ are done: reuse it for the output rows
    float one[NT][2];
#pragma unroll
    for (int mt = 0; mt < NT; ++mt) { one[mt][0] = 1.f; one[mt][1] = 1.f; }
    as_store_tile<NT>(tQ, o, one, g, tq);
    if (p.lse && tq == 0) {
#pragma unroll
      for (int mt = 0; mt < NT; ++mt)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int r = mt * 16 + g + 8 * hf;
          if (r < S) p.lse[(tok0 + (long long)r * p.tok_stride) * p.heads + h] = (m2[mt][hf] + log2f(l[mt][hf])) * 0.6931471805599453f;
        }
    }
    __syncwarp();
    as_unstage<NT>(p.out + h * 64, p.ldo, tok0, p.tok_stride, S, lane, tQ);
    __syncwarp();
  }
}

template <int NT>
__global__ void __launch_bounds__(AS_WARPS * 32) attn_small_bwd_kernel(const SmallAttnP p) {
  extern __shared__ __align__(16) uint8_t as_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;
  constexpr uint32_t TILE = 16 * NT * AS_ROW * 2;
  constexpr uint32_t STAT = 16 * NT * 3 * 4;      // per query row: log2-domain max, 1 / l, delta
  const uint32_t tQ = smem_u32(as_smem) + warp * (5 * TILE + STAT), tK = tQ + TILE, tV = tK + TILE, tD = tV + TILE, tO = tD + TILE;
  float* stat = reinterpret_cast<float*>(as_smem + warp * (5 * TILE + STAT) + 5 * TILE);
  const int S = p.S;
  const long long total = p.nseq * p.heads;
  const float qs = p.scale * AS_LOG2E;
  for (long long pi = (long long)blockIdx.x * AS_WARPS + warp; pi < total; pi += (long long)gridDim.x * AS_WARPS) {
    const long long seq = pi / p.heads;
    const int h = (int)(pi - seq * p.heads);
    const long long outer = seq / p.inner;
    const long long tok0 = outer * p.outer_stride + (seq - outer * p.inner) * p.inner_stride;
    as_stage<NT>(p.q + h * 64, p.ldq, tok0, p.tok_stride, S, lane, tQ);
    as_stage<NT>(p.k + h * 64, p.ldk, tok0, p.tok_stride, S, lane, tK);
    as_stage<NT>(p.v + h * 64, p.ldv, tok0, p.tok_stride, S, lane, tV);
    as_stage<NT>(p.dout + h * 64, p.lddo, tok0, p.tok_stride, S, lane, tD);
    __syncwarp();
    // ---- query-major pass: P, dP, delta, dS, dQ = dS K
    {
      float s[NT][2 * NT][4], dp[NT][2 * NT][4];
      as_kmajor_product<NT>(s, tQ, tK, g, tq);
      float m2[NT][2], l[NT][2];
      as_softmax<NT>(s, qs, S, tq, m2, l);
      as_kmajor_product<NT>(dp, tD, tV, g, tq);
#pragma unroll
      for (int mt = 0; mt < NT; ++mt) {
        float d0 = 0.f, d1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
          for (int i = 0; i < 2; ++i) { d0 = fmaf(s[mt][nt][i], dp[mt][nt][i], d0); d1 = fmaf(s[mt][nt][2 + i], dp[mt][nt][2 + i], d1); }
        d0 = quad_sum(d0);
        d1 = quad_sum(d1);
#pragma unroll
        for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            s[mt][nt][i] = s[mt][nt][i] * (dp[mt][nt][i] - d0) * p.scale;              // dS (masked keys: P = 0)
            s[mt][nt][2 + i] = s[mt][nt][2 + i] * (dp[mt][nt][2 + i] - d1) * p.scale;
          }
        if (tq == 0) {
          float* st0 = stat + (mt * 16 + g) * 3;
          st0[0] = m2[mt][0]; st0[1] = 1.0f / l[mt][0]; st0[2] = d0;
          st0[24] = m2[mt][1]; st0[25] = 1.0f / l[mt][1]; st0[26] = d1;                   // row g + 8
        }
      }
      float dq[NT][8][4];
      as_pv_product<NT>(dq, s, tK, lane);
      float one[NT][2];
#pragma unroll
      for (int mt = 0; mt < NT; ++mt) { one[mt][0] = 1.f; one[mt][1] = 1.f; }
      as_store_tile<NT>(tO, dq, one, g, tq);
    }
    __syncwarp();
    as_unstage<NT>(p.dq + h * 64, p.lddq, tok0, p.tok_stride, S, lane, tO);
    __syncwarp();
    // ---- key-major pass: P^T, dS^T from S^T = K Q^T and dP^T = V dO^T with the per-query statistics; dV = P^T dO, dK = dS^T Q
    {
      float st[NT][2 * NT][4], dpt[NT][2 * NT][4];
      as_kmajor_product<NT>(st, tK, tQ, g, tq);       // rows = keys, columns = queries
      as_kmajor_product<NT>(dpt, tV, tD, g, tq);
#pragma unroll
      for (int mt = 0; mt < NT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float* sq = stat + (nt * 8 + 2 * tq + i) * 3;       // statistics of query column nt * 8 + 2 tq + i
            const float pa = exp2_fast(st[mt][nt][i] * qs - sq[0]) * sq[1];
            const float pb = exp2_fast(st[mt][nt][2 + i] * qs - sq[0]) * sq[1];
            st[mt][nt][i] = pa;
            st[mt][nt][2 + i] = pb;
            dpt[mt][nt][i] = pa * (dpt[mt][nt][i] - sq[2]) * p.scale;
            dpt[mt][nt][2 + i] = pb * (dpt[mt][nt][2 + i] - sq[2]) * p.scale;
          }
      float acc[NT][8][4];
      float one[NT][2];
#pragma unroll
      for (int mt = 0; mt < NT; ++mt) { one[mt][0] = 1.f; one[mt][1] = 1.f; }
      as_pv_product<NT>(acc, st, tD, lane);            // dV[key][d] = sum_q P^T[key][q] dO[q][d]
      as_store_tile<NT>(tO, acc, one, g, tq);
      __syncwarp();
      as_unstage<NT>(p.dv + h * 64, p.lddv, tok0, p.tok_stride, S, lane, tO);
      __syncwarp();
      as_pv_product<NT>(acc, dpt, tQ, lane);           // dK[key][d] = sum_q dS^T[key][q] Q[q][d]
      as_store_tile<NT>(tO, acc, one, g, tq);
      __syncwarp();
      as_unstage<NT>(p.dk + h * 64, p.lddk, tok0, p.tok_stride, S, lane, tO);
    }
    __syncwarp();
  }
}

}  // namespace svdx

using namespace svdx;

// eligible: strided short sequences (the temporal attention); env SVDX_ATTN_SMALL=0 routes them back to the wgmma kernels
bool svdx_attention_small_eligible(const SvdxAttn* d) {
  static int on = -1;
  if (on < 0) { const char* e = getenv("SVDX_ATTN_SMALL"); on = (e && e[0] == '0') ? 0 : 1; }
  return on && d && d->inner > 1 && d->S > 0 && d->S <= 32;
}

static int small_fill(const SvdxAttn* d, SmallAttnP& p, bool bwd) {
  if (!d->q || !d->k || !d->v || !d->o) return svdx_fail(SVDX_E_BADARG, "attention(small): null pointer");
  if (d->heads <= 0 || d->nseq <= 0 || d->inner <= 0 || d->nseq % d->inner) return svdx_fail(SVDX_E_BADARG, "attention(small): bad sequence geometry");
  if ((d->ldq % 8) || (d->ldk % 8) || (d->ldv % 8) || (d->ldo % 8)) return svdx_fail(SVDX_E_BADARG, "attention(small): leading dims must be multiples of 8");
  const int64_t cols = (int64_t)d->heads * 64;
  if (d->ldq < cols || d->ldk < cols || d->ldv < cols || d->ldo < cols)
    return svdx_fail(SVDX_E_BADARG, "attention(small): ldq / ldk / ldv / ldo < heads * 64");
  const uintptr_t al = reinterpret_cast<uintptr_t>(d->q) | reinterpret_cast<uintptr_t>(d->k) | reinterpret_cast<uintptr_t>(d->v) | reinterpret_cast<uintptr_t>(d->o);
  if (al & 15) return svdx_fail(SVDX_E_BADARG, "attention(small): operands must be 16 B aligned");
  memset(&p, 0, sizeof(p));
  p.q = reinterpret_cast<const bf16*>(d->q); p.k = reinterpret_cast<const bf16*>(d->k); p.v = reinterpret_cast<const bf16*>(d->v);
  p.out = reinterpret_cast<bf16*>(d->o);
  p.ldq = d->ldq; p.ldk = d->ldk; p.ldv = d->ldv; p.ldo = d->ldo;
  p.nseq = d->nseq; p.heads = d->heads; p.S = d->S; p.inner = d->inner;
  p.outer_stride = d->outer_stride; p.inner_stride = d->inner_stride; p.tok_stride = d->tok_stride;
  p.scale = d->scale; p.lse = d->lse;
  if (bwd) {
    if (!d->dout || !d->dq || !d->dk || !d->dv) return svdx_fail(SVDX_E_BADARG, "attention_bwd(small): null pointer");
    if ((d->lddo % 8) || (d->lddq % 8) || (d->lddk % 8) || (d->lddv % 8)) return svdx_fail(SVDX_E_BADARG, "attention_bwd(small): leading dims");
    if (d->lddo < cols || d->lddq < cols || d->lddk < cols || d->lddv < cols)
      return svdx_fail(SVDX_E_BADARG, "attention_bwd(small): lddo / lddq / lddk / lddv < heads * 64");
    const uintptr_t a2 = reinterpret_cast<uintptr_t>(d->dout) | reinterpret_cast<uintptr_t>(d->dq) | reinterpret_cast<uintptr_t>(d->dk) | reinterpret_cast<uintptr_t>(d->dv);
    if (a2 & 15) return svdx_fail(SVDX_E_BADARG, "attention_bwd(small): operands must be 16 B aligned");
    p.dout = reinterpret_cast<const bf16*>(d->dout); p.lddo = d->lddo;
    p.dq = reinterpret_cast<bf16*>(d->dq); p.dk = reinterpret_cast<bf16*>(d->dk); p.dv = reinterpret_cast<bf16*>(d->dv);
    p.lddq = d->lddq; p.lddk = d->lddk; p.lddv = d->lddv;
  }
  return SVDX_OK;
}

template <typename K>
static int small_launch(K kernel, const SmallAttnP& p, size_t smem, cudaStream_t st, bool* attr_flags, const char* what) {
  const int slot = svdx_device_slot();
  if (!attr_flags[slot]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return svdx_fail_cuda(e, what);
    attr_flags[slot] = true;
  }
  const long long total = p.nseq * p.heads;
  long long ctas = (total + AS_WARPS - 1) / AS_WARPS;
  const long long cap = 16LL * svdx_num_sms();
  if (ctas > cap) ctas = cap;
  kernel<<<(unsigned)ctas, AS_WARPS * 32, smem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return svdx_fail_cuda(e, what);
  return SVDX_OK;
}

int svdx_attention_small_fwd(const SvdxAttn* d, cudaStream_t st) {
  SmallAttnP p;
  int rc = small_fill(d, p, false);
  if (rc) return rc;
  static bool f1[SVDX_MAX_DEVICES] = {false}, f2[SVDX_MAX_DEVICES] = {false};
  if (d->S <= 16) return small_launch(attn_small_fwd_kernel<1>, p, (size_t)AS_WARPS * 3 * 16 * AS_ROW * 2, st, f1, "attention_fwd(small)");
  return small_launch(attn_small_fwd_kernel<2>, p, (size_t)AS_WARPS * 3 * 32 * AS_ROW * 2, st, f2, "attention_fwd(small)");
}

int svdx_attention_small_bwd(const SvdxAttn* d, cudaStream_t st) {
  SmallAttnP p;
  int rc = small_fill(d, p, true);
  if (rc) return rc;
  static bool f1[SVDX_MAX_DEVICES] = {false}, f2[SVDX_MAX_DEVICES] = {false};
  if (d->S <= 16) return small_launch(attn_small_bwd_kernel<1>, p, (size_t)AS_WARPS * (5 * 16 * AS_ROW * 2 + 16 * 3 * 4), st, f1, "attention_bwd(small)");
  return small_launch(attn_small_bwd_kernel<2>, p, (size_t)AS_WARPS * (5 * 32 * AS_ROW * 2 + 32 * 3 * 4), st, f2, "attention_bwd(small)");
}
