// Scaled-dot-product attention (head_dim 64, no mask), forward and backward, on wgmma (sm_90a).
//
// Replaces AttnProcessor2_0 -> F.scaled_dot_product_attention [D: diffusers models/attention_processor.py]
// for BasicTransformerBlock.attn1 (spatial, S = H*W per frame) and
// TemporalBasicTransformerBlock.attn1 (temporal, S = T per pixel) of the SVD UNet
// (reference: src/unet_spatio_temporal_condition.py:170-233).
//
// Layout: q/k/v/o are column slices of token-major [tokens][ld] bf16 matrices (channels-last
// activations), head h = columns [64h, 64h+64). One 128-row tile holds G interleaved sequences
// x RT = 128/G tokens (tile row r -> sequence r % G, token r / G); spatial attention uses G = 1,
// temporal attention packs G = 8 neighbouring pixels (T <= 16) so the tensor-core tile is full and
// the strided token rows are gathered by ONE 4-D TMA box. Cross-sequence score entries are masked.
//
// Every kernel: one TMA producer warp and two consumer warpgroups; warpgroup g owns rows [64g, 64g + 64) of the tile.
// Scores are computed 64 columns at a time into wgmma register fragments, the element-wise work runs on those
// registers, and the bf16 probabilities / score gradients feed the next wgmma directly as register A operands.
//   forward  : S = Q K^T -> online softmax (exp2) -> O += P V (V as MN-major B operand)
//   backward : bwd_dq  (CTA per query tile, loops key tiles):  dQ += dS K
//              bwd_dkv (CTA per key tile, loops query tiles):  dV += P^T dO, dK += dS^T Q
//              with P = exp(scale*S - lse) recomputed, dS = P o (dP - delta) * scale.
#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"

namespace svdx {

constexpr int AT_THREADS = 288;   // two consumer warpgroups (warps 0..7) + the TMA producer (warp 8)
constexpr int AT_PRODUCER = 8;
constexpr int AT_CONSUMER_WARPS = 8;
constexpr int TILE_BYTES = 128 * 64 * 2;  // one [128 rows][64 cols] bf16 operand tile, 16 KB
constexpr float LOG2E = 1.4426950408889634f;

struct AttnKParams {
  CUtensorMap tq, tk, tv, tdo;  // 4-D maps: (col, inner, token, outer), box (64, G, RT, 1)
  int heads, S, G, RT, inner_groups, tiles, gshift, gmask;
  long long outer_stride, inner_stride, tok_stride;
  float scale;
  bf16* o; long long ldo;
  float* lse;     // [tokens][heads]
  float* delta;   // [tokens][heads]
  bf16* dq; long long lddq;
  bf16* dk; long long lddk;
  bf16* dv; long long lddv;
};

struct RowInfo {
  long long token;  // global token row
  int g;            // sequence slot inside the tile
  bool valid;
};

SVDX_DEVINL RowInfo row_info(const AttnKParams& p, int r, int tile, int outer, int inner0) {
  RowInfo ri;
  const int t = tile * p.RT + (r >> p.gshift);
  ri.g = r & p.gmask;
  ri.valid = t < p.S;
  ri.token = (long long)outer * p.outer_stride + (long long)(inner0 + ri.g) * p.inner_stride + (long long)t * p.tok_stride;
  return ri;
}

SVDX_DEVINL float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// [64 rows x 64 cols] (=) A[64 rows x 64] * B[64 rows x 64]^T, both K-major 128B-swizzled tiles of 128-byte rows; committed,
// not waited for
SVDX_DEVINL void mma_abt64(float (&d)[32], uint32_t a_rows, uint32_t b_rows) {
  const uint64_t a = make_smem_desc_sw128(a_rows, 16, 1024), b = make_smem_desc_sw128(b_rows, 16, 1024);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_ss_n64<0, 0>(d, a + 2 * ks, b + 2 * ks, ks > 0 ? 1u : 0u);
  wgmma_commit();
}
// acc[64 x 64] += P[64 x 64] (a D fragment, rounded to bf16) * B[64 rows x 64 cols] (rows = the contraction, MN-major);
// committed, not waited for
SVDX_DEVINL void mma_pb64(float (&acc)[32], const float (&p)[32], uint32_t b_rows) {
  const uint64_t b = make_smem_desc_sw128(b_rows, 8192, 1024);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    wgmma_rs_n64_tb(acc, pack_bf16x2(p[8 * ks], p[8 * ks + 1]), pack_bf16x2(p[8 * ks + 2], p[8 * ks + 3]),
                    pack_bf16x2(p[8 * ks + 4], p[8 * ks + 5]), pack_bf16x2(p[8 * ks + 6], p[8 * ks + 7]), b + (2048 >> 4) * ks, 1u);
  wgmma_commit();
}
// column (inside a 64-column fragment) of D-fragment register i of this lane; its row is row_lo + 8 * frag_hi(i)
SVDX_DEVINL int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }
SVDX_DEVINL int frag_hi(int i) { return (i >> 1) & 1; }
SVDX_DEVINL float quad_max(float v) { return fmaxf(fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1)), __shfl_xor_sync(0xffffffffu, fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1)), 2)); }
SVDX_DEVINL float quad_sum(float v) { v += __shfl_xor_sync(0xffffffffu, v, 1); return v + __shfl_xor_sync(0xffffffffu, v, 2); }

// the 32 bf16 values of a D fragment of rows row_lo / row_lo + 8, scaled by inv[hi], to 64 consecutive columns of two rows
SVDX_DEVINL void store_frag_rows(bf16* row_lo, bf16* row_hi, const float (&d)[32], float inv_lo, float inv_hi, int lane) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = 8 * j + 2 * (lane & 3);
    if (row_lo) *reinterpret_cast<uint32_t*>(row_lo + c) = pack_bf16x2(d[4 * j] * inv_lo, d[4 * j + 1] * inv_lo);
    if (row_hi) *reinterpret_cast<uint32_t*>(row_hi + c) = pack_bf16x2(d[4 * j + 2] * inv_hi, d[4 * j + 3] * inv_hi);
  }
}

SVDX_DEVINL void decode_block(const AttnKParams& p, int& tile, int& head, int& outer, int& inner0) {
  tile = blockIdx.x;
  head = blockIdx.y;
  outer = blockIdx.z / p.inner_groups;
  inner0 = (blockIdx.z % p.inner_groups) * p.G;
}

// a consumer warp is done with a ring slot
SVDX_DEVINL void release(uint32_t bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

// =====================================================================================
// forward. smem: Q | KV ring 2 x (K,V). O accumulates in registers; the running maximum of a row is updated every key
// block and O / l rescaled with it (flash-attention 2).
constexpr int FWD_KV_STAGES = 2;
constexpr int FWD_SMEM = 1024 + TILE_BYTES + FWD_KV_STAGES * 2 * TILE_BYTES + 256;

__global__ void __launch_bounds__(AT_THREADS, 1) attn_fwd_kernel(const __grid_constant__ AttnKParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sKV = sQ + TILE_BYTES;
  const uint32_t sBar = sKV + FWD_KV_STAGES * 2 * TILE_BYTES;
  const uint32_t b_qfull = sBar;
  const uint32_t b_kvfull = sBar + 8;          // [2]
  const uint32_t b_kvempty = sBar + 8 * 3;     // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int tile, head, outer, inner0;
  decode_block(p, tile, head, outer, inner0);
  const int nkv = p.tiles;

  if (warp == AT_PRODUCER && lane == 0) {
    prefetch_tmap(&p.tq); prefetch_tmap(&p.tk); prefetch_tmap(&p.tv);
    mbar_init(b_qfull, 1);
    for (int i = 0; i < FWD_KV_STAGES; ++i) { mbar_init(b_kvfull + 8 * i, 1); mbar_init(b_kvempty + 8 * i, AT_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == AT_PRODUCER) {
    if (lane == 0) {
      mbar_expect_tx(b_qfull, TILE_BYTES);
      tma_load_4d(&p.tq, b_qfull, sQ, head * 64, inner0, tile * p.RT, outer);
      for (int j = 0; j < nkv; ++j) {
        const int st = j % FWD_KV_STAGES;
        mbar_wait_mma(b_kvempty + 8 * st, ((j / FWD_KV_STAGES) & 1) ^ 1);
        mbar_expect_tx(b_kvfull + 8 * st, 2 * TILE_BYTES);
        tma_load_4d(&p.tk, b_kvfull + 8 * st, sKV + st * 2 * TILE_BYTES, head * 64, inner0, j * p.RT, outer);
        tma_load_4d(&p.tv, b_kvfull + 8 * st, sKV + st * 2 * TILE_BYTES + TILE_BYTES, head * 64, inner0, j * p.RT, outer);
      }
    }
    return;
  }
  const int wg = warp >> 2;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: r_lo, r_lo + 8
  const RowInfo ri[2] = {row_info(p, r_lo, tile, outer, inner0), row_info(p, r_lo + 8, tile, outer, inner0)};
  const float sc = p.scale * LOG2E;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this lane's partial row sums
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait_mma(b_qfull, 0);
  for (int j = 0; j < nkv; ++j) {
    const int st = j % FWD_KV_STAGES;
    const uint32_t sK = sKV + st * 2 * TILE_BYTES, sV = sK + TILE_BYTES;
    mbar_wait_mma(b_kvfull + 8 * st, (j / FWD_KV_STAGES) & 1);
    float s0[32], s1[32];
    mma_abt64(s0, sQ + wg * 8192, sK);
    mma_abt64(s1, sQ + wg * 8192, sK + 8192);
    wgmma_wait<0>();
    reg_fence(s0); reg_fence(s1);
    const int kvalid = p.S - j * p.RT;                 // valid key tokens in this block
    if (!(p.G == 1 && kvalid >= 128)) {                // warp-uniform: something to mask
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c0 = frag_col(i, lane), c1 = 64 + c0;
        const RowInfo& r = ri[frag_hi(i)];
        if (!(((c0 & p.gmask) == r.g) && ((c0 >> p.gshift) < kvalid))) s0[i] = -INFINITY;
        if (!(((c1 & p.gmask) == r.g) && ((c1 >> p.gshift) < kvalid))) s1[i] = -INFINITY;
      }
    }
    float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) bm[frag_hi(i)] = fmaxf(bm[frag_hi(i)], fmaxf(s0[i], s1[i]));
    float msc[2], alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float m_new = fmaxf(m_run[h], quad_max(bm[h]));
      const float m_use = m_new == -INFINITY ? 0.f : m_new;   // a row with no visible key so far (padding rows)
      alpha[h] = fast_exp2((m_run[h] - m_use) * sc);
      m_run[h] = m_new;
      msc[h] = m_use * sc;
      l_run[h] *= alpha[h];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int h = frag_hi(i);
      o[i] *= alpha[h];
      // probabilities: the row sum uses the fp32 values (the bf16 rounding of P averages out, as in flash-attention)
      s0[i] = fast_exp2(fmaf(s0[i], sc, -msc[h]));
      s1[i] = fast_exp2(fmaf(s1[i], sc, -msc[h]));
      l_run[h] += s0[i] + s1[i];
    }
    mma_pb64(o, s0, sV);
    mma_pb64(o, s1, sV + 8192);
    wgmma_wait<0>();
    reg_fence(o);
    release(b_kvempty + 8 * st, lane);
  }
  // epilogue: O / l
  bf16* rows[2];
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float l = quad_sum(l_run[h]);
    const float m_use = m_run[h] == -INFINITY ? 0.f : m_run[h];
    inv[h] = 1.f / l;
    rows[h] = ri[h].valid ? p.o + ri[h].token * p.ldo + head * 64 : nullptr;
    if (ri[h].valid && p.lse && (lane & 3) == 0) p.lse[ri[h].token * p.heads + head] = m_use * p.scale + __logf(l);
  }
  store_frag_rows(rows[0], rows[1], o, inv[0], inv[1], lane);
}

// =====================================================================================
// backward, dQ:  CTA owns a query tile, loops key tiles (two 64-key halves each).
// smem: Q | dO | KV ring 2 x (K,V).
constexpr int BWD_STAGES = 2;
constexpr int BDQ_SMEM = 1024 + 2 * TILE_BYTES + BWD_STAGES * 2 * TILE_BYTES + 256;

__global__ void __launch_bounds__(AT_THREADS, 1) attn_bwd_dq_kernel(const __grid_constant__ AttnKParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base, sDO = sQ + TILE_BYTES;
  const uint32_t sKV = sDO + TILE_BYTES;
  const uint32_t sBar = sKV + BWD_STAGES * 2 * TILE_BYTES;
  const uint32_t b_qfull = sBar;
  const uint32_t b_kvfull = sBar + 8;        // [2]
  const uint32_t b_kvempty = sBar + 8 * 3;   // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int tile, head, outer, inner0;
  decode_block(p, tile, head, outer, inner0);
  const int nkv = p.tiles;

  if (warp == AT_PRODUCER && lane == 0) {
    prefetch_tmap(&p.tq); prefetch_tmap(&p.tk); prefetch_tmap(&p.tv); prefetch_tmap(&p.tdo);
    mbar_init(b_qfull, 1);
    for (int i = 0; i < BWD_STAGES; ++i) { mbar_init(b_kvfull + 8 * i, 1); mbar_init(b_kvempty + 8 * i, AT_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == AT_PRODUCER) {
    if (lane == 0) {
      mbar_expect_tx(b_qfull, 2 * TILE_BYTES);
      tma_load_4d(&p.tq, b_qfull, sQ, head * 64, inner0, tile * p.RT, outer);
      tma_load_4d(&p.tdo, b_qfull, sDO, head * 64, inner0, tile * p.RT, outer);
      for (int j = 0; j < nkv; ++j) {
        const int st = j % BWD_STAGES;
        mbar_wait_mma(b_kvempty + 8 * st, ((j / BWD_STAGES) & 1) ^ 1);
        mbar_expect_tx(b_kvfull + 8 * st, 2 * TILE_BYTES);
        tma_load_4d(&p.tk, b_kvfull + 8 * st, sKV + st * 2 * TILE_BYTES, head * 64, inner0, j * p.RT, outer);
        tma_load_4d(&p.tv, b_kvfull + 8 * st, sKV + st * 2 * TILE_BYTES + TILE_BYTES, head * 64, inner0, j * p.RT, outer);
      }
    }
    return;
  }
  const int wg = warp >> 2;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const RowInfo ri[2] = {row_info(p, r_lo, tile, outer, inner0), row_info(p, r_lo + 8, tile, outer, inner0)};
  const float sc = p.scale * LOG2E;
  float lse2[2], dlt[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lse2[h] = ri[h].valid ? p.lse[ri[h].token * p.heads + head] * LOG2E : 0.f;
    dlt[h] = ri[h].valid ? p.delta[ri[h].token * p.heads + head] : 0.f;
  }
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait_mma(b_qfull, 0);
  for (int j = 0; j < nkv; ++j) {
    const int st = j % BWD_STAGES;
    const uint32_t sK = sKV + st * 2 * TILE_BYTES, sV = sK + TILE_BYTES;
    mbar_wait_mma(b_kvfull + 8 * st, (j / BWD_STAGES) & 1);
    const int kvalid = p.S - j * p.RT;
    const bool nomask = (p.G == 1) && (kvalid >= 128);
#pragma unroll 1
    for (int kh = 0; kh < 2; ++kh) {
      float s[32], dp[32];
      mma_abt64(s, sQ + wg * 8192, sK + kh * 8192);     // S_h  = Q K_h^T
      mma_abt64(dp, sDO + wg * 8192, sV + kh * 8192);   // dP_h = dO V_h^T
      wgmma_wait<0>();
      reg_fence(s); reg_fence(dp);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = kh * 64 + frag_col(i, lane), h = frag_hi(i);
        const bool ok = ri[h].valid && (nomask || (((c & p.gmask) == ri[h].g) && ((c >> p.gshift) < kvalid)));
        const float pr = ok ? fast_exp2(fmaf(s[i], sc, -lse2[h])) * p.scale : 0.f;
        s[i] = pr * (dp[i] - dlt[h]);
      }
      mma_pb64(dq, s, sK + kh * 8192);                  // dQ += dS_h K_h
      wgmma_wait<0>();
      reg_fence(dq);
    }
    release(b_kvempty + 8 * st, lane);
  }
  store_frag_rows(ri[0].valid ? p.dq + ri[0].token * p.lddq + head * 64 : nullptr,
                  ri[1].valid ? p.dq + ri[1].token * p.lddq + head * 64 : nullptr, dq, 1.f, 1.f, lane);
}

// =====================================================================================
// backward, dK/dV: CTA owns a key tile, loops query tiles (two 64-query halves each). Scores are computed transposed
// (S^T = K Q^T, dP^T = V dO^T) so that P^T / dS^T are the A operands of dV += P^T dO and dK += dS^T Q.
// smem: K | V | Q/dO ring 2 | lse/delta of the current query tile
constexpr int BKV_SMEM = 1024 + 2 * TILE_BYTES + BWD_STAGES * 2 * TILE_BYTES + 1024 + 256;

__global__ void __launch_bounds__(AT_THREADS, 1) attn_bwd_dkv_kernel(const __grid_constant__ AttnKParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = base, sV = sK + TILE_BYTES;
  const uint32_t sQD = sV + TILE_BYTES;
  const uint32_t sVec = sQD + BWD_STAGES * 2 * TILE_BYTES;  // float lse2[128], delta[128]
  const uint32_t sBar = sVec + 1024;
  const uint32_t b_kvfull = sBar;
  const uint32_t b_qfull = sBar + 8;        // [2]
  const uint32_t b_qempty = sBar + 8 * 3;   // [2]
  float* vec = reinterpret_cast<float*>(smem_raw + (sVec - smem_u32(smem_raw)));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int tile, head, outer, inner0;
  decode_block(p, tile, head, outer, inner0);
  const int nq = p.tiles;

  if (warp == AT_PRODUCER && lane == 0) {
    prefetch_tmap(&p.tq); prefetch_tmap(&p.tk); prefetch_tmap(&p.tv); prefetch_tmap(&p.tdo);
    mbar_init(b_kvfull, 1);
    for (int i = 0; i < BWD_STAGES; ++i) { mbar_init(b_qfull + 8 * i, 1); mbar_init(b_qempty + 8 * i, AT_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == AT_PRODUCER) {
    if (lane == 0) {
      mbar_expect_tx(b_kvfull, 2 * TILE_BYTES);
      tma_load_4d(&p.tk, b_kvfull, sK, head * 64, inner0, tile * p.RT, outer);
      tma_load_4d(&p.tv, b_kvfull, sV, head * 64, inner0, tile * p.RT, outer);
      for (int i = 0; i < nq; ++i) {
        const int st = i % BWD_STAGES;
        mbar_wait_mma(b_qempty + 8 * st, ((i / BWD_STAGES) & 1) ^ 1);
        mbar_expect_tx(b_qfull + 8 * st, 2 * TILE_BYTES);
        tma_load_4d(&p.tq, b_qfull + 8 * st, sQD + st * 2 * TILE_BYTES, head * 64, inner0, i * p.RT, outer);
        tma_load_4d(&p.tdo, b_qfull + 8 * st, sQD + st * 2 * TILE_BYTES + TILE_BYTES, head * 64, inner0, i * p.RT, outer);
      }
    }
    return;
  }
  const int wg = warp >> 2;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's key rows: r_lo, r_lo + 8
  const RowInfo ki[2] = {row_info(p, r_lo, tile, outer, inner0), row_info(p, r_lo + 8, tile, outer, inner0)};
  const float sc = p.scale * LOG2E;
  // lse (threads 0..127) / delta (128..255) of query row threadIdx.x % 128 of a tile; +inf lse -> p = 0 for padding queries
  const int vr = threadIdx.x & 127;
  auto load_stat = [&](int i) -> float {
    const RowInfo qi = row_info(p, vr, i, outer, inner0);
    if (threadIdx.x < 128) return qi.valid ? p.lse[qi.token * p.heads + head] * LOG2E : INFINITY;
    return qi.valid ? p.delta[qi.token * p.heads + head] : 0.f;
  };
  float stat = load_stat(0);
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  mbar_wait_mma(b_kvfull, 0);
  for (int i = 0; i < nq; ++i) {
    // stage lse/delta of the 128 queries of tile i (column vectors of the transposed scores); the values of the
    // next tile are requested right away so that their latency hides behind this tile's work
    named_bar_sync(1, 32 * AT_CONSUMER_WARPS);  // previous iteration finished reading vec[]
    vec[threadIdx.x] = stat;
    named_bar_sync(1, 32 * AT_CONSUMER_WARPS);
    if (i + 1 < nq) stat = load_stat(i + 1);
    const int st = i % BWD_STAGES;
    const uint32_t sQ = sQD + st * 2 * TILE_BYTES, sDO = sQ + TILE_BYTES;
    mbar_wait_mma(b_qfull + 8 * st, (i / BWD_STAGES) & 1);
#pragma unroll 1
    for (int qh = 0; qh < 2; ++qh) {
      float s[32], dp[32];
      mma_abt64(s, sK + wg * 8192, sQ + qh * 8192);     // S^T_h  = K Q_h^T
      mma_abt64(dp, sV + wg * 8192, sDO + qh * 8192);   // dP^T_h = V dO_h^T
      wgmma_wait<0>();
      reg_fence(s); reg_fence(dp);
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const int c = qh * 64 + frag_col(k, lane);       // query column
        const RowInfo& r = ki[frag_hi(k)];
        // G == 1: invalid query columns carry lse = +inf -> p = 0
        const bool ok = r.valid && (p.G == 1 || (c & p.gmask) == r.g);
        const float pr = ok ? fast_exp2(fmaf(s[k], sc, -vec[c])) : 0.f;
        s[k] = pr;
        dp[k] = (pr * p.scale) * (dp[k] - vec[128 + c]);
      }
      mma_pb64(dv, s, sDO + qh * 8192);                  // dV += P^T_h dO_h
      mma_pb64(dk, dp, sQ + qh * 8192);                  // dK += dS^T_h Q_h
      wgmma_wait<0>();
      reg_fence(dv); reg_fence(dk);
    }
    release(b_qempty + 8 * st, lane);
  }
  store_frag_rows(ki[0].valid ? p.dv + ki[0].token * p.lddv + head * 64 : nullptr,
                  ki[1].valid ? p.dv + ki[1].token * p.lddv + head * 64 : nullptr, dv, 1.f, 1.f, lane);
  store_frag_rows(ki[0].valid ? p.dk + ki[0].token * p.lddk + head * 64 : nullptr,
                  ki[1].valid ? p.dk + ki[1].token * p.lddk + head * 64 : nullptr, dk, 1.f, 1.f, lane);
}

// delta[token row][head] = sum_d dO * O   — one warp per (sequence, token, head); the token row follows the descriptor's
// geometry as row_info does, so only the rows the backward kernels read are written
__global__ void attn_delta_kernel(const bf16* __restrict__ o, long long ldo, const bf16* __restrict__ dout, long long lddo,
                                  long long nseq, int S, int inner, long long outer_stride, long long inner_stride,
                                  long long tok_stride, int heads, float* __restrict__ delta) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= nseq * S * heads) return;
  const long long st = w / heads;                    // sequence * S + token
  const int h = (int)(w - st * heads);
  const long long seq = st / S;
  const long long t = st - seq * S;
  const long long outer = seq / inner;
  const long long tok = outer * outer_stride + (seq - outer * inner) * inner_stride + t * tok_stride;
  const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(o + tok * ldo + h * 64 + 2 * lane));
  const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + tok * lddo + h * 64 + 2 * lane));
  const float s = warp_sum(a.x * b.x + a.y * b.y);
  if (lane == 0) delta[tok * heads + h] = s;
}

}  // namespace svdx

using namespace svdx;

static int attn_make_map(CUtensorMap* m, const void* ptr, int64_t ld, int cols, const SvdxAttn* d, int G, int RT) {
  const int outer = d->nseq / d->inner;
  uint64_t dims[4] = {(uint64_t)cols, (uint64_t)d->inner, (uint64_t)d->S, (uint64_t)outer};
  uint64_t strides[3] = {(uint64_t)(d->inner_stride * ld * 2), (uint64_t)(d->tok_stride * ld * 2), (uint64_t)(d->outer_stride * ld * 2)};
  if (d->inner == 1) strides[0] = (uint64_t)ld * 2;  // extent-1 dimension: any legal stride
  uint32_t box[4] = {64, (uint32_t)G, (uint32_t)RT, 1};
  return svdx_make_tmap(m, ptr, 4, dims, strides, box);
}

static int attn_setup(const SvdxAttn* d, AttnKParams& p, bool bwd, dim3& grid) {
  if (!d || !d->q || !d->k || !d->v) return svdx_fail(SVDX_E_BADARG, "attention: null pointer");
  if (d->heads <= 0 || d->S <= 0 || d->nseq <= 0 || d->inner <= 0 || d->nseq % d->inner) return svdx_fail(SVDX_E_BADARG, "attention: bad sequence geometry");
  if ((d->ldq % 8) || (d->ldk % 8) || (d->ldv % 8)) return svdx_fail(SVDX_E_BADARG, "attention: leading dims must be multiples of 8");
  const int64_t cols = (int64_t)d->heads * 64;
  if (d->ldq < cols || d->ldk < cols || d->ldv < cols) return svdx_fail(SVDX_E_BADARG, "attention: ldq / ldk / ldv < heads * 64");
  if (bwd) {
    if (!d->dout || !d->dq || !d->dk || !d->dv || !d->lse || !d->delta || !d->o) return svdx_fail(SVDX_E_BADARG, "attention_bwd: null pointer");
    if ((d->lddo % 8) || (d->lddq % 8) || (d->lddk % 8) || (d->lddv % 8) || (d->ldo % 8)) return svdx_fail(SVDX_E_BADARG, "attention_bwd: leading dims");
    if (d->lddo < cols || d->lddq < cols || d->lddk < cols || d->lddv < cols || d->ldo < cols)
      return svdx_fail(SVDX_E_BADARG, "attention_bwd: ldo / lddo / lddq / lddk / lddv < heads * 64");
  } else {
    if (!d->o || (d->ldo % 8)) return svdx_fail(SVDX_E_BADARG, "attention_fwd: output");
    if (d->ldo < cols) return svdx_fail(SVDX_E_BADARG, "attention_fwd: ldo < heads * 64");
  }
  // o / dq / dk / dv are written as 4-byte column pairs (store_frag_rows), and o is read so by the delta kernel
  const uintptr_t out_al = reinterpret_cast<uintptr_t>(d->o) | (bwd ? reinterpret_cast<uintptr_t>(d->dq) | reinterpret_cast<uintptr_t>(d->dk) |
                                                                        reinterpret_cast<uintptr_t>(d->dv) : 0);
  if (out_al & 3) return svdx_fail(SVDX_E_BADARG, "attention: o / dq / dk / dv must be 4 B aligned");
  memset(&p, 0, sizeof(p));
  int G = 1;
  if (d->inner > 1) {
    // pack G sequences per tile: largest power of two with G * S <= 128 that divides inner
    G = 1;
    while (G * 2 * d->S <= 128 && d->inner % (G * 2) == 0 && G < 64) G *= 2;
  }
  const int RT = 128 / G;
  if (d->inner > 1 && d->S > RT) return svdx_fail(SVDX_E_BADARG, "attention: strided sequences longer than 128 tokens are not supported");
  p.G = G; p.RT = RT; p.S = d->S; p.heads = d->heads;
  p.gmask = G - 1; p.gshift = 0;
  while ((1 << p.gshift) < G) ++p.gshift;
  p.inner_groups = d->inner / G;
  p.tiles = (d->S + RT - 1) / RT;
  p.outer_stride = d->outer_stride; p.inner_stride = d->inner_stride; p.tok_stride = d->tok_stride;
  p.scale = d->scale;
  const long long gz = (long long)(d->nseq / d->inner) * p.inner_groups;
  if (gz > 65535 || d->heads > 65535) return svdx_fail(SVDX_E_BADARG, "attention: grid too large");
  grid = dim3(p.tiles, d->heads, (unsigned)gz);
  p.o = reinterpret_cast<bf16*>(d->o); p.ldo = d->ldo;
  p.lse = d->lse; p.delta = d->delta;
  p.dq = reinterpret_cast<bf16*>(d->dq); p.lddq = d->lddq;
  p.dk = reinterpret_cast<bf16*>(d->dk); p.lddk = d->lddk;
  p.dv = reinterpret_cast<bf16*>(d->dv); p.lddv = d->lddv;
  // every argument check is above: the tensor maps need the driver
  int rc;
  if ((rc = attn_make_map(&p.tq, d->q, d->ldq, (int)cols, d, G, RT))) return rc;
  if ((rc = attn_make_map(&p.tk, d->k, d->ldk, (int)cols, d, G, RT))) return rc;
  if ((rc = attn_make_map(&p.tv, d->v, d->ldv, (int)cols, d, G, RT))) return rc;
  if (bwd && (rc = attn_make_map(&p.tdo, d->dout, d->lddo, (int)cols, d, G, RT))) return rc;
  return 0;
}

// attention_small.cu: CUDA-core kernels for strided short sequences (temporal attention, S <= 32) — HBM-bound work
bool svdx_attention_small_eligible(const SvdxAttn* d);
int svdx_attention_small_fwd(const SvdxAttn* d, cudaStream_t st);
int svdx_attention_small_bwd(const SvdxAttn* d, cudaStream_t st);

extern "C" int svdx_attention_fwd(const SvdxAttn* d, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (svdx_attention_small_eligible(d)) return svdx_attention_small_fwd(d, st);
  AttnKParams p;
  dim3 grid;
  int rc = attn_setup(d, p, false, grid);
  if (rc) return rc;
  static bool attr[SVDX_MAX_DEVICES] = {false};
  const int slot = svdx_device_slot();
  if (!attr[slot]) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM);
    if (e != cudaSuccess) return svdx_fail_cuda(e, "attention_fwd: smem attribute");
    attr[slot] = true;
  }
  attn_fwd_kernel<<<grid, AT_THREADS, FWD_SMEM, st>>>(p);
  SVDX_CHECK_LAUNCH("attention_fwd");
  return SVDX_OK;
}

extern "C" int svdx_attention_bwd(const SvdxAttn* d, void* stream_v) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (svdx_attention_small_eligible(d)) return svdx_attention_small_bwd(d, st);
  AttnKParams p;
  dim3 grid;
  int rc = attn_setup(d, p, true, grid);
  if (rc) return rc;
  static bool attr[SVDX_MAX_DEVICES] = {false};
  const int slot = svdx_device_slot();
  if (!attr[slot]) {
    cudaError_t e = cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BDQ_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BKV_SMEM);
    if (e != cudaSuccess) return svdx_fail_cuda(e, "attention_bwd: smem attribute");
    attr[slot] = true;
  }
  const long long warps = (long long)d->nseq * d->S * d->heads;
  attn_delta_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const bf16*>(d->o), d->ldo, reinterpret_cast<const bf16*>(d->dout), d->lddo, d->nseq, d->S, d->inner,
      d->outer_stride, d->inner_stride, d->tok_stride, d->heads, d->delta);
  attn_bwd_dq_kernel<<<grid, AT_THREADS, BDQ_SMEM, st>>>(p);
  attn_bwd_dkv_kernel<<<grid, AT_THREADS, BKV_SMEM, st>>>(p);
  SVDX_CHECK_LAUNCH("attention_bwd");
  return SVDX_OK;
}
