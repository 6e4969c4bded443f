// Shared pieces of the wgmma tapgemm kernel (tapgemm.cu): kernel parameter block, tile geometry and the fused epilogue
// of one accumulator tile.
#pragma once
#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"

namespace svdx {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int MAX_BN = 160;                           // widest tile: 80 accumulator registers per thread
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int B_STAGE_BYTES = MAX_BN * BLOCK_K * 2;   // 20 KB
constexpr int NUM_EPI_WARPS = 8;   // the two consumer warpgroups: wgmma main loop, then the epilogue of the tile
constexpr int PRODUCER_WARP = NUM_EPI_WARPS;
constexpr int NUM_THREADS = 32 * NUM_EPI_WARPS + 32;
// EPI_GENERIC parks the finished fp32 accumulator tile in shared memory, one 128-row x MAX_BN tile; rows padded by 16 bytes
// so that the epilogue's row-per-lane 16-byte reads are conflict-free
constexpr int ACC_LD = MAX_BN + 4;
constexpr int ACC_BYTES = BLOCK_M * ACC_LD * 4;
constexpr int EPI_STAGE_BYTES = 4096;  // per epilogue warp: 2 x (32 rows x 64 B) bf16 halves or 1 x (32 rows x 128 B) fp32
// operand ring depth: the parked tile leaves room for 3 stages; the register epilogues give its 84 KB to two more
constexpr int STAGES_PARKED = 3;
constexpr int STAGES_REGS = 5;
constexpr int smem_bytes(int stages, bool parked) {
  return 1024 + stages * (A_STAGE_BYTES + B_STAGE_BYTES) + (parked ? ACC_BYTES : 0) + NUM_EPI_WARPS * EPI_STAGE_BYTES + 256;
}
static_assert(smem_bytes(STAGES_PARKED, true) <= 227 * 1024, "tapgemm shared memory exceeds the 227 KB a block may use");
static_assert(smem_bytes(STAGES_REGS, false) <= 227 * 1024, "tapgemm shared memory exceeds the 227 KB a block may use");
static_assert(16 * STAGES_REGS <= 256, "ring barriers must fit their 256-byte region");
static_assert((ACC_BYTES % 1024) == 0 && (B_STAGE_BYTES % 1024) == 0, "staging buffers must stay 1024-byte aligned");

struct __align__(64) TapGemmKParams {
  CUtensorMap tma;
  CUtensorMap tmb;
  CUtensorMap tma_bh[4];  // CONV2D: boxes of 2, 4, 8, 16 image rows (tma itself = 1 row)
  int max_bh_log2;
  int a_mode, a_mn, b_mn, b_mode, kb_per_group;
  int rows_per_group, groups, tiles_per_group;
  int W, H, nimg;
  int wtiles;          // CONV2D with W > 128 (W % 128 == 0): a tile = 128 consecutive pixels of ONE image row, wtiles = W / 128 (else 0)
  int im2col;          // the image operand (CONV2D A: tma, 128 pixels; b_mode 1 B: tmb, 64 pixels) is an im2col map: widths
                       // the row boxes cannot tile (neither W | 128 nor 128 | W for A, W | 64 / 64 | W for B)
  int num_taps;
  int tap_d0[SVDX_MAX_TAPS], tap_d1[SVDX_MAX_TAPS], tap_d2[SVDX_MAX_TAPS];
  int M, N, K;
  int block_n, m_tiles, n_tiles, split_k, kb_total, kb_per_split, kb_per_tap;
  // epilogue
  void* out;
  long long ldo;
  int out_dtype, geglu;
  const float* bias;
  const float* rowbias;
  int rowbias_div;
  long long ldrb;
  const bf16* res1;
  long long ldr1;
  const bf16* res2;
  long long ldr2;
  const float* scales;
  bf16* pre;
  long long ldpre;
  CUtensorMap tmo;     // output (bf16: 32x32 box, 64B swizzle; fp32: 32x32 box, 128B swizzle), dims {n_out, rows, groups}
  CUtensorMap tmo16;   // EPI_F32: the fp32 output map of tmo with 16-row boxes (one per consumer warp)
  CUtensorMap tmpre;   // GEGLU pre-activation [M, N]
  float* gn_sum;       // fused GroupNorm statistics of the output (per slab m / gn_rows, per channel): [slab][2][gn_ld]
  long long gn_ld;
  int gn_rows;
  // GroupNorm BACKWARD statistics fused into the epilogue of the GEMM / conv that writes dy = dL/d(GroupNorm output)
  const bf16* gnb_x;   // the GroupNorm's INPUT (channels [0, gnb_c1)), and gnb_x2 the concatenated second source
  long long gnb_ldx;
  const bf16* gnb_x2;
  long long gnb_ldx2;
  int gnb_c1;
  const float* gnb_ab; // [slab][2][N]: forward scale / shift per channel (y = act(x * scale + shift))
  float* gnb_sum;      // [slab][2][N], zero on entry: sum(e), sum(e * x), e = dy * act'(x * scale + shift)
  int gnb_rows, gnb_silu;
  int tma_store;       // epilogue stores through shared memory + TMA (tmo / tmpre valid)
  int epi_mode;        // EPI_GENERIC / EPI_FAST / EPI_GEGLU / EPI_RES: which kernel instantiation runs
  int probe;   // dev switch SVDX_EPI_PROBE: 1 = epilogue without global stores, 2 = no epilogue work at all
  int interleave;      // tmo is the 4-D phase view {n_out, W, H, nimg} of a 2x-upsampled output (EPI_FAST_IL*)
  int act;             // SVDX_ACT_GELU / SVDX_ACT_QUICK_GELU applied after the bias (EPI_FAST_ACT)
  bf16* il_out;        // interleave: output row 0 of the phase (out + (2 W phase_h + phase_w) * ldo), for il_store_next_row
};


// 32 consecutive fp32 accumulator columns [col, col + 32) of one tile row (row = the row's shared-memory address)
SVDX_DEVINL void acc_ld32(uint32_t row, int col, uint32_t (&r)[32]) {
  const uint32_t a = row + col * 4;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r[4 * k]), "=r"(r[4 * k + 1]), "=r"(r[4 * k + 2]), "=r"(r[4 * k + 3])
                 : "r"(a + 16 * k));
}

// output row of epilogue thread r (0..127) of m-tile mt, and whether it exists
SVDX_DEVINL void tile_row(const TapGemmKParams& p, int mt, int r, long long& m, bool& row_ok) {
  if (p.a_mode == SVDX_A_ROWS && !p.a_mn) {
    const int g = mt / p.tiles_per_group;
    const int t = mt - g * p.tiles_per_group;
    const int rin = t * BLOCK_M + r;
    row_ok = rin < p.rows_per_group;
    m = (long long)g * p.rows_per_group + rin;
  } else {
    m = (long long)mt * BLOCK_M + r;
    row_ok = m < p.M;
  }
}

// ---- conv A tiles: the 128 pixels of a tile are R = 128 / W consecutive image rows, fetched as a few multi-row TMA
// boxes (image borders and tile/image straddling decide the split). The split depends on the tile only, so it is
// computed once per tile with lane l of the producer warp keeping box l; per k-block every lane that owns a box
// issues its TMA. (A per-k-block scalar decomposition costs ~1.5-3 k cycles and makes the producer thread the
// bottleneck of a 3x3 convolution.)
struct ConvBox {
  int lg, hh, n;
  uint32_t dst_off;
  bool nvalid, active;
};
SVDX_DEVINL void conv_tile_boxes(const TapGemmKParams& p, int t, int lane, ConvBox& mine) {
  const int R = BLOCK_M / p.W;
  int rowid = t * R, left = R, idx = 0;
  uint32_t off = 0;
  mine.active = false; mine.lg = 0; mine.hh = 0; mine.n = 0; mine.dst_off = 0; mine.nvalid = false;
  while (left > 0) {
    const int n = rowid / p.H;
    const int h = rowid - n * p.H;
    int run = min(left, p.H - h);
    int hh = h;
    while (run > 0) {
      const int lg = min(p.max_bh_log2, 31 - __clz(run));
      const int bh = 1 << lg;
      if (idx == lane) { mine.lg = lg; mine.hh = hh; mine.n = n; mine.nvalid = n < p.nimg; mine.dst_off = off; mine.active = true; }
      off += bh * p.W * 128;
      hh += bh; run -= bh; left -= bh; rowid += bh; ++idx;
    }
  }
}

// ---- staged stores: a warp writes its 32-row x 32-column chunk into shared memory (one row per lane, swizzled so
// that the 16-byte writes are conflict-free) and one lane hands it to the TMA unit. The global writes become full
// 64/128-byte row segments issued asynchronously, instead of 32 scattered 16-byte sectors per store instruction
// (scattered stores make the short-K GEMMs epilogue-bound).
// Rows past the end of the group / matrix and columns past n_out are clipped by the tensor map.
struct EpiStage {
  uint32_t base;   // this warp's 4 KB staging region (1024-aligned)
  uint32_t off;    // bf16 and EPI_F32: alternates between the two 2 KB halves
  int row0, grp;   // tensor-map coordinates of this warp's first row
};

SVDX_DEVINL void stage_store_bf16(const CUtensorMap* tm, EpiStage& st, int lane, const float (&f)[32], int col) {
  if (lane == 0) bulk_wait_read<1>();   // the half written two stores ago has been read out
  __syncwarp();
  const uint32_t buf = st.base + st.off;
  const uint32_t row = buf + lane * 64;
  const int sw = (lane >> 1) & 3;       // CU_TENSOR_MAP_SWIZZLE_64B: 16-byte chunk index ^= address bits [7:8]
#pragma unroll
  for (int j = 0; j < 4; ++j)
    st_shared_v4(row + ((j ^ sw) << 4), pack_bf16x2(f[8 * j], f[8 * j + 1]), pack_bf16x2(f[8 * j + 2], f[8 * j + 3]),
                 pack_bf16x2(f[8 * j + 4], f[8 * j + 5]), pack_bf16x2(f[8 * j + 6], f[8 * j + 7]));
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) { tma_store_3d(tm, buf, col, st.row0, st.grp); bulk_commit(); }
  st.off ^= 2048;
}

SVDX_DEVINL void stage_store_f32(const CUtensorMap* tm, EpiStage& st, int lane, const float (&f)[32], int col, bool reduce) {
  if (lane == 0) bulk_wait_read<0>();
  __syncwarp();
  const uint32_t row = st.base + lane * 128;
  const int sw = lane & 7;              // CU_TENSOR_MAP_SWIZZLE_128B
#pragma unroll
  for (int j = 0; j < 8; ++j)
    st_shared_v4(row + ((j ^ sw) << 4), __float_as_uint(f[4 * j]), __float_as_uint(f[4 * j + 1]), __float_as_uint(f[4 * j + 2]),
                 __float_as_uint(f[4 * j + 3]));
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) {
    if (reduce) tma_reduce_add_3d(tm, st.base, col, st.row0, st.grp);
    else tma_store_3d(tm, st.base, col, st.row0, st.grp);
    bulk_commit();
  }
}

// ---- GroupNorm statistics of the output, fused into the epilogue: column sums (and sums of squares) of one staged
// 32-row x 32-column bf16 chunk, i.e. of exactly the values the TMA store writes. Lane l takes the column pair l % 16 and
// the rows of parity l / 16 (two 64-byte rows per wavefront: conflict-free with the 64B swizzle), the two halves are
// combined with one shuffle and lanes 0..15 issue two red.global.add.v2.f32. Rows are walked slab by slab (a slab = gn_rows
// consecutive rows = one frame or one clip), so tiles that straddle frames (5x8 latents) stay correct.
// m0 = global row index of the chunk's row 0, valid_rows = how many of its 32 rows exist.
SVDX_DEVINL void gn_chunk_sums(const TapGemmKParams& p, uint32_t buf, int lane, int col0, int n_out_total, long long m0, int valid_rows) {
  const int pr = lane & 15, h = lane >> 4;
  const uint32_t in_chunk = (uint32_t)(pr & 3) * 4u;
  const int jch = pr >> 2;
  long long slab = m0 / p.gn_rows;
  int left = p.gn_rows - (int)(m0 - slab * p.gn_rows);
  int r = 0;
  while (r < valid_rows) {                                     // warp-uniform trip count
    const int seg_end = min(valid_rows, r + left);
    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
    for (int rr = r + ((h ^ r) & 1); rr < seg_end; rr += 2) {
      uint32_t w;
      asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(buf + rr * 64 + ((uint32_t)(jch ^ ((rr >> 1) & 3)) << 4) + in_chunk));
      const float2 v = unpack_bf16x2(w);
      s0 += v.x; s1 += v.y;
      q0 = fmaf(v.x, v.x, q0); q1 = fmaf(v.y, v.y, q1);
    }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
    q0 += __shfl_xor_sync(0xffffffffu, q0, 16); q1 += __shfl_xor_sync(0xffffffffu, q1, 16);
    const int col = col0 + 2 * pr;
    if (h == 0 && col < n_out_total) {
      float* d = p.gn_sum + (2 * slab) * p.gn_ld + col;
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(s0), "f"(s1) : "memory");
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d + p.gn_ld), "f"(q0), "f"(q1) : "memory");
    }
    r = seg_end; ++slab; left = p.gn_rows;
  }
}

// ---- specialised epilogues (kernel template parameter EPI): the hot shapes have short K, so the per-chunk instruction
// count of the epilogue decides their speed. Every EPI but EPI_GENERIC and EPI_F32 assumes a bf16 output written through TMA,
// whole 32-column chunks (n_out % 32 == 0), 16-byte aligned bias rows and a K-major A operand, and reads the accumulator straight
// from the wgmma registers (epilogue_regs); EPI_F32 is the fp32 counterpart (epilogue_f32); everything else parks the tile
// and takes the generic epilogue_tile below.
constexpr int EPI_GENERIC = 0, EPI_FAST = 1, EPI_GEGLU = 2, EPI_RES = 3;
// + fused GroupNorm statistics of the output (separate instantiations: the plain ones keep their register budget)
constexpr int EPI_FAST_GN = 4, EPI_RES_GN = 5;
// + fused GroupNorm BACKWARD sums (the output is the gradient of a GroupNorm's output)
constexpr int EPI_FAST_GNB = 6;
// plain epilogue with the interleaved (upsample phase) store, without / with fused GroupNorm statistics
constexpr int EPI_FAST_IL = 7, EPI_FAST_IL_GN = 8;
// plain epilogue + activation (act(acc + bias)): its own instantiation, so the others keep their register budget
constexpr int EPI_FAST_ACT = 9;
// fp32 output through TMA (store or reduce-add: weight gradients, split-K partials), optionally scaled by scales[0]; any
// operand majors, ragged N; no bias / row-bias / residuals (epilogue_f32)
constexpr int EPI_F32 = 10;

// the activations of EPI_FAST_ACT: GELU (erf) and quick_gelu x * sigmoid(1.702 x)
template <int N>
SVDX_DEVINL void act_n(float (&f)[N], int act) {
  if (act == SVDX_ACT_GELU) {
#pragma unroll
    for (int i = 0; i < N; ++i) f[i] = gelu_erf_f(f[i]);
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) f[i] = __fdividef(f[i], 1.0f + __expf(-1.702f * f[i]));
  }
}

// TMA store of one staged 32-row chunk whose first row is row0 of group grp. Interleaved: the chunk is 32 consecutive pixels
// of the low-res geometry, addressed through the 4-D phase view {column, w, h, image}. W < 32: the box is 32 / W whole rows
// (whole images per chunk: checked on the host). W >= 32: the box is 32 pixels of one row, clipped at W by the map; the
// pixels of a chunk that run past the end of the row are written by il_store_next_row.
template <bool IL>
SVDX_DEVINL void store_chunk(const TapGemmKParams& p, uint32_t src, int col, int row0, int grp) {
  if constexpr (IL) {
    const int w0 = row0 % p.W, r = row0 / p.W;
    tma_store_4d(&p.tmo, src, col, w0, r % p.H, r / p.H);
  } else {
    tma_store_3d(&p.tmo, src, col, row0, grp);
  }
}

// Interleaved store, W >= 32: a chunk whose first pixel w0 has fewer than 32 pixels left in its row (only at widths that are
// not multiples of 32) continues in the next row, or in row 0 of the next image. The TMA store above wrote the part in the
// first row. Each lane whose pixel lies in the next row writes its own 64-byte row from the staged (64B-swizzled) chunk.
// Low-res pixel row r = n * H + h, column w lands on output row 4 W r + 2 w of the phase base.
SVDX_DEVINL void il_store_next_row(const TapGemmKParams& p, uint32_t src, int col, int row0, int lane) {
  const int k = p.W - row0 % p.W;   // pixels of the chunk in its first row
  if (p.W < 32 || k >= 32 || lane < k || row0 + lane >= p.M) return;
  const long long orow = 4LL * p.W * (row0 / p.W + 1) + 2 * (lane - k);
  uint4* dst = reinterpret_cast<uint4*>(p.il_out + orow * p.ldo + col);
  const uint32_t row = src + lane * 64;
  const int sw = (lane >> 1) & 3;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(row + ((j ^ sw) << 4)));
    dst[j] = v;
  }
}

// Epilogue operands that are read per chunk (the residual of EPI_RES, the GroupNorm input of EPI_FAST_GNB) are usually not in L2
// any more; a warp has ONE chunk's loads in flight, so the fetch is latency-bound. Each epilogue warp therefore requests its 32 rows x bn columns of the tile
// into L2 BEFORE its main loop: the lines arrive while the tensor cores work. Lane = row; the two warps of a lane
// quarter take alternate 128-byte lines.
SVDX_DEVINL void prefetch_rows_l2(const bf16* base, long long ld, long long m0, int valid_rows, int col0, int ncols, int lane, int half) {
  if (!base || lane >= valid_rows) return;
  const char* row = reinterpret_cast<const char*>(base + (m0 + lane) * ld + col0);
  const int bytes = ncols * 2;
  for (int b = half * 128; b < bytes; b += 256) asm volatile("prefetch.global.L2 [%0];" ::"l"(row + b));
}
SVDX_DEVINL void prefetch_epilogue_operands(const TapGemmKParams& p, int epi, long long m0, int valid_rows, int n0, int bn_out, int n_out_total,
                                            int lane, int half) {
  const int ncols = min(bn_out, n_out_total - n0);
  if (ncols <= 0) return;
  if (epi == EPI_RES || epi == EPI_RES_GN) {
    prefetch_rows_l2(p.res1, p.ldr1, m0, valid_rows, n0, ncols, lane, half);
    prefetch_rows_l2(p.res2, p.ldr2, m0, valid_rows, n0, ncols, lane, half);
  } else if (epi == EPI_FAST_GNB) {
    if (n0 < p.gnb_c1) prefetch_rows_l2(p.gnb_x, p.gnb_ldx, m0, valid_rows, n0, min(ncols, p.gnb_c1 - n0), lane, half);
    if (n0 + ncols > p.gnb_c1) {
      const int c0 = max(n0, p.gnb_c1);
      prefetch_rows_l2(p.gnb_x2, p.gnb_ldx2, m0, valid_rows, c0 - p.gnb_c1, n0 + ncols - c0, lane, half);
    }
  }
}

// ---- GroupNorm backward, pass 1, fused into the epilogue that WRITES dy (the dgrad conv / GEMM whose input was the
// GroupNorm(+SiLU) output): per (slab, channel) S = sum_rows e and SX = sum_rows e * x with e = dy * act'(x * scale + shift),
// from the staged bf16 dy chunk (exactly the values stored) and the matching 32 x 32 chunk of the GroupNorm input x staged
// beside it. The consumer (svdx_groupnorm_bwd_fused) folds channels into groups: s1 = sum_c gamma_c S_c,
// s2 = rstd * (sum_c gamma_c SX_c - mean * s1); dgamma_c = rstd * (SX_c - mean * S_c), dbeta_c = S_c. Same lane layout as
// gn_chunk_sums (lane = column pair x row parity), slabs walked segment by segment.
// ROWS: the rows the buffers hold (a 32-row chunk, or one warp's 16-row half of it).
template <int ROWS = 32>
SVDX_DEVINL void gnb_chunk_sums(const TapGemmKParams& p, uint32_t buf_dy, uint32_t buf_x, int lane, int col0, int n_out_total, long long m0,
                                int valid_rows) {
  const int pr = lane & 15, h = lane >> 4;
  const uint32_t in_chunk = (uint32_t)(pr & 3) * 4u;
  const int jch = pr >> 2;
  long long slab = m0 / p.gnb_rows;
  int left = p.gnb_rows - (int)(m0 - slab * p.gnb_rows);
  const int col = col0 + 2 * pr;
  const bool col_ok = col < n_out_total;
  int r = 0;
  while (r < valid_rows) {                                     // warp-uniform trip count
    const int seg_end = min(valid_rows, r + left);
    float2 A = make_float2(0.f, 0.f), B = make_float2(0.f, 0.f);
    if (col_ok && p.gnb_silu) {
      A = *reinterpret_cast<const float2*>(p.gnb_ab + (2 * slab) * p.N + col);
      B = *reinterpret_cast<const float2*>(p.gnb_ab + (2 * slab + 1) * p.N + col);
    }
    float s0 = 0.f, s1 = 0.f, x0 = 0.f, x1 = 0.f;
    if (r == 0 && seg_end == ROWS) {
      // the common case (all ROWS rows inside one slab): rows h, h + 2, ... in unrolled batches of 8 so that the
      // sigmoid chains (ex2 -> rcp) of different rows overlap; the rolled loop below ran one dependent chain at a time
#pragma unroll
      for (int b = 0; b < ROWS / 16; ++b) {
        uint32_t wd[8], wx[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int rr = h + 2 * (8 * b + i);
          const uint32_t off = rr * 64 + ((uint32_t)(jch ^ ((rr >> 1) & 3)) << 4) + in_chunk;
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(wd[i]) : "r"(buf_dy + off));
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(wx[i]) : "r"(buf_x + off));
        }
        float e0[8], e1[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float2 d = unpack_bf16x2(wd[i]), xv = unpack_bf16x2(wx[i]);
          e0[i] = d.x; e1[i] = d.y;
          if (p.gnb_silu) {
            e0[i] *= silu_grad_f(fmaf(xv.x, A.x, B.x));
            e1[i] *= silu_grad_f(fmaf(xv.y, A.y, B.y));
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float2 xv = unpack_bf16x2(wx[i]);
          s0 += e0[i]; s1 += e1[i];
          x0 = fmaf(e0[i], xv.x, x0); x1 = fmaf(e1[i], xv.y, x1);
        }
      }
    } else {
      for (int rr = r + ((h ^ r) & 1); rr < seg_end; rr += 2) {
        const uint32_t off = rr * 64 + ((uint32_t)(jch ^ ((rr >> 1) & 3)) << 4) + in_chunk;
        uint32_t wd, wx;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(wd) : "r"(buf_dy + off));
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(wx) : "r"(buf_x + off));
        const float2 d = unpack_bf16x2(wd), xv = unpack_bf16x2(wx);
        float e0 = d.x, e1 = d.y;
        if (p.gnb_silu) {
          e0 *= silu_grad_f(fmaf(xv.x, A.x, B.x));
          e1 *= silu_grad_f(fmaf(xv.y, A.y, B.y));
        }
        s0 += e0; s1 += e1;
        x0 = fmaf(e0, xv.x, x0); x1 = fmaf(e1, xv.y, x1);
      }
    }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
    x0 += __shfl_xor_sync(0xffffffffu, x0, 16); x1 += __shfl_xor_sync(0xffffffffu, x1, 16);
    if (h == 0 && col_ok) {
      float* d = p.gnb_sum + (2 * slab) * p.N + col;
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(s0), "f"(s1) : "memory");
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d + p.N), "f"(x0), "f"(x1) : "memory");
    }
    r = seg_end; ++slab; left = p.gnb_rows;
  }
}

// ---- register epilogues (every EPI but EPI_GENERIC): the accumulator stays in the wgmma fragment registers. Consumer warp
// w holds tile rows 16 w + lane / 4 + 8 h (h = 0, 1); its register 4 j + 2 h + e is column 8 j + 2 (lane % 4) + e. The two
// warps of a pair (w = 2 q, 2 q + 1) own the 32-row quarter q: per 32-column chunk each stages its 16 rows as bf16 with
// stmatrix into one 2 KB slot (32 rows x 64 B, 64B swizzle) of the pair's 8 KB, they meet on the pair's named barrier and
// lane 0 of the first warp issues the 32 x 32 TMA store. The fused GroupNorm sums and the interleaved next-row stores read
// the staged chunk as the parked epilogue did: each warp sums its own 16 rows, and the next-row stores alternate between the
// two warps. Per element the arithmetic is the
// parked epilogue's: bias, row-bias, scale, residuals, GEGLU / activation, round to bf16, in that order.
struct PairStage {
  uint32_t slots;   // the pair's 8 KB staging region: four 2 KB slots
  int bar;          // the pair's named barrier (2..5)
  int sub;          // 0: rows 0-15 of the quarter, issues the stores; 1: rows 16-31
  uint32_t round;   // chunks staged so far: the slot ring position, carried across tiles
};
struct EpiTile {
  int n0, n_out_total, row0, grp, valid_rows;   // row0 / grp: tensor-map coordinates of the quarter's first row
  long long m0;                                 // global row of the quarter's first row; valid_rows of its 32 exist
  long long m[2];                               // global rows 16 w + lane / 4 + 8 h of this thread
  bool ok[2];
};

// byte offset of row r, 16-byte column piece j, in a 64B-swizzled slot (rows 64 B apart: 16 r and 16 (r & ~15) swizzle alike)
SVDX_DEVINL uint32_t sw64(int r, int j) { return (uint32_t)(r * 64 + ((j ^ ((r >> 1) & 3)) << 4)); }
// the row this lane addresses for stmatrix / ldmatrix x4 number x of a warp's 16 x 32 chunk: matrix lane / 8 of the four
// covers column piece 2 x + (lane / 8) / 2 and rows 8 ((lane / 8) % 2) + [0, 8); register k of the x4 is fragment
// register pair (j, h) = (2 x + k / 2, k % 2)
SVDX_DEVINL uint32_t frag_row_addr(uint32_t base16, int lane, int x) {
  const int mi = lane >> 3;
  return base16 + sw64(8 * (mi & 1) + (lane & 7), 2 * x + (mi >> 1));
}
SVDX_DEVINL void stmatrix_x4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
SVDX_DEVINL void ldmatrix_x4(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr) : "memory");
}
// a chunk's 16 fragment values (f[4 j + 2 h + e]) -> this warp's 16 rows of a slot, bf16 (cvt.rn.bf16x2)
SVDX_DEVINL void stage_frag16(uint32_t base16, int lane, const float (&f)[16]) {
#pragma unroll
  for (int x = 0; x < 2; ++x)
    stmatrix_x4(frag_row_addr(base16, lane, x), pack_bf16x2(f[8 * x], f[8 * x + 1]), pack_bf16x2(f[8 * x + 2], f[8 * x + 3]),
                pack_bf16x2(f[8 * x + 4], f[8 * x + 5]), pack_bf16x2(f[8 * x + 6], f[8 * x + 7]));
}
// 16 rows x 32 bf16 columns of a row-major operand, fetched coalesced (lane: 16-byte piece lane % 4 of rows lane / 4 and
// lane / 4 + 8, 8 rows x 64 B per instruction); rows >= nrows read as zero
SVDX_DEVINL void load_rows16(const bf16* base, long long ld, int nrows, int lane, uint4 (&v)[2]) {
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int rr = (lane >> 2) + 8 * j;
    v[j] = rr < nrows ? *reinterpret_cast<const uint4*>(base + (long long)rr * ld + (lane & 3) * 8) : make_uint4(0u, 0u, 0u, 0u);
  }
}
SVDX_DEVINL void stage_rows16(uint32_t base16, int lane, const uint4 (&v)[2]) {
#pragma unroll
  for (int j = 0; j < 2; ++j) st_shared_v4(base16 + sw64((lane >> 2) + 8 * j, lane & 3), v[j].x, v[j].y, v[j].z, v[j].w);
}

template <int EPI, int BN>
SVDX_DEVINL void epilogue_regs(const TapGemmKParams& p, const float (&acc)[BN / 2], PairStage& ps, const EpiTile& t, int lane, float s_acc,
                               float s_r1, float s_r2) {
  constexpr bool GEGLU = EPI == EPI_GEGLU;
  constexpr bool RES = EPI == EPI_RES || EPI == EPI_RES_GN;
  constexpr bool GN = EPI == EPI_FAST_GN || EPI == EPI_RES_GN || EPI == EPI_FAST_IL_GN;
  constexpr bool IL = EPI == EPI_FAST_IL || EPI == EPI_FAST_IL_GN;
  constexpr bool GNB = EPI == EPI_FAST_GNB;
  constexpr int BN_OUT = GEGLU ? BN / 2 : BN;
  const int cq = 2 * (lane & 3);
  const bool issuer = ps.sub == 0 && lane == 0;
  const bool save_pre = GEGLU && p.pre != nullptr;
  const int vr = t.valid_rows - 16 * ps.sub;             // rows of this warp's 16 that exist
  const long long mw = t.m0 + 16 * ps.sub;               // global row of this warp's first row
  const float* bias = p.bias;
  // rows past the end read row 0's operands: they are clipped by the store and skipped by the sums
  const float* rb[2] = {nullptr, nullptr};
  const bf16* r2[2] = {nullptr, nullptr};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!GEGLU && p.rowbias) rb[h] = p.rowbias + (t.ok[h] ? t.m[h] / p.rowbias_div : 0) * p.ldrb;
    if (RES && p.res2) r2[h] = p.res2 + (t.ok[h] ? t.m[h] : 0) * p.ldr2;
  }
#pragma unroll
  for (int ch = 0; ch < BN_OUT / 32; ++ch) {
    const int col0 = t.n0 + 32 * ch;
    if (col0 >= t.n_out_total) break;                     // pair-uniform
    // slots: a ring of four single-chunk slots (wait until the store three chunks back has been read before the barrier
    // that frees its slot); GNB: dy | x slot pairs, alternating; GEGLU with pre: value | gate | output, fixed
    const uint32_t slot = ps.slots + 2048u * (GNB ? 2 * (ps.round & 1) : save_pre ? 2 : (ps.round & 3));
    const uint32_t mine = slot + 1024u * ps.sub;
    uint4 xa[2];                                          // RES: res1 rows; GNB: the GroupNorm input rows
    if constexpr (RES) {
      if (p.res1) load_rows16(p.res1 + mw * p.ldr1 + col0, p.ldr1, vr, lane, xa);
    }
    if constexpr (GNB) {
      const bool src1 = col0 < p.gnb_c1;
      const long long xld = src1 ? p.gnb_ldx : p.gnb_ldx2;
      load_rows16((src1 ? p.gnb_x + col0 : p.gnb_x2 + (col0 - p.gnb_c1)) + mw * xld, xld, vr, lane, xa);
    }
    uint32_t a2[8];
    if constexpr (RES) {
      if (p.res2) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a2[k] = *reinterpret_cast<const uint32_t*>(r2[k & 1] + col0 + 8 * (k >> 1) + cq);
      }
    }
    float f[16], g[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      f[i] = acc[16 * ch + i];
      if constexpr (GEGLU) g[i] = acc[BN_OUT / 2 + 16 * ch + i];
    }
    if (bias) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col0 + 8 * j + cq));
        f[4 * j] += b.x; f[4 * j + 1] += b.y; f[4 * j + 2] += b.x; f[4 * j + 3] += b.y;
        if constexpr (GEGLU) {
          const float2 bg = __ldg(reinterpret_cast<const float2*>(bias + p.N / 2 + col0 + 8 * j + cq));
          g[4 * j] += bg.x; g[4 * j + 1] += bg.y; g[4 * j + 2] += bg.x; g[4 * j + 3] += bg.y;
        }
      }
    }
    if (!GEGLU && p.rowbias) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(rb[k & 1] + col0 + 8 * (k >> 1) + cq));
        f[2 * k] += b.x; f[2 * k + 1] += b.y;
      }
    }
    if constexpr (EPI == EPI_FAST_ACT) act_n(f, p.act);
    if constexpr (RES) {
      if (p.scales) {
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] = __fmul_rn(f[i], s_acc);
      }
      if (p.res1) {
        // the coalesced rows go through this warp's half of the slot that is about to receive its output, back in
        // fragment order
        uint32_t a1[8];
        stage_rows16(mine, lane, xa);
        __syncwarp();
        ldmatrix_x4(frag_row_addr(mine, lane, 0), a1[0], a1[1], a1[2], a1[3]);
        ldmatrix_x4(frag_row_addr(mine, lane, 1), a1[4], a1[5], a1[6], a1[7]);
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float2 a = unpack_bf16x2(a1[k]);
          f[2 * k] = __fmaf_rn(s_r1, a.x, f[2 * k]); f[2 * k + 1] = __fmaf_rn(s_r1, a.y, f[2 * k + 1]);
        }
      }
      if (p.res2) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float2 a = unpack_bf16x2(a2[k]);
          f[2 * k] = __fmaf_rn(s_r2, a.x, f[2 * k]); f[2 * k + 1] = __fmaf_rn(s_r2, a.y, f[2 * k + 1]);
        }
      }
    }
    if constexpr (GEGLU) {
      if (save_pre) {
        // the bf16 pre-activation: value and gate columns through slots 0 and 1
        stage_frag16(ps.slots + 1024u * ps.sub, lane, f);
        stage_frag16(ps.slots + 2048u + 1024u * ps.sub, lane, g);
        fence_proxy_async_smem();
        if (issuer) bulk_wait_read<0>();                 // the previous chunk's output store has left slot 2
        named_bar_sync(ps.bar, 64);
        if (issuer) {
          tma_store_3d(&p.tmpre, ps.slots, col0, t.row0, t.grp);
          tma_store_3d(&p.tmpre, ps.slots + 2048u, p.N / 2 + col0, t.row0, t.grp);
          bulk_commit();
        }
      }
      // the reference applies GEGLU on the bf16-rounded projection (autocast F.linear output)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float fv = __bfloat162float(__float2bfloat16(f[i]));
        const float gv = __bfloat162float(__float2bfloat16(g[i]));
        f[i] = fv * gelu_erf_f(gv);
      }
    }
    stage_frag16(mine, lane, f);
    if constexpr (GNB) stage_rows16(mine + 2048u, lane, xa);
    fence_proxy_async_smem();
    if (issuer) {
      if (GNB || save_pre) bulk_wait_read<0>();
      else bulk_wait_read<2>();
    }
    named_bar_sync(ps.bar, 64);
    if (issuer) { store_chunk<IL>(p, slot, col0, t.row0, t.grp); bulk_commit(); }
    if constexpr (IL) {
      if ((ps.round & 1) == (uint32_t)ps.sub) il_store_next_row(p, slot, col0, t.row0, lane);
    }
    // each warp sums its own 16 rows of the staged chunk, so the two warps of a pair run their sums at the same time
    if constexpr (GN) gn_chunk_sums(p, mine, lane, col0, t.n_out_total, mw, max(0, min(16, vr)));
    if constexpr (GNB) gnb_chunk_sums<16>(p, mine, mine + 2048u, lane, col0, t.n_out_total, mw, max(0, min(16, vr)));
    ++ps.round;
  }
}

// EPI_F32: each consumer warp stages its own 16 rows x 32 columns of a chunk as fp32 (2 KB, the 128B swizzle of tmo) with
// st.shared.v2 straight from the fragments, alternating between the two halves of its 4 KB region, and its lane 0 issues
// the 16-row TMA store or reduce-add (tmo16). No pair barrier: the two warps of a quarter run their chunks independently.
// Per element the arithmetic is the parked epilogue's: acc, times scales[0] when given.
template <int BN>
SVDX_DEVINL void epilogue_f32(const TapGemmKParams& p, const float (&acc)[BN / 2], EpiStage& st, const EpiTile& t, int sub, int lane,
                              float s_acc) {
  const bool reduce = p.out_dtype == SVDX_OUT_F32_ATOMIC;
  // fragment register 4 j + 2 h + e: row lane / 4 + 8 h, columns 8 j + 2 (lane % 4) + e = 16-byte piece 2 j + (lane % 4) / 2,
  // 8-byte half lane % 2; rows lane / 4 and lane / 4 + 8 swizzle alike (128B swizzle: piece ^= row % 8)
  const uint32_t row_off = (uint32_t)(lane >> 2) * 128u + 8u * (lane & 1);
  const int sw = lane >> 2, pc = (lane & 3) >> 1;
#pragma unroll
  for (int ch = 0; ch < BN / 32; ++ch) {
    const int col0 = t.n0 + 32 * ch;
    if (col0 >= t.n_out_total) break;                     // warp-uniform
    if (lane == 0) bulk_wait_read<1>();                   // the half written two chunks ago has been read out
    __syncwarp();
    const uint32_t buf = st.base + st.off + row_off;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t a = buf + ((uint32_t)((2 * j + pc) ^ sw) << 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float x = acc[16 * ch + 4 * j + 2 * h], y = acc[16 * ch + 4 * j + 2 * h + 1];
        if (p.scales) { x *= s_acc; y *= s_acc; }
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + h * 1024u), "f"(x), "f"(y) : "memory");
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      const uint32_t src = st.base + st.off;
      if (reduce) tma_reduce_add_3d(&p.tmo16, src, col0, t.row0 + 16 * sub, t.grp);
      else tma_store_3d(&p.tmo16, src, col0, t.row0 + 16 * sub, t.grp);
      bulk_commit();
    }
    st.off ^= 2048;
  }
}

// Epilogue of one accumulator tile for one thread (= one output row): this warp takes the 32-column
// chunks half, half+2, ...; bias / row-bias / GEGLU / residuals / scales, then staged TMA stores (or direct 16-byte
// stores when the output cannot be described by a tensor map).
SVDX_DEVINL void epilogue_tile(const TapGemmKParams& p, uint32_t t_base, long long m, bool row_ok, int n0, int half, int bn_out,
                               int n_out_total, float s_acc, float s_r1, float s_r2, EpiStage& st, int lane) {
      if (p.probe == 2) return;
      const float* rb = (p.rowbias && row_ok) ? p.rowbias + (m / p.rowbias_div) * p.ldrb : nullptr;
      for (int c = half * 32; c < bn_out; c += 64) {
        uint32_t v[32];
        uint32_t gte[32];
        const int col0 = n0 + c;
        if (col0 >= n_out_total) break;   // warp-uniform
        const bool full_chunk = (col0 + 32 <= n_out_total);
        // issue the global reads of this chunk before reading the accumulator so their latency overlaps
        uint4 rr1[4], rr2[4];
        if (row_ok && full_chunk) {
          if (p.res1) {
            const uint4* r1p = reinterpret_cast<const uint4*>(p.res1 + m * p.ldr1 + col0);
#pragma unroll
            for (int k = 0; k < 4; ++k) rr1[k] = r1p[k];
          }
          if (p.res2) {
            const uint4* r2p = reinterpret_cast<const uint4*>(p.res2 + m * p.ldr2 + col0);
#pragma unroll
            for (int k = 0; k < 4; ++k) rr2[k] = r2p[k];
          }
        }
        __syncwarp();
        acc_ld32(t_base, c, v);
        if (p.geglu) acc_ld32(t_base, bn_out + c, gte);
        float f[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(v[i]);
        if (p.geglu) {
          float g[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) g[i] = __uint_as_float(gte[i]);
          if (p.bias) {
            if (full_chunk && ((p.N / 2) & 3) == 0) {
              const float4* bv = reinterpret_cast<const float4*>(p.bias + col0);
              const float4* bg = reinterpret_cast<const float4*>(p.bias + p.N / 2 + col0);
#pragma unroll
              for (int k = 0; k < 8; ++k) {
                const float4 x4 = __ldg(bv + k), y4 = __ldg(bg + k);
                f[4 * k] += x4.x; f[4 * k + 1] += x4.y; f[4 * k + 2] += x4.z; f[4 * k + 3] += x4.w;
                g[4 * k] += y4.x; g[4 * k + 1] += y4.y; g[4 * k + 2] += y4.z; g[4 * k + 3] += y4.w;
              }
            } else {
#pragma unroll
              for (int i = 0; i < 32; ++i) {
                if (full_chunk || col0 + i < n_out_total) {
                  f[i] += __ldg(p.bias + col0 + i);
                  g[i] += __ldg(p.bias + p.N / 2 + col0 + i);
                }
              }
            }
          }
          if (p.pre) {
            if (p.tma_store) {
              stage_store_bf16(&p.tmpre, st, lane, f, col0);
              stage_store_bf16(&p.tmpre, st, lane, g, p.N / 2 + col0);
            } else if (row_ok) {
              bf16* pv = p.pre + m * p.ldpre + col0;
              bf16* pg = pv + p.N / 2;
              if (full_chunk) {
#pragma unroll
                for (int i = 0; i < 32; i += 8) {
                  uint4 a, b;
                  a.x = pack_bf16x2(f[i], f[i + 1]); a.y = pack_bf16x2(f[i + 2], f[i + 3]);
                  a.z = pack_bf16x2(f[i + 4], f[i + 5]); a.w = pack_bf16x2(f[i + 6], f[i + 7]);
                  b.x = pack_bf16x2(g[i], g[i + 1]); b.y = pack_bf16x2(g[i + 2], g[i + 3]);
                  b.z = pack_bf16x2(g[i + 4], g[i + 5]); b.w = pack_bf16x2(g[i + 6], g[i + 7]);
                  *reinterpret_cast<uint4*>(pv + i) = a;
                  *reinterpret_cast<uint4*>(pg + i) = b;
                }
              } else {
                for (int i = 0; i < 32; ++i)
                  if (col0 + i < n_out_total) { pv[i] = __float2bfloat16(f[i]); pg[i] = __float2bfloat16(g[i]); }
              }
            }
          }
          // the reference applies GEGLU on the bf16-rounded projection (autocast F.linear output)
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float fv = __bfloat162float(__float2bfloat16(f[i]));
            const float gv = __bfloat162float(__float2bfloat16(g[i]));
            f[i] = fv * gelu_erf_f(gv);
          }
        } else {
          if (p.bias) {
            if (full_chunk) {
              const float4* bp = reinterpret_cast<const float4*>(p.bias + col0);
#pragma unroll
              for (int k = 0; k < 8; ++k) {
                const float4 b4 = __ldg(bp + k);
                f[4 * k] += b4.x; f[4 * k + 1] += b4.y; f[4 * k + 2] += b4.z; f[4 * k + 3] += b4.w;
              }
            } else {
              for (int i = 0; i < 32; ++i)
                if (col0 + i < n_out_total) f[i] += __ldg(p.bias + col0 + i);
            }
          }
        }
        if (rb) {
          if (full_chunk && (reinterpret_cast<uintptr_t>(rb + col0) & 15) == 0) {
            const float4* bp = reinterpret_cast<const float4*>(rb + col0);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const float4 b4 = __ldg(bp + k);
              f[4 * k] += b4.x; f[4 * k + 1] += b4.y; f[4 * k + 2] += b4.z; f[4 * k + 3] += b4.w;
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (full_chunk || col0 + i < n_out_total) f[i] += __ldg(rb + col0 + i);
          }
        }
        if (p.scales) {
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] *= s_acc;
        }
        if (p.res1 && row_ok) {
          const bf16* r1 = p.res1 + m * p.ldr1 + col0;
          if (full_chunk) {
#pragma unroll
            for (int i = 0; i < 32; i += 8) {
              const uint4 u = rr1[i >> 3];
              float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c2 = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
              f[i] += s_r1 * a.x; f[i + 1] += s_r1 * a.y; f[i + 2] += s_r1 * b.x; f[i + 3] += s_r1 * b.y;
              f[i + 4] += s_r1 * c2.x; f[i + 5] += s_r1 * c2.y; f[i + 6] += s_r1 * d.x; f[i + 7] += s_r1 * d.y;
            }
          } else {
            for (int i = 0; i < 32; ++i)
              if (col0 + i < n_out_total) f[i] += s_r1 * __bfloat162float(r1[i]);
          }
        }
        if (p.res2 && row_ok) {
          const bf16* r2 = p.res2 + m * p.ldr2 + col0;
          if (full_chunk) {
#pragma unroll
            for (int i = 0; i < 32; i += 8) {
              const uint4 u = rr2[i >> 3];
              float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c2 = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
              f[i] += s_r2 * a.x; f[i + 1] += s_r2 * a.y; f[i + 2] += s_r2 * b.x; f[i + 3] += s_r2 * b.y;
              f[i + 4] += s_r2 * c2.x; f[i + 5] += s_r2 * c2.y; f[i + 6] += s_r2 * d.x; f[i + 7] += s_r2 * d.y;
            }
          } else {
            for (int i = 0; i < 32; ++i)
              if (col0 + i < n_out_total) f[i] += s_r2 * __bfloat162float(r2[i]);
          }
        }
        // ---- store
        if (p.probe == 1) {
          float acc = 0.f;
#pragma unroll
          for (int i = 0; i < 32; ++i) acc += f[i];
          if (acc == 123.456f) reinterpret_cast<float*>(p.out)[0] = acc;   // keeps the math alive
        } else if (p.tma_store) {
          if (p.out_dtype == SVDX_OUT_BF16) stage_store_bf16(&p.tmo, st, lane, f, col0);
          else stage_store_f32(&p.tmo, st, lane, f, col0, p.out_dtype == SVDX_OUT_F32_ATOMIC);
        } else if (!row_ok) {
          // nothing to write for rows past the end
        } else if (p.out_dtype == SVDX_OUT_BF16) {
          bf16* o = reinterpret_cast<bf16*>(p.out) + m * p.ldo + col0;
          if (full_chunk) {
#pragma unroll
            for (int i = 0; i < 32; i += 8) {
              uint4 a;
              a.x = pack_bf16x2(f[i], f[i + 1]); a.y = pack_bf16x2(f[i + 2], f[i + 3]);
              a.z = pack_bf16x2(f[i + 4], f[i + 5]); a.w = pack_bf16x2(f[i + 6], f[i + 7]);
              *reinterpret_cast<uint4*>(o + i) = a;
            }
          } else {
            for (int i = 0; i < 32; ++i)
              if (col0 + i < n_out_total) o[i] = __float2bfloat16(f[i]);
          }
        } else if (p.out_dtype == SVDX_OUT_F32) {
          float* o = reinterpret_cast<float*>(p.out) + m * p.ldo + col0;
          if (full_chunk) {
#pragma unroll
            for (int i = 0; i < 32; i += 4)
              *reinterpret_cast<float4*>(o + i) = make_float4(f[i], f[i + 1], f[i + 2], f[i + 3]);
          } else {
            for (int i = 0; i < 32; ++i)
              if (col0 + i < n_out_total) o[i] = f[i];
          }
        } else {
          float* o = reinterpret_cast<float*>(p.out) + m * p.ldo + col0;
          if (full_chunk) {
#pragma unroll
            for (int i = 0; i < 32; i += 4)   // 16-byte vector reductions: 4x fewer L2 atomic requests
              asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + i), "f"(f[i]), "f"(f[i + 1]), "f"(f[i + 2]), "f"(f[i + 3])
                           : "memory");
          } else {
            for (int i = 0; i < 32; ++i)
              if (col0 + i < n_out_total) atomicAdd(o + i, f[i]);
          }
        }
      }
}

}  // namespace svdx

// host: validates the descriptor and fills the kernel parameter block.
int svdx_tapgemm_fill(const SvdxTapGemm* d, svdx::TapGemmKParams& p);
