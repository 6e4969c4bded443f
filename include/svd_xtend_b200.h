/*
 * svd_xtend_b200 — C ABI of the H100-native (sm_90a) SVD spatio-temporal UNet hot path.
 *
 * Every entry point takes raw device pointers, explicit shapes/strides and a CUDA stream
 * (passed as void* == cudaStream_t). Contract for ALL functions:
 *   - return 0 on success, <0 on error (see SVDX_E_*); never throw, never allocate or free
 *     device memory, never synchronise the device; re-entrant across streams;
 *   - bf16 = __nv_bfloat16 storage, fp32 accumulation everywhere.
 *
 * The reference (pixeli99/SVD_Xtend) is pure Python on top of diffusers; the operator each entry
 * replaces is therefore the ATen/cuDNN/cuBLAS call reached from the reference's module code.
 * The replaced interface is cited per function as  <reference file:line> -> <diffusers op [D]>.
 * "[D]" = code that lives in the un-vendored diffusers dependency (SURVEY.md Appendix B).
 */
#ifndef SVD_XTEND_B200_H_
#define SVD_XTEND_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SVDX_OK 0
#define SVDX_E_BADARG (-1)     /* unsupported shape / alignment / null pointer */
#define SVDX_E_CUDA (-2)       /* CUDA runtime / driver error on launch */
#define SVDX_E_NODRIVER (-3)   /* cuTensorMapEncodeTiled entry point unavailable */

#define SVDX_MAX_TAPS 27

/* A-operand addressing modes of svdx_tapgemm */
#define SVDX_A_ROWS 0    /* A is [groups][rows_per_group][K] (a plain matrix when groups==1);
                            tap t reads rows shifted by tap_d0[t] inside the group, rows outside
                            the group read as zero (this is the (3,1,1) temporal conv / a linear) */
#define SVDX_A_CONV2D 1  /* A is [nimg][H][W][K] channels-last; tap t reads pixel (h+tap_d1[t],
                            w+tap_d0[t]) of image n+tap_d2[t]; out-of-image reads are zero
                            (3x3 conv padding=1, and the parity-plane form of the stride-2 conv).
                            Any width W: when 128 % W == 0 or W % 128 == 0 the tile's pixels are
                            fetched as shifted row boxes; at every other width as one TMA im2col
                            load per k-block (taps then need |tap_d0|, |tap_d1| <= 1). The two
                            forms give bit-identical results, with or without interleave. */

#define SVDX_OUT_BF16 0
#define SVDX_OUT_F32 1
#define SVDX_OUT_F32_ATOMIC 2  /* out += result (fp32 red.add), used by split-K weight gradients */
/* fp32 outputs (SVDX_OUT_F32 / SVDX_OUT_F32_ATOMIC) without bias / rowbias / res1 / res2 / GEGLU run an epilogue from the
 * accumulator registers (scales[0] applied; any operand majors and b_mode, any N, split-K); fp32 outputs with those operands
 * run the generic epilogue. Both give bit-identical stores. fp32 rows must be 16-byte aligned (ldo % 4 == 0). */

/*
 * svdx_tapgemm — the one tensor-core contraction of the path (wgmma, register accumulators,
 * TMA-fed 128B-swizzled shared memory, warp-specialised persistent CTAs):
 *
 *     acc[m, n] = sum_{t < num_taps} sum_{k < K}  A_t[m, k] * B[n, t*K + k]
 *     v         = acc + bias[n] + rowbias[m / rowbias_div, n]
 *     v         = geglu ? v[:, :N/2] * gelu_erf(v[:, N/2:]) : v
 *     out[m, n] = scales[0] * v + scales[1] * res1[m, n] + scales[2] * res2[m, n]
 *
 * Replaces, with the epilogue fused:
 *   F.linear      — Attention.to_q/to_k/to_v/to_out, FeedForward proj/out, proj_in/proj_out,
 *                   time_emb_proj, TimestepEmbedding  [D]; reached from
 *                   src/unet_spatio_temporal_condition.py:138-144,170-233
 *   F.conv2d 3x3  — ResnetBlock2D.conv1/conv2, Downsample2D, Upsample2D.conv [D], conv_in/conv_out
 *                   (src/unet_spatio_temporal_condition.py:128-133,241-246)
 *   F.conv2d 1x1  — ResnetBlock2D.conv_shortcut [D]
 *   F.conv3d (3,1,1) — TemporalResnetBlock.conv1/conv2 [D]
 *   GEGLU, AlphaBlender, residual adds [D] (epilogue)
 * and their data/weight gradients (dgrad = same contraction on transposed weights; wgrad =
 * a_major_mn = b_major_mn = 1 with SVDX_OUT_F32_ATOMIC).
 */
typedef struct SvdxTapGemm {
  /* A operand (bf16) */
  const void* a;
  int64_t lda;          /* elements between consecutive rows/pixels */
  int32_t a_mode;       /* SVDX_A_ROWS / SVDX_A_CONV2D */
  int32_t a_major_mn;   /* 0: A[m][k] k contiguous. 1 (ROWS, groups==1 only): memory is [k][m], m contiguous; a bf16 output runs
                           the generic epilogue, so no gn_sum / gnb sums / act / interleave / block_n 320 */
  int32_t rows_per_group, groups;      /* ROWS   */
  int32_t W, H, nimg;                  /* CONV2D (and b_mode 1): any W > 0; see SVDX_A_CONV2D for how each width is tiled */
  int32_t num_taps;
  int32_t tap_d0[SVDX_MAX_TAPS];
  int32_t tap_d1[SVDX_MAX_TAPS];
  int32_t tap_d2[SVDX_MAX_TAPS];
  /* B operand (bf16): [N][num_taps*K] (k contiguous), or if b_major_mn: memory [K][N], n contiguous */
  const void* b;
  int64_t ldb;
  int32_t b_major_mn;   /* 1: with a bf16 output, bias / rowbias only (with res1 / res2 / scales it runs the generic epilogue);
                           no gn_sum / gnb sums / act / interleave / GEGLU */
  int32_t b_mode;       /* weight-gradient forms (a_major_mn = b_major_mn = 1): 0 plain [K][N];
                           1: B is a channels-last image tensor [nimg][H][W][N], contraction row p (an output
                              pixel) reads pixel shifted by (tap_d0[0], tap_d1[0]) of image +tap_d2[0], zero outside
                              (dW of a 3x3 conv tap); K = images*H*W output pixels;
                           2: B is [groups][rows_per_group][N], contraction row reads row + tap_d0[0] of its
                              group, zero outside (dW of a (3,1,1) temporal conv tap) */
  /* problem */
  int32_t M, N, K;      /* M output rows, N = B rows (before GEGLU halving), K = contraction per tap */
  int32_t block_n;      /* multiple of 32, <= 256 (multiple of 64 when b_major_mn); 320 = 320-column tiles (run as two 160-wide tiles)
                           (two N = 160 MMAs per k-step on one A stage): M >= 512, N % 320 == 0, bf16 TMA-store epilogues only */
  int32_t split_k;      /* >= 1; > 1 requires SVDX_OUT_F32_ATOMIC */
  /* epilogue */
  void* out;
  int64_t ldo;
  int32_t out_dtype;
  int32_t geglu;        /* out has N/2 columns */
  const float* bias;    /* [N] or NULL */
  const float* rowbias; /* [ceil(M/rowbias_div)][ldrb] or NULL */
  int32_t rowbias_div;
  int64_t ldrb;
  const void* res1;     /* bf16 [M][ldr1] or NULL */
  int64_t ldr1;
  const void* res2;
  int64_t ldr2;
  const float* scales;  /* device float[3] {acc, res1, res2} or NULL (= 1,1,1) */
  void* pre;            /* geglu: bf16 [M][ldpre] pre-activation (value | gate) saved for backward, or NULL */
  int64_t ldpre;
  /* GroupNorm statistics of the OUTPUT, fused into the epilogue ("GroupNorm fused into the conv epilogue"): when gn_sum is
   * not NULL the epilogue also accumulates, per statistics slab s = m / gn_rows and output channel n, the sum and the sum
   * of squares of the bf16 values it stores:  gn_sum[(2*s + 0) * gn_ld + n] += out[m][n],  gn_sum[(2*s + 1) * gn_ld + n] +=
   * out[m][n]^2  (fp32 red.add; column sums of each staged 32x32 chunk, warp-reduced). gn_rows = rows per slab (H*W per
   * frame for the spatial GroupNorms, T*H*W per clip for the temporal ones); the buffer must be zero on entry. The consumer
   * (svdx_groupnorm_apply_fused) folds channels into groups, so a later channel concatenation needs no extra pass.
   * Requires a bf16 output written through the TMA-store epilogues (N % 32 == 0, 16-byte aligned rows), no split-K, no GEGLU. */
  float* gn_sum;
  int64_t gn_ld;        /* floats per (slab, moment) row, >= N */
  int32_t gn_rows;
  /* GroupNorm BACKWARD statistics fused into the epilogue (pass 1 of F.group_norm's backward): set on the GEMM / conv that
   * WRITES dy = dL/d(GroupNorm output) — the data gradient of the conv that consumed the normalised tensor. gnb_x (channels
   * [0, gnb_c1)) and gnb_x2 (the rest; NULL = single source) are the GroupNorm's bf16 INPUT, gnb_ab[(2*s + 0) * N + n] /
   * [(2*s + 1) * N + n] the forward scale / shift of channel n in statistics slab s = m / gnb_rows (written by
   * svdx_groupnorm_apply_fused, y = act(x * scale + shift); only read when gnb_silu). The epilogue accumulates
   *   gnb_sum[(2*s + 0) * N + n] += e,  gnb_sum[(2*s + 1) * N + n] += e * x[m][n],   e = dy[m][n] * act'(x * scale + shift)
   * on the bf16 values it stores (buffer zero on entry); svdx_groupnorm_bwd_fused turns them into dx / dgamma / dbeta with ONE
   * pass over x and dy. Requires the plain bf16 TMA-store epilogue (no residual / scales / GEGLU / split-K / gn_sum), N even. */
  const void* gnb_x;
  int64_t gnb_ldx;
  const void* gnb_x2;
  int64_t gnb_ldx2;
  int32_t gnb_c1;
  const float* gnb_ab;
  float* gnb_sum;
  int32_t gnb_rows;
  int32_t gnb_silu;
  /* Interleaved store: the phase form of Upsample2D [D] (nearest 2x upsample, then a 3x3 conv with padding 1), which is four
   * 2x2-tap convolutions on the LOW-RES input, one per output parity (phase_h, phase_w). When interleave != 0 (CONV2D mode),
   * output row (n, h, w) of the low-res geometry {W, H, nimg} is written to row (n*2H + 2h + phase_h) * 2W + 2w + phase_w of
   * the [nimg][2H][2W][ldo] high-res output, so the four launches fill it without the upsampled input ever existing.
   * gn_sum slabs still count low-res rows (gn_rows = H*W: the four phases of a frame accumulate into one slab).
   * Requires the plain bf16 TMA-store epilogue (bias only: no rowbias / residual / scales / GEGLU / split-K / gnb sums).
   * W >= 32: any W and H (a 32-row store chunk that crosses into the next image row or image is stored in two pieces).
   * W < 32: W | 32 and H*W % 32 == 0 (each 32-row store chunk is whole rows of one image). */
  int32_t interleave;
  int32_t phase_h, phase_w;
  /* Activation epilogue (the MLP fc1 of the CLIP image encoder [transformers CLIPMLP]): out = act(acc + bias), bf16, with
   * act = SVDX_ACT_GELU (erf form, gelu_erf_f) or SVDX_ACT_QUICK_GELU (x * sigmoid(1.702 x)); SVDX_ACT_NONE (0) = no activation.
   * Requires the plain bf16 TMA-store epilogue (bias only: no rowbias / residual / scales / GEGLU / split-K / gn_sum / gnb sums /
   * interleave; N % 32 == 0, 16-byte aligned rows). */
  int32_t act;
} SvdxTapGemm;

#define SVDX_ACT_NONE 0
#define SVDX_ACT_GELU 1
#define SVDX_ACT_QUICK_GELU 2

int svdx_tapgemm(const SvdxTapGemm* desc, void* stream);

/* Second half of a split-K svdx_tapgemm (fp32 partial sums accumulated with SVDX_OUT_F32_ATOMIC into ws): applies the
 * same epilogue  out = scales[0]*(ws + bias + rowbias[m / rowbias_div]) + scales[1]*res1 + scales[2]*res2  -> bf16.
 * Used for the 5x8 / 10x16 latent levels where M gives too few output tiles to fill the SMs.
 * The workspace is CONSUMED: every element read is reset to zero, so a caller can keep one zeroed workspace per shape
 * and never memset it again. */
int svdx_splitk_epilogue(float* ws, int64_t ldw, void* out, int64_t ldo, int64_t rows, int32_t cols, const float* bias,
                         const float* rowbias, int32_t rowbias_div, int64_t ldrb, const void* res1, int64_t ldr1,
                         const void* res2, int64_t ldr2, const float* scales, void* stream);

/* number of SMs the persistent kernels size their grids to (queried once) */
int svdx_num_sms(void);
/* enable peer access from the current device to peer_device (needed before svdx_adamw_step_p2p dereferences arenas that live on,
 * or were IPC-mapped from, that GPU); idempotent; fails when the GPUs have no P2P path */
int svdx_enable_peer_access(int32_t peer_device);
/* CUDA IPC of a device buffer between the processes of one node (one process per GPU). export: the 64-byte handle of the
 * allocation that contains ptr + ptr's byte offset inside it. import (call it with the CONSUMING GPU current): maps the
 * allocation into this process for that GPU (peer access enabled lazily) and returns the address corresponding to ptr. An
 * allocation can be imported once per process; the mapping lives until the process exits. */
int svdx_ipc_export(const void* ptr, void* handle64_out, int64_t* offset_out);
int svdx_ipc_import(const void* handle64, int64_t offset, void** ptr_out);
/* sizeof(SvdxTapGemm) (which==0) / sizeof(SvdxAttn) (which==1): lets bindings verify their struct layout */
int svdx_struct_size(int which);
/* human-readable last error of this thread */
const char* svdx_last_error(void);

/* ------------------------------------------------------------------ normalisation
 * GroupNorm(32)+SiLU over channels-last activations, replaces F.group_norm + F.silu of
 * ResnetBlock2D.norm1/norm2, TemporalResnetBlock.norm1/norm2 (stats over T*H*W),
 * TransformerSpatioTemporalModel.norm [D], conv_norm_out (src/unet_spatio_temporal_condition.py:238-239,480-481).
 * x is [ngroups_outer][rows][C] bf16 where one statistics group spans `rows` rows x (C/32) channels.
 * A second source x2 (C2 channels) is concatenated along channels (the up-block torch.cat).
 */
/* Per-(slab, channel) sums of a tensor no producing epilogue covered: sums[(2*s + 0) * ld + c] += x, sums[(2*s + 1) * ld + c]
 * += x^2 over the rows of slab s, exactly the gn_sum contract of svdx_tapgemm (sums zero on entry, 16-byte aligned,
 * ld >= C1 + C2, ld % 4 == 0). */
int svdx_groupnorm_sums(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2,
                        int32_t outer, int32_t rows, float* sums, int64_t ld, void* stream);
/* GroupNorm(+SiLU) apply from per-CHANNEL sums (gn_sum of the producing svdx_tapgemm epilogues, or svdx_groupnorm_sums):
 * csum1 / csum2 are the [outer][2][ld] fp32 sum / sum-of-squares arrays of the two channel-concatenated sources (csum2 NULL
 * when C2 == 0). Every CTA first folds the channels of its slab into the group statistics (shared memory), the CTA with
 * blockIdx.x == 0 of each slab also writes mean / rstd [outer][groups] for the backward. gamma / beta must be 16-byte
 * aligned. ab_out (optional): fp32 [outer][2][C], receives the per-channel scale / shift of every slab
 * (y = act(x * scale + shift)): the gnb_ab table of the GroupNorm-backward sums (svdx_tapgemm, svdx_groupnorm_bwd_sums). */
int svdx_groupnorm_apply_fused(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2,
                               int32_t outer, int32_t rows, int32_t num_groups, float eps,
                               const float* csum1, int64_t ldc1, const float* csum2, int64_t ldc2,
                               float* mean, float* rstd, const float* gamma, const float* beta,
                               int32_t fuse_silu, void* y, int64_t ldy, float* ab_out, void* stream);
/* Backward pass 1 for a dy no dgrad epilogue covered: the gnb_sum contract of svdx_tapgemm, sums[(2*s + 0) * C + c] += e,
 * sums[(2*s + 1) * C + c] += e * x, e = dy * silu'(x * scale + shift) with scale / shift from the ab table of
 * svdx_groupnorm_apply_fused (read only when fuse_silu). sums: fp32 [outer][2][C], zero on entry, 16-byte aligned. */
int svdx_groupnorm_bwd_sums(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2,
                            const void* dy, int64_t lddy, int32_t outer, int32_t rows, const float* ab, int32_t fuse_silu,
                            float* sums, void* stream);
/* backward pass 2: csum = the [outer][2][C] sums of pass 1 (svdx_tapgemm gnb_sum or svdx_groupnorm_bwd_sums). One launch,
 * one pass over x and dy: every CTA folds the channel sums into the group sums, dgamma / dbeta (optional, fp32, accumulated)
 * come straight from the channel sums. dres (optional, bf16 [outer*rows][lddres], single-source form only): a gradient
 * already accumulated on x through its residual use; dx = GroupNorm backward + dres in the same pass. */
int svdx_groupnorm_bwd_fused(const void* x, int64_t ldx, int32_t C1, const void* x2, int64_t ldx2, int32_t C2,
                             const void* dy, int64_t lddy, int32_t outer, int32_t rows, int32_t num_groups,
                             const float* mean, const float* rstd, const float* gamma, const float* beta,
                             int32_t fuse_silu, const float* csum, void* dx, int64_t lddx, void* dx2, int64_t lddx2,
                             float* dgamma, float* dbeta, const void* dres, int64_t lddres, void* stream);

/* LayerNorm over the last dim (C <= 2560, C % 8 == 0), replaces F.layer_norm of
 * BasicTransformerBlock.norm1-3 / TemporalBasicTransformerBlock.norm_in,norm1-3 [D].
 * addvec (optional, [ceil(rows/add_div)][C] fp32): row r gets addvec[r / add_div] added before normalisation and
 * the bf16 sum is written to xsum (the "hidden_states + emb" of TransformerSpatioTemporalModel [D]). */
int svdx_layernorm_fwd(const void* x, int64_t ldx, int32_t rows, int32_t C, const float* gamma, const float* beta,
                       float eps, void* y, int64_t ldy, float* mean, float* rstd,
                       const float* addvec, int32_t add_div, void* xsum, int64_t ldxs, void* stream);
int svdx_layernorm_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, int32_t rows, int32_t C,
                       const float* gamma, const float* mean, const float* rstd,
                       void* dx, int64_t lddx, const void* dres, int64_t lddres,
                       float* dgamma, float* dbeta, void* stream);

/* ------------------------------------------------------------------ attention
 * Scaled-dot-product attention, head_dim 64, no mask, replaces
 * AttnProcessor2_0 -> F.scaled_dot_product_attention [D].
 * q/k/v/o are column slices of token-major [tokens][ld] bf16 matrices; head h uses columns
 * [h*64, h*64+64). A sequence s (0 <= s < nseq) has its i-th token at row  seq_base(s) + i*tok_stride
 * with seq_base(s) = (s / inner) * outer_stride + (s % inner) * inner_stride:
 *   spatial  (per frame over H*W):  inner = 1,  outer_stride = HW, tok_stride = 1
 *   temporal (per pixel over T):    inner = HW, outer_stride = T*HW, inner_stride = 1, tok_stride = HW
 * Rows that belong to no sequence are neither read nor written. Strided sequences (inner > 1) need S <= 128.
 * lse fp32 (natural-log sum-exp of the scaled scores, saved for backward) and the backward's delta workspace are
 * [token row][heads]: the value of token row r and head h is at [r * heads + h], so both must hold
 * (largest token row + 1) * heads floats. Only the entries of token rows are written.
 * Every ld is a multiple of 8 and at least heads*64; q / k / v / dout are 16-byte aligned, o / dq / dk / dv 4-byte
 * aligned (16-byte aligned when inner > 1 and S <= 32). */
typedef struct SvdxAttn {
  const void* q; const void* k; const void* v; void* o;
  int64_t ldq, ldk, ldv, ldo;
  int32_t nseq, heads, S;
  int32_t inner;
  int64_t outer_stride, inner_stride, tok_stride;
  float scale;
  float* lse;
  /* backward only */
  const void* dout; int64_t lddo;
  void* dq; void* dk; void* dv; int64_t lddq, lddk, lddv;
  float* delta;     /* workspace [token row][heads], sized as lse */
} SvdxAttn;
int svdx_attention_fwd(const SvdxAttn* d, void* stream);
int svdx_attention_bwd(const SvdxAttn* d, void* stream);

/* Head dim 80, forward only: the self-attention of the CLIP ViT-H/14 image encoder [transformers CLIPAttention -> SDPA,
 * 16 heads x 80, no mask]. Sequence s (0 <= s < nseq) is rows [s*S, s*S + S) of the token-major q / k / v / o matrices;
 * head h uses columns [80h, 80h + 80) of each (column slices of the fused q|k|v GEMM output allowed):
 *   o = softmax(scale * q k^T) v     over all S keys (any S >= 1), fp32 softmax, bf16 in / out.
 * q/k/v: ld % 8 == 0, 16-byte aligned; o: even ld, 4-byte aligned. Rows of o outside [0, nseq*S) are never written. */
int svdx_attention_hd80_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                            int64_t ldo, int32_t nseq, int32_t heads, int32_t S, float scale, void* stream);

/* ------------------------------------------------------------------ CLIP image preprocessing
 * The conditioning frame -> the A operand of the patch-embedding GEMM in one pass (train_svd.py:857-876 encode_image:
 * _resize_with_antialiasing(x, (224, 224)) -> (x + 1) / 2 -> CLIPImageProcessor normalisation -> Conv2d(3, C, 14, stride 14)).
 * x: contiguous NCHW [B][3][H][W] (x_strides = its 4 element strides, checked as torch defines contiguity: the stride of a
 * size-1 dimension is ignored, so a batch-1 frame slice of a video is accepted), dtype code x_dtype (0 fp32, 1 bf16, 2 fp16).
 * Per output pixel (oy, ox) of the out_size^2 image and channel c:
 *   blurred(y, x) = sum_a gy[a] sum_b gx[b] x[c][refl(y + a - (ky-1)/2)][refl(x + b - (kx-1)/2)]    (reflect padding)
 *   v = bicubic(blurred; A = -0.75, align_corners, border-clamped taps) at (oy * (H-1)/(out_size-1), ox * (W-1)/(out_size-1))
 *   out = v * affine[c] + affine[3 + c]
 * gy / gx: HOST arrays of ky / kx fp32 weights (odd sizes <= SVDX_CLIP_MAX_TAPS, (k-1)/2 < the dimension, as torch's reflect pad);
 * affine: HOST float[6] {a_0, a_1, a_2, b_0, b_1, b_2}. All three are copied into the launch (graph-capturable).
 * out: bf16 [B * (1 + P^2)][ldo], P = out_size / patch: row 0 of each image is all zero (the class-token slot), row 1 + py*P + px
 * holds patch (py, px) with column c*patch^2 + ky*patch + kx (the conv weight's (c, kh, kw) order); columns [3*patch^2, Kp) are
 * zero, Kp = 3*patch^2 rounded up to 64 (ldo >= Kp). ky = kx = 1 with H = W = out_size reproduces x exactly (rounded to bf16). */
#define SVDX_CLIP_MAX_TAPS 63
int svdx_clip_preprocess(const void* x, int32_t x_dtype, const int64_t* x_strides, int32_t B, int32_t H, int32_t W,
                         const float* gy, int32_t ky, const float* gx, int32_t kx, const float* affine,
                         int32_t out_size, int32_t patch, void* out, int64_t ldo, void* stream);

/* ------------------------------------------------------------------ elementwise / layout */
/* weights -> bf16, optionally re-laid-out. src_bf16 is the SOURCE DTYPE CODE used by every entry of this section:
 * 0 = fp32, 1 = bf16, 2 = fp16 (train_svd_lora.py:669 moves the frozen UNet to fp16 / bf16 `weight_dtype`).
 *   mode 0: plain copy           dst[n][k]           = src[n][k]
 *   mode 1: transpose            dst[k][n]           = src[n][k]            (dgrad operand of a linear)
 *   mode 2: conv OIHW -> O(HW)I  dst[o][t][i(pad)]   = src[o][i][t]         (fwd operand; taps = kh*kw or kt)
 *   mode 3: conv OIHW -> I(HW)O  dst[i][t][o]        = src[o][i][t]         (dgrad operand; the caller negates tap offsets)
 * i_pad >= I pads the input-channel axis with zeros (conv_in: 8 -> 64). */
int svdx_prep_weight(const void* src, int32_t src_bf16, void* dst, int32_t mode,
                     int32_t O, int32_t I, int32_t taps, int32_t i_pad, void* stream);
/* adjoint of svdx_prep_weight mode 2: dst[o][i][t] += src[o][t][i] (fp32; src row = taps*i_pad, dst = OIHW gradient) */
int svdx_unprep_conv_grad(const float* src, float* dst, int32_t O, int32_t I, int32_t taps, int32_t i_pad, void* stream);
/* sum over all elements of dy * (a - b) (bf16 inputs) accumulated into out[0] (fp32): AlphaBlender mix_factor gradient */
int svdx_dot_diff(const void* dy, const void* a, const void* b, int64_t n, float* out, void* stream);
/* y = dy * silu'(x) on fp32 vectors (time-embedding MLP backward) */
int svdx_silu_bwd_f32(const float* x, const float* dy, float* dx, int64_t n, void* stream);
int svdx_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream);
int svdx_cast_bf16_f32(const void* src, float* dst, int64_t n, void* stream);
int svdx_cast_f16_f32(const void* src, float* dst, int64_t n, void* stream);
/* NCHW (dtype code 0/1/2) -> [N][H][W][c_pad] bf16 (zero padded channels) and back (to an NCHW tensor of dtype code dst_bf16) */
int svdx_nchw_to_nhwc(const void* src, int32_t src_bf16, void* dst, int32_t N, int32_t C, int32_t H, int32_t W,
                      int32_t c_pad, void* stream);
int svdx_nhwc_to_nchw(const void* src, int64_t lds, void* dst, int32_t dst_bf16, int32_t N, int32_t C, int32_t H,
                      int32_t W, void* stream);
/* The temporal VAE decoder's tail [D: TemporalDecoder.time_conv_out]: a Conv3d(C, C, (3,1,1), padding (1,0,0)) over the frames
 * of each clip (zero frames past the clip edges), fused with the token-major -> NCHW conversion and the output cast:
 *   y[n][o][p] = bias[o] + sum_{i, k} w[(o*C + i)*3 + k] * x[(n + k - 1) * H*W + p][i]      (clip b = n / T, n + k - 1 in clip b)
 * x: fp32 [N*H*W][ldx] (the conv_out output, ldx % 4 == 0, 16-byte aligned, ldx >= C rounded up to 4), C <= 8, N = B*T;
 * w fp32 [C][C][3], bias fp32 [C] or NULL; y NCHW [N][C][H][W] of dtype code y_dtype (0 fp32, 1 bf16, 2 fp16). One pass. */
int svdx_time_conv_out(const float* x, int64_t ldx, int32_t N, int32_t T, int32_t C, int32_t H, int32_t W, const float* w,
                       const float* bias, void* y, int32_t y_dtype, void* stream);
/* nearest 2x upsample, channels-last (F.interpolate of Upsample2D [D]) and its adjoint (2x2 sum) */
int svdx_upsample2x(const void* src, void* dst, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
int svdx_upsample2x_bwd(const void* dsrc, void* ddst, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
/* parity planes for the stride-2 conv: dst[(p*2+q)*N + n][H/2][W/2][C] = src[n][2h+p][2w+q][C], and adjoint */
int svdx_space_to_planes(const void* src, void* dst, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
int svdx_planes_to_space(const void* src, void* dst, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
/* channel concat / split of channels-last tensors (torch.cat(dim=1) of the up blocks) */
int svdx_concat_channels(const void* a, int32_t Ca, const void* b, int32_t Cb, void* dst, int64_t rows, void* stream);
int svdx_split_channels(const void* src, void* a, int32_t Ca, void* b, int32_t Cb, int64_t rows, int32_t accumulate_a,
                        void* stream);
/* y = a + b (bf16), y = silu(x) for fp32 vectors, column sums (bias gradients) */
int svdx_add_bf16(const void* a, const void* b, void* y, int64_t n, void* stream);
int svdx_axpby_bf16(const void* a, const void* b, const float* scales, void* y, int64_t n, void* stream);
int svdx_silu_f32(const float* x, float* y, int64_t n, void* stream);
int svdx_colsum(const void* x, int64_t ldx, int64_t rows, int32_t cols, float* out, int32_t accumulate, void* stream);
/* GEGLU backward: dpre[m][:h] = dout*gelu(gate); dpre[m][h:] = dout*value*gelu'(gate). bias_grad (optional, fp32 [2h], accumulated):
 * += column sums of the dpre values written — the bias gradient of the GEGLU projection, fused into the same pass */
int svdx_geglu_bwd(const void* pre, int64_t ldpre, const void* dout, int64_t lddo, void* dpre, int64_t lddpre,
                   int64_t rows, int32_t h, float* bias_grad, void* stream);
/* y[r][:] = softmax(scale * x[r][:]) over bf16 rows (fp32 arithmetic, in place allowed). Used by the VAE encoder's mid-block
 * attention (1 head of dim 512, [D] AutoencoderKLTemporalDecoder.encoder.mid_block.attentions.0): scores = Q K^T and P V go through
 * svdx_tapgemm, the row softmax through this kernel. */
int svdx_softmax_rows(const void* x, int64_t ldx, int64_t rows, int32_t cols, float scale, void* y, int64_t ldy, void* stream);
/* Skinny products of the per-clip conditioning vectors ([B, C] rows: TimestepEmbedding MLPs, every resnet's time_emb_proj, the
 * 1-key image cross-attention to_out(to_v(e)) [D], their LoRA side paths and their data gradients):
 *   out[m][n] = scale * sum_k a[m][k] * w[n][k] + bias[n]  (+ out[m][n] when accumulate != 0),
 * M <= 8 rows, bf16 operands, fp32 accumulation, bf16 (SVDX_OUT_BF16) or fp32 (SVDX_OUT_F32) output. A weight-streaming GEMV
 * (one warp per output column): the 128-row tensor-core tiles of svdx_tapgemm would be > 99 % padding here. */
int svdx_gemv(const void* a, int64_t lda, const void* w, int64_t ldw, int32_t M, int32_t N, int32_t K, const float* bias,
              void* out, int64_t ldo, int32_t out_dtype, float scale, int32_t accumulate, void* stream);
/* ...and their weight gradients: g[o][k] += scale[0] * sum_{t < T} dy[t][o] * x[t][k], T <= 8 (scale NULL = 1) */
int svdx_outer_accum(const void* dy, int64_t lddy, const void* x, int64_t ldx, int32_t T, int32_t O, int32_t K,
                     const float* scale, float* g, int64_t ldg, void* stream);
/* AlphaBlender epilogue scale triples from mix_factor, a = sigmoid(mix_factor); writes float[16]:
 *   out[0..3]   = {1-a, a, 1-a, 0}      transformer blend  out = a*x_spatial + (1-a)*(acc + residual)
 *   out[4..7]   = {1-a, 1, 0, a*(1-a)}  resnet blend       out = x_spatial + (1-a)*acc
 *   out[8..11]  = {1-a, 0, 0, 0}        accumulator-only triple (gradient GEMMs of a blended forward)
 *   out[12..15] = {a, 0, 1-a, 0}        {s, 0} pairs for svdx_axpby_bf16 (gradients of the residual operands) */
int svdx_blend_scales(const float* mix_factor, float* out16, void* stream);
/* fused multi-tensor AdamW on a flat fp32 buffer (torch.optim.AdamW of train_svd.py:767-773); when shadow_bf16 is given
 * the updated parameters are also written as bf16 at the same flat offsets (the forward GEMM operands). Every
 * step-varying scalar is in DEVICE memory, so that the update can be captured in a CUDA graph and replayed:
 * state = float[8] {lr, beta1, beta2, eps, weight_decay, step, 1-beta1^step, 1-beta2^step}. The call first advances
 * step and the bias corrections on the device (a 1-thread kernel), then updates; the host changes the learning rate by
 * writing state[0] (lr scheduler of train_svd.py:790-796). Two launches. Optional arguments, NULL for none:
 *   ema, ema_state: the update also advances the fp32 EMA buffer ema[0 .. n) (16-byte aligned) at the same flat offsets from
 *     the freshly updated masters, and the tick also advances ema_state (the EMA state below, 8-byte aligned). Pass both or
 *     neither: one without the other is SVDX_E_BADARG.
 *   grad_mul: a DEVICE float (4-byte aligned) the gradient is also scaled by, read by the update kernel, so the applied gradient
 *     is g * (grad_scale * grad_mul[0]); at grad_scale = 1 that is g * grad_mul[0], the product torch's in-place g.mul_(coef)
 *     gives. Gradient clipping passes out + 1 of svdx_clip_coef, so the clip is decided on the device and a captured step
 *     needs no host sync.
 * With all three NULL the update is plain AdamW. */
int svdx_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, float* state, float grad_scale, void* shadow_bf16,
                    float* ema, double* ema_state, const float* grad_mul, void* stream);
/* Data-parallel optimizer step over NVLink peer memory (one process per GPU, every rank's gradient and bf16 operand arenas
 * mapped into every process with CUDA IPC): reduce-scatter + AdamW + all-gather as ONE kernel. This rank owns [lo, lo + n):
 * it loads that slice of grads[r] (r = 0 .. world-1, the FULL arenas, peer-mapped), sums in rank order, applies AdamW with
 * grad_scale (= 1 / world) to its local p / m / v slices (length n) and stores the bf16 value to shadows[r][lo + i] of every
 * rank. The caller provides the cross-rank ordering: all gradients final before the launch, no rank reads its shadow or
 * clears its gradients until every rank's launch has completed. tick != 0 also advances the device step count / bias
 * corrections in state[5..7] (svdx_adamw_step's state layout), and ema_state with an EMA. grads[r]: 16-byte aligned,
 * shadows[r]: 8-byte aligned. ema (this rank's slice: length n, 16-byte aligned, no peer traffic), ema_state and grad_mul as in
 * svdx_adamw_step. Two launches with tick, one without. Replaces DistributedDataParallel's all-reduce + torch.optim.AdamW of
 * train_svd.py:767-773,815-824,1044-1049 at N > 1. */
int svdx_adamw_step_p2p(float* p, float* m, float* v, const void* const* grads, void* const* shadows, int32_t world, int64_t lo,
                        int64_t n, float* state, float grad_scale, int32_t tick, float* ema, double* ema_state,
                        const float* grad_mul, void* stream);

/* Global gradient norm for clipping (torch.nn.utils.clip_grad_norm_ with norm type 2: train_svd.py's --max_grad_norm,
 * :468-470, :1044-1049), computed and applied on the device so that a captured step clips without a host sync.
 * sumsq: DEVICE double[1 + 1024]; sumsq[0] receives the result, sumsq[1 ..] is the per-block scratch of the first stage.
 * svdx_grad_sumsq: sumsq[0] = sum over i < n of (double)g[i]^2 (g 16-byte aligned: the gradient arena or a slice of it). The
 * partition over blocks depends on n only, the partials are fp64 and a second one-block kernel sums them in index order:
 * identical bits for the same input, launch after launch and replay after replay. Two launches, no host access.
 * svdx_grad_sumsq_p2p: the same over the slice [lo, lo + n) of the rank-order sum of grads[0 .. world) (svdx_adamw_step_p2p's
 * peer-mapped arenas, summed exactly as that kernel sums them, up to four ranks' loads in flight), so the norm is that of the
 * gradient svdx_adamw_step_p2p applies. lo and n multiples of 4. Two launches.
 * svdx_clip_coef: one thread. From sumsq[0], a DEVICE max_norm and the host scale (1 / world under the sharded optimizers, so
 * the norm is that of the mean gradient), writes the DEVICE pair out = {total_norm, coef}:
 *   total_norm = fl(fl(sqrt(sumsq[0])) * scale),  coef = min(max_norm / (total_norm + 1e-6f), 1)
 * in fp32 with torch's roundings (the division is reciprocal, then multiply). The clamp propagates NaN as torch.clamp does; an
 * infinite norm gives coef = 0. Pass out + 1 as grad_mul of the update. */
int svdx_grad_sumsq(const float* g, int64_t n, double* sumsq, void* stream);
int svdx_grad_sumsq_p2p(const void* const* grads, int32_t world, int64_t lo, int64_t n, double* sumsq, void* stream);
int svdx_clip_coef(const double* sumsq, const float* max_norm, float scale, float* out, void* stream);

/* Exponential moving average of the weights (train_svd.py:676-679 EMAModel, :1053-1054 ema_unet.step(unet.parameters())
 * -> [D] diffusers.training_utils.EMAModel.step: get_decay on the host, then per parameter tensor
 * s.sub_((1 - d) * (s - p)) if p.requires_grad else s.copy_(p)).
 * ema_state = double[9] in DEVICE memory: {optimization_step, decay, min_decay, update_after_step, use_ema_warmup (0/1),
 * inv_gamma, power, cur_decay_value, 1 - cur_decay_value}. Every entry point that takes it (the AdamW updates given an
 * ema_state, and svdx_ema_multi) first advances the step and evaluates EMAModel.get_decay in fp64 on the device (a 1-thread
 * kernel, capturable in a CUDA graph), then applies e = e - (float)(1 - d) * (e - p) with three separately rounded fp32
 * operations: bit-identical to the torch ops.
 *
 * svdx_ema_multi: the EMA update over many tensors in one launch (EMAModel.step over parameters outside a fused optimizer).
 * jobs: device array of {float* shadow; const float* param; int64 n}; block_prefix[j] = first 4096-element block of job j,
 * total_blocks = sum of ceil(n_j / 4096). Two launches (tick + update). */
int svdx_ema_multi(const void* jobs, const int32_t* block_prefix, int32_t njobs, int32_t total_blocks, double* ema_state,
                   void* stream);

/* Block-wise 8-bit AdamW (train_svd.py --use_8bit_adam: bitsandbytes.optim.AdamW8bit with its defaults; the update is stated
 * in oracle/svd_adam8bit_oracle.py). One launch over many fp32 parameters, each a job of the DEVICE array
 *   {float* p; const float* g; void* s1; void* s2; float* absmax1; float* absmax2; bf16* shadow; float* ema; int64 n; int64 quant}
 * quant != 0: s1 / s2 are uint8 codes [n] into qmap1 (signed dynamic map, for m) / qmap2 (unsigned dynamic map, for v), with
 * one fp32 absmax per 256-element block and moment (absmax[ceil(n / 256)]); blocks start at the parameter's first element.
 * quant == 0: s1 / s2 are fp32 m / v [n] (parameters below min_8bit_size). shadow (optional): bf16 copy of the new p.
 * block_prefix[j] = first 256-element block of job j, total_blocks = sum of ceil(n_j / 256). qmap1 / qmap2: DEVICE float[256],
 * sorted, shared by every job of the launch. state = svdx_adamw_step's float[8] (device, advanced by a 1-thread tick first), so
 * the pair can be captured in a CUDA graph and replayed. Every operation is rounded separately (no FMA); no atomics. Aligned
 * jobs (p, g, fp32 states, shadow, EMA 16-byte; codes 8-byte) take 16-byte loads, others a scalar path. ema_state (optional,
 * 8-byte aligned): the update also advances every job's fp32 EMA buffer job.ema from the new p, by svdx_adamw_step's rule, and
 * the tick advances ema_state; NULL: no EMA, job.ema is ignored. grad_mul (optional) as in svdx_adamw_step. Two launches. */
int svdx_adamw8bit_step(const void* jobs, const int32_t* block_prefix, int32_t njobs, int32_t total_blocks, const float* qmap1,
                        const float* qmap2, float* state, float grad_scale, double* ema_state, const float* grad_mul, void* stream);

/* Sharded block-wise 8-bit AdamW over NVLink peer memory (P2PShardedAdamW8bit): reduce-scatter + svdx_adamw8bit_step +
 * all-gather as ONE kernel, replacing DistributedDataParallel's all-reduce + bitsandbytes.optim.AdamW8bit of
 * train_svd.py:746-773,815-824,1044-1049 at N > 1. jobs: DEVICE array of this rank's sub-jobs
 *   {float* p; void* s1; void* s2; float* absmax1; float* absmax2; float* ema; int64 off; int64 n; int64 quant}
 * each a whole number of 256-element blocks of one parameter (a parameter that straddles a shard boundary is split by block
 * range; s1 / s2 / absmax1 / absmax2 / ema point at the sub-job's first block), p / state / EMA this rank's local buffers, and
 * off the arena offset of p[0]. Per element the gradient is sum over r = 0 .. world-1, in rank order from 0, of grads[r][off + i]
 * (the FULL gradient arenas, peer-mapped, as svdx_adamw_step_p2p sums), times grad_scale (= 1 / world) and grad_mul[0] when
 * grad_mul is not NULL; the update is svdx_adamw8bit_step's, bit for bit (same roundings, block absmax and maps; no FMA, no
 * atomics); the new bf16 value is stored to shadows[r][off + i] of every rank. tick != 0 first advances state (and ema_state
 * when given) as svdx_adamw_step_p2p does. ema_state NULL: no EMA; otherwise every job's ema is advanced as in
 * svdx_adamw8bit_step. The caller orders the ranks around the launch as for svdx_adamw_step_p2p. grads[r] / shadows[r]: 16-byte
 * aligned; world 1 .. 16. Two launches with tick, one without. */
int svdx_adamw8bit_p2p(const void* jobs, const int32_t* block_prefix, int32_t njobs, int32_t total_blocks, const float* qmap1,
                       const float* qmap2, const void* const* grads, void* const* shadows, int32_t world, float* state,
                       float grad_scale, int32_t tick, double* ema_state, const float* grad_mul, void* stream);

/* Batch assembly of a training step from video frames (train_svd.py:942-1017; svd_xtend_b200.video_train). Every operation is
 * rounded separately (no FMA), in the reference's order.
 * svdx_vae_frames_in: the VAE encoder's input rows, bf16 [(B*F + B) * H*W][c_pad] (token-major, channels >= 3 zero), as
 * svdx_nchw_to_nhwc writes them: rows of frame n < B*F are the clip frames x[b][f] (n = b*F + f); rows of frame B*F + b are the
 * noise-augmented conditioning frame fl(fl(eps[b] * sigma_c[b]) + x[b][0]) (:957-958). x: [B][F][3][H][W] of dtype code
 * x_dtype (0 fp32, 1 bf16); eps: fp32 [B][3][H][W]; sigma_c: DEVICE fp32 [B]. One launch. */
int svdx_vae_frames_in(const void* x, int32_t x_dtype, const float* cond_eps, const float* cond_sigma, int32_t B, int32_t F,
                       int32_t H, int32_t W, int32_t c_pad, void* dst, void* stream);
/* svdx_vae_frames_in_range: the rows of svdx_vae_frames_in for the frames [first, first + count) of its B*(F+1) frame index space
 * only, into dst [count * H*W][c_pad] (for an encode in frame chunks). Same values, one launch. */
int svdx_vae_frames_in_range(const void* x, int32_t x_dtype, const float* cond_eps, const float* cond_sigma, int32_t B, int32_t F,
                             int32_t H, int32_t W, int32_t first, int32_t count, int32_t c_pad, void* dst, void* stream);
/* Decoded uint8 frames (csrc/frames.cu). Resize = what Pillow's Image.resize((W, H)) returns for an RGB image with its default
 * BICUBIC filter: 8-bpc two-pass resample, horizontal first into a uint8 intermediate, then vertical, 22-bit fixed-point taps.
 * svdx_resize_taps_ksize: taps per output pixel along an axis of in_size -> out_size (or < 0 on bad sizes).
 * svdx_resize_taps (HOST): the taps of that axis, int32 [out_size][2 + ksize]: first source index, tap count, ksize weights.
 * svdx_frames_u8_in: from uint8 frames src [B][F][H0][W0][3] (HWC, RGB) and DEVICE copies of the taps of H0 -> H (taps_y) and
 * W0 -> W (taps_x), the rows of svdx_vae_frames_in for the frames [first, first + count) into dst [count * H*W][c_pad] (c_pad a
 * multiple of 8, dst 16-byte aligned), where x = fl(fl(resize(src) / 127.5f) - 1) (train_svd.py's DummyDataset); for each
 * conditioning frame B*F + b in the range, also the clean first frame x[b][0] into first_frames fp32 [B][3][H][W] (may be NULL).
 * One launch.
 * svdx_resize_taps_box_ksize / svdx_resize_taps_box (HOST): the same for Image.resize(size, box=...) along one axis: the source
 * interval [in0, in1) (Pillow's float box bounds) -> out_size. SVDX_E_BADARG unless 0 <= in0 <= in1 <= in_size (Pillow's box
 * rules; a box of zero extent is valid) and both are finite. svdx_resize_taps is the box [0, in_size), bit for bit. Pillow copies
 * an axis with out_size == in_size and the box [0, in_size); those taps are the identity, so the resize stays bit exact.
 * svdx_frames_u8_in_clips: svdx_frames_u8_in for clips of different source sizes and boxes. Clip b (frames F*b .. F*b + F-1 and
 * conditioning frame B*F + b) is described by the DEVICE descriptor descs[b]: its frame f is the uint8 [H0][W0][3] image at byte
 * start + f*H0*W0*3 of src, and its output row y / column x uses tap row ty_off + y of taps_y / tx_off + x of taps_x. The tap
 * tables are int32 [ty_rows][2 + ksize_y] and [tx_rows][2 + ksize_x]: one fixed row stride, the largest ksize of any clip, each
 * row as svdx_resize_taps(_box) writes it, zero padded. A descriptor whose frames do not fit in src_bytes, or whose tap rows do
 * not fit in the tables, reads nothing (those frames come out as u = 0), and tap rows are clamped to the clip's source size.
 * Same rows, rounding and frame range as svdx_frames_u8_in; svdx_frames_u8_in is the case where every clip shares one descriptor
 * and runs the same kernel. One launch. */
typedef struct svdx_clip_desc {
  int64_t start;               /* byte offset of the clip's frame 0 in src */
  int32_t H0, W0;              /* its source size */
  int32_t ty_off, tx_off;      /* its first tap rows in taps_y / taps_x */
} svdx_clip_desc;
int svdx_resize_taps_ksize(int32_t in_size, int32_t out_size);
int svdx_resize_taps(int32_t in_size, int32_t out_size, int32_t* taps);
int svdx_resize_taps_box_ksize(int32_t in_size, int32_t out_size, float in0, float in1);
int svdx_resize_taps_box(int32_t in_size, int32_t out_size, float in0, float in1, int32_t* taps);
int svdx_frames_u8_in(const uint8_t* src, int32_t H0, int32_t W0, const int32_t* taps_y, int32_t ksize_y, const int32_t* taps_x,
                      int32_t ksize_x, const float* cond_eps, const float* cond_sigma, int32_t B, int32_t F, int32_t H, int32_t W,
                      int32_t first, int32_t count, int32_t c_pad, void* dst, float* first_frames, void* stream);
int svdx_frames_u8_in_clips(const uint8_t* src, int64_t src_bytes, const svdx_clip_desc* descs, const int32_t* taps_y,
                            int32_t ty_rows, int32_t ksize_y, const int32_t* taps_x, int32_t tx_rows, int32_t ksize_x,
                            const float* cond_eps, const float* cond_sigma, int32_t B, int32_t F, int32_t H, int32_t W, int32_t first,
                            int32_t count, int32_t c_pad, void* dst, float* first_frames, void* stream);
/* svdx_edm_prepare: from the fp32 moments [B*(F+1)][2C][h][w] of that encode (mean, then logvar), per latent element
 *   z = mean + exp(0.5 * clamp(logvar, -30, 20)) * eps,  latent = z * sf,  noisy = latent + noise * sigma[b]
 * (:948, :287, :951, :967) and the conditioning latents c = (z_c * sf) * (1 / sf) of frame B*F + b (:959-960: torch's division of
 * a CUDA tensor by a scalar multiplies by the fp32 reciprocal), writes (all fp32)
 *   sample  [B][F][2C][h][w]: channels < C noisy / sqrt(sigma^2 + 1) (:972), channels >= C image_mask[b] * c (:1008-1017);
 *   noisy   [B][F][C][h][w];  latents [B][F][C][h][w] (the target).
 * latent_eps, noise: fp32 [B*F][C][h][w]; cond_latent_eps: fp32 [B][C][h][w]; sigma, image_mask: DEVICE fp32 [B]. One launch. */
int svdx_edm_prepare(const float* moments, const float* latent_eps, const float* noise, const float* cond_latent_eps,
                     const float* sigma, const float* image_mask, float scaling_factor, int32_t B, int32_t F, int32_t C,
                     int32_t h, int32_t w, float* sample, float* noisy, float* latents, void* stream);

/* many bf16 transposes dst[i][o] = src_base[src_off + o*I + i] in one launch (dgrad operands of all trainable linears).
 * jobs: device array of {int64 src_off; void* dst; int32 O; int32 I}; tile_prefix[j] = first 32x32 tile of job j. */
int svdx_multi_transpose(const void* src_base, const void* jobs, const int32_t* tile_prefix, int32_t njobs, int32_t total_tiles,
                         void* stream);

/* LoRA fuse / unfuse (UNet fuse_lora / unfuse_lora): many base weights W [N, K] updated in place in one launch,
 *   W[n,k] = round(fl(W[n,k] + tot)),  tot = sum over the job's terms, in order, of fl(scale * acc),
 *   acc = sum over j < r, in order, of fl(B[n,j] * A[j,k])   (every product and sum rounded separately, no FMA; the
 *   final rounding to bf16 / fp16 is to nearest even). oracle/svd_lora_oracle.py states the same in torch ops.
 * jobs: device array of {void* w; int64 n; int64 k; int32 dtype; int32 term0; int32 nterms; int32 pad} (40 bytes);
 * terms: device array of {const void* a [r, K]; const void* b [N, r]; int32 r (>= 1); int32 dtype; float scale; int32 pad}
 * (32 bytes); job j uses terms[term0 .. term0 + nterms). dtype codes as above (0 fp32, 1 bf16, 2 fp16), a and b of one term
 * share one. tile_prefix[j] = first 64x64 tile of job j, total_tiles = sum of ceil(n/64) * ceil(k/64). An unfuse is a
 * fuse with negated scales: it restores W to within one unit in the last place of its dtype. */
int svdx_lora_merge(const void* jobs, const void* terms, const int32_t* tile_prefix, int32_t njobs, int32_t total_tiles,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVD_XTEND_B200_H_ */
