// The CLIP image encoder's own kernels (CLIPVisionModelWithProjection, ViT-H/14 [transformers]; the frozen image encoder of
// the SVD pipeline): everything else in the encoder runs on svdx_tapgemm, svdx_layernorm_fwd and svdx_gemv.
//
// svdx_clip_preprocess: the conditioning frame -> the A operand of the patch-embedding GEMM in one pass over the image.
//   Each output element is one (image, patch, c, ky, kx) pixel of the 224x224 model input: it evaluates the bicubic resize
//   (align_corners, A = -0.75, border-clamped taps) of the Gaussian-blurred image, blurring each of the 16 bicubic taps on the fly
//   from the two 1-D kernels (reflect padding, x then y as the reference filters), then applies the per-channel normalisation
//   affine and stores bf16. Nothing of the blurred or resized image is materialised.
//
// svdx_attention_hd80_fwd: dense unmasked SDPA with head dim 80 (ViT-H: 1280 = 16 x 80), forward only. attention.cu is built
//   around 64-column heads (128-byte swizzled rows, 64-column maps and epilogue); attention here is ~3 % of the encoder's FLOPs
//   (21 MFLOP per image, head and layer at S = 257), so it gets the warp-level shape of attention_small.cu instead: one CTA per
//   (sequence, head, 64-query block), four warps of 16 query rows, mma.sync m16n8k16, K / V blocks of 64 keys staged with
//   cp.async into padded shared-memory rows, online softmax in registers (ex2), keys >= S masked, query rows >= S not stored.
#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"

namespace svdx {

// ------------------------------------------------------------------------------------------------ preprocess
struct ClipPrepP {
  const void* x;
  int B, H, W;
  int ky, kx;                                 // odd Gaussian kernel sizes, reflect padding (k - 1) / 2
  float gy[SVDX_CLIP_MAX_TAPS], gx[SVDX_CLIP_MAX_TAPS];
  float a[3], b[3];                           // y = v * a[c] + b[c]
  double sy, sx;                              // align_corners source scale (in - 1) / (out - 1): source coordinates in fp64,
                                              // an fp32 coordinate misplaces a tap by ~1e-5 pixel at 1024 columns
  int OS, PS, P, K, Kp;                       // output size, patch size, patches per side, 3 * PS^2, padded K
  bf16* out;
  long long ldo;
  long long total;
};

template <typename T>
SVDX_DEVINL float ld_px(const T* p) { return static_cast<float>(*p); }
template <>
SVDX_DEVINL float ld_px<bf16>(const bf16* p) { return __bfloat162float(*p); }
template <>
SVDX_DEVINL float ld_px<__half>(const __half* p) { return __half2float(*p); }

SVDX_DEVINL int reflect_idx(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// torch's upsample_bicubic2d coefficients (cubic convolution, A = -0.75) of the taps at offsets -1, 0, 1, 2
SVDX_DEVINL void cubic_coeffs(float t, float (&c)[4]) {
  constexpr float A = -0.75f;
  auto cc1 = [](float x) { return ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f; };
  auto cc2 = [](float x) { return ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A; };
  c[0] = cc2(t + 1.0f);
  c[1] = cc1(t);
  c[2] = cc1(1.0f - t);
  c[3] = cc2(2.0f - t);
}

template <typename T>
__global__ void __launch_bounds__(256) clip_preprocess_kernel(const __grid_constant__ ClipPrepP p) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.total) return;
  const int col = (int)(idx % p.Kp);
  const long long row = idx / p.Kp;
  const int per_img = 1 + p.P * p.P;
  const int img = (int)(row / per_img);
  const int r = (int)(row - (long long)img * per_img);
  float v = 0.f;
  if (r > 0 && col < p.K) {                   // row 0 of every image is the class-token slot; columns >= K are padding
    const int pp = p.PS * p.PS;
    const int c = col / pp, rem = col - c * pp;
    const int dy = rem / p.PS, dx = rem - dy * p.PS;
    const int py = (r - 1) / p.P, px = (r - 1) - py * p.P;
    const int oy = py * p.PS + dy, ox = px * p.PS + dx;
    const double ry = p.sy * oy, rx = p.sx * ox;
    const int iy = (int)floor(ry), ix = (int)floor(rx);
    float cy[4], cx[4];
    cubic_coeffs((float)(ry - iy), cy);
    cubic_coeffs((float)(rx - ix), cx);
    const T* plane = reinterpret_cast<const T*>(p.x) + ((long long)img * 3 + c) * p.H * p.W;
    const int hy = (p.ky - 1) / 2, hx = (p.kx - 1) / 2;
    float rows[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int yy = min(max(iy - 1 + i, 0), p.H - 1);
      float tap[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int xx = min(max(ix - 1 + j, 0), p.W - 1);
        float blur = 0.f;                     // separable Gaussian at (yy, xx): rows blurred along x, then combined along y
        for (int a = 0; a < p.ky; ++a) {
          const T* src = plane + (long long)reflect_idx(yy + a - hy, p.H) * p.W;
          float s = 0.f;
          for (int b = 0; b < p.kx; ++b) s = fmaf(p.gx[b], ld_px(src + reflect_idx(xx + b - hx, p.W)), s);
          blur = fmaf(p.gy[a], s, blur);
        }
        tap[j] = blur;
      }
      rows[i] = tap[0] * cx[0] + tap[1] * cx[1] + tap[2] * cx[2] + tap[3] * cx[3];
    }
    const float val = rows[0] * cy[0] + rows[1] * cy[1] + rows[2] * cy[2] + rows[3] * cy[3];
    v = fmaf(val, p.a[c], p.b[c]);
  }
  p.out[row * p.ldo + col] = __float2bfloat16(v);
}

// ------------------------------------------------------------------------------------------------ attention, head dim 80
constexpr int A80_D = 80;
constexpr int A80_ROW = 88;        // bf16 per staged row: 80 + 8 pad (176 B: conflict-free fragment loads / ldmatrix rows)
constexpr int A80_BLK = 64;        // queries per CTA and keys per staged block
constexpr int A80_WARPS = 4;
constexpr float A80_LOG2E = 1.4426950408889634f;

struct Attn80P {
  const bf16 *q, *k, *v;
  bf16* o;
  long long ldq, ldk, ldv, ldo;
  int S;
  float qs;                        // scale * log2(e)
};

SVDX_DEVINL void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
SVDX_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
SVDX_DEVINL void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

SVDX_DEVINL uint32_t a80_lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
SVDX_DEVINL void a80_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// rows [r0, r0 + 64) of one head slice ([S][80] at `base`, row stride ld) -> a [64][A80_ROW] tile; rows >= S are zero-filled
SVDX_DEVINL void a80_stage(const bf16* base, long long ld, int r0, int S, uint32_t tile) {
  for (int i = threadIdx.x; i < A80_BLK * (A80_D / 8); i += A80_WARPS * 32) {
    const int r = i / (A80_D / 8), c = i - r * (A80_D / 8);
    const bool ok = r0 + r < S;
    cp_async16(tile + (uint32_t)(r * A80_ROW + c * 8) * 2u, base + (long long)(ok ? r0 + r : 0) * ld + c * 8, ok);
  }
}

__global__ void __launch_bounds__(A80_WARPS * 32) attn_hd80_fwd_kernel(const Attn80P p) {
  __shared__ __align__(16) bf16 sm[3 * A80_BLK * A80_ROW];
  const uint32_t tQ = smem_u32(sm), tK = tQ + A80_BLK * A80_ROW * 2, tV = tK + A80_BLK * A80_ROW * 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;
  const int q0 = blockIdx.x * A80_BLK, h = blockIdx.y;
  const long long tok0 = (long long)blockIdx.z * p.S;
  const bf16* qb = p.q + tok0 * p.ldq + h * A80_D;
  const bf16* kb_ = p.k + tok0 * p.ldk + h * A80_D;
  const bf16* vb = p.v + tok0 * p.ldv + h * A80_D;
  const int S = p.S;
  const int nkb = (S + A80_BLK - 1) / A80_BLK;

  a80_stage(qb + (long long)q0 * p.ldq, p.ldq, 0, S - q0, tQ);
  a80_stage(kb_, p.ldk, 0, S, tK);
  cp_async_commit();
  a80_stage(vb, p.ldv, 0, S, tV);
  cp_async_commit();

  uint32_t qa[5][4];
  float o[10][4];
#pragma unroll
  for (int dn = 0; dn < 10; ++dn)
#pragma unroll
    for (int i = 0; i < 4; ++i) o[dn][i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // log2-domain row maxima, this thread's partial row sums

  for (int kb = 0; kb < nkb; ++kb) {
    cp_async_wait<1>();                      // Q and this block's K have landed
    __syncthreads();
    if (kb == 0) {
#pragma unroll
      for (int ks = 0; ks < 5; ++ks) {
        const uint32_t base = tQ + (uint32_t)((warp * 16 + g) * A80_ROW + ks * 16 + 2 * tq) * 2u;
        qa[ks][0] = a80_lds32(base);
        qa[ks][1] = a80_lds32(base + 8 * A80_ROW * 2);
        qa[ks][2] = a80_lds32(base + 16);
        qa[ks][3] = a80_lds32(base + 8 * A80_ROW * 2 + 16);
      }
    }
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) s[nt][i] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 5; ++ks)
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const uint32_t bb = tK + (uint32_t)((nt * 8 + g) * A80_ROW + ks * 16 + 2 * tq) * 2u;
        a80_mma(s[nt], qa[ks], a80_lds32(bb), a80_lds32(bb + 16));
      }
    // online softmax over this block's keys (rows g and g + 8 of the warp's 16)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const bool ok = kb * A80_BLK + nt * 8 + 2 * tq + i < S;
        s[nt][i] = ok ? s[nt][i] * p.qs : -INFINITY;
        s[nt][2 + i] = ok ? s[nt][2 + i] * p.qs : -INFINITY;
        mx0 = fmaxf(mx0, s[nt][i]);
        mx1 = fmaxf(mx1, s[nt][2 + i]);
      }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);     // finite: every key block holds at least one key < S
    const float al0 = exp2_fast(m0 - n0), al1 = exp2_fast(m1 - n1);
    m0 = n0; m1 = n1;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        s[nt][i] = exp2_fast(s[nt][i] - n0);
        s[nt][2 + i] = exp2_fast(s[nt][2 + i] - n1);
        r0 += s[nt][i];
        r1 += s[nt][2 + i];
      }
    l0 = l0 * al0 + r0;
    l1 = l1 * al1 + r1;
#pragma unroll
    for (int dn = 0; dn < 10; ++dn) { o[dn][0] *= al0; o[dn][1] *= al0; o[dn][2] *= al1; o[dn][3] *= al1; }
    cp_async_wait<0>();                      // this block's V has landed
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int dn = 0; dn < 10; ++dn) {
        uint32_t b0, b1;
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
                     : "=r"(b0), "=r"(b1) : "r"(tV + (uint32_t)((kk * 16 + (lane & 15)) * A80_ROW + dn * 8) * 2u));
        a80_mma(o[dn], a, b0, b1);
      }
    }
    __syncthreads();                         // every warp is done with this block's K and V
    if (kb + 1 < nkb) {
      a80_stage(kb_, p.ldk, (kb + 1) * A80_BLK, S, tK);
      cp_async_commit();
      a80_stage(vb, p.ldv, (kb + 1) * A80_BLK, S, tV);
      cp_async_commit();
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  const int qa0 = q0 + warp * 16 + g, qa1 = qa0 + 8;
  bf16* ob = p.o + tok0 * p.ldo + h * A80_D + 2 * tq;
#pragma unroll
  for (int dn = 0; dn < 10; ++dn) {
    if (qa0 < S) *reinterpret_cast<uint32_t*>(ob + (long long)qa0 * p.ldo + dn * 8) = pack_bf16x2(o[dn][0] * i0, o[dn][1] * i0);
    if (qa1 < S) *reinterpret_cast<uint32_t*>(ob + (long long)qa1 * p.ldo + dn * 8) = pack_bf16x2(o[dn][2] * i1, o[dn][3] * i1);
  }
}

}  // namespace svdx

using namespace svdx;

extern "C" int svdx_clip_preprocess(const void* x, int32_t x_dtype, const int64_t* x_strides, int32_t B, int32_t H, int32_t W,
                                    const float* gy, int32_t ky, const float* gx, int32_t kx, const float* affine,
                                    int32_t out_size, int32_t patch, void* out, int64_t ldo, void* stream) {
  if (!x || !x_strides || !gy || !gx || !affine || !out || B <= 0 || H <= 0 || W <= 0 || x_dtype < 0 || x_dtype > 2)
    return svdx_fail(SVDX_E_BADARG, "clip_preprocess: null pointer or bad shape / dtype code");
  // contiguity as torch defines it: the stride of a size-1 dimension is never used, so it is not checked (a batch-1 frame
  // slice video[:, 0] keeps the video's batch stride and is still contiguous)
  if ((W > 1 && x_strides[3] != 1) || (H > 1 && x_strides[2] != W) || x_strides[1] != (int64_t)H * W ||
      (B > 1 && x_strides[0] != 3LL * H * W))
    return svdx_fail(SVDX_E_BADARG, "clip_preprocess: the image must be a contiguous NCHW [B, 3, H, W] tensor");
  if (ky < 1 || kx < 1 || ky > SVDX_CLIP_MAX_TAPS || kx > SVDX_CLIP_MAX_TAPS || !(ky & 1) || !(kx & 1))
    return svdx_fail(SVDX_E_BADARG, "clip_preprocess: Gaussian kernel sizes must be odd and <= SVDX_CLIP_MAX_TAPS (63)");
  if ((ky - 1) / 2 >= H || (kx - 1) / 2 >= W)
    return svdx_fail(SVDX_E_BADARG, "clip_preprocess: reflect padding must be smaller than the input dimension");
  if (out_size < 2 || patch < 1 || out_size % patch) return svdx_fail(SVDX_E_BADARG, "clip_preprocess: out_size must be a multiple of patch");
  const int K = 3 * patch * patch;
  if (ldo < ((K + 63) / 64) * 64) return svdx_fail(SVDX_E_BADARG, "clip_preprocess: ldo must hold K = 3 * patch^2 rounded up to 64");
  ClipPrepP p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.B = B; p.H = H; p.W = W; p.ky = ky; p.kx = kx;
  for (int i = 0; i < ky; ++i) p.gy[i] = gy[i];
  for (int i = 0; i < kx; ++i) p.gx[i] = gx[i];
  for (int c = 0; c < 3; ++c) { p.a[c] = affine[c]; p.b[c] = affine[3 + c]; }
  p.sy = (double)(H - 1) / (double)(out_size - 1);
  p.sx = (double)(W - 1) / (double)(out_size - 1);
  p.OS = out_size; p.PS = patch; p.P = out_size / patch; p.K = K; p.Kp = (K + 63) / 64 * 64;
  p.out = reinterpret_cast<bf16*>(out); p.ldo = ldo;
  p.total = (long long)B * (1 + p.P * p.P) * p.Kp;
  const unsigned blocks = (unsigned)((p.total + 255) / 256);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (x_dtype == 1) clip_preprocess_kernel<bf16><<<blocks, 256, 0, st>>>(p);
  else if (x_dtype == 2) clip_preprocess_kernel<__half><<<blocks, 256, 0, st>>>(p);
  else clip_preprocess_kernel<float><<<blocks, 256, 0, st>>>(p);
  SVDX_CHECK_LAUNCH("clip_preprocess");
  return SVDX_OK;
}

extern "C" int svdx_attention_hd80_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                                       int64_t ldo, int32_t nseq, int32_t heads, int32_t S, float scale, void* stream) {
  if (!q || !k || !v || !o || nseq <= 0 || heads <= 0 || S <= 0 || nseq > 65535 || heads > 65535)
    return svdx_fail(SVDX_E_BADARG, "attention_hd80_fwd: null pointer or bad geometry");
  if ((ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 2) || ldq < heads * 80 || ldk < heads * 80 || ldv < heads * 80 || ldo < heads * 80)
    return svdx_fail(SVDX_E_BADARG, "attention_hd80_fwd: q/k/v rows need ld % 8 == 0 and ld >= heads * 80, o rows ld even");
  const uintptr_t al = reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v);
  if ((al & 15) || (reinterpret_cast<uintptr_t>(o) & 3)) return svdx_fail(SVDX_E_BADARG, "attention_hd80_fwd: q/k/v 16 B and o 4 B aligned");
  Attn80P p;
  p.q = reinterpret_cast<const bf16*>(q); p.k = reinterpret_cast<const bf16*>(k); p.v = reinterpret_cast<const bf16*>(v);
  p.o = reinterpret_cast<bf16*>(o);
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.S = S;
  p.qs = scale * A80_LOG2E;
  dim3 grid((unsigned)((S + A80_BLK - 1) / A80_BLK), (unsigned)heads, (unsigned)nseq);
  attn_hd80_fwd_kernel<<<grid, A80_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  SVDX_CHECK_LAUNCH("attention_hd80_fwd");
  return SVDX_OK;
}
