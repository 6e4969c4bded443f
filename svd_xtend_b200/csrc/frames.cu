// Decoded video frames -> the VAE encoder's input rows of a training step (svd_xtend_b200.video_train, uint8 input form).
//
// svdx_resize_taps (host): the per-output-pixel taps of Pillow's 8-bpc BICUBIC resample along one axis, the filter
//   `Image.resize((W, H))` applies to an RGB image by default (Pillow's libImaging/Resample.c): a = -0.5, support 2 scaled by the
//   downscale factor (antialiasing), weights in double, normalised by their sum, then 22-bit fixed point rounded half away from
//   zero. Computed on the host, once per (source, target) size, in the same double operations as Pillow.
// svdx_frames_u8_in: uint8 HWC RGB frames [B][F][H0][W0][3] -> the horizontal pass (clamped to a uint8 intermediate), the
//   vertical pass (clamped to uint8), u / 127.5f - 1 (train_svd.py's DummyDataset) -> bf16 encoder rows over a frame range, in
//   svdx_vae_frames_in's layout and rounding, plus the clean first frame of each clip in fp32 for the CLIP encoder.
//   One launch, one thread per output pixel: the uint8 intermediate of the horizontal pass is recomputed per vertical tap in
//   registers instead of going through global memory (each source row is read from L1 / L2 by the neighbouring threads).
#include <cmath>
#include <cstdint>

#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"

namespace svdx {

constexpr int kPrecisionBits = 32 - 8 - 2;

// Pillow's bicubic_filter (a = -0.5), same operation order
static double bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

static int taps_ksize(int in_size, int out_size) {
  double filterscale = (double)(float)in_size / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  return (int)std::ceil(2.0 * filterscale) * 2 + 1;
}

SVDX_DEVINL int clip8(int v) {
  v >>= kPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// frame n of the range: n < B*F is clip frame n = b*F + f; n = B*F + b is the conditioning frame of clip b (its frame 0, noise
// augmented). taps_y / taps_x: per output row / column [lo, count, k_0 .. k_{ksize-1}].
__global__ void __launch_bounds__(256) frames_u8_in_kernel(
    const uint8_t* __restrict__ src, int H0, int W0, const int* __restrict__ taps_y, int ks_y, const int* __restrict__ taps_x,
    int ks_x, const float* __restrict__ eps, const float* __restrict__ sigma_c, int B, int F, int H, int W, int first, int c_pad,
    bf16* __restrict__ dst, float* __restrict__ first_frames) {
  const int hw = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  const int n = first + (int)blockIdx.y;
  const int y = p / W, x = p - (p / W) * W;
  const long long sn = n < B * F ? n : (long long)(n - B * F) * F;
  const uint8_t* s = src + sn * H0 * W0 * 3;
  const int* ty = taps_y + (long long)y * (ks_y + 2);
  const int* tx = taps_x + (long long)x * (ks_x + 2);
  const int y0 = ty[0], ny = ty[1], x0 = tx[0], nx = tx[1];
  const int half = 1 << (kPrecisionBits - 1);
  int a0 = half, a1 = half, a2 = half;
  for (int j = 0; j < ny; ++j) {
    const uint8_t* row = s + ((long long)(y0 + j) * W0 + x0) * 3;
    int h0 = half, h1 = half, h2 = half;
    for (int i = 0; i < nx; ++i) {
      const int k = tx[2 + i];
      h0 += (int)row[3 * i] * k;
      h1 += (int)row[3 * i + 1] * k;
      h2 += (int)row[3 * i + 2] * k;
    }
    const int k = ty[2 + j];
    a0 += clip8(h0) * k;
    a1 += clip8(h1) * k;
    a2 += clip8(h2) * k;
  }
  float v[3] = {(float)clip8(a0), (float)clip8(a1), (float)clip8(a2)};
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = __fsub_rn(__fdiv_rn(v[c], 127.5f), 1.f);
  if (n >= B * F) {
    const int b = n - B * F;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long e = ((long long)b * 3 + c) * hw + p;
      if (first_frames) first_frames[e] = v[c];
      v[c] = __fadd_rn(__fmul_rn(eps[e], sigma_c[b]), v[c]);
    }
  }
  // c_pad is a multiple of 8: one 16-byte store with the three channels, then zeros
  uint4* out = reinterpret_cast<uint4*>(dst + ((long long)blockIdx.y * hw + p) * c_pad);
  __align__(16) bf16 head[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) head[c] = __float2bfloat16(c < 3 ? v[c] : 0.f);
  out[0] = *reinterpret_cast<const uint4*>(head);
  for (int q = 1; q < c_pad / 8; ++q) out[q] = make_uint4(0, 0, 0, 0);
}

}  // namespace svdx

using namespace svdx;

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int svdx_resize_taps_ksize(int32_t in_size, int32_t out_size) {
  if (in_size <= 0 || out_size <= 0) return svdx_fail(SVDX_E_BADARG, "resize_taps_ksize: sizes must be positive");
  return taps_ksize(in_size, out_size);
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the box [0, in_size) -> out_size
extern "C" int svdx_resize_taps(int32_t in_size, int32_t out_size, int32_t* taps) {
  if (in_size <= 0 || out_size <= 0 || !taps) return svdx_fail(SVDX_E_BADARG, "resize_taps: bad arguments");
  const float in0 = 0.f, in1 = (float)in_size;
  const double scale = (double)(in1 - in0) / out_size;
  double filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  const int ksize = (int)std::ceil(support) * 2 + 1;
  double* k = new double[ksize];
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    int x = 0;
    for (; x < xmax; ++x) {
      const double w = bicubic((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    for (; x < ksize; ++x) k[x] = 0;
    int32_t* t = taps + (long long)xx * (ksize + 2);
    t[0] = xmin;
    t[1] = xmax;
    for (x = 0; x < ksize; ++x)
      t[2 + x] = k[x] < 0 ? (int)(-0.5 + k[x] * (1 << kPrecisionBits)) : (int)(0.5 + k[x] * (1 << kPrecisionBits));
  }
  delete[] k;
  return SVDX_OK;
}

extern "C" int svdx_frames_u8_in(const uint8_t* src, int32_t H0, int32_t W0, const int32_t* taps_y, int32_t ksize_y,
                                 const int32_t* taps_x, int32_t ksize_x, const float* cond_eps, const float* cond_sigma, int32_t B,
                                 int32_t F, int32_t H, int32_t W, int32_t first, int32_t count, int32_t c_pad, void* dst,
                                 float* first_frames, void* stream) {
  if (!src || !taps_y || !taps_x || !cond_eps || !cond_sigma || !dst || B <= 0 || F <= 0 || H <= 0 || W <= 0 || H0 <= 0 ||
      W0 <= 0 || ksize_y != taps_ksize(H0, H) || ksize_x != taps_ksize(W0, W) || c_pad < 8 || c_pad % 8 ||
      (reinterpret_cast<uintptr_t>(dst) & 15) || first < 0 || count <= 0 || count > 65535 || first + count > B * (F + 1))
    return svdx_fail(SVDX_E_BADARG, "frames_u8_in: bad arguments (uint8 frames [B, F, H0, W0, 3], taps of svdx_resize_taps, "
                                    "c_pad a multiple of 8, 16-byte aligned dst, 0 <= first < first + count <= B*(F+1))");
  const dim3 grid((unsigned)((H * W + 255) / 256), (unsigned)count);
  frames_u8_in_kernel<<<grid, 256, 0, ST(stream)>>>(src, H0, W0, taps_y, ksize_y, taps_x, ksize_x, cond_eps, cond_sigma, B, F, H, W,
                                                     first, c_pad, reinterpret_cast<bf16*>(dst), first_frames);
  SVDX_CHECK_LAUNCH("frames_u8_in");
  return SVDX_OK;
}
