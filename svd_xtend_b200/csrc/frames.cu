// Decoded video frames -> the VAE encoder's input rows of a training step (svd_xtend_b200.video_train, uint8 input form).
//
// svdx_resize_taps (host): the per-output-pixel taps of Pillow's 8-bpc BICUBIC resample along one axis, the filter
//   `Image.resize((W, H))` applies to an RGB image by default (Pillow's libImaging/Resample.c): a = -0.5, support 2 scaled by the
//   downscale factor (antialiasing), weights in double, normalised by their sum, then 22-bit fixed point rounded half away from
//   zero. Computed on the host, once per (source, target) size, in the same double operations as Pillow. The box form is
//   `Image.resize(size, box=...)`: the taps of the source interval [in0, in1) (float bounds, as Pillow stores them).
// svdx_frames_u8_in: uint8 HWC RGB frames [B][F][H0][W0][3] -> the horizontal pass (clamped to a uint8 intermediate), the
//   vertical pass (clamped to uint8), u / 127.5f - 1 (train_svd.py's DummyDataset) -> bf16 encoder rows over a frame range, in
//   svdx_vae_frames_in's layout and rounding, plus the clean first frame of each clip in fp32 for the CLIP encoder.
//   One launch, one thread per output pixel: the uint8 intermediate of the horizontal pass is recomputed per vertical tap in
//   registers instead of going through global memory (each source row is read from L1 / L2 by the neighbouring threads).
// svdx_frames_u8_in_clips: the same kernel with one descriptor per clip (svdx_clip_desc: where the clip starts, its source size
//   and its tap rows), so that the clips of one launch may have different source sizes and crop boxes. svdx_frames_u8_in is the
//   case where every clip shares one descriptor.
//
// Pillow runs a pass only when `out != in || box_lo != 0 || box_hi != in` on that axis and copies the axis otherwise. The taps
// of the box [0, in) with out == in are the identity (one weight of exactly 1 << 22), so the kernel runs both passes always and
// gets the copy bit for bit.
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

// Pillow's ksize for the box [in0, in1) -> out_size: the scale is (double)(in1 - in0) / out_size with in1 - in0 in float
static int taps_ksize(float in0, float in1, int out_size) {
  double filterscale = (double)(in1 - in0) / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  return (int)std::ceil(2.0 * filterscale) * 2 + 1;
}

static int taps_ksize(int in_size, int out_size) { return taps_ksize(0.f, (float)in_size, out_size); }

// Pillow's box rules (`box offset can't be negative`, `box can't exceed original image size`, `box can't be empty`), plus a
// finite box; a box of zero extent is accepted, as Pillow accepts it
static bool box_ok(int in_size, float in0, float in1) {
  return std::isfinite(in0) && std::isfinite(in1) && in0 >= 0.f && in1 <= (float)in_size && in1 - in0 >= 0.f;
}

SVDX_DEVINL int clip8(int v) {
  v >>= kPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// frame n of the range: n < B*F is frame f = n % F of clip b = n / F; n = B*F + b is the conditioning frame of clip b (its frame
// 0, noise augmented). Clip b's descriptor is descs[b], or d0 for every clip when descs is NULL; its frame f starts at byte
// b * clip_stride + start + f * H0*W0*3 of src. taps_y / taps_x: rows [lo, count, k_0 .. k_{ks-1}], the clip's output row y at
// row ty_off + y. A descriptor whose frames or tap rows do not fit in src_bytes / ty_rows / tx_rows reads nothing (its frames
// come out as u = 0), and tap rows are clamped to the clip's source size, so device data never leads outside the buffers.
__global__ void __launch_bounds__(256) frames_u8_in_kernel(
    const uint8_t* __restrict__ src, long long src_bytes, long long clip_stride, const svdx_clip_desc* __restrict__ descs,
    svdx_clip_desc d0, const int* __restrict__ taps_y, int ty_rows, int ks_y, const int* __restrict__ taps_x, int tx_rows,
    int ks_x, const float* __restrict__ eps, const float* __restrict__ sigma_c, int B, int F, int H, int W, int first, int c_pad,
    bf16* __restrict__ dst, float* __restrict__ first_frames) {
  const int hw = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  const int n = first + (int)blockIdx.y;
  const int y = p / W, x = p - (p / W) * W;
  const int b = n < B * F ? n / F : n - B * F;
  const int f = n < B * F ? n - b * F : 0;
  const svdx_clip_desc d = descs ? descs[b] : d0;
  const long long start = b * clip_stride + d.start;
  const long long avail = src_bytes - start;
  const bool ok = d.H0 > 0 && d.W0 > 0 && start >= 0 && avail > 0 && d.W0 <= avail / 3 / F &&
                  d.H0 <= avail / ((long long)d.W0 * 3 * F) && d.ty_off >= 0 && d.ty_off <= ty_rows - H && d.tx_off >= 0 &&
                  d.tx_off <= tx_rows - W;
  const int H0 = ok ? d.H0 : 1, W0 = ok ? d.W0 : 1;
  const uint8_t* s = src + (ok ? start + (long long)f * H0 * W0 * 3 : 0);
  const int* ty = taps_y + (long long)((ok ? d.ty_off : 0) + y) * (ks_y + 2);
  const int* tx = taps_x + (long long)((ok ? d.tx_off : 0) + x) * (ks_x + 2);
  int y0 = 0, ny = 0, x0 = 0, nx = 0;
  if (ok) {
    y0 = min(max(ty[0], 0), H0);
    ny = min(max(ty[1], 0), min(ks_y, H0 - y0));
    x0 = min(max(tx[0], 0), W0);
    nx = min(max(tx[1], 0), min(ks_x, W0 - x0));
  }
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

extern "C" int svdx_resize_taps_box_ksize(int32_t in_size, int32_t out_size, float in0, float in1) {
  if (in_size <= 0 || out_size <= 0 || !box_ok(in_size, in0, in1))
    return svdx_fail(SVDX_E_BADARG, "resize_taps_box_ksize: sizes must be positive and 0 <= in0 <= in1 <= in_size");
  return taps_ksize(in0, in1, out_size);
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the box [in0, in1) of an axis of in_size -> out_size
extern "C" int svdx_resize_taps_box(int32_t in_size, int32_t out_size, float in0, float in1, int32_t* taps) {
  if (in_size <= 0 || out_size <= 0 || !taps || !box_ok(in_size, in0, in1))
    return svdx_fail(SVDX_E_BADARG, "resize_taps_box: bad arguments (positive sizes, 0 <= in0 <= in1 <= in_size)");
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

// the box [0, in_size)
extern "C" int svdx_resize_taps(int32_t in_size, int32_t out_size, int32_t* taps) {
  if (in_size <= 0 || out_size <= 0 || !taps) return svdx_fail(SVDX_E_BADARG, "resize_taps: bad arguments");
  return svdx_resize_taps_box(in_size, out_size, 0.f, (float)in_size, taps);
}

static bool range_ok(int32_t B, int32_t F, int32_t first, int32_t count) {
  return first >= 0 && count > 0 && count <= 65535 && (long long)first + count <= (long long)B * (F + 1);
}

static int launch_frames(const uint8_t* src, long long src_bytes, long long clip_stride, const svdx_clip_desc* descs,
                         svdx_clip_desc d0, const int32_t* taps_y, int ty_rows, int ks_y, const int32_t* taps_x, int tx_rows,
                         int ks_x, const float* cond_eps, const float* cond_sigma, int B, int F, int H, int W, int first, int count,
                         int c_pad, void* dst, float* first_frames, void* stream, const char* what) {
  const dim3 grid((unsigned)((H * W + 255) / 256), (unsigned)count);
  frames_u8_in_kernel<<<grid, 256, 0, ST(stream)>>>(src, src_bytes, clip_stride, descs, d0, taps_y, ty_rows, ks_y, taps_x, tx_rows,
                                                     ks_x, cond_eps, cond_sigma, B, F, H, W, first, c_pad,
                                                     reinterpret_cast<bf16*>(dst), first_frames);
  SVDX_CHECK_LAUNCH(what);
  return SVDX_OK;
}

extern "C" int svdx_frames_u8_in(const uint8_t* src, int32_t H0, int32_t W0, const int32_t* taps_y, int32_t ksize_y,
                                 const int32_t* taps_x, int32_t ksize_x, const float* cond_eps, const float* cond_sigma, int32_t B,
                                 int32_t F, int32_t H, int32_t W, int32_t first, int32_t count, int32_t c_pad, void* dst,
                                 float* first_frames, void* stream) {
  if (!src || !taps_y || !taps_x || !cond_eps || !cond_sigma || !dst || B <= 0 || F <= 0 || H <= 0 || W <= 0 || H0 <= 0 ||
      W0 <= 0 || ksize_y != taps_ksize(H0, H) || ksize_x != taps_ksize(W0, W) || c_pad < 8 || c_pad % 8 ||
      (reinterpret_cast<uintptr_t>(dst) & 15) || !range_ok(B, F, first, count))
    return svdx_fail(SVDX_E_BADARG, "frames_u8_in: bad arguments (uint8 frames [B, F, H0, W0, 3], taps of svdx_resize_taps, "
                                    "c_pad a multiple of 8, 16-byte aligned dst, 0 <= first < first + count <= B*(F+1))");
  const long long clip = (long long)F * H0 * W0 * 3;
  const svdx_clip_desc d0 = {0, H0, W0, 0, 0};
  return launch_frames(src, clip * B, clip, nullptr, d0, taps_y, H, ksize_y, taps_x, W, ksize_x, cond_eps, cond_sigma, B, F, H, W,
                       first, count, c_pad, dst, first_frames, stream, "frames_u8_in");
}

extern "C" int svdx_frames_u8_in_clips(const uint8_t* src, int64_t src_bytes, const svdx_clip_desc* descs, const int32_t* taps_y,
                                       int32_t ty_rows, int32_t ksize_y, const int32_t* taps_x, int32_t tx_rows, int32_t ksize_x,
                                       const float* cond_eps, const float* cond_sigma, int32_t B, int32_t F, int32_t H, int32_t W,
                                       int32_t first, int32_t count, int32_t c_pad, void* dst, float* first_frames, void* stream) {
  if (!src || src_bytes <= 0 || !descs || (reinterpret_cast<uintptr_t>(descs) & 7) || !taps_y || !taps_x || !cond_eps ||
      !cond_sigma || !dst || B <= 0 || F <= 0 || H <= 0 || W <= 0 || ksize_y < 1 || ksize_x < 1 || ty_rows < H || tx_rows < W ||
      c_pad < 8 || c_pad % 8 || (reinterpret_cast<uintptr_t>(dst) & 15) || !range_ok(B, F, first, count))
    return svdx_fail(SVDX_E_BADARG, "frames_u8_in_clips: bad arguments (src_bytes > 0, 8-byte aligned descs [B], tap tables of "
                                    "at least H / W rows of 2 + ksize >= 3, c_pad a multiple of 8, 16-byte aligned dst, "
                                    "0 <= first < first + count <= B*(F+1))");
  const svdx_clip_desc none = {0, 0, 0, 0, 0};
  return launch_frames(src, src_bytes, 0, descs, none, taps_y, ty_rows, ksize_y, taps_x, tx_rows, ksize_x, cond_eps, cond_sigma, B,
                       F, H, W, first, count, c_pad, dst, first_frames, stream, "frames_u8_in_clips");
}
