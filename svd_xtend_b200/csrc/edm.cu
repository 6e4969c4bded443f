// The batch assembly of a training step from video frames (train_svd.py:942-1017), around the frozen VAE encoder:
//
// svdx_vae_frames_in: the clip frames and the noise-augmented conditioning frames -> the VAE encoder's bf16 input rows in one
//   pass, so that ONE encode of B*(F+1) frames replaces the reference's two (the encoder is per frame: GroupNorm per frame, no
//   temporal layers). The concatenated fp32 frame batch is never materialised.
// svdx_edm_prepare: the encoder's moments -> posterior samples, EDM noising, input scaling and the conditioning channels of the
//   UNet input, the noisy latents and the target, one thread per latent element.
//
// Every operation is rounded separately (__fmul_rn / __fadd_rn / __fdiv_rn / __fsqrt_rn, no contraction) in the reference's
// order, so the torch statement in oracle/svd_train_batch_oracle.py reproduces the outputs bit for bit on the same inputs.
#include "common.cuh"
#include "../../include/svd_xtend_b200.h"
#include "host_util.h"

namespace svdx {

SVDX_DEVINL float ld_pix(const void* x, int bf, long long i) {
  return bf ? __bfloat162float(reinterpret_cast<const bf16*>(x)[i]) : reinterpret_cast<const float*>(x)[i];
}

// row n < B*F: clip frame n = b*F + f; row B*F + b: fl(fl(eps[b] * sigma_c[b]) + x[b, 0]). dst holds the rows of the frames
// [first, first + count).
__global__ void vae_frames_in_kernel(const void* __restrict__ x, int x_bf16, const float* __restrict__ eps,
                                     const float* __restrict__ sigma_c, int B, int F, int H, int W, int first, int count, int c_pad,
                                     bf16* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long hw = (long long)H * W;
  const long long total = (long long)count * hw * c_pad;
  if (idx >= total) return;
  const int c = (int)(idx % c_pad);
  const long long pix = idx / c_pad;
  const long long p = pix % hw;
  const int n = first + (int)(pix / hw);
  float v = 0.f;
  if (c < 3) {
    if (n < B * F) {
      v = ld_pix(x, x_bf16, ((long long)n * 3 + c) * hw + p);
    } else {
      const int b = n - B * F;
      const float x0 = ld_pix(x, x_bf16, ((long long)b * F * 3 + c) * hw + p);
      v = __fadd_rn(__fmul_rn(eps[((long long)b * 3 + c) * hw + p], sigma_c[b]), x0);
    }
  }
  dst[idx] = __float2bfloat16(v);
}

// posterior sample of one latent element from the moments row n (mean at channel c, logvar at C + c)
SVDX_DEVINL float posterior(const float* __restrict__ mom, long long n, int c, int C, long long hw, long long p, float e) {
  const float mean = mom[(n * 2 * C + c) * hw + p];
  float lv = mom[(n * 2 * C + C + c) * hw + p];
  lv = lv < -30.f ? -30.f : (lv > 20.f ? 20.f : lv);          // torch.clamp (a NaN passes through)
  const float sd = expf(__fmul_rn(0.5f, lv));
  return __fadd_rn(mean, __fmul_rn(sd, e));
}

__global__ void edm_prepare_kernel(const float* __restrict__ mom, const float* __restrict__ latent_eps,
                                   const float* __restrict__ noise, const float* __restrict__ cond_eps,
                                   const float* __restrict__ sigma, const float* __restrict__ image_mask, float sf,
                                   int B, int F, int C, long long hw, float* __restrict__ sample, float* __restrict__ noisy,
                                   float* __restrict__ latents) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * F * C * hw;
  if (idx >= total) return;
  const long long p = idx % hw;
  const int c = (int)((idx / hw) % C);
  const long long n = idx / (hw * C);          // frame b*F + f
  const int b = (int)(n / F);
  const float s = sigma[b];
  const float lat = __fmul_rn(posterior(mom, n, c, C, hw, p, latent_eps[idx]), sf);
  const float nz = __fadd_rn(lat, __fmul_rn(noise[idx], s));
  const float inp = __fdiv_rn(nz, __fsqrt_rn(__fadd_rn(__fmul_rn(s, s), 1.f)));
  const long long nc = (long long)B * F + b;
  const float zc = posterior(mom, nc, c, C, hw, p, cond_eps[((long long)b * C + c) * hw + p]);
  // torch divides a CUDA tensor by a Python scalar as a multiplication by the scalar's fp32 reciprocal (:960 on the GPU)
  const float cond = __fmul_rn(__fmul_rn(zc, sf), __fdiv_rn(1.f, sf));
  latents[idx] = lat;
  noisy[idx] = nz;
  sample[(n * 2 * C + c) * hw + p] = inp;
  sample[(n * 2 * C + C + c) * hw + p] = __fmul_rn(image_mask[b], cond);
}

}  // namespace svdx

using namespace svdx;

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int svdx_vae_frames_in(const void* x, int32_t x_dtype, const float* cond_eps, const float* cond_sigma, int32_t B,
                                  int32_t F, int32_t H, int32_t W, int32_t c_pad, void* dst, void* stream) {
  if (!x || !cond_eps || !cond_sigma || !dst || B <= 0 || F <= 0 || H <= 0 || W <= 0 || c_pad < 3 || (x_dtype != 0 && x_dtype != 1))
    return svdx_fail(SVDX_E_BADARG, "vae_frames_in: bad arguments (fp32 / bf16 frames [B, F, 3, H, W], c_pad >= 3)");
  return svdx_vae_frames_in_range(x, x_dtype, cond_eps, cond_sigma, B, F, H, W, 0, B * (F + 1), c_pad, dst, stream);
}

extern "C" int svdx_vae_frames_in_range(const void* x, int32_t x_dtype, const float* cond_eps, const float* cond_sigma, int32_t B,
                                        int32_t F, int32_t H, int32_t W, int32_t first, int32_t count, int32_t c_pad, void* dst,
                                        void* stream) {
  if (!x || !cond_eps || !cond_sigma || !dst || B <= 0 || F <= 0 || H <= 0 || W <= 0 || c_pad < 3 || (x_dtype != 0 && x_dtype != 1) ||
      first < 0 || count <= 0 || first + count > B * (F + 1))
    return svdx_fail(SVDX_E_BADARG, "vae_frames_in_range: bad arguments (fp32 / bf16 frames [B, F, 3, H, W], c_pad >= 3, "
                                    "0 <= first < first + count <= B*(F+1))");
  const long long total = (long long)count * H * W * c_pad;
  vae_frames_in_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ST(stream)>>>(x, x_dtype, cond_eps, cond_sigma, B, F, H, W, first,
                                                                                count, c_pad, reinterpret_cast<bf16*>(dst));
  SVDX_CHECK_LAUNCH("vae_frames_in");
  return SVDX_OK;
}

extern "C" int svdx_edm_prepare(const float* moments, const float* latent_eps, const float* noise, const float* cond_latent_eps,
                                const float* sigma, const float* image_mask, float scaling_factor, int32_t B, int32_t F, int32_t C,
                                int32_t h, int32_t w, float* sample, float* noisy, float* latents, void* stream) {
  if (!moments || !latent_eps || !noise || !cond_latent_eps || !sigma || !image_mask || !sample || !noisy || !latents || B <= 0 ||
      F <= 0 || C <= 0 || h <= 0 || w <= 0)
    return svdx_fail(SVDX_E_BADARG, "edm_prepare: bad arguments");
  const long long total = (long long)B * F * C * h * w;
  edm_prepare_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ST(stream)>>>(moments, latent_eps, noise, cond_latent_eps, sigma,
                                                                              image_mask, scaling_factor, B, F, C, (long long)h * w,
                                                                              sample, noisy, latents);
  SVDX_CHECK_LAUNCH("edm_prepare");
  return SVDX_OK;
}
