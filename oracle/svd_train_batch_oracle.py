"""ORACLE — test infrastructure only. Plain-torch statement of the batch assembly of train_svd.py's training step (:942-1017)
over GIVEN encoder moments, image embeddings and random draws, and of its loss (:1025-1036): what
svd_xtend_b200.video_train.assemble_train_batch (kernels svdx_vae_frames_in / svdx_edm_prepare) computes. Line numbers are
/root/reference/train_svd.py's. Runs in the dtype of its inputs (fp32 on the GPU for the bitwise kernel tests, fp64 on the
CPU against tests/golden/train_batch_golden.pt).

Draws, by name (svd_xtend_b200.video_train.draw_train_noise): latent_eps, noise, cond_u, cond_pixel_eps, cond_latent_eps,
sigma_u and, with conditioning dropout, dropout_u.
"""
from __future__ import annotations

import torch

from oracle.svd_unet_oracle import edm_loss  # noqa: F401  (train_svd.py:1025-1036)


def log_normal(u: torch.Tensor, loc: float, scale: float) -> torch.Tensor:
    """rand_log_normal (:64-67) from its uniform draw u, in fp32 as the reference draws it"""
    u = u.float() * (1 - 2e-7) + 1e-7
    return torch.distributions.Normal(loc, scale).icdf(u).exp()


def posterior(moments: torch.Tensor, eps: torch.Tensor) -> torch.Tensor:
    """latent_dist.sample() of tensor_to_vae_latent (:287): mean + exp(0.5 * clamp(logvar, -30, 20)) * eps"""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
    return mean + std * eps


def frames_in(pixel_values: torch.Tensor, cond_pixel_eps: torch.Tensor, cond_sigma: torch.Tensor) -> torch.Tensor:
    """the VAE's input frames [B*F + B, 3, H, W] in the inputs' dtype: the clip frames (:948), then the noise-augmented
    conditioning frames randn_like(x0) * cond_sigma + x0 (:957-958)"""
    B, F = pixel_values.shape[:2]
    x = pixel_values
    cond = cond_pixel_eps.reshape(B, 3, *x.shape[-2:]) * cond_sigma.reshape(B, 1, 1, 1) + x[:, 0]
    return torch.cat([x.reshape(B * F, *x.shape[2:]), cond])


def dropout_masks(r: torch.Tensor, p: float):
    """(prompt dropped [B] bool, image_mask [B]) of the conditioning dropout (:993-1008), compared in r's dtype (fp32) as the
    reference does: r < 2p drops the image embedding, p <= r < 3p the conditioning latents"""
    prompt = r < 2 * p
    image_mask = 1 - (r >= p).to(r.dtype) * (r < 3 * p).to(r.dtype)
    return prompt, image_mask


def prepare(moments, latent_eps, noise, cond_latent_eps, sigma, image_mask, scaling_factor):
    """svdx_edm_prepare: moments [B*(F+1), 2C, h, w] (the clip frames, then the conditioning frames) -> (sample, noisy, latents)"""
    B = sigma.shape[0]
    N, C2, h, w = moments.shape
    F, C = N // B - 1, C2 // 2
    s = sigma.reshape(B, 1, 1, 1, 1)
    latents = (posterior(moments[:B * F], latent_eps.reshape(B * F, C, h, w)) * scaling_factor).reshape(B, F, C, h, w)  # :948
    noisy = latents + noise.reshape(B, F, C, h, w) * s                                                            # :968
    inp = noisy / (s * s + 1).sqrt()                                                # :972, the scale in sigma's dtype
    cond = posterior(moments[B * F:], cond_latent_eps.reshape(B, C, h, w)) * scaling_factor / scaling_factor      # :959-960
    cond = image_mask.reshape(B, 1, 1, 1) * cond                                                                  # :1008
    sample = torch.cat([inp, cond.unsqueeze(1).repeat(1, F, 1, 1, 1)], dim=2)                                     # :1014-1017
    return sample, noisy, latents


def train_batch(clip_moments, cond_moments, image_embeds, draws, *, scaling_factor=0.18215, conditioning_dropout_prob=None,
                fps=7, motion_bucket_id=127, dtype=torch.float64):
    """the UNet batch of one step (the keys of workload.synthetic_batch) in `dtype`, from the moments of the clip frames
    [B*F, 2C, h, w] and of the conditioning frames [B, 2C, h, w], the CLIP embeddings of the clean first frames [B, D] and the
    draws. The sigmas are drawn in fp32 (rand_log_normal's default dtype) and stay fp32, as in the reference: sigmas, timestep,
    and the input scale sqrt(sigma^2 + 1) are fp32 quantities, widened where they meet the latents. added_time_ids carry each clip's own
    conditioning sigma (the reference uses clip 0's for all, :981)."""
    B = image_embeds.shape[0]
    c = lambda t: t.to(dtype)       # noqa: E731
    cond_sigma = c(log_normal(draws["cond_u"], -3.0, 0.5))                   # :954
    sigma = log_normal(draws["sigma_u"], 0.7, 1.6)                           # :964, stays fp32 (:965-967)
    ehs = c(image_embeds).unsqueeze(1)                                       # :975
    image_mask = torch.ones(B, dtype=dtype)
    if conditioning_dropout_prob is not None:
        prompt, image_mask = dropout_masks(draws["dropout_u"].float(), conditioning_dropout_prob)
        ehs = torch.where(prompt.reshape(B, 1, 1), torch.zeros_like(ehs), ehs)       # :996-999
        image_mask = c(image_mask)
    moments = torch.cat([c(clip_moments), c(cond_moments)])
    sample, noisy, latents = prepare(moments, c(draws["latent_eps"]), c(draws["noise"]), c(draws["cond_latent_eps"]), sigma,
                                     image_mask.to(moments.device), scaling_factor)
    added_time_ids = torch.stack([torch.full((B,), float(fps), dtype=dtype), torch.full((B,), float(motion_bucket_id), dtype=dtype),
                                  cond_sigma.cpu()], dim=1).to(moments.device)                 # :981-987
    return dict(sample=sample, timestep=c(0.25 * sigma.log()), encoder_hidden_states=ehs, added_time_ids=added_time_ids,
                latents=latents, noisy=noisy, sigmas=sigma.reshape(B, 1, 1, 1, 1))
