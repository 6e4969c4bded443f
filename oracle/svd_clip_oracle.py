"""ORACLE — test infrastructure only. Plain-PyTorch restatement of the CLIP image encoder of the SVD pipeline and of the
image-to-video composition around it:

  * transformers' `CLIPVisionModelWithProjection` (ViT-H/14 in the SVD checkpoint's `image_encoder/`): patch embedding (a
    stride-14 conv without bias), class token, position embedding, `pre_layrnorm`, pre-LN encoder layers (q/k/v/out
    projections with biases, unmasked SDPA at scale head_dim^-1/2, fc1 -> gelu / quick_gelu -> fc2), `post_layernorm` of token 0,
    `visual_projection` without bias. Module / parameter names and registration order follow the transformers state dict.
  * the reference's conditioning-image preprocessing (train_svd.py:857-876 `encode_image`, and diffusers'
    `StableVideoDiffusionPipeline._encode_image` [D]): an anti-aliased resize to 224x224 (a separable Gaussian blur with
    reflect padding, then a bicubic interpolation with align_corners=True), (x + 1) / 2, CLIPImageProcessor's normalisation.
  * the patch-row layout the H100 encoder's preprocess kernel writes (`patchify`).
  * `image_to_video`: [D] StableVideoDiffusionPipeline.__call__ with output_type="pt" on top of the sampling and decoder oracles.

tests/golden/clip_golden.pt pins `CLIPVisionModelWithProjection` against transformers and `resize_with_antialiasing` against the
reference's own function (tests/golden/make_clip_golden.py). fp32 or fp64, whatever dtype the parameters / inputs have.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

CLIP_CONFIG = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=32, patch_size=14,
                   image_size=224, projection_dim=1024, layer_norm_eps=1e-5, hidden_act="gelu", num_channels=3)
# head dim 80 like ViT-H, so the tiny model runs the same attention kernel
TINY_CLIP_CONFIG = dict(hidden_size=160, intermediate_size=640, num_attention_heads=2, num_hidden_layers=2, patch_size=14,
                        image_size=224, projection_dim=96, layer_norm_eps=1e-5, hidden_act="gelu", num_channels=3)

# CLIPImageProcessor's defaults (the SVD checkpoint's feature_extractor/preprocessor_config.json carries the same values)
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def activation(name: str):
    if name == "gelu":
        return F.gelu
    if name == "quick_gelu":
        return lambda x: x * torch.sigmoid(1.702 * x)
    raise ValueError(f"unsupported hidden_act {name!r}")


class _Embeddings(nn.Module):
    def __init__(self, C, patch, image_size, channels):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.randn(C))
        self.patch_embedding = nn.Conv2d(channels, C, patch, stride=patch, bias=False)
        self.position_embedding = nn.Embedding((image_size // patch) ** 2 + 1, C)

    def forward(self, x):
        p = self.patch_embedding(x.to(self.patch_embedding.weight.dtype)).flatten(2).transpose(1, 2)
        cls = self.class_embedding.expand(x.shape[0], 1, -1)
        return torch.cat([cls, p], dim=1) + self.position_embedding.weight[None]


class _Attention(nn.Module):
    def __init__(self, C, heads):
        super().__init__()
        self.heads = heads
        self.k_proj = nn.Linear(C, C)
        self.v_proj = nn.Linear(C, C)
        self.q_proj = nn.Linear(C, C)
        self.out_proj = nn.Linear(C, C)

    def forward(self, x):
        B, S, C = x.shape
        d = C // self.heads
        q, k, v = (f(x).view(B, S, self.heads, d).transpose(1, 2) for f in (self.q_proj, self.k_proj, self.v_proj))
        a = torch.softmax((q @ k.transpose(-1, -2)) * d ** -0.5, dim=-1) @ v
        return self.out_proj(a.transpose(1, 2).reshape(B, S, C))


class _MLP(nn.Module):
    def __init__(self, C, I, act):
        super().__init__()
        self.act = activation(act)
        self.fc1 = nn.Linear(C, I)
        self.fc2 = nn.Linear(I, C)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class _Layer(nn.Module):
    def __init__(self, C, I, heads, eps, act):
        super().__init__()
        self.self_attn = _Attention(C, heads)
        self.layer_norm1 = nn.LayerNorm(C, eps=eps)
        self.mlp = _MLP(C, I, act)
        self.layer_norm2 = nn.LayerNorm(C, eps=eps)

    def forward(self, x):
        x = x + self.self_attn(self.layer_norm1(x))
        return x + self.mlp(self.layer_norm2(x))


class _Encoder(nn.Module):
    def __init__(self, C, I, heads, layers, eps, act):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(C, I, heads, eps, act) for _ in range(layers)])


class _VisionTransformer(nn.Module):
    def __init__(self, C, I, heads, layers, patch, image_size, channels, eps, act):
        super().__init__()
        self.embeddings = _Embeddings(C, patch, image_size, channels)
        self.pre_layrnorm = nn.LayerNorm(C, eps=eps)
        self.encoder = _Encoder(C, I, heads, layers, eps, act)
        self.post_layernorm = nn.LayerNorm(C, eps=eps)


class CLIPVisionModelWithProjection(nn.Module):
    def __init__(self, hidden_size=768, intermediate_size=3072, num_attention_heads=12, num_hidden_layers=12, patch_size=32,
                 image_size=224, projection_dim=512, layer_norm_eps=1e-5, hidden_act="quick_gelu", num_channels=3, **ignored):
        super().__init__()
        activation(hidden_act)
        self.config = SimpleNamespace(hidden_size=hidden_size, intermediate_size=intermediate_size, num_attention_heads=num_attention_heads,
                                      num_hidden_layers=num_hidden_layers, patch_size=patch_size, image_size=image_size,
                                      projection_dim=projection_dim, layer_norm_eps=layer_norm_eps, hidden_act=hidden_act,
                                      num_channels=num_channels)
        self.vision_model = _VisionTransformer(hidden_size, intermediate_size, num_attention_heads, num_hidden_layers, patch_size,
                                               image_size, num_channels, layer_norm_eps, hidden_act)
        self.visual_projection = nn.Linear(hidden_size, projection_dim, bias=False)

    def forward(self, pixel_values):
        vm = self.vision_model
        x = vm.pre_layrnorm(vm.embeddings(pixel_values))
        for layer in vm.encoder.layers:
            x = layer(x)
        pooled = vm.post_layernorm(x[:, 0])
        return SimpleNamespace(image_embeds=self.visual_projection(pooled), last_hidden_state=x)


def integer_init_(model: nn.Module, seed: int) -> nn.Module:
    """deterministic parameters from integer draws scaled by powers of two (exact in fp32 and fp64, the same on every CPU):
    weights ~ k / 2^(3 + log2 fan_in / 2), biases k / 256, LayerNorm weights 1 + k / 64, embeddings k / 16, k small integers"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            k = torch.randint(-8, 9, p.shape, generator=g).to(p.dtype)
            if "norm" in n and n.endswith("weight"):
                p.copy_(1.0 + k / 64)
            elif n.endswith("bias"):
                p.copy_(k / 256)
            elif "embedding" in n and "patch" not in n:
                p.copy_(k / 16)
            else:
                fan_in = p[0].numel()
                p.copy_(k * 2.0 ** -(3 + round(math.log2(fan_in) / 2)))
    return model


def integer_pixels(shape, seed: int, dtype=torch.float64) -> torch.Tensor:
    """seeded inputs in [-1, 1] on a 1/128 grid"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-128, 129, shape, generator=g) / 128).to(dtype)


# ------------------------------------------------------------------------------------------------------------ preprocessing
def antialias_params(h: int, w: int, size=(224, 224)):
    """Gaussian sigmas and odd kernel sizes (y, x) of the anti-aliasing blur before a resize of h x w to `size`: sigma is half
    the excess of the down-scale factor (at least 0.001), the kernel spans four sigmas (at least 3 taps), made odd."""
    sig = (max((h / size[0] - 1.0) / 2.0, 0.001), max((w / size[1] - 1.0) / 2.0, 0.001))
    ks = [int(max(4.0 * s, 3)) for s in sig]
    ks = tuple(k + 1 if k % 2 == 0 else k for k in ks)
    return sig, ks


def gaussian_1d(k: int, sigma: float, dtype=torch.float32) -> torch.Tensor:
    """normalised Gaussian weights at the k integer offsets centred on k // 2, evaluated in `dtype` (the input's dtype)"""
    s = torch.tensor([[sigma]], dtype=dtype)
    x = torch.arange(k, dtype=dtype) - k // 2
    if k % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * s.pow(2.0)))
    return (g / g.sum(-1, keepdim=True))[0]


def gaussian_blur(x: torch.Tensor, gy: torch.Tensor, gx: torch.Tensor) -> torch.Tensor:
    """separable depthwise blur with reflect padding: along x first, then along y"""
    C = x.shape[1]
    ky, kx = gy.numel(), gx.numel()
    px, py = (kx - 1) // 2, (ky - 1) // 2
    h = F.conv2d(F.pad(x, (px, kx - 1 - px, 0, 0), mode="reflect"), gx.to(x.dtype).view(1, 1, 1, kx).expand(C, 1, 1, kx), groups=C)
    return F.conv2d(F.pad(h, (0, 0, py, ky - 1 - py), mode="reflect"), gy.to(x.dtype).view(1, 1, ky, 1).expand(C, 1, ky, 1), groups=C)


def resize_with_antialiasing(x: torch.Tensor, size=(224, 224)) -> torch.Tensor:
    """the reference's anti-aliased resize (train_svd.py `_resize_with_antialiasing`, restated): Gaussian blur, then bicubic
    interpolation with align_corners=True"""
    (sy, sx), (ky, kx) = antialias_params(x.shape[-2], x.shape[-1], size)
    x = gaussian_blur(x, gaussian_1d(ky, sy, x.dtype).to(x.device), gaussian_1d(kx, sx, x.dtype).to(x.device))
    return F.interpolate(x, size=size, mode="bicubic", align_corners=True)


def normalize(x: torch.Tensor, mean=CLIP_MEAN, std=CLIP_STD) -> torch.Tensor:
    m = torch.tensor(mean, dtype=x.dtype, device=x.device).view(1, -1, 1, 1)
    s = torch.tensor(std, dtype=x.dtype, device=x.device).view(1, -1, 1, 1)
    return (x - m) / s


def clip_input(pixel_values: torch.Tensor, image_size: int = 224, mean=CLIP_MEAN, std=CLIP_STD) -> torch.Tensor:
    """train_svd.py:857-871: images in [-1, 1] -> the normalised CLIP input"""
    x = resize_with_antialiasing(pixel_values, (image_size, image_size))
    return normalize((x + 1.0) / 2.0, mean, std)


def encode_image(model: CLIPVisionModelWithProjection, pixel_values: torch.Tensor, mean=CLIP_MEAN, std=CLIP_STD) -> torch.Tensor:
    x = clip_input(pixel_values.to(next(model.parameters()).dtype), model.config.image_size, mean, std)
    return model(x).image_embeds


def patchify(x: torch.Tensor, patch: int = 14, k_pad: int = 640) -> torch.Tensor:
    """[B, 3, S, S] -> [B * (1 + P^2), k_pad]: row 0 of each image zero (class slot), then patches in raster order, columns in
    the conv weight's (c, ky, kx) order, zero-padded from 3 * patch^2 to k_pad"""
    B, C, H, W = x.shape
    P = H // patch
    p = x.reshape(B, C, P, patch, P, patch).permute(0, 2, 4, 1, 3, 5).reshape(B, P * P, C * patch * patch)
    out = torch.zeros(B, 1 + P * P, k_pad, dtype=x.dtype, device=x.device)
    out[:, 1:, :C * patch * patch] = p
    return out.reshape(B * (1 + P * P), k_pad)


# ------------------------------------------------------------------------------------------------------------ image -> video
def image_to_video(unet, vae, image_encoder, image, *, num_frames, num_inference_steps=25, min_guidance_scale=1.0,
                   max_guidance_scale=3.0, fps=7, motion_bucket_id=127, noise_aug_strength=0.02, decode_chunk_size=None,
                   generator=None, latents=None, mean=CLIP_MEAN, std=CLIP_STD):
    """[D] StableVideoDiffusionPipeline.__call__(output_type="pt") on an image [B, 3, H, W] in [0, 1]: CLIP embedding of the
    image, noise-augmented conditioning latents (VAE mode, unscaled; the generator's FIRST draw), Euler / CFG sampling from the
    generator's SECOND draw (or `latents`), chunked temporal decode, frames [B, F, 3, H, W] in [0, 1]."""
    from .svd_sampling_oracle import sample_latents
    from .svd_vae_decoder_oracle import decode_latents
    x = image * 2.0 - 1.0
    gen_dev = x.device if generator is None else generator.device
    emb = encode_image(image_encoder, x, mean, std).unsqueeze(1)
    noise = torch.randn(x.shape, generator=generator, device=gen_dev, dtype=x.dtype).to(x.device)
    cond = x + noise_aug_strength * noise
    image_latents = vae.encode(cond).latent_dist.mode()
    B, _, h, w = image_latents.shape
    if latents is None:
        latents = torch.randn(B, num_frames, 4, h, w, generator=generator, device=gen_dev, dtype=torch.float32).to(x.device)
    lat = sample_latents(unet, image_latents.float(), emb.float(), num_frames=num_frames, fps=fps, motion_bucket_id=motion_bucket_id,
                         noise_aug_strength=noise_aug_strength, num_inference_steps=num_inference_steps,
                         min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale, noise=latents.float())
    frames = decode_latents(vae, lat, decode_chunk_size)
    return (frames / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4)
