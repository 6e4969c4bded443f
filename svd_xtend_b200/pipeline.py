"""Image -> video on H100 without diffusers or transformers: [D] StableVideoDiffusionPipeline.__call__ with output_type="pt"
(the validation loop of train_svd.py:1106-1140 and infer_svd.ipynb cell 3), chained from the package's own stages:

    CLIP embedding (clip.encode_image) -> noise-augmented conditioning latents (vae.encode(...).latent_dist.mode(), unscaled)
    -> Euler / CFG sampling (sampling.VideoLatentSampler) -> chunked temporal decode (sampling.decode_latents) -> frames in [0, 1]

Random draws, in this order, all from `generator` (on the generator's own device, CPU or CUDA, then moved to the image's
device, as diffusers' `randn_tensor` does): (1) the conditioning-image noise of noise_aug_strength (the image's shape), (2) the
initial video latents [B, F, 4, h, w] unless `latents` is given. The same generator state therefore reproduces a pipeline
call from the stages composed by hand.
"""
from __future__ import annotations

import os
from types import SimpleNamespace
from typing import Optional

import torch

from .clip import CLIP_MEAN, CLIP_STD, CLIPVisionModelWithProjection, encode_image, image_processor_stats
from .sampling import VideoLatentSampler, decode_latents
from .unet import UNetSpatioTemporalConditionModel
from .vae import AutoencoderKLTemporalDecoder


class ImageToVideoPipeline:
    def __init__(self, unet, vae, image_encoder, image_mean=CLIP_MEAN, image_std=CLIP_STD, use_cuda_graph: bool = True):
        if vae.decoder is None:
            raise ValueError("ImageToVideoPipeline needs the VAE decoder (AutoencoderKLTemporalDecoder(with_decoder=True))")
        self.unet, self.vae, self.image_encoder = unet, vae, image_encoder
        self.image_mean, self.image_std = tuple(image_mean), tuple(image_std)
        self.sampler = VideoLatentSampler(unet, use_cuda_graph=use_cuda_graph)

    @classmethod
    def from_pretrained(cls, path: str, variant: Optional[str] = None, torch_dtype=None, **kw):
        """loads unet/, vae/ (with the decoder), image_encoder/ and the normalisation of feature_extractor/"""
        unet = UNetSpatioTemporalConditionModel.from_pretrained(path, subfolder="unet", variant=variant, torch_dtype=torch_dtype)
        vae = AutoencoderKLTemporalDecoder.from_pretrained(path, subfolder="vae", variant=variant, torch_dtype=torch_dtype, with_decoder=True)
        enc = CLIPVisionModelWithProjection.from_pretrained(path, subfolder="image_encoder", variant=variant, torch_dtype=torch_dtype)
        fe = os.path.join(path, "feature_extractor", "preprocessor_config.json")
        mean, std = image_processor_stats(path) if os.path.exists(fe) else (CLIP_MEAN, CLIP_STD)
        for m in (unet, vae, enc):
            m.requires_grad_(False).eval()
        return cls(unet, vae, enc, image_mean=mean, image_std=std, **kw)

    def to(self, device):
        for m in (self.unet, self.vae, self.image_encoder):
            m.to(device)
        return self

    # ---- LoRA adapters of the UNet (diffusers' pipeline method names; the file format lives in svd_xtend_b200.lora)
    def load_lora_weights(self, pretrained_model_name_or_path_or_dict, adapter_name: Optional[str] = None,
                          weight_name: Optional[str] = None) -> str:
        return self.unet.load_lora_adapter(pretrained_model_name_or_path_or_dict, adapter_name=adapter_name, weight_name=weight_name)

    @staticmethod
    def save_lora_weights(save_directory: str, unet_lora_layers, weight_name: Optional[str] = None, safe_serialization: bool = True,
                          **kwargs) -> str:
        from .lora import save_lora_weights
        return save_lora_weights(save_directory, unet_lora_layers, weight_name=weight_name, safe_serialization=safe_serialization)

    def set_adapters(self, adapter_names, adapter_weights=None):
        self.unet.set_adapters(adapter_names, adapter_weights)

    def fuse_lora(self, lora_scale: float = 1.0, adapter_names=None):
        self.unet.fuse_lora(lora_scale=lora_scale, adapter_names=adapter_names)

    def unfuse_lora(self):
        self.unet.unfuse_lora()

    def unload_lora_weights(self):
        self.unet.unload_lora()

    def disable_lora(self):
        self.unet.disable_lora()

    def enable_lora(self):
        self.unet.enable_lora()

    @torch.no_grad()
    def __call__(self, image: torch.Tensor, *, num_frames: Optional[int] = None, num_inference_steps: int = 25,
                 min_guidance_scale: float = 1.0, max_guidance_scale: float = 3.0, fps: int = 7, motion_bucket_id: int = 127,
                 noise_aug_strength: float = 0.02, decode_chunk_size: Optional[int] = None, generator: Optional[torch.Generator] = None,
                 latents: Optional[torch.Tensor] = None):
        """image [B, 3, H, W] in [0, 1], already at the output size -> object with `.frames` [B, F, 3, H, W] fp32 in [0, 1]"""
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError(f"image must be [B, 3, H, W] in [0, 1], got {tuple(image.shape)}")
        F = self.unet.config.num_frames if num_frames is None else int(num_frames)
        x = image.float() * 2.0 - 1.0
        gen_dev = x.device if generator is None else generator.device      # draws happen on the generator's device, as randn_tensor [D]
        emb = encode_image(self.image_encoder, x, self.image_mean, self.image_std)
        noise = torch.randn(x.shape, generator=generator, device=gen_dev, dtype=x.dtype).to(x.device)            # draw 1
        cond = x + noise_aug_strength * noise
        image_latents = self.vae.encode(cond.to(self.vae.dtype)).latent_dist.mode()
        B, _, h, w = image_latents.shape
        if latents is None:
            latents = torch.randn(B, F, 4, h, w, generator=generator, device=gen_dev, dtype=torch.float32).to(x.device)   # draw 2
        lat = self.sampler(image_latents.float(), emb.float().unsqueeze(1), num_frames=F, fps=fps, motion_bucket_id=motion_bucket_id,
                           noise_aug_strength=noise_aug_strength, num_inference_steps=num_inference_steps,
                           min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale, noise=latents.float())
        frames = decode_latents(self.vae, lat.to(self.vae.dtype), decode_chunk_size)
        return SimpleNamespace(frames=(frames / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4).contiguous())
