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

import json
import math
import os
import shutil
from types import SimpleNamespace
from typing import Optional

import numpy as np
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
                 latents: Optional[torch.Tensor] = None, sigma_min: float = 0.002, sigma_max: float = 700.0):
        """image [B, 3, H, W] in [0, 1], already at the output size -> object with `.frames` [B, F, 3, H, W] fp32 in [0, 1].
        sigma_min / sigma_max: the range of the Karras sigmas (the scheduler config's)"""
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError(f"image must be [B, 3, H, W] in [0, 1], got {tuple(image.shape)}")
        lat = self._sample(image, image, num_frames=num_frames, num_inference_steps=num_inference_steps,
                           min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale, fps=fps,
                           motion_bucket_id=motion_bucket_id, noise_aug_strength=noise_aug_strength, generator=generator,
                           latents=latents, sigma_min=sigma_min, sigma_max=sigma_max)
        return SimpleNamespace(frames=self._decode(lat, decode_chunk_size))

    def _sample(self, clip_image: torch.Tensor, vae_image: torch.Tensor, *, num_frames, num_inference_steps, min_guidance_scale,
                max_guidance_scale, fps, motion_bucket_id, noise_aug_strength, generator, latents, sigma_min, sigma_max):
        """CLIP embedding of clip_image (any size), conditioning latents of vae_image (the output size), sampling -> the
        denoised latents [B, F, 4, h, w] fp32. Both images [B, 3, *, *] in [0, 1]."""
        F = self.unet.config.num_frames if num_frames is None else int(num_frames)
        x = vae_image.float() * 2.0 - 1.0
        gen_dev = x.device if generator is None else generator.device      # draws happen on the generator's device, as randn_tensor [D]
        emb = encode_image(self.image_encoder, x if clip_image is vae_image else clip_image.float() * 2.0 - 1.0,
                           self.image_mean, self.image_std)
        noise = torch.randn(x.shape, generator=generator, device=gen_dev, dtype=x.dtype).to(x.device)            # draw 1
        cond = x + noise_aug_strength * noise
        image_latents = self.vae.encode(cond.to(self.vae.dtype)).latent_dist.mode()
        B, _, h, w = image_latents.shape
        if latents is None:
            latents = torch.randn(B, F, 4, h, w, generator=generator, device=gen_dev, dtype=torch.float32).to(x.device)   # draw 2
        return self.sampler(image_latents.float(), emb.float().unsqueeze(1), num_frames=F, fps=fps, motion_bucket_id=motion_bucket_id,
                            noise_aug_strength=noise_aug_strength, num_inference_steps=num_inference_steps,
                            min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale, noise=latents.float(),
                            sigma_min=sigma_min, sigma_max=sigma_max)

    def _decode(self, lat: torch.Tensor, decode_chunk_size: Optional[int]) -> torch.Tensor:
        """denoised latents -> frames [B, F, 3, H, W] fp32 in [0, 1]"""
        frames = decode_latents(self.vae, lat.to(self.vae.dtype), decode_chunk_size)
        return (frames / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4).contiguous()


# [D] EulerDiscreteScheduler keys whose value the SVD configuration fixes (the sampler implements exactly that configuration:
# Karras sigmas with rho 7, v-prediction, continuous timesteps 0.25 ln sigma, init_noise_sigma sqrt(sigma_max^2 + 1), a final
# sigma of zero), and keys that do not change the sigmas or timesteps once those hold (the betas only give the sigma range
# when sigma_min / sigma_max are unset, and those two are required here).
_SCHEDULER_FIXED = dict(_class_name="EulerDiscreteScheduler", prediction_type="v_prediction", use_karras_sigmas=True,
                        timestep_type="continuous", timestep_spacing="leading", final_sigmas_type="zero",
                        use_exponential_sigmas=False, use_beta_sigmas=False, rescale_betas_zero_snr=False)
_SCHEDULER_FREE = {"_diffusers_version", "beta_start", "beta_end", "beta_schedule", "trained_betas", "num_train_timesteps",
                   "steps_offset", "interpolation_type", "clip_sample", "set_alpha_to_one", "skip_prk_steps"}


def scheduler_sigma_range(cfg: dict):
    """(sigma_min, sigma_max) of a scheduler_config.json in the SVD Euler-Karras configuration; any other class, setting or
    unknown key raises ValueError naming the key"""
    for k, v in cfg.items():
        if k in ("sigma_min", "sigma_max") or k in _SCHEDULER_FREE:
            continue
        if k not in _SCHEDULER_FIXED:
            raise ValueError(f"scheduler_config.json: unsupported key {k!r} (the sampler implements the SVD Euler-Karras configuration)")
        if v != _SCHEDULER_FIXED[k]:
            raise ValueError(f"scheduler_config.json: {k}={v!r} is not supported (the sampler implements {k}={_SCHEDULER_FIXED[k]!r})")
    if cfg.get("_class_name") != _SCHEDULER_FIXED["_class_name"]:
        raise ValueError("scheduler_config.json: _class_name must be 'EulerDiscreteScheduler'")
    for k in ("prediction_type", "use_karras_sigmas", "timestep_type"):
        if k not in cfg:
            raise ValueError(f"scheduler_config.json: {k} is missing (the sampler needs {k}={_SCHEDULER_FIXED[k]!r})")
    lo, hi = cfg.get("sigma_min"), cfg.get("sigma_max")
    for k, v in (("sigma_min", lo), ("sigma_max", hi)):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v <= 0:
            raise ValueError(f"scheduler_config.json: {k}={v!r} must be a positive finite number")
    if lo >= hi:
        raise ValueError(f"scheduler_config.json: sigma_min={lo!r} must be below sigma_max={hi!r}")
    return float(lo), float(hi)


# model_index.json: (library, class) of each component, as diffusers' loader reads them [D]
MODEL_INDEX = dict(feature_extractor=["transformers", "CLIPImageProcessor"], image_encoder=["transformers", "CLIPVisionModelWithProjection"],
                   scheduler=["diffusers", "EulerDiscreteScheduler"], unet=["diffusers", "UNetSpatioTemporalConditionModel"],
                   vae=["diffusers", "AutoencoderKLTemporalDecoder"])
OUTPUT_TYPES = ("pil", "np", "pt", "latent")


class StableVideoDiffusionPipeline(ImageToVideoPipeline):
    """[D] diffusers' StableVideoDiffusionPipeline call surface over ImageToVideoPipeline: the same stages, kernels and
    generator draws, built from the modules a training script passes (train_svd.py's validation loop and final save).
    Components passed to `from_pretrained` are used as they are: never cast, moved or frozen."""

    def __init__(self, unet, vae, image_encoder, image_mean=CLIP_MEAN, image_std=CLIP_STD, sigma_min: float = 0.002,
                 sigma_max: float = 700.0, source: Optional[str] = None, loaded=()):
        super().__init__(unet, vae, image_encoder, image_mean=image_mean, image_std=image_std)
        self.sigma_min, self.sigma_max = float(sigma_min), float(sigma_max)
        self.source = source                 # the directory scheduler/ and feature_extractor/ came from (save_pretrained copies them)
        self._loaded = tuple(loaded)         # the components this pipeline loaded itself: the only ones `to` moves

    @classmethod
    def from_pretrained(cls, path: str, unet=None, vae=None, image_encoder=None, revision: Optional[str] = None, torch_dtype=None,
                        variant: Optional[str] = None, **ignored):
        """loads from the local directory `path` only the components not passed (the VAE with its decoder), in torch_dtype;
        reads scheduler/scheduler_config.json (the SVD Euler-Karras configuration) and feature_extractor/'s normalisation"""
        if revision is not None:
            raise ValueError(f"StableVideoDiffusionPipeline.from_pretrained: revision={revision!r} is not supported (local directories only)")
        if not os.path.isdir(path):
            raise ValueError(f"StableVideoDiffusionPipeline.from_pretrained: {path!r} is not a local directory (hub downloads are not supported)")
        with open(os.path.join(path, "scheduler", "scheduler_config.json")) as f:
            sigma_min, sigma_max = scheduler_sigma_range(json.load(f))
        fe = os.path.join(path, "feature_extractor", "preprocessor_config.json")
        mean, std = image_processor_stats(path) if os.path.exists(fe) else (CLIP_MEAN, CLIP_STD)
        loaded = []
        if unet is None:
            unet = UNetSpatioTemporalConditionModel.from_pretrained(path, subfolder="unet", variant=variant, torch_dtype=torch_dtype)
            loaded.append(unet)
        if vae is None:
            vae = AutoencoderKLTemporalDecoder.from_pretrained(path, subfolder="vae", variant=variant, torch_dtype=torch_dtype, with_decoder=True)
            loaded.append(vae)
        if image_encoder is None:
            image_encoder = CLIPVisionModelWithProjection.from_pretrained(path, subfolder="image_encoder", variant=variant,
                                                                          torch_dtype=torch_dtype)
            loaded.append(image_encoder)
        for m in loaded:
            m.requires_grad_(False).eval()
        return cls(unet, vae, image_encoder, image_mean=mean, image_std=std, sigma_min=sigma_min, sigma_max=sigma_max, source=path,
                   loaded=loaded)

    def to(self, device):
        """moves the components this pipeline loaded; passed components stay where their owner keeps them"""
        for m in self._loaded:
            m.to(device)
        return self

    def set_progress_bar_config(self, **kwargs):
        """accepted for diffusers' surface; the sampler prints nothing"""

    def save_pretrained(self, save_directory: str, safe_serialization: bool = True, **kwargs):
        """diffusers' pipeline layout: model_index.json, unet/, vae/ (with the decoder), image_encoder/, and scheduler/ and
        feature_extractor/ copied from the directory the pipeline was loaded from"""
        os.makedirs(save_directory, exist_ok=True)
        version = "0.24.0"                   # the diffusers release that added SVD, unless the source directory names one
        src_index = None if self.source is None else os.path.join(self.source, "model_index.json")
        if src_index is not None and os.path.exists(src_index):
            with open(src_index) as f:
                version = json.load(f).get("_diffusers_version", version)
        index = dict(_class_name="StableVideoDiffusionPipeline", _diffusers_version=version, **MODEL_INDEX)
        with open(os.path.join(save_directory, "model_index.json"), "w") as f:
            json.dump(index, f, indent=2)
        self.unet.save_pretrained(os.path.join(save_directory, "unet"), safe_serialization=safe_serialization)
        self.vae.save_pretrained(os.path.join(save_directory, "vae"), safe_serialization=safe_serialization)
        self.image_encoder.save_pretrained(os.path.join(save_directory, "image_encoder"), safe_serialization=safe_serialization)
        if self.source is not None and os.path.abspath(self.source) != os.path.abspath(save_directory):
            for sub in ("scheduler", "feature_extractor"):
                if os.path.isdir(os.path.join(self.source, sub)):
                    shutil.copytree(os.path.join(self.source, sub), os.path.join(save_directory, sub), dirs_exist_ok=True)

    def _images(self, image, height: int, width: int):
        """(CLIP image, VAE image): [B, 3, *, *] fp32 in [0, 1] on the pipeline's device. PIL images go to CLIP as given and to
        the VAE resized on the host with Pillow's LANCZOS filter (diffusers' VideoProcessor [D]); a tensor must already be
        [B, 3, height, width]."""
        dev = self.vae.device
        if isinstance(image, torch.Tensor):
            if image.dim() != 4 or image.shape[1] != 3:
                raise ValueError(f"image tensor must be [B, 3, H, W] in [0, 1], got {tuple(image.shape)}")
            if tuple(image.shape[-2:]) != (height, width):
                raise ValueError(f"image tensor is {image.shape[-2]}x{image.shape[-1]}; a tensor input must already be at "
                                 f"height x width = {height}x{width} (PIL inputs are resized)")
            image = image.to(dev)
            return image, image
        from PIL import Image
        images = list(image) if isinstance(image, (list, tuple)) else [image]
        if not images or not all(isinstance(im, Image.Image) for im in images):
            raise ValueError("image must be a PIL image, a list of PIL images or a [B, 3, H, W] tensor")
        if any(im.mode != "RGB" for im in images) or len({im.size for im in images}) != 1:
            raise ValueError("PIL images must be RGB and all of one size")

        def to_tensor(ims):
            a = torch.from_numpy(np.stack([np.asarray(im) for im in ims]))
            return (a.permute(0, 3, 1, 2).float() / 255.0).to(dev)
        clip = to_tensor(images)
        if images[0].size == (width, height):
            return clip, clip
        return clip, to_tensor([im.resize((width, height), resample=Image.Resampling.LANCZOS) for im in images])

    @torch.no_grad()
    def __call__(self, image, height: int = 576, width: int = 1024, num_frames: Optional[int] = None, num_inference_steps: int = 25,
                 min_guidance_scale: float = 1.0, max_guidance_scale: float = 3.0, fps: int = 7, motion_bucket_id: int = 127,
                 noise_aug_strength: float = 0.02, decode_chunk_size: Optional[int] = None, num_videos_per_prompt: int = 1,
                 generator: Optional[torch.Generator] = None, latents: Optional[torch.Tensor] = None, output_type: str = "pil",
                 return_dict: bool = True, **unsupported):
        """[D] StableVideoDiffusionPipeline.__call__. `.frames[b]` is a list of F PIL images (output_type "pil"), or the
        frames as [B, F, H, W, 3] numpy ("np") / [B, F, 3, H, W] tensor ("pt") in [0, 1], or the denoised latents [B, F, 4, h, w]
        ("latent"). With return_dict=False the frames alone are returned."""
        if unsupported:
            raise ValueError(f"StableVideoDiffusionPipeline: unsupported argument(s) {sorted(unsupported)}")
        if num_videos_per_prompt != 1:
            raise ValueError(f"num_videos_per_prompt={num_videos_per_prompt} is not supported (only 1)")
        if generator is not None and not isinstance(generator, torch.Generator):
            raise ValueError("generator must be one torch.Generator (a list of generators is not supported)")
        if output_type not in OUTPUT_TYPES:
            raise ValueError(f"output_type={output_type!r} is not supported (one of {OUTPUT_TYPES})")
        if height % 8 or width % 8 or height <= 0 or width <= 0:
            raise ValueError(f"height and width must be positive multiples of 8, got {height}x{width}")
        if decode_chunk_size is not None and decode_chunk_size < 1:
            raise ValueError("decode_chunk_size must be >= 1")
        F = self.unet.config.num_frames if num_frames is None else int(num_frames)
        clip_image, vae_image = self._images(image, height, width)
        f = 1 << (len(self.vae.config.block_out_channels) - 1)
        want = (vae_image.shape[0], F, self.vae.config.latent_channels, height // f, width // f)
        if latents is not None and tuple(latents.shape) != want:
            raise ValueError(f"latents must be {list(want)}, got {list(latents.shape)}")
        lat = self._sample(clip_image, vae_image, num_frames=F, num_inference_steps=num_inference_steps,
                           min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale, fps=fps,
                           motion_bucket_id=motion_bucket_id, noise_aug_strength=noise_aug_strength, generator=generator,
                           latents=latents, sigma_min=self.sigma_min, sigma_max=self.sigma_max)
        frames = lat if output_type == "latent" else postprocess_video(self._decode(lat, decode_chunk_size), output_type)
        return SimpleNamespace(frames=frames) if return_dict else frames


def postprocess_video(frames: torch.Tensor, output_type: str):
    """[D] VideoProcessor.postprocess_video of frames [B, F, 3, H, W] in [0, 1]: "pt" as they are, "np" [B, F, H, W, 3] fp32,
    "pil" one list of F PIL images per video, uint8 = round(x * 255)"""
    if output_type == "pt":
        return frames
    arr = frames.permute(0, 1, 3, 4, 2).cpu().float().numpy()
    if output_type == "np":
        return arr
    from PIL import Image
    u8 = (arr * 255).round().astype("uint8")
    return [[Image.fromarray(f) for f in video] for video in u8]
