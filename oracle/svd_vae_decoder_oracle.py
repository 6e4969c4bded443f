"""ORACLE — test infrastructure only. Plain-PyTorch restatement of the temporal VAE DECODER the reference's inference path
reaches through diffusers' `StableVideoDiffusionPipeline.decode_latents` (train_svd.py validation, decode_chunk_size=8;
infer_svd.ipynb cell 3: 14 frames at 576x1024, decode_chunk_size=8):

    frames = vae.decode(latents / scaling_factor, num_frames=chunk).sample      (chunk by chunk)

[D] = diffusers models/autoencoders/autoencoder_kl_temporal_decoder.py (AutoencoderKLTemporalDecoder.decode),
models/autoencoders/vae.py TemporalDecoder, models/unets/unet_3d_blocks.py MidBlockTemporalDecoder / UpBlockTemporalDecoder,
models/resnet.py SpatioTemporalResBlock / TemporalResnetBlock / AlphaBlender, models/upsampling.py Upsample2D — absent from
/root/reference and restated from the published algorithm (diffusers 0.29-0.31): PARITY UNPINNED against diffusers
(tests/test_decoder_vs_diffusers.py A/Bs this file wherever diffusers is importable; SURVEY.md Appendix D lists the recalled
items). The encode path stays in oracle/svd_vae_oracle.py; `AutoencoderKLTemporalDecoder(..., with_decoder=True)` here adds
`decoder.*` and `decode`. fp32, module / parameter names follow the diffusers state dict.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from .svd_vae_oracle import AutoencoderKLTemporalDecoder as _EncodeOnly
from .svd_vae_oracle import ResnetBlock2D, VaeAttention


class TemporalResnetBlock(nn.Module):
    """[D] resnet.py TemporalResnetBlock(temb_channels=None): GroupNorm(32) statistics over (C/32, T, H, W) of each clip,
    two Conv3d (3,1,1) with padding (1,0,0), residual."""

    def __init__(self, in_channels, out_channels, eps=1e-6):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv3d(in_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))
        self.norm2 = nn.GroupNorm(32, out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))
        self.nonlinearity = nn.SiLU()

    def forward(self, x):                                   # x [B, C, T, H, W]
        h = self.conv1(self.nonlinearity(self.norm1(x)))
        h = self.conv2(self.dropout(self.nonlinearity(self.norm2(h))))
        return x + h


class AlphaBlender(nn.Module):
    """[D] resnet.py AlphaBlender(merge_strategy="learned", switch_spatial_to_temporal_mix): alpha = sigmoid(mix_factor),
    flipped to 1 - alpha when switched; out = alpha * x_spatial + (1 - alpha) * x_temporal."""

    def __init__(self, alpha, switch_spatial_to_temporal_mix=False):
        super().__init__()
        self.switch_spatial_to_temporal_mix = switch_spatial_to_temporal_mix
        self.mix_factor = nn.Parameter(torch.tensor([float(alpha)]))

    def forward(self, x_spatial, x_temporal):
        alpha = torch.sigmoid(self.mix_factor)
        if self.switch_spatial_to_temporal_mix:
            alpha = 1.0 - alpha
        return alpha * x_spatial + (1.0 - alpha) * x_temporal


class SpatioTemporalResBlock(nn.Module):
    """[D] resnet.py SpatioTemporalResBlock as the temporal decoder builds it: eps 1e-6, temporal_eps 1e-5, no temb,
    merge_factor 0.0, merge_strategy "learned", switch_spatial_to_temporal_mix=True."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.spatial_res_block = ResnetBlock2D(in_channels, out_channels, eps=1e-6)
        self.temporal_res_block = TemporalResnetBlock(out_channels, out_channels, eps=1e-5)
        self.time_mixer = AlphaBlender(0.0, switch_spatial_to_temporal_mix=True)

    def forward(self, x, num_frames):
        x = self.spatial_res_block(x)
        bf, c, h, w = x.shape
        xs = x.reshape(bf // num_frames, num_frames, c, h, w).permute(0, 2, 1, 3, 4)
        xt = self.temporal_res_block(xs)
        out = self.time_mixer(xs, xt)
        return out.permute(0, 2, 1, 3, 4).reshape(bf, c, h, w)


class MidBlockTemporalDecoder(nn.Module):
    """[D] unet_3d_blocks.py MidBlockTemporalDecoder: resnets[0], then (attention, resnet) pairs over resnets[1:] (zip)."""

    def __init__(self, channels, num_layers):
        super().__init__()
        self.attentions = nn.ModuleList([VaeAttention(channels)])
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(channels, channels) for _ in range(num_layers)])

    def forward(self, x, num_frames):
        x = self.resnets[0](x, num_frames)
        for resnet, attn in zip(self.resnets[1:], self.attentions):
            x = attn(x)
            x = resnet(x, num_frames)
        return x


class Upsample2D(nn.Module):
    """[D] upsampling.py Upsample2D(use_conv=True): nearest 2x, then a 3x3 conv with padding 1."""

    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class UpBlockTemporalDecoder(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(in_channels if i == 0 else out_channels, out_channels) for i in range(num_layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels)]) if add_upsample else None

    def forward(self, x, num_frames):
        for r in self.resnets:
            x = r(x, num_frames)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                x = u(x)
        return x


class TemporalDecoder(nn.Module):
    """[D] vae.py TemporalDecoder: conv_in -> mid -> up blocks over the reversed block_out_channels -> GroupNorm + SiLU ->
    conv_out (3x3) -> time_conv_out, a Conv3d(3, 3, (3,1,1), padding (1,0,0)) over the frames of the call."""

    def __init__(self, in_channels, out_channels, block_out_channels, layers_per_block):
        super().__init__()
        boc = list(block_out_channels)
        self.conv_in = nn.Conv2d(in_channels, boc[-1], 3, padding=1)
        self.mid_block = MidBlockTemporalDecoder(boc[-1], layers_per_block)
        rev = list(reversed(boc))
        self.up_blocks = nn.ModuleList([])
        oc = rev[0]
        for i, c in enumerate(rev):
            ic, oc = oc, c
            self.up_blocks.append(UpBlockTemporalDecoder(ic, oc, layers_per_block + 1, add_upsample=i != len(rev) - 1))
        self.conv_norm_out = nn.GroupNorm(32, boc[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(boc[0], out_channels, 3, padding=1)
        self.time_conv_out = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, z, num_frames):
        x = self.conv_in(z)
        x = self.mid_block(x, num_frames)
        for b in self.up_blocks:
            x = b(x, num_frames)
        x = self.conv_out(self.conv_act(self.conv_norm_out(x)))
        bf, c, h, w = x.shape
        x = x.reshape(bf // num_frames, num_frames, c, h, w).permute(0, 2, 1, 3, 4)
        x = self.time_conv_out(x)
        return x.permute(0, 2, 1, 3, 4).reshape(bf, c, h, w)


class AutoencoderKLTemporalDecoder(_EncodeOnly):
    """encode path of oracle/svd_vae_oracle.py plus, with with_decoder=True, `decoder.*` and [D] decode (no post_quant_conv;
    image_only_indicator is all zeros, which the "learned" AlphaBlender ignores)."""

    def __init__(self, in_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2, scaling_factor=0.18215,
                 with_decoder=False):
        super().__init__(in_channels, latent_channels, block_out_channels, layers_per_block, scaling_factor)
        self.decoder = TemporalDecoder(latent_channels, in_channels, block_out_channels, layers_per_block) if with_decoder else None

    def decode(self, z, num_frames):
        """z [B*F, latent, h, w] -> .sample [B*F, 3, 8h, 8w] (for 4 levels)"""
        return SimpleNamespace(sample=self.decoder(z, num_frames))


def decode_latents(vae, latents, decode_chunk_size=None):
    """[D] StableVideoDiffusionPipeline.decode_latents: latents [B, F, 4, h, w] -> frames [B, 3, F, H, W] fp32. Chunks of
    decode_chunk_size flattened frames (default: F) are decoded as separate clips (num_frames = chunk length)."""
    b, f = latents.shape[:2]
    chunk = f if decode_chunk_size is None else decode_chunk_size
    lat = latents.flatten(0, 1) * (1.0 / vae.config.scaling_factor)
    frames = []
    for i in range(0, lat.shape[0], chunk):
        part = lat[i:i + chunk]
        frames.append(vae.decode(part, num_frames=part.shape[0]).sample)
    frames = torch.cat(frames, dim=0)
    return frames.reshape(-1, f, *frames.shape[1:]).permute(0, 2, 1, 3, 4).float()
