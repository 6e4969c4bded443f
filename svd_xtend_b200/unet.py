"""Drop-in `UNetSpatioTemporalConditionModel` for pixeli99/SVD_Xtend on H100.

Host-side mirror of /root/reference/src/unet_spatio_temporal_condition.py (class at :32, forward
signature at :357-364, attention-processor plugin API at :248-321, gradient-checkpointing flag at
:68,:323-325, forward chunking at :328-355) and of the diffusers block classes it instantiates
(SURVEY.md Appendix B/C). The module tree exists to HOLD parameters under the reference's exact
names (so `from_pretrained` state dicts, the `'temporal_transformer_block' in name` filter of
train_svd.py:761-766 and PEFT's target matching at train_svd_lora.py:659-664 all work unchanged);
the arithmetic never goes through `nn.Module.forward` of those holders — `forward()` below drives
the sm_90a kernels through `engine.Engine` (token-major channels-last bf16, hand-rolled tape).
There is no PyTorch/CPU fallback: without the native library or a CUDA device forward raises.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import raw
from .engine import Engine, Geom, Var, bf16, F32


# ----------------------------------------------------------------------------- parameter holders
class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels: int, time_embed_dim: int, out_dim: Optional[int] = None):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, out_dim if out_dim is not None else time_embed_dim)


class SvdxAttnProcessor:
    """The attention 'processor' of this build: wgmma flash attention for self-attention and the exact
    1-key collapse for the image cross-attention. Kept as an object so that the reference's
    `attn_processors` / `set_attn_processor` API (src/unet_spatio_temporal_condition.py:248-308) round-trips."""

    def __repr__(self):
        return "SvdxAttnProcessor(sm_90a)"


# Processors whose arithmetic IS plain scaled-dot-product attention (softmax(q k^T / sqrt(d)) v followed by to_out): the
# diffusers classes the reference can install — `AttnProcessor()` by set_default_attn_processor
# (src/unet_spatio_temporal_condition.py:310-321), `AttnProcessor2_0` (the constructor default [D]) and
# `XFormersAttnProcessor` (enable_xformers_memory_efficient_attention, train_svd.py:681-693). Setting one of them keeps the
# object (the dict API round-trips) and the sm_90a kernel computes the same function. Any OTHER processor would change
# the arithmetic (the reference calls it, :276-308); it cannot run on this path, so it is rejected instead of being
# silently ignored.
_SDPA_EQUIVALENT_PROCESSORS = ("SvdxAttnProcessor", "AttnProcessor", "AttnProcessor2_0", "XFormersAttnProcessor")


def _check_processor(processor):
    name = type(processor).__name__
    if name not in _SDPA_EQUIVALENT_PROCESSORS:
        raise ValueError(
            f"svd_xtend_b200: attention processor {name!r} is not supported — the H100 path computes plain scaled-dot-product "
            f"attention in one fused kernel and cannot call a custom processor; accepted (arithmetically identical): "
            f"{', '.join(_SDPA_EQUIVALENT_PROCESSORS)}")
    return processor


class Attention(nn.Module):
    def __init__(self, query_dim: int, cross_attention_dim: Optional[int] = None, heads: int = 8, dim_head: int = 64):
        super().__init__()
        if dim_head != 64:
            raise ValueError("svd_xtend_b200 attention kernels are specialised for head_dim 64 (the SVD UNet value)")
        self.inner_dim = dim_head * heads
        self.heads = heads
        self.scale = dim_head ** -0.5
        kv_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.to_q = nn.Linear(query_dim, self.inner_dim, bias=False)
        self.to_k = nn.Linear(kv_dim, self.inner_dim, bias=False)
        self.to_v = nn.Linear(kv_dim, self.inner_dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(self.inner_dim, query_dim, bias=True), nn.Dropout(0.0)])
        self.processor = SvdxAttnProcessor()

    def get_processor(self):
        return self.processor

    def set_processor(self, processor):
        self.processor = _check_processor(processor)


class GEGLU(nn.Module):
    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    def __init__(self, dim: int, dim_out: Optional[int] = None, mult: int = 4):
        super().__init__()
        inner_dim = int(dim * mult)
        self.net = nn.ModuleList([GEGLU(dim, inner_dim), nn.Dropout(0.0), nn.Linear(inner_dim, dim_out if dim_out is not None else dim)])


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, head_dim, cross_attention_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-5)
        self.attn1 = Attention(dim, None, heads, head_dim)
        self.norm2 = nn.LayerNorm(dim, eps=1e-5)
        self.attn2 = Attention(dim, cross_attention_dim, heads, head_dim)
        self.norm3 = nn.LayerNorm(dim, eps=1e-5)
        self.ff = FeedForward(dim)
        self._chunk_size, self._chunk_dim = None, 0

    def set_chunk_feed_forward(self, chunk_size, dim=0):
        # feed-forward chunking is a memory optimisation of the reference; the fused GEGLU GEMM makes it moot
        self._chunk_size, self._chunk_dim = chunk_size, dim


class TemporalBasicTransformerBlock(nn.Module):
    def __init__(self, dim, time_mix_inner_dim, heads, head_dim, cross_attention_dim):
        super().__init__()
        if dim != time_mix_inner_dim:
            raise ValueError("only dim == time_mix_inner_dim (the SVD topology) is supported")
        self.is_res = True
        self.norm_in = nn.LayerNorm(dim)
        self.ff_in = FeedForward(dim, dim_out=time_mix_inner_dim)
        self.norm1 = nn.LayerNorm(time_mix_inner_dim)
        self.attn1 = Attention(time_mix_inner_dim, None, heads, head_dim)
        self.norm2 = nn.LayerNorm(time_mix_inner_dim)
        self.attn2 = Attention(time_mix_inner_dim, cross_attention_dim, heads, head_dim)
        self.norm3 = nn.LayerNorm(time_mix_inner_dim)
        self.ff = FeedForward(time_mix_inner_dim)
        self._chunk_size, self._chunk_dim = None, 0

    def set_chunk_feed_forward(self, chunk_size, dim=0):
        self._chunk_size, self._chunk_dim = chunk_size, dim


class AlphaBlender(nn.Module):
    def __init__(self, alpha: float):
        super().__init__()
        self.register_parameter("mix_factor", nn.Parameter(torch.tensor([float(alpha)])))


class ResnetBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, temb_channels, eps):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, stride=1, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(32, out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, stride=1, padding=1)
        self.nonlinearity = nn.SiLU()
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None


class TemporalResnetBlock(nn.Module):
    def __init__(self, in_channels, out_channels, temb_channels, eps):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv3d(in_channels, out_channels, (3, 1, 1), stride=1, padding=(1, 0, 0))
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(32, out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv3d(out_channels, out_channels, (3, 1, 1), stride=1, padding=(1, 0, 0))
        self.nonlinearity = nn.SiLU()


class SpatioTemporalResBlock(nn.Module):
    def __init__(self, in_channels, out_channels, temb_channels, eps):
        super().__init__()
        self.spatial_res_block = ResnetBlock2D(in_channels, out_channels, temb_channels, eps)
        self.temporal_res_block = TemporalResnetBlock(out_channels, out_channels, temb_channels, eps)
        self.time_mixer = AlphaBlender(0.5)


class Downsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=1)


class Upsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)


class TransformerSpatioTemporalModel(nn.Module):
    def __init__(self, heads, head_dim, in_channels, num_layers=1, cross_attention_dim=None):
        super().__init__()
        if num_layers != 1:
            raise ValueError("svd_xtend_b200 supports transformer_layers_per_block == 1 (the SVD topology)")
        inner = heads * head_dim
        self.heads = heads
        self.in_channels = in_channels
        self.norm = nn.GroupNorm(32, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, head_dim, cross_attention_dim)])
        self.temporal_transformer_blocks = nn.ModuleList([TemporalBasicTransformerBlock(inner, inner, heads, head_dim, cross_attention_dim)])
        self.time_pos_embed = TimestepEmbedding(in_channels, in_channels * 4, out_dim=in_channels)
        self.time_mixer = AlphaBlender(0.5)
        self.proj_out = nn.Linear(inner, in_channels)
        self.gradient_checkpointing = False


class DownBlockSpatioTemporal(nn.Module):
    has_cross_attention = False

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, add_downsample=True):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(in_channels if i == 0 else out_channels, out_channels, temb_channels, 1e-5)
                                      for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels)]) if add_downsample else None
        self.gradient_checkpointing = False


class CrossAttnDownBlockSpatioTemporal(nn.Module):
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, transformer_layers_per_block=1,
                 num_attention_heads=1, cross_attention_dim=1280, add_downsample=True):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(in_channels if i == 0 else out_channels, out_channels, temb_channels, 1e-6)
                                      for i in range(num_layers)])
        self.attentions = nn.ModuleList([TransformerSpatioTemporalModel(num_attention_heads, out_channels // num_attention_heads,
                                                                        out_channels, transformer_layers_per_block, cross_attention_dim)
                                         for _ in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels)]) if add_downsample else None
        self.gradient_checkpointing = False


class UNetMidBlockSpatioTemporal(nn.Module):
    has_cross_attention = True

    def __init__(self, in_channels, temb_channels, num_layers=1, transformer_layers_per_block=1, num_attention_heads=1,
                 cross_attention_dim=1280):
        super().__init__()
        resnets = [SpatioTemporalResBlock(in_channels, in_channels, temb_channels, 1e-5)]
        attentions = []
        for _ in range(num_layers):
            attentions.append(TransformerSpatioTemporalModel(num_attention_heads, in_channels // num_attention_heads, in_channels,
                                                             transformer_layers_per_block, cross_attention_dim))
            resnets.append(SpatioTemporalResBlock(in_channels, in_channels, temb_channels, 1e-5))
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)
        self.gradient_checkpointing = False


class UpBlockSpatioTemporal(nn.Module):
    has_cross_attention = False

    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, num_layers=1, add_upsample=True):
        super().__init__()
        resnets = []
        for i in range(num_layers):
            res_skip = in_channels if i == num_layers - 1 else out_channels
            res_in = prev_output_channel if i == 0 else out_channels
            resnets.append(SpatioTemporalResBlock(res_in + res_skip, out_channels, temb_channels, 1e-6))
        self.resnets = nn.ModuleList(resnets)
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels)]) if add_upsample else None
        self.gradient_checkpointing = False


class CrossAttnUpBlockSpatioTemporal(nn.Module):
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, prev_output_channel, temb_channels, num_layers=1,
                 transformer_layers_per_block=1, num_attention_heads=1, cross_attention_dim=1280, add_upsample=True):
        super().__init__()
        resnets, attentions = [], []
        for i in range(num_layers):
            res_skip = in_channels if i == num_layers - 1 else out_channels
            res_in = prev_output_channel if i == 0 else out_channels
            resnets.append(SpatioTemporalResBlock(res_in + res_skip, out_channels, temb_channels, 1e-6))
            attentions.append(TransformerSpatioTemporalModel(num_attention_heads, out_channels // num_attention_heads, out_channels,
                                                             transformer_layers_per_block, cross_attention_dim))
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels)]) if add_upsample else None
        self.gradient_checkpointing = False


@dataclass
class UNetSpatioTemporalConditionOutput:
    """src/unet_spatio_temporal_condition.py:19-29"""
    sample: torch.Tensor = None

    def __getitem__(self, i):
        return (self.sample,)[i]


class LoraLinear(nn.Module):
    """PEFT-compatible LoRA wrapper layout (base_layer + lora_A/lora_B ModuleDicts keyed by adapter name), so that
    parameter names match what `unet.add_adapter(LoraConfig)` of train_svd_lora.py:659-671 produces:
    `<linear>.base_layer.weight`, `<linear>.lora_A.default.weight` [r,in], `<linear>.lora_B.default.weight` [out,r].
    Per adapter, under PEFT's names: `r`, `lora_alpha`, `scaling` (= lora_alpha / r), the user weight of `set_adapters`
    (`adapter_weights`, default 1.0), and whether it is merged into the base weight (`merged_adapters`, with the fp32 scale it
    was merged with in `merged_scales`, so that an unmerge subtracts the same term)."""

    def __init__(self, base: nn.Linear, r: int, lora_alpha: float, adapter_name: str = "default", init: str = "gaussian"):
        super().__init__()
        self.base_layer = base
        self.in_features, self.out_features = base.in_features, base.out_features
        self.lora_A = nn.ModuleDict()
        self.lora_B = nn.ModuleDict()
        self.r, self.lora_alpha, self.scaling, self.adapter_weights = {}, {}, {}, {}
        self.active_adapters: List[str] = []
        self.merged_adapters: List[str] = []
        self.merged_scales: Dict[str, float] = {}
        self.disable_adapters = False
        self.add(adapter_name, r, lora_alpha, init)

    def add(self, adapter_name: str, r: int, lora_alpha: float, init: str = "gaussian"):
        A = nn.Linear(self.in_features, r, bias=False)
        B = nn.Linear(r, self.out_features, bias=False)
        with torch.no_grad():
            if init == "gaussian":
                nn.init.normal_(A.weight, std=1.0 / r)
            else:
                nn.init.kaiming_uniform_(A.weight, a=math.sqrt(5))
            nn.init.zeros_(B.weight)
        dev, dt = self.base_layer.weight.device, self.base_layer.weight.dtype
        self.lora_A[adapter_name] = A.to(device=dev, dtype=dt)
        self.lora_B[adapter_name] = B.to(device=dev, dtype=dt)
        self.r[adapter_name], self.lora_alpha[adapter_name] = r, lora_alpha
        self.scaling[adapter_name] = lora_alpha / r
        self.adapter_weights[adapter_name] = 1.0

    def remove(self, adapter_name: str):
        for d in (self.lora_A, self.lora_B):
            del d[adapter_name]
        for d in (self.r, self.lora_alpha, self.scaling, self.adapter_weights):
            d.pop(adapter_name)
        self.active_adapters = [n for n in self.active_adapters if n != adapter_name]

    @property
    def merged(self) -> bool:
        return bool(self.merged_adapters)

    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias


def _lora_of(lin: nn.Module, off: int = 0) -> list:
    """[(col_offset, out_features, A, B, scaling * weight)] of a LoRA-wrapped linear (ours or PEFT's): one term per active,
    unmerged adapter; none when the layer is plain or its adapters are disabled."""
    if not hasattr(lin, "lora_A") or not hasattr(lin, "base_layer") or getattr(lin, "disable_adapters", False):
        return []
    merged = set(getattr(lin, "merged_adapters", ()))
    weights = getattr(lin, "adapter_weights", {})
    return [(off, lin.lora_B[n].weight.shape[0], lin.lora_A[n].weight, lin.lora_B[n].weight, float(lin.scaling[n]) * weights.get(n, 1.0))
            for n in getattr(lin, "active_adapters", list(lin.lora_A.keys())) if n in lin.lora_A and n not in merged]


def _sinusoid(t: torch.Tensor, dim: int) -> torch.Tensor:
    """Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0) [D: embeddings.py]; fp32, tiny."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F32, device=t.device) / half)
    e = t[:, None].float() * freqs[None, :]
    return torch.cat([torch.cos(e), torch.sin(e)], dim=-1)


_DEFAULT_CONFIG = dict(
    sample_size=None, in_channels=8, out_channels=4,
    down_block_types=("CrossAttnDownBlockSpatioTemporal",) * 3 + ("DownBlockSpatioTemporal",),
    up_block_types=("UpBlockSpatioTemporal",) + ("CrossAttnUpBlockSpatioTemporal",) * 3,
    block_out_channels=(320, 640, 1280, 1280), addition_time_embed_dim=256,
    projection_class_embeddings_input_dim=768, layers_per_block=2, cross_attention_dim=1024,
    transformer_layers_per_block=1, num_attention_heads=(5, 10, 20, 20), num_frames=25,
)


class _Config(SimpleNamespace):
    def __getitem__(self, k):
        return getattr(self, k)

    def get(self, k, default=None):
        return getattr(self, k, default)

    def to_dict(self):
        return {k: (list(v) if isinstance(v, tuple) else v) for k, v in vars(self).items()}


class UNetSpatioTemporalConditionModel(nn.Module):
    """H100-native replacement with the constructor, attributes and forward of
    src/unet_spatio_temporal_condition.py:32-490."""

    _supports_gradient_checkpointing = True  # :68
    config_name = "config.json"

    def __init__(self, sample_size=None, in_channels=8, out_channels=4,
                 down_block_types=_DEFAULT_CONFIG["down_block_types"], up_block_types=_DEFAULT_CONFIG["up_block_types"],
                 block_out_channels=(320, 640, 1280, 1280), addition_time_embed_dim=256,
                 projection_class_embeddings_input_dim=768, layers_per_block=2, cross_attention_dim=1024,
                 transformer_layers_per_block=1, num_attention_heads=(5, 10, 20, 20), num_frames=25):
        super().__init__()
        self.config = _Config(sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
                              down_block_types=tuple(down_block_types), up_block_types=tuple(up_block_types),
                              block_out_channels=tuple(block_out_channels), addition_time_embed_dim=addition_time_embed_dim,
                              projection_class_embeddings_input_dim=projection_class_embeddings_input_dim,
                              layers_per_block=layers_per_block, cross_attention_dim=cross_attention_dim,
                              transformer_layers_per_block=transformer_layers_per_block,
                              num_attention_heads=num_attention_heads, num_frames=num_frames)
        self.sample_size = sample_size
        # input checks, same messages' intent as :102-125
        if len(down_block_types) != len(up_block_types):
            raise ValueError(f"Must provide the same number of `down_block_types` as `up_block_types`. `down_block_types`: {down_block_types}. `up_block_types`: {up_block_types}.")
        if len(block_out_channels) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. `block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        if not isinstance(num_attention_heads, int) and len(num_attention_heads) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `num_attention_heads` as `down_block_types`. `num_attention_heads`: {num_attention_heads}. `down_block_types`: {down_block_types}.")
        if isinstance(cross_attention_dim, list) and len(cross_attention_dim) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `cross_attention_dim` as `down_block_types`. `cross_attention_dim`: {cross_attention_dim}. `down_block_types`: {down_block_types}.")
        if not isinstance(layers_per_block, int) and len(layers_per_block) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `layers_per_block` as `down_block_types`. `layers_per_block`: {layers_per_block}. `down_block_types`: {down_block_types}.")

        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], kernel_size=3, padding=1)
        time_embed_dim = block_out_channels[0] * 4
        self.time_embedding = TimestepEmbedding(block_out_channels[0], time_embed_dim)
        self.add_embedding = TimestepEmbedding(projection_class_embeddings_input_dim, time_embed_dim)

        n = len(down_block_types)
        if isinstance(num_attention_heads, int):
            num_attention_heads = (num_attention_heads,) * n
        if isinstance(cross_attention_dim, int):
            cross_attention_dim = (cross_attention_dim,) * n
        if isinstance(layers_per_block, int):
            layers_per_block = [layers_per_block] * n
        if isinstance(transformer_layers_per_block, int):
            transformer_layers_per_block = [transformer_layers_per_block] * n

        self.down_blocks = nn.ModuleList([])
        self.up_blocks = nn.ModuleList([])
        output_channel = block_out_channels[0]
        for i, t in enumerate(down_block_types):
            input_channel, output_channel = output_channel, block_out_channels[i]
            is_final = i == n - 1
            if t == "DownBlockSpatioTemporal":
                blk = DownBlockSpatioTemporal(input_channel, output_channel, time_embed_dim, layers_per_block[i], not is_final)
            elif t == "CrossAttnDownBlockSpatioTemporal":
                blk = CrossAttnDownBlockSpatioTemporal(input_channel, output_channel, time_embed_dim, layers_per_block[i],
                                                       transformer_layers_per_block[i], num_attention_heads[i],
                                                       cross_attention_dim[i], not is_final)
            else:
                raise ValueError(f"{t} does not exist.")
            self.down_blocks.append(blk)

        self.mid_block = UNetMidBlockSpatioTemporal(block_out_channels[-1], time_embed_dim, 1, transformer_layers_per_block[-1],
                                                    num_attention_heads[-1], cross_attention_dim[-1])

        self.num_upsamplers = 0
        rev_ch = list(reversed(block_out_channels))
        rev_heads = list(reversed(num_attention_heads))
        rev_layers = list(reversed(layers_per_block))
        rev_xdim = list(reversed(cross_attention_dim))
        rev_tl = list(reversed(transformer_layers_per_block))
        output_channel = rev_ch[0]
        for i, t in enumerate(up_block_types):
            is_final = i == n - 1
            prev_output_channel, output_channel = output_channel, rev_ch[i]
            input_channel = rev_ch[min(i + 1, n - 1)]
            add_up = not is_final
            self.num_upsamplers += int(add_up)
            if t == "UpBlockSpatioTemporal":
                blk = UpBlockSpatioTemporal(input_channel, prev_output_channel, output_channel, time_embed_dim, rev_layers[i] + 1, add_up)
            elif t == "CrossAttnUpBlockSpatioTemporal":
                blk = CrossAttnUpBlockSpatioTemporal(input_channel, output_channel, prev_output_channel, time_embed_dim,
                                                     rev_layers[i] + 1, rev_tl[i], rev_heads[i], rev_xdim[i], add_up)
            else:
                raise ValueError(f"{t} does not exist.")
            self.up_blocks.append(blk)

        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[0], num_groups=32, eps=1e-5)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, kernel_size=3, padding=1)

        self._engine = Engine()
        self._resblocks: List[SpatioTemporalResBlock] = [m for m in self.modules() if isinstance(m, SpatioTemporalResBlock)]
        self.grad_hook = None   # callable(list_of_params) invoked as soon as parameter gradients are final (DDP overlap)
        self._arena = None
        self._graphs = None     # autograph.GraphRunner: shape-keyed CUDA graphs of this module's forward / backward
        self.peft_config: Dict[str, object] = {}     # adapter name -> the config object add_adapter was given (PEFT's attribute)
        self.lora_stamp = 0     # moves on every change of adapter state: captured graphs keyed on it are re-captured
        self._active_adapters: List[str] = []
        self._fuse_calls: List[list] = []    # per fuse_lora call: (LoraLinear, [(name, -scale)]), what unfuse_lora subtracts

    # ------------------------------------------------------------------ training plumbing (svd_xtend_b200.train)
    def attach_arena(self, arena):
        """Accumulate parameter gradients directly into `arena.grad` views (see train.ParamArena)."""
        self._arena = arena
        self._engine.grad_views = arena.grad_views if arena is not None else {}
        self._engine.arena = arena
        self._engine.wc.clear()

    def enable_cuda_graphs(self, warmup: int = 2):
        """Serve `forward` / `backward` of the unchanged training script from shape-keyed CUDA graphs (svd_xtend_b200.autograph):
        after `warmup` eager calls per input signature the ~2 200 launches of a step become two graph launches. Needs fp32
        trainable parameters (they are re-homed into a flat arena). Call after `requires_grad_` / `add_adapter` set-up."""
        from . import autograph
        return autograph.enable(self, warmup)

    def disable_cuda_graphs(self):
        self._graphs = None

    def refresh_trainable_operands(self, shadow_current: bool = False):
        """Re-prepare the bf16 operand layouts of all trainable parameters (after an optimizer / out-of-band update).
        With a ParamArena the plain operands are views of its bf16 shadow (kept current by FusedAdamW) and all
        transposed (dgrad) operands are refreshed by ONE svdx_multi_transpose launch."""
        if self._arena is not None:
            if not shadow_current:          # the updater did not maintain the bf16 shadow (e.g. torch.optim.AdamW)
                self._arena.refresh_shadow()
            self._arena.refresh_transposes()
            self._arena.mark_synced()
        self._engine.wc.refresh_trainable()

    @property
    def kernel_launches(self) -> int:
        return raw.LAUNCHES[0]

    # ------------------------------------------------------------------ reference helper API
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def attn_processors(self) -> Dict[str, object]:
        """src/unet_spatio_temporal_condition.py:248-274"""
        procs = {}

        def rec(name, module):
            if hasattr(module, "get_processor"):
                procs[f"{name}.processor"] = module.get_processor()
            for sub, child in module.named_children():
                rec(f"{name}.{sub}", child)

        for name, module in self.named_children():
            rec(name, module)
        return procs

    def set_attn_processor(self, processor):
        """src/unet_spatio_temporal_condition.py:276-308"""
        count = len(self.attn_processors.keys())
        if isinstance(processor, dict) and len(processor) != count:
            raise ValueError(
                f"A dict of processors was passed, but the number of processors {len(processor)} does not match the"
                f" number of attention layers: {count}. Please make sure to pass {count} processor classes.")

        def rec(name, module, processor):
            if hasattr(module, "set_processor"):
                if not isinstance(processor, dict):
                    module.set_processor(processor)
                else:
                    module.set_processor(processor.pop(f"{name}.processor"))
            for sub, child in module.named_children():
                rec(f"{name}.{sub}", child, processor)

        for name, module in self.named_children():
            rec(name, module, processor)

    def set_default_attn_processor(self):
        """:310-321 — the default processor of this build is the sm_90a one."""
        self.set_attn_processor(SvdxAttnProcessor())

    def _set_gradient_checkpointing(self, module, value=False):
        if hasattr(module, "gradient_checkpointing"):
            module.gradient_checkpointing = value

    def enable_gradient_checkpointing(self):
        self.apply(lambda m: self._set_gradient_checkpointing(m, True))

    def disable_gradient_checkpointing(self):
        self.apply(lambda m: self._set_gradient_checkpointing(m, False))

    @property
    def is_gradient_checkpointing(self):
        return any(getattr(m, "gradient_checkpointing", False) for m in self.modules())

    def enable_xformers_memory_efficient_attention(self, *a, **k):
        """train_svd.py:681-693 calls this behind a flag; attention here is already a fused flash kernel."""
        return None

    def enable_forward_chunking(self, chunk_size: Optional[int] = None, dim: int = 0) -> None:
        """src/unet_spatio_temporal_condition.py:328-355"""
        if dim not in [0, 1]:
            raise ValueError(f"Make sure to set `dim` to either 0 or 1, not {dim}")
        chunk_size = chunk_size or 1
        for m in self.modules():
            if hasattr(m, "set_chunk_feed_forward"):
                m.set_chunk_feed_forward(chunk_size=chunk_size, dim=dim)

    def add_adapter(self, adapter_config, adapter_name: str = "default"):
        """LoRA injection with the surface of diffusers' PeftAdapterMixin.add_adapter (train_svd_lora.py:671): wraps
        every nn.Linear whose name ends with one of `target_modules` (to_k, to_q, to_v, to_out.0 at :659-664), or adds the
        adapter to such a layer that is already wrapped, freezes the base model and leaves only the new adapter's lora_A /
        lora_B trainable. The config object is kept as `peft_config[adapter_name]`; the new adapter becomes the active one."""
        self._check_new_adapter_name(adapter_name)
        targets = list(getattr(adapter_config, "target_modules"))
        r = int(getattr(adapter_config, "r"))
        alpha = float(getattr(adapter_config, "lora_alpha", r))
        init = getattr(adapter_config, "init_lora_weights", True)
        init = "gaussian" if init == "gaussian" else "kaiming"
        slots = [(full, parent, child_name, child) for full, parent, child_name, child in self._linear_slots()
                 if any(full == t or full.endswith("." + t) for t in targets)]
        if not slots:
            raise ValueError(f"add_adapter: no module matched target_modules={targets}")
        adaptable = self._adaptable()
        refused = [full for full, _, _, _ in slots if full not in adaptable]
        if refused:
            raise ValueError(f"add_adapter: target_modules={targets} match linears without a LoRA side path on this build "
                             f"(only the attention projections to_q / to_k / to_v / to_out.0 take one): {refused[:8]}")
        matched = [(parent, child_name, child) for _, parent, child_name, child in slots]
        self.requires_grad_(False)
        self._inject(adapter_name, [(parent, child_name, child, r, alpha, init) for parent, child_name, child in matched])
        self.peft_config[adapter_name] = adapter_config
        return len(matched)

    # ------------------------------------------------------------------ LoRA adapters (diffusers' adapter API)
    def _linear_slots(self):
        """(full name, parent, attribute, module) of every nn.Linear or LoraLinear of the model (not the linears inside a
        LoraLinear)"""
        inside = tuple(n + "." for n, m in self.named_modules() if isinstance(m, LoraLinear))
        out = []
        for parent_name, parent in list(self.named_modules()):
            if isinstance(parent, LoraLinear) or (inside and (parent_name + ".").startswith(inside)):
                continue
            for child_name, child in list(parent.named_children()):
                if isinstance(child, (nn.Linear, LoraLinear)):
                    out.append((f"{parent_name}.{child_name}" if parent_name else child_name, parent, child_name, child))
        return out

    def _adaptable(self) -> set:
        """full names of the linears that take a LoRA side path in forward and backward (`_lora_of` call sites): the
        attention projections. attn2.to_q / to_k are among them: their output never reaches the result (one key), in the
        reference as here, so an adapter on them changes nothing either way."""
        out = set()
        for name, m in self.named_modules():
            if isinstance(m, Attention):
                out.update(f"{name}.{p}" for p in ("to_q", "to_k", "to_v", "to_out.0"))
        return out

    def _lora_layers(self) -> List[LoraLinear]:
        return [m for m in self.modules() if isinstance(m, LoraLinear)]

    def _check_new_adapter_name(self, adapter_name: str):
        if not isinstance(adapter_name, str) or not adapter_name or "." in adapter_name:
            raise ValueError(f"adapter name must be a non-empty string without '.', got {adapter_name!r}")
        if adapter_name in self.peft_config:
            raise ValueError(f"adapter {adapter_name!r} already exists; delete_adapters it first or choose another name")

    def _inject(self, adapter_name: str, slots):
        """slots: (parent, attribute, nn.Linear or LoraLinear, r, lora_alpha, init). Adds the adapter to every slot and makes
        it the only active adapter."""
        for parent, child_name, child, r, alpha, init in slots:
            if isinstance(child, LoraLinear):
                child.add(adapter_name, r, alpha, init)
            else:
                setattr(parent, child_name, LoraLinear(child, r, alpha, adapter_name, init))
        self._engine.wc.clear()
        self._set_active([adapter_name])

    def _set_active(self, names: List[str], weights: Optional[List[float]] = None):
        for layer in self._lora_layers():
            layer.active_adapters = [n for n in names if n in layer.lora_A]
            if weights is not None:
                for n, w in zip(names, weights):
                    if n in layer.adapter_weights:
                        layer.adapter_weights[n] = float(w)
        self._active_adapters = list(names)
        self.lora_stamp += 1

    def _check_known(self, names, what: str):
        unknown = [n for n in names if n not in self.peft_config]
        if unknown:
            raise ValueError(f"{what}: unknown adapter(s) {unknown}; present: {list(self.peft_config)}")

    def _check_not_fused(self, names, what: str):
        fused = sorted({n for layer in self._lora_layers() for n in layer.merged_adapters if n in names})
        if fused:
            raise ValueError(f"{what}: adapter(s) {fused} are fused into the base weights; unfuse_lora() first")

    def active_adapters(self) -> List[str]:
        """names of the active adapters (empty when there are none)"""
        return [n for n in getattr(self, "_active_adapters", []) if n in self.peft_config]

    def set_adapters(self, adapter_names, weights=None):
        """make `adapter_names` (a name or a list) the active adapters, each with its weight (a number for all, a list, or
        None for 1.0): the layer output is W x + sum over active adapters of weight * scaling * B A x"""
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        if weights is None:
            weights = [1.0] * len(names)
        elif not isinstance(weights, (list, tuple)):
            weights = [weights] * len(names)
        if len(weights) != len(names):
            raise ValueError(f"set_adapters: {len(names)} adapter names but {len(weights)} weights")
        self._check_known(names, "set_adapters")
        self._check_not_fused(names, "set_adapters")
        self._set_active(names, [float(w) for w in weights])

    def disable_lora(self):
        """run the base model alone (adapters already fused stay in the base weights)"""
        for layer in self._lora_layers():
            layer.disable_adapters = True
        self.lora_stamp += 1

    def enable_lora(self):
        for layer in self._lora_layers():
            layer.disable_adapters = False
        self.lora_stamp += 1

    def delete_adapters(self, adapter_names):
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        self._check_known(names, "delete_adapters")
        self._check_not_fused(names, "delete_adapters")
        for layer in self._lora_layers():
            for n in names:
                if n in layer.lora_A:
                    layer.remove(n)
        for n in names:
            self.peft_config.pop(n)
        self._engine.wc.clear()
        self._set_active([n for n in self.active_adapters() if n not in names])

    def unload_lora(self):
        """remove every LoRA wrapper and put the plain nn.Linear back; adapters fused into the base weights stay there"""
        for _, parent, child_name, child in self._linear_slots():
            if isinstance(child, LoraLinear):
                setattr(parent, child_name, child.base_layer)
        self.peft_config.clear()
        self._fuse_calls = []
        self._engine.wc.clear()
        self._set_active([])

    def _merge(self, items, what: str):
        """items: (LoraLinear, [(adapter name, fp32-rounded scale)]) -> one svdx_lora_merge launch over their base weights"""
        from . import lora
        for layer, _ in items:
            w = layer.base_layer.weight
            if not w.is_cuda:
                raise RuntimeError(f"svd_xtend_b200: {what} runs on the CUDA kernels only; there is no CPU fallback (move the UNet to the GPU)")
            if w.requires_grad:
                raise ValueError(f"{what}: a base weight is trainable; fusing into a trainable base is not supported")
        lora.merge_into_base([(layer.base_layer.weight, [(layer.lora_A[n].weight, layer.lora_B[n].weight, s) for n, s in terms])
                              for layer, terms in items])
        torch.autograd.graph.increment_version([layer.base_layer.weight for layer, _ in items])
        self.lora_stamp += 1

    def fuse_lora(self, lora_scale: float = 1.0, adapter_names=None):
        """merge the active (or named) adapters into the base weights in place, in one kernel launch: each layer then holds
        W + lora_scale * weight * scaling * B A, so state_dict / save_pretrained see the merged weights. Adapters already
        fused are skipped."""
        names = self.active_adapters() if adapter_names is None else \
            ([adapter_names] if isinstance(adapter_names, str) else list(adapter_names))
        self._check_known(names, "fuse_lora")
        items = []
        for layer in self._lora_layers():
            terms = [(n, float(torch.tensor(float(lora_scale) * layer.adapter_weights[n] * layer.scaling[n], dtype=F32)))
                     for n in names if n in layer.lora_A and n not in layer.merged_adapters]
            if terms:
                items.append((layer, terms))
        if not items:
            return
        self._merge(items, "fuse_lora")
        for layer, terms in items:
            for n, s in terms:
                layer.merged_adapters.append(n)
                layer.merged_scales[n] = s
        self._fuse_calls.append([(layer, [(n, -s) for n, s in terms]) for layer, terms in items])

    def unfuse_lora(self):
        """subtract every fused adapter from the base weights again, undoing the fuse_lora calls last first, one launch each:
        each call's terms are subtracted with exactly the negated sum that call added, so every call leaves at most one ulp of
        the base dtype behind (at the larger of the weight's magnitudes before and after that fuse)"""
        calls, self._fuse_calls = self._fuse_calls, []
        for items in reversed(calls):
            self._merge(items, "unfuse_lora")
        for layer in self._lora_layers():
            layer.merged_adapters, layer.merged_scales = [], {}

    def load_lora_adapter(self, pretrained_model_name_or_path_or_dict, adapter_name: Optional[str] = None,
                          weight_name: Optional[str] = None):
        """load a LoRA file written by save_lora_weights (or a directory holding one, or its state dict) as a new adapter
        (svd_xtend_b200.lora.load_into); it becomes the active adapter. Returns the adapter name."""
        from . import lora
        return lora.load_into(self, pretrained_model_name_or_path_or_dict, adapter_name, weight_name)

    def register_to_config(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self.config, k, v)

    # ------------------------------------------------------------------ (de)serialisation (diffusers layout)
    def save_pretrained(self, save_directory: str, safe_serialization: bool = True, **kwargs):
        os.makedirs(save_directory, exist_ok=True)
        cfg = self.config.to_dict()
        cfg["_class_name"] = "UNetSpatioTemporalConditionModel"
        with open(os.path.join(save_directory, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2)
        sd = {k: v.detach().cpu().contiguous() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, "diffusion_pytorch_model.safetensors"))
        else:
            torch.save(sd, os.path.join(save_directory, "diffusion_pytorch_model.bin"))

    @classmethod
    def from_config(cls, config):
        cfg = dict(config.to_dict() if hasattr(config, "to_dict") else config)
        cfg = {k: v for k, v in cfg.items() if k in _DEFAULT_CONFIG}
        return cls(**cfg)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, subfolder: Optional[str] = None, torch_dtype=None,
                        variant: Optional[str] = None, low_cpu_mem_usage: bool = True, **kwargs):
        """Local-directory loader with the keyword surface train_svd.py:651-656 uses."""
        d = pretrained_model_name_or_path if subfolder is None else os.path.join(pretrained_model_name_or_path, subfolder)
        with open(os.path.join(d, cls.config_name)) as f:
            cfg = json.load(f)
        model = cls.from_config(cfg)
        stems = ["diffusion_pytorch_model"] if variant is None else [f"diffusion_pytorch_model.{variant}", "diffusion_pytorch_model"]
        sd = None
        for stem in stems:
            p = os.path.join(d, stem + ".safetensors")
            if os.path.exists(p):
                from safetensors.torch import load_file
                sd = load_file(p)
                break
            p = os.path.join(d, stem + ".bin")
            if os.path.exists(p):
                sd = torch.load(p, map_location="cpu")
                break
        if sd is None:
            raise FileNotFoundError(f"no diffusion_pytorch_model weights under {d}")
        sd = {k: v.to(torch.float32) if torch_dtype is None else v.to(torch_dtype) for k, v in sd.items()}
        model.load_state_dict(sd, strict=True)
        if torch_dtype is not None:
            model.to(torch_dtype)
        return model

    # ------------------------------------------------------------------ forward
    def forward(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int], encoder_hidden_states: torch.Tensor,
                added_time_ids: torch.Tensor, return_dict: bool = True):
        """Same contract as src/unet_spatio_temporal_condition.py:357-490."""
        self._check_latent_size(sample)
        if not sample.is_cuda:
            raise RuntimeError("svd_xtend_b200: the UNet hot path only runs on a CUDA (sm_90a) device; there is no CPU fallback")
        self._validate(sample)
        timesteps = timestep
        if not torch.is_tensor(timesteps):
            dtype = torch.float64 if isinstance(timestep, float) else torch.int64
            timesteps = torch.tensor([timesteps], dtype=dtype, device=sample.device)
        elif len(timesteps.shape) == 0:
            timesteps = timesteps[None].to(sample.device)
        batch_size = sample.shape[0]
        timesteps = timesteps.expand(batch_size)

        trainable = [p for p in self.parameters() if p.requires_grad]
        record = torch.is_grad_enabled() and len(trainable) > 0
        out = _UNetFn.apply(self, record, sample, timesteps, encoder_hidden_states, added_time_ids, *trainable)
        if not return_dict:
            return (out,)
        return UNetSpatioTemporalConditionOutput(sample=out)

    def _check_latent_size(self, sample: torch.Tensor):
        """every down block but the last halves the latent, and each up block concatenates the skip of the same size: the
        latent height and width must be multiples of 2^(down blocks - 1). Any such size runs (the convolutions take any width)."""
        f = 1 << (len(self.down_blocks) - 1)
        H, W = sample.shape[-2], sample.shape[-1]
        if H % f or W % f:
            raise ValueError(f"svd_xtend_b200: the latent height and width must be multiples of 2^(number of down blocks - 1) = {f} "
                             f"for the skip connections to line up; got {H}x{W}")

    def _validate(self, sample: torch.Tensor):
        """boundary checks, cached on (parameter count, dtype/device signature): every parameter on the sample's device
        and of a dtype the weight-preparation kernels can read (fp32 / bf16 / fp16; anything else would be misread)."""
        sig = (sample.device, tuple((p.dtype, p.device) for p in self.parameters()))
        if getattr(self, "_validated_sig", None) != sig:
            for n, p in self.named_parameters():
                if p.device != sample.device:
                    raise RuntimeError("svd_xtend_b200: all parameters must live on the device of `sample`")
                raw.dtype_code(p, f"parameter {n}")
            self._validated_sig = sig

    # the tape-driven network -------------------------------------------------
    def _run(self, sample, timesteps, encoder_hidden_states, added_time_ids) -> Tuple[torch.Tensor, Var, Geom]:
        E = self._engine
        B, T, Cin, H, W = sample.shape
        dev = sample.device
        g = Geom(B, T, H, W)
        N = B * T
        cfg = self.config

        # ---- 1. time embeddings (:403-416): tiny; sinusoid in torch, MLPs through the GEMM kernel
        emb1 = self._mlp(E, _sinusoid(timesteps.to(dev), cfg.block_out_channels[0]), self.time_embedding)
        t_ids = _sinusoid(added_time_ids.flatten().to(dev), cfg.addition_time_embed_dim).reshape(B, -1)
        emb = E.add_f32(emb1, self._mlp(E, t_ids, self.add_embedding))            # [B, 1280] fp32
        semb = E.silu_cast(emb)                                                   # nonlinearity(temb), shared by all resnets
        projs = []
        for rb in self._resblocks:
            projs += [rb.spatial_res_block.time_emb_proj, rb.temporal_res_block.time_emb_proj]
        temb_slices = {}
        if semb.needs_grad or any(p.weight.requires_grad or p.bias.requires_grad for p in projs):
            for p in projs:      # differentiable path: one small GEMM per projection
                temb_slices[p] = E.linear(semb, p.weight, p.bias, out_f32=True)
        else:
            # frozen (the scripted configuration): every resnet's time_emb_proj in ONE GEMM
            w_all = E.w_lin_cat([p.weight for p in projs], False)
            b_all = E.wc.get(("tembbias",) + tuple(id(p.bias) for p in projs), [p.bias for p in projs], (w_all.shape[0],),
                             lambda buf: buf.copy_(torch.cat([p.bias.detach().float() for p in projs])), dtype=F32)
            temb_all = torch.empty(B, w_all.shape[0], device=dev, dtype=F32)
            raw.tapgemm_auto(semb.data, w_all, temb_all, M=B, N=w_all.shape[0], K=w_all.shape[1], bias=b_all)
            o0 = 0
            for p in projs:
                temb_slices[p] = Var(temb_all[:, o0:o0 + p.out_features])
                o0 += p.out_features
        temb = temb_slices     # per forward (closures of checkpointed blocks keep THIS forward's projections)

        # image embedding per clip (encoder_hidden_states is [B,1,1024]; :425 repeats it per frame)
        enc = Var(encoder_hidden_states.reshape(B, -1).to(bf16).contiguous())

        # ---- 2. conv_in (:420-428)
        x_nchw = sample.reshape(N, Cin, H, W).contiguous()
        cpad = 64
        x0 = torch.empty(N * H * W, cpad, device=dev, dtype=bf16)
        raw.nchw_to_nhwc(x_nchw if x_nchw.dtype in (F32, bf16, torch.float16) else x_nchw.float(), x0, N, Cin, H, W, cpad)
        x = E.conv2d_3x3(Var(x0), g, self.conv_in, i_pad=cpad, gn_rows=g.HW)

        # ---- 3. down (:432-448)
        skips = [(x, g)]
        for blk in self.down_blocks:
            for j, res in enumerate(blk.resnets):
                x = self._res(E, blk, res, x, g, temb)
                if blk.has_cross_attention:
                    x = self._transformer(E, blk.attentions[j], x, g, enc)
                skips.append((x, g))
            if blk.downsamplers is not None:
                p = E.space_to_planes(x, g)
                g = g.down()
                x = E.conv2d_3x3(p, g, blk.downsamplers[0].conv, planes=True, gn_rows=g.HW)
                skips.append((x, g))

        # ---- 4. mid (:451-456)
        x = self._resblock(E, self.mid_block.resnets[0], x, g, temb)     # [D]: the first mid resnet is never checkpointed
        for attn, res in zip(self.mid_block.attentions, self.mid_block.resnets[1:]):
            x = self._transformer(E, attn, x, g, enc)
            x = self._res(E, self.mid_block, res, x, g, temb)

        # ---- 5. up (:459-477)
        for blk in self.up_blocks:
            for j, res in enumerate(blk.resnets):
                skip, _ = skips.pop()
                x = E.concat(x, skip)
                x = self._res(E, blk, res, x, g, temb)
                if blk.has_cross_attention:
                    x = self._transformer(E, blk.attentions[j], x, g, enc)
            if blk.upsamplers is not None:
                u = E.upsample2x(x, g)
                g = g.up()
                x = E.conv2d_3x3(u, g, blk.upsamplers[0].conv, gn_rows=g.HW)

        # ---- 6. post-process (:480-485)
        h = E.groupnorm(x, self.conv_norm_out, outer=N, rows=g.HW, silu=True)
        y = E.conv2d_3x3(h, g, self.conv_out, n_pad=8)
        Cout = cfg.out_channels
        out = torch.empty(B, T, Cout, H, W, device=dev, dtype=sample.dtype if sample.dtype in (F32, bf16, torch.float16) else F32)
        raw.nhwc_to_nchw(y.data, out, N, Cout, H, W)
        return out, y, g

    def _mlp(self, E: Engine, x32: torch.Tensor, mlp: TimestepEmbedding) -> Var:
        """TimestepEmbedding on a few rows: Linear -> SiLU -> Linear, fp32 in/out, bf16 operands."""
        dev = x32.device
        xb = raw.cast_f32_bf16(x32.contiguous().float(), torch.empty(x32.shape, device=dev, dtype=bf16))
        h = E.linear(Var(xb), mlp.linear_1.weight, mlp.linear_1.bias, out_f32=True)
        return E.linear(E.silu_cast(h), mlp.linear_2.weight, mlp.linear_2.bias, out_f32=True)

    def _blend(self, E: Engine, mixer: AlphaBlender) -> torch.Tensor:
        """device float[16] epilogue scale triples (svdx_blend_scales layout) of an AlphaBlender (image_only_indicator is all zeros, :430)."""
        mix = mixer.mix_factor
        return E.wc.get(("blend", id(mix)), [mix], (16,), lambda buf: raw.blend_scales(E.vec_f32(mix), buf), dtype=F32)

    def _res(self, E: Engine, owner: nn.Module, res: SpatioTemporalResBlock, x: Var, g: Geom, temb) -> Var:
        """a resnet of a down/mid/up block, gradient-checkpointed when the owner's flag is set ([D] unet_3d_blocks.py)."""
        if self.training and getattr(owner, "gradient_checkpointing", False):
            return E.checkpoint(lambda v: self._resblock(E, res, v, g, temb), x)
        return self._resblock(E, res, x, g, temb)

    def _resblock(self, E: Engine, blk: SpatioTemporalResBlock, x: Var, g: Geom, temb) -> Var:
        """SpatioTemporalResBlock [D: resnet.py]: spatial ResnetBlock2D -> TemporalResnetBlock -> AlphaBlender."""
        sp, tp = blk.spatial_res_block, blk.temporal_res_block
        N = g.B * g.T
        per_clip = g.T * g.HW
        h = E.groupnorm(x, sp.norm1, outer=N, rows=g.HW, silu=True)
        h = E.conv2d_3x3(h, g, sp.conv1, rowbias=temb[sp.time_emb_proj], rowbias_div=per_clip, gn_rows=g.HW)
        h = E.groupnorm(h, sp.norm2, outer=N, rows=g.HW, silu=True)
        xs = x if sp.conv_shortcut is None else E.linear(x, sp.conv_shortcut.weight, sp.conv_shortcut.bias)
        hs = E.conv2d_3x3(h, g, sp.conv2, res1=xs, gn_rows=per_clip)     # -> temporal norm1: statistics per clip
        t = E.groupnorm(hs, tp.norm1, outer=g.B, rows=per_clip, silu=True)
        t = E.conv_temporal(t, g, tp.conv1, rowbias=temb[tp.time_emb_proj], rowbias_div=per_clip, gn_rows=per_clip)
        t = E.groupnorm(t, tp.norm2, outer=g.B, rows=per_clip, silu=True)
        s8 = self._blend(E, blk.time_mixer)
        # alpha*hs + (1-alpha)*(hs + conv) = hs + (1-alpha)*conv
        return E.conv_temporal(t, g, tp.conv2, res1=hs, scales=s8[4:7], res1_unit=True, blend=(blk.time_mixer.mix_factor, s8[1:2]),
                               gn_rows=g.HW)     # block output: the next GroupNorm (resnet norm1 / transformer norm / concat) is per frame

    @staticmethod
    def _qkv_lora(attn: Attention):
        C = attn.inner_dim
        return _lora_of(attn.to_q, 0) + _lora_of(attn.to_k, C) + _lora_of(attn.to_v, 2 * C)

    def _cross_vec(self, E: Engine, attn2: Attention, enc: Var) -> Var:
        """Image cross-attention has ONE key/value token (train_svd.py:1000-1001), so softmax == 1 and the
        attention output is to_out(to_v(e)) for every query of the clip (SURVEY.md §0 quirk 3): a [B, C]
        vector, added through the row-bias epilogue. to_q / to_k / norm2 receive exactly zero gradient."""
        v = E.linear(enc, attn2.to_v.weight, lora=_lora_of(attn2.to_v))
        c = E.linear(v, attn2.to_out[0].weight, attn2.to_out[0].bias, lora=_lora_of(attn2.to_out[0]))
        return E.cast_to_f32(c)

    def _frame_emb(self, E: Engine, tr: TransformerSpatioTemporalModel, g: Geom):
        """time_pos_embed(Timesteps(arange(T))) [D: transformer_temporal.py] -> fp32 [B*T, C]; input independent, so it
        is cached while its MLP is frozen. Returns (tensor, Var-or-None for the gradient path)."""
        mlp = tr.time_pos_embed
        params = [mlp.linear_1.weight, mlp.linear_1.bias, mlp.linear_2.weight, mlp.linear_2.bias]
        C = tr.in_channels

        def sinus(dev):
            return _sinusoid(torch.arange(g.T, device=dev).repeat(g.B), C)
        if E.recording and any(p.requires_grad for p in params):
            v = self._mlp(E, sinus(params[0].device), mlp)
            return v.data, v
        return E.wc.get(("frame_emb", id(tr), g.B, g.T), params, (g.B * g.T, C),
                        lambda buf: buf.copy_(self._mlp(E, sinus(buf.device), mlp).data), dtype=F32), None

    def _transformer(self, E: Engine, tr: TransformerSpatioTemporalModel, x_in: Var, g: Geom, enc: Var) -> Var:
        """TransformerSpatioTemporalModel [D]: GN -> proj_in -> spatial block -> temporal block -> blend -> proj_out -> +x."""
        N = g.B * g.T
        per_clip = g.T * g.HW
        heads = tr.heads
        sb, tb = tr.transformer_blocks[0], tr.temporal_transformer_blocks[0]
        if self.grad_hook is not None and E.recording:
            ready = [p for p in tr.parameters() if p.requires_grad]
            if ready:  # recorded first => runs last in this block's backward: its parameter gradients are final
                E.record(lambda ready=ready: self.grad_hook(ready))
        h = E.groupnorm(x_in, tr.norm, outer=N, rows=g.HW, silu=False)
        x0 = E.linear(h, tr.proj_in.weight, tr.proj_in.bias)
        # spatial BasicTransformerBlock ([D] transformer_temporal.py checkpoints only this block)
        def spatial(x0: Var) -> Var:
            _, n1 = E.layernorm(x0, sb.norm1)
            qkv = E.linear(n1, None, fused=[sb.attn1.to_q.weight, sb.attn1.to_k.weight, sb.attn1.to_v.weight], lora=self._qkv_lora(sb.attn1))
            a = E.attention(qkv, heads, g, temporal=False)
            x1 = E.linear(a, sb.attn1.to_out[0].weight, sb.attn1.to_out[0].bias, res1=x0,
                          rowbias=self._cross_vec(E, sb.attn2, enc), rowbias_div=per_clip, lora=_lora_of(sb.attn1.to_out[0]))
            _, n3 = E.layernorm(x1, sb.norm3)
            ff = E.linear(n3, sb.ff.net[0].proj.weight, sb.ff.net[0].proj.bias, geglu=True)
            return E.linear(ff, sb.ff.net[2].weight, sb.ff.net[2].bias, res1=x1)

        if self.training and tr.gradient_checkpointing:
            x2 = E.checkpoint(spatial, x0)
        else:
            x2 = spatial(x0)
        # TemporalBasicTransformerBlock on the same token layout (frames are HW rows apart)
        femb, femb_var = self._frame_emb(E, tr, g)
        xm, ni = E.layernorm(x2, tb.norm_in, addvec=femb, add_div=g.HW, addvec_var=femb_var)
        ff = E.linear(ni, tb.ff_in.net[0].proj.weight, tb.ff_in.net[0].proj.bias, geglu=True)
        y1 = E.linear(ff, tb.ff_in.net[2].weight, tb.ff_in.net[2].bias, res1=xm)
        _, n1 = E.layernorm(y1, tb.norm1)
        qkv = E.linear(n1, None, fused=[tb.attn1.to_q.weight, tb.attn1.to_k.weight, tb.attn1.to_v.weight], lora=self._qkv_lora(tb.attn1))
        a = E.attention(qkv, heads, g, temporal=True)
        y2 = E.linear(a, tb.attn1.to_out[0].weight, tb.attn1.to_out[0].bias, res1=y1,
                      rowbias=self._cross_vec(E, tb.attn2, enc), rowbias_div=per_clip, lora=_lora_of(tb.attn1.to_out[0]))
        _, n3 = E.layernorm(y2, tb.norm3)
        ff = E.linear(n3, tb.ff.net[0].proj.weight, tb.ff.net[0].proj.bias, geglu=True)
        s8 = self._blend(E, tr.time_mixer)
        # alpha*x_spatial + (1-alpha)*(ff + y2)
        xb = E.linear(ff, tb.ff.net[2].weight, tb.ff.net[2].bias, res1=x2, res2=y2, scales=s8[0:3],
                      blend=(tr.time_mixer.mix_factor, s8[1:2]))
        return E.linear(xb, tr.proj_out.weight, tr.proj_out.bias, res1=x_in, gn_rows=g.HW)


class _UNetFn(torch.autograd.Function):
    """One autograd node for the whole UNet: forward records the engine tape, backward replays it.
    Parameter gradients are accumulated in fp32 by the kernels and attached to `.grad` directly."""

    @staticmethod
    def forward(ctx, model: UNetSpatioTemporalConditionModel, record: bool, sample, timesteps, enc, added_time_ids, *params):
        E = model._engine
        ctx.model, ctx.params = model, params
        ctx.n_out = model.config.out_channels
        ctx.entry = None
        if model._graphs is not None:
            served = model._graphs.forward(record, sample, timesteps, enc, added_time_ids)
            if served is not None:
                out, ctx.entry = served
                ctx.y, ctx.g, ctx.tape = ctx.entry.y, ctx.entry.geom, None
                return out
        if model._arena is not None and model._arena.stale():
            # an optimizer other than FusedAdamW, load_state_dict or an EMA copy-back touched the fp32 masters: the bf16
            # shadow / transposed operands are re-derived before they are used (a captured forward does this in-graph)
            model.refresh_trainable_operands(shadow_current=False)
        E.begin(recording=record)
        out, y, g = model._run(sample, timesteps, enc, added_time_ids)
        ctx.y, ctx.g = y, g
        ctx.tape = E.detach_tape()      # this forward's tape lives on ITS autograd node (ADVICE r1: no cross-forward clobbering)
        return out

    @staticmethod
    def backward(ctx, dout):
        model, y, g, params = ctx.model, ctx.y, ctx.g, ctx.params
        E = model._engine
        N = g.B * g.T
        views = E.grad_views
        if views and all(p.grad is None for p in params if p in views):
            # optimizer.zero_grad(set_to_none=True) (train_svd.py:1049) dropped the .grad views: the flat gradient arena the
            # kernels accumulate into must start this backward at zero, or gradients would pile up across steps
            model._arena.zero_grad()
        captured = ctx.entry is not None
        if captured:
            entry, ctx.entry = ctx.entry, None
            if not entry.pending_backward:
                raise RuntimeError("svd_xtend_b200: backward called twice on the same forward (retain_graph is not supported)")
            E.pgrads = dict(model._graphs.backward(entry, dout, ctx.n_out))      # static buffers of the captured backward
        else:
            d = dout.reshape(N, ctx.n_out, g.H, g.W).contiguous()
            if d.dtype not in (F32, bf16):
                d = d.float()
            dy = torch.empty(N * g.H * g.W, y.data.shape[1], device=d.device, dtype=bf16)
            raw.nchw_to_nhwc(d, dy, N, ctx.n_out, g.H, g.W, y.data.shape[1])
            E.add_grad(y, dy)
            tape, ctx.tape = ctx.tape, None
            if tape is None:
                raise RuntimeError("svd_xtend_b200: backward called twice on the same forward (retain_graph is not supported)")
            E.run_backward(tape)
        for p in params:
            if p in views:
                p.grad = views[p]        # the kernels accumulated straight into the arena
                continue
            gp = E.pgrads.get(p)
            if gp is None:
                gp = torch.zeros(p.shape, device=p.device, dtype=F32)   # e.g. attn2.to_q/to_k/norm2: exactly zero
            if p.dtype != F32:
                gp = gp.to(p.dtype)
            elif captured:
                # a captured backward re-fills the same static buffer on every replay: .grad is a copy of it, so that a
                # second backward without zero_grad (gradient accumulation) adds to the first instead of replacing it
                gp = gp.clone()
            if p.grad is None:
                p.grad = gp
            else:
                p.grad.add_(gp)
        E.pgrads = {}
        if model.grad_hook is not None:
            model.grad_hook(None)       # None = everything is final
        return (None,) * (6 + len(params))
