"""`AutoencoderKLTemporalDecoder.encode` on H100 — SURVEY.md §8f-1: the VAE encode that sits on the critical path of every
training step of the reference (`tensor_to_vae_latent`, /root/reference/train_svd.py:283-291, called at :948 for the clip and
at :959 for the noise-augmented conditioning frame):

    latents = vae.encode(frames).latent_dist.sample() * vae.config.scaling_factor

Same kernels as the UNet (one channels-last bf16 token matrix for the whole encoder): 3x3 convolutions as tap-shifted TMA
boxes on wgmma (`svdx_tapgemm`, here also for images wider than one 128-pixel tile: 320x512 frames), GroupNorm statistics
fused into the producing conv epilogue, GroupNorm+SiLU apply, the stride-2 convs over parity planes (the VAE's
pad-(0,1,0,1) form), and the mid block's single-head dim-512 attention as QK^T / row-softmax / PV GEMMs (its S x S score
matrix is small). Forward only: the VAE is frozen (`vae.requires_grad_(False)`, train_svd.py:659) — gradients are refused.

Module / parameter names follow the diffusers state dict of `AutoencoderKLTemporalDecoder` (encoder.* and quant_conv);
`from_pretrained` ignores the decoder.* tensors (the temporal decoder is outside this path). No PyTorch / CPU fallback.
"""
from __future__ import annotations

import json
import os
from types import SimpleNamespace
from typing import Optional

import torch
import torch.nn as nn

from . import raw
from .engine import Engine, F32, Geom, Var, bf16


class _Resnet(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, cin, eps=1e-6, affine=True)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(32, cout, eps=1e-6, affine=True)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None


class _Down(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)


class _DownBlock(nn.Module):
    def __init__(self, cin, cout, layers, add_down):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout) for i in range(layers)])
        self.downsamplers = nn.ModuleList([_Down(cout)]) if add_down else None


class _Attn(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.group_norm = nn.GroupNorm(32, c, eps=1e-6, affine=True)
        self.to_q = nn.Linear(c, c)
        self.to_k = nn.Linear(c, c)
        self.to_v = nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])


class _Mid(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(c, c), _Resnet(c, c)])
        self.attentions = nn.ModuleList([_Attn(c)])


class _Encoder(nn.Module):
    def __init__(self, cin, latent, boc, layers):
        super().__init__()
        self.conv_in = nn.Conv2d(cin, boc[0], 3, padding=1)
        blocks, oc = [], boc[0]
        for i, c in enumerate(boc):
            ic, oc = oc, c
            blocks.append(_DownBlock(ic, oc, layers, i != len(boc) - 1))
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = _Mid(boc[-1])
        self.conv_norm_out = nn.GroupNorm(32, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], 2 * latent, 3, padding=1)


class DiagonalGaussianDistribution:
    """[D] vae.py DiagonalGaussianDistribution over the [N, 2*latent, h, w] moments (tiny tensors: plain torch ops)."""

    def __init__(self, parameters: torch.Tensor):
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        if noise is None:
            noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


class AutoencoderKLTemporalDecoder(nn.Module):
    """encode-side replacement of diffusers' AutoencoderKLTemporalDecoder (train_svd.py:649-650, :673, :283-291)."""

    config_name = "config.json"

    def __init__(self, in_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 scaling_factor=0.18215, **ignored):
        super().__init__()
        self.config = SimpleNamespace(in_channels=in_channels, latent_channels=latent_channels, block_out_channels=tuple(block_out_channels),
                                      layers_per_block=layers_per_block, scaling_factor=scaling_factor)
        if any(c % 32 for c in block_out_channels):
            raise ValueError("block_out_channels must be multiples of 32 (GroupNorm(32) and 32-column epilogue chunks)")
        self.encoder = _Encoder(in_channels, latent_channels, tuple(block_out_channels), layers_per_block)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self._engine = Engine()

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, torch_dtype=None, variant: Optional[str] = None, **kw):
        d = path if subfolder is None else os.path.join(path, subfolder)
        with open(os.path.join(d, cls.config_name)) as f:
            cfg = json.load(f)
        model = cls(**{k: v for k, v in cfg.items() if k in ("in_channels", "latent_channels", "block_out_channels", "layers_per_block", "scaling_factor")})
        stems = ["diffusion_pytorch_model"] if variant is None else [f"diffusion_pytorch_model.{variant}", "diffusion_pytorch_model"]
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
        else:
            raise FileNotFoundError(f"no diffusion_pytorch_model weights under {d}")
        sd = {k: v for k, v in sd.items() if not k.startswith("decoder.")}      # the temporal decoder is not part of this path
        model.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
        if torch_dtype is not None:
            model.to(torch_dtype)
        return model

    # ------------------------------------------------------------------ the encode path
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [N, 3, H, W] (H, W multiples of 2^(levels-1); W | 128 or 128 | W at every level) -> object with `.latent_dist`"""
        if not x.is_cuda:
            raise RuntimeError("svd_xtend_b200: the VAE encode path only runs on a CUDA (sm_90a) device; there is no CPU fallback")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("svd_xtend_b200: AutoencoderKLTemporalDecoder.encode is forward-only (the reference freezes the VAE, "
                               "train_svd.py:659); call vae.requires_grad_(False) / use torch.no_grad()")
        for n, p in self.named_parameters():
            raw.dtype_code(p, f"parameter {n}")
        moments = self._run(x)
        dist = DiagonalGaussianDistribution(moments)
        if not return_dict:
            return (dist,)
        return SimpleNamespace(latent_dist=dist)

    def _resnet(self, E: Engine, r: _Resnet, x: Var, g: Geom, gn_rows: int) -> Var:
        n = g.B * g.T
        h = E.groupnorm(x, r.norm1, outer=n, rows=g.HW, silu=True)
        h = E.conv2d_3x3(h, g, r.conv1, gn_rows=gn_rows)
        h = E.groupnorm(h, r.norm2, outer=n, rows=g.HW, silu=True)
        xs = x if r.conv_shortcut is None else E.linear(x, r.conv_shortcut.weight, r.conv_shortcut.bias)
        return E.conv2d_3x3(h, g, r.conv2, res1=xs, gn_rows=gn_rows)

    def _attention(self, E: Engine, a: _Attn, x: Var, g: Geom) -> Var:
        """[D] Attention(heads = 1, dim_head = C, residual_connection, group_norm): per frame softmax(Q K^T / sqrt(C)) V"""
        n, S, C = g.B * g.T, g.HW, x.cols
        hn = E.groupnorm(x, a.group_norm, outer=n, rows=S, silu=False)
        ws = [a.to_q.weight, a.to_k.weight, a.to_v.weight]
        bs = [a.to_q.bias, a.to_k.bias, a.to_v.bias]
        bcat = E.wc.get(("vae_qkv_bias",) + tuple(id(b) for b in bs), bs, (3 * C,),
                        lambda buf: buf.copy_(torch.cat([b.detach().float() for b in bs])), dtype=F32)
        qkv = E.linear(hn, None, bcat, fused=ws).data
        o = torch.empty(n * S, C, device=qkv.device, dtype=bf16)
        scores = torch.empty(S, S, device=qkv.device, dtype=bf16)
        for f in range(n):
            rows = slice(f * S, (f + 1) * S)
            raw.tapgemm(qkv[rows, :C], qkv[rows, C:2 * C], scores, M=S, N=S, K=C)
            raw.softmax_rows(scores, scores, scale=C ** -0.5)
            # P V with V read in place as an MN-major B operand ([keys][C], row stride 3C): no transpose of V
            raw.tapgemm(scores, qkv[rows, 2 * C:], o[rows], M=S, N=C, K=S, b_mn=True, ldb=qkv.stride(0))
        return E.linear(Var(o), a.to_out[0].weight, a.to_out[0].bias, res1=x, gn_rows=S)

    def _run(self, x: torch.Tensor) -> torch.Tensor:
        E = self._engine
        enc = self.encoder
        N, Cin, H, W = x.shape
        dev = x.device
        E.begin(recording=False)
        g = Geom(N, 1, H, W)
        cpad = 64
        x0 = torch.empty(N * H * W, cpad, device=dev, dtype=bf16)
        xin = x.contiguous()
        raw.nchw_to_nhwc(xin if xin.dtype in (F32, bf16, torch.float16) else xin.float(), x0, N, Cin, H, W, cpad)
        h = E.conv2d_3x3(Var(x0), g, enc.conv_in, i_pad=cpad, gn_rows=g.HW)
        for blk in enc.down_blocks:
            for r in blk.resnets:
                h = self._resnet(E, r, h, g, g.HW)
            if blk.downsamplers is not None:
                p = E.space_to_planes(h, g)
                g = g.down()
                h = E.conv2d_3x3(p, g, blk.downsamplers[0].conv, planes=True, planes_pad0=True, gn_rows=g.HW)
        mid = enc.mid_block
        h = self._resnet(E, mid.resnets[0], h, g, g.HW)
        h = self._attention(E, mid.attentions[0], h, g)
        h = self._resnet(E, mid.resnets[1], h, g, g.HW)
        h = E.groupnorm(h, enc.conv_norm_out, outer=N, rows=g.HW, silu=True)
        C2 = 2 * self.config.latent_channels
        y = E.conv2d_3x3(h, g, enc.conv_out, n_pad=(C2 + 7) // 8 * 8)
        if y.cols != C2:
            raise ValueError("latent_channels must be a multiple of 4")
        m = E.linear(y, self.quant_conv.weight, self.quant_conv.bias)
        out = torch.empty(N, C2, g.H, g.W, device=dev, dtype=F32)
        raw.nhwc_to_nchw(m.data, out, N, C2, g.H, g.W)
        return out.to(x.dtype) if x.dtype in (bf16, torch.float16) else out


def tensor_to_vae_latent(t: torch.Tensor, vae: AutoencoderKLTemporalDecoder, noise: Optional[torch.Tensor] = None, generator=None) -> torch.Tensor:
    """train_svd.py:283-291: [B, F, 3, H, W] frames -> scaled latents [B, F, 4, H/8, W/8]"""
    b, f = t.shape[:2]
    with torch.no_grad():
        latents = vae.encode(t.flatten(0, 1)).latent_dist.sample(generator=generator, noise=noise)
    return latents.reshape(b, f, *latents.shape[1:]) * vae.config.scaling_factor
