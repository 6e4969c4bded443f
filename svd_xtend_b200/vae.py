"""`AutoencoderKLTemporalDecoder.encode` on H100 — SURVEY.md §8f-1: the VAE encode that sits on the critical path of every
training step of the reference (`tensor_to_vae_latent`, /root/reference/train_svd.py:283-291, called at :948 for the clip and
at :959 for the noise-augmented conditioning frame):

    latents = vae.encode(frames).latent_dist.sample() * vae.config.scaling_factor

Same kernels as the UNet (one channels-last bf16 token matrix for the whole encoder): 3x3 convolutions as tap-shifted TMA
boxes on wgmma (`svdx_tapgemm`, here also for images wider than one 128-pixel tile: 320x512 frames), GroupNorm statistics
fused into the producing conv epilogue, GroupNorm+SiLU apply, the stride-2 convs over parity planes (the VAE's
pad-(0,1,0,1) form), and the mid block's single-head dim-512 attention as QK^T / row-softmax / PV GEMMs (its S x S score
matrix is small). Forward only: the VAE is frozen (`vae.requires_grad_(False)`, train_svd.py:659) — gradients are refused.

Decode (built with `with_decoder=True`): the temporal decoder of the inference path (StableVideoDiffusionPipeline.decode_latents,
see sampling.decode_latents) on the same kernels — per-frame spatial resnets, per-clip temporal resnets ((3,1,1) convs with
GroupNorm statistics over T*H*W) mixed by the switched AlphaBlender in the conv epilogue, the same mid-block attention, and
Upsample2D as four 2x2-tap phase convolutions that store straight into the upsampled tensor (`svdx_tapgemm` interleaved
store); the tail (3-channel conv_out in fp32, the (3,1,1) time_conv_out, NCHW output) is `svdx_time_conv_out`.

Module / parameter names follow the diffusers state dict of `AutoencoderKLTemporalDecoder` (encoder.*, quant_conv, decoder.*);
`from_pretrained` ignores the decoder.* tensors unless with_decoder=True. No PyTorch / CPU fallback.
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
from .unet import _Config


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


class _TemporalRes(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, c, eps=1e-5, affine=True)
        self.conv1 = nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))
        self.norm2 = nn.GroupNorm(32, c, eps=1e-5, affine=True)
        self.conv2 = nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))


class _Mixer(nn.Module):
    def __init__(self):
        super().__init__()
        self.mix_factor = nn.Parameter(torch.zeros(1))


class _STRes(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.spatial_res_block = _Resnet(cin, cout)
        self.temporal_res_block = _TemporalRes(cout)
        self.time_mixer = _Mixer()


class _DecMid(nn.Module):
    def __init__(self, c, layers):
        super().__init__()
        self.attentions = nn.ModuleList([_Attn(c)])
        self.resnets = nn.ModuleList([_STRes(c, c) for _ in range(layers)])


class _Up(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)


class _UpBlock(nn.Module):
    def __init__(self, cin, cout, layers, add_up):
        super().__init__()
        self.resnets = nn.ModuleList([_STRes(cin if i == 0 else cout, cout) for i in range(layers)])
        self.upsamplers = nn.ModuleList([_Up(cout)]) if add_up else None


class _Decoder(nn.Module):
    def __init__(self, latent, cout, boc, layers):
        super().__init__()
        self.conv_in = nn.Conv2d(latent, boc[-1], 3, padding=1)
        self.mid_block = _DecMid(boc[-1], layers)
        rev = list(reversed(boc))
        blocks, oc = [], rev[0]
        for i, c in enumerate(rev):
            ic, oc = oc, c
            blocks.append(_UpBlock(ic, oc, layers + 1, i != len(rev) - 1))
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = nn.GroupNorm(32, boc[0], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[0], cout, 3, padding=1)
        self.time_conv_out = nn.Conv3d(cout, cout, (3, 1, 1), padding=(1, 0, 0))


# Upsample2D as four 2x2-tap convolutions on the low-res input, one per output parity: output row 2h + ph of
# conv3x3(nearest2x(x)) reads upsampled rows 2h + ph - 1 .. 2h + ph + 1, i.e. low-res rows {h-1, h, h} (ph = 0) or {h, h, h+1}
# (ph = 1). Kernel rows that read the same low-res row are summed; columns fold the same way. Zero padding of the high-res
# border is exactly an out-of-image low-res read.
_PHASE_FOLD = (((0,), (1, 2)), ((0, 1), (2,)))      # [parity][low-res tap a] -> 3x3 kernel rows (columns) summed into it
PHASES = ((0, 0), (0, 1), (1, 0), (1, 1))


def fold_upsample_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """3x3 conv weight [O, I, 3, 3] -> the four phase kernels [4, O, I, 2, 2] (index 2*ph + pw). Phase (ph, pw) at low-res
    pixel (h, w) is sum_{a, b} k[:, :, a, b] x[h + a - 1 + ph, w + b - 1 + pw] (see `phase_taps`)."""
    out = []
    for ph in (0, 1):
        rows = torch.stack([w[:, :, list(s), :].sum(2) for s in _PHASE_FOLD[ph]], 2)
        for pw in (0, 1):
            out.append(torch.stack([rows[:, :, :, list(s)].sum(3) for s in _PHASE_FOLD[pw]], 3))
    return torch.stack(out)


def phase_taps(ph: int, pw: int):
    """svdx_tapgemm CONV2D taps (dw, dh, dn) of phase (ph, pw), in the [a][b] order of the folded kernel"""
    return tuple((b - 1 + pw, a - 1 + ph, 0) for a in range(2) for b in range(2))


def _mid_attention(E: Engine, a: _Attn, x: Var, g: Geom) -> Var:
    """[D] Attention(heads = 1, dim_head = C, residual_connection, group_norm): per frame softmax(Q K^T / sqrt(C)) V
    (the mid block of the encoder and of the temporal decoder)"""
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
    """replacement of diffusers' AutoencoderKLTemporalDecoder: encode (train_svd.py:649-650, :673, :283-291) and, when built
    with_decoder=True, the temporal decode of the inference path (StableVideoDiffusionPipeline.decode_latents)."""

    config_name = "config.json"

    def __init__(self, in_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 scaling_factor=0.18215, with_decoder=False, force_upcast=True, **config):
        """keyword arguments this model does not use (config.json's `out_channels`, `sample_size`, `down_block_types`, ...) are
        kept on `self.config` and written back by `save_pretrained`"""
        super().__init__()
        self.config = _Config(**config)
        self.config.__dict__.update(in_channels=in_channels, latent_channels=latent_channels, block_out_channels=tuple(block_out_channels),
                                    layers_per_block=layers_per_block, scaling_factor=scaling_factor, force_upcast=force_upcast)
        if any(c % 32 for c in block_out_channels):
            raise ValueError("block_out_channels must be multiples of 32 (GroupNorm(32) and 32-column epilogue chunks)")
        self.encoder = _Encoder(in_channels, latent_channels, tuple(block_out_channels), layers_per_block)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.decoder = _Decoder(latent_channels, in_channels, tuple(block_out_channels), layers_per_block) if with_decoder else None
        self._engine = Engine()

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, torch_dtype=None, variant: Optional[str] = None,
                        with_decoder: bool = False, revision: Optional[str] = None, low_cpu_mem_usage: bool = True, **kw):
        """with_decoder=False (the training path) drops the decoder.* tensors; True loads them too, strictly. Local directories
        only: a `revision` or a path that is not a directory raises ValueError. Every key of config.json is kept on `config`."""
        if revision is not None:
            raise ValueError(f"AutoencoderKLTemporalDecoder.from_pretrained: revision={revision!r} is not supported (local directories only)")
        if not os.path.isdir(path):
            raise ValueError(f"AutoencoderKLTemporalDecoder.from_pretrained: {path!r} is not a local directory (hub downloads are not supported)")
        d = path if subfolder is None else os.path.join(path, subfolder)
        with open(os.path.join(d, cls.config_name)) as f:
            cfg = json.load(f)
        cfg.pop("with_decoder", None)
        model = cls(**cfg, with_decoder=with_decoder)
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
        if not with_decoder:
            sd = {k: v for k, v in sd.items() if not k.startswith("decoder.")}      # the temporal decoder is not part of this model
        model.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
        if torch_dtype is not None:
            model.to(torch_dtype)
        return model

    def save_pretrained(self, save_directory: str, safe_serialization: bool = True, variant: Optional[str] = None, **kwargs):
        """diffusers' layout: config.json (every config key, `_class_name` AutoencoderKLTemporalDecoder) and
        diffusion_pytorch_model[.variant].safetensors (or .bin) with diffusers' keys, decoder.* included when built with it"""
        os.makedirs(save_directory, exist_ok=True)
        cfg = self.config.to_dict()
        cfg["_class_name"] = "AutoencoderKLTemporalDecoder"
        with open(os.path.join(save_directory, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2)
        stem = "diffusion_pytorch_model" + ("" if variant is None else f".{variant}")
        sd = {k: v.detach().cpu().contiguous() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, stem + ".safetensors"))
        else:
            torch.save(sd, os.path.join(save_directory, stem + ".bin"))

    def forward(self, sample: torch.Tensor, sample_posterior: bool = False, return_dict: bool = True,
                generator: Optional[torch.Generator] = None, num_frames: int = 1):
        """[D] AutoencoderKLTemporalDecoder.forward: encode, the posterior's mode (or a sample), decode in clips of num_frames"""
        posterior = self.encode(sample).latent_dist
        z = posterior.sample(generator=generator) if sample_posterior else posterior.mode()
        dec = self.decode(z, num_frames=num_frames).sample
        return SimpleNamespace(sample=dec) if return_dict else (dec,)

    # ------------------------------------------------------------------ the encode path
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [N, 3, H, W] (H, W multiples of 2^(levels-1), any such size) -> object with `.latent_dist`"""
        f = 1 << (len(self.config.block_out_channels) - 1)
        if x.shape[-2] % f or x.shape[-1] % f:
            raise ValueError(f"encode: the frame height and width must be multiples of 2^(levels - 1) = {f} (one stride-2 "
                             f"downsample per level but the last); got {x.shape[-2]}x{x.shape[-1]}")
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
        return _mid_attention(E, a, x, g)

    def _run(self, x: torch.Tensor) -> torch.Tensor:
        N, Cin, H, W = x.shape
        x0 = torch.empty(N * H * W, self.ROW_PAD, device=x.device, dtype=bf16)
        xin = x.contiguous()
        raw.nchw_to_nhwc(xin if xin.dtype in (F32, bf16, torch.float16) else xin.float(), x0, N, Cin, H, W, self.ROW_PAD)
        out = self._run_rows(x0, N, H, W)
        return out.to(x.dtype) if x.dtype in (bf16, torch.float16) else out

    ROW_PAD = 64          # columns of the encoder's input rows (conv_in's channels zero padded to one 64-wide k-block)

    def _run_rows(self, x0: torch.Tensor, N: int, H: int, W: int) -> torch.Tensor:
        """the encoder on its bf16 input rows x0 [N*H*W, ROW_PAD] (token-major, as svdx_nchw_to_nhwc writes them) -> the fp32
        NCHW moments [N, 2*latent_channels, H/f, W/f]"""
        E = self._engine
        enc = self.encoder
        dev = x0.device
        E.begin(recording=False)
        g = Geom(N, 1, H, W)
        cpad = self.ROW_PAD
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
        return out

    # ------------------------------------------------------------------ the decode path
    def decode(self, z: torch.Tensor, num_frames: int, return_dict: bool = True):
        """[D] AutoencoderKLTemporalDecoder.decode: z [B*F, latent, h, w] (F = num_frames, one clip of F frames per B) ->
        object with `.sample` [B*F, 3, h * 2^(levels-1), w * 2^(levels-1)]. The temporal layers see the F frames of each clip."""
        if self.decoder is None:
            raise RuntimeError("svd_xtend_b200: this AutoencoderKLTemporalDecoder was built without the decoder "
                               "(construct / from_pretrained with with_decoder=True)")
        N, Cl, h, w = z.shape
        if num_frames < 1 or N % num_frames:
            raise ValueError(f"decode: {N} latent frames are not a whole number of clips of num_frames={num_frames}")
        if Cl != self.config.latent_channels:
            raise ValueError(f"decode: expected {self.config.latent_channels} latent channels, got {Cl}")
        self._check_decode_geometry(h, w)
        if not z.is_cuda:
            raise RuntimeError("svd_xtend_b200: the VAE decode path only runs on a CUDA (sm_90a) device; there is no CPU fallback")
        if torch.is_grad_enabled() and (z.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("svd_xtend_b200: AutoencoderKLTemporalDecoder.decode is forward-only; "
                               "call vae.requires_grad_(False) / use torch.no_grad()")
        for n, p in self.named_parameters():
            raw.dtype_code(p, f"parameter {n}")
        sample = self._run_decode(z, num_frames)
        if not return_dict:
            return (sample,)
        return SimpleNamespace(sample=sample)

    def _check_decode_geometry(self, h: int, w: int):
        """A level at least 32 pixels wide takes any width and height: the 3x3 convs read widths the row boxes cannot tile
        through im2col loads, and the phase-form upsample splits a 32-pixel store chunk that crosses image rows. A narrower
        level needs W | 128 (below 32 the same as W | 32: a store chunk is whole image rows), and if it is upsampled also
        H*W % 32 == 0 (a chunk is whole images). For latents whose sides are multiples of 8 (every size the UNet takes) this
        accepts every width except 24, i.e. 192-pixel-wide frames."""
        levels = len(self.config.block_out_channels)
        for lv in range(levels):
            H, W = h << lv, w << lv
            if W < 32 and 128 % W:
                raise ValueError(f"decode: latent width {w} gives width {W} at level {lv}; a level narrower than 32 pixels needs W | 128")
            if lv < levels - 1 and W < 32 and (H * W) % 32:
                raise ValueError(f"decode: the 2x upsample at {H}x{W} needs H*W % 32 == 0 when W < 32")

    def _stres(self, E: Engine, blk: _STRes, x: Var, g: Geom) -> Var:
        """[D] SpatioTemporalResBlock of the temporal decoder: ResnetBlock2D -> TemporalResnetBlock -> AlphaBlender with
        switch_spatial_to_temporal_mix, i.e. out = hs + sigmoid(mix) * h_t: the resnet blend triple of svdx_blend_scales at -mix"""
        sp, tp = blk.spatial_res_block, blk.temporal_res_block
        n, per_clip = g.B * g.T, g.T * g.HW
        h = E.groupnorm(x, sp.norm1, outer=n, rows=g.HW, silu=True)
        h = E.conv2d_3x3(h, g, sp.conv1, gn_rows=g.HW)
        h = E.groupnorm(h, sp.norm2, outer=n, rows=g.HW, silu=True)
        xs = x if sp.conv_shortcut is None else E.linear(x, sp.conv_shortcut.weight, sp.conv_shortcut.bias)
        hs = E.conv2d_3x3(h, g, sp.conv2, res1=xs, gn_rows=per_clip)       # -> temporal norm1: statistics per clip
        t = E.groupnorm(hs, tp.norm1, outer=g.B, rows=per_clip, silu=True)
        t = E.conv_temporal(t, g, tp.conv1, gn_rows=per_clip)
        t = E.groupnorm(t, tp.norm2, outer=g.B, rows=per_clip, silu=True)
        mix = blk.time_mixer.mix_factor
        s16 = E.wc.get(("blend_switched", id(mix)), [mix], (16,), lambda buf: raw.blend_scales(-E.vec_f32(mix), buf), dtype=F32)
        return E.conv_temporal(t, g, tp.conv2, res1=hs, scales=s16[4:7], res1_unit=True, gn_rows=g.HW)

    def _upsample_conv(self, E: Engine, conv: nn.Conv2d, x: Var, g: Geom) -> Var:
        """Upsample2D (nearest 2x + 3x3 conv) as four phase convolutions of 4 taps at the low-res geometry g, each storing its
        parity straight into the high-res output. Their fused GroupNorm sums accumulate into one per-frame slab."""
        w = conv.weight
        O, I = w.shape[0], w.shape[1]

        def build(buf):
            k = fold_upsample_conv_weight(w.detach().float())
            for i in range(4):
                raw.prep_weight(k[i].contiguous(), buf[i], 2, O, I, 4, I)
        wf = E.wc.get(("phase", id(w)), [w], (4, O, 4 * I), build)
        nimg = g.B * g.T
        M = nimg * g.HW
        out = E.empty(4 * M, O, x.data)
        sink = E.stat_zeros(nimg * 2 * O, out.device).view(nimg, 2, O)
        b32 = E.vec_f32(conv.bias)
        for i, (ph, pw) in enumerate(PHASES):
            raw.tapgemm(x.data, wf[i], out, M=M, N=O, K=I, mode=raw.A_CONV2D, taps=phase_taps(ph, pw), conv_whn=(g.W, g.H, nimg),
                        bias=b32, gn_sum=sink, gn_rows=g.HW, phase=(ph, pw))
        y = Var(out)
        y.csum = (4 * g.HW, [(sink, O)])
        return y

    def _run_decode(self, z: torch.Tensor, T: int) -> torch.Tensor:
        E = self._engine
        dec = self.decoder
        N, Cl, h, w = z.shape
        dev = z.device
        E.begin(recording=False)
        g = Geom(N // T, T, h, w)
        cpad = 64
        x0 = torch.empty(N * h * w, cpad, device=dev, dtype=bf16)
        zin = z.contiguous()
        raw.nchw_to_nhwc(zin if zin.dtype in (F32, bf16, torch.float16) else zin.float(), x0, N, Cl, h, w, cpad)
        x = E.conv2d_3x3(Var(x0), g, dec.conv_in, i_pad=cpad, gn_rows=g.HW)
        mid = dec.mid_block
        x = self._stres(E, mid.resnets[0], x, g)
        for r, a in zip(mid.resnets[1:], mid.attentions):
            x = _mid_attention(E, a, x, g)
            x = self._stres(E, r, x, g)
        for blk in dec.up_blocks:
            for r in blk.resnets:
                x = self._stres(E, r, x, g)
            if blk.upsamplers is not None:
                x = self._upsample_conv(E, blk.upsamplers[0].conv, x, g)
                g = g.up()
        x = E.groupnorm(x, dec.conv_norm_out, outer=N, rows=g.HW, silu=True)
        # conv_out in fp32 into an 8-column buffer (3 valid): the frames are rounded once, by time_conv_out's output cast
        Cout = dec.conv_out.weight.shape[0]
        y = torch.empty(g.M, 8, device=dev, dtype=F32)
        raw.tapgemm(x.data, E.w_conv(dec.conv_out.weight, False), y, M=g.M, N=Cout, K=x.cols, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS,
                    conv_whn=(g.W, g.H, N), bias=E.vec_f32(dec.conv_out.bias), block_n=32)
        out = torch.empty(N, Cout, g.H, g.W, device=dev, dtype=z.dtype if z.dtype in (bf16, torch.float16) else F32)
        return raw.time_conv_out(y, E.vec_f32(dec.time_conv_out.weight), E.vec_f32(dec.time_conv_out.bias), out, T)


class AutoencoderKLTemporalDecoderWithDecoder(AutoencoderKLTemporalDecoder):
    """the class svd_xtend_b200.shim installs as `diffusers.AutoencoderKLTemporalDecoder`: diffusers' class always has the
    temporal decoder, so `from_pretrained` loads it unless told otherwise (the package's own default stays encoder-only)"""

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, torch_dtype=None, variant: Optional[str] = None,
                        with_decoder: bool = True, **kw):
        return super().from_pretrained(path, subfolder=subfolder, torch_dtype=torch_dtype, variant=variant, with_decoder=with_decoder, **kw)


def tensor_to_vae_latent(t: torch.Tensor, vae: AutoencoderKLTemporalDecoder, noise: Optional[torch.Tensor] = None, generator=None) -> torch.Tensor:
    """train_svd.py:283-291: [B, F, 3, H, W] frames -> scaled latents [B, F, 4, H/8, W/8]"""
    b, f = t.shape[:2]
    with torch.no_grad():
        latents = vae.encode(t.flatten(0, 1)).latent_dist.sample(generator=generator, noise=noise)
    return latents.reshape(b, f, *latents.shape[1:]) * vae.config.scaling_factor
