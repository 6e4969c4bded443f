"""`CLIPVisionModelWithProjection` on H100: the frozen CLIP image encoder of SVD (the checkpoint's `image_encoder/`, ViT-H/14),
which turns the conditioning frame into the `[B, 1, 1024]` `encoder_hidden_states` the UNet cross-attends to — every training
step (train_svd.py:975-976 -> `encode_image`, :857-876) and every validation / inference video ([D]
StableVideoDiffusionPipeline._encode_image).

One token-major bf16 matrix `[B * 257, 1280]` for the whole encoder, on the project's kernels:
  * `svdx_clip_preprocess`: resize (Gaussian blur + bicubic), normalisation and patchify of the image in one pass, straight
    into the A operand of the patch-embedding GEMM (`encode_image`); the identity form of the same kernel patchifies an
    already-normalised 224 x 224 input (`forward`);
  * the patch embedding is one `svdx_tapgemm` whose residual operand is a cached `[B * 257, C]` table (row 0 = class embedding
    + position 0, rows 1.. = positions 1..): the class token and the positions cost nothing extra;
  * per layer: LayerNorm (`svdx_layernorm_fwd`), the fused q|k|v GEMM, `svdx_attention_hd80_fwd`, out_proj with the residual
    epilogue, LayerNorm, fc1 with the activation epilogue (gelu / quick_gelu), fc2 with the residual epilogue;
  * post_layernorm of the B class rows and `visual_projection` as `svdx_gemv`.

Forward only (the encoder is frozen: train_svd.py:660), CUDA only, fp32 / bf16 / fp16 parameters; bf16 operand copies come from
the engine's weight cache and are prepared once. Parameter names are transformers' (`vision_model.*`, `visual_projection.weight`).
"""
from __future__ import annotations

import json
import os
from types import SimpleNamespace
from typing import Optional, Sequence

import torch
import torch.nn as nn

from . import raw
from .engine import Engine, F32, Var, bf16

# CLIPImageProcessor's default normalisation (also the SVD checkpoint's feature_extractor/preprocessor_config.json)
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
_ACTS = {"gelu": raw.ACT_GELU, "quick_gelu": raw.ACT_QUICK_GELU}
_HEAD_DIM = 80


class _Embeddings(nn.Module):
    def __init__(self, C, patch, image_size, channels):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.randn(C))
        self.patch_embedding = nn.Conv2d(channels, C, patch, stride=patch, bias=False)
        self.position_embedding = nn.Embedding((image_size // patch) ** 2 + 1, C)


class _Attention(nn.Module):
    def __init__(self, C):
        super().__init__()
        self.k_proj = nn.Linear(C, C)
        self.v_proj = nn.Linear(C, C)
        self.q_proj = nn.Linear(C, C)
        self.out_proj = nn.Linear(C, C)


class _MLP(nn.Module):
    def __init__(self, C, I):
        super().__init__()
        self.fc1 = nn.Linear(C, I)
        self.fc2 = nn.Linear(I, C)


class _Layer(nn.Module):
    def __init__(self, C, I, eps):
        super().__init__()
        self.self_attn = _Attention(C)
        self.layer_norm1 = nn.LayerNorm(C, eps=eps)
        self.mlp = _MLP(C, I)
        self.layer_norm2 = nn.LayerNorm(C, eps=eps)


class _Encoder(nn.Module):
    def __init__(self, C, I, layers, eps):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(C, I, eps) for _ in range(layers)])


class _VisionTransformer(nn.Module):
    def __init__(self, C, I, layers, patch, image_size, channels, eps):
        super().__init__()
        self.embeddings = _Embeddings(C, patch, image_size, channels)
        self.pre_layrnorm = nn.LayerNorm(C, eps=eps)
        self.encoder = _Encoder(C, I, layers, eps)
        self.post_layernorm = nn.LayerNorm(C, eps=eps)


def antialias_kernels(h: int, w: int, size: int):
    """(gy, gx): the 1-D Gaussian weights of the anti-aliasing blur before resizing h x w to size x size, computed in fp32 the
    way train_svd.py's `_resize_with_antialiasing` does: sigma = max((factor - 1) / 2, 0.001) per axis, int(max(4 sigma, 3))
    taps made odd, weights exp(-x^2 / (2 sigma^2)) normalised to sum 1."""
    out = []
    for n in (h, w):
        sigma = max((n / size - 1.0) / 2.0, 0.001)
        k = int(max(4.0 * sigma, 3))
        k += 1 - k % 2
        s = torch.tensor([[sigma]], dtype=F32)
        x = torch.arange(k, dtype=F32) - k // 2
        g = torch.exp(-x.pow(2.0) / (2 * s.pow(2.0)))
        out.append((g / g.sum(-1, keepdim=True))[0].tolist())
    return out[0], out[1]


def image_processor_stats(path: str, subfolder: Optional[str] = "feature_extractor"):
    """(image_mean, image_std) of a `preprocessor_config.json` (CLIPImageProcessor's defaults for keys it does not set)"""
    d = path if subfolder is None else os.path.join(path, subfolder)
    with open(os.path.join(d, "preprocessor_config.json")) as f:
        cfg = json.load(f)
    mean, std = tuple(float(v) for v in cfg.get("image_mean", CLIP_MEAN)), tuple(float(v) for v in cfg.get("image_std", CLIP_STD))
    if len(mean) != 3 or len(std) != 3:
        raise ValueError("preprocessor_config.json: image_mean / image_std must have 3 entries")
    return mean, std


def clip_flops(config=None, image_size: Optional[int] = None) -> dict:
    """algorithmic FLOPs of one image through CLIPVisionModelWithProjection, counted from shapes, per family"""
    c = SimpleNamespace(**config) if isinstance(config, dict) else config
    img = image_size if image_size is not None else c.image_size
    P = img // c.patch_size
    S, C, I, L = 1 + P * P, c.hidden_size, c.intermediate_size, c.num_hidden_layers
    fl = dict(linear=L * 2.0 * S * C * (4 * C + 2 * I), attention=L * 4.0 * S * S * C,
              patch_embedding=2.0 * P * P * 3 * c.patch_size ** 2 * C, projection=2.0 * C * c.projection_dim)
    fl["total"] = sum(fl.values())
    return fl


class CLIPVisionModelWithProjection(nn.Module):
    """replacement of transformers' CLIPVisionModelWithProjection (the SVD image encoder), forward only"""

    config_name = "config.json"

    def __init__(self, hidden_size=768, intermediate_size=3072, num_attention_heads=12, num_hidden_layers=12, patch_size=32,
                 image_size=224, projection_dim=512, layer_norm_eps=1e-5, hidden_act="quick_gelu", num_channels=3, **ignored):
        super().__init__()
        if hidden_act not in _ACTS:
            raise ValueError(f"svd_xtend_b200: unsupported hidden_act {hidden_act!r} (supported: gelu, quick_gelu)")
        if hidden_size % num_attention_heads or hidden_size // num_attention_heads != _HEAD_DIM:
            raise ValueError(f"svd_xtend_b200: the CLIP attention kernel needs head dim {_HEAD_DIM} "
                             f"(hidden_size {hidden_size} / {num_attention_heads} heads)")
        if num_channels != 3 or image_size % patch_size or hidden_size % 32 or intermediate_size % 32 or projection_dim % 8:
            raise ValueError("svd_xtend_b200: CLIP config needs 3 channels, image_size % patch_size == 0, hidden_size and "
                             "intermediate_size multiples of 32, projection_dim a multiple of 8")
        self.config = SimpleNamespace(hidden_size=hidden_size, intermediate_size=intermediate_size, num_attention_heads=num_attention_heads,
                                      num_hidden_layers=num_hidden_layers, patch_size=patch_size, image_size=image_size,
                                      projection_dim=projection_dim, layer_norm_eps=layer_norm_eps, hidden_act=hidden_act,
                                      num_channels=num_channels)
        self.vision_model = _VisionTransformer(hidden_size, intermediate_size, num_hidden_layers, patch_size, image_size, num_channels,
                                               layer_norm_eps)
        self.visual_projection = nn.Linear(hidden_size, projection_dim, bias=False)
        self._engine = Engine()

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = "image_encoder", torch_dtype=None, variant: Optional[str] = None,
                        **ignored):
        """reads `config.json` and `model[.variant].safetensors` (or `pytorch_model[.variant].bin`), loaded strictly"""
        d = path if subfolder is None else os.path.join(path, subfolder)
        with open(os.path.join(d, cls.config_name)) as f:
            cfg = json.load(f)
        model = cls(**{k: v for k, v in cfg.items() if k in ("hidden_size", "intermediate_size", "num_attention_heads", "num_hidden_layers",
                                                              "patch_size", "image_size", "projection_dim", "layer_norm_eps",
                                                              "hidden_act", "num_channels")})
        sd = None
        for stem, ext in ([] if variant is None else [(f"model.{variant}", "safetensors"), (f"pytorch_model.{variant}", "bin")]) + \
                [("model", "safetensors"), ("pytorch_model", "bin")]:
            p = os.path.join(d, f"{stem}.{ext}")
            if os.path.exists(p):
                if ext == "safetensors":
                    from safetensors.torch import load_file
                    sd = load_file(p)
                else:
                    sd = torch.load(p, map_location="cpu")
                break
        if sd is None:
            raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin under {d}")
        sd.pop("vision_model.embeddings.position_ids", None)          # a buffer older transformers versions saved
        model.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
        if torch_dtype is not None:
            model.to(torch_dtype)
        return model

    def save_pretrained(self, save_directory: str, safe_serialization: bool = True, **kwargs):
        """transformers' layout: config.json (a `clip_vision_model` config) and model.safetensors (or pytorch_model.bin) with
        the keys `from_pretrained` reads"""
        os.makedirs(save_directory, exist_ok=True)
        cfg = dict(vars(self.config), architectures=["CLIPVisionModelWithProjection"], model_type="clip_vision_model",
                   torch_dtype=str(self.dtype).replace("torch.", ""))
        with open(os.path.join(save_directory, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2)
        sd = {k: v.detach().cpu().contiguous() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, "model.safetensors"), metadata={"format": "pt"})
        else:
            torch.save(sd, os.path.join(save_directory, "pytorch_model.bin"))

    # ------------------------------------------------------------------ entry points
    def _guard(self, x: torch.Tensor, what: str):
        if not x.is_cuda:
            raise RuntimeError(f"svd_xtend_b200: CLIPVisionModelWithProjection.{what} only runs on a CUDA (sm_90a) device; "
                               "there is no CPU fallback")
        grad = torch.is_grad_enabled()
        needs_grad = grad and x.requires_grad
        for n, p in self.named_parameters():          # one walk: supported dtypes (a misread buffer is out of bounds) and grads
            raw.dtype_code(p, f"parameter {n}")
            needs_grad = needs_grad or (grad and p.requires_grad)
        if needs_grad:
            raise RuntimeError(f"svd_xtend_b200: CLIPVisionModelWithProjection.{what} is forward-only (the reference freezes the "
                               "image encoder, train_svd.py:660); call image_encoder.requires_grad_(False) / use torch.no_grad()")
        raw.dtype_code(x, "pixel_values")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"svd_xtend_b200: pixel_values must be [B, 3, H, W], got {tuple(x.shape)}")

    def forward(self, pixel_values: torch.Tensor, return_dict: bool = True):
        """pixel_values: already-normalised [B, 3, image_size, image_size] -> object with `.image_embeds` [B, projection_dim] (parameter
        dtype) and `.last_hidden_state` [B, 1 + P^2, hidden_size] (the encoder output before post_layernorm)"""
        self._guard(pixel_values, "forward")
        n = self.config.image_size
        if pixel_values.shape[-2:] != (n, n):
            raise ValueError(f"Input image size ({pixel_values.shape[-2]}*{pixel_values.shape[-1]}) doesn't match model ({n}*{n}).")
        rows = self._rows(pixel_values.contiguous(), [1.0], [1.0], (1.0, 1.0, 1.0, 0.0, 0.0, 0.0))
        emb, hidden = self._run(rows, pixel_values.shape[0])
        emb, hidden = emb.to(self.dtype), hidden.to(self.dtype)
        out = SimpleNamespace(image_embeds=emb, last_hidden_state=hidden)
        return out if return_dict else (emb, hidden)

    def _rows(self, x: torch.Tensor, gy: Sequence[float], gx: Sequence[float], affine) -> torch.Tensor:
        c = self.config
        P = c.image_size // c.patch_size
        kp = (3 * c.patch_size ** 2 + 63) // 64 * 64
        rows = torch.empty(x.shape[0] * (1 + P * P), kp, device=x.device, dtype=bf16)
        return raw.clip_preprocess(x, gy, gx, affine, rows, out_size=c.image_size, patch=c.patch_size)

    def _patch_operands(self, B: int):
        E, emb, c = self._engine, self.vision_model.embeddings, self.config
        w, cls, pos = emb.patch_embedding.weight, emb.class_embedding, emb.position_embedding.weight
        C, K = c.hidden_size, 3 * c.patch_size ** 2
        kp = (K + 63) // 64 * 64
        wp = E.wc.get(("clip_patch", id(w)), [w], (C, kp), lambda buf: raw.prep_weight(w.detach().reshape(C, K), buf, 2, C, K, 1, kp))

        def table(buf):
            t = pos.detach().float().clone()
            t[0] += cls.detach().float()
            buf.copy_(t.repeat(B, 1))
        tab = E.wc.get(("clip_pos_table", id(cls), id(pos), B), [cls, pos], (B * pos.shape[0], C), table)
        return wp, tab, kp

    def _layernorm(self, x: torch.Tensor, ln: nn.LayerNorm) -> torch.Tensor:
        E = self._engine
        y = torch.empty(x.shape[0], x.shape[1], device=x.device, dtype=bf16)
        raw.layernorm_fwd(x, E.vec_f32(ln.weight), E.vec_f32(ln.bias), ln.eps, y)
        return y

    def _run(self, rows: torch.Tensor, B: int):
        """patch rows [B * S, kp] -> (image_embeds fp32 [B, projection_dim], encoder output bf16 [B, S, hidden_size])"""
        E = self._engine
        c = self.config
        vm = self.vision_model
        C, I, heads = c.hidden_size, c.intermediate_size, c.num_attention_heads
        S = 1 + (c.image_size // c.patch_size) ** 2
        M = B * S
        dev = rows.device
        E.begin(recording=False)
        wp, tab, kp = self._patch_operands(B)
        emb = torch.empty(M, C, device=dev, dtype=bf16)
        raw.tapgemm_auto(rows, wp, emb, M=M, N=C, K=kp, res1=tab)
        x = Var(self._layernorm(emb, vm.pre_layrnorm))
        act = _ACTS[c.hidden_act]
        for layer in vm.encoder.layers:
            a = layer.self_attn
            h = Var(self._layernorm(x.data, layer.layer_norm1))
            bs = [a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]
            bcat = E.wc.get(("clip_qkv_bias",) + tuple(id(b) for b in bs), bs, (3 * C,),
                            lambda buf, bs=bs: buf.copy_(torch.cat([b.detach().float() for b in bs])), dtype=F32)
            qkv = E.linear(h, None, bcat, fused=[a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]).data
            o = torch.empty(M, C, device=dev, dtype=bf16)
            raw.attention_hd80_fwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], o, heads=heads, S=S, nseq=B, scale=_HEAD_DIM ** -0.5)
            x = E.linear(Var(o), a.out_proj.weight, a.out_proj.bias, res1=x)
            h = self._layernorm(x.data, layer.layer_norm2)
            f = torch.empty(M, I, device=dev, dtype=bf16)
            raw.tapgemm_auto(h, E.w_lin(layer.mlp.fc1.weight, False), f, M=M, N=I, K=C, bias=E.vec_f32(layer.mlp.fc1.bias), act=act)
            x = E.linear(Var(f), layer.mlp.fc2.weight, layer.mlp.fc2.bias, res1=x)
        pooled = self._layernorm(x.data.view(B, S * C)[:, :C], vm.post_layernorm)
        wproj = E.w_lin(self.visual_projection.weight, False)
        out = torch.empty(B, c.projection_dim, device=dev, dtype=F32)
        for b0 in range(0, B, 8):
            b1 = min(B, b0 + 8)
            raw.gemv(pooled[b0:b1], wproj, out[b0:b1], M=b1 - b0, N=c.projection_dim, K=C)
        return out, x.data.view(B, S, C)


def encode_image(image_encoder: CLIPVisionModelWithProjection, pixel_values: torch.Tensor, image_mean=CLIP_MEAN, image_std=CLIP_STD):
    """train_svd.py:857-876: images in [-1, 1] of any size [B, 3, H, W] -> image_embeds [B, projection_dim] (parameter dtype).
    The anti-aliased resize to image_size, (x + 1) / 2 and the normalisation by image_mean / image_std run as ONE
    svdx_clip_preprocess launch that writes the patch-embedding operand."""
    m = image_encoder
    m._guard(pixel_values, "encode_image")
    H, W = pixel_values.shape[-2:]
    gy, gx = antialias_kernels(H, W, m.config.image_size)
    # ((v + 1) / 2 - mean) / std = v * (0.5 / std) + (0.5 - mean) / std
    affine = [0.5 / s for s in image_std] + [(0.5 - mu) / s for mu, s in zip(image_mean, image_std)]
    rows = m._rows(pixel_values.contiguous(), gy, gx, affine)
    return m._run(rows, pixel_values.shape[0])[0].to(m.dtype)
