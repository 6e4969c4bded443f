"""A training step from video frames on H100: the body of train_svd.py's training loop (:942-1036) from the clip's pixels to the
optimizer update, with the package's frozen VAE encoder and CLIP image encoder in front of the UNet.

    step = VideoTrainStep(unet, vae, image_encoder, opt, frames_shape=(1, 14, 320, 512), conditioning_dropout_prob=0.1,
                          generator=torch.Generator("cuda").manual_seed(0))
    loss = step(pixel_values)           # [B, F, 3, H, W] in [-1, 1], fp32 or bf16; the 0-dim device loss

Per step: the random draws (`draw_train_noise`) happen eagerly, outside any graph; then `assemble_train_batch` builds the
UNet batch (the dict `workload.synthetic_batch` returns) and the step runs forward, `workload.edm_loss`, backward and the
optimizer, all inside one captured `train.GraphedStep`. The batch assembly is two kernels of csrc/edm.cu around one VAE encode:
`svdx_vae_frames_in` writes the encoder's input rows of the B*F clip frames and the B noise-augmented conditioning frames (one
encode of B*(F+1) frames replaces the reference's two: the encoder works frame by frame), and `svdx_edm_prepare` turns the
moments into the posterior samples, the noisy latents, the target and the UNet input. The per-clip scalars (log-normal sigmas,
timesteps, time ids, dropout masks) are O(B) torch ops. oracle/svd_train_batch_oracle.py states the same in torch.

Decoded uint8 frames [B, F, H0, W0, 3] (VideoTrainStep(source_size=...), assemble_train_batch(size=...)) take the place of
`svdx_vae_frames_in` with `svdx_frames_u8_in` (csrc/frames.cu), which resizes them as Pillow's Image.resize does
(oracle/svd_resize_oracle.py) and normalises them as train_svd.py's DummyDataset does. encode_chunk_size encodes the frames in
chunks.

Clips of mixed source sizes (VideoTrainStep(max_source_size=...), assemble_train_batch with a list of B uint8 clips
[F, H0_b, W0_b, 3]) go through `svdx_frames_u8_in_clips`, the same kernel with one descriptor per clip (ClipSlots), optionally
with a Pillow crop box per clip. FrameFolderClips reads train_svd.py's folder layout and picks clips as its DummyDataset does.
"""
from __future__ import annotations

import os
import random
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import raw
from .clip import CLIP_MEAN, CLIP_STD, encode_image
from .workload import edm_loss

F32 = torch.float32

# (name, kind) in the reference's draw order: posterior sample of the clip (:948 -> :287), the EDM noise (:951), the uniform of
# the conditioning sigma (:954 -> :66), the conditioning-frame noise (:957-958), the posterior sample of the conditioning frame
# (:959), the uniform of the EDM sigma (:964) and the conditioning-dropout uniform (:993, only when dropout is on)
DRAWS = (("latent_eps", "randn"), ("noise", "randn"), ("cond_u", "rand"), ("cond_pixel_eps", "randn"), ("cond_latent_eps", "randn"),
         ("sigma_u", "rand"), ("dropout_u", "rand"))


def draw_shapes(B: int, F: int, H: int, W: int, conditioning_dropout: bool = True) -> Dict[str, tuple]:
    """name -> shape of every draw of one step, in draw order (h = H / 8, w = W / 8)"""
    h, w = H // 8, W // 8
    shapes = dict(latent_eps=(B * F, 4, h, w), noise=(B, F, 4, h, w), cond_u=(B,), cond_pixel_eps=(B, 3, H, W),
                  cond_latent_eps=(B, 4, h, w), sigma_u=(B,), dropout_u=(B,))
    if not conditioning_dropout:
        del shapes["dropout_u"]
    return shapes


def draw_train_noise(B: int, F: int, H: int, W: int, generator: Optional[torch.Generator] = None, device="cuda",
                     conditioning_dropout: bool = True) -> Dict[str, torch.Tensor]:
    """The random draws of one training step from frames [B, F, 3, H, W], as named fp32 tensors on `device`, drawn in this
    order (h = H / 8, w = W / 8):

        1 latent_eps       [B*F, 4, h, w]   randn   posterior sample of the clip frames
        2 noise            [B, F, 4, h, w]  randn   EDM noise
        3 cond_u           [B]              rand    uniform of the conditioning sigma, LogNormal(-3, 0.5)
        4 cond_pixel_eps   [B, 3, H, W]     randn   noise augmentation of the conditioning frame
        5 cond_latent_eps  [B, 4, h, w]     randn   posterior sample of the conditioning frame
        6 sigma_u          [B]              rand    uniform of the EDM sigma, LogNormal(0.7, 1.6)
        7 dropout_u        [B]              rand    conditioning dropout (only when conditioning_dropout)

    Each is drawn from `generator` on the generator's own device (CPU or CUDA; the default generator of `device` when None) and
    then moved to `device`, as diffusers' randn_tensor does, so a CPU generator gives the same values on any device."""
    gdev = torch.device(device) if generator is None else generator.device
    kinds = dict(DRAWS)
    return {name: getattr(torch, kinds[name])(shape, generator=generator, device=gdev, dtype=F32).to(device)
            for name, shape in draw_shapes(B, F, H, W, conditioning_dropout).items()}


def log_normal(u: torch.Tensor, loc: float, scale: float) -> torch.Tensor:
    """rand_log_normal (train_svd.py:64-67) from its uniform draw u, in fp32"""
    return torch.distributions.Normal(loc, scale).icdf(u * (1 - 2e-7) + 1e-7).exp()


def _unet_dims(unet_config):
    """(in_channels, cross_attention_dim, addition_time_embed_dim, add_embedding in_features) of a UNet or its config"""
    cfg = getattr(unet_config, "config", unet_config)
    add = getattr(unet_config, "add_embedding", None)
    in_features = add.linear_1.in_features if add is not None else cfg.projection_class_embeddings_input_dim
    return cfg.in_channels, cfg.cross_attention_dim, cfg.addition_time_embed_dim, in_features


def _check_u8_frames(frames, size):
    """(B, F, H, W) of uint8 frames [B, F, H0, W0, 3] to be resized to size = (H, W); ValueError / TypeError otherwise"""
    if size is None:
        raise TypeError(f"pixel_values has dtype {frames.dtype}; uint8 frames [B, F, H0, W0, 3] need the training size=(H, W)")
    if frames.dim() != 5 or frames.shape[-1] != 3:
        raise ValueError(f"uint8 frames must be [B, F, H0, W0, 3] (HWC, RGB), got {tuple(frames.shape)}")
    H, W = (int(v) for v in size)
    return frames.shape[0], frames.shape[1], H, W


def _check_box(box, H0: int, W0: int, b: int):
    """clip b's box (x0, y0, x1, y1) in fp32, as Pillow stores it; ValueError naming the clip for a box Pillow refuses (negative
    offset, beyond the frame, x1 < x0 or y1 < y0) or one that is not finite"""
    if box is None:
        return None
    if len(box) != 4:
        raise ValueError(f"clip {b}: box must be None or (x0, y0, x1, y1), got {box!r}")
    x0, y0, x1, y1 = (np.float32(v) for v in box)
    if not all(np.isfinite(v) for v in (x0, y0, x1, y1)):
        raise ValueError(f"clip {b}: box {tuple(box)} must be finite")
    if x0 < 0 or y0 < 0:
        raise ValueError(f"clip {b}: box {tuple(box)}: box offset can't be negative")
    if x1 > W0 or y1 > H0:
        raise ValueError(f"clip {b}: box {tuple(box)} can't exceed its frames' size {W0}x{H0} (W x H)")
    if x1 - x0 < 0 or y1 - y0 < 0:
        raise ValueError(f"clip {b}: box {tuple(box)} can't be empty (x1 < x0 or y1 < y0)")
    return float(x0), float(y0), float(x1), float(y1)


def check_clips(clips, size, boxes=None, B: Optional[int] = None, F: Optional[int] = None, capacity=None):
    """(B, F, H, W, boxes) of a list of B uint8 clips [F, H0_b, W0_b, 3] to be resized to size = (H, W), each with its box (None or
    Pillow's (x0, y0, x1, y1)), before any launch: TypeError for a dtype other than uint8, ValueError naming the clip for the
    wrong clip or frame count (B / F when given), channels other than 3, a clip larger than capacity = (H0max, W0max) or a bad
    box"""
    if size is None:
        raise TypeError("uint8 clips [F, H0, W0, 3] need the training size=(H, W)")
    H, W = (int(v) for v in size)
    clips = list(clips)
    if not clips or (B is not None and len(clips) != B):
        raise ValueError(f"expected a list of {B if B is not None else 'B >= 1'} clips, got {len(clips)}")
    boxes = [None] * len(clips) if boxes is None else list(boxes)
    if len(boxes) != len(clips):
        raise ValueError(f"boxes must hold one entry (None or (x0, y0, x1, y1)) per clip: {len(clips)} clips, {len(boxes)} boxes")
    out = []
    for b, (c, box) in enumerate(zip(clips, boxes)):
        if not isinstance(c, torch.Tensor):
            raise TypeError(f"clip {b}: expected a uint8 tensor [F, H0, W0, 3], got {type(c).__name__}")
        if c.dtype != torch.uint8:
            raise TypeError(f"clip {b}: dtype {c.dtype}; the mixed-size form takes uint8 frames [F, H0, W0, 3]")
        if c.dim() != 4 or c.shape[-1] != 3:
            raise ValueError(f"clip {b}: uint8 frames must be [F, H0, W0, 3] (HWC, RGB, 3 channels), got {tuple(c.shape)}")
        want_f = F if F is not None else clips[0].shape[0]
        if c.shape[0] != want_f or c.shape[0] < 1:
            raise ValueError(f"clip {b}: {c.shape[0]} frames, expected {want_f}")
        H0, W0 = int(c.shape[1]), int(c.shape[2])
        if H0 < 1 or W0 < 1:
            raise ValueError(f"clip {b}: empty frames {H0}x{W0}")
        if capacity is not None and (H0 > capacity[0] or W0 > capacity[1]):
            raise ValueError(f"clip {b}: frames of {H0}x{W0} exceed the step's max_source_size {capacity[0]}x{capacity[1]}")
        out.append(_check_box(box, H0, W0, b))
    return len(clips), int(clips[0].shape[0]), H, W, out


def check_train_inputs(vae, image_encoder, unet_config, pixel_values, draws, conditioning_dropout_prob=None, size=None,
                       encode_chunk_size=None, boxes=None):
    """every check of assemble_train_batch, before any launch: ValueError / TypeError for what does not fit, RuntimeError for
    models or tensors off the GPU (there is no CPU path)"""
    if encode_chunk_size is not None and (int(encode_chunk_size) != encode_chunk_size or encode_chunk_size < 1):
        raise ValueError(f"encode_chunk_size must be None or a positive number of frames, got {encode_chunk_size!r}")
    if boxes is not None and not isinstance(pixel_values, (list, tuple)):
        raise ValueError("boxes are taken with a list of uint8 clips only")
    on_gpu = []
    if isinstance(pixel_values, ClipSlots):
        B, F, H, W = pixel_values.B, pixel_values.F, pixel_values.H, pixel_values.W
        on_gpu.append(pixel_values.slots.is_cuda)
    elif isinstance(pixel_values, (list, tuple)):
        B, F, H, W, _ = check_clips(pixel_values, size, boxes)
    elif pixel_values.dtype == torch.uint8:
        B, F, H, W = _check_u8_frames(pixel_values, size)
        on_gpu.append(pixel_values.is_cuda)
    else:
        if pixel_values.dim() != 5 or pixel_values.shape[2] != 3:
            raise ValueError(f"pixel_values must be [B, F, 3, H, W], got {tuple(pixel_values.shape)}")
        if pixel_values.dtype not in (F32, torch.bfloat16):
            raise TypeError(f"pixel_values has dtype {pixel_values.dtype}; supported: float32, bfloat16 (uint8 with size=(H, W))")
        B, F, _, H, W = pixel_values.shape
        if size is not None and tuple(int(v) for v in size) != (H, W):
            raise ValueError(f"size={tuple(size)} given for float frames of {H}x{W}; float frames are used at their own size")
        on_gpu.append(pixel_values.is_cuda)
    if H % 64 or W % 64:
        raise ValueError(f"frame height and width must be multiples of 64 (the UNet's latents, H/8 x W/8, need sides that are "
                         f"multiples of 8); got {H}x{W}")
    in_ch, cross, add_dim, add_in = _unet_dims(unet_config)
    lc = vae.config.latent_channels
    if 2 * lc != in_ch:
        raise ValueError(f"the VAE's latent_channels x 2 = {2 * lc} must equal the UNet's in_channels = {in_ch} (noisy latents "
                         "concatenated with the conditioning latents)")
    if lc != 4 or 1 << (len(vae.config.block_out_channels) - 1) != 8:
        raise ValueError("the VAE must have 4 latent channels and downsample by 8 (the draws are [., 4, H/8, W/8])")
    if image_encoder.config.projection_dim != cross:
        raise ValueError(f"the CLIP projection_dim {image_encoder.config.projection_dim} must equal the UNet's cross_attention_dim {cross}")
    if add_dim * 3 != add_in:
        raise ValueError(f"Model expects an added time embedding vector of length {add_in}, but a vector of {add_dim * 3} was "
                         "created (addition_time_embed_dim x 3 time ids). The model has an incorrect config.")
    shapes = draw_shapes(B, F, H, W, conditioning_dropout_prob is not None)
    for name, shape in shapes.items():
        t = draws.get(name)
        if t is None or t.dtype != F32 or tuple(t.shape) != shape:
            raise ValueError(f"draws[{name!r}] must be an fp32 tensor of shape {shape} (draw_train_noise), got "
                             f"{None if t is None else (tuple(t.shape), t.dtype)}")
    for n, p in list(vae.named_parameters()) + list(image_encoder.named_parameters()):
        raw.dtype_code(p, f"parameter {n}")
    on_gpu += [vae.device.type == "cuda", image_encoder.device.type == "cuda"] + [draws[n].is_cuda for n in shapes]
    if not all(on_gpu):
        raise RuntimeError("svd_xtend_b200: assemble_train_batch only runs on a CUDA (sm_90a) device (frames, draws, VAE and image "
                           "encoder); there is no CPU fallback")
    return B, F, H, W


_TAPS: Dict[tuple, torch.Tensor] = {}


def _device_taps(in_size: int, out_size: int, device) -> torch.Tensor:
    """the resize taps of one axis on `device`, made once per (sizes, device): a step replayed from a CUDA graph reads the copy
    its eager warm-up made"""
    key = (in_size, out_size, str(device))
    if key not in _TAPS:
        _TAPS[key] = raw.resize_taps(in_size, out_size).to(device)
    return _TAPS[key]


_HOST_TAPS: Dict[tuple, np.ndarray] = {}


def _host_taps(in_size: int, out_size: int, lo: float, hi: float) -> np.ndarray:
    """resize_taps of the box [lo, hi) of one axis on the host, made once per (sizes, box)"""
    key = (in_size, out_size, lo, hi)
    if key not in _HOST_TAPS:
        box = None if (lo, hi) == (0.0, float(in_size)) else (lo, hi)
        _HOST_TAPS[key] = raw.resize_taps(in_size, out_size, box).numpy()
    return _HOST_TAPS[key]


class ClipSlots:
    """Device buffers that hold B uint8 clips of up to (H0max, W0max) source pixels, F frames each, for one resize to (H, W)
    (svdx_frames_u8_in_clips): one slot of F*H0max*W0max*3 bytes per clip, and one int32 table with the clips' descriptors and
    tap rows (raw.clip_descs, raw.resize_taps; the tap rows of one axis have the stride of the largest ksize the capacity
    allows). Both stay at fixed addresses, so a captured graph that reads them follows what `load` puts there.

    load(clips, boxes) checks the clips (check_clips), then makes one asynchronous copy per clip of only that clip's bytes (pinned
    host or device memory), and, when the sizes or boxes differ from the previous load, computes the table on the host (taps
    cached per size and box) into a pinned staging buffer and copies it to the device. The staging buffer is rewritten only
    after the previous copy from it has completed (an event)."""

    def __init__(self, B: int, F: int, size, capacity, device):
        self.B, self.F = int(B), int(F)
        self.H, self.W = (int(v) for v in size)
        self.capacity = tuple(int(v) for v in capacity)
        H0m, W0m = self.capacity
        if self.B < 1 or self.F < 1 or min(self.H, self.W, H0m, W0m) < 1:
            raise ValueError(f"ClipSlots needs B, F, the size and the capacity positive, got B={B} F={F} size={size} "
                             f"capacity={capacity}")
        self.slot = self.F * H0m * W0m * 3
        self.slots = torch.zeros(self.B, self.slot, device=device, dtype=torch.uint8)
        self.ks_y = raw.resize_taps(H0m, self.H).shape[1] - 2
        self.ks_x = raw.resize_taps(W0m, self.W).shape[1] - 2
        ny, nx = self.B * self.H * (2 + self.ks_y), self.B * self.W * (2 + self.ks_x)
        n = 6 * self.B + ny + nx
        self.table = torch.zeros(n, device=device, dtype=torch.int32)
        self.descs = self.table[:6 * self.B].view(torch.int64).view(self.B, 3)
        self.taps_y = self.table[6 * self.B:6 * self.B + ny].view(self.B * self.H, 2 + self.ks_y)
        self.taps_x = self.table[6 * self.B + ny:].view(self.B * self.W, 2 + self.ks_x)
        self._staging = torch.zeros(n, dtype=torch.int32, pin_memory=True)
        self._copied = torch.cuda.Event()
        self._loaded = None

    def check(self, clips, boxes=None):
        return check_clips(clips, (self.H, self.W), boxes, B=self.B, F=self.F, capacity=self.capacity)[4]

    def load(self, clips: Sequence[torch.Tensor], boxes=None) -> None:
        fboxes = self.check(clips, boxes)
        for b, c in enumerate(clips):
            n = c.numel()
            self.slots[b, :n].view(c.shape).copy_(c, non_blocking=True)
        key = tuple((tuple(c.shape[1:3]), bx) for c, bx in zip(clips, fboxes))
        if key != self._loaded:
            self._copied.synchronize()              # the previous table copy has read the staging buffer
            self._write_table(key)
            self.table.copy_(self._staging, non_blocking=True)
            self._copied.record()
            self._loaded = key

    def _write_table(self, key) -> None:
        B, H, W = self.B, self.H, self.W
        host = self._staging.numpy()
        ty = host[6 * B:6 * B + B * H * (2 + self.ks_y)].reshape(B * H, 2 + self.ks_y)
        tx = host[6 * B + B * H * (2 + self.ks_y):].reshape(B * W, 2 + self.ks_x)
        ty[:] = 0
        tx[:] = 0
        for b, ((H0, W0), box) in enumerate(key):
            x0, y0, x1, y1 = (0.0, 0.0, float(W0), float(H0)) if box is None else box
            t = _host_taps(H0, H, y0, y1)
            ty[b * H:(b + 1) * H, :t.shape[1]] = t
            t = _host_taps(W0, W, x0, x1)
            tx[b * W:(b + 1) * W, :t.shape[1]] = t
        d = raw.clip_descs([b * self.slot for b in range(B)], [k[0] for k in key], [b * H for b in range(B)],
                           [b * W for b in range(B)])
        host[:6 * B] = d.view(torch.int32).reshape(-1).numpy()

    def fill(self, rows, first, count, cond_eps, cond_sigma, first_frames, c_pad):
        raw.frames_u8_in_clips(self.slots, self.descs, self.taps_y, self.taps_x, cond_eps, cond_sigma, rows, (self.H, self.W),
                               self.F, first, count, first_frames, c_pad)


def assemble_train_batch(vae, image_encoder, unet_config, pixel_values: torch.Tensor, draws: Dict[str, torch.Tensor], *,
                         conditioning_dropout_prob: Optional[float] = None, fps: int = 7, motion_bucket_id: int = 127,
                         image_mean=CLIP_MEAN, image_std=CLIP_STD, size: Optional[Tuple[int, int]] = None,
                         encode_chunk_size: Optional[int] = None, boxes=None) -> Dict[str, torch.Tensor]:
    """train_svd.py:944-1017 from the frames pixel_values [B, F, 3, H, W] (in [-1, 1]) and the step's draws (draw_train_noise) ->
    the UNet batch, the dict workload.synthetic_batch returns: sample [B, F, 8, h, w], timestep [B], encoder_hidden_states
    [B, 1, cross_dim], added_time_ids [B, 3], latents / noisy [B, F, 4, h, w] and sigmas [B, 1, 1, 1, 1], all fp32.

    pixel_values may also be decoded uint8 frames [B, F, H0, W0, 3] (HWC, RGB) with the training size=(H, W): each frame is
    resized as Pillow's Image.resize((W, H)) does (BICUBIC, 8 bits per channel) and normalised as u / 127.5 - 1, as train_svd.py's
    DummyDataset does on the CPU, in the kernel that writes the encoder's input rows (svdx_frames_u8_in).

    pixel_values may also be a list of B uint8 clips [F, H0_b, W0_b, 3] of different source sizes (pinned host or device memory)
    with the training size=(H, W), and boxes a list of None or Pillow's (x0, y0, x1, y1) per clip: clip b is resized as
    Image.resize((W, H), box=boxes[b]) does (svdx_frames_u8_in_clips). Without boxes, the result equals that of the [B, F, H0,
    W0, 3] form for the same pixels. A ClipSlots that holds loaded clips is taken as well.

    encode_chunk_size: None encodes the B*(F+1) frames at once; a number encodes that many frames at a time (as decode_chunk_size
    in sampling.decode_latents), which bounds the encoder's activations. The encoder works frame by frame, so only the order of
    its fp32 GroupNorm-statistics atomics differs.

    unet_config: the UNet or its config. The VAE and the image encoder run forward only. Unlike the reference, every clip's
    added_time_ids carry its own conditioning sigma, and everything before the UNet is fp32 (INTEGRATION.md §3.2)."""
    B, F, H, W = check_train_inputs(vae, image_encoder, unet_config, pixel_values, draws, conditioning_dropout_prob, size,
                                    encode_chunk_size, boxes)
    dev = pixel_values.device if isinstance(pixel_values, torch.Tensor) else vae.device
    clips = pixel_values
    if isinstance(clips, (list, tuple)):
        clips = ClipSlots(B, F, (H, W), (max(c.shape[1] for c in pixel_values), max(c.shape[2] for c in pixel_values)), dev)
        clips.load(pixel_values, boxes)
    x = None if isinstance(clips, ClipSlots) else pixel_values.contiguous()
    cond_sigma = log_normal(draws["cond_u"], -3.0, 0.5)          # :954
    sigma = log_normal(draws["sigma_u"], 0.7, 1.6)               # :964
    N, pad = B * (F + 1), vae.ROW_PAD
    with torch.no_grad():
        if x is None:
            first_frames = torch.empty(B, 3, H, W, device=dev, dtype=F32)

            def fill(rows, first, count):
                clips.fill(rows, first, count, draws["cond_pixel_eps"], cond_sigma, first_frames, pad)
        elif x.dtype == torch.uint8:
            taps_y, taps_x = _device_taps(x.shape[2], H, dev), _device_taps(x.shape[3], W, dev)
            first_frames = torch.empty(B, 3, H, W, device=dev, dtype=F32)

            def fill(rows, first, count):
                raw.frames_u8_in(x, taps_y, taps_x, draws["cond_pixel_eps"], cond_sigma, rows, (H, W), first, count, first_frames, pad)
        else:
            first_frames = x[:, 0]

            def fill(rows, first, count):
                raw.vae_frames_in_range(x, draws["cond_pixel_eps"], cond_sigma, rows, first, count, pad)
        if encode_chunk_size is None:
            rows = torch.empty(N * H * W, pad, device=dev, dtype=torch.bfloat16)
            if x is None or x.dtype == torch.uint8:
                fill(rows, 0, N)
            else:
                raw.vae_frames_in(x, draws["cond_pixel_eps"], cond_sigma, rows, pad)
            moments = vae._run_rows(rows, N, H, W)
            del rows
        else:
            moments = None
            for first in range(0, N, int(encode_chunk_size)):
                count = min(int(encode_chunk_size), N - first)
                rows = torch.empty(count * H * W, pad, device=dev, dtype=torch.bfloat16)
                fill(rows, first, count)
                m = vae._run_rows(rows, count, H, W)
                if moments is None:
                    moments = torch.empty((N,) + tuple(m.shape[1:]), device=dev, dtype=m.dtype)
                moments[first:first + count].copy_(m)
                del rows, m
        emb = encode_image(image_encoder, first_frames, image_mean, image_std).float()      # the clean first frame (:975)
    ehs = emb.unsqueeze(1)
    if conditioning_dropout_prob is None:
        image_mask = torch.ones(B, device=dev, dtype=F32)
    else:
        p = conditioning_dropout_prob
        r = draws["dropout_u"]
        ehs = torch.where((r < 2 * p).reshape(B, 1, 1), torch.zeros_like(ehs), ehs)            # :996-999
        image_mask = 1 - (r >= p).to(F32) * (r < 3 * p).to(F32)                                # :1003-1008
    h, w = H // 8, W // 8
    sample = torch.empty(B, F, 8, h, w, device=dev, dtype=F32)
    noisy = torch.empty(B, F, 4, h, w, device=dev, dtype=F32)
    latents = torch.empty(B, F, 4, h, w, device=dev, dtype=F32)
    raw.edm_prepare(moments, draws["latent_eps"], draws["noise"], draws["cond_latent_eps"], sigma, image_mask,
                    vae.config.scaling_factor, sample, noisy, latents)
    added_time_ids = torch.stack([torch.full_like(cond_sigma, float(fps)), torch.full_like(cond_sigma, float(motion_bucket_id)),
                                  cond_sigma], dim=1)
    return dict(sample=sample, timestep=0.25 * sigma.log(), encoder_hidden_states=ehs, added_time_ids=added_time_ids,
                latents=latents, noisy=noisy, sigmas=sigma.reshape(B, 1, 1, 1, 1))


class VideoTrainStep:
    """One training step from frames: `step(pixel_values)` -> the 0-dim device loss.

    Each call copies the frames [B, F, 3, H, W] (frames_shape; fp32 or bf16, pinned host or device memory) into a static device
    buffer, draws the step's noise eagerly (draw_train_noise, from `generator`) into static buffers, and replays one captured
    train.GraphedStep: opt.zero_grad -> assemble_train_batch -> UNet forward -> workload.edm_loss -> backward -> opt.step().
    cuda_graph=False runs the same function eagerly. Any optimizer of the package works (its on_updated hook should refresh the
    UNet's operands, as for any GraphedStep); `opt.lr = ...` between calls takes effect. Construction leaves the weights, the
    optimizer's moments and step count, an attached EMA and the generator's state as they were.

    source_size=(H0, W0): the step takes decoded uint8 frames [B, F, H0, W0, 3] (HWC, RGB; pinned host or device memory) instead,
    copied 1 byte per channel into a uint8 static buffer and resized on the GPU to frames_shape's H x W as Pillow's
    Image.resize((W, H)) does (assemble_train_batch). encode_chunk_size: encode that many frames at a time (assemble_train_batch).

    max_source_size=(H0max, W0max) (not with source_size): `step(clips, boxes=None)` takes a list of B uint8 clips [F, H0_b, W0_b,
    3] of any sizes up to that capacity, and per clip None or a Pillow crop box (x0, y0, x1, y1); clip b is resized as
    Image.resize((W, H), box=boxes[b]) does. The step holds one slot of F*H0max*W0max*3 bytes per clip and copies only each
    clip's own bytes; the per-clip descriptors and taps are made on the host and copied before the replay (ClipSlots), so sizes
    and boxes may change from call to call without a new capture.

    The graphed form keeps the snapshot it restores after the capture in pinned host memory (train.GraphedStep), which with
    encode_chunk_size is what lets the default size of train_svd.py (25 x 576 x 1024) fit on one 80 GB card.

    gradient_accumulation_steps=k > 1 (train_svd.py --gradient_accumulation_steps, accelerate's `accumulate`): every call runs one
    micro-step (frames and draws -> batch -> UNet -> edm_loss -> (loss / k).backward(), adding into the gradient arena) and
    returns that micro-batch's unscaled loss; calls k, 2k, ... also run the update (opt.step(), clipping included when the
    optimizer has max_grad_norm, then opt.zero_grad()). `step.sync_gradients` is True after a call that updated, as accelerate's
    flag: step a scheduler, log or save there. The micro-step and the update are two captured train.GraphedSteps; construction
    leaves the gradient arena zeroed, so the first window starts clean. k = 1 is the single captured step above."""

    def __init__(self, unet, vae, image_encoder, opt, *, frames_shape, conditioning_dropout_prob: Optional[float] = None,
                 generator: Optional[torch.Generator] = None, fps: int = 7, motion_bucket_id: int = 127, image_mean=CLIP_MEAN,
                 image_std=CLIP_STD, cuda_graph: bool = True, source_size: Optional[Tuple[int, int]] = None,
                 encode_chunk_size: Optional[int] = None, gradient_accumulation_steps: int = 1,
                 max_source_size: Optional[Tuple[int, int]] = None):
        k = gradient_accumulation_steps
        if not isinstance(k, int) or isinstance(k, bool) or k < 1:
            raise ValueError(f"gradient_accumulation_steps must be an int >= 1, got {k!r}")
        self.accumulation_steps = k
        self.sync_gradients = False          # True after a call that applied an optimizer update
        self._calls = 0
        if source_size is not None and max_source_size is not None:
            raise ValueError("source_size and max_source_size are mutually exclusive: one source size, or clips of sizes up to "
                             "max_source_size")
        if vae.device.type != "cuda":
            raise RuntimeError("svd_xtend_b200: VideoTrainStep only runs on a CUDA (sm_90a) device; there is no CPU fallback")
        self.unet, self.vae, self.image_encoder, self.opt = unet, vae, image_encoder, opt
        self.B, self.F, self.H, self.W = (int(v) for v in frames_shape)
        self.dropout = conditioning_dropout_prob
        self.source_size = None if source_size is None else tuple(int(v) for v in source_size)
        self.kw = dict(conditioning_dropout_prob=conditioning_dropout_prob, fps=fps, motion_bucket_id=motion_bucket_id,
                       image_mean=image_mean, image_std=image_std, encode_chunk_size=encode_chunk_size)
        dev = vae.device
        self.device = dev
        if self.source_size is not None:
            H0, W0 = self.source_size
            if H0 <= 0 or W0 <= 0:
                raise ValueError(f"source_size must be two positive sides (H0, W0), got {source_size}")
            self.kw["size"] = (self.H, self.W)
            frames = torch.zeros(self.B, self.F, H0, W0, 3, device=dev, dtype=torch.uint8)
        elif max_source_size is not None:
            cap = tuple(int(v) for v in max_source_size)
            if len(cap) != 2 or min(cap) <= 0:
                raise ValueError(f"max_source_size must be two positive sides (H0max, W0max), got {max_source_size}")
            self.kw["size"] = (self.H, self.W)
            frames = ClipSlots(self.B, self.F, (self.H, self.W), cap, dev)
            frames.load([torch.zeros(self.F, cap[0], cap[1], 3, device=dev, dtype=torch.uint8)] * self.B)
        else:
            frames = torch.zeros(self.B, self.F, 3, self.H, self.W, device=dev, dtype=F32)
        self.generator = generator if generator is not None else torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
        self.static = {"pixel_values": frames}
        gstate = self.generator.get_state()
        self.static.update(self.draw())
        check_train_inputs(vae, image_encoder, unet, self.static["pixel_values"], self.static, conditioning_dropout_prob,
                           self.kw.get("size"), encode_chunk_size)
        self.graphed = None
        self.graphed_update = None
        if cuda_graph:
            from .train import GraphedStep

            def restored():
                self.generator.set_state(gstate)
                unet.refresh_trainable_operands(shadow_current=opt.arena.shadow is not None)

            if k == 1:
                self.graphed = GraphedStep(self._step, self.static, warmup=2, restore=opt.snapshot_tensors(), on_restored=restored,
                                           restore_on_host=True)
            else:
                # the micro-step changes nothing but the gradient arena, which is zeroed below
                self.graphed = GraphedStep(self._micro, self.static, warmup=2, restore=None)
                self.graphed_update = GraphedStep(lambda _s: self._update(), {}, warmup=2, restore=opt.snapshot_tensors(),
                                                  on_restored=restored, restore_on_host=True)
        else:
            self.generator.set_state(gstate)
        if k > 1:
            opt.arena.zero_grad()

    def draw(self) -> Dict[str, torch.Tensor]:
        return draw_train_noise(self.B, self.F, self.H, self.W, generator=self.generator, device=self.device,
                                conditioning_dropout=self.dropout is not None)

    def _step(self, s: Dict[str, torch.Tensor]) -> torch.Tensor:
        self.opt.zero_grad()
        loss = self._micro(s)
        self.opt.step()
        return loss

    def _micro(self, s: Dict[str, torch.Tensor]) -> torch.Tensor:
        """batch -> UNet -> loss -> backward of (loss / k), adding into the gradient arena; the unscaled loss"""
        b = assemble_train_batch(self.vae, self.image_encoder, self.unet, s["pixel_values"], s, **self.kw)
        pred = self.unet(b["sample"], b["timestep"], b["encoder_hidden_states"], added_time_ids=b["added_time_ids"]).sample
        loss = edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"])
        (loss if self.accumulation_steps == 1 else loss / self.accumulation_steps).backward()
        return loss.detach()

    def _update(self) -> None:
        self.opt.step()
        self.opt.zero_grad()

    def check_frames(self, pixel_values, boxes=None) -> None:
        """ValueError / TypeError unless pixel_values (and boxes) are what this step was built for"""
        clips = self.static["pixel_values"]
        if isinstance(clips, ClipSlots):
            if not isinstance(pixel_values, (list, tuple)):
                raise TypeError(f"VideoTrainStep was built for a list of {self.B} uint8 clips (max_source_size), got "
                                f"{type(pixel_values).__name__}")
            clips.check(pixel_values, boxes)
            return
        if boxes is not None:
            raise ValueError("boxes are taken by a step built with max_source_size only")
        if self.source_size is not None:
            want = (self.B, self.F) + self.source_size + (3,)
            if pixel_values.dtype != torch.uint8:
                raise TypeError(f"VideoTrainStep was built for uint8 frames (source_size), got dtype {pixel_values.dtype}")
            if pixel_values.dim() == 5 and pixel_values.shape[-1] != 3:
                raise ValueError(f"uint8 frames must have 3 (RGB) channels, last dimension of {tuple(pixel_values.shape)}")
            if tuple(pixel_values.shape) != want:
                raise ValueError(f"VideoTrainStep was built for uint8 frames {want}, got {tuple(pixel_values.shape)}")
            return
        if tuple(pixel_values.shape) != (self.B, self.F, 3, self.H, self.W):
            raise ValueError(f"VideoTrainStep was built for frames {(self.B, self.F, 3, self.H, self.W)}, got {tuple(pixel_values.shape)}")
        if pixel_values.dtype not in (F32, torch.bfloat16):
            raise TypeError(f"pixel_values has dtype {pixel_values.dtype}; supported: float32, bfloat16")

    def __call__(self, pixel_values, boxes=None) -> torch.Tensor:
        self.check_frames(pixel_values, boxes)
        if isinstance(self.static["pixel_values"], ClipSlots):
            self.static["pixel_values"].load(pixel_values, boxes)
        else:
            self.static["pixel_values"].copy_(pixel_values, non_blocking=True)
        for k, v in self.draw().items():
            self.static[k].copy_(v)
        self._calls += 1
        self.sync_gradients = self._calls % self.accumulation_steps == 0
        if self.accumulation_steps == 1:
            return self.graphed.replay() if self.graphed is not None else self._step(self.static)
        loss = self.graphed.replay() if self.graphed is not None else self._micro(self.static)
        if self.sync_gradients:
            if self.graphed_update is not None:
                self.graphed_update.replay()
            else:
                self._update()
        return loss


class FrameFolderClips(torch.utils.data.Dataset):
    """train_svd.py's folder layout (one folder of frame images per video under base_folder) as uint8 clips at the frames' own
    size, for VideoTrainStep(max_source_size=...): item i is {"pixel_values": uint8 [F, H0, W0, 3], "size": (H0, W0)}.

    Clips are picked as the reference's DummyDataset picks them, with the same calls on Python's global `random` in the same order
    over the same os.listdir order (a folder by random.choice, its sorted frame names, random.randint for the first frame), so a
    seeded run reads the same clips; a folder with fewer than sample_frames frames raises the same ValueError. Frames are decoded
    with Pillow and not resized (the step resizes them on the GPU). A frame that is not RGB, or a clip whose frames differ in
    size, raises ValueError naming the file. `collate` turns a batch into the list of clips the step takes."""

    def __init__(self, base_folder: str, sample_frames: int, num_samples: int = 100000):
        self.num_samples = num_samples
        self.base_folder = base_folder
        self.folders = os.listdir(self.base_folder)
        self.sample_frames = sample_frames

    def __len__(self) -> int:
        return self.num_samples

    def select(self) -> Tuple[str, List[str]]:
        """(folder path, the names of the clip's frames), drawn from the global `random` as DummyDataset.__getitem__ draws"""
        chosen_folder = random.choice(self.folders)
        folder_path = os.path.join(self.base_folder, chosen_folder)
        frames = os.listdir(folder_path)
        frames.sort()
        if len(frames) < self.sample_frames:
            raise ValueError(f"The selected folder '{chosen_folder}' contains fewer than `{self.sample_frames}` frames.")
        start_idx = random.randint(0, len(frames) - self.sample_frames)
        return folder_path, frames[start_idx:start_idx + self.sample_frames]

    def __getitem__(self, idx):
        from PIL import Image
        folder_path, names = self.select()
        out, size = [], None
        for name in names:
            path = os.path.join(folder_path, name)
            with Image.open(path) as img:
                if img.mode != "RGB":
                    raise ValueError(f"{path}: frame mode {img.mode}; FrameFolderClips takes RGB frames (convert them in the loader)")
                a = np.asarray(img)
            if size is None:
                size = a.shape[:2]
            elif a.shape[:2] != size:
                raise ValueError(f"{path}: frame of {a.shape[0]}x{a.shape[1]} in a clip of {size[0]}x{size[1]} frames; the frames "
                                 "of one clip share one size")
            out.append(a)
        return {"pixel_values": torch.from_numpy(np.stack(out)), "size": tuple(int(v) for v in size)}

    @staticmethod
    def collate(batch) -> List[torch.Tensor]:
        """the list of uint8 clips [F, H0_b, W0_b, 3] that VideoTrainStep(max_source_size=...) takes"""
        return [item["pixel_values"] for item in batch]
