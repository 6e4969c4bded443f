#!/usr/bin/env python
"""Gradient accumulation and gradient-norm clipping of the training step from video frames (VideoTrainStep) on one H100, one
JSON line.

    python scripts/bench_grad_accum.py --config 2 [--steps K] [--warmup W]
    python scripts/bench_grad_accum.py --config 4 [--steps K] [--warmup W]

Seeded default-init SVD UNet (the config's trainable set and gradient checkpointing), VAE encoder and CLIP ViT-H image encoder,
FusedAdamW, B = 1, conditioning dropout 0.1, frames from a device buffer.
  --config 2: ms per call of the graphed step at gradient_accumulation_steps 1 and 4, timed in alternating windows of 4K calls
    (medians of 3); the update graph of k = 4 alone; svdx_grad_sumsq + svdx_clip_coef over the as-scripted gradient arena
    (CUDA events over 50 launches) with the bytes they read and the rate; the k = 1 step with and without max_grad_norm, in
    alternating windows of K calls.
  --config 4: 25 x 576 x 1024 at k = 2 with bf16 VAE / CLIP and encode_chunk_size 2: ms per call and the peak
    torch.cuda.max_memory_allocated.
Every line carries the card's name and power limit, read in the same run. Writes nothing to the source tree.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def _models(cfg, frozen_bf16, dev):
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.train import ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    from svd_xtend_b200.workload import SVD_CONFIG
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        vae = AutoencoderKLTemporalDecoder(**VAE_CONFIG)
        clip = CLIPVisionModelWithProjection(**CLIP_CONFIG)
    for m in (unet, vae, clip):
        m.requires_grad_(False)
    if frozen_bf16:                     # train_svd.py:665-673 under --mixed_precision=bf16
        vae.to(torch.bfloat16)
        clip.to(torch.bfloat16)
    vae.eval()
    clip.eval()
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:          # train_svd.py:761-766
            p.requires_grad_(True)
    unet.train()
    if cfg["grad_ckpt"]:
        unet.enable_gradient_checkpointing()
    arena = ParamArena(unet)
    unet.attach_arena(arena)
    return unet, vae, clip, arena


def _opt(unet, arena, max_grad_norm=None):
    from svd_xtend_b200.train import FusedAdamW
    opt = FusedAdamW(arena, lr=1e-5, max_grad_norm=max_grad_norm)
    opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
    return opt


def _windows(forms, calls, rounds=3):
    """ms per call of each form, alternating windows of `calls` calls"""
    times = {k: [] for k in forms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, fn in forms.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(calls):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / calls)
    return {k: {"ms_per_call": round(statistics.median(ts), 3), "windows_ms": [round(t, 3) for t in ts]} for k, ts in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, choices=(2, 4), default=2)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_grad_accum.py needs a CUDA device: the step has no CPU fallback")
    from scripts.bench_decode import power_limit_w
    from svd_xtend_b200 import raw
    from svd_xtend_b200.video_train import VideoTrainStep
    from svd_xtend_b200.workload import BENCH_CONFIGS

    dev = torch.device("cuda", 0)
    cfg = BENCH_CONFIGS[args.config]
    F, H, W = cfg["frames"], 8 * cfg["h"], 8 * cfg["w"]
    steps, warmup = max(args.steps, 1), max(args.warmup, 1)
    unet, vae, clip, arena = _models(cfg, args.config == 4, dev)
    x = (torch.rand(1, F, 3, H, W, generator=torch.Generator().manual_seed(5)) * 2 - 1).to(dev)
    kw = dict(frames_shape=(1, F, H, W), conditioning_dropout_prob=0.1)
    res = {"metric": "grad_accum", "config": args.config, "frames": F, "pixels": [H, W], "batch": 1,
           "trainable_params": sum(p.numel() for p in arena.params), "arena_numel": arena.numel}

    if args.config == 4:
        opt = _opt(unet, arena, max_grad_norm=1.0)
        torch.cuda.reset_peak_memory_stats()
        step = VideoTrainStep(unet, vae, clip, opt, generator=torch.Generator(dev).manual_seed(0), encode_chunk_size=2,
                              gradient_accumulation_steps=2, **kw)
        res["built_max_allocated_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        for _ in range(2 * warmup):
            step(x)
        res["k2"] = _windows({"k2": lambda: step(x)}, 2 * steps)["k2"]
        res["max_memory_allocated_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        res["grad_norm"] = float(opt.grad_norm.item())
    else:
        opt = _opt(unet, arena)
        s1 = VideoTrainStep(unet, vae, clip, opt, generator=torch.Generator(dev).manual_seed(0), **kw)
        s4 = VideoTrainStep(unet, vae, clip, opt, generator=torch.Generator(dev).manual_seed(0), gradient_accumulation_steps=4, **kw)
        for _ in range(4 * warmup):
            s1(x)
            s4(x)
        res["accumulation"] = _windows({"k1": lambda: s1(x), "k4": lambda: s4(x)}, 4 * steps)
        res["update_graph_alone"] = _windows({"update": s4.graphed_update.replay}, 4 * steps)["update"]
        del s4
        torch.cuda.empty_cache()

        # the norm kernels over the as-scripted gradient arena
        sumsq = torch.zeros(1 + raw.SUMSQ_PARTIALS, device=dev, dtype=torch.float64)
        mx, out = torch.ones(1, device=dev), torch.zeros(2, device=dev)
        arena.grad.normal_()
        for _ in range(5):
            raw.grad_sumsq(arena.grad, sumsq)
            raw.clip_coef(sumsq, mx, 1.0, out)
        n_iter = 50
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n_iter):
            raw.grad_sumsq(arena.grad, sumsq)
            raw.clip_coef(sumsq, mx, 1.0, out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n_iter
        nbytes = 4 * arena.numel
        res["norm_kernels"] = {"ms": round(ms, 4), "bytes_read": nbytes, "achieved_gb_per_s": round(nbytes / ms / 1e6, 1),
                               "datasheet_floor_ms_at_3.35TB/s": round(nbytes / 3.35e12 * 1e3, 4)}
        arena.zero_grad()

        # the k = 1 step with and without clipping: two optimizers over the one arena (their own moments)
        opt_c = _opt(unet, arena, max_grad_norm=1.0)
        s1c = VideoTrainStep(unet, vae, clip, opt_c, generator=torch.Generator(dev).manual_seed(0), **kw)
        for _ in range(warmup):
            s1(x)
            s1c(x)
        res["clip"] = _windows({"no_clip": lambda: s1(x), "max_grad_norm": lambda: s1c(x)}, steps)
        res["grad_norm"] = float(opt_c.grad_norm.item())
        res["max_memory_allocated_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    res.update(device=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(0))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
