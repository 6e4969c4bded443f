#!/usr/bin/env python
"""Training step from video frames (svd_xtend_b200.video_train.VideoTrainStep) on the H100 path, one JSON line.

    python scripts/bench_video_train.py --config 2|4 [--steps K] [--warmup W] [--forms graphed,eager,latent_only]
                                        [--input float|u8|mixed] [--source 1080x1920] [--sources 1080x1920,360x640,...]
                                        [--encode-chunk N] [--frozen-dtype fp32|bf16]

Seeded default-init SVD UNet (the config's trainable set and gradient checkpointing), VAE encoder and CLIP ViT-H image encoder,
FusedAdamW, B = 1, conditioning dropout 0.1. The forms of the step (--forms, default all three), timed in alternating windows of
K steps, medians of 3:
  * graphed: VideoTrainStep (frames -> VAE encode -> CLIP -> batch assembly -> UNet -> loss -> backward -> AdamW, one graph),
    frames from a device buffer, draws made eagerly each step;
  * eager: the same VideoTrainStep with cuda_graph=False;
  * latent_only: the latent-input graphed step bench.py times (workload.synthetic_batch, no VAE / CLIP).
--input u8 feeds decoded uint8 frames [1, F, H0, W0, 3] of --source size from pinned host memory (resized on the GPU as Pillow's
Image.resize does); float feeds fp32 frames [1, F, 3, H, W] from a device buffer. --encode-chunk N encodes N frames at a time.
--input mixed feeds a list of uint8 clips [F, H0_b, W0_b, 3] from pinned host memory to a VideoTrainStep(max_source_size=...)
whose capacity is the largest of --sources; each call takes the next size of --sources (clips of one call cycle through it too),
so the sizes change from call to call. The forms graphed_u8 (source_size = the first of --sources) and graphed_float (fp32 frames)
may be added to --forms to time the single-size and float steps in the same session. With --input mixed the report also has the
resize kernel alone (svdx_frames_u8_in_clips over all B*(F+1) frames, CUDA events, median of 20) and the bytes it reads (each
source pixel once) and writes (the bf16 rows and the fp32 first frames), computed from the shapes.
--frozen-dtype: the VAE's and CLIP's weights, fp32 (default) or bf16 as train_svd.py holds them under --mixed_precision=bf16.
Reports ms per step and frames/s of each form, torch.cuda.max_memory_allocated / memory_reserved after each form's
construction, after the warm-up and after the timed windows, the card's name and power limit, and the SM clock sampled during
the timed windows. A form that does not fit on the card is reported as failed. Writes nothing to the source tree.
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


def _mem():
    return {"max_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
            "reserved_gib": round(torch.cuda.memory_reserved() / 2 ** 30, 2)}


def _kernel_alone(clips, capacity, F, H, W, dev):
    """svdx_frames_u8_in_clips over the B*(F+1) frames of each call's clips, CUDA events, median of 20 per size; the bytes it
    must move, from the shapes: every source pixel of the clip read once, the bf16 rows (64 channels) and the fp32 first frame
    written"""
    from svd_xtend_b200.video_train import ClipSlots, log_normal
    out = []
    for cs in clips:
        slots = ClipSlots(len(cs), F, (H, W), capacity, dev)
        slots.load(cs)
        B = len(cs)
        eps, sig = torch.zeros(B, 3, H, W, device=dev), log_normal(torch.full((B,), 0.5, device=dev), -3.0, 0.5)
        rows = torch.empty(B * (F + 1) * H * W, 64, device=dev, dtype=torch.bfloat16)
        x0 = torch.empty(B, 3, H, W, device=dev)
        for _ in range(3):
            slots.fill(rows, 0, B * (F + 1), eps, sig, x0, 64)
        ts = []
        for _ in range(20):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            slots.fill(rows, 0, B * (F + 1), eps, sig, x0, 64)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = statistics.median(ts)
        read = sum(c.numel() for c in cs) + eps.numel() * 4
        written = rows.numel() * 2 + x0.numel() * 4
        out.append({"source": list(cs[0].shape[1:3]), "ms": round(ms, 4), "bytes_read": read, "bytes_written": written,
                    "gb_per_s": round((read + written) / ms / 1e6, 1)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, choices=(2, 4), default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--forms", default="graphed,eager,latent_only")
    ap.add_argument("--input", choices=("float", "u8", "mixed"), default="float")
    ap.add_argument("--source", default="1080x1920", help="H0xW0 of the uint8 frames (--input u8)")
    ap.add_argument("--sources", default="1080x1920,720x1280,360x640,1080x1440", help="H0xW0 sizes of the clips (--input mixed)")
    ap.add_argument("--encode-chunk", type=int, default=None)
    ap.add_argument("--frozen-dtype", choices=("fp32", "bf16"), default="fp32")
    args = ap.parse_args()
    wanted = [f for f in args.forms.split(",") if f]
    if not wanted or any(f not in ("graphed", "eager", "latent_only", "graphed_u8", "graphed_float") for f in wanted):
        raise SystemExit(f"--forms: a comma-separated subset of graphed,eager,latent_only,graphed_u8,graphed_float, got {args.forms!r}")
    H0, W0 = (int(v) for v in args.source.lower().split("x"))
    sources = [tuple(int(v) for v in s.lower().split("x")) for s in args.sources.split(",") if s]
    if args.input == "mixed":
        H0, W0 = sources[0]
    if not torch.cuda.is_available():
        raise RuntimeError("bench_video_train.py needs a CUDA device: the step has no CPU fallback")

    from bench import ClockSampler
    from oracle.svd_clip_oracle import CLIP_CONFIG          # the SVD checkpoint's image_encoder/ and vae/ configurations
    from oracle.svd_vae_oracle import VAE_CONFIG
    from scripts.bench_decode import power_limit_w
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.train import FusedAdamW, GraphedStep, ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    from svd_xtend_b200.video_train import VideoTrainStep
    from svd_xtend_b200.workload import BENCH_CONFIGS, SVD_CONFIG, edm_loss, synthetic_batch

    dev = torch.device("cuda", 0)
    cfg = BENCH_CONFIGS[args.config]
    F, H, W = cfg["frames"], 8 * cfg["h"], 8 * cfg["w"]
    steps, warmup = max(args.steps, 1), max(args.warmup, 1)
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        vae = AutoencoderKLTemporalDecoder(**VAE_CONFIG)
        clip = CLIPVisionModelWithProjection(**CLIP_CONFIG)
    for m in (unet, vae, clip):
        m.to(dev).requires_grad_(False)
    if args.frozen_dtype == "bf16":             # train_svd.py:665-673
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
    opt = FusedAdamW(arena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
    g = torch.Generator(device="cpu").manual_seed(5)
    if args.input == "u8":
        frames = torch.randint(0, 256, (1, F, H0, W0, 3), generator=g, dtype=torch.uint8).pin_memory()
    else:
        frames = (torch.rand(1, F, 3, H, W, generator=g) * 2 - 1).to(dev)
    if args.input == "mixed":
        clips = [[torch.randint(0, 256, (F, h0, w0, 3), generator=g, dtype=torch.uint8).pin_memory()] for h0, w0 in sources]
        u8_frames = clips[0][0][None]
        float_frames = frames
        frames = clips
        calls = [0]

        def next_clips():
            calls[0] += 1
            return clips[calls[0] % len(clips)]
    memory = {"models": _mem()}

    forms, failed = {}, {}
    kw = dict(frames_shape=(1, F, H, W), conditioning_dropout_prob=0.1, generator=torch.Generator(dev).manual_seed(0),
              source_size=(H0, W0) if args.input == "u8" else None, encode_chunk_size=args.encode_chunk)
    if args.input == "mixed":
        kw["max_source_size"] = (max(s[0] for s in sources), max(s[1] for s in sources))

    def oom(name, e):
        failed[name] = f"OutOfMemoryError: {str(e).splitlines()[0]}"
        torch.cuda.empty_cache()

    if "graphed" in wanted:
        try:
            graphed = VideoTrainStep(unet, vae, clip, opt, **kw)
            forms["graphed"] = (lambda: graphed(next_clips())) if args.input == "mixed" else (lambda: graphed(frames))
        except torch.OutOfMemoryError as e:
            oom("graphed", e)
        memory["graphed_built"] = _mem()
    for name in ("graphed_u8", "graphed_float"):
        if name in wanted:
            if args.input != "mixed":
                raise SystemExit(f"--forms {name} is a comparison of --input mixed")
            try:
                other = dict(kw, max_source_size=None, source_size=(H0, W0) if name == "graphed_u8" else None)
                st = VideoTrainStep(unet, vae, clip, opt, **other)
                x = u8_frames if name == "graphed_u8" else float_frames
                forms[name] = (lambda st=st, x=x: st(x))
            except torch.OutOfMemoryError as e:
                oom(name, e)
            memory[name + "_built"] = _mem()
    if "latent_only" in wanted:
        b = {k: v.to(dev) for k, v in synthetic_batch(1, F, cfg["h"], cfg["w"], seed=1234).items()}

        def latent_step(bb):
            arena.zero_grad()
            pred = unet(bb["sample"], bb["timestep"], bb["encoder_hidden_states"], added_time_ids=bb["added_time_ids"]).sample
            loss = edm_loss(pred.float(), bb["noisy"], bb["latents"], bb["sigmas"])
            loss.backward()
            opt.step()
            return loss
        try:
            latent = GraphedStep(latent_step, b, warmup=3, restore=opt.snapshot_tensors(),
                                 on_restored=lambda: unet.refresh_trainable_operands(shadow_current=True))
            forms["latent_only"] = latent.replay
        except torch.OutOfMemoryError as e:
            oom("latent_only", e)
        memory["latent_only_built"] = _mem()
    if "eager" in wanted:
        eager = VideoTrainStep(unet, vae, clip, opt, cuda_graph=False, **kw)
        forms["eager"] = (lambda: eager(next_clips())) if args.input == "mixed" else (lambda: eager(frames))
    for k in list(forms):
        try:
            for _ in range(warmup):
                forms[k]()
            torch.cuda.synchronize()
        except torch.OutOfMemoryError as e:
            forms.pop(k)
            oom(k, e)
    memory["warmed_up"] = _mem()

    clocks = ClockSampler(0)
    c0 = clocks.count()
    times = {k: [] for k in forms}
    loss = None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        for k, fn in forms.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                loss = fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / steps)
    c1 = clocks.count()
    clk = clocks.stop(c0, c1)
    memory["timed"] = _mem()
    res = {}
    for k, ts in times.items():
        ms = statistics.median(ts)
        res[k] = {"ms_per_step": round(ms, 3), "frames_per_s": round(F * 1e3 / ms, 2), "windows_ms": [round(t, 3) for t in ts]}
    res.update({k: {"failed": v} for k, v in failed.items()})
    kernel = _kernel_alone(clips, kw["max_source_size"], F, H, W, dev) if args.input == "mixed" else None
    print(json.dumps({"metric": "video_train_step", "config": args.config, "frames": F, "pixels": [H, W], "batch": 1,
                      "input": args.input, "source": [H0, W0] if args.input == "u8" else None,
                      "sources": sources if args.input == "mixed" else None, "resize_kernel": kernel, "encode_chunk": args.encode_chunk,
                      "frozen_dtype": args.frozen_dtype, "steps_per_window": steps, "forms": res,
                      "final_loss": None if loss is None else float(loss.float().item()),
                      "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), "memory": memory,
                      "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "sm_clock": clk}))


if __name__ == "__main__":
    main()
