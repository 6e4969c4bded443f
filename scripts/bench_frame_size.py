#!/usr/bin/env python
"""Frame-orientation benchmark on the H100 path, one JSON line.

    python scripts/bench_frame_size.py [--steps K] [--warmup W]

Landscape frames keep every conv width on the row-box tiles (W | 128 or 128 | W); the same frames in portrait put every level
on the im2col path. Both have identical FLOPs, so the ratio is the cost (or gain) of im2col loads:
  1. the config-2 train step of bench.py (seeded default-init SVD UNet, as-scripted trainable set, FusedAdamW, one CUDA graph),
     captured twice in one process: 14 x 320x512 (latent 40x64) and 14 x 512x320 (latent 64x40); the two graphs are replayed
     in alternating windows of K replays, medians of 3;
  2. the VAE encode (no grad, eager) of 14 frames at 576x1024 and at 1024x576, alternating, CUDA events, medians of 3;
  3. the temporal VAE decode (`sampling.decode_latents`, decode_chunk_size 8) of 14 frames at 576x1024 (latent 72x128) and at
     1024x576 (latent 128x72), alternating, CUDA events, medians of 3. In portrait the phase-form upsample stores cross image
     rows (widths 72, 144, 288).
Also reported: the card name, its power limit and SM clock, read in one query. Writes nothing to the source tree.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card_details(index=0):
    """name, power limit (W) and current SM clock (MHz) from one nvidia-smi query"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits", "-i", str(index)],
                           capture_output=True, text=True, timeout=20)
        name, pl, clk = (s.strip() for s in r.stdout.strip().splitlines()[0].split(","))
        return {"card": name, "power_limit_w": float(pl), "sm_clock_mhz": float(clk)}
    except Exception:
        return {"card": torch.cuda.get_device_name(index), "power_limit_w": None, "sm_clock_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.sampling import decode_latents
    from svd_xtend_b200.train import FusedAdamW, GraphedStep, ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    from svd_xtend_b200.workload import SVD_CONFIG, edm_loss, synthetic_batch

    if not torch.cuda.is_available():
        raise RuntimeError("bench_frame_size.py needs a CUDA device: the kernels have no CPU fallback")
    dev = torch.device("cuda", 0)
    steps, warmup = max(args.steps, 1), max(args.warmup, 2)
    frames = 14
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(fn, n):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    # ---- 1. the captured train step, landscape vs portrait
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
    unet.to(dev).requires_grad_(False)
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:   # train_svd.py:761-766
            p.requires_grad_(True)
    unet.train()
    arena = ParamArena(unet)
    unet.attach_arena(arena)
    opt = FusedAdamW(arena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)

    def step(bb):
        arena.zero_grad()
        pred = unet(bb["sample"], bb["timestep"], bb["encoder_hidden_states"], added_time_ids=bb["added_time_ids"]).sample
        loss = edm_loss(pred.float(), bb["noisy"], bb["latents"], bb["sigmas"])
        loss.backward()
        opt.step()
        return loss

    shapes = {"landscape": (40, 64), "portrait": (64, 40)}
    graphs = {}
    for k, (h, w) in shapes.items():
        b = {kk: v.to(dev) for kk, v in synthetic_batch(1, frames, h, w, seed=1234).items()}
        graphs[k] = GraphedStep(step, b, warmup=warmup)
    for g in graphs.values():
        window(g.replay, 2)
    ms = {k: [] for k in graphs}
    for _ in range(3):
        for k, g in graphs.items():
            ms[k].append(window(g.replay, steps))
    finite = bool(torch.isfinite(arena.data).all())
    med = {k: statistics.median(v) for k, v in ms.items()}
    train = {f"{k}_ms": med[k] for k in med}
    train.update({f"{k}_frames_per_s": frames * 1e3 / med[k] for k in med})
    train.update({"portrait_over_landscape": med["portrait"] / med["landscape"], "windows_ms": ms, "finite": finite,
                  "what": (f"config 2 train step in one CUDA graph, {frames} x 320x512 (latent 40x64) vs {frames} x 512x320 "
                           f"(latent 64x40), alternating windows of {steps} replays, medians of 3")})
    del graphs, opt, arena, unet
    gc.collect()
    torch.cuda.empty_cache()

    # ---- 2. the VAE encode, landscape vs portrait
    torch.manual_seed(5)
    with torch.device(dev):
        vae = AutoencoderKLTemporalDecoder(**VAE_CONFIG, with_decoder=True)
    vae.to(dev).eval().requires_grad_(False)
    g = torch.Generator(device="cpu").manual_seed(11)
    xs = {"landscape": (torch.rand(frames, 3, 576, 1024, generator=g) * 2 - 1).to(dev),
          "portrait": (torch.rand(frames, 3, 1024, 576, generator=g) * 2 - 1).to(dev)}
    vms = {k: [] for k in xs}
    with torch.no_grad():
        for x in xs.values():
            vae.encode(x)
        for _ in range(3):
            for k, x in xs.items():
                vms[k].append(window(lambda x=x: vae.encode(x), 3))
    vmed = {k: statistics.median(v) for k, v in vms.items()}
    enc = {f"{k}_ms": vmed[k] for k in vmed}
    enc.update({"portrait_over_landscape": vmed["portrait"] / vmed["landscape"], "windows_ms": vms,
                "what": f"VAE encode of {frames} frames, 576x1024 vs 1024x576, no grad, eager, alternating windows of 3, medians of 3"})
    del xs
    torch.cuda.empty_cache()

    # ---- 3. the temporal VAE decode, landscape vs portrait
    lats = {"landscape": torch.randn(1, frames, 4, 72, 128, generator=g).to(dev),
            "portrait": torch.randn(1, frames, 4, 128, 72, generator=g).to(dev)}
    dms = {k: [] for k in lats}
    with torch.no_grad():
        for lat in lats.values():
            decode_latents(vae, lat, 8)
        for _ in range(3):
            for k, lat in lats.items():
                dms[k].append(window(lambda lat=lat: decode_latents(vae, lat, 8), 3))
    dmed = {k: statistics.median(v) for k, v in dms.items()}
    dec = {f"{k}_ms": dmed[k] for k in dmed}
    dec.update({"portrait_over_landscape": dmed["portrait"] / dmed["landscape"], "windows_ms": dms,
                "what": (f"decode_latents of {frames} frames, decode_chunk_size 8, 576x1024 vs 1024x576, no grad, eager, alternating "
                         f"windows of 3, medians of 3")})

    line = {"metric": "portrait / landscape time of the config-2 train step (same FLOPs)", "value": train["portrait_over_landscape"],
            "unit": "ratio", "higher_is_better": False, "steps": steps, "warmup": warmup,
            "data": "seeded default-init weights, synthetic batch", **card_details(0), "train_step": train, "vae_encode": enc, "vae_decode": dec}
    sys.stdout.flush()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
