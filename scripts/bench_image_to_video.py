#!/usr/bin/env python
"""Image-to-video benchmark on the H100 path, one JSON line.

    python scripts/bench_image_to_video.py --stage clip [--steps K] [--warmup W] [--no-gpu-baseline]
    python scripts/bench_image_to_video.py --stage all  [--steps K] [--warmup W]

--stage clip: `clip.encode_image` (resize + normalise + the ViT-H/14 image encoder) from 576x1024 (infer_svd.ipynb) and
  320x512 (train_svd.py) images at B = 1 and 2: ms per image (CUDA events over K calls after W warm-up calls), TFLOP/s from
  the shape-counted `clip_flops`, and the oracle (fp32 weights) under torch bf16 autocast on the same GPU — transformers'
  CLIPVisionModelWithProjection in bf16 too where transformers is importable.
--stage all: `ImageToVideoPipeline` for the notebook's 14 x 576x1024 clip (25 steps, decode_chunk_size 8), whole call and
  broken into CLIP / VAE encode / sampling / decode.
Seeded default-init weights. Prints the card name and its power limit with the numbers. Writes nothing to the source tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench_decode import power_limit_w  # noqa: E402

CLIP_WORKLOADS = ((576, 1024, 1), (576, 1024, 2), (320, 512, 1), (320, 512, 2))


def _timer():
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n_warm, n_steps):
        out = None
        for _ in range(n_warm):
            out = fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n_steps):
            out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n_steps, out
    return timed


def stage_clip(args, dev):
    from oracle.svd_clip_oracle import CLIP_CONFIG, CLIPVisionModelWithProjection as Oracle, encode_image as oracle_encode
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection, clip_flops, encode_image
    torch.manual_seed(1234)
    with torch.device(dev):
        enc = CLIPVisionModelWithProjection(**CLIP_CONFIG)
    enc.requires_grad_(False).eval()
    timed = _timer()
    gflop = clip_flops(CLIP_CONFIG)["total"] / 1e9
    ora = hf = None
    if not args.no_gpu_baseline:
        with torch.device(dev):
            ora = Oracle(**CLIP_CONFIG)
        ora.load_state_dict(enc.state_dict())
        ora.requires_grad_(False).eval()
        try:
            import transformers
            with torch.device(dev):
                hf = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**CLIP_CONFIG))
            hf.load_state_dict(enc.state_dict())
            hf.to(torch.bfloat16).requires_grad_(False).eval()
        except Exception:       # noqa: BLE001
            hf = None
    results = []
    for H, W, B in CLIP_WORKLOADS:
        x = torch.rand(B, 3, H, W, device=dev, generator=torch.Generator(dev).manual_seed(H + W + B)) * 2 - 1
        with torch.no_grad():
            ms, out = timed(lambda: encode_image(enc, x), args.warmup, args.steps)
        r = {"image": [H, W], "batch": B, "ms_per_call": ms, "ms_per_image": ms / B, "gflop_per_image": gflop,
             "tflops": gflop * B / ms, "finite": bool(torch.isfinite(out).all())}
        if ora is not None:
            def eager():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                    return oracle_encode(ora, x)
            ms_e, _ = timed(eager, 1, args.steps)
            r["oracle_bf16_autocast"] = {"ms_per_image": ms_e / B, "speedup_of_ours": ms_e / ms}
        if hf is not None:
            from oracle.svd_clip_oracle import clip_input

            def trans():
                with torch.no_grad():
                    return hf(pixel_values=clip_input(x).to(torch.bfloat16)).image_embeds
            ms_t, _ = timed(trans, 1, args.steps)
            r["transformers_bf16"] = {"ms_per_image": ms_t / B, "speedup_of_ours": ms_t / ms}
        results.append(r)
    return {"metric": "CLIP image encoder (encode_image) ms per image @ 576x1024, B=1", "value": results[0]["ms_per_image"],
            "unit": "ms", "higher_is_better": False, "workloads": results}


def stage_all(args, dev):
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from oracle.svd_unet_oracle import SVD_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection, encode_image
    from svd_xtend_b200.pipeline import ImageToVideoPipeline
    from svd_xtend_b200.sampling import decode_latents
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        vae = AutoencoderKLTemporalDecoder(with_decoder=True)
        enc = CLIPVisionModelWithProjection(**CLIP_CONFIG)
    for m in (unet, vae, enc):
        m.requires_grad_(False).eval()
    pipe = ImageToVideoPipeline(unet, vae, enc)
    F_, H, W, steps_inf, chunk = 14, 576, 1024, 25, 8
    image = torch.rand(1, 3, H, W, device=dev, generator=torch.Generator(dev).manual_seed(7))
    timed = _timer()
    kw = dict(num_frames=F_, num_inference_steps=steps_inf, decode_chunk_size=chunk)
    ms_total, frames = timed(lambda: pipe(image, generator=torch.Generator(dev).manual_seed(1), **kw).frames, args.warmup, args.steps)
    x = image * 2 - 1
    with torch.no_grad():
        ms_clip, emb = timed(lambda: encode_image(enc, x), 1, args.steps)
        ms_vae, lat0 = timed(lambda: vae.encode(x).latent_dist.mode(), 1, args.steps)
        noise = torch.randn(1, F_, 4, H // 8, W // 8, device=dev)
        ms_samp, lat = timed(lambda: pipe.sampler(lat0, emb.unsqueeze(1), num_frames=F_, num_inference_steps=steps_inf, noise=noise), 1, args.steps)
        ms_dec, _ = timed(lambda: decode_latents(vae, lat, chunk), 1, args.steps)
    r = {"frames": F_, "pixels": [H, W], "num_inference_steps": steps_inf, "decode_chunk_size": chunk, "ms_per_video": ms_total,
         "stages_ms": {"clip": ms_clip, "vae_encode": ms_vae, "sampling": ms_samp, "decode": ms_dec},
         "finite": bool(torch.isfinite(frames).all())}
    return {"metric": "image-to-video ms per 14x576x1024 video (25 steps, decode_chunk_size 8)", "value": ms_total, "unit": "ms",
            "higher_is_better": False, "workloads": [r]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", choices=("clip", "all"), default="clip")
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=None)
    ap.add_argument("--no-gpu-baseline", action="store_true", help="--stage clip: skip the oracle / transformers timings")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_image_to_video.py needs a CUDA device: the encoder and the pipeline have no CPU fallback")
    args.steps = max(1, args.steps if args.steps is not None else (10 if args.stage == "clip" else 1))
    args.warmup = max(1, args.warmup if args.warmup is not None else (3 if args.stage == "clip" else 1))
    dev = torch.device("cuda", 0)
    line = stage_clip(args, dev) if args.stage == "clip" else stage_all(args, dev)
    line.update(steps=args.steps, warmup=args.warmup, dtype="bf16", data="seeded default-init weights, random images",
                card=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(0))
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
