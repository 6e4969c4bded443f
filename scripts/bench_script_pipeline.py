#!/usr/bin/env python
"""What the unchanged training script spends on the drop-in VAE and pipeline, one JSON line.

    python scripts/bench_script_pipeline.py [--windows N] [--calls K] [--validations V] [--skip-encode] [--skip-validation]

encode: the script's per-step encode (`tensor_to_vae_latent`, train_svd.py:283-291, called on the B*F clip frames and on the
  noise-augmented first frame) at config 2 (14 x 320 x 512) and config 4 (25 x 576 x 1024), with fp16 and bf16 weights and
  frames: this package's VAE, and the oracle VAE (oracle/svd_vae_oracle.py) under torch autocast in the same dtype (cuDNN) as
  the stand-in for diffusers' eager VAE. Per-step ms = both calls, median over alternating windows of K steps (CUDA events).
validation: one validation of train_svd.py (from_pretrained with the training modules, the call at 14 x 320 x 512, 25 steps,
  decode_chunk_size 8, under fp16 autocast, then del + empty_cache) with a config-2 training UNet resident (fp32 masters,
  gradient checkpointing, enable_cuda_graphs, torch AdamW, three steps taken). Wall time around work that ends in a device
  synchronise, median over V validations, and the peak max_memory_allocated. Next to it: the eager oracle composition
  (oracle/svd_clip_oracle.image_to_video, fp32 UNet, fp16 VAE and CLIP, fp16 autocast) on the same card.
Seeded default-init weights. Prints the card name and power limit. Writes nothing to the source tree.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from bench_decode import power_limit_w  # noqa: E402

GIB = 2.0 ** 30
SVD_SCHEDULER = {"_class_name": "EulerDiscreteScheduler", "beta_end": 0.012, "beta_schedule": "scaled_linear", "beta_start": 0.00085,
                 "clip_sample": False, "interpolation_type": "linear", "num_train_timesteps": 1000, "prediction_type": "v_prediction",
                 "set_alpha_to_one": False, "sigma_max": 700.0, "sigma_min": 0.002, "skip_prk_steps": True, "steps_offset": 1,
                 "timestep_spacing": "leading", "timestep_type": "continuous", "trained_betas": None, "use_karras_sigmas": True}


def _events_ms(fn, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


def _script_step_encode(vae, frames, cond):
    """tensor_to_vae_latent twice, as train_svd.py:948 and :959 call it"""
    b, f = frames.shape[:2]
    lat = vae.encode(frames.flatten(0, 1)).latent_dist.sample()
    lat = lat.reshape(b, f, *lat.shape[1:]) * vae.config.scaling_factor
    c = vae.encode(cond.flatten(0, 1)).latent_dist.sample()
    return lat, c.reshape(b, 1, *c.shape[1:]) * vae.config.scaling_factor


def bench_encode(args, dev):
    from oracle.svd_vae_oracle import VAE_CONFIG, AutoencoderKLTemporalDecoder as Oracle
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(1234)
    with torch.device(dev):
        ours32 = AutoencoderKLTemporalDecoder(**VAE_CONFIG)
        ora32 = Oracle(**VAE_CONFIG)
    ora32.load_state_dict(ours32.state_dict())
    results = []
    for dtype in (torch.float16, torch.bfloat16):
        ours = AutoencoderKLTemporalDecoder(**VAE_CONFIG).to(dev)
        ours.load_state_dict(ours32.state_dict())
        ours.to(dtype).requires_grad_(False)
        ora = Oracle(**VAE_CONFIG).to(dev)
        ora.load_state_dict(ora32.state_dict())
        ora.to(dtype).requires_grad_(False)
        for name, F_, H, W in (("config 2", 14, 320, 512), ("config 4", 25, 576, 1024)):
            g = torch.Generator(dev).manual_seed(F_ + H)
            frames = (torch.rand(1, F_, 3, H, W, device=dev, generator=g) * 2 - 1).to(dtype)
            cond = (frames[:, :1].float() + 0.02 * torch.randn(1, 1, 3, H, W, device=dev, generator=g)).to(dtype)

            def run_ours():
                with torch.no_grad():
                    return _script_step_encode(ours, frames, cond)

            def run_oracle():
                with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
                    return _script_step_encode(ora, frames, cond)
            r = {"workload": name, "frames": F_, "pixels": [H, W], "weights": str(dtype).replace("torch.", "")}
            forms = {"ours": run_ours, "oracle_autocast": run_oracle}
            alive = dict(forms)
            samples = {k: [] for k in forms}
            for k, fn in forms.items():          # warm-up: algorithm selection, first launches
                try:
                    for _ in range(2):
                        fn()
                    torch.cuda.synchronize()
                except torch.OutOfMemoryError:
                    alive.pop(k)
                    r[k] = "out of memory"
                    torch.cuda.empty_cache()
            for _ in range(args.windows):
                for k, fn in alive.items():
                    samples[k].append(_events_ms(fn, args.calls))
            for k in alive:
                r[k] = {"ms_per_step": statistics.median(samples[k]), "windows_ms": samples[k]}
            if "ours" in alive and "oracle_autocast" in alive:
                r["speedup_of_ours"] = r["oracle_autocast"]["ms_per_step"] / r["ours"]["ms_per_step"]
            results.append(r)
            print(json.dumps({"partial": r}), file=sys.stderr, flush=True)
            del frames, cond
            torch.cuda.empty_cache()
        del ours, ora
        torch.cuda.empty_cache()
    return results


def bench_validation(args, dev):
    from PIL import Image
    import numpy as np
    from oracle.svd_clip_oracle import CLIP_CONFIG, CLIPVisionModelWithProjection as OClip, image_to_video
    from oracle.svd_unet_oracle import SVD_CONFIG, UNetSpatioTemporalConditionModel as OUnet, edm_loss, synthetic_batch
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as OVae
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.pipeline import StableVideoDiffusionPipeline
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        vae = AutoencoderKLTemporalDecoder(with_decoder=True)
        enc = CLIPVisionModelWithProjection(**CLIP_CONFIG)
    vae.to(torch.float16).requires_grad_(False)
    enc.to(torch.float16).requires_grad_(False)
    unet.requires_grad_(False)
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:      # train_svd.py:761-766
            p.requires_grad_(True)
    unet.train()
    unet.enable_gradient_checkpointing()
    unet.enable_cuda_graphs()
    opt = torch.optim.AdamW([p for p in unet.parameters() if p.requires_grad], lr=1e-5)
    batch = synthetic_batch(1, 14, 40, 64, seed=7, device=dev)
    for _ in range(3):
        with torch.autocast("cuda", dtype=torch.float16):
            pred = unet(batch["sample"], batch["timestep"], batch["encoder_hidden_states"], batch["added_time_ids"]).sample
        edm_loss(pred.float(), batch["noisy"], batch["latents"], batch["sigmas"]).backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated() / GIB
    image = Image.fromarray(np.random.default_rng(3).integers(0, 256, (320, 512, 3), dtype=np.uint8))
    call = dict(height=320, width=512, num_frames=14, decode_chunk_size=8, motion_bucket_id=127, fps=7, noise_aug_strength=0.02,
                num_inference_steps=25)
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "scheduler"))
        with open(os.path.join(d, "scheduler", "scheduler_config.json"), "w") as f:
            json.dump(SVD_SCHEDULER, f)

        def validation():
            pipe = StableVideoDiffusionPipeline.from_pretrained(d, unet=unet, image_encoder=enc, vae=vae, torch_dtype=torch.float16)
            pipe = pipe.to(dev)
            pipe.set_progress_bar_config(disable=True)
            with torch.autocast("cuda", enabled=True):
                frames = pipe(image, **call).frames[0]
            del pipe
            torch.cuda.empty_cache()
            return frames
        times, peaks = [], []
        for _ in range(args.validations):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            frames = validation()
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
            peaks.append(torch.cuda.max_memory_allocated() / GIB)
    r = {"workload": "validation 14 x 320 x 512, 25 steps, decode_chunk_size 8, fp16 autocast", "resident_training_gib": resident,
         "ours": {"ms_per_validation": statistics.median(times), "runs_ms": times, "peak_gib": max(peaks),
                  "frames": len(frames)}}
    # the eager oracle composition, the training UNet's weights in fp32 under fp16 autocast
    try:
        ou, ov, oc = OUnet(**SVD_CONFIG).to(dev), OVae(with_decoder=True).to(dev), OClip(**CLIP_CONFIG).to(dev)
        ou.load_state_dict(unet.state_dict())
        ov.load_state_dict(vae.state_dict())
        oc.load_state_dict(enc.state_dict())
        ov.to(torch.float16)
        oc.to(torch.float16)
        for m in (ou, ov, oc):
            m.requires_grad_(False).eval()
        x = torch.from_numpy(np.asarray(image).copy()).permute(2, 0, 1)[None].float().div(255).to(dev)
        kw = dict(num_frames=14, num_inference_steps=25, decode_chunk_size=8)
        otimes, opeaks = [], []
        for _ in range(max(1, args.validations - 1)):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            with torch.no_grad(), torch.autocast("cuda", enabled=True):
                image_to_video(ou, ov, oc, x, **kw)
            torch.cuda.synchronize()
            otimes.append((time.perf_counter() - t0) * 1e3)
            opeaks.append(torch.cuda.max_memory_allocated() / GIB)
        r["oracle_eager_fp16_autocast"] = {"ms_per_validation": statistics.median(otimes), "runs_ms": otimes,
                                           "peak_gib_including_both_models": max(opeaks)}
    except Exception as e:      # noqa: BLE001  (reported, not hidden)
        import traceback
        where = traceback.extract_tb(e.__traceback__)[-1]
        r["oracle_eager_fp16_autocast"] = f"not measured: {type(e).__name__}: {str(e)[:200]} ({where.filename}:{where.lineno})"
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5, help="script steps per timed window")
    ap.add_argument("--validations", type=int, default=3)
    ap.add_argument("--skip-encode", action="store_true")
    ap.add_argument("--skip-validation", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_script_pipeline.py needs a CUDA device: the VAE and the pipeline have no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    line = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
            "data": "seeded default-init weights, random frames"}
    if not args.skip_encode:
        line["script_step_encode"] = bench_encode(args, dev)
    if not args.skip_validation:
        line["validation"] = bench_validation(args, dev)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
