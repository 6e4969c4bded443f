#!/usr/bin/env python
"""Temporal VAE decode benchmark: `sampling.decode_latents` on the H100 path, one JSON line.

    python scripts/bench_decode.py [--steps K] [--warmup W] [--no-gpu-baseline]

Two workloads of the reference's inference path, 14 frames each, decode_chunk_size 8: 576x1024 (infer_svd.ipynb cell 3) and
320x512 (train_svd.py validation). Seeded default-init weights, randn latents. Reported per workload: ms per clip (CUDA events
over K calls after W warm-up calls), frames/s, the algorithmic TFLOP counted from shapes (`decoder_flops`, in the reference's
upsample-then-conv form and as this package executes it) and the TFLOP/s, against the same peaks bench.py uses; the card
name and its power limit; and the same decode of the oracle (fp32 weights) under torch bf16 autocast on the same GPU (cuDNN).
Writes nothing to the source tree.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

WORKLOADS = (("infer_svd.ipynb: 14 frames 576x1024, decode_chunk_size 8", 14, 72, 128, 8),
             ("train_svd.py validation: 14 frames 320x512, decode_chunk_size 8", 14, 40, 64, 8))


def decoder_flops(boc, layers, latent_c, out_c, h, w, frames, phase_form):
    """multiply-adds x 2 of the temporal decoder on `frames` frames of latent h x w, counted from shapes: convolutions,
    1x1 shortcuts, the mid-block attention (projections + S x S products). phase_form=False counts Upsample2D as the reference
    executes it (a 3x3 conv on the 2x-upsampled tensor), True as the four 2x2-tap phase convolutions this package runs."""
    H, W = h, w
    macs = H * W * latent_c * boc[-1] * 9

    def stres(cin, cout, hw):
        return hw * (9 * cin * cout + 9 * cout * cout + (cin * cout if cin != cout else 0) + 2 * 3 * cout * cout)

    c = boc[-1]
    macs += layers * stres(c, c, H * W)
    if layers >= 2:                        # MidBlockTemporalDecoder calls its attention only between two resnets
        S = H * W
        macs += S * 4 * c * c + 2 * S * S * c
    rev = list(reversed(boc))
    prev = rev[0]
    for i, c in enumerate(rev):
        for j in range(layers + 1):
            macs += stres(prev if j == 0 else c, c, H * W)
        prev = c
        if i != len(rev) - 1:
            macs += (16 if phase_form else 36) * c * c * H * W
            H, W = 2 * H, 2 * W
    macs += H * W * (9 * boc[0] * out_c + 3 * out_c * out_c)
    return 2.0 * macs * frames


def power_limit_w(index):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-gpu-baseline", action="store_true", help="skip the torch-eager bf16-autocast oracle timing")
    args = ap.parse_args()

    from bench import peaks
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as Oracle, decode_latents as oracle_decode_latents
    from svd_xtend_b200.sampling import decode_latents
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder

    if not torch.cuda.is_available():
        raise RuntimeError("bench_decode.py needs a CUDA device: the decode path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    with torch.device(dev):
        vae = AutoencoderKLTemporalDecoder(with_decoder=True)
    vae.to(dev).requires_grad_(False).eval()
    cfg = vae.config
    sustained, _, _, peak_src = peaks()
    steps, warmup = max(args.steps, 1), max(args.warmup, 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n_warm, n_steps):
        for _ in range(n_warm):
            out = fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n_steps):
            out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n_steps, out

    results = []
    for name, F_, h, w, chunk in WORKLOADS:
        g = torch.Generator(device="cpu").manual_seed(4321)
        lat = (torch.randn(1, F_, cfg.latent_channels, h, w, generator=g) * cfg.scaling_factor).to(dev)
        ms, frames_out = timed(lambda: decode_latents(vae, lat, decode_chunk_size=chunk), warmup, steps)
        fl = lambda phase: decoder_flops(cfg.block_out_channels, cfg.layers_per_block, cfg.latent_channels, cfg.in_channels, h, w, F_, phase) / 1e12
        tf_ref, tf_exe = fl(False), fl(True)
        r = {"workload": name, "frames": F_, "pixels": [8 * h, 8 * w], "decode_chunk_size": chunk, "ms_per_clip": ms,
             "frames_per_s": F_ * 1000.0 / ms, "tflop_reference_form": tf_ref, "tflop_executed": tf_exe,
             "tflops_reference_form": tf_ref / (ms / 1e3), "tflops_executed": tf_exe / (ms / 1e3),
             "fraction_of_peak_executed": tf_exe / (ms / 1e3) / sustained, "finite": bool(torch.isfinite(frames_out).all())}
        del frames_out
        torch.cuda.empty_cache()
        if not args.no_gpu_baseline:
            try:
                with torch.device(dev):
                    ora = Oracle(**{k: getattr(cfg, k) for k in ("in_channels", "latent_channels", "block_out_channels",
                                                                  "layers_per_block", "scaling_factor")}, with_decoder=True)
                ora.load_state_dict(vae.state_dict())
                ora.to(dev).requires_grad_(False).eval()

                def eager():
                    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                        return oracle_decode_latents(ora, lat, decode_chunk_size=chunk)
                ms_e, _ = timed(eager, 1, min(steps, 3))
                r["torch_bf16_autocast"] = {"ms_per_clip": ms_e, "frames_per_s": F_ * 1000.0 / ms_e, "tflops_reference_form": tf_ref / (ms_e / 1e3),
                                            "speedup_of_ours": ms_e / ms}
                del ora
            except Exception as e:      # noqa: BLE001
                r["torch_bf16_autocast"] = {"failed": f"{type(e).__name__}: {e}"}
            torch.cuda.empty_cache()
        results.append(r)
    line = {"metric": "SVD temporal VAE decode frames/sec @ 14x576x1024 (decode_chunk_size 8)", "value": results[0]["frames_per_s"],
            "unit": "frames/s", "higher_is_better": True, "steps": steps, "warmup": warmup, "dtype": "bf16",
            "data": "seeded default-init weights, randn latents x scaling_factor",
            "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
            "peak_tflops": sustained, "peak_source": peak_src, "workloads": results}
    sys.stdout.flush()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
