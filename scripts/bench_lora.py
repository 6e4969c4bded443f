#!/usr/bin/env python
"""LoRA at sampling time on the H100 path: what the side path costs a denoising step, and what fusing costs. One JSON line.

    python scripts/bench_lora.py [--steps K] [--warmup W]

SVD configuration, seeded default-init weights in bf16 (nothing downloaded), 14 frames at 576 × 1024 (latents 72 × 128) with
classifier-free guidance (a 2-clip UNet batch). Measurements, in one process on one GPU:
  1. one graphed denoising step (VideoLatentSampler's captured step) in four states, each its own UNet with the same base
     weights: base; rank-64 adapter on to_q / to_k / to_v / to_out.0 (256 linears), unfused; rank-4 adapter, unfused; the
     rank-64 adapter fused. The four graphs are replayed in alternating windows of K replays, CUDA events, medians of 3;
  2. fuse_lora + unfuse_lora of the rank-64 adapter (two svdx_lora_merge launches), host enqueue to device completion, against
     the per-layer torch merge PEFT does (`W += s * (B @ A)` in a Python loop, then the same with -s), alternating windows,
     medians of 3.
Also reported: the merge's operations and HBM bytes counted from shapes, the card name and its power limit. Writes nothing to
the source tree.
"""
import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.bench_decode import power_limit_w  # noqa: E402

TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    from svd_xtend_b200 import lora
    from svd_xtend_b200.sampling import VideoLatentSampler
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.workload import SVD_CONFIG

    if not torch.cuda.is_available():
        raise RuntimeError("bench_lora.py needs a CUDA device: the LoRA merge and the UNet have no CPU fallback")
    dev = torch.device("cuda", 0)
    steps, warmup = max(args.steps, 1), max(args.warmup, 1)
    frames, h, w = 14, 576 // 8, 1024 // 8

    torch.manual_seed(1234)
    with torch.device(dev):
        base = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
    base.to(dev, torch.bfloat16).requires_grad_(False).eval()
    sd = base.state_dict()

    def adapted(r, fuse):
        with torch.device(dev):
            u = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        u.to(dev, torch.bfloat16).load_state_dict(sd)
        g = torch.Generator(dev).manual_seed(r)
        u.add_adapter(SimpleNamespace(r=r, lora_alpha=r, init_lora_weights="gaussian", target_modules=TARGETS))
        with torch.no_grad():
            for m in u.modules():
                if hasattr(m, "lora_B"):
                    m.lora_B["default"].weight.normal_(0, 0.02, generator=g)
        u.requires_grad_(False).eval()
        if fuse:
            u.fuse_lora()
        return u

    states = {"base": base, "r64_unfused": adapted(64, False), "r4_unfused": adapted(4, False), "r64_fused": adapted(64, True)}
    n_layers = sum(1 for m in states["r64_unfused"].modules() if hasattr(m, "lora_A"))

    g = torch.Generator(dev).manual_seed(7)
    lat = torch.randn(1, 4, h, w, generator=g, device=dev)
    emb = torch.randn(1, 1, SVD_CONFIG["cross_attention_dim"], generator=g, device=dev)
    noise = torch.randn(1, frames, 4, h, w, generator=g, device=dev)
    samplers = {}
    for name, u in states.items():
        s = VideoLatentSampler(u)
        for _ in range(warmup):       # the first call captures the step; the rest replay it
            s(lat, emb, num_frames=frames, num_inference_steps=1, noise=noise)
        samplers[name] = s

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(fn, n):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    times = {k: [] for k in samplers}
    for _ in range(3):
        for k, s in samplers.items():
            times[k].append(window(s._graph.replay, steps))
    step = {k: statistics.median(v) for k, v in times.items()}
    finite = all(bool(torch.isfinite(s._st["latents"]).all()) for s in samplers.values())

    # fuse + unfuse of the rank-64 adapter against PEFT's per-layer torch merge
    u = states["r64_unfused"]
    layers = [m for m in u.modules() if hasattr(m, "lora_A")]
    items = [(m.base_layer.weight, [(m.lora_A["default"].weight, m.lora_B["default"].weight, 1.0)]) for m in layers]
    flops, nbytes = lora.merge_cost(items)

    @torch.no_grad()
    def peft_merge():
        for sgn in (1.0, -1.0):
            for m in layers:
                m.base_layer.weight.data += (m.lora_B["default"].weight @ m.lora_A["default"].weight) * (sgn * m.scaling["default"])

    def ours():
        u.fuse_lora()
        u.unfuse_lora()

    ours()
    peft_merge()
    ours_ms, peft_ms = [], []
    for _ in range(3):
        ours_ms.append(window(ours, steps))
        peft_ms.append(window(peft_merge, steps))
    fuse = {"fuse_plus_unfuse_ms": statistics.median(ours_ms), "peft_loop_ms": statistics.median(peft_ms),
            "fuse_plus_unfuse_ms_windows": ours_ms, "peft_loop_ms_windows": peft_ms, "layers": n_layers,
            "merge_flops_per_fuse": flops, "merge_bytes_per_fuse": nbytes,
            "merge_tbps": 2 * nbytes / (statistics.median(ours_ms) * 1e-3) / 1e12,
            "what": ("fuse_lora + unfuse_lora of the rank-64 adapter (two svdx_lora_merge launches, bf16 base, bf16 factors) vs the "
                     "per-layer torch loop W += s * (B @ A) then with -s, host enqueue to device completion, CUDA events, "
                     f"alternating windows of {steps}, medians of 3")}
    side64 = step["r64_unfused"] - step["base"]
    line = {"metric": "LoRA rank-64 side path: added ms per graphed denoising step (14 x 576 x 1024, CFG)", "value": side64,
            "unit": "ms", "higher_is_better": False, "steps": steps, "warmup": warmup,
            "data": "seeded default-init SVD UNet, bf16 weights, synthetic latents", "card": torch.cuda.get_device_name(dev),
            "power_limit_w": power_limit_w(0),
            "denoising_step_ms": step, "denoising_step_ms_windows": times, "finite": finite,
            "side_path_share_r64": side64 / step["r64_unfused"], "side_path_share_r4": (step["r4_unfused"] - step["base"]) / step["r4_unfused"],
            "fuse_pays_after_steps": (fuse["fuse_plus_unfuse_ms"] / side64) if side64 > 0 else None,
            "fuse": fuse}
    sys.stdout.flush()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
