#!/usr/bin/env python
"""EMA-of-the-weights benchmark (train_svd.py --use_ema, :676-679, :1053-1054) on the H100 path, one JSON line.

    python scripts/bench_ema.py [--steps K] [--warmup W]

Two measurements on the same GPU, in the same process:
  1. the config-2 train step of bench.py (seeded default-init SVD UNet, as-scripted trainable set, FusedAdamW, one CUDA graph)
     captured twice, plain and with an EMA of the whole model attached to the optimizer (FusedAdamW.attach_ema: the EMA of the
     fp32 masters is updated in the AdamW pass); the two graphs are replayed in alternating windows of K replays, medians of 3;
  2. EMAModel.step(unet.parameters()) over the same model: the reference's per-tensor loop (oracle/svd_ema_oracle.py, the
     restatement of diffusers' foreach=False step) against svd_xtend_b200.ema.EMAModel (one tick + one multi-tensor launch),
     host enqueue to device completion, alternating windows, medians of 2.
Also reported: the HBM bytes each form needs, counted from shapes, the card name and its power limit. Writes nothing to the
source tree.
"""
import argparse
import gc
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.bench_decode import power_limit_w  # noqa: E402


def ema_bytes(params):
    """HBM bytes of one EMA step, from shapes: the reference loop runs three fp32 tensor ops per trainable tensor
    (s - p: 12 B, (1 - d) * x: 8 B, s.sub_(x): 12 B per element) and copies every frozen tensor (8 B); the drop-in reads s and
    p and writes s (12 B) and copies nothing; inside the fused AdamW pass the EMA adds a read and a write of s (8 B)."""
    n_train = sum(p.numel() for p in params if p.requires_grad)
    n_frozen = sum(p.numel() for p in params if not p.requires_grad)
    return {"reference_loop": 32 * n_train + 8 * n_frozen, "dropin": 12 * n_train, "fused_in_adamw": 8 * n_train,
            "trainable_params": n_train, "frozen_params": n_frozen}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    from oracle.svd_ema_oracle import EMAModel as RefEMA
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.train import FusedAdamW, GraphedStep, ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.workload import BENCH_CONFIGS, SVD_CONFIG, edm_loss, synthetic_batch

    if not torch.cuda.is_available():
        raise RuntimeError("bench_ema.py needs a CUDA device: the EMA kernels have no CPU fallback")
    dev = torch.device("cuda", 0)
    cfg = BENCH_CONFIGS[2]        # two captured steps of config 4 do not fit on one 80 GB card together
    steps, warmup = max(args.steps, 1), max(args.warmup, 2)

    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
    unet.to(dev).requires_grad_(False)
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:   # train_svd.py:761-766
            p.requires_grad_(True)
    unet.train()
    params = list(unet.parameters())
    ema = EMAModel(params)                      # train_svd.py:678 builds it over unet.parameters(), before the arena exists
    arena = ParamArena(unet)
    unet.attach_arena(arena)
    opt = FusedAdamW(arena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
    b = {k: v.to(dev) for k, v in synthetic_batch(1, cfg["frames"], cfg["h"], cfg["w"], seed=1234).items()}

    def step(bb):
        arena.zero_grad()
        pred = unet(bb["sample"], bb["timestep"], bb["encoder_hidden_states"], added_time_ids=bb["added_time_ids"]).sample
        loss = edm_loss(pred.float(), bb["noisy"], bb["latents"], bb["sigmas"])
        loss.backward()
        opt.step()
        return loss

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(fn, n):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    g_plain = GraphedStep(step, b, warmup=warmup)
    opt.attach_ema(ema)
    g_ema = GraphedStep(step, b, warmup=warmup)
    for g in (g_plain, g_ema):
        window(g.replay, 2)
    plain, with_ema = [], []
    for _ in range(3):
        plain.append(window(g_plain.replay, steps))
        with_ema.append(window(g_ema.replay, steps))
    finite = bool(torch.isfinite(ema._flat).all()) and bool(torch.isfinite(arena.data).all())
    step_res = {"step_ms": statistics.median(plain), "step_with_ema_ms": statistics.median(with_ema),
                "ema_in_step_ms": statistics.median(with_ema) - statistics.median(plain),
                "step_ms_windows": plain, "step_with_ema_ms_windows": with_ema, "finite": finite,
                "what": (f"config 2 train step in one CUDA graph, plain vs FusedAdamW.attach_ema, alternating windows of "
                         f"{steps} replays, medians of 3")}
    opt.ema = None
    del g_plain, g_ema, ema
    gc.collect()
    torch.cuda.empty_cache()

    ref = RefEMA(params)
    ours = EMAModel(params)
    ref.step(params)
    ours.step(params)
    ref_ms, ours_ms = [], []
    for _ in range(2):
        ref_ms.append(window(lambda: ref.step(params), 3))
        ours_ms.append(window(lambda: ours.step(params), steps))
    nbytes = ema_bytes(params)
    ema_step = {"reference_loop_ms": statistics.median(ref_ms), "dropin_ms": statistics.median(ours_ms),
                "reference_loop_ms_windows": ref_ms, "dropin_ms_windows": ours_ms,
                "tensors": len(params), "trainable_tensors": sum(1 for p in params if p.requires_grad),
                "what": ("EMAModel.step(unet.parameters()): oracle restatement of diffusers' per-tensor loop (foreach=False) vs "
                         "svd_xtend_b200.ema.EMAModel, host enqueue to device completion, CUDA events, medians of 2 windows")}
    line = {"metric": "EMA of the UNet weights: added ms per captured train step", "value": step_res["ema_in_step_ms"], "unit": "ms",
            "higher_is_better": False, "config": 2, "steps": steps, "warmup": warmup,
            "data": "seeded default-init weights, synthetic batch", "card": torch.cuda.get_device_name(dev),
            "power_limit_w": power_limit_w(0), "train_step": step_res, "ema_step": ema_step, "bytes_per_step": nbytes}
    sys.stdout.flush()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
