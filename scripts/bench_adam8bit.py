#!/usr/bin/env python
"""8-bit AdamW benchmark (train_svd.py --use_8bit_adam) on the H100 path, one JSON line.

    python scripts/bench_adam8bit.py [--steps K] [--warmup W]
    python scripts/bench_adam8bit.py --sharded nccl|p2p --world N

--sharded times the sharded forms' update instead (see `sharded()` below); without it:

Measured in one process on one GPU:
  1. the config-2 train step of bench.py (seeded default-init SVD UNet, as-scripted trainable set, one CUDA graph) captured
     twice, with FusedAdamW and with FusedAdamW8bit, replayed in alternating windows of K replays, medians of 3;
  2. the optimizer pass alone on the config-2 arena (tick + update, without the operand refresh of `on_updated`), both forms,
     CUDA events over many launches, with the achieved GB/s against the bytes each form needs (30 B / parameter for fp32
     moments, about 18 B for 8-bit codes);
  3. the script's loop: torch.optim.AdamW (foreach) against AdamW8bit.step on the same parameter list, host enqueue to device
     completion, alternating windows, medians of 3;
  4. memory: optimizer-state bytes counted from shapes, and torch.cuda.max_memory_allocated over one eager config-2 step with the
     as-scripted set and with the whole UNet trainable, under each fused optimizer.
Also reported: the card name and its power limit. Writes nothing to the source tree.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sharded", choices=("nccl", "p2p"), default=None)
    ap.add_argument("--world", type=int, default=1)
    args = ap.parse_args()
    if args.sharded is not None:
        return sharded(args.sharded, args.world)

    from svd_xtend_b200.optim8bit import AdamW8bit, state_bytes, update_bytes
    from svd_xtend_b200.train import FusedAdamW, FusedAdamW8bit, GraphedStep, ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.workload import BENCH_CONFIGS, SVD_CONFIG, edm_loss, synthetic_batch

    if not torch.cuda.is_available():
        raise RuntimeError("bench_adam8bit.py needs a CUDA device: the optimizer kernels have no CPU fallback")
    dev = torch.device("cuda", 0)
    cfg = BENCH_CONFIGS[2]
    steps, warmup = max(args.steps, 1), max(args.warmup, 2)
    b = {k: v.to(dev) for k, v in synthetic_batch(1, cfg["frames"], cfg["h"], cfg["w"], seed=1234).items()}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(fn, n):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    def model(whole: bool):
        torch.manual_seed(1234)
        with torch.device(dev):
            unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        unet.requires_grad_(whole)
        if not whole:
            for n, p in unet.named_parameters():
                if "temporal_transformer_block" in n:      # train_svd.py:761-766
                    p.requires_grad_(True)
        unet.train()
        return unet

    def step_fn(unet, arena, opt):
        def step(bb):
            arena.zero_grad()
            pred = unet(bb["sample"], bb["timestep"], bb["encoder_hidden_states"], added_time_ids=bb["added_time_ids"]).sample
            loss = edm_loss(pred.float(), bb["noisy"], bb["latents"], bb["sigmas"])
            loss.backward()
            opt.step()
            return loss
        return step

    # ---- 1 + 2: captured train step and the optimizer pass alone, both forms, one arena --------------------------------
    unet = model(False)
    arena = ParamArena(unet)
    unet.attach_arena(arena)
    ntrain = arena.numel
    o32 = FusedAdamW(arena, lr=1e-5)
    o8 = FusedAdamW8bit(arena, lr=1e-5)
    for o in (o32, o8):
        o.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
    g32 = GraphedStep(step_fn(unet, arena, o32), b, warmup=warmup, restore=o32.snapshot_tensors() + o8.snapshot_tensors())
    g8 = GraphedStep(step_fn(unet, arena, o8), b, warmup=warmup, restore=o32.snapshot_tensors() + o8.snapshot_tensors())
    for g in (g32, g8):
        window(g.replay, 2)
    t32, t8 = [], []
    for _ in range(3):
        t32.append(window(g32.replay, steps))
        t8.append(window(g8.replay, steps))
    finite = bool(torch.isfinite(arena.data).all())
    train_step = {"fused_adamw_ms": statistics.median(t32), "fused_adamw8bit_ms": statistics.median(t8),
                  "fused_adamw_ms_windows": t32, "fused_adamw8bit_ms_windows": t8, "finite": finite,
                  "what": f"config 2 train step in one CUDA graph, FusedAdamW vs FusedAdamW8bit, alternating windows of {steps} replays, medians of 3"}
    del g32, g8
    gc.collect()
    torch.cuda.empty_cache()
    n8 = sum(p.numel() for p, _, q, _, _ in o8.layout if q)
    nparam = sum(p.numel() for p in arena.params)
    bytes32 = 30.0 * arena.numel                          # the fp32 kernel runs over the whole arena, padding included
    bytes8 = update_bytes(n8, nparam - n8, shadow=True, ema=False)
    arena.grad.normal_()
    for o in (o32, o8):
        o.on_updated = None                               # the update alone: no transposed-operand refresh after it
    launches = 50
    for o in (o32, o8):
        window(lambda: o.step(), 3)
    p32, p8 = [], []
    for _ in range(3):
        p32.append(window(lambda: o32.step(), launches))
        p8.append(window(lambda: o8.step(), launches))
    opt_pass = {"fused_adamw_ms": statistics.median(p32), "fused_adamw8bit_ms": statistics.median(p8),
                "fused_adamw_gbps": bytes32 / statistics.median(p32) / 1e6, "fused_adamw8bit_gbps": bytes8 / statistics.median(p8) / 1e6,
                "fused_adamw_bytes": bytes32, "fused_adamw8bit_bytes": bytes8, "params": nparam, "params_8bit": n8,
                "what": f"optimizer step alone (tick + update, no operand refresh) on the config-2 arena, CUDA events over {launches} launches, medians of 3"}

    # ---- 3: the script's loop ----------------------------------------------------------------------------------------
    params = list(arena.params)
    for p in params:
        p.grad = arena.grad_views[p]
    ref = torch.optim.AdamW(params, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, foreach=True)
    ours = AdamW8bit(params, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    ref.step()
    ours.step()
    s32, s8 = [], []
    for _ in range(3):
        s32.append(window(ref.step, 5))
        s8.append(window(ours.step, 20))
    script = {"torch_adamw_foreach_ms": statistics.median(s32), "adamw8bit_ms": statistics.median(s8),
              "torch_adamw_foreach_ms_windows": s32, "adamw8bit_ms_windows": s8, "tensors": len(params),
              "what": "optimizer.step() over the as-scripted parameter list, host enqueue to device completion, medians of 3 windows"}
    for p in params:
        p.grad = None
    del ref, ours, o32, o8, unet, arena, params
    gc.collect()
    torch.cuda.empty_cache()

    # ---- 4: memory ---------------------------------------------------------------------------------------------------
    memory = {}
    for whole in (False, True):
        for name, cls in (("fused_adamw", FusedAdamW), ("fused_adamw8bit", FusedAdamW8bit)):
            torch.cuda.reset_peak_memory_stats(dev)
            unet = model(whole)
            arena = ParamArena(unet)
            unet.attach_arena(arena)
            opt = cls(arena, lr=1e-5)
            opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
            step_fn(unet, arena, opt)(b)
            torch.cuda.synchronize()
            key = ("whole_unet_" if whole else "as_scripted_") + name
            memory[key + "_max_allocated_gb"] = torch.cuda.max_memory_allocated(dev) / 1e9
            numels = [p.numel() for p in arena.params]
            memory[("whole_unet" if whole else "as_scripted") + "_params"] = sum(numels)
            memory[key + "_state_gb"] = (8 * sum(numels) if cls is FusedAdamW else state_bytes(numels)) / 1e9
            del unet, arena, opt
            gc.collect()
            torch.cuda.empty_cache()

    line = {"metric": "8-bit AdamW: config-2 captured train step", "value": train_step["fused_adamw8bit_ms"], "unit": "ms",
            "higher_is_better": False, "config": 2, "steps": steps, "warmup": warmup, "trainable_params": ntrain,
            "data": "seeded default-init weights, synthetic batch", "card": torch.cuda.get_device_name(dev),
            "power_limit_w": power_limit_w(0), "train_step": train_step, "optimizer_pass": opt_pass, "script_loop": script,
            "memory": memory}
    sys.stdout.flush()
    print(json.dumps(line), flush=True)


HBM_TBPS = 3.35     # H100 SXM data-sheet HBM3 bandwidth


def sharded(form: str, world: int):
    """One rank's optimizer update of ShardedAdamW8bit (form "nccl") or P2PShardedAdamW8bit ("p2p") at world size `world`, on the
    config-2 arena (the as-scripted trainable set, 397,620,480 parameters) and on the whole UNet, CUDA events over many launches.

    world 1 times the real optimizer's step(). At world N > 1 the N ranks are emulated on one device: rank 0's optimizer is built
    over its own arena with torch.distributed stood in for, and the peer pointer lists point at local buffers, one gradient and
    one shadow slice per rank (only the owned slice [lo, hi) of a peer arena is ever addressed, so each peer buffer covers just
    that slice). These are LOCAL-HBM timings, not NVLink: the peers' gradient reads and shadow writes go to this card's memory.
    "p2p" times the one-kernel step (tick + svdx_adamw8bit_p2p, the fences left out); "nccl" times the svdx_adamw8bit_step launch
    over rank 0's sub-jobs only (tick + update; the reduce-scatter and the all-gather are not measured). Bytes are counted from
    shapes (svd_xtend_b200.optim8bit.update_bytes: the local HBM traffic, the emulated peer traffic included)."""
    from types import SimpleNamespace

    import torch.distributed as dist

    from oracle.svd_unet_oracle import SVD_CONFIG
    from svd_xtend_b200 import train
    from svd_xtend_b200.optim8bit import update_bytes
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel

    if not torch.cuda.is_available():
        raise RuntimeError("bench_adam8bit.py needs a CUDA device: the optimizer kernels have no CPU fallback")
    if not 1 <= world <= 16:
        raise ValueError("--world is 1 .. 16")
    dev = torch.device("cuda", 0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cls = train.P2PShardedAdamW8bit if form == "p2p" else train.ShardedAdamW8bit
    out = {}
    for which in ("as_scripted", "whole_unet"):
        with torch.device("meta"):
            m = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        shapes = [p.shape for n, p in m.named_parameters() if which == "whole_unet" or "temporal_transformer_block" in n]
        net = torch.nn.Module()
        net.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.empty(s, device=dev).normal_(0, 0.02)) for s in shapes])
        arena = train.ParamArena(net, pad_to=world * 256, block=256)
        arena.grad.normal_()
        peers = None
        saved = train.dist, train.map_peer_buffers
        if world > 1:
            shard = arena.numel // world
            peers = [(torch.empty(shard, device=dev).normal_(), torch.empty(shard, device=dev, dtype=torch.bfloat16))
                     for _ in range(world - 1)]
            train.dist = SimpleNamespace(is_initialized=lambda: True, get_world_size=lambda group=None: world,
                                         get_rank=lambda group=None: 0, get_backend=lambda group=None: "nccl",
                                         ReduceOp=dist.ReduceOp, all_reduce=lambda *a, **k: None)
            # rank 0 owns [0, shard): a peer slice buffer is addressed from the peer arena's base, here its own start
            train.map_peer_buffers = lambda t, group=None: [t.data_ptr()] + [(g if t.dtype == torch.float32 else s).data_ptr()
                                                                              for g, s in peers]
        try:
            opt = cls(arena, lr=1e-5)
            if form == "nccl" and world > 1:
                def fn():
                    opt._launch(1.0 / world, None)
            else:
                def fn():
                    opt.step()
            for _ in range(3):
                fn()
            launches = 20
            times = []
            for _ in range(3):
                torch.cuda.synchronize()
                e0.record()
                for _ in range(launches):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) / launches)
        finally:
            train.dist, train.map_peer_buffers = saved
        n8 = sum(n for _, _, n, q, _, _ in opt.subjobs if q)
        n32 = sum(n for _, _, n, q, _, _ in opt.subjobs if not q)
        nbytes = update_bytes(n8, n32, shadow=True, ema=False, world=world if form == "p2p" else 1)
        ms = statistics.median(times)
        out[which] = {"ms": ms, "ms_windows": times, "params": sum(p.numel() for p in arena.params), "rank_params": n8 + n32,
                      "rank_params_8bit": n8, "bytes": nbytes, "gbps": nbytes / ms / 1e6,
                      "share_of_hbm_peak": nbytes / ms / 1e6 / (HBM_TBPS * 1e3), "finite": bool(torch.isfinite(arena.data).all())}
        del opt, arena, net, peers, m
        gc.collect()
        torch.cuda.empty_cache()
    what = ("the optimizer's step()" if world == 1 else
            "rank 0's launch of N emulated ranks on one card (LOCAL-HBM timing, not NVLink): "
            + ("tick + svdx_adamw8bit_p2p" if form == "p2p" else "tick + svdx_adamw8bit_step over its sub-jobs, without the NCCL collectives"))
    line = {"metric": f"sharded 8-bit AdamW ({form}) update, one rank of {world}", "value": out["as_scripted"]["ms"], "unit": "ms",
            "higher_is_better": False, "form": form, "world": world, "what": what + ", CUDA events over 20 launches, medians of 3",
            "hbm_peak_tbps": HBM_TBPS, "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), **out}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
