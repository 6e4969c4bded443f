#!/usr/bin/env python
"""Time one state_dict() and one load_state_dict() of the fp32 fused optimizers over the config-2 arena (the as-scripted
temporal set of the SVD UNet, 397.6 M parameters), one JSON line.

    python scripts/bench_optim_checkpoint.py [--rounds R]

FusedAdamW and ShardedAdamW at world 1 (its state_dict gathers through the temporary arena-length buffer, here without peers),
host clock around calls that end in a device synchronise, medians of R rounds. Moments are seeded random values. Also
reported: the card name and its power limit. Writes nothing to the source tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.bench_decode import power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    from svd_xtend_b200.train import FusedAdamW, ParamArena, ShardedAdamW
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.workload import SVD_CONFIG

    if not torch.cuda.is_available():
        raise RuntimeError("bench_optim_checkpoint.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    with torch.device(dev):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
    unet.requires_grad_(False)
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:   # train_svd.py:761-766
            p.requires_grad_(True)
    arena = ParamArena(unet)
    n_params = sum(p.numel() for p in arena.params)
    out = {}
    for name, cls in (("FusedAdamW", FusedAdamW), ("ShardedAdamW_world1", ShardedAdamW)):
        opt = cls(arena, lr=1e-5)
        g = torch.Generator(device=dev).manual_seed(7)
        for p, o in zip(arena.params, arena.offsets):
            opt.m[o:o + p.numel()].copy_(torch.randn(p.numel(), generator=g, device=dev))
            opt.v[o:o + p.numel()].copy_(torch.rand(p.numel(), generator=g, device=dev))
        opt.state[5] = 1000.0
        m0 = opt.m.clone()
        save_s, load_s = [], []
        for _ in range(max(args.rounds, 1)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sd = opt.state_dict()
            save_s.append(time.perf_counter() - t0)
            opt.m.zero_()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            opt.load_state_dict(sd)
            torch.cuda.synchronize()
            load_s.append(time.perf_counter() - t0)
            del sd
        assert torch.equal(opt.m, m0) and opt.t == 1000
        out[name] = {"state_dict_s": statistics.median(save_s), "load_state_dict_s": statistics.median(load_s),
                     "state_dict_s_rounds": save_s, "load_state_dict_s_rounds": load_s}
        del opt, m0
        torch.cuda.empty_cache()
    line = {"metric": "optimizer checkpoint of the config-2 arena: seconds per state_dict() / load_state_dict()",
            "params": n_params, "moment_bytes": 8 * n_params, "rounds": args.rounds, "card": torch.cuda.get_device_name(dev),
            "power_limit_w": power_limit_w(0), "host_cpus": os.cpu_count(), **out}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
