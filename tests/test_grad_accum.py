"""Gradient accumulation and global gradient-norm clipping without a GPU: argument validation of
VideoTrainStep(gradient_accumulation_steps=...) and of the fused optimizers' max_grad_norm, the clip-coefficient rule of
svdx_clip_coef restated in torch against torch.nn.utils.clip_grad_norm_, and the sharded optimizers' norm combination (each rank's
fp64 partial, summed over the ranks, then the 1 / N scale) at world size 2 over gloo."""
import math
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _cpu_arena():
    from svd_xtend_b200.train import ParamArena
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.Linear(5, 3))
    return ParamArena(net)


@pytest.mark.parametrize("k", [0, -1, 1.0, 2.5, "2", True, None])
def test_gradient_accumulation_steps_must_be_a_positive_int(k):
    from svd_xtend_b200.video_train import VideoTrainStep
    with pytest.raises(ValueError, match="gradient_accumulation_steps"):
        VideoTrainStep(None, None, None, None, frames_shape=(1, 4, 64, 64), gradient_accumulation_steps=k)


@pytest.mark.parametrize("cls", ["FusedAdamW", "FusedAdamW8bit", "ShardedAdamW", "P2PShardedAdamW"])
@pytest.mark.parametrize("bad", [0.0, -1.0, float("inf"), float("nan"), "x", True])
def test_max_grad_norm_must_be_positive_and_finite(cls, bad):
    from svd_xtend_b200 import train
    with pytest.raises(ValueError, match="max_grad_norm"):
        getattr(train, cls)(_cpu_arena(), max_grad_norm=bad)


def test_max_grad_norm_setter():
    from svd_xtend_b200.train import FusedAdamW
    plain = FusedAdamW(_cpu_arena())
    assert plain.max_grad_norm is None
    with pytest.raises(ValueError, match="without clipping"):
        plain.max_grad_norm = 1.0
    with pytest.raises(ValueError, match="without clipping"):
        plain.grad_norm
    opt = FusedAdamW(_cpu_arena(), max_grad_norm=2.0)
    assert opt.max_grad_norm == 2.0 and opt.grad_norm.dim() == 0 and opt.grad_norm.dtype == torch.float32
    addr = opt._max_norm_dev.data_ptr()
    opt.max_grad_norm = 0.5
    assert opt.max_grad_norm == 0.5 and opt._max_norm_dev.item() == 0.5 and opt._max_norm_dev.data_ptr() == addr
    for bad in (0.0, -2.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="max_grad_norm"):
            opt.max_grad_norm = bad
    assert opt.max_grad_norm == 0.5


def clip_coef_rule(sumsq: torch.Tensor, max_norm: float, scale: float = 1.0):
    """svdx_clip_coef in torch ops: (total_norm, coef) from the fp64 sum of squares"""
    total = torch.sqrt(sumsq.double()).float() * torch.tensor(scale, dtype=torch.float32)
    coef = torch.reciprocal(total + torch.tensor(1e-6, dtype=torch.float32)) * torch.tensor(max_norm, dtype=torch.float32)
    coef = torch.where(coef > 1, torch.ones_like(coef), coef)          # keeps NaN, as torch.clamp(max=1) does
    return total, coef


@pytest.mark.parametrize("case", ["below", "at", "above", "inf", "nan"])
def test_clip_coefficient_rule_matches_clip_grad_norm(case):
    """the coefficient svdx_clip_coef applies, from torch's own total norm, scales the gradient exactly as clip_grad_norm_ does,
    NaN and infinite norms included; the fp64 sum-of-squares norm is torch's norm to within 1e-6"""
    g = torch.Generator().manual_seed(3)
    grads = [torch.randn(37, 11, generator=g), torch.randn(129, generator=g)]
    norm = math.sqrt(sum(float((x.double() ** 2).sum()) for x in grads))
    max_norm = {"below": 2 * norm, "at": norm, "above": norm / 3, "inf": 1.0, "nan": 1.0}[case]
    if case == "inf":
        grads[0][3, 4] = float("inf")
    if case == "nan":
        grads[1][7] = float("nan")
    params = [torch.nn.Parameter(torch.zeros_like(x)) for x in grads]
    for p, x in zip(params, grads):
        p.grad = x.clone()
    total = torch.nn.utils.clip_grad_norm_(params, max_norm)
    sumsq = sum((x.double() ** 2).sum() for x in grads)
    mine, coef = clip_coef_rule(sumsq, max_norm)
    _, coef_from_torch_norm = clip_coef_rule(total.double() ** 2, max_norm)
    if case == "nan":
        assert math.isnan(total.item()) and math.isnan(mine.item()) and math.isnan(coef.item())
    elif case == "inf":
        assert math.isinf(total.item()) and math.isinf(mine.item()) and coef.item() == 0.0
    else:
        assert abs(mine.item() - total.item()) <= 1e-6 * total.item()
        assert (coef.item() == 1.0) == (case == "below")
        # the rule itself, fed torch's norm, gives torch's scaled gradients bit for bit
        coef_t = torch.clamp(max_norm / (total + 1e-6), max=1.0)
        assert torch.equal(coef_t, coef_from_torch_norm.float())
    for p, x in zip(params, grads):
        torch.testing.assert_close(p.grad, x * coef_from_torch_norm.float(), rtol=0, atol=0, equal_nan=True)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from svd_xtend_b200.train import ParamArena, ShardedAdamW, all_reduce_sumsq
        torch.manual_seed(0)
        net = torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.Linear(53, 11))
        arena = ParamArena(net, pad_to=world * 64)
        opt = ShardedAdamW(arena, max_grad_norm=1.0)
        grads = [torch.randn(arena.numel, generator=torch.Generator().manual_seed(10 + r)) for r in range(world)]
        arena.grad.copy_(grads[rank])
        shard = opt.reduce_scatter_grads()         # this rank's slice of the summed gradient
        opt._sumsq[0] = (shard.double() ** 2).sum()
        all_reduce_sumsq(opt._sumsq[:1], opt.world, opt.group)
        total, _ = clip_coef_rule(opt._sumsq[0], 1.0, 1.0 / opt.world)
        mean = sum(grads) / world
        q.put((rank, total.item(), torch.linalg.vector_norm(mean.double()).item()))
    finally:
        dist.destroy_process_group()


def test_sharded_norm_is_the_norm_of_the_mean_gradient():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_worker, args=(world, _free_port(), q), nprocs=world, join=True)
    got = sorted(q.get() for _ in range(world))
    assert got[0][1] == got[1][1], "every rank computes the same norm"
    for _, total, ref in got:
        assert abs(total - ref) <= 1e-6 * ref, (total, ref)
