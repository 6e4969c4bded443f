"""world_size-2 gloo test of the sharded EMA plumbing: each rank advances its [lo, hi) slice of the EMA buffer,
ShardedAdamW.gather_ema() assembles every slice in place, and the EMA refuses to be read between a step and a gather."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_ddp_cpu import _free_port


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from svd_xtend_b200.ema import EMAModel
        from svd_xtend_b200.train import ParamArena, ShardedAdamW
        torch.manual_seed(0)
        net = torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.Linear(53, 7), torch.nn.Linear(7, 200))
        net[1].requires_grad_(False)
        arena = ParamArena(net, pad_to=world * 64)
        opt = ShardedAdamW(arena, lr=1e-3)
        ema = EMAModel(net.parameters())
        opt.attach_ema(ema)
        flat = ema._flat
        assert flat.numel() == arena.numel and torch.equal(flat, arena.data)      # the initial EMA is the initial weights
        # what one sharded step leaves behind: this rank's slice advanced, the device counter moved, the rest stale
        flat[opt.lo:opt.hi] = float(rank + 10)
        ema._state[0] += 1
        try:
            ema.copy_to(net.parameters())
            raise AssertionError("copy_to accepted an EMA that was not gathered")
        except RuntimeError:
            pass
        opt.gather_ema()
        n = arena.numel // world
        assert all(torch.all(flat[r * n:(r + 1) * n] == float(r + 10)) for r in range(world))
        sd = ema.state_dict()
        assert sd["optimization_step"] == 1
        ema.copy_to(net.parameters())
        ps = list(net.parameters())
        for p, o in zip(arena.params, arena.offsets):
            assert torch.equal(p.detach().view(-1), flat[o:o + p.numel()])
        assert ema.shadow_params[2] is not None and ema.shadow_params[2].data_ptr() == ps[2].data_ptr()
        assert flat.data_ptr() in [t.data_ptr() for t in opt.snapshot_tensors()]
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_sharded_ema_gather_world2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
