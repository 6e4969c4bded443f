"""Checkpoints of the fp32 fused optimizers in torch.optim.AdamW's layout, on CPU arenas (no kernel runs): the layout
functions on odd parameter sizes, every refused dict, the round trip through torch.optim.AdamW, and ShardedAdamW's collective
state_dict at world 3 reloaded at worlds 2 and 1 over gloo."""
import io
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SIZES = [(1,), (63,), (64,), (65,), (7, 11), (130,), (3, 5, 7), (200,)]


class _Net(torch.nn.Module):
    def __init__(self, sizes=SIZES, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(s, generator=g)) for s in sizes])


def _fill(arena, buf, seed):
    """random values at the parameters' arena offsets, zero padding"""
    g = torch.Generator().manual_seed(seed)
    buf.zero_()
    for p, o in zip(arena.params, arena.offsets):
        buf[o:o + p.numel()] = torch.rand(p.numel(), generator=g) + 0.1
    return buf


def _arena_opt(cls=None, seed=0, **kw):
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    arena = ParamArena(_Net(seed=seed), pad_to=kw.pop("pad_to", 64))
    return arena, (cls or FusedAdamW)(arena, **kw)


def test_layout_round_trip_odd_sizes_and_any_range():
    from svd_xtend_b200.train import adamw_state_dict, load_adamw_state_dict
    arena, _ = _arena_opt(pad_to=192)
    assert arena.numel % 192 == 0 and any(o % 64 == 0 and p.numel() % 64 for p, o in zip(arena.params, arena.offsets))
    m, v = _fill(arena, torch.empty(arena.numel), 1), _fill(arena, torch.empty(arena.numel), 2)
    hyper = dict(lr=3e-4, betas=(0.8, 0.99), eps=1e-7, weight_decay=0.05)
    sd = adamw_state_dict(arena, 5, hyper, (m, v))
    assert sd["param_groups"][0]["params"] == list(range(len(SIZES)))
    for i, (p, o) in enumerate(zip(arena.params, arena.offsets)):
        st = sd["state"][i]
        assert st["step"].dtype == torch.float32 and st["step"].dim() == 0 and st["step"].item() == 5
        assert st["exp_avg"].shape == p.shape and torch.equal(st["exp_avg"].reshape(-1), m[o:o + p.numel()])
        assert torch.equal(st["exp_avg_sq"].reshape(-1), v[o:o + p.numel()])
        assert st["exp_avg"].data_ptr() != m.data_ptr()                       # a copy, not a view of the live buffer
    # any [lo, hi) range: whole arena, shard boundaries inside parameters and inside padding
    for lo, hi in [(0, arena.numel), (0, 64), (64, 192), (100, 260), (192, arena.numel), (arena.numel - 64, arena.numel)]:
        m2, v2 = torch.full((hi - lo,), -1.0), torch.full((hi - lo,), -1.0)
        h = load_adamw_state_dict(arena, sd, m2, v2, lo)
        assert torch.equal(m2, m[lo:hi]) and torch.equal(v2, v[lo:hi]), (lo, hi)        # padding written as zero
        assert h["step"] == 5 and h["lr"] == 3e-4 and h["betas"] == (0.8, 0.99) and h["eps"] == 1e-7 and h["weight_decay"] == 0.05


def test_group_keys_follow_torch_and_extra_keys_survive():
    arena, opt = _arena_opt(lr=2e-3)
    opt.param_groups[0]["initial_lr"] = 2e-3                                  # what a torch lr scheduler adds
    g = opt.state_dict()["param_groups"][0]
    ref = torch.optim.AdamW([torch.zeros(1)], lr=2e-3).state_dict()["param_groups"][0]
    assert set(g) == set(ref) | {"initial_lr"} and g["lr"] == 2e-3
    _, fresh = _arena_opt(lr=9.0)
    fresh.load_state_dict(opt.state_dict())
    assert fresh.param_groups[0]["initial_lr"] == 2e-3 and fresh.lr == 2e-3
    assert fresh.param_groups[0]["params"] is fresh.arena.params


def _good_sd(opt, seed=3):
    _fill(opt.arena, opt.m, seed)
    _fill(opt.arena, opt.v, seed + 1)
    opt.state[5] = 4.0
    return opt.state_dict()


def _malformed(sd):
    """name -> a copy of sd broken in one way"""
    def edit(fn):
        d = torch.load(_buf(sd), weights_only=False)
        fn(d)
        return d
    out = {
        "two groups": edit(lambda d: d["param_groups"].append(dict(d["param_groups"][0]))),
        "one parameter too few": edit(lambda d: d["param_groups"][0]["params"].pop()),
        "one parameter too many": edit(lambda d: d["param_groups"][0]["params"].append(len(SIZES))),
        "moment shape": edit(lambda d: d["state"][4].update(exp_avg=torch.zeros(11, 7))),
        "moment numel": edit(lambda d: d["state"][1].update(exp_avg_sq=torch.zeros(64))),
        "integer moment": edit(lambda d: d["state"][0].update(exp_avg=torch.zeros(1, dtype=torch.int32))),
        "missing entry": edit(lambda d: d["state"].pop(6)),
        "missing moment": edit(lambda d: d["state"][2].pop("exp_avg_sq")),
        "different steps": edit(lambda d: d["state"][3].update(step=torch.tensor(5.0))),
        "fractional step": edit(lambda d: [s.update(step=torch.tensor(2.5)) for s in d["state"].values()]),
        "amsgrad": edit(lambda d: d["param_groups"][0].update(amsgrad=True)),
        "maximize": edit(lambda d: d["param_groups"][0].update(maximize=True)),
        "coupled weight decay": edit(lambda d: d["param_groups"][0].update(decoupled_weight_decay=False)),
        "no lr": edit(lambda d: d["param_groups"][0].pop("lr")),
    }
    return out


def _buf(obj):
    b = io.BytesIO()
    torch.save(obj, b)
    b.seek(0)
    return b


@pytest.mark.parametrize("sharded", [False, True])
def test_every_malformed_dict_is_refused_before_any_write(sharded):
    from svd_xtend_b200.train import ShardedAdamW
    _, src = _arena_opt(seed=5)
    sd = _good_sd(src)
    arena, opt = _arena_opt(ShardedAdamW if sharded else None, seed=5, lr=1e-4)
    _fill(arena, opt.m, 11)
    _fill(arena, opt.v, 12)
    opt.state[5] = 9.0
    before = [t.clone() for t in (opt.m, opt.v, opt.state)]
    for name, bad in _malformed(sd).items():
        with pytest.raises(ValueError) as e:
            opt.load_state_dict(bad)
        for t, b in zip((opt.m, opt.v, opt.state), before):
            assert torch.equal(t, b), name
        if name in ("moment shape", "moment numel", "integer moment", "missing entry", "missing moment", "different steps"):
            idx = {"moment shape": 4, "moment numel": 1, "integer moment": 0, "missing entry": 6, "missing moment": 2, "different steps": 3}
            assert f"[{idx[name]}]" in str(e.value), (name, e.value)
    assert opt.lr == 1e-4 and opt.t == 9
    opt.load_state_dict(sd)                                           # the intact dict loads
    assert torch.equal(opt.m, src.m) and torch.equal(opt.v, src.v) and opt.t == 4


def test_floating_moments_are_cast_to_fp32():
    _, src = _arena_opt()
    sd = _good_sd(src)
    for st in sd["state"].values():
        st["exp_avg"] = st["exp_avg"].double()
        st["exp_avg_sq"] = st["exp_avg_sq"].to(torch.bfloat16)
        st["step"] = 4                                               # older torch releases saved a Python number
    _, opt = _arena_opt()
    opt.load_state_dict(sd)
    assert torch.equal(opt.m, src.m)
    assert torch.equal(opt.v, src.v.to(torch.bfloat16).float())
    assert opt.state.dtype == torch.float32 and opt.t == 4


def test_round_trip_through_torch_adamw():
    net = _Net(seed=7)
    params = list(net.parameters())
    ref = torch.optim.AdamW(params, lr=1e-2, betas=(0.85, 0.995), eps=1e-6, weight_decay=0.03)
    g = torch.Generator().manual_seed(8)
    for _ in range(3):
        for p in params:
            p.grad = torch.randn(p.shape, generator=g)
        ref.step()
    sd = ref.state_dict()
    arena, opt = _arena_opt(seed=7, lr=5.0)
    opt.load_state_dict(sd)
    assert opt.t == 3 and opt.lr == 1e-2 and opt.betas == (0.85, 0.995) and opt.eps == 1e-6 and opt.weight_decay == 0.03
    assert opt.state.tolist()[:6] == torch.tensor([1e-2, 0.85, 0.995, 1e-6, 0.03, 3.0]).tolist()
    back = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(s)) for s in SIZES], lr=7.0)
    back.load_state_dict(opt.state_dict())
    out = back.state_dict()
    assert set(out["param_groups"][0]) == set(sd["param_groups"][0])
    assert {k: x for k, x in out["param_groups"][0].items() if k != "params"} == \
           {k: x for k, x in sd["param_groups"][0].items() if k != "params"}
    for i in range(len(SIZES)):
        a, b = out["state"][i], sd["state"][i]
        assert set(a) == set(b)
        for k in a:
            assert torch.equal(a[k], b[k]) and a[k].dtype == b[k].dtype, (i, k)


# ---------------------------------------------------------------------------------------------------------- gloo, world 3 -> 2 -> 1
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _expected(arena, which):
    """the full arena-length moment every world must reproduce: distinct per element, zero padding"""
    out = torch.zeros(arena.numel)
    for p, o in zip(arena.params, arena.offsets):
        out[o:o + p.numel()] = torch.arange(o, o + p.numel(), dtype=torch.float32) * (0.5 if which == 0 else 0.25) + 1 + which
    return out


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from svd_xtend_b200.train import ParamArena, ShardedAdamW
        sub2 = dist.new_group([0, 1])
        ones = [dist.new_group([r]) for r in range(world)]
        arena = ParamArena(_Net(), pad_to=3 * 64)
        opt = ShardedAdamW(arena, lr=2e-4, betas=(0.8, 0.95), weight_decay=0.1)
        assert opt.world == 3
        m_full, v_full = _expected(arena, 0), _expected(arena, 1)
        opt.m.copy_(m_full[opt.lo:opt.hi])                            # each rank holds only its own slice
        opt.v.copy_(v_full[opt.lo:opt.hi])
        opt.state[5] = 12.0
        sd = opt.state_dict()                                          # collective
        assert opt.t == 12 and torch.equal(opt.m, m_full[opt.lo:opt.hi])   # the gather left the shards alone
        for i, (p, o) in enumerate(zip(arena.params, arena.offsets)):
            assert torch.equal(sd["state"][i]["exp_avg"].reshape(-1), m_full[o:o + p.numel()]), i
            assert torch.equal(sd["state"][i]["exp_avg_sq"].reshape(-1), v_full[o:o + p.numel()]), i
            assert sd["state"][i]["step"].item() == 12
        sd = torch.load(_buf(sd), weights_only=True)
        # world 2 (ranks 0 and 1) and world 1 (every rank alone): local loads, each rank's slice exact
        for group, w in ((sub2, 2), (ones[rank], 1)):
            if w == 2 and rank == 2:
                continue
            a = ParamArena(_Net(seed=1), pad_to=w * 64)
            o2 = ShardedAdamW(a, lr=9.0, group=group)
            assert o2.world == w
            o2.load_state_dict(sd)
            mf, vf = _expected(a, 0), _expected(a, 1)
            assert torch.equal(o2.m, mf[o2.lo:o2.hi]) and torch.equal(o2.v, vf[o2.lo:o2.hi]), w
            assert o2.t == 12 and o2.lr == 2e-4 and o2.betas == (0.8, 0.95) and o2.weight_decay == pytest.approx(0.1)
        # the world-2 state_dict (collective over the pair) equals the world-3 one
        if rank < 2:
            a = ParamArena(_Net(seed=1), pad_to=2 * 64)
            o2 = ShardedAdamW(a, group=sub2)
            o2.load_state_dict(sd)
            sd2 = o2.state_dict()
            for i in sd["state"]:
                for k in sd["state"][i]:
                    assert torch.equal(sd2["state"][i][k], sd["state"][i][k]), (i, k)
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_sharded_state_dict_world3_reloads_at_world2_and_world1_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 3, port, q)) for r in range(3)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok"), (2, "ok")], res
