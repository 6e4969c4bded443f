"""GPU tests of the fp32 fused optimizers' checkpoints on the tiny UNet's arena: a resumed run continues bit for bit (eager, inside
a captured GraphedStep with the state loaded in place, with an attached EMA), the dicts interchange with torch.optim.AdamW, and
ShardedAdamW / P2PShardedAdamW at world 1 resume from their own dicts and from FusedAdamW's. Gradients are seeded per step
rather than taken from a backward: the backward's fp32 atomics are not bit-reproducible, and what is resumed is the optimizer."""
import io

import pytest
import torch

from test_unet_gpu import DEV, _build, _train_filter

pytestmark = pytest.mark.gpu


def _cls(name):
    from svd_xtend_b200.train import FusedAdamW, P2PShardedAdamW, ShardedAdamW
    return {"fused": FusedAdamW, "sharded": ShardedAdamW, "p2p": P2PShardedAdamW}[name]


def _model(seed):
    from oracle.svd_unet_oracle import TINY_CONFIG
    _, m = _build(TINY_CONFIG, seed=seed)
    _train_filter(m)
    m.train()
    return m


def _setup(model, name, **kw):
    from svd_xtend_b200.train import ParamArena
    arena = ParamArena(model)
    model.attach_arena(arena)
    opt = _cls(name)(arena, **(kw or dict(lr=2e-3, weight_decay=1e-2)))
    opt.on_updated = lambda: model.refresh_trainable_operands(shadow_current=True)
    return arena, opt


# hyperparameters of an optimizer that is about to load a dict: all of them must come from the dict
OTHER = dict(lr=9.0, betas=(0.5, 0.6), eps=1e-3, weight_decay=0.5)


def _flat_grad(arena, t):
    """step t's gradient arena: seeded per parameter, magnitudes 1e-3 .. 1e-1, zero padding"""
    g = torch.Generator(device=DEV).manual_seed(1000 + t)
    out = torch.zeros_like(arena.grad)
    for i, (p, o) in enumerate(zip(arena.params, arena.offsets)):
        out[o:o + p.numel()] = torch.randn(p.numel(), generator=g, device=DEV) * 10.0 ** (i % 3 - 3)
    return out


def _lr(t):
    return 2e-3 / (1 + 0.1 * t)


def _steps(opt, arena, ts):
    for t in ts:
        opt.lr = _lr(t)
        arena.grad.copy_(_flat_grad(arena, t))
        opt.step()
    torch.cuda.synchronize()


def _save(obj):
    b = io.BytesIO()
    torch.save(obj, b)
    b.seek(0)
    return b


def _assert_same(a, b, what=""):
    for x, y, k in zip(a, b, ("masters", "m", "v", "state", "shadow", "ema", "ema state")):
        assert torch.equal(x, y), (what, k)


@pytest.mark.parametrize("name", ["fused", "sharded", "p2p"])
def test_eager_resume_continues_bit_exactly(name):
    """6 steps straight == 3 steps, torch.save / torch.load of weights and optimizer, a fresh model / arena / optimizer, 3 steps"""
    ma = _model(5)
    aa, oa = _setup(ma, name)
    _steps(oa, aa, range(6))
    mb = _model(5)
    ab, ob = _setup(mb, name)
    _steps(ob, ab, range(3))
    ck = _save({"model": mb.state_dict(), "opt": ob.state_dict()})
    del mb, ab, ob
    ck = torch.load(ck, weights_only=True)
    assert all(st["exp_avg"].device.type == "cpu" for st in ck["opt"]["state"].values())
    mc = _model(6)                                   # another initialisation: everything comes from the checkpoint
    mc.load_state_dict(ck["model"])
    ac, oc = _setup(mc, name, **OTHER)
    oc.load_state_dict(ck["opt"])
    assert oc.t == 3 and oc.lr == _lr(2) and oc.betas == (0.9, 0.999) and oc.weight_decay == 1e-2 and oc.eps == 1e-8
    _steps(oc, ac, range(3, 6))
    assert oc.t == 6
    _assert_same(oa.snapshot_tensors(), oc.snapshot_tensors(), name)


@pytest.mark.parametrize("src,dst", [("fused", "sharded"), ("fused", "p2p"), ("sharded", "fused"), ("p2p", "fused")])
def test_dicts_interchange_between_the_fused_forms(src, dst):
    m1 = _model(7)
    a1, o1 = _setup(m1, src)
    _steps(o1, a1, range(3))
    m2 = _model(8)
    m2.load_state_dict(m1.state_dict())
    a2, o2 = _setup(m2, dst, **OTHER)
    o2.load_state_dict(o1.state_dict())
    torch.cuda.synchronize()
    assert torch.equal(o1.m, o2.m) and torch.equal(o1.v, o2.v) and torch.equal(o1.state[:6], o2.state[:6])
    _steps(o1, a1, range(3, 5))
    _steps(o2, a2, range(3, 5))
    if "p2p" not in (src, dst):                      # the same kernel (svdx_adamw_step) on both sides
        _assert_same(o1.snapshot_tensors(), o2.snapshot_tensors())
    else:                                            # svdx_adamw_step_p2p: the same arithmetic in another kernel
        d = (a1.data - a2.data).abs().max().item()
        assert d <= 1e-6 * a1.data.abs().max().item(), d
        assert o1.t == o2.t == 5


@pytest.mark.parametrize("with_ema", [False, True])
def test_graphed_step_continues_bit_exactly_after_an_in_place_load(with_ema):
    """capture, replay 3 times, save; replay 3 more (run A); load the saved state into the same buffers, replay 3 more (run B)"""
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.train import GraphedStep
    m = _model(9)
    ema = EMAModel(m.parameters(), update_after_step=1) if with_ema else None
    arena, opt = _setup(m, "fused")
    if with_ema:
        opt.attach_ema(ema)
    grad_in = torch.zeros_like(arena.grad)

    def fn(b):
        arena.grad.copy_(b["grad"])
        opt.step()

    graphed = GraphedStep(fn, {"grad": grad_in}, warmup=2, restore=opt.snapshot_tensors(),
                          on_restored=lambda: m.refresh_trainable_operands(shadow_current=True))

    def run(ts):
        for t in ts:
            opt.lr = _lr(t)
            graphed({"grad": _flat_grad(arena, t)})
        torch.cuda.synchronize()

    run(range(3))
    ck = {"model": m.state_dict(), "opt": opt.state_dict()}
    if with_ema:
        ck["ema"] = ema.state_dict()
        ema3 = ema._flat.clone()
    ck = _save(ck)
    run(range(3, 6))
    run_a = [t.clone() for t in opt.snapshot_tensors()]
    ck = torch.load(ck, weights_only=True)
    m.load_state_dict(ck["model"])                    # in place: the parameters are views of the arena
    arena.refresh_shadow()
    opt.load_state_dict(ck["opt"])
    if with_ema:
        flat = ema._flat
        ema.load_state_dict(ck["ema"])
        torch.cuda.synchronize()
        assert ema._flat is flat and torch.equal(flat, ema3) and ema.optimization_step == 3   # landed in the optimizer's EMA buffer
    assert opt.t == 3
    run(range(3, 6))
    run_b = opt.snapshot_tensors()
    assert len(run_b) == (7 if with_ema else 5)
    _assert_same(run_a, run_b)
    if with_ema:
        assert ema.optimization_step == 6


def test_interchange_with_torch_adamw_and_one_update_each():
    m = _model(11)
    arena, opt = _setup(m, "fused")
    _steps(opt, arena, range(3))
    params = [torch.nn.Parameter(p.detach().clone()) for p in arena.params]
    ref = torch.optim.AdamW(params, lr=5.0)
    ref.load_state_dict(opt.state_dict())
    rsd = ref.state_dict()
    assert rsd["param_groups"][0]["lr"] == opt.lr and rsd["param_groups"][0]["betas"] == (0.9, 0.999)
    for i, (p, q) in enumerate(zip(arena.params, params)):
        st = ref.state[q]
        assert st["step"].item() == 3.0 and st["step"].dtype == torch.float32
        o = arena.offset_of[p]
        assert torch.equal(st["exp_avg"].reshape(-1), opt.m[o:o + p.numel()]) and torch.equal(st["exp_avg_sq"].reshape(-1), opt.v[o:o + p.numel()])
    # and back: torch.optim.AdamW's dict into a fresh FusedAdamW
    m2 = _model(12)
    m2.load_state_dict(m.state_dict())
    a2, o2 = _setup(m2, "fused", **OTHER)
    o2.load_state_dict(rsd)
    torch.cuda.synchronize()
    assert torch.equal(o2.m, opt.m) and torch.equal(o2.v, opt.v) and o2.t == 3 and o2.lr == opt.lr
    # one update of each from the same state and gradient
    g = _flat_grad(arena, 3)
    arena.grad.copy_(g)
    for p, q in zip(arena.params, params):
        q.grad = arena.grad_views[p].clone()
    before = arena.data.clone()
    opt.step()
    ref.step()
    torch.cuda.synchronize()
    # each result against fp32 eps times the magnitudes of the terms it sums (o2 still holds the moments before the update).
    # The two arithmetics round differently (torch: lerp, host-side double bias corrections, a true division; the kernel:
    # b1*m + (1-b1)*g, powf on the device, rsqrtf, contracted FMAs), and the kernel holds the betas as fp32: 1 - fp32(0.999)
    # is 1.3e-5 (108 eps) relative away from torch's double 1 - 0.999, which enters v and, through v and 1 - b2^t, the weights.
    # Measured on an H100 80GB HBM3 (700 W): weights 157, m 3.4, v 109 of these units; bounded with a quarter more.
    eps = torch.finfo(torch.float32).eps
    worst = {"weights": 0.0, "m": 0.0, "v": 0.0}
    for p, q in zip(arena.params, params):
        o, n = arena.offset_of[p], p.numel()
        gi, m0, v0, p0 = g[o:o + n], o2.m[o:o + n], o2.v[o:o + n], before[o:o + n]
        st = ref.state[q]
        terms = {"weights": (p.detach().reshape(-1), q.detach().reshape(-1), p0.abs() + (q.detach().reshape(-1) - p0).abs()),
                 "m": (opt.m[o:o + n], st["exp_avg"].reshape(-1), 0.9 * m0.abs() + 0.1 * gi.abs()),
                 "v": (opt.v[o:o + n], st["exp_avg_sq"].reshape(-1), 0.999 * v0 + 0.001 * gi * gi)}
        for k, (x, y, mag) in terms.items():
            worst[k] = max(worst[k], ((x - y).abs() / (eps * mag + 1e-38)).max().item())
    print("fused vs torch.optim.AdamW, one update, max |difference| in units of eps32 * term magnitudes:", worst)
    assert worst["weights"] <= 200 and worst["m"] <= 5 and worst["v"] <= 140, worst
    assert ref.state[params[0]]["step"].item() == 4 == opt.t
