"""GPU tests of the block-wise 8-bit AdamW: svdx_adamw8bit against oracle/svd_adam8bit_oracle.py BIT FOR BIT (codes, absmax,
masters, bf16 shadow, fp32 small-parameter states) through FusedAdamW8bit and the drop-in AdamW8bit, on the config-2 arena of
the SVD UNet, under CUDA-graph replay, with an attached EMA, across the two front ends, and in the unchanged script's loop."""
import pytest
import torch

from oracle import svd_adam8bit_oracle as O
from test_unet_gpu import DEV, _build, _rel, _train_filter

pytestmark = pytest.mark.gpu


class _Net(torch.nn.Module):
    def __init__(self, sizes, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(n, generator=g).to(DEV)) for n in sizes])


class _Ref:
    """the oracle's copy of a FusedAdamW8bit's masters and state"""

    def __init__(self, opt):
        self.opt = opt
        self.items = []
        for p, *_r in opt.layout:
            sv = {k: (v if k.startswith("qmap") else v.clone()) for k, v in opt.state_views(p).items()}
            self.items.append((p, p.detach().clone(), sv))

    def step(self, grads, grad_scale=1.0):
        """apply the oracle with the optimizer's own state after its tick (bias corrections are not recomputed)"""
        for (p, pr, sv), g in zip(self.items, grads):
            if "absmax1" in sv:
                O.step_8bit(pr, g, sv["state1"], sv["state2"], sv["absmax1"], sv["absmax2"], sv["qmap1"], sv["qmap2"], self.opt.state,
                            grad_scale)
            else:
                O.step_fp32(pr, g, sv["state1"], sv["state2"], self.opt.state, grad_scale)

    def check(self, what=""):
        a = self.opt.arena
        for p, pr, sv in self.items:
            assert torch.equal(p.detach(), pr), what
            o = a.offset_of[p]
            assert torch.equal(a.shadow[o:o + p.numel()], pr.reshape(-1).to(torch.bfloat16)), what
            mine = self.opt.state_views(p)
            for k in ("state1", "state2", "absmax1", "absmax2"):
                if k in sv:
                    assert torch.equal(mine[k], sv[k]), (what, k, p.numel())


SIZES = [1, 255, 256, 257, 4095, 4096, 1_000_003, 5000, 70000]


def _rand_grads(arena, seed, zero_index=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    with torch.no_grad():
        for i, p in enumerate(arena.params):
            v = arena.grad_views[p]
            if i == zero_index:
                v.zero_()
            else:
                v.copy_(torch.randn(v.shape, generator=g, device=DEV) * (10.0 ** (i % 5 - 3)))
            out.append(v.clone())
    return out


@pytest.mark.parametrize("grad_scale", [1.0, 0.37])
def test_kernel_equals_oracle_bit_for_bit(grad_scale):
    from svd_xtend_b200 import raw
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    net = _Net(SIZES)
    arena = ParamArena(net)
    opt = FusedAdamW8bit(arena, lr=1e-2, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    ref = _Ref(opt)
    for t in range(1, 5):
        opt.lr = 1e-2 / t
        grads = _rand_grads(arena, 100 + t, zero_index=SIZES.index(5000))       # an all-zero-gradient 8-bit tensor
        l0 = raw.LAUNCHES[0]
        opt.step(grad_scale)
        assert raw.LAUNCHES[0] - l0 == 2                       # tick + ONE launch over every parameter
        ref.step(grads, grad_scale)
        torch.cuda.synchronize()
        ref.check(t)
        assert opt.t == t
    zero = int((opt.qmap1 == 0).nonzero().item())
    sv = opt.state_views(arena.params[SIZES.index(5000)])
    assert bool((sv["absmax1"] == 0).all()) and bool((sv["state1"] == zero).all())
    assert bool((sv["state2"] == 0).all())                   # the unsigned map's 0.0 is its first code


def test_two_runs_are_bit_identical():
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    outs = []
    for _ in range(2):
        arena = ParamArena(_Net([1_000_003, 300, 8192], seed=5))
        opt = FusedAdamW8bit(arena, lr=3e-3)
        for t in range(3):
            _rand_grads(arena, 7 + t)
            opt.step()
        torch.cuda.synchronize()
        outs.append([x.clone() for x in opt.snapshot_tensors()])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_graph_replay_equals_eager_and_snapshot_restores():
    from svd_xtend_b200.train import FusedAdamW8bit, GraphedStep, ParamArena
    sizes = [4096 * 3 + 17, 100, 300000]
    a1, a2 = ParamArena(_Net(sizes, seed=9)), ParamArena(_Net(sizes, seed=9))
    o1, o2 = FusedAdamW8bit(a1, lr=1e-3), FusedAdamW8bit(a2, lr=1e-3)
    before = [t.clone() for t in o2.snapshot_tensors()]

    def fn(b):
        o2.step(0.5)
        return None

    graphed = GraphedStep(fn, {"grad": a2.grad}, warmup=2, restore=o2.snapshot_tensors())
    for x, y in zip(o2.snapshot_tensors(), before):
        assert torch.equal(x, y)                               # warm-up and capture left every state tensor as it was
    for t in range(1, 6):
        o1.lr = o2.lr = 1e-3 * t
        g = torch.randn(a1.numel, device=DEV)
        a1.grad.copy_(g)
        o1.step(0.5)
        graphed({"grad": g})
        torch.cuda.synchronize()
        for x, y in zip(o1.snapshot_tensors(), o2.snapshot_tensors()):
            assert torch.equal(x, y), t


def test_attached_ema_equals_fused_adamw8bit_plus_ema_oracle():
    from oracle.svd_ema_oracle import get_decay
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    sizes = [5000, 33, 4096]
    n1, n2 = _Net(sizes, seed=4), _Net(sizes, seed=4)
    a1, a2 = ParamArena(n1), ParamArena(n2)
    o1, o2 = FusedAdamW8bit(a1, lr=2e-3), FusedAdamW8bit(a2, lr=2e-3)
    ema = EMAModel(n2.parameters(), update_after_step=1)
    o2.attach_ema(ema)
    e = a2.data.clone()
    for t in range(1, 6):
        g = torch.randn(a1.numel, device=DEV)
        a1.grad.copy_(g)
        a2.grad.copy_(g)
        o1.step()
        o2.step()
        e.sub_((1 - get_decay(t, update_after_step=1)) * (e - a1.data))
        torch.cuda.synchronize()
        for x, y in zip(o1.snapshot_tensors(), o2.snapshot_tensors()):
            assert torch.equal(x, y), t
        assert torch.equal(ema._flat, e), t


def test_fused_state_dict_gives_the_same_next_step_in_the_drop_in():
    from svd_xtend_b200.optim8bit import AdamW8bit
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    sizes = [5000, 10, 70000]
    arena = ParamArena(_Net(sizes, seed=2))
    fused = FusedAdamW8bit(arena, lr=1e-3, weight_decay=0.05)
    for t in range(3):
        _rand_grads(arena, 40 + t)
        fused.step()
    sd = fused.state_dict()
    params = [torch.nn.Parameter(p.detach().clone()) for p in arena.params]
    drop = AdamW8bit(params, lr=5.0)                          # the loaded group carries lr / weight decay
    drop.load_state_dict(sd)
    grads = _rand_grads(arena, 50)
    for p, g in zip(params, grads):
        p.grad = g.clone()
    fused.step()
    drop.step()
    torch.cuda.synchronize()
    for p, q in zip(arena.params, params):
        assert torch.equal(p.detach(), q.detach())
        a, b = fused.state_views(p), drop.state[q]
        for k in ("state1", "state2", "absmax1", "absmax2"):
            if k in a:
                assert torch.equal(a[k], b[k]), k
    assert drop.state_dict()["state"][0]["step"] == 4 == fused.t


def test_config2_arena_five_steps_equal_the_oracle_and_forward_uses_the_new_masters():
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    from svd_xtend_b200.workload import BENCH_CONFIGS, SVD_CONFIG, edm_loss, synthetic_batch
    cfg = BENCH_CONFIGS[2]
    torch.manual_seed(1234)
    with torch.device(DEV):
        unet = Ours(**SVD_CONFIG)
    _train_filter(unet)
    unet.train()
    arena = ParamArena(unet)
    unet.attach_arena(arena)
    assert arena.numel >= 397_620_480
    opt = FusedAdamW8bit(arena, lr=1e-5)
    opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
    assert any(q for _, _, q, _, _ in opt.layout) and not all(q for _, _, q, _, _ in opt.layout)
    ref = _Ref(opt)
    b = {k: v.to(DEV) for k, v in synthetic_batch(1, cfg["frames"], cfg["h"], cfg["w"], seed=1234).items()}
    for t in range(1, 6):
        opt.lr = 1e-5 * (1.0 + 0.5 * t)
        arena.zero_grad()
        pred = unet(b["sample"], b["timestep"], b["encoder_hidden_states"], added_time_ids=b["added_time_ids"]).sample
        edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"]).backward()
        grads = [arena.grad_views[p].clone() for p in arena.params]
        opt.step()
        ref.step(grads)
        torch.cuda.synchronize()
        ref.check(t)
        del grads
    del ref
    torch.cuda.empty_cache()
    small = synthetic_batch(1, cfg["frames"], 16, 16, seed=77)
    small = {k: v.to(DEV) for k, v in small.items()}
    with torch.no_grad():
        out = unet(small["sample"], small["timestep"], small["encoder_hidden_states"], added_time_ids=small["added_time_ids"]).sample
        sd = unet.state_dict()
        with torch.device(DEV):
            fresh = Ours(**SVD_CONFIG)
        fresh.load_state_dict(sd)
        ref_out = fresh(small["sample"], small["timestep"], small["encoder_hidden_states"], added_time_ids=small["added_time_ids"]).sample
    torch.cuda.synchronize()
    _assert_operands_follow_masters(unet, arena)
    assert _rel(out, ref_out) < 2.5e-2, _rel(out, ref_out)        # the bf16 tolerance of tests/test_ema_gpu.py's same check


def _assert_operands_follow_masters(model, arena):
    """the bf16 operands the last forward used (shadow and dgrad transposes) are exactly those re-derived from the masters"""
    shadow = arena.shadow.clone()
    transposes = [dst.clone() for _, dst, _, _ in arena._tjobs]
    assert transposes
    model.refresh_trainable_operands()                   # full re-derivation: cast of the fp32 masters, then the transposes
    torch.cuda.synchronize()
    assert torch.equal(arena.shadow, shadow)
    for (_, dst, _, _), b in zip(arena._tjobs, transposes):
        assert torch.equal(dst, b)


@pytest.mark.parametrize("graphs", [False, True])
def test_unchanged_script_loop_with_drop_in(graphs):
    """train_svd.py --use_8bit_adam: autocast forward, loss.backward(), bnb.optim.AdamW8bit (the drop-in) with LambdaLR,
    optimizer.zero_grad(set_to_none=True); every step equals the oracle, and the next forward runs on the new masters"""
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.optim8bit import AdamW8bit
    from svd_xtend_b200.train import ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    from test_boundary_gpu import _call, _tiny_batch
    from test_unet_gpu import _loss
    _, ours = _build(TINY_CONFIG, seed=61)
    _train_filter(ours)
    ours.train()
    if graphs:
        ours.enable_cuda_graphs(warmup=2)
    else:
        ours.attach_arena(ParamArena(ours))
    params = [p for p in ours.parameters() if p.requires_grad]
    opt = AdamW8bit(params, lr=3e-3, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 1.0 / (1 + s))
    batch = _tiny_batch(71)
    refs = []
    for p in params:
        st = {}
        if p.numel() >= 4096:
            nb = (p.numel() + 255) // 256
            st = dict(state1=torch.zeros_like(p, dtype=torch.uint8), state2=torch.zeros_like(p, dtype=torch.uint8),
                      absmax1=torch.zeros(nb, device=DEV), absmax2=torch.zeros(nb, device=DEV))
        else:
            st = dict(state1=torch.zeros_like(p), state2=torch.zeros_like(p))
        refs.append((p.detach().clone(), st))
    for step in range(5):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, loss = _loss(ours, batch)
        loss.backward()
        grads = [p.grad.detach().clone() for p in params]
        opt.step()
        state = opt._dev[0][0]
        for (pr, st), p, g in zip(refs, params, grads):
            if "absmax1" in st:
                O.step_8bit(pr, g, st["state1"], st["state2"], st["absmax1"], st["absmax2"], opt.state[p]["qmap1"], opt.state[p]["qmap2"],
                            state)
            else:
                O.step_fp32(pr, g, st["state1"], st["state2"], state)
        sched.step()
        opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        assert state[0].item() == pytest.approx(3e-3 / (1 + step), rel=1e-6)
        for (pr, st), p in zip(refs, params):
            assert torch.equal(p.detach(), pr), step
            for k in ("state1", "state2", "absmax1", "absmax2"):
                if k in st:
                    assert torch.equal(opt.state[p][k], st[k]), (step, k)
    with torch.no_grad():
        out = _call(ours, batch)                         # the operands follow the updated masters (version counters moved)
        fresh = Ours(**TINY_CONFIG).to(DEV)
        fresh.load_state_dict(ours.state_dict())
        ref_out = _call(fresh, batch)
    torch.cuda.synchronize()
    arena = ours._arena
    assert torch.equal(arena.shadow, arena.data.to(torch.bfloat16))
    _assert_operands_follow_masters(ours, arena)
    assert _rel(out, ref_out) < 2.5e-2, _rel(out, ref_out)


def test_training_tracks_fp32_adamw():
    """20 tiny-config steps on one batch: the loss trajectory under AdamW8bit stays within 5 % of torch.optim.AdamW's"""
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.optim8bit import AdamW8bit
    from svd_xtend_b200.train import ParamArena
    from test_boundary_gpu import _tiny_batch
    from test_unet_gpu import _loss
    batch = _tiny_batch(81, b=2)
    curves = []
    for use8 in (False, True):
        _, m = _build(TINY_CONFIG, seed=83)
        _train_filter(m)
        m.train()
        m.attach_arena(ParamArena(m))
        ps = [p for p in m.parameters() if p.requires_grad]
        opt = AdamW8bit(ps, lr=1e-3, min_8bit_size=256) if use8 else torch.optim.AdamW(ps, lr=1e-3)
        losses = []
        for _ in range(20):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                _, loss = _loss(m, batch)
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
            losses.append(loss.item())
        curves.append(losses)
    l32, l8 = curves
    assert l32[-1] < 0.9 * l32[0]                           # the run actually trains
    for a, b in zip(l32, l8):
        assert abs(a - b) <= 0.05 * a, (l32, l8)


@pytest.mark.parametrize("offset", [0, 1])
def test_midpoint_ties_and_misaligned_views(offset):
    """m' / A1' exactly on midpoints of the signed map goes to the lower code, just above it to the upper one: beta1 = 0 makes
    m' = g, and each block holds one |g| = 1 (A1' = 1). offset = 1 makes the parameter and its gradient views one element
    past a 16-byte boundary, so the whole job takes the kernel's scalar path; offset = 0 the vector path. Both equal the
    oracle bit for bit."""
    from svd_xtend_b200.optim8bit import AdamW8bit, dynamic_map
    n = 4096 + 300                                            # 18 blocks, the last one partial
    q = dynamic_map(True)
    mid = O.midpoints(q)
    ks = torch.arange(n) % 255
    vals = mid[ks].clone()
    up = torch.arange(n) % 3 == 1
    vals[up] = torch.nextafter(vals[up], torch.full_like(vals[up], 2.0))
    vals[torch.arange(n) % 256 == 0] = 1.0                    # the block maximum
    want = (ks + up.long()).to(torch.uint8)
    want[torch.arange(n) % 256 == 0] = 255
    base_p = torch.randn(n + 4, device=DEV)
    base_g = torch.zeros(n + 4, device=DEV)
    base_g[offset:offset + n] = vals.to(DEV)
    p = torch.nn.Parameter(base_p[offset:offset + n])
    p.grad = base_g[offset:offset + n]
    assert (p.data_ptr() % 16 == 0) == (offset == 0)
    small = torch.nn.Parameter(torch.randn(100, device=DEV)[offset:offset + 50])
    small.grad = torch.randn(100, device=DEV)[offset:offset + 50]
    ref_p, ref_small = p.detach().clone(), small.detach().clone()
    outside = torch.cat([base_p[:offset], base_p[offset + n:]]).clone()
    opt = AdamW8bit([p, small], lr=1e-3, betas=(0.0, 0.999), weight_decay=0.0)
    opt.step()
    torch.cuda.synchronize()
    st = opt.state[p]
    assert torch.equal(st["state1"].cpu(), want)
    assert bool((st["absmax1"] == 1.0).all())
    state = opt._dev[0][0]
    r = {"state1": torch.zeros(n, dtype=torch.uint8, device=DEV), "state2": torch.zeros(n, dtype=torch.uint8, device=DEV),
         "absmax1": torch.zeros(18, device=DEV), "absmax2": torch.zeros(18, device=DEV)}
    O.step_8bit(ref_p, p.grad, r["state1"], r["state2"], r["absmax1"], r["absmax2"], st["qmap1"], st["qmap2"], state)
    m32, v32 = torch.zeros(50, device=DEV), torch.zeros(50, device=DEV)
    O.step_fp32(ref_small, small.grad, m32, v32, state)
    assert torch.equal(p.detach(), ref_p) and torch.equal(small.detach(), ref_small)
    for k in r:
        assert torch.equal(st[k], r[k]), k
    assert torch.equal(opt.state[small]["state1"], m32) and torch.equal(opt.state[small]["state2"], v32)
    assert torch.equal(torch.cat([base_p[:offset], base_p[offset + n:]]), outside)     # nothing written outside the view
