"""GPU tests of the sharded 8-bit AdamW (ShardedAdamW8bit, P2PShardedAdamW8bit and the svdx_adamw8bit_p2p kernel).

Worlds of N ranks are emulated on one device: every rank has its own model, arena and optimizer, the peer pointer lists point
at the local buffers, and a stand-in for torch.distributed hands each rank what its collectives would give. Each rank's launch
must leave exactly what FusedAdamW8bit.step(grad_scale=1/N) leaves over the rank-order sum of the gradients, bit for bit, in the
blocks it owns, and nothing else."""
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist

from test_unet_gpu import DEV

pytestmark = pytest.mark.gpu

SIZES = [1, 255, 256, 257, 4095, 4096, 100_003, 5000, 70000, 33, 262_144 + 129]


class _Net(torch.nn.Module):
    def __init__(self, sizes, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(n, generator=g).to(DEV)) for n in sizes])


class _World:
    """N emulated ranks of one sharded 8-bit form, plus the unsharded FusedAdamW8bit reference over the same layout"""

    def __init__(self, monkeypatch, form, world, max_grad_norm=None, ema=False, sizes=SIZES, lr=1e-2):
        from svd_xtend_b200 import train
        from svd_xtend_b200.ema import EMAModel
        self.train, self.mp, self.world = train, monkeypatch, world
        kw = dict(lr=lr, weight_decay=1e-2, max_grad_norm=max_grad_norm)
        self.nets = [_Net(sizes) for _ in range(world + 1)]
        self.arenas = [train.ParamArena(n, pad_to=world * 256, block=256) for n in self.nets]
        self.ref = train.FusedAdamW8bit(self.arenas[-1], **kw)
        self.emas = [EMAModel(n.parameters(), update_after_step=1) for n in self.nets] if ema else None
        if ema:
            self.ref.attach_ema(self.emas[-1])
        monkeypatch.setattr(train, "map_peer_buffers",
                            lambda t, group=None: [(a.grad if t.dtype == torch.float32 else a.shadow).data_ptr() for a in self.arenas[:-1]])
        cls = getattr(train, form)
        self.opts = []
        for r in range(world):
            with self.rank(r):
                self.opts.append(cls(self.arenas[r], **kw))
            if ema:
                self.opts[r].attach_ema(self.emas[r])
        self.gsum = None
        self.sumsq_total = None

    def rank(self, r):
        w = self

        def all_reduce(t, op=None, group=None):
            if t.dtype == torch.float64:               # the clip's sum of squares: every rank's partial
                t.copy_(w.sumsq_total)
            # the fences' flag: nothing to order on one device

        def reduce_scatter_tensor(out, inp, op=None, group=None):
            out.copy_(w.gsum[w.opts[r].lo:w.opts[r].hi])

        def all_gather_into_tensor(out, inp, group=None):
            lo, hi = w.opts[r].lo, w.opts[r].hi
            for a in w.arenas[:-1]:
                (a.shadow if out.dtype == torch.bfloat16 else a.data)[lo:hi].copy_(out[lo:hi])

        fake = SimpleNamespace(is_initialized=lambda: True, get_world_size=lambda group=None: w.world,
                               get_rank=lambda group=None: r, get_backend=lambda group=None: "nccl", ReduceOp=dist.ReduceOp,
                               all_reduce=all_reduce, reduce_scatter_tensor=reduce_scatter_tensor,
                               all_gather_into_tensor=all_gather_into_tensor)
        return _Patch(self.mp, self.train, fake)

    def set_grads(self, t):
        """seeded gradients per rank (different per rank), and their rank-order sum into the reference's arena"""
        self.gsum = torch.zeros_like(self.arenas[-1].grad)
        for r, a in enumerate(self.arenas[:-1]):
            g = torch.Generator(device=DEV).manual_seed(1000 * t + r)
            for i, p in enumerate(a.params):
                a.grad_views[p].copy_(torch.randn(p.shape, generator=g, device=DEV) * 10.0 ** (i % 4 - 3))
            self.gsum += a.grad
        self.arenas[-1].grad.copy_(self.gsum)
        from svd_xtend_b200 import raw
        if self.ref._clip is not None:                 # what the all-reduce of the ranks' partials gives
            parts = torch.zeros(1 + raw.SUMSQ_PARTIALS, device=DEV, dtype=torch.float64)
            total = torch.zeros(1, device=DEV, dtype=torch.float64)
            for o in self.opts:
                if o.__class__.__name__.startswith("P2P"):
                    raw.grad_sumsq_p2p(o.peer_grad, o.lo, o.hi - o.lo, parts)
                else:
                    raw.grad_sumsq(self.gsum[o.lo:o.hi], parts)
                total += parts[:1]
            self.sumsq_total = total

    def set_lr(self, lr):
        for o in [*self.opts, self.ref]:
            o.lr = lr

    def step_ranks(self, check_untouched=True):
        for r, o in enumerate(self.opts):
            before = [(a.data.clone(), a.shadow.clone()) for a in self.arenas[:-1]]
            ema_before = self.emas[r]._flat.clone() if self.emas else None
            with self.rank(r):
                o.step()
            torch.cuda.synchronize()
            if not check_untouched:
                continue
            lo, hi = o.lo, o.hi
            for k, (a, (d0, s0)) in enumerate(zip(self.arenas[:-1], before)):
                out = torch.ones(a.numel, dtype=torch.bool, device=DEV)
                out[lo:hi] = False
                assert torch.equal(a.shadow[out], s0[out]), ("shadow written outside the owner's blocks", r, k)
                assert torch.equal(a.data[out], d0[out]), ("masters written outside the owner's blocks", r, k)
            if self.emas:
                out = torch.ones(ema_before.numel(), dtype=torch.bool, device=DEV)
                out[lo:hi] = False
                assert torch.equal(self.emas[r]._flat[out], ema_before[out])

    def check(self, what):
        ref = self.ref
        for r, o in enumerate(self.opts):
            (c0, c1), (b0, b1), (f0, f1) = o.ranges
            a = self.arenas[r]
            assert torch.equal(a.data[o.lo:o.hi], self.arenas[-1].data[o.lo:o.hi]), (what, r, "masters")
            for name, (x, y) in (("codes1", (c0, c1)), ("codes2", (c0, c1)), ("absmax1", (b0, b1)), ("absmax2", (b0, b1)),
                                 ("m32", (f0, f1)), ("v32", (f0, f1))):
                assert torch.equal(getattr(o, name), getattr(ref, name)[x:y]), (what, r, name)
            assert torch.equal(a.shadow, self.arenas[-1].data.to(torch.bfloat16)), (what, r, "shadow")
            if self.emas:
                assert torch.equal(self.emas[r]._flat[o.lo:o.hi], self.emas[-1]._flat[o.lo:o.hi]), (what, r, "ema")
            if ref._clip is not None:
                assert torch.equal(o.grad_norm, ref.grad_norm), (what, r, "grad_norm")
            assert o.t == ref.t


class _Patch:
    def __init__(self, mp, module, fake):
        self.mp, self.module, self.fake = mp, module, fake

    def __enter__(self):
        self.mp.setattr(self.module, "dist", self.fake)

    def __exit__(self, *exc):
        self.mp.setattr(self.module, "dist", dist)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("form", ["P2PShardedAdamW8bit", "ShardedAdamW8bit"])
@pytest.mark.parametrize("clip,ema", [(False, False), (True, False), (False, True), (True, True)])
def test_emulated_ranks_equal_fused_adamw8bit_on_the_summed_gradient(monkeypatch, world, form, clip, ema):
    w = _World(monkeypatch, form, world, max_grad_norm=0.5 if clip else None, ema=ema)
    for t in range(1, 4):
        w.set_lr(1e-2 / t)
        w.set_grads(t)
        w.step_ranks()
        w.ref.step(1.0 / world)
        torch.cuda.synchronize()
        w.check(t)
    if clip:
        assert w.ref.grad_norm.item() > 0.5          # the clip was active


def test_p2p_kernel_equals_the_oracle_on_the_rank_sum(monkeypatch):
    """one emulated world-3 step through svdx_adamw8bit_p2p against oracle/svd_adam8bit_oracle.py directly"""
    from oracle import svd_adam8bit_oracle as O
    w = _World(monkeypatch, "P2PShardedAdamW8bit", 3)
    ref = w.ref
    items = []
    for p, off, quant, so, bo in ref.layout:
        items.append((p, p.detach().clone(), {k: (v if k.startswith("qmap") else v.clone()) for k, v in ref.state_views(p).items()}))
    w.set_grads(1)
    w.step_ranks(check_untouched=False)
    state = w.opts[0].state
    torch.cuda.synchronize()
    for (p, pr, sv), q in zip(items, w.arenas[-1].params):
        g = w.gsum[w.arenas[-1].offset_of[q]:w.arenas[-1].offset_of[q] + p.numel()].view(p.shape)
        if "absmax1" in sv:
            O.step_8bit(pr, g, sv["state1"], sv["state2"], sv["absmax1"], sv["absmax2"], sv["qmap1"], sv["qmap2"], state, 1.0 / 3)
        else:
            O.step_fp32(pr, g, sv["state1"], sv["state2"], state, 1.0 / 3)
    for r, o in enumerate(w.opts):
        a = w.arenas[r]
        for p, off, n, quant, si, bi in o.subjobs:
            i = o._index[p]
            pr, sv = items[i][1], items[i][2]
            d = off - w.arenas[r].offset_of[p]
            assert torch.equal(a.data[off:off + n], pr.reshape(-1)[d:d + n]), (r, i)
            if quant:
                (c0, _), (b0, _), _ = o.ranges
                assert torch.equal(o.codes1[si - c0:si - c0 + n], sv["state1"].reshape(-1)[d:d + n])
                assert torch.equal(o.codes2[si - c0:si - c0 + n], sv["state2"].reshape(-1)[d:d + n])
                nb = (n + 255) // 256
                assert torch.equal(o.absmax1[bi - b0:bi - b0 + nb], sv["absmax1"][d // 256:d // 256 + nb])
                assert torch.equal(o.absmax2[bi - b0:bi - b0 + nb], sv["absmax2"][d // 256:d // 256 + nb])


@pytest.mark.parametrize("form", ["ShardedAdamW8bit", "P2PShardedAdamW8bit"])
def test_world_one_graphed_step_equals_fused_adamw8bit_and_restores(form):
    from svd_xtend_b200 import train
    sizes = [4096 * 3 + 17, 100, 300000, 5000]
    a1, a2 = train.ParamArena(_Net(sizes, seed=9), pad_to=256, block=256), train.ParamArena(_Net(sizes, seed=9), pad_to=256, block=256)
    o1 = train.FusedAdamW8bit(a1, lr=1e-3, max_grad_norm=1.0)
    o2 = getattr(train, form)(a2, lr=1e-3, max_grad_norm=1.0)
    before = [t.clone() for t in o2.snapshot_tensors()]
    graphed = train.GraphedStep(lambda b: o2.step(), {"grad": a2.grad}, warmup=2, restore=o2.snapshot_tensors())
    for x, y in zip(o2.snapshot_tensors(), before):
        assert torch.equal(x, y)                               # warm-up and capture left every state tensor as it was
    for t in range(1, 6):
        o1.lr = o2.lr = 1e-3 * t
        g = torch.randn(a1.numel, device=DEV) * (0.01 if t % 2 else 1.0)
        a1.grad.copy_(g)
        o1.step()
        graphed({"grad": g})
        torch.cuda.synchronize()
        for x, y in zip(o1.snapshot_tensors(), o2.snapshot_tensors()):
            assert torch.equal(x, y), t
        assert torch.equal(o1.grad_norm, o2.grad_norm)


def _sd_equal(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert list(a["state"]) == list(b["state"])
    for i in a["state"]:
        assert list(a["state"][i]) == list(b["state"][i])
        for k, v in a["state"][i].items():
            assert torch.equal(v, b["state"][i][k]) if isinstance(v, torch.Tensor) else v == b["state"][i][k], (i, k)


def test_checkpoints_move_between_the_sharded_and_the_fused_form(monkeypatch):
    from svd_xtend_b200 import train
    from svd_xtend_b200.optim8bit import AdamW8bit
    # world-4 run, state_dict (collective), into FusedAdamW8bit, continue; against the uninterrupted reference
    w = _World(monkeypatch, "P2PShardedAdamW8bit", 4)
    for t in range(1, 4):
        w.set_lr(1e-2 / t)
        w.set_grads(t)
        w.step_ranks(check_untouched=False)
        w.ref.step(0.25)
    torch.cuda.synchronize()
    names = list(w.opts[0]._moment_buffers)
    calls = [0]

    def gather(out, src, group=None):
        name = names[calls[0] % len(names)]
        calls[0] += 1
        width = src.numel()
        for k, o in enumerate(w.opts):
            mine = getattr(o, name)
            out[k * width:k * width + mine.numel()].copy_(mine)

    sds = []
    for r in range(4):
        with w.rank(r):
            monkeypatch.setattr(w.train.dist, "all_gather_into_tensor", gather)
            sds.append(w.opts[r].state_dict())
    ref_sd = w.ref.state_dict()
    for sd in sds:
        _sd_equal(sd, ref_sd)
    resumed = train.FusedAdamW8bit(train.ParamArena(_Net(SIZES), pad_to=4 * 256, block=256), lr=1.0)
    resumed.arena.data.copy_(w.arenas[-1].data)
    resumed.arena.refresh_shadow()
    resumed.load_state_dict(sds[1])
    drop = AdamW8bit([torch.nn.Parameter(p.detach().clone()) for p in w.nets[-1].parameters()])
    drop.load_state_dict(sds[2])                           # the drop-in accepts the sharded dict
    for t in range(4, 6):
        w.set_lr(1e-2 / t)
        resumed.lr = 1e-2 / t
        w.set_grads(t)
        resumed.arena.grad.copy_(w.gsum)
        resumed.step(0.25)
        w.ref.step(0.25)
        torch.cuda.synchronize()
        for x, y in zip(resumed.snapshot_tensors(), w.ref.snapshot_tensors()):
            assert torch.equal(x, y), t

    # a FusedAdamW8bit dict into an emulated world-2 form, continue; against the uninterrupted reference
    w2 = _World(monkeypatch, "P2PShardedAdamW8bit", 2)
    for t in range(1, 3):
        w2.set_lr(1e-2 / t)
        w2.set_grads(t)
        w2.ref.step(0.5)
    torch.cuda.synchronize()
    sd = w2.ref.state_dict()
    for r, o in enumerate(w2.opts):
        o.load_state_dict(sd)
        w2.arenas[r].data.copy_(w2.arenas[-1].data)
        w2.arenas[r].refresh_shadow()
    for t in range(3, 5):
        w2.set_lr(1e-2 / t)
        w2.set_grads(t)
        w2.step_ranks()
        w2.ref.step(0.5)
        torch.cuda.synchronize()
        w2.check(t)


@pytest.mark.parametrize("form", ["ShardedAdamW8bit", "P2PShardedAdamW8bit"])
def test_video_train_step_accumulating_two_matches_fused_adamw8bit(form):
    """VideoTrainStep(gradient_accumulation_steps=2), captured, with a sharded form at world 1: every update equals FusedAdamW8bit
    on the same accumulated gradient, bit for bit. The backward rounds differently from run to run, so the reference is a twin
    FusedAdamW8bit whose step is captured into the same graph, just before the sharded one, on a copy of the gradient it reads."""
    from test_video_train_gpu import _frames, _pairs, _tiny_cfgs
    from svd_xtend_b200 import train
    from svd_xtend_b200.video_train import VideoTrainStep
    torch.backends.cuda.matmul.allow_tf32 = False
    x = [_frames(1, 4, 64, 128, 40 + i) for i in range(4)]
    (_, v), (_, c), (_, u) = _pairs(7, *_tiny_cfgs())
    arena = train.ParamArena(u, pad_to=256, block=256)
    u.attach_arena(arena)
    twin_net = torch.nn.Module()
    twin_net.ps = torch.nn.ParameterList([torch.nn.Parameter(p.detach().clone()) for p in arena.params])
    twin = train.ParamArena(twin_net, pad_to=256, block=256)
    assert twin.offsets == arena.offsets
    ref = train.FusedAdamW8bit(twin, lr=1e-4, max_grad_norm=1.0)
    opt = getattr(train, form)(arena, lr=1e-4, max_grad_norm=1.0)
    opt.on_updated = lambda: u.refresh_trainable_operands(shadow_current=True)
    step_, snap_ = opt.step, opt.snapshot_tensors

    def step():
        twin.grad.copy_(arena.grad)
        ref.step()
        step_()

    opt.step = step
    opt.snapshot_tensors = lambda: snap_() + ref.snapshot_tensors()     # the capture's warm-up steps are undone for both
    w0 = arena.data.clone()
    vts = VideoTrainStep(u, v, c, opt, frames_shape=(1, 4, 64, 128), conditioning_dropout_prob=0.1,
                         generator=torch.Generator(DEV).manual_seed(123), gradient_accumulation_steps=2)
    assert torch.equal(arena.data, w0) and torch.equal(twin.data, w0) and ref.t == 0 and opt.t == 0
    syncs = []
    for i in range(4):
        if i == 2:
            opt.lr = ref.lr = 5e-5
        vts(x[i])
        syncs.append(vts.sync_gradients)
        torch.cuda.synchronize()
        if vts.sync_gradients:
            for a_, b_ in zip(snap_(), ref.snapshot_tensors()):
                assert torch.equal(a_, b_), i
    assert syncs == [False, True, False, True] and opt.t == 2 and not torch.equal(arena.data, w0)
