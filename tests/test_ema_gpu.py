"""GPU tests of the weight EMA: the fused AdamW + EMA kernels, the multi-tensor EMA kernel, the device decay schedule over
graph replays, an attached EMA inside a captured GraphedStep, and the unchanged script's validation loop with the drop-in
EMAModel. Arithmetic is compared BIT FOR BIT against torch's `s.sub_((1 - d) * (s - p))`."""
import numpy as np
import pytest
import torch

from test_ema import CONFIGS
from test_unet_gpu import DEV, _build, _loss, _rel, _train_filter

pytestmark = pytest.mark.gpu


def _rand(n, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * scale).to(DEV)


def _ema_state(**kw):
    from svd_xtend_b200.ema import EMAModel
    return EMAModel([torch.zeros(1, device=DEV)], **kw)._state


@pytest.mark.parametrize("n", [4096, 10003])
def test_adamw_graph_ema_is_adamw_graph_plus_torch_ema(n):
    from oracle.svd_ema_oracle import get_decay
    from svd_xtend_b200 import raw
    p, g = _rand(n, 1), _rand(n, 2)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    state = torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0], device=DEV)
    sh = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    e = p.clone()
    est = _ema_state()
    ref = [t.clone() for t in (p, m, v, state, sh)]
    e_ref = p.clone()
    for t in range(1, 5):
        raw.adamw_graph(p, g, m, v, state, 0.5, shadow=sh, ema=e, ema_state=est)
        raw.adamw_graph(ref[0], g, ref[1], ref[2], ref[3], 0.5, shadow=ref[4])
        e_ref.sub_((1 - get_decay(t)) * (e_ref - ref[0]))
        torch.cuda.synchronize()
        for a, b in zip((p, m, v, state, sh), ref):
            assert torch.equal(a, b), t
        assert torch.equal(e, e_ref), t
    assert int(est[0].item()) == 4


@pytest.mark.parametrize("world,rank", [(1, 0), (2, 1), (3, 2)])
def test_adamw_p2p_ema_matches_p2p_and_touches_only_the_slice(world, rank):
    from oracle.svd_ema_oracle import get_decay
    from svd_xtend_b200 import raw
    n = 4096
    lo = rank * n
    grads = [_rand(n * world, 30 + r) for r in range(world)]
    shadows = [torch.full((n * world,), 7.0, device=DEV, dtype=torch.bfloat16) for _ in range(world)]
    shadows_ref = [s.clone() for s in shadows]
    p = _rand(n, 50)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    state = torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0], device=DEV)
    p_ref, m_ref, v_ref, state_ref = p.clone(), m.clone(), v.clone(), state.clone()
    ema_full = torch.full((n * world,), -3.0, device=DEV)
    ema_full[lo:lo + n] = p
    e_ref = p.clone()
    est = _ema_state(update_after_step=1)
    for t in range(1, 4):
        raw.adamw_p2p(p, m, v, grads, shadows, lo, state, 1.0 / world, ema=ema_full[lo:lo + n], ema_state=est)
        raw.adamw_p2p(p_ref, m_ref, v_ref, grads, shadows_ref, lo, state_ref, 1.0 / world)
        e_ref.sub_((1 - get_decay(t, update_after_step=1)) * (e_ref - p_ref))
    torch.cuda.synchronize()
    assert torch.equal(p, p_ref) and torch.equal(m, m_ref) and torch.equal(v, v_ref) and torch.equal(state, state_ref)
    assert all(torch.equal(a, b) for a, b in zip(shadows, shadows_ref))
    assert torch.equal(ema_full[lo:lo + n], e_ref)
    rest = torch.cat([ema_full[:lo], ema_full[lo + n:]])
    assert bool((rest == -3.0).all())


def test_multi_tensor_ema_equals_oracle_with_two_launches_and_no_idle_copies():
    from oracle.svd_ema_oracle import EMAModel as Oracle
    from svd_xtend_b200 import raw
    from svd_xtend_b200.ema import EMAModel
    torch.manual_seed(0)
    big = torch.randn(5000, device=DEV)
    params = [torch.nn.Parameter(torch.randn(s, device=DEV), requires_grad=rg)
              for s, rg in [((64, 33), True), ((7,), False), ((4096,), True), ((3, 5, 7), True), ((129,), False), ((12289,), True)]]
    odd = torch.nn.Parameter(big[1:1001])            # a view that is not 16-byte aligned: the scalar path
    params.append(odd)
    ours = EMAModel(params, update_after_step=2)
    ora = Oracle(params, update_after_step=2)
    frozen_shadows = [s for s, p in zip(ours.shadow_params, params) if not p.requires_grad]
    for t in range(6):
        with torch.no_grad():
            for i, p in enumerate(params):
                if p.requires_grad:
                    p.add_(torch.randn_like(p) * 0.1)
            if t == 4:
                params[1].add_(1.0)                       # a frozen tensor moved: the next step copies it
        v_frozen = [s._version for s in frozen_shadows]
        l0 = raw.LAUNCHES[0]
        ours.step(params)
        assert raw.LAUNCHES[0] - l0 == 2
        ora.step(params)
        torch.cuda.synchronize()
        copied = [s._version != v for s, v in zip(frozen_shadows, v_frozen)]
        assert copied == ([True, False] if t == 4 else [False, False]), t
        for a, b in zip(ours.shadow_params, ora.shadow_params):
            assert torch.equal(a, b), t
        assert ours.cur_decay_value == ora.cur_decay_value and ours.optimization_step == ora.optimization_step


@pytest.mark.parametrize("name", list(CONFIGS))
def test_device_decay_over_graph_replays(name):
    from oracle.svd_ema_oracle import get_decay
    from svd_xtend_b200.ema import EMAModel
    kw = CONFIGS[name]
    p = torch.nn.Parameter(torch.randn(4096, device=DEV))
    ema = EMAModel([p], **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ema.step([p])                                    # builds the job table (t = 1)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ema.step([p])
    ema.optimization_step = 1                            # the capture itself did not run the kernels; keep the count honest
    pow_sched = kw.get("use_ema_warmup", False)
    for start in (1, 2 ** 31):
        ema.optimization_step = start
        for t in range(start + 1, start + 40):
            graph.replay()
            torch.cuda.synchronize()
            assert ema.optimization_step == t
            want = np.float32(get_decay(t, **kw))
            got = np.float32(ema.cur_decay_value)
            omd_want, omd_got = np.float32(1 - get_decay(t, **kw)), np.float32(ema._state[8].item())
            if pow_sched:
                assert abs(int(got.view(np.int32)) - int(want.view(np.int32))) <= 1, (t, got, want)
                assert abs(int(omd_got.view(np.int32)) - int(omd_want.view(np.int32))) <= 1, (t, omd_got, omd_want)
            else:
                assert got == want and omd_got == omd_want, (t, got, want)


def test_attached_ema_in_graphed_step_follows_the_oracle_recurrence():
    from oracle.svd_ema_oracle import get_decay
    from oracle.svd_unet_oracle import TINY_CONFIG, edm_loss
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.train import FusedAdamW, GraphedStep, ParamArena
    _, ours = _build(TINY_CONFIG, seed=23)
    _train_filter(ours)
    ours.train()
    ema = EMAModel(ours.parameters())
    arena = ParamArena(ours)
    ours.attach_arena(arena)
    opt = FusedAdamW(arena, lr=2e-3, weight_decay=1e-2)
    opt.attach_ema(ema)
    opt.on_updated = lambda: ours.refresh_trainable_operands(shadow_current=True)
    e = arena.data.clone()
    assert torch.equal(ema._flat, e)
    from test_boundary_gpu import _tiny_batch
    batch = _tiny_batch(31)

    def step(b):
        arena.zero_grad()
        pred = ours(b["sample"], b["timestep"], b["encoder_hidden_states"], added_time_ids=b["added_time_ids"]).sample
        loss = edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"])
        loss.backward()
        opt.step()
        return loss

    graphed = GraphedStep(step, batch, warmup=3, restore=opt.snapshot_tensors(),
                          on_restored=lambda: ours.refresh_trainable_operands(shadow_current=True))
    assert torch.equal(ema._flat, e) and ema.optimization_step == 0     # warm-up / capture left the EMA alone
    with pytest.raises(RuntimeError, match="attached"):
        ema.step(ours.parameters())
    for t in range(1, 7):
        graphed(batch)
        torch.cuda.synchronize()
        e.sub_((1 - get_decay(t)) * (e - arena.data))
        assert torch.equal(ema._flat, e), t
    assert ema.optimization_step == 6
    ps = list(ours.parameters())
    i = next(k for k, p in enumerate(ps) if p.requires_grad)
    o = arena.offset_of[ps[i]]
    assert torch.equal(ema.shadow_params[i].reshape(-1), e[o:o + ps[i].numel()])


@pytest.mark.parametrize("graphs", [False, True])
def test_script_validation_loop_with_drop_in_ema(graphs):
    """train_svd.py --use_ema with the unchanged loop: torch.optim.AdamW, ema.step after every optimizer step, then
    store / copy_to / validation forward / restore (:1101-1104, :1152-1154)"""
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.train import ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    from test_boundary_gpu import _call, _tiny_batch
    oracle, ours = _build(TINY_CONFIG, seed=29)
    _train_filter(ours)
    ours.train()
    ema = EMAModel(ours.parameters(), model_cls=Ours, model_config=ours.config)
    runner = ours.enable_cuda_graphs(warmup=2) if graphs else None
    if not graphs:
        ours.attach_arena(ParamArena(ours))
    arena = ours._arena
    opt = torch.optim.AdamW([p for p in ours.parameters() if p.requires_grad], lr=3e-3, weight_decay=1e-2)
    batch, vbatch = _tiny_batch(41), _tiny_batch(42)
    for _ in range(5):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, loss = _loss(ours, batch)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        ema.step(ours.parameters())
    with torch.no_grad():
        _call(ours, vbatch)                   # operands current for the training weights
    torch.cuda.synchronize()
    train_entry = [e for e in runner.entries.values() if e.g_bwd is not None] if graphs else None
    masters = [p.detach().clone() for p in ours.parameters()]
    shadow = arena.shadow.clone()
    transposes = [dst.clone() for _, dst, _, _ in arena._tjobs]
    ema.store(ours.parameters())
    ema.copy_to(ours.parameters())
    with torch.no_grad():
        out = _call(ours, vbatch)
        fresh = Ours(**TINY_CONFIG).to(DEV)
        fresh.load_state_dict(ours.state_dict())
        ref_ours = _call(fresh, vbatch)
        oracle.load_state_dict(ours.state_dict())
        ref = _call(oracle, vbatch)
    torch.cuda.synchronize()
    assert _rel(out, ref) < 2e-2 and _rel(out, ref_ours) < 2.5e-2, (_rel(out, ref), _rel(out, ref_ours))
    for p, s in zip(ours.parameters(), ema.shadow_params):
        assert torch.equal(p, s)
    ema.restore(ours.parameters())
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = _loss(ours, batch)          # the next training step re-derives the operands from the restored masters
    loss.backward()
    torch.cuda.synchronize()
    for p, b in zip(ours.parameters(), masters):
        assert torch.equal(p, b)
    assert torch.equal(arena.shadow, shadow)
    for (_, dst, _, _), b in zip(arena._tjobs, transposes):
        assert torch.equal(dst, b)
    if graphs:
        now = [e for e in runner.entries.values() if e.g_bwd is not None]
        assert len(train_entry) == 1 and now and now[0] is train_entry[0], "validation dropped the captured training graphs"
