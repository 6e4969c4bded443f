"""Gradient accumulation and global gradient-norm clipping on the H100: the deterministic sum-of-squares kernels against fp64
torch, the clipped fused updates against clip_grad_norm_ + torch.optim.AdamW and bit for bit against the unclipped update fed
the clipped gradient, two backward passes without zero_grad against the sum of the two (eager, captured with an arena, and
captured without one), and VideoTrainStep(gradient_accumulation_steps=2) against its eager form and against one B = 2 step."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _release_earlier_graphs():
    """the steps of earlier tests hold CUDA graphs in reference cycles (optimizer hooks): free them before a new capture"""
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    yield


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _sumsq_buf():
    from svd_xtend_b200 import raw
    return torch.full((1 + raw.SUMSQ_PARTIALS,), float("nan"), device=DEV, dtype=torch.float64)


# ---- 1. the norm kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4 * 1000 + 3, 397_620_480, 0])
def test_grad_sumsq_matches_fp64_and_repeats_bit_for_bit(n):
    """n = 0 stands for an all-zero gradient of 4099 elements; 397,620,480 is the as-scripted trainable arena"""
    from svd_xtend_b200 import raw
    if n == 0:
        g = torch.zeros(4099, device=DEV)
    else:
        g = torch.empty(n, device=DEV).normal_(0.0, 1e-3, generator=torch.Generator(DEV).manual_seed(n))
    s1, s2 = _sumsq_buf(), _sumsq_buf()
    raw.grad_sumsq(g, s1)
    raw.grad_sumsq(g, s2)
    ref = sum((c.double() ** 2).sum().item() for c in g.split(1 << 24))
    got = s1[0].item()
    assert torch.equal(s1[0], s2[0])
    assert abs(got - ref) <= 1e-10 * ref if ref else got == 0.0
    graph = torch.cuda.CUDAGraph()             # and inside a captured graph, replay after replay
    s3 = _sumsq_buf()
    with torch.cuda.graph(graph):
        raw.grad_sumsq(g, s3)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(s3[0], s1[0])


@pytest.mark.parametrize("world,rank", [(1, 0), (2, 1), (5, 3)])
def test_grad_sumsq_p2p_is_the_sumsq_of_the_rank_order_sum(world, rank):
    """one device, the 'peer' arenas local tensors (as the svdx_adamw_step_p2p test does)"""
    from svd_xtend_b200 import raw
    n_total = 8192 * world
    n = n_total // world
    lo = rank * n
    grads = [torch.randn(n_total, device=DEV, generator=torch.Generator(DEV).manual_seed(30 + r)) for r in range(world)]
    gsum = grads[0][lo:lo + n].clone()
    for r in range(1, world):
        gsum += grads[r][lo:lo + n]
    s_p2p, s_ref = _sumsq_buf(), _sumsq_buf()
    raw.grad_sumsq_p2p(grads, lo, n, s_p2p)
    raw.grad_sumsq(gsum, s_ref)
    torch.cuda.synchronize()
    assert torch.equal(s_p2p[0], s_ref[0])


def test_clip_coef_kernel_nan_inf_and_clamp():
    from svd_xtend_b200 import raw
    out = torch.zeros(2, device=DEV)
    mx = torch.tensor([2.0], device=DEV)
    for sumsq, scale, want_coef in ((1.0, 1.0, 1.0), (16.0, 1.0, None), (16.0, 0.25, 1.0), (float("inf"), 1.0, 0.0),
                                    (float("nan"), 1.0, "nan")):
        s = torch.tensor([sumsq], device=DEV, dtype=torch.float64)
        raw.clip_coef(s, mx, scale, out)
        total, coef = out.tolist()
        t_ref = torch.sqrt(torch.tensor(sumsq, dtype=torch.float64)).float() * scale
        c_ref = torch.clamp(2.0 / (t_ref + 1e-6), max=1.0)
        if want_coef == "nan":
            assert coef != coef and total != total
        else:
            assert total == t_ref.item() and coef == c_ref.item()
            if want_coef is not None:
                assert coef == want_coef


# ---- 2. clipped updates ----------------------------------------------------------------------------------------------------------
def _tiny_net(seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(64, 96), torch.nn.Linear(96, 40), torch.nn.Linear(40, 7)).to(DEV)


def _fill_grads(arena, seed, scale):
    g = torch.Generator(DEV).manual_seed(seed)
    arena.zero_grad()
    for p in arena.params:
        arena.grad_views[p].copy_(torch.randn(p.shape, device=DEV, generator=g) * scale)


@pytest.mark.parametrize("max_norm", [0.05, 1e3])
def test_fused_adamw_clip_matches_torch(max_norm):
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    torch.backends.cuda.matmul.allow_tf32 = False
    net, ref = _tiny_net(1), _tiny_net(1)
    arena = ParamArena(net)
    opt = FusedAdamW(arena, lr=1e-3, weight_decay=1e-2, max_grad_norm=max_norm)
    topt = torch.optim.AdamW(ref.parameters(), lr=1e-3, weight_decay=1e-2)
    for step in range(3):
        _fill_grads(arena, 100 + step, 0.1)
        for p, q in zip(arena.params, ref.parameters()):
            q.grad = arena.grad_views[p].clone()
        g_before = arena.grad.clone()
        opt.step()
        tnorm = torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        topt.step()
        torch.cuda.synchronize()
        assert abs(opt.grad_norm.item() - tnorm.item()) <= 1e-6 * tnorm.item()
        assert torch.equal(arena.grad, g_before), "the gradient arena is not rescaled"
        for p, q in zip(arena.params, ref.parameters()):
            assert torch.allclose(p, q, rtol=1e-5, atol=1e-6), (step, (p - q).abs().max().item())
    assert (opt._clip[1].item() < 1.0) == (max_norm < 1)


def _pair(form, seed, ema=False, **kw):
    """two optimizers of one form over two copies of one arena: the clipped one and the unclipped reference"""
    from svd_xtend_b200 import train
    from svd_xtend_b200.ema import EMAModel
    out = []
    for clip in (True, False):
        net = _tiny_net(seed)
        arena = train.ParamArena(net)
        cls = getattr(train, form)
        opt = cls(arena, lr=1e-3, max_grad_norm=0.05 if clip else None, **kw)
        if ema:
            opt.attach_ema(EMAModel(net.parameters(), decay=0.9))
        out.append((arena, opt))
    return out


@pytest.mark.parametrize("form,ema", [("FusedAdamW", False), ("FusedAdamW", True), ("FusedAdamW8bit", False),
                                      ("FusedAdamW8bit", True)])
def test_clipped_update_is_the_unclipped_update_of_the_clipped_gradient(form, ema):
    """bit for bit: the clipped step against the unclipped step fed arena.grad * coef (the device's own coefficient)"""
    kw = {"min_8bit_size": 1024} if form == "FusedAdamW8bit" else {}
    (a1, o1), (a2, o2) = _pair(form, 3, ema=ema, **kw)
    for step in range(3):
        _fill_grads(a1, 200 + step, 0.1)
        o1.step()
        a2.grad.copy_(a1.grad * o1._clip[1])
        o2.step()
        torch.cuda.synchronize()
        assert o1._clip[1].item() < 1.0
        assert torch.equal(a1.data, a2.data) and torch.equal(a1.shadow, a2.shadow)
        if ema:
            assert torch.equal(o1.ema._flat, o2.ema._flat)


@pytest.mark.parametrize("form", ["FusedAdamW", "FusedAdamW8bit"])
def test_clip_acts_on_the_gradient_scaled_by_grad_scale(form):
    """step(grad_scale=0.5) on g is bit for bit step() on 0.5 * g (a power of two: every product is exact), norm included"""
    from svd_xtend_b200 import train
    kw = {"min_8bit_size": 1024} if form == "FusedAdamW8bit" else {}
    (a1, o1), (a2, o2) = [(a, getattr(train, form)(a, lr=1e-3, max_grad_norm=0.05, **kw))
                          for a in (train.ParamArena(_tiny_net(5)), train.ParamArena(_tiny_net(5)))]
    for step in range(2):
        _fill_grads(a1, 400 + step, 0.1)
        a2.grad.copy_(a1.grad * 0.5)
        o1.step(grad_scale=0.5)
        o2.step()
        torch.cuda.synchronize()
        assert o1._clip[1].item() < 1.0
        assert torch.equal(o1.grad_norm, o2.grad_norm) and torch.equal(a1.data, a2.data)


def test_sharded_forms_at_world_one_equal_fused_adamw():
    from svd_xtend_b200.train import FusedAdamW, P2PShardedAdamW, ParamArena, ShardedAdamW
    runs = []
    for cls in (FusedAdamW, ShardedAdamW, P2PShardedAdamW):
        arena = ParamArena(_tiny_net(4))
        opt = cls(arena, lr=1e-3, max_grad_norm=0.05)
        for step in range(3):
            _fill_grads(arena, 300 + step, 0.1)
            opt.step()
        torch.cuda.synchronize()
        runs.append((arena.data.clone(), arena.shadow.clone(), opt.grad_norm.clone(), opt._clip.clone()))
    for r in runs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(runs[0], r))


def test_grad_mul_of_one_and_none_give_the_same_bits():
    from svd_xtend_b200 import raw
    n = 4099
    g = torch.Generator(DEV).manual_seed(5)
    p0, grad = torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)
    one = torch.ones(1, device=DEV)
    res = []
    for gm in (None, one):
        p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        state = torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0], device=DEV)
        for _ in range(2):
            raw.adamw_graph(p, grad, m, v, state, 0.5, grad_mul=gm)
        res.append((p, m, v))
    assert all(torch.equal(x, y) for x, y in zip(*res))


# ---- 3. accumulation in the engine -----------------------------------------------------------------------------------------------
def _engine_model(mode):
    from types import SimpleNamespace
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.train import ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    torch.manual_seed(41)
    with torch.device(DEV):
        m = UNetSpatioTemporalConditionModel(**TINY_CONFIG)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
    if mode == "mixed":
        m.to(torch.bfloat16)
    m.add_adapter(SimpleNamespace(r=4, lora_alpha=4, init_lora_weights="gaussian", target_modules=["to_k", "to_q", "to_v", "to_out.0"]))
    m.requires_grad_(True)                     # every parameter trainable, the adapter's factors too
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "lora" in n:
                p.data = p.data.float()        # mixed: bf16 base + fp32 LoRA factors, so no arena
        for mod in m.modules():
            if hasattr(mod, "lora_B"):
                mod.lora_B["default"].weight.normal_(0, 0.05)
    m.train()
    if mode == "eager":
        m.attach_arena(ParamArena(m))
    else:
        m.enable_cuda_graphs(warmup=2)
        assert (m._arena is None) == (mode == "mixed")
    return m


def _grads(m, batches, zero=True):
    from oracle.svd_unet_oracle import edm_loss
    params = [p for p in m.parameters() if p.requires_grad]
    if zero:
        for p in params:
            p.grad = None
    for b in batches:
        x = {k: (v.to(torch.bfloat16) if v.is_floating_point() and next(m.parameters()).dtype == torch.bfloat16
                 and k in ("sample", "encoder_hidden_states", "added_time_ids") else v) for k, v in b.items()}
        pred = m(x["sample"], x["timestep"], x["encoder_hidden_states"], x["added_time_ids"]).sample
        edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"]).backward()
    torch.cuda.synchronize()
    return [p.grad.float().clone() for p in params]


@pytest.mark.parametrize("mode", ["eager", "graphs", "mixed"])
def test_two_backwards_without_zero_grad_sum_their_gradients(mode):
    """every parameter-gradient writer adds into .grad: backward(A) + backward(B) without zero_grad equals grad(A) + grad(B).
    Every parameter and a LoRA adapter trainable. eager: with an arena; graphs: under enable_cuda_graphs (arena); mixed: bf16
    base and fp32 adapter under enable_cuda_graphs (no arena: the captured backward's static gradient buffers)"""
    from oracle.svd_unet_oracle import TINY_CONFIG, synthetic_batch
    m = _engine_model(mode)
    A, B = (synthetic_batch(1, 4, 16, 16, seed=s, device=DEV, cross_dim=TINY_CONFIG["cross_attention_dim"]) for s in (61, 62))
    for _ in range(3):                          # warm-up and capture (graph modes), then every call below replays
        _grads(m, [A])
    ga, ga2, gb = _grads(m, [A]), _grads(m, [A]), _grads(m, [B])
    gab = _grads(m, [A, B])
    names = [n for n, p in m.named_parameters() if p.requires_grad]
    lora = [i for i, n in enumerate(names) if "lora" in n]
    assert lora and len(lora) < len(names)
    for what, ix in (("all", range(len(ga))), ("lora", lora)):
        flat = lambda gs: torch.cat([gs[i].reshape(-1) for i in ix])
        spread = _rel(flat(ga2), flat(ga))
        err = _rel(flat(gab), flat([x + y for x, y in zip(ga, gb)]))
        print(f"{mode} {what}: spread {spread:.3e} accumulated-vs-sum {err:.3e}")
        tol = 1e-2 if mode == "mixed" and what == "all" else 1e-5     # bf16 .grad of bf16 parameters: one bf16 rounding of the sum
        assert err <= 4 * spread + tol
    if m._graphs is not None:
        assert any(e.calls >= 6 for e in m._graphs.entries.values() if e.g_bwd is not None)


# ---- 4. VideoTrainStep at k = 2 --------------------------------------------------------------------------------------------------
def _video_setup(seed, k, cuda_graph, frames=(1, 4, 64, 128), ema=False, max_grad_norm=None):
    from test_video_train_gpu import _pairs, _tiny_cfgs
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    from svd_xtend_b200.video_train import VideoTrainStep
    (_, v), (_, c), (_, u) = _pairs(seed, *_tiny_cfgs())
    e = EMAModel(u.parameters()) if ema else None
    arena = ParamArena(u)
    u.attach_arena(arena)
    opt = FusedAdamW(arena, lr=1e-4, max_grad_norm=max_grad_norm)
    if e is not None:
        opt.attach_ema(e)
    opt.on_updated = lambda: u.refresh_trainable_operands(shadow_current=True)
    gen = torch.Generator(DEV).manual_seed(123)
    arena.grad.fill_(1.0)                     # construction must leave the arena zeroed
    step = VideoTrainStep(u, v, c, opt, frames_shape=frames, conditioning_dropout_prob=0.1, generator=gen, cuda_graph=cuda_graph,
                          gradient_accumulation_steps=k)
    torch.cuda.synchronize()
    assert bool((arena.grad == 0).all()) if k > 1 else True
    if max_grad_norm is not None:
        assert opt.grad_norm.item() == 0.0, "the capture's warm-up updates must not leave their norm behind"
    return step, opt, arena


def test_video_step_k2_graphed_matches_eager():
    from test_video_train_gpu import _frames
    torch.backends.cuda.matmul.allow_tf32 = False
    x = [_frames(1, 4, 64, 128, 40 + i) for i in range(4)]

    def run(graph):
        step, opt, arena = _video_setup(7, 2, graph, ema=True)
        losses, syncs = [], []
        for i in range(4):
            if i == 2:
                opt.lr = 5e-5
            losses.append(step(x[i]).item())
            syncs.append(step.sync_gradients)
            if i == 2:
                g_mid = arena.grad.clone()
        torch.cuda.synchronize()
        assert syncs == [False, True, False, True]
        assert opt.t == 2 and opt.ema._state[0].item() == 2.0
        assert bool((arena.grad == 0).all())
        return losses, g_mid, arena.data.clone()

    l1, g1, p1 = run(False)
    l2, g2, p2 = run(False)
    lg, gg, pg = run(True)
    spread_l = max(abs(a - b) for a, b in zip(l1, l2))
    spread_g, spread_p = _rel(g2, g1), _rel(p2, p1)
    dl, dgr, dp = max(abs(a - b) for a, b in zip(lg, l1)), _rel(gg, g1), _rel(pg, p1)
    print(f"k=2: losses eager {l1} graphed {lg}; grad spread {spread_g:.3e} graphed-eager {dgr:.3e}; weights spread "
          f"{spread_p:.3e} graphed-eager {dp:.3e}")
    assert dl <= 4 * spread_l + 1e-6 * max(map(abs, l1))
    assert dgr <= 4 * spread_g + 1e-6
    assert dp <= 4 * spread_p + 1e-7


def test_two_micro_steps_equal_one_batch_of_two():
    """k = 2 with B = 1 against k = 1 with B = 2 over the same frames and draws: the same gradient (so the 1 / k of the micro-step
    is right: the window's gradient is the mean over its clips, as the B = 2 step's is), the same clipped update and the same
    grad_norm, within the spread of two identical runs"""
    from test_video_train_gpu import _frames
    torch.backends.cuda.matmul.allow_tf32 = False
    x = [_frames(1, 4, 64, 128, 70 + i) for i in range(2)]
    clip = 0.05                                 # active on both sides: the update depends on the gradient's scale

    def accumulated(graph, draws=None):
        step, opt, arena = _video_setup(9, 2, graph, max_grad_norm=clip)
        seen, window = [], []
        draw = step.draw
        if draws is None:
            step.draw = lambda: seen.append(draw()) or seen[-1]
        else:
            step.draw = lambda: seen.append(draws[len(seen)]) or seen[-1]
        if not graph:                             # the window's gradient, just before the update consumes it
            update = step._update
            step._update = lambda: (window.append(arena.grad.clone()), update())
        losses = [step(xi).item() for xi in x]
        torch.cuda.synchronize()
        return losses, arena.data.clone(), opt.grad_norm.item(), (window[0] if window else None), seen

    def batched(draws):
        step, opt, arena = _video_setup(9, 1, True, frames=(2, 4, 64, 128), max_grad_norm=clip)
        both = {k: torch.cat([d[k] for d in draws]) for k in draws[0]}
        step.draw = lambda: both
        loss = step(torch.cat(x)).item()
        torch.cuda.synchronize()
        return loss, arena.data.clone(), opt.grad_norm.item(), arena.grad.clone()    # k = 1 zeroes at the start of a step

    la, pa, na, _, seen = accumulated(True)
    la2, pa2, na2, _, _ = accumulated(True)
    le, pe, ne, ge, _ = accumulated(False, seen)
    lb, pb, nb, gb = batched(seen)
    lb2, pb2, nb2, gb2 = batched(seen)
    spread_p = max(_rel(pa2, pa), _rel(pb2, pb))
    spread_g = _rel(gb2, gb)
    spread_n = max(abs(na2 - na), abs(nb2 - nb)) / nb
    dp, dg, dn = _rel(pa, pb), _rel(ge, gb), abs(na - nb) / nb
    print(f"accumulated losses {la} batched {lb}; gradient eager-accumulated-vs-batched {dg:.3e} (spread {spread_g:.3e}); "
          f"grad_norm graphed {na:.6g} eager {ne:.6g} batched {nb:.6g} (rel diff {dn:.3e}, spread {spread_n:.3e}); weights "
          f"{dp:.3e} (spread {spread_p:.3e})")
    assert nb > clip and na > clip, "the clip must be active for the update to depend on the gradient's scale"
    assert abs(sum(la) / 2 - lb) <= 1e-3 * abs(lb)
    assert dg <= 4 * spread_g + 1e-3              # B = 1 and B = 2 also differ in bf16 rounding (losses: ~2e-4)
    assert dn <= 4 * max(spread_n, spread_g) + 1e-3 and abs(ne - na) / na <= 4 * max(spread_n, spread_g) + 1e-3
    assert dp <= 4 * spread_p + 1e-6


# ---- 5. config 4 at k = 2 --------------------------------------------------------------------------------------------------------
def test_config4_k2_fits_one_card():
    """25 x 576 x 1024 (train_svd.py's default size), B = 1, the as-scripted trainable set, bf16 VAE / CLIP, encode_chunk_size 2:
    the two captured graphs of k = 2 build and replay a window on one 80 GB card"""
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    from svd_xtend_b200.video_train import VideoTrainStep
    from svd_xtend_b200.workload import BENCH_CONFIGS, SVD_CONFIG
    cfg = BENCH_CONFIGS[4]
    F, H, W = cfg["frames"], 8 * cfg["h"], 8 * cfg["w"]
    torch.manual_seed(1234)
    with torch.device(DEV):
        unet = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
        vae = AutoencoderKLTemporalDecoder(**VAE_CONFIG)
        clip = CLIPVisionModelWithProjection(**CLIP_CONFIG)
    for m in (unet, vae, clip):
        m.requires_grad_(False)
    vae.to(torch.bfloat16).eval()
    clip.to(torch.bfloat16).eval()
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:
            p.requires_grad_(True)
    unet.train()
    if cfg["grad_ckpt"]:
        unet.enable_gradient_checkpointing()
    arena = ParamArena(unet)
    unet.attach_arena(arena)
    opt = FusedAdamW(arena, lr=1e-5, max_grad_norm=1.0)
    opt.on_updated = lambda: unet.refresh_trainable_operands(shadow_current=True)
    torch.cuda.reset_peak_memory_stats()
    step = VideoTrainStep(unet, vae, clip, opt, frames_shape=(1, F, H, W), conditioning_dropout_prob=0.1,
                          generator=torch.Generator(DEV).manual_seed(0), encode_chunk_size=2, gradient_accumulation_steps=2)
    x = (torch.rand(1, F, 3, H, W, generator=torch.Generator().manual_seed(5)) * 2 - 1).to(DEV)
    losses = [step(x).item() for _ in range(2)]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"config 4, k = 2: losses {losses}, grad norm {opt.grad_norm.item():.4g}, peak max_memory_allocated {peak:.2f} GiB "
          f"on {torch.cuda.get_device_name(0)}")
    assert step.sync_gradients and opt.t == 1
    assert all(l == l for l in losses) and opt.grad_norm.item() > 0
    assert peak < 80
