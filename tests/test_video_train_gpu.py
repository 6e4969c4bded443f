"""Training from video frames on the H100 (svd_xtend_b200.video_train): the two batch-assembly kernels bit for bit against the
oracle (oracle/svd_train_batch_oracle.py), the tiny composition VAE -> CLIP -> UNet -> loss -> backward against the oracle
models, the captured VideoTrainStep against its eager form, and the SVD configuration against the hand composition of the
package's stages."""
import pytest
import torch

DEV = "cuda:0"
TINY_VAE = dict(in_channels=3, latent_channels=4, block_out_channels=(64, 64, 128, 128), layers_per_block=1, scaling_factor=0.18215)


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _frames(B, F, H, W, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, F, 3, H, W, generator=g) * 2 - 1).to(DEV, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(64, 128), (128, 64)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_frames_in_bitwise(H, W, dtype):
    from oracle.svd_train_batch_oracle import frames_in
    from svd_xtend_b200 import raw
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    B, F = 2, 3
    x = _frames(B, F, H, W, 1, dtype)
    eps = torch.randn(B, 3, H, W, device=DEV)
    sig = torch.tensor([0.05, 0.2], device=DEV)
    rows = torch.full((B * (F + 1) * H * W, 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    raw.vae_frames_in(x, eps, sig, rows)
    ref = frames_in(x.float(), eps, sig)
    want = ref.permute(0, 2, 3, 1).reshape(-1, 3).to(torch.bfloat16)
    assert torch.equal(rows[:, :3].view(torch.int16), want.view(torch.int16))
    assert torch.equal(rows[:, 3:].float(), torch.zeros_like(rows[:, 3:].float()))
    clip_rows = torch.empty(B * F * H * W, 64, device=DEV, dtype=torch.bfloat16)
    raw.nchw_to_nhwc(x.reshape(B * F, 3, H, W), clip_rows, B * F, 3, H, W, 64)
    assert torch.equal(rows[:B * F * H * W].view(torch.int16), clip_rows.view(torch.int16))
    # one encode of the rows is the encode of the concatenated frames (encode = the row conversion + _run_rows). Two encodes of
    # the same input differ in the last bits (fp32 atomics of the GroupNorm statistics), so the bound is their spread.
    torch.manual_seed(3)
    with torch.device(DEV):
        vae = AutoencoderKLTemporalDecoder(**TINY_VAE).requires_grad_(False)
    with torch.no_grad():
        got = vae._run_rows(rows, B * (F + 1), H, W).to(dtype)
        e1, e2 = (vae.encode(ref.to(dtype)).latent_dist for _ in range(2))
    m1, m2 = (torch.cat([e.mean, e.logvar], 1) for e in (e1, e2))
    spread = _rel(m2, m1)
    print(f"frames-in encode {H}x{W} {dtype}: rel-l2 to encode {_rel(got, m1):.3e} (two encodes {spread:.3e})")
    assert _rel(got, m1) <= 4 * spread + 1e-6


@pytest.mark.gpu
def test_edm_prepare_bitwise():
    from oracle.svd_train_batch_oracle import prepare
    from svd_xtend_b200 import raw
    B, F, h, w = 4, 3, 8, 16
    g = torch.Generator(device=DEV).manual_seed(5)
    mom = torch.randn(B * (F + 1), 8, h, w, device=DEV, generator=g) * 3
    mom[:, 4:].mul_(8)                                   # logvars beyond both clamp bounds
    le, nz = (torch.randn(B * F, 4, h, w, device=DEV, generator=g) for _ in range(2))
    ce = torch.randn(B, 4, h, w, device=DEV, generator=g)
    sigma = torch.tensor([0.02, 1.0, 7.5, 80.0], device=DEV)
    mask = torch.tensor([1.0, 0.0, 0.0, 1.0], device=DEV)            # the four dropout regions give masks 1, 0, 0, 1
    sample = torch.empty(B, F, 8, h, w, device=DEV)
    noisy, lat = torch.empty(B, F, 4, h, w, device=DEV), torch.empty(B, F, 4, h, w, device=DEV)
    raw.edm_prepare(mom, le, nz, ce, sigma, mask, 0.18215, sample, noisy, lat)
    rs, rn, rl = prepare(mom, le, nz, ce, sigma, mask, 0.18215)
    for a, b, what in ((sample, rs, "sample"), (noisy, rn, "noisy"), (lat, rl, "latents")):
        assert torch.equal(a.view(torch.int32), b.contiguous().view(torch.int32)), (what, (a - b).abs().max().item())


def _pairs(seed, vae_cfg, unet_cfg, clip_cfg):
    from oracle.svd_clip_oracle import CLIPVisionModelWithProjection as OClip
    from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as OUnet
    from oracle.svd_vae_oracle import AutoencoderKLTemporalDecoder as OVae
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(seed)
    out = []
    for O, P, kw in ((OVae, AutoencoderKLTemporalDecoder, vae_cfg), (OClip, CLIPVisionModelWithProjection, clip_cfg),
                     (OUnet, UNetSpatioTemporalConditionModel, unet_cfg)):
        o = O(**kw).to(DEV)
        with torch.no_grad():
            for n, p in o.named_parameters():
                if "norm" in n:
                    p.add_(0.1 * torch.randn_like(p))
        with torch.device(DEV):
            ours = P(**kw)
        ours.load_state_dict(o.state_dict())
        out.append((o.eval().requires_grad_(False), ours.eval().requires_grad_(False)))
    for m in (out[2][0], out[2][1]):
        for n, p in m.named_parameters():
            if "temporal_transformer_block" in n:           # train_svd.py:761-766
                p.requires_grad_(True)
        m.train()
    return out


def _tiny_cfgs():
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from oracle.svd_unet_oracle import TINY_CONFIG
    return TINY_VAE, TINY_CONFIG, dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"])


@pytest.mark.gpu
def test_tiny_composition_matches_oracle():
    from oracle.svd_clip_oracle import encode_image as oracle_encode_image
    from oracle.svd_train_batch_oracle import edm_loss as oracle_loss, frames_in, log_normal, train_batch
    from svd_xtend_b200.video_train import assemble_train_batch, draw_train_noise
    from svd_xtend_b200.workload import edm_loss
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    (ov, v), (oc, c), (ou, u) = _pairs(31, *_tiny_cfgs())
    B, F, H, W, p = 2, 4, 64, 128, 0.1
    x = _frames(B, F, H, W, 2)
    d = draw_train_noise(B, F, H, W, generator=torch.Generator().manual_seed(9), device=DEV)
    d["dropout_u"] = torch.tensor([0.5, 0.15], device=DEV)          # clip 0 keeps both conditionings, clip 1 drops both
    b = assemble_train_batch(v, c, u, x, d, conditioning_dropout_prob=p)
    pred = u(b["sample"], b["timestep"], b["encoder_hidden_states"], added_time_ids=b["added_time_ids"]).sample
    loss = edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"])
    loss.backward()
    torch.cuda.synchronize()

    def oracle(autocast):
        for prm in ou.parameters():
            prm.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            with torch.no_grad():
                frames = frames_in(x, d["cond_pixel_eps"], log_normal(d["cond_u"], -3.0, 0.5))
                mom = ov.quant_conv(ov.encoder(frames)).float()
                emb = oracle_encode_image(oc, x[:, 0]).float()
            ob = train_batch(mom[:B * F], mom[B * F:], emb, d, conditioning_dropout_prob=p, dtype=torch.float32)
            op = ou(ob["sample"], ob["timestep"], ob["encoder_hidden_states"], added_time_ids=ob["added_time_ids"]).sample
        ol = oracle_loss(op.float(), ob["noisy"], ob["latents"], ob["sigmas"])
        ol.backward()
        return ob, op.detach().float(), ol.detach(), {n: prm.grad.clone() for n, prm in ou.named_parameters() if prm.requires_grad}

    ob, op, ol, og = oracle(False)
    _, ap, al, ag = oracle(True)
    for k in ("sample", "noisy", "latents", "encoder_hidden_states"):
        e = _rel(b[k], ob[k])
        print(f"batch {k}: rel-l2 {e:.3e}")
        assert e <= 2e-2, k
    for k in ("timestep", "added_time_ids", "sigmas"):
        assert torch.allclose(b[k], ob[k], rtol=1e-6, atol=0), k
    assert (b["encoder_hidden_states"][1] == 0).all() and (b["sample"][1, :, 4:] == 0).all()
    e, ea = _rel(pred, op), _rel(ap, op)
    print(f"prediction rel-l2 {e:.3e} (oracle under bf16 autocast {ea:.3e}); loss {loss.item():.5f} oracle {ol.item():.5f}")
    assert e <= max(2 * ea, 2e-2)
    grads = dict(u.named_parameters())
    worst = 0.0
    for n, gref in og.items():
        eg, eag = _rel(grads[n].grad, gref), _rel(ag[n], gref)
        worst = max(worst, eg)
        assert eg <= max(3 * eag, 5e-2), (n, eg, eag)
    print(f"gradients: worst rel-l2 {worst:.3e} over {len(og)} tensors")


def _train_setup(seed, optim="fused", cfgs=None, frames=(1, 4, 64, 128), dropout=0.1, cuda_graph=True, grad_ckpt=False):
    from svd_xtend_b200.train import FusedAdamW, FusedAdamW8bit, ParamArena
    from svd_xtend_b200.video_train import VideoTrainStep
    (_, v), (_, c), (_, u) = _pairs(seed, *(cfgs or _tiny_cfgs()))
    if grad_ckpt:
        u.enable_gradient_checkpointing()
    arena = ParamArena(u)
    u.attach_arena(arena)
    opt = (FusedAdamW if optim == "fused" else FusedAdamW8bit)(arena, lr=1e-4)
    opt.on_updated = lambda: u.refresh_trainable_operands(shadow_current=True)
    gen = torch.Generator(DEV).manual_seed(123)
    snap = [t.clone() for t in opt.snapshot_tensors()]
    gstate = gen.get_state()
    step = VideoTrainStep(u, v, c, opt, frames_shape=frames, conditioning_dropout_prob=dropout, generator=gen, cuda_graph=cuda_graph)
    torch.cuda.synchronize()
    unchanged = all(torch.equal(a, b) for a, b in zip(snap, opt.snapshot_tensors())) and torch.equal(gstate, gen.get_state())
    seen = []
    draw = step.draw

    def recording_draw():
        dd = draw()
        seen.append({k: t.clone() for k, t in dd.items()})
        return dd
    step.draw = recording_draw
    return step, opt, arena, seen, unchanged


@pytest.mark.gpu
@pytest.mark.parametrize("optim", ["fused", "8bit"])
def test_graphed_step_matches_eager(optim):
    torch.backends.cuda.matmul.allow_tf32 = False
    x = [_frames(1, 4, 64, 128, 40 + i) for i in range(3)]

    def run(graph):
        step, opt, arena, seen, unchanged = _train_setup(7, optim=optim, cuda_graph=graph)
        assert unchanged, "construction changed the weights, the optimizer state or the generator"
        losses = []
        for i in range(3):
            if i == 2:
                opt.lr = 5e-5
            losses.append(step(x[i]).item())
        torch.cuda.synchronize()
        assert opt.t == 3
        return losses, arena.grad.clone(), arena.data.clone(), seen

    l1, g1, p1, d1 = run(False)
    l2, g2, p2, d2 = run(False)
    lg, gg, pg, dg = run(True)
    for a, b in zip(d1, dg):
        assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    spread_l = max(abs(a - b) for a, b in zip(l1, l2))
    spread_g, spread_p = _rel(g2, g1), _rel(p2, p1)
    dl = max(abs(a - b) for a, b in zip(lg, l1))
    dgr, dp = _rel(gg, g1), _rel(pg, p1)
    print(f"{optim}: losses eager {l1} graphed {lg}; loss spread {spread_l:.3e} graphed-eager {dl:.3e}; grad spread {spread_g:.3e} "
          f"graphed-eager {dgr:.3e}; weights spread {spread_p:.3e} graphed-eager {dp:.3e}")
    assert all(map(lambda t: t == t, lg))
    assert dl <= 4 * spread_l + 1e-6 * max(map(abs, l1))
    assert dgr <= 4 * spread_g + 1e-6
    assert dp <= 4 * spread_p + 1e-7


@pytest.mark.gpu
def test_svd_config_graphed_step_matches_hand_composition():
    """14 x 320 x 512, B = 1, the as-scripted trainable set, FusedAdamW: the graphed step against the package's stages composed by
    hand (eager assemble_train_batch + UNet + edm_loss + backward) on the same draws, within the spread of repeated eager runs"""
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from svd_xtend_b200.video_train import assemble_train_batch
    from svd_xtend_b200.workload import SVD_CONFIG, edm_loss
    from oracle.svd_vae_oracle import VAE_CONFIG
    cfgs = (VAE_CONFIG, SVD_CONFIG, CLIP_CONFIG)
    x = _frames(1, 14, 320, 512, 50)
    step, opt, arena, seen, unchanged = _train_setup(8, cfgs=cfgs, frames=(1, 14, 320, 512))
    assert unchanged
    u = step.unet
    w0 = arena.data.clone()
    loss = step(x).item()
    torch.cuda.synchronize()
    g_graph = arena.grad.clone()
    assert loss == loss and abs(loss) < float("inf")
    arena.data.copy_(w0)
    arena.refresh_shadow()
    u.refresh_trainable_operands(shadow_current=True)
    # The GroupNorm channel sums are added across CTAs by atomics in a varying order, so the loss moves by ~3e-5 relative from
    # run to run. One pair of eager runs is too small a sample of that spread: a graphed loss within the noise fell outside 4x one
    # pair's difference about one time in ten. The loss spread is the largest difference over four eager reruns.
    hand = []
    for i in range(5):
        arena.zero_grad()
        b = assemble_train_batch(step.vae, step.image_encoder, u, x, seen[0], conditioning_dropout_prob=0.1)
        pred = u(b["sample"], b["timestep"], b["encoder_hidden_states"], added_time_ids=b["added_time_ids"]).sample
        lh = edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"])
        lh.backward()
        torch.cuda.synchronize()
        hand.append((lh.item(), arena.grad.clone() if i < 2 else None))
    spread = _rel(hand[1][1], hand[0][1])
    e = _rel(g_graph, hand[0][1])
    spread_l = max(abs(h - hand[0][0]) for h, _ in hand[1:])
    print(f"SVD config: loss graphed {loss:.5f} hand {' / '.join(f'{h:.5f}' for h, _ in hand)}; grad rel-l2 {e:.3e} (eager spread "
          f"{spread:.3e}); max memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert e <= 4 * spread + 1e-6
    assert abs(loss - hand[0][0]) <= 4 * spread_l + 1e-5 * abs(hand[0][0])
