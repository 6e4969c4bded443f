"""Training from decoded uint8 frames on the H100 (svd_xtend_b200.video_train, kernel svdx_frames_u8_in): the GPU resize against
Pillow's recorded outputs and the numpy oracle (oracle/svd_resize_oracle.py) bit for bit, its encoder rows against
svdx_vae_frames_in's rows of the oracle-resized frames, the encode in frame chunks, the uint8-input VideoTrainStep against its
eager form and against the float-input step, and the graphed step at train_svd.py's default size (25 x 576 x 1024) on one card."""
import os

import numpy as np
import pytest
import torch

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_golden.pt")
TINY_VAE = dict(in_channels=3, latent_channels=4, block_out_channels=(64, 64, 128, 128), layers_per_block=1, scaling_factor=0.18215)
bf16 = torch.bfloat16


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _u8(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)


def _oracle_frames(u8, H, W):
    """[B, F, H0, W0, 3] uint8 -> the oracle's resized, normalised fp32 frames [B, F, 3, H, W] (DummyDataset)"""
    from oracle.svd_resize_oracle import normalize, resize
    B, F = u8.shape[:2]
    out = np.stack([np.stack([normalize(resize(u8[b, f].numpy(), (W, H))) for f in range(F)]) for b in range(B)])
    return torch.from_numpy(out).permute(0, 1, 4, 2, 3).contiguous()


def _kernel(src, H, W, eps, sig, first=0, count=None):
    from svd_xtend_b200 import raw
    B, F, H0, W0, _ = src.shape
    count = B * (F + 1) - first if count is None else count
    ty, tx = raw.resize_taps(H0, H).to(DEV), raw.resize_taps(W0, W).to(DEV)
    rows = torch.full((count * H * W, 64), float("nan"), device=DEV, dtype=bf16)
    x0 = torch.full((B, 3, H, W), float("nan"), device=DEV)
    raw.frames_u8_in(src.to(DEV), ty, tx, eps, sig, rows, (H, W), first, count, x0)
    return rows, x0


def _cases():
    from oracle.svd_resize_oracle import source_frame, unpack_image
    g = torch.load(GOLDEN)
    out = [(c["name"], source_frame(c["seed"], *c["source"]), tuple(c["size"]), unpack_image(c["out"], tuple(c["size"]) + (3,)))
           for c in g["cases"]]
    src = _u8((1080, 1920, 3), 77)
    out.append(("1080x1920_to_576x1024", src, (576, 1024), None))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(8))
def test_kernel_resize_bitwise(i):
    """the clean first frame the kernel writes is normalize(resize(u8)): equal bit for bit to Pillow's golden output (and the
    oracle's), so the resize itself is Pillow's"""
    from oracle.svd_resize_oracle import normalize, resize
    name, src, (H, W), golden = _cases()[i]
    want_u8 = resize(src.numpy(), (W, H))
    if golden is not None:
        assert np.array_equal(want_u8, golden), name
    eps = torch.zeros(1, 3, H, W, device=DEV)
    sig = torch.zeros(1, device=DEV)
    rows, x0 = _kernel(src[None, None], H, W, eps, sig)
    want = torch.from_numpy(normalize(want_u8)).permute(2, 0, 1).to(DEV)
    assert torch.equal(x0[0].view(torch.int32), want.view(torch.int32)), name
    hw = H * W
    want_rows = want.permute(1, 2, 0).reshape(hw, 3).to(bf16)
    assert torch.equal(rows[:hw, :3].view(torch.int16), want_rows.view(torch.int16)), name
    assert torch.equal(rows[:, 3:].float(), torch.zeros_like(rows[:, 3:].float()))


@pytest.mark.gpu
def test_u8_rows_match_frames_in():
    """rows of uint8 frames = svdx_vae_frames_in rows of the oracle-resized, normalised frames, bit for bit: the clip frames and
    the noise-augmented conditioning frames, for the whole frame space and for frame ranges (uint8 and float forms)"""
    from svd_xtend_b200 import raw
    B, F, H0, W0, H, W = 2, 3, 150, 250, 64, 128
    src = _u8((B, F, H0, W0, 3), 3)
    x = _oracle_frames(src, H, W).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    eps = torch.randn(B, 3, H, W, device=DEV, generator=g)
    sig = torch.tensor([0.05, 0.3], device=DEV)
    ref = torch.empty(B * (F + 1) * H * W, 64, device=DEV, dtype=bf16)
    raw.vae_frames_in(x, eps, sig, ref)
    rows, x0 = _kernel(src, H, W, eps, sig)
    assert torch.equal(rows.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(x0.view(torch.int32), x[:, 0].contiguous().view(torch.int32))
    hw = H * W
    for first, count in ((0, 1), (4, 4), (5, 2), (7, 1)):
        part, x0p = _kernel(src, H, W, eps, sig, first, count)
        assert torch.equal(part.view(torch.int16), ref[first * hw:(first + count) * hw].view(torch.int16)), (first, count)
        fl = torch.empty(count * hw, 64, device=DEV, dtype=bf16)
        raw.vae_frames_in_range(x, eps, sig, fl, first, count)
        assert torch.equal(fl.view(torch.int16), ref[first * hw:(first + count) * hw].view(torch.int16)), (first, count)
        for b in range(B):                        # the clean first frame is written with the conditioning frame B*F + b
            if first <= B * F + b < first + count:
                assert torch.equal(x0p[b].view(torch.int32), x[b, 0].contiguous().view(torch.int32))


def _pairs(seed, vae_cfg, unet_cfg, clip_cfg):
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(seed)
    with torch.device(DEV):
        v = AutoencoderKLTemporalDecoder(**vae_cfg)
        c = CLIPVisionModelWithProjection(**clip_cfg)
        u = UNetSpatioTemporalConditionModel(**unet_cfg)
    for m in (v, c, u):
        m.eval().requires_grad_(False)
    for n, p in u.named_parameters():
        if "temporal_transformer_block" in n:           # train_svd.py:761-766
            p.requires_grad_(True)
    u.train()
    return v, c, u


def _tiny_cfgs():
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from oracle.svd_unet_oracle import TINY_CONFIG
    return TINY_VAE, TINY_CONFIG, dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"])


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["float", "u8"])
def test_chunked_encode_matches_one_encode(form):
    from svd_xtend_b200.video_train import assemble_train_batch, draw_train_noise
    v, c, u = _pairs(21, *_tiny_cfgs())
    B, F, H, W = 1, 4, 64, 128
    src = _u8((B, F, 96, 160, 3), 5)
    x = src.to(DEV) if form == "u8" else _oracle_frames(src, H, W).to(DEV)
    kw = dict(size=(H, W)) if form == "u8" else {}
    d = draw_train_noise(B, F, H, W, generator=torch.Generator().manual_seed(9), device=DEV)
    one = [assemble_train_batch(v, c, u, x, d, conditioning_dropout_prob=0.1, **kw) for _ in range(3)]
    spread = max(_rel(one[i]["sample"], one[0]["sample"]) for i in (1, 2))
    for chunk in (1, 3, B * (F + 1)):
        b = assemble_train_batch(v, c, u, x, d, conditioning_dropout_prob=0.1, encode_chunk_size=chunk, **kw)
        e = _rel(b["sample"], one[0]["sample"])
        print(f"{form} encode_chunk_size={chunk}: sample rel-l2 {e:.3e} (two encodes {spread:.3e})")
        assert e <= 4 * spread + 1e-6, chunk
        for k in ("encoder_hidden_states", "timestep", "added_time_ids", "sigmas"):
            assert torch.equal(b[k], one[0][k]), k


def _step(seed, source_size=None, cuda_graph=True, chunk=None, frames=(1, 4, 64, 128), cfgs=None, frozen_dtype=None, grad_ckpt=False,
          check_unchanged=True):
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    from svd_xtend_b200.video_train import VideoTrainStep
    v, c, u = _pairs(seed, *(cfgs or _tiny_cfgs()))
    if frozen_dtype is not None:
        v.to(frozen_dtype)
        c.to(frozen_dtype)
    if grad_ckpt:
        u.enable_gradient_checkpointing()
    arena = ParamArena(u)
    u.attach_arena(arena)
    opt = FusedAdamW(arena, lr=1e-4)
    opt.on_updated = lambda: u.refresh_trainable_operands(shadow_current=True)
    gen = torch.Generator(DEV).manual_seed(123)
    snap = [t.clone() for t in opt.snapshot_tensors()] if check_unchanged else []
    step = VideoTrainStep(u, v, c, opt, frames_shape=frames, conditioning_dropout_prob=0.1, generator=gen, cuda_graph=cuda_graph,
                          source_size=source_size, encode_chunk_size=chunk)
    torch.cuda.synchronize()
    unchanged = all(torch.equal(a, b) for a, b in zip(snap, opt.snapshot_tensors())) if check_unchanged else None
    return step, opt, arena, unchanged


@pytest.mark.gpu
def test_u8_graphed_step_matches_eager_and_float_step():
    torch.backends.cuda.matmul.allow_tf32 = False
    src = [_u8((1, 4, 90, 200, 3), 60 + i) for i in range(3)]
    pinned = [s.pin_memory() for s in src]
    flt = [_oracle_frames(s, 64, 128).to(DEV) for s in src]

    def run(graph, u8=True, chunk=2):
        step, opt, arena, unchanged = _step(7, source_size=(90, 200) if u8 else None, cuda_graph=graph, chunk=chunk)
        assert unchanged, "construction changed the weights or the optimizer state"
        losses = [step(pinned[i] if u8 else flt[i]).item() for i in range(3)]
        torch.cuda.synchronize()
        return losses, arena.grad.clone(), arena.data.clone()

    l1, g1, p1 = run(False)
    l2, g2, p2 = run(False)
    lg, gg, pg = run(True)
    lf, gf, pf = run(True, u8=False)
    spread_l = max(abs(a - b) for a, b in zip(l1, l2))
    spread_g, spread_p = _rel(g2, g1), _rel(p2, p1)
    for name, (l, g, p) in (("graphed u8", (lg, gg, pg)), ("graphed float", (lf, gf, pf))):
        dl = max(abs(a - b) for a, b in zip(l, l1))
        print(f"{name}: losses {l} eager u8 {l1}; loss spread {spread_l:.3e} diff {dl:.3e}; grad spread {spread_g:.3e} diff "
              f"{_rel(g, g1):.3e}; weights spread {spread_p:.3e} diff {_rel(p, p1):.3e}")
        assert all(t == t for t in l)
        assert dl <= 4 * spread_l + 1e-6 * max(map(abs, l1))
        assert _rel(g, g1) <= 4 * spread_g + 1e-6
        assert _rel(p, p1) <= 4 * spread_p + 1e-7


@pytest.mark.gpu
def test_u8_step_rejects_other_frames():
    step, _, _, _ = _step(3, source_size=(90, 200), cuda_graph=False)
    with pytest.raises(TypeError, match="uint8"):
        step(torch.zeros(1, 4, 90, 200, 3, device=DEV))
    with pytest.raises(ValueError, match="3 \\(RGB\\)"):
        step(torch.zeros(1, 4, 90, 200, 4, device=DEV, dtype=torch.uint8))
    with pytest.raises(ValueError, match="built for uint8 frames"):
        step(torch.zeros(1, 4, 90, 198, 3, device=DEV, dtype=torch.uint8))


@pytest.mark.gpu
def test_config4_graphed_step_fits_80gb():
    """train_svd.py's defaults, 25 x 576 x 1024 and B = 1, from decoded 1080 x 1920 uint8 frames: fp32 UNet with the as-scripted
    trainable set and gradient checkpointing, VAE and CLIP in bf16, FusedAdamW, conditioning dropout 0.1, the graphed step with
    the encode in chunks of 2 frames; it builds and replays two steps with a finite loss"""
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.workload import SVD_CONFIG
    if torch.cuda.get_device_properties(0).total_memory < 79 * 2 ** 30:
        pytest.skip("needs an 80 GB card")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    step, _, _, _ = _step(11, source_size=(1080, 1920), chunk=2, frames=(1, 25, 576, 1024), cfgs=(VAE_CONFIG, SVD_CONFIG, CLIP_CONFIG),
                          frozen_dtype=bf16, grad_ckpt=True, check_unchanged=False)      # no device copy of the optimizer state
    built = torch.cuda.max_memory_allocated()
    src = _u8((1, 25, 1080, 1920, 3), 90).pin_memory()
    losses = [step(src).item() for _ in range(2)]
    torch.cuda.synchronize()
    print(f"config 4 from uint8 1080x1920 frames: losses {losses}; peak allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB "
          f"(after construction {built / 2**30:.2f}), reserved {torch.cuda.memory_reserved() / 2**30:.2f} GiB of "
          f"{torch.cuda.get_device_properties(0).total_memory / 2**30:.1f}")
    assert all(l == l and abs(l) < float("inf") for l in losses)
