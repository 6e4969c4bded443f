"""Frame sizes whose widths the row-box conv tiles cannot cover (neither W | 128 nor 128 | W): svdx_tapgemm takes them through
TMA im2col loads. The im2col path must compute exactly what the box path computes: the same conv on the input zero-padded on
the right to a width the boxes tile, cropped back, is bitwise equal (same operand bytes, same k order, same epilogue). On top,
the kernels are checked against torch fp32 math and the whole UNet / sampler / VAE encoder against their fp32 oracles at
portrait and square sizes."""
import pytest
import torch
import torch.nn.functional as F

from test_unet_gpu import DEV, _build, _loss, _rel, _train_filter

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
WIDTHS = (5, 9, 10, 12, 18, 20, 24, 36, 40, 48, 72, 80, 96, 144, 160, 192, 288, 320, 576)


@pytest.fixture(scope="module")
def raw():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from svd_xtend_b200 import raw
    return raw


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _box_width(W):
    """the narrowest width >= W that the row boxes tile"""
    return 128 if W <= 128 else -(-W // 128) * 128


def _height(W, nimg, min_m=0):
    """a height whose tiles straddle image rows and images: H*W % 128 != 0 and M % 128 != 0 (and M >= min_m)"""
    for H in [7, 5, 3] + list(range(9, 64, 2)):
        if (H * W) % 128 and (nimg * H * W) % 128 and nimg * H * W >= min_m:
            return H
    raise AssertionError(W)


def _padw(t, Wp):
    """[n, H, W, C] -> [n, H, Wp, C], zeros on the right"""
    return F.pad(t, (0, 0, 0, Wp - t.shape[2]))


def _conv(raw, x, wk, Cout, taps, out_rows, W, H, nimg, auto=False, **kw):
    """x [nimg_tensor, H, W, C] channels-last; out [out_rows, Cout]"""
    out = torch.full((out_rows, Cout), float("nan"), device=DEV, dtype=bf16)
    fn = raw.tapgemm_auto if auto else raw.tapgemm
    fn(x.reshape(-1, x.shape[-1]), wk, out, M=out_rows, N=Cout, K=x.shape[-1], mode=raw.A_CONV2D, taps=taps, conv_whn=(W, H, nimg), **kw)
    return out


def _crop(out, n, H, Wp, W):
    return out.view(n, H, Wp, -1)[:, :, :W].reshape(n * H * W, -1)


def _weights(Cin, Cout, seed):
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=seed).to(bf16)
    return w, w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)


def _torch_conv(x, w, bias=None, **kw):
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, **kw)
    return y.permute(0, 2, 3, 1).reshape(-1, w.shape[0])


def _close(got, ref, what):
    err = (got.float() - ref).abs()
    tol = 1.5e-2 * ref.abs().max().item() + 1.5e-2 * ref.abs()
    rel = ((got.float() - ref).norm() / ref.norm()).item()
    assert not (err > tol).any() and rel < 1e-2, f"{what}: max err {err.max().item():.4g}, rel-l2 {rel:.4g}"


# ------------------------------------------------------------------------------------------------ bit identity, forward
@pytest.mark.parametrize("W", WIDTHS)
def test_forward_bitwise_equal_to_the_box_path(raw, W):
    """bias + per-image rowbias + residual with scales, against the same launch at the padded width; and against torch"""
    nimg = 3
    H = _height(W, nimg)
    Cin, Cout = (64, 64) if W >= 288 else (96, 160)
    Wp = _box_width(W)
    x = _rand(nimg, H, W, Cin, seed=1).to(bf16)
    w, wk = _weights(Cin, Cout, 2)
    bias = _rand(Cout, seed=3)
    rb = _rand(nimg, Cout, seed=4)
    res = _rand(nimg, H, W, Cout, seed=5).to(bf16)
    scales = torch.tensor([0.7, 1.0, 0.0], device=DEV)
    M, Mp = nimg * H * W, nimg * H * Wp
    kw = dict(bias=bias, rowbias=rb, scales=scales)
    got = _conv(raw, x, wk, Cout, raw.CONV3x3_TAPS, M, W, H, nimg, rowbias_div=H * W, res1=res.view(M, Cout), **kw)
    box = _conv(raw, _padw(x, Wp), wk, Cout, raw.CONV3x3_TAPS, Mp, Wp, H, nimg, rowbias_div=H * Wp,
                res1=_padw(res, Wp).view(Mp, Cout), **kw)
    torch.cuda.synchronize()
    assert torch.equal(got, _crop(box, nimg, H, Wp, W)), f"W={W}: im2col and box outputs differ"
    ref = 0.7 * (_torch_conv(x, w, bias, padding=1) + rb.repeat_interleave(H * W, 0)) + res.float().view(M, Cout)
    _close(got, ref, f"conv W={W}")


@pytest.mark.parametrize("H,W,nimg", [(8, 5, 14), (16, 9, 14)])
def test_portrait_bottom_level_bitwise_equal(raw, H, W, nimg):
    """the L3 images of the 512x320 and 1024x576 portrait latents, 14 frames"""
    Cin = Cout = 128
    Wp = _box_width(W)
    x = _rand(nimg, H, W, Cin, seed=6).to(bf16)
    w, wk = _weights(Cin, Cout, 7)
    bias = _rand(Cout, seed=8)
    got = _conv(raw, x, wk, Cout, raw.CONV3x3_TAPS, nimg * H * W, W, H, nimg, bias=bias)
    box = _conv(raw, _padw(x, Wp), wk, Cout, raw.CONV3x3_TAPS, nimg * H * Wp, Wp, H, nimg, bias=bias)
    torch.cuda.synchronize()
    assert torch.equal(got, _crop(box, nimg, H, Wp, W))
    _close(got, _torch_conv(x, w, bias, padding=1), f"conv {H}x{W}")


@pytest.mark.parametrize("W", [9, 36, 72, 320])
def test_block_n_320_bitwise_equal(raw, W):
    nimg = 3
    H = _height(W, nimg, min_m=512)
    Cin, Cout = 64, 640
    Wp = _box_width(W)
    x = _rand(nimg, H, W, Cin, seed=9).to(bf16)
    w, wk = _weights(Cin, Cout, 10)
    bias = _rand(Cout, seed=11)
    M = nimg * H * W
    assert M >= 512
    got = _conv(raw, x, wk, Cout, raw.CONV3x3_TAPS, M, W, H, nimg, bias=bias, block_n=320)
    box = _conv(raw, _padw(x, Wp), wk, Cout, raw.CONV3x3_TAPS, nimg * H * Wp, Wp, H, nimg, bias=bias, block_n=320)
    torch.cuda.synchronize()
    assert torch.equal(got, _crop(box, nimg, H, Wp, W))
    _close(got, _torch_conv(x, w, bias, padding=1), f"block_n 320 W={W}")


@pytest.mark.parametrize("H,W", [(8, 5), (16, 9), (10, 12)])
def test_split_k_matches_the_box_path_within_fp32_round_off(raw, H, W):
    """small-M convs take tapgemm_auto's split-K path (fp32 atomics: the sums are reordered, so equality holds to round-off)"""
    nimg, Cin, Cout = 14, 256, 512
    Wp = _box_width(W)
    M = nimg * H * W
    assert raw.split_plan(True, M, Cout, Cin, 9) is not None
    x = _rand(nimg, H, W, Cin, seed=12).to(bf16)
    w, wk = _weights(Cin, Cout, 13)
    bias = _rand(Cout, seed=14)
    res = _rand(nimg, H, W, Cout, seed=15).to(bf16)
    scales = torch.tensor([0.4, 1.0, 0.0], device=DEV)
    got = _conv(raw, x, wk, Cout, raw.CONV3x3_TAPS, M, W, H, nimg, auto=True, bias=bias, res1=res.view(M, Cout), scales=scales)
    box = _conv(raw, _padw(x, Wp), wk, Cout, raw.CONV3x3_TAPS, nimg * H * Wp, Wp, H, nimg, auto=True, bias=bias,
                res1=_padw(res, Wp).view(-1, Cout), scales=scales)
    torch.cuda.synchronize()
    b = _crop(box, nimg, H, Wp, W).float()
    assert ((got.float() - b).abs() <= 2 ** -7 * b.abs() + 1e-5).all()
    _close(got, 0.4 * _torch_conv(x, w, bias, padding=1) + res.float().view(M, Cout), f"split-K {H}x{W}")


@pytest.mark.parametrize("W", [5, 9, 36, 72, 288])
def test_dgrad_negated_taps_bitwise_equal(raw, W):
    """the input gradient of a 3x3 conv: the taps negated, K = the padded output channels (8: the UNet's conv_out)"""
    from svd_xtend_b200.engine import _neg_taps
    nimg = 3
    H = _height(W, nimg)
    Wp = _box_width(W)
    for Cin, Cout in ((8, 320), (128, 64)):
        dy = _rand(nimg, H, W, Cin, seed=16).to(bf16)
        wt = _rand(Cout, 9 * Cin, scale=(9 * Cin) ** -0.5, seed=17).to(bf16)
        taps = _neg_taps(raw.CONV3x3_TAPS)
        got = _conv(raw, dy, wt, Cout, taps, nimg * H * W, W, H, nimg)
        box = _conv(raw, _padw(dy, Wp), wt, Cout, taps, nimg * H * Wp, Wp, H, nimg)
        torch.cuda.synchronize()
        assert torch.equal(got, _crop(box, nimg, H, Wp, W)), (W, Cin)


def _planes(x):
    N = x.shape[0]
    p = torch.empty(4 * N, x.shape[1] // 2, x.shape[2] // 2, x.shape[3], device=DEV, dtype=x.dtype)
    for a in range(2):
        for b in range(2):
            p[(a * 2 + b) * N:(a * 2 + b + 1) * N] = x[:, a::2, b::2]
    return p


@pytest.mark.parametrize("Wi", [72, 18, 576])
@pytest.mark.parametrize("pad0", [False, True])
def test_stride2_plane_tables_bitwise_equal(raw, Wi, pad0):
    """both parity-plane tables: the UNet's Downsample2D (padding 1) and the VAE encoder's F.pad(0,1,0,1) + padding 0"""
    N, C, Cout = 3, 64, 128
    Hi = 10 if Wi < 576 else 6
    Ho, Wo = Hi // 2, Wi // 2
    Wp = _box_width(Wo)
    x = _rand(N, Hi, Wi, C, seed=18).to(bf16)
    w, wk = _weights(C, Cout, 19)
    table = ((0, 0), (1, 0), (0, 1)) if pad0 else ((1, -1), (0, 0), (1, 0))
    taps = []
    for kh in range(3):
        for kw in range(3):
            ph, dh = table[kh]
            pw, dw = table[kw]
            taps.append((dw, dh, (ph * 2 + pw) * N))
    planes = _planes(x)
    got = _conv(raw, planes, wk, Cout, taps, N * Ho * Wo, Wo, Ho, 4 * N)
    box = _conv(raw, _padw(planes, Wp), wk, Cout, taps, N * Ho * Wp, Wp, Ho, 4 * N)
    torch.cuda.synchronize()
    assert torch.equal(got, _crop(box, N, Ho, Wp, Wo))
    ref = _torch_conv(F.pad(x, (0, 0, 0, 1, 0, 1)), w, stride=2) if pad0 else _torch_conv(x, w, stride=2, padding=1)
    _close(got, ref, f"stride-2 planes {Wi}->{Wo} pad0={pad0}")


# ------------------------------------------------------------------------------------------------ fused GroupNorm sums
@pytest.mark.parametrize("H,W,nimg", [(8, 5, 14), (16, 9, 14), (7, 36, 3), (5, 144, 2)])
def test_gn_sum_equals_groupnorm_sums(raw, H, W, nimg):
    Cin, Cout = 64, 320
    x = _rand(nimg, H, W, Cin, seed=20).to(bf16)
    w, wk = _weights(Cin, Cout, 21)
    bias = _rand(Cout, seed=22)
    rows = H * W
    sums = torch.zeros(nimg, 2, Cout, device=DEV)
    out = _conv(raw, x, wk, Cout, raw.CONV3x3_TAPS, nimg * rows, W, H, nimg, bias=bias, gn_sum=sums, gn_rows=rows)
    alone = raw.groupnorm_sums(out, None, nimg, rows)
    torch.cuda.synchronize()
    _close(out, _torch_conv(x, w, bias, padding=1), f"conv + gn_sum {H}x{W}")
    err = ((alone - sums).abs().amax((0, 2)) / (sums.abs().amax((0, 2)) + 1e-9)).max().item()
    assert err < 4e-5, f"groupnorm_sums vs the epilogue's gn_sum: {err:.3g}"


@pytest.mark.parametrize("H,W,nimg", [(16, 9, 14), (7, 36, 3)])
def test_gnb_sums_equal_groupnorm_bwd_sums(raw, H, W, nimg):
    Cin, Cout = 128, 320
    M, rows = nimg * H * W, H * W
    g = _rand(nimg, H, W, Cin, seed=23).to(bf16)
    w, wk = _weights(Cin, Cout, 24)
    x = (_rand(M, Cout, seed=25) + 0.3).to(bf16)
    gamma = _rand(Cout, seed=26) * 0.2 + 1.0
    beta = _rand(Cout, seed=27) * 0.1
    y = torch.empty(M, Cout, device=DEV, dtype=bf16)
    ab = torch.empty(nimg, 2, Cout, device=DEV)
    raw.groupnorm_apply_fused(x, None, nimg, rows, 1e-5, raw.groupnorm_sums(x, None, nimg, rows), None, gamma, beta, True, y, ab=ab)
    sums = torch.zeros(nimg, 2, Cout, device=DEV)
    dy = _conv(raw, g, wk, Cout, raw.CONV3x3_TAPS, M, W, H, nimg, gnb=dict(x=x, x2=None, ab=ab, rows=rows, silu=True, sum=sums))
    alone = raw.groupnorm_bwd_sums(x, None, dy, nimg, rows, ab, True)
    torch.cuda.synchronize()
    _close(dy, _torch_conv(g, w, padding=1), f"dgrad + gnb {H}x{W}")
    tol = 2e-3 * sums[:, 0].abs().max().item() + 1e-4
    assert (alone[:, 0] - sums[:, 0]).abs().max().item() < tol
    assert (alone[:, 1] - sums[:, 1]).abs().max().item() < 2e-3 * sums[:, 1].abs().max().item() + 1e-4


# ------------------------------------------------------------------------------------------------ conv weight gradient
@pytest.mark.parametrize("W", [9, 36, 72, 96, 144])
def test_weight_gradient_im2col_b(raw, W):
    """b_mode 1 at widths with neither W | 64 nor 64 | W: 64-pixel im2col loads of the shifted input, against fp64"""
    nimg = 3
    H = _height(W, nimg)
    Cin, Cout = 128, 64
    x = _rand(nimg, H, W, Cin, seed=28).to(bf16)
    dy = _rand(nimg, H, W, Cout, scale=0.1, seed=29).to(bf16)
    M = nimg * H * W
    ws = torch.zeros(Cout, 9 * Cin, device=DEV)
    for t, tap in enumerate(raw.CONV3x3_TAPS):
        raw.tapgemm(dy.view(M, Cout), x.view(M, Cin), ws[:, t * Cin:(t + 1) * Cin], M=Cout, N=Cin, K=M, a_mn=True, b_mn=True, b_mode=1,
                    taps=(tap,), conv_whn=(W, H, nimg), split_k=2, out_dtype=raw.OUT_F32_ATOMIC, ldo=9 * Cin)
    gw = torch.zeros(Cout, Cin, 3, 3, device=DEV)
    raw.unprep_conv_grad(ws, gw, Cout, Cin, 9, Cin)
    torch.cuda.synchronize()
    wr = torch.zeros(Cout, Cin, 3, 3, device=DEV, dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double().permute(0, 3, 1, 2), wr, padding=1).backward(dy.double().permute(0, 3, 1, 2))
    ref = wr.grad.float()
    err = (gw - ref).abs()
    assert (err <= 3e-3 * ref.abs().max().item() + 3e-3 * ref.abs()).all(), f"W={W}: max err {err.max().item():.4g}"


def test_weight_gradient_stride2_planes_im2col_b(raw):
    """the UNet Downsample2D weight gradient at 72 -> 36 (plane width 36: im2col B with a plane offset)"""
    N, Hi, Wi, C, Cout = 2, 10, 72, 64, 64
    Ho, Wo = Hi // 2, Wi // 2
    x = _rand(N, Hi, Wi, C, seed=30).to(bf16)
    dy = _rand(N, Ho, Wo, Cout, scale=0.1, seed=31).to(bf16)
    planes = _planes(x)
    M = N * Ho * Wo
    ws = torch.zeros(Cout, 9 * C, device=DEV)
    t = 0
    for kh in range(3):
        for kw in range(3):
            ph, dh = ((1, -1), (0, 0), (1, 0))[kh]
            pw, dw = ((1, -1), (0, 0), (1, 0))[kw]
            raw.tapgemm(dy.view(M, Cout), planes.view(-1, C), ws[:, t * C:(t + 1) * C], M=Cout, N=C, K=M, a_mn=True, b_mn=True, b_mode=1,
                        taps=((dw, dh, (ph * 2 + pw) * N),), conv_whn=(Wo, Ho, 4 * N), split_k=2, out_dtype=raw.OUT_F32_ATOMIC, ldo=9 * C)
            t += 1
    gw = torch.zeros(Cout, C, 3, 3, device=DEV)
    raw.unprep_conv_grad(ws, gw, Cout, C, 9, C)
    torch.cuda.synchronize()
    wr = torch.zeros(Cout, C, 3, 3, device=DEV, dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double().permute(0, 3, 1, 2), wr, stride=2, padding=1).backward(dy.double().permute(0, 3, 1, 2))
    ref = wr.grad.float()
    assert ((gw - ref).abs() <= 3e-3 * ref.abs().max().item() + 3e-3 * ref.abs()).all()


# ------------------------------------------------------------------------------------------------ the whole model
def _grads_vs_oracle(oracle, ours, batch, all_params=False):
    pred_ref, loss_ref = _loss(oracle, batch)
    loss_ref.backward()
    g_ref = {n: p.grad.clone() for n, p in oracle.named_parameters() if p.requires_grad}
    oracle.zero_grad(set_to_none=True)
    pred_ac, loss_ac = _loss(oracle, batch, autocast=True)
    loss_ac.backward()
    g_ac = {n: p.grad.clone() for n, p in oracle.named_parameters() if p.requires_grad}
    oracle.zero_grad(set_to_none=True)
    e_ac = _rel(pred_ac, pred_ref)
    del pred_ac, loss_ac
    torch.cuda.empty_cache()
    pred, loss = _loss(ours, batch)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(pred).all()
    e_out = _rel(pred, pred_ref)
    assert e_out <= max(2 * e_ac, 2e-2), f"output rel-l2 {e_out:.4g} vs autocast {e_ac:.4g}"
    bad, n_cmp = [], 0
    for n, p in ours.named_parameters():
        if not p.requires_grad:
            continue
        assert p.grad is not None, n
        ref = g_ref[n]
        if ref.abs().max() == 0:
            assert p.grad.abs().max() == 0, n
            continue
        e, ea = _rel(p.grad, ref), _rel(g_ac[n], ref)
        # mix_factor gradients are scalars made of differences of nearly equal bf16 tensors (see test_unet_gpu)
        tol = max(0.2, 2 * ea) if (all_params and n.endswith("mix_factor")) else max(3 * ea, 5e-2)
        n_cmp += 1
        if e > tol:
            bad.append((n, round(e, 4), round(ea, 4)))
    assert not bad, bad[:10]
    return n_cmp


def test_tiny_train_step_at_16x24():
    from oracle.svd_unet_oracle import TINY_CONFIG, synthetic_batch
    oracle, ours = _build(TINY_CONFIG, seed=2)
    for m in (oracle, ours):
        _train_filter(m)
        m.train()
    batch = synthetic_batch(2, 4, 16, 24, seed=99, device=DEV, cross_dim=TINY_CONFIG["cross_attention_dim"])
    assert _grads_vs_oracle(oracle, ours, batch) > 10


def test_tiny_full_finetune_at_16x24():
    """every parameter trainable: conv weight gradients at widths 24 and 12 (im2col B) included"""
    from oracle.svd_unet_oracle import TINY_CONFIG, synthetic_batch
    oracle, ours = _build(TINY_CONFIG, seed=6)
    for m in (oracle, ours):
        m.requires_grad_(True)
        m.train()
    batch = synthetic_batch(2, 4, 16, 24, seed=98, device=DEV, cross_dim=TINY_CONFIG["cross_attention_dim"])
    assert _grads_vs_oracle(oracle, ours, batch, all_params=True) > 100


def test_svd_config_train_step_portrait_64x40():
    """config 2 of BASELINE.json in portrait: 14 frames of 512x320 (latent 64x40: every level on the im2col path)"""
    from oracle.svd_unet_oracle import SVD_CONFIG, synthetic_batch
    oracle, ours = _build(SVD_CONFIG, seed=11)
    for m in (oracle, ours):
        _train_filter(m)
        m.train()
    batch = synthetic_batch(1, 14, 64, 40, seed=1234, device=DEV)
    assert _grads_vs_oracle(oracle, ours, batch) > 300


@pytest.mark.parametrize("h,w,T", [(128, 72, 4), (96, 96, 4)])
def test_svd_config_forward_large_portrait_and_square(h, w, T):
    """1024x576 portrait and 768x768 square latents; 4 frames keep the fp32 oracle's materialised attention in memory"""
    from oracle.svd_unet_oracle import SVD_CONFIG, synthetic_batch
    oracle, ours = _build(SVD_CONFIG, seed=12)
    oracle.eval()
    ours.eval()
    batch = synthetic_batch(1, T, h, w, seed=4321, device=DEV)
    args = (batch["sample"], batch["timestep"], batch["encoder_hidden_states"], batch["added_time_ids"])
    with torch.no_grad():
        ref = oracle(*args).sample
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = oracle(*args).sample
        out = ours(*args).sample
    torch.cuda.synchronize()
    e, ea = _rel(out, ref), _rel(ac, ref)
    print(f"svd forward {h}x{w}: rel-l2 {e:.4g} (autocast {ea:.4g})")
    assert torch.isfinite(out).all() and e <= max(2 * ea, 2e-2), (e, ea)


def test_cuda_graph_replay_at_64x40_equals_eager():
    from oracle.svd_unet_oracle import SVD_CONFIG, synthetic_batch
    _, ours = _build(SVD_CONFIG, seed=13)
    _train_filter(ours)
    ours.train()
    batch = synthetic_batch(1, 14, 64, 40, seed=77, device=DEV)
    args = (batch["sample"], batch["timestep"], batch["encoder_hidden_states"], batch["added_time_ids"])

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            pred = ours(*args).sample
        (pred.float() ** 2).mean().backward()
        return pred.detach().clone(), {n: p.grad.clone() for n, p in ours.named_parameters() if p.requires_grad}

    # the script's loop: forward, backward, optimizer step, zero_grad; captured after the warm-up calls
    runner = ours.enable_cuda_graphs(warmup=2)
    opt = torch.optim.AdamW([p for p in ours.parameters() if p.requires_grad], lr=1e-6)
    for _ in range(4):
        step()
        opt.step()
        opt.zero_grad(set_to_none=True)
    p_graph, g_graph = step()
    torch.cuda.synchronize()
    ent = [e for e in runner.entries.values() if e.g_bwd is not None]
    assert len(ent) == 1 and ent[0].calls == 5, "the training step must have been captured and replayed"
    ours.zero_grad(set_to_none=True)
    ours.disable_cuda_graphs()
    p_eager, g_eager = step()
    torch.cuda.synchronize()
    # fp32 atomics (GroupNorm statistics, split-K) make two runs differ at bf16-rounding level: the bounds of
    # test_boundary_gpu's replay-versus-eager check
    assert _rel(p_graph, p_eager) < 3e-2
    for n in g_eager:
        if g_eager[n].abs().max() > 0:
            assert _rel(g_graph[n], g_eager[n]) < 5e-2, n


def test_sampler_two_steps_at_64x40():
    from oracle.svd_sampling_oracle import sample_latents
    from oracle.svd_unet_oracle import SVD_CONFIG
    from svd_xtend_b200.sampling import VideoLatentSampler
    oracle, ours = _build(SVD_CONFIG, seed=14)
    oracle.eval()
    g = torch.Generator(device="cpu").manual_seed(8)
    B, T, h, w = 1, 14, 64, 40
    image_latents = torch.randn(B, 4, h, w, generator=g).to(DEV)
    emb = torch.randn(B, 1, SVD_CONFIG["cross_attention_dim"], generator=g).to(DEV)
    noise = torch.randn(B, T, 4, h, w, generator=g).to(DEV)
    kw = dict(num_frames=T, fps=7, motion_bucket_id=127, noise_aug_strength=0.02, num_inference_steps=2, min_guidance_scale=1.0,
              max_guidance_scale=3.0, noise=noise)
    with torch.no_grad():
        ref = sample_latents(oracle, image_latents, emb, **kw)
    out = VideoLatentSampler(ours)(image_latents, emb, **kw)
    torch.cuda.synchronize()
    assert out.shape == ref.shape == (B, T, 4, h, w) and torch.isfinite(out).all()
    e = _rel(out, ref)
    print("portrait sampling rel-l2 after 2 steps", e)
    assert e < 4e-2, e


@pytest.mark.parametrize("H,W", [(512, 320), (1024, 576)])
def test_vae_encode_portrait(H, W):
    from oracle.svd_vae_oracle import VAE_CONFIG
    from test_vae import _build as _build_vae
    oracle, ours = _build_vae(VAE_CONFIG, seed=5, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(12)
    N = 2
    x = (torch.randn(N, 3, H, W, generator=g) * 0.5).clamp(-1, 1).to(DEV)
    with torch.no_grad():
        ref = oracle.encode(x).latent_dist
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = oracle.encode(x).latent_dist
        got = ours.encode(x).latent_dist
    torch.cuda.synchronize()
    assert got.mean.shape == ref.mean.shape == (N, 4, H // 8, W // 8)
    ref_m, ac_m, got_m = (torch.cat([d.mean, d.logvar], 1) for d in (ref, ac, got))
    e, ea = _rel(got_m, ref_m), _rel(ac_m.float(), ref_m)
    print(f"vae encode {H}x{W}: moments rel-l2 {e:.4g} (autocast {ea:.4g})")
    assert torch.isfinite(got_m).all() and e <= max(2 * ea, 2e-2), (e, ea)
