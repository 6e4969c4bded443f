"""GPU parity of svdx_tapgemm (wgmma contraction) against fp32 torch math on the same bf16 inputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16


def _dev():
    return torch.device("cuda:0")


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(_dev())


def _close(got, ref, rtol=1.5e-2, atol=None, what=""):
    got = got.float()
    ref = ref.float()
    if atol is None:
        atol = 1.5e-2 * ref.abs().max().item()
    err = (got - ref).abs()
    bad = err > (atol + rtol * ref.abs())
    rel = (got - ref).norm() / (ref.norm() + 1e-12)
    assert not bad.any() and rel < 1e-2, (
        f"{what}: {bad.sum().item()} / {bad.numel()} mismatches, max err {err.max().item():.4g}, rel-l2 {rel.item():.4g}, "
        f"first bad idx {bad.nonzero()[:4].tolist()}")


@pytest.fixture(scope="module")
def raw():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from svd_xtend_b200 import raw
    return raw


@pytest.mark.parametrize("M,N,K", [(128, 32, 64), (256, 320, 320), (1000, 640, 1024), (35840, 320, 320), (560, 1280, 2560), (14, 1280, 320)])
def test_linear_bias(raw, M, N, K):
    a = _rand(M, K, seed=1).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=2).to(bf16)
    bias = _rand(N, seed=3)
    out = torch.full((M, N), float("nan"), device=_dev(), dtype=bf16)
    raw.tapgemm(a, w, out, M=M, N=N, K=K, bias=bias)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias
    _close(out, ref, what=f"linear {M}x{N}x{K}")


def test_linear_f32_out_and_strided(raw):
    M, N, K = 300, 96, 192
    abig = _rand(M, K + 64, seed=4).to(bf16)
    a = abig[:, 64:]            # column-sliced view, lda = K + 64
    w = _rand(N, K, scale=K ** -0.5, seed=5).to(bf16)
    out = torch.zeros(M, N, device=_dev(), dtype=torch.float32)
    raw.tapgemm(a, w, out, M=M, N=N, K=K)
    torch.cuda.synchronize()
    _close(out, a.float() @ w.float().t(), rtol=1e-3, atol=1e-3, what="f32 out")


def test_geglu(raw):
    M, C = 512, 320
    a = _rand(M, C, seed=6).to(bf16)
    w = _rand(8 * C, C, scale=C ** -0.5, seed=7).to(bf16)
    bias = _rand(8 * C, scale=0.1, seed=8)
    out = torch.empty(M, 4 * C, device=_dev(), dtype=bf16)
    pre = torch.empty(M, 8 * C, device=_dev(), dtype=bf16)
    raw.tapgemm(a, w, out, M=M, N=8 * C, K=C, bias=bias, geglu=True, pre=pre)
    torch.cuda.synchronize()
    proj = a.float() @ w.float().t() + bias
    _close(pre, proj, what="geglu pre")
    pr = proj.to(bf16).float()
    ref = pr[:, : 4 * C] * F.gelu(pr[:, 4 * C:])
    _close(out, ref, what="geglu out")


def test_residual_blend(raw):
    M, N, K = 640, 320, 1280
    a = _rand(M, K, seed=9).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=10).to(bf16)
    bias = _rand(N, seed=11)
    r1 = _rand(M, N, seed=12).to(bf16)
    r2 = _rand(M, N, seed=13).to(bf16)
    scales = torch.tensor([0.378, 0.622, 0.378], device=_dev())
    out = torch.empty(M, N, device=_dev(), dtype=bf16)
    raw.tapgemm(a, w, out, M=M, N=N, K=K, bias=bias, res1=r1, res2=r2, scales=scales)
    torch.cuda.synchronize()
    ref = scales[0] * (a.float() @ w.float().t() + bias) + scales[1] * r1.float() + scales[2] * r2.float()
    _close(out, ref, what="residual blend")


def test_rowbias(raw):
    M, N, K, div = 14 * 40, 320, 320, 40
    a = _rand(M, K, seed=14).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=15).to(bf16)
    rb = _rand(M // div, N, seed=16)
    out = torch.empty(M, N, device=_dev(), dtype=bf16)
    raw.tapgemm(a, w, out, M=M, N=N, K=K, rowbias=rb, rowbias_div=div)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + rb.repeat_interleave(div, 0)
    _close(out, ref, what="rowbias")


@pytest.mark.parametrize("B,T,HW,C", [(1, 14, 160, 320), (2, 5, 40, 640), (1, 14, 2560, 320)])
def test_temporal_conv(raw, B, T, HW, C):
    # TemporalResnetBlock conv (3,1,1): x [B,T,HW,C] channels-last, w [Cout, Cin, 3]
    Cout = C
    x = _rand(B, T, HW, C, seed=17).to(bf16)
    w = _rand(Cout, C, 3, scale=(3 * C) ** -0.5, seed=18).to(bf16)
    bias = _rand(Cout, seed=19)
    wk = w.permute(0, 2, 1).contiguous().view(Cout, 3 * C)  # [Cout][tap][Cin]
    out = torch.empty(B * T * HW, Cout, device=_dev(), dtype=bf16)
    taps = [(-HW, 0, 0), (0, 0, 0), (HW, 0, 0)]
    raw.tapgemm(x.view(-1, C), wk, out, M=B * T * HW, N=Cout, K=C, taps=taps, rows_per_group=T * HW, groups=B, bias=bias)
    torch.cuda.synchronize()
    x5 = x.float().permute(0, 3, 1, 2).reshape(B, C, T, HW, 1)
    ref = F.conv3d(x5, w.float().view(Cout, C, 3, 1, 1), bias, padding=(1, 0, 0))
    ref = ref.reshape(B, Cout, T, HW).permute(0, 2, 3, 1).reshape(-1, Cout)
    _close(out, ref, what="temporal conv")


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(3, 40, 64, 64, 320), (14, 5, 8, 128, 160), (5, 10, 16, 320, 64), (2, 20, 32, 192, 320)])
def test_conv3x3(raw, N, H, W, Cin, Cout):
    x = _rand(N, H, W, Cin, seed=20).to(bf16)   # channels-last
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=21).to(bf16)
    bias = _rand(Cout, seed=22)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)  # [Cout][kh][kw][Cin]
    out = torch.empty(N * H * W, Cout, device=_dev(), dtype=bf16)
    raw.tapgemm(x.view(-1, Cin), wk, out, M=N * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS,
                conv_whn=(W, H, N), bias=bias)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    _close(out, ref, what="conv3x3")


def test_conv3x3_stride2_planes(raw):
    # Downsample2D: stride-2 conv as 9 taps over 4 parity planes
    N, H, W, C, Cout = 3, 20, 32, 128, 128
    x = _rand(N, H, W, C, seed=23).to(bf16)
    w = _rand(Cout, C, 3, 3, scale=(9 * C) ** -0.5, seed=24).to(bf16)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * C)
    Ho, Wo = H // 2, W // 2
    planes = torch.empty(4 * N, Ho, Wo, C, device=_dev(), dtype=bf16)
    for p in range(2):
        for q in range(2):
            planes[(p * 2 + q) * N:(p * 2 + q + 1) * N] = x[:, p::2, q::2]
    taps = []
    for kh in range(3):
        for kw in range(3):
            ph, dh = ((1, -1), (0, 0), (1, 0))[kh]
            pw, dw = ((1, -1), (0, 0), (1, 0))[kw]
            taps.append((dw, dh, (ph * 2 + pw) * N))
    out = torch.empty(N * Ho * Wo, Cout, device=_dev(), dtype=bf16)
    raw.tapgemm(planes.view(-1, C), wk, out, M=N * Ho * Wo, N=Cout, K=C, mode=raw.A_CONV2D, taps=taps, conv_whn=(Wo, Ho, 4 * N))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), None, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    _close(out, ref, what="conv stride 2")


@pytest.mark.parametrize("Mtok,Nout,Kin,split", [(512, 128, 64, 1), (2240, 320, 1280, 4), (35840, 2560, 320, 8)])
def test_wgrad_mn_major(raw, Mtok, Nout, Kin, split):
    # dW[Nout, Kin] = dY[Mtok, Nout]^T @ X[Mtok, Kin]: both operands MN-major
    dy = _rand(Mtok, Nout, scale=0.1, seed=25).to(bf16)
    x = _rand(Mtok, Kin, seed=26).to(bf16)
    dw = torch.zeros(Nout, Kin, device=_dev(), dtype=torch.float32)
    raw.tapgemm(dy, x, dw, M=Nout, N=Kin, K=Mtok, a_mn=True, b_mn=True, split_k=split, out_dtype=raw.OUT_F32_ATOMIC)
    torch.cuda.synchronize()
    ref = dy.float().t() @ x.float()
    _close(dw, ref, rtol=2e-3, atol=2e-3 * ref.abs().max().item(), what="wgrad")


@pytest.mark.parametrize("N,H,W,Cin,Cout,split", [(3, 40, 64, 64, 128, 4), (14, 5, 8, 128, 192, 2), (2, 10, 16, 320, 64, 1), (1, 4, 128, 64, 64, 1)])
def test_conv3x3_weight_gradient(raw, N, H, W, Cin, Cout, split):
    x = _rand(N, H, W, Cin, seed=30).to(bf16)
    dy = _rand(N, H, W, Cout, scale=0.1, seed=31).to(bf16)
    M = N * H * W
    ws = torch.zeros(Cout, 9 * Cin, device=_dev(), dtype=torch.float32)
    for t, tap in enumerate(raw.CONV3x3_TAPS):
        raw.tapgemm(dy.view(M, Cout), x.view(M, Cin), ws[:, t * Cin:(t + 1) * Cin], M=Cout, N=Cin, K=M, a_mn=True, b_mn=True, b_mode=1,
                    taps=(tap,), conv_whn=(W, H, N), split_k=split, out_dtype=raw.OUT_F32_ATOMIC, ldo=9 * Cin)
    gw = torch.zeros(Cout, Cin, 3, 3, device=_dev())
    raw.unprep_conv_grad(ws, gw, Cout, Cin, 9, Cin)
    torch.cuda.synchronize()
    w = torch.zeros(Cout, Cin, 3, 3, device=_dev(), requires_grad=True)
    F.conv2d(x.float().permute(0, 3, 1, 2), w, padding=1).backward(dy.float().permute(0, 3, 1, 2))
    _close(gw, w.grad, rtol=3e-3, atol=3e-3 * w.grad.abs().max().item(), what="conv wgrad")


def test_conv_stride2_planes_weight_gradient(raw):
    N, H, W, C, Cout = 3, 20, 32, 128, 64
    x = _rand(N, H, W, C, seed=32).to(bf16)
    Ho, Wo = H // 2, W // 2
    dy = _rand(N, Ho, Wo, Cout, scale=0.1, seed=33).to(bf16)
    planes = torch.empty(4 * N, Ho, Wo, C, device=_dev(), dtype=bf16)
    for p in range(2):
        for q in range(2):
            planes[(p * 2 + q) * N:(p * 2 + q + 1) * N] = x[:, p::2, q::2]
    M = N * Ho * Wo
    ws = torch.zeros(Cout, 9 * C, device=_dev(), dtype=torch.float32)
    t = 0
    for kh in range(3):
        for kw in range(3):
            ph, dh = ((1, -1), (0, 0), (1, 0))[kh]
            pw, dw = ((1, -1), (0, 0), (1, 0))[kw]
            raw.tapgemm(dy.view(M, Cout), planes.view(-1, C), ws[:, t * C:(t + 1) * C], M=Cout, N=C, K=M, a_mn=True, b_mn=True, b_mode=1,
                        taps=((dw, dh, (ph * 2 + pw) * N),), conv_whn=(Wo, Ho, 4 * N), split_k=2, out_dtype=raw.OUT_F32_ATOMIC, ldo=9 * C)
            t += 1
    gw = torch.zeros(Cout, C, 3, 3, device=_dev())
    raw.unprep_conv_grad(ws, gw, Cout, C, 9, C)
    torch.cuda.synchronize()
    w = torch.zeros(Cout, C, 3, 3, device=_dev(), requires_grad=True)
    F.conv2d(x.float().permute(0, 3, 1, 2), w, stride=2, padding=1).backward(dy.float().permute(0, 3, 1, 2))
    _close(gw, w.grad, rtol=3e-3, atol=3e-3 * w.grad.abs().max().item(), what="stride-2 conv wgrad")


@pytest.mark.parametrize("B,T,HW,C,split", [(1, 14, 160, 128, 4), (2, 5, 40, 64, 1), (2, 14, 40, 192, 2)])
def test_temporal_conv_weight_gradient(raw, B, T, HW, C, split):
    Cout = C
    x = _rand(B, T, HW, C, seed=34).to(bf16)
    dy = _rand(B, T, HW, Cout, scale=0.1, seed=35).to(bf16)
    M = B * T * HW
    ws = torch.zeros(Cout, 3 * C, device=_dev(), dtype=torch.float32)
    for t, sh in enumerate((-HW, 0, HW)):
        raw.tapgemm(dy.view(M, Cout), x.view(M, C), ws[:, t * C:(t + 1) * C], M=Cout, N=C, K=M, a_mn=True, b_mn=True, b_mode=2,
                    taps=((sh, 0, 0),), rows_per_group=T * HW, groups=B, split_k=split, out_dtype=raw.OUT_F32_ATOMIC, ldo=3 * C)
    gw = torch.zeros(Cout, C, 3, device=_dev())
    raw.unprep_conv_grad(ws, gw, Cout, C, 3, C)
    torch.cuda.synchronize()
    w = torch.zeros(Cout, C, 3, 1, 1, device=_dev(), requires_grad=True)
    x5 = x.float().permute(0, 3, 1, 2).reshape(B, C, T, HW, 1)
    d5 = dy.float().permute(0, 3, 1, 2).reshape(B, Cout, T, HW, 1)
    F.conv3d(x5, w, padding=(1, 0, 0)).backward(d5)
    _close(gw, w.grad.view(Cout, C, 3), rtol=3e-3, atol=3e-3 * w.grad.abs().max().item(), what="temporal conv wgrad")


def test_dot_diff_and_silu_bwd(raw):
    n = 8 * 12345
    dy, a, b = (_rand(n, seed=s).to(bf16) for s in (36, 37, 38))
    out = torch.zeros(1, device=_dev())
    raw.dot_diff(dy, a, b, out)
    x = _rand(1000, seed=39)
    g = _rand(1000, seed=40)
    dx = torch.empty_like(x)
    raw.silu_bwd_f32(x, g, dx)
    torch.cuda.synchronize()
    ref = (dy.float() * (a.float() - b.float())).sum()
    assert abs(out.item() - ref.item()) < 2e-3 * dy.float().abs().sum().item() ** 0.5 + 1e-2 * abs(ref.item())
    xr = x.clone().requires_grad_(True)
    F.silu(xr).backward(g)
    assert torch.allclose(dx, xr.grad, atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(14, 5, 8, 256, 512), (14, 10, 16, 128, 320)])
def test_conv3x3_auto_split_k(raw, N, H, W, Cin, Cout):
    """small-M convs (5x8 / 10x16 latents) take the split-K + svdx_splitk_epilogue path with the full epilogue"""
    x = _rand(N, H, W, Cin, seed=41).to(bf16)
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=42).to(bf16)
    bias = _rand(Cout, seed=43)
    M = N * H * W
    rb = _rand(2, Cout, seed=44)
    res = _rand(M, Cout, seed=45).to(bf16)
    scales = torch.tensor([0.4, 1.0, 0.0], device=_dev())
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)
    out = torch.empty(M, Cout, device=_dev(), dtype=bf16)
    raw.tapgemm_auto(x.view(-1, Cin), wk, out, M=M, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS, conv_whn=(W, H, N),
                     bias=bias, rowbias=rb, rowbias_div=M // 2, res1=res, scales=scales)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    ref = 0.4 * (ref + rb.repeat_interleave(M // 2, 0)) + res.float()
    _close(out, ref, what="conv split-k")
    # the fp32 workspace is cached per shape and re-zeroed by the epilogue: a second launch must give the same result
    out2 = torch.empty_like(out)
    raw.tapgemm_auto(x.view(-1, Cin), wk, out2, M=M, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS, conv_whn=(W, H, N),
                     bias=bias, rowbias=rb, rowbias_div=M // 2, res1=res, scales=scales)
    torch.cuda.synchronize()
    _close(out2, ref, what="conv split-k (workspace reuse)")


def _check_gn_sums(sums, out, rows_per_slab, what):
    """sums [slabs, 2, C] against fp64 column sums of the STORED bf16 output"""
    slabs, _, C = sums.shape
    o = out.double().view(slabs, rows_per_slab, C)
    ref1, ref2 = o.sum(1), (o * o).sum(1)
    e1 = (sums[:, 0].double() - ref1).abs().max().item() / (ref1.abs().max().item() + 1e-9)
    e2 = (sums[:, 1].double() - ref2).abs().max().item() / (ref2.abs().max().item() + 1e-9)
    assert e1 < 2e-5 and e2 < 2e-5, f"{what}: channel-sum error {e1:.3g} / {e2:.3g}"


@pytest.mark.parametrize("M,N,K,rows", [(35840, 320, 320, 2560), (2240, 640, 1280, 160), (560, 1280, 640, 40), (280, 320, 128, 40),
                                        (1024, 64, 64, 256), (4480, 1280, 320, 2240)])
@pytest.mark.parametrize("res", [False, True])
def test_fused_groupnorm_sums_linear(raw, M, N, K, rows, res):
    """gn_sum of svdx_tapgemm: per (slab, channel) sum / sum of squares of the stored output, plain and residual epilogues,
    M >= 512 and M < 512, slabs aligned (2560, 160) and NOT aligned (40) to the 32-row warp slices."""
    a = _rand(M, K, seed=1).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=2).to(bf16)
    bias = _rand(N, seed=3)
    r1 = _rand(M, N, seed=4).to(bf16) if res else None
    out = torch.empty(M, N, device=_dev(), dtype=bf16)
    sums = torch.zeros(M // rows, 2, N, device=_dev())
    raw.tapgemm(a, w, out, M=M, N=N, K=K, bias=bias, res1=r1, gn_sum=sums, gn_rows=rows)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias + (r1.float() if res else 0)
    _close(out, ref, what="linear + gn_sum")
    _check_gn_sums(sums, out, rows, f"linear {M}x{N}x{K} rows {rows} res {res}")
    # the stand-alone channel-sum kernel writes the buffer the epilogue wrote
    alone = raw.groupnorm_sums(out, None, M // rows, rows)
    _check_gn_sums(alone, out, rows, f"groupnorm_sums {M}x{N} rows {rows}")
    err = ((alone - sums).abs().amax((0, 2)) / (sums.abs().amax((0, 2)) + 1e-9)).max().item()
    assert err < 4e-5, f"groupnorm_sums vs the epilogue's gn_sum: {err:.3g}"


@pytest.mark.parametrize("N,H,W,Cin,Cout,per_clip", [(14, 40, 64, 64, 320, False), (14, 5, 8, 128, 160, False), (14, 10, 16, 320, 640, True),
                                                       (4, 20, 32, 192, 320, True)])
def test_fused_groupnorm_sums_conv3x3(raw, N, H, W, Cin, Cout, per_clip):
    x = _rand(N, H, W, Cin, seed=20).to(bf16)
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=21).to(bf16)
    bias = _rand(Cout, seed=22)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)
    out = torch.empty(N * H * W, Cout, device=_dev(), dtype=bf16)
    rows = N * H * W if per_clip else H * W
    sums = torch.zeros(N * H * W // rows, 2, Cout, device=_dev())
    raw.tapgemm(x.view(-1, Cin), wk, out, M=N * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS,
                conv_whn=(W, H, N), bias=bias, gn_sum=sums, gn_rows=rows)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    _close(out, ref, what="conv3x3 + gn_sum")
    _check_gn_sums(sums, out, rows, f"conv {N}x{H}x{W} {Cin}->{Cout}")


def test_fused_groupnorm_sums_temporal_conv_grouped(raw):
    """grouped ROWS mode (B = 2 clips): slab index must follow the GLOBAL row (group * rows_per_group + row)"""
    B, T, HW, C = 2, 5, 40, 320
    x = _rand(B, T, HW, C, seed=17).to(bf16)
    w = _rand(C, C, 3, scale=(3 * C) ** -0.5, seed=18).to(bf16)
    wk = w.permute(0, 2, 1).contiguous().view(C, 3 * C)
    out = torch.empty(B * T * HW, C, device=_dev(), dtype=bf16)
    taps = [(-HW, 0, 0), (0, 0, 0), (HW, 0, 0)]
    for rows in (HW, T * HW):
        sums = torch.zeros(B * T * HW // rows, 2, C, device=_dev())
        raw.tapgemm(x.view(-1, C), wk, out, M=B * T * HW, N=C, K=C, taps=taps, rows_per_group=T * HW, groups=B, gn_sum=sums, gn_rows=rows)
        torch.cuda.synchronize()
        _check_gn_sums(sums, out, rows, f"temporal conv slab {rows}")


@pytest.mark.parametrize("M,N,K,f32", [(1, 1280, 1024, False), (2, 320, 320, True), (1, 40320, 1280, True), (5, 640, 640, False), (8, 96, 64, True)])
def test_gemv_and_outer_accum_for_conditioning_vectors(raw, M, N, K, f32):
    """M <= 8 rows (time-embedding MLPs, time_emb_proj, the 1-key cross-attention vectors): tapgemm_auto routes them to the
    weight-streaming GEMV; their weight gradient is an outer-product accumulation."""
    a = _rand(M, K, seed=1).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=2).to(bf16)
    bias = _rand(N, seed=3)
    out = torch.full((M, N), float("nan"), device=_dev(), dtype=torch.float32 if f32 else bf16)
    launches = raw.LAUNCHES[0]
    raw.tapgemm_auto(a, w, out, M=M, N=N, K=K, bias=bias)
    torch.cuda.synchronize()
    assert raw.LAUNCHES[0] - launches == 1
    _close(out, a.float() @ w.float().t() + bias, what=f"gemv {M}x{N}x{K}")
    # LoRA side path form: out += scale * a w^T
    prev = out.clone()
    raw.gemv(a, w, out, M=M, N=N, K=K, scale=0.5, accumulate=True)
    torch.cuda.synchronize()
    _close(out, prev.float() + 0.5 * (a.float() @ w.float().t()), what="gemv accumulate")
    dy = _rand(M, N, seed=4).to(bf16)
    g = torch.full((N, K), 0.25, device=_dev())
    sc = torch.tensor([0.5], device=_dev())
    raw.outer_accum(dy, a, g, sc)
    torch.cuda.synchronize()
    _close(g, 0.25 + 0.5 * dy.float().t() @ a.float(), what="outer_accum")


# ---- 320-wide tile requests (block_n = 320): validated like any width, computed as 160-wide tiles
@pytest.mark.parametrize("M,N,K", [(35840, 320, 320), (2560, 640, 1280), (8960, 640, 2560), (1000, 320, 192), (70000, 960, 64)])
@pytest.mark.parametrize("res,gn", [(False, False), (True, False), (False, True), (True, True)])
def test_wide_tile_linear(raw, M, N, K, res, gn):
    a = _rand(M, K, seed=1).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=2).to(bf16)
    bias = _rand(N, seed=3)
    r1 = _rand(M, N, seed=4).to(bf16) if res else None
    out = torch.full((M, N), float("nan"), device=_dev(), dtype=bf16)
    rows = M // 5 if M % 5 == 0 else M
    sums = torch.zeros(M // rows, 2, N, device=_dev()) if gn else None
    raw.tapgemm(a, w, out, M=M, N=N, K=K, bias=bias, res1=r1, block_n=320, **({"gn_sum": sums, "gn_rows": rows} if gn else {}))
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias + (r1.float() if res else 0)
    _close(out, ref, what=f"wide linear {M}x{N}x{K} res {res}")
    if gn:
        _check_gn_sums(sums, out, rows, f"wide linear {M}x{N}x{K} rows {rows} res {res}")
    # the same problem through the 160-wide tiles must give the same values (same k order, same epilogue arithmetic)
    out2 = torch.empty_like(out)
    raw.tapgemm(a, w, out2, M=M, N=N, K=K, bias=bias, res1=r1, block_n=160)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(14, 40, 64, 320, 320), (14, 20, 32, 640, 640), (3, 40, 64, 64, 320), (14, 10, 16, 128, 640)])
def test_wide_tile_conv3x3(raw, N, H, W, Cin, Cout):
    x = _rand(N, H, W, Cin, seed=20).to(bf16)
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=21).to(bf16)
    bias = _rand(Cout, seed=22)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)
    out = torch.full((N * H * W, Cout), float("nan"), device=_dev(), dtype=bf16)
    sums = torch.zeros(N, 2, Cout, device=_dev())
    raw.tapgemm(x.view(-1, Cin), wk, out, M=N * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS,
                conv_whn=(W, H, N), bias=bias, gn_sum=sums, gn_rows=H * W, block_n=320)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    _close(out, ref, what="wide conv3x3")
    _check_gn_sums(sums, out, H * W, f"wide conv {N}x{H}x{W} {Cin}->{Cout}")


def test_wide_tile_rejected_where_unsupported(raw):
    a = _rand(1024, 64, seed=1).to(bf16)
    w = _rand(640, 64, seed=2).to(bf16)
    with pytest.raises(RuntimeError):      # (SvdxError is a RuntimeError) fp32 output: the generic epilogue has no wide form
        raw.tapgemm(a, w, torch.zeros(1024, 640, device=_dev()), M=1024, N=640, K=64, block_n=320)
    with pytest.raises(RuntimeError):      # N not a multiple of 320
        raw.tapgemm(a, w[:480], torch.empty(1024, 480, device=_dev(), dtype=bf16), M=1024, N=480, K=64, block_n=320)
    with pytest.raises(RuntimeError):      # small M: 1-CTA kernel
        raw.tapgemm(a[:256], w, torch.empty(256, 640, device=_dev(), dtype=bf16), M=256, N=640, K=64, block_n=320)


# ---- GroupNorm backward, pass 1 fused into the epilogue that writes dy (gnb_*), + svdx_groupnorm_bwd_fused
def _gnb_reference(x, dy, outer, rows, gamma, beta, silu):
    C = x.shape[1]
    xr = x.float().reshape(outer, rows, C).permute(0, 2, 1).requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    ref = F.group_norm(xr, 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref.backward(dy.float().view(outer, rows, C).permute(0, 2, 1))
    return xr.grad.permute(0, 2, 1).reshape(outer * rows, C), g.grad, b.grad


@pytest.mark.parametrize("M,N,K,rows,bn", [(35840, 320, 640, 2560, 320), (35840, 320, 640, 2560, 160), (2240, 640, 1280, 160, None),
                                           (560, 1280, 64, 40, None), (280, 320, 128, 40, None), (4480, 1280, 320, 2240, None)])
@pytest.mark.parametrize("silu,concat", [(True, False), (False, False), (True, True)])
def test_groupnorm_backward_sums_of_the_dgrad_epilogue_and_the_standalone_kernel(raw, M, N, K, rows, bn, silu, concat):
    """the GEMM writes dy (the gradient of a GroupNorm output) and accumulates sum e, sum e*x per (slab, channel); the fused
    backward kernel turns them into dx / dgamma / dbeta: compared with F.group_norm's backward on the bf16 dy it stored"""
    outer = M // rows
    a = _rand(M, K, seed=1).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=2).to(bf16)
    x = (_rand(M, N, seed=5) + 0.5).to(bf16)                      # the GroupNorm input
    gamma = _rand(N, seed=7) * 0.2 + 1.0
    beta = _rand(N, seed=8) * 0.1
    C1 = N // 2 if concat else N
    x1 = x[:, :C1] if concat else x
    x2 = x[:, C1:] if concat else None
    cs = raw.groupnorm_sums(x1, x2, outer, rows)
    y = torch.empty(M, N, device=_dev(), dtype=bf16)
    ab = torch.empty(outer, 2, N, device=_dev())
    mean, rstd = raw.groupnorm_apply_fused(x1, x2, outer, rows, 1e-5, cs, cs[:, :, C1:] if concat else None, gamma, beta, silu, y, ab=ab)
    torch.cuda.synchronize()
    cpg = N // 32
    scale = rstd.view(outer, 32).repeat_interleave(cpg, 1) * gamma
    shift = beta - mean.view(outer, 32).repeat_interleave(cpg, 1) * scale
    assert torch.allclose(ab[:, 0], scale, rtol=1e-5, atol=1e-6) and torch.allclose(ab[:, 1], shift, rtol=1e-5, atol=1e-5)
    dy = torch.full((M, N), float("nan"), device=_dev(), dtype=bf16)
    sums = torch.zeros(outer, 2, N, device=_dev())
    raw.tapgemm(a, w, dy, M=M, N=N, K=K, block_n=bn, gnb=dict(x=x1, x2=x2, ab=ab, rows=rows, silu=silu, sum=sums))
    torch.cuda.synchronize()
    _close(dy, a.float() @ w.float().t(), what="dy")
    # the sums against fp32 math on the stored bf16 dy
    z = x.float() * scale.repeat_interleave(rows, 0) + shift.repeat_interleave(rows, 0)
    e = dy.float() * ((torch.sigmoid(z) * (1 + z * (1 - torch.sigmoid(z)))) if silu else 1.0)
    S = e.view(outer, rows, N).sum(1)
    SX = (e * x.float()).view(outer, rows, N).sum(1)
    tol = 2e-3 * (e.abs().view(outer, rows, N).sum(1).max().item())
    assert (sums[:, 0] - S).abs().max().item() < tol and (sums[:, 1] - SX).abs().max().item() < 2 * tol
    # the stand-alone pass 1 on the same dy and scale / shift table writes the epilogue's sums
    alone = raw.groupnorm_bwd_sums(x1, x2, dy, outer, rows, ab, silu)
    assert (alone[:, 0] - sums[:, 0]).abs().max().item() < tol and (alone[:, 1] - sums[:, 1]).abs().max().item() < 2 * tol
    dx = torch.full((M, N), float("nan"), device=_dev(), dtype=bf16)
    dgamma = torch.zeros(N, device=_dev())
    dbeta = torch.zeros(N, device=_dev())
    dres = _rand(M, N, seed=10).to(bf16) if not concat else None
    raw.groupnorm_bwd_fused(x1, x2, dy, outer, rows, mean, rstd, gamma, beta, silu, sums, dx[:, :C1] if concat else dx,
                            dx[:, C1:] if concat else None, dgamma, dbeta, dres=dres)
    torch.cuda.synchronize()
    dxr, dgr, dbr = _gnb_reference(x, dy, outer, rows, gamma, beta, silu)
    _close(dx, dxr + (dres.float() if dres is not None else 0), what="fused groupnorm dx")
    _close(dgamma, dgr, what="fused groupnorm dgamma")
    _close(dbeta, dbr, what="fused groupnorm dbeta")


def test_groupnorm_backward_sums_of_a_conv3x3_dgrad(raw):
    Nimg, H, W, Cin, Cout = 14, 20, 32, 128, 640
    M = Nimg * H * W
    g = _rand(Nimg, H, W, Cin, seed=20).to(bf16)
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=21).to(bf16)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)
    x = (_rand(M, Cout, seed=5) + 0.3).to(bf16)
    gamma = _rand(Cout, seed=7) * 0.2 + 1.0
    beta = _rand(Cout, seed=8) * 0.1
    rows = H * W
    y = torch.empty(M, Cout, device=_dev(), dtype=bf16)
    ab = torch.empty(Nimg, 2, Cout, device=_dev())
    mean, rstd = raw.groupnorm_apply_fused(x, None, Nimg, rows, 1e-5, raw.groupnorm_sums(x, None, Nimg, rows), None, gamma, beta, True, y, ab=ab)
    dy = torch.empty(M, Cout, device=_dev(), dtype=bf16)
    sums = torch.zeros(Nimg, 2, Cout, device=_dev())
    raw.tapgemm(g.view(-1, Cin), wk, dy, M=M, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS, conv_whn=(W, H, Nimg),
                gnb=dict(x=x, x2=None, ab=ab, rows=rows, silu=True, sum=sums))
    dx = torch.empty(M, Cout, device=_dev(), dtype=bf16)
    raw.groupnorm_bwd_fused(x, None, dy, Nimg, rows, mean, rstd, gamma, beta, True, sums, dx, None)
    torch.cuda.synchronize()
    dxr, _, _ = _gnb_reference(x, dy, Nimg, rows, gamma, beta, True)
    _close(dx, dxr, what="conv dgrad + fused groupnorm backward")
