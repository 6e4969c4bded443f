"""SURVEY.md §8f-1 — VAE encode (train_svd.py:283-291, :948, :959) on the H100 path against the oracle restatement of
diffusers' AutoencoderKLTemporalDecoder.encode (oracle/svd_vae_oracle.py). Tolerance as for the UNet: rel-L2 of the moments
<= max(2 x err(oracle under torch bf16 autocast), 2e-2) against the fp32 oracle."""
import pytest
import torch

DEV = "cuda:0"


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def _build(cfg, seed=0, device="cpu"):
    from oracle.svd_vae_oracle import AutoencoderKLTemporalDecoder as Oracle
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder as Ours
    torch.manual_seed(seed)
    oracle = Oracle(**cfg)
    with torch.no_grad():
        for n, p in oracle.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
    ours = Ours(**cfg)
    ours.load_state_dict(oracle.state_dict())
    return oracle.to(device).eval().requires_grad_(False), ours.to(device).eval().requires_grad_(False)


def test_state_dict_contract_and_census():
    from oracle.svd_vae_oracle import VAE_CONFIG, AutoencoderKLTemporalDecoder as Oracle
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder as Ours
    with torch.device("meta"):
        a, b = Ours(**VAE_CONFIG), Oracle(**VAE_CONFIG)
    ka = [(k, tuple(v.shape)) for k, v in a.state_dict().items()]
    assert ka == [(k, tuple(v.shape)) for k, v in b.state_dict().items()]
    assert sum(v.numel() for v in a.state_dict().values()) == 34_163_664       # encoder + quant_conv of the SD / SVD VAE
    assert all(k.startswith(("encoder.", "quant_conv.")) for k, _ in ka)
    assert a.config.scaling_factor == 0.18215


def test_encode_is_forward_only_and_has_no_cpu_path():
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder as Ours
    m = Ours(**TINY_VAE_CONFIG)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.encode(torch.zeros(1, 3, 16, 128))


def test_oracle_downsample_is_pad_right_bottom():
    """the restated Downsample2D: F.pad(x, (0,1,0,1)) + stride-2 conv == the parity-plane taps the CUDA path uses"""
    from oracle.svd_vae_oracle import Downsample2D
    torch.manual_seed(0)
    d = Downsample2D(4)
    x = torch.randn(2, 4, 6, 8)
    y = d(x)
    w, b = d.conv.weight, d.conv.bias
    ref = torch.zeros_like(y)
    xp = torch.zeros(2, 4, 7, 9)
    xp[:, :, :6, :8] = x
    for kh in range(3):
        for kw in range(3):
            ref += torch.einsum("oi,bihw->bohw", w[:, :, kh, kw], xp[:, :, kh:kh + 6:2, kw:kw + 8:2])
    assert torch.allclose(y, ref + b[None, :, None, None], atol=1e-5)


@pytest.mark.gpu
def test_softmax_rows_kernel():
    from svd_xtend_b200 import raw
    for rows, cols, scale in ((128, 128, 0.044), (77, 2560, 0.044), (5, 9216, 1.0)):
        x = (torch.randn(rows, cols, device=DEV) * 8).to(torch.bfloat16)
        y = torch.empty_like(x)
        raw.softmax_rows(x, y, scale)
        torch.cuda.synchronize()
        ref = torch.softmax(x.float() * scale, dim=-1)
        assert (y.float() - ref).abs().max().item() < 2e-2 * ref.max().item() + 1e-4
        assert torch.allclose(y.float().sum(-1), torch.ones(rows, device=DEV), atol=2e-2)


@pytest.mark.gpu
def test_tapgemm_mixed_major_pv_and_wide_conv():
    """the two kernel forms the VAE adds: K-major A with an MN-major B (P V with V read in place) and 3x3 conv tiles on images
    wider than 128 pixels"""
    import torch.nn.functional as F
    from svd_xtend_b200 import raw
    bf16 = torch.bfloat16
    g = torch.Generator(device="cpu").manual_seed(3)
    S, C = 384, 512
    p = torch.softmax(torch.randn(S, S, generator=g), -1).to(DEV, bf16)
    qkv = torch.randn(S, 3 * C, generator=g).to(DEV, bf16)
    o = torch.empty(S, C, device=DEV, dtype=bf16)
    raw.tapgemm(p, qkv[:, 2 * C:], o, M=S, N=C, K=S, b_mn=True, ldb=qkv.stride(0))
    torch.cuda.synchronize()
    ref = p.float() @ qkv[:, 2 * C:].float()
    assert _rel(o, ref) < 1e-2, _rel(o, ref)
    for (N, H, W, Cin, Cout) in ((2, 6, 256, 64, 128), (1, 4, 512, 64, 64), (3, 5, 128, 128, 64)):
        x = torch.randn(N, H, W, Cin, generator=g).to(DEV, bf16)
        w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(DEV, bf16)
        bias = torch.randn(Cout, generator=g).to(DEV)
        wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)
        out = torch.empty(N * H * W, Cout, device=DEV, dtype=bf16)
        sums = torch.zeros(N, 2, Cout, device=DEV)
        raw.tapgemm(x.view(-1, Cin), wk, out, M=N * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS, conv_whn=(W, H, N),
                    bias=bias, gn_sum=sums, gn_rows=H * W)
        torch.cuda.synchronize()
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
        assert _rel(out, ref) < 1e-2, (W, _rel(out, ref))
        o3 = out.double().view(N, H * W, Cout)
        assert (sums[:, 0].double() - o3.sum(1)).abs().max().item() < 2e-5 * o3.sum(1).abs().max().item() + 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,N,H,W", [("tiny", 3, 16, 256), ("tiny", 2, 32, 64), ("full", 2, 64, 128), ("full", 1, 320, 512)])
def test_vae_encode_matches_oracle(cfg_name, N, H, W):
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG, VAE_CONFIG, tensor_to_vae_latent as oracle_latents
    from svd_xtend_b200.vae import tensor_to_vae_latent
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = TINY_VAE_CONFIG if cfg_name == "tiny" else VAE_CONFIG
    oracle, ours = _build(cfg, seed=5, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(11)
    x = (torch.randn(N, 3, H, W, generator=g) * 0.5).clamp(-1, 1).to(DEV)
    with torch.no_grad():
        ref = oracle.encode(x).latent_dist
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = oracle.encode(x).latent_dist
        got = ours.encode(x).latent_dist
    torch.cuda.synchronize()
    lv = len(cfg["block_out_channels"]) - 1
    assert got.mean.shape == ref.mean.shape == (N, 4, H >> lv, W >> lv)
    ref_m, ac_m, got_m = (torch.cat([d.mean, d.logvar], 1) for d in (ref, ac, got))
    e, ea = _rel(got_m, ref_m), _rel(ac_m.float(), ref_m)
    print(f"vae {cfg_name} {N}x{H}x{W}: moments rel-l2 {e:.4g} (torch bf16 autocast {ea:.4g})")
    assert torch.isfinite(got_m).all()
    assert e <= max(2 * ea, 2e-2), (e, ea)
    # the caller's function (train_svd.py:283-291) with a shared noise draw
    noise = torch.randn(ref.mean.shape, generator=g).to(DEV)
    a = tensor_to_vae_latent(x[None], ours, noise=noise)
    b = oracle_latents(x[None], oracle, noise=noise)
    assert a.shape == b.shape == (1, N, 4, H >> lv, W >> lv)
    assert _rel(a, b) <= max(2 * ea, 2e-2) * 1.5
    with pytest.raises(RuntimeError, match="forward-only"):
        ours.requires_grad_(True)
        ours.encode(x)
