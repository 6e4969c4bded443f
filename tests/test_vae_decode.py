"""Temporal VAE decode (StableVideoDiffusionPipeline.decode_latents -> AutoencoderKLTemporalDecoder.decode) on the H100 path
against the oracle restatement of diffusers' TemporalDecoder (oracle/svd_vae_decoder_oracle.py), the two kernels it adds
(the interleaved-store phase form of Upsample2D in svdx_tapgemm, svdx_time_conv_out) and the host logic around them.
Decode tolerance as for the encode: rel-L2 <= max(2 x err(oracle under torch bf16 autocast), 2e-2) against the fp32 oracle."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

DEV = "cuda:0"
bf16 = torch.bfloat16


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _build(cfg, seed=0, device="cpu"):
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as Oracle
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder as Ours
    torch.manual_seed(seed)
    oracle = Oracle(**cfg, with_decoder=True)
    with torch.no_grad():
        for n, p in oracle.named_parameters():
            if "norm" in n or "mix_factor" in n:
                p.add_(0.1 * torch.randn_like(p))
    ours = Ours(**cfg, with_decoder=True)
    ours.load_state_dict(oracle.state_dict())
    return oracle.to(device).eval().requires_grad_(False), ours.to(device).eval().requires_grad_(False)


# ----------------------------------------------------------------------------------------------------------- CPU
def test_state_dict_contract_and_decoder_census():
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as Oracle
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder as Ours
    with torch.device("meta"):
        a, b = Ours(**VAE_CONFIG, with_decoder=True), Oracle(**VAE_CONFIG, with_decoder=True)
        plain = Ours(**VAE_CONFIG)
    ka = [(k, tuple(v.shape)) for k, v in a.state_dict().items()]
    assert ka == [(k, tuple(v.shape)) for k, v in b.state_dict().items()]
    dec = [(k, n) for k, n in ka if k.startswith("decoder.")]
    assert len(dec) == 266
    assert sum(torch.Size(s).numel() for _, s in dec) == 63_579_183
    assert sum(v.numel() for v in a.state_dict().values()) == 97_742_847
    assert a.decoder.mid_block.resnets[0].temporal_res_block.norm1.eps == 1e-5
    assert a.decoder.mid_block.resnets[0].spatial_res_block.norm1.eps == 1e-6
    # the default stays encode-only
    assert plain.decoder is None and all(k.startswith(("encoder.", "quant_conv.")) for k in plain.state_dict())


@pytest.mark.parametrize("n,H,W", [(1, 4, 6), (2, 5, 7), (3, 6, 3), (2, 1, 1)])
def test_upsample_phase_fold_identity(n, H, W):
    """conv3x3(nearest2x(x)) == the four folded 2x2-tap phase convolutions at the low-res geometry, interleaved (fp64)"""
    from svd_xtend_b200.vae import PHASES, fold_upsample_conv_weight, phase_taps
    g = torch.Generator().manual_seed(n * 100 + H * 10 + W)
    I, O = 5, 3
    x = torch.randn(n, I, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(O, I, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, padding=1)
    k = fold_upsample_conv_weight(w)
    assert k.shape == (4, O, I, 2, 2)
    out = torch.zeros_like(ref)
    xp = F.pad(x, (1, 1, 1, 1))
    for i, (ph, pw) in enumerate(PHASES):
        y = F.conv2d(xp, k[i])[..., ph:ph + H, pw:pw + W]
        # the same phase through the device tap list: k[:, :, a, b] reads x[h + dh, w + dw]
        yt = torch.zeros_like(y)
        for t, (dw, dh, dn) in enumerate(phase_taps(ph, pw)):
            assert dn == 0
            a, b = divmod(t, 2)
            yt += torch.einsum("oi,nihw->nohw", k[i][:, :, a, b], xp[:, :, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W])
        assert (yt - y).abs().max().item() < 1e-12
        out[..., ph::2, pw::2] = y
    assert (out - ref).abs().max().item() < 1e-12 * max(1.0, ref.abs().max().item())


def test_oracle_switched_alpha_blender():
    from oracle.svd_vae_decoder_oracle import AlphaBlender
    torch.manual_seed(0)
    m = AlphaBlender(0.0, switch_spatial_to_temporal_mix=True)
    with torch.no_grad():
        m.mix_factor.fill_(0.37)
    xs, ht = torch.randn(2, 8, 3, 4, 4), torch.randn(2, 8, 3, 4, 4)
    ref = xs + torch.sigmoid(torch.tensor(0.37)) * ht
    assert torch.allclose(m(xs, xs + ht), ref, atol=1e-6)


def test_oracle_decode_latents_chunks_are_separate_clips():
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as Oracle, decode_latents
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    torch.manual_seed(3)
    vae = Oracle(**TINY_VAE_CONFIG, with_decoder=True).eval()
    lat = torch.randn(1, 14, 4, 4, 8)
    with torch.no_grad():
        out = decode_latents(vae, lat, decode_chunk_size=8)
        sf = 1.0 / vae.config.scaling_factor
        a = vae.decode(lat[0, :8] * sf, num_frames=8).sample
        b = vae.decode(lat[0, 8:] * sf, num_frames=6).sample
        whole = decode_latents(vae, lat, decode_chunk_size=14)
    assert out.shape == (1, 3, 14, 8, 16) and out.dtype == torch.float32
    sep = torch.cat([a, b]).permute(1, 0, 2, 3)[None]
    assert torch.allclose(out, sep, atol=1e-6)
    assert torch.allclose(decode_latents(vae, lat), whole)           # default chunk = all frames
    assert _rel(out, whole) > 1e-4                                   # the temporal layers see where the clips are cut


def test_decode_guards_without_gpu():
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder as Ours
    m = Ours(**TINY_VAE_CONFIG, with_decoder=True).requires_grad_(False)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.decode(torch.zeros(2, 4, 4, 8), num_frames=2)
    with pytest.raises(ValueError, match="num_frames"):
        m.decode(torch.zeros(3, 4, 4, 8), num_frames=2)
    with pytest.raises(ValueError, match="128"):
        m.decode(torch.zeros(1, 4, 4, 24), num_frames=1)               # width 24 does not tile the 128-pixel conv tiles
    with pytest.raises(ValueError, match="% 32"):
        m.decode(torch.zeros(1, 4, 3, 8), num_frames=1)                # 3 x 8 low-res: a 32-pixel store chunk straddles images
    with pytest.raises(RuntimeError, match="with_decoder"):
        Ours(**TINY_VAE_CONFIG).decode(torch.zeros(1, 4, 4, 8), num_frames=1)


def test_decode_benchmark_flop_count():
    """scripts/bench_decode.py counts the decoder's work from shapes; the phase form removes 20 of the 36 tap-products per
    low-res pixel of every Upsample2D conv"""
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "bench_decode.py")
    spec = importlib.util.spec_from_file_location("bench_decode", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    boc = (128, 256, 512, 512)
    ref = mod.decoder_flops(boc, 2, 4, 3, 72, 128, 1, False)
    exe = mod.decoder_flops(boc, 2, 4, 3, 72, 128, 1, True)
    assert 6.9e12 < ref < 7.0e12                                      # ~6.9 TFLOP per 576x1024 frame
    up = sum(c * c * (72 * 128 << 2 * i) for i, c in enumerate((512, 512, 256)))
    assert ref - exe == 2.0 * 20 * up
    assert 1.85e12 < mod.decoder_flops(boc, 2, 4, 3, 40, 64, 1, False) < 1.95e12
    assert mod.decoder_flops(boc, 2, 4, 3, 40, 64, 14, False) == 14 * mod.decoder_flops(boc, 2, 4, 3, 40, 64, 1, False)


def test_time_conv_out_rejects_bad_arguments_without_gpu():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200._lib import load
    lib = load()
    p = ctypes.c_void_p(1024)           # never dereferenced: every call below fails validation first
    assert lib.svdx_time_conv_out(None, 8, 2, 2, 3, 4, 4, p, None, p, 0, None) == -1
    assert lib.svdx_time_conv_out(p, 8, 3, 2, 3, 4, 4, p, None, p, 0, None) == -1      # N not a multiple of T
    assert lib.svdx_time_conv_out(p, 16, 2, 2, 9, 4, 4, p, None, p, 0, None) == -1     # C > 8
    assert lib.svdx_time_conv_out(p, 6, 2, 2, 3, 4, 4, p, None, p, 0, None) == -1      # ldx % 4
    assert lib.svdx_time_conv_out(p, 8, 2, 2, 3, 4, 4, p, None, p, 3, None) == -1      # output dtype code
    assert b"time_conv_out" in lib.svdx_last_error()


# ----------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("n,H,W,Cin,Cout", [(3, 8, 16, 128, 128), (2, 6, 64, 256, 256), (2, 4, 128, 512, 512), (2, 3, 256, 256, 128),
                                            (1, 2, 512, 128, 128), (5, 2, 16, 128, 256)])
def test_interleaved_phase_conv_matches_upsample_conv(n, H, W, Cin, Cout):
    from svd_xtend_b200 import raw
    from svd_xtend_b200.vae import PHASES, fold_upsample_conv_weight, phase_taps
    g = torch.Generator(device="cpu").manual_seed(n + H + W + Cin)
    x = torch.randn(n, H, W, Cin, generator=g).to(DEV, bf16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(DEV)
    bias = torch.randn(Cout, generator=g).to(DEV)
    k = fold_upsample_conv_weight(w)
    out = torch.full((n * 4 * H * W, Cout), float("nan"), device=DEV, dtype=bf16)
    sums = torch.zeros(n, 2, Cout, device=DEV)
    for i, (ph, pw) in enumerate(PHASES):
        wk = k[i].permute(0, 2, 3, 1).reshape(Cout, 4 * Cin).to(bf16).contiguous()
        raw.tapgemm(x.view(-1, Cin), wk, out, M=n * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=phase_taps(ph, pw), conv_whn=(W, H, n),
                    bias=bias, gn_sum=sums, gn_rows=H * W, phase=(ph, pw))
    torch.cuda.synchronize()
    xr = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    ref = F.conv2d(xr, w, bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert torch.isfinite(out.float()).all()                      # every high-res row was written by exactly one phase
    e = _rel(out, ref)
    assert e < 1e-2, (W, e)
    o3 = out.double().view(n, 4 * H * W, Cout)
    for m, s in ((0, o3.sum(1)), (1, (o3 * o3).sum(1))):
        assert (sums[:, m].double() - s).abs().max().item() < 2e-5 * s.abs().max().item() + 1e-3


@pytest.mark.gpu
def test_interleaved_store_rejects_epilogue_operands():
    from svd_xtend_b200 import raw
    from svd_xtend_b200._lib import SvdxError
    x = torch.zeros(64, 128, device=DEV, dtype=bf16)
    wk = torch.zeros(128, 4 * 128, device=DEV, dtype=bf16)
    out = torch.zeros(256, 128, device=DEV, dtype=bf16)
    kw = dict(M=64, N=128, K=128, mode=raw.A_CONV2D, taps=((0, 0, 0),) * 4, conv_whn=(16, 4, 1), phase=(0, 1))
    with pytest.raises(SvdxError, match="interleave"):
        raw.tapgemm(x, wk, out, res1=out[:64], **kw)
    with pytest.raises(SvdxError, match="interleave"):
        raw.tapgemm(x, wk, torch.zeros(256, 128, device=DEV), **kw)           # fp32 output
    with pytest.raises(SvdxError, match="interleave"):
        raw.tapgemm(x, wk, out, **dict(kw, M=48, conv_whn=(16, 3, 1)))       # 3 x 16 low-res rows: chunks straddle images


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 6, 8, 14])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_time_conv_out_matches_conv3d(T, dtype):
    from svd_xtend_b200 import raw
    g = torch.Generator(device="cpu").manual_seed(T)
    B, C, H, W = 2, 3, 5, 7
    N = B * T
    x = torch.randn(N * H * W, 8, generator=g).to(DEV)
    w = torch.randn(C, C, 3, 1, 1, generator=g).to(DEV)
    b = torch.randn(C, generator=g).to(DEV)
    out = torch.empty(N, C, H, W, device=DEV, dtype=dtype)
    raw.time_conv_out(x, w, b, out, T)
    torch.cuda.synchronize()
    xi = x[:, :C].reshape(B, T, H, W, C).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(xi, w, b, padding=(1, 0, 0)).permute(0, 2, 1, 3, 4).reshape(N, C, H, W)
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert (out.float() - ref).abs().max().item() <= tol * ref.abs().max().item()
    # the clip-edge frames (zero padding at both ends of each clip, not across clips)
    for t in {0, T - 1}:
        assert torch.allclose(out.float()[t::T], ref[t::T], atol=tol * ref.abs().max().item())


def _decode_parity(cfg, T, h, w, seed=5, nclips=1):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _build(cfg, seed=seed, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    z = torch.randn(nclips * T, cfg["latent_channels"], h, w, generator=g).to(DEV)
    with torch.no_grad():
        ref = oracle.decode(z, num_frames=T).sample
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = oracle.decode(z, num_frames=T).sample
        got = ours.decode(z, num_frames=T).sample
    torch.cuda.synchronize()
    up = 1 << (len(cfg["block_out_channels"]) - 1)
    assert got.shape == ref.shape == (nclips * T, 3, h * up, w * up) and got.dtype == torch.float32
    assert torch.isfinite(got).all()
    e, ea = _rel(got, ref), _rel(ac.float(), ref)
    print(f"decode {cfg['block_out_channels']} T={T} {h}x{w}: rel-l2 {e:.4g} (torch bf16 autocast {ea:.4g})")
    assert e <= max(2 * ea, 2e-2), (e, ea)
    return oracle, ours, z


@pytest.mark.gpu
@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("T,h,w,nclips", [(1, 8, 16, 1), (3, 4, 32, 1), (5, 8, 8, 1), (2, 6, 16, 2)])
def test_decode_tiny_matches_oracle(layers, T, h, w, nclips):
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    _decode_parity(dict(TINY_VAE_CONFIG, layers_per_block=layers), T, h, w, nclips=nclips)


@pytest.mark.gpu
def test_decode_full_config_small_latent_and_guards():
    from oracle.svd_vae_oracle import VAE_CONFIG
    oracle, ours, z = _decode_parity(VAE_CONFIG, 3, 8, 16)
    with torch.no_grad():
        half = ours.decode(z.to(bf16), num_frames=3).sample           # output dtype follows the input, as for encode
    assert half.dtype == bf16
    with pytest.raises(RuntimeError, match="forward-only"):
        ours.requires_grad_(True)
        ours.decode(z, num_frames=3)


@pytest.mark.gpu
def test_decode_576x1024_chunk_of_two():
    """the notebook's frame size: 1024-pixel-wide conv tiles and the S = 9216 mid-block attention"""
    from oracle.svd_vae_oracle import VAE_CONFIG
    _decode_parity(VAE_CONFIG, 2, 72, 128)


@pytest.mark.gpu
def test_decode_latents_14_frames_320x512_chunk_8():
    from oracle.svd_vae_decoder_oracle import decode_latents as oracle_decode_latents
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.sampling import decode_latents
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _build(VAE_CONFIG, seed=9, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(10)
    lat = (torch.randn(1, 14, 4, 40, 64, generator=g) * VAE_CONFIG["scaling_factor"]).to(DEV)
    with torch.no_grad():
        ref = oracle_decode_latents(oracle, lat, decode_chunk_size=8)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = oracle_decode_latents(oracle, lat, decode_chunk_size=8)
    got = decode_latents(ours, lat, decode_chunk_size=8)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (1, 3, 14, 320, 512) and got.dtype == torch.float32
    e, ea = _rel(got, ref), _rel(ac.float(), ref)
    print(f"decode_latents 14 x 320x512 chunk 8: rel-l2 {e:.4g} (torch bf16 autocast {ea:.4g})")
    assert e <= max(2 * ea, 2e-2), (e, ea)


@pytest.mark.gpu
def test_sample_then_decode_end_to_end():
    """VideoLatentSampler -> decode_latents on the tiny UNet and tiny VAE against the oracle loop -> oracle decode_latents"""
    from oracle.svd_sampling_oracle import sample_latents
    from oracle.svd_unet_oracle import TINY_CONFIG
    from oracle.svd_vae_decoder_oracle import decode_latents as oracle_decode_latents
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.sampling import VideoLatentSampler, decode_latents
    from test_unet_gpu import _build as build_unet
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle_unet, unet = build_unet(TINY_CONFIG, seed=41)
    oracle_unet.eval()
    oracle_vae, vae = _build(TINY_VAE_CONFIG, seed=42, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(7)
    B, T, h, w = 1, 4, 16, 16
    image_latents = torch.randn(B, 4, h, w, generator=g).to(DEV)
    emb = torch.randn(B, 1, TINY_CONFIG["cross_attention_dim"], generator=g).to(DEV)
    noise = torch.randn(B, T, 4, h, w, generator=g).to(DEV)
    kw = dict(num_frames=T, num_inference_steps=4, min_guidance_scale=1.0, max_guidance_scale=3.0, noise=noise)
    with torch.no_grad():
        ref = oracle_decode_latents(oracle_vae, sample_latents(oracle_unet, image_latents, emb, **kw), decode_chunk_size=3)
    got = decode_latents(vae, VideoLatentSampler(unet)(image_latents, emb, **kw), decode_chunk_size=3)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (B, 3, T, 2 * h, 2 * w) and torch.isfinite(got).all()
    e = _rel(got, ref)
    print("sample + decode rel-l2", e)
    assert e < 4e-2, e
