"""Decode at frame widths the row-box conv tiles cannot cover (portrait 512x320 and 1024x576, square 768x768, 640x384): the
phase-form Upsample2D runs its interleaved store on the im2col A path, and a 32-pixel store chunk may cross image rows and
images. The phase launches must compute exactly what they compute at a width the boxes tile (the input zero-padded on the
right, the output cropped back), and the whole decoder and pipeline must match their fp32 oracles at those sizes."""
import pytest
import torch
import torch.nn.functional as F

from test_pipeline_gpu import _models
from test_vae_decode import _build, _decode_parity, _rel

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16 = torch.bfloat16


def _box_width(W):
    """the narrowest width >= W that the row boxes tile"""
    if W > 128:
        return -(-W // 128) * 128
    return next(b for b in (1, 2, 4, 8, 16, 32, 64, 128) if b >= W)


def _phase_conv(x, w, bias):
    """the four phase launches of Upsample2D's conv on channels-last x [n, H, W, Cin] -> ([n*2H*2W, Cout] prefilled with NaN,
    the fused gn_sum [n, 2, Cout])"""
    from svd_xtend_b200 import raw
    from svd_xtend_b200.vae import PHASES, fold_upsample_conv_weight, phase_taps
    n, H, W, Cin = x.shape
    Cout = w.shape[0]
    k = fold_upsample_conv_weight(w)
    out = torch.full((n * 4 * H * W, Cout), float("nan"), device=DEV, dtype=bf16)
    sums = torch.zeros(n, 2, Cout, device=DEV)
    for i, (ph, pw) in enumerate(PHASES):
        wk = k[i].permute(0, 2, 3, 1).reshape(Cout, 4 * Cin).to(bf16).contiguous()
        raw.tapgemm(x.reshape(-1, Cin), wk, out, M=n * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=phase_taps(ph, pw),
                    conv_whn=(W, H, n), bias=bias, gn_sum=sums, gn_rows=H * W, phase=(ph, pw), block_n=128)
    return out, sums


# (n, H, W, Cin, Cout): chunks straddle image rows (W not a multiple of 32), wide widths that are not multiples of 128, and
# 3 x 40 where H*W % 32 != 0, so chunks also straddle images and the gn_sum slabs split mid-chunk
SHAPES = [(2, 5, 40, 128, 128), (2, 3, 72, 256, 128), (3, 4, 36, 128, 256), (2, 5, 48, 128, 128), (2, 7, 33, 128, 128),
          (2, 3, 144, 128, 128), (2, 2, 288, 128, 128), (2, 2, 576, 128, 128), (3, 3, 40, 128, 128)]


@pytest.mark.parametrize("n,H,W,Cin,Cout", SHAPES)
def test_interleaved_phase_conv_at_any_width(n, H, W, Cin, Cout):
    g = torch.Generator(device="cpu").manual_seed(n + H + W + Cin)
    x = torch.randn(n, H, W, Cin, generator=g).to(DEV, bf16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(DEV)
    bias = torch.randn(Cout, generator=g).to(DEV)
    out, sums = _phase_conv(x, w, bias)
    Wp = _box_width(W)
    outp, _ = _phase_conv(F.pad(x, (0, 0, 0, Wp - W)), w, bias)
    torch.cuda.synchronize()
    xr = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    ref = F.conv2d(xr, w, bias, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert torch.isfinite(out.float()).all()                      # every high-res row was written by one of the phases
    e = _rel(out, ref)
    assert e < 1e-2, (W, e)
    # the same launches at a width the boxes tile, cropped back: bitwise equal (and nothing was written past a row's end)
    crop = outp.view(n, 2 * H, 2 * Wp, Cout)[:, :, :2 * W].reshape(-1, Cout)
    assert torch.equal(out, crop), f"W={W}: the row-crossing store differs from the box-width launch"
    o3 = out.double().view(n, 4 * H * W, Cout)
    for m, s in ((0, o3.sum(1)), (1, (o3 * o3).sum(1))):
        assert (sums[:, m].double() - s).abs().max().item() < 2e-5 * s.abs().max().item() + 1e-3


def test_interleave_below_32_that_does_not_divide_32_is_refused():
    from svd_xtend_b200 import raw
    from svd_xtend_b200._lib import SvdxError
    x = torch.zeros(96, 128, device=DEV, dtype=bf16)
    wk = torch.zeros(128, 4 * 128, device=DEV, dtype=bf16)
    out = torch.zeros(4 * 96, 128, device=DEV, dtype=bf16)
    with pytest.raises(SvdxError, match="interleave"):
        raw.tapgemm(x, wk, out, M=96, N=128, K=128, mode=raw.A_CONV2D, taps=((0, 0, 0),) * 4, conv_whn=(24, 4, 1), phase=(0, 1))


# ------------------------------------------------------------------------------------------------ the decoder
@pytest.mark.parametrize("h,w", [(64, 40), (128, 72), (96, 96), (80, 48)])
def test_decode_svd_config_portrait_and_square(h, w):
    """512x320 and 1024x576 portrait, 768x768 square, 640x384 portrait frames"""
    from oracle.svd_vae_oracle import VAE_CONFIG
    _decode_parity(VAE_CONFIG, 2, h, w)


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("T,h,w,nclips", [(3, 6, 36, 2), (2, 10, 40, 2)])
def test_decode_tiny_at_row_crossing_widths(layers, T, h, w, nclips):
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    _decode_parity(dict(TINY_VAE_CONFIG, layers_per_block=layers), T, h, w, nclips=nclips)


def test_decode_latents_14_frames_512x320_portrait_chunk_8():
    from oracle.svd_vae_decoder_oracle import decode_latents as oracle_decode_latents
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.sampling import decode_latents
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _build(VAE_CONFIG, seed=19, device=DEV)
    g = torch.Generator(device="cpu").manual_seed(20)
    lat = (torch.randn(1, 14, 4, 64, 40, generator=g) * VAE_CONFIG["scaling_factor"]).to(DEV)
    with torch.no_grad():
        ref = oracle_decode_latents(oracle, lat, decode_chunk_size=8)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = oracle_decode_latents(oracle, lat, decode_chunk_size=8)
    got = decode_latents(ours, lat, decode_chunk_size=8)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (1, 3, 14, 512, 320) and got.dtype == torch.float32
    e, ea = _rel(got, ref), _rel(ac.float(), ref)
    print(f"decode_latents 14 x 512x320 chunk 8: rel-l2 {e:.4g} (torch bf16 autocast {ea:.4g})")
    assert e <= max(2 * ea, 2e-2), (e, ea)


# ------------------------------------------------------------------------------------------------ image to video
@pytest.mark.parametrize("H,W", [(96, 72), (80, 80)])
def test_tiny_pipeline_portrait_and_square_match_oracle_composition(H, W):
    """tiny-VAE levels of 36 / 72 and 40 / 80 pixels: every decoder level on the im2col path with row-crossing stores"""
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG, image_to_video
    from oracle.svd_unet_oracle import TINY_CONFIG
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.pipeline import ImageToVideoPipeline
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    (ou, u), (ov, v), (oc, c) = _models(TINY_CONFIG, TINY_VAE_CONFIG, dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"]), 23)
    image = torch.rand(1, 3, H, W, device=DEV)
    kw = dict(num_frames=4, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.02)
    out = ImageToVideoPipeline(u, v, c)(image, generator=torch.Generator(DEV).manual_seed(5), **kw).frames
    with torch.no_grad():
        ref = image_to_video(ou, ov, oc, image, generator=torch.Generator(DEV).manual_seed(5), **kw)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = image_to_video(ou, ov, oc, image, generator=torch.Generator(DEV).manual_seed(5), **kw)
    torch.cuda.synchronize()
    assert out.shape == ref.shape == (1, 4, 3, H, W) and out.dtype == torch.float32
    e, e_ac = _rel(out, ref), _rel(ac.float(), ref)
    print(f"tiny image-to-video {H}x{W}: rel-l2 {e:.3e} (oracle under bf16 autocast {e_ac:.3e})")
    assert torch.isfinite(out).all() and out.min() >= 0 and out.max() <= 1
    assert e <= max(2 * e_ac, 2e-2), (e, e_ac)


def test_svd_pipeline_portrait_512x320_equals_hand_composition():
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from oracle.svd_unet_oracle import SVD_CONFIG
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection, encode_image
    from svd_xtend_b200.pipeline import ImageToVideoPipeline
    from svd_xtend_b200.sampling import VideoLatentSampler, decode_latents
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(3)
    with torch.device(DEV):
        u = UNetSpatioTemporalConditionModel(**SVD_CONFIG).requires_grad_(False).eval()
        v = AutoencoderKLTemporalDecoder(**VAE_CONFIG, with_decoder=True).requires_grad_(False).eval()
        c = CLIPVisionModelWithProjection(**CLIP_CONFIG).requires_grad_(False).eval()
    image = torch.rand(1, 3, 512, 320, device=DEV)
    kw = dict(num_frames=14, num_inference_steps=2, decode_chunk_size=8)
    out = ImageToVideoPipeline(u, v, c)(image, generator=torch.Generator(DEV).manual_seed(9), **kw).frames

    def hand():
        g = torch.Generator(DEV).manual_seed(9)
        with torch.no_grad():
            x = image * 2 - 1
            emb = encode_image(c, x)
            cond = x + 0.02 * torch.randn(x.shape, generator=g, device=DEV)
            lat0 = v.encode(cond).latent_dist.mode()
            noise = torch.randn(1, 14, 4, 64, 40, generator=g, device=DEV)
            lat = VideoLatentSampler(u)(lat0, emb.unsqueeze(1), num_frames=14, num_inference_steps=2, noise=noise)
            return (decode_latents(v, lat, 8) / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4)
    ref, ref2 = hand(), hand()
    torch.cuda.synchronize()
    assert out.shape == (1, 14, 3, 512, 320) and torch.isfinite(out).all() and out.min() >= 0 and out.max() <= 1
    # bitwise when the stages are reproducible, else within 4x the run-to-run spread of two hand compositions (the fp32
    # atomics of the fused GroupNorm sums and split-K GEMMs reorder sums), as in test_pipeline_gpu
    if torch.equal(ref, ref2):
        print("hand composition reproducible: bit-for-bit comparison")
        assert torch.equal(out, ref)
    else:
        spread = _rel(ref2, ref)
        print(f"hand composition not reproducible (run-to-run spread {spread:.3e}): pipeline vs hand {_rel(out, ref):.3e}")
        assert _rel(out, ref) <= 4 * spread
