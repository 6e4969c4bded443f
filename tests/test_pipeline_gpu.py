"""Image -> video end to end (svd_xtend_b200.pipeline.ImageToVideoPipeline): against the oracle composition of diffusers'
StableVideoDiffusionPipeline (oracle/svd_clip_oracle.image_to_video) at tiny configs, and against the hand composition of the
package's stages at the SVD configs with the same generator draws."""
import pytest
import torch

DEV = "cuda:0"


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _models(unet_cfg, vae_cfg, clip_cfg, seed):
    from oracle.svd_clip_oracle import CLIPVisionModelWithProjection as OClip
    from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as OUnet
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as OVae
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(seed)
    pairs = []
    for O, P, kw in ((OUnet, UNetSpatioTemporalConditionModel, unet_cfg), (OVae, AutoencoderKLTemporalDecoder, dict(vae_cfg, with_decoder=True)),
                     (OClip, CLIPVisionModelWithProjection, clip_cfg)):
        o = O(**kw).to(DEV)
        with torch.no_grad():
            for n, p in o.named_parameters():
                if "norm" in n:
                    p.add_(0.1 * torch.randn_like(p))
        with torch.device(DEV):
            ours = P(**kw)
        ours.load_state_dict(o.state_dict())
        pairs.append((o.eval().requires_grad_(False), ours.eval().requires_grad_(False)))
    return pairs


@pytest.mark.gpu
def test_tiny_pipeline_matches_oracle_composition():
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG, image_to_video
    from oracle.svd_unet_oracle import TINY_CONFIG
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.pipeline import ImageToVideoPipeline
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    (ou, u), (ov, v), (oc, c) = _models(TINY_CONFIG, TINY_VAE_CONFIG, dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"]), 21)
    image = torch.rand(1, 3, 32, 32, device=DEV)
    kw = dict(num_frames=4, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.02)
    pipe = ImageToVideoPipeline(u, v, c)
    # a CUDA generator, and a CPU generator (drawn on the CPU, then moved, as diffusers' randn_tensor does)
    for gdev in (DEV, "cpu"):
        out = pipe(image, generator=torch.Generator(gdev).manual_seed(5), **kw).frames
        with torch.no_grad():
            ref = image_to_video(ou, ov, oc, image, generator=torch.Generator(gdev).manual_seed(5), **kw)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                ac = image_to_video(ou, ov, oc, image, generator=torch.Generator(gdev).manual_seed(5), **kw)
        torch.cuda.synchronize()
        assert out.shape == ref.shape == (1, 4, 3, 32, 32) and out.dtype == torch.float32
        e, e_ac = _rel(out, ref), _rel(ac.float(), ref)
        print(f"tiny image-to-video ({gdev} generator) rel-l2 {e:.3e} (oracle under bf16 autocast {e_ac:.3e})")
        assert torch.isfinite(out).all() and out.min() >= 0 and out.max() <= 1
        assert e <= max(2 * e_ac, 2e-2), (e, e_ac)


@pytest.mark.gpu
def test_svd_pipeline_equals_hand_composition():
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from oracle.svd_unet_oracle import SVD_CONFIG
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.clip import encode_image
    from svd_xtend_b200.pipeline import ImageToVideoPipeline
    from svd_xtend_b200.sampling import VideoLatentSampler, decode_latents
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(2)
    with torch.device(DEV):
        u = UNetSpatioTemporalConditionModel(**SVD_CONFIG).requires_grad_(False).eval()
        v = AutoencoderKLTemporalDecoder(**VAE_CONFIG, with_decoder=True).requires_grad_(False).eval()
        c = CLIPVisionModelWithProjection(**CLIP_CONFIG).requires_grad_(False).eval()
    image = torch.rand(1, 3, 320, 512, device=DEV)
    kw = dict(num_frames=14, num_inference_steps=2, decode_chunk_size=8)
    out = ImageToVideoPipeline(u, v, c)(image, generator=torch.Generator(DEV).manual_seed(9), **kw).frames

    def hand():
        g = torch.Generator(DEV).manual_seed(9)
        with torch.no_grad():
            x = image * 2 - 1
            emb = encode_image(c, x)
            cond = x + 0.02 * torch.randn(x.shape, generator=g, device=DEV)
            lat0 = v.encode(cond).latent_dist.mode()
            noise = torch.randn(1, 14, 4, 40, 64, generator=g, device=DEV)
            lat = VideoLatentSampler(u)(lat0, emb.unsqueeze(1), num_frames=14, num_inference_steps=2, noise=noise)
            return (decode_latents(v, lat, 8) / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4)
    ref, ref2 = hand(), hand()
    torch.cuda.synchronize()
    assert out.shape == (1, 14, 3, 320, 512) and torch.isfinite(out).all() and out.min() >= 0 and out.max() <= 1
    # Bit equality is required whenever the stages are reproducible. At these configs they are not: the fused GroupNorm sums
    # and the split-K GEMMs accumulate with fp32 atomics, so two hand compositions differ at the bf16 noise floor (~1e-2
    # rel-L2), and the pipeline must then stay within that run-to-run spread. A wrong draw order or a missing stage is off
    # by orders of magnitude more (the draws are unit-variance noise).
    if torch.equal(ref, ref2):
        print("hand composition reproducible: bit-for-bit comparison")
        assert torch.equal(out, ref)
    else:
        spread = _rel(ref2, ref)
        print(f"hand composition not reproducible (run-to-run spread {spread:.3e}): pipeline vs hand {_rel(out, ref):.3e}")
        assert _rel(out, ref) <= 4 * spread
