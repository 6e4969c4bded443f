"""Inference path (SURVEY.md §8f-3, UNet-facing part): Euler / classifier-free-guidance sampling loop around the forward-only
H100 UNet against the oracle restatement of diffusers' StableVideoDiffusionPipeline loop (oracle/svd_sampling_oracle.py)."""
import pytest
import torch

from test_unet_gpu import DEV, _build, _rel


def test_karras_sigmas_host_logic():
    from oracle.svd_sampling_oracle import karras_sigmas as ref
    from svd_xtend_b200.sampling import karras_sigmas
    for n in (1, 2, 25, 30):
        a, b = karras_sigmas(n), ref(n)
        assert a.shape == (n + 1,) and torch.equal(a, b)
        assert abs(float(a[0]) - 700.0) < 1e-3 and float(a[-1]) == 0.0 and (n == 1 or abs(float(a[-2]) - 0.002) < 1e-6)
        assert all(float(a[i]) > float(a[i + 1]) for i in range(n))


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_sampling_loop_matches_oracle(graph):
    from oracle.svd_sampling_oracle import sample_latents
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.sampling import VideoLatentSampler
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _build(TINY_CONFIG, seed=41)
    oracle.eval()
    g = torch.Generator(device="cpu").manual_seed(7)
    B, T, h, w = 1, 4, 16, 16
    image_latents = torch.randn(B, 4, h, w, generator=g).to(DEV)
    emb = torch.randn(B, 1, TINY_CONFIG["cross_attention_dim"], generator=g).to(DEV)
    noise = torch.randn(B, T, 4, h, w, generator=g).to(DEV)
    kw = dict(num_frames=T, fps=7, motion_bucket_id=127, noise_aug_strength=0.02, num_inference_steps=4, min_guidance_scale=1.0,
              max_guidance_scale=3.0, noise=noise)
    with torch.no_grad():
        ref = sample_latents(oracle, image_latents, emb, **kw)
    sampler = VideoLatentSampler(ours, use_cuda_graph=graph)
    out = sampler(image_latents, emb, **kw)
    out2 = sampler(image_latents, emb, **kw)       # second call re-uses the captured step
    torch.cuda.synchronize()
    assert out.shape == ref.shape == (B, T, 4, h, w) and torch.isfinite(out).all()
    e = _rel(out, ref)
    print("sampling rel-l2 after 4 steps", e, "graph" if graph else "eager")
    assert e < 4e-2, e                 # bf16 UNet, errors compound over the steps
    assert _rel(out2, out) < 4e-2
