"""The drop-in StableVideoDiffusionPipeline and VAE on the H100 (tiny configs written to tmp_path): passed modules left as
they are, the call against ImageToVideoPipeline and against the composition by hand, the output conversions, fp16 VAE weights
and their force_upcast round trip against the fp32 oracle, the script's per-step encode in its three dtypes, and train_svd.py's
validation sequence between training steps of a graphed UNet with an EMA or a LoRA adapter."""
import gc
import os
import weakref
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_script_pipeline import write_tiny_checkpoint

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KW = dict(height=32, width=32, num_frames=4, num_inference_steps=3, decode_chunk_size=3)


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _agree(got, ref, ref2, what):
    """the rule of tests/test_pipeline_gpu.py for two compositions of the same stages: bit equality when the stages are
    reproducible, otherwise within 4x their run-to-run spread (fp32 atomics in the fused GroupNorm sums / split-K GEMMs)"""
    if torch.equal(ref, ref2):
        assert torch.equal(got, ref), (what, _rel(got, ref))
    else:
        spread = _rel(ref2, ref)
        print(f"{what}: not reproducible (spread {spread:.3e}), got vs ref {_rel(got, ref):.3e}")
        assert _rel(got, ref) <= 4 * spread, what


def _models(tmp_path, seed=0):
    unet, vae, enc = write_tiny_checkpoint(str(tmp_path), seed=seed)
    for m in (unet, vae, enc):
        m.to(DEV).requires_grad_(False).eval()
    return unet, vae, enc


def test_passed_modules_untouched_and_call_matches_image_to_video(tmp_path):
    from svd_xtend_b200.pipeline import ImageToVideoPipeline, StableVideoDiffusionPipeline, postprocess_video
    unet, vae, enc = _models(tmp_path)
    vae.to(torch.bfloat16)
    unet.train()
    for n, p in unet.named_parameters():
        p.requires_grad_("temporal_transformer_block" in n)
    state = [(p.dtype, p.device, p.requires_grad, p.data_ptr(), p._version) for m in (unet, vae, enc) for p in m.parameters()]
    pipe = StableVideoDiffusionPipeline.from_pretrained(str(tmp_path), unet=unet, vae=vae, image_encoder=enc, torch_dtype=torch.float16)
    pipe.to(DEV)
    pipe.set_progress_bar_config(disable=True)
    image = torch.rand(1, 3, 32, 32, device=DEV)
    out = {}
    for t in ("pt", "np", "pil", "latent"):
        out[t] = pipe(image, generator=torch.Generator(DEV).manual_seed(5), output_type=t, **KW).frames
    torch.cuda.synchronize()
    assert [(p.dtype, p.device, p.requires_grad, p.data_ptr(), p._version) for m in (unet, vae, enc) for p in m.parameters()] == state
    assert unet.training
    i2v = ImageToVideoPipeline(unet, vae, enc, image_mean=pipe.image_mean, image_std=pipe.image_std)
    kw = {k: v for k, v in KW.items() if k not in ("height", "width")}
    ref = i2v(image, generator=torch.Generator(DEV).manual_seed(5), **kw).frames
    ref2 = i2v(image, generator=torch.Generator(DEV).manual_seed(5), **kw).frames
    assert out["pt"].shape == (1, 4, 3, 32, 32) and out["pt"].dtype == torch.float32
    _agree(out["pt"], ref, ref2, "pt vs ImageToVideoPipeline")
    assert out["latent"].shape == (1, 4, 4, 16, 16)          # the tiny VAE downsamples by 2
    pt_np = postprocess_video(out["pt"], "np")
    assert out["np"].shape == (1, 4, 32, 32, 3) and out["np"].dtype == np.float32
    pil = out["pil"]
    assert len(pil) == 1 and len(pil[0]) == 4 and pil[0][0].size == (32, 32)
    if torch.equal(ref, ref2):
        assert np.array_equal(out["np"], pt_np)
        for f in range(4):
            assert np.array_equal(np.asarray(pil[0][f]), (pt_np[0, f] * 255).round().astype(np.uint8))
    else:
        assert _rel(torch.from_numpy(out["np"]), torch.from_numpy(pt_np)) <= 4 * _rel(ref2, ref)
    frames = pipe(image, generator=torch.Generator(DEV).manual_seed(5), output_type="pt", return_dict=False, **KW)
    assert isinstance(frames, torch.Tensor) and frames.shape == out["pt"].shape


def test_pil_input_of_another_size_against_the_composition_by_hand(tmp_path, monkeypatch):
    from PIL import Image
    from svd_xtend_b200 import pipeline as P
    from svd_xtend_b200.clip import encode_image
    from svd_xtend_b200.sampling import decode_latents
    unet, vae, enc = _models(tmp_path, seed=3)
    pipe = P.StableVideoDiffusionPipeline.from_pretrained(str(tmp_path), unet=unet, vae=vae, image_encoder=enc)
    rng = np.random.default_rng(4)
    pil = Image.fromarray(rng.integers(0, 256, (72, 56, 3), dtype=np.uint8))          # 56 wide, 72 high
    seen = {}
    monkeypatch.setattr(P, "encode_image", lambda m, x, *a: (seen.__setitem__("clip", x.clone()), encode_image(m, x, *a))[1])
    vae_encode = vae.encode
    monkeypatch.setattr(vae, "encode", lambda x, *a, **k: (seen.__setitem__("vae", x.clone()), vae_encode(x, *a, **k))[1])
    got = pipe(pil, generator=torch.Generator(DEV).manual_seed(8), output_type="pt", **KW).frames
    monkeypatch.undo()

    def t(im):
        return torch.from_numpy(np.asarray(im).copy()).permute(2, 0, 1)[None].float().div(255).to(DEV)

    def hand():
        g = torch.Generator(DEV).manual_seed(8)
        with torch.no_grad():
            xc = t(pil) * 2 - 1                                                     # CLIP: the image as given
            xv = t(pil.resize((32, 32), resample=Image.Resampling.LANCZOS)) * 2 - 1   # VAE: Pillow-resized to height x width
            emb = encode_image(enc, xc, pipe.image_mean, pipe.image_std)
            cond = xv + 0.02 * torch.randn(xv.shape, generator=g, device=DEV)
            lat0 = vae.encode(cond).latent_dist.mode()
            noise = torch.randn(1, 4, 4, 16, 16, generator=g, device=DEV)
            lat = pipe.sampler(lat0, emb.unsqueeze(1), num_frames=4, num_inference_steps=3, noise=noise)
            out = (decode_latents(vae, lat, 3) / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4)
            return out, xc, cond
    (ref, xc, cond), (ref2, _, _) = hand(), hand()
    torch.cuda.synchronize()
    # the stage inputs are exact: CLIP got the 72 x 56 original, the VAE the LANCZOS-resized image plus the first draw
    assert seen["clip"].shape == (1, 3, 72, 56) and torch.equal(seen["clip"], xc)
    assert seen["vae"].shape == (1, 3, 32, 32) and torch.equal(seen["vae"], cond)
    _agree(got, ref, ref2, "PIL 72x56 vs hand")


def test_fp16_vae_against_fp32_oracle_and_force_upcast_round_trip():
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as Oracle
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(6)
    oracle = Oracle(**TINY_VAE_CONFIG, with_decoder=True)
    with torch.no_grad():
        for n, p in oracle.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
        for p in oracle.parameters():
            p.copy_(p.half().float())                   # fp16-representable weights: the fp16 model holds them exactly
    oracle = oracle.to(DEV).eval().requires_grad_(False)
    vae16 = AutoencoderKLTemporalDecoder(**TINY_VAE_CONFIG, with_decoder=True)
    vae16.load_state_dict(oracle.state_dict())
    vae16 = vae16.to(DEV).half().requires_grad_(False)
    vae32 = AutoencoderKLTemporalDecoder(**TINY_VAE_CONFIG, with_decoder=True)
    vae32.load_state_dict(oracle.state_dict())
    vae32 = vae32.to(DEV).requires_grad_(False)
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(4, 3, 32, 64, generator=g) * 0.5).clamp(-1, 1).to(DEV)
    z = torch.randn(4, 4, 16, 32, generator=g).to(DEV)
    with torch.no_grad():
        ref_m = oracle.encode(x).latent_dist
        ref_d = oracle.decode(z, num_frames=4).sample
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac_m = oracle.encode(x).latent_dist
            ac_d = oracle.decode(z, num_frames=4).sample
        got_m = vae16.encode(x.half()).latent_dist
        got_d = vae16.decode(z.half(), num_frames=4).sample
    torch.cuda.synchronize()
    assert got_m.mean.dtype == torch.float16 and got_d.dtype == torch.float16
    cat = lambda d: torch.cat([d.mean, d.logvar], 1).float()   # noqa: E731
    for what, got, ref, ac in (("encode", cat(got_m), cat(ref_m), cat(ac_m)), ("decode", got_d, ref_d, ac_d)):
        e, ea = _rel(got.float(), ref), _rel(ac.float(), ref)
        print(f"fp16 VAE {what}: rel-l2 {e:.4g} (torch bf16 autocast {ea:.4g})")
        assert torch.isfinite(got).all() and e <= max(2 * ea, 2e-2), (what, e, ea)
    # diffusers' force_upcast sequence: fp16 -> fp32 for the encode -> fp16 for the decode, on the same module
    with torch.no_grad():
        vae16.to(torch.float32)
        up_m = vae16.encode(x).latent_dist.mode()
        vae16.to(torch.float16)
        up_d = vae16.decode(z, num_frames=4).sample
        r_m, r2_m = vae32.encode(x).latent_dist.mode(), vae32.encode(x).latent_dist.mode()
        r_d, r2_d = vae32.decode(z, num_frames=4).sample, vae32.decode(z, num_frames=4).sample
    torch.cuda.synchronize()
    assert vae16.dtype == torch.float16 and up_m.dtype == up_d.dtype == torch.float32
    _agree(up_m, r_m, r2_m, "upcast encode vs fp32 VAE")
    _agree(up_d, r_d, r2_d, "fp16 decode after the round trip vs fp32 VAE")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_script_per_step_encode_draws_like_torch_randn(dtype):
    """tensor_to_vae_latent (train_svd.py:283-291) with the VAE and the frames in the script's weight dtype: the sample is
    mean + std * torch.randn(shape, dtype) from the global CUDA generator, and leaves that generator where randn would"""
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoderWithDecoder as V
    torch.manual_seed(9)
    vae = V(**TINY_VAE_CONFIG).to(DEV, dtype=dtype).requires_grad_(False)
    t = (torch.rand(2, 3, 3, 32, 32, device=DEV) * 2 - 1).to(dtype)
    dist = vae.encode(t.flatten(0, 1)).latent_dist
    assert dist.mean.dtype == dtype
    torch.cuda.manual_seed(123)
    lat = dist.sample()
    after = torch.randn(8, device=DEV)
    torch.cuda.manual_seed(123)
    noise = torch.randn(dist.mean.shape, device=DEV, dtype=dist.mean.dtype)
    assert torch.equal(lat, dist.mean + dist.std * noise)
    assert torch.equal(after, torch.randn(8, device=DEV))
    scaled = lat.reshape(2, 3, *lat.shape[1:]) * vae.config.scaling_factor
    assert scaled.shape == (2, 3, 4, 16, 16) and torch.isfinite(scaled).all()


@pytest.mark.parametrize("mode", ["ema", "lora"])
def test_validation_between_training_steps(tmp_path, mode):
    """train_svd.py:1093-1157 (and train_svd_lora.py's loop) on a graphed training UNet: (EMA store / copy_to), the pipeline
    built from the training modules under fp16 autocast, (restore), del pipeline, empty_cache -- twice -- then the next step
    and the final save."""
    from PIL import Image
    from oracle.svd_unet_oracle import edm_loss, synthetic_batch, TINY_CONFIG
    from svd_xtend_b200.ema import EMAModel
    from svd_xtend_b200.pipeline import ImageToVideoPipeline, StableVideoDiffusionPipeline
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as U
    unet, vae, enc = _models(tmp_path, seed=11)
    vae.half()
    enc.half()
    unet.train()
    if mode == "ema":
        for n, p in unet.named_parameters():
            p.requires_grad_("temporal_transformer_block" in n)
    else:
        unet.add_adapter(SimpleNamespace(r=4, lora_alpha=4, init_lora_weights="gaussian",
                                         target_modules=["to_k", "to_q", "to_v", "to_out.0"]))
    unet.enable_gradient_checkpointing()
    ema = EMAModel(unet.parameters(), model_cls=U, model_config=unet.config) if mode == "ema" else None
    runner = unet.enable_cuda_graphs(warmup=2)
    arena = unet._arena
    assert arena is not None
    opt = torch.optim.AdamW([p for p in unet.parameters() if p.requires_grad], lr=3e-3, weight_decay=1e-2)
    batch = synthetic_batch(1, 4, 16, 16, seed=41, device=DEV, cross_dim=TINY_CONFIG["cross_attention_dim"])

    def train_step():
        with torch.autocast("cuda", dtype=torch.float16):
            pred = unet(batch["sample"], batch["timestep"], batch["encoder_hidden_states"], batch["added_time_ids"]).sample
        loss = edm_loss(pred.float(), batch["noisy"], batch["latents"], batch["sigmas"])
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        if ema is not None:
            ema.step(unet.parameters())
        return loss
    for _ in range(4):
        train_step()
    torch.cuda.synchronize()
    train_entries = [e for e in runner.entries.values() if e.g_bwd is not None]
    assert len(train_entries) == 1
    image = Image.fromarray(np.random.default_rng(2).integers(0, 256, (40, 48, 3), dtype=np.uint8))
    for _ in range(2):
        masters = [p.detach().clone() for p in unet.parameters()]
        if ema is not None:
            ema.store(unet.parameters())
            ema.copy_to(unet.parameters())
        pipe = StableVideoDiffusionPipeline.from_pretrained(str(tmp_path), unet=unet, image_encoder=enc, vae=vae, revision=None,
                                                            torch_dtype=torch.float16)
        pipe = pipe.to(DEV)
        pipe.set_progress_bar_config(disable=True)
        with torch.autocast("cuda", enabled=True):
            frames = pipe(image.resize((32, 32)), height=32, width=32, num_frames=4, decode_chunk_size=8, motion_bucket_id=127,
                          fps=7, noise_aug_strength=0.02, num_inference_steps=3).frames[0]
        assert len(frames) == 4 and all(np.isfinite(np.asarray(f, dtype=np.float32)).all() for f in frames)
        if ema is not None:
            ema.restore(unet.parameters())
        sampler = weakref.ref(pipe.sampler)
        assert pipe.sampler._graph is not None
        del pipe
        torch.cuda.empty_cache()
        assert sampler() is None, "the pipeline's sampler, and with it its graph and static buffers, outlived the pipeline"
        torch.cuda.synchronize()
        assert unet.training and unet.is_gradient_checkpointing
        for p, b in zip(unet.parameters(), masters):
            assert torch.equal(p, b)
        now = [e for e in runner.entries.values() if e.g_bwd is not None]
        assert len(now) == 1 and now[0] is train_entries[0], "validation dropped the captured training graphs"
        assert len(runner.entries) == 1, "the sampling signature left a graph in the module"
        loss = train_step()
        torch.cuda.synchronize()
        assert torch.isfinite(loss)
        assert [e for e in runner.entries.values() if e.g_bwd is not None][0] is train_entries[0]
    # the final save (train_svd.py:1166-1180), read back by the package's own loader
    pipe = StableVideoDiffusionPipeline.from_pretrained(str(tmp_path), image_encoder=enc, vae=vae, unet=unet, revision=None)
    pipe.save_pretrained(str(tmp_path / "out"))
    if mode == "ema":
        back = ImageToVideoPipeline.from_pretrained(str(tmp_path / "out"))
        for a, b in ((unet, back.unet), (vae, back.vae), (enc, back.image_encoder)):
            sa, sb = a.state_dict(), b.state_dict()
            assert list(sa) == list(sb) and all(torch.equal(sa[k].cpu(), sb[k].to(sa[k].dtype)) for k in sa)
    del pipe
    gc.collect()


def test_diffusers_loads_the_saved_directory(tmp_path):
    diffusers = pytest.importorskip("diffusers")
    from svd_xtend_b200.pipeline import StableVideoDiffusionPipeline
    unet, vae, enc = _models(tmp_path / "src")
    StableVideoDiffusionPipeline.from_pretrained(str(tmp_path / "src"), unet=unet, vae=vae, image_encoder=enc).save_pretrained(
        str(tmp_path / "out"))
    assert os.path.exists(tmp_path / "out" / "model_index.json")
    pipe = diffusers.StableVideoDiffusionPipeline.from_pretrained(str(tmp_path / "out"))
    assert type(pipe.scheduler).__name__ == "EulerDiscreteScheduler"
