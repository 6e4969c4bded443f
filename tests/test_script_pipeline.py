"""The drop-in VAE and StableVideoDiffusionPipeline the unchanged training scripts get from the shim, without a GPU: the shim
installs them under diffusers' names, the VAE's diffusers contract (config keys, forward signature, save / load, local
directories only), the scheduler configurations the sampler accepts, model_index.json, and argument checks that raise before
any launch."""
import importlib
import inspect
import json
import os
import sys
import types

import pytest
import torch

from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
from oracle.svd_unet_oracle import TINY_CONFIG
from oracle.svd_vae_oracle import TINY_VAE_CONFIG

# diffusers' scheduler/scheduler_config.json of the SVD checkpoints [D]
SVD_SCHEDULER = {"_class_name": "EulerDiscreteScheduler", "_diffusers_version": "0.24.0.dev0", "beta_end": 0.012,
                 "beta_schedule": "scaled_linear", "beta_start": 0.00085, "clip_sample": False, "interpolation_type": "linear",
                 "num_train_timesteps": 1000, "prediction_type": "v_prediction", "set_alpha_to_one": False, "sigma_max": 700.0,
                 "sigma_min": 0.002, "skip_prk_steps": True, "steps_offset": 1, "timestep_spacing": "leading",
                 "timestep_type": "continuous", "trained_betas": None, "use_karras_sigmas": True}
# diffusers' vae/config.json of the SVD checkpoints [D]
SVD_VAE_CONFIG_EXTRA = {"_class_name": "AutoencoderKLTemporalDecoder", "_diffusers_version": "0.24.0.dev0",
                        "down_block_types": ["DownEncoderBlock2D"] * 4, "force_upcast": True, "out_channels": 3, "sample_size": 768}


def write_tiny_checkpoint(root, seed=0, unet_cfg=None, vae_cfg=None, clip_cfg=None):
    """a complete local SVD-layout directory at tiny configs: unet/, vae/ (with decoder), image_encoder/, scheduler/,
    feature_extractor/. Returns the three models as written (fp32, CPU)."""
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(seed)
    unet = UNetSpatioTemporalConditionModel(**(unet_cfg or TINY_CONFIG))
    vae = AutoencoderKLTemporalDecoder(**(vae_cfg or TINY_VAE_CONFIG), **SVD_VAE_CONFIG_EXTRA, with_decoder=True)
    enc = CLIPVisionModelWithProjection(**(clip_cfg or dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"])))
    with torch.no_grad():
        for m in (vae, enc):
            for n, p in m.named_parameters():
                if "norm" in n:
                    p.add_(0.1 * torch.randn_like(p))
    unet.save_pretrained(os.path.join(root, "unet"))
    vae.save_pretrained(os.path.join(root, "vae"))
    enc.save_pretrained(os.path.join(root, "image_encoder"))
    os.makedirs(os.path.join(root, "scheduler"), exist_ok=True)
    with open(os.path.join(root, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump(SVD_SCHEDULER, f)
    os.makedirs(os.path.join(root, "feature_extractor"), exist_ok=True)
    with open(os.path.join(root, "feature_extractor", "preprocessor_config.json"), "w") as f:
        json.dump({"image_mean": [0.5, 0.45, 0.4], "image_std": [0.25, 0.26, 0.27], "feature_extractor_type": "CLIPFeatureExtractor"}, f)
    return unet, vae, enc


def test_shim_installs_vae_and_pipeline_under_diffusers_names(monkeypatch):
    from svd_xtend_b200 import shim
    from svd_xtend_b200.pipeline import StableVideoDiffusionPipeline
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder, AutoencoderKLTemporalDecoderWithDecoder
    fake = types.ModuleType("diffusers")
    fake.__path__ = []
    fake.AutoencoderKLTemporalDecoder = fake.StableVideoDiffusionPipeline = object
    pipes = types.ModuleType("diffusers.pipelines")
    pipes.__path__ = []
    monkeypatch.setitem(sys.modules, "diffusers", fake)
    monkeypatch.setitem(sys.modules, "diffusers.pipelines", pipes)
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)
    monkeypatch.setattr(shim, "install_clip", lambda: False)      # keep an installed transformers untouched for later tests
    shim.install(use_8bit_adam=False)
    from diffusers import AutoencoderKLTemporalDecoder as V, StableVideoDiffusionPipeline as P  # noqa: the stand-in
    assert V is AutoencoderKLTemporalDecoderWithDecoder and issubclass(V, AutoencoderKLTemporalDecoder)
    assert P is StableVideoDiffusionPipeline and importlib.import_module("diffusers.pipelines").StableVideoDiffusionPipeline is P
    assert hasattr(P, "save_lora_weights") and shim.install_lora_writer(P) is False      # the drop-in has its own writer
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)


def test_vae_config_keys_survive_save_and_load(tmp_path):
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder, AutoencoderKLTemporalDecoderWithDecoder
    _, vae, _ = write_tiny_checkpoint(str(tmp_path))
    with open(tmp_path / "vae" / "config.json") as f:
        cfg = json.load(f)
    assert cfg["_class_name"] == "AutoencoderKLTemporalDecoder"
    for k, v in SVD_VAE_CONFIG_EXTRA.items():
        assert cfg[k] == v, k
    # the package default stays encoder-only; the shim's class loads the decoder
    enc_only = AutoencoderKLTemporalDecoder.from_pretrained(str(tmp_path), subfolder="vae", revision=None, low_cpu_mem_usage=False)
    assert enc_only.decoder is None
    full = AutoencoderKLTemporalDecoderWithDecoder.from_pretrained(str(tmp_path), subfolder="vae")
    assert full.decoder is not None
    for k in ("force_upcast", "out_channels", "sample_size", "down_block_types", "scaling_factor", "_diffusers_version"):
        assert getattr(full.config, k) == cfg[k], k
    assert full.config.force_upcast is True and full.config["scaling_factor"] == 0.18215
    sd, sd2 = vae.state_dict(), full.state_dict()
    assert list(sd) == list(sd2) and all(torch.equal(sd[k], sd2[k]) for k in sd)
    # a variant file, written and read back with the decoder
    full.save_pretrained(str(tmp_path / "v2"), variant="fp16")
    assert (tmp_path / "v2" / "diffusion_pytorch_model.fp16.safetensors").exists()
    again = AutoencoderKLTemporalDecoder.from_pretrained(str(tmp_path / "v2"), variant="fp16", with_decoder=True)
    assert all(torch.equal(a, b) for a, b in zip(again.state_dict().values(), sd.values()))
    with open(tmp_path / "v2" / "config.json") as f:
        assert json.load(f) == cfg


def test_vae_forward_signature_and_loader_refusals(tmp_path):
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    params = inspect.signature(AutoencoderKLTemporalDecoder.forward).parameters
    assert list(params)[1:] == ["sample", "sample_posterior", "return_dict", "generator", "num_frames"]
    assert params["num_frames"].default == 1 and params["sample_posterior"].default is False
    write_tiny_checkpoint(str(tmp_path))
    with pytest.raises(ValueError, match="revision"):
        AutoencoderKLTemporalDecoder.from_pretrained(str(tmp_path), subfolder="vae", revision="main")
    with pytest.raises(ValueError, match="local directory"):
        AutoencoderKLTemporalDecoder.from_pretrained("stabilityai/stable-video-diffusion-img2vid-xt", subfolder="vae")
    with pytest.raises(ValueError, match="local directory"):
        AutoencoderKLTemporalDecoder.from_pretrained(str(tmp_path / "vae" / "config.json"))
    m = AutoencoderKLTemporalDecoder(**TINY_VAE_CONFIG, with_decoder=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(2, 3, 16, 16), num_frames=2)


def test_scheduler_configs():
    from svd_xtend_b200.pipeline import scheduler_sigma_range
    assert scheduler_sigma_range(SVD_SCHEDULER) == (0.002, 700.0)
    assert scheduler_sigma_range({**SVD_SCHEDULER, "sigma_min": 0.01, "sigma_max": 80}) == (0.01, 80.0)
    assert scheduler_sigma_range({**SVD_SCHEDULER, "final_sigmas_type": "zero", "use_exponential_sigmas": False}) == (0.002, 700.0)
    bad = [("_class_name", "EulerAncestralDiscreteScheduler"), ("prediction_type", "epsilon"), ("use_karras_sigmas", False),
           ("timestep_type", "discrete"), ("timestep_spacing", "trailing"), ("final_sigmas_type", "sigma_min"),
           ("use_beta_sigmas", True), ("rescale_betas_zero_snr", True), ("sigma_min", None), ("sigma_max", "700"),
           ("sigma_min", -1.0), ("sigma_max", float("inf")), ("shift", 1.0)]
    for k, v in bad:
        with pytest.raises(ValueError, match=k):
            scheduler_sigma_range({**SVD_SCHEDULER, k: v})
    for k in ("_class_name", "prediction_type", "use_karras_sigmas", "timestep_type", "sigma_min", "sigma_max"):
        with pytest.raises(ValueError, match=k):
            scheduler_sigma_range({kk: v for kk, v in SVD_SCHEDULER.items() if kk != k})
    with pytest.raises(ValueError, match="sigma_min"):
        scheduler_sigma_range({**SVD_SCHEDULER, "sigma_min": 800.0})


def test_karras_sigmas_take_the_config_range():
    from svd_xtend_b200.sampling import karras_sigmas
    s = karras_sigmas(25, 0.01, 80.0)
    assert torch.allclose(s[[0, 24, 25]], torch.tensor([80.0, 0.01, 0.0]))
    assert torch.equal(karras_sigmas(25), karras_sigmas(25, 0.002, 700.0))


def test_pipeline_from_pretrained_save_and_model_index(tmp_path):
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.pipeline import ImageToVideoPipeline, StableVideoDiffusionPipeline
    src, out = str(tmp_path / "src"), str(tmp_path / "out")
    unet, vae, enc = write_tiny_checkpoint(src)
    with open(os.path.join(src, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump({**SVD_SCHEDULER, "sigma_min": 0.01, "sigma_max": 80.0}, f)
    pipe = StableVideoDiffusionPipeline.from_pretrained(src, revision=None, torch_dtype=torch.float16, variant="fp16")
    assert (pipe.sigma_min, pipe.sigma_max) == (0.01, 80.0)
    assert pipe.image_mean == (0.5, 0.45, 0.4) and pipe.image_std == (0.25, 0.26, 0.27)
    assert pipe.vae.decoder is not None and pipe.unet.dtype == pipe.vae.dtype == pipe.image_encoder.dtype == torch.float16
    assert not any(p.requires_grad for m in (pipe.unet, pipe.vae, pipe.image_encoder) for p in m.parameters())
    pipe.set_progress_bar_config(disable=True)
    pipe.save_pretrained(out)
    with open(os.path.join(out, "model_index.json")) as f:
        index = json.load(f)
    assert index == {"_class_name": "StableVideoDiffusionPipeline", "_diffusers_version": "0.24.0",
                     "feature_extractor": ["transformers", "CLIPImageProcessor"],
                     "image_encoder": ["transformers", "CLIPVisionModelWithProjection"],
                     "scheduler": ["diffusers", "EulerDiscreteScheduler"],
                     "unet": ["diffusers", "UNetSpatioTemporalConditionModel"],
                     "vae": ["diffusers", "AutoencoderKLTemporalDecoder"]}
    for sub, name in (("scheduler", "scheduler_config.json"), ("feature_extractor", "preprocessor_config.json")):
        with open(os.path.join(src, sub, name)) as a, open(os.path.join(out, sub, name)) as b:
            assert a.read() == b.read()
    with open(os.path.join(out, "image_encoder", "config.json")) as f:
        ccfg = json.load(f)
    assert ccfg["model_type"] == "clip_vision_model" and ccfg["architectures"] == ["CLIPVisionModelWithProjection"]
    for cls in (ImageToVideoPipeline, StableVideoDiffusionPipeline):
        back = cls.from_pretrained(out)
        for a, b in ((pipe.unet, back.unet), (pipe.vae, back.vae), (pipe.image_encoder, back.image_encoder)):
            sa, sb = a.state_dict(), b.state_dict()
            assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k].to(sa[k].dtype)) for k in sa)
    enc2 = CLIPVisionModelWithProjection.from_pretrained(out)
    assert all(torch.equal(a, b) for a, b in zip(enc2.state_dict().values(), pipe.image_encoder.state_dict().values()))
    with pytest.raises(ValueError, match="revision"):
        StableVideoDiffusionPipeline.from_pretrained(src, revision="v1")
    with pytest.raises(ValueError, match="local directory"):
        StableVideoDiffusionPipeline.from_pretrained(str(tmp_path / "missing"))


def test_passed_components_are_left_alone_and_bad_calls_raise_before_any_launch(tmp_path, monkeypatch):
    from PIL import Image
    from svd_xtend_b200 import raw
    from svd_xtend_b200.pipeline import StableVideoDiffusionPipeline
    unet, vae, enc = write_tiny_checkpoint(str(tmp_path))
    unet.train()
    for n, p in unet.named_parameters():
        p.requires_grad_("temporal_transformer_block" in n)
    before = [(p.dtype, p.device, p.requires_grad, p.data_ptr()) for m in (unet, vae, enc) for p in m.parameters()]
    pipe = StableVideoDiffusionPipeline.from_pretrained(str(tmp_path), unet=unet, vae=vae, image_encoder=enc, torch_dtype=torch.float16)
    pipe.to("cpu")
    assert pipe.unet is unet and pipe.vae is vae and pipe.image_encoder is enc and unet.training
    assert [(p.dtype, p.device, p.requires_grad, p.data_ptr()) for m in (unet, vae, enc) for p in m.parameters()] == before
    img = Image.new("RGB", (48, 40))
    launches = raw.LAUNCHES[0]
    monkeypatch.setattr(raw, "load", lambda: (_ for _ in ()).throw(AssertionError("a kernel was launched")))
    cases = [dict(num_videos_per_prompt=2), dict(generator=[torch.Generator()]), dict(output_type="gif"),
             dict(callback_on_step_end=print), dict(height=36), dict(decode_chunk_size=0),
             dict(latents=torch.zeros(1, 4, 4, 4, 4), num_frames=4)]
    for kw in cases:
        with pytest.raises(ValueError):
            pipe(img, **{"height": 32, "width": 32, **kw})
    with pytest.raises(ValueError, match="height x width"):
        pipe(torch.rand(1, 3, 40, 48), height=32, width=32)
    with pytest.raises(ValueError, match="RGB"):
        pipe(img.convert("L"), height=32, width=32)
    with pytest.raises(ValueError, match="one size"):
        pipe([img, Image.new("RGB", (32, 32))], height=32, width=32)
    assert raw.LAUNCHES[0] == launches


def test_postprocess_conversions():
    import numpy as np
    from svd_xtend_b200.pipeline import postprocess_video
    torch.manual_seed(0)
    frames = torch.rand(2, 3, 3, 5, 7)
    frames[0, 0, 0, 0, :3] = torch.tensor([0.5 / 255, 1.5 / 255, 1.0])
    assert postprocess_video(frames, "pt") is frames
    arr = postprocess_video(frames, "np")
    assert arr.shape == (2, 3, 5, 7, 3) and arr.dtype == np.float32 and np.array_equal(arr, frames.permute(0, 1, 3, 4, 2).numpy())
    pil = postprocess_video(frames, "pil")
    assert len(pil) == 2 and all(len(v) == 3 for v in pil) and pil[0][0].size == (7, 5) and pil[0][0].mode == "RGB"
    for b in range(2):
        for f in range(3):
            assert np.array_equal(np.asarray(pil[b][f]), (arr[b, f] * 255).round().astype(np.uint8))
