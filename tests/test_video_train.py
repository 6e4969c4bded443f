"""Training from video frames, without a GPU: the oracle of the batch assembly (oracle/svd_train_batch_oracle.py) against the
reference's own step body (tests/golden/train_batch_golden.pt, made by tests/golden/make_train_batch_golden.py), the draw
contract of svd_xtend_b200.video_train.draw_train_noise, and the input checks of assemble_train_batch."""
import os

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_batch_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _close(a, b, what, tol=1e-12):
    a, b = a.double(), b.double()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if a.numel() == 0:
        return
    err = (a - b).abs().max().item()
    assert err <= tol * max(1.0, b.abs().max().item()), (what, err)


def _draws(case):
    return {name: v for name, _, v in case["draws"]}


def test_golden_covers_the_dropout_regions_and_boundaries(golden):
    from oracle.svd_train_batch_oracle import dropout_masks
    seen = set()
    for c in golden["cases"]:
        if c["p"] is None:
            continue
        r = _draws(c)["dropout_u"]
        prompt, image = dropout_masks(r, c["p"])
        seen.add((bool(prompt[0]), float(image[0])))
    assert seen == {(True, 1.0), (True, 0.0), (False, 0.0), (False, 1.0)}
    at = {c["name"]: _draws(c)["dropout_u"][0].item() for c in golden["cases"] if c["name"].startswith("at_")}
    f32 = lambda v: torch.tensor(v, dtype=torch.float32).item()      # noqa: E731
    assert at == {"at_p": f32(0.1), "at_2p": f32(0.2), "at_3p": f32(0.1 * 3)}


@pytest.mark.parametrize("name", ["drop_prompt", "drop_both", "drop_image", "drop_none", "at_p", "at_2p", "at_3p", "no_dropout",
                                  "natural", "batch2"])
def test_oracle_reproduces_reference_step(golden, name):
    from oracle.svd_train_batch_oracle import edm_loss, frames_in, log_normal, train_batch
    c = next(c for c in golden["cases"] if c["name"] == name)
    d = _draws(c)
    B, F = c["B"], c["F"]
    b = train_batch(c["clip_moments"], c["cond_moments"], c["image_embeds"], d, scaling_factor=golden["scaling_factor"],
                    conditioning_dropout_prob=c["p"])
    for k, ref in (("sample", c["sample"]), ("latents", c["latents"]), ("noisy", c["noisy"]), ("sigmas", c["sigmas"])):
        _close(b[k], ref, k)
    _close(b["timestep"], c["timestep"].reshape(B), "timestep")
    _close(b["encoder_hidden_states"], c["encoder_hidden_states"].reshape(B, 1, -1), "encoder_hidden_states")
    # the reference carries clip 0's conditioning sigma in every clip's time ids (:955); here each clip has its own
    _close(b["added_time_ids"][:1], c["added_time_ids"][:1], "added_time_ids")
    _close(b["added_time_ids"][1:, :2], c["added_time_ids"][1:, :2], "added_time_ids")
    if B > 1:
        assert not torch.equal(b["added_time_ids"][1:, 2], c["added_time_ids"][1:, 2])
        _close(b["added_time_ids"][:, 2], log_normal(d["cond_u"], -3.0, 0.5).double(), "per-clip sigma_c")
    # the VAE's inputs: the clip frames, then the noise-augmented conditioning frames
    x = frames_in(c["pixel_values"], d["cond_pixel_eps"].double(), log_normal(d["cond_u"], -3.0, 0.5).double())
    _close(x[:B * F], c["clip_frames"], "clip frames")
    _close(x[B * F:], c["cond_frames"], "conditioning frames")
    # the loss (fp32, as the reference computes it) and its gradient with respect to the prediction
    pred = c["model_pred"].clone().requires_grad_(True)
    loss = edm_loss(pred, b["noisy"], b["latents"], b["sigmas"])
    loss.backward()
    _close(loss, c["loss"], "loss")
    _close(pred.grad, c["dloss_dpred"], "dloss/dpred")


def test_draw_sequence_matches_reference_order(golden):
    from svd_xtend_b200.video_train import DRAWS, draw_train_noise
    for c in golden["cases"]:
        got = draw_train_noise(c["B"], c["F"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]), device="cpu",
                               conditioning_dropout=c["p"] is not None)
        assert list(got) == [n for n, _, _ in c["draws"]] == [n for n, _ in DRAWS if c["p"] is not None or n != "dropout_u"]
        for name, shape, v in c["draws"]:
            # the reference draws the conditioning-frame noise as [B, 1, 3, H, W] (randn_like of frame 0 kept as a clip)
            assert got[name].shape == tuple(s for i, s in enumerate(shape) if not (name == "cond_pixel_eps" and i == 1)), name
            assert got[name].dtype == torch.float32
            if name not in c["replaced"]:
                assert torch.equal(got[name], v.reshape(got[name].shape)), (c["name"], name)


def test_draws_equal_sequential_torch_draws():
    from svd_xtend_b200.video_train import DRAWS, draw_shapes, draw_train_noise
    got = draw_train_noise(2, 3, 64, 128, generator=torch.Generator().manual_seed(7), device="cpu")
    g = torch.Generator().manual_seed(7)
    for (name, kind), (name2, shape) in zip(DRAWS, draw_shapes(2, 3, 64, 128).items()):
        assert name == name2
        assert torch.equal(got[name], getattr(torch, kind)(shape, generator=g))
    assert draw_shapes(2, 3, 64, 128)["latent_eps"] == (6, 4, 8, 16)
    assert "dropout_u" not in draw_train_noise(1, 2, 64, 64, generator=torch.Generator(), device="cpu", conditioning_dropout=False)


def _models(vae_blocks=(32, 32, 32, 32), proj=64, add_dim=32):
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from oracle.svd_unet_oracle import TINY_CONFIG
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    vae = AutoencoderKLTemporalDecoder(**dict(TINY_VAE_CONFIG, block_out_channels=vae_blocks)).requires_grad_(False)
    clip = CLIPVisionModelWithProjection(**dict(TINY_CLIP_CONFIG, projection_dim=proj)).requires_grad_(False)
    unet = UNetSpatioTemporalConditionModel(**dict(TINY_CONFIG, addition_time_embed_dim=add_dim))
    return vae, clip, unet


def test_assemble_checks_inputs_before_any_launch(monkeypatch):
    from svd_xtend_b200 import raw
    from svd_xtend_b200.video_train import assemble_train_batch, draw_train_noise

    def no_launch(*a, **k):
        raise AssertionError("launched")
    for name in ("vae_frames_in", "edm_prepare", "nchw_to_nhwc", "tapgemm", "clip_preprocess"):
        monkeypatch.setattr(raw, name, no_launch)
    vae, clip, unet = _models()
    x = torch.zeros(1, 2, 3, 64, 128)
    d = draw_train_noise(1, 2, 64, 128, generator=torch.Generator(), device="cpu")
    kw = dict(conditioning_dropout_prob=0.1)
    with pytest.raises(ValueError, match="multiples of 64"):
        assemble_train_batch(vae, clip, unet, torch.zeros(1, 2, 3, 64, 96), d, **kw)
    with pytest.raises(TypeError, match="float16"):
        assemble_train_batch(vae, clip, unet, x.half(), d, **kw)
    with pytest.raises(ValueError, match="in_channels"):
        assemble_train_batch(vae, clip, unet.config.__class__(**dict(unet.config.to_dict(), in_channels=6)), x, d, **kw)
    bad_clip = _models(proj=96)[1]
    with pytest.raises(ValueError, match="projection_dim"):
        assemble_train_batch(vae, bad_clip, unet, x, d, **kw)
    bad_unet = _models(add_dim=16)[2]
    with pytest.raises(ValueError, match="added time embedding"):
        assemble_train_batch(vae, clip, bad_unet, x, d, **kw)
    with pytest.raises(ValueError, match="dropout_u"):
        assemble_train_batch(vae, clip, unet, x, {k: v for k, v in d.items() if k != "dropout_u"}, **kw)
    with pytest.raises(ValueError, match="downsample by 8"):
        assemble_train_batch(_models(vae_blocks=(32, 32))[0], clip, unet, x, d, **kw)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        assemble_train_batch(vae, clip, unet, x, d, **kw)
