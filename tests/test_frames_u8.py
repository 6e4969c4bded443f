"""Decoded uint8 frames for training (no GPU): the numpy restatement of Pillow's BICUBIC resize (oracle/svd_resize_oracle.py)
against Pillow's recorded outputs (tests/golden/resize_golden.pt) bit for bit, the library's host-side resize taps against the
oracle's, DummyDataset's normalisation, and the argument checks of the uint8 form, which fire before any launch."""
import os

import numpy as np
import pytest
import torch

from oracle.svd_resize_oracle import normalize, pack_image, resize, source_frame, taps, unpack_image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_golden.pt")


def _golden():
    g = torch.load(GOLDEN)
    return [(c, source_frame(c["seed"], *c["source"]).numpy()) for c in g["cases"]]


@pytest.mark.parametrize("i", range(7))
def test_oracle_matches_pillow_golden(i):
    c, src = _golden()[i]
    H, W = c["size"]
    got = resize(src, (W, H))
    assert got.dtype == np.uint8 and got.shape == (H, W, 3)
    assert np.array_equal(got, unpack_image(c["out"], (H, W, 3))), c["name"]


def test_golden_covers_the_cases():
    names = [c["name"] for c, _ in _golden()]
    assert len(names) == 7
    for c, src in _golden():
        (H0, W0), (H, W) = c["source"], c["size"]
        assert src.shape == (H0, W0, 3)
    sizes = {(tuple(c["source"]), tuple(c["size"])) for c, _ in _golden()}
    assert os.path.getsize(GOLDEN) < 256 * 1024
    assert ((360, 640), (320, 512)) in sizes and ((187, 333), (64, 128)) in sizes and ((144, 256), (320, 512)) in sizes
    assert any(s[0] == d[0] and s[1] != d[1] for s, d in sizes) and any(s[1] == d[1] and s[0] != d[0] for s, d in sizes)
    assert any(s == d for s, d in sizes)


def test_oracle_matches_pillow_random_sizes():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(11)
    sizes = [((1080, 1920), (576, 1024)), ((5, 3), (17, 200)), ((37, 1000), (401, 7))]
    sizes += [((int(rng.integers(1, 400)), int(rng.integers(1, 400))), (int(rng.integers(1, 400)), int(rng.integers(1, 400))))
              for _ in range(12)]
    for (H0, W0), (H, W) in sizes:
        img = rng.integers(0, 256, (H0, W0, 3), dtype=np.uint8)
        want = np.asarray(Image.fromarray(img).resize((W, H)))
        assert np.array_equal(resize(img, (W, H)), want), ((H0, W0), (H, W))


@pytest.mark.parametrize("n_in,n_out", [(640, 512), (333, 128), (144, 320), (1920, 1024), (1080, 576), (96, 96), (7, 300), (3000, 5)])
def test_library_taps_match_oracle(n_in, n_out):
    from svd_xtend_b200 import build, raw
    build.build()
    t = raw.resize_taps(n_in, n_out).numpy()
    lo, cnt, k = taps(n_in, n_out)
    assert t.shape == (n_out, 2 + k.shape[1])
    assert np.array_equal(t[:, 0], lo) and np.array_equal(t[:, 1], cnt) and np.array_equal(t[:, 2:], k)
    # every row sums to one in 22-bit fixed point up to the rounding of each tap
    assert np.all(np.abs(k.sum(1) - (1 << 22)) <= k.shape[1])


def test_source_frames_and_packing():
    a, b = source_frame(3, 144, 256), source_frame(3, 144, 256)
    assert a.dtype == torch.uint8 and a.shape == (144, 256, 3) and torch.equal(a, b)
    assert not torch.equal(a, source_frame(4, 144, 256))
    v = a.numpy()
    assert (v == 0).any() and (v == 255).any() and len(np.unique(v)) == 256
    img = np.random.default_rng(2).integers(0, 256, (7, 9, 3), dtype=np.uint8)
    for im in (v, img):
        assert np.array_equal(unpack_image(pack_image(im), im.shape), im)


def test_identity_taps_are_exact():
    lo, cnt, k = taps(64, 64)
    img = np.random.default_rng(1).integers(0, 256, (64, 64, 3), dtype=np.uint8)
    from oracle.svd_resize_oracle import _pass
    assert np.array_equal(_pass(img, 64, 1), img) and np.array_equal(_pass(img, 64, 0), img)


def test_normalize_is_dummy_dataset():
    u = np.arange(256, dtype=np.uint8)
    want = (torch.from_numpy(u.copy()).float() / 127.5 - 1).numpy()
    got = normalize(u)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32))
    assert got[0] == -1.0 and got[255] == 1.0
    # a division, not a multiplication by the fp32 reciprocal: the two differ for some u
    recip = (u.astype(np.float32) * np.float32(1 / 127.5)) - np.float32(1)
    assert not np.array_equal(recip, got)


def _models():
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    vae = AutoencoderKLTemporalDecoder(in_channels=3, latent_channels=4, block_out_channels=(64, 64, 128, 128), layers_per_block=1)
    clip = CLIPVisionModelWithProjection(**dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"]))
    unet = UNetSpatioTemporalConditionModel(**TINY_CONFIG)
    return vae, clip, unet


def test_u8_argument_checks_before_any_launch(monkeypatch):
    from svd_xtend_b200 import raw
    from svd_xtend_b200.video_train import VideoTrainStep, assemble_train_batch, draw_train_noise

    def no_launch(*a, **k):
        raise AssertionError("launched before the checks")
    for name in ("frames_u8_in", "vae_frames_in", "vae_frames_in_range", "edm_prepare", "nchw_to_nhwc", "tapgemm", "clip_preprocess",
                 "resize_taps"):
        monkeypatch.setattr(raw, name, no_launch)
    vae, clip, unet = _models()
    d = draw_train_noise(1, 2, 64, 128, generator=torch.Generator(), device="cpu")
    kw = dict(conditioning_dropout_prob=0.1)
    x = torch.zeros(1, 2, 90, 160, 3, dtype=torch.uint8)
    with pytest.raises(TypeError, match="size"):
        assemble_train_batch(vae, clip, unet, x, d, **kw)
    with pytest.raises(ValueError, match="HWC"):
        assemble_train_batch(vae, clip, unet, torch.zeros(1, 2, 90, 160, 4, dtype=torch.uint8), d, size=(64, 128), **kw)
    with pytest.raises(ValueError, match="HWC"):
        assemble_train_batch(vae, clip, unet, torch.zeros(2, 90, 160, 3, dtype=torch.uint8), d, size=(64, 128), **kw)
    with pytest.raises(ValueError, match="multiples of 64"):
        assemble_train_batch(vae, clip, unet, x, d, size=(64, 96), **kw)
    with pytest.raises(ValueError, match="latent_eps"):
        assemble_train_batch(vae, clip, unet, x, d, size=(128, 128), **kw)
    with pytest.raises(ValueError, match="encode_chunk_size"):
        assemble_train_batch(vae, clip, unet, x, d, size=(64, 128), encode_chunk_size=0, **kw)
    with pytest.raises(ValueError, match="size="):
        assemble_train_batch(vae, clip, unet, torch.zeros(1, 2, 3, 64, 128), d, size=(128, 128), **kw)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        assemble_train_batch(vae, clip, unet, x, d, size=(64, 128), encode_chunk_size=2, **kw)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        VideoTrainStep(unet, vae, clip, None, frames_shape=(1, 2, 64, 128), source_size=(90, 160))


def test_raw_u8_argument_checks(monkeypatch):
    from svd_xtend_b200 import raw
    monkeypatch.setattr(raw, "load", lambda: (_ for _ in ()).throw(AssertionError("reached the library")))
    B, F, H, W = 1, 2, 64, 128
    src = torch.zeros(B, F, 90, 160, 3, dtype=torch.uint8)
    ty, tx = torch.zeros(H, 9, dtype=torch.int32), torch.zeros(W, 9, dtype=torch.int32)
    eps, sig = torch.zeros(B, 3, H, W), torch.zeros(B)
    rows = torch.zeros(3 * H * W, 64, dtype=torch.bfloat16)
    with pytest.raises(TypeError, match="uint8"):
        raw.frames_u8_in(src.float(), ty, tx, eps, sig, rows, (H, W), 0, 3)
    with pytest.raises(ValueError, match="frames \\[2, 5\\)"):
        raw.frames_u8_in(src, ty, tx, eps, sig, rows, (H, W), 2, 3)
    with pytest.raises(ValueError, match="taps_x"):
        raw.frames_u8_in(src, ty, ty, eps, sig, rows, (H, W), 0, 3)
    with pytest.raises(ValueError, match="dst"):
        raw.frames_u8_in(src, ty, tx, eps, sig, rows[:-1], (H, W), 0, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        raw.frames_u8_in(src, ty, tx, eps, sig, rows, (H, W), 0, 3)
    x = torch.zeros(B, F, 3, H, W)
    with pytest.raises(ValueError, match="not within"):
        raw.vae_frames_in_range(x, eps, sig, rows, 1, 3)
