"""Clips of mixed source sizes and crop boxes (no GPU): the crop-box resize oracle (tests/resize_box_oracle.py) against Pillow's
recorded outputs (tests/golden/resize_box_golden.pt) bit for bit, the library's box taps against the oracle's and, for the box
[0, in), against the taps of the no-box form, the argument checks of the mixed-size form, which fire before any launch, and
FrameFolderClips' clip selection against the reference's DummyDataset (tests/golden/frame_folder_golden.pt)."""
import os
import random

import numpy as np
import pytest
import torch

from oracle.svd_resize_oracle import source_frame, taps, unpack_image
from resize_box_oracle import resize_box, taps_box

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_box_golden.pt")
FOLDERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frame_folder_golden.pt")


def _golden():
    return torch.load(GOLDEN)["cases"]


@pytest.mark.parametrize("i", range(14))
def test_box_oracle_matches_pillow_golden(i):
    c = _golden()[i]
    (H0, W0), (H, W) = c["source"], c["size"]
    got = resize_box(source_frame(c["seed"], H0, W0).numpy(), (W, H), c["box"])
    assert got.dtype == np.uint8 and got.shape == (H, W, 3)
    assert np.array_equal(got, unpack_image(c["out"], (H, W, 3))), c["name"]


def test_box_golden_covers_the_cases():
    cases = _golden()
    assert len(cases) == 14 and os.path.getsize(GOLDEN) < 256 * 1024
    clips = {}
    for c in cases:
        if c["clip"] >= 0:
            clips.setdefault(c["clip"], []).append(c)
    assert sorted(clips) == [0, 1, 2] and all(len(v) == 2 for v in clips.values())
    assert len({tuple(v[0]["source"]) for v in clips.values()}) == 3                  # three source sizes, one target size
    assert len({tuple(c["size"]) for v in clips.values() for c in v}) == 1
    boxed = [(c["source"], c["size"], c["box"]) for c in cases if c["box"] is not None]
    assert any(s[0] < d[0] for s, d, _ in boxed) and any(s[0] > d[0] for s, d, _ in boxed)          # up and down
    assert any(b[0] % 1 or b[1] % 1 for _, _, b in boxed)                                          # fractional offsets
    assert any(b == [0, 0, s[1], s[0]] for s, _, b in boxed)                                       # the box equal to the frame
    assert any(s[0] == d[0] and b[1] % 1 for s, d, b in boxed)                                     # kept side, fractional box
    assert any(s[0] == d[0] and b[1] == 0 and b[3] != s[0] for s, d, b in boxed)                   # kept side, zero offset
    assert any(c["box"] is None and c["source"][0] == c["size"][0] for c in cases)                 # one axis only


def test_box_oracle_matches_pillow_random():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(17)
    for t in range(60):
        H0, W0, H, W = (int(v) for v in rng.integers(1, 90, 4))
        img = rng.integers(0, 256, (H0, W0, 3), dtype=np.uint8)
        if t % 3 == 0:
            box = (float(rng.uniform(0, W0 / 2)), float(rng.uniform(0, H0 / 2)), float(rng.uniform(W0 / 2, W0)),
                   float(rng.uniform(H0 / 2, H0)))
        elif t % 3 == 1:
            x0, y0 = int(rng.integers(0, W0)), int(rng.integers(0, H0))
            box = (x0, y0, int(rng.integers(x0, W0 + 1)), int(rng.integers(y0, H0 + 1)))
        else:
            H, box = H0, (0, float(rng.choice([0.0, 0.25, 1.0])), W0, H0)                          # the height kept
        want = np.asarray(Image.fromarray(img).resize((W, H), box=box))
        assert np.array_equal(resize_box(img, (W, H), box), want), ((H0, W0), (H, W), box)


@pytest.mark.parametrize("n_in,n_out", [(640, 512), (333, 128), (96, 96), (7, 300)])
def test_full_box_oracle_taps_are_the_no_box_taps(n_in, n_out):
    for a, b in zip(taps_box(n_in, n_out, 0, n_in), taps(n_in, n_out)):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("n_in,n_out,box", [(640, 512, (0, 640)), (640, 128, (17.3, 600.9)), (96, 96, (0.5, 96)),
                                            (96, 96, (0, 90)), (40, 128, (3.5, 39.25)), (300, 64, (22, 278)), (5, 9, (2, 2)),
                                            (1920, 1024, (0, 1920)), (1080, 576, (60, 1020))])
def test_library_box_taps_match_oracle(n_in, n_out, box):
    from svd_xtend_b200 import build, raw
    build.build()
    t = raw.resize_taps(n_in, n_out, box).numpy()
    lo, cnt, k = taps_box(n_in, n_out, *box)
    assert t.shape == (n_out, 2 + k.shape[1])
    assert np.array_equal(t[:, 0], lo) and np.array_equal(t[:, 1], cnt) and np.array_equal(t[:, 2:], k)
    if box == (0, n_in):
        assert np.array_equal(t, raw.resize_taps(n_in, n_out).numpy())


def test_library_box_taps_reject_bad_boxes():
    from svd_xtend_b200 import build, raw
    build.build()
    for box in ((-1, 5), (0, 11), (6, 5), (float("nan"), 5)):
        with pytest.raises(ValueError, match="box"):
            raw.resize_taps(10, 4, box)
    lib = raw.load()
    assert lib.svdx_resize_taps_box_ksize(10, 4, 6.0, 5.0) < 0
    assert lib.svdx_resize_taps_box(10, 4, 0.0, 10.5, None) < 0


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


def test_mixed_argument_checks_before_any_launch(monkeypatch):
    from svd_xtend_b200 import raw
    from svd_xtend_b200.video_train import VideoTrainStep, assemble_train_batch, check_clips, draw_train_noise

    def no_launch(*a, **k):
        raise AssertionError("launched before the checks")
    for name in ("frames_u8_in", "frames_u8_in_clips", "vae_frames_in", "vae_frames_in_range", "edm_prepare", "nchw_to_nhwc",
                 "tapgemm", "clip_preprocess", "resize_taps", "clip_descs"):
        monkeypatch.setattr(raw, name, no_launch)
    vae, clip, unet = _models()
    d = draw_train_noise(2, 2, 64, 128, generator=torch.Generator(), device="cpu")
    kw = dict(conditioning_dropout_prob=0.1, size=(64, 128))
    u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8)         # noqa: E731
    good = [u8(2, 90, 160, 3), u8(2, 40, 96, 3)]

    def rejects(exc, match, clips, boxes=None):
        with pytest.raises(exc, match=match):
            assemble_train_batch(vae, clip, unet, clips, d, boxes=boxes, **kw)
    rejects(TypeError, "clip 1: dtype torch.float32", [good[0], torch.zeros(2, 40, 96, 3)])
    rejects(ValueError, "clip 1: 3 frames, expected 2", [good[0], u8(3, 40, 96, 3)])
    rejects(ValueError, "clip 0: .*3 channels", [u8(2, 90, 160, 4), good[1]])
    rejects(ValueError, "clip 1: .*3 channels", [good[0], u8(40, 96, 3)])
    rejects(ValueError, "clip 1: .*offset can't be negative", good, [None, (-0.5, 0, 10, 10)])
    rejects(ValueError, "clip 0: .*can't exceed", good, [(0, 0, 160.5, 90), None])
    rejects(ValueError, "clip 1: .*can't be empty", good, [None, (10, 5, 9, 20)])
    rejects(ValueError, "clip 1: .*finite", good, [None, (0, 0, float("inf"), 20)])
    rejects(ValueError, "one entry .* per clip", good, [None])
    rejects(ValueError, "latent_eps", good + [u8(2, 30, 30, 3)])                 # three clips for draws of two
    with pytest.raises(ValueError, match="boxes are taken with a list"):
        assemble_train_batch(vae, clip, unet, u8(2, 2, 90, 160, 3), d, boxes=[None, None], **kw)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        assemble_train_batch(vae, clip, unet, good, d, boxes=[None, (0, 0, 96, 40)], **kw)
    # the checks a step built with max_source_size=(90, 160) and B = 2, F = 2 runs (ClipSlots.check)
    with pytest.raises(ValueError, match="list of 2 clips, got 3"):
        check_clips(good + [good[1]], (64, 128), B=2, F=2, capacity=(90, 160))
    with pytest.raises(ValueError, match="clip 1: 3 frames, expected 2"):
        check_clips([good[0], u8(3, 40, 96, 3)], (64, 128), B=2, F=2, capacity=(90, 160))
    with pytest.raises(ValueError, match="clip 1: frames of 40x170 exceed the step's max_source_size 90x160"):
        check_clips([good[0], u8(2, 40, 170, 3)], (64, 128), B=2, F=2, capacity=(90, 160))
    assert check_clips(good, (64, 128), [None, (0.5, 1, 96, 40)], B=2, F=2, capacity=(90, 160))[4] == [None, (0.5, 1.0, 96.0, 40.0)]
    with pytest.raises(ValueError, match="mutually exclusive"):
        VideoTrainStep(unet, vae, clip, None, frames_shape=(2, 2, 64, 128), source_size=(90, 160), max_source_size=(90, 160))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        VideoTrainStep(unet, vae, clip, None, frames_shape=(2, 2, 64, 128), max_source_size=(90, 160))


def test_raw_clips_argument_checks(monkeypatch):
    from svd_xtend_b200 import raw
    monkeypatch.setattr(raw, "load", lambda: (_ for _ in ()).throw(AssertionError("reached the library")))
    B, F, H, W = 2, 2, 64, 128
    src = torch.zeros(1000, dtype=torch.uint8)
    descs = torch.zeros(B, 3, dtype=torch.int64)
    ty, tx = torch.zeros(B * H, 9, dtype=torch.int32), torch.zeros(B * W, 9, dtype=torch.int32)
    eps, sig = torch.zeros(B, 3, H, W), torch.zeros(B)
    rows = torch.zeros(3 * H * W, 64, dtype=torch.bfloat16)
    args = lambda **o: [o.get(k, v) for k, v in (("src", src), ("descs", descs), ("ty", ty), ("tx", tx), ("eps", eps),   # noqa: E731
                                                  ("sig", sig), ("rows", rows))]
    with pytest.raises(TypeError, match="uint8"):
        raw.frames_u8_in_clips(*args(src=src.float()), (H, W), F, 0, 3)
    with pytest.raises(ValueError, match="descs"):
        raw.frames_u8_in_clips(*args(descs=descs.int()), (H, W), F, 0, 3)
    with pytest.raises(ValueError, match="taps_x"):
        raw.frames_u8_in_clips(*args(tx=tx[:W - 1]), (H, W), F, 0, 3)
    with pytest.raises(ValueError, match="frames \\[5, 8\\)"):
        raw.frames_u8_in_clips(*args(), (H, W), F, 5, 3)
    with pytest.raises(ValueError, match="dst"):
        raw.frames_u8_in_clips(*args(rows=rows[:-1]), (H, W), F, 0, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        raw.frames_u8_in_clips(*args(), (H, W), F, 0, 3)


def test_clip_descs_layout():
    from svd_xtend_b200 import raw
    d = raw.clip_descs([0, 3 << 33], [(90, 160), (40, 96)], [0, 64], [0, 128])
    assert d.dtype == torch.int64 and d.shape == (2, 3)
    w = d.view(torch.int32).view(2, 6)
    assert d[1, 0] == 3 << 33 and w[0, 2:].tolist() == [90, 160, 0, 0] and w[1, 2:].tolist() == [40, 96, 64, 128]


def test_frame_folder_selection_matches_reference(monkeypatch):
    from svd_xtend_b200.video_train import FrameFolderClips
    g = torch.load(FOLDERS)
    base, tree = g["base"], g["tree"]
    monkeypatch.setattr(os, "listdir", lambda p: list(g["order"]) if p == base else list(tree[os.path.relpath(p, base)]))
    ds = FrameFolderClips(base, g["sample_frames"])
    assert len(ds) == 100000
    state = random.getstate()
    try:
        random.seed(g["seed"])
        for i, want in enumerate(g["picks"]):
            if "error" in want:
                with pytest.raises(ValueError) as e:
                    ds.select()
                assert str(e.value) == want["error"], i
            else:
                assert ds.select() == (want["folder"], want["frames"]), i
    finally:
        random.setstate(state)
    assert sum("error" in p for p in g["picks"]) >= 1 and len({p.get("folder") for p in g["picks"]}) >= 4


def test_frame_folder_decodes_native_size_and_rejects(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    from svd_xtend_b200.video_train import FrameFolderClips
    rng = np.random.default_rng(3)
    frames = {"a": [rng.integers(0, 256, (12, 20, 3), dtype=np.uint8) for _ in range(3)]}
    for name, fr in frames.items():
        (tmp_path / name).mkdir()
        for i, f in enumerate(fr):
            Image.fromarray(f).save(tmp_path / name / f"{i}.png")
    ds = FrameFolderClips(str(tmp_path), 3)
    random.seed(0)
    item = ds[0]
    assert item["size"] == (12, 20) and item["pixel_values"].dtype == torch.uint8
    assert np.array_equal(item["pixel_values"].numpy(), np.stack(frames["a"]))
    batch = FrameFolderClips.collate([item, item])
    assert isinstance(batch, list) and len(batch) == 2 and batch[0].shape == (3, 12, 20, 3)
    Image.fromarray(frames["a"][0][:, :10]).save(tmp_path / "a" / "1.png")
    with pytest.raises(ValueError, match="1.png: frame of 12x10"):
        ds[0]
    Image.fromarray(frames["a"][0][..., 0]).save(tmp_path / "a" / "1.png")
    with pytest.raises(ValueError, match="1.png: frame mode L"):
        ds[0]
