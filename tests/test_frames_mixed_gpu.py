"""Clips of mixed source sizes and crop boxes on the H100 (svd_xtend_b200.video_train.ClipSlots, kernel svdx_frames_u8_in_clips):
one launch over three clips of three sizes against Pillow's recorded outputs bit for bit, the table-driven launch against
svdx_frames_u8_in when every clip has one size, a descriptor that does not fit reading nothing, the encode in frame chunks, and a
graphed VideoTrainStep(max_source_size=...) called with changing sizes and boxes against its eager form and against the float
step fed the oracle's resized frames."""
import os

import numpy as np
import pytest
import torch

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_box_golden.pt")
TINY_VAE = dict(in_channels=3, latent_channels=4, block_out_channels=(64, 64, 128, 128), layers_per_block=1, scaling_factor=0.18215)
bf16 = torch.bfloat16


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _u8(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)


def _oracle_frames(clips, boxes, H, W):
    """list of uint8 [F, H0, W0, 3] -> the oracle's resized, normalised fp32 frames [B, F, 3, H, W] (DummyDataset with boxes)"""
    from oracle.svd_resize_oracle import normalize
    from resize_box_oracle import resize_box
    out = np.stack([np.stack([normalize(resize_box(c[f].cpu().numpy(), (W, H), bx)) for f in range(c.shape[0])])
                    for c, bx in zip(clips, boxes)])
    return torch.from_numpy(out).permute(0, 1, 4, 2, 3).contiguous()


def _fill(slots, eps, sig, first=0, count=None):
    count = slots.B * (slots.F + 1) - first if count is None else count
    rows = torch.full((count * slots.H * slots.W, 64), float("nan"), device=DEV, dtype=bf16)
    x0 = torch.full((slots.B, 3, slots.H, slots.W), float("nan"), device=DEV)
    slots.fill(rows, first, count, eps, sig, x0, 64)
    return rows, x0


def _golden_clips():
    from oracle.svd_resize_oracle import source_frame, unpack_image
    cases = [c for c in torch.load(GOLDEN)["cases"] if c["clip"] >= 0]
    clips, boxes, want = [], [], []
    for b in sorted({c["clip"] for c in cases}):
        cs = [c for c in cases if c["clip"] == b]
        clips.append(torch.stack([source_frame(c["seed"], *c["source"]) for c in cs]))
        boxes.append(cs[0]["box"])
        want.append(np.stack([unpack_image(c["out"], tuple(c["size"]) + (3,)) for c in cs]))
    return clips, boxes, want, tuple(cases[0]["size"])


@pytest.mark.gpu
def test_one_launch_of_three_sizes_matches_pillow():
    """three clips of three source sizes, two with boxes, in one launch: every clip frame's row and every clean first frame
    equal normalize(Pillow's output) bit for bit; the conditioning rows with sigma = 0 as well; a frame range gives the same"""
    from oracle.svd_resize_oracle import normalize
    from svd_xtend_b200.video_train import ClipSlots
    clips, boxes, want, (H, W) = _golden_clips()
    B, F = len(clips), clips[0].shape[0]
    assert B == 3 and len({c.shape for c in clips}) == 3
    slots = ClipSlots(B, F, (H, W), (max(c.shape[1] for c in clips), max(c.shape[2] for c in clips)), DEV)
    slots.load([c.pin_memory() for c in clips], boxes)
    eps, sig = torch.zeros(B, 3, H, W, device=DEV), torch.zeros(B, device=DEV)
    rows, x0 = _fill(slots, eps, sig)
    hw = H * W
    for b in range(B):
        ref = torch.from_numpy(normalize(want[b])).to(DEV)                      # [F, H, W, 3]
        for f in range(F):
            n = b * F + f
            got = rows[n * hw:(n + 1) * hw, :3]
            assert torch.equal(got.view(torch.int16), ref[f].reshape(hw, 3).to(bf16).view(torch.int16)), (b, f)
        assert torch.equal(x0[b].view(torch.int32), ref[0].permute(2, 0, 1).contiguous().view(torch.int32)), b
        n = B * F + b
        assert torch.equal(rows[n * hw:(n + 1) * hw, :3].view(torch.int16), ref[0].reshape(hw, 3).to(bf16).view(torch.int16)), b
    assert torch.equal(rows[:, 3:].float(), torch.zeros_like(rows[:, 3:].float()))
    for first, count in ((0, 1), (2, 3), (5, 4)):
        part, _ = _fill(slots, eps, sig, first, count)
        assert torch.equal(part.view(torch.int16), rows[first * hw:(first + count) * hw].view(torch.int16)), (first, count)


@pytest.mark.gpu
def test_one_size_matches_frames_u8_in():
    """every clip at one size, no boxes: the table-driven launch and svdx_frames_u8_in write the same rows and first frames,
    bit for bit, noise-augmented conditioning frames included"""
    from svd_xtend_b200 import raw
    from svd_xtend_b200.video_train import ClipSlots
    B, F, H0, W0, H, W = 2, 3, 150, 250, 64, 128
    src = _u8((B, F, H0, W0, 3), 3).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    eps = torch.randn(B, 3, H, W, device=DEV, generator=g)
    sig = torch.tensor([0.05, 0.3], device=DEV)
    ty, tx = raw.resize_taps(H0, H).to(DEV), raw.resize_taps(W0, W).to(DEV)
    ref = torch.empty(B * (F + 1) * H * W, 64, device=DEV, dtype=bf16)
    ref_x0 = torch.empty(B, 3, H, W, device=DEV)
    raw.frames_u8_in(src, ty, tx, eps, sig, ref, (H, W), 0, B * (F + 1), ref_x0)
    for cap in ((H0, W0), (200, 300)):                       # a capacity larger than the clips changes nothing
        slots = ClipSlots(B, F, (H, W), cap, DEV)
        slots.load(list(src))
        rows, x0 = _fill(slots, eps, sig)
        assert torch.equal(rows.view(torch.int16), ref.view(torch.int16)), cap
        assert torch.equal(x0.view(torch.int32), ref_x0.view(torch.int32)), cap


@pytest.mark.gpu
def test_descriptor_that_does_not_fit_reads_nothing():
    """a descriptor whose frames lie beyond the source buffer, or whose tap rows lie beyond the tables, gives u = 0 (-1 after
    the normalisation) for its clip, and the other clip is unchanged"""
    from svd_xtend_b200 import raw
    from svd_xtend_b200.video_train import ClipSlots
    B, F, H, W = 2, 2, 64, 128
    slots = ClipSlots(B, F, (H, W), (90, 160), DEV)
    slots.load([_u8((F, 90, 160, 3), 8).to(DEV), _u8((F, 60, 100, 3), 9).to(DEV)])
    eps, sig = torch.zeros(B, 3, H, W, device=DEV), torch.zeros(B, device=DEV)
    good, _ = _fill(slots, eps, sig)
    hw = H * W
    for bad in (raw.clip_descs([0, slots.slots.numel()], [(90, 160), (60, 100)], [0, H], [0, W]),
                raw.clip_descs([0, slots.slot], [(90, 160), (60, 100)], [0, 2 * H], [0, W]),
                raw.clip_descs([0, slots.slot], [(90, 160), (2 ** 30, 2 ** 30)], [0, H], [0, W])):
        slots.descs.copy_(bad)
        rows, _ = _fill(slots, eps, sig)
        for n in (2, 3, 5):                                  # clip 1's frames and its conditioning frame
            assert torch.equal(rows[n * hw:(n + 1) * hw, :3].float(), torch.full((hw, 3), -1.0, device=DEV)), n
        for n in (0, 1, 4):
            assert torch.equal(rows[n * hw:(n + 1) * hw].view(torch.int16), good[n * hw:(n + 1) * hw].view(torch.int16)), n


def _pairs(seed):
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.manual_seed(seed)
    with torch.device(DEV):
        v = AutoencoderKLTemporalDecoder(**TINY_VAE)
        c = CLIPVisionModelWithProjection(**dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"]))
        u = UNetSpatioTemporalConditionModel(**TINY_CONFIG)
    for m in (v, c, u):
        m.eval().requires_grad_(False)
    for n, p in u.named_parameters():
        if "temporal_transformer_block" in n:           # train_svd.py:761-766
            p.requires_grad_(True)
    u.train()
    return v, c, u


# per call: the two clips' source sizes and boxes
CALLS = [
    (((90, 200), None), ((64, 128), None)),
    (((120, 220), (10.5, 3.25, 210.0, 117.75)), ((40, 96), None)),
    (((64, 300), (0, 0, 256, 64)), ((120, 220), (0, 0, 220, 120))),
]


def _calls():
    return [([_u8((2,) + s + (3,), 100 + 10 * i + b) for b, (s, _) in enumerate(c)], [bx for _, bx in c]) for i, c in enumerate(CALLS)]


@pytest.mark.gpu
def test_chunked_encode_matches_one_encode_mixed():
    from svd_xtend_b200.video_train import assemble_train_batch, draw_train_noise
    v, c, u = _pairs(21)
    B, F, H, W = 2, 2, 64, 128
    clips, boxes = _calls()[1]
    clips = [x.to(DEV) for x in clips]
    d = draw_train_noise(B, F, H, W, generator=torch.Generator().manual_seed(9), device=DEV)
    kw = dict(conditioning_dropout_prob=0.1, size=(H, W), boxes=boxes)
    one = [assemble_train_batch(v, c, u, clips, d, **kw) for _ in range(3)]
    spread = max(_rel(one[i]["sample"], one[0]["sample"]) for i in (1, 2))
    for chunk in (1, 4, B * (F + 1)):
        b = assemble_train_batch(v, c, u, clips, d, encode_chunk_size=chunk, **kw)
        e = _rel(b["sample"], one[0]["sample"])
        print(f"mixed encode_chunk_size={chunk}: sample rel-l2 {e:.3e} (two encodes {spread:.3e})")
        assert e <= 4 * spread + 1e-6, chunk
        for k in ("encoder_hidden_states", "timestep", "added_time_ids", "sigmas"):
            assert torch.equal(b[k], one[0][k]), k


def _step(seed, cuda_graph=True, mixed=True, chunk=2):
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    from svd_xtend_b200.video_train import VideoTrainStep
    v, c, u = _pairs(seed)
    arena = ParamArena(u)
    u.attach_arena(arena)
    opt = FusedAdamW(arena, lr=1e-4)
    opt.on_updated = lambda: u.refresh_trainable_operands(shadow_current=True)
    gen = torch.Generator(DEV).manual_seed(123)
    snap = [t.clone() for t in opt.snapshot_tensors()]
    step = VideoTrainStep(u, v, c, opt, frames_shape=(2, 2, 64, 128), conditioning_dropout_prob=0.1, generator=gen,
                          cuda_graph=cuda_graph, max_source_size=(120, 300) if mixed else None, encode_chunk_size=chunk)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(snap, opt.snapshot_tensors())), "construction changed the optimizer state"
    return step, arena


@pytest.mark.gpu
def test_mixed_graphed_step_matches_eager_and_float_step():
    """a graphed max_source_size step called three times with changing sizes and boxes captures once; the rows and CLIP frames
    it reads equal those of assemble_train_batch's eager list form; losses, gradients and weights agree with the eager step and
    with the float step fed the oracle's resized frames within four times the spread of two eager runs"""
    from svd_xtend_b200.video_train import ClipSlots
    torch.backends.cuda.matmul.allow_tf32 = False
    calls = _calls()
    pinned = [([c.pin_memory() for c in clips], boxes) for clips, boxes in calls]
    flt = [_oracle_frames(clips, boxes, 64, 128).to(DEV) for clips, boxes in calls]

    def run(graph, mixed=True):
        step, arena = _step(7, cuda_graph=graph, mixed=mixed)
        graph_obj = step.graphed.graph if graph else None
        losses = []
        for i in range(3):
            losses.append(step(*pinned[i]).item() if mixed else step(flt[i]).item())
            if mixed and graph:
                assert step.graphed.graph is graph_obj
                s = step.static
                cs = log_normal(s["cond_u"])
                got, got_x0 = _fill(s["pixel_values"], s["cond_pixel_eps"], cs)
                fresh = ClipSlots(2, 2, (64, 128), (max(c.shape[1] for c in pinned[i][0]), max(c.shape[2] for c in pinned[i][0])),
                                  DEV)
                fresh.load(pinned[i][0], pinned[i][1])
                want, want_x0 = _fill(fresh, s["cond_pixel_eps"], cs)
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), i
                assert torch.equal(got_x0.view(torch.int32), want_x0.view(torch.int32)), i
                ref = flt[i][:, 0].contiguous()
                assert torch.equal(got_x0.view(torch.int32), ref.view(torch.int32)), i
        torch.cuda.synchronize()
        return losses, arena.grad.clone(), arena.data.clone()

    def log_normal(u):
        from svd_xtend_b200.video_train import log_normal as ln
        return ln(u, -3.0, 0.5)

    l1, g1, p1 = run(False)
    l2, g2, p2 = run(False)
    lg, gg, pg = run(True)
    lf, gf, pf = run(True, mixed=False)
    spread_l = max(abs(a - b) for a, b in zip(l1, l2))
    spread_g, spread_p = _rel(g2, g1), _rel(p2, p1)
    for name, (l, g, p) in (("graphed mixed", (lg, gg, pg)), ("graphed float", (lf, gf, pf))):
        dl = max(abs(a - b) for a, b in zip(l, l1))
        print(f"{name}: losses {l} eager mixed {l1}; loss spread {spread_l:.3e} diff {dl:.3e}; grad spread {spread_g:.3e} diff "
              f"{_rel(g, g1):.3e}; weights spread {spread_p:.3e} diff {_rel(p, p1):.3e}")
        assert all(t == t for t in l)
        assert dl <= 4 * spread_l + 1e-6 * max(map(abs, l1))
        assert _rel(g, g1) <= 4 * spread_g + 1e-6
        assert _rel(p, p1) <= 4 * spread_p + 1e-7


@pytest.mark.gpu
def test_mixed_step_rejects_other_clips():
    step, _ = _step(3, cuda_graph=False)
    ok = [_u8((2, 90, 200, 3), 1), _u8((2, 64, 128, 3), 2)]
    with pytest.raises(TypeError, match="list of 2 uint8 clips"):
        step(torch.zeros(2, 2, 90, 200, 3, device=DEV, dtype=torch.uint8))
    with pytest.raises(TypeError, match="clip 1: dtype"):
        step([ok[0], ok[1].float()])
    with pytest.raises(ValueError, match="list of 2 clips, got 1"):
        step(ok[:1])
    with pytest.raises(ValueError, match="clip 0: frames of 121x200 exceed"):
        step([_u8((2, 121, 200, 3), 1), ok[1]])
    with pytest.raises(ValueError, match="clip 1: 3 frames"):
        step([ok[0], _u8((3, 64, 128, 3), 2)])
    with pytest.raises(ValueError, match="clip 0: .*can't exceed"):
        step(ok, [(0, 0, 201, 90), None])
    loss = step(ok, [None, (1.5, 0, 128, 63)]).item()
    assert loss == loss and abs(loss) < float("inf")
