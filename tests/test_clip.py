"""CLIP image encoder (transformers' CLIPVisionModelWithProjection, the SVD `image_encoder/`) on the H100 path against the
oracle restatement (oracle/svd_clip_oracle.py), which tests/golden/clip_golden.pt pins to transformers and to the reference's
own `_resize_with_antialiasing`; the three kernels it adds (svdx_clip_preprocess, the activation epilogue of svdx_tapgemm,
svdx_attention_hd80_fwd) and the host logic around them. Encoder tolerance as for the VAE: rel-L2 <= max(2 x err(oracle under
torch bf16 autocast), 2e-2) against the fp32 oracle."""
import ctypes
import json
import os

import pytest
import torch
import torch.nn.functional as F

DEV = "cuda:0"
bf16 = torch.bfloat16
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clip_golden.pt")


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _golden():
    return torch.load(GOLDEN, weights_only=False)


# ----------------------------------------------------------------------------------------------------------- CPU
def test_state_dict_contract_and_census():
    from oracle.svd_clip_oracle import CLIP_CONFIG, CLIPVisionModelWithProjection as Oracle
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection as Ours
    with torch.device("meta"):
        a, b = Ours(**CLIP_CONFIG), Oracle(**CLIP_CONFIG)
    ka = [(k, tuple(v.shape)) for k, v in a.state_dict().items()]
    assert ka == [(k, tuple(v.shape)) for k, v in b.state_dict().items()]
    assert len(ka) == 520
    assert sum(torch.Size(s).numel() for _, s in ka) == 632_076_800
    assert ka[0] == ("vision_model.embeddings.class_embedding", (1280,))
    assert ka[-1] == ("visual_projection.weight", (1024, 1280))


def test_state_dict_keys_equal_transformers():
    tr = pytest.importorskip("transformers")
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection as Ours
    with torch.device("meta"):
        hf = tr.CLIPVisionModelWithProjection(tr.CLIPVisionConfig(**CLIP_CONFIG))
        ours = Ours(**CLIP_CONFIG)
    assert [(k, tuple(v.shape)) for k, v in hf.state_dict().items()] == [(k, tuple(v.shape)) for k, v in ours.state_dict().items()]


@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
def test_oracle_reproduces_transformers_golden(act):
    from oracle.svd_clip_oracle import CLIPVisionModelWithProjection as Oracle, integer_init_, integer_pixels
    g = _golden()["clip"][act]
    m = integer_init_(Oracle(**g["config"]).double(), g["param_seed"])
    with torch.no_grad():
        r = m(integer_pixels((2, 3, 224, 224), g["input_seed"]))
    assert _rel(r.image_embeds, g["image_embeds"]) < 1e-12
    assert _rel(r.last_hidden_state[:, ::8], g["last_hidden_state_every8"]) < 1e-12


@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
def test_oracle_matches_live_transformers_fp32(act):
    tr = pytest.importorskip("transformers")
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG, CLIPVisionModelWithProjection as Oracle
    cfg = dict(TINY_CLIP_CONFIG, hidden_act=act)
    torch.manual_seed(5)
    m = Oracle(**cfg).eval()
    hf = tr.CLIPVisionModelWithProjection(tr.CLIPVisionConfig(**cfg)).eval()
    hf.load_state_dict(m.state_dict(), strict=True)
    x = torch.randn(2, 3, 224, 224)
    with torch.no_grad():
        a, b = m(x), hf(pixel_values=x)
    assert _rel(a.image_embeds, b.image_embeds) < 1e-5
    assert _rel(a.last_hidden_state, b.last_hidden_state) < 1e-5


def test_oracle_resize_reproduces_reference_golden():
    from oracle.svd_clip_oracle import integer_pixels, resize_with_antialiasing
    for (h, w), g in _golden()["resize"].items():
        y = resize_with_antialiasing(integer_pixels((1, 3, h, w), g["seed"]), (224, 224))
        assert y.shape == (1, 3, 224, 224)
        assert (y.flatten()[g["index"].long()] - g["values"]).abs().max().item() < 1e-12
        assert abs(y.sum().item() - g["sum"]) < 1e-9 * max(1.0, abs(g["sum"]))
        assert abs((y * y).sum().item() - g["sumsq"]) < 1e-9 * g["sumsq"]


def test_host_gaussians_match_oracle():
    from oracle.svd_clip_oracle import antialias_params, gaussian_1d
    from svd_xtend_b200.clip import antialias_kernels
    for h, w in ((576, 1024), (320, 512), (100, 150), (224, 224), (291, 397), (2160, 3840)):
        (sy, sx), (ky, kx) = antialias_params(h, w)
        gy, gx = antialias_kernels(h, w, 224)
        assert (len(gy), len(gx)) == (ky, kx) and ky % 2 == kx % 2 == 1
        assert torch.equal(torch.tensor(gy), gaussian_1d(ky, sy)) and torch.equal(torch.tensor(gx), gaussian_1d(kx, sx))
    assert [len(v) for v in antialias_kernels(576, 1024, 224)] == [3, 7]


def test_default_normalisation_equals_clip_image_processor():
    tr = pytest.importorskip("transformers")
    from svd_xtend_b200.clip import CLIP_MEAN, CLIP_STD
    p = tr.CLIPImageProcessor()
    assert tuple(p.image_mean) == CLIP_MEAN and tuple(p.image_std) == CLIP_STD


def test_preprocessor_config_parsing(tmp_path):
    from svd_xtend_b200.clip import CLIP_MEAN, CLIP_STD, image_processor_stats
    d = tmp_path / "feature_extractor"
    d.mkdir()
    (d / "preprocessor_config.json").write_text(json.dumps({"image_mean": [0.5, 0.25, 0.125], "image_std": [1, 2, 4], "crop_size": 224}))
    assert image_processor_stats(str(tmp_path)) == ((0.5, 0.25, 0.125), (1.0, 2.0, 4.0))
    (d / "preprocessor_config.json").write_text(json.dumps({"do_normalize": True}))
    assert image_processor_stats(str(tmp_path)) == (CLIP_MEAN, CLIP_STD)


def test_clip_flops_census():
    from oracle.svd_clip_oracle import CLIP_CONFIG
    from svd_xtend_b200.clip import clip_flops
    f = clip_flops(CLIP_CONFIG)
    assert round(f["total"] / 1e9, 2) == 334.59
    assert round(f["linear"] / 1e9, 2) == 323.38 and round(f["attention"] / 1e9, 2) == 10.82
    assert round(f["patch_embedding"] / 1e9, 2) == 0.39 and round(f["projection"] / 1e9, 3) == 0.003


def test_guards_and_loading_without_gpu(tmp_path):
    from safetensors.torch import save_file
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection as Ours, encode_image
    with pytest.raises(ValueError, match="head dim"):
        Ours(**dict(TINY_CLIP_CONFIG, num_attention_heads=4))
    with pytest.raises(ValueError, match="hidden_act"):
        Ours(**dict(TINY_CLIP_CONFIG, hidden_act="relu"))
    m = Ours(**TINY_CLIP_CONFIG).requires_grad_(False)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 224, 224))
    with pytest.raises(RuntimeError, match="CUDA"):
        encode_image(m, torch.zeros(1, 3, 64, 64))
    m.requires_grad_(True)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 224, 224))
    # from_pretrained: config.json + model.fp16.safetensors, strict, the old position_ids buffer tolerated
    d = tmp_path / "image_encoder"
    d.mkdir()
    (d / "config.json").write_text(json.dumps(dict(TINY_CLIP_CONFIG, architectures=["CLIPVisionModelWithProjection"])))
    sd = {k: v.half().contiguous() for k, v in m.state_dict().items()}
    sd["vision_model.embeddings.position_ids"] = torch.arange(257)[None]
    save_file(sd, str(d / "model.fp16.safetensors"))
    m2 = Ours.from_pretrained(str(tmp_path), variant="fp16", torch_dtype=torch.float16)
    assert m2.dtype == torch.float16 and m2.config.hidden_act == "gelu"
    for k, v in m2.state_dict().items():
        assert torch.equal(v, m.state_dict()[k].half())
    del sd["visual_projection.weight"]
    save_file(sd, str(d / "model.fp16.safetensors"))
    with pytest.raises(RuntimeError, match="visual_projection"):
        Ours.from_pretrained(str(tmp_path), variant="fp16")


def test_preprocess_rejects_bad_arguments_without_gpu():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200._lib import load
    lib = load()
    c_f = ctypes.c_float
    one, seven = (c_f * 1)(1.0), (c_f * 65)(*([0.0] * 65))
    aff = (c_f * 6)(1, 1, 1, 0, 0, 0)
    fake = ctypes.c_void_p(1 << 20)

    def call(strides, H, W, ky, gy, kx, gx):
        s = (ctypes.c_int64 * 4)(*strides)
        return lib.svdx_clip_preprocess(fake, 0, s, 1, H, W, gy, ky, gx, kx, aff, 224, 14, fake, 640, None)
    cont = (3 * 64 * 64, 64 * 64, 64, 1)
    assert call((3 * 64 * 64, 64 * 64, 1, 64), 64, 64, 1, one, 1, one) == -1               # non-contiguous (transposed)
    assert b"contiguous" in lib.svdx_last_error()
    assert call(cont, 64, 64, 65, seven, 1, one) == -1                                      # beyond SVDX_CLIP_MAX_TAPS
    assert call(cont, 64, 64, 4, seven, 1, one) == -1                                       # even kernel
    assert b"63" in lib.svdx_last_error()
    assert call((3 * 4 * 64, 4 * 64, 64, 1), 4, 64, 9, seven, 1, one) == -1                 # reflect pad 4 >= H = 4
    assert b"reflect" in lib.svdx_last_error()


def test_shim_installs_the_image_encoder():
    tr = pytest.importorskip("transformers")
    from svd_xtend_b200 import shim
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection as Ours
    before = tr.CLIPVisionModelWithProjection
    try:
        assert shim.install_clip() is True
        from transformers import CLIPVisionModelWithProjection as got
        assert got is Ours
    finally:
        tr.CLIPVisionModelWithProjection = before
        import transformers.models.clip as mc
        mc.CLIPVisionModelWithProjection = before


# ----------------------------------------------------------------------------------------------------------- GPU: kernels
def _within_one_bf16_ulp(out, ref64):
    """|out - bf16(ref)| <= one bf16 ulp at |bf16(ref)|; below 2^-8 the ulp is taken as 2^-15 (an absolute floor: the affine
    v * a_c + b_c cancels there, and its fp32 rounding, ~1e-7 of the operands, is all that is left of the value)"""
    r = ref64.to(bf16).double()
    ulp = torch.exp2(torch.floor(torch.log2(r.abs().clamp_min(2.0 ** -8))) - 7)
    return ((out.double() - r).abs() / ulp).max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(576, 1024), (320, 512), (100, 150), (224, 224)])
@pytest.mark.parametrize("dtype", [torch.float32, bf16, torch.float16])
@pytest.mark.parametrize("B", [1, 3])
def test_preprocess_matches_oracle(H, W, dtype, B):
    from oracle.svd_clip_oracle import CLIP_MEAN, CLIP_STD, clip_input, patchify
    from svd_xtend_b200 import raw
    from svd_xtend_b200.clip import antialias_kernels
    g = torch.Generator().manual_seed(H * 7 + W + B)
    x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dtype)
    ref = patchify(clip_input(x.double(), 224, CLIP_MEAN, CLIP_STD))
    gy, gx = antialias_kernels(H, W, 224)
    aff = [0.5 / s for s in CLIP_STD] + [(0.5 - m) / s for m, s in zip(CLIP_MEAN, CLIP_STD)]
    out = torch.full((B * 257, 640), float("nan"), device=DEV, dtype=bf16)
    raw.clip_preprocess(x.to(DEV), gy, gx, aff, out, out_size=224, patch=14)
    out = out.cpu()
    rows = out.view(B, 257, 640)
    assert torch.equal(rows[:, 0], torch.zeros_like(rows[:, 0])) and torch.equal(rows[:, :, 588:], torch.zeros_like(rows[:, :, 588:]))
    d = _within_one_bf16_ulp(out, ref)
    assert d <= 1.0, d
    if (H, W) == (224, 224):
        # kernel size 1 + identity resize + identity affine: the input itself, patchified
        ident = torch.empty_like(out, device=DEV)
        raw.clip_preprocess(x.to(DEV), [1.0], [1.0], [1, 1, 1, 0, 0, 0], ident, out_size=224, patch=14)
        assert torch.equal(ident.cpu(), patchify(x.float()).to(bf16))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_preprocess_and_encode_accept_batch1_frame_slices(dtype):
    """train_svd.py:975-976 encodes `pixel_values[:, 0].float()` of a [1, F, 3, H, W] batch: a view that keeps the video's
    batch stride. torch calls it contiguous (a size-1 dimension's stride is never used), and so does svdx_clip_preprocess."""
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    from svd_xtend_b200 import raw
    from svd_xtend_b200.clip import antialias_kernels, encode_image
    video = (torch.rand(1, 14, 3, 320, 512, device=DEV) * 2 - 1).to(dtype)
    frame = video[:, 0].float()
    assert frame.is_contiguous() and frame.stride(0) == 14 * 3 * 320 * 512
    gy, gx = antialias_kernels(320, 512, 224)
    aff = [1.0, 1.0, 1.0, 0.0, 0.0, 0.0]
    a, b = (torch.empty(257, 640, device=DEV, dtype=bf16) for _ in range(2))
    raw.clip_preprocess(frame, gy, gx, aff, a, out_size=224, patch=14)
    raw.clip_preprocess(frame.clone(), gy, gx, aff, b, out_size=224, patch=14)
    assert torch.equal(a, b)
    _, ours = _pair(TINY_CLIP_CONFIG, seed=4)
    with torch.no_grad():
        e1, e2 = encode_image(ours, frame), encode_image(ours, frame.clone())
    assert torch.equal(e1, e2)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
@pytest.mark.parametrize("M,N,K", [(257, 5120, 1280), (514, 640, 160), (2, 1280, 640), (64, 1280, 5120)])
def test_activation_epilogue(act, M, N, K):
    from svd_xtend_b200 import raw
    from svd_xtend_b200._lib import SvdxError
    code = dict(gelu=raw.ACT_GELU, quick_gelu=raw.ACT_QUICK_GELU)[act]
    if (M, N, K) == (64, 1280, 5120):
        assert raw.split_plan(True, M, N, K) is not None          # a split-K shape without the activation: launched whole with it
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    x = torch.randn(M, K, device=DEV, generator=g).to(bf16)
    w = (torch.randn(N, K, device=DEV, generator=g) * K ** -0.5).to(bf16)
    b = torch.randn(N, device=DEV, generator=g)
    out = torch.empty(M, N, device=DEV, dtype=bf16)
    raw.tapgemm_auto(x, w, out, M=M, N=N, K=K, bias=b, act=code)
    z = x.float() @ w.float().t() + b
    ref = F.gelu(z) if act == "gelu" else z * torch.sigmoid(1.702 * z)
    e = _rel(out.float(), ref)
    assert e < 4e-3, e
    assert (out.float() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())
    with pytest.raises(SvdxError, match="act"):
        raw.tapgemm(x, w, out, M=M, N=N, K=K, bias=b, act=code, res1=out)     # activation with a residual: refused


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 5, 64, 65, 257, 577])
@pytest.mark.parametrize("heads", [2, 16])
def test_attention_hd80_matches_sdpa(S, heads):
    from svd_xtend_b200 import raw
    B = 1 + S % 3
    C = heads * 80
    g = torch.Generator(device=DEV).manual_seed(S * 31 + heads)
    qkv = (torch.randn(B * S, 3 * C, device=DEV, generator=g) * 1.5).to(bf16)
    sentinel = 7.0
    o_full = torch.full((B * S + 64, C + 32), sentinel, device=DEV, dtype=bf16)
    raw.attention_hd80_fwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], o_full[:, :C], heads=heads, S=S, nseq=B, scale=80 ** -0.5)
    q, k, v = (qkv[:, i * C:(i + 1) * C].float().view(B, S, heads, 80).transpose(1, 2) for i in range(3))
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B * S, C)
    out = o_full[:B * S, :C].float()
    assert _rel(out, ref) < 1e-2 and (out - ref).abs().max().item() < 3e-2
    assert bool((o_full[B * S:] == sentinel).all()) and bool((o_full[:, C:] == sentinel).all())     # rows past S never written


# ----------------------------------------------------------------------------------------------------------- GPU: the encoder
def _pair(cfg, seed, device=DEV):
    from oracle.svd_clip_oracle import CLIPVisionModelWithProjection as Oracle
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection as Ours
    torch.manual_seed(seed)
    with torch.device(device):
        oracle = Oracle(**cfg)
        with torch.no_grad():
            for n, p in oracle.named_parameters():
                if "norm" in n:
                    p.add_(0.1 * torch.randn_like(p))
        ours = Ours(**cfg)
    ours.load_state_dict(oracle.state_dict())
    return oracle.eval().requires_grad_(False), ours.eval().requires_grad_(False)


def _check(ours_out, run_oracle, what):
    """rel-L2 of ours against the fp32 oracle within max(2 x the oracle's own error under bf16 autocast, 2e-2)"""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ref = run_oracle()
        with torch.autocast("cuda", dtype=bf16):
            ac = run_oracle()
    e, e_ac = _rel(ours_out.float(), ref), _rel(ac.float(), ref)
    print(f"{what}: rel-l2 {e:.3e} (oracle under bf16 autocast {e_ac:.3e})")
    assert torch.isfinite(ours_out).all()
    assert e <= max(2 * e_ac, 2e-2), (e, e_ac)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
def test_tiny_encoder_matches_oracle(act):
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG
    oracle, ours = _pair(dict(TINY_CLIP_CONFIG, hidden_act=act), seed=3)
    x = torch.randn(3, 3, 224, 224, device=DEV)
    with torch.no_grad():
        out = ours(x)
    assert out.image_embeds.shape == (3, 96) and out.image_embeds.dtype == torch.float32
    _check(out.image_embeds, lambda: oracle(x).image_embeds, f"tiny {act} image_embeds")
    _check(out.last_hidden_state, lambda: oracle(x).last_hidden_state, f"tiny {act} last_hidden_state")
    with pytest.raises(ValueError, match="doesn't match"):
        ours(torch.zeros(1, 3, 112, 112, device=DEV))
    with pytest.raises(RuntimeError, match="forward-only"):
        ours.requires_grad_(True)(x)


@pytest.fixture(scope="module")
def svd_pair():
    from oracle.svd_clip_oracle import CLIP_CONFIG
    return _pair(CLIP_CONFIG, seed=11)


@pytest.mark.gpu
def test_svd_encoder_forward_matches_oracle(svd_pair):
    oracle, ours = svd_pair
    x = torch.randn(2, 3, 224, 224, device=DEV)
    with torch.no_grad():
        out = ours(x).image_embeds
    assert out.shape == (2, 1024)
    _check(out, lambda: oracle(x).image_embeds, "svd forward B=2")


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(576, 1024), (320, 512)])
def test_svd_encode_image_matches_oracle(svd_pair, H, W):
    from oracle.svd_clip_oracle import encode_image as oracle_encode
    from svd_xtend_b200.clip import encode_image
    oracle, ours = svd_pair
    x = torch.rand(2, 3, H, W, device=DEV) * 2 - 1
    with torch.no_grad():
        out = encode_image(ours, x)
    _check(out, lambda: oracle_encode(oracle, x), f"svd encode_image {H}x{W}")


@pytest.mark.gpu
def test_svd_encoder_fp16_parameters(svd_pair):
    """fp16 parameters (the pipeline's variant="fp16") against the fp32 oracle holding the same fp16-rounded weights: the model
    converted in place after fp32 calls (its cached operands are rebuilt from the new parameters, layer by layer) and a
    model built in fp16 agree with it"""
    from oracle.svd_clip_oracle import encode_image as oracle_encode
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection as Ours, encode_image
    oracle, ours = svd_pair
    half = ours.to(torch.float16)
    oracle.load_state_dict({k: v.float() for k, v in half.state_dict().items()})
    with torch.device(DEV):
        fresh = Ours(**vars(ours.config)).to(torch.float16)
    fresh.load_state_dict(half.state_dict())
    fresh.requires_grad_(False)
    x = torch.rand(1, 3, 320, 512, device=DEV) * 2 - 1
    for m, what in ((half, "converted"), (fresh, "built in fp16")):
        with torch.no_grad():
            out = encode_image(m, x)
        assert out.dtype == torch.float16
        _check(out, lambda: oracle_encode(oracle, x), f"svd encode_image fp16 parameters, {what}")
