"""LoRA adapters on the H100: svdx_lora_merge bit for bit against oracle/svd_lora_oracle.py, fuse / unfuse round trips, two
loaded adapters on the tiny UNet against the merged-weight oracle (forward and training), and the pipeline with a loaded
adapter, fused and unfused, including the sampler's re-capture after the weights or the adapter state change."""
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# ----------------------------------------------------------------------------- kernel
SHAPES = [(320, 320), (640, 640), (1280, 1280), (320, 1024), (1280, 1024), (100, 70), (1, 1), (65, 129), (33, 200)]
RANKS = [1, 4, 64, 80]          # 80: more than one 64-rank shared-memory chunk
SCALES = [1.0, 0.5, -0.75]


@pytest.mark.parametrize("wdtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("fdtype", [torch.float32, torch.bfloat16])
def test_merge_kernel_bit_exact_against_oracle(wdtype, fdtype):
    from oracle.svd_lora_oracle import merge, ulp
    from svd_xtend_b200.lora import merge_into_base
    g = torch.Generator(DEV).manual_seed(11)
    items = []
    for i, (N, K) in enumerate(SHAPES):
        w = torch.randn(N, K, device=DEV, generator=g).to(wdtype)
        terms = []
        for t, s in enumerate(SCALES):
            r = RANKS[(i + t) % len(RANKS)]
            terms.append((torch.randn(r, K, device=DEV, generator=g).div(r).to(fdtype),
                          torch.randn(N, r, device=DEV, generator=g).mul(0.05).to(fdtype), s))
        items.append((w, terms))
    base = [w.clone() for w, _ in items]
    fused_ref = [merge(w, terms) for w, terms in items]
    merge_into_base(items)                                   # fuse: every job in one launch
    torch.cuda.synchronize()
    for (w, _), ref, (N, K) in zip(items, fused_ref, SHAPES):
        assert torch.equal(w, ref), (N, K, wdtype, fdtype, (w.double() - ref.double()).abs().max().item())
    unfused_ref = [merge(w, [(A, B, -s) for A, B, s in terms]) for w, terms in items]
    merge_into_base([(w, [(A, B, -s) for A, B, s in terms]) for w, terms in items])     # unfuse
    torch.cuda.synchronize()
    for (w, _), ref, b0, f in zip(items, unfused_ref, base, fused_ref):
        assert torch.equal(w, ref)
        # fuse -> unfuse: within one ulp of the dtype at the larger of the base and fused magnitudes
        mag = torch.maximum(torch.maximum(b0.double().abs(), f.double().abs()), w.double().abs())
        assert ((w.double() - b0.double()).abs() <= ulp(mag, wdtype)).all()


# ----------------------------------------------------------------------------- tiny UNet, two adapters
def _build(cfg, seed):
    from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as Oracle
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    torch.manual_seed(seed)
    oracle = Oracle(**cfg).to(DEV)
    with torch.no_grad():
        for n, p in oracle.named_parameters():
            if "norm" in n and n.endswith("weight"):
                p.add_(0.1 * torch.randn_like(p))
            if "norm" in n and n.endswith("bias"):
                p.add_(0.05 * torch.randn_like(p))
            if n.endswith("mix_factor"):
                p.add_(0.3 * torch.randn_like(p))
    with torch.device(DEV):
        ours = Ours(**cfg)
    ours.load_state_dict(oracle.state_dict())
    return oracle, ours


def _adapter_sd(unet, r, seed, alpha=None, up_std=0.05):
    """a LoRA file's state dict (diffusers keys) for every attention linear of `unet`"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, mod in unet.named_modules():
        if isinstance(mod, torch.nn.Linear) and any(name.endswith("." + t) for t in TARGETS):
            sd[f"unet.{name}.lora.down.weight"] = torch.randn(r, mod.in_features, generator=g) / r
            sd[f"unet.{name}.lora.up.weight"] = torch.randn(mod.out_features, r, generator=g) * up_std
            if alpha is not None:
                sd[f"unet.{name}.alpha"] = torch.tensor(float(alpha))
    return sd


def _merged_state(base_sd, adapters):
    """oracle state dict with W + sum weight * scaling * B A; adapters = [(file sd, scaling, weight)]"""
    sd = {k: v.clone() for k, v in base_sd.items()}
    for asd, scaling, weight in adapters:
        for k, down in asd.items():
            if not k.endswith(".lora.down.weight"):
                continue
            m = k[len("unet."):-len(".lora.down.weight")]
            up = asd[k.replace(".lora.down.weight", ".lora.up.weight")]
            sd[m + ".weight"] += scaling * weight * (up.to(DEV).double() @ down.to(DEV).double()).float()
    return sd


def _load_two(tmp_path, ours):
    from svd_xtend_b200.lora import save_lora_weights
    sd_a = _adapter_sd(ours, 4, seed=1, alpha=8)             # scaling 2
    sd_b = _adapter_sd(ours, 16, seed=2)                     # no alpha: lora_alpha = r, scaling 1
    save_lora_weights(str(tmp_path / "a"), sd_a)
    assert ours.load_lora_adapter(str(tmp_path / "a"), adapter_name="a") == "a"
    assert ours.load_lora_adapter(sd_b, adapter_name="b") == "b"
    return sd_a, sd_b


def test_tiny_unet_two_adapters_unfused_fused_disabled(tmp_path):
    from oracle.svd_lora_oracle import merge
    from oracle.svd_unet_oracle import TINY_CONFIG, synthetic_batch
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _build(TINY_CONFIG, seed=31)
    base_sd = {k: v.clone() for k, v in oracle.state_dict().items()}
    sd_a, sd_b = _load_two(tmp_path, ours)
    ours.set_adapters(["a", "b"], [1.0, 0.5])
    oracle.eval()
    ours.eval()
    batch = synthetic_batch(1, 4, 16, 16, seed=17, device=DEV, cross_dim=TINY_CONFIG["cross_attention_dim"])
    args = (batch["sample"], batch["timestep"], batch["encoder_hidden_states"], batch["added_time_ids"])
    with torch.no_grad():
        base_ref = oracle(*args).sample
        oracle.load_state_dict(_merged_state(base_sd, [(sd_a, 2.0, 1.0), (sd_b, 1.0, 0.5)]))
        ref = oracle(*args).sample
        unfused = ours(*args).sample
        ours.disable_lora()
        disabled = ours(*args).sample
        ours.enable_lora()
    assert _rel(ref, base_ref) > 0.05                        # the adapters matter
    assert _rel(unfused, ref) < 2e-2, _rel(unfused, ref)
    assert _rel(disabled, base_ref) < 2e-2, _rel(disabled, base_ref)

    with pytest.raises(ValueError):
        ours.fuse_lora()                                     # base weights still trainable
    ours.requires_grad_(False)
    q = ours.down_blocks[0].attentions[0].transformer_blocks[0].attn1.to_q
    w0 = q.base_layer.weight.clone()
    terms = [(q.lora_A[n].weight, q.lora_B[n].weight, s) for n, s in (("a", 2.0), ("b", 0.5))]
    ours.fuse_lora()
    wf = q.base_layer.weight.clone()
    assert torch.equal(wf, merge(w0, terms))                           # the kernel's merge, in the model
    assert q.merged_adapters == ["a", "b"]
    with pytest.raises(ValueError):
        ours.set_adapters(["a"])
    with pytest.raises(ValueError):
        ours.delete_adapters("b")
    with torch.no_grad():
        fused = ours(*args).sample
    assert _rel(fused, ref) < 2e-2, _rel(fused, ref)
    ours.unfuse_lora()
    assert q.merged_adapters == []
    from oracle.svd_lora_oracle import ulp
    w1 = q.base_layer.weight.double()
    mag = torch.maximum(torch.maximum(w0.double().abs(), wf.double().abs()), w1.abs())
    assert ((w1 - w0.double()).abs() <= ulp(mag, torch.float32)).all()


def test_tiny_train_one_adapter_while_other_is_fused(tmp_path):
    from oracle.svd_unet_oracle import TINY_CONFIG, edm_loss, synthetic_batch
    torch.backends.cuda.matmul.allow_tf32 = False
    oracle, ours = _build(TINY_CONFIG, seed=32)
    base_sd = {k: v.clone() for k, v in oracle.state_dict().items()}
    sd_a, sd_b = _load_two(tmp_path, ours)
    ours.requires_grad_(False)
    ours.set_adapters(["a", "b"], [1.0, 0.5])
    ours.fuse_lora(adapter_names=["b"])
    for n, p in ours.named_parameters():
        if ".lora_A.a." in n or ".lora_B.a." in n:
            p.requires_grad_(True)
    oracle.load_state_dict(_merged_state(base_sd, [(sd_a, 2.0, 1.0), (sd_b, 1.0, 0.5)]))
    oracle.requires_grad_(False)
    lin = {}
    for name, mod in ours.named_modules():
        if hasattr(mod, "lora_A"):
            lin[name] = mod
            dict(oracle.named_parameters())[name + ".weight"].requires_grad_(True)
    oracle.train()
    ours.train()
    batch = synthetic_batch(1, 4, 16, 16, seed=99, device=DEV, cross_dim=TINY_CONFIG["cross_attention_dim"])

    def loss(model):
        pred = model(batch["sample"], batch["timestep"], batch["encoder_hidden_states"], batch["added_time_ids"]).sample
        return pred, edm_loss(pred.float(), batch["noisy"], batch["latents"], batch["sigmas"])
    pred_ref, l_ref = loss(oracle)
    l_ref.backward()
    pred, l = loss(ours)
    l.backward()
    torch.cuda.synchronize()
    assert _rel(pred, pred_ref) < 2e-2
    gw = dict(oracle.named_parameters())
    bad = []
    for name, mod in lin.items():
        assert mod.lora_A["b"].weight.grad is None and mod.lora_B["b"].weight.grad is None
        dW = gw[name + ".weight"].grad
        A, B = mod.lora_A["a"].weight, mod.lora_B["a"].weight
        for gr, ref, tag in ((A.grad, 2.0 * B.detach().t() @ dW, "A"), (B.grad, 2.0 * dW @ A.detach().t(), "B")):
            if ref.abs().max() == 0:
                assert gr.abs().max() == 0
                continue
            e = _rel(gr, ref)
            if e > 8e-2:
                bad.append((name, tag, round(e, 4)))
    assert not bad, bad[:8]


def test_unfuse_undoes_separate_fuse_calls_last_first(tmp_path):
    """two fuse_lora calls round W twice; unfuse_lora subtracts each call's own terms, last call first, so the result is the
    oracle's four merges in that order, bit for bit"""
    from oracle.svd_lora_oracle import merge
    from oracle.svd_unet_oracle import TINY_CONFIG
    _, ours = _build(TINY_CONFIG, seed=33)
    for dt in (torch.float32, torch.bfloat16):
        ours.unload_lora()
        ours.to(dt)
        _load_two(tmp_path / str(dt), ours)
        ours.requires_grad_(False)
        ours.set_adapters(["a", "b"], [1.0, 0.5])
        layers = [m for m in ours.modules() if hasattr(m, "lora_A")]
        w0 = [m.base_layer.weight.clone() for m in layers]
        ours.fuse_lora(adapter_names="a")
        ours.fuse_lora(lora_scale=0.75, adapter_names=["b"])
        ours.unfuse_lora()
        for m, w in zip(layers, w0):
            ta = [(m.lora_A["a"].weight, m.lora_B["a"].weight, 2.0)]
            tb = [(m.lora_A["b"].weight, m.lora_B["b"].weight, 0.375)]
            neg = lambda t: [(A, B, -s) for A, B, s in t]
            ref = merge(merge(merge(merge(w, ta), tb), neg(tb)), neg(ta))
            assert torch.equal(m.base_layer.weight, ref)
            assert m.merged_adapters == []


# ----------------------------------------------------------------------------- pipeline
def test_tiny_pipeline_with_loaded_adapter(tmp_path):
    from oracle.svd_clip_oracle import TINY_CLIP_CONFIG, image_to_video
    from oracle.svd_clip_oracle import CLIPVisionModelWithProjection as OClip
    from oracle.svd_unet_oracle import TINY_CONFIG
    from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as OUnet
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as OVae
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.clip import CLIPVisionModelWithProjection
    from svd_xtend_b200.pipeline import ImageToVideoPipeline
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(41)
    pairs = []
    for O, P, kw in ((OUnet, UNetSpatioTemporalConditionModel, TINY_CONFIG), (OVae, AutoencoderKLTemporalDecoder, dict(TINY_VAE_CONFIG, with_decoder=True)),
                     (OClip, CLIPVisionModelWithProjection, dict(TINY_CLIP_CONFIG, projection_dim=TINY_CONFIG["cross_attention_dim"]))):
        o = O(**kw).to(DEV)
        with torch.no_grad():
            for n, p in o.named_parameters():
                if "norm" in n:
                    p.add_(0.1 * torch.randn_like(p))
        with torch.device(DEV):
            m = P(**kw)
        m.load_state_dict(o.state_dict())
        pairs.append((o.eval().requires_grad_(False), m.eval().requires_grad_(False)))
    (ou, u), (ov, v), (oc, c) = pairs
    image = torch.rand(1, 3, 32, 32, device=DEV)
    kw = dict(num_frames=4, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.02)
    pipe = ImageToVideoPipeline(u, v, c)
    eager = ImageToVideoPipeline(u, v, c, use_cuda_graph=False)

    def run(p):
        return p(image, generator=torch.Generator(DEV).manual_seed(5), **kw).frames

    def oracle_run(autocast=False):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            return image_to_video(ou, ov, oc, image, generator=torch.Generator(DEV).manual_seed(5), **kw).float()

    # run-to-run spread (fp32 atomics, DESIGN.md §4): it varies from pair to pair, so take the largest of the pairs of four base
    # runs, graphed and eager, and allow twice that
    runs = [run(pipe), run(pipe), run(eager), run(eager)]
    base = runs[0]
    same = max(2 * max(_rel(a, b) for i, a in enumerate(runs) for b in runs[i + 1:]), 1e-2)

    def recaptured(prev=None):
        """the graphed sampler agrees with the eager one within the eager runs' own spread in the current state (a strong
        adapter amplifies the run-to-run noise); when `prev` is given, the state change moved the result by more than twice
        that, so the graphed result is closer to the new state than a replay of the stale capture (`prev`) could be"""
        graphed, e1, e2 = run(pipe), run(eager), run(eager)
        tol_state = max(same, 2 * _rel(e2, e1))
        print(f"graphed vs eager {_rel(graphed, e1):.3e}, eager vs eager {_rel(e2, e1):.3e}, tolerance {tol_state:.3e}"
              + ("" if prev is None else f", moved {_rel(e1, prev):.3e}"))
        if prev is not None:
            assert _rel(e1, prev) > 2 * tol_state, (_rel(e1, prev), tol_state)
        assert _rel(graphed, e1) <= tol_state, (_rel(graphed, e1), tol_state)
        return graphed

    base_sd = {k: v.clone() for k, v in ou.state_dict().items()}
    sd = _adapter_sd(u, 8, seed=3, up_std=0.3)
    ImageToVideoPipeline.save_lora_weights(str(tmp_path), {k[len("unet."):]: t for k, t in sd.items()})
    assert pipe.load_lora_weights(str(tmp_path)) == "default_0"
    ou.load_state_dict(_merged_state(base_sd, [(sd, 1.0, 1.0)]))
    ref, ref_ac = oracle_run(), oracle_run(True)
    tol = max(2 * _rel(ref_ac, ref), 2e-2)
    unfused = recaptured(base)                               # loading the adapter
    assert _rel(unfused, ref) <= tol, (_rel(unfused, ref), tol)

    pipe.fuse_lora()
    fused = recaptured()                                     # fuse: the merged weights were captured again
    assert _rel(fused, ref) <= tol, (_rel(fused, ref), tol)

    pipe.set_adapters([])            # no active adapter: after the unfuse the UNet is the base model again
    pipe.unfuse_lora()
    back = recaptured(fused)
    assert _rel(back, base) <= same, (_rel(back, base), same)

    pipe.set_adapters("default_0", 2.0)                     # set_adapters: the side path at twice the scale
    doubled = recaptured(back)

    # load_state_dict rewrites the base weights: the graphed sampler must not replay the old operands
    pipe.unload_lora_weights()
    plain = run(pipe)
    assert _rel(plain, doubled) > 2 * same
    torch.manual_seed(9)
    new_sd = {k: t + 0.2 * torch.randn_like(t) if k.endswith(("to_v.weight", "to_out.0.weight")) else t for k, t in u.state_dict().items()}
    u.load_state_dict(new_sd)
    recaptured(plain)
