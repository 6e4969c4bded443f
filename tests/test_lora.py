"""LoRA adapters without a GPU: the on-disk format (svd_xtend_b200.lora) round trip and its rejections, the UNet's adapter
bookkeeping, the shim's save_lora_weights patch, and the merge oracle against an fp64 merge."""
import os
from types import SimpleNamespace

import pytest
import torch
import torch.nn as nn

TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]


def _unet(seed=0):
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    torch.manual_seed(seed)
    return UNetSpatioTemporalConditionModel(**TINY_CONFIG)


def _adapted(r, seed=0, name="default"):
    u = _unet(seed)
    u.add_adapter(SimpleNamespace(r=r, lora_alpha=r, init_lora_weights="gaussian", target_modules=TARGETS), name)
    with torch.no_grad():
        for m in u.modules():
            if hasattr(m, "lora_B"):
                m.lora_B[name].weight.normal_(0, 0.05)
    return u


def _snapshot(u):
    return ({k: v.clone() for k, v in u.state_dict().items()}, dict(u.peft_config), u.lora_stamp, u.active_adapters())


def _unchanged(u, snap):
    sd, cfg, stamp, active = snap
    now = u.state_dict()
    return (now.keys() == sd.keys() and all(torch.equal(now[k], v) for k, v in sd.items()) and u.peft_config == cfg
            and u.lora_stamp == stamp and u.active_adapters() == active)


@pytest.mark.parametrize("r", [4, 16])
@pytest.mark.parametrize("spelling", ["peft", "diffusers"])
@pytest.mark.parametrize("prefix", [False, True])
@pytest.mark.parametrize("alpha", [False, True])
@pytest.mark.parametrize("source", ["dict", "safetensors", "bin"])
def test_round_trip_bit_equal(tmp_path, r, spelling, prefix, alpha, source):
    from svd_xtend_b200.lora import lora_adapter_state_dict, save_lora_weights
    src = _adapted(r, seed=1)
    sd = {}
    for k, v in lora_adapter_state_dict(src, "default").items():
        if spelling == "diffusers":
            k = k.replace(".lora_A.weight", ".lora.down.weight").replace(".lora_B.weight", ".lora.up.weight")
        sd[("unet." if prefix else "") + k] = v
    if alpha:
        mods = {k.rsplit(".lora", 1)[0] for k in sd}
        for m in mods:
            sd[m + ".alpha"] = torch.tensor(2.0 * r)
    if source == "dict":
        arg = sd
    else:
        path = save_lora_weights(str(tmp_path), sd, safe_serialization=(source == "safetensors"))
        assert os.path.basename(path) == ("pytorch_lora_weights.safetensors" if source == "safetensors" else "pytorch_lora_weights.bin")
        if source == "safetensors":
            from safetensors.torch import load_file
            keys = load_file(path).keys()
        else:
            keys = torch.load(path).keys()
        assert all(k.startswith("unet.") and (k.endswith((".lora.down.weight", ".lora.up.weight", ".alpha"))) for k in keys)
        arg = str(tmp_path)
    dst = _unet(seed=2)
    name = dst.load_lora_adapter(arg, adapter_name="mine")
    assert name == "mine" and dst.active_adapters() == ["mine"] and "mine" in dst.peft_config
    n = 0
    src_layers = dict(src.named_modules())
    for full, mod in dst.named_modules():
        if not hasattr(mod, "lora_A"):
            continue
        s = src_layers[full]
        assert torch.equal(mod.lora_A["mine"].weight, s.lora_A["default"].weight)
        assert torch.equal(mod.lora_B["mine"].weight, s.lora_B["default"].weight)
        assert mod.r["mine"] == r and mod.scaling["mine"] == (2.0 if alpha else 1.0)
        assert not mod.lora_A["mine"].weight.requires_grad
        n += 1
    assert n == 64


def test_unnamed_loads_take_the_next_free_default_name():
    from svd_xtend_b200.lora import lora_adapter_state_dict
    sd = lora_adapter_state_dict(_adapted(4), "default")
    u = _unet()
    assert u.load_lora_adapter(sd) == "default_0"
    assert u.load_lora_adapter(sd) == "default_1"
    assert u.active_adapters() == ["default_1"]


def _good_sd():
    from svd_xtend_b200.lora import lora_adapter_state_dict
    return {"unet." + k: v for k, v in lora_adapter_state_dict(_adapted(4), "default").items()}


def _malformed():
    cases = {}
    sd = _good_sd()
    k0 = next(iter(sd))
    bad = dict(sd)
    bad["unet.down_blocks.0.attentions.0.no_such.to_q.lora_A.weight"] = torch.zeros(4, 64)
    bad["unet.down_blocks.0.attentions.0.no_such.to_q.lora_B.weight"] = torch.zeros(64, 4)
    cases["no such module"] = bad
    bad = dict(sd)
    bad["unet.conv_in.lora_A.weight"] = torch.zeros(4, 8)      # a Conv2d, not an nn.Linear
    bad["unet.conv_in.lora_B.weight"] = torch.zeros(64, 4)
    cases["not a linear"] = bad
    cases["other component"] = dict(sd, **{"text_encoder.text_model.encoder.layers.0.self_attn.q_proj.lora_A.weight": torch.zeros(4, 8)})
    bad = dict(sd)
    bad.pop(k0.replace("lora_A", "lora_B") if "lora_A" in k0 else k0)
    cases["unpaired"] = bad
    bad = dict(sd)
    bad[k0] = torch.zeros(sd[k0].shape[0], sd[k0].shape[1] + 1)
    cases["shape"] = bad
    bad = dict(sd)
    ka = [k for k in sd if k.endswith("lora_A.weight")][0]
    bad[ka] = torch.zeros(5, sd[ka].shape[1])                   # rank differs from its up factor
    cases["rank mismatch"] = bad
    cases["not a lora key"] = dict(sd, **{"unet.conv_in.weight": torch.zeros(3)})
    # real nn.Linear layers, but without a LoRA side path: unfused they would be ignored, fused they would not
    for tag, mod, (out_f, in_f) in (("proj_in", "down_blocks.0.attentions.0.proj_in", (64, 64)),
                                    ("ff.net.2", "down_blocks.0.attentions.0.transformer_blocks.0.ff.net.2", (64, 256)),
                                    ("time_embedding", "time_embedding.linear_1", (256, 64))):
        cases[f"no side path: {tag}"] = dict(sd, **{f"unet.{mod}.lora.down.weight": torch.zeros(4, in_f),
                                                   f"unet.{mod}.lora.up.weight": torch.zeros(out_f, 4)})
    cases["empty"] = {}
    return cases


@pytest.mark.parametrize("case", list(_malformed()))
def test_malformed_files_are_rejected_without_change(case):
    sd = _malformed()[case]
    u = _adapted(4, seed=3, name="present")
    snap = _snapshot(u)
    with pytest.raises(ValueError):
        u.load_lora_adapter(sd, adapter_name="new")
    assert _unchanged(u, snap)


def test_existing_adapter_name_is_rejected_without_change():
    u = _adapted(4, seed=3, name="present")
    snap = _snapshot(u)
    with pytest.raises(ValueError):
        u.load_lora_adapter(_good_sd(), adapter_name="present")
    with pytest.raises(ValueError):
        u.add_adapter(SimpleNamespace(r=4, lora_alpha=4, target_modules=TARGETS), "present")
    assert _unchanged(u, snap)


def test_adapter_bookkeeping_and_stamp():
    from svd_xtend_b200.unet import LoraLinear, _lora_of
    u = _unet()
    stamps = [u.lora_stamp]

    def moved():
        stamps.append(u.lora_stamp)
        return stamps[-1] != stamps[-2]

    cfg_a = SimpleNamespace(r=4, lora_alpha=8, init_lora_weights="gaussian", target_modules=TARGETS)
    assert u.add_adapter(cfg_a, "a") == 64 and moved()
    assert u.peft_config["a"] is cfg_a
    cfg_b = SimpleNamespace(r=8, lora_alpha=8, init_lora_weights=True, target_modules=["to_q"])
    assert u.add_adapter(cfg_b, "b") == 16 and moved()       # to_q layers are already LoraLinear: the adapter is added to them
    assert u.peft_config["b"] is cfg_b and u.active_adapters() == ["b"]
    trainable = [k for k, p in u.named_parameters() if p.requires_grad]
    assert len(trainable) == 32 and all(".b." in k for k in trainable)
    q = u.down_blocks[0].attentions[0].transformer_blocks[0].attn1.to_q
    k = u.down_blocks[0].attentions[0].transformer_blocks[0].attn1.to_k
    assert isinstance(q, LoraLinear) and set(q.lora_A) == {"a", "b"} and set(k.lora_A) == {"a"}
    assert [t[4] for t in _lora_of(q)] == [1.0] and _lora_of(k) == []

    u.set_adapters(["a", "b"], [1.0, 0.5])
    assert moved() and u.active_adapters() == ["a", "b"]
    assert [t[4] for t in _lora_of(q)] == [2.0, 0.5] and [t[4] for t in _lora_of(k)] == [2.0]
    assert [t[0] for t in _lora_of(q, 64)] == [64, 64]
    u.set_adapters("a", 0.25)
    assert moved() and [t[4] for t in _lora_of(q)] == [0.5]
    with pytest.raises(ValueError):
        u.set_adapters(["a", "nope"])
    with pytest.raises(ValueError):
        u.set_adapters(["a", "b"], [1.0])
    u.set_adapters(["a", "b"])
    moved()

    u.disable_lora()
    assert moved() and _lora_of(q) == [] and _lora_of(k) == []
    u.enable_lora()
    assert moved() and len(_lora_of(q)) == 2

    u.delete_adapters("a")
    assert moved() and "a" not in u.peft_config and u.active_adapters() == ["b"]
    assert set(q.lora_A) == {"b"} and set(k.lora_A) == set() and not any(".a." in n for n, _ in u.named_parameters())
    with pytest.raises(ValueError):
        u.delete_adapters("a")

    w_before = q.base_layer.weight
    u.unload_lora()
    assert moved() and u.peft_config == {} and u.active_adapters() == []
    assert not any(isinstance(m, LoraLinear) for m in u.modules())
    q2 = u.down_blocks[0].attentions[0].transformer_blocks[0].attn1.to_q
    assert type(q2) is nn.Linear and q2.weight is w_before
    assert not any("lora" in n or "base_layer" in n for n in u.state_dict())


def test_fuse_on_cpu_raises_the_no_fallback_error():
    u = _adapted(4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        u.fuse_lora()


def test_add_adapter_keeps_its_init_and_count():
    """the first adapter's factors come out of the same random stream as before adapters could be stacked"""
    u = _unet(seed=0)
    torch.manual_seed(7)
    n = u.add_adapter(SimpleNamespace(r=4, lora_alpha=4, init_lora_weights="gaussian", target_modules=TARGETS))
    assert n == 64
    torch.manual_seed(7)
    ref_A = nn.Linear(64, 4, bias=False)
    nn.Linear(4, 64, bias=False)
    nn.init.normal_(ref_A.weight, std=0.25)
    first = u.down_blocks[0].attentions[0].transformer_blocks[0].attn1.to_q
    assert torch.equal(first.lora_A["default"].weight, ref_A.weight)
    assert torch.count_nonzero(first.lora_B["default"].weight) == 0
    with pytest.raises(ValueError):
        _unet().add_adapter(SimpleNamespace(r=4, lora_alpha=4, target_modules=["no_such_module"]))


def test_shim_patches_save_lora_weights_only_where_missing():
    from svd_xtend_b200 import lora
    from svd_xtend_b200.shim import install_lora_writer

    class Lacking:
        pass

    def own(*a, **k):
        return "own"

    class Having:
        save_lora_weights = staticmethod(own)

    assert install_lora_writer(Lacking) is True
    assert Lacking.save_lora_weights is lora.save_lora_weights
    assert install_lora_writer(Having) is False
    assert Having.save_lora_weights is own
    assert install_lora_writer(None) is False


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("fdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("r", [1, 4, 64, 80])
def test_oracle_merge_within_one_ulp_of_fp64(dtype, fdtype, r):
    from oracle.svd_lora_oracle import merge, merge_fp64, ulp
    g = torch.Generator().manual_seed(r)
    N, K = 96, 130
    w = ((torch.rand(N, K, generator=g) * 0.5 + 0.5) * torch.randn(N, K, generator=g).sign()).to(dtype)
    terms = [(torch.randn(r, K, generator=g).to(fdtype) / r, (torch.randn(N, r, generator=g) * 0.01).to(fdtype), s)
             for s in (1.0, 0.5, -0.75)]
    got, ref = merge(w, terms), merge_fp64(w, terms)
    assert got.dtype == dtype
    diff = (got.double() - ref.double()).abs()
    assert (diff <= ulp(torch.maximum(got.double().abs(), ref.double().abs()), dtype)).all()
    assert not torch.equal(got, w)


def test_peft_state_dict_round_trip(tmp_path):
    """the script's own call: convert_state_dict_to_diffusers(get_peft_model_state_dict(unet)) -> save_lora_weights -> load"""
    peft = pytest.importorskip("peft")
    pytest.importorskip("diffusers")
    from diffusers.utils import convert_state_dict_to_diffusers
    from peft.utils import get_peft_model_state_dict
    from svd_xtend_b200.lora import save_lora_weights
    u = _unet(seed=4)
    u.add_adapter(peft.LoraConfig(r=4, lora_alpha=4, init_lora_weights="gaussian", target_modules=TARGETS))
    with torch.no_grad():
        for m in u.modules():
            if hasattr(m, "lora_B"):
                m.lora_B["default"].weight.normal_(0, 0.05)
    sd = convert_state_dict_to_diffusers(get_peft_model_state_dict(u))
    save_lora_weights(str(tmp_path), sd, safe_serialization=True)
    v = _unet(seed=5)
    v.load_lora_adapter(str(tmp_path), adapter_name="x")
    src = dict(u.named_modules())
    for full, mod in v.named_modules():
        if hasattr(mod, "lora_A"):
            assert torch.equal(mod.lora_A["x"].weight, src[full].lora_A["default"].weight)
            assert torch.equal(mod.lora_B["x"].weight, src[full].lora_B["default"].weight)


@pytest.mark.parametrize("targets", [["proj_in"], ["to_q", "ff.net.2"], ["linear_1"]])
def test_add_adapter_refuses_linears_without_a_side_path(targets):
    u = _adapted(4, seed=3, name="present")
    snap = _snapshot(u)
    with pytest.raises(ValueError, match="side path"):
        u.add_adapter(SimpleNamespace(r=4, lora_alpha=4, init_lora_weights="gaussian", target_modules=targets), "new")
    assert _unchanged(u, snap)


def test_alpha_other_than_rank_survives_write_and_read(tmp_path):
    from svd_xtend_b200.lora import lora_adapter_state_dict, save_lora_weights
    sd = _good_sd()
    for m in {k.rsplit(".lora", 1)[0] for k in sd}:
        sd[m + ".alpha"] = torch.tensor(12.0)                  # r = 4: scaling 3
    u = _unet(seed=6)
    u.load_lora_adapter(sd, adapter_name="x")
    out = lora_adapter_state_dict(u, "x")
    assert sum(k.endswith(".alpha") for k in out) == 64
    save_lora_weights(str(tmp_path), out)
    v = _unet(seed=7)
    v.load_lora_adapter(str(tmp_path), adapter_name="y")
    layers = [m for m in v.modules() if hasattr(m, "lora_A")]
    assert len(layers) == 64 and all(m.scaling["y"] == 3.0 and m.lora_alpha["y"] == 12.0 for m in layers)
    # alpha == r writes no alpha: the dict is what PEFT returns
    assert not any(k.endswith(".alpha") for k in lora_adapter_state_dict(_adapted(4), "default"))


def test_graph_runner_drops_entries_of_earlier_adapter_states():
    """every adapter change starts a new entry; the entries (and graph pools) of earlier states are released, except one
    whose backward is still pending"""
    from svd_xtend_b200.autograph import GraphRunner
    u = _adapted(4)
    runner = GraphRunner(u, warmup=5)          # within warm-up: the calls return before touching a device
    x = torch.zeros(1, 4, 8, 16, 16)
    args = (x, torch.zeros(1), torch.zeros(1, 1, 64), torch.zeros(1, 3))
    assert runner.forward(False, *args) is None
    assert len(runner.entries) == 1
    u.set_adapters("default", 0.5)
    runner.forward(False, *args)
    assert len(runner.entries) == 1 and next(iter(runner.entries))[-1] == u.lora_stamp
    next(iter(runner.entries.values())).pending_backward = True
    u.disable_lora()
    runner.forward(False, *args)
    assert len(runner.entries) == 2            # the pending one stays until its backward has run
    for e in runner.entries.values():
        e.pending_backward = False
    u.enable_lora()
    runner.forward(False, *args)
    assert len(runner.entries) == 1 and next(iter(runner.entries))[-1] == u.lora_stamp
