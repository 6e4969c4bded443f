"""CPU tests of the host-side mirror: construction, naming contract, helper API, no-CPU-fallback."""
import os

import pytest
import torch

from oracle.svd_unet_oracle import SVD_CONFIG, TINY_CONFIG
from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as Oracle
from svd_xtend_b200.engine import Geom
from svd_xtend_b200.raw import pick_block_n
from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours


def test_same_parameter_names_and_shapes_as_oracle():
    with torch.device("meta"):
        a, b = Ours(**SVD_CONFIG), Oracle(**SVD_CONFIG)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa.keys()) == list(sb.keys())
    assert all(sa[k].shape == sb[k].shape for k in sa)
    assert sum(p.numel() for p in a.parameters()) == 1_524_623_082


def test_trainable_filter_of_train_svd():
    """train_svd.py:761-766 selects parameters by name substring."""
    with torch.device("meta"):
        m = Ours(**SVD_CONFIG)
    n = sum(p.numel() for k, p in m.named_parameters() if "temporal_transformer_block" in k)
    assert n == 397_620_480


def test_constructor_errors_match_reference():
    with pytest.raises(ValueError, match="down_block_types"):
        Ours(**{**TINY_CONFIG, "up_block_types": ("UpBlockSpatioTemporal",)})
    with pytest.raises(ValueError, match="block_out_channels"):
        Ours(**{**TINY_CONFIG, "block_out_channels": (64,)})
    with pytest.raises(ValueError, match="num_attention_heads"):
        Ours(**{**TINY_CONFIG, "num_attention_heads": (1, 2, 3)})
    with pytest.raises(ValueError):
        Ours(**{**TINY_CONFIG, "down_block_types": ("Nope", "DownBlockSpatioTemporal")})


def test_helper_api_surface():
    m = Ours(**TINY_CONFIG)
    assert m.config.addition_time_embed_dim == 32 and m.config["in_channels"] == 8   # train_svd.py:887-889
    assert m.add_embedding.linear_1.in_features == 96
    procs = m.attn_processors
    assert len(procs) == 16 and all(k.endswith(".processor") for k in procs)
    assert "down_blocks.0.attentions.0.transformer_blocks.0.attn1.processor" in procs
    m.set_attn_processor(dict(procs))
    with pytest.raises(ValueError, match="number of processors"):
        m.set_attn_processor({"x": 1})
    m.set_default_attn_processor()
    assert not m.is_gradient_checkpointing
    m.enable_gradient_checkpointing()
    assert m.is_gradient_checkpointing
    with pytest.raises(ValueError):
        m.enable_forward_chunking(dim=2)
    m.enable_forward_chunking(2, dim=1)
    m.enable_xformers_memory_efficient_attention()


def test_no_cpu_fallback():
    m = Ours(**TINY_CONFIG)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(1, 2, 8, 16, 16), torch.zeros(1), torch.zeros(1, 1, 64), torch.zeros(1, 3))


def test_save_load_roundtrip(tmp_path):
    torch.manual_seed(1)
    m = Ours(**TINY_CONFIG)
    m.save_pretrained(os.path.join(tmp_path, "unet"))
    m2 = Ours.from_pretrained(str(tmp_path), subfolder="unet", low_cpu_mem_usage=True, variant="fp16")
    for (ka, va), (kb, vb) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    oracle = Oracle(**TINY_CONFIG)
    oracle.load_state_dict(m.state_dict())       # same key contract both ways


def test_tile_selection_and_geometry():
    assert pick_block_n(320) == 160 and pick_block_n(1280) == 256 and pick_block_n(960) == 160
    assert pick_block_n(320, True) == 64 and pick_block_n(1280, True) == 256
    assert pick_block_n(4) == 32
    g = Geom(2, 14, 40, 64)
    assert g.M == 2 * 14 * 2560 and g.down().HW == 640 and g.down().up().W == 64


def test_shim_installs_the_replacement_under_both_reference_import_paths(monkeypatch):
    """svd_xtend_b200.shim.install(): `from diffusers import UNetSpatioTemporalConditionModel` (train_svd.py:49) and
    `from src.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel` (train_svd_lora.py:60) must both
    resolve to the H100 class. diffusers is absent here, so a stand-in package plays its role."""
    import importlib
    import sys
    import types
    from svd_xtend_b200 import shim
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    fake = types.ModuleType("diffusers")
    fake.__path__ = []
    fake.UNetSpatioTemporalConditionModel = object
    sub = types.ModuleType("diffusers.models")
    sub.__path__ = []
    sub.UNetSpatioTemporalConditionModel = object
    monkeypatch.setitem(sys.modules, "diffusers", fake)
    monkeypatch.setitem(sys.modules, "diffusers.models", sub)
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)
    shim.install()
    assert importlib.import_module("diffusers").UNetSpatioTemporalConditionModel is Ours
    assert importlib.import_module("diffusers.models").UNetSpatioTemporalConditionModel is Ours
    from src.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel as viaSrc   # noqa: the shim's module
    assert viaSrc is Ours
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)


def test_shim_fails_loudly_without_diffusers(monkeypatch):
    import sys
    import pytest
    from svd_xtend_b200 import shim
    monkeypatch.setitem(sys.modules, "diffusers", None)      # import diffusers -> ModuleNotFoundError
    with pytest.raises(RuntimeError, match="diffusers"):
        shim.install()


def test_wide_tile_rule():
    """320-wide tile requests: only where the alternative is 160-wide tiles, the contraction is long, and the launch has the
    bf16 TMA-store epilogue (raw._wide_tile_ok mirrors the library's conditions)"""
    from svd_xtend_b200 import raw
    bf16 = torch.bfloat16
    out = torch.empty(1024, 640, dtype=bf16)
    common = dict(ldo=None, geglu=False, a_mn=False, b_mn=False, b_mode=0, split_k=1, out_dtype=None, bias=None, rowbias=None)
    assert raw._wide_tile_ok(1024, 640, 2560, out, **common)
    assert raw._wide_tile_ok(35840, 320, 2880, torch.empty(8, 320, dtype=bf16), **common)
    assert not raw._wide_tile_ok(1024, 640, 640, out, **common)                       # short contraction
    assert not raw._wide_tile_ok(1024, 1280, 5120, torch.empty(8, 1280, dtype=bf16), **common)   # 256-wide tiles divide N
    assert not raw._wide_tile_ok(256, 640, 2560, out, **common)                        # small M
    assert not raw._wide_tile_ok(1024, 480, 2560, torch.empty(8, 480, dtype=bf16), **common)     # N % 320
    assert not raw._wide_tile_ok(1024, 640, 2560, torch.empty(8, 640), **common)       # fp32 output
    assert not raw._wide_tile_ok(1024, 640, 2560, out, **{**common, "geglu": True})
    assert not raw._wide_tile_ok(1024, 640, 2560, out, **{**common, "split_k": 4})
    assert not raw._wide_tile_ok(1024, 640, 2560, out, **{**common, "a_mn": True, "b_mn": True})


def test_groupnorm_backward_fusion_is_decided_per_launch():
    """Engine._gnb_for: the dgrad epilogue carries the GroupNorm-backward sums only when it is the first writer of that
    gradient, has the plain epilogue (no scales), the widths match and the launch is not split-K"""
    from svd_xtend_b200 import raw
    from svd_xtend_b200.engine import Engine, Var
    E = Engine()
    M, rows = 35840, 2560
    x = torch.zeros(M, 320, dtype=torch.bfloat16)
    y = Var(torch.zeros(M, 320, dtype=torch.bfloat16), needs_grad=True)
    y.gnb = dict(x=x, x2=None, ab=torch.zeros(M // rows, 2, 320), rows=rows, silu=True, C=320)
    E._stat_arena = torch.zeros(1 << 16)
    g = E._gnb_for(y, M, 320, 320, 9, None, "cpu")
    assert g is not None and g["sum"].shape == (M // rows, 2, 320) and g["rows"] == rows and g["x"] is x
    assert E._gnb_for(y, M, 320, 320, 9, torch.ones(3), "cpu") is None                 # scaled accumulation (LoRA / blend)
    assert E._gnb_for(y, M, 640, 320, 9, None, "cpu") is None                          # not this GroupNorm's width
    assert E._gnb_for(y, M - 64, 320, 320, 9, None, "cpu") is None                     # rows do not tile into slabs
    y.grad = torch.zeros(8, 320, dtype=torch.bfloat16)
    assert E._gnb_for(y, M, 320, 320, 9, None, "cpu") is None                          # somebody already wrote this gradient
    y.grad = None
    assert E._gnb_for(Var(x, True), M, 320, 320, 9, None, "cpu") is None               # not a GroupNorm output
    # small levels run split-K (fp32 workspace + epilogue kernel): no fused sums there
    small = Var(torch.zeros(2560, 320, dtype=torch.bfloat16), needs_grad=True)
    small.gnb = dict(x=x[:2560], x2=None, ab=torch.zeros(2, 2, 320), rows=1280, silu=True, C=320)
    assert raw.split_plan(True, 2560, 320, 320, 9) is not None and E._gnb_for(small, 2560, 320, 320, 9, None, "cpu") is None
    # a second accumulation invalidates sums computed for the first
    y.gnb_sums = (g["sum"], torch.zeros(1))
    E.add_grad(y, torch.zeros(8, 320, dtype=torch.bfloat16))
    assert y.gnb_sums is None


def test_peer_memory_optimizer_step_api_exists():
    from svd_xtend_b200 import _lib, train
    assert issubclass(train.P2PShardedAdamW, train.ShardedAdamW)
    for name in ("svdx_adamw_step_p2p", "svdx_ipc_export", "svdx_ipc_import", "svdx_enable_peer_access"):
        assert name in _lib._PROTOS
