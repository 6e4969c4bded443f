"""CPU tests of the block-wise 8-bit AdamW (oracle/svd_adam8bit_oracle.py, svd_xtend_b200.optim8bit, train.FusedAdamW8bit): the
quantisation maps, the quantiser's tie and zero rules, the block layout over real ParamArena offsets, the drop-in's argument
checks and scheduler compatibility, state-dict round trips, the shim and the C-ABI argument checks."""
import ctypes
import sys
import types

import numpy as np
import pytest
import torch

from oracle import svd_adam8bit_oracle as O


# ------------------------------------------------------------------------------------------------------------- maps
@pytest.mark.parametrize("signed", [True, False])
def test_maps_are_256_sorted_with_zero_and_one_and_equal_the_oracle(signed):
    from svd_xtend_b200.optim8bit import dynamic_map
    q = dynamic_map(signed)
    assert q.dtype == torch.float32 and q.numel() == 256
    assert bool((q[1:] > q[:-1]).all())                       # strictly sorted: 0.0 appears once
    assert 0.0 in q.tolist() and 1.0 in q.tolist()
    assert q.max().item() == 1.0
    if signed:
        assert q.min().item() < 0 and int((q < 0).sum()) == 127 and int((q > 0).sum()) == 128
    else:
        assert q.min().item() == 0.0
    assert torch.equal(q, O.create_dynamic_map(signed))


# ------------------------------------------------------------------------------------------------------------- quantiser
def test_quantiser_midpoint_ties_go_to_the_lower_code():
    q = O.create_dynamic_map(True)
    mid = O.midpoints(q)
    k = 200
    a = torch.tensor(1.0)
    # one block whose absmax is 1.0: x = value exactly
    x = torch.zeros(256)
    x[0] = 1.0
    x[1] = mid[k]                                              # exact midpoint -> lower code k
    x[2] = torch.nextafter(mid[k], torch.tensor(2.0))         # just above -> k + 1
    x[3] = q[k]                                                # a code value maps to itself
    codes, absmax = O.quantize(x, q, signed=True)
    assert absmax.item() == a.item()
    assert codes[1].item() == k and codes[2].item() == k + 1 and codes[3].item() == k
    assert codes[0].item() == 255                              # 1.0 is the largest code


@pytest.mark.parametrize("signed", [True, False])
def test_all_zero_block_stores_the_code_of_zero(signed):
    q = O.create_dynamic_map(signed)
    x = torch.zeros(300)
    x[260] = 0.5                                              # block 1 non-zero, block 0 all zero
    codes, absmax = O.quantize(x, q, signed=signed)
    zero = int((q == 0).nonzero().item())
    assert absmax[0].item() == 0.0 and absmax[1].item() == 0.5
    assert bool((codes[:256] == zero).all())
    assert O.dequantize(codes, absmax, q)[:256].abs().max().item() == 0.0
    assert O.dequantize(codes, absmax, q)[260].item() == 0.5


def test_quantiser_roundtrip_error_is_bounded_by_the_map_spacing():
    torch.manual_seed(0)
    q = O.create_dynamic_map(True)
    x = torch.randn(1000) * 1e-3
    codes, absmax = O.quantize(x, q, signed=True)
    y = O.dequantize(codes, absmax, q)
    idx = torch.arange(1000) // 256
    assert bool(((y - x).abs() <= 0.08 * absmax[idx] + 1e-12).all())


def test_oracle_step_fp32_equals_torch_adamw_semantics():
    """the fp32-state branch of the oracle is AdamW (bias-corrected, decoupled weight decay) up to rounding order"""
    torch.manual_seed(1)
    p = torch.randn(100)
    p_ref = torch.nn.Parameter(p.clone())
    opt = torch.optim.AdamW([p_ref], lr=1e-2, weight_decay=1e-2, foreach=False)
    m, v = torch.zeros(100), torch.zeros(100)
    state = torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0])
    for _ in range(3):
        g = torch.randn(100)
        O.tick(state)
        O.step_fp32(p, g, m, v, state)
        p_ref.grad = g.clone()
        opt.step()
    assert torch.allclose(p, p_ref.detach(), rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------- layout
class _Net(torch.nn.Module):
    def __init__(self, sizes):
        super().__init__()
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(n)) for n in sizes])


SIZES = [1, 255, 256, 257, 4095, 4096, 4097, 70000, 513]


def test_block_layout_over_arena_offsets():
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    net = _Net(SIZES)
    arena = ParamArena(net)
    opt = FusedAdamW8bit(arena, lr=1e-3)
    rows = opt.job_rows()
    assert rows.shape == (len(SIZES), 10)
    base, gbase = arena.data.data_ptr(), arena.grad.data_ptr()
    covered = np.zeros(arena.numel, dtype=np.int32)
    for r, (p, off, quant, so, bo) in zip(rows, opt.layout):
        n = p.numel()
        assert off == arena.offset_of[p]
        assert r[0] - base == 4 * off and r[1] - gbase == 4 * off
        assert r[8] == n and bool(r[9]) == quant == (n >= 4096)
        assert r[6] == 0 and r[7] == 0                          # CPU arena: no shadow, no EMA
        nb = (n + 255) // 256
        starts = [off + 256 * k for k in range(nb)]
        ends = [min(s + 256, off + n) for s in starts]
        assert ends[-1] - starts[-1] == (n - 256 * (nb - 1))   # partial last block
        for s, e in zip(starts, ends):
            covered[s:e] += 1
        if quant:
            assert r[4] - opt.absmax1.data_ptr() == 4 * bo and r[5] - opt.absmax2.data_ptr() == 4 * bo
            assert r[2] - opt.codes1.data_ptr() == so and so % 256 == 0
            sv = opt.state_views(p)
            assert sv["state1"].dtype == torch.uint8 and sv["state1"].shape == p.shape and sv["absmax1"].numel() == nb
        else:
            assert r[4] == 0 and r[5] == 0
            assert r[2] - opt.m32.data_ptr() == 4 * so
            assert opt.state_views(p)["state1"].dtype == torch.float32
    # every element of every parameter is in exactly one block, arena padding in none
    in_param = np.zeros(arena.numel, dtype=np.int32)
    for p in arena.params:
        o = arena.offset_of[p]
        in_param[o:o + p.numel()] = 1
    assert np.array_equal(covered, in_param)
    assert opt.codes1.numel() == sum(((n + 255) // 256) * 256 for n in SIZES if n >= 4096)
    assert opt.absmax1.numel() == sum((n + 255) // 256 for n in SIZES if n >= 4096)


@pytest.mark.parametrize("n,quant", [(4095, False), (4096, True)])
def test_min_8bit_size_boundary(n, quant):
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    arena = ParamArena(_Net([n]))
    assert FusedAdamW8bit(arena).layout[0][2] == quant
    assert FusedAdamW8bit(arena, min_8bit_size=n + 1).layout[0][2] is False


def test_job_table_prefix():
    from svd_xtend_b200.optim8bit import JobTable, job_row
    t = JobTable("cpu")
    rows = np.array([job_row(0, 0, 0, 0, 0, 0, 0, 0, n, n >= 4096) for n in (1, 256, 257, 5000)], dtype=np.int64)
    t.set(rows)
    assert t.prefix.tolist() == [0, 1, 2, 4] and t.blocks == 4 + 20 and t.njobs == 4
    assert t.dev.numel() == 4 * 80
    dev0 = t.dev
    t.set(rows.copy())
    assert t.dev is dev0                                       # unchanged pointers: no re-upload


def test_byte_counts():
    from svd_xtend_b200.optim8bit import state_bytes, update_bytes
    assert state_bytes([4096]) == 2 * 4096 + 8 * 16
    assert state_bytes([4095]) == 8 * 4095
    assert update_bytes(256, 0, shadow=True, ema=False) == 18 * 256 + 16
    assert update_bytes(0, 64, shadow=True, ema=False) == 30 * 64
    assert update_bytes(0, 64, shadow=True, ema=True) == 38 * 64
    # the as-scripted trainable set of the SVD UNet (all 8-bit, whole blocks): 2.03125 bytes per parameter
    assert abs(state_bytes([397_620_480]) / 397_620_480 - 2.03125) < 1e-6


# ------------------------------------------------------------------------------------------------------------- drop-in
def _params():
    return [torch.nn.Parameter(torch.randn(5000)), torch.nn.Parameter(torch.randn(10))]


@pytest.mark.parametrize("kw", [dict(amsgrad=True), dict(percentile_clipping=95), dict(block_wise=False), dict(is_paged=True),
                                dict(args=object()), dict(lr=-1.0), dict(betas=(1.0, 0.999))])
def test_drop_in_rejects_unsupported_arguments(kw):
    from svd_xtend_b200.optim8bit import AdamW8bit
    with pytest.raises(ValueError):
        AdamW8bit(_params(), **kw)


@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step\\(\\)`")
def test_drop_in_constructor_defaults_and_scheduler():
    from svd_xtend_b200.optim8bit import AdamW8bit
    opt = AdamW8bit(_params(), lr=1e-4, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    g = opt.param_groups[0]
    assert g["lr"] == 1e-4 and g["min_8bit_size"] == 4096 and g["block_wise"] and not g["amsgrad"]
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 1.0 / (s + 1))
    assert isinstance(opt, torch.optim.Optimizer)
    for k in range(1, 4):
        sched.step()
        assert opt.param_groups[0]["lr"] == pytest.approx(1e-4 / (k + 1))


def test_drop_in_rejects_cpu_and_non_fp32_tensors():
    from svd_xtend_b200.optim8bit import AdamW8bit
    ps = _params()
    for p in ps:
        p.grad = torch.zeros_like(p)
    with pytest.raises(TypeError, match="CUDA"):
        AdamW8bit(ps).step()
    h = [torch.nn.Parameter(torch.randn(10, dtype=torch.float16))]
    h[0].grad = torch.zeros_like(h[0])
    with pytest.raises(TypeError, match="float32"):
        AdamW8bit(h).step()


def test_fused_state_dict_round_trip_and_load_into_drop_in():
    from svd_xtend_b200.optim8bit import AdamW8bit
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    torch.manual_seed(3)
    net = _Net([5000, 10, 4096])
    arena = ParamArena(net)
    opt = FusedAdamW8bit(arena, lr=2e-3, betas=(0.8, 0.99), weight_decay=0.1, eps=1e-6)
    for p in arena.params:
        sv = opt.state_views(p)
        for k in ("state1", "state2"):
            sv[k].copy_(torch.randint(0, 255, sv[k].shape, dtype=torch.uint8) if sv[k].dtype == torch.uint8 else torch.randn(sv[k].shape))
        for k in ("absmax1", "absmax2"):
            if k in sv:
                sv[k].copy_(torch.rand(sv[k].shape))
    opt.state[5] = 7.0
    sd = opt.state_dict()
    assert set(sd["state"][0]) == {"state1", "state2", "qmap1", "qmap2", "absmax1", "absmax2", "step"}
    assert set(sd["state"][1]) == {"state1", "state2", "step"}
    assert sd["state"][0]["step"] == 7 and sd["state"][0]["state1"].shape == (5000,) and sd["state"][0]["absmax1"].shape == (20,)
    assert sd["state"][1]["state1"].dtype == torch.float32
    other = FusedAdamW8bit(ParamArena(_Net([5000, 10, 4096])))
    other.load_state_dict(sd)
    assert other.t == 7 and other.lr == 2e-3 and other.state[1].item() == pytest.approx(0.8)
    for a, b in ((opt.codes1, other.codes1), (opt.codes2, other.codes2), (opt.absmax1, other.absmax1), (opt.m32, other.m32),
                 (opt.v32, other.v32)):
        assert torch.equal(a, b)
    # the same dict loads into the drop-in (bitsandbytes' per-parameter layout); uint8 codes stay uint8
    drop = AdamW8bit(list(_Net([5000, 10, 4096]).parameters()))
    drop.load_state_dict(sd)
    ps = drop.param_groups[0]["params"]
    assert drop.state[ps[0]]["state1"].dtype == torch.uint8 and torch.equal(drop.state[ps[0]]["state1"], sd["state"][0]["state1"])
    assert drop.state[ps[0]]["qmap1"] is drop.state[ps[2]]["qmap1"]
    assert drop.param_groups[0]["lr"] == 2e-3 and tuple(drop.param_groups[0]["betas"]) == (0.8, 0.99)
    back = drop.state_dict()
    assert back["state"][0]["step"] == 7
    other.load_state_dict(back)
    assert torch.equal(other.codes1, opt.codes1)


def test_fused_load_rejects_a_mismatched_layout():
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    sd = FusedAdamW8bit(ParamArena(_Net([5000, 10]))).state_dict()
    with pytest.raises(ValueError):
        FusedAdamW8bit(ParamArena(_Net([5000, 10, 7]))).load_state_dict(sd)
    with pytest.raises(ValueError):
        FusedAdamW8bit(ParamArena(_Net([10, 5000]))).load_state_dict(sd)


# ------------------------------------------------------------------------------------------------------------- shim
def test_shim_registers_a_stand_in_without_bitsandbytes(monkeypatch):
    from svd_xtend_b200 import shim
    from svd_xtend_b200.optim8bit import AdamW8bit
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)
    real_import = __import__("importlib").import_module

    def fake_import(name, *a, **k):
        if name.startswith("bitsandbytes") and name not in sys.modules:
            raise ModuleNotFoundError(name)
        return real_import(name, *a, **k)

    monkeypatch.setattr(shim.importlib, "import_module", fake_import)
    bnb = shim.install_adam8bit()
    assert getattr(bnb, "__svdx_standin__", False) is True
    import bitsandbytes
    assert bitsandbytes is bnb and bitsandbytes.optim.AdamW8bit is AdamW8bit
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)


def test_shim_patches_an_installed_bitsandbytes(monkeypatch):
    from svd_xtend_b200 import shim
    from svd_xtend_b200.optim8bit import AdamW8bit
    fake = types.ModuleType("bitsandbytes")
    fake.__path__ = []
    optim = types.ModuleType("bitsandbytes.optim")
    optim.AdamW8bit = object
    fake.optim = optim
    monkeypatch.setitem(sys.modules, "bitsandbytes", fake)
    monkeypatch.setitem(sys.modules, "bitsandbytes.optim", optim)
    assert shim.install_adam8bit() is fake
    assert optim.AdamW8bit is AdamW8bit and not hasattr(fake, "__svdx_standin__")


def test_stand_in_keeps_find_spec_working_and_other_libraries_see_no_bitsandbytes(monkeypatch):
    """with the stand-in installed, importlib.util.find_spec still answers (a module with __spec__ None makes it raise), and
    transformers, which gates its quantisation integrations on a bitsandbytes version, still reports none available"""
    import importlib.util
    from svd_xtend_b200 import shim
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)
    if importlib.util.find_spec("bitsandbytes") is not None:
        pytest.skip("a real bitsandbytes is installed: no stand-in")
    bnb = shim.install_adam8bit()
    assert bnb.__svdx_standin__
    spec = importlib.util.find_spec("bitsandbytes")
    assert spec is not None and spec.name == "bitsandbytes"
    assert importlib.util.find_spec("bitsandbytes.optim").name == "bitsandbytes.optim"
    try:
        from transformers.utils import import_utils as tiu
    except Exception:
        tiu = None
    if tiu is not None and hasattr(tiu, "is_bitsandbytes_available"):
        fn = tiu.is_bitsandbytes_available
        getattr(fn, "cache_clear", lambda: None)()
        try:
            assert fn() is False
        finally:
            getattr(fn, "cache_clear", lambda: None)()
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)


def _fake_diffusers(monkeypatch):
    fake = types.ModuleType("diffusers")
    fake.__path__ = []
    tu = types.ModuleType("diffusers.training_utils")
    fake.training_utils = tu
    monkeypatch.setitem(sys.modules, "diffusers", fake)
    monkeypatch.setitem(sys.modules, "diffusers.training_utils", tu)
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)


@pytest.mark.parametrize("argv,planted", [(["--use_ema"], False), (["--use_8bit_adam", "--use_ema"], True), (["--use_8bit"], True)])
def test_shim_installs_the_optimizer_only_for_use_8bit_adam(monkeypatch, argv, planted):
    import importlib.util
    from svd_xtend_b200 import shim
    from svd_xtend_b200.optim8bit import AdamW8bit
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)
    if importlib.util.find_spec("bitsandbytes") is not None:
        pytest.skip("a real bitsandbytes is installed")
    _fake_diffusers(monkeypatch)
    monkeypatch.setattr(shim, "install_clip", lambda: False)   # keep an installed transformers untouched for later tests
    assert shim.wants_8bit_adam(argv) == planted
    shim.install(use_8bit_adam=shim.wants_8bit_adam(argv))
    assert ("bitsandbytes" in sys.modules) == planted
    if planted:
        assert sys.modules["bitsandbytes"].optim.AdamW8bit is AdamW8bit
    monkeypatch.setattr(sys, "argv", ["train_svd.py"] + argv)
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)
    shim.install()                                            # None: read from sys.argv
    assert ("bitsandbytes" in sys.modules) == planted
    monkeypatch.delitem(sys.modules, "bitsandbytes", raising=False)
    monkeypatch.delitem(sys.modules, "bitsandbytes.optim", raising=False)
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)


# ------------------------------------------------------------------------------------------------------------- checkpoints
def _valid_state(n, min_8bit_size=4096):
    if n >= min_8bit_size:
        nb = (n + 255) // 256
        return {"state1": torch.zeros(n, dtype=torch.uint8), "state2": torch.zeros(n, dtype=torch.uint8),
                "qmap1": O.create_dynamic_map(True), "qmap2": O.create_dynamic_map(False),
                "absmax1": torch.zeros(nb), "absmax2": torch.zeros(nb), "step": 3}
    return {"state1": torch.zeros(n), "state2": torch.zeros(n), "step": 3}


@pytest.mark.parametrize("key,bad", [("state2", torch.zeros(4999, dtype=torch.uint8)), ("state1", torch.zeros(5000)),
                                     ("absmax1", torch.zeros(19)), ("absmax2", torch.zeros(20, dtype=torch.float64).half()),
                                     ("qmap2", torch.zeros(255)), ("absmax1", None)])
def test_checkpoint_state_is_validated_against_the_parameter(key, bad):
    from svd_xtend_b200.optim8bit import AdamW8bit
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    st = _valid_state(5000)
    if bad is None:
        del st[key]
    else:
        st[key] = bad
    sd = {"state": {0: st, 1: _valid_state(10)},
          "param_groups": [{"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 1e-2, "min_8bit_size": 4096,
                            "params": [0, 1]}]}
    fused = FusedAdamW8bit(ParamArena(_Net([5000, 10])))
    drop = AdamW8bit(list(_Net([5000, 10]).parameters()))
    if key == "absmax2":                       # a half-precision absmax is converted by the drop-in, refused by the fused form
        drop.load_state_dict(sd)
        with pytest.raises(ValueError, match="absmax2"):
            fused.load_state_dict(sd)
        return
    for opt in (fused, drop):
        with pytest.raises(ValueError, match=key):
            opt.load_state_dict(sd)
    # the valid dict loads into both
    sd["state"][0] = _valid_state(5000)
    fused.load_state_dict(sd)
    drop.load_state_dict(sd)


def test_missing_parameter_state_is_reported():
    from svd_xtend_b200.optim8bit import AdamW8bit
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    sd = {"state": {0: _valid_state(5000)},
          "param_groups": [{"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 1e-2, "min_8bit_size": 4096,
                            "params": [0, 1]}]}
    with pytest.raises(ValueError, match=r"no state for parameters \[1\]"):
        FusedAdamW8bit(ParamArena(_Net([5000, 10]))).load_state_dict(sd)
    drop = AdamW8bit(list(_Net([5000, 10]).parameters()))
    drop.load_state_dict(sd)                   # the drop-in starts that parameter from zero state, as bitsandbytes does
    assert len(drop.state) == 1
    sd["state"][7] = _valid_state(10)
    with pytest.raises(ValueError, match="no group holds"):
        drop.load_state_dict(sd)


# ------------------------------------------------------------------------------------------------------------- ABI
def test_abi_rejects_null_and_misaligned_buffers():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200 import _lib
    lib = _lib.load()
    assert lib.svdx_adamw8bit(None, None, 1, 1, None, None, None, 1.0, None) == -1
    assert b"adamw8bit" in lib.svdx_last_error()
    buf = (ctypes.c_double * 64)()
    a = ctypes.addressof(buf)
    assert lib.svdx_adamw8bit(a + 4, a, 1, 1, a, a, a, 1.0, None) == -1          # job table not 8-byte aligned
    assert lib.svdx_adamw8bit(a, a, 0, 1, a, a, a, 1.0, None) == -1              # no jobs
    assert lib.svdx_adamw8bit_ema(a, a, 1, 1, a, a, a, 1.0, None, None) == -1    # EMA form without ema_state
    assert lib.svdx_adamw8bit_ema(a, a, 1, 1, a, a, a, 1.0, a + 4, None) == -1   # misaligned ema_state
