"""CPU tests of the weight EMA (svd_xtend_b200.ema.EMAModel, oracle/svd_ema_oracle.py): the decay schedule, serialisation,
the version-counter behaviour of copy_to / restore, the shim, the C-ABI argument checks and the sharded EMA plumbing."""
import ctypes
import json
import os

import pytest
import torch

from oracle import svd_ema_oracle as O
from svd_xtend_b200 import ema as E

CONFIGS = {
    "default": dict(),
    "update_after_step_3": dict(update_after_step=3),
    "warmup_power_3_4": dict(use_ema_warmup=True, power=3 / 4),
    "min_decay_0_5": dict(min_decay=0.5),
    "cap_0_99": dict(decay=0.99),
}


def test_get_decay_hand_values():
    for g in (O.get_decay, E.get_decay):
        assert g(1) == 0.0 and g(2) == 2 / 11 and g(10) == 10 / 19
        assert g(10 ** 6) == 0.9999                                          # (1 + s) / (10 + s) capped at decay
        assert g(4, update_after_step=3) == 0.0 and g(5, update_after_step=3) == 2 / 11
        assert g(2, use_ema_warmup=True, power=3 / 4) == 1 - 2 ** -0.75
        assert g(3, use_ema_warmup=True, power=3 / 4, inv_gamma=2.0) == 1 - 2 ** -0.75
        assert g(1, min_decay=0.5) == 0.0                                    # the s <= 0 branch returns before min_decay
        assert g(2, min_decay=0.5) == 0.5 and g(100, min_decay=0.5) == 100 / 109
        assert g(1000, decay=0.99) == 0.99 and g(20, decay=0.99) == 20 / 29
    for name, kw in CONFIGS.items():
        assert [O.get_decay(t, **kw) for t in range(1, 60)] == [E.get_decay(t, **kw) for t in range(1, 60)], name


def test_oracle_step_is_the_diffusers_recurrence():
    w = torch.nn.Parameter(torch.tensor([1.0, 2.0, 3.0]))
    f = torch.nn.Parameter(torch.tensor([5.0]), requires_grad=False)
    ema = O.EMAModel([w, f])
    with torch.no_grad():
        w.add_(1.0)
        f.add_(1.0)
    ema.step([w, f])                          # t = 1: d = 0, s -= 1 * (s - p)
    assert ema.cur_decay_value == 0.0 and torch.equal(ema.shadow_params[0], w.detach()) and ema.shadow_params[1].item() == 6.0
    with torch.no_grad():
        w.add_(11.0)
    ema.step([w, f])                          # t = 2: d = 2/11
    s = torch.tensor([2.0, 3.0, 4.0])
    s.sub_((1 - 2 / 11) * (s - w.detach()))
    assert torch.equal(ema.shadow_params[0], s) and ema.optimization_step == 2


def _params():
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.Linear(5, 3))
    net[1].requires_grad_(False)
    return net


def test_state_dict_keys_and_round_trip():
    net = _params()
    ema = E.EMAModel(net.parameters(), decay=0.999, min_decay=0.1, update_after_step=2, use_ema_warmup=True, inv_gamma=2.0, power=0.75)
    sd = ema.state_dict()
    assert set(sd) == set(O.EMAModel(net.parameters()).state_dict()) == set(O.STATE_KEYS) | {"shadow_params"}
    assert sd["optimization_step"] == 0 and sd["decay"] == 0.999 and sd["use_ema_warmup"] is True and len(sd["shadow_params"]) == 4
    other = E.EMAModel(net.parameters())
    sd2 = dict(sd, optimization_step=17, shadow_params=[s + 1 for s in sd["shadow_params"]])
    other.load_state_dict(sd2)
    got = other.state_dict()
    for k in O.STATE_KEYS:
        assert got[k] == sd2[k], k
    assert all(torch.equal(a, b) for a, b in zip(got["shadow_params"], sd2["shadow_params"]))
    with pytest.raises(ValueError):
        other.load_state_dict({"decay": 1.5})
    with pytest.raises(ValueError):
        other.load_state_dict({"optimization_step": 1.0})


def test_data_write_does_not_move_the_version_but_copy_to_does():
    """diffusers' copy_to writes through p.data, invisible to version-counter staleness checks; ours moves the counter"""
    p = torch.nn.Parameter(torch.zeros(4))
    p.data.copy_(torch.ones(4))
    assert p._version == 0
    net = _params()
    ema = E.EMAModel(net.parameters())
    ora = O.EMAModel(net.parameters())
    with torch.no_grad():
        for s in ema.shadow_params[:2] + ora.shadow_params[:2]:       # the trainable tensors' EMA moved away from them
            s.add_(0.5)
    v0 = [q._version for q in net.parameters()]
    ora.copy_to(net.parameters())
    assert [q._version for q in net.parameters()] == v0
    with torch.no_grad():
        for q, b in zip(net.parameters(), O.EMAModel(net.parameters()).shadow_params):
            q.data.copy_(b - 0.5 if q.requires_grad else b)
    before = [q.detach().clone() for q in net.parameters()]
    ema.store(net.parameters())
    ema.copy_to(net.parameters())
    assert [q._version > v for q, v in zip(net.parameters(), v0)] == [True, True, False, False]
    assert all(torch.equal(q, s) for q, s in zip(net.parameters(), ema.shadow_params))
    ema.restore(net.parameters())
    assert all(torch.equal(q, b) for q, b in zip(net.parameters(), before))
    with pytest.raises(RuntimeError, match="store"):
        ema.restore(net.parameters())


def test_copy_to_skips_frozen_tensors_known_equal_to_their_shadow():
    net = _params()
    ema = E.EMAModel(net.parameters())
    frozen = [q for q in net.parameters() if not q.requires_grad]
    v0 = [q._version for q in frozen]
    ema.store(net.parameters())
    assert [c is None for c in ema.temp_stored_params] == [False, False, True, True]
    ema.copy_to(net.parameters())
    assert [q._version for q in frozen] == v0
    ema.restore(net.parameters())
    with torch.no_grad():
        frozen[0].add_(1.0)                   # moved since the shadow was taken: copy_to writes the (old) shadow back
    ema.copy_to(net.parameters())
    assert frozen[0]._version > v0[0] and torch.equal(frozen[0], ema.shadow_params[2])


def test_step_has_no_cpu_fallback():
    net = _params()
    ema = E.EMAModel(net.parameters())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ema.step(net.parameters())


def test_save_pretrained_from_pretrained_tiny_unet(tmp_path):
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    torch.manual_seed(3)
    unet = Ours(**TINY_CONFIG)
    ema = E.EMAModel(unet.parameters(), decay=0.995, update_after_step=5, model_cls=Ours, model_config=unet.config)
    with torch.no_grad():
        for s in ema.shadow_params:
            s.mul_(0.5)
    ema.optimization_step = 123
    d = str(tmp_path / "unet_ema")
    ema.save_pretrained(d)
    cfg = json.load(open(os.path.join(d, "config.json")))
    assert {k: cfg[k] for k in O.STATE_KEYS} == {k: v for k, v in ema.state_dict().items() if k != "shadow_params"}
    assert cfg["in_channels"] == unet.config.in_channels and cfg["_class_name"] == "UNetSpatioTemporalConditionModel"
    loaded = Ours.from_pretrained(d)                      # the EMA weights as a model directory
    for q, s in zip(loaded.parameters(), ema.shadow_params):
        assert torch.equal(q, s)
    back = E.EMAModel.from_pretrained(d, Ours)            # train_svd.py:710-712
    assert back.optimization_step == 123 and back.decay == 0.995 and back.update_after_step == 5
    for a, b in zip(back.shadow_params, ema.shadow_params):
        assert torch.equal(a, b)
    assert not hasattr(unet.config, "decay")              # the live model's config is untouched
    with pytest.raises(ValueError, match="model_cls"):
        E.EMAModel(unet.parameters()).save_pretrained(d)


def test_shim_installs_the_ema_as_diffusers_training_utils(monkeypatch):
    import importlib
    import sys
    import types
    from svd_xtend_b200 import shim
    fake = types.ModuleType("diffusers")
    fake.__path__ = []
    tu = types.ModuleType("diffusers.training_utils")
    tu.EMAModel = object
    fake.training_utils = tu
    monkeypatch.setitem(sys.modules, "diffusers", fake)
    monkeypatch.setitem(sys.modules, "diffusers.training_utils", tu)
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)
    shim.install()
    assert importlib.import_module("diffusers.training_utils").EMAModel is E.EMAModel
    monkeypatch.delitem(sys.modules, "src", raising=False)
    monkeypatch.delitem(sys.modules, "src.unet_spatio_temporal_condition", raising=False)


def test_attach_rules_on_cpu_arena():
    from svd_xtend_b200.train import FusedAdamW, ParamArena
    net = _params()
    init = [q.detach().clone() for q in net.parameters()]
    arena = ParamArena(net)
    opt = FusedAdamW(arena)
    with pytest.raises(ValueError, match="cover"):
        opt.attach_ema(E.EMAModel(list(net.parameters())[:1]))
    ema = E.EMAModel(net.parameters())
    opt.attach_ema(ema)
    ps = list(net.parameters())
    assert all(torch.equal(s, q) for s, q in zip(ema.shadow_params, init))
    assert ema.shadow_params[2].data_ptr() == ps[2].data_ptr()                # a frozen tensor's EMA is the tensor
    off = arena.offset_of[ps[0]]
    assert ema.shadow_params[0].data_ptr() == ema._flat[off:].data_ptr()      # arena shadows live at the arena offsets
    assert ema._flat.data_ptr() in [t.data_ptr() for t in opt.snapshot_tensors()]
    with pytest.raises(RuntimeError, match="attached"):
        ema.step(net.parameters())


def test_adamw_step_abi_rejects_bad_ema_arguments():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200 import _lib
    lib = _lib.load()
    assert lib.svdx_ema_multi(None, None, 0, 0, None, None) == -1
    assert b"ema_multi" in lib.svdx_last_error()
    assert lib.svdx_adamw_step(None, None, None, None, 0, None, 1.0, None, None, None, None, None) == -1
    buf = (ctypes.c_double * 16)()
    misaligned = ctypes.addressof(buf) + 4
    assert lib.svdx_adamw_step_p2p(None, None, None, None, None, 1, 0, 4, None, 1.0, 1, None, misaligned, None, None) == -1
    assert b"adamw_step_p2p" in lib.svdx_last_error()
    # every other argument valid: an EMA buffer without its state, or the state without a buffer, is refused
    a = (ctypes.addressof(buf) + 15) & ~15
    arenas = (ctypes.c_void_p * 1)(a)
    for ema, ema_state in ((a, None), (None, a)):
        assert lib.svdx_adamw_step(a, a, a, a, 4, a, 1.0, None, ema, ema_state, None, None) == -1
        assert b"adamw_step: bad arguments" in lib.svdx_last_error()
        assert lib.svdx_adamw_step_p2p(a, a, a, arenas, arenas, 1, 0, 4, a, 1.0, 1, ema, ema_state, None, None) == -1
        assert b"adamw_step_p2p: bad arguments" in lib.svdx_last_error()
    for name in ("svdx_adamw_step", "svdx_adamw_step_p2p", "svdx_ema_multi"):
        assert name in _lib._PROTOS
    # the per-option entry points that svdx_adamw_step / _step_p2p / svdx_adamw8bit_step replace are not exported, so a binding
    # written for them fails on a missing symbol rather than dropping the EMA or the clip
    for name in ("svdx_adamw_graph", "svdx_adamw_graph_ema", "svdx_adamw_graph_mul", "svdx_adamw_graph_ema_mul", "svdx_adamw_p2p",
                 "svdx_adamw_p2p_ema", "svdx_adamw_p2p_mul", "svdx_adamw_p2p_ema_mul", "svdx_adamw8bit", "svdx_adamw8bit_ema",
                 "svdx_adamw8bit_mul", "svdx_adamw8bit_ema_mul"):
        assert not hasattr(lib, name), name


def test_bench_ema_counts_bytes_from_shapes():
    """scripts/bench_ema.py: the per-step HBM bytes of the three EMA forms; on the SVD UNet these are the figures the step
    times are read against (21.7 GB for the reference loop, 4.77 GB for the drop-in, 3.18 GB inside AdamW)"""
    import importlib.util
    from oracle.svd_unet_oracle import SVD_CONFIG
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "bench_ema.py")
    spec = importlib.util.spec_from_file_location("bench_ema", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    net = _params()
    assert mod.ema_bytes(list(net.parameters())) == {"reference_loop": 32 * 40 + 8 * 18, "dropin": 12 * 40, "fused_in_adamw": 8 * 40,
                                                    "trainable_params": 40, "frozen_params": 18}
    with torch.device("meta"):
        unet = Ours(**SVD_CONFIG)
    unet.requires_grad_(False)
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:
            p.requires_grad_(True)
    b = mod.ema_bytes(list(unet.parameters()))
    assert b["trainable_params"] == 397_620_480 and b["frozen_params"] == 1_127_002_602
    assert b["reference_loop"] == 21_739_876_176 and b["dropin"] == 4_771_445_760 and b["fused_in_adamw"] == 3_180_963_840
