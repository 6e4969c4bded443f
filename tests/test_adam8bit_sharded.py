"""CPU tests of the sharded 8-bit AdamW layout: ParamArena's opt-in block alignment (the default offsets unchanged), the per-rank
sub-jobs of ShardedAdamW8bit / P2PShardedAdamW8bit over the SVD UNet's parameter lists and hand-made sizes at worlds 1, 2, 3, 4
and 8, the misbuilt-arena errors, and the argument checks of svdx_adamw8bit_p2p."""
import ctypes

import pytest
import torch

WORLDS = [1, 2, 3, 4, 8]


class _Net(torch.nn.Module):
    def __init__(self, sizes):
        super().__init__()
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.zeros(n)) for n in sizes])


def _svd_params(which):
    from oracle.svd_unet_oracle import SVD_CONFIG
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    with torch.device("meta"):
        m = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
    if which == "scripted":                    # train_svd.py:761-766
        m.requires_grad_(False)
        for n, p in m.named_parameters():
            if "temporal_transformer_block" in n:
                p.requires_grad_(True)
    return m


@pytest.mark.parametrize("which", ["scripted", "whole"])
def test_default_arena_offsets_are_the_64_element_rule(which):
    from svd_xtend_b200.train import ParamArena
    m = _svd_params(which)
    ps = [p for p in m.parameters() if p.requires_grad]
    sizes = [p.numel() for p in ps]
    for pad_to in (64, 8 * 64):
        arena = ParamArena(m, pad_to=pad_to)
        off, want = 0, []
        for n in sizes:
            want.append(off)
            off += (n + 63) // 64 * 64
        assert arena.offsets == want
        assert arena.numel == (off + pad_to - 1) // pad_to * pad_to


def _check_sharding(net, world, min_8bit_size=4096):
    """every quantisation block in one shard; each parameter's sub-jobs over the ranks cover it once, 8-bit ones in whole blocks;
    sub-job state / absmax indices equal FusedAdamW8bit's; the ranks' state ranges tile the unsharded buffers"""
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena, ShardedAdamW8bit
    arena = ParamArena(net, pad_to=world * 256, block=256)
    assert arena.numel % (world * 256) == 0
    shard = arena.numel // world
    ref = FusedAdamW8bit(arena, min_8bit_size=min_8bit_size)          # the unsharded layout over the same arena
    opt = ShardedAdamW8bit(arena, min_8bit_size=min_8bit_size)        # world 1 here; the ranks' sub-jobs come from _subjobs
    assert opt.layout == ref.layout
    by_param = {}
    ranges = []
    for r in range(world):
        jobs, rng = opt._subjobs(r * shard, (r + 1) * shard)
        ranges.append(rng)
        for p, a, n, quant, si, bi in jobs:
            assert r * shard <= a and a + n <= (r + 1) * shard
            by_param.setdefault(p, []).append((a, n, quant, si, bi))
    for p, off, quant, so, bo in ref.layout:
        n = p.numel()
        assert quant == (n >= min_8bit_size)
        if quant:
            assert off % 256 == 0
            for k in range((n + 255) // 256):
                s, e = off + 256 * k, min(off + 256 * (k + 1), off + n)
                assert s // shard == (e - 1) // shard              # the block lies in one shard
        subs = sorted(by_param[p])
        pos = off
        for a, m, q, si, bi in subs:
            assert a == pos and q == quant
            assert si == so + (a - off)                            # state index into the unsharded buffers
            if quant:
                assert (a - off) % 256 == 0 and bi == bo + (a - off) // 256
                assert a + m == off + n or m % 256 == 0            # whole blocks, the last may be partial
            else:
                assert (a - off) % 64 == 0
            pos = a + m
        assert pos == off + n
    # the owned ranges of the unsharded code / absmax / fp32 buffers tile them in rank order
    totals = (ref.codes1.numel(), ref.absmax1.numel(), ref.m32.numel())
    for k in range(3):
        spans = [rng[k] for rng in ranges if rng[k] != (0, 0)]
        assert sum(y - x for x, y in spans) == totals[k]
        for (x0, y0), (x1, y1) in zip(spans, spans[1:]):
            assert y0 == x1
    return arena, by_param


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("which", ["scripted", "whole"])
def test_svd_parameter_lists_shard_on_block_boundaries(world, which):
    _check_sharding(_svd_params(which), world)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("min_8bit_size", [4096, 1])
def test_hand_made_sizes_and_a_parameter_across_every_boundary(world, min_8bit_size):
    sizes = [256, 257, 4096, 100, 300_000 + 77, 33]
    net = _Net(sizes)
    arena, by_param = _check_sharding(net, world, min_8bit_size)
    big = net.ps[4]
    off = arena.offset_of[big]
    shard = arena.numel // world
    for r in range(1, world):
        assert off < r * shard < off + big.numel()                 # the big parameter straddles every shard boundary
    assert len(by_param[big]) == world


def test_block_alignment_leaves_views_and_the_fused_layout_alone():
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena
    sizes = [1, 255, 256, 257, 4095, 4096, 4097, 70000, 513]
    a64, a256 = ParamArena(_Net(sizes)), ParamArena(_Net(sizes), block=256)
    assert all(o % 256 == 0 for o in a256.offsets)
    l64, l256 = FusedAdamW8bit(a64).layout, FusedAdamW8bit(a256).layout
    assert [x[2:] for x in l64] == [x[2:] for x in l256]           # same state and absmax offsets, only arena offsets move
    with pytest.raises(ValueError, match="multiple of 64"):
        ParamArena(_Net(sizes), block=96)


@pytest.mark.parametrize("cls", ["ShardedAdamW8bit", "P2PShardedAdamW8bit"])
def test_misbuilt_arena_is_refused_with_the_constructor_to_use(cls):
    from svd_xtend_b200 import train
    sizes = [5000, 10, 70000]
    for arena in (train.ParamArena(_Net(sizes)), train.ParamArena(_Net(sizes), pad_to=256)):
        with pytest.raises(ValueError, match=r"ParamArena\(\.\.\., pad_to=256, block=256\)"):
            getattr(train, cls)(arena)


def test_cpu_state_dict_and_load_round_trip_at_world_one():
    from svd_xtend_b200.train import FusedAdamW8bit, ParamArena, ShardedAdamW8bit
    sizes = [5000, 10, 70000, 300]
    g = torch.Generator().manual_seed(0)
    fused = FusedAdamW8bit(ParamArena(_Net(sizes), pad_to=256, block=256))
    for x in fused.snapshot_tensors()[1:7]:
        x.copy_((torch.rand(x.shape, generator=g) * 200).to(x.dtype))
    sd = fused.state_dict()
    sharded = ShardedAdamW8bit(ParamArena(_Net(sizes), pad_to=256, block=256))
    sharded.load_state_dict(sd)
    sd2 = sharded.state_dict()
    assert sd2["param_groups"] == sd["param_groups"]
    for i in sd["state"]:
        assert list(sd2["state"][i]) == list(sd["state"][i])
        for k, v in sd["state"][i].items():
            assert torch.equal(v, sd2["state"][i][k]) if isinstance(v, torch.Tensor) else v == sd2["state"][i][k]
    bad = {**sd, "state": {**sd["state"], 0: {**sd["state"][0], "absmax1": torch.zeros(3)}}}
    before = [t.clone() for t in sharded.snapshot_tensors()]
    with pytest.raises(ValueError, match="absmax1"):
        sharded.load_state_dict(bad)
    assert all(torch.equal(a, b) for a, b in zip(before, sharded.snapshot_tensors()))


def test_abi_rejects_bad_p2p_arguments():
    from svd_xtend_b200 import build
    build.build()
    from svd_xtend_b200 import _lib
    lib = _lib.load()
    buf = (ctypes.c_double * 64)()
    a = ctypes.addressof(buf)
    arenas = (ctypes.c_void_p * 2)(a, a)
    null_peer = (ctypes.c_void_p * 2)(a, None)
    odd_peer = (ctypes.c_void_p * 2)(a, a + 8)

    def call(jobs=a, prefix=a, njobs=1, blocks=1, q1=a, q2=a, grads=arenas, shadows=arenas, world=2, state=a, ema_state=None,
             grad_mul=None):
        return lib.svdx_adamw8bit_p2p(jobs, prefix, njobs, blocks, q1, q2, grads, shadows, world, state, 0.5, 1, ema_state,
                                      grad_mul, None)

    for kw in (dict(jobs=None), dict(prefix=None), dict(q1=None), dict(q2=None), dict(state=None), dict(grads=None),
               dict(shadows=None), dict(njobs=0), dict(blocks=0), dict(world=0), dict(world=17), dict(jobs=a + 4),
               dict(prefix=a + 2), dict(ema_state=a + 4), dict(grad_mul=a + 2)):
        assert call(**kw) == -1, kw
        assert b"adamw8bit_p2p" in lib.svdx_last_error()
    for kw in (dict(grads=null_peer), dict(shadows=null_peer), dict(grads=odd_peer), dict(shadows=odd_peer)):
        assert call(**kw) == -1, kw
        assert b"peer arena" in lib.svdx_last_error()
