"""raw.wgrad_plan: the (tile width, token split) of a weight-gradient launch, on the CPU with the H100's 132 SMs."""
import pytest

from svd_xtend_b200 import raw

# (O, K, M) of the weight gradients of the config-2 step: the temporal transformer blocks' projections at the four UNet
# levels (q|k|v fused, GEGLU proj, ff out, ...), and rank-64 LoRA factors of config 5
SHAPES = [(O, K, M) for M in (35840, 8960, 2240, 560) for C in (320, 640, 1280) for O, K in
          ((C, C), (3 * C, C), (8 * C, C), (C, 4 * C), (4 * C, C))] + \
         [(64, 320, 35840), (320, 64, 35840), (64, 1280, 2240), (1280, 64, 2240), (64, 64, 560)]


@pytest.fixture(autouse=True)
def h100_sms(monkeypatch):
    monkeypatch.setattr(raw, "_NUM_SMS", [132])


@pytest.mark.parametrize("O,K,M", SHAPES)
def test_plan_is_a_launch_the_library_runs(O, K, M):
    bn, split = raw.wgrad_plan(O, K, M)
    assert bn in (64, 128)                      # MN-major B: 64-column boxes, at most 128 columns per tile
    n_tiles = -(-K // bn)
    assert n_tiles * bn >= K > (n_tiles - 1) * bn   # every column covered, no empty tile
    kb = -(-M // 64)
    assert 1 <= split <= kb
    kb_per_split = -(-kb // split)
    assert -(-kb // kb_per_split) == split      # no split the library would drop as empty


@pytest.mark.parametrize("O,K,M", [(64, 64, 560), (320, 64, 35840), (1280, 64, 2240)])
def test_narrow_shapes_keep_64(O, K, M):
    assert raw.wgrad_plan(O, K, M)[0] == 64


def test_long_contraction_fills_the_sms():
    """GEGLU proj at level 0 (dW [2560, 320] over 35,840 tokens): 60 tiles of 128 x 128 leave most SMs idle, so the
    tokens are split until the CTAs cover the SMs"""
    bn, split = raw.wgrad_plan(2560, 320, 35840)
    tiles = 20 * -(-320 // bn)
    assert tiles * split >= 120
