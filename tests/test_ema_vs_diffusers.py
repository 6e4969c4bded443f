"""A/B of oracle/svd_ema_oracle.py against the REAL diffusers.training_utils.EMAModel — runs wherever `diffusers` is
importable, skips elsewhere (diffusers is not installable offline). Pins the decay sequence, the shadows after N steps on
mixed trainable / frozen tensors, and the state_dict keys, for every schedule the CPU tests use."""
import pytest
import torch

diffusers = pytest.importorskip("diffusers", reason="diffusers is not installed on this box: the EMA oracle cannot be A/B-ed against it here")

from test_ema import CONFIGS  # noqa: E402


@pytest.mark.parametrize("name", list(CONFIGS))
def test_ema_oracle_matches_diffusers(name):
    from diffusers.training_utils import EMAModel as Real
    from oracle.svd_ema_oracle import EMAModel as Oracle
    kw = CONFIGS[name]
    torch.manual_seed(7)
    params = [torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(4), requires_grad=False), torch.nn.Parameter(torch.randn(9))]
    real, ora = Real(params, **kw), Oracle(params, **kw)
    assert set(real.state_dict()) == set(ora.state_dict())
    for t in range(1, 40):
        assert real.get_decay(t) == ora.get_decay(t), t
    for _ in range(12):
        with torch.no_grad():
            for p in params:
                p.add_(0.1 * torch.randn_like(p))
        real.step(params)
        ora.step(params)
        assert real.cur_decay_value == ora.cur_decay_value
        for a, b in zip(real.shadow_params, ora.shadow_params):
            assert torch.equal(a, b)
    sr, so = real.state_dict(), ora.state_dict()
    assert {k: v for k, v in sr.items() if k != "shadow_params"} == {k: v for k, v in so.items() if k != "shadow_params"}
