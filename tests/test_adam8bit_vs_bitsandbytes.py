"""A/B against bitsandbytes wherever a real bitsandbytes is installed (skipped otherwise, and on the shim's stand-in): the two
quantisation maps equal `bitsandbytes.functional.create_dynamic_map`, and a few AdamW8bit steps of the drop-in stay close to
`bnb.optim.AdamW8bit` on the same parameters and gradients. The step is compared within a tolerance, not bit for bit:
bitsandbytes arranges the update algebra differently (its kernel fuses operations the oracle rounds separately)."""
import pytest
import torch

bnb = pytest.importorskip("bitsandbytes")
if getattr(bnb, "__svdx_standin__", False):
    pytest.skip("the shim's stand-in, not bitsandbytes", allow_module_level=True)


@pytest.mark.parametrize("signed", [True, False])
def test_maps_equal_bitsandbytes(signed):
    from bitsandbytes.functional import create_dynamic_map
    from svd_xtend_b200.optim8bit import dynamic_map
    assert torch.equal(dynamic_map(signed), create_dynamic_map(signed=signed).float().cpu())


@pytest.mark.gpu
def test_steps_track_bitsandbytes():
    from svd_xtend_b200.optim8bit import AdamW8bit
    torch.manual_seed(0)
    ref = [torch.nn.Parameter(torch.randn(n, device="cuda")) for n in (70000, 4096, 100)]
    ours = [torch.nn.Parameter(p.detach().clone()) for p in ref]
    o_ref = bnb.optim.AdamW8bit(ref, lr=1e-3)
    o_ours = AdamW8bit(ours, lr=1e-3)
    for _ in range(5):
        for a, b in zip(ref, ours):
            g = torch.randn_like(a)
            a.grad, b.grad = g.clone(), g.clone()
        o_ref.step()
        o_ours.step()
    torch.cuda.synchronize()
    for a, b in zip(ref, ours):
        assert (a - b).abs().max().item() < 1e-4
