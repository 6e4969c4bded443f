"""A/B of the temporal VAE decoder oracle (oracle/svd_vae_decoder_oracle.py) against the REAL diffusers
AutoencoderKLTemporalDecoder — runs wherever `diffusers` is importable, skips loudly elsewhere (the decoder restatement then
stays "parity unpinned", like the UNet and encoder oracles; SURVEY.md Appendix D lists the recalled items it would pin).

Same seeded state dict (norms, biases and the AlphaBlender mix factors perturbed so that every term shows) loaded strictly
into both, the same latents decoded as clips of T frames on the CPU in fp32; tolerance 1e-5 rel-L2."""
import pytest
import torch

diffusers = pytest.importorskip("diffusers", reason="diffusers is not installed on this box: the decoder oracle cannot be A/B-ed "
                                                    "against it here (parity stays UNPINNED)")


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.mark.parametrize("layers", [1, 2])
def test_decoder_matches_diffusers(layers):
    from diffusers import AutoencoderKLTemporalDecoder as Real
    from oracle.svd_vae_decoder_oracle import AutoencoderKLTemporalDecoder as Oracle
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    cfg = dict(TINY_VAE_CONFIG, layers_per_block=layers)
    torch.manual_seed(20261015)
    ora = Oracle(**cfg, with_decoder=True).eval()
    with torch.no_grad():
        for n, p in ora.named_parameters():
            if "norm" in n or n.endswith("bias") or n.endswith("mix_factor"):
                p.add_(0.1 * torch.randn_like(p))
    real = Real(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * len(cfg["block_out_channels"]),
                block_out_channels=cfg["block_out_channels"], layers_per_block=layers, latent_channels=4).eval()
    assert sorted(real.state_dict()) == sorted(ora.state_dict())
    real.load_state_dict(ora.state_dict(), strict=True)
    eps_real = {n: m.eps for n, m in real.named_modules() if isinstance(m, torch.nn.GroupNorm)}
    assert eps_real == {n: m.eps for n, m in ora.named_modules() if isinstance(m, torch.nn.GroupNorm)}
    z = torch.randn(2 * 3, 4, 8, 8)
    with torch.no_grad():
        a = real.decode(z, num_frames=3).sample
        b = ora.decode(z, num_frames=3).sample
    e = _rel(b, a)
    print("decoder oracle vs diffusers", diffusers.__version__, "rel-l2", e)
    assert e < 1e-5, e
