"""The temporal decode's frame-size rule at the public boundary (no GPU needed): a decoder level at least 32 pixels wide takes
any width; a narrower level needs W | 128 (and, if it is upsampled, H*W % 32 == 0). Sizes the rule accepts get past it and
stop at the device check."""
import pytest
import torch


def _svd_vae():
    from oracle.svd_vae_oracle import VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    with torch.device("meta"):
        return AutoencoderKLTemporalDecoder(**VAE_CONFIG, with_decoder=True).requires_grad_(False)


@pytest.mark.parametrize("h,w", [(64, 40), (128, 72), (96, 96), (80, 48), (40, 64), (72, 128)])
def test_svd_decode_portrait_square_and_landscape_reach_the_device_check(h, w):
    """512x320 / 1024x576 portrait, 768x768 square, 640x384 portrait; 320x512 / 576x1024 landscape as before"""
    m = _svd_vae()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.decode(torch.zeros(2, 4, h, w, device="meta"), num_frames=2)


@pytest.mark.parametrize("h,w", [(6, 36), (10, 40), (3, 33), (5, 48), (4, 72)])
def test_tiny_decode_row_crossing_widths_reach_the_device_check(h, w):
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    m = AutoencoderKLTemporalDecoder(**TINY_VAE_CONFIG, with_decoder=True).requires_grad_(False)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.decode(torch.zeros(2, 4, h, w), num_frames=2)


def test_unet_sized_latents_decode_at_every_width_but_24():
    """latents with sides that are multiples of 8 (every size the UNet takes), up to 160: only the 24-wide latent
    (192-pixel-wide frames) is refused"""
    m = _svd_vae()
    refused = []
    for h in range(8, 161, 8):
        for w in range(8, 161, 8):
            try:
                m.decode(torch.zeros(1, 4, h, w, device="meta"), num_frames=1)
            except ValueError as e:
                assert "128" in str(e), (h, w, str(e))
                refused.append((h, w))
            except RuntimeError as e:
                assert "CUDA" in str(e), (h, w, str(e))
    assert refused == [(h, 24) for h in range(8, 161, 8)]
