"""Frame-size rules at the public boundary (no GPU needed): the UNet and the VAE encoder take any latent / frame whose height
and width are multiples of 2^(levels - 1), and refuse every other size with a ValueError before any launch."""
import pytest
import torch

from oracle.svd_unet_oracle import TINY_CONFIG


def _unet():
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    return UNetSpatioTemporalConditionModel(**TINY_CONFIG)


@pytest.mark.parametrize("h,w", [(16, 15), (15, 16), (9, 24)])
def test_unet_refuses_a_latent_the_skips_cannot_line_up(h, w):
    m = _unet()      # 2 down blocks: multiples of 2
    with pytest.raises(ValueError, match=r"multiples of 2\^\(number of down blocks - 1\) = 2"):
        m(torch.zeros(1, 2, 8, h, w), torch.zeros(1), torch.zeros(1, 1, 64), torch.zeros(1, 3))


@pytest.mark.parametrize("h,w", [(16, 24), (16, 18), (10, 6)])
def test_unet_valid_sizes_still_reach_the_device_check(h, w):
    m = _unet()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(1, 2, 8, h, w), torch.zeros(1), torch.zeros(1, 1, 64), torch.zeros(1, 3))


def test_svd_topology_rule_is_8():
    from oracle.svd_unet_oracle import SVD_CONFIG
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
    with torch.device("meta"):
        m = UNetSpatioTemporalConditionModel(**SVD_CONFIG)
    with pytest.raises(ValueError, match="= 8"):
        m._check_latent_size(torch.zeros(1, 1, 8, 64, 36, device="meta"))
    for h, w in ((64, 40), (128, 72), (96, 96), (80, 48)):       # 512x320, 1024x576, 768x768, 640x384 frames
        m._check_latent_size(torch.zeros(1, 1, 8, h, w, device="meta"))


def test_vae_encode_frame_size_rule():
    from oracle.svd_vae_oracle import TINY_VAE_CONFIG
    from svd_xtend_b200.vae import AutoencoderKLTemporalDecoder
    m = AutoencoderKLTemporalDecoder(**TINY_VAE_CONFIG)
    f = 1 << (len(TINY_VAE_CONFIG["block_out_channels"]) - 1)
    with pytest.raises(ValueError, match=f"multiples of 2\\^\\(levels - 1\\) = {f}"):
        m.encode(torch.zeros(1, 3, 4 * f, 3 * f + 1))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.encode(torch.zeros(1, 3, 4 * f, 5 * f))        # a width neither dividing nor divided by 128 passes the boundary
