"""Generates tests/golden/resize_golden.pt: what Pillow's Image.resize((W, H)) returns for seeded RGB frames, with its default
filter (BICUBIC), the resize train_svd.py's DummyDataset applies to every frame.

    python tests/golden/make_resize_golden.py            (needs Pillow)

Each case stores its name, the seed and source size [H0, W0] of its input (oracle/svd_resize_oracle.py's `source_frame`
regenerates it), the target size [H, W] and Pillow's uint8 output [H, W, 3] in `pack_image`'s lossless form (row differences,
deflated; `unpack_image` restores it), which keeps the file near 100 kB. tests/test_frames_u8.py holds
oracle/svd_resize_oracle.py to these outputs bit for bit, and tests/test_frames_u8_gpu.py the kernel.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.svd_resize_oracle import pack_image, source_frame, unpack_image  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resize_golden.pt")

# name, seed, (H0, W0), (H, W)
CASES = (
    ("down_640x360_to_512x320", 1, (360, 640), (320, 512)),
    ("down_non_integer_333x187_to_128x64", 2, (187, 333), (64, 128)),
    ("up_256x144_to_512x320", 3, (144, 256), (320, 512)),
    ("width_only_300x200_to_128x200", 4, (200, 300), (200, 128)),
    ("height_only_160x250_to_160x96", 5, (250, 160), (96, 160)),
    ("down_width_up_height_200x60_to_64x128", 6, (60, 200), (128, 64)),
    ("identity_96x64", 7, (64, 96), (64, 96)),
)


def main():
    import PIL
    from PIL import Image
    cases = []
    for name, seed, (H0, W0), (H, W) in CASES:
        img = Image.fromarray(source_frame(seed, H0, W0).numpy())
        out = np.asarray(img.resize((W, H)))
        packed = pack_image(out)
        assert np.array_equal(unpack_image(packed, out.shape), out)
        cases.append(dict(name=name, seed=seed, source=[H0, W0], size=[H, W], out=packed))
    torch.save(dict(pillow=PIL.__version__, cases=cases), OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, Pillow {PIL.__version__})")


if __name__ == "__main__":
    main()
