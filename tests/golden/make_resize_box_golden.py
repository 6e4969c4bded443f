"""Generates tests/golden/resize_box_golden.pt: what Pillow's Image.resize((W, H), box=...) returns for seeded RGB frames of mixed
sizes, with and without crop boxes, with its default filter (BICUBIC).

    python tests/golden/make_resize_box_golden.py            (needs Pillow)

Each case stores its name, the seed and source size [H0, W0] of its input (oracle/svd_resize_oracle.py's `source_frame`
regenerates it), the target size [H, W], the box (x0, y0, x1, y1) or None, the clip it belongs to (or -1) and Pillow's uint8
output in `pack_image`'s lossless form. The cases of clips 0, 1 and 2 are two frames each of three clips of different source sizes
resized to one training size, 64 x 128: the GPU test resizes them in one launch. The others cover the axis rules one at a time.
tests/test_frames_mixed.py holds tests/resize_box_oracle.py to these outputs bit for bit, and tests/test_frames_mixed_gpu.py the
kernel.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.svd_resize_oracle import pack_image, source_frame, unpack_image  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resize_box_golden.pt")

# name, seed, (H0, W0), (H, W), box, clip
CASES = (
    ("clip0_down_250x150_f0", 11, (150, 250), (64, 128), None, 0),
    ("clip0_down_250x150_f1", 12, (150, 250), (64, 128), None, 0),
    ("clip1_up_fractional_box_96x40_f0", 21, (40, 96), (64, 128), (3.5, 2.25, 90.75, 39.5), 1),
    ("clip1_up_fractional_box_96x40_f1", 22, (40, 96), (64, 128), (3.5, 2.25, 90.75, 39.5), 1),
    ("clip2_down_aspect_crop_300x200_f0", 31, (200, 300), (64, 128), (22, 0, 278, 128), 2),
    ("clip2_down_aspect_crop_300x200_f1", 32, (200, 300), (64, 128), (22, 0, 278, 128), 2),
    ("width_only_300x64_to_128x64", 41, (64, 300), (64, 128), None, -1),
    ("height_kept_fractional_y_box_200x64", 42, (64, 200), (64, 128), (0, 0.5, 200, 64), -1),
    ("height_kept_zero_offset_short_box_200x64", 43, (64, 200), (64, 128), (0, 0, 200, 61), -1),
    ("box_equal_to_frame_160x90", 44, (90, 160), (64, 128), (0, 0, 160, 90), -1),
    ("integer_crop_of_output_size_200x100", 45, (100, 200), (64, 128), (10, 20, 138, 84), -1),
    ("fractional_crop_of_output_size_200x100", 46, (100, 200), (64, 128), (10.5, 20.25, 138.5, 84.25), -1),
    ("identity_with_full_box_128x64", 47, (64, 128), (64, 128), (0, 0, 128, 64), -1),
    ("down_box_both_offsets_333x187", 48, (187, 333), (64, 128), (17.3, 9.6, 301.9, 180.1), -1),
)


def main():
    import PIL
    from PIL import Image
    cases = []
    for name, seed, (H0, W0), (H, W), box, clip in CASES:
        img = Image.fromarray(source_frame(seed, H0, W0).numpy())
        out = np.asarray(img.resize((W, H), box=box))
        packed = pack_image(out)
        assert np.array_equal(unpack_image(packed, out.shape), out)
        cases.append(dict(name=name, seed=seed, source=[H0, W0], size=[H, W], box=None if box is None else [float(v) for v in box],
                          clip=clip, out=packed))
    torch.save(dict(pillow=PIL.__version__, cases=cases), OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, Pillow {PIL.__version__})")


if __name__ == "__main__":
    main()
