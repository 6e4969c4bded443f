"""ORACLE — test infrastructure only. The crop-box form of oracle/svd_resize_oracle.py: what Pillow's
`Image.resize((W, H), box=(x0, y0, x1, y1))` returns for an RGB uint8 image with its default BICUBIC filter, in numpy integer
arithmetic. The tests of the mixed-size uint8 input (svd_xtend_b200.video_train) hold the library's box taps and the GPU resize
to it, and it to Pillow's recorded outputs (tests/golden/resize_box_golden.pt).

    taps_box(in_size, out_size, lo, hi) -> (first source index [out], tap count [out], int64 fixed-point weights [out, ksize])
    resize_box(img, (W, H), box=None)    -> uint8 [H, W, 3], bit for bit Image.resize((W, H), box=box)

Pillow keeps the box in fp32. An axis is resampled when `out != in or lo != 0 or hi != in` and copied otherwise; with the box
(0, in) the taps are those of oracle/svd_resize_oracle.py's `taps(in, out)`.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.svd_resize_oracle import PRECISION_BITS, _clip8, bicubic


def taps_box(in_size: int, out_size: int, lo: float, hi: float):
    """precompute_coeffs over the box [lo, hi) (fp32 bounds) + normalize_coeffs_8bpc"""
    lo, hi = np.float32(lo), np.float32(hi)
    scale = float(hi - lo) / out_size                          # the extent in fp32, the scale in double
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    first = np.zeros(out_size, np.int64)
    cnt = np.zeros(out_size, np.int64)
    k = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = float(lo) + (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)             # C casts truncate toward zero
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = bicubic((np.arange(xmax) + xmin - center + 0.5) * ss)
        ww = 0.0
        for v in w:                                            # the sum in Pillow's order
            ww += float(v)
        if ww != 0.0:
            w = w / ww
        fixed = np.where(w < 0, np.trunc(-0.5 + w * (1 << PRECISION_BITS)), np.trunc(0.5 + w * (1 << PRECISION_BITS)))
        first[xx], cnt[xx] = xmin, xmax
        k[xx, :xmax] = fixed.astype(np.int64)
    return first, cnt, k


def _pass(img: np.ndarray, out_size: int, axis: int, lo: float, hi: float) -> np.ndarray:
    """one 8-bpc pass along axis (1: horizontal, 0: vertical) of an [H, W, 3] uint8 image over the box [lo, hi)"""
    first, cnt, k = taps_box(img.shape[axis], out_size, lo, hi)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((out_size,) + src.shape[1:], np.uint8)
    for o in range(out_size):
        seg = src[first[o]:first[o] + cnt[o]]
        acc = (1 << (PRECISION_BITS - 1)) + np.tensordot(k[o, :cnt[o]], seg, axes=(0, 0))
        out[o] = _clip8(acc)
    return np.moveaxis(out, 0, axis)


def check_box(box, H0: int, W0: int):
    """the box in fp32, or ValueError with Pillow's message for a box Pillow refuses (plus a non-finite one)"""
    x0, y0, x1, y1 = (np.float32(v) for v in box)
    if not all(np.isfinite(v) for v in (x0, y0, x1, y1)):
        raise ValueError("box must be finite")
    if x0 < 0 or y0 < 0:
        raise ValueError("box offset can't be negative")
    if x1 > W0 or y1 > H0:
        raise ValueError("box can't exceed original image size")
    if x1 - x0 < 0 or y1 - y0 < 0:
        raise ValueError("box can't be empty")
    return x0, y0, x1, y1


def resize_box(img: np.ndarray, size, box=None) -> np.ndarray:
    """Image.fromarray(img).resize(size, box=box) for an RGB uint8 img [H0, W0, 3] and size = (W, H): the horizontal pass first
    (into a uint8 intermediate), then the vertical one, each only where Pillow runs it"""
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"resize_box: expected a uint8 [H, W, 3] RGB image, got {img.dtype} {img.shape}")
    H0, W0 = img.shape[:2]
    W, H = (int(v) for v in size)
    x0, y0, x1, y1 = check_box((0, 0, W0, H0) if box is None else box, H0, W0)
    out = img
    if W != W0 or x0 != 0 or x1 != W0:
        out = _pass(out, W, 1, x0, x1)
    if H != H0 or y0 != 0 or y1 != H0:
        out = _pass(out, H, 0, y0, y1)
    return out.copy()
