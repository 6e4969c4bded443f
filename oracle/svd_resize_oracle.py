"""ORACLE — test infrastructure only. Numpy restatement of what train_svd.py's DummyDataset does to a decoded RGB frame
(`img.resize((width, height))`, then `float() / 127.5 - 1`): Pillow's 8-bpc BICUBIC resample (libImaging/Resample.c,
`precompute_coeffs`, `normalize_coeffs_8bpc`, `ImagingResampleHorizontal_8bpc` / `ImagingResampleVertical_8bpc`) in integer
arithmetic, and the fp32 normalisation. What svd_xtend_b200's svdx_frames_u8_in computes before the encoder rows.

    taps(in_size, out_size)            -> (first source index [out], tap count [out], int64 fixed-point weights [out, ksize])
    resize(img, (W, H))                -> uint8 [H, W, 3], bit for bit Image.resize((W, H)) of an RGB image
    normalize(u8)                      -> fp32 fl(fl(u / 127.5f) - 1)
    source_frame(seed, H0, W0)         -> the seeded uint8 input [H0, W0, 3] of a case of tests/golden/resize_golden.pt
    pack_image / unpack_image          -> the compressed form in which that file stores each uint8 output
"""
from __future__ import annotations

import math
import zlib

import numpy as np
import torch

PRECISION_BITS = 32 - 8 - 2


def bicubic(x: np.ndarray) -> np.ndarray:
    """bicubic_filter, a = -0.5, evaluated in double with Pillow's operation order"""
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def taps(in_size: int, out_size: int):
    """precompute_coeffs over the box [0, in_size) + normalize_coeffs_8bpc"""
    scale = float(np.float32(in_size)) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    lo = np.zeros(out_size, np.int64)
    cnt = np.zeros(out_size, np.int64)
    k = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
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
        lo[xx], cnt[xx] = xmin, xmax
        k[xx, :xmax] = fixed.astype(np.int64)
    return lo, cnt, k


def _clip8(acc: np.ndarray) -> np.ndarray:
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def _pass(img: np.ndarray, out_size: int, axis: int) -> np.ndarray:
    """one 8-bpc pass along axis (1: horizontal, 0: vertical) of an [H, W, 3] uint8 image"""
    lo, cnt, k = taps(img.shape[axis], out_size)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((out_size,) + src.shape[1:], np.uint8)
    for o in range(out_size):
        seg = src[lo[o]:lo[o] + cnt[o]]
        acc = (1 << (PRECISION_BITS - 1)) + np.tensordot(k[o, :cnt[o]], seg, axes=(0, 0))
        out[o] = _clip8(acc)
    return np.moveaxis(out, 0, axis)


def resize(img: np.ndarray, size) -> np.ndarray:
    """Image.fromarray(img).resize(size) for an RGB uint8 img [H0, W0, 3] and size = (W, H): the horizontal pass first (into a
    uint8 intermediate), then the vertical one; a pass is skipped where that side is unchanged, the image returned as is when
    both are"""
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"resize: expected a uint8 [H, W, 3] RGB image, got {img.dtype} {img.shape}")
    W, H = (int(v) for v in size)
    out = img
    if W != img.shape[1]:
        out = _pass(out, W, 1)
    if H != img.shape[0]:
        out = _pass(out, H, 0)
    return out.copy()


def normalize(u8: np.ndarray) -> np.ndarray:
    """DummyDataset's `torch.tensor(np.array(img)).float() / 127.5 - 1`, rounded in fp32 after each operation"""
    return (u8.astype(np.float32) / np.float32(127.5)) - np.float32(1.0)


def source_frame(seed: int, H0: int, W0: int) -> torch.Tensor:
    """the seeded uint8 RGB frame [H0, W0, 3] of a golden case (tests/golden/make_resize_golden.py), built in integer arithmetic
    only so that every machine regenerates the same bytes: per channel a folded linear ramp (smooth gradients and creases), six
    saturated rectangles (sharp edges, whose bicubic overshoot is clamped to 0 / 255) and one patch of uniform noise"""
    g = torch.Generator().manual_seed(seed)

    def r(lo, hi, n=()):
        return torch.randint(lo, hi, n, generator=g, dtype=torch.int64)
    y = torch.arange(H0).view(H0, 1, 1)
    x = torch.arange(W0).view(1, W0, 1)
    t = (r(-6, 7, (3,)) * y + r(-6, 7, (3,)) * x + r(0, 512, (3,))) % 512
    img = torch.where(t < 256, t, 511 - t)
    for _ in range(6):
        y0, x0 = int(r(0, H0)), int(r(0, W0))
        img[y0:y0 + int(r(1, H0 // 3 + 2)), x0:x0 + int(r(1, W0 // 3 + 2))] = r(0, 2, (3,)) * 255
    y0, x0 = int(r(0, max(1, H0 - H0 // 6))), int(r(0, max(1, W0 - W0 // 6)))
    ph, pw = min(H0 // 6 + 1, H0 - y0), min(W0 // 6 + 1, W0 - x0)
    img[y0:y0 + ph, x0:x0 + pw] = r(0, 256, (ph, pw, 3))
    return img.to(torch.uint8)


def pack_image(img: np.ndarray) -> torch.Tensor:
    """uint8 [H, W, 3] -> the stored form of a golden output: each row's differences of neighbouring pixels (mod 256, the first
    pixel as is), deflated; a uint8 tensor of the compressed bytes"""
    d = img.astype(np.uint8).copy()
    d[:, 1:] = img[:, 1:] - img[:, :-1]
    return torch.frombuffer(bytearray(zlib.compress(d.tobytes(), 9)), dtype=torch.uint8)


def unpack_image(packed: torch.Tensor, shape) -> np.ndarray:
    """inverse of pack_image: the uint8 image of `shape` [H, W, 3]"""
    d = np.frombuffer(zlib.decompress(packed.numpy().tobytes()), dtype=np.uint8).reshape(tuple(shape))
    return np.cumsum(d, axis=1, dtype=np.uint8)
