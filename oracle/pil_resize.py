"""Pillow's BILINEAR resize of a uint8 RGB image, restated in numpy (Pillow's src/libImaging/Resample.c, 8 bits per
channel) — what learning/utils/wrappers.py:39-54's ResizeWrapper computes through scipy.misc.imresize, and the
reference the device pass (k_resize_pil) is compared with at any shape, without Pillow.

Per axis, `inp` source pixels -> `out` output pixels, in double:
    scale = inp / out, fs = max(scale, 1), support = fs, ksize = 2 * ceil(support) + 1
    center = (i + 0.5) * scale, xmin = max(0, (int)(center - support + 0.5)), xmax = min(inp, (int)(center + support + 0.5))
    w_k = tri((k + xmin - center + 0.5) * (1 / fs)) for k < xmax - xmin, tri(t) = max(0, 1 - |t|); w /= sum(w)
    fixed point: (int)(0.5 + w * 2^22)
A pass: acc = 2^21 + sum px * w (int32), u8 = 0 if acc <= 0, 255 if acc >= 255 << 22, else acc >> 22.  The
horizontal pass runs first, the vertical one on its uint8 output; an axis that keeps its size is an exact copy.
"""
from __future__ import annotations

import hashlib
import math

import numpy as np

PRECISION_BITS = 22


def axis_coeffs(inp: int, out: int):
    """(xmin[out], weights int64[out][ksize]) of one axis; weights past a pixel's own count are zero."""
    scale = inp / out
    fs = max(scale, 1.0)
    support, ss = fs, 1.0 / fs
    ksize = int(math.ceil(support)) * 2 + 1
    xmins = np.zeros(out, np.int64)
    kk = np.zeros((out, ksize), np.int64)
    for i in range(out):
        center = (i + 0.5) * scale
        xmin = max(0, int(center - support + 0.5))
        xmax = min(inp, int(center + support + 0.5))
        w = []
        for x in range(xmax - xmin):
            t = abs((x + xmin - center + 0.5) * ss)
            w.append(1.0 - t if t < 1.0 else 0.0)
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        xmins[i] = xmin
        kk[i, :len(w)] = [int(0.5 + v * (1 << PRECISION_BITS)) for v in w]
    return xmins, kk


def _pass(img: np.ndarray, out: int, axis: int) -> np.ndarray:
    inp = img.shape[axis]
    xmins, kk = axis_coeffs(inp, out)
    idx = np.minimum(xmins[:, None] + np.arange(kk.shape[1])[None, :], inp - 1)   # zero taps past the edge: any index
    src = np.take(img.astype(np.int64), idx, axis=axis)                          # axis -> (out, ksize)
    wshape = [1] * src.ndim
    wshape[axis], wshape[axis + 1] = kk.shape
    acc = (1 << (PRECISION_BITS - 1)) + (src * kk.reshape(wshape)).sum(axis=axis + 1)
    return np.where(acc <= 0, 0, np.where(acc >= 255 << PRECISION_BITS, 255, acc >> PRECISION_BITS)).astype(np.uint8)


def resize(img: np.ndarray, out_w: int, out_h: int) -> np.ndarray:
    """PIL.Image.fromarray(img).resize((out_w, out_h), BILINEAR) of u8 [..., H, W, 3] (leading axes: a batch)."""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim < 3 or img.shape[-1] != 3:
        raise ValueError("expects uint8 [..., H, W, 3]")
    h_ax, w_ax = img.ndim - 3, img.ndim - 2
    if img.shape[w_ax] != out_w:
        img = _pass(img, out_w, w_ax)
    if img.shape[h_ax] != out_h:
        img = _pass(img, out_h, h_ax)
    return np.ascontiguousarray(img)


def imresize_standin(arr, size, interp="bilinear", mode=None):
    """scipy.misc.imresize as scipy 1.2 had it, for what LW's ResizeWrapper passes: a uint8 RGB frame and a
    (height, width, 3) tuple.  toimage() hands uint8 data to Pillow unchanged and imresize() swaps the size to
    Pillow's (width, height).  Anything else raises."""
    from PIL import Image
    arr = np.asarray(arr)
    if interp != "bilinear" or mode is not None or arr.dtype != np.uint8 or arr.ndim != 3 or arr.shape[2] != 3:
        raise NotImplementedError("stand-in covers uint8 RGB frames with interp='bilinear' only")
    if not isinstance(size, tuple) or len(size) != 3 or size[2] != 3:
        raise NotImplementedError("stand-in covers a (height, width, 3) size only")
    im = Image.fromarray(arr)
    return np.array(im.resize((size[1], size[0]), Image.BILINEAR))


# golden fixture tests/golden/lw_resize.npz: source sizes (w, h) and the LW shapes resized to from each
SOURCES = {"640x480": [(120, 160, 3), (84, 84, 3), (48, 64, 3), (120, 640, 3), (15, 20, 3)],
           "160x120": [(80, 80, 3), (120, 160, 3), (240, 320, 3)],
           "100x76": [(120, 160, 3), (30, 41, 3)]}
# outputs of at most this many pixels are stored whole (a failing comparison shows where); larger ones only as the
# SHA-256 of their bytes, which pins them just as exactly and keeps the file small (resized noise does not compress)
GOLDEN_ARRAY_MAX_PIXELS = 84 * 84


def golden_key(tag: str, shape) -> str:
    return f"lw_{tag}_{shape[0]}x{shape[1]}"


def canned_frames(seed: int, w: int, h: int) -> np.ndarray:
    """u8 [3][h][w][3]: noise, a smooth gradient, and blocks saturated at 0 and 255 over noise (one rng per size)."""
    rng = np.random.default_rng([seed, w, h])
    frames = rng.integers(0, 256, (3, h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    frames[1] = np.stack([(xx * 255 // w), (yy * 255 // h), ((xx + yy) * 255 // (h + w))], -1).astype(np.uint8)
    sat = frames[2]
    sat[: h // 2, : w // 3] = 0
    sat[h // 3:, w // 2:] = 255
    sat[h // 4: h // 4 + max(1, h // 8), :, 1] = 255     # one saturated channel across the frame
    sat[:, w // 5: w // 5 + 3] = (0, 255, 0)             # a thin hard-edged stripe
    return frames


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
