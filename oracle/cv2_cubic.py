"""OpenCV's scalar INTER_CUBIC resize of a uint8 image, restated in numpy, integer-exact: what
src/gym_duckietown/wrappers.py:111-141's ResizeWrapper computes with cv2.resize, and the reference the device pass
(k_resize_band / k_resize, tables from dts_set_resize) is compared with at any shape, without OpenCV.

Per axis, `src` pixels -> `dst` pixels:
    scale = 1 / (dst / src) in double, fx = float32((d + 0.5) * scale - 0.5), sx = floor(fx), fx -= sx
    c[0..2] = interpolateCubic(fx) with A = -0.75 in float32, in OpenCV's operation order; c[3] = 1 - c0 - c1 - c2
    taps = rint(2048 * c) (half to even: cvRound), indices sx - 1 + k clamped to 0 .. src - 1
The horizontal pass sums px * tap exactly (int32 in OpenCV, int64 here); the vertical pass sums those with the row
taps, then (v + 2^21) >> 22 (arithmetic shift), saturated to 0..255.  This is the arithmetic of OpenCV's scalar
fixed-point code.  cv2.resize itself runs a vectorised vertical pass that sums in float32 and rounds ties to even, so
it differs by 1 LSB on a few percent of values; with cv2.setUseOptimized(False) still on the few whose sum lies at a
half LSB.
"""
from __future__ import annotations

import numpy as np

COEF_BITS = 11                      # INTER_RESIZE_COEF_BITS: taps are 2048 * w
SHIFT = 2 * COEF_BITS               # both passes' scale, removed at the end
CHUNK_BYTES = 256 << 20             # int64 intermediates per chunk of frames


def axis_weights(src: int, dst: int):
    """(sx int64[dst], c float32[dst][4]): first tap's unclamped source index + 1 and the float32 cubic weights."""
    scale = 1.0 / (dst / src)
    fx = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(fx)
    x = (fx - sx).astype(np.float32)
    A, one = np.float32(-0.75), np.float32(1)
    c = np.empty((dst, 4), np.float32)
    c[:, 0] = ((A * (x + one) - np.float32(5) * A) * (x + one) + np.float32(8) * A) * (x + one) - np.float32(4) * A
    c[:, 1] = ((A + np.float32(2)) * x - (A + np.float32(3))) * x * x + one
    c[:, 2] = ((A + np.float32(2)) * (one - x) - (A + np.float32(3))) * (one - x) * (one - x) + one
    c[:, 3] = one - c[:, 0] - c[:, 1] - c[:, 2]
    return sx.astype(np.int64), c


def axis_table(src: int, dst: int):
    """(idx int64[dst][4], taps int64[dst][4]) of one axis: the clamped source indices and the 11-bit taps."""
    sx, c = axis_weights(src, dst)
    idx = np.clip(sx[:, None] - 1 + np.arange(4)[None, :], 0, src - 1)
    taps = np.rint(c * np.float32(1 << COEF_BITS)).astype(np.int64)
    return idx, taps


def _resize_chunk(frames, xi, xw, yi, yw):
    rows, ry = np.unique(yi, return_inverse=True)            # the horizontal pass runs on the rows the taps read
    ry = ry.reshape(yi.shape)
    src = frames[:, rows].astype(np.int64)                     # [n][rows][W][3]
    h = sum(src[:, :, xi[:, k]] * xw[None, None, :, k, None] for k in range(4))         # [n][rows][ow][3]
    v = sum(h[:, ry[:, k]] * yw[None, :, k, None, None] for k in range(4))              # [n][oh][ow][3]
    return np.clip((v + (1 << (SHIFT - 1))) >> SHIFT, 0, 255).astype(np.uint8)


def resize(frames: np.ndarray, ow: int, oh: int) -> np.ndarray:
    """cv2.resize(frame, (ow, oh), interpolation=cv2.INTER_CUBIC) of u8 [..., H, W, 3] (leading axes: a batch),
    as OpenCV's scalar path computes it."""
    frames = np.asarray(frames)
    if frames.dtype != np.uint8 or frames.ndim < 3 or frames.shape[-1] != 3:
        raise ValueError("expects uint8 [..., H, W, 3]")
    lead, (H, W) = frames.shape[:-3], frames.shape[-3:-1]
    flat = frames.reshape((-1, H, W, 3))
    xi, xw = axis_table(W, ow)
    yi, yw = axis_table(H, oh)
    per_frame = 8 * 3 * ow * (len(np.unique(yi)) + oh) + 8 * len(np.unique(yi)) * W * 3
    step = max(1, CHUNK_BYTES // per_frame)
    out = np.empty((flat.shape[0], oh, ow, 3), np.uint8)
    for i in range(0, flat.shape[0], step):
        out[i:i + step] = _resize_chunk(flat[i:i + step], xi, xw, yi, yw)
    return out.reshape(lead + (oh, ow, 3))
