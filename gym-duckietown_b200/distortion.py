"""Fisheye look-up table of the reference's `Distortion` (distortion.py:10-125, 138-256), built once
on the host; the per-frame gather `out[y,x] = img[rint(rmapy[y,x]), rint(rmapx[y,x])]` is fused into
the render kernel (dts_set_fisheye_lut).  `camera_rand` (carnivalmirror) is out of scope.

The LUT must equal the reference's bit for bit (tests/golden/fisheye.npz pins it), which means
reproducing two order-dependent details of its construction: duplicate targets in the scatter keep
the LAST contribution, and holes are filled in Python-set iteration order.
"""
from __future__ import annotations

import itertools

import cv2
import numpy as np

# K, D of the raw (distorted) camera — distortion.py:16-30
CAMERA_MATRIX = np.reshape([305.5718893575089, 0, 303.0797142544728, 0, 308.8338858195428, 231.8845403702499,
                            0, 0, 1], (3, 3))
DISTORTION_COEFS = np.reshape([-0.2, 0.0305, 0.0005859930422629722, -0.0006697840226199427, 0], (1, 5))
# P of the rectified image UndistortWrapper emits — wrappers.py:184-198
RECTIFIED_PROJECTION = np.reshape([220.2460277141687, 0, 301.8668918355899, 0, 0, 238.6758484095299, 227.0880056118307,
                                   0, 0, 0, 1, 0], (3, 4))
_SPLAT = [(-1, -1, 7), (-1, 0, 10), (-1, 1, 7), (0, -1, 10), (0, 0, 20), (0, 1, 10), (1, -1, 7), (1, 0, 10), (1, 1, 7)]


def rectify_maps(width: int, height: int):
    """UndistortWrapper's (mapx, mapy), float32 [height][width] each (wrappers.py:210-225): the map it builds at the
    observation's size, with K and D of the raw camera, R = I and its own P.  The wrapper's observation is
    `cv2.remap(pinhole_frame, mapx, mapy, INTER_NEAREST)`: frame[rint(mapy), rint(mapx)], 0 outside the frame."""
    return cv2.initUndistortRectifyMap(CAMERA_MATRIX, DISTORTION_COEFS, np.eye(3), RECTIFIED_PROJECTION,
                                       (int(width), int(height)), cv2.CV_32FC1)


def invert_map(mapx: np.ndarray, mapy: np.ndarray):
    """Approximate inverse of a rectification map by weighted splatting (distortion.py:138-216)."""
    H, W = mapx.shape[:2]
    acc_w = np.zeros(H * W, np.float32)
    acc_x = np.zeros(H * W, np.float32)
    acc_y = np.zeros(H * W, np.float32)
    cx = np.clip(mapx.astype(np.int32), 2, W - 2)
    cy = np.clip(mapy.astype(np.int32), 2, H - 2)
    src_x = np.tile(np.arange(W, dtype=np.int32), (H, 1))
    src_y = np.repeat(np.arange(H, dtype=np.int32)[:, None], W, 1)
    for di, dj, w in _SPLAT:
        flat = ((cy + di) * W + (cx + dj)).ravel()
        # NOT np.add.at: the reference's fancy-index "+=" keeps only the last duplicate
        acc_w[flat] = acc_w[flat] + w
        acc_x[flat] = acc_x[flat] + (w * src_x).ravel()
        acc_y[flat] = acc_y[flat] + (w * src_y).ravel()
    rx = np.full(H * W, np.nan, np.float32)
    ry = np.full(H * W, np.nan, np.float32)
    hit = acc_w > 0
    rx[hit] = acc_x[hit] / acc_w[hit]
    ry[hit] = acc_y[hit] / acc_w[hit]
    rx, ry = rx.reshape(H, W), ry.reshape(H, W)
    fill_holes(rx, ry)
    return rx, ry


def fill_holes(rx: np.ndarray, ry: np.ndarray, R: int = 2):
    """Nearest filled neighbour within radius R, repeated until stable (distortion.py:218-256).
    Offsets are (a-R-1, b-R-1) for a,b in range(2R+1) — the reference's off-by-one window — stably
    sorted by length; holes are visited in the iteration order of a Python set built row-major."""
    H, W = rx.shape
    F = 2 * R + 1
    offs = [(a - R - 1, b - R - 1) for a, b in itertools.product(range(F), range(F))]
    offs = [o for o in offs if np.hypot(o[0], o[1]) <= R]
    offs.sort(key=lambda o: np.hypot(o[0], o[1]))
    holes = set()
    for i, j in np.argwhere(np.isnan(rx)):
        holes.add((int(i), int(j)))
    while holes:
        filled = 0
        for i, j in list(holes):
            for di, dj in offs:
                u, v = i + di, j + dj
                if 0 <= u < H and 0 <= v < W and not np.isnan(rx[u, v]):
                    rx[i, j], ry[i, j] = rx[u, v], ry[u, v]
                    filled += 1
                    holes.remove((i, j))
                    break
        if filled == 0:
            break


class Distortion:
    def __init__(self, width: int = 640, height: int = 480):
        self.W, self.H = 640, 480  # the calibration's image size (distortion.py:13-14)
        self.camera_matrix, self.distortion_coefs = CAMERA_MATRIX, DISTORTION_COEFS
        self.new_camera_matrix, _ = cv2.getOptimalNewCameraMatrix(
            cameraMatrix=self.camera_matrix, distCoeffs=self.distortion_coefs, imageSize=(self.W, self.H), alpha=0)
        # maps are built for the OBSERVATION's size with the same K (distortion.py:97-109)
        self.mapx, self.mapy = cv2.initUndistortRectifyMap(
            cameraMatrix=self.camera_matrix, distCoeffs=self.distortion_coefs, R=np.eye(3),
            newCameraMatrix=self.new_camera_matrix, size=(width, height), m1type=cv2.CV_32FC1)
        self.rmapx, self.rmapy = invert_map(self.mapx, self.mapy)

    def distort(self, observation: np.ndarray) -> np.ndarray:
        """Host reference of the fused gather (numpy): used by tests and by callers holding numpy frames."""
        ix = np.rint(self.rmapx).astype(np.int64)
        iy = np.rint(self.rmapy).astype(np.int64)
        H, W = observation.shape[:2]
        ok = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
        out = np.zeros_like(observation)
        out[ok] = observation[iy[ok], ix[ok]]
        return out

    def undistort(self, observation: np.ndarray) -> np.ndarray:
        """Distortion._undistort (distortion.py:127-136): remaps with this camera model's maps, whose new camera
        matrix comes from getOptimalNewCameraMatrix.  Not UndistortWrapper's map, which uses the wrapper's own P
        (rectify_maps); at 640x480 the two differ by up to 18 px."""
        return cv2.remap(observation, self.mapx, self.mapy, cv2.INTER_NEAREST)
