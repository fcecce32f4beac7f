"""Fisheye look-up table of the reference's `Distortion` (distortion.py:10-125, 138-256), built once
on the host; the per-frame gather `out[y,x] = img[rint(rmapy[y,x]), rint(rmapx[y,x])]` is fused into
the render kernel (dts_set_fisheye_lut).  Under `camera_rand` every camera has its own calibration K, D
(`draw_calibrations`) and its own LUT (`Distortion(width, height, K, D)`), gathered per env (dts_set_fisheye_luts).

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
# The order camera_rand draws a calibration's parameters in: carnivalmirror's ranges dict (distortion.py:65-75)
CALIBRATION_KEYS = ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3")
# Extra seed word of the calibration stream: a stream of its own, apart from the envs' reset streams
CAMERA_RAND_SEED_WORD = 0x63616D72
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


def calibration_ranges(camera_matrix=CAMERA_MATRIX, distortion_coefs=DISTORTION_COEFS) -> dict:
    """Distortion.randomize_camera's ranges (distortion.py:65-75): every parameter within (0.95 v, 1.05 v) of its base
    value, written (low, high) as the reference writes them, so low > high for a negative base value (p2)."""
    K, D = np.asarray(camera_matrix, float), np.reshape(np.asarray(distortion_coefs, float), (1, 5))
    base = (K[0, 0], K[1, 1], K[0, 2], K[1, 2], D[0, 0], D[0, 1], D[0, 2], D[0, 3], D[0, 4])
    return {k: (0.95 * v, 1.05 * v) for k, v in zip(CALIBRATION_KEYS, base)}


def calibration_stream(seed=None) -> np.random.Generator:
    """The stream camera calibrations are drawn from: PCG64 seeded from `seed` and CAMERA_RAND_SEED_WORD (fresh entropy
    for seed None).  It is not an env's reset stream, so resets stay draw for draw the reference's; the reference
    draws from carnivalmirror's own generator, not the Simulator's, either."""
    words = None if seed is None else [int(seed), CAMERA_RAND_SEED_WORD]
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(words)))


def draw_calibration(rng: np.random.Generator):
    """One camera_rand calibration: fx, fy, cx, cy, k1, k2, p1, p2, k3, in that order, each uniform over its range in
    `calibration_ranges()`.  Generator.uniform refuses low > high (p2's range as the reference writes it), so each is
    drawn between the smaller and the larger bound; k3's range is (0, 0), so k3 is 0.  Returns K [[fx, 0, cx], [0, fy,
    cy], [0, 0, 1]] and D [[k1, k2, p1, p2, k3]].  (carnivalmirror's own draws are not reproduced: DESIGN §5a.)"""
    v = {k: rng.uniform(min(lo, hi), max(lo, hi)) for k, (lo, hi) in calibration_ranges().items()}
    K = np.array([[v["fx"], 0, v["cx"]], [0, v["fy"], v["cy"]], [0, 0, 1]], float)
    D = np.array([[v["k1"], v["k2"], v["p1"], v["p2"], v["k3"]]], float)
    return K, D


def draw_calibrations(count: int, seed=None) -> list:
    """`count` calibrations (K, D) from calibration_stream(seed), in order."""
    rng = calibration_stream(seed)
    return [draw_calibration(rng) for _ in range(count)]


class Distortion:
    def __init__(self, width: int = 640, height: int = 480, camera_matrix=None, distortion_coefs=None):
        """The fisheye LUT of a camera with calibration K = `camera_matrix`, D = `distortion_coefs` (default: the
        reference's own), built as the reference builds it for an observation of width x height."""
        self.W, self.H = 640, 480  # the calibration's image size (distortion.py:13-14)
        self.camera_matrix = CAMERA_MATRIX if camera_matrix is None else np.reshape(np.asarray(camera_matrix, float), (3, 3))
        self.distortion_coefs = DISTORTION_COEFS if distortion_coefs is None else \
            np.reshape(np.asarray(distortion_coefs, float), (1, 5))
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
