#!/usr/bin/env python3
"""Generate tests/golden/undistort.npz by running the REFERENCE's own src/gym_duckietown/wrappers.py UndistortWrapper
(stub-imported through oracle/refstub.py, like oracle/make_golden_lw.py) on canned frames.

Run in the build container only (needs /root/reference and cv2):   python oracle/make_golden_undistort.py

The wrapper sits on a stand-in env with `distortion=True`; its construction must set `unwrapped.undistort`.  Per size
it builds its map on the first observation (cv2.initUndistortRectifyMap with its K, D, I, P at the observation's size)
and returns cv2.remap(frame, mapx, mapy, INTER_NEAREST).  The cv2 version that computed them is recorded.

Keys: seed, cv2_version, frames_sha_<w>x<h> (the canned frames, pil_resize.canned_frames(seed, w, h)),
mapx_sha_<w>x<h> / mapy_sha_<w>x<h> = SHA-256 of the wrapper's float32 maps, out_sha_<w>x<h> = SHA-256 of u8 [3][h][w][3],
what observation() returned for the three frames, and out_<w>x<h> = those frames where w * h <= 160 * 120.
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import pil_resize  # noqa: E402
import refstub  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SIZES = [(640, 480), (160, 120), (84, 84), (90, 70)]
ARRAY_MAX_PIXELS = 160 * 120


def gen_undistort(seed=29):
    import cv2
    refstub.install()
    W_ = importlib.import_module("gym_duckietown.wrappers")
    spaces = sys.modules["gym.spaces"]
    out = {"seed": np.int64(seed), "cv2_version": cv2.__version__}
    for w, h in SIZES:
        tag = f"{w}x{h}"
        frames = pil_resize.canned_frames(seed, w, h)

        class Env:   # a Simulator(distortion=True) as the wrapper sees it
            metadata, reward_range = {}, (-1000, 1000)
            action_space = spaces.Box(low=-1, high=1, shape=(2,), dtype=np.float32)
            observation_space = spaces.Box(low=0, high=255, shape=(h, w, 3), dtype=np.uint8)
            distortion, undistort = True, False

            @property
            def unwrapped(self):
                return self

        env = Env()
        uw = W_.UndistortWrapper(env)
        assert env.undistort is True
        got = np.stack([uw.observation(f) for f in frames])
        assert got.dtype == np.uint8 and got.shape == (3, h, w, 3)
        mx, my = uw.mapx, uw.mapy
        assert mx.dtype == np.float32 and mx.shape == (h, w) and my.shape == (h, w)
        out[f"frames_sha_{tag}"] = pil_resize.sha(frames)
        out[f"mapx_sha_{tag}"] = pil_resize.sha(mx)
        out[f"mapy_sha_{tag}"] = pil_resize.sha(my)
        out[f"out_sha_{tag}"] = pil_resize.sha(got)
        if w * h <= ARRAY_MAX_PIXELS:
            out[f"out_{tag}"] = got
    np.savez_compressed(os.path.join(OUT, "undistort.npz"), **out)
    print("undistort:", sorted(out))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gen_undistort()
