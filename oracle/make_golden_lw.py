#!/usr/bin/env python3
"""Generate tests/golden/lw_resize.npz by running the REFERENCE's own learning/utils/wrappers.py ResizeWrapper
(stub-imported through oracle/refstub.py, like oracle/make_golden.py's generators) on canned frames.

Run in the build container only (needs /root/reference and Pillow):   python oracle/make_golden_lw.py

The wrapper calls `scipy.misc.imresize(observation, self.shape)`, which scipy >= 1.3 no longer has.  A stand-in with
scipy 1.2's semantics for what the wrapper passes it (uint8 RGB frame, (h, w, 3) size; pil_resize.imresize_standin)
is installed as scipy.misc for the run; the Pillow version that computed the frames is recorded in the file.

Keys: seed, pillow_version, frames_sha_<src> (the canned frames, pil_resize.canned_frames(seed, w, h)),
lw_<src>_<h>x<w>_sha = SHA-256 of u8 [3][h][w][3], what ResizeWrapper(env, shape=(h, w, 3)).observation(frame)
returned for the three frames, and lw_<src>_<h>x<w> = those frames themselves where h * w <=
pil_resize.GOLDEN_ARRAY_MAX_PIXELS.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import pil_resize  # noqa: E402
import refstub  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def gen_lw_resize(seed=23):
    import PIL
    refstub.install()
    sys.path.insert(0, "/root/reference")
    import scipy
    misc = types.ModuleType("scipy.misc")
    misc.imresize = pil_resize.imresize_standin
    sys.modules["scipy.misc"] = misc
    scipy.misc = misc
    LW = importlib.import_module("learning.utils.wrappers")
    spaces = sys.modules["gym.spaces"]
    out = {"seed": np.int64(seed), "pillow_version": PIL.__version__}
    for tag, shapes in pil_resize.SOURCES.items():
        w, h = map(int, tag.split("x"))
        frames = pil_resize.canned_frames(seed, w, h)

        class Env:   # what launch_env()'s Simulator looks like to the wrapper
            metadata, reward_range = {}, (-1000, 1000)
            action_space = spaces.Box(low=-1, high=1, shape=(2,), dtype=np.float32)
            observation_space = spaces.Box(low=np.zeros((h, w, 3), np.uint8), high=np.full((h, w, 3), 255, np.uint8),
                                           shape=(h, w, 3), dtype=np.uint8)

            @property
            def unwrapped(self):
                return self

        out[f"frames_sha_{tag}"] = pil_resize.sha(frames)
        for shape in shapes:
            rz = LW.ResizeWrapper(Env(), shape=shape)
            assert tuple(rz.observation_space.shape) == shape
            got = np.stack([rz.observation(f) for f in frames])
            assert got.dtype == np.uint8 and got.shape == (3,) + shape
            key = pil_resize.golden_key(tag, shape)
            out[key + "_sha"] = pil_resize.sha(got)
            if shape[0] * shape[1] <= pil_resize.GOLDEN_ARRAY_MAX_PIXELS:
                out[key] = got
    np.savez_compressed(os.path.join(OUT, "lw_resize.npz"), **out)
    print("lw_resize:", sorted(out))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gen_lw_resize()
