"""UndistortWrapper (src/gym_duckietown/wrappers.py:145-227) on the CPU: the product's map builder
(distortion.rectify_maps) and a round-half-even gather through it against what the reference class returned
(tests/golden/undistort.npz, oracle/make_golden_undistort.py), and the raster oracle's fused gather under that map
against cv2.remap of its plain frame — the reference the GPU tests compare the device's rectified frames with."""
import os

import numpy as np

import pil_resize as P
from test_gpu_fisheye import THREADS, lsb_diff, numpy_gather, random_poses

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "undistort.npz")
SIZES = [(640, 480), (160, 120), (84, 84), (90, 70)]


def golden_outputs(g, w, h, frames):
    """What the reference class returned for `frames`: stored whole up to 160x120; for 640x480 only its digest, which
    the numpy gather must match before it stands in for it."""
    tag = f"{w}x{h}"
    if f"out_{tag}" in g.files:
        return g[f"out_{tag}"]
    from gym_duckietown_b200.distortion import rectify_maps
    want = numpy_gather(frames, *rectify_maps(w, h))
    assert P.sha(want) == str(g[f"out_sha_{tag}"]), tag
    return want


def test_map_builder_equals_the_reference_wrappers_map():
    from gym_duckietown_b200.distortion import rectify_maps
    g = np.load(GOLD)
    for w, h in SIZES:
        mx, my = rectify_maps(w, h)
        assert mx.dtype == np.float32 and mx.shape == (h, w) and my.shape == (h, w)
        assert P.sha(mx) == str(g[f"mapx_sha_{w}x{h}"]) and P.sha(my) == str(g[f"mapy_sha_{w}x{h}"]), (w, h)


def test_gather_through_the_map_equals_the_reference_wrapper():
    """round half to even, 0 where the map leaves the frame: byte for byte what the wrapper's cv2.remap returned"""
    from gym_duckietown_b200.distortion import rectify_maps
    g = np.load(GOLD)
    for w, h in SIZES:
        frames = P.canned_frames(int(g["seed"]), w, h)
        assert P.sha(frames) == str(g[f"frames_sha_{w}x{h}"]), (w, h)
        got = numpy_gather(frames, *rectify_maps(w, h))
        want = golden_outputs(g, w, h, frames)
        assert np.array_equal(got, want), (w, h, lsb_diff(got, want))
        assert P.sha(got) == str(g[f"out_sha_{w}x{h}"])
        assert (got == 0).all(-1).any(), "the map was expected to leave some pixels without a source"


def test_the_wrappers_map_is_not_the_distortion_models():
    """Distortion.undistort uses getOptimalNewCameraMatrix's K, not the wrapper's P"""
    from gym_duckietown_b200.distortion import Distortion, rectify_maps
    mx, my = rectify_maps(640, 480)
    d = Distortion(640, 480)
    assert max(np.abs(mx - d.mapx).max(), np.abs(my - d.mapy).max()) > 10


def test_oracle_rectified_render_equals_cv2_remap_of_its_plain_frame():
    import cv2
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.distortion import rectify_maps

    md = maps.load_map("loop_obstacles")
    sc = orc.OracleScene(md)
    for w, h in ((160, 120), (84, 84)):
        px, pz, ang = random_poses(md, 6, 8)
        eps = [orc.default_episode() for _ in px]
        mx, my = rectify_maps(w, h)
        plain = sc.render_batch(px, pz, ang, eps, w, h, False, threads=THREADS)
        fused = sc.render_batch(px, pz, ang, eps, w, h, False, lut=(mx, my), threads=THREADS)
        for k in range(len(px)):
            want = cv2.remap(plain[k], mx, my, cv2.INTER_NEAREST)
            assert np.array_equal(fused[k], want), (w, h, k, lsb_diff(fused[k], want))
        assert fused.std() > 10
