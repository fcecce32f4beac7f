#!/usr/bin/env python3
"""Generate the camera_rand fixtures under tests/golden/ by executing the REFERENCE's own code (oracle/refstub.py), as
oracle/make_golden.py does for the others.  Needs the reference source tree; the fixtures are committed.

    python tools/make_golden_camera_rand.py

  camera_rand.npz          Distortion(camera_rand=True) (distortion.py:46-83) with carnivalmirror.ParameterSampler
                           stubbed: the `ranges` / `cal_width` / `cal_height` the reference hands the sampler, and for
                           fixed calibrations (the base values, corners of the range box, interior points) the digest,
                           a sub-sample and the new camera matrix of the LUT it builds, at 640x480 and at 160x120 (the
                           reference builds its maps at the size of the first image it distorts, distortion.py:92-111)
  reset_camrand_<map>.npz  Simulator.reset() with camera_rand=True, distortion=True, domain_rand=False (S:611-614)
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import make_golden as mg  # noqa: E402
import refstub  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SIZES = ((640, 480), (160, 120))


def fixed_calibrations():
    """(K, D) of the calibrations the stubbed sampler hands out, in order: the base values, three corners of the range
    box and three interior points (k3's range is (0, 0): always 0)."""
    K0 = np.reshape([305.5718893575089, 0, 303.0797142544728, 0, 308.8338858195428, 231.8845403702499, 0, 0, 1], (3, 3))
    D0 = np.array([-0.2, 0.0305, 0.0005859930422629722, -0.0006697840226199427, 0])
    base = np.array([K0[0, 0], K0[1, 1], K0[0, 2], K0[1, 2], *D0])
    scales = [np.ones(9), np.full(9, 0.95), np.full(9, 1.05), np.array([0.95, 1.05] * 4 + [1.0])]
    rng = np.random.default_rng(17)
    scales += [rng.uniform(0.95, 1.05, 9) for _ in range(3)]
    out = []
    for s in scales:
        v = base * s
        out.append((np.array([[v[0], 0, v[2]], [0, v[1], v[3]], [0, 0, 1]]), np.array(v[4:9])))
    return out


def gen_camera_rand():
    refstub.install()
    import gym_duckietown.distortion as rd

    cals = fixed_calibrations()
    seen = []

    class Calibration:
        def __init__(self, K, D, cal_height):
            self.K, self.D, self.cal_height = K, D, cal_height

        def get_K(self, height):
            assert height == self.cal_height   # carnivalmirror's rescale to another height is not exercised
            return self.K.copy()

        def get_D(self):
            return self.D.copy()

    class ParameterSampler:
        def __init__(self, ranges, cal_width, cal_height):
            seen.append((dict(ranges), cal_width, cal_height))
            self.cal_height = cal_height

        def next(self):
            K, D = cals[len(seen) - 1]
            return Calibration(K, D, self.cal_height)

    rd.cm.ParameterSampler = ParameterSampler
    out = {"K": np.stack([K for K, _ in cals]), "D": np.stack([D for _, D in cals])}
    for W, H in SIZES:
        seen.clear()
        sha_x, sha_y, sub_x, sub_y, ncm = [], [], [], [], []
        for _ in cals:
            d = rd.Distortion(camera_rand=True)
            d.distort(np.zeros((H, W, 3), np.uint8))
            rx, ry = d.rmapx.astype(np.float32), d.rmapy.astype(np.float32)
            sha_x.append(hashlib.sha256(rx.tobytes()).hexdigest()); sha_y.append(hashlib.sha256(ry.tobytes()).hexdigest())
            sub_x.append(rx[::8, ::8]); sub_y.append(ry[::8, ::8]); ncm.append(d.new_camera_matrix)
        tag = f"{W}x{H}"
        out[f"sha_rmapx_{tag}"], out[f"sha_rmapy_{tag}"] = np.array(sha_x), np.array(sha_y)
        out[f"rmapx_sub_{tag}"], out[f"rmapy_sub_{tag}"] = np.stack(sub_x), np.stack(sub_y)
        out[f"new_camera_matrix_{tag}"] = np.stack(ncm)
    ranges, cal_w, cal_h = seen[0]
    assert all(s[0] == ranges and s[1:] == (cal_w, cal_h) for s in seen)
    out["range_keys"] = np.array(list(ranges))
    out["ranges"] = np.array([ranges[k] for k in ranges], float)
    out["cal_width"], out["cal_height"] = np.array(cal_w), np.array(cal_h)
    np.savez_compressed(os.path.join(OUT, "camera_rand.npz"), **out)
    print(f"camera_rand: {len(cals)} calibrations x {len(SIZES)} sizes")


def gen_reset_camrand(name: str, seeds=range(12)):
    raw = mg.raw_map(name)
    S, C, G, O = refstub.modules()
    rows = {k: [] for k in ("cur_pos", "cur_angle", "wheel_dist", "cam_height", "cam_angle", "cam_fov_y",
                            "horizon_color", "ground_color")}
    for seed in seeds:
        sim = refstub.build_reference_sim(raw, mg.extents_for(raw), domain_rand=False, seed=int(seed))
        sim.distortion, sim.camera_rand = True, True   # Simulator(distortion=True, camera_rand=True), S:352-358
        for episode in range(2):
            sim.reset()
            rows["cur_pos"].append(np.array(sim.cur_pos, float)); rows["cur_angle"].append(float(sim.cur_angle))
            rows["wheel_dist"].append(float(sim.wheel_dist))
            rows["cam_height"].append(float(np.ravel(sim.cam_height)[0]))
            rows["cam_angle"].append(float(np.ravel(sim.cam_angle[0])[0]))
            rows["cam_fov_y"].append(float(np.ravel(sim.cam_fov_y)[0]))
            rows["horizon_color"].append(np.array(sim.horizon_color, float))
            rows["ground_color"].append(np.array(sim.ground_color, float))
    out = {k: np.array(v) for k, v in rows.items()}
    out["seeds"] = np.array(list(seeds))
    np.savez_compressed(os.path.join(OUT, f"reset_camrand_{name}.npz"), **out)
    print(f"reset_camrand_{name}: {len(out['seeds'])} seeds x 2 episodes")


if __name__ == "__main__":
    gen_camera_rand()
    for m in mg.MAPS:
        gen_reset_camrand(m)
