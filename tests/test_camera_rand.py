"""camera_rand on the host: the calibration ranges and LUTs against the reference's own Distortion(camera_rand=True)
(tests/golden/camera_rand.npz, carnivalmirror's sampler stubbed with fixed calibrations), the calibration draw, and
the host resets against the reference's reset() with camera_rand and distortion on (reset_camrand_<map>.npz)."""
import hashlib
import os

import numpy as np
import pytest

from gym_duckietown_b200 import maps
from gym_duckietown_b200.distortion import (CALIBRATION_KEYS, Distortion, calibration_ranges, draw_calibration,
                                             draw_calibrations)
from gym_duckietown_b200.episode import EpisodeSampler
from test_reset_sampler import MAPS, oracle_query


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "camera_rand.npz"))


def test_ranges_are_the_references(golden):
    """What the reference hands carnivalmirror.ParameterSampler equals calibration_ranges(), key order included."""
    assert tuple(golden["range_keys"]) == CALIBRATION_KEYS
    ranges = calibration_ranges()
    assert list(ranges) == list(CALIBRATION_KEYS)
    assert np.array_equal(golden["ranges"], np.array([ranges[k] for k in CALIBRATION_KEYS]))
    assert int(golden["cal_width"]) == 640 and int(golden["cal_height"]) == 480


@pytest.mark.parametrize("W,H", [(640, 480), (160, 120)])
def test_luts_match_reference(golden, W, H):
    """Distortion(W, H, K, D) builds, for every fixed calibration, the LUT the reference builds, bit for bit."""
    tag = f"{W}x{H}"
    for c in range(len(golden["K"])):
        d = Distortion(W, H, golden["K"][c], golden["D"][c])
        rx, ry = d.rmapx.astype(np.float32), d.rmapy.astype(np.float32)
        assert np.array_equal(d.new_camera_matrix, golden[f"new_camera_matrix_{tag}"][c])
        assert np.array_equal(rx[::8, ::8], golden[f"rmapx_sub_{tag}"][c])
        assert np.array_equal(ry[::8, ::8], golden[f"rmapy_sub_{tag}"][c])
        assert hashlib.sha256(rx.tobytes()).hexdigest() == str(golden[f"sha_rmapx_{tag}"][c])
        assert hashlib.sha256(ry.tobytes()).hexdigest() == str(golden[f"sha_rmapy_{tag}"][c])


def test_default_calibration_unchanged(golden):
    """Distortion() without K, D is the base calibration, the first of the fixed ones."""
    d = Distortion(160, 120)
    assert hashlib.sha256(d.rmapx.astype(np.float32).tobytes()).hexdigest() == str(golden["sha_rmapx_160x120"][0])


def test_draws_deterministic_and_in_range():
    a, b, c = draw_calibrations(32, seed=5), draw_calibrations(32, seed=5), draw_calibrations(32, seed=6)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))
    assert not np.array_equal(a[0][0], c[0][0])
    ranges = calibration_ranges()
    for K, D in a:
        assert K.shape == (3, 3) and D.shape == (1, 5)
        assert K[0, 1] == K[1, 0] == K[2, 0] == K[2, 1] == 0 and K[2, 2] == 1
        vals = dict(zip(CALIBRATION_KEYS, [K[0, 0], K[1, 1], K[0, 2], K[1, 2], *D[0]]))
        for k, (lo, hi) in ranges.items():
            assert min(lo, hi) <= vals[k] <= max(lo, hi), k
        assert D[0, 4] == 0.0
    # p2 is negative: its range is written (low, high) with low > high, and is drawn all the same
    assert ranges["p2"][0] > ranges["p2"][1]
    assert len({float(D[0, 3]) for _, D in a}) == 32


def test_draw_stream_is_not_a_reset_stream():
    """The calibrations come from a stream of their own: seed s does not give the draws of np_random(s)."""
    from gym_duckietown_b200.episode import np_random
    K, _ = draw_calibration(np_random(5))
    assert not np.array_equal(K, draw_calibrations(1, seed=5)[0][0])


@pytest.mark.parametrize("name", MAPS)
def test_reset_draws_match_reference(golden_dir, name):
    """EpisodeSampler(camera_rand=True, domain_rand=False) is the reference's reset() with camera_rand and distortion
    on, draw for draw: the camera height / angle / FOV are applied, nothing else of DR is."""
    g = np.load(os.path.join(golden_dir, f"reset_camrand_{name}.npz"))
    md = maps.load_map(name)
    seeds = [int(v) for v in g["seeds"]]
    s = EpisodeSampler(len(seeds), domain_rand=False, camera_rand=True)
    s.seed(seeds)
    envs = list(range(len(seeds)))
    for ep in range(2):
        out = s.sample(envs, [md] * len(envs), oracle_query(md))
        rows = np.arange(len(envs)) * 2 + ep
        assert np.array_equal(out["pos_x"], g["cur_pos"][rows, 0])
        assert np.array_equal(out["pos_z"], g["cur_pos"][rows, 2])
        assert np.array_equal(out["angle"], g["cur_angle"][rows])
        assert np.array_equal(out["wheel_dist"], g["wheel_dist"][rows])
        assert np.array_equal(out["cam_height"], g["cam_height"][rows])
        assert np.array_equal(out["cam_angle_deg"], g["cam_angle"][rows])
        assert np.array_equal(out["cam_fov_y_deg"], g["cam_fov_y"][rows])
        assert np.array_equal(out["horizon_color"], g["horizon_color"][rows])
        assert np.array_equal(out["ground_color"], g["ground_color"][rows])
        assert not np.any(out["cam_noise"])
    assert len(set(g["cam_height"].tolist())) > 1   # the perturbation is on
