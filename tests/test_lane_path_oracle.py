"""The lane path's oracle (tests/lane_path_oracle.py, DESIGN.md section 5 item 18) without a GPU: it walks the chain the
reference's own closest_curve_point walks (the lane_path goldens), its point 0 gives the reference's lane pose (the
logic goldens), every point lies on a drivable tile, on a straight tile aligned with the lane the points keep one right
offset, on the looped maps an in-lane walk finds every point, and the ctypes signatures match the header."""
import os
import re

import numpy as np
import pytest

import lane_path_oracle as lo
from gym_duckietown_b200 import maps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
GOLDEN_MAPS = ["small_loop", "loop_obstacles", "udem1", "loop_trafficlights"]
LOOPED = ["small_loop", "loop_obstacles", "udem1"]   # every lane of these runs on round the map


@pytest.mark.parametrize("name", GOLDEN_MAPS)
def test_walk_is_the_references(name):
    """Every point of every chain, the ambiguous ones too: numpy takes its sines and arctangents from the same libm as
    the reference, so only the sums' order differs"""
    g = np.load(os.path.join(GOLD, f"lane_path_{name}.npz"))
    md = maps.load_map(name)
    K = g["q"].shape[2]
    assert K == 64 and list(g["spacing"]) == [0.05, 0.1, 0.3]
    for s, ds in enumerate(g["spacing"]):
        q, t, count, _ = lo.walk(md, g["poses"], K, float(ds))
        assert np.array_equal(count, g["count"][s]), (name, ds)
        for arr, want in ((q, g["q"][s]), (t, g["t"][s])):
            assert np.array_equal(np.isnan(arr), np.isnan(want)), (name, ds)
            ok = ~np.isnan(want)
            assert np.abs(arr[ok] - want[ok]).max() <= 1e-12, (name, ds)
    assert (g["count"] == K).any() and (g["count"] == 0).any()


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles", "udem1"])
def test_point_zero_is_the_lane_pose(name):
    """get_lane_pos2's dist and angle_rad from point 0's row: dist = -forward sin(yaw) - right cos(yaw), angle = yaw"""
    g = np.load(os.path.join(GOLD, f"logic_{name}.npz"))
    md = maps.load_map(name)
    poses = g["poses"]
    q, t, count, amb = lo.walk(md, poses, 1, 0.1)
    assert np.array_equal(count == 1, g["inlane"].astype(bool))
    pts = lo.agent_frame(poses, q, t)[:, 0]
    dist, ang = lo.lane_pose(pts)
    m = g["inlane"].astype(bool) & ~amb[:, 0]
    assert m.sum() > 0.5 * len(poses)
    assert np.abs(dist[m] - g["dist"][m]).max() <= 1e-12
    # acos(dot) loses digits where the heading lies along the tangent or against it: 1 ulp of dot over sin(angle)
    dd = np.clip(g["dot"][m], -1, 1)
    bar = 1e-12 + 4e-16 / np.maximum(np.sqrt(1 - dd * dd), 1e-8)
    err = np.abs((ang[m] - g["ang"][m] + np.pi) % (2 * np.pi) - np.pi)
    assert (err <= bar).all(), err.max()


@pytest.mark.parametrize("name", GOLDEN_MAPS)
def test_every_point_lies_on_its_drivable_tile(name):
    md = maps.load_map(name)
    poses = np.asarray(np.load(os.path.join(GOLD, f"lane_path_{name}.npz"))["poses"])
    ts = md.tile_size
    for ds in (0.05, 0.3):
        q, t, count, _ = lo.walk(md, poses, 64, ds)
        assert count.sum() > 0
        for e in np.flatnonzero(count):
            qx = np.r_[poses[e, 0], q[e, :count[e] - 1, 0] + ds * t[e, :count[e] - 1, 0]]   # each point's query
            qz = np.r_[poses[e, 1], q[e, :count[e] - 1, 2] + ds * t[e, :count[e] - 1, 2]]
            i, j = np.floor(qx / ts), np.floor(qz / ts)
            idx = (j * md.grid_w + i).astype(np.int64)
            assert (md.tile_drivable[idx] != 0).all()
            p = q[e, :count[e]]
            assert ((p[:, 0] >= i * ts - 1e-12) & (p[:, 0] <= (i + 1) * ts + 1e-12)).all(), (name, e)
            assert ((p[:, 2] >= j * ts - 1e-12) & (p[:, 2] <= (j + 1) * ts + 1e-12)).all(), (name, e)
            assert np.allclose(p[:, 1], 0.0) and np.allclose(np.linalg.norm(t[e, :count[e]], axis=1), 1.0)


@pytest.mark.parametrize("name", GOLDEN_MAPS)
def test_straight_tiles_keep_one_right_offset(name):
    """An agent on a straight tile's right lane, heading along it: the points on that tile share its right offset"""
    md = maps.load_map(name)
    ts = md.tile_size
    straight = maps.TILE_KINDS.index("straight")
    cv = lo.Curves(md)
    n_tiles = 0
    for idx in np.flatnonzero(md.tile_kind == straight):
        i, j = idx % md.grid_w, idx // md.grid_w
        for a0 in (0.0, np.pi / 2, np.pi, -np.pi / 2):
            x, z = np.array([(i + 0.5) * ts]), np.array([(j + 0.5) * ts])
            found, q0, t0, _ = lo.closest_curve_point(cv, x, z, np.array([a0]))
            if not found[0]:
                continue
            heading = np.arctan2(-t0[0, 2], t0[0, 0])
            pose = np.array([[q0[0, 0] - 0.2 * t0[0, 0], q0[0, 2] - 0.2 * t0[0, 2], heading]])
            q, t, count, _ = lo.walk(md, pose, 64, 0.05)
            pts = lo.agent_frame(pose, q, t)[0, :count[0]]
            on = (np.floor(q[0, :count[0], 0] / ts) == i) & (np.floor(q[0, :count[0], 2] / ts) == j)
            assert on.sum() >= 3
            assert np.abs(pts[on, 1] - pts[on, 1][0]).max() <= 1e-12, (name, i, j, a0)
            assert np.abs(pts[on, 2]).max() <= 1e-12
            n_tiles += 1
    assert n_tiles > 0


@pytest.mark.parametrize("name", LOOPED)
def test_looped_maps_find_every_point(name):
    g = np.load(os.path.join(GOLD, f"logic_{name}.npz"))
    md = maps.load_map(name)
    inlane = g["inlane"].astype(bool)
    for ds in (0.05, 0.1, 0.3):   # (a step longer than a tile's half-width can leave a curve tile's road)
        _, _, count, _ = lo.walk(md, g["poses"][inlane], 64, ds)
        assert (count == 64).all(), (name, ds, np.unique(count))


def test_ctypes_signatures_match_the_header():
    import ctypes as C
    from gym_duckietown_b200 import lib as L
    with open(os.path.join(ROOT, "include", "dtsim.h")) as f:
        h = f.read()
    lib = L.load()
    for name in ("dts_set_lane_path_target", "dts_render_lane_path"):
        args = re.search(r"int " + name + r"\(([^)]*)\);", h).group(1)
        want = []
        for a in args.split(","):
            a = a.strip()
            if re.fullmatch(r"int \w+", a):
                want.append(C.c_int)
            elif re.fullmatch(r"double \w+", a):
                want.append(C.c_double)
            else:
                assert "*" in a, a
                want.append(C.c_void_p)
        assert getattr(lib, name).argtypes == want, name
    assert re.search(r"#define DTS_LANE_PATH_MAX_POINTS 64\b", h)
