"""The range scan oracle (tests/scan_oracle.py, DESIGN.md section 5 item 16) without a GPU: hand-built maps with walls,
empty cells and square objects at known distances, the tie and visibility rules, the ray directions, and on every
shipped map the scan's defining property checked against the bird's-eye oracle's labels at random poses.  Also: every
shipped footprint is strictly convex, and the ctypes struct matches the header."""
import math
import os
import re

import numpy as np
import pytest

import bev_oracle as bo
import scan_oracle as so
from gym_duckietown_b200 import maps

TS = 0.585
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def hand_scene(rows, squares=()):
    """A scene of MapFormat1 tile rows and axis-aligned square footprints (cx, cz, half side), object o = squares[o]"""
    md = maps.interpret_map({"tile_size": TS, "tiles": rows, "objects": []}, "hand")
    sc = bo.BevScene(md)
    sc.corners = [np.array([[cx - h, cz - h], [cx + h, cz - h], [cx + h, cz + h], [cx - h, cz + h]]) for cx, cz, h in
                  squares]
    sc.slot_of = {}
    return sc


ROAD5 = [["straight/E"] * 5 for _ in range(5)]


def one_ray(sc, x, z, angle, max_range=5.0, **kw):
    rng, hit, amb = so.scan(sc, x, z, angle, (1, 2 * math.pi, max_range, 0.0, 0.0), **kw)
    return float(rng[0]), int(hit[0]), bool(amb[0])


def test_wall_of_tiles_that_are_not_drivable():
    """Grass in column 3 of a road: a ray along +x from x = 0.3 stops at x = 3 ts on the grass tile of its row."""
    rows = [["straight/E", "straight/E", "straight/E", "grass", "straight/E"] for _ in range(3)]
    sc = hand_scene(rows)
    z = 1.5 * TS
    rng, hit, amb = one_ray(sc, 0.3, z, 0.0)
    assert not amb and hit == 2 + 3 * 3 + 1 and rng == pytest.approx(3 * TS - 0.3, abs=1e-12)
    # at an angle: the wall is met at x = 3 ts, the row where the ray is then
    a = 0.2
    rng, hit, amb = one_ray(sc, 0.3, z, a)
    t = (3 * TS - 0.3) / math.cos(a)
    j = math.floor((z - t * math.sin(a)) / TS)
    assert not amb and hit == 2 + 3 * 3 + j and rng == pytest.approx(t, abs=1e-12)


def test_leaving_the_grid_or_an_empty_cell_gives_the_ground():
    rows = [["straight/E", "straight/E", "empty", "straight/E"] for _ in range(3)]
    sc = hand_scene(rows)
    z = 1.5 * TS
    assert one_ray(sc, 0.3, z, math.pi) == (pytest.approx(0.3, abs=1e-12), 1, False)   # off the grid at x = 0
    assert one_ray(sc, 0.3, z, 0.0) == (pytest.approx(2 * TS - 0.3, abs=1e-12), 1, False)   # the empty column
    rng, hit, _ = one_ray(sc, 3.5 * TS, z, 0.0)
    assert hit == 1 and rng == pytest.approx(0.5 * TS, abs=1e-12)


@pytest.mark.parametrize("side", range(4))
def test_square_object_at_a_known_distance_on_each_side(side):
    a = side * math.pi / 2
    x, z = 2.5 * TS + 0.01, 2.5 * TS + 0.02
    cx, cz = x + 0.5 * math.cos(a), z - 0.5 * math.sin(a)
    sc = hand_scene(ROAD5, [(cx, cz, 0.05)])
    rng, hit, amb = one_ray(sc, x, z, a)
    assert not amb and hit == 2 + 25 + 0 and rng == pytest.approx(0.45, abs=1e-12)
    # the ray pointing the other way misses it and leaves the grid
    rng, hit, amb = one_ray(sc, x, z, a + math.pi)
    assert hit == 1 and rng > 1.0


def test_origin_inside_a_footprint_gives_zero_and_its_label():
    x, z = 2.5 * TS, 2.5 * TS
    sc = hand_scene(ROAD5, [(0.3, 0.3, 0.05), (x + 0.01, z, 0.04)])
    rng, hit, amb = so.scan(sc, x, z, 0.4, (16, 2 * math.pi, 2.0, 0.0, 0.0))
    assert (rng == 0).all() and (hit == 2 + 25 + 1).all() and not amb.any()


def test_origin_on_a_tile_that_is_not_drivable_gives_zero_and_its_label():
    rows = [["straight/E", "grass"], ["straight/E", "straight/E"]]
    sc = hand_scene(rows)
    rng, hit, _ = so.scan(sc, 1.5 * TS, 0.5 * TS, 1.0, (8, 2 * math.pi, 2.0, 0.0, 0.0))
    assert (rng == 0).all() and (hit == 2 + 1 * 2 + 0).all()


def test_overlapping_footprints_the_smallest_index_wins():
    """Two squares whose near edges coincide: the ray enters both at once and names the first of them."""
    x, z = 2.5 * TS, 2.5 * TS + 0.001
    big, small = (x + 0.5, z, 0.1), (x + 0.45, z, 0.05)
    for order, want in (((big, small), 0), ((small, big), 0)):
        sc = hand_scene(ROAD5, order)
        rng, hit, _ = one_ray(sc, x, z, 0.0)
        assert hit == 2 + 25 + want and rng == pytest.approx(0.4, abs=1e-12)
    # the nearer one wins whatever its index
    sc = hand_scene(ROAD5, [(x + 0.8, z, 0.05), (x + 0.4, z, 0.05)])
    assert one_ray(sc, x, z, 0.0)[:2] == (pytest.approx(0.35, abs=1e-12), 2 + 25 + 1)


def test_an_object_wins_over_a_cell_boundary_at_the_same_t():
    rows = [["straight/E", "straight/E", "grass"] for _ in range(3)]
    x, z = 0.5 * TS, 1.5 * TS
    sc = hand_scene(rows, [(2 * TS + 0.05, z, 0.05)])   # its near edge on the grass tile's edge
    rng, hit, _ = one_ray(sc, x, z, 0.0)
    assert hit == 2 + 9 + 0 and rng == pytest.approx(1.5 * TS, abs=1e-12)


def test_a_hidden_object_stops_nothing():
    x, z = 2.5 * TS, 2.5 * TS + 0.01
    sc = hand_scene(ROAD5, [(x + 0.3, z, 0.05)])
    hidden = np.zeros(8, np.uint32)
    hidden[0] = 1
    assert one_ray(sc, x, z, 0.0)[1] == 2 + 25
    rng, hit, _ = one_ray(sc, x, z, 0.0, hidden=hidden)
    assert hit == 1 and rng == pytest.approx(5 * TS - x, abs=1e-12)


def test_nothing_within_max_range_gives_hit_zero():
    rows = [["straight/E", "straight/E", "straight/E", "grass"] for _ in range(3)]
    sc = hand_scene(rows)
    assert one_ray(sc, 0.3, 1.5 * TS, 0.0, max_range=1.0) == (1.0, 0, False)
    assert one_ray(sc, 0.3, 1.5 * TS, 0.0, max_range=3 * TS - 0.3 + 1e-3)[1] == 2 + 9 + 1


def test_ray_directions():
    """One ray points straight ahead; fov = 2 pi gives R distinct directions, ray 0 the leftmost; an origin offset moves
    the origin ahead and to the right of the agent."""
    a = 0.7
    ox, oz, dx, dz = so.rays(1.0, 2.0, a, (1, 1.3, 2.0, 0.0, 0.0))
    assert (ox, oz) == (1.0, 2.0) and dx[0] == math.cos(a) and dz[0] == -math.sin(a)
    for R in (2, 7, 64, 360, 4096):
        _, _, dx, dz = so.rays(0.0, 0.0, a, (R, 2 * math.pi, 2.0, 0.0, 0.0))
        ang = np.sort(np.mod(np.arctan2(-dz, dx), 2 * math.pi))
        gaps = np.diff(np.concatenate([ang, ang[:1] + 2 * math.pi]))
        assert np.allclose(gaps, 2 * math.pi / R, atol=1e-9)
    _, _, dx, dz = so.rays(0.0, 0.0, 0.0, (3, 1.0, 2.0, 0.0, 0.0))
    assert -dz[0] > 0 > -dz[2] and dz[1] == 0   # left of the heading is -z at angle 0 (get_right_vec is +z)
    ox, oz, _, _ = so.rays(1.0, 2.0, 0.0, (1, 1.0, 2.0, 0.3, 0.1))
    assert (ox, oz) == pytest.approx((1.3, 2.1))


def test_every_shipped_footprint_is_strictly_convex():
    for name in maps.list_maps():
        md = maps.load_map(name)
        for o in md.objects:
            assert so.strictly_convex(np.asarray(o.corners, np.float64)), (name, o.kind)
        for d in md.dyn_objects:
            assert so.strictly_convex(np.asarray(d.corners, np.float64)), (name, "dynamic")


def random_road_poses(md, n, seed):
    rng = np.random.default_rng(seed)
    tiles = [(i, j) for j in range(md.grid_h) for i in range(md.grid_w) if md.tile_drivable[j * md.grid_w + i]]
    pick = rng.integers(0, len(tiles), n)
    ij = np.array([tiles[k] for k in pick], np.float64)
    x = (ij[:, 0] + rng.uniform(0.05, 0.95, n)) * md.tile_size
    z = (ij[:, 1] + rng.uniform(0.05, 0.95, n)) * md.tile_size
    return x, z, rng.uniform(-math.pi, math.pi, n)


@pytest.mark.parametrize("name", sorted(maps.list_maps()))
def test_property_against_the_birds_eye_labels(name):
    """Along every unambiguous ray: just before t* the point is not blocked, just after it the point is blocked and
    its bird's-eye label is hit (at t* = 0 the origin is); beyond max_range, hit 0 and nothing blocks before it."""
    md = maps.load_map(name)
    sc = bo.BevScene(md)
    feet = sc.footprints()
    n_amb = n_all = n_obj = 0
    for cfg in ((64, 2 * math.pi, 2.0, 0.0, 0.0), (33, 1.2, 6.0, 0.1, -0.05)):
        px, pz, ang = random_road_poses(md, 24, 11)
        for e in range(24):
            rng, hit, amb = so.scan(sc, px[e], pz[e], ang[e], cfg)
            ox, oz, dx, dz = so.rays(px[e], pz[e], ang[e], cfg)
            ok = ~amb
            n_amb += int(amb.sum())
            n_all += amb.size
            before = np.maximum(rng - so.EPS, 0)
            b0, _ = so.blocked_label(sc, ox + before * dx, oz + before * dz, feet)
            assert not (b0 & ok & (rng > so.EPS)).any(), f"{name} env {e}: blocked before t*"
            after = np.where(hit == 0, rng, rng + so.EPS)
            b1, lab1 = so.blocked_label(sc, ox + after * dx, oz + after * dz, feet)
            stop = ok & (hit != 0) & (rng > 0)
            assert (b1[stop] & (lab1[stop] == hit[stop])).all(), f"{name} env {e}: hit does not name the blocker"
            org = ok & (rng == 0)
            if org.any():
                bo_, lo = so.blocked_label(sc, np.float64(ox), np.float64(oz), feet)
                assert bo_ and (hit[org] == lo).all()
            assert (rng[hit == 0] == cfg[2]).all()
            n_obj += int((hit >= 2 + sc.n_cells).sum())
    assert n_amb < 0.01 * n_all
    if md.objects:
        assert n_obj > 0, f"{name}: no ray met an object"


def test_ctypes_struct_matches_the_header():
    import ctypes as C
    from gym_duckietown_b200 import lib as L
    with open(os.path.join(ROOT, "include", "dtsim.h")) as f:
        h = f.read()
    body = re.search(r"typedef struct \{([^{}]*)\} dts_scan_config;", h).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(n.strip(), ctype) for n in names.split(",")]
    ctypes_of = {"int32_t": C.c_int32, "double": C.c_double}
    assert [(n, ctypes_of[t]) for n, t in fields] == list(L.ScanConfig._fields_)
    assert C.sizeof(L.ScanConfig) == 40 and L.ScanConfig.fov.offset == 8
