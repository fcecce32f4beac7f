"""The bird's-eye oracle (tests/bev_oracle.py, DESIGN.md section 5 item 12) on the CPU: hand-built maps whose grids are
written out by hand, at every tile angle; the same texel rule checked against the rasteriser's own markings and labels
by casting each pixel's ray onto the ground; and the footprints the map blob hands the library."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import bev_oracle as bo
from gym_duckietown_b200 import assets
from gym_duckietown_b200 import lib as L
from gym_duckietown_b200 import maps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W_, Y_ = assets.MARK_WHITE, assets.MARK_YELLOW
ORIENT = ["S", "E", "N", "W"]


def hand_map(rows, objects=(), ts=1.0):
    return maps.interpret_map({"tile_size": ts, "tiles": rows, "objects": list(objects)}, "hand")


def painted(n=4, column=None, row=None):
    """An n x n class plane of bare tile (1) with texel column `column` white and texel row `row` yellow"""
    p = np.full((n, n), assets.MARK_TILE, np.uint8)
    if column is not None:
        p[:, column] = W_
    if row is not None:
        p[row, :] = Y_
    return p


def one_tile_scene(angle, plane):
    md = hand_map([[f"straight/{ORIENT[angle]}"]])
    sc = bo.BevScene(md)
    sc.classes[int(sc.tile_tex[0])] = plane
    return sc


# The 4 x 4 grid of 0.25 m cells over the one 1 m tile, the agent at its centre facing +x (angle 0): row r lies at
# x = 0.875 - 0.25 r (row 0 ahead), column c at z = 0.125 + 0.25 c (the agent's right is +z).
GRID = (4, 4, 0.25, 2.0, 2.0)
# texel column 0 painted white: where the white line lands in the grid, per tile angle S, E, N, W
WHITE_COLUMN = {
    0: [[2, 2, 2, 2], [1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1]],
    1: [[2, 1, 1, 1], [2, 1, 1, 1], [2, 1, 1, 1], [2, 1, 1, 1]],
    2: [[1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1], [2, 2, 2, 2]],
    3: [[1, 1, 1, 2], [1, 1, 1, 2], [1, 1, 1, 2], [1, 1, 1, 2]],
}
# texel row 0 painted yellow
YELLOW_ROW = {
    0: [[3, 1, 1, 1], [3, 1, 1, 1], [3, 1, 1, 1], [3, 1, 1, 1]],
    1: [[1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1], [3, 3, 3, 3]],
    2: [[1, 1, 1, 3], [1, 1, 1, 3], [1, 1, 1, 3], [1, 1, 1, 3]],
    3: [[3, 3, 3, 3], [1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1]],
}
# texel column 0 white, the agent turned to face -z (angle pi / 2): row r at z = 0.125 + 0.25 r, column c at
# x = 0.125 + 0.25 c
WHITE_COLUMN_TURNED = {
    0: [[1, 1, 1, 2], [1, 1, 1, 2], [1, 1, 1, 2], [1, 1, 1, 2]],
    1: [[2, 2, 2, 2], [1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1]],
    2: [[2, 1, 1, 1], [2, 1, 1, 1], [2, 1, 1, 1], [2, 1, 1, 1]],
    3: [[1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1], [2, 2, 2, 2]],
}


@pytest.mark.parametrize("angle", range(4))
def test_one_tile_paint_lands_where_the_tile_angle_puts_it(angle):
    for plane, want, pose in ((painted(column=0), WHITE_COLUMN, 0.0), (painted(row=0), YELLOW_ROW, 0.0),
                              (painted(column=0), WHITE_COLUMN_TURNED, math.pi / 2)):
        sc = one_tile_scene(angle, plane)
        lab, mk, amb, _ = bo.bev_grid(sc, 0.5, 0.5, pose, GRID)
        assert not amb.any()
        assert (lab == 2).all()                      # the one cell (0, 0): 2 + 0 * grid_h + 0
        assert np.array_equal(mk, np.array(want[angle])), (angle, pose, mk)


def test_one_tile_off_the_grid_is_ground_without_paint():
    sc = one_tile_scene(0, painted(column=0))
    # 8 x 2 cells of 0.25 m ahead of an agent at the tile's far edge (x = 1, facing +x): rows 0-3 beyond it
    lab, mk, amb, _ = bo.bev_grid(sc, 1.0, 0.5, 0.0, (2, 8, 0.25, 1.0, 4.0))
    assert not amb.any()
    assert np.array_equal(lab[:, 0], [1, 1, 1, 1, 2, 2, 2, 2]) and np.array_equal(mk[:4], np.zeros((4, 2)))
    assert np.array_equal(mk[4:, 0], [2, 1, 1, 1])   # back on the tile: texel column tu = floor(4 (1 - x)) with angle S


def test_two_by_two_labels_name_each_cell_and_leave_empty_ones_ground():
    md = hand_map([["straight/E", "curve_left/N"], ["empty", "grass"]])
    sc = bo.BevScene(md)
    # agent near (1, 1) facing +x; 4 x 4 cells of 0.5 m: rows at x ~ 1.75, 1.25, 0.75, 0.25, columns at z ~ 0.25 .. 1.75
    # (moved off the texel edges a power-of-two texture has at multiples of 1/4 tile)
    lab, mk, amb, _ = bo.bev_grid(sc, 1.01, 1.013, 0.0, (4, 4, 0.5, 2.0, 2.0))
    assert not amb.any()
    # cell (i, j) has label 2 + 2 i + j; (0, 1) is empty -> 1
    want = [[4, 4, 5, 5], [4, 4, 5, 5], [2, 2, 1, 1], [2, 2, 1, 1]]
    assert np.array_equal(lab, np.array(want)), lab
    assert (mk[lab == 1] == 0).all() and (mk[lab >= 2] >= 1).all()
    # the grass tile's texture is bare tile everywhere
    assert (mk[lab == 5] == assets.MARK_TILE).all()


def test_objects_take_the_smallest_index_skip_hidden_ones_and_leave_markings():
    objs = [{"kind": "duckie", "pos": [0.5, 0.5], "height": 0.06}, {"kind": "duckie", "pos": [0.5, 0.5], "height": 0.06}]
    md = hand_map([["straight/S"]], objs)
    sc = bo.BevScene(md)
    sc.classes[int(sc.tile_tex[0])] = painted(column=0)
    # footprints by hand: object 0 the square [0.5, 1] x [0, 0.5], object 1 [0.25, 0.75] x [0.25, 0.75]
    sc.corners = [np.array([[0.5, 0.0], [1.0, 0.0], [1.0, 0.5], [0.5, 0.5]]),
                  np.array([[0.75, 0.25], [0.25, 0.25], [0.25, 0.75], [0.75, 0.75]])]   # (the other winding)
    n = 1
    lab, mk, amb, _ = bo.bev_grid(sc, 0.5, 0.5, 0.0, GRID)
    o0, o1, tile = 2 + n, 3 + n, 2
    want = [[o0, o0, tile, tile], [o0, o0, o1, tile], [tile, o1, o1, tile], [tile, tile, tile, tile]]
    assert not amb.any()
    assert np.array_equal(lab, np.array(want)), lab
    assert np.array_equal(mk, np.array(WHITE_COLUMN[0]))   # paint under the objects is still reported
    hidden = np.zeros(8, np.uint32)
    hidden[0] = 1
    lab, _, _, _ = bo.bev_grid(sc, 0.5, 0.5, 0.0, GRID, hidden=hidden)
    want = [[tile] * 4, [tile, o1, o1, tile], [tile, o1, o1, tile], [tile] * 4]
    assert np.array_equal(lab, np.array(want)), lab


def test_a_cell_on_a_footprint_edge_is_ambiguous_and_a_moved_obstacle_moves():
    objs = [{"kind": "duckie", "pos": [0.5, 0.5], "height": 0.06, "static": False}]
    md = hand_map([["straight/S"]], objs)
    sc = bo.BevScene(md)
    sc.classes[int(sc.tile_tex[0])] = painted()
    sq = np.array([[0.5, 0.0], [1.0, 0.0], [1.0, 0.375], [0.5, 0.375]])   # an edge through column 1's centres
    lab, _, amb, _ = bo.bev_grid(sc, 0.5, 0.5, 0.0, GRID, env_corners=[sq])
    assert amb[:2, 1].all() and amb.sum() == 2
    assert (lab[:2, 1] == 3).all() and (lab[:2, 0] == 3).all() and (lab[2:] == 2).all()
    moved = sq - [0.5, 0.0]
    lab, _, _, _ = bo.bev_grid(sc, 0.5, 0.5, 0.0, GRID, env_corners=[moved])
    assert (lab[:2] == 2).all() and (lab[2:, 0] == 3).all()


# ------------------------------------------------------------------------------------------------ camera cross-check
@pytest.fixture(scope="module")
def built():
    import oracle as orc
    orc.build()
    return orc


SAMPLES = [(-0.125, -0.375), (0.375, -0.125), (-0.375, 0.125), (0.125, 0.375)]   # 4x MSAA, from the pixel centre
JITTER = [(0, 0), (1 / 64, 0), (-1 / 64, 0), (0, 1 / 64), (0, -1 / 64)]            # the vertices' 1/64 px snap


def ground_points(V, P, W, H, dx=0.0, dy=0.0):
    """Where each pixel's ray through (x + .5 + dx, y + .5 + dy) meets the plane y = 0: (x, z) [H, W]"""
    R, t = V[:, :3], V[:, 3]
    c, r = np.meshgrid(np.arange(W) + 0.5 + dx, np.arange(H) + 0.5 + dy)
    nx, ny = c / W * 2 - 1, 1 - r / H * 2
    d_eye = np.stack([nx / P[0], ny / P[1], -np.ones_like(nx)], -1)
    o_w, d_w = -R.T @ t, d_eye @ R          # R.T @ d for every pixel
    s = -o_w[1] / d_w[..., 1]
    return o_w[0] + d_w[..., 0] * s, o_w[2] + d_w[..., 2] * s


@pytest.mark.parametrize("name,top_down", [("small_loop", False), ("udem1", False), ("loop_obstacles", False),
                                           ("small_loop", True), ("udem1", True)])
def test_ground_under_each_tile_pixel_is_what_the_rasteriser_shows(name, top_down, built):
    """Every pixel whose raster label is a tile: the ground point its centre ray meets, classified by the oracle (objects
    left out: the camera sees the ground there), gives the rasteriser's label and marking for at least 99 % of those
    whose samples all meet the centre's tile.  Every other one shows its label through one of its samples, or its
    marking within one texel or 1/64 px."""
    import label_oracle
    import marking_oracle
    md = maps.load_map(name)
    osc, sc = built.OracleScene(md), bo.BevScene(md)
    n_cells = md.grid_w * md.grid_h
    W, H = (320, 240) if top_down else (160, 120)
    rng = np.random.default_rng(9)
    poses = []
    while len(poses) < (2 if top_down else 6):
        i, j = md.drivable_tiles[rng.integers(len(md.drivable_tiles))]
        poses.append(((i + rng.uniform(0.2, 0.8)) * md.tile_size, (j + rng.uniform(0.2, 0.8)) * md.tile_size,
                      rng.uniform(-np.pi, np.pi)))
    texel = md.tile_size / min(sc.classes[t].shape[1] for t in set(sc.tile_tex[sc.tile_tex >= 0].tolist()))
    near = [(a * texel, b * texel) for a in (-1, 0, 1) for b in (-1, 0, 1) if a or b]
    n_px = n_bad = 0
    for px, pz, ang in poses:
        _, _, lab, mk = marking_oracle.render(osc, px, pz, ang, W=W, H=H, top_down=top_down)
        dbg = label_oracle.debug_frame(osc, px, pz, ang, W=W, H=H, top_down=top_down)
        V, P = dbg["V"].reshape(3, 4), dbg["P"].astype(np.float64)
        tile_px = (lab >= 2) & (lab < 2 + n_cells)
        x, z = ground_points(V, P, W, H)
        gl, gm = bo.classify_points(sc, x, z, [])
        bad = tile_px & ~((gl == lab) & (gm == mk))
        # The label is decided by the pixel's four samples (render spec item 5; either vertical convention), so a label
        # that differs must be the oracle's through one of them, give or take the rasteriser's 1/64 px snap: at a tile's
        # border a sample can see the tile while the centre ray does not, and the marking of such a pixel is then taken
        # at the centre from outside its tile.  A marking that differs under the right label must be the oracle's within
        # one texel or 1/64 px.
        ok_label, border = np.zeros_like(bad), np.zeros_like(bad)
        for sx, sy in SAMPLES:
            for flip in (1, -1):
                for jx, jy in JITTER:
                    xs, zs = ground_points(V, P, W, H, sx + jx, flip * sy + jy)
                    sl = bo.classify_points(sc, xs, zs, [])[0]
                    ok_label |= sl == lab
                    border |= sl != gl
        # the bar counts the pixels whose samples all meet the centre's tile (or all miss the grid alike)
        n_px += int((tile_px & ~border).sum())
        n_bad += int((bad & ~border).sum())
        ok_mark = np.zeros_like(bad)
        probes = [(x + dx, z + dz) for dx, dz in near]
        probes += [ground_points(V, P, W, H, dx, dy) for dx, dy in ((1 / 64, 0), (-1 / 64, 0), (0, 1 / 64), (0, -1 / 64))]
        for xs, zs in probes:
            al, am = bo.classify_points(sc, xs, zs, [])
            ok_mark |= (al == lab) & (am == mk)
        far = bad & np.where(gl != lab, ~ok_label, ~ok_mark)
        assert not far.any(), (name, top_down, (px, pz, ang), np.argwhere(far)[:5])
    assert n_px > 1000 and n_bad <= 0.01 * n_px, (n_bad, n_px)


# ------------------------------------------------------------------------------------------------ blob footprints
def test_blob_hands_over_every_objects_corners():
    for name in ("udem1", "loop_dyn_duckiebots", "loop_trafficlights", "small_loop"):
        md = maps.load_map(name)
        h = L.MapBlobHolder(md)
        assert h.blob.obj_corners
        got = np.ctypeslib.as_array(ctypes.cast(h.blob.obj_corners, ctypes.POINTER(ctypes.c_double)),
                                    (max(1, len(md.objects)) * 8,))
        want = np.array([o.corners for o in md.objects], np.float64).reshape(-1)
        assert np.array_equal(got[:want.size], want), name
        assert all(np.array_equal(o.corners, maps.obb_corners(o.pos, md.meshes[o.mesh_id].min_coords,
                                                              md.meshes[o.mesh_id].max_coords, o.angle, o.scale))
                   for o in md.objects)


def test_ctypes_bev_config_and_blob_match_the_header():
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dtsim.h"
    int main(){ printf("%zu %zu %zu %zu %zu %zu\n", sizeof(dts_bev_config), offsetof(dts_bev_config, cell),
      offsetof(dts_bev_config, origin_x), offsetof(dts_bev_config, origin_y), sizeof(dts_map_blob),
      offsetof(dts_map_blob, obj_corners)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "bev_layout_probe")
        subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe], input=src, text=True,
                       check=True)
        vals = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert vals == [ctypes.sizeof(L.BevConfig), L.BevConfig.cell.offset, L.BevConfig.origin_x.offset,
                    L.BevConfig.origin_y.offset, ctypes.sizeof(L.MapBlob), L.MapBlob.obj_corners.offset]
