"""The bird's-eye visibility oracle (tests/bev_view_oracle.py, DESIGN.md section 5 item 15) tied to the raster oracle's
own frames, without a GPU: flat one-tile and two-by-two maps at every tile angle, a duckie placed by hand ahead of the
agent (pinhole, the default fisheye and one camera_rand table), and for the pinhole camera the cell <-> pixel link both
ways (the depth the rasteriser measured where a visible cell lands, and tile pixels cast onto the ground and projected
back)."""
import numpy as np
import pytest

import bev_oracle as bo
import bev_view_oracle as vo
import flow_oracle as fo
import label_oracle
import oracle as orc
from gym_duckietown_b200 import maps

W, H = 160, 120
CFG = (64, 64, 0.03, 32.0, 48.0)   # the default grid: 1.44 m ahead, 0.48 m behind
ORIENT = ["S", "E", "N", "W"]
CAMERAS = ["pinhole", "fisheye", "camera_rand"]
# Cast back, pinhole: every tile pixel of these frames lands within half a pixel of its own centre (measured 1.0).
CAST_BAR = 0.99

_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def built():
    orc.build()


def camera(kind):
    """None for the pinhole camera; the default fisheye; table 2 of a camera_rand pool of 4"""
    if kind == "pinhole":
        return None
    if kind not in _MODELS:
        from gym_duckietown_b200.distortion import Distortion, draw_calibrations
        if kind == "fisheye":
            _MODELS[kind] = Distortion(W, H)
        else:
            K, D = draw_calibrations(4, 3)[2]
            _MODELS[kind] = Distortion(W, H, K, D)
    return _MODELS[kind]


def hand_map(rows, objects=()):
    return maps.interpret_map({"tile_size": 0.585, "tiles": rows, "objects": list(objects)}, "hand")


def view(md, pose, kind, cfg=CFG):
    """The oracle's answer for the camera at pose over the raster oracle's frame, with that frame's depth, labels, V, P"""
    m = camera(kind)
    osc, bsc = orc.OracleScene(md), bo.BevScene(md)
    _, dep, lab = label_oracle.render_batch(osc, [pose[0]], [pose[1]], [pose[2]], W=W, H=H,
                                            lut=(m.rmapx, m.rmapy) if m else None)
    dbg = label_oracle.debug_frame(osc, *pose, W=W, H=H)
    grid = bo.bev_grid(bsc, *pose, cfg)
    r = vo.visibility(bsc, pose, cfg, grid, dbg["V"], dbg["P"], lab[0], (m.mapx, m.mapy) if m else None)
    return r, grid, dep[0], lab[0], dbg["V"].reshape(3, 4), dbg["P"].astype(np.float64)


def plane_depth(V, P, u, v, y0):
    """Eye depth where the pinhole ray through (u, v) (pixel units) meets the plane y = y0"""
    R, t = V[:, :3], V[:, 3]
    d_eye = np.stack([(2 * u / W - 1) / P[0], (1 - 2 * v / H) / P[1], -np.ones_like(u)], -1)
    o_w, d_w = -R.T @ t, d_eye @ R
    return (y0 - o_w[1]) / d_w[..., 1]


def world_point(V, P, u, v, y0):
    R, t = V[:, :3], V[:, 3]
    d_eye = np.stack([(2 * u / W - 1) / P[0], (1 - 2 * v / H) / P[1], -np.ones_like(u)], -1)
    o_w, d_w = -R.T @ t, d_eye @ R
    s = (y0 - o_w[1]) / d_w[..., 1]
    return o_w[0] + d_w[..., 0] * s, o_w[1] + d_w[..., 1] * s, o_w[2] + d_w[..., 2] * s


def tile_edge_cells(grid, r=1):
    """cells within r cells of a cell with another label"""
    lab = grid[0]
    out = np.zeros(lab.shape, bool)
    pad = np.pad(lab, r, mode="edge")
    h, w = lab.shape
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            out |= pad[r + dy:r + dy + h, r + dx:r + dx + w] != lab
    return out


@pytest.mark.parametrize("kind", CAMERAS)
@pytest.mark.parametrize("layout", ["one", "two"])
def test_flat_maps_at_every_tile_angle(kind, layout):
    n_vis = n_occ = 0
    for angle in range(4):
        rows = [[f"straight/{ORIENT[angle]}"]] if layout == "one" else \
            [[f"straight/{ORIENT[angle]}", f"curve_left/{ORIENT[angle]}"], [f"3way_left/{ORIENT[angle]}", "asphalt"]]
        md = hand_map(rows)
        ts = md.tile_size
        for heading in (0.3, 2.2, -1.9):
            pose = (0.5 * ts + 0.013, 0.5 * ts - 0.021, heading)
            r, grid, dep, lab, V, P = view(md, pose, kind)
            val, w = r["value"], r["w"]
            x, z = bo.cell_centres(*pose, *CFG)
            y1 = vo.project(V.ravel(), P, W, H, x, vo.surface_height(bo.BevScene(md), x, z), z)["y1"]
            where = (layout, angle, heading, kind)
            assert (val[w <= vo.NEAR] == vo.OUTSIDE).all(), where            # behind the camera
            assert (val[(w > vo.NEAR) & (y1 > H + 2)] == vo.OUTSIDE).all(), where   # below the frame's bottom edge
            tile = (grid[0] >= 2) & ~r["ambiguous"] & ~tile_edge_cells(grid)
            inframe = tile & ~np.isnan(r["q"][..., 0])
            assert (val[inframe] == vo.VISIBLE).all(), (where, np.argwhere(inframe & (val != vo.VISIBLE))[:5])
            # The ground quad lies 8 mm below the tiles, so a tile's edge hides a strip of ground beyond it: away from
            # the edges between two tiles (whose labels differ a pixel from the edge), the only occluded cells are ground
            # cells whose ray crosses the tiles' plane over a tile (one-tile map, pinhole; the fisheye's gather moves q up to a
            # pixel)
            occ = (val == vo.OCCLUDED) & ~(tile_edge_cells(grid) & (grid[0] >= 2))
            assert layout == "two" or (grid[0][occ] == 1).all(), where
            o = -V[:, :3].T @ V[:, 3]
            s = o[1] / (o[1] - vo.GROUND_Y)
            cross = bo.classify_points(bo.BevScene(md), o[0] + s * (x[occ] - o[0]), o[2] + s * (z[occ] - o[2]), [])[0]
            assert kind != "pinhole" or layout == "two" or (cross >= 2).all(), where
            n_vis += int(inframe.sum())
            n_occ += int(occ.sum())
    assert n_vis > 400 and n_occ > 0


@pytest.mark.parametrize("kind", CAMERAS)
def test_a_duckie_hides_the_cells_behind_it(kind):
    ts = 0.585
    md = hand_map([["straight/E"] * 4], [{"kind": "duckie", "pos": [1.25, 0.5], "height": 0.06}])
    pose = (0.3, 0.5 * ts, 0.0)   # facing +x, the duckie 0.43 m ahead
    r, grid, dep, lab, V, P = view(md, pose, kind)
    duck = 2 + md.grid_w * md.grid_h
    val = r["value"]
    occ = (val == vo.OCCLUDED) & ~tile_edge_cells(grid)   # (not the edges between tiles, whose labels differ)
    assert occ.sum() >= 10, occ.sum()
    q = r["q"][occ]
    cx, cy = np.floor(q[:, 0] - 0.5).astype(int), np.floor(q[:, 1] - 0.5).astype(int)
    shows = np.zeros(len(q), bool)
    deeper = np.zeros(len(q), bool)
    for j in (0, 1):
        for i in (0, 1):
            sx, sy = np.clip(cx + i, 0, W - 1), np.clip(cy + j, 0, H - 1)
            hit = lab[sy, sx] == duck
            shows |= hit
            deeper |= hit & (r["w"][occ] > dep[sy, sx])
    # every hidden cell is behind the duckie on its ray (under the fisheye all but its gather's strays, here 1 of 19)
    bar = 1.0 if kind == "pinhole" else 0.9
    assert shows.mean() >= bar and deeper.mean() >= bar, (shows.mean(), deeper.mean())
    # the cells beside it: tile cells whose pixels show no duckie are visible
    cc = np.nan_to_num(r["q"], nan=-10.0)
    near_duck = np.zeros(val.shape, bool)
    for j in (-1, 0, 1, 2):
        for i in (-1, 0, 1, 2):
            sx = np.clip(np.floor(cc[..., 0] - 0.5).astype(int) + i, 0, W - 1)
            sy = np.clip(np.floor(cc[..., 1] - 0.5).astype(int) + j, 0, H - 1)
            near_duck |= lab[sy, sx] == duck
    beside = (grid[0] >= 2) & (grid[0] < duck) & ~near_duck & ~np.isnan(r["q"][..., 0]) & ~tile_edge_cells(grid)
    assert beside.sum() > 200 and (val[beside] == vo.VISIBLE).all()


@pytest.mark.parametrize("kind", ["pinhole"])
def test_visible_cells_land_at_their_own_depth(kind):
    """A visible tile cell's eye depth lies within the depths of the ground under the pixel nearest q"""
    md = maps.load_map("small_loop")
    rng = np.random.default_rng(5)
    checked = 0
    m = camera(kind)
    src = fo.src_of_lut(m.rmapx, m.rmapy) if m else None
    for k in range(3):
        i, j = md.drivable_tiles[rng.integers(len(md.drivable_tiles))]
        pose = ((i + rng.uniform(0.3, 0.7)) * md.tile_size, (j + rng.uniform(0.3, 0.7)) * md.tile_size,
                rng.uniform(-np.pi, np.pi))
        r, grid, dep, lab, V, P = view(md, pose, kind)
        sel = (r["value"] == vo.VISIBLE) & (grid[0] >= 2) & (grid[0] < 2 + md.grid_w * md.grid_h) & ~r["ambiguous"]
        sel &= ~tile_edge_cells(grid)
        q = r["q"][sel]
        ix, iy = np.floor(q[:, 0]).astype(int), np.floor(q[:, 1]).astype(int)
        sx, sy = (ix, iy) if src is None else (src[0][iy, ix], src[1][iy, ix])
        pad = 0.0 if src is None else 1.0
        corners = [plane_depth(V, P, sx + a, sy + b, 0.0) for a in (-pad, 1 + pad) for b in (-pad, 1 + pad)]
        lo, hi = np.minimum.reduce(corners), np.maximum.reduce(corners)
        w = r["w"][sel]
        assert ((w >= lo * (1 - 1e-3)) & (w <= hi * (1 + 1e-3))).all(), (kind, k)
        assert np.all(np.abs(dep[iy, ix] - w) <= (hi - lo) + 1e-3 * w), (kind, k)
        checked += int(sel.sum())
    assert checked > 1000


@pytest.mark.parametrize("kind", ["pinhole"])
def test_tile_pixels_cast_onto_the_ground_come_back_to_themselves(kind):
    md = maps.load_map("udem1")
    rng = np.random.default_rng(7)
    m = camera(kind)
    src = fo.src_of_lut(m.rmapx, m.rmapy) if m else None
    n_px = n_ok = 0
    for k in range(3):
        i, j = md.drivable_tiles[rng.integers(len(md.drivable_tiles))]
        pose = ((i + rng.uniform(0.3, 0.7)) * md.tile_size, (j + rng.uniform(0.3, 0.7)) * md.tile_size,
                rng.uniform(-np.pi, np.pi))
        r, grid, dep, lab, V, P = view(md, pose, kind)
        py, px = np.mgrid[0:H, 0:W]
        sx, sy = (px, py) if src is None else src
        tile = (lab >= 2) & (lab < 2 + md.grid_w * md.grid_h) & (sx >= 0)
        x, y, z = world_point(V, P, sx[tile] + 0.5, sy[tile] + 0.5, 0.0)
        p = vo.project(V.ravel(), P, W, H, x, y, z, (m.mapx, m.mapy) if m else None)
        err = np.hypot(p["qx"] - (px[tile] + 0.5), p["qy"] - (py[tile] + 0.5))
        n_px += int(tile.sum())
        n_ok += int((err <= 0.5).sum())
    assert n_px > 5000 and n_ok >= CAST_BAR * n_px, (kind, n_ok / n_px)
