"""The flow oracle (tests/flow_oracle.py, DESIGN.md section 5 item 13) tied to the rasteriser without a GPU: frames of two
consecutive states from the raster, depth and label oracles (pinhole and fisheye cameras on small_loop, loop_obstacles
and udem1, and an obstacle that moved), and two checks that pin the flow's sign, its row direction, the half-pixel
convention and the fisheye's forward map against the renders themselves.

- Label warp: a pixel with valid flow whose previous position q = p + flow lies in the previous frame, at least one pixel
  from any label edge there, and not occluded (the previous depth at q is at least the point's depth in the previous
  camera x (1 - 1e-3)), shows the same item at q in the previous frame.
- Depth warp: a road-tile pixel's point lies, in the previous pinhole frame, at the depth that frame measured at its
  pinhole position (inverse depth interpolated bilinearly, which is exact on a plane), within 1e-3 relative.
"""
import numpy as np
import pytest

import flow_oracle as fo
import label_oracle
import oracle as orc

W, H = 160, 120
# Bars, from what the checks measure here (10 pose pairs per map at 160 x 120).  Label warp, pinhole: 0.99995-0.99997
# (the misses are pixels on an object's silhouette).  Fisheye: 0.9881-0.9914, moved obstacle 0.9981: the fisheye frame is
# a nearest-neighbour gather whose source pixel lies up to half a pinhole pixel off the inverse of F at the output pixel,
# and its inverse map is a splatted approximation of F's inverse, so q lands a pixel off near edges.  Depth warp:
# 0.9870-0.9940; the misses are tiles more than 2 m away, where the snapping of vertices to 1/64 px moves a tile's depth
# plane by more than 1e-3 relative (DESIGN.md section 5 item 9).
LABEL_BAR = {False: 0.999, True: 0.985}
DEPTH_BAR = 0.985


@pytest.fixture(scope="module", autouse=True)
def built():
    orc.build()


def label_warp(flow, lab, lab_prev, dep_prev, z_prev):
    """(pixels whose previous position shows their item, pixels checked) of one frame"""
    h, w = lab.shape
    y, x = np.mgrid[0:h, 0:w]
    ok = ~np.isnan(flow[..., 0])
    qx = np.where(ok, x + 0.5 + flow[..., 0], -10.0)
    qy = np.where(ok, y + 0.5 + flow[..., 1], -10.0)
    ix, iy = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    ok &= (ix >= 1) & (ix <= w - 2) & (iy >= 1) & (iy <= h - 2)
    uniform = np.ones((h, w), bool)   # the 3 x 3 block around a pixel of the previous frame shows one item
    pad = np.pad(lab_prev, 1, mode="edge")
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            uniform &= pad[1 + dy:1 + dy + h, 1 + dx:1 + dx + w] == lab_prev
    cx, cy = np.clip(ix, 0, w - 1), np.clip(iy, 0, h - 1)
    ok &= uniform[cy, cx]
    ok &= dep_prev[cy, cx] >= np.where(ok, z_prev, 0) * (1 - 1e-3)   # not hidden in the previous frame
    hits = ok & (lab_prev[cy, cx] == lab)
    return int(hits.sum()), int(ok.sum())


def depth_warp(x1, y1, z_prev, lab, lab_prev_pin, dep_prev_pin, n_tiles):
    """(road-tile pixels whose point lies at the previous pinhole frame's depth within 1e-3 relative, pixels checked)"""
    h, w = lab_prev_pin.shape
    tile = (lab >= 2) & (lab <= 1 + n_tiles) & ~np.isnan(x1)
    ix, iy = np.where(tile, x1 - 0.5, -10.0), np.where(tile, y1 - 0.5, -10.0)
    x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
    ok = tile & (x0 >= 0) & (x0 <= w - 2) & (y0 >= 0) & (y0 <= h - 2)
    cx, cy = np.clip(x0, 0, w - 2), np.clip(y0, 0, h - 2)
    taps = [(cy, cx), (cy, cx + 1), (cy + 1, cx), (cy + 1, cx + 1)]
    for ty, tx in taps:   # every tap on a road tile (one plane), none hidden by an object
        ok &= (lab_prev_pin[ty, tx] >= 2) & (lab_prev_pin[ty, tx] <= 1 + n_tiles)
    inv = [np.where(ok, 1.0 / np.where(ok, dep_prev_pin[ty, tx], 1.0), 0.0) for ty, tx in taps]
    ax, ay = ix - cx, iy - cy
    q = (inv[0] * (1 - ax) + inv[1] * ax) * (1 - ay) + (inv[2] * (1 - ax) + inv[3] * ax) * ay
    with np.errstate(divide="ignore", invalid="ignore"):
        hits = ok & (np.abs(1.0 / q - z_prev) <= 1e-3 * z_prev)
    return int(hits.sum()), int(ok.sum())


def scene(name):
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    return md, orc.OracleScene(md)


def pose_pairs(md, n, seed):
    """n cameras on drivable tiles and where each is one step later: up to 6 cm ahead, up to 0.1 rad turned"""
    rng = np.random.default_rng(seed)
    tiles = [md.drivable_tiles[k] for k in rng.integers(0, len(md.drivable_tiles), n)]
    ts = md.tile_size
    px = np.array([(i + rng.uniform(0.2, 0.8)) * ts for i, _ in tiles])
    pz = np.array([(j + rng.uniform(0.2, 0.8)) * ts for _, j in tiles])
    a = rng.uniform(-np.pi, np.pi, n)
    d, t = rng.uniform(0.0, 0.06, n), rng.uniform(-0.1, 0.1, n)
    return (px, pz, a), (px + d * np.cos(a), pz - d * np.sin(a), a + t)


_MODELS = {}


def fisheye():
    if "m" not in _MODELS:
        from gym_duckietown_b200.distortion import Distortion
        _MODELS["m"] = Distortion(W, H)
    return _MODELS["m"]


def frame(sc, p, lut):
    """(depth, labels) of the camera p, and its V, P"""
    _, dep, lab = label_oracle.render_batch(sc, [p[0]], [p[1]], [p[2]], W=W, H=H, lut=lut)
    dbg = label_oracle.debug_frame(sc, p[0], p[1], p[2], W=W, H=H)
    return dep[0], lab[0], dbg["V"], dbg["P"]


def warps(md, sc, p0, p1, fish, moves=None, move=None):
    """Both checks for one pair of states; `move(sc, k)` puts the scene's moving object in state k first"""
    m = fisheye() if fish else None
    lut = (m.rmapx, m.rmapy) if fish else None
    src = fo.src_of_lut(*lut) if fish else None
    fwd = (m.mapx, m.mapy) if fish else None
    n_tiles = md.grid_w * md.grid_h
    if move:
        move(sc, 0)
    dep0, lab0, V0, _ = frame(sc, p0, lut)
    dep0p, lab0p, _, _ = frame(sc, p0, None)
    if move:
        move(sc, 1)
    dep1, lab1, V1, P1 = frame(sc, p1, lut)
    r = fo.flow(dep1, lab1, P1, V0, V1, n_tiles, len(md.objects), moves, src=src, fwd=fwd)
    lw = label_warp(r["flow"], lab1, lab0, dep0, r["z_prev"])
    dw = depth_warp(r["x1"], r["y1"], r["z_prev"], lab1, lab0p, dep0p, n_tiles)
    return lw, dw


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles", "udem1"])
@pytest.mark.parametrize("fish", [False, True])
def test_label_and_depth_warps(name, fish):
    md, sc = scene(name)
    (px0, pz0, a0), (px1, pz1, a1) = pose_pairs(md, 10, 21)
    lh = lt = dh = dt = 0
    for k in range(len(px0)):
        (a, b), (c, d) = warps(md, sc, (px0[k], pz0[k], a0[k]), (px1[k], pz1[k], a1[k]), fish)
        lh, lt, dh, dt = lh + a, lt + b, dh + c, dt + d
    assert lt > 20000 and dt > 10000
    assert lh >= LABEL_BAR[fish] * lt, f"label warp {lh} / {lt}"
    assert dh >= DEPTH_BAR * dt, f"depth warp {dh} / {dt}"


@pytest.mark.parametrize("fish", [False, True])
def test_warps_with_a_moved_obstacle(fish):
    """loop_obstacles with object 0 moved 4 cm and turned 12 degrees between the frames, seen from 0.35 m behind it"""
    md, sc = scene("loop_obstacles")
    ob = md.objects[0]
    x, y, z = (float(v) for v in ob.pos)
    deg = float(np.rad2deg(ob.angle))
    states = [((x, y, z), deg), ((x + 0.03, y, z - 0.025), deg + 12.0)]

    def move(s, k):
        s.set_object_pose(0, *states[k])
    moves = {0: ((np.float32(states[0][0][0]), np.float32(states[0][0][2]), np.float32(states[0][1])),
                 (np.float32(states[1][0][0]), np.float32(states[1][0][2]), np.float32(states[1][1])))}
    lh = lt = 0
    try:
        for k, a in enumerate(np.linspace(-np.pi, np.pi, 8, endpoint=False)):
            p0 = (x - 0.35 * np.cos(a), z + 0.35 * np.sin(a), a)
            p1 = (p0[0] + 0.01, p0[1], a + 0.02)
            (h, t), _ = warps(md, sc, p0, p1, fish, moves, move)
            lh, lt = lh + h, lt + t
    finally:
        sc.set_object_pose(0, (x, y, z), deg)
    assert lt > 20000
    assert lh >= LABEL_BAR[fish] * lt, f"label warp {lh} / {lt}"


def test_still_scene_has_zero_flow():
    """The same camera twice: every defined pixel's flow is 0 to 1e-9 px (the oracle in float64)"""
    md, sc = scene("udem1")
    (px0, pz0, a0), _ = pose_pairs(md, 3, 5)
    for k in range(3):
        p = (px0[k], pz0[k], a0[k])
        dep, lab, V, P = frame(sc, p, None)
        r = fo.flow(dep, lab, P, V, V, md.grid_w * md.grid_h, len(md.objects))
        f = r["flow"][~np.isnan(r["flow"][..., 0])]
        assert f.size and np.abs(f).max() < 1e-9
