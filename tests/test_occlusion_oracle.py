"""The occlusion oracle (tests/occlusion_oracle.py, DESIGN.md section 5 item 14) tied to the rasteriser without a GPU:
frames of the raster, depth and label oracles, pinhole and fisheye, in scenes where what was hidden is known without
the pixel rule.

- A still camera and an obstacle moved by hand: road the obstacle covered is occluded, road far from it is visible.
- A flat world (small_loop, no objects) seen from a moving camera: nothing can be occluded.
- A static obstacle and a moving, turning camera: the previous frame rendered again with the obstacle hidden (the
  episode's `hidden` mask) says which road pixels only the obstacle hid.
- A duckie turned 180 degrees in place: the side it now shows was its far side.  With an unturned duckie seen from a
  moving camera, this check sets tau.
"""
import numpy as np
import pytest

import flow_oracle as fo
import label_oracle
import occlusion_oracle as oo
import oracle as orc
from test_flow_oracle import W, H, fisheye, pose_pairs, scene

# Bars, from what the checks measure here at 160 x 120 (DESIGN.md section 5 item 14 lists the numbers).
# Flat world, share of in-frame pixels called occluded: pinhole 3.0e-3, fisheye 1.5e-2 (the fisheye's nearest-neighbour
# gather puts q a pixel off near label edges, as tests/test_flow_oracle.py measures).  The duckie checks set tau: at
# tau = 0.01 / 0.02 / 0.03 / 0.05 the turned duckie's newly seen side is occluded for 0.931 / 0.881 / 0.847 / 0.797 of its
# pinhole pixels (fisheye 0.941 / 0.896 / 0.861 / 0.802), and an unturned duckie seen from a moving camera is visible for
# 0.946 / 0.978 / 0.987 / 0.993 (fisheye 0.902 / 0.963 / 0.978 / 0.987).  0.02 misclassifies the least of both together.
FLAT_OCCLUDED_BAR = {False: 5e-3, True: 0.02}
TURN_OCCLUDED_BAR = 0.86      # turned duckie: share of its newly seen side called occluded
STILL_VISIBLE_BAR = 0.95      # a duckie that did not turn, seen from a moving camera: share called visible


@pytest.fixture(scope="module", autouse=True)
def built():
    orc.build()


def render(sc, p, fish, ep=None):
    """depth, labels, V, P of camera p = (x, z, angle)"""
    m = fisheye() if fish else None
    lut = (m.rmapx, m.rmapy) if fish else None
    _, dep, lab = label_oracle.render_batch(sc, [p[0]], [p[1]], [p[2]], [ep] if ep is not None else None, W=W, H=H,
                                            lut=lut)
    dbg = label_oracle.debug_frame(sc, p[0], p[1], p[2], W=W, H=H)
    return dep[0], lab[0], dbg["V"], dbg["P"]


def flow_of(md, cur, prev_V, fish, moves=None):
    dep, lab, V, P = cur
    m = fisheye() if fish else None
    src = fo.src_of_lut(m.rmapx, m.rmapy) if fish else None
    fwd = (m.mapx, m.mapy) if fish else None
    return fo.flow(dep, lab, P, prev_V, V, md.grid_w * md.grid_h, len(md.objects), moves, src=src, fwd=fwd)


def near(mask, r=1):
    """pixels within r (Chebyshev) of a pixel of mask"""
    out = mask.copy()
    pad = np.pad(mask, r)
    h, w = mask.shape
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            out |= pad[r + dy:r + dy + h, r + dx:r + dx + w]
    return out


def hidden_episode(o):
    words = [0] * 8
    words[o // 32] |= 1 << (o % 32)
    return orc.default_episode(hidden=words)


def road(lab, n_tiles):
    return (lab >= 1) & (lab <= 1 + n_tiles)


@pytest.mark.parametrize("fish", [False, True])
def test_still_camera_and_a_moved_obstacle(fish):
    """loop_obstacles' object 0 moved 4 cm and turned 12 degrees in front of a still camera 0.35 m away"""
    md, sc = scene("loop_obstacles")
    ob = md.objects[0]
    x, y, z = (float(v) for v in ob.pos)
    deg = float(np.rad2deg(ob.angle))
    states = [((x, y, z), deg), ((x + 0.03, y, z - 0.025), deg + 12.0)]
    moves = {0: tuple((np.float32(s[0][0]), np.float32(s[0][2]), np.float32(s[1])) for s in states)}
    n_tiles, obj = md.grid_w * md.grid_h, 2 + md.grid_w * md.grid_h
    occ_n = vis_n = 0
    try:
        for a in np.linspace(-np.pi, np.pi, 8, endpoint=False):
            p = (x - 0.35 * np.cos(a), z + 0.35 * np.sin(a), a)
            sc.set_object_pose(0, *states[0])
            prev = render(sc, p, fish)
            sc.set_object_pose(0, *states[1])
            cur = render(sc, p, fish)
            r = oo.occlusion(flow_of(md, cur, prev[2], fish, moves), cur[1], n_tiles, prev[0], prev[1])
            was, now = prev[1] == obj, cur[1] == obj
            uncovered = was & road(cur[1], n_tiles) & ~near(~was) & (r["mask"] != oo.NONE)
            far = road(cur[1], n_tiles) & ~near(was | now) & (r["mask"] != oo.NONE)
            assert (r["mask"][uncovered] == oo.OCCLUDED).all()
            assert (r["mask"][far] == oo.VISIBLE).all()
            occ_n, vis_n = occ_n + int(uncovered.sum()), vis_n + int(far.sum())
    finally:
        sc.set_object_pose(0, (x, y, z), deg)
    assert occ_n > 100 and vis_n > 20000, (occ_n, vis_n)


@pytest.mark.parametrize("fish", [False, True])
def test_flat_world_has_nothing_occluded(fish):
    md, sc = scene("small_loop")
    assert not md.objects
    (px0, pz0, a0), (px1, pz1, a1) = pose_pairs(md, 10, 31)
    occluded = total = 0
    for k in range(len(px0)):
        prev = render(sc, (px0[k], pz0[k], a0[k]), fish)
        cur = render(sc, (px1[k], pz1[k], a1[k]), fish)
        r = oo.occlusion(flow_of(md, cur, prev[2], fish), cur[1], md.grid_w * md.grid_h, prev[0], prev[1])
        m = r["mask"]
        occluded += int((m == oo.OCCLUDED).sum())
        total += int(((m == oo.OCCLUDED) | (m == oo.VISIBLE)).sum())
    print(f"flat world, fisheye {fish}: occluded {occluded} of {total} = {occluded / total:.2e}")
    assert total > 50000
    assert occluded <= FLAT_OCCLUDED_BAR[fish] * total


@pytest.mark.parametrize("fish", [False, True])
def test_hiding_a_static_obstacle(fish):
    """loop_obstacles, a camera 0.3 m from object o stepping sideways and turning: the previous frame rendered again
    without o.  A road pixel whose candidates show only o there, and only its own road without o, is occluded; where o is
    in no candidate of either render, the masks against the two renders agree."""
    md, sc = scene("loop_obstacles")
    n_tiles = md.grid_w * md.grid_h
    must = agree = 0
    for o in range(4):
        x, _, z = (float(v) for v in md.objects[o].pos)
        obj = 2 + n_tiles + o
        for a in np.linspace(-np.pi, np.pi, 6, endpoint=False):
            p0 = (x - 0.3 * np.cos(a), z + 0.3 * np.sin(a), a)
            p1 = (p0[0] + 0.03 * np.sin(a), p0[1] + 0.03 * np.cos(a), a - 0.05)   # 3 cm to the side, turned
            prev = render(sc, p0, fish)
            bare = render(sc, p0, fish, hidden_episode(o))
            cur = render(sc, p1, fish)
            fl = flow_of(md, cur, prev[2], fish)
            r = oo.occlusion(fl, cur[1], n_tiles, prev[0], prev[1])
            rb = oo.occlusion(fl, cur[1], n_tiles, bare[0], bare[1])
            h, w = cur[1].shape
            py, px = np.mgrid[0:h, 0:w]
            ok = (r["mask"] == oo.VISIBLE) | (r["mask"] == oo.OCCLUDED)
            qx = np.where(ok, px + np.nan_to_num(fl["flow"][..., 0]), 0)   # q - 0.5
            qy = np.where(ok, py + np.nan_to_num(fl["flow"][..., 1]), 0)
            cx, cy = np.floor(qx).astype(int), np.floor(qy).astype(int)
            all_o, all_road, any_o = ok.copy(), ok.copy(), np.zeros_like(ok)
            for j in (0, 1):
                for i in (0, 1):
                    inb = (cx + i >= 0) & (cx + i < w) & (cy + j >= 0) & (cy + j < h)
                    sx, sy = np.clip(cx + i, 0, w - 1), np.clip(cy + j, 0, h - 1)
                    all_o &= ~inb | (prev[1][sy, sx] == obj)
                    all_road &= ~inb | (bare[1][sy, sx] == cur[1])
                    any_o |= inb & ((prev[1][sy, sx] == obj) | (bare[1][sy, sx] == obj))
            hid = all_o & all_road & road(cur[1], n_tiles)
            assert (r["mask"][hid] == oo.OCCLUDED).all()
            assert (rb["mask"][hid] == oo.VISIBLE).all()
            clear = ok & ~any_o
            assert np.array_equal(r["mask"][clear], rb["mask"][clear])
            must, agree = must + int(hid.sum()), agree + int(clear.sum())
    print(f"hidden obstacle, fisheye {fish}: {must} road pixels only the obstacle hid, {agree} clear")
    assert must > 200 and agree > 50000


def duckie_frames(md, sc, turn, cam_move, fish, tau=oo.TAU):
    """loop_obstacles' duckie 0 turned by `turn` degrees in place, seen from 0.2 m by a camera that moves `cam_move`
    (dx, dz, dangle).  Returns (mask, newly seen) over the duckie's pixels: newly seen where the point's previous
    position is more than 5 mm farther from the camera, horizontally, than the duckie's axis."""
    ob = md.objects[0]
    x, y, z = (float(v) for v in ob.pos)
    deg = float(np.rad2deg(ob.angle))
    n_tiles = md.grid_w * md.grid_h
    obj = 2 + n_tiles
    masks, newly = [], []
    try:
        for a in np.linspace(-np.pi, np.pi, 8, endpoint=False):
            p0 = (x - 0.2 * np.cos(a), z + 0.2 * np.sin(a), a)
            p1 = (p0[0] + cam_move[0], p0[1] + cam_move[1], a + cam_move[2])
            sc.set_object_pose(0, (x, y, z), deg)
            prev = render(sc, p0, fish)
            sc.set_object_pose(0, (x, y, z), deg + turn)
            cur = render(sc, p1, fish)
            moves = {0: ((np.float32(x), np.float32(z), np.float32(deg)), (np.float32(x), np.float32(z),
                                                                           np.float32(deg + turn)))}
            fl = flow_of(md, cur, prev[2], fish, moves)
            r = oo.occlusion(fl, cur[1], n_tiles, prev[0], prev[1], tau=tau)
            # the point's previous world position, from its previous eye position
            d, P = cur[0].astype(np.float64), cur[3]
            sel = (cur[1] == obj) & ~np.isnan(fl["z_prev"])
            if fish:
                m = fisheye()
                sx, sy = fo.src_of_lut(m.rmapx, m.rmapy)
            else:
                sy, sx = np.mgrid[0:H, 0:W]
            E = np.stack([(2 * (sx + 0.5) / W - 1) * d / float(P[0]), (1 - 2 * (sy + 0.5) / H) * d / float(P[1]), -d,
                          np.ones_like(d)], -1)[sel]
            Xw = E @ np.linalg.inv(fo.rigid(cur[2])).T @ fo.mesh_motion(*moves[0]).T
            dist = np.hypot(Xw[:, 0] - p0[0], Xw[:, 2] - p0[1])
            masks.append(r["mask"][sel])
            newly.append(dist > np.hypot(x - p0[0], z - p0[1]) + 0.005)
    finally:
        sc.set_object_pose(0, (x, y, z), deg)
    return np.concatenate(masks), np.concatenate(newly)


@pytest.mark.parametrize("fish", [False, True])
def test_duckie_turned_in_place_hides_its_new_side(fish):
    md, sc = scene("loop_obstacles")
    m, newly = duckie_frames(md, sc, 180.0, (0.0, 0.0, 0.0), fish)
    sel = newly & ((m == oo.VISIBLE) | (m == oo.OCCLUDED))
    share = (m[sel] == oo.OCCLUDED).mean()
    print(f"turned duckie, fisheye {fish}: {sel.sum()} newly seen pixels, occluded {share:.4f}")
    assert sel.sum() > 300
    assert share >= TURN_OCCLUDED_BAR


@pytest.mark.parametrize("fish", [False, True])
def test_duckie_that_did_not_turn_stays_visible(fish):
    md, sc = scene("loop_obstacles")
    m, _ = duckie_frames(md, sc, 0.0, (0.01, 0.005, 0.03), fish)
    sel = (m == oo.VISIBLE) | (m == oo.OCCLUDED)
    share = (m[sel] == oo.VISIBLE).mean()
    print(f"unturned duckie, fisheye {fish}: {sel.sum()} pixels, visible {share:.4f}")
    assert sel.sum() > 1000
    assert share >= STILL_VISIBLE_BAR
