"""The depth image of the render spec (DESIGN.md section 5, item 9) as the CPU depth oracle computes it
(tests/depth_oracle.py: the raster oracle's source with the depth insertions), pinned to geometry the spec does not
define: on small_loop frames the depth of a pixel that lies well inside a road tile equals the
analytic distance — the camera ray through the pixel centre meets the plane y = 0, and the hit point's distance along
the view axis is the depth — with the camera taken from the frame's own V and P (orr_debug_frame).

How close: the spec snaps vertices to 1/64 px and builds the 1/w plane from the snapped positions, so the plane is that
of a tile whose corners moved by up to 1/128 px, extrapolated over the half of the quad its triangle does not cover.
1/w is linear in the image row and zero on the horizon, so a shift of e pixels is a relative depth error of e / (rows
below the horizon): the bar is 1/16 px of shift (0.032 px is the most seen over 40 poses), which is 1e-3 relative forty
rows below the horizon and 1e-2 at 10 m.  A wrong plane, a wrong vertex or the far / near planes' z in place of w would
miss it by orders of magnitude.  Sky pixels are 0, and the depth does not depend on the colours drawn."""
import numpy as np
import pytest

import depth_oracle

W, H = 160, 120


@pytest.fixture(scope="module")
def scene():
    import oracle as orc
    from gym_duckietown_b200 import maps
    orc.lib().orr_set_tile_mode(1)
    md = maps.load_map("small_loop")
    return orc, md, orc.OracleScene(md)


def poses(md, n, seed):
    rng = np.random.default_rng(seed)
    cells = np.array(md.drivable_tiles)[rng.integers(len(md.drivable_tiles), size=n)]
    return [((c[0] + rng.uniform(0.2, 0.8)) * md.tile_size, (c[1] + rng.uniform(0.2, 0.8)) * md.tile_size,
             rng.uniform(-np.pi, np.pi)) for c in cells]


def plane_hits(V, P):
    """Per pixel centre: eye-space depth of the ray's hit with the plane y = 0 (inf where the ray does not descend to
    it) and the hit's world (x, z)."""
    V = V.reshape(3, 4)
    R, t = V[:, :3], V[:, 3]
    cam = -R.T @ t
    xs, ys = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    ndx, ndy = 2.0 * xs / W - 1.0, 1.0 - 2.0 * ys / H
    d_eye = np.stack([ndx / float(P[0]), ndy / float(P[1]), -np.ones_like(ndx)], -1)   # depth 1 along the view axis
    d_world = d_eye @ R            # R^T applied to every direction
    with np.errstate(divide="ignore", invalid="ignore"):
        s = -cam[1] / d_world[..., 1]
    s = np.where((d_world[..., 1] < 0) & (s > 0), s, np.inf)
    with np.errstate(invalid="ignore"):
        hit = cam + s[..., None] * d_world
    return s, hit[..., 0], hit[..., 2]


def test_road_depth_is_the_ray_plane_distance_and_sky_is_zero(scene):
    orc, md, sc = scene
    ts = md.tile_size
    checked = 0
    for px, pz, ang in poses(md, 12, 7):
        rgb, depth = depth_oracle.render(sc, px, pz, ang, None, W, H)
        assert depth.dtype == np.float32 and depth.shape == (H, W)
        assert np.array_equal(rgb, sc.render(px, pz, ang, None, W, H)), "the depth oracle's frame is not the raster oracle's"
        f = sc.debug_frame(px, pz, ang, None, W, H)
        s, hx, hz = plane_hits(f["V"], f["P"])
        # pixels whose whole footprint lies in ONE road tile: the hit is 3 % of a tile away from the tile's border and
        # the neighbouring pixel centres fall in the same tile (so no sample sees another surface), nearer than the far
        # plane's tenth, and not behind an object (small_loop has none)
        with np.errstate(invalid="ignore"):
            ci, cj = np.floor(hx / ts), np.floor(hz / ts)
            fx, fz = hx / ts - ci, hz / ts - cj
        ok = np.isfinite(s) & (s < 10.0) & (fx > 0.03) & (fx < 0.97) & (fz > 0.03) & (fz < 0.97)
        ok &= (ci >= 0) & (ci < md.grid_w) & (cj >= 0) & (cj < md.grid_h)
        road = np.zeros_like(ok)
        idx = np.flatnonzero(ok)
        kinds = np.asarray(md.tile_kind).reshape(md.grid_h, md.grid_w)
        road.flat[idx] = kinds[cj.flat[idx].astype(int), ci.flat[idx].astype(int)] >= 0
        same = np.ones_like(ok)
        for dy, dx in ((0, 1), (1, 0), (0, -1), (-1, 0)):
            sh_i, sh_j = np.roll(ci, (dy, dx), (0, 1)), np.roll(cj, (dy, dx), (0, 1))
            same &= (sh_i == ci) & (sh_j == cj)
        same[0, :] = same[-1, :] = False
        same[:, 0] = same[:, -1] = False
        sel = ok & road & same
        assert sel.sum() > 500, "the pose shows too little road to check"
        with np.errstate(divide="ignore", invalid="ignore"):
            q = 1.0 / s
            rows = q / np.abs(np.gradient(q, axis=0))          # rows below the horizon: 1/w is linear in y and 0 there
            shift = (np.abs(depth - s) / s * rows)[sel]
        assert shift.max() < 1.0 / 16, f"pose {(px, pz, ang)}: depth is off the ray / plane distance by {shift.max():.3f} px"
        checked += int(sel.sum())
        # above the horizon nothing is drawn: the ray neither meets the road plane nor the ground quad 8 mm below it
        sky = ~np.isfinite(s)
        sky[1:, :] &= sky[:-1, :]          # ... and a row clear of the horizon line itself
        sky[:-1, :] &= sky[1:, :]
        sky[-1, :] = False
        assert sky.sum() > 1000
        assert (depth[sky] == 0.0).all(), "sky pixels carry a depth"
        assert (depth[~sky] >= 0.0).all() and np.isfinite(depth).all()
    assert checked > 20000


def test_depth_ignores_colours_and_follows_the_camera(scene):
    orc, md, sc = scene
    px, pz, ang = poses(md, 1, 3)[0]
    _, base = depth_oracle.render(sc, px, pz, ang, None, W, H)
    seg_rgb, seg = depth_oracle.render(sc, px, pz, ang, None, W, H, segment=True)
    assert np.array_equal(seg, base), "segment=True changed the depth"
    assert np.array_equal(seg_rgb, sc.render(px, pz, ang, None, W, H, segment=True))
    assert not np.array_equal(seg_rgb, sc.render(px, pz, ang, None, W, H))
    dark = orc.default_episode(ambient=(0.05, 0.05, 0.05), diffuse=(0.9, 0.2, 0.1), horizon=(0.1, 0.2, 0.3), ground=(0.4, 0.1, 0.2))
    _, d2 = depth_oracle.render(sc, px, pz, ang, dark, W, H)
    assert np.array_equal(d2, base), "light / sky / ground colours changed the depth"
    tall = orc.default_episode(cam_height=0.13, cam_angle_deg=15.0)
    _, d3 = depth_oracle.render(sc, px, pz, ang, tall, W, H, domain_rand=True)
    assert not np.array_equal(d3, base), "the camera's height and pitch did not change the depth"


def test_depth_goes_through_the_gather_like_the_frame(scene):
    """Under a LUT the depth of an output pixel is the plain depth at the source pixel, 0 where there is none."""
    orc, md, sc = scene
    px, pz, ang = poses(md, 1, 5)[0]
    _, plain = depth_oracle.render(sc, px, pz, ang, None, W, H)
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    rx, ry = (W - 1 - x) + 0.25, y + 3.0          # mirrored, shifted down: the last three rows have no source
    rx[5, 7] = np.nan
    rgb, got = depth_oracle.render(sc, px, pz, ang, None, W, H, lut=(rx, ry))
    assert np.array_equal(rgb, sc.render(px, pz, ang, None, W, H, lut=(rx, ry)))
    want = np.zeros_like(plain)
    want[:H - 3] = plain[3:, ::-1]
    want[5, 7] = 0.0
    assert np.array_equal(got, want)


def test_depth_oracle_frames_are_the_raster_oracles_in_both_tile_modes_and_views(scene):
    """The second build of the raster oracle draws what the first draws: a batch of frames in tile mode 1 and 0, and the
    top-down view."""
    orc, md, sc = scene
    P = np.array(poses(md, 6, 9))
    eps = [orc.default_episode() for _ in P]
    try:
        for tile_mode in (1, 0):
            orc.lib().orr_set_tile_mode(tile_mode)
            want = sc.render_batch(P[:, 0], P[:, 1], P[:, 2], eps, W, H, False, threads=2)
            got, dep = depth_oracle.render_batch(sc, P[:, 0], P[:, 1], P[:, 2], eps, W, H, tile_mode=tile_mode)
            assert np.array_equal(got, want), f"tile mode {tile_mode}"
            assert (dep > 0).mean() > 0.3
    finally:
        orc.lib().orr_set_tile_mode(1)
    top, dep = depth_oracle.render(sc, P[0, 0], P[0, 1], P[0, 2], None, W, H, top_down=True)
    assert np.array_equal(top, sc.render(P[0, 0], P[0, 1], P[0, 2], None, W, H, top_down=True))
    assert dep.min() > 1.0      # the camera hangs above the map: everything is far, nothing is sky
