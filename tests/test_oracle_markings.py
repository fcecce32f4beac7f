"""The marking oracle (tests/marking_oracle.py, render spec item 11) on the CPU: its frames, depth and labels are the
label oracle's, its markings are non-zero exactly where the label is a textured cell, they do not change with segment or
domain randomisation, and in a view from above a pixel whose centre falls well inside a painted line shows its paint."""
import numpy as np
import pytest

import label_oracle
import marking_oracle
import oracle as orc
from gym_duckietown_b200 import assets


@pytest.fixture(scope="module", autouse=True)
def built():
    orc.build()


def scene(name):
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    return md, orc.OracleScene(md)


def drivable_poses(md, n, seed):
    rng = np.random.default_rng(seed)
    tiles = [md.drivable_tiles[k] for k in rng.integers(0, len(md.drivable_tiles), n)]
    ts = md.tile_size
    px = np.array([(i + rng.uniform(0.1, 0.9)) * ts for i, _ in tiles])
    pz = np.array([(j + rng.uniform(0.1, 0.9)) * ts for _, j in tiles])
    return px, pz, rng.uniform(-np.pi, np.pi, n)


def textured_cell(md, lab):
    """label image -> where it is a grid cell whose tile has a texture (every present tile kind has one)"""
    n_cells = md.grid_w * md.grid_h
    cell = lab.astype(np.int64) - 2
    ok = (cell >= 0) & (cell < n_cells)
    i, j = np.where(ok, cell // md.grid_h, 0), np.where(ok, cell % md.grid_h, 0)
    kind = np.asarray(md.tile_kind)[j * md.grid_w + i]
    return ok & (kind >= 0)


@pytest.mark.parametrize("name,tile_mode,mode", [
    ("small_loop", 1, {}), ("udem1", 1, {}), ("loop_obstacles", 0, {}), ("udem1", 0, {"segment": True}),
    ("udem1", 1, {"segment": True}), ("loop_obstacles", 1, {"top_down": True}), ("small_loop", 0, {"top_down": True}),
])
def test_frames_depth_labels_are_the_label_oracles(name, tile_mode, mode):
    md, sc = scene(name)
    px, pz, ang = drivable_poses(md, 12, 3)
    W, H = 96, 72
    rgb, dep, lab, mk = marking_oracle.render_batch(sc, px, pz, ang, W=W, H=H, tile_mode=tile_mode, **mode)
    rgb_l, dep_l, lab_l = label_oracle.render_batch(sc, px, pz, ang, W=W, H=H, tile_mode=tile_mode, **mode)
    assert np.array_equal(rgb, rgb_l)
    assert np.array_equal(dep.view(np.int32), dep_l.view(np.int32))
    assert np.array_equal(lab, lab_l)
    assert mk.max() <= assets.MARK_RED
    assert np.array_equal(mk != 0, textured_cell(md, lab))
    assert (mk == assets.MARK_TILE).any() and (mk >= assets.MARK_WHITE).any()


def test_segment_and_domain_randomisation_leave_markings_unchanged():
    md, sc = scene("udem1")
    px, pz, ang = drivable_poses(md, 8, 5)
    for tile_mode in (0, 1):
        _, _, _, mk = marking_oracle.render_batch(sc, px, pz, ang, tile_mode=tile_mode)
        _, _, _, seg = marking_oracle.render_batch(sc, px, pz, ang, segment=True, tile_mode=tile_mode)
        assert np.array_equal(mk, seg)
        eps = [orc.default_episode() for _ in range(8)]
        for k, ep in enumerate(eps):     # other light, colours and horizon: the same visibility and texels
            ep.horizon[0], ep.ground[1] = 0.1 * k, 0.05 * k
            ep.light_eye[0] = 0.2 + 0.1 * k
            ep.ambient[1] = 0.05 * k
        _, _, _, dr = marking_oracle.render_batch(sc, px, pz, ang, eps, tile_mode=tile_mode)
        assert np.array_equal(mk, dr)


def test_top_down_pixels_inside_paint_show_it():
    """small_loop from above: a pixel whose centre, mapped back through the camera to the ground plane and into its
    tile's texture, falls well inside the stand-in's yellow dash or white line (its 8 neighbours painted alike, so the
    filter's erosion keeps it, and the centre away from a texel edge) carries 3 / 2."""
    md, sc = scene("small_loop")
    W, H = 640, 480
    _, _, lab, mk = marking_oracle.render(sc, 0.5, 0.5, 0.3, W=W, H=H, top_down=True)
    dbg = label_oracle.debug_frame(sc, 0.5, 0.5, 0.3, W=W, H=H, top_down=True)
    V, P = dbg["V"].reshape(3, 4), dbg["P"]
    R, t = V[:, :3], V[:, 3]
    n_cells = md.grid_w * md.grid_h
    checked = {assets.MARK_YELLOW: 0, assets.MARK_WHITE: 0}
    ts = md.tile_size
    for r in range(H):
        for c in range(W):
            v = int(lab[r, c]) - 2
            if not 0 <= v < n_cells:
                continue
            i, j = v // md.grid_h, v % md.grid_h
            kind = md.tile_kind[j * md.grid_w + i]
            # the ray through the pixel centre, met with the plane y = 0
            nx, ny = (c + 0.5) / W * 2 - 1, 1 - (r + 0.5) / H * 2
            d_eye = np.array([nx / P[0], ny / P[1], -1.0])
            o_w, d_w = -R.T @ t, R.T @ d_eye
            p = o_w + d_w * (-o_w[1] / d_w[1])
            # tile-local coordinates (the tile is drawn with Ry(angle * 90 + 180)) and the texture's u, v
            lx, lz = p[0] - (i + 0.5) * ts, p[2] - (j + 0.5) * ts
            q = (int(md.tile_angle[j * md.grid_w + i]) + 2) & 3
            cs, sn = [1, 0, -1, 0][q], [0, 1, 0, -1][q]
            ax, az = cs * lx - sn * lz, sn * lx + cs * lz
            u, vv = ax / ts + 0.5, 0.5 - az / ts
            tex = assets.tile_texture(assets_kind(kind))
            n = tex.shape[0]
            tu, tv = u * n, vv * n
            if min(tu % 1, 1 - tu % 1, tv % 1, 1 - tv % 1) < 0.2:
                continue   # near a texel edge: rounding may pick the neighbour
            col = tex[int(tv) % n, int(tu) % n, :3].astype(int)
            for want, rgb in ((assets.MARK_YELLOW, (235, 200, 30)), (assets.MARK_WHITE, (235, 235, 235))):
                block = tex[np.arange(int(tv) - 1, int(tv) + 2) % n][:, np.arange(int(tu) - 1, int(tu) + 2) % n, :3]
                if (col == rgb).all() and (block == rgb).all():
                    assert mk[r, c] == want, (r, c, i, j, u, vv)
                    checked[want] += 1
    assert checked[assets.MARK_YELLOW] > 10 and checked[assets.MARK_WHITE] > 10, checked


def assets_kind(kind_id):
    from gym_duckietown_b200.maps import TILE_KINDS
    return TILE_KINDS[int(kind_id)]
