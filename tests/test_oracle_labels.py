"""The label oracle (tests/label_oracle.py, render spec item 10) on the CPU: its frames and depth are those of the
raster and depth oracles, and its labels are checked against geometry computed independently of the rasteriser — where
a grid cell's centre lands in a top-down view, which prop stands in front of a camera — and against the item numbering
of orr_debug_frame, which label_table must follow."""
import numpy as np
import pytest

import depth_oracle
import label_oracle
import oracle as orc


@pytest.fixture(scope="module", autouse=True)
def built():
    orc.build()


def scene(name):
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    return md, orc.OracleScene(md)


def drivable_poses(md, n, seed):
    """n cameras on drivable tiles, anywhere inside them, facing anywhere"""
    rng = np.random.default_rng(seed)
    tiles = [md.drivable_tiles[k] for k in rng.integers(0, len(md.drivable_tiles), n)]
    ts = md.tile_size
    px = np.array([(i + rng.uniform(0.1, 0.9)) * ts for i, _ in tiles])
    pz = np.array([(j + rng.uniform(0.1, 0.9)) * ts for _, j in tiles])
    return px, pz, rng.uniform(-np.pi, np.pi, n)


@pytest.mark.parametrize("name,tile_mode,mode", [
    ("small_loop", 1, {}), ("udem1", 1, {}), ("loop_obstacles", 0, {}), ("udem1", 1, {"segment": True}),
    ("loop_obstacles", 1, {"top_down": True}),
])
def test_frames_and_depth_are_the_other_oracles(name, tile_mode, mode):
    """Byte for byte the raster oracle's frames, bit for bit the depth oracle's depth; label 0 exactly where depth is 0."""
    md, sc = scene(name)
    px, pz, ang = drivable_poses(md, 12, 3)
    W, H = 96, 72
    rgb, dep, lab = label_oracle.render_batch(sc, px, pz, ang, W=W, H=H, tile_mode=tile_mode, **mode)
    rgb_d, dep_d = depth_oracle.render_batch(sc, px, pz, ang, W=W, H=H, tile_mode=tile_mode, **mode)
    assert np.array_equal(rgb, rgb_d)
    assert np.array_equal(dep.view(np.int32), dep_d.view(np.int32))
    if tile_mode == 1:   # (the raster oracle's own tile mode is the analytic one unless set)
        for k in range(3):
            assert np.array_equal(rgb[k], sc.render(px[k], pz[k], ang[k], None, W, H, **mode))
    assert np.array_equal(lab != 0, dep != 0)
    n_cells, n_obj = md.grid_w * md.grid_h, len(md.objects)
    assert lab.min() >= 0 and lab.max() <= 2 + n_cells + n_obj
    if not mode.get("top_down"):
        assert not (lab == 2 + n_cells + n_obj).any(), "the agent's own mesh is drawn in top-down views only"


def test_segment_and_domain_randomisation_leave_labels_unchanged():
    md, sc = scene("udem1")
    px, pz, ang = drivable_poses(md, 8, 5)
    _, _, lab = label_oracle.render_batch(sc, px, pz, ang)
    _, _, seg = label_oracle.render_batch(sc, px, pz, ang, segment=True)
    assert np.array_equal(lab, seg)
    eps = [orc.default_episode() for _ in range(8)]
    for k, ep in enumerate(eps):     # other light, colours and horizon: the same visibility
        ep.horizon[0], ep.ground[1] = 0.1 * k, 0.05 * k
        ep.light_eye[0] = 0.2 + 0.1 * k
    _, _, dr = label_oracle.render_batch(sc, px, pz, ang, eps)
    assert np.array_equal(lab, dr)


def project(dbg, W, H, x, z):
    """pixel (col, row) of the world point (x, 0, z) under the frame's camera V and projection P"""
    V, P = dbg["V"].reshape(3, 4), dbg["P"]
    ex, ey, ez = V @ np.array([x, 0.0, z, 1.0])
    nx, ny = P[0] * ex / -ez, P[1] * ey / -ez
    return int(np.floor((nx + 1) * 0.5 * W)), int(np.floor((1 - ny) * 0.5 * H))


@pytest.mark.parametrize("name", ["small_loop", "udem1", "loop_obstacles"])
def test_top_down_cell_centres_carry_their_cells_label(name):
    """In the view from above the map, the pixel a non-empty cell's centre projects to shows that cell — or an object
    (or the agent) standing on it."""
    md, sc = scene(name)
    W, H = 320, 240
    px, pz, ang = drivable_poses(md, 1, 7)
    _, _, lab = label_oracle.render(sc, px[0], pz[0], ang[0], W=W, H=H, top_down=True)
    dbg = label_oracle.debug_frame(sc, px[0], pz[0], ang[0], W=W, H=H, top_down=True)
    n_cells = md.grid_w * md.grid_h
    seen = covered = 0
    for i in range(md.grid_w):
        for j in range(md.grid_h):
            if md.tile_kind[j * md.grid_w + i] < 0:
                continue
            c, r = project(dbg, W, H, (i + 0.5) * md.tile_size, (j + 0.5) * md.tile_size)
            assert 0 <= c < W and 0 <= r < H, "the top-down view shows the whole map"
            v = int(lab[r, c])
            assert v == 2 + i * md.grid_h + j or v >= 2 + n_cells, f"cell ({i}, {j}) centre shows label {v}"
            seen += 1
            covered += v == 2 + i * md.grid_h + j
    assert covered >= seen * 0.8


def test_a_camera_facing_a_prop_sees_its_label_at_the_image_centre():
    """udem1: for every prop, a camera parked 0.3 .. 1 m in front of it and facing it, from eight directions, sees the
    prop's label at the image centre for some of those poses (the camera looks down, so the nearest poses see a low
    prop's base; a farther one can stand behind another prop)."""
    md, sc = scene("udem1")
    W, H = 160, 120
    n_cells = md.grid_w * md.grid_h
    for o, ob in enumerate(md.objects):
        P = [(ob.pos[0] - d * np.cos(a), ob.pos[2] + d * np.sin(a), a)
             for d in np.arange(0.3, 1.01, 0.1) for a in np.linspace(-np.pi, np.pi, 8, endpoint=False)]
        P = np.array(P)
        _, dep, lab = label_oracle.render_batch(sc, P[:, 0], P[:, 1], P[:, 2], W=W, H=H)
        hit = lab[:, H // 2, W // 2] == 2 + n_cells + o
        assert hit.any(), f"object {o} ({ob.kind}) is never seen at the image centre"
        assert (dep[hit, H // 2, W // 2] < 1.1).all()     # and it is near


@pytest.mark.parametrize("name", ["udem1", "loop_obstacles"])
def test_label_table_follows_the_oracles_item_numbering(name):
    """label_table()[1 + item] is orr_debug_frame's item: the ground, every cell (transform zero exactly where the cell is
    empty, else placed at the cell's centre), every object (placed at its position), and the agent last."""
    from gym_duckietown_b200.batched_env import label_table
    md, sc = scene(name)
    dbg = sc.debug_frame(0.5, 0.5, 0.3)
    table = label_table(md)
    n_cells = md.grid_w * md.grid_h
    assert len(table) == 1 + len(dbg["item_mv"]) + 1 and table[0] == ("none",) and table[-1] == ("agent",)
    assert table[1] == ("ground",)
    V = dbg["V"].reshape(3, 4)
    for item in range(1, len(dbg["item_mv"])):
        ent, mv = table[1 + item], dbg["item_mv"][item].reshape(3, 4)
        if item <= n_cells:
            _, i, j, kind = ent
            assert ent[0] == "tile" and (item - 1) == i * md.grid_h + j
            assert (kind is None) == (not mv.any())
            centre = np.array([(i + 0.5) * md.tile_size, 0.0, (j + 0.5) * md.tile_size])
        else:
            _, o, kind = ent
            assert ent[0] == "object" and o == item - 1 - n_cells and kind == md.objects[o].kind
            centre = np.asarray(md.objects[o].pos, np.float64)
        if mv.any():
            assert np.allclose(mv[:, 3], V[:, :3] @ centre + V[:, 3], atol=1e-4)
