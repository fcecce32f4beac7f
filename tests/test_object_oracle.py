"""The object boxes' oracle (tests/object_oracle.py, DESIGN.md section 5 item 17) without a GPU: its footprints are the
maps' own, its mesh extent is the reference ObjMesh's, its boxes hold every vertex the reference hands OpenGL for each
object (the gltrace goldens) and touch each of their six faces, the raster oracle's object pixels lie inside the
projected boxes, hand-built cases fix the signs of the agent frame and the yaw, and the ctypes signatures match the
header."""
import os
import re
import types

import numpy as np
import pytest

import bev_view_oracle as vo
import label_oracle
import object_oracle as oo
import oracle as orc
from gym_duckietown_b200 import maps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
W, H = 160, 120


def test_box_corners_are_the_maps_footprints():
    from gym_duckietown_b200 import lib as L
    for name in maps.list_maps():
        md = maps.load_map(name)
        blob = L.MapBlobHolder(md).keep.get("obj_corners")
        for o, (c, y0, y1) in enumerate(oo.world_boxes(md)):
            assert np.array_equal(c, md.objects[o].corners), (name, o)
            assert np.array_equal(c, np.asarray(blob[o]).reshape(4, 2)), (name, o)
            assert y1 > y0, (name, o)


def test_mesh_extent_is_the_reference_objmesh_extent(tmp_path):
    from gym_duckietown_b200 import assets
    from test_obj_loader import MTL, OBJ
    (tmp_path / "prop.obj").write_text(OBJ)
    (tmp_path / "prop.mtl").write_text(MTL)
    ref = np.load(os.path.join(GOLD, "objmesh_prop.npz"))
    mesh = assets.load_obj(str(tmp_path / "prop.obj"), "prop")
    md = types.SimpleNamespace(meshes=[mesh], objects=[types.SimpleNamespace(mesh_id=0)])
    assert oo.mesh_extent_y(md, 0) == (float(ref["min_coords"][1]), float(ref["max_coords"][1]))
    for name in maps.list_maps():   # and every shipped object's, as the library's ObjMesh keeps it
        md = maps.load_map(name)
        for o, ob in enumerate(md.objects):
            mesh = md.meshes[ob.mesh_id]
            assert oo.mesh_extent_y(md, o) == (float(mesh.min_coords[1]), float(mesh.max_coords[1]))


@pytest.mark.parametrize("name", ["loop_obstacles", "udem1"])
def test_boxes_hold_every_traced_vertex_and_touch_every_face(name):
    md = maps.load_map(name)
    g = np.load(os.path.join(GOLD, f"gltrace_{name}.npz"))
    boxes = oo.world_boxes(md)
    cells = [(i, j) for i in range(md.grid_w) for j in range(md.grid_h)]
    n_present = sum(md.tile_kind[j * md.grid_w + i] >= 0 for i, j in cells)
    checked = set()
    for f in np.flatnonzero(g["f_mode"] == 0):
        lo = int(g["f_draw0"][f])
        view = g["f_view"][f].reshape(4, 4)
        vis = [o for o in range(len(md.objects)) if g["f_visible"][f][o]]
        for k, o in enumerate(vis):
            model = np.linalg.solve(view, g["d_mv"][lo + 2 + n_present + k].reshape(4, 4))
            v = np.asarray(md.meshes[md.objects[o].mesh_id].tri_pos, np.float64).reshape(-1, 3)
            p = v @ model[:3, :3].T + model[:3, 3]
            c, y0, y1 = boxes[o]
            u, w = c[1] - c[0], c[3] - c[0]
            a = (p[:, [0, 2]] - c[0]) @ (u / np.linalg.norm(u))
            b = (p[:, [0, 2]] - c[0]) @ (w / np.linalg.norm(w))
            for got, lo_, hi_ in ((a, 0.0, np.linalg.norm(u)), (b, 0.0, np.linalg.norm(w)), (p[:, 1], y0, y1)):
                assert got.min() >= lo_ - 1e-6 and got.max() <= hi_ + 1e-6, (f, o, got.min(), got.max(), lo_, hi_)
                assert abs(got.min() - lo_) <= 1e-6 and abs(got.max() - hi_) <= 1e-6, (f, o, got.min(), lo_, got.max(), hi_)
            checked.add(o)
    assert len(checked) == len(md.objects) or len(checked) >= 4, checked


def hand_map(objects):
    return maps.interpret_map({"tile_size": 0.585, "tiles": [["straight/E"] * 4] * 3, "objects": list(objects)}, "hand")


@pytest.mark.parametrize("name,poses", [
    ("loop_obstacles", None), ("udem1", None),
    ("hand", [(0.3, 0.8775, 0.0), (0.35, 0.85, 0.2), (0.3, 0.9, -0.25)])])
def test_object_pixels_lie_inside_the_projected_boxes(name, poses):
    orc.build()
    if name == "hand":
        md = hand_map([{"kind": "duckie", "pos": [1.25, 1.5], "height": 0.06, "rotate": 30},
                       {"kind": "cone", "pos": [1.6, 1.2], "rotate": -70}])
        px, pz, ang = (np.array(v) for v in zip(*poses))
    else:
        md = maps.load_map(name)
        rng = np.random.default_rng(7)
        cells = np.array(md.drivable_tiles)[rng.integers(len(md.drivable_tiles), size=12)]
        px = (cells[:, 0] + rng.uniform(size=12)) * md.tile_size
        pz = (cells[:, 1] + rng.uniform(size=12)) * md.tile_size
        ang = rng.uniform(-np.pi, np.pi, size=12)
    sc = orc.OracleScene(md)
    _, _, lab = label_oracle.render_batch(sc, px, pz, ang, W=W, H=H)
    n_cells, n_obj = md.grid_w * md.grid_h, len(md.objects)
    checked = 0
    for e in range(len(px)):
        dbg = label_oracle.debug_frame(sc, px[e], pz[e], ang[e], W=W, H=H)
        _, _, q, _ = oo.objects(md, (px[e], pz[e], ang[e]), n_obj, camera=(dbg["V"], dbg["P"], W, H, None))
        o_img = lab[e].astype(np.int64) - 2 - n_cells
        for o in range(n_obj):
            ys, xs = np.nonzero(o_img == o)
            if not len(xs):
                continue
            c, y0, y1 = oo.world_boxes(md)[o]
            pts = oo.box_points(c, y0, y1)[:8]
            w = vo.project(dbg["V"], dbg["P"], W, H, pts[:, 0], pts[:, 1], pts[:, 2])["w"]
            if not (w > vo.NEAR).all():
                continue
            qx, qy = q[o, :8, 0], q[o, :8, 1]
            assert (xs + 0.5 >= qx.min() - 1).all() and (xs + 0.5 <= qx.max() + 1).all(), (name, e, o)
            assert (ys + 0.5 >= qy.min() - 1).all() and (ys + 0.5 <= qy.max() + 1).all(), (name, e, o)
            checked += 1
    assert checked >= 2, checked


@pytest.mark.parametrize("agent,place,rot,fwd,right,yaw", [
    (0.0, (1.0, 0.0), 0.0, 1.0, 0.0, 0.0),                      # straight ahead, same heading
    (0.0, (0.0, 0.5), 0.0, 0.0, 0.5, 0.0),                      # on the right: +z is right of heading +x
    (np.pi / 2, (0.0, -1.0), 0.0, 1.0, 0.0, -np.pi / 2),        # heading -z: ahead is -z; the object turned right of it
    (0.3, None, 0.3 + np.pi / 2, None, None, np.pi / 2),        # +90 degrees: counter-clockwise from above
    (0.3, None, 0.3 - np.pi / 2, None, None, -np.pi / 2),       # -90 degrees
    (0.3, None, 0.3 + np.pi, None, None, np.pi),                # 180 degrees: pi, not -pi
    (-np.pi, None, 0.0, None, None, np.pi)])
def test_hand_built_signs(agent, place, rot, fwd, right, yaw):
    pos = np.array([3.0, 0.0, 2.0]) if place is None else np.array([place[0], 0.0, place[1]])
    lo, hi = np.array([-0.1, 0.0, -0.05]), np.array([0.1, 0.2, 0.05])
    c = maps.obb_corners(pos, lo, hi, rot, 1.0)
    box = oo.agent_box(c, 0.0, 0.2, 0.0, 0.0, agent)
    if fwd is not None:
        assert abs(box[0] - fwd) < 1e-12 and abs(box[1] - right) < 1e-12, box
    assert abs(box[3] - 0.2) < 1e-12 and abs(box[4] - 0.1) < 1e-12 and abs(box[5] - 0.2) < 1e-12
    assert abs(box[6] - yaw) < 1e-12 and -np.pi < box[6] <= np.pi, box
    # the agent frame inverts the bird's-eye grid's: the centre maps back to the world
    ca, sa = np.cos(agent), np.sin(agent)
    f, r = box[0], box[1]
    assert np.allclose([f * ca + r * sa, -f * sa + r * ca], c.mean(0), atol=1e-12)


@pytest.mark.parametrize("angle", [0.0, 0.4, np.pi / 2, np.pi, -2.5])
def test_a_turned_duckiebot_keeps_its_heading(angle):
    """A Duckiebot's turning step writes its corners in agent_boundbox's order (back-left, back-right, front-right,
    front-left; as dts_logic.cuh does, collision.py:9-31): its box still runs along its heading, length robot_length"""
    from gym_duckietown_b200.maps import DYN_DUCKIEBOT
    md = maps.load_map("loop_dyn_duckiebots")
    s, d = next((s, d) for s, d in enumerate(md.dyn_objects) if d.kind == DYN_DUCKIEBOT)
    p = np.array([1.0, 2.0])
    f, r = np.array([np.cos(angle), -np.sin(angle)]), np.array([np.sin(angle), np.cos(angle)])
    hw, hl = d.robot_width / 2, d.robot_length / 2
    c = np.array([p - hw * r - hl * f, p + hw * r - hl * f, p + hw * r + hl * f, p - hw * r + hl * f])
    dyn = [o.corners for o in md.dyn_objects]
    dyn[s] = c
    angles = [o.angle for o in md.dyn_objects]
    angles[s] = angle
    for agent in (0.0, 1.1, -2.0):
        box = oo.objects(md, (0.0, 0.0, agent), len(md.objects), dyn, dyn_angles=angles)[0][d.object_index]
        want = (angle - agent + np.pi) % (2 * np.pi) - np.pi
        assert abs((box[6] - want + np.pi) % (2 * np.pi) - np.pi) < 1e-12, (box[6], want)
        assert abs(box[3] - d.robot_length) < 1e-12 and abs(box[4] - d.robot_width) < 1e-12
    # at load, in generate_corners' order, the same rule keeps c0 -> c1
    for o_s, o in enumerate(md.dyn_objects):
        box = oo.objects(md, (0.0, 0.0, 0.0), len(md.objects))[0][o.object_index]
        want = (o.angle + np.pi) % (2 * np.pi) - np.pi
        assert abs((box[6] - want + np.pi) % (2 * np.pi) - np.pi) < 1e-12, (o_s, box[6], o.angle)


def test_ctypes_signatures_match_the_header():
    import ctypes as C
    from gym_duckietown_b200 import lib as L
    with open(os.path.join(ROOT, "include", "dtsim.h")) as f:
        h = f.read()
    lib = L.load()
    kinds = {"int": C.c_int, "void*": C.c_void_p}
    for name in ("dts_set_object_target", "dts_render_objects", "dts_object_pixels"):
        args = re.search(r"int " + name + r"\(([^)]*)\);", h).group(1)
        want = [C.c_int if re.fullmatch(r"int \w+", a.strip()) else C.c_void_p for a in args.split(",")]
        assert all("*" in a or re.fullmatch(r"int \w+", a.strip()) for a in args.split(",")), args
        assert getattr(lib, name).argtypes == want, name
    assert (L.OBJECT_STATE_NAMES, oo.NONE, oo.SHOWN, oo.HIDDEN) == (("none", "shown", "hidden"), 0, 1, 2)
    for k, v in enumerate(L.OBJECT_STATE_NAMES):
        assert re.search(rf"DTS_OBJECT_{v.upper()} = {k}\b", h), v
