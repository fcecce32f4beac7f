"""A float64 numpy restatement of the object boxes (dts_set_object_target, DESIGN.md section 5 item 17): test
infrastructure, written from the spec rather than from the kernel.

For one env: every object's footprint (its map's corners, or the env's copy for an object with a dynamic slot), its
mesh's object-space y extent, the env's pose and hidden-object mask give the box in the agent's frame and its state;
the frame's camera (and under the fisheye the env's forward map) gives where the box's corners land, through the bird's-
eye visibility oracle's projection.  Also the pixel statistics of a label image (object_boxes(), dts_object_pixels)."""
import numpy as np

import bev_view_oracle as vo

NONE, SHOWN, HIDDEN = range(3)


def mesh_extent_y(md, o):
    """(min_y, max_y) of object o's mesh over its vertices, as uploaded: ObjMesh.min_coords[1] / max_coords[1]"""
    v = np.asarray(md.meshes[md.objects[o].mesh_id].tri_pos, np.float32)[..., 1]
    return float(v.min()), float(v.max())


def heading_first(c, angle):
    """A Duckiebot's corners with c0 -> c1 along get_dir_vec(angle): as they are in generate_corners' order (the map's),
    from c1 in agent_boundbox's (back-left, back-right, front-right, front-left; what its turning step writes)"""
    f = np.array([np.cos(angle), -np.sin(angle)])
    return np.roll(c, -1, axis=0) if abs((c[2] - c[1]) @ f) > abs((c[1] - c[0]) @ f) else c


def world_boxes(md, dyn_corners=None, dyn_angles=None):
    """[(corners [4, 2] x-z, y0, y1)] of every object of the map: dyn_corners[slot] ([n_dyn][4][2]) for an object with a
    dynamic slot (default: where the map puts it), a Duckiebot's put in heading order by its dyn_angles[slot] (default:
    its angle at load)"""
    from gym_duckietown_b200.maps import DYN_DUCKIEBOT
    slot_of = {d.object_index: s for s, d in enumerate(md.dyn_objects)}
    out = []
    for o, ob in enumerate(md.objects):
        s = slot_of.get(o)
        c = np.asarray(dyn_corners[s] if s is not None and dyn_corners is not None else ob.corners, np.float64)
        if s is not None and md.dyn_objects[s].kind == DYN_DUCKIEBOT:
            c = heading_first(c, md.dyn_objects[s].angle if dyn_angles is None else dyn_angles[s])
        lo, hi = mesh_extent_y(md, o)
        scale, y = float(np.float32(ob.scale)), float(ob.pos[1])
        out.append((c, y + scale * lo, y + scale * hi))
    return out


def box_points(c, y0, y1):
    """The 8 corners (c0..c3 at y0, then at y1) and the centre, [9, 3]"""
    pts = [(c[k, 0], y0, c[k, 1]) for k in range(4)] + [(c[k, 0], y1, c[k, 1]) for k in range(4)]
    pts.append((c[:, 0].mean(), (y0 + y1) / 2, c[:, 1].mean()))
    return np.array(pts, np.float64)


def agent_box(c, y0, y1, px, pz, angle):
    """[7]: forward, right, up of the centre, length, width, height, yaw"""
    ca, sa = np.cos(angle), np.sin(angle)
    mx, mz = c[:, 0].mean(), c[:, 1].mean()
    dx, dz = mx - px, mz - pz
    e, w = c[1] - c[0], c[2] - c[1]
    yaw = np.arctan2(-(e[0] * sa + e[1] * ca), e[0] * ca - e[1] * sa)
    if yaw <= -np.pi:
        yaw = np.pi
    return np.array([dx * ca - dz * sa, dx * sa + dz * ca, (y0 + y1) / 2, np.hypot(*e), np.hypot(*w), y1 - y0, yaw])


def objects(md, pose, max_objects, dyn_corners=None, hidden=None, camera=None, dyn_angles=None):
    """One env.  pose: (pos_x, pos_z, angle); dyn_corners / dyn_angles: its obstacles' corners [n_dyn][4][2] and
    DTS_DYN_ANGLE [n_dyn] (None: the map's); hidden: its u32 [8] mask (or None); camera: None (no frame drawn) or
    (V f64 [12], P f32 [4], W, H, fwd) with fwd (Fx, Fy) of the env's fisheye table or None.

    Returns boxes f64 [O, 7] (NaN for NONE), state u8 [O], corners f64 [O, 9, 2] (NaN where the spec says) and
    ambiguous bool [O, 9]: a point at a near or far plane, or at the edge of F's footprint."""
    boxes = np.full((max_objects, 7), np.nan)
    state = np.zeros(max_objects, np.uint8)
    px = np.full((max_objects, 9, 2), np.nan)
    amb = np.zeros((max_objects, 9), bool)
    for o, (c, y0, y1) in enumerate(world_boxes(md, dyn_corners, dyn_angles)):
        hid = hidden is not None and (int(hidden[o >> 5]) >> (o & 31)) & 1
        state[o] = HIDDEN if hid else SHOWN
        boxes[o] = agent_box(c, y0, y1, *pose)
        if camera is not None:
            V, P, W, H, fwd = camera
            p = box_points(c, y0, y1)
            r = vo.project(V, P, W, H, p[:, 0], p[:, 1], p[:, 2], fwd)
            ok = r["front"] & r["foot"]
            px[o, :, 0] = np.where(ok, r["qx"], np.nan)
            px[o, :, 1] = np.where(ok, r["qy"], np.nan)
            amb[o] = r["ambiguous"]
    return boxes, state, px, amb


def pixel_stats(labels, n_cells, n_objects, max_objects):
    """One env's label image i16 [H, W] -> (pixels i32 [O], boxes i32 [O, 4]): object o = label - 2 - n_cells where
    0 <= o < n_objects; the count of its pixels and their inclusive x0, y0, x1, y1, -1 where the count is 0"""
    o = np.asarray(labels, np.int64) - 2 - n_cells
    hit = (o >= 0) & (o < n_objects)
    ys, xs = np.nonzero(hit)
    ob = o[hit]
    pixels = np.bincount(ob, minlength=max_objects)[:max_objects].astype(np.int32)
    boxes = np.full((max_objects, 4), -1, np.int32)
    for k in np.flatnonzero(pixels):
        m = ob == k
        boxes[k] = (xs[m].min(), ys[m].min(), xs[m].max(), ys[m].max())
    return pixels, boxes
