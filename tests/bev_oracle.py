"""A float64 numpy restatement of the bird's-eye map (dts_set_bev_target, DESIGN.md section 5 item 12): test
infrastructure, written from the spec and the reference rather than from the kernel.

A cell's centre is placed on the ground with the agent's get_dir_vec (cos a, -sin a) and get_right_vec (sin a, cos a)
(simulator.py:2056-2073); its tile is get_grid_coords (S:1134); its texel comes from inverting the tile's model transform
T((i + .5) ts, 0, (j + .5) ts) Ry(angle * 90 + 180) (S:1870-1873) and _init_vlists' vertex / uv rule (S:394-401); its
object is the smallest index whose footprint, generate_corners (collision.py:64-79), holds it.  The textures and their
texel classes are the scene's, from the product's blob builder, as the marking oracle takes them.

The device's cos / sin may differ from libm's by an ulp, so a cell is ambiguous when moving its centre by 1e-9 m in x
or z changes its answer: such a cell may take any of those answers (`check`)."""
import math

import numpy as np

EPS = 1e-9   # metres: the perturbation that marks a cell ambiguous
_PERTURB = ((EPS, 0.0), (-EPS, 0.0), (0.0, EPS), (0.0, -EPS))


class BevScene:
    """What the map says about every point of the ground: tiles, their textures and texel classes, and footprints."""

    def __init__(self, md):
        from gym_duckietown_b200 import lib as L
        holder = L.MapBlobHolder(md)
        self.md = md
        self.ts = float(md.tile_size)
        self.gw, self.gh = md.grid_w, md.grid_h
        self.n_cells = md.grid_w * md.grid_h
        self.kind = np.asarray(md.tile_kind, np.int64)
        self.angle = np.asarray(md.tile_angle, np.int64)
        self.tile_tex = np.asarray(holder.keep["tex"], np.int64)
        self.classes = [np.asarray(c, np.uint8) for c in holder.keep["tex_cls"]]
        self.corners = [np.asarray(o.corners, np.float64) for o in md.objects]
        self.slot_of = {d.object_index: s for s, d in enumerate(md.dyn_objects)}

    def footprints(self, dyn_corners=None, hidden=None):
        """[(object index, corners [4, 2])] in index order: hidden objects left out, objects with a dynamic slot at
        dyn_corners[slot] (default: where the map puts them)."""
        out = []
        for o, c in enumerate(self.corners):
            if hidden is not None and (int(hidden[o >> 5]) >> (o & 31)) & 1:
                continue
            s = self.slot_of.get(o)
            out.append((o, np.asarray(dyn_corners[s], np.float64) if s is not None and dyn_corners is not None else c))
        return out


def holds(c, x, z):
    """The four cross products (c[k+1] - c[k]) x (p - c[k]) all >= 0 or all <= 0"""
    pos = np.ones(np.shape(x), bool)
    neg = np.ones(np.shape(x), bool)
    for k in range(4):
        ax, az = c[k]
        bx, bz = c[(k + 1) % 4]
        cr = (bx - ax) * (z - az) - (bz - az) * (x - ax)
        pos &= cr >= 0
        neg &= cr <= 0
    return pos | neg


def classify_points(sc: BevScene, x, z, feet):
    """(labels int64, markings int64) of the ground points (x, z), with footprints `feet` (BevScene.footprints)."""
    x, z = np.asarray(x, np.float64), np.asarray(z, np.float64)
    ts = sc.ts
    label = np.ones(x.shape, np.int64)
    mark = np.zeros(x.shape, np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        fi, fj = np.floor(x / ts), np.floor(z / ts)
    inside = (fi >= 0) & (fi < sc.gw) & (fj >= 0) & (fj < sc.gh)
    i, j = np.where(inside, fi, 0).astype(np.int64), np.where(inside, fj, 0).astype(np.int64)
    idx = j * sc.gw + i
    on = inside & (sc.kind[idx] >= 0)
    label[on] = 2 + i[on] * sc.gh + j[on]
    tex = np.where(on, sc.tile_tex[idx], -1)
    for t in np.unique(tex[tex >= 0]):
        sel = tex == t
        ii, jj = i[sel], j[sel]
        lx, lz = x[sel] - (ii + 0.5) * ts, z[sel] - (jj + 0.5) * ts
        # Ry(theta) maps local (a, b) to (cos a + sin b, -sin a + cos b); its transpose undoes it.  theta is a multiple
        # of 90 degrees, so cos and sin are exactly 0 or +-1.
        q = (sc.angle[idx[sel]] + 2) % 4
        cs, sn = np.array([1.0, 0.0, -1.0, 0.0])[q], np.array([0.0, 1.0, 0.0, -1.0])[q]
        ax, az = cs * lx - sn * lz, sn * lx + cs * lz
        pu, pv = (ax + ts / 2) / ts, (az + ts / 2) / ts
        u, v = pu, 1 - pv
        plane = sc.classes[t]
        th, tw = plane.shape
        tu, tv = np.floor(u * tw).astype(np.int64) % tw, np.floor(v * th).astype(np.int64) % th
        mark[sel] = plane[tv, tu]
    done = np.zeros(x.shape, bool)
    for o, c in feet:
        hit = holds(c, x, z) & ~done
        label[hit] = 2 + sc.n_cells + o
        done |= hit
    return label, mark


def classify(sc: BevScene, x, z, env_corners=None, hidden=None):
    """(label, marking) of ground point(s) (x, z) for an env whose dynamic obstacles have corners env_corners
    [n_dyn][4][2] (None: their load-time ones) and whose hidden-object mask is `hidden` (u32 [8], or None)."""
    return classify_points(sc, x, z, sc.footprints(env_corners, hidden))


def cell_centres(px, pz, angle, width, height, cell, origin_x, origin_y):
    """Centres (x, z) [height, width] of the grid's cells, in the spec's order of float64 operations."""
    ca, sa = math.cos(angle), math.sin(angle)
    r = np.arange(height, dtype=np.float64)[:, None]
    c = np.arange(width, dtype=np.float64)[None, :]
    f = (origin_y - (r + 0.5)) * cell
    l = ((c + 0.5) - origin_x) * cell
    x = px + f * ca + l * sa
    z = pz - f * sa + l * ca
    return x, z


def bev_grid(sc: BevScene, px, pz, angle, cfg, env_corners=None, hidden=None):
    """One env's grid: (labels, markings, ambiguous, alternatives) — int64 [H, W] each, a bool [H, W], and the labels /
    markings [4, H, W] at the four perturbed centres.  cfg = (width, height, cell, origin_x, origin_y)."""
    width, height, cell, ox, oy = cfg
    x, z = cell_centres(px, pz, angle, width, height, cell, ox, oy)
    feet = sc.footprints(env_corners, hidden)
    lab, mk = classify_points(sc, x, z, feet)
    alt_l, alt_m = [], []
    for dx, dz in _PERTURB:
        a, b = classify_points(sc, x + dx, z + dz, feet)
        alt_l.append(a)
        alt_m.append(b)
    alt_l, alt_m = np.stack(alt_l), np.stack(alt_m)
    amb = ((alt_l != lab) | (alt_m != mk)).any(0)
    return lab, mk, amb, (alt_l, alt_m)


def bev_batch(scenes, map_id, px, pz, angle, cfg, dyn_corners=None, hidden=None):
    """Every env's grid: scenes[map_id[e]] at pose e; dyn_corners[e]: env e's [n_dyn][4][2] of its map (or None);
    hidden[e]: its u32 [8] mask (or None).  Returns lists of bev_grid's four results."""
    out = []
    for e in range(len(px)):
        sc = scenes[int(map_id[e])]
        out.append(bev_grid(sc, float(px[e]), float(pz[e]), float(angle[e]), cfg,
                            None if dyn_corners is None else dyn_corners[e], None if hidden is None else hidden[e]))
    return out


def check(got_labels, got_marks, expected, what=""):
    """The bar: every cell that is not ambiguous equal bit for bit; every ambiguous cell equal to its centre's answer or
    one of its perturbed answers; ambiguous cells under 1e-4 of all cells.  got_*: [N, H, W] arrays; expected: bev_batch's
    list."""
    n_amb = n_all = 0
    for e, (lab, mk, amb, (alt_l, alt_m)) in enumerate(expected):
        gl, gm = np.asarray(got_labels[e]).astype(np.int64), np.asarray(got_marks[e]).astype(np.int64)
        bad = ~amb & ((gl != lab) | (gm != mk))
        if bad.any():
            r, c = np.argwhere(bad)[0]
            raise AssertionError(f"{what} env {e}: {int(bad.sum())} unambiguous cells differ, first ({r}, {c}): got "
                                 f"label {gl[r, c]} marking {gm[r, c]}, want {lab[r, c]} {mk[r, c]}")
        ok = ((gl == lab) & (gm == mk)) | ((alt_l == gl) & (alt_m == gm)).any(0)
        if (amb & ~ok).any():
            r, c = np.argwhere(amb & ~ok)[0]
            raise AssertionError(f"{what} env {e}: ambiguous cell ({r}, {c}) is none of its answers")
        n_amb += int(amb.sum())
        n_all += amb.size
    assert n_amb < 1e-4 * n_all or n_amb == 0, f"{what}: {n_amb} of {n_all} cells are ambiguous"
    return n_amb
