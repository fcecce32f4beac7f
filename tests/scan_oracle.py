"""A float64 numpy restatement of the range scan (dts_set_scan_target, DESIGN.md section 5 item 16): test
infrastructure, written from the spec rather than from the kernel.

A ray leaves the origin (the bird's-eye grid's offset formulas) along get_dir_vec(a + phi_k).  It is blocked where a
strictly convex footprint of an object not hidden this episode holds the point (bev_oracle.holds), or where
_drivable_pos (S:1411-1428) is false.  Objects are met where the ray crosses one of the footprint's edge segments, or at
0 when the footprint holds the origin.  Tiles are met at every crossing of a grid line x = m ts or z = n ts, all of them
at once rather than cell by cell: the cell a crossing enters is the one across that line.

The device's cos / sin may differ from libm's by an ulp, so a ray is ambiguous when the runner-up candidate's t lies
within EPS of t*, when the ray passes within EPS of a footprint or tile corner before t*, or when the origin lies within
EPS of a footprint edge or a grid line.  An ambiguous ray may take any answer (`check`)."""
import math

import numpy as np

import bev_oracle as bo

EPS = 1e-6   # metres


def strictly_convex(c):
    """The four cross products (c[k+1] - c[k]) x (c[k+2] - c[k+1]) all > 0 or all < 0"""
    s = [(c[(k + 1) % 4][0] - c[k][0]) * (c[(k + 2) % 4][1] - c[k][1]) -
         (c[(k + 1) % 4][1] - c[k][1]) * (c[(k + 2) % 4][0] - c[k][0]) for k in range(4)]
    return all(v > 0 for v in s) or all(v < 0 for v in s)


def tile_drivable(sc: bo.BevScene, x, z):
    """_drivable_pos (S:1411-1428) of the points (x, z): on the grid, on a tile, and that tile drivable"""
    x, z = np.asarray(x, np.float64), np.asarray(z, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        fi, fj = np.floor(x / sc.ts), np.floor(z / sc.ts)
    inside = (fi >= 0) & (fi < sc.gw) & (fj >= 0) & (fj < sc.gh)
    idx = np.where(inside, fj, 0).astype(np.int64) * sc.gw + np.where(inside, fi, 0).astype(np.int64)
    drv = np.asarray(sc.md.tile_drivable, bool)
    return inside & (sc.kind[idx] >= 0) & drv[idx]


def blocked_label(sc, x, z, feet):
    """(blocked, label) of points: label is the bird's-eye label; blocked when it is an object or the point is not
    drivable.  feet: the footprints that block (strictly convex ones)."""
    lab, _ = bo.classify_points(sc, x, z, feet)
    return (lab >= 2 + sc.n_cells) | ~tile_drivable(sc, x, z), lab


def rays(px, pz, angle, cfg):
    """origin (ox, oz) and directions (dx, dz) [R] of cfg = (n_rays, fov, max_range, forward, right)"""
    R, fov, _, f, r = cfg
    ca, sa = math.cos(angle), math.sin(angle)
    ox, oz = px + f * ca + r * sa, pz - f * sa + r * ca
    k = np.arange(R, dtype=np.float64)
    phi = fov * (0.5 - (k + 0.5) / R)
    a = angle + phi
    return ox, oz, np.cos(a), -np.sin(a)


def _cross(ax, az, bx, bz):
    return ax * bz - az * bx


def _segment_t(ox, oz, dx, dz, c0, c1):
    """t >= 0 where each ray meets the segment c0 -> c1 (inf where it does not); parallel rays do not meet it"""
    ex, ez = c1[0] - c0[0], c1[1] - c0[1]
    den = _cross(dx, dz, ex, ez)
    wx, wz = c0[0] - ox, c0[1] - oz
    with np.errstate(divide="ignore", invalid="ignore"):
        t = _cross(wx, wz, ex, ez) / den
        u = _cross(wx, wz, dx, dz) / den
    ok = (den != 0) & (t >= 0) & (u >= 0) & (u <= 1)
    return np.where(ok, t, np.inf)


def scan(sc: bo.BevScene, px, pz, angle, cfg, env_corners=None, hidden=None):
    """One env's scan: (range float64 [R], hit int64 [R], ambiguous bool [R]), cfg = (n_rays, fov, max_range, forward,
    right); env_corners / hidden as bev_oracle.classify's."""
    R, _, max_range, _, _ = cfg
    ox, oz, dx, dz = rays(px, pz, angle, cfg)
    feet = [(o, c) for o, c in sc.footprints(env_corners, hidden) if strictly_convex(c)]
    n_cells, ts = sc.n_cells, sc.ts
    # candidates: (t [R], label [R]) per object, then the tiles
    cands = []
    for o, c in feet:
        t = np.full(R, np.inf)
        for k in range(4):
            t = np.minimum(t, _segment_t(ox, oz, dx, dz, c[k], c[(k + 1) % 4]))
        if bo.holds(c, np.float64(ox), np.float64(oz)):
            t[:] = 0.0
        cands.append((t, np.full(R, 2 + n_cells + o)))
    # tiles: every grid-line crossing enters the cell across the line
    tile_t = np.full(R, np.inf)
    tile_lab = np.ones(R, np.int64)
    org_blocked, org_label = blocked_label(sc, np.float64(ox), np.float64(oz), feet)
    if not tile_drivable(sc, ox, oz):
        tile_t[:] = 0.0
        fi, fj = math.floor(ox / ts), math.floor(oz / ts)
        on = 0 <= fi < sc.gw and 0 <= fj < sc.gh and sc.kind[fj * sc.gw + fi] >= 0
        tile_lab[:] = 2 + fi * sc.gh + fj if on else 1
    else:
        for axis, n_lines in ((0, sc.gw), (1, sc.gh)):
            lines = np.arange(n_lines + 1, dtype=np.float64)[None, :] * ts
            o_a, d_a = (ox, dx) if axis == 0 else (oz, dz)
            o_b, d_b = (oz, dz) if axis == 0 else (ox, dx)
            with np.errstate(divide="ignore", invalid="ignore"):
                t = (lines - o_a) / d_a[:, None]
            t = np.where((d_a[:, None] != 0) & (t >= 0), t, np.inf)
            m = np.arange(n_lines + 1)[None, :]
            a_cell = np.where(d_a[:, None] > 0, m, m - 1)
            with np.errstate(invalid="ignore"):
                b_cell = np.floor((o_b + np.where(np.isfinite(t), t, 0) * d_b[:, None]) / ts)
            i, j = (a_cell, b_cell) if axis == 0 else (b_cell, a_cell)
            inside = (i >= 0) & (i < sc.gw) & (j >= 0) & (j < sc.gh)
            idx = np.where(inside, j, 0).astype(np.int64) * sc.gw + np.where(inside, i, 0).astype(np.int64)
            road = inside & (sc.kind[idx] >= 0)
            drv = road & np.asarray(sc.md.tile_drivable, bool)[idx]
            t = np.where(drv, np.inf, t)
            best = np.argmin(t, axis=1)
            tb = t[np.arange(R), best]
            lab = np.where(road[np.arange(R), best], 2 + (i * sc.gh + j)[np.arange(R), best].astype(np.int64), 1)
            take = tb < tile_t
            tile_t, tile_lab = np.where(take, tb, tile_t), np.where(take, lab, tile_lab)
    cands.append((tile_t, tile_lab))
    # t*: the smallest candidate; objects come first in index order, so argmin keeps the object at a tie
    T = np.stack([t for t, _ in cands])
    L = np.stack([lab for _, lab in cands])
    first = np.argmin(T, axis=0)
    t_star = T[first, np.arange(R)]
    hit = L[first, np.arange(R)]
    if org_blocked:
        t_star[:], hit[:] = 0.0, org_label
    far = t_star > max_range
    rng = np.where(far, max_range, t_star)
    hit = np.where(far, 0, hit)
    # ambiguity
    T2 = np.concatenate([T, np.full((1, R), float(max_range))])
    amb = ((np.abs(T2 - rng[None, :]) < EPS).sum(0) >= 2) & (rng > 0)   # at 0 the origin's own label decides
    corners = [c for _, c in feet] + [np.stack(np.meshgrid(np.arange(sc.gw + 1) * ts, np.arange(sc.gh + 1) * ts),
                                               -1).reshape(-1, 2)]
    pts = np.concatenate(corners)
    wx, wz = pts[:, 0][None, :] - ox, pts[:, 1][None, :] - oz
    along = wx * dx[:, None] + wz * dz[:, None]
    perp = np.abs(wx * dz[:, None] - wz * dx[:, None])
    amb |= ((perp < EPS) & (along > -EPS) & (along < rng[:, None] + EPS)).any(1)
    edge_near = any(_point_segment_dist(ox, oz, c[k], c[(k + 1) % 4]) < EPS for _, c in feet for k in range(4))
    grid_near = (abs(ox / ts - round(ox / ts)) * ts < EPS) or (abs(oz / ts - round(oz / ts)) * ts < EPS)
    if edge_near or grid_near:
        amb[:] = True
    return rng, hit, amb


def _point_segment_dist(px, pz, a, b):
    ex, ez = b[0] - a[0], b[1] - a[1]
    u = min(1.0, max(0.0, ((px - a[0]) * ex + (pz - a[1]) * ez) / (ex * ex + ez * ez)))
    return math.hypot(px - a[0] - u * ex, pz - a[1] - u * ez)


def scan_batch(scenes, map_id, px, pz, angle, cfg, dyn_corners=None, hidden=None):
    """Every env's scan: scenes[map_id[e]] at pose e, as bev_oracle.bev_batch takes them.  Returns a list of scan's
    three results."""
    return [scan(scenes[int(map_id[e])], float(px[e]), float(pz[e]), float(angle[e]), cfg,
                 None if dyn_corners is None else dyn_corners[e], None if hidden is None else hidden[e])
            for e in range(len(px))]


def check(got_range, got_hit, expected, what="", tol=1e-5):
    """The bar: on every ray that is not ambiguous, range within tol metres and hit equal; fewer than 1 % of the rays
    ambiguous.  got_*: [N, R] arrays; expected: scan_batch's list.  Returns the number of ambiguous rays."""
    n_amb = n_all = 0
    for e, (rng, hit, amb) in enumerate(expected):
        gr, gh = np.asarray(got_range[e], np.float64), np.asarray(got_hit[e]).astype(np.int64)
        bad = ~amb & ((np.abs(gr - rng) > tol) | (gh != hit))
        if bad.any():
            k = int(np.flatnonzero(bad)[0])
            raise AssertionError(f"{what} env {e}: {int(bad.sum())} unambiguous rays differ, first ray {k}: got "
                                 f"range {gr[k]!r} hit {gh[k]}, want {rng[k]!r} {hit[k]}")
        n_amb += int(amb.sum())
        n_all += amb.size
    assert n_amb < 0.01 * n_all or n_amb == 0, f"{what}: {n_amb} of {n_all} rays are ambiguous"
    return n_amb
