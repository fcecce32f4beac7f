"""A float64 numpy restatement of the lane path (dts_set_lane_path_target, DESIGN.md section 5 item 18): test
infrastructure, written from the spec rather than from the kernel.

closest_curve_point is restated over many queries at once: the tile under each query, the tile's curve whose chord
(every chord divided by the one Frobenius norm of them all, summed curve by curve) is best aligned with the heading,
then bezier_closest's 8-level bisection.  The walk steps `spacing` along each tangent and takes the next curve by the
tangent's heading.  Each point also carries whether it is ambiguous: where the device's sincos / atan2 may differ from
libm's by an ulp, a different curve, bisection branch or tile could follow, so that point and the rest of its chain
are not held to the oracle.  The frame's camera (and under the fisheye the env's forward map) gives where each point
lands, through the bird's-eye visibility oracle's projection."""
import numpy as np

import bev_view_oracle as vo

AMB_DOT = 1e-9     # the top two chords' dot products closer than this
AMB_DIST = 1e-12   # a bisection level's two distances closer than this
AMB_EDGE = 1e-9    # a query this close to a tile edge (metres)


class Curves:
    """A map's curves per tile, padded: cp [tiles, C, 4, 3], n [tiles] (0: no tile, or not drivable)"""

    def __init__(self, md):
        self.md = md
        nt = md.grid_w * md.grid_h
        cmax = max(int(md.tile_curve_cnt.max()), 1)
        self.cp = np.zeros((nt, cmax, 4, 3))
        self.n = np.where((md.tile_kind >= 0) & (md.tile_drivable != 0), md.tile_curve_cnt, 0).astype(np.int64)
        for idx in np.flatnonzero(self.n):
            o, c = int(md.tile_curve_off[idx]), int(md.tile_curve_cnt[idx])
            self.cp[idx, :c] = md.curves[o:o + c]


def bezier(cp, t):
    """cp [n, 4, 3], t [n] -> [n, 3], in the order bezier_at sums"""
    s = 1 - t
    b = [s * s * s, 3 * t * (s * s), 3 * (t * t) * s, t * t * t]
    p = b[0][:, None] * cp[:, 0]
    for k in range(1, 4):
        p = p + b[k][:, None] * cp[:, k]
    return p


def closest_curve_point(cv, x, z, angle):
    """Queries (x, 0, z) with headings angle, each [n] -> (found [n], q [n, 3], t [n, 3], ambiguous [n])"""
    md = cv.md
    ts = md.tile_size
    n = len(x)
    fi, fj = np.floor(x / ts), np.floor(z / ts)
    on = (fi >= 0) & (fi < md.grid_w) & (fj >= 0) & (fj < md.grid_h)
    idx = np.where(on, fj * md.grid_w + fi, 0).astype(np.int64)
    nc = np.where(on, cv.n[idx], 0)
    found = nc > 0
    # a query on a tile edge may fall into either tile
    fx, fz = x / ts, z / ts
    amb = (np.abs(fx - np.round(fx)) * ts < AMB_EDGE) | (np.abs(fz - np.round(fz)) * ts < AMB_EDGE)
    q = np.full((n, 3), np.nan)
    tg = np.full((n, 3), np.nan)
    e = np.flatnonzero(found)
    if not len(e):
        return found, q, tg, amb
    cps = cv.cp[idx[e]]                                   # [m, C, 4, 3]
    valid = np.arange(cps.shape[1])[None, :] < nc[e, None]
    h = np.where(valid[..., None], cps[:, :, 3] - cps[:, :, 0], 0.0)
    fro = np.zeros(len(e))
    for c in range(cps.shape[1]):
        for d in range(3):
            fro = fro + h[:, c, d] * h[:, c, d]
    fro = np.sqrt(fro)
    dirx, dirz = np.cos(angle[e]), -np.sin(angle[e])
    dots = (h[:, :, 0] / fro[:, None]) * dirx[:, None] + (h[:, :, 2] / fro[:, None]) * dirz[:, None]
    dots = np.where(valid, dots, -np.inf)
    best = np.argmax(dots, axis=1)                         # the first maximum
    srt = np.sort(dots, axis=1)
    amb[e] |= (nc[e] > 1) & (srt[:, -1] - srt[:, -2] < AMB_DOT)
    cp = cps[np.arange(len(e)), best]                      # [m, 4, 3]
    p = np.stack([x[e], np.zeros(len(e)), z[e]], 1)
    lo, hi = np.zeros(len(e)), np.ones(len(e))
    for _ in range(8):
        mid = (lo + hi) * 0.5
        a, b = bezier(cp, lo), bezier(cp, hi)
        dlo = np.sqrt((a[:, 0] - p[:, 0]) ** 2 + a[:, 1] * a[:, 1] + (a[:, 2] - p[:, 2]) ** 2)
        dhi = np.sqrt((b[:, 0] - p[:, 0]) ** 2 + b[:, 1] * b[:, 1] + (b[:, 2] - p[:, 2]) ** 2)
        amb[e] |= np.abs(dlo - dhi) < AMB_DIST
        go_lo = dlo < dhi
        hi = np.where(go_lo, mid, hi)
        lo = np.where(go_lo, lo, mid)
    t = (lo + hi) * 0.5
    s = 1 - t
    q[e] = bezier(cp, t)
    d = (3 * (s * s))[:, None] * (cp[:, 1] - cp[:, 0])
    d = d + (6 * s * t)[:, None] * (cp[:, 2] - cp[:, 1])
    d = d + (3 * (t * t))[:, None] * (cp[:, 3] - cp[:, 2])
    tg[e] = d / np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])[:, None]
    return found, q, tg, amb


def walk(md, poses, n_points, spacing, curves=None):
    """poses [n, 3] (pos_x, pos_z, angle) -> q [n, K, 3], t [n, K, 3] (NaN past the count), count [n], and ambiguous
    [n, K]: the first ambiguous point of each chain and every point after it"""
    cv = curves or Curves(md)
    poses = np.asarray(poses, np.float64)
    n = len(poses)
    q = np.full((n, n_points, 3), np.nan)
    t = np.full((n, n_points, 3), np.nan)
    count = np.zeros(n, np.int64)
    amb = np.zeros((n, n_points), bool)
    x, z, a = poses[:, 0].copy(), poses[:, 1].copy(), poses[:, 2].copy()
    live = np.ones(n, bool)
    tainted = np.zeros(n, bool)
    for k in range(n_points):
        e = np.flatnonzero(live)
        if not len(e):
            break
        found, qk, tk, ak = closest_curve_point(cv, x[e], z[e], a[e])
        tainted[e] |= ak
        amb[e, k] = tainted[e]
        f = e[found]
        q[f, k], t[f, k] = qk[found], tk[found]
        count[f] = k + 1
        live[e[~found]] = False
        a[f] = np.arctan2(-t[f, k, 2], t[f, k, 0])
        x[f] = q[f, k, 0] + spacing * t[f, k, 0]
        z[f] = q[f, k, 2] + spacing * t[f, k, 2]
    # past a chain's end: ambiguous when its last call was
    for e in np.flatnonzero(tainted):
        amb[e, np.argmax(amb[e]):] = True
    return q, t, count, amb


def agent_frame(poses, q, t):
    """[n, K, 3]: forward, right of each point from the agent, and the tangent's yaw against its heading in (-pi, pi]"""
    poses = np.asarray(poses, np.float64)
    ca, sa = np.cos(poses[:, 2])[:, None], np.sin(poses[:, 2])[:, None]
    dx, dz = q[..., 0] - poses[:, 0, None], q[..., 2] - poses[:, 1, None]
    fe, re = t[..., 0] * ca - t[..., 2] * sa, t[..., 0] * sa + t[..., 2] * ca
    yaw = np.arctan2(-re, fe)
    yaw = np.where(yaw <= -np.pi, np.pi, yaw)
    return np.stack([dx * ca - dz * sa, dx * sa + dz * ca, yaw], -1)


def lane_pose(points):
    """Point 0's lane pose from its agent-frame row: (dist, angle_rad) of get_lane_pos2"""
    f, r, yaw = points[..., 0], points[..., 1], points[..., 2]
    return -f * np.sin(yaw) - r * np.cos(yaw), yaw


def pixels(q, count, camera):
    """One env's points q [K, 3] through camera (V f64 [12], P f32 [4], W, H, fwd) as item 17 projects a corner ->
    px [K, 2] (NaN where the spec says) and ambiguous [K]: at a near or far plane, or at the edge of F's footprint"""
    K = len(q)
    px = np.full((K, 2), np.nan)
    amb = np.zeros(K, bool)
    if camera is None or count == 0:
        return px, amb
    V, P, W, H, fwd = camera
    p = q[:count]
    r = vo.project(V, P, W, H, p[:, 0], p[:, 1], p[:, 2], fwd)
    ok = r["front"] & r["foot"]
    px[:count, 0] = np.where(ok, r["qx"], np.nan)
    px[:count, 1] = np.where(ok, r["qy"], np.nan)
    amb[:count] = r["ambiguous"]
    return px, amb
