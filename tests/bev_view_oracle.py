"""A float64 numpy restatement of the bird's-eye grid's camera visibility (dts_set_bev_visibility_target, DESIGN.md
section 5 item 15): test infrastructure, written from the spec rather than from the kernel.

Inputs: the grid oracle's answer for the env (tests/bev_oracle.py), the frame's camera V and float32 P00 / P11, its own
label image and, under the fisheye, the forward map F of the env's table.  Every cell gets a bitmask of the values it
may take and its position q in the frame.  A cell is ambiguous, and may take any value of its mask, where the grid
oracle calls it ambiguous (its label, and with a tile edge its surface height, may differ), where q lies within eps of
a pixel-centre line (the four-pixel neighbourhood changes) or of the frame's edge, where -e_z lies within 1e-6 relative
of the near or far plane, or under the fisheye where F's footprint margin is at most 1e-4 px (as tests/flow_oracle.py).
eps is 1e-6 px for the pinhole frame, and under the fisheye 2^-10 px, the bar of q itself, as the device reads F in
float32."""
import numpy as np

import bev_oracle as bo

UNKNOWN, VISIBLE, OCCLUDED, OUTSIDE = range(4)
NAMES = ("unknown", "visible", "occluded", "outside")
GROUND_Y = float(np.float32(-0.8 * 0.01))   # the ground quad's height, a GLfloat
NEAR, FAR = 0.04, 100.0
EPS_PLANE = 1e-6
EPS_PX = 1e-6
EPS_PX_FISHEYE = 2.0 ** -10
EPS_FOOT = 1e-4


def surface_height(sc: bo.BevScene, x, z):
    """0 on a road tile, the ground quad's height elsewhere"""
    with np.errstate(invalid="ignore", over="ignore"):
        fi, fj = np.floor(x / sc.ts), np.floor(z / sc.ts)
    inside = (fi >= 0) & (fi < sc.gw) & (fj >= 0) & (fj < sc.gh)
    i, j = np.where(inside, fi, 0).astype(np.int64), np.where(inside, fj, 0).astype(np.int64)
    road = inside & (sc.kind[j * sc.gw + i] >= 0)
    return np.where(road, 0.0, GROUND_Y)


def bilinear_clamped(F, x, y):
    """F [H, W] at positions (x, y) with OpenCV's index = position - 0.5, the index clamped to the table; (values,
    margin): margin the index's distance in px from the edge of the domain (negative outside)"""
    H, W = F.shape
    ix, iy = x - 0.5, y - 0.5
    margin = np.minimum(np.minimum(ix, (W - 1) - ix), np.minimum(iy, (H - 1) - iy))
    cx, cy = np.clip(np.nan_to_num(ix), 0, W - 1), np.clip(np.nan_to_num(iy), 0, H - 1)
    x0 = np.minimum(np.floor(cx).astype(np.int64), max(W - 2, 0))
    y0 = np.minimum(np.floor(cy).astype(np.int64), max(H - 2, 0))
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = cx - x0, cy - y0
    top = F[y0, x0] * (1 - ax) + F[y0, x1] * ax
    bot = F[y1, x0] * (1 - ax) + F[y1, x1] * ax
    return top * (1 - ay) + bot * ay, np.where(np.isnan(margin), -np.inf, margin)


def project(V, P, W, H, x, y, z, fwd=None) -> dict:
    """World points (x, y, z) through the frame's camera: w = -e_z, the pinhole position (x1, y1), q (through F under the
    fisheye), and where they may be ambiguous"""
    V = np.reshape(np.asarray(V, np.float64), (3, 4))
    P00, P11 = float(np.float32(P[0])), float(np.float32(P[1]))
    ex = V[0, 0] * x + V[0, 1] * y + V[0, 2] * z + V[0, 3]
    ey = V[1, 0] * x + V[1, 1] * y + V[1, 2] * z + V[1, 3]
    w = -(V[2, 0] * x + V[2, 1] * y + V[2, 2] * z + V[2, 3])
    front = (w > NEAR) & (w <= FAR)
    amb = (np.abs(w - NEAR) <= EPS_PLANE * NEAR) | (np.abs(w - FAR) <= EPS_PLANE * FAR)
    with np.errstate(divide="ignore", invalid="ignore"):
        x1 = (P00 * ex / w + 1) * W / 2
        y1 = (1 - P11 * ey / w) * H / 2
    if fwd is None:
        qx, qy, foot = x1, y1, np.ones(np.shape(x1), bool)
    else:
        Fx, Fy = (np.asarray(f, np.float64) for f in fwd)
        qx, margin = bilinear_clamped(Fx, x1, y1)
        qy, _ = bilinear_clamped(Fy, x1, y1)
        foot = margin >= 0
        amb |= front & (np.abs(margin) <= EPS_FOOT)
    return dict(w=w, x1=x1, y1=y1, qx=qx, qy=qy, front=front, foot=foot, ambiguous=amb)


def _neighbourhood(lab, qx, qy, frame, eps):
    """(value, bits): the value from the pixels floor(q - 0.5) + {0, 1} in the frame, and the values of every
    neighbourhood floor(q - 0.5 +- eps) may pick"""
    H, W = frame.shape
    qx, qy = np.nan_to_num(qx, nan=-10.0), np.nan_to_num(qy, nan=-10.0)
    fr = np.asarray(frame).astype(np.int64)
    bits = np.zeros(np.shape(lab), np.uint8)
    value = None
    for ox in (0.0, -eps, eps):
        for oy in (0.0, -eps, eps):
            cx, cy = np.floor(qx - 0.5 + ox).astype(np.int64), np.floor(qy - 0.5 + oy).astype(np.int64)
            seen, shown = np.zeros(np.shape(lab), bool), np.zeros(np.shape(lab), bool)
            for j in (0, 1):
                for i in (0, 1):
                    sx, sy = cx + i, cy + j
                    ok = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H)
                    s = fr[np.clip(sy, 0, H - 1), np.clip(sx, 0, W - 1)]
                    seen |= ok & (s == lab)
                    shown |= ok & (s != 0)
            v = np.where(seen, VISIBLE, np.where(shown, OCCLUDED, OUTSIDE)).astype(np.uint8)
            bits |= (np.uint8(1) << v).astype(np.uint8)
            if value is None:
                value = v
    return value, bits


def _answer(lab, x, y, z, V, P, frame, fwd):
    H, W = frame.shape
    eps = EPS_PX if fwd is None else EPS_PX_FISHEYE
    p = project(V, P, W, H, x, y, z, fwd)
    qx, qy = p["qx"], p["qy"]
    with np.errstate(invalid="ignore"):
        inframe = (qx >= 0) & (qx < W) & (qy >= 0) & (qy < H)
        edge = (np.minimum(np.abs(qx), np.abs(qx - W)) <= eps) | (np.minimum(np.abs(qy), np.abs(qy - H)) <= eps)
    reach = p["front"] & p["foot"] & inframe
    inner, inner_bits = _neighbourhood(lab, qx, qy, frame, eps)
    value = np.where(reach, inner, OUTSIDE).astype(np.uint8)
    out = np.uint8(1 << OUTSIDE)
    bits = np.where(reach, inner_bits, out).astype(np.uint8)
    amb = p["ambiguous"] | (p["front"] & p["foot"] & edge) | (reach & (inner_bits != (np.uint8(1) << inner)))
    bits |= np.where(p["ambiguous"] | (p["front"] & p["foot"] & edge), inner_bits | out, 0).astype(np.uint8)
    q = np.stack([qx, qy], -1)
    q[value == OUTSIDE] = np.nan
    return value, bits, q, amb


def visibility(sc: bo.BevScene, pose, cfg, grid, V, P, frame, fwd=None) -> dict:
    """One env's cells.  pose: (pos_x, pos_z, angle) the grid was taken at; cfg: (width, height, cell, origin_x,
    origin_y); grid: bo.bev_grid's result at that pose; V f64 [12] / P f32 [4]: the frame's camera; frame: its label image
    i16 [H, W]; fwd: (Fx, Fy) of the env's fisheye table, None for the pinhole frame.

    Returns value u8 [h, w] (VISIBLE, OCCLUDED or OUTSIDE), allowed u8 [h, w] (bit v set where v is an answer),
    q f64 [h, w, 2] (NaN where OUTSIDE), w = -e_z f64 [h, w] and ambiguous bool [h, w]."""
    lab, _, amb_bev, (alt_l, _) = grid
    x, z = bo.cell_centres(*pose, *cfg)
    y = surface_height(sc, x, z)
    value, allowed, q, amb = _answer(lab, x, y, z, V, P, frame, fwd)
    if amb_bev.any():   # any of the cell's labels, on either surface
        for cand in [lab] + list(alt_l):
            for yy in (0.0, GROUND_Y):
                _, b, _, _ = _answer(cand, x, np.full_like(y, yy), z, V, P, frame, fwd)
                allowed |= np.where(amb_bev, b, 0).astype(np.uint8)
    amb |= amb_bev
    V3 = np.reshape(np.asarray(V, np.float64), (3, 4))
    w = -(V3[2, 0] * x + V3[2, 1] * y + V3[2, 2] * z + V3[2, 3])
    assert ((allowed >> value) & 1).all()
    return dict(value=value, allowed=allowed, q=q, w=w, ambiguous=amb)
