"""The float64 oracle of the motion-flow image (DESIGN.md section 5 item 13, dts_set_flow_target): test infrastructure.

It restates the definition pixel by pixel in numpy float64 from the inputs a render leaves — the frame's own depth and
labels, P00 / P11 and the two frames' cameras V (dts_debug_frame, or the raster oracle's orr_debug_frame), the poses of
whatever moved, the remap table and the forward map F — without the device's composed float32 matrices.  A pixel is
ambiguous where a rounding of the device's float32 arithmetic may flip its NaN: e'_z within 1e-6 relative of the near
plane, or (x', y') within 1e-4 px of the edge of F's domain.
"""
import numpy as np

NEAR = 0.04


def ry(deg) -> np.ndarray:
    """Ry of glRotatef(deg, 0, 1, 0), the render's convention: x' = c x + s z, z' = -s x + c z"""
    t = float(deg) * 0.017453292519943295
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def rigid(V) -> np.ndarray:
    """row-major 3x4 [R|t] -> 4x4"""
    M = np.eye(4)
    M[:3] = np.reshape(np.asarray(V, np.float64), (3, 4))
    return M


def mesh_motion(prev, cur) -> np.ndarray:
    """T(p_prev) Ry(r_prev) Ry(r_cur)^-1 T(p_cur)^-1 of a mesh placed at (x, z, deg), each value rounded to float32 as the
    render passes them to glTranslatef / glRotatef (4x4)"""
    def place(p):
        x, z, deg = (float(np.float32(v)) for v in p)
        M = np.eye(4)
        M[:3, :3] = ry(deg)
        M[0, 3], M[2, 3] = x, z
        return M
    return place(prev) @ np.linalg.inv(place(cur))


def src_of_lut(rmapx, rmapy):
    """The source pixel (sx, sy) of every output pixel of a remap LUT, as the renderer builds it: rint in float32
    (half to even), -1 where it leaves the frame"""
    rx, ry_ = np.asarray(rmapx, np.float32), np.asarray(rmapy, np.float32)
    H, W = rx.shape
    fin = (np.abs(rx) < 2 ** 30) & (np.abs(ry_) < 2 ** 30)
    sx = np.where(fin, np.rint(np.where(fin, rx, 0)), -1).astype(np.int64)
    sy = np.where(fin, np.rint(np.where(fin, ry_, 0)), -1).astype(np.int64)
    ok = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H)
    return np.where(ok, sx, -1), np.where(ok, sy, -1)


def bilinear(F, x, y):
    """F [H, W] at positions (x, y) (index = position - 0.5), OpenCV's bilinear; (values, inside, margin), margin the
    distance in px of the index from the edge of the domain [0, W-1] x [0, H-1] (negative outside)"""
    H, W = F.shape
    ix, iy = x - 0.5, y - 0.5
    margin = np.minimum(np.minimum(ix, (W - 1) - ix), np.minimum(iy, (H - 1) - iy))
    inside = margin >= 0
    cx, cy = np.where(inside, ix, 0.0), np.where(inside, iy, 0.0)
    x0 = np.minimum(np.floor(cx).astype(np.int64), max(W - 2, 0))
    y0 = np.minimum(np.floor(cy).astype(np.int64), max(H - 2, 0))
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = cx - x0, cy - y0
    top = F[y0, x0] * (1 - ax) + F[y0, x1] * ax
    bot = F[y1, x0] * (1 - ax) + F[y1, x1] * ax
    return top * (1 - ay) + bot * ay, inside, margin


def flow(depth, labels, P, V_prev, V_cur, n_tiles, n_objects, moves=None, agent=None, src=None, fwd=None,
         rectify=False) -> dict:
    """The flow of one frame.

    depth f32 [H, W], labels i16 [H, W]: the frame's own images.  P: (P00, P11, ...) float32 of the frame.  V_prev,
    V_cur: the two frames' cameras, f64 row-major 3x4.  moves: {object index o: ((x, z, deg) before, (x, z, deg) now)}
    for every object that moves (its label 2 + n_tiles + o); agent: the same pair for the agent's own mesh (label
    2 + n_tiles + n_objects, top-down views).  src: (sx, sy) int [H, W] of a remap (src_of_lut), None for the pinhole
    frame.  fwd: (Fx, Fy) [H, W] forward map of the remap's camera model.  rectify: every pixel NaN.

    Returns flow f64 [H, W, 2] (NaN where undefined), ambiguous bool [H, W], z_prev = -e'_z (the point's depth in the
    previous camera) and x1, y1 (its pinhole position there), f64 [H, W] each, NaN where not computed."""
    d = np.asarray(depth, np.float64)
    lab = np.asarray(labels).astype(np.int64)
    H, W = d.shape
    if src is None:
        sy, sx = np.mgrid[0:H, 0:W]
    else:
        sx, sy = src
    xs, ys = sx + 0.5, sy + 0.5
    P00, P11 = float(np.float32(P[0])), float(np.float32(P[1]))
    E = np.stack([(2 * xs / W - 1) * d / P00, (1 - 2 * ys / H) * d / P11, -d, np.ones_like(d)], -1)   # [H, W, 4]
    Xw = E @ np.linalg.inv(rigid(V_cur)).T
    # every pixel's motion: the identity, or its item's
    Xp = Xw.copy()
    items = dict(moves or {})
    for o, (prev, cur) in items.items():
        m = lab == 2 + n_tiles + o
        Xp[m] = Xw[m] @ mesh_motion(prev, cur).T
    if agent is not None:
        m = lab == 2 + n_tiles + n_objects
        Xp[m] = Xw[m] @ mesh_motion(*agent).T
    e = Xp @ rigid(V_prev).T
    ez = e[..., 2]
    valid = (d > 0) & (sx >= 0) & (not rectify)
    front = ez < -NEAR
    amb = valid & (np.abs(ez + NEAR) <= 1e-6 * NEAR)
    with np.errstate(divide="ignore", invalid="ignore"):
        x1 = (P00 * e[..., 0] / -ez + 1) * W / 2
        y1 = (1 - P11 * e[..., 1] / -ez) * H / 2
    ok = valid & front
    out = np.full((H, W, 2), np.nan)
    if fwd is None:
        out[..., 0] = np.where(ok, x1 - xs, np.nan)
        out[..., 1] = np.where(ok, y1 - ys, np.nan)
    else:
        Fx, Fy = (np.asarray(f, np.float64) for f in fwd)
        bx = np.where(ok, x1, 0.5)
        by = np.where(ok, y1, 0.5)
        ax_, inside, margin = bilinear(Fx, bx, by)
        ay_, _, _ = bilinear(Fy, bx, by)
        sxv, syv = np.where(ok, xs, 0.5), np.where(ok, ys, 0.5)
        b0, _, _ = bilinear(Fx, sxv, syv)
        b1, _, _ = bilinear(Fy, sxv, syv)
        good = ok & inside
        amb |= ok & (np.abs(margin) <= 1e-4)
        out[..., 0] = np.where(good, ax_ - b0, np.nan)
        out[..., 1] = np.where(good, ay_ - b1, np.nan)
    z_prev = np.where(ok, -ez, np.nan)
    return dict(flow=out, ambiguous=amb, z_prev=z_prev, x1=np.where(ok, x1, np.nan), y1=np.where(ok, y1, np.nan))
