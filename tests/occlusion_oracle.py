"""The float64 oracle of the occlusion mask (DESIGN.md section 5 item 14, dts_set_occlusion_target): test
infrastructure.

It restates the pixel rule in numpy float64 from flow_oracle.flow's result for a frame, the frame's labels and the
previous frame's depth and labels (the render of the recorded state in the same view).  Besides the mask it returns,
for every pixel, the set of answers a float32 restatement may give: where q - 0.5 lies within eps of an integer (the
candidates may shift by one), q within eps of the frame's edge (outside or not), a mesh's depth test within 1e-4 z'
of tau z', or flow's own oracle calls the pixel ambiguous (its NaN may flip).  eps = max(2^-9, 2e-5 |flow|), twice the
flow image's own bar.
"""
import numpy as np

TAU = 0.02
NONE, VISIBLE, OCCLUDED, OUTSIDE, UNKNOWN = range(5)
NAMES = ("none", "visible", "occluded", "outside", "unknown")
EPS_Q = 2.0 ** -9
EPS_TAU = 1e-4


def occlusion(fl, labels, n_tiles, depth_prev=None, labels_prev=None, tau=TAU) -> dict:
    """The mask of one frame.

    fl: flow_oracle.flow(...) of the frame; labels i16 [H, W]: the frame's labels; n_tiles: the map's grid cells;
    depth_prev f32 / labels_prev i16 [H, W]: the previous frame, None where no render of it was kept (UNKNOWN).

    Returns mask u8 [H, W]; allowed u8 [H, W], bit v set where v is an answer; ambiguous bool [H, W] (more than one)."""
    f = fl["flow"]
    H, W = labels.shape
    lab = np.asarray(labels).astype(np.int64)
    defined = ~np.isnan(f[..., 0])
    fx, fy = np.where(defined, f[..., 0], 0.0), np.where(defined, f[..., 1], 0.0)
    py, px = np.mgrid[0:H, 0:W]
    qx, qy = px + 0.5 + fx, py + 0.5 + fy
    ex, ey = np.maximum(EPS_Q, 2e-5 * np.abs(fx)), np.maximum(EPS_Q, 2e-5 * np.abs(fy))
    inside = (qx >= 0) & (qx < W) & (qy >= 0) & (qy < H)
    edge = (np.minimum(np.abs(qx), np.abs(qx - W)) <= ex) | (np.minimum(np.abs(qy), np.abs(qy - H)) <= ey)
    # inside-frame answers: nominal, strict (every float32 rounding visible) and lenient (some rounding visible)
    if depth_prev is None:
        vis_nom = vis_strict = vis_len = None
    else:
        dprev = np.asarray(depth_prev, np.float64)
        lprev = np.asarray(labels_prev).astype(np.int64)
        z = np.where(defined, fl["z_prev"], 0.0)
        flat = (lab >= 1) & (lab <= 1 + n_tiles)
        nx, ny = np.floor(qx - 0.5).astype(np.int64), np.floor(qy - 0.5).astype(np.int64)
        lox, hix = np.floor(qx - 0.5 - ex).astype(np.int64), np.floor(qx - 0.5 + ex).astype(np.int64)
        loy, hiy = np.floor(qy - 0.5 - ey).astype(np.int64), np.floor(qy - 0.5 + ey).astype(np.int64)
        vis_nom, vis_strict, vis_len = (np.zeros((H, W), bool) for _ in range(3))
        for dy in range(3):
            for dx in range(3):
                cx, cy = lox + dx, loy + dy
                ok = defined & (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
                sx, sy = np.clip(cx, 0, W - 1), np.clip(cy, 0, H - 1)
                same = ok & (lprev[sy, sx] == lab)
                dd = np.abs(dprev[sy, sx] - z)
                nom = same & (flat | (dd <= tau * z))
                strict = same & (flat | (dd <= (tau - EPS_TAU) * z))
                len_ = same & (flat | (dd <= (tau + EPS_TAU) * z))
                in_nom = (cx - nx >= 0) & (cx - nx <= 1) & (cy - ny >= 0) & (cy - ny <= 1)
                in_all = (cx >= hix) & (cx <= lox + 1) & (cy >= hiy) & (cy <= loy + 1)   # a candidate under every rounding
                in_any = (cx <= hix + 1) & (cy <= hiy + 1)                                 # under some rounding
                vis_nom |= nom & in_nom
                vis_strict |= strict & in_all
                vis_len |= len_ & in_any
    mask = np.full((H, W), NONE, np.uint8)
    mask[defined & ~inside] = OUTSIDE
    sel = defined & inside
    if vis_nom is None:
        mask[sel] = UNKNOWN
    else:
        mask[sel] = np.where(vis_nom[sel], VISIBLE, OCCLUDED)
    # every answer
    bit = lambda v: np.uint8(1 << v)
    inner = np.zeros((H, W), np.uint8)   # the answers when q is in the frame
    if vis_nom is None:
        inner[:] = bit(UNKNOWN)
    else:
        inner |= np.where(vis_len, bit(VISIBLE), 0).astype(np.uint8)
        inner |= np.where(~vis_strict, bit(OCCLUDED), 0).astype(np.uint8)
    allowed = np.where(defined & ~inside, bit(OUTSIDE), 0).astype(np.uint8)
    allowed |= np.where(defined & inside, inner, 0).astype(np.uint8)
    allowed |= np.where(defined & edge, bit(OUTSIDE) | inner, 0).astype(np.uint8)
    allowed |= np.where(~defined, bit(NONE), 0).astype(np.uint8)
    flip = fl["ambiguous"]   # flow's NaN may flip: none, or any answer of a defined flow
    allowed |= np.where(flip & defined, bit(NONE), 0).astype(np.uint8)
    allowed |= np.where(flip & ~defined, np.uint8(0x1f), 0).astype(np.uint8)
    popcount = sum((allowed >> v) & 1 for v in range(5))
    assert ((allowed >> mask) & 1).all()
    return dict(mask=mask, allowed=allowed, ambiguous=popcount > 1)
