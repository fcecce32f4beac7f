"""src/gym_duckietown/wrappers.py's ResizeWrapper (cv2.resize, INTER_CUBIC): the numpy restatement in
oracle/cv2_cubic.py, which the GPU tests hold the device pass to at 0 LSB, pinned against what the reference class
returned (tests/golden/wrappers.npz), against OpenCV itself where it imports, and against a float64 convolution.
Also the host arithmetic of the device's band plan (plan_resize_bands in dts_post.cu), so that the GPU sweep below
keeps reaching every branch of k_resize_band / k_resize."""
import os

import numpy as np
import pytest

import cv2_cubic as C
from test_reference_wrappers import canned_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "wrappers.npz")

# ((camera w, h), (target w, h), output rows per band of k_resize_band (0: the untiled k_resize))
SWEEP = [((160, 120), (84, 84), 16),       # the c2 benchmark shape; tallest band, just under the 40 KB budget
         ((160, 120), (80, 80), 16),
         ((160, 120), (64, 48), 11),
         ((640, 480), (84, 84), 2),
         ((640, 480), (80, 80), 2),
         ((640, 480), (64, 48), 2),
         ((640, 480), (160, 120), 2),
         ((640, 480), (20, 15), 1),        # 32x reduction
         ((800, 600), (2000, 8), 1),       # single rows above 48 KB: the shared-memory opt-in
         ((800, 600), (4096, 8), 0),       # no band fits in 200 KB: the untiled kernel
         ((160, 120), (83, 61), 12),       # output rows of 249 bytes: the non-word store
         ((162, 121), (84, 40), 8),        # source rows of 486 bytes: byte staging, word store
         ((162, 121), (53, 40), 11),       # byte staging, non-word store
         ((160, 120), (320, 240), 9),      # 2x upscale
         ((33, 17), (100, 50), 16),        # upscale on both axes: both borders clamp
         ((160, 120), (1, 1), 16),
         ((160, 120), (1, 84), 16),
         ((160, 120), (84, 1), 16),
         ((84, 84), (84, 84), 16)]         # identity
SWEEP_IDS = [f"{w}x{h}-{ow}x{oh}" for (w, h), (ow, oh), _ in SWEEP]

BAND_SMEM = 40 * 1024            # kResizeBandSmem
OPT_IN_MAX = 200 * 1024          # single-row bands may opt in up to this much dynamic shared memory


def band_smem(W, ow, cap):
    return ow * 16 + ((cap * W * 3 + 15) & ~15) + cap * ow * 3 * 4 + 16


def plan_bands(W, ow, oh, yidx):
    """(rows per band, largest source-row span, shared memory) as plan_resize_bands picks them; (0, 0, 0): untiled."""
    for R in range(16, 0, -1):
        cap = max(int(yidx[min(r0 + R, oh) - 1, 3] - yidx[r0, 0]) + 1 for r0 in range(0, oh, R))
        smem = band_smem(W, ow, cap)
        if smem <= BAND_SMEM or (R == 1 and smem <= OPT_IN_MAX):
            return R, cap, smem
    return 0, 0, 0


def staging(W, H, oh, yidx, R, cap, n_envs):
    """{'int4', 'bytes'}: how k_resize_band copies each band's source rows (16-byte loads need an aligned band whose
    byte count is a multiple of 16; the frames tensor itself is 16-byte aligned)."""
    kinds = set()
    for env in range(n_envs):
        for r0 in range(0, oh, R):
            s_lo, s_hi = int(yidx[r0, 0]), int(yidx[min(r0 + R, oh) - 1, 3])
            off, nbytes = env * W * H * 3 + s_lo * W * 3, min(s_hi - s_lo + 1, cap) * W * 3
            kinds.add("int4" if off % 16 == 0 and nbytes % 16 == 0 else "bytes")
    return kinds


def sweep_frames(n, w, h, seed):
    """u8 [n][h][w][3], n >= 6: noise, a one-pixel 0/255 checkerboard, a coarser checkerboard whose channels differ,
    0/255 step edges, and noise with saturated blocks.  The cubic's negative lobes overshoot past 0 and 255 at every
    hard edge, so both clips and negative accumulators occur."""
    rng = np.random.default_rng([seed, w, h])
    f = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    f[1] = np.where((xx + yy) % 2, 255, 0)[..., None]
    f[2] = np.stack([np.where((xx // 3 + yy // 2) % 2, 255, 0), np.where((xx // 2 + yy // 3) % 2, 0, 255),
                     np.where((xx // 5 + yy) % 2, 255, 0)], -1)
    f[3] = np.where(xx < w // 2, 0, 255)[..., None]
    f[3, h // 3:] = 255 - f[3, h // 3:]
    f[3, :, w // 4: w // 4 + 1, 1] = 255
    f[5, : h // 2, : w // 3] = 0
    f[5, h // 3:, w // 2:] = 255
    return f


def test_sweep_plans_and_covers_every_branch_of_the_device_pass():
    """The band height each sweep shape gets, and that the sweep as a whole runs every branch: R = 16, 1 < R < 16,
    R = 1 within 40 KB and with the opt-in, the untiled kernel, word and non-word stores, 16-byte and byte staging."""
    seen = set()
    for (w, h), (ow, oh), rows in SWEEP:
        yidx, _ = C.axis_table(h, oh)
        R, cap, smem = plan_bands(w, ow, oh, yidx)
        assert R == rows, ((w, h), (ow, oh), R)
        if R == 0:
            seen.add("untiled")
            continue
        seen.add("R=16" if R == 16 else "R=1" if R == 1 else "1<R<16")
        if R == 1:
            seen.add("opt-in" if smem > 48 * 1024 else "R=1 in budget")
        seen.add("word" if (ow * 3) % 4 == 0 else "non-word")
        seen |= staging(w, h, oh, yidx, R, cap, 6)
    assert seen == {"R=16", "1<R<16", "R=1", "R=1 in budget", "opt-in", "untiled", "word", "non-word", "int4", "bytes"}
    y = C.axis_table(120, 84)[0]
    assert plan_bands(160, 84, 84, y) == (16, 26, 40048)       # the benchmark shape: 912 B under the budget
    assert plan_bands(800, 2000, 8, C.axis_table(600, 8)[0]) == (1, 4, 137616)


# ------------------------------------------------------------------------------------------------ the tap tables
TABLE_AXES = [(120, 84), (160, 84), (480, 15), (640, 20), (600, 8), (800, 4096), (800, 2000), (120, 240), (17, 50),
              (33, 100), (160, 1), (84, 84), (121, 40), (162, 53), (1, 5)]


@pytest.mark.parametrize("src,dst", TABLE_AXES)
def test_tables_index_the_image_in_order_and_taps_sum_to_one(src, dst):
    idx, taps = C.axis_table(src, dst)
    assert idx.shape == taps.shape == (dst, 4)
    assert idx.min() >= 0 and idx.max() <= src - 1
    assert (np.diff(idx, axis=1) >= 0).all() and (np.diff(idx, axis=0) >= 0).all()
    assert np.abs(taps.sum(1) - 2048).max() <= 1            # measured: rint() of four weights loses at most 1
    assert np.abs(taps).max() <= 2048


def test_identity_axis_is_an_exact_copy():
    idx, taps = C.axis_table(84, 84)
    assert np.array_equal(idx[:, 1], np.arange(84)) and (taps == [0, 2048, 0, 0]).all()
    f = sweep_frames(6, 84, 84, 0)
    assert np.array_equal(C.resize(f, 84, 84), f)


def test_tables_follow_opencv_sampling_and_rounding():
    """fx = float32((d + 0.5) * scale - 0.5); taps rint(2048 c), half to even, against the float32 weights."""
    sx, c = C.axis_weights(120, 84)
    assert c.dtype == np.float32 and np.array_equal(c.sum(1, dtype=np.float64).round(5), np.ones(84))
    idx, taps = C.axis_table(120, 84)
    assert np.array_equal(taps, np.rint(c.astype(np.float64) * 2048).astype(np.int64))
    assert np.array_equal(idx[:, 0], np.clip(sx - 1, 0, 119))
    assert sx[0] == 0 and sx[-1] == 118                     # (83.5 * 120/84 - 0.5) = 118.79
    assert C.axis_weights(17, 50)[0][0] == -1               # upscales start left of the image


# ------------------------------------------------------------------------------------------------ against the golden
# fraction of values the restatement moves by 1 LSB from the reference class's frames (OpenCV's vectorised vertical
# pass sums in float32), measured, with a little headroom
GOLDEN_FRACTION = {"160x120_80x80": 0.025, "160x120_84x84": 0.061, "160x120_64x48": 0.0,
                   "640x480_80x80": 0.043, "640x480_84x84": 0.044, "640x480_64x48": 0.068}


@pytest.mark.parametrize("key", list(GOLDEN_FRACTION))
def test_restatement_against_the_reference_resize_wrapper(key):
    g = np.load(GOLD)
    tag, size = key.split("_")
    (w, h), (rw, rh) = (map(int, s.split("x")) for s in (tag, size))
    frames = canned_frames(int(g["seed"]), h, w)
    want = g[f"resize_{key}"].transpose(0, 3, 2, 1)          # the wrapper's [C][W][H] -> [H][W][C]
    d = np.abs(C.resize(frames, rw, rh).astype(int) - want)
    assert d.max() <= 1 and (d > 0).mean() <= GOLDEN_FRACTION[key], (int(d.max()), float((d > 0).mean()))


# ------------------------------------------------------------------------------------------------ against OpenCV
# sweep shapes where OpenCV with setUseOptimized(False) equals the restatement on every value of sweep_frames.  At
# the others a few values differ by 1, all with the exact sum at (within float32 rounding of) a half LSB before the
# shift: its vertical pass still sums in float32 and rounds ties to even, where the fixed-point code rounds them up
CV2_SCALAR_EXACT = {"160x120-84x84", "160x120-64x48", "640x480-84x84", "162x121-84x40", "162x121-53x40",
                    "160x120-1x1", "160x120-1x84", "160x120-84x1", "84x84-84x84"}


def unshifted(frames, ow, oh, at):
    """The integer vertical sums (before the rounding shift) of the output values at the indices `at`."""
    H, W = frames.shape[1:3]
    xi, xw = C.axis_table(W, ow)
    yi, yw = C.axis_table(H, oh)
    return np.array([sum(int(yw[y, r]) * sum(int(frames[n, yi[y, r], xi[x, k], c]) * int(xw[x, k]) for k in range(4))
                         for r in range(4)) for n, y, x, c in at], np.int64)


@pytest.fixture
def cv2_mod():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    yield cv2
    cv2.setUseOptimized(was)


@pytest.mark.parametrize("cam,target,rows", SWEEP, ids=SWEEP_IDS)
def test_restatement_against_opencv(cam, target, rows, cv2_mod):
    cv2 = cv2_mod
    (w, h), (ow, oh) = cam, target
    frames = sweep_frames(6, w, h, 11)
    got = C.resize(frames, ow, oh)

    def cv2_resize():
        return np.stack([cv2.resize(f, (ow, oh), interpolation=cv2.INTER_CUBIC) for f in frames])

    cv2.setUseOptimized(True)
    d = np.abs(got.astype(int) - cv2_resize())
    assert d.max() <= 1, int(d.max())
    cv2.setUseOptimized(False)
    scalar = cv2_resize()
    at = np.argwhere(got != scalar)
    if f"{w}x{h}-{ow}x{oh}" in CV2_SCALAR_EXACT:
        assert len(at) == 0, len(at)
        return
    v, cv, mine = unshifted(frames, ow, oh, at), scalar[tuple(at.T)].astype(int), got[tuple(at.T)].astype(int)
    off_half = np.abs(v % (1 << 22) - (1 << 21))
    assert off_half.max() <= 1 << 8 and (np.abs(cv - mine) == 1).all()        # only sums at a half LSB differ ...
    tie = off_half == 0
    assert np.array_equal(mine[tie], (v[tie] >> 22) + 1)                        # ... which the shift rounds up
    assert np.array_equal(cv[tie], (v[tie] >> 22) + (v[tie] >> 22) % 2)         # and OpenCV to even


# ------------------------------------------------------------------------------------------------ against float64
def float64_resize(frames, ow, oh):
    """Separable convolution with the a = -0.75 cubic evaluated in float64 at the double-precision sample position,
    same clamping, rounded to nearest: no tap quantisation, no float32."""
    def axis(src, dst):
        fx = (np.arange(dst) + 0.5) * (src / dst) - 0.5
        sx = np.floor(fx)
        t = np.abs((fx - sx)[:, None] - (np.arange(4) - 1)[None, :])               # distance to taps sx-1 .. sx+2
        a = -0.75
        w = np.where(t <= 1, ((a + 2) * t - (a + 3)) * t * t + 1, ((a * t - 5 * a) * t + 8 * a) * t - 4 * a)
        return np.clip(sx[:, None].astype(int) - 1 + np.arange(4), 0, src - 1), w
    H, W = frames.shape[1:3]
    xi, xw = axis(W, ow)
    yi, yw = axis(H, oh)
    f = frames.astype(np.float64)
    hsum = sum(f[:, :, xi[:, k]] * xw[None, None, :, k, None] for k in range(4))
    return np.clip(np.rint(sum(hsum[:, yi[:, k]] * yw[None, :, k, None, None] for k in range(4))), 0, 255)


@pytest.mark.parametrize("cam,target,rows", SWEEP, ids=SWEEP_IDS)
def test_restatement_against_a_float64_convolution(cam, target, rows):
    (w, h), (ow, oh) = cam, target
    frames = sweep_frames(6, w, h, 12)
    d = np.abs(C.resize(frames, ow, oh) - float64_resize(frames, ow, oh))
    assert d.max() <= 1, float(d.max())                     # measured: 11-bit taps move values by at most 1 LSB


def test_restatement_batches_and_chunks_like_single_frames(monkeypatch):
    frames = sweep_frames(6, 160, 120, 13)
    whole = C.resize(frames, 84, 84)
    monkeypatch.setattr(C, "CHUNK_BYTES", 1)                # one frame per chunk
    assert np.array_equal(C.resize(frames.reshape(2, 3, 120, 160, 3), 84, 84), whole.reshape(2, 3, 84, 84, 3))
    assert np.array_equal(np.stack([C.resize(f, 84, 84) for f in frames]), whole)
    with pytest.raises(ValueError):
        C.resize(frames.astype(np.float32), 84, 84)
