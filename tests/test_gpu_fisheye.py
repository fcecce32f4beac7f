"""The fused fisheye gather (DTS_FLAG_DISTORTION) against the CPU raster oracle under LUTs whose answer is known
exactly, and the frame-memory overflow contract.

Under the fisheye a coarse bin is the bounding box of the source pixels its output pixels name, so the binning (the
two inverse indices, the home-cell range grown by ext_x / ext_y), the fine-bin boxes, the empty-bin path and the
per-lane source lookup only meet their edge cases under LUTs other than the real one: boxes far from their bin,
boxes spanning several cells, bins with no valid source, half-integer and non-finite entries.  The bar is the
oracle's frame, 0 LSB on every channel value."""
import os

import numpy as np
import pytest


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


THREADS = os.cpu_count() or 1
KINDS = ["identity", "mirror_x", "rot180", "transpose", "shift", "ties", "specials", "zoom", "jitter", "permutation", "real"]
KINDS_FULL_RES = ["identity", "mirror_x", "jitter", "real"]   # 640x480: the kinds whose boxes pass the int32 edge bound


def kinds_for(W, H):
    if (W, H) == (640, 480):
        return KINDS_FULL_RES
    return [k for k in KINDS if k != "transpose" or W == H]


def make_lut(kind, W, H, real=None):
    """float32 (rmapx, rmapy) [H][W] of one synthetic LUT kind; `real` supplies the Distortion LUT for "real"."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    if kind == "identity":
        return x, y
    if kind == "mirror_x":       # boxes far from their output bin
        return W - 1 - x, y
    if kind == "rot180":
        return W - 1 - x, H - 1 - y
    if kind == "transpose":      # a 32x8 output bin reads an 8x32 source box: ext_y > 0
        assert W == H
        return y.copy(), x.copy()
    if kind == "shift":          # whole coarse bins without a source, partly valid fine bins
        return x + 37, y - 13
    if kind == "ties":           # x.5: round half to even; -0.5 -> 0 (valid), W - 0.5 -> W (invalid for even W)
        rx, ry = x + 0.5, y + 0.5
        rx[:, 0] = -0.5
        ry[0, :] = -0.5
        return rx, ry
    if kind == "specials":       # non-finite and out-of-int-range entries are invalid (black)
        rng = np.random.default_rng(11)
        rx, ry = x.copy(), y.copy()
        vals = np.array([np.nan, np.inf, -np.inf, 1e10, -1e10, 3e9], np.float32)
        for m in (rx, ry):
            pick = rng.random((H, W)) < 0.01
            m[pick] = vals[rng.integers(len(vals), size=int(pick.sum()))]
        return rx, ry
    if kind == "zoom":           # many output pixels on one source pixel
        return 4 * (x // 4) + 1, 2 * (y // 2)
    if kind == "jitter":         # boxes spanning 2-3 cells
        rng = np.random.default_rng(12)
        return x + rng.integers(-6, 7, (H, W)), y + rng.integers(-6, 7, (H, W))
    if kind == "permutation":    # every box is the whole image: every prim in every bin, lists of > 32 records
        p = np.random.default_rng(13).permutation(W * H).reshape(H, W)
        return (p % W).astype(np.float32), (p // W).astype(np.float32)
    if kind == "real":
        return real.rmapx, real.rmapy
    raise ValueError(kind)


def numpy_gather(frames, rx, ry):
    """out[y, x] = frame[rint(ry), rint(rx)] where that lies in the image (finite entries only), else 0."""
    H, W = rx.shape
    ok = np.isfinite(rx) & np.isfinite(ry)
    ix, iy = np.where(ok, np.rint(rx), -1.0), np.where(ok, np.rint(ry), -1.0)
    ok &= (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    out = np.zeros_like(frames)
    out[:, ok] = frames[:, iy[ok].astype(np.int64), ix[ok].astype(np.int64)]
    return out


def random_poses(md, N, seed):
    """N cameras on random points of random drivable tiles, random headings."""
    rng = np.random.default_rng(seed)
    cells = np.array(md.drivable_tiles)[rng.integers(len(md.drivable_tiles), size=N)]
    px = (cells[:, 0] + rng.uniform(size=N)) * md.tile_size
    pz = (cells[:, 1] + rng.uniform(size=N)) * md.tile_size
    return px, pz, rng.uniform(-np.pi, np.pi, size=N)


def lsb_diff(got, ref):
    d = np.abs(got.astype(np.int16) - ref.astype(np.int16))
    return int(d.max()), int((d > 0).sum())


def test_oracle_gather_equals_numpy_gather():
    """CPU only: for every LUT kind the oracle's fused gather equals a numpy gather of its plain frame, which pins the
    reference the GPU tests below compare with (rint half to even, non-finite / out-of-range entries black)."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.distortion import Distortion

    md = maps.load_map("loop_obstacles")
    sc = orc.OracleScene(md)
    for W, H in ((160, 120), (84, 84)):
        px, pz, ang = random_poses(md, 4, 7)
        eps = [orc.default_episode() for _ in px]
        plain = sc.render_batch(px, pz, ang, eps, W, H, False, threads=THREADS)
        real = Distortion(W, H)
        for kind in kinds_for(W, H):
            rx, ry = make_lut(kind, W, H, real)
            fused = sc.render_batch(px, pz, ang, eps, W, H, False, lut=(rx, ry), threads=THREADS)
            want = numpy_gather(plain, rx, ry)
            assert np.array_equal(fused, want), f"{kind} {W}x{H}: max diff {lsb_diff(fused, want)}"
            if kind in ("ties", "specials", "shift"):
                assert (want == 0).all(-1).any(), f"{kind}: the LUT was meant to leave some pixels without a source"
        assert np.array_equal(real.distort(plain[0]), numpy_gather(plain[:1], real.rmapx, real.rmapy)[0])


def _render_twice(env, torch):
    a = env.render_obs().clone()
    b = env.render_obs(out=torch.empty_like(a))
    torch.cuda.synchronize()
    assert torch.equal(a, b), "two renders of the same state differ"
    return a.cpu().numpy()


def _check_kinds(env, torch, md, kinds, px, pz, ang, chw_f32=False):
    """Install each LUT kind, render, compare with the oracle; returns the kinds that differ, with their diffs."""
    import oracle as orc
    W, H = env.camera_width, env.camera_height
    sc = orc.OracleScene(md)
    eps = [orc.default_episode() for _ in px]
    bad = []
    for kind in kinds:
        rx, ry = make_lut(kind, W, H, env.camera_model)
        env.sim.set_fisheye_lut(rx, ry)
        got = _render_twice(env, torch)
        ref = sc.render_batch(px, pz, ang, eps, W, H, False, lut=(rx, ry), threads=THREADS)
        if chw_f32:
            want = (ref.transpose(0, 3, 1, 2) / 255.0).astype(np.float32)
            if not np.array_equal(got, want):
                bad.append((kind, lsb_diff(np.rint(got * 255.0).astype(np.uint8), ref.transpose(0, 3, 1, 2))))
        else:
            mx, n = lsb_diff(got, ref)
            if mx:
                bad.append((kind, (mx, n)))
        assert ref.std() > 10, f"{kind}: the oracle's frames are blank"
    env.check()
    return bad


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
@pytest.mark.parametrize("W,H,fmt", [
    (160, 120, "hwc_u8"),    # k_raster_solo / k_raster_flat / k_raster<false, true>
    (84, 84, "hwc_u8"),      # lean, partial fine bins on the right and bottom edges; square: the transpose LUT
    (90, 70, "hwc_u8"),      # W % 4 != 0: k_raster<false, true> alone, partial bins on both edges
    (160, 120, "chw_f32"),   # k_raster<true, true>
    (640, 480, "hwc_u8"),    # > 128 coarse bins: k_bin with 4 warps
])
def test_lut_family_vs_oracle(name, W, H, fmt, torch_cuda):
    """Every synthetic LUT kind on 256 random drivable-tile cameras: each frame equals the oracle's (0 LSB), a second
    render of the same state is byte-equal, and no frame ran out of frame memory.  The list of kinds that differ, with
    (max diff, values that differ), is the failure message."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv

    md = maps.load_map(name)
    N = 256
    px, pz, ang = random_poses(md, N, 2025)
    env = BatchedDuckietownEnv(N, name, camera_width=W, camera_height=H, domain_rand=False, distortion=True, seed=5)
    if fmt == "chw_f32":
        env.set_output_format(obs_layout="chw", obs_dtype="float32")
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    bad = _check_kinds(env, torch, md, kinds_for(W, H), px, pz, ang, chw_f32=fmt == "chw_f32")
    env.close()
    assert not bad, f"{name} {W}x{H} {fmt}: frames differ from the oracle under {bad}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
def test_lut_batch_scale_vs_oracle(name, torch_cuda):
    """2048 cameras at 160x120: the batch sizes at which k_raster_flat hands bins back to k_raster and rare bins
    (depth ties, long lists) occur, under the identity, permutation and real LUTs."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv

    md = maps.load_map(name)
    N, W, H = 2048, 160, 120
    px, pz, ang = random_poses(md, N, 2024)
    env = BatchedDuckietownEnv(N, name, camera_width=W, camera_height=H, domain_rand=False, distortion=True, seed=5)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    bad = _check_kinds(env, torch, md, ["identity", "permutation", "real"], px, pz, ang)
    env.close()
    assert not bad, f"{name}: frames differ from the oracle under {bad}"


@pytest.mark.gpu
def test_fisheye_c4_semantics_vs_oracle(torch_cuda):
    """The benchmark's fisheye config: udem1, 640x480, real LUT, domain randomisation, 64 envs after reset() with
    host-drawn episode parameters.  The oracle's fused gather equals the product's numpy gather (Distortion.distort) of
    the oracle's plain frame, and the GPU's frames equal the oracle's (0 LSB)."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from test_gpu_render import oracle_episode

    N, W, H = 64, 640, 480
    env = BatchedDuckietownEnv(N, "udem1", camera_width=W, camera_height=H, domain_rand=True, distortion=True, seed=50)
    captured = {}
    orig = env.sim.reset
    env.sim.reset = lambda mask, params, stream=0: (captured.update(params), orig(mask, params, stream))[1]
    gpu = env.reset().cpu().numpy()
    env.check()
    st = {k: v.cpu().numpy() for k, v in env.state.items()}
    sc = orc.OracleScene(maps.load_map("udem1"))
    eps = [oracle_episode(orc, captured, k) for k in range(N)]
    lut = (env.camera_model.rmapx, env.camera_model.rmapy)
    cpu = sc.render_batch(st["pos_x"], st["pos_z"], st["angle"], eps, W, H, True, lut=lut, threads=THREADS)
    undist = sc.render_batch(st["pos_x"], st["pos_z"], st["angle"], eps, W, H, True, threads=THREADS)
    for k in range(N):
        assert np.array_equal(env.camera_model.distort(undist[k]), cpu[k]), k   # oracle gather == product's numpy gather
    mx, n = lsb_diff(gpu, cpu)
    assert mx == 0, f"max diff {mx} LSB on {n} channel values"
    env.close()


@pytest.mark.gpu
def test_too_wide_lut_is_refused_and_the_previous_stays(torch_cuda):
    """A LUT that sends one coarse output bin to both far corners of the image would overflow the rasteriser's int32
    edge functions: set_fisheye_lut raises, and the LUT set before stays in effect."""
    torch = torch_cuda
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.lib import DtsError

    N, W, H = 8, 640, 480
    env = BatchedDuckietownEnv(N, "udem1", camera_width=W, camera_height=H, domain_rand=False, distortion=True, seed=3)
    env.reset(render=False)
    before = _render_twice(env, torch)
    rx, ry = make_lut("identity", W, H)
    rx[0:8, 0:16], ry[0:8, 0:16] = 0, 0                      # coarse bin 0: half its pixels on (0, 0) ...
    rx[0:8, 16:32], ry[0:8, 16:32] = W - 1, H - 1            # ... half on (639, 479)
    with pytest.raises(DtsError, match="too wide for the rasteriser's int32 edge functions"):
        env.sim.set_fisheye_lut(rx, ry)
    after = _render_twice(env, torch)
    assert np.array_equal(before, after)
    env.check()
    env.close()


@pytest.mark.gpu
def test_lut_of_the_wrong_shape_is_refused(torch_cuda):
    """rmapx and rmapy must be two 2-D arrays of the camera's shape; the library reads H x W floats from each."""
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.lib import DtsError

    W, H = 84, 84
    env = BatchedDuckietownEnv(2, "small_loop", camera_width=W, camera_height=H, domain_rand=False, distortion=True, seed=3)
    rx, ry = make_lut("identity", W, H)
    for a, b in ((rx, ry[:40]), (rx[:, :40], ry), (rx.ravel(), ry.ravel()), (rx[None], ry[None])):
        with pytest.raises(ValueError, match="fisheye LUT"):
            env.sim.set_fisheye_lut(a, b)
    with pytest.raises(DtsError, match="but the camera is"):
        env.sim.set_fisheye_lut(rx[:40, :40], ry[:40, :40])
    env.sim.set_fisheye_lut(rx, ry)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fisheye", [False, True], ids=["plain", "permutation"])
def test_frame_memory_overflow_contract(fisheye, monkeypatch, torch_cuda):
    """A pair pool of exactly one env's bound (DTS_PAIR_POOL_GB tiny) for 64 envs: some frames fit, the rest do not.
    A frame that fits equals the oracle's; one that does not is the clear colour everywhere (black where the LUT gives no
    source), its overflow flag is set, status bit 0 is set and env.check() raises."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.lib import DtsError

    monkeypatch.setenv("DTS_PAIR_POOL_GB", "1e-6")   # read when the frame memory is reserved, at the first render
    name, N, W, H = "small_loop", 64, 160, 120
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 31)
    env = BatchedDuckietownEnv(N, name, camera_width=W, camera_height=H, domain_rand=False, distortion=fisheye, seed=5)
    lut = None
    if fisheye:
        lut = make_lut("permutation", W, H)
        env.sim.set_fisheye_lut(*lut)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    got = env.render_obs().cpu().numpy()
    n_cells = md.grid_w * md.grid_h
    over = np.array([env.sim.debug_frame(k, n_cells)["overflow"] for k in range(N)])
    assert set(over.tolist()) == {0, 1}, f"{int(over.sum())} of {N} frames overflowed: pick N so that both outcomes occur"
    sc = orc.OracleScene(md)
    fit = np.flatnonzero(over == 0)
    ref = sc.render_batch(px[fit], pz[fit], ang[fit], [orc.default_episode() for _ in fit], W, H, False, lut=lut,
                          threads=THREADS)
    mx, n = lsb_diff(got[fit], ref)
    assert mx == 0, f"frames that fit: max diff {mx} LSB on {n} channel values"
    no_source = np.zeros((H, W), bool) if lut is None else (numpy_gather(np.ones((1, H, W, 1), np.uint8), *lut)[0, ..., 0] == 0)
    for k in np.flatnonzero(over == 1):
        h = env.sim.debug_episode(int(k))["horizon"].astype(np.float32)
        clear = np.minimum(np.rint(h * np.float32(255.0)), 255).astype(np.uint8)
        want = np.where(no_source[..., None], np.uint8(0), clear[None, None, :])
        assert np.array_equal(got[k], np.broadcast_to(want, got[k].shape)), \
            f"env {k} overflowed but is not the clear colour: {int((got[k] != want).any(-1).sum())} pixels differ"
    assert env.sim.status() & 1
    with pytest.raises(DtsError):
        env.check()
    env.close()
