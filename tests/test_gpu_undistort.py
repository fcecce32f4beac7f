"""UndistortWrapper (src/gym_duckietown/wrappers.py:145-227) on the device: the rectification gathered by the fused
fisheye kernels through a second table (dts_set_rectify_lut, DTS_RENDER_RECTIFY), the pinhole mode behind
`undistort` (DTS_RENDER_PINHOLE), the wrapper's stacking rules and the single-env adapter.

The bar is the raster oracle's rectified frame (its fused gather under the wrapper's map, which tests/test_undistort.py
holds to cv2.remap of its plain frame), 0 LSB on every channel value; the map itself is pinned by
tests/golden/undistort.npz."""
import numpy as np
import pytest

from test_gpu_fisheye import THREADS, lsb_diff, random_poses

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, name, w, h, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, distortion=True, seed=5)
    args.update(kw)
    return BatchedDuckietownEnv(n, name, **args)


def rect_lut(w, h):
    from gym_duckietown_b200.distortion import rectify_maps
    return rectify_maps(w, h)


def obs_render_twice(env, torch):
    """The reset / step observation of the current state (the env's base render mode), rendered twice."""
    a, b = torch.empty_like(env.obs), torch.empty_like(env.obs)
    env.sim.render(a.data_ptr(), env._stream())
    env.sim.render(b.data_ptr(), env._stream())
    torch.cuda.synchronize()
    assert torch.equal(a, b), "two renders of the same state differ"
    return a.cpu().numpy()


def oracle_frames(md, px, pz, ang, w, h, lut=None, eps=None, domain_rand=False):
    import oracle as orc
    eps = eps or [orc.default_episode() for _ in px]
    return orc.OracleScene(md).render_batch(px, pz, ang, eps, w, h, domain_rand, lut=lut, threads=THREADS)


def device_episodes(env):
    """Oracle episodes holding what the device drew for each env (domain randomisation, device resets)."""
    import oracle as orc
    eps = []
    for k in range(env.num_envs):
        r = env.sim.debug_episode(k)
        eps.append(orc.default_episode(cam_height=float(r["cam_height"]), cam_angle_deg=float(r["cam_angle_deg"]),
                                       cam_fov_y_deg=float(r["cam_fov_y_deg"]), cam_noise=r["cam_noise"],
                                       horizon=r["horizon"], ambient=r["ambient"], diffuse=r["diffuse"],
                                       light_eye=r["light_eye"], ground=r["ground"], hidden=[int(v) for v in r["hidden"]]))
    return eps


def check_u8(got, want, what):
    mx, n = lsb_diff(got, want)
    assert mx == 0, f"{what}: max diff {mx} LSB on {n} channel values"


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
@pytest.mark.parametrize("W,H,fmt", [(640, 480, "hwc_u8"), (160, 120, "hwc_u8"), (84, 84, "hwc_u8"), (90, 70, "hwc_u8"),
                                     (160, 120, "chw_f32")])
def test_rectified_frames_vs_oracle(name, W, H, fmt, torch_cuda):
    """256 random drivable-tile cameras under UndistortWrapper (NormalizeWrapper and ImgWrapper above it for
    chw_f32): the observation equals the oracle's rectified frame and a second render is byte-equal."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps, wrappers as Wr

    md = maps.load_map(name)
    N = 256
    px, pz, ang = random_poses(md, N, 2026)
    env = make_env(N, name, W, H)
    w = Wr.UndistortWrapper(env)
    if fmt == "chw_f32":
        w = Wr.ImgWrapper(Wr.NormalizeWrapper(w))
        assert tuple(w.observation_space.shape) == (3, H, W)
    else:
        assert tuple(w.observation_space.shape) == (H, W, 3)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    got = obs_render_twice(env, torch)
    ref = oracle_frames(md, px, pz, ang, W, H, lut=rect_lut(W, H))
    assert ref.std() > 10
    if fmt == "chw_f32":
        assert np.array_equal(got, (ref.transpose(0, 3, 1, 2) / 255.0).astype(np.float32)), \
            lsb_diff(np.rint(got * 255.0).astype(np.uint8), ref.transpose(0, 3, 1, 2))
    else:
        check_u8(got, ref, f"{name} {W}x{H}")
    env.check()
    env.close()


def test_training_camera_reset_and_auto_reset_steps_vs_oracle(torch_cuda):
    """launch_env()'s camera (udem1, 640x480, distortion) with domain randomisation, 64 envs, device auto-reset: the
    observations of UndistortWrapper(env).reset() and of the steps after it, through episode ends, equal the oracle's
    rectified frames of the same state and episode."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps, wrappers as Wr

    N, W, H = 64, 640, 480
    md = maps.load_map("udem1")
    env = make_env(N, "udem1", W, H, domain_rand=True, seed=50, device_reset=True, auto_reset=True, max_steps=3)
    w = Wr.UndistortWrapper(env)
    lut = rect_lut(W, H)
    rng = np.random.default_rng(6)
    ended = 0
    for t in range(5):
        if t == 0:
            obs = w.reset()
        else:
            acts = torch.from_numpy(rng.uniform(-1, 1, (N, 2)).astype(np.float32)).to(env.device)
            obs, _, done, _ = w.step(acts)
            ended += int(done.sum().item())
        got = obs.cpu().numpy()
        st = {k: v.cpu().numpy() for k, v in env.state.items()}
        ref = oracle_frames(md, st["pos_x"], st["pos_z"], st["angle"], W, H, lut=lut, eps=device_episodes(env),
                            domain_rand=True)
        check_u8(got, ref, f"step {t}")
    assert ended >= N, f"only {ended} episodes ended: the auto-reset path was not exercised"
    env.check()
    env.close()


def test_render_obs_and_undistort_mode_semantics(torch_cuda):
    """Under the wrapper render_obs() and render_obs(segment=True) are the pinhole frames and the observation stays
    rectified; `undistort = True` alone gives pinhole step observations; back to False, the frames are byte-equal to
    those of a fresh distortion=True env."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps, wrappers as Wr

    name, N, W, H = "loop_obstacles", 16, 160, 120
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 77)
    poses = dict(pos_x=px, pos_z=pz, angle=ang)
    sc = orc.OracleScene(md)

    env = make_env(N, name, W, H)
    Wr.UndistortWrapper(env)
    assert env.undistort
    env.sim.reset(None, poses)
    check_u8(env.render_obs().cpu().numpy(), oracle_frames(md, px, pz, ang, W, H), "render_obs()")
    seg = env.render_obs(segment=True).cpu().numpy()
    check_u8(seg, np.stack([sc.render(px[k], pz[k], ang[k], None, W, H, False, segment=True) for k in range(N)]),
             "render_obs(segment=True)")
    check_u8(obs_render_twice(env, torch), oracle_frames(md, px, pz, ang, W, H, lut=rect_lut(W, H)), "observation")
    env.close()

    zero = torch.zeros((N, 2), dtype=torch.float32, device="cuda")
    a, fresh = make_env(N, name, W, H), make_env(N, name, W, H)
    for e in (a, fresh):
        e.sim.reset(None, poses)
    a.undistort = True
    obs = a.step(zero)[0].cpu().numpy()
    st = {k: v.cpu().numpy() for k, v in a.state.items()}
    check_u8(obs, oracle_frames(md, st["pos_x"], st["pos_z"], st["angle"], W, H), "undistort = True step")
    fresh.step(zero)
    a.undistort = False
    got, want = a.step(zero)[0].cpu().numpy(), fresh.step(zero)[0].cpu().numpy()
    assert np.array_equal(got, want), "undistort = False: not the fresh env's frames"
    st = {k: v.cpu().numpy() for k, v in a.state.items()}
    check_u8(got, oracle_frames(md, st["pos_x"], st["pos_z"], st["angle"], W, H,
                                lut=(a.camera_model.rmapx, a.camera_model.rmapy)), "undistort = False step")
    assert np.array_equal(a.render_obs().cpu().numpy(), fresh.render_obs().cpu().numpy())
    a.close(); fresh.close()


def test_rectified_step_launches_as_many_kernels_as_a_fisheye_step(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import wrappers as Wr
    N, W, H = 32, 160, 120
    fish, rect = make_env(N, "udem1", W, H), make_env(N, "udem1", W, H)
    w = Wr.UndistortWrapper(rect)
    counts = []
    for e, stepper in ((fish, fish), (rect, w)):
        e.reset(render=False)
        stepper.step(torch.zeros((N, 2), dtype=torch.float32, device=e.device))
        c0 = e.launch_count()
        stepper.step(torch.zeros((N, 2), dtype=torch.float32, device=e.device))
        counts.append(e.launch_count() - c0)
    assert counts[0] == counts[1], counts
    fish.close(); rect.close()


@pytest.mark.parametrize("W,H,resize", [(160, 120, "cv2_84x84"), (640, 480, "pil_160x120")])
def test_resize_above_undistort(W, H, resize, torch_cuda):
    """ResizeWrapper(UndistortWrapper(env)) (cv2's and the learning scripts' Pillow filter): the observation is the
    resize pass applied to the wrapper's full-size rectified frames."""
    torch = torch_cuda
    from gym_duckietown_b200 import learning_wrappers as LW, maps, wrappers as Wr
    name, N = "udem1", 8
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 5)
    full_env, rz_env = make_env(N, name, W, H), make_env(N, name, W, H)
    full = Wr.UndistortWrapper(full_env)
    rz = Wr.ResizeWrapper(Wr.UndistortWrapper(rz_env), resize_w=84, resize_h=84) if resize.startswith("cv2") else \
        LW.ResizeWrapper(Wr.UndistortWrapper(rz_env), shape=(120, 160, 3))
    zero = torch.zeros((N, 2), dtype=torch.float32, device="cuda")
    for e in (full_env, rz_env):
        e.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    frames = full.step(zero)[0].clone()
    got = rz.step(zero)[0].cpu().numpy().copy()
    st = {k: v.cpu().numpy() for k, v in full_env.state.items()}
    check_u8(frames.cpu().numpy(), oracle_frames(md, st["pos_x"], st["pos_z"], st["angle"], W, H, lut=rect_lut(W, H)),
             "full-size rectified frames")
    want = rz_env.sim_resize_only(frames).cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got, want)
    full_env.close(); rz_env.close()


def test_batch_scale_vs_oracle(torch_cuda):
    """2048 cameras at 160x120: the rectification's source boxes fit the batch's pair pool (env.check() clean) and
    every frame equals the oracle's."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps, wrappers as Wr
    name, N, W, H = "loop_obstacles", 2048, 160, 120
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 2027)
    env = make_env(N, name, W, H)
    Wr.UndistortWrapper(env)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    got = obs_render_twice(env, torch)
    env.check()
    check_u8(got, oracle_frames(md, px, pz, ang, W, H, lut=rect_lut(W, H)), "2048 cameras")
    env.close()


def test_single_env_adapter(torch_cuda):
    """Simulator(distortion=True) with `undistort = True` returns pinhole frames (what the reference's own
    UndistortWrapper then remaps on the host); cv2.remap of them equals the fused wrapper's observation."""
    import cv2
    from gym_duckietown_b200 import wrappers as Wr
    from gym_duckietown_b200.simulator import Simulator
    W, H = 160, 120
    kw = dict(map_name="udem1", camera_width=W, camera_height=H, domain_rand=False, seed=12)
    host, fused, pinhole = Simulator(distortion=True, **kw), Wr.UndistortWrapper(Simulator(distortion=True, **kw)), \
        Simulator(distortion=False, **kw)
    host.undistort = True
    assert host.undistort and host._b.undistort and fused.unwrapped.undistort
    mx, my = rect_lut(W, H)
    a = np.array([0.4, 0.2], np.float32)
    for t in range(3):
        if t == 0:
            o_host, o_fused, o_pin = host.reset(), fused.reset(), pinhole.reset()
        else:
            o_host, o_fused, o_pin = host.step(a)[0], fused.step(a)[0], pinhole.step(a)[0]
        assert isinstance(o_fused, np.ndarray) and o_fused.shape == (H, W, 3) and o_fused.dtype == np.uint8
        assert np.array_equal(o_host, o_pin), t
        assert np.array_equal(cv2.remap(o_host, mx, my, cv2.INTER_NEAREST), o_fused), t
        assert o_fused.std() > 10
    for s in (host, fused, pinhole):
        s.close()


def test_refusals(torch_cuda):
    from gym_duckietown_b200 import learning_wrappers as LW, wrappers as Wr
    W, H = 84, 84
    with pytest.raises(AssertionError, match="Distortion is false, no need for this wrapper"):
        Wr.UndistortWrapper(make_env(2, "small_loop", W, H, distortion=False))
    for below in (lambda e: Wr.ResizeWrapper(e, 40, 40), lambda e: LW.ResizeWrapper(e, shape=(42, 42, 3)),
                  Wr.ImgWrapper, Wr.PyTorchObsWrapper):
        env = make_env(2, "small_loop", W, H)
        with pytest.raises(ValueError):
            Wr.UndistortWrapper(below(env))
        assert not env.undistort and env.rectification is None
        env.close()
    env = make_env(2, "small_loop", W, H)
    with pytest.raises(ValueError, match="MotionBlurWrapper"):
        Wr.UndistortWrapper(Wr.MotionBlurWrapper(env))
    assert not env.undistort
    env.close()
    env = make_env(2, "small_loop", W, H)
    with pytest.raises(ValueError, match="MotionBlurWrapper"):
        Wr.MotionBlurWrapper(Wr.UndistortWrapper(env))
    env.close()


def test_rectify_lut_refusals_keep_the_previous_table(torch_cuda):
    """A table too wide for the int32 edge functions or of the wrong shape is refused and the one set before stays in
    effect; a handle without DTS_FLAG_DISTORTION refuses any; a cleared table fails DTS_RENDER_RECTIFY renders."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps, wrappers as Wr
    from gym_duckietown_b200.lib import DtsError
    from test_gpu_fisheye import make_lut

    name, N, W, H = "udem1", 8, 640, 480
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 3)
    env = make_env(N, name, W, H)
    Wr.UndistortWrapper(env)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    before = obs_render_twice(env, torch)
    check_u8(before, oracle_frames(md, px, pz, ang, W, H, lut=rect_lut(W, H)), "rectified")
    rx, ry = make_lut("identity", W, H)
    rx[0:8, 0:16], ry[0:8, 0:16] = 0, 0
    rx[0:8, 16:32], ry[0:8, 16:32] = W - 1, H - 1
    with pytest.raises(DtsError, match="too wide for the rasteriser's int32 edge functions"):
        env.set_rectification(rx, ry)
    mx, my = rect_lut(W, H)
    for a, b in ((mx, my[:40]), (mx.ravel(), my.ravel())):
        with pytest.raises(ValueError, match="rectification LUT"):
            env.set_rectification(a, b)
    with pytest.raises(DtsError, match="but the camera is"):
        env.set_rectification(mx[:40, :40], my[:40, :40])
    assert np.array_equal(obs_render_twice(env, torch), before)
    env.sim.set_rectify_lut(None, None)
    with pytest.raises(DtsError, match="no rectification LUT"):
        env.sim.render(env.obs.data_ptr(), env._stream())
    env.set_rectification(None, None)     # undistort alone: pinhole observations
    check_u8(obs_render_twice(env, torch), oracle_frames(md, px, pz, ang, W, H), "pinhole after clearing")
    env.check()
    env.close()
    plain = make_env(2, name, 160, 120, distortion=False)
    with pytest.raises(DtsError, match="DTS_FLAG_DISTORTION"):
        plain.sim.set_rectify_lut(*rect_lut(160, 120))
    plain.close()
