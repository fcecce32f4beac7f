"""Wrapper fusion (SURVEY 8f-3): the reference's observation / reward / action wrappers emitted directly by the
step kernels (dts_set_output_format) must equal the wrapper's numpy semantics applied to the plain outputs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(name, n, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=160, camera_height=120, domain_rand=False, seed=1000)
    args.update(kw)
    return BatchedDuckietownEnv(n, name, **args)


@pytest.mark.parametrize("size,distortion", [((160, 120), False), ((84, 84), False), ((100, 76), False), ((160, 120), True),
                                           ((101, 75), False), ((160, 120), "camera_rand_pool"), ((160, 120), "rectified")])
def test_observation_layouts_and_normalisation(size, distortion, torch_cuda):
    """ImgWrapper transpose(2,0,1) LW:86, PyTorchObsWrapper transpose(2,1,0) W:110, NormalizeWrapper obs/255 LW:66-70.
    101x75: a width that is no multiple of 4; also a camera_rand pool of four fisheye tables and the rectification."""
    torch = torch_cuda
    W, H = size
    kw = dict(distortion=bool(distortion))
    if distortion == "camera_rand_pool":
        kw.update(camera_rand=True, camera_rand_pool=4)
    env = make_env("udem1", 12, camera_width=W, camera_height=H, domain_rand=True, **kw)
    if distortion == "rectified":
        from gym_duckietown_b200.distortion import rectify_maps
        env.set_rectification(*rectify_maps(W, H))
        env.undistort = True

    def render():   # in the env's own render mode (under undistort render_obs() would draw the pinhole frame)
        env.sim.render(env.obs.data_ptr(), env._stream())
        return env.obs.cpu().numpy()
    env.reset(render=False)
    base = render().copy()                                # u8 [N,H,W,3]
    assert base.std() > 10
    for layout, perm in (("hwc", (0, 1, 2)), ("chw", (2, 0, 1)), ("cwh", (2, 1, 0))):
        for dtype in ("uint8", "float32"):
            env.set_output_format(obs_layout=layout, obs_dtype=dtype)
            got = render()
            want = np.stack([f.transpose(perm) for f in base])
            if dtype == "float32":
                ref64 = want / 255.0                         # what NormalizeWrapper computes (float64)
                assert got.dtype == np.float32 and np.array_equal(got, ref64.astype(np.float32))
            else:
                assert got.dtype == np.uint8 and np.array_equal(got, want)
    # and through step(): the obs of the step is already in the wrapper format
    env.set_output_format(obs_layout="chw", obs_dtype="float32")
    acts = torch.zeros(12, 2, device=env.device)
    obs, *_ = env.step(acts)
    env.set_output_format(obs_layout="hwc", obs_dtype="uint8")
    plain = render()
    assert np.array_equal(obs.cpu().numpy(), (plain.transpose(0, 3, 1, 2) / 255.0).astype(np.float32))
    env.close()


def test_wrapper_classes_configure_the_fused_path(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import wrappers as Wr
    env = make_env("small_loop", 8)
    w = Wr.DtRewardWrapper(Wr.ActionWrapper(Wr.ImgWrapper(Wr.NormalizeWrapper(env))))
    assert w.unwrapped is env
    assert env.output_format == dict(obs_layout="chw", obs_dtype="float32", reward="dt", discrete_actions=False,
                                     action_vel_scale=0.8)
    sp = w.observation_space
    assert tuple(sp.shape) == (3, 120, 160) and sp.dtype == np.float32
    w.reset()
    obs, rew, done, info = w.step(torch.full((8, 2), 0.3, device=env.device))
    assert obs.shape == (8, 3, 120, 160) and obs.dtype == torch.float32 and 0.0 <= float(obs.min()) and float(obs.max()) <= 1.0
    assert tuple(Wr.PyTorchObsWrapper(make_env("small_loop", 2)).observation_space.shape) == (3, 160, 120)
    rz = Wr.ResizeWrapper(Wr.PyTorchObsWrapper(make_env("small_loop", 2)), resize_w=84, resize_h=84)
    assert tuple(rz.observation_space.shape) == (3, 84, 84)
    obs = rz.reset()
    assert tuple(obs.shape) == (2, 3, 84, 84) and obs.dtype == torch.uint8 and float(obs.float().std()) > 5
    env.close()


@pytest.mark.parametrize("mode", ["discrete", "scaled"])
def test_action_and_reward_wrappers_vs_oracle(mode, torch_cuda):
    """DiscreteWrapper W:18-30 / ActionWrapper LW:110-112 feed DuckietownEnv.step with float64 [vel, steering];
    DtRewardWrapper LW:94-102 maps the reward.  The oracle env is driven with those float64 actions."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps, wrappers as Wr
    N, T = 32, 80
    env = make_env("loop_obstacles", N)
    env.reset(render=False)
    torch.cuda.synchronize()
    st0 = {k: v.cpu().numpy().copy() for k, v in env.state.items()}
    om = orc.OracleMap(maps.load_map("loop_obstacles"))
    cpu = [orc.OracleEnv(om, st0["pos_x"][k], st0["pos_z"][k], st0["angle"][k]) for k in range(N)]
    rng = np.random.default_rng(11)
    w = Wr.DtRewardWrapper(Wr.DiscreteWrapper(env) if mode == "discrete" else Wr.ActionWrapper(env))
    table = {0: (0.6, 1.0), 1: (0.6, -1.0), 2: (0.7, 0.0)}
    seen = set()
    for t in range(T):
        if mode == "discrete":
            ids = rng.integers(0, 3, N)
            _, rew, done, info = w.step(torch.from_numpy(ids).to(env.device), render=False)
            acts = [table[int(i)] for i in ids]
        else:
            a32 = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
            _, rew, done, info = w.step(torch.from_numpy(a32).to(env.device), render=False)
            acts = [(float(a[0]) * 0.8, float(a[1])) for a in a32]
        s = {k: v.cpu().numpy() for k, v in info.items()}
        r32 = rew.cpu().numpy()
        for k in range(N):
            o = cpu[k].step(acts[k])
            assert abs(s["pos_x"][k] - o.pos_x) <= 1e-9 and abs(s["pos_z"][k] - o.pos_z) <= 1e-9, (t, k)
            assert s["done_code"][k] == o.done_code, (t, k)
            want = -10.0 if o.reward == -1000 else (o.reward + 10 if o.reward > 0 else o.reward + 4)
            seen.add(0 if o.reward == -1000 else (1 if o.reward > 0 else 2))
            assert abs(r32[k] - want) <= 1e-5 * max(1.0, abs(want)), (t, k)
            assert abs(s["reward"][k] - o.reward) <= 1e-9 * max(1.0, abs(o.reward))     # the state keeps the raw reward
    assert seen == {0, 1, 2}
    env.close()


def test_motion_blur_wrapper_equals_numpy_average_of_the_substep_frames(torch_cuda):
    """MotionBlurWrapper LW:8-54: three update_physics(action) at delta_time / 3 with a render before each and one after,
    np.average(window, axis=0, weights=[0.8, 0.15, 0.04, 0.01]) in float64; reward / done of the final state."""
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L, wrappers as Wr
    N = 6
    a = make_env("loop_obstacles", N, action_mode="pwm")
    b = make_env("loop_obstacles", N, action_mode="pwm")
    a.reset(); b.reset()
    w = Wr.MotionBlurWrapper(a)
    b.sim.set_timing((1.0 / 30) / 3, 1, L.ACTION_PWM)
    assert w.observation_space.dtype == np.float64
    rng = np.random.default_rng(3)
    for t in range(4):
        act = torch.from_numpy(rng.uniform(-1, 1, (N, 2)).astype(np.float32)).to(a.device)
        blurred, rew, done, info = w.step(act)
        window = []
        for k in range(3):
            window.append(b.render_obs().cpu().numpy().copy())
            _, rew_b, done_b, _ = b.step(act, render=False)
        window.append(b.render_obs().cpu().numpy().copy())
        want = np.average(window, axis=0, weights=[0.8, 0.15, 0.04, 0.01])
        got = blurred.cpu().numpy()
        assert got.dtype == np.float64 and np.array_equal(got, want), float(np.abs(got - want).max())
        assert torch.equal(rew, rew_b) and torch.equal(done, done_b)
        assert int(a.state["step_count"][0]) == 3 * (t + 1)
    a.close(); b.close()
