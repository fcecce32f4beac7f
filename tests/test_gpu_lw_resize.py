"""The device pass of learning/utils/wrappers.py's ResizeWrapper (dts_set_resize_filter(DTS_RESIZE_PIL_BILINEAR),
Pillow's bilinear in 8-bit fixed point) and the reference training scripts' wrapper stack built on it:
0 LSB against the reference class's output (tests/golden/lw_resize.npz) and against the numpy restatement
(oracle/pil_resize.py) at other shapes, in every layout and dtype."""
import os

import numpy as np
import pytest

import pil_resize as P

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "lw_resize.npz")
LAYOUTS = {"hwc": (0, 1, 2, 3), "chw": (0, 3, 1, 2), "cwh": (0, 3, 2, 1)}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, w, h, name="small_loop", **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, seed=1)
    args.update(kw)
    return BatchedDuckietownEnv(n, name, **args)


def check_all_formats(env, src, want_hwc):
    """sim_resize_only(src) in the three layouts, u8 and float32, against want_hwc u8 [N][h][w][3]."""
    for layout, perm in LAYOUTS.items():
        want = want_hwc.transpose(perm)
        for dtype in ("uint8", "float32"):
            env.set_output_format(obs_layout=layout, obs_dtype=dtype)
            got = env.sim_resize_only(src).cpu().numpy()
            if dtype == "float32":
                assert got.dtype == np.float32 and np.array_equal(got, (want / 255.0).astype(np.float32)), (layout, dtype)
            else:
                d = np.abs(got.astype(int) - want.astype(int))
                assert got.dtype == np.uint8 and d.max() == 0, (layout, dtype, int(d.max()), float((d > 0).mean()))
    env.set_output_format(obs_layout="hwc", obs_dtype="uint8")


def golden_frames(g, tag, shape, frames):
    """What the reference class returned for `frames`: stored whole for small targets; for the others only its
    digest is stored, which the restatement's output must match before it stands in for it."""
    key = P.golden_key(tag, shape)
    if key in g.files:
        return g[key]
    want = P.resize(frames, shape[1], shape[0])
    assert P.sha(want) == str(g[key + "_sha"]), key
    return want


@pytest.mark.parametrize("tag", list(P.SOURCES))
def test_device_pass_equals_the_reference_resize_wrapper(tag, torch_cuda):
    torch = torch_cuda
    g = np.load(GOLD)
    w, h = map(int, tag.split("x"))
    frames = P.canned_frames(int(g["seed"]), w, h)
    env = make_env(3, w, h)
    env.reset(render=False)
    src = torch.from_numpy(frames).to(env.device)
    for shape in P.SOURCES[tag]:
        env.set_resize(shape[1], shape[0], method="pil_bilinear")
        assert env.resize == (shape[1], shape[0]) and env.resize_method == "pil_bilinear"
        check_all_formats(env, src, golden_frames(g, tag, shape, frames))
    env.close()


# (camera w, h) -> (target w, h): the training size, the largest permitted reduction (1/32 per axis: 65 taps),
# widths whose rows are not whole words (non-word stores), cameras whose rows are not whole 4-pixel groups (byte
# staging), one-axis changes, an identity and upscales
SWEEP = [((640, 480), (160, 120)), ((640, 480), (20, 15)), ((800, 600), (25, 19)), ((640, 480), (84, 84)),
         ((100, 76), (41, 30)), ((162, 121), (53, 40)), ((98, 50), (37, 50)), ((160, 120), (160, 37)),
         ((84, 84), (84, 84)), ((160, 120), (320, 240)), ((33, 17), (101, 7))]


@pytest.mark.parametrize("cam,target", SWEEP)
def test_device_pass_equals_the_restatement_on_random_frames(cam, target, torch_cuda):
    torch = torch_cuda
    (w, h), (ow, oh) = cam, target
    rng = np.random.default_rng(w * 1000 + ow)
    frames = rng.integers(0, 256, (5, h, w, 3), dtype=np.uint8)
    frames[1, : h // 2] = 255
    frames[1, :, : w // 3] = 0
    env = make_env(5, w, h)
    env.reset(render=False)
    env.set_resize(ow, oh, method="pil_bilinear")
    check_all_formats(env, torch.from_numpy(frames).to(env.device), P.resize(frames, ow, oh))
    env.close()


def test_a_target_beyond_the_tap_bound_is_refused_and_the_previous_setting_stays(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    env = make_env(2, 640, 480)
    env.reset(render=False)
    env.set_resize(160, 120, method="pil_bilinear")
    with pytest.raises(L.DtsError, match="taps"):
        env.set_resize(19, 15, method="pil_bilinear")        # 640 / 19 > 32: 69 taps per output column
    with pytest.raises(ValueError):
        env.set_resize(80, 60, method="lanczos")
    assert env.resize == (160, 120) and env.resize_method == "pil_bilinear" and tuple(env.obs.shape) == (2, 120, 160, 3)
    frames = np.random.default_rng(2).integers(0, 256, (2, 480, 640, 3), dtype=np.uint8)
    got = env.sim_resize_only(torch.from_numpy(frames).to(env.device)).cpu().numpy()
    assert np.array_equal(got, P.resize(frames, 160, 120))
    env.close()


def lw_stack(env, shape=(120, 160, 3)):
    from gym_duckietown_b200 import learning_wrappers as LW
    return LW.DtRewardWrapper(LW.ActionWrapper(LW.ImgWrapper(LW.NormalizeWrapper(LW.ResizeWrapper(env, shape=shape)))))


def plain_frames(b):
    """render_obs() of the current state without the stack's format: full-size u8 HWC."""
    b.set_resize(None, None)
    b.set_output_format(obs_layout="hwc", obs_dtype="uint8")
    plain = b.render_obs().cpu().numpy().copy()
    b.set_output_format(obs_layout="chw", obs_dtype="float32")
    b.set_resize(160, 120, method="pil_bilinear")
    return plain


@pytest.mark.parametrize("name,domain_rand", [("udem1", False), ("udem1", True), ("loop_obstacles", False)])
def test_training_stack_on_the_launch_env_camera(name, domain_rand, torch_cuda):
    """learning/utils/env.py's launch_env (640x480, distortion on) under the stack the reference training scripts
    build: every step's obs is the restatement of the plain render, normalised and transposed, at 0 LSB."""
    torch = torch_cuda
    N = 8
    b = make_env(N, 640, 480, name, distortion=True, domain_rand=domain_rand, seed=31)
    env = lw_stack(b)
    sp = env.observation_space
    assert tuple(sp.shape) == (3, 120, 160) and sp.dtype == np.float32
    assert b.output_format["obs_layout"] == "chw" and b.output_format["obs_dtype"] == "float32"
    env.reset()
    rng = np.random.default_rng(4)
    for t in range(3):
        acts = torch.from_numpy(rng.uniform(-1, 1, (N, 2)).astype(np.float32)).to(b.device)
        obs, rew, done, info = env.step(acts)
        assert tuple(obs.shape) == (N, 3, 120, 160) and obs.dtype == torch.float32
        got = obs.cpu().numpy().copy()
        plain = plain_frames(b)
        assert plain.std() > 10
        want = (P.resize(plain, 160, 120).transpose(0, 3, 1, 2) / 255.0).astype(np.float32)
        assert np.array_equal(got, want), (t, float(np.abs(got - want).max()))
    b.close()


def test_training_stack_on_the_single_env_adapter_matches_env_0(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200.simulator import DuckietownEnv
    kw = dict(camera_width=640, camera_height=480, distortion=True, domain_rand=False, seed=12)
    single = lw_stack(DuckietownEnv(map_name="udem1", **kw))
    b = make_env(3, 640, 480, "udem1", **kw)
    b.reset(render=False)                 # the adapter resets once on construction
    batched = lw_stack(b)
    assert tuple(single.observation_space.shape) == (3, 120, 160)
    o1, ob = single.reset(), batched.reset()
    assert isinstance(o1, np.ndarray) and o1.shape == (3, 120, 160) and o1.dtype == np.float32
    assert np.array_equal(o1, ob[0].cpu().numpy())
    a = np.array([0.4, 0.2], np.float32)
    o1, r1, d1, _ = single.step(a)
    ob, rb, db, _ = batched.step(torch.from_numpy(np.tile(a, (3, 1))).to(b.device))
    assert np.array_equal(o1, ob[0].cpu().numpy()) and o1.std() > 0.02
    single.close()
    b.close()


def test_resize_wrapper_refuses_a_second_resize_and_a_non_rgb_shape(torch_cuda):
    from gym_duckietown_b200 import learning_wrappers as LW, wrappers as Wr
    env = make_env(2, 160, 120)
    with pytest.raises(ValueError):
        LW.ResizeWrapper(env, shape=(60, 80, 1))
    assert env.resize is None
    LW.ResizeWrapper(env, shape=(60, 80, 3))
    with pytest.raises(ValueError, match="resize"):
        LW.ResizeWrapper(env, shape=(30, 40, 3))
    assert env.resize == (80, 60)
    env.close()
    assert LW.NormalizeWrapper is Wr.NormalizeWrapper and LW.MotionBlurWrapper is Wr.MotionBlurWrapper


def test_cv2_resize_wrapper_unchanged_after_the_pillow_filter_was_used(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import wrappers as Wr
    frames = np.random.default_rng(8).integers(0, 256, (3, 120, 160, 3), dtype=np.uint8)
    a, b = make_env(3, 160, 120), make_env(3, 160, 120)
    for e in (a, b):
        e.reset(render=False)
    src = torch.from_numpy(frames).to(a.device)
    Wr.ResizeWrapper(a, resize_w=84, resize_h=84)
    want = a.sim_resize_only(src).cpu().numpy().copy()
    b.set_resize(84, 84, method="pil_bilinear")
    pil = b.sim_resize_only(src).cpu().numpy().copy()
    assert np.array_equal(pil, P.resize(frames, 84, 84)) and not np.array_equal(pil, want)
    b.set_resize(None, None)
    Wr.ResizeWrapper(b, resize_w=84, resize_h=84)
    assert b.resize_method == "cv2_cubic"
    assert np.array_equal(b.sim_resize_only(src).cpu().numpy(), want)
    a.close(); b.close()
