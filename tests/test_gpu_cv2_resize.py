"""The device pass of src/gym_duckietown/wrappers.py's ResizeWrapper (dts_set_resize: cv2 INTER_CUBIC in 8-bit fixed
point) against the integer restatement oracle/cv2_cubic.py at 0 LSB, in every layout and dtype, through the tiled
k_resize_band and, under DTS_RESIZE_UNTILED=1, the untiled k_resize.  The sweep's shapes and which branch each one
takes are in test_cv2_resize.py."""
import numpy as np
import pytest

import cv2_cubic as C
from test_cv2_resize import SWEEP, SWEEP_IDS, sweep_frames

pytestmark = pytest.mark.gpu

LAYOUTS = {"hwc": (0, 1, 2, 3), "chw": (0, 3, 1, 2), "cwh": (0, 3, 2, 1)}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(params=[False, True], ids=["tiled", "untiled"])
def untiled(request, monkeypatch):
    """The plan is made by set_resize: the variable must be in place before it and stay until the env is closed."""
    if request.param:
        monkeypatch.setenv("DTS_RESIZE_UNTILED", "1")
    else:
        monkeypatch.delenv("DTS_RESIZE_UNTILED", raising=False)
    return request.param


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


@pytest.mark.parametrize("cam,target,rows", SWEEP, ids=SWEEP_IDS)
def test_device_resize_equals_the_restatement(cam, target, rows, untiled, torch_cuda):
    torch = torch_cuda
    (w, h), (ow, oh) = cam, target
    frames = sweep_frames(6, w, h, 21)
    env = make_env(6, w, h)
    env.reset(render=False)
    env.set_resize(ow, oh)
    assert env.resize == (ow, oh) and env.resize_method == "cv2_cubic"
    check_all_formats(env, torch.from_numpy(frames).to(env.device), C.resize(frames, ow, oh))
    env.close()


def plain_frames(b, ow, oh):
    """render_obs() of the current state at the camera's size, with the resize switched off (then on again)."""
    b.set_resize(None, None)
    plain = b.render_obs().cpu().numpy().copy()
    b.set_resize(ow, oh)
    return plain


def test_rendered_steps_under_resize_wrapper_equal_the_restatement(untiled, torch_cuda):
    """The c2 benchmark's shape: 256 envs of small_loop at 160x120 under ResizeWrapper(84, 84).  Each step's
    observation is the restatement of that step's full-size render.  Untiled, 256 x 84 x 84 pixels are more than
    k_resize's grid, so its grid-stride loop runs more than once per thread."""
    torch = torch_cuda
    from gym_duckietown_b200 import wrappers as Wr
    N = 256
    b = make_env(N, 160, 120)
    env = Wr.ResizeWrapper(b, resize_w=84, resize_h=84)
    obs = env.reset()
    assert tuple(obs.shape) == (N, 84, 84, 3) and obs.dtype == torch.uint8
    rng = np.random.default_rng(6)
    for t in range(3):
        acts = torch.from_numpy(rng.uniform(-1, 1, (N, 2)).astype(np.float32)).to(b.device)
        obs, _, _, _ = env.step(acts)
        got = obs.cpu().numpy().copy()
        plain = plain_frames(b, 84, 84)
        assert plain.std() > 10
        want = C.resize(plain, 84, 84)
        d = np.abs(got.astype(int) - want.astype(int))
        assert d.max() == 0, (t, int(d.max()), float((d > 0).mean()))
    b.close()
