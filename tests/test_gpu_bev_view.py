"""The bird's-eye grid's camera visibility on the device (dts_set_bev_visibility_target, DESIGN.md section 5 item 15)
against the float64 oracle (tests/bev_view_oracle.py), fed with the device's own cameras (frame_cameras()) and label
images: every cell takes one of the oracle's answers, and its pixel lies within one float32 ulp of the oracle's q
(pinhole) or 2^-10 px (fisheye).  Over 30-step rollouts with random actions and domain randomisation on every map,
pinhole, fisheye, a camera_rand pool, undistort, top-down and segment views, a two-map batch, a grid coarser than a
tile and a 1 x 1 grid.  Also: the lifecycle (unrendered steps, render_bev, repeats, auto-reset with terminal frames,
loads, the rectification), frame_cameras() against dts_debug_frame, refused calls, that the feature changes no other
output, its launches, and the forward maps it shares with flow."""
import numpy as np
import pytest

import bev_view_oracle as vo
from test_gpu_bev import config_of, expected, scene
from test_gpu_depth import poses_of
from test_gpu_flow import MAPS, model_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, names, w=96, h=72, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=True, seed=11, bev_visibility=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def host(env):
    import torch
    torch.cuda.synchronize()
    return env.bev_visibility.cpu().numpy().copy(), env.bev_pixels.cpu().numpy().copy()


def actions(torch, rng, n, device):
    return torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=device)


def check(env, what, fisheye=None):
    """Every env's cells against the oracle for its current state and last frame; returns the count of each value"""
    V, P = (t.cpu().numpy() for t in env.frame_cameras())
    want = expected(env)
    vis, pix = host(env)
    lab = env.labels.cpu().numpy()
    px, pz, ang = poses_of(env)
    mid = env.state["map_id"].cpu().numpy()
    fish = env.distortion and not env.undistort if fisheye is None else fisheye
    seen = np.zeros(4, np.int64)
    amb = 0
    for e in range(env.num_envs):
        md = env.maps[int(mid[e])]
        m = model_of(env, e) if fish else None
        r = vo.visibility(scene(md), (px[e], pz[e], ang[e]), config_of(env), want[e], V[e].ravel(), P[e], lab[e],
                          (m.mapx, m.mapy) if fish else None)
        where = f"{what} env {e}"
        ok = ((r["allowed"] >> vis[e]) & 1) == 1
        assert ok.all(), f"{where}: {np.argwhere(~ok)[:5]} device {vis[e][~ok][:5]} oracle {r['value'][~ok][:5]}"
        has = (vis[e] == vo.VISIBLE) | (vis[e] == vo.OCCLUDED)
        nan = np.isnan(pix[e])
        assert np.array_equal(nan[..., 0], ~has) and np.array_equal(nan[..., 1], ~has), f"{where}: NaN pattern"
        cmp = has & ~r["ambiguous"]
        q, d = r["q"][cmp], pix[e][cmp].astype(np.float64)
        bar = 2.0 ** -10 if fish else np.spacing(np.abs(q).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(q)
        err = np.abs(d - q)
        assert (err <= bar).all(), f"{where}: pixel off by {err.max():.3g} px"
        seen += np.bincount(vis[e].ravel(), minlength=4)
        amb += int(r["ambiguous"].sum())
    return seen, amb


CASES = [(m, "pinhole") for m in MAPS] + [
    ("udem1", "fisheye"), ("loop_dyn_duckiebots", "fisheye"), ("loop_pedestrians", "camera_rand"),
    ("udem1", "undistort"), ("loop_dyn_duckiebots", "top_down"), ("udem1", "segment"),
    (("small_loop", "loop_dyn_duckiebots"), "pinhole"), ("udem1", "coarse"), ("loop_obstacles", "one_cell")]


@pytest.mark.parametrize("names,view", CASES)
def test_rollout_against_the_oracle(torch_cuda, names, view):
    torch = torch_cuda
    n = 4
    kw = dict(distortion=view in ("fisheye", "camera_rand", "undistort"), camera_rand=view == "camera_rand")
    if view == "camera_rand":
        kw["camera_rand_pool"] = 4
    if view == "coarse":
        kw.update(bev_shape=(6, 6), bev_cell=0.8, bev_origin=(3.0, 4.0))
    if view == "one_cell":
        kw.update(bev_shape=(1, 1), bev_cell=0.1, bev_origin=(0.5, 4.0))
    if isinstance(names, tuple):
        kw["cycle_maps"] = True
    env = make_env(n, names, **kw)
    if view == "undistort":
        env.undistort = True
    if isinstance(names, tuple):
        env.reset()
    env.reset()
    mode = dict(top_down=view == "top_down", segment=view == "segment")
    step_renders = not (mode["top_down"] or mode["segment"])
    rng = np.random.default_rng(4)
    seen = np.zeros(4, np.int64)
    amb = 0
    for k in range(30):
        if step_renders:
            env.step(actions(torch, rng, n, env.device))
        else:
            env.step(actions(torch, rng, n, env.device), render=False)
            env.render_obs(**mode)
        s, a = check(env, f"{names} {view} step {k}")
        seen, amb = seen + s, amb + a
    assert seen[vo.UNKNOWN] == 0
    if view != "one_cell":
        assert seen[vo.VISIBLE] > 0 and (seen[vo.OUTSIDE] > 0 or view == "top_down"), seen   # (top-down: all in view)
    assert amb <= 1e-3 * seen.sum() + 1, (amb, seen)


def test_unrendered_steps_and_render_bev_are_unknown(torch_cuda):
    torch = torch_cuda
    n = 4
    env = make_env(n, "udem1")
    env.reset()
    rng = np.random.default_rng(3)
    env.step(actions(torch, rng, n, env.device))
    assert (host(env)[0] == vo.VISIBLE).any()
    env.step(actions(torch, rng, n, env.device), render=False)
    vis, pix = host(env)
    assert (vis == vo.UNKNOWN).all() and np.isnan(pix).all()
    env.render_obs()
    assert (host(env)[0] == vo.VISIBLE).any()
    env.render_bev()
    vis, pix = host(env)
    assert (vis == vo.UNKNOWN).all() and np.isnan(pix).all()


def test_render_obs_repeats_the_step(torch_cuda):
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_pedestrians", distortion=True)
    env.reset()
    rng = np.random.default_rng(6)
    for k in range(4):
        env.step(actions(torch, rng, n, env.device))
        vis, pix = host(env)
        env.render_obs()
        v2, p2 = host(env)
        assert np.array_equal(vis, v2) and np.array_equal(pix.view(np.uint32), p2.view(np.uint32))


def test_auto_reset_rows_match_their_obs_rows(torch_cuda):
    """Ended envs are checked against their respawned first frame, the others against the step's frame"""
    torch = torch_cuda
    n = 16
    env = make_env(n, "small_loop", auto_reset=True, device_reset=True, max_steps=5, terminal_obs=True)
    env.reset()
    rng = np.random.default_rng(2)
    respawned = 0
    for k in range(12):
        ep0 = env.state["episode"].cpu().numpy().copy()
        env.step(actions(torch, rng, n, env.device))
        respawned += int((env.state["episode"].cpu().numpy() != ep0).sum())
        check(env, f"auto-reset step {k}")
    assert respawned > 0


@pytest.mark.parametrize("how", ["load_state", "copy_envs"])
def test_loads_then_render_obs(torch_cuda, how):
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_dyn_duckiebots")
    env.reset()
    rng = np.random.default_rng(9)
    recs = env.save_state()
    for k in range(5):
        env.step(actions(torch, rng, n, env.device))
    if how == "load_state":
        env.load_state(recs)
    else:
        env.copy_envs([3, 2, 1, 0])
    env.render_obs()
    check(env, how)


def test_rectified_render_is_unknown_and_python_refuses_it(torch_cuda):
    from gym_duckietown_b200.distortion import rectify_maps
    torch = torch_cuda
    n = 2
    env = make_env(n, "small_loop", distortion=True)
    m = env.camera_model
    with pytest.raises(ValueError):
        env.set_rectification(m.mapx, m.mapy)
    env.reset()
    env.step(torch.full((n, 2), 0.5, dtype=torch.float32, device=env.device))
    assert (host(env)[0] == vo.VISIBLE).any()
    rx, ry = rectify_maps(env.camera_width, env.camera_height)
    env.sim.set_rectify_lut(rx, ry)
    env.sim.set_render_mode(rectify=True)
    env.render_obs()
    vis, pix = host(env)
    assert (vis == vo.UNKNOWN).all() and np.isnan(pix).all()


def test_frame_cameras_equal_debug_frame(torch_cuda):
    torch = torch_cuda
    n = 6
    rng = np.random.default_rng(1)
    for kw, mode in ((dict(), {}), (dict(distortion=True), {}), (dict(distortion=True, camera_rand=True,
                                                                       camera_rand_pool=3), {}),
                     (dict(), dict(top_down=True)),
                     (dict(auto_reset=True, device_reset=True, max_steps=3, terminal_obs=True), {})):
        env = make_env(n, "loop_obstacles", **kw)
        env.reset()
        for k in range(4):
            env.step(actions(torch, rng, n, env.device))
            if mode:
                env.render_obs(**mode)
            V, P = (t.cpu().numpy() for t in env.frame_cameras())
            assert V.shape == (n, 3, 4) and V.dtype == np.float64 and P.shape == (n, 4) and P.dtype == np.float32
            for e in range(n):
                d = env.sim.debug_frame(e, 0)
                assert np.array_equal(V[e].ravel().view(np.uint64), d["V"].view(np.uint64)), (kw, mode, e)
                assert np.array_equal(P[e].view(np.uint32), d["P"].view(np.uint32)), (kw, mode, e)


def test_frame_cameras_fail_before_the_first_render(torch_cuda):
    from gym_duckietown_b200 import lib as L
    env = make_env(2, "small_loop", bev_visibility=False)
    with pytest.raises(L.DtsError):
        env.frame_cameras()


def test_refusals_leave_the_previous_setting(torch_cuda):
    from gym_duckietown_b200 import lib as L
    torch = torch_cuda
    n = 2
    vis = torch.zeros((n, 64, 64), dtype=torch.uint8, device="cuda")
    pix = torch.zeros((n, 64, 64, 2), dtype=torch.float32, device="cuda")
    no_grid = make_env(n, "small_loop", bev_visibility=False, labels=True)
    with pytest.raises(L.DtsError):   # no bird's-eye label target
        no_grid.sim.set_bev_visibility_target(vis.data_ptr(), pix.data_ptr())
    no_labels = make_env(n, "small_loop", bev_visibility=False, bev=True)
    with pytest.raises(L.DtsError):   # no camera label target
        no_labels.sim.set_bev_visibility_target(vis.data_ptr(), pix.data_ptr())
    env = make_env(n, "small_loop", distortion=True)
    twin = make_env(n, "small_loop", distortion=True)
    m = env.camera_model
    with pytest.raises(L.DtsError):   # a pixel target not 8-byte aligned
        env.sim.set_bev_visibility_target(vis.data_ptr(), pix.data_ptr() + 4, m.mapx, m.mapy)
    with pytest.raises(L.DtsError):   # two forward maps for a pool of one table
        env.sim.set_bev_visibility_target(vis.data_ptr(), pix.data_ptr(), np.stack([m.mapx] * 2),
                                          np.stack([m.mapy] * 2))
    with pytest.raises(L.DtsError):   # it reads the label image
        env.sim.set_label_target(None)
    with pytest.raises(L.DtsError):   # and the grid's labels
        env.sim.set_bev_target(None, None, None)
    with pytest.raises(L.DtsError):
        env.sim.set_bev_target(env.bev_config, None, env.bev_markings.data_ptr())
    from gym_duckietown_b200 import lib
    c = env.bev_config
    with pytest.raises(L.DtsError):   # another grid shape
        env.sim.set_bev_target(lib.BevConfig(c.width // 2, c.height, c.cell, c.origin_x, c.origin_y),
                               env.bev_labels.data_ptr(), env.bev_markings.data_ptr())
    act = torch.full((n, 2), 0.7, dtype=torch.float32, device=env.device)
    for e_ in (env, twin):
        e_.reset()
        e_.step(act)
    a, b = host(env), host(twin)
    assert (a[0] == vo.VISIBLE).any()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    check(env, "after refusals")


def test_changes_no_other_output_and_launches_one_kernel(torch_cuda):
    torch = torch_cuda
    n = 4
    kw = dict(depth=True, labels=True, markings=True, bev=True, flow_occlusion=True)
    on = make_env(n, "loop_dyn_duckiebots", **kw)
    off = make_env(n, "loop_dyn_duckiebots", bev_visibility=False, **kw)
    rng = np.random.default_rng(8)
    for e_ in (on, off):
        e_.reset()
    c_on, c_off = on.launch_count(), off.launch_count()
    names = ("obs", "depth", "labels", "markings", "bev_labels", "bev_markings", "flow", "flow_occlusion")
    for k in range(6):
        act = actions(torch, rng, n, on.device)
        for e_ in (on, off):
            e_.step(act, render=k % 3 != 1)
        for name in names:
            x, y = getattr(on, name).cpu().numpy(), getattr(off, name).cpu().numpy()
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (name, k)
    for e_ in (on, off):
        e_.render_obs()
        e_.render_bev()
    assert on.launch_count() - c_on == off.launch_count() - c_off + 6 + 2   # one per grid-writing call
    for name in names:
        x, y = getattr(on, name).cpu().numpy(), getattr(off, name).cpu().numpy()
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    # off again: nothing new launches
    on.sim.set_bev_visibility_target(None, None)
    c_on, c_off = on.launch_count(), off.launch_count()
    act = actions(torch, rng, n, on.device)
    for e_ in (on, off):
        e_.step(act)
    assert on.launch_count() - c_on == off.launch_count() - c_off


def test_flow_and_visibility_share_the_forward_maps(torch_cuda):
    """Clearing flow keeps the fisheye forward maps for the visibility, and clearing the visibility keeps them for flow"""
    torch = torch_cuda
    n = 4
    rng = np.random.default_rng(12)
    a = make_env(n, "udem1", distortion=True, flow=True)
    a.reset()
    a.sim.set_flow_target(None)
    for k in range(3):
        a.step(actions(torch, rng, n, a.device))
        check(a, f"flow cleared, step {k}")
    b, twin = make_env(n, "udem1", distortion=True, flow=True), make_env(n, "udem1", distortion=True, flow=True,
                                                                          bev_visibility=False)
    b.sim.set_bev_visibility_target(None, None)
    for e_ in (b, twin):
        e_.reset()
    for k in range(3):
        act = actions(torch, rng, n, b.device)
        b.step(act), twin.step(act)
        assert np.array_equal(b.flow.cpu().numpy().view(np.uint32), twin.flow.cpu().numpy().view(np.uint32))
    assert not np.isnan(b.flow.cpu().numpy()).all()
