"""The lane path on the device (dts_set_lane_path_target, DESIGN.md section 5 item 18) against the float64 oracle
(tests/lane_path_oracle.py), fed with the device's own poses and cameras (frame_cameras()): points within 1e-6 m, yaw
within 1e-6 rad, counts exact, and every unambiguous pixel within one float32 ulp (pinhole, top-down) or 2^-10 px
(fisheye, a camera_rand pool).  A point is ambiguous where the device's sincos / atan2 may pick another curve,
bisection branch or tile than libm's (that point and the rest of its chain go unchecked), or where item 17's pixel rules
say so; fewer than 1 % of the points of a case may be.  Over seeded rollouts with device auto-reset on every map and a
two-map batch, 1 to 4096 envs, 1 to 64 points and several spacings.  Also where the pixels are NaN, terminal frames,
refused calls, the forward maps it shares, the launches it adds, the outputs it leaves alone, and Simulator."""
import numpy as np
import pytest

import lane_path_oracle as lo
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
    args = dict(camera_width=w, camera_height=h, domain_rand=True, seed=11, lane_path=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def actions(torch, rng, n, device):
    return torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=device)


def check(env, what, spacing, drew=True, fisheye=None):
    """Every env's rows against the oracle for its current state and, where `drew`, its last frame; returns the number
    of points compared and of ambiguous ones"""
    import torch
    torch.cuda.synchronize()
    pts, count, px = (t.cpu().numpy() for t in (env.lane_path, env.lane_path_count, env.lane_path_px))
    N, K = pts.shape[:2]
    V, P = (t.cpu().numpy() for t in env.frame_cameras()) if drew else (None, None)
    x, z, a = poses_of(env)
    poses = np.stack([x, z, a], 1)
    mid = env.state["map_id"].cpu().numpy()
    fish = env.distortion and not env.undistort if fisheye is None else fisheye
    q, t = np.full((N, K, 3), np.nan), np.full((N, K, 3), np.nan)
    want_n, amb = np.zeros(N, np.int64), np.zeros((N, K), bool)
    for m in np.unique(mid):
        e = np.flatnonzero(mid == m)
        q[e], t[e], want_n[e], amb[e] = lo.walk(env.maps[int(m)], poses[e], K, spacing)
    want = lo.agent_frame(poses, q, t)
    clean = ~amb.any(1)
    assert np.array_equal(count[clean], want_n[clean]), f"{what}: count"
    live = np.arange(K)[None, :] < count[:, None]
    assert np.isnan(pts[~live]).all() and np.isnan(px[~live]).all(), f"{what}: rows past the count"
    ok = ~amb & (np.arange(K)[None, :] < want_n[:, None])
    got = pts.astype(np.float64)
    assert not np.isnan(got[ok]).any(), f"{what}: NaN point"
    err = np.abs(got[ok][:, :2] - want[ok][:, :2])
    assert err.size == 0 or err.max() <= 1e-6, f"{what}: point off by {err.max():.3g} m"
    yerr = np.abs((got[ok][:, 2] - want[ok][:, 2] + np.pi) % (2 * np.pi) - np.pi)
    assert yerr.size == 0 or yerr.max() <= 1e-6, f"{what}: yaw off by {yerr.max():.3g}"
    n_amb = int(amb.sum())
    n_cmp = int(ok.sum())
    if drew:
        for e in range(N):
            m = model_of(env, e) if fish else None
            cam = (V[e].ravel(), P[e], env.camera_width, env.camera_height, (m.mapx, m.mapy) if fish else None)
            wp, pamb = lo.pixels(q[e], int(want_n[e]), cam)
            cmp = (ok[e] & ~pamb)[:, None] & np.ones((K, 2), bool)
            g = px[e].astype(np.float64)
            assert np.array_equal(np.isnan(g)[cmp], np.isnan(wp)[cmp]), f"{what} env {e}: pixel NaN pattern"
            both = cmp & ~np.isnan(wp)
            bar = 2.0 ** -10 if fish else np.spacing(np.abs(wp[both]).astype(np.float32)).astype(np.float64) + \
                1e-9 * np.abs(wp[both])
            perr = np.abs(g[both] - wp[both])
            assert (perr <= bar).all(), f"{what} env {e}: pixel off by {perr.max():.3g} px"
            n_amb += int((ok[e] & pamb).sum())
    else:
        assert np.isnan(px).all(), f"{what}: pixels without a frame"
    return n_cmp, n_amb


CASES = [(m, 37, 16, 0.1, "pinhole") for m in MAPS] + [
    ("udem1", 1, 1, 0.05, "pinhole"), ("loop_obstacles", 4096, 64, 0.3, "pinhole"), ("udem1", 4096, 16, 0.1, "fisheye"),
    ("udem1", 37, 64, 0.05, "fisheye"), ("loop_pedestrians", 37, 16, 0.2, "camera_rand"),
    ("loop_trafficlights", 37, 64, 0.1, "top_down"), (("small_loop", "loop_obstacles"), 37, 16, 0.1, "pinhole"),
    ("small_loop", 37, 64, 1.0, "pinhole")]


@pytest.mark.parametrize("names,n,K,ds,view", CASES)
def test_rollout_against_the_oracle(torch_cuda, names, n, K, ds, view):
    torch = torch_cuda
    kw = dict(distortion=view in ("fisheye", "camera_rand"), camera_rand=view == "camera_rand", auto_reset=True,
              device_reset=True, max_steps=9, lane_path_points=K, lane_path_spacing=ds)
    if view == "camera_rand":
        kw["camera_rand_pool"] = 4
    if isinstance(names, tuple):
        kw["cycle_maps"] = True
    env = make_env(n, names, **kw)
    env.reset()
    if isinstance(names, tuple):
        env.reset(mask=torch.arange(n, device=env.device) % 2 == 0)
    rng = np.random.default_rng(n * 100 + K)
    n_cmp = n_amb = 0
    found = 0
    for k in range(3 if n == 4096 else 12):
        act = actions(torch, rng, n, env.device)
        if view == "top_down":
            env.step(act, render=False)
            env.render_obs(top_down=True)
            c, a = check(env, f"{names} {view} step {k}", ds, fisheye=False)
        else:
            env.step(act)
            c, a = check(env, f"{names} {view} step {k}", ds)
        n_cmp, n_amb = n_cmp + c, n_amb + a
        found += int(env.lane_path_count.sum().item())
    assert n_cmp > 0 and found > 0
    assert n_amb < 0.01 * (n_cmp + n_amb), (n_amb, n_cmp)


def test_pixels_are_nan_without_a_pinhole_or_fisheye_frame(torch_cuda):
    from gym_duckietown_b200.distortion import rectify_maps
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_obstacles", distortion=True)
    rx, ry = rectify_maps(env.camera_width, env.camera_height)
    env.set_rectification(rx, ry)
    env.undistort = True
    env.reset()
    act = torch.full((n, 2), 0.5, dtype=torch.float32, device=env.device)
    env.step(act)
    check(env, "rectified", 0.1, drew=False)
    plain = make_env(n, "udem1")
    plain.reset()
    plain.step(act, render=False)
    check(plain, "render=False", 0.1, drew=False)
    plain.step(act)
    assert not np.isnan(plain.lane_path_px.cpu().numpy()).all()
    plain.reset(render=False)
    plain.render_lane_path()
    check(plain, "render_lane_path", 0.1, drew=False)
    assert int(plain.lane_path_count.sum().item()) > 0


def test_terminal_steps_show_the_respawned_state(torch_cuda):
    torch = torch_cuda
    n = 16
    env = make_env(n, "loop_pedestrians", auto_reset=True, device_reset=True, terminal_obs=True, max_steps=5)
    env.reset()
    rng = np.random.default_rng(6)
    ended = 0
    for k in range(14):
        _, _, done, _ = env.step(actions(torch, rng, n, env.device))
        ended += int(done.sum())
        check(env, f"terminal step {k}", 0.1)
    assert ended > 0
    env.step(actions(torch, rng, n, env.device), render=False)
    check(env, "terminal step without a render", 0.1, drew=False)


def test_refusals_leave_the_previous_target(torch_cuda):
    from gym_duckietown_b200 import lib as L
    torch = torch_cuda
    n = 4
    env, twin = make_env(n, "udem1"), make_env(n, "udem1")
    other = torch.zeros((n, 64, 3), dtype=torch.float32, device=env.device)
    cnt = torch.zeros(n + 1, dtype=torch.int16, device=env.device)
    for K, ds in ((0, 0.1), (65, 0.1), (16, 0.0), (16, -0.1), (16, 1.01), (16, float("nan")), (16, float("inf"))):
        with pytest.raises(L.DtsError):
            env.sim.set_lane_path_target(K, ds, other.data_ptr(), None, None)
    with pytest.raises(L.DtsError):
        env.sim.set_lane_path_target(16, 0.1, other.data_ptr() + 2, None, None)
    with pytest.raises(L.DtsError):
        env.sim.set_lane_path_target(16, 0.1, None, None, other.data_ptr() + 2)
    with pytest.raises(L.DtsError):
        env.sim.set_lane_path_target(16, 0.1, None, cnt.data_ptr() + 1, None)
    fx = np.zeros((1, env.camera_height, env.camera_width), np.float32)
    with pytest.raises(L.DtsError):   # forward maps on a handle without the fisheye
        env.sim.set_lane_path_target(16, 0.1, other.data_ptr(), None, None, fx, fx)
    act = torch.full((n, 2), 0.6, dtype=torch.float32, device=env.device)
    for e_ in (env, twin):
        e_.reset()
        e_.step(act)
    assert (other.cpu().numpy() == 0).all() and (cnt.cpu().numpy() == 0).all()   # never written
    for name in ("lane_path", "lane_path_count", "lane_path_px"):
        x, y = getattr(env, name).cpu().numpy(), getattr(twin, name).cpu().numpy()
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    check(env, "after refusals", 0.1)
    env.sim.set_lane_path_target(0, 0.0, None, None, None)   # off
    with pytest.raises(L.DtsError):
        env.sim.render_lane_path()


ORDERS = [("flow", "bev_visibility", "objects", "lane_path"), ("lane_path", "objects", "bev_visibility", "flow"),
          ("objects", "lane_path", "flow", "bev_visibility"), ("bev_visibility", "flow", "lane_path", "objects")]


def clear(env, name):
    if name == "flow":
        env.sim.set_flow_target(None)
    elif name == "bev_visibility":
        env.sim.set_bev_visibility_target(None, None)
    elif name == "objects":
        env.sim.set_object_target(0, None, None, None)
    else:
        env.sim.set_lane_path_target(0, 0.0, None, None, None)


@pytest.mark.parametrize("order", ORDERS)
def test_targets_share_the_forward_maps(torch_cuda, order):
    """Cleared one by one in each order, the fisheye forward maps stay while any target still reads them: every fisheye
    step with a reader left renders (a reader without the maps fails it), and the lane path's pixels, while it is set,
    are the oracle's through them.  Set again after the last one, it takes the maps again."""
    torch = torch_cuda
    n = 4
    rng = np.random.default_rng(13)
    env = make_env(n, "udem1", distortion=True, depth=True, labels=True, bev=True, flow=True, bev_visibility=True,
                   objects=True)
    env.reset()
    for k, name in enumerate(order):
        clear(env, name)
        env.step(actions(torch, rng, n, env.device))
        if "lane_path" not in order[:k + 1]:
            check(env, f"{order[:k + 1]} cleared", 0.1)
    env.sim.set_lane_path_target(16, 0.1, env.lane_path.data_ptr(), env.lane_path_count.data_ptr(),
                                 env.lane_path_px.data_ptr(), np.stack([env.camera_model.mapx]),
                                 np.stack([env.camera_model.mapy]))
    env.step(actions(torch, rng, n, env.device))
    check(env, "set again", 0.1)


def test_launches_one_kernel_and_changes_no_other_output(torch_cuda):
    torch = torch_cuda
    n = 8
    kw = dict(depth=True, labels=True, markings=True, bev=True, scan=True, bev_visibility=True, objects=True,
              auto_reset=True, device_reset=True, terminal_obs=True, max_steps=4)
    on = make_env(n, "loop_dyn_duckiebots", **kw)
    off = make_env(n, "loop_dyn_duckiebots", **dict(kw, lane_path=False))
    rng = np.random.default_rng(8)
    for e_ in (on, off):
        e_.reset()
    c_on, c_off = on.launch_count(), off.launch_count()
    names = ("obs", "terminal_obs", "depth", "labels", "markings", "bev_labels", "bev_markings", "bev_visibility",
             "bev_pixels", "scan_range", "scan_hit", "object_boxes3d", "object_state", "object_corners_px")
    for k in range(6):
        act = actions(torch, rng, n, on.device)
        for e_ in (on, off):
            e_.step(act, render=k % 3 != 1)
    for e_ in (on, off):
        e_.render_obs()
        e_.render_bev()
    assert on.launch_count() - c_on == off.launch_count() - c_off + 6 + 1   # steps and render_obs; not render_bev
    for name in names:
        x, y = getattr(on, name).cpu().numpy(), getattr(off, name).cpu().numpy()
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    on.sim.set_lane_path_target(0, 0.0, None, None, None)   # off again: nothing new launches
    c_on, c_off = on.launch_count(), off.launch_count()
    for k in range(3):
        act = actions(torch, rng, n, on.device)
        for e_ in (on, off):
            e_.step(act, render=k != 1)
    assert on.launch_count() - c_on == off.launch_count() - c_off


def test_simulator_gives_env_zero(torch_cuda):
    from gym_duckietown_b200.simulator import Simulator
    sim = Simulator("udem1", camera_width=96, camera_height=72, seed=3, domain_rand=False, lane_path=True,
                    lane_path_points=8, lane_path_spacing=0.2)
    sim.reset()
    sim.step([0.4, 0.4])
    b = sim._b
    check(b, "Simulator", 0.2)
    assert sim.lane_path.shape == (8, 3) and sim.lane_path_px.shape == (8, 2)
    assert np.array_equal(sim.lane_path.view(np.uint32), b.lane_path[0].cpu().numpy().view(np.uint32))
    assert np.array_equal(sim.lane_path_px.view(np.uint32), b.lane_path_px[0].cpu().numpy().view(np.uint32))
    assert sim.lane_path_count == int(b.lane_path_count[0].item()) > 0
    plain = Simulator("udem1", camera_width=96, camera_height=72, seed=3, domain_rand=False)
    assert plain.lane_path is None and plain.lane_path_count is None and plain.lane_path_px is None
