"""The object boxes on the device (dts_set_object_target, DESIGN.md section 5 item 17) against the float64 oracle
(tests/object_oracle.py), fed with the device's own poses, obstacles, hidden masks and cameras (frame_cameras()):
boxes within 1e-6 m / 1e-6 rad, states exact, and every unambiguous corner pixel within one float32 ulp (pinhole) or
2^-10 px (fisheye, a camera_rand pool).  Over 30-step rollouts on every map, the fisheye, a camera_rand pool, undistort,
the rectification, top-down and segment views, steps without a render, device auto-reset with terminal frames, hidden
optional objects and a two-map batch with unequal object counts.  Also k_object_pixels (object_boxes()) against a numpy
reduction at 4096 x 160x120 and at odd sizes, refused calls, and the launches the target adds."""
import numpy as np
import pytest

import object_oracle as oo
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
    args = dict(camera_width=w, camera_height=h, domain_rand=True, seed=11, objects=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def actions(torch, rng, n, device):
    return torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=device)


def dyn_corners(env, field=None):
    """Every env's obstacles' corners [n_dyn][4][2] (or, given a DTS_DYN_* field, that field [n_dyn]), or None where its
    map has none"""
    import torch
    from gym_duckietown_b200 import lib as L
    n = env.num_envs
    mid = env.state["map_id"].cpu().numpy()
    dyn = {}
    for m in range(len(env.maps)):
        arr, nd = env.sim.dyn_state(m)
        if nd:
            a = torch.as_tensor(arr, device=env.device).cpu().numpy().reshape(L.DYN_FIELDS, nd, n)
            dyn[m] = a[L.DYN_CORNERS:L.DYN_CORNERS + 8] if field is None else a[field]
    if field is not None:
        return [dyn[int(mid[e])][:, e] if int(mid[e]) in dyn else None for e in range(n)]
    return [dyn[int(mid[e])][:, :, e].T.reshape(-1, 4, 2) if int(mid[e]) in dyn else None for e in range(n)]


def check(env, what, drew=True, fisheye=None):
    """Every env's rows against the oracle for its current state and, where `drew`, its last frame; returns the number
    of points compared and of ambiguous ones, and the count of each state"""
    import torch
    torch.cuda.synchronize()
    boxes, state, px = (t.cpu().numpy() for t in (env.object_boxes3d, env.object_state, env.object_corners_px))
    O = boxes.shape[1]
    V, P = (t.cpu().numpy() for t in env.frame_cameras()) if drew else (None, None)
    x, z, a = poses_of(env)
    mid = env.state["map_id"].cpu().numpy()
    corners = dyn_corners(env)
    from gym_duckietown_b200 import lib as L
    angles = dyn_corners(env, L.DYN_ANGLE)
    fish = env.distortion and not env.undistort if fisheye is None else fisheye
    n_cmp = n_amb = 0
    states = np.zeros(3, np.int64)
    for e in range(env.num_envs):
        md = env.maps[int(mid[e])]
        hidden = env.sim.debug_episode(e)["hidden"]
        cam = None
        if drew:
            m = model_of(env, e) if fish else None
            cam = (V[e].ravel(), P[e], env.camera_width, env.camera_height, (m.mapx, m.mapy) if fish else None)
        b, s, q, amb = oo.objects(md, (x[e], z[e], a[e]), O, corners[e], hidden, cam, angles[e])
        where = f"{what} env {e}"
        assert np.array_equal(state[e], s), f"{where}: state {state[e]} oracle {s}"
        assert np.array_equal(np.isnan(boxes[e]), np.isnan(b)), f"{where}: box NaN pattern"
        ok = ~np.isnan(b)
        err = np.abs(boxes[e][ok].astype(np.float64) - b[ok])
        assert (err <= 1e-6).all(), f"{where}: box off by {err.max():.3g}"
        got, want = px[e].astype(np.float64), q
        cmp = ~amb[..., None] & np.ones_like(want, bool)
        assert np.array_equal(np.isnan(got)[cmp], np.isnan(want)[cmp]), f"{where}: corner NaN pattern"
        both = cmp & ~np.isnan(want)
        bar = 2.0 ** -10 if fish else np.spacing(np.abs(want[both]).astype(np.float32)).astype(np.float64) + \
            1e-9 * np.abs(want[both])
        err = np.abs(got[both] - want[both])
        assert (err <= bar).all(), f"{where}: corner off by {err.max():.3g} px"
        n_cmp += int(both.sum())
        n_amb += int(amb.sum())
        states += np.bincount(s, minlength=3)
    return n_cmp, n_amb, states


CASES = [(m, "pinhole") for m in MAPS if m != "small_loop"] + [
    ("udem1", "fisheye"), ("loop_dyn_duckiebots", "fisheye"), ("loop_pedestrians", "camera_rand"),
    ("udem1", "undistort"), ("loop_dyn_duckiebots", "top_down"), ("udem1", "segment"),
    (("small_loop", "loop_obstacles"), "pinhole"), ("loop_pedestrians", "no_render")]


@pytest.mark.parametrize("names,view", CASES)
def test_rollout_against_the_oracle(torch_cuda, names, view):
    torch = torch_cuda
    n = 4
    kw = dict(distortion=view in ("fisheye", "camera_rand", "undistort"), camera_rand=view == "camera_rand")
    if view == "camera_rand":
        kw["camera_rand_pool"] = 4
    if isinstance(names, tuple):
        kw["cycle_maps"] = True
    env = make_env(n, names, **kw)
    if view == "undistort":
        env.undistort = True
    env.reset()
    if isinstance(names, tuple):   # the even envs on the second map: half the batch has no objects
        env.reset(mask=torch.arange(n, device=env.device) % 2 == 0)
    mode = dict(top_down=view == "top_down", segment=view == "segment")
    rng = np.random.default_rng(4)
    n_cmp = n_amb = 0
    states = np.zeros(3, np.int64)
    for k in range(30):
        act = actions(torch, rng, n, env.device)
        if view == "no_render":
            env.step(act, render=False)
            c, a, s = check(env, f"{names} {view} step {k}", drew=False)
            assert np.isnan(env.object_corners_px.cpu().numpy()).all()
        elif mode["top_down"] or mode["segment"]:
            env.step(act, render=False)
            env.render_obs(**mode)
            c, a, s = check(env, f"{names} {view} step {k}", fisheye=False)
        else:
            env.step(act)
            c, a, s = check(env, f"{names} {view} step {k}")
        n_cmp, n_amb, states = n_cmp + c, n_amb + a, states + s
    assert states[oo.SHOWN] > 0
    assert view == "no_render" or n_cmp > 0
    assert n_amb <= 1e-3 * max(n_cmp, 1) + 1, (n_amb, n_cmp)
    if isinstance(names, tuple):
        assert states[oo.NONE] > 0
        b = env.object_boxes3d.cpu().numpy()
        assert np.isnan(b[env.object_state.cpu().numpy() == oo.NONE]).all()


def test_duckiebot_yaw_follows_its_heading(torch_cuda):
    """Tied to the obstacles' own state, not to the corner order: each Duckiebot's yaw is its DTS_DYN_ANGLE minus the
    agent's angle, before and after its turning step rewrites its corners in agent_boundbox's order, and its length
    then lies along its heading (robot_length)"""
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200.maps import DYN_DUCKIEBOT
    torch = torch_cuda
    n = 8
    env = make_env(n, "loop_dyn_duckiebots", domain_rand=False)
    env.reset()
    md = env.maps[0]
    bots = [(s, d) for s, d in enumerate(md.dyn_objects) if d.kind == DYN_DUCKIEBOT]
    assert bots
    rng = np.random.default_rng(5)
    turned = 0
    for k in range(40):
        env.step(actions(torch, rng, n, env.device))
        torch.cuda.synchronize()
        boxes = env.object_boxes3d.cpu().numpy().astype(np.float64)
        ang = dyn_corners(env, L.DYN_ANGLE)
        agent = env.state["angle"].cpu().numpy()
        for e in range(n):
            for s, d in bots:
                want = ang[e][s] - agent[e]
                diff = (boxes[e, d.object_index, 6] - want + np.pi) % (2 * np.pi) - np.pi
                assert abs(diff) <= 1e-6, (k, e, s, boxes[e, d.object_index, 6], want)
                if ang[e][s] != d.angle:   # it has turned: its corners are agent_boundbox's
                    turned += 1
                    assert abs(boxes[e, d.object_index, 3] - d.robot_length) <= 1e-6, (k, e, s)
                    assert abs(boxes[e, d.object_index, 4] - d.robot_width) <= 1e-6, (k, e, s)
        check(env, f"duckiebots step {k}")
    assert turned > 0


def test_hidden_optional_objects_have_boxes(torch_cuda):
    torch = torch_cuda
    n = 16
    env = make_env(n, "udem1", domain_rand=True)
    env.reset()
    rng = np.random.default_rng(2)
    env.step(actions(torch, rng, n, env.device))
    _, _, states = check(env, "udem1 domain_rand")
    assert states[oo.HIDDEN] > 0 and states[oo.SHOWN] > 0, states


def test_device_reset_with_terminal_frames(torch_cuda):
    torch = torch_cuda
    n = 8
    env = make_env(n, "loop_pedestrians", auto_reset=True, device_reset=True, terminal_obs=True, max_steps=7)
    env.reset()
    rng = np.random.default_rng(6)
    ended = 0
    for k in range(30):
        _, _, done, _ = env.step(actions(torch, rng, n, env.device))
        ended += int(done.sum())
        check(env, f"auto-reset step {k}")
    assert ended > 0
    env.step(actions(torch, rng, n, env.device), render=False)
    check(env, "auto-reset step without a render", drew=False)


@pytest.mark.parametrize("how", ["reset", "load_state", "copy_envs"])
def test_render_objects_after_state_changes(torch_cuda, how):
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_dyn_duckiebots")
    env.reset()
    rng = np.random.default_rng(3)
    for k in range(5):
        env.step(actions(torch, rng, n, env.device))
    if how == "reset":
        env.reset(render=False)
    elif how == "load_state":
        recs = env.save_state()
        for k in range(3):
            env.step(actions(torch, rng, n, env.device))
        env.load_state(recs)
    else:
        env.copy_envs([3, 2, 1, 0])
    env.render_objects()
    check(env, how, drew=False)
    assert np.isnan(env.object_corners_px.cpu().numpy()).all()
    env.render_obs()
    check(env, how + " then rendered")


def test_rectified_frames_give_nan_corners(torch_cuda):
    from gym_duckietown_b200.distortion import rectify_maps
    torch = torch_cuda
    n = 2
    env = make_env(n, "loop_obstacles", distortion=True)
    rx, ry = rectify_maps(env.camera_width, env.camera_height)
    env.set_rectification(rx, ry)
    env.undistort = True
    env.reset()
    env.step(torch.full((n, 2), 0.5, dtype=torch.float32, device=env.device))
    check(env, "rectified", drew=False)
    assert np.isnan(env.object_corners_px.cpu().numpy()).all()
    assert (env.object_state.cpu().numpy() == oo.SHOWN).all()


def numpy_object_boxes(env, labels):
    """object_boxes()'s rule restated in numpy, every env at once"""
    n, h, w = labels.shape
    O = max(len(md.objects) for md in env.maps)
    mid = env.state["map_id"].cpu().numpy()
    cells = np.array([md.grid_w * md.grid_h for md in env.maps])[mid]
    nobj = np.array([len(md.objects) for md in env.maps])[mid]
    o = labels.astype(np.int64) - 2 - cells[:, None, None]
    hit = (o >= 0) & (o < nobj[:, None, None])
    e, y, x = np.nonzero(hit)
    slot = e * O + o[hit]
    pixels = np.bincount(slot, minlength=n * O).astype(np.int32)
    boxes = np.full((n * O, 4), -1, np.int32)
    for col, v in ((0, x), (1, y)):
        order = np.lexsort((v, slot))
        s, vs = slot[order], v[order]
        first = np.r_[True, s[1:] != s[:-1]]
        last = np.r_[s[1:] != s[:-1], True]
        boxes[s[first], col] = vs[first]
        boxes[s[last], col + 2] = vs[last]
    return pixels.reshape(n, O), boxes.reshape(n, O, 4)


def test_object_pixels_at_the_benchmark_size(torch_cuda):
    torch = torch_cuda
    env = make_env(4096, "udem1", w=160, h=120, objects=False, labels=True)
    env.reset()
    rng = np.random.default_rng(0)
    env.step(actions(torch, rng, 4096, env.device))
    pixels, boxes = env.object_boxes()
    torch.cuda.synchronize()
    want_p, want_b = numpy_object_boxes(env, env.labels.cpu().numpy())
    assert pixels.dtype == torch.int32 and boxes.dtype == torch.int32
    assert np.array_equal(pixels.cpu().numpy(), want_p) and np.array_equal(boxes.cpu().numpy(), want_b)
    assert want_p.sum() > 0


@pytest.mark.parametrize("w,h", [(1, 1), (3, 799), (799, 3), (101, 75), (13, 7)])
def test_object_pixels_at_odd_sizes(torch_cuda, w, h):
    """Synthetic label images: blocks of one object, noise of every label value (some past the map's objects)"""
    torch = torch_cuda
    n = 5
    env = make_env(n, ["loop_obstacles", "udem1"], w=w, h=h, objects=False, labels=True, cycle_maps=True)
    env.reset()
    env.reset(mask=torch.arange(n, device=env.device) % 2 == 0)   # maps 1, 0, 1, 0, 1
    rng = np.random.default_rng(w * 1000 + h)
    top = 2 + 25 * 25 + 30
    lab = rng.integers(0, top, (n, h, w)).astype(np.int16)
    mid = env.state["map_id"].cpu().numpy()
    for e in range(n):
        md = env.maps[int(mid[e])]
        base = 2 + md.grid_w * md.grid_h
        for k in range(4):
            y0, x0 = rng.integers(0, h), rng.integers(0, w)
            lab[e, y0:y0 + rng.integers(1, 40), x0:x0 + rng.integers(1, 40)] = base + rng.integers(0, len(md.objects))
    env.labels.copy_(torch.from_numpy(lab).to(env.device))
    pixels, boxes = env.object_boxes()
    torch.cuda.synchronize()
    want_p, want_b = numpy_object_boxes(env, lab)
    assert np.array_equal(pixels.cpu().numpy(), want_p), (w, h)
    assert np.array_equal(boxes.cpu().numpy(), want_b), (w, h)


def test_refusals_leave_the_previous_target(torch_cuda):
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200.maps import load_map
    torch = torch_cuda
    n = 2
    env = make_env(n, "loop_obstacles")
    twin = make_env(n, "loop_obstacles")
    O = env.object_state.shape[1]
    other = torch.zeros((n, 32, 7), dtype=torch.float32, device=env.device)
    for bad in (0, O - 1, 257):   # (DTS_MAX_OBJECTS is 256)
        with pytest.raises(L.DtsError):
            env.sim.set_object_target(bad, other.data_ptr(), None, None)
    with pytest.raises(L.DtsError):   # a box target not aligned to its element size
        env.sim.set_object_target(O, env.object_boxes3d.data_ptr() + 2, None, None)
    with pytest.raises(L.DtsError):   # the map has more objects than the target holds
        env.sim.upload_map(0, load_map("udem1"), None)
    act = torch.full((n, 2), 0.6, dtype=torch.float32, device=env.device)
    for e_ in (env, twin):
        e_.reset()
        e_.step(act)
    assert np.isnan(other.cpu().numpy()).sum() == 0   # never written
    for name in ("object_boxes3d", "object_state", "object_corners_px"):
        x, y = getattr(env, name).cpu().numpy(), getattr(twin, name).cpu().numpy()
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    check(env, "after refusals")


def test_a_map_without_objects_gives_empty_outputs(torch_cuda):
    torch = torch_cuda
    env = make_env(2, "small_loop")
    env.reset()
    c = env.launch_count()
    env.step(torch.zeros((2, 2), dtype=torch.float32, device=env.device))
    b, s, q = env.render_objects()
    assert b.shape == (2, 0, 7) and s.shape == (2, 0) and q.shape == (2, 0, 9, 2)
    plain = make_env(2, "small_loop", objects=False)
    plain.reset()
    c_plain = plain.launch_count()
    plain.step(torch.zeros((2, 2), dtype=torch.float32, device=env.device))
    assert env.launch_count() - c == plain.launch_count() - c_plain


def test_launches_one_kernel_and_changes_no_other_output(torch_cuda):
    torch = torch_cuda
    n = 4
    kw = dict(depth=True, labels=True, bev=True, scan=True, bev_visibility=True, auto_reset=True, device_reset=True,
              terminal_obs=True, max_steps=4)
    on = make_env(n, "loop_dyn_duckiebots", **kw)
    off = make_env(n, "loop_dyn_duckiebots", **dict(kw, objects=False))
    rng = np.random.default_rng(8)
    for e_ in (on, off):
        e_.reset()
    c_on, c_off = on.launch_count(), off.launch_count()
    names = ("obs", "terminal_obs", "depth", "labels", "bev_labels", "bev_visibility", "bev_pixels", "scan_range")
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
    on.sim.set_object_target(0, None, None, None)   # off again: nothing new launches
    c_on, c_off = on.launch_count(), off.launch_count()
    for k in range(3):
        act = actions(torch, rng, n, on.device)
        for e_ in (on, off):
            e_.step(act, render=k != 1)
    assert on.launch_count() - c_on == off.launch_count() - c_off
