"""The motion-flow image on the device (dts_set_flow_target, DESIGN.md section 5 item 13) against the float64 oracle
(tests/flow_oracle.py): every pixel that is not ambiguous within max(2^-10 px, 1e-5 |flow|), with the same NaN pattern,
over 50-step rollouts with random actions and domain randomisation on every map, pinhole, fisheye, a camera_rand pool,
top-down and segment views and a two-map batch.  Also: the label and depth warps of tests/test_flow_oracle.py on
consecutive device frames, zero flow where nothing moved, the lifecycle (resets, auto-reset, terminal frames, loads,
renders after a step), refused calls, and that flow changes no other output and adds only its own launches."""
import numpy as np
import pytest

import flow_oracle as fo
from test_flow_oracle import LABEL_BAR, label_warp

pytestmark = pytest.mark.gpu

MAPS = ["small_loop", "small_loop_only_duckies", "loop_obstacles", "loop_only_duckies", "loop_pedestrians",
        "loop_dyn_duckiebots", "loop_trafficlights", "udem1"]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, names, w=96, h=72, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=True, seed=11, flow=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def snap(env):
    """The state flow is taken against: poses, episodes, map ids and every map's obstacles"""
    import torch
    from gym_duckietown_b200 import lib as L
    torch.cuda.synchronize()
    st = {k: env.state[k].cpu().numpy().copy() for k in ("pos_x", "pos_z", "angle", "episode", "map_id")}
    dyn = {}
    for m in range(len(env.maps)):
        arr, nd = env.sim.dyn_state(m)
        dyn[m] = torch.as_tensor(arr, device=env.device).cpu().numpy().reshape(L.DYN_FIELDS, nd, env.num_envs).copy() \
            if nd else None
    return st, dyn


def frames(env):
    """V, P of every env's last frame"""
    out = []
    for e in range(env.num_envs):
        md = env.maps[int(env.state["map_id"][e])]
        d = env.sim.debug_frame(e, md.grid_w * md.grid_h)
        out.append((d["V"].copy(), d["P"].copy()))
    return out


def model_of(env, e):
    return env.camera_models[env.calibration_of_env[e]] if env.camera_rand else env.camera_model


def oracle(env, e, before, after, Vp, Vc, P, depth, labels, top_down=False, fisheye=None):
    """flow_oracle.flow for env e across one step, from snapshots before and after it"""
    (s0, d0), (s1, d1) = before, after
    mid = int(s1["map_id"][e])
    md = env.maps[mid]
    moves = {}
    for s, dobj in enumerate(md.dyn_objects):
        if dobj.kind == 3:   # a traffic light does not move
            continue
        b, a = d0[mid][:, s, e], d1[mid][:, s, e]
        moves[dobj.object_index] = ((b[0], b[1], b[3]), (a[0], a[1], a[3]))
    agent = None
    if top_down:
        agent = ((s0["pos_x"][e], s0["pos_z"][e], s0["angle"][e] * 180.0 / 3.141592653589793),
                 (s1["pos_x"][e], s1["pos_z"][e], s1["angle"][e] * 180.0 / 3.141592653589793))
    src = fwd = None
    if fisheye if fisheye is not None else env.distortion:
        m = model_of(env, e)
        src, fwd = fo.src_of_lut(m.rmapx, m.rmapy), (m.mapx, m.mapy)
    return fo.flow(depth, labels, P, Vp, Vc, md.grid_w * md.grid_h, len(md.objects), moves, agent, src, fwd)


def compare(dev, orc, what):
    f, amb = orc["flow"], orc["ambiguous"]
    nd, no = np.isnan(dev).any(-1), np.isnan(f).any(-1)
    assert np.isnan(dev).all(-1)[nd].all(), f"{what}: a pixel with one NaN component"
    assert np.array_equal(nd[~amb], no[~amb]), f"{what}: NaN pattern differs at {np.argwhere((nd != no) & ~amb)[:5]}"
    both = ~nd & ~no & ~amb
    err = np.abs(dev[both].astype(np.float64) - f[both])
    bar = np.maximum(2.0 ** -10, 1e-5 * np.abs(f[both]))
    assert (err <= bar).all(), f"{what}: max error {err.max():.3g} px (flow {np.abs(f[both]).max():.3g})"
    return int(both.sum()), int(amb.sum())


CASES = [(m, "pinhole") for m in MAPS] + [
    ("udem1", "fisheye"), ("loop_dyn_duckiebots", "fisheye"), ("loop_pedestrians", "camera_rand"),
    ("small_loop", "camera_rand"), ("loop_dyn_duckiebots", "top_down"), ("loop_pedestrians", "top_down"),
    ("udem1", "top_down"), ("udem1", "segment"), ("loop_obstacles", "segment"),
    (("small_loop", "loop_dyn_duckiebots"), "pinhole")]


@pytest.mark.parametrize("names,view", CASES)
def test_rollout_against_the_oracle(torch_cuda, names, view):
    torch = torch_cuda
    n = 4
    kw = dict(distortion=view in ("fisheye", "camera_rand"), camera_rand=view == "camera_rand")
    if view == "camera_rand":
        kw["camera_rand_pool"] = 4
    if isinstance(names, tuple):
        kw["cycle_maps"] = True
    env = make_env(n, names, **kw)
    if isinstance(names, tuple):
        env.reset()   # (the second reset moves every other env to the next map)
    env.reset()
    mode = dict(top_down=view == "top_down", segment=view == "segment")
    step_renders = view in ("pinhole", "fisheye", "camera_rand")
    if not step_renders:
        env.render_obs(**mode)
    prev = frames(env)
    rng = np.random.default_rng(4)
    checked = ambiguous = 0
    for k in range(50):
        before = snap(env)
        act = torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=env.device)
        if step_renders:
            env.step(act)
        else:
            env.step(act, render=False)
            env.render_obs(**mode)
        after = snap(env)
        cur = frames(env)
        flow, dep, lab = (t.cpu().numpy() for t in (env.flow, env.depth, env.labels))
        for e in range(n):
            assert after[0]["episode"][e] == before[0]["episode"][e]
            Vp = cur[e][0] if view == "top_down" else prev[e][0]
            orc = oracle(env, e, before, after, Vp, cur[e][0], cur[e][1], dep[e], lab[e], top_down=view == "top_down")
            c, _ = compare(flow[e], orc, f"{names} {view} step {k} env {e}")
            amb = orc["ambiguous"]
            if env.distortion:   # a still point whose source is an edge pixel of the pinhole frame sits on the edge of
                # F's domain (every such pixel during the command delay after a reset): ambiguous, and expected so
                sx, sy = fo.src_of_lut(model_of(env, e).rmapx, model_of(env, e).rmapy)
                amb = amb & ~((sx == 0) | (sy == 0) | (sx == dep[e].shape[1] - 1) | (sy == dep[e].shape[0] - 1))
            checked, ambiguous = checked + c, ambiguous + int(amb.sum())
        prev = cur
    assert checked > 0.15 * 50 * n * dep[0].size   # (sky and the fisheye's black corners)
    assert ambiguous <= 1e-3 * checked


@pytest.mark.parametrize("names,view", [("loop_dyn_duckiebots", "pinhole"), ("loop_pedestrians", "pinhole"),
                                        ("udem1", "pinhole"), ("udem1", "fisheye"), ("loop_dyn_duckiebots", "top_down")])
def test_label_warp_on_device_frames(torch_cuda, names, view):
    """The label warp of tests/test_flow_oracle.py on consecutive device frames: the device's flow carries each pixel to
    one showing the same item in the previous frame (bars from that file)"""
    torch = torch_cuda
    n = 4
    env = make_env(n, names, w=160, h=120, distortion=view == "fisheye", domain_rand=False)
    env.reset()
    top = view == "top_down"
    if top:
        env.render_obs(top_down=True)
    prev = frames(env)
    rng = np.random.default_rng(9)
    hits = total = 0
    for k in range(20):
        dep0, lab0 = env.depth.cpu().numpy().copy(), env.labels.cpu().numpy().copy()
        before = snap(env)
        act = torch.as_tensor(np.c_[rng.uniform(0.3, 1, n), rng.uniform(-1, 1, n)], dtype=torch.float32,
                              device=env.device)
        if top:
            env.step(act, render=False)
            env.render_obs(top_down=True)
        else:
            env.step(act)
        after = snap(env)
        cur = frames(env)
        flow, dep, lab = (t.cpu().numpy() for t in (env.flow, env.depth, env.labels))
        for e in range(n):
            Vp = cur[e][0] if top else prev[e][0]
            orc = oracle(env, e, before, after, Vp, cur[e][0], cur[e][1], dep[e], lab[e], top_down=top)
            h, t = label_warp(flow[e], lab[e], lab0[e], dep0[e], orc["z_prev"])
            hits, total = hits + h, total + t
        prev = cur
    assert total > 20000
    assert hits >= LABEL_BAR[view == "fisheye"] * total, f"label warp: {hits} of {total}"


def test_zero_motion(torch_cuda):
    """An env whose pose and obstacles did not change bit for bit across a step: its static items' flow is 0 to 1e-4
    px; in top-down views the ground and tiles' flow is 0 to 1e-4 px in every env"""
    torch = torch_cuda
    n = 16
    env = make_env(n, "small_loop")
    env.reset()
    before = snap(env)
    env.step(torch.zeros((n, 2), dtype=torch.float32, device=env.device))
    after = snap(env)
    still = [e for e in range(n) if all(before[0][k][e] == after[0][k][e] for k in ("pos_x", "pos_z", "angle"))]
    assert still, "a zero command from rest moved every env"
    flow, lab = env.flow.cpu().numpy(), env.labels.cpu().numpy()
    n_tiles = env.maps[0].grid_w * env.maps[0].grid_h
    for e in still:
        static = (lab[e] >= 1) & (lab[e] <= 1 + n_tiles)
        assert static.sum() > 0
        assert np.abs(flow[e][static]).max() <= 1e-4
    env.step(torch.full((n, 2), 0.8, dtype=torch.float32, device=env.device), render=False)
    env.render_obs(top_down=True)
    flow, lab = env.flow.cpu().numpy(), env.labels.cpu().numpy()
    ground = (lab >= 1) & (lab <= 1 + n_tiles)
    assert ground.sum() > 0
    assert np.abs(flow[ground]).max() <= 1e-4


def test_first_frames_are_nan(torch_cuda):
    torch = torch_cuda
    for device_reset in (False, True):
        env = make_env(4, "loop_obstacles", device_reset=device_reset)
        env.reset()
        assert np.isnan(env.flow.cpu().numpy()).all()
        env.step(torch.full((4, 2), 0.5, dtype=torch.float32, device=env.device))
        assert not np.isnan(env.flow.cpu().numpy()).all()
        env.reset()
        assert np.isnan(env.flow.cpu().numpy()).all()


def test_auto_reset_rows(torch_cuda):
    """Respawned rows are NaN; the others carry the step's flow.  After step_terminal, flow rows match obs rows."""
    torch = torch_cuda
    for terminal in (False, True):
        n = 32
        env = make_env(n, "small_loop", auto_reset=True, device_reset=True, max_steps=6, terminal_obs=terminal)
        env.reset()
        rng = np.random.default_rng(2)
        seen = 0
        for k in range(14):
            ep0 = env.state["episode"].cpu().numpy().copy()
            act = torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=env.device)
            env.step(act)
            ep1 = env.state["episode"].cpu().numpy()
            flow, dep = env.flow.cpu().numpy(), env.depth.cpu().numpy()
            for e in range(n):
                if ep1[e] != ep0[e]:
                    assert np.isnan(flow[e]).all()
                    seen += 1
                else:
                    assert (~np.isnan(flow[e][..., 0])).sum() >= 0.3 * (dep[e] > 0).sum()
        assert seen > 0


def test_load_state_and_copy_envs_forget_the_previous_frame(torch_cuda):
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_dyn_duckiebots")
    env.reset()
    act = torch.full((n, 2), 0.6, dtype=torch.float32, device=env.device)
    env.step(act)
    rec = env.save_state()
    env.step(act)
    env.load_state(rec)
    env.render_obs()
    assert np.isnan(env.flow.cpu().numpy()).all()
    env.step(act)
    assert not np.isnan(env.flow.cpu().numpy()).all()
    env.copy_envs([0] * n)
    env.render_obs()
    assert np.isnan(env.flow.cpu().numpy()).all()
    env.step(act)
    assert not np.isnan(env.flow.cpu().numpy()).all()


def test_renders_after_a_step(torch_cuda):
    """render_obs() after a step gives the step's flow bytes; after step(render=False) it gives that step's flow"""
    torch = torch_cuda
    n = 4
    a, b = make_env(n, "loop_pedestrians"), make_env(n, "loop_pedestrians")
    a.reset(), b.reset()
    rng = np.random.default_rng(6)
    for k in range(5):
        act = torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=a.device)
        a.step(act)
        fa = a.flow.cpu().numpy().copy()
        a.render_obs()
        assert np.array_equal(a.flow.cpu().numpy().view(np.uint32), fa.view(np.uint32))
        b.step(act, render=False)
        b.render_obs()
        assert np.array_equal(b.flow.cpu().numpy().view(np.uint32), fa.view(np.uint32))


def test_resize_and_output_format_leave_flow_unchanged(torch_cuda):
    torch = torch_cuda
    n = 4
    a, b = make_env(n, "udem1"), make_env(n, "udem1")
    b.set_resize(84, 84).set_output_format(obs_layout="chw", obs_dtype="float32")
    a.reset(), b.reset()
    rng = np.random.default_rng(7)
    for k in range(4):
        act = torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=a.device)
        a.step(act), b.step(act)
        assert np.array_equal(a.flow.cpu().numpy().view(np.uint32), b.flow.cpu().numpy().view(np.uint32))


def test_refusals_leave_the_previous_setting(torch_cuda):
    from gym_duckietown_b200 import lib as L
    torch = torch_cuda
    n = 2
    plain = make_env(n, "small_loop", flow=False, depth=True)
    buf = torch.zeros((n, 72, 96, 2), dtype=torch.float32, device=plain.device)
    with pytest.raises(L.DtsError):   # no label target
        plain.sim.set_flow_target(buf.data_ptr())
    env = make_env(n, "small_loop", distortion=True)
    twin = make_env(n, "small_loop", distortion=True)
    m = env.camera_model
    with pytest.raises(L.DtsError):   # two forward maps for a pool of one table
        env.sim.set_flow_target(env.flow.data_ptr(), np.stack([m.mapx] * 2), np.stack([m.mapy] * 2))
    with pytest.raises(L.DtsError):   # the flow image reads the depth and label images
        env.sim.set_depth_target(None)
    with pytest.raises(L.DtsError):
        env.sim.set_label_target(None)
    with pytest.raises(ValueError):   # the rectification has no forward map
        env.set_rectification(m.mapx, m.mapy)
    act = torch.full((n, 2), 0.7, dtype=torch.float32, device=env.device)
    for e_ in (env, twin):
        e_.reset()
        e_.step(act)
    assert not np.isnan(env.flow.cpu().numpy()).all()
    assert np.array_equal(env.flow.cpu().numpy().view(np.uint32), twin.flow.cpu().numpy().view(np.uint32))
    assert np.array_equal(env.obs.cpu().numpy(), twin.obs.cpu().numpy())


def test_flow_changes_no_other_output_and_launches_only_k_flow(torch_cuda):
    torch = torch_cuda
    n = 4
    kw = dict(depth=True, labels=True, markings=True, bev=True)
    on, off = make_env(n, "loop_dyn_duckiebots", **kw), make_env(n, "loop_dyn_duckiebots", flow=False, **kw)
    rng = np.random.default_rng(8)
    for e_ in (on, off):
        e_.reset()
    c_on, c_off = on.launch_count(), off.launch_count()
    for k in range(6):
        act = torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=on.device)
        for e_ in (on, off):
            e_.step(act)
        for name in ("obs", "depth", "labels", "markings", "bev_labels", "bev_markings"):
            x, y = getattr(on, name).cpu().numpy(), getattr(off, name).cpu().numpy()
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    # per step, k_flow_record before k_step_logic and k_flow after the rasterisers, nothing else
    assert on.launch_count() - c_on == off.launch_count() - c_off + 2 * 6
    recs = on.save_state()
    c_on = on.launch_count()
    on.load_state(recs)
    assert on.launch_count() - c_on == 2   # the load and the record's invalidation
