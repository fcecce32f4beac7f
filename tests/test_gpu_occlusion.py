"""The occlusion mask on the device (dts_set_occlusion_target, DESIGN.md section 5 item 14) against the float64 oracle
(tests/occlusion_oracle.py), fed with the device's own flow oracle inputs and its own previous depth and labels: every
pixel takes one of the oracle's answers, and only ambiguous pixels have more than one.  Over 50-step rollouts with
random actions and domain randomisation on every map, pinhole, fisheye, a camera_rand pool, top-down and segment
views and a two-map batch.  Also: the slots' lifecycle (resets, repeats, unrendered steps, other views between steps,
auto-reset, terminal frames, loads, map uploads), refused calls, that the mask changes no other output, and its
launches."""
import numpy as np
import pytest

import flow_oracle as fo
import occlusion_oracle as oo
from test_gpu_flow import CASES, frames, model_of, oracle, snap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, names, w=96, h=72, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=True, seed=11, flow_occlusion=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def host(env):
    return tuple(t.cpu().numpy().copy() for t in (env.flow_occlusion, env.flow, env.depth, env.labels))


def actions(torch, rng, n, device):
    return torch.as_tensor(rng.uniform(-1, 1, (n, 2)), dtype=torch.float32, device=device)


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
        env.reset()
    env.reset()
    mode = dict(top_down=view == "top_down", segment=view == "segment")
    step_renders = view in ("pinhole", "fisheye", "camera_rand")
    if not step_renders:
        env.render_obs(**mode)
    prev = frames(env)
    rng = np.random.default_rng(4)
    checked = ambiguous = 0
    seen = np.zeros(5, np.int64)
    for k in range(50):
        before = snap(env)
        _, _, dep0, lab0 = host(env)   # the frame of the state the step starts from, in this view
        if step_renders:
            env.step(actions(torch, rng, n, env.device))
        else:
            env.step(actions(torch, rng, n, env.device), render=False)
            env.render_obs(**mode)
        after = snap(env)
        cur = frames(env)
        occ, flow, dep, lab = host(env)
        for e in range(n):
            md = env.maps[int(after[0]["map_id"][e])]
            Vp = cur[e][0] if view == "top_down" else prev[e][0]
            fl = oracle(env, e, before, after, Vp, cur[e][0], cur[e][1], dep[e], lab[e], top_down=view == "top_down")
            r = oo.occlusion(fl, lab[e], md.grid_w * md.grid_h, dep0[e], lab0[e])
            ok = ((r["allowed"] >> occ[e]) & 1) == 1
            where = f"{names} {view} step {k} env {e}"
            assert ok.all(), f"{where}: {np.argwhere(~ok)[:5]} device {occ[e][~ok][:5]} oracle {r['mask'][~ok][:5]}"
            amb = r["ambiguous"]
            if env.distortion:   # still points on the edge of F's domain: ambiguous flow, and expected so
                sx, sy = fo.src_of_lut(model_of(env, e).rmapx, model_of(env, e).rmapy)
                amb = amb & ~((sx == 0) | (sy == 0) | (sx == dep[e].shape[1] - 1) | (sy == dep[e].shape[0] - 1))
            checked += int((~np.isnan(fl["flow"][..., 0])).sum())
            ambiguous += int(amb.sum())
            seen += np.bincount(occ[e].ravel(), minlength=5)
        prev = cur
    assert seen[oo.UNKNOWN] == 0   # every step's previous frame was rendered in this view
    assert seen[oo.VISIBLE] > 0.5 * checked
    assert ambiguous <= 2e-3 * checked, (ambiguous, checked)


def test_reset_gives_none_and_render_obs_repeats(torch_cuda):
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_pedestrians")
    env.reset()
    assert (host(env)[0] == oo.NONE).all()
    rng = np.random.default_rng(6)
    for k in range(5):
        env.step(actions(torch, rng, n, env.device))
        m = host(env)[0]
        assert (m != oo.UNKNOWN).all() and (m == oo.VISIBLE).any()
        env.render_obs()
        assert np.array_equal(host(env)[0], m)


def test_unrendered_step_makes_the_next_one_unknown(torch_cuda):
    torch = torch_cuda
    n = 4
    env = make_env(n, "udem1")
    env.reset()
    rng = np.random.default_rng(3)
    env.step(actions(torch, rng, n, env.device), render=False)
    env.step(actions(torch, rng, n, env.device))
    occ, flow, _, _ = host(env)
    defined = ~np.isnan(flow[..., 0])
    assert np.isin(occ[defined], [oo.OUTSIDE, oo.UNKNOWN]).all() and (occ == oo.UNKNOWN).any()
    env.step(actions(torch, rng, n, env.device))   # that step's frame was rendered: known again
    assert (host(env)[0] != oo.UNKNOWN).all()


def test_top_down_render_between_steps(torch_cuda):
    """A top-down render between two steps gives its own mask (unknown: no top-down frame was kept) and leaves the next
    step's mask as without it"""
    torch = torch_cuda
    n = 4
    a, b = make_env(n, "loop_dyn_duckiebots"), make_env(n, "loop_dyn_duckiebots")
    a.reset(), b.reset()
    rng = np.random.default_rng(5)
    for k in range(4):
        act = actions(torch, rng, n, a.device)
        a.step(act), b.step(act)
        a.render_obs(top_down=True)
        occ, flow, _, _ = host(a)
        assert np.isin(occ[~np.isnan(flow[..., 0])], [oo.OUTSIDE, oo.UNKNOWN]).all()
        act = actions(torch, rng, n, a.device)
        a.step(act), b.step(act)
        assert np.array_equal(host(a)[0], host(b)[0])


def test_auto_reset_and_terminal_rows(torch_cuda):
    """Respawned rows are NONE; their next step has a mask, as the respawned frame was kept"""
    torch = torch_cuda
    for terminal in (False, True):
        n = 32
        env = make_env(n, "small_loop", auto_reset=True, device_reset=True, max_steps=6, terminal_obs=terminal)
        env.reset()
        rng = np.random.default_rng(2)
        respawned = 0
        for k in range(14):
            ep0 = env.state["episode"].cpu().numpy().copy()
            env.step(actions(torch, rng, n, env.device))
            ep1 = env.state["episode"].cpu().numpy()
            occ, flow, _, _ = host(env)
            assert (occ != oo.UNKNOWN).all()
            for e in range(n):
                if ep1[e] != ep0[e]:
                    assert (occ[e] == oo.NONE).all()
                    respawned += 1
                else:
                    assert np.array_equal(occ[e] == oo.NONE, np.isnan(flow[e][..., 0]))
        assert respawned > 0


@pytest.mark.parametrize("how", ["load_state", "copy_envs", "map_upload"])
def test_loads_and_map_uploads_empty_the_slots(torch_cuda, how):
    """Each forgets the envs' previous frames: right after it a render gives NONE and keeps its frame for the next step;
    a step without that render finds no frame of its starting state (UNKNOWN), although one was rendered before"""
    torch = torch_cuda
    n = 4
    env = make_env(n, "loop_dyn_duckiebots")
    env.reset()
    act = torch.full((n, 2), 0.6, dtype=torch.float32, device=env.device)
    env.step(act)
    if how == "load_state":
        env.load_state(env.save_state())   # the very state whose frame a slot holds
    elif how == "copy_envs":
        env.copy_envs(list(range(n)))
    else:
        env.sim.upload_map(0, env.maps[0])
    env.render_obs()
    assert (host(env)[0] == oo.NONE).all()   # (no flow record either)
    env.step(act)   # its previous frame is the render after the load
    assert (host(env)[0] != oo.UNKNOWN).all() and (host(env)[0] == oo.VISIBLE).any()
    env.step(act)
    if how == "load_state":
        env.load_state(env.save_state())
    elif how == "copy_envs":
        env.copy_envs(list(range(n)))
    else:
        env.sim.upload_map(0, env.maps[0])
    env.step(act)
    occ, flow, _, _ = host(env)
    assert np.isin(occ[~np.isnan(flow[..., 0])], [oo.OUTSIDE, oo.UNKNOWN]).all()


def test_refusals_leave_the_previous_setting(torch_cuda):
    from gym_duckietown_b200 import lib as L
    torch = torch_cuda
    n = 2
    plain = make_env(n, "small_loop", flow_occlusion=False, depth=True, labels=True)
    buf = torch.zeros((n, 72, 96), dtype=torch.uint8, device=plain.device)
    with pytest.raises(L.DtsError):   # no flow target
        plain.sim.set_occlusion_target(buf.data_ptr())
    env, twin = make_env(n, "small_loop"), make_env(n, "small_loop")
    with pytest.raises(L.DtsError):   # the mask is taken with the flow image
        env.sim.set_flow_target(None)
    act = torch.full((n, 2), 0.7, dtype=torch.float32, device=env.device)
    for e_ in (env, twin):
        e_.reset()
        e_.step(act)
        e_.step(act)
    assert (host(env)[0] == oo.VISIBLE).any()
    for a, b in zip(host(env), host(twin)):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    # off, then on again: the slots start empty, so the first step has flow but no previous frame
    env.sim.set_occlusion_target(None)
    env.sim.set_flow_target(None)
    env.step(act)
    env.sim.set_flow_target(env.flow.data_ptr())
    env.sim.set_occlusion_target(env.flow_occlusion.data_ptr())
    env.step(act)
    occ, flow, _, _ = host(env)
    assert np.isin(occ[~np.isnan(flow[..., 0])], [oo.OUTSIDE, oo.UNKNOWN]).all() and (occ == oo.UNKNOWN).any()
    env.step(act)   # against the frame the previous step kept
    m = host(env)[0]
    assert (m != oo.UNKNOWN).all() and (m == oo.VISIBLE).any()


def test_mask_changes_no_other_output_and_launches_only_k_occ_commit(torch_cuda):
    torch = torch_cuda
    n = 4
    kw = dict(depth=True, labels=True, markings=True, bev=True, flow=True)
    on = make_env(n, "loop_dyn_duckiebots", **kw)
    off = make_env(n, "loop_dyn_duckiebots", flow_occlusion=False, **kw)
    rng = np.random.default_rng(8)
    for e_ in (on, off):
        e_.reset()
    c_on, c_off = on.launch_count(), off.launch_count()
    for k in range(6):
        act = actions(torch, rng, n, on.device)
        for e_ in (on, off):
            e_.step(act)
        for name in ("obs", "depth", "labels", "markings", "flow", "bev_labels", "bev_markings"):
            x, y = getattr(on, name).cpu().numpy(), getattr(off, name).cpu().numpy()
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    assert on.launch_count() - c_on == off.launch_count() - c_off + 6   # k_occ_commit after every step's k_flow
    recs = on.save_state()
    c_on = on.launch_count()
    on.load_state(recs)
    assert on.launch_count() - c_on == 2   # the load and the record's and slots' invalidation
