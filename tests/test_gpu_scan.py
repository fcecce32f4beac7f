"""The range scan on the device (dts_set_scan_target, DESIGN.md section 5 item 16) against the float64 oracle
(tests/scan_oracle.py): range within 1e-5 m and hit exactly on every ray that is not ambiguous, and fewer than 1 % of
the rays ambiguous.  Cases: every map, 1 to 4096 rays, narrow and full fields of view, ranges from 5 cm to 20 m,
offset origins, a two-map batch, moving obstacles over 200 steps without rendering, hidden optional objects, auto-reset
with terminal frames, and the calls that change the state without a render.  Also: the scan changes no other output,
an unset target launches nothing, a refused configuration leaves the previous one in effect, and the single-env
adapter exposes it."""
import math

import numpy as np
import pytest

import scan_oracle as so
from test_gpu_bev import place, scene
from test_gpu_depth import poses_of
from test_gpu_fisheye import random_poses

pytestmark = pytest.mark.gpu

MAPS = ["loop_dyn_duckiebots", "loop_obstacles", "loop_only_duckies", "loop_pedestrians", "loop_trafficlights",
        "small_loop", "small_loop_only_duckies", "udem1"]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def scan_env(n, names, w=32, h=24, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, seed=5, scan=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def config_of(env):
    c = env.scan_config
    return (c.n_rays, c.fov, c.max_range, c.origin_forward, c.origin_right)


def expected(env):
    """The oracle's scans for every env's current state: its pose, map, hidden objects and obstacles' corners."""
    import torch
    from gym_duckietown_b200 import lib as L
    n = env.num_envs
    px, pz, ang = poses_of(env)
    mid = env.state["map_id"].cpu().numpy()
    hidden = np.stack([env.sim.debug_episode(e)["hidden"] for e in range(n)])
    dyn = {}
    for m in range(len(env.maps)):
        arr, nd = env.sim.dyn_state(m)
        if nd:
            a = torch.as_tensor(arr, device=env.device).cpu().numpy().reshape(L.DYN_FIELDS, nd, n)
            dyn[m] = a[L.DYN_CORNERS:L.DYN_CORNERS + 8]
    corners = [dyn[int(mid[e])][:, :, e].T.reshape(-1, 4, 2) if int(mid[e]) in dyn else None for e in range(n)]
    return so.scan_batch([scene(md) for md in env.maps], mid, px, pz, ang, config_of(env), corners, hidden)


def check_env(env, what):
    import torch
    torch.cuda.synchronize()
    want = expected(env)
    so.check(env.scan_range.cpu().numpy(), env.scan_hit.cpu().numpy(), want, what)
    return want


def objects_hit(env, want):
    n_cells = [md.grid_w * md.grid_h for md in env.maps]
    mid = env.state["map_id"].cpu().numpy()
    return sum(int((hit >= 2 + n_cells[int(mid[e])]).sum()) for e, (_, hit, _) in enumerate(want))


@pytest.mark.parametrize("name", MAPS)
def test_every_map_at_the_defaults(name, torch_cuda):
    """reset() and a render: the scans of 64 agents on random road points equal the oracle's."""
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    env = scan_env(64, name)
    assert tuple(env.scan_range.shape) == (64, 64) and env.scan_range.dtype == torch_cuda.float32
    assert env.scan_hit.dtype == torch_cuda.int16 and config_of(env) == (64, 2 * math.pi, 2.0, 0.0, 0.0)
    env.reset()
    place(env, *random_poses(md, 64, 17))
    env.render_obs()
    want = check_env(env, name)
    if md.objects:
        assert objects_hit(env, want) > 0, f"{name}: no ray met an object"
    assert (env.scan_hit >= 2).any()
    env.close()


@pytest.mark.parametrize("rays,fov,max_range,origin", [
    (1, 2 * math.pi, 2.0, (0.0, 0.0)), (7, 0.3, 0.05, (0.0, 0.0)), (64, 2 * math.pi, 20.0, (0.1, -0.05)),
    (360, 2 * math.pi, 3.0, (0.0, 0.0)), (4096, 2 * math.pi, 1.0, (-0.2, 0.3)), (64, 1e-3, 5.0, (0.0, 0.0)),
    (7, 2 * math.pi, 0.5, (0.0, 0.0)), (360, 1.5, 20.0, (0.05, 0.0)),
])
def test_configurations(rays, fov, max_range, origin, torch_cuda):
    """udem1 and loop_obstacles, 48 agents each, after reset(render=False) + render_scan()."""
    from gym_duckietown_b200 import maps
    for name in ("udem1", "loop_obstacles"):
        md = maps.load_map(name)
        env = scan_env(48, name, scan_rays=rays, scan_fov=fov, scan_range=max_range, scan_origin=origin)
        env.reset(render=False)
        place(env, *random_poses(md, 48, 23))
        env.scan_range.fill_(-7); env.scan_hit.fill_(-7)
        env.render_scan()
        check_env(env, f"{name} {rays} rays fov {fov} range {max_range} origin {origin}")
        env.close()


def test_batch_of_two_maps(torch_cuda):
    from gym_duckietown_b200 import maps
    names = ["loop_obstacles", "udem1"]
    mds = [maps.load_map(n) for n in names]
    env = scan_env(64, names, scan_rays=90, scan_range=3.0)
    mid = (np.arange(64) % 2).astype(np.int32)
    P = np.zeros((64, 3))
    for m in range(2):
        k = np.flatnonzero(mid == m)
        P[k] = np.stack(random_poses(mds[m], len(k), 50 + m), axis=1)
    place(env, P[:, 0], P[:, 1], P[:, 2], mid)
    env.render_scan()
    want = check_env(env, "two maps")
    assert objects_hit(env, want) > 0
    env.close()


@pytest.mark.parametrize("name", ["loop_dyn_duckiebots", "loop_pedestrians"])
def test_moving_obstacles_over_200_steps_without_rendering(name, torch_cuda):
    """Device resets and auto-reset, step(render=False) for 200 steps: every 10th step's scans equal the oracle's with
    the obstacles' corners where dts_get_dyn_state has them."""
    torch = torch_cuda
    env = scan_env(32, name, device_reset=True, auto_reset=True, max_steps=80, scan_range=4.0)
    env.reset(render=False)
    env.render_scan()
    check_env(env, f"{name} reset")
    g = torch.Generator(device="cuda").manual_seed(7)
    seen, first = 0, env.scan_range.clone()
    for t in range(200):
        a = torch.rand((32, 2), device="cuda", generator=g)
        a[:, 0] = 0.1 + 0.4 * a[:, 0]
        a[:, 1] = a[:, 1] * 2 - 1
        env.scan_range.fill_(-7)
        env.step(a, render=False)
        if t % 10 == 9:
            want = check_env(env, f"{name} step {t}")
            seen += objects_hit(env, want)
    assert seen > 0 and not torch.equal(first, env.scan_range)
    env.close()


def test_hidden_optional_objects_under_domain_rand(torch_cuda):
    env = scan_env(64, "udem1", domain_rand=True, device_reset=True, scan_range=6.0)
    env.reset()
    hidden = np.stack([env.sim.debug_episode(e)["hidden"] for e in range(64)])
    assert hidden.any(), "no env hid an optional object"
    check_env(env, "domain_rand")
    env.close()


def test_step_terminal_rows_are_the_respawned_state(torch_cuda):
    torch = torch_cuda
    env = scan_env(32, "loop_obstacles", domain_rand=True, device_reset=True, auto_reset=True, terminal_obs=True,
                   max_steps=5)
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(3)
    ended = 0
    for t in range(12):
        a = torch.rand((32, 2), device="cuda", generator=g)
        env.scan_range.fill_(-7)
        _, _, done, _ = env.step(a, render=t % 3 != 2)
        check_env(env, f"terminal step {t}")
        ended += int(done.sum())
    assert ended >= 32
    env.close()


def test_render_scan_after_reset_load_state_and_copy_envs(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map("udem1")
    env = scan_env(16, "udem1", device_reset=True)
    env.reset(render=False)
    env.render_scan()
    check_env(env, "reset(render=False)")
    saved = env.save_state()
    first = env.scan_range.clone(), env.scan_hit.clone()
    place(env, *random_poses(md, 16, 99))
    env.render_scan()
    check_env(env, "moved")
    env.load_state(saved)
    env.render_scan()
    assert torch.equal(env.scan_range, first[0]) and torch.equal(env.scan_hit, first[1])
    src = torch.tensor([3] * 8 + [-1] * 8)
    before = env.scan_range.clone()
    env.copy_envs(src)
    env.render_scan()
    assert torch.equal(env.scan_range[:8], before[3].expand(8, -1))
    assert torch.equal(env.scan_range[8:], before[8:])
    check_env(env, "copy_envs")
    env.close()


def test_scan_changes_no_other_output_and_an_unset_target_launches_nothing(torch_cuda):
    """obs, reward, done, depth, labels and the bird's-eye grids are the same bits with the scan on and off; a step
    launches one kernel more with it on, and with it off the tensors are not written."""
    torch = torch_cuda
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    kw = dict(camera_width=160, camera_height=120, domain_rand=True, seed=4, device_reset=True, auto_reset=True,
              depth=True, labels=True, bev=True, max_steps=8)
    env, plain = BatchedDuckietownEnv(32, "udem1", scan=True, **kw), BatchedDuckietownEnv(32, "udem1", **kw)
    assert plain.scan_range is None and plain.scan_hit is None
    env.reset(); plain.reset()
    g = torch.Generator(device="cuda").manual_seed(5)
    for t in range(10):
        a = torch.rand((32, 2), device="cuda", generator=g)
        n0, p0 = env.launch_count(), plain.launch_count()
        out = env.step(a, render=t % 4 != 3)
        ref = plain.step(a, render=t % 4 != 3)
        torch.cuda.synchronize()
        assert env.launch_count() - n0 == plain.launch_count() - p0 + 1
        for x, y in zip(out[:3], ref[:3]):
            assert torch.equal(x, y), f"step {t}"
        for name in ("depth", "labels", "bev_labels", "bev_markings"):
            assert torch.equal(getattr(env, name).view(torch.uint8), getattr(plain, name).view(torch.uint8)), (name, t)
    env.sim.set_scan_target(None, None, None)
    env.scan_range.fill_(-7); env.scan_hit.fill_(77)
    n0, p0 = env.launch_count(), plain.launch_count()
    a = torch.rand((32, 2), device="cuda", generator=g)
    env.step(a); plain.step(a)
    env.step(a, render=False); plain.step(a, render=False)
    env.render_obs(); plain.render_obs()
    torch.cuda.synchronize()
    assert env.launch_count() - n0 == plain.launch_count() - p0
    assert (env.scan_range == -7).all() and (env.scan_hit == 77).all()
    with pytest.raises(Exception):
        env.render_scan()
    env.close(); plain.close()


def test_refused_configurations_leave_the_previous_one(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    env = scan_env(8, "udem1", device_reset=True)
    env.reset(render=False)
    env.render_scan()
    good = env.scan_range.clone(), env.scan_hit.clone()
    rp, hp = env.scan_range.data_ptr(), env.scan_hit.data_ptr()
    nan, inf = float("nan"), float("inf")
    bad = [L.ScanConfig(0, 1.0, 2.0, 0, 0), L.ScanConfig(4097, 1.0, 2.0, 0, 0), L.ScanConfig(64, 0.0, 2.0, 0, 0),
           L.ScanConfig(64, -1.0, 2.0, 0, 0), L.ScanConfig(64, 2 * math.pi + 1e-9, 2.0, 0, 0),
           L.ScanConfig(64, nan, 2.0, 0, 0), L.ScanConfig(64, 1.0, 0.0, 0, 0), L.ScanConfig(64, 1.0, -2.0, 0, 0),
           L.ScanConfig(64, 1.0, inf, 0, 0), L.ScanConfig(64, 1.0, nan, 0, 0), L.ScanConfig(64, 1.0, 2.0, nan, 0),
           L.ScanConfig(64, 1.0, 2.0, 0, inf)]
    for cfg in bad:
        with pytest.raises(L.DtsError):
            env.sim.set_scan_target(cfg, rp, hp)
    with pytest.raises(L.DtsError):
        env.sim.set_scan_target(L.ScanConfig(64, 1.0, 2.0, 0, 0), rp + 2, hp)   # range not 4-byte aligned
    with pytest.raises(L.DtsError):
        env.sim.set_scan_target(L.ScanConfig(64, 1.0, 2.0, 0, 0), rp, hp + 1)   # hit not 2-byte aligned
    env.scan_range.fill_(-7); env.scan_hit.fill_(77)
    env.render_scan()
    assert torch.equal(env.scan_range, good[0]) and torch.equal(env.scan_hit, good[1])
    env.close()


def test_single_env_adapter_exposes_the_scan(torch_cuda):
    from gym_duckietown_b200.simulator import DuckietownEnv
    e = DuckietownEnv(map_name="loop_obstacles", domain_rand=False, camera_width=32, camera_height=24, seed=4, scan=True,
                      scan_rays=90)
    for step in range(3):
        if step:
            e.step(np.array([0.4, 0.2]))
        r, h = e.scan_range, e.scan_hit
        assert r.shape == (90,) and r.dtype == np.float32 and h.shape == (90,) and h.dtype == np.int16
        so.check(r[None], h[None], expected(e._b), f"adapter step {step}")
    e.close()
