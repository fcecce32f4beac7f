"""The navigation task on the device (DTS_FLAG_NAV, DESIGN.md §6c): goal draws against the reference's own
DuckietownNav.reset (tests/golden/nav_<map>.npz), the arrival test inside the step kernel, auto-reset rollouts against
the CPU oracle with the host sampler's resets, snapshots, and the refusals."""
import copy
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATIC_MAPS = ["small_loop", "loop_obstacles", "udem1"]
MAPS = STATIC_MAPS + ["loop_dyn_duckiebots"]
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(name, n, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=32, camera_height=24, domain_rand=False, seed=0, nav=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, name, **args)


def stream_rows(env):
    return np.array([[s["state"]["state"] >> 64, s["state"]["state"] & M64, s["has_uint32"], s["uinteger"]]
                     for s in env.sim.debug_streams()], np.uint64)


def host(env, torch):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in env.state.items()}


def check_resets(env, g, tag, torch, streams=True):
    n = env.num_envs
    for ep in range(2):
        env.reset(render=False)
        s = host(env, torch)
        rows = np.arange(n) * 2 + ep
        assert np.array_equal(s["pos_x"], g[f"{tag}_cur_pos"][rows, 0]), (tag, ep)
        assert np.array_equal(s["pos_z"], g[f"{tag}_cur_pos"][rows, 2]), (tag, ep)
        assert np.array_equal(s["angle"], g[f"{tag}_cur_angle"][rows]), (tag, ep)
        assert np.array_equal(env.goal_tile.cpu().numpy(), g[f"{tag}_goal"][rows]), (tag, ep)
        if streams:
            assert np.array_equal(stream_rows(env), g[f"{tag}_stream"][rows]), (tag, ep)


@pytest.mark.parametrize("name", MAPS)
@pytest.mark.parametrize("dr", [False, True])
@pytest.mark.parametrize("device_reset", [True, False])
def test_goal_draws_match_reference(name, dr, device_reset, golden_dir, torch_cuda):
    """dts_reset_random draws the goal on the device; a host reset draws it in EpisodeSampler and hands it over with
    dts_set_goals.  Both equal the reference's DuckietownNav.reset for the same seeds, and the device stream stands where
    the reference's does afterwards."""
    g = np.load(os.path.join(golden_dir, f"nav_{name}.npz"))
    tag = "dr" if dr else "nodr"
    env = make_env(name, len(g["seeds"]), domain_rand=dr, device_reset=device_reset)
    try:
        check_resets(env, g, tag, torch_cuda, streams=device_reset)
        if not device_reset:
            got = np.array([[s["state"]["state"] >> 64, s["state"]["state"] & M64, s["has_uint32"], s["uinteger"]]
                            for s in (r.bit_generator.state for r in env.sampler.rngs)], np.uint64)
            assert np.array_equal(got, g[f"{tag}_stream"][np.arange(len(g['seeds'])) * 2 + 1])
    finally:
        env.close()


@pytest.mark.parametrize("device_reset", [True, False])
def test_goal_draws_after_fixed_starts_match_reference(device_reset, golden_dir, torch_cuda):
    from gym_duckietown_b200 import maps
    g = np.load(os.path.join(golden_dir, "nav_udem1.npz"))
    base = maps.load_map("udem1")
    md_tile = copy.deepcopy(base); md_tile.start_tile = tuple(int(v) for v in g["start_tile"])
    md_pose = copy.deepcopy(md_tile)
    sp = g["start_pose"]
    md_pose.start_pose = [[float(sp[0]), float(sp[1]), float(sp[2])], float(sp[3])]
    cases = {"user": (base, dict(user_tile_start=tuple(int(v) for v in g["user_tile_start"]))),
             "tile": (md_tile, {}), "pose": (md_pose, {})}
    for tag, (md, kw) in cases.items():
        env = make_env(md, 12, device_reset=device_reset, **kw)
        try:
            check_resets(env, g, tag, torch_cuda, streams=device_reset)
        finally:
            env.close()


@pytest.mark.parametrize("name", STATIC_MAPS)
@pytest.mark.parametrize("reward", ["raw", "dt"])
def test_arrival_in_the_step_kernel(name, reward, golden_dir, torch_cuda):
    """Agents placed at the fixture's poses and stepped with a zero action (they stay put): with nav, reward, done and
    done_code are exactly the nav-off step's with DuckietownNav.step's goal test on top, and equal the reference's
    DuckietownNav.step on every pose not on a tile edge."""
    torch = torch_cuda
    from test_nav import nav_done_reward
    g = np.load(os.path.join(golden_dir, f"nav_{name}.npz"))
    keep = g["step_count"] < 1500
    poses, want_r, want_d = g["step_poses"][keep], g["step_reward"][keep], g["step_done"][keep]
    n = len(poses)
    goal = g["step_goal"]
    outs = []
    for nav in (False, True):
        env = make_env(name, n, nav=nav)
        env.set_output_format(reward=reward)
        try:
            env.sim.reset(None, dict(pos_x=poses[:, 0], pos_z=poses[:, 1], angle=poses[:, 2]), env._stream())
            if nav:
                env.sim.set_goals(None, torch.from_numpy(np.tile(goal.astype(np.int16), (n, 1))).cuda().data_ptr(),
                                  env._stream())
                assert np.array_equal(env.goal_tile.cpu().numpy(), np.tile(goal, (n, 1)))
            _, rew, done, _ = env.step(torch.zeros((n, 2), device=env.device), render=False)
            s = host(env, torch)
            outs.append((rew.cpu().numpy().copy(), done.cpu().numpy().copy(), s))
        finally:
            env.close()
    (r0, d0, s0), (r1, d1, s1) = outs
    at = (s1["tile_i"] == goal[0]) & (s1["tile_j"] == goal[1])
    assert at.sum() > 10 and np.array_equal(s0["tile_i"], s1["tile_i"]) and np.array_equal(s0["tile_j"], s1["tile_j"])
    assert np.array_equal(d1, d0 | at)
    assert np.array_equal(s1["done_code"], np.where(at, 3, s0["done_code"]))
    assert np.array_equal(r1, np.where(at, np.float32(1010.0 if reward == "dt" else 1000.0), r0))
    assert np.array_equal(s1["reward"], np.where(at, 1000.0, s0["reward"]))
    # against the reference, away from tile edges (a zero-action step round-trips the pose through the cartesian frame)
    from gym_duckietown_b200 import maps
    ts = maps.load_map(name).tile_size
    frac = np.stack([poses[:, 0] / ts, poses[:, 1] / ts], 1) % 1.0
    inner = ((frac > 1e-9) & (frac < 1 - 1e-9)).all(1)
    assert np.array_equal(d1[inner], want_d[inner])
    if reward == "raw":
        assert np.allclose(s1["reward"][inner], want_r[inner], rtol=1e-5, atol=1e-5)


def rollout_case(torch, names, n, steps, frame_skip=1, reward="raw", terminal=False, seed=900):
    """Device auto-reset against the reference-style loop `step; if done: reset` built from the CPU oracle (step), the
    goal test, and the host sampler (resets: same numpy streams, nav on)."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.episode import EpisodeSampler
    from test_nav import nav_done_reward
    from test_reset_sampler import oracle_query
    names = [names] if isinstance(names, str) else names
    mds = [maps.load_map(m) for m in names]
    oms = [orc.OracleMap(md) for md in mds]
    rnd = len(names) > 1
    env = make_env(names if rnd else names[0], n, device_reset=True, auto_reset=True, max_steps=150, seed=seed,
                   frame_skip=frame_skip, randomize_maps_on_reset=rnd, terminal_obs=terminal)
    env.set_output_format(reward=reward)
    hs = EpisodeSampler(n, domain_rand=False, nav=True)
    hs.seed([seed + k for k in range(n)])
    mid = np.zeros(n, int)

    def host_reset(k):
        if rnd:
            mid[k] = int(hs.rngs[k].integers(0, len(names)))
        r = hs.sample([k], [mds[mid[k]]], oracle_query(mds[mid[k]]))
        return orc.OracleEnv(oms[mid[k]], r["pos_x"][0], r["pos_z"][0], r["angle"][0], wheel_dist=r["wheel_dist"][0],
                             max_steps=150, frame_skip=frame_skip), tuple(r["goal"][0]), r
    try:
        env.reset(render=False)
        cpu = [host_reset(k) for k in range(n)]
        goals = env.goal_tile.cpu().numpy()
        assert all(tuple(goals[k]) == cpu[k][1] for k in range(n))
        acts = np.random.default_rng(seed).uniform(-1, 1, (steps, n, 2)).astype(np.float32)
        acts[:, :, 0] = 0.3 + 0.7 * np.abs(acts[:, :, 0])   # drive on: episodes end at goals, off the road, max_steps
        acts[:, :, 1] *= 0.5
        codes = np.zeros(4, int)
        for t in range(steps):
            _, rew, done, _ = env.step(torch.from_numpy(acts[t]).to(env.device), render=terminal)
            s = host(env, torch)
            r32, d = rew.cpu().numpy(), done.cpu().numpy()
            goals = env.goal_tile.cpu().numpy()
            for k in range(n):
                o = cpu[k][0].step(acts[t, k])
                want_r, want_d, want_c = nav_done_reward(o, cpu[k][1])
                if reward == "dt":
                    want_r = -10.0 if want_r == -1000.0 else (want_r + 10 if want_r > 0 else want_r + 4)
                assert bool(d[k]) == want_d and s["done_code"][k] == want_c, (t, k)
                assert abs(r32[k] - want_r) <= 1e-5 * max(1.0, abs(want_r)), (t, k)
                codes[want_c] += 1
                if want_d:
                    cpu[k] = host_reset(k)
                    r = cpu[k][2]
                    assert s["pos_x"][k] == r["pos_x"][0] and s["angle"][k] == r["angle"][0], (t, k)
                    assert tuple(goals[k]) == cpu[k][1] and s["map_id"][k] == mid[k], (t, k)
        # the device streams stand where the host sampler's do
        assert np.array_equal(stream_rows(env), np.array(
            [[st["state"]["state"] >> 64, st["state"]["state"] & M64, st["has_uint32"], st["uinteger"]]
             for st in (g.bit_generator.state for g in hs.rngs)], np.uint64))
        return codes
    finally:
        env.close()


@pytest.mark.parametrize("case", [
    dict(names="small_loop", n=64, steps=300),
    dict(names="udem1", n=64, steps=300, frame_skip=2, reward="dt"),
    dict(names="loop_obstacles", n=48, steps=200, terminal=True),
    dict(names=["small_loop", "udem1"], n=48, steps=250),
    dict(names="small_loop", n=4096, steps=40, terminal=True),
])
def test_auto_reset_rollout_vs_oracle(case, torch_cuda):
    codes = rollout_case(torch_cuda, **case)
    assert codes[3] > 5 and codes[1] + codes[2] > 0, codes   # goals reached, and other endings too


def test_goal_reached_at_scale(torch_cuda):
    """4096 envs started just short of their goal: on the tile next to it, 2 mm from the edge they share, facing it,
    and driven straight on.  Every env's first episode ends at the goal (once the command delay has passed) with reward
    1000, and the next one starts in the same step with a new goal."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map("small_loop")
    n = 4096
    env = make_env("small_loop", n, device_reset=True, auto_reset=True, seed=3)
    try:
        env.reset(render=False)
        goals = env.goal_tile.cpu().numpy().astype(int)
        ts = md.tile_size
        drv = set(md.drivable_tiles)
        px, pz, ang = np.zeros(n), np.zeros(n), np.zeros(n)
        for k, (gi, gj) in enumerate(goals):   # a drivable 4-neighbour of the goal, 2 mm short of their shared edge
            for di, dj, a in ((-1, 0, 0.0), (1, 0, np.pi), (0, -1, -np.pi / 2), (0, 1, np.pi / 2)):
                if (gi + di, gj + dj) in drv:
                    break
            px[k] = (gi + 0.5) * ts + di * (0.5 * ts + 0.002)
            pz[k] = (gj + 0.5) * ts + dj * (0.5 * ts + 0.002)
            ang[k] = a
        env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang), env._stream())
        first = np.full(n, np.nan)
        goal_after = np.zeros((n, 2), int)
        acts = torch.tensor([[1.0, 0.0]] * n, device=env.device)
        for _ in range(30):
            _, rew, done, _ = env.step(acts, render=False)
            s, d, r, g = host(env, torch), done.cpu().numpy(), rew.cpu().numpy(), env.goal_tile.cpu().numpy()
            new = d & np.isnan(first)
            assert (s["step_count"][new] == 0).all()   # respawned in the same step
            first[new], goal_after[new] = r[new], g[new]
        assert (first == 1000).all(), np.unique(first, return_counts=True)
        assert (goal_after != goals).any(1).mean() > 0.5   # new goals
    finally:
        env.close()


def test_snapshots_resume_a_nav_run_bit_for_bit(torch_cuda):
    torch = torch_cuda
    n, t0, t1 = 96, 25, 60
    env = make_env("udem1", n, device_reset=True, auto_reset=True, seed=44, max_steps=80)
    try:
        env.reset(render=False)
        acts = torch.from_numpy(np.random.default_rng(1).uniform(0.2, 1, (t0 + t1, n, 2)).astype(np.float32)).cuda()
        for t in range(t0):
            env.step(acts[t], render=False)
        rec = env.save_state()

        def run():
            out = []
            for t in range(t0, t0 + t1):
                _, r, d, _ = env.step(acts[t], render=False)
                out.append((r.clone(), d.clone(), env.goal_tile, env.state["pos_x"].clone()))
            return out
        a = run()
        env.load_state(rec)
        b = run()
        for x, y in zip(a, b):
            for u, v in zip(x, y):
                assert torch.equal(u, v)
        assert any(x[1].any() for x in a)   # episodes ended, and respawned with new goals, in the resumed run
        # copy_envs carries the goal
        src = torch.arange(n).flip(0)
        g = env.goal_tile
        env.copy_envs(src)
        assert torch.equal(env.goal_tile, g.flip(0))
    finally:
        env.close()


def test_nav_off_runs_are_the_parents_byte_for_byte(golden_dir, torch_cuda):
    """Seeded runs without nav (device and host resets, auto-reset with terminal frames, domain and dynamics
    randomisation, moving obstacles, random maps): every frame, reward, done flag, terminal frame, stream and final
    state equal what the commit before DTS_FLAG_NAV recorded (tests/nav_off_baseline.py)."""
    from nav_off_baseline import record
    want = np.load(os.path.join(golden_dir, "nav_off_baseline.npz"))
    got = record()
    assert sorted(got) == sorted(want.files)
    bad = [k for k in want.files if not np.array_equal(got[k], want[k])]
    assert not bad, bad


def test_nav_off_keeps_the_goal_planes_zero_and_the_launch_counts(torch_cuda):
    torch = torch_cuda
    envs = [make_env("small_loop", 64, device_reset=True, auto_reset=True, seed=8, nav=nav) for nav in (False, True)]
    try:
        acts = torch.full((64, 2), 0.6, device="cuda")
        for e in envs:
            e.reset(render=False)
            for _ in range(50):
                e.step(acts, render=True)
        torch.cuda.synchronize()
        assert envs[0].launch_count() == envs[1].launch_count()
        off = envs[0].sim.goal_arrays()
        assert all(not torch.as_tensor(v, device="cuda").any() for v in off.values())
        assert envs[1].goal_tile.any()
        with pytest.raises(ValueError):
            envs[0].goal_tile
    finally:
        for e in envs:
            e.close()


def one_drivable(md):
    md = copy.deepcopy(md)
    keep = md.drivable_tiles[0]
    drv = np.zeros_like(md.tile_drivable)
    drv[keep[1] * md.grid_w + keep[0]] = 1
    md.tile_drivable, md.drivable_tiles = drv, [keep]
    return md


def wide(md, w=256):
    md = copy.deepcopy(md)
    pad = lambda a, v: np.concatenate([a.reshape(md.grid_h, md.grid_w),
                                       np.full((md.grid_h, w - md.grid_w), v, a.dtype)], 1).ravel()
    md.tile_kind, md.tile_angle, md.tile_drivable = pad(md.tile_kind, -1), pad(md.tile_angle, 0), pad(md.tile_drivable, 0)
    md.tile_curve_off, md.tile_curve_cnt = pad(md.tile_curve_off, 0), pad(md.tile_curve_cnt, 0)
    md.grid_w = w
    return md


def test_refusals(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200 import maps
    base = maps.load_map("small_loop")
    for bad in (one_drivable(base), wide(base)):
        with pytest.raises(L.DtsError, match="DTS_FLAG_NAV"):
            make_env(bad, 4)
        make_env(bad, 4, nav=False).close()   # the same maps without nav upload
    env = make_env("small_loop", 8, device_reset=True)
    try:
        env.reset(render=False)
        fp = env.state_fingerprint
        for bad in (one_drivable(base), wide(base)):   # a refused upload leaves the slot as it was
            with pytest.raises(L.DtsError, match="DTS_FLAG_NAV"):
                env.sim.upload_map(0, bad)
            assert env.state_fingerprint == fp
        env.reset(render=False)
        goals = torch.zeros((8, 2), dtype=torch.int16, device="cuda")
        with pytest.raises(L.DtsError, match="aligned"):
            env.sim.set_goals(None, goals.data_ptr() + 1, env._stream())
        # drivable goals are taken
        goals[:] = torch.tensor(base.drivable_tiles[-1], dtype=torch.int16)
        env.sim.set_goals(None, goals.data_ptr(), env._stream())
        assert torch.equal(env.goal_tile, goals) and env.sim.status() == 0
        env.step(torch.zeros((8, 2), device="cuda"), render=False)
    finally:
        env.close()
    # an entry off the grid or on a tile that is not drivable leaves that env's goal and sets status bit 2, after which
    # steps and renders fail
    undrivable = next((i, j) for j in range(base.grid_h) for i in range(base.grid_w)
                      if not base.tile_drivable[j * base.grid_w + i])
    for bad in ((base.grid_w, 0), (-1, 0), undrivable):
        env = make_env("small_loop", 8, device_reset=True)
        try:
            env.reset(render=False)
            before = env.goal_tile
            goals = torch.tensor([base.drivable_tiles[0]] * 8, dtype=torch.int16, device="cuda")
            goals[3] = torch.tensor(bad, dtype=torch.int16)
            env.sim.set_goals(None, goals.data_ptr(), env._stream())
            want = goals.clone()
            want[3] = before[3]
            assert torch.equal(env.goal_tile, want), bad
            torch.cuda.synchronize()
            assert env.sim.status() == 4
            with pytest.raises(L.DtsError, match="dts_set_goals met a goal"):
                env.step(torch.zeros((8, 2), device="cuda"), render=False)
        finally:
            env.close()
    plain = make_env("small_loop", 8, nav=False)
    try:
        goals = torch.zeros((8, 2), dtype=torch.int16, device="cuda")
        with pytest.raises(L.DtsError, match="without DTS_FLAG_NAV"):
            plain.sim.set_goals(None, goals.data_ptr(), plain._stream())
    finally:
        plain.close()


def test_simulator_nav_and_lf(torch_cuda):
    import gym_duckietown_b200 as gd
    sim = gd.DuckietownNav(map_name="small_loop", domain_rand=False, camera_width=32, camera_height=24, seed=5)
    try:
        g = sim.goal_tile
        assert g["coords"] in sim.drivable_tiles and g["coords"] != sim.get_grid_coords(sim.cur_pos) and g["drivable"]
        md = sim._b.maps[0]
        from gym_duckietown_b200.maps import TILE_KINDS
        assert g["kind"] == TILE_KINDS[int(md.tile_kind[g["coords"][1] * md.grid_w + g["coords"][0]])]
        for _ in range(5):
            obs, r, d, info = sim.step([0.3, 0.0])
            assert info["goal_tile"] == sim.goal_tile
    finally:
        sim.close()
    lf = gd.DuckietownLF(map_name="small_loop", domain_rand=False, camera_width=32, camera_height=24, seed=5)
    try:
        assert isinstance(lf, gd.DuckietownEnv) and not lf._b.nav
    finally:
        lf.close()
