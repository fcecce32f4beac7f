"""The bird's-eye map on the device (dts_set_bev_target, DESIGN.md section 5 item 12) against the float64 oracle
(tests/bev_oracle.py): every cell that is not ambiguous bit for bit, every ambiguous one equal to one of its answers,
and fewer than 1e-4 of the cells ambiguous.  Cases: every map, grid shapes from 1 x 1 to 2048 x 1, cells finer than a
texel and coarser than a tile, an origin off the grid, two-map batches, moving obstacles over 200 steps, hidden optional
objects, steps without rendering, auto-reset with terminal frames, and the calls that change the state without a
render.  Also: the agent's own cell names its tile, the grids change no other output, an unset target launches nothing
and writes nothing, and a refused configuration leaves the previous one in effect."""
import numpy as np
import pytest

import bev_oracle as bo
from test_gpu_depth import poses_of
from test_gpu_fisheye import random_poses

pytestmark = pytest.mark.gpu

_SCENES = {}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def scene(md):
    if md.name not in _SCENES:
        _SCENES[md.name] = bo.BevScene(md)
    return _SCENES[md.name]


def bev_env(n, names, shape=(64, 64), cell=0.03, origin=None, w=32, h=24, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, seed=5, bev=True, bev_shape=shape, bev_cell=cell,
                bev_origin=origin)
    args.update(kw)
    return BatchedDuckietownEnv(n, names, **args)


def config_of(env):
    c = env.bev_config
    return (c.width, c.height, c.cell, c.origin_x, c.origin_y)


def expected(env):
    """The oracle's grids for every env's current state: its pose, map, hidden objects and obstacles' corners."""
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
    return bo.bev_batch([scene(md) for md in env.maps], mid, px, pz, ang, config_of(env), corners, hidden)


def check_env(env, what):
    import torch
    torch.cuda.synchronize()
    want = expected(env)
    bo.check(env.bev_labels.cpu().numpy(), env.bev_markings.cpu().numpy(), want, what)
    return want


def place(env, px, pz, ang, map_id=None, **extra):
    n = env.num_envs
    p = dict(pos_x=np.asarray(px, float).copy(), pos_z=np.asarray(pz, float).copy(), angle=np.asarray(ang, float).copy(),
             map_id=np.zeros(n, np.int32) if map_id is None else np.asarray(map_id, np.int32))
    p.update(extra)
    env.sim.reset(None, p, env._stream())


def object_labels_seen(env, want):
    n_cells = [md.grid_w * md.grid_h for md in env.maps]
    mid = env.state["map_id"].cpu().numpy()
    return sum(int((lab >= 2 + n_cells[int(mid[e])]).sum()) for e, (lab, _, _, _) in enumerate(want))


@pytest.mark.parametrize("name", ["loop_dyn_duckiebots", "loop_obstacles", "loop_only_duckies", "loop_pedestrians",
                                  "loop_trafficlights", "small_loop", "small_loop_only_duckies", "udem1"])
def test_every_map_at_the_default_grid(name, torch_cuda):
    """reset() (host-drawn episodes, rendered): the grids of 64 agents on random road points equal the oracle's."""
    from gym_duckietown_b200 import maps
    assert name in maps.list_maps()
    md = maps.load_map(name)
    env = bev_env(64, name)
    assert tuple(env.bev_labels.shape) == (64, 64, 64) and env.bev_labels.dtype == torch_cuda.int16
    assert env.bev_markings.dtype == torch_cuda.uint8 and (env.bev_config.origin_x, env.bev_config.origin_y) == (32, 48)
    env.reset()
    px, pz, ang = random_poses(md, 64, 17)
    place(env, px, pz, ang)
    env.render_obs()
    want = check_env(env, name)
    if md.objects:
        assert object_labels_seen(env, want) > 0, f"{name}: no object in any grid"
    assert (env.bev_markings >= 2).any(), f"{name}: no paint in any grid"
    env.close()


@pytest.mark.parametrize("shape,cell,origin", [
    ((64, 64), 0.03, None), ((48, 96), 0.03, None), ((1, 1), 0.03, None), ((1, 2048), 0.03, None),
    ((64, 64), 0.001, None), ((16, 16), 0.8, None), ((64, 64), 0.03, (-10.0, 80.5)), ((2048, 1), 0.002, (0.5, 1000.0)),
])
def test_grid_configurations(shape, cell, origin, torch_cuda):
    """udem1, 48 agents, after reset(render=False) + render_bev(): non-square, 1 x 1, 2048 x 1 and 1 x 2048 grids, a
    cell smaller than a texel (1 mm; a texel is 2.3 mm), a cell larger than a tile, an origin outside the grid."""
    from gym_duckietown_b200 import maps
    md = maps.load_map("udem1")
    env = bev_env(48, "udem1", shape, cell, origin)
    env.reset(render=False)
    px, pz, ang = random_poses(md, 48, 23)
    place(env, px, pz, ang)
    env.bev_labels.fill_(-7)
    env.render_bev()
    check_env(env, f"{shape} cell {cell} origin {origin}")
    env.close()


def test_batch_of_two_maps(torch_cuda):
    from gym_duckietown_b200 import maps
    names = ["loop_obstacles", "udem1"]
    mds = [maps.load_map(n) for n in names]
    env = bev_env(64, names)
    mid = (np.arange(64) % 2).astype(np.int32)
    P = np.zeros((64, 3))
    for m in range(2):
        k = np.flatnonzero(mid == m)
        P[k] = np.stack(random_poses(mds[m], len(k), 50 + m), axis=1)
    place(env, P[:, 0], P[:, 1], P[:, 2], mid)
    env.render_bev()
    want = check_env(env, "two maps")
    assert object_labels_seen(env, want) > 0
    env.close()


@pytest.mark.parametrize("name", ["loop_dyn_duckiebots", "loop_pedestrians"])
def test_moving_obstacles_over_200_steps_without_rendering(name, torch_cuda):
    """Device resets and auto-reset, step(render=False) for 200 steps: every 10th step's grids equal the oracle's with
    the obstacles' corners where dts_get_dyn_state has them; an obstacle's label moves with it."""
    torch = torch_cuda
    env = bev_env(32, name, device_reset=True, auto_reset=True, max_steps=80)
    env.reset(render=False)
    env.render_bev()
    check_env(env, f"{name} reset")
    g = torch.Generator(device="cuda").manual_seed(7)
    seen, first = 0, env.bev_labels.clone()
    for t in range(200):
        a = torch.rand((32, 2), device="cuda", generator=g)
        a[:, 0] = 0.1 + 0.4 * a[:, 0]
        a[:, 1] = a[:, 1] * 2 - 1
        env.bev_labels.fill_(-7)
        env.step(a, render=False)
        if t % 10 == 9:
            want = check_env(env, f"{name} step {t}")
            seen += object_labels_seen(env, want)
    assert seen > 0 and not torch.equal(first, env.bev_labels)
    env.close()


def test_hidden_optional_objects_under_domain_rand(torch_cuda):
    """udem1 under domain_rand with device resets: some envs hide optional objects, and their grids skip them."""
    env = bev_env(64, "udem1", domain_rand=True, device_reset=True)
    env.reset()
    hidden = np.stack([env.sim.debug_episode(e)["hidden"] for e in range(64)])
    assert hidden.any(), "no env hid an optional object"
    check_env(env, "domain_rand")
    env.close()


def test_step_terminal_rows_are_the_respawned_state(torch_cuda):
    """terminal_obs under auto-reset (dts_step_terminal): after every step each row is the oracle's of the state obs
    shows, for ended envs their next episode's first state, with rendering and without."""
    torch = torch_cuda
    env = bev_env(32, "loop_obstacles", domain_rand=True, device_reset=True, auto_reset=True, terminal_obs=True,
                  max_steps=5)
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(3)
    ended = 0
    for t in range(12):
        a = torch.rand((32, 2), device="cuda", generator=g)
        env.bev_labels.fill_(-7)
        _, _, done, _ = env.step(a, render=t % 3 != 2)
        check_env(env, f"terminal step {t}")
        ended += int(done.sum())
    assert ended >= 32
    env.close()


def test_render_bev_after_reset_load_state_and_copy_envs(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map("udem1")
    env = bev_env(16, "udem1", device_reset=True)
    env.reset(render=False)
    env.render_bev()
    check_env(env, "reset(render=False)")
    saved = env.save_state()
    first = env.bev_labels.clone(), env.bev_markings.clone()
    px, pz, ang = random_poses(md, 16, 99)
    place(env, px, pz, ang)
    env.render_bev()
    check_env(env, "moved")
    env.load_state(saved)
    env.render_bev()
    assert torch.equal(env.bev_labels, first[0]) and torch.equal(env.bev_markings, first[1])
    src = torch.tensor([3] * 8 + [-1] * 8)
    before = env.bev_labels.clone()
    env.copy_envs(src)
    env.render_bev()
    assert torch.equal(env.bev_labels[:8], before[3].expand(8, -1, -1))
    assert torch.equal(env.bev_labels[8:], before[8:])
    check_env(env, "copy_envs")
    env.close()


def test_the_agents_own_cell_names_its_tile(torch_cuda):
    """With the origin on a cell centre, that cell's centre is the agent's position: its label is (tile_i, tile_j)'s."""
    env = bev_env(64, "udem1", origin=(32.5, 48.5), device_reset=True)
    md = env.maps[0]
    n_cells = md.grid_w * md.grid_h
    env.reset(render=False)
    env.render_bev()
    own = env.bev_labels[:, 48, 32].cpu().numpy().astype(int)
    ti, tj = env.state["tile_i"].cpu().numpy(), env.state["tile_j"].cpu().numpy()
    on_tile = own < 2 + n_cells
    assert on_tile.sum() >= 60
    assert np.array_equal(own[on_tile], 2 + ti[on_tile] * md.grid_h + tj[on_tile])
    env.close()


def test_bev_changes_no_other_output_and_an_unset_target_launches_nothing(torch_cuda):
    """obs, depth, labels, markings, reward and done are the same bits with the grids on and off; with them off the
    tensors are not written and a step launches what it launches without them, one kernel more with them on."""
    torch = torch_cuda
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    kw = dict(camera_width=160, camera_height=120, domain_rand=True, seed=4, device_reset=True, auto_reset=True,
              depth=True, labels=True, markings=True, max_steps=8)
    env, plain = BatchedDuckietownEnv(32, "udem1", bev=True, **kw), BatchedDuckietownEnv(32, "udem1", **kw)
    assert plain.bev_labels is None and plain.bev_markings is None
    env.reset(); plain.reset()
    g = torch.Generator(device="cuda").manual_seed(5)
    for t in range(10):
        a = torch.rand((32, 2), device="cuda", generator=g)
        n0, p0 = env.launch_count(), plain.launch_count()
        out = env.step(a)
        ref = plain.step(a)
        torch.cuda.synchronize()
        assert env.launch_count() - n0 == plain.launch_count() - p0 + 1
        for x, y in zip(out[:3], ref[:3]):
            assert torch.equal(x, y), f"step {t}"
        for name in ("depth", "labels", "markings"):
            assert torch.equal(getattr(env, name).view(torch.uint8), getattr(plain, name).view(torch.uint8)), (name, t)
    env.sim.set_bev_target(None, None, None)
    env.bev_labels.fill_(-7); env.bev_markings.fill_(77)
    n0, p0 = env.launch_count(), plain.launch_count()
    a = torch.rand((32, 2), device="cuda", generator=g)
    env.step(a); plain.step(a)
    env.step(a, render=False); plain.step(a, render=False)
    env.render_obs(); plain.render_obs()
    torch.cuda.synchronize()
    assert env.launch_count() - n0 == plain.launch_count() - p0
    assert (env.bev_labels == -7).all() and (env.bev_markings == 77).all()
    with pytest.raises(Exception):
        env.render_bev()
    env.close(); plain.close()


def test_refused_configurations_leave_the_previous_one(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    env = bev_env(8, "udem1", device_reset=True)
    env.reset(render=False)
    env.render_bev()
    good = env.bev_labels.clone(), env.bev_markings.clone()
    lab, mk = env.bev_labels.data_ptr(), env.bev_markings.data_ptr()
    bad = [L.BevConfig(0, 64, 0.03, 32, 48), L.BevConfig(64, 2049, 0.03, 32, 48), L.BevConfig(64, 64, 0.0, 32, 48),
           L.BevConfig(64, 64, -0.03, 32, 48), L.BevConfig(64, 64, float("nan"), 32, 48),
           L.BevConfig(64, 64, float("inf"), 32, 48), L.BevConfig(64, 64, 0.03, float("nan"), 48),
           L.BevConfig(64, 64, 0.03, 32, float("inf"))]
    for cfg in bad:
        with pytest.raises(L.DtsError):
            env.sim.set_bev_target(cfg, lab, mk)
    with pytest.raises(L.DtsError):
        env.sim.set_bev_target(L.BevConfig(64, 64, 0.03, 32, 48), lab + 1, mk)   # labels not 2-byte aligned
    env.bev_labels.fill_(-7); env.bev_markings.fill_(77)
    env.render_bev()
    assert torch.equal(env.bev_labels, good[0]) and torch.equal(env.bev_markings, good[1])
    env.close()


def test_single_env_adapter_exposes_the_grids(torch_cuda):
    from gym_duckietown_b200.simulator import DuckietownEnv
    e = DuckietownEnv(map_name="loop_obstacles", domain_rand=False, camera_width=32, camera_height=24, seed=4, bev=True,
                      bev_shape=(32, 48))
    for step in range(3):
        if step:
            e.step(np.array([0.4, 0.2]))
        g, m = e.bev_labels, e.bev_markings
        assert g.shape == (32, 48) and g.dtype == np.int16 and m.shape == (32, 48) and m.dtype == np.uint8
        want = expected(e._b)
        bo.check(g[None], m[None], want, f"adapter step {step}")
    e.close()
