"""The lane-marking image the rasterisers write beside every observation (dts_set_marking_target, render spec item 11)
against the CPU marking oracle's (tests/marking_oracle.py: the label oracle's source with the marking insertions), bit
for bit: the two agree on the label's winners, evaluate the same f32 u, v for each at the pixel centre, and take the
same smallest class among them, which does not depend on the order it is taken in.

The raster paths are the label tests' (tests/test_gpu_labels.py, whose helpers are reused): bins inside one prim, flat
bins with their queued edge pixels and the bins handed back, mesh bins and tiny triangles, both tile modes, domain
randomisation, the fisheye / rectification gather and a camera_rand pool, top-down views, wrapper layouts and resize,
the listed second pass of dts_step_terminal, and two-map batches.  Every case also checks that the marking instances
change nothing else: obs, depth and labels are the same bits with markings on and off, and markings alone are the
markings written beside labels and depth."""
import numpy as np
import pytest

import marking_oracle
from test_gpu_camera_rand import install, pool_of
from test_gpu_depth import assert_same_bits, make_env, poses_of
from test_gpu_fisheye import random_poses
from test_gpu_labels import assert_same_labels
from test_gpu_render import oracle_episode
from test_gpu_undistort import device_episodes, rect_lut

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def oracle_batch(md, px, pz, ang, w, h, eps=None, domain_rand=False, lut=None, **mode):
    """(frames, depth, labels, markings u8 [n, h, w]) of the marking oracle"""
    import oracle as orc
    return marking_oracle.render_batch(orc.OracleScene(md), px, pz, ang, eps, w, h, domain_rand, lut=lut, **mode)


def marked_env(n, name, w=160, h=120, **kw):
    return make_env(n, name, w, h, labels=True, markings=True, **kw)


def render_again(env, kw):
    """render_obs(**kw) into a fresh buffer: (obs, depth, labels, markings) copies of what it wrote"""
    import torch
    out = env.render_obs(out=torch.empty_like(env.obs), **kw)
    torch.cuda.synchronize()
    return tuple(None if t is None else t.clone() for t in (out, env.depth, env.labels, env.markings))


def assert_markings_change_nothing(env, what, **kw):
    """With the env's targets as set (markings, labels, depth): the same render with the marking target off gives the
    same obs / depth / labels bits; markings alone, and markings beside labels alone or depth alone, give the same
    markings; and with the marking target off the markings tensor is not written."""
    import torch
    obs, dep, lab, mk = render_again(env, kw)
    env.sim.set_marking_target(None)
    env.markings.fill_(77)
    o2, d2, l2, _ = render_again(env, kw)
    assert torch.equal(o2, obs), f"{what}: obs differs with markings off"
    assert torch.equal(d2.view(torch.int32), dep.view(torch.int32)), f"{what}: depth differs with markings off"
    assert torch.equal(l2, lab), f"{what}: labels differ with markings off"
    assert (env.markings == 77).all(), f"{what}: markings were written with no target set"
    env.sim.set_marking_target(env.markings.data_ptr())
    for depth_on, labels_on in ((False, False), (True, False), (False, True)):
        env.sim.set_depth_target(env.depth.data_ptr() if depth_on else None)
        env.sim.set_label_target(env.labels.data_ptr() if labels_on else None)
        env.markings.fill_(77)
        o3, _, _, m3 = render_again(env, kw)
        assert torch.equal(o3, obs) and torch.equal(m3, mk), f"{what}: depth {depth_on} labels {labels_on}"
    env.sim.set_depth_target(env.depth.data_ptr())
    env.sim.set_label_target(env.labels.data_ptr())
    return mk


def assert_same_markings(got, want, what):
    assert_same_labels(got, want, what + " (markings)")


@pytest.mark.parametrize("name,W,H,dr,tess", [
    ("small_loop", 160, 120, False, False), ("loop_obstacles", 160, 120, False, False), ("udem1", 160, 120, True, False),
    ("small_loop", 84, 84, True, False), ("small_loop", 160, 120, False, True), ("udem1", 160, 120, True, True),
    ("loop_obstacles", 90, 70, False, False), ("udem1", 320, 240, False, False),
])
def test_first_frame_markings_vs_oracle(name, W, H, dr, tess, torch_cuda):
    """reset() with host-drawn episode parameters: markings, labels, depth and frame equal the oracle's; markings != 0
    exactly where the label is a textured cell; and the marking instances change nothing else."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps

    N = 48
    md = maps.load_map(name)
    env = marked_env(N, name, W, H, domain_rand=dr, seed=1000, tessellate_tiles=tess)
    assert env.markings.shape == (N, H, W) and env.markings.dtype == torch.uint8
    captured = {}
    orig = env.sim.reset
    env.sim.reset = lambda mask, params, stream=0: (captured.update(params), orig(mask, params, stream))[1]
    obs = env.reset().clone()
    px, pz, ang = poses_of(env)
    eps = [oracle_episode(orc, captured, k) for k in range(N)]
    rgb, dep, lab, mk = oracle_batch(md, px, pz, ang, W, H, eps, dr, tile_mode=0 if tess else 1)
    assert_same_markings(env.markings, mk, f"{name} {W}x{H}")
    assert_same_labels(env.labels, lab, f"{name} {W}x{H}")
    assert_same_bits(env.depth, dep, f"{name} {W}x{H}")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    n_cells = md.grid_w * md.grid_h
    assert np.array_equal(mk != 0, (lab >= 2) & (lab < 2 + n_cells))
    assert {1, 2}.issubset(set(np.unique(mk).tolist()))
    assert_markings_change_nothing(env, f"{name} {W}x{H}")
    env.check()
    env.close()


@pytest.mark.parametrize("name,W,H", [("loop_obstacles", 160, 120), ("udem1", 84, 84)])
def test_markings_near_props_vs_oracle(name, W, H, torch_cuda):
    """Agents parked 0.15 .. 2.5 m from the map's props, facing them: props hide the road (marking 0 on their pixels)."""
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    rng = np.random.default_rng(5)
    poses = []
    for o in md.objects:
        for d in (0.15, 0.3, 0.5, 0.8, 1.2, 1.8, 2.5):
            a = rng.uniform(-np.pi, np.pi)
            poses.append((o.pos[0] - d * np.cos(a), o.pos[2] + d * np.sin(a), a + rng.uniform(-0.25, 0.25)))
    P = np.array(poses[:96])
    N = len(P)
    env = marked_env(N, name, W, H, seed=3)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), map_id=np.zeros(N, np.int32)),
                  env._stream())
    env.render_obs()
    _, _, lab, mk = oracle_batch(md, P[:, 0], P[:, 1], P[:, 2], W, H)
    assert_same_markings(env.markings, mk, f"props {name} {W}x{H}")
    assert (mk[lab >= 2 + md.grid_w * md.grid_h] == 0).all() and (lab >= 2 + md.grid_w * md.grid_h).any()
    assert_markings_change_nothing(env, f"props {name}")
    env.check()
    env.close()


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
def test_large_batch_markings_exact_and_order_independent(name, torch_cuda):
    """2048 random cameras: markings equal the oracle's; the same cameras in two other orders give the same markings
    camera for camera; segment=True and domain-randomised colours leave them unchanged."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    N, W, H = 2048, 160, 120
    px, pz, ang = random_poses(md, N, 2024)
    env = marked_env(N, name, W, H)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    first = env.markings.clone()
    _, _, _, mk = oracle_batch(md, px, pz, ang, W, H)
    assert_same_markings(first, mk, f"large batch {name}")
    env.render_obs(segment=True)
    assert torch.equal(env.markings, first), "segment=True changed the markings"
    rng = np.random.default_rng(8)
    for perm in (np.arange(N)[::-1].copy(), rng.permutation(N)):
        env.sim.reset(None, dict(pos_x=px[perm].copy(), pos_z=pz[perm].copy(), angle=ang[perm].copy()))
        env.render_obs()
        idx = torch.from_numpy(perm).to(env.device)
        assert torch.equal(env.markings, first[idx]), "markings depend on the order of the batch"
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang, horizon_color=rng.uniform(0, 1, (N, 3)).astype(np.float32),
                             light_ambient=rng.uniform(0, 0.5, (N, 3)).astype(np.float32),
                             ground_color=rng.uniform(0, 1, (N, 3)).astype(np.float32)))
    env.render_obs()
    assert torch.equal(env.markings, first), "lighting and colours changed the markings"
    assert_markings_change_nothing(env, f"large batch {name}")
    env.check()
    env.close()


@pytest.mark.parametrize("name,W,H,N", [("udem1", 160, 120, 96), ("small_loop", 84, 84, 96)])
def test_markings_follow_fisheye_pinhole_rectification_and_top_down(name, W, H, N, torch_cuda):
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 31)
    env = marked_env(N, name, W, H, distortion=True)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    fish = (env.camera_model.rmapx, env.camera_model.rmapy)
    obs = env.render_obs()
    rgb, _, _, mk = oracle_batch(md, px, pz, ang, W, H, lut=fish)
    assert_same_markings(env.markings, mk, "fisheye")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    assert_markings_change_nothing(env, "fisheye")
    env.undistort = True
    env.render_obs()
    _, _, _, pin = oracle_batch(md, px, pz, ang, W, H)
    assert_same_markings(env.markings, pin, "pinhole")
    lut = rect_lut(W, H)
    env.set_rectification(*lut)
    env.sim.render(env.obs.data_ptr(), env._stream())     # the reset / step observation: rectified
    _, _, _, rect = oracle_batch(md, px, pz, ang, W, H, lut=lut)
    assert_same_markings(env.markings, rect, "rectified")
    env.render_obs(top_down=True)
    k = min(N, 12)
    _, _, top_lab, top = oracle_batch(md, px[:k], pz[:k], ang[:k], W, H, top_down=True)
    assert_same_markings(env.markings[:k], top, "top-down")
    assert (top_lab == 2 + md.grid_w * md.grid_h + len(md.objects)).any() and (top >= 2).any()
    assert_markings_change_nothing(env, "top-down", top_down=True)
    env.check()
    env.close()


def test_markings_follow_a_camera_rand_pool(torch_cuda):
    """A pool of fisheye tables, env e on table e mod K: each env's markings are the oracle's through its own table."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    name, N, W, H = "small_loop", 128, 160, 120
    md = maps.load_map(name)
    env = marked_env(N, name, W, H, distortion=True)
    luts = pool_of(["identity", "mirror_x", "jitter", "permutation", "real"], W, H)
    tab = np.arange(N) % len(luts)
    install(env, luts, tab)
    px, pz, ang = random_poses(md, N, 2026)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    got = env.markings.cpu().numpy()
    sc = orc.OracleScene(md)
    for t, lut in enumerate(luts):
        idx = np.flatnonzero(tab == t)
        _, _, _, mk = marking_oracle.render_batch(sc, px[idx], pz[idx], ang[idx], None, W, H, lut=lut)
        assert_same_markings(got[idx], mk, f"table {t}")
    assert_markings_change_nothing(env, "camera_rand pool")
    env.check()
    env.close()


@pytest.mark.parametrize("setup", ["chw_f32", "cwh_u8", "resize_cv2", "resize_pil_chw_f32"])
def test_markings_keep_their_layout_and_size_under_wrapper_formats_and_resize(setup, torch_cuda):
    from gym_duckietown_b200 import maps
    name, N, W, H = "loop_obstacles", 64, 160, 120
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 77)
    env = marked_env(N, name, W, H)
    if "chw_f32" in setup:
        env.set_output_format(obs_layout="chw", obs_dtype="float32")
    if setup == "cwh_u8":
        env.set_output_format(obs_layout="cwh")
    if setup.startswith("resize"):
        env.set_resize(84, 84, method="cv2_cubic" if "cv2" in setup else "pil_bilinear")
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    assert tuple(env.markings.shape) == (N, H, W)
    _, _, _, mk = oracle_batch(md, px, pz, ang, W, H)
    assert_same_markings(env.markings, mk, setup)
    assert_markings_change_nothing(env, setup)
    env.check()
    env.close()


def test_auto_reset_rollout_with_terminal_obs_markings_match_obs(torch_cuda):
    """Device auto-reset with terminal_obs=True: after every step env.markings is the oracle's of the state obs shows
    (for ended envs redrawn by the listed pass), and obs, terminal_obs, reward, done equal those of the same env
    without markings."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    name = "loop_obstacles"
    md = maps.load_map(name)
    N, W, H, T = 48, 160, 120, 12
    kw = dict(domain_rand=True, seed=11, device_reset=True, auto_reset=True, terminal_obs=True, max_steps=6)
    env, plain = marked_env(N, name, W, H, **kw), make_env(N, name, W, H, labels=True, **kw)
    assert plain.markings is None
    env.reset(); plain.reset()
    g = torch.Generator(device="cuda").manual_seed(3)
    ended = 0
    for t in range(T):
        a = torch.rand((N, 2), device="cuda", generator=g)
        a[:, 0] = 0.2 + 0.8 * a[:, 0]
        a[:, 1] = a[:, 1] * 2 - 1
        obs, rew, done, _ = env.step(a)
        obs2, rew2, done2, _ = plain.step(a)
        torch.cuda.synchronize()
        assert torch.equal(obs, obs2) and torch.equal(rew, rew2) and torch.equal(done, done2), f"step {t}"
        assert torch.equal(env.terminal_obs, plain.terminal_obs), f"step {t}"
        assert torch.equal(env.labels, plain.labels), f"step {t}"
        assert torch.equal(env.depth.view(torch.int32), plain.depth.view(torch.int32)), f"step {t}"
        ended += int(done.sum())
        px, pz, ang = poses_of(env)
        _, _, _, mk = oracle_batch(md, px, pz, ang, W, H, device_episodes(env), True)
        assert_same_markings(env.markings, mk, f"{name} step {t} ({int(done.sum())} envs ended)")
    assert ended >= N, f"only {ended} episodes ended"
    env.check(); plain.check()
    env.close(); plain.close()


def test_batch_of_two_maps_markings_come_from_each_envs_map(torch_cuda):
    import oracle as orc
    from gym_duckietown_b200 import maps
    names = ["small_loop", "udem1"]
    mds = [maps.load_map(n) for n in names]
    N, W, H = 64, 160, 120
    env = marked_env(N, names, W, H, seed=2)
    mid = (np.arange(N) % 2).astype(np.int32)
    P = np.zeros((N, 3))
    for m in range(2):
        k = np.flatnonzero(mid == m)
        P[k] = np.stack(random_poses(mds[m], len(k), 40 + m), axis=1)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), map_id=mid))
    env.render_obs()
    got = env.markings.cpu().numpy()
    for m in range(2):
        k = np.flatnonzero(mid == m)
        _, _, _, mk = marking_oracle.render_batch(orc.OracleScene(mds[m]), P[k, 0], P[k, 1], P[k, 2], W=W, H=H)
        assert_same_markings(got[k], mk, f"map {names[m]}")
    assert_markings_change_nothing(env, "two maps")
    env.check()
    env.close()


def test_single_env_adapter_exposes_markings(torch_cuda):
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.simulator import DuckietownEnv
    W, H = 160, 120
    e = DuckietownEnv(map_name="small_loop", domain_rand=False, camera_width=W, camera_height=H, seed=4, markings=True)
    assert e.labels is None and e.depth is None
    md = maps.load_map("small_loop")
    for step in range(3):
        if step:
            e.step(np.array([0.6, 0.3]))
        m = e.markings
        assert isinstance(m, np.ndarray) and m.shape == (H, W) and m.dtype == np.uint8
        _, _, _, mk = oracle_batch(md, [e.cur_pos[0]], [e.cur_pos[2]], [e.cur_angle], W, H)
        assert_same_markings(m, mk[0], f"adapter step {step}")
    e.close()
