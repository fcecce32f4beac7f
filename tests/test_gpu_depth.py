"""The depth image the rasterisers write beside every observation (dts_set_depth_target, render spec item 9) against the
CPU depth oracle's (tests/depth_oracle.py: the raster oracle's source with the depth insertions), bit for bit: the two agree on which prims win a pixel's samples and evaluate the same f32 expression for
each winner's 1/w, and a maximum of exact values does not depend on the order it is taken in.

Every raster path is reached through the shapes the RGB tests use: small_loop (bins inside one prim, flat bins and the
ones handed back), loop_obstacles and udem1 (mesh bins, one-lane tiny triangles, lists streamed in chunks), both tile
modes, domain randomisation, the fused fisheye / rectification gather, wrapper layouts (the general rasteriser alone),
cameras whose size is no multiple of the bin size, and the listed second pass of dts_step_terminal."""
import numpy as np
import pytest

import depth_oracle
from test_gpu_fisheye import random_poses
from test_gpu_render import oracle_episode
from test_gpu_undistort import device_episodes, rect_lut

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, name, w=160, h=120, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, seed=5, depth=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, name, **args)


def oracle_batch(md, px, pz, ang, w, h, eps=None, domain_rand=False, lut=None, **mode):
    """(frames u8 [n, h, w, 3], depth f32 [n, h, w]) of the depth oracle; mode: segment, top_down, tile_mode."""
    import oracle as orc
    return depth_oracle.render_batch(orc.OracleScene(md), px, pz, ang, eps, w, h, domain_rand, lut=lut, **mode)


def assert_same_bits(got, want, what):
    """`got` (a CUDA or numpy f32 array) and the oracle's depth hold the same bit patterns."""
    import torch
    g = torch.as_tensor(got).cpu().contiguous().view(torch.int32)
    w = torch.from_numpy(np.ascontiguousarray(want)).view(torch.int32)
    if not torch.equal(g, w):
        bad = (g != w)
        gf, wf = g.view(torch.float32)[bad], w.view(torch.float32)[bad]
        where = torch.nonzero(bad)[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} depth values differ, first at {where}: "
                             f"{gf[0].item()!r} vs the oracle's {wf[0].item()!r}; largest gap {float((gf - wf).abs().max()):.3e}")


def poses_of(env):
    st = {k: v.cpu().numpy() for k, v in env.state.items()}
    return st["pos_x"], st["pos_z"], st["angle"]


@pytest.mark.parametrize("name,W,H,dr,tess", [
    ("small_loop", 160, 120, False, False), ("loop_obstacles", 160, 120, False, False), ("udem1", 160, 120, True, False),
    ("small_loop", 84, 84, True, False), ("small_loop", 160, 120, False, True), ("udem1", 160, 120, True, True),
    ("loop_obstacles", 90, 70, False, False), ("udem1", 320, 240, False, False),
])
def test_first_frame_depth_vs_oracle(name, W, H, dr, tess, torch_cuda):
    """reset() with host-drawn episode parameters: the depth equals the oracle's, the frame equals the oracle's, and the
    frame equals, byte for byte, the one the same env draws with no depth target.  84x84 ends in half a coarse bin on
    both axes; 90x70 is no multiple of 4 wide, so the general rasteriser draws all of it."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps

    N = 48
    env = make_env(N, name, W, H, domain_rand=dr, seed=1000, tessellate_tiles=tess)
    assert env.depth.shape == (N, H, W) and env.depth.dtype == torch.float32 and env.depth.device == env.device
    captured = {}
    orig = env.sim.reset
    env.sim.reset = lambda mask, params, stream=0: (captured.update(params), orig(mask, params, stream))[1]
    obs = env.reset().clone()
    px, pz, ang = poses_of(env)
    eps = [oracle_episode(orc, captured, k) for k in range(N)]
    rgb, dep = oracle_batch(maps.load_map(name), px, pz, ang, W, H, eps, dr, tile_mode=0 if tess else 1)
    assert_same_bits(env.depth, dep, f"{name} {W}x{H}")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    assert (dep == 0).mean() > 0.05 and (dep > 0).mean() > 0.3     # sky and surfaces both present
    env.sim.set_depth_target(None)
    assert torch.equal(env.render_obs(out=torch.empty_like(obs)), obs), "the frame drawn with depth differs from the frame without"
    env.check()
    env.close()


@pytest.mark.parametrize("name,W,H", [("loop_obstacles", 160, 120), ("udem1", 160, 120), ("udem1", 84, 84)])
def test_depth_near_props_vs_oracle(name, W, H, torch_cuda):
    """Agents parked 0.15 .. 2.5 m from the map's props, facing them: triangles from dozens of pixels down to sub-pixel
    size, so winners come from warp-wide visits, from the one-lane tiny-triangle buffer and from the merge of the two."""
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
    env = make_env(N, name, W, H, seed=3)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), map_id=np.zeros(N, np.int32)),
                  env._stream())
    obs = env.render_obs()
    rgb, dep = oracle_batch(md, P[:, 0], P[:, 1], P[:, 2], W, H)
    assert_same_bits(env.depth, dep, f"props {name} {W}x{H}")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    assert dep[dep > 0].min() < 0.2     # something stands right in front of a camera
    env.check()
    env.close()


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
def test_large_batch_depth_exact_and_order_independent(name, torch_cuda):
    """2048 random cameras of one map (rare events — bins handed back by the flat rasteriser, depth ties, lists of more
    than 32 records — only show up in large batches): depth equals the oracle's; the same cameras in two other orders
    of the batch give the same depth camera for camera, and segment=True does too."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps

    md = maps.load_map(name)
    N, W, H = 2048, 160, 120
    px, pz, ang = random_poses(md, N, 2024)
    env = make_env(N, name, W, H)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    first = env.depth.clone()
    _, dep = oracle_batch(md, px, pz, ang, W, H)
    assert_same_bits(first, dep, f"large batch {name}")
    env.render_obs(segment=True)
    assert torch.equal(env.depth.view(torch.int32), first.view(torch.int32)), "segment=True changed the depth"
    rng = np.random.default_rng(8)
    for perm in (np.arange(N)[::-1].copy(), rng.permutation(N)):
        env.sim.reset(None, dict(pos_x=px[perm].copy(), pos_z=pz[perm].copy(), angle=ang[perm].copy()))
        env.render_obs()
        idx = torch.from_numpy(perm).to(env.device)
        assert torch.equal(env.depth.view(torch.int32), first[idx].view(torch.int32)), "depth depends on the order of the batch"
    env.check()
    env.close()


@pytest.mark.parametrize("name,W,H,N", [("udem1", 160, 120, 96), ("small_loop", 84, 84, 96), ("udem1", 640, 480, 8)])
def test_depth_follows_fisheye_pinhole_rectification_and_top_down(name, W, H, N, torch_cuda):
    """A `distortion` env: the fisheye frame's depth is the oracle's depth gathered through the fisheye LUT (0 where it
    names no source); under `undistort` it is the pinhole depth, with a rectification installed the depth gathered
    through that map; render_obs(top_down=True) gives the depth of the camera above the map."""
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 31)
    env = make_env(N, name, W, H, distortion=True)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    fish = (env.camera_model.rmapx, env.camera_model.rmapy)
    obs = env.render_obs()
    rgb, dep = oracle_batch(md, px, pz, ang, W, H, lut=fish)
    assert_same_bits(env.depth, dep, "fisheye")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    env.undistort = True
    env.render_obs()
    _, pin = oracle_batch(md, px, pz, ang, W, H)
    assert_same_bits(env.depth, pin, "pinhole")
    assert not np.array_equal(pin, dep)
    lut = rect_lut(W, H)
    env.set_rectification(*lut)
    env.sim.render(env.obs.data_ptr(), env._stream())     # the reset / step observation: rectified
    _, rect = oracle_batch(md, px, pz, ang, W, H, lut=lut)
    assert_same_bits(env.depth, rect, "rectified")
    env.render_obs(top_down=True)
    _, top = oracle_batch(md, px[:12], pz[:12], ang[:12], W, H, top_down=True)
    assert_same_bits(env.depth[:min(N, 12)], top[:min(N, 12)], "top-down")
    env.check()
    env.close()


@pytest.mark.parametrize("setup", ["chw_f32", "cwh_u8", "resize_cv2", "resize_pil_chw_f32"])
def test_depth_keeps_its_layout_and_size_under_wrapper_formats_and_resize(setup, torch_cuda):
    """dts_set_output_format and dts_set_resize change obs, not depth: f32 [N, H, W] at the camera size, the oracle's
    bits.  (A wrapper layout sends every bin through the general rasteriser.)"""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    name, N, W, H = "loop_obstacles", 64, 160, 120
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 77)
    env = make_env(N, name, W, H)
    if "chw_f32" in setup:
        env.set_output_format(obs_layout="chw", obs_dtype="float32")
    if setup == "cwh_u8":
        env.set_output_format(obs_layout="cwh")
    if setup.startswith("resize"):
        env.set_resize(84, 84, method="cv2_cubic" if "cv2" in setup else "pil_bilinear")
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    obs = env.render_obs()
    assert tuple(env.depth.shape) == (N, H, W)
    rgb, dep = oracle_batch(md, px, pz, ang, W, H)
    assert_same_bits(env.depth, dep, setup)
    if setup == "chw_f32":
        assert np.array_equal(obs.cpu().numpy(), (rgb.transpose(0, 3, 1, 2) / 255.0).astype(np.float32))
    if setup == "cwh_u8":
        assert np.array_equal(obs.cpu().numpy(), rgb.transpose(0, 3, 2, 1))
    env.check()
    env.close()


@pytest.mark.parametrize("name,dr", [("small_loop", False), ("loop_obstacles", True)])
def test_auto_reset_rollout_with_terminal_obs_depth_matches_obs(name, dr, torch_cuda):
    """Device auto-reset with terminal_obs=True (dts_step_terminal): after every step env.depth is the oracle's depth of
    the state obs shows — for the envs that ended, the first frame of their next episode, redrawn by the pass over the
    listed envs alone — and obs, reward, done equal those of the same env without depth."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    N, W, H, T = 48, 160, 120, 14
    kw = dict(domain_rand=dr, seed=11, device_reset=True, auto_reset=True, terminal_obs=True, max_steps=6)
    env, plain = make_env(N, name, W, H, **kw), make_env(N, name, W, H, depth=False, **kw)
    assert plain.depth is None
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
        ended += int(done.sum())
        px, pz, ang = poses_of(env)
        _, dep = oracle_batch(md, px, pz, ang, W, H, device_episodes(env) if dr else None, dr)
        assert_same_bits(env.depth, dep, f"{name} step {t} ({int(done.sum())} envs ended)")
    assert ended >= N, f"only {ended} episodes ended"
    env.check(); plain.check()
    env.close(); plain.close()


def test_null_target_stops_the_writes_and_a_new_one_resumes(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    name, N, W, H = "small_loop", 32, 160, 120
    md = maps.load_map(name)
    env = make_env(N, name, W, H, seed=9)
    env.reset()
    px, pz, ang = poses_of(env)
    _, dep = oracle_batch(md, px, pz, ang, W, H)
    assert_same_bits(env.depth, dep, "before")
    env.sim.set_depth_target(None)
    env.depth.fill_(-7.0)
    env.render_obs()
    acts = torch.zeros((N, 2), device=env.device)
    env.step(acts)
    torch.cuda.synchronize()
    assert (env.depth == -7.0).all(), "depth was written with no target set"
    other = torch.full_like(env.depth, -1.0)
    env.sim.set_depth_target(other.data_ptr())
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    assert_same_bits(other, dep, "new target")
    assert (env.depth == -7.0).all()
    with pytest.raises(Exception):
        env.sim.set_depth_target(other.data_ptr() + 2)      # not a float address
    env.check()
    counters = env.sim.debug_counters()
    assert int(counters[0]) == 0 and not (env.sim.status() & 1)
    env.close()


def test_single_env_adapter_exposes_depth(torch_cuda):
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.simulator import DuckietownEnv
    W, H = 160, 120
    e = DuckietownEnv(map_name="loop_obstacles", domain_rand=False, camera_width=W, camera_height=H, seed=4, depth=True)
    off = DuckietownEnv(map_name="small_loop", domain_rand=False, camera_width=W, camera_height=H, seed=4)
    assert off.depth is None
    off.close()
    md = maps.load_map("loop_obstacles")
    for step in range(3):
        if step:
            e.step(np.array([0.6, 0.3]))
        d = e.depth
        assert isinstance(d, np.ndarray) and d.shape == (H, W) and d.dtype == np.float32
        _, dep = oracle_batch(md, [e.cur_pos[0]], [e.cur_pos[2]], [e.cur_angle], W, H)
        assert_same_bits(d, dep[0], f"adapter step {step}")
    e.render(mode="rgb_array")          # the 800x600 view has no depth and leaves this one alone
    assert np.array_equal(e.depth, d)
    e.close()
