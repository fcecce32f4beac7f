"""camera_rand on the device: a pool of fisheye LUTs, env e gathered through LUT lut_of_env[e] (dts_set_fisheye_luts),
against the CPU label oracle rendering each env through its own LUT (frames, depth and labels, bit for bit).

Mixed batches use test_gpu_fisheye.py's synthetic LUT kinds, env e on kind e mod K, so that envs side by side in one
launch bin and gather through tables whose boxes, inverse indices and home-cell ranges differ.  small_loop reaches
k_raster_solo, k_raster_flat and the bins it hands back, loop_obstacles the mesh bins of k_raster; the wrapper format
reaches k_raster's other instance, and terminal_obs the env-list second pass of dts_step_terminal."""
import os

import numpy as np
import pytest

import label_oracle
from test_gpu_depth import make_env, poses_of
from test_gpu_fisheye import lsb_diff, make_lut, random_poses
from test_gpu_undistort import device_episodes

pytestmark = pytest.mark.gpu

MIXED_KINDS = ["identity", "mirror_x", "shift", "ties", "specials", "zoom", "jitter", "permutation", "real"]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def pool_of(kinds, W, H):
    from gym_duckietown_b200.distortion import Distortion
    real = Distortion(W, H)
    luts = [make_lut(k, W, H, real) for k in kinds]
    return [(np.asarray(x, np.float32), np.asarray(y, np.float32)) for x, y in luts]


def install(env, luts, tab):
    env.sim.set_fisheye_luts(np.stack([x for x, _ in luts]), np.stack([y for _, y in luts]), tab)


def oracle_per_env(md, px, pz, ang, W, H, luts, tab, eps=None, domain_rand=False):
    """(frames, depth, labels) of the label oracle, env k rendered through luts[tab[k]]"""
    import oracle as orc
    sc = orc.OracleScene(md)
    n = len(px)
    frames, dep, lab = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32), np.zeros((n, H, W), np.int16)
    for t, lut in enumerate(luts):
        idx = np.flatnonzero(np.asarray(tab) == t)
        if len(idx) == 0:
            continue
        f, d, l = label_oracle.render_batch(sc, px[idx], pz[idx], ang[idx], [eps[i] for i in idx] if eps else None, W, H,
                                            domain_rand, lut=lut)
        frames[idx], dep[idx], lab[idx] = f, d, l
    return frames, dep, lab


def check_env(env, md, luts, tab, what, eps=None, domain_rand=False, chw_f32=False):
    import torch
    torch.cuda.synchronize()
    W, H = env.camera_width, env.camera_height
    px, pz, ang = poses_of(env)
    f, d, l = oracle_per_env(md, px, pz, ang, W, H, luts, tab, eps, domain_rand)
    got = env.obs.cpu().numpy()
    if chw_f32:
        want = (f.transpose(0, 3, 1, 2) / 255.0).astype(np.float32)
        assert np.array_equal(got, want), f"{what}: frames differ"
    else:
        mx, n = lsb_diff(got, f)
        assert mx == 0, f"{what}: frames differ by up to {mx} LSB on {n} values"
    assert np.array_equal(env.depth.cpu().numpy().view(np.uint32), d.view(np.uint32)), f"{what}: depth differs"
    assert np.array_equal(env.labels.cpu().numpy(), l), f"{what}: labels differ"
    assert f.std() > 10, f"{what}: the oracle's frames are blank"


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
@pytest.mark.parametrize("fmt", ["hwc_u8", "chw_f32"])
def test_mixed_tables_vs_oracle(name, fmt, torch_cuda):
    """256 cameras at 160x120, env e on synthetic kind e mod 9: frames at 0 LSB, depth and labels bit for bit."""
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    N, W, H = 256, 160, 120
    env = make_env(N, name, W, H, distortion=True, labels=True)
    if fmt == "chw_f32":
        env.set_output_format(obs_layout="chw", obs_dtype="float32")
    luts = pool_of(MIXED_KINDS, W, H)
    tab = np.arange(N) % len(luts)
    install(env, luts, tab)
    px, pz, ang = random_poses(md, N, 2026)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    check_env(env, md, luts, tab, f"{name} {fmt}", chw_f32=fmt == "chw_f32")
    # a shuffled assignment: each env's frame follows its own table, not its neighbours'
    tab2 = np.random.default_rng(4).integers(0, len(luts), N)
    install(env, luts, tab2)
    env.render_obs()
    check_env(env, md, luts, tab2, f"{name} {fmt} shuffled", chw_f32=fmt == "chw_f32")
    env.check()
    env.close()


def test_mixed_tables_at_640x480_vs_oracle(torch_cuda):
    """640x480 (k_bin with four warps per env): the kinds whose boxes pass the int32 edge bound there, mixed."""
    from gym_duckietown_b200 import maps
    md = maps.load_map("udem1")
    N, W, H = 24, 640, 480
    env = make_env(N, "udem1", W, H, distortion=True, labels=True)
    luts = pool_of(["identity", "mirror_x", "jitter", "real"], W, H)
    tab = np.arange(N) % len(luts)
    install(env, luts, tab)
    px, pz, ang = random_poses(md, N, 7)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    check_env(env, md, luts, tab, "udem1 640x480")
    env.check()
    env.close()


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
def test_terminal_obs_rollout_vs_oracle(name, torch_cuda):
    """Device auto-reset with terminal_obs=True: envs on different tables end, and the listed second pass redraws them
    through their own tables.  After every step obs, depth and labels equal the oracle's."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    N, W, H, T = 48, 160, 120, 12
    env = make_env(N, name, W, H, distortion=True, labels=True, seed=11, device_reset=True, auto_reset=True,
                   terminal_obs=True, max_steps=5)
    luts = pool_of(["identity", "mirror_x", "jitter", "permutation", "real"], W, H)
    tab = np.arange(N) % len(luts)
    install(env, luts, tab)
    env.reset()
    check_env(env, md, luts, tab, f"{name} reset", eps=device_episodes(env))
    g = torch.Generator(device="cuda").manual_seed(5)
    ended_tables = set()
    for t in range(T):
        a = torch.rand((N, 2), device="cuda", generator=g)
        a[:, 0] = 0.2 + 0.8 * a[:, 0]
        a[:, 1] = a[:, 1] * 2 - 1
        _, _, done, _ = env.step(a)
        ended_tables |= set(tab[done.cpu().numpy()].tolist())
        # (a re-spawned env's light comes through the previous episode's model-view, S:581: the device's episodes)
        check_env(env, md, luts, tab, f"{name} step {t} ({int(done.sum())} ended)", eps=device_episodes(env))
    assert ended_tables == set(range(len(luts))), f"only envs on tables {sorted(ended_tables)} ended"
    env.check()
    env.close()


def test_pool_of_one_table_equals_single_lut(torch_cuda):
    """A pool of one table, and a pool of two equal tables (the pool kernels), draw the frames dts_set_fisheye_lut draws
    with that table, byte for byte."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map("loop_obstacles")
    N, W, H = 512, 160, 120
    env = make_env(N, "loop_obstacles", W, H, distortion=True, labels=True)
    px, pz, ang = random_poses(md, N, 9)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    rx, ry = env.camera_model.rmapx, env.camera_model.rmapy
    env.sim.set_fisheye_lut(rx, ry)
    want = [t.clone() for t in (env.render_obs(), env.depth, env.labels)]
    for luts, tab in (([(rx, ry)], np.zeros(N)), ([(rx, ry), (rx, ry)], np.arange(N) % 2)):
        install(env, luts, tab)
        got = (env.render_obs(), env.depth, env.labels)
        torch.cuda.synchronize()
        for a, b, what in zip(got, want, ("obs", "depth", "labels")):
            assert torch.equal(a, b), f"{len(luts)} table(s): {what} differs from the single LUT's"
    env.check()
    env.close()


@pytest.mark.parametrize("W,H", [(160, 120), (84, 84)])
def test_real_pool_vs_oracle(W, H, torch_cuda):
    """camera_rand=True, distortion=True: four drawn calibrations, env g on calibration g mod 4 (env_id_offset counts),
    device resets drawing the camera height / angle / FOV; every env's frame equals the oracle's through its
    calibration's host-built LUT."""
    from gym_duckietown_b200 import maps
    md = maps.load_map("loop_obstacles")
    N = 64
    env = make_env(N, "loop_obstacles", W, H, distortion=True, camera_rand=True, camera_rand_pool=4, labels=True,
                   seed=21, device_reset=True, env_id_offset=3)
    assert env.camera_rand and len(env.calibrations) == 4
    assert np.array_equal(env.calibration_of_env, (3 + np.arange(N)) % 4)
    assert len({m.rmapx.tobytes() for m in env.camera_models}) == 4
    env.reset()
    eps = device_episodes(env)
    assert len({e.cam_fov_y_deg for e in eps}) > 1
    luts = [(m.rmapx, m.rmapy) for m in env.camera_models]
    check_env(env, md, luts, env.calibration_of_env, f"real pool {W}x{H}", eps=eps)
    env.check()
    env.close()


def test_refused_pool_keeps_the_previous_tables(torch_cuda):
    """A pool with one table too wide for the edge functions, an assignment outside the pool, or a pool on a handle
    without DTS_FLAG_DISTORTION is refused; the previous tables and assignment keep rendering exactly as before."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.lib import DtsError
    md = maps.load_map("small_loop")
    N, W, H = 16, 640, 480
    env = make_env(N, "small_loop", W, H, distortion=True, labels=True)
    px, pz, ang = random_poses(md, N, 3)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    luts = pool_of(["identity", "mirror_x", "real"], W, H)
    tab = np.arange(N) % 3
    install(env, luts, tab)
    before = [t.clone() for t in (env.render_obs(), env.depth, env.labels)]
    wide_x, wide_y = make_lut("identity", W, H)
    wide_x[0:8, 0:16], wide_y[0:8, 0:16] = 0, 0
    wide_x[0:8, 16:32], wide_y[0:8, 16:32] = W - 1, H - 1
    with pytest.raises(DtsError, match="fisheye LUT 1 sends output bin 0 .* too wide"):
        install(env, [luts[0], (wide_x, wide_y), luts[2]], np.zeros(N))
    with pytest.raises(DtsError, match="is not a table of the pool"):
        install(env, luts[:2], np.full(N, 2))
    after = (env.render_obs(), env.depth, env.labels)
    torch.cuda.synchronize()
    for a, b in zip(after, before):
        assert torch.equal(a, b)
    plain = make_env(2, "small_loop", 32, 32, depth=False)
    with pytest.raises(DtsError, match="without DTS_FLAG_DISTORTION"):
        plain.sim.set_fisheye_luts(np.zeros((2, 32, 32), np.float32), np.zeros((2, 32, 32), np.float32), [0, 1])
    env.check()
    env.close(); plain.close()


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles", "udem1"])
def test_device_reset_reproduces_reference(name, golden_dir, torch_cuda):
    """Device resets (DTS_FLAG_CAMERA_RAND, domain_rand off) are the reference's reset() with camera_rand and distortion
    on (reset_camrand_<map>.npz), draw for draw; auto_reset re-spawns the same way."""
    torch = torch_cuda
    g = np.load(os.path.join(golden_dir, f"reset_camrand_{name}.npz"))
    n = len(g["seeds"])
    assert list(g["seeds"]) == list(range(n))
    for auto in (False, True):
        env = make_env(n, name, 32, 32, depth=False, distortion=True, camera_rand=True, camera_rand_pool=1, seed=0,
                       device_reset=True, auto_reset=auto, max_steps=1)
        for ep in range(2):
            if ep == 0 or not auto:
                env.reset(render=False)
            else:   # one step of max_steps=1 ends every episode, and auto_reset re-spawns on the device
                _, _, done, _ = env.step(torch.zeros((n, 2), device="cuda"), render=False)
                assert bool(done.all())
            torch.cuda.synchronize()
            st = {k: v.cpu().numpy() for k, v in env.state.items()}
            rows = np.arange(n) * 2 + ep
            assert np.array_equal(st["pos_x"], g["cur_pos"][rows, 0]), (auto, ep)
            assert np.array_equal(st["angle"], g["cur_angle"][rows]), (auto, ep)
            for k in range(n):
                r, row = env.sim.debug_episode(k), rows[k]
                assert r["cam_height"] == np.float32(g["cam_height"][row])
                assert r["cam_angle_deg"] == np.float32(g["cam_angle"][row])
                assert r["cam_fov_y_deg"] == np.float32(g["cam_fov_y"][row])
                assert not np.any(r["cam_noise"])
                assert np.array_equal(r["horizon"], g["horizon_color"][row].astype(np.float32))
        env.close()


def test_camera_rand_without_distortion_changes_nothing(torch_cuda):
    """As in the reference (S:352-358), camera_rand takes effect only with distortion: without it the env, its resets
    (host and device) and its frames are those of an env built without the flag."""
    torch = torch_cuda
    for device_reset in (False, True):
        a = make_env(32, "loop_obstacles", 64, 48, camera_rand=True, seed=4, device_reset=device_reset)
        b = make_env(32, "loop_obstacles", 64, 48, seed=4, device_reset=device_reset)
        assert not a.camera_rand and a.calibrations is None
        for _ in range(2):
            oa, ob = a.reset(), b.reset()
            torch.cuda.synchronize()
            assert torch.equal(oa, ob) and torch.equal(a.depth, b.depth)
            assert all(torch.equal(a.state[k], b.state[k]) for k in a.state)
            assert all(a.sim.debug_episode(k)["cam_height"] == b.sim.debug_episode(k)["cam_height"] for k in range(32))
        a.close(); b.close()


def test_copy_envs_and_load_state_keep_each_envs_calibration(torch_cuda):
    """The calibration belongs to the env: after copy_envs the destination draws its copied state through its own
    table, and records loaded into another env of the pool are drawn through that env's."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map("small_loop")
    N, W, H = 8, 160, 120
    env = make_env(N, "small_loop", W, H, distortion=True, camera_rand=True, camera_rand_pool=4, labels=True, seed=8,
                   device_reset=True)
    env.reset()
    luts = [(m.rmapx, m.rmapy) for m in env.camera_models]
    tab = env.calibration_of_env
    src = np.array([1, -1, 3, -1, -1, -1, 4, 6])
    env.copy_envs(src)
    env.render_obs()
    eps = device_episodes(env)
    check_env(env, md, luts, tab, "after copy_envs", eps=eps)
    px, pz, _ = poses_of(env)
    assert px[0] == px[1] and px[2] == px[3]                            # the same state ...
    assert not torch.equal(env.obs[0], env.obs[1])                      # ... seen through another lens
    env.check()
    env.close()


def test_state_dict_round_trip_and_mismatched_pool(torch_cuda):
    """state_dict carries the pool's calibrations and assignment under camera_rand: it round-trips into an env with the
    same pool, and an env with another pool (another seed, or none) refuses it and keeps its state."""
    torch = torch_cuda
    kw = dict(distortion=True, camera_rand=True, camera_rand_pool=3, device_reset=True, depth=False)
    a = make_env(6, "small_loop", 64, 48, seed=30, **kw)
    a.reset()
    for _ in range(3):
        a.step(torch.full((6, 2), 0.3, device="cuda"))
    d = a.state_dict()
    assert d["camera_rand"]["K"].shape == (3, 3, 3) and d["camera_rand"]["D"].shape == (3, 1, 5)
    b = make_env(6, "small_loop", 64, 48, seed=30, **kw)
    b.reset()
    b.load_state_dict(d)
    assert torch.equal(a.render_obs().clone(), b.render_obs())
    a.step(torch.full((6, 2), 0.5, device="cuda")); b.step(torch.full((6, 2), 0.5, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(a.obs, b.obs)
    other = make_env(6, "small_loop", 64, 48, seed=31, **kw)
    none = make_env(6, "small_loop", 64, 48, seed=30, distortion=True, device_reset=True, depth=False)
    for env in (other, none):
        env.reset()
        recs = env.save_state()
        with pytest.raises(ValueError, match="camera_rand calibrations differ"):
            env.load_state_dict(d)
        assert torch.equal(env.save_state(), recs)
    with pytest.raises(ValueError, match="camera_rand calibrations differ"):
        a.load_state_dict(none.state_dict())
    for env in (a, b, other, none):
        env.close()
