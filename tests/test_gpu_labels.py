"""The label image the rasterisers write beside every observation (dts_set_label_target, render spec item 10) against the
CPU label oracle's (tests/label_oracle.py: the depth oracle's source with the label insertions), bit for bit: the two
agree on which prims win a pixel's samples, evaluate the same f32 1/w for each winner, and take the same maximum with
the same exact tie-break, which does not depend on the order it is taken in.

The raster paths are reached through the shapes tests/test_gpu_depth.py uses: small_loop (bins inside one prim, flat
bins and the ones handed back), loop_obstacles and udem1 (mesh bins, one-lane tiny triangles, lists streamed in chunks),
both tile modes, domain randomisation, the fused fisheye / rectification gather, top-down views (the agent's own mesh),
wrapper layouts and resize, cameras whose size is no multiple of the bin size, the listed second pass of
dts_step_terminal, and batches mixing two maps."""
import numpy as np
import pytest

import label_oracle
from test_gpu_depth import assert_same_bits, make_env, poses_of
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


def oracle_batch(md, px, pz, ang, w, h, eps=None, domain_rand=False, lut=None, **mode):
    """(frames u8 [n, h, w, 3], depth f32 [n, h, w], labels i16 [n, h, w]) of the label oracle"""
    import oracle as orc
    return label_oracle.render_batch(orc.OracleScene(md), px, pz, ang, eps, w, h, domain_rand, lut=lut, **mode)


def assert_same_labels(got, want, what):
    import torch
    g = torch.as_tensor(got).cpu().numpy()
    if not np.array_equal(g, want):
        bad = np.argwhere(g != want)
        k = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {g.size} labels differ, first at {list(k)}: {g[k]} vs the oracle's "
                             f"{want[k]}")


def labelled_env(n, name, w=160, h=120, **kw):
    return make_env(n, name, w, h, labels=True, **kw)


@pytest.mark.parametrize("name,W,H,dr,tess", [
    ("small_loop", 160, 120, False, False), ("loop_obstacles", 160, 120, False, False), ("udem1", 160, 120, True, False),
    ("small_loop", 84, 84, True, False), ("small_loop", 160, 120, False, True), ("udem1", 160, 120, True, True),
    ("loop_obstacles", 90, 70, False, False), ("udem1", 320, 240, False, False),
])
def test_first_frame_labels_vs_oracle(name, W, H, dr, tess, torch_cuda):
    """reset() with host-drawn episode parameters: labels, depth and frame equal the oracle's; label != 0 exactly where
    depth != 0; labels alone (no depth target) are the same labels; and with neither target the frame is the same."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps

    N = 48
    env = labelled_env(N, name, W, H, domain_rand=dr, seed=1000, tessellate_tiles=tess)
    assert env.labels.shape == (N, H, W) and env.labels.dtype == torch.int16 and env.labels.device == env.device
    captured = {}
    orig = env.sim.reset
    env.sim.reset = lambda mask, params, stream=0: (captured.update(params), orig(mask, params, stream))[1]
    obs = env.reset().clone()
    px, pz, ang = poses_of(env)
    eps = [oracle_episode(orc, captured, k) for k in range(N)]
    rgb, dep, lab = oracle_batch(maps.load_map(name), px, pz, ang, W, H, eps, dr, tile_mode=0 if tess else 1)
    assert_same_labels(env.labels, lab, f"{name} {W}x{H}")
    assert_same_bits(env.depth, dep, f"{name} {W}x{H}")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    assert torch.equal(env.labels != 0, env.depth != 0)
    assert len(np.unique(lab)) > 3
    depth = env.depth.clone()
    env.sim.set_depth_target(None)            # labels alone
    env.labels.zero_()
    assert torch.equal(env.render_obs(out=torch.empty_like(obs)), obs)
    assert_same_labels(env.labels, lab, f"{name} {W}x{H} labels alone")
    env.sim.set_depth_target(env.depth.data_ptr())
    env.sim.set_label_target(None)            # depth alone: the same depth bits and frame
    env.depth.zero_()
    assert torch.equal(env.render_obs(out=torch.empty_like(obs)), obs)
    assert torch.equal(env.depth.view(torch.int32), depth.view(torch.int32))
    env.sim.set_depth_target(None)
    assert torch.equal(env.render_obs(out=torch.empty_like(obs)), obs)
    env.check()
    env.close()


@pytest.mark.parametrize("name,W,H", [("loop_obstacles", 160, 120), ("udem1", 160, 120), ("udem1", 84, 84)])
def test_labels_near_props_vs_oracle(name, W, H, torch_cuda):
    """Agents parked 0.15 .. 2.5 m from the map's props, facing them: winners from warp-wide visits, from the one-lane
    tiny-triangle buffer and from the merge of the two; every pixel's label names one object of the list."""
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
    env = labelled_env(N, name, W, H, seed=3)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), map_id=np.zeros(N, np.int32)),
                  env._stream())
    obs = env.render_obs()
    rgb, dep, lab = oracle_batch(md, P[:, 0], P[:, 1], P[:, 2], W, H)
    assert_same_labels(env.labels, lab, f"props {name} {W}x{H}")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    n_cells = md.grid_w * md.grid_h
    assert len(np.unique(lab[lab >= 2 + n_cells])) >= min(len(md.objects), 8)     # many props are seen
    env.check()
    env.close()


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
def test_large_batch_labels_exact_and_order_independent(name, torch_cuda):
    """2048 random cameras of one map (bins handed back by the flat rasteriser, depth ties and long lists show up in
    large batches): labels equal the oracle's; the same cameras in two other orders give the same labels camera for
    camera, and segment=True does too."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps

    md = maps.load_map(name)
    N, W, H = 2048, 160, 120
    px, pz, ang = random_poses(md, N, 2024)
    env = labelled_env(N, name, W, H)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    first = env.labels.clone()
    _, _, lab = oracle_batch(md, px, pz, ang, W, H)
    assert_same_labels(first, lab, f"large batch {name}")
    env.render_obs(segment=True)
    assert torch.equal(env.labels, first), "segment=True changed the labels"
    rng = np.random.default_rng(8)
    for perm in (np.arange(N)[::-1].copy(), rng.permutation(N)):
        env.sim.reset(None, dict(pos_x=px[perm].copy(), pos_z=pz[perm].copy(), angle=ang[perm].copy()))
        env.render_obs()
        idx = torch.from_numpy(perm).to(env.device)
        assert torch.equal(env.labels, first[idx]), "labels depend on the order of the batch"
    env.check()
    env.close()


@pytest.mark.parametrize("name,W,H,N", [("udem1", 160, 120, 96), ("small_loop", 84, 84, 96), ("udem1", 640, 480, 8)])
def test_labels_follow_fisheye_pinhole_rectification_and_top_down(name, W, H, N, torch_cuda):
    """The fisheye frame's labels are the oracle's gathered through the fisheye LUT (0 where it names no source); under
    `undistort` the pinhole labels, with a rectification installed those gathered through it; render_obs(top_down=True)
    the labels of the camera above the map, the agent's own mesh among them."""
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 31)
    env = labelled_env(N, name, W, H, distortion=True)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    fish = (env.camera_model.rmapx, env.camera_model.rmapy)
    obs = env.render_obs()
    rgb, dep, lab = oracle_batch(md, px, pz, ang, W, H, lut=fish)
    assert_same_labels(env.labels, lab, "fisheye")
    assert np.array_equal(obs.cpu().numpy(), rgb)
    assert np.array_equal(lab != 0, dep != 0)
    env.undistort = True
    env.render_obs()
    _, _, pin = oracle_batch(md, px, pz, ang, W, H)
    assert_same_labels(env.labels, pin, "pinhole")
    lut = rect_lut(W, H)
    env.set_rectification(*lut)
    env.sim.render(env.obs.data_ptr(), env._stream())     # the reset / step observation: rectified
    _, _, rect = oracle_batch(md, px, pz, ang, W, H, lut=lut)
    assert_same_labels(env.labels, rect, "rectified")
    env.render_obs(top_down=True)
    k = min(N, 12)
    _, _, top = oracle_batch(md, px[:k], pz[:k], ang[:k], W, H, top_down=True)
    assert_same_labels(env.labels[:k], top, "top-down")
    assert (top == 2 + md.grid_w * md.grid_h + len(md.objects)).any(), "the agent's mesh is in the top-down view"
    env.check()
    env.close()


@pytest.mark.parametrize("setup", ["chw_f32", "cwh_u8", "resize_cv2", "resize_pil_chw_f32"])
def test_labels_keep_their_layout_and_size_under_wrapper_formats_and_resize(setup, torch_cuda):
    from gym_duckietown_b200 import maps
    name, N, W, H = "loop_obstacles", 64, 160, 120
    md = maps.load_map(name)
    px, pz, ang = random_poses(md, N, 77)
    env = labelled_env(N, name, W, H)
    if "chw_f32" in setup:
        env.set_output_format(obs_layout="chw", obs_dtype="float32")
    if setup == "cwh_u8":
        env.set_output_format(obs_layout="cwh")
    if setup.startswith("resize"):
        env.set_resize(84, 84, method="cv2_cubic" if "cv2" in setup else "pil_bilinear")
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    assert tuple(env.labels.shape) == (N, H, W)
    _, _, lab = oracle_batch(md, px, pz, ang, W, H)
    assert_same_labels(env.labels, lab, setup)
    env.check()
    env.close()


@pytest.mark.parametrize("name,dr", [("small_loop", False), ("loop_obstacles", True)])
def test_auto_reset_rollout_with_terminal_obs_labels_match_obs(name, dr, torch_cuda):
    """Device auto-reset with terminal_obs=True: after every step env.labels is the oracle's labels of the state obs
    shows (for ended envs redrawn by the listed pass), and obs, reward, done equal those of the same env without labels."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    N, W, H, T = 48, 160, 120, 14
    kw = dict(domain_rand=dr, seed=11, device_reset=True, auto_reset=True, terminal_obs=True, max_steps=6)
    env, plain = labelled_env(N, name, W, H, depth=False, **kw), make_env(N, name, W, H, depth=False, **kw)
    assert plain.labels is None
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
        _, _, lab = oracle_batch(md, px, pz, ang, W, H, device_episodes(env) if dr else None, dr)
        assert_same_labels(env.labels, lab, f"{name} step {t} ({int(done.sum())} envs ended)")
    assert ended >= N, f"only {ended} episodes ended"
    env.check(); plain.check()
    env.close(); plain.close()


def test_batch_of_two_maps_labels_refer_to_each_envs_map(torch_cuda):
    import oracle as orc
    from gym_duckietown_b200 import maps
    names = ["small_loop", "udem1"]
    mds = [maps.load_map(n) for n in names]
    N, W, H = 64, 160, 120
    env = labelled_env(N, names, W, H, seed=2)
    mid = (np.arange(N) % 2).astype(np.int32)
    P = np.zeros((N, 3))
    for m in range(2):
        k = np.flatnonzero(mid == m)
        P[k] = np.stack(random_poses(mds[m], len(k), 40 + m), axis=1)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), map_id=mid))
    env.render_obs()
    got = env.labels.cpu().numpy()
    for m in range(2):
        k = np.flatnonzero(mid == m)
        _, _, lab = label_oracle.render_batch(orc.OracleScene(mds[m]), P[k, 0], P[k, 1], P[k, 2], W=W, H=H)
        assert_same_labels(got[k], lab, f"map {names[m]}")
        assert got[k].max() < len(env.label_table(m))
    env.check()
    env.close()


def test_hidden_objects_never_appear(torch_cuda):
    """Objects hidden for an episode (obj_hidden, as domain randomisation hides optional ones) have no pixel."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    name, W, H = "udem1", 160, 120
    md = maps.load_map(name)
    rng = np.random.default_rng(6)
    P = []
    for o in md.objects:
        for d in (0.3, 0.8):
            a = rng.uniform(-np.pi, np.pi)
            P.append((o.pos[0] - d * np.cos(a), o.pos[2] + d * np.sin(a), a))
    P = np.array(P)
    N = len(P)
    hidden = np.zeros((N, 8), np.uint32)
    for e in range(N):
        for o in range(len(md.objects)):
            if (e + o) % 2 == 0:
                hidden[e, o >> 5] |= np.uint32(1 << (o & 31))
    env = labelled_env(N, name, W, H, seed=3)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), obj_hidden=hidden))
    env.render_obs()
    got = env.labels.cpu().numpy()
    eps = [orc.default_episode() for _ in range(N)]
    for e, ep in enumerate(eps):
        for i in range(8):
            ep.hidden[i] = int(hidden[e, i])
    _, _, lab = oracle_batch(md, P[:, 0], P[:, 1], P[:, 2], W, H, eps)
    assert_same_labels(got, lab, "hidden objects")
    n_cells = md.grid_w * md.grid_h
    shown = 0
    for e in range(N):
        objs = set((np.unique(got[e]) - 2 - n_cells).tolist()) & set(range(len(md.objects)))
        assert not any((e + o) % 2 == 0 for o in objs), f"env {e} shows a hidden object"
        shown += len(objs)
    assert shown > N // 2
    env.check()
    env.close()


def test_null_target_stops_the_writes_and_misaligned_targets_are_refused(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    name, N, W, H = "small_loop", 32, 160, 120
    md = maps.load_map(name)
    env = labelled_env(N, name, W, H, seed=9, depth=False)
    env.reset()
    px, pz, ang = poses_of(env)
    _, _, lab = oracle_batch(md, px, pz, ang, W, H)
    assert_same_labels(env.labels, lab, "before")
    env.sim.set_label_target(None)
    env.labels.fill_(-7)
    env.render_obs()
    env.step(torch.zeros((N, 2), device=env.device))
    torch.cuda.synchronize()
    assert (env.labels == -7).all(), "labels were written with no target set"
    other = torch.full_like(env.labels, -1)
    env.sim.set_label_target(other.data_ptr())
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    env.render_obs()
    assert_same_labels(other, lab, "new target")
    assert (env.labels == -7).all()
    with pytest.raises(Exception):
        env.sim.set_label_target(other.data_ptr() + 1)      # not an int16 address
    env.check()
    env.close()


def test_object_boxes_equal_a_numpy_reduction(torch_cuda):
    from gym_duckietown_b200 import maps
    names = ["loop_obstacles", "udem1"]
    mds = [maps.load_map(n) for n in names]
    N, W, H = 48, 160, 120
    env = labelled_env(N, names, W, H, seed=4)
    mid = (np.arange(N) % 2).astype(np.int32)
    P = []
    rng = np.random.default_rng(1)
    for e in range(N):
        objs = mds[mid[e]].objects
        o = objs[e % len(objs)]
        d, a = rng.uniform(0.3, 1.5), rng.uniform(-np.pi, np.pi)
        P.append((o.pos[0] - d * np.cos(a), o.pos[2] + d * np.sin(a), a))
    P = np.array(P)
    env.sim.reset(None, dict(pos_x=P[:, 0].copy(), pos_z=P[:, 1].copy(), angle=P[:, 2].copy(), map_id=mid))
    env.render_obs()
    pixels, boxes = env.object_boxes()
    n_obj = max(len(md.objects) for md in mds)
    assert pixels.shape == (N, n_obj) and boxes.shape == (N, n_obj, 4)
    lab = env.labels.cpu().numpy()
    want_px, want_box = np.zeros((N, n_obj), np.int32), np.full((N, n_obj, 4), -1, np.int32)
    for e in range(N):
        md = mds[mid[e]]
        for o in range(len(md.objects)):
            ys, xs = np.nonzero(lab[e] == 2 + md.grid_w * md.grid_h + o)
            want_px[e, o] = len(xs)
            if len(xs):
                want_box[e, o] = (xs.min(), ys.min(), xs.max(), ys.max())
    assert np.array_equal(pixels.cpu().numpy(), want_px)
    assert np.array_equal(boxes.cpu().numpy(), want_box)
    assert (want_px > 0).sum() >= N // 2
    env.check()
    env.close()


def test_single_env_adapter_exposes_labels(torch_cuda):
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.simulator import DuckietownEnv
    W, H = 160, 120
    e = DuckietownEnv(map_name="loop_obstacles", domain_rand=False, camera_width=W, camera_height=H, seed=4, labels=True)
    off = DuckietownEnv(map_name="small_loop", domain_rand=False, camera_width=W, camera_height=H, seed=4)
    assert off.labels is None
    off.close()
    md = maps.load_map("loop_obstacles")
    for step in range(3):
        if step:
            e.step(np.array([0.6, 0.3]))
        lb = e.labels
        assert isinstance(lb, np.ndarray) and lb.shape == (H, W) and lb.dtype == np.int16
        _, _, lab = oracle_batch(md, [e.cur_pos[0]], [e.cur_pos[2]], [e.cur_angle], W, H)
        assert_same_labels(lb, lab[0], f"adapter step {step}")
    e.render(mode="rgb_array")          # the 800x600 view has no labels and leaves these alone
    assert np.array_equal(e.labels, lb)
    e.close()
