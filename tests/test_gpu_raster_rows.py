"""k_raster's two ways of picking its work: the rows k_bin and k_raster_flat put on its list, or every row of every env.

With packed u8 HWC output k_raster_solo clears the empty coarse bins (without a LUT) and draws the bins inside one prim,
k_raster_flat the flat ones, so k_raster draws only the rows k_bin listed (a bin that neither took) and the rows of the
bins k_raster_flat hands back.  On a gathering step k_raster walks every row instead, since it ships each finished row,
the ones the others drew included, to every rank.  The same state drawn both ways must give the same bytes in obs and
in every image: a row missing from the list would keep the previous contents there.  Each case draws once without a
gather (the list) and once with FusedObsGather(env, 0, 1) armed (every row), over buffers filled with other bytes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, name, w=160, h=120, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, seed=9)
    args.update(kw)
    return BatchedDuckietownEnv(n, name, **args)


def random_poses(env, n, seed):
    """n cameras on random drivable tiles of map 0, any heading"""
    md = env.maps[0]
    rng = np.random.default_rng(seed)
    cells = np.array(md.drivable_tiles)[rng.integers(len(md.drivable_tiles), size=n)]
    px = (cells[:, 0] + rng.uniform(size=n)) * md.tile_size
    pz = (cells[:, 1] + rng.uniform(size=n)) * md.tile_size
    return px, pz, rng.uniform(-np.pi, np.pi, size=n)


def place(env, px, pz, ang):
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))


def targets(env):
    return [env.obs] + [getattr(env, k) for k in ("depth", "labels", "markings") if getattr(env, k, None) is not None]


def images(env, torch):
    """obs and every image target of the last render, as bytes"""
    torch.cuda.synchronize()
    out = {"obs": env.obs.contiguous().view(-1).view(torch.uint8).clone()}
    for k in ("depth", "labels", "markings"):
        t = getattr(env, k, None)
        if t is not None:
            out[k] = t.contiguous().view(-1).view(torch.uint8).clone()
    return out


def assert_both_walks_agree(env, torch, render=None, gather=None):
    """Draws the env's current state twice through `render` (default: dts_render in the env's own mode, fisheye and
    rectification included): from k_raster's row list, then on a gathering step, each over targets filled with other
    bytes.  obs and every image must be equal byte for byte, and the gather's slot must be obs."""
    from gym_duckietown_b200.dist import FusedObsGather
    render = render or (lambda: env.sim.render(env.obs.data_ptr(), env._stream()))
    g = gather or FusedObsGather(env, 0, 1)
    for t in targets(env):
        t.fill_(0x3C if t.dtype == torch.uint8 else 3)
    render()
    listed = images(env, torch)
    for t in targets(env):
        t.fill_(0x5A if t.dtype == torch.uint8 else 7)
    g.arm()
    render()
    full = images(env, torch)
    slot = g.finish()[0]
    assert torch.equal(slot.contiguous().view(-1).view(torch.uint8), full["obs"]), "the gather's slot is not obs"
    assert listed.keys() == full.keys()
    for k in listed:
        diff = int((listed[k] != full[k]).sum())
        assert diff == 0, f"{k}: {diff} bytes differ between the row list and the walk over every row"
    assert float(env.obs.float().std()) > 5, "not a rendered frame"
    return g


def test_large_batch_with_hand_backs(torch_cuda):
    """2048 random cameras on small_loop (the batch where k_raster_flat hands bins back to k_raster), with depth and
    labels; then the same cameras with markings."""
    torch = torch_cuda
    for kw in (dict(depth=True, labels=True), dict(markings=True)):
        env = make_env(2048, "small_loop", **kw)
        place(env, *random_poses(env, 2048, 2024))
        assert_both_walks_agree(env, torch)
        env.check()
        env.close()


def test_mesh_rows_loop_obstacles(torch_cuda):
    """loop_obstacles: the duckies' and cones' bins (mesh and tiny triangles) stay k_raster's, on rows beside bins the
    lean kernels drew; depth, labels and markings"""
    torch = torch_cuda
    env = make_env(512, "loop_obstacles", depth=True, labels=True, markings=True)
    place(env, *random_poses(env, 512, 7))
    assert_both_walks_agree(env, torch)
    env.check()
    env.close()


def test_cameras_at_the_horizon(torch_cuda):
    """Cameras on the map's border looking out over the bare ground: rows of sky and ground only, which k_raster does
    not draw at all, and rows of the horizon, where empty bins meet ground bins"""
    torch = torch_cuda
    n = 256
    env = make_env(n, "small_loop", depth=True, labels=True)
    md = env.maps[0]
    rng = np.random.default_rng(3)
    side = rng.integers(4, size=n)
    t = rng.uniform(0.0, 1.0, size=n)
    gw, gh = md.grid_w * md.tile_size, md.grid_h * md.tile_size
    px = np.where(side == 0, 0.05, np.where(side == 1, gw - 0.05, t * gw))
    pz = np.where(side == 2, 0.05, np.where(side == 3, gh - 0.05, t * gh))
    out = np.array([np.pi, 0.0, np.pi / 2, -np.pi / 2])[side]   # looking out of the map, +- up to 57 degrees
    place(env, px, pz, out + rng.uniform(-1.0, 1.0, size=n))
    assert_both_walks_agree(env, torch)
    env.check()
    env.close()


@pytest.mark.parametrize("W,H", [(100, 76), (96, 60)])
def test_border_bins(W, H, torch_cuda):
    """Cameras whose right column of coarse bins is narrower than 32 pixels and whose last row of bins is 4 rows high:
    the empty bins there are cleared row by row up to the image's edge"""
    torch = torch_cuda
    env = make_env(256, "small_loop", W, H, depth=True, labels=True, markings=True)
    place(env, *random_poses(env, 256, 13))
    assert_both_walks_agree(env, torch)
    env.check()
    env.close()


def test_domain_rand_horizon_per_env(torch_cuda):
    """domain_rand: every env clears its empty bins to its own horizon colour"""
    torch = torch_cuda
    env = make_env(512, "loop_obstacles", domain_rand=True, depth=True, labels=True)
    env.reset()
    assert_both_walks_agree(env, torch)
    env.check()
    env.close()


@pytest.mark.parametrize("view", ["segment", "top_down"])
def test_segment_and_top_down_views(view, torch_cuda):
    """segment (empty bins magenta) and top-down views, through render_obs"""
    torch = torch_cuda
    env = make_env(256, "loop_obstacles", labels=True)
    place(env, *random_poses(env, 256, 11))
    assert_both_walks_agree(env, torch, render=lambda: env.render_obs(**{view: True}))
    env.check()
    env.close()


@pytest.mark.parametrize("lens", ["fisheye", "camera_rand_pool", "undistort"])
def test_remapped_frames(lens, torch_cuda):
    """The fisheye LUT, a camera_rand pool of four LUTs and UndistortWrapper's rectification: k_raster clears the empty
    bins there (0 where the LUT names no source), on the rows k_bin lists"""
    torch = torch_cuda
    kw = dict(distortion=True, depth=True, labels=True)
    if lens == "camera_rand_pool":
        kw.update(camera_rand=True, camera_rand_pool=4)
    env = make_env(256, "loop_obstacles", **kw)
    if lens == "undistort":
        from gym_duckietown_b200.distortion import rectify_maps
        env.set_rectification(*rectify_maps(env.camera_width, env.camera_height))
        env.undistort = True
    place(env, *random_poses(env, 256, 5))
    assert_both_walks_agree(env, torch)
    env.check()
    env.close()


def test_terminal_step_second_pass(torch_cuda):
    """dts_step_terminal with envs ending: its second pass draws the listed envs from their rows on the list.  What obs
    holds after the step is the frame of every env's current state, which a gathering render draws over every row."""
    torch = torch_cuda
    n = 256
    env = make_env(n, "loop_obstacles", auto_reset=True, device_reset=True, terminal_obs=True, max_steps=6,
                   depth=True, labels=True)
    env.reset()
    from gym_duckietown_b200.dist import FusedObsGather
    g = FusedObsGather(env, 0, 1)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(4)
    acts = torch.rand((6, n, 2), device=env.device, generator=gen) * 2 - 1
    for t in range(6):
        if t == 2:   # the odd envs start over: only the even ones reach max_steps on the last step
            env.reset(mask=torch.arange(n, device=env.device) % 2 == 1)
        _, _, done, _ = env.step(acts[t])
    torch.cuda.synchronize()
    assert 0 < int(done.sum()) < n, "no env (or every env) ended on the last step"
    stepped = images(env, torch)
    assert_both_walks_agree(env, torch, gather=g)
    again = images(env, torch)
    for k in stepped:
        assert torch.equal(stepped[k], again[k]), f"{k}: the terminal step's frames differ from a render of the same state"
    env.check()
    env.close()


def test_frame_memory_overflow_still_raises(monkeypatch, torch_cuda):
    """A pair pool of one env's bound for 64 envs: the frames that did not fit are the clear colour everywhere whether
    k_raster walks its list or every row, the overflow is flagged, env.check() raises, and the next render is refused."""
    torch = torch_cuda
    from gym_duckietown_b200.dist import FusedObsGather
    from gym_duckietown_b200.lib import DtsError
    monkeypatch.setenv("DTS_PAIR_POOL_GB", "1e-6")   # read when the frame memory is reserved, at the first render
    n = 64
    frames, overs = [], []
    for gathered in (False, True):
        env = make_env(n, "small_loop")
        place(env, *random_poses(env, n, 31))
        g = FusedObsGather(env, 0, 1)
        env.obs.fill_(0x5A)
        if gathered:
            g.arm()
        env.sim.render(env.obs.data_ptr(), env._stream())
        torch.cuda.synchronize()
        n_cells = env.maps[0].grid_w * env.maps[0].grid_h
        over = np.array([env.sim.debug_frame(k, n_cells)["overflow"] for k in range(n)])
        assert set(over.tolist()) == {0, 1}, f"{int(over.sum())} of {n} frames overflowed: pick n so that both occur"
        got = env.obs.cpu().numpy()
        for k in np.flatnonzero(over == 1):
            h = env.sim.debug_episode(int(k))["horizon"].astype(np.float32)
            clear = np.minimum(np.rint(h * np.float32(255.0)), 255).astype(np.uint8)
            assert (got[k] == clear).all(), f"env {k} overflowed but is not the clear colour"
        assert env.sim.status() & 1
        with pytest.raises(DtsError):
            env.check()
        with pytest.raises(DtsError, match="overflowed its render frame memory"):
            env.sim.render(env.obs.data_ptr(), env._stream())
        frames.append(got)
        overs.append(over)
        env.close()
    # which envs overflow depends on the order the envs reach the pool: compare those that fit or overflowed in both
    same = overs[0] == overs[1]
    assert same.any()
    assert np.array_equal(frames[0][same], frames[1][same])
