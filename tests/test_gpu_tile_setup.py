"""Road tiles of tile mode 1 are set up one lane per tile (k_tiles): a warp per env takes the map's grid cells 32 at a
time, and only the tiles that need the clipper (or whose snapped quad is not strictly convex) go through the warp-wide
triangle path, one at a time.

Pinned here:
  - what a frame leaves in frame memory does not depend on the batch around it: per env, the prim count, the lattice
    count and the lit lattice of every grid cell are the same in a batch of its own, permuted inside a larger batch,
    and in a render over a device list of envs (dts_step_terminal's second pass);
  - frames equal the raster oracle at 0 LSB on loop_obstacles (56 grid cells: two chunks of lanes) and at hand-placed
    poses that put tiles across the near plane and the guard band (the fallback path)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H = 160, 120


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(autouse=True)
def _tile_mode_1():
    import oracle as orc
    orc.lib().orr_set_tile_mode(1)
    yield


def random_poses(md, n, seed):
    rng = np.random.default_rng(seed)
    cells = np.array(md.drivable_tiles)[rng.integers(len(md.drivable_tiles), size=n)]
    px = (cells[:, 0] + rng.uniform(size=n)) * md.tile_size
    pz = (cells[:, 1] + rng.uniform(size=n)) * md.tile_size
    return px, pz, rng.uniform(-np.pi, np.pi, size=n)


def frame_memory(env, envs, n_cells):
    out = []
    for e in envs:
        d = env.sim.debug_frame(int(e), n_cells)
        assert d["overflow"] == 0
        out.append((d["n_prims"], d["n_lat"], d["lattice"]))
    return out


def assert_same_frame_memory(a, b, what):
    for k, ((pa, la, xa), (pb, lb, xb)) in enumerate(zip(a, b)):
        assert (pa, la) == (pb, lb), f"{what}, env {k}: n_prims / n_lat {pa} / {la} vs {pb} / {lb}"
        assert np.array_equal(xa, xb, equal_nan=True), f"{what}, env {k}: lattice by cell differs"


@pytest.mark.parametrize("name", ["small_loop", "loop_obstacles"])
def test_frame_memory_does_not_depend_on_the_batch(name, torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv

    md = maps.load_map(name)
    n_cells = md.grid_w * md.grid_h
    n, extra = 96, 61
    px, pz, ang = random_poses(md, n, 31)
    a = BatchedDuckietownEnv(n, name, camera_width=W, camera_height=H, domain_rand=False, seed=5)
    a.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    fa = a.render_obs().clone()
    torch.cuda.synchronize()
    mem_a = frame_memory(a, range(n), n_cells)
    assert sum(m[1] for m in mem_a) > 4 * n

    # the same envs at permuted places of a larger batch, among other cameras
    perm = np.random.default_rng(7).permutation(n + extra)
    qx, qz, qa = random_poses(md, n + extra, 32)
    qx[perm[:n]], qz[perm[:n]], qa[perm[:n]] = px, pz, ang
    b = BatchedDuckietownEnv(n + extra, name, camera_width=W, camera_height=H, domain_rand=False, seed=5)
    b.sim.reset(None, dict(pos_x=qx, pos_z=qz, angle=qa))
    fb = b.render_obs().clone()
    torch.cuda.synchronize()
    assert torch.equal(fa, fb[torch.as_tensor(perm[:n], device=fb.device)]), "frames differ inside a larger batch"
    assert_same_frame_memory(mem_a, frame_memory(b, perm[:n], n_cells), "permuted in a larger batch")
    a.close()
    b.close()

    # a render over a device list: every episode ends after one step, so dts_step_terminal's second pass lists every
    # env (in the order they were appended) and draws the respawned states; then a full render of the same states
    c = BatchedDuckietownEnv(n, name, camera_width=W, camera_height=H, domain_rand=False, seed=9, device_reset=True,
                             max_steps=1, auto_reset=True, terminal_obs=True)
    c.reset()
    act = torch.zeros((n, 2), device="cuda")
    act[:, 0] = 0.5
    _, _, done, _ = c.step(act)
    torch.cuda.synchronize()
    assert bool(done.all())
    listed_obs = c.obs.clone()
    mem_listed = frame_memory(c, range(n), n_cells)
    full_obs = c.render_obs().clone()
    torch.cuda.synchronize()
    assert torch.equal(listed_obs, full_obs), "listed render differs from the full render of the same states"
    assert_same_frame_memory(mem_listed, frame_memory(c, range(n), n_cells), "listed render")
    c.close()


def hand_placed_poses(md):
    """Cameras on tile corners and borders, at the map's edge, looking along and across the grid: the tile under the
    camera crosses the near plane, and neighbours reach far past the image into the guard band."""
    ts, gw, gh = md.tile_size, md.grid_w, md.grid_h
    pts = []
    for (i, j) in [(1, 1), (2, 1), (1, 2), (gw - 2, gh - 2), (gw // 2, gh // 2)]:
        for (dx, dz) in [(0.0, 0.0), (0.5, 0.0), (0.0, 0.5), (0.02, 0.98), (0.999, 0.5)]:
            for k in range(8):
                pts.append(((i + dx) * ts, (j + dz) * ts, -np.pi + k * np.pi / 4 + (0.013 if dx == 0.02 else 0.0)))
    for k in range(16):   # the map's border, facing out and along it
        pts.append((0.01 * ts, (0.5 + k % 4) * ts, np.pi * (k // 4) / 2))
    return [np.array(v, dtype=np.float64) for v in zip(*pts)]


@pytest.mark.parametrize("name,seed", [("loop_obstacles", 11), ("small_loop", None)])
def test_frames_match_the_oracle(name, seed, torch_cuda):
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv

    md = maps.load_map(name)
    if seed is None:
        px, pz, ang = hand_placed_poses(md)
    else:
        px, pz, ang = random_poses(md, 512, seed)
        hx, hz, ha = hand_placed_poses(md)
        px, pz, ang = np.concatenate([px, hx]), np.concatenate([pz, hz]), np.concatenate([ang, ha])
    n = len(px)
    env = BatchedDuckietownEnv(n, name, camera_width=W, camera_height=H, domain_rand=False, seed=5)
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang))
    gpu = env.render_obs().cpu().numpy()
    sc = orc.OracleScene(md)
    cpu = sc.render_batch(px, pz, ang, [orc.default_episode() for _ in range(n)], W, H, False, threads=os.cpu_count() or 1)
    diff = np.abs(gpu.astype(np.int16) - cpu.astype(np.int16))
    assert diff.max() == 0, f"{name}: {int((diff > 0).sum())} channel values differ from the oracle (max {diff.max()} LSB)"
    env.close()
