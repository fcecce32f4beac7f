"""The snapshot record layout, pinned byte for byte (dts_save_state, DESIGN.md §2 "Snapshots").

Save/load round trips pass for any layout that agrees with itself, so they cannot tell a row left out, two rows swapped
or the rows reordered.  Here each env's record is built on the host from the documented order, out of values read
through other entry points (state arrays, device streams, the raw RenderEp, the obstacles' state) and values known
right after a host-parameter reset, and save_state() must equal it.  Every env gets its own pose, wheel distance, trim,
camera and lights, and its own stream, so a misplaced row shows as a mismatch.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "include", "dtsim.h")) as _f:
    MAX_DELAY = int(re.search(r"#define DTS_MAX_DELAY (\d+)", _f.read()).group(1))
N = 45   # not a multiple of the save kernel's 32-env groups


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def host_params(mds, mid, rng):
    """dts_episode_params that differ in every env: a pose inside its map, wheel_dist, trim, camera, lights, mask."""
    n = len(mid)
    ts = np.array([mds[m].tile_size for m in mid])
    gw, gh = np.array([mds[m].grid_w for m in mid]), np.array([mds[m].grid_h for m in mid])
    f32 = lambda lo, hi, *shape: rng.uniform(lo, hi, (n,) + shape).astype(np.float32)
    return dict(map_id=mid.astype(np.int32), pos_x=rng.uniform(0.1, 0.9, n) * gw * ts,
                pos_z=rng.uniform(0.1, 0.9, n) * gh * ts, angle=rng.uniform(-np.pi, np.pi, n),
                wheel_dist=rng.uniform(0.09, 0.11, n), trim=rng.normal(0, 0.02, n),
                cam_height=f32(0.09, 0.12), cam_angle_deg=f32(-20, -10), cam_fov_y_deg=f32(50, 70),
                cam_noise=f32(-0.005, 0.005, 3), horizon_color=f32(0, 1, 3), light_ambient=f32(0, 1, 3),
                light_diffuse=f32(0, 1, 3), light_pos=f32(-2, 2, 4), ground_color=f32(0, 1, 3),
                obj_hidden=rng.integers(0, 2 ** 32, (n, 8), dtype=np.uint32))


def expected_records(env, mds, p):
    """Each env's record in the documented order: RenderEp; the 16 doubles; the delay line; the stream; every map
    slot's obstacles; the five int32s; the three bytes; zero padding to a multiple of 16."""
    import torch
    torch.cuda.synchronize()
    n = env.num_envs
    st = {k: v.cpu().numpy() for k, v in env.state.items()}
    rep = np.zeros((n, 144), np.uint8)
    for e in range(n):
        assert env.sim.lib.dts_debug_episode(env.sim.h, e, rep[e].ctypes.data_as(C.c_void_p)) == 0
    grid_h = np.array([mds[m].grid_h for m in st["map_id"]])
    ts = np.array([mds[m].tile_size for m in st["map_id"]])
    zero = np.zeros(n)
    # right after the reset: cartesian pose from the simulator one (S:1629-1638), no velocity, an empty delay line
    f64 = [p["pos_x"], grid_h * ts - p["pos_z"], p["angle"], zero, zero, st["pos_x"], st["pos_z"], st["angle"],
           st["speed"], st["reward"], st["lane_dist"], st["lane_dot"], st["lane_angle_rad"], st["prox_penalty"],
           st["wheel_dist"], p["trim"]] + [zero] * (2 * MAX_DELAY)
    streams = env.sim.debug_streams()
    m64 = (1 << 64) - 1
    rows = [np.array([(s["state"]["state"] >> 64, s["state"]["state"] & m64, s["state"]["inc"] >> 64,
                       s["state"]["inc"] & m64, s["has_uint32"], s["uinteger"]) for s in streams], np.uint64).T]
    for m in range(len(mds)):
        arr, nd = env.sim.dyn_state(m)
        if nd:
            rows.append(torch.as_tensor(arr, device=env.device).cpu().numpy().reshape(-1, n))
    cols = [rep] + [np.asarray(r, np.float64) for r in f64] + [r for block in rows for r in block]
    cols += [st[k] for k in ("step_count", "tile_i", "tile_j", "map_id", "episode", "done_code", "in_lane", "collided")]
    rec = np.concatenate([np.ascontiguousarray(c).view(np.uint8).reshape(n, -1) for c in cols], axis=1)
    pad = -rec.shape[1] % 16
    return np.concatenate([rec, np.zeros((n, pad), np.uint8)], axis=1)


@pytest.mark.parametrize("maps_,want_bytes", [(["small_loop"], 608), (["loop_dyn_duckiebots"], 1040),
                                              (["small_loop", "loop_dyn_duckiebots"], 1040)])
def test_record_layout_is_the_documented_one(maps_, want_bytes, torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    env = BatchedDuckietownEnv(N, maps_ if len(maps_) > 1 else maps_[0], camera_width=64, camera_height=48,
                               domain_rand=False, seed=5)
    try:
        mds = env.maps
        rng = np.random.default_rng(17)
        env.reset()
        g = torch.Generator(device="cuda").manual_seed(2)
        for _ in range(3):   # the obstacles walk, and every env has an episode behind it
            env.step(torch.rand((N, 2), device="cuda", generator=g) * 2 - 1)
        env.sim.seed_streams([np.random.default_rng([23, e]) for e in range(N)])
        mid = np.arange(N) % len(mds)
        p = host_params(mds, mid, rng)
        env.sim.reset(None, p, env._stream())
        want = expected_records(env, mds, p)
        got = env.save_state()
        torch.cuda.synchronize()
        got = got.cpu().numpy()
        assert env.sim.state_info()[0] == want.shape[1] == want_bytes
        assert got.shape == want.shape
        bad = np.flatnonzero((got != want).any(0))
        assert len(bad) == 0, f"record bytes {bad[:16].tolist()} differ from the documented layout"
        # the rows really carry per-env values: no two envs' records share their stream or their RenderEp
        assert len({bytes(r) for r in want[:, :144]}) == N and len({bytes(r) for r in want}) == N
    finally:
        env.close()
