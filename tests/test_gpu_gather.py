"""The fused end-of-rollout gather (dts_gather_*): the last step's rasteriser stores the frames into slot `rank` of every
rank's gather buffer besides the caller's tensor.

Every case fills the whole buffer with a sentinel byte, takes unarmed steps, arms, and takes one step (or a reset), then
checks (a) the slot equals `obs` byte for byte, (b) every other byte still holds the sentinel, and (c) the next unarmed
step leaves the buffer as it was.  The paths that write the slot: whole 8-row blocks of a packed u8 HWC frame shipped
with 16-byte vectors or, where a frame, a block or a slot is not 16-byte aligned, byte by byte; the wrapper layouts and
float32 stored per bin; the fisheye, a camera_rand pool of fisheye tables and the rectification.  One process on one GPU
covers world = 1; world = 2 and 3 run as that many processes sharing one GPU (cudaIpc handles open across processes on
one device), so that every slot offset and every peer store is exercised.  tools/check_fused_gather.py compares the
fused buffer with the NCCL all-gather across GPUs."""
import ctypes as C
import os
import signal
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xA5
STEPS = 8   # unarmed steps before the armed one: a command acts 0.15 s (5 steps) after it is issued


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, maps="small_loop", w=160, h=120, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=w, camera_height=h, domain_rand=False, seed=21, auto_reset=True, device_reset=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, maps, **args)


def forward_actions(torch, env, steps, seed=3):
    """Velocity in [0.2, 1], steering in [-1, 1]: once the commands act, every step moves the camera."""
    g = torch.Generator(device=env.device)
    g.manual_seed(seed)
    a = torch.rand((steps, env.num_envs, 2), device=env.device, generator=g)
    a[..., 0] = a[..., 0] * 0.8 + 0.2
    a[..., 1] = a[..., 1] * 2 - 1
    return a


def obs_bytes(env):
    import torch
    return env.obs.contiguous().view(-1).view(torch.uint8)


def batch_bytes(env):
    return env.obs.numel() * env.obs.element_size()


class Gather:
    """A gather buffer allocated through the C ABI with any bytes_per_rank; in one process only its own rank's
    buffer can be mapped (world 1)."""

    def __init__(self, env, bytes_per_rank, rank=0, world=1):
        import torch
        from gym_duckietown_b200.lib import _CudaArray
        self.env, self.bytes_per_rank, self.rank, self.world = env, bytes_per_rank, rank, world
        sim = env.sim
        self.handle = (C.c_uint8 * 64)()
        buf = C.c_void_p()
        sim._check(sim.lib.dts_gather_alloc(sim.h, bytes_per_rank, rank, world, self.handle, C.byref(buf)),
                   "dts_gather_alloc")
        self.buf = torch.as_tensor(_CudaArray(buf.value, world * bytes_per_rank, np.uint8), device=env.device)

    def open(self):
        sim = self.env.sim
        handles = np.frombuffer(bytes(self.handle) * self.world, np.uint8).copy()
        sim._check(sim.lib.dts_gather_open(sim.h, handles.ctypes.data_as(C.c_void_p)), "dts_gather_open")

    def arm(self):
        sim = self.env.sim
        sim._check(sim.lib.dts_gather_next(sim.h), "dts_gather_next")

    def assert_sentinel(self, what):
        assert bool((self.buf == SENTINEL).all()), f"{what} wrote the gather buffer"


def gathered_step(torch, env, extra=0, steps=STEPS, reset=False, seed=3, at_armed=None):
    """Sentinel, `steps` unarmed steps, arm, one step (or reset = dts_render); checks (a), (b) and (c), and calls
    at_armed(env) right after the armed call.  Returns the armed call's obs (a copy) and done."""
    batch = batch_bytes(env)
    g = Gather(env, batch + extra)
    g.open()
    g.buf.fill_(SENTINEL)
    acts = forward_actions(torch, env, steps + 2, seed)
    for t in range(steps):
        env.step(acts[t])
    torch.cuda.synchronize()
    g.assert_sentinel("an unarmed step")
    g.arm()
    done = None
    if reset:
        env.reset()
    else:
        _, _, done, _ = env.step(acts[steps])
    torch.cuda.synchronize()
    assert torch.equal(g.buf[:batch], obs_bytes(env)), "(a) the slot is not the armed call's obs"
    assert bool((g.buf[batch:] == SENTINEL).all()), "(b) the armed call wrote past the batch"
    if at_armed:
        at_armed(env)
    armed, kept = env.obs.clone(), g.buf.clone()
    done = None if done is None else done.clone()
    env.obs.zero_()
    env.step(acts[steps + 1])
    torch.cuda.synchronize()
    assert torch.equal(g.buf, kept), "(c) the unarmed step after the armed one wrote the gather buffer"
    assert_rendered(env.obs)                   # ... though it did render
    return armed, done


def assert_rendered(obs):
    """A real frame batch, not a clear colour: u8 values spread, float32 the same in [0, 1]."""
    o = obs.float() * (255.0 if obs.is_floating_point() else 1.0)
    assert float(o.std()) > 10


def oracle_frames(env, name):
    """The raster oracle's frames of every env's current pose (default episode: no domain randomisation)."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    orc.lib().orr_set_tile_mode(1)
    sc = orc.OracleScene(maps.load_map(name))
    st = {k: v.cpu().numpy() for k, v in env.state.items()}
    W, H = env.camera_width, env.camera_height
    return np.stack([sc.render(st["pos_x"][k], st["pos_z"][k], st["angle"][k], None, W, H, False)
                     for k in range(env.num_envs)])


@pytest.mark.parametrize("fmt", [("hwc", "uint8"), ("chw", "float32")])
def test_fused_gather_world1_equals_obs(fmt):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.dist import FusedObsGather

    env = BatchedDuckietownEnv(40, "loop_obstacles", camera_width=160, camera_height=120, domain_rand=False, seed=5,
                               auto_reset=True, device_reset=True)
    env.set_output_format(obs_layout=fmt[0], obs_dtype=fmt[1])
    env.reset()
    g = FusedObsGather(env, 0, 1)
    acts = torch.rand((6, 40, 2), device=env.device) * 2 - 1
    for t in range(5):
        env.step(acts[t])
    assert float(g.gathered.float().abs().sum()) == 0.0          # nothing written before arm()
    g.arm()
    obs, *_ = env.step(acts[5])
    out = g.finish()
    assert out.shape == (1,) + tuple(obs.shape) and torch.equal(out[0], obs) and float(obs.float().std()) > (1 if fmt[1] == 'uint8' else 0.02)
    before = out.clone()
    env.step(acts[0])                                               # not armed: the gather buffer keeps the rollout's frames
    torch.cuda.synchronize()
    assert torch.equal(g.gathered, before)
    env.check()
    env.close()


@pytest.mark.parametrize("reset", [False, True])
def test_lean_packed_u8_ships_every_row(reset, torch_cuda):
    """small_loop 160x120, packed u8 HWC: k_raster_solo, k_raster_flat and k_raster all draw bins, and some rows are drawn
    by the first two alone; every row reaches the slot.  reset=True: the armed call is a reset's dts_render."""
    torch = torch_cuda
    env = make_env(48, "small_loop")
    env.reset()
    armed, _ = gathered_step(torch, env, extra=4096, reset=reset)
    assert_rendered(armed)
    env.check()
    env.close()


@pytest.mark.parametrize("W,H", [(100, 76), (101, 75)])
def test_packed_u8_odd_sizes_equal_obs_and_oracle(W, H, torch_cuda):
    """100x76: the lean rasterisers with a 4-row last block of rows (16-byte aligned).  101x75: W % 4 != 0, so every bin
    goes through the general store and the rows are shipped after it; a 3-row last block, and every odd env's frame
    starts at an odd byte, so the rows go byte by byte.  The armed frames are the raster oracle's at 0 LSB."""
    torch = torch_cuda
    env = make_env(32, "loop_obstacles", W, H, auto_reset=False, device_reset=False)   # host resets: default episodes
    env.reset()

    def vs_oracle(e):
        assert np.array_equal(e.obs.cpu().numpy(), oracle_frames(e, "loop_obstacles")), "the armed frames are not the oracle's"
    armed, _ = gathered_step(torch, env, extra=1000 + W, at_armed=vs_oracle)
    assert_rendered(armed)
    env.check()
    env.close()


@pytest.mark.parametrize("W,H", [(160, 120), (101, 75)])
@pytest.mark.parametrize("layout,dtype", [("hwc", "float32"), ("chw", "uint8"), ("chw", "float32"), ("cwh", "uint8"),
                                          ("cwh", "float32")])
def test_wrapper_formats_are_stored_per_bin(layout, dtype, W, H, torch_cuda):
    """Every layout / dtype other than packed u8 HWC: the resolve stores each bin into the caller's tensor and into
    every peer's slot (the planar u8 fast store is not used while a gather is armed)."""
    torch = torch_cuda
    env = make_env(40, "loop_obstacles", W, H)
    env.set_output_format(obs_layout=layout, obs_dtype=dtype)
    env.reset()
    armed, _ = gathered_step(torch, env, extra=4099)
    assert_rendered(armed)
    env.check()
    env.close()


@pytest.mark.parametrize("lens", ["fisheye", "camera_rand_pool", "rectified"])
def test_fisheye_pool_and_rectification(lens, torch_cuda):
    """The remapping rasterisers: the fisheye LUT, a camera_rand pool of four LUTs (the kRemapPool instances, each env
    through its own table) and UndistortWrapper's rectification."""
    torch = torch_cuda
    kw = dict(distortion=True)
    if lens == "camera_rand_pool":
        kw.update(camera_rand=True, camera_rand_pool=4)
    env = make_env(48, "loop_obstacles", **kw)
    if lens == "camera_rand_pool":
        assert len(set(env.calibration_of_env.tolist())) == 4
    if lens == "rectified":
        from gym_duckietown_b200.distortion import rectify_maps
        env.set_rectification(*rectify_maps(env.camera_width, env.camera_height))
        env.undistort = True
    env.reset()
    armed, _ = gathered_step(torch, env, extra=64)
    assert_rendered(armed)
    env.check()
    env.close()


@pytest.mark.parametrize("W,H", [(160, 120), (101, 75)])
def test_depth_and_labels_are_unchanged_by_the_gather(W, H, torch_cuda):
    """With depth and label targets set, the gathering step's obs, depth and labels are byte for byte those of an
    unarmed run of the same seed and actions; the slot carries obs only."""
    torch = torch_cuda
    kw = dict(depth=True, labels=True)
    env, plain = make_env(40, "loop_obstacles", W, H, **kw), make_env(40, "loop_obstacles", W, H, **kw)
    env.reset()
    plain.reset()

    def vs_unarmed(e):
        acts = forward_actions(torch, plain, STEPS + 2)    # gathered_step's actions: the unarmed steps, the armed one
        for t in range(STEPS + 1):
            plain.step(acts[t])
        torch.cuda.synchronize()
        assert torch.equal(e.obs, plain.obs)
        assert torch.equal(e.depth.view(torch.int32), plain.depth.view(torch.int32))
        assert torch.equal(e.labels, plain.labels)
        assert bool((e.labels != 0).any()) and float(e.depth.max()) > 0
    gathered_step(torch, env, extra=512, at_armed=vs_unarmed)
    env.check()
    env.close()
    plain.close()


def test_multi_map_cycled_batch_with_envs_ending_on_the_gathered_step(torch_cuda):
    """bench c5's shape: six maps cycled on reset, device auto-reset, and a short max_steps, so that envs end on the
    gathered step and the slot holds their next episode's first frame, as obs does."""
    torch = torch_cuda
    names = ["small_loop", "loop_obstacles", "udem1", "loop_pedestrians", "loop_dyn_duckiebots", "loop_trafficlights"]
    env = make_env(64, names, cycle_maps=True, max_steps=STEPS + 1)   # the armed step is the episodes' last
    env.reset()
    envs = torch.arange(64, device=env.device)
    for j in range(1, 6):                      # each reset moves an env to the next map: env e ends on map e mod 6
        env.reset(mask=envs % 6 >= j)
    assert torch.equal(env.state["map_id"].long(), envs % 6)
    armed, done = gathered_step(torch, env, extra=96)
    assert bool(done.any()), "no env ended on the gathered step"
    assert_rendered(armed)
    env.check()
    env.close()


# ---- refusals: each leaves the state, obs and the gather buffer as they were -----------------------------------------
def snapshot(torch, env):
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in env.state.items()}, env.obs.clone()


def assert_unchanged(torch, env, snap, what):
    torch.cuda.synchronize()
    state, obs = snap
    for k, v in env.state.items():
        assert torch.equal(v, state[k]), f"{what}: state[{k!r}] advanced"
    assert torch.equal(env.obs, obs), f"{what}: obs was written"


def test_refuses_a_batch_that_outgrows_its_buffer(torch_cuda):
    """The buffer is sized for u8 frames; obs switched to float32 afterwards is four times larger.  FusedObsGather.arm()
    and dts_gather_next refuse to arm; a step or render armed before the switch is refused before it launches anything,
    and the gather stays armed for the next call whose batch fits."""
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200.dist import FusedObsGather
    env = make_env(32, "loop_obstacles")
    env.reset()
    g = FusedObsGather(env, 0, 1)
    g.gathered.view(torch.uint8).fill_(SENTINEL)
    batch = batch_bytes(env)
    acts = forward_actions(torch, env, 3)
    env.step(acts[0])
    env.set_output_format(obs_dtype="float32")
    env.step(acts[0])
    sim = env.sim
    snap = snapshot(torch, env)
    with pytest.raises(ValueError, match="was built for observations torch.uint8"):
        g.arm()
    assert sim.lib.dts_gather_next(sim.h) != 0
    assert sim.lib.dts_last_error(sim.h).decode() == (f"the fused gather holds {batch} bytes per rank (dts_gather_alloc) "
                                                      f"but the observation batch is {4 * batch} bytes in the current "
                                                      f"output format")
    assert_unchanged(torch, env, snap, "a refused arm")
    env.step(acts[1])                          # not armed: a float32 step writes no buffer
    assert bool((g.gathered.view(torch.uint8) == SENTINEL).all())
    # armed while u8, then switched: dts_step and dts_render refuse
    env.set_output_format(obs_dtype="uint8")
    g.arm()
    env.set_output_format(obs_dtype="float32")
    env.obs.fill_(0.5)
    snap = snapshot(torch, env)
    with pytest.raises(L.DtsError, match=f"dts_step: the fused gather holds {batch} bytes per rank .* batch is {4 * batch} bytes"):
        env.step(acts[2])
    assert_unchanged(torch, env, snap, "refused dts_step")
    with pytest.raises(L.DtsError, match=f"dts_render: the fused gather holds {batch} bytes per rank"):
        sim.render(env.obs.data_ptr(), env._stream())
    assert_unchanged(torch, env, snap, "refused dts_render")
    assert bool((g.gathered.view(torch.uint8) == SENTINEL).all())
    # still armed: the first step that fits writes the slot
    env.set_output_format(obs_dtype="uint8")
    obs, *_ = env.step(acts[2])
    out = g.finish()
    assert torch.equal(out[0], obs)
    env.check()
    env.close()


def test_refuses_resize_while_armed(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    env = make_env(32, "small_loop")
    env.reset()
    g = Gather(env, batch_bytes(env))
    g.open()
    g.buf.fill_(SENTINEL)
    acts = forward_actions(torch, env, 2)
    g.arm()
    env.set_resize(84, 84)
    snap = snapshot(torch, env)
    with pytest.raises(L.DtsError, match="dts_step: the fused gather writes the rasteriser's own output: not combined with dts_set_resize"):
        env.step(acts[0])
    assert_unchanged(torch, env, snap, "refused dts_step")
    with pytest.raises(L.DtsError, match="dts_render: the fused gather .* not combined with dts_set_resize"):
        env.sim.render(env.obs.data_ptr(), env._stream())
    assert_unchanged(torch, env, snap, "refused dts_render")
    g.assert_sentinel("a refused call")
    env.set_resize(None, None)
    env.step(acts[1])                          # still armed
    torch.cuda.synchronize()
    assert torch.equal(g.buf, obs_bytes(env))
    env.check()
    env.close()


def test_refuses_bad_allocations_and_unmapped_peers(torch_cuda):
    torch = torch_cuda
    env = make_env(32, "small_loop")
    env.reset()
    sim = env.sim
    batch = batch_bytes(env)
    snap = snapshot(torch, env)

    def refused(call, message):
        assert call() != 0
        assert sim.lib.dts_last_error(sim.h).decode() == message

    refused(lambda: sim.lib.dts_gather_next(sim.h), "dts_gather_alloc first")
    for rank, world in ((1, 1), (-1, 2), (2, 2), (0, 0), (0, 9)):
        handle, buf = (C.c_uint8 * 64)(), C.c_void_p()
        refused(lambda: sim.lib.dts_gather_alloc(sim.h, batch, rank, world, handle, C.byref(buf)),
                f"bad rank {rank} / world {world} (max 8)")
        assert buf.value is None
    g = Gather(env, batch, rank=0, world=2)    # rank 1's buffer is never opened
    g.buf.fill_(SENTINEL)
    handle, buf = (C.c_uint8 * 64)(), C.c_void_p()
    refused(lambda: sim.lib.dts_gather_alloc(sim.h, batch, 0, 1, handle, C.byref(buf)), "gather buffer already allocated")
    assert buf.value is None
    refused(lambda: sim.lib.dts_gather_next(sim.h), "dts_gather_open first (rank 1 not mapped)")
    assert_unchanged(torch, env, snap, "a refused dts_gather_*")
    env.step(forward_actions(torch, env, 1)[0])   # not armed
    torch.cuda.synchronize()
    g.assert_sentinel("a step after the refused dts_gather_next")
    env.check()
    env.close()


# ---- several ranks: one process per rank, all on one GPU, handles exchanged over gloo --------------------------------
_WORKER = r'''
import ctypes as C
import os
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import torch
import torch.distributed as dist

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
SENTINEL = 0xA5
try:   # every rank needs a CUDA context of its own on the one device
    torch.zeros(1, device="cuda:0")
    why = ""
except RuntimeError as e:
    why = str(e)
whys = [None] * world
dist.all_gather_object(whys, why)
if any(whys):
    busy = all("busy or unavailable" in w for w in whys if w)
    if rank == 0:
        print(("SKIP: " if busy else "FAIL: ") + "; ".join(w.splitlines()[0] for w in whys if w), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if busy else 1)

from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
from gym_duckietown_b200.lib import _CudaArray

N = 32
# name, camera, layout, dtype, bytes_per_rank - batch (8: every slot of rank >= 1 is misaligned for 16-byte stores)
CASES = [("lean_u8", 160, 120, "hwc", "uint8", 0), ("odd_u8", 101, 75, "hwc", "uint8", 0),
         ("chw_f32", 160, 120, "chw", "float32", 0), ("misaligned_u8", 160, 120, "hwc", "uint8", 8)]
for name, W, H, layout, dtype, extra in CASES:
    env = BatchedDuckietownEnv(N, "loop_obstacles", device=0, camera_width=W, camera_height=H, domain_rand=False,
                               seed=77, auto_reset=True, device_reset=True, env_id_offset=rank * N)
    env.set_output_format(obs_layout=layout, obs_dtype=dtype)
    env.reset()
    batch = env.obs.numel() * env.obs.element_size()
    bpr = batch + extra
    sim = env.sim
    handle, ptr = (C.c_uint8 * 64)(), C.c_void_p()
    sim._check(sim.lib.dts_gather_alloc(sim.h, bpr, rank, world, handle, C.byref(ptr)), "dts_gather_alloc")
    mine = torch.tensor(list(handle), dtype=torch.uint8)
    handles = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(handles, mine)
    host = torch.stack(handles).numpy()
    sim._check(sim.lib.dts_gather_open(sim.h, host.ctypes.data_as(C.c_void_p)), "dts_gather_open")
    buf = torch.as_tensor(_CudaArray(ptr.value, world * bpr, np.uint8), device=env.device)
    buf.fill_(SENTINEL)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(5 + rank)
    acts = torch.rand((5, N, 2), device=env.device, generator=gen) * 2 - 1
    for t in range(3):
        env.step(acts[t])
    torch.cuda.synchronize()
    dist.barrier()                         # every buffer holds the sentinel before any rank's armed step
    sim._check(sim.lib.dts_gather_next(sim.h), "dts_gather_next")
    env.step(acts[3])
    torch.cuda.synchronize()
    dist.barrier()                         # every rank's stores into every buffer have landed
    obs = env.obs.contiguous().view(-1).view(torch.uint8).cpu()
    assert float(env.obs.float().std()) > (10 if dtype == "uint8" else 0.04), name
    all_obs = [torch.empty_like(obs) for _ in range(world)]
    dist.all_gather(all_obs, obs)
    got = buf.cpu()
    all_bufs = [torch.empty_like(got) for _ in range(world)]
    dist.all_gather(all_bufs, got)
    for r in range(world):
        assert torch.equal(got[r * bpr:r * bpr + batch], all_obs[r]), f"{name}: slot {r} of rank {rank}'s buffer is not rank {r}'s obs"
        assert bool((got[r * bpr + batch:(r + 1) * bpr] == SENTINEL).all()), f"{name}: rank {rank}'s buffer written past slot {r}"
        assert torch.equal(all_bufs[r], got), f"{name}: the buffers of ranks {r} and {rank} differ"
        assert r == 0 or not torch.equal(all_obs[r], all_obs[0]), f"{name}: ranks 0 and {r} hold the same shard"
    env.step(acts[4])                      # not armed
    torch.cuda.synchronize()
    dist.barrier()
    assert torch.equal(buf.cpu(), got), f"{name}: an unarmed step wrote rank {rank}'s buffer"
    env.check()
    del buf
    dist.barrier()                         # no rank frees its buffer while another still reads it
    env.close()
    if rank == 0:
        print(f"CASE_OK {name}", flush=True)
dist.destroy_process_group()
'''


@pytest.mark.parametrize("world,port", [(2, 29547), (3, 29548)])
def test_ranks_on_one_gpu_fill_every_slot_of_every_buffer(world, port, tmp_path, torch_cuda):
    """`world` processes on one GPU, each with its shard (env_id_offset = rank * N) and its gather buffer, handles
    exchanged over gloo: after the armed step, slot r of every rank's buffer is rank r's obs, every buffer is the same,
    the bytes past each slot's batch keep the sentinel, and the shards differ.  Packed u8 at 160x120 (16-byte rows) and
    101x75 (bytes), CHW float32 (per bin), and slots 8 bytes longer than the batch (rank >= 1 falls back to bytes)."""
    from gym_duckietown_b200 import lib as L
    L.load()                                   # built and current before the workers load it
    script = tmp_path / "gather_worker.py"
    script.write_text(_WORKER % {"root": ROOT})
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                         stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        out, err = p.communicate(timeout=300)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)       # the launcher and every worker
        out, err = p.communicate()
        pytest.fail(f"world {world} did not finish in 300 s:\n{out[-2000:]}{err[-3000:]}")
    skip = [l for l in out.splitlines() if l.startswith("SKIP: ")]
    if skip:
        pytest.skip(f"a second CUDA context on the device was refused (exclusive compute mode): {skip[0][6:]}")
    assert p.returncode == 0, out[-2000:] + err[-4000:]
    assert [l for l in out.splitlines() if l.startswith("CASE_OK")] == \
        ["CASE_OK lean_u8", "CASE_OK odd_u8", "CASE_OK chw_f32", "CASE_OK misaligned_u8"], out[-2000:] + err[-2000:]
