"""CPU suite: (1) libdtsim.so loads and exports every symbol include/dtsim.h declares (no compute call);
(2) the ctypes structs have the C layout; (3) multi-GPU host logic on 2 gloo ranks: env shards are
contiguous index blocks, seeds follow the GLOBAL env index, so episode draws do not depend on the
number of ranks, and the 128-byte communicator id reaches every rank."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from gym_duckietown_b200 import build as b
    from gym_duckietown_b200 import lib as L
    path = b.build()
    lib = ctypes.CDLL(path)
    hdr = open(os.path.join(ROOT, "include", "dtsim.h")).read()
    declared = set(re.findall(r"\b(dts_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(L.EXPORTS), declared ^ set(L.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    # cuobjdump: the library carries sm_90a code only — every embedded cubin is sm_90a, and no PTX to JIT elsewhere
    out = subprocess.run(["cuobjdump", "-lelf", path], capture_output=True, text=True).stdout
    elfs = [l for l in out.splitlines() if l.startswith("ELF file")]
    assert elfs and all(re.findall(r"\.(sm_\w+)\.cubin", l) == ["sm_90a"] for l in elfs), out
    ptx = subprocess.run(["cuobjdump", "-lptx", path], capture_output=True, text=True)
    assert not re.search(r"^PTX file\s+\d+:", ptx.stdout, re.M), ptx.stdout


def test_ctypes_struct_layout_matches_header():
    from gym_duckietown_b200 import lib as L
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "dtsim.h"
    int main(){ printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d\n", sizeof(dts_config), offsetof(dts_config, frame_rate),
      offsetof(dts_config, seed), sizeof(dts_map_blob), sizeof(dts_episode_params), sizeof(dts_state_view), sizeof(dts_object),
      sizeof(dts_dyn_object), offsetof(dts_dyn_object, safety_radius), offsetof(dts_map_blob, dyn), (int)DTS_DYN_FIELDS); return 0; }
    '''
    exe = os.path.join(ROOT, "tests", "_layout_probe")
    subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe], input=src, text=True, check=True)
    vals = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    os.remove(exe)
    assert vals == [ctypes.sizeof(L.Config), L.Config.frame_rate.offset, L.Config.seed.offset, ctypes.sizeof(L.MapBlob),
                    ctypes.sizeof(L.EpisodeParams), ctypes.sizeof(L.StateView), ctypes.sizeof(L.Object),
                    ctypes.sizeof(L.DynObjectC), L.DynObjectC.safety_radius.offset, L.MapBlob.dyn.offset, L.DYN_FIELDS]


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "gym-duckietown_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "liborc" not in text and "dt_oracle" not in text, f


_WORKER = r'''
import os, sys
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests")); sys.path.insert(0, os.path.join(%(root)r, "oracle"))
from gym_duckietown_b200 import maps
from gym_duckietown_b200.episode import EpisodeSampler
from test_reset_sampler import oracle_query
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
N_local, base_seed = 6, 1000
md = maps.load_map("loop_obstacles")
offset = rank * N_local                                  # contiguous block [rank*N, (rank+1)*N)
s = EpisodeSampler(N_local, domain_rand=True)
s.seed([base_seed + offset + k for k in range(N_local)]) # seeds by GLOBAL env index
out = s.sample(list(range(N_local)), [md] * N_local, oracle_query(md))
mine = torch.tensor(np.stack([out["pos_x"], out["pos_z"], out["angle"], out["wheel_dist"]], 1))
gathered = [torch.zeros_like(mine) for _ in range(world)]
dist.all_gather(gathered, mine)                          # the obs all-gather's host-side shape logic
uid = torch.arange(128, dtype=torch.uint8) if rank == 0 else torch.zeros(128, dtype=torch.uint8)
dist.broadcast(uid, src=0)                               # communicator id handshake (dist.py)
assert uid.tolist() == list(range(128))
if rank == 0:
    ref = EpisodeSampler(N_local * world, domain_rand=True)
    ref.seed([base_seed + k for k in range(N_local * world)])
    o = ref.sample(list(range(N_local * world)), [md] * (N_local * world), oracle_query(md))
    want = np.stack([o["pos_x"], o["pos_z"], o["angle"], o["wheel_dist"]], 1)
    got = torch.cat(gathered, 0).numpy()
    assert np.array_equal(got, want), "episode draws depend on the number of ranks"
    print("SHARDING_OK")
dist.destroy_process_group()
'''


def test_two_rank_sharding_is_rank_count_independent(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER % {"root": ROOT})
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29533", str(script)],
                       capture_output=True, text=True, timeout=280)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "SHARDING_OK" in r.stdout


def test_map_blob_flattening_of_dynamic_objects_and_traffic_light_cards():
    """Host logic only (no GPU): the dts_map_blob built for maps with `static: false` obstacles and traffic lights."""
    import ctypes as C
    from gym_duckietown_b200 import lib as L, maps
    for name in ("loop_pedestrians", "loop_dyn_duckiebots", "loop_trafficlights", "udem1"):
        md = maps.load_map(name)
        h = L.MapBlobHolder(md)
        b = h.blob
        assert b.n_dyn == len(md.dyn_objects) <= 32 and b.n_objects == len(md.objects)
        objs = C.cast(b.objects, C.POINTER(L.Object))
        dyn = C.cast(b.dyn, C.POINTER(L.DynObjectC))
        slots = [objs[i].dyn_slot for i in range(b.n_objects)]
        assert sorted(s for s in slots if s >= 0) == list(range(b.n_dyn))          # every slot used exactly once
        for s in range(b.n_dyn):
            o = dyn[s].object_index
            assert objs[o].dyn_slot == s and dyn[s].kind == md.dyn_objects[s].kind
            assert [dyn[s].pos[k] for k in range(3)] == [float(v) for v in md.objects[o].pos]
            if dyn[s].kind == maps.DYN_TRAFFICLIGHT:
                assert 0 <= objs[o].alt_tex_from < b.n_textures and 0 <= objs[o].alt_tex_to < b.n_textures
                assert objs[o].alt_tex_from != objs[o].alt_tex_to
                assert not md.objects[o].collidable
            else:
                assert objs[o].alt_tex_from == -1 and not md.objects[o].static
        # update order = object order (S:1570-1584)
        assert [dyn[s].object_index for s in range(b.n_dyn)] == sorted(dyn[s].object_index for s in range(b.n_dyn))
    md = maps.load_map("small_loop")
    assert L.MapBlobHolder(md, user_tile_start=(2, 1)).blob.start_tile[:] == [2, 1]
    assert L.MapBlobHolder(md).blob.start_tile[:] == [-1, -1] and L.MapBlobHolder(md).blob.has_start_pose == 0


def test_no_cpu_fallback_without_cuda():
    """The product has no CPU path: on a box without a CUDA device every entry into the simulator classes raises
    (loudly, with the reason) instead of computing something some other way."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for the CPU-only container")
    import gym_duckietown_b200 as gd
    from gym_duckietown_b200 import gymshim, lib as L
    with pytest.raises(L.DtsError, match="CUDA"):
        gd.BatchedDuckietownEnv(2, "small_loop", camera_width=32, camera_height=24)
    with pytest.raises(L.DtsError, match="CUDA"):
        gd.Simulator("small_loop")
    with pytest.raises(L.DtsError, match="CUDA"):
        gymshim.make("Duckietown-small_loop-v0")
    # the C ABI itself refuses too: no device -> dts_create fails with cudaSetDevice's message
    lib = L.load()
    h = ctypes.c_void_p()
    cfg = L.default_config(num_envs=2, cam_width=32, cam_height=24)
    assert lib.dts_create(ctypes.byref(cfg), ctypes.byref(h)) != 0
    assert b"cuda" in lib.dts_last_error(None).lower()


def test_module_level_helpers_match_reference(golden_dir):
    """get_dir_vec / get_right_vec / _actual_center / get_agent_corners (S:2056-2118), which user scripts import from
    the simulator module, against values computed by the reference's own functions."""
    import os
    import numpy as np
    from gym_duckietown_b200 import simulator as sim
    g = np.load(os.path.join(golden_dir, "helpers.npz"))
    for k, (p, a) in enumerate(zip(g["poses"], g["angles"])):
        assert np.array_equal(sim.get_dir_vec(a), g["dir_vec"][k]) and np.array_equal(sim.get_right_vec(a), g["right_vec"][k])
        assert np.array_equal(sim._actual_center(p, a), g["center"][k])
        assert np.array_equal(sim.get_agent_corners(p, a), g["corners"][k])
