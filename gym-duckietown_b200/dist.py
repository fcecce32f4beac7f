"""Multi-GPU: envs shard by contiguous index blocks (rank r owns global envs [r*N, (r+1)*N), seeds by
global index), the step path has no collective; one NCCL all-gather moves the end-of-rollout
observation batch (SURVEY 8e).  The all-gather runs inside libdtsim.so (dts_allgather_obs) on a
communicator created from a unique id that is broadcast with torch.distributed."""
from __future__ import annotations

import ctypes as C
import glob
import os

import torch
import torch.distributed as dist


def bind_to_gpu_numa(device_index: int) -> dict:
    """Pin this process to the CPUs of the NUMA node the GPU hangs off (PCI sysfs), BEFORE pinned host buffers are
    allocated: first-touch then places them on that node and the D2H stream does not cross the socket link.  One
    process per GPU (torchrun) otherwise inherits an all-CPU mask.  Returns what was done (for the bench record)."""
    import subprocess
    bus = subprocess.run(["nvidia-smi", "--query-gpu=pci.bus_id", "--format=csv,noheader", "-i", str(device_index)],
                         capture_output=True, text=True, timeout=10).stdout.strip().lower()
    if not bus:
        return {"bound": False, "why": "nvidia-smi gave no bus id"}
    if len(bus.split(":")[0]) == 8:   # 00000000:1B:00.0 -> 0000:1b:00.0
        bus = bus[4:]
    node_path = f"/sys/bus/pci/devices/{bus}/numa_node"
    if not os.path.exists(node_path):
        return {"bound": False, "why": f"{node_path} missing"}
    node = int(open(node_path).read().strip())
    if node < 0:
        return {"bound": False, "why": "numa_node = -1 (single node)"}
    txt = open(f"/sys/devices/system/node/node{node}/cpulist").read().strip()
    cpus = set()
    for part in txt.split(","):
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    allowed = cpus & set(os.sched_getaffinity(0))
    if not allowed:
        return {"bound": False, "why": f"no allowed CPU on node {node}"}
    os.sched_setaffinity(0, allowed)
    return {"bound": True, "node": node, "cpus": len(allowed)}


def find_libnccl() -> str:
    """The NCCL that torch itself loaded (nvidia-nccl wheel), else the system one."""
    cands = []
    try:
        import nvidia.nccl  # type: ignore
        for p in nvidia.nccl.__path__:
            cands += glob.glob(os.path.join(p, "lib", "libnccl.so*"))
    except Exception:
        pass
    cands += glob.glob(os.path.join(os.path.dirname(torch.__file__), "lib", "libnccl.so*"))
    cands += glob.glob("/usr/lib/x86_64-linux-gnu/libnccl.so*")
    if not cands:
        raise RuntimeError("libnccl.so not found")
    return cands[0]


class ObsAllGather:
    def __init__(self, env, rank: int, world: int):
        self.env, self.rank, self.world = env, rank, world
        sim = env.sim
        sim._check(sim.lib.dts_comm_load(sim.h, find_libnccl().encode()), "dts_comm_load")
        uid = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            buf = (C.c_uint8 * 128)()
            sim._check(sim.lib.dts_comm_unique_id(sim.h, buf), "dts_comm_unique_id")
            uid = torch.tensor(list(buf), dtype=torch.uint8)
        uid = uid.to(env.device)
        dist.broadcast(uid, src=0)
        host = uid.cpu().numpy()
        sim._check(sim.lib.dts_comm_init(sim.h, host.ctypes.data_as(C.c_void_p), rank, world), "dts_comm_init")

    def all_gather(self, out: torch.Tensor, src: torch.Tensor = None) -> torch.Tensor:
        """out: u8[world, N, H, W, 3] on this device; src defaults to the env's obs batch."""
        src = self.env.obs if src is None else src
        assert out.is_contiguous() and src.is_contiguous() and out.numel() == self.world * src.numel()
        sim = self.env.sim
        sim._check(sim.lib.dts_allgather_obs(sim.h, src.data_ptr(), out.data_ptr(), src.numel() * src.element_size(),
                                             torch.cuda.current_stream(self.env.device).cuda_stream),
                   "dts_allgather_obs")
        return out


class FusedObsGather:
    """The end-of-rollout observation exchange FUSED into the last step's rasteriser (dts_gather_*): every rank maps the
    other ranks' gather buffers as peer memory (cudaIpc over NVLink / NVSwitch) and its k_raster ships each finished
    block of 8 whole image rows of a packed u8 HWC frame into all of them while it renders; the other layouts and float32
    are stored per 8x4 pixel bin.  No separate collective pass: the transfer rides under the rasterisation.  The buffers
    are sized for `env.obs` as it is at construction (one gather per env): `arm()` refuses while `set_output_format` /
    `set_resize` have left it another dtype or shape.  Usage per rollout:

        g.arm()                      # before the rollout's LAST env.step(): that step also fills the gather buffers
        env.step(actions)
        batch = g.finish()           # stream sync + barrier: [world, *env.obs.shape] (this rank's copy) is complete
    """

    def __init__(self, env, rank: int, world: int):
        self.env, self.rank, self.world = env, rank, world
        sim = env.sim
        self.dtype, self.shape = env.obs.dtype, tuple(env.obs.shape)
        nbytes = env.obs.numel() * env.obs.element_size()
        handle = (C.c_uint8 * 64)()
        buf = C.c_void_p()
        sim._check(sim.lib.dts_gather_alloc(sim.h, nbytes, rank, world, handle, C.byref(buf)), "dts_gather_alloc")
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=env.device)
        allh = [torch.empty_like(mine) for _ in range(world)]
        if world > 1:
            dist.all_gather(allh, mine)
        else:
            allh = [mine]
        host = torch.stack(allh).cpu().numpy()
        sim._check(sim.lib.dts_gather_open(sim.h, host.ctypes.data_as(C.c_void_p)), "dts_gather_open")
        from .lib import _CudaArray
        import numpy as np
        flat = torch.as_tensor(_CudaArray(buf.value, world * nbytes, np.uint8), device=env.device)
        self.gathered = flat.view(env.obs.dtype).view((world,) + tuple(env.obs.shape))
        if world > 1:
            dist.barrier()   # every rank has opened every buffer before anyone writes

    def arm(self):
        obs = self.env.obs
        if obs.dtype != self.dtype or tuple(obs.shape) != self.shape:
            raise ValueError(f"FusedObsGather was built for observations {self.dtype} {list(self.shape)}, but env.obs is now "
                             f"{obs.dtype} {list(obs.shape)}: choose the output format before creating the gather")
        sim = self.env.sim
        sim._check(sim.lib.dts_gather_next(sim.h), "dts_gather_next")

    def finish(self) -> torch.Tensor:
        torch.cuda.current_stream(self.env.device).synchronize()   # my stores to every peer have landed
        if self.world > 1:
            dist.barrier()                                         # ... and everybody else's into mine
        return self.gathered
