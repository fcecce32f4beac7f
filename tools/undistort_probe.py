"""What UndistortWrapper costs on the device.

launch_env()'s camera (udem1, 640x480, fisheye distortion on, domain_rand off) for N envs with device auto-reset,
stepped on the device with random actions, in four configurations:
  fisheye     the env's own observations (fused fisheye gather)
  undistort   wrappers.UndistortWrapper(env): the rectification gathered by the same kernels through its own table
  pinhole     env.undistort = True: no gather
  lw stack    learning_wrappers' DtRewardWrapper(ActionWrapper(ImgWrapper(NormalizeWrapper(ResizeWrapper(
              UndistortWrapper(env)))))) -> 160x120 float32 CHW
Reports device ms per step of each (host clock around `steps` steps that end in a synchronise, after `warmup` steps),
the configurations interleaved over `rounds` rounds so that the spread between rounds is measured in the same run,
and the share of output pixels each gather leaves without a source.  The card's name and power limit are printed with
the numbers.

    python tools/undistort_probe.py [--envs 4096] [--steps 50] [--warmup 10] [--rounds 3] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gym_duckietown_b200 import learning_wrappers as LW, wrappers as Wr  # noqa: E402
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402
from gym_duckietown_b200.distortion import Distortion, rectify_maps  # noqa: E402

CONFIGS = ["fisheye", "undistort", "pinhole", "lw_stack"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def launch_env(n, seed=1):
    return BatchedDuckietownEnv(n, "udem1", camera_width=640, camera_height=480, distortion=True, domain_rand=False,
                                seed=seed, auto_reset=True, device_reset=True)


def select(kind, env, uw):
    """Put `env`, wrapped by UndistortWrapper `uw`, into one of the first three configurations."""
    if kind == "fisheye":
        env.undistort = False
    elif kind == "undistort":
        env.set_rectification(uw.mapx, uw.mapy)
        env.undistort = True
    else:
        env.set_rectification(None, None)
        env.undistort = True


def device_ms(w, acts, steps, warmup):
    for t in range(warmup):
        w.step(acts[t % len(acts)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        w.step(acts[t % len(acts)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def no_source_share(mx, my, W=640, H=480):
    ok = np.isfinite(mx) & np.isfinite(my)
    ix, iy = np.where(ok, np.rint(mx), -1), np.where(ok, np.rint(my), -1)
    return float(1.0 - ((ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    d = Distortion(640, 480)
    res = {"card": card(), "envs": a.envs, "steps": a.steps, "camera": "udem1 640x480 distortion",
           "no_source_share": {"fisheye": no_source_share(d.rmapx, d.rmapy),
                               "undistort": no_source_share(*rectify_maps(640, 480))}}
    print("card:", res["card"], flush=True)
    print("output pixels without a source:", res["no_source_share"], flush=True)
    # one env switched between the three full-size configurations, one under the LW stack (each holds ~3.8 GB of frames
    # and its own pair pool at 4096 envs)
    env, lw_env = launch_env(a.envs), launch_env(a.envs)
    uw = Wr.UndistortWrapper(env)
    lw = LW.DtRewardWrapper(LW.ActionWrapper(LW.ImgWrapper(LW.NormalizeWrapper(LW.ResizeWrapper(
        Wr.UndistortWrapper(lw_env))))))
    uw.reset()
    lw.reset()
    acts = torch.rand((16, a.envs, 2), device="cuda") * 2 - 1
    runs = {k: [] for k in CONFIGS}
    for r in range(a.rounds):
        for kind in CONFIGS:
            if kind != "lw_stack":
                select(kind, env, uw)
            runs[kind].append(device_ms(lw if kind == "lw_stack" else uw, acts, a.steps, a.warmup))
        print("round %d: " % r + ", ".join("%s %.3f" % (k, runs[k][-1]) for k in CONFIGS) + " ms/step", flush=True)
    env.check()
    lw_env.check()
    res["ms_per_step"] = runs
    res["median_ms_per_step"] = {k: float(np.median(v)) for k, v in runs.items()}
    print("median ms/step:", {k: round(v, 3) for k, v in res["median_ms_per_step"].items()}, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
