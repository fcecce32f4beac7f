"""What the reference training scripts' wrapper stack costs on the device.

learning/utils/env.py's launch_env camera (640x480, fisheye distortion on, domain_rand off) for N envs, stepped on the
device with random actions:
  plain      full-size u8 HWC frames, no wrapper
  lw stack   learning_wrappers' DtRewardWrapper(ActionWrapper(ImgWrapper(NormalizeWrapper(ResizeWrapper(env)))))
             -> 160x120 float32 CHW (Pillow bilinear resize pass after the render)
and reports ms per step of each, the resize pass's time (profile level 2's "post" interval, and the pass alone on
the frames, timed with CUDA events), the pass's source bytes (N x W x H x 3 per step) over that time against the
H100 SXM data sheet's 3.35 TB/s, and HostPipeline's end-to-end rate with full-size frames and with the stack.
The card's name and power limit are printed with the numbers.

    python tools/lw_stack_probe.py [--envs 4096] [--steps 100] [--warmup 10] [--e2e-envs 1024] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import deque

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gym_duckietown_b200 import learning_wrappers as LW  # noqa: E402
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv, HostPipeline  # noqa: E402

DATASHEET_BW = 3.35e12   # H100 SXM HBM3, bytes/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def launch_env(n, seed=1):
    return BatchedDuckietownEnv(n, "udem1", camera_width=640, camera_height=480, distortion=True, domain_rand=False,
                                seed=seed, auto_reset=True, device_reset=True)


def stack(env):
    return LW.DtRewardWrapper(LW.ActionWrapper(LW.ImgWrapper(LW.NormalizeWrapper(LW.ResizeWrapper(env)))))


def device_ms(w, acts, steps, warmup):
    for t in range(warmup):
        w.step(acts[t % len(acts)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        w.step(acts[t % len(acts)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def post_ms(b, acts, steps):
    b.sim.profile(2)
    b.sim.profile_read()
    for t in range(steps):
        b.step(acts[t % len(acts)])
    ms, frames = b.sim.profile_read()
    b.sim.profile(0)
    return ms["post"] / max(frames, 1), {k: v / max(frames, 1) for k, v in ms.items()}


def pass_ms(b, frames, reps):
    for _ in range(3):
        b.sim_resize_only(frames)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        b.sim_resize_only(frames)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def e2e_rate(b, steps, warmup, depth=2):
    n = b.num_envs
    h_act = (torch.rand((8, n, 2)) * 2 - 1).pin_memory()
    pipe = HostPipeline(b, depth=depth)
    for t in range(warmup):
        pipe.result(pipe.submit(h_act[t % 8]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pend = deque()
    for t in range(steps):
        pend.append(pipe.submit(h_act[t % 8]))
        if len(pend) >= depth:
            pipe.result(pend.popleft())
    while pend:
        pipe.result(pend.popleft())
    dt = (time.perf_counter() - t0) / steps
    return n / dt, dt * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--e2e-envs", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "envs": a.envs, "steps": a.steps, "camera": "640x480 distortion", "lw_shape": [120, 160, 3]}
    print("card:", res["card"], flush=True)
    b = launch_env(a.envs)
    b.reset()
    acts = torch.rand((16, a.envs, 2), device=b.device) * 2 - 1
    res["plain_ms_per_step"] = device_ms(b, acts, a.steps, a.warmup)
    print("plain (640x480 u8 HWC)  %.3f ms/step" % res["plain_ms_per_step"], flush=True)
    w = stack(b)
    res["lw_ms_per_step"] = device_ms(w, acts, a.steps, a.warmup)
    print("lw stack (160x120 f32 CHW)  %.3f ms/step" % res["lw_ms_per_step"], flush=True)
    res["lw_post_ms"], res["lw_profile_ms"] = post_ms(b, acts, a.steps)
    frames = torch.randint(0, 256, (a.envs, 480, 640, 3), dtype=torch.uint8, device=b.device)
    res["pass_ms"] = pass_ms(b, frames, a.steps)
    src_bytes = a.envs * 640 * 480 * 3
    out_bytes = a.envs * 160 * 120 * 3 * 4
    for key in ("lw_post_ms", "pass_ms"):
        ms = res[key]
        res[key + "_src_TBps"] = src_bytes / (ms * 1e-3) / 1e12
        res[key + "_share_of_datasheet"] = src_bytes / (ms * 1e-3) / DATASHEET_BW
    res["src_bytes_per_step"] = src_bytes
    res["out_bytes_per_step"] = out_bytes
    res["datasheet_floor_ms"] = (src_bytes + out_bytes) / DATASHEET_BW * 1e3
    print("resize pass: post interval %.3f ms/step, alone %.3f ms; source %.2f GB -> %.2f TB/s (%.0f %% of 3.35 TB/s); "
          "data-sheet floor (read + write) %.3f ms" % (res["lw_post_ms"], res["pass_ms"], src_bytes / 1e9,
          res["pass_ms_src_TBps"], 100 * res["pass_ms_share_of_datasheet"], res["datasheet_floor_ms"]), flush=True)
    print("profile level 2, ms per step:", {k: round(v, 3) for k, v in res["lw_profile_ms"].items()}, flush=True)
    b.close()
    del frames, b, w
    torch.cuda.empty_cache()
    # host-facing: HostPipeline copies every step's observations to pinned host memory
    full = launch_env(a.e2e_envs)
    full.reset()
    res["e2e_full_env_steps_per_s"], res["e2e_full_ms"] = e2e_rate(full, a.steps, a.warmup)
    lw = launch_env(a.e2e_envs)
    stack(lw)
    lw.reset()
    res["e2e_lw_env_steps_per_s"], res["e2e_lw_ms"] = e2e_rate(lw, a.steps, a.warmup)
    print("HostPipeline e2e at %d envs: full-size u8 %.0f env-steps/s (%.3f ms/step), lw stack %.0f env-steps/s "
          "(%.3f ms/step)" % (a.e2e_envs, res["e2e_full_env_steps_per_s"], res["e2e_full_ms"],
                              res["e2e_lw_env_steps_per_s"], res["e2e_lw_ms"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
