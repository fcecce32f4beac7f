"""What the object outputs cost (dts_set_object_target: one k_objects launch per step; dts_object_pixels: one
k_object_pixels launch per object_boxes() call).

For each map — small_loop, loop_obstacles, udem1 at 4096 envs of 160x120 — ONE env with labels=True and objects=True
under device auto-reset and bench.py's uniform random actions in [-1, 1], stepped in two arms that alternate from round
to round: the object target off and on.  The same handle runs both, so they differ in nothing but the k_objects launch.
Measured:
  - env-steps/s of step() with a render, host clock around `steps` steps ending in a synchronise, after `warmup`;
  - k_objects without a frame: CUDA events around `steps` render_objects() calls, ms per call;
  - k_objects after a render and k_object_pixels: their CUDA time per launch from torch.profiler over `steps` steps
    and object_boxes() calls, in a run of its own after the timed rounds;
  - object_boxes(): CUDA events around `steps` calls, ms per call, against the torch scatter chain it replaces (kept
    here as `torch_object_boxes`, the previous implementation; `steps` / 10 calls), after checking that both agree.
Reports the median and spread over the rounds and prints one JSON line with the card's name, power limit and SM clocks
read before and after in the same run.

    python tools/object_probe.py [--maps small_loop,loop_obstacles,udem1] [--steps 100] [--warmup 10] [--rounds 5]
                                 [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402

ENVS, WIDTH, HEIGHT = 4096, 160, 120


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def torch_object_boxes(env):
    """object_boxes() as the library computed it in torch before k_object_pixels"""
    n, h, w = env.labels.shape
    n_obj = max((len(md.objects) for md in env.maps), default=0)
    dev = env.device
    cells = torch.tensor([md.grid_w * md.grid_h for md in env.maps], dtype=torch.int64, device=dev)
    nobj = torch.tensor([len(md.objects) for md in env.maps], dtype=torch.int64, device=dev)
    mid = env.state["map_id"].to(torch.int64)
    o = env.labels.to(torch.int64) - 2 - cells[mid].view(n, 1, 1)
    hit = (o >= 0) & (o < nobj[mid].view(n, 1, 1))
    e = torch.arange(n, device=dev).view(n, 1, 1).expand(n, h, w)
    ys = torch.arange(h, device=dev).view(1, h, 1).expand(n, h, w)
    xs = torch.arange(w, device=dev).view(1, 1, w).expand(n, h, w)
    slot = (e * max(n_obj, 1) + o)[hit]
    pixels = torch.zeros(n * max(n_obj, 1), dtype=torch.int64, device=dev).scatter_add_(0, slot, torch.ones_like(slot))
    big = torch.iinfo(torch.int64).max
    lo_x = torch.full_like(pixels, big).scatter_reduce_(0, slot, xs[hit], "amin")
    lo_y = torch.full_like(pixels, big).scatter_reduce_(0, slot, ys[hit], "amin")
    hi_x = torch.full_like(pixels, -1).scatter_reduce_(0, slot, xs[hit], "amax")
    hi_y = torch.full_like(pixels, -1).scatter_reduce_(0, slot, ys[hit], "amax")
    boxes = torch.stack([lo_x, lo_y, hi_x, hi_y], dim=1)
    boxes[pixels == 0] = -1
    return pixels.view(n, -1)[:, :n_obj].to(torch.int32), boxes.view(n, -1, 4)[:, :n_obj].to(torch.int32)


def set_arm(env, on):
    if on:
        env.sim.set_object_target(env.object_state.shape[1], env.object_boxes3d.data_ptr(), env.object_state.data_ptr(),
                                  env.object_corners_px.data_ptr())
    else:
        env.sim.set_object_target(0, None, None, None)


def step_rate(env, acts, steps, warmup):
    for t in range(warmup):
        env.step(acts[t % len(acts)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        env.step(acts[t % len(acts)])
    torch.cuda.synchronize()
    return env.num_envs * steps / (time.perf_counter() - t0)


def call_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def kernel_us(env, acts, steps):
    """CUDA time per launch of k_objects (after a render) and k_object_pixels, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(steps):
            env.step(acts[t % len(acts)])
            env.object_boxes()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in ("k_objects", "k_object_pixels"):
            if f"::{k}(" in ev.key or f"{k}E" in ev.key:   # demangled or mangled
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                out[k] = {"us_per_launch": t / max(ev.count, 1), "launches": ev.count}
    return out


def probe_map(name, steps, warmup, rounds):
    env = BatchedDuckietownEnv(ENVS, name, camera_width=WIDTH, camera_height=HEIGHT, domain_rand=False, seed=0,
                               device_reset=True, auto_reset=True, labels=True, objects=True)
    env.reset()
    n_obj = env.object_state.shape[1]
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = [torch.rand((ENVS, 2), device="cuda", generator=g) * 2 - 1 for _ in range(16)]
    out = {"objects": n_obj}
    if not n_obj:   # nothing to launch: the target is never set
        out["env_steps_per_s"] = step_rate(env, acts, steps, warmup)
        env.close()
        return out
    res = {"off": [], "on": []}
    k_ms = []
    for r in range(rounds):
        for arm in (("off", "on") if r % 2 == 0 else ("on", "off")):
            set_arm(env, arm == "on")
            res[arm].append(step_rate(env, acts, steps, warmup))
        set_arm(env, True)
        k_ms.append(call_ms(env.render_objects, steps, warmup))
    p_new, b_new = env.object_boxes()
    p_old, b_old = torch_object_boxes(env)
    same = bool(torch.equal(p_new, p_old) and torch.equal(b_new, b_old))
    new_ms = [call_ms(env.object_boxes, steps, warmup) for _ in range(rounds)]
    old_ms = [call_ms(lambda: torch_object_boxes(env), max(steps // 10, 1), 2) for _ in range(rounds)]
    stats = lambda x: {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x))}  # noqa: E731
    out.update({arm: {"env_steps_per_s": stats(v)} for arm, v in res.items()})
    out["step_cost_ms"] = ENVS * (1 / out["on"]["env_steps_per_s"]["median"] -
                                  1 / out["off"]["env_steps_per_s"]["median"]) * 1e3
    out["k_objects_no_frame_ms"] = stats(k_ms)
    out["object_boxes_ms"] = {"kernel": stats(new_ms), "torch": stats(old_ms), "equal": same}
    out["profiler"] = kernel_us(env, acts, min(steps, 20))
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", default="small_loop,loop_obstacles,udem1")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("object_probe needs a CUDA device")
    line = {"card_before": card()}
    line["maps"] = {m: probe_map(m, args.steps, args.warmup, args.rounds) for m in args.maps.split(",")}
    line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
