"""What the lane path costs (dts_set_lane_path_target: one k_lane_path launch per step).

For each map — small_loop and udem1 at 4096 envs of 160x120 — and each K of 16 and 64 points (0.1 m apart), ONE env
under device auto-reset and bench.py's uniform random actions in [-1, 1], stepped in two arms that alternate from round
to round: the lane path target off and on.  The same handle runs both, so they differ in nothing but the k_lane_path
launch.  Measured:
  - env-steps/s of step() with a render and of step(render=False), host clock around `steps` steps ending in a
    synchronise, after `warmup`;
  - k_lane_path alone: CUDA events around `steps` render_lane_path() calls, ms per call.
Reports the median and spread over the rounds and prints one JSON line with the card's name, power limit and SM clocks
read before and after in the same run.

    python tools/lane_path_probe.py [--maps small_loop,udem1] [--points 16,64] [--steps 100] [--warmup 10]
                                    [--rounds 5] [--out FILE.json]
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

ENVS, WIDTH, HEIGHT, SPACING = 4096, 160, 120, 0.1


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def set_arm(env, on):
    if on:
        env.sim.set_lane_path_target(env.lane_path.shape[1], SPACING, env.lane_path.data_ptr(),
                                     env.lane_path_count.data_ptr(), env.lane_path_px.data_ptr())
    else:
        env.sim.set_lane_path_target(0, 0.0, None, None, None)


def step_rate(env, acts, steps, warmup, render):
    for t in range(warmup):
        env.step(acts[t % len(acts)], render=render)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        env.step(acts[t % len(acts)], render=render)
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


def probe(name, K, steps, warmup, rounds):
    env = BatchedDuckietownEnv(ENVS, name, camera_width=WIDTH, camera_height=HEIGHT, domain_rand=False, seed=0,
                               device_reset=True, auto_reset=True, lane_path=True, lane_path_points=K,
                               lane_path_spacing=SPACING)
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = [torch.rand((ENVS, 2), device="cuda", generator=g) * 2 - 1 for _ in range(16)]
    stats = lambda x: {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x))}  # noqa: E731
    out = {}
    for render in (True, False):
        res = {"off": [], "on": []}
        for r in range(rounds):
            for arm in (("off", "on") if r % 2 == 0 else ("on", "off")):
                set_arm(env, arm == "on")
                res[arm].append(step_rate(env, acts, steps, warmup, render))
        key = "step" if render else "step_no_render"
        out[key] = {arm: {"env_steps_per_s": stats(v)} for arm, v in res.items()}
        out[key]["step_cost_ms"] = ENVS * (1 / out[key]["on"]["env_steps_per_s"]["median"] -
                                           1 / out[key]["off"]["env_steps_per_s"]["median"]) * 1e3
    set_arm(env, True)
    out["k_lane_path_ms"] = stats([call_ms(env.render_lane_path, steps, warmup) for _ in range(rounds)])
    torch.cuda.synchronize()
    out["mean_count"] = float(env.lane_path_count.float().mean().item())
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", default="small_loop,udem1")
    ap.add_argument("--points", default="16,64")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lane_path_probe needs a CUDA device")
    line = {"card_before": card(), "envs": ENVS, "camera": [WIDTH, HEIGHT], "spacing": SPACING}
    line["maps"] = {m: {f"K{k}": probe(m, int(k), args.steps, args.warmup, args.rounds)
                        for k in args.points.split(",")} for m in args.maps.split(",")}
    line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
