"""What the range scan costs (dts_set_scan_target: one k_scan launch per step, a thread per ray, one f32 and one i16
store per ray).

For each shape — c2: small_loop, c3: loop_obstacles (4096 envs, 160x120) — ONE env under device auto-reset and
bench.py's uniform random actions in [-1, 1], stepped in arms that rotate from round to round: the scan off, and 1, 64
and 360 rays over the full circle to 2 m.  The same handle runs every arm, so they differ in nothing but the k_scan
launch.  Two measurements per arm:
  - env-steps/s of step(render=False), the mode the scan opens: no rasteriser at all (host clock around `steps` steps
    ending in a synchronise, after `warmup`);
  - k_scan alone: CUDA events around `steps` render_scan() calls (off: not run), ms per call.
Reports the median and spread over the rounds and prints one JSON line with the card's name, power limit and SM clocks
read before and after in the same run.

--bench-ab PARENT also runs `bench.py --no-cpu-baseline` from the tree PARENT (built) and from this one, alternated
`--bench-rounds` times with `--bench-steps` / `--bench-warmup`, each with the scan off (bench.py never sets it), and
reports c2 (the headline) to c5 env-steps/s of both.  `--configs none` skips the scan arms.

    python tools/scan_probe.py [--configs c2,c3] [--steps 100] [--warmup 10] [--rounds 5] [--bench-ab DIR]
                               [--bench-rounds 2] [--bench-steps 100] [--bench-warmup 10] [--out FILE.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gym_duckietown_b200 import lib as L  # noqa: E402
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402

SHAPES = {
    "c2": dict(map="small_loop", envs=4096, width=160, height=120),
    "c3": dict(map="loop_obstacles", envs=4096, width=160, height=120),
}
ARMS = {"off": None, "rays1": 1, "rays64": 64, "rays360": 360}
RANGE = 2.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def set_arm(env, arm):
    r = ARMS[arm]
    if r is None:
        env.sim.set_scan_target(None, None, None)
    else:   # the first num_envs * r elements of the 360-ray tensors, laid out [num_envs][r]
        env.sim.set_scan_target(L.ScanConfig(r, 2 * math.pi, RANGE, 0.0, 0.0), env.scan_range.data_ptr(),
                                env.scan_hit.data_ptr())


def step_rate(env, acts, steps, warmup):
    for t in range(warmup):
        env.step(acts[t % len(acts)], render=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        env.step(acts[t % len(acts)], render=False)
    torch.cuda.synchronize()
    return env.num_envs * steps / (time.perf_counter() - t0)


def scan_ms(env, steps, warmup):
    for _ in range(warmup):
        env.render_scan()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        env.render_scan()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def probe_shape(name, steps, warmup, rounds):
    s = SHAPES[name]
    env = BatchedDuckietownEnv(s["envs"], s["map"], camera_width=s["width"], camera_height=s["height"],
                               domain_rand=False, seed=0, device_reset=True, auto_reset=True, scan=True,
                               scan_rays=max(r for r in ARMS.values() if r))
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = [torch.rand((s["envs"], 2), device="cuda", generator=g) * 2 - 1 for _ in range(16)]
    res = {a: {"env_steps_per_s": [], "k_scan_ms": []} for a in ARMS}
    arms = list(ARMS)
    for r in range(rounds):
        for arm in arms[r % len(arms):] + arms[:r % len(arms)]:
            set_arm(env, arm)
            res[arm]["env_steps_per_s"].append(step_rate(env, acts, steps, warmup))
            if ARMS[arm]:
                res[arm]["k_scan_ms"].append(scan_ms(env, steps, warmup))
    env.close()
    out = {}
    for arm, v in res.items():
        out[arm] = {k: {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x))}
                    for k, x in v.items() if x}
    base = out["off"]["env_steps_per_s"]["median"]
    for arm in arms[1:]:
        out[arm]["step_cost_ms"] = s["envs"] * (1 / out[arm]["env_steps_per_s"]["median"] - 1 / base) * 1e3
    return out


def bench_configs(tree, steps, warmup):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
           str(warmup), "--no-cpu-baseline"]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    line = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    out = {"c2": line["value"]}
    for k, v in line.get("configs", {}).items():
        out[k] = v.get("value", v.get("error"))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--bench-ab", metavar="PARENT", default=None)
    ap.add_argument("--bench-rounds", type=int, default=2)
    ap.add_argument("--bench-steps", type=int, default=100)
    ap.add_argument("--bench-warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("scan_probe needs a CUDA device")
    line = {"card_before": card()}
    line["shapes"] = {c: probe_shape(c, args.steps, args.warmup, args.rounds)
                      for c in args.configs.split(",") if c != "none"}
    if args.bench_ab:
        ab = {"parent": [], "this": []}
        for _ in range(args.bench_rounds):
            ab["parent"].append(bench_configs(os.path.abspath(args.bench_ab), args.bench_steps, args.bench_warmup))
            ab["this"].append(bench_configs(ROOT, args.bench_steps, args.bench_warmup))
        line["bench_ab"] = ab
    line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
