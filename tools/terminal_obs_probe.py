"""What keeping the terminal frames under device auto-reset costs.

For each map (c2: small_loop, c3: loop_obstacles; 4096 envs at 160x120, domain_rand off, bench.py's uniform random
actions in [-1, 1]), five arms alternated in one process, `rounds` times:
  a       auto_reset=True: the first frame of the next episode only (what bench.py runs)
  b       auto_reset=True, terminal_obs=True: also the terminal frames (dts_step_terminal: a second render over the envs
          that ended)
  c       the reference-style loop that also gives them: auto_reset=False, step(), then reset(mask=done), whose reset
          re-renders the whole batch
  a_idle, b_idle   a and b with zero actions, where no episode ends: b_idle - a_idle is the fixed cost of the empty
                   second pass
Reports device ms/step of each arm (host clock around `steps` steps ending in a synchronise, after `warmup` steps),
medians over the rounds, and the mean fraction of envs that ended per step under the random actions.  Prints one JSON
line, with the card's name, power limit and SM clock read in the same run.

    python tools/terminal_obs_probe.py [--envs 4096] [--steps 100] [--warmup 10] [--rounds 3] [--out FILE.json]
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
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402

MAPS = {"c2": "small_loop", "c3": "loop_obstacles"}
ARMS = ["a", "b", "c", "a_idle", "b_idle"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def make(n, name, **kw):
    return BatchedDuckietownEnv(n, name, camera_width=160, camera_height=120, domain_rand=False, seed=1,
                                device_reset=True, **kw)


def run(arm, envs, acts, idle, steps, t0=0):
    """`steps` steps of one arm; returns nothing (the caller times it)."""
    if arm == "c":
        e = envs["c"]
        for t in range(steps):
            _, _, done, _ = e.step(acts[(t0 + t) % len(acts)])
            e.reset(mask=done)
        return
    e = envs[arm[0]]
    for t in range(steps):
        e.step(idle if arm.endswith("_idle") else acts[(t0 + t) % len(acts)])


def device_ms(arm, envs, acts, idle, steps, warmup):
    run(arm, envs, acts, idle, warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(arm, envs, acts, idle, steps, warmup)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def ended_fraction(envs, acts, steps):
    """Mean fraction of envs whose episode ended per step, on the auto-reset env under the random actions."""
    e = envs["a"]
    tot = torch.zeros((), dtype=torch.float64, device=e.device)
    for t in range(steps):
        _, _, done, _ = e.step(acts[t % len(acts)])
        tot += done.double().mean()
    return float(tot) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "envs": a.envs, "steps": a.steps, "camera": "160x120", "actions": "uniform [-1, 1]",
           "configs": {}}
    for cfg in a.configs.split(","):
        name = MAPS[cfg]
        envs = {"a": make(a.envs, name, auto_reset=True), "b": make(a.envs, name, auto_reset=True, terminal_obs=True),
                "c": make(a.envs, name)}
        for e in envs.values():
            e.reset()
        g = torch.Generator(device="cuda").manual_seed(0)
        acts = torch.rand((16, a.envs, 2), device="cuda", generator=g) * 2 - 1
        idle = torch.zeros((a.envs, 2), device="cuda")
        runs = {k: [] for k in ARMS}
        for r in range(a.rounds):
            for arm in ARMS:
                runs[arm].append(device_ms(arm, envs, acts, idle, a.steps, a.warmup))
            print(f"{cfg} round {r}: " + ", ".join(f"{k} {runs[k][-1]:.3f}" for k in ARMS) + " ms/step",
                  file=sys.stderr, flush=True)
        frac = ended_fraction(envs, acts, a.steps)
        for e in envs.values():
            e.check()
        med = {k: float(np.median(v)) for k, v in runs.items()}
        res["configs"][cfg] = {"map": name, "ms_per_step": runs, "median_ms_per_step": med, "ended_fraction": frac,
                               "b_minus_a_ms": med["b"] - med["a"], "b_idle_minus_a_idle_ms": med["b_idle"] - med["a_idle"],
                               "b_beats_c": med["b"] < med["c"]}
        for e in envs.values():
            e.close()
        del envs
        torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
