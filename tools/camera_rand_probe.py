"""What a pool of fisheye LUTs costs (camera_rand: dts_set_fisheye_luts, the rasterisers' kRemapPool instances) against
the one-LUT path (dts_set_fisheye_lut).

Shapes: c4 (udem1, 640x480, fisheye, domain randomisation, `--c4-envs`, default 2048) and f160 (loop_obstacles, 160x120,
fisheye, domain randomisation, 4096 envs).  ONE env per shape under device auto-reset and bench.py's uniform random
actions in [-1, 1]; the arms install, on the same handle, the real LUT alone ("single") or a pool of K distinct tables
("K16", "K64", env e on table e mod K), and are stepped in an order that rotates from round to round.  A pool of one
table is the single arm by construction (dts_set_fisheye_luts launches the one-table kernels for it).  The pool's tables
are the real LUT shifted by a different whole-pixel offset each (up to +-6 px): distinct tables of the real one's shape,
so that they take K times its memory (1.2 MB of source indices each at 640x480), without building K calibrations' maps
on the host.  Reports ms per step of each arm (host clock around `steps` steps ending in a synchronise, after `warmup`
steps of that arm), the median and the spread over the rounds, and from a separate pass under dts_profile_enable(2) the
ms per frame of each render kernel bracket.  Prints one JSON line with the card's name, power limit and SM clocks read
before and after in the same run.

    python tools/camera_rand_probe.py [--configs c4,f160] [--steps 100] [--warmup 10] [--rounds 4] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402
from depth_probe import card, run  # noqa: E402

SHAPES = {
    "c4": dict(map="udem1", envs=2048, width=640, height=480),
    "f160": dict(map="loop_obstacles", envs=4096, width=160, height=120),
}
ARMS = ["single", "K16", "K64"]


def pool(real, K, seed=0):
    rng = np.random.default_rng(seed)
    offs = [(0, 0)] + [tuple(rng.integers(-6, 7, 2)) for _ in range(K - 1)]
    return (np.stack([real.rmapx + dx for dx, _ in offs]).astype(np.float32),
            np.stack([real.rmapy + dy for _, dy in offs]).astype(np.float32))


def set_arm(env, arm, pools):
    if arm == "single":
        env.sim.set_fisheye_lut(env.camera_model.rmapx, env.camera_model.rmapy)
    else:
        rx, ry = pools[arm]
        env.sim.set_fisheye_luts(rx, ry, np.arange(env.num_envs) % len(rx))


def step_ms(env, acts, steps, warmup):
    run(env, acts, warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(env, acts, steps, warmup)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def kernel_ms(env, acts, steps):
    """ms per frame of each render kernel bracket, events at every boundary."""
    run(env, acts, 5)
    env.sim.profile(2)
    env.sim.profile_read()
    run(env, acts, steps)
    ms, frames = env.sim.profile_read()
    env.sim.profile(0)
    return {k: v / max(frames, 1) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c4,f160")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--c4-envs", type=int, default=SHAPES["c4"]["envs"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "actions": "uniform [-1, 1]", "configs": {}}
    for cfg in a.configs.split(","):
        c = dict(SHAPES[cfg])
        if cfg == "c4":
            c["envs"] = a.c4_envs
        env = BatchedDuckietownEnv(c["envs"], c["map"], camera_width=c["width"], camera_height=c["height"],
                                   domain_rand=True, distortion=True, seed=1, device_reset=True, auto_reset=True)
        pools = {arm: pool(env.camera_model, int(arm[1:])) for arm in ARMS if arm != "single"}
        env.reset()
        g = torch.Generator(device="cuda").manual_seed(0)
        acts = torch.rand((16, c["envs"], 2), device="cuda", generator=g) * 2 - 1
        runs = {k: [] for k in ARMS}
        for r in range(a.rounds):
            for arm in ARMS[r % 3:] + ARMS[:r % 3]:     # no arm always runs first
                set_arm(env, arm, pools)
                runs[arm].append(step_ms(env, acts, a.steps, a.warmup))
            print(f"{cfg} round {r}: " + ", ".join(f"{k} {runs[k][-1]:.3f}" for k in ARMS) + " ms/step", file=sys.stderr, flush=True)
        kern = {}
        for arm in ARMS:
            set_arm(env, arm, pools)
            kern[arm] = kernel_ms(env, acts, min(a.steps, 50))
        env.check()
        med = {k: float(np.median(v)) for k, v in runs.items()}
        res["configs"][cfg] = {
            **c, "ms_per_step": runs, "median_ms_per_step": med,
            "spread_ms_per_step": {k: [float(min(v)), float(max(v))] for k, v in runs.items()},
            "kernel_ms_per_frame": kern, "src_xy_bytes_per_table": c["width"] * c["height"] * 4}
        for arm in ARMS[1:]:
            res["configs"][cfg].update({f"{arm}_over_single": med[arm] / med["single"],
                                        f"{arm}_minus_single_ms": med[arm] - med["single"]})
        env.close()
        del env
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
