"""What the bird's-eye map costs (dts_set_bev_target: one k_bev launch per step, a thread per cell, one i16 and one u8
store per cell).

For each benchmark shape — c2: small_loop, c3: loop_obstacles (4096 envs, 160x120) — ONE env under device auto-reset and
bench.py's uniform random actions in [-1, 1], stepped in arms that rotate from round to round: the grids off, 64x64 and
128x128 (0.03 m cells, the default origin).  The same handle runs every arm, so they differ in nothing but the k_bev
launch.  Three measurements per arm:
  - ms per step of step() with rendering (host clock around `steps` steps ending in a synchronise, after `warmup`);
  - env-steps/s of step(render=False), the mode the grids open: no rasteriser at all;
  - k_bev alone: CUDA events around `steps` render_bev() calls (off: not run), ms per call and the bytes it stores over
    that time.
Reports the median and spread over the rounds and prints one JSON line with the card's name, power limit and SM clocks
read before and after in the same run.

    python tools/bev_probe.py [--configs c2,c3] [--steps 100] [--warmup 10] [--rounds 5] [--out FILE.json]

--visibility measures the camera visibility of the grid instead (dts_set_bev_visibility_target: one k_bev_view launch
per step, after the render).  For each shape, with the pinhole camera and with --distortion's fisheye, one env with a
64x64 grid and the label image on is stepped in two alternating arms: the grid alone and the grid plus visibility.
Per arm: ms per step of step() with rendering, and render_obs() alone timed with CUDA events over `steps` calls; the
difference of the second between the arms is k_bev_view's time.

    python tools/bev_probe.py --visibility [--configs c2,c3] [--steps 100] [--warmup 10] [--rounds 5] [--out FILE.json]
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
from gym_duckietown_b200 import lib as L  # noqa: E402
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402

SHAPES = {
    "c2": dict(map="small_loop", envs=4096, width=160, height=120),
    "c3": dict(map="loop_obstacles", envs=4096, width=160, height=120),
}
GRIDS = {"off": None, "bev64": 64, "bev128": 128}
CELL = 0.03


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def set_arm(env, arm):
    n = GRIDS[arm]
    if n is None:
        env.sim.set_bev_target(None, None, None)
    else:   # the first num_envs * n * n elements of the 128 x 128 tensors, laid out [num_envs][n][n]
        env.sim.set_bev_target(L.BevConfig(n, n, CELL, n / 2, 3 * n / 4), env.bev_labels.data_ptr(),
                               env.bev_markings.data_ptr())


def run(env, acts, steps, render, t0=0):
    for t in range(steps):
        env.step(acts[(t0 + t) % len(acts)], render=render)


def host_ms(env, arm, acts, steps, warmup, render):
    set_arm(env, arm)
    run(env, acts, warmup, render)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(env, acts, steps, render, warmup)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def kernel_ms(env, arm, steps):
    if GRIDS[arm] is None:
        return 0.0
    set_arm(env, arm)
    for _ in range(5):
        env.sim.render_bev(env._stream())
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        env.sim.render_bev(env._stream())
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def render_ms(env, steps):
    for _ in range(5):
        env.render_obs()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        env.render_obs()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def visibility(a):
    res = {"card": card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "actions": "uniform [-1, 1]",
           "grid": [64, 64], "cell_m": CELL, "configs": {}}
    arms = ["grid", "grid+vis"]
    for cfg in a.configs.split(","):
        for fish in (False, True):
            c = dict(SHAPES[cfg])
            env = BatchedDuckietownEnv(c["envs"], c["map"], camera_width=c["width"], camera_height=c["height"],
                                       domain_rand=False, seed=1, device_reset=True, auto_reset=True,
                                       bev_shape=(64, 64), bev_cell=CELL, bev_visibility=True, distortion=fish)
            env.reset()
            fwd = (env.camera_model.mapx, env.camera_model.mapy) if fish else ()

            def set_vis(on):
                if on:
                    env.sim.set_bev_visibility_target(env.bev_visibility.data_ptr(), env.bev_pixels.data_ptr(), *fwd)
                else:
                    env.sim.set_bev_visibility_target(None, None)

            g = torch.Generator(device="cuda").manual_seed(0)
            acts = torch.rand((16, c["envs"], 2), device="cuda", generator=g) * 2 - 1
            step = {k: [] for k in arms}
            rend = {k: [] for k in arms}
            for r in range(a.rounds):
                for arm in arms[r % 2:] + arms[:r % 2]:
                    set_vis(arm == "grid+vis")
                    run(env, acts, a.warmup, True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run(env, acts, a.steps, True, a.warmup)
                    torch.cuda.synchronize()
                    step[arm].append((time.perf_counter() - t0) / a.steps * 1e3)
                    rend[arm].append(render_ms(env, a.steps))
                print(f"{cfg} {'fisheye' if fish else 'pinhole'} round {r}: " +
                      ", ".join(f"{k} {step[k][-1]:.3f} / {rend[k][-1]:.4f}" for k in arms) +
                      " ms (step / render_obs)", file=sys.stderr, flush=True)
            env.check()
            med = lambda d: {k: float(np.median(v)) for k, v in d.items()}
            spread = lambda d: {k: [float(min(v)), float(max(v))] for k, v in d.items()}
            diffs = [v - g_ for v, g_ in zip(rend["grid+vis"], rend["grid"])]
            res["configs"][f"{cfg}_{'fisheye' if fish else 'pinhole'}"] = {
                **c, "ms_per_step": med(step), "spread_ms_per_step": spread(step), "render_obs_ms": med(rend),
                "spread_render_obs_ms": spread(rend), "k_bev_view_ms": float(np.median(diffs)),
                "spread_k_bev_view_ms": [float(min(diffs)), float(max(diffs))]}
            env.close()
            del env
            torch.cuda.empty_cache()
    res["card_after"] = card()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--visibility", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    if a.visibility:
        emit(visibility(a), a.out)
        return
    arms = list(GRIDS)
    res = {"card": card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "actions": "uniform [-1, 1]",
           "cell_m": CELL, "configs": {}}
    for cfg in a.configs.split(","):
        c = dict(SHAPES[cfg])
        env = BatchedDuckietownEnv(c["envs"], c["map"], camera_width=c["width"], camera_height=c["height"],
                                   domain_rand=False, seed=1, device_reset=True, auto_reset=True, bev=True,
                                   bev_shape=(128, 128), bev_cell=CELL)
        env.reset()
        g = torch.Generator(device="cuda").manual_seed(0)
        acts = torch.rand((16, c["envs"], 2), device="cuda", generator=g) * 2 - 1
        runs = {k: [] for k in arms}
        blind = {k: [] for k in arms}
        kern = {k: [] for k in arms}
        for r in range(a.rounds):
            for arm in arms[r % 3:] + arms[:r % 3]:     # no arm always runs first
                runs[arm].append(host_ms(env, arm, acts, a.steps, a.warmup, True))
                blind[arm].append(host_ms(env, arm, acts, a.steps, a.warmup, False))
                kern[arm].append(kernel_ms(env, arm, a.steps))
            print(f"{cfg} round {r}: " + ", ".join(f"{k} {runs[k][-1]:.3f} / {blind[k][-1]:.3f} / {kern[k][-1]:.4f}"
                                                   for k in arms) + " ms (step / step without render / k_bev)",
                  file=sys.stderr, flush=True)
        env.check()
        med = lambda d: {k: float(np.median(v)) for k, v in d.items()}
        spread = lambda d: {k: [float(min(v)), float(max(v))] for k, v in d.items()}
        m_run, m_blind, m_kern = med(runs), med(blind), med(kern)
        out = {**c, "ms_per_step": m_run, "spread_ms_per_step": spread(runs),
               "ms_per_step_no_render": m_blind, "spread_ms_per_step_no_render": spread(blind),
               "env_steps_per_s_no_render": {k: c["envs"] / (v * 1e-3) for k, v in m_blind.items()},
               "k_bev_ms": m_kern, "spread_k_bev_ms": spread(kern)}
        for arm in arms[1:]:
            n = GRIDS[arm]
            bytes_ = c["envs"] * n * n * 3
            out[f"{arm}_minus_off_ms"] = m_run[arm] - m_run["off"]
            out[f"{arm}_no_render_minus_off_ms"] = m_blind[arm] - m_blind["off"]
            out[f"{arm}_bytes_per_step"] = bytes_
            out[f"{arm}_k_bev_store_GBps"] = bytes_ / (m_kern[arm] * 1e-3) / 1e9
        res["configs"][cfg] = out
        env.close()
        del env
        torch.cuda.empty_cache()
    res["card_after"] = card()
    emit(res, a.out)


def emit(res, out):
    line = json.dumps(res)
    print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
