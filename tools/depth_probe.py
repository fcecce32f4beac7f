"""What the depth image costs (dts_set_depth_target: the rasterisers' depth instances, one f32 store per pixel), and
with --labels what the label image costs (dts_set_label_target: their label instances, one i16 store per pixel and a
draw-item lookup per winner), alone and together with depth, and with --markings what the lane-marking image costs
(dts_set_marking_target: the rasterisers' marking instances, one u8 store per pixel and a texel-class load per winner),
alone and together with labels, and with --flow what the motion-flow image costs (dts_set_flow_target: k_flow after the
rasterisers, reading depth, labels and the remap, one float2 store per pixel) on top of depth and labels, and with
--flow --occlusion what the occlusion mask adds to flow (dts_set_occlusion_target: k_flow's mask instance, which also
stores the frame into a slot and reads four candidates from the other, then k_occ_commit).

For each benchmark shape — c2: small_loop, c3: loop_obstacles (4096 envs, 160x120), c4: udem1, 640x480, fisheye, domain
randomisation (`--c4-envs`, default 2048: the depth tensor is 1.2 MB per env there) — ONE env under device auto-reset
and bench.py's uniform random actions in [-1, 1], stepped with the depth target off and on in alternating arms, `rounds`
times.  The same handle runs both arms, so the arms differ in nothing but the kernels launched.
With --labels the arms are off / depth / labels / both, with --markings off / labels / markings / labels+markings (no
depth target in either), taken in an order that rotates from round to round; with --flow depth+labels / flow (depth,
labels and flow), alternated; with --flow --occlusion depth+labels / flow / flow+occlusion, in a rotating order.
k_flow's own time is the "post" bracket of the flow arm less that of depth+labels (the bracket holds nothing else
without a resize), and the mask's k_flow and k_occ_commit that of flow+occlusion less that of depth+labels.
Reports ms per step of each arm (host clock around `steps` steps ending in a synchronise, after `warmup` steps of that
arm), the median and the spread (min .. max) over the rounds, and, from a separate pass under dts_profile_enable(2)
(events at every kernel boundary, so not an end-to-end number), the ms per frame of each render kernel bracket; k_raster's
bracket holds the three rasterisers.  Prints one JSON line with the card's name, power limit and SM clocks read before
and after in the same run.

    python tools/depth_probe.py [--configs c2,c3,c4] [--steps 100] [--warmup 10] [--rounds 5] [--labels | --markings | --flow]
                                [--occlusion] [--out FILE.json]
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

SHAPES = {
    "c2": dict(map="small_loop", envs=4096, width=160, height=120, domain_rand=False, distortion=False),
    "c3": dict(map="loop_obstacles", envs=4096, width=160, height=120, domain_rand=False, distortion=False),
    "c4": dict(map="udem1", envs=2048, width=640, height=480, domain_rand=True, distortion=True),
}
ARMS = ["off", "on"]
LABEL_ARMS = ["off", "depth", "labels", "both"]
MARKING_ARMS = ["off", "labels", "markings", "labels+markings"]
FLOW_ARMS = ["depth+labels", "flow"]
OCCLUSION_ARMS = ["depth+labels", "flow", "flow+occlusion"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def set_arm(env, arm):
    if env.flow is not None:   # depth and labels stay on: the flow image reads them
        if env.flow_occlusion is not None:   # (the mask goes off before flow, and on after it)
            env.sim.set_occlusion_target(None)
        if arm in ("flow", "flow+occlusion"):   # (under the fisheye, with the forward maps of the pool's tables)
            models = env.camera_models if env.camera_rand else [env.camera_model] if env.distortion else []
            env.sim.set_flow_target(env.flow.data_ptr(), *((np.stack([m.mapx for m in models]),
                                                            np.stack([m.mapy for m in models])) if models else ()))
        else:
            env.sim.set_flow_target(None)
        if arm == "flow+occlusion":
            env.sim.set_occlusion_target(env.flow_occlusion.data_ptr())
        return
    env.sim.set_depth_target(env.depth.data_ptr() if arm in ("on", "depth", "both") else None)
    if env.labels is not None:
        env.sim.set_label_target(env.labels.data_ptr() if arm in ("labels", "both", "labels+markings") else None)
    if env.markings is not None:
        env.sim.set_marking_target(env.markings.data_ptr() if arm in ("markings", "labels+markings") else None)


def run(env, acts, steps, t0=0):
    for t in range(steps):
        env.step(acts[(t0 + t) % len(acts)])


def device_ms(env, arm, acts, steps, warmup):
    set_arm(env, arm)
    run(env, acts, warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(env, acts, steps, warmup)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def kernel_ms(env, arm, acts, steps):
    """ms per frame of each render kernel bracket, events at every boundary."""
    set_arm(env, arm)
    run(env, acts, 5)
    env.sim.profile(2)
    env.sim.profile_read()
    run(env, acts, steps)
    ms, frames = env.sim.profile_read()
    env.sim.profile(0)
    return {k: v / max(frames, 1) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3,c4")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--c4-envs", type=int, default=SHAPES["c4"]["envs"])
    ap.add_argument("--labels", action="store_true", help="arms off / depth / labels / both")
    ap.add_argument("--markings", action="store_true", help="arms off / labels / markings / labels+markings")
    ap.add_argument("--flow", action="store_true", help="arms depth+labels / depth+labels+flow")
    ap.add_argument("--occlusion", action="store_true", help="with --flow: arms depth+labels / flow / flow+occlusion")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.occlusion and not a.flow:
        sys.exit("--occlusion goes with --flow")
    arms = (OCCLUSION_ARMS if a.occlusion else FLOW_ARMS) if a.flow else MARKING_ARMS if a.markings else LABEL_ARMS if a.labels else ARMS
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "actions": "uniform [-1, 1]", "configs": {}}
    for cfg in a.configs.split(","):
        c = dict(SHAPES[cfg])
        if cfg == "c4":
            c["envs"] = a.c4_envs
        env = BatchedDuckietownEnv(c["envs"], c["map"], camera_width=c["width"], camera_height=c["height"],
                                   domain_rand=c["domain_rand"], distortion=c["distortion"], seed=1, device_reset=True,
                                   auto_reset=True, depth=True, labels=a.labels or a.markings, markings=a.markings,
                                   flow=a.flow, flow_occlusion=a.occlusion)
        env.reset()
        g = torch.Generator(device="cuda").manual_seed(0)
        acts = torch.rand((16, c["envs"], 2), device="cuda", generator=g) * 2 - 1
        runs = {k: [] for k in arms}
        for r in range(a.rounds):
            order = (arms if r % 2 == 0 else arms[::-1]) if len(arms) == 2 else arms[r % len(arms):] + arms[:r % len(arms)]
            for arm in order:     # no arm always runs first
                runs[arm].append(device_ms(env, arm, acts, a.steps, a.warmup))
            print(f"{cfg} round {r}: " + ", ".join(f"{k} {runs[k][-1]:.3f}" for k in arms) + " ms/step", file=sys.stderr, flush=True)
        kern = {arm: kernel_ms(env, arm, acts, min(a.steps, 50)) for arm in arms}
        env.check()
        med = {k: float(np.median(v)) for k, v in runs.items()}
        px = c["envs"] * c["width"] * c["height"]
        res["configs"][cfg] = {
            **c, "ms_per_step": runs, "median_ms_per_step": med,
            "spread_ms_per_step": {k: [float(min(v)), float(max(v))] for k, v in runs.items()},
            "kernel_ms_per_frame": kern, "obs_bytes_per_step": px * 3, "depth_bytes_per_step": px * 4,
            "labels_bytes_per_step": px * 2, "markings_bytes_per_step": px, "flow_bytes_per_step": px * 8}
        base = arms[0]
        for arm in arms[1:]:
            res["configs"][cfg].update({f"{arm}_minus_{base}_ms": med[arm] - med[base], f"{arm}_over_{base}": med[arm] / med[base],
                                        f"k_raster_{arm}_minus_{base}_ms": kern[arm]["k_raster"] - kern[base]["k_raster"]})
        if a.flow:
            res["configs"][cfg]["k_flow_ms_per_frame"] = kern["flow"]["post"] - kern[base]["post"]
        if a.occlusion:
            res["configs"][cfg]["k_flow_occlusion_ms_per_frame"] = kern["flow+occlusion"]["post"] - kern[base]["post"]
            res["configs"][cfg]["occlusion_bytes_per_step"] = px * (1 + 6 + 4 * 6)   # mask, slot write, 4 candidates
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
