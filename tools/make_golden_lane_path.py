#!/usr/bin/env python3
"""Generate the lane path fixtures under tests/golden/ by executing the REFERENCE's own code (oracle/refstub.py), as
oracle/make_golden.py does for the others.  Needs the reference source tree; the fixtures are committed.

    python tools/make_golden_lane_path.py

  lane_path_<map>.npz   the walk of DESIGN.md section 5 item 18 through the reference's own
                        Simulator.closest_curve_point (simulator.py:1337-1369): from each pose of make_golden's
                        sample_poses mix, (q0, t0) = ccp((x, 0, z), angle), then (q_{k+1}, t_{k+1}) = ccp(q_k + ds t_k,
                        atan2(-t_k.z, t_k.x)) until K points or the first None, for every ds of SPACINGS.
                        poses [n, 3] (x, z, angle); spacing [S]; count [S, n]; q, t [S, n, K, 3] (NaN past count)
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import make_golden as mg  # noqa: E402
import refstub  # noqa: E402
from gym_duckietown_b200 import maps  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
MAPS = ["small_loop", "loop_obstacles", "udem1", "loop_trafficlights"]   # udem1 and loop_trafficlights have 3-way tiles
SPACINGS = (0.05, 0.1, 0.3)
K = 64


def gen_lane_path(name: str, n=128, seed=31):
    raw = mg.raw_map(name)
    md = maps.load_map(name)
    sim = refstub.build_reference_sim(raw, mg.extents_for(raw))
    poses = mg.sample_poses(md, n, np.random.default_rng(seed))
    q = np.full((len(SPACINGS), n, K, 3), np.nan)
    t = np.full((len(SPACINGS), n, K, 3), np.nan)
    count = np.zeros((len(SPACINGS), n), np.int16)
    for s, ds in enumerate(SPACINGS):
        for e, (x, z, a) in enumerate(poses):
            pos, angle = np.array([x, 0.0, z]), a
            for k in range(K):
                p, tg = sim.closest_curve_point(pos, angle)
                if p is None:
                    break
                q[s, e, k], t[s, e, k] = p, tg
                count[s, e] = k + 1
                angle = np.arctan2(-tg[2], tg[0])
                pos = p + ds * tg
    np.savez_compressed(os.path.join(OUT, f"lane_path_{name}.npz"), poses=poses, spacing=np.array(SPACINGS),
                        count=count, q=q, t=t)
    print(f"lane_path_{name}: {n} poses, mean count {count.mean(1)}")


if __name__ == "__main__":
    refstub.install()
    for m in MAPS:
        gen_lane_path(m)
