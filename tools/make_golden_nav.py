#!/usr/bin/env python3
"""Generate the navigation fixtures under tests/golden/ by executing the REFERENCE's own code (oracle/refstub.py), as
oracle/make_golden.py does for the others.  Needs the reference source tree; the fixtures are committed.

    python tools/make_golden_nav.py

The reference's DuckietownNav (envs/duckietown_env.py:89-127) cannot run as written: its reset and step call
themselves, and its `np_random.randint` does not exist on the Generator the reference's seeding returns.  The
methods' own source is compiled here with exactly those three tokens corrected (DuckietownNav.reset -> DuckietownEnv.reset,
DuckietownNav.step -> DuckietownEnv.step, randint -> integers) and run on a reference Simulator built by refstub.

  nav_<map>.npz   for seeds 0..23, domain_rand off ("nodr") and on ("dr"), two episodes from one stream (row 2 * seed +
                  episode): cur_pos, cur_angle, the goal tile's coords `goal` [2], and the stream after the reset
                  (`stream` [4]: state >> 64, state & (2^64 - 1), has_uint32, uinteger).  For udem1 also the fixed
                  starts of reset_start_udem1.npz (user_tile_start, the map's start_tile, start_pose), domain_rand off:
                  <case>_cur_pos, <case>_cur_angle, <case>_goal, <case>_stream.  Then DuckietownNav.step's arrival test
                  on make_golden's pose mix, each against the goal of nodr row 0: step_poses [n, 3], step_count [n],
                  step_reward [n], step_done [n], step_goal [2].
"""
from __future__ import annotations

import copy
import inspect
import os
import sys
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import make_golden as mg  # noqa: E402
import refstub  # noqa: E402
from gym_duckietown_b200 import maps  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
MAPS = ["small_loop", "loop_obstacles", "udem1", "loop_dyn_duckiebots"]
SEEDS = range(24)
M64 = (1 << 64) - 1


def corrected_nav():
    """DuckietownNav with its reset and step compiled from the reference's source, the three defects corrected."""
    refstub.install()
    from gym_duckietown.envs import duckietown_env as E
    if getattr(E.DuckietownNav, "_corrected", False):
        return E
    E.DuckietownNav._corrected = True
    ns = dict(vars(E))
    for meth, fixes in (("reset", [("DuckietownNav.reset(self)", "DuckietownEnv.reset(self)"),
                                   ("np_random.randint(", "np_random.integers(")]),
                        ("step", [("DuckietownNav.step(self, action)", "DuckietownEnv.step(self, action)")])):
        src = textwrap.dedent(inspect.getsource(getattr(E.DuckietownNav, meth)))
        for a, b in fixes:
            assert src.count(a) == 1, (meth, a)
            src = src.replace(a, b)
        exec(compile(src, E.__file__, "exec"), ns)
        setattr(E.DuckietownNav, meth, ns[meth])
    return E


def stream_words(sim):
    st = sim.np_random.bit_generator.state
    s = st["state"]["state"]
    return [s >> 64, s & M64, st["has_uint32"], st["uinteger"]]


def run_resets(E, raw, dr, seeds, **kw):
    rows = {k: [] for k in ("cur_pos", "cur_angle", "goal", "stream")}
    for seed in seeds:
        sim = refstub.build_reference_sim(raw, mg.extents_for(raw), domain_rand=dr, seed=int(seed), cls=E.DuckietownNav,
                                          **kw)
        S = refstub.modules()[0]
        S.gl.glLightfv = lambda *a: None

        class _GLf:
            def __mul__(self, n):
                return lambda *v: np.array(v, dtype=np.float32)
        S.gl.GLfloat = _GLf()
        for episode in range(2):
            sim.reset()
            rows["cur_pos"].append(np.array(sim.cur_pos, float)); rows["cur_angle"].append(float(sim.cur_angle))
            rows["goal"].append(np.array(sim.goal_tile["coords"], np.int64))
            rows["stream"].append(np.array(stream_words(sim), np.uint64))
    return {k: np.array(v) for k, v in rows.items()}, sim


def arrival(E, sim, md, n=1536, seed=7):
    """DuckietownNav.step's test on sampled poses: DuckietownEnv.step stands in as _compute_done_reward of the pose."""
    rng = np.random.default_rng(seed)
    poses = mg.sample_poses(md, n, rng)
    steps = rng.integers(0, 4, n)
    reward, done = [], []
    orig = E.DuckietownEnv.step

    def env_step(self, action):
        d = self._compute_done_reward()
        return None, float(d.reward), bool(d.done), {}
    E.DuckietownEnv.step = env_step
    try:
        for (x, z, a), st in zip(poses, steps):
            sim.cur_pos, sim.cur_angle = np.array([x, 0.0, z]), a
            sim.step_count = sim.max_steps if st == 0 else int(st)
            _, r, d, info = sim.step(None)
            assert info["goal_tile"] is sim.goal_tile
            reward.append(float(r)); done.append(bool(d))
    finally:
        E.DuckietownEnv.step = orig
    return dict(step_poses=poses, step_count=np.where(steps == 0, sim.max_steps, steps).astype(np.int32),
                step_reward=np.array(reward), step_done=np.array(done),
                step_goal=np.array(sim.goal_tile["coords"], np.int64))


def gen_nav(name: str):
    E = corrected_nav()
    raw = mg.raw_map(name)
    out = {"seeds": np.array(list(SEEDS))}
    for tag, dr in (("nodr", False), ("dr", True)):
        rows, _ = run_resets(E, raw, dr, SEEDS)
        out.update({f"{tag}_{k}": v for k, v in rows.items()})
    # the arrival test against the goal of seed 0's first episode (domain_rand off)
    first = refstub.build_reference_sim(raw, mg.extents_for(raw), seed=0, cls=E.DuckietownNav)
    S = refstub.modules()[0]
    S.gl.glLightfv = lambda *a: None
    first.reset()
    assert list(first.goal_tile["coords"]) == list(out["nodr_goal"][0])
    out.update(arrival(E, first, maps.load_map(name)))
    if name == "udem1":   # the fixed starts of reset_start_udem1.npz
        cases = {"user": (raw, dict(user_tile_start=(1, 1))),
                 "tile": (dict(copy.deepcopy(raw), start_tile=[3, 1]), {}),
                 "pose": (dict(copy.deepcopy(raw), start_tile=[3, 1], start_pose=[[0.21, 0.0, 0.33], 1.4]), {})}
        for tag, (mp, kw) in cases.items():
            rows, _ = run_resets(E, mp, False, range(12), **kw)
            out.update({f"{tag}_{k}": v for k, v in rows.items()})
        out["start_tile"], out["start_pose"], out["user_tile_start"] = \
            np.array([3, 1]), np.array([0.21, 0.0, 0.33, 1.4]), np.array([1, 1])
    np.savez_compressed(os.path.join(OUT, f"nav_{name}.npz"), **out)
    print(f"nav_{name}: {len(SEEDS)} seeds x 2 episodes x (dr off/on), {len(out['step_poses'])} arrival poses, "
          f"{int(out['step_done'].sum())} done, {int((out['step_reward'] == 1000).sum())} at the goal")


if __name__ == "__main__":
    for m in MAPS:
        gen_nav(m)
