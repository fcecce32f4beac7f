"""The navigation task (DuckietownNav, DESIGN.md §6c) on the CPU: the host EpisodeSampler's goal draw against the
reference's own DuckietownNav.reset (tests/golden/nav_<map>.npz, tools/make_golden_nav.py), the arrival test's fixture
against the oracle's done / reward with the goal test applied, and the C ABI's new names and signatures."""
import copy
import os
import re

import numpy as np
import pytest

import oracle as orc
from gym_duckietown_b200 import maps
from gym_duckietown_b200.episode import EpisodeSampler
from test_reset_sampler import oracle_query

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAPS = ["small_loop", "loop_obstacles", "udem1", "loop_dyn_duckiebots"]
STATIC_MAPS = MAPS[:3]
M64 = (1 << 64) - 1


def stream_words(g):
    st = g.bit_generator.state
    return [st["state"]["state"] >> 64, st["state"]["state"] & M64, st["has_uint32"], st["uinteger"]]


def nav_done_reward(o, goal):
    """DuckietownNav.step (envs/duckietown_env.py:119-125) on top of a step's outputs: (reward, done, done_code)."""
    if (o.tile_i, o.tile_j) == tuple(goal):
        return 1000.0, True, 3
    return o.reward, bool(o.done), o.done_code


def check_sampler(g, tag, md, seeds, **kw):
    s = EpisodeSampler(len(seeds), domain_rand=tag == "dr", nav=True, **kw)
    s.seed(seeds)
    envs = list(range(len(seeds)))
    for ep in range(2):
        out = s.sample(envs, [md] * len(envs), oracle_query(md))
        rows = np.arange(len(envs)) * 2 + ep
        assert np.array_equal(out["pos_x"], g[f"{tag}_cur_pos"][rows, 0]), (tag, ep)
        assert np.array_equal(out["pos_z"], g[f"{tag}_cur_pos"][rows, 2]), (tag, ep)
        assert np.array_equal(out["angle"], g[f"{tag}_cur_angle"][rows]), (tag, ep)
        assert np.array_equal(out["goal"], g[f"{tag}_goal"][rows]), (tag, ep)
        # the stream stands where the reference's does after the goal loop: the next reset draws alike
        got = np.array([stream_words(s.rngs[e]) for e in envs], np.uint64)
        assert np.array_equal(got, g[f"{tag}_stream"][rows]), (tag, ep)
        start = np.stack([np.floor(out["pos_x"] / md.tile_size), np.floor(out["pos_z"] / md.tile_size)], 1)
        assert not (start == out["goal"]).all(1).any()
        assert all(tuple(t) in md.drivable_tiles for t in out["goal"])


@pytest.mark.parametrize("name", MAPS)
def test_host_goal_draws_match_reference(name, golden_dir):
    g = np.load(os.path.join(golden_dir, f"nav_{name}.npz"))
    md = maps.load_map(name)
    for tag in ("nodr", "dr"):
        check_sampler(g, tag, md, [int(v) for v in g["seeds"]])


def test_host_goal_draws_after_fixed_starts_match_reference(golden_dir):
    """user_tile_start, the map's start_tile and start_pose (no spawn loop at all): the goal avoids the start tile."""
    g = np.load(os.path.join(golden_dir, "nav_udem1.npz"))
    base = maps.load_map("udem1")
    md_tile = copy.deepcopy(base); md_tile.start_tile = tuple(int(v) for v in g["start_tile"])
    md_pose = copy.deepcopy(md_tile)
    sp = g["start_pose"]
    md_pose.start_pose = [[float(sp[0]), float(sp[1]), float(sp[2])], float(sp[3])]
    cases = {"user": (base, dict(user_tile_start=tuple(int(v) for v in g["user_tile_start"]))),
             "tile": (md_tile, {}), "pose": (md_pose, {})}
    for tag, (md, kw) in cases.items():
        check_sampler(g, tag, md, list(range(12)), **kw)


def test_nav_off_draws_nothing_more(golden_dir):
    """Without nav the sampler's streams stand where the plain reset leaves them: the goal loop's draws are the only
    difference between the two."""
    g = np.load(os.path.join(golden_dir, "nav_small_loop.npz"))
    md = maps.load_map("small_loop")
    seeds = [int(v) for v in g["seeds"]]
    plain, nav = (EpisodeSampler(len(seeds), domain_rand=False, nav=v) for v in (False, True))
    plain.seed(seeds); nav.seed(seeds)
    a = plain.sample(list(range(len(seeds))), [md] * len(seeds), oracle_query(md))
    b = nav.sample(list(range(len(seeds))), [md] * len(seeds), oracle_query(md))
    assert "goal" not in a and "goal" in b
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    for e in range(len(seeds)):   # replaying the goal loop on the plain stream lands where the nav stream is
        EpisodeSampler._draw_goal(plain.rngs[e], md, a["pos_x"][e], a["pos_z"][e])
        assert stream_words(plain.rngs[e]) == stream_words(nav.rngs[e])


@pytest.mark.parametrize("name", STATIC_MAPS)
def test_arrival_fixture_is_the_step_with_the_goal_test(name, golden_dir):
    """The reference's DuckietownNav.step on sampled poses equals the oracle's _compute_done_reward with the goal test
    of DESIGN §6c on top: the restatement the device tests hold the step kernel to.  (The oracle's done_reward leaves
    moving obstacles out of the proximity penalty, so the maps without them.)"""
    g = np.load(os.path.join(golden_dir, f"nav_{name}.npz"))
    om = orc.OracleMap(maps.load_map(name))
    goal = tuple(int(v) for v in g["step_goal"])
    at_goal = 0
    for (x, z, a), st, r, d in zip(g["step_poses"], g["step_count"], g["step_reward"], g["step_done"]):
        o = om.done_reward(x, z, a, int(st))
        rew, done, code = nav_done_reward(o, goal)
        assert done == bool(d) and abs(rew - r) <= 1e-9 * max(1.0, abs(r)), (x, z, a, st)
        at_goal += code == 3
    assert at_goal > 10


def test_sampler_refuses_a_map_with_one_drivable_tile():
    md = copy.deepcopy(maps.load_map("small_loop"))
    md.drivable_tiles = md.drivable_tiles[:1]
    with pytest.raises(ValueError, match="two drivable tiles"):
        EpisodeSampler._draw_goal(np.random.default_rng(0), md, 0.0, 0.0)


def test_header_names_and_ctypes_signatures():
    from gym_duckietown_b200 import lib as L
    import gym_duckietown_b200 as gd
    hdr = open(os.path.join(ROOT, "include", "dtsim.h")).read()
    assert int(re.search(r"DTS_FLAG_NAV = (\d+)", hdr).group(1)) == L.FLAG_NAV == 64
    assert int(re.search(r"DTS_GOAL_REACHED = (\d+)", hdr).group(1)) == L.GOAL_REACHED == 3
    assert gd.DONE_CODE_NAMES[L.GOAL_REACHED] == "goal-reached" and len(gd.DONE_CODE_NAMES) == 4
    lib = L.load()
    for name in ("dts_set_goals", "dts_get_goals"):
        params = re.search(r"int %s\(([^)]*)\)" % name, hdr).group(1).split(",")
        assert len(getattr(lib, name).argtypes) == len(params), name
    assert "dts_set_goals" in L.EXPORTS and "dts_get_goals" in L.EXPORTS
