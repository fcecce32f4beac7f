"""The C oracle's wheel path held to tests/dynamics_ref.py, an independent float64 restatement whose pose update is
scipy's matrix exponential of the twist rather than the closed form (DESIGN.md §4), and the command delay rule and
delay-line depth the oracle shares with the device.  CPU only."""
import ctypes as C
import os
import re
from fractions import Fraction

import numpy as np
import pytest

import dynamics_ref as ref
import oracle as orc
from gym_duckietown_b200 import maps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Measured over the cases below: the closed form and the expm reference differ by at most 8.9e-16 m in position (two
# ulps of coordinates in [-5, 5]), 4.4e-16 in theta, 1.1e-16 m/s in u and 1.8e-15 rad/s in w (the reference groups the
# forcing terms differently).  The bars keep a margin of about 10x.  Before the lateral term was computed as
# 2 sin^2(a/2) / a, turns of 1e-9 to 1e-7 cost up to 1.1e-11 m here, from 1 - cos(a) cancelling.
POSE_BAR = 1e-14
VEL_BAR = 2e-14
RATES = [15, 20, 24, 30, 40, 60, 90, 100]
DELAYS = [Fraction(1, 30), Fraction(1, 10), Fraction(3, 20), Fraction(0)]


def _define(path, name):
    with open(os.path.join(ROOT, path)) as f:
        return int(re.search(rf"#define {name} (\d+)", f.read()).group(1))


def test_delay_line_is_as_deep_in_the_oracle_as_on_the_device():
    depth = _define("include/dtsim.h", "DTS_MAX_DELAY")
    assert _define("oracle/dt_oracle.h", "ORC_MAX_DELAY") == depth
    assert orc.ORC_MAX_DELAY == depth and len(orc.OrcDynState().fifo) == depth


@pytest.mark.parametrize("rate", RATES)
def test_delay_rule_gives_the_exact_step_count(rate):
    """A command issued at t acts on the intervals starting at or after t + delay: ceil(delay · rate) steps, computed
    exactly here.  Exact multiples (0.1 s at 20 Hz, 1/30 s at 30 or 60 Hz) must not round up to one step more.  The
    oracle env is checked to first move on the step after that count, its delay line filled to that depth."""
    om = orc.OracleMap(maps.load_map("small_loop"))
    for delay in DELAYS:
        want = -(-delay.numerator * rate // delay.denominator)
        assert orc.delay_steps(float(delay), 1.0 / rate) == want, (rate, delay)
        env = orc.OracleEnv(om, 1.0, 1.0, 0.0, action_mode=0, dt=1.0 / rate, model=dict(delay=float(delay)))
        assert env.dp.delay_steps == want
        for k in range(want):
            assert env.step([0.8, 0.6]).speed == 0.0, (rate, delay, k)
        assert np.all(np.asarray(env.s.fifo)[:want] == [0.8, 0.6]) and np.all(np.asarray(env.s.fifo)[want:] == 0.0)
        assert env.step([0.8, 0.6]).speed > 0.0, (rate, delay)


def test_a_delay_longer_than_the_line_is_refused():
    assert orc.delay_steps(0.16, 0.01) == orc.ORC_MAX_DELAY
    orc.dyn_params(0.01, delay=0.16)                        # 16 steps: the line's full depth
    with pytest.raises(ValueError, match="delay line"):
        orc.dyn_params(1.0 / 120, delay=0.15)               # 18 steps
    with pytest.raises(TypeError):
        orc.dyn_params(1.0 / 30, u4=1.0)


def test_oracle_runs_at_90_hz_within_its_delay_line():
    """MotionBlurWrapper's 1/90 s sub-steps: 14 delay steps, more than the 8 the oracle's line once held."""
    om = orc.OracleMap(maps.load_map("small_loop"))
    env = orc.OracleEnv(om, 1.0, 1.0, 0.0, action_mode=0, dt=1.0 / 90)
    assert env.dp.delay_steps == 14 and orc.OrcDynState.fifo.size == 16 * orc.ORC_MAX_DELAY
    for k in range(14):
        assert env.step([1.0, 1.0]).speed == 0.0
    assert env.step([1.0, 1.0]).speed > 0.0


def oracle_step(model, trim, dt, state, fifo, cmd, d):
    p = orc.dyn_params(dt, trim, **model)
    p.delay_steps = d
    s = orc.OrcDynState(*state[:5])
    for k in range(orc.ORC_MAX_DELAY):
        s.fifo[k][0], s.fifo[k][1] = fifo[k]
    orc.lib().orc_dyn_step(C.byref(s), C.byref(p), (C.c_double * 2)(*cmd), C.c_double(dt))
    return np.array([s.x, s.y, s.theta, s.u, s.w]), np.array(s.fifo)


def reference_step(model, trim, dt, state, fifo, cmd, d):
    acting, line = ref.delay_push(fifo[:d], cmd, d)
    full = np.asarray(fifo, np.float64).copy()
    full[:d] = line
    return np.array(ref.db18_step(*state[:5], acting, model, trim, dt)), full


def random_cases(rng, n):
    for _ in range(n):
        model = {k: v * rng.uniform(0.5, 1.5) for k, v in ref.MODEL_ALL.items()}
        model = {k: v * rng.choice([-1.0, 1.0]) if k in ("u2", "u3", "w2", "w3") else v for k, v in model.items()}
        dt = 1.0 / rng.uniform(15, 100)
        state = [rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(-7, 7), rng.uniform(-1, 1), rng.uniform(-9, 9)]
        fifo = rng.uniform(-1.6, 1.6, (orc.ORC_MAX_DELAY, 2))
        yield model, rng.normal(0, 0.1), dt, state, fifo, rng.uniform(-1, 1, 2), int(rng.integers(0, 17))


def turn_cases(rng):
    dt = 1.0 / 30
    for a in ref.turn_values():
        for trim in (-0.07, 0.05):
            u = rng.uniform(0.2, 0.8)
            w, got = ref.w_for_turn(a, u, ref.MODEL_TURN, trim, dt)
            assert got == a, (a, got)
            state = [rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(-7, 7), u, w]
            fifo = np.zeros((orc.ORC_MAX_DELAY, 2))
            fifo[1:] = rng.uniform(-1, 1, (orc.ORC_MAX_DELAY - 1, 2))
            yield ref.MODEL_TURN, trim, dt, state, fifo, rng.uniform(-1, 1, 2), 5


def test_oracle_step_vs_expm_reference():
    """One model step from random states, constants, trims, rates and delay lines (duties beyond [-1, 1] waiting in
    the line, so the model's own clip acts), and from states whose turn a = dt·w' is one of ref.turn_values()."""
    rng = np.random.default_rng(2024)
    worst = 0.0
    cases = list(random_cases(rng, 3000)) + list(turn_cases(rng))
    for model, trim, dt, state, fifo, cmd, d in cases:
        got, got_fifo = oracle_step(model, trim, dt, state, fifo, cmd, d)
        want, want_fifo = reference_step(model, trim, dt, state, fifo, cmd, d)
        assert np.array_equal(got_fifo, want_fifo)
        err = np.abs(got[:2] - want[:2]).max()
        worst = max(worst, err)
        assert err <= POSE_BAR, (model, trim, dt, state, err)
        assert np.abs(got[2:] - want[2:]).max() <= VEL_BAR, (got[2:], want[2:])
    assert worst > 0.0      # the two really are computed differently


def test_action_map_vs_reference_restatement(golden_dir):
    """The oracle's action map equals the restatement bit for bit, for both configurations of action_map.npz."""
    g = np.load(os.path.join(golden_dir, "action_map.npz"))
    for cfg in g["cfgs"]:
        for q in range(len(g["actions"])):
            a = (float(g["actions"][q, 0]), float(g["actions"][q, 1]), float(g["wheel_dist"][q]))
            assert orc.action_map(*a, *cfg) == ref.action_map(*a, *cfg), (cfg, q)
