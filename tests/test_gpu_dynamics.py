"""The step kernel's wheel path on the device, across the model's whole configuration (DESIGN.md §4): one step from
crafted snapshot records against the C oracle and the expm reference (tests/dynamics_ref.py), the action map against
the reference's own output, the command delay rule at every frame rate, trajectories at non-default constants, rates
and frame skips, MotionBlurWrapper's 1/90 s sub-steps, and the model's steady states."""
import os
import re
from contextlib import contextmanager
from unittest import mock

import numpy as np
import pytest

import dynamics_ref as ref
from test_dynamics_ref import DELAYS, POSE_BAR, RATES, oracle_step, reference_step, turn_cases

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "include", "dtsim.h")) as _f:
    MAX_DELAY = int(re.search(r"#define DTS_MAX_DELAY (\d+)", _f.read()).group(1))
# A snapshot record (include/dtsim.h, "dts_save_state"): the 144-byte RenderEp, then these 16 doubles, then the delay
# line fifo[DTS_MAX_DELAY][2] (slot 0 the oldest).
F64 = ("cx", "cy", "ctheta", "vu", "vw", "pos_x", "pos_z", "angle", "speed", "reward", "lane_dist", "lane_dot",
       "lane_angle", "prox", "wheel_dist", "trim")
I = {k: i for i, k in enumerate(F64)}
FIFO = len(F64)
REC0, REC1 = 144, 144 + 8 * (len(F64) + 2 * MAX_DELAY)
# CUDA's sincos and glibc's sin / cos may round differently.  Measured on an H100 over every one-step case below, the
# position came out bit-identical to the oracle's (0 ulp) and the wrapped angle within 1 ulp; the bars allow 2.
XPOS_ULP = 2
ANGLE_ULP = 2


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@contextmanager
def _model(model):
    """Build envs whose dts_config carries `model` (keys of oracle.DB18_NOMINAL) in its dyn_* fields."""
    from gym_duckietown_b200 import lib as L
    base = L.default_config
    fields = {f"dyn_{k}": float(v) for k, v in (model or {}).items()}
    with mock.patch.object(L, "default_config", lambda **kw: base(**kw, **fields)):
        yield


def make_env(name, n, model=None, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=32, camera_height=24, domain_rand=False, seed=1000)
    args.update(kw)
    with _model(model):
        return BatchedDuckietownEnv(n, name, **args)


def records(env):
    import torch
    rec = env.save_state()
    torch.cuda.synchronize()
    return rec, rec.cpu().numpy()


def doubles(host):
    """[n, 16 + 2 * DTS_MAX_DELAY] float64: the record's doubles and its delay line."""
    return np.ascontiguousarray(host[:, REC0:REC1]).view(np.float64)


def step_from(env, d64, actions):
    """Load records whose doubles are `d64` (the rest as the env has it now), take one step without rendering, and
    return the doubles of the records saved after it."""
    import torch
    rec, host = records(env)
    host[:, REC0:REC1] = np.ascontiguousarray(d64, np.float64).view(np.uint8)
    env.load_state(torch.from_numpy(host).to(env.device), fingerprint=rec.fingerprint)
    env.step(torch.from_numpy(np.asarray(actions, np.float32)).to(env.device), render=False)
    return doubles(records(env)[1])


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def wrapped(a, b):
    d = np.abs(np.asarray(a) - np.asarray(b))
    return np.minimum(d, 2 * np.pi - d)


# ------------------------------------------------------------------------------------------------ one step
def crafted_cases(rng, n):
    """(state, trim, delay line, action) per env for MODEL_ALL: random states and trims of both signs, headings at the
    +-pi wrap, duties beyond [-1, 1] waiting in the delay line and issued now."""
    out = []
    for k in range(n):
        th = rng.uniform(-7, 7)
        if k % 4 == 1:
            th = rng.choice([np.pi, -np.pi, 3 * np.pi]) + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-15, -3)
        state = [rng.uniform(0.3, 1.5), rng.uniform(0.3, 1.5), th, rng.uniform(-0.8, 0.8), rng.uniform(-9, 9)]
        trim = rng.choice([-1, 1]) * rng.uniform(0.01, 0.1)
        fifo = rng.uniform(-1.6, 1.6, (MAX_DELAY, 2))
        out.append((state, trim, fifo, rng.uniform(-1.5, 1.5, 2)))
    return out


@pytest.mark.parametrize("which", ["all_constants", "turns"])
def test_one_step_from_crafted_states(which, torch_cuda):
    """Every env starts from its own crafted record; after one step the kernel's 16 doubles and delay line must equal
    the oracle's step: bit for bit where the operations are the same (u, w, theta, the delay line, pos_x), within
    XPOS_ULP / ANGLE_ULP where sincos differs, and within POSE_BAR of the expm reference."""
    import oracle as orc
    rng = np.random.default_rng(77 if which == "all_constants" else 78)
    dt, D = 1.0 / 30, 5
    if which == "all_constants":
        model, cases = ref.MODEL_ALL, crafted_cases(rng, 96)
    else:
        model = ref.MODEL_TURN
        cases = [(st, trim, fifo, cmd) for _, trim, _, st, fifo, cmd, _ in turn_cases(rng)]
        for st, *_ in cases:
            st[0], st[1] = rng.uniform(0.3, 1.5), rng.uniform(0.3, 1.5)
    n = len(cases)
    env = make_env("small_loop", n, model, action_mode="pwm")
    try:
        env.reset(render=False)
        d64 = doubles(records(env)[1]).copy()
        for e, (st, trim, fifo, _) in enumerate(cases):
            d64[e, :5] = st
            d64[e, I["trim"]] = trim
            d64[e, FIFO:] = np.asarray(fifo).ravel()
        acts = np.array([c[3] for c in cases], np.float32)
        got = step_from(env, d64, acts)
        gh_ts = env.maps[0].grid_h * env.maps[0].tile_size
        worst = dict(pos_ulp=0.0, angle_ulp=0.0, ref=0.0)
        for e, (st, trim, fifo, _) in enumerate(cases):
            cmd = np.clip(acts[e].astype(np.float64), -1, 1)
            want, want_fifo = oracle_step(model, trim, dt, st, fifo, cmd, D)
            assert np.array_equal(got[e, 2:5], want[2:]), (e, got[e, 2:5], want[2:])
            assert np.array_equal(got[e, FIFO:].reshape(-1, 2), want_fifo), e
            assert got[e, I["pos_x"]] == got[e, 0] and got[e, I["pos_z"]] == gh_ts - got[e, 1]
            pu = ulps(got[e, :2], want[:2]).max()
            s, c = np.sin(want[2]), np.cos(want[2])
            au = wrapped(got[e, I["angle"]], np.arctan2(s, c)) / np.spacing(np.pi)
            rpos = np.array(reference_step(model, trim, dt, st, fifo, cmd, D)[0][:2])
            rerr = np.abs(got[e, :2] - rpos).max()
            worst = dict(pos_ulp=max(worst["pos_ulp"], pu), angle_ulp=max(worst["angle_ulp"], au),
                         ref=max(worst["ref"], rerr))
            assert pu <= XPOS_ULP and au <= ANGLE_ULP and rerr <= POSE_BAR, (e, pu, au, rerr)
        print(f"\none step, {which}: {worst}")
        if which == "turns":
            turned = got[:, 2] - np.array([c[0][2] for c in cases])
            assert np.any((np.abs(turned) > 0) & (np.abs(turned) < 2e-9))   # the Taylor branch and its neighbours ran
    finally:
        env.close()


# ------------------------------------------------------------------------------------------------ action map
def _mapped(env, actions, wheel_dist):
    """The duty the step issues for `actions`: the newest slot (D - 1) of a delay line that was empty."""
    D = 5
    rec = doubles(records(env)[1]).copy()
    rec[:, FIFO:] = 0.0
    rec[:, I["wheel_dist"]] = wheel_dist
    got = step_from(env, rec, actions)
    line = got[:, FIFO:].reshape(-1, MAX_DELAY, 2)
    assert not line[:, :D - 1].any() and not line[:, D:].any()
    return line[:, D - 1]


@pytest.mark.parametrize("cfg_index", [0, 1])
def test_action_map_vs_reference_golden(cfg_index, golden_dir, torch_cuda):
    """Both configurations of action_map.npz (the defaults; gain 0.8, trim 0.05, radius 0.03, k 25, limit 0.9), all
    512 actions, each env at the golden wheel distance: the issued duty matches the reference's output to 2e-6 (its
    float32 arithmetic, as in test_oracle_logic) and the oracle's action map bit for bit.  Then ActionWrapper's
    action_vel_scale = 0.8 and DiscreteWrapper's ids 0, 1, 2, against the oracle bit for bit."""
    import oracle as orc
    g = np.load(os.path.join(golden_dir, "action_map.npz"))
    cfg = [float(v) for v in g["cfgs"][cfg_index]]
    acts, wd = g["actions"].astype(np.float32), g["wheel_dist"]
    n = len(acts)
    env = make_env("small_loop", n, None, action_mode="vel_steer", **dict(zip(("gain", "trim", "radius", "k", "limit"), cfg)))
    try:
        env.reset(render=False)

        def want(vel):
            return np.array([np.clip(orc.action_map(vel[q], acts[q, 1], wd[q], *cfg), -1, 1) for q in range(n)])

        got = _mapped(env, acts, wd)
        assert np.abs(got - g["vels"][cfg_index]).max() <= 2e-6
        assert np.array_equal(got, want(acts[:, 0].astype(np.float64)))
        env.set_output_format(action_vel_scale=0.8)
        assert np.array_equal(_mapped(env, acts, wd), want(acts[:, 0].astype(np.float64) * 0.8))
        env.set_output_format(action_vel_scale=1.0, discrete_actions=True)
        ids = np.arange(n) % 3
        table = {0: (0.6, 1.0), 1: (0.6, -1.0), 2: (0.7, 0.0)}
        got = _mapped(env, np.stack([ids, np.zeros(n)], 1), wd)
        exp = np.array([np.clip(orc.action_map(*table[i], wd[q], *cfg), -1, 1) for q, i in enumerate(ids)])
        assert np.array_equal(got, exp)
    finally:
        env.close()


# ------------------------------------------------------------------------------------------------ delay rule
def _issued_line(env, rate):
    """Reset, issue one PWM command, and return the delay line and whether the robot started moving (its speed u;
    the reported speed can be an ulp off zero, as pos_z does not round-trip through the cartesian y exactly)."""
    env.reset(render=False)
    got = step_from(env, doubles(records(env)[1]), np.full((env.num_envs, 2), (0.8, 0.6), np.float32))
    return got[0, FIFO:].reshape(MAX_DELAY, 2), got[0, I["vu"]] != 0.0


@pytest.mark.parametrize("delay", DELAYS, ids=[str(d) for d in DELAYS])
def test_delay_rule_matches_the_oracle_at_every_rate(delay, torch_cuda):
    """For 15 ... 100 Hz, through dts_create and through dts_set_timing: the command issued lands in slot d - 1 of an
    empty line, the robot first moves after d steps, and d is what the oracle computes."""
    import oracle as orc
    from gym_duckietown_b200 import lib as L
    cmd = np.array([np.float32(0.8), np.float32(0.6)], np.float64)
    by_timing = make_env("small_loop", 1, dict(delay=float(delay)), action_mode="pwm")
    try:
        for rate in RATES:
            d = orc.delay_steps(float(delay), 1.0 / rate)
            assert d == -(-delay.numerator * rate // delay.denominator)
            by_create = make_env("small_loop", 1, dict(delay=float(delay)), action_mode="pwm", frame_rate=rate)
            by_timing.sim.set_timing(1.0 / rate, 1, L.ACTION_PWM)
            for env in (by_create, by_timing):
                line, moved = _issued_line(env, rate)
                want = np.zeros((MAX_DELAY, 2))
                if d:
                    want[d - 1] = cmd
                assert np.array_equal(line, want), (rate, float(delay), d, line[:, 0])
                assert moved == (d == 0), (rate, float(delay))
            by_create.close()
    finally:
        by_timing.close()


def test_delay_beyond_the_line_is_refused_and_leaves_timing_as_it_was(torch_cuda):
    """0.15 s at 120 Hz is 18 steps, more than DTS_MAX_DELAY: dts_create refuses it, and a refused dts_set_timing
    leaves dt, frame_skip, action_mode and the delay as they were (the env steps exactly as an untouched twin)."""
    import torch
    from gym_duckietown_b200 import lib as L
    with pytest.raises(L.DtsError, match="DTS_MAX_DELAY"):
        make_env("small_loop", 1, frame_rate=120)
    make_env("small_loop", 1, dict(delay=0.16), frame_rate=100).close()   # exactly 16 steps: accepted
    a = make_env("small_loop", 8, ref.MODEL_ALL, frame_rate=20)
    b = make_env("small_loop", 8, ref.MODEL_ALL, frame_rate=20)
    try:
        with pytest.raises(L.DtsError, match="DTS_MAX_DELAY"):
            a.sim.set_timing(1.0 / 120, 2, L.ACTION_PWM)
        a.reset(render=False)
        b.reset(render=False)
        rng = np.random.default_rng(9)
        for _ in range(8):
            act = torch.from_numpy(rng.uniform(-1, 1, (8, 2)).astype(np.float32)).to(a.device)
            a.step(act, render=False)
            b.step(act, render=False)
        assert np.array_equal(records(a)[1], records(b)[1])
        assert int(a.state["step_count"][0]) == 8
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ trajectories
# Measured on an H100 over the 12 trajectory runs: pose and speed within 4.0e-14 of the oracle, reward within 3.8e-14
# (relative to max(1, |reward|)).  The bars keep a margin of about 25x.
TRAJ_POSE = 1e-12
TRAJ_REWARD = 1e-12


@pytest.mark.parametrize("name", ["small_loop", "loop_dyn_duckiebots"])
@pytest.mark.parametrize("rate,frame_skip", [(20, 1), (20, 2), (60, 1), (60, 2), (90, 1), (90, 2)])
def test_trajectory_at_non_default_model_vs_oracle(name, rate, frame_skip, golden_dir, torch_cuda):
    """64 envs x 300 steps with every model constant non-zero, at 20, 60 and 90 Hz (3, 9 and 14 delay steps): flags
    bit-exact, pose, speed and reward to the measured bars.  On loop_dyn_duckiebots the obstacles step with dt too."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps
    N, T = 64, 300
    md = maps.load_map(name)
    wiggle = None
    if md.dyn_objects:
        wiggle = np.load(os.path.join(golden_dir, f"dynamic_{name}.npz"))["wiggle"]
        for d, w in zip(md.dyn_objects, wiggle):
            d.wiggle = float(w)
    mode = "pwm" if md.dyn_objects else "vel_steer"
    env = make_env(md, N, ref.MODEL_ALL, action_mode=mode, frame_rate=rate, frame_skip=frame_skip, max_steps=250)
    try:
        env.reset(render=False)
        torch.cuda.synchronize()
        st0 = {k: v.cpu().numpy().copy() for k, v in env.state.items()}
        om = orc.OracleMap(md)
        cpu = [orc.OracleEnv(om, st0["pos_x"][k], st0["pos_z"][k], st0["angle"][k], wheel_dist=st0["wheel_dist"][k],
                             action_mode=1 if mode == "vel_steer" else 0, max_steps=250, frame_skip=frame_skip,
                             dt=1.0 / rate, model=ref.MODEL_ALL,
                             dynamics=orc.OracleDynamics(om, wiggle=wiggle) if wiggle is not None else None)
               for k in range(N)]
        assert cpu[0].dp.delay_steps == {20: 3, 60: 9, 90: 14}[rate]
        acts = np.random.default_rng(rate * 10 + frame_skip).uniform(-1, 1, (T, N, 2)).astype(np.float32)
        acts[:, : N // 4, 0] = 0.15 if mode == "vel_steer" else 0.3
        acts[:, : N // 4, 1] *= 0.3
        acts[:, : N // 8] = 0.0
        worst = np.zeros(2)
        codes = set()
        for t in range(T):
            _, rew, done, info = env.step(torch.from_numpy(acts[t]).to(env.device), render=False)
            s = {k: v.cpu().numpy() for k, v in info.items()}
            d = done.cpu().numpy()
            o = [cpu[k].step(acts[t, k]) for k in range(N)]
            want = {f: np.array([getattr(x, f) for x in o]) for f in
                    ("pos_x", "pos_z", "angle", "speed", "reward", "tile_i", "tile_j", "done", "done_code",
                     "collided", "in_lane", "step_count")}
            for f, g in (("tile_i", "tile_i"), ("tile_j", "tile_j"), ("done_code", "done_code"),
                         ("collided", "collided"), ("in_lane", "in_lane"), ("step_count", "step_count")):
                assert np.array_equal(s[g].astype(np.int64), want[f].astype(np.int64)), (t, f)
            assert np.array_equal(d.astype(bool), want["done"].astype(bool)), t
            pose = max(np.abs(s["pos_x"] - want["pos_x"]).max(), np.abs(s["pos_z"] - want["pos_z"]).max(),
                       wrapped(s["angle"], want["angle"]).max(), np.abs(s["speed"] - want["speed"]).max())
            rw = (np.abs(s["reward"] - want["reward"]) / np.maximum(1.0, np.abs(want["reward"]))).max()
            worst = np.maximum(worst, (pose, rw))
            assert pose <= TRAJ_POSE and rw <= TRAJ_REWARD, (t, pose, rw)
            codes.update(int(c) for c in want["done_code"])
        print(f"\ntrajectory {name} {rate} Hz fs {frame_skip}: pose {worst[0]:.3g} reward {worst[1]:.3g} codes {codes}")
        assert 0 in codes and 1 in codes
    finally:
        env.close()


# ------------------------------------------------------------------------------------------------ MotionBlurWrapper
def test_motion_blur_wrapper_vs_oracle(torch_cuda):
    """10 wrapper steps = 30 sub-steps of 1/90 s, past the 14-step delay, with per-env PWM actions: after each, pose,
    speed, reward and done equal an oracle env at dt = 1/90 stepped three times."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps, wrappers as Wr
    N = 16
    env = make_env("loop_obstacles", N, action_mode="pwm")
    try:
        env.reset(render=False)
        torch.cuda.synchronize()
        st0 = {k: v.cpu().numpy().copy() for k, v in env.state.items()}
        om = orc.OracleMap(maps.load_map("loop_obstacles"))
        cpu = [orc.OracleEnv(om, st0["pos_x"][k], st0["pos_z"][k], st0["angle"][k], action_mode=0, dt=1.0 / 90)
               for k in range(N)]
        assert cpu[0].dp.delay_steps == 14
        w = Wr.MotionBlurWrapper(env)
        rng = np.random.default_rng(4)
        for t in range(10):
            a = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
            a[: N // 2] = np.abs(a[: N // 2]) * 0.5 + 0.5          # half of them drive forwards
            _, rew, done, info = w.step(torch.from_numpy(a).to(env.device))
            s = {k: v.cpu().numpy() for k, v in info.items()}
            r, d = rew.cpu().numpy(), done.cpu().numpy()
            for k in range(N):
                for _ in range(3):
                    o = cpu[k].step(a[k])
                assert abs(s["pos_x"][k] - o.pos_x) <= TRAJ_POSE and abs(s["pos_z"][k] - o.pos_z) <= TRAJ_POSE, (t, k)
                assert wrapped(s["angle"][k], o.angle) <= TRAJ_POSE and abs(s["speed"][k] - o.speed) <= TRAJ_POSE
                assert abs(s["reward"][k] - o.reward) <= TRAJ_REWARD * max(1.0, abs(o.reward)), (t, k)
                assert abs(r[k] - np.float32(o.reward)) <= 1e-3 * max(1.0, abs(o.reward))
                assert bool(d[k]) == bool(o.done) and s["done_code"][k] == o.done_code, (t, k)
            assert int(s["step_count"][0]) == 3 * (t + 1)
        assert (s["speed"][: N // 2] > 0).all()                  # past the delay: they move
    finally:
        env.close()


def test_steady_states_on_the_device(torch_cuda):
    """The nominal model's steady states, as the oracle's anchors check them: 0.6 m/s at duty (1, 1), 7.5 rad/s at
    (-1, +1)."""
    env = make_env("small_loop", 2, action_mode="pwm")
    try:
        env.reset(render=False)
        import torch
        act = torch.tensor([[1.0, 1.0], [-1.0, 1.0]], device=env.device)
        for _ in range(200):
            env.step(act, render=False)
        d64 = doubles(records(env)[1])
        assert abs(d64[0, I["vu"]] - 0.6) < 1e-6 and abs(d64[0, I["vw"]]) < 1e-12
        assert abs(d64[1, I["vw"]] - 7.5) < 1e-6 and abs(d64[1, I["vu"]]) < 1e-12
    finally:
        env.close()
