"""Terminal frames under device auto-reset (terminal_obs=True, dts_step_terminal).

The reference's step() returns the terminal frame of an episode that ended (render_obs() S:1677, before the caller's
reset()).  Under auto_reset the batched env returns the next episode's first frame in `obs`; with terminal_obs=True it
also writes the terminal frame of every env that ended into `terminal_obs`.  It does so with a second render over a
device list of the ended envs only.

The bars, all bit-identical (0 LSB):
  - against the reference-style loop on a handle without auto-reset (step, then reset(mask=done)): the same done and
    reward, terminal_obs[done] == that loop's step observation, obs == its observation after the reset;
  - against the same env with terminal_obs off: the same obs, reward, done and state on every step, so the deferred
    respawn leaves the state and the PCG64 draws exactly where the in-kernel one does;
  - rows of envs that did not end keep what terminal_obs held, and a step where nothing ends changes nothing.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H = 160, 120


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, maps="small_loop", **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=W, camera_height=H, domain_rand=False, seed=11, device_reset=True)
    args.update(kw)
    return BatchedDuckietownEnv(n, maps, **args)


def forward_actions(torch, steps, n, seed=3):
    """Random actions biased forward: velocity in [0.2, 1], steering in [-1, 1].  Both kinds of termination happen:
    invalid poses off the road, and max_steps."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.rand((steps, n, 2), device="cuda", generator=g)
    a[..., 0] = 0.2 + 0.8 * a[..., 0]
    a[..., 1] = a[..., 1] * 2 - 1
    return a


def assert_same_state(a, b, what):
    for k in a:
        assert np.array_equal(a[k].cpu().numpy(), b[k].cpu().numpy(), equal_nan=True), f"{what}: state[{k!r}] differs"


# ---------------------------------------------------------------------------------------------- the reference loop
LOOP_CASES = {
    "small_loop": dict(maps="small_loop"),
    "loop_obstacles": dict(maps="loop_obstacles"),
    "loop_dyn_duckiebots": dict(maps="loop_dyn_duckiebots"),
    "domain_rand": dict(maps="loop_obstacles", domain_rand=True),
}


@pytest.mark.parametrize("case", sorted(LOOP_CASES))
def test_matches_reference_style_loop(torch_cuda, case):
    torch = torch_cuda
    n, steps, kw = 48, 60, dict(LOOP_CASES[case])
    maps = kw.pop("maps")
    a = make_env(n, maps, max_steps=12, auto_reset=True, terminal_obs=True, **kw)
    b = make_env(n, maps, max_steps=12, **kw)
    a.reset()
    b.reset()
    torch.cuda.synchronize()
    assert torch.equal(a.obs, b.obs)
    acts = forward_actions(torch, steps, n)
    codes = set()
    for t in range(steps):
        _, ra, da, sa = a.step(acts[t])
        ob, rb, db, sb = b.step(acts[t])
        torch.cuda.synchronize()
        assert torch.equal(da, db), f"step {t}: done differs"
        assert torch.equal(ra, rb), f"step {t}: reward differs"
        assert torch.equal(a.terminal_obs[da], ob[db]), f"step {t}: terminal frames differ"
        codes |= set(sb["done_code"][db].tolist())
        b.reset(mask=db)
        torch.cuda.synchronize()
        assert torch.equal(a.obs, b.obs), f"step {t}: the first frames of the new episodes differ"
    episodes = a.state["episode"].cpu().numpy()
    assert episodes.min() >= 3, episodes   # (the first reset counts one)
    assert codes == {1, 2}, f"termination kinds seen: {codes}"
    a.check()
    b.check()
    a.close()
    b.close()


# ---------------------------------------------------------------------------------- nothing else changes
def setup_fmt(layout, dtype):
    return lambda e: e.set_output_format(obs_layout=layout, obs_dtype=dtype)


def setup_resize(method):
    return lambda e: e.set_resize(84, 84, method=method)


def setup_rectify(e):
    from gym_duckietown_b200.distortion import rectify_maps
    e.set_rectification(*rectify_maps(e.camera_width, e.camera_height))
    e.undistort = True


SAME_CASES = {
    "hwc_u8": (dict(), setup_fmt("hwc", "uint8")),
    "chw_f32": (dict(), setup_fmt("chw", "float32")),
    "cwh_u8": (dict(), setup_fmt("cwh", "uint8")),
    "resize_cv2_cubic": (dict(), setup_resize("cv2_cubic")),
    "resize_pil_bilinear_chw_f32": (dict(), lambda e: (setup_fmt("chw", "float32")(e), setup_resize("pil_bilinear")(e))),
    "fisheye_640x480": (dict(n=8, camera_width=640, camera_height=480, distortion=True, maps="udem1"), None),
    "rectify_640x480": (dict(n=8, camera_width=640, camera_height=480, distortion=True, maps="udem1"), setup_rectify),
    "cycle_maps": (dict(maps=["small_loop", "loop_obstacles"], cycle_maps=True), None),
    "randomize_maps_on_reset": (dict(maps=["small_loop", "loop_dyn_duckiebots"], randomize_maps_on_reset=True,
                                     domain_rand=True), None),
    "frame_skip3_dynamics_rand": (dict(frame_skip=3, dynamics_rand=True, domain_rand=True, maps="loop_dyn_duckiebots"),
                                  None),
}


@pytest.mark.parametrize("case", sorted(SAME_CASES))
def test_changes_nothing_else(torch_cuda, case):
    torch = torch_cuda
    kw, setup = SAME_CASES[case]
    kw = dict(kw)
    n, maps = kw.pop("n", 40), kw.pop("maps", "small_loop")
    steps = 30 if n >= 40 else 20
    a = make_env(n, maps, max_steps=8, auto_reset=True, terminal_obs=True, **kw)
    c = make_env(n, maps, max_steps=8, auto_reset=True, **kw)
    for e in (a, c):
        if setup:
            setup(e)
        e.reset()
    assert a.terminal_obs.shape == a.obs.shape and a.terminal_obs.dtype == a.obs.dtype
    acts = forward_actions(torch, steps, n, seed=5)
    ended = 0
    for t in range(steps):
        oa, ra, da, sa = a.step(acts[t])
        oc, rc, dc, sc = c.step(acts[t])
        torch.cuda.synchronize()
        assert torch.equal(oa, oc), f"step {t}: obs differs"
        assert torch.equal(ra, rc) and torch.equal(da, dc), f"step {t}: reward / done differ"
        assert_same_state(sa, sc, f"step {t}")
        ended += int(da.sum())
    assert ended >= n, f"only {ended} episodes ended"
    a.check()
    c.check()
    a.close()
    c.close()


def test_wrappers_reach_terminal_obs(torch_cuda):
    from gym_duckietown_b200 import wrappers as Wr
    env = make_env(4, auto_reset=True, terminal_obs=True)
    w = Wr.PyTorchObsWrapper(env)
    assert w.terminal_obs is env.terminal_obs and tuple(env.terminal_obs.shape) == (4, 3, W, H)
    env.close()


# ---------------------------------------------------------------------------------------------- edges
def test_step_where_nothing_ends(torch_cuda):
    torch = torch_cuda
    n = 32
    a = make_env(n, "loop_obstacles", auto_reset=True, terminal_obs=True)
    c = make_env(n, "loop_obstacles", auto_reset=True)
    a.reset()
    c.reset()
    a.terminal_obs.fill_(77)
    still = torch.zeros((n, 2), device="cuda")
    for t in range(3):
        oa, _, da, _ = a.step(still)
        oc, _, dc, _ = c.step(still)
        torch.cuda.synchronize()
        assert not bool(da.any()) and not bool(dc.any())
        assert torch.equal(oa, oc), f"step {t}: obs differs"
        assert bool((a.terminal_obs == 77).all()), f"step {t}: terminal_obs was written"
    a.close()
    c.close()


def test_every_env_ends_every_step(torch_cuda):
    torch = torch_cuda
    n, steps = 40, 6
    a = make_env(n, "loop_obstacles", max_steps=1, auto_reset=True, terminal_obs=True)
    b = make_env(n, "loop_obstacles", max_steps=1)
    a.reset()
    b.reset()
    acts = forward_actions(torch, steps, n, seed=9)
    for t in range(steps):
        a.terminal_obs.fill_(77)
        _, ra, da, _ = a.step(acts[t])
        ob, rb, db, _ = b.step(acts[t])
        torch.cuda.synchronize()
        assert bool(da.all()) and torch.equal(da, db) and torch.equal(ra, rb)
        assert torch.equal(a.terminal_obs, ob), f"step {t}: terminal frames differ"
        b.reset(mask=db)
        torch.cuda.synchronize()
        assert torch.equal(a.obs, b.obs), f"step {t}: first frames differ"
    a.close()
    b.close()


@pytest.mark.parametrize("fmt", [("hwc", "uint8"), ("cwh", "float32")])
def test_rows_not_done_keep_their_sentinel(torch_cuda, fmt):
    torch = torch_cuda
    n, steps = 48, 30
    a = make_env(n, "loop_obstacles", max_steps=9, auto_reset=True, terminal_obs=True)
    b = make_env(n, "loop_obstacles", max_steps=9)
    for e in (a, b):
        e.set_output_format(obs_layout=fmt[0], obs_dtype=fmt[1])
        e.reset()
    acts = forward_actions(torch, steps, n, seed=13)
    half = (torch.arange(n, device="cuda") % 2) == 0
    some = 0
    for t in range(steps):
        if t == 4:   # restart every other env: from here on their max_steps endings fall between the others'
            a.reset(mask=half)
            b.reset(mask=half)
        a.terminal_obs.fill_(0.5 if fmt[1] == "float32" else 201)
        sentinel = a.terminal_obs.clone()
        _, _, da, _ = a.step(acts[t])
        ob, _, db, _ = b.step(acts[t])
        torch.cuda.synchronize()
        assert torch.equal(a.terminal_obs[~da], sentinel[~da]), f"step {t}: a row that did not end was written"
        assert torch.equal(a.terminal_obs[da], ob[db]), f"step {t}: terminal frames differ"
        some += int(0 < int(da.sum()) < n)
        b.reset(mask=db)
    assert some >= 3, "too few steps with a mix of ended and running envs"
    a.close()
    b.close()


def test_render_off_still_respawns(torch_cuda):
    torch = torch_cuda
    n, steps = 32, 20
    a = make_env(n, max_steps=5, auto_reset=True, terminal_obs=True)
    c = make_env(n, max_steps=5, auto_reset=True)
    a.reset()
    c.reset()
    a.terminal_obs.fill_(9)
    acts = forward_actions(torch, steps, n, seed=2)
    for t in range(steps):
        _, ra, da, sa = a.step(acts[t], render=False)
        _, rc, dc, sc = c.step(acts[t], render=False)
        torch.cuda.synchronize()
        assert torch.equal(ra, rc) and torch.equal(da, dc)
        assert_same_state(sa, sc, f"step {t}")
    assert bool((a.terminal_obs == 9).all())
    a.close()
    c.close()


# ------------------------------------------------------------------------------------ large batch and refusals
def test_4096_envs_repeatable(torch_cuda):
    torch = torch_cuda
    n, steps = 4096, 100
    runs = [make_env(n, "small_loop", max_steps=40, auto_reset=True, terminal_obs=True, seed=1) for _ in range(2)]
    for e in runs:
        e.reset()
        e.terminal_obs.zero_()
    g = torch.Generator(device="cuda").manual_seed(0)
    ended = 0
    for t in range(steps):
        act = torch.rand((n, 2), device="cuda", generator=g) * 2 - 1
        out = [e.step(act) for e in runs]
        torch.cuda.synchronize()
        assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])
        assert torch.equal(runs[0].terminal_obs, runs[1].terminal_obs), f"step {t}: terminal frames differ"
        ended += int(out[0][2].sum())
    assert ended >= 2 * n, ended
    for e in runs:
        e.check()   # no render ran out of frame memory
        e.close()


def test_refusals(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200.dist import FusedObsGather
    with pytest.raises(ValueError):
        make_env(4, terminal_obs=True)                       # no auto_reset
    plain = make_env(4)
    plain.reset()
    act = torch.zeros((4, 2), device="cuda")
    with pytest.raises(L.DtsError, match="AUTO_RESET"):
        plain.sim.step_terminal(act.data_ptr(), plain.obs.data_ptr(), torch.empty_like(plain.obs).data_ptr(),
                                plain.reward.data_ptr(), plain._done_u8.data_ptr(), plain._stream())
    plain.close()
    env = make_env(4, auto_reset=True, terminal_obs=True)
    env.reset()
    with pytest.raises(L.DtsError, match="obs_dev"):
        env.sim.step_terminal(act.data_ptr(), env.obs.data_ptr(), env.obs.data_ptr(), env.reward.data_ptr(),
                              env._done_u8.data_ptr(), env._stream())
    g = FusedObsGather(env, 0, 1)
    g.arm()
    with pytest.raises(L.DtsError, match="gather"):
        env.step(act)
    torch.cuda.synchronize()
    assert float(g.gathered.float().abs().sum()) == 0.0      # the refused step wrote nothing there
    env.close()
