"""Snapshots of the envs' simulator state (dts_save_state / dts_load_state, BatchedDuckietownEnv.save_state /
load_state / copy_envs / state_dict).

Every comparison is bit for bit:
  - resume in place: run, save, run on with resets of both kinds (invalid pose and max_steps) inside the window, load,
    replay the same actions: every step's obs, reward, done, terminal frames, state arrays, device streams, obstacles
    of every map and render record are those of the first run;
  - resume in a new env: state_dict -> torch.save -> torch.load -> load_state_dict into a fresh env with the same
    keywords, which then continues exactly as the original;
  - copy_envs: copied envs step as their sources do, the others as in a run without the copy;
  - a masked load leaves the unmasked envs as they were; render_obs straight after a load draws the saved state;
  - refusals (other maps, a map uploaded since, wrong shape / dtype / device) raise and change nothing; a record naming
    an empty map slot is not loaded and stops the next step;
  - Simulator.render("rgb_array") through a snapshot equals an 800x600 env that took the same actions.
"""
import io

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H = 160, 120
N = 32


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def make_env(n, maps="small_loop", **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=W, camera_height=H, domain_rand=False, seed=11)
    args.update(kw)
    return BatchedDuckietownEnv(n, maps, **args)


def forward_actions(torch, steps, n, seed=3):
    """Random actions biased forward: velocity in [0.2, 1], steering in [-1, 1], so that some envs leave the road."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.rand((steps, n, 2), device="cuda", generator=g)
    a[..., 0] = 0.2 + 0.8 * a[..., 0]
    a[..., 1] = a[..., 1] * 2 - 1
    return a


def mixed_actions(torch, steps, n, seed=3):
    """Even envs drive straight at full speed and leave the road (invalid pose); odd envs creep and stay on it until
    max_steps."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.rand((steps, n, 2), device="cuda", generator=g)
    a[..., 0] = 0.05 + 0.15 * a[..., 0]
    a[..., 1] = 0.2 * a[..., 1] - 0.1
    a[:, ::2, 0], a[:, ::2, 1] = 1.0, 0.0
    return a


def step(env, act):
    """One step; under host resets the envs that ended are reset (the reference loop).  Returns what it produced."""
    obs, rew, done, _ = env.step(act)
    out = dict(obs=obs.clone(), reward=rew.clone(), done=done.clone(), done_code=env.state["done_code"].clone())
    if env.terminal_obs is not None:
        out["terminal"] = env.terminal_obs[done].clone()
    if not env.device_reset and bool(done.any()):
        env.reset(mask=done)
        out["obs_after_reset"] = env.obs.clone()
    return out


def full_state(env):
    """Everything of the env's state that can be read from outside: state arrays, device streams, every map's
    obstacles, every env's render record."""
    import torch
    torch.cuda.synchronize()
    st = {k: v.cpu().numpy().copy() for k, v in env.state.items()}
    st["streams"] = np.array([[s["state"]["state"], s["state"]["inc"], s["has_uint32"], s["uinteger"]]
                              for s in env.sim.debug_streams()], dtype=object)
    for m in range(len(env.maps)):
        arr, nd = env.sim.dyn_state(m)
        if nd:
            st[f"dyn{m}"] = torch.as_tensor(arr, device=env.device).cpu().numpy().reshape(-1, env.num_envs).copy()
    eps = [env.sim.debug_episode(e) for e in range(env.num_envs)]
    for k in eps[0]:
        st["ep_" + k] = np.stack([np.asarray(ep[k]) for ep in eps])
    return st


def env_rows(st, envs):
    """The rows of a full_state() of the listed envs (env axis last for the obstacles)."""
    return {k: (v[:, envs] if k.startswith("dyn") else v[envs]) for k, v in st.items()}


def assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        if isinstance(a[k], np.ndarray) and a[k].dtype != object:
            assert np.array_equal(a[k], b[k], equal_nan=True), f"{what}: {k} differs"
        else:
            assert np.array_equal(a[k], b[k]), f"{what}: {k} differs"


def assert_same_outputs(a, b, what):
    assert a.keys() == b.keys(), f"{what}: {sorted(a)} vs {sorted(b)}"
    for k in a:
        assert a[k].shape == b[k].shape and bool((a[k] == b[k]).all()), f"{what}: {k} differs"


def run(env, acts, t0, t1):
    """Steps t0 .. t1-1; per step the outputs and the full state after it."""
    trace = []
    for t in range(t0, t1):
        trace.append((step(env, acts[t]), full_state(env)))
    return trace


def compare_traces(a, b, what):
    assert len(a) == len(b)
    for t, ((oa, sa), (ob, sb)) in enumerate(zip(a, b)):
        assert_same_outputs(oa, ob, f"{what} step {t}")
        assert_same(sa, sb, f"{what} step {t}")


DEV = dict(device_reset=True, auto_reset=True)
RESUME_CASES = {
    "small_loop_host": dict(maps="small_loop"),
    "loop_obstacles_terminal": dict(maps="loop_obstacles", terminal_obs=True, **DEV),
    "loop_pedestrians": dict(maps="loop_pedestrians", domain_rand=True, **DEV),
    "loop_dyn_duckiebots": dict(maps="loop_dyn_duckiebots", **DEV),
    "domain_dynamics_rand": dict(maps="loop_obstacles", domain_rand=True, dynamics_rand=True, **DEV),
    "cycle_maps": dict(maps=["small_loop", "loop_dyn_duckiebots"], cycle_maps=True, **DEV),
    "randomize_maps": dict(maps=["loop_pedestrians", "loop_dyn_duckiebots"], randomize_maps_on_reset=True, **DEV),
    "distortion": dict(maps="small_loop", distortion=True, **DEV),
}
T1, T2 = 20, 50


@pytest.mark.parametrize("case", sorted(RESUME_CASES))
def test_resume_in_place(torch_cuda, case):
    torch = torch_cuda
    kw = dict(RESUME_CASES[case])
    env = make_env(N, kw.pop("maps"), max_steps=40, **kw)
    env.reset()
    acts = mixed_actions(torch, T1 + T2, N)
    for t in range(T1):
        step(env, acts[t])
    host = not env.device_reset
    saved = env.state_dict() if host else env.save_state()   # host resets: the sampler's streams come along
    at_save = full_state(env)
    first = run(env, acts, T1, T1 + T2)
    done_any = torch.stack([o["done"] for o, _ in first]).any(0)
    assert bool(done_any.any()), "no episode ended inside the replayed window"
    codes = torch.cat([o["done_code"][o["done"]] for o, _ in first]).unique().tolist()
    assert set(codes) == {1, 2}, f"episodes must end both ways (invalid pose, max_steps): {codes}"
    if host:
        env.load_state_dict(saved)
    else:
        env.load_state(saved)
    assert_same(full_state(env), at_save, "state straight after the load")
    compare_traces(first, run(env, acts, T1, T1 + T2), case)


@pytest.mark.parametrize("case", ["device_reset", "host_reset"])
def test_resume_in_fresh_env(torch_cuda, case):
    torch = torch_cuda
    if case == "device_reset":
        kw = dict(maps="loop_dyn_duckiebots", domain_rand=True, terminal_obs=True, **DEV)
    else:
        kw = dict(maps=["small_loop", "loop_pedestrians"], randomize_maps_on_reset=True)
    maps = kw.pop("maps")
    a = make_env(N, maps, max_steps=9, **kw)
    a.reset()
    acts = forward_actions(torch, T1 + T2, N, seed=5)
    for t in range(T1):
        step(a, acts[t])
    buf = io.BytesIO()
    torch.save(a.state_dict(), buf)
    buf.seek(0)
    b = make_env(N, maps, max_steps=9, **kw)
    b.load_state_dict(torch.load(buf))
    assert_same(full_state(b), full_state(a), "fresh env after load_state_dict")
    compare_traces(run(a, acts, T1, T1 + T2), run(b, acts, T1, T1 + T2), case)


COPY_SOURCES = {
    "permutation": lambda g: np.random.default_rng(g).permutation(N),
    "many_to_one": lambda g: np.array([-1 if e % 5 == 0 else (3 if e < N // 2 else 17) for e in range(N)]),
}


@pytest.mark.parametrize("reset", ["device", "host"])
@pytest.mark.parametrize("sources", sorted(COPY_SOURCES))
def test_copy_envs(torch_cuda, reset, sources):
    torch = torch_cuda
    kw = dict(maps="loop_dyn_duckiebots", domain_rand=True, **DEV) if reset == "device" else \
        dict(maps=["small_loop", "loop_pedestrians"], cycle_maps=True)
    maps = kw.pop("maps")
    a = make_env(N, maps, max_steps=9, **kw)    # gets the copy
    b = make_env(N, maps, max_steps=9, **kw)    # runs on without it
    a.reset()
    b.reset()
    acts = forward_actions(torch, T1 + T2, N, seed=9)
    for t in range(T1):
        step(a, acts[t])
        step(b, acts[t])
    src = COPY_SOURCES[sources](1)
    a.copy_envs(torch.as_tensor(src))
    who = np.where(src >= 0, src, np.arange(N))     # the env of b that env e of a now is
    who_d = torch.as_tensor(who, device="cuda")
    assert_same(full_state(a), env_rows(full_state(b), who), "straight after copy_envs")
    for t in range(T1, T1 + T2):
        oa = step(a, acts[t][who_d])
        ob = step(b, acts[t])
        sa, sb = full_state(a), full_state(b)
        assert torch.equal(oa["obs"], ob["obs"][who_d]), f"step {t}: obs"
        assert torch.equal(oa["reward"], ob["reward"][who_d]) and torch.equal(oa["done"], ob["done"][who_d]), f"step {t}"
        if "obs_after_reset" in oa or "obs_after_reset" in ob:
            assert torch.equal(a.obs, b.obs[who_d]), f"step {t}: obs after the host reset"
        assert_same(sa, env_rows(sb, who), f"step {t}")


def test_masked_load_leaves_unmasked_envs(torch_cuda):
    torch = torch_cuda
    env = make_env(N, ["loop_dyn_duckiebots", "loop_pedestrians"], max_steps=9, randomize_maps_on_reset=True,
                   domain_rand=True, terminal_obs=True, **DEV)
    env.reset()
    acts = forward_actions(torch, 2 * T1, N, seed=13)
    for t in range(T1):
        step(env, acts[t])
    old = env.save_state()
    old_state = full_state(env)
    for t in range(T1, 2 * T1):
        step(env, acts[t])
    torch.cuda.synchronize()
    now = env.save_state()
    now_state = full_state(env)
    obs, term = env.obs.clone(), env.terminal_obs.clone()
    mask = torch.zeros(N, dtype=torch.bool, device="cuda")
    mask[::3] = True
    env.load_state(old, mask=mask)
    after = full_state(env)
    m = mask.cpu().numpy()
    assert_same(env_rows(after, np.flatnonzero(~m)), env_rows(now_state, np.flatnonzero(~m)), "unmasked envs")
    assert_same(env_rows(after, np.flatnonzero(m)), env_rows(old_state, np.flatnonzero(m)), "masked envs")
    assert torch.equal(env.save_state(), torch.where(mask[:, None], old, now)), "records after the masked load"
    assert torch.equal(env.obs, obs) and torch.equal(env.terminal_obs, term), "a load rewrites no output buffer"
    # and the unmasked envs step on as they would have: against a twin that never loaded
    twin = make_env(N, ["loop_dyn_duckiebots", "loop_pedestrians"], max_steps=9, randomize_maps_on_reset=True,
                    domain_rand=True, terminal_obs=True, **DEV)
    twin.load_state(now)
    keep = torch.nonzero(~mask).flatten()
    for t in range(10):
        oa, ob = step(env, acts[t]), step(twin, acts[t])
        for k in ("obs", "reward", "done"):
            assert torch.equal(oa[k][keep], ob[k][keep]), f"step {t}: {k} of an unmasked env"


@pytest.mark.parametrize("mode", ["plain", "segment", "top_down"])
def test_render_straight_after_load(torch_cuda, mode):
    torch = torch_cuda
    env = make_env(N, "loop_dyn_duckiebots", domain_rand=True, max_steps=30, **DEV)
    env.reset()
    acts = forward_actions(torch, 2 * T1, N, seed=17)
    for t in range(T1):
        step(env, acts[t])
    kw = dict(segment=mode == "segment", top_down=mode == "top_down")
    want = env.render_obs(out=torch.empty_like(env.obs), **kw).clone()
    rec = env.save_state()
    for t in range(T1, 2 * T1):
        step(env, acts[t])
    env.load_state(rec)
    got = env.render_obs(out=torch.empty_like(env.obs), **kw)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_refusals_change_nothing(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200.maps import load_map
    env = make_env(N, "small_loop", max_steps=30, **DEV)
    env.reset()
    acts = forward_actions(torch, 5, N)
    for t in range(5):
        step(env, acts[t])
    rec = env.save_state()
    other = make_env(N, "loop_obstacles", **DEV)   # another map in slot 0, a record of the same size
    assert other.save_state().shape == rec.shape and other.state_fingerprint != env.state_fingerprint
    step(env, acts[0])
    before = full_state(env)
    rec_now = env.save_state()
    bad = [
        dict(records=rec, fingerprint=other.state_fingerprint),
        dict(records=rec[:, :-16].contiguous(), fingerprint=rec.fingerprint),
        dict(records=rec.view(torch.int8), fingerprint=rec.fingerprint),
        dict(records=rec.cpu(), fingerprint=rec.fingerprint),
        dict(records=rec.clone()),   # no fingerprint attached
    ]
    for b in bad:
        with pytest.raises((L.DtsError, ValueError)):
            env.load_state(b["records"], fingerprint=b.get("fingerprint"))
    assert_same(full_state(env), before, "after the refused loads")
    # the same content uploaded again keeps the fingerprint; another map in the slot changes it, and records saved
    # before that upload are refused
    fp = env.state_fingerprint
    env.sim.upload_map(0, load_map("small_loop"))
    assert env.state_fingerprint == fp
    env.sim.upload_map(0, load_map("loop_obstacles"))
    assert env.state_fingerprint == other.state_fingerprint != fp
    after_upload = full_state(env)
    with pytest.raises(L.DtsError, match="fingerprint"):
        env.load_state(rec_now)
    assert_same(full_state(env), after_upload, "after the refused load of records from before the upload")


def test_record_naming_an_empty_slot_is_not_loaded(torch_cuda):
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L
    env = make_env(N, ["small_loop", "loop_obstacles"], randomize_maps_on_reset=True, **DEV)
    env.reset()
    torch.cuda.synchronize()
    mids = env.state["map_id"].cpu().numpy()
    assert 0 < mids.sum() < N, "both maps should be in use"
    rec = env.save_state()
    # the record's map id: the only 4-byte column that holds every env's map id
    words = rec.view(torch.int32).cpu().numpy()
    cols = [c for c in range(words.shape[1]) if np.array_equal(words[:, c], mids)]
    assert len(cols) == 1, cols
    before = full_state(env)
    edited = rec.clone()
    edited.view(torch.int32)[5, cols[0]] = 2        # max_maps = 2: slot 2 does not exist
    edited.view(torch.int32)[9, cols[0]] = -1
    env.load_state(edited, fingerprint=rec.fingerprint)
    torch.cuda.synchronize()
    assert env.sim.status() & 2
    after = full_state(env)
    assert_same(env_rows(after, [5, 9]), env_rows(before, [5, 9]), "the refused envs keep their state")
    with pytest.raises(L.DtsError, match="map_id"):
        env.step(forward_actions(torch, 1, N)[0])
    with pytest.raises(L.DtsError, match="map_id"):
        env.render_obs()


def test_human_view_is_a_snapshot(torch_cuda):
    """Simulator.render('rgb_array') builds its 800x600 view from this env's snapshot: it equals the observation of an
    800x600 env with the same seed and keywords that took the same actions, obstacles included."""
    torch = torch_cuda
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.simulator import Simulator
    sim = Simulator("loop_dyn_duckiebots", camera_width=W, camera_height=H, seed=5, domain_rand=True)
    big = BatchedDuckietownEnv(1, "loop_dyn_duckiebots", camera_width=800, camera_height=600, seed=5, domain_rand=True,
                               action_mode="pwm")
    big.reset()
    g = np.random.default_rng(2)
    for t in range(24):
        a = np.array([0.3 + 0.5 * g.random(), 0.3 + 0.5 * g.random()], np.float32)
        sim.step(a)
        big.step(torch.from_numpy(a[None]).cuda())
        if t % 6 == 5:
            view = sim.render("rgb_array")
            assert view.shape == (600, 800, 3)
            assert np.array_equal(view, big.obs[0].cpu().numpy()), f"step {t}"
    _, nd = big.sim.dyn_state(0)
    assert nd > 0
    sim.close()
    big.close()
