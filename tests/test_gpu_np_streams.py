"""The device's numpy-compatible random streams (np_random.cuh) against numpy itself, draw for draw and bit for bit.

Every device reset, auto-reset and domain-randomised obstacle walk draws from the env's `NpStream`, a restatement of
numpy's `Generator(PCG64)`.  Here each of its methods runs through `dts_debug_draw` at the ranges the product uses and
at the edges of numpy's branches (Lemire rejection, the 32-bit / raw / 64-bit integer regimes, the ziggurat's tail),
and the device resets and walks are replayed on the host with numpy.  Every comparison is exact, and every case also
compares the stream state afterwards (state, inc, has_uint32, uinteger) with `Generator.bit_generator.state`."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ZIGGURAT_R = 3.6541528853610087963519472518   # the ziggurat's last layer: beyond it a draw came from the tail branch


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def generators(seeds):
    return [np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(s)))) for s in seeds]


def bare_sim(n):
    """A handle with no map: enough for seed_streams / debug_draw / debug_streams."""
    from gym_duckietown_b200 import lib as L
    return L.Sim(L.default_config(num_envs=n, cam_width=16, cam_height=16))


def device_draws(torch, sim, ops):
    from gym_duckietown_b200 import lib as L   # noqa: F401
    total = sum(int(op[1]) for op in ops)
    out = torch.empty((sim.cfg.num_envs, total), dtype=torch.int64, device="cuda")
    sim.debug_draw(ops, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return out.cpu().numpy().view(np.uint64)


def host_draws(g, ops):
    """What numpy draws for the program, as the device writes it: u64 bits of each value."""
    from gym_duckietown_b200 import lib as L
    parts = []
    for kind, count, a, b in ops:
        if kind == L.DRAW_NEXT64:
            v = np.asarray(g.bit_generator.random_raw(count), np.uint64)
        elif kind == L.DRAW_NEXT32:
            v = g.integers(0, 2 ** 32, size=count, dtype=np.uint32).astype(np.uint64)
        elif kind == L.DRAW_UNIFORM:
            v = g.uniform(a, b, size=count).view(np.uint64)
        elif kind == L.DRAW_INTEGERS:
            v = g.integers(a, b, size=count).astype(np.int64).view(np.uint64)
        else:
            v = g.normal(a, b, size=count).view(np.uint64)
        parts.append(v)
    return np.concatenate(parts)


def assert_streams_equal(sim, gens, what=""):
    dev = sim.debug_streams()
    bad = [e for e, g in enumerate(gens) if dev[e] != g.bit_generator.state]
    assert not bad, (what, len(bad), bad[:4], [(dev[e], gens[e].bit_generator.state) for e in bad[:1]])


def run_and_compare(torch, sim, gens, ops, what):
    dev = device_draws(torch, sim, ops)
    host = np.stack([host_draws(g, ops) for g in gens])
    bad = np.flatnonzero((dev != host).any(axis=1))
    assert not len(bad), (what, len(bad), bad[:4], np.flatnonzero(dev[bad[0]] != host[bad[0]])[:8])
    assert_streams_equal(sim, gens, what)
    return dev


def seeded(torch, n, seed0, odd_prefix=False):
    """n device streams equal to numpy Generators seeded seed0 .. seed0 + n - 1; odd_prefix: each first draws an odd
    number of 32-bit values on the host, so every stream is uploaded with its cached half pending (has_uint32 = 1)."""
    gens = generators(range(seed0, seed0 + n))
    if odd_prefix:
        rng = np.random.default_rng(seed0)
        for g in gens:
            g.integers(0, 2 ** 32, size=2 * int(rng.integers(0, 4)) + 1, dtype=np.uint32)
        assert all(g.bit_generator.state["has_uint32"] == 1 for g in gens)
    sim = bare_sim(n)
    sim.seed_streams(gens)
    assert_streams_equal(sim, gens, "upload")
    return sim, gens


# ------------------------------------------------------------------------------------------------------ the methods
def test_raw_draws(torch_cuda):
    """next64 = random_raw(), next32 = integers(0, 2**32, dtype=uint32): odd counts leave the cached half pending
    across the 64-bit draws that follow."""
    from gym_duckietown_b200 import lib as L
    sim, gens = seeded(torch_cuda, 4096, 11)
    ops = [(L.DRAW_NEXT64, 64, 0, 0), (L.DRAW_NEXT32, 33, 0, 0), (L.DRAW_NEXT64, 5, 0, 0), (L.DRAW_NEXT32, 1, 0, 0),
           (L.DRAW_NEXT64, 1, 0, 0), (L.DRAW_NEXT32, 3, 0, 0)]
    run_and_compare(torch_cuda, sim, gens, ops, "raw")
    assert all(g.bit_generator.state["has_uint32"] == 1 for g in gens)   # the program ends with a half cached
    sim.close()


def test_uniform_at_the_products_ranges(torch_cuda):
    """Spawn tiles (ti, ti + 1) and the angle (0, 2 pi), the _perturb ranges 1 +- s, the default table's ranges, the
    distractor triangles' and a negative range.  (The spawn loop's `* tile_size` is checked by the reset cases.)"""
    from gym_duckietown_b200 import lib as L
    sim, gens = seeded(torch_cuda, 4096, 20_000)
    ranges = [(float(t), float(t + 1)) for t in range(8)] + [(0.0, 2 * math.pi)]
    ranges += [(1 - s, 1 + s) for s in (0.1, 0.2, 0.3, 0.4, 0.99)]
    ranges += [(0.8, 1.2), (0.92, 1.08), (-0.005, 0.005), (-150.0, 150.0), (170.0, 220.0)]
    ranges += [(-20.0, 20.0), (-0.6, -0.3), (0.0, 0.9), (-7.25, -3.5)]
    ops = [(L.DRAW_UNIFORM, 3 + k % 4, a, b) for k, (a, b) in enumerate(ranges)]
    run_and_compare(torch_cuda, sim, gens, ops, "uniform")
    sim.close()


def lemire_rejections(states, skip32, lo, hi, count):
    """How many draws numpy's Lemire loop rejects for `count` integers(lo, hi) after `skip32` 32-bit draws, summed over
    the generator states."""
    rng = hi - 1 - lo
    rej = 0
    for st in states:
        g = np.random.Generator(np.random.PCG64())
        g.bit_generator.state = st
        g.integers(0, 2 ** 32, size=skip32, dtype=np.uint32)
        if rng < 2 ** 32 - 1:
            excl = rng + 1
            thr = (2 ** 32 - 1 - rng) % excl
            u = g.integers(0, 2 ** 32, size=4 * count + 64, dtype=np.uint32).astype(np.uint64)
            ok = ((u * np.uint64(excl)) & np.uint64(0xFFFFFFFF)) >= np.uint64(thr)
        else:
            excl = rng + 1
            thr = (2 ** 64 - 1 - rng) % excl
            u = g.bit_generator.random_raw(4 * count + 64)
            ok = np.array([(int(v) * excl) % 2 ** 64 >= thr for v in u])
        rej += int(np.flatnonzero(ok)[count - 1]) + 1 - count
    return rej


def test_integers_every_regime(torch_cuda):
    """integers(lo, hi) at the product's ranges (1, 2, 4, 17, every map's drivable-tile count), where the 32-bit Lemire
    loop rejects a quarter of the draws (3 * 2**29), around 2**31 and 2**32 (the raw 32-bit draw at 2**32), and on
    numpy's 64-bit path (2**32 + 1, 2**33, 3 * 2**61, whose loop also rejects a quarter), with negative lows."""
    from gym_duckietown_b200 import lib as L, maps
    torch = torch_cuda
    sim, gens = seeded(torch, 4096, 30_000)
    n_drv = sorted({len(maps.load_map(m).drivable_tiles) for m in ("small_loop", "loop_obstacles", "udem1",
                                                                  "loop_pedestrians", "loop_dyn_duckiebots")})
    his = [1, 2, 4, 17] + n_drv + [3 * 2 ** 29, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1,
                                   2 ** 33, 3 * 2 ** 61]
    bounds = [(0, h) for h in his] + [(-5, 12), (-(2 ** 31), 2 ** 31), (-(2 ** 40), 2 ** 40 + 3), (-(2 ** 62), 2 ** 62)]
    rejected = {}
    for k, (lo, hi) in enumerate(bounds):   # one program per range, so that a failure names its range
        ops = [(L.DRAW_NEXT32, 1 + k % 2, 0, 0), (L.DRAW_INTEGERS, 7, lo, hi)]
        starts = [g.bit_generator.state for g in gens]
        dev = run_and_compare(torch, sim, gens, ops, f"integers({lo}, {hi})")
        if hi in (3 * 2 ** 29, 3 * 2 ** 61):
            rejected[hi] = lemire_rejections(starts, 1 + k % 2, lo, hi, 7)
        vals = dev[:, -7:].view(np.int64)
        assert vals.min() >= lo and vals.max() < hi
        if hi == 1:
            assert np.all(vals == 0)
    print(f"\nLemire rejections reached: 32-bit loop {rejected[3 * 2 ** 29]}, 64-bit loop {rejected[3 * 2 ** 61]} "
          f"of {4096 * 7} draws each")
    assert rejected[3 * 2 ** 29] > 4096 * 7 // 8 and rejected[3 * 2 ** 61] > 4096 * 7 // 8
    sim.close()


def test_normal_reaches_the_ziggurat_tail(torch_cuda):
    """2**25 and more normal draws at (0, 1), the trim's (0, 0.02) and the walk speed's (0.02, 0.005), in chunks: the
    tail branch (log1p, ~1 in 3,900 draws) and the wedges (exp) are taken thousands of times."""
    from gym_duckietown_b200 import lib as L
    torch = torch_cuda
    n, per = 4096, 1024
    sim, gens = seeded(torch, n, 40_000)
    params = [(0.0, 1.0), (0.0, 0.02), (0.02, 0.005)]
    tail = drawn = 0
    for chunk in range(3):
        ops = [(L.DRAW_NEXT32, 1, 0, 0)] + [(L.DRAW_NORMAL, per, a, b) for a, b in params]
        dev = run_and_compare(torch, sim, gens, ops, f"normal chunk {chunk}")
        for j, (loc, scale) in enumerate(params):
            x = dev[:, 1 + j * per:1 + (j + 1) * per].copy().view(np.float64)
            tail += int((np.abs(x - loc) / scale > ZIGGURAT_R).sum())
            drawn += x.size
    print(f"\nnormal: {drawn} draws, {tail} beyond the ziggurat's R = {ZIGGURAT_R} (tail branch)")
    assert drawn >= 2 ** 25 and tail >= 4000
    sim.close()


def test_interleaved_programs_from_a_pending_half(torch_cuda):
    """Random mixes of all five kinds, 4,096 ops each, from streams uploaded with numpy's cached 32-bit half pending:
    the half must survive the upload, the 64-bit draws in between, and come out where numpy takes it."""
    from gym_duckietown_b200 import lib as L
    torch = torch_cuda
    sim, gens = seeded(torch, 128, 50_000, odd_prefix=True)
    rng = np.random.default_rng(5)
    int_bounds = [(0, 2), (0, 4), (0, 17), (0, 18), (0, 3 * 2 ** 29), (0, 2 ** 32), (0, 2 ** 33), (-9, 3),
                  (0, 3 * 2 ** 61), (0, 2 ** 31 + 1)]
    uniform_ranges = [(0.0, 1.0), (0.7, 1.3), (0.0, 0.9), (-150.0, 150.0), (0.0, 2 * math.pi)]
    normal_params = [(0.0, 1.0), (0.02, 0.005), (0.0, 0.02)]
    for prog in range(2):
        ops = []
        for kind in rng.integers(0, 5, size=4096):
            count = int(rng.integers(1, 4))
            if kind == L.DRAW_INTEGERS:
                lo, hi = int_bounds[rng.integers(len(int_bounds))]
                ops.append((L.DRAW_INTEGERS, count, lo, hi))
            elif kind in (L.DRAW_UNIFORM, L.DRAW_NORMAL):
                table = uniform_ranges if kind == L.DRAW_UNIFORM else normal_params
                a, b = table[rng.integers(len(table))]
                ops.append((int(kind), count, a, b))
            else:
                ops.append((int(kind), count, 0, 0))
        run_and_compare(torch, sim, gens, ops, f"program {prog}")
    sim.close()


def test_refuses_empty_integer_ranges(torch_cuda):
    """Generator.integers raises on low >= high: so do dts_create for a randomization table's int key and
    dts_debug_draw, instead of drawing garbage."""
    from gym_duckietown_b200 import lib as L
    from gym_duckietown_b200.episode import DEFAULT_DR_CONFIG
    for low, high in ((4, 4), (5, 2), (0, 2.0 ** 64)):
        cfg = dict(DEFAULT_DR_CONFIG, horz_mode={"type": "int", "low": low, "high": high})
        c = L.default_config(num_envs=2, cam_width=16, cam_height=16, dr_ops=L.dr_ops_from_config(cfg))
        with pytest.raises(L.DtsError, match="dts_dr_op 4: int draw needs low < high"):
            L.Sim(c)
    sim = bare_sim(2)
    out = torch_cuda.zeros((2, 1), dtype=torch_cuda.int64, device="cuda")
    with pytest.raises(L.DtsError, match="integers needs lo < hi"):
        sim.debug_draw([(L.DRAW_INTEGERS, 1, 3, 3)], out.data_ptr())
    sim.close()


# ------------------------------------------------------------------------------------------ device resets at scale
def oracle_spawn_query(md):
    """The spawn predicates from the C oracle (_valid_pose(1.3), get_lane_pos2) and _inconvenient_spawn in numpy."""
    import oracle as orc
    om = orc.OracleMap(md)
    pos = np.array([o.pos for o in md.objects], np.float64).reshape(-1, 3)
    rad = np.array([max(o.max_coords) * 0.5 * o.scale + 0.25 for o in md.objects])

    def query(x, z, a, safety, hidden):
        n = len(x)
        outd, outi = np.full((n, 4), np.nan), np.zeros((n, 8), np.int32)
        for q in range(n):
            o = om.done_reward(x[q], z[q], a[q], 0)
            outd[q] = (o.lane_dist, o.lane_dot, o.lane_angle, o.prox)
            outi[q, 0] = om.valid_pose(x[q], z[q], a[q], safety)
            outi[q, 3] = o.in_lane
        if len(pos):
            d = np.sqrt((pos[None, :, 0] - x[:, None]) ** 2 + (pos[None, :, 1] - 0.0) ** 2 + (pos[None, :, 2] - z[:, None]) ** 2)
            oi = np.arange(len(pos))
            vis = ((hidden[:, oi >> 5] >> (oi & 31)) & 1) == 0
            outi[:, 4] = ((d < rad[None]) & vis).any(axis=1)
        return outd, outi
    return query


RESET_CASES = {
    "small_loop": dict(maps=["small_loop"]),
    "loop_obstacles_dr_notris": dict(maps=["loop_obstacles"], domain_rand=True, num_tris_distractors=0),
    "udem1_dr_dynrand_tris40": dict(maps=["udem1"], domain_rand=True, dynamics_rand=True, num_tris_distractors=40),
    "mixed_random_maps_dr": dict(maps=["small_loop", "loop_obstacles", "udem1"], domain_rand=True,
                                 randomize_maps_on_reset=True),
    "cycle_maps": dict(maps=["small_loop", "loop_obstacles", "udem1"], cycle_maps=True),
    "custom_table": dict(maps=["loop_obstacles"], domain_rand=True, dynamics_rand=True, randomization_config={
        "camera_angle": {"type": "uniform", "low": 0.8, "high": 1.2},
        "camera_fov_y": {"type": "uniform", "low": 0.8, "high": 1.2},
        "camera_height": {"type": "uniform", "low": 0.92, "high": 1.08},
        "camera_noise": {"type": "normal", "loc": 0, "scale": 0.01, "size": 3},
        "horz_mode": {"type": "int", "low": 0, "high": 4},
        "int5": {"type": "int", "low": -3, "high": 9, "size": 5},
        "light_pos": {"type": "uniform", "low": [-150, 170, -150], "high": [150, 220, 150], "size": 3},
        "normal4": {"type": "normal", "loc": 0.5, "scale": 2.0, "size": 4},
        "trim": {"type": "normal", "loc": 0, "scale": 0.02},
        "wide": {"type": "int", "low": 0, "high": 2 ** 33},
    }),
}


@pytest.mark.parametrize("case", list(RESET_CASES))
def test_device_reset_equals_numpy_replay(case, torch_cuda):
    """4096 envs, 3 episodes of dts_reset_random against EpisodeSampler replaying the same resets with numpy: the
    streams afterwards, pose, wheel_dist and the render record must equal what the host drew."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.episode import EpisodeSampler
    kw = dict(RESET_CASES[case])
    names = kw.pop("maps")
    n, seed = 4096, 7000
    mds = [maps.load_map(m) for m in names]
    env = BatchedDuckietownEnv(n, mds, camera_width=32, camera_height=32, seed=seed, device_reset=True,
                               domain_rand=kw.get("domain_rand", False), **{k: v for k, v in kw.items() if k != "domain_rand"})
    host = EpisodeSampler(n, domain_rand=kw.get("domain_rand", False), dynamics_rand=kw.get("dynamics_rand", False),
                          num_tris_distractors=kw.get("num_tris_distractors", 12),
                          randomization_config=kw.get("randomization_config"))
    host.seed([seed + k for k in range(n)])
    queries = [oracle_spawn_query(md) for md in mds]
    map_ids = np.zeros(n, np.int64)
    envs = list(range(n))
    for ep in range(3):
        env.reset(render=False)
        if kw.get("randomize_maps_on_reset"):
            map_ids = np.array([int(host.rngs[e].integers(0, len(mds))) for e in envs])
        elif kw.get("cycle_maps") and ep > 0:
            map_ids = (map_ids + 1) % len(mds)
        want = host.sample(envs, [mds[m] for m in map_ids],
                           lambda k, x, z, a, sf, hid: queries[map_ids[k]](x, z, a, sf, hid))
        assert_streams_equal(env.sim, host.rngs, (case, ep))
        torch.cuda.synchronize()
        st = {k: v.cpu().numpy() for k, v in env.state.items()}
        assert np.array_equal(st["map_id"], map_ids), (case, ep)
        for key in ("pos_x", "pos_z", "angle", "wheel_dist"):
            bad = np.flatnonzero(st[key] != want[key])
            assert not len(bad), (case, ep, key, bad[:4], st[key][bad[:2]], want[key][bad[:2]])
        rec = [env.sim.debug_episode(e) for e in envs]
        for dev_key, host_key in (("cam_height", "cam_height"), ("cam_angle_deg", "cam_angle_deg"),
                                  ("cam_fov_y_deg", "cam_fov_y_deg"), ("cam_noise", "cam_noise"),
                                  ("horizon", "horizon_color"), ("ambient", "light_ambient"), ("diffuse", "light_diffuse"),
                                  ("ground", "ground_color"), ("hidden", "obj_hidden")):
            got = np.array([r[dev_key] for r in rec])
            exp = want[host_key].astype(got.dtype).reshape(got.shape)
            bad = np.flatnonzero((got != exp).reshape(n, -1).any(axis=1))
            assert not len(bad), (case, ep, dev_key, bad[:4], got[bad[:1]], exp[bad[:1]])
        if ep == 0:   # first reset: GL_LIGHT0 captured under the identity modelview, i.e. the drawn position itself
            got = np.array([r["light_eye"] for r in rec])
            assert np.array_equal(got, want["light_pos"].astype(np.float32)), case
    env.close()


# -------------------------------------------------------------------------------------- obstacle walks under DR
def test_domain_rand_walks_draw_what_numpy_draws(torch_cuda):
    """loop_pedestrians under domain_rand, 256 parked envs: every duckie that ends a walk takes v = normal(0.02, 0.005)
    and w = integers(0, 17) from its env's stream in slot order.  The new speed must be -sign(old) |v|, the wait
    3 + w, and the stream afterwards numpy's, step by step until every duckie has ended two walks."""
    from gym_duckietown_b200 import lib as L, maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    torch = torch_cuda
    md = maps.load_map("loop_pedestrians")
    assert all(d.kind == maps.DYN_DUCKIE for d in md.dyn_objects)
    n = 256
    env = BatchedDuckietownEnv(n, md, camera_width=32, camera_height=32, seed=900, domain_rand=True, device_reset=True)
    env.reset(render=False)
    zero = torch.zeros(n, 2, device=env.device)
    ended = np.zeros((len(md.dyn_objects), n), np.int64)
    t = 0
    while ended.min() < 2:
        assert t < 1500, ("some duckie has not ended two walks", t, int(ended.min()))
        before_streams, before = env.sim.debug_streams(), dyn_host(env, torch)
        env.step(zero, render=False)
        after = dyn_host(env, torch)
        gens = []
        for e in range(n):
            g = np.random.Generator(np.random.PCG64())
            g.bit_generator.state = before_streams[e]
            for s in np.flatnonzero((before[L.DYN_ACTIVE, :, e] == 1) & (after[L.DYN_ACTIVE, :, e] == 0)):
                v, w = g.normal(0.02, 0.005), g.integers(0, 17)
                old = before[L.DYN_VEL, s, e]
                assert after[L.DYN_VEL, s, e] == -1 * np.sign(old) * abs(v), (t, e, s)
                assert after[L.DYN_WAIT, s, e] == float(3 + w), (t, e, s)
                ended[s, e] += 1
            gens.append(g)
        assert_streams_equal(env.sim, gens, ("walk step", t))
        t += 1
    print(f"\nwalks: {int(ended.sum())} ended in {t} steps, each duckie of each env at least twice")
    env.close()


def dyn_host(env, torch):
    from gym_duckietown_b200 import lib as L
    arr, nd = env.sim.dyn_state(0)
    return torch.as_tensor(arr, device=env.device).view(L.DYN_FIELDS, nd, env.num_envs).cpu().numpy()


def test_walks_and_auto_reset_share_the_stream(torch_cuda):
    """As above with auto-reset and a short max_steps: where an env also ended, its respawn continues the stream from
    the post-walk state, and EpisodeSampler replays it from there (spawn predicates from dts_query_poses, which sees
    the obstacles where the step left them).  A twin env stepping through dts_step_terminal (respawn in
    k_respawn_ended) must keep streams, obstacles and poses equal to the dts_step one at every step."""
    from gym_duckietown_b200 import lib as L, maps
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    from gym_duckietown_b200.episode import EpisodeSampler
    torch = torch_cuda
    md = maps.load_map("loop_pedestrians")
    n, seed = 256, 1900
    kw = dict(camera_width=32, camera_height=32, seed=seed, domain_rand=True, device_reset=True, auto_reset=True,
              max_steps=90)
    env = BatchedDuckietownEnv(n, md, **kw)
    twin = BatchedDuckietownEnv(n, md, terminal_obs=True, **kw)
    host = EpisodeSampler(n, domain_rand=True)
    env.reset(render=False); twin.reset(render=False)
    host.episodes[:] = 1
    zero = torch.zeros(n, 2, device=env.device)
    walks = resets = 0
    for t in range(700):
        before_streams, before = env.sim.debug_streams(), dyn_host(env, torch)
        _, _, done, _ = env.step(zero, render=False)
        twin.step(zero, render=False)
        done = done.cpu().numpy()
        after = dyn_host(env, torch)
        st = {k: v.cpu().numpy() for k, v in env.state.items()}
        for e in range(n):
            g = np.random.Generator(np.random.PCG64())
            g.bit_generator.state = before_streams[e]
            for s in np.flatnonzero((before[L.DYN_ACTIVE, :, e] == 1) & (after[L.DYN_ACTIVE, :, e] == 0)):
                v, w = g.normal(0.02, 0.005), g.integers(0, 17)
                assert after[L.DYN_VEL, s, e] == -1 * np.sign(before[L.DYN_VEL, s, e]) * abs(v), (t, e, s)
                assert after[L.DYN_WAIT, s, e] == float(3 + w), (t, e, s)
                walks += 1
            host.rngs[e] = g
            if done[e]:
                q = (lambda e_: lambda k, x, z, a, sf, hid: env.sim.query_poses(0, x, z, a, sf, hid, dyn_env=e_))(e)
                want = host.sample([e], [md], q)
                for key in ("pos_x", "pos_z", "angle", "wheel_dist"):
                    assert st[key][e] == want[key][0], (t, e, key)
                resets += 1
        assert_streams_equal(env.sim, host.rngs, ("auto-reset step", t))
        assert twin.sim.debug_streams() == env.sim.debug_streams(), t
        assert np.array_equal(dyn_host(twin, torch), after), t
        tw = {k: v.cpu().numpy() for k, v in twin.state.items()}
        for key in ("pos_x", "pos_z", "angle", "wheel_dist", "episode", "step_count"):
            assert np.array_equal(tw[key], st[key]), (t, key)
    print(f"\nauto-reset: {walks} walks ended, {resets} resets in 700 steps")
    assert walks > 2 * n and resets >= 7 * n
    env.close(); twin.close()
