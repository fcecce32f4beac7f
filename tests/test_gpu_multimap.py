"""Batches that mix maps, against the CPU oracle and the reference goldens.

Every kernel on the hot path looks up the env's own map: k_frame_setup (the top-down camera), k_cull and k_geometry (which
items exist), the three rasterisers (the texture pool), the step logic and respawn (grid, curves, obstacles), and the
frame memory is sized from the largest uploaded map.  A batch of one map cannot tell `maps[S.map_id[env]]` from
`maps[0]`, nor frame memory sized from one map from memory sized from all of them.  Here every env's frame, step and
obstacle state is held to what the oracle computes for that env's own map, bit-exact for frames.
"""
import copy
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 1
# bench.py's c5 maps.  udem1 (the largest texture pool and the most props) sits in slot 0, so that a kernel reading slot
# 0's tables for every env reads valid memory and shows up as wrong pixels.
C5 = ["udem1", "small_loop", "loop_obstacles", "loop_pedestrians", "loop_dyn_duckiebots", "loop_trafficlights"]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(autouse=True)
def _default_tile_mode():
    import oracle as orc
    orc.lib().orr_set_tile_mode(1)
    yield
    orc.lib().orr_set_tile_mode(1)


# ------------------------------------------------------------------------------------------------------------ helpers
def make_env(maps_, n, **kw):
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    args = dict(camera_width=160, camera_height=120, domain_rand=False, seed=1000)
    args.update(kw)
    return BatchedDuckietownEnv(n, maps_, **args)


def load_md(name, golden_dir):
    from gym_duckietown_b200 import maps
    md = maps.load_map(name)
    g = np.load(os.path.join(golden_dir, f"dynamic_{name}.npz"))
    for d, w in zip(md.dyn_objects, g["wiggle"]):   # the reference draws the wiggle from the unseeded global RNG
        d.wiggle = float(w)
    return md, g


def trafficlight_md(golden_dir):
    """loop_trafficlights with the frequencies and first patterns of the golden's plain run."""
    from gym_duckietown_b200 import maps
    g = np.load(os.path.join(golden_dir, "trafficlight_loop_trafficlights.npz"))
    md = copy.deepcopy(maps.load_map("loop_trafficlights"))
    tl = [i for i, d in enumerate(md.dyn_objects) if d.kind == maps.DYN_TRAFFICLIGHT]
    for k, i in enumerate(tl):
        md.dyn_objects[i].freq, md.dyn_objects[i].pattern = float(g["plain_freq"][k]), int(g["plain_pattern0"][k])
    return md, g, tl


def dyn_host(env, torch, map_id):
    from gym_duckietown_b200 import lib as L
    arr, nd = env.sim.dyn_state(map_id)
    if not nd:
        return np.zeros((L.DYN_FIELDS, 0, env.num_envs))
    return torch.as_tensor(arr, device=env.device).view(L.DYN_FIELDS, nd, env.num_envs).cpu().numpy()


def oracle_scene(md):
    """The map's scene as it is at load time: the traffic-light card is the last light's pattern."""
    import oracle as orc
    sc = orc.OracleScene(md)
    sc.set_trafficlight_card(orc.OracleDynamics(orc.OracleMap(md)).shown_card)
    return sc


def oracle_episode(params, k):
    """The oracle's episode record from host-drawn reset params (first episode: identity modelview)."""
    import oracle as orc
    ep = orc.default_episode()
    ep.cam_height = float(params["cam_height"][k]); ep.cam_angle_deg = float(params["cam_angle_deg"][k])
    ep.cam_fov_y_deg = float(params["cam_fov_y_deg"][k])
    for name, field in (("cam_noise", "cam_noise"), ("horizon_color", "horizon"), ("light_ambient", "ambient"),
                        ("light_diffuse", "diffuse"), ("ground_color", "ground")):
        for i in range(3):
            getattr(ep, field)[i] = float(np.float32(params[name][k][i]))
    for i in range(4):
        ep.light_eye[i] = float(np.float32(params["light_pos"][k][i]))
    for i in range(8):
        ep.hidden[i] = int(params["obj_hidden"][k][i])
    return ep


def recorded_episode(r):
    """The oracle's episode record from the device's (dts_debug_episode)."""
    import oracle as orc
    return orc.default_episode(cam_height=float(r["cam_height"]), cam_angle_deg=float(r["cam_angle_deg"]),
                               cam_fov_y_deg=float(r["cam_fov_y_deg"]), cam_noise=r["cam_noise"], horizon=r["horizon"],
                               ambient=r["ambient"], diffuse=r["diffuse"], light_eye=r["light_eye"], ground=r["ground"],
                               hidden=[int(v) for v in r["hidden"]])


def oracle_frames(scenes, mid, px, pz, ang, eps, W, H, dr=False, lut=None):
    """Each env's frame on its own map, one oracle batch per map."""
    out = np.zeros((len(mid), H, W, 3), np.uint8)
    for m in np.unique(mid):
        sel = np.flatnonzero(mid == m)
        out[sel] = scenes[m].render_batch(px[sel], pz[sel], ang[sel], [eps[k] for k in sel], W, H, dr, lut=lut,
                                          threads=THREADS)
    return out


def assert_exact(got, want, tag):
    diff = np.abs(got.astype(np.int16) - want.astype(np.int16)).reshape(len(got), -1).max(1)
    bad = np.flatnonzero(diff)
    assert len(bad) == 0, f"{tag}: {len(bad)} frames differ from the oracle (envs {bad[:8].tolist()}, max {diff.max()} LSB)"


def poses_for(md, rng, n):
    """n camera poses on one map: random drivable cells, and every third one facing a prop from 0.15 .. 2.5 m (props'
    triangles from screen-filling down to sub-pixel size)."""
    ts = md.tile_size
    cells = np.array(md.drivable_tiles)
    out = np.zeros((n, 3))
    for i in range(n):
        if md.objects and i % 3 == 0:
            o = md.objects[rng.integers(len(md.objects))]
            d, a = rng.choice([0.15, 0.3, 0.5, 0.8, 1.2, 1.8, 2.5]), rng.uniform(-np.pi, np.pi)
            out[i] = (o.pos[0] - d * np.cos(a), o.pos[2] + d * np.sin(a), a + rng.uniform(-0.25, 0.25))
        else:
            c = cells[rng.integers(len(cells))]
            out[i] = ((c[0] + rng.uniform()) * ts, (c[1] + rng.uniform()) * ts, rng.uniform(-np.pi, np.pi))
    return out


def mixed_layout(mds, n, seed):
    """Map ids: env k on k % len(mds) for the first half, a seeded shuffle of the same for the second (every warp and
    CTA meets several maps, in no regular order); poses drawn on each env's own map."""
    rng = np.random.default_rng(seed)
    mid = np.arange(n, dtype=np.int32) % len(mds)
    mid[n // 2:] = rng.permutation(mid[n // 2:])
    P = np.zeros((n, 3))
    for m, md in enumerate(mds):
        sel = np.flatnonzero(mid == m)
        P[sel] = poses_for(md, rng, len(sel))
    return mid, P[:, 0].copy(), P[:, 1].copy(), P[:, 2].copy()


def place(env, mid, px, pz, ang):
    env.sim.reset(None, dict(pos_x=px, pos_z=pz, angle=ang, map_id=mid), env._stream())


# ------------------------------------------------------------------------------------------- 1. mixed-batch frames
FRAME_CASES = {
    "160x120_1500": dict(n=1500, W=160, H=120),
    "84x84": dict(n=384, W=84, H=84),
    "320x240_dr": dict(n=192, W=320, H=240, dr=True),
    "tessellated": dict(n=384, W=160, H=120, tess=True),
    "fisheye": dict(n=384, W=160, H=120, distortion=True),
    "chw_f32": dict(n=384, W=160, H=120, fmt=("chw", "float32")),
}


@pytest.mark.parametrize("case", list(FRAME_CASES))
def test_mixed_batch_frames_vs_oracle(case, torch_cuda):
    """The six c5 maps in one batch: every env's frame equals the oracle's frame on that env's map, 0 LSB."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    c = FRAME_CASES[case]
    n, W, H, dr, tess = c["n"], c["W"], c["H"], c.get("dr", False), c.get("tess", False)
    mds = [maps.load_map(m) for m in C5]
    mid, px, pz, ang = mixed_layout(mds, n, seed=11)
    orc.lib().orr_set_tile_mode(0 if tess else 1)
    env = make_env(C5, n, camera_width=W, camera_height=H, domain_rand=dr, tessellate_tiles=tess,
                   distortion=c.get("distortion", False), seed=41)
    if "fmt" in c:
        env.set_output_format(obs_layout=c["fmt"][0], obs_dtype=c["fmt"][1])
    if dr:
        # host-drawn DR for each env's own map (obj_hidden included), at the poses chosen here
        captured = {}
        orig = env.sim.reset

        def reset_at_poses(mask, params, stream=0):
            params = dict(params, pos_x=px, pos_z=pz, angle=ang)
            captured.update(params)
            return orig(mask, params, stream)
        env.sim.reset = reset_at_poses
        env.map_ids[:] = mid
        got = env.reset().cpu().numpy()
        assert np.array_equal(captured["map_id"], mid)
        assert captured["obj_hidden"][mid == 0].any(), "no optional prop of udem1 was hidden"
        eps = [oracle_episode(captured, k) for k in range(n)]
    else:
        place(env, mid, px, pz, ang)
        got = env.render_obs().cpu().numpy()
        eps = [orc.default_episode() for _ in range(n)]
    assert np.array_equal(env.state["map_id"].cpu().numpy(), mid)
    lut = (env.camera_model.rmapx, env.camera_model.rmapy) if c.get("distortion") else None
    want = oracle_frames([oracle_scene(md) for md in mds], mid, px, pz, ang, eps, W, H, dr, lut)
    if "fmt" in c:
        ref = (want.transpose(0, 3, 1, 2) / 255.0).astype(np.float32)
        if not np.array_equal(got, ref):
            assert_exact(np.rint(got * 255.0).astype(np.uint8), want.transpose(0, 3, 1, 2), case)
            raise AssertionError(f"{case}: float32 values are not u8 / 255")
    else:
        assert_exact(got, want, case)
    assert got.std() > 0.05 if "fmt" in c else got.std() > 10
    env.check()
    env.close()


def test_mixed_batch_permutation_and_isolation(torch_cuda):
    """The same (map, pose) set in a permuted env order gives the permuted frames, byte for byte; and each frame is the
    frame a batch of that env's map alone gives for that pose."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    n = 600
    mds = [maps.load_map(m) for m in C5]
    mid, px, pz, ang = mixed_layout(mds, n, seed=12)
    env = make_env(C5, n)
    place(env, mid, px, pz, ang)
    base = env.render_obs().clone()
    perm = np.random.default_rng(3).permutation(n)
    place(env, mid[perm], px[perm], pz[perm], ang[perm])
    permuted = env.render_obs()
    torch.cuda.synchronize()
    assert torch.equal(permuted, base[torch.as_tensor(perm, device=env.device)]), "frames depend on the env order"
    env.check()
    env.close()
    base = base.cpu().numpy()
    for m, name in enumerate(C5):
        sel = np.flatnonzero(mid == m)
        solo = make_env(name, len(sel))
        place(solo, np.zeros(len(sel), np.int32), px[sel], pz[sel], ang[sel])
        alone = solo.render_obs().cpu().numpy()
        assert_exact(base[sel], alone, f"isolation_{name}")
        solo.check()
        solo.close()


# ------------------------------------------------------------------------- 2. obstacles and traffic lights, mixed
def test_mixed_batch_obstacles_and_traffic_lights(golden_dir, torch_cuda):
    """Pedestrians, duckiebots and traffic lights in one batch with two static maps, envs interleaved: each env's
    obstacles on its own map follow the reference's trace, its slots on the other maps keep their load-time state, and
    its frames show its own obstacles and card."""
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L, maps
    ped, g_ped = load_md("loop_pedestrians", golden_dir)
    bots, g_bots = load_md("loop_dyn_duckiebots", golden_dir)
    tlmd, g_tl, tl = trafficlight_md(golden_dir)
    mds = [ped, bots, tlmd, maps.load_map("small_loop"), maps.load_map("loop_obstacles")]
    golden = {0: g_ped, 1: g_bots}
    n, T = 40, 263                    # past the first card flip (step 149) and into the pedestrians' walk (steps 240-269)
    flip = int(np.flatnonzero(np.diff(g_tl["plain_shown"]))[0]) + 1
    assert flip + 5 < T - 1 and T <= 400
    when = (100, flip + 5, T - 1)     # the steps whose frames are compared: card 0, card 1, pedestrians walking
    mid = np.arange(n, dtype=np.int32) % len(mds)
    rng = np.random.default_rng(21)
    px, pz, ang = np.zeros(n), np.zeros(n), np.zeros(n)
    for k in range(n):                # look at one of the env's obstacles from 0.45 m (where it is at the last step)
        m, a = mid[k], rng.uniform(-np.pi, np.pi)
        if m in golden:
            s = (k // len(mds)) % len(mds[m].dyn_objects)
            ox, oz = golden[m]["pos"][T - 1, s, 0], golden[m]["pos"][T - 1, s, 2]
        elif m == 2:
            o = tlmd.objects[tlmd.dyn_objects[tl[(k // len(mds)) % len(tl)]].object_index]
            ox, oz = o.pos[0], o.pos[2]
        else:
            px[k], pz[k], ang[k] = poses_for(mds[m], rng, 1)[0]
            continue
        px[k], pz[k], ang[k] = ox - 0.45 * np.cos(a), oz + 0.45 * np.sin(a), a
    env = make_env(mds, n)
    place(env, mid, px, pz, ang)
    init = {m: dyn_host(env, torch, m) for m in range(len(mds))}
    zero = torch.zeros(n, 2, device=env.device)
    frames = {}
    for t in range(T):
        obs, *_ = env.step(zero, render=t in when)
        if t in when:
            frames[t] = (obs.cpu().numpy().copy(), {m: dyn_host(env, torch, m) for m in range(len(mds))})
        if t % 9 and t not in when and t != T - 1:
            continue
        for m in range(3):
            st = dyn_host(env, torch, m)
            on, off = mid == m, mid != m
            assert np.array_equal(st[:, :, off], init[m][:, :, off]), (t, m, "slots of envs on other maps changed")
            if m in golden:
                g = golden[m]
                assert np.abs(st[L.DYN_PX][:, on] - g["pos"][t, :, 0:1]).max() <= 1e-9, (t, m)
                assert np.abs(st[L.DYN_PZ][:, on] - g["pos"][t, :, 2:3]).max() <= 1e-9, (t, m)
                assert np.abs(st[L.DYN_YROT][:, on] - g["y_rot"][t][:, None]).max() <= 1e-7, (t, m)
                if m == 0:
                    assert np.array_equal(st[L.DYN_ACTIVE][:, on] != 0, np.repeat(g["active"][t][:, None], on.sum(), 1)), t
            else:
                assert (st[L.DYN_PATTERN][tl][:, on] == g_tl["plain_pattern"][t][:, None]).all(), t
                assert (st[L.DYN_SHOWN, tl[0], on] == g_tl["plain_shown"][t]).all(), t
    assert g_ped["active"][T - 1].any()                   # the pedestrians are walking
    state = {k: v.cpu().numpy() for k, v in env.state.items()}
    scenes = [oracle_scene(md) for md in mds]
    cards = set()
    for t, (got, dst) in frames.items():
        want = np.zeros_like(got)
        for k in range(n):
            m, sc = mid[k], scenes[mid[k]]
            for s, d in enumerate(mds[m].dyn_objects):   # this env's obstacles, where its own state has them
                if d.kind != maps.DYN_TRAFFICLIGHT:
                    sc.set_object_pose(d.object_index, (dst[m][L.DYN_PX, s, k], d.pos[1], dst[m][L.DYN_PZ, s, k]),
                                       dst[m][L.DYN_YROT, s, k])
            if m == 2:
                cards.add(int(dst[m][L.DYN_SHOWN, tl[0], k]))
                sc.set_trafficlight_card(int(dst[m][L.DYN_SHOWN, tl[0], k]))
            want[k] = sc.render(state["pos_x"][k], state["pos_z"][k], state["angle"][k], W=160, H=120)
        assert_exact(got, want, f"obstacles_t{t}")
    assert cards == {0, 1}
    # the obstacles are in view: the load-time scenes give other frames
    got, still = frames[T - 1][0], [oracle_scene(md) for md in mds[:2]]
    moved = sum(int(np.any(still[mid[k]].render(state["pos_x"][k], state["pos_z"][k], state["angle"][k]) != got[k]))
                for k in range(n) if mid[k] in golden)
    assert moved >= 8, moved
    env.check()
    env.close()


# ------------------------------------------------------------------------------------ 3. segment and top-down views
@pytest.mark.parametrize("segment,top_down", [(True, False), (False, True), (True, True)])
def test_mixed_batch_segment_and_top_down_vs_oracle(segment, top_down, torch_cuda):
    """The top-down camera frames each env's own map (5 x 5 or 8 x 7 tiles) and draws the agent's mesh at its pose;
    segmentation textures come from each env's map."""
    from gym_duckietown_b200 import maps
    names = ["udem1", "small_loop", "loop_obstacles", "loop_trafficlights"]
    mds = [maps.load_map(m) for m in names]
    n = 64
    mid, px, pz, ang = mixed_layout(mds, n, seed=13)
    env = make_env(names, n)
    place(env, mid, px, pz, ang)
    got = env.render_obs(segment=segment, top_down=top_down).cpu().numpy()
    scenes = [oracle_scene(md) for md in mds]
    want = np.stack([scenes[mid[k]].render(px[k], pz[k], ang[k], None, 160, 120, segment=segment, top_down=top_down)
                     for k in range(n)])
    assert_exact(got, want, f"modes_{int(segment)}{int(top_down)}")
    env.check()
    env.close()


# ------------------------------------------------------------------------------------- 4. frame-memory sizing
@pytest.mark.parametrize("tess", [False, True])
def test_frame_memory_sized_from_the_largest_map(tess, torch_cuda):
    """[small_loop, udem1] with every env on slot 1: the small map in slot 0 must not size the frame memory."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    orc.lib().orr_set_tile_mode(0 if tess else 1)
    md = maps.load_map("udem1")
    n = 256
    P = poses_for(md, np.random.default_rng(14), n)
    env = make_env(["small_loop", "udem1"], n, tessellate_tiles=tess)
    place(env, np.ones(n, np.int32), P[:, 0].copy(), P[:, 1].copy(), P[:, 2].copy())
    got = env.render_obs().cpu().numpy()
    env.check()
    want = oracle_scene(md).render_batch(P[:, 0], P[:, 1], P[:, 2], [orc.default_episode() for _ in range(n)], 160, 120,
                                         threads=THREADS)
    assert_exact(got, want, f"sized_{'tess' if tess else 'quad'}")
    env.close()


def test_upload_map_resizes_frame_memory(torch_cuda):
    """Render on [small_loop, small_loop]; upload udem1 into slot 1 and move the envs there: the next render sizes its
    frame memory for udem1.  Then shrink it again with small_loop."""
    import oracle as orc
    from gym_duckietown_b200 import maps
    small, big = maps.load_map("small_loop"), maps.load_map("udem1")
    n = 256
    rng = np.random.default_rng(15)
    env = make_env(["small_loop", "small_loop"], n)
    ones = np.ones(n, np.int32)
    eps = [orc.default_episode() for _ in range(n)]
    for i, (tag, md) in enumerate((("small_loop", small), ("udem1", big), ("small_loop_again", small))):
        if i:
            env.sim.upload_map(1, md)
        P = poses_for(md, rng, n)
        place(env, ones, P[:, 0].copy(), P[:, 1].copy(), P[:, 2].copy())
        got = env.render_obs().cpu().numpy()
        env.check()
        want = oracle_scene(md).render_batch(P[:, 0], P[:, 1], P[:, 2], eps, 160, 120, threads=THREADS)
        assert_exact(got, want, f"upload_{tag}")
    env.close()


def _texture(h, w, hgt, backed):
    """Texture 0 of the blob becomes w x hgt; `backed`: over a zeroed buffer of that size, else over the old texels."""
    from gym_duckietown_b200 import lib as L
    texs = h.keep["texs"]
    if backed:
        h.keep["big"] = np.zeros((hgt, w, 4), np.uint8)
    texs[0] = L.Texture(w, hgt, h.keep["big"].ctypes.data if backed else texs[0].rgba)


def _set(arr, i, **kw):
    for k, v in kw.items():
        setattr(arr[i], k, v)


# Every refusal of dts_upload_map, on a fresh blob of loop_pedestrians (6 objects, the first 4 of them the pedestrians
# of dyn slots 0-3; 2 meshes of 148 and 72 triangles; 8 textures): (slot, corruption, the error it gets)
REFUSED_UPLOADS = {
    "map_id": (2, lambda h: None, "bad map_id 2"),
    "too_many_objects": (0, lambda h: setattr(h.blob, "n_objects", 257), "map has 257 objects, limit 256"),
    "bad_grid": (0, lambda h: setattr(h.blob, "grid_w", 0), "invalid tile grid"),
    "n_dyn": (0, lambda h: setattr(h.blob, "n_dyn", 33), "map has 33 dynamic obstacles, limit 32"),
    "mesh_id": (0, lambda h: _set(h.keep["objs"], 5, mesh_id=2), "object 5: bad mesh_id"),
    "alt_texture": (0, lambda h: _set(h.keep["objs"], 5, alt_tex_to=h.blob.n_textures), "object 5: alt texture out of range"),
    "dyn_slot": (0, lambda h: _set(h.keep["objs"], 4, dyn_slot=4), "object 4: dyn_slot 4 out of range"),
    "not_power_of_two": (0, lambda h: _texture(h, 255, 256, False), "texture 0: 255x256 is not a power of two"),
    "side_over_2^15": (0, lambda h: _texture(h, 65536, 1, True), "texture 0: 65536x1 too large"),
    "pool_over_4GB": (0, lambda h: _texture(h, 32768, 32768, False), "textures exceed 4 GB"),
    "mesh_past_n_tris": (0, lambda h: _set(h.keep["meshes"], 1, tri_count=73), "mesh 1: triangles 148 .. 221 past n_tris 220"),
    "dyn_kind": (0, lambda h: _set(h.keep["dyn"], 0, kind=9), "dyn 0: bad kind 9"),
    "dyn_back_pointer": (0, lambda h: _set(h.keep["dyn"], 0, object_index=4),
                         "dyn 0: object_index 4 does not point back to this slot"),
}


@pytest.mark.parametrize("case", list(REFUSED_UPLOADS))
def test_refused_upload_leaves_the_slot_as_it_was(case, torch_cuda):
    """A blob dts_upload_map refuses changes nothing: slot 0 keeps its map on the host and the device, the next frames
    are the frames before it, bit for bit and equal to the oracle's, and the batch still steps."""
    import ctypes as C
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import lib as L, maps
    md = maps.load_map("loop_pedestrians")
    n = 128
    P = poses_for(md, np.random.default_rng(17), n)
    env = make_env(["loop_pedestrians", "loop_pedestrians"], n)
    place(env, np.zeros(n, np.int32), P[:, 0].copy(), P[:, 1].copy(), P[:, 2].copy())
    before = env.render_obs().clone()
    slot, corrupt, message = REFUSED_UPLOADS[case]
    holder = L.MapBlobHolder(md)
    corrupt(holder)
    sim = env.sim
    assert sim.lib.dts_upload_map(sim.h, slot, C.byref(holder.blob)) != 0
    assert sim.lib.dts_last_error(sim.h).decode() == message
    after = env.render_obs()
    torch.cuda.synchronize()
    assert torch.equal(after, before), f"{case}: the frames changed"
    want = oracle_scene(md).render_batch(P[:, 0], P[:, 1], P[:, 2], [orc.default_episode() for _ in range(n)], 160, 120,
                                         threads=THREADS)
    assert_exact(after.cpu().numpy(), want, f"refused_{case}")
    env.check()
    env.step(torch.zeros(n, 2, device=env.device))
    env.check()
    env.close()


# -------------------------------------------------------------------------------------- 5. step logic, mixed
def test_mixed_batch_trajectory_vs_oracle(golden_dir, torch_cuda):
    """test_trajectory_vs_oracle with env k on map k % 5, static and dynamic maps, auto-reset off."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps
    ped, g_ped = load_md("loop_pedestrians", golden_dir)
    bots, g_bots = load_md("loop_dyn_duckiebots", golden_dir)
    mds = [maps.load_map("small_loop"), maps.load_map("loop_obstacles"), maps.load_map("udem1"), ped, bots]
    wiggle = {3: g_ped["wiggle"], 4: g_bots["wiggle"]}
    N, T = 80, 300
    mid = np.arange(N, dtype=np.int32) % len(mds)
    env = make_env(mds, N, max_steps=250)
    env.map_ids[:] = mid
    env.reset(render=False)
    torch.cuda.synchronize()
    st0 = {k: v.cpu().numpy().copy() for k, v in env.state.items()}
    assert np.array_equal(st0["map_id"], mid)
    oms = [orc.OracleMap(md) for md in mds]
    cpu = [orc.OracleEnv(oms[mid[k]], st0["pos_x"][k], st0["pos_z"][k], st0["angle"][k], wheel_dist=st0["wheel_dist"][k],
                         max_steps=250,
                         dynamics=orc.OracleDynamics(oms[mid[k]], wiggle=wiggle[mid[k]]) if mid[k] in wiggle else None)
           for k in range(N)]
    acts = np.random.default_rng(1234).uniform(-1, 1, (T, N, 2)).astype(np.float32)
    acts[:, : N // 4, 0] = 0.12       # gentle forward actions keep some envs alive
    acts[:, : N // 4, 1] *= 0.3
    acts[:, : N // 8, :] = 0.0        # parked: max_steps
    codes = {m: set() for m in range(len(mds))}
    for t in range(T):
        _, rew, done, info = env.step(torch.from_numpy(acts[t]).to(env.device), render=False)
        s = {k: v.cpu().numpy() for k, v in info.items()}
        d = done.cpu().numpy()
        for k in range(N):
            o = cpu[k].step(acts[t, k])
            assert (s["tile_i"][k], s["tile_j"][k]) == (o.tile_i, o.tile_j), (t, k)
            assert bool(d[k]) == bool(o.done) and s["done_code"][k] == o.done_code, (t, k)
            assert bool(s["collided"][k]) == bool(o.collided), (t, k)
            assert s["step_count"][k] == o.step_count, (t, k)
            assert abs(s["pos_x"][k] - o.pos_x) <= 1e-5 and abs(s["pos_z"][k] - o.pos_z) <= 1e-5, (t, k)
            dang = abs(s["angle"][k] - o.angle)
            assert min(dang, abs(dang - 2 * np.pi)) <= 1e-5, (t, k)
            assert abs(s["reward"][k] - o.reward) <= 1e-5 * max(1.0, abs(o.reward)), (t, k)
            assert abs(s["prox_penalty"][k] - o.prox) <= 1e-9, (t, k)
            codes[mid[k]].add(int(o.done_code))
    assert set().union(*codes.values()) == {0, 1, 2}, codes
    assert all(2 in codes[m] for m in range(3)), codes   # on every static map some envs lived to max_steps
    env.check()
    env.close()


# ----------------------------------------------------------------- 6. cycle_maps auto-reset, reference-style loop
def test_cycle_maps_auto_reset_vs_reference_style_loop(torch_cuda):
    """MultiMapEnv under device auto-reset: the map advances on every reset after the first; every spawn equals the host
    sampler's on the env's next map, and every terminal frame equals the oracle's on the map the episode ran on."""
    torch = torch_cuda
    import oracle as orc
    from gym_duckietown_b200 import maps
    from gym_duckietown_b200.episode import EpisodeSampler
    from test_reset_sampler import oracle_query

    names = ["small_loop", "loop_obstacles", "udem1"]
    mds = [maps.load_map(m) for m in names]
    N, T, W, H = 24, 300, 160, 120
    kw = dict(seed=500, device_reset=True, cycle_maps=True, max_steps=60)
    env = make_env(names, N, auto_reset=True, terminal_obs=True, **kw)
    ref = make_env(names, N, **kw)    # the same streams, reset by the caller: its state holds the terminal poses
    env.reset()
    ref.reset(render=False)
    torch.cuda.synchronize()
    host = EpisodeSampler(N, domain_rand=False)
    host.seed([500 + k for k in range(N)])
    qs = [oracle_query(md) for md in mds]
    oms = [orc.OracleMap(md) for md in mds]
    cur = np.zeros(N, np.int32)
    first = host.sample(list(range(N)), [mds[0]] * N, qs[0])
    cpu = [orc.OracleEnv(oms[0], first["pos_x"][k], first["pos_z"][k], first["angle"][k],
                         wheel_dist=first["wheel_dist"][k], max_steps=60) for k in range(N)]
    st = {k: v.cpu().numpy() for k, v in env.state.items()}
    assert np.array_equal(st["map_id"], cur)
    assert np.array_equal(st["pos_x"], first["pos_x"]) and np.array_equal(st["angle"], first["angle"])
    records = [env.sim.debug_episode(k) for k in range(N)]
    terminal = []                     # (frame, map, pose, episode record)
    acts = np.random.default_rng(3).uniform(-1, 1, (T, N, 2)).astype(np.float32)
    acts[:, :, 0] = np.abs(acts[:, :, 0])
    for t in range(T):
        a = torch.from_numpy(acts[t]).to(env.device)
        _, rew, done, info = env.step(a)
        _, _, rdone, rinfo = ref.step(a, render=False)
        s = {k: v.cpu().numpy() for k, v in info.items()}
        r = {k: v.cpu().numpy() for k, v in rinfo.items()}
        d = done.cpu().numpy()
        assert np.array_equal(d, rdone.cpu().numpy()), t
        tobs = env.terminal_obs.cpu().numpy() if d.any() else None
        for k in range(N):
            o = cpu[k].step(acts[t, k])
            assert bool(d[k]) == bool(o.done) and s["done_code"][k] == o.done_code, (t, k)
            assert abs(s["reward"][k] - o.reward) <= 1e-5 * max(1.0, abs(o.reward)), (t, k)
            if not o.done:
                assert abs(s["pos_x"][k] - o.pos_x) <= 1e-5 and abs(s["pos_z"][k] - o.pos_z) <= 1e-5, (t, k)
                continue
            assert abs(r["pos_x"][k] - o.pos_x) <= 1e-5 and abs(r["pos_z"][k] - o.pos_z) <= 1e-5, (t, k)
            terminal.append((tobs[k].copy(), cur[k], (r["pos_x"][k], r["pos_z"][k], r["angle"][k]), records[k]))
            cur[k] = (cur[k] + 1) % len(mds)              # MultiMapEnv.reset: the next map
            nxt = host.sample([k], [mds[cur[k]]], qs[cur[k]])
            assert s["map_id"][k] == cur[k], (t, k)
            assert (s["pos_x"][k], s["pos_z"][k], s["angle"][k]) == (nxt["pos_x"][0], nxt["pos_z"][0], nxt["angle"][0]), (t, k)
            assert s["step_count"][k] == 0
            cpu[k] = orc.OracleEnv(oms[cur[k]], nxt["pos_x"][0], nxt["pos_z"][0], nxt["angle"][0],
                                   wheel_dist=nxt["wheel_dist"][0], max_steps=60)
            records[k] = env.sim.debug_episode(k)
        if d.any():
            ref.reset(mask=rdone, render=False)
    assert len(terminal) > 3 * N and len({m for _, m, _, _ in terminal}) == len(mds)
    scenes = [oracle_scene(md) for md in mds]
    got = np.stack([f for f, _, _, _ in terminal])
    want = np.stack([scenes[m].render(p[0], p[1], p[2], recorded_episode(rec), W, H) for _, m, p, rec in terminal])
    assert_exact(got, want, "terminal_frames")
    env.check()
    env.close()
    ref.close()


# ------------------------------------------------------------------- 7. per-map obstacle clocks under cycle_maps
def test_cycle_maps_keeps_each_maps_obstacle_clock(golden_dir, torch_cuda):
    """MultiMapEnv holds one Simulator per map: an env's obstacles on a map advance only while the env is on that map,
    and cycling away and back does not reset them."""
    torch = torch_cuda
    from gym_duckietown_b200 import lib as L, maps
    ped, g_ped = load_md("loop_pedestrians", golden_dir)
    bots, g_bots = load_md("loop_dyn_duckiebots", golden_dir)
    mds = [ped, maps.load_map("small_loop"), bots]
    golden = {0: g_ped, 2: g_bots}
    # per env: how many steps each episode lasts (maps 0, 1, 2, 0, ... in turn)
    sched = [[600], [100, 50, 200, 250], [250, 30, 320], [10] * 60, [300, 300], [5, 400, 100, 95]]
    T = 600
    assert all(sum(s) == T for s in sched)
    N = len(sched)
    spent = np.zeros((N, len(mds)), int)
    for e, s in enumerate(sched):
        for i, steps in enumerate(s):
            spent[e, i % len(mds)] += steps
    assert spent[:, 0].max() <= 640 and spent[:, 2].max() <= 400    # inside the reference's traces
    ends = [set(np.cumsum(s)[:-1].tolist()) for s in sched]
    env = make_env(mds, N, device_reset=True, cycle_maps=True, max_steps=5000)
    env.reset(render=False)
    init = {m: dyn_host(env, torch, m) for m in golden}
    zero = torch.zeros(N, 2, device=env.device)
    for t in range(T):
        due = [e for e in range(N) if t in ends[e]]
        if due:
            mask = torch.zeros(N, dtype=torch.uint8, device=env.device)
            mask[due] = 1
            env.reset(mask=mask, render=False)
        env.step(zero, render=False)
    mid = env.state["map_id"].cpu().numpy()
    assert np.array_equal(mid, np.array([(len(s) - 1) % len(mds) for s in sched]))
    for m, g in golden.items():
        st = dyn_host(env, torch, m)
        for e in range(N):
            if spent[e, m] == 0:
                assert np.array_equal(st[:, :, e], init[m][:, :, e]), (m, e)
                continue
            i = spent[e, m] - 1
            assert np.abs(st[L.DYN_PX, :, e] - g["pos"][i, :, 0]).max() <= 1e-9, (m, e, i)
            assert np.abs(st[L.DYN_PZ, :, e] - g["pos"][i, :, 2]).max() <= 1e-9, (m, e, i)
            assert np.abs(st[L.DYN_YROT, :, e] - g["y_rot"][i]).max() <= 1e-7, (m, e, i)
            if m == 0:
                assert np.array_equal(st[L.DYN_ACTIVE, :, e] != 0, g["active"][i]), (m, e, i)
    env.check()
    env.close()


# ------------------------------------------------------------ 8. randomize_maps_on_reset, DR, device reset
def test_randomize_maps_device_reset_first_frames_vs_oracle(torch_cuda):
    """The first frame of episodes 1 to 3 under randomize_maps_on_reset with DR drawn on the device: each env's frame on
    the map it drew, with the render record (hidden props, stale light) the device reports."""
    torch = torch_cuda
    from gym_duckietown_b200 import maps
    names = ["small_loop", "udem1", "loop_trafficlights", "loop_pedestrians"]
    mds = [maps.load_map(m) for m in names]
    scenes = [oracle_scene(md) for md in mds]
    N, W, H = 48, 160, 120
    env = make_env(names, N, domain_rand=True, device_reset=True, randomize_maps_on_reset=True, seed=300)
    acts = torch.full((N, 2), 0.4, device=env.device)
    seen, hidden_on_udem1 = set(), 0
    for ep in range(3):
        got = env.reset().cpu().numpy()
        st = {k: v.cpu().numpy() for k, v in env.state.items()}
        assert (st["episode"] == ep + 1).all()
        mid = st["map_id"]
        seen |= set(mid.tolist())
        recs = [env.sim.debug_episode(k) for k in range(N)]
        hidden_on_udem1 += sum(int(recs[k]["hidden"].any()) for k in range(N) if mid[k] == 1)
        want = np.stack([scenes[mid[k]].render(st["pos_x"][k], st["pos_z"][k], st["angle"][k], recorded_episode(recs[k]),
                                               W, H, True) for k in range(N)])
        assert_exact(got, want, f"random_maps_ep{ep + 1}")
        for _ in range(6):
            env.step(acts, render=False)
    assert seen == set(range(len(names))) and hidden_on_udem1 > 0
    env.check()
    env.close()
