"""ctypes front-end of the CPU oracle (oracle/*.c).  TEST INFRASTRUCTURE — see oracle/README.md.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import
this module.  The product package never does.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liborc.so")
SOURCES = ["dt_oracle_logic.c", "dt_oracle_raster.c", "dt_oracle_batch.c", "dt_oracle_dynamic.c"]


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, s) for s in SOURCES if os.path.exists(os.path.join(HERE, s))]
    deps = srcs + [os.path.join(HERE, "dt_oracle.h")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(s) for s in deps):
        return LIB
    # -ffp-contract=off: no silent FMA contraction, so the float arithmetic is exactly what the
    # source says (the raster oracle's fp32 spec relies on it); -mfma only makes fmaf() an instruction.
    cmd = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
           "-mfma", "-mavx2", "-o", LIB] + srcs + ["-lm"]
    subprocess.check_call(cmd)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_proximity.restype = C.c_double
        _lib.orc_dyn_proximity.restype = C.c_double
    return _lib


class OrcMap(C.Structure):
    _fields_ = [("tile_size", C.c_double), ("grid_w", C.c_int32), ("grid_h", C.c_int32),
                ("tile_kind", C.c_void_p), ("tile_drivable", C.c_void_p), ("tile_curve_off", C.c_void_p),
                ("tile_curve_cnt", C.c_void_p), ("curves", C.c_void_p), ("n_coll", C.c_int32),
                ("coll_corners", C.c_void_p), ("coll_norms", C.c_void_p), ("coll_centers", C.c_void_p),
                ("coll_radii", C.c_void_p)]


class OrcDynParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("u1", "u2", "u3", "w1", "w2", "w3", "uar", "ual", "war", "wal")] + \
               [("delay_steps", C.c_int32)]


ORC_MAX_DELAY = 16   # dt_oracle.h; the delay line is as deep as the device's (DTS_MAX_DELAY)


class OrcDynState(C.Structure):
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("theta", C.c_double), ("u", C.c_double),
                ("w", C.c_double), ("fifo", (C.c_double * 2) * ORC_MAX_DELAY)]


class OrcStepOut(C.Structure):
    _fields_ = [("pos_x", C.c_double), ("pos_z", C.c_double), ("angle", C.c_double), ("speed", C.c_double),
                ("reward", C.c_double), ("lane_dist", C.c_double), ("lane_dot", C.c_double),
                ("lane_angle", C.c_double), ("prox", C.c_double), ("tile_i", C.c_int32), ("tile_j", C.c_int32),
                ("step_count", C.c_int32), ("done", C.c_uint8), ("done_code", C.c_uint8), ("in_lane", C.c_uint8),
                ("collided", C.c_uint8), ("drivable4", C.c_uint8)]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class OracleMap:
    """Holds contiguous copies of a MapData's arrays and the orc_map struct pointing at them."""

    def __init__(self, md):
        self.md = md
        self._keep = dict(
            kind=np.ascontiguousarray(md.tile_kind, np.int8), drv=np.ascontiguousarray(md.tile_drivable, np.uint8),
            coff=np.ascontiguousarray(md.tile_curve_off, np.int32), ccnt=np.ascontiguousarray(md.tile_curve_cnt, np.int32),
            curves=np.ascontiguousarray(md.curves, np.float64),
            cc=np.ascontiguousarray(md.coll_corners, np.float64), cn=np.ascontiguousarray(md.coll_norms, np.float64),
            ce=np.ascontiguousarray(md.coll_centers, np.float64), cr=np.ascontiguousarray(md.coll_radii, np.float64))
        k = self._keep
        self.c = OrcMap(md.tile_size, md.grid_w, md.grid_h, _p(k["kind"]), _p(k["drv"]), _p(k["coff"]), _p(k["ccnt"]),
                        _p(k["curves"]), md.n_coll, _p(k["cc"]), _p(k["cn"]), _p(k["ce"]), _p(k["cr"]))

    def done_reward(self, px, pz, angle, step_count, max_steps=1500, robot_speed=1.2) -> OrcStepOut:
        o = OrcStepOut()
        lib().orc_done_reward(C.byref(self.c), C.c_double(px), C.c_double(pz), C.c_double(angle), C.c_int(step_count),
                              C.c_int(max_steps), C.c_double(robot_speed), C.byref(o))
        return o

    def valid_pose(self, px, pz, angle, sf=1.0) -> bool:
        return bool(lib().orc_valid_pose(C.byref(self.c), C.c_double(px), C.c_double(pz), C.c_double(angle),
                                         C.c_double(sf), None, None))

    def collision(self, px, pz, angle) -> bool:
        return bool(lib().orc_collision(C.byref(self.c), C.c_double(px), C.c_double(pz), C.c_double(angle)))

    def proximity(self, px, pz, angle) -> float:
        return float(lib().orc_proximity(C.byref(self.c), C.c_double(px), C.c_double(pz), C.c_double(angle)))


def action_map(vel, steer, wheel_dist, gain=1.0, trim=0.0, radius=0.0318, k=27.0, limit=1.0):
    out = (C.c_double * 2)()
    lib().orc_action_map(*(C.c_double(float(v)) for v in (vel, steer, wheel_dist, gain, trim, radius, k, limit)), out)
    return out[0], out[1]


# get_DB18_nominal as restated in DESIGN.md §4 (parity unpinned): the ten model constants and the command delay in
# seconds, under the names dts_config gives them without their `dyn_` prefix.
DB18_NOMINAL = dict(u1=5.0, u2=0.0, u3=0.0, w1=4.0, w2=0.0, w3=0.0, uar=1.5, ual=1.5, war=15.0, wal=15.0, delay=0.15)


def delay_steps(delay: float, dt: float) -> int:
    """Integration steps a command waits before it acts: the fewest whose span reaches `delay` (dts_create /
    dts_set_timing, the same expression in the same float64 arithmetic)."""
    d = 0
    while d * dt < delay - 1e-12:
        d += 1
    return d


def dyn_params(dt=1.0 / 30, trim=0.0, **model) -> OrcDynParams:
    """OrcDynParams of the model `DB18_NOMINAL` updated with `model` (any of its keys), stepped at `dt`, with the
    per-env `trim` folded into the gains as the device folds it in (get_DB18_uncalibrated: right gains * (1 + trim),
    left gains * (1 - trim)).  A delay longer than the delay line can hold is refused, as dts_create refuses it."""
    unknown = set(model) - set(DB18_NOMINAL)
    if unknown:
        raise TypeError(f"unknown dynamics constants {sorted(unknown)}")
    p = dict(DB18_NOMINAL, **model)
    d = delay_steps(p["delay"], dt)
    if d > ORC_MAX_DELAY:
        raise ValueError(f"a delay of {p['delay']} s is {d} steps of {dt} s: the delay line holds {ORC_MAX_DELAY}")
    return OrcDynParams(p["u1"], p["u2"], p["u3"], p["w1"], p["w2"], p["w3"], p["uar"] * (1.0 + trim),
                        p["ual"] * (1.0 - trim), p["war"] * (1.0 + trim), p["wal"] * (1.0 - trim), d)


def default_dyn_params(dt=1.0 / 30, delay=0.15, trim=0.0) -> OrcDynParams:
    """get_DB18_nominal / get_DB18_uncalibrated as restated in DESIGN.md (parity unpinned)."""
    return dyn_params(dt, trim, delay=delay)


class OracleEnv:
    """One reference-style env stepped by the C oracle: the CPU side of every trajectory parity test."""

    def __init__(self, omap: OracleMap, px, pz, angle, *, wheel_dist=0.102, action_mode=1, max_steps=1500,
                 frame_skip=1, dt=1.0 / 30, robot_speed=1.2, env5=(1.0, 0.0, 0.0318, 27.0, 1.0), trim=0.0,
                 dynamics=None, model=None):
        """model: the wheel model's constants and command delay, any keys of DB18_NOMINAL (the dts_config fields
        dyn_u1 ... dyn_wal, dyn_delay); the others keep their nominal values."""
        self.m = omap
        self.dynamics = dynamics          # OracleDynamics: this env's moving obstacles (stepped with the agent)
        self.dp = dyn_params(dt, trim, **(model or {}))
        self.s = OrcDynState()
        lib().orc_cartesian_from_weird(C.byref(omap.c), C.c_double(px), C.c_double(pz), C.c_double(angle), C.byref(self.s))
        self.step_count = C.c_int(0)
        self.px, self.pz = C.c_double(px), C.c_double(pz)
        self.wheel_dist, self.action_mode, self.max_steps = wheel_dist, action_mode, max_steps
        self.frame_skip, self.dt, self.robot_speed = frame_skip, dt, robot_speed
        self.env5 = (C.c_double * 5)(*env5)

    def step(self, action) -> OrcStepOut:
        o = OrcStepOut()
        a = (C.c_double * 2)(float(action[0]), float(action[1]))
        if self.dynamics is not None:
            d = self.dynamics
            lib().orc_step_dynamic(C.byref(self.m.c), C.byref(self.dp), C.byref(self.s), C.byref(self.step_count),
                                   C.byref(self.px), C.byref(self.pz), a, C.c_int(self.action_mode),
                                   C.c_double(self.wheel_dist), self.env5, C.c_int(self.frame_skip),
                                   C.c_double(self.dt), C.c_int(self.max_steps), C.c_double(self.robot_speed),
                                   d.objs, C.c_int(d.n), C.byref(o))
            return o
        lib().orc_step(C.byref(self.m.c), C.byref(self.dp), C.byref(self.s), C.byref(self.step_count),
                       C.byref(self.px), C.byref(self.pz), a, C.c_int(self.action_mode), C.c_double(self.wheel_dist),
                       self.env5, C.c_int(self.frame_skip), C.c_double(self.dt), C.c_int(self.max_steps),
                       C.c_double(self.robot_speed), C.byref(o))
        return o


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))


# ----------------------------------------------------------------------------- raster oracle
class OrrTexture(C.Structure):
    _fields_ = [("w", C.c_int32), ("h", C.c_int32), ("rgba", C.c_void_p)]


class OrrObject(C.Structure):
    _fields_ = [("pos", C.c_float * 3), ("scale", C.c_float), ("y_rot_deg", C.c_float), ("tri_offset", C.c_int32),
                ("tri_count", C.c_int32), ("tex_from", C.c_int32), ("tex_to", C.c_int32), ("seg_tex", C.c_int32)]


class OrrScene(C.Structure):
    _fields_ = [("tile_size", C.c_double), ("grid_w", C.c_int32), ("grid_h", C.c_int32), ("tile_kind", C.c_void_p),
                ("tile_angle", C.c_void_p), ("tile_tex", C.c_void_p), ("n_objects", C.c_int32), ("objects", C.c_void_p),
                ("tri_pos", C.c_void_p), ("tri_nrm", C.c_void_p), ("tri_uv", C.c_void_p), ("tri_col", C.c_void_p),
                ("tri_tex", C.c_void_p), ("n_textures", C.c_int32), ("textures", C.c_void_p),
                ("tex_segment", C.c_void_p), ("agent", OrrObject)]


class OrrEpisode(C.Structure):
    _fields_ = [("cam_height", C.c_float), ("cam_angle_deg", C.c_float), ("cam_fov_y_deg", C.c_float),
                ("cam_noise", C.c_float * 3), ("horizon", C.c_float * 3), ("ambient", C.c_float * 3),
                ("diffuse", C.c_float * 3), ("light_eye", C.c_float * 4), ("ground", C.c_float * 3),
                ("hidden", C.c_uint32 * 8)]


def default_episode(**kw) -> OrrEpisode:
    """Non-randomized values of Simulator.reset() (S:546-614): what dts_reset uses for NULL params."""
    ep = OrrEpisode(0.108, 19.15, 75.0, (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(0.45, 0.82, 1.0),
                    (C.c_float * 3)(0.25, 0.25, 0.25), (C.c_float * 3)(0.35, 0.35, 0.35),
                    (C.c_float * 4)(0, 3, 0, 1), (C.c_float * 3)(0.15, 0.15, 0.15), (C.c_uint32 * 8)())
    for k, v in kw.items():
        cur = getattr(ep, k)
        if hasattr(cur, "__len__"):
            for i, x in enumerate(v):
                cur[i] = x
        else:
            setattr(ep, k, v)
    return ep


class OracleScene:
    """orr_scene for a MapData; array flattening shared with the product's blob builder (data only)."""

    def __init__(self, md):
        from gym_duckietown_b200.lib import MapBlobHolder
        self.holder = h = MapBlobHolder(md)
        k = h.keep
        self.objs = (OrrObject * max(1, len(md.objects)))()
        for i, o in enumerate(md.objects):
            src = k["objs"][i]
            me = k["meshes"][o.mesh_id]
            self.objs[i] = OrrObject((C.c_float * 3)(*[float(v) for v in src.pos]), src.scale, src.y_rot_deg, me.tri_offset,
                                     me.tri_count, -1, -1, me.seg_flat_tex)
        self.texs = (OrrTexture * max(1, len(k["tex_imgs"])))()
        for i, im in enumerate(k["tex_imgs"]):
            self.texs[i] = OrrTexture(im.shape[1], im.shape[0], im.ctypes.data)
        self.c = OrrScene(md.tile_size, md.grid_w, md.grid_h, _p(k["kind"]), _p(k["angle"]), _p(k["tex"]),
                          len(md.objects), C.cast(self.objs, C.c_void_p), _p(k["tpos"]), _p(k["tnrm"]), _p(k["tuv"]),
                          _p(k["tcol"]), _p(k["ttex"]), len(k["tex_imgs"]), C.cast(self.texs, C.c_void_p), _p(k["seg"]),
                          OrrObject((C.c_float * 3)(0, 0, 0), 1.0, 0.0, k["meshes"][h.agent_mesh].tri_offset,
                                    k["meshes"][h.agent_mesh].tri_count, -1, -1, k["meshes"][h.agent_mesh].seg_flat_tex))

    def set_trafficlight_card(self, pattern: int):
        """Which card the mesh shared by all traffic lights shows (TrafficLightObj O:453,462)."""
        src = self.holder.keep["objs"]
        for i in range(self.c.n_objects):
            on = pattern and src[i].alt_tex_from >= 0
            self.objs[i].tex_from, self.objs[i].tex_to = (src[i].alt_tex_from, src[i].alt_tex_to) if on else (-1, -1)

    def set_object_pose(self, i, pos, y_rot_deg):
        """Move object i (a dynamic obstacle of one env) before rendering that env's frame."""
        for k in range(3):
            self.objs[i].pos[k] = float(pos[k])
        self.objs[i].y_rot_deg = float(y_rot_deg)

    def render(self, px, pz, angle, ep: OrrEpisode = None, W=160, H=120, domain_rand=False, lut=None, segment=False,
               top_down=False) -> np.ndarray:
        ep = ep or default_episode()
        if segment or top_down:
            lib().orr_set_render_mode((1 if segment else 0) | (2 if top_down else 0))
            try:
                return self.render(px, pz, angle, ep, W, H, domain_rand, lut)
            finally:
                lib().orr_set_render_mode(0)
        out = np.zeros((H, W, 3), np.uint8)
        lx = ly = None
        if lut is not None:
            lx, ly = np.ascontiguousarray(lut[0], np.float32), np.ascontiguousarray(lut[1], np.float32)
        lib().orr_render(C.byref(self.c), C.c_double(px), C.c_double(pz), C.c_double(angle), C.byref(ep), W, H,
                         int(domain_rand), _p(lx) if lx is not None else None, _p(ly) if ly is not None else None, _p(out))
        return out

    def debug_frame(self, px, pz, angle, ep: OrrEpisode = None, W=160, H=120, domain_rand=False) -> dict:
        """Transforms and lit tile lattices the raster oracle uses for one frame (orr_debug_frame): V f64[12], P f32[4]
        (P00 P11 P22 P23), item_mv f32[items,12], item_n f32[items,9], lattice f32[cells,64,3]; items = ground, every
        grid cell (i outer, j inner), objects."""
        ep = ep or default_episode()
        cells = self.c.grid_w * self.c.grid_h
        items = 1 + cells + self.c.n_objects
        V, P = np.zeros(12), np.zeros(4, np.float32)
        mv, nn = np.zeros((items, 12), np.float32), np.zeros((items, 9), np.float32)
        lat = np.zeros((cells, 64, 3), np.float32)
        lib().orr_debug_frame(C.byref(self.c), C.c_double(px), C.c_double(pz), C.c_double(angle), C.byref(ep), W, H,
                              int(domain_rand), _p(V), _p(P), _p(mv), _p(nn), _p(lat))
        return dict(V=V, P=P, item_mv=mv, item_n=nn, lattice=lat)

    def render_batch(self, px, pz, angle, eps, W=160, H=120, domain_rand=False, lut=None, threads=1) -> np.ndarray:
        n = len(px)
        out = np.zeros((n, H, W, 3), np.uint8)
        arr = (OrrEpisode * n)(*eps)
        a = [np.ascontiguousarray(v, np.float64) for v in (px, pz, angle)]
        lx = ly = None
        if lut is not None:
            lx, ly = np.ascontiguousarray(lut[0], np.float32), np.ascontiguousarray(lut[1], np.float32)
        lib().orr_render_batch(C.byref(self.c), n, _p(a[0]), _p(a[1]), _p(a[2]), arr, W, H, int(domain_rand),
                               _p(lx) if lx is not None else None, _p(ly) if ly is not None else None, _p(out),
                               int(threads))
        return out


class OrcEnv(C.Structure):
    _fields_ = [("s", OrcDynState), ("step_count", C.c_int32), ("px", C.c_double), ("pz", C.c_double),
                ("px0", C.c_double), ("pz0", C.c_double), ("ang0", C.c_double)]


class OracleBatch:
    """n reference-style envs stepped + rendered on host cores (one env per OpenMP task)."""

    def __init__(self, md, px, pz, angle, *, W=160, H=120, action_mode=1, max_steps=1500, threads=None):
        self.om, self.sc = OracleMap(md), OracleScene(md)
        self.n, self.W, self.H = len(px), W, H
        self.envs = (OrcEnv * self.n)()
        for k in range(self.n):
            lib().orc_env_init(C.byref(self.om.c), C.byref(self.envs[k]), C.c_double(px[k]), C.c_double(pz[k]),
                               C.c_double(angle[k]))
        self.eps = (OrrEpisode * self.n)(*[default_episode() for _ in range(self.n)])
        self.dp = default_dyn_params()
        self.env5 = (C.c_double * 5)(1.0, 0.0, 0.0318, 27.0, 1.0)
        self.action_mode, self.max_steps = action_mode, max_steps
        self.threads = threads or os.cpu_count() or 1
        self.obs = np.zeros((self.n, H, W, 3), np.uint8)
        self.reward = np.zeros(self.n, np.float32)
        self.done = np.zeros(self.n, np.uint8)

    def step(self, actions: np.ndarray, render=True):
        a = np.ascontiguousarray(actions, np.float32)
        lib().orc_full_step_batch(C.byref(self.om.c), C.byref(self.sc.c), C.byref(self.dp), self.n, self.envs, _p(a),
                                  self.action_mode, C.c_double(0.102), self.env5, 1, C.c_double(1.0 / 30),
                                  self.max_steps, C.c_double(1.2), self.eps, self.W, self.H, int(render), _p(self.obs),
                                  _p(self.reward), _p(self.done), self.threads)
        return self.obs, self.reward, self.done


class OrcDyn(C.Structure):
    _fields_ = [("kind", C.c_int32), ("active", C.c_int32), ("pos", C.c_double * 3), ("angle", C.c_double),
                ("y_rot", C.c_double), ("corners", (C.c_double * 2) * 4), ("norm", C.c_double * 4),
                ("safety_radius", C.c_double), ("walk_distance", C.c_double), ("vel", C.c_double),
                ("wait_time", C.c_double), ("wiggle", C.c_double), ("time", C.c_double), ("start", C.c_double * 3),
                ("heading", C.c_double * 3)] + [(n, C.c_double) for n in (
                    "follow_dist", "velocity", "gain", "trim", "radius", "k", "limit", "wheel_dist", "robot_width",
                    "robot_length", "freq")] + [("tl_first", C.c_int32), ("shown", C.c_int32)]


class OracleDynamics:
    """The dynamic obstacles of one env (MapData.dyn_objects), stepped by the C oracle."""

    def __init__(self, omap: OracleMap, wiggle=None, freq=None, pattern=None):
        """wiggle / freq / pattern: per dynamic object overrides of what the reference draws from the global RNG."""
        md = omap.md
        self.m, self.n = omap, len(md.dyn_objects)
        self.objs = (OrcDyn * max(1, self.n))()
        for i, d in enumerate(md.dyn_objects):
            o = self.objs[i]
            o.kind, o.active = d.kind, 0
            for k in range(3):
                o.pos[k] = float(d.pos[k]); o.start[k] = float(d.pos[k])
            o.angle = d.angle
            o.y_rot = float(np.rad2deg(d.angle))                       # O:57
            for k in range(4):
                o.corners[k][0], o.corners[k][1] = float(d.corners[k][0]), float(d.corners[k][1])
            for k in range(4):
                o.norm[k] = float(np.ravel(d.axes)[k])
            o.safety_radius, o.walk_distance, o.vel, o.wait_time = d.safety_radius, d.walk_distance, d.vel, d.wait_time
            o.wiggle = d.wiggle if wiggle is None else float(wiggle[i])
            o.freq = d.freq if freq is None else float(freq[i])
            if d.kind == 3:
                o.active = int(d.pattern if pattern is None else pattern[i])
            o.time = 0.0
            o.heading[0], o.heading[1], o.heading[2] = math.cos(d.angle), 0.0, -math.sin(d.angle)   # heading_vec C:222
            (o.follow_dist, o.velocity, o.gain, o.trim, o.radius, o.k, o.limit, o.wheel_dist, o.robot_width,
             o.robot_length) = (d.follow_dist, d.velocity, d.gain, d.trim, d.radius, d.k, d.limit, d.wheel_dist,
                                d.robot_width, d.robot_length)

        tls = [i for i, d in enumerate(md.dyn_objects) if d.kind == 3]
        for i in range(self.n):
            self.objs[i].tl_first = tls[0] if tls else -1
        if tls:
            self.objs[tls[0]].shown = self.objs[tls[-1]].active     # constructors assign in order: the last one shows

    @property
    def shown_card(self) -> int:
        t = self.objs[0].tl_first
        return int(self.objs[t].shown) if t >= 0 else 0

    def step(self, dt=1.0 / 30):
        lib().orc_dyn_step_all(C.byref(self.m.c), self.objs, self.n, C.c_double(dt))

    def collision(self, px, pz, angle) -> bool:
        return bool(lib().orc_dyn_collision(self.objs, self.n, C.c_double(px), C.c_double(pz), C.c_double(angle)))

    def proximity(self, px, pz, angle) -> float:
        return float(lib().orc_dyn_proximity(self.objs, self.n, C.c_double(px), C.c_double(pz), C.c_double(angle)))
