"""Host-side `Simulator.reset()` sampling, draw-for-draw compatible with the reference.

The reference draws every per-episode quantity from `self.np_random`, a
`numpy.random.Generator(PCG64(SeedSequence(seed)))` (simulator.py:1043-1045 via gym.utils.seeding),
in a fixed order (simulator.py:546-736, randomization/randomizer.py:36-91; SURVEY 8a row P0).
`EpisodeSampler` keeps one such generator per env and replays that order with the same numpy calls,
so seeds produce the reference's poses and DR values.  The spawn-rejection predicates
(`_inconvenient_spawn`, `_valid_pose(safety_factor=1.3)`, `get_lane_pos2`) are evaluated by the CUDA
library (`dts_query_poses`) on candidate batches; the stream position afterwards is exactly the
reference's because candidates are drawn from a copy of the bit-generator state and the real
generator is then advanced by the accepted attempt count.
"""
from __future__ import annotations

import copy
import math
from typing import Dict, List, Optional, Sequence

import numpy as np

from .maps import MapData

# constants simulator.py:108-177 and randomizer.py:8-16 / config/default_dr.json
BLUE_SKY = np.array([0.45, 0.82, 1])
WALL_COLOR = np.array([0.64, 0.71, 0.28])
DIM = 0.5
CAMERA_ANGLE, CAMERA_FOV_Y, CAMERA_FLOOR_DIST, WHEEL_DIST = 19.15, 75, 0.108, 0.102
MAX_SPAWN_ATTEMPTS = 5000
_CHUNK = 16
# randomization/config/default_dr.json (== randomizer.py DEFAULT_CONFIG)
DEFAULT_DR_CONFIG = {
    "horz_mode": {"type": "int", "low": 0, "high": 4},
    "light_pos": {"type": "uniform", "low": [-150, 170, -150], "high": [150, 220, 150], "size": 3},
    "camera_noise": {"type": "uniform", "low": -0.005, "high": 0.005, "size": 3},
    "trim": {"type": "normal", "loc": 0, "scale": 0.02},
    "camera_height": {"type": "uniform", "low": 0.92, "high": 1.08},
    "camera_angle": {"type": "uniform", "low": 0.8, "high": 1.2},
    "camera_fov_y": {"type": "uniform", "low": 0.8, "high": 1.2},
}
_DR_REQUIRED = ("camera_angle", "camera_fov_y", "camera_height", "camera_noise", "horz_mode", "light_pos", "trim")


def load_dr_config(cfg) -> dict:
    """`Randomizer(randomization_config_fp=...)` (randomizer.py:19-33): a dict, a JSON file path, or None for
    default_dr.json.  Every key the simulator reads must be present: the reference falls back to
    DEFAULT_CONFIG[k]["default"], which does not exist (KeyError, randomizer.py:84)."""
    if cfg is None:
        return dict(DEFAULT_DR_CONFIG)
    if not isinstance(cfg, dict):
        import json
        with open(cfg) as f:
            cfg = json.load(f)
    missing = [k for k in _DR_REQUIRED if k not in cfg]
    if missing:
        raise KeyError(f"randomization config lacks {missing}: the reference's Randomizer raises KeyError('default') for them")
    return dict(cfg)


def np_random(seed=None) -> np.random.Generator:
    """gym.utils.seeding.np_random for gym>=0.21 (the `.integers` calls at S:654,675 require it)."""
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


class EpisodeSampler:
    def __init__(self, num_envs: int, *, domain_rand: bool, dynamics_rand: bool = False, camera_rand: bool = False,
                 accept_start_angle_deg: float = 60.0, num_tris_distractors: int = 12,
                 color_ground=(0.15, 0.15, 0.15), color_sky=BLUE_SKY, user_tile_start=None, randomization_config=None,
                 nav: bool = False):
        self.n = num_envs
        self.nav = nav   # DuckietownNav.reset: a goal tile drawn after the spawn loop
        self.domain_rand = domain_rand
        self.dynamics_rand = dynamics_rand
        self.camera_rand = camera_rand
        self.accept = accept_start_angle_deg
        self.num_tris = num_tris_distractors
        self.color_ground = np.array(color_ground)
        self.color_sky = np.array(list(color_sky))
        self.user_tile_start = user_tile_start
        self.dr_config = load_dr_config(randomization_config)
        self.dr_keys = sorted(self.dr_config)   # randomizer.py:33
        self.last_horizon = [np.array(self.color_sky, dtype=float) for _ in range(num_envs)]
        self.rngs: List[np.random.Generator] = [np_random(None) for _ in range(num_envs)]
        self.episodes = np.zeros(num_envs, np.int64)

    def seed(self, seeds: Sequence[Optional[int]], envs: Optional[Sequence[int]] = None):
        envs = range(self.n) if envs is None else envs
        for e, s in zip(envs, seeds):
            self.rngs[e] = np_random(s)

    def _perturb(self, rng, val, scale=0.1):  # S:1065-1085
        val = np.array(val)
        if not self.domain_rand:
            return val
        noise = rng.uniform(low=1 - scale, high=1 + scale, size=val.shape)
        if val.size == 4:
            noise[3] = 1
        return val * noise

    def _randomize(self, rng) -> dict:
        """Randomizer.randomize (randomizer.py:36-91): every key in sorted order with the reference's numpy calls."""
        out = {}
        for k in self.dr_keys:
            d = self.dr_config[k]
            size = d.get("size", 1)
            if d["type"] == "int":
                out[k] = rng.integers(low=d["low"], high=d["high"], size=size)
            elif d["type"] == "uniform":
                out[k] = rng.uniform(low=d["low"], high=d["high"], size=size)
            elif d["type"] == "normal":
                out[k] = rng.normal(loc=d["loc"], scale=d["scale"], size=size)
            else:
                raise NotImplementedError("You've specified an unsupported distribution type")
        return out

    def _pre_spawn(self, rng, md: MapData, env: int = 0) -> dict:
        """Everything reset() draws before the start tile (S:546-656), in order."""
        out = {}
        # Randomizer.randomize — keys sorted, drawn whether or not DR is on (randomizer.py:33,46-89)
        st = self._randomize(rng)
        camera_angle, camera_fov_y, camera_height = st["camera_angle"], st["camera_fov_y"], st["camera_height"]
        camera_noise, horz_mode, light_pos_r, trim = st["camera_noise"], st["horz_mode"], st["light_pos"], st["trim"]
        if self.domain_rand:  # S:551-562
            hm = int(horz_mode[0])
            if hm == 0:
                horizon = self._perturb(rng, self.color_sky)
            elif hm == 1:
                horizon = self._perturb(rng, WALL_COLOR)
            elif hm == 2:
                horizon = self._perturb(rng, [0.15, 0.15, 0.15], 0.4)
            elif hm == 3:
                horizon = self._perturb(rng, [0.9, 0.9, 0.9], 0.4)
            else:
                horizon = self.last_horizon[env]   # no branch assigns: the attribute keeps its previous value
            light_pos = np.array([light_pos_r[0], light_pos_r[1], light_pos_r[2], 0.0])  # 3 floats in a 4-array
        else:
            horizon = self.color_sky
            light_pos = np.array([0.0, 3.0, 0.0, 1.0])  # S:570
        ambient = self._perturb(rng, np.array([0.50 * DIM, 0.50 * DIM, 0.50 * DIM, 1]), 0.3)
        diffuse = self._perturb(rng, np.array([0.70 * DIM, 0.70 * DIM, 0.70 * DIM, 1]), 0.99)
        ground = self._perturb(rng, np.array(self.color_ground), 0.3)
        wheel_dist = self._perturb(rng, WHEEL_DIST)
        cam_height, cam_angle, cam_fov = CAMERA_FLOOR_DIST, CAMERA_ANGLE, CAMERA_FOV_Y
        if self.domain_rand or self.camera_rand:  # S:611-614
            cam_height = cam_height * camera_height[0]
            cam_angle = CAMERA_ANGLE * camera_angle[0]
            cam_fov = cam_fov * camera_fov_y[0]
        for _ in range(0, 3 * self.num_tris):  # distractors S:621-629: drawn, never visible (SURVEY R2)
            rng.uniform(low=[-20, -0.6, -20], high=[20, -0.3, 20], size=(3,))
            c = rng.uniform(low=0, high=0.9)
            self._perturb(rng, [c, c, c], 0.1)
        for k in md.tile_kind:  # per-tile colour S:634-645 (no visible effect, SURVEY R4); every cell has a tile
            if k < 0:
                raise ValueError("reference reset() cannot handle maps with empty cells (S:637)")
            self._perturb(rng, [1, 1, 1, 1], 0.2)
        hidden = np.zeros(8, np.uint32)
        for oi, obj in enumerate(md.objects):  # S:648-656
            self._perturb(rng, [1, 1, 1, 1], 0.3)
            if obj.optional and self.domain_rand:
                if not (rng.integers(0, 2) == 0):
                    hidden[oi >> 5] |= np.uint32(1 << (oi & 31))
        self.last_horizon[env] = np.array(horizon, dtype=float)
        out.update(cam_height=cam_height, cam_angle_deg=cam_angle, cam_fov_y_deg=cam_fov,
                   cam_noise=camera_noise if self.domain_rand else np.zeros(3), horizon_color=horizon,
                   light_ambient=ambient[:3], light_diffuse=diffuse[:3], light_pos=light_pos, ground_color=ground,
                   wheel_dist=float(wheel_dist), trim=float(trim[0]) if self.dynamics_rand else 0.0,
                   obj_hidden=hidden)
        return out

    def sample(self, envs: Sequence[int], maps: Sequence[MapData], query) -> Dict[str, np.ndarray]:
        """Draw one reset for each env in `envs` (env e uses map `maps[k]`).
        `query(map_index_in_maps, x, z, angle, safety, hidden) -> (f64[n,4], i32[n,8])` = dts_query_poses.
        Returns dense arrays of length len(envs)."""
        recs = []
        todo = []
        for k, e in enumerate(envs):
            rng, md = self.rngs[e], maps[k]
            r = self._pre_spawn(rng, md, e)
            if self.user_tile_start is not None:  # S:659-666
                ti, tj = self.user_tile_start
                if not (0 <= ti < md.grid_w and 0 <= tj < md.grid_h) or md.tile_kind[tj * md.grid_w + ti] < 0:
                    raise Exception("The tile specified does not exist.")
            elif md.start_tile is not None:
                ti, tj = md.start_tile
            else:
                if not md.drivable_tiles:
                    raise Exception("There are no drivable tiles. Use start_tile or self.user_tile_start")
                ti, tj = md.drivable_tiles[int(rng.integers(0, len(md.drivable_tiles)))]
            r["tile"] = (ti, tj)
            if md.start_pose is not None:  # S:679-688
                r["pos_x"] = ti * md.tile_size + md.start_pose[0][0]
                r["pos_z"] = tj * md.tile_size + md.start_pose[0][2]
                r["angle"] = md.start_pose[1]
            else:
                todo.append(k)
            r["light_stale"] = 0 if self.episodes[e] == 0 else 1  # S:581: identity modelview only at first reset
            self.episodes[e] += 1
            recs.append(r)
        # spawn loop S:692-736, batched across envs in chunks of candidate attempts
        attempts = {k: 0 for k in todo}
        while todo:
            cand = []
            for k in todo:
                rng = self.rngs[envs[k]]
                probe = np.random.Generator(copy.deepcopy(rng.bit_generator))
                ti, tj = recs[k]["tile"]
                ts = maps[k].tile_size
                m = min(_CHUNK, MAX_SPAWN_ATTEMPTS - attempts[k])
                xs, zs, an = np.empty(m), np.empty(m), np.empty(m)
                for a in range(m):
                    xs[a] = probe.uniform(ti, ti + 1) * ts
                    zs[a] = probe.uniform(tj, tj + 1) * ts
                    an[a] = probe.uniform(0, 2 * math.pi)
                cand.append((k, xs, zs, an))
            nxt = []
            by_map: Dict[int, list] = {}
            for c in cand:
                by_map.setdefault(id(maps[c[0]]), []).append(c)
            for group in by_map.values():
                x = np.concatenate([g[1] for g in group]); z = np.concatenate([g[2] for g in group])
                a = np.concatenate([g[3] for g in group])
                hid = np.concatenate([np.repeat(recs[g[0]]["obj_hidden"][None], len(g[1]), 0) for g in group])
                outd, outi = query(group[0][0], x, z, a, 1.3, hid)
                off = 0
                for (k, xs, zs, an) in group:
                    m = len(xs)
                    ok = ((outi[off:off + m, 4] == 0) & (outi[off:off + m, 0] == 1) & (outi[off:off + m, 3] == 1))
                    deg = np.rad2deg(outd[off:off + m, 2])
                    ok &= (-self.accept < deg) & (deg < self.accept)
                    rng = self.rngs[envs[k]]
                    hit = np.flatnonzero(ok)
                    used = (hit[0] + 1) if len(hit) else m
                    ti, tj = recs[k]["tile"]
                    for _ in range(used):  # advance the real stream exactly as the reference would have
                        rng.uniform(ti, ti + 1); rng.uniform(tj, tj + 1); rng.uniform(0, 2 * math.pi)
                    attempts[k] += used
                    if len(hit):
                        recs[k].update(pos_x=xs[hit[0]], pos_z=zs[hit[0]], angle=an[hit[0]])
                    elif attempts[k] >= MAX_SPAWN_ATTEMPTS:
                        recs[k].update(pos_x=1.0, pos_z=1.0, angle=1.0)  # S:732-736 fallback
                    else:
                        nxt.append(k)
                    off += m
            todo = nxt
        if self.nav:   # DuckietownNav.reset (envs/duckietown_env.py:97-111, randint read as integers)
            for k, e in enumerate(envs):
                recs[k]["goal"] = self._draw_goal(self.rngs[e], maps[k], recs[k]["pos_x"], recs[k]["pos_z"])
        keys = ["pos_x", "pos_z", "angle", "wheel_dist", "trim", "cam_height", "cam_angle_deg", "cam_fov_y_deg",
                "cam_noise", "horizon_color", "light_ambient", "light_diffuse", "light_pos", "light_stale",
                "ground_color", "obj_hidden"] + (["goal"] if self.nav else [])
        return {k: np.array([r[k] for r in recs]) for k in keys}

    @staticmethod
    def _draw_goal(rng, md: MapData, x: float, z: float) -> tuple:
        """A drivable tile other than get_grid_coords((x, 0, z)) (S:1134), drawn until one is."""
        if len(md.drivable_tiles) < 2:   # assert len(self.drivable_tiles) > 1, envs/duckietown_env.py:106
            raise ValueError("navigation needs a map with at least two drivable tiles")
        start = (math.floor(x / md.tile_size), math.floor(z / md.tile_size))
        while True:
            goal = tuple(md.drivable_tiles[int(rng.integers(0, len(md.drivable_tiles)))])
            if goal != start:
                return goal
