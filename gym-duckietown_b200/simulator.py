"""Single-env adapters with the reference's `gym.Env` surface (old 4-tuple API), backed by a
one-env `BatchedDuckietownEnv` on the GPU.  Same constructor keywords, attributes and helper methods
callers rely on (SURVEY.md 1 / 8b): simulator.py:188-232 (Simulator), envs/duckietown_env.py
(DuckietownEnv), envs/multimap_env.py (MultiMapEnv).  Observations come back as numpy uint8 HxWx3,
so the reference's wrappers (wrappers.py) work unchanged on top of these classes.  DuckietownLF and DuckietownNav are
the two tasks of envs/duckietown_env.py.
"""
from __future__ import annotations

from collections import namedtuple
from typing import Optional, Tuple

import numpy as np

from . import lib as L
from .gymshim import Env, spaces
from .maps import load_map

LanePosition0 = namedtuple("LanePosition", "dist dot_dir angle_deg angle_rad")


class LanePosition(LanePosition0):  # S:182-185
    def as_json_dict(self):
        return dict(dist=self.dist, dot_dir=self.dot_dir, angle_deg=self.angle_deg, angle_rad=self.angle_rad)


class NotInLane(Exception):
    """Raised when the Duckiebot is not in a lane (exceptions.py:14)."""


DEFAULT_MAP_NAME = "udem1"

# module-level constants and helpers user scripts import from gym_duckietown.simulator (S:118-177, S:2056-2118)
CAMERA_FORWARD_DIST, ROBOT_WIDTH, ROBOT_LENGTH, WHEEL_DIST = 0.066, 0.13 + 0.02, 0.18, 0.102
WINDOW_WIDTH, WINDOW_HEIGHT = 800, 600   # S:100-101
DEFAULT_ROBOT_SPEED, DEFAULT_FRAMERATE, DEFAULT_MAX_STEPS = 1.20, 30, 1500
REWARD_INVALID_POSE = -1000


def get_dir_vec(cur_angle: float) -> np.ndarray:
    """Unit vector the robot points along, x right / z towards the viewer (S:2056-2064)."""
    return np.array([np.cos(cur_angle), 0.0, -np.sin(cur_angle)])


def get_right_vec(cur_angle: float) -> np.ndarray:
    """Unit vector to the robot's right (S:2066-2074)."""
    return np.array([np.sin(cur_angle), 0.0, np.cos(cur_angle)])


def _actual_center(pos, angle) -> np.ndarray:
    """Centre of the robot's footprint: the camera sits CAMERA_FORWARD_DIST ahead of the rear end (S:2102-2110)."""
    return np.asarray(pos, float) + (CAMERA_FORWARD_DIST - ROBOT_LENGTH / 2) * get_dir_vec(angle)


def get_agent_corners(pos, angle) -> np.ndarray:
    """[4,2] (x,z) corners of the robot's bounding box around `_actual_center(pos, angle)` (S:2113-2118, C:9-34)."""
    c, f, r = _actual_center(pos, angle), get_dir_vec(angle), get_right_vec(angle)
    hw, hl = 0.5 * ROBOT_WIDTH, 0.5 * ROBOT_LENGTH
    pts = [c - hw * r - hl * f, c + hw * r - hl * f, c + hw * r + hl * f, c - hw * r + hl * f]
    return np.array([[p_[0], p_[2]] for p_ in pts])


class Simulator(Env):
    metadata = {"render.modes": ["rgb_array"], "video.frames_per_second": 30}
    _action_mode = "pwm"  # Simulator.step takes wheel duty cycles (S:1669)

    def __init__(self, map_name: str = DEFAULT_MAP_NAME, max_steps: int = 1500, draw_curve: bool = False,
                 draw_bbox: bool = False, domain_rand: bool = True, frame_rate: float = 30, frame_skip: int = 1,
                 camera_width: int = 640, camera_height: int = 480, robot_speed: float = 1.2,
                 accept_start_angle_deg=60, full_transparency: bool = False, user_tile_start=None,
                 seed: Optional[int] = None, distortion: bool = False, dynamics_rand: bool = False,
                 camera_rand: bool = False, randomize_maps_on_reset: bool = False, num_tris_distractors: int = 12,
                 color_ground=(0.15, 0.15, 0.15), color_sky=(0.45, 0.82, 1), style: str = "photos",
                 enable_leds: bool = False, device: int = 0, depth: bool = False, labels: bool = False,
                 markings: bool = False, bev: bool = False, flow: bool = False, flow_occlusion: bool = False,
                 bev_visibility: bool = False, scan: bool = False, objects: bool = False,
                 lane_path: bool = False, **env_kwargs):
        if draw_curve or draw_bbox or enable_leds:
            raise NotImplementedError("draw_curve / draw_bbox / enable_leds are debug modes outside the hot path "
                                      "(SURVEY 8f-4)")
        from .batched_env import BatchedDuckietownEnv  # needs torch + CUDA: fail here, loudly, if absent
        self.map_name = map_name
        self.max_steps, self.domain_rand, self.full_transparency = max_steps, domain_rand, full_transparency
        self.frame_rate, self.delta_time, self.frame_skip = frame_rate, 1.0 / frame_rate, frame_skip
        self.camera_width, self.camera_height, self.robot_speed = camera_width, camera_height, robot_speed
        self.accept_start_angle_deg = accept_start_angle_deg
        self.distortion, self.dynamics_rand = distortion, dynamics_rand
        self.seed_value = seed
        self.randomize_maps_on_reset = randomize_maps_on_reset
        map_arg = map_name
        if randomize_maps_on_reset:   # S:373-378: every map file except calibration* / regress*; reset() draws one
            from .maps import list_maps
            self.map_names = [m for m in list_maps() if not m.startswith(("calibration", "regress"))]
            map_arg = self.map_names
            env_kwargs = dict(env_kwargs, randomize_maps_on_reset=True)
        self._env_kwargs = dict(
            device=device, max_steps=max_steps, domain_rand=domain_rand, frame_rate=frame_rate,
            frame_skip=frame_skip, camera_width=camera_width, camera_height=camera_height, robot_speed=robot_speed,
            accept_start_angle_deg=accept_start_angle_deg, user_tile_start=user_tile_start, seed=seed,
            distortion=distortion, dynamics_rand=dynamics_rand, camera_rand=camera_rand,
            camera_rand_pool=env_kwargs.pop("camera_rand_pool", 1),   # one camera per Simulator (distortion.py:46-47)
            color_ground=color_ground, color_sky=color_sky, num_tris_distractors=num_tris_distractors,
            action_mode=self._action_mode, depth=depth, labels=labels, markings=markings, bev=bev, flow=flow,
            flow_occlusion=flow_occlusion, bev_visibility=bev_visibility, scan=scan, objects=objects, lane_path=lane_path,
            **env_kwargs)
        self._b = BatchedDuckietownEnv(1, map_arg, **self._env_kwargs)
        self._adopt_map()
        self.action_space = spaces.Box(low=-1, high=1, shape=(2,), dtype=np.float32)              # S:309
        self.observation_space = spaces.Box(low=0, high=255, shape=(camera_height, camera_width, 3), dtype=np.uint8)
        self.reward_range = (-1000, 1000)
        self.cam_offset = np.array([0, 0, 0])
        self.last_action = np.array([0, 0])
        self.wheelVels = np.array([0, 0])
        self.timestamp = 0.0
        self.reset()

    def _map_index(self) -> int:
        return int(self._b.map_ids[0]) if not self._b.device_reset else int(self._b.state["map_id"][0].item())

    def _adopt_map(self):
        """Map-dependent attributes of the reference Simulator (S:793-879) for the env's current map."""
        md = self._b.maps[self._map_index()]
        self.road_tile_size, self.grid_width, self.grid_height = md.tile_size, md.grid_w, md.grid_h
        self.drivable_tiles, self.objects = md.drivable_tiles, md.objects
        if self.randomize_maps_on_reset:
            self.map_name = self.map_names[self._map_index()]

    # ------------------------------------------------------------------ gym.Env
    def seed(self, seed=None):
        self._b.sampler.seed([seed])
        return [seed]

    def reset(self, segment: bool = False):
        obs = self._b.reset(render=not segment)
        if segment:   # S:760: the first observation is render_obs(segment=segment)
            obs = self._b.render_obs(segment=True)
        self.timestamp = 0.0
        self._adopt_map()
        return self._obs_numpy(obs)

    def step(self, action):
        import torch
        a = np.asarray(action, dtype=np.float32).reshape(1, 2)
        obs, rew, done, _ = self._b.step(torch.from_numpy(a).to(self._b.device))
        self.timestamp += self.delta_time * self.frame_skip
        self.last_action = np.clip(np.asarray(action, dtype=float), -1, 1) if self._action_mode == "pwm" else np.asarray(action)
        self.wheelVels = self.last_action * self.robot_speed
        o = self._obs_numpy(obs)
        st = self._scalars()
        misc = self.get_agent_info(st)
        code = int(st["done_code"])
        misc["Simulator"]["msg"] = {0: "", 1: "Stopping the simulator because we are at an invalid pose.",
                                    2: "Stopping the simulator because we reached max_steps = %s" % self.max_steps,
                                    3: ""}[code]   # DuckietownNav's arrival sets no message
        return o, float(st["reward"]), bool(code != 0), misc

    def render_obs(self, segment: bool = False):
        return self._obs_numpy(self._b.render_obs(segment=segment))

    def _human_view(self):
        """A second 1-env handle at WINDOW_WIDTH x WINDOW_HEIGHT (S:100-101, 340) put into this env's state: what
        `_render_img(WINDOW_WIDTH, WINDOW_HEIGHT, multi_fbo_human, ...)` draws (S:1988-1996).  It is built with this
        env's keywords and maps (so its records have the same fingerprint), without the fisheye, and takes this env's
        whole state as a snapshot."""
        from .batched_env import BatchedDuckietownEnv
        if getattr(self, "_human", None) is None:
            kw = dict(self._env_kwargs, camera_width=WINDOW_WIDTH, camera_height=WINDOW_HEIGHT, distortion=False,
                      terminal_obs=False, depth=False, labels=False, markings=False, bev=False, flow=False,
                      flow_occlusion=False, bev_visibility=False, scan=False, objects=False, lane_path=False)
            self._human = BatchedDuckietownEnv(1, list(self._b.maps), **kw)
        self._human.load_state(self._b.save_state())
        return self._human

    def render(self, mode: str = "human", close: bool = False, segment: bool = False):
        """S:1974-2054.  "rgb_array" / "top_down" return the WINDOW_WIDTH x WINDOW_HEIGHT image; "human" / "free_cam" open a
        pyglet window in the reference (interactive UI: not provided).  The fisheye model is not applied to this view."""
        assert mode in ["human", "top_down", "free_cam", "rgb_array"]
        if close:
            return None
        if mode in ("human", "free_cam"):
            raise NotImplementedError("window rendering (human / free_cam) is interactive UI; use rgb_array or top_down")
        h = self._human_view()
        return h.render_obs(segment=segment, top_down=(mode == "top_down"))[0].cpu().numpy()

    def close(self):
        if getattr(self, "_human", None) is not None:
            self._human.close()
        self._b.close()

    # ------------------------------------------------------------------ state the reference exposes as attributes
    def _obs_numpy(self, obs):
        return obs[0].cpu().numpy()

    def _scalars(self):
        return {k: v[0].item() for k, v in self._b.state.items()}

    @property
    def undistort(self) -> bool:
        """S:361, set by the reference's UndistortWrapper: True returns pinhole frames instead of fisheye ones (S:1969-1970),
        which that wrapper then remaps on the host.  Kept by the batched env (BatchedDuckietownEnv.undistort)."""
        return self._b.undistort

    @undistort.setter
    def undistort(self, value: bool):
        self._b.undistort = value

    @property
    def depth(self) -> Optional[np.ndarray]:
        """With depth=True: float32 [camera_height, camera_width], the depth image of the observation last returned by
        reset / step / render_obs (BatchedDuckietownEnv.depth); else None."""
        d = self._b.depth
        return None if d is None else d[0].cpu().numpy()

    @property
    def labels(self) -> Optional[np.ndarray]:
        """With labels=True: int16 [camera_height, camera_width], the label image of the observation last returned by
        reset / step / render_obs (BatchedDuckietownEnv.labels, named by BatchedDuckietownEnv.label_table); else None."""
        lb = self._b.labels
        return None if lb is None else lb[0].cpu().numpy()

    @property
    def markings(self) -> Optional[np.ndarray]:
        """With markings=True: uint8 [camera_height, camera_width], the lane-marking image of the observation last
        returned by reset / step / render_obs (BatchedDuckietownEnv.markings, named by MARKING_NAMES); else None."""
        mk = self._b.markings
        return None if mk is None else mk[0].cpu().numpy()

    @property
    def bev_labels(self) -> Optional[np.ndarray]:
        """With bev=True: int16 [height, width], the bird's-eye label grid around the agent in the state last returned by
        reset / step / render_obs (BatchedDuckietownEnv.bev_labels, named by BatchedDuckietownEnv.label_table); else
        None.  `bev_shape`, `bev_cell` and `bev_origin` pass through to the batched env."""
        g = self._b.bev_labels
        return None if g is None else g[0].cpu().numpy()

    @property
    def bev_markings(self) -> Optional[np.ndarray]:
        """With bev=True: uint8 [height, width], the lane paint under each cell of the bird's-eye grid
        (BatchedDuckietownEnv.bev_markings, named by MARKING_NAMES); else None."""
        g = self._b.bev_markings
        return None if g is None else g[0].cpu().numpy()

    @property
    def scan_range(self) -> Optional[np.ndarray]:
        """With scan=True: float32 [scan_rays], how far each ray of the range scan around the agent runs in the state last
        returned by reset / step / render_obs (BatchedDuckietownEnv.scan_range); else None.  `scan_rays`, `scan_fov`,
        `scan_range` and `scan_origin` pass through to the batched env."""
        r = self._b.scan_range
        return None if r is None else r[0].cpu().numpy()

    @property
    def scan_hit(self) -> Optional[np.ndarray]:
        """With scan=True: int16 [scan_rays], what stops each ray, named by BatchedDuckietownEnv.label_table
        (BatchedDuckietownEnv.scan_hit); else None."""
        h = self._b.scan_hit
        return None if h is None else h[0].cpu().numpy()

    @property
    def object_boxes3d(self) -> Optional[np.ndarray]:
        """With objects=True: float32 [O, 7], every object's 3D box around the agent (forward, right, up of its centre,
        length, width, height, yaw) in the state last returned by reset / step / render_obs
        (BatchedDuckietownEnv.object_boxes3d); else None."""
        b = self._b.object_boxes3d
        return None if b is None else b[0].cpu().numpy()

    @property
    def object_state(self) -> Optional[np.ndarray]:
        """With objects=True: uint8 [O], each slot's OBJECT_STATE_NAMES value (BatchedDuckietownEnv.object_state);
        else None."""
        s = self._b.object_state
        return None if s is None else s[0].cpu().numpy()

    @property
    def object_corners_px(self) -> Optional[np.ndarray]:
        """With objects=True: float32 [O, 9, 2], where each box's 8 corners and centre land in the frame last returned
        (BatchedDuckietownEnv.object_corners_px); else None."""
        c = self._b.object_corners_px
        return None if c is None else c[0].cpu().numpy()

    @property
    def lane_path(self) -> Optional[np.ndarray]:
        """With lane_path=True: float32 [K, 3], the lane path ahead of the agent (forward, right, yaw of each point) in
        the state last returned by reset / step / render_obs (BatchedDuckietownEnv.lane_path); else None."""
        p = self._b.lane_path
        return None if p is None else p[0].cpu().numpy()

    @property
    def lane_path_count(self) -> Optional[int]:
        """With lane_path=True: how many of lane_path's points were found (BatchedDuckietownEnv.lane_path_count);
        else None."""
        c = self._b.lane_path_count
        return None if c is None else int(c[0].item())

    @property
    def lane_path_px(self) -> Optional[np.ndarray]:
        """With lane_path=True: float32 [K, 2], where each lane path point lands in the frame last returned
        (BatchedDuckietownEnv.lane_path_px); else None."""
        p = self._b.lane_path_px
        return None if p is None else p[0].cpu().numpy()

    @property
    def flow(self) -> Optional[np.ndarray]:
        """With flow=True: float32 [camera_height, camera_width, 2], the backward flow of the frame last returned by reset /
        step / render_obs — for each pixel, where the surface point it shows was at the start of the last step minus
        where it is now, in pixels, x right and y down; NaN for sky and when there is no earlier frame in the episode
        (BatchedDuckietownEnv.flow); else None.  flow=True also turns on depth and labels."""
        f = self._b.flow
        return None if f is None else f[0].cpu().numpy()

    @property
    def flow_occlusion(self) -> Optional[np.ndarray]:
        """With flow_occlusion=True: uint8 [camera_height, camera_width], whether each pixel of `flow` was in view at its
        previous position, named by OCCLUSION_NAMES (BatchedDuckietownEnv.flow_occlusion); else None.
        flow_occlusion=True also turns on flow, depth and labels."""
        o = self._b.flow_occlusion
        return None if o is None else o[0].cpu().numpy()

    @property
    def bev_visibility(self) -> Optional[np.ndarray]:
        """With bev_visibility=True: uint8 [height, width], whether the frame last returned by reset / step / render_obs
        shows each cell of the bird's-eye grid, named by BEV_VISIBILITY_NAMES (BatchedDuckietownEnv.bev_visibility);
        else None.  bev_visibility=True also turns on bev and labels."""
        v = self._b.bev_visibility
        return None if v is None else v[0].cpu().numpy()

    @property
    def bev_pixels(self) -> Optional[np.ndarray]:
        """With bev_visibility=True: float32 [height, width, 2], where each cell lands in that frame, in camera pixels
        (BatchedDuckietownEnv.bev_pixels); else None."""
        p = self._b.bev_pixels
        return None if p is None else p[0].cpu().numpy()

    @property
    def cur_pos(self):
        s = self._b.state
        return np.array([s["pos_x"][0].item(), 0.0, s["pos_z"][0].item()])

    @property
    def cur_angle(self):
        return self._b.state["angle"][0].item()

    @property
    def step_count(self):
        return int(self._b.state["step_count"][0].item())

    @property
    def speed(self):
        return self._b.state["speed"][0].item()

    @property
    def wheel_dist(self):
        return self._b.state["wheel_dist"][0].item()

    # ------------------------------------------------------------------ helper methods callers use
    def _query(self, pos, angle, safety=1.0):
        outd, outi = self._b.sim.query_poses(self._map_index(), np.array([pos[0]]), np.array([pos[2]]), np.array([angle]), safety, dyn_env=0, stream=self._b._stream())
        return outd[0], outi[0]

    def get_grid_coords(self, abs_pos) -> Tuple[int, int]:  # S:1134
        d, i = self._query(abs_pos, 0.0)
        return int(i[5]), int(i[6])

    def _drivable_pos(self, pos) -> bool:  # S:1411
        return bool(self._query(pos, 0.0)[1][7])

    def _valid_pose(self, pos, angle, safety_factor: float = 1.0) -> bool:  # S:1494
        return bool(self._query(pos, angle, safety_factor)[1][0])

    def _collision_at(self, pos, angle) -> bool:
        """`env._collision(get_agent_corners(pos, angle))` (S:1473 as used by run_tests.py:50)."""
        return bool(self._query(pos, angle)[1][1])

    def proximity_penalty2(self, pos, angle) -> float:  # S:1430
        return float(self._query(pos, angle)[0][3])

    def get_lane_pos2(self, pos, angle) -> LanePosition:  # S:1371
        d, i = self._query(pos, angle)
        if not i[3]:
            raise NotInLane(f"Point not in lane: {pos}")
        return LanePosition(dist=d[0], dot_dir=d[1], angle_deg=float(np.rad2deg(d[2])), angle_rad=d[2])

    def get_agent_info(self, st=None) -> dict:  # S:1586-1627
        st = st or self._scalars()
        info = {"action": list(self.last_action)}
        if self.full_transparency:
            if st["in_lane"]:
                info["lane_position"] = LanePosition(st["lane_dist"], st["lane_dot"], float(np.rad2deg(st["lane_angle_rad"])),
                                                     st["lane_angle_rad"]).as_json_dict()
            info["robot_speed"] = st["speed"]
            info["proximity_penalty"] = st["prox_penalty"]
            info["cur_pos"] = [float(st["pos_x"]), 0.0, float(st["pos_z"])]
            info["cur_angle"] = float(st["angle"])
            info["wheel_velocities"] = [self.wheelVels[0], self.wheelVels[1]]
            info["timestamp"] = self.timestamp
            info["tile_coords"] = [int(st["tile_i"]), int(st["tile_j"])]
        return {"Simulator": info}


class DuckietownEnv(Simulator):
    """[vel, steering] control (envs/duckietown_env.py:9-72); the action map runs inside the step kernel."""
    _action_mode = "vel_steer"

    def __init__(self, gain=1.0, trim=0.0, radius=0.0318, k=27.0, limit=1.0, **kwargs):
        self.gain, self.trim, self.radius, self.k, self.limit = gain, trim, radius, k, limit
        Simulator.__init__(self, gain=gain, trim=trim, radius=radius, k=k, limit=limit, **kwargs)
        self.action_space = spaces.Box(low=np.array([-1, -1]), high=np.array([1, 1]), dtype=np.float32)

    def step(self, action):
        vel, angle = action
        baseline = self.wheel_dist
        obs, reward, done, info = Simulator.step(self, action)
        omega_r = (vel + 0.5 * angle * baseline) / self.radius   # E:50-51, reported in info only
        omega_l = (vel - 0.5 * angle * baseline) / self.radius
        info["DuckietownEnv"] = {"k": self.k, "gain": self.gain, "train": self.trim, "radius": self.radius,
                                 "omega_r": omega_r, "omega_l": omega_l}
        return obs, reward, done, info


class DuckietownLF(DuckietownEnv):
    """The lane-following task (envs/duckietown_env.py:75-86): DuckietownEnv itself."""


class DuckietownNav(DuckietownEnv):
    """The navigation task (envs/duckietown_env.py:89-127) as its author meant it: every reset also draws a goal tile
    other than the start tile, and the episode ends with reward 1000 when the agent reaches it.  The reference's class
    cannot run (its reset and step call themselves, and its Generator has no randint); here they are read as calls to
    DuckietownEnv and `integers`, and the draw and the arrival test run inside the batched env (nav=True)."""

    def __init__(self, **kwargs):
        DuckietownEnv.__init__(self, nav=True, **kwargs)

    @property
    def goal_tile(self) -> dict:
        """The episode's goal tile as the reference's tile dict holds it (S:838-860): "coords" (i, j), one of
        `drivable_tiles`, "kind", "angle" (0..3) and "drivable".  The reference's dict also holds the tile's GL texture
        and colour and its curves, which are not given here; and a new dict is returned on every access, so compare
        goals by their coords, not with `is`."""
        from .maps import TILE_KINDS
        i, j = (int(v) for v in self._b.goal_tile[0].tolist())
        md = self._b.maps[self._map_index()]
        t = j * md.grid_w + i
        return {"coords": (i, j), "kind": TILE_KINDS[int(md.tile_kind[t])], "angle": int(md.tile_angle[t]),
                "drivable": bool(md.tile_drivable[t])}

    def step(self, action):
        obs, reward, done, info = DuckietownEnv.step(self, action)
        info["goal_tile"] = self.goal_tile
        return obs, reward, done, info


class MultiMapEnv(Env):
    """Round-robin over several maps on reset (envs/multimap_env.py:7-91)."""

    def __init__(self, map_names=("loop_only_duckies", "small_loop_only_duckies"), **kwargs):
        self.env_list = [DuckietownEnv(map_name=m, **kwargs) for m in map_names]
        e = self.env_list[0]
        self.action_space, self.observation_space, self.reward_range = e.action_space, e.observation_space, e.reward_range
        self.cur_env_idx = 0

    def seed(self, seed=None):
        for env in self.env_list:
            env.seed(seed)
        return [seed]

    def reset(self):
        self.cur_env_idx = (self.cur_env_idx + 1) % len(self.env_list)
        return self.env_list[self.cur_env_idx].reset()

    def step(self, action):
        return self.env_list[self.cur_env_idx].step(action)

    def render(self, mode="rgb_array", close=False):
        return self.env_list[self.cur_env_idx].render(mode, close)

    def close(self):
        for env in self.env_list:
            env.close()

    @property
    def step_count(self):
        return self.env_list[self.cur_env_idx].step_count
