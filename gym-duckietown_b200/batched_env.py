"""BatchedDuckietownEnv — N independent Duckietown agents per GPU behind the reference's reset/step API.

`step(actions)` is `Simulator.step()` (simulator.py:1669-1683) for every env at once: the action and
observation buffers are caller-visible torch CUDA tensors, the work runs on
`torch.cuda.current_stream()` inside libdtsim.so, nothing synchronises.  Constructor keywords are the
reference's (simulator.py:207-232, envs/duckietown_env.py:15) plus `num_envs`, `device`,
`auto_reset`, `device_reset`, `terminal_obs`, `depth`, `labels`, `markings`, `flow`, `flow_occlusion`,
`camera_rand_pool`, the `bev*` keywords (`bev_visibility` among them), the `scan*` keywords, `objects` and the
`lane_path*` keywords and `nav`.

`camera_rand=True` (with `distortion=True`; without it the flag does nothing, as in the reference, S:352-358) gives the
envs a spread of lenses: `camera_rand_pool` calibrations K, D are drawn once, at construction, within the reference's
ranges (distortion.py:58-83; `distortion.draw_calibrations`, from a stream seeded by `seed`), each gets the fisheye LUT
the reference builds for it, and env g (global index, `env_id_offset + e`) is gathered through calibration
`g % camera_rand_pool` in every render — frames, depth and labels.  camera_rand_pool = num_envs is the reference's one
camera per Simulator.  Resets then apply the drawn camera height / angle / FOV even without domain_rand (S:611-614).
The calibration belongs to the env, not to its state: snapshots do not carry it, and an env keeps its own across
`load_state` / `copy_envs`.  Building the LUTs takes about 0.5 s per calibration at 160x120 and 1-2 s at 640x480.

Under `auto_reset` the observation a step returns for an env whose episode ended is the first frame of its next
episode.  `terminal_obs=True` also keeps the frame the reference's step() returns there (the terminal frame, before
the caller's reset()), in `env.terminal_obs` — what SB3's `terminal_observation` / gymnasium's `final_obs` carry, for
value bootstrapping on truncation.  Only the rows of envs that ended (`done`) are written; the others keep what they
held.  The ended envs are drawn a second time, so the cost grows with how many ended, not with num_envs.  It holds a
second obs-sized buffer: 236 MB at 4096 envs x 160x120 u8, 7.5 GB at 8192 envs x 640x480 u8.

`depth=True` allocates `env.depth`, float32 [num_envs, camera_height, camera_width], which every render (`reset`,
`step`, `render_obs`) fills beside the observation it draws: the eye-space depth in metres of the nearest surface a
pixel's samples see, 0 for sky and for pixels the fisheye / rectification gives no source (dts_set_depth_target).  It is
the depth of the frame just rendered, so it follows `undistort`, the rectification, `top_down` and `segment` (which
leaves it unchanged), and under `auto_reset` an ended env's row is its next episode's first frame, as in `obs`.  It stays
at the camera size and in this layout under `set_resize` and `set_output_format`.  The depth of the terminal frames
(`terminal_obs=True`) is not kept, and the multi-GPU gathers carry observations only.

`labels=True` allocates `env.labels`, int16 [num_envs, camera_height, camera_width], filled by the same renders: which
draw item each pixel shows (dts_set_label_target) — 0 nothing, 1 the ground, then one value per grid cell, per object of
the map and for the agent's own mesh; `label_table(map_id)` names them.  It is the surface the depth image measures, so
with both on `labels != 0` exactly where `depth != 0`; it follows the render modes, sizes and auto-reset as depth does,
and lighting, textures, domain randomisation and `segment` leave it unchanged.  `object_boxes()` reduces it to every
object's pixel count and bounding box.

`markings=True` allocates `env.markings`, uint8 [num_envs, camera_height, camera_width], filled by the same renders: the
lane paint each pixel shows (dts_set_marking_target), named by MARKING_NAMES — 0 no road tile (sky, ground, objects, no
fisheye source), 1 a road tile's unpainted surface, 2 white, 3 yellow, 4 red — the class of the texel its label winner
samples at the pixel centre.  It needs no label image and follows the render modes, sizes and auto-reset as labels do;
lighting, domain randomisation and `segment` leave it unchanged.

`bev=True` allocates `env.bev_labels`, int16, and `env.bev_markings`, uint8, both [num_envs, height, width] for
`bev_shape=(height, width)`: a bird's-eye grid fixed to each agent (dts_set_bev_target), sampled from the map rather than
rendered.  Row 0 is the farthest ahead and column 0 the leftmost, so it reads like an image of the ground seen from
above with the agent facing up; a cell is `bev_cell` metres, and the agent sits at `bev_origin=(x, y)` in cells, by
default (width / 2, 3 * height / 4): 1.44 m ahead and 0.48 m behind at the defaults.  A cell's label uses the label
image's numbering (`label_table`): the first object whose footprint holds the cell centre (hidden optional objects
skipped, moving obstacles where they are now), else the road tile under it, else 1, the ground; its marking is the
MARKING_NAMES class of the texel under it, 0 off the tiles, objects or not.  Every `step` writes them, with
`render=False` too (under `auto_reset`, an ended env's row is its next episode's first state, as in `obs`), and so
does every render; `render_bev()` writes them alone, e.g. after `reset(render=False)`, `load_state` or `copy_envs`.
They do not depend on the camera, the render modes, sizes or formats, and snapshots and gathers do not carry them.

`scan=True` allocates `env.scan_range`, float32, and `env.scan_hit`, int16, both [num_envs, scan_rays]: a range scan
around each agent (dts_set_scan_target), cast on the map rather than rendered.  Ray k leaves at fov * (0.5 - (k + 0.5)
/ scan_rays) to the left of the heading, for `scan_fov` radians (2 pi by default: the full circle), so ray 0 is the
leftmost and one ray points straight ahead; the rays start `scan_origin=(forward, right)` metres from the agent's
position.  `scan_range` holds how far each ray runs before it meets an object's footprint (hidden optional objects
skipped, moving obstacles where they are now) or ground the reference does not drive on (an empty cell, a tile that is
not drivable, off the map), up to `scan_range` metres (2.0 by default); 0 when the origin itself is blocked.  `scan_hit`
names what stopped it in the label image's numbering (`label_table`): the object, the tile that is not drivable, 1
for an empty cell or off the map, 0 for nothing within range.  Every `step` writes them, with `render=False` too
(under `auto_reset`, an ended env's row is its next episode's first state), and so does every render;
`render_scan()` writes them alone.  They do not depend on the camera, the render modes, sizes or formats, and
snapshots and gathers do not carry them.

`flow=True` allocates `env.flow`, float32 [num_envs, camera_height, camera_width, 2], filled by the same renders: the
backward motion flow (dts_set_flow_target) — for each pixel, (dx, dy) in pixels, x right and y down, from where the
surface point it shows is now to where it was in the previous frame, the camera and scene at the start of the env's
last `step`.  It is computed from the depth and label images, so it turns on `depth` and `labels` (allocating
`env.depth` and `env.labels` if they were not asked for); the ground, tiles, static objects and traffic lights stay put,
moving obstacles and the agent's own mesh (top-down) move with their poses.  Under the fisheye both ends go through the
env's camera model's forward map (`camera_model(s).mapx / mapy`).  NaN for sky, for points behind the previous camera,
and for every pixel of an env without a previous frame in its episode: after `reset` (host or device), in the rows
auto-reset respawned, and after `load_state` / `copy_envs` until the next step.  A point hidden in the previous frame
still gets its motion; `flow_occlusion` says which were in view.  `render_obs()` after a step gives the step's flow
again, and after `step(render=False)` that step's.  It stays at the camera size and in this layout under `set_resize`
and `set_output_format`; a flow env refuses `set_rectification`, whose remap has no forward map.  Snapshots and gathers
do not carry it.

`flow_occlusion=True` allocates `env.flow_occlusion`, uint8 [num_envs, camera_height, camera_width], written with
`env.flow` (dts_set_occlusion_target; it turns on `flow`, and through it `depth` and `labels`): whether each pixel's
surface point was in view at its position q = pixel centre + flow in the previous frame, named by OCCLUSION_NAMES —
0 none (flow is NaN), 1 visible (one of the four pixels around q showed the same item there, and a mesh at the
point's depth within 2 %), 2 occluded (something else was there), 3 outside (q leaves the frame), 4 unknown (the
previous frame was never rendered in this view, e.g. after `step(render=False)`).  Under the fisheye most points that
leave the view have NaN flow, so 0.  The library keeps the previous frames itself, two depth and label images per env
(12 bytes per camera pixel: 944 MB at 4096 envs of 160 x 120), so `render_obs()` after a step repeats the step's mask,
and a `render_obs(top_down=True)` between two steps leaves the next step's mask intact.  The terminal frames' masks are
not kept; `load_state`, `copy_envs` and a map upload forget the envs' previous frames.

`bev_visibility=True` allocates `env.bev_visibility`, uint8 [num_envs, height, width], and `env.bev_pixels`, float32
[num_envs, height, width, 2], in the bird's-eye grid's shape (dts_set_bev_visibility_target; it turns on `bev` and
`labels`): for each cell, whether the frame in `obs` shows it and where.  The cell's surface point — its centre on the
road tile or on the ground quad, 8 mm lower (for an object cell, the surface under the object) — is projected through
that frame's camera, and under the fisheye through the env's forward map, to q in camera pixels (pixel centres at +0.5,
as `flow`), which `bev_pixels` holds.  `bev_visibility` names the answer by BEV_VISIBILITY_NAMES: 0 unknown (no frame
was drawn: `step(render=False)`, `render_bev()`), 1 visible (one of the four pixels around q shows the cell's grid
label), 3 outside (behind the camera, beyond its near or far plane, off the frame, off the forward map, or all four
pixels show nothing: sky or no fisheye source), 2 occluded (something else is in front of it).  `bev_pixels` is NaN
for unknown and outside.  Under `auto_reset` a row matches its `obs` row.  A visibility env refuses
`set_rectification`, whose remap has no forward map.  `frame_cameras()` returns every env's camera of its last frame,
on the device, to turn `bev_pixels` or `depth` into rays.  Snapshots and gathers do not carry them.

`objects=True` allocates, for O = the most objects any of the env's maps has (object_boxes()'s O), `env.object_boxes3d`,
float32 [num_envs, O, 7], `env.object_state`, uint8 [num_envs, O], and `env.object_corners_px`, float32 [num_envs, O,
9, 2] (dts_set_object_target): every object's 3D box around each agent, slot o being object o of the env's map.  A box
is the object's footprint of the bird's-eye map (moving obstacles where they are now), raised over the mesh's height;
its row holds the centre's (forward, right, up) in metres from the agent, as the bird's-eye grid's axes, then length
(along the object's heading; for a Duckiebot that has turned, its collision box's robot_length), width, height and yaw,
the object's heading minus the agent's in (-pi, pi], counter-clockwise from above.  `object_state` names each slot by OBJECT_STATE_NAMES: 0 none (the map has fewer
objects; the box is NaN), 1 shown, 2 hidden this episode (the box is still given: the reference still collides with
it).  `object_corners_px` holds where the box's 8 corners (the four footprint corners at the bottom, then at the top)
and its centre land in the frame in `obs`, in camera pixels as `bev_pixels`: NaN behind the camera or beyond its near
or far plane, kept outside the frame for the pinhole and top-down views, NaN where the fisheye's forward map has no
value; every point NaN after `step(render=False)`, under the rectification and in `render_objects()`, which writes the
boxes and states alone, e.g. after `reset(render=False)`, `load_state` or `copy_envs`.  Every `step` and render writes
them, last in the call; under `auto_reset` a row matches its `obs` row.  Snapshots and gathers do not carry them.

`lane_path=True` allocates, for K = `lane_path_points` (1 to 64, default 16), `env.lane_path`, float32 [num_envs, K, 3],
`env.lane_path_count`, int16 [num_envs], and `env.lane_path_px`, float32 [num_envs, K, 2] (dts_set_lane_path_target):
the lane ahead of each agent as points on its lane's centre curve, found by the reference's closest_curve_point.  Point
0 is the closest point to the agent for its heading, the anchor of the lane pose; each later point is the closest point
to a step of `lane_path_spacing` metres (0 < spacing <= 1, default 0.1) along the previous point's tangent, so the
spacing is nominal.  A row holds the point's (forward, right) in metres from the agent, as `object_boxes3d`'s centre,
then the yaw of the lane's tangent there against the agent's heading in (-pi, pi], counter-clockwise from above.
`lane_path_count` says how many points were found: the walk stops at K or where it leaves the drivable tiles (0 when
the agent is off them); later rows are NaN.  On 3-way and 4-way tiles the curve best aligned with the heading is taken,
as the reference's rule does, and it can switch curves within a tile: the path does not choose a route.
`lane_path_px` holds where each point lands in the frame in `obs`, in camera pixels as `object_corners_px`, NaN as
there: after `step(render=False)`, under the rectification and in `render_lane_path()`, which writes the points and
counts alone.  Every `step` and render writes them, last in the call; under `auto_reset` a row matches its `obs` row.
Snapshots and gathers do not carry them.

`nav=True` poses the reference's navigation task, DuckietownNav (envs/duckietown_env.py:89-127, its two calls to itself
read as calls to DuckietownEnv and its `randint` as `integers`), for every env: each reset, host or device, draws a
goal tile from the env's own stream after everything else the reset draws, uniformly among the map's drivable tiles
and again until it is not the tile the agent starts on; `env.goal_tile`, int16 [num_envs, 2], holds (i, j).  A step
that ends on the goal tile ends the episode with reward 1000 (1010 under the `dt` reward) and done_code 3,
"goal-reached" (DONE_CODE_NAMES), whatever the step would have ended with otherwise; auto-reset and `terminal_obs`
then treat it as any other ended episode.  Every map needs at least two drivable tiles and at most 255 tiles a side.
The goal is part of the env's state: snapshots carry it.  Without `nav` nothing is drawn and no goal is tested.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import lib as L
from .assets import MARKING_NAMES  # noqa: F401  (the names of env.markings' values)
from .lib import BEV_VISIBILITY_NAMES  # noqa: F401  (the names of env.bev_visibility's values)
from .lib import DONE_CODE_NAMES  # noqa: F401  (the names of the done codes)
from .lib import OBJECT_STATE_NAMES  # noqa: F401  (the names of env.object_state's values)
from .lib import OCCLUSION_NAMES  # noqa: F401  (the names of env.flow_occlusion's values)
from .episode import EpisodeSampler
from .maps import TILE_KINDS, MapData, load_map


def label_table(md: MapData) -> list:
    """What each label value of the map stands for, indexed by the value (render spec item 10): ("none",), ("ground",),
    ("tile", i, j, kind) for every grid cell (i outer, j inner; kind is None for an empty cell, whose label never
    appears), ("object", o, kind) for entry o of the map's object list, and ("agent",) last."""
    table = [("none",), ("ground",)]
    for i in range(md.grid_w):
        for j in range(md.grid_h):
            k = int(md.tile_kind[j * md.grid_w + i])
            table.append(("tile", i, j, TILE_KINDS[k] if k >= 0 else None))
    table += [("object", o, ob.kind) for o, ob in enumerate(md.objects)]
    table.append(("agent",))
    return table


class BatchedDuckietownEnv:
    def __init__(self, num_envs: int, map_name: Union[str, Sequence[str]] = "udem1", *, device: int = 0,
                 max_steps: int = 1500, domain_rand: bool = True, frame_rate: float = 30, frame_skip: int = 1,
                 camera_width: int = 640, camera_height: int = 480, robot_speed: float = 1.2,
                 accept_start_angle_deg: float = 60, user_tile_start=None, seed: Optional[int] = None,
                 distortion: bool = False, dynamics_rand: bool = False, camera_rand: bool = False,
                 color_ground=(0.15, 0.15, 0.15), color_sky=(0.45, 0.82, 1), num_tris_distractors: int = 12,
                 gain=1.0, trim=0.0, radius=0.0318, k=27.0, limit=1.0,
                 action_mode: str = "vel_steer", auto_reset: bool = False, device_reset: bool = False,
                 cycle_maps: bool = False, env_id_offset: int = 0, tessellate_tiles: bool = False,
                 randomize_maps_on_reset: bool = False, randomization_config=None, terminal_obs: bool = False,
                 depth: bool = False, labels: bool = False, camera_rand_pool: int = 16, markings: bool = False,
                 bev: bool = False, bev_shape=(64, 64), bev_cell: float = 0.03, bev_origin=None, flow: bool = False,
                 flow_occlusion: bool = False, bev_visibility: bool = False, scan: bool = False, scan_rays: int = 64,
                 scan_fov: float = 2 * np.pi, scan_range: float = 2.0, scan_origin=(0.0, 0.0), objects: bool = False,
                 lane_path: bool = False, lane_path_points: int = 16, lane_path_spacing: float = 0.1,
                 nav: bool = False):
        if not torch.cuda.is_available():
            raise L.DtsError("BatchedDuckietownEnv needs a CUDA device; there is no CPU implementation")
        camera_rand = bool(camera_rand and distortion)   # S:353-356: camera_rand only with distortion
        flow = flow or flow_occlusion                    # the mask is taken with the flow image
        depth, labels = depth or flow, labels or flow    # the flow image is taken from both
        bev, labels = bev or bev_visibility, labels or bev_visibility   # the visibility compares their labels
        if camera_rand and not 1 <= int(camera_rand_pool) <= 65536:
            raise ValueError(f"camera_rand_pool must be 1 to 65536, not {camera_rand_pool}")
        self.camera_rand = camera_rand
        names = [map_name] if isinstance(map_name, (str, MapData)) else list(map_name)
        self.maps: List[MapData] = [n if isinstance(n, MapData) else load_map(n) for n in names]   # parsed maps pass through
        self.num_envs, self.device_index = num_envs, device
        self.device = torch.device("cuda", device)
        self.camera_width, self.camera_height = camera_width, camera_height
        self.max_steps, self.domain_rand, self.distortion = max_steps, domain_rand, distortion
        self.frame_rate, self.delta_time, self.frame_skip = frame_rate, 1.0 / frame_rate, frame_skip
        self.robot_speed = robot_speed
        self.auto_reset, self.device_reset, self.cycle_maps = auto_reset, device_reset, cycle_maps
        self.randomize_maps_on_reset = randomize_maps_on_reset
        if cycle_maps and randomize_maps_on_reset:
            raise ValueError("cycle_maps (MultiMapEnv) and randomize_maps_on_reset are two different reset policies")
        if auto_reset and not device_reset:
            raise ValueError("auto_reset re-spawns on the device: pass device_reset=True")
        if terminal_obs and not auto_reset:
            raise ValueError("terminal_obs keeps the frame auto_reset replaces: without auto_reset, step() already "
                             "returns the terminal frame")
        self._keep_terminal = terminal_obs
        flags = (L.FLAG_AUTO_RESET if auto_reset else 0) | (L.FLAG_DOMAIN_RAND if domain_rand else 0) | \
                (L.FLAG_DISTORTION if distortion else 0) | (L.FLAG_DYNAMICS_RAND if dynamics_rand else 0) | \
                (L.FLAG_TESSELLATE if tessellate_tiles else 0) | (L.FLAG_CAMERA_RAND if camera_rand else 0) | \
                (L.FLAG_NAV if nav else 0)
        self.nav = nav
        self.cfg = L.default_config(
            num_envs=num_envs, device=device, cam_width=camera_width, cam_height=camera_height, max_steps=max_steps,
            frame_skip=int(frame_skip), action_mode=L.ACTION_VEL_STEER if action_mode == "vel_steer" else L.ACTION_PWM,
            flags=flags, max_maps=len(self.maps), cycle_maps=len(self.maps) if cycle_maps else 0,
            random_maps=len(self.maps) if randomize_maps_on_reset else 0,
            frame_rate=float(frame_rate), robot_speed=robot_speed, accept_start_angle_deg=float(accept_start_angle_deg),
            gain=gain, trim=trim, radius=radius, k=k, limit=limit, seed=0 if seed is None else int(seed),
            env_id_offset=env_id_offset, num_tris_distractors=int(num_tris_distractors),
            color_sky=tuple(color_sky), color_ground=tuple(color_ground))
        if randomization_config is not None:   # Randomizer(randomization_config_fp=...) randomizer.py:19-33
            from .episode import load_dr_config
            L.set_dr_ops(self.cfg, L.dr_ops_from_config(load_dr_config(randomization_config)))
        self.sim = L.Sim(self.cfg)
        for i, md in enumerate(self.maps):
            self.sim.upload_map(i, md, tuple(user_tile_start) if user_tile_start else None)
        # camera_rand: the calibrations (K, D) of the pool and the one of every env, else None
        self.calibrations: Optional[list] = None
        self.calibration_of_env: Optional[np.ndarray] = None
        if camera_rand:
            from .distortion import Distortion, draw_calibrations
            self.calibrations = draw_calibrations(int(camera_rand_pool), seed)
            self.camera_models = [Distortion(camera_width, camera_height, K, D) for K, D in self.calibrations]
            self.calibration_of_env = (env_id_offset + np.arange(num_envs)) % len(self.calibrations)
            self.sim.set_fisheye_luts(np.stack([m.rmapx for m in self.camera_models]),
                                      np.stack([m.rmapy for m in self.camera_models]), self.calibration_of_env)
        elif distortion:
            from .distortion import Distortion
            self.camera_model = Distortion(camera_width, camera_height)
            self.sim.set_fisheye_lut(self.camera_model.rmapx, self.camera_model.rmapy)
        with torch.cuda.device(self.device):
            self.obs = torch.zeros((num_envs, camera_height, camera_width, 3), dtype=torch.uint8, device=self.device)
            # the terminal frames of the envs that ended on a step (terminal_obs=True), in obs's shape and dtype
            self.terminal_obs: Optional[torch.Tensor] = torch.zeros_like(self.obs) if terminal_obs else None
            # the depth image of the frames in obs (depth=True); the renders write it on the device
            self.depth: Optional[torch.Tensor] = torch.zeros(
                (num_envs, camera_height, camera_width), dtype=torch.float32, device=self.device) if depth else None
            # the label image of the frames in obs (labels=True); the renders write it on the device
            self.labels: Optional[torch.Tensor] = torch.zeros(
                (num_envs, camera_height, camera_width), dtype=torch.int16, device=self.device) if labels else None
            # the lane-marking image of the frames in obs (markings=True); the renders write it on the device
            self.markings: Optional[torch.Tensor] = torch.zeros(
                (num_envs, camera_height, camera_width), dtype=torch.uint8, device=self.device) if markings else None
            # the bird's-eye grids (bev=True); every step and render writes them on the device
            bh, bw = (int(v) for v in bev_shape)
            self.bev_labels: Optional[torch.Tensor] = torch.zeros(
                (num_envs, bh, bw), dtype=torch.int16, device=self.device) if bev else None
            self.bev_markings: Optional[torch.Tensor] = torch.zeros(
                (num_envs, bh, bw), dtype=torch.uint8, device=self.device) if bev else None
            # the backward flow of the frames in obs (flow=True); the renders write it on the device
            self.flow: Optional[torch.Tensor] = torch.zeros(
                (num_envs, camera_height, camera_width, 2), dtype=torch.float32, device=self.device) if flow else None
            # which of those pixels were in view in the previous frame (flow_occlusion=True), OCCLUSION_NAMES
            self.flow_occlusion: Optional[torch.Tensor] = torch.zeros(
                (num_envs, camera_height, camera_width), dtype=torch.uint8, device=self.device) if flow_occlusion else None
            # whether the frames in obs show each cell of the grid, and where (bev_visibility=True), BEV_VISIBILITY_NAMES
            self.bev_visibility: Optional[torch.Tensor] = torch.zeros(
                (num_envs, bh, bw), dtype=torch.uint8, device=self.device) if bev_visibility else None
            self.bev_pixels: Optional[torch.Tensor] = torch.zeros(
                (num_envs, bh, bw, 2), dtype=torch.float32, device=self.device) if bev_visibility else None
            # the range scans (scan=True); every step and render writes them on the device
            self.scan_range: Optional[torch.Tensor] = torch.zeros(
                (num_envs, int(scan_rays)), dtype=torch.float32, device=self.device) if scan else None
            self.scan_hit: Optional[torch.Tensor] = torch.zeros(
                (num_envs, int(scan_rays)), dtype=torch.int16, device=self.device) if scan else None
            # the object boxes (objects=True), OBJECT_STATE_NAMES; every step and render writes them on the device
            n_obj = self._max_objects()
            self.object_boxes3d: Optional[torch.Tensor] = torch.full(
                (num_envs, n_obj, 7), float("nan"), dtype=torch.float32, device=self.device) if objects else None
            self.object_state: Optional[torch.Tensor] = torch.zeros(
                (num_envs, n_obj), dtype=torch.uint8, device=self.device) if objects else None
            self.object_corners_px: Optional[torch.Tensor] = torch.full(
                (num_envs, n_obj, 9, 2), float("nan"), dtype=torch.float32, device=self.device) if objects else None
            # the lane path (lane_path=True); every step and render writes it on the device
            n_pts = int(lane_path_points)
            self.lane_path: Optional[torch.Tensor] = torch.full(
                (num_envs, n_pts, 3), float("nan"), dtype=torch.float32, device=self.device) if lane_path else None
            self.lane_path_count: Optional[torch.Tensor] = torch.zeros(
                num_envs, dtype=torch.int16, device=self.device) if lane_path else None
            self.lane_path_px: Optional[torch.Tensor] = torch.full(
                (num_envs, n_pts, 2), float("nan"), dtype=torch.float32, device=self.device) if lane_path else None
            self.reward = torch.zeros(num_envs, dtype=torch.float32, device=self.device)
            self._done_u8 = torch.zeros(num_envs, dtype=torch.uint8, device=self.device)
            self.state: Dict[str, torch.Tensor] = {
                k_: torch.as_tensor(v, device=self.device) for k_, v in self.sim.state_arrays().items()}
            # the goal tiles (nav=True), library-owned uint8 [num_envs] each
            self._goal = {k_: torch.as_tensor(v, device=self.device) for k_, v in self.sim.goal_arrays().items()}
        self.sampler = EpisodeSampler(
            num_envs, domain_rand=domain_rand, dynamics_rand=dynamics_rand, camera_rand=camera_rand,
            accept_start_angle_deg=accept_start_angle_deg,
            num_tris_distractors=num_tris_distractors, color_ground=color_ground, color_sky=color_sky,
            user_tile_start=user_tile_start, randomization_config=randomization_config, nav=nav)
        self.map_ids = np.zeros(num_envs, np.int32)
        self._first_reset = True
        self.resize = None
        self.resize_method = None
        self._undistort = False      # Simulator.undistort: no fisheye on any render
        self.rectification = None    # (mapx, mapy) UndistortWrapper installed for reset / step observations
        self.output_format = dict(obs_layout="hwc", obs_dtype="uint8", reward="raw", discrete_actions=False,
                                  action_vel_scale=1.0)
        if depth:
            self.sim.set_depth_target(self.depth.data_ptr())
        if labels:
            self.sim.set_label_target(self.labels.data_ptr())
        if markings:
            self.sim.set_marking_target(self.markings.data_ptr())
        if bev:
            ox, oy = (bw / 2, 3 * bh / 4) if bev_origin is None else (float(v) for v in bev_origin)
            self.bev_config = L.BevConfig(bw, bh, float(bev_cell), float(ox), float(oy))
            self.sim.set_bev_target(self.bev_config, self.bev_labels.data_ptr(), self.bev_markings.data_ptr())
        if scan:
            fwd_off, right_off = (float(v) for v in scan_origin)
            self.scan_config = L.ScanConfig(int(scan_rays), float(scan_fov), float(scan_range), fwd_off, right_off)
            self.sim.set_scan_target(self.scan_config, self.scan_range.data_ptr(), self.scan_hit.data_ptr())
        # the forward maps of the fisheye tables, in the pool's order
        models = self.camera_models if camera_rand else [self.camera_model] if distortion else None
        fwd = (np.stack([m.mapx for m in models]), np.stack([m.mapy for m in models])) if models else ()
        if flow:
            self.sim.set_flow_target(self.flow.data_ptr(), *fwd)
        if flow_occlusion:
            self.sim.set_occlusion_target(self.flow_occlusion.data_ptr())
        if bev_visibility:
            self.sim.set_bev_visibility_target(self.bev_visibility.data_ptr(), self.bev_pixels.data_ptr(), *fwd)
        if objects and n_obj:   # (maps without objects: nothing to write)
            self.sim.set_object_target(n_obj, self.object_boxes3d.data_ptr(), self.object_state.data_ptr(),
                                       self.object_corners_px.data_ptr(), *fwd)
        if lane_path:
            self.sim.set_lane_path_target(n_pts, lane_path_spacing, self.lane_path.data_ptr(),
                                          self.lane_path_count.data_ptr(), self.lane_path_px.data_ptr(), *fwd)
        self.seed(seed)

    def set_output_format(self, obs_layout: Optional[str] = None, obs_dtype: Optional[str] = None,
                          reward: Optional[str] = None, discrete_actions: Optional[bool] = None,
                          action_vel_scale: Optional[float] = None):
        """Fuse the reference's wrapper stack into the step kernels (dts_set_output_format): obs_layout 'hwc' |
        'chw' (ImgWrapper) | 'cwh' (PyTorchObsWrapper), obs_dtype 'uint8' | 'float32' (NormalizeWrapper: /255),
        reward 'raw' | 'dt' (DtRewardWrapper), discrete_actions (DiscreteWrapper: ids in actions[:, 0]),
        action_vel_scale (ActionWrapper: 0.8).  Re-allocates `self.obs` in the new shape / dtype.  A layout or dtype
        other than 'hwc' 'uint8' without a resize costs a staging frame of num_envs x H x W x 3 bytes on the device
        (236 MB at 4096 envs of 160x120, 7.5 GB at 8192 of 640x480): the frame is drawn there and a format pass writes
        `self.obs`.  A failed allocation raises and leaves the previous format in effect."""
        f = self.output_format
        for key, val in (("obs_layout", obs_layout), ("obs_dtype", obs_dtype), ("reward", reward),
                         ("discrete_actions", discrete_actions), ("action_vel_scale", action_vel_scale)):
            if val is not None:
                f[key] = val
        lay = {"hwc": L.OBS_HWC, "chw": L.OBS_CHW, "cwh": L.OBS_CWH}[f["obs_layout"]]
        dt = {"uint8": L.OBS_U8, "float32": L.OBS_F32_UNIT}[f["obs_dtype"]]
        rw = {"raw": L.REWARD_RAW, "dt": L.REWARD_DT}[f["reward"]]
        self.sim.set_output_format(lay, dt, rw, L.ACTIONS_DISCRETE3 if f["discrete_actions"] else L.ACTIONS_CONTINUOUS,
                                   f["action_vel_scale"])
        self._alloc_obs()
        return self

    @property
    def obs_size(self):
        """(height, width) of the observations the env emits: the camera's, or the fused ResizeWrapper's target."""
        return (self.resize[1], self.resize[0]) if self.resize else (self.camera_height, self.camera_width)

    def _alloc_obs(self):
        f = self.output_format
        H, W = self.obs_size
        shape = {"hwc": (H, W, 3), "chw": (3, H, W), "cwh": (3, W, H)}[f["obs_layout"]]
        with torch.cuda.device(self.device):
            self.obs = torch.zeros((self.num_envs,) + shape, device=self.device,
                                   dtype=torch.uint8 if f["obs_dtype"] == "uint8" else torch.float32)
            if self._keep_terminal:
                self.terminal_obs = torch.zeros_like(self.obs)

    RESIZE_METHODS = {"cv2_cubic": L.RESIZE_CV2_CUBIC, "pil_bilinear": L.RESIZE_PIL_BILINEAR}

    def set_resize(self, resize_w: Optional[int], resize_h: Optional[int], method: str = "cv2_cubic"):
        """A resize wrapper on the device: render at the camera size, emit `resize_w` x `resize_h` observations in the
        current layout / dtype.  method 'cv2_cubic': src/gym_duckietown/wrappers.py:111-141's ResizeWrapper
        (cv2.INTER_CUBIC's 8-bit fixed-point arithmetic); 'pil_bilinear': learning/utils/wrappers.py:39-54's
        (scipy.misc.imresize = Pillow's bilinear, bit-exact; targets of at least 1/32 of the camera per axis).  None
        switches off.  A target the device refuses raises and leaves the previous setting in effect."""
        if method not in self.RESIZE_METHODS:
            raise ValueError(f"resize method must be one of {sorted(self.RESIZE_METHODS)}, not {method!r}")
        resize = (int(resize_w), int(resize_h)) if resize_w else None
        self.sim.set_resize(*(resize or (0, 0)), filter=self.RESIZE_METHODS[method])
        self.resize, self.resize_method = resize, method if resize else None
        self._alloc_obs()
        return self

    def sim_resize_only(self, frames: torch.Tensor) -> torch.Tensor:
        """The device ResizeWrapper pass on caller-supplied full-size frames u8[N, H, W, 3] -> self.obs."""
        if tuple(frames.shape) != (self.num_envs, self.camera_height, self.camera_width, 3) or frames.dtype != torch.uint8:
            raise ValueError("frames must be uint8 [num_envs, camera_height, camera_width, 3]")
        frames = frames.to(self.device).contiguous()
        self.sim.resize_frames(frames.data_ptr(), self.obs.data_ptr(), self._stream())
        return self.obs

    @property
    def undistort(self) -> bool:
        """Simulator.undistort (S:361), which UndistortWrapper sets: True skips the fisheye gather of a `distortion` env
        (S:1969-1970), so every render is the pinhole frame, and reset / step observations go through the installed
        rectification if there is one.  On an env without distortion it changes nothing."""
        return self._undistort

    @undistort.setter
    def undistort(self, value: bool):
        self._undistort = bool(value)
        self.sim.set_render_mode(**self._base_mode())

    def set_rectification(self, mapx: Optional[np.ndarray], mapy: Optional[np.ndarray]):
        """UndistortWrapper's `cv2.remap(obs, mapx, mapy, INTER_NEAREST)` of reset / step observations, fused into the
        render (dts_set_rectify_lut): each output pixel is rendered at the source pixel the map names.  Applies while
        `undistort` is True; needs an env built with distortion=True.  None, None removes it.  A map the device refuses
        raises and leaves the previous one in effect.  Refused (ValueError) on a flow or bev_visibility env: the
        rectification's remap has no forward map, so its frames would have neither."""
        if self.flow is not None:
            raise ValueError("set_rectification: the flow image cannot follow the rectification (no forward map); "
                             "build the env without flow=True")
        if self.bev_visibility is not None:
            raise ValueError("set_rectification: the bird's-eye visibility cannot follow the rectification (no forward "
                             "map); build the env without bev_visibility=True")
        self.sim.set_rectify_lut(mapx, mapy)
        self.rectification = None if mapx is None and mapy is None else (mapx, mapy)
        self.sim.set_render_mode(**self._base_mode())
        return self

    def _base_mode(self) -> dict:
        """The render mode of reset / step observations."""
        return dict(pinhole=self._undistort, rectify=self._undistort and self.rectification is not None)

    # ------------------------------------------------------------------ gym-like surface
    def seed(self, seed=None):
        """Env k gets seed+k (global index), like one reference env per seed (S:1043-1045)."""
        off = self.cfg.env_id_offset
        seeds = [None if seed is None else int(seed) + off + k for k in range(self.num_envs)]
        self.sampler.seed(seeds)
        if self.device_reset:   # the device continues the very same numpy streams (np_random.cuh)
            self.sim.seed_streams(self.sampler.rngs)
        return seeds

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def reset(self, mask: Optional[torch.Tensor] = None, render: bool = True) -> torch.Tensor:
        """Simulator.reset() (S:528-763) for the masked envs (all if None); returns the obs batch."""
        mask_ptr = None
        if mask is not None:
            mask = mask.to(device=self.device, dtype=torch.uint8).contiguous()
            mask_ptr = mask.data_ptr()
        if self.device_reset:
            self.sim.reset_random(mask_ptr, self._stream())
        else:
            envs = list(range(self.num_envs)) if mask is None else torch.nonzero(mask).flatten().tolist()
            if envs:
                if self.cycle_maps and not self._first_reset:  # MultiMapEnv.reset, envs/multimap_env.py:46
                    self.map_ids[envs] = (self.map_ids[envs] + 1) % len(self.maps)
                if self.randomize_maps_on_reset:   # np_random.choice(self.map_names) S:541-542: first draw of the reset
                    for e in envs:
                        self.map_ids[e] = int(self.sampler.rngs[e].integers(0, len(self.maps)))
                    # _load_map (S:544) comes before the spawn loop: re-create the drawn maps' obstacles first, so that
                    # the spawn predicates below see them at their load-time places.  Only the map id and the
                    # obstacles change here: pose / camera of the episode that just ended stay in place for the
                    # stale-modelview light capture of the reset proper (S:581).
                    self.sim.assign_maps(mask_ptr, self.map_ids.copy(), self._stream())
                dense = self.sampler.sample(envs, [self.maps[self.map_ids[e]] for e in envs], self._query_for(envs))
                params = {}
                for key, val in dense.items():
                    full = np.zeros((self.num_envs,) + val.shape[1:], val.dtype)
                    full[envs] = val
                    params[key] = full
                params["map_id"] = self.map_ids.copy()
                goals = params.pop("goal", None)
                self.sim.reset(mask_ptr, params, self._stream())
                if goals is not None:   # stream-ordered after the reset it belongs to
                    g = torch.from_numpy(goals.astype(np.int16)).to(self.device)
                    self.sim.set_goals(mask_ptr, g.data_ptr(), self._stream())
        self._first_reset = False
        if render:
            self.sim.render(self.obs.data_ptr(), self._stream())
        return self.obs

    @property
    def goal_tile(self) -> torch.Tensor:
        """int16 [num_envs, 2]: every env's goal tile (i, j) under nav=True (a copy, on the current stream)."""
        if not self.nav:
            raise ValueError("goal_tile needs nav=True")
        return torch.stack([self._goal["goal_i"], self._goal["goal_j"]], 1).to(torch.int16)

    def _query_for(self, envs):
        def query(k, x, z, a, safety, hidden):
            return self.sim.query_poses(int(self.map_ids[envs[k]]), x, z, a, safety, hidden, dyn_env=int(envs[k]),
                                        stream=self._stream())
        return query

    def step(self, actions: torch.Tensor, render: bool = True, out=None):
        """actions f32[N,2] on this device: [vel, steering] (DuckietownEnv.step) or wheel duty
        (Simulator.step) depending on action_mode.  Returns (obs u8[N,H,W,3], reward f32[N], done bool[N], info).
        `out=(obs, reward, done_u8)` writes into caller-provided CUDA tensors instead of the env's own.
        Under terminal_obs=True the terminal frames of the envs that ended go to `self.terminal_obs` (dts_step_terminal)."""
        if actions.device != self.device or actions.dtype != torch.float32 or tuple(actions.shape) != (self.num_envs, 2):
            raise ValueError("actions must be a float32 CUDA tensor of shape [num_envs, 2] on the env's device")
        actions = actions.contiguous()
        obs, reward, done = (self.obs, self.reward, self._done_u8) if out is None else out
        if self._keep_terminal:
            self.sim.step_terminal(actions.data_ptr(), obs.data_ptr() if render else None,
                                   self.terminal_obs.data_ptr() if render else None, reward.data_ptr(), done.data_ptr(),
                                   self._stream())
        else:
            self.sim.step(actions.data_ptr(), obs.data_ptr() if render else None, reward.data_ptr(), done.data_ptr(),
                          self._stream())
        return obs, reward, done.view(torch.bool), self.state

    def render_obs(self, segment: bool = False, top_down: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """render_obs(segment) (S:1953-1972) of the current state; `top_down` gives _render_img(top_down=True)'s camera.
        Under `undistort` this is the pinhole frame: UndistortWrapper rectifies only reset / step observations."""
        tgt = self.obs if out is None else out
        base = self._base_mode()
        mode = dict(segment=segment, top_down=top_down, pinhole=self._undistort, rectify=False)
        if segment or top_down or base["rectify"]:
            self.sim.set_render_mode(**mode)
            try:
                self.sim.render(tgt.data_ptr(), self._stream())
            finally:
                self.sim.set_render_mode(**base)
        else:
            self.sim.render(tgt.data_ptr(), self._stream())
        return tgt

    def frame_cameras(self):
        """(V float64 [num_envs, 3, 4], P float32 [num_envs, 4]) on the device: every env's camera of its last frame,
        the model-view [R|t] and gluPerspective's P00, P11, P22, P23 (dts_get_frame_cameras), written on the current
        stream.  Raises before the first render."""
        with torch.cuda.device(self.device):
            V = torch.empty((self.num_envs, 3, 4), dtype=torch.float64, device=self.device)
            P = torch.empty((self.num_envs, 4), dtype=torch.float32, device=self.device)
            self.sim.get_frame_cameras(V.data_ptr(), P.data_ptr(), self._stream())
        return V, P

    def render_bev(self):
        """Write `bev_labels` / `bev_markings` for the current state (dts_render_bev), without rendering a frame."""
        if self.bev_labels is None:
            raise ValueError("render_bev needs bev=True")
        self.sim.render_bev(self._stream())
        return self.bev_labels, self.bev_markings

    def render_scan(self):
        """Write `scan_range` / `scan_hit` for the current state (dts_render_scan), without rendering a frame."""
        if self.scan_range is None:
            raise ValueError("render_scan needs scan=True")
        self.sim.render_scan(self._stream())
        return self.scan_range, self.scan_hit

    def render_objects(self):
        """Write `object_boxes3d` / `object_state` for the current state (dts_render_objects), without rendering a
        frame; `object_corners_px` becomes NaN."""
        if self.object_boxes3d is None:
            raise ValueError("render_objects needs objects=True")
        if self.object_boxes3d.shape[1]:
            self.sim.render_objects(self._stream())
        return self.object_boxes3d, self.object_state, self.object_corners_px

    def render_lane_path(self):
        """Write `lane_path` / `lane_path_count` for the current state (dts_render_lane_path), without rendering a
        frame; `lane_path_px` becomes NaN."""
        if self.lane_path is None:
            raise ValueError("render_lane_path needs lane_path=True")
        self.sim.render_lane_path(self._stream())
        return self.lane_path, self.lane_path_count, self.lane_path_px

    # labels -------------------------------------------------------------------------------------
    def label_table(self, map_id: int = 0) -> list:
        """What each label value of map `map_id` stands for (module-level `label_table`)."""
        return label_table(self.maps[map_id])

    def object_boxes(self):
        """From `labels` (labels=True), on the device: (pixels int32 [num_envs, max_objects], boxes int32 [num_envs,
        max_objects, 4]) — how many pixels of each env's frame show object o of its map, and their bounding box x0, y0,
        x1, y1 (inclusive); -1 where the object shows no pixel.  max_objects is the most objects any of the maps has."""
        if self.labels is None:
            raise ValueError("object_boxes needs labels=True")
        n, n_obj = self.num_envs, self._max_objects()
        with torch.cuda.device(self.device):
            pixels = torch.empty((n, n_obj), dtype=torch.int32, device=self.device)
            boxes = torch.empty((n, n_obj, 4), dtype=torch.int32, device=self.device)
        if n_obj:
            self.sim.object_pixels(self.labels.data_ptr(), pixels.data_ptr(), boxes.data_ptr(), n_obj, self._stream())
        return pixels, boxes

    def _max_objects(self) -> int:
        """The most objects any of the env's maps has: object_boxes()'s and the object boxes' O"""
        return max((len(md.objects) for md in self.maps), default=0)

    # snapshots ----------------------------------------------------------------------------------
    @property
    def state_fingerprint(self) -> int:
        """Identifies the record layout and the maps this env's records refer to (dts_state_info); a map upload
        changes it."""
        return self.sim.state_info()[1]

    def save_state(self, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Every env's complete simulator state as one record per env: uint8 [num_envs, record_bytes] on the env's
        device, written on the current stream without synchronising (dts_save_state).  The tensor's `fingerprint`
        attribute is `state_fingerprint` at save time; `load_state` checks it."""
        rb, fp = self.sim.state_info()
        if out is None:
            out = torch.empty((self.num_envs, rb), dtype=torch.uint8, device=self.device)
        else:
            self._check_records(out, "out")
        self.sim.save_state(out.data_ptr(), self._stream())
        out.fingerprint = fp
        return out

    def _check_records(self, records: torch.Tensor, what: str):
        rb = self.sim.state_info()[0]
        if not isinstance(records, torch.Tensor) or records.device != self.device or records.dtype != torch.uint8 \
                or tuple(records.shape) != (self.num_envs, rb) or not records.is_contiguous():
            raise ValueError(f"{what} must be a contiguous uint8 tensor [num_envs, {rb}] on {self.device}")

    def load_state(self, records: torch.Tensor, mask: Optional[torch.Tensor] = None, fingerprint: Optional[int] = None):
        """Env e (every env, or those where `mask` is true) takes record e of `records` as its complete state
        (dts_load_state), on the current stream without synchronising.  `fingerprint` defaults to the one `save_state`
        attached to `records`; one that is not this env's `state_fingerprint` (other maps, a map re-uploaded since)
        raises and changes nothing.  `render_obs()` then draws the loaded state; `self.obs` is left as it was.  Only
        the device state is loaded: `load_state_dict` / `copy_envs` also carry the host-side reset state."""
        self._check_records(records, "records")
        if fingerprint is None:
            fingerprint = getattr(records, "fingerprint", None)
            if fingerprint is None:
                raise ValueError("records carry no fingerprint: pass the fingerprint of the env that saved them")
        mask_ptr = None
        if mask is not None:
            if tuple(mask.shape) != (self.num_envs,):
                raise ValueError("mask must have one entry per env")
            mask = mask.to(device=self.device, dtype=torch.uint8).contiguous()
            mask_ptr = mask.data_ptr()
        self.sim.load_state(mask_ptr, records.data_ptr(), int(fingerprint), self._stream())

    def _host_state(self) -> dict:
        """The host-side per-env reset state: what host resets draw from (sampler streams, last horizon, reset count)
        and the map ids host resets assign."""
        s = self.sampler
        return dict(rngs=[g.bit_generator.state for g in s.rngs], last_horizon=[np.array(h, float) for h in s.last_horizon],
                    episodes=s.episodes.copy(), map_ids=self.map_ids.copy())

    def _set_host_state(self, h: dict, envs, src):
        s = self.sampler
        for e, k in zip(envs, src):
            s.rngs[e].bit_generator.state = h["rngs"][k]
            s.last_horizon[e] = np.array(h["last_horizon"][k], float)
            s.episodes[e] = h["episodes"][k]
            self.map_ids[e] = h["map_ids"][k]

    def copy_envs(self, src) -> None:
        """Env e becomes a copy of env src[e] as it was before the call; src[e] = -1 keeps env e.  `src` is int64
        [num_envs].  On the device this is `load_state(save_state()[src], src >= 0)`; the host-side reset state is
        copied too, so envs under host resets branch correctly."""
        src = torch.as_tensor(src, dtype=torch.int64)
        if tuple(src.shape) != (self.num_envs,):
            raise ValueError("src must have one entry per env")
        src_h = src.cpu().numpy()
        if ((src_h < -1) | (src_h >= self.num_envs)).any():
            raise ValueError("src entries must be -1 or an env index")
        src_d = src.to(self.device)
        recs = self.save_state()
        gathered = recs[src_d.clamp(min=0)]
        self.load_state(gathered, mask=src_d >= 0, fingerprint=recs.fingerprint)
        envs = np.flatnonzero(src_h >= 0)
        self._set_host_state(self._host_state(), envs, src_h[envs])

    def state_dict(self) -> dict:
        """Everything needed to continue this batch elsewhere: every env's record (on the CPU), its fingerprint and the
        host-side reset state, in types `torch.save` / `torch.load` round-trip.  Synchronises.  Load it into an env
        built with the same keywords (`load_state_dict`).  Under camera_rand it also holds the calibrations and each
        env's, which the env must have too: a resume sees the same lenses."""
        h = self._host_state()
        recs = self.save_state()
        d = {"records": recs.cpu(), "fingerprint": int(recs.fingerprint), "rngs": h["rngs"],
             "last_horizon": torch.from_numpy(np.stack(h["last_horizon"])),
             "episodes": torch.from_numpy(h["episodes"]), "map_ids": torch.from_numpy(h["map_ids"]),
             "first_reset": bool(self._first_reset)}
        if self.camera_rand:
            d["camera_rand"] = self._camera_rand_state()
        return d

    def _camera_rand_state(self) -> dict:
        return {"K": torch.from_numpy(np.stack([K for K, _ in self.calibrations])),
                "D": torch.from_numpy(np.stack([D for _, D in self.calibrations])),
                "calibration_of_env": torch.from_numpy(self.calibration_of_env.astype(np.int64))}

    def load_state_dict(self, d: dict) -> None:
        """Continue from `state_dict()`: every env's device and host state.  A fingerprint from other maps, or camera_rand
        calibrations other than this env's, raise and change nothing."""
        mine, theirs = (self._camera_rand_state() if self.camera_rand else None), d.get("camera_rand")
        if (mine is None) != (theirs is None) or (mine is not None and any(
                mine[k].shape != theirs[k].shape or not torch.equal(mine[k], theirs[k].to(mine[k].dtype)) for k in mine)):
            raise ValueError("the state's camera_rand calibrations differ from this env's")
        recs = d["records"].to(self.device).contiguous()
        self.load_state(recs, fingerprint=int(d["fingerprint"]))
        h = dict(rngs=d["rngs"], last_horizon=list(d["last_horizon"].numpy()), episodes=d["episodes"].numpy(),
                 map_ids=d["map_ids"].numpy())
        envs = np.arange(self.num_envs)
        self._set_host_state(h, envs, envs)
        self._first_reset = bool(d["first_reset"])

    # convenience views --------------------------------------------------------------------------
    @property
    def cur_pos(self) -> torch.Tensor:
        s = self.state
        return torch.stack([s["pos_x"], torch.zeros_like(s["pos_x"]), s["pos_z"]], dim=1)

    @property
    def cur_angle(self) -> torch.Tensor:
        return self.state["angle"]

    def launch_count(self) -> int:
        return self.sim.launch_count()

    def check(self):
        """Synchronise and raise if any render since creation ran out of its frame-memory capacity (prim slab or bin
        lists, sized from the scene's upper bounds at the first render) — such frames are left at the clear colour."""
        torch.cuda.synchronize(self.device)
        if int(self.sim.debug_counters()[0]) != 0 or (self.sim.status() & 1):
            raise L.DtsError("render frame memory overflowed: some frames were not drawn")

    def close(self):
        self.sim.close()


class HostPipeline:
    """Host-facing stepping with the copies taken off the critical path.

    `submit(actions_host)` enqueues: pinned-host -> device copy of the actions, `dts_step`, and a
    device -> pinned-host copy of obs / reward / done on a second stream; `result(ticket)` blocks until
    that step's host buffers are complete.  With `depth` slots in flight the PCIe transfer of step k
    overlaps the kernels of step k+1 (callers whose next action does not depend on the previous
    observation — replay, open-loop or random-action rollouts as in the reference's benchmark.py — get the
    full overlap; a closed-loop caller simply calls result() before the next submit())."""

    def __init__(self, env: BatchedDuckietownEnv, depth: int = 2):
        self.env, self.depth = env, depth
        dev, n = env.device, env.num_envs
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.slots = []
        for _ in range(depth):
            self.slots.append(dict(
                act=torch.empty((n, 2), dtype=torch.float32, device=dev),
                obs=torch.empty_like(env.obs), rew=torch.empty_like(env.reward), done=torch.empty_like(env._done_u8),
                h_obs=torch.empty(tuple(env.obs.shape), dtype=env.obs.dtype).pin_memory(),
                h_rew=torch.empty(n, dtype=torch.float32).pin_memory(),
                h_done=torch.empty(n, dtype=torch.uint8).pin_memory(),
                computed=torch.cuda.Event(), copied=torch.cuda.Event(), busy=False))
        self.ticket = 0

    def submit(self, actions_host: torch.Tensor) -> int:
        """actions_host: float32 [N,2] CPU tensor (pinned for a truly asynchronous copy)."""
        s = self.slots[self.ticket % self.depth]
        cur = torch.cuda.current_stream(self.env.device)
        if s["busy"]:
            cur.wait_event(s["copied"])          # the slot's previous D2H must be done before we overwrite its buffers
        s["act"].copy_(actions_host, non_blocking=True)
        self.env.step(s["act"], out=(s["obs"], s["rew"], s["done"]))
        s["computed"].record(cur)
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(s["computed"])
            s["h_obs"].copy_(s["obs"], non_blocking=True)
            s["h_rew"].copy_(s["rew"], non_blocking=True)
            s["h_done"].copy_(s["done"], non_blocking=True)
            s["copied"].record(self.copy_stream)
        s["busy"] = True
        self.ticket += 1
        return self.ticket - 1

    def result(self, ticket: int):
        """(obs u8[N,H,W,3], reward f32[N], done bool[N]) pinned host tensors of that step; valid until the slot
        is reused `depth` submits later."""
        s = self.slots[ticket % self.depth]
        s["copied"].synchronize()
        return s["h_obs"], s["h_rew"], s["h_done"].view(torch.bool)
