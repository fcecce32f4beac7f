/* dtsim.h — C ABI of libdtsim.so, the H100-native batched Duckietown step() hot path.
 *
 * The reference (duckietown/gym-duckietown @5c2a586) has no FFI for this path: Simulator.step()
 * is Python all the way down to the OpenGL driver.  This header is the boundary we introduce
 * beneath its gym.Env surface (SURVEY.md 8b).  Every entry point names the reference code it
 * replaces (paths relative to /root/reference/src/gym_duckietown).  Plain C, POD structs, raw
 * pointers and sizes; no torch types.  All device work is stream-ordered on the cudaStream_t the
 * caller passes (as a void*; NULL = legacy default stream); no entry point synchronises.
 *
 * Return value: 0 = ok, non-zero = error; dts_last_error() gives the message.
 */
#ifndef DTSIM_H
#define DTSIM_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DTS_ABI_VERSION 3
#define DTS_MAX_DELAY 16     /* command-delay line depth (steps): 0.15 s at up to 100 Hz (MotionBlurWrapper steps at 90 Hz) */
#define DTS_MAX_OBJECTS 256  /* per map; visibility bitmask is 8 x u32 */
#define DTS_LANE_PATH_MAX_POINTS 64  /* points per env of dts_set_lane_path_target */

typedef struct dts_sim dts_sim; /* opaque, one per GPU, not thread-safe */

/* done_code values (simulator.py:1685-1705 DoneRewardInfo.done_code) */
enum { DTS_IN_PROGRESS = 0, DTS_INVALID_POSE = 1, DTS_MAX_STEPS = 2 };
/* action_mode */
enum { DTS_ACTION_PWM = 0,      /* Simulator.step(action=[u_left,u_right])        simulator.py:1669 */
       DTS_ACTION_VEL_STEER = 1 /* DuckietownEnv.step(action=[vel, steering])  envs/duckietown_env.py:36-59 */ };
/* flags */
enum { DTS_FLAG_AUTO_RESET = 1,   /* done envs are re-spawned on device inside dts_step / dts_step_terminal */
       DTS_FLAG_DOMAIN_RAND = 2,  /* simulator.py:213  (camera noise S:1768, DR sampling in device resets) */
       DTS_FLAG_DISTORTION = 4,   /* simulator.py:223  fisheye gather fused into the render (distortion.py:118) */
       DTS_FLAG_DYNAMICS_RAND = 8,/* simulator.py:224  per-env trim on the motor gains (S:746-748) */
       DTS_FLAG_TESSELLATE = 16,  /* draw every road tile as the literal 7x7 quads of simulator.py:386-507
                                     instead of one quad + analytic lattice lighting (DESIGN.md render spec) */
       DTS_FLAG_CAMERA_RAND = 32  /* simulator.py:225 camera_rand: device resets apply the drawn camera height / angle
                                     / FOV without DTS_FLAG_DOMAIN_RAND too (S:611-614); the calibrations are the
                                     caller's (dts_set_fisheye_luts) */ };

/* One entry of the reference's domain-randomization table (randomization/randomizer.py:19-89): Randomizer.randomize
 * draws every key of the JSON config in SORTED key order from the env's np_random, whether or not domain_rand is on
 * (S:546).  `target` says which render / dynamics parameter the draw feeds; keys the simulator never reads are still
 * drawn (DTS_DR_NONE) so that the stream stays aligned with the reference. */
enum { DTS_DR_INT = 0,      /* rng.integers(low, high, size)   randomizer.py:55-58 */
       DTS_DR_UNIFORM = 1,  /* rng.uniform(low, high, size)    randomizer.py:69 */
       DTS_DR_NORMAL = 2    /* rng.normal(loc, scale, size)    randomizer.py:77 */ };
enum { DTS_DR_NONE = 0, DTS_DR_CAMERA_ANGLE, DTS_DR_CAMERA_FOV_Y, DTS_DR_CAMERA_HEIGHT, DTS_DR_CAMERA_NOISE,
       DTS_DR_HORZ_MODE, DTS_DR_LIGHT_POS, DTS_DR_TRIM };
#define DTS_MAX_DR_OPS 16
typedef struct {
  int32_t type, size, target, reserved;
  double a[3], b[3];        /* low / loc and high / scale; element k of a size-3 draw uses a[k], b[k]; size > 3 uses [0] */
} dts_dr_op;

typedef struct {
  int32_t abi_version;      /* DTS_ABI_VERSION */
  int32_t num_envs;         /* N independent agents on this GPU */
  int32_t device;           /* CUDA ordinal */
  int32_t cam_width;        /* simulator.py:216 (default 640) */
  int32_t cam_height;       /* simulator.py:217 (default 480) */
  int32_t max_steps;        /* simulator.py:210 (1500) */
  int32_t frame_skip;       /* simulator.py:215 (1) */
  int32_t action_mode;
  int32_t flags;
  int32_t max_maps;         /* slots for dts_upload_map */
  int32_t cycle_maps;       /* >0: every reset advances the env's map id modulo this count
                               (MultiMapEnv.reset round-robin, envs/multimap_env.py:44-49) */
  int32_t random_maps;      /* >0: every reset draws the env's map uniformly from the first `random_maps` slots and
                               re-creates its obstacles (randomize_maps_on_reset: np_random.choice + _load_map, S:541-544) */
  double frame_rate;        /* simulator.py:214 (30) */
  double robot_speed;       /* simulator.py:218 (1.2): the constant used in the reward, S:1702 */
  double accept_start_angle_deg; /* simulator.py:219 (60), device-side spawn only */
  /* DuckietownEnv constructor (envs/duckietown_env.py:15-33) */
  double gain, trim, radius, k, limit;
  /* duckietown_world DB18 PWM dynamics — source absent, restated (DESIGN.md "dynamics"):
   *   u' = u + dt(-u1 u - u2 w + u3 w^2 + uar*R + ual*L),  w' = w + dt(-w1 w - w2 u - w3 u w + war*R - wal*L)
   *   q' = q * exp(dt * [u', 0, w']),  commands delayed by `delay` seconds.            call sites S:746-755, S:2083-2086 */
  double dyn_u1, dyn_u2, dyn_u3, dyn_w1, dyn_w2, dyn_w3, dyn_uar, dyn_ual, dyn_war, dyn_wal;
  double dyn_delay;         /* 0.15 (S:748-750) */
  uint64_t seed;            /* device-side spawn/DR streams: stream k = hash(seed, global_env_id) */
  int64_t env_id_offset;    /* global index of local env 0 (multi-GPU shards keep seeds GPU-count independent) */
  /* Simulator.__init__ keywords that reset() reads (simulator.py:226-230): device resets honour them */
  int32_t num_tris_distractors; /* 12: 3*n vertices drawn per reset S:621-629 (never visible, draws consumed) */
  int32_t n_dr_ops;         /* 0 = the reference's default_dr.json; else the custom table below, in sorted key order */
  double color_sky[3];      /* BLUE_SKY S:108 (float64 like the Python floats _perturb multiplies) */
  double color_ground[3];   /* (0.15, 0.15, 0.15) S:228 */
  dts_dr_op dr_ops[DTS_MAX_DR_OPS];
} dts_config;

typedef struct { int32_t width, height; const uint8_t* rgba; /* [height][width][4], row 0 = t=0 */ } dts_texture;

typedef struct {            /* one placed prop: objects.py:33-66 (WorldObj), render O:123-148 */
  double pos[3];            /* float64 like WorldObj.pos (_inconvenient_spawn S:1461-1471); rendered as float32 */
  float scale;
  float y_rot_deg;
  int32_t mesh_id;
  int32_t optional;         /* hidden w.p. 1/2 at reset under domain_rand (S:653-654) */
  int32_t dyn_slot;         /* -1: static; else index into dts_map_blob.dyn — pose / card come from the per-env state */
  int32_t alt_tex_from;     /* traffic light: triangles textured `alt_tex_from` show `alt_tex_to` while the shared */
  int32_t alt_tex_to;       /*   card is on pattern 1 (mesh.textures[0] = texs[pattern] O:453,462); -1 = none */
  int32_t reserved;
} dts_object;

/* One `static: false` obstacle (S:973-1017): DuckieObj pedestrian O:339-432 or DuckiebotObj lane follower
 * O:180-336, with its state at map load.  Every env carries its own copy of the evolving state (per map), which
 * like the reference's object list survives resets.  Under domain_rand the reference draws vel / wait_time /
 * follow_dist ... from the GLOBAL numpy RNG at construction (O:348-350, O:197-205): the host supplies them. */
enum { DTS_DYN_DUCKIE = 1, DTS_DYN_DUCKIEBOT = 2,
       DTS_DYN_TRAFFICLIGHT = 3 /* TrafficLightObj O:434-462: static, never collides; flips its card every freq s */ };
#define DTS_MAX_DYN 32
typedef struct {
  int32_t kind;             /* DTS_DYN_* */
  int32_t object_index;     /* entry of objects[] carrying mesh / scale / height */
  double pos[3], angle;     /* WorldObj.pos, .angle O:54-57 */
  double corners[4][2];     /* obj_corners (x,z) O:60 */
  double norms[2][2];       /* obj_norm rows O:61 — the duckiebot never refreshes them (O:306-336) */
  double safety_radius;     /* O:66 */
  double walk_distance, vel, wait_time, wiggle;                       /* DuckieObj O:343-366 */
  double follow_dist, velocity, gain, trim, radius, k, limit, wheel_dist, robot_width, robot_length; /* O:196-227 */
  double freq;              /* TrafficLightObj O:445-450 (5; randint(4,7) under domain_rand) */
  int32_t pattern;          /* starting pattern (0; randint(0,2) under domain_rand) */
  int32_t reserved;
} dts_dyn_object;

/* Per-env state of one dynamic obstacle: DTS_DYN_FIELDS doubles, device layout [field][slot][env]. */
enum { DTS_DYN_PX = 0, DTS_DYN_PZ, DTS_DYN_ANGLE, DTS_DYN_YROT, DTS_DYN_CORNERS /* 8: x0 z0 .. x3 z3 */,
       DTS_DYN_START_X = 12, DTS_DYN_START_Z, DTS_DYN_WAIT, DTS_DYN_VEL, DTS_DYN_TIME, DTS_DYN_ACTIVE, DTS_DYN_FIELDS,
       /* traffic lights reuse two fields: their own pattern, and — in the FIRST light's slot — the card the mesh
        * they all share currently shows (every flip assigns it; the last writer wins, like the reference) */
       DTS_DYN_PATTERN = DTS_DYN_ACTIVE, DTS_DYN_SHOWN = DTS_DYN_WAIT };

typedef struct {
  int32_t tri_offset, tri_count;
  int32_t seg_flat_tex;     /* texture every triangle of this mesh shows under segment=True: the flat class colour
                               gen_segmentation_color(mesh_name) (objmesh.py:260-290); -1 = none */
  int32_t reserved;
} dts_mesh;

/* What the reference's wrapper stacks do to actions, observations and rewards, fused into the step kernels
 * (SURVEY 8f-3).  W = src/gym_duckietown/wrappers.py, LW = learning/utils/wrappers.py. */
enum { DTS_OBS_HWC = 0,     /* render_obs S:1953-1972: [H][W][3] */
       DTS_OBS_CHW = 1,     /* ImgWrapper LW:73-87 transpose(2,0,1): [3][H][W] */
       DTS_OBS_CWH = 2      /* PyTorchObsWrapper W:93-110 transpose(2,1,0): [3][W][H] */ };
enum { DTS_OBS_U8 = 0,
       DTS_OBS_F32_UNIT = 1 /* NormalizeWrapper LW:56-70: (obs - 0) / (255 - 0) as float32 */ };
enum { DTS_REWARD_RAW = 0,
       DTS_REWARD_DT = 1    /* DtRewardWrapper LW:90-102: -1000 -> -10, r > 0 -> r + 10, else r + 4 */ };
enum { DTS_ACTIONS_CONTINUOUS = 0,
       DTS_ACTIONS_DISCRETE3 = 1 /* DiscreteWrapper W:8-33: 0 left [0.6,+1], 1 right [0.6,-1], 2 forward [0.7,0];
                                    actions[e][0] carries the id, actions[e][1] is ignored */ };
typedef struct {
  int32_t obs_layout, obs_dtype, reward_mode, action_map;
  double action_vel_scale;  /* ActionWrapper LW:106-112: action[0] * 0.8 before the env sees it (1.0 = off) */
} dts_output_format;

/* Everything the hot path reads about one map, prepared on the host (maps.py):
 * tile grid S:788-860, curves S:1151-1335, static collidables S:1019-1038 / S:919-931,
 * meshes objmesh.py:65-293, textures graphics.py:70-169. All pointers are HOST memory, copied. */
typedef struct {
  double tile_size;
  int32_t grid_w, grid_h;
  const int8_t* tile_kind;        /* [grid_h*grid_w], -1 = no tile */
  const int8_t* tile_angle;       /* 0..3 (S,E,N,W) */
  const uint8_t* tile_drivable;
  const int16_t* tile_tex;        /* texture index per tile, -1 = none */
  const int32_t* tile_curve_off;  /* first curve of the tile */
  const int32_t* tile_curve_cnt;  /* 0, 2, 6 or 12 */
  int32_t n_curves;
  const double* curves;           /* [n_curves][4][3] */
  int32_t n_coll;
  const double* coll_corners;     /* [n_coll][2][4]  x row, z row */
  const double* coll_norms;       /* [n_coll][2][2]  two SAT axes as rows */
  const double* coll_centers;     /* [n_coll][3] */
  const double* coll_radii;       /* [n_coll] safety radii */
  int32_t n_objects;
  const dts_object* objects;
  int32_t n_meshes;
  const dts_mesh* meshes;
  int32_t n_tris;
  const float* tri_pos;           /* [n_tris][3][3] */
  const float* tri_nrm;           /* [n_tris][3][3] */
  const float* tri_uv;            /* [n_tris][3][2] */
  const float* tri_col;           /* [n_tris][3][3] */
  const int16_t* tri_tex;         /* [n_tris] texture index, -1 = untextured */
  int32_t n_textures;
  const dts_texture* textures;
  int32_t start_tile[2];          /* `user_tile_start` (S:659-662) else map `start_tile` (S:867-871) else {-1,-1}: device resets spawn there */
  int32_t n_dyn;                  /* <= DTS_MAX_DYN */
  int32_t has_start_pose;         /* map `start_pose` (S:874-876): device resets then place the agent at start_pose */
  const dts_dyn_object* dyn;      /* [n_dyn] in the order of the map's object list (update order S:1570-1584) */
  double start_pose[3];           /* x offset, z offset inside the start tile, angle (S:679-686) */
  const int16_t* tex_segment;     /* [n_textures] what Texture.bind(segment=True) / get_mesh(name, True) show instead of texture t
                                     (graphics.py:52-56, 70-130; objmesh.py:268-290); NULL or -1 = unchanged */
  int32_t agent_mesh;             /* mesh drawn at the agent's pose in top-down views (self.mesh, S:864, S:1923-1929); -1 = none */
  int32_t reserved2;
  const uint8_t* tex_class;       /* texel classes of every texture in texture order, width*height each (row 0 = t=0, as
                                     rgba), values of dts_set_marking_target; NULL = all 0 */
  const double* obj_corners;      /* [n_objects][4][2] (x, z): every object's footprint obj_corners (generate_corners
                                     C:64-79, O:60, computed for every object S:885), for dts_set_bev_target; finite.
                                     Objects with a dyn_slot take their env's DTS_DYN_CORNERS instead.  NULL = static
                                     objects have no footprint in the bird's-eye map */
} dts_map_blob;

/* Per-episode inputs produced by Simulator.reset() (simulator.py:528-763, SURVEY 8a row P0), one
 * entry per env of the batch (SoA, HOST pointers, length num_envs; entries of unmasked envs are
 * ignored).  Any pointer may be NULL = keep the reference's non-randomized default. */
typedef struct {
  const int32_t* map_id;
  const double* pos_x;  const double* pos_z;  const double* angle;   /* cur_pos / cur_angle S:740-741 */
  const double* wheel_dist;      /* S:597 */
  const double* trim;            /* S:747 (dynamics_rand) */
  const float* cam_height;       /* S:602,612 */
  const float* cam_angle_deg;    /* S:605,613 */
  const float* cam_fov_y_deg;    /* S:608,614 */
  const float* cam_noise;        /* [N][3] S:1768-1769 */
  const float* horizon_color;    /* [N][3] S:551-562 */
  const float* light_ambient;    /* [N][3] S:573-574 */
  const float* light_diffuse;    /* [N][3] S:575-576 */
  const float* light_pos;        /* [N][4] S:565-570, S:581 */
  const int32_t* light_stale;    /* [N] 0: GL_POSITION captured under identity modelview (first reset);
                                        1: under the previous frame's camera matrix (S:581, SURVEY app. B-11) */
  const float* ground_color;     /* [N][3] S:594 */
  const uint32_t* obj_hidden;    /* [N][8] bit o set = object o invisible this episode (S:653-656) */
} dts_episode_params;

/* Device pointers to the library-owned SoA state (all length num_envs unless noted). */
typedef struct {
  double* pos_x; double* pos_z; double* angle;     /* cur_pos[0], cur_pos[2], cur_angle */
  double* speed;                                   /* S:1568 */
  double* reward;                                  /* f64 shadow of the f32 reward output */
  double* lane_dist; double* lane_dot; double* lane_angle_rad;   /* LanePosition S:1409 (NaN if not in lane) */
  double* prox_penalty;                            /* S:1430-1459 */
  double* wheel_dist;
  int32_t* step_count;
  int32_t* tile_i; int32_t* tile_j;                /* get_grid_coords(cur_pos) S:1134 */
  int32_t* map_id;
  int32_t* episode;                                /* resets so far */
  uint8_t* done_code;
  uint8_t* in_lane;
  uint8_t* collided;                               /* _collision() of the current pose S:1473 */
} dts_state_view;

/* Simulator.__init__ (simulator.py:207-384) minus map loading. */
int dts_create(const dts_config* cfg, dts_sim** out);
/* Simulator._load_map/_interpret_map/_load_objects (simulator.py:765-931) : device copy of one map into slot map_id
 * (< max_maps), in place of the slot's previous map; synchronises the device.  The whole blob is checked, and the new
 * map's device memory allocated and filled, before the slot changes: a refused blob or a failed allocation returns
 * nonzero and leaves the slot as it was, its previous map (or none) still in effect.  A successful upload re-creates
 * the map's dynamic obstacles for every env, and the next render re-sizes frame memory for the new set of maps. */
int dts_upload_map(dts_sim* sim, int map_id, const dts_map_blob* blob);
/* Distortion.rmapx/rmapy (distortion.py:85-125): LUT of the fused fisheye gather, [H][W] each (HOST pointers).  The
 * rasteriser renders every output pixel AT the source position rint(rmap) names — obs[y,x] = undistorted[rint(rmapy),
 * rint(rmapx)], 0 when that falls outside (distortion.py:118, cv2.remap INTER_NEAREST / BORDER_CONSTANT) — so no
 * undistorted frame is materialised and no second pass runs.  Fails if the LUT scatters one 32x8 output bin over a
 * source region too wide for the rasteriser's int32 edge functions. */
int dts_set_fisheye_lut(dts_sim* sim, const float* rmapx, const float* rmapy, int width, int height);
/* camera_rand (distortion.py:46-83): a pool of `count` fisheye LUTs, one per camera calibration, float [count][H][W]
 * each of rmapx / rmapy (HOST), and the LUT of every env, lut_of_env int32 [num_envs] (HOST), each entry in
 * [0, count).  Env e's frames, and its depth and labels, are gathered through LUT lut_of_env[e], in every render.
 * Each LUT is validated as dts_set_fisheye_lut validates its one; a refused call leaves the previous tables and
 * assignment in effect.  Only on a DTS_FLAG_DISTORTION handle.  count = 1 is dts_set_fisheye_lut. */
int dts_set_fisheye_luts(dts_sim* sim, int count, const float* rmapx, const float* rmapy, int width, int height,
                         const int32_t* lut_of_env);
/* UndistortWrapper's rectification (wrappers.py:206-227: cv2.remap(frame, mapx, mapy, INTER_NEAREST) of the pinhole
 * frame, with mapx/mapy from cv2.initUndistortRectifyMap(K, D, I, P, (W, H), CV_32FC1)): a second LUT [H][W] each (HOST
 * pointers), gathered by the same fused kernels as the fisheye's under DTS_RENDER_RECTIFY, so the rectified frame
 * costs no extra pass.  Validated like dts_set_fisheye_lut (camera-sized only; non-finite or huge entries name no
 * source; a LUT too wide for the edge functions is refused and the previous one stays in effect).  Only on a handle
 * created with DTS_FLAG_DISTORTION, whose pair pool is sized for gathers.  NULL, NULL clears it. */
int dts_set_rectify_lut(dts_sim* sim, const float* mapx, const float* mapy, int width, int height);
/* Simulator.reset() (simulator.py:528-763) with host-drawn episode parameters.
 * mask_dev: device u8[num_envs] (NULL = all). */
int dts_reset(dts_sim* sim, const uint8_t* mask_dev, const dts_episode_params* params, void* stream);
/* Simulator.seed() (simulator.py:1043-1045): one numpy PCG64 stream per env for the DEVICE-side resets.
 * streams[N][6] (HOST) = state_hi, state_lo, inc_hi, inc_lo, has_uint32, uinteger of
 * numpy.random.Generator(PCG64(SeedSequence(seed))).bit_generator.state; mask_host u8[N] or NULL = all. */
int dts_seed_streams(dts_sim* sim, const uint8_t* mask_host, const uint64_t* streams);
/* Simulator.reset() with pose / DR drawn ON THE DEVICE from the env's numpy-compatible stream, draw for draw
 * in the reference's order (np_random.cuh): same seeds -> same episodes as the reference. */
int dts_reset_random(dts_sim* sim, const uint8_t* mask_dev, void* stream);
/* Simulator.step() (simulator.py:1669-1683) for all envs: actions f32[N][2] -> obs u8[N][H][W][3]
 * (NULL = skip rendering), reward f32[N], done u8[N]. All DEVICE pointers. */
int dts_step(dts_sim* sim, const float* actions_dev, void* obs_dev, float* reward_dev, uint8_t* done_dev,
             void* stream);
/* dts_step that also returns the TERMINAL frames, on a DTS_FLAG_AUTO_RESET handle: for every env whose episode ended
 * (done = 1), terminal_obs_dev's row gets what the reference's step() returns there (render_obs() S:1677, before the
 * caller's reset()), and obs_dev's row the first frame of the next episode, as from dts_step.  Rows of envs that did
 * not end keep what terminal_obs_dev held.  terminal_obs_dev has obs_dev's size (layout, dtype, resize) and must not
 * be obs_dev.  Stream order: k_step_logic without the respawn, the render of all envs into obs_dev, k_respawn_ended
 * (the respawn, state and draws bit for bit those of dts_step, and a device list of the ended envs), k_copy_rows (their
 * rows -> terminal_obs_dev) and a second render into obs_dev over the listed envs only, whose kernels exit at once when
 * nothing ended.  Launches: 2 R + 3, R being dts_render's (5, or 7 when the rasteriser writes packed u8 HWC of a width divisible by 4, +1
 * with a resize), plus a 4-byte memset; obs_dev = NULL (no render): 2; one more with a bird's-eye target (dts_set_bev_target),
 * one more with a range scan target (dts_set_scan_target), one more with an object target (dts_set_object_target), and
 * one more with a lane path target (dts_set_lane_path_target).  Fails without DTS_FLAG_AUTO_RESET, with
 * terminal_obs_dev == obs_dev, and while a fused gather is armed (dts_gather_next), which it does not write.  The
 * second pass is not timed by dts_profile_*.  Never synchronises. */
int dts_step_terminal(dts_sim* sim, const float* actions_dev, void* obs_dev, void* terminal_obs_dev, float* reward_dev,
                      uint8_t* done_dev, void* stream);
/* Simulator.render_obs() (simulator.py:1953-1972) of the current state. */
int dts_render(dts_sim* sim, void* obs_dev, void* stream);
/* Render variants of _render_img (S:1707-1951) for subsequent dts_render / dts_step calls (0 = the agent camera):
 *   DTS_RENDER_SEGMENT   segment=True: lighting off (S:1730-1733), magenta clear + ground (S:1752, 1808), no distractors
 *                        (S:1814), segmentation textures / flat per-class mesh colours
 *   DTS_RENDER_TOP_DOWN  top_down=True: camera above the map centre looking down (S:1786-1798), the agent's own mesh drawn
 *                        at cur_pos (S:1923-1929)
 *   DTS_RENDER_PINHOLE   Simulator.undistort = True: the fisheye gather of DTS_FLAG_DISTORTION is skipped (S:1969-1970,
 *                        2001-2002), the pinhole frame is emitted
 *   DTS_RENDER_RECTIFY   UndistortWrapper's observation (wrappers.py:206-227): the pinhole frame gathered through the
 *                        dts_set_rectify_lut table; implies PINHOLE.  dts_render fails while no such table is set. */
enum { DTS_RENDER_SEGMENT = 1, DTS_RENDER_TOP_DOWN = 2, DTS_RENDER_PINHOLE = 4, DTS_RENDER_RECTIFY = 8 };
int dts_set_render_mode(dts_sim* sim, int mode);
/* Depth image beside every observation (render spec item 9, DESIGN.md section 5): every later render of this handle —
 * dts_render, dts_step, dts_step_terminal, whatever the render mode — also writes depth_dev, float32
 * [num_envs][cam_height][cam_width], always in that layout and at the camera size whatever dts_set_output_format and
 * dts_set_resize say.  A pixel holds the eye-space depth in metres (clip-space w, the distance along the view axis) of
 * the nearest surface any of its four samples sees: 1 / (the largest 1/w, evaluated at the pixel centre exactly as
 * shading evaluates it, among the distinct winners of the samples).  0: no sample is covered (sky), or the fisheye /
 * rectification table names no source pixel.  No averaging, no quantisation, no far-plane clamp.  Lighting, textures and
 * DTS_RENDER_SEGMENT leave it unchanged; the camera values of domain randomisation do not.  Sticky, like
 * dts_set_render_mode.  The memory is the caller's and must stay valid while it is set; NULL (the default) turns depth
 * off, and the renders launch the very kernels they launch without this call.  A pass over listed envs (the second pass
 * of dts_step_terminal) writes only those envs' rows, so after dts_step_terminal row e matches obs_dev row e; the
 * terminal frames' depth is not kept.  The fused gather (dts_gather_next) carries observations only. */
int dts_set_depth_target(dts_sim* sim, float* depth_dev);
/* Label image beside every observation (render spec item 10, DESIGN.md section 5): every later render of this handle —
 * dts_render, dts_step, dts_step_terminal, whatever the render mode — also writes labels_dev, int16
 * [num_envs][cam_height][cam_width], always in that layout and at the camera size whatever dts_set_output_format and
 * dts_set_resize say.  A pixel holds which draw item it shows: 0 none (no sample covered, or the fisheye / rectification
 * table names no source pixel), 1 the ground quad, 2 + i * grid_h + j the road tile at grid cell (i, j), 2 + n_cells + o
 * object o of the map's object list (dts_map_blob.objects, static and dynamic alike), 2 + n_cells + n_objects the agent's
 * own mesh (top-down views), where n_cells = grid_w * grid_h.  Of the distinct winners of the pixel's four samples it is
 * the one with the largest 1/w at the pixel centre (the surface dts_set_depth_target's depth is taken from), and among
 * equal ones the smallest label; so with both targets set, label != 0 exactly where depth != 0.  No averaging at edges.
 * Lighting, textures, domain-randomised colours and DTS_RENDER_SEGMENT leave it unchanged.  Sticky, like
 * dts_set_render_mode.  The memory is the caller's, 2-byte aligned, and must stay valid while it is set; NULL (the
 * default) turns labels off, and the renders launch the very kernels they launch without this call.  Refused while an
 * uploaded map's largest label exceeds 32767, and while it is set dts_upload_map refuses such a map.  A pass over listed
 * envs (the second pass of dts_step_terminal) writes only those envs' rows, so after dts_step_terminal row e matches
 * obs_dev row e; the terminal frames' labels are not kept.  The fused gather (dts_gather_next) carries observations only. */
int dts_set_label_target(dts_sim* sim, int16_t* labels_dev);
/* Lane-marking image beside every observation (render spec item 11, DESIGN.md section 5): every later render of this
 * handle — dts_render, dts_step, dts_step_terminal, whatever the render mode — also writes markings_dev, uint8
 * [num_envs][cam_height][cam_width], always in that layout and at the camera size whatever dts_set_output_format and
 * dts_set_resize say.  A pixel holds the class of the texel its label winner samples (dts_map_blob.tex_class): 0 none
 * (no road tile: sky, no fisheye / rectification source, the ground, objects, the agent, untextured prims), 1 a road
 * tile's unpainted surface, 2 white, 3 yellow, 4 red paint.  Of the pixel's distinct winners with the label's 1/w and
 * the label's value (dts_set_label_target), each gives the class at texel (floor(u * w) mod w, floor(v * h) mod h) of
 * its texture, u, v as shading computes them at the pixel centre; the pixel takes the smallest.  So markings != 0
 * exactly where the label is a grid cell whose tile has a texture.  Lighting, domain-randomised colours and
 * DTS_RENDER_SEGMENT leave it unchanged.  Independent of the depth and label targets: any of the three may be set.
 * Sticky, like dts_set_render_mode.  The memory is the caller's and must stay valid while it is set; NULL (the default)
 * turns markings off, and the renders launch the very kernels they launch without this call.  A pass over listed envs
 * (the second pass of dts_step_terminal) writes only those envs' rows; the terminal frames' markings are not kept.  The
 * fused gather (dts_gather_next) carries observations only. */
int dts_set_marking_target(dts_sim* sim, uint8_t* markings_dev);
/* Bird's-eye map around every agent (DESIGN.md section 5, item 12): a grid of `height` x `width` cells fixed to the
 * agent, sampled from the map itself rather than rendered.  Row 0 is the farthest ahead and column 0 the leftmost, so
 * the grid reads like an image of the ground seen from above with the agent facing up.  The agent sits at (origin_x,
 * origin_y), in cells, and a cell is `cell` metres on a side.  In float64: with ca, sa = cos, sin of the env's angle,
 * cell (r, c) has f = (origin_y - (r + 0.5)) * cell, l = ((c + 0.5) - origin_x) * cell and its centre at
 * x = pos_x + f * ca + l * sa, z = pos_z - f * sa + l * ca (get_dir_vec, get_right_vec S:2056-2073). */
typedef struct {
  int32_t width, height;    /* cells, 1 to 2048 each */
  double cell;              /* metres per cell, finite and > 0 */
  double origin_x, origin_y;/* the agent's position in grid coordinates (cells), finite */
} dts_bev_config;
/* Sets the bird's-eye targets: labels_dev int16 [num_envs][height][width] (2-byte aligned) and markings_dev uint8
 * [num_envs][height][width], either of them NULL.  A cell's label uses the numbering of dts_set_label_target: 2 + n_cells
 * + o for the smallest object index o whose footprint (dts_map_blob.obj_corners, or the env's DTS_DYN_CORNERS for an
 * object with a dyn_slot) contains the cell centre, the four cross products (c[k+1] - c[k]) x (p - c[k]) all >= 0 or
 * all <= 0, objects hidden this episode skipped (the reference still collides with a hidden optional object); else
 * 2 + i * grid_h + j on the road tile at (i, j) = (floor(x / tile_size), floor(z / tile_size)) (get_grid_coords S:1134);
 * else 1, the ground, outside the grid included.  0 and the agent's label never appear.  A cell's marking is the
 * class (dts_set_marking_target's values) of the texel of its tile's texture under the centre: the inverse of the
 * tile's model transform T((i + .5) ts, 0, (j + .5) ts) Ry(angle * 90 + 180) gives lx, lz, then u = (lx + ts/2) / ts,
 * v = 1 - (lz + ts/2) / ts and the texel (floor(u * w) mod w, floor(v * h) mod h); 0 off the tiles or on a tile without
 * texture.  Objects do not change markings.
 * Written once per dts_step and dts_step_terminal (after the respawn: a row shows the state the returned obs row shows,
 * whether or not obs_dev is NULL), once per dts_render and by dts_render_bev; not by a call refused before it launches.
 * Independent of the render mode, fisheye, rectification, resize, output format and the per-pixel targets.  Sticky; the
 * memory is the caller's and must stay valid while it is set.  A NULL config, or both pointers NULL, turns it off, and
 * then no call launches anything for it.  A refused config returns 1 and leaves the previous target in effect.  Refused
 * with labels while an uploaded map's largest label exceeds 32767, and while so set dts_upload_map refuses such a map.
 * An output, not state: snapshots and the gathers do not carry it. */
int dts_set_bev_target(dts_sim* sim, const dts_bev_config* cfg, int16_t* labels_dev, uint8_t* markings_dev);
/* The bird's-eye targets of the current state (after dts_reset without a render, dts_load_state, ...): one launch,
 * stream-ordered.  Fails while no target is set. */
int dts_render_bev(dts_sim* sim, void* stream);
/* Range scan around every agent (DESIGN.md section 5, item 16): n_rays rays on the ground plane, each cast from one
 * origin until an object or undrivable ground stops it.  In float64, with px, pz, a the env's pos_x, pos_z, angle and
 * ca, sa = cos a, sin a: the origin is ox = px + f ca + r sa, oz = pz - f sa + r ca (f, r = origin_forward,
 * origin_right: dts_bev_config's formulas); ray k (0 <= k < n_rays) leaves at phi_k = fov (0.5 - (k + 0.5) / n_rays) to
 * the left of the heading, along get_dir_vec(a + phi_k) = (cos(a + phi_k), -sin(a + phi_k)), so ray 0 is the leftmost
 * and one ray points straight ahead; fov = 2 pi covers the circle with no ray twice.  A point p blocks a ray when (a) its
 * bird's-eye label (dts_set_bev_target) is an object: a footprint of an object not hidden this episode holds it, which
 * is what the camera sees (traffic lights included), not the reference's collision set; or (b) _drivable_pos(p)
 * (S:1411-1428) is false: off the grid, an empty cell or a tile that is not drivable.  A footprint that is not strictly
 * convex (its four corners do not turn one way) stops no ray; no shipped map has one.
 * range_dev float32 [num_envs][n_rays]: t* = inf { t >= 0 : origin + t dir blocked }, max_range when no point within
 * max_range is blocked, 0 when the origin is.  hit_dev int16 [num_envs][n_rays], in dts_set_label_target's numbering:
 * 2 + n_cells + o for the smallest object index o whose footprint the ray enters at t* (an object wins over a cell
 * boundary at the same t); else 2 + i * grid_h + j for the tile at (i, j) that is not drivable and that the ray enters;
 * else 1 (an empty cell or off the grid); 0 when nothing is met within max_range; when the origin is blocked, the
 * origin's own bird's-eye label.
 * Written once per dts_step and dts_step_terminal (after the respawn: a row shows the state the returned obs row shows,
 * whether or not obs_dev is NULL), once per dts_render and by dts_render_scan; not by a call refused before it launches.
 * Independent of the render mode, fisheye, rectification, resize, output format and every other target. */
typedef struct {
  int32_t n_rays;           /* 1 to 4096 */
  double fov;               /* radians, in (0, 2 pi] */
  double max_range;         /* metres, finite and > 0 */
  double origin_forward, origin_right;   /* metres, finite */
} dts_scan_config;
/* Sets the range scan targets range_dev (4-byte aligned) and hit_dev (2-byte aligned), either of them NULL.  Sticky;
 * the memory is the caller's and must stay valid while it is set.  A NULL config, or both pointers NULL, turns it off,
 * and then no call launches anything for it.  A refused config returns 1 and leaves the previous target in effect.
 * Refused with hit_dev while an uploaded map's largest label exceeds 32767, and while so set dts_upload_map refuses
 * such a map.  An output, not state: snapshots and the gathers do not carry it. */
int dts_set_scan_target(dts_sim* sim, const dts_scan_config* cfg, float* range_dev, int16_t* hit_dev);
/* The range scan of the current state (after dts_reset without a render, dts_load_state, ...): one launch,
 * stream-ordered.  Fails while no target is set. */
int dts_render_scan(dts_sim* sim, void* stream);
/* Motion-flow image beside every observation (DESIGN.md section 5, item 13): every later render of this handle that
 * writes obs — dts_render, dts_step, dts_step_terminal, whatever the render mode — also writes flow_dev, float32
 * [num_envs][cam_height][cam_width][2], always in that layout and at the camera size whatever dts_set_output_format and
 * dts_set_resize say.  A pixel holds (dx, dy) in output pixels, x to the right and y down: BACKWARD flow, the position
 * the surface point it shows had in the previous frame minus its position in this one.  The previous frame is the
 * camera and scene at the start of the env's most recent dts_step / dts_step_terminal (before its frame_skip ticks),
 * in the same episode: a kernel launched just before k_step_logic (k_flow_record) records the agent's pose, every dynamic
 * slot's position and heading and the episode number.  The surface point is the one the depth and label images name (dts_set_depth_target,
 * dts_set_label_target): unprojected from the pixel centre of its pinhole source pixel (under the fisheye, the table's
 * source), moved with its draw item (ground, tiles, static objects and traffic lights stay; a moving obstacle and, in
 * top-down views, the agent's mesh move with their pose, rounded to float as the render places them), and projected
 * through the previous camera.  Under the fisheye the pinhole positions at both ends go through the forward map of the
 * env's table, sampled bilinearly (OpenCV's convention: index = position - 0.5).  NaN where: the depth is 0 (sky, no
 * source pixel); the env has no previous frame (nothing stepped since dts_set_flow_target, a map upload, a reset or
 * respawn, or a dts_load_state of that env); the render is DTS_RENDER_RECTIFY; the point was not in front of the previous
 * camera's near plane; or, under the fisheye, the forward map's footprint leaves the table.  A point hidden in the
 * previous frame still gets its motion: dts_set_occlusion_target says which pixels were in view there.  After a step, dts_render gives the step's flow again; after a step
 * without a render, the next render gives that step's.  A pass over listed envs (the second pass of dts_step_terminal)
 * writes only those envs' rows — NaN, as they respawned — so row e matches obs_dev row e; the terminal frames' flow is
 * not kept.
 * fwd_x / fwd_y: HOST float32 [n_tables][cam_height][cam_width], the forward maps F (distortion.Distortion's mapx / mapy:
 * the distorted output position of every pinhole position) of the fisheye tables, one per table of the pool and in its
 * order, on a DTS_FLAG_DISTORTION handle; NULL, NULL, 0 without.  A fisheye LUT set afterwards drops them, and renders
 * through it fail until this is called again.  Refused (non-zero, the previous setting kept) unless the depth and label
 * targets are set, with a wrong n_tables, or a flow_dev not 8-byte aligned; while it is set, clearing the depth or
 * label target is refused.  Sticky; the memory is the caller's and must stay valid while it is set.  NULL turns it off,
 * and then the renders launch the very kernels they launch without this call.  With it set, every render launches one
 * more kernel (k_flow), and dts_step, dts_step_terminal and dts_load_state one more each.  Synchronises.  An output, not state: snapshots and the gathers do not
 * carry it, nor the record. */
int dts_set_flow_target(dts_sim* sim, float* flow_dev, const float* fwd_x, const float* fwd_y, int n_tables);
/* Occlusion mask beside the flow image (DESIGN.md section 5, item 14): every later render that writes flow_dev also
 * writes occ_dev, uint8 [num_envs][cam_height][cam_width], one DTS_OCC_* value per pixel, checked in this order:
 *   DTS_OCC_NONE      the pixel's flow is NaN
 *   DTS_OCC_OUTSIDE   q = p + 0.5 + flow, the pixel's position in the previous frame, lies outside [0, W) x [0, H)
 *   DTS_OCC_UNKNOWN   no render of the recorded state (the start of the env's last step) in this view was kept
 *   DTS_OCC_VISIBLE   one of the up to four pixels around q, (floor(q - 0.5) + {0, 1}) clipped to the frame, showed the
 *                     same label in that render and, unless the label is the ground or a road tile, a depth within
 *                     2 % of the point's depth in the previous camera
 *   DTS_OCC_OCCLUDED  otherwise: the previous frame shows something else at q
 * Under the fisheye most points that leave the view already have NaN flow (F's footprint leaves the table): NONE.
 * The previous frames are kept by the library: two slots per env of a depth and a label image (12 bytes per pixel
 * across both), each tagged with the episode, step_count and view (the DTS_RENDER_TOP_DOWN, _PINHOLE and _RECTIFY bits;
 * not _SEGMENT) of the frame it holds.  A render reads the slot of its flow record's state in its view, if there is one,
 * and writes its own frame into the other slot, or with no match into the one written less recently.  So dts_render
 * after a step repeats the step's mask; after a step without a render the next step's mask is UNKNOWN; a render in
 * another view between two steps leaves the next step's mask intact; after dts_step_terminal row e matches obs_dev row
 * e (respawned envs NONE; the terminal frames' masks are not kept, but the respawned frames are, so their next step
 * has a mask).  The slots are emptied by this call, dts_set_flow_target, a map upload, and dts_load_state for the
 * loaded envs.
 * Refused (non-zero, the previous setting kept) unless a flow target is set, or when the slots cannot be allocated;
 * while it is set, clearing the flow target is refused.  Sticky; the memory is the caller's and must stay valid while
 * it is set.  NULL turns it off, and then the renders launch the very kernels they launch without this call.  With it
 * set, every render launches one more kernel (k_occ_commit, after k_flow) and k_flow is its mask-writing instance;
 * dts_step, dts_step_terminal and dts_load_state launch what they launch with flow alone.  Synchronises.  An output,
 * not state: snapshots and the gathers carry neither it nor the slots. */
enum { DTS_OCC_NONE = 0, DTS_OCC_VISIBLE = 1, DTS_OCC_OCCLUDED = 2, DTS_OCC_OUTSIDE = 3, DTS_OCC_UNKNOWN = 4 };
int dts_set_occlusion_target(dts_sim* sim, uint8_t* occ_dev);
/* Camera visibility of the bird's-eye grid (DESIGN.md section 5, item 15): for every cell of dts_set_bev_target's grid,
 * whether the frame drawn for its env shows it, and where it lands in that frame.  In float64: the cell centre (x, z) of
 * dts_bev_config at height y = 0 on a road tile (i, j) = (floor(x / tile_size), floor(z / tile_size)) and the ground
 * quad's (float)(-0.8 * 0.01) elsewhere — for a cell whose label is an object, the surface under it — goes through the
 * frame's camera V to the eye point e = V (x, y, z, 1) and, with the frame's float32 P00 / P11, to
 * x1 = (P00 ex / -ez + 1) W / 2, y1 = (1 - P11 ey / -ez) H / 2.  Outside unless 0.04 < -ez <= 100 (gluPerspective's
 * planes).  Without a remap q = (x1, y1); under the fisheye (one table or a camera_rand pool) q is the env's forward map
 * F at (x1, y1), read as dts_set_flow_target reads it, and the cell is outside where F's footprint leaves the table.
 * Outside unless q lies in [0, W) x [0, H).  Then the up to four pixels (floor(q - 0.5) + {0, 1}) clipped to the frame,
 * in the frame's label image, decide, in this order:
 *   DTS_BEVVIS_VISIBLE   one of them shows the cell's grid label
 *   DTS_BEVVIS_OUTSIDE   all of them show 0 (sky, no fisheye source pixel, beyond the ground quad)
 *   DTS_BEVVIS_OCCLUDED  otherwise
 *   DTS_BEVVIS_UNKNOWN   every cell of an env this call drew no frame for, or drew DTS_RENDER_RECTIFY
 * vis_dev: uint8 [num_envs][height][width]; pix_dev: float32 [num_envs][height][width][2] (8-byte aligned), q in camera
 * pixels with pixel centres at +0.5 as the flow image's, NaN for UNKNOWN and OUTSIDE.  Either may be NULL; both NULL
 * turns it off, and then every call launches exactly what it launches without it.  fwd_x / fwd_y / n_tables: as
 * dts_set_flow_target's, and the two share the forward maps: clearing one keeps them for the other, and a fisheye LUT
 * set afterwards drops them for both.  Refused (non-zero, the previous setting kept) unless a bird's-eye label target and
 * a label target are set, with a wrong n_tables or a pix_dev not 8-byte aligned; while it is set, clearing either label
 * target and a dts_set_bev_target of another width or height are refused.  With it set, every call that writes the grid
 * (dts_step, dts_step_terminal, dts_render, dts_render_bev) launches one more kernel, k_bev_view, last in the call: after
 * dts_step with obs_dev and dts_render against the frame just drawn (in its mode), after dts_step_terminal with obs_dev
 * against the frame in obs_dev row e (the respawned first frame where the episode ended); after dts_step without obs_dev,
 * dts_step_terminal without obs_dev and dts_render_bev every cell is UNKNOWN.  Sticky; the memory is the caller's and
 * must stay valid while it is set.  Synchronises.  An output, not state: snapshots and the gathers do not carry it. */
enum { DTS_BEVVIS_UNKNOWN = 0, DTS_BEVVIS_VISIBLE = 1, DTS_BEVVIS_OCCLUDED = 2, DTS_BEVVIS_OUTSIDE = 3 };
int dts_set_bev_visibility_target(dts_sim* sim, uint8_t* vis_dev, float* pix_dev, const float* fwd_x, const float* fwd_y,
                                  int n_tables);
/* The camera of every env's last frame, as k_frame_setup built it: V_dev float64 [num_envs][12] (row-major 3x4 [R|t]) and
 * P_dev float32 [num_envs][4] (P00, P11, P22, P23 of gluPerspective), device memory.  Stream-ordered, one launch; fails
 * before the handle's first render (and after a map upload, until the next render). */
int dts_get_frame_cameras(dts_sim* sim, double* V_dev, float* P_dev, void* stream);
/* Object boxes around every agent (DESIGN.md section 5, item 17): for each env e and object slot o < max_objects, the
 * 3D box of object o of e's map and where it lands in the frame drawn for e.  Box: its four corners in x-z are the
 * object's footprint of the bird's-eye map (dts_map_blob.obj_corners, or env e's DTS_DYN_CORNERS for an object with a
 * dynamic slot), ordered so that c0 -> c1 runs along the object's heading: generate_corners' order (C:64-79), c0 (min
 * x, min z), c1 (max x, min z), c2, c3, as the map and the load-time obstacles have them; for a Duckiebot whose turning
 * step has rewritten them in agent_boundbox's order (back-left, back-right, front-right, front-left, collision.py:9-31),
 * (c1, c2, c3, c0) — chosen by which of c0 -> c1 and c1 -> c2 lies along get_dir_vec(DTS_DYN_ANGLE); its span in y is pos_y + scale min_y to pos_y + scale max_y, min_y / max_y the mesh's object-space
 * extent (ObjMesh.min_coords / max_coords, objmesh.py:228-232, over the mesh's vertices as uploaded).  In float64, with
 * px, pz, a the env's pos_x, pos_z, angle and ca, sa = cos a, sin a (the bird's-eye grid's frame, item 12, inverted):
 *   boxes_dev float32 [num_envs][max_objects][7]: forward, right, up of the centre (the mean of c0..c3 at the middle of
 *     the span; forward = dx ca - dz sa, right = dx sa + dz ca for dx, dz = centre - (px, pz), up = y), then
 *     length = |c1 - c0|, width = |c2 - c1|, height = y1 - y0, and yaw = atan2(-right(c1 - c0), forward(c1 - c0)) in
 *     (-pi, pi]: the object's heading minus the agent's, counter-clockwise from above.  NaN for DTS_OBJECT_NONE.
 *   state_dev uint8 [num_envs][max_objects]: DTS_OBJECT_NONE (o >= the map's object count, or a map uploaded without
 *     footprints), DTS_OBJECT_SHOWN, or DTS_OBJECT_HIDDEN (an optional object hidden this episode; the reference still
 *     collides with it, so its box is given).
 *   corners_dev float32 [num_envs][max_objects][9][2]: the 8 box corners (c0..c3 at y0, then c0..c3 at y1) and the box
 *     centre through the frame's camera as dts_set_bev_visibility_target projects a cell: x1, y1 where 0.04 < -ez <= 100,
 *     else NaN; without a remap q = (x1, y1), kept when it lies outside the frame; under the fisheye (one table or a
 *     camera_rand pool) q = F(x1, y1), NaN where F's footprint leaves the table.  Every point NaN for an env this call
 *     drew no frame for, for a frame drawn with DTS_RENDER_RECTIFY, and for DTS_OBJECT_NONE.
 * Any output may be NULL; all NULL turns it off, and then every call launches exactly what it launches without it.
 * fwd_x / fwd_y / n_tables: as dts_set_flow_target's, shared with the flow image and the bird's-eye visibility on the same
 * terms.  Refused (non-zero, the previous target kept) for max_objects outside 1 to DTS_MAX_OBJECTS, while an uploaded
 * map has more objects than max_objects, with outputs not aligned to their element size, with wrong forward maps, or
 * when an allocation fails; while it is set, dts_upload_map refuses a map with more objects than max_objects.  With it
 * set, dts_step, dts_step_terminal and dts_render launch one more kernel, k_objects, last in the call (after
 * k_bev_view): a row shows the state obs row e shows, the respawned first state where dts_step_terminal's episode ended,
 * and boxes and state are written without obs_dev too.  Sticky; the memory is the caller's and must stay valid while it
 * is set.  Synchronises.  An output, not state: snapshots and the gathers do not carry it. */
enum { DTS_OBJECT_NONE = 0, DTS_OBJECT_SHOWN = 1, DTS_OBJECT_HIDDEN = 2 };
int dts_set_object_target(dts_sim* sim, int max_objects, float* boxes_dev, uint8_t* state_dev, float* corners_dev,
                          const float* fwd_x, const float* fwd_y, int n_tables);
/* The object boxes and states of the current state (after dts_reset without a render, dts_load_state, ...), every corner
 * NaN: one launch, stream-ordered.  Fails while no target is set. */
int dts_render_objects(dts_sim* sim, void* stream);
/* The lane path ahead of every agent (DESIGN.md section 5, item 18): points along its lane's centre curve, in the
 * agent's frame and in the frame drawn for it.  ccp(p, a) below is closest_curve_point (S:1337-1369) as the step's lane
 * pose takes it: the tile under p (get_grid_coords), none off the grid or on a tile that is not drivable; the curve of
 * that tile whose chord P3 - P0, every chord divided by the one Frobenius norm of them all, has the largest dot product
 * with get_dir_vec(a) (the first at a tie); then bezier_closest's 8-level bisection for p and the point and unit
 * tangent there.  Per env e, in float64, with px, pz, a its pos_x, pos_z, angle:
 *   (q0, t0) = ccp((px, 0, pz), a); for k = 0, 1, ...: a_k = atan2(-t_k.z, t_k.x) (the tangent's heading, so that
 *   get_dir_vec(a_k) lies along t_k) and (q_{k+1}, t_{k+1}) = ccp(q_k + spacing t_k, a_k); the walk ends at n_points
 *   points or at the first call that finds none, and count is how many it found.
 * Point 0 takes the agent's heading, so it is the anchor of get_lane_pos2 (the lane pose); each later point takes the
 * previous tangent's, so the walk follows the lane around curves.  On 3-way and 4-way tiles the best-aligned chord picks
 * the curve as the reference's rule does, and it can switch curves partway through a tile: the walk does not choose a
 * route.  Spacing is nominal: a point is the bisection's closest point to a step of `spacing` along the tangent.
 *   points_dev float32 [num_envs][n_points][3]: forward, right of q_k (dx ca - dz sa, dx sa + dz ca for dx, dz =
 *     q_k - (px, pz), ca, sa = cos a, sin a, item 17's formulas), then yaw = atan2(-right(t_k), forward(t_k)) in
 *     (-pi, pi], -pi given as pi: the tangent's heading minus the agent's, counter-clockwise from above.  NaN for k >=
 *     count.  Point 0's lane pose: dist = -forward sin(yaw) - right cos(yaw) and angle_rad = yaw.
 *   count_dev int16 [num_envs].
 *   px_dev float32 [num_envs][n_points][2]: q_k (at its own y: 0, the curves are flat) through the frame's camera as
 *     dts_set_object_target projects a box corner: where 0.04 < -ez <= 100, kept outside the frame for the pinhole and
 *     top-down views, through F under the fisheye or a camera_rand pool (NaN where F's footprint leaves the table).
 *     NaN under DTS_RENDER_RECTIFY, for an env the call drew no frame for, and for k >= count.
 * Any output may be NULL; all NULL turns it off, and then every call launches exactly what it launches without it.
 * fwd_x / fwd_y / n_tables: as dts_set_flow_target's, shared with the flow image, the bird's-eye visibility and the
 * object target on the same terms.  Refused (non-zero, the previous target kept) for n_points outside 1 to
 * DTS_LANE_PATH_MAX_POINTS, spacing outside (0, 1] m or not finite, points_dev / px_dev not aligned to 4 bytes or
 * count_dev to 2, or wrong forward maps.  With it set, dts_step, dts_step_terminal and dts_render launch one more
 * kernel, k_lane_path, last in the call (after k_objects): a row shows the state obs row e shows, the respawned first
 * state where dts_step_terminal's episode ended, and points and count are written without obs_dev too.  Sticky; the
 * memory is the caller's and must stay valid while it is set.  Synchronises.  An output, not state: snapshots and the
 * gathers do not carry it. */
int dts_set_lane_path_target(dts_sim* sim, int n_points, double spacing, float* points_dev, int16_t* count_dev,
                             float* px_dev, const float* fwd_x, const float* fwd_y, int n_tables);
/* The lane path of the current state (after dts_reset without a render, dts_load_state, ...), every pixel NaN: one
 * launch, stream-ordered.  Fails while no target is set. */
int dts_render_lane_path(dts_sim* sim, void* stream);
/* Every env's object pixel statistics from a caller's label image labels_dev int16 [num_envs][cam_height][cam_width]
 * (dts_set_label_target's numbering, against the map each env has now): o = label - 2 - grid_w * grid_h is object o
 * where 0 <= o < the map's object count.  pixels_dev int32 [num_envs][max_objects]: how many pixels show object o;
 * boxes_dev int32 [num_envs][max_objects][4]: their inclusive bounds x0, y0, x1, y1, all -1 where the count is 0 (and
 * for o at or past the map's object count).  Refused for max_objects outside 1 to DTS_MAX_OBJECTS, NULL or misaligned
 * pointers.  One launch, k_object_pixels, stream-ordered. */
int dts_object_pixels(dts_sim* sim, const int16_t* labels_dev, int32_t* pixels_dev, int32_t* boxes_dev, int max_objects,
                      void* stream);
/* Select the fused wrapper behaviour for subsequent dts_step / dts_render calls (default: all zero, scale 1).
 * obs_dev then holds num_envs * 3 * H * W elements of uint8 or float32 in the chosen layout.  The renderer draws packed
 * uint8 HWC; for any other layout or dtype without a resize (dts_set_resize) it draws into a library staging frame of
 * num_envs * cam_height * cam_width * 3 bytes, and a format pass writes obs_dev.  A call that changes the layout or dtype
 * synchronises the device first, as it may allocate or free that frame; a failed allocation returns an error and leaves
 * the previous format in effect. */
int dts_set_output_format(dts_sim* sim, const dts_output_format* fmt);
/* ResizeWrapper (wrappers.py:111-141: cv2.resize(obs, (resize_w, resize_h), interpolation=cv2.INTER_CUBIC)) on the device:
 * subsequent dts_step / dts_render calls render at the camera size into a library buffer and write obs_dev as
 * num_envs x 3 x out_h x out_w elements in the selected layout / dtype (OpenCV's 8-bit fixed-point bicubic; matches cv2
 * within 1 LSB).  out_w = out_h = 0 switches it off. */
int dts_set_resize(dts_sim* sim, int out_w, int out_h);
/* The same resize slot with a choice of filter.  DTS_RESIZE_CV2_CUBIC is dts_set_resize.  DTS_RESIZE_PIL_BILINEAR is
 * learning/utils/wrappers.py:39-54's ResizeWrapper: scipy.misc.imresize(obs, (out_h, out_w, 3)), which for a uint8 RGB
 * frame is PIL.Image.resize((out_w, out_h), BILINEAR) — Pillow's 8-bit fixed-point triangle filter, widened by the
 * scale factor when it shrinks; bit-exact.  That filter takes targets of at least 1/32 of the camera size per axis
 * (at most 65 taps per output pixel): a smaller one is refused and the previous setting stays in effect.
 * out_w = out_h = 0 switches resizing off whatever the filter. */
enum { DTS_RESIZE_CV2_CUBIC = 0, DTS_RESIZE_PIL_BILINEAR = 1 };
int dts_set_resize_filter(dts_sim* sim, int out_w, int out_h, int filter);
/* MotionBlurWrapper (learning/utils/wrappers.py:8-54): out f64[n] = np.average of four u8 frame batches with `weights`
 * (numpy's evaluation order), and the knobs that wrapper turns on the wrapped env: delta_time / frame_skip (it divides
 * env.delta_time by 3 and drives update_physics itself, LW:13-14) and the action convention (wheel commands). */
int dts_blend4(dts_sim* sim, const uint8_t* const frames_dev[4], const double weights[4], double* out_dev, uint64_t n, void* stream);
int dts_set_timing(dts_sim* sim, double delta_time, int frame_skip, int action_mode);
/* The resize pass alone, on caller-supplied frames: src u8[num_envs][cam_h][cam_w][3] -> dst in the selected layout / dtype. */
int dts_resize_frames(dts_sim* sim, const uint8_t* src_dev, void* dst_dev, void* stream);
int dts_get_state(dts_sim* sim, dts_state_view* out);
/* Batched pose predicates for host callers — the de-facto public helpers of Simulator:
 * _valid_pose (S:1494), _collision(get_agent_corners()) (S:1473, run_tests.py:50), get_lane_pos2 (S:1371),
 * proximity_penalty2 (S:1430), _inconvenient_spawn (S:1461), get_grid_coords (S:1134), _drivable_pos (S:1411).
 * HOST pointers, synchronous. query[n][4] = x, z, angle, safety_factor; hidden[n][8] object-visibility
 * bitmasks or NULL; out_f64[n][4] = lane dist, dot_dir, angle_rad (NaN when not in a lane), proximity;
 * out_i32[n][8] = valid, collision (offset once), collision (as _valid_pose sees it), in_lane,
 * inconvenient_spawn, tile_i, tile_j, drivable.  Dynamic obstacles are taken where env `dyn_env` currently has
 * them (check_collision O:265/368, proximity O:271/374, x.pos in S:1466); dyn_env < 0 ignores them. */
int dts_query_poses(dts_sim* sim, int map_id, int dyn_env, int n, const double* query, const uint32_t* hidden,
                    double* out_f64, int32_t* out_i32, void* stream);
/* randomize_maps_on_reset, host-drawn (S:541-544): give the masked envs the map ids in map_id_host[N] and re-create
 * those maps' obstacles for them (_load_map) WITHOUT touching pose, episode counter or render record — the reset that
 * follows still sees the previous episode's last camera (stale GL_LIGHT0 position, S:581). */
int dts_assign_maps(dts_sim* sim, const uint8_t* mask_dev, const int32_t* map_id_host, void* stream);
/* Device pointer to the dynamic-obstacle state of map `map_id`: f64[DTS_DYN_FIELDS][n_dyn][num_envs] (NULL, 0 for a
 * map without dynamic obstacles).  Re-uploading the map puts every env's obstacles back to their load-time state. */
int dts_get_dyn_state(dts_sim* sim, int map_id, double** state_dev, int32_t* n_dyn);
/* End-of-rollout observation all-gather across the GPU shards of one box (SURVEY 8e); the step path
 * itself has no collective.  libnccl is dlopen'ed from `libnccl_path` (the torch-bundled copy); rank 0
 * creates a unique id, the caller broadcasts its 128 bytes (torch.distributed), every rank inits.
 * send: u8[bytes_per_rank] on this GPU, recv: u8[world*bytes_per_rank]. */
int dts_comm_load(dts_sim* sim, const char* libnccl_path);
int dts_comm_unique_id(dts_sim* sim, uint8_t out[128]);
int dts_comm_init(dts_sim* sim, const uint8_t id[128], int rank, int world);
int dts_allgather_obs(dts_sim* sim, const void* send_dev, void* recv_dev, uint64_t bytes_per_rank, void* stream);
/* Sticky status, readable WITHOUT synchronising (mapped host words the kernels write): bit 0 = some frame since
 * creation overflowed its render frame memory (prim slab / bin lists) and was left incomplete; bit 1 = a
 * dts_load_state was handed a record whose map_id names no uploaded map (that env was not loaded).  dts_step and
 * dts_render return non-zero once either is set (the call that set it may be one or two calls back). */
int dts_status(dts_sim* sim);
/* Snapshots: every env's complete simulator state as one record, saved from and loaded into the library's own arrays
 * on the device, for resuming a run exactly or branching envs from a state.  A record holds everything a step, a reset
 * or a render reads about its env:
 *   - the dynamics (cartesian pose cx cy ctheta, velocities vu vw, motor trim) and the command-delay line
 *     fifo[DTS_MAX_DELAY][2], pending duty cycles included;
 *   - the simulator-frame pose and the per-step outputs that dts_get_state points to: pos_x pos_z angle speed reward
 *     lane_dist lane_dot lane_angle_rad prox_penalty wheel_dist step_count tile_i tile_j map_id episode done_code
 *     in_lane collided;
 *   - the env's numpy PCG64 stream (as dts_seed_streams takes it);
 *   - the per-episode render record (camera height / angle / fov and noise, horizon, light, ground colour, hidden
 *     objects: dts_debug_episode's 144 bytes);
 *   - for EVERY map slot that has dynamic obstacles, the env's copy of that map's obstacle state (dts_get_dyn_state,
 *     the traffic lights' shared card included): an env that comes back to a map finds its obstacles where it left them.
 * Not in a record, because they are not env state: reset staging buffers, frame memory, output buffers and the
 * handle's configuration (camera size, output format, resize, render mode, timing, flags, frame_rate, DR table).
 * Loading records into a handle configured differently is the caller's business.
 *
 * dts_state_info: record_bytes = one env's record size (a multiple of 16); fingerprint = a hash of the record layout
 * version, DTS_MAX_DELAY and, per map slot, the content of the map uploaded there (0 for an empty slot).  Any map
 * upload changes it, so records saved before one no longer load.  Host only. */
int dts_state_info(dts_sim* sim, uint64_t* record_bytes, uint64_t* fingerprint);
/* Every env's record -> records_dev, device u8[num_envs][record_bytes].  One launch, stream-ordered, never synchronises. */
int dts_save_state(dts_sim* sim, void* records_dev, void* stream);
/* Every env e of mask_dev (device u8[num_envs]; NULL = all) takes record e of records_dev as its complete state.
 * `fingerprint` is the dts_state_info fingerprint of the handle that saved them: it is checked on the host first, and
 * on a mismatch nothing is launched, no env changes and the call fails.  A record whose map_id names no uploaded map
 * is not loaded (the env keeps its state) and sets status bit 1.  One launch, never synchronises.  Device resets are
 * allowed afterwards, as after dts_seed_streams: the streams came with the records. */
int dts_load_state(dts_sim* sim, const uint8_t* mask_dev, const void* records_dev, uint64_t fingerprint, void* stream);
/* Per-kernel device timing of the render launches (bench.py's roofline): when enabled, every dts_render brackets its
 * kernels with CUDA events on the caller's stream.  dts_profile_read synchronises, returns the summed milliseconds of
 * [0] k_frame_setup, [1] k_geometry, [2] k_bin, [3] k_raster, [4] post passes (resize) and the number of frames
 * they cover, and clears the accumulators. */
int dts_profile_enable(dts_sim* sim, int level);   /* 0 off; 1 events around k_raster only; 2 around every render kernel */
int dts_profile_read(dts_sim* sim, double ms_out[8], int64_t* frames);
/* FUSED end-of-rollout gather (the path's one exchange step, SURVEY 8e) — instead of running an all-gather after the last
 * step, the last step's rasteriser stores every frame straight into the gather buffers of all GPUs of the box:
 *   dts_gather_alloc   this rank's buffer u8[world][bytes_per_rank] (returned in *buf_dev) and its 64-byte cudaIpc handle;
 *   dts_gather_open    the other ranks' handles (the caller exchanges them, e.g. torch.distributed all_gather), mapped
 *                      as peer memory (NVLink / NVSwitch);
 *   dts_gather_next    the NEXT dts_step / dts_render also writes its observations, in the selected layout / dtype,
 *                      to slot `rank` of every rank's buffer while it rasterises (one extra store per peer and word).
 * A rank's buffer is complete once every rank's step has finished: the caller orders that (stream sync + barrier), exactly
 * as it orders the use of an all-gather's output.  dts_allgather_obs remains as the NCCL baseline of the same exchange.
 * Slot `rank` starts at byte rank * bytes_per_rank, and the armed dts_step / dts_render writes its first num_envs * cam_h *
 * cam_w * 3 * elem bytes (elem 1 for DTS_OBS_U8, 4 for DTS_OBS_F32_UNIT); no call writes the rest of the buffer, which
 * dts_gather_alloc zeroes.
 * bytes_per_rank is fixed here, so:
 *   dts_gather_next    fails, and does not arm, while that batch is larger than bytes_per_rank;
 *   dts_step, dts_render  fail while a gather is armed and a resize target is set (dts_set_resize: the gather carries the
 *                      rasteriser's camera-sized output) or the batch, in the current output format, is larger than
 *                      bytes_per_rank.  They check before launching anything: a refused call runs no step logic, writes
 *                      no buffer and leaves the gather armed;
 *   dts_step_terminal  fails while a gather is armed (it does not write one).
 * dts_gather_alloc fails for a rank outside [0, world), a world outside [1, 8], and on a handle that has
 * allocated one already; dts_gather_next fails before dts_gather_alloc and before dts_gather_open has mapped every other
 * rank's buffer. */
int dts_gather_alloc(dts_sim* sim, uint64_t bytes_per_rank, int rank, int world, uint8_t handle_out[64], void** buf_dev);
int dts_gather_open(dts_sim* sim, const uint8_t* handles /* [world][64] */);
int dts_gather_next(dts_sim* sim);
/* Number of kernel launches issued by this handle so far (bench.py's gpu_launches). */
uint64_t dts_launch_count(dts_sim* sim);
/* debug: the env's per-episode render record as 36 x 32-bit words (cam_height, cam_angle_deg, cam_fov_y_deg, -,
 * cam_noise[3], -, horizon[3], -, ambient[3], -, diffuse[3], -, light_eye[4], ground[3], -, hidden u32[8]). */
int dts_debug_episode(dts_sim* sim, int env, void* out144);
/* debug (tests/test_gpu_gltrace.py): what k_frame_setup / k_geometry produced for `env` in the last dts_render — camera
 * model-view V (row-major 3x4, float64), projection P00 P11 P22 P23, counts = {prims, lattices, overflow, (prim, bin) pairs of the whole batch}, and the lit
 * 8x8 lattice [n_cells][64][3] of every emitted road tile by grid cell i * grid_h + j (NaN where culled).  Synchronises. */
int dts_debug_frame(dts_sim* sim, int env, double V[12], float P[4], int32_t counts[4], float* lattice_by_cell, int n_cells);
/* 32 diagnostic counters: [0] != 0 -> a render scratch buffer overflowed (frame incomplete). */
int dts_debug_counters(dts_sim* sim, int32_t out[32]);
/* debug (tests/test_gpu_np_streams.py): every env's numpy PCG64 stream as out_host[N][6] = state_hi, state_lo, inc_hi,
 * inc_lo, has_uint32, uinteger — the layout dts_seed_streams takes.  Synchronises. */
int dts_debug_streams(dts_sim* sim, uint64_t* out_host);
/* debug: one short program of draws, run by every env from its own stream through the NpStream methods the device
 * resets call.  Op k draws `count` values of `kind`; draw i of the program goes to out_dev[env][i] (u64[N][total]):
 * integers as int64, doubles as their bit patterns, next32 zero-extended.  The env's stream advances as the draws
 * did.  Device output, stream-ordered; integers need lo < hi, as numpy does. */
enum { DTS_DRAW_NEXT64 = 0,   /* bit_generator.random_raw() */
       DTS_DRAW_NEXT32 = 1,   /* integers(0, 2**32, dtype=np.uint32) */
       DTS_DRAW_UNIFORM = 2,  /* uniform(a, b) */
       DTS_DRAW_INTEGERS = 3, /* integers(lo, hi) */
       DTS_DRAW_NORMAL = 4    /* normal(a, b) */ };
typedef struct {
  int32_t kind, count;
  double a, b;              /* uniform / normal */
  int64_t lo, hi;           /* integers */
} dts_draw_op;
int dts_debug_draw(dts_sim* sim, const dts_draw_op* ops, int n_ops, uint64_t* out_dev, void* stream);
const char* dts_last_error(dts_sim* sim); /* sim may be NULL: error of the last failed dts_create */
void dts_destroy(dts_sim* sim);

#ifdef __cplusplus
}
#endif
#endif /* DTSIM_H */
