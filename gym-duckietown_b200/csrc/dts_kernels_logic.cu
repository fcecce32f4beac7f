// dts_kernels_logic.cu — one thread per env: Simulator.step() minus rendering, resets, pose queries.
// HBM traffic per env-step: ~30 doubles read + ~20 written (SoA, coalesced); the map (grid, curves,
// OBBs) is a few KB shared by all envs and stays in L1/L2.  Latency-bound, reported as us/launch.
#include "dts_camera.cuh"
#include "dts_kernels.h"
#include "dts_logic.cuh"

namespace dts {

__device__ __forceinline__ void default_render_ep(RenderEp& r) {
  r.cam_height = 0.108f; r.cam_angle_deg = 19.15f; r.cam_fov_y_deg = 75.0f; r.pad0 = 0;   // S:119-127
  r.cam_noise[0] = r.cam_noise[1] = r.cam_noise[2] = 0.f; r.pad1 = 0;
  r.horizon[0] = 0.45f; r.horizon[1] = 0.82f; r.horizon[2] = 1.0f; r.pad2 = 0;             // BLUE_SKY S:108
  r.ambient[0] = r.ambient[1] = r.ambient[2] = 0.25f; r.pad3 = 0;                          // 0.5*DIM S:573
  r.diffuse[0] = r.diffuse[1] = r.diffuse[2] = 0.35f; r.pad4 = 0;                          // 0.7*DIM S:575
  r.light_eye[0] = 0.f; r.light_eye[1] = 3.f; r.light_eye[2] = 0.f; r.light_eye[3] = 1.f;  // S:570, identity modelview
  r.ground[0] = r.ground[1] = r.ground[2] = 0.15f; r.pad5 = 0;                             // S:228
  for (int k = 0; k < 8; k++) r.hidden[k] = 0u;
}

// Fill the per-step outputs for the env's current pose: get_agent_info fields + _compute_done_reward S:1685-1705.
// `arrival`: DuckietownNav.step's goal test, which overrides whatever _compute_done_reward decided (a step's only).
__device__ inline void evaluate_pose(const DState& S, const DMap& m, const StepCfg& c, int e, double px, double pz,
                                     double ang, int step_count, float* reward, uint8_t* done, bool arrival = false) {
  int ti, tj;
  tile_at(m, px, pz, ti, tj);
  const DynRef dyn = dyn_ref(m, S.n, e);
  const LanePose lp = lane_pose(m, px, pz, ang);
  const double pen = proximity_penalty(m, px, pz, ang) + dynamic_proximity(dyn, px, pz, ang);   // S:1454-1457
  bool hit;
  const bool ok = valid_pose(m, dyn, px, pz, ang, 1.0, &hit);
  double rew;
  uint8_t code;
  if (!ok) { rew = kRewardInvalidPose; code = DTS_INVALID_POSE; }
  else if (step_count >= c.max_steps) { rew = 0.0; code = DTS_MAX_STEPS; }
  else {
    code = DTS_IN_PROGRESS;
    rew = lp.in_lane ? (+1.0 * c.robot_speed * lp.dot_dir + -10 * fabs(lp.dist) + +40 * pen) : 40 * pen;  // S:1654-1667
  }
  if (arrival && ti == S.goal_i[e] && tj == S.goal_j[e]) { rew = kRewardGoal; code = DTS_GOAL_REACHED; }   // envs/duckietown_env.py:119-125
  S.tile_i[e] = ti; S.tile_j[e] = tj;
  S.lane_dist[e] = lp.dist; S.lane_dot[e] = lp.dot_dir; S.lane_angle[e] = lp.angle_rad; S.in_lane[e] = lp.in_lane;
  S.prox[e] = pen; S.collided[e] = hit; S.reward[e] = rew; S.done_code[e] = code;
  if (reward) {
    double out = rew;
    if (c.reward_mode == DTS_REWARD_DT) out = rew == -1000.0 ? -10.0 : (rew > 0 ? rew + 10 : rew + 4);   // LW:94-102
    reward[e] = (float)out;
  }
  if (done) done[e] = code != DTS_IN_PROGRESS;
}

__device__ __forceinline__ void load_stream(const DState& S, int e, NpStream& rs) {
  const int n = S.n;
  rs.state = ((unsigned __int128)S.rng[0 * n + e] << 64) | S.rng[1 * n + e];
  rs.inc = ((unsigned __int128)S.rng[2 * n + e] << 64) | S.rng[3 * n + e];
  rs.has32 = (uint32_t)S.rng[4 * n + e];
  rs.cache32 = (uint32_t)S.rng[5 * n + e];
}
__device__ __forceinline__ void store_stream(const DState& S, int e, const NpStream& rs) {
  const int n = S.n;
  S.rng[0 * n + e] = (uint64_t)(rs.state >> 64); S.rng[1 * n + e] = (uint64_t)rs.state;
  S.rng[4 * n + e] = rs.has32; S.rng[5 * n + e] = rs.cache32;
}

__device__ inline void set_pose(const DState& S, const DMap& m, int e, double px, double pz, double ang) {
  S.pos_x[e] = px; S.pos_z[e] = pz; S.angle[e] = ang;
  S.cx[e] = px; S.cy[e] = m.grid_h * m.tile_size - pz; S.ctheta[e] = ang;   // cartesian_from_weird S:1629-1638
  S.vu[e] = 0.0; S.vw[e] = 0.0;                                           // init_vel = 0 S:743
  for (int k = 0; k < DTS_MAX_DELAY; k++) { S.fifo[(k * 2 + 0) * S.n + e] = 0.0; S.fifo[(k * 2 + 1) * S.n + e] = 0.0; }
  S.step_count[e] = 0; S.speed[e] = 0.0;                                  // S:535-539
}

// _load_map re-creates the map's objects (S:541-544 under randomize_maps_on_reset): this env's obstacles go back
// to their load-time state.
__device__ inline void reinit_dynamic(const DMap& m, int n, int e) {
  for (int k = 0; k < DTS_DYN_FIELDS * m.n_dyn; k++) m.dyn_state[(size_t)k * n + e] = m.dyn_init[k];
}

// Device-side Simulator.reset() (S:528-763): DR sampling + spawn rejection loop on the env's numpy-compatible
// PCG64 stream, draw for draw in the reference's order (randomizer.py:46-89 sorted keys, then S:551-736).
__device__ inline void respawn(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, int e) {
  const int n = S.n;
  NpStream rs;
  load_stream(S, e, rs);
  const bool dr = (c.flags & DTS_FLAG_DOMAIN_RAND) != 0;
  RenderEp old = S.rep[e];
  double Vprev[12];
  camera_view(S.pos_x[e], S.pos_z[e], S.angle[e], old, dr, Vprev);
  const bool first = S.episode[e] == 0;
  int mid = S.map_id[e];
  if (n_maps_cycle > 0 && !first) mid = (mid + 1) % n_maps_cycle;   // MultiMapEnv.reset envs/multimap_env.py:44-49
  if (n_maps_cycle < 0) mid = rs.integers(0, -n_maps_cycle);          // np_random.choice(map_names) S:541-542
  S.map_id[e] = mid;
  const DMap& m = maps[mid];
  if (n_maps_cycle < 0) reinit_dynamic(m, n, e);                     // _load_map S:544
  RenderEp r;
  default_render_ep(r);
  // Randomizer.randomize: every key of the table in sorted order — drawn whether or not DR is on
  // (randomizer.py:33,46-89, S:546); c.dr_ops is default_dr.json unless the caller supplied its own table
  double cam_angle = 1.0, cam_fov = 1.0, cam_h = 1.0, noise[3] = {0.0, 0.0, 0.0}, lp3[3] = {0.0, 3.0, 0.0}, trim = 0.0;
  int horz = 0;
  for (int oi = 0; oi < c.n_dr_ops; oi++) {
    const dts_dr_op& op = c.dr_ops[oi];
    for (int k = 0; k < op.size; k++) {
      const int kk = (op.size <= 3) ? k : 0;
      double v;
      if (op.type == DTS_DR_INT) v = (double)rs.integers((int64_t)op.a[kk], (int64_t)op.b[kk]);
      else if (op.type == DTS_DR_UNIFORM) v = rs.uniform(op.a[kk], op.b[kk]);
      else v = rs.normal(op.a[kk], op.b[kk]);
      switch (op.target) {
        case DTS_DR_CAMERA_ANGLE: if (k == 0) cam_angle = v; break;
        case DTS_DR_CAMERA_FOV_Y: if (k == 0) cam_fov = v; break;
        case DTS_DR_CAMERA_HEIGHT: if (k == 0) cam_h = v; break;
        case DTS_DR_CAMERA_NOISE: if (k < 3) noise[k] = v; break;
        case DTS_DR_HORZ_MODE: if (k == 0) horz = (int)v; break;
        case DTS_DR_LIGHT_POS: if (k < 3) lp3[k] = v; break;
        case DTS_DR_TRIM: if (k == 0) trim = v; break;
        default: break;
      }
    }
  }
  float lpos[4] = {0.f, 3.f, 0.f, 1.f};
  for (int k = 0; k < 3; k++) { r.horizon[k] = (float)c.color_sky[k]; r.ground[k] = (float)c.color_ground[k]; }   // S:562, S:594
  double wheel = 0.102;
  if (dr) {
    const double base[4][3] = {{c.color_sky[0], c.color_sky[1], c.color_sky[2]},
                               {0.64, 0.71, 0.28}, {0.15, 0.15, 0.15}, {0.9, 0.9, 0.9}};
    if (horz >= 0 && horz < 4) {                                              // S:551-560
      const double hs = horz < 2 ? 0.1 : 0.4;
      for (int k = 0; k < 3; k++) r.horizon[k] = (float)(base[horz][k] * rs.uniform(1.0 - hs, 1.0 + hs));
    } else {
      for (int k = 0; k < 3; k++) r.horizon[k] = old.horizon[k];              // no branch taken: the attribute keeps its value
    }
    lpos[0] = (float)lp3[0]; lpos[1] = (float)lp3[1]; lpos[2] = (float)lp3[2]; lpos[3] = 0.f;  // 3 floats into a 4-array: w = 0
    double p4[4];
    for (int k = 0; k < 4; k++) p4[k] = rs.uniform(1.0 - 0.3, 1.0 + 0.3);     // _perturb(ambient, 0.3) S:574
    for (int k = 0; k < 3; k++) r.ambient[k] = (float)(0.25 * p4[k]);
    for (int k = 0; k < 4; k++) p4[k] = rs.uniform(1.0 - 0.99, 1.0 + 0.99);   // _perturb(diffuse, 0.99) S:576
    for (int k = 0; k < 3; k++) r.diffuse[k] = (float)(0.35 * p4[k]);
    for (int k = 0; k < 3; k++) r.ground[k] = (float)(c.color_ground[k] * rs.uniform(1.0 - 0.3, 1.0 + 0.3));  // S:594
    wheel = 0.102 * rs.uniform(1.0 - 0.1, 1.0 + 0.1);                         // S:597
    for (int k = 0; k < 3; k++) r.cam_noise[k] = (float)noise[k];             // S:1768: domain_rand only
  }
  if (dr || (c.flags & DTS_FLAG_CAMERA_RAND)) {                               // S:611-614: domain_rand or camera_rand
    r.cam_height = (float)(0.108 * cam_h);
    r.cam_angle_deg = (float)(19.15 * cam_angle);
    r.cam_fov_y_deg = (float)(75.0 * cam_fov);
  }
  // distractor triangles S:621-629: never visible (below the ground plane) but their draws are consumed
  for (int t = 0; t < 3 * c.num_tris_distractors; t++) {
    rs.next64(); rs.next64(); rs.next64();      // uniform(low=[-20,-0.6,-20], high=[20,-0.3,20], size=3)
    rs.next64();                                // c = uniform(0, 0.9)
    if (dr) { rs.next64(); rs.next64(); rs.next64(); }   // _perturb([c,c,c], 0.1)
  }
  if (dr) {
    for (int t = 0; t < m.n_tiles; t++)         // tile["color"] = _perturb([1,1,1,1], 0.2) S:645 (no visible effect)
      if (m.tile_kind[t] >= 0) { rs.next64(); rs.next64(); rs.next64(); rs.next64(); }
    for (int o = 0; o < m.n_objects; o++) {     // S:648-656
      rs.next64(); rs.next64(); rs.next64(); rs.next64();   // obj.color = _perturb([1,1,1,1], 0.3)
      if (m.objects[o].optional && !(rs.integers(0, 2) == 0)) r.hidden[o >> 5] |= 1u << (o & 31);
    }
  }
  if (first) { for (int k = 0; k < 4; k++) r.light_eye[k] = lpos[k]; }       // identity modelview at first reset
  else light_to_eye(Vprev, lpos, r.light_eye);                               // stale modelview S:581
  S.wheel_dist[e] = wheel;
  S.trim[e] = (c.flags & DTS_FLAG_DYNAMICS_RAND) ? trim : 0.0;               // S:746-750
  // start tile S:659-676, spawn loop S:692-736
  int ti = 0, tj = 0;
  if (m.start_i >= 0) { ti = m.start_i; tj = m.start_j; }
  else if (m.n_drivable > 0) { const int t = rs.integers(0, m.n_drivable); ti = m.drivable_ij[2 * t]; tj = m.drivable_ij[2 * t + 1]; }
  double px = 1.0, pz = 1.0, ang = 1.0;                                      // fallback S:735-736
  const DynRef dyn = dyn_ref(m, n, e);
  if (m.has_start_pose) {   // S:679-686: the map fixes the pose inside the start tile; nothing is drawn
    px = ti * m.tile_size + m.start_pose[0]; pz = tj * m.tile_size + m.start_pose[1]; ang = m.start_pose[2];
  }
  for (int attempt = 0; attempt < kMaxSpawnAttempts && m.n_drivable > 0 && !m.has_start_pose; attempt++) {
    const double x = rs.uniform((double)ti, (double)(ti + 1)) * m.tile_size, z = rs.uniform((double)tj, (double)(tj + 1)) * m.tile_size;
    const double a = rs.uniform(0.0, 2 * 3.141592653589793);
    if (inconvenient_spawn(m, dyn, r.hidden, x, z)) continue;
    if (!valid_pose(m, dyn, x, z, a, 1.3, nullptr)) continue;
    const LanePose lp = lane_pose(m, x, z, a);
    if (!lp.in_lane) continue;
    const double deg = lp.angle_rad * 57.29577951308232;                    // np.rad2deg S:1406
    if (!(-c.accept_angle_deg < deg && deg < c.accept_angle_deg)) continue;
    px = x; pz = z; ang = a;
    break;
  }
  if (c.flags & DTS_FLAG_NAV) {   // DuckietownNav.reset: a goal tile other than the start's (upload keeps n_drivable >= 2)
    int si, sj, gi, gj;
    tile_at(m, px, pz, si, sj);
    do {
      const int t = rs.integers(0, m.n_drivable);
      gi = m.drivable_ij[2 * t]; gj = m.drivable_ij[2 * t + 1];
    } while (gi == si && gj == sj);
    S.goal_i[e] = (uint8_t)gi; S.goal_j[e] = (uint8_t)gj;
  }
  set_pose(S, m, e, px, pz, ang);
  S.rep[e] = r;
  store_stream(S, e, rs);
  S.episode[e] += 1;
}

__global__ void __launch_bounds__(128) k_step_logic(DState S, const DMap* __restrict__ maps, StepCfg c,
                                                    int n_maps_cycle, const float* __restrict__ actions,
                                                    float* __restrict__ reward, uint8_t* __restrict__ done) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n) return;
  const DMap& m = maps[S.map_id[e]];
  const float2 act = reinterpret_cast<const float2*>(actions)[e];
  double a0 = (double)act.x, a1 = (double)act.y;
  if (c.action_map == DTS_ACTIONS_DISCRETE3) {            // DiscreteWrapper.action W:18-30
    const int id = (int)act.x;
    a0 = id == 2 ? 0.7 : 0.6;
    a1 = id == 0 ? 1.0 : (id == 1 ? -1.0 : 0.0);
  }
  a0 = a0 * c.action_vel_scale;                           // ActionWrapper.action LW:110-112 (scale 1.0: exact no-op)
  double ul = a0, ur = a1;
  if (c.action_mode == DTS_ACTION_VEL_STEER) action_to_pwm(a0, a1, S.wheel_dist[e], c, ul, ur);
  ul = clampd(ul, -1.0, 1.0);   // np.clip S:1670
  ur = clampd(ur, -1.0, 1.0);
  double x = S.cx[e], y = S.cy[e], th = S.ctheta[e], u = S.vu[e], w = S.vw[e];
  double px = S.pos_x[e], pz = S.pos_z[e], ang = S.angle[e], speed = 0.0;
  int steps = S.step_count[e];
  const double trim = S.trim[e];
  const int D = c.dyn.delay_steps;
  const DynRef dyn = dyn_ref(m, S.n, e);
  NpStream rs;
  const bool dyn_rand = dyn.n_dyn > 0 && (c.flags & DTS_FLAG_DOMAIN_RAND) && (S.rng[3 * S.n + e] & 1ull);  // seeded stream
  if (dyn_rand) load_stream(S, e, rs);
  for (int f = 0; f < c.frame_skip; f++) {   // update_physics S:1551-1584
    double l = ul, r = ur;
    if (D > 0) {  // delay line: the command issued now acts D steps later
      l = S.fifo[0 * S.n + e]; r = S.fifo[1 * S.n + e];
      for (int k = 0; k + 1 < D; k++) {
        S.fifo[(2 * k) * S.n + e] = S.fifo[(2 * k + 2) * S.n + e];
        S.fifo[(2 * k + 1) * S.n + e] = S.fifo[(2 * k + 3) * S.n + e];
      }
      S.fifo[(2 * (D - 1)) * S.n + e] = ul; S.fifo[(2 * (D - 1) + 1) * S.n + e] = ur;
    }
    const double ppx = px, ppz = pz;
    dynamics_step(x, y, th, u, w, l, r, c.dyn, trim, c.dt);
    px = x; pz = m.grid_h * m.tile_size - y;          // weird_from_cartesian S:1640-1652
    double sn, cs;
    sincos(th, &sn, &cs);
    ang = atan2(sn, cs);
    steps++;
    speed = sqrt((px - ppx) * (px - ppx) + (pz - ppz) * (pz - ppz)) / c.dt;
    if (dyn.n_dyn > 0) dyn_step_all(m, dyn, c.dt, dyn_rand ? &rs : nullptr);   // S:1570-1584
  }
  if (dyn_rand) store_stream(S, e, rs);
  S.cx[e] = x; S.cy[e] = y; S.ctheta[e] = th; S.vu[e] = u; S.vw[e] = w;
  S.pos_x[e] = px; S.pos_z[e] = pz; S.angle[e] = ang; S.speed[e] = speed; S.step_count[e] = steps;
  evaluate_pose(S, m, c, e, px, pz, ang, steps, reward, done, (c.flags & DTS_FLAG_NAV) != 0);
  if ((c.flags & DTS_FLAG_AUTO_RESET) && S.done_code[e] != DTS_IN_PROGRESS) respawn(S, maps, c, n_maps_cycle, e);
}

__global__ void __launch_bounds__(128) k_reset_random(DState S, const DMap* __restrict__ maps, StepCfg c,
                                                      int n_maps_cycle, const uint8_t* __restrict__ mask) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n || (mask && !mask[e])) return;
  respawn(S, maps, c, n_maps_cycle, e);
  const DMap& m = maps[S.map_id[e]];
  evaluate_pose(S, m, c, e, S.pos_x[e], S.pos_z[e], S.angle[e], 0, nullptr, nullptr);
}

// dts_step_terminal's auto-reset, run after the terminal frames are rendered: k_step_logic ran with
// DTS_FLAG_AUTO_RESET cleared, so this is the same respawn() on the same state, and the env's PCG64 stream continues
// where the step's dyn_rand draws left it.  The envs that respawn are appended to `ended` (warp-aggregated).
__global__ void __launch_bounds__(128) k_respawn_ended(DState S, const DMap* __restrict__ maps, StepCfg c, int n_maps_cycle,
                                                       int32_t* __restrict__ ended, int32_t* __restrict__ n_ended) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const bool end = e < S.n && S.done_code[e] != DTS_IN_PROGRESS;
  const unsigned m = __ballot_sync(0xffffffffu, end);
  if (!m) return;
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == __ffs(m) - 1) base = atomicAdd(n_ended, __popc(m));
  base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
  if (!end) return;
  ended[base + __popc(m & ((1u << lane) - 1u))] = e;
  respawn(S, maps, c, n_maps_cycle, e);
}

// dts_reset with host-drawn parameters (already copied to device staging arrays in `p`)
__global__ void __launch_bounds__(128) k_reset_params(DState S, const DMap* __restrict__ maps, StepCfg c,
                                                      const uint8_t* __restrict__ mask, dts_episode_params p) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n || (mask && !mask[e])) return;
  RenderEp old = S.rep[e];
  double Vprev[12];
  camera_view(S.pos_x[e], S.pos_z[e], S.angle[e], old, (c.flags & DTS_FLAG_DOMAIN_RAND) != 0, Vprev);
  if (p.map_id) S.map_id[e] = p.map_id[e];
  const DMap& m = maps[S.map_id[e]];
  if (c.random_maps > 0) reinit_dynamic(m, S.n, e);   // the host drew the map (S:541-544): objects are re-created
  RenderEp r;
  default_render_ep(r);
  for (int k = 0; k < 3; k++) { r.horizon[k] = (float)c.color_sky[k]; r.ground[k] = (float)c.color_ground[k]; }
  if (p.cam_height) r.cam_height = p.cam_height[e];
  if (p.cam_angle_deg) r.cam_angle_deg = p.cam_angle_deg[e];
  if (p.cam_fov_y_deg) r.cam_fov_y_deg = p.cam_fov_y_deg[e];
  float lpos[4] = {0.f, 3.f, 0.f, 1.f};
  for (int k = 0; k < 3; k++) {
    if (p.cam_noise) r.cam_noise[k] = p.cam_noise[3 * e + k];
    if (p.horizon_color) r.horizon[k] = p.horizon_color[3 * e + k];
    if (p.light_ambient) r.ambient[k] = p.light_ambient[3 * e + k];
    if (p.light_diffuse) r.diffuse[k] = p.light_diffuse[3 * e + k];
    if (p.ground_color) r.ground[k] = p.ground_color[3 * e + k];
  }
  if (p.light_pos) for (int k = 0; k < 4; k++) lpos[k] = p.light_pos[4 * e + k];
  if (p.light_stale && p.light_stale[e]) light_to_eye(Vprev, lpos, r.light_eye);
  else for (int k = 0; k < 4; k++) r.light_eye[k] = lpos[k];
  if (p.obj_hidden) for (int k = 0; k < 8; k++) r.hidden[k] = p.obj_hidden[8 * e + k];
  S.wheel_dist[e] = p.wheel_dist ? p.wheel_dist[e] : 0.102;
  S.trim[e] = p.trim ? p.trim[e] : 0.0;
  const double px = p.pos_x ? p.pos_x[e] : 1.0, pz = p.pos_z ? p.pos_z[e] : 1.0, ang = p.angle ? p.angle[e] : 1.0;
  set_pose(S, m, e, px, pz, ang);
  S.rep[e] = r;
  S.episode[e] += 1;
  evaluate_pose(S, m, c, e, px, pz, ang, 0, nullptr, nullptr);
}

// dts_set_goals: a host reset's goal tiles.  One that is not a drivable tile of its env's map is not taken: the env
// keeps its goal and `refused` (a status word) is set
__global__ void __launch_bounds__(128) k_set_goals(DState S, const DMap* __restrict__ maps, const uint8_t* __restrict__ mask,
                                                   const int16_t* __restrict__ goals, int32_t* refused) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n || (mask && !mask[e])) return;
  const DMap& m = maps[S.map_id[e]];
  const int gi = goals[2 * e], gj = goals[2 * e + 1];
  const int idx = gj * m.grid_w + gi;
  if (gi < 0 || gi >= m.grid_w || gj < 0 || gj >= m.grid_h || m.tile_kind[idx] < 0 || !m.tile_drivable[idx]) {
    *reinterpret_cast<volatile int32_t*>(refused) = 1;
    return;
  }
  S.goal_i[e] = (uint8_t)gi; S.goal_j[e] = (uint8_t)gj;
}

// randomize_maps_on_reset with a host-drawn map (S:541-544): new map id + its obstacles re-created (_load_map),
// nothing else — pose, episode counter and render record stay those of the episode that just ended, so the reset
// that follows captures GL_LIGHT0 under the right stale modelview (S:581).
__global__ void __launch_bounds__(128) k_assign_maps(DState S, const DMap* __restrict__ maps,
                                                     const uint8_t* __restrict__ mask, const int32_t* __restrict__ map_id) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n || (mask && !mask[e])) return;
  S.map_id[e] = map_id[e];
  reinit_dynamic(maps[map_id[e]], S.n, e);
}

// Batched pose predicates for host callers: _valid_pose / _collision / get_lane_pos2 /
// proximity_penalty2 / _inconvenient_spawn of arbitrary poses (used by the host-side reset).
__global__ void __launch_bounds__(128) k_query(const DMap* __restrict__ maps, int map_id, int dyn_env, int n_envs, int n,
                                               const double* __restrict__ q /*[n][4] x z angle safety*/,
                                               const uint32_t* __restrict__ hidden /*[n][8] or null*/,
                                               double* __restrict__ outd /*[n][4] dist dot angle prox*/,
                                               int32_t* __restrict__ outi /*[n][8]*/) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const DMap& m = maps[map_id];
  const double x = q[4 * t], z = q[4 * t + 1], a = q[4 * t + 2], sf = q[4 * t + 3];
  const DynRef dyn = dyn_ref(m, n_envs, dyn_env);
  bool hit2;
  const bool ok = valid_pose(m, dyn, x, z, a, sf, &hit2);
  double sn, cs;
  sincos(a, &sn, &cs);
  const bool hit1 = agent_hits_static(m, x + kCentreOff * cs, z + kCentreOff * -sn, a) ||   // run_tests.py:50 usage
                    agent_hits_dynamic(dyn, x + kCentreOff * cs, z + kCentreOff * -sn, a);
  const LanePose lp = lane_pose(m, x, z, a);
  const bool bad = inconvenient_spawn(m, dyn, hidden ? hidden + 8 * t : nullptr, x, z);
  int ti, tj;
  const int idx = tile_at(m, x, z, ti, tj);
  outd[4 * t] = lp.dist; outd[4 * t + 1] = lp.dot_dir; outd[4 * t + 2] = lp.angle_rad;
  outd[4 * t + 3] = proximity_penalty(m, x, z, a) + dynamic_proximity(dyn, x, z, a);
  outi[8 * t] = ok; outi[8 * t + 1] = hit1; outi[8 * t + 2] = hit2; outi[8 * t + 3] = lp.in_lane;
  outi[8 * t + 4] = bad; outi[8 * t + 5] = ti; outi[8 * t + 6] = tj;
  outi[8 * t + 7] = idx >= 0 && m.tile_drivable[idx];
}

// dts_debug_draw: the env's stream runs a program of NpStream calls; draw i -> out[e * total + i]
__global__ void __launch_bounds__(128) k_debug_draw(DState S, const dts_draw_op* __restrict__ ops, int n_ops, int64_t total,
                                                    uint64_t* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n) return;
  NpStream rs;
  load_stream(S, e, rs);
  uint64_t* o = out + (size_t)e * total;
  for (int k = 0; k < n_ops; k++) {
    const dts_draw_op op = ops[k];
    for (int i = 0; i < op.count; i++) {
      uint64_t v;
      switch (op.kind) {
        case DTS_DRAW_NEXT64: v = rs.next64(); break;
        case DTS_DRAW_NEXT32: v = rs.next32(); break;
        case DTS_DRAW_UNIFORM: v = (uint64_t)__double_as_longlong(rs.uniform(op.a, op.b)); break;
        case DTS_DRAW_INTEGERS: v = (uint64_t)rs.integers(op.lo, op.hi); break;
        default: v = (uint64_t)__double_as_longlong(rs.normal(op.a, op.b)); break;
      }
      *o++ = v;
    }
  }
  store_stream(S, e, rs);
}

// ------------------------------------------------------------------ launchers
void launch_step_logic(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, const float* actions,
                       float* reward, uint8_t* done, cudaStream_t st) {
  k_step_logic<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, c, n_maps_cycle, actions, reward, done);
}
void launch_reset_random(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, const uint8_t* mask,
                         cudaStream_t st) {
  k_reset_random<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, c, n_maps_cycle, mask);
}
void launch_respawn_ended(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, int32_t* ended,
                          int32_t* n_ended, cudaStream_t st) {
  k_respawn_ended<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, c, n_maps_cycle, ended, n_ended);
}
void launch_reset_params(const DState& S, const DMap* maps, const StepCfg& c, const uint8_t* mask,
                         const dts_episode_params& p, cudaStream_t st) {
  k_reset_params<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, c, mask, p);
}
void launch_set_goals(const DState& S, const DMap* maps, const uint8_t* mask, const int16_t* goals, int32_t* refused,
                      cudaStream_t st) {
  k_set_goals<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, mask, goals, refused);
}
void launch_assign_maps(const DState& S, const DMap* maps, const uint8_t* mask, const int32_t* map_id, cudaStream_t st) {
  k_assign_maps<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, mask, map_id);
}
void launch_query(const DMap* maps, int map_id, int dyn_env, int n_envs, int n, const double* q, const uint32_t* hidden,
                  double* outd, int32_t* outi, cudaStream_t st) {
  k_query<<<(n + 127) / 128, 128, 0, st>>>(maps, map_id, dyn_env, n_envs, n, q, hidden, outd, outi);
}
void launch_debug_draw(const DState& S, const dts_draw_op* ops, int n_ops, int64_t total, uint64_t* out, cudaStream_t st) {
  k_debug_draw<<<(S.n + 127) / 128, 128, 0, st>>>(S, ops, n_ops, total, out);
}

}  // namespace dts
