// dts_logic.cuh — device functions for the non-rendering half of Simulator.step():
// action map, delayed PWM dynamics, tile lookup, valid-pose, OBB SAT, safety circles, lane pose,
// reward/done, and the device-side spawn.  float64 like the reference (numpy defaults).
// Citations: S = simulator.py, C = collision.py, G = graphics.py, E = envs/duckietown_env.py.
#pragma once
#include "dts_common.cuh"
#include "np_random.cuh"

namespace dts {

// robot constants S:118-177
constexpr double kRobotWidth = 0.13 + 0.02;
constexpr double kRobotLength = 0.18;
constexpr double kCamForward = 0.066;
constexpr double kCentreOff = kCamForward - (kRobotLength / 2);          // _actual_center S:2109
constexpr double kAgentSafetyRad = ((kRobotLength > kRobotWidth ? kRobotLength : kRobotWidth) / 2) * 1.8;  // S:153
constexpr double kRewardInvalidPose = -1000.0;                           // S:175
constexpr double kRewardGoal = 1000.0;                                   // DuckietownNav.step envs/duckietown_env.py:125
constexpr int kMaxSpawnAttempts = 5000;                                  // S:177

struct LanePose { double dist, dot_dir, angle_rad; bool in_lane; };

__device__ __forceinline__ double clampd(double v, double lo, double hi) { return fmax(lo, fmin(hi, v)); }

// E:36-59 — [vel, steering] -> (u_left, u_right), clamped to +-limit
__device__ __forceinline__ void action_to_pwm(double vel, double steer, double baseline, const StepCfg& c,
                                              double& u_l, double& u_r) {
  const double k_r_inv = (c.gain + c.trim) / c.k;
  const double k_l_inv = (c.gain - c.trim) / c.k;
  const double omega_r = (vel + 0.5 * steer * baseline) / c.radius;
  const double omega_l = (vel - 0.5 * steer * baseline) / c.radius;
  u_r = fmax(fmin(omega_r * k_r_inv, c.limit), -c.limit);
  u_l = fmax(fmin(omega_l * k_l_inv, c.limit), -c.limit);
}

// get_grid_coords S:1134-1149 + _get_tile S:1053-1063. Returns flat tile index or -1.
__device__ __forceinline__ int tile_at(const DMap& m, double x, double z, int& i, int& j) {
  i = (int)floor(x / m.tile_size);
  j = (int)floor(z / m.tile_size);
  if (i < 0 || i >= m.grid_w || j < 0 || j >= m.grid_h) return -1;
  const int idx = j * m.grid_w + i;
  return m.tile_kind[idx] < 0 ? -1 : idx;
}
// _drivable_pos S:1411-1428
__device__ __forceinline__ bool drivable_at(const DMap& m, double x, double z) {
  int i, j;
  const int idx = tile_at(m, x, z, i, j);
  return idx >= 0 && m.tile_drivable[idx] != 0;
}

__device__ __forceinline__ void project4(double ax, double az, const double* xs, const double* zs, double& lo,
                                         double& hi) {
  double v = ax * xs[0] + az * zs[0];
  lo = v; hi = v;
#pragma unroll
  for (int k = 1; k < 4; k++) {
    v = ax * xs[k] + az * zs[k];
    lo = fmin(lo, v);
    hi = fmax(hi, v);
  }
}
// C:50-61 closed-interval overlap
__device__ __forceinline__ bool intervals_touch(double a0, double a1, double b0, double b1) {
  return (a0 <= b0 && b0 <= a1) || (b0 <= a0 && a0 <= b1);
}

// _collision S:1473-1492 / intersects C:129-159 for the agent box centred at (bx,bz).
// Agent SAT axes = right / forward unit vectors (eigenvectors of the 0.15x0.18 corner covariance,
// C:99-106, up to sign and order, to which the interval test is indifferent).
__device__ inline bool agent_hits_static(const DMap& m, double bx, double bz, double angle) {
  if (m.n_coll == 0) return false;
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double fx = cs, fz = -sn, rx = sn, rz = cs;  // get_dir_vec / get_right_vec S:2056-2073
  const double hw = 0.5 * kRobotWidth, hl = 0.5 * kRobotLength;
  double ax[4], az[4];  // agent_boundbox C:9-34 corner order
  ax[0] = bx - hw * rx - hl * fx; az[0] = bz - hw * rz - hl * fz;
  ax[1] = bx + hw * rx - hl * fx; az[1] = bz + hw * rz - hl * fz;
  ax[2] = bx + hw * rx + hl * fx; az[2] = bz + hw * rz + hl * fz;
  ax[3] = bx - hw * rx + hl * fx; az[3] = bz - hw * rz + hl * fz;
  double aR0, aR1, aF0, aF1;
  project4(rx, rz, ax, az, aR0, aR1);
  project4(fx, fz, ax, az, aF0, aF1);
  for (int k = 0; k < m.n_coll; k++) {
    const double* ox = m.coll_corners + k * 8;
    const double* oz = ox + 4;
    const double* on = m.coll_norms + k * 4;
    double lo, hi, lo2, hi2;
    project4(rx, rz, ox, oz, lo, hi);
    if (!intervals_touch(aR0, aR1, lo, hi)) continue;
    project4(fx, fz, ox, oz, lo, hi);
    if (!intervals_touch(aF0, aF1, lo, hi)) continue;
    project4(on[0], on[1], ax, az, lo, hi);
    project4(on[0], on[1], ox, oz, lo2, hi2);
    if (!intervals_touch(lo, hi, lo2, hi2)) continue;
    project4(on[2], on[3], ax, az, lo, hi);
    project4(on[2], on[3], ox, oz, lo2, hi2);
    if (!intervals_touch(lo, hi, lo2, hi2)) continue;
    return true;
  }
  return false;
}

__device__ inline bool agent_hits_dynamic(const DynRef& d, double bx, double bz, double angle);

// _valid_pose S:1494-1534.  NB the collision box is built from the already-shifted centre and
// get_agent_corners shifts it again (S:1502 + S:1521 -> S:2114): offset applied twice.
__device__ inline bool valid_pose(const DMap& m, const DynRef& d, double px, double pz, double angle, double safety,
                                  bool* collided) {
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double fx = cs, fz = -sn, rx = sn, rz = cs;
  const double qx = px + kCentreOff * fx, qz = pz + kCentreOff * fz;
  const double sw = safety * 0.5 * kRobotWidth, sl = safety * 0.5 * kRobotLength;
  const bool all_drivable = drivable_at(m, qx, qz) && drivable_at(m, qx - sw * rx, qz - sw * rz) &&
                            drivable_at(m, qx + sw * rx, qz + sw * rz) && drivable_at(m, qx + sl * fx, qz + sl * fz);
  const bool hit = agent_hits_static(m, qx + kCentreOff * fx, qz + kCentreOff * fz, angle) ||
                   agent_hits_dynamic(d, qx + kCentreOff * fx, qz + kCentreOff * fz, angle);   // S:1481-1489
  if (collided) *collided = hit;
  return !hit && all_drivable;
}

// proximity_penalty2 S:1430-1459 with C:189-211
__device__ inline double proximity_penalty(const DMap& m, double px, double pz, double angle) {
  if (m.n_coll == 0) return 0.0;
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double qx = px + kCentreOff * cs, qz = pz + kCentreOff * -sn;
  bool touching = false;
  double acc = 0.0;
  for (int k = 0; k < m.n_coll; k++) {
    const double* c = m.coll_centers + 3 * k;
    const double dx = c[0] - qx, dy = c[1], dz = c[2] - qz;
    const double d = sqrt(dx * dx + dy * dy + dz * dz);
    const double r2 = m.coll_radii[k];
    const double dif = kAgentSafetyRad - r2, sum = kAgentSafetyRad + r2;
    if ((dif * dif <= d * d && d * d <= sum * sum) || d < fabs(dif)) touching = true;
    const double s = d - kAgentSafetyRad - r2;
    if (s < 0) acc += s;
  }
  return touching ? acc : 0.0;
}

__device__ __forceinline__ void bezier_at(const double* cp, double t, double& x, double& y, double& z) {  // G:286-297
  const double s = 1 - t;
  const double b0 = s * s * s, b1 = 3 * t * (s * s), b2 = 3 * (t * t) * s, b3 = t * t * t;
  x = b0 * cp[0]; x += b1 * cp[3]; x += b2 * cp[6]; x += b3 * cp[9];
  y = b0 * cp[1]; y += b1 * cp[4]; y += b2 * cp[7]; y += b3 * cp[10];
  z = b0 * cp[2]; z += b1 * cp[5]; z += b2 * cp[8]; z += b3 * cp[11];
}

// closest_curve_point S:1337-1369: point q and unit tangent t of the tile's best-aligned curve; false off-road.
__device__ inline bool closest_curve_point(const DMap& m, double px, double pz, double angle, double q[3], double t3[3]) {
  int ti, tj;
  const int idx = tile_at(m, px, pz, ti, tj);
  if (idx < 0 || !m.tile_drivable[idx]) return false;
  const double* cv = m.curves + (size_t)m.tile_curve_off[idx] * 12;
  const int nc = m.tile_curve_cnt[idx];
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double dirx = cs, dirz = -sn;
  // argmax_c (P3-P0).dir — S:1355-1362 divide every chord by ONE Frobenius norm, kept for the rounding
  double fro = 0.0;
  for (int c = 0; c < nc; c++) {
    const double hx = cv[c * 12 + 9] - cv[c * 12], hy = cv[c * 12 + 10] - cv[c * 12 + 1], hz = cv[c * 12 + 11] - cv[c * 12 + 2];
    fro += hx * hx; fro += hy * hy; fro += hz * hz;
  }
  fro = sqrt(fro);
  int best = 0;
  double bestv = -1e300;
  for (int c = 0; c < nc; c++) {
    const double hx = (cv[c * 12 + 9] - cv[c * 12]) / fro, hz = (cv[c * 12 + 11] - cv[c * 12 + 2]) / fro;
    const double v = hx * dirx + hz * dirz;
    if (v > bestv) { bestv = v; best = c; }  // first maximum wins (np.argmax)
  }
  const double* cp = cv + best * 12;
  double lo = 0.0, hi = 1.0;  // bezier_closest G:316-333
#pragma unroll 1
  for (int lvl = 0; lvl < 8; lvl++) {
    const double mid = (lo + hi) * 0.5;
    double ax, ay, az, bx, by, bz;
    bezier_at(cp, lo, ax, ay, az);
    bezier_at(cp, hi, bx, by, bz);
    const double dlo = sqrt((ax - px) * (ax - px) + ay * ay + (az - pz) * (az - pz));
    const double dhi = sqrt((bx - px) * (bx - px) + by * by + (bz - pz) * (bz - pz));
    if (dlo < dhi) hi = mid; else lo = mid;
  }
  const double t = (lo + hi) * 0.5, s = 1 - t;
  bezier_at(cp, t, q[0], q[1], q[2]);
  double tx = 3 * (s * s) * (cp[3] - cp[0]); tx += 6 * s * t * (cp[6] - cp[3]); tx += 3 * (t * t) * (cp[9] - cp[6]);   // G:300-313
  double ty = 3 * (s * s) * (cp[4] - cp[1]); ty += 6 * s * t * (cp[7] - cp[4]); ty += 3 * (t * t) * (cp[10] - cp[7]);
  double tz = 3 * (s * s) * (cp[5] - cp[2]); tz += 6 * s * t * (cp[8] - cp[5]); tz += 3 * (t * t) * (cp[11] - cp[8]);
  const double nrm = sqrt(tx * tx + ty * ty + tz * tz);
  t3[0] = tx / nrm; t3[1] = ty / nrm; t3[2] = tz / nrm;
  return true;
}

// get_lane_pos2 S:1371-1409
__device__ inline LanePose lane_pose(const DMap& m, double px, double pz, double angle) {
  LanePose r;
  r.dist = r.dot_dir = r.angle_rad = __longlong_as_double(0x7ff8000000000000LL);
  r.in_lane = false;
  double q[3], t3[3];
  if (!closest_curve_point(m, px, pz, angle, q, t3)) return r;
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double dirx = cs, dirz = -sn, tx = t3[0], tz = t3[2];
  const double dd = clampd(dirx * tx + dirz * tz, -1.0, 1.0);
  const double rvx = -tz, rvz = tx;  // cross(tangent, +y)
  r.dist = (px - q[0]) * rvx + (pz - q[2]) * rvz;
  r.angle_rad = acos(dd);
  if (dirx * rvx + dirz * rvz < 0) r.angle_rad = -r.angle_rad;
  r.dot_dir = dd;
  r.in_lane = true;
  return r;
}

// ------------------------------------------------------------------ dynamic obstacles (objects.py, O:)
// DuckieObj.step O:396-422 + finish_walk O:424-432.  `rs` != nullptr: domain_rand draws (the reference takes them
// from the global numpy RNG; here the env's stream supplies them).
__device__ inline void duckie_step(const DynRef& d, int s, double dt, NpStream* rs) {
  const DDyn& p = d.par[s];
  const double time = d.f(DTS_DYN_TIME, s) + dt;
  d.f(DTS_DYN_TIME, s) = time;
  if (d.f(DTS_DYN_ACTIVE, s) == 0.0) {
    const double w = d.f(DTS_DYN_WAIT, s) - dt;
    d.f(DTS_DYN_WAIT, s) = w;
    if (w <= 0) d.f(DTS_DYN_ACTIVE, s) = 1.0;
    return;
  }
  double sn, cs;
  sincos(p.angle0, &sn, &cs);
  double vel = d.f(DTS_DYN_VEL, s);
  const double vx = cs * vel, vz = -sn * vel;                         // heading_vec C:222 * vel
  const double px = d.f(DTS_DYN_PX, s) + vx, pz = d.f(DTS_DYN_PZ, s) + vz;
  d.f(DTS_DYN_PX, s) = px; d.f(DTS_DYN_PZ, s) = pz;
#pragma unroll
  for (int k = 0; k < 4; k++) { d.f(DTS_DYN_CORNERS + 2 * k, s) += vx; d.f(DTS_DYN_CORNERS + 2 * k + 1, s) += vz; }
  const double dx = px - d.f(DTS_DYN_START_X, s), dz = pz - d.f(DTS_DYN_START_Z, s);
  double angle = d.f(DTS_DYN_ANGLE, s);
  if (sqrt(dx * dx + 0.0 + dz * dz) > p.walk_distance) {
    d.f(DTS_DYN_START_X, s) = px; d.f(DTS_DYN_START_Z, s) = pz;
    angle += 3.141592653589793;
    d.f(DTS_DYN_ANGLE, s) = angle;
    d.f(DTS_DYN_ACTIVE, s) = 0.0;
    if (rs) {
      vel = -1 * (vel > 0 ? 1.0 : (vel < 0 ? -1.0 : 0.0)) * fabs(rs->normal(0.02, 0.005));
      d.f(DTS_DYN_WAIT, s) = (double)(3 + rs->integers(0, 17));        // randint(3, 20)
    } else {
      vel *= -1;
      d.f(DTS_DYN_WAIT, s) = 8.0;
    }
    d.f(DTS_DYN_VEL, s) = vel;
  }
  d.f(DTS_DYN_YROT, s) = (angle + p.wiggle * sin(48 * time)) * (180 / 3.141592653589793);
}

// DuckiebotObj.step_duckiebot O:229-263 + _update_pos O:281-336
__device__ inline void duckiebot_step(const DMap& m, const DynRef& d, int s, double dt) {
  const DDyn& p = d.par[s];
  const double px = d.f(DTS_DYN_PX, s), pz = d.f(DTS_DYN_PZ, s), angle = d.f(DTS_DYN_ANGLE, s);
  double cp[3], ct[3], cur[3], tmp[3];
  if (!closest_curve_point(m, px, pz, angle, cp, ct)) return;         // the reference raises; here the bot stops
  double lookup = p.follow_dist;
  bool found = false;
  for (int it = 0; it < 1000 && !found; it++) {
    found = closest_curve_point(m, cp[0] + ct[0] * lookup, cp[2] + ct[2] * lookup, angle, cur, tmp);
    if (!found) lookup *= 0.5;
  }
  if (!found) return;
  double vx = cur[0] - px, vy = cur[1] - p.pos_y, vz = cur[2] - pz;
  const double nn = sqrt(vx * vx + vy * vy + vz * vz);
  vx /= nn; vy /= nn; vz /= nn;
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double steer = p.gain * -(sn * vx + 0 * vy + cs * vz);
  const double k_r_inv = (p.gain + p.trim) / p.k, k_l_inv = (p.gain - p.trim) / p.k;
  const double omega_r = (p.velocity + 0.5 * steer * p.wheel_dist) / p.radius;
  const double omega_l = (p.velocity - 0.5 * steer * p.wheel_dist) / p.radius;
  const double ur = fmax(fmin(omega_r * k_r_inv, p.limit), -p.limit), ul = fmax(fmin(omega_l * k_l_inv, p.limit), -p.limit);
  if (ul == ur) {                                                      // O:305-307: box and y_rot not refreshed
    d.f(DTS_DYN_PX, s) = px + dt * ul * cs;
    d.f(DTS_DYN_PZ, s) = pz + dt * ul * -sn;
    return;
  }
  const double w = (ur - ul) / p.wheel_dist;
  const double r = (p.wheel_dist * (ul + ur)) / (2 * (ul - ur));
  const double rot = w * dt;
  const double icx = px + r * sn, icz = pz + r * cs;
  double srot, crot;
  sincos(rot, &srot, &crot);
  const double ddx = px - icx, ddy = pz - icz;                          // rotate_point G:254-265
  const double ndx = ddx * crot + ddy * srot, ndy = ddy * crot - ddx * srot;
  const double nx = icx + ndx, nz = icz + ndy, na = angle + rot;
  d.f(DTS_DYN_PX, s) = nx; d.f(DTS_DYN_PZ, s) = nz; d.f(DTS_DYN_ANGLE, s) = na;
  d.f(DTS_DYN_YROT, s) += rot * 180 / 3.141592653589793;
  sincos(na, &sn, &cs);
  const double fx = cs, fz = -sn, sx = sn, sz = cs, hw = 0.5 * p.robot_width, hl = 0.5 * p.robot_length;
  d.f(DTS_DYN_CORNERS + 0, s) = nx - hw * sx - hl * fx; d.f(DTS_DYN_CORNERS + 1, s) = nz - hw * sz - hl * fz;
  d.f(DTS_DYN_CORNERS + 2, s) = nx + hw * sx - hl * fx; d.f(DTS_DYN_CORNERS + 3, s) = nz + hw * sz - hl * fz;
  d.f(DTS_DYN_CORNERS + 4, s) = nx + hw * sx + hl * fx; d.f(DTS_DYN_CORNERS + 5, s) = nz + hw * sz + hl * fz;
  d.f(DTS_DYN_CORNERS + 6, s) = nx - hw * sx + hl * fx; d.f(DTS_DYN_CORNERS + 7, s) = nz - hw * sz + hl * fz;
}

// TrafficLightObj.step O:455-462: `round(time, 3) % freq == 0` flips the pattern and re-assigns the SHARED mesh's card
__device__ inline void trafficlight_step(const DynRef& d, int s, double dt) {
  const DDyn& p = d.par[s];
  const double time = d.f(DTS_DYN_TIME, s) + dt;
  d.f(DTS_DYN_TIME, s) = time;
  const long long ms = llrint(time * 1000.0), per = llrint(p.freq * 1000.0);
  if (per > 0 && ms % per == 0) {
    const double pat = d.f(DTS_DYN_PATTERN, s) == 0.0 ? 1.0 : 0.0;
    d.f(DTS_DYN_PATTERN, s) = pat;
    d.f(DTS_DYN_SHOWN, p.tl_first) = pat;
  }
}

// the object loop of update_physics S:1570-1584
__device__ inline void dyn_step_all(const DMap& m, const DynRef& d, double dt, NpStream* rs) {
  for (int s = 0; s < d.n_dyn; s++) {
    const int kind = d.par[s].kind;
    if (kind == DTS_DYN_DUCKIEBOT) duckiebot_step(m, d, s, dt);
    else if (kind == DTS_DYN_TRAFFICLIGHT) trafficlight_step(d, s, dt);
    else duckie_step(d, s, dt, rs);
  }
}

// check_collision O:265-269 / O:368-372 -> intersects_single_obj C:162-186, agent box centred at (bx,bz)
__device__ inline bool agent_hits_dynamic(const DynRef& d, double bx, double bz, double angle) {
  if (d.n_dyn == 0) return false;
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double fx = cs, fz = -sn, rx = sn, rz = cs, hw = 0.5 * kRobotWidth, hl = 0.5 * kRobotLength;
  double ax[4], az[4];
  ax[0] = bx - hw * rx - hl * fx; az[0] = bz - hw * rz - hl * fz;
  ax[1] = bx + hw * rx - hl * fx; az[1] = bz + hw * rz - hl * fz;
  ax[2] = bx + hw * rx + hl * fx; az[2] = bz + hw * rz + hl * fz;
  ax[3] = bx - hw * rx + hl * fx; az[3] = bz - hw * rz + hl * fz;
  double aR0, aR1, aF0, aF1;
  project4(rx, rz, ax, az, aR0, aR1);
  project4(fx, fz, ax, az, aF0, aF1);
  for (int s = 0; s < d.n_dyn; s++) {
    if (d.par[s].kind == DTS_DYN_TRAFFICLIGHT) continue;   // a static WorldObj: check_collision is False (O:150-158)
    double ox[4], oz[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { ox[k] = d.f(DTS_DYN_CORNERS + 2 * k, s); oz[k] = d.f(DTS_DYN_CORNERS + 2 * k + 1, s); }
    const double* on = d.par[s].norms;
    double lo, hi, lo2, hi2;
    project4(rx, rz, ox, oz, lo, hi);
    if (!intervals_touch(aR0, aR1, lo, hi)) continue;
    project4(fx, fz, ox, oz, lo, hi);
    if (!intervals_touch(aF0, aF1, lo, hi)) continue;
    project4(on[0], on[1], ax, az, lo, hi);
    project4(on[0], on[1], ox, oz, lo2, hi2);
    if (!intervals_touch(lo, hi, lo2, hi2)) continue;
    project4(on[2], on[3], ax, az, lo, hi);
    project4(on[2], on[3], ox, oz, lo2, hi2);
    if (!intervals_touch(lo, hi, lo2, hi2)) continue;
    return true;
  }
  return false;
}

// obj.proximity O:271-279 / O:374-383 summed as in S:1455-1457
__device__ inline double dynamic_proximity(const DynRef& d, double px, double pz, double angle) {
  if (d.n_dyn == 0) return 0.0;
  double sn, cs;
  sincos(angle, &sn, &cs);
  const double qx = px + kCentreOff * cs, qz = pz + kCentreOff * -sn;
  double acc = 0.0;
  for (int s = 0; s < d.n_dyn; s++) {
    if (d.par[s].kind == DTS_DYN_TRAFFICLIGHT) continue;   // static WorldObj.proximity is 0 (O:160-168)
    const double dx = qx - d.f(DTS_DYN_PX, s), dy = 0 - d.par[s].pos_y, dz = qz - d.f(DTS_DYN_PZ, s);
    const double sc = sqrt(dx * dx + dy * dy + dz * dz) - kAgentSafetyRad - d.par[s].safety_radius;
    acc += sc < 0 ? sc : 0.0;
  }
  return acc;
}

// _inconvenient_spawn S:1461-1471 over the visible objects, dynamic ones where they currently are
__device__ inline bool inconvenient_spawn(const DMap& m, const DynRef& d, const uint32_t* hidden, double x, double z) {
  for (int o = 0; o < m.n_objects; o++) {
    if (hidden && (hidden[o >> 5] >> (o & 31) & 1u)) continue;
    const DObject& ob = m.objects[o];
    double ox = ob.dpos[0], oz = ob.dpos[2];
    if (ob.dyn_slot >= 0 && d.n_dyn > 0) { ox = d.f(DTS_DYN_PX, ob.dyn_slot); oz = d.f(DTS_DYN_PZ, ob.dyn_slot); }
    const double dx = ox - x, dy = ob.dpos[1], dz = oz - z;
    if (sqrt(dx * dx + dy * dy + dz * dz) < (double)ob.spawn_rad) return true;
  }
  return false;
}

// One integration step of the restated duckietown_world model (DESIGN.md "dynamics"; call site S:2083-2086).
__device__ __forceinline__ void dynamics_step(double& x, double& y, double& th, double& u, double& w, double l,
                                              double r, const DynParams& p, double trim, double dt) {
  l = clampd(l, -1.0, 1.0);
  r = clampd(r, -1.0, 1.0);
  const double uar = p.uar * (1.0 + trim), ual = p.ual * (1.0 - trim);
  const double war = p.war * (1.0 + trim), wal = p.wal * (1.0 - trim);
  const double du = -p.u1 * u - p.u2 * w + p.u3 * w * w + (uar * r + ual * l);
  const double dw = -p.w1 * w - p.w2 * u - p.w3 * u * w + (war * r - wal * l);
  const double u1 = u + dt * du, w1 = w + dt * dw;
  const double a = dt * w1, vx = dt * u1;
  double sa, ca;  // sin(a)/a, (1-cos a)/a, the latter as 2 sin^2(a/2)/a: 1 - cos(a) cancels to nothing below |a| ~ 1e-7
  if (fabs(a) < 1e-9) { sa = 1.0 - a * a / 6.0; ca = a / 2.0; }
  else { double sh, ch; sincos(0.5 * a, &sh, &ch); sa = 2.0 * sh * ch / a; ca = 2.0 * sh * sh / a; }
  const double tx = sa * vx, ty = ca * vx;
  double sn, cs;
  sincos(th, &sn, &cs);
  x += cs * tx - sn * ty;
  y += sn * tx + cs * ty;
  th += a;
  u = u1;
  w = w1;
}

}  // namespace dts
