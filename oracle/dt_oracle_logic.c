/* dt_oracle_logic.c — CPU ORACLE (test infrastructure, NOT product code).
 *
 * Plain-C float64 restatement of the non-rendering half of gym-duckietown's Simulator.step():
 * action map, delayed PWM dynamics, tile lookup, valid-pose, OBB SAT collision, safety circles,
 * lane pose, reward/done.  Each function cites the reference lines it follows (paths relative to
 * /root/reference/src/gym_duckietown).  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this; the product (libdtsim.so) never does.
 *
 * Pinning: everything except orc_dyn_step is checked against the reference's own code executed
 * through oracle/refstub.py (tests/golden/logic_*.npz, tests/test_oracle_vs_reference.py).
 * orc_dyn_step restates duckietown_world (absent, un-pinned dependency): PARITY UNPINNED.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "dt_oracle.h"


/* robot constants simulator.py:118-177 */
static const double ROBOT_WIDTH = 0.13 + 0.02;
static const double ROBOT_LENGTH = 0.18;
static const double CAMERA_FORWARD_DIST = 0.066;
#define AGENT_SAFETY_RAD ((fmax(ROBOT_LENGTH, ROBOT_WIDTH) / 2) * 1.8)

/* envs/duckietown_env.py:36-59 — [vel, steering] -> clamped wheel duty (left, right) */
void orc_action_map(double vel, double steer, double wheel_dist, double gain, double trim, double radius,
                    double k, double limit, double out_lr[2]) {
  double k_r_inv = (gain + trim) / k;
  double k_l_inv = (gain - trim) / k;
  double omega_r = (vel + 0.5 * steer * wheel_dist) / radius;
  double omega_l = (vel - 0.5 * steer * wheel_dist) / radius;
  double u_r = omega_r * k_r_inv;
  double u_l = omega_l * k_l_inv;
  out_lr[1] = fmax(fmin(u_r, limit), -limit);
  out_lr[0] = fmax(fmin(u_l, limit), -limit);
}

/* duckietown_world pwm_dynamics + delay + SE(2) exponential (restated, call sites S:2083-2086).
 * `cmd` is the command issued NOW (already clipped to [-1,1] by Simulator.step S:1670). */
void orc_dyn_step(orc_dyn_state* s, const orc_dyn_params* p, const double cmd_lr[2], double dt) {
  double l, r;
  int d = p->delay_steps;
  if (d > 0) {
    l = s->fifo[0][0];
    r = s->fifo[0][1];
    for (int i = 0; i + 1 < d; i++) { s->fifo[i][0] = s->fifo[i + 1][0]; s->fifo[i][1] = s->fifo[i + 1][1]; }
    s->fifo[d - 1][0] = cmd_lr[0];
    s->fifo[d - 1][1] = cmd_lr[1];
  } else { l = cmd_lr[0]; r = cmd_lr[1]; }
  /* the dynamic model clips the duty cycle again */
  l = fmax(-1.0, fmin(1.0, l));
  r = fmax(-1.0, fmin(1.0, r));
  double u = s->u, w = s->w;
  double du = -p->u1 * u - p->u2 * w + p->u3 * w * w + (p->uar * r + p->ual * l);
  double dw = -p->w1 * w - p->w2 * u - p->w3 * u * w + (p->war * r - p->wal * l);
  double u1 = u + dt * du;
  double w1 = w + dt * dw;
  /* q' = q * expm(dt * [[0,-w,u],[w,0,0],[0,0,0]]) : closed form of the SE(2) exponential */
  double a = dt * w1, vx = dt * u1;
  double sa, ca;
  /* sin(a)/a , (1-cos a)/a, the latter as 2 sin^2(a/2)/a: 1 - cos(a) cancels to nothing below |a| ~ 1e-7 */
  if (fabs(a) < 1e-9) { sa = 1.0 - a * a / 6.0; ca = a / 2.0; }
  else { double sh = sin(0.5 * a), ch = cos(0.5 * a); sa = 2.0 * sh * ch / a; ca = 2.0 * sh * sh / a; }
  double tx = sa * vx, ty = ca * vx; /* body-frame translation (lateral velocity is 0) */
  double c = cos(s->theta), sn = sin(s->theta);
  s->x += c * tx - sn * ty;
  s->y += sn * tx + c * ty;
  s->theta += a;
  s->u = u1;
  s->w = w1;
}

/* weird_from_cartesian S:1640-1652: pos = [x, 0, H*ts - y], angle = atan2(sin, cos) in (-pi, pi] */
void orc_weird_from_cartesian(const orc_map* m, const orc_dyn_state* s, double* px, double* pz, double* ang) {
  *px = s->x;
  *pz = m->grid_h * m->tile_size - s->y;
  *ang = atan2(sin(s->theta), cos(s->theta));
}
/* cartesian_from_weird S:1629-1638 */
void orc_cartesian_from_weird(const orc_map* m, double px, double pz, double ang, orc_dyn_state* s) {
  s->x = px;
  s->y = m->grid_h * m->tile_size - pz;
  s->theta = ang;
}

/* get_grid_coords S:1134-1149 + _get_tile S:1053-1063 + _drivable_pos S:1411-1428 */
static int tile_index(const orc_map* m, double x, double z, int* oi, int* oj) {
  int i = (int)floor(x / m->tile_size);
  int j = (int)floor(z / m->tile_size);
  if (oi) *oi = i;
  if (oj) *oj = j;
  if (i < 0 || i >= m->grid_w || j < 0 || j >= m->grid_h) return -1;
  int idx = j * m->grid_w + i;
  if (m->tile_kind[idx] < 0) return -1;
  return idx;
}
int orc_drivable_pos(const orc_map* m, double x, double z) {
  int idx = tile_index(m, x, z, 0, 0);
  return idx >= 0 && m->tile_drivable[idx];
}

static void minmax4(const double ax[2], const double* cx, const double* cz, double* lo, double* hi) {
  double mn = INFINITY, mx = -INFINITY;
  for (int k = 0; k < 4; k++) {
    double v = ax[0] * cx[k] + ax[1] * cz[k];
    if (v < mn) mn = v;
    if (v > mx) mx = v;
  }
  *lo = mn; *hi = mx;
}
/* collision.overlaps / is_between_ordered C:50-61 (closed intervals) */
static int overlaps(double min1, double max1, double min2, double max2) {
  return (min1 <= min2 && min2 <= max1) || (min2 <= min1 && min1 <= max2);
}

/* agent_boundbox C:9-34 via get_agent_corners S:2112-2116; corner order as in the reference */
void orc_agent_corners(double px, double pz, double angle, double cx[4], double cz[4]) {
  double fx = cos(angle), fz = -sin(angle);       /* get_dir_vec S:2056 */
  double rx = sin(angle), rz = cos(angle);        /* get_right_vec S:2066 */
  double off = CAMERA_FORWARD_DIST - (ROBOT_LENGTH / 2);  /* _actual_center S:2102-2109 */
  double tx = px + off * fx, tz = pz + off * fz;
  double hw = 0.5 * ROBOT_WIDTH, hl = 0.5 * ROBOT_LENGTH;
  cx[0] = tx - hw * rx - hl * fx; cz[0] = tz - hw * rz - hl * fz;
  cx[1] = tx + hw * rx - hl * fx; cz[1] = tz + hw * rz - hl * fz;
  cx[2] = tx + hw * rx + hl * fx; cz[2] = tz + hw * rz + hl * fz;
  cx[3] = tx - hw * rx + hl * fx; cz[3] = tz - hw * rz + hl * fz;
}

/* _collision S:1473-1492 + intersects C:129-159.  The agent's SAT axes: generate_norm (C:99-106)
 * takes eigenvectors of the corner covariance; for the non-square 0.15 x 0.18 footprint those are
 * the box axes (up to sign/order, which the symmetric interval test ignores), so the oracle uses
 * the right / forward unit vectors directly. Pinned against the LAPACK path by the golden vectors. */
int orc_collision(const orc_map* m, double px, double pz, double angle) {
  if (m->n_coll == 0) return 0;
  double cx[4], cz[4];
  orc_agent_corners(px, pz, angle, cx, cz);
  double an[2][2] = {{sin(angle), cos(angle)}, {cos(angle), -sin(angle)}};
  double dd_lo[2], dd_hi[2];
  for (int a = 0; a < 2; a++) minmax4(an[a], cx, cz, &dd_lo[a], &dd_hi[a]);
  for (int k = 0; k < m->n_coll; k++) {
    const double* ox = m->coll_corners + (size_t)k * 8;
    const double* oz = ox + 4;
    const double* on = m->coll_norms + (size_t)k * 4;
    double lo, hi, lo2, hi2;
    int hit = 1;
    for (int a = 0; a < 2 && hit; a++) {
      minmax4(an[a], ox, oz, &lo, &hi);
      if (!overlaps(dd_lo[a], dd_hi[a], lo, hi)) hit = 0;
    }
    for (int a = 0; a < 2 && hit; a++) {
      minmax4(on + 2 * a, cx, cz, &lo, &hi);
      minmax4(on + 2 * a, ox, oz, &lo2, &hi2);
      if (!overlaps(lo, hi, lo2, hi2)) hit = 0;
    }
    if (hit) return 1;
  }
  return 0;
}

/* _valid_pose S:1494-1534 */
int orc_valid_pose(const orc_map* m, double px, double pz, double angle, double safety_factor, uint8_t* collided,
                   uint8_t* all_drivable) {
  double fx = cos(angle), fz = -sin(angle);
  double rx = sin(angle), rz = cos(angle);
  double off = CAMERA_FORWARD_DIST - (ROBOT_LENGTH / 2);
  double cxp = px + off * fx, czp = pz + off * fz;
  double sw = safety_factor * 0.5 * ROBOT_WIDTH, sl = safety_factor * 0.5 * ROBOT_LENGTH;
  int drv = orc_drivable_pos(m, cxp, czp) && orc_drivable_pos(m, cxp - sw * rx, czp - sw * rz) &&
            orc_drivable_pos(m, cxp + sw * rx, czp + sw * rz) && orc_drivable_pos(m, cxp + sl * fx, czp + sl * fz);
  /* get_agent_corners(pos, angle) is called with the ALREADY shifted centre (S:1502,1521): the
   * offset is applied twice for the collision box. */
  int col = orc_collision(m, cxp, czp, angle);
  if (collided) *collided = (uint8_t)col;
  if (all_drivable) *all_drivable = (uint8_t)drv;
  return !col && drv;
}

/* proximity_penalty2 S:1430-1459, safety_circle_intersection/overlap C:189-211 */
double orc_proximity(const orc_map* m, double px, double pz, double angle) {
  if (m->n_coll == 0) return 0.0;
  double off = CAMERA_FORWARD_DIST - (ROBOT_LENGTH / 2);
  double cx = px + off * cos(angle), cz = pz + off * -sin(angle);
  int any = 0;
  double sum = 0.0;
  for (int k = 0; k < m->n_coll; k++) {
    const double* c = m->coll_centers + 3 * (size_t)k;
    double dx = c[0] - cx, dy = c[1] - 0.0, dz = c[2] - cz;
    double d = sqrt(dx * dx + dy * dy + dz * dz);
    double r1 = AGENT_SAFETY_RAD, r2 = m->coll_radii[k];
    int inter = ((r1 - r2) * (r1 - r2) <= d * d) && (d * d <= (r1 + r2) * (r1 + r2));
    int env = d < fabs(r1 - r2);
    if (inter || env) any = 1;
    double sc = d - r1 - r2;
    if (sc < 0) sum += sc;
  }
  return any ? sum : 0.0;
}

static void bez_point(const double* cp, double t, double out[3]) {  /* G:286-297 */
  double a = (1 - t) * (1 - t) * (1 - t), b = 3 * t * ((1 - t) * (1 - t)), c = 3 * (t * t) * (1 - t), d = t * t * t;
  for (int k = 0; k < 3; k++) {
    double p = a * cp[k];
    p += b * cp[3 + k];
    p += c * cp[6 + k];
    p += d * cp[9 + k];
    out[k] = p;
  }
}

/* closest_curve_point S:1337-1369: point on the best-aligned lane curve of the tile under (px,pz) and the
 * unit tangent there.  Returns 0 when there is no drivable tile. */
int orc_closest_curve_point(const orc_map* m, double px, double pz, double angle, double pnt[3], double tan3[3]) {
  int idx = tile_index(m, px, pz, 0, 0);
  if (idx < 0 || !m->tile_drivable[idx]) return 0;
  const double* cv = m->curves + (size_t)m->tile_curve_off[idx] * 12;
  int nc = m->tile_curve_cnt[idx];
  double dirx = cos(angle), dirz = -sin(angle);
  /* argmax of (P3-P0).dir ; the common Frobenius normalisation (S:1356) does not change the order */
  double fro = 0.0;
  for (int c = 0; c < nc; c++)
    for (int k = 0; k < 3; k++) { double h = cv[c * 12 + 9 + k] - cv[c * 12 + k]; fro += h * h; }
  fro = sqrt(fro);
  int best = 0; double bestv = -INFINITY;
  for (int c = 0; c < nc; c++) {
    double hx = (cv[c * 12 + 9] - cv[c * 12 + 0]) / fro, hz = (cv[c * 12 + 11] - cv[c * 12 + 2]) / fro;
    double v = hx * dirx + hz * dirz;
    if (v > bestv) { bestv = v; best = c; }
  }
  const double* cp = cv + best * 12;
  /* bezier_closest G:316-333: 8 bisection levels on endpoint distance */
  double tb = 0.0, tt = 1.0;
  for (int n = 8; n > 0; n--) {
    double mid = (tb + tt) * 0.5, pb[3], pt[3];
    bez_point(cp, tb, pb);
    bez_point(cp, tt, pt);
    double db = sqrt((pb[0] - px) * (pb[0] - px) + pb[1] * pb[1] + (pb[2] - pz) * (pb[2] - pz));
    double dtp = sqrt((pt[0] - px) * (pt[0] - px) + pt[1] * pt[1] + (pt[2] - pz) * (pt[2] - pz));
    if (db < dtp) tt = mid; else tb = mid;
  }
  double t = (tb + tt) * 0.5;
  bez_point(cp, t, pnt);
  /* bezier_tangent G:300-313 */
  for (int k = 0; k < 3; k++) {
    double p = 3 * ((1 - t) * (1 - t)) * (cp[3 + k] - cp[k]);
    p += 6 * (1 - t) * t * (cp[6 + k] - cp[3 + k]);
    p += 3 * (t * t) * (cp[9 + k] - cp[6 + k]);
    tan3[k] = p;
  }
  double nrm = sqrt(tan3[0] * tan3[0] + tan3[1] * tan3[1] + tan3[2] * tan3[2]);
  for (int k = 0; k < 3; k++) tan3[k] /= nrm;
  return 1;
}

/* get_lane_pos2 S:1371-1409. Returns 0 if not in a lane. */
int orc_lane_pos(const orc_map* m, double px, double pz, double angle, double* dist, double* dot_dir,
                 double* angle_rad) {
  double pnt[3], tan3[3];
  if (!orc_closest_curve_point(m, px, pz, angle, pnt, tan3)) return 0;
  double dirx = cos(angle), dirz = -sin(angle);
  double dd = dirx * tan3[0] + dirz * tan3[2];
  if (dd > 1.0) dd = 1.0;
  if (dd < -1.0) dd = -1.0;
  double rvx = -tan3[2], rvz = tan3[0];  /* cross(tangent, up) with tangent.y == 0 */
  *dist = (px - pnt[0]) * rvx + (pz - pnt[2]) * rvz;
  double ar = acos(dd);
  if (dirx * rvx + dirz * rvz < 0) ar = -ar;
  *dot_dir = dd;
  *angle_rad = ar;
  return 1;
}

/* _compute_done_reward S:1685-1705 + compute_reward S:1654-1667 */
void orc_done_reward(const orc_map* m, double px, double pz, double angle, int step_count, int max_steps,
                     double robot_speed, orc_step_out* o) {
  o->pos_x = px; o->pos_z = pz; o->angle = angle; o->step_count = step_count;
  tile_index(m, px, pz, &o->tile_i, &o->tile_j);
  o->lane_dist = o->lane_dot = o->lane_angle = NAN;
  o->in_lane = (uint8_t)orc_lane_pos(m, px, pz, angle, &o->lane_dist, &o->lane_dot, &o->lane_angle);
  o->prox = orc_proximity(m, px, pz, angle);
  int valid = orc_valid_pose(m, px, pz, angle, 1.0, &o->collided, &o->drivable4);
  if (!valid) { o->done = 1; o->done_code = 1; o->reward = -1000.0; }
  else if (step_count >= max_steps) { o->done = 1; o->done_code = 2; o->reward = 0.0; }
  else {
    o->done = 0; o->done_code = 0;
    if (o->in_lane) o->reward = +1.0 * robot_speed * o->lane_dot + -10 * fabs(o->lane_dist) + +40 * o->prox;
    else o->reward = 40 * o->prox;
  }
}

/* Simulator.step S:1669-1683 (frame_skip physics updates, then done/reward) for ONE env.
 * `action` is what the caller hands to env.step: wheel duty if action_mode==0, [vel, steer] if 1. */
void orc_step(const orc_map* m, const orc_dyn_params* dp, orc_dyn_state* s, int* step_count, double* last_px,
              double* last_pz, const double action[2], int action_mode, double wheel_dist, const double env5[5],
              int frame_skip, double dt, int max_steps, double robot_speed, orc_step_out* o) {
  double cmd[2] = {action[0], action[1]};
  if (action_mode == 1) orc_action_map(action[0], action[1], wheel_dist, env5[0], env5[1], env5[2], env5[3], env5[4], cmd);
  cmd[0] = fmax(-1.0, fmin(1.0, cmd[0]));  /* np.clip S:1670 */
  cmd[1] = fmax(-1.0, fmin(1.0, cmd[1]));
  double px = *last_px, pz = *last_pz, ang = 0, speed = 0;
  for (int f = 0; f < frame_skip; f++) {  /* update_physics S:1551-1568 */
    double ppx = px, ppz = pz;
    orc_dyn_step(s, dp, cmd, dt);
    orc_weird_from_cartesian(m, s, &px, &pz, &ang);
    (*step_count)++;
    speed = sqrt((px - ppx) * (px - ppx) + (pz - ppz) * (pz - ppz)) / dt;
  }
  *last_px = px; *last_pz = pz;
  orc_done_reward(m, px, pz, ang, *step_count, max_steps, robot_speed, o);
  o->speed = speed;
}
