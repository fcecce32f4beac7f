/* dt_oracle.h — types and prototypes of the CPU oracle (TEST INFRASTRUCTURE, see the .c headers). */
#ifndef DT_ORACLE_H
#define DT_ORACLE_H
#include <stdint.h>

#define ORC_MAX_DELAY 16 /* = DTS_MAX_DELAY (include/dtsim.h); tests/test_dynamics_ref.py holds the two equal */

typedef struct {
  double tile_size;
  int32_t grid_w, grid_h;
  const int8_t* tile_kind;
  const uint8_t* tile_drivable;
  const int32_t* tile_curve_off;
  const int32_t* tile_curve_cnt;
  const double* curves; /* [nc][4][3] */
  int32_t n_coll;
  const double* coll_corners; /* [K][2][4] */
  const double* coll_norms;   /* [K][2][2] */
  const double* coll_centers; /* [K][3] */
  const double* coll_radii;   /* [K] */
} orc_map;

typedef struct {
  double u1, u2, u3, w1, w2, w3, uar, ual, war, wal;
  int32_t delay_steps; /* commands issued at step k act from step k+delay_steps on */
} orc_dyn_params;

typedef struct {
  double x, y, theta; /* cartesian pose q (duckietown_world frame) */
  double u, w;        /* longitudinal / angular velocity */
  double fifo[ORC_MAX_DELAY][2]; /* pending (left,right) commands, [0] = oldest */
} orc_dyn_state;

typedef struct {
  double pos_x, pos_z, angle, speed;
  double reward;
  double lane_dist, lane_dot, lane_angle;
  double prox;
  int32_t tile_i, tile_j, step_count;
  uint8_t done, done_code, in_lane, collided, drivable4;
} orc_step_out;

typedef struct { int32_t w, h; const uint8_t* rgba; } orr_texture;
typedef struct {
  float pos[3]; float scale; float y_rot_deg; int32_t tri_offset, tri_count;
  int32_t tex_from, tex_to; /* triangles textured tex_from draw tex_to instead (traffic-light card); -1 = off */
  int32_t seg_tex;          /* segment=True: every triangle shows this flat class-colour texture (objmesh.py:260-290) */
} orr_object;

typedef struct {
  double tile_size;
  int32_t grid_w, grid_h;
  const int8_t* tile_kind;
  const int8_t* tile_angle;
  const int16_t* tile_tex;
  int32_t n_objects;
  const orr_object* objects;
  const float* tri_pos; /* [T][3][3] */
  const float* tri_nrm;
  const float* tri_uv;  /* [T][3][2] */
  const float* tri_col;
  const int16_t* tri_tex;
  int32_t n_textures;
  const orr_texture* textures;
  const int16_t* tex_segment; /* [n_textures] Texture.bind(segment=True) replacement (graphics.py:52-56) */
  orr_object agent;           /* top-down views: the agent's own mesh (tri_count 0 = none), S:1923-1929 */
} orr_scene;

typedef struct { /* mirrors the product's per-episode render record */
  float cam_height, cam_angle_deg, cam_fov_y_deg;
  float cam_noise[3], horizon[3], ambient[3], diffuse[3], light_eye[4], ground[3];
  uint32_t hidden[8];
} orr_episode;

typedef struct {   /* one dynamic obstacle (objects.py DuckieObj / DuckiebotObj) */
  int32_t kind;      /* 1 duckie pedestrian, 2 duckiebot follower, 3 traffic light */
  int32_t active;    /* DuckieObj.pedestrian_active */
  double pos[3], angle, y_rot;
  double corners[4][2];
  double norm[4];    /* obj_norm rows */
  double safety_radius;
  double walk_distance, vel, wait_time, wiggle, time, start[3], heading[3];
  double follow_dist, velocity, gain, trim, radius, k, limit, wheel_dist, robot_width, robot_length;
  double freq;       /* kind 3 (TrafficLightObj): `active` is its pattern */
  int32_t tl_first;  /* index of the first traffic light: its `shown` is the card of the mesh they all share */
  int32_t shown;
} orc_dyn;

int orc_closest_curve_point(const orc_map* m, double px, double pz, double angle, double pnt[3], double tan3[3]);
void orc_agent_corners(double px, double pz, double angle, double cx[4], double cz[4]);
void orc_dyn_step_all(const orc_map* m, orc_dyn* objs, int n, double dt);
int orc_dyn_collision(const orc_dyn* objs, int n, double px, double pz, double angle);
double orc_dyn_proximity(const orc_dyn* objs, int n, double px, double pz, double angle);
int orc_valid_pose_dyn(const orc_map* m, const orc_dyn* objs, int n, double px, double pz, double angle,
                       double safety_factor, uint8_t* collided);
void orc_step_dynamic(const orc_map* m, const orc_dyn_params* dp, orc_dyn_state* s, int* step_count, double* last_px,
                      double* last_pz, const double action[2], int action_mode, double wheel_dist,
                      const double env5[5], int frame_skip, double dt, int max_steps, double robot_speed,
                      orc_dyn* objs, int n, orc_step_out* o);
void orc_action_map(double vel, double steer, double wheel_dist, double gain, double trim, double radius, double k,
                    double limit, double out_lr[2]);
void orc_dyn_step(orc_dyn_state* s, const orc_dyn_params* p, const double cmd_lr[2], double dt);
void orc_weird_from_cartesian(const orc_map* m, const orc_dyn_state* s, double* px, double* pz, double* ang);
void orc_cartesian_from_weird(const orc_map* m, double px, double pz, double ang, orc_dyn_state* s);
int orc_valid_pose(const orc_map* m, double px, double pz, double angle, double safety_factor, uint8_t* collided,
                   uint8_t* all_drivable);
void orc_done_reward(const orc_map* m, double px, double pz, double angle, int step_count, int max_steps,
                     double robot_speed, orc_step_out* o);
void orc_step(const orc_map* m, const orc_dyn_params* dp, orc_dyn_state* s, int* step_count, double* last_px,
              double* last_pz, const double action[2], int action_mode, double wheel_dist, const double env5[5],
              int frame_skip, double dt, int max_steps, double robot_speed, orc_step_out* o);
void orr_render(const orr_scene* sc, double px, double pz, double angle, const orr_episode* ep, int W, int H,
                int domain_rand, const float* lut_x, const float* lut_y, uint8_t* out);
void orr_set_render_mode(int mode); /* 1 = segment=True, 2 = top_down=True (simulator.py:1707-1951) */
void orr_debug_frame(const orr_scene* sc, double px, double pz, double angle, const orr_episode* ep, int W, int H,
                     int domain_rand, double* V_out, float* P_out, float* item_mv, float* item_n, float* lattice);
/* test-side statistics of the triangles handed to the rasteriser since the last reset (single-threaded use):
 * [0] set-up triangles on screen, [1] no sample position in their box, [2] no covered sample, [3] box <= 2x2 px, [4] <= 4x4 px, [5] quads */
void orr_stats_read(long long out[8], int reset);
#endif
