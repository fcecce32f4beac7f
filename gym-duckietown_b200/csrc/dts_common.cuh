// dts_common.cuh — device-side data layout shared by the dtsim kernels (sm_90a only).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/dtsim.h"

namespace dts {

// ------------------------------------------------------------------ map data resident in HBM
// One DMap per uploaded map; all pointers are device memory owned by the handle.  Read-only on
// the hot path and shared by every env, so it lives in L2 after the first touch.
struct DObject {
  float pos[3];
  float scale;
  float y_rot_deg;
  int32_t mesh_id;
  int32_t optional;
  float spawn_rad;   // max(max_coords)*0.5*scale + MIN_SPAWN_OBJ_DIST   (simulator.py:1467)
  int32_t tri_offset, tri_count;
  float bound_rad;   // object-space bounding radius (culling)
  float centre[3];   // object-space bounding-sphere centre
  int32_t dyn_slot;  // -1 static; else slot of the per-env dynamic state that supplies pos / y_rot / card
  int32_t alt_from, alt_to;   // traffic-light card swap (texture ids), -1 none
  int32_t seg_tex;            // flat class-colour texture of the mesh under segment=True (-1 none)
  int32_t tri_base;           // triangles of the map's objects before this one (the agent: of all of them), so that its
                              // draw ids start at 2 + the tiles' ids + tri_base (label images, render spec item 10)
  double dpos[3];    // float64 position (x.pos in _inconvenient_spawn S:1466)
};

// A dynamic obstacle's constants (dts_dyn_object); its evolving state lives in DMap::dyn_state.
struct DDyn {
  int32_t kind, object_index;
  double pos_y;
  double norms[4];
  double safety_radius;
  double walk_distance, wiggle, angle0;   // duckie: heading = heading_vec(angle at load) never changes (O:357)
  double follow_dist, velocity, gain, trim, radius, k, limit, wheel_dist, robot_width, robot_length;
  double freq;        // traffic light
  int32_t tl_first;   // slot of the map's first traffic light (holds the shared card), -1 if none
  int32_t pad;
};

// Textures of a map live in ONE pool allocation; `info` is what a prim carries to find its texels without a dependent
// table lookup: (byte offset in the pool >> 8) | log2(w) << 24 | log2(h) << 28.
struct DTexture { const uint8_t* rgba; int32_t w, h; uint32_t info, pad; };

struct DMap {
  double tile_size;
  int32_t grid_w, grid_h;
  int32_t n_tiles;              // grid_w * grid_h
  const int8_t* tile_kind;
  const int8_t* tile_angle;
  const uint8_t* tile_drivable;
  const int16_t* tile_tex;
  const int32_t* tile_curve_off;
  const int32_t* tile_curve_cnt;
  const double* curves;         // [n][4][3]
  int32_t n_coll;
  const double* coll_corners;   // [K][2][4]
  const double* coll_norms;     // [K][2][2]
  const double* coll_centers;   // [K][3]
  const double* coll_radii;     // [K]
  int32_t start_i, start_j;     // user_tile_start / map `start_tile` (S:659-671) or -1
  int32_t has_start_pose;       // map `start_pose` S:679-686
  double start_pose[3];         // x, z offset inside the start tile, angle
  int32_t n_drivable;
  const int32_t* drivable_ij;   // [n_drivable][2] in reference scan order (S:806-860)
  int32_t n_objects;
  const DObject* objects;
  int32_t n_tris;
  const float* tri_pos;         // [T][3][3]
  const float* tri_nrm;
  const float* tri_uv;          // [T][3][2]
  const float* tri_col;         // [T][3][3]
  const int16_t* tri_tex;
  int32_t n_textures;
  uint32_t tex_class_off;       // the texel classes (dts_map_blob.tex_class) start at tex_pool + tex_class_off, one byte
                                // per texel at the texture's texel offset, (info & 0xffffff) << 6 (in what was padding)
  const DTexture* textures;
  const uint8_t* tex_pool;      // all RGBA8 textures, each 256-byte aligned, then the texel classes
  const int16_t* tex_segment;   // [n_textures] segment=True replacement of each texture (or the same index)
  DObject agent;                // top-down views: the agent's own mesh (tri_count 0 = none)
  int32_t n_dyn;
  const DDyn* dyn;              // [n_dyn]
  double* dyn_state;            // [DTS_DYN_FIELDS][n_dyn][num_envs]: mutable, per env, survives resets
  const double* dyn_init;       // [DTS_DYN_FIELDS][n_dyn] load-time values (a map reload re-creates the obstacles)
  int32_t valid;
  const double* obj_corners;    // [n_objects][4][2] footprints (x, z) of the bird's-eye map; null: the blob had none
};

// One env's view of its map's dynamic obstacles.
struct DynRef {
  const DDyn* par;
  double* st;
  int32_t n_dyn, n_envs, e;
  __device__ __forceinline__ double& f(int field, int slot) const {
    return st[((size_t)field * n_dyn + slot) * n_envs + e];
  }
};
__device__ __forceinline__ DynRef dyn_ref(const DMap& m, int n_envs, int e) {
  return DynRef{m.dyn, m.dyn_state, e >= 0 ? m.n_dyn : 0, n_envs, e};
}

// ------------------------------------------------------------------ per-env state, SoA in HBM
// One thread per env in the logic kernels: consecutive threads touch consecutive doubles.  kStateArrays (dts_state.cu)
// lists every array once: a new one is allocated and snapshotted by adding it there, and the build fails until it is.
struct DState {
  int32_t n;
  // dynamics (cartesian frame of duckietown_world: x right, y up; S:1629-1652)
  double *cx, *cy, *ctheta, *vu, *vw;
  double* fifo;          // [DTS_MAX_DELAY][2][n]  pending (left,right) duty, slot 0 = oldest
  // simulator-frame pose and per-step outputs
  double *pos_x, *pos_z, *angle, *speed, *reward, *lane_dist, *lane_dot, *lane_angle, *prox;
  double *wheel_dist, *trim;
  int32_t *step_count, *tile_i, *tile_j, *map_id, *episode;
  uint8_t *done_code, *in_lane, *collided;
  uint64_t* rng;         // [6][n] numpy PCG64 stream per env: state hi, lo, inc hi, lo, has_uint32, cached uint32
  struct RenderEp* rep;  // [n] per-episode render parameters (AoS: one CTA reads one record)
  uint8_t *goal_i, *goal_j;   // DTS_FLAG_NAV: the episode's goal tile (such maps are at most 255 tiles a side); else 0
};

// Per-episode render inputs (simulator.py:546-614, 1768): 144 bytes, seven 16-byte groups and the hidden mask, read by
// one CTA per frame.
struct __align__(16) RenderEp {
  float cam_height, cam_angle_deg, cam_fov_y_deg, pad0;
  float cam_noise[3]; float pad1;
  float horizon[3]; float pad2;
  float ambient[3]; float pad3;       // GL_LIGHT0 ambient
  float diffuse[3]; float pad4;       // GL_LIGHT0 diffuse
  float light_eye[4];                 // GL_POSITION as stored by GL: already in eye space
  float ground[3]; float pad5;
  uint32_t hidden[8];                 // bit o = object o invisible
};
static_assert(sizeof(RenderEp) == 144, "dts_debug_episode copies 144 bytes, and the records' sizes count them");

struct DynParams { double u1, u2, u3, w1, w2, w3, uar, ual, war, wal; int32_t delay_steps; };

struct StepCfg {
  double dt, robot_speed, accept_angle_deg;
  double gain, trim, radius, k, limit;
  DynParams dyn;
  int32_t frame_skip, max_steps, action_mode, flags;
  int32_t reward_mode, action_map;      // dts_output_format
  int32_t random_maps, pad0;
  double action_vel_scale;
  uint64_t seed;
  int64_t env_id_offset;
  // Simulator.__init__ keywords read by reset() (S:226-230) and the Randomizer table (randomizer.py:19-89)
  int32_t num_tris_distractors, n_dr_ops;
  double color_sky[3], color_ground[3];
  dts_dr_op dr_ops[DTS_MAX_DR_OPS];
};

// One pixel in a wrapper layout / dtype (dts_output_format): element index of channel c at (x, y)
__device__ __forceinline__ size_t fmt_index(int layout, int x, int y, int c, int W, int H) {
  return layout == DTS_OBS_CHW ? ((size_t)c * H + y) * W + x
       : layout == DTS_OBS_CWH ? ((size_t)c * W + x) * H + y
                               : ((size_t)y * W + x) * 3 + c;
}
// A value v (0..255) as DTS_OBS_F32_UNIT stores it: NormalizeWrapper's v / 255 (LW:66-70)
__device__ __forceinline__ float unit_f32(unsigned v) { return (float)v / 255.0f; }
// Channel c of it, value v (0..255): u8, or float32 v / 255
__device__ __forceinline__ void store_elem_fmt(void* frame, int layout, int dtype, int x, int y, int c, int W, int H, unsigned v) {
  const size_t i = fmt_index(layout, x, y, c, W, H);
  if (dtype == DTS_OBS_F32_UNIT) reinterpret_cast<float*>(frame)[i] = unit_f32(v);
  else reinterpret_cast<uint8_t*>(frame)[i] = (uint8_t)v;
}
__device__ __forceinline__ void store_px_fmt(void* frame, int layout, int dtype, int x, int y, int W, int H, unsigned rgb) {
#pragma unroll
  for (int c = 0; c < 3; c++) store_elem_fmt(frame, layout, dtype, x, y, c, W, H, (rgb >> (8 * c)) & 255u);
}

// Object o's footprint in env `env` of `ne` (DESIGN.md section 5 items 12 and 17): the env's copy of the obstacle's
// corners for an object with a dynamic slot, else the map's obj_corners; false when the map has no footprints.  nd: the
// map's n_dyn (callers looping over objects read it once)
__device__ __forceinline__ bool object_footprint(const DMap& m, size_t nd, size_t ne, int env, int o, double x[4],
                                                 double z[4]) {
  const int slot = m.objects[o].dyn_slot;
  if (slot >= 0) {
    for (int k = 0; k < 4; k++) {
      x[k] = m.dyn_state[((size_t)(DTS_DYN_CORNERS + 2 * k) * nd + slot) * ne + env];
      z[k] = m.dyn_state[((size_t)(DTS_DYN_CORNERS + 2 * k + 1) * nd + slot) * ne + env];
    }
    return true;
  }
  if (!m.obj_corners) return false;
  for (int k = 0; k < 4; k++) {
    x[k] = __ldg(m.obj_corners + (size_t)o * 8 + 2 * k);
    z[k] = __ldg(m.obj_corners + (size_t)o * 8 + 2 * k + 1);
  }
  return true;
}

// A pass over a device env list (RenderCfg::env_list): the number of slots drawn, and the env of slot s < that number
__device__ __forceinline__ int n_listed(const int32_t* list, const int32_t* count, int n_envs) { return list ? __ldg(count) : n_envs; }
__device__ __forceinline__ int listed_env(const int32_t* list, int slot) { return list ? __ldg(list + slot) : slot; }

}  // namespace dts
