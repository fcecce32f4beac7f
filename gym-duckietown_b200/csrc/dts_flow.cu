// dts_flow.cu — the motion-flow image (dts_set_flow_target, DESIGN.md section 5 item 13): for every output pixel, where
// the surface point it shows was in the env's previous frame (the camera and obstacles at the start of its last step,
// recorded by k_flow_record just before k_step_logic), minus where it is now, in output pixels.  The surface is the one the render's own depth and
// label images name, so the pass runs after the rasterisers over the same envs.  Per env the camera motion and one motion
// per dynamic slot are composed in float64 and rounded once to float32 3x4 matrices in shared memory; a pixel then costs
// an unprojection, one 3x4 product, one divide and, under the fisheye, two bilinear reads of the forward map.
#include "dts_camera.cuh"
#include "dts_kernels.h"

namespace dts {
namespace {

constexpr int kFlowThreads = 256;
constexpr int kFlowPxPerThread = 64;   // pixels per CTA = 16384: a 160 x 120 frame is two CTAs per env, so the setup is
                                       // paid twice per env, not ten times
constexpr int kFlowPxPerCta = kFlowThreads * kFlowPxPerThread;
constexpr int kFlowBatch = 8;          // pixels per thread whose depth and label loads are issued together
constexpr int kFlowMats = 2 + DTS_MAX_OBJECTS;   // the scene's, the agent's, one per dynamic slot (at most one per object)
constexpr float kNear = 0.04f;                    // gluPerspective's near plane (S:1761)
constexpr float kOccTau = 0.02f;                  // a mesh point is visible within this share of its depth (DESIGN.md
                                                  // section 5 item 14 measures it)

// out = A * B for row-major 3x4 rigid transforms (the implied fourth row 0 0 0 1)
__device__ inline void compose(const double* A, const double* B, double* out) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++)
      out[4 * r + c] = A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c] + A[4 * r + 2] * B[8 + c] + (c == 3 ? A[4 * r + 3] : 0.0);
}

// The world motion of a mesh drawn at glTranslatef(x, y, z) glRotatef(deg, 0, 1, 0) (GLfloat arguments, as the render
// rounds them) from its current placement to its previous one: T(p_prev) Ry(r_prev) Ry(r_cur)^-1 T(p_cur)^-1.  The
// scale and the height cancel.
__device__ inline void mesh_motion(float px0, float pz0, float deg0, float px1, float pz1, float deg1, double* W) {
  double s0, c0, s1, c1;
  sincos((double)deg0 * kDeg2Rad, &s0, &c0);
  sincos((double)deg1 * kDeg2Rad, &s1, &c1);
  const double A[12] = {c0, 0, s0, (double)px0, 0, 1, 0, 0, -s0, 0, c0, (double)pz0};   // T(p_prev) Ry(r_prev)
  const double B[12] = {c1, 0, -s1, -(c1 * (double)px1 - s1 * (double)pz1),               // Ry(r_cur)^T T(-p_cur)
                        0, 1, 0, 0,
                        s1, 0, c1, -(s1 * (double)px1 + c1 * (double)pz1)};
  compose(A, B, W);
}

// The render-mode bits that change a frame's depth and labels: an occlusion slot's frame is of one view
__device__ __forceinline__ int occ_view(int mode) {
  return mode & (DTS_RENDER_TOP_DOWN | DTS_RENDER_PINHOLE | DTS_RENDER_RECTIFY);
}

// An env's occlusion slots for this render (valid: its flow record is this episode's): .x the slot holding the frame of
// the recorded state in this view, -1 if none; .y the slot this frame goes to, the other one, or with no match the one
// written less recently.  k_flow and k_occ_commit compute it from the same tags, which only k_occ_commit changes.
__device__ __forceinline__ int2 occ_slots(const OcclusionTarget& o, const FlowRecord& rec, const DState& S, int env,
                                          int view, bool valid) {
  const size_t n = S.n;
  int rs = -1;
  if (valid) {
    const int ep = __ldg(rec.episode + env), sc = __ldg(rec.episode + n + env);
    for (int s = 0; s < 2; s++)
      if (__ldg(o.tag + (3 * s) * n + env) == ep && __ldg(o.tag + (3 * s + 1) * n + env) == sc &&
          __ldg(o.tag + (3 * s + 2) * n + env) == view)
        rs = s;
  }
  return make_int2(rs, rs >= 0 ? 1 - rs : 1 - (int)__ldg(o.newest + env));
}

// grid (listed env, chunk of kFlowPxPerCta output pixels); one thread per pixel of the chunk at a time.  kOcc: also the
// occlusion mask (dts_set_occlusion_target) from the slot of the recorded state, and this frame into the other slot.
template <bool kOcc>
__global__ void __launch_bounds__(kFlowThreads) k_flow(DState S, const DMap* __restrict__ maps, RenderCfg rc,
                                                       const FrameCtx* __restrict__ ctx, AuxTargets aux, FlowTarget f,
                                                       FlowRemap rm, OcclusionTarget o) {
  __shared__ float mats[kFlowMats][12];   // 0: ground, tiles and static objects; 1: the agent's mesh; 2 + s: dynamic slot s
  __shared__ double Vp[12], Vi[12];       // the previous frame's camera, the inverse of this frame's
  const int slot = blockIdx.x;
  if (slot >= n_listed(rc.env_list, rc.env_count, rc.n_envs)) return;
  const int env = listed_env(rc.env_list, slot);
  const DMap& m = maps[S.map_id[env]];
  const FrameCtx& c = ctx[env];
  // the record is this episode's (resets, respawns and loads change or clear its number); no forward map for rectified
  const bool valid = !rm.rectify && __ldg(f.rec.episode + env) == S.episode[env];
  const int n_dyn = m.n_dyn, W = rc.width, H = rc.height;
  if (valid) {
    if (threadIdx.x == 0) {   // the same camera the previous frame's k_frame_setup built, from the recorded pose
      const RenderEp ep = S.rep[env];
      if (rc.mode & DTS_RENDER_TOP_DOWN)
        top_down_view((double)m.grid_w, (double)m.grid_h, m.tile_size, (double)ep.cam_fov_y_deg, Vp);
      else
        camera_view(f.rec.pose[env], f.rec.pose[S.n + env], f.rec.pose[2 * S.n + env], ep,
                    (rc.flags & DTS_FLAG_DOMAIN_RAND) != 0, Vp);
    } else if (threadIdx.x == 32) {   // V is rigid: its inverse is [R^T | -R^T t]
      double V[12];
      for (int k = 0; k < 12; k++) V[k] = c.V[k];
      for (int r = 0; r < 3; r++) {
        for (int k = 0; k < 3; k++) Vi[4 * r + k] = V[4 * k + r];
        Vi[4 * r + 3] = -(V[r] * V[3] + V[4 + r] * V[7] + V[8 + r] * V[11]);
      }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 2 + n_dyn; k += kFlowThreads) {
      double Wm[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0}, T[12], M[12];
      if (k == 1) {   // glTranslatef(*cur_pos); glRotatef(cur_angle * 180 / pi, 0, 1, 0), as item_visible rounds them
        const double* pp = f.rec.pose;
        mesh_motion((float)pp[env], (float)pp[S.n + env], (float)(pp[2 * S.n + env] * 180.0 / 3.141592653589793),
                    (float)S.pos_x[env], (float)S.pos_z[env], (float)(S.angle[env] * 180.0 / 3.141592653589793), Wm);
      } else if (k >= 2 && m.dyn[k - 2].kind != DTS_DYN_TRAFFICLIGHT) {   // a moving obstacle (a light's pose is fixed)
        const size_t nd = n_dyn, ne = S.n, s = k - 2, md = f.rec.max_dyn;
        const double* d = f.rec.dyn;
        mesh_motion((float)d[(0 * md + s) * ne + env], (float)d[(1 * md + s) * ne + env], (float)d[(2 * md + s) * ne + env],
                    (float)m.dyn_state[((size_t)DTS_DYN_PX * nd + s) * ne + env],
                    (float)m.dyn_state[((size_t)DTS_DYN_PZ * nd + s) * ne + env],
                    (float)m.dyn_state[((size_t)DTS_DYN_YROT * nd + s) * ne + env], Wm);
      }
      compose(Wm, Vi, T);
      compose(Vp, T, M);
      for (int q = 0; q < 12; q++) mats[k][q] = (float)M[q];
    }
    __syncthreads();
  }
  const int hw = W * H, n_tiles = m.n_tiles, agent = 2 + m.n_tiles + m.n_objects;
  const size_t row = (size_t)env * hw;
  const float P00 = c.P00, P11 = c.P11, fw = (float)W, fh = (float)H;
  const int table = rm.table_of_env ? __ldg(rm.table_of_env + env) : 0;
  const int32_t* src = rm.src_xy ? rm.src_xy + (size_t)table * hw : nullptr;
  const float2* fwd = rm.fwd ? rm.fwd + (size_t)table * hw : nullptr;
  float2* out = reinterpret_cast<float2*>(f.out) + row;
  const float nan = __int_as_float(0x7fc00000);
  int2 occ = make_int2(-1, 0);   // (the slot read, -1: none; the slot written)
  if constexpr (kOcc) occ = occ_slots(o, f.rec, S, env, occ_view(rc.mode), valid);
  const size_t slot_px = (size_t)S.n * hw;
  const float* dprev = o.depth + max(occ.x, 0) * slot_px + row;   // (read only where occ.x >= 0)
  const int16_t* lprev = o.labels + max(occ.x, 0) * slot_px + row;
  const int t0 = blockIdx.y * kFlowPxPerCta + threadIdx.x;
  for (int k0 = 0; k0 < kFlowPxPerThread; k0 += kFlowBatch) {
    if (t0 + k0 * kFlowThreads >= hw) break;
    float db[kFlowBatch];   // a batch of pixels' loads in flight before any of them is used
    int16_t lb[kFlowBatch];
#pragma unroll
    for (int b = 0; b < kFlowBatch; b++) {
      const int t = t0 + (k0 + b) * kFlowThreads;
      db[b] = (kOcc || valid) && t < hw ? __ldg(aux.depth + row + t) : 0.0f;   // (kOcc: every frame goes to a slot)
      lb[b] = (kOcc || valid) && t < hw ? __ldg(aux.labels + row + t) : (int16_t)0;
    }
#pragma unroll
    for (int b = 0; b < kFlowBatch; b++) {
    const int t = t0 + (k0 + b) * kFlowThreads;
    if (t >= hw) break;
    float2 flow = make_float2(nan, nan);
    float zp = 0.0f;   // the point's depth in the previous camera, where flow is defined
    const float d = db[b];
    if ((!kOcc || valid) && d > 0.0f) {   // (0: sky, or no source pixel)
      int sx, sy;
      if (src) {
        const int v = __ldg(src + t);
        sx = (int)(int16_t)(v & 0xffff); sy = v >> 16;
      } else {
        sy = t / W; sx = t - sy * W;
      }
      const int lab = lb[b];
      int mi = 0;
      if (lab == agent) mi = 1;
      else if (lab > 1 + n_tiles) {
        const int ds = __ldg(&m.objects[lab - 2 - n_tiles].dyn_slot);
        mi = ds >= 0 ? 2 + ds : 0;
      }
      const float* M = mats[mi];
      const float xs = (float)sx + 0.5f, ys = (float)sy + 0.5f;
      const float ex = (2.0f * xs / fw - 1.0f) * d / P00, ey = (1.0f - 2.0f * ys / fh) * d / P11, ez = -d;
      const float qx = M[0] * ex + M[1] * ey + M[2] * ez + M[3];
      const float qy = M[4] * ex + M[5] * ey + M[6] * ez + M[7];
      const float qz = M[8] * ex + M[9] * ey + M[10] * ez + M[11];
      if (qz < -kNear) {
        zp = -qz;
        const float iz = 1.0f / -qz;
        const float x1 = (P00 * qx * iz + 1.0f) * fw * 0.5f, y1 = (1.0f - P11 * qy * iz) * fh * 0.5f;
        if (!fwd) {
          flow = make_float2(x1 - xs, y1 - ys);
        } else {   // both ends through the same forward map, so a still point gives 0 up to the matrices' rounding
          float2 a, b;
          if (forward_map(fwd, W, H, x1, y1, a) && forward_map(fwd, W, H, xs, ys, b)) flow = make_float2(a.x - b.x, a.y - b.y);
        }
      }
    }
    out[t] = flow;
    if constexpr (kOcc) {   // DESIGN.md section 5 item 14
      const int lab = lb[b];
      uint8_t mv = DTS_OCC_NONE;
      if (flow.x == flow.x) {   // (NaN in both components or neither)
        const int py = t / W, px = t - py * W;
        const float qx = (float)px + 0.5f + flow.x, qy = (float)py + 0.5f + flow.y;
        if (!(qx >= 0.0f && qx < fw && qy >= 0.0f && qy < fh)) {
          mv = DTS_OCC_OUTSIDE;
        } else if (occ.x < 0) {
          mv = DTS_OCC_UNKNOWN;
        } else {   // visible where one of the four pixels around q shows the item, and a mesh at the point's depth
          mv = DTS_OCC_OCCLUDED;
          const bool flat = lab <= 1 + n_tiles;   // ground or a road tile: cannot hide part of itself
          const int cx = (int)floorf(qx - 0.5f), cy = (int)floorf(qy - 0.5f);
#pragma unroll
          for (int j = 0; j < 2; j++)
#pragma unroll
            for (int i = 0; i < 2; i++) {
              const int x = cx + i, y = cy + j;
              if (x < 0 || x >= W || y < 0 || y >= H) continue;
              const int c = y * W + x;
              if (__ldg(lprev + c) == lab && (flat || fabsf(__ldg(dprev + c) - zp) <= kOccTau * zp)) mv = DTS_OCC_VISIBLE;
            }
        }
      }
      o.out[row + t] = mv;
      o.depth[occ.y * slot_px + row + t] = d;   // this frame, the previous one of the next step's mask
      o.labels[occ.y * slot_px + row + t] = (int16_t)lab;
    }
    }
  }
}

// thread per listed env, after k_flow: the slot k_flow wrote now holds this frame.  (Not in k_flow itself, whose other
// CTAs of the env may still be choosing their slots from the tags.)
__global__ void __launch_bounds__(128) k_occ_commit(DState S, RenderCfg rc, FlowRecord rec, OcclusionTarget o,
                                                    bool rectify) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= n_listed(rc.env_list, rc.env_count, rc.n_envs)) return;
  const int env = listed_env(rc.env_list, slot);
  const int view = occ_view(rc.mode);
  const int ws = occ_slots(o, rec, S, env, view, !rectify && __ldg(rec.episode + env) == S.episode[env]).y;
  const size_t n = S.n;
  o.tag[(3 * ws) * n + env] = S.episode[env];
  o.tag[(3 * ws + 1) * n + env] = S.step_count[env];
  o.tag[(3 * ws + 2) * n + env] = view;
  o.newest[env] = (uint8_t)ws;
}

// thread per env: the pose and obstacles the step is about to move, and the episode they belong to
__global__ void __launch_bounds__(128) k_flow_record(DState S, const DMap* __restrict__ maps, FlowRecord rec) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S.n) return;
  const DMap& m = maps[S.map_id[e]];
  rec.pose[e] = S.pos_x[e]; rec.pose[S.n + e] = S.pos_z[e]; rec.pose[2 * S.n + e] = S.angle[e];
  const int fields[3] = {DTS_DYN_PX, DTS_DYN_PZ, DTS_DYN_YROT};
  for (int k = 0; k < m.n_dyn; k++)
    for (int f = 0; f < 3; f++)
      rec.dyn[((size_t)f * rec.max_dyn + k) * S.n + e] = m.dyn_state[((size_t)fields[f] * m.n_dyn + k) * S.n + e];
  rec.episode[e] = S.episode[e];
  rec.episode[S.n + e] = S.step_count[e];
}

// occ_tag: null, or the occlusion slots' tags, whose frames the env forgets with its record
__global__ void k_flow_forget(int32_t* __restrict__ episode, int32_t* __restrict__ occ_tag,
                              const uint8_t* __restrict__ mask, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n && (!mask || mask[e])) {
    episode[e] = -1;
    if (occ_tag) occ_tag[e] = occ_tag[3 * (size_t)n + e] = -1;
  }
}

}  // namespace

std::string flow_record_alloc(FlowRecord& rec, int n_envs, int max_dyn) {
  FlowRecord r{nullptr, nullptr, nullptr, max_dyn};
  const size_t n = n_envs;
  cudaError_t e = cudaMalloc(&r.pose, 3 * n * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&r.dyn, 3 * (size_t)(max_dyn > 0 ? max_dyn : 1) * n * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&r.episode, 2 * n * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMemset(r.episode, 0xff, 2 * n * sizeof(int32_t));   // -1: no previous frame
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    flow_record_free(r);
    return std::string("flow record allocation failed: ") + cudaGetErrorString(e);
  }
  rec = r;
  return "";
}

void flow_record_free(FlowRecord& rec) {
  cudaFree(rec.pose);
  cudaFree(rec.dyn);
  cudaFree(rec.episode);
  rec = FlowRecord{};
}

void launch_flow_record(const DState& S, const DMap* maps, const FlowRecord& rec, cudaStream_t st) {
  k_flow_record<<<(S.n + 127) / 128, 128, 0, st>>>(S, maps, rec);
}

void launch_flow_forget(const FlowRecord& rec, const OcclusionTarget& occ, const uint8_t* mask, int n_envs,
                        cudaStream_t st) {
  k_flow_forget<<<(n_envs + 127) / 128, 128, 0, st>>>(rec.episode, occ.tag, mask, n_envs);
}

std::string occlusion_alloc(OcclusionTarget& occ, uint8_t* out, int n_envs, int width, int height) {
  OcclusionTarget o{out, nullptr, nullptr, nullptr, nullptr};
  const size_t n = n_envs, px = 2 * n * width * height;
  cudaError_t e = cudaMalloc(&o.depth, px * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&o.labels, px * sizeof(int16_t));
  if (e == cudaSuccess) e = cudaMalloc(&o.tag, 6 * n * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&o.newest, n);
  if (e == cudaSuccess) e = cudaMemset(o.newest, 0, n);
  if (e == cudaSuccess) e = cudaMemset(o.tag, 0xff, 6 * n * sizeof(int32_t));   // episode -1: empty
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    occlusion_free(o);
    cudaGetLastError();   // (a failed allocation is refused, not left for the next launch to report)
    return std::string("occlusion slot allocation (") + std::to_string(px * 6 + 25 * n) + " B) failed: " +
           cudaGetErrorString(e);
  }
  occ = o;
  return "";
}

std::string occlusion_empty(const OcclusionTarget& occ, int n_envs) {
  cudaError_t e = cudaMemset(occ.tag, 0xff, 6 * (size_t)n_envs * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return e == cudaSuccess ? "" : std::string("emptying the occlusion slots failed: ") + cudaGetErrorString(e);
}

void occlusion_free(OcclusionTarget& occ) {
  cudaFree(occ.depth);
  cudaFree(occ.labels);
  cudaFree(occ.tag);
  cudaFree(occ.newest);
  occ = OcclusionTarget{};
}

int launch_flow(const DState& S, const DMap* maps, const RenderCfg& rc, const FrameCtx* ctx, const AuxTargets& aux,
                const FlowTarget& f, const FlowRemap& rm, const OcclusionTarget& occ, cudaStream_t st) {
  const int hw = rc.width * rc.height;
  const dim3 grid(rc.n_envs, (hw + kFlowPxPerCta - 1) / kFlowPxPerCta);
  if (!occ.out) {
    k_flow<false><<<grid, kFlowThreads, 0, st>>>(S, maps, rc, ctx, aux, f, rm, occ);
    return 1;
  }
  k_flow<true><<<grid, kFlowThreads, 0, st>>>(S, maps, rc, ctx, aux, f, rm, occ);
  k_occ_commit<<<(rc.n_envs + 127) / 128, 128, 0, st>>>(S, rc, f.rec, occ, rm.rectify);
  return 2;
}

}  // namespace dts
