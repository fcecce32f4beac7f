// dts_objects.cu — object-level outputs.  k_objects: every object's 3D box around every agent and where its corners land
// in the frame the call drew (dts_set_object_target, DESIGN.md section 5 item 17), a thread per (env, object slot), in
// float64 in the order the spec states (-fmad=false keeps every product and sum separately rounded, as numpy's are).
// k_object_pixels: each object's visible pixel count and bounding box in a label image (dts_object_pixels).
#include <climits>

#include "dts_camera.cuh"
#include "dts_kernels.h"

namespace dts {
namespace {

constexpr int kObjThreads = 256;
constexpr int kBoxFloats = 7;          // forward, right, up, length, width, height, yaw
constexpr int kCornerFloats = 9 * 2;   // 8 box corners and the centre, x and y in pixels

// grid: kObjThreads consecutive (env, slot) pairs per CTA, slot fastest.  Each thread stages its row in shared memory and
// the CTA stores its contiguous run of every output with consecutive threads on consecutive words.
__global__ void __launch_bounds__(kObjThreads) k_objects(DState S, const DMap* __restrict__ maps,
                                                         const float2* const* __restrict__ extent, ObjectTarget t,
                                                         const FrameCtx* __restrict__ ctx, int W, int H, FlowRemap rm,
                                                         bool drew) {
  __shared__ float box_s[kObjThreads * kBoxFloats];
  __shared__ float px_s[kObjThreads * kCornerFloats];
  __shared__ uint8_t state_s[kObjThreads];
  const int O = t.max_objects;
  const long long total = (long long)S.n * O, first = (long long)blockIdx.x * kObjThreads;
  const long long at = first + threadIdx.x;
  const float nan = __int_as_float(0x7fc00000);
  float* box = box_s + threadIdx.x * kBoxFloats;
  float* px = px_s + threadIdx.x * kCornerFloats;
  for (int k = 0; k < kBoxFloats; k++) box[k] = nan;
  for (int k = 0; k < kCornerFloats; k++) px[k] = nan;
  state_s[threadIdx.x] = DTS_OBJECT_NONE;
  if (at < total) {
    const int env = (int)(at / O), o = (int)(at - (long long)env * O);
    const int map_id = S.map_id[env];
    const DMap& m = maps[map_id];
    double cx[4], cz[4];
    if (o < m.n_objects && object_footprint(m, m.n_dyn, S.n, env, o, cx, cz)) {
      // c0 -> c1 along the heading.  A Duckiebot's turning step rewrites its corners in agent_boundbox's order
      // (back-left, back-right, front-right, front-left; collision.py:9-31), whose heading edge is c1 -> c2: the edge
      // that lies along get_dir_vec(DTS_DYN_ANGLE) says which order the corners are in.
      const int slot = m.objects[o].dyn_slot;
      if (slot >= 0 && m.dyn[slot].kind == DTS_DYN_DUCKIEBOT) {
        double sh, ch;
        sincos(m.dyn_state[((size_t)DTS_DYN_ANGLE * m.n_dyn + slot) * S.n + env], &sh, &ch);
        const double a01 = fabs((cx[1] - cx[0]) * ch - (cz[1] - cz[0]) * sh);
        const double a12 = fabs((cx[2] - cx[1]) * ch - (cz[2] - cz[1]) * sh);
        if (a12 > a01) {
          const double x0 = cx[0], z0 = cz[0];
          for (int k = 0; k < 3; k++) { cx[k] = cx[k + 1]; cz[k] = cz[k + 1]; }
          cx[3] = x0; cz[3] = z0;
        }
      }
      const uint32_t* hidden = S.rep[env].hidden;
      state_s[threadIdx.x] = (hidden[o >> 5] >> (o & 31) & 1u) ? DTS_OBJECT_HIDDEN : DTS_OBJECT_SHOWN;
      const DObject& d = m.objects[o];
      const float2 ext = extent[map_id][o];
      const double scale = d.scale, y0 = d.dpos[1] + scale * (double)ext.x, y1 = d.dpos[1] + scale * (double)ext.y;
      const double px0 = S.pos_x[env], pz0 = S.pos_z[env];
      double sa, ca;
      sincos(S.angle[env], &sa, &ca);
      const double mx = (((cx[0] + cx[1]) + cx[2]) + cx[3]) / 4.0, mz = (((cz[0] + cz[1]) + cz[2]) + cz[3]) / 4.0;
      const double my = (y0 + y1) / 2.0;
      const double dx = mx - px0, dz = mz - pz0;
      const double ex = cx[1] - cx[0], ez = cz[1] - cz[0];   // c0 -> c1: the object's heading
      const double wx = cx[2] - cx[1], wz = cz[2] - cz[1];
      const double fe = ex * ca - ez * sa, re = ex * sa + ez * ca;
      double yaw = atan2(-re, fe);
      if (yaw <= -M_PI) yaw = M_PI;   // (-pi, pi]
      box[0] = (float)(dx * ca - dz * sa);
      box[1] = (float)(dx * sa + dz * ca);
      box[2] = (float)my;
      box[3] = (float)sqrt(ex * ex + ez * ez);
      box[4] = (float)sqrt(wx * wx + wz * wz);
      box[5] = (float)(y1 - y0);
      box[6] = (float)yaw;
      if (drew && !rm.rectify) {
        const FrameCtx& c = ctx[env];
        const double* V = c.V;
        const double P00 = c.P00, P11 = c.P11;
        const float2* fwd =
            rm.fwd ? rm.fwd + (size_t)(rm.table_of_env ? __ldg(rm.table_of_env + env) : 0) * W * H : nullptr;
        for (int k = 0; k < 9; k++) {
          const double x = k < 8 ? cx[k & 3] : mx, y = k < 4 ? y0 : k < 8 ? y1 : my, z = k < 8 ? cz[k & 3] : mz;
          float2 q;
          if (!project_to_frame(V, P00, P11, fwd, W, H, x, y, z, q)) continue;
          px[2 * k] = q.x;
          px[2 * k + 1] = q.y;
        }
      }
    }
  }
  __syncthreads();
  const int n = (int)(total - first < kObjThreads ? total - first : kObjThreads);
  if (t.boxes)
    for (int i = threadIdx.x; i < n * kBoxFloats; i += kObjThreads) t.boxes[first * kBoxFloats + i] = box_s[i];
  if (t.corners) {
    float* out = reinterpret_cast<float*>(t.corners) + first * kCornerFloats;
    for (int i = threadIdx.x; i < n * kCornerFloats; i += kObjThreads) out[i] = px_s[i];
  }
  if (t.state && threadIdx.x < n) t.state[first + threadIdx.x] = state_s[threadIdx.x];
}

constexpr int kPixThreads = 256;

// One pixel of the label image at (x, y), for every lane of the warp at once (`in`: the lane has a pixel): the lanes
// showing the same object add their count and bounds in one shared atomic each, from the group's lowest lane.
__device__ __forceinline__ void count_pixel(int label, int x, int y, bool in, int lane, int base, int n_obj,
                                            int* cnt, int* x0, int* y0, int* x1, int* y1) {
  const int o = label - base;
  const int key = in && o >= 0 && o < n_obj ? o : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  if (key < 0) return;
  const int lx = __reduce_min_sync(peers, (unsigned)x), hx = __reduce_max_sync(peers, (unsigned)x);
  const int ly = __reduce_min_sync(peers, (unsigned)y), hy = __reduce_max_sync(peers, (unsigned)y);
  if (lane == __ffs(peers) - 1) {
    atomicAdd(cnt + key, __popc(peers));
    atomicMin(x0 + key, lx); atomicMax(x1 + key, hx);
    atomicMin(y0 + key, ly); atomicMax(y1 + key, hy);
  }
}

// grid: one CTA per env.  The image is read as one run of W * H labels: a scalar head up to 16-byte alignment, 16-byte
// loads of 8 labels, and a scalar tail, so any W and any row alignment is read whole.  Every warp steps through its
// share in lockstep, so that count_pixel's warp intrinsics see all 32 lanes.
__global__ void __launch_bounds__(kPixThreads) k_object_pixels(DState S, const DMap* __restrict__ maps,
                                                               const int16_t* __restrict__ labels, int W, int H,
                                                               int32_t* pixels, int32_t* boxes, int max_objects) {
  __shared__ int cnt[DTS_MAX_OBJECTS], x0[DTS_MAX_OBJECTS], y0[DTS_MAX_OBJECTS], x1[DTS_MAX_OBJECTS], y1[DTS_MAX_OBJECTS];
  const int env = blockIdx.x;
  const DMap& m = maps[S.map_id[env]];
  const int n_obj = m.n_objects, base = 2 + m.n_tiles;   // object o's label (render spec item 10)
  for (int o = threadIdx.x; o < DTS_MAX_OBJECTS; o += kPixThreads) {
    cnt[o] = 0; x0[o] = INT_MAX; y0[o] = INT_MAX; x1[o] = -1; y1[o] = -1;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = kPixThreads / 32;
  const int n = W * H;
  const int16_t* img = labels + (size_t)env * n;
  const int head = min((int)((16 - (reinterpret_cast<uintptr_t>(img) & 15)) & 15) / 2, n);
  const int n_vec = (n - head) / 8, tail = head + n_vec * 8;
  // the head and the tail: fewer than 16 labels
  if (warp == 0) {
    const int p = lane < head ? lane : tail + (lane - head);
    const bool in = lane < head || (p < n && lane - head < 8);
    const int label = in ? __ldg(img + p) : 0;
    count_pixel(label, in ? p % W : 0, in ? p / W : 0, in, lane, base, n_obj, cnt, x0, y0, x1, y1);
  }
  const int4* vec = reinterpret_cast<const int4*>(img + head);
  for (int b = warp * 32; b < n_vec; b += warps * 32) {
    const int i = b + lane;
    const bool in = i < n_vec;
    int4 v = make_int4(0, 0, 0, 0);
    if (in) v = __ldg(vec + i);
    const int p = head + i * 8;
    int y = in ? p / W : 0, x = in ? p - y * W : 0;
    const int words[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int label = (int16_t)(words[k >> 1] >> (16 * (k & 1)) & 0xffff);
      count_pixel(label, x, y, in, lane, base, n_obj, cnt, x0, y0, x1, y1);
      if (++x == W) { x = 0; y++; }
    }
  }
  __syncthreads();
  for (int o = threadIdx.x; o < max_objects; o += kPixThreads) {
    const size_t r = (size_t)env * max_objects + o;
    const int c = o < n_obj ? cnt[o] : 0;
    pixels[r] = c;
    boxes[4 * r] = c ? x0[o] : -1;
    boxes[4 * r + 1] = c ? y0[o] : -1;
    boxes[4 * r + 2] = c ? x1[o] : -1;
    boxes[4 * r + 3] = c ? y1[o] : -1;
  }
}

}  // namespace

void launch_objects(const DState& S, const DMap* maps, const float2* const* extent, const ObjectTarget& t,
                    const FrameCtx* ctx, int W, int H, const FlowRemap& rm, bool drew_frame, cudaStream_t st) {
  const long long total = (long long)S.n * t.max_objects;
  k_objects<<<(unsigned)((total + kObjThreads - 1) / kObjThreads), kObjThreads, 0, st>>>(S, maps, extent, t, ctx, W, H,
                                                                                        rm, drew_frame);
}

void launch_object_pixels(const DState& S, const DMap* maps, const int16_t* labels, int W, int H, int32_t* pixels,
                          int32_t* boxes, int max_objects, cudaStream_t st) {
  k_object_pixels<<<S.n, kPixThreads, 0, st>>>(S, maps, labels, W, H, pixels, boxes, max_objects);
}

}  // namespace dts
