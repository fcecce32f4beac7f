// dts_path.cu — the lane path ahead of every agent (dts_set_lane_path_target, DESIGN.md section 5 item 18): a walk of
// closest_curve_point calls along the lane's centre curve, each from a step of `spacing` along the previous tangent, in
// float64 in the order the spec states (-fmad=false keeps every product and sum separately rounded, as numpy's are).
#include "dts_camera.cuh"
#include "dts_kernels.h"
#include "dts_logic.cuh"

namespace dts {
namespace {

// The walk is serial in k, so a thread per env, and its cost is the latency of one thread's chain of K calls.  A CTA of
// one warp spreads the envs over every SM: at 4096 envs that is 128 warps, about one per SM.  CTAs of 16 or 8 threads,
// which put more warps on each SM, measured within 7 % of it on an H100.
constexpr int kPathThreads = 32;

// grid: a thread per env.  Each thread stores its own rows straight to global memory: a row is K points of 12 B and K
// pixels of 8 B, and the writes of a warp's 32 rows fill their sectors in L2 over the walk.
__global__ void __launch_bounds__(kPathThreads) k_lane_path(DState S, const DMap* __restrict__ maps, LanePathTarget t,
                                                            const FrameCtx* __restrict__ ctx, int W, int H,
                                                            FlowRemap rm, bool drew) {
  const int env = blockIdx.x * kPathThreads + threadIdx.x;
  if (env >= S.n) return;
  const DMap& m = maps[S.map_id[env]];
  const int K = t.n_points;
  const double ds = t.spacing;
  const double px0 = S.pos_x[env], pz0 = S.pos_z[env];
  double sa, ca;
  sincos(S.angle[env], &sa, &ca);
  const float nan = __int_as_float(0x7fc00000);
  float* pts = t.points ? t.points + (size_t)env * K * 3 : nullptr;
  float* pix = t.px ? t.px + (size_t)env * K * 2 : nullptr;
  const bool project = pix && drew && !rm.rectify;
  const double* V = nullptr;
  double P00 = 0.0, P11 = 0.0;
  const float2* fwd = nullptr;
  if (project) {
    const FrameCtx& c = ctx[env];
    V = c.V;
    P00 = c.P00;
    P11 = c.P11;
    fwd = rm.fwd ? rm.fwd + (size_t)(rm.table_of_env ? __ldg(rm.table_of_env + env) : 0) * W * H : nullptr;
  }
  double qx = px0, qz = pz0, heading = S.angle[env];   // the query of point k and the heading its curve is chosen by
  int n = 0;
#pragma unroll 1
  for (; n < K; n++) {
    double q[3], tg[3];
    if (!closest_curve_point(m, qx, qz, heading, q, tg)) break;
    if (pts) {
      const double dx = q[0] - px0, dz = q[2] - pz0;
      const double fe = tg[0] * ca - tg[2] * sa, re = tg[0] * sa + tg[2] * ca;
      double yaw = atan2(-re, fe);
      if (yaw <= -M_PI) yaw = M_PI;   // (-pi, pi]
      pts[3 * n] = (float)(dx * ca - dz * sa);
      pts[3 * n + 1] = (float)(dx * sa + dz * ca);
      pts[3 * n + 2] = (float)yaw;
    }
    if (pix) {
      float2 p = make_float2(nan, nan);
      if (project && !project_to_frame(V, P00, P11, fwd, W, H, q[0], q[1], q[2], p)) p = make_float2(nan, nan);
      pix[2 * n] = p.x;
      pix[2 * n + 1] = p.y;
    }
    heading = atan2(-tg[2], tg[0]);   // get_dir_vec(heading) lies along the tangent
    qx = q[0] + ds * tg[0];
    qz = q[2] + ds * tg[2];
  }
  if (t.count) t.count[env] = (int16_t)n;
  for (int k = n; k < K; k++) {
    if (pts) { pts[3 * k] = nan; pts[3 * k + 1] = nan; pts[3 * k + 2] = nan; }
    if (pix) { pix[2 * k] = nan; pix[2 * k + 1] = nan; }
  }
}

}  // namespace

void launch_lane_path(const DState& S, const DMap* maps, const LanePathTarget& t, const FrameCtx* ctx, int W, int H,
                      const FlowRemap& rm, bool drew_frame, cudaStream_t st) {
  k_lane_path<<<(S.n + kPathThreads - 1) / kPathThreads, kPathThreads, 0, st>>>(S, maps, t, ctx, W, H, rm, drew_frame);
}

}  // namespace dts
