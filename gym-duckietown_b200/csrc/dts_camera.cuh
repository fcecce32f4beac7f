// dts_camera.cuh — agent camera matrices of _render_img (simulator.py:1758-1803), float64,
// row-major 3x4 [R|t].  Shared by the render kernel and by the device reset (the reference captures
// GL_LIGHT0's position under whatever modelview the previous frame left, S:581); and the fisheye's forward map.
#pragma once
#include "dts_common.cuh"

namespace dts {

constexpr double kDeg2Rad = 0.017453292519943295;

// modelview = Rx(cam_angle) * T(0,0,CAMERA_FORWARD_DIST) * gluLookAt(eye, eye+dir, +y)   S:1780-1803
__host__ __device__ inline void camera_view(double px, double pz, double angle, const RenderEp& ep, bool domain_rand,
                                            double V[12]) {
  double ex = px, ey = 0.0, ez = pz;
  if (domain_rand) { ex += (double)ep.cam_noise[0]; ey += (double)ep.cam_noise[1]; ez += (double)ep.cam_noise[2]; }  // S:1768-1769
  ey += (double)ep.cam_height;                                                                                       // S:1780
  double fx = cos(angle), fy = 0.0, fz = -sin(angle);  // get_dir_vec S:2056
  const double fn = sqrt(fx * fx + fy * fy + fz * fz);
  fx /= fn; fy /= fn; fz /= fn;
  // s = f x up, up = (0,1,0)
  double sx = fy * 0.0 - fz * 1.0, sy = fz * 0.0 - fx * 0.0, sz = fx * 1.0 - fy * 0.0;
  const double sn = sqrt(sx * sx + sy * sy + sz * sz);
  sx /= sn; sy /= sn; sz /= sn;
  const double ux = sy * fz - sz * fy, uy = sz * fx - sx * fz, uz = sx * fy - sy * fx;  // u = s x f
  double L[12] = {sx, sy, sz, -(sx * ex + sy * ey + sz * ez),
                  ux, uy, uz, -(ux * ex + uy * ey + uz * ez),
                  -fx, -fy, -fz, (fx * ex + fy * ey + fz * ez)};
  L[11] += (double)0.066f;  // glTranslatef(0, 0, CAMERA_FORWARD_DIST) S:1784: a GLfloat argument (S:131)
  const double th = (double)ep.cam_angle_deg * kDeg2Rad;
  const double c = cos(th), s = sin(th);
  for (int k = 0; k < 4; k++) {
    V[k] = L[k];
    V[4 + k] = c * L[4 + k] - s * L[8 + k];
    V[8 + k] = s * L[4 + k] + c * L[8 + k];
  }
}

// top_down=True (S:1786-1798): gluLookAt from (a, H, b) to (a, 0, b - 0.01), up +y, a / b = half the map extents,
// H = (max(a, b) + 0.1) / tan(fov_y / 2); no camera tilt / forward offset in this view.
__host__ __device__ inline void top_down_view(double grid_w, double grid_h, double tile_size, double fov_y_deg, double V[12]) {
  const double a = (grid_w * tile_size) / 2, b = (grid_h * tile_size) / 2;
  const double H = ((a > b ? a : b) + 0.1) / tan(fov_y_deg * kDeg2Rad / 2);
  const double ex = a, ey = H, ez = b;
  double fx = 0.0, fy = 0.0 - H, fz = (b - 0.01) - b;
  const double fn = sqrt(fx * fx + fy * fy + fz * fz);
  fx /= fn; fy /= fn; fz /= fn;
  double sx = fy * 0.0 - fz * 1.0, sy = fz * 0.0 - fx * 0.0, sz = fx * 1.0 - fy * 0.0;   // s = f x up
  const double sn = sqrt(sx * sx + sy * sy + sz * sz);
  sx /= sn; sy /= sn; sz /= sn;
  const double ux = sy * fz - sz * fy, uy = sz * fx - sx * fz, uz = sx * fy - sy * fx;   // u = s x f
  const double L[12] = {sx, sy, sz, -(sx * ex + sy * ey + sz * ez),
                        ux, uy, uz, -(ux * ex + uy * ey + uz * ez),
                        -fx, -fy, -fz, (fx * ex + fy * ey + fz * ez)};
  for (int k = 0; k < 12; k++) V[k] = L[k];
}

// Bilinear read of a forward map F [H][W] (the flow image's and the bird's-eye visibility's; OpenCV's convention: table
// index = position - 0.5); false where the footprint leaves it
__device__ __forceinline__ bool forward_map(const float2* __restrict__ F, int W, int H, float x, float y, float2& out) {
  const float ix = x - 0.5f, iy = y - 0.5f;
  if (!(ix >= 0.0f && ix <= (float)(W - 1) && iy >= 0.0f && iy <= (float)(H - 1))) return false;   // (NaN: false)
  const int x0 = min((int)ix, max(W - 2, 0)), y0 = min((int)iy, max(H - 2, 0));
  const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  const float ax = ix - (float)x0, ay = iy - (float)y0;
  const float2 f00 = __ldg(F + (size_t)y0 * W + x0), f01 = __ldg(F + (size_t)y0 * W + x1);
  const float2 f10 = __ldg(F + (size_t)y1 * W + x0), f11 = __ldg(F + (size_t)y1 * W + x1);
  const float tx = f00.x + ax * (f01.x - f00.x), ty = f00.y + ax * (f01.y - f00.y);
  const float bx = f10.x + ax * (f11.x - f10.x), by = f10.y + ax * (f11.y - f10.y);
  out = make_float2(tx + ay * (bx - tx), ty + ay * (by - ty));
  return true;
}

// A world point (x, y, z) to the pixel q of a W x H frame drawn under modelview V and gluPerspective's P00, P11, then
// through the forward map `fwd` unless it is null (the pinhole and top-down views).  False where the point does not lie
// within the near and far planes (0.04 < -ez <= 100, S:1761) or F's footprint leaves the table; a point outside the
// frame is kept.
__device__ __forceinline__ bool project_to_frame(const double* V, double P00, double P11, const float2* __restrict__ fwd,
                                                 int W, int H, double x, double y, double z, float2& q) {
  const double ex = V[0] * x + V[1] * y + V[2] * z + V[3];
  const double ey = V[4] * x + V[5] * y + V[6] * z + V[7];
  const double w = -(V[8] * x + V[9] * y + V[10] * z + V[11]);
  if (!(w > 0.04 && w <= 100.0)) return false;
  const double iw = 1.0 / w;
  const double qx = (P00 * (ex * iw) + 1.0) * (0.5 * W), qy = (1.0 - P11 * (ey * iw)) * (0.5 * H);
  q = make_float2((float)qx, (float)qy);
  return !fwd || forward_map(fwd, W, H, (float)qx, (float)qy, q);
}

// Eye-space GL_POSITION for a light given under modelview V: positional (w=1) or direction (w=0).
__host__ __device__ inline void light_to_eye(const double V[12], const float lp[4], float out[4]) {
  const double x = lp[0], y = lp[1], z = lp[2], w = lp[3];
  out[0] = (float)(V[0] * x + V[1] * y + V[2] * z + V[3] * w);
  out[1] = (float)(V[4] * x + V[5] * y + V[6] * z + V[7] * w);
  out[2] = (float)(V[8] * x + V[9] * y + V[10] * z + V[11] * w);
  out[3] = (float)w;
}

}  // namespace dts
