// dts_render.cu — batched software rasteriser for the agent camera (Simulator._render_img,
// simulator.py:1707-1951) on sm_90a (H100).  No tensor cores: there is no dense contraction here.
//
// Stream-ordered kernels per frame batch (k_cull, a work-list pre-pass for k_geometry, and k_raster_solo / k_raster_flat,
// the lean rasterisers of coarse bins lying inside one prim / holding only road tiles and ground, are described at their
// definitions):
//   k_frame_setup  thread per env: camera matrices (f64), gluPerspective, counters -> FrameCtx[env]
//   k_tiles        warp per env, lane per road tile (tile mode 1): the ground and the map's tiles.  A road tile is ONE
//                  quad: its 8x8 lit lattice goes to the env's table and the Gouraud interpolant is evaluated per
//                  pixel (render spec tile mode 1); RenderCfg.tessellate switches to the literal 98 triangles (mode 0),
//                  which k_geometry draws like meshes.
//   k_geometry     warp per (env, draw item) over the whole GPU: placed meshes (and in tile mode 0 the ground and the
//                  tiles).  Model-view f64->f32, fixed-function per-vertex lighting, frustum cull, near + guard-band
//                  clip, snap to 1/64 px, triangle setup -> 128-byte PrimRec appended to the env's slab.
//   k_bin          warp per env: exact (prim, 32x8-px coarse bin) pairs — count, warp scan, scatter — then, dense
//                  over the pairs (one pair per lane), the 80-byte BinRec each pair needs for visibility: edge
//                  functions re-based to the bin corner (exact in 64 bits, then int32), per-fine-bin reject /
//                  trivial-accept bits, the depth plane.  A bin's records are contiguous in HBM.
//   k_raster       persistent warps pull rows of coarse bins (any env) from one global counter.  The bin's records
//                  arrive in shared memory by bulk-async copy (cp.async.bulk + mbarrier, double-buffered per warp:
//                  the next chunk of 32 records lands while the current one is rasterised).  Visibility first: every
//                  lane owns one pixel of an 8x4 fine bin with its 4 MSAA samples (depth + winning prim) in
//                  registers.  Shading is DEFERRED: once per distinct winner of the pixel (1 for interior pixels,
//                  2 on an edge), fetched from the PrimRec by index — overdraw costs no shading.  Bins with one
//                  fully covering prim skip the depth pass.  Box resolve -> u8, rows packed with shuffles and
//                  stored as 32-bit words.
// The passes over finished frames (ResizeWrappers, MotionBlurWrapper, terminal-frame copies) are in dts_post.cu.
// Arithmetic follows the render spec of DESIGN.md (the CPU checker implements the same spec) bit for bit
// (compiled with -fmad=false; fmaf() is spelled out where the spec has one).
//
// Image targets (AuxTargets, the three rasterisers' last kernel parameter): besides obs, every pixel's eye-space depth
// (f32 [N][H][W], render spec item 9), label (the draw item + 1, i16, item 10) and lane marking (the texel class, u8,
// item 11).  Template parameter kAux, a set of kAuxDepth / kAuxLabels / kAuxMarks, is the images an instance writes,
// and launch_render picks it from the targets that are set (aux_set); without targets the launches are the plain
// kernels.  Labels and markings both take the label's winner among a pixel's winners.  A marking instance stores the
// depth where that target is set, a pointer test in these instances only (stores_depth), instead of a compiled depth +
// markings variant of each.  The instances are kAuxSets.
//
// HBM traffic per env-frame: obs store W*H*3 B (compulsory; + W*H*4 B of depth, W*H*2 B of labels and W*H B of markings where asked for) + PrimRec slab / BinRec lists / lattice table
// (tens of KB per env, written by k_geometry / k_bin and read once by k_raster) + texels (shared, L2-resident).
#include <algorithm>
#include <cstddef>
#include <cstdlib>
#include <iterator>
#include <type_traits>
#include <utility>
#include <vector>

#include "dts_camera.cuh"
#include "dts_kernels.h"

namespace dts {

// LUT remap, fused into the rasteriser (distortion.py:118 for the fisheye, UndistortWrapper's rectification alike:
// obs[y, x] = undistorted[rint(rmapy), rint(rmapx)]): the rasteriser renders each OUTPUT pixel at the source position
// the table names, so no undistorted frame is ever written.  Prims are binned against the source-pixel bounding boxes of
// the output bins.  All device pointers, built by renderer_set_lut.
// A pool of tables (dts_set_fisheye_luts, camera_rand) is held in one RemapTab: the tables' arrays concatenated, table
// t's src_xy / cbox / fbox / cell_start / home_start t strides in (every table has the camera's sizes), the CSR starts
// holding positions in the concatenated cell_bins / home_ent, ext_x / ext_y the largest over the tables, and
// table_of_env naming each env's table.  The kRemapPool instances offset the pointers by it (remap_of_env); the
// kRemapTable instances read the table as it is.
struct RemapTab {
  const int32_t* src_xy;   // [H][W]  sx | sy << 16 (int16 each); sx = -32768: source outside the image -> 0
  const short4* cbox;      // [cbins]    source bounding box (x0, y0, x1, y1) of a 32x8 coarse output bin; x1 < x0: empty
  const short4* fbox;      // [cbins][8] the same for each of its 8x4 fine bins
  // inverse index for binning small prims: the output coarse bins whose source box meets cell c of a 32x8-px grid laid
  // over the SOURCE image (CSR: cell_bins[cell_start[c] .. cell_start[c + 1]))
  const int32_t* cell_start;   // [cbins + 1]
  const uint16_t* cell_bins;
  // second inverse index for prims spanning many cells: every output bin listed ONCE, under the source cell holding the
  // top-left corner of its box (CSR); an entry is (x0 | y0 << 16, x1 | y1 << 16, bin, 0).  ext_x / ext_y: how many
  // cells a box reaches to the right of / below its home cell at most
  const int32_t* home_start;   // [cbins + 1]
  const int4* home_ent;
  int ext_x, ext_y;
  const uint16_t* table_of_env;   // [n_envs] a pool's table index of every env; null unless a pool of more than one table
  int count;                      // tables held
  const float2* fwd;              // [count][H][W] forward maps of the flow image (renderer_set_flow_maps), or null
};
// How the rasterisers map output pixels to source pixels: not at all, through one table, or through each env's table of
// a pool (the template value kRemap of k_bin and the rasterisers)
constexpr int kRemapNone = 0, kRemapTable = 1, kRemapPool = 2;

namespace {

#ifndef DTS_STATS
#define DTS_STATS 0         // 1: k_raster counts bins / prim visits / shading rounds into the diagnostic counters (tools/raster_stats.py)
#endif
#if DTS_STATS
#define DTS_COUNT(slot, n) do { if (lane == 0) atomicAdd(err + (slot), (n)); } while (0)
#else
#define DTS_COUNT(slot, n) do { } while (0)
#endif
// Occupancy: threads per CTA of the three rasterisers, and the resident CTAs per SM each kernel is compiled for
// (register budget 65536 / (threads * CTAs)).  Swept on H100 at c2: DESIGN.md §10.
constexpr int kThreads = 256;
constexpr int kRasterMinCtas = 3;   // k_raster
constexpr int kSoloMinCtas = 3;     // k_raster_solo
constexpr int kFlatMinCtas = 4;     // k_raster_flat
constexpr int kGeoWarps = 1;        // k_geometry: warps per CTA ...
constexpr int kGeoMinCtas = 32;     // ... and CTAs per SM
constexpr int kTileWarps = 4;       // k_tiles: warps (envs) per CTA ...
constexpr int kTileMinCtas = 4;     // ... and CTAs per SM (35 KB of shared memory each; 119 registers, no spills: at 6
                                    // or 5 CTAs, 80 or 96 registers, the lane phase spills)
constexpr int kWarps = kThreads / 32;
constexpr int kBinW = 8, kBinH = 4;   // fine bin = one warp's pixel block (one pixel per lane)
constexpr int kCFX = 4, kCFY = 2;     // coarse bin = 4 x 2 fine bins = 32 x 8 px: unit of binning and staging
constexpr int kCoarseW = kBinW * kCFX, kCoarseH = kBinH * kCFY;
constexpr int kStage = 32;        // prims staged per pass and warp
constexpr float kGuard = 4.0f;
constexpr int kSub = 64;          // sub-pixel units per pixel
constexpr int kTessTris = 98;     // spec tile mode 0: a road tile is its literal 7x7 quads, two triangles each
// Draw ids of one road tile: its triangles in tile mode 0; in tile mode 1 its quad, or the two triangles it splits into
__host__ __device__ constexpr int tile_draw_ids(bool tess) { return tess ? kTessTris : 2; }
// Draw items of a frame: the ground (item 0), the tiles, the placed objects, and last the agent's own mesh
__host__ __device__ constexpr int agent_item(int n_tiles, int n_objects) { return 1 + n_tiles + n_objects; }
// MSAA sample offsets in 1/64 px, (.375,.125)(.875,.375)(.125,.625)(.625,.875); constexpr so that the
// unrolled sample loops fold them into immediates
__host__ __device__ constexpr int sample_x(int s) { return s == 0 ? 24 : (s == 1 ? 56 : (s == 2 ? 8 : 40)); }
__host__ __device__ constexpr int sample_y(int s) { return s == 0 ? 8 : (s == 1 ? 24 : (s == 2 ? 40 : 56)); }

struct Vtx { float cx, cy, cz, cw, r, g, b, u, v; };

struct __align__(16) PrimRec {   // 128 B in the env's slab, words grouped for 128-bit loads
  int32_t X0, Y0, X1, Y1;        // w0  snapped vertices in cyclic order, orientation normalised (area > 0)
  int32_t X2, Y2, X3, Y3;        // w1  vertex 3: 4th corner of a quad, else a copy of vertex 0
  float z0, zx, zy;              // w2  depth plane anchored at vertex 0 (f0, d/dx, d/dy per pixel)
  int32_t id;                    //     draw id (GL_LESS ties go to the earlier draw)
  float q0, qx, qy, u0;          // w3  q = 1/w, then u*q, v*q, r*q, g*q, b*q
  float ux, uy, v0, vx;          // w4
  float vy;                      // w5
  int32_t ltq;                   //     (lattice slot + 1) | (texture index + 1) << 16 | quad << 24
  uint32_t tex;                  //     DTexture::info of the prim's texture (pool offset >> 8 | log2 w << 24 | log2 h << 28)
  float r0;
  float rx, ry, g0, gx;          // w6
  float gy, b0, bx, by;          // w7
};
static_assert(sizeof(PrimRec) == 128, "PrimRec must be 128 bytes");
static_assert(offsetof(PrimRec, q0) == 48 && offsetof(PrimRec, vy) == 80 && offsetof(PrimRec, rx) == 96, "PrimRec word groups");

struct __align__(16) BinRec {    // 80 B per (prim, coarse bin) pair: what visibility needs, re-based to the bin corner
  int32_t E0[4], A[4], B[4];     // E_k(x,y) = E0_k + A_k*x + B_k*y, x,y in 1/64 px from the bin corner (triangles: E_3 = 0)
  float z0, zx, zy;              // depth plane
  int32_t id;                    // draw id
  int32_t x0, y0;                // anchor vertex relative to the bin corner (sub-pixels)
  uint32_t prim_flags;           // prim index | per fine bin f of the coarse bin: bit 16+f = may touch, bit 24+f = every sample inside
  int32_t kind;                  // kKind* bits
};
static_assert(sizeof(BinRec) == 80, "BinRec layout");
// BinRec::kind, written by k_bin (build_binrec) and read by the rasterisers
constexpr int kKindQuad = 1;     // 4 edges
constexpr int kKindGround = 2;   // the ground quad (draw id < 2)
constexpr int kKindTiny = 4;     // tiny triangle: its pixel box inside the coarse bin is at most 4x4 and sits in the unused
                                 // 4th-edge slots: E0[3] = x0 | y0 << 16, A[3] = x1 | y1 << 16 (pixels from the bin corner, inclusive)
constexpr int kKindFlat = 8;     // road tile of tile mode 1: lies in the plane y = 0
constexpr unsigned kNoPrim = 0xffffu;   // sample not covered by any prim: clear colour

struct Xform { float MV[12], N[9]; };

struct __align__(16) GeoWarp {    // per warp of k_geometry, shared memory
  int32_t unlit, pad_[3];        // segment=True: GL_LIGHTING off, the vertex colour is the material colour (S:1730-1733)
  RenderEp ep;
  double V[12];
  float P00, P11, P22, P23;
  Xform x;                       // model-view / normal matrix of the warp's draw item (warp-uniform)
  Vtx corners[4];
  Vtx poly[2][12];               // ping-pong polygon of the warp-parallel clipper
};
using Shared = GeoWarp;           // shade_vertex reads ep and P from it

// MV = V * T(t) * S(sc) * Ry(c,s), N = rot(V) * Ry / sc — float64 then rounded (spec).  Entry (r, k) of the 3x4
// matrix, and of N for the rotation part (k < 3).
__device__ __forceinline__ void model_view_entry(const double* V, double tx, double ty, double tz, double sc, double c,
                                                 double s, int r, int k, Xform& x) {
  if (k < 3) {
    const double R0 = k == 0 ? c : (k == 1 ? 0.0 : s), R1 = k == 1 ? 1.0 : 0.0, R2 = k == 0 ? -s : (k == 1 ? 0.0 : c);
    const double a = V[4 * r + 0] * R0 + V[4 * r + 1] * R1 + V[4 * r + 2] * R2;
    x.MV[4 * r + k] = (float)(a * sc);
    x.N[3 * r + k] = (float)(sc == 1.0 ? a : a / sc);   // x / 1.0 == x exactly
  } else {
    x.MV[4 * r + 3] = (float)(V[4 * r + 0] * tx + V[4 * r + 1] * ty + V[4 * r + 2] * tz + V[4 * r + 3]);
  }
}
// Warp form: lanes 0..11 each produce one entry into the warp's shared Xform.
__device__ __forceinline__ void model_view(const double* V, double tx, double ty, double tz, double sc, double c,
                                           double s, Xform& x, int lane) {
  __syncwarp();
  if (lane < 12) model_view_entry(V, tx, ty, tz, sc, c, s, lane >> 2, lane & 3, x);
  __syncwarp();
}

// Of the geometry pass's big device functions, shade_vertex and the clipper are inlined and setup_and_emit is not: inlined,
// setup_and_emit alone is a dozen copies of a large function, more SASS than the instruction cache holds.

// fixed-function transform & lighting of one vertex (float32, operation order = spec)
__device__ __forceinline__ Vtx shade_vertex(const Xform& x, const Shared& sh, float px, float py, float pz, float nx,
                                            float ny, float nz, float cr, float cg, float cb, float u, float v) {
  float e[3], ne[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
    float t = x.MV[4 * r] * px;
    t = t + x.MV[4 * r + 1] * py;
    t = t + x.MV[4 * r + 2] * pz;
    e[r] = t + x.MV[4 * r + 3];
    float q = x.N[3 * r] * nx;
    q = q + x.N[3 * r + 1] * ny;
    ne[r] = q + x.N[3 * r + 2] * nz;
  }
  const float* lp = sh.ep.light_eye;
  float lx, ly, lz;
  if (lp[3] == 0.0f) { lx = lp[0]; ly = lp[1]; lz = lp[2]; }
  else { lx = lp[0] - e[0]; ly = lp[1] - e[1]; lz = lp[2] - e[2]; }
  float len = lx * lx;
  len = len + ly * ly;
  len = len + lz * lz;
  len = sqrtf(len);
  float ndl = 0.0f;
  if (len > 0.0f) {
    lx = lx / len; ly = ly / len; lz = lz / len;
    ndl = ne[0] * lx;
    ndl = ndl + ne[1] * ly;
    ndl = ndl + ne[2] * lz;
    if (!(ndl > 0.0f)) ndl = 0.0f;
  }
  Vtx o;
  const float col[3] = {cr, cg, cb};
  float lit[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    float s = 0.3f + sh.ep.ambient[k];
    s = s + ndl * sh.ep.diffuse[k];
    const float c = sh.unlit ? col[k] : col[k] * s;
    lit[k] = c < 0.0f ? 0.0f : (c > 1.0f ? 1.0f : c);
  }
  o.r = lit[0]; o.g = lit[1]; o.b = lit[2];
  o.u = u; o.v = v;
  o.cx = sh.P00 * e[0];
  o.cy = sh.P11 * e[1];
  o.cz = sh.P22 * e[2] + sh.P23;
  o.cw = -e[2];
  return o;
}

// Road tile S:1852-1884: its lattice vertex (a, b) of the 8x8 grid (a: u index along x, b: v index along z), lit white
__device__ __forceinline__ Vtx tile_vertex(const Xform& x, const Shared& sh, double ts, int a, int b) {
  const float lx = (float)(-ts / 2 + ((double)a / 7.0) * ts), lz = (float)(-ts / 2 + ((double)b / 7.0) * ts);
  return shade_vertex(x, sh, lx, 0.0f, lz, 0.f, 1.f, 0.f, 1.f, 1.f, 1.f, (float)((double)a / 7.0), (float)(1.0 - (double)b / 7.0));
}
// ... and its placement: glTranslatef((i + 0.5) * TS, 0, (j + 0.5) * TS) S:1870 (GLfloat arguments), glRotatef(angle*90+180) S:1873
struct TilePose { double tx, tz, cs, sn; };
__device__ __forceinline__ TilePose tile_pose(const DMap& m, int ti, int tj) {
  const int quarter = (m.tile_angle[tj * m.grid_w + ti] + 2) & 3;
  const double ts = m.tile_size;
  return TilePose{(double)(float)((ti + 0.5) * ts), (double)(float)((tj + 0.5) * ts),
                  quarter == 0 ? 1.0 : (quarter == 2 ? -1.0 : 0.0), quarter == 1 ? 1.0 : (quarter == 3 ? -1.0 : 0.0)};
}

__device__ __forceinline__ float plane_dist(const Vtx& a, int pl) {
  switch (pl) {
    case 0: return a.cz + a.cw;
    case 1: return a.cw - a.cz;
    case 2: return a.cx + kGuard * a.cw;
    case 3: return kGuard * a.cw - a.cx;
    case 4: return a.cy + kGuard * a.cw;
    default: return kGuard * a.cw - a.cy;
  }
}

// 0 = visible without clipping, 1 = needs the clipper, 2 = invisible (outside one true-frustum plane)
__device__ __forceinline__ int classify(const Vtx& a, const Vtx& b, const Vtx& c) {
  const Vtx* v[3] = {&a, &b, &c};
  int out[6] = {0, 0, 0, 0, 0, 0}, need = 0;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float x = v[k]->cx, y = v[k]->cy, z = v[k]->cz, w = v[k]->cw;
    out[0] += !(z + w >= 0.0f); out[1] += !(w - z >= 0.0f);
    out[2] += x < -w; out[3] += x > w; out[4] += y < -w; out[5] += y > w;
    need |= !(x + kGuard * w >= 0.0f) | !(kGuard * w - x >= 0.0f) | !(y + kGuard * w >= 0.0f) |
            !(kGuard * w - y >= 0.0f);
  }
  need |= out[0] | out[1];
#pragma unroll
  for (int p = 0; p < 6; p++) if (out[p] == 3) return 2;
  return need ? 1 : 0;
}

struct EmitCtx {
  const DTexture* textures;
  GeoWarp* gw;
  FrameCtx* ctx;
  PrimRec* prims;          // this env's slab
  int max_prims, W, H;
};

// screen mapping + triangle setup (spec steps 5-7) and append to the slab
// With `d` the prim is the QUAD a,b,c,d (spec tile mode 1: an unclipped road tile): planes of triangle (a,b,c),
// coverage by four edges.  Returns false — nothing emitted — if the snapped quad is not strictly convex; the
// caller then draws the two triangles (a,b,c)(a,c,d) instead.
__device__ __noinline__ bool setup_and_emit(const EmitCtx& ec, const Vtx& a, const Vtx& b, const Vtx& c, int id,
                                            int tex, int lat, const Vtx* d = nullptr) {
  const Vtx* vs[3] = {&a, &b, &c};
  int X[3], Y[3];
  float zw[3], q[3];
  const float Wf = (float)ec.W, Hf = (float)ec.H;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float iw = 1.0f / vs[k]->cw;
    const float nx = vs[k]->cx * iw, ny = vs[k]->cy * iw, nz = vs[k]->cz * iw;
    const float sx = (nx * 0.5f + 0.5f) * Wf;
    const float sy = (0.5f - ny * 0.5f) * Hf;
    X[k] = (int)rintf(sx * 64.0f);
    Y[k] = (int)rintf(sy * 64.0f);
    zw[k] = nz * 0.5f + 0.5f;
    q[k] = iw;
  }
  const long long area2 = (long long)(X[1] - X[0]) * (Y[2] - Y[0]) - (long long)(X[2] - X[0]) * (Y[1] - Y[0]);
  if (area2 == 0) return false;
  const int i1 = area2 < 0 ? 2 : 1, i2 = area2 < 0 ? 1 : 2;
  const int x0 = X[0], y0 = Y[0], x1 = X[i1], y1 = Y[i1], x2 = X[i2], y2 = Y[i2];
  int minx = min(x0, min(x1, x2)), maxx = max(x0, max(x1, x2));
  int miny = min(y0, min(y1, y2)), maxy = max(y0, max(y1, y2));
  int qx[4] = {x0, x1, x2, 0}, qy[4] = {y0, y1, y2, 0};   // quad: cyclic order with positive orientation
  if (d) {
    const float iw = 1.0f / d->cw;
    const float sx = ((d->cx * iw) * 0.5f + 0.5f) * Wf, sy = (0.5f - (d->cy * iw) * 0.5f) * Hf;
    const int X3 = (int)rintf(sx * 64.0f), Y3 = (int)rintf(sy * 64.0f);
    if (area2 > 0) { qx[1] = X[1]; qy[1] = Y[1]; qx[2] = X[2]; qy[2] = Y[2]; qx[3] = X3; qy[3] = Y3; }       // a b c d
    else { qx[1] = X3; qy[1] = Y3; qx[2] = X[2]; qy[2] = Y[2]; qx[3] = X[1]; qy[3] = Y[1]; }                 // a d c b
#pragma unroll
    for (int k = 0; k < 4; k++) {   // strictly convex: every corner turns the same (positive) way
      const int k1 = (k + 1) & 3, k2 = (k + 2) & 3;
      const long long cr = (long long)(qx[k1] - qx[k]) * (qy[k2] - qy[k1]) - (long long)(qx[k2] - qx[k1]) * (qy[k1] - qy[k]);
      if (cr <= 0) return false;
    }
    minx = min(minx, X3); maxx = max(maxx, X3); miny = min(miny, Y3); maxy = max(maxy, Y3);
  }
  const int px0 = max(minx >> 6, 0), px1 = min(maxx >> 6, ec.W - 1);
  const int py0 = max(miny >> 6, 0), py1 = min(maxy >> 6, ec.H - 1);
  if (px0 > px1 || py0 > py1) return true;   // off screen: emitted nothing, and nothing is what it covers
  if (!d && (maxx >> 6) - (minx >> 6) < 3 && (maxy >> 6) - (miny >> 6) < 3) {   // (the unclamped box: everything below stays small)
    // A small triangle that covers NO sample position draws nothing — half the triangles of a distant mesh at
    // 160x120 — so it needs no record, no bin pair and no visit by the rasteriser.  Same integer edge functions and
    // fill rule as the coverage test proper (build_binrec / k_raster); coordinates relative to vertex 0 stay in int32.
    const int ex[3] = {x1 - x0, x2 - x1, x0 - x2}, ey[3] = {y1 - y0, y2 - y1, y0 - y2};
    const int ax[3] = {0, x1 - x0, x2 - x0}, ay[3] = {0, y1 - y0, y2 - y0};
    int e00[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const int bias = (ey[k] > 0 || (ey[k] == 0 && ex[k] < 0)) ? 0 : 1;
      e00[k] = ex[k] * (py0 * kSub - y0 - ay[k]) - ey[k] * (px0 * kSub - x0 - ax[k]) - bias;
    }
    bool any = false;
    for (int py = 0; py <= py1 - py0; py++)
      for (int px = 0; px <= px1 - px0; px++) {
#pragma unroll
        for (int s = 0; s < 4; s++) {
          const int sx = px * kSub + sample_x(s), sy = py * kSub + sample_y(s);
          const int e0 = e00[0] + ex[0] * sy - ey[0] * sx, e1 = e00[1] + ex[1] * sy - ey[1] * sx, e2 = e00[2] + ex[2] * sy - ey[2] * sx;
          any |= (e0 | e1 | e2) >= 0;
        }
      }
    if (!any) return true;
  }
  PrimRec r;
  r.X0 = x0; r.Y0 = y0; r.X1 = x1; r.Y1 = y1; r.X2 = x2; r.Y2 = y2; r.X3 = x0; r.Y3 = y0;
  const float dx1 = (float)(x1 - x0) * 0.015625f, dy1 = (float)(y1 - y0) * 0.015625f;
  const float dx2 = (float)(x2 - x0) * 0.015625f, dy2 = (float)(y2 - y0) * 0.015625f;
  const float areaf = dx1 * dy2 - dx2 * dy1;
  const float ia = 1.0f / areaf;
  const Vtx* p0 = vs[0]; const Vtx* p1 = vs[i1]; const Vtx* p2 = vs[i2];
  const float q0 = q[0], q1 = q[i1], q2 = q[i2];
  const float v0[7] = {zw[0], q0, p0->u * q0, p0->v * q0, p0->r * q0, p0->g * q0, p0->b * q0};
  const float v1[7] = {zw[i1], q1, p1->u * q1, p1->v * q1, p1->r * q1, p1->g * q1, p1->b * q1};
  const float v2[7] = {zw[i2], q2, p2->u * q2, p2->v * q2, p2->r * q2, p2->g * q2, p2->b * q2};
  float f0[7], fx[7], fy[7];
#pragma unroll
  for (int at = 0; at < 7; at++) {
    const float d1 = v1[at] - v0[at], d2 = v2[at] - v0[at];
    f0[at] = v0[at];
    fx[at] = (d1 * dy2 - d2 * dy1) * ia;
    fy[at] = (d2 * dx1 - d1 * dx2) * ia;
  }
  r.z0 = f0[0]; r.zx = fx[0]; r.zy = fy[0];
  r.q0 = f0[1]; r.qx = fx[1]; r.qy = fy[1];
  r.u0 = f0[2]; r.ux = fx[2]; r.uy = fy[2];
  r.v0 = f0[3]; r.vx = fx[3]; r.vy = fy[3];
  r.r0 = f0[4]; r.rx = fx[4]; r.ry = fy[4];
  r.g0 = f0[5]; r.gx = fx[5]; r.gy = fy[5];
  r.b0 = f0[6]; r.bx = fx[6]; r.by = fy[6];
  r.id = id;
  r.ltq = (lat + 1) | ((tex + 1) << 16);
  r.tex = tex >= 0 ? ec.textures[tex].info : 0u;
  if (d) {   // vertices in cyclic order; planes stay those of triangle (a,b,c) anchored at a
    r.ltq |= 1 << 24;
    r.X1 = qx[1]; r.Y1 = qy[1]; r.X2 = qx[2]; r.Y2 = qy[2]; r.X3 = qx[3]; r.Y3 = qy[3];
  }
  // the slab slot: one atomic for all the lanes emitting together (a warp draws one env at a time, so they share ctx)
  const unsigned act = __activemask();
  const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
  int slot = 0;
  if (lane == leader) slot = atomicAdd(&ec.ctx->n_prims, __popc(act));
  slot = __shfl_sync(act, slot, leader) + __popc(act & ((1u << lane) - 1u));
  if (slot >= ec.max_prims) { ec.ctx->overflow = 1; return true; }
  const int4* src = reinterpret_cast<const int4*>(&r);
  int4* dst = reinterpret_cast<int4*>(ec.prims + slot);
#pragma unroll
  for (int k = 0; k < 8; k++) dst[k] = src[k];
  return true;
}

__device__ __forceinline__ Vtx clip_lerp(const Vtx& in, const Vtx& out, float din, float dout) {
  const float t = din / (din - dout);
  Vtx o;
  const float* a = reinterpret_cast<const float*>(&in);
  const float* b = reinterpret_cast<const float*>(&out);
  float* c = reinterpret_cast<float*>(&o);
#pragma unroll
  for (int k = 0; k < 9; k++) { const float d = b[k] - a[k]; c[k] = a[k] + t * d; }
  return o;
}

// Sutherland-Hodgman against near, far and the guard band (spec step 4), then a triangle fan — executed by the
// WHOLE warp for one triangle: lane k owns polygon vertex k, neighbours' plane distances come by shuffle, output
// slots by ballot prefix sums, so a plane costs a few dozen instructions instead of a serial loop over vertices.
// Same arithmetic, same vertex order (hence the same fan) as the serial formulation of the spec.
__device__ __forceinline__ void clip_and_emit_warp(const EmitCtx& ec, const Vtx& a, const Vtx& b, const Vtx& c, int id,
                                                   int tex, int lat, int lane) {
  for (int p2 = 0; p2 < 6; p2++) {   // the spec's trivial reject looks at the ORIGINAL triangle, guard planes
    const int cnt = !(plane_dist(a, p2) >= 0.0f) + !(plane_dist(b, p2) >= 0.0f) + !(plane_dist(c, p2) >= 0.0f);
    if (cnt == 3) return;
  }
  GeoWarp& g = *ec.gw;
  __syncwarp();
  if (lane == 0) { g.poly[0][0] = a; g.poly[0][1] = b; g.poly[0][2] = c; }
  __syncwarp();
  int n = 3, cur = 0;
  for (int pl = 0; pl < 6; pl++) {
    const Vtx* P = g.poly[cur];
    const float dk = lane < n ? plane_dist(P[lane], pl) : 0.0f;
    const bool in1 = dk >= 0.0f;
    const unsigned valid = (1u << n) - 1u;
    const unsigned out_mask = __ballot_sync(0xffffffffu, lane < n && !in1);
    if (!out_mask) continue;
    const int k2 = (lane + 1 == n) ? 0 : lane + 1;
    const float dn = __shfl_sync(0xffffffffu, dk, k2 & 31);
    const bool in2 = dn >= 0.0f;
    const bool cross = lane < n && (in1 != in2);
    const unsigned keep_mask = __ballot_sync(0xffffffffu, lane < n && in1) & valid;
    const unsigned cross_mask = __ballot_sync(0xffffffffu, cross) & valid;
    const unsigned below = (1u << lane) - 1u;
    int pos = __popc(keep_mask & below) + __popc(cross_mask & below);
    Vtx* T = g.poly[cur ^ 1];
    if (lane < n) {
      if (in1) T[pos++] = P[lane];
      if (in1 && !in2) T[pos] = clip_lerp(P[lane], P[k2], dk, dn);
      else if (!in1 && in2) T[pos] = clip_lerp(P[k2], P[lane], dn, dk);
    }
    n = __popc(keep_mask) + __popc(cross_mask);
    cur ^= 1;
    __syncwarp();
    if (n < 3) return;
  }
  const Vtx* P = g.poly[cur];
  if (lane + 2 < n) setup_and_emit(ec, P[0], P[lane + 1], P[lane + 2], id, tex, lat);
  __syncwarp();
}

// one warp-uniform triangle (ground, analytic tile): classify once, lane 0 emits or the warp clips
__device__ __forceinline__ void process_triangle_uniform(const EmitCtx& ec, const Vtx& a, const Vtx& b, const Vtx& c,
                                                         int id, int tex, int lat, int lane) {
  const int cls = classify(a, b, c);
  if (cls == 2) return;
  if (cls == 0) { if (lane == 0) setup_and_emit(ec, a, b, c, id, tex, lat); }
  else clip_and_emit_warp(ec, a, b, c, id, tex, lat, lane);
}

// one triangle per lane (meshes, tessellated tiles): unclipped ones are emitted in place, the rare ones that
// need clipping are broadcast lane by lane to the warp-parallel clipper
__device__ __forceinline__ void process_triangle_lanes(const EmitCtx& ec, bool have, const Vtx& a, const Vtx& b,
                                                       const Vtx& c, int id, int tex, int lat, int lane) {
  const int cls = have ? classify(a, b, c) : 2;
  if (cls == 0) setup_and_emit(ec, a, b, c, id, tex, lat);
  unsigned need = __ballot_sync(0xffffffffu, cls == 1);
  while (need) {
    const int src = __ffs(need) - 1;
    need &= need - 1;
    Vtx va, vb, vc;
    const float* fa = reinterpret_cast<const float*>(&a);
    const float* fb = reinterpret_cast<const float*>(&b);
    const float* fc = reinterpret_cast<const float*>(&c);
#pragma unroll
    for (int k = 0; k < 9; k++) {
      reinterpret_cast<float*>(&va)[k] = __shfl_sync(0xffffffffu, fa[k], src);
      reinterpret_cast<float*>(&vb)[k] = __shfl_sync(0xffffffffu, fb[k], src);
      reinterpret_cast<float*>(&vc)[k] = __shfl_sync(0xffffffffu, fc[k], src);
    }
    const int sid = __shfl_sync(0xffffffffu, id, src), stex = __shfl_sync(0xffffffffu, tex, src);
    clip_and_emit_warp(ec, va, vb, vc, sid, stex, lat, lane);
  }
}

// conservative prim / box overlap: false only if one edge has every sample position of the box
// [x_lo, x_hi] x [y_lo, y_hi] (sub-pixels) on its outside
__device__ __forceinline__ bool box_overlaps(const int qx[4], const int qy[4], int n, int x_lo, int x_hi, int y_lo, int y_hi) {
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (k >= n) break;
    const int k1 = (k + 1) & 3;   // a triangle's vertex 3 aliases vertex 0
    const int dx = qx[k1] - qx[k], dy = qy[k1] - qy[k];
    // E(x,y) = dx*(y-ay) - dy*(x-ax); maximise over the box
    const int xs = (-dy > 0) ? x_hi : x_lo;
    const int ys = (dx > 0) ? y_hi : y_lo;
    const long long e = (long long)dx * (ys - qy[k]) - (long long)dy * (xs - qx[k]);
    if (e < 0) return false;
  }
  return true;
}
__device__ __forceinline__ bool bin_overlaps(const int qx[4], const int qy[4], int n, int ox, int oy) {
  return box_overlaps(qx, qy, n, ox + 8, ox + (kCoarseW - 1) * kSub + 56, oy + 8, oy + (kCoarseH - 1) * kSub + 56);
}

// The visibility record of prim `p` for the coarse bin whose corner is (ox, oy) sub-pixels: edge functions re-based
// to the corner (exact in 64 bits, then int32: inside the coarse bin |A*x + B*y| < 2^30), exact reject /
// trivial-accept bits for each of the bin's 8 fine bins, depth plane, draw id.
// With `fb` (LUT remap) the bin's pixels are wherever the LUT sends its output pixels: (ox, oy) is the corner of
// their source bounding box and fb[f] the source box of fine bin f; the bits then speak about every pixel of that box.
// Returns the fine bins every sample of which the prim covers (bits 0-7) | kRecGround | kRecFlatOk.
constexpr unsigned kRecGround = 0x100u;   // the ground quad
constexpr unsigned kRecFlatOk = 0x200u;   // a flat road tile or the ground quad, and not drawn by the tiny-triangle path
__device__ __forceinline__ unsigned build_binrec(const PrimRec* __restrict__ pr, int p, int ox, int oy, BinRec* __restrict__ out,
                                                 const short4* __restrict__ fb = nullptr) {
  const int4 w0 = __ldg(reinterpret_cast<const int4*>(pr));
  const int4 w1 = __ldg(reinterpret_cast<const int4*>(pr) + 1);
  const float4 w2 = __ldg(reinterpret_cast<const float4*>(pr) + 2);
  const int ltq = __ldg(&pr->ltq);
  const int quad = (ltq >> 24) & 1;
  const int flat = (ltq & 0xffff) ? kKindFlat : 0;   // a road tile of tile mode 1 (it carries a lattice)
  const int qx[4] = {w0.x, w0.z, w1.x, w1.z}, qy[4] = {w0.y, w0.w, w1.y, w1.w};
  const int nv = quad ? 4 : 3;
  unsigned live = 0xffu, inside = 0xffu;
  int E0[4] = {0, 0, 0, 0}, A[4] = {0, 0, 0, 0}, B[4] = {0, 0, 0, 0};   // triangles: a fourth edge that every sample passes
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (k >= nv) break;
    const int ka = k, kb = (k + 1) & 3;   // edge k: vertex k -> k+1 (a triangle's vertex 3 is a copy of vertex 0)
    const int dx = qx[kb] - qx[ka], dy = qy[kb] - qy[ka];
    const int bias = (dy > 0 || (dy == 0 && dx < 0)) ? 0 : 1;
    long long e0 = (long long)dx * (oy - qy[ka]) - (long long)dy * (ox - qx[ka]) - bias;
    if (e0 < -(1LL << 30)) live = 0;          // negative for every sample of the coarse bin
    if (e0 > (1LL << 30)) e0 = (1LL << 30);   // positive for every sample: keep the sign, stay in int32
    if (e0 < -(1LL << 30)) e0 = -(1LL << 30);
    const int a = -dy, b = dx, e = (int)e0;
    E0[k] = e; A[k] = a; B[k] = b;
    if (fb) {
      // (remap: the fine bins' source boxes are handled after the edge loop, one box load per fine bin)
    } else {
      // extremes of A*x + B*y over one fine bin's sample span x in [8, 504], y in [8, 248]
      const int hi = (a > 0 ? a * 504 : a * 8) + (b > 0 ? b * 248 : b * 8);
      const int lo = (a > 0 ? a * 8 : a * 504) + (b > 0 ? b * 8 : b * 248);
#pragma unroll
      for (int f = 0; f < 8; f++) {
        const int ef = e + a * ((f & 3) * kBinW * kSub) + b * ((f >> 2) * kBinH * kSub);
        if (ef + hi < 0) live &= ~(1u << f);
        if (ef + lo < 0) inside &= ~(1u << f);
      }
    }
  }
  if (fb) {
#pragma unroll 1
    for (int f = 0; f < 8; f++) {
      const short4 q = fb[f];
      if (q.z < q.x) { live &= ~(1u << f); continue; }   // no pixel of this fine bin has a source inside the image
      const int X0 = q.x * kSub - ox + 8, X1 = q.z * kSub - ox + 56, Y0 = q.y * kSub - oy + 8, Y1 = q.w * kSub - oy + 56;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        if (k >= nv) break;
        const int a = A[k], b = B[k], e = E0[k];
        const int hi = (a > 0 ? a * X1 : a * X0) + (b > 0 ? b * Y1 : b * Y0);
        const int lo = (a > 0 ? a * X0 : a * X1) + (b > 0 ? b * Y0 : b * Y1);
        if (e + hi < 0) live &= ~(1u << f);
        if (e + lo < 0) inside &= ~(1u << f);
      }
    }
  }
  int tiny = 0;
  if (!fb && !quad && live) {
    // small triangles (a 6 cm duckie is 148 triangles in a dozen pixels) are rasterised one per LANE in k_raster instead
    // of one per warp: they carry their pixel box
    const int minx = min(qx[0], min(qx[1], qx[2])) - ox, maxx = max(qx[0], max(qx[1], qx[2])) - ox;
    const int miny = min(qy[0], min(qy[1], qy[2])) - oy, maxy = max(qy[0], max(qy[1], qy[2])) - oy;
    const int x0 = max(minx >> 6, 0), x1 = min(maxx >> 6, kCoarseW - 1), y0 = max(miny >> 6, 0), y1 = min(maxy >> 6, kCoarseH - 1);
    if (x1 - x0 < 4 && y1 - y0 < 4 && x1 >= x0 && y1 >= y0) {
      tiny = kKindTiny;
      E0[3] = x0 | (y0 << 16); A[3] = x1 | (y1 << 16);
    }
  }
  const int id = __float_as_int(w2.w);
  int4* o = reinterpret_cast<int4*>(out);
  o[0] = make_int4(E0[0], E0[1], E0[2], E0[3]);
  o[1] = make_int4(A[0], A[1], A[2], A[3]);
  o[2] = make_int4(B[0], B[1], B[2], B[3]);
  o[3] = make_int4(__float_as_int(w2.x), __float_as_int(w2.y), __float_as_int(w2.z), id);
  o[4] = make_int4(qx[0] - ox, qy[0] - oy, (int)((unsigned)p | (live << 16) | ((inside & live) << 24)),
                   (quad ? kKindQuad : 0) | (id < 2 ? kKindGround : 0) | tiny | flat);
  return (inside & live) | (id < 2 ? kRecGround : 0u) | ((flat || id < 2) && !tiny ? kRecFlatOk : 0u);
}

// Fragment colour of prim `w` of the env's slab at the pixel whose centre is (pxa + 32, pya + 32) sub-pixels (spec steps
// 5-6 and 8): perspective-correct u,v (+ rgb for meshes / ground), analytic lattice lighting for road tiles,
// bilinear REPEAT texel, MODULATE.  Deferred shading: each lane may shade a different prim.  Split in two so that a
// coarse bin lying inside ONE prim fetches the prim's planes once for its 256 pixels.
// `qq_out` (depth target, render spec item 9) receives the prim's clamped 1/w at the pixel centre: the very value the
// perspective divide uses.  `cls_out` (marking target, render spec item 11) receives the class of the texel
// (floor(u * tw) mod tw, floor(v * th) mod th) of the prim's texture from `cls_pool` (the map's texel classes, at the
// texture's texel offset), u, v those the texel fetch uses; 0 for an untextured prim.
struct ShadeIn {
  const PrimRec* pr;
  int x0, y0;
  float q0, qx, qy, u0, ux, uy, v0, vx, vy, r0;
  int ltq;
  unsigned tex;
};
__device__ __forceinline__ ShadeIn load_shade(const PrimRec* __restrict__ prims, unsigned w) {
  const PrimRec* pr = prims + w;
  const int2 xy0 = __ldg(reinterpret_cast<const int2*>(pr));
  const float4 w3 = __ldg(reinterpret_cast<const float4*>(pr) + 3);   // q0 qx qy u0
  const float4 w4 = __ldg(reinterpret_cast<const float4*>(pr) + 4);   // ux uy v0 vx
  const float4 w5 = __ldg(reinterpret_cast<const float4*>(pr) + 5);   // vy ltq tex r0
  ShadeIn si;
  si.pr = pr; si.x0 = xy0.x; si.y0 = xy0.y;
  si.q0 = w3.x; si.qx = w3.y; si.qy = w3.z; si.u0 = w3.w;
  si.ux = w4.x; si.uy = w4.y; si.v0 = w4.z; si.vx = w4.w;
  si.vy = w5.x; si.ltq = __float_as_int(w5.y); si.tex = __float_as_uint(w5.z); si.r0 = w5.w;
  return si;
}
__device__ __forceinline__ void shade_eval(const ShadeIn& si, const uint8_t* __restrict__ tex_pool, const float4* __restrict__ lat_tab,
                                           int pxa, int pya, float c3[3], float* qq_out = nullptr,
                                           const uint8_t* __restrict__ cls_pool = nullptr, int* cls_out = nullptr) {
  const float cdx = (float)(pxa + 32 - si.x0) * 0.015625f, cdy = (float)(pya + 32 - si.y0) * 0.015625f;
  float qq = fmaf(si.qy, cdy, fmaf(si.qx, cdx, si.q0));
  if (!(qq > 1e-20f)) qq = 1e-20f;
  if (qq_out) *qq_out = qq;
  const float rq = 1.0f / qq;
  const float u = fmaf(si.uy, cdy, fmaf(si.ux, cdx, si.u0)) * rq;
  const float v = fmaf(si.vy, cdy, fmaf(si.vx, cdx, si.v0)) * rq;
  const int ltq = si.ltq;
  const int lat = (ltq & 0xffff) - 1;
  if (lat >= 0) {
    // analytic road tile: Gouraud interpolant of the lit 8x8 lattice at (u,v)
    const float fa_ = u * 7.0f, fb_ = (1.0f - v) * 7.0f;
    int ia = __float2int_rd(fa_), ib = __float2int_rd(fb_);   // (int)floorf(.)
    ia = ia < 0 ? 0 : (ia > 6 ? 6 : ia);
    ib = ib < 0 ? 0 : (ib > 6 ? 6 : ib);
    const float fa = fa_ - (float)ia, fb = fb_ - (float)ib;
    const float4* L = lat_tab + lat * 64 + ia * 8 + ib;
    // the cell's two triangles share c00 and c11; pick the third corner and the order of the two weights
    // instead of branching (same arithmetic, three loads instead of four)
    const bool lower = fb <= fa;
    const float4 c00 = L[0], c11 = L[9], cm = L[lower ? 8 : 1];
    const float t1 = lower ? fa : fb, t2 = lower ? fb : fa;
    c3[0] = fmaf(t2, c11.x - cm.x, fmaf(t1, cm.x - c00.x, c00.x));
    c3[1] = fmaf(t2, c11.y - cm.y, fmaf(t1, cm.y - c00.y, c00.y));
    c3[2] = fmaf(t2, c11.z - cm.z, fmaf(t1, cm.z - c00.z, c00.z));
  } else {
    const float4 w6 = __ldg(reinterpret_cast<const float4*>(si.pr) + 6);    // rx ry g0 gx
    const float4 w7 = __ldg(reinterpret_cast<const float4*>(si.pr) + 7);    // gy b0 bx by
    c3[0] = fmaf(w6.y, cdy, fmaf(w6.x, cdx, si.r0)) * rq;
    c3[1] = fmaf(w7.x, cdy, fmaf(w6.w, cdx, w6.z)) * rq;
    c3[2] = fmaf(w7.w, cdy, fmaf(w7.z, cdx, w7.y)) * rq;
  }
  if (cls_out) *cls_out = 0;
  if (ltq & 0x00ff0000) {
    const unsigned ti = si.tex;
    const int lw = (ti >> 24) & 15, lh = ti >> 28;
    const int tw = 1 << lw, th = 1 << lh;
    const float twf = __int_as_float((127 + lw) << 23), thf = __int_as_float((127 + lh) << 23);   // (float)tw: a power of two
    const float tx = u * twf - 0.5f, ty = v * thf - 0.5f;
    const int txi = __float2int_rd(tx), tyi = __float2int_rd(ty);   // floorf(.) as the int the wrap needs; exact back in float
    const float ffx = tx - (float)txi, ffy = ty - (float)tyi;
    // texel indices as unsigned 32-bit values (below 2^30): each address is one wide multiply-add onto the texture base
    const unsigned ti0 = (unsigned)txi & (tw - 1), ti1 = (ti0 + 1) & (tw - 1);
    const unsigned tj0 = (unsigned)tyi & (th - 1), tj1 = (tj0 + 1) & (th - 1);
    const unsigned r0 = tj0 << lw, r1 = tj1 << lw;
    const uchar4* tp = reinterpret_cast<const uchar4*>(tex_pool + ((size_t)(ti & 0xffffffu) << 8));
    const uchar4 t00 = __ldg(tp + (r0 + ti0)), t10 = __ldg(tp + (r0 + ti1));
    const uchar4 t01 = __ldg(tp + (r1 + ti0)), t11 = __ldg(tp + (r1 + ti1));
    const float a0[3] = {(float)t00.x, (float)t00.y, (float)t00.z}, a1[3] = {(float)t10.x, (float)t10.y, (float)t10.z};
    const float b0[3] = {(float)t01.x, (float)t01.y, (float)t01.z}, b1[3] = {(float)t11.x, (float)t11.y, (float)t11.z};
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      const float ta = fmaf(ffx, a1[ch] - a0[ch], a0[ch]);
      const float tb = fmaf(ffx, b1[ch] - b0[ch], b0[ch]);
      const float tc = fmaf(ffy, tb - ta, ta);
      c3[ch] = tc * (c3[ch] * 0.00392156862745098f);
    }
    if (cls_out) {   // (u * twf is exact: a power of two)
      const unsigned cu = (unsigned)__float2int_rd(u * twf) & (tw - 1), cv = (unsigned)__float2int_rd(v * thf) & (th - 1);
      *cls_out = __ldg(cls_pool + ((size_t)(ti & 0xffffffu) << 6) + ((cv << lw) + cu));
    }
  }
}
__device__ __forceinline__ void shade_prim(const PrimRec* __restrict__ prims, unsigned w, const uint8_t* __restrict__ tex_pool,
                                           const float4* __restrict__ lat_tab, int pxa, int pya, float c3[3], float* qq_out = nullptr,
                                           const uint8_t* __restrict__ cls_pool = nullptr, int* cls_out = nullptr) {
  const ShadeIn si = load_shade(prims, w);
  shade_eval(si, tex_pool, lat_tab, pxa, pya, c3, qq_out, cls_pool, cls_out);
}

// ---- bulk-async copy (TMA, 1-D) + mbarrier: global -> shared without register staging
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
  } while (!ok);
}

// u8 = rint(255 * clamp(c)) packed r | g<<8 | b<<16 (resolve of 4 equal samples is the value itself).  The
// float->unsigned conversion rounds to nearest-even and saturates below at 0 (NaN -> 0), min() saturates above:
// identical to clamping c to [0, 1] first.
__device__ __forceinline__ unsigned pack_rgb(float r, float g, float b) {
  const unsigned ur = min(__float2uint_rn(r * 255.0f), 255u);
  const unsigned ug = min(__float2uint_rn(g * 255.0f), 255u);
  const unsigned ub = min(__float2uint_rn(b * 255.0f), 255u);
  return ur | (ug << 8) | (ub << 16);
}

// one 8x4 bin of packed pixels -> global memory: rows of 24 bytes as 6 aligned words built with shuffles.
// The lane-constant parts (shuffle sources, shift, byte offset inside a bin) are computed once per kernel (StoreLane).
struct StoreLane {
  int src_lo, src_hi;   // lanes holding the two pixels this lane's output word straddles
  int sh8;              // bit offset of the word inside lo | hi << 24
  int off;              // byte offset of the word from the bin's first byte: (lane >> 3) * W * 3 + 4 * (lane & 7)
  int j, row;           // word index in the row (only 0..5 store), row inside the bin
};
__device__ __forceinline__ StoreLane make_store_lane(int lane, int W) {
  StoreLane sl;
  const int j = lane & 7, rowbase = lane & ~7;
  const int p0 = (4 * j) / 3;
  sl.sh8 = (4 * j - 3 * p0) * 8;
  sl.src_lo = rowbase + min(p0, 7);
  sl.src_hi = rowbase + min(p0 + 1, 7);
  sl.off = (lane >> 3) * W * 3 + 4 * j;
  sl.j = j; sl.row = lane >> 3;
  return sl;
}
// `bin0` = address of the bin's first byte (warp-uniform); rows_ok = how many of the bin's 4 rows are inside the image
__device__ __forceinline__ void store_bin_fast(uint8_t* __restrict__ bin0, const StoreLane& sl, unsigned rgb, int rows_ok) {
  const unsigned lo = __shfl_sync(0xffffffffu, rgb, sl.src_lo);
  const unsigned hi = __shfl_sync(0xffffffffu, rgb, sl.src_hi);
  const unsigned word = __funnelshift_r(lo | (hi << 24), hi >> 8, sl.sh8);   // (lo | hi << 24) >> sh8, low 32 bits
  if (sl.j < 6 && sl.row < rows_ok) *reinterpret_cast<unsigned*>(bin0 + sl.off) = word;
}
// byte form (any width, bins cut by the right border): a lane stores its own pixel
__device__ __forceinline__ void store_bin_bytes(uint8_t* __restrict__ out, unsigned rgb, int lane, int bx, int by, int W, int H) {
  const int gx = bx * kBinW + (lane & 7), gy = by * kBinH + (lane >> 3);
  if (gx < W && gy < H) {
    uint8_t* d = out + ((size_t)gy * W + gx) * 3;
    d[0] = (uint8_t)(rgb & 255); d[1] = (uint8_t)((rgb >> 8) & 255); d[2] = (uint8_t)(rgb >> 16);
  }
}

// The fine bins of coarse bin (cbx, cby) that lie inside the image, as bits f = column | row << 2: all 8 except on the
// right / bottom border.  `rows` = fine_rows_in_image(cby, H), which k_raster computes once per row of coarse bins.
__device__ __forceinline__ unsigned fine_rows_in_image(int cby, int H) { return ((cby * kCFY + 1) * kBinH < H) ? 0xffu : 0x0fu; }
__device__ __forceinline__ unsigned fine_in_image(int cbx, unsigned rows, int W) {
  const int nx = min(kCFX, (W - cbx * kCoarseW + kBinW - 1) / kBinW);   // fine-bin columns inside the image: 1..4
  const unsigned cols = (1u << nx) - 1u;
  return rows & (cols | (cols << 4));
}

// LUT remap: the source pixel the table names for this lane's output pixel of fine bin (bx, by), in sub-pixels, and
// whether there is one (none: cv2.remap BORDER_CONSTANT, black).  Lanes past the image edge read a clamped entry; their
// pixels are not stored.
struct RemapPx { bool valid; int x, y; };
__device__ __forceinline__ RemapPx remap_source(const RemapTab& rt, int bx, int by, int lane, int W, int H) {
  const int gx = min(bx * kBinW + (lane & 7), W - 1), gy = min(by * kBinH + (lane >> 3), H - 1);
  const int sxy = __ldg(rt.src_xy + gy * W + gx);
  const int sx = (int)(short)(sxy & 0xffff), sy = sxy >> 16;
  return RemapPx{sx != -32768, sx * kSub, sy * kSub};
}
// The table of env `env` in a pool
__device__ __forceinline__ RemapTab remap_of_env(RemapTab rt, int env, int W, int H, int cbins) {
  const int t = __ldg(rt.table_of_env + env);
  rt.src_xy += (size_t)t * W * H;
  rt.cbox += (size_t)t * cbins;
  rt.fbox += (size_t)t * cbins * (kCFX * kCFY);
  rt.cell_start += (size_t)t * (cbins + 1);
  rt.home_start += (size_t)t * (cbins + 1);
  return rt;
}

// One fine bin of a packed u8 HWC frame, the store all three rasterisers share: whole words where the image's rows are
// (W % 4 == 0) and the bin lies inside it, else a byte per channel
__device__ __forceinline__ void store_bin(uint8_t* __restrict__ out, const StoreLane& sl, unsigned rgb, int lane, int bx, int by,
                                          int W, int H) {
  if ((W & 3) == 0 && bx * kBinW + kBinW <= W)
    store_bin_fast(out + ((size_t)(by * kBinH) * W + bx * kBinW) * 3, sl, rgb, min(kBinH, H - by * kBinH));
  else
    store_bin_bytes(out, rgb, lane, bx, by, W, H);
}

// Depth target (render spec item 9): the eye-space depth of a pixel is 1 / (the largest 1/w among the distinct winners
// of its samples), 0 where no sample is covered (`qmax` 0: a prim's 1/w is at least 1e-20) or the gather has no source.
__device__ __forceinline__ float depth_of(float qmax, bool px_valid = true) { return (px_valid && qmax > 0.0f) ? 1.0f / qmax : 0.0f; }
// One fine bin of the depth frame `dep` (f32 [H][W] of one env): a lane stores its own pixel.  The 8 lanes of a bin row
// write 32 contiguous bytes — one whole sector wherever W is a multiple of 8 — so wider per-lane stores packed with
// shuffles would move the same sectors.
__device__ __forceinline__ void store_depth(float* __restrict__ dep, float d, int lane, int bx, int by, int W, int H) {
  const int gx = bx * kBinW + (lane & 7), gy = by * kBinH + (lane >> 3);
  if (gx < W && gy < H) dep[(size_t)gy * W + gx] = d;
}

// Label target (render spec item 10): a pixel's label is 1 + the draw item of the winner depth selects (the largest 1/w;
// among equal ones the smallest label), 0 where no sample is covered or the gather has no source.  Items: the ground
// (draw ids 0, 1), grid cell t = i * grid_h + j (tile_draw_ids ids each), object o (its tri_count ids each, from
// tri_base on), the agent's mesh.  What a label instance needs of its env's map to turn a draw id into a label:
struct LabelMap { const DObject* objects; int n_cells, n_objects, agent_base, tess; };
__device__ __forceinline__ LabelMap label_map(const DMap& m, int tess) {
  return LabelMap{m.objects, m.grid_w * m.grid_h, m.n_objects, m.agent.tri_base, tess};
}
// ground and road tiles only (all k_raster_flat ever sees)
__device__ __forceinline__ int tile_label(int tess, int id) {
  return id < 2 ? 1 : 2 + (tess ? (id - 2) / kTessTris : (id - 2) >> 1);
}
__device__ __forceinline__ int label_of_id(const LabelMap& lm, int id) {
  const int r = id - 2 - tile_draw_ids(lm.tess != 0) * lm.n_cells;   // triangle index among the meshes' draw ids
  if (r < 0) return tile_label(lm.tess, id);
  if (r >= lm.agent_base) return 2 + lm.n_cells + lm.n_objects;
  // the last object whose tri_base <= r (objects without triangles share the tri_base of the object after them)
  int lo = 0, hi = lm.n_objects - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&lm.objects[mid].tri_base) <= r) lo = mid; else hi = mid - 1;
  }
  return 2 + lm.n_cells + lo;
}
// The marking frame `mf` (u8 [H][W] of one env): a lane stores its own pixel, 1 byte.
__device__ __forceinline__ void store_marking(uint8_t* __restrict__ mf, int v, int lane, int bx, int by, int W, int H) {
  const int gx = bx * kBinW + (lane & 7), gy = by * kBinH + (lane >> 3);
  if (gx < W && gy < H) mf[(size_t)gy * W + gx] = (uint8_t)v;
}
// The label frame `lf` (i16 [H][W] of one env): a lane stores its own pixel, 2 bytes.  The 8 lanes of a bin row write 16
// contiguous bytes — half a 32-byte sector — so pairs packed into 4-byte stores with a shuffle would write the same
// sectors, for a shuffle more per pixel.
__device__ __forceinline__ void store_label(int16_t* __restrict__ lf, int v, int lane, int bx, int by, int W, int H) {
  const int gx = bx * kBinW + (lane & 7), gy = by * kBinH + (lane >> 3);
  if (gx < W && gy < H) lf[(size_t)gy * W + gx] = (int16_t)v;
}

// The images a rasteriser instance writes (kAux, a set of these) and what they ask of it
constexpr int kAuxDepth = 1, kAuxLabels = 2, kAuxMarks = 4;
// the label's winner is taken: for the label, and for the marking, which is the class that winner shows
__host__ __device__ constexpr bool takes_winner(int aux) { return (aux & (kAuxLabels | kAuxMarks)) != 0; }
// depth may be stored: by a depth instance, and by a marking instance where the depth target is set
__host__ __device__ constexpr bool may_store_depth(int aux) { return (aux & (kAuxDepth | kAuxMarks)) != 0; }
// a winner's 1/w is needed: for the depth, or to take the label's winner
__host__ __device__ constexpr bool needs_qq(int aux) { return takes_winner(aux) || may_store_depth(aux); }
// depth is stored: always by a depth instance, by a marking instance where the depth target `depth` is set
template <int kAux>
__device__ __forceinline__ bool stores_depth(const float* depth) { return (kAux & kAuxDepth) || ((kAux & kAuxMarks) && depth); }

// One env's frames of the image targets, each [H][W] at `off`.  (The targets and an offset rather than three frame
// pointers: the depth test then reads the kernel parameter, and the pointers cost no registers across a bin.)
struct AuxFrames { AuxTargets t; size_t off; };
__device__ __forceinline__ AuxFrames aux_frames(const AuxTargets& aux, int env, int W, int H) {
  return AuxFrames{aux, (size_t)env * W * H};
}
// One fine bin of each image the instance writes, in the order depth, label, marking: a lane stores its own pixel
template <int kAux>
__device__ __forceinline__ void store_aux(const AuxFrames& af, float depth, int label, int mark, int lane, int bx, int by, int W,
                                          int H) {
  if (stores_depth<kAux>(af.t.depth)) store_depth(af.t.depth + af.off, depth, lane, bx, by, W, H);
  if (kAux & kAuxLabels) store_label(af.t.labels + af.off, label, lane, bx, by, W, H);
  if (kAux & kAuxMarks) store_marking(af.t.marks + af.off, mark, lane, bx, by, W, H);
}

// A pixel's image state over its winners: the largest 1/w (0: none yet), the label of the winner it picks and the
// marking (0: none)
struct AuxPx { float qmax; int lab, mk; };
// One more winner `w` of a pixel (a prim index), its 1/w `qq` (> 0), label_of(w) and texel class `c`: the pixel keeps
// the largest 1/w and, among equal ones, the smallest label; with markings, the smallest class among the winners that
// have both (two triangles of one tile, in tile mode 0 or clipped, can).  Maxima over exact values with exact
// tie-breaks: the order does not matter.
template <int kAux, typename LabelOf>
__device__ __forceinline__ void take_winner(AuxPx& pix, float qq, unsigned w, int c, const LabelOf& label_of) {
  if (!(qq >= pix.qmax)) return;   // (a farther winner: its label is not looked up)
  const int l = label_of(w);
  if (qq > pix.qmax || l < pix.lab) {
    pix.qmax = qq; pix.lab = l;
    if constexpr ((kAux & kAuxMarks) != 0) pix.mk = c;
  } else if constexpr ((kAux & kAuxMarks) != 0) {
    if (l == pix.lab) pix.mk = min(pix.mk, c);
  }
}

// glClearColor: the env's horizon colour, or on the segment view glClearColor(255, 0, 255) clamped to magenta (S:1752)
__device__ __forceinline__ void clear_colour(const DState& S, const RenderCfg& rc, int env, float clr[3]) {
  const bool seg = (rc.mode & DTS_RENDER_SEGMENT) != 0;
  clr[0] = seg ? 1.0f : S.rep[env].horizon[0];
  clr[1] = seg ? 0.0f : S.rep[env].horizon[1];
  clr[2] = seg ? 1.0f : S.rep[env].horizon[2];
}

}  // namespace

// ------------------------------------------------------------------------------------------------ frame memory
struct FrameMem {
  FrameCtx* ctx;        // [N]
  PrimRec* prims;       // [N][max_prims]
  uint32_t* pairs;      // [pool]  prim | coarse bin << 16, grouped by env and coarse bin (k_bin pass 1).  One pool for the
  BinRec* recs;         // [pool]  batch: an env takes exactly the entries it needs (atomic cursor work[1]), densely packed
  int* bin_count;       // [N][cbins]
  int* bin_start;       // [N][cbins]  pool index of the bin's first pair / record
  float4* lat;          // [N][max_lat][64]
  uint2* geo_list;      // [N * items_max] (env, draw item) pairs that passed k_cull
  uint2* solo;          // [N * cbins] (env, coarse bin | prim << 16): coarse bins lying inside one prim (k_bin -> k_raster_solo)
  uint2* flat;          // [N * cbins] (env, coarse bin | record count << 16): flat bins, only road tiles and ground (k_bin -> k_raster_flat)
  uint2* empty;         // [N * cbins] (env, coarse bin): bins without records, cleared by k_raster_solo (k_bin, no LUT)
  uint2* rows;          // [N * cbins_y] (env, coarse row): the rows k_raster still has to draw (k_bin, k_raster_flat -> k_raster)
  int* row_flag;        // [N][cbins_y] nonzero once the row is on `rows` (cleared by k_bin for its env)
  int* work;            // global counters, zeroed per frame: the kWork* slots
  int32_t* status;      // mapped host word (dts_status): bit 0 = a frame ran out of frame memory
};
constexpr int kWorkRaster = 0;     // k_raster's next work item
constexpr int kWorkPairPool = 1;   // pair-pool cursor (k_bin)
constexpr int kWorkGeoList = 2;    // geo_list length (k_cull -> k_geometry)
constexpr int kWorkSoloList = 3;   // solo list length (k_bin -> k_raster_solo)
constexpr int kWorkFlatList = 4;   // flat list length (k_bin -> k_raster_flat)
constexpr int kWorkRowList = 5;    // row list length (k_bin, k_raster_flat's hand-backs -> k_raster)
constexpr int kWorkEmptyList = 6;  // empty list length (k_bin -> k_raster_solo)

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

struct Renderer {
  int n, W, H, flags;        // envs, camera and DTS_FLAG_* of the handle
  int sms;                   // launch sizes are SMs x resident CTAs per SM of each kernel
  int cbins;                 // coarse bins per frame
  // frame sizes, set with the frame memory from the uploaded maps: PrimRec slab and lattice slots per env, draw items
  // per env, and entries of the batch's pair pool
  int max_prims = 0, max_lat = 0, items_max = 0, pool = 0;
  void* frame = nullptr;     // frame memory (null: not reserved since the last map upload)
  FrameMem fm{};             // ... carved
  RemapTab fish{};           // the fisheye remap (null until a LUT is set): one table, or a pool of them
  RemapTab rect{};           // UndistortWrapper's rectification (null unless set)
};

// The one statement of the frame-memory layout: points `f` into the allocation at `base` and returns its size, so
// carving from base 0 sizes it.
__host__ size_t carve(const Renderer& r, uintptr_t base, FrameMem& f) {
  const size_t n = r.n;
  size_t o = 0;
  auto take = [&](auto*& p, size_t count) {
    p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + o);
    o += align256(count * sizeof(*p));
  };
  take(f.work, 64);
  take(f.ctx, n);
  take(f.bin_count, n * r.cbins);
  take(f.bin_start, n * r.cbins);
  take(f.prims, n * r.max_prims);
  take(f.pairs, r.pool);
  take(f.recs, r.pool);
  take(f.lat, n * r.max_lat * 64);
  take(f.geo_list, n * r.items_max);
  take(f.solo, n * r.cbins);
  take(f.flat, n * r.cbins);
  const size_t cbins_y = (r.H + kCoarseH - 1) / kCoarseH;
  take(f.empty, n * r.cbins);
  take(f.rows, n * cbins_y);
  take(f.row_flag, n * cbins_y);
  return o + 256;   // (+ 256 B of slack past the last list)
}

// ------------------------------------------------------------------------------------------------ k_frame_setup
__global__ void __launch_bounds__(128) k_frame_setup(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= n_listed(rc.env_list, rc.env_count, rc.n_envs)) return;
  const int env = listed_env(rc.env_list, slot);
  FrameCtx& c = fm.ctx[env];
  const RenderEp ep = S.rep[env];
  double V[12];
  if (rc.mode & DTS_RENDER_TOP_DOWN) {
    const DMap& m = maps[S.map_id[env]];
    top_down_view((double)m.grid_w, (double)m.grid_h, m.tile_size, (double)ep.cam_fov_y_deg, V);
  } else {
    camera_view(S.pos_x[env], S.pos_z[env], S.angle[env], ep, (rc.flags & DTS_FLAG_DOMAIN_RAND) != 0, V);
  }
#pragma unroll
  for (int k = 0; k < 12; k++) c.V[k] = V[k];
  const double f = 1.0 / tan((double)ep.cam_fov_y_deg * kDeg2Rad / 2.0), aspect = (double)rc.width / (double)rc.height;
  const double zn = 0.04, zf = 100.0;                                     // gluPerspective S:1761
  c.P00 = (float)(f / aspect); c.P11 = (float)f;
  c.P22 = (float)((zf + zn) / (zn - zf)); c.P23 = (float)(2.0 * zf * zn / (zn - zf));
  c.n_prims = 0; c.n_lat = 0; c.overflow = 0; c.pad = 0;
}

// Conservative bounding-sphere cull in eye space against the four side planes and near: true only if the sphere
// — hence everything inside it — lies outside one plane (margins cover the f32 rounding of the test itself).
__device__ __forceinline__ bool sphere_outside(float P00, float P11, float cx_, float cy_, float cz_, float rad) {
  const float hx = rsqrtf(P00 * P00 + 1.0f), hy = rsqrtf(P11 * P11 + 1.0f);
  bool out = cz_ - rad > -0.04f;                                  // entirely behind the near plane
  out |= (P00 * cx_ + cz_) * hx > rad * 1.01f;                    // right plane: P00*x <= -z
  out |= (-P00 * cx_ + cz_) * hx > rad * 1.01f;
  out |= (P11 * cy_ + cz_) * hy > rad * 1.01f;
  out |= (-P11 * cy_ + cz_) * hy > rad * 1.01f;
  return out;
}
// world point -> eye space with the f64 camera matrix (row-major 3x4)
__device__ __forceinline__ void eye_point(const double* V, double wx, double wy, double wz, float& ex, float& ey, float& ez) {
  ex = (float)(V[0] * wx + V[1] * wy + V[2] * wz + V[3]);
  ey = (float)(V[4] * wx + V[5] * wy + V[6] * wz + V[7]);
  ez = (float)(V[8] * wx + V[9] * wy + V[10] * wz + V[11]);
}

// Does draw item `item` of env `env` need any work this frame?  Conservative bounding-sphere test against the view
// frustum before anything is transformed (most (env, item) pairs end here), plus the values the mesh path needs later:
// the obstacle's per-env pose.  Run once per pair by k_cull (one thread each) and again by the warp that draws the item.
struct ItemPose { int dyn_kind; float opx, opz, orot; bool agent_item; };
__device__ __forceinline__ bool item_visible(const DState& S, const DMap& m, const RenderCfg& rc, const FrameCtx& ctx, int env,
                                             int item, ItemPose& ip) {
  const int n_tiles = m.grid_w * m.grid_h;
  ip.dyn_kind = 0; ip.opx = 0.f; ip.opz = 0.f; ip.orot = 0.f;
  ip.agent_item = item == agent_item(n_tiles, m.n_objects);   // top-down views draw the agent's own mesh last (S:1923-1929)
  if (item > agent_item(n_tiles, m.n_objects)) return false;
  if (ip.agent_item && (!(rc.mode & DTS_RENDER_TOP_DOWN) || m.agent.tri_count == 0)) return false;
  if (item >= 1 && item <= n_tiles) {
    const int t = item - 1, ti = t / m.grid_h, tj = t - ti * m.grid_h;
    if (m.tile_kind[tj * m.grid_w + ti] < 0) return false;
    const double ts = m.tile_size;
    float ex, ey, ez;
    eye_point(ctx.V, (ti + 0.5) * ts, 0.0, (tj + 0.5) * ts, ex, ey, ez);
    if (sphere_outside(ctx.P00, ctx.P11, ex, ey, ez, (float)(ts * 0.7071067811865476) * 1.001f + 1e-4f)) return false;
  } else if (item > n_tiles) {
    const int o = item - 1 - n_tiles;
    if (!ip.agent_item && (S.rep[env].hidden[o >> 5] >> (o & 31) & 1u)) return false;
    const DObject& ob = ip.agent_item ? m.agent : m.objects[o];
    ip.opx = ob.pos[0]; ip.opz = ob.pos[2]; ip.orot = ob.y_rot_deg;
    if (ip.agent_item) {   // glTranslatef(*cur_pos); glRotatef(cur_angle * 180 / pi, 0, 1, 0): GLfloat arguments
      ip.opx = (float)S.pos_x[env]; ip.opz = (float)S.pos_z[env];
      ip.orot = (float)(S.angle[env] * 180.0 / 3.141592653589793);
    }
    if (ob.dyn_slot >= 0) {
      ip.dyn_kind = m.dyn[ob.dyn_slot].kind;
      if (ip.dyn_kind != DTS_DYN_TRAFFICLIGHT) {   // a moving obstacle: this env's pos / y_rot, rounded to float like glTranslatef / glRotatef
        const size_t nd = m.n_dyn, ne = rc.n_envs;
        ip.opx = (float)m.dyn_state[((size_t)DTS_DYN_PX * nd + ob.dyn_slot) * ne + env];
        ip.opz = (float)m.dyn_state[((size_t)DTS_DYN_PZ * nd + ob.dyn_slot) * ne + env];
        ip.orot = (float)m.dyn_state[((size_t)DTS_DYN_YROT * nd + ob.dyn_slot) * ne + env];
      }
    }
    double sn, cs;
    sincos((double)ip.orot * kDeg2Rad, &sn, &cs);
    const double sc = (double)ob.scale, ccx = ob.centre[0], ccy = ob.centre[1], ccz = ob.centre[2];
    float ex, ey, ez;   // T(pos) S(scale) Ry(rot) applied to the bounding-sphere centre
    eye_point(ctx.V, (double)ip.opx + sc * (cs * ccx + sn * ccz), (double)ob.pos[1] + sc * ccy, (double)ip.opz + sc * (-sn * ccx + cs * ccz), ex, ey, ez);
    if (sphere_outside(ctx.P00, ctx.P11, ex, ey, ez, ob.bound_rad * ob.scale * 1.002f + 2e-4f)) return false;
  }
  return true;
}

// ------------------------------------------------------------------------------------------------ k_cull
// thread per (env, draw item), item-major: the pairs that survive item_visible() go to a compact work list (warp-
// aggregated atomic append), so that k_geometry spends warps only on items that will emit something.  In tile mode 1
// the ground and the road tiles are k_tiles' work, so only the placed meshes and the agent's own are listed.
__global__ void __launch_bounds__(256) k_cull(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm, int items_max,
                                              int32_t* __restrict__ err) {
  const size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const int item = (int)(g / rc.n_envs), slot = (int)(g - (size_t)item * rc.n_envs);
  bool vis = false;
  int env = 0;
  if (item < items_max && slot < n_listed(rc.env_list, rc.env_count, rc.n_envs)) {
    env = listed_env(rc.env_list, slot);
    const DMap& m = maps[S.map_id[env]];
    ItemPose ip;
    vis = (rc.tessellate || item > m.grid_w * m.grid_h) && item_visible(S, m, rc, fm.ctx[env], env, item, ip);
  }
  const unsigned m = __ballot_sync(0xffffffffu, vis);
  if (!m) return;
  const int lane = threadIdx.x & 31;
  DTS_COUNT(28, __popc(m));
  int base = 0;
  if (lane == __ffs(m) - 1) base = atomicAdd(fm.work + kWorkGeoList, __popc(m));
  base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
  if (vis) fm.geo_list[base + __popc(m & ((1u << lane) - 1u))] = make_uint2((unsigned)env, (unsigned)item);
}

// ------------------------------------------------------------------------------------------------ k_geometry
// The per-env state a geometry warp reads from shared memory: light and material (RenderEp), camera, projection, the
// unlit flag.  `sh` must be free: the caller has synchronised the warp since its last use.
__device__ __forceinline__ void load_geo_warp(GeoWarp& sh, const DState& S, const FrameCtx& ctx, int env, bool seg, int lane) {
  for (int k = lane; k < (int)(sizeof(RenderEp) / 4); k += 32)
    reinterpret_cast<uint32_t*>(&sh.ep)[k] = reinterpret_cast<const uint32_t*>(&S.rep[env])[k];
  if (lane < 12) sh.V[lane] = ctx.V[lane];
  if (lane == 12) { sh.P00 = ctx.P00; sh.P11 = ctx.P11; sh.P22 = ctx.P22; sh.P23 = ctx.P23; sh.unlit = seg ? 1 : 0; }
  __syncwarp();
}

// ground quad S:1805-1812 (draw ids 0, 1): glScalef(50,0.01,50) applied to (+-1,-0.8,+-1), world-space +y normal
__device__ __forceinline__ void draw_ground(const EmitCtx& ec, GeoWarp& sh, bool seg, int lane) {
  model_view(sh.V, 0.0, 0.0, 0.0, 1.0, 1.0, 0.0, sh.x, lane);
  const float gy = (float)(-0.8 * 0.01);
  const float P[4][3] = {{-50.f, gy, 50.f}, {-50.f, gy, -50.f}, {50.f, gy, -50.f}, {50.f, gy, 50.f}};
  const float magenta[3] = {255.f, 0.f, 255.f};   // glColor3f(255, 0, 255) S:1808: clamped to (1, 0, 1) as a vertex colour
  const float* g = seg ? magenta : sh.ep.ground;
  const int pl_ = lane & 3;   // lanes 0..3 light the four corners, the two triangles (0,1,2)(0,2,3) are then warp-uniform
  const Vtx mine = shade_vertex(sh.x, sh, P[pl_][0], P[pl_][1], P[pl_][2], 0.f, 1.f, 0.f, g[0], g[1], g[2], 0.f, 0.f);
  if (lane < 4) sh.corners[lane] = mine;
  __syncwarp();
  process_triangle_uniform(ec, sh.corners[0], sh.corners[1], sh.corners[2], 0, -1, -1, lane);
  process_triangle_uniform(ec, sh.corners[0], sh.corners[2], sh.corners[3], 1, -1, -1, lane);
}

// One warp per CTA, 64 registers, 32 CTAs per SM: the kernel is latency-bound (short dependent chains), so resident warps
// matter more than spills.  Each warp draws the (env, item) pairs of k_cull's work list, grid-strided: in tile mode 1 the
// placed meshes only (k_tiles draws the ground and the road tiles), in tile mode 0 every item.
template <bool kTess>   // true: spec tile mode 0 (DTS_FLAG_TESSELLATE), the literal 98 triangles per road tile
__device__ __forceinline__ void geometry_item(const DState& S, const DMap* __restrict__ maps, const RenderCfg& rc, const FrameMem& fm,
                                              int max_prims, int32_t* __restrict__ err, int env, int item, int lane, GeoWarp& sh) {
  const DMap& m = maps[S.map_id[env]];
  const int n_tiles = m.grid_w * m.grid_h;
  const bool seg = (rc.mode & DTS_RENDER_SEGMENT) != 0;
  const int W = rc.width, H = rc.height;
  FrameCtx& ctx = fm.ctx[env];
  ItemPose ip;
  if (!item_visible(S, m, rc, ctx, env, item, ip)) return;
  const bool agent_item = ip.agent_item;
  const int dyn_kind = ip.dyn_kind;
  const float opx = ip.opx, opz = ip.opz, orot = ip.orot;
  __syncwarp();   // the previous item of this warp is done with the shared GeoWarp
  load_geo_warp(sh, S, ctx, env, seg, lane);
  EmitCtx ec{m.textures, &sh, &ctx, fm.prims + (size_t)env * max_prims, max_prims, W, H};
  const int tris_per_tile = tile_draw_ids(kTess);
  Xform& x = sh.x;
  if (item <= n_tiles) {
    if constexpr (kTess) {
      if (item == 0) {
        draw_ground(ec, sh, seg, lane);
      } else {
        // road tile S:1852-1884: draw order i outer, j inner
        const int t = item - 1, ti = t / m.grid_h, tj = t - ti * m.grid_h;
        const int idx = tj * m.grid_w + ti;
        const TilePose tp = tile_pose(m, ti, tj);
        const double ts = m.tile_size;
        model_view(sh.V, tp.tx, 0.0, tp.tz, 1.0, tp.cs, tp.sn, x, lane);
        int tex = m.tile_tex[idx];
        if (seg && tex >= 0) tex = m.tex_segment[tex];   // Texture.bind(segment=True) G:52-56
        const int base_id = 2 + tris_per_tile * t;
        // frustum-cull the whole tile on its 8x8 lattice, two vertices per lane
        int outside[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int vi = lane + 32 * h;
          const Vtx v = tile_vertex(x, sh, ts, vi >> 3, vi & 7);
          outside[0] += !(v.cz + v.cw >= 0.0f); outside[1] += !(v.cw - v.cz >= 0.0f);
          outside[2] += v.cx < -v.cw; outside[3] += v.cx > v.cw; outside[4] += v.cy < -v.cw; outside[5] += v.cy > v.cw;
        }
        bool culled = false;
#pragma unroll
        for (int p = 0; p < 6; p++) culled |= __all_sync(0xffffffffu, outside[p] == 2);
        if (culled) return;
        // literal vertex list S:407-433 (spec tile mode 0): 7x7 quads, (0,1,2)(0,2,3) split, 3 shades / triangle
        for (int k0 = 0; k0 < kTessTris; k0 += 32) {
          const int k = k0 + lane;
          Vtx v[3];
          if (k < kTessTris) {
            const int quad = k >> 1, half = k & 1, a = quad / 7, b = quad - 7 * a;
#pragma unroll
            for (int j = 0; j < 3; j++) {
              const int aa = j == 0 ? a : (j == 1 ? a + 1 : (half == 0 ? a + 1 : a));
              const int bb = j == 0 ? b : (j == 1 ? (half == 0 ? b : b + 1) : b + 1);
              v[j] = tile_vertex(x, sh, ts, aa, bb);
            }
          }
          process_triangle_lanes(ec, k < kTessTris, v[0], v[1], v[2], base_id + k, tex, -1, lane);
        }
      }
    }
  } else {
    // placed mesh S:1905-1907, O:123-148: T(pos) S(scale) Ry(y_rot)
    const int o = item - 1 - n_tiles;
    const DObject& ob = agent_item ? m.agent : m.objects[o];
    int alt_from = -2;        // traffic-light card on pattern 1: swap this texture id for ob.alt_to
    if (dyn_kind == DTS_DYN_TRAFFICLIGHT) {
      const size_t nd = m.n_dyn, ne = rc.n_envs;
      if (m.dyn_state[((size_t)DTS_DYN_SHOWN * nd + m.dyn[ob.dyn_slot].tl_first) * ne + env] != 0.0) alt_from = ob.alt_from;
    }
    double sn, cs;
    sincos((double)orot * kDeg2Rad, &sn, &cs);
    model_view(sh.V, (double)opx, (double)ob.pos[1], (double)opz, (double)ob.scale, cs, sn, x, lane);
    int base_id = 2 + tris_per_tile * n_tiles;
    for (int q = 0; q < o; q++) base_id += m.objects[q].tri_count;   // (the agent item follows every object)
    for (int k0 = 0; k0 < ob.tri_count; k0 += 32) {
      const int k = k0 + lane;
      Vtx v[3];
      int ttex = -1;
      if (k < ob.tri_count) {
        const size_t ti = (size_t)ob.tri_offset + k;
        const float* p = m.tri_pos + ti * 9;
        const float* n = m.tri_nrm + ti * 9;
        const float* uv = m.tri_uv + ti * 6;
        const float* c = m.tri_col + ti * 9;
#pragma unroll
        for (int j = 0; j < 3; j++)
          v[j] = shade_vertex(x, sh, p[3 * j], p[3 * j + 1], p[3 * j + 2], n[3 * j], n[3 * j + 1], n[3 * j + 2],
                              c[3 * j], c[3 * j + 1], c[3 * j + 2], uv[2 * j], uv[2 * j + 1]);
        ttex = m.tri_tex[ti];
        if (ttex == alt_from) ttex = ob.alt_to;
        if (seg) ttex = ob.seg_tex;   // get_mesh(name, segment=True): every chunk shows the flat class colour (M:268-290)
      }
      process_triangle_lanes(ec, k < ob.tri_count, v[0], v[1], v[2], base_id + k, ttex, -1, lane);
      }
  }
  if (lane == 0 && ctx.overflow) { atomicOr(err, 1); *reinterpret_cast<volatile int32_t*>(fm.status) = 1; }
}

template <bool kTess>
__global__ void __launch_bounds__(kGeoWarps * 32, kGeoMinCtas)
k_geometry(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm, int max_prims, int32_t* __restrict__ err) {
  __shared__ GeoWarp gws[kGeoWarps];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int n_list = fm.work[kWorkGeoList];   // written by k_cull
  for (int wi = blockIdx.x * kGeoWarps + wib; wi < n_list; wi += gridDim.x * kGeoWarps) {
    const uint2 e = fm.geo_list[wi];
    geometry_item<kTess>(S, maps, rc, fm, max_prims, err, (int)e.x, (int)e.y, lane, gws[wib]);
  }
}

// ------------------------------------------------------------------------------------------------ k_tiles
// Tile mode 1: the ground and every road tile of one env (one listed slot) per warp.  The lanes take the map's grid cells
// 32 at a time, a tile per lane: bounding-sphere test, model-view (the f64 entries of model_view_entry), the four corners
// lit and culled against the frustum, and — where no clipping is needed — the quad set up and emitted, all 32 tiles at
// once.  Lattice and prim slots come from one atomic per warp.  Then the whole warp lights the 64 lattice vertices of
// each surviving tile, two per lane, from the transform its lane left in shared memory; tiles that need the clipper, and
// quads that are not strictly convex after snapping, go one at a time through the warp-wide triangle path, as does the
// ground quad.  Same expressions as a tile drawn by one warp, so the prims and lattices are bit-identical; only their
// slots in the env's slab come in another order.
struct TileLanes {
  Xform x[32];      // the transform of lane k's tile
  Vtx c[32][4];     // its corners (0,0) (7,0) (7,7) (0,7), uncoloured: the quad's vertices
};
__global__ void __launch_bounds__(kTileWarps * 32, kTileMinCtas)
k_tiles(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm, int max_prims, int max_lat, int32_t* __restrict__ err) {
  __shared__ GeoWarp gws[kTileWarps];
  __shared__ TileLanes tls[kTileWarps];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int slot = blockIdx.x * kTileWarps + wib;
  if (slot >= n_listed(rc.env_list, rc.env_count, rc.n_envs)) return;   // (the whole warp)
  const int env = listed_env(rc.env_list, slot);
  GeoWarp& sh = gws[wib];
  TileLanes& tl = tls[wib];
  const DMap& m = maps[S.map_id[env]];
  FrameCtx& ctx = fm.ctx[env];
  const bool seg = (rc.mode & DTS_RENDER_SEGMENT) != 0;
  load_geo_warp(sh, S, ctx, env, seg, lane);
  const EmitCtx ec{m.textures, &sh, &ctx, fm.prims + (size_t)env * max_prims, max_prims, rc.width, rc.height};
  float4* lat_tab = fm.lat + (size_t)env * max_lat * 64;
  const int n_tiles = m.grid_w * m.grid_h;
  const double ts = m.tile_size;
  for (int t0 = 0; t0 < n_tiles; t0 += 32) {
    // lane phase: tile t (draw order i outer, j inner, S:1852-1884)
    const int t = t0 + lane, ti = t / m.grid_h, tj = t - ti * m.grid_h, idx = tj * m.grid_w + ti;
    bool live = false;
    if (t < n_tiles && m.tile_kind[idx] >= 0) {
      float ex, ey, ez;   // (item_visible's test of the tile)
      eye_point(sh.V, (ti + 0.5) * ts, 0.0, (tj + 0.5) * ts, ex, ey, ez);
      live = !sphere_outside(sh.P00, sh.P11, ex, ey, ez, (float)(ts * 0.7071067811865476) * 1.001f + 1e-4f);
    }
#if DTS_STATS
    const unsigned in_sphere = __ballot_sync(0xffffffffu, live);   // (the whole warp: DTS_COUNT is lane 0 alone)
    DTS_COUNT(29, __popc(in_sphere));
#endif
    Vtx* cn = tl.c[lane];
    if (live) {
      const TilePose tp = tile_pose(m, ti, tj);
      Xform x;
#pragma unroll
      for (int e = 0; e < 12; e++) model_view_entry(sh.V, tp.tx, 0.0, tp.tz, 1.0, tp.cs, tp.sn, e >> 2, e & 3, x);
      tl.x[lane] = x;
      // the prim is the quad of the 4 corners: cull on those before lighting the lattice
      int out[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        Vtx v = tile_vertex(x, sh, ts, (k == 1 || k == 2) ? 7 : 0, k >= 2 ? 7 : 0);
        out[0] += !(v.cz + v.cw >= 0.0f); out[1] += !(v.cw - v.cz >= 0.0f);
        out[2] += v.cx < -v.cw; out[3] += v.cx > v.cw; out[4] += v.cy < -v.cw; out[5] += v.cy > v.cw;
        v.r = 0.f; v.g = 0.f; v.b = 0.f;
        cn[k] = v;
      }
#pragma unroll
      for (int p = 0; p < 6; p++) live &= out[p] != 4;
    }
    const unsigned lit = __ballot_sync(0xffffffffu, live);
    if (!lit) continue;
    int lat = 0;
    if (lane == 0) lat = atomicAdd(&ctx.n_lat, __popc(lit));
    lat = __shfl_sync(0xffffffffu, lat, 0) + __popc(lit & ((1u << lane) - 1u));
    if (live && lat >= max_lat) { ctx.overflow = 1; live = false; }
    int tex = -1;
    bool clip = false;   // drawn by the warp-wide path
    if (live) {
      tex = m.tile_tex[idx];
      if (seg && tex >= 0) tex = m.tex_segment[tex];   // Texture.bind(segment=True) G:52-56
      // a tile that needs no clipping is ONE quad prim (its diagonal then splits no bin); otherwise two triangles
      clip = !(classify(cn[0], cn[1], cn[2]) == 0 && classify(cn[0], cn[2], cn[3]) == 0 &&
               setup_and_emit(ec, cn[0], cn[1], cn[2], 2 + 2 * t, tex, lat, &cn[3]));
    }
    __syncwarp();
    // warp phase: the lattice colours of each surviving tile -> table
    for (unsigned todo = __ballot_sync(0xffffffffu, live); todo; todo &= todo - 1) {
      const int src = __ffs(todo) - 1, s = __shfl_sync(0xffffffffu, lat, src);
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int vi = lane + 32 * h;
        const Vtx v = tile_vertex(tl.x[src], sh, ts, vi >> 3, vi & 7);
        lat_tab[s * 64 + vi] = make_float4(v.r, v.g, v.b, 0.0f);
      }
    }
    // ... and the tiles the lanes could not emit as one quad: triangles (0,1,2)(0,2,3), clipped where needed
    for (unsigned todo = __ballot_sync(0xffffffffu, clip); todo; todo &= todo - 1) {
      const int src = __ffs(todo) - 1, id = 2 + 2 * (t0 + src);
      const int stex = __shfl_sync(0xffffffffu, tex, src), slat = __shfl_sync(0xffffffffu, lat, src);
      const Vtx* c = tl.c[src];
      process_triangle_uniform(ec, c[0], c[1], c[2], id, stex, slat, lane);
      process_triangle_uniform(ec, c[0], c[2], c[3], id + 1, stex, slat, lane);
    }
    __syncwarp();   // before the next chunk's lanes overwrite their TileLanes entries
  }
  draw_ground(ec, sh, seg, lane);
  __syncwarp();
  if (lane == 0 && ctx.overflow) { atomicOr(err, 1); *reinterpret_cast<volatile int32_t*>(fm.status) = 1; }
}

// ------------------------------------------------------------------------------------------------ k_bin
// CTA (1 or 4 warps) per env, the env's prims striped over the warps.  Pass 1: exact-size lists of (prim, 32x8-px coarse bin)
// pairs — count (shared-memory atomics), scan, scatter; prims with a small bounding box are binned by it, larger ones
// test each bin of the box against their edges, one bin per lane.  Pass 2, dense over the pairs (one per thread, so a
// screen-filling prim costs no more lanes than a sliver): the pair's BinRec.
// Then the lists of the bins k_raster_solo and k_raster_flat draw, and the list of the rows k_raster still has to draw.
constexpr int kBinWarps = 4;
constexpr int kCountMask = 0xfffff, kGroundInc = 1 << 20;   // a bin's counter: records | ground-quad records << 20
constexpr int kFlatBin = -0x7fffffff - 1;   // bin_count of a flat bin (k_raster_flat); solo bins hold -(prim + 1) >= -65536
constexpr int kEmptyBin = kFlatBin + 1;     // bin_count of an empty bin (no records) that k_raster_solo clears
constexpr int kSoloMark = 2;   // no_flat[] bit of a solo bin (bit 0: not flat)
// Row `cby` of `env` onto k_raster's list, unless it is there already (`row_flag`: k_bin clears its env's flags)
__device__ __forceinline__ void row_to_list(const FrameMem& fm, int env, int cby, int cbins_y) {
  if (atomicOr(fm.row_flag + (size_t)env * cbins_y + cby, 1) == 0)
    fm.rows[atomicAdd(fm.work + kWorkRowList, 1)] = make_uint2((unsigned)env, (unsigned)cby);
}
// Every row of `env` onto k_raster's list, its flags set (the CTA's threads tid of nthr)
__device__ __forceinline__ void list_every_row(const FrameMem& fm, int env, int cbins_y, int tid, int nthr) {
  for (int r = tid; r < cbins_y; r += nthr) {
    fm.row_flag[(size_t)env * cbins_y + r] = 1;
    fm.rows[atomicAdd(fm.work + kWorkRowList, 1)] = make_uint2((unsigned)env, (unsigned)r);
  }
}
// kListed: the frame draws the envs of rc.env_list.  (Its own instance: an env id loaded from the list stays live across
// the kernel, where blockIdx.x is re-read for free, and would cost the remap instances registers and spills.)
template <int kRemap, bool kListed>   // kRemap other than kRemapNone: bins are the LUT's source boxes of the output bins
__global__ void __launch_bounds__(kBinWarps * 32, 8)   // 64 registers: 32 one-warp CTAs per SM at small cameras
k_bin(RenderCfg rc, FrameMem fm, RemapTab rts, int max_prims, int max_pairs, int32_t* __restrict__ err) {
  extern __shared__ int bin_smem[];
  __shared__ int s_total, s_base, s_ok;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, tid = threadIdx.x;
  if (kListed && (int)blockIdx.x >= __ldg(rc.env_count)) return;   // (the whole CTA)
  const int env = kListed ? __ldg(rc.env_list + blockIdx.x) : (int)blockIdx.x, nthr = blockDim.x;   // 1 warp per env for small cameras, 4 for large ones (launch_render)
  const int W = rc.width, H = rc.height;
  const int cbins_x = (W + kCoarseW - 1) / kCoarseW, cbins_y = (H + kCoarseH - 1) / kCoarseH, cbins = cbins_x * cbins_y;
  const RemapTab rt = kRemap == kRemapPool ? remap_of_env(rts, env, W, H, cbins) : rts;
  int* cnt = bin_smem;
  int* start = cnt + cbins;
  const PrimRec* prims = fm.prims + (size_t)env * max_prims;
  uint32_t* pairs = fm.pairs;
  const int n = min(fm.ctx[env].n_prims, max_prims);
  for (int pass = 0; pass < 2; pass++) {
    for (int b = tid; b < cbins; b += nthr) cnt[b] = 0;
    __syncthreads();
    for (int p0 = wib * 32; p0 < n; p0 += nthr) {
      const int p = p0 + lane;
      const bool have = p < n;
      int qx[4] = {0, 0, 0, 0}, qy[4] = {0, 0, 0, 0}, nv = 3, ginc = 1;
      if (have) {
        const int4 w0 = __ldg(reinterpret_cast<const int4*>(prims + p));
        const int4 w1 = __ldg(reinterpret_cast<const int4*>(prims + p) + 1);
        qx[0] = w0.x; qx[1] = w0.z; qx[2] = w1.x; qx[3] = w1.z;
        qy[0] = w0.y; qy[1] = w0.w; qy[2] = w1.y; qy[3] = w1.w;
        nv = ((__ldg(&prims[p].ltq) >> 24) & 1) ? 4 : 3;   // vertex 3 of a triangle repeats vertex 0
        if (__ldg(&prims[p].id) < 2) ginc = 1 + kGroundInc;   // the ground quad's records are counted in the upper bits too
      }
      const int minx = min(min(qx[0], qx[1]), min(qx[2], qx[3])), maxx = max(max(qx[0], qx[1]), max(qx[2], qx[3]));
      const int miny = min(min(qy[0], qy[1]), min(qy[2], qy[3])), maxy = max(max(qy[0], qy[1]), max(qy[2], qy[3]));
      // pixel bounding box, and (identity bins) the range of coarse bins it meets
      const int pminx = max(minx >> 6, 0), pmaxx = min(maxx >> 6, W - 1), pminy = max(miny >> 6, 0), pmaxy = min(maxy >> 6, H - 1);
      const int bx0 = pminx / kCoarseW, by0 = pminy / kCoarseH, bx1 = pmaxx / kCoarseW, by1 = pmaxy / kCoarseH;
      // A prim that may meet many bins is handed to the whole warp (one bin per lane and round) instead of one lane
      // walking all of them while 31 wait: the ground quad and the near tiles span hundreds of bins.
      const bool big = have && (bx1 - bx0 + 1) * (by1 - by0 + 1) > 8;   // (remap: source cells under the prim's box)
      if (have && !big) {
        if (kRemap != kRemapNone) {
          // the output bins whose SOURCE box meets the prim, through the inverse index: the source cells under the prim's
          // pixel box (the same 32x8 grid), each with its list of output bins.  A bin listed by several of those cells
          // is taken from the first one only (the cell holding the top-left corner of box ∩ prim-cell-range).
          for (int cy = by0; cy <= by1; cy++)
            for (int cx = bx0; cx <= bx1; cx++) {
              const int c = cy * cbins_x + cx;
              for (int q = rt.cell_start[c]; q < rt.cell_start[c + 1]; q++) {
                const int b = rt.cell_bins[q];
                const short4 cb = rt.cbox[b];
                if (pmaxx < cb.x || pminx > cb.z || pmaxy < cb.y || pminy > cb.w) continue;
                if (cx != max(bx0, cb.x / kCoarseW) || cy != max(by0, cb.y / kCoarseH)) continue;   // counted from another cell
                const int pos = atomicAdd(&cnt[b], ginc) & kCountMask;
                if (pass == 1) pairs[start[b] + pos] = (uint32_t)p | ((uint32_t)b << 16);
              }
            }
        } else {
          const bool large = (bx1 - bx0 + 1) * (by1 - by0 + 1) > 4;
          for (int by = by0; by <= by1; by++)
            for (int bx = bx0; bx <= bx1; bx++) {
              if (large && !bin_overlaps(qx, qy, nv, bx * kCoarseW * kSub, by * kCoarseH * kSub)) continue;
              const int b = by * cbins_x + bx;
              const int pos = atomicAdd(&cnt[b], ginc) & kCountMask;
              if (pass == 1) pairs[start[b] + pos] = (uint32_t)p | ((uint32_t)b << 16);
            }
        }
      }
      unsigned bigs = __ballot_sync(0xffffffffu, big);
      while (bigs) {
        const int src = __ffs(bigs) - 1;
        bigs &= bigs - 1;
        int vx[4], vy[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { vx[k] = __shfl_sync(0xffffffffu, qx[k], src); vy[k] = __shfl_sync(0xffffffffu, qy[k], src); }
        const int snv = __shfl_sync(0xffffffffu, nv, src), sp = p0 + src, sginc = __shfl_sync(0xffffffffu, ginc, src);
        if (kRemap != kRemapNone) {
          // one HOME cell per lane and round: every output bin is listed once, under the source cell holding the top-left
          // corner of its source box (second inverse index), so a prim spanning many cells meets each candidate bin once;
          // the range of home cells is the prim's cell range grown up / left by the largest box extent of the LUT
          const int sminx = __shfl_sync(0xffffffffu, pminx, src), smaxx = __shfl_sync(0xffffffffu, pmaxx, src);
          const int sminy = __shfl_sync(0xffffffffu, pminy, src), smaxy = __shfl_sync(0xffffffffu, pmaxy, src);
          const int hx0 = max(__shfl_sync(0xffffffffu, bx0, src) - rt.ext_x, 0), sbx1 = __shfl_sync(0xffffffffu, bx1, src);
          const int hy0 = max(__shfl_sync(0xffffffffu, by0, src) - rt.ext_y, 0), sby1 = __shfl_sync(0xffffffffu, by1, src);
          const int nbx = sbx1 - hx0 + 1, nb = nbx * (sby1 - hy0 + 1);
          for (int i = lane; i < nb; i += 32) {
            const int cy = hy0 + i / nbx, cx = hx0 + i % nbx, c = cy * cbins_x + cx;
            const int q1 = __ldg(rt.home_start + c + 1);
            for (int q = __ldg(rt.home_start + c); q < q1; q++) {
              const int4 e = __ldg(rt.home_ent + q);   // x0 | y0 << 16, x1 | y1 << 16, bin
              const int x0 = (int)(short)(e.x & 0xffff), y0 = e.x >> 16, x1 = (int)(short)(e.y & 0xffff), y1 = e.y >> 16;
              if (smaxx < x0 || sminx > x1 || smaxy < y0 || sminy > y1) continue;
              if (!box_overlaps(vx, vy, snv, x0 * kSub + 8, x1 * kSub + 56, y0 * kSub + 8, y1 * kSub + 56)) continue;
              const int pos = atomicAdd(&cnt[e.z], sginc) & kCountMask;
              if (pass == 1) pairs[start[e.z] + pos] = (uint32_t)sp | ((uint32_t)e.z << 16);
            }
          }
        } else {
          const int sbx0 = __shfl_sync(0xffffffffu, bx0, src), sbx1 = __shfl_sync(0xffffffffu, bx1, src);
          const int sby0 = __shfl_sync(0xffffffffu, by0, src), sby1 = __shfl_sync(0xffffffffu, by1, src);
          const int nbx = sbx1 - sbx0 + 1, nb = nbx * (sby1 - sby0 + 1);
          for (int i = lane; i < nb; i += 32) {
            const int by = sby0 + i / nbx, bx = sbx0 + i % nbx;
            if (!bin_overlaps(vx, vy, snv, bx * kCoarseW * kSub, by * kCoarseH * kSub)) continue;
            const int b = by * cbins_x + bx;
            const int pos = atomicAdd(&cnt[b], sginc) & kCountMask;
            if (pass == 1) pairs[start[b] + pos] = (uint32_t)sp | ((uint32_t)b << 16);
          }
        }
      }
    }
    __syncthreads();
    if (pass == 0) {
      if (wib == 0) {
        int carry = 0;
        for (int b0 = 0; b0 < cbins; b0 += 32) {
          const int b = b0 + lane;
          const int v = b < cbins ? (cnt[b] & kCountMask) : 0;
          int inc = v;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) { const int t_ = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t_; }
          if (b < cbins) start[b] = carry + inc - v;
          carry += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (lane == 0) {   // this env's run of the batch-wide pair pool
          const unsigned base = atomicAdd(reinterpret_cast<unsigned*>(fm.work) + kWorkPairPool, (unsigned)carry);
          s_total = carry; s_base = (int)base;
          s_ok = (unsigned long long)base + (unsigned)carry <= (unsigned long long)max_pairs;
        }
      }
      __syncthreads();
      const int base = s_base;
      const bool ok = s_ok != 0;
      for (int b = tid; b < cbins; b += nthr) {
        start[b] += base;
        fm.bin_count[(size_t)env * cbins + b] = ok ? (cnt[b] & kCountMask) : 0;   // lists that do not fit: the frame stays clear
        fm.bin_start[(size_t)env * cbins + b] = start[b];
      }
      if (!ok) {
        if (tid == 0) { fm.ctx[env].overflow = 1; atomicOr(err, 1); *reinterpret_cast<volatile int32_t*>(fm.status) = 1; }
        list_every_row(fm, env, cbins_y, tid, nthr);   // every bin holds count 0: k_raster clears the whole frame
        return;
      }
    }
  }
  // pass 2: one pair per thread -> its visibility record (the pairs were written by other threads of this CTA: the
  // barrier above orders those writes before these reads)
  const int pair0 = s_base, total = s_total;
  // start[] is free from here on: per coarse bin, nonzero once a record rules the bin out of k_raster_flat (a mesh
  // triangle, a tiny triangle, or a solo bin, which also sets kSoloMark)
  int* no_flat = start;
  for (int b = tid; b < cbins; b += nthr) no_flat[b] = 0;
  for (int r = tid; r < cbins_y; r += nthr) fm.row_flag[(size_t)env * cbins_y + r] = 0;
  __syncthreads();
  BinRec* recs = fm.recs;
  for (int i = pair0 + tid; i < pair0 + total; i += nthr) {
    const uint32_t pair = pairs[i];
    const int p = (int)(pair & 0xffffu), b = (int)(pair >> 16);
    const int cby = b / cbins_x, cbx = b - cby * cbins_x;
    unsigned r;
    if (kRemap != kRemapNone) {
      const short4 cb = rt.cbox[b];
      r = build_binrec(prims + p, p, cb.x * kSub, cb.y * kSub, recs + i, rt.fbox + (size_t)b * 8);
    } else {
      r = build_binrec(prims + p, p, cbx * kCoarseW * kSub, cby * kCoarseH * kSub, recs + i);
    }
    // the coarse bin lies inside this prim and holds no other (besides the ground, hidden below it): no visibility
    // work at all -> the bin goes to k_raster_solo, and k_raster skips it (negative count)
    const int c = cnt[b];
    const unsigned valid = fine_in_image(cbx, fine_rows_in_image(cby, H), W);
    // (... or it is the bin's only record: a stretch of bare ground)
    const bool alone = (r & kRecGround) ? (c & kCountMask) == 1 : (c & kCountMask) - (c >> 20) == 1;
    if (alone && (r & valid) == valid) {
      fm.bin_count[(size_t)env * cbins + b] = -(p + 1);
      const int slot = atomicAdd(fm.work + kWorkSoloList, 1);
      fm.solo[slot] = make_uint2((unsigned)env, (unsigned)b | ((unsigned)p << 16));
      atomicOr(&no_flat[b], 1 | kSoloMark);
    }
    if (!(r & kRecFlatOk)) atomicOr(&no_flat[b], 1);
  }
  // flat bins: 1..kStage records, every one a flat road tile or the ground quad, not solo -> k_raster_flat's list, and
  // k_raster skips them (kFlatBin) unless k_raster_flat hands one back.  Empty bins, without a LUT and where the image's
  // rows are whole words -> k_raster_solo's empty list, which clears them, and k_raster skips them (kEmptyBin).  A row
  // holding any other bin -> k_raster's list.
  __syncthreads();
  for (int b0 = wib * 32; b0 < cbins; b0 += nthr) {
    const int b = b0 + lane, c = b < cbins ? (cnt[b] & kCountMask) : 0;
    const bool flat = c >= 1 && c <= kStage && !no_flat[b];
    // (otherwise k_raster clears them, per pixel: clear_empty_bins stores whole words, and the LUT can name no source)
    const bool empty = kRemap == kRemapNone && (W & 3) == 0 && b < cbins && c == 0;
    const unsigned m = __ballot_sync(0xffffffffu, flat), me = __ballot_sync(0xffffffffu, empty);
    if (m) {
      int base = 0;
      if (lane == 0) base = atomicAdd(fm.work + kWorkFlatList, __popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (flat) {
        fm.bin_count[(size_t)env * cbins + b] = kFlatBin;
        fm.flat[base + __popc(m & ((1u << lane) - 1u))] = make_uint2((unsigned)env, (unsigned)b | ((unsigned)c << 16));
      }
    }
    if (me) {
      DTS_COUNT(30, __popc(me));
      int base = 0;
      if (lane == 0) base = atomicAdd(fm.work + kWorkEmptyList, __popc(me));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (empty) {
        fm.bin_count[(size_t)env * cbins + b] = kEmptyBin;
        fm.empty[base + __popc(me & ((1u << lane) - 1u))] = make_uint2((unsigned)env, (unsigned)b);
      }
    }
    // (a gathering step ships every row from k_raster: all of them on its list)
    if (b < cbins && (rc.all_rows || (!flat && !empty && !(no_flat[b] & kSoloMark)))) row_to_list(fm, env, b / cbins_x, cbins_y);
  }
}

// A finished run of image rows -> every rank's gather buffer (peer memory over NVLink): 16-byte vectors, 512 contiguous
// bytes per warp store.  The rows were written by this very warp (__syncwarp orders those stores before these loads).
__device__ __noinline__ void gather_rows_out(const uint8_t* __restrict__ src, const GatherTab& gt, size_t off, size_t nbytes, int lane) {
  __syncwarp();
  const uint8_t* s = src + off;
  if (((reinterpret_cast<size_t>(s) | nbytes) & 15) == 0) {
    bool aligned = true;
    for (int p = 0; p < gt.n; p++) aligned &= (reinterpret_cast<size_t>(gt.base[p] + off) & 15) == 0;
    if (aligned) {
      for (size_t i = (size_t)lane * 16; i < nbytes; i += 512) {
        const int4 v = __ldcg(reinterpret_cast<const int4*>(s + i));   // from L2, where this warp's stores went
        for (int p = 0; p < gt.n; p++) *reinterpret_cast<int4*>(gt.base[p] + off + i) = v;
      }
      return;
    }
  }
  for (size_t i = lane; i < nbytes; i += 32) {
    const uint8_t v = __ldcg(s + i);
    for (int p = 0; p < gt.n; p++) gt.base[p][off + i] = v;
  }
}

constexpr size_t kRasterSmem = (sizeof(BinRec) * 2 * kStage + 16 + 128 * sizeof(unsigned long long)) * kWarps;
// order-preserving map of a float onto unsigned (and back): depth keys of the tiny-triangle buffer
__device__ __forceinline__ unsigned float_key(float f) { const unsigned b = __float_as_uint(f); return b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u); }
__device__ __forceinline__ float key_float(unsigned k) { return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu)); }

// The MSAA samples of the pixel at (pxc, pyc) (sub-pixels from the coarse bin corner) that record `br` covers, as bits 0-3
__device__ __forceinline__ int sample_mask(const BinRec& br, int pxc, int pyc) {
  const int4 E = *reinterpret_cast<const int4*>(br.E0);
  const int4 A = *reinterpret_cast<const int4*>(br.A);
  const int4 B = *reinterpret_cast<const int4*>(br.B);
  const int ec0 = E.x + A.x * pxc + B.x * pyc;
  const int ec1 = E.y + A.y * pxc + B.y * pyc;
  const int ec2 = E.z + A.z * pxc + B.z * pyc;
  int mask = 0;
  if (br.kind & kKindQuad) {
    const int ec3 = E.w + A.w * pxc + B.w * pyc;
#pragma unroll
    for (int s = 0; s < 4; s++) {
      const int e0 = ec0 + A.x * sample_x(s) + B.x * sample_y(s);
      const int e1 = ec1 + A.y * sample_x(s) + B.y * sample_y(s);
      const int e2 = ec2 + A.z * sample_x(s) + B.z * sample_y(s);
      const int e3 = ec3 + A.w * sample_x(s) + B.w * sample_y(s);
      if ((e0 | e1 | e2 | e3) >= 0) mask |= 1 << s;
    }
  } else {
#pragma unroll
    for (int s = 0; s < 4; s++) {
      const int e0 = ec0 + A.x * sample_x(s) + B.x * sample_y(s);
      const int e1 = ec1 + A.y * sample_x(s) + B.y * sample_y(s);
      const int e2 = ec2 + A.z * sample_x(s) + B.z * sample_y(s);
      if ((e0 | e1 | e2) >= 0) mask |= 1 << s;
    }
  }
  return mask;
}

// Deferred shading of one pixel whose visibility is resolved (winner prim per MSAA sample, kNoPrim = clear colour): shaded
// once per distinct winner at the pixel centre (pxa, pya), then the box resolve -> packed u8.
// resolve_edge is the part after the first winner wn[0] is shaded (colour c3): the pixel's other distinct winners, shaded
// in rounds of the whole warp (a lane with nothing pending idles), and the box resolve (s01 + s23) * 0.25 into c3, with
// s01 = c(wn0) + c(wn1), s23 = c(wn2) + c(wn3).  Each shade depends only on (prim, position) and each half has two
// addends, so neither the lane nor the order in which the winners are shaded changes a bit.  Called by the whole warp.
// `pix` comes in as the first winner's (0s: none) and leaves as the pixel's: the largest 1/w over its winners (a maximum
// of exact values, so the order does not matter there either), and where kAux takes the label's winner, its label and
// marking (take_winner; label_of(w): the label of prim w; the class coming from `cls_pool`).
template <int kAux, typename LabelOf>
__device__ __forceinline__ void resolve_edge(const unsigned wn[4], float c3[3], const float clr[3], const PrimRec* __restrict__ prims,
                                             const uint8_t* __restrict__ tex_pool, const float4* __restrict__ lat_tab, int pxa, int pya,
                                             int lane, int32_t* __restrict__ err, AuxPx& pix, const LabelOf& label_of,
                                             const uint8_t* __restrict__ cls_pool) {
  (void)lane; (void)err;   // (DTS_STATS counters)
  float s01[3] = {c3[0], c3[1], c3[2]}, s23[3] = {0.f, 0.f, 0.f};   // 0 + c == c
  unsigned pend = 0xeu;
  if (wn[1] == wn[0]) { pend &= ~2u; s01[0] = s01[0] + c3[0]; s01[1] = s01[1] + c3[1]; s01[2] = s01[2] + c3[2]; }
#pragma unroll
  for (int t = 2; t < 4; t++)
    if (wn[t] == wn[0]) { pend &= ~(1u << t); s23[0] = s23[0] + c3[0]; s23[1] = s23[1] + c3[1]; s23[2] = s23[2] + c3[2]; }
#pragma unroll 1
  while (__any_sync(0xffffffffu, pend != 0u)) {
    DTS_COUNT(12, 1);
    if (pend) {
      const int s = __ffs(pend) - 1;
      const unsigned w = s == 1 ? wn[1] : (s == 2 ? wn[2] : wn[3]);
      float d3[3] = {clr[0], clr[1], clr[2]};
      float qq = 0.0f;
      int c = 0;
      if (w != kNoPrim)
        shade_prim(prims, w, tex_pool, lat_tab, pxa, pya, d3, needs_qq(kAux) ? &qq : nullptr, cls_pool,
                   (kAux & kAuxMarks) ? &c : nullptr);
      if (takes_winner(kAux)) {
        if (w != kNoPrim) take_winner<kAux>(pix, qq, w, c, label_of);
      } else if (kAux & kAuxDepth) {
        pix.qmax = fmaxf(pix.qmax, qq);
      }
#pragma unroll
      for (int t = 1; t < 4; t++)
        if ((pend >> t & 1u) && wn[t] == w) {
          pend &= ~(1u << t);
          if (t < 2) { s01[0] = s01[0] + d3[0]; s01[1] = s01[1] + d3[1]; s01[2] = s01[2] + d3[2]; }
          else { s23[0] = s23[0] + d3[0]; s23[1] = s23[1] + d3[1]; s23[2] = s23[2] + d3[2]; }
        }
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ch++) c3[ch] = (s01[ch] + s23[ch]) * 0.25f;
}
// The whole resolve of one fine bin's pixels (k_raster).  `simple`: the caller knows that every sample of the whole fine
// bin has the same winner.  `pix` receives the pixel's image state (resolve_edge), 0s if it has no winner.
template <int kAux, typename LabelOf>
__device__ __forceinline__ unsigned shade_resolve(const unsigned wn[4], bool simple, const float clr[3], const PrimRec* __restrict__ prims,
                                                  const uint8_t* __restrict__ tex_pool, const float4* __restrict__ lat_tab, int pxa,
                                                  int pya, int lane, int32_t* __restrict__ err, AuxPx& pix, const LabelOf& label_of,
                                                  const uint8_t* __restrict__ cls_pool) {
  const bool same = wn[1] == wn[0] && wn[2] == wn[0] && wn[3] == wn[0];
  const bool all_same = simple || __all_sync(0xffffffffu, same);
  float c3[3] = {clr[0], clr[1], clr[2]};
  pix = AuxPx{};
  if (wn[0] != kNoPrim) {   // every lane: its first winner
    shade_prim(prims, wn[0], tex_pool, lat_tab, pxa, pya, c3, needs_qq(kAux) ? &pix.qmax : nullptr, cls_pool,
               (kAux & kAuxMarks) ? &pix.mk : nullptr);
    if (takes_winner(kAux)) pix.lab = label_of(wn[0]);
  }
  if (!all_same)   // (four equal samples: the mean is the value itself)
    resolve_edge<kAux>(wn, c3, clr, prims, tex_pool, lat_tab, pxa, pya, lane, err, pix, label_of, cls_pool);
  return pack_rgb(c3[0], c3[1], c3[2]);
}

// ------------------------------------------------------------------------------------------------ k_raster
// A work item is one row of coarse bins of one env, from the list k_bin and k_raster_flat built: the rows holding a bin
// that neither k_raster_solo nor k_raster_flat drew, or on a gathering step every row.
template <int kRemap, int kAux>        // kRemap other than kRemapNone: every lane renders the SOURCE pixel the LUT names
                                       // for its output pixel;
                                       // kAux: the images written beside obs (AuxTargets)
__global__ void __launch_bounds__(kThreads, kRasterMinCtas)
k_raster(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm, RemapTab rts, GatherTab gt,
         uint8_t* __restrict__ obs, int max_prims, int max_pairs, int max_lat, int32_t* __restrict__ err, AuxTargets aux) {
  // dynamic shared memory (kRasterSmem bytes): per warp two chunks of records in flight, their mbarriers, and a 128-sample
  // depth / winner buffer for the tiny triangles of the fine bin being drawn
  extern __shared__ __align__(128) unsigned char raster_smem[];
  BinRec (*stages)[2][kStage] = reinterpret_cast<BinRec (*)[2][kStage]>(raster_smem);
  uint64_t (*bars)[2] = reinterpret_cast<uint64_t (*)[2]>(raster_smem + sizeof(BinRec) * kWarps * 2 * kStage);
  unsigned long long* zb = reinterpret_cast<unsigned long long*>(raster_smem + sizeof(BinRec) * kWarps * 2 * kStage + 16 * kWarps) +
                           128 * (threadIdx.x >> 5);
  const int W = rc.width, H = rc.height;
  const int cbins_x = (W + kCoarseW - 1) / kCoarseW, cbins_y = (H + kCoarseH - 1) / kCoarseH, cbins = cbins_x * cbins_y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t frame_bytes = (size_t)W * H * 3;
  const int pxs = (lane & 7) * kSub, pys = (lane >> 3) * kSub;   // this lane's pixel inside a fine bin (sub-pixels)
  const StoreLane sl = make_store_lane(lane, W);
  uint64_t* bar = bars[warp];
  if (lane == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); mbar_fence_init(); }
  __syncwarp();
  uint32_t parity = 0;   // bit s: the phase the next wait on slot s completes
  int cs = 0, ps = 0;    // consumer / producer slot
  const int n_work = fm.work[kWorkRowList];
  int work = 0;
  if (lane == 0) work = atomicAdd(fm.work + kWorkRaster, 1);
  work = __shfl_sync(0xffffffffu, work, 0);
  while (work < n_work) {
    int next_work = 0;
    if (lane == 0) next_work = atomicAdd(fm.work + kWorkRaster, 1);   // consumed after this row: latency hidden
    const uint2 row = fm.rows[work];
    const int env = (int)row.x, cby = (int)row.y;
    const RemapTab rt = kRemap == kRemapPool ? remap_of_env(rts, env, W, H, cbins) : rts;
    const DMap& m = maps[S.map_id[env]];
    const uint8_t* tex_pool = m.tex_pool;
    const PrimRec* prims = fm.prims + (size_t)env * max_prims;
    const BinRec* recs = fm.recs;   // bin_start holds pool indices
    const float4* lat_tab = fm.lat + (size_t)env * max_lat * 64;
    const size_t env_off = (size_t)env * frame_bytes;
    uint8_t* out = obs + env_off;
    const AuxFrames af = aux_frames(aux, env, W, H);
    const uint8_t* cls_pool = (kAux & kAuxMarks) ? tex_pool + m.tex_class_off : nullptr;
    LabelMap lm{};
    if constexpr (takes_winner(kAux)) lm = label_map(m, rc.tessellate);
    auto label_of = [&](unsigned w) { return label_of_id(lm, __ldg(&prims[w].id)); };
    // one fine bin -> obs and the images (the caller's tensors only: the gather carries obs)
    auto emit = [&](unsigned rgb, float depth, int label, int mark, int bx, int by) {
      store_aux<kAux>(af, depth, label, mark, lane, bx, by, W, H);
      store_bin(out, sl, rgb, lane, bx, by, W, H);
    };
    float clr[3];
    clear_colour(S, rc, env, clr);
    const unsigned clear_rgb = pack_rgb(clr[0], clr[1], clr[2]);
    // lane l holds the list of coarse bin (cby, l)
    int my_cnt = 0, my_start = 0;
    if (lane < cbins_x) {
      my_cnt = fm.bin_count[(size_t)env * cbins + cby * cbins_x + lane];
      my_start = fm.bin_start[(size_t)env * cbins + cby * cbins_x + lane];
    }
    const unsigned nz = __ballot_sync(0xffffffffu, my_cnt > 0);
    // ---- producer: walks the row's chunk sequence one chunk ahead of the consumer.  A list of <= 32 records is
    // ONE chunk shared by the bin's 8 fine bins; a longer list is streamed chunk by chunk for each fine bin in turn
    // (the records are ready-made, re-reading them from L2 costs no arithmetic).
    int pcbx = nz ? __ffs(nz) - 1 : 32, pf = 0, pc = 0;
    const unsigned rows_in = fine_rows_in_image(cby, H);
    auto fine_valid = [&](int cbx, int f) -> bool { return (fine_in_image(cbx, rows_in, W) >> f) & 1u; };
    auto next_bin = [&]() {
      const unsigned rem = nz & ~((2u << pcbx) - 1u);
      pcbx = rem ? __ffs(rem) - 1 : 32;
      pf = 0; pc = 0;
    };
    auto issue = [&]() {
      if (pcbx >= 32) return;
      const int n = __shfl_sync(0xffffffffu, my_cnt, pcbx), st = __shfl_sync(0xffffffffu, my_start, pcbx);
      if (n > kStage) while (pf < kCFX * kCFY && !fine_valid(pcbx, pf)) pf++;   // fine bins outside the image are not visited
      if (n > kStage && pf >= kCFX * kCFY) { next_bin(); return; }               // (cannot happen: fine bin 0 is always inside)
      const int nch = min(kStage, n - pc);
      if (lane == 0) {
        mbar_expect_tx(&bar[ps], (uint32_t)(nch * sizeof(BinRec)));
        bulk_load(stages[warp][ps], recs + st + pc, (uint32_t)(nch * sizeof(BinRec)), &bar[ps]);
      }
      ps ^= 1;
      if (n <= kStage) { next_bin(); return; }
      pc += kStage;
      if (pc >= n) {
        pc = 0; pf++;
        while (pf < kCFX * kCFY && !fine_valid(pcbx, pf)) pf++;
        if (pf >= kCFX * kCFY) next_bin();
      }
    };
    issue();
    for (int cbx = 0; cbx < cbins_x; cbx++) {
      const int count = __shfl_sync(0xffffffffu, my_cnt, cbx);
      if (count < 0) continue;   // drawn by k_raster_solo (a bin inside one prim, or kEmptyBin) or k_raster_flat (kFlatBin)
      const unsigned fvalid = fine_in_image(cbx, rows_in, W);
      DTS_COUNT(8, 1);
      if (count == 0) {
        DTS_COUNT(9, 1);
#pragma unroll 1
        for (int f = 0; f < kCFX * kCFY; f++)
          if ((fvalid >> f) & 1u) {
            const int bx = cbx * kCFX + (f & 3), by = cby * kCFY + (f >> 2);
            unsigned rgb = clear_rgb;
            if (kRemap != kRemapNone && !remap_source(rt, bx, by, lane, W, H).valid) rgb = 0u;
            emit(rgb, 0.0f, 0, 0, bx, by);
          }
        continue;
      }
      const bool single = count <= kStage;
      DTS_COUNT(10, count);
      if (!single) { DTS_COUNT(14, 1); DTS_COUNT(15, count); }
      int ox = cbx * kCoarseW * kSub, oy = cby * kCoarseH * kSub;   // coarse bin corner, sub-pixels
      if (kRemap != kRemapNone) { const short4 cb = rt.cbox[cby * cbins_x + cbx]; ox = cb.x * kSub; oy = cb.y * kSub; }   // ... of its source box
#pragma unroll 1
      for (int g = 0; g < (single ? 1 : kCFX * kCFY); g++) {
        if (!single && !((fvalid >> g) & 1u)) continue;
        float z[4];
        unsigned wn[4];   // per sample: depth and winning prim (index into the env's slab)
        bool zb_used = false;   // tiny triangles of this fine bin went through the shared depth / winner buffer
#pragma unroll 1
        for (int c0 = 0; c0 < count; c0 += kStage) {
          // ---- acquire this chunk; the next one starts loading into the other slot meanwhile
          __syncwarp();   // every lane is done with the slot the producer is about to refill
          issue();
          mbar_wait(&bar[cs], (parity >> cs) & 1u);
          parity ^= 1u << cs;
          const BinRec* stage = stages[warp][cs];
          cs ^= 1;
          const int nch = min(kStage, count - c0);
          uint2 mine = make_uint2(0u, 0u);
          if (lane < nch) mine = *reinterpret_cast<const uint2*>(&stage[lane].prim_flags);
          const bool first = c0 == 0, last = c0 + kStage >= count;
          const unsigned ground_bits = __ballot_sync(0xffffffffu, (mine.y & kKindGround) != 0u);   // the ground quad's records in this chunk
          const unsigned tiny_bits = kRemap != kRemapNone ? 0u : __ballot_sync(0xffffffffu, (mine.y & kKindTiny) != 0u);   // one-per-lane triangles
          const unsigned flat_bits = __ballot_sync(0xffffffffu, (mine.y & kKindFlat) != 0u);   // road tiles (plane y = 0)
#if DTS_STATS
          if (single) {   // census: coarse bins lying inside ONE prim (besides the ground)
            const unsigned ng_ = __ballot_sync(0xffffffffu, !(mine.y & kKindGround) && ((mine.x >> 16) & fvalid) != 0u);
            const unsigned ngfull_ = __ballot_sync(0xffffffffu, !(mine.y & kKindGround) && ((mine.x >> 24) & fvalid) == fvalid);
            if (ng_ && !(ng_ & (ng_ - 1)) && (ng_ & ngfull_)) { DTS_COUNT(22, 1); DTS_COUNT(23, __popc(fvalid)); }
          }
#endif
#pragma unroll 1
          for (int f = (single ? 0 : g); f < (single ? kCFX * kCFY : g + 1); f++) {
            if (!((fvalid >> f) & 1u)) continue;
            const int bx = cbx * kCFX + (f & 3), by = cby * kCFY + (f >> 2);   // fine bin
            int pxc = pxs + (f & 3) * kBinW * kSub, pyc = pys + (f >> 2) * kBinH * kSub;   // this lane's pixel, coarse-relative
            bool px_valid = true;
            if (kRemap != kRemapNone) {
              const RemapPx src = remap_source(rt, bx, by, lane, W, H);
              px_valid = src.valid;
              pxc = src.x - ox; pyc = src.y - oy;
            }
            const bool live = (mine.x >> (16 + f)) & 1u;
            const unsigned live_mask = __ballot_sync(0xffffffffu, live);
            const unsigned ground_mask = live_mask & ground_bits;
            bool simple = false;
            if (single) {
              // ---- simple bin: ONE prim (besides the ground quad) and it covers every sample of the bin.
              // All four samples then carry its colour (depth cleared to 1 passes, the ground lies below
              // every other surface and fails GL_LESS), and the mean of four equal floats is exact.
              const unsigned full_mask = __ballot_sync(0xffffffffu, live && ((mine.x >> (24 + f)) & 1u));
              const unsigned others = live_mask & ~ground_mask;
              const unsigned pick = others ? others : live_mask;
              if (pick && !(pick & (pick - 1)) && (pick & full_mask)) {
                simple = true;
                DTS_COUNT(13, 1);
                const unsigned w = stage[__ffs(pick) - 1].prim_flags & 0xffffu;
                wn[0] = w; wn[1] = w; wn[2] = w; wn[3] = w;
              }
            }
            // every prim of the bin besides the ground quad is a road tile: the tiles are coplanar and (up to slivers where
            // two neighbours snapped their shared border differently) disjoint, so a sample belongs to the one tile that
            // covers it — no depth arithmetic; the ground lies below them and takes what is left.  A sample that turns
            // out to be covered twice sends the whole bin through the depth-tested path (exactly the spec's answer).
            bool coplanar = single && !(live_mask & ~ground_mask & ~flat_bits);
            if (coplanar && !simple) DTS_COUNT(20, 1);
            if (!simple) {
              if (first) {
#pragma unroll
                for (int s = 0; s < 4; s++) { z[s] = 1.0f; wn[s] = kNoPrim; }
                zb_used = false;
              }
              // ---- visibility: everything else first, the ground quad last (it is almost always hidden)
#pragma unroll 1
              for (int phase = 0; phase < 2; phase++) {
                unsigned todo = phase == 0 ? (live_mask & ~ground_mask & ~tiny_bits) : ground_mask;
                // every sample of the bin already belongs to a surface above the ground plane: the ground quad
                // (y = -0.008, below everything else) cannot pass GL_LESS anywhere — same argument as the simple bin
                if (phase == 1 && todo &&
                    __all_sync(0xffffffffu, wn[0] != kNoPrim && wn[1] != kNoPrim && wn[2] != kNoPrim && wn[3] != kNoPrim))
                  todo = 0;
                int seen = 0, twice = 0;   // (coverage-only mode) samples of this pixel covered so far / covered by two tiles
                while (todo) {
                  const int k = __ffs(todo) - 1;
                  todo &= todo - 1;
                  const BinRec& br = stage[k];
                  const uint32_t pflags = br.prim_flags;
                  DTS_COUNT(16, 1);
                  if ((pflags >> (24 + f)) & 1u) DTS_COUNT(17, 1);
                  int mask = 15;
                  if (!((pflags >> (24 + f)) & 1u)) {
                    mask = sample_mask(br, pxc, pyc);
                    if (!mask) continue;
                  }
                  if (coplanar && phase == 0) {
                    twice |= seen & mask;
                    seen |= mask;
#pragma unroll
                    for (int s = 0; s < 4; s++)
                      if (mask >> s & 1) wn[s] = pflags & 0xffffu;
                    continue;
                  }
                  // ---- depth of the covered samples, GL_LESS in draw order
                  const float4 zp = *reinterpret_cast<const float4*>(&br.z0);   // z0 zx zy id
                  const int2 xy0 = *reinterpret_cast<const int2*>(&br.x0);
                  const float cdx = (float)(pxc + 32 - xy0.x) * 0.015625f, cdy = (float)(pyc + 32 - xy0.y) * 0.015625f;
                  float zs[4];
                  int lt = 0, eq = 0;
#pragma unroll
                  for (int s = 0; s < 4; s++) {
                    // sample offset from the pixel centre is a multiple of 1/64: cdx + off is exact, i.e.
                    // identical to the spec's (float)(X_sample - x0) / 64
                    const float sdx = cdx + (float)(sample_x(s) - 32) * 0.015625f, sdy = cdy + (float)(sample_y(s) - 32) * 0.015625f;
                    zs[s] = fmaf(zp.z, sdy, fmaf(zp.y, sdx, zp.x));
                    lt |= (zs[s] < z[s]) << s;
                    eq |= (zs[s] == z[s]) << s;
                  }
                  int pass_mask = mask & lt;
                  const int tie = mask & eq;
                  if (tie) {   // exact depth ties are rare: the earlier draw keeps the sample (its id comes from the slab)
                    const int my_id = __float_as_int(zp.w);
#pragma unroll
                    for (int s = 0; s < 4; s++)
                      if ((tie >> s & 1) && wn[s] != kNoPrim && my_id < __ldg(&prims[wn[s]].id)) pass_mask |= 1 << s;
                  }
                  if (!pass_mask) continue;
                  const unsigned me = pflags & 0xffffu;
#pragma unroll
                  for (int s = 0; s < 4; s++)
                    if (pass_mask >> s & 1) { z[s] = zs[s]; wn[s] = me; }
                }
                if (coplanar && phase == 0) {
                  if (__any_sync(0xffffffffu, twice != 0)) {   // rare: start the bin over, depth-tested
                    coplanar = false;
                    DTS_COUNT(21, 1);
#pragma unroll
                    for (int s = 0; s < 4; s++) wn[s] = kNoPrim;
                    phase = -1;
                  } else {
#pragma unroll
                    for (int s = 0; s < 4; s++)
                      if (seen >> s & 1) z[s] = -1.0f;   // the ground (phase 1) can neither pass nor tie there
                  }
                }
              }
            }
            if (kRemap == kRemapNone && !simple && (live_mask & tiny_bits)) {
              // ---- tiny triangles, ONE PER LANE: each lane walks the few pixels of its triangle inside this fine bin and
              // resolves GL_LESS (ties to the lower draw id) with a 64-bit atomicMin on depth | id | prim per sample —
              // 32 triangles per pass instead of one warp-wide visit per triangle
              if (!zb_used) {
                zb_used = true;
#pragma unroll
                for (int s = 0; s < 4; s++) zb[lane * 4 + s] = ~0ull;
                __syncwarp();
              }
              DTS_COUNT(18, 1);
              DTS_COUNT(19, __popc(live_mask & tiny_bits));
              if ((live_mask & tiny_bits) >> lane & 1u) {
                const BinRec& br = stage[lane];
                const int4 E = *reinterpret_cast<const int4*>(br.E0);
                const int4 A = *reinterpret_cast<const int4*>(br.A);
                const int4 B = *reinterpret_cast<const int4*>(br.B);
                const float4 zp = *reinterpret_cast<const float4*>(&br.z0);
                const int2 xy0 = *reinterpret_cast<const int2*>(&br.x0);
                const int fx0 = (f & 3) * kBinW, fy0 = (f >> 2) * kBinH;
                const int x_lo = max(E.w & 0xffff, fx0), x_hi = min(A.w & 0xffff, fx0 + kBinW - 1);
                const int y_lo = max(E.w >> 16, fy0), y_hi = min(A.w >> 16, fy0 + kBinH - 1);
                const unsigned long long tail = ((unsigned long long)(unsigned)__float_as_int(zp.w) << 16) | (br.prim_flags & 0xffffu);
                for (int py = y_lo; py <= y_hi; py++)
                  for (int px = x_lo; px <= x_hi; px++) {
                    const int X = px * kSub, Y = py * kSub;
                    const int ec0 = E.x + A.x * X + B.x * Y, ec1 = E.y + A.y * X + B.y * Y, ec2 = E.z + A.z * X + B.z * Y;
#pragma unroll
                    for (int s = 0; s < 4; s++) {
                      const int e0 = ec0 + A.x * sample_x(s) + B.x * sample_y(s);
                      const int e1 = ec1 + A.y * sample_x(s) + B.y * sample_y(s);
                      const int e2 = ec2 + A.z * sample_x(s) + B.z * sample_y(s);
                      if ((e0 | e1 | e2) < 0) continue;
                      const float sdx = (float)(X + sample_x(s) - xy0.x) * 0.015625f, sdy = (float)(Y + sample_y(s) - xy0.y) * 0.015625f;
                      const float zs = fmaf(zp.z, sdy, fmaf(zp.y, sdx, zp.x));
                      atomicMin(&zb[((py - fy0) * kBinW + (px - fx0)) * 4 + s], ((unsigned long long)float_key(zs) << 32) | tail);
                    }
                  }
              }
              __syncwarp();
            }
            if (!(last || simple)) continue;
            if (kRemap == kRemapNone && !simple && zb_used) {
              // merge the tiny triangles' winners into the per-sample state: GL_LESS, ties to the lower draw id
#pragma unroll
              for (int s = 0; s < 4; s++) {
                const unsigned long long k = zb[lane * 4 + s];
                if (k == ~0ull) continue;
                const float zt = key_float((unsigned)(k >> 32));
                bool win = zt < z[s];
                if (zt == z[s] && wn[s] != kNoPrim) win = (int)((k >> 16) & 0xffffu) < __ldg(&prims[wn[s]].id);
                if (win) { z[s] = zt; wn[s] = (unsigned)(k & 0xffffu); }
              }
              __syncwarp();   // the buffer is re-initialised by the next fine bin
            }
            // ---- deferred shading: once per distinct winner of this pixel, then the box resolve
            DTS_COUNT(11, 1);
            AuxPx pix;
            unsigned rgb = shade_resolve<kAux>(wn, simple, clr, prims, tex_pool, lat_tab, ox + pxc, oy + pyc, lane, err, pix,
                                               label_of, cls_pool);
            if (kRemap != kRemapNone && !px_valid) rgb = 0u;   // cv2.remap BORDER_CONSTANT
            emit(rgb, depth_of(pix.qmax, px_valid), px_valid ? pix.lab : 0, px_valid ? pix.mk : 0, bx, by);
          }
        }
      }
    }
    // On a gathering step the frame goes to the peers in BLOCKS: a work item is 8 whole image rows = one contiguous run of
    // bytes, copied to every rank's gather buffer with 16-byte vector stores once the item is drawn (NVLink wants long
    // writes: per-bin 4-byte stores reach a fifth of the link rate)
    if (gt.n > 0) {   // the item's rows are complete: ship them to every rank
      const int rows = min(kCoarseH, H - cby * kCoarseH);
      gather_rows_out(obs, gt, env_off + (size_t)cby * kCoarseH * W * 3, (size_t)rows * W * 3, lane);
    }
    work = __shfl_sync(0xffffffffu, next_work, 0);
  }
}

// ------------------------------------------------------------------------------------------------ k_raster_solo
// k_bin's empty bins (no LUT, W % 4 == 0): the clear colour in obs, 0 in every image.  A bin waits on two dependent
// loads (its entry, then its env's horizon), so a warp takes eight bins at once, one lane loading each, and then stores
// them one after the other, a whole image row of the bin per store: the row's pixels of obs as words (W % 4 == 0: the
// row starts on a word and its 3 * 32 bytes, or 3 * a multiple of 4 at the right border, are whole words), cycling
// through the three words of the packed colour, and each image's row, a lane per pixel.
template <int kAux>
__device__ __forceinline__ void clear_empty_bins(const DState& S, const RenderCfg& rc, const FrameMem& fm, uint8_t* __restrict__ obs,
                                                 const AuxTargets& aux) {
  constexpr int kBatch = 8;
  const int W = rc.width, H = rc.height;
  const int cbins_x = (W + kCoarseW - 1) / kCoarseW;
  const int lane = threadIdx.x & 31, n = fm.work[kWorkEmptyList];
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int i0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * kBatch; i0 < n; i0 += warps * kBatch) {
    uint2 e = make_uint2(0u, 0u);
    unsigned rgb = 0u;
    if (lane < kBatch && i0 + lane < n) {
      e = fm.empty[i0 + lane];
      float clr[3];
      clear_colour(S, rc, (int)e.x, clr);
      rgb = pack_rgb(clr[0], clr[1], clr[2]);   // bytes r g b 0
    }
#pragma unroll 1
    for (int j = 0; j < min(kBatch, n - i0); j++) {
      const int env = (int)__shfl_sync(0xffffffffu, e.x, j), b = (int)__shfl_sync(0xffffffffu, e.y, j);
      const unsigned c = __shfl_sync(0xffffffffu, rgb, j);
      const int cby = b / cbins_x, x0 = (b - cby * cbins_x) * kCoarseW;
      const int px = min(kCoarseW, W - x0), rows = min(kCoarseH, H - cby * kCoarseH);
      // word k of a row holds channels k, k+1, k+2, k+3 (mod 3) of the colour
      const int k3 = lane % 3;
      const unsigned word = k3 == 0 ? (c | (c << 24)) : (k3 == 1 ? ((c >> 8) | (c << 16)) : ((c >> 16) | (c << 8)));
      const size_t pix0 = (size_t)env * W * H + (size_t)(cby * kCoarseH) * W + x0;
#pragma unroll 1
      for (int r = 0; r < rows; r++) {
        const size_t pix = pix0 + (size_t)r * W;
        if (lane < px * 3 / 4) reinterpret_cast<unsigned*>(obs + pix * 3)[lane] = word;
        if (lane < px) {
          if (stores_depth<kAux>(aux.depth)) aux.depth[pix + lane] = 0.0f;
          if (kAux & kAuxLabels) aux.labels[pix + lane] = 0;
          if (kAux & kAuxMarks) aux.marks[pix + lane] = 0;
        }
      }
    }
  }
}

// Coarse bins that lie inside ONE prim (k_bin found: one record besides the ground quad, covering every sample of every
// fine bin — 22 of the 55 non-empty coarse bins of a c2 frame, 40 % of the shaded pixels) need no records, no staging, no
// visibility state: a warp fetches the prim's planes once and shades the bin's 256 pixels.  A separate kernel so that the
// lean loop gets its own register allocation (the same fast path inside k_raster cost more than it saved).
// Without a LUT, where the image's rows are whole words, the empty bins come here first (k_bin's empty list: the sky, 20
// of a c2 frame's 75 bins), so that k_raster does not walk their rows: the clear colour, and 0 in every image, as
// k_raster writes them (clear_empty_bins).  Runs before k_raster.
// Images: the 1/w the shading divides by gives the depth, the bin's one prim the label of every pixel with a source, and
// the texel it shows there the marking.
template <int kRemap, int kAux>   // kRemap other than kRemapNone: each lane shades the source pixel the LUT names for its output pixel
__global__ void __launch_bounds__(kThreads, kSoloMinCtas) k_raster_solo(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm,
                                                                        RemapTab rts, uint8_t* __restrict__ obs, int max_prims, int max_lat,
                                                                        AuxTargets aux) {
  const int W = rc.width, H = rc.height;
  const int cbins_x = (W + kCoarseW - 1) / kCoarseW;
  const int lane = threadIdx.x & 31;
  const StoreLane sl = make_store_lane(lane, W);
  const size_t frame_bytes = (size_t)W * H * 3;
  if (kRemap == kRemapNone) clear_empty_bins<kAux>(S, rc, fm, obs, aux);
  const int n = fm.work[kWorkSoloList];
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const uint2 e = fm.solo[i];
    const int env = (int)e.x, b = (int)(e.y & 0xffffu);
    const unsigned p = e.y >> 16;
    const int cby = b / cbins_x, cbx = b - cby * cbins_x;
    const RemapTab rt = kRemap == kRemapPool ? remap_of_env(rts, env, W, H, cbins_x * ((H + kCoarseH - 1) / kCoarseH)) : rts;
    uint8_t* out = obs + (size_t)env * frame_bytes;
    // fine bins inside the image as loop bounds rather than fine_in_image(): the mask test costs this loop machine code
    const int nx = min(kCFX, (W - cbx * kCoarseW + kBinW - 1) / kBinW);
    const int ny = ((cby * kCFY + 1) * kBinH < H) ? 2 : 1;
    const uint8_t* tex_pool = maps[S.map_id[env]].tex_pool;
    const float4* lat_tab = fm.lat + (size_t)env * max_lat * 64;
    const ShadeIn si = load_shade(fm.prims + (size_t)env * max_prims, p);
    int lab = 0;
    if constexpr ((kAux & kAuxLabels) != 0)
      lab = label_of_id(label_map(maps[S.map_id[env]], rc.tessellate), __ldg(&fm.prims[(size_t)env * max_prims + p].id));
    const uint8_t* cls_pool = (kAux & kAuxMarks) ? tex_pool + maps[S.map_id[env]].tex_class_off : nullptr;
    const AuxFrames af = aux_frames(aux, env, W, H);
#pragma unroll 1
    for (int fy = 0; fy < ny; fy++)
#pragma unroll 1
    for (int fx = 0; fx < nx; fx++) {
      const int bx = cbx * kCFX + fx, by = cby * kCFY + fy;
      int pxa = (bx * kBinW + (lane & 7)) * kSub, pya = (by * kBinH + (lane >> 3)) * kSub;
      bool px_valid = true;
      if (kRemap != kRemapNone) {
        const RemapPx src = remap_source(rt, bx, by, lane, W, H);
        px_valid = src.valid;
        pxa = src.x; pya = src.y;
      }
      float c3[3], qq = 0.0f;
      int mk = 0;
      shade_eval(si, tex_pool, lat_tab, pxa, pya, c3, may_store_depth(kAux) ? &qq : nullptr, cls_pool,
                 (kAux & kAuxMarks) ? &mk : nullptr);
      unsigned rgb = pack_rgb(c3[0], c3[1], c3[2]);
      if (kRemap != kRemapNone && !px_valid) rgb = 0u;
      store_bin(out, sl, rgb, lane, bx, by, W, H);
      store_aux<kAux>(af, depth_of(qq, px_valid), px_valid ? lab : 0, px_valid ? mk : 0, lane, bx, by, W, H);
    }
  }
}

// ------------------------------------------------------------------------------------------------ k_raster_flat
// Coarse bins of at most kStage records that are all flat road tiles or the ground quad (k_bin's flat list: most of the
// bins neither empty nor solo on a map without objects).  The tiles lie in the plane y = 0 and, up to slivers where two
// neighbours snapped their shared border differently, do not overlap, so a sample belongs to the one tile that covers it:
// no depth arithmetic.  The ground quad lies below every tile and takes the samples no tile covers, where its depth
// passes GL_LESS against the cleared 1.0; samples nothing covers keep the clear colour.  The answer is k_raster's
// coverage-only path, in a kernel of its own so that it is not held to k_raster's register allocation
// (depth state, the tiny-triangle buffer, chunk streaming, the gather).
// Edge pixels are shaded across the whole coarse bin: each fine bin shades every pixel's first winner, and a pixel with
// more than one distinct winner (about a quarter of a general fine bin's lanes) joins a per-warp queue instead of keeping
// the warp for a round at a quarter of its lanes.  Whenever 32 pixels are queued, and after the bin's last fine bin, each
// lane takes one and shades its other winners (resolve_edge: the same bits whichever lane shades them).  The bin's
// colours collect in shared memory and are stored once the bin is done.
// Hand-back: a sample covered by two tiles (or by two ground records) is not resolved here.  The warp drops the bin's
// queue and colours, restores its record count, puts its row on k_raster's list, and k_raster, launched next on the
// stream, draws the whole bin depth-tested.
// Images need no plane in shared memory.  A lane stores a one-winner pixel's images as soon as it has shaded it, and a
// queued pixel's when its other winners are resolved; the queue carries the first winner's 1/w in a third array (2 KB:
// 46 KB per CTA, still four CTAs per SM) and its class in the high half of the entry's slot word, and the first label
// is looked up again from the first winner, which the queue holds.  Only the ground and road tiles come here, so a label
// is arithmetic on the draw id (tile_label).  A bin handed back may have stored some images already: k_raster rewrites
// the whole bin, colour and images.
// Runs after k_raster_solo.
constexpr int kEdgeQ = 64;   // queue ring: flushed at 32 entries, so at most 31 + 32 wait at once
template <int kRemap, int kAux>   // kRemap other than kRemapNone: each lane covers and shades the source pixel the LUT names
                                  // for its output pixel
__global__ void __launch_bounds__(kThreads, kFlatMinCtas) k_raster_flat(const DState S, const DMap* __restrict__ maps, RenderCfg rc, FrameMem fm,
                                                                        RemapTab rts, uint8_t* __restrict__ obs, int max_prims, int max_lat,
                                                                        int32_t* __restrict__ err, AuxTargets aux) {
  __shared__ BinRec stages[kWarps][kStage];   // per warp: the records of its bin
  __shared__ unsigned bin_rgb[kWarps][kCFX * kCFY * 32];   // per warp: packed colour of pixel `lane` of fine bin f at f * 32 + lane
  // per warp: the edge-pixel queue, an entry in two words: (pixel slot, pxa, pya, wn0 | wn1 << 16), (wn2 | wn3 << 16, first colour)
  __shared__ uint4 edge_q[kWarps][2][kEdgeQ];
  const int W = rc.width, H = rc.height;
  const int cbins_x = (W + kCoarseW - 1) / kCoarseW, cbins = cbins_x * ((H + kCoarseH - 1) / kCoarseH);
  const int lane = threadIdx.x & 31;
  BinRec* stage = stages[threadIdx.x >> 5];
  unsigned* rgb_buf = bin_rgb[threadIdx.x >> 5];
  uint4 (*q)[kEdgeQ] = edge_q[threadIdx.x >> 5];
  float* q_qq = nullptr;   // per queue entry, the first winner's 1/w
  if constexpr (needs_qq(kAux)) {
    __shared__ float edge_qq[kWarps][kEdgeQ];
    q_qq = edge_qq[threadIdx.x >> 5];
  }
  const size_t frame_bytes = (size_t)W * H * 3;
  const int pxs = (lane & 7) * kSub, pys = (lane >> 3) * kSub;   // this lane's pixel inside a fine bin (sub-pixels)
  const int warps = (gridDim.x * blockDim.x) >> 5;
  // (the list length is read per bin, from L1: held across the bin it would take a register)
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < __ldg(fm.work + kWorkFlatList); i += warps) {
    const uint2 e = fm.flat[i];
    const int env = (int)e.x, b = (int)(e.y & 0xffffu), count = (int)(e.y >> 16);
    const int cby = b / cbins_x, cbx = b - cby * cbins_x;
    const RemapTab rt = kRemap == kRemapPool ? remap_of_env(rts, env, W, H, cbins) : rts;
    DTS_COUNT(24, 1);
    // ---- stage the records: one per lane, five 128-bit loads
    uint2 mine = make_uint2(0u, 0u);   // prim_flags, kind
    __syncwarp();   // every lane is done with the previous bin's records
    if (lane < count) {
      const int4* src = reinterpret_cast<const int4*>(fm.recs + fm.bin_start[(size_t)env * cbins + b] + lane);
      int4* dst = reinterpret_cast<int4*>(stage + lane);
      int4 v[5];
#pragma unroll
      for (int k = 0; k < 5; k++) v[k] = __ldg(src + k);
#pragma unroll
      for (int k = 0; k < 5; k++) dst[k] = v[k];
      mine = make_uint2((unsigned)v[4].z, (unsigned)v[4].w);
    }
    __syncwarp();
    const unsigned ground_bits = __ballot_sync(0xffffffffu, (mine.y & kKindGround) != 0u);
    const uint8_t* tex_pool = maps[S.map_id[env]].tex_pool;
    const PrimRec* prims = fm.prims + (size_t)env * max_prims;
    const float4* lat_tab = fm.lat + (size_t)env * max_lat * 64;
    uint8_t* out = obs + (size_t)env * frame_bytes;
    const AuxFrames af = aux_frames(aux, env, W, H);
    const uint8_t* cls_pool = (kAux & kAuxMarks) ? tex_pool + maps[S.map_id[env]].tex_class_off : nullptr;
    auto label_of = [&](unsigned w) { return tile_label(rc.tessellate, __ldg(&prims[w].id)); };
    float clr[3];
    clear_colour(S, rc, env, clr);
    int ox = cbx * kCoarseW * kSub, oy = cby * kCoarseH * kSub;   // coarse bin corner, sub-pixels
    if (kRemap != kRemapNone) { const short4 cb = rt.cbox[b]; ox = cb.x * kSub; oy = cb.y * kSub; }   // ... of its source box
    // fine bins inside the image as column / row counts rather than fine_in_image(), as in k_raster_solo
    const int nx = min(kCFX, (W - cbx * kCoarseW + kBinW - 1) / kBinW);
    const int ny = ((cby * kCFY + 1) * kBinH < H) ? 2 : 1;
    unsigned qs = 0;   // edge-pixel queue: entries head = qs >> 16 .. tail - 1 = (qs & 0xffff) - 1, modulo kEdgeQ (one register)
    int f = 0;
#pragma unroll 1
    for (; f < kCFX * kCFY; f++) {
      if ((f & 3) >= nx || (f >> 2) >= ny) continue;
      const int bx = cbx * kCFX + (f & 3), by = cby * kCFY + (f >> 2);   // fine bin
      int pxc = pxs + (f & 3) * kBinW * kSub, pyc = pys + (f >> 2) * kBinH * kSub;   // this lane's pixel, coarse-relative
      bool px_valid = true;
      if (kRemap != kRemapNone) {
        const RemapPx src = remap_source(rt, bx, by, lane, W, H);
        px_valid = src.valid;
        pxc = src.x - ox; pyc = src.y - oy;
      }
      const bool live = (mine.x >> (16 + f)) & 1u;
      const unsigned live_mask = __ballot_sync(0xffffffffu, live);
      const unsigned full_mask = __ballot_sync(0xffffffffu, live && ((mine.x >> (24 + f)) & 1u));
      const unsigned ground_mask = live_mask & ground_bits, tiles = live_mask & ~ground_mask;
      // one prim covering every sample of the fine bin (a lone ground record, too: k_raster's simple bin)
      const unsigned pick = tiles ? tiles : live_mask;
      const bool simple = pick && !(pick & (pick - 1)) && (pick & full_mask);
      unsigned wn[4] = {kNoPrim, kNoPrim, kNoPrim, kNoPrim};
      if (simple) {
        const unsigned w = stage[__ffs(pick) - 1].prim_flags & 0xffffu;
        wn[0] = w; wn[1] = w; wn[2] = w; wn[3] = w;
      } else {
        int seen = 0, twice = 0;   // samples of this pixel covered so far / covered twice
        for (unsigned todo = tiles; todo; todo &= todo - 1) {
          const BinRec& br = stage[__ffs(todo) - 1];
          const uint32_t pflags = br.prim_flags;
          const int mask = ((pflags >> (24 + f)) & 1u) ? 15 : sample_mask(br, pxc, pyc);
          twice |= seen & mask;
          seen |= mask;
#pragma unroll
          for (int s = 0; s < 4; s++)
            if (mask >> s & 1) wn[s] = pflags & 0xffffu;
        }
        // the ground quad on the samples no tile covers (none left anywhere in the fine bin: it is hidden)
        unsigned todo = __all_sync(0xffffffffu, seen == 15) ? 0u : ground_mask;
        for (; todo; todo &= todo - 1) {
          const BinRec& br = stage[__ffs(todo) - 1];
          const uint32_t pflags = br.prim_flags;
          const int mask = (((pflags >> (24 + f)) & 1u) ? 15 : sample_mask(br, pxc, pyc)) & ~(seen & 15);
          if (!mask) continue;
          twice |= (seen >> 4) & mask;
          seen |= mask << 4;
          // GL_LESS against the cleared depth 1.0, the depth plane evaluated exactly as k_raster does
          const float4 zp = *reinterpret_cast<const float4*>(&br.z0);   // z0 zx zy id
          const int2 xy0 = *reinterpret_cast<const int2*>(&br.x0);
          const float cdx = (float)(pxc + 32 - xy0.x) * 0.015625f, cdy = (float)(pyc + 32 - xy0.y) * 0.015625f;
#pragma unroll
          for (int s = 0; s < 4; s++) {
            const float sdx = cdx + (float)(sample_x(s) - 32) * 0.015625f, sdy = cdy + (float)(sample_y(s) - 32) * 0.015625f;
            if ((mask >> s & 1) && fmaf(zp.z, sdy, fmaf(zp.y, sdx, zp.x)) < 1.0f) wn[s] = pflags & 0xffffu;
          }
        }
        if (__any_sync(0xffffffffu, twice != 0)) {   // rare: k_raster draws the bin, depth-tested
          DTS_COUNT(25, 1);
          if (lane == 0) {
            fm.bin_count[(size_t)env * cbins + b] = count;
            row_to_list(fm, env, cby, (H + kCoarseH - 1) / kCoarseH);
          }
          break;
        }
      }
      // ---- every lane: its first winner.  One winner: the pixel is done.  More: it waits in the queue.  (A pixel the
      // LUT gives no source is black either way.)
      float c3[3] = {clr[0], clr[1], clr[2]}, qq0 = 0.0f;
      int c0 = 0;
      if (wn[0] != kNoPrim)
        shade_prim(prims, wn[0], tex_pool, lat_tab, ox + pxc, oy + pyc, c3, needs_qq(kAux) ? &qq0 : nullptr, cls_pool,
                   (kAux & kAuxMarks) ? &c0 : nullptr);
      const bool edge = px_valid && !(wn[1] == wn[0] && wn[2] == wn[0] && wn[3] == wn[0]);
      const unsigned edges = __ballot_sync(0xffffffffu, edge);
      const unsigned slot = f * 32 + lane;
      if (edge) {
        const int e = (qs + __popc(edges & ((1u << lane) - 1u))) & (kEdgeQ - 1);
        q[0][e] = make_uint4((kAux & kAuxMarks) ? slot | (unsigned)c0 << 16 : slot, (unsigned)(ox + pxc), (unsigned)(oy + pyc),
                             wn[0] | (wn[1] << 16));
        q[1][e] = make_uint4(wn[2] | (wn[3] << 16), __float_as_uint(c3[0]), __float_as_uint(c3[1]), __float_as_uint(c3[2]));
        if (needs_qq(kAux)) q_qq[e] = qq0;
      } else {
        rgb_buf[slot] = (kRemap != kRemapNone && !px_valid) ? 0u : pack_rgb(c3[0], c3[1], c3[2]);
        const int lab = ((kAux & kAuxLabels) && px_valid && wn[0] != kNoPrim) ? label_of(wn[0]) : 0;
        store_aux<kAux>(af, depth_of(qq0, px_valid), lab, px_valid ? c0 : 0, lane, bx, by, W, H);   // (c0 = 0 without a winner)
      }
      qs += __popc(edges);
      DTS_COUNT(26, __popc(edges));
      // ---- the queued pixels' other winners, one pixel per lane: 32 at a time, and what is left after the last fine bin
#pragma unroll 1
      for (int nq = (qs & 0xffffu) - (qs >> 16); nq >= 32 || (nq > 0 && f == (ny - 1) * kCFX + nx - 1); nq = (qs & 0xffffu) - (qs >> 16)) {
        DTS_COUNT(27, 1);
        const int take = min(nq, 32);
        __syncwarp();   // the entries were written by other lanes
        unsigned qw[4] = {0u, 0u, 0u, 0u};   // (lanes without an entry: one winner, nothing to shade)
        float q3[3] = {0.f, 0.f, 0.f};
        AuxPx qpix{};
        unsigned qslot = 0u;
        int qx = 0, qy = 0;
        if (lane < take) {
          const int e = ((qs >> 16) + lane) & (kEdgeQ - 1);
          const uint4 a = q[0][e], c = q[1][e];
          qslot = (kAux & kAuxMarks) ? a.x & 0xffffu : a.x; qx = (int)a.y; qy = (int)a.z;
          if (kAux & kAuxMarks) qpix.mk = (int)(a.x >> 16);
          qw[0] = a.w & 0xffffu; qw[1] = a.w >> 16; qw[2] = c.x & 0xffffu; qw[3] = c.x >> 16;
          q3[0] = __uint_as_float(c.y); q3[1] = __uint_as_float(c.z); q3[2] = __uint_as_float(c.w);
          if (needs_qq(kAux)) qpix.qmax = q_qq[e];
          if (takes_winner(kAux) && qw[0] != kNoPrim) qpix.lab = label_of(qw[0]);
        }
        resolve_edge<kAux>(qw, q3, clr, prims, tex_pool, lat_tab, qx, qy, lane, err, qpix, label_of, cls_pool);
        if (lane < take) rgb_buf[qslot] = pack_rgb(q3[0], q3[1], q3[2]);
        // the queued pixel `qslot` = fine bin * 32 + lane-in-bin: its images go straight to the frames (queued pixels
        // have a source)
        if (lane < take)
          store_aux<kAux>(af, depth_of(qpix.qmax), qpix.lab, qpix.mk, (int)(qslot & 31u), cbx * kCFX + (int)((qslot >> 5) & 3u),
                          cby * kCFY + (int)(qslot >> 7), W, H);
        qs += (unsigned)take << 16;
        __syncwarp();   // read before the next fine bin's entries overwrite the ring
      }
    }
    if (f < kCFX * kCFY) continue;   // handed back
    __syncwarp();   // queued pixels' colours were written by other lanes
    const StoreLane sl = make_store_lane(lane, W);   // (made here: held across the bin it would cost registers)
#pragma unroll 1
    for (int f = 0; f < kCFX * kCFY; f++) {
      if ((f & 3) >= nx || (f >> 2) >= ny) continue;
      store_bin(out, sl, rgb_buf[f * 32 + lane], lane, cbx * kCFX + (f & 3), cby * kCFY + (f >> 2), W, H);
    }
  }
}

// ------------------------------------------------------------------------------------------------ the renderer
static void free_remap(RemapTab& t) {
  const void* p[] = {t.src_xy, t.cbox, t.fbox, t.cell_start, t.cell_bins, t.home_start, t.home_ent, t.table_of_env, t.fwd};
  for (const void* q : p) cudaFree(const_cast<void*>(q));
  t = RemapTab{};
}

void renderer_release_frame(Renderer& r) {
  cudaFree(r.frame);
  r.frame = nullptr;
}

void renderer_destroy(Renderer* r) {
  if (r) { renderer_release_frame(*r); free_remap(r->fish); free_remap(r->rect); }
  delete r;
}

std::string renderer_prepare(Renderer& r, const std::vector<MapCounts>& counts, int mode, bool forward) {
  if (!r.frame) {
    // prims k_geometry emits per road tile: the literal triangles of tile mode 0, or the quad of tile mode 1, which a
    // clip splits into two triangles and fans into a few more
    const int tile_prims = (r.flags & DTS_FLAG_TESSELLATE) ? kTessTris : 6;
    long long max_tris = 2;
    int max_lat = 1, items_max = 1;
    for (const MapCounts& m : counts) {
      if (!m.n_tiles) continue;   // an empty slot
      const long long t = 2 + (long long)tile_prims * m.n_tiles + m.n_tris;   // the ground quad's two triangles, the tiles, the meshes
      max_tris = std::max(max_tris, t);
      max_lat = std::max(max_lat, m.n_tiles);
      items_max = std::max(items_max, agent_item(m.n_tiles, m.n_objects) + 1);
    }
    const long long max_prims = max_tris + max_tris / 4 + 64;   // clipping can add fan triangles
    if (items_max > 65535) return "scene too large: " + std::to_string(items_max) + " draw items per frame (limit 65535)";
    if (max_prims > 65535) return "scene too large: " + std::to_string(max_prims) + " triangles per frame (limit 65535)";
    // (prim, coarse bin) pairs k_bin emits per env at most: the ground fan (<= 8 x cbins), a few screen-filling tiles
    // and one screen-filling prop; under the fused fisheye the bins are overlapping source boxes (x ~4).  The batch
    // shares ONE pool, each env taking exactly what its frame needs: capacity = that bound x num_envs, capped at
    // DTS_PAIR_POOL_GB (default 16) of pairs and records — a typical frame uses a small fraction of its bound.
    const long long per_env = (3LL * max_prims + 24LL * r.cbins + 256) * ((r.flags & DTS_FLAG_DISTORTION) ? 4 : 1);
    double pool_gb = 16.0;
    if (const char* e = getenv("DTS_PAIR_POOL_GB")) pool_gb = atof(e) > 0 ? atof(e) : pool_gb;
    const long long cap = (long long)(pool_gb * 1073741824.0 / (double)(sizeof(uint32_t) + sizeof(BinRec)));
    const long long pool = std::max(std::min({per_env * r.n, cap, 2000000000LL}), per_env);
    r.max_prims = (int)max_prims; r.max_lat = max_lat; r.items_max = items_max; r.pool = (int)pool;
    const size_t bytes = carve(r, 0, r.fm);
    const cudaError_t e = cudaMalloc(&r.frame, bytes);
    if (e != cudaSuccess) {
      r.frame = nullptr;
      return "render scratch cudaMalloc(" + std::to_string(bytes) + ") failed: " + cudaGetErrorString(e);
    }
    carve(r, reinterpret_cast<uintptr_t>(r.frame), r.fm);
  }
  if ((r.flags & DTS_FLAG_DISTORTION) && !r.fish.src_xy) return "distortion enabled but no fisheye LUT set";
  if ((mode & DTS_RENDER_RECTIFY) && !r.rect.src_xy) return "DTS_RENDER_RECTIFY but no rectification LUT set";
  if (forward && (r.flags & DTS_FLAG_DISTORTION) && !(mode & (DTS_RENDER_PINHOLE | DTS_RENDER_RECTIFY)) && !r.fish.fwd)
    return "a flow, bird's-eye visibility, object or lane path target is set but the fisheye tables have no forward maps: "
           "a fisheye LUT set after dts_set_flow_target / dts_set_bev_visibility_target / dts_set_object_target / "
           "dts_set_lane_path_target drops them, so set that target again";
  return "";
}

std::string renderer_set_flow_maps(Renderer& r, int count, const float* fwd_x, const float* fwd_y) {
  if (!fwd_x || !fwd_y) {
    cudaFree(const_cast<float2*>(r.fish.fwd));
    r.fish.fwd = nullptr;
    return "";
  }
  if (!r.fish.src_xy || count != r.fish.count)
    return "the flow image's forward maps are " + std::to_string(count) + " tables but the fisheye pool holds " +
           std::to_string(r.fish.src_xy ? r.fish.count : 0);
  const size_t n = (size_t)count * r.W * r.H;
  std::vector<float2> f(n);
  for (size_t k = 0; k < n; k++) f[k] = make_float2(fwd_x[k], fwd_y[k]);
  void* d = nullptr;
  cudaError_t e = cudaMalloc(&d, n * sizeof(float2));
  if (e == cudaSuccess) e = cudaMemcpy(d, f.data(), n * sizeof(float2), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d);
    return std::string("flow forward map upload failed: ") + cudaGetErrorString(e);
  }
  cudaFree(const_cast<float2*>(r.fish.fwd));
  r.fish.fwd = static_cast<const float2*>(d);
  return "";
}

std::string renderer_set_lut(Renderer& r, bool rectify, int count, const float* rmapx, const float* rmapy,
                             const int32_t* lut_of_env) {
  // distortion.py:118 gathers img[rint(rmapy), rint(rmapx)], UndistortWrapper (wrappers.py:227) the same with its own
  // map.  The rasteriser renders those source pixels directly: per output pixel the source position, per fine / coarse
  // output bin the bounding box of its source pixels (the bins prims are sorted into).
  RemapTab& slot = rectify ? r.rect : r.fish;
  const char* what = rectify ? "rectification LUT" : "fisheye LUT";
  if (!rmapx || !rmapy) {
    free_remap(slot);
    return "";
  }
  const int W = r.W, H = r.H, cbx_n = (W + kCoarseW - 1) / kCoarseW, cbins = r.cbins;
  const size_t px = (size_t)W * H;
  // the tables of a pool, concatenated (RemapTab): every per-table array is appended, so that the CSR starts pushed below
  // are positions in the concatenated lists
  std::vector<int32_t> src(px * count);
  const short4 empty = make_short4(32767, 32767, -32768, -32768);
  std::vector<short4> cbox((size_t)cbins * count, empty), fbox((size_t)cbins * count * kCFX * kCFY, empty);
  std::vector<int32_t> cell_start, home_start;
  std::vector<uint16_t> cell_bins;
  std::vector<int4> home_ent;   // with the box
  int ext_x = 0, ext_y = 0;
  auto grow = [](short4& b, int x, int y) {
    b.x = (short)(x < b.x ? x : b.x); b.y = (short)(y < b.y ? y : b.y);
    b.z = (short)(x > b.z ? x : b.z); b.w = (short)(y > b.w ? y : b.w);
  };
  for (int t = 0; t < count; t++) {
    const float* mx = rmapx + px * t;
    const float* my = rmapy + px * t;
    int32_t* tsrc = src.data() + px * t;
    short4* tcbox = cbox.data() + (size_t)cbins * t;
    short4* tfbox = fbox.data() + (size_t)cbins * t * kCFX * kCFY;
    const std::string name = count > 1 ? std::string(what) + " " + std::to_string(t) : std::string(what);
    for (int y = 0; y < H; y++)
      for (int x = 0; x < W; x++) {
        const float fx = mx[(size_t)y * W + x], fy = my[(size_t)y * W + x];
        // round half to even (numpy's rint); NaN, inf and huge entries are out of range before any float -> int conversion,
        // which would be undefined for them
        const bool finite = fabsf(fx) < 1073741824.0f && fabsf(fy) < 1073741824.0f;
        const int sx = finite ? (int)rintf(fx) : -1, sy = finite ? (int)rintf(fy) : -1;
        const bool ok = sx >= 0 && sx < W && sy >= 0 && sy < H;
        tsrc[(size_t)y * W + x] = ok ? (int32_t)((uint32_t)(sx & 0xffff) | ((uint32_t)sy << 16)) : (int32_t)0x80008000u;
        if (!ok) continue;
        const int cb = (y / kCoarseH) * cbx_n + x / kCoarseW, f = (y % kCoarseH / kBinH) * kCFX + x % kCoarseW / kBinW;
        grow(tcbox[cb], sx, sy); grow(tfbox[(size_t)cb * kCFX * kCFY + f], sx, sy);
      }
    // int32 edge functions inside a coarse bin need |A x + B y| < 2^30 over its source box, where (guard band) |A| <=
    // kEdge * H, |B| <= kEdge * W, x <= kSub * w, y <= kSub * h  ->  H * w + W * h < 2^30 / (kEdge * kSub)
    constexpr long long kEdge = (long long)(kGuard + 1) * kSub;
    for (int b = 0; b < cbins; b++) {
      if (tcbox[b].z < tcbox[b].x) continue;
      const long long w = tcbox[b].z - tcbox[b].x + 2, h = tcbox[b].w - tcbox[b].y + 2;
      if ((long long)H * w + (long long)W * h >= (1LL << 30) / (kEdge * kSub))
        return name + " sends output bin " + std::to_string(b) + " to a " + std::to_string(w) + "x" + std::to_string(h) +
               " px source region: too wide for the rasteriser's int32 edge functions";
    }
    // two inverse indices over source cells (the coarse grid laid over the source image): per cell, the output bins whose
    // source box meets it, and the output bins whose box has its top-left corner there, each bin under one HOME cell
    std::vector<std::vector<int>> meets(cbins), homes(cbins);
    for (int b = 0; b < cbins; b++) {
      const short4 q = tcbox[b];
      if (q.z < q.x) continue;
      const int cx0 = q.x / kCoarseW, cy0 = q.y / kCoarseH, cx1 = q.z / kCoarseW, cy1 = q.w / kCoarseH;
      for (int cy = cy0; cy <= cy1; cy++)
        for (int cx = cx0; cx <= cx1; cx++) meets[cy * cbx_n + cx].push_back(b);
      homes[cy0 * cbx_n + cx0].push_back(b);
      ext_x = std::max(ext_x, cx1 - cx0);
      ext_y = std::max(ext_y, cy1 - cy0);
    }
    for (int c = 0; c < cbins; c++) {
      cell_start.push_back((int32_t)cell_bins.size());
      home_start.push_back((int32_t)home_ent.size());
      for (int b : meets[c]) cell_bins.push_back((uint16_t)b);
      for (int b : homes[c])
        home_ent.push_back(make_int4((int)((uint32_t)(uint16_t)tcbox[b].x | ((uint32_t)(uint16_t)tcbox[b].y << 16)),
                                     (int)((uint32_t)(uint16_t)tcbox[b].z | ((uint32_t)(uint16_t)tcbox[b].w << 16)), b, 0));
    }
    cell_start.push_back((int32_t)cell_bins.size());
    home_start.push_back((int32_t)home_ent.size());
  }
  if (cell_bins.empty()) cell_bins.push_back(0);
  if (home_ent.empty()) home_ent.push_back(make_int4(0, 0, 0, 0));
  std::vector<uint16_t> tab;
  if (count > 1)
    for (int e = 0; e < r.n; e++) tab.push_back((uint16_t)lut_of_env[e]);
  RemapTab t{};
  cudaError_t e = cudaSuccess;
  auto upload = [&](auto& dst, const auto& v) {
    void* d = nullptr;
    if (e == cudaSuccess) e = cudaMalloc(&d, v.size() * sizeof(v[0]));
    if (e != cudaSuccess) return;
    dst = reinterpret_cast<std::remove_reference_t<decltype(dst)>>(d);
    e = cudaMemcpy(d, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
  };
  upload(t.src_xy, src); upload(t.cbox, cbox); upload(t.fbox, fbox);
  upload(t.cell_start, cell_start); upload(t.cell_bins, cell_bins);
  upload(t.home_start, home_start); upload(t.home_ent, home_ent);
  if (!tab.empty()) upload(t.table_of_env, tab);
  if (e != cudaSuccess) {
    free_remap(t);
    return std::string(what) + " table upload failed: " + cudaGetErrorString(e);
  }
  t.ext_x = ext_x; t.ext_y = ext_y; t.count = count;
  free_remap(slot);
  slot = t;
  return "";
}

const FrameCtx* renderer_frame_ctx(const Renderer& r) { return r.frame ? r.fm.ctx : nullptr; }

// the table a render in `mode` is remapped through, if any: the rectification (DTS_RENDER_RECTIFY), none
// (DTS_RENDER_PINHOLE or no DTS_FLAG_DISTORTION) or the fisheye
static const RemapTab* remap_of(const Renderer& r, int flags, int mode) {
  return (mode & DTS_RENDER_RECTIFY) ? &r.rect
       : ((flags & DTS_FLAG_DISTORTION) && !(mode & DTS_RENDER_PINHOLE)) ? &r.fish : nullptr;
}

FlowRemap renderer_remap(const Renderer& r, int mode) {
  const RemapTab* lut = remap_of(r, r.flags, mode);
  const RemapTab rt = lut ? *lut : RemapTab{};
  return FlowRemap{rt.src_xy, rt.table_of_env, rt.fwd, (mode & DTS_RENDER_RECTIFY) != 0};
}

// Test hook (dts_debug_frame): what k_frame_setup / k_geometry left in frame memory for one env of the last render —
// the camera model-view and projection, the prim / lattice counts, and the lit 8x8 lattice of every road tile that
// was emitted, re-ordered by grid cell (i * grid_h + j; cells that were culled stay NaN).
std::string debug_frame_copy(const Renderer& r, int env, double* V, float* P, int32_t* counts, float* lattice_by_cell,
                             int n_cells) {
  if (!r.frame) return "nothing rendered yet";
  if (r.flags & DTS_FLAG_TESSELLATE) return "dts_debug_frame reads the analytic-tile lattice (tile mode 1)";
  const FrameMem& fm = r.fm;
  const int max_prims = r.max_prims, max_lat = r.max_lat, tris_per_tile = tile_draw_ids(false);
  FrameCtx c;
  if (cudaMemcpy(&c, fm.ctx + env, sizeof c, cudaMemcpyDeviceToHost) != cudaSuccess) return "debug_frame_copy failed";
  for (int k = 0; k < 12; k++) V[k] = c.V[k];
  P[0] = c.P00; P[1] = c.P11; P[2] = c.P22; P[3] = c.P23;
  counts[0] = c.n_prims; counts[1] = c.n_lat; counts[2] = c.overflow; counts[3] = 0;
  cudaMemcpy(&counts[3], fm.work + kWorkPairPool, sizeof(int32_t), cudaMemcpyDeviceToHost);   // (prim, coarse bin) pairs of the whole batch
  const int np = c.n_prims < max_prims ? c.n_prims : max_prims;
  std::vector<PrimRec> prims(np > 0 ? np : 1);
  std::vector<float4> lat((size_t)max_lat * 64);
  int rc = 0;
  if (np && cudaMemcpy(prims.data(), fm.prims + (size_t)env * max_prims, (size_t)np * sizeof(PrimRec), cudaMemcpyDeviceToHost) != cudaSuccess) rc = 1;
  if (cudaMemcpy(lat.data(), fm.lat + (size_t)env * max_lat * 64, (size_t)max_lat * 64 * sizeof(float4), cudaMemcpyDeviceToHost) != cudaSuccess) rc = 1;
  for (int k = 0; k < n_cells * 64 * 3; k++) lattice_by_cell[k] = nanf("");
  for (int p = 0; p < np && !rc; p++) {
    const int slot = (prims[p].ltq & 0xffff) - 1;
    if (slot < 0 || slot >= max_lat) continue;
    const int cell = (prims[p].id - 2) / tris_per_tile;   // tiles are drawn i outer, j inner: cell = i * grid_h + j
    if (cell < 0 || cell >= n_cells) continue;
    for (int v = 0; v < 64; v++) {
      lattice_by_cell[(cell * 64 + v) * 3 + 0] = lat[slot * 64 + v].x;
      lattice_by_cell[(cell * 64 + v) * 3 + 1] = lat[slot * 64 + v].y;
      lattice_by_cell[(cell * 64 + v) * 3 + 2] = lat[slot * 64 + v].z;
    }
  }
  return rc ? "debug_frame_copy failed" : "";
}

// The image sets the rasterisers are compiled for.  Depth + markings has none of its own: it runs the marking instance,
// which stores the depth where that target is set.
constexpr int kAuxSets[] = {0, kAuxDepth, kAuxLabels, kAuxDepth | kAuxLabels, kAuxMarks, kAuxLabels | kAuxMarks};
// The image set a render with these targets runs
static int aux_set(const AuxTargets& a) {
  return (a.labels ? kAuxLabels : 0) | (a.marks ? kAuxMarks : a.depth ? kAuxDepth : 0);
}
// The remap modes k_bin and the rasterisers are compiled for
constexpr int kRemapModes[] = {kRemapNone, kRemapTable, kRemapPool};
// f(std::integral_constant<int, v>{}) for every value v of kList (kAuxSets, kRemapModes)
template <const auto& kList, typename F, size_t... I>
static void each_of(F& f, std::index_sequence<I...>) { (f(std::integral_constant<int, kList[I]>{}), ...); }
template <const auto& kList, typename F>
static void for_each_of(F f) { each_of<kList>(f, std::make_index_sequence<std::size(kList)>{}); }

int launch_render(const Renderer& r, const DState& S, const DMap* maps, const RenderCfg& rc, const AuxTargets& aux,
                  const FlowTarget& flow, const OcclusionTarget& occ, void* obs_any, const GatherTab& gather, int32_t* err_flag, int32_t* status_dev,
                  cudaEvent_t* marks, int mark_level, cudaStream_t st) {
  uint8_t* obs = reinterpret_cast<uint8_t*>(obs_any);
  // the table the frame is remapped through, if any.  A table with a per-env index is a pool (kRemapPool); one table,
  // of either kind, is kRemapTable.
  const RemapTab* lut = remap_of(r, rc.flags, rc.mode);
  const RemapTab rt = lut ? *lut : RemapTab{};
  const int remap = !lut ? kRemapNone : rt.table_of_env ? kRemapPool : kRemapTable;
  FrameMem fm = r.fm;
  fm.status = status_dev;
  int mk = 0;
  // level 2: an event at every kernel boundary; level 1: only the two around k_raster (marks 3 and 4), so that the
  // timed region of a benchmark carries two event records per step instead of six
  auto mark = [&]() { if (marks && (mark_level >= 2 || mk == 3 || mk == 4)) cudaEventRecord(marks[mk], st); mk++; };
  cudaMemsetAsync(fm.work, 0, 256, st);
  mark();
  k_frame_setup<<<(rc.n_envs + 127) / 128, 128, 0, st>>>(S, maps, rc, fm);
  mark();
  const size_t pairs_total = (size_t)rc.n_envs * r.items_max;
  k_cull<<<(unsigned)((pairs_total + 255) / 256), 256, 0, st>>>(S, maps, rc, fm, r.items_max, err_flag);
  int launches = 7;
  if (!rc.tessellate) {   // (inside the k_geometry event bracket: it is geometry time)
    k_tiles<<<(rc.n_envs + kTileWarps - 1) / kTileWarps, kTileWarps * 32, 0, st>>>(S, maps, rc, fm, r.max_prims, r.max_lat, err_flag);
    launches++;
  }
  const auto geometry = rc.tessellate ? k_geometry<true> : k_geometry<false>;
  geometry<<<r.sms * kGeoMinCtas / kGeoWarps, kGeoWarps * 32, 0, st>>>(S, maps, rc, fm, r.max_prims, err_flag);
  mark();
  // (at most 20 KB: dts_create caps the camera at 800x800, 2,500 coarse bins, so no opt-in past 48 KB is needed)
  const size_t bin_smem_bytes = (size_t)2 * r.cbins * sizeof(int);
  const int bin_grid = rc.n_envs;   // CTA per env: one warp where a frame has few bins and prims (160x120: 75 bins — more warps
  // only add barriers and CTA launches), four for large cameras (640x480)
  const int bin_threads = r.cbins > 128 ? kBinWarps * 32 : 32;
  for_each_of<kRemapModes>([&](auto remap_c) {
    constexpr int R = decltype(remap_c)::value;
    if (R != remap) return;
    const auto bin = rc.env_list ? k_bin<R, true> : k_bin<R, false>;
    bin<<<bin_grid, bin_threads, bin_smem_bytes, st>>>(rc, fm, rt, r.max_prims, r.pool, err_flag);
  });
  mark();
  const int aux_run = aux_set(aux);   // the rasterisers' instances for the images asked for (no target: the plain ones)
  for_each_of<kAuxSets>([&](auto aux_c) {
    for_each_of<kRemapModes>([&](auto remap_c) {
      constexpr int A = decltype(aux_c)::value, R = decltype(remap_c)::value;
      if (A != aux_run || R != remap) return;
      // (all three inside the k_raster event bracket: it is rasterisation time)
      k_raster_solo<R, A><<<r.sms * kSoloMinCtas, kThreads, 0, st>>>(S, maps, rc, fm, rt, obs, r.max_prims, r.max_lat, aux);
      // before k_raster, which draws the bins k_raster_flat hands back
      k_raster_flat<R, A><<<r.sms * kFlatMinCtas, kThreads, 0, st>>>(S, maps, rc, fm, rt, obs, r.max_prims, r.max_lat,
                                                                      err_flag, aux);
      k_raster<R, A><<<r.sms * kRasterMinCtas, kThreads, kRasterSmem, st>>>(S, maps, rc, fm, rt, gather, obs, r.max_prims,
                                                                            r.pool, r.max_lat, err_flag, aux);
    });
  });
  mark();
  if (flow.out) {   // (inside the post-pass event bracket)
    launches += launch_flow(S, maps, rc, fm.ctx, aux, flow, renderer_remap(r, rc.mode), occ, st);
  }
  mark();   // (post passes: launched by the caller)
  return launches;
}

// (after launch_render: instantiated before k_bin, k_raster would move k_bin's dynamic shared memory from offset 16 to 128)
Renderer* renderer_create(const dts_config& cfg) {
  Renderer* r = new Renderer();
  r->n = cfg.num_envs; r->W = cfg.cam_width; r->H = cfg.cam_height; r->flags = cfg.flags;
  r->sms = 132;
  cudaDeviceGetAttribute(&r->sms, cudaDevAttrMultiProcessorCount, cfg.device);
  r->cbins = ((r->W + kCoarseW - 1) / kCoarseW) * ((r->H + kCoarseH - 1) / kCoarseH);
  // k_raster's shared memory is past the 48 KB default; the opt-in holds for the kernel as loaded on this device
  for_each_of<kAuxSets>([](auto aux_c) {
    for_each_of<kRemapModes>([&](auto remap_c) {
      constexpr int A = decltype(aux_c)::value, R = decltype(remap_c)::value;
      cudaFuncSetAttribute(k_raster<R, A>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRasterSmem);
    });
  });
  return r;
}

}  // namespace dts
