// dts_bev.cu — the bird's-eye map (dts_set_bev_target, DESIGN.md section 5 item 12): a grid of cells fixed to every
// agent, each point-sampled from the map's own tables at its centre — the tile under it, the class of the texel under it
// and the first object whose footprint holds it.  No rasteriser: a thread per cell, float64 in the order the spec states
// (-fmad=false keeps every product and sum separately rounded, as numpy's are).  k_bev_view then says, cell by cell,
// whether the frame the call drew shows the grid (dts_set_bev_visibility_target, item 15).  k_scan casts the range scan
// (dts_set_scan_target, item 16) from the same footprints and the reference's drivability rule.
#include "dts_camera.cuh"
#include "dts_kernels.h"
#include "dts_logic.cuh"

namespace dts {
namespace {

constexpr int kBevThreads = 256;
constexpr int kBevCellsPerThread = 4;   // cells per CTA = 1024: a 64 x 64 grid is four CTAs per env
constexpr int kBevCellsPerCta = kBevThreads * kBevCellsPerThread;

struct BevFootprint { double x[4], z[4]; };

// (b - a) x (p - a)
__device__ __forceinline__ double edge_cross(double ax, double az, double bx, double bz, double px, double pz) {
  return (bx - ax) * (pz - az) - (bz - az) * (px - ax);
}

// the four cross products (c[k+1] - c[k]) x (p - c[k]) all >= 0 or all <= 0
__device__ __forceinline__ bool footprint_holds(const BevFootprint& q, double px, double pz) {
  bool pos = true, neg = true;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int n = (k + 1) & 3;
    const double c = edge_cross(q.x[k], q.z[k], q.x[n], q.z[n], px, pz);
    pos &= c >= 0.0;
    neg &= c <= 0.0;
  }
  return pos || neg;
}

// A strictly convex quad holds exactly its own closed area, up to the rounding of the cross products, so none of its
// points lies outside the corners' box widened by `margin`: cells and objects outside it are skipped without changing
// the result.  Any other quad (degenerate: its rule can hold points outside it) gets an unbounded box.
__device__ __forceinline__ void footprint_box(const BevFootprint& q, double box[4]) {
  bool pos = true, neg = true;
  double x0 = q.x[0], x1 = q.x[0], z0 = q.z[0], z1 = q.z[0];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int n = (k + 1) & 3, n2 = (k + 2) & 3;
    const double t = edge_cross(q.x[k], q.z[k], q.x[n], q.z[n], q.x[n2], q.z[n2]);
    pos &= t > 0.0;
    neg &= t < 0.0;
    x0 = fmin(x0, q.x[k]); x1 = fmax(x1, q.x[k]);
    z0 = fmin(z0, q.z[k]); z1 = fmax(z1, q.z[k]);
  }
  const double margin = 1e-9 * (1.0 + fmax(fmax(fabs(x0), fabs(x1)), fmax(fabs(z0), fabs(z1))));
  const bool bounded = pos || neg;
  box[0] = bounded ? x0 - margin : -INFINITY; box[1] = bounded ? x1 + margin : INFINITY;
  box[2] = bounded ? z0 - margin : -INFINITY; box[3] = bounded ? z1 + margin : INFINITY;
}

// Can a footprint with this box hold a point of the disc (wx, wz, wr)?  (The disc's own rounding is covered by a margin.)
__device__ __forceinline__ bool box_meets(const double box[4], double wx, double wz, double wr) {
  const double m = wr + 1e-9 * (1.0 + fabs(wx) + fabs(wz) + wr);
  return box[0] <= wx + m && box[1] >= wx - m && box[2] <= wz + m && box[3] >= wz - m;
}

// Called by one whole warp: the footprints of env `env`'s objects that are not hidden this episode and whose box meets
// the disc (wx, wz, wr), in index order, into foot / foot_box / foot_obj, which have room for every object of the map.
// Returns how many, on every lane.
__device__ __forceinline__ int gather_footprints(const DState& S, const DMap& m, int env, int lane, double wx, double wz,
                                                 double wr, BevFootprint* foot, double (*foot_box)[4], int16_t* foot_obj) {
  int count = 0;
  const uint32_t* hidden = S.rep[env].hidden;
  const size_t nd = m.n_dyn, ne = S.n;
  for (int base = 0; base < m.n_objects; base += 32) {
    const int o = base + lane;
    BevFootprint q;
    double box[4];
    bool keep = false;
    if (o < m.n_objects && !(hidden[o >> 5] >> (o & 31) & 1u)) {
      keep = object_footprint(m, nd, ne, env, o, q.x, q.z);
      if (keep) footprint_box(q, box);
      keep = keep && box_meets(box, wx, wz, wr);
    }
    const unsigned ball = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int at = count + __popc(ball & ((1u << lane) - 1u));
      foot[at] = q;
      for (int k = 0; k < 4; k++) foot_box[at][k] = box[k];
      foot_obj[at] = (int16_t)o;
    }
    count += __popc(ball);
  }
  return count;
}

// grid (env, chunk of kBevCellsPerCta cells), one thread per cell of the chunk at a time, rows stored contiguously
__global__ void __launch_bounds__(kBevThreads) k_bev(DState S, const DMap* __restrict__ maps, BevTarget b) {
  __shared__ BevFootprint foot[DTS_MAX_OBJECTS];   // the objects whose footprint can meet the window, in index order
  __shared__ double foot_box[DTS_MAX_OBJECTS][4];   // x0 x1 z0 z1 outside which the footprint holds no point
  __shared__ int16_t foot_obj[DTS_MAX_OBJECTS];     // (room for every object a map may have: no fallback is needed)
  __shared__ int n_foot;
  __shared__ double pose[4];                        // pos_x, pos_z, cos, sin of the env's angle
  const int env = blockIdx.x;
  const DMap& m = maps[S.map_id[env]];
  const dts_bev_config g = b.cfg;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    const double px = S.pos_x[env], pz = S.pos_z[env];
    double sa, ca;
    sincos(S.angle[env], &sa, &ca);
    if (lane == 0) { pose[0] = px; pose[1] = pz; pose[2] = ca; pose[3] = sa; }
    int count = 0;
    if (b.labels) {
      // the window's bounding disc: the grid's middle, half its diagonal
      const double fc = (g.origin_y - 0.5 * g.height) * g.cell, lc = (0.5 * g.width - g.origin_x) * g.cell;
      const double wx = px + fc * ca + lc * sa, wz = pz - fc * sa + lc * ca;
      const double wr = 0.5 * g.cell * sqrt((double)g.width * g.width + (double)g.height * g.height);
      count = gather_footprints(S, m, env, lane, wx, wz, wr, foot, foot_box, foot_obj);
    }
    if (lane == 0) n_foot = count;
  }
  __syncthreads();
  const double px = pose[0], pz = pose[1], ca = pose[2], sa = pose[3];
  const double ts = m.tile_size;
  const int gw = m.grid_w, gh = m.grid_h, n_foot_env = n_foot;
  const int n_cells = g.width * g.height;
  const size_t row = (size_t)env * n_cells;
  const uint8_t* cls_pool = m.tex_pool + m.tex_class_off;
  for (int k = 0; k < kBevCellsPerThread; k++) {
    const int t = blockIdx.y * kBevCellsPerCta + k * kBevThreads + threadIdx.x;
    if (t >= n_cells) break;
    const int r = t / g.width, c = t - r * g.width;
    const double f = (g.origin_y - (r + 0.5)) * g.cell, l = ((c + 0.5) - g.origin_x) * g.cell;
    const double x = px + f * ca + l * sa, z = pz - f * sa + l * ca;
    int label = 1, mark = 0;
    const double fi = floor(x / ts), fj = floor(z / ts);   // get_grid_coords S:1134, compared before any int conversion
    if (fi >= 0.0 && fi < gw && fj >= 0.0 && fj < gh) {
      const int i = (int)fi, j = (int)fj, idx = j * gw + i;
      if (__ldg(m.tile_kind + idx) >= 0) {
        label = 2 + i * gh + j;
        const int tex = __ldg(m.tile_tex + idx);
        if (b.marks && tex >= 0) {
          // tile-local point: T((i + .5) ts, 0, (j + .5) ts) Ry(angle * 90 + 180) inverted, its cos / sin exact 0 / +-1
          const double lx = x - (i + 0.5) * ts, lz = z - (j + 0.5) * ts;
          const int q = (__ldg(m.tile_angle + idx) + 2) & 3;
          const double ax = q == 0 ? lx : q == 1 ? -lz : q == 2 ? -lx : lz;
          const double az = q == 0 ? lz : q == 1 ? lx : q == 2 ? -lz : -lx;
          const double u = (ax + 0.5 * ts) / ts, v = 1.0 - (az + 0.5 * ts) / ts;   // _init_vlists S:394-401
          const int tw = __ldg(&m.textures[tex].w), th = __ldg(&m.textures[tex].h);
          const uint32_t info = __ldg(&m.textures[tex].info);
          const int tu = (int)floor(u * tw) & (tw - 1), tv = (int)floor(v * th) & (th - 1);   // power-of-two sides
          mark = __ldg(cls_pool + ((size_t)(info & 0xffffffu) << 6) + (size_t)tv * tw + tu);
        }
      }
    }
    if (b.labels) {
      for (int s = 0; s < n_foot_env; s++) {
        if (x < foot_box[s][0] || x > foot_box[s][1] || z < foot_box[s][2] || z > foot_box[s][3]) continue;
        if (footprint_holds(foot[s], x, z)) { label = 2 + m.n_tiles + foot_obj[s]; break; }
      }
      b.labels[row + t] = (int16_t)label;
    }
    if (b.marks) b.marks[row + t] = (uint8_t)mark;
  }
}

constexpr int kScanThreads = 256;          // the most threads of a CTA, and the most rays of one env it casts
constexpr int kScanMaxEnvs = 32;           // the most envs of a CTA
constexpr int kScanSmem = 40 * 1024;       // the most bytes of gathered footprints a CTA holds

// The shared memory of one env's gathered footprints, in doubles: foot[cap], foot_box[cap][4], foot_obj[cap]
__host__ __device__ __forceinline__ int scan_slot_doubles(int cap) { return cap * 12 + (cap + 3) / 4; }

// Where ray (ox, oz) + t (dx, dz), t >= 0, enters the strictly convex footprint q (its four edge half-planes, Cyrus-Beck,
// the side taken from the corners' orientation): max(t_in, 0) where t_in <= t_out and t_out >= 0, else INFINITY.
__device__ __forceinline__ double footprint_entry(const BevFootprint& q, double ox, double oz, double dx, double dz) {
  const double side = edge_cross(q.x[0], q.z[0], q.x[1], q.z[1], q.x[2], q.z[2]) > 0.0 ? 1.0 : -1.0;
  double t0 = -INFINITY, t1 = INFINITY;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int n = (k + 1) & 3;
    const double num = side * edge_cross(q.x[k], q.z[k], q.x[n], q.z[n], ox, oz);   // inside: num + t den >= 0
    const double den = side * ((q.x[n] - q.x[k]) * dz - (q.z[n] - q.z[k]) * dx);
    if (den > 0.0) t0 = fmax(t0, -num / den);
    else if (den < 0.0) t1 = fmin(t1, -num / den);
    else if (num < 0.0) t1 = -INFINITY;   // parallel to the edge, outside it
  }
  return t0 <= t1 && t1 >= 0.0 ? fmax(t0, 0.0) : INFINITY;
}

// grid (CTAs of `envs` consecutive envs, chunks of kScanThreads rays): thread (slot, k) casts ray k of env
// blockIdx.x * envs + slot, its rays stored contiguously.  A warp gathers each env's footprints within max_range of
// the origin once, into `cap` entries of dynamic shared memory per env (cap: the most objects of an uploaded map).
__global__ void __launch_bounds__(kScanThreads) k_scan(DState S, const DMap* __restrict__ maps, ScanTarget sc, int cap,
                                                       int envs) {
  extern __shared__ double scan_mem[];
  __shared__ double origin[kScanMaxEnvs][2];
  __shared__ int n_foot[kScanMaxEnvs];
  const dts_scan_config g = sc.cfg;
  const int R = g.n_rays, per = R < kScanThreads ? R : kScanThreads;
  const int stride = scan_slot_doubles(cap);
  const int lane = threadIdx.x & 31;
  for (int s = threadIdx.x >> 5; s < envs; s += blockDim.x >> 5) {
    const int env = blockIdx.x * envs + s;
    if (env >= S.n) break;
    const DMap& m = maps[S.map_id[env]];
    double sa, ca;
    sincos(S.angle[env], &sa, &ca);
    const double f = g.origin_forward, r = g.origin_right;
    const double ox = S.pos_x[env] + f * ca + r * sa, oz = S.pos_z[env] - f * sa + r * ca;
    double* slot = scan_mem + (size_t)s * stride;
    const int count = gather_footprints(S, m, env, lane, ox, oz, g.max_range, reinterpret_cast<BevFootprint*>(slot),
                                        reinterpret_cast<double(*)[4]>(slot + cap * 8),
                                        reinterpret_cast<int16_t*>(slot + cap * 12));
    if (lane == 0) { origin[s][0] = ox; origin[s][1] = oz; n_foot[s] = count; }
  }
  __syncthreads();
  const int s = threadIdx.x / per, k = blockIdx.y * per + (threadIdx.x - s * per);
  const int env = blockIdx.x * envs + s;
  if (s >= envs || env >= S.n || k >= R) return;
  const DMap& m = maps[S.map_id[env]];
  const double* slot = scan_mem + (size_t)s * stride;
  const BevFootprint* foot = reinterpret_cast<const BevFootprint*>(slot);
  const double(*foot_box)[4] = reinterpret_cast<const double(*)[4]>(slot + cap * 8);
  const int16_t* foot_obj = reinterpret_cast<const int16_t*>(slot + cap * 12);
  const double ox = origin[s][0], oz = origin[s][1];
  double sd, cd;
  sincos(S.angle[env] + g.fov * (0.5 - (k + 0.5) / R), &sd, &cd);
  const double dx = cd, dz = -sd;   // get_dir_vec
  // objects: the first footprint entered, the smallest index among equals
  double t_obj = INFINITY;
  int hit = 0;
  for (int q = 0, n = n_foot[s]; q < n; q++) {
    if (foot_box[q][0] == -INFINITY) continue;   // not strictly convex: stops no ray
    const double t = footprint_entry(foot[q], ox, oz, dx, dz);
    if (t < t_obj) { t_obj = t; hit = 2 + m.n_tiles + foot_obj[q]; }
  }
  // tiles: the cells the ray crosses, from the origin's, up to the first that is not drivable (_drivable_pos S:1411);
  // it leaves the grid within grid_w + grid_h steps, and off the grid nothing is drivable
  const double ts = m.tile_size, limit = fmin(t_obj, g.max_range);
  double fi = floor(ox / ts), fj = floor(oz / ts), t_tile = INFINITY;
  if (!drivable_at(m, ox, oz)) {
    t_tile = 0.0;
  } else {
    int i = (int)fi, j = (int)fj;
    const int si = dx > 0.0 ? 1 : -1, sj = dz > 0.0 ? 1 : -1;
    for (int step = 0; step < m.grid_w + m.grid_h + 2; step++) {
      const double tx = dx != 0.0 ? ((i + (si > 0)) * ts - ox) / dx : INFINITY;
      const double tz = dz != 0.0 ? ((j + (sj > 0)) * ts - oz) / dz : INFINITY;
      const double t = fmax(fmin(tx, tz), 0.0);
      if (t > limit) break;
      if (tx <= tz) i += si;
      if (tz <= tx) j += sj;
      if (!drivable_at(m, (i + 0.5) * ts, (j + 0.5) * ts)) { t_tile = t; fi = i; fj = j; break; }
    }
  }
  double t = t_obj;
  if (t_tile < t_obj) {   // an object wins a tie
    t = t_tile;
    const bool road = fi >= 0.0 && fi < m.grid_w && fj >= 0.0 && fj < m.grid_h &&
                      __ldg(m.tile_kind + (int)fj * m.grid_w + (int)fi) >= 0;
    hit = road ? 2 + (int)fi * m.grid_h + (int)fj : 1;
  }
  if (!(t <= g.max_range)) { t = g.max_range; hit = 0; }
  const size_t at = (size_t)env * R + k;
  if (sc.range) sc.range[at] = (float)t;
  if (sc.hit) sc.hit[at] = (int16_t)hit;
}

constexpr int kViewThreads = 256;
constexpr int kViewCellsPerThread = 4;
constexpr int kViewCellsPerCta = kViewThreads * kViewCellsPerThread;
constexpr double kGroundY = (double)(float)(-0.8 * 0.01);   // the ground quad's height (draw_ground, S:1805-1812)

// grid (env, chunk of kViewCellsPerCta cells), one thread per cell of the chunk at a time, rows stored contiguously.
// The cell centres are k_bev's, bit for bit, so a cell's surface (road tile or ground) is the one its label was taken on.
__global__ void __launch_bounds__(kViewThreads) k_bev_view(DState S, const DMap* __restrict__ maps, BevTarget b,
                                                           BevViewTarget v, const FrameCtx* __restrict__ ctx,
                                                           const int16_t* __restrict__ labels, int W, int H,
                                                           FlowRemap rm, bool drew) {
  __shared__ double cam[12];          // the frame's V
  __shared__ double pose[4];          // pos_x, pos_z, cos, sin of the env's angle
  __shared__ float proj[2];           // the frame's P00, P11
  __shared__ const float2* fwd;       // the env's forward map, null: the pinhole frame
  __shared__ bool known;              // a frame was drawn, not through the rectification
  const int env = blockIdx.x;
  if (threadIdx.x == 0) {
    double sa, ca;
    sincos(S.angle[env], &sa, &ca);
    pose[0] = S.pos_x[env]; pose[1] = S.pos_z[env]; pose[2] = ca; pose[3] = sa;
    known = drew && !rm.rectify;
    if (known) {
      const FrameCtx& c = ctx[env];
      for (int k = 0; k < 12; k++) cam[k] = c.V[k];
      proj[0] = c.P00; proj[1] = c.P11;
      fwd = rm.fwd ? rm.fwd + (size_t)(rm.table_of_env ? __ldg(rm.table_of_env + env) : 0) * W * H : nullptr;
    }
  }
  __syncthreads();
  const dts_bev_config g = b.cfg;
  const DMap& m = maps[S.map_id[env]];
  const double px = pose[0], pz = pose[1], ca = pose[2], sa = pose[3], ts = m.tile_size;
  const int gw = m.grid_w, gh = m.grid_h;
  const int n_cells = g.width * g.height;
  const size_t row = (size_t)env * n_cells;
  const int16_t* frame = labels + (size_t)env * W * H;
  const float nan = __int_as_float(0x7fc00000);
  for (int k = 0; k < kViewCellsPerThread; k++) {
    const int t = blockIdx.y * kViewCellsPerCta + k * kViewThreads + threadIdx.x;
    if (t >= n_cells) break;
    uint8_t val = DTS_BEVVIS_UNKNOWN;
    float2 pix = make_float2(nan, nan);
    if (known) {
      val = DTS_BEVVIS_OUTSIDE;
      const int r = t / g.width, c = t - r * g.width;
      const double f = (g.origin_y - (r + 0.5)) * g.cell, l = ((c + 0.5) - g.origin_x) * g.cell;
      const double x = px + f * ca + l * sa, z = pz - f * sa + l * ca;
      const double fi = floor(x / ts), fj = floor(z / ts);
      const bool road = fi >= 0.0 && fi < gw && fj >= 0.0 && fj < gh && __ldg(m.tile_kind + (int)fj * gw + (int)fi) >= 0;
      const double y = road ? 0.0 : kGroundY;
      const int lab = b.labels[row + t];
      const double ex = cam[0] * x + cam[1] * y + cam[2] * z + cam[3];
      const double ey = cam[4] * x + cam[5] * y + cam[6] * z + cam[7];
      const double w = -(cam[8] * x + cam[9] * y + cam[10] * z + cam[11]);
      if (w > 0.04 && w <= 100.0) {   // gluPerspective's near and far planes (S:1761)
        const double iw = 1.0 / w;
        double qx = ((double)proj[0] * (ex * iw) + 1.0) * (0.5 * W), qy = (1.0 - (double)proj[1] * (ey * iw)) * (0.5 * H);
        bool in = true;
        if (fwd) {
          float2 o;
          in = forward_map(fwd, W, H, (float)qx, (float)qy, o);
          qx = o.x; qy = o.y;
        }
        if (in && qx >= 0.0 && qx < W && qy >= 0.0 && qy < H) {
          const int cx = (int)floor(qx - 0.5), cy = (int)floor(qy - 0.5);
          bool seen = false, shown = false;
#pragma unroll
          for (int j = 0; j < 2; j++)
#pragma unroll
            for (int i = 0; i < 2; i++) {
              const int sx = cx + i, sy = cy + j;
              if (sx < 0 || sx >= W || sy < 0 || sy >= H) continue;
              const int s = __ldg(frame + sy * W + sx);
              seen |= s == lab;
              shown |= s != 0;
            }
          if (seen || shown) {
            val = seen ? DTS_BEVVIS_VISIBLE : DTS_BEVVIS_OCCLUDED;
            pix = make_float2((float)qx, (float)qy);
          }
        }
      }
    }
    if (v.vis) v.vis[row + t] = val;
    if (v.pix) v.pix[row + t] = pix;
  }
}

// thread per env: the camera k_frame_setup left in frame memory
__global__ void __launch_bounds__(128) k_frame_cameras(const FrameCtx* __restrict__ ctx, int n, double* V, float* P) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const FrameCtx& c = ctx[e];
  for (int k = 0; k < 12; k++) V[(size_t)e * 12 + k] = c.V[k];
  P[(size_t)e * 4] = c.P00; P[(size_t)e * 4 + 1] = c.P11; P[(size_t)e * 4 + 2] = c.P22; P[(size_t)e * 4 + 3] = c.P23;
}

}  // namespace

void launch_bev(const DState& S, const DMap* maps, const BevTarget& b, cudaStream_t st) {
  const int n_cells = b.cfg.width * b.cfg.height;
  const dim3 grid(S.n, (n_cells + kBevCellsPerCta - 1) / kBevCellsPerCta);
  k_bev<<<grid, kBevThreads, 0, st>>>(S, maps, b);
}

void launch_scan(const DState& S, const DMap* maps, const ScanTarget& sc, int max_objects, cudaStream_t st) {
  const int R = sc.cfg.n_rays, per = R < kScanThreads ? R : kScanThreads;
  const int cap = max_objects > 1 ? max_objects : 1;
  const size_t slot_bytes = sizeof(double) * scan_slot_doubles(cap);
  const int fit = (int)(kScanSmem / slot_bytes);   // >= 1: DTS_MAX_OBJECTS footprints take 25,088 B
  int envs = kScanThreads / per;
  if (envs > kScanMaxEnvs) envs = kScanMaxEnvs;
  if (envs > fit) envs = fit;
  const int threads = (envs * per + 31) / 32 * 32;
  const dim3 grid((S.n + envs - 1) / envs, (R + per - 1) / per);
  k_scan<<<grid, threads, envs * slot_bytes, st>>>(S, maps, sc, cap, envs);
}

void launch_bev_view(const DState& S, const DMap* maps, const BevTarget& b, const BevViewTarget& v, const FrameCtx* ctx,
                     const int16_t* labels, int W, int H, const FlowRemap& rm, bool drew_frame, cudaStream_t st) {
  const int n_cells = b.cfg.width * b.cfg.height;
  const dim3 grid(S.n, (n_cells + kViewCellsPerCta - 1) / kViewCellsPerCta);
  k_bev_view<<<grid, kViewThreads, 0, st>>>(S, maps, b, v, ctx, labels, W, H, rm, drew_frame);
}

void launch_frame_cameras(const FrameCtx* ctx, int n_envs, double* V, float* P, cudaStream_t st) {
  k_frame_cameras<<<(n_envs + 127) / 128, 128, 0, st>>>(ctx, n_envs, V, P);
}

}  // namespace dts
