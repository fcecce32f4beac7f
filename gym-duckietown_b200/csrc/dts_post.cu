// dts_post.cu — the passes over finished frames: the ResizeWrappers (k_resize_band, k_resize, k_resize_pil), the output
// format pass (k_format) and the Resizer that owns their tables and staging frame, MotionBlurWrapper's k_blend4,
// dts_step_terminal's k_copy_rows.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "dts_kernels.h"

namespace dts {

// SMs of the current device: grid-stride kernels cap their grid at a multiple of it
static size_t device_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? (size_t)sms : 1;
}

// Pillow's bilinear resize (k_resize_pil): both axes' fixed-point tap tables and the band plan
struct PilTab {
  int W, H, ow, oh;   // camera and target size
  int tx, ty;         // taps per output column / row: the most any one has; the others are padded with zero taps
  int band, cap;      // output rows per CTA, source rows a band spans at most
  int pitch, ow3p;    // shared-memory row pitch of the staged source (32-bit words) and of the horizontal result (bytes)
  size_t smem;        // dynamic shared memory per CTA
  int32_t* tab;       // device: xs[ow] (first source column), xw[ow][tx] (22-bit weights), ys[oh], yw[oh][ty]; null: off
};

struct Resizer {
  int n, W, H;                         // envs and camera of the handle
  int filter = DTS_RESIZE_CV2_CUBIC, ow = 0, oh = 0;   // DTS_RESIZE_* and the target; 0 x 0: off
  int layout = DTS_OBS_HWC, dtype = DTS_OBS_U8;        // the caller's obs (dts_set_output_format)
  uint8_t* staging = nullptr;          // [n][H][W][3] the full-size frames (null unless staged())
  int16_t* cubic = nullptr;            // cv2: the tap tables [ow][8] then [oh][8] (null unless cv2 is set), and
  int band = 0, cap = 0;               // k_resize_band's plan (plan_resize_bands; band 0: the untiled k_resize)
  PilTab pil{};                        // Pillow: tap tables and band plan (null unless Pillow is set)
};

// The rasterisers draw into the staging frame, and a post pass writes obs, whenever obs is not their packed u8 HWC frame
// at the camera size
static bool staged(const Resizer& z) { return z.ow || z.layout != DTS_OBS_HWC || z.dtype != DTS_OBS_U8; }

constexpr size_t kSmemOptInMax = 200 * 1024;   // dynamic shared memory of the largest band plan either filter makes

// ------------------------------------------------------------------------------------------------ k_resize
// One entry of a cv2 tap table (8 int16 read as an int4): four source indices, then their four taps
struct CubicTaps { int i[4], w[4]; };
__device__ __forceinline__ CubicTaps cubic_taps(int4 a) {
  return CubicTaps{{(short)(a.x & 0xffff), a.x >> 16, (short)(a.y & 0xffff), a.y >> 16},
                   {(short)(a.z & 0xffff), a.z >> 16, (short)(a.w & 0xffff), a.w >> 16}};
}

// ResizeWrapper (wrappers.py:111-141): cv2.resize(..., interpolation=cv2.INTER_CUBIC) of the rendered frame, on the
// device, so that a training stack's 84x84 payload (21 KB per env instead of 57.6 KB) is what crosses PCIe.  OpenCV's
// 8-bit bicubic is fixed point: per output column / row four int16 taps = cvRound(2048 * w_k(frac)), w = the a = -0.75
// cubic kernel evaluated in float32 at frac = (d + 0.5) * scale - 0.5 - floor(.), source indices clamped to the
// image; horizontal pass in int32, then (sum_k beta_k * row_k + 2^21) >> 22, saturated.  The tap tables are built on
// the host (cubic_axis_table).  One thread per output pixel (3 channels); reads the full-size u8 HWC render.
__global__ void __launch_bounds__(256) k_resize(const uint8_t* __restrict__ src, int W, int H, int ow, int oh, int n_envs,
                                                const int16_t* __restrict__ xtab /*[ow][8]: 4 indices, 4 taps*/,
                                                const int16_t* __restrict__ ytab /*[oh][8]*/, void* __restrict__ dst, int layout,
                                                int dtype, const int32_t* __restrict__ env_list, const int32_t* __restrict__ env_count) {
  const size_t total = (size_t)n_listed(env_list, env_count, n_envs) * ow * oh;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(g % ow), y = (int)((g / ow) % oh);
    const size_t env = (size_t)listed_env(env_list, (int)(g / ((size_t)ow * oh)));
    const CubicTaps cx = cubic_taps(__ldg(reinterpret_cast<const int4*>(xtab + 8 * x)));
    const CubicTaps cy = cubic_taps(__ldg(reinterpret_cast<const int4*>(ytab + 8 * y)));
    const uint8_t* frame = src + env * (size_t)W * H * 3;
    long long acc[3] = {0, 0, 0};
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const uint8_t* row = frame + (size_t)cy.i[r] * W * 3;
      int h0 = 0, h1 = 0, h2 = 0;
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const uint8_t* px = row + cx.i[c] * 3;
        h0 += (int)px[0] * cx.w[c]; h1 += (int)px[1] * cx.w[c]; h2 += (int)px[2] * cx.w[c];
      }
      acc[0] += (long long)h0 * cy.w[r]; acc[1] += (long long)h1 * cy.w[r]; acc[2] += (long long)h2 * cy.w[r];
    }
    unsigned rgb = 0;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      long long v = (acc[ch] + (1LL << 21)) >> 22;
      v = v < 0 ? 0 : (v > 255 ? 255 : v);
      rgb |= (unsigned)v << (8 * ch);
    }
    void* out = reinterpret_cast<uint8_t*>(dst) + env * (size_t)ow * oh * 3 * (dtype == DTS_OBS_F32_UNIT ? 4 : 1);
    store_px_fmt(out, layout, dtype, x, y, ow, oh, rgb);
  }
}

// The same resize, tiled: a CTA per (band of `R` output rows, env).  The band's source rows (contiguous bytes of the
// render) are copied to shared memory with 16-byte loads, the horizontal pass runs once per source row into an int32
// buffer in shared memory, the vertical pass reads it and writes four output bytes per thread as one word — instead
// of every output pixel fetching its own 48 source bytes from global memory (k_resize above: 0.49 ms at 4096 x
// 160x120 -> 84x84).  Integer arithmetic identical to k_resize.  `cap` = the largest source-row span of any band
// (computed on the host from the same tap table).
__global__ void __launch_bounds__(256) k_resize_band(const uint8_t* __restrict__ src, int W, int H, int ow, int oh,
                                                     const int16_t* __restrict__ xtab, const int16_t* __restrict__ ytab,
                                                     void* __restrict__ dst, int layout, int dtype, int R, int cap,
                                                     const int32_t* __restrict__ env_list, const int32_t* __restrict__ env_count) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  const int bands = (oh + R - 1) / R;
  const int slot = blockIdx.x / bands, r0 = (blockIdx.x - slot * bands) * R, r1 = min(r0 + R, oh);
  if (env_list && slot >= __ldg(env_count)) return;   // (the whole CTA)
  const int env = listed_env(env_list, slot);
  const int s_lo = ytab[8 * r0], s_hi = ytab[8 * (r1 - 1) + 3], nrows = min(s_hi - s_lo + 1, cap);
  const int rowb = W * 3, ow3 = ow * 3;
  int4* xt = reinterpret_cast<int4*>(rs_smem);                                      // [ow] tap table
  uint8_t* sb = rs_smem + (size_t)ow * 16;                                          // [cap][rowb] source bytes
  int* hb = reinterpret_cast<int*>(sb + (((size_t)cap * rowb + 15) & ~(size_t)15));   // [cap][ow3] horizontal sums
  const uint8_t* band = src + (size_t)env * W * H * 3 + (size_t)s_lo * rowb;
  const int nbytes = nrows * rowb;
  if ((reinterpret_cast<uintptr_t>(band) & 15) == 0 && (nbytes & 15) == 0) {
    for (int i = threadIdx.x; i < nbytes / 16; i += blockDim.x) reinterpret_cast<int4*>(sb)[i] = __ldg(reinterpret_cast<const int4*>(band) + i);
  } else {
    for (int i = threadIdx.x; i < nbytes; i += blockDim.x) sb[i] = __ldg(band + i);
  }
  for (int i = threadIdx.x; i < ow; i += blockDim.x) xt[i] = __ldg(reinterpret_cast<const int4*>(xtab) + i);
  __syncthreads();
  // horizontal pass: a warp per source row, a lane per output column (no index divisions), three channels
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int x = lane; x < ow; x += 32) {
    const CubicTaps cx = cubic_taps(xt[x]);
    for (int row = warp; row < nrows; row += nwarps) {
      const uint8_t* rp = sb + row * rowb;
      int h0 = 0, h1 = 0, h2 = 0;
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const uint8_t* px = rp + cx.i[c] * 3;
        h0 += (int)px[0] * cx.w[c]; h1 += (int)px[1] * cx.w[c]; h2 += (int)px[2] * cx.w[c];
      }
      int* hp = hb + row * ow3 + x * 3;
      hp[0] = h0; hp[1] = h1; hp[2] = h2;
    }
  }
  __syncthreads();
  // vertical pass
  const size_t out_elem = dtype == DTS_OBS_F32_UNIT ? 4 : 1;
  uint8_t* out = reinterpret_cast<uint8_t*>(dst) + (size_t)env * ow3 * oh * out_elem;
  const bool words = layout == DTS_OBS_HWC && dtype == DTS_OBS_U8 && (ow3 & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0;
  if (words) {
    const int wpr = ow3 / 4;   // words per output row
    for (int y = r0 + warp; y < r1; y += nwarps) {   // a warp per output row, a lane per word of four bytes
      const CubicTaps cy = cubic_taps(__ldg(reinterpret_cast<const int4*>(ytab) + y));
      for (int j = lane; j < wpr; j += 32) {
        const int e = 4 * j;
        // int32 like OpenCV's own vertical pass (|sum| <= 255 * sum|xw| * sum|yw| < 2^31 for cubic taps: 255 * 2621^2 = 1.75e9)
        int acc[4] = {0, 0, 0, 0};
#pragma unroll
        for (int r = 0; r < 4; r++) {
          const int4 hv = *reinterpret_cast<const int4*>(hb + (cy.i[r] - s_lo) * ow3 + e);
          acc[0] += hv.x * cy.w[r]; acc[1] += hv.y * cy.w[r]; acc[2] += hv.z * cy.w[r]; acc[3] += hv.w * cy.w[r];
        }
        unsigned word = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const int v = min(max((acc[k] + (1 << 21)) >> 22, 0), 255);
          word |= (unsigned)v << (8 * k);
        }
        *reinterpret_cast<unsigned*>(out + (size_t)y * ow3 + e) = word;
      }
    }
  } else {
    for (int i = threadIdx.x; i < (r1 - r0) * ow3; i += blockDim.x) {
      const int yy = i / ow3, e = i - yy * ow3, y = r0 + yy, x = e / 3, ch = e - 3 * x;
      const CubicTaps cy = cubic_taps(__ldg(reinterpret_cast<const int4*>(ytab) + y));
      long long acc = 0;
#pragma unroll
      for (int r = 0; r < 4; r++) acc += (long long)hb[(cy.i[r] - s_lo) * ow3 + e] * cy.w[r];
      long long v = (acc + (1LL << 21)) >> 22;
      v = v < 0 ? 0 : (v > 255 ? 255 : v);
      store_elem_fmt(out, layout, dtype, x, y, ch, ow, oh, (unsigned)v);
    }
  }
}

// dynamic shared memory of k_resize_band for a band spanning `cap` source rows
static size_t resize_band_smem(int W, int ow, int cap) {
  return (size_t)ow * 16 + (((size_t)cap * W * 3 + 15) & ~(size_t)15) + (size_t)cap * ow * 3 * 4 + 16;   // (+16: word loads may run past the last row)
}

constexpr size_t kResizeBandSmem = 40 * 1024;   // shared memory a band may take and still leave room for several CTAs per SM

// k_resize_band's plan for z's target and row tap table `ytab` ([oh][8]): the tallest band (<= 16 output rows) whose
// source rows + horizontal sums fit in kResizeBandSmem, or single rows in up to kSmemOptInMax; otherwise, and under
// DTS_RESIZE_UNTILED=1, the untiled kernel (band 0)
static void plan_resize_bands(Resizer& z, const int16_t* ytab) {
  const int W = z.W, ow = z.ow, oh = z.oh;
  z.band = z.cap = 0;
  const char* untiled = getenv("DTS_RESIZE_UNTILED");
  if (untiled && untiled[0] == '1') return;
  for (int R = 16; R >= 1; R--) {
    int cap = 0;
    for (int r0 = 0; r0 < oh; r0 += R) {
      const int r1 = std::min(r0 + R, oh);
      cap = std::max(cap, (int)ytab[(size_t)8 * (r1 - 1) + 3] - (int)ytab[(size_t)8 * r0] + 1);
    }
    const size_t smem = resize_band_smem(W, ow, cap);
    if (smem <= kResizeBandSmem || (R == 1 && smem <= kSmemOptInMax)) { z.band = R; z.cap = cap; return; }
  }
}

// cv2.resize INTER_CUBIC tap table of one axis, appended to `tab` (OpenCV resize(): fx = (float)((d + 0.5) * scale - 0.5),
// interpolateCubic with A = -0.75 in float32, taps = saturate_cast<short>(w * 2048), indices clamped to the image)
static void cubic_axis_table(int src, int dst, std::vector<int16_t>& tab) {
  const size_t base = tab.size();
  tab.resize(base + (size_t)dst * 8, 0);
  const double inv = (double)dst / (double)src, scale = 1.0 / inv;
  for (int d = 0; d < dst; d++) {
    float fx = (float)((d + 0.5) * scale - 0.5);
    const int sx = (int)floorf(fx);
    fx -= (float)sx;
    const float A = -0.75f, x = fx;
    float c[4];
    c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
    c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
    c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
    c[3] = 1.f - c[0] - c[1] - c[2];
    for (int k = 0; k < 4; k++) {
      int idx = sx - 1 + k;
      idx = idx < 0 ? 0 : (idx > src - 1 ? src - 1 : idx);
      tab[base + (size_t)d * 8 + k] = (int16_t)idx;
      tab[base + (size_t)d * 8 + 4 + k] = (int16_t)lrintf(c[k] * 2048.0f);
    }
  }
}

// ------------------------------------------------------------------------------------------------ k_resize_pil
// learning/utils/wrappers.py:39-54's ResizeWrapper: scipy.misc.imresize(obs, shape), which for a uint8 RGB frame is
// PIL.Image.resize((w, h), BILINEAR), in Pillow's 8-bit arithmetic (Resample.c): per axis a triangle filter widened by
// the scale factor when it shrinks (7 taps per output pixel at 640 -> 160), weights normalised in double and rounded
// to 22-bit fixed point (tables: pil_axis); the horizontal pass first, acc = 2^21 + sum px * w in int32, clipped to
// u8, then the vertical pass on those bytes.
// A CTA per (band of `band` output rows, env).  The band's source rows pass through shared memory kPilChunk at a time,
// one pixel per 32-bit word; a warp takes one output column of those rows, a lane per row, its two half-warps the even
// and odd taps (row pitch = 2 mod 32 words, so the 32 lanes read 32 different banks).  The horizontal results, u8 like
// Pillow's intermediate image, stay in shared memory for the whole band (480 B per source row at 160 wide); the
// vertical pass reads them a word (four bytes of an output row) per lane.
constexpr int kPilChunk = 16;                   // source rows staged at a time: one per lane of a half-warp
constexpr size_t kPilSmem = 74 * 1024;          // a band plan that fits keeps three CTAs per SM
constexpr int kPilMaxTaps = 65;                 // Pillow's ksize at a 32x reduction

__device__ __forceinline__ unsigned pil_clip8(int acc) { return (unsigned)min(max(acc >> 22, 0), 255); }

__global__ void __launch_bounds__(256) k_resize_pil(const uint8_t* __restrict__ src, const PilTab t, void* __restrict__ dst,
                                                    int layout, int dtype, const int32_t* __restrict__ env_list,
                                                    const int32_t* __restrict__ env_count) {
  extern __shared__ __align__(16) unsigned char pil_smem[];
  const int W = t.W, H = t.H, ow = t.ow, oh = t.oh, ow3 = ow * 3, pitch = t.pitch, ow3p = t.ow3p;
  const int bands = (oh + t.band - 1) / t.band;
  const int slot = blockIdx.x / bands, r0 = (blockIdx.x - slot * bands) * t.band, r1 = min(r0 + t.band, oh);
  if (env_list && slot >= __ldg(env_count)) return;   // (the whole CTA)
  const int env = listed_env(env_list, slot);
  const int32_t* __restrict__ xs = t.tab;
  const int32_t* __restrict__ xw = xs + ow;
  const int32_t* __restrict__ ys = xw + (size_t)ow * t.tx;
  const int32_t* __restrict__ yw = ys + oh;
  const int lo = __ldg(ys + r0), hi = __ldg(ys + r1 - 1) + t.ty;   // the band's source rows [lo, hi)
  uint32_t* stage = reinterpret_cast<uint32_t*>(pil_smem);         // [kPilChunk][pitch] source pixels, RGBX
  uint8_t* inter = pil_smem + (size_t)kPilChunk * pitch * 4;       // [cap][ow3p] horizontal result, u8 RGB
  const uint8_t* frame = src + (size_t)env * W * H * 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int hr = lane & 15, half = lane >> 4;
  // four pixels = three aligned words when rows are whole groups of four and the frame is word-aligned
  const bool words_in = (W & 3) == 0 && (reinterpret_cast<uintptr_t>(frame) & 3) == 0;
  for (int c0 = lo; c0 < hi; c0 += kPilChunk) {
    const int nr = min(kPilChunk, hi - c0);
    if (words_in) {
      const int groups = W >> 2, items = nr * groups;
      const uint32_t* rows = reinterpret_cast<const uint32_t*>(frame + (size_t)c0 * W * 3);
      for (int i0 = threadIdx.x; i0 < items; i0 += 4 * blockDim.x) {
        uint32_t v[4][3];
#pragma unroll
        for (int q = 0; q < 4; q++) {   // all loads first: 48 B per thread in flight
          const int i = i0 + q * blockDim.x;
          if (i < items) { v[q][0] = __ldg(rows + 3 * i); v[q][1] = __ldg(rows + 3 * i + 1); v[q][2] = __ldg(rows + 3 * i + 2); }
        }
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int i = i0 + q * blockDim.x;
          if (i >= items) break;
          const int r = i / groups, g = i - r * groups;
          uint2* d = reinterpret_cast<uint2*>(stage + r * pitch + 4 * g);   // (pitch even: 8-byte aligned)
          d[0] = make_uint2(v[q][0], __byte_perm(v[q][0], v[q][1], 0x0543));
          d[1] = make_uint2(__byte_perm(v[q][1], v[q][2], 0x0432), v[q][2] >> 8);
        }
      }
    } else {
      for (int i = threadIdx.x; i < nr * W; i += blockDim.x) {
        const int r = i / W, x = i - r * W;
        const uint8_t* p = frame + ((size_t)(c0 + r) * W + x) * 3;
        stage[r * pitch + x] = (uint32_t)__ldg(p) | ((uint32_t)__ldg(p + 1) << 8) | ((uint32_t)__ldg(p + 2) << 16);
      }
    }
    __syncthreads();
    // horizontal pass: a warp per output column, lane hr = staged row, half = even / odd taps
    for (int x = warp; x < ow; x += nwarps) {
      const uint32_t* sp = stage + hr * pitch + __ldg(xs + x);
      const int32_t* wx = xw + (size_t)x * t.tx;
      int a0 = 0, a1 = 0, a2 = 0;
      for (int k = half; k < t.tx; k += 2) {
        const int w = __ldg(wx + k);
        const uint32_t v = sp[k];
        a0 += (int)(v & 255u) * w;
        a1 += (int)__byte_perm(v, 0, 0x4441) * w;
        a2 += (int)__byte_perm(v, 0, 0x4442) * w;
      }
      a0 += __shfl_xor_sync(0xffffffffu, a0, 16);
      a1 += __shfl_xor_sync(0xffffffffu, a1, 16);
      a2 += __shfl_xor_sync(0xffffffffu, a2, 16);
      if (half == 0 && hr < nr) {
        uint8_t* o = inter + (size_t)(c0 - lo + hr) * ow3p + 3 * x;
        o[0] = (uint8_t)pil_clip8(a0 + (1 << 21));
        o[1] = (uint8_t)pil_clip8(a1 + (1 << 21));
        o[2] = (uint8_t)pil_clip8(a2 + (1 << 21));
      }
    }
    __syncthreads();
  }
  // vertical pass: a warp per output row, a lane per word of four bytes of it
  const size_t out_elem = dtype == DTS_OBS_F32_UNIT ? 4 : 1;
  uint8_t* out = reinterpret_cast<uint8_t*>(dst) + (size_t)env * ow3 * oh * out_elem;
  const bool words_out = layout == DTS_OBS_HWC && dtype == DTS_OBS_U8 && (ow3 & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0;
  const int wpr = (ow3 + 3) >> 2, ipw = ow3p >> 2;
  for (int y = r0 + warp; y < r1; y += nwarps) {
    const uint32_t* col = reinterpret_cast<const uint32_t*>(inter + (size_t)(__ldg(ys + y) - lo) * ow3p);
    const int32_t* wy = yw + (size_t)y * t.ty;
    for (int j = lane; j < wpr; j += 32) {
      int a[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
      for (int k = 0; k < t.ty; k++) {
        const int w = __ldg(wy + k);
        const uint32_t v = col[k * ipw + j];
        a[0] += (int)(v & 255u) * w;
        a[1] += (int)__byte_perm(v, 0, 0x4441) * w;
        a[2] += (int)__byte_perm(v, 0, 0x4442) * w;
        a[3] += (int)(v >> 24) * w;
      }
      const int e = 4 * j;
      if (words_out) {
        *reinterpret_cast<uint32_t*>(out + (size_t)y * ow3 + e) =
            pil_clip8(a[0]) | (pil_clip8(a[1]) << 8) | (pil_clip8(a[2]) << 16) | (pil_clip8(a[3]) << 24);
        continue;
      }
#pragma unroll
      for (int q = 0; q < 4; q++) {
        if (e + q >= ow3) break;
        const int x = (e + q) / 3, ch = e + q - 3 * x;
        store_elem_fmt(out, layout, dtype, x, y, ch, ow, oh, pil_clip8(a[q]));
      }
    }
  }
}

// Pillow's precompute_coeffs (Resample.c) for one axis, bilinear filter, then normalize_coeffs_8bpc: per output index
// the first source index and `taps` weights, the window moved left where it would run past the last source pixel
// (its extra taps are zero).  Returns Pillow's ksize for the scale.
static int pil_axis(int in, int out, std::vector<int32_t>& start, std::vector<int32_t>& w, int& taps) {
  const double scale = (double)in / out, fs = scale < 1.0 ? 1.0 : scale, support = fs, ss = 1.0 / fs;
  const int ksize = (int)ceil(support) * 2 + 1;
  if (ksize > kPilMaxTaps) return ksize;
  std::vector<int> lo(out), n(out);
  std::vector<int32_t> kk((size_t)out * ksize, 0);
  taps = 1;
  for (int i = 0; i < out; i++) {
    const double center = (i + 0.5) * scale;
    int xmin = (int)(center - support + 0.5), xmax = (int)(center + support + 0.5);
    if (xmin < 0) xmin = 0;
    if (xmax > in) xmax = in;
    const int cnt = std::min(xmax - xmin, ksize);
    double k[kPilMaxTaps], ww = 0.0;
    for (int x = 0; x < cnt; x++) {
      double u = (x + xmin - center + 0.5) * ss;
      if (u < 0.0) u = -u;
      k[x] = u < 1.0 ? 1.0 - u : 0.0;
      ww += k[x];
    }
    for (int x = 0; x < cnt; x++) {
      if (ww != 0.0) k[x] /= ww;
      kk[(size_t)i * ksize + x] = (int32_t)(0.5 + k[x] * (1 << 22));   // the weights are >= 0
    }
    lo[i] = xmin; n[i] = cnt;
    taps = std::max(taps, cnt);
  }
  start.assign(out, 0);
  w.assign((size_t)out * taps, 0);
  for (int i = 0; i < out; i++) {
    const int s = std::min(lo[i], in - taps);
    start[i] = s;
    for (int x = 0; x < n[i]; x++) w[(size_t)i * taps + lo[i] - s + x] = kk[(size_t)i * ksize + x];
  }
  return ksize;
}

// ------------------------------------------------------------------------------------------------ the resizer
// A filter's tables -> a new device allocation at *dst (left as it is if that fails); then, if the plan takes more than
// the default 48 KB of shared memory, its kernel's opt-in to the largest plan's, which holds on the current device
template <typename T>
static std::string upload(const char* filter, T** dst, const std::vector<T>& v, const void* kernel, size_t smem) {
  void* d = nullptr;
  cudaError_t e = cudaMalloc(&d, v.size() * sizeof(T));
  if (e == cudaSuccess) { *dst = reinterpret_cast<T*>(d); e = cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice); }
  if (e == cudaSuccess && smem > 48 * 1024) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOptInMax);
  return e == cudaSuccess ? "" : std::string(filter) + " resize table upload failed: " + cudaGetErrorString(e);
}

// The cv2 filter's tables and band plan for z's target
static std::string cubic_tables(Resizer& z) {
  std::vector<int16_t> tab;   // [ow][8] then [oh][8]
  cubic_axis_table(z.W, z.ow, tab);
  cubic_axis_table(z.H, z.oh, tab);
  plan_resize_bands(z, tab.data() + (size_t)8 * z.ow);
  return upload("cv2", &z.cubic, tab, (const void*)k_resize_band, z.band ? resize_band_smem(z.W, z.ow, z.cap) : 0);
}

// The Pillow filter's tables and band plan for z's target
static std::string pil_tables(Resizer& z) {
  PilTab& t = z.pil;
  const int ow = z.ow, oh = z.oh;
  t.W = z.W; t.H = z.H; t.ow = ow; t.oh = oh;
  std::vector<int32_t> xs, xw, ys, yw;
  const int kx = pil_axis(z.W, ow, xs, xw, t.tx), ky = pil_axis(z.H, oh, ys, yw, t.ty);
  if (kx > kPilMaxTaps || ky > kPilMaxTaps)
    return "Pillow bilinear resize " + std::to_string(z.W) + "x" + std::to_string(z.H) + " -> " + std::to_string(ow) + "x" +
           std::to_string(oh) + " needs " + std::to_string(std::max(kx, ky)) + " taps per output pixel; the device pass takes " +
           "at most " + std::to_string(kPilMaxTaps) + " (targets of at least 1/32 of the camera size per axis)";
  t.pitch = z.W + ((2 - z.W) & 31);                 // = 2 mod 32: the 16 rows x 2 tap parities of a warp hit 32 banks
  t.ow3p = (ow * 3 + 3) & ~3;
  if (((t.ow3p >> 2) & 1) == 0) t.ow3p += 4;        // an odd word pitch: a column's 16 rows are stored to 16 banks
  // band height: the least staged rows (whole chunks) over the frame, within kPilSmem if any plan is, else the least
  // shared memory; ties go to taller bands (fewer CTAs)
  const size_t stage = (size_t)kPilChunk * t.pitch * 4;
  long long best_rows = -1;
  size_t best_smem = 0;
  for (int R = 1; R <= std::min(oh, 64); R++) {
    int cap = 0;
    long long rows = 0;
    for (int r0 = 0; r0 < oh; r0 += R) {
      const int r1 = std::min(r0 + R, oh), span = ys[r1 - 1] + t.ty - ys[r0];
      cap = std::max(cap, span);
      rows += (span + kPilChunk - 1) / kPilChunk * kPilChunk;
    }
    const size_t smem = stage + (size_t)cap * t.ow3p;
    if (smem > kSmemOptInMax) continue;
    const bool fits = smem <= kPilSmem, best_fits = best_rows >= 0 && best_smem <= kPilSmem;
    const bool better = best_rows < 0 || (fits && !best_fits) ||
                        (fits == best_fits && (fits ? rows <= best_rows : smem < best_smem));
    if (better) { best_rows = rows; best_smem = smem; t.band = R; t.cap = cap; }
  }
  if (best_rows < 0)
    return "Pillow bilinear resize to " + std::to_string(ow) + "x" + std::to_string(oh) + ": a single output row needs more " +
           "than " + std::to_string(kSmemOptInMax / 1024) + " KB of shared memory";
  t.smem = best_smem;
  std::vector<int32_t> tab;
  for (const auto* v : {&xs, &xw, &ys, &yw}) tab.insert(tab.end(), v->begin(), v->end());
  return upload("Pillow", &t.tab, tab, (const void*)k_resize_pil, t.smem);
}

Resizer* resizer_create(const dts_config& cfg) { return new Resizer{cfg.num_envs, cfg.cam_width, cfg.cam_height}; }

void resizer_destroy(Resizer* z) {
  if (z) { cudaFree(z->staging); cudaFree(z->cubic); cudaFree(z->pil.tab); }
  delete z;
}

// z <- t, a setting built beside it (`e`: the error building it failed with, if any): t keeps z's staging frame or gets a
// new one if staged(t) needs one.  What the setting that is left over holds and z does not is freed.
static std::string replace(Resizer& z, Resizer& t, std::string e) {
  t.staging = staged(t) ? z.staging : nullptr;
  if (e.empty() && staged(t) && !t.staging) {
    void* p = nullptr;
    const cudaError_t ce = cudaMalloc(&p, (size_t)t.n * t.W * t.H * 3);
    if (ce == cudaSuccess) t.staging = reinterpret_cast<uint8_t*>(p);
    else e = std::string("staging frame cudaMalloc failed: ") + cudaGetErrorString(ce);
  }
  if (e.empty()) std::swap(z, t);   // t: the setting to release, the previous one or the one that failed
  if (t.staging != z.staging) cudaFree(t.staging);
  if (t.cubic != z.cubic) cudaFree(t.cubic);
  if (t.pil.tab != z.pil.tab) cudaFree(t.pil.tab);
  return e;
}

std::string resizer_set(Resizer& z, int filter, int ow, int oh) {
  Resizer t{z.n, z.W, z.H, filter, ow, oh, z.layout, z.dtype};
  const std::string e = !ow ? "" : filter == DTS_RESIZE_PIL_BILINEAR ? pil_tables(t) : cubic_tables(t);
  return replace(z, t, e);
}

std::string resizer_set_format(Resizer& z, int layout, int dtype) {
  Resizer t = z;   // (the same tables)
  t.layout = layout; t.dtype = dtype;
  return replace(z, t, "");
}

ResizeTarget resizer_target(const Resizer& z) { return ResizeTarget{z.ow, z.oh, z.staging}; }

void launch_resize(const Resizer& z, const uint8_t* src, void* dst, int layout, int dtype, const int32_t* env_list,
                   const int32_t* env_count, cudaStream_t st) {
  if (z.filter == DTS_RESIZE_PIL_BILINEAR) {
    const PilTab& t = z.pil;
    const unsigned grid = (unsigned)(((t.oh + t.band - 1) / t.band) * (size_t)z.n);
    k_resize_pil<<<grid, 256, t.smem, st>>>(src, t, dst, layout, dtype, env_list, env_count);
    return;
  }
  const int16_t *xtab = z.cubic, *ytab = z.cubic + (size_t)8 * z.ow;
  if (z.band > 0) {   // tiled form (plan_resize_bands found a band height whose rows fit in shared memory)
    k_resize_band<<<(unsigned)(((z.oh + z.band - 1) / z.band) * (size_t)z.n), 256, resize_band_smem(z.W, z.ow, z.cap), st>>>(
        src, z.W, z.H, z.ow, z.oh, xtab, ytab, dst, layout, dtype, z.band, z.cap, env_list, env_count);
    return;
  }
  const size_t total = (size_t)z.n * z.ow * z.oh;
  const size_t cap = device_sms() * 16;
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  k_resize<<<blocks, 256, 0, st>>>(src, z.W, z.H, z.ow, z.oh, z.n, xtab, ytab, dst, layout, dtype, env_list, env_count);
}

// ------------------------------------------------------------------------------------------------ k_format
// The staging frames at the camera size -> the caller's layout / dtype (dts_set_output_format) and, on a gathering step,
// every peer's gather slot at the same offset: a thread per pixel, grid-stride over the listed envs' pixels.  HWC
// (float32 here: packed u8 HWC is not staged without a resize) where W * H % 32 == 0, so that a warp's 32 pixels are
// consecutive in one frame: the lanes take the warp's 96 elements interleaved, each the staging byte of the same index,
// so that a warp's stores are contiguous instead of three 12-byte-strided float stores.
__global__ void __launch_bounds__(256) k_format(const uint8_t* __restrict__ src, int W, int H, int n_envs, void* __restrict__ dst,
                                                int layout, int dtype, GatherTab gt, const int32_t* __restrict__ env_list,
                                                const int32_t* __restrict__ env_count) {
  const size_t px = (size_t)W * H, frame_bytes = px * 3 * (dtype == DTS_OBS_F32_UNIT ? 4 : 1);
  const bool interleave = layout == DTS_OBS_HWC && px % 32 == 0;
  const size_t total = (size_t)n_listed(env_list, env_count, n_envs) * px;
  const int lane = threadIdx.x & 31;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
    const size_t env = (size_t)listed_env(env_list, (int)(g / px)), i = g % px;
    const uint8_t* s = src + env * px * 3;
    const unsigned rgb = interleave ? 0u : (unsigned)s[3 * i] | ((unsigned)s[3 * i + 1] << 8) | ((unsigned)s[3 * i + 2] << 16);
#pragma unroll
    for (int p = -1; p < DTS_MAX_PEERS; p++) {   // obs, then the peers' slots (constant indices: gt stays in the parameter space)
      if (p >= gt.n) break;
      uint8_t* out = (p < 0 ? reinterpret_cast<uint8_t*>(dst) : gt.base[p < 0 ? 0 : p]) + env * frame_bytes;
      if (interleave) {
#pragma unroll
        for (size_t j = 0, e = (i - lane) * 3 + lane; j < 3; j++, e += 32) reinterpret_cast<float*>(out)[e] = unit_f32(s[e]);
      } else {
        store_px_fmt(out, layout, dtype, (int)(i % W), (int)(i / W), W, H, rgb);
      }
    }
  }
}

void launch_format(const Resizer& z, void* dst, const GatherTab& gt, const int32_t* env_list, const int32_t* env_count,
                   cudaStream_t st) {
  const size_t blocks = ((size_t)z.n * z.W * z.H + 255) / 256, cap = device_sms() * 16;
  k_format<<<(unsigned)std::min(blocks, cap), 256, 0, st>>>(z.staging, z.W, z.H, z.n, dst, z.layout, z.dtype, gt, env_list,
                                                            env_count);
}

// ------------------------------------------------------------------------------------------------ k_blend4
// MotionBlurWrapper (learning/utils/wrappers.py:8-54): np.average(window, axis=0, weights=[0.8, 0.15, 0.04, 0.01]) of four
// uint8 frames -> float64, in numpy's order: products in float64, summed frame by frame, divided by the weight sum.
__global__ void __launch_bounds__(256) k_blend4(const uint8_t* __restrict__ f0, const uint8_t* __restrict__ f1,
                                                const uint8_t* __restrict__ f2, const uint8_t* __restrict__ f3, double w0,
                                                double w1, double w2, double w3, double scl, double* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double a = (double)f0[i] * w0;
    a = a + (double)f1[i] * w1;
    a = a + (double)f2[i] * w2;
    a = a + (double)f3[i] * w3;
    out[i] = a / scl;
  }
}

void launch_blend4(const uint8_t* const f[4], const double w[4], double* out, size_t n, cudaStream_t st) {
  const double scl = ((w[0] + w[1]) + w[2]) + w[3];   // numpy: wgt.sum() of four float64 (pairwise == sequential below 8 terms)
  const size_t blocks = (n + 255) / 256, cap = device_sms() * 32;
  k_blend4<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, st>>>(f[0], f[1], f[2], f[3], w[0], w[1], w[2], w[3], scl, out, n);
}

// ------------------------------------------------------------------------------------------------ k_copy_rows
// dts_step_terminal's terminal frames: the observation rows of the envs that ended -> the same rows of the terminal
// buffer, a CTA per listed env (grid-strided over the list), 16-byte vectors when both rows and the row size allow them.
__global__ void __launch_bounds__(256) k_copy_rows(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t row_bytes,
                                                   const int32_t* __restrict__ list, const int32_t* __restrict__ count) {
  const int n = __ldg(count);
  for (int s = blockIdx.x; s < n; s += gridDim.x) {
    const size_t off = (size_t)__ldg(list + s) * row_bytes;
    const uint8_t* a = src + off;
    uint8_t* b = dst + off;
    if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | row_bytes) & 15) == 0) {
      for (size_t i = threadIdx.x; i < row_bytes / 16; i += blockDim.x)
        reinterpret_cast<int4*>(b)[i] = __ldg(reinterpret_cast<const int4*>(a) + i);
    } else {
      for (size_t i = threadIdx.x; i < row_bytes; i += blockDim.x) b[i] = __ldg(a + i);
    }
  }
}

void launch_copy_rows(const void* src, void* dst, size_t row_bytes, const int32_t* list, const int32_t* count, int n_envs,
                      cudaStream_t st) {
  const size_t cap = device_sms() * 8, blocks = (size_t)n_envs < cap ? (size_t)n_envs : cap;
  k_copy_rows<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(src), reinterpret_cast<uint8_t*>(dst), row_bytes,
                                                list, count);
}

}  // namespace dts
