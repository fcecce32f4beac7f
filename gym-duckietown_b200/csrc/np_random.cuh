// np_random.cuh — NumPy-compatible random streams on the device.
//
// The reference draws every reset quantity from `numpy.random.Generator(PCG64(SeedSequence(seed)))`
// (simulator.py:1043-1045 via gym.utils.seeding.np_random; draw sites simulator.py:546-736,
// randomization/randomizer.py:36-91).  To let DEVICE-side resets (dts_reset_random / auto-reset) stay on
// that stream draw for draw, this header restates the published algorithms behind the four numpy calls the
// reference makes:
//   PCG64 (pcg_setseq_128_xsl_rr_64): state = state * 0x2360ED051FC65DA44385DF649FCCF645 + inc (mod 2^128),
//          output rotr64(hi ^ lo, hi >> 58) of the NEW state; 32-bit draws return the low half and cache the high
//   Generator.uniform(lo, hi)   = lo + (hi - lo) * (next64 >> 11) * 2^-53
//   Generator.integers(lo, hi)  = random_bounded_uint64's regimes on int64 bounds: Lemire's nearly-divisionless
//          rejection on 32-bit draws below 2^32 - 1, one raw 32-bit draw at 2^32 - 1, Lemire on 64-bit draws above
//   Generator.normal(loc, sc)   = loc + sc * ziggurat(256 layers), tables in np_ziggurat_tables.h
// The host seeds the streams (numpy itself computes SeedSequence -> initial state) and uploads
// (state, inc, has_uint32, uinteger) per env with dts_seed_streams.  tests/test_gpu_np_streams.py runs every
// method here (dts_debug_draw) and the device resets and obstacle walks against numpy draw for draw, bit for bit,
// stream state included; tests/test_gpu_logic.py checks device resets against the reference's own golden vectors.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "np_ziggurat_tables.h"

namespace dts {

__host__ __device__ inline int32_t np_hi_word(double x) { uint64_t u; memcpy(&u, &x, 8); return (int32_t)(u >> 32); }
__host__ __device__ inline double np_with_hi_word(double x, int32_t hi) {
  uint64_t u;
  memcpy(&u, &x, 8);
  u = (u & 0xFFFFFFFFull) | ((uint64_t)(uint32_t)hi << 32);
  memcpy(&x, &u, 8);
  return x;
}

// log1p as numpy's ziggurat tail gets it: npy_log1p is the host libm's log1p, and glibc's (sysdeps/ieee754/dbl-64/
// s_log1p.c: fdlibm's reduction, an Estrin-order polynomial) runs as the variant built for FMA on hosts that have it, so
// every fma() below is a product the compiler fused there.  With the build's -fmad=false nothing else is fused; compiled
// for the host, this returned glibc 2.39's bits on 2 * 10^8 of the ziggurat's arguments -next_double() and on every high
// word near its branch points.  (With CUDA's log1p, 10 of 4,096 streams left numpy within 3,072 normal draws each.)  A
// host without FMA runs glibc's other variant, and numpy's own tail draws then differ from these in the last bits.
__host__ __device__ inline double np_log1p(double x) {
  const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10, two54 = 1.80143985094819840000e+16;
  const double Lp1 = 6.666666666666735130e-01, Lp2 = 3.999999999940941908e-01, Lp3 = 2.857142874366239149e-01,
               Lp4 = 2.222219843214978396e-01, Lp5 = 1.818357216161805012e-01, Lp6 = 1.531383769920937332e-01,
               Lp7 = 1.479819860511658591e-01;
  const int32_t hx = np_hi_word(x), ax = hx & 0x7fffffff;
  double f = 0.0, c = 0.0;
  int32_t k = 1, hu = 0;
  if (hx < 0x3FDA827A) {                                  // x < 0.41422
    if (ax >= 0x3ff00000) return x == -1.0 ? -two54 / 0.0 : (x - x) / (x - x);
    if (ax < 0x3e200000) return ax < 0x3c900000 ? x : fma(-(x * x), 0.5, x);   // |x| < 2^-29
    if (hx > 0 || hx <= (int32_t)0xbfd2bec3) { k = 0; f = x; hu = 1; }         // -0.2929 < x < 0.41422
  }
  if (hx >= 0x7ff00000) return x + x;
  if (k != 0) {
    double u;
    if (hx < 0x43400000) {
      u = 1.0 + x;
      hu = np_hi_word(u);
      k = (hu >> 20) - 1023;
      c = (k > 0) ? 1.0 - (u - x) : x - (u - 1.0);      // correction term
      c /= u;
    } else {
      u = x;
      hu = np_hi_word(u);
      k = (hu >> 20) - 1023;
      c = 0.0;
    }
    hu &= 0x000fffff;
    if (hu < 0x6a09e) {
      u = np_with_hi_word(u, hu | 0x3ff00000);          // normalise u
    } else {
      k += 1;
      u = np_with_hi_word(u, hu | 0x3fe00000);          // normalise u / 2
      hu = (0x00100000 - hu) >> 2;
    }
    f = u - 1.0;
  }
  const double hfsq = 0.5 * f * f, dk = (double)k;
  if (hu == 0) {                                          // |f| < 2^-20
    if (f == 0.0) return k == 0 ? 0.0 : fma(dk, ln2_hi, fma(dk, ln2_lo, c));
    const double R = hfsq * fma(-0.66666666666666666, f, 1.0);
    return k == 0 ? f - R : fma(dk, ln2_hi, -((R - fma(dk, ln2_lo, c)) - f));
  }
  const double s = f / (2.0 + f), z = s * s, z2 = z * z, z4 = z2 * z2, z6 = z4 * z2;
  const double R2 = fma(z, Lp3, Lp2), R3 = fma(z, Lp5, Lp4), R4 = fma(z, Lp7, Lp6);
  const double R = fma(z6, R4, fma(z4, R3, fma(z, Lp1, z2 * R2)));
  if (k == 0) return f - (hfsq - s * (hfsq + R));
  return fma(dk, ln2_hi, -((hfsq - (s * (hfsq + R) + fma(dk, ln2_lo, c))) - f));
}

struct NpStream {
  unsigned __int128 state, inc;
  uint32_t has32, cache32;

  __device__ __forceinline__ uint64_t next64() {
    const unsigned __int128 mult = ((unsigned __int128)0x2360ED051FC65DA4ULL << 64) | 0x4385DF649FCCF645ULL;
    state = state * mult + inc;
    const uint64_t hi = (uint64_t)(state >> 64), lo = (uint64_t)state;
    const uint64_t x = hi ^ lo;
    const unsigned rot = (unsigned)(hi >> 58);
    return (x >> rot) | (x << ((64u - rot) & 63u));
  }
  __device__ __forceinline__ uint32_t next32() {
    if (has32) { has32 = 0; return cache32; }
    const uint64_t n = next64();
    has32 = 1;
    cache32 = (uint32_t)(n >> 32);
    return (uint32_t)n;
  }
  __device__ __forceinline__ double next_double() { return (double)(next64() >> 11) * (1.0 / 9007199254740992.0); }
  __device__ __forceinline__ double uniform(double lo, double hi) { return lo + (hi - lo) * next_double(); }
  // Generator.integers(lo, hi) for int64 (hi exclusive, lo < hi): numpy's random_bounded_uint64 on rng = hi - 1 - lo.
  // rng 0 draws nothing; below 2^32 - 1, 32-bit Lemire on next32 (so it uses and leaves the cached half); exactly
  // 2^32 - 1, one raw next32; above, 64-bit Lemire with a 128-bit product.  (numpy's raw next64 at rng = 2^64 - 1
  // needs a range wider than int64 bounds can give.)
  __device__ inline int64_t integers(int64_t lo, int64_t hi) {
    const uint64_t rng = (uint64_t)hi - (uint64_t)lo - 1u;
    if (rng == 0) return lo;
    if (rng < 0xFFFFFFFFull) {
      const uint32_t rng_excl = (uint32_t)rng + 1u;
      uint64_t m = (uint64_t)next32() * rng_excl;
      uint32_t leftover = (uint32_t)m;
      if (leftover < rng_excl) {
        const uint32_t threshold = (0xFFFFFFFFu - (uint32_t)rng) % rng_excl;
        while (leftover < threshold) { m = (uint64_t)next32() * rng_excl; leftover = (uint32_t)m; }
      }
      return (int64_t)((uint64_t)lo + (m >> 32));
    }
    if (rng == 0xFFFFFFFFull) return (int64_t)((uint64_t)lo + next32());
    const uint64_t rng_excl = rng + 1u;
    unsigned __int128 m = (unsigned __int128)next64() * rng_excl;
    uint64_t leftover = (uint64_t)m;
    if (leftover < rng_excl) {
      const uint64_t threshold = (~0ull - rng) % rng_excl;
      while (leftover < threshold) { m = (unsigned __int128)next64() * rng_excl; leftover = (uint64_t)m; }
    }
    return (int64_t)((uint64_t)lo + (uint64_t)(m >> 64));
  }
  __device__ inline double standard_normal() {
    const double R = 3.6541528853610087963519472518, INV_R = 0.27366123732975827203338247596;
    for (;;) {
      uint64_t r = next64();
      const int idx = (int)(r & 0xff);
      r >>= 8;
      const int sign = (int)(r & 1);
      const uint64_t rabs = (r >> 1) & 0x000fffffffffffffULL;
      double x = (double)rabs * np_wi_double[idx];
      if (sign) x = -x;
      if (rabs < np_ki_double[idx]) return x;
      if (idx == 0) {
        for (;;) {
          const double xx = -INV_R * np_log1p(-next_double());
          const double yy = -np_log1p(-next_double());
          if (yy + yy > xx * xx) return ((rabs >> 8) & 1) ? -(R + xx) : R + xx;
        }
      } else if (((np_fi_double[idx - 1] - np_fi_double[idx]) * next_double() + np_fi_double[idx]) < exp(-0.5 * x * x)) {
        return x;
      }
    }
  }
  __device__ __forceinline__ double normal(double loc, double scale) { return loc + scale * standard_normal(); }
};

}  // namespace dts
