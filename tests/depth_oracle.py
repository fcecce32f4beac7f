"""The CPU oracle of the depth image (render spec item 9, DESIGN.md section 5): test infrastructure, like oracle/.

The depth of a pixel is defined from the raster oracle's own visibility, so the depth oracle is the raster oracle
(oracle/dt_oracle_raster.c) itself, compiled a second time with the few insertions in PATCH: a buffer beside the depth
buffer that keeps, per sample, the winning triangle's 1/w at the pixel centre exactly as shading clamps it, and at the
resolve `1 / max` of a pixel's four entries (0 where none is covered or the LUT names no source).  The raster oracle's
source stays as it is and nothing of it is duplicated; every insertion names the text it follows and must find it
exactly once, so a change of the oracle that moves one fails here instead of being missed.  The frames this build
returns are the raster oracle's (tests/test_oracle_depth.py holds them to it byte for byte).

The library is built with the raster oracle's compiler flags into the user's temporary directory, keyed by a hash of the
patched source, so the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "oracle", "dt_oracle_raster.c")

# (text of the raster oracle, what is put in its place): each replacement is the text itself plus an insertion
PATCH = [
    # the buffer: [H][W][4], the winner's clamped 1/w at the pixel centre; 0 = sample not covered
    ("  float* depth; /* [H][W][4] */\n} framebuf;\n",
     "  float* depth; /* [H][W][4] */\n  float* q;\n} framebuf;\n"
     "static _Thread_local float* tl_depth_out = 0; /* f32 [H][W] of the frame being drawn, or none */\n"
     "static _Thread_local float* tl_q = 0;\n"
     "static _Thread_local size_t tl_q_px = 0;\n"),
    # a sample that passes GL_LESS takes the triangle's 1/w with its colour (qq: shading's clamped value)
    ("          fb->depth[si] = z;\n", "          fb->depth[si] = z;\n          fb->q[si] = qq;\n"),
    ("  fb.depth = tl_depth;\n",
     "  fb.depth = tl_depth;\n"
     "  if (tl_q_px < (size_t)W * H) { free(tl_q); tl_q_px = (size_t)W * H; tl_q = (float*)malloc(sizeof(float) * tl_q_px * 4); }\n"
     "  fb.q = tl_q;\n"),
    ("    fb.depth[k] = 1.0f;\n", "    fb.depth[k] = 1.0f;\n    fb.q[k] = 0.0f;\n"),
    # resolve: the nearest surface any sample of the (source) pixel sees; a maximum of exact values, whatever the order
    ("        out[((size_t)y * W + xx) * 3 + ch] = v;\n      }\n",
     "        out[((size_t)y * W + xx) * 3 + ch] = v;\n      }\n"
     "      if (tl_depth_out) {\n"
     "        float qmax = 0.0f;\n"
     "        if (valid)\n"
     "          for (int s = 0; s < 4; s++) { const float q = fb.q[((size_t)sy * W + sx) * 4 + s]; if (q > qmax) qmax = q; }\n"
     "        tl_depth_out[(size_t)y * W + xx] = qmax > 0.0f ? 1.0f / qmax : 0.0f;\n"
     "      }\n"),
]
ENTRY = """
/* orr_render_batch, and every env's depth image into depth_out f32 [n][H][W] */
void orr_render_batch_depth(const orr_scene* sc, int n, const double* px, const double* pz, const double* angle,
                            const orr_episode* eps, int W, int H, int domain_rand, const float* lut_x, const float* lut_y,
                            uint8_t* out, float* depth_out, int threads) {
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int e = 0; e < n; e++) {
    tl_depth_out = depth_out + (size_t)e * W * H;
    orr_render(sc, px[e], pz[e], angle[e], &eps[e], W, H, domain_rand, lut_x, lut_y, out + (size_t)e * W * H * 3);
    tl_depth_out = 0;
  }
}
"""
THREADS = os.cpu_count() or 1


def patched_source() -> str:
    src = open(SOURCE).read()
    for old, new in PATCH:
        if src.count(old) != 1:
            raise RuntimeError(f"oracle/dt_oracle_raster.c no longer has exactly one {old!r}: the depth insertion after it "
                               "must be placed again")
        src = src.replace(old, new)
    return src + ENTRY


_lib = None


def lib():
    global _lib
    if _lib is None:
        src = patched_source()
        cmd = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-mfma",
               "-mavx2", "-I", os.path.join(ROOT, "oracle")]     # oracle.build()'s flags: the same arithmetic
        key = hashlib.sha256((src + " ".join(cmd)).encode()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"dts_depth_oracle_{os.getuid()}_{key}.so")
        if not os.path.exists(so):
            with tempfile.TemporaryDirectory() as d:
                c = os.path.join(d, "depth_oracle.c")
                with open(c, "w") as f:
                    f.write(src)
                subprocess.check_call(cmd + ["-o", os.path.join(d, "out.so"), c, "-lm"])
                os.replace(os.path.join(d, "out.so"), so)     # complete or absent, also with several test processes
        _lib = C.CDLL(so)
    return _lib


def render_batch(sc, px, pz, angle, eps=None, W=160, H=120, domain_rand=False, lut=None, segment=False, top_down=False,
                 tile_mode=1, threads=THREADS):
    """(frames u8 [n, H, W, 3], depth f32 [n, H, W]) of the cameras (px, pz, angle) of `sc`, an oracle.OracleScene;
    eps: their oracle episodes (default: the non-randomised one).  This build has its own copy of the raster oracle's
    tile and render modes, so they are arguments."""
    n = len(px)
    eps = eps or [orc.default_episode() for _ in range(n)]
    arr = (orc.OrrEpisode * n)(*eps)
    a = [np.ascontiguousarray(v, np.float64) for v in (px, pz, angle)]
    out, dep = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32)
    lx = ly = None
    if lut is not None:
        lx, ly = np.ascontiguousarray(lut[0], np.float32), np.ascontiguousarray(lut[1], np.float32)
    p = lambda v: None if v is None else v.ctypes.data_as(C.c_void_p)
    L = lib()
    L.orr_set_tile_mode(int(tile_mode))
    L.orr_set_render_mode((1 if segment else 0) | (2 if top_down else 0))
    L.orr_render_batch_depth(C.byref(sc.c), n, p(a[0]), p(a[1]), p(a[2]), arr, W, H, int(domain_rand), p(lx), p(ly), p(out),
                             p(dep), int(threads))
    return out, dep


def render(sc, px, pz, angle, ep=None, W=160, H=120, domain_rand=False, **kw):
    """(frame u8 [H, W, 3], depth f32 [H, W]) of one camera."""
    out, dep = render_batch(sc, [px], [pz], [angle], [ep] if ep is not None else None, W, H, domain_rand, threads=1, **kw)
    return out[0], dep[0]
