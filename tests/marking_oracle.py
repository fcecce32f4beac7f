"""The CPU oracle of the lane-marking image (render spec item 11, DESIGN.md section 5): test infrastructure, like oracle/.

A pixel's marking is defined from the label oracle's own visibility, so the marking oracle is the label oracle's source
(tests/label_oracle.py: the depth oracle's with the label insertions) with the few insertions in PATCH: where shading
has computed u, v at the pixel centre, the class of the texel (floor(u * w) mod w, floor(v * h) mod h) of the
triangle's texture (0 untextured); one more value per sample, that class of the triangle that passed GL_LESS there
(beside its 1/w and item); and at the resolve, among the samples with the label's 1/w and the label's value, the
smallest class, 0 where the label is 0.  Every insertion names the text it follows and must find it exactly once.

The texel classes are the scene's: oracle.OracleScene builds its textures with the product's blob builder, whose
keep["tex_cls"] holds one uint8 [h, w] plane per texture in the same order; render_batch hands them to this build
beside the scene, so oracle/'s scene struct stays as it is.  One build returns the frames, depth and labels of the label
oracle (tests/test_oracle_markings.py holds them to it byte for byte) and the markings.  It is built by
depth_oracle.lib(), handed this source for one call, as the label oracle is."""
import ctypes as C

import numpy as np

import depth_oracle
import label_oracle
import oracle as orc

# (text of the label oracle's source, what is put in its place): each replacement is the text itself plus an insertion
PATCH = [
    # the class per sample ([H][W][4]) and where the classes come from
    ("  int* item;\n} framebuf;\n",
     "  int* item;\n  int* cls;\n} framebuf;\n"
     "static _Thread_local uint8_t* tl_mark_out = 0; /* u8 [H][W] of the frame being drawn, or none */\n"
     "static _Thread_local const orr_texture* tl_tex_base = 0; /* the scene's textures */\n"
     "static _Thread_local const uint8_t* const* tl_class_of = 0; /* texture t's texel classes, [h][w] */\n"
     "static _Thread_local int* tl_cls = 0;\n"
     "static _Thread_local size_t tl_cls_px = 0;\n"),
    # the class of the texel shading's u, v fall in, at the pixel centre
    ("      const float u = at[2] * rq, v = at[3] * rq;\n",
     "      const float u = at[2] * rq, v = at[3] * rq;\n"
     "      int cls_cur = 0;\n"
     "      if (tex && tl_class_of) {\n"
     "        const int cu = ((int)floorf(u * (float)tex->w)) & (tex->w - 1), cv = ((int)floorf(v * (float)tex->h)) & (tex->h - 1);\n"
     "        cls_cur = tl_class_of[tex - tl_tex_base][(size_t)cv * tex->w + cu];\n"
     "      }\n"),
    # a sample that passes GL_LESS takes the triangle's class with its 1/w and item
    ("          fb->item[si] = tl_item_cur;\n", "          fb->item[si] = tl_item_cur;\n          fb->cls[si] = cls_cur;\n"),
    ("  fb.item = tl_item;\n",
     "  fb.item = tl_item;\n"
     "  if (tl_cls_px < (size_t)W * H) { free(tl_cls); tl_cls_px = (size_t)W * H; tl_cls = (int*)malloc(sizeof(int) * tl_cls_px * 4); }\n"
     "  fb.cls = tl_cls;\n"),
    ("    fb.item[k] = -1;\n", "    fb.item[k] = -1;\n    fb.cls[k] = 0;\n"),
    # resolve: the label's surface as in the label insertion, then the smallest class among its samples
    ("        tl_label_out[(size_t)y * W + xx] = (int16_t)lab;\n      }\n",
     "        tl_label_out[(size_t)y * W + xx] = (int16_t)lab;\n      }\n"
     "      if (tl_mark_out) {\n"
     "        float qbest = 0.0f;\n"
     "        int lab = 0, mk = 0;\n"
     "        if (valid)\n"
     "          for (int s = 0; s < 4; s++) {\n"
     "            const size_t k = ((size_t)sy * W + sx) * 4 + s;\n"
     "            const float q = fb.q[k];\n"
     "            const int l = fb.item[k] + 1, c = fb.cls[k];\n"
     "            if (!(q > 0.0f)) continue;\n"
     "            if (q > qbest || (q == qbest && l < lab)) { qbest = q; lab = l; mk = c; }\n"
     "            else if (q == qbest && l == lab && c < mk) mk = c;\n"
     "          }\n"
     "        tl_mark_out[(size_t)y * W + xx] = (uint8_t)mk;\n"
     "      }\n"),
]
ENTRY = """
/* orr_render_batch_labels, and every env's marking image into marks_out u8 [n][H][W]; class_of[t]: texture t's classes */
void orr_render_batch_markings(const orr_scene* sc, int n, const double* px, const double* pz, const double* angle,
                               const orr_episode* eps, int W, int H, int domain_rand, const float* lut_x, const float* lut_y,
                               uint8_t* out, float* depth_out, int16_t* labels_out, uint8_t* marks_out,
                               const uint8_t* const* class_of, int threads) {
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int e = 0; e < n; e++) {
    tl_depth_out = depth_out + (size_t)e * W * H;
    tl_label_out = labels_out + (size_t)e * W * H;
    tl_mark_out = marks_out + (size_t)e * W * H;
    tl_tex_base = sc->textures;
    tl_class_of = class_of;
    orr_render(sc, px[e], pz[e], angle[e], &eps[e], W, H, domain_rand, lut_x, lut_y, out + (size_t)e * W * H * 3);
    tl_depth_out = 0;
    tl_label_out = 0;
    tl_mark_out = 0;
    tl_class_of = 0;
  }
}
"""


def patched_source() -> str:
    src = label_oracle.patched_source()
    for old, new in PATCH:
        if src.count(old) != 1:
            raise RuntimeError(f"the label oracle's source no longer has exactly one {old!r}: the marking insertion after "
                               "it must be placed again")
        src = src.replace(old, new)
    return src + ENTRY


_lib = None


def lib():
    global _lib
    if _lib is None:
        # as label_oracle.lib(): the depth oracle's builder compiles this source once, then gets its own back
        src = patched_source()
        saved = depth_oracle._lib, depth_oracle.patched_source
        depth_oracle._lib, depth_oracle.patched_source = None, lambda: src
        try:
            _lib = depth_oracle.lib()
        finally:
            depth_oracle._lib, depth_oracle.patched_source = saved
    return _lib


def class_planes(sc) -> list:
    """The texel classes of every texture of `sc`, an oracle.OracleScene, in its texture order (uint8 [h, w] each)."""
    return sc.holder.keep["tex_cls"]


def render_batch(sc, px, pz, angle, eps=None, W=160, H=120, domain_rand=False, lut=None, segment=False, top_down=False,
                 tile_mode=1, threads=depth_oracle.THREADS):
    """(frames u8 [n, H, W, 3], depth f32 [n, H, W], labels i16 [n, H, W], markings u8 [n, H, W]) of the cameras
    (px, pz, angle) of `sc`, an oracle.OracleScene; eps: their oracle episodes (default: the non-randomised one)."""
    n = len(px)
    eps = eps or [orc.default_episode() for _ in range(n)]
    arr = (orc.OrrEpisode * n)(*eps)
    a = [np.ascontiguousarray(v, np.float64) for v in (px, pz, angle)]
    out, dep = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32)
    lab, mk = np.zeros((n, H, W), np.int16), np.zeros((n, H, W), np.uint8)
    planes = [np.ascontiguousarray(c, np.uint8) for c in class_planes(sc)]
    class_of = (C.c_void_p * max(1, len(planes)))(*[c.ctypes.data for c in planes])
    lx = ly = None
    if lut is not None:
        lx, ly = np.ascontiguousarray(lut[0], np.float32), np.ascontiguousarray(lut[1], np.float32)
    p = lambda v: None if v is None else v.ctypes.data_as(C.c_void_p)
    L = lib()
    L.orr_set_tile_mode(int(tile_mode))
    L.orr_set_render_mode((1 if segment else 0) | (2 if top_down else 0))
    L.orr_render_batch_markings(C.byref(sc.c), n, p(a[0]), p(a[1]), p(a[2]), arr, W, H, int(domain_rand), p(lx), p(ly),
                                p(out), p(dep), p(lab), p(mk), class_of, int(threads))
    return out, dep, lab, mk


def render(sc, px, pz, angle, ep=None, W=160, H=120, domain_rand=False, **kw):
    """(frame u8 [H, W, 3], depth f32 [H, W], labels i16 [H, W], markings u8 [H, W]) of one camera."""
    out, dep, lab, mk = render_batch(sc, [px], [pz], [angle], [ep] if ep is not None else None, W, H, domain_rand,
                                     threads=1, **kw)
    return out[0], dep[0], lab[0], mk[0]
