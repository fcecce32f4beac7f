"""The CPU oracle of the label image (render spec item 10, DESIGN.md section 5): test infrastructure, like oracle/.

A pixel's label is defined from the raster oracle's own visibility, as its depth is, so the label oracle is the depth
oracle's source (tests/depth_oracle.py: oracle/dt_oracle_raster.c with the depth insertions) with the few insertions in
PATCH: the draw item orr_render is drawing — set before the ground, each grid cell, each object and the agent's mesh —,
one more value per sample, the item of the triangle that passed GL_LESS there (beside its 1/w), and at the resolve
1 + the item of the sample with the largest 1/w, the smallest such label among equal ones, 0 where no sample is covered
or the LUT names no source.  Every insertion names the text it follows and must find it exactly once.  One build
returns the frames (the raster oracle's), the depth (the depth oracle's) and the labels; tests/test_oracle_labels.py
holds the first two to those oracles.  It is built by depth_oracle.lib() itself — the depth oracle's builder, handed this
source for one call — so it gets the same compiler flags and lands in the temporary directory under a key of its own
source."""
import ctypes as C

import numpy as np

import depth_oracle
import oracle as orc

# (text of the depth oracle's source, what is put in its place): each replacement is the text itself plus an insertion
PATCH = [
    # the item per sample ([H][W][4], -1 = not covered) and the item being drawn
    ("  float* q;\n} framebuf;\n",
     "  float* q;\n  int* item;\n} framebuf;\n"
     "static _Thread_local int tl_item_cur = 0; /* draw item of the triangles being drawn */\n"
     "static _Thread_local int16_t* tl_label_out = 0; /* i16 [H][W] of the frame being drawn, or none */\n"
     "static _Thread_local int* tl_item = 0;\n"
     "static _Thread_local size_t tl_item_px = 0;\n"),
    # a sample that passes GL_LESS takes the triangle's item with its 1/w
    ("          fb->q[si] = qq;\n", "          fb->q[si] = qq;\n          fb->item[si] = tl_item_cur;\n"),
    ("  fb.q = tl_q;\n",
     "  fb.q = tl_q;\n"
     "  if (tl_item_px < (size_t)W * H) { free(tl_item); tl_item_px = (size_t)W * H; tl_item = (int*)malloc(sizeof(int) * tl_item_px * 4); }\n"
     "  fb.item = tl_item;\n"),
    ("    fb.q[k] = 0.0f;\n", "    fb.q[k] = 0.0f;\n    fb.item[k] = -1;\n"),
    # the three draw sections of orr_render: ground (item 0), grid cell i * grid_h + j (1 + that), object o / the agent
    ("    model_view(V, zero3, 1.0, 1.0, 0.0, x.MV, x.N);\n",
     "    model_view(V, zero3, 1.0, 1.0, 0.0, x.MV, x.N);\n    tl_item_cur = 0;\n"),
    ("      int tile_tex = sc->tile_tex[idx];\n",
     "      int tile_tex = sc->tile_tex[idx];\n      tl_item_cur = 1 + i * sc->grid_h + j;\n"),
    ("    model_view(V, t, (double)ob->scale, cos(th), sin(th), x.MV, x.N);\n    for (int k = 0; k < ob->tri_count; k++) {\n",
     "    model_view(V, t, (double)ob->scale, cos(th), sin(th), x.MV, x.N);\n    for (int k = 0; k < ob->tri_count; k++) {\n"
     "      tl_item_cur = 1 + sc->grid_w * sc->grid_h + o;\n"),
    # resolve: the label of the nearest surface; a maximum of exact values with an exact tie-break, whatever the order
    ("        tl_depth_out[(size_t)y * W + xx] = qmax > 0.0f ? 1.0f / qmax : 0.0f;\n      }\n",
     "        tl_depth_out[(size_t)y * W + xx] = qmax > 0.0f ? 1.0f / qmax : 0.0f;\n      }\n"
     "      if (tl_label_out) {\n"
     "        float qbest = 0.0f;\n"
     "        int lab = 0;\n"
     "        if (valid)\n"
     "          for (int s = 0; s < 4; s++) {\n"
     "            const size_t k = ((size_t)sy * W + sx) * 4 + s;\n"
     "            const float q = fb.q[k];\n"
     "            const int l = fb.item[k] + 1;\n"
     "            if (q > 0.0f && (q > qbest || (q == qbest && l < lab))) { qbest = q; lab = l; }\n"
     "          }\n"
     "        tl_label_out[(size_t)y * W + xx] = (int16_t)lab;\n"
     "      }\n"),
]
ENTRY = """
/* orr_render_batch, and every env's depth image into depth_out f32 [n][H][W] and label image into labels_out i16 [n][H][W] */
void orr_render_batch_labels(const orr_scene* sc, int n, const double* px, const double* pz, const double* angle,
                             const orr_episode* eps, int W, int H, int domain_rand, const float* lut_x, const float* lut_y,
                             uint8_t* out, float* depth_out, int16_t* labels_out, int threads) {
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int e = 0; e < n; e++) {
    tl_depth_out = depth_out + (size_t)e * W * H;
    tl_label_out = labels_out + (size_t)e * W * H;
    orr_render(sc, px[e], pz[e], angle[e], &eps[e], W, H, domain_rand, lut_x, lut_y, out + (size_t)e * W * H * 3);
    tl_depth_out = 0;
    tl_label_out = 0;
  }
}
"""


def patched_source() -> str:
    src = depth_oracle.patched_source()
    for old, new in PATCH:
        if src.count(old) != 1:
            raise RuntimeError(f"the depth oracle's source no longer has exactly one {old!r}: the label insertion after "
                               "it must be placed again")
        src = src.replace(old, new)
    return src + ENTRY


_lib = None


def lib():
    global _lib
    if _lib is None:
        # depth_oracle.lib() compiles whatever its patched_source() returns (cached by a hash of that source) and keeps
        # the result in its _lib: let it build this source once, then give it back its own source and library
        src = patched_source()
        saved = depth_oracle._lib, depth_oracle.patched_source
        depth_oracle._lib, depth_oracle.patched_source = None, lambda: src
        try:
            _lib = depth_oracle.lib()
        finally:
            depth_oracle._lib, depth_oracle.patched_source = saved
    return _lib


def render_batch(sc, px, pz, angle, eps=None, W=160, H=120, domain_rand=False, lut=None, segment=False, top_down=False,
                 tile_mode=1, threads=depth_oracle.THREADS):
    """(frames u8 [n, H, W, 3], depth f32 [n, H, W], labels i16 [n, H, W]) of the cameras (px, pz, angle) of `sc`, an
    oracle.OracleScene; eps: their oracle episodes (default: the non-randomised one)."""
    n = len(px)
    eps = eps or [orc.default_episode() for _ in range(n)]
    arr = (orc.OrrEpisode * n)(*eps)
    a = [np.ascontiguousarray(v, np.float64) for v in (px, pz, angle)]
    out, dep, lab = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32), np.zeros((n, H, W), np.int16)
    lx = ly = None
    if lut is not None:
        lx, ly = np.ascontiguousarray(lut[0], np.float32), np.ascontiguousarray(lut[1], np.float32)
    p = lambda v: None if v is None else v.ctypes.data_as(C.c_void_p)
    L = lib()
    L.orr_set_tile_mode(int(tile_mode))
    L.orr_set_render_mode((1 if segment else 0) | (2 if top_down else 0))
    L.orr_render_batch_labels(C.byref(sc.c), n, p(a[0]), p(a[1]), p(a[2]), arr, W, H, int(domain_rand), p(lx), p(ly),
                              p(out), p(dep), p(lab), int(threads))
    return out, dep, lab


def debug_frame(sc, px, pz, angle, ep=None, W=160, H=120, top_down=False) -> dict:
    """orr_debug_frame of this build (its render mode: top_down gives the camera above the map), as
    oracle.OracleScene.debug_frame returns it."""
    ep = ep or orc.default_episode()
    cells = sc.c.grid_w * sc.c.grid_h
    n_items = 1 + cells + sc.c.n_objects
    V, P = np.zeros(12, np.float64), np.zeros(4, np.float32)
    mv, nn = np.zeros((n_items, 12), np.float32), np.zeros((n_items, 9), np.float32)
    lat = np.zeros((cells, 64, 3), np.float32)
    p = lambda v: v.ctypes.data_as(C.c_void_p)
    L = lib()
    L.orr_set_render_mode(2 if top_down else 0)
    L.orr_debug_frame(C.byref(sc.c), C.c_double(px), C.c_double(pz), C.c_double(angle), C.byref(ep), W, H, 0, p(V), p(P),
                      p(mv), p(nn), p(lat))
    return dict(V=V, P=P, item_mv=mv, item_n=nn, lattice=lat)


def render(sc, px, pz, angle, ep=None, W=160, H=120, domain_rand=False, **kw):
    """(frame u8 [H, W, 3], depth f32 [H, W], labels i16 [H, W]) of one camera."""
    out, dep, lab = render_batch(sc, [px], [pz], [angle], [ep] if ep is not None else None, W, H, domain_rand, threads=1,
                                 **kw)
    return out[0], dep[0], lab[0]
