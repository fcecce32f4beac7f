"""Stand-in assets: procedural tile textures and low-poly prop meshes, plus an OBJ/MTL reader.

The reference takes every mesh (`*.obj/*.mtl`), texture and all but two maps from the un-vendored
pip package duckietown-world (objmesh.py:37, simulator.py:638,779) — none of it exists in
`/root/reference`.  This module produces deterministic replacements so that both sides of every
parity test (CUDA kernels and CPU oracle) see the same triangles and texels.  Mesh post-processing
follows the reference loader exactly where it matters for the hot path:
  * re-centring, including the `max(axis=0).min(axis=0)` quirk          objmesh.py:217-232
  * per-vertex colour = material Kd, uv = (0,0) when absent             objmesh.py:184-212
  * textures are RGBA8, bilinear, REPEAT wrap, origin bottom-left       graphics.py:140-169 (pyglet)
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from functools import lru_cache
from typing import Dict, List, Optional, Tuple

import numpy as np

TEX_SIZE = 256


@dataclass
class Mesh:
    name: str
    tri_pos: np.ndarray  # f32 [F,3,3]
    tri_nrm: np.ndarray  # f32 [F,3,3]
    tri_uv: np.ndarray  # f32 [F,3,2]
    tri_col: np.ndarray  # f32 [F,3,3]
    tri_tex: np.ndarray  # i16 [F]   index into `textures`, -1 = untextured chunk
    textures: List[np.ndarray] = field(default_factory=list)  # RGBA8 [h,w,4], row 0 = t=0
    alt_textures: Dict[int, np.ndarray] = field(default_factory=dict)  # texture slot -> the image a TrafficLightObj swaps in
    min_coords: np.ndarray = None
    max_coords: np.ndarray = None

    def recentre(self) -> "Mesh":
        """Base at y=0, centred in x/z — with the reference's quirk (objmesh.py:217-232)."""
        v = self.tri_pos
        min_c = v.min(axis=0).min(axis=0)
        max_c = v.max(axis=0).min(axis=0)  # sic: max over faces, then MIN over the 3 corners
        mean_c = (min_c + max_c) / 2
        v[:, :, 1] -= min_c[1]
        v[:, :, 0] -= mean_c[0]
        v[:, :, 2] -= mean_c[2]
        self.min_coords = v.min(axis=0).min(axis=0)
        self.max_coords = v.max(axis=0).max(axis=0)
        return self


# ----------------------------------------------------------------------------- mesh builders
class _Soup:
    def __init__(self):
        self.p, self.n, self.t, self.c, self.x = [], [], [], [], []

    def tri(self, p, n, col, uv=((0, 0), (0, 0), (0, 0)), tex=-1):
        self.p.append(p)
        self.n.append(n)
        self.t.append(uv)
        self.c.append([col] * 3)
        self.x.append(tex)

    def quad(self, a, b, c, d, col, tex=-1, uvs=((0, 0), (1, 0), (1, 1), (0, 1))):
        a, b, c, d = (np.asarray(v, float) for v in (a, b, c, d))
        n = np.cross(b - a, c - a)
        n = n / (np.linalg.norm(n) + 1e-30)
        self.tri([a, b, c], [n] * 3, col, (uvs[0], uvs[1], uvs[2]), tex)
        self.tri([a, c, d], [n] * 3, col, (uvs[0], uvs[2], uvs[3]), tex)

    def box(self, lo, hi, col, tex=-1):
        x0, y0, z0 = lo
        x1, y1, z1 = hi
        self.quad((x0, y0, z1), (x1, y0, z1), (x1, y1, z1), (x0, y1, z1), col, tex)  # +z
        self.quad((x1, y0, z0), (x0, y0, z0), (x0, y1, z0), (x1, y1, z0), col, tex)  # -z
        self.quad((x1, y0, z1), (x1, y0, z0), (x1, y1, z0), (x1, y1, z1), col, tex)  # +x
        self.quad((x0, y0, z0), (x0, y0, z1), (x0, y1, z1), (x0, y1, z0), col, tex)  # -x
        self.quad((x0, y1, z1), (x1, y1, z1), (x1, y1, z0), (x0, y1, z0), col, tex)  # +y
        self.quad((x0, y0, z0), (x1, y0, z0), (x1, y0, z1), (x0, y0, z1), col, tex)  # -y

    def ellipsoid(self, centre, radii, col, nu=8, nv=5):
        """Smooth-shaded lat/long ellipsoid: nu segments around, nv stacks."""
        cx, cy, cz = centre
        rx, ry, rz = radii

        def pt(iu, iv):
            th = 2 * math.pi * iu / nu
            ph = math.pi * iv / nv
            d = np.array([math.sin(ph) * math.cos(th), math.cos(ph), math.sin(ph) * math.sin(th)])
            p = np.array([cx + rx * d[0], cy + ry * d[1], cz + rz * d[2]])
            n = np.array([d[0] / rx, d[1] / ry, d[2] / rz])
            return p, n / np.linalg.norm(n)

        for iv in range(nv):
            for iu in range(nu):
                (p00, n00), (p10, n10) = pt(iu, iv), pt(iu + 1, iv)
                (p01, n01), (p11, n11) = pt(iu, iv + 1), pt(iu + 1, iv + 1)
                if iv > 0:
                    self.tri([p00, p10, p11], [n00, n10, n11], col)
                if iv < nv - 1:
                    self.tri([p00, p11, p01], [n00, n11, n01], col)

    def cone(self, base_c, r, h, col, nu=10):
        cx, cy, cz = base_c
        apex = np.array([cx, cy + h, cz])
        for iu in range(nu):
            a0, a1 = 2 * math.pi * iu / nu, 2 * math.pi * (iu + 1) / nu
            p0 = np.array([cx + r * math.cos(a0), cy, cz + r * math.sin(a0)])
            p1 = np.array([cx + r * math.cos(a1), cy, cz + r * math.sin(a1)])
            n0 = np.array([math.cos(a0) * h, r, math.sin(a0) * h])
            n1 = np.array([math.cos(a1) * h, r, math.sin(a1) * h])
            n0, n1 = n0 / np.linalg.norm(n0), n1 / np.linalg.norm(n1)
            nm = (n0 + n1) / np.linalg.norm(n0 + n1)
            self.tri([p1, p0, apex], [n1, n0, nm], col)

    def mesh(self, name, textures=()):
        return Mesh(
            name=name,
            tri_pos=np.array(self.p, np.float32), tri_nrm=np.array(self.n, np.float32),
            tri_uv=np.array(self.t, np.float32), tri_col=np.array(self.c, np.float32),
            tri_tex=np.array(self.x, np.int16), textures=list(textures)).recentre()


def _sign_texture(kind: str) -> np.ndarray:
    """Deterministic 64x64 RGBA plate: white border + a kind-hashed colour block pattern."""
    n = 64
    h = sum((i + 1) * ord(ch) for i, ch in enumerate(kind))
    rng = np.random.default_rng(h)
    img = np.full((n, n, 4), 255, np.uint8)
    base = rng.integers(40, 220, 3)
    cells = rng.integers(0, 2, (6, 6))
    for a in range(6):
        for b in range(6):
            col = base if cells[a, b] else (20, 20, 20)
            img[8 + a * 8: 16 + a * 8, 8 + b * 8: 16 + b * 8, :3] = col
    return img


def _build_duckie():
    s = _Soup()
    yellow, orange, black = (0.95, 0.80, 0.10), (0.95, 0.45, 0.05), (0.05, 0.05, 0.05)
    s.ellipsoid((0.0, 0.45, 0.0), (0.45, 0.40, 0.60), yellow)  # body
    s.ellipsoid((0.0, 1.05, 0.35), (0.32, 0.30, 0.32), yellow, nu=8, nv=4)  # head
    s.box((-0.12, 0.95, 0.62), (0.12, 1.05, 0.85), orange)  # beak
    s.box((-0.20, 1.12, 0.60), (-0.12, 1.20, 0.66), black)  # eyes
    s.box((0.12, 1.12, 0.60), (0.20, 1.20, 0.66), black)
    return s.mesh("duckie")


def _build_cone():
    s = _Soup()
    s.box((-0.14, 0.0, -0.14), (0.14, 0.02, 0.14), (0.1, 0.1, 0.1))
    s.cone((0.0, 0.02, 0.0), 0.10, 0.30, (0.95, 0.35, 0.05))
    return s.mesh("cone")


def _build_tree():
    s = _Soup()
    s.box((-0.03, 0.0, -0.03), (0.03, 0.18, 0.03), (0.35, 0.22, 0.10))
    s.cone((0.0, 0.12, 0.0), 0.16, 0.22, (0.10, 0.45, 0.12))
    s.cone((0.0, 0.24, 0.0), 0.12, 0.20, (0.12, 0.52, 0.14))
    return s.mesh("tree")


def _build_house():
    s = _Soup()
    s.box((-0.30, 0.0, -0.22), (0.30, 0.28, 0.22), (0.80, 0.72, 0.60))
    # gable roof
    r = (0.55, 0.15, 0.12)
    s.quad((-0.32, 0.28, 0.24), (0.32, 0.28, 0.24), (0.32, 0.45, 0.0), (-0.32, 0.45, 0.0), r)
    s.quad((0.32, 0.28, -0.24), (-0.32, 0.28, -0.24), (-0.32, 0.45, 0.0), (0.32, 0.45, 0.0), r)
    s.box((-0.06, 0.0, 0.22), (0.06, 0.16, 0.225), (0.30, 0.18, 0.08))
    return s.mesh("house")


def _build_barrier():
    s = _Soup()
    s.box((-0.25, 0.0, -0.04), (0.25, 0.10, 0.04), (0.90, 0.90, 0.90))
    s.box((-0.25, 0.10, -0.03), (0.25, 0.14, 0.03), (0.85, 0.10, 0.10))
    return s.mesh("barrier")


def _build_vehicle(name, body, cab):
    s = _Soup()
    s.box((-0.10, 0.02, -0.22), (0.10, 0.14, 0.22), body)
    s.box((-0.09, 0.14, -0.05), (0.09, 0.22, 0.20), cab)
    for sx in (-0.11, 0.09):
        for sz in (-0.16, 0.12):
            s.box((sx, 0.0, sz), (sx + 0.02, 0.06, sz + 0.06), (0.05, 0.05, 0.05))
    return s.mesh(name)


def _build_sign(kind: str):
    s = _Soup()
    grey = (0.55, 0.55, 0.55)
    s.box((-0.006, 0.0, -0.006), (0.006, 0.10, 0.006), grey)  # pole
    s.box((-0.035, 0.10, -0.004), (0.035, 0.17, 0.0), grey)  # back plate
    # textured face (material "April_Tag" in the reference gets map_Kd = f"{kind}.png", S:965-970)
    s.quad((-0.035, 0.10, 0.0005), (0.035, 0.10, 0.0005), (0.035, 0.17, 0.0005), (-0.035, 0.17, 0.0005),
           (1.0, 1.0, 1.0), tex=0)
    return s.mesh("sign_generic:" + kind, textures=[_sign_texture(kind)])


def _trafficlight_card(pattern: int) -> np.ndarray:
    """Stand-in for trafficlight_card{0,1}.jpg (O:438-441): a dark card with a red and a green lamp whose lit one
    depends on the pattern; the card wraps the four faces of the head, so opposite directions see opposite lamps."""
    n = 64
    img = np.zeros((n, n, 4), np.uint8)
    img[..., :3] = (28, 28, 30)
    img[..., 3] = 255
    yy, xx = np.mgrid[0:n, 0:n]
    for half in (0, 1):                       # left half of the card: N/S faces, right half: E/W faces
        lit_green = (pattern == 0) == (half == 0)
        cx = 16 + 32 * half
        for cy, col_on, col_off, on in ((44, (235, 40, 30), (70, 14, 12), not lit_green),
                                        (20, (40, 230, 60), (14, 66, 20), lit_green)):
            img[(xx - cx) ** 2 + (yy - cy) ** 2 <= 81, :3] = col_on if on else col_off
    return img


def _build_trafficlight():
    s = _Soup()
    s.box((-0.01, 0.0, -0.01), (0.01, 0.30, 0.01), (0.2, 0.2, 0.2))
    x0, x1, y0, y1 = -0.04, 0.04, 0.30, 0.42
    white = (1.0, 1.0, 1.0)
    # head: four card faces (material 0 of the mesh — the texture TrafficLightObj swaps, O:453,462), plain lids
    s.quad((x0, y0, x1), (x1, y0, x1), (x1, y1, x1), (x0, y1, x1), white, 0, ((0.0, 0), (0.5, 0), (0.5, 1), (0.0, 1)))   # +z
    s.quad((x1, y0, x0), (x0, y0, x0), (x0, y1, x0), (x1, y1, x0), white, 0, ((0.0, 0), (0.5, 0), (0.5, 1), (0.0, 1)))   # -z
    s.quad((x1, y0, x1), (x1, y0, x0), (x1, y1, x0), (x1, y1, x1), white, 0, ((0.5, 0), (1.0, 0), (1.0, 1), (0.5, 1)))   # +x
    s.quad((x0, y0, x0), (x0, y0, x1), (x0, y1, x1), (x0, y1, x0), white, 0, ((0.5, 0), (1.0, 0), (1.0, 1), (0.5, 1)))   # -x
    s.quad((x0, y1, x1), (x1, y1, x1), (x1, y1, x0), (x0, y1, x0), (0.15, 0.15, 0.15))
    s.quad((x0, y0, x0), (x1, y0, x0), (x1, y0, x1), (x0, y0, x1), (0.15, 0.15, 0.15))
    m = s.mesh("trafficlight", textures=[_trafficlight_card(0)])
    m.alt_textures = {0: _trafficlight_card(1)}
    return m


_BUILDERS = {
    "duckie": _build_duckie,
    "cone": _build_cone,
    "tree": _build_tree,
    "house": _build_house,
    "barrier": _build_barrier,
    "bus": lambda: _build_vehicle("bus", (0.95, 0.75, 0.10), (0.60, 0.75, 0.90)),
    "truck": lambda: _build_vehicle("truck", (0.20, 0.35, 0.70), (0.85, 0.85, 0.85)),
    "duckiebot": lambda: _build_vehicle("duckiebot", (0.80, 0.10, 0.10), (0.20, 0.20, 0.20)),
    "trafficlight": _build_trafficlight,
}

_MESH_CACHE: Dict[str, Mesh] = {}
MESH_SEARCH_PATH: List[str] = []  # directories holding real <kind>.obj/.mtl, searched first


def get_mesh(kind: str) -> Mesh:
    """Mesh for an object kind (cached like objmesh.get_mesh, M:28-50).  Real OBJ files found on
    MESH_SEARCH_PATH win over the procedural stand-ins."""
    key = kind
    if key in _MESH_CACHE:
        return _MESH_CACHE[key]
    file_kind = "sign_generic" if kind.startswith("sign") else kind
    for d in MESH_SEARCH_PATH:
        p = os.path.join(d, f"{file_kind}.obj")
        if os.path.isfile(p):
            _MESH_CACHE[key] = load_obj(p, kind)
            return _MESH_CACHE[key]
    if kind.startswith("sign"):
        m = _build_sign(kind)
    elif kind in _BUILDERS:
        m = _BUILDERS[kind]()
    else:
        raise KeyError(f"no mesh for object kind {kind!r}")
    _MESH_CACHE[key] = m
    return m


def mesh_extents() -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    """kind -> (min_coords, max_coords); handed to the reference-code harness in tests."""
    return {k: (get_mesh(k).min_coords, get_mesh(k).max_coords) for k in _BUILDERS}


# ----------------------------------------------------------------------------- segmentation assets (render_obs(segment=True))
def gen_segmentation_color(name: str) -> List[int]:
    """ObjMesh's per-class colour (objmesh.py:260-266): the decimal character codes of the mesh name concatenated,
    cut into 3-digit groups, each `% 255`; the first three groups."""
    hashed = "".join(str(ord(ch)) for ch in name)
    col = [int(hashed[i:i + 3]) % 255 for i in range(0, len(hashed), 3)][:3]
    assert len(col) == 3
    return col


def should_segment_out(tex_path: str) -> bool:
    """graphics.py:59-67: which textures are replaced by one flat colour; the others keep their lane markings."""
    for yes in ["sign", "trafficlight", "asphalt"]:
        if yes in tex_path:
            return True
    for no in ["left", "right", "way", "curve", "straight"]:
        if no in tex_path:
            return False
    return True


def flat_texture(rgb) -> np.ndarray:
    """load_texture(..., segment=True) of a segmented-out texture (graphics.py:92-98): every texel = `rgb`."""
    t = np.zeros((1, 1, 4), np.uint8)
    t[0, 0, :3] = [int(v) & 255 for v in rgb]
    t[0, 0, 3] = 255
    return t


def segment_tile_texture(kind: str, rgba: np.ndarray, style: str = "photos") -> np.ndarray:
    """Texture.bind(segment=True) for a road tile (graphics.py:52-56, 70-130): the texture path decides — grass, floor,
    asphalt are flattened to black; tiles with lane markings keep what survives the reference's HSV filter (everything
    outside H 0-179 / S 0-100 / V 0-160, i.e. bright or saturated paint, minus pixels that lose an 8-neighbour)."""
    path = f"tiles-processed/{style}/{kind}/texture"
    if should_segment_out(path):
        return flat_texture([0, 0, 0])
    try:
        import cv2
    except ImportError as e:   # the reference needs cv2 for this too
        raise RuntimeError("segmentation textures need OpenCV (cv2), as in the reference (graphics.py:100-121)") from e
    im = np.ascontiguousarray(rgba[:, :, 2::-1])             # cv2.imread gives BGR
    hsv = cv2.cvtColor(im, cv2.COLOR_BGR2HSV)
    mask = cv2.inRange(hsv, np.array([0, 0, 0], np.uint8), np.array([179, 100, 160], np.uint8))
    mask = cv2.bitwise_not(mask)
    k1 = np.array([[0, 0, 0], [0, 1, 0], [0, 0, 0]], np.uint8)
    k2 = np.array([[1, 1, 1], [1, 0, 1], [1, 1, 1]], np.uint8)
    h1 = cv2.morphologyEx(mask, cv2.MORPH_ERODE, k1)
    h2 = cv2.morphologyEx(h1, cv2.MORPH_ERODE, k2)
    mask = cv2.bitwise_and(h1, h2)
    res = cv2.bitwise_and(hsv, hsv, mask=mask)
    bgr = cv2.cvtColor(res, cv2.COLOR_HSV2BGR)
    out = np.full(rgba.shape, 255, np.uint8)
    out[:, :, :3] = bgr[:, :, ::-1]
    return out


# ----------------------------------------------------------------------------- lane-marking classes (render spec item 11)
MARKING_NAMES = ("none", "tile", "white", "yellow", "red")
MARK_NONE, MARK_TILE, MARK_WHITE, MARK_YELLOW, MARK_RED = range(5)


def tile_texel_classes(kind: str, rgba: np.ndarray, style: str = "photos") -> np.ndarray:
    """uint8 [h, w], row 0 = t=0 as the texels: the marking class of every texel of road tile `kind`'s texture `rgba`.
    Paint is what the reference's own filter keeps, segment_tile_texture(kind, rgba) not black (so a kind it flattens
    has none, and the erosion trims a texel off each side of a line); an unpainted texel is MARK_TILE.  A painted texel's
    class comes from OpenCV's HSV of the texel itself (H 0-179, S and V 0-255): S <= 100 white, else 11 <= H <= 45
    yellow, else red.  The thresholds are this project's: the reference has no classes."""
    h, w = rgba.shape[:2]
    cls = np.full((h, w), MARK_TILE, np.uint8)
    if should_segment_out(f"tiles-processed/{style}/{kind}/texture"):
        return cls
    import cv2   # (segment_tile_texture has already required it)
    paint = segment_tile_texture(kind, rgba, style)[:, :, :3].any(axis=2)
    hsv = cv2.cvtColor(np.ascontiguousarray(rgba[:, :, 2::-1]), cv2.COLOR_BGR2HSV)
    hue, sat = hsv[:, :, 0], hsv[:, :, 1]
    painted = np.where(sat <= 100, MARK_WHITE, np.where((hue >= 11) & (hue <= 45), MARK_YELLOW, MARK_RED))
    cls[paint] = painted[paint]
    return cls


def mesh_texel_classes(rgba: np.ndarray) -> np.ndarray:
    """uint8 [h, w] of zeros: a mesh's texels (signs, traffic-light cards, flat segment colours) are never road."""
    return np.zeros(rgba.shape[:2], np.uint8)


# ----------------------------------------------------------------------------- OBJ / MTL reader
def load_obj(path: str, name: str, texture_loader=None) -> Mesh:
    """Wavefront reader with the reference loader's semantics (objmesh.py:65-293): triangles only,
    faces sorted by material, per-vertex colour = Kd (default white), uv (0,0) when absent,
    default material picks `<name>.png` if it exists, then `recentre()`."""
    model_dir, file_name = os.path.split(path)
    stem = file_name.split(".")[0]
    materials: Dict[str, dict] = {"": {"Kd": np.array([1.0, 1.0, 1.0])}}
    if os.path.isfile(os.path.join(model_dir, stem + ".png")):
        materials[""]["map_Kd"] = os.path.join(model_dir, stem + ".png")
    mtl_path = os.path.join(model_dir, stem + ".mtl")
    if os.path.isfile(mtl_path):
        cur = None
        for line in open(mtl_path):
            tok = line.split()
            if not tok or tok[0].startswith("#"):
                continue
            if tok[0] == "newmtl":
                cur = {}
                materials[tok[1]] = cur
            elif tok[0] == "Kd" and cur is not None:
                cur["Kd"] = np.array([float(v) for v in tok[1:4]])
            elif tok[0] == "map_Kd" and cur is not None:
                cur["map_Kd"] = os.path.join(model_dir, tok[-1])
    verts, texs, norms, faces = [], [], [], []
    cur_mtl = ""
    for line in open(path):
        tok = line.split()
        if not tok or tok[0].startswith("#"):
            continue
        if tok[0] == "v":
            verts.append([float(v) for v in tok[1:4]])
        elif tok[0] == "vt":
            texs.append([float(v) for v in tok[1:3]])
        elif tok[0] == "vn":
            norms.append([float(v) for v in tok[1:4]])
        elif tok[0] == "usemtl":
            cur_mtl = tok[1] if tok[1] in materials else ""
        elif tok[0] == "f":
            assert len(tok) == 4, "only triangle faces are supported"
            face = [[int(i) for i in t.split("/") if i != ""] for t in tok[1:]]
            faces.append((face, cur_mtl))
    faces.sort(key=lambda f: f[1])
    tex_index: Dict[str, int] = {}
    textures: List[np.ndarray] = []
    s = _Soup()
    for face, mtl in faces:
        m = materials[mtl]
        col = tuple(m.get("Kd", np.array([1.0, 1.0, 1.0])))
        tex = -1
        if "map_Kd" in m and texture_loader is not None:
            if m["map_Kd"] not in tex_index:
                tex_index[m["map_Kd"]] = len(textures)
                textures.append(texture_loader(m["map_Kd"]))
            tex = tex_index[m["map_Kd"]]
        p, n, t = [], [], []
        for idx in face:
            if len(idx) == 3:
                p.append(verts[idx[0] - 1]); t.append(texs[idx[1] - 1]); n.append(norms[idx[2] - 1])
            else:
                p.append(verts[idx[0] - 1]); n.append(norms[idx[1] - 1]); t.append([0, 0])
        s.tri(p, n, col, t, tex)
    return s.mesh(name, textures)


# ----------------------------------------------------------------------------- tile textures
def _value_noise(n: int, seed: int, octaves=(8, 32, 128)) -> np.ndarray:
    rng = np.random.default_rng(seed)
    out = np.zeros((n, n))
    yy, xx = np.mgrid[0:n, 0:n]
    for o in octaves:
        g = rng.random((o + 1, o + 1))
        fx, fy = xx * o / n, yy * o / n
        ix, iy = fx.astype(int), fy.astype(int)
        tx, ty = fx - ix, fy - iy
        a = g[iy, ix] * (1 - tx) + g[iy, ix + 1] * tx
        b = g[iy + 1, ix] * (1 - tx) + g[iy + 1, ix + 1] * tx
        out += (a * (1 - ty) + b * ty) / len(octaves)
    return out


def _bezier_samples(template, m=48):
    t = np.linspace(0, 1, m)[:, None]
    p = np.array(template, float)
    return ((1 - t) ** 3) * p[0] + 3 * t * (1 - t) ** 2 * p[1] + 3 * t ** 2 * (1 - t) * p[2] + t ** 3 * p[3]


@lru_cache(maxsize=None)
def tile_texture(kind: str, n: int = TEX_SIZE) -> np.ndarray:
    """RGBA8 [n,n,4], row 0 = texture t=0.  Drivable kinds get asphalt + lane paint laid out
    around the same Bezier templates the lane-pose code uses: a texel (u,v) shows template point
    (0.5-u, v-0.5), because tiles are drawn with Ry(angle*90+180) (S:1872-1873) and uv=(pu,1-pv)
    (S:394-401) while the curves are rotated by angle*90 only (S:1331)."""
    from .maps import _TEMPLATES  # local import: maps imports assets

    seed = 1000 + sum(ord(c) for c in kind)
    noise = _value_noise(n, seed)
    img = np.zeros((n, n, 4), np.uint8)
    img[..., 3] = 255
    if kind == "grass":
        base = np.array([60, 140, 50])[None, None, :] * (0.75 + 0.5 * noise[..., None])
        img[..., :3] = np.clip(base, 0, 255)
        return img
    if kind == "floor":
        base = np.array([170, 150, 120])[None, None, :] * (0.85 + 0.3 * noise[..., None])
        img[..., :3] = np.clip(base, 0, 255)
        return img
    asphalt = np.array([55, 55, 58])[None, None, :] * (0.8 + 0.4 * noise[..., None])
    rgb = np.clip(asphalt, 0, 255)
    key = "3way" if kind.startswith("3way") else kind
    if key in _TEMPLATES:
        v, u = np.mgrid[0:n, 0:n]
        px = 0.5 - (u + 0.5) / n
        pz = (v + 0.5) / n - 0.5
        q = np.stack([px, pz], -1)[:, :, None, :]
        dists = []
        for tpl in _TEMPLATES[key]:
            s = _bezier_samples(tpl)[None, None, :, :]
            dists.append(np.sqrt(((q - s) ** 2).sum(-1)).min(-1))
        d = np.sort(np.stack(dists, -1), -1)
        d1, d2 = d[..., 0], d[..., 1]
        yellow = (np.abs(d1 - 0.2) < 0.012) & (np.abs(d2 - 0.2) < 0.03)
        dash = ((np.floor((px + pz + 1.0) * 10) % 2) == 0)
        white = (np.abs(d1 - 0.23) < 0.012) & (d2 > 0.3)
        rgb[yellow & dash] = (235, 200, 30)
        rgb[white] = (235, 235, 235)
    img[..., :3] = rgb
    return img
