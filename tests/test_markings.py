"""The texel classes behind the lane-marking image (render spec item 11): assets.tile_texel_classes on every stand-in
tile texture, and the planes the blob builder hands the library and the oracle, one per texture in texture order."""
import numpy as np
import pytest

from gym_duckietown_b200 import assets
from gym_duckietown_b200 import lib as L
from gym_duckietown_b200.maps import TILE_KINDS, load_map

M = assets


@pytest.mark.parametrize("kind", TILE_KINDS)
def test_paint_is_what_the_segment_filter_keeps(kind):
    tex = assets.tile_texture(kind)
    cls = assets.tile_texel_classes(kind, tex)
    assert cls.shape == tex.shape[:2] and cls.dtype == np.uint8
    assert set(np.unique(cls)) <= {M.MARK_TILE, M.MARK_WHITE, M.MARK_YELLOW, M.MARK_RED}
    paint = assets.segment_tile_texture(kind, tex)[:, :, :3].any(axis=2)
    if paint.shape == cls.shape:
        assert np.array_equal(cls != M.MARK_TILE, paint)
    else:   # a kind the filter flattens: no paint at all
        assert not paint.any() and (cls == M.MARK_TILE).all()


@pytest.mark.parametrize("kind", ["grass", "floor", "asphalt"])
def test_flattened_kinds_are_all_tile(kind):
    assert (assets.tile_texel_classes(kind, assets.tile_texture(kind)) == M.MARK_TILE).all()


def stand_in_paint(kind):
    """(yellow, white, asphalt) texel masks of the stand-in texture by its colours: the paint it was drawn with"""
    rgb = assets.tile_texture(kind)[:, :, :3].astype(int)
    yellow = (rgb == (235, 200, 30)).all(-1)
    white = (rgb == (235, 235, 235)).all(-1)
    return yellow, white, ~(yellow | white)


def interior(mask):
    """texels of `mask` whose 8 neighbours are in it too (the reference filter's erosion trims the rest)"""
    m = np.pad(mask, 1)
    out = np.ones_like(mask)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            out &= m[1 + dy:1 + dy + mask.shape[0], 1 + dx:1 + dx + mask.shape[1]]
    return out


@pytest.mark.parametrize("kind", ["straight", "curve_left", "curve_right", "3way_left", "4way"])
def test_stand_in_paint_classes(kind):
    """The stand-in yellow dashes are yellow, white lines white, asphalt plain tile; paint loses at most its rim."""
    cls = assets.tile_texel_classes(kind, assets.tile_texture(kind))
    yellow, white, asphalt = stand_in_paint(kind)
    assert (cls[asphalt] == M.MARK_TILE).all()
    assert np.isin(cls[yellow], (M.MARK_TILE, M.MARK_YELLOW)).all()
    assert np.isin(cls[white], (M.MARK_TILE, M.MARK_WHITE)).all()
    assert (cls[interior(yellow)] == M.MARK_YELLOW).all() and (cls[interior(white)] == M.MARK_WHITE).all()
    assert (cls == M.MARK_YELLOW).sum() + (cls == M.MARK_WHITE).sum() > 0


def test_a_red_bar_is_red():
    tex = assets.tile_texture("straight").copy()
    tex[100:110, 20:200, :3] = (220, 30, 40)        # a stop line: H 178, S 220
    cls = assets.tile_texel_classes("straight", tex)
    assert (cls[101:109, 21:199] == M.MARK_RED).all()
    assert np.isin(cls[100:110, 20:200], (M.MARK_TILE, M.MARK_RED)).all()


def test_hsv_thresholds():
    """One painted texel block per colour: S <= 100 white; else 11 <= H <= 45 yellow; else red."""
    tex = assets.tile_texture("straight").copy()
    cols = {(230, 230, 200): M.MARK_WHITE, (235, 200, 30): M.MARK_YELLOW, (240, 120, 20): M.MARK_YELLOW,
            (60, 200, 60): M.MARK_RED, (200, 40, 200): M.MARK_RED}
    for k, c in enumerate(cols):
        tex[10 + 20 * k:20 + 20 * k, 100:120, :3] = c
    cls = assets.tile_texel_classes("straight", tex)
    for k, want in enumerate(cols.values()):
        assert (cls[11 + 20 * k:19 + 20 * k, 101:119] == want).all(), list(cols)[k]


def test_blob_planes():
    """Every texture gets a plane of its own size, in texture order: tile kinds classified, meshes' textures 0, and each
    segment replacement the plane of the texture it replaces (a flattened kind's 1x1 replacement: one MARK_TILE)."""
    md = load_map("udem1")
    h = L.MapBlobHolder(md)
    k = h.keep
    planes, imgs, seg = k["tex_cls"], k["tex_imgs"], k["seg"]
    assert len(planes) == len(imgs)
    assert all(p.shape == im.shape[:2] and p.dtype == np.uint8 for p, im in zip(planes, imgs))
    assert np.array_equal(k["tex_class"], np.concatenate([p.ravel() for p in planes]))
    kinds = sorted(set(int(x) for x in md.tile_kind if x >= 0))
    assert h.n_tile_tex == len(kinds)
    for ti, kid in enumerate(kinds):
        assert np.array_equal(planes[ti], assets.tile_texel_classes(TILE_KINDS[kid], imgs[ti]))
        s = int(seg[ti])
        assert s != ti
        if planes[s].shape == planes[ti].shape:
            assert np.array_equal(planes[s], planes[ti])
        else:
            assert planes[s].shape == (1, 1) and planes[s][0, 0] == M.MARK_TILE and (planes[ti] == M.MARK_TILE).all()
    tile_seg = {int(seg[ti]) for ti in range(h.n_tile_tex)}
    for t in range(h.n_tile_tex, len(planes)):
        if t not in tile_seg:
            assert not planes[t].any(), f"texture {t} belongs to a mesh"
    assert h.blob.tex_class == k["tex_class"].ctypes.data


def test_marking_names_are_exported():
    import gym_duckietown_b200 as g
    assert g.MARKING_NAMES == ("none", "tile", "white", "yellow", "red")
