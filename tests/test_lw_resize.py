"""learning/utils/wrappers.py's ResizeWrapper (scipy.misc.imresize = Pillow BILINEAR): the numpy restatement in
oracle/pil_resize.py, which the GPU tests compare the device pass with, against what the reference class returned
(tests/golden/lw_resize.npz, oracle/make_golden_lw.py) and, where Pillow is importable, against Pillow itself."""
import os

import numpy as np
import pytest

import pil_resize as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "lw_resize.npz")

CASES = [(tag, shape) for tag, shapes in P.SOURCES.items() for shape in shapes]


def test_golden_covers_the_listed_sizes_and_frames_regenerate_from_the_seed():
    g = np.load(GOLD)
    for tag in P.SOURCES:
        w, h = map(int, tag.split("x"))
        assert P.sha(P.canned_frames(int(g["seed"]), w, h)) == str(g[f"frames_sha_{tag}"]), tag
    for tag, shape in CASES:
        key = P.golden_key(tag, shape)
        assert len(str(g[key + "_sha"])) == 64
        if shape[0] * shape[1] <= P.GOLDEN_ARRAY_MAX_PIXELS:
            assert g[key].shape == (3,) + shape and P.sha(g[key]) == str(g[key + "_sha"])
        else:
            assert key not in g.files


def check_against_golden(g, tag, shape, got):
    """`got` u8 [3][h][w][3] is what the reference class returned: its digest, and the frames where they are stored."""
    key = P.golden_key(tag, shape)
    if key in g.files:
        assert np.array_equal(got, g[key])
    assert P.sha(got) == str(g[key + "_sha"])


@pytest.mark.parametrize("tag,shape", CASES)
def test_restatement_equals_the_reference_resize_wrapper(tag, shape):
    g = np.load(GOLD)
    w, h = map(int, tag.split("x"))
    frames = P.canned_frames(int(g["seed"]), w, h)
    check_against_golden(g, tag, shape, P.resize(frames, shape[1], shape[0]))
    check_against_golden(g, tag, shape, np.stack([P.resize(f, shape[1], shape[0]) for f in frames]))   # per frame


@pytest.mark.parametrize("tag,shape", CASES)
def test_imresize_standin_reproduces_the_golden(tag, shape):
    pytest.importorskip("PIL")
    g = np.load(GOLD)
    w, h = map(int, tag.split("x"))
    frames = P.canned_frames(int(g["seed"]), w, h)
    check_against_golden(g, tag, shape, np.stack([P.imresize_standin(f, shape) for f in frames]))


def test_imresize_standin_refuses_what_scipy_1_2_would_have_converted():
    pytest.importorskip("PIL")
    img = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(NotImplementedError):
        P.imresize_standin(img.astype(np.float32), (4, 4, 3))
    with pytest.raises(NotImplementedError):
        P.imresize_standin(img, (4, 4))
    with pytest.raises(NotImplementedError):
        P.imresize_standin(img, (4, 4, 3), interp="bicubic")


def test_restatement_equals_pillow_on_a_sweep_of_shapes():
    pytest.importorskip("PIL")
    from PIL import Image
    rng = np.random.default_rng(5)
    cases = [(640, 480, 160, 120), (640, 480, 84, 84), (640, 480, 20, 15), (640, 480, 640, 120), (640, 480, 160, 480),
             (160, 120, 84, 84), (100, 76, 160, 120), (101, 77, 33, 19), (7, 5, 3, 9), (1, 1, 4, 3), (33, 17, 1, 1)]
    for _ in range(30):
        w, h = (int(v) for v in rng.integers(1, 240, 2))
        cases.append((w, h, int(rng.integers(w // 32 + 1, 330)), int(rng.integers(h // 32 + 1, 330))))
    for w, h, ow, oh in cases:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if rng.random() < 0.5:
            img[: h // 2] = 255
            img[:, : w // 3] = 0
        want = np.array(Image.fromarray(img).resize((ow, oh), Image.BILINEAR))
        assert np.array_equal(P.resize(img, ow, oh), want), (w, h, ow, oh)


def test_identity_axis_is_an_exact_copy():
    xmin, kk = P.axis_coeffs(160, 160)
    assert np.array_equal(xmin, np.arange(160)) and (kk[:, 0] == 1 << 22).all() and (kk[:, 1:] == 0).all()
