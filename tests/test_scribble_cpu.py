"""Pins the scribble oracle (oracle/scribble_oracle.py) against cv2 itself and against a direct cv2 transcription of
the reference's make_scribble (controlnet.py:436-454) and xdog lines (controlnet.py:476-482) — CPU only."""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import hed_oracle as HO  # noqa: E402
from oracle import scribble_oracle as S  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINES = [np.array(a, np.uint8) for a in ([[0, 0, 0], [1, 1, 1], [0, 0, 0]], [[0, 1, 0], [0, 1, 0], [0, 1, 0]],
                                         [[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[0, 0, 1], [0, 1, 0], [1, 0, 0]])]


def _cv_nms(g, t):
    y = np.zeros_like(g)
    for f in LINES:
        np.putmask(y, cv2.dilate(g, kernel=f) == g, g)
    z = np.zeros_like(y, dtype=np.uint8)
    z[y > t] = 255
    return z


def _cv_make_scribble(hed_u8):
    r = _cv_nms(cv2.GaussianBlur(hed_u8.astype(np.float32), (0, 0), 3.0), 127)
    r = cv2.GaussianBlur(r, (0, 0), 3.0)
    r[r > 4] = 255
    r[r < 255] = 0
    return r


def _cv_xdog(img, threshold):
    g1 = cv2.GaussianBlur(img.astype(np.float32), (0, 0), 0.5)
    g2 = cv2.GaussianBlur(img.astype(np.float32), (0, 0), 5.0)
    dog = (255 - np.min(g2 - g1, axis=2)).clip(0, 255).astype(np.uint8)
    result = np.zeros_like(img, dtype=np.uint8)
    result[2 * (255 - dog) > threshold] = 255
    return result[..., 0], dog


def _gray_images():
    rng = np.random.RandomState(0)
    yield "random", rng.randint(0, 256, (40, 50)).astype(np.uint8)
    yield "sparse", (rng.rand(64, 80) > 0.97).astype(np.uint8) * 255
    yield "flat", np.full((20, 30), 77, np.uint8)
    yield "9x7", rng.randint(0, 256, (9, 7)).astype(np.uint8)
    yield "3x2", rng.randint(0, 256, (3, 2)).astype(np.uint8)
    yield "1x5", rng.randint(0, 256, (1, 5)).astype(np.uint8)
    yield "1x1", np.array([[200]], np.uint8)
    yield "hed", HO.hed_image(5, 61, 45)[..., 0]


def _hed_like(seed, H, W):
    """A soft-edge-like uint8 map: bright ridges along the level-0.5 contours of a smooth field, dark elsewhere."""
    f = HO.hed_image(seed, H, W)[..., 0].astype(np.float64) / 255.0
    return np.rint(255 * np.exp(-(f - 0.5) ** 2 / 0.004)).astype(np.uint8)


def test_taps_match_opencv():
    for sigma in (0.5, 3.0, 5.0):
        n = S.ksize(sigma, False)
        assert np.array_equal(S.float_taps(sigma), cv2.getGaussianKernel(n, sigma, ktype=cv2.CV_32F).ravel())
    assert S.ksize(3.0, False) == 25 and S.ksize(0.5, False) == 5 and S.ksize(5.0, False) == 41
    assert S.ksize(3.0, True) == 19
    f = S.fixed_taps(3.0)
    # an impulse through a 19x1 blur (the vertical kernel is the fixed-point 1.0) shows the integer taps
    img = np.zeros((1, 64), np.uint8)
    img[0, 32] = 255
    probe = cv2.GaussianBlur(img, (19, 1), 3.0, sigmaY=3.0)[0, 32 - 9:32 + 10].astype(np.int64)
    assert np.array_equal(f, probe) and f.sum() == 256
    assert not np.array_equal(f, np.round(S.gaussian_taps(19, 3.0) * 256))      # not the naively rounded taps


@pytest.mark.parametrize("name,img", list(_gray_images()), ids=[n for n, _ in _gray_images()])
def test_u8_blur_bit_exact(name, img):
    assert np.array_equal(S.blur_u8(img), cv2.GaussianBlur(img, (0, 0), 3.0)), name


@pytest.mark.parametrize("name,img", list(_gray_images()), ids=[n for n, _ in _gray_images()])
def test_float_blurs_close_to_cv2(name, img):
    for sigma in (0.5, 3.0, 5.0):
        ref = cv2.GaussianBlur(img.astype(np.float32), (0, 0), sigma).astype(np.float64)
        err = np.abs(S.blur_f64(img, sigma) - ref).max()
        assert err <= 1e-6 * max(np.abs(ref).max(), 1.0), (name, sigma, err)
        assert err <= S.TOL / 2, (name, sigma, err)         # the tolerance covers cv2's float32 rounding twice over


def test_float_blur_rgb_close_to_cv2():
    img = S.scribble_image(3, 70, 90)
    for sigma in (0.5, 5.0):
        ref = cv2.GaussianBlur(img.astype(np.float32), (0, 0), sigma).astype(np.float64)
        err = np.abs(S.blur_f64(img, sigma) - ref).max()
        assert err <= 1e-6 * 255 and err <= S.TOL / 2, (sigma, err)


@pytest.mark.parametrize("seed,H,W", [(1, 97, 131), (2, 64, 64), (3, 9, 7), (4, 1, 17), (5, 40, 3)])
def test_nms_matches_dilate(seed, H, W):
    g = cv2.GaussianBlur(_hed_like(seed, H, W).astype(np.float32), (0, 0), 3.0)
    flat = np.full((H, W), 130.0, np.float32)
    for m in (g, flat, np.round(g / 8) * 8):                # smooth maps, a plateau, and many exact ties
        zc, zp = S.nms_threshold(m)
        ref = _cv_nms(m, 127) == 255
        assert np.array_equal(zc, ref) and np.array_equal(zp, ref)


@pytest.mark.parametrize("seed,H,W", [(1, 97, 131), (2, 64, 64), (3, 9, 7), (6, 128, 96), (7, 33, 31)])
def test_make_scribble_matches_cv2(seed, H, W):
    hed = _hed_like(seed, H, W)
    ref = _cv_make_scribble(hed)
    out, exempt = S.make_scribble(hed)
    assert not ((out != ref) & ~exempt).any()
    assert exempt.mean() <= 1e-3, exempt.mean()
    assert 0.005 < (ref == 255).mean() < 0.995 or min(H, W) < 16


def test_make_scribble_matches_golden():
    z = np.load(os.path.join(ROOT, "tests", "golden", "scribble_outputs.npz"))
    i = 0
    while f"case_{i}" in z:
        out, exempt = S.make_scribble(z[f"hed_{i}"])
        ref = z[f"scribble_{i}"]
        assert not ((out != ref) & ~exempt).any() and exempt.mean() <= 1e-3, i
        assert 0.05 < (ref == 255).mean() < 0.95, f"case {i} is nearly constant"
        i += 1
    assert i == 4


@pytest.mark.parametrize("seed,H,W", [(1, 97, 131), (2, 256, 256), (3, 9, 7), (4, 33, 31)])
@pytest.mark.parametrize("threshold", [0, 32, 200])
def test_xdog_matches_cv2(seed, H, W, threshold):
    img = S.scribble_image(seed, H, W)
    ref, dog_cv = _cv_xdog(img, threshold)
    out, exempt, dog = S.xdog(img, threshold)
    assert not ((out != ref) & ~exempt).any()
    assert exempt.mean() <= 1e-3, exempt.mean()
    near = np.abs(S.xdog_value(img) - np.round(S.xdog_value(img))) <= S.TOL
    assert not ((dog != dog_cv) & ~near).any()


def test_xdog_uint8_wrap():
    # numpy evaluates 2 * (255 - dog) in uint8: 255 - dog = 128 wraps to 0 (no edge), 200 to 144, 144 to 32
    dog = np.array([127, 55, 111, 238, 255, 0], np.uint8)
    assert (2 * (255 - dog)).dtype == np.uint8
    assert list(S.xdog_from_dog(dog, 32)) == list(2 * (255 - dog) > 32) == [False, True, False, True, False, True]
    # on an image: the darkest strokes land in the wrap range and are edges at threshold 32, not at 200
    img = S.scribble_image(2, 256, 256)
    _, _, dog = S.xdog(img, 32)
    inv = 255 - dog.astype(np.int64)
    wrap = inv >= 128
    assert wrap.sum() >= 100
    ref32, _ = _cv_xdog(img, 32)
    e = (2 * inv) % 256
    assert np.array_equal(ref32[wrap] == 255, e[wrap] > 32)
    assert ((ref32 == 0) & wrap).any() and ((ref32 == 255) & wrap).any()   # the wrap both drops and keeps strokes
