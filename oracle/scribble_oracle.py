"""CPU restatement of the scribble pre-processing of ControlNet.preprocess(type='scribble').  TEST INFRASTRUCTURE —
only tests/ and tools/ may import this module.  It does not import cv2: the GPU tests use it on machines without it.

Reference path: lib/model_zoo/controlnet.py:432-491.
  method='hed'  apply_hed, then make_scribble (:436-454): cv2.GaussianBlur(float32(u8), (0,0), 3) -> keep the pixels
                that equal cv2.dilate along at least one of four 3-tap lines -> `> 127` -> 255 -> cv2.GaussianBlur of
                that uint8 map with sigma 3 -> 255 where `> 4`.
  method='xdog' (:476-482) g1, g2 = float32 cv2.GaussianBlur(rgb_u8) with sigma 0.5 and 5; dog =
                uint8(clip(255 - min_c(g2 - g1), 0, 255)); 255 where uint8(2 * uint8(255 - dog)) > threshold (the
                numpy uint8 product wraps mod 256).
OpenCV's operators are restated from its published algorithm (modules/imgproc/src/smooth.*): kernel size
round(sigma * (3 for uint8, 4 for float32) * 2 + 1) | 1; taps exp(-x^2 / (2 sigma^2)) in float64 normalised by the
reciprocal of their sum (getGaussianKernel), rounded to float32 for float images; for uint8 images 8-fractional-bit
integer taps rounded from the outside in with the rounding error carried forward (the centre tap takes the rest of
256), integer row and column sums and (sum + 2^15) >> 16.  BORDER_REFLECT_101 everywhere; cv2.dilate ignores pixels
outside the image.  tests/test_scribble_cpu.py pins all of it against cv2 itself.

The uint8 blur here is exact.  The float blurs are computed in float64 from the float32 taps, i.e. without the float32
rounding that cv2 and the GPU each add in their own order; decisions that depend on them are therefore returned as
(certain, possible) pairs with the deciding margin widened by TOL, and a pixel is *exempt* when the two disagree.
"""
import numpy as np

# Deciding-margin tolerance of the float32 blurs, in the units of the maps (0..255): 16 float32 ulps at 255.  The
# float32 blurs of cv2 are within 9e-5 of the float64 blur on 0..255 maps (tests/test_scribble_cpu.py checks TOL / 2).
TOL = 16 * 2.0 ** -16


def ksize(sigma, u8):
    return int(round(sigma * (3 if u8 else 4) * 2 + 1)) | 1


def gaussian_taps(n, sigma):
    """getGaussianKernel(n, sigma) in float64."""
    s2 = -0.125 / (sigma * sigma)
    h = (n - 1) // 2
    v = np.array([np.exp(float((1 - n + 2 * i) ** 2) * s2) for i in range(h)], np.float64)
    total = 0.0
    for t in v:                                              # sequential sum, as OpenCV does
        total += t
    mul = 1.0 / (total * 2.0 + 1.0)
    k = np.empty(n, np.float64)
    k[:h] = v * mul
    k[n - h:] = k[:h][::-1]
    k[h] = mul
    return k


def float_taps(sigma):
    """The float32 taps of a float32 image's GaussianBlur."""
    return gaussian_taps(ksize(sigma, False), sigma).astype(np.float32)


def fixed_taps(sigma):
    """The 8-fractional-bit integer taps of a uint8 image's GaussianBlur (they sum to 256)."""
    k = gaussian_taps(ksize(sigma, True), sigma)
    n = len(k)
    f = np.zeros(n, np.int64)
    err = 0.0
    for i in range(n // 2):
        a = k[i] * 256.0 + err
        v = int(np.rint(a))
        err = a - v
        f[i] = f[n - 1 - i] = v
    f[n // 2] = 256 - 2 * int(f[:n // 2].sum())
    return f


def reflect101(i, n):
    if n == 1:
        return 0
    while i < 0 or i >= n:
        i = -i if i < 0 else 2 * (n - 1) - i
    return i


def _sep(img, k, acc_dtype):
    """Separable filter with BORDER_REFLECT_101 (rows, then columns) on an [H, W] or [H, W, C] array."""
    H, W = img.shape[:2]
    r = len(k) // 2
    xs = np.array([reflect101(i, W) for i in range(-r, W + r)])
    ys = np.array([reflect101(i, H) for i in range(-r, H + r)])
    a = img.astype(acc_dtype)
    row = sum(acc_dtype(k[j]) * a[:, xs[j:j + W]] for j in range(len(k)))
    return sum(acc_dtype(k[i]) * row[ys[i:i + H]] for i in range(len(k)))


def blur_u8(img, sigma=3.0):
    """cv2.GaussianBlur(img_u8, (0, 0), sigma), bit-exact."""
    c = _sep(np.asarray(img, np.uint8), fixed_taps(sigma), np.int64)
    return ((c + (1 << 15)) >> 16).clip(0, 255).astype(np.uint8)


def blur_f64(img, sigma):
    """cv2.GaussianBlur(float32(img), (0, 0), sigma) in float64 arithmetic (float32 taps)."""
    return _sep(np.asarray(img, np.float32), float_taps(sigma).astype(np.float64), np.float64)


LINES = ((0, 1), (1, 0), (1, 1), (1, -1))                   # the four 3-tap dilate kernels of make_scribble's nms


def nms_margin(g):
    """max over the four lines of min(g - neighbour) over the line's in-image neighbours: cv2.dilate(g, line) == g
    for some line exactly when the margin is >= 0 (+inf on a 1x1 image)."""
    g = np.asarray(g, np.float64)
    H, W = g.shape
    p = np.full((H + 2, W + 2), -np.inf)
    p[1:-1, 1:-1] = g
    best = np.full((H, W), -np.inf)
    for dy, dx in LINES:
        a = p[1 - dy:H + 1 - dy, 1 - dx:W + 1 - dx]
        b = p[1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx]
        best = np.maximum(best, np.minimum(g - a, g - b))
    return best


def nms_threshold(g, tol=0.0):
    """nms(., 127) after the blur -> (certain, possible) boolean maps of z == 255: the decision with every margin
    lowered, and raised, by tol (both are the exact decision when tol == 0)."""
    m = nms_margin(g)
    g = np.asarray(g, np.float64)
    return (m - tol >= 0) & (g - tol > 127), (m + tol >= 0) & (g + tol > 127)


def make_scribble(hed_u8, tol=TOL):
    """make_scribble of a uint8 [H, W] HED map -> (uint8 scribble map 0/255, exempt mask).  Exempt pixels are those
    whose output changes when the NMS / `> 127` decisions that lie within tol of a tie go the other way."""
    zc, zp = nms_threshold(blur_f64(hed_u8, 3.0), tol)
    lo = blur_u8(zc.astype(np.uint8) * 255) > 4
    hi = blur_u8(zp.astype(np.uint8) * 255) > 4
    return np.where(lo, 255, 0).astype(np.uint8), lo != hi


def xdog_value(img_u8):
    """255 - min_c(g2 - g1) in float64 for an [H, W, 3] uint8 image (before the clip and uint8 truncation)."""
    d = blur_f64(img_u8, 5.0) - blur_f64(img_u8, 0.5)
    return 255.0 - d.min(axis=2)


def xdog_from_dog(dog, threshold):
    """The thresholding lines with numpy's uint8 arithmetic: uint8(2 * uint8(255 - dog)) > threshold."""
    dog = np.asarray(dog, np.uint8)
    e = (2 * (255 - dog.astype(np.int64))) % 256
    return e > threshold


def xdog(img_u8, threshold=32, tol=TOL):
    """-> (uint8 map 0/255, exempt mask, dog): exempt where the truncation of 255 - min_c(g2 - g1) moved by +-tol
    changes the decision."""
    v = xdog_value(img_u8)
    dogs = [np.floor(np.clip(v + s, 0, 255)).astype(np.uint8) for s in (-tol, 0.0, tol)]
    e = [xdog_from_dog(d, threshold) for d in dogs]
    return np.where(e[1], 255, 0).astype(np.uint8), (e[0] != e[1]) | (e[2] != e[1]), dogs[1]


def scribble_image(seed, H, W):
    """HxWx3 uint8 test image for xdog: a smooth coloured background with thin dark strokes and dots of several
    strengths, so that 255 - dog spans 0..255, the uint8 wrap range (>= 128) included."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.empty((H, W, 3), np.float64)
    for c in range(3):
        fy, fx, ph = rng.uniform(0.01, 0.08), rng.uniform(0.01, 0.08), rng.uniform(0, 6.3)
        img[..., c] = 200 + 40 * np.sin(fy * yy + ph) * np.cos(fx * xx)
    for _ in range(max(4, H * W // 400)):
        depth = rng.uniform(20, 255)
        if rng.rand() < 0.5:                                 # a 1-2 pixel wide line
            y, x0, x1 = rng.randint(0, H), rng.randint(0, W), rng.randint(0, W)
            img[y:y + rng.randint(1, 3), min(x0, x1):max(x0, x1) + 1] -= depth
        else:                                                # a dot
            y, x = rng.randint(0, H), rng.randint(0, W)
            img[y:y + 2, x:x + 2] -= depth
    img += rng.normal(0, 3, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)
