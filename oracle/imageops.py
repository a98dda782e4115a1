"""ORACLE (test infrastructure, not product): NumPy models of the three fixed-point image algorithms the app's host
code runs around the pipelines, restated from their published descriptions and pinned byte for byte against the
libraries themselves in tests/test_app_flow_cpu.py:

- `resize`: Pillow's `Image.resize` for modes L / RGB with BILINEAR, BICUBIC (a = -0.5) or LANCZOS (3 lobes). The
  coefficient tables are computed in double precision, normalised, and quantised to 22 fractional bits; the image
  goes through a horizontal then a vertical integer pass, each clipped to uint8. A pass whose size does not change
  is skipped; when neither changes the result is a copy.
- `gaussian_blur`: Pillow's `ImageFilter.GaussianBlur`, an extended box blur (three horizontal then three vertical
  passes, edges replicated) whose box radius comes from the float32 formula of Gwosdek et al. (SSVM 2011).
- `canny`: OpenCV's `cv2.Canny(img, low, high)` with aperture 3 and the L1 norm, for 1 or 3 channels. Hysteresis is
  stated as a set: a pixel that survives non-maximum suppression with magnitude > low is an edge iff it is
  8-connected, through such pixels, to one with magnitude > high.
"""
from __future__ import annotations

import math

import numpy as np

PRECISION_BITS = 22  # 32 - 8 - 2: Pillow's 8-bit resampling precision


def _bilinear(x: float) -> float:
    x = -x if x < 0.0 else x
    return 1.0 - x if x < 1.0 else 0.0


def _bicubic(x: float) -> float:
    a = -0.5
    x = -x if x < 0.0 else x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


FILTERS = {"bilinear": (1.0, _bilinear), "bicubic": (2.0, _bicubic), "lanczos": (3.0, _lanczos)}


def resample_coeffs(in_size: int, out_size: int, name: str):
    """(xmin [out], k [out, taps] int64): the fixed-point taps of each output pixel (zero past its count)"""
    support0, fn = FILTERS[name]
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = support0 * fs
    ss = 1.0 / fs
    rows = []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [fn((x + xmin - center + 0.5) * ss) for x in range(n)]
        total = 0.0
        for v in w:
            total += v
        if total != 0.0:
            w = [v / total for v in w]
        rows.append((xmin, [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
                            for v in w]))
    taps = max(len(k) for _, k in rows)
    xmin = np.array([r[0] for r in rows], np.int64)
    k = np.zeros((out_size, taps), np.int64)
    for i, (_, kk) in enumerate(rows):
        k[i, :len(kk)] = kk
    return xmin, k


def _resample_axis(a: np.ndarray, axis: int, out_size: int, name: str) -> np.ndarray:
    a = np.moveaxis(a.astype(np.int64), axis, -1)
    in_size = a.shape[-1]
    xmin, k = resample_coeffs(in_size, out_size, name)
    acc = np.full(a.shape[:-1] + (out_size,), 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(k.shape[1]):
        idx = np.minimum(xmin + t, in_size - 1)  # k = 0 past a pixel's tap count
        acc += a[..., idx] * k[:, t]
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, -1, axis)


def resize(img: np.ndarray, size, name: str = "bicubic") -> np.ndarray:
    """Image.fromarray(img).resize(size=(w, h), resample=name) for uint8 [h, w] or [h, w, 3]"""
    w, h = size
    out = img.copy()
    if w != img.shape[1]:
        out = _resample_axis(out, 1, w, name)
    if h != img.shape[0]:
        out = _resample_axis(out, 0, h, name)
    return out


def box_radius(radius: float) -> np.float32:
    """the extended box radius Pillow's GaussianBlur runs three passes of (float32, as Pillow computes it)"""
    f = np.float32
    sigma2 = f(f(radius) * f(radius)) / f(3)
    L = f(math.sqrt(12.0 * float(sigma2) + 1.0))
    l = f(math.floor((float(L) - 1.0) / 2.0))
    a = (f(2) * l + f(1)) * (l * (l + f(1)) - f(3) * sigma2)
    a = a / (f(6) * (sigma2 - (l + f(1)) * (l + f(1))))
    return f(l + a)


def box_weights(fr: np.float32):
    """(integer radius, centre weight ww, end-tap weight fw) in 24-bit fixed point"""
    r = int(fr)
    ww = int(np.float32(1 << 24) / (fr * np.float32(2) + np.float32(1)))
    fw = ((1 << 24) - (2 * r + 1) * ww) // 2
    return r, ww, fw


def _box_pass(a: np.ndarray, axis: int, fr: np.float32) -> np.ndarray:
    r, ww, fw = box_weights(fr)
    a = np.moveaxis(a.astype(np.int64), axis, -1)
    n = a.shape[-1]
    x = np.arange(n)
    acc = np.zeros(a.shape, np.int64)
    for i in range(-r, r + 1):
        acc += a[..., np.clip(x + i, 0, n - 1)]
    far = a[..., np.clip(x - r - 1, 0, n - 1)] + a[..., np.clip(x + r + 1, 0, n - 1)]
    out = ((acc * ww + far * fw + (1 << 23)) >> 24).astype(np.uint8)
    return np.moveaxis(out, -1, axis)


def gaussian_blur(img: np.ndarray, radius: float) -> np.ndarray:
    """Image.fromarray(img).filter(ImageFilter.GaussianBlur(radius)) for uint8 [h, w] or [h, w, 3]"""
    out = img.copy()
    if radius == 0:
        return out
    fr = box_radius(radius)
    for axis in (1, 0):
        for _ in range(3):
            out = _box_pass(out, axis, fr)
    return out


TG22 = int(0.4142135623730950488016887242097 * (1 << 15) + 0.5)  # tan(22.5 deg) in 15 fractional bits


def sobel_l1(img: np.ndarray):
    """(dx, dy, |dx| + |dy|) of the 3x3 Sobel with replicated borders; for 3 channels each pixel takes the channel
    with the largest magnitude (the first on ties)"""
    a = img.astype(np.int64)
    if a.ndim == 2:
        a = a[..., None]
    p = np.pad(a, ((1, 1), (1, 1), (0, 0)), mode="edge")
    h, w = a.shape[:2]

    def s(dy, dx):
        return p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]

    dx = (s(-1, 1) + 2 * s(0, 1) + s(1, 1)) - (s(-1, -1) + 2 * s(0, -1) + s(1, -1))
    dy = (s(1, -1) + 2 * s(1, 0) + s(1, 1)) - (s(-1, -1) + 2 * s(-1, 0) + s(-1, 1))
    mag = np.abs(dx) + np.abs(dy)
    c = np.argmax(mag, axis=2)[..., None]
    take = lambda t: np.take_along_axis(t, c, axis=2)[..., 0]  # noqa: E731
    return take(dx), take(dy), take(mag)


def canny_thresholds(low: float, high: float):
    if low > high:
        low, high = high, low
    return math.floor(low), math.floor(high)


def canny_classes(img: np.ndarray, low: float, high: float) -> np.ndarray:
    """0: not a candidate, 1: survives suppression with magnitude > low, 2: and > high"""
    lo, hi = canny_thresholds(low, high)
    dx, dy, m = sobel_l1(img)
    h, w = m.shape
    mp = np.pad(m, 1)  # neighbours outside the image have magnitude 0

    def nb(oy, ox):
        return mp[1 + oy:1 + oy + h, 1 + ox:1 + ox + w]

    ax = np.abs(dx)
    ay = np.abs(dy) << 15
    tg22x = ax * TG22
    tg67x = tg22x + (ax << 16)
    s = np.where((dx ^ dy) < 0, -1, 1)
    horiz = (m > nb(0, -1)) & (m >= nb(0, 1))
    vert = (m > nb(-1, 0)) & (m >= nb(1, 0))
    diag_p = (m > nb(-1, -1)) & (m > nb(1, 1))  # s = +1: previous row j - 1, next row j + 1
    diag_n = (m > nb(-1, 1)) & (m > nb(1, -1))  # s = -1
    keep = np.where(ay < tg22x, horiz, np.where(ay > tg67x, vert, np.where(s > 0, diag_p, diag_n)))
    keep &= m > lo
    return np.where(keep, np.where(m > hi, 2, 1), 0).astype(np.uint8)


def canny(img: np.ndarray, low: float, high: float) -> np.ndarray:
    """cv2.Canny(img, low, high) (aperture 3, L1) for uint8 [h, w] or [h, w, 3]: uint8 [h, w] in {0, 255}"""
    from scipy import ndimage

    cls = canny_classes(img, low, high)
    lab, n = ndimage.label(cls > 0, structure=np.ones((3, 3), bool))
    strong = np.zeros(n + 1, bool)
    strong[lab[cls == 2]] = True
    strong[0] = False
    return np.where(strong[lab], 255, 0).astype(np.uint8)
