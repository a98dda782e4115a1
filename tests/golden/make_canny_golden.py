"""Writes tests/golden/canny_cases.npz: inputs and `cv2.Canny(img, low, high)` outputs (aperture 3, L1 norm) for the
device Canny (tests/test_imageops_gpu.py) and its NumPy model (tests/test_app_flow_cpu.py), on machines without cv2.

Cases: random, smooth and structured images, 1 and 3 channels, sizes from 1 x 1 to 848 x 640, and equal, swapped,
zero and fractional thresholds. Deterministic: `python tests/golden/make_canny_golden.py` rewrites the same bytes."""
import os

import cv2
import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "canny_cases.npz")


def _smooth(rng, h, w, c):
    a = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    return cv2.GaussianBlur(a, (7, 7), 2.0).reshape(h, w, c) if min(h, w) > 3 else a


def _structured(rng, h, w, c):
    y, x = np.mgrid[0:h, 0:w]
    a = np.zeros((h, w, c), np.uint8)
    for ch in range(c):
        cx, cy, r = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(4, max(5, min(h, w) / 2))
        disc = ((x - cx) ** 2 + (y - cy) ** 2 < r * r) * 200
        stripes = ((x + 2 * y + 7 * ch) // 9 % 2) * 40
        a[..., ch] = np.clip(disc + stripes + 10, 0, 255)
    return a


def _random(rng, h, w, c):
    return rng.integers(0, 256, (h, w, c), dtype=np.uint8)


CASES = [  # (kind, h, w, channels, low, high)
    ("random", 1, 1, 1, 100, 200), ("random", 1, 1, 3, 0, 0), ("random", 1, 9, 1, 50, 100),
    ("random", 7, 1, 3, 50, 100), ("random", 2, 2, 3, 10, 10), ("random", 16, 33, 1, 100, 200),
    ("random", 31, 65, 3, 300, 600), ("random", 64, 64, 3, 200, 100), ("smooth", 17, 40, 1, 5, 15),
    ("smooth", 64, 96, 3, 20, 40), ("smooth", 100, 130, 1, 0, 0), ("smooth", 120, 160, 3, 12.7, 30.2),
    ("structured", 48, 80, 1, 100, 200), ("structured", 97, 33, 3, 100, 200), ("structured", 128, 128, 3, 50, 50),
    ("structured", 200, 300, 3, 200, 100), ("structured", 480, 640, 3, 100, 200), ("smooth", 240, 320, 3, 20, 40),
    ("structured", 640, 848, 3, 100, 200), ("structured", 640, 848, 1, 60, 120),
]


def main():
    rng = np.random.default_rng(20261018)
    data = {}
    for i, (kind, h, w, c, lo, hi) in enumerate(CASES):
        img = {"random": _random, "smooth": _smooth, "structured": _structured}[kind](rng, h, w, c)
        img = img[..., 0] if c == 1 else img
        data[f"in_{i}"] = img
        data[f"out_{i}"] = cv2.Canny(img, lo, hi)
        data[f"thr_{i}"] = np.array([lo, hi], np.float64)
    data["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **data)
    print(f"wrote {len(CASES)} cases to {OUT}")


if __name__ == "__main__":
    main()
