"""Time the app's host pre / post-processing (oracle/app_flow.py's PIL / NumPy / cv2 steps) against the controller's
device steps (powerpaint_b200/imageops.py), per stage, at three upload sizes; the denoising loop is not part of it.

Stages (ref:app.py:258-387,405-473; canvas = the 640-short-side size rounded down to multiples of 8):
  pre     upload resize to 640 short side, resize to the canvas, mask resize
  hole    the v2 hole fill
  post    red overlay, Gaussian blur (radius 4) and paste-back, with the downloads of the returned images
  canny   control-image resize and Canny (100, 200)
Host numbers are wall time; device numbers are wall time (from the PIL upload to the PIL downloads, synchronised) and
CUDA-event time of the same span. Prints the host CPU model and thread count and the GPU name and power limit.

    python tools/measure_app_flow.py [--reps 20]
"""
from __future__ import annotations

import argparse
import os
import platform
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
from PIL import Image, ImageFilter

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from powerpaint_b200 import imageops as io  # noqa: E402
from powerpaint_b200.controller import short_side_size  # noqa: E402

UPLOADS = [(4032, 3024), (1920, 1080), (640, 480)]


def _cpu_model() -> str:
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    try:
        for line in subprocess.run(["lscpu"], capture_output=True, text=True, timeout=30).stdout.splitlines():
            if line.startswith("Model name"):
                return line.split(":", 1)[1].strip()
    except (OSError, subprocess.TimeoutExpired):
        pass
    return platform.processor() or "unknown"


def _gpu() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return q or torch.cuda.get_device_name()


def _inputs(w, h):
    rng = np.random.default_rng(0)
    y, x = np.mgrid[0:h, 0:w]
    img = np.stack([x * 255 // w, y * 255 // h, (x + y) % 256], -1).astype(np.int32) + rng.integers(0, 30, (h, w, 3))
    m = np.zeros((h, w, 3), np.uint8)
    m[h // 4:h // 2, w // 3:2 * w // 3] = 255
    return Image.fromarray(np.clip(img, 0, 255).astype(np.uint8)), Image.fromarray(m)


def host_stages(img, mask):
    t = {}
    s = time.perf_counter()
    a = img.convert("RGB").resize(short_side_size(img.size, 640))
    H, W = a.size[0] - a.size[0] % 8, a.size[1] - a.size[1] % 8
    a, m = a.resize((H, W)), mask.resize((H, W))
    t["pre"] = time.perf_counter() - s
    s = time.perf_counter()
    Image.fromarray((np.array(a) * (1 - np.array(m) / 255.0)).astype(np.uint8))
    t["hole"] = time.perf_counter() - s
    res = a  # stands in for the pipeline's result
    s = time.perf_counter()
    mn = np.array(m.convert("RGB")).astype("float")
    red = np.array(res).astype("float")
    red[:, :, 0], red[:, :, 1], red[:, :, 2] = 180.0, 0, 0
    Image.fromarray((np.array(res).astype("float") * (1 - mn / 512.0) + mn / 512.0 * red).astype("uint8"))
    mb = np.asarray(m.convert("RGB").filter(ImageFilter.GaussianBlur(radius=4))) / 255.0
    Image.fromarray(np.uint8((np.asarray(res) / 255.0 * mb + (1 - mb) * (np.asarray(a) / 255.0)) * 255))
    t["post"] = time.perf_counter() - s
    try:
        import cv2

        s = time.perf_counter()
        cv2.Canny(np.array(img.resize((H, W))), 100, 200)
        t["canny"] = time.perf_counter() - s
    except ImportError:
        t["canny"] = float("nan")
    return t, (H, W)


def device_stages(img, mask, HW):
    H, W = HW
    t, ev = {}, {}

    def span(name, fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s = time.perf_counter()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        t[name] = time.perf_counter() - s
        ev[name] = e0.elapsed_time(e1) / 1e3
        return out

    def pre():
        a = io.resize(io.to_device(img), short_side_size(img.size, 640))
        return io.resize(a, (H, W)), io.resize(io.to_device(mask), (H, W))

    a, m = span("pre", pre)
    span("hole", lambda: io.hole_fill(a, m))
    span("post", lambda: (io.to_pil(io.red_overlay(a, m)), io.to_pil(io.paste_back(a, io.gaussian_blur(m, 4), a))))
    span("canny", lambda: io.to_pil(io.canny(io.resize(io.to_device(img), (H, W)), 100, 200)))
    return t, ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measure_app_flow needs a GPU (the device side has no CPU path)")
    print(f"host CPU: {_cpu_model()}, {os.cpu_count()} threads, torch threads {torch.get_num_threads()}")
    print(f"GPU: {_gpu()}")
    print("upload | canvas | stage | host ms | device wall ms | device event ms")
    for w, h in UPLOADS:
        img, mask = _inputs(w, h)
        host, dev, evs = {}, {}, {}
        for r in range(args.reps + 2):  # two warm-up rounds (tables, allocator, module load)
            ht, HW = host_stages(img, mask)
            dt, de = device_stages(img, mask, HW)
            if r >= 2:
                for k in ht:
                    host.setdefault(k, []).append(ht[k])
                    dev.setdefault(k, []).append(dt[k])
                    evs.setdefault(k, []).append(de[k])
        for k in host:
            print(f"{w}x{h} | {HW[0]}x{HW[1]} | {k} | {statistics.median(host[k]) * 1e3:.2f} | "
                  f"{statistics.median(dev[k]) * 1e3:.2f} | {statistics.median(evs[k]) * 1e3:.2f}")


if __name__ == "__main__":
    main()
