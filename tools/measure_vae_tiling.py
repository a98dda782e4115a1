"""Time and peak device memory of VAE encode / decode, untiled and tiled (AutoencoderKL.enable_tiling), at SD-1.5
widths with synthetic weights and the SD-1.5 tile size (sample_size 512).

    python tools/measure_vae_tiling.py [--reps 5] [--json OUT]

Rows: untiled and tiled decode / encode of a 1024 x 1024 image, tiled decode / encode at 1024 x 1360 and 2048 x 2728
(the app's 3:4 outpainting canvases expanded 2 x 2 and 4 x 4). Each row records its plan from an empty plan cache
(the recording and graph capture are not timed), runs once to warm up, then times `--reps` calls with CUDA events and
reports the median. Peak memory is torch's max_memory_allocated over the first call, from a reset. The card's name
and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch

    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing can be measured")
    dev = torch.device("cuda:0")
    vae = AutoencoderKL.synthetic(seed=4321, sample_size=512).to(dev)
    eng = vae.engine()
    g = torch.Generator(device=dev).manual_seed(0)
    vae.decode(torch.randn(1, 4, 16, 16, device=dev, generator=g))  # weights packed before any measurement
    rows = []
    for op, tiled, H, W in (("decode", False, 1024, 1024), ("decode", True, 1024, 1024),
                            ("encode", False, 1024, 1024), ("encode", True, 1024, 1024),
                            ("decode", True, 1360, 1024), ("encode", True, 1360, 1024),
                            ("decode", True, 2728, 2048), ("encode", True, 2728, 2048)):
        if op == "decode":
            arg = torch.randn(1, 4, H // 8, W // 8, device=dev, generator=g)
            fn = (lambda a=arg: vae.tiled_decode(a).sample) if tiled else (lambda a=arg: vae._decode(a, True, False).sample)
        else:
            arg = torch.rand(1, 3, H, W, device=dev, generator=g) * 2 - 1
            fn = ((lambda a=arg: vae.tiled_encode(a).latent_dist.mean) if tiled
                  else (lambda a=arg: vae._encode(a, True, False).latent_dist.mean))
        eng._plans.clear()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        times.sort()
        tiles = len(vae.tile_geometry(op == "encode", *((H, W) if op == "encode" else (H // 8, W // 8))).tiles)
        rows.append(dict(op=op, tiled=tiled, height=H, width=W, tiles=tiles if tiled else 1,
                         ms_median=times[len(times) // 2], ms_min=times[0], peak_gib=peak / 2 ** 30))
        del arg, fn
    name, limit = _card()
    print(f"device: {name}, power limit {limit}; synthetic SD-1.5 VAE weights, sample_size 512, batch 1")
    print(f"{'op':7} {'mode':8} {'canvas (H x W)':>15} {'tiles':>6} {'median ms':>10} {'min ms':>8} {'peak GiB':>9}")
    for r in rows:
        print(f"{r['op']:7} {'tiled' if r['tiled'] else 'untiled':8} {r['height']:>7} x {r['width']:<5} {r['tiles']:>6} "
              f"{r['ms_median']:>10.1f} {r['ms_min']:>8.1f} {r['peak_gib']:>9.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=name, power_limit=limit, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
