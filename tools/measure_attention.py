#!/usr/bin/env python
"""Times every attention shape of the C2 and C4 denoising step, and compares builds of the library.

    python tools/measure_attention.py [--lib PATH ...] [--rounds 3] [--config C2 --config C4] [--out DIR]

The shapes are those the step programs record (as tools/profile_step.py records them): self-attention at d = 40 over
4 096 / 16 384 tokens, d = 80 over 1 024, d = 160 over 256, and the 77-key cross-attention. Each shape runs on seeded
inputs at the recorded pitches. Its time is CUDA events over windows of at least 200 ms (median of three windows).
Reported per shape: µs per launch, algorithmic TFLOP/s (4·B·H·Nq·Nk·d) and the exponential floor: every 128 x 128
score block takes 16 384 MUFU.EX2, at 16 per SM per clock 1 024 SM clocks, over the SMs at the SM clock sampled
right after the timing.

Each --lib (default: the in-tree library) is timed in subprocesses of their own with PP_B200_LIB set, since the
library is loaded once per process; the libraries alternate, --rounds times. The first round also keeps the outputs:
every library after the first is compared with the first one (bit-identical or rel-L2 / max |diff|). The card's name,
power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

FIELDS = ("batch", "heads", "d", "nq", "nk", "q_ld", "k_ld", "vt_ld", "o_ld", "q_batch_stride", "k_batch_stride",
          "vt_fp16")
EX2_PER_SM_CLK = 16
WINDOW_S = 0.2


def smi(q):
    import torch

    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), (x.strip() for x in out.split(","))))


def record_shapes(configs):
    """distinct attention shapes of each config's step program, with launches per step"""
    import torch

    import bench
    import profile_step

    dev = torch.device("cuda", 0)
    shapes = {}
    for name in configs:
        den, st, descs = profile_step.record_step(bench.CONFIGS[name], dev)
        for d in descs:
            if d.kind != "attn":
                continue
            f = {k: int(getattr(d.c, k)) for k in FIELDS}
            f["scale"] = float(d.c.scale)
            key = json.dumps(f, sort_keys=True)
            per = shapes.setdefault(key, dict(f, configs={}))["configs"]
            per[name] = per.get(name, 0) + 1
        del den, st, descs
        torch.cuda.empty_cache()
    return sorted(shapes.values(), key=lambda s: -s["batch"] * s["heads"] * s["nq"] * s["nk"] * s["d"])


def build(f, seed):
    import torch

    from powerpaint_b200 import _native as nat
    from powerpaint_b200 import ops as o

    g = torch.Generator(device="cuda").manual_seed(seed)
    B, H, dh, nq, nk = f["batch"], f["heads"], f["d"], f["nq"], f["nk"]
    C = H * dh
    q = torch.randn((B - 1) * f["q_batch_stride"] + nq * f["q_ld"], device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn((B - 1) * f["k_batch_stride"] + nk * f["k_ld"], device="cuda", generator=g).to(torch.bfloat16)
    vt = torch.randn(B * C * f["vt_ld"], device="cuda", generator=g).to(torch.float16 if f["vt_fp16"] else torch.bfloat16)
    out = torch.zeros(B * nq * f["o_ld"], device="cuda", dtype=torch.bfloat16)
    d = nat.AttnDesc()
    for key in FIELDS:
        setattr(d, key, f[key])
    d.scale = f["scale"]
    d.q, d.k, d.vt, d.out = q.data_ptr(), k.data_ptr(), vt.data_ptr(), out.data_ptr()
    return o.Desc("attn", d, [q, k, vt, out]), out.view(B * nq, f["o_ld"])[:, :C]


def child(shapes_path, save_dir):
    import torch

    from powerpaint_b200 import ops as o

    torch.cuda.set_device(0)
    shapes = json.load(open(shapes_path))
    res = []
    for i, f in enumerate(shapes):
        desc, out = build(f, seed=1234 + i)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def window(n):
            e0.record()
            for _ in range(n):
                o.run(desc)
            e1.record()
            torch.cuda.synchronize()
            return 1e3 * e0.elapsed_time(e1) / n  # µs per launch

        window(3)  # warm-up
        n = max(10, int(math.ceil(1.2 * WINDOW_S * 1e6 / window(10))))
        wins = [window(n) for _ in range(3)]
        clk = smi("clocks.sm")["clocks.sm"]
        res.append(dict(us=statistics.median(wins), launches_per_window=n, sm_mhz=float(clk)))
        if save_dir:
            torch.save(out.clone().cpu(), os.path.join(save_dir, f"out{i}.pt"))
        del desc, out
    print("RESULT " + json.dumps(res))


def compare(dir_a, dir_b, n):
    import torch

    rows = []
    for i in range(n):
        a = torch.load(os.path.join(dir_a, f"out{i}.pt")).double()
        b = torch.load(os.path.join(dir_b, f"out{i}.pt")).double()
        same = torch.equal(torch.load(os.path.join(dir_a, f"out{i}.pt")).view(torch.int16),
                           torch.load(os.path.join(dir_b, f"out{i}.pt")).view(torch.int16))
        rel = ((a - b).norm() / a.norm()).item()
        rows.append(dict(bit_identical=same, rel_l2=rel, max_abs=(a - b).abs().max().item()))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="library build to time (repeatable; default: the in-tree one)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--config", action="append", choices=("C2", "C4"))
    ap.add_argument("--out", help="write measure_attention.json there")
    ap.add_argument("--child", help=argparse.SUPPRESS)
    ap.add_argument("--save", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child, args.save)

    import torch

    if not torch.cuda.is_available():
        print("measure_attention.py: no CUDA device", file=sys.stderr)
        return 2
    card = smi("name,power.limit,clocks.max.sm")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    libs = args.lib or [""]
    shapes = record_shapes(args.config or ["C2", "C4"])
    torch.cuda.empty_cache()
    print(f"card: {card['name']}, power limit {card['power.limit']} W, max SM clock {card['clocks.max.sm']} MHz, "
          f"{sms} SMs; {len(shapes)} attention shapes")
    tmp = tempfile.mkdtemp(prefix="pp_measure_attention_")
    shapes_path = os.path.join(tmp, "shapes.json")
    json.dump(shapes, open(shapes_path, "w"))
    runs = {i: [] for i in range(len(libs))}
    for r in range(args.rounds):
        for i, lib in enumerate(libs):
            env = dict(os.environ)
            env.pop("PP_B200_LIB", None)
            if lib:
                env["PP_B200_LIB"] = os.path.abspath(lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--child", shapes_path]
            if r == 0:
                os.makedirs(os.path.join(tmp, f"lib{i}"), exist_ok=True)
                cmd += ["--save", os.path.join(tmp, f"lib{i}")]
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
            if p.returncode != 0 or not line:
                print(p.stdout[-3000:], p.stderr[-3000:], file=sys.stderr)
                return 1
            runs[i].append(json.loads(line[0][7:]))
    report = dict(card=card, sms=sms, libs=[lib or "in-tree" for lib in libs], shapes=[])
    for k, f in enumerate(shapes):
        blocks = f["batch"] * f["heads"] * math.ceil(f["nq"] / 128) * math.ceil(f["nk"] / 128)
        flops = 4.0 * f["batch"] * f["heads"] * f["nq"] * f["nk"] * f["d"]
        entry = dict(shape={x: f[x] for x in ("batch", "heads", "d", "nq", "nk", "vt_fp16")},
                     launches_per_step=f["configs"], per_lib=[])
        for i in range(len(libs)):
            us = [run[k]["us"] for run in runs[i]]
            mhz = statistics.median(run[k]["sm_mhz"] for run in runs[i])
            med = statistics.median(us)
            floor_us = blocks * (128 * 128 / EX2_PER_SM_CLK) / sms / mhz  # SM clocks / MHz = µs
            entry["per_lib"].append(dict(us_median=med, us_min=min(us), us_max=max(us), tflops=flops / med / 1e6,
                                         sm_mhz_median=mhz, mufu_floor_us=floor_us, floor_share=floor_us / med))
        report["shapes"].append(entry)
    if len(libs) > 1:
        for i in range(1, len(libs)):
            for k, row in enumerate(compare(os.path.join(tmp, "lib0"), os.path.join(tmp, f"lib{i}"), len(shapes))):
                report["shapes"][k]["per_lib"][i]["vs_first"] = row
    print(f"{'shape (B x H, d, Nq x Nk, P)':38s} {'per step':>14s} " + " ".join(
        f"{'lib' + str(i) + ' µs [min, max]':>26s} {'TFLOP/s':>7s} {'MHz':>5s} {'floor%':>6s}" for i in range(len(libs))))
    for e in report["shapes"]:
        s = e["shape"]
        name = f"{s['batch']}x{s['heads']}, d={s['d']}, {s['nq']}x{s['nk']}, {'f16' if s['vt_fp16'] else 'bf16'}"
        cells = []
        for pl in e["per_lib"]:
            cells.append(f"{pl['us_median']:9.1f} [{pl['us_min']:7.1f}, {pl['us_max']:7.1f}] {pl['tflops']:7.0f} "
                         f"{pl['sm_mhz_median']:5.0f} {100 * pl['floor_share']:5.1f}%")
        per = ",".join(f"{c}:{n}" for c, n in e["launches_per_step"].items())
        print(f"{name:38s} {per:>14s} " + " ".join(cells))
        for i, pl in enumerate(e["per_lib"][1:], 1):
            v = pl["vs_first"]
            print(f"{'':38s} lib{i} vs lib0: {pl['us_median'] / e['per_lib'][0]['us_median'] - 1:+.1%} time, "
                  + ("bit-identical" if v["bit_identical"] else f"rel-L2 {v['rel_l2']:.2e}, max |diff| {v['max_abs']:.2e}"))
    for i, lib in enumerate(report["libs"]):
        print(f"lib{i}: {lib}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "measure_attention.json"), "w") as fh:
            json.dump(report, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
