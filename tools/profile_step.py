#!/usr/bin/env python
"""Per-kernel profile of one denoising step program on the GPU (a run of its own, separate from bench.py).

    python tools/profile_step.py [--config C2 [--config C4]] [--steps 10] [--sweep-block-n] [--out DIR]

For each config it builds the bench's pipeline and inputs, runs the loop once to record the step program, times 50
CUDA-graph replays of it with events (the step time bench.py reports as `ms_per_ddim_step`), then replays it `--steps`
times as plain launches under torch.profiler and prints, per kernel variant: launches per step, device µs per step,
share of the step's kernel time, and for the GEMM / attention variants the algorithmic TFLOP/s of the launches the
program recorded for it (2·M·N·K per GEMM, 4·Nq·Nk·d per attention head; from the descriptors, not the tiles run).

--sweep-block-n times every distinct plain / GEGLU GEMM of the step once per legal tile width (CUDA events, the
statistics and split-K attachments removed so that every width runs the same work) against the width the library
picks, as evidence for the tile-width rule in gemm_conv.cu (`pick_block_n`).
--out DIR writes profile_<config>.json there. The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

GEMM_NAME = re.compile(r"gemm_conv_kernel<(\d+), (\d+), (true|false)>")
ATTN_NAME = re.compile(r"attn_fwd_kernel<(\d+), (true|false)>")


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), (x.strip() for x in out.split(","))))


def gemm_flops(c) -> float:
    from powerpaint_b200 import _native as N

    if c.a_mode == N.PP_A_MATRIX:
        m, taps = c.M, 1
    elif c.a_mode == N.PP_A_CONV3X3:
        m, taps = c.nb * c.h * c.w, 9
    elif c.a_mode == N.PP_A_CONV3X3_S2:
        m, taps = c.nb * ((c.h + 1) // 2) * ((c.w + 1) // 2), 9
    else:
        m, taps = c.nb * (c.h // 2) * (c.w // 2), 9
    return 2.0 * m * c.N * taps * (c.c0 + c.c1)


def variant_key(desc):
    from powerpaint_b200 import ops

    if desc.kind == "gemm":
        bn, mode, ks = ops.gemm_variant(desc)
        return f"gemm_conv_kernel<{bn}, {mode}, {'true' if ks == 2 else 'false'}>"
    dv, f16 = ops.attention_variant(desc)
    return f"attn_fwd_kernel<{dv}, {'true' if f16 else 'false'}>"


def kernel_key(name: str) -> str:
    m = GEMM_NAME.search(name) or ATTN_NAME.search(name)
    if m:
        return m.group(0)
    return re.sub(r"^void |\(.*$", "", name).replace("pp::", "").strip()


def record_step(cfg, dev):
    """the bench's loop, recorded once; returns (plan state, [descriptors of the step program])"""
    from powerpaint_b200 import ops

    added = defaultdict(list)
    orig_add = ops.Program.add

    def add(self, desc):
        added[id(self)].append(desc)
        return orig_add(self, desc)

    ops.Program.add = add
    try:
        pipe = bench.build_pipeline(cfg, dev)
        den = pipe.denoiser()
        pipe.scheduler.set_timesteps(bench.DDIM_STEPS)
        kw = bench.resident_inputs(cfg, dev, 0)
        den.run(timesteps=pipe.scheduler.timesteps, coef=pipe.scheduler.step_coefficients(),
                guidance_scale=bench.GUIDANCE, **kw)
    finally:
        ops.Program.add = orig_add
    torch.cuda.synchronize()
    st = next(reversed(den._cache.values()))
    return den, st, [d for d in added[id(st["program"])] if d.kind in ("gemm", "attn")]


def replay(den, st, n, graph):
    """n <= 50 replays of the step program from step 0 (the device step counter indexes the timestep table)"""
    prog = st["program"]
    with torch.cuda.stream(den._stream):
        st["step_idx"].zero_()
        for _ in range(n):
            prog.launch() if graph else prog.run()


def graph_step_ms(den, st):
    torch.cuda.synchronize()
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(bench.DDIM_STEPS + 1)]
    with torch.cuda.stream(den._stream):
        st["step_idx"].zero_()
        evs[0].record()
        for i in range(bench.DDIM_STEPS):
            st["program"].launch()
            evs[i + 1].record()
    torch.cuda.synchronize()
    ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(5, bench.DDIM_STEPS - 5))
    return sum(ms) / len(ms), ms[0], ms[-1]


def kernel_profile(den, st, steps):
    from torch.profiler import ProfilerActivity, profile

    replay(den, st, 3, graph=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        replay(den, st, steps, graph=False)
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0, 0.0])  # kernel key -> [launches, device µs], summed over the profiled steps
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            k = kernel_key(e.name)
            per[k][0] += 1
            per[k][1] += e.device_time_total
    return {k: (n / steps, us / steps) for k, (n, us) in per.items()}


def sweep_block_n(descs, reps=20):
    """device µs of each distinct plain / GEGLU GEMM of the step at every legal tile width (events over `reps`)"""
    from powerpaint_b200 import _native as N
    from powerpaint_b200 import ops

    seen, rows = {}, []
    for d in descs:
        c = d.c
        if d.kind != "gemm" or c.epilogue not in (N.PP_EPI_PLAIN, N.PP_EPI_GEGLU):
            continue
        shape = (c.a_mode, c.nb, c.h, c.w, c.M, c.N, c.c0, c.c1, c.epilogue)
        if shape in seen:
            rows[seen[shape]]["count"] += 1
            continue
        base = type(c).from_buffer_copy(c)
        for f in ("chan_stats", "row_stats", "row_final", "row_ticket", "splitk_ws", "splitk_flags"):
            setattr(base, f, 0)
        base.block_n = 0
        default = ops.gemm_variant(ops.Desc("gemm", base, d.keep))[0]
        times = {}
        for bn in (64, 128, 160, 256):
            if c.epilogue == N.PP_EPI_GEGLU and (bn not in (128, 256) or c.N % bn):
                continue
            t = type(base).from_buffer_copy(base)
            t.block_n = bn
            dd = ops.Desc("gemm", t, d.keep)
            for _ in range(3):
                ops.run(dd)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ops.run(dd)
            e1.record()
            torch.cuda.synchronize()
            times[bn] = 1e3 * e0.elapsed_time(e1) / reps
        seen[shape] = len(rows)
        rows.append(dict(shape=dict(a_mode=c.a_mode, nb=c.nb, h=c.h, w=c.w, M=c.M, N=c.N, c0=c.c0, c1=c.c1,
                                    geglu=c.epilogue == N.PP_EPI_GEGLU),
                         count=1, flops=gemm_flops(c), default=default, us=times))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", action="append", choices=sorted(bench.CONFIGS))
    ap.add_argument("--steps", type=int, default=10, help="profiled replays of the step program (at most 50)")
    ap.add_argument("--sweep-block-n", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("profile_step.py: no CUDA device", file=sys.stderr)
        return 2
    if not 1 <= args.steps <= bench.DDIM_STEPS:
        ap.error(f"--steps must be in [1, {bench.DDIM_STEPS}]")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    lib = os.environ.get("PP_B200_LIB") or "in-tree libpowerpaint_b200.so"
    print(f"card: {gpu}  library: {lib}")
    for name in args.config or ["C2"]:
        cfg = bench.CONFIGS[name]
        den, st, descs = record_step(cfg, dev)
        flops = defaultdict(float)
        recorded = defaultdict(int)
        for d in descs:
            k = variant_key(d)
            recorded[k] += 1
            flops[k] += gemm_flops(d.c) if d.kind == "gemm" else 4.0 * d.c.batch * d.c.heads * d.c.nq * d.c.nk * d.c.d
        replay(den, st, 3, graph=True)
        step_ms, lo, hi = graph_step_ms(den, st)
        kp = kernel_profile(den, st, args.steps)
        total_us = sum(us for _, us in kp.values())
        step_flops = cfg["flops_per_image_step"] * cfg["batch"]
        print(f"\n[{name}] step program: {step_ms:.3f} ms per step (graph replay, events; min {lo:.3f} max {hi:.3f}), "
              f"{step_flops / step_ms / 1e9:.0f} TFLOP/s algorithmic; kernel time under the profiler "
              f"{total_us / 1e3:.3f} ms per step over {args.steps} steps")
        print(f"{'kernel variant':44s} {'launches':>8s} {'recorded':>8s} {'µs/step':>10s} {'share':>7s} {'TFLOP/s':>8s}")
        rows = []
        for k, (n, us) in sorted(kp.items(), key=lambda kv: -kv[1][1]):
            tf = flops[k] / (us * 1e6) if k in flops and us > 0 else None
            rows.append(dict(kernel=k, launches_per_step=n, recorded=recorded.get(k, 0), us_per_step=us,
                             share=us / total_us, tflops=tf, flops_per_step=flops.get(k, 0.0)))
            print(f"{k:44s} {n:8.1f} {recorded.get(k, 0) or '':>8} {us:10.1f} {100 * us / total_us:6.1f}% "
                  f"{'' if tf is None else f'{tf:8.0f}'}")
        res = dict(config=name, card=gpu, library=lib, step_ms=step_ms, step_ms_min=lo, step_ms_max=hi,
                   kernel_us_per_step=total_us, profiled_steps=args.steps, kernels=rows)
        if args.sweep_block_n:
            sw = sweep_block_n(descs)
            res["block_n_sweep"] = sw
            print(f"\n[{name}] tile-width sweep (µs per launch; * = the library's pick; launches per step)")
            gain = 0.0
            for r in sw:
                s = r["shape"]
                best = min(r["us"], key=r["us"].get)
                gain += r["count"] * (r["us"][r["default"]] - r["us"][best])
                cells = " ".join(f"{bn}{'*' if bn == r['default'] else ' '}={us:8.1f}" for bn, us in r["us"].items())
                kind = "conv" if s["a_mode"] else "gemm"
                m = s["M"] if not s["a_mode"] else f"{s['nb']}x{s['h']}x{s['w']}"
                print(f"  {kind} M={m} N={s['N']} K={s['c0'] + s['c1']}{' geglu' if s['geglu'] else ''} x{r['count']}: "
                      f"{cells}  best={best}")
            print(f"[{name}] all best widths together would save {gain:.0f} µs per step ({100 * gain / 1e3 / step_ms:.1f} %)")
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, f"profile_{name}.json"), "w") as f:
                json.dump(res, f, indent=1)
        del den, st, descs
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
