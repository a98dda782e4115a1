#!/usr/bin/env python
"""Times every GEMM / conv launch of the C2 and C4 denoising step, and compares builds of the library.

    python tools/measure_gemm.py [--lib PATH ...] [--rounds 3] [--config C2 --config C4] [--trace] [--out DIR]

The launches are those the step programs record (tools/profile_step.py's `record_step`); launches with the same
descriptor shape are timed once and counted per step. Each runs on its recorded buffers and pitches, with every input
it reads (A sources, residuals, row vector, bias, LayerNorm pair and weight sums) refilled from a seed first. Its
time is CUDA events over one window of at least 200 ms per round; the libraries alternate, each round in a child
process of its own with PP_B200_LIB set (the library is loaded once per process), and the report gives the median
(min-max) over the rounds, with algorithmic TFLOP/s (`profile_step.gemm_flops`: 2·M·N·K). The card's name, power
limit and the SM clock sampled after each window are read in the same run.

Before its timing each launch runs once on the seeded inputs, and its outputs (the output tensor and, where attached,
the GroupNorm partial sums and the LayerNorm records and pairs) are hashed and sampled; every library after the first
is compared with the first one (bit-identical, or rel-L2 of the sample).

--trace reads the per-tile clocks a library built with PP_EXTRA_NVCC_FLAGS=-DGEMM_TRACE records for CTA 0 of the
seeded run (`pp_debug_gemm_trace`): median SM clocks per tile of the main loop (slot 14 -> 5) and of the epilogue
(slot 5 -> 10), for the epilogue flavours that record those slots (modes 0 / 3 / 4 / 5). The epilogue is split into
its fragment arithmetic and stmatrix, residual and row-vector waits included ("math", 5 -> 6), the staging barrier
("stage", 6 -> 7; in mode 3 also the ticket verdict) and the TMA store issue, GroupNorm statistics pass and mode-3
fold ("tail", 7 -> 10). Each is a median over the tiles on its own, so the parts need not add up to the epilogue.
"""
from __future__ import annotations

import argparse
import ctypes
import hashlib
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

WINDOW_S = 0.2
SAMPLE = 1 << 20  # elements kept per output for the rel-L2 of a non-identical launch
# descriptor fields that make up a launch's shape (pointers excluded; attachments as presence flags)
SHAPE = ("a_mode", "epilogue", "c0", "c1", "lda0", "lda1", "nb", "h", "w", "M", "N", "ldb", "rows_per_group",
         "rowvec_ld", "ldr1", "ldr2", "act", "ldc", "out_fp32", "t_rows", "t_ld", "t_fp16", "trans_from_col")
PRESENT = ("bias", "rowvec", "res1", "res2", "alpha_dev", "chan_stats", "ln_stats", "row_stats", "splitk_ws", "a1",
           "out_t")


def smi(q):
    import torch

    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), (x.strip() for x in out.split(","))))


def shape_key(c, variant):
    f = {k: int(getattr(c, k)) for k in SHAPE}
    f.update({k: bool(getattr(c, k)) for k in PRESENT})
    f["alpha"] = float(c.alpha)
    f["variant"] = variant
    return json.dumps(f, sort_keys=True)


def distinct_launches(configs, dev):
    """[(config, key, desc, launches per step, program state)] of the distinct GEMM launches, in program order"""
    import bench
    import profile_step

    out, states = [], []
    for name in configs:
        den, st, descs = profile_step.record_step(bench.CONFIGS[name], dev)
        states.append((den, st))
        seen = {}
        for d in descs:
            if d.kind != "gemm":
                continue
            key = shape_key(d.c, profile_step.variant_key(d))
            if key in seen:
                seen[key][3] += 1
            else:
                seen[key] = [name, key, d, 1, st]
        out += list(seen.values())
    return out, states


def seed_inputs(desc, seed):
    """refill every buffer the launch reads (everything but the weights) from `seed`"""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    a0, a1, _w, _out, bias, rowvec, res1, res2 = desc.keep[:8]
    ins = [a0, a1, bias, rowvec, res1, res2]
    if desc.c.ln_stats:
        st, u = desc.keep[12:14]
        st.copy_(torch.stack([torch.rand(st.shape[0], device="cuda", generator=g) + 0.5,
                              torch.randn(st.shape[0], device="cuda", generator=g)], dim=1))
        ins.append(u)
    for t in ins:
        if t is not None and t.is_floating_point():
            t.copy_(torch.randn(t.shape, device="cuda", generator=g).to(t.dtype))


def outputs(desc):
    import torch

    from powerpaint_b200 import _native as N

    keep = [t for t in desc.keep if isinstance(t, torch.Tensor)]
    by_ptr = {N.ptr(t): t for t in keep}
    outs = {"out": by_ptr.get(desc.c.out)}
    for k in ("out_t", "chan_stats", "row_stats", "row_final"):
        if getattr(desc.c, k):
            outs[k] = by_ptr.get(getattr(desc.c, k))
    return {k: t for k, t in outs.items() if t is not None}


def digest(t):
    import torch

    flat = t.detach().contiguous().view(-1)
    raw = flat.view(torch.uint8) if flat.element_size() == 1 else flat.view({2: torch.int16, 4: torch.int32}[flat.element_size()])
    h = hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest()
    step = max(1, flat.numel() // SAMPLE)
    return h, flat[::step].float().cpu()


def read_trace():
    from powerpaint_b200 import _native as N

    try:
        fn = N.lib().pp_debug_gemm_trace
    except AttributeError:
        return None
    buf = (ctypes.c_longlong * (64 * 32))()
    if fn(buf, 64 * 32) != 0:
        return None
    t = [[buf[i * 32 + s] for s in range(32)] for i in range(64)]
    # The buffer keeps entries of earlier launches, and clock64 is per SM (CTA 0 of another launch may have run on
    # another SM), so the tiles of this launch are the chain from tile 0 in which each tile starts right after the
    # previous one ended.
    main, epi, math, stage, tail = [], [], [], [], []
    for i, row in enumerate(t):
        if i and not 0 <= row[15] - t[i - 1][10] < 100_000:
            break
        if not t[i][15] <= row[14] < row[5] <= row[6] <= row[7] <= row[10]:
            break
        main.append(row[5] - row[14])
        epi.append(row[10] - row[5])
        math.append(row[6] - row[5])
        stage.append(row[7] - row[6])
        tail.append(row[10] - row[7])
    if not main:
        return None
    med = statistics.median
    return dict(tiles=len(main), main_clk=med(main), epi_clk=med(epi), math_clk=med(math), stage_clk=med(stage),
                tail_clk=med(tail))


def child(configs, save_dir, trace):
    import torch

    from powerpaint_b200 import ops as o

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    launches, _states = distinct_launches(configs, dev)
    res = []
    for i, (name, key, desc, per_step, st) in enumerate(launches):
        st["step_idx"].zero_()  # the device step counter indexes the side-net scale table
        seed_inputs(desc, 1234 + i)
        o.run(desc)
        torch.cuda.synchronize()
        tr = read_trace() if trace else None
        if save_dir:
            torch.save({k: digest(t) for k, t in outputs(desc).items()}, os.path.join(save_dir, f"out{i}.pt"))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def window(n):
            e0.record()
            for _ in range(n):
                o.run(desc)
            e1.record()
            torch.cuda.synchronize()
            return 1e3 * e0.elapsed_time(e1) / n  # µs per launch

        us = 0.0
        if not trace:
            window(3)
            n = max(10, int(math.ceil(1.2 * WINDOW_S * 1e6 / window(10))))
            us = window(n)
        res.append(dict(config=name, key=key, per_step=per_step, us=us, trace=tr,
                        sm_mhz=float(smi("clocks.sm")["clocks.sm"]) if not trace else 0.0))
    print("RESULT " + json.dumps(res))


def compare(dir_a, dir_b, n):
    import torch

    rows = []
    for i in range(n):
        a = torch.load(os.path.join(dir_a, f"out{i}.pt"))
        b = torch.load(os.path.join(dir_b, f"out{i}.pt"))
        row = {}
        for k in a:
            same = a[k][0] == b[k][0]
            x, y = a[k][1].double(), b[k][1].double()
            row[k] = dict(bit_identical=same, rel_l2=0.0 if same else ((x - y).norm() / x.norm().clamp_min(1e-30)).item())
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="library build to time (repeatable; default: the in-tree one)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--config", action="append", choices=("C2", "C4"))
    ap.add_argument("--trace", action="store_true", help="per-tile clocks of -DGEMM_TRACE builds instead of times")
    ap.add_argument("--out", help="write measure_gemm.json there")
    ap.add_argument("--child", help=argparse.SUPPRESS)
    ap.add_argument("--save", help=argparse.SUPPRESS)
    args = ap.parse_args()
    configs = args.config or ["C2", "C4"]
    if args.child:
        return child(configs, args.save, args.trace)

    import torch

    if not torch.cuda.is_available():
        print("measure_gemm.py: no CUDA device", file=sys.stderr)
        return 2
    card = smi("name,power.limit,clocks.max.sm")
    print(f"card: {card['name']}, power limit {card['power.limit']} W, max SM clock {card['clocks.max.sm']} MHz")
    libs = args.lib or [""]
    tmp = tempfile.mkdtemp(prefix="pp_measure_gemm_")
    runs = {i: [] for i in range(len(libs))}
    for r in range(1 if args.trace else args.rounds):
        for i, lib in enumerate(libs):
            env = dict(os.environ)
            env.pop("PP_B200_LIB", None)
            if lib:
                env["PP_B200_LIB"] = os.path.abspath(lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "x"] + sum((["--config", c] for c in configs), [])
            if args.trace:
                cmd.append("--trace")
            if r == 0:
                os.makedirs(os.path.join(tmp, f"lib{i}"), exist_ok=True)
                cmd += ["--save", os.path.join(tmp, f"lib{i}")]
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
            if p.returncode != 0 or not line:
                print(p.stdout[-3000:], p.stderr[-3000:], file=sys.stderr)
                return 1
            runs[i].append(json.loads(line[0][7:]))
            print(f"round {r + 1}, lib{i}: {len(runs[i][-1])} launches", file=sys.stderr, flush=True)
    import profile_step  # noqa: F401  (gemm_flops needs the descriptor; recompute from the key)
    from powerpaint_b200 import _native as N

    n = len(runs[0][0])
    cmp = [compare(os.path.join(tmp, "lib0"), os.path.join(tmp, f"lib{i}"), n) for i in range(1, len(libs))]
    report = dict(card=card, libs=[lib or "in-tree" for lib in libs], launches=[])
    for k in range(n):
        first = runs[0][0][k]
        f = json.loads(first["key"])
        c = N.GemmDesc()
        for x in ("a_mode", "M", "N", "nb", "h", "w", "c0", "c1"):
            setattr(c, x, f[x])
        flops = profile_step.gemm_flops(c)
        entry = dict(config=first["config"], variant=f["variant"], per_step=first["per_step"], flops=flops,
                     shape={x: f[x] for x in ("a_mode", "M", "N", "nb", "h", "w", "c0", "c1", "epilogue")}, per_lib=[])
        for i in range(len(libs)):
            rs = [run[k] for run in runs[i]]
            us = [x["us"] for x in rs]
            pl = dict(trace=rs[0]["trace"])
            if not args.trace:
                med = statistics.median(us)
                pl.update(us_median=med, us_min=min(us), us_max=max(us), tflops=flops / med / 1e6,
                          sm_mhz_median=statistics.median(x["sm_mhz"] for x in rs))
            if i:
                pl["vs_first"] = cmp[i - 1][k]
            entry["per_lib"].append(pl)
        report["launches"].append(entry)
    for e in report["launches"]:
        s = e["shape"]
        geo = f"M={s['M']}" if s["a_mode"] == 0 else f"{s['nb']}x{s['h']}x{s['w']} conv{s['a_mode']}"
        name = f"{e['config']} {e['variant'].replace('gemm_conv_kernel', '')} {geo} N={s['N']} K={s['c0'] + s['c1']}"
        cells = []
        for pl in e["per_lib"]:
            if args.trace:
                t = pl["trace"]
                cells.append(f"main {t['main_clk']:8.0f} epi {t['epi_clk']:6.0f} = math {t['math_clk']:6.0f} + stage "
                             f"{t['stage_clk']:6.0f} + tail {t['tail_clk']:6.0f} clk ({t['tiles']} tiles)"
                             if t else "no trace")
            else:
                cells.append(f"{pl['us_median']:8.1f} [{pl['us_min']:7.1f}, {pl['us_max']:7.1f}] µs {pl['tflops']:5.0f} TF "
                             f"{pl['sm_mhz_median']:5.0f} MHz")
            if "vs_first" in pl:
                diff = {k: v for k, v in pl["vs_first"].items() if not v["bit_identical"]}
                cells.append("bit-identical" if not diff else
                             "differs: " + ", ".join(f"{k} rel-L2 {v['rel_l2']:.2e}" for k, v in diff.items()))
        print(f"{name:62s} x{e['per_step']:<3d} " + " | ".join(cells))
    if not args.trace:
        for i in range(len(libs)):
            for cfg in configs:
                tot = sum(e["per_lib"][i]["us_median"] * e["per_step"] for e in report["launches"] if e["config"] == cfg)
                print(f"lib{i} {cfg}: {tot / 1e3:.2f} ms of GEMM per step (sum of launch medians)")
    for i, lib in enumerate(report["libs"]):
        print(f"lib{i}: {lib}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "measure_gemm_trace.json" if args.trace else "measure_gemm.json"), "w") as fh:
            json.dump(report, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
