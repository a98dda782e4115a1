"""What drawing the stochastic samplers' noise on the device buys: ms per step of the fused loop with host-drawn noise
(`noise_fn`, the step program run op by op) against device-drawn noise (`randn_draws`, one CUDA graph replay per
step), and a `RequestBatcher` serving stochastic requests against serial calls.

    python tools/measure_stochastic.py [--steps 50] [--windows 5] [--requests 16] [--json OUT]

Loop arms: PowerPaint v1 on synthetic SD-1.5 weights at the C2 shape (512 x 512, CFG), Euler ancestral and DDIM with
eta = 1, batch 8 and batch 1. Each (sampler, batch) runs in a process of its own, so no plan, allocator or clock state
carries from one case to the next; inside it the host and device arms alternate over `--windows` timed windows of
`--steps` steps each, timed with CUDA events after a warm-up call of each arm. The host arm's window includes its
per-step draw and copy, which is what a caller pays. The final latents of both arms are compared bit for bit.

Serving arms: v1 with Euler ancestral and with DDIM eta = 1, `--requests` requests at 512 x 512 with steps from 20-30,
each seeded with its own CUDA generator: serial `pipe(...)` calls against the batcher with 4 and 8 slots. The card's
name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_schedulers import _card  # noqa: E402

H = 512


def _scheduler(name):
    from powerpaint_b200.schedulers import DDIMScheduler, EulerAncestralDiscreteScheduler

    return EulerAncestralDiscreteScheduler.from_config(DDIMScheduler().config) if name == "euler_a" else DDIMScheduler()


def loop_case(sampler: str, batch: int, steps: int, windows: int) -> dict:
    import torch

    import bench
    from powerpaint_b200.pipelines import common

    dev = torch.device("cuda:0")
    pipe = bench.build_pipeline(dict(mode="v1"), dev)
    den = pipe.denoiser()
    sch = _scheduler(sampler)
    sch.set_timesteps(steps)
    g = torch.Generator(device=dev).manual_seed(0)
    h = H // 8
    lat = torch.randn(batch, 4, h, h, device=dev, generator=g) * float(sch.init_noise_sigma)
    emb = torch.randn(2 * batch, 77, 768, device=dev, generator=g) * 0.5
    extra = torch.cat([(torch.rand(batch, 1, h, h, device=dev, generator=g) > 0.5).float(),
                       torch.randn(batch, 4, h, h, device=dev, generator=g)], 1)
    run = dict(latents=lat, prompt_embeds=emb, timesteps=sch.timesteps, guidance_scale=7.5, extra=extra)
    if sampler == "euler_a":
        run.update(coef=sch.step_coefficients(), scoef=sch.solver_coefficients())
    else:
        run.update(coef=sch.step_coefficients(sch.timesteps, eta=1.0))

    def arm(device_noise: bool, seed: int):
        gen = torch.Generator(device=dev).manual_seed(seed)
        if device_noise:
            return dict(randn_draws=common.device_randn_draws(gen, lat.shape, dev, steps))
        return dict(noise_fn=lambda i: torch.randn(lat.shape, generator=gen, device=dev))

    def timed(device_noise: bool, seed: int):
        kw = arm(device_noise, seed)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = den.run(**run, **kw)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps, out

    for dn in (False, True):  # warm-up: both plans recorded, the device plan's graph captured
        timed(dn, 1)
    res = {"host": [], "device": []}
    outs = {}
    for w in range(windows):
        for dn, k in ((False, "host"), (True, "device")) if w % 2 == 0 else ((True, "device"), (False, "host")):
            ms, outs[k] = timed(dn, 100 + w)
            res[k].append(ms)
    host, device = statistics.median(res["host"]), statistics.median(res["device"])
    return dict(sampler=sampler, batch=batch, steps=steps, host_ms_per_step=host, device_ms_per_step=device,
                host_windows=res["host"], device_windows=res["device"], speedup=host / device,
                same_latents=bool(torch.equal(outs["host"], outs["device"])))


def serving(requests: int) -> dict:
    import torch

    import bench
    from powerpaint_b200.serving import RequestBatcher

    dev = torch.device("cuda:0")
    out = {}
    for sampler, eta, label in (("euler_a", 0.0, "Euler ancestral"), ("ddim", 1.0, "DDIM eta=1")):
        pipe = bench.build_pipeline(dict(mode="v1"), dev)
        pipe.scheduler = _scheduler(sampler)
        g = torch.Generator().manual_seed(11)
        reqs = []
        for _ in range(requests):
            mask = torch.zeros(1, 1, H, H)
            mask[:, :, H // 4:3 * H // 4, H // 4:3 * H // 4] = 1
            reqs.append(dict(image=torch.rand(1, 3, H, H, generator=g) * 2 - 1, mask=mask,
                             prompt_embeds=torch.randn(1, 77, 768, generator=g) * 0.5,
                             negative_prompt_embeds=torch.randn(1, 77, 768, generator=g) * 0.5,
                             num_inference_steps=int(torch.randint(20, 31, (1,), generator=g)), guidance_scale=7.5,
                             eta=eta, output_type="pil", height=H, width=H))

        def serial(rs):
            t0 = time.perf_counter()
            for i, kw in enumerate(rs):
                pipe(generator=torch.Generator(device=dev).manual_seed(i), **kw)
            return time.perf_counter() - t0

        def batched(b, rs):
            t0 = time.perf_counter()
            hs = [b.submit(generator=torch.Generator(device=dev).manual_seed(i), **kw) for i, kw in enumerate(rs)]
            b.run()
            [h.result() for h in hs]
            return time.perf_counter() - t0

        batchers = {S: RequestBatcher(pipe, S, H, H) for S in (4, 8)}
        warm = [dict(r, num_inference_steps=2) for r in reqs[:8]]
        serial(warm[:1])
        for b in batchers.values():
            batched(b, warm)
        w = out[label] = {"serial images/s": requests / serial(reqs)}
        for S, b in batchers.items():
            w[f"batcher S={S} images/s"] = requests / batched(b, reqs)
            assert b.plans_recorded == 1
        print(f"{label:16s} " + "  ".join(f"{k} {v:.2f}" for k, v in w.items()))
        del pipe, batchers
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--case", default=None, help=argparse.SUPPRESS)  # sampler:batch, run in a child process
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing can be measured")
    if args.case:
        sampler, batch = args.case.split(":")
        print(json.dumps(loop_case(sampler, int(batch), args.steps, args.windows)))
        return
    name, limit = _card()
    out = dict(card=name, power_limit=limit, shape=f"v1 {H}x{H}, CFG", loops=[], serving=None)
    for sampler in ("euler_a", "ddim_eta1"):
        for batch in (8, 1):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", f"{sampler.split('_eta')[0]}:{batch}",
                                "--steps", str(args.steps), "--windows", str(args.windows)],
                               capture_output=True, text=True, cwd=ROOT)
            if r.returncode != 0:
                raise SystemExit(f"case {sampler} batch {batch} failed:\n{r.stdout}\n{r.stderr}")
            res = json.loads(r.stdout.strip().splitlines()[-1])
            res["sampler"] = sampler
            out["loops"].append(res)
            print(f"{sampler:10s} batch {batch}: host-drawn (eager) {res['host_ms_per_step']:.2f} ms/step, device-drawn "
                  f"(graph) {res['device_ms_per_step']:.2f} ms/step, x{res['speedup']:.3f}, same latents "
                  f"{res['same_latents']}  windows host {['%.2f' % v for v in res['host_windows']]} device "
                  f"{['%.2f' % v for v in res['device_windows']]}")
    out["serving"] = serving(args.requests)
    print(f"card: {name}, power limit {limit}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
