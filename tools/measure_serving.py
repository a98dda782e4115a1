"""Throughput and latency of a stream of mixed requests: serial `pipe(...)` calls against `RequestBatcher`.

    python tools/measure_serving.py [--requests 32] [--rounds 1] [--json OUT]

Synthetic SD-1.5 weights at 512 x 512. The workload is a seeded stream of requests, every one submitted at t = 0, with
steps drawn from 20-50 and guidance from {5, 7.5, 10, 12}. Two workloads: PowerPaint v1 with DDIM, and BrushNet with
UniPC (the v2 app's sampler). Arms, alternated within each round: serial `pipe(...)` calls (one request at a time, what
a single-worker app queue does), the batcher with 4 slots and with 8 slots. Every arm returns PIL images, so a request
is complete when its host copy exists.

Reported per workload and arm: images/s over the whole stream, mean and p90 completion latency from t = 0, and the
rel-L2 of every batched image against its serial counterpart (uint8 pixels as floats). Also the replay time per step of
the slotted program against `FusedDenoiser`'s program at batch S, which shows the cost of the per-slot launches. The
card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_schedulers import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--replay-steps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from powerpaint_b200.schedulers import DDIMScheduler, UniPCMultistepScheduler
    from powerpaint_b200.serving import RequestBatcher

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing can be measured")
    dev = torch.device("cuda:0")
    H = 512

    def stream(mode, seed):
        g = torch.Generator().manual_seed(seed)
        out = []
        for i in range(args.requests):
            steps = int(torch.randint(20, 51, (1,), generator=g))
            guidance = [5.0, 7.5, 10.0, 12.0][int(torch.randint(0, 4, (1,), generator=g))]
            img = torch.rand(1, 3, H, H, generator=g) * 2 - 1
            kw = dict(image=img, prompt_embeds=torch.randn(1, 77, 768, generator=g) * 0.5,
                      negative_prompt_embeds=torch.randn(1, 77, 768, generator=g) * 0.5, num_inference_steps=steps,
                      guidance_scale=guidance, output_type="pil", height=H, width=H)
            if mode == "brushnet":
                mask = torch.ones(1, 3, H, H)
                mask[:, :, H // 4:3 * H // 4, H // 4:3 * H // 4] = -1.0
                kw.update(mask=mask, prompt_embedsU=torch.randn(2, 77, 768, generator=g) * 0.5)
            else:
                mask = torch.zeros(1, 1, H, H)
                mask[:, :, H // 4:3 * H // 4, H // 4:3 * H // 4] = 1
                kw.update(mask=mask)
            out.append(kw)
        return out

    def serial(pipe, reqs):
        torch.manual_seed(7)
        t0 = time.perf_counter()
        imgs, done = [], []
        for i, kw in enumerate(reqs):
            imgs.append(pipe(generator=torch.Generator(device=dev).manual_seed(i), **kw).images[0])
            done.append(time.perf_counter() - t0)
        return imgs, done, time.perf_counter() - t0

    def batched(b, reqs):
        torch.manual_seed(7)
        t0 = time.perf_counter()
        hs = [b.submit(generator=torch.Generator(device=dev).manual_seed(i), **kw) for i, kw in enumerate(reqs)]
        b.run()
        total = time.perf_counter() - t0
        return [h.result().images[0] for h in hs], [h.finished_at - t0 for h in hs], total

    def rel(a, b):
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-12))

    def events_ms(fn, n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(n)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n

    name, limit = _card()
    out = dict(card=name, power_limit=limit, requests=args.requests, rounds=args.rounds, size=H, workloads={})
    for mode, sched, label in (("v1", DDIMScheduler, "v1 DDIM"), ("brushnet", UniPCMultistepScheduler,
                                                                     "BrushNet UniPC")):
        pipe = bench.build_pipeline(dict(mode=mode), dev)
        pipe.scheduler = sched()
        reqs = stream(mode, 11)
        batchers = {S: RequestBatcher(pipe, S, H, H) for S in (4, 8)}
        # warm-up: every arm's plan recorded and captured before any timed pass
        warm = [dict(r, num_inference_steps=2) for r in reqs[:8]]
        serial(pipe, warm[:1])
        for b in batchers.values():
            batched(b, warm)
        torch.cuda.synchronize()
        arms = {"serial": lambda: serial(pipe, reqs)}
        arms.update({f"batcher S={S}": (lambda b=b: batched(b, reqs)) for S, b in batchers.items()})
        res = {k: dict(total=[], mean=[], p90=[]) for k in arms}
        images = {}
        for _ in range(args.rounds):
            for k, run in arms.items():
                imgs, done, total = run()
                images[k] = imgs
                res[k]["total"].append(total)
                res[k]["mean"].append(statistics.mean(done))
                res[k]["p90"].append(float(np.percentile(done, 90)))
        w = out["workloads"][label] = {}
        for k, r in res.items():
            tot = statistics.median(r["total"])
            w[k] = dict(images_per_s=args.requests / tot, stream_s=tot, latency_mean_s=statistics.median(r["mean"]),
                        latency_p90_s=statistics.median(r["p90"]))
            if k != "serial":
                rels = [rel(a, b) for a, b in zip(images[k], images["serial"])]
                w[k]["rel_l2_vs_serial_max"] = max(rels)
                w[k]["rel_l2_vs_serial_mean"] = statistics.mean(rels)
            print(f"{label:15s} {k:13s} {w[k]['images_per_s']:6.2f} img/s  latency mean {w[k]['latency_mean_s']:6.2f} s"
                  f"  p90 {w[k]['latency_p90_s']:6.2f} s" + (f"  rel-L2 max {w[k]['rel_l2_vs_serial_max']:.2e}"
                                                              if k != "serial" else ""))
        assert all(b.plans_recorded == 1 for b in batchers.values()), "a slotted plan was re-recorded"
        # per-step replay: the slotted program of S slots against FusedDenoiser's program at batch S
        for S, b in batchers.items():
            den = pipe.denoiser()
            lat = torch.randn(S, 4, H // 8, H // 8, device=dev)
            emb = torch.randn(2 * S, 77, 768, device=dev) * 0.5
            s = sched()
            s.set_timesteps(args.replay_steps)
            kw = dict(latents=lat, prompt_embeds=emb, timesteps=s.timesteps, coef=s.step_coefficients(),
                      guidance_scale=7.5)
            if mode == "brushnet":
                kw.update(extra=torch.randn(2 * S, 5, H // 8, H // 8, device=dev), side_prompt_embeds=emb,
                          ucoef=s.unipc_coefficients())
            else:
                kw.update(extra=torch.randn(S, 5, H // 8, H // 8, device=dev))
            den.run(**kw)
            prog = next(p for key, p in den._cache.items() if key[0] == S)["program"]
            fused = [events_ms(lambda n: [prog.launch() for _ in range(n)], args.replay_steps) for _ in range(3)]
            slotted = [events_ms(b.plan.replay, args.replay_steps) for _ in range(3)]
            w[f"replay S={S}"] = dict(slotted_step_ms=statistics.median(slotted), fused_step_ms=statistics.median(fused),
                                      slotted_launches=b.plan.launches_per_step, fused_launches=prog.num_launches)
            print(f"{label:15s} replay S={S}: slotted {statistics.median(slotted):.2f} ms/step "
                  f"({b.plan.launches_per_step} launches), FusedDenoiser batch {S} {statistics.median(fused):.2f} "
                  f"ms/step ({prog.num_launches} launches)")
        del pipe, batchers
        torch.cuda.empty_cache()
    print(f"card: {name}, power limit {limit}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
