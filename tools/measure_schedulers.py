"""Step time and loop throughput of the fused loop per scheduler at the C2 shape (PowerPaint v1, 8 images of
512 x 512 with classifier-free guidance: UNet batch 16, 64 x 64 latents), synthetic SD-1.5 weights.

    python tools/measure_schedulers.py [--rounds 5] [--json OUT]

Rows:
* DDIM and DPM-Solver++ 2M on the graph path (one captured step replayed per step), 20 steps each;
* Euler ancestral and DDIM with eta = 1 on the noise path (program replay without a graph; each step's noise drawn
  on a CPU generator and copied to the device, as the pipelines draw it with a CPU generator), 20 steps each;
* loop images/s of DDIM at 50 steps and DPM-Solver++ 2M at 20 steps.
All loops are alternated `--rounds` times in the same process; per-step time = loop time / steps (it includes the
per-call set-up before the loop). One denoiser holds the plans of all four step kinds (DDIM / solver, with and without
noise), recorded and captured in a warm-up pass; the tool checks that no plan is re-recorded inside the timed window.
Times are CUDA events, the median over the rounds is reported with the card's name and power limit, read in the same
run. Output quality of the schedulers is not measured: the weights are synthetic.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch

    from oracle.unet import UNetConfig
    from powerpaint_b200.denoise import FusedDenoiser
    from powerpaint_b200.engine import NetConfig
    from powerpaint_b200.models import UNet2DConditionModel, synthetic_state_dict
    from powerpaint_b200.pipelines.common import randn_tensor
    from powerpaint_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing can be measured")
    dev = torch.device("cuda:0")
    o = UNetConfig.sd15(9)
    cfg = NetConfig(in_channels=9, block_out_channels=o.block_out_channels, attention_head_dim=o.attention_head_dim,
                    cross_attention_dim=o.cross_attention_dim, norm_num_groups=o.norm_num_groups)
    unet = UNet2DConditionModel.from_state_dict(cfg, synthetic_state_dict(cfg, "unet", 1234)).to(dev)
    den = FusedDenoiser(unet)
    den.MAX_PLANS = 4  # one plan per step kind, so no timed loop records or captures
    B, h = 8, 64
    g = torch.Generator(device=dev).manual_seed(0)
    lat = torch.randn(B, 4, h, h, device=dev, generator=g)
    emb = torch.randn(2 * B, 77, 768, device=dev, generator=g) * 0.5
    extra = torch.randn(B, 5, h, h, device=dev, generator=g)

    cpu_gen = torch.Generator().manual_seed(1)

    def noise_fn(i):
        return randn_tensor((B, 4, h, h), generator=cpu_gen, device=dev, dtype=torch.float32)

    def loop(name, steps):
        eta = 0.0
        if name.startswith("ddim"):
            s = DDIMScheduler()
            s.set_timesteps(steps)
            kw = {}
            if name == "ddim_eta":
                eta, kw["noise_fn"] = 1.0, noise_fn
        else:
            cls = DPMSolverMultistepScheduler if name == "dpmpp_2m" else EulerAncestralDiscreteScheduler
            s = cls.from_config(DDIMScheduler().config)
            s.set_timesteps(steps)
            kw = dict(scoef=s.solver_coefficients())
            if s.stochastic:
                kw["noise_fn"] = noise_fn
        coef = s.step_coefficients(eta=eta)

        def run():
            return den.run(latents=lat, prompt_embeds=emb, timesteps=s.timesteps, coef=coef, guidance_scale=7.5,
                           extra=extra, **kw)
        return run

    cases = {"ddim_20": loop("ddim", 20), "dpmpp_2m_20": loop("dpmpp_2m", 20), "euler_a_20": loop("euler_a", 20),
             "ddim_eta_20": loop("ddim_eta", 20), "ddim_50": loop("ddim", 50)}
    steps = {"ddim_20": 20, "dpmpp_2m_20": 20, "euler_a_20": 20, "ddim_eta_20": 20, "ddim_50": 50}
    for run in cases.values():  # record + capture + first replay
        run()
    torch.cuda.synchronize()
    plans = dict(den._cache)  # held, so a re-recorded plan can never reuse an evicted one's identity
    if len(plans) != 4:
        raise SystemExit(f"expected 4 recorded plans after the warm-up, found {len(plans)}")
    times = {k: [] for k in cases}
    for _ in range(args.rounds):
        for k, run in cases.items():  # alternated within each round
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
    if len(den._cache) != len(plans) or any(den._cache.get(k) is not v for k, v in plans.items()):
        raise SystemExit("a plan was re-recorded inside the timed window: the times include recording")
    name, limit = _card()
    out = dict(card=name, power_limit=limit, shape="C2: v1, 8 x 512^2, CFG (UNet batch 16)", rounds=args.rounds,
               rows={})
    for k, ts in times.items():
        med = statistics.median(ts)
        out["rows"][k] = dict(loop_ms=med, step_ms=med / steps[k], images_per_s=B / (med / 1e3),
                              spread_ms=[min(ts), max(ts)])
        print(f"{k:12s} loop {med:9.1f} ms  step {med / steps[k]:7.2f} ms  {B / (med / 1e3):6.2f} images/s "
              f"(min {min(ts):.1f}, max {max(ts):.1f})")
    print(f"card: {name}, power limit {limit}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
