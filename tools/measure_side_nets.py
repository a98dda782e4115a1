"""Step time of the fused loop with the side-net options, synthetic SD-1.5 weights, DDIM, graph replay.

    python tools/measure_side_nets.py [--rounds 5] [--steps 20] [--json OUT]

Rows:
* at the C5 per-GPU shape (PowerPaint v1 + ControlNet, 2 images of 512 x 512 with classifier-free guidance: UNet batch
  4, 64 x 64 latents): one ControlNet, two ControlNets, one ControlNet in guess mode;
* at the C3 per-GPU shape (PowerPaint v2 BrushNet, 4 images of 512 x 512 with CFG: UNet batch 8): BrushNet, BrushNet in
  guess mode.
Each row has its own denoiser; every plan is recorded and captured in a warm-up pass, and the tool checks that none is
re-recorded inside the timed window. The rows are alternated `--rounds` times in the same process; per-step time =
loop time / steps (it includes the per-call set-up before the loop). Times are CUDA events; the median over the rounds
is reported with the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_schedulers import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch

    from oracle.unet import UNetConfig
    from powerpaint_b200.denoise import FusedDenoiser
    from powerpaint_b200.engine import NetConfig
    from powerpaint_b200.models import BrushNetModel, ControlNetModel, UNet2DConditionModel, synthetic_state_dict
    from powerpaint_b200.schedulers import DDIMScheduler

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing can be measured")
    dev = torch.device("cuda:0")

    def model(cls, kind, cin, seed):
        o = UNetConfig.sd15(cin)
        cfg = NetConfig(in_channels=cin, block_out_channels=o.block_out_channels,
                        attention_head_dim=o.attention_head_dim, cross_attention_dim=o.cross_attention_dim,
                        norm_num_groups=o.norm_num_groups)
        return cls.from_state_dict(cfg, synthetic_state_dict(cfg, kind, seed)).to(dev)

    u9, u4 = model(UNet2DConditionModel, "unet", 9, 1234), model(UNet2DConditionModel, "unet", 4, 1234)
    cns = [model(ControlNetModel, "controlnet", 4, 77), model(ControlNetModel, "controlnet", 4, 78)]
    bn = model(BrushNetModel, "brushnet", 4, 99)
    s = DDIMScheduler()
    s.set_timesteps(args.steps)
    ts, coef = s.timesteps, s.step_coefficients()
    g = torch.Generator(device=dev).manual_seed(0)
    h = 64

    def controlnet_row(K, guess):
        B = 2
        den = FusedDenoiser(u9, cns[:K], "controlnet")
        lat = torch.randn(B, 4, h, h, device=dev, generator=g)
        emb = torch.randn(2 * B, 77, 768, device=dev, generator=g) * 0.5
        extra = torch.randn(B, 5, h, h, device=dev, generator=g)
        ctl = [torch.rand(B if guess else 2 * B, 3, 8 * h, 8 * h, device=dev, generator=g) for _ in range(K)]
        kw = dict(control_image=ctl, side_scale=[0.5] * K) if K > 1 else dict(control_image=ctl[0], side_scale=0.5)

        def run():
            return den.run(latents=lat, prompt_embeds=emb, side_prompt_embeds=emb, timesteps=ts, coef=coef,
                           guidance_scale=7.5, extra=extra, guess_mode=guess, **kw)
        return den, run

    def brushnet_row(guess):
        B = 4
        den = FusedDenoiser(u4, bn, "brushnet")
        lat = torch.randn(B, 4, h, h, device=dev, generator=g)
        emb_t = torch.randn(2 * B, 77, 768, device=dev, generator=g) * 0.5
        emb_u = torch.randn(2 * B, 77, 768, device=dev, generator=g) * 0.5
        cond = torch.randn(B if guess else 2 * B, 5, h, h, device=dev, generator=g)

        def run():
            return den.run(latents=lat, prompt_embeds=emb_u, side_prompt_embeds=emb_t, timesteps=ts, coef=coef,
                           guidance_scale=7.5, extra=cond, side_scale=1.0, guess_mode=guess)
        return den, run

    rows = {"C5 v1 + 1 ControlNet": controlnet_row(1, False), "C5 v1 + 2 ControlNets": controlnet_row(2, False),
            "C5 v1 + 1 ControlNet, guess mode": controlnet_row(1, True),
            "C3 BrushNet": brushnet_row(False), "C3 BrushNet, guess mode": brushnet_row(True)}
    for _, run in rows.values():  # record + capture + first replay
        run()
    torch.cuda.synchronize()
    plans = {k: dict(den._cache) for k, (den, _) in rows.items()}
    if any(len(p) != 1 for p in plans.values()):
        raise SystemExit("expected one recorded plan per row after the warm-up")
    times = {k: [] for k in rows}
    for _ in range(args.rounds):
        for k, (_, run) in rows.items():  # alternated within each round
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
    for k, (den, _) in rows.items():
        if len(den._cache) != 1 or any(den._cache.get(key) is not v for key, v in plans[k].items()):
            raise SystemExit(f"{k}: a plan was re-recorded inside the timed window")
    name, limit = _card()
    out = dict(card=name, power_limit=limit, steps=args.steps, rounds=args.rounds, rows={})
    for k, tt in times.items():
        med = statistics.median(tt)
        out["rows"][k] = dict(loop_ms=med, step_ms=med / args.steps, spread_ms=[min(tt), max(tt)])
        print(f"{k:34s} step {med / args.steps:7.2f} ms  (loop min {min(tt):.1f}, median {med:.1f}, max {max(tt):.1f})")
    print(f"card: {name}, power limit {limit}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
