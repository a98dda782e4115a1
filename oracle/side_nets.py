"""Side-net options over the fp32 oracle nets of oracle/unet.py (which stays unchanged): guess mode's per-residual
scaling, global pooling (`global_pool_conditions`) and the Multi-ControlNet sum.

Restated from the reference's BrushNet forward (powerpaint/models/BrushNet_CA.py:905-943) and, for the ControlNet,
from diffusers 0.27.0 `ControlNetModel.forward` / `MultiControlNetModel.forward` as recalled:
  - guess mode and not pooled: residual k is multiplied by logspace(-1, 0, n)[k] * conditioning_scale (n = 13 for a
    ControlNet, 28 for a BrushNet); otherwise every residual by conditioning_scale;
  - pooled: each residual is replaced by its spatial mean, [B, C, 1, 1], which the UNet broadcast-adds;
  - Multi-ControlNet: the nets' residuals are summed in net order.
The oracle nets multiply by their `conditioning_scale` argument; they are called with 1 here and scaled after, which
is the same map (the zero-convs are linear in that factor).
"""
from __future__ import annotations

from typing import List, Sequence

import torch


def guess_scales(n: int) -> torch.Tensor:
    """logspace(-1, 0, n) in float64: 10 ** (-1 + k / (n - 1))"""
    return torch.logspace(-1, 0, n, dtype=torch.float64)


def scale_and_pool(residuals: List[torch.Tensor], conditioning_scale: float, guess_mode: bool,
                   pool: bool) -> List[torch.Tensor]:
    """the scaling then pooling tail of a side net's forward, over its residuals in order (down..., mid[, up...])"""
    n = len(residuals)
    if guess_mode and not pool:
        s = guess_scales(n).to(residuals[0].device) * conditioning_scale
        out = [r * s[k].to(r.dtype) for k, r in enumerate(residuals)]
    else:
        out = [r * conditioning_scale for r in residuals]
    if pool:
        out = [torch.mean(r, dim=(2, 3), keepdim=True) for r in out]
    return out


@torch.no_grad()
def controlnet(net, sample, timestep, emb, cond, conditioning_scale: float = 1.0, guess_mode: bool = False,
               pool: bool = False):
    """(down[12], mid) of an oracle ControlNet with the guess-mode / pooling options"""
    down, mid = net(sample, timestep, emb, cond, 1.0)
    res = scale_and_pool(list(down) + [mid], conditioning_scale, guess_mode, pool)
    return res[:-1], res[-1]


@torch.no_grad()
def brushnet(net, sample, timestep, emb, cond, conditioning_scale: float = 1.0, guess_mode: bool = False,
             pool: bool = False):
    """(down[12], mid, up[15]) of an oracle BrushNet with the guess-mode / pooling options"""
    down, mid, up = net(sample, timestep, emb, cond, 1.0)
    nd = len(down)
    res = scale_and_pool(list(down) + [mid] + list(up), conditioning_scale, guess_mode, pool)
    return res[:nd], res[nd], res[nd + 1:]


@torch.no_grad()
def multi_controlnet(nets: Sequence, pools: Sequence[bool], sample, timestep, emb, conds: Sequence[torch.Tensor],
                     scales: Sequence[float], guess_mode: bool = False):
    """the Multi-ControlNet sum, net 0 first (nets without a scale or image are dropped, as `zip` does)"""
    down = mid = None
    for i, (cond, scale, net, pool) in enumerate(zip(conds, scales, nets, pools)):
        d, m = controlnet(net, sample, timestep, emb, cond, scale, guess_mode, pool)
        if i == 0:
            down, mid = d, m
        else:
            down = [a + b for a, b in zip(down, d)]
            mid = mid + m
    return down, mid


@torch.no_grad()
def loop_controlnet(unet, nets, pools, sched, latents, prompt_embeds, mask, masked_image_latents, control_images,
                    guidance_scale: float, scales, keeps=None, guess_mode: bool = False):
    """the ControlNet loop of pipeline_PowerPaint_ControlNet.py:1663-1735 with K nets, guess mode and pooling.
    control_images: K tensors of B rows (doubled here for CFG unless guess mode, :855-856); keeps[k][i] =
    `controlnet_keep[i][k]`. Under guess mode + CFG the nets see the conditional half only and the unconditional
    half of every residual is zero (:1669-1701)."""
    do_cfg = guidance_scale > 1.0
    B = latents.shape[0]
    if do_cfg:
        mask = torch.cat([mask] * 2)
        masked_image_latents = torch.cat([masked_image_latents] * 2)
    half = guess_mode and do_cfg
    conds = [c if half or not do_cfg else torch.cat([c] * 2) for c in control_images]
    for i, t in enumerate(sched.timesteps):
        x4 = torch.cat([latents] * 2) if do_cfg else latents
        xc, ec = (latents, prompt_embeds[B:]) if half else (x4, prompt_embeds)
        cs = [s * (keeps[k][i] if keeps is not None else 1.0) for k, s in enumerate(scales)]
        d, m = multi_controlnet(nets, pools, xc, int(t), ec, conds, cs, guess_mode)
        if half:
            d = [torch.cat([torch.zeros_like(r), r]) for r in d]
            m = torch.cat([torch.zeros_like(m), m])
        x9 = torch.cat([x4, mask, masked_image_latents], dim=1)
        eps = unet(x9, int(t), prompt_embeds, down_block_additional_residuals=d, mid_block_additional_residual=m)
        if do_cfg:
            a, c = eps.chunk(2)
            eps = a + guidance_scale * (c - a)
        latents = sched.step(eps, int(t), latents)
    return latents


@torch.no_grad()
def loop_brushnet(unet, net, pool: bool, sched, latents, prompt_embeds_task, prompt_embeds_u, conditioning_latents,
                  guidance_scale: float, conditioning_scale: float = 1.0, guess_mode: bool = False):
    """the BrushNet loop of pipeline_PowerPaint_Brushnet_CA.py:1384-1449 with guess mode and pooling.
    conditioning_latents: the rows the BrushNet sees (2B under CFG, B in guess mode, whose images are not doubled)"""
    do_cfg = guidance_scale > 1.0
    B = latents.shape[0]
    half = guess_mode and do_cfg
    for i, t in enumerate(sched.timesteps):
        x = torch.cat([latents] * 2) if do_cfg else latents
        xc, ec = (latents, prompt_embeds_task[B:]) if half else (x, prompt_embeds_task)
        d, m, u = brushnet(net, xc, int(t), ec, conditioning_latents, conditioning_scale, guess_mode, pool)
        if half:
            d = [torch.cat([torch.zeros_like(r), r]) for r in d]
            m = torch.cat([torch.zeros_like(m), m])
            u = [torch.cat([torch.zeros_like(r), r]) for r in u]
        eps = unet(x, int(t), prompt_embeds_u, down_block_add_samples=d, mid_block_add_sample=m,
                   up_block_add_samples=u)
        if do_cfg:
            a, c = eps.chunk(2)
            eps = a + guidance_scale * (c - a)
        latents = sched.step(eps, int(t), latents)
    return latents
