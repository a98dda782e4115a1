"""The fused denoising loop: one recorded CUDA program per step, replayed as a CUDA graph.

Replaces the body of the reference loops
  v1          powerpaint/pipelines/pipeline_PowerPaint.py:988-1035
  v2 BrushNet powerpaint/pipelines/pipeline_PowerPaint_Brushnet_CA.py:1384-1449
  ControlNet  powerpaint/pipelines/pipeline_PowerPaint_ControlNet.py:1663-1735
i.e. per step: CFG duplication + channel concat -> [BrushNet | ControlNet] -> UNet -> CFG combine ->
DDIMScheduler.step. Here the step is a single `pp_program`:

    [side net forward]  ->  UNet forward (side-net residuals ride the UNet epilogues)
                        ->  pp_cfg_ddim_step: eps = u + s (c - u); x_{t-1}; writes the NEXT step's
                            bf16 channels-last net input for both CFG halves; bumps the step counter

The per-step scalars (timestep, DDIM coefficients, guidance scale) live in device tables indexed
by a device-side step counter, so one captured graph serves all steps; nothing crosses PCIe
inside the loop (the reference uploads `t` every step, unet_2d_condition.py:926). Step-invariant
work is hoisted: cross-attention K/V of the prompt(s), ControlNet's conditioning embedding, and
the constant input channels (mask, masked-image latents, BrushNet condition) are converted once.

All nets read ONE shared input buffer [n, h*w, 16]: channels 0..3 = latents, 4.. = the constant
channels of whichever net consumes them; nets that do not consume a channel carry zero weights
for it (weights are zero-padded at pack time), so no per-net concat exists. The constant channels are
written once per call; the step kernel only refreshes the four latent channels.

Per-step coefficient row (8 floats, `coef[step]`): 0-4 DDIM (sqrt(a_t), sqrt(1-a_t), sqrt(a_prev),
sqrt(1-a_prev-sigma^2), sigma), 5 guidance scale, 6 spare, 7 the 4-channel blend's sqrt(alpha_bar). The side nets'
conditioning scale x keep flag of the step (`brushnet_keep` / `controlnet_keep`, Brushnet_CA.py:1369-1376,1403-1409,
ControlNet.py:1652-1658) sits in a [MAX_STEPS, K] table, one column per side net. A recorded plan therefore serves
every guidance / conditioning scale and every control_guidance window.

Side-net options (the reference's `guess_mode`, `global_pool_conditions` and MultiControlNetModel):
- guess mode under CFG: the side net runs on the conditional half only (x_in[B:2B], the conditional prompt rows, B
  control images) and its zero-convs write the conditional rows of the 2B-row residual buffers the UNet reads. The
  unconditional rows are zeroed when the plan is recorded and never written again (ControlNet.py:1669-1701,
  Brushnet_CA.py:1394-1427). Residual k is scaled by the recorded constant logspace(-1, 0, n)[k] (`guess_mode_alphas`).
- global pooling: a pooled net's residuals are replaced by their spatial mean, broadcast to full size
  (pp_pool_broadcast); the logspace factors do not apply to it.
- K ControlNets record into the same program and activation pool, in net order; net k's zero-convs add net k-1's
  residuals through the epilogue's second residual, so the last net writes the sum the UNet reads.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Callable, Optional

import torch

from . import ops
from .engine import NetEngine, Pool, SideOutputs, guess_mode_alphas, lru_get
from .schedulers import PLMS_RING

MAX_STEPS = 1000
X_IN_C = 16
COEF_GUIDANCE = 5


class FusedDenoiser:
    """mode: 'v1' (UNet, 9-ch), 'brushnet' (BrushNet + 4-ch UNet), 'controlnet' (ControlNet + 9-ch UNet). For
    'controlnet', `side` may also be a list of ControlNets or a MultiControlNetModel (its `.nets`)."""

    def __init__(self, unet, side=None, mode: str = "v1"):
        if mode not in ("v1", "brushnet", "controlnet"):
            raise ValueError(mode)
        if (mode == "v1") != (side is None):
            raise ValueError("side net must be given exactly for modes 'brushnet' / 'controlnet'")
        sides = list(getattr(side, "nets", side)) if isinstance(side, (list, tuple)) or hasattr(side, "nets") \
            else ([side] if side is not None else [])
        if mode == "brushnet" and len(sides) != 1:
            raise ValueError("mode 'brushnet' takes exactly one BrushNet")
        if mode == "controlnet" and not sides:
            raise ValueError("mode 'controlnet' needs at least one ControlNet")
        self.unet = unet
        self.sides = sides
        self.side = sides[0] if sides else None
        self.mode = mode
        # recorded plans, least recently used first; a plan owns its activation pool (a few GB at C2), so only
        # MAX_PLANS shapes are kept
        self._cache: "OrderedDict[tuple, dict]" = OrderedDict()
        self._stream: Optional[torch.cuda.Stream] = None

    MAX_PLANS = 2

    # ------------------------------------------------------------------ plan
    def _get(self, B: int, h: int, w: int, do_cfg: bool, ctx_len: int, with_noise: bool,
             extra_per_copy: bool, sched: str = "ddim", blend: bool = False, guess: bool = False,
             device_noise: bool = False) -> dict:
        pools = tuple(bool(getattr(s.config, "global_pool_conditions", False)) for s in self.sides)
        # the key carries the parameter generation of each model: `load_state_dict` / `.to()` invalidate it,
        # and the cached entry keeps its engines alive, so a recycled id() can never alias a stale program
        key = (B, h, w, do_cfg, ctx_len, with_noise, device_noise, extra_per_copy, sched, blend, len(self.sides), guess,
               pools, self.unet.generation, tuple(s.generation for s in self.sides))
        for k in [k for k in self._cache if k[-2:] != key[-2:]]:  # (unet generation, side generations)
            del self._cache[k]  # plans recorded against replaced weights
        return lru_get(self._cache, key, self.MAX_PLANS, lambda: self._record(
            B, h, w, do_cfg, ctx_len, with_noise, extra_per_copy, sched, blend, guess, pools, device_noise))

    def _record(self, B, h, w, do_cfg, ctx_len, with_noise, extra_per_copy, sched, blend, guess, pools,
                device_noise=False) -> dict:
        """`with_noise`: the step reads host-drawn noise from st["noise"]; `device_noise`: the step kernel draws it
        from the B-entry pp_randn_draw table st["draws"]"""
        K = len(self.sides)
        dev = self.unet.device
        nb = 2 * B if do_cfg else B
        ns = B if guess and do_cfg else nb  # rows the side nets run on: the conditional half in guess mode
        ue: NetEngine = self.unet.engine()
        prog, ctxprog = ops.Program(), ops.Program()
        x_in = torch.zeros(nb, h * w, X_IN_C, dtype=torch.bfloat16, device=dev)
        timesteps = torch.zeros(MAX_STEPS, dtype=torch.float32, device=dev)
        step_idx = torch.zeros(1, dtype=torch.int32, device=dev)
        coef = torch.zeros(MAX_STEPS, 8, dtype=torch.float32, device=dev)
        side_scale = torch.zeros(MAX_STEPS, max(K, 1), dtype=torch.float32, device=dev)  # scale x keep per step, net
        pool = Pool(dev)  # the nets of one step share one activation pool
        common = dict(pool=pool, program=prog, ctx_program=ctxprog, steps=(timesteps, step_idx))
        st = dict(B=B, nb=nb, ns=ns, h=h, w=w, do_cfg=do_cfg, x_in=x_in, timesteps=timesteps, step_idx=step_idx,
                  coef=coef, side_scale=side_scale, program=prog, ctx_program=ctxprog, graph=False,
                  with_noise=with_noise, extra_per_copy=extra_per_copy,
                  engines=(ue,) + tuple(s.engine() for s in self.sides))
        side_x = x_in[nb - ns:]  # contiguous: the CFG halves are stacked [uncond; cond]
        down_s, mid_s, up_s = ue._state_shapes(nb, h, w)
        nd = len(down_s)
        # 2B-row residual buffers the UNet reads, in residual order; rows the side nets never write stay zero
        shapes = {"v1": [], "brushnet": down_s + [mid_s] + up_s, "controlnet": down_s + [mid_s]}[self.mode]
        res = [pool.tensor(nb, hh * ww, c, zero=True) for (c, hh, ww) in shapes]
        side_plans = []
        for k, net in enumerate(self.sides):  # in net order; the last one writes the side-net rows of `res`
            prev = side_plans[-1].outputs["down"] + [side_plans[-1].outputs["mid"]] if side_plans else None
            side = SideOutputs(scale=(side_scale[:, k], step_idx, K),
                               alphas=guess_mode_alphas(len(res)) if guess and not pools[k] else None,
                               global_pool=pools[k], prev=prev,
                               targets=[b[nb - ns:].reshape(-1, b.shape[-1]) for b in res] if k == K - 1 else None)
            side_plans.append(net.engine()._build_plan(ns, h, w, ctx_len, x_in=side_x, side=side, **common))
        uplan = ue._build_plan(nb, h, w, ctx_len, x_in=x_in, **common,
                               adds=(res[:nd], res[nd], res[nd + 1:]) if self.mode == "brushnet" else None,
                               cn=(res[:nd], res[nd]) if self.mode == "controlnet" else None)
        st["uplan"], st["side_plans"], st["residuals"] = uplan, side_plans, res
        # fp32 master latents and the constant channels (channels-last)
        n_extra = nb if extra_per_copy else B
        st["latents"] = torch.zeros(B, h * w, 4, dtype=torch.float32, device=dev)
        st["extra"] = torch.zeros(n_extra, h * w, 5, dtype=torch.float32, device=dev)
        st["noise"] = torch.zeros(B, h * w, 4, dtype=torch.float32, device=dev)
        # one entry per latent row at most (a list of generators); the entries a call does not use match no row
        st["draws"] = torch.zeros(B * ops.RANDN_DRAW_BYTES, dtype=torch.uint8, device=dev) if device_noise else None
        if sched == "unipc":
            # UniPCMultistepScheduler (the v2 app's scheduler, app.py:197): multistep state lives next to the latents
            for k in ("last_sample", "m1", "m2"):
                st[k] = torch.zeros(B, h * w, 4, dtype=torch.float32, device=dev)
            st["ucoef"] = torch.zeros(MAX_STEPS, 12, dtype=torch.float32, device=dev)
            prog.add(ops.unipc_desc(eps=uplan.outputs["eps"], eps_fp32=True, eps_ld=4, latents=st["latents"],
                                    last_sample=st["last_sample"], m1=st["m1"], m2=st["m2"], coef=coef,
                                    ucoef=st["ucoef"], step_idx=step_idx, advance_step=True, do_cfg=do_cfg, batch=B,
                                    hw=h * w, next_in=x_in, next_c=X_IN_C, n_copies=2 if do_cfg else 1))
        elif sched == "solver":
            # DPM-Solver++ / Euler / Euler-ancestral: the previous x0 prediction lives next to the latents
            st["m1"] = torch.zeros(B, h * w, 4, dtype=torch.float32, device=dev)
            st["scoef"] = torch.zeros(MAX_STEPS, 8, dtype=torch.float32, device=dev)
            prog.add(ops.solver_desc(eps=uplan.outputs["eps"], eps_fp32=True, eps_ld=4, latents=st["latents"],
                                     m1=st["m1"], coef=coef, scoef=st["scoef"], step_idx=step_idx, advance_step=True,
                                     do_cfg=do_cfg, batch=B, hw=h * w, noise=st["noise"] if with_noise else None,
                                     draws=st["draws"], next_in=x_in, next_c=X_IN_C, n_copies=2 if do_cfg else 1))
        else:
            if blend:  # 4-channel UNet: known region kept on the noised original after every step
                st["blend_x0"] = torch.zeros(h * w, 4, dtype=torch.float32, device=dev)
                st["blend_mask"] = torch.zeros(h * w, dtype=torch.float32, device=dev)
                st["blend_noise"] = torch.zeros(B, h * w, 4, dtype=torch.float32, device=dev)
        if sched == "plms":
            # PNDM / PLMS (the v1 checkpoint's scheduler): the first step's sample and a ring of 3 earlier eps
            st["cur_sample"] = torch.zeros(B, h * w, 4, dtype=torch.float32, device=dev)
            st["ets"] = torch.zeros(PLMS_RING, B, h * w, 4, dtype=torch.float32, device=dev)
            st["pcoef"] = torch.zeros(MAX_STEPS, 8, dtype=torch.float32, device=dev)
            prog.add(ops.plms_desc(eps=uplan.outputs["eps"], eps_fp32=True, eps_ld=4, latents=st["latents"],
                                   cur_sample=st["cur_sample"], ets=st["ets"], coef=coef, pcoef=st["pcoef"],
                                   step_idx=step_idx, advance_step=True, do_cfg=do_cfg, batch=B, hw=h * w,
                                   next_in=x_in, next_c=X_IN_C, n_copies=2 if do_cfg else 1,
                                   blend_x0=st.get("blend_x0"), blend_mask=st.get("blend_mask"),
                                   blend_noise=st.get("blend_noise")))
        elif sched == "ddim":
            prog.add(ops.cfg_ddim_desc(eps=uplan.outputs["eps"], eps_fp32=True, eps_ld=4, latents=st["latents"],
                                       coef=coef, step_idx=step_idx, advance_step=True,
                                       noise=st["noise"] if with_noise else None, draws=st["draws"], guidance_scale=0.0,
                                       guidance_from_coef=True, do_cfg=do_cfg, batch=B, hw=h * w, next_in=x_in,
                                       next_c=X_IN_C, n_copies=2 if do_cfg else 1, extra=None, extra_c=0,
                                       blend_x0=st.get("blend_x0"), blend_mask=st.get("blend_mask"),
                                       blend_noise=st.get("blend_noise")))
        st["bytes"] = pool.bytes
        return st

    def record_slots(self, S: int, h: int, w: int, sched: str = "ddim", ctx_len: int = 77) -> "SlottedPlan":
        """A step program with S independent slots (`SlottedPlan`); one pipeline mode, one latent size, classifier-free
        guidance always on. Records nothing into the plan cache of `run`."""
        if self.mode == "controlnet" and len(self.sides) != 1:
            raise NotImplementedError("slotted plans take one ControlNet")
        if any(getattr(s.config, "global_pool_conditions", False) for s in self.sides):
            raise NotImplementedError("slotted plans take no globally pooled side net")
        return SlottedPlan(self, S, h, w, sched, ctx_len)

    @property
    def launches_per_step(self) -> int:
        return max((s["program"].num_launches for s in self._cache.values()), default=0)

    # ------------------------------------------------------------------ run
    def _fill_x_in(self, st: dict, latents_only: bool = False, scale: float = 1.0):
        B, do_cfg, x_in = st["B"], st["do_cfg"], st["x_in"]
        lat16 = (st["latents"] * scale if scale != 1.0 else st["latents"]).to(torch.bfloat16)
        for cpy in range(2 if do_cfg else 1):
            x_in[cpy * B:(cpy + 1) * B, :, :4] = lat16
            if not latents_only:
                ex = st["extra"][cpy * B:(cpy + 1) * B] if st["extra_per_copy"] else st["extra"]
                x_in[cpy * B:(cpy + 1) * B, :, 4:9] = ex.to(torch.bfloat16)

    @torch.no_grad()
    def run(self, *, latents: torch.Tensor, prompt_embeds: torch.Tensor, timesteps, coef: torch.Tensor,
            guidance_scale: float, extra: Optional[torch.Tensor] = None,
            side_prompt_embeds: Optional[torch.Tensor] = None, control_image: Optional[torch.Tensor] = None,
            side_scale=1.0, side_keep=None,
            noise_fn: Optional[Callable[[int], torch.Tensor]] = None, ucoef: Optional[torch.Tensor] = None,
            scoef: Optional[torch.Tensor] = None, pcoef: Optional[torch.Tensor] = None, blend: Optional[dict] = None,
            callback: Optional[Callable[[int, int, torch.Tensor], Optional[torch.Tensor]]] = None,
            use_graph: bool = True, guess_mode: bool = False, randn_draws=None) -> torch.Tensor:
        """latents [B,4,h,w]; prompt_embeds [nb,77,768] for the UNet (negative half first when CFG);
        extra [B or nb,5,h,w] = constant channels (v1/controlnet: mask + masked-image latents;
        brushnet: conditioning latents + mask; nb rows = one set per CFG half); side_prompt_embeds
        for the side net; `side_scale` x `side_keep[i]` (default 1) scales the side net's residuals at step i;
        coef [n,8] from `DDIMScheduler.step_coefficients`; `noise_fn(i)` supplies
        the eta > 0 variance noise of step i; `ucoef` [n,12] (`UniPCMultistepScheduler.unipc_coefficients`) selects
        the UniPC step kernel instead of DDIM; `scoef` [n,8] (`solver_coefficients` of DPMSolverMultistepScheduler,
        EulerDiscreteScheduler, EulerAncestralDiscreteScheduler) selects `pp_solver_step`, with `noise_fn(i)` the
        noise of a stochastic step and column 7 of row 0 the input scale of the first step; `pcoef` [n,8]
        (`PNDMScheduler.plms_coefficients`) selects `pp_plms_step`, whose rows carry the whole PLMS state machine
        (a callback's replacement latents after step 0 only feed step 1's net input: that step restarts from the
        sample step 0 started at, as in diffusers); `blend` = dict(x0 [1,4,h,w], mask [1,1,h,w], noise [B,4,h,w],
        sqrt_alpha [n]) is the 4-channel-UNet blend (ref pipeline_PowerPaint.py:1025-1035).
        `randn_draws` (exclusive with `noise_fn`): the noise of the stochastic steps drawn by the step kernels, rows of
        pp_randn_draw fields (`pipelines.common.device_randn_draws`) covering the B latent rows; step i draws
        at offset0 + i * offset_per_step, so the loop stays one CUDA graph.
        `callback(i, t, latents_nchw)` may return replacement
        latents. Returns the final latents [B,4,h,w] fp32.
        K ControlNets: `side_scale` a list of K floats, `side_keep` None or a list of K per-step lists,
        `control_image` a list of K tensors. `guess_mode`: the side nets' residuals are scaled by logspace(-1, 0, n)
        (pooled nets excepted) and, under CFG, the side nets see only the conditional half: `side_prompt_embeds` may
        then be the 2B rows (the conditional B are used) or B rows, control images have B rows."""
        B, _, h, w = latents.shape
        nb = prompt_embeds.shape[0]
        do_cfg = nb == 2 * B
        if not do_cfg and nb != B:
            raise ValueError("prompt_embeds batch must be B or 2B")
        n_steps = len(timesteps)
        if n_steps > MAX_STEPS:
            raise ValueError(f"at most {MAX_STEPS} steps")
        extra_per_copy = extra is not None and do_cfg and extra.shape[0] == nb
        if extra is not None and extra.shape[0] not in (B, nb):
            raise ValueError("extra batch must be B or 2B")
        dev = self.unet.device
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=dev)
        K = len(self.sides)
        multi = isinstance(side_scale, (list, tuple))
        scales = [float(v) for v in side_scale] if multi else [float(side_scale)] * max(K, 1)
        keeps = (list(side_keep) if multi else [side_keep]) if side_keep is not None else [None] * len(scales)
        if K and (len(scales) != K or len(keeps) != K or (K > 1 and not multi)):
            raise ValueError(f"{K} side nets: side_scale and side_keep need one entry per net")
        for kp in keeps:
            if kp is not None and len(kp) != n_steps:
                raise ValueError("side_keep needs one entry per step")
        cur = torch.cuda.current_stream(dev)
        self._stream.wait_stream(cur)
        with torch.cuda.device(dev), torch.cuda.stream(self._stream):
            if sum(c is not None for c in (ucoef, scoef, pcoef)) > 1:
                raise ValueError("ucoef, scoef and pcoef select different step kernels: pass one")
            sched = "unipc" if ucoef is not None else "solver" if scoef is not None else \
                "plms" if pcoef is not None else "ddim"
            if noise_fn is not None and randn_draws is not None:
                raise ValueError("noise_fn and randn_draws are exclusive: pass one")
            stochastic = noise_fn is not None or randn_draws is not None
            if sched == "plms" and stochastic:
                raise NotImplementedError("PNDM has no stochastic step: noise_fn is DDIM / solver-only")
            if sched == "unipc" and (stochastic or blend is not None):
                raise NotImplementedError("eta / the 4-channel blend are DDIM-only on the fused path")
            if sched == "solver" and blend is not None:
                raise NotImplementedError("the 4-channel blend is DDIM-only on the fused path")
            st = self._get(B, h, w, do_cfg, prompt_embeds.shape[1], noise_fn is not None, extra_per_copy, sched,
                           blend is not None, bool(guess_mode) and K > 0, randn_draws is not None)
            if randn_draws is not None:
                if any(not (0 <= d[4] and d[4] + d[5] <= B) for d in randn_draws):
                    raise ValueError(f"randn_draws: rows outside the {B} latent rows")
                st["draws"].copy_(ops.randn_draw_bytes(randn_draws, B).to(dev))
            if sched == "unipc":
                if len(ucoef) != n_steps:
                    raise ValueError("ucoef needs one row per step")
                st["ucoef"][:n_steps].copy_(ucoef.to(dev, torch.float32))
                for k in ("last_sample", "m1", "m2"):
                    st[k].zero_()
            if sched == "plms":
                if len(pcoef) != n_steps:
                    raise ValueError("pcoef needs one row per step")
                st["pcoef"][:n_steps].copy_(pcoef.to(dev, torch.float32))
                st["cur_sample"].zero_()
                st["ets"].zero_()
            in_scale = lambda i: 1.0  # noqa: E731  (scale_model_input of step i)
            if sched == "solver":
                if len(scoef) != n_steps:
                    raise ValueError("scoef needs one row per step")
                sc = scoef.to(torch.float32).cpu()
                st["scoef"][:n_steps].copy_(sc.to(dev))
                st["m1"].zero_()
                in_scale = lambda i: float(sc[i, 7]) if i < n_steps else 1.0  # noqa: E731
            # ---- per-call inputs (all outside the loop)
            st["latents"].copy_(ops.nhwc_fp32_from_nchw(latents.to(dev)))
            if extra is not None:
                st["extra"].copy_(ops.nhwc_fp32_from_nchw(extra.to(dev)))
            else:
                st["extra"].zero_()
            self._fill_x_in(st, scale=in_scale(0))
            ts = torch.as_tensor([float(t) for t in timesteps], dtype=torch.float32)
            st["timesteps"][:n_steps].copy_(ts.to(dev))
            cf = coef.clone().float()
            cf[:, COEF_GUIDANCE] = float(guidance_scale)
            ss = torch.zeros(n_steps, max(K, 1))
            for k, (scale, kp) in enumerate(zip(scales, keeps)):
                keep = torch.ones(n_steps) if kp is None else torch.tensor([float(v) for v in kp])
                ss[:, k] = scale * keep
            st["side_scale"][:n_steps].copy_(ss.to(dev))
            if blend is not None:
                cf[:, 7] = torch.as_tensor(blend["sqrt_alpha"], dtype=torch.float32)
                st["blend_x0"].copy_(ops.nhwc_fp32_from_nchw(blend["x0"][:1].to(dev))[0])
                st["blend_mask"].copy_(blend["mask"][:1].to(dev, torch.float32).reshape(-1))
                st["blend_noise"].copy_(ops.nhwc_fp32_from_nchw(blend["noise"].to(dev)))
            st["coef"][:n_steps].copy_(cf.to(dev))
            st["step_idx"].zero_()
            st["uplan"].inputs["ctx"].copy_(prompt_embeds.to(dev, torch.bfloat16))
            if st["side_plans"]:
                if side_prompt_embeds is None:
                    raise ValueError("side_prompt_embeds required")
                ns = st["ns"]
                spe = side_prompt_embeds[-ns:] if side_prompt_embeds.shape[0] == nb else side_prompt_embeds
                images = control_image if isinstance(control_image, (list, tuple)) else [control_image]
                if self.mode == "controlnet" and (control_image is None or len(images) != K):
                    raise ValueError(f"control_image required: one per ControlNet ({K})")
                for k, sp in enumerate(st["side_plans"]):
                    sp.inputs["ctx"].copy_(spe.to(dev, torch.bfloat16))
                    if self.mode == "controlnet":
                        ci = sp.inputs["cond_in"]
                        ci.copy_(ops.nchw_to_nhwc(images[k].to(dev).float().contiguous(), ci.shape[-1]).view_as(ci))
                        sp.cond_program.run()
            st["ctx_program"].run()
            # ---- the loop
            prog = st["program"]
            if use_graph and callback is None and noise_fn is None:
                if not st["graph"]:
                    prog.build_graph()  # capture does not execute: device state is untouched
                    st["graph"] = True
                for _ in range(n_steps):
                    prog.launch()
            else:
                for i in range(n_steps):
                    if noise_fn is not None:
                        st["noise"].copy_(ops.nhwc_fp32_from_nchw(noise_fn(i).to(dev)))
                    prog.run()
                    if callback is not None:
                        cur_lat = ops.nchw_from_nhwc_fp32(st["latents"], h, w)
                        new = callback(i, timesteps[i], cur_lat)
                        if new is not None and new is not cur_lat:
                            st["latents"].copy_(ops.nhwc_fp32_from_nchw(new.to(dev)))
                            self._fill_x_in(st, latents_only=True, scale=in_scale(i + 1))
            out = ops.nchw_from_nhwc_fp32(st["latents"], h, w).clone()
        cur.wait_stream(self._stream)
        out.record_stream(cur)
        return out


# A slot's table row that leaves its latents where they are: x_{t-1} = x_t, no history written. An idle slot replays
# these rows, so its rows of the net input stay finite while other slots step.
_HOLD = {"coef": [1.0, 0.0, 1.0, 0.0, 0.0, 1.0, 0.0, 0.0],
         "ucoef": [0.0] * 7 + [1.0] + [0.0] * 4,          # use_c = 0, x_next = x
         "scoef": [0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 1.0],  # x_next = x, input scale 1
         "pcoef": [1.0, 0.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0]}  # x_next = x, no ring slot, no saved sample
_SCHED_TABLE = {"ddim": None, "unipc": "ucoef", "solver": "scoef", "plms": "pcoef"}


def _upload(dst: torch.Tensor, src: torch.Tensor) -> None:
    """dst <- src without a host synchronisation: a host tensor is staged in pinned memory and copied asynchronously
    (the pinned block is not reused before the copy has run)"""
    if src.device.type == "cpu":
        src = src.to(dst.dtype).contiguous().pin_memory()
        dst.copy_(src, non_blocking=True)
    else:
        dst.copy_(src)


class SlottedPlan:
    """One step program over S slots, each an independent request with its own step count, guidance scale, inputs,
    side-net scale and, for DDIM with eta > 0 and the stochastic solvers, its own device-drawn noise. Slot s owns the UNet rows 2s (unconditional) and 2s + 1 (conditional): the CFG pair of a slot is
    contiguous, so every step kernel runs unchanged on one slot (batch 1, two copies of the next input).

    Per slot the device holds a timestep table, an 8-float coefficient table (guidance in column 5), a side-net
    scale x keep table, a step counter, the scheduler state and one pp_randn_draw entry (batch 1). Each replay records, besides the shared nets, one time
    embedding per slot, one step launch per slot (advancing that slot's counter) and, for a side net, one zero-conv
    launch per slot and residual. `admit` loads a request's loop inputs (what the pipeline hands `FusedDenoiser.run`)
    into a slot, `hold` parks a slot on rows that keep its latents fixed, `replay(k)` runs k steps of every slot."""

    def __init__(self, fd: FusedDenoiser, S: int, h: int, w: int, sched: str, ctx_len: int):
        if S < 1:
            raise ValueError("a slotted plan needs at least one slot")
        if sched not in _SCHED_TABLE:
            raise ValueError(f"scheduler kind {sched!r}: one of {sorted(_SCHED_TABLE)}")
        self.fd, self.S, self.h, self.w, self.sched, self.ctx_len = fd, S, h, w, sched, ctx_len
        dev = fd.unet.device
        hw, nb = h * w, 2 * S
        f32 = dict(dtype=torch.float32, device=dev)
        ue: NetEngine = fd.unet.engine()
        self.program, self.ctx_program = ops.Program(), ops.Program()
        self.x_in = torch.zeros(nb, hw, X_IN_C, dtype=torch.bfloat16, device=dev)
        self.timesteps = torch.zeros(S, MAX_STEPS, **f32)
        self.step_idx = torch.zeros(S, dtype=torch.int32, device=dev)
        self.coef = torch.zeros(S, MAX_STEPS, 8, **f32)
        self.side_scale = torch.zeros(S, MAX_STEPS, 1, **f32)
        self.latents = torch.zeros(S, hw, 4, **f32)
        # the ddim / solver step launches always carry their slot's draw entry: a slot whose step has sigma / r[5]
        # equal to 0 (deterministic requests, the hold rows) draws nothing, so one plan serves every request
        self.draws = torch.zeros(S, ops.RANDN_DRAW_BYTES, dtype=torch.uint8, device=dev)
        self.pool = pool = Pool(dev)
        steps = [(self.timesteps[s], self.step_idx[s:s + 1]) for s in range(S)]
        common = dict(pool=pool, program=self.program, ctx_program=self.ctx_program, steps=steps)
        down_s, mid_s, up_s = ue._state_shapes(nb, h, w)
        nd = len(down_s)
        shapes = {"v1": [], "brushnet": down_s + [mid_s] + up_s, "controlnet": down_s + [mid_s]}[fd.mode]
        res = [pool.tensor(nb, hh * ww, c, zero=True) for (c, hh, ww) in shapes]
        self.side_plan = None
        if fd.side is not None:
            side = SideOutputs(scale=(self.side_scale[0, :, 0], self.step_idx[:1], 1),
                               targets=[b.reshape(-1, b.shape[-1]) for b in res],
                               slot_scales=[(self.side_scale[s], self.step_idx[s:s + 1], 1) for s in range(S)])
            self.side_plan = fd.side.engine()._build_plan(nb, h, w, ctx_len, x_in=self.x_in, side=side, **common)
        self.uplan = ue._build_plan(nb, h, w, ctx_len, x_in=self.x_in, **common,
                                    adds=(res[:nd], res[nd], res[nd + 1:]) if fd.mode == "brushnet" else None,
                                    cn=(res[:nd], res[nd]) if fd.mode == "controlnet" else None)
        self.state = {}  # scheduler state, one entry per slot per tensor
        table = _SCHED_TABLE[sched]
        if table is not None:
            self.state[table] = torch.zeros(S, MAX_STEPS, len(_HOLD[table]), **f32)
        if sched == "unipc":
            for k in ("last_sample", "m1", "m2"):
                self.state[k] = torch.zeros(S, hw, 4, **f32)
        elif sched == "solver":
            self.state["m1"] = torch.zeros(S, hw, 4, **f32)
        elif sched == "plms":
            self.state["cur_sample"] = torch.zeros(S, hw, 4, **f32)
            # one ring per slot: the kernel's ring stride is batch x hw, so slots cannot share one [RING, S, hw, 4] ring
            self.state["ets"] = [torch.zeros(PLMS_RING, 1, hw, 4, **f32) for _ in range(S)]
        eps = self.uplan.outputs["eps"]
        for s in range(S):
            slot = dict(eps=eps[2 * s:2 * s + 2], eps_fp32=True, eps_ld=4, latents=self.latents[s:s + 1],
                        coef=self.coef[s], step_idx=self.step_idx[s:s + 1], advance_step=True, do_cfg=True, batch=1,
                        hw=hw, next_in=self.x_in[2 * s:2 * s + 2], next_c=X_IN_C, n_copies=2)
            st = {k: v[s] if k in _HOLD or isinstance(v, list) else v[s:s + 1] for k, v in self.state.items()}
            if sched == "unipc":
                self.program.add(ops.unipc_desc(**slot, last_sample=st["last_sample"], m1=st["m1"], m2=st["m2"],
                                                ucoef=st["ucoef"]))
            elif sched == "solver":
                self.program.add(ops.solver_desc(**slot, m1=st["m1"], scoef=st["scoef"], draws=self.draws[s]))
            elif sched == "plms":
                self.program.add(ops.plms_desc(**slot, cur_sample=st["cur_sample"], ets=st["ets"], pcoef=st["pcoef"]))
            else:
                self.program.add(ops.cfg_ddim_desc(**slot, noise=None, draws=self.draws[s], guidance_scale=0.0,
                                                   guidance_from_coef=True))
        self.bytes = pool.bytes
        self.graph = False
        # the hold rows of every table, on the device: parking a slot is a device-to-device copy
        self._hold = {name: torch.tensor(_HOLD[name], **f32).expand(MAX_STEPS, len(_HOLD[name])).contiguous()
                      for name in ("coef", table) if name is not None}
        for s in range(S):
            self.hold(s)

    @property
    def launches_per_step(self) -> int:
        return self.program.num_launches

    def hold(self, s: int) -> None:
        """park slot s: latents zero, every table row a hold row, counter zero (its other input channels keep their
        last, finite values)"""
        self.latents[s].zero_()
        self.x_in[2 * s:2 * s + 2, :, :4].zero_()
        self.timesteps[s].zero_()
        self.side_scale[s].zero_()
        for name in ("coef", _SCHED_TABLE[self.sched]):
            if name is not None:
                t = self.coef if name == "coef" else self.state[name]
                t[s].copy_(self._hold[name])
        self.reset_counter(s)

    def reset_counter(self, s: int) -> None:
        self.step_idx[s:s + 1].zero_()

    def admit(self, s: int, *, latents, prompt_embeds, timesteps, coef, guidance_scale, extra=None,
              side_prompt_embeds=None, control_image=None, side_scale=1.0, side_keep=None, noise_fn=None, ucoef=None,
              scoef=None, pcoef=None, blend=None, callback=None, guess_mode=False, randn_draws=None) -> int:
        """load one request's loop inputs (the keywords the pipelines pass `FusedDenoiser.run`, for one image under
        classifier-free guidance) into slot s and re-run the per-prompt programs; returns the request's step count"""
        h, w, dev = self.h, self.w, self.x_in.device
        if noise_fn is not None or blend is not None or callback is not None or guess_mode:
            raise NotImplementedError("slots take no host-drawn noise, 4-channel blend, callback or guess mode")
        if randn_draws is not None and (self.sched not in ("ddim", "solver") or len(randn_draws) != 1
                                        or tuple(randn_draws[0][4:]) != (0, 1)):
            raise ValueError("a slot's device-drawn noise is one draw of its one latent row (DDIM / solver plans)")
        if tuple(latents.shape) != (1, 4, h, w) or prompt_embeds.shape[0] != 2:
            raise ValueError(f"a slot takes one {h}x{w} latent and its [negative; positive] prompt rows")
        given = {"ucoef": ucoef, "scoef": scoef, "pcoef": pcoef}
        table = _SCHED_TABLE[self.sched]
        if any(v is not None for k, v in given.items() if k != table) or (table and given[table] is None):
            raise ValueError(f"the plan was recorded for scheduler kind {self.sched!r}")
        n = len(timesteps)
        if not 1 <= n <= MAX_STEPS:
            raise ValueError(f"1 to {MAX_STEPS} steps")
        rows = slice(2 * s, 2 * s + 2)
        in_scale = 1.0
        if table is not None:
            tab = given[table].to(torch.float32)
            if len(tab) != n:
                raise ValueError(f"{table} needs one row per step")
            _upload(self.state[table][s, :n], tab)
            if table == "scoef":
                in_scale = float(tab[0, 7])
            for k, v in self.state.items():
                if k != table:
                    v[s].zero_()
        lat = ops.nhwc_fp32_from_nchw(latents.to(dev, torch.float32))
        self.latents[s:s + 1].copy_(lat)
        self.x_in[rows, :, :4] = (lat * in_scale if in_scale != 1.0 else lat).to(torch.bfloat16)
        if extra is not None:
            self.x_in[rows, :, 4:9] = ops.nhwc_fp32_from_nchw(extra.to(dev, torch.float32)).to(torch.bfloat16)
        else:
            self.x_in[rows, :, 4:9] = 0
        _upload(self.timesteps[s, :n], torch.as_tensor([float(t) for t in timesteps], dtype=torch.float32))
        cf = coef.clone().float()
        cf[:, COEF_GUIDANCE] = float(guidance_scale)
        _upload(self.coef[s, :n], cf)
        keep = torch.ones(n) if side_keep is None else torch.tensor([float(v) for v in side_keep])
        if len(keep) != n:
            raise ValueError("side_keep needs one entry per step")
        _upload(self.side_scale[s, :n, 0], float(side_scale) * keep)
        self.uplan.inputs["ctx"][rows].copy_(prompt_embeds.to(dev, torch.bfloat16))
        if self.side_plan is not None:
            if side_prompt_embeds is None:
                raise ValueError("side_prompt_embeds required")
            self.side_plan.inputs["ctx"][rows].copy_(side_prompt_embeds[-2:].to(dev, torch.bfloat16))
            if self.fd.mode == "controlnet":
                img = control_image[0] if isinstance(control_image, (list, tuple)) else control_image
                if img is None or img.shape[0] != 2:
                    raise ValueError("control_image: one image per CFG half")
                ci = self.side_plan.inputs["cond_in"]
                ci[rows].copy_(ops.nchw_to_nhwc(img.to(dev).float().contiguous(), ci.shape[-1]).view_as(ci[rows]))
                self.side_plan.cond_program.run()
        _upload(self.draws[s], ops.randn_draw_bytes(randn_draws or [], 1))
        self.ctx_program.run()
        self.reset_counter(s)
        return n

    def replay(self, k: int) -> None:
        """k steps of every slot: the captured graph, captured on first use"""
        if not self.graph:
            self.program.build_graph()
            self.graph = True
        for _ in range(k):
            self.program.launch()

    def slot_latents(self, s: int) -> torch.Tensor:
        """slot s's latents [1, 4, h, w] fp32 (a copy)"""
        return ops.nchw_from_nhwc_fp32(self.latents[s:s + 1], self.h, self.w).clone()
