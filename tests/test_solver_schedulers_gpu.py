"""GPU tests of `pp_solver_step` and of the fused loops with DPMSolverMultistepScheduler, EulerDiscreteScheduler and
EulerAncestralDiscreteScheduler: the kernel against a float64 evaluation of its row formula, the eager
`scheduler.step` against the stepwise oracles (oracle/dpmsolver.py, oracle/euler.py), and the three loops against fp32
oracle loops driven by the oracle schedulers, held to DESIGN's trajectory bounds (rel-L2 <= 5e-2, cosine >= 0.999 at
SD-1.5 width; cosine >= 0.998 for the tiny nets, as in test_pipelines_gpu.py)."""
import pytest
import torch

from oracle.dpmsolver import DPMSolverOracle
from oracle.euler import EulerAncestralOracle, EulerOracle
from powerpaint_b200.schedulers import (DDIMScheduler, DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                        EulerDiscreteScheduler)
from test_pipelines_gpu import _cos, _nets, _rel

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _fp32_exact():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _ref_step(eps, x, m1, noise, scoef, coef, step, do_cfg, B):
    """float64 evaluation of the row formula (include/powerpaint_b200.h, pp_solver_desc)"""
    r = scoef[step].double()
    e = eps.double()
    if do_cfg:
        u, c = e[:B], e[B:2 * B]
        e = u + float(coef[step, 5]) * (c - u)
    else:
        e = e[:B]
    mt = r[0] * x.double() + r[1] * e
    xn = r[2] * x.double() + r[3] * mt + r[4] * m1.double() + (r[5] * noise.double() if noise is not None else 0)
    return xn, mt, r[6] * xn


def test_solver_step_kernel_matches_the_row_formula_and_replays_bit_identically():
    from powerpaint_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(0)
    B, hw, C = 2, 37 * 13, 16
    scoef = torch.randn(3, 8, device=DEV, generator=g)
    coef = torch.zeros(3, 8, device=DEV)
    coef[:, 5] = torch.tensor([7.5, 3.0, 1.5])
    for do_cfg in (False, True):
        for with_noise in (False, True):
            for n_copies in (1, 2, 3):
                for eps_kind in ("fp32_vec", "bf16_strided"):
                    nb = 2 * B if do_cfg else B
                    if eps_kind == "fp32_vec":
                        eps, eps_fp32, eps_ld = torch.randn(nb, hw, 4, device=DEV, generator=g), True, 4
                        eps_view = eps
                    else:
                        eps = torch.randn(nb, hw, 8, device=DEV, generator=g).to(torch.bfloat16)
                        eps_fp32, eps_ld, eps_view = False, 8, eps[..., :4].float()
                    x0 = torch.randn(B, hw, 4, device=DEV, generator=g)
                    m0 = torch.randn(B, hw, 4, device=DEV, generator=g)
                    nz = torch.randn(B, hw, 4, device=DEV, generator=g) if with_noise else None
                    outs = []
                    for mode in ("eager", "program", "graph"):
                        lat, m1 = x0.clone(), m0.clone()
                        nxt = torch.zeros(n_copies * B, hw, C, dtype=torch.bfloat16, device=DEV)
                        idx = torch.tensor([1], dtype=torch.int32, device=DEV)
                        d = ops.solver_desc(eps=eps, eps_fp32=eps_fp32, eps_ld=eps_ld, latents=lat, m1=m1, coef=coef,
                                            scoef=scoef, step_idx=idx, advance_step=mode != "eager", do_cfg=do_cfg,
                                            batch=B, hw=hw, noise=nz, next_in=nxt, next_c=C, n_copies=n_copies)
                        if mode == "eager":
                            ops.run(d)
                        else:
                            p = ops.Program()
                            p.add(d)
                            if mode == "graph":
                                p.build_graph()
                                p.launch()
                            else:
                                p.run()
                            assert int(idx) == 2
                        torch.cuda.synchronize()
                        outs.append((lat, m1, nxt))
                    xn, mt, ni = _ref_step(eps_view, x0, m0, nz, scoef, coef, 1, do_cfg, B)
                    lat, m1, nxt = outs[0]
                    tol = 1e-5 * max(1.0, float(xn.abs().max()))
                    assert (lat.double() - xn).abs().max() < tol and (m1.double() - mt).abs().max() < tol
                    for c in range(n_copies):
                        blk = nxt[c * B:(c + 1) * B]
                        assert (blk[..., :4].double() - ni).abs().max() <= 8e-3 * max(1.0, float(ni.abs().max()))
                        # bit for bit: bf16 of the fp32 product r6 * x_next of the stored x_next
                        assert torch.equal(blk[..., :4], (scoef[1, 6] * lat).to(torch.bfloat16))
                        assert (blk[..., 4:] == 0).all()
                    for lat2, m12, nxt2 in outs[1:]:
                        assert torch.equal(lat2, lat) and torch.equal(m12, m1) and torch.equal(nxt2, nxt)


def _eager_vs_oracle(sp, so, steps, B=2, h=8):
    sp.set_timesteps(steps)
    so.set_timesteps(steps)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 4, h, h, generator=g) * float(sp.init_noise_sigma)
    x_o, x_p = x.double(), x.to(DEV)
    gp, go = torch.Generator().manual_seed(11), torch.Generator().manual_seed(11)
    for t in so.timesteps:
        eps = torch.randn(B, 4, h, h, generator=g)
        x_o = so.step(eps.double(), t, x_o, generator=go)
        x_p = sp.step(eps.to(DEV), t, x_p, generator=gp).prev_sample
    assert torch.equal(torch.randn(3, generator=gp), torch.randn(3, generator=go))  # same draws consumed
    return _rel(x_p.cpu(), x_o)


def test_eager_step_matches_the_oracle_step():
    base = DDIMScheduler().config
    sde = dict(algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min")
    assert _eager_vs_oracle(DPMSolverMultistepScheduler.from_config(base, use_karras_sigmas=True),
                            DPMSolverOracle(use_karras_sigmas=True), 12) < 1e-5
    assert _eager_vs_oracle(DPMSolverMultistepScheduler.from_config(base, **sde), DPMSolverOracle(**sde), 9) < 1e-5
    assert _eager_vs_oracle(EulerDiscreteScheduler.from_config(base), EulerOracle(),
                            7) < 1e-5
    assert _eager_vs_oracle(EulerAncestralDiscreteScheduler.from_config(base), EulerAncestralOracle(), 7) < 1e-5
    # an fp32 channels_last sample is read, never written
    s = DPMSolverMultistepScheduler.from_config(base)
    s.set_timesteps(5)
    x = torch.randn(1, 4, 8, 8, device=DEV).to(memory_format=torch.channels_last)
    keep = x.clone()
    out = s.step(torch.randn_like(x), s.timesteps[0], x).prev_sample
    assert torch.equal(x, keep) and not torch.equal(out, keep)


SCHEDS = {
    "dpmpp_2m": (lambda: DPMSolverMultistepScheduler.from_config(DDIMScheduler().config),
                 lambda: DPMSolverOracle()),
    "sde_dpmpp_2m": (lambda: DPMSolverMultistepScheduler.from_config(
        DDIMScheduler().config, algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min"),
        lambda: DPMSolverOracle(algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min")),
    "euler_a": (lambda: EulerAncestralDiscreteScheduler.from_config(DDIMScheduler().config),
                lambda: EulerAncestralOracle()),
}


@torch.no_grad()
def _oracle_loop(mode, om_u, om_s, so, lat, emb, extra, ctrl, gs, side_scale, noise):
    """the reference loops with `scale_model_input` before the nets (v1 :993, Brushnet_CA :1391, ControlNet :1666) and
    the step's noise taken from `noise[i]`"""
    B = lat.shape[0]
    for i, t in enumerate(so.timesteps):
        x = so.scale_model_input(torch.cat([lat] * 2), t).float()
        if mode == "v1":
            eps = om_u(torch.cat([x, torch.cat([extra] * 2)], 1), int(t), emb)
        elif mode == "brushnet":
            d, m, u = om_s(x, int(t), emb, extra, side_scale)
            eps = om_u(x, int(t), emb, down_block_add_samples=d, mid_block_add_sample=m, up_block_add_samples=u)
        else:
            d, m = om_s(x, int(t), emb, ctrl, side_scale)
            eps = om_u(torch.cat([x, torch.cat([extra] * 2)], 1), int(t), emb, down_block_additional_residuals=d,
                       mid_block_additional_residual=m)
        u_, c_ = eps.chunk(2)
        eps = u_ + gs * (c_ - u_)
        lat = so.step(eps, t, lat, variance_noise=noise[i] if noise is not None else None).float()
    assert lat.shape[0] == B
    return lat


@pytest.mark.parametrize("mode", ["v1", "brushnet", "controlnet"])
@pytest.mark.parametrize("sched", ["dpmpp_2m", "sde_dpmpp_2m", "euler_a"])
def test_loops_tiny_against_the_oracle_loop(mode, sched):
    from powerpaint_b200.denoise import FusedDenoiser

    kinds = {"v1": (9, [("unet", 9, 1234)]), "brushnet": (4, [("unet", 4, 1234), ("brushnet", 4, 99)]),
             "controlnet": (9, [("unet", 9, 1234), ("controlnet", 4, 77)])}[mode]
    nets = _nets(*kinds)
    om_u, pm_u, o = nets["unet"]
    side = nets.get("brushnet") or nets.get("controlnet")
    g = torch.Generator(device=DEV).manual_seed(4)
    B, h, steps = 2, 8, 8
    sp, so = SCHEDS[sched][0](), SCHEDS[sched][1]()
    sp.set_timesteps(steps)
    so.set_timesteps(steps)
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g) * float(sp.init_noise_sigma)
    emb = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    extra = torch.randn(2 * B if mode == "brushnet" else B, 5, h, h, device=DEV, generator=g)
    ctrl = torch.cat([torch.rand(B, 3, 8 * h, 8 * h, device=DEV, generator=g)] * 2) if mode == "controlnet" else None
    noise = [torch.randn(B, 4, h, h, device=DEV, generator=g) for _ in range(steps)] if sp.stochastic else None
    so.sigmas = so.sigmas.float().to(DEV)
    so.timesteps = so.timesteps.to(DEV)
    ref = _oracle_loop(mode, om_u, side[0] if side else None, so, lat, emb, extra, ctrl, 7.5, 0.8, noise)
    den = FusedDenoiser(pm_u, side[1] if side else None, mode)
    got = den.run(latents=lat, prompt_embeds=emb, timesteps=sp.timesteps, coef=sp.step_coefficients(),
                  scoef=sp.solver_coefficients(), guidance_scale=7.5, extra=extra,
                  side_prompt_embeds=emb if side else None, control_image=ctrl, side_scale=0.8,
                  noise_fn=(lambda i: noise[i]) if noise is not None else None)
    assert torch.isfinite(got).all()
    # the tiny-config bound of test_pipelines_gpu.py: the randomly initialised tiny nets amplify bf16 rounding
    assert _rel(got, ref) < 5e-2 and _cos(got, ref) > 0.998, (mode, sched, _rel(got, ref), _cos(got, ref))
    if noise is None:
        assert den._cache[next(iter(den._cache))]["graph"], "the deterministic solver replays one CUDA graph"
    # two runs of the same call: bit-identical latents
    again = den.run(latents=lat, prompt_embeds=emb, timesteps=sp.timesteps, coef=sp.step_coefficients(),
                    scoef=sp.solver_coefficients(), guidance_scale=7.5, extra=extra,
                    side_prompt_embeds=emb if side else None, control_image=ctrl, side_scale=0.8,
                    noise_fn=(lambda i: noise[i]) if noise is not None else None)
    assert torch.equal(got, again)


def test_loop_v1_sd15_512_dpmpp_2m_karras_20_steps():
    """SD-1.5-width v1 UNet, 512 x 512 (64 x 64 latents), one image x CFG, DPM-Solver++ 2M Karras, 20 steps"""
    from powerpaint_b200.denoise import FusedDenoiser

    nets = _nets(9, [("unet", 9, 1234)], tiny=False)
    om, pm, o = nets["unet"]
    g = torch.Generator(device=DEV).manual_seed(6)
    B, h, steps = 1, 64, 20
    sp = DPMSolverMultistepScheduler.from_config(DDIMScheduler().config, use_karras_sigmas=True)
    so = DPMSolverOracle(use_karras_sigmas=True)
    sp.set_timesteps(steps)
    so.set_timesteps(steps)
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g)
    emb = torch.randn(2 * B, 77, 768, device=DEV, generator=g) * 0.5
    extra = torch.cat([(torch.rand(B, 1, h, h, device=DEV, generator=g) > 0.5).float(),
                       torch.randn(B, 4, h, h, device=DEV, generator=g)], 1)
    so.sigmas = so.sigmas.float().to(DEV)
    so.timesteps = so.timesteps.to(DEV)
    ref = _oracle_loop("v1", om, None, so, lat, emb, extra, None, 7.5, 1.0, None)
    got = FusedDenoiser(pm).run(latents=lat, prompt_embeds=emb, timesteps=sp.timesteps, coef=sp.step_coefficients(),
                                scoef=sp.solver_coefficients(), guidance_scale=7.5, extra=extra)
    assert torch.isfinite(got).all()
    assert _rel(got, ref) < 5e-2 and _cos(got, ref) > 0.999, (_rel(got, ref), _cos(got, ref))


def test_pipeline_v1_seeded_call_is_deterministic():
    """the public `__call__` with Euler ancestral (noise path) and a seeded generator: two calls, identical latents"""
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline

    nets = _nets(9, [("unet", 9, 1234)])
    _, pm, o = nets["unet"]
    pipe = StableDiffusionInpaintPipeline(vae=AutoencoderKLOracle.synthetic(tiny=True).to(DEV), text_encoder=None,
                                          tokenizer=None, unet=pm, safety_checker=None,
                                          scheduler=EulerAncestralDiscreteScheduler.from_config(DDIMScheduler().config))
    g = torch.Generator().manual_seed(1)
    img = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    mask = (torch.rand(1, 1, 64, 64, generator=g) > 0.5).float()
    pe = (torch.randn(1, 77, o.cross_attention_dim, generator=g) * 0.5).to(DEV)
    outs = [pipe(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=pe * 0.5, height=64, width=64,
                 num_inference_steps=6, generator=torch.Generator().manual_seed(3), output_type="latent",
                 return_dict=False)[0] for _ in range(2)]
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
