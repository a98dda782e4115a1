"""CPU tests of DPMSolverMultistepScheduler, EulerDiscreteScheduler and EulerAncestralDiscreteScheduler: the folded
rows `pp_solver_step` applies against the stepwise float64 oracles (oracle/dpmsolver.py, oracle/euler.py), known
answers of the schedules, orders of accuracy on the closed-form Gaussian problem, the config surface, and the host
side of the pipelines' `__call__` against the reference's own `__call__` (tests/golden/pipeline_solver_call.npz)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle.dpmsolver import DPMSolverOracle
from oracle.euler import EulerAncestralOracle, EulerOracle
from powerpaint_b200.schedulers import (DDIMScheduler, DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                        EulerDiscreteScheduler, UniPCMultistepScheduler)
from test_scheduler import _gaussian_denoiser_eps

HERE = os.path.dirname(os.path.abspath(__file__))

DPM_CONFIGS = [dict(algorithm_type=a, solver_order=o, solver_type=t, final_sigmas_type=f, use_karras_sigmas=k)
               for a in ("dpmsolver++", "sde-dpmsolver++") for o in (1, 2) for t in ("midpoint", "heun")
               for f in ("zero", "sigma_min") for k in (False, True) if not (o == 1 and t == "heun")]
DPM_CONFIGS += [dict(euler_at_final=True, final_sigmas_type="sigma_min"),
                dict(lower_order_final=False, final_sigmas_type="sigma_min")]
EULER_CONFIGS = [dict(use_karras_sigmas=k) for k in (False, True)]
SPACINGS = [dict(timestep_spacing="leading", steps_offset=1), dict(timestep_spacing="linspace", steps_offset=0),
            dict(timestep_spacing="trailing", steps_offset=0)]


def _pair(family, cfg, spacing):
    sd = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    if family == "dpm":
        return DPMSolverOracle(**sd, **cfg, **spacing), DPMSolverMultistepScheduler(**sd, **cfg, **spacing)
    if family == "euler":
        return EulerOracle(**sd, **cfg, **spacing), EulerDiscreteScheduler(**sd, **cfg, **spacing)
    return EulerAncestralOracle(**sd, **cfg, **spacing), EulerAncestralDiscreteScheduler(**sd, **cfg, **spacing)


def _apply(r, x, m1, eps, noise):
    """the row formula of pp_solver_step (include/powerpaint_b200.h)"""
    mt = r[0] * x + r[1] * eps
    return r[2] * x + r[3] * mt + r[4] * m1 + r[5] * noise, mt


def _cases():
    for fam, cfgs in (("dpm", DPM_CONFIGS), ("euler", EULER_CONFIGS), ("euler_a", EULER_CONFIGS)):
        for cfg in cfgs:
            for spacing in SPACINGS:
                yield fam, cfg, spacing


def test_folded_rows_equal_the_stepwise_oracle_for_every_accepted_configuration():
    """5 / 10 / 25 / 50 steps (crossing lower_order_final's 15-step switch), full and strength < 1 starts, random
    tensors, float64: the folded rows reproduce the oracle step by step (same noise for the stochastic variants)"""
    checked = 0
    for fam, cfg, spacing in _cases():
        for n in (5, 10, 25, 50):
            for frac in (1.0, 0.6):
                o, s = _pair(fam, cfg, spacing)
                o.set_timesteps(n)
                s.set_timesteps(n)
                assert np.allclose(o.timesteps.double().numpy(), s.timesteps.double().numpy()), (fam, cfg, spacing)
                first = n - int(n * frac)
                rows = s.solver_coefficients(first=first).double()
                assert rows.shape == (n - first, 8)
                g = torch.Generator().manual_seed(n + first)
                x = torch.randn(2, 4, 4, 4, generator=g, dtype=torch.float64) * 3
                xo, xs, m1 = x.clone(), x.clone(), torch.zeros_like(x)
                for i, t in enumerate(o.timesteps[first:]):
                    eps = torch.randn(2, 4, 4, 4, generator=g, dtype=torch.float64)
                    nz = torch.randn(2, 4, 4, 4, generator=g, dtype=torch.float64)
                    xo = o.step(eps, t, xo, variance_noise=nz)
                    xs, m1 = _apply(rows[i], xs, m1, eps, nz)
                    # the next step's input scale (column 6) is the scale_model_input factor of the next row (column 7)
                    if i + 1 < len(rows):
                        assert abs(float(rows[i, 6] - rows[i + 1, 7])) < 1e-7
                assert torch.isfinite(xs).all()
                if not torch.isfinite(xo).all():
                    # heun over a zero-length last step (Karras sigmas end at sigma_min, repeated by final_sigmas_type
                    # sigma_min): the restated update divides 0 by 0, the folded row is the identity
                    assert cfg.get("solver_type") == "heun" and cfg["use_karras_sigmas"] and n >= 15
                    continue
                rel = ((xs - xo).norm() / xo.norm()).item()
                assert rel < 1e-5, (fam, cfg, spacing, n, first, rel)
                checked += 1
    assert checked > 0.9 * (len(DPM_CONFIGS) + 2 * len(EULER_CONFIGS)) * len(SPACINGS) * 8


def test_known_answers():
    s = EulerDiscreteScheduler.from_config(DDIMScheduler().config)
    s.set_timesteps(50)
    assert float(s.timesteps[0]) == 981.0 and float(s.timesteps[-1]) == 1.0 and s.timesteps.dtype == torch.float32
    ac = s.alphas_cumprod.double()
    assert abs(s.sigmas[0] - math.sqrt((1 - ac[981]) / ac[981])) < 1e-5 and s.sigmas[-1] == 0.0
    # init_noise_sigma: sqrt(sigma_max^2 + 1) for leading spacing, sigma_max for linspace / trailing
    assert abs(s.init_noise_sigma - math.sqrt(s.sigmas[0] ** 2 + 1)) < 1e-9
    for spacing in ("linspace", "trailing"):
        e = EulerDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                                   timestep_spacing=spacing)
        e.set_timesteps(30)
        assert float(e.timesteps[0]) == 999.0 and e.init_noise_sigma == float(e.sigmas.max())
        assert abs(e.init_noise_sigma - math.sqrt((1 - ac[999]) / ac[999])) < 1e-4
    d = DPMSolverMultistepScheduler.from_config(DDIMScheduler().config)
    d.set_timesteps(20)
    assert d.init_noise_sigma == 1.0 and d.timesteps.tolist()[:2] == [941, 894] and int(d.timesteps[-1]) == 48
    assert d.sigmas[-1] == 0.0
    # Karras sigmas: the closed form with rho = 7 between the training schedule's extremes
    for n in (5, 20):
        k = DPMSolverMultistepScheduler.from_config(DDIMScheduler().config, use_karras_sigmas=True)
        k.set_timesteps(n)
        smin, smax = math.sqrt((1 - ac[0]) / ac[0]), math.sqrt((1 - ac[999]) / ac[999])
        want = [(smax ** (1 / 7) + i / (n - 1) * (smin ** (1 / 7) - smax ** (1 / 7))) ** 7 for i in range(n)]
        assert np.allclose(k.sigmas[:-1], want, rtol=1e-5), (k.sigmas, want)
        assert int(k.timesteps[0]) == 999 and int(k.timesteps[-1]) == 0
        ek = EulerDiscreteScheduler.from_config(DDIMScheduler().config, use_karras_sigmas=True)
        ek.set_timesteps(n)
        lo, hi = ek._train_sigmas[1], ek._train_sigmas[951 if n == 20 else 801]  # the spaced schedule's extremes
        want = [(hi ** (1 / 7) + i / (n - 1) * (lo ** (1 / 7) - hi ** (1 / 7))) ** 7 for i in range(n)]
        assert np.allclose(ek.sigmas[:-1], want, rtol=1e-5)
        assert any(float(t) != round(float(t)) for t in ek.timesteps)  # fractional timesteps stay unrounded


# ----------------------------------------------------------------------------------- orders of accuracy
S2 = 0.25
X_INIT = torch.tensor([1.3, -0.7, 0.2], dtype=torch.float64)


def _alpha_sigma(row):
    """(alpha, sigma) of the row's own step from m = r0 x + r1 eps (VP: 1 / alpha, -sigma / alpha; VE: 1, -s)"""
    return 1.0 / float(row[0]), -float(row[1]) / float(row[0])


def _product_error(sched, n, k, rows_hook=None):
    sched.set_timesteps(n)
    assert int(round(float(sched.timesteps[k]))) == 199
    rows = sched.solver_coefficients().double()
    if rows_hook is not None:
        rows = rows_hook(rows)
    x, m1 = X_INIT.clone(), torch.zeros(3, dtype=torch.float64)
    for i in range(k):
        a, s = _alpha_sigma(rows[i])
        x, m1 = _apply(rows[i], x, m1, _gaussian_denoiser_eps(x, a, s, S2), 0.0)
    a0, s0 = _alpha_sigma(rows[0])
    a1, s1 = _alpha_sigma(rows[k])
    ref = X_INIT * math.sqrt(a1 * a1 * S2 + s1 * s1) / math.sqrt(a0 * a0 * S2 + s0 * s0)
    return ((x - ref).norm() / ref.norm()).item()


def _oracle_error(o, n, k):
    o.set_timesteps(n)
    vp = isinstance(o, DPMSolverOracle)

    def a_s(i):
        sg = float(o.sigmas[i])
        return (1 / math.sqrt(sg * sg + 1), sg / math.sqrt(sg * sg + 1)) if vp else (1.0, sg)

    x = X_INIT.clone()
    for i in range(k):
        a, s = a_s(i)
        x = o.step(_gaussian_denoiser_eps(x, a, s, S2), o.timesteps[i], x, variance_noise=torch.zeros(3))
    a0, s0 = a_s(0)
    a1, s1 = a_s(k)
    ref = X_INIT * math.sqrt(a1 * a1 * S2 + s1 * s1) / math.sqrt(a0 * a0 * S2 + s0 * s0)
    return ((x - ref).norm() / ref.norm()).item()


GRID = [(10, 8), (20, 16), (40, 32)]  # trailing spacing: steps of 100 / 50 / 25 from t = 999 down to t = 199
SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", timestep_spacing="trailing")


def _orders(errs):
    return [math.log2(errs[i] / errs[i + 1]) for i in range(len(errs) - 1)]


def test_orders_of_accuracy_on_the_closed_form_gaussian_flow():
    """data ~ N(0, s^2): the probability-flow ODE is exact and the optimal denoiser linear (test_scheduler.py), so the
    global error is measurable exactly. DPM-Solver++ 1 and Euler are first order, DPM-Solver++ 2M (midpoint, heun)
    second order — for the folded rows and the stepwise oracle alike; a wrong h, r or alpha_t factor drops it."""
    cases = {"dpm1": (dict(solver_order=1), (0.8, 1.3)), "dpm2_mid": (dict(solver_type="midpoint"), (1.7, 2.4)),
             "dpm2_heun": (dict(solver_type="heun"), (1.7, 2.4))}
    for name, (cfg, (lo, hi)) in cases.items():
        ep = [_product_error(DPMSolverMultistepScheduler(**SD, **cfg), n, k) for n, k in GRID]
        eo = [_oracle_error(DPMSolverOracle(**SD, **cfg), n, k) for n, k in GRID]
        assert all(lo < o < hi for o in _orders(ep)), (name, ep, _orders(ep))
        assert all(lo < o < hi for o in _orders(eo)), (name, eo, _orders(eo))
        assert all(abs(a - b) <= 1e-3 * b for a, b in zip(ep, eo)), (ep, eo)
    ee = [_product_error(EulerDiscreteScheduler(**SD), n, k) for n, k in GRID]
    eo = [_oracle_error(EulerOracle(**SD), n, k) for n, k in GRID]
    assert all(0.8 < o < 1.3 for o in _orders(ee)) and all(0.8 < o < 1.3 for o in _orders(eo)), (ee, eo)

    # wrong factors: r (the step ratio h_0 / h) off by 10 %, h off by 10 %, alpha_t dropped from the D1 term
    def wrong_r(rows):
        rows = rows.clone()
        d = 0.1 * rows[:, 4]
        rows[:, 3] += d
        rows[:, 4] -= d
        return rows

    def wrong_h(rows):
        rows = rows.clone()
        rows[1:, 3] *= 1.1
        return rows

    def wrong_alpha(rows):
        rows = rows.clone()
        s = rows[:, 0].clone()  # 1 / alpha_s: a D1 coefficient in alpha_s rather than alpha_t
        rows[:, 3] += rows[:, 4] * (s - 1)
        rows[:, 4] *= s
        return rows

    for hook in (wrong_r, wrong_h, wrong_alpha):
        ew = [_product_error(DPMSolverMultistepScheduler(**SD), n, k, hook) for n, k in GRID]
        assert min(_orders(ew)) < 1.4, (hook.__name__, ew, _orders(ew))


def _stochastic_variance_error(make_product, make_oracle, n, k):
    """|Var(x_k) - (alpha_k^2 s^2 + sigma_k^2)| / target for the folded rows (x, m1 recursion) and for the oracle.
    Exact: every tensor is a vector of coefficients on (x_T, noise_0, noise_1, ...), independent normals of variance
    (Var_T, 1, 1, ...), so Var(x_k) is the scaled sum of squares of x_k's coefficients"""
    s = make_product()
    s.set_timesteps(n)
    rows = s.solver_coefficients().double()
    a0, s0 = _alpha_sigma(rows[0])
    var_t = a0 * a0 * S2 + s0 * s0
    dim = 1 + k
    scale = torch.ones(dim, dtype=torch.float64)
    scale[0] = math.sqrt(var_t)

    def unit(j):
        e = torch.zeros(dim, dtype=torch.float64)
        e[j] = 1.0
        return e

    x0 = unit(0)
    x, m1 = x0.clone(), torch.zeros(dim, dtype=torch.float64)
    for i in range(k):
        a, sg = _alpha_sigma(rows[i])
        x, m1 = _apply(rows[i], x, m1, _gaussian_denoiser_eps(x, a, sg, S2), unit(1 + i))
    a1, s1 = _alpha_sigma(rows[k])
    target = a1 * a1 * S2 + s1 * s1
    err_p = abs(float(((x * scale) ** 2).sum()) - target) / target
    o = make_oracle()
    o.set_timesteps(n)
    xo = x0.clone()
    for i in range(k):
        a, sg = _alpha_sigma(rows[i])
        xo = o.step(_gaussian_denoiser_eps(xo, a, sg, S2), o.timesteps[i], xo, variance_noise=unit(1 + i))
    err_o = abs(float(((xo * scale) ** 2).sum()) - target) / target
    return err_p, err_o


def test_stochastic_variants_converge_in_distribution():
    """SDE-DPM-Solver++ and Euler ancestral with the linear (Gaussian-data) denoiser: the state is updated linearly plus
    Gaussian noise, so Var(x_k) follows an exact recursion (no sampling) and must converge to alpha^2 s^2 + sigma^2,
    with at least first order for SDE-DPM++ 1 and Euler ancestral (measured 0.955, 0.977 on this grid; the two give the
    same variances). For SDE-DPM++ 2M (midpoint) the float64 oracle recursion converges with second order (measured
    1.949, 1.965), and the folded rows match it. The grid is one halving finer than the ODE tests': on the coarser one
    the first-order schemes are still in the pre-asymptotic range (0.906, 0.955)."""
    sde = dict(algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min")
    cases = {
        "sde1": (lambda: DPMSolverMultistepScheduler(**SD, **sde, solver_order=1),
                 lambda: DPMSolverOracle(**SD, **sde, solver_order=1), 0.9),
        "euler_a": (lambda: EulerAncestralDiscreteScheduler(**SD), lambda: EulerAncestralOracle(**SD), 0.9),
        "sde2": (lambda: DPMSolverMultistepScheduler(**SD, **sde), lambda: DPMSolverOracle(**SD, **sde), 1.8),
    }
    for name, (mp, mo, min_order) in cases.items():
        errs = [_stochastic_variance_error(mp, mo, n, k) for n, k in ((20, 16), (40, 32), (80, 64))]
        ep, eo = [e[0] for e in errs], [e[1] for e in errs]
        assert all(o > min_order for o in _orders(ep)), (name, ep, _orders(ep))
        assert all(o > min_order for o in _orders(eo)), (name, eo, _orders(eo))
        assert all(abs(a - b) <= 1e-3 * b + 1e-12 for a, b in zip(ep, eo)), (name, ep, eo)


# ----------------------------------------------------------------------------------- config surface
def test_config_surface(tmp_path):
    ddim, unipc = DDIMScheduler(), UniPCMultistepScheduler.from_config(DDIMScheduler().config)
    for cls in (DPMSolverMultistepScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler):
        for base in (ddim, unipc):
            s = cls.from_config(base.config)  # the app's swap-by-config pattern; foreign keys are dropped
            assert s.config.timestep_spacing == "leading" and s.config.steps_offset == 1 and s.kind == "solver"
            assert "clip_sample" not in s.config and "predict_x0" not in s.config
            assert torch.equal(s.alphas_cumprod, ddim.alphas_cumprod)
        s = cls.from_config(ddim.config, use_karras_sigmas=True)
        s.save_pretrained(str(tmp_path / cls.__name__))
        s2 = cls.from_pretrained(str(tmp_path / cls.__name__))
        assert vars(s2.config) == vars(s.config)
        s.set_timesteps(12)
        s2.set_timesteps(12)
        assert torch.equal(s.timesteps, s2.timesteps) and torch.equal(s.solver_coefficients(), s2.solver_coefficients())
        with pytest.raises(NotImplementedError, match="prediction_type"):
            cls(prediction_type="v_prediction")
        with pytest.raises(NotImplementedError, match="timestep_spacing"):
            cls(timestep_spacing="karras")
        with pytest.raises(RuntimeError):  # CPU tensors: there is no CPU step
            s.step(torch.zeros(1, 4, 8, 8), s.timesteps[0], torch.zeros(1, 4, 8, 8))
    assert DPMSolverMultistepScheduler.from_config(unipc.config).config.solver_type == "midpoint"  # bh2 -> midpoint
    for kw, key in ((dict(algorithm_type="dpmsolver"), "algorithm_type"),
                    (dict(algorithm_type="sde-dpmsolver"), "algorithm_type"), (dict(solver_order=3), "solver_order"),
                    (dict(use_lu_lambdas=True), "use_lu_lambdas"), (dict(thresholding=True), "thresholding"),
                    (dict(solver_type="euler"), "solver_type"), (dict(final_sigmas_type="denoise_to_zero"),
                                                                 "final_sigmas_type"),
                    (dict(variance_type="learned_range"), "variance_type")):
        with pytest.raises(NotImplementedError, match=key):
            DPMSolverMultistepScheduler(**kw)
    for cls in (EulerDiscreteScheduler, EulerAncestralDiscreteScheduler):
        for kw, key in ((dict(interpolation_type="log_linear"), "interpolation_type"),
                        (dict(timestep_type="continuous"), "timestep_type")):
            with pytest.raises(NotImplementedError, match=key):
                cls(**kw)
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(use_karras_sigmas=True)  # UniPC's own restrictions stay
    # scale_model_input / add_noise: VE for Euler, VP for DPM-Solver++
    e = EulerDiscreteScheduler.from_config(ddim.config)
    e.set_timesteps(10)
    x = torch.ones(1, 4, 2, 2)
    assert torch.allclose(e.scale_model_input(x, e.timesteps[3]), x / math.sqrt(e.sigmas[3] ** 2 + 1))
    assert torch.allclose(e.add_noise(x, x, e.timesteps[2:3]), x * (1 + e.sigmas[2]))
    d = DPMSolverMultistepScheduler.from_config(ddim.config)
    d.set_timesteps(10)
    a = 1 / math.sqrt(d.sigmas[2] ** 2 + 1)
    assert torch.equal(d.scale_model_input(x, d.timesteps[3]), x)
    assert torch.allclose(d.add_noise(x, x, d.timesteps[2:3]), x * (a + d.sigmas[2] * a))


def test_pipeline_directory_loads_the_stored_solver_class(tmp_path):
    """scheduler_config.json storing one of the new classes builds it; PNDM still falls back to DDIM with a warning"""
    import json

    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline as P

    base = {k: v for k, v in vars(DDIMScheduler().config).items()}
    for cls in (DPMSolverMultistepScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler, None):
        name = cls.__name__ if cls else "PNDMScheduler"
        d = tmp_path / name
        d.mkdir()
        cfg = dict(base, _class_name=name, use_karras_sigmas=True)
        (d / "scheduler_config.json").write_text(json.dumps(cfg))
        if cls is None:
            with pytest.warns(UserWarning, match="PNDMScheduler is replaced by DDIMScheduler"):
                s = P._load_component("scheduler", str(d), ["diffusers", name], None, None)
            assert type(s) is DDIMScheduler
        else:
            s = P._load_component("scheduler", str(d), ["diffusers", name], None, None)
            assert type(s) is cls and s.config.use_karras_sigmas and s.config.steps_offset == 1


# ----------------------------------------------------------------------------------- host side of __call__
class _SolverDenoiser:
    """what FusedDenoiser.run computes with `scoef`, in fp32 torch on the CPU (test stand-in only): the input scale of
    step i is row i column 7, the noise of a stochastic step comes from noise_fn(i)"""

    def __init__(self, unet, brushnet=None):
        self.unet, self.brushnet = unet, brushnet

    @torch.no_grad()
    def run(self, *, latents, prompt_embeds, timesteps, coef, guidance_scale, extra, noise_fn=None, callback=None,
            ucoef=None, scoef=None, blend=None, side_prompt_embeds=None, side_scale=1.0, side_keep=None):
        assert ucoef is None and blend is None and scoef is not None and len(scoef) == len(timesteps)
        do_cfg = guidance_scale > 1.0
        m1 = torch.zeros_like(latents)
        for i, t in enumerate(timesteps):
            r = [float(v) for v in scoef[i]]
            xin = latents * r[7]
            if self.brushnet is None:
                x = torch.cat([torch.cat([xin] * 2) if do_cfg else xin, torch.cat([extra] * 2) if do_cfg else extra], 1)
                eps = self.unet(x, int(t), prompt_embeds)
            else:
                x = torch.cat([xin] * 2) if do_cfg else xin
                d, m, u = self.brushnet(x, int(t), side_prompt_embeds, extra,
                                        side_scale * (side_keep[i] if side_keep is not None else 1.0))
                eps = self.unet(x, int(t), prompt_embeds, down_block_add_samples=d, mid_block_add_sample=m,
                                up_block_add_samples=u)
            if do_cfg:
                u_, c_ = eps.chunk(2)
                eps = u_ + guidance_scale * (c_ - u_)
            noise = noise_fn(i) if noise_fn is not None else 0.0
            latents, m1 = _apply(r, latents, m1, eps, noise)
        return latents


def _solver(name):
    import sys

    sys.path.insert(0, os.path.join(HERE, "golden"))
    base = DDIMScheduler().config
    return {"dpmpp_2m_karras": lambda: DPMSolverMultistepScheduler.from_config(base, use_karras_sigmas=True),
            "sde_dpmpp_2m": lambda: DPMSolverMultistepScheduler.from_config(
                base, algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min"),
            "euler_a": lambda: EulerAncestralDiscreteScheduler.from_config(base)}[name]()


@pytest.mark.parametrize("name,sched,strength,steps", [
    ("v1_dpmpp_2m_karras", "dpmpp_2m_karras", 1.0, 5), ("v1_euler_a", "euler_a", 1.0, 4),
    ("v1_sde_dpmpp_2m_strength", "sde_dpmpp_2m", 0.5, 8), ("v1_euler_a_strength", "euler_a", 0.6, 5)])
def test_v1_call_with_solver_equals_reference_call_golden(name, sched, strength, steps):
    import test_pipeline_golden as G
    from oracle.unet import UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline

    gold = np.load(os.path.join(HERE, "golden", "pipeline_solver_call.npz"))
    om, sd = G._oracle(UNet2DConditionOracle, 9, "unet", 77)
    pipe = StableDiffusionInpaintPipeline(vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=None,
                                          tokenizer=None, unet=UNet2DConditionModel.from_state_dict(G._cfg(9), sd),
                                          scheduler=_solver(sched), safety_checker=None)
    fake = _SolverDenoiser(om)
    pipe.denoiser = lambda: fake
    img, mask, pe, ne = G._call_inputs()
    out = pipe(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=G.H, width=G.W,
               strength=strength, num_inference_steps=steps, guidance_scale=7.5, generator=G._generators(False),
               output_type="latent", return_dict=False)[0]
    ref = torch.from_numpy(gold[f"{name}_latents"])
    assert out.shape == ref.shape and G._rel(out, ref) < 5e-5, G._rel(out, ref)


@pytest.mark.parametrize("name,sched,steps", [("brushnet_dpmpp_2m_karras", "dpmpp_2m_karras", 4),
                                              ("brushnet_euler_a", "euler_a", 3)])
def test_brushnet_call_with_solver_equals_reference_call_golden(name, sched, steps):
    import test_pipeline_golden as G
    from oracle.unet import BrushNetOracle, UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import BrushNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionPowerPaintBrushNetPipeline

    gold = np.load(os.path.join(HERE, "golden", "pipeline_solver_call.npz"))
    ou, sd_u = G._oracle(UNet2DConditionOracle, 4, "unet", 11)
    ob, sd_b = G._oracle(BrushNetOracle, 4, "brushnet", 12)
    tok, te, te_b = G._text_stack()
    pipe = StableDiffusionPowerPaintBrushNetPipeline(
        vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=te, text_encoder_brushnet=te_b, tokenizer=tok,
        unet=UNet2DConditionModel.from_state_dict(G._cfg(4), sd_u),
        brushnet=BrushNetModel.from_state_dict(G._cfg(4), sd_b), scheduler=_solver(sched), safety_checker=None)
    fake = _SolverDenoiser(ou, ob)
    pipe.denoiser = lambda: fake
    img, mask = G._brushnet_inputs()
    torch.manual_seed(123)
    with torch.no_grad():
        out = pipe(**G.PROMPTS, tradoff=0.7, tradoff_nag=0.4, image=img, mask=mask, generator=G._generators(False),
                   num_inference_steps=steps, guidance_scale=7.5, brushnet_conditioning_scale=1.0,
                   output_type="latent", return_dict=False)[0]
    ref = torch.from_numpy(gold[f"{name}_latents"])
    assert out.shape == ref.shape and G._rel(out, ref) < 5e-5, G._rel(out, ref)
