"""CPU tests of PNDMScheduler with skip_prk_steps (PLMS): known answers of its N + 1 timesteps, the folded rows
`pp_plms_step` applies against the stepwise float64 oracle (oracle/pndm.py), second order of accuracy on the
closed-form Gaussian problem, the config surface and refusals, the new descriptor's layout, and the host side of the
three pipelines' `__call__` against the reference's own `__call__` (tests/golden/pipeline_pndm_call.npz)."""
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle.pndm import PNDMOracle
from powerpaint_b200.schedulers import DDIMScheduler, PNDMScheduler, _PlmsFold
from test_scheduler import _gaussian_denoiser_eps

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", skip_prk_steps=True,
          set_alpha_to_one=False, steps_offset=1)  # the SD-1.5 inpainting checkpoint's scheduler_config.json
SPACINGS = [dict(timestep_spacing="leading", steps_offset=1), dict(timestep_spacing="linspace", steps_offset=0),
            dict(timestep_spacing="trailing", steps_offset=0)]


def _pair(spacing=None, **kw):
    cfg = dict(SD, **(spacing or {}), **kw)
    oracle_cfg = {k: v for k, v in cfg.items() if k != "skip_prk_steps"}
    return PNDMOracle(**oracle_cfg), PNDMScheduler(**cfg)


def _apply(r, x, cur, ets, eps):
    """the row formula of pp_plms_step (include/powerpaint_b200.h); returns (x_next, cur, ets)"""
    r = [float(v) for v in r]
    xn = r[0] * x + r[1] * cur + r[2] * eps + r[3] * ets[0] + r[4] * ets[1] + r[5] * ets[2]
    ets = list(ets)
    if r[7] != 0:
        cur = x
    if r[6] >= 0:
        ets[int(r[6])] = eps
    return xn, cur, ets


def _run_rows(rows, x, eps_fn):
    cur, ets = torch.zeros_like(x), [torch.zeros_like(x)] * 3
    for i, r in enumerate(rows):
        x, cur, ets = _apply(r, x, cur, ets, eps_fn(i, x))
    return x


# ----------------------------------------------------------------------------------- timesteps
def test_timestep_known_answers():
    s = PNDMScheduler(**SD)
    s.set_timesteps(50)
    ts = s.timesteps.tolist()
    assert len(ts) == 51 and ts[:4] == [981, 961, 961, 941] and ts[-1] == 1 and s.timesteps.dtype == torch.int64
    assert ts[3:] == list(range(941, 0, -20)) and s.num_inference_steps == 50
    s.set_timesteps(10)
    assert s.timesteps.tolist() == [901, 801, 801, 701, 601, 501, 401, 301, 201, 101, 1]
    lin = PNDMScheduler(**dict(SD, timestep_spacing="linspace", steps_offset=0))
    lin.set_timesteps(10)
    assert lin.timesteps.tolist() == [999, 888, 888, 777, 666, 555, 444, 333, 222, 111, 0]
    tr = PNDMScheduler(**dict(SD, timestep_spacing="trailing", steps_offset=0))
    tr.set_timesteps(10)
    assert tr.timesteps.tolist() == [999, 899, 899, 799, 699, 599, 499, 399, 299, 199, 99]
    for spacing in SPACINGS:
        for n in (1, 2, 7, 25, 50):
            o, p = _pair(spacing)
            o.set_timesteps(n)
            p.set_timesteps(n)
            assert torch.equal(o.timesteps, p.timesteps), (spacing, n)
            assert len(p.timesteps) == (n + 1 if n > 1 else 1)
    # strength < 1 slices the N + 1 entries (get_timesteps, ref:pipeline_PowerPaint.py:855-860)
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline as P

    pipe = P.__new__(P)
    pipe.scheduler = PNDMScheduler(**SD)
    for n, strength, want in ((5, 0.6, [601, 401, 201, 1]), (5, 0.8, [601, 601, 401, 201, 1]), (10, 0.5, [501, 401, 301,
                                                                                                     201, 101, 1])):
        pipe.scheduler.set_timesteps(n)
        ts, steps = pipe.get_timesteps(n, strength, "cpu")
        assert ts.tolist() == want and len(ts) - steps == 1, (n, strength, ts, steps)
    assert pipe.scheduler.init_noise_sigma == 1.0 and pipe.scheduler.order == 1
    x = torch.randn(1, 4, 2, 2)
    assert pipe.scheduler.scale_model_input(x, 981) is x


# ----------------------------------------------------------------------------------- folded rows
def test_folded_rows_equal_the_stepwise_oracle():
    """float64, random eps sequences, every spacing, full runs and strength suffixes (including a slice that starts
    at the repeated timestep, where the Heun restart steps back up by one ratio): relative error <= 1e-6"""
    checked = 0
    for spacing in SPACINGS:
        for n in (1, 2, 3, 4, 5, 10, 50):
            for first in sorted({0, 1, 2, 3, n // 2}):
                o, p = _pair(spacing)
                o.set_timesteps(n)
                p.set_timesteps(n)
                if first >= len(p.timesteps):
                    continue
                rows = p.plms_coefficients(first=first, dtype=torch.float64)
                assert rows.shape == (len(p.timesteps) - first, 8)
                g = torch.Generator().manual_seed(100 * n + first)
                x = torch.randn(2, 4, 3, 5, generator=g, dtype=torch.float64) * 2
                eps = [torch.randn(2, 4, 3, 5, generator=g, dtype=torch.float64) for _ in range(len(rows))]
                xo = x.clone()
                for i, t in enumerate(o.timesteps[first:]):
                    xo = o.step(eps[i], t, xo)
                xs = _run_rows(rows, x.clone(), lambda i, _x: eps[i])
                rel = ((xs - xo).norm() / xo.norm()).item()
                assert rel <= 1e-6, (spacing, n, first, rel)
                checked += 1
    assert checked >= 60
    # the fp32 table the kernel reads holds the same rows; slot indices and flags are exact
    p = PNDMScheduler(**SD)
    p.set_timesteps(50)
    r32, r64 = p.plms_coefficients(), p.plms_coefficients(dtype=torch.float64)
    assert r32.dtype == torch.float32 and torch.allclose(r32.double(), r64, rtol=1e-7, atol=0)
    assert r32[:, 6].tolist()[:6] == [0, -1, 1, 2, 0, 1] and r32[:, 7].tolist()[:3] == [1, 0, 0]
    assert r32[1, 0] == 0 and r32[1, 1] != 0 and (r32[2:, 1] == 0).all()  # counter 1 restarts from cur_sample


def test_row_structure_of_each_counter():
    """the weights of each row type: m = eps (counter 0), (eps + e0) / 2 from cur_sample (counter 1), then
    Adams-Bashforth 2 / 3 / 4 on the ring, the newest remembered eps first"""
    p = PNDMScheduler(**SD)
    p.set_timesteps(50)
    rows = p.plms_coefficients(dtype=torch.float64)
    for i, ab in ((0, [1.0]), (1, [0.5, 0.5]), (2, [3 / 2, -1 / 2]), (3, [23 / 12, -16 / 12, 5 / 12]),
                  (4, [55 / 24, -59 / 24, 37 / 24, -9 / 24]), (7, [55 / 24, -59 / 24, 37 / 24, -9 / 24])):
        r = rows[i]
        k = -float(r[2]) / ab[0]
        newest = {1: [0], 2: [0], 3: [1, 0], 4: [2, 1, 0], 7: [2, 1, 0]}.get(i, [])  # slots, newest first
        got = [float(r[3 + s]) for s in newest]
        assert np.allclose(got, [-k * w for w in ab[1:]], rtol=1e-12), (i, got)
        assert sum(float(r[3 + s]) != 0 for s in range(3)) == len(ab) - 1


# ----------------------------------------------------------------------------------- order of accuracy
S2 = 0.25
X_INIT = torch.tensor([1.3, -0.7, 0.2], dtype=torch.float64)
STOP = 201


def _ac(sched):
    return sched.alphas_cumprod.double()


def _ref(ac, t0):
    a0, s0 = math.sqrt(ac[t0]), math.sqrt(1 - ac[t0])
    a1, s1 = math.sqrt(ac[STOP]), math.sqrt(1 - ac[STOP])
    return X_INIT * math.sqrt(a1 * a1 * S2 + s1 * s1) / math.sqrt(a0 * a0 * S2 + s0 * s0)


def _eps(ac, t, x):
    return _gaussian_denoiser_eps(x, math.sqrt(ac[t]), math.sqrt(1 - ac[t]), S2)


def _stop_index(ts, ratio):
    """the row whose step ends at t = STOP (counter >= 2: the first two rows end at the same timestep)"""
    return next(i for i in range(2, len(ts)) if int(ts[i]) - ratio == STOP)


def _product_error(n):
    p = PNDMScheduler(**SD)
    p.set_timesteps(n)
    ts, ac = p.timesteps, _ac(p)
    k = _stop_index(ts, 1000 // n)
    rows = p.plms_coefficients(dtype=torch.float64)[:k + 1]
    x = _run_rows(rows, X_INIT.clone(), lambda i, x: _eps(ac, int(ts[i]), x))
    ref = _ref(ac, int(ts[0]))
    return ((x - ref).norm() / ref.norm()).item()


def _oracle_error(n):
    o, _ = _pair()
    o.set_timesteps(n)
    ts, ac = o.timesteps, o.alphas_cumprod.double()
    x = X_INIT.clone()
    for i in range(_stop_index(ts, 1000 // n) + 1):
        x = o.step(_eps(ac, int(ts[i]), x), ts[i], x)
    ref = _ref(ac, int(ts[0]))
    return ((x - ref).norm() / ref.norm()).item()


def _orders(errs):
    return [math.log2(errs[i] / errs[i + 1]) for i in range(len(errs) - 1)]


def test_plms_is_second_order_on_the_closed_form_gaussian_flow():
    """data ~ N(0, s^2) (test_scheduler.py): the probability-flow ODE has a closed form and the optimal denoiser is
    linear, so the global error at t = 201 is exact to measure. N = 50 / 100 / 200 leading steps: PLMS converges with
    second order (an fp64 restatement measured 6.8e-5, 1.8e-5, 4.7e-6), the folded rows and the oracle alike; DDIM
    on the same grid is first order. A wrong Adams-Bashforth weight (-8 for -9) stops convergence."""
    grid = (50, 100, 200)
    ep = [_product_error(n) for n in grid]
    eo = [_oracle_error(n) for n in grid]
    for errs in (ep, eo):
        assert all(1.7 < o < 2.3 for o in _orders(errs)), (errs, _orders(errs))
        assert errs[-1] < 1e-5, errs
    assert all(abs(a - b) <= 1e-6 * b for a, b in zip(ep, eo)), (ep, eo)
    saved = dict(_PlmsFold.AB)
    try:
        _PlmsFold.AB[4] = (55 / 24, -59 / 24, 37 / 24, -8 / 24)
        bad = [_product_error(n) for n in grid]
    finally:
        _PlmsFold.AB.clear()
        _PlmsFold.AB.update(saved)
    assert max(_orders(bad)) < 0.5, (bad, _orders(bad))
    assert _product_error(50) == ep[0]


# ----------------------------------------------------------------------------------- config surface, ABI
def test_config_surface_and_refusals(tmp_path):
    with pytest.raises(NotImplementedError, match="skip_prk_steps"):
        PNDMScheduler()  # diffusers' default is the Runge-Kutta warm-up
    with pytest.raises(NotImplementedError, match="skip_prk_steps"):
        PNDMScheduler.from_config(DDIMScheduler().config)  # a config without the key gets that default
    with pytest.raises(NotImplementedError, match="prediction_type"):
        PNDMScheduler(skip_prk_steps=True, prediction_type="v_prediction")
    with pytest.raises(NotImplementedError, match="timestep_spacing"):
        PNDMScheduler(skip_prk_steps=True, timestep_spacing="karras")
    s = PNDMScheduler.from_config(DDIMScheduler().config, skip_prk_steps=True)
    assert s.kind == "plms" and s.config.steps_offset == 1 and s.config.timestep_spacing == "leading"
    assert "clip_sample" not in s.config and torch.equal(s.alphas_cumprod, DDIMScheduler().alphas_cumprod)
    assert set(vars(s.config)) == {"num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "trained_betas",
                                   "skip_prk_steps", "set_alpha_to_one", "prediction_type", "timestep_spacing",
                                   "steps_offset"}
    s.save_pretrained(str(tmp_path / "scheduler"))
    s2 = PNDMScheduler.from_pretrained(str(tmp_path), subfolder="scheduler")
    assert vars(s2.config) == vars(s.config)
    s.set_timesteps(12)
    s2.set_timesteps(12)
    assert torch.equal(s.timesteps, s2.timesteps) and torch.equal(s.plms_coefficients(), s2.plms_coefficients())
    x = torch.ones(1, 4, 2, 2)
    a = float(s.alphas_cumprod[s.timesteps[3]])
    assert torch.allclose(s.add_noise(x, 2 * x, s.timesteps[3:4]), x * (math.sqrt(a) + 2 * math.sqrt(1 - a)))
    with pytest.raises(RuntimeError):  # CPU tensors: there is no CPU step
        s.step(torch.zeros(1, 4, 8, 8), s.timesteps[0], torch.zeros(1, 4, 8, 8))
    # the pipelines' signature sniffing passes neither eta nor generator (PNDM's step takes neither)
    import inspect

    assert not {"eta", "generator"} & set(inspect.signature(s.step).parameters)
    # set_alpha_to_one selects the final alpha_bar of a step past t = 0
    one = PNDMScheduler(**dict(SD, set_alpha_to_one=True, timestep_spacing="linspace", steps_offset=0))
    zero = PNDMScheduler(**dict(SD, timestep_spacing="linspace", steps_offset=0))
    for sch in (one, zero):
        sch.set_timesteps(10)
    assert not torch.equal(one.plms_coefficients()[-1], zero.plms_coefficients()[-1])


def test_loading_keeps_the_ddim_fallback_and_names_the_opt_in(tmp_path):
    import json

    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline as P

    d = tmp_path / "scheduler"
    d.mkdir()
    cfg = dict(vars(DDIMScheduler().config), _class_name="PNDMScheduler", skip_prk_steps=True)
    (d / "scheduler_config.json").write_text(json.dumps(cfg))
    with pytest.warns(UserWarning, match="PNDMScheduler is replaced by DDIMScheduler") as w:
        s = P._load_component("scheduler", str(d), ["diffusers", "PNDMScheduler"], None, None)
    assert type(s) is DDIMScheduler and "PNDMScheduler.from_pretrained" in str(w[0].message)
    p = PNDMScheduler.from_pretrained(str(tmp_path), subfolder="scheduler")  # the opt-in
    assert p.config.skip_prk_steps and p.config.steps_offset == 1


def test_plms_descriptor_matches_the_header(tmp_path):
    import ctypes
    import shutil
    import subprocess

    from powerpaint_b200 import _native as N

    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    cls, cname = N.PlmsDesc, "pp_plms_desc"
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "powerpaint_b200.h"', 'int main(void) {',
             f'  printf("{cname} %zu\\n", sizeof({cname}));']
    lines += [f'  printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in cls._fields_]
    lines.append("  return 0; }")
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                        str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = dict(ln.split(" ", 1) for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                         check=True).stdout.splitlines())
    assert int(out[cname]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f"{cname}.{f}"]) == getattr(cls, f).offset, f
    assert "pp_plms_step" in N.EXPORTED_SYMBOLS and "pp_program_add_plms_step" in N.EXPORTED_SYMBOLS


def test_plms_kernel_waits_on_its_predecessor_grid():
    src = open(os.path.join(ROOT, "powerpaint_b200", "csrc", "elementwise.cu")).read()
    m = re.search(r"__global__ void plms_step_kernel\([^)]*\)\s*\{", src)
    assert m, "plms_step_kernel not found"
    body = src[m.end():]
    assert body.lstrip().startswith("pdl_wait();"), body[:80]


# ----------------------------------------------------------------------------------- host side of __call__
class _PlmsDenoiser:
    """what FusedDenoiser.run computes with `pcoef`, in fp32 torch on the CPU over the oracle nets (test stand-in
    only): the PLMS rows, the 4-channel blend, side nets with their per-step scale, and a callback that may replace
    the latents"""

    def __init__(self, unet, sides=(), mode="v1"):
        self.unet, self.sides, self.mode = unet, list(sides), mode

    @torch.no_grad()
    def run(self, *, latents, prompt_embeds, timesteps, coef, guidance_scale, extra=None, noise_fn=None,
            callback=None, ucoef=None, pcoef=None, blend=None, side_prompt_embeds=None, side_scale=1.0,
            side_keep=None, control_image=None):
        from oracle import side_nets as osn

        assert ucoef is None and noise_fn is None and pcoef is not None and len(pcoef) == len(timesteps)
        do_cfg = guidance_scale > 1.0
        cur, ets = torch.zeros_like(latents), [torch.zeros_like(latents)] * 3
        for i, t in enumerate(timesteps):
            x = torch.cat([latents] * 2) if do_cfg else latents
            scale = side_scale * (side_keep[i] if side_keep is not None else 1.0)
            if self.mode == "v1":
                eps = self.unet(torch.cat([x, torch.cat([extra] * 2) if do_cfg else extra], 1) if extra is not None
                                else x, int(t), prompt_embeds)
            elif self.mode == "controlnet":
                d, m = osn.multi_controlnet(self.sides, (False,), x, int(t), side_prompt_embeds, [control_image],
                                            [scale], False)
                eps = self.unet(torch.cat([x, torch.cat([extra] * 2) if do_cfg else extra], 1), int(t),
                                prompt_embeds, down_block_additional_residuals=d, mid_block_additional_residual=m)
            else:
                d, m, u = self.sides[0](x, int(t), side_prompt_embeds, extra, scale)
                eps = self.unet(x, int(t), prompt_embeds, down_block_add_samples=d, mid_block_add_sample=m,
                                up_block_add_samples=u)
            if do_cfg:
                a, c = eps.chunk(2)
                eps = a + guidance_scale * (c - a)
            latents, cur, ets = _apply(pcoef[i], latents, cur, ets, eps)
            if blend is not None:
                sa = float(blend["sqrt_alpha"][i])
                known = sa * blend["x0"][:1] + math.sqrt(max(1 - sa * sa, 0.0)) * blend["noise"]
                latents = (1 - blend["mask"][:1]) * known + blend["mask"][:1] * latents
            if callback is not None:
                new = callback(i, t, latents)
                if new is not None:
                    latents = new
        return latents


def _gold(key):
    return np.load(os.path.join(HERE, "golden", "pipeline_pndm_call.npz"))[key]


def _sched():
    return PNDMScheduler.from_config(DDIMScheduler().config, skip_prk_steps=True)


def _check(out, seen, name):
    import test_pipeline_golden as G

    ref = torch.from_numpy(_gold(f"{name}_latents"))
    assert out.shape == ref.shape and G._rel(out, ref) < 5e-5, (name, G._rel(out, ref))
    assert seen == [tuple(v) for v in _gold(f"{name}_callback").tolist()], (name, seen)


@pytest.mark.parametrize("name,cin,strength,steps", [
    ("v1_full", 9, 1.0, 4), ("v1_strength", 9, 0.6, 5), ("v1_strength_restart", 9, 0.8, 5),
    ("v1_unet4", 4, 1.0, 4), ("v1_unet4_strength", 4, 0.6, 5)])
def test_v1_call_with_pndm_equals_reference_call_golden(name, cin, strength, steps):
    """N + 1 timesteps and their strength slices, the callback skipping the warm-up step, the 4-channel blend"""
    import test_pipeline_golden as G
    from oracle.unet import UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline

    om, sd = G._oracle(UNet2DConditionOracle, cin, "unet", {9: 77, 4: 78}[cin])
    pipe = StableDiffusionInpaintPipeline(vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=None,
                                          tokenizer=None, unet=UNet2DConditionModel.from_state_dict(G._cfg(cin), sd),
                                          scheduler=_sched(), safety_checker=None)
    fake = _PlmsDenoiser(om)
    pipe.denoiser = lambda: fake
    img, mask, pe, ne = G._call_inputs()
    seen = []
    out = pipe(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=G.H, width=G.W,
               strength=strength, num_inference_steps=steps, guidance_scale=7.5, generator=G._generators(False),
               output_type="latent", return_dict=False, callback=lambda i, t, x: seen.append((i, int(t))))[0]
    _check(out, seen, name)


def test_controlnet_call_with_pndm_equals_reference_call_golden():
    """the control-guidance window is computed over the N + 1 timesteps"""
    import test_pipeline_golden as G
    from oracle.unet import ControlNetOracle, UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import ControlNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionControlNetInpaintPipeline

    ou, sd_u = G._oracle(UNet2DConditionOracle, 9, "unet", 5)
    oc, sd_c = G._oracle(ControlNetOracle, 4, "controlnet", 6)
    pipe = StableDiffusionControlNetInpaintPipeline(
        vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=None, tokenizer=None,
        unet=UNet2DConditionModel.from_state_dict(G._cfg(9), sd_u),
        controlnet=ControlNetModel.from_state_dict(G._cfg(4), sd_c), scheduler=_sched(), safety_checker=None)
    fake = _PlmsDenoiser(ou, [oc], "controlnet")
    pipe.denoiser = lambda: fake
    img, mask, pe, ne = G._call_inputs()
    ctl = torch.rand(G.B, 3, G.H, G.W, generator=torch.Generator().manual_seed(31))
    seen = []
    out = pipe(image=img, mask=mask, control_image=ctl, prompt_embeds=pe, negative_prompt_embeds=ne, height=G.H,
               width=G.W, generator=G._generators(False), output_type="latent", return_dict=False,
               callback=lambda i, t, x: seen.append((i, int(t))), num_inference_steps=4, guidance_scale=7.5,
               controlnet_conditioning_scale=0.8, control_guidance_start=0.25, control_guidance_end=0.7)[0]
    _check(out, seen, "controlnet_window")


def test_brushnet_call_with_pndm_equals_reference_call_golden():
    """`brushnet_keep` over N + 1 timesteps, `num_timesteps`, the legacy callback skipping the warm-up step"""
    import test_pipeline_golden as G
    from oracle.unet import BrushNetOracle, UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import BrushNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionPowerPaintBrushNetPipeline

    ou, sd_u = G._oracle(UNet2DConditionOracle, 4, "unet", 11)
    ob, sd_b = G._oracle(BrushNetOracle, 4, "brushnet", 12)
    tok, te, te_b = G._text_stack()
    pipe = StableDiffusionPowerPaintBrushNetPipeline(
        vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=te, text_encoder_brushnet=te_b, tokenizer=tok,
        unet=UNet2DConditionModel.from_state_dict(G._cfg(4), sd_u),
        brushnet=BrushNetModel.from_state_dict(G._cfg(4), sd_b), scheduler=_sched(), safety_checker=None)
    fake = _PlmsDenoiser(ou, [ob], "brushnet")
    pipe.denoiser = lambda: fake
    img, mask = G._brushnet_inputs()
    seen = []
    torch.manual_seed(123)
    with torch.no_grad():
        out = pipe(**G.PROMPTS, tradoff=0.7, tradoff_nag=0.4, image=img, mask=mask, generator=G._generators(False),
                   num_inference_steps=3, guidance_scale=7.5, brushnet_conditioning_scale=1.0,
                   control_guidance_end=0.6, output_type="latent", return_dict=False,
                   callback=lambda i, t, x: seen.append((i, int(t))), callback_steps=1)[0]
    _check(out, seen, "brushnet_window")
    assert pipe.num_timesteps == 4
