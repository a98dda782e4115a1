"""CPU tests of the side-net options (guess mode, global pooling, several ControlNets): the logspace factors, the
oracle's pooling and sum order against closed forms, the new descriptor's layout, the reference's checks of a
Multi-ControlNet call, and what the pipelines' host side hands to the fused denoiser."""
import os

import pytest
import torch

from oracle import side_nets as osn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_guess_mode_factors_are_logspace_in_fp32():
    from powerpaint_b200.engine import guess_mode_alphas

    for n in (13, 28):
        got = guess_mode_alphas(n)
        closed = [10.0 ** (-1.0 + k / (n - 1)) for k in range(n)]
        assert len(got) == n and got[0] == pytest.approx(0.1, rel=1e-7) and got[-1] == 1.0
        # fp32 values: one fp32 rounding of the closed form
        assert all(abs(a - b) <= 2.0 ** -23 * b * 2 for a, b in zip(got, closed))
        assert all(float(torch.tensor(a, dtype=torch.float32)) == a for a in got)
        assert list(osn.guess_scales(n)) == pytest.approx(closed, rel=1e-14)


def test_oracle_scaling_pooling_and_sum_order_closed_forms():
    g = torch.Generator().manual_seed(0)
    res = [torch.randn(2, 3, 4, 5, generator=g, dtype=torch.float64) for _ in range(13)]
    s = osn.guess_scales(13)
    out = osn.scale_and_pool(res, 0.5, guess_mode=True, pool=False)
    assert all(torch.equal(o, r * (s[k] * 0.5)) for k, (o, r) in enumerate(zip(out, res)))
    # a pooled net skips the logspace factors, then averages over the pixels
    out = osn.scale_and_pool(res, 0.5, guess_mode=True, pool=True)
    for o, r in zip(out, res):
        assert o.shape == (2, 3, 1, 1)
        assert torch.allclose(o, (r * 0.5).sum((2, 3), keepdim=True) / 20, rtol=1e-14)
    # no guess mode: the conditioning scale alone
    out = osn.scale_and_pool(res, 0.25, guess_mode=False, pool=False)
    assert all(torch.equal(o, r * 0.25) for o, r in zip(out, res))

    class Net:  # residuals = the inputs themselves, in fixed channels
        def __init__(self, c):
            self.c = c

        def __call__(self, x, t, emb, cond, scale):
            return [x * self.c * scale] * 2, x * self.c * scale * 2

    x = torch.randn(1, 2, 3, 3, generator=g, dtype=torch.float64)
    d, m = osn.multi_controlnet([Net(1.0), Net(3.0), Net(5.0)], (False, True, False), x, 0, None, [None] * 3,
                                [0.5, 0.25])  # zip: the third net has no scale and is dropped
    assert torch.allclose(d[0], x * 0.5 + (x * 0.75).mean((2, 3), keepdim=True))
    assert torch.allclose(m, x * 1.0 + (x * 1.5).mean((2, 3), keepdim=True))


def test_pool_broadcast_descriptor_matches_the_header(tmp_path):
    import shutil
    import subprocess

    from powerpaint_b200 import _native as N

    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    cls, cname = N.PoolBroadcastDesc, "pp_pool_broadcast_desc"
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
    import ctypes

    assert int(out[cname]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f"{cname}.{f}"]) == getattr(cls, f).offset, f
    assert "pp_pool_broadcast" in N.EXPORTED_SYMBOLS and "pp_program_add_pool_broadcast" in N.EXPORTED_SYMBOLS


def _tiny_cfg(cin):
    from oracle.unet import UNetConfig
    from powerpaint_b200.engine import NetConfig

    o = UNetConfig.tiny(cin)
    return o, NetConfig(in_channels=cin, block_out_channels=o.block_out_channels, attention_head_dim=o.attention_head_dim,
                        cross_attention_dim=o.cross_attention_dim, norm_num_groups=o.norm_num_groups)


class _Recorder:
    """stand-in for FusedDenoiser.run: records what the pipeline hands over and returns the latents"""

    def __init__(self):
        self.kw = None

    def run(self, **kw):
        self.kw = kw
        return kw["latents"]


def _cn_pipe(nets):
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionControlNetInpaintPipeline
    from powerpaint_b200.schedulers import DDIMScheduler

    pipe = StableDiffusionControlNetInpaintPipeline(vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=None,
                                                    tokenizer=None, unet=UNet2DConditionModel(_tiny_cfg(9)[1]),
                                                    controlnet=nets, scheduler=DDIMScheduler())
    rec = _Recorder()
    pipe.denoiser = lambda: rec
    return pipe, rec


def _cn_inputs(B=1, H=64, cross=32):
    g = torch.Generator().manual_seed(3)
    img = torch.rand(B, 3, H, H, generator=g) * 2 - 1
    mask = torch.zeros(B, 1, H, H)
    mask[:, :, 16:48, 8:40] = 1
    pe = torch.randn(B, 77, cross, generator=g) * 0.5
    ne = torch.randn(B, 77, cross, generator=g) * 0.5
    ctl = [torch.rand(B, 3, H, H, generator=g) for _ in range(3)]
    return img, mask, pe, ne, ctl


def test_invalid_multi_controlnet_calls_raise_what_the_reference_raises():
    """the reference's own exceptions for invalid calls with two ControlNets (tests/golden/
    pipeline_controlnet_multi_errors.json, recorded by make_side_net_golden.py from its `__call__`)"""
    import json

    from powerpaint_b200.models import ControlNetModel

    with open(os.path.join(ROOT, "tests", "golden", "pipeline_controlnet_multi_errors.json")) as f:
        gold = json.load(f)
    pipe, _ = _cn_pipe([ControlNetModel(_tiny_cfg(4)[1]), ControlNetModel(_tiny_cfg(4)[1])])
    img, mask, pe, ne, ctl = golden_cn_inputs()
    cases = multi_error_cases(img, mask, pe, ne, ctl)
    assert sorted(cases) == sorted(gold) and all(v[0] != "no error" for v in gold.values())
    for name, kw in cases.items():
        kind, msg = gold[name]
        with pytest.raises(Exception) as ei:
            pipe(**kw)
        assert (type(ei.value).__name__, str(ei.value)) == (kind, msg), name


# ---------------------------------------------------------------- the reference's `__call__` (pipeline_side_net_call.npz)
# == tests/golden/make_side_net_golden.py: inputs, case tables, invalid calls
GB, GS = 2, 64
CN_SEEDS = (6, 61, 62)
CONTROLNET_CASES = {
    "cn_two_nets_windows": ((False, False), dict(num_inference_steps=5, guidance_scale=7.5,
                                                 controlnet_conditioning_scale=[0.5, 0.8],
                                                 control_guidance_start=[0.0, 0.2], control_guidance_end=[1.0, 0.6])),
    "cn_two_nets_default_window": ((False, False), dict(num_inference_steps=3, guidance_scale=7.5,
                                                        controlnet_conditioning_scale=0.6)),
    "cn_three_nets_guess": ((False, False, False), dict(num_inference_steps=3, guidance_scale=7.5, guess_mode=True,
                                                        controlnet_conditioning_scale=[0.5, 0.8, 1.0])),
    "cn_guess_cfg": ((False,), dict(num_inference_steps=4, guidance_scale=7.5, guess_mode=True,
                                    controlnet_conditioning_scale=0.7)),
    "cn_guess_no_cfg": ((False,), dict(num_inference_steps=3, guidance_scale=1.0, guess_mode=True,
                                       controlnet_conditioning_scale=0.7)),
    "cn_pooled": ((True,), dict(num_inference_steps=3, guidance_scale=7.5, controlnet_conditioning_scale=0.9)),
    "cn_pooled_then_plain": ((True, False), dict(num_inference_steps=3, guidance_scale=7.5,
                                                 controlnet_conditioning_scale=[0.9, 0.6])),
}
BRUSHNET_CASES = {
    "bn_guess": (False, dict(num_inference_steps=3, guidance_scale=7.5, guess_mode=True,
                             brushnet_conditioning_scale=0.8)),
    "bn_guess_window": (False, dict(num_inference_steps=4, guidance_scale=5.0, guess_mode=True,
                                    brushnet_conditioning_scale=1.0, control_guidance_end=0.6)),
    "bn_pooled": (True, dict(num_inference_steps=3, guidance_scale=7.5, brushnet_conditioning_scale=1.0)),
}


def _golden_path():
    import sys

    d = os.path.join(ROOT, "tests", "golden")
    if d not in sys.path:
        sys.path.insert(0, d)


def golden_cn_inputs():
    _golden_path()
    from pipeline_cases import sized_inputs

    img, mask, pe, ne, ctl = sized_inputs(GB, GS, GS, 64, 71)
    g = torch.Generator().manual_seed(72)
    return img, mask, pe, ne, [ctl] + [torch.rand(GB, 3, GS, GS, generator=g) for _ in range(2)]


def golden_bn_inputs():
    g = torch.Generator().manual_seed(73)
    img = torch.rand(GB, 3, GS, GS, generator=g)
    mask = torch.ones(GB, 3, GS, GS)
    mask[0, :, 8:40, 16:40] = 0
    mask[1, :, 20:60, 4:30] = 0
    return img * mask, mask


def multi_error_cases(img, mask, pe, ne, ctl):
    base = dict(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=GS, width=GS,
                num_inference_steps=2, output_type="latent", return_dict=False)
    two = [ctl[0], ctl[1]]
    return {
        "image_not_a_list": dict(base, control_image=ctl[0]),
        "one_image_for_two_nets": dict(base, control_image=[ctl[0]]),
        "three_images_for_two_nets": dict(base, control_image=ctl),
        "nested_images": dict(base, control_image=[[ctl[0]], [ctl[1]]]),
        "nested_scales": dict(base, control_image=two, controlnet_conditioning_scale=[[0.5], [0.5]]),
        "start_end_lengths": dict(base, control_image=two, control_guidance_start=[0.0, 0.1],
                                  control_guidance_end=[1.0]),
        "three_windows_for_two_nets": dict(base, control_image=two, control_guidance_start=[0.0, 0.1, 0.2]),
        "three_ends_for_two_nets": dict(base, control_image=two, control_guidance_end=[1.0, 0.9, 0.8]),
        "start_after_end": dict(base, control_image=two, control_guidance_start=[0.0, 0.7],
                                control_guidance_end=[1.0, 0.5]),
        "scale_not_a_float": dict(base, control_image=two, controlnet_conditioning_scale=1),
    }


class SideNetDenoiser:
    """what FusedDenoiser.run computes with side nets, in fp32 torch over the oracle nets (test stand-in only):
    K ControlNets or one BrushNet, guess mode (the conditional half under CFG), pooled nets, coefficient-row DDIM"""

    def __init__(self, unet, sides, pools, mode):
        self.unet, self.sides, self.pools, self.mode = unet, sides, pools, mode

    @torch.no_grad()
    def run(self, *, latents, prompt_embeds, side_prompt_embeds, timesteps, coef, guidance_scale, extra, side_scale,
            side_keep=None, control_image=None, guess_mode=False, noise_fn=None, callback=None, ucoef=None):
        do_cfg = guidance_scale > 1.0
        B = latents.shape[0]
        multi = isinstance(side_scale, list)
        scales, keeps = (side_scale, side_keep) if multi else ([side_scale], [side_keep])
        keeps = keeps if keeps is not None else [None] * len(scales)
        images = control_image if isinstance(control_image, list) else [control_image]
        half = guess_mode and do_cfg
        spe = side_prompt_embeds[-B:] if half and side_prompt_embeds.shape[0] == 2 * B else side_prompt_embeds

        def pad(r):
            return torch.cat([torch.zeros_like(r), r]) if half else r
        for i, t in enumerate(timesteps):
            x = torch.cat([latents] * 2) if do_cfg else latents
            xs = latents if half else x
            cs = [s * (k[i] if k is not None else 1.0) for s, k in zip(scales, keeps)]
            if self.mode == "controlnet":
                d, m = osn.multi_controlnet(self.sides, self.pools, xs, int(t), spe, images, cs, guess_mode)
                ex = torch.cat([extra] * 2) if do_cfg else extra
                eps = self.unet(torch.cat([x, ex], 1), int(t), prompt_embeds,
                                down_block_additional_residuals=[pad(r) for r in d],
                                mid_block_additional_residual=pad(m))
            else:
                d, m, u = osn.brushnet(self.sides[0], xs, int(t), spe, extra, cs[0], guess_mode, self.pools[0])
                eps = self.unet(x, int(t), prompt_embeds, down_block_add_samples=[pad(r) for r in d],
                                mid_block_add_sample=pad(m), up_block_add_samples=[pad(r) for r in u])
            if do_cfg:
                a, c = eps.chunk(2)
                eps = a + guidance_scale * (c - a)
            sa, s1a, sap, dirc, _ = [float(v) for v in coef[i, :5]]
            latents = sap * ((latents - s1a * eps) / sa) + dirc * eps
        return latents


def controlnet_golden_pipe(pools, device="cpu"):
    """the product pipeline with the fixture's weights; (pipe, oracle UNet, oracle ControlNets)"""
    from oracle.unet import ControlNetOracle, UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import ControlNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionControlNetInpaintPipeline
    from powerpaint_b200.schedulers import DDIMScheduler
    from test_pipeline_golden import _cfg, _oracle

    ou, sd_u = _oracle(UNet2DConditionOracle, 9, "unet", 5)
    ocs, pcs = [], []
    for k, pool in enumerate(pools):
        oc, sd_c = _oracle(ControlNetOracle, 4, "controlnet", CN_SEEDS[k])
        pc = ControlNetModel.from_state_dict(_cfg(4), sd_c).to(device)
        pc.config.global_pool_conditions = pool
        ocs.append(oc)
        pcs.append(pc)
    pipe = StableDiffusionControlNetInpaintPipeline(
        vae=AutoencoderKLOracle.synthetic(tiny=True).to(device), text_encoder=None, tokenizer=None,
        unet=UNet2DConditionModel.from_state_dict(_cfg(9), sd_u).to(device),
        controlnet=pcs[0] if len(pcs) == 1 else pcs, scheduler=DDIMScheduler(), safety_checker=None)
    return pipe, ou, ocs


def controlnet_golden_call(pipe, name):
    pools, kw = CONTROLNET_CASES[name]
    img, mask, pe, ne, ctl = golden_cn_inputs()
    control = ctl[0] if len(pools) == 1 else ctl[:len(pools)]
    with torch.no_grad():
        return pipe(image=img, mask=mask, control_image=control, prompt_embeds=pe, negative_prompt_embeds=ne,
                    height=GS, width=GS, generator=torch.Generator().manual_seed(13), output_type="latent",
                    return_dict=False, **kw)[0]


def brushnet_golden_pipe(pool):
    """the product BrushNet pipeline (CPU) with the fixture's weights and text stack; (pipe, oracle UNet, BrushNet)"""
    from oracle.unet import BrushNetOracle, UNet2DConditionOracle
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import BrushNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionPowerPaintBrushNetPipeline
    from powerpaint_b200.schedulers import DDIMScheduler
    from test_pipeline_golden import _cfg, _oracle, _text_stack

    ou, sd_u = _oracle(UNet2DConditionOracle, 4, "unet", 11)
    ob, sd_b = _oracle(BrushNetOracle, 4, "brushnet", 12)
    tok, te, te_b = _text_stack()
    bn = BrushNetModel.from_state_dict(_cfg(4), sd_b)
    bn.config.global_pool_conditions = pool
    pipe = StableDiffusionPowerPaintBrushNetPipeline(
        vae=AutoencoderKLOracle.synthetic(tiny=True), text_encoder=te, text_encoder_brushnet=te_b, tokenizer=tok,
        unet=UNet2DConditionModel.from_state_dict(_cfg(4), sd_u), brushnet=bn, scheduler=DDIMScheduler(),
        safety_checker=None)
    return pipe, ou, ob


def brushnet_golden_call(pipe, name):
    from test_pipeline_golden import PROMPTS

    _, kw = BRUSHNET_CASES[name]
    img, mask = golden_bn_inputs()
    torch.manual_seed(123)  # the conditioning latents come from the global generator, as in the reference
    with torch.no_grad():
        return pipe(**PROMPTS, tradoff=0.7, tradoff_nag=0.4, image=img, mask=mask,
                    generator=torch.Generator().manual_seed(4), output_type="latent", return_dict=False, **kw)[0]


def _gold(key):
    import numpy as np

    return torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "pipeline_side_net_call.npz"))[key])


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize("name", list(CONTROLNET_CASES))
def test_controlnet_side_net_call_equals_reference_call_golden(name):
    """the product's ControlNet `__call__` host side with an fp32 stand-in denoiser against the reference's own
    `__call__` (several nets, guidance windows, guess mode with and without CFG, pooled nets)"""
    pools, _ = CONTROLNET_CASES[name]
    pipe, ou, ocs = controlnet_golden_pipe(pools)
    pipe.denoiser = lambda: SideNetDenoiser(ou, ocs, pools, "controlnet")
    out = controlnet_golden_call(pipe, name)
    ref = _gold(f"{name}_latents")
    assert out.shape == ref.shape and _rel(out, ref) < 5e-5, _rel(out, ref)


@pytest.mark.parametrize("name", list(BRUSHNET_CASES))
def test_brushnet_side_net_call_equals_reference_call_golden(name):
    """the product's BrushNet `__call__` host side (guess mode: images not doubled, B VAE draws from the global RNG;
    pooled BrushNet) with an fp32 stand-in denoiser against the reference's own `__call__`"""
    pool, _ = BRUSHNET_CASES[name]
    pipe, ou, ob = brushnet_golden_pipe(pool)
    pipe.denoiser = lambda: SideNetDenoiser(ou, [ob], (pool,), "brushnet")
    out = brushnet_golden_call(pipe, name)
    ref = _gold(f"{name}_latents")
    assert out.shape == ref.shape and _rel(out, ref) < 5e-5, _rel(out, ref)


def test_multi_controlnet_call_hands_per_net_inputs_to_the_denoiser():
    from powerpaint_b200.models import ControlNetModel, MultiControlNetModel

    nets = [ControlNetModel(_tiny_cfg(4)[1]) for _ in range(3)]
    pipe, rec = _cn_pipe(nets)
    assert isinstance(pipe.controlnet, MultiControlNetModel) and len(pipe.controlnet.nets) == 3
    img, mask, pe, ne, ctl = _cn_inputs()
    steps = 4
    pipe(image=img, mask=mask, control_image=ctl, prompt_embeds=pe, negative_prompt_embeds=ne,
         num_inference_steps=steps, guidance_scale=7.5, controlnet_conditioning_scale=0.7,
         control_guidance_start=[0.0, 0.25, 0.0], control_guidance_end=[1.0, 1.0, 0.5], output_type="latent")
    kw = rec.kw
    assert kw["side_scale"] == [0.7, 0.7, 0.7]  # a float scale is replicated to every net (:1533)
    assert kw["side_keep"] == [[1.0] * 4, [0.0, 1.0, 1.0, 1.0], [1.0, 1.0, 0.0, 0.0]]
    assert [tuple(c.shape) for c in kw["control_image"]] == [(2, 3, 64, 64)] * 3  # doubled for CFG
    assert "guess_mode" not in kw
    # guess mode: the control images are not doubled; a scale list shorter than the nets drops the rest (zip)
    pipe(image=img, mask=mask, control_image=ctl, prompt_embeds=pe, negative_prompt_embeds=ne,
         num_inference_steps=steps, guidance_scale=7.5, controlnet_conditioning_scale=[0.5, 0.8], guess_mode=True,
         control_guidance_start=[0.0] * 3, control_guidance_end=[1.0] * 3, output_type="latent")
    kw = rec.kw
    assert kw["guess_mode"] is True and kw["side_scale"] == [0.5, 0.8, 0.0]
    assert [tuple(c.shape) for c in kw["control_image"]] == [(1, 3, 64, 64)] * 3
    # a pooled first net forces guess mode (:1536-1541)
    nets[0].config.global_pool_conditions = True
    pipe(image=img, mask=mask, control_image=ctl, prompt_embeds=pe, negative_prompt_embeds=ne,
         num_inference_steps=steps, guidance_scale=7.5, control_guidance_start=[0.0] * 3,
         control_guidance_end=[1.0] * 3, output_type="latent")
    assert rec.kw["guess_mode"] is True


def test_single_controlnet_call_is_unchanged_without_guess_mode():
    from powerpaint_b200.models import ControlNetModel

    pipe, rec = _cn_pipe(ControlNetModel(_tiny_cfg(4)[1]))
    img, mask, pe, ne, ctl = _cn_inputs()
    pipe(image=img, mask=mask, control_image=ctl[0], prompt_embeds=pe, negative_prompt_embeds=ne,
         num_inference_steps=3, guidance_scale=7.5, controlnet_conditioning_scale=0.5, output_type="latent")
    kw = rec.kw
    assert kw["side_scale"] == 0.5 and kw["side_keep"] == [1.0] * 3 and "guess_mode" not in kw
    assert tuple(kw["control_image"].shape) == (2, 3, 64, 64)
    pipe(image=img, mask=mask, control_image=ctl[0], prompt_embeds=pe, negative_prompt_embeds=ne,
         num_inference_steps=3, guidance_scale=7.5, controlnet_conditioning_scale=0.5, guess_mode=True,
         output_type="latent")
    assert rec.kw["guess_mode"] is True and tuple(rec.kw["control_image"].shape) == (1, 3, 64, 64)


def test_brushnet_guess_mode_encodes_one_set_of_conditioning_latents():
    """under guess mode the image and mask are not doubled, so the VAE encode draws B samples from the global RNG,
    not 2B (:1300-1345)"""
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import BrushNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import StableDiffusionPowerPaintBrushNetPipeline
    from powerpaint_b200.schedulers import DDIMScheduler

    o, n = _tiny_cfg(4)
    vae = AutoencoderKLOracle.synthetic(tiny=True)
    pipe = StableDiffusionPowerPaintBrushNetPipeline(vae=vae, text_encoder=None, text_encoder_brushnet=None,
                                                     tokenizer=None, unet=UNet2DConditionModel(n),
                                                     brushnet=BrushNetModel(n), scheduler=DDIMScheduler())
    rec = _Recorder()
    pipe.denoiser = lambda: rec
    B, H = 1, 64
    g = torch.Generator().manual_seed(5)
    img = torch.rand(B, 3, H, H, generator=g) * 2 - 1
    mask = torch.ones(B, 3, H, H)
    mask[:, :, 16:48, 16:48] = -1.0
    pe = torch.randn(B, 77, o.cross_attention_dim, generator=g) * 0.5
    ne = torch.randn(B, 77, o.cross_attention_dim, generator=g) * 0.5
    peU = torch.randn(2 * B, 77, o.cross_attention_dim, generator=g) * 0.5
    lat = torch.randn(B, 4, H // 8, H // 8, generator=g)  # given: the call draws nothing for the initial latents
    for guess, pool in ((True, False), (False, True)):
        pipe.brushnet.config.global_pool_conditions = pool
        torch.manual_seed(123)
        pipe(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, prompt_embedsU=peU, latents=lat,
             num_inference_steps=3, guidance_scale=7.5, guess_mode=guess, output_type="latent",
             brushnet_conditioning_scale=0.8)
        after = torch.randn(4)
        kw = rec.kw
        assert kw["guess_mode"] is True and kw["extra"].shape[0] == B
        torch.manual_seed(123)
        want = vae.encode(img).latent_dist.sample() * vae.config.scaling_factor
        assert torch.allclose(kw["extra"][:, :4], want, atol=1e-5)
        assert torch.equal(after, torch.randn(4)), "the global RNG advanced by B samples, as the reference's does"
    pipe.brushnet.config.global_pool_conditions = False
    pipe(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, prompt_embedsU=peU,
         num_inference_steps=3, guidance_scale=7.5, output_type="latent", brushnet_conditioning_scale=0.8)
    assert rec.kw["extra"].shape[0] == 2 * B and "guess_mode" not in rec.kw


def test_side_net_configs_with_global_pooling_load():
    from powerpaint_b200.loading import net_config_from_diffusers
    from powerpaint_b200.models import BrushNetModel, ControlNetModel

    for cls in (ControlNetModel, BrushNetModel):
        m = cls.from_config(dict(global_pool_conditions=True, block_out_channels=[32, 64, 64, 64], in_channels=4))
        assert m.config.global_pool_conditions is True
        assert cls.from_config(dict(in_channels=4)).config.global_pool_conditions is False
    with pytest.raises(NotImplementedError, match="global_pool_conditions"):
        net_config_from_diffusers(dict(global_pool_conditions=True), "unet")
