"""Generate tests/golden/pipeline_side_net_call.npz and pipeline_controlnet_multi_errors.json: the REFERENCE's own
ControlNet and BrushNet `__call__` with several ControlNets, guess mode and globally pooled side nets.

    PP_REFERENCE_DIR=<checkout of open-mmlab/PowerPaint> python tests/golden/make_side_net_golden.py

Same set-up as make_pipeline_golden.py: the reference pipelines, UNet and BrushNet are imported unmodified over
tests/golden/diffusers_shim, with synthetic weights and the oracle VAE / DDIM. The ControlNet and MultiControlNetModel
the ControlNet pipeline imports from diffusers are defined here (the shim's ControlNet refuses guess mode and its
MultiControlNetModel refuses to be built, so that the older fixtures keep pinning what they pin): the oracle
ControlNet with diffusers 0.27.0's guess-mode scaling and global pooling, and the multi-net sum in net order, both as
recalled (oracle/side_nets.py). The BrushNet is the reference's own, whose forward does its scaling and pooling itself
(BrushNet_CA.py:905-943). What the fixture pins is the host side of `__call__`: the guidance-window and scale
alignment per net, which images are doubled under guess mode, the conditional-half batching, the zero residuals of the
unconditional half, and (BrushNet) the B-sample VAE draw of guess mode.
"""
import os

import numpy as np
import torch

import make_pipeline_golden as G  # noqa: E402  (sets sys.path: shim, reference, repository root)
from diffusers.models import AutoencoderKL  # noqa: E402
from diffusers.schedulers import DDIMScheduler  # noqa: E402

from make_unet_golden import CROSS, cfg, ref_unet  # noqa: E402
from oracle import side_nets as osn  # noqa: E402
from oracle.unet import ControlNetOracle, UNetConfig  # noqa: E402
from powerpaint_b200.models import synthetic_state_dict  # noqa: E402

B, S = 2, 64  # two images of 64 x 64 (8 x 8 latents: a size the tiny GPU loops already run)
CN_SEEDS = (6, 61, 62)  # ControlNet k: synthetic weights of seed CN_SEEDS[k]


class SideControlNet(ControlNetOracle):
    """the oracle ControlNet behind diffusers' ControlNetModel call signature, with guess mode and global pooling"""

    def __init__(self, global_pool_conditions=False):
        super().__init__(UNetConfig.tiny(4))
        self.global_pool_conditions = global_pool_conditions

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def config(self):
        from diffusers.configuration_utils import FrozenDict

        return FrozenDict(global_pool_conditions=self.global_pool_conditions)

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                guess_mode=False, return_dict=True, **kw):
        return osn.controlnet(super().forward, sample, timestep, encoder_hidden_states, controlnet_cond,
                              conditioning_scale, guess_mode, self.global_pool_conditions)


class MultiControlNetModel(torch.nn.Module):
    """diffusers 0.27.0 MultiControlNetModel as recalled: `.nets`, the residuals summed in net order"""

    def __init__(self, controlnets):
        super().__init__()
        self.nets = torch.nn.ModuleList(controlnets)

    @property
    def dtype(self):
        return self.nets[0].dtype

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale, guess_mode=False,
                return_dict=True, **kw):
        down = mid = None
        for i, (image, scale, net) in enumerate(zip(controlnet_cond, conditioning_scale, self.nets)):
            d, m = net(sample, timestep, encoder_hidden_states, image, scale, guess_mode=guess_mode)
            if i == 0:
                down, mid = d, m
            else:
                down = [a + b for a, b in zip(down, d)]
                mid = mid + m
        return down, mid


def controlnets(pools):
    nets = []
    for k, pool in enumerate(pools):
        cn = SideControlNet(pool).eval()
        cn.load_state_dict(synthetic_state_dict(cfg(4), "controlnet", CN_SEEDS[k]), strict=True)
        nets.append(cn)
    return nets


def cn_inputs():
    """image in [-1, 1], mask, prompt / negative embeddings and three control images"""
    from pipeline_cases import sized_inputs

    img, mask, pe, ne, ctl = sized_inputs(B, S, S, CROSS, 71)
    g = torch.Generator().manual_seed(72)
    return img, mask, pe, ne, [ctl] + [torch.rand(B, 3, S, S, generator=g) for _ in range(2)]


# name -> (ControlNet pools (one per net), call kwargs beyond the inputs). A single-entry pool tuple passes the net
# itself, more entries a list (wrapped in MultiControlNetModel by the pipeline, :306).
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
BRUSHNET_CASES = {  # name -> (pooled, call kwargs). guidance_scale <= 1 is not a case: the reference's
    # encode_prompt concatenates a None then (:627)
    "bn_guess": (False, dict(num_inference_steps=3, guidance_scale=7.5, guess_mode=True,
                             brushnet_conditioning_scale=0.8)),
    "bn_guess_window": (False, dict(num_inference_steps=4, guidance_scale=5.0, guess_mode=True,
                                    brushnet_conditioning_scale=1.0, control_guidance_end=0.6)),
    "bn_pooled": (True, dict(num_inference_steps=3, guidance_scale=7.5, brushnet_conditioning_scale=1.0)),
}


def brushnet_inputs():
    """image in [0, 1], mask whose zeros mark the hole (make_pipeline_golden.brushnet_inputs at 64 x 64)"""
    g = torch.Generator().manual_seed(73)
    img = torch.rand(B, 3, S, S, generator=g)
    mask = torch.ones(B, 3, S, S)
    mask[0, :, 8:40, 16:40] = 0
    mask[1, :, 20:60, 4:30] = 0
    return img * mask, mask


def multi_error_cases(img, mask, pe, ne, ctl):
    """invalid calls with two ControlNets: name -> kwargs"""
    base = dict(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=S, width=S,
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


@torch.no_grad()
def main():
    import powerpaint.pipelines.pipeline_PowerPaint_ControlNet as ref_cn

    # the diffusers names the reference pipeline module resolves at call time
    ref_cn.ControlNetModel, ref_cn.MultiControlNetModel = SideControlNet, MultiControlNetModel
    u9 = ref_unet(9)
    u9.load_state_dict(synthetic_state_dict(cfg(9), "unet", 5), strict=True)
    img, mask, pe, ne, ctl = cn_inputs()
    out = {}
    for name, (pools, kw) in CONTROLNET_CASES.items():
        nets = controlnets(pools)
        pipe = ref_cn.StableDiffusionControlNetInpaintPipeline(
            vae=AutoencoderKL.synthetic(tiny=True), text_encoder=None, tokenizer=None, unet=u9,
            controlnet=nets[0] if len(nets) == 1 else nets, scheduler=DDIMScheduler(), safety_checker=None,
            feature_extractor=None, requires_safety_checker=False)
        control = ctl[0] if len(nets) == 1 else ctl[:len(nets)]
        lat = pipe(image=img, mask=mask, control_image=control, prompt_embeds=pe, negative_prompt_embeds=ne,
                   height=S, width=S, generator=torch.Generator().manual_seed(13), output_type="latent",
                   return_dict=False, **kw)[0]
        out[f"{name}_latents"] = lat.numpy()
        print(name, tuple(lat.shape), float(lat.abs().mean()))
    pipe = ref_cn.StableDiffusionControlNetInpaintPipeline(
        vae=AutoencoderKL.synthetic(tiny=True), text_encoder=None, tokenizer=None, unet=u9,
        controlnet=controlnets((False, False)), scheduler=DDIMScheduler(), safety_checker=None,
        feature_extractor=None, requires_safety_checker=False)
    G.record_errors(pipe, multi_error_cases(img, mask, pe, ne, ctl), "pipeline_controlnet_multi_errors.json")

    import copy

    from powerpaint.models.BrushNet_CA import BrushNetModel as RefBrushNet
    from powerpaint.pipelines.pipeline_PowerPaint_Brushnet_CA import StableDiffusionPowerPaintBrushNetPipeline as RefBN

    u4 = ref_unet(4)
    u4.load_state_dict(synthetic_state_dict(cfg(4), "unet", 11), strict=True)
    tok, te, te_b = G.text_stack()
    bimg, bmask = brushnet_inputs()
    for name, (pool, kw) in BRUSHNET_CASES.items():
        bn = copy.deepcopy(RefBrushNet.from_unet(ref_unet(4), conditioning_channels=5)).eval()
        bn.load_state_dict(synthetic_state_dict(cfg(4), "brushnet", 12), strict=True)
        bn.register_to_config(global_pool_conditions=pool)
        pipe = RefBN(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=te, text_encoder_brushnet=te_b, tokenizer=tok,
                     unet=u4, brushnet=bn, scheduler=DDIMScheduler(), safety_checker=None, feature_extractor=None,
                     requires_safety_checker=False)
        torch.manual_seed(123)  # the conditioning latents are sampled from the GLOBAL generator (:1335)
        lat = pipe(**G.PROMPTS, tradoff=0.7, tradoff_nag=0.4, image=bimg, mask=bmask,
                   generator=torch.Generator().manual_seed(4), output_type="latent", return_dict=False, **kw)[0]
        out[f"{name}_latents"] = lat.numpy()
        print(name, tuple(lat.shape), float(lat.abs().mean()))
    G.save("pipeline_side_net_call.npz", out)


if __name__ == "__main__":
    main()
