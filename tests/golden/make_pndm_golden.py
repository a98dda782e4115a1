"""Generate tests/golden/pipeline_pndm_call.npz: the REFERENCE's own v1, ControlNet and BrushNet `__call__` with the
PNDM (PLMS) scheduler the v1 checkpoint stores.

    PP_REFERENCE_DIR=<checkout of open-mmlab/PowerPaint> python tests/golden/make_pndm_golden.py

Same set-up as make_pipeline_golden.py (reference pipelines, UNet and BrushNet imported unmodified over
tests/golden/diffusers_shim, synthetic weights, the oracle VAE and ControlNet); the scheduler is the stepwise oracle
(oracle/pndm.py) behind diffusers' call contract (`PNDMScheduler` below). What the fixture pins is how the pipelines
walk PNDM's N + 1 timesteps: strength slicing of that list, the legacy callback skipping the warm-up step
(`num_warmup_steps = 1`), the 4-channel blend noised to `timesteps[i + 1]`, the control-guidance window over
N + 1 entries, and that no `eta` / `generator` reaches `step`.
"""
import os

import numpy as np
import torch

import make_pipeline_golden as G  # noqa: E402  (sets sys.path: shim, reference, repository root)
from diffusers.configuration_utils import FrozenDict  # noqa: E402
from diffusers.models import AutoencoderKL  # noqa: E402
from oracle.pndm import PNDMOracle  # noqa: E402

from make_unet_golden import cfg, ref_unet  # noqa: E402
from powerpaint_b200.models import synthetic_state_dict  # noqa: E402

V1_CASES = {  # name -> (UNet input channels, strength, steps)
    "v1_full": (9, 1.0, 4),
    "v1_strength": (9, 0.6, 5),  # the slice starts past the repeated timestep
    "v1_strength_restart": (9, 0.8, 5),  # the slice starts AT the repeated timestep: the Heun restart then steps back up
    "v1_unet4": (4, 1.0, 4),
    "v1_unet4_strength": (4, 0.6, 5),
}
CONTROLNET_CASES = {
    "controlnet_window": dict(num_inference_steps=4, guidance_scale=7.5, controlnet_conditioning_scale=0.8,
                              control_guidance_start=0.25, control_guidance_end=0.7),
}
# GPU fixtures (tests/test_pndm_gpu.py repeats these): latent sizes the tiny GPU tests already exercise
GPU_V1 = dict(size=128, seed=51, gen_seed=11, kw=dict(num_inference_steps=6, guidance_scale=7.5))
GPU_CONTROLNET = dict(size=64, seed=53, gen_seed=13,
                      kw=dict(num_inference_steps=6, guidance_scale=7.5, controlnet_conditioning_scale=0.5,
                              control_guidance_start=0.0, control_guidance_end=0.7))


class PNDMScheduler(PNDMOracle):
    """the oracle PNDM with the diffusers call contract the reference pipelines use, and the SD-1.x checkpoints'
    `skip_prk_steps: true`; `step` takes neither `eta` nor `generator`, as diffusers' does, so the pipelines'
    signature sniffing passes none"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self._internal_dict = FrozenDict(steps_offset=self.steps_offset, num_train_timesteps=self.T,
                                         skip_prk_steps=True)

    @property
    def config(self):
        return self._internal_dict

    def step(self, model_output, timestep, sample, return_dict: bool = True):
        return (super().step(model_output, timestep, sample),)


def sched():
    return PNDMScheduler(set_alpha_to_one=False, steps_offset=1)


@torch.no_grad()
def main():
    from pipeline_cases import sized_inputs

    out = {}
    unets = {}
    for cin, seed in ((9, 77), (4, 78)):
        unets[cin] = ref_unet(cin)
        unets[cin].load_state_dict(synthetic_state_dict(cfg(cin), "unet", seed), strict=True)
    img, mask, pe, ne = G.call_inputs()

    def v1_pipe(cin):
        return G.RefPipe(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=None, tokenizer=None, unet=unets[cin],
                         scheduler=sched(), safety_checker=None, feature_extractor=None, requires_safety_checker=False)

    for name, (cin, strength, steps) in V1_CASES.items():
        seen = []
        lat = v1_pipe(cin)(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=G.H, width=G.W,
                           strength=strength, num_inference_steps=steps, guidance_scale=7.5,
                           generator=G.generators(False), output_type="latent", return_dict=False,
                           callback=lambda i, t, x: seen.append((i, int(t))))[0]
        out[f"{name}_latents"] = lat.numpy()
        out[f"{name}_callback"] = np.array(seen, dtype=np.int64).reshape(-1, 2)
        print(name, tuple(lat.shape), seen, float(lat.abs().mean()))
    gi, gm, gpe, gne, _ = sized_inputs(G.B, GPU_V1["size"], GPU_V1["size"], G.CROSS, GPU_V1["seed"])
    lat = v1_pipe(9)(image=gi, mask=gm, prompt_embeds=gpe, negative_prompt_embeds=gne, height=GPU_V1["size"],
                     width=GPU_V1["size"], generator=torch.Generator().manual_seed(GPU_V1["gen_seed"]),
                     output_type="latent", return_dict=False, **GPU_V1["kw"])[0]
    out["gpu_v1_latents"] = lat.numpy()
    print("gpu_v1", tuple(lat.shape), float(lat.abs().mean()))

    from diffusers.models import ControlNetModel
    from oracle.unet import UNetConfig
    from powerpaint.pipelines.pipeline_PowerPaint_ControlNet import StableDiffusionControlNetInpaintPipeline as RefCN

    u9 = ref_unet(9)
    u9.load_state_dict(synthetic_state_dict(cfg(9), "unet", 5), strict=True)
    cn = ControlNetModel(UNetConfig.tiny(4)).eval()
    cn.load_state_dict(synthetic_state_dict(cfg(4), "controlnet", 6), strict=True)
    pipe = RefCN(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=None, tokenizer=None, unet=u9, controlnet=cn,
                 scheduler=sched(), safety_checker=None, feature_extractor=None, requires_safety_checker=False)
    ctl = torch.rand(G.B, 3, G.H, G.W, generator=torch.Generator().manual_seed(31))
    for name, kw in CONTROLNET_CASES.items():
        seen = []
        lat = pipe(image=img, mask=mask, control_image=ctl, prompt_embeds=pe, negative_prompt_embeds=ne, height=G.H,
                   width=G.W, generator=G.generators(False), output_type="latent", return_dict=False,
                   callback=lambda i, t, x: seen.append((i, int(t))), **kw)[0]
        out[f"{name}_latents"] = lat.numpy()
        out[f"{name}_callback"] = np.array(seen, dtype=np.int64).reshape(-1, 2)
        print(name, tuple(lat.shape), seen, float(lat.abs().mean()))
    s = GPU_CONTROLNET["size"]
    gi, gm, gpe, gne, gctl = sized_inputs(G.B, s, s, G.CROSS, GPU_CONTROLNET["seed"])
    lat = pipe(image=gi, mask=gm, control_image=gctl, prompt_embeds=gpe, negative_prompt_embeds=gne, height=s, width=s,
               generator=torch.Generator().manual_seed(GPU_CONTROLNET["gen_seed"]), output_type="latent",
               return_dict=False, **GPU_CONTROLNET["kw"])[0]
    out["gpu_controlnet_latents"] = lat.numpy()
    print("gpu_controlnet", tuple(lat.shape), float(lat.abs().mean()))

    import copy

    from powerpaint.models.BrushNet_CA import BrushNetModel as RefBrushNet
    from powerpaint.pipelines.pipeline_PowerPaint_Brushnet_CA import StableDiffusionPowerPaintBrushNetPipeline as RefBN

    u4 = ref_unet(4)
    u4.load_state_dict(synthetic_state_dict(cfg(4), "unet", 11), strict=True)
    bn = copy.deepcopy(RefBrushNet.from_unet(ref_unet(4), conditioning_channels=5)).eval()
    bn.load_state_dict(synthetic_state_dict(cfg(4), "brushnet", 12), strict=True)
    tok, te, te_b = G.text_stack()
    bimg, bmask = G.brushnet_inputs()
    pipe = RefBN(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=te, text_encoder_brushnet=te_b, tokenizer=tok,
                 unet=u4, brushnet=bn, scheduler=sched(), safety_checker=None, feature_extractor=None,
                 requires_safety_checker=False)
    seen = []
    torch.manual_seed(123)  # the conditioning latents are sampled from the GLOBAL generator
    lat = pipe(**G.PROMPTS, tradoff=0.7, tradoff_nag=0.4, image=bimg, mask=bmask, generator=G.generators(False),
               num_inference_steps=3, guidance_scale=7.5, brushnet_conditioning_scale=1.0, control_guidance_end=0.6,
               output_type="latent", return_dict=False, callback=lambda i, t, x: seen.append((i, int(t))),
               callback_steps=1)[0]
    out["brushnet_window_latents"] = lat.numpy()
    out["brushnet_window_callback"] = np.array(seen, dtype=np.int64).reshape(-1, 2)
    print("brushnet_window", tuple(lat.shape), seen, float(lat.abs().mean()))
    path = os.path.join(os.environ.get("PP_GOLDEN_OUT", G.HERE), "pipeline_pndm_call.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
