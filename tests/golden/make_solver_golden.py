"""Generate tests/golden/pipeline_solver_call.npz: the REFERENCE's own v1 and BrushNet `__call__` with the
DPM-Solver++ and Euler-ancestral schedulers.

    PP_REFERENCE_DIR=<checkout of open-mmlab/PowerPaint> python tests/golden/make_solver_golden.py

Same set-up as make_pipeline_golden.py (reference pipelines, UNet and BrushNet imported unmodified over
tests/golden/diffusers_shim, synthetic weights, the oracle VAE); the scheduler behind the diffusers call contract is
the stepwise oracle (oracle/dpmsolver.py, oracle/euler.py). What the fixture pins is where the pipeline puts
`init_noise_sigma`, `scale_model_input` and `add_noise`, and the order in which the scheduler's `step` draws its noise
from the caller's generator.
"""
import os

import numpy as np
import torch

import make_pipeline_golden as G  # noqa: E402  (sets sys.path: shim, reference, repository root)
from diffusers.models import AutoencoderKL  # noqa: E402
from oracle.dpmsolver import DPMSolverOracle  # noqa: E402
from oracle.euler import EulerAncestralOracle  # noqa: E402

from make_unet_golden import cfg, ref_unet  # noqa: E402
from powerpaint_b200.models import synthetic_state_dict  # noqa: E402

# name -> (oracle class, its arguments beyond the SD schedule); the product side builds the same through `from_config`
SCHEDULERS = {
    "dpmpp_2m_karras": (DPMSolverOracle, dict(use_karras_sigmas=True)),
    "sde_dpmpp_2m": (DPMSolverOracle, dict(algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min")),
    "euler_a": (EulerAncestralOracle, {}),
}
V1_CASES = {  # name -> (scheduler, strength, steps)
    "v1_dpmpp_2m_karras": ("dpmpp_2m_karras", 1.0, 5),
    "v1_euler_a": ("euler_a", 1.0, 4),
    "v1_sde_dpmpp_2m_strength": ("sde_dpmpp_2m", 0.5, 8),
    "v1_euler_a_strength": ("euler_a", 0.6, 5),
}
BRUSHNET_CASES = {"brushnet_dpmpp_2m_karras": ("dpmpp_2m_karras", 4), "brushnet_euler_a": ("euler_a", 3)}


def scheduler(name):
    """the oracle scheduler with the call contract the reference pipelines use"""
    base, kw = SCHEDULERS[name]

    class Sched(base):
        @property
        def config(self):
            return dict(num_train_timesteps=self.T)

        def set_timesteps(self, n, device=None):
            super().set_timesteps(n)

        def step(self, model_output, timestep, sample, generator=None, return_dict=True):
            return (super().step(model_output, timestep, sample, generator=generator),)

    return Sched(**kw)


@torch.no_grad()
def main():
    out = {}
    unet = ref_unet(9)
    unet.load_state_dict(synthetic_state_dict(cfg(9), "unet", 77), strict=True)
    img, mask, pe, ne = G.call_inputs()
    for name, (sched, strength, steps) in V1_CASES.items():
        pipe = G.RefPipe(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=None, tokenizer=None, unet=unet,
                         scheduler=scheduler(sched), safety_checker=None, feature_extractor=None,
                         requires_safety_checker=False)
        lat = pipe(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=G.H, width=G.W,
                   strength=strength, num_inference_steps=steps, guidance_scale=7.5, generator=G.generators(False),
                   output_type="latent", return_dict=False)[0]
        out[f"{name}_latents"] = lat.numpy()
        print(name, tuple(lat.shape), float(lat.abs().mean()))
    import copy

    from powerpaint.models.BrushNet_CA import BrushNetModel as RefBrushNet
    from powerpaint.pipelines.pipeline_PowerPaint_Brushnet_CA import StableDiffusionPowerPaintBrushNetPipeline as RefBN

    u4 = ref_unet(4)
    u4.load_state_dict(synthetic_state_dict(cfg(4), "unet", 11), strict=True)
    bn = copy.deepcopy(RefBrushNet.from_unet(ref_unet(4), conditioning_channels=5)).eval()
    bn.load_state_dict(synthetic_state_dict(cfg(4), "brushnet", 12), strict=True)
    tok, te, te_b = G.text_stack()
    bimg, bmask = G.brushnet_inputs()
    for name, (sched, steps) in BRUSHNET_CASES.items():
        pipe = RefBN(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=te, text_encoder_brushnet=te_b, tokenizer=tok,
                     unet=u4, brushnet=bn, scheduler=scheduler(sched), safety_checker=None, feature_extractor=None,
                     requires_safety_checker=False)
        torch.manual_seed(123)  # the conditioning latents are sampled from the GLOBAL generator
        lat = pipe(**G.PROMPTS, tradoff=0.7, tradoff_nag=0.4, image=bimg, mask=bmask, generator=G.generators(False),
                   num_inference_steps=steps, guidance_scale=7.5, brushnet_conditioning_scale=1.0,
                   output_type="latent", return_dict=False)[0]
        out[f"{name}_latents"] = lat.numpy()
        print(name, tuple(lat.shape), float(lat.abs().mean()))
    path = os.path.join(os.environ.get("PP_GOLDEN_OUT", G.HERE), "pipeline_solver_call.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
