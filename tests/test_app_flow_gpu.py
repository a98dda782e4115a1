"""GPU: `PowerPaintController` returns the app's bytes. Each request runs twice over the SAME tiny synthetic product
pipelines with the same seeds: once through oracle/app_flow.py (the app's PIL / NumPy / cv2 host code, PIL images into
the pipelines) and once through the controller (uint8 CUDA tensors in, every image step on the device). The returned
PIL images must be identical."""
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))


def _text():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from synthetic_clip import make_text_encoder, make_tokenizer

    from powerpaint_b200.models import CLIPTextModel
    from powerpaint_b200.utils import TokenizerWrapper, add_tokens

    tok = TokenizerWrapper.from_tokenizer(make_tokenizer())
    te = CLIPTextModel.from_transformers(make_text_encoder(len(tok.wrapped), hidden=64, seed=0))
    add_tokens(tokenizer=tok, text_encoder=te, placeholder_tokens=["P_ctxt", "P_shape", "P_obj"],
               initialize_tokens=["a", "a", "a"], num_vectors_per_token=10)
    return tok, te.to(DEV)


def _net(cls, cin, seed):
    from oracle.unet import UNetConfig
    from powerpaint_b200.engine import NetConfig

    o = UNetConfig.tiny(cin)
    n = NetConfig(in_channels=cin, block_out_channels=o.block_out_channels, attention_head_dim=o.attention_head_dim,
                  cross_attention_dim=o.cross_attention_dim, norm_num_groups=o.norm_num_groups)
    return cls.synthetic(n, seed).to(DEV)


@pytest.fixture(scope="module")
def pipes():
    from powerpaint_b200.models import BrushNetModel, ControlNetModel, UNet2DConditionModel
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL
    from powerpaint_b200.pipelines import (StableDiffusionControlNetInpaintPipeline, StableDiffusionInpaintPipeline,
                                           StableDiffusionPowerPaintBrushNetPipeline)
    from powerpaint_b200.schedulers import DDIMScheduler

    tok, te = _text()
    vae = AutoencoderKL.synthetic(tiny=True).to(DEV)
    unet9 = _net(UNet2DConditionModel, 9, 1234)
    v1 = StableDiffusionInpaintPipeline(vae=vae, text_encoder=te, tokenizer=tok, unet=unet9, scheduler=DDIMScheduler(),
                                        safety_checker=None)
    cn = StableDiffusionControlNetInpaintPipeline(vae=vae, text_encoder=te, tokenizer=tok, unet=unet9,
                                                  controlnet=_net(ControlNetModel, 4, 77), scheduler=DDIMScheduler(),
                                                  safety_checker=None)
    v2 = StableDiffusionPowerPaintBrushNetPipeline(vae=vae, text_encoder=te, text_encoder_brushnet=te, tokenizer=tok,
                                                   unet=_net(UNet2DConditionModel, 4, 4321),
                                                   brushnet=_net(BrushNetModel, 4, 99), scheduler=DDIMScheduler(),
                                                   safety_checker=None)
    return {"ppt-v1": v1, "ppt-v2": v2, "control": cn}


def _upload(w, h, seed, mask_mode="RGB"):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = np.stack([(x * 255 // w), (y * 255 // h), ((x + y) * 3) % 256], -1) + rng.integers(0, 40, (h, w, 3))
    img = Image.fromarray(np.clip(img, 0, 255).astype(np.uint8))
    m = np.zeros((h, w), np.uint8)
    m[h // 4:3 * h // 4, w // 3:2 * w // 3] = 255
    return {"image": img, "mask": Image.fromarray(m).convert(mask_mode)}


def _same(got, want):
    assert len(got) == len(want)
    for g_list, w_list in zip(got, want):
        assert len(g_list) == len(w_list)
        for g, w in zip(g_list, w_list):
            assert g.size == w.size and g.mode == w.mode, (g.size, w.size, g.mode, w.mode)
            a, b = np.asarray(g), np.asarray(w)
            assert np.array_equal(a, b), f"{int((a != b).sum())} bytes differ (max {int(np.abs(a.astype(int) - b).max())})"


def _both(pipes, version, method, *args, control=None, loader=None, annotators=None):
    from oracle.app_flow import AppFlowOracle
    from powerpaint_b200.controller import PowerPaintController

    pipe = pipes[version]
    want = getattr(AppFlowOracle(pipe, version, control, loader, annotators), method)(*args)
    torch.cuda.synchronize()
    got = getattr(PowerPaintController(pipe, version, control, loader, annotators), method)(*args)
    return got, want


@pytest.mark.parametrize("version", ["ppt-v1", "ppt-v2"])
@pytest.mark.parametrize("task", ["text-guided", "shape-guided", "object-removal", "image-outpainting"])
def test_predict_equals_the_app(pipes, task, version):
    ratios = (1.5, 1.25) if task == "image-outpainting" else (None, None)
    up = _upload(90, 70, seed=len(task))
    args = (up, "a cat", 0.6, 3, 7.5, 21, "dog", task, *ratios)
    got, want = _both(pipes, version, "predict", dict(up), *args[1:])
    _same(got, want)


@pytest.mark.parametrize("ratios", [(1, 2), (2, 1), (1, 1)])
def test_outpainting_ratios_equal_the_app(pipes, ratios):
    up = _upload(60, 80, seed=4)
    got, want = _both(pipes, "ppt-v1", "predict", dict(up), "sky", 1.0, 2, 7.5, 5, "", "image-outpainting", *ratios)
    _same(got, want)


def test_predict_controlnet_canny_equals_the_app(pipes):
    pytest.importorskip("cv2")
    loads = []
    up = _upload(100, 75, seed=8, mask_mode="L")
    ctrl = _upload(120, 90, seed=9)["image"]
    args = (dict(up), ctrl, "canny", "a chair", 3, 7.5, 33, "blurry", 0.8)
    got, want = _both(pipes, "ppt-v1", "predict_controlnet", *args, control=pipes["control"], loader=loads.append)
    _same(got, want)
    assert loads == []
    # an annotator's output is uploaded and resized on the device; a control-type change calls the loader
    pose = lambda im: im.resize((64, 48)).convert("L")  # noqa: E731
    args = (dict(up), ctrl, "pose", "a chair", 2, 7.5, 34, "blurry", 0.8)
    got, want = _both(pipes, "ppt-v1", "predict_controlnet", *args, control=pipes["control"], loader=loads.append,
                      annotators={"pose": pose})
    _same(got, want)
    assert loads == ["pose", "pose"]


def test_infer_equals_the_app(pipes):
    pytest.importorskip("cv2")
    from oracle.app_flow import AppFlowOracle
    from powerpaint_b200.controller import PowerPaintController

    up = _upload(80, 100, seed=12)
    common = dict(text_guided_prompt="a cat", text_guided_negative_prompt="dog", shape_guided_prompt="a chair",
                  shape_guided_negative_prompt="wall", fitting_degree=0.5, ddim_steps=2, scale=7.0, seed=3,
                  vertical_expansion_ratio=1.2, horizontal_expansion_ratio=1.2, outpaint_prompt="sky",
                  outpaint_negative_prompt="", removal_prompt="", removal_negative_prompt="photo")
    for version, task, control in [("ppt-v1", "object-removal", False), ("ppt-v2", "image-outpainting", False),
                                   ("ppt-v1", "text-guided", True)]:
        kw = dict(common, task=task, enable_control=control, input_control_image=up["image"], control_type="canny",
                  controlnet_conditioning_scale=0.7)
        want = AppFlowOracle(pipes[version], version, pipes["control"]).infer(dict(up), **kw)
        ctl = PowerPaintController(pipes[version], version, pipes["control"])
        got = ctl.infer(dict(up), **kw)
        _same(got, want)
        plan = ctl.prepare_request(dict(up), **kw)  # the two halves a batching server runs around its own loop
        _same(ctl.finish_request(ctl.run(plan), plan), want)
