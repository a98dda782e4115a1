"""ORACLE (test infrastructure, not product): the reference app's host-side request flow (ref:app.py:29-64,222-543)
restated with PIL, NumPy and cv2, over whatever pipelines it is given.

`AppFlowOracle(pipe, version, control_pipe, controlnet_loader, annotators)` has the app's `predict`,
`predict_controlnet` and `infer`: the same resizes, canvas, prompts, seeding, pipeline keywords (PIL images in, PIL
images out) and post-processing, so tests/test_app_flow_gpu.py can hold `powerpaint_b200.controller` to the app's
bytes over the same product pipelines. The Gradio UI, the model loading and the annotator networks are the app's own
and not restated: `controlnet_loader(control_type)` and `annotators[name](pil)` stand in for them.
"""
from __future__ import annotations

import random

import numpy as np
import torch
from PIL import Image, ImageFilter

_QUALITY = ", worst quality, low quality, normal quality, bad quality, blurry "


def seed_everything(seed):
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    np.random.seed(seed)
    random.seed(seed)


def task_prompts(prompt, negative_prompt, task, version):
    """(promptA, promptB, negative_promptA, negative_promptB) of a task"""
    v1 = version == "ppt-v1"
    if task in ("object-removal", "image-outpainting"):
        pos = "empty scene blur " + prompt if v1 else ""
        neg = negative_prompt if v1 else ""
        return pos + " P_ctxt", pos + " P_ctxt", neg + " P_obj", neg + " P_obj"
    pos = prompt if v1 else ""
    neg = negative_prompt + _QUALITY if v1 else ""
    if task == "shape-guided":
        return pos + " P_shape", pos + " P_ctxt", neg + "P_shape", neg + "P_ctxt"
    return pos + " P_obj", pos + " P_obj", neg + "P_obj", neg + "P_obj"


def _short_side(img, side):
    w, h = img.convert("RGB").size
    size = (side, int(h / w * side)) if w < h else (int(w / h * side), side)
    return img.convert("RGB").resize(size)


def _to_multiple_of_8(image, mask):
    a = np.array(image.convert("RGB"))
    rows, cols = a.shape[0] - a.shape[0] % 8, a.shape[1] - a.shape[1] % 8
    return image.resize((cols, rows)), mask.resize((cols, rows)), cols, rows


def _red_overlay(result, mask_rgb):
    m = mask_rgb.astype("float")
    red = np.array(result).astype("float")
    red[:, :, 0], red[:, :, 1], red[:, :, 2] = 180.0, 0, 0
    return Image.fromarray((np.array(result).astype("float") * (1 - m / 512.0) + m / 512.0 * red).astype("uint8"))


class AppFlowOracle:
    def __init__(self, pipe, version, control_pipe=None, controlnet_loader=None, annotators=None):
        self.pipe, self.version, self.control_pipe = pipe, version, control_pipe
        self.controlnet_loader = controlnet_loader
        self.annotators = annotators or {}
        self.current_control = "canny"

    def load_controlnet(self, control_type):
        if self.current_control != control_type:
            if self.controlnet_loader is not None:
                self.controlnet_loader(control_type)
            self.current_control = control_type

    def predict(self, input_image, prompt, fitting_degree, ddim_steps, scale, seed, negative_prompt, task,
                vertical_expansion_ratio, horizontal_expansion_ratio):
        image = _short_side(input_image["image"], 512 if task == "image-outpainting" else 640)
        mask = input_image["mask"]
        if vertical_expansion_ratio is not None and horizontal_expansion_ratio is not None:
            vr, hr = vertical_expansion_ratio, horizontal_expansion_ratio
            o_w, o_h = image.size
            c_w, c_h = int(hr * o_w), int(vr * o_h)
            top, left = int((c_h - o_h) / 2.0), int((c_w - o_w) / 2.0)
            canvas = np.full((c_h, c_w, 3), 127, np.uint8)
            canvas[top:top + o_h, left:left + o_w, :] = np.array(image)
            m = np.full((c_h, c_w, 3), 255, np.uint8)
            g = 10
            if vr == 1 and hr != 1:
                m[top:top + o_h, left + g:left + o_w - g, :] = 0
            elif vr != 1 and hr != 1:
                m[top + g:top + o_h - g, left + g:left + o_w - g, :] = 0
            elif vr != 1 and hr == 1:
                m[top + g:top + o_h - g, left:left + o_w, :] = 0
            image, mask = Image.fromarray(canvas), Image.fromarray(m)
        if self.version != "ppt-v1":
            prompt = prompt + {"image-outpainting": " empty scene", "object-removal": " empty scene blur"}.get(task, "")
        pa, pb, na, nb = task_prompts(prompt, negative_prompt, task, self.version)
        image, mask, H, W = _to_multiple_of_8(image, mask)
        seed_everything(seed)
        if self.version == "ppt-v1":
            result = self.pipe(promptA=pa, promptB=pb, tradoff=fitting_degree, tradoff_nag=fitting_degree,
                               negative_promptA=na, negative_promptB=nb, image=image.convert("RGB"),
                               mask=mask.convert("RGB"), width=H, height=W, guidance_scale=scale,
                               num_inference_steps=ddim_steps).images[0]
        else:
            filled = np.array(image) * (1 - np.array(mask) / 255.0)
            image = Image.fromarray(filled.astype(np.uint8)).convert("RGB")
            result = self.pipe(promptA=pa, promptB=pb, promptU=prompt, tradoff=fitting_degree,
                               tradoff_nag=fitting_degree, image=image.convert("RGB"), mask=mask.convert("RGB"),
                               num_inference_steps=ddim_steps, generator=torch.Generator("cuda").manual_seed(seed),
                               brushnet_conditioning_scale=1.0, negative_promptA=na, negative_promptB=nb,
                               negative_promptU=negative_prompt, guidance_scale=scale, width=H, height=W).images[0]
        result_m = _red_overlay(result, np.array(mask.convert("RGB")))
        return [result], [mask.convert("RGB"), result_m]

    def predict_controlnet(self, input_image, input_control_image, control_type, prompt, ddim_steps, scale, seed,
                           negative_prompt, controlnet_conditioning_scale):
        image = _short_side(input_image["image"], 640)
        image, mask, H, W = _to_multiple_of_8(image, input_image["mask"])
        if control_type != self.current_control:
            self.load_controlnet(control_type)
        if control_type == "canny":
            import cv2

            edges = cv2.Canny(np.array(input_control_image.resize((H, W))), 100, 200)[:, :, None]
            control = Image.fromarray(np.concatenate([edges] * 3, axis=2))
        elif control_type == "pose":
            control = self.annotators["pose"](input_control_image)
        elif control_type == "depth":
            control = self.annotators["depth"](input_control_image.resize((H, W)))
        else:
            control = self.annotators["hed"](input_control_image)
        mask_rgb = np.array(mask.convert("RGB"))
        control = control.resize((H, W))
        seed_everything(seed)
        result = self.control_pipe(promptA=prompt + " P_obj", promptB=prompt + " P_obj", tradoff=1.0, tradoff_nag=1.0,
                                   negative_promptA=negative_prompt, negative_promptB=negative_prompt,
                                   image=image.convert("RGB"), mask=mask.convert("RGB"), control_image=control,
                                   width=H, height=W, guidance_scale=scale,
                                   controlnet_conditioning_scale=controlnet_conditioning_scale,
                                   num_inference_steps=ddim_steps).images[0]
        result_m = _red_overlay(result, mask_rgb)
        mb = np.asarray(mask.convert("RGB").filter(ImageFilter.GaussianBlur(radius=4))) / 255.0
        ours = np.asarray(result) / 255.0 * mb + (1 - mb) * (np.asarray(image.convert("RGB")) / 255.0)
        return [image.convert("RGB"), Image.fromarray(np.uint8(ours * 255))], [control, result_m]

    def infer(self, input_image, text_guided_prompt, text_guided_negative_prompt, shape_guided_prompt,
              shape_guided_negative_prompt, fitting_degree, ddim_steps, scale, seed, task, vertical_expansion_ratio,
              horizontal_expansion_ratio, outpaint_prompt, outpaint_negative_prompt, removal_prompt,
              removal_negative_prompt, enable_control=False, input_control_image=None, control_type="canny",
              controlnet_conditioning_scale=None):
        if task == "image-outpainting":
            return self.predict(input_image, outpaint_prompt, fitting_degree, ddim_steps, scale, seed,
                                outpaint_negative_prompt, task, vertical_expansion_ratio, horizontal_expansion_ratio)
        if task == "shape-guided":
            prompt, negative_prompt = shape_guided_prompt, shape_guided_negative_prompt
        elif task == "object-removal":
            prompt, negative_prompt = removal_prompt, removal_negative_prompt
        else:
            task, prompt, negative_prompt = "text-guided", text_guided_prompt, text_guided_negative_prompt
        if self.version == "ppt-v1" and enable_control and task == "text-guided":
            return self.predict_controlnet(input_image, input_control_image, control_type, prompt, ddim_steps, scale,
                                           seed, negative_prompt, controlnet_conditioning_scale)
        return self.predict(input_image, prompt, fitting_degree, ddim_steps, scale, seed, negative_prompt, task, None,
                            None)

