"""`PowerPaintController`: the app's request handling (ref:app.py:29-64,245-543) around the kernel-backed pipelines,
with every image step on the device (DESIGN.md §6b).

The app resizes the upload and the mask with Pillow, builds the outpainting canvas and the v2 hole fill with NumPy,
runs `cv2.Canny` for the ControlNet, and makes the red mask preview and the Gaussian-blurred paste-back on the host.
Here the upload crosses PCIe once, each of those steps is one of `imageops`' byte-exact kernels, the pipelines take
the uint8 CUDA tensors their PIL path would have built (`output_type="uint8"` leaves the result on the device), and
the returned PIL images are the only downloads. The returned lists equal the app's own, byte for byte, over the same
pipelines and seeds.

Gradio stays with the app: swap its `PowerPaintController` for this one (INTEGRATION.md E). The pose, HED and depth
annotators are networks the app loads itself; pass them as `annotators={"pose": f, "hed": f, "depth": f}` (PIL in,
PIL out). `controlnet_loader(control_type)` swaps the ControlNet, as the app's `load_controlnet` does.

A server that batches requests (`RequestBatcher`, INTEGRATION.md D) runs the two halves around its own loop:
`plan = prepare_request(...)`, `plan.pipe(**plan.kwargs)` (or `batcher(**plan.kwargs)`), `finish_request(result, plan)`.
"""
from __future__ import annotations

import inspect
import random
from dataclasses import dataclass, field
from typing import Callable, Dict, Optional, Tuple

import numpy as np
import torch

from . import imageops as io

BLURRY_GAP = 10  # px of the canvas mask that overlap the original image (ref:app.py:284)


def set_seed(seed: int) -> None:
    """the app's `set_seed` (ref:app.py:29-34)"""
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    np.random.seed(seed)
    random.seed(seed)


def add_task(prompt: str, negative_prompt: str, control_type: str, version: str) -> Tuple[str, str, str, str]:
    """the task prompts (ref:app.py:37-64): (promptA, promptB, negative_promptA, negative_promptB)"""
    pos = neg = ""
    v1 = version == "ppt-v1"
    quality = ", worst quality, low quality, normal quality, bad quality, blurry "
    if control_type in ("object-removal", "image-outpainting"):
        if v1:
            pos, neg = "empty scene blur " + prompt, negative_prompt
        return pos + " P_ctxt", pos + " P_ctxt", neg + " P_obj", neg + " P_obj"
    if control_type == "shape-guided":
        if v1:
            pos, neg = prompt, negative_prompt + quality
        return pos + " P_shape", pos + " P_ctxt", neg + "P_shape", neg + "P_ctxt"
    if v1:
        pos, neg = prompt, negative_prompt + quality
    return pos + " P_obj", pos + " P_obj", neg + "P_obj", neg + "P_obj"


def short_side_size(size: Tuple[int, int], side: int) -> Tuple[int, int]:
    """the app's resize target: the short side to `side`, the long side scaled and truncated"""
    w, h = size
    return (side, int(h / w * side)) if w < h else (int(w / h * side), side)


def _span(n: int, start: int, stop: int) -> Tuple[int, int]:
    """[start, stop) of the NumPy slice a[start:stop] over n elements (negative ends count from the end)"""
    r = range(n)[start:stop]
    return (r.start, r.stop) if len(r) else (0, 0)


@dataclass
class Canvas:
    """the outpainting canvas (ref:app.py:271-307): size, where the image goes, the mask's zero rectangle"""
    width: int
    height: int
    top: int
    left: int
    hole: Tuple[int, int, int, int]  # rows [0]:[1], columns [2]:[3]


def outpaint_canvas(size: Tuple[int, int], vertical_ratio: float, horizontal_ratio: float) -> Canvas:
    o_w, o_h = size
    c_w, c_h = int(horizontal_ratio * o_w), int(vertical_ratio * o_h)
    if c_w < o_w or c_h < o_h:
        raise ValueError(f"expansion ratios ({vertical_ratio}, {horizontal_ratio}) shrink the {o_w}x{o_h} image")
    top, left = int((c_h - o_h) / 2.0), int((c_w - o_w) / 2.0)
    g = BLURRY_GAP
    if vertical_ratio == 1 and horizontal_ratio != 1:
        rows, cols = (top, top + o_h), (left + g, left + o_w - g)
    elif vertical_ratio != 1 and horizontal_ratio != 1:
        rows, cols = (top + g, top + o_h - g), (left + g, left + o_w - g)
    elif vertical_ratio != 1 and horizontal_ratio == 1:
        rows, cols = (top + g, top + o_h - g), (left, left + o_w)
    else:  # (1, 1): the app leaves the whole mask at 255
        rows, cols = (0, 0), (0, 0)
    return Canvas(c_w, c_h, top, left, _span(c_h, *rows) + _span(c_w, *cols))


@dataclass
class RequestPlan:
    """What one request does, decided on the host from the upload's size and the request's parameters. `kwargs` are
    the pipeline call's keywords; `prepare_request` adds the images to them."""
    kind: str  # "predict" or "predict_controlnet"
    version: str
    task: str
    resized: Tuple[int, int]  # (w, h) after the short-side resize
    canvas: Optional[Canvas]
    H: int  # the app's naming: H is the width, W the height (both multiples of 8)
    W: int
    pipe_name: str  # "pipe" or "control_pipe"
    kwargs: dict
    seed: int
    control_type: Optional[str] = None
    state: dict = field(default_factory=dict)

    @property
    def pipe(self):
        return self.state["pipe"]


class PowerPaintController:
    """The app's controller (ref:app.py:83-543) over already-built pipelines: `predict`, `predict_controlnet` and
    `infer` take the app's parameters and return the app's lists of PIL images."""

    def __init__(self, pipe, version: str, control_pipe=None, controlnet_loader: Optional[Callable] = None,
                 annotators: Optional[Dict[str, Callable]] = None):
        self.pipe, self.version, self.control_pipe = pipe, version, control_pipe
        self.controlnet_loader = controlnet_loader
        self.annotators = dict(annotators or {})
        self.current_control = "canny"

    # ------------------------------------------------------------------ host plans
    def plan_predict(self, image_size, prompt, fitting_degree, ddim_steps, scale, seed, negative_prompt, task,
                     vertical_expansion_ratio, horizontal_expansion_ratio) -> RequestPlan:
        side = 512 if task == "image-outpainting" else 640
        resized = short_side_size(image_size, side)
        canvas = None
        if vertical_expansion_ratio is not None and horizontal_expansion_ratio is not None:
            canvas = outpaint_canvas(resized, vertical_expansion_ratio, horizontal_expansion_ratio)
        if self.version != "ppt-v1":
            if task == "image-outpainting":
                prompt = prompt + " empty scene"
            if task == "object-removal":
                prompt = prompt + " empty scene blur"
        pa, pb, na, nb = add_task(prompt, negative_prompt, task, self.version)
        w, h = (canvas.width, canvas.height) if canvas else resized
        H, W = w - w % 8, h - h % 8
        kw = dict(promptA=pa, promptB=pb, tradoff=fitting_degree, tradoff_nag=fitting_degree, negative_promptA=na,
                  negative_promptB=nb)
        if self.version == "ppt-v1":
            kw.update(width=H, height=W, guidance_scale=scale, num_inference_steps=ddim_steps)
        else:
            kw.update(promptU=prompt, num_inference_steps=ddim_steps, brushnet_conditioning_scale=1.0,
                      negative_promptU=negative_prompt, guidance_scale=scale, width=H, height=W)
        return RequestPlan("predict", self.version, task, resized, canvas, H, W, "pipe", kw, seed)

    def plan_controlnet(self, image_size, control_type, prompt, ddim_steps, scale, seed, negative_prompt,
                        controlnet_conditioning_scale) -> RequestPlan:
        resized = short_side_size(image_size, 640)
        H, W = resized[0] - resized[0] % 8, resized[1] - resized[1] % 8
        kw = dict(promptA=prompt + " P_obj", promptB=prompt + " P_obj", tradoff=1.0, tradoff_nag=1.0,
                  negative_promptA=negative_prompt, negative_promptB=negative_prompt, width=H, height=W,
                  guidance_scale=scale, controlnet_conditioning_scale=controlnet_conditioning_scale,
                  num_inference_steps=ddim_steps)
        return RequestPlan("predict_controlnet", self.version, "text-guided", resized, None, H, W, "control_pipe", kw,
                           seed, control_type)

    def plan_request(self, input_image, text_guided_prompt, text_guided_negative_prompt, shape_guided_prompt,
                     shape_guided_negative_prompt, fitting_degree, ddim_steps, scale, seed, task,
                     vertical_expansion_ratio, horizontal_expansion_ratio, outpaint_prompt, outpaint_negative_prompt,
                     removal_prompt, removal_negative_prompt, enable_control=False, input_control_image=None,
                     control_type="canny", controlnet_conditioning_scale=None) -> RequestPlan:
        """`infer`'s dispatch (ref:app.py:475-543) to the plan of `predict` or `predict_controlnet`"""
        size = input_image["image"].size
        if task == "image-outpainting":
            return self.plan_predict(size, outpaint_prompt, fitting_degree, ddim_steps, scale, seed,
                                     outpaint_negative_prompt, task, vertical_expansion_ratio,
                                     horizontal_expansion_ratio)
        prompts = {"text-guided": (text_guided_prompt, text_guided_negative_prompt),
                   "shape-guided": (shape_guided_prompt, shape_guided_negative_prompt),
                   "object-removal": (removal_prompt, removal_negative_prompt)}
        if task not in prompts:
            task = "text-guided"
        prompt, negative_prompt = prompts[task]
        if self.version == "ppt-v1" and enable_control and task == "text-guided":
            return self.plan_controlnet(size, control_type, prompt, ddim_steps, scale, seed, negative_prompt,
                                        controlnet_conditioning_scale)
        return self.plan_predict(size, prompt, fitting_degree, ddim_steps, scale, seed, negative_prompt, task, None,
                                 None)

    # ------------------------------------------------------------------ device halves
    def _prepare(self, plan: RequestPlan, input_image, input_control_image=None) -> RequestPlan:
        st = plan.state
        if plan.kind == "predict_controlnet":
            self._require_annotator(plan.control_type)
        image = _rgb(io.to_device(input_image["image"]))
        image = io.resize(image, plan.resized)
        mask = io.to_device(input_image["mask"])
        if plan.canvas is not None:
            c = plan.canvas
            image, mask = io.outpaint_canvas(image, (c.height, c.width), (c.top, c.left), c.hole)
        image = io.resize(image, (plan.H, plan.W))
        mask = io.resize(mask, (plan.H, plan.W))
        st.update(image=image, mask=mask)
        kw = dict(plan.kwargs, output_type="uint8")
        if plan.kind == "predict":
            if self.version == "ppt-v1":
                kw.update(image=_nchw(image), mask=_nchw(io.luma(mask) if mask.shape[2] == 3 else mask))
            else:
                image = io.hole_fill(image, mask)
                st["image"] = image
                kw.update(image=_unit(image), mask=_unit(_rgb(mask)),
                          generator=torch.Generator("cuda").manual_seed(plan.seed))
            st["pipe"] = self.pipe
        else:
            if plan.control_type != self.current_control:
                self.load_controlnet(plan.control_type)
            control = self._control_image(plan, input_control_image)
            control = io.resize(control, (plan.H, plan.W))
            st["control"] = control
            kw.update(image=_nchw(image), mask=_nchw(io.luma(mask) if mask.shape[2] == 3 else mask),
                      control_image=_nchw(_rgb(control)))
            st["pipe"] = self.control_pipe
        plan.kwargs = kw
        return plan

    def _require_annotator(self, control_type):
        if control_type != "canny":
            name = control_type if control_type in ("pose", "depth") else "hed"
            if name not in self.annotators:
                raise ValueError(f"control type {control_type!r} needs the {name!r} annotator: pass "
                                 f"annotators={{{name!r}: callable}} to PowerPaintController")

    def _control_image(self, plan: RequestPlan, pil):
        """the ControlNet condition before its final resize (ref:app.py:419-433)"""
        if plan.control_type == "canny":
            edges = io.canny(io.resize(io.to_device(pil), (plan.H, plan.W)), 100, 200)
            return edges.expand(-1, -1, 3).contiguous()
        if plan.control_type == "pose":
            return io.to_device(self.annotators["pose"](pil))
        if plan.control_type == "depth":
            small = io.to_pil(io.resize(io.to_device(pil), (plan.H, plan.W)))
            return io.to_device(self.annotators["depth"](small))
        return io.to_device(self.annotators["hed"](pil))

    def prepare_request(self, input_image, *args, **kwargs) -> RequestPlan:
        """`infer`'s arguments -> the plan, with its images uploaded and pre-processed on the device. Run
        `set_seed(plan.seed)` and `plan.pipe(**plan.kwargs)` (what `run` does), then `finish_request`."""
        bound = inspect.signature(self.plan_request).bind(input_image, *args, **kwargs)
        plan = self.plan_request(*bound.args, **bound.kwargs)
        return self._prepare(plan, input_image, bound.arguments.get("input_control_image"))

    @staticmethod
    def run(plan: RequestPlan):
        set_seed(plan.seed)
        return plan.pipe(**plan.kwargs).images

    def finish_request(self, result, plan: RequestPlan):
        """the pipeline's uint8 result ([1, h, w, 3] or [h, w, 3] on the device) -> the app's two lists of PIL
        images"""
        res = result[0] if result.ndim == 4 else result
        st = plan.state
        mask = _rgb(st["mask"])
        result_m = io.red_overlay(res, mask)
        if plan.kind == "predict":  # the app's paste-back here is dead code (ref:app.py:377-385)
            return [io.to_pil(res)], [io.to_pil(mask), io.to_pil(result_m)]
        paste = io.paste_back(res, io.gaussian_blur(mask, 4), st["image"])
        return [io.to_pil(st["image"]), io.to_pil(paste)], [io.to_pil(st["control"]), io.to_pil(result_m)]

    # ------------------------------------------------------------------ the app's methods
    def load_controlnet(self, control_type):
        """ref:app.py:222-243: a different ControlNet when the control type changes"""
        if self.current_control != control_type:
            if self.controlnet_loader is not None:
                self.controlnet_loader(control_type)
            self.current_control = control_type

    def predict(self, input_image, prompt, fitting_degree, ddim_steps, scale, seed, negative_prompt, task,
                vertical_expansion_ratio, horizontal_expansion_ratio):
        plan = self.plan_predict(input_image["image"].size, prompt, fitting_degree, ddim_steps, scale, seed,
                                 negative_prompt, task, vertical_expansion_ratio, horizontal_expansion_ratio)
        plan = self._prepare(plan, input_image)
        return self.finish_request(self.run(plan), plan)

    def predict_controlnet(self, input_image, input_control_image, control_type, prompt, ddim_steps, scale, seed,
                           negative_prompt, controlnet_conditioning_scale):
        plan = self.plan_controlnet(input_image["image"].size, control_type, prompt, ddim_steps, scale, seed,
                                    negative_prompt, controlnet_conditioning_scale)
        plan = self._prepare(plan, input_image, input_control_image)
        return self.finish_request(self.run(plan), plan)

    def infer(self, input_image, *args, **kwargs):
        plan = self.prepare_request(input_image, *args, **kwargs)
        return self.finish_request(self.run(plan), plan)


def _rgb(u8: torch.Tensor) -> torch.Tensor:
    """`convert("RGB")` of an L image (an RGB one is returned as is)"""
    return u8 if u8.shape[2] == 3 else u8.expand(-1, -1, 3).contiguous()


def _nchw(u8: torch.Tensor) -> torch.Tensor:
    """[h, w, c] -> the pipelines' uint8 [1, c, h, w]"""
    return u8.permute(2, 0, 1).unsqueeze(0).contiguous()


def _unit(u8: torch.Tensor) -> torch.Tensor:
    """[h, w, c] -> float32 [1, c, h, w] = u8 / 255, rounded as the BrushNet pipeline's PIL path rounds it (NumPy's
    true division). The pipeline's own uint8-tensor branch divides by a host scalar, which torch evaluates on the
    device as a multiplication by 1/255: one ulp apart on some values, and a different image after the loop."""
    x = _nchw(u8).float()
    return x / torch.full_like(x, 255.0)
