"""CPU tests of the app's request path (DESIGN.md §6b): the NumPy models of oracle/imageops.py against Pillow and cv2
byte for byte, the controller's host tables and plans against the libraries and against oracle/app_flow.py, and
argument checks of the new C entry points, which fail before they touch a device."""
import ctypes as C
import os

import numpy as np
import pytest
from PIL import Image, ImageFilter

from oracle import imageops as O

HERE = os.path.dirname(os.path.abspath(__file__))
FILTERS = {"bilinear": Image.Resampling.BILINEAR, "bicubic": Image.Resampling.BICUBIC,
           "lanczos": Image.Resampling.LANCZOS}
# (in_h, in_w, out_h, out_w): downscales by 1.01x .. 12x, upscales, 1-pixel sides, one axis unchanged
RESIZE_SHAPES = [(101, 99, 100, 98), (240, 320, 20, 27), (480, 640, 640, 853), (1, 7, 5, 1), (9, 1, 1, 13),
                 (37, 53, 37, 200), (64, 64, 5, 64), (30, 31, 360, 20), (200, 300, 17, 25), (3024, 4032, 40, 336)]
BLUR_RADII = [0.5, 1, 2, 3, 4, 7.5]


def _image(rng, h, w, mode):
    return rng.integers(0, 256, (h, w) if mode == "L" else (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("name", sorted(FILTERS))
def test_resize_model_equals_pillow(name, mode):
    rng = np.random.default_rng(1)
    for h, w, oh, ow in RESIZE_SHAPES:
        a = _image(rng, h, w, mode)
        want = np.asarray(Image.fromarray(a).resize((ow, oh), FILTERS[name]))
        assert np.array_equal(O.resize(a, (ow, oh), name), want), (h, w, oh, ow)


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_gaussian_blur_model_equals_pillow(mode):
    rng = np.random.default_rng(2)
    for r in BLUR_RADII:
        a = _image(rng, 61, 47, mode)
        a[20:40, 10:30] = 255
        want = np.asarray(Image.fromarray(a).filter(ImageFilter.GaussianBlur(r)))
        assert np.array_equal(O.gaussian_blur(a, r), want), r


def _canny_cases():
    z = np.load(os.path.join(HERE, "golden", "canny_cases.npz"))
    n = len([k for k in z.files if k.startswith("in_")])
    return [(z[f"in_{i}"], *z[f"thr_{i}"], z[f"out_{i}"]) for i in range(n)]


def test_canny_model_equals_cv2_fixtures():
    cases = _canny_cases()
    assert len(cases) >= 20
    for img, lo, hi, want in cases:
        assert np.array_equal(O.canny(img, lo, hi), want), (img.shape, lo, hi)


def test_canny_model_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for h, w, c, lo, hi in [(1, 1, 1, 0, 0), (5, 3, 3, 10, 20), (64, 80, 1, 50, 150), (90, 70, 3, 150, 50),
                            (128, 96, 3, 30, 30)]:
        a = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
        a = (cv2.GaussianBlur(a, (5, 5), 1.2).reshape(h, w, c) if min(h, w) > 4 else a)
        a = a[..., 0] if c == 1 else a
        assert np.array_equal(O.canny(a, lo, hi), cv2.Canny(a, lo, hi)), (h, w, c, lo, hi)


@pytest.mark.parametrize("name", sorted(FILTERS))
def test_product_resample_tables_equal_the_model(name):
    """the controller's vectorised table builder == the scalar restatement pinned to Pillow above"""
    from powerpaint_b200.imageops import resample_tables

    for n_in, n_out in [(99, 98), (4032, 853), (3024, 640), (853, 848), (1, 5), (7, 1), (31, 360), (640, 17)]:
        bounds, k = resample_tables(n_in, n_out, FILTERS[name])
        xmin, kk = O.resample_coeffs(n_in, n_out, name)
        assert np.array_equal(bounds[:, 0], xmin)
        assert np.array_equal(k, kk[:, :k.shape[1]]) and not kk[:, k.shape[1]:].any()
        assert all(not k[i, n:].any() for i, n in enumerate(bounds[:, 1]))


def _lib():
    from powerpaint_b200 import _native as N

    return N, N.lib()


def test_gaussian_box_radius_is_pillows():
    N, lib = _lib()
    for r in [0.2, 0.5, 1, 1.5, 2, 3, 4, 7.5, 10, 33.3]:
        assert np.float32(lib.pp_gaussian_box_radius(r, 3)) == O.box_radius(r), r


def _fails(status, lib, words):
    assert status != 0
    msg = lib.pp_last_error().decode()
    assert all(w in msg for w in words), msg


def test_entry_points_reject_invalid_arguments_before_touching_the_device():
    N, lib = _lib()
    p = C.c_void_p(16)  # never dereferenced: every call below fails its argument checks first
    _fails(lib.pp_resample_u8(p, p, p, 0, 4, 2, 2, 3, p, p, 1, p, p, 1, None), lib, ["zero size"])
    _fails(lib.pp_resample_u8(None, p, p, 4, 4, 2, 2, 3, p, p, 1, p, p, 1, None), lib, ["null"])
    _fails(lib.pp_resample_u8(p, p, p, 4, 4, 2, 2, 4, p, p, 1, p, p, 1, None), lib, ["4 channels"])
    _fails(lib.pp_resample_u8(p, p, p, 4, 4, 4, 2, 3, None, p, 1, None, None, 0, None), lib, ["horizontal"])
    _fails(lib.pp_resample_u8(p, None, p, 4, 4, 2, 2, 3, p, p, 1, p, p, 1, None), lib, ["scratch"])
    _fails(lib.pp_box_blur_u8(p, C.c_void_p(32), C.c_void_p(48), 4, 0, 3, 1.0, 3, None), lib, ["zero size"])
    _fails(lib.pp_box_blur_u8(p, C.c_void_p(32), C.c_void_p(48), 4, 4, 2, 1.0, 3, None), lib, ["2 channels"])
    _fails(lib.pp_box_blur_u8(p, C.c_void_p(32), C.c_void_p(48), 4, 4, 3, 0.0, 3, None), lib, ["radius"])
    _fails(lib.pp_box_blur_u8(p, p, C.c_void_p(48), 4, 4, 3, 1.0, 3, None), lib, ["distinct"])
    assert lib.pp_canny_workspace_bytes(0, 5) == -1
    ws = lib.pp_canny_workspace_bytes(8, 8)
    _fails(lib.pp_canny_u8(p, p, None, ws, 8, 8, 3, 1.0, 2.0, None), lib, ["null"])
    _fails(lib.pp_canny_u8(p, p, p, ws, 0, 8, 3, 1.0, 2.0, None), lib, ["zero size"])
    _fails(lib.pp_canny_u8(p, p, p, ws, 8, 8, 4, 1.0, 2.0, None), lib, ["4 channels"])
    _fails(lib.pp_canny_u8(p, p, p, ws - 1, 8, 8, 3, 1.0, 2.0, None), lib, ["workspace"])
    _fails(lib.pp_canny_u8(p, p, p, ws, 8, 8, 1, float("nan"), 2.0, None), lib, ["thresholds"])
    _fails(lib.pp_outpaint_canvas_u8(p, 10, 10, p, p, 9, 20, 0, 0, 0, 0, 0, 0, None), lib, ["does not fit"])
    _fails(lib.pp_outpaint_canvas_u8(p, 10, 10, p, None, 20, 20, 0, 0, 0, 0, 0, 0, None), lib, ["null"])
    _fails(lib.pp_app_blend_u8(7, p, p, p, p, 4, 4, 3, None), lib, ["unknown op 7"])
    _fails(lib.pp_app_blend_u8(N.PP_BLEND_PASTE, p, p, None, p, 4, 4, 3, None), lib, ["null"])
    _fails(lib.pp_app_blend_u8(N.PP_BLEND_RED_OVERLAY, p, p, None, p, 4, 4, 2, None), lib, ["2 channels"])
    _fails(lib.pp_app_blend_u8(N.PP_BLEND_LUMA, p, None, None, p, 0, 4, 0, None), lib, ["zero size"])


# ---------------------------------------------------------------------------------------- controller plans
class _StubPipe:
    """records each call's keywords and returns a grey image of the requested size"""

    def __init__(self):
        self.calls = []

    def __call__(self, **kw):
        self.calls.append(kw)
        from types import SimpleNamespace

        return SimpleNamespace(images=[Image.new("RGB", (kw["width"], kw["height"]), (90, 120, 150))])


def _upload(w, h, seed=0, mask_mode="RGB"):
    rng = np.random.default_rng(seed)
    img = Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    m = np.zeros((h, w), np.uint8)
    m[h // 4:h // 2, w // 3:w // 2] = 255
    mask = Image.fromarray(m).convert(mask_mode)
    return {"image": img, "mask": mask}


INFER_TASKS = ["text-guided", "shape-guided", "object-removal", "image-outpainting", "something-else"]
RATIOS = [(1, 2), (2, 1), (1.5, 1.5), (1, 1)]


def _infer_args(task, ratio=(1, 2), enable_control=False, control_image=None, control_type="canny"):
    return dict(text_guided_prompt="a cat", text_guided_negative_prompt="dog", shape_guided_prompt="a chair",
                shape_guided_negative_prompt="wall", fitting_degree=0.7, ddim_steps=3, scale=6.5, seed=11, task=task,
                vertical_expansion_ratio=ratio[0], horizontal_expansion_ratio=ratio[1], outpaint_prompt="sky",
                outpaint_negative_prompt="blur", removal_prompt="", removal_negative_prompt="photo",
                enable_control=enable_control, input_control_image=control_image, control_type=control_type,
                controlnet_conditioning_scale=0.5)


def _expected_images(plan, upload, version):
    """the pipeline inputs the plan's geometry implies, built with PIL / NumPy on the host"""
    from powerpaint_b200.controller import short_side_size

    img = upload["image"].convert("RGB").resize(short_side_size(upload["image"].size, 640 if plan.canvas is None
                                                                 else 512))
    mask = upload["mask"]
    if plan.canvas is not None:
        c = plan.canvas
        canvas = np.full((c.height, c.width, 3), 127, np.uint8)
        a = np.asarray(img)
        canvas[c.top:c.top + a.shape[0], c.left:c.left + a.shape[1]] = a
        m = np.full((c.height, c.width, 3), 255, np.uint8)
        m[c.hole[0]:c.hole[1], c.hole[2]:c.hole[3]] = 0
        img, mask = Image.fromarray(canvas), Image.fromarray(m)
    img, mask = img.resize((plan.H, plan.W)), mask.resize((plan.H, plan.W))
    if version != "ppt-v1" and plan.kind == "predict":
        img = Image.fromarray((np.array(img) * (1 - np.array(mask) / 255.0)).astype(np.uint8))
    return img, mask


def _compare(plan, call, upload, version):
    images = {k: call.pop(k) for k in ("image", "mask", "control_image") if k in call}
    gen = call.pop("generator", None)
    assert (gen is not None) == (version != "ppt-v1" and plan.kind == "predict")
    assert plan.kwargs == call
    img, mask = _expected_images(plan, upload, version)
    assert np.array_equal(np.asarray(images["image"]), np.asarray(img.convert("RGB")))
    assert np.array_equal(np.asarray(images["mask"]), np.asarray(mask.convert("RGB")))


@pytest.mark.parametrize("version", ["ppt-v1", "ppt-v2"])
@pytest.mark.parametrize("task", INFER_TASKS)
def test_controller_plan_equals_the_app_flow(task, version, monkeypatch):
    import torch

    from oracle.app_flow import AppFlowOracle
    from powerpaint_b200.controller import PowerPaintController

    class _Gen:  # the v2 flow seeds a CUDA generator; the stub pipelines never draw from it
        def __init__(self, device):
            self.device = device

        def manual_seed(self, seed):
            self.seed = seed
            return self

    monkeypatch.setattr(torch, "Generator", _Gen)

    for size in [(96, 72), (60, 150)]:
        for ratio in (RATIOS if task == "image-outpainting" else [(None, None)]):
            upload = _upload(*size)
            pipe = _StubPipe()
            args = _infer_args(task, ratio)
            AppFlowOracle(pipe, version).infer(dict(upload), **args)
            plan = PowerPaintController(pipe, version).plan_request(dict(upload), **args)
            assert plan.kind == "predict" and plan.pipe_name == "pipe"
            assert (plan.canvas is not None) == (task == "image-outpainting")
            _compare(plan, pipe.calls[0], upload, version)


def test_controller_plan_equals_the_app_flow_controlnet():
    pytest.importorskip("cv2")
    from oracle.app_flow import AppFlowOracle
    from powerpaint_b200.controller import PowerPaintController

    loaded = []
    upload = _upload(120, 90, mask_mode="L")
    pipe, cpipe = _StubPipe(), _StubPipe()
    ctrl_img = _upload(50, 40, seed=3)["image"]
    args = _infer_args("text-guided", enable_control=True, control_image=ctrl_img)
    AppFlowOracle(pipe, "ppt-v1", cpipe, loaded.append).infer(dict(upload), **args)
    plan = PowerPaintController(pipe, "ppt-v1", cpipe, loaded.append).plan_request(dict(upload), **args)
    assert not pipe.calls and plan.kind == "predict_controlnet" and plan.pipe_name == "control_pipe"
    call = cpipe.calls[0]
    assert call["control_image"].size == (plan.H, plan.W)
    _compare(plan, call, upload, "ppt-v1")
    assert loaded == []  # canny is the controller's initial control type
    # v2 has no ControlNet path: the request goes to predict
    plan = PowerPaintController(pipe, "ppt-v2", cpipe).plan_request(dict(upload), **args)
    assert plan.kind == "predict"


def test_outpaint_canvas_geometry_cases():
    from powerpaint_b200.controller import outpaint_canvas

    c = outpaint_canvas((680, 512), 1, 2)
    assert (c.width, c.height, c.top, c.left, c.hole) == (1360, 512, 0, 340, (0, 512, 350, 1010))
    c = outpaint_canvas((680, 512), 2, 1)
    assert (c.width, c.height, c.top, c.left, c.hole) == (680, 1024, 256, 0, (266, 758, 0, 680))
    c = outpaint_canvas((680, 512), 1.5, 1.5)
    assert (c.width, c.height, c.top, c.left, c.hole) == (1020, 768, 128, 170, (138, 630, 180, 840))
    assert outpaint_canvas((680, 512), 1, 1).hole == (0, 0, 0, 0)
    with pytest.raises(ValueError, match="shrink"):
        outpaint_canvas((680, 512), 0.9, 1)


def test_missing_annotator_is_named_before_any_device_work():
    from powerpaint_b200.controller import PowerPaintController

    ctl = PowerPaintController(_StubPipe(), "ppt-v1", _StubPipe(), annotators={"pose": lambda im: im})
    upload = _upload(64, 64)
    for ctype, name in [("depth", "depth"), ("hed", "hed"), ("scribble", "hed")]:
        with pytest.raises(ValueError, match=repr(name)):
            ctl.prepare_request(dict(upload), **_infer_args("text-guided", enable_control=True,
                                                             control_image=upload["image"], control_type=ctype))
