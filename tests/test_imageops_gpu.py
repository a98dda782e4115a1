"""GPU tests of powerpaint_b200/imageops.py: resize and Gaussian blur equal live Pillow, Canny equals cv2 (fixtures,
and live when cv2 is installed), the app's per-pixel steps equal their NumPy expressions; byte for byte. Every
output is written between sentinel bytes that must survive, each op run twice gives identical bytes, and invalid
arguments raise."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageFilter

from powerpaint_b200 import _native as N
from powerpaint_b200 import imageops as io

pytestmark = pytest.mark.gpu

DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
PAD = 4096
SENTINEL = 0xA5
FILTERS = [Image.Resampling.BILINEAR, Image.Resampling.BICUBIC, Image.Resampling.LANCZOS]
RESIZE_SHAPES = [(101, 99, 100, 98), (240, 320, 20, 27), (480, 640, 640, 853), (1, 7, 5, 1), (9, 1, 1, 13),
                 (37, 53, 37, 200), (64, 64, 5, 64), (30, 31, 360, 20), (200, 300, 17, 25), (3024, 4032, 640, 848),
                 (640, 853, 640, 848), (3024, 4032, 640, 853), (50, 60, 50, 60)]


def _guarded(shape):
    """(buffer, view): `view` of `shape` inside a buffer of sentinel bytes"""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * PAD,), SENTINEL, dtype=torch.uint8, device=DEV)
    return buf, buf[PAD:PAD + n].view(*shape)


def _intact(buf, n):
    assert bool((buf[:PAD] == SENTINEL).all()) and bool((buf[PAD + n:] == SENTINEL).all()), "write outside the output"


def _dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a if a.ndim == 3 else a[..., None])).to(DEV)


def _host(t: torch.Tensor) -> np.ndarray:
    a = t.cpu().numpy()
    return a[..., 0] if a.shape[2] == 1 else a


def _pattern(rng, h, w, c):
    if h * w > 1 << 20:  # large uploads: a smooth photo-like field plus noise
        y, x = np.mgrid[0:h, 0:w]
        base = (np.sin(x / 37.0) * 60 + np.cos(y / 23.0) * 60 + 128)[..., None] + rng.normal(0, 12, (h, w, c))
        return np.clip(base, 0, 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w, c), dtype=np.uint8)


def _resize_guarded(src, ow, oh, resample):
    h, w, c = src.shape
    buf, out = _guarded((oh, ow, c))
    bx = kx = by = ky = None
    if ow != w:
        bx, kx = io._device_tables(w, ow, resample, src.device)
    if oh != h:
        by, ky = io._device_tables(h, oh, resample, src.device)
    tmp = torch.empty(h, ow, c, dtype=torch.uint8, device=DEV)
    N.check(N.lib().pp_resample_u8(N.ptr(src), N.ptr(tmp), N.ptr(out), h, w, oh, ow, c, N.ptr(bx), N.ptr(kx),
                                   0 if kx is None else kx.shape[1], N.ptr(by), N.ptr(ky),
                                   0 if ky is None else ky.shape[1], N.current_stream()), "resample")
    torch.cuda.synchronize()
    _intact(buf, out.numel())
    return out


@pytest.mark.parametrize("c", [1, 3])
@pytest.mark.parametrize("resample", FILTERS, ids=lambda f: f.name)
def test_resize_equals_pillow(resample, c):
    rng = np.random.default_rng(int(resample) * 10 + c)
    for h, w, oh, ow in RESIZE_SHAPES:
        a = _pattern(rng, h, w, c)
        pil = Image.fromarray(a if c == 3 else a[..., 0])
        want = np.asarray(pil.resize((ow, oh), resample))
        src = _dev(a)
        got = _resize_guarded(src, ow, oh, resample)
        assert np.array_equal(_host(got), want), (h, w, oh, ow)
        again = io.resize(src, (ow, oh), resample)
        assert torch.equal(got, again), "two runs differ"
        if (oh, ow) == (h, w):
            assert again.data_ptr() != src.data_ptr()  # a copy, as Pillow's


@pytest.mark.parametrize("c", [1, 3])
def test_gaussian_blur_equals_pillow(c):
    rng = np.random.default_rng(7 + c)
    for (h, w) in [(61, 47), (1, 9), (640, 848), (5, 1)]:
        for r in [0.5, 1, 2, 3, 4, 7.5]:
            a = _pattern(rng, h, w, c)
            a[h // 3:h // 2, w // 4:w // 2] = 255
            pil = Image.fromarray(a if c == 3 else a[..., 0])
            want = np.asarray(pil.filter(ImageFilter.GaussianBlur(r)))
            src = _dev(a)
            buf, out = _guarded(src.shape)
            tmp = torch.empty_like(src)
            box = N.lib().pp_gaussian_box_radius(r, 3)
            N.check(N.lib().pp_box_blur_u8(N.ptr(src), N.ptr(tmp), N.ptr(out), h, w, c, box, 3, N.current_stream()),
                    "box blur")
            torch.cuda.synchronize()
            _intact(buf, out.numel())
            assert np.array_equal(_host(out), want), (h, w, r)
            assert torch.equal(out, io.gaussian_blur(src, r)), "two runs differ"
    src = _dev(_pattern(rng, 8, 8, c))
    assert torch.equal(io.gaussian_blur(src, 0), src)


def _canny_guarded(src, lo, hi):
    h, w, c = src.shape
    buf, out = _guarded((h, w, 1))
    nbytes = N.lib().pp_canny_workspace_bytes(h, w)
    wbuf, ws = _guarded((nbytes,))
    N.check(N.lib().pp_canny_u8(N.ptr(src), N.ptr(out), N.ptr(ws), nbytes, h, w, c, lo, hi, N.current_stream()),
            "canny")
    torch.cuda.synchronize()
    _intact(buf, out.numel())
    _intact(wbuf, nbytes)
    return out


def test_canny_equals_cv2_fixtures():
    z = np.load(os.path.join(HERE, "golden", "canny_cases.npz"))
    n = len([k for k in z.files if k.startswith("in_")])
    assert n >= 20
    for i in range(n):
        img, (lo, hi), want = z[f"in_{i}"], z[f"thr_{i}"], z[f"out_{i}"]
        src = _dev(img)
        got = _canny_guarded(src, float(lo), float(hi))
        assert np.array_equal(_host(got), want), (i, img.shape, lo, hi)
        assert torch.equal(got, io.canny(src, lo, hi)), "two runs differ"


def test_canny_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    for (h, w, c, lo, hi) in [(640, 848, 3, 100, 200), (853, 640, 1, 30, 90), (333, 517, 3, 0, 0),
                              (64, 2048, 3, 40, 40), (2048, 33, 1, 250, 20)]:
        a = _pattern(rng, h, w, c)
        a = cv2.GaussianBlur(a, (5, 5), 1.0).reshape(h, w, c)
        img = a if c == 3 else a[..., 0]
        got = _canny_guarded(_dev(img), lo, hi)
        assert np.array_equal(_host(got), cv2.Canny(img, lo, hi)), (h, w, c, lo, hi)


def test_app_blends_equal_numpy():
    rng = np.random.default_rng(5)
    h, w = 67, 91
    res = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    mask3 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    mask3[:10] = 255
    mask3[10:20] = 0
    mask1 = mask3[..., :1].copy()
    d = {k: _dev(v) for k, v in dict(res=res, img=img, mask3=mask3, mask1=mask1).items()}
    red = res.astype("float") * 1
    red[:, :, 0], red[:, :, 1], red[:, :, 2] = 180.0, 0, 0
    for m, dm in ((mask3, d["mask3"]), (np.repeat(mask1, 3, 2), d["mask1"])):
        cases = [
            (N.PP_BLEND_HOLE_FILL, d["img"], dm, None, (img * (1 - m / 255.0)).astype(np.uint8)),
            (N.PP_BLEND_RED_OVERLAY, d["res"], dm, None,
             (res.astype("float") * (1 - m.astype("float") / 512.0) + m.astype("float") / 512.0 * red).astype("uint8")),
            (N.PP_BLEND_PASTE, d["res"], dm, d["img"],
             np.uint8((res / 255.0 * (m / 255.0) + (1 - m / 255.0) * (img / 255.0)) * 255)),
        ]
        for op, a, b, c, want in cases:
            buf, out = _guarded((h, w, 3))
            N.check(N.lib().pp_app_blend_u8(op, N.ptr(a), N.ptr(b), N.ptr(c), N.ptr(out), h, w, b.shape[2],
                                            N.current_stream()), "blend")
            torch.cuda.synchronize()
            _intact(buf, out.numel())
            assert np.array_equal(_host(out), want), op
            again = {N.PP_BLEND_HOLE_FILL: lambda: io.hole_fill(a, b), N.PP_BLEND_RED_OVERLAY: lambda: io.red_overlay(a, b),
                     N.PP_BLEND_PASTE: lambda: io.paste_back(a, b, c)}[op]()
            assert torch.equal(out, again), "two runs differ"
    want = np.asarray(Image.fromarray(mask3).convert("L"))
    assert np.array_equal(_host(io.luma(d["mask3"])), want)


def test_outpaint_canvas_and_host_transfers():
    rng = np.random.default_rng(6)
    a = rng.integers(0, 256, (40, 50, 3), dtype=np.uint8)
    src = io.to_device(Image.fromarray(a))
    assert src.is_cuda and src.shape == (40, 50, 3)
    img_buf, img = _guarded((70, 90, 3))
    mask_buf, mask = _guarded((70, 90, 3))
    N.check(N.lib().pp_outpaint_canvas_u8(N.ptr(src), 40, 50, N.ptr(img), N.ptr(mask), 70, 90, 15, 20, 25, 45, 30,
                                          60, N.current_stream()), "canvas")
    torch.cuda.synchronize()
    _intact(img_buf, img.numel())
    _intact(mask_buf, mask.numel())
    want = np.full((70, 90, 3), 127, np.uint8)
    want[15:55, 20:70] = a
    wm = np.full((70, 90, 3), 255, np.uint8)
    wm[25:45, 30:60] = 0
    assert np.array_equal(img.cpu().numpy(), want) and np.array_equal(mask.cpu().numpy(), wm)
    i2, m2 = io.outpaint_canvas(src, (70, 90), (15, 20), (25, 45, 30, 60))
    assert torch.equal(i2, img) and torch.equal(m2, mask)
    # to_device / to_pil: RGB, L, RGBA (alpha dropped); other modes are refused by name
    assert np.array_equal(np.asarray(io.to_pil(src)), a)
    gray = Image.fromarray(a[..., 0])
    assert io.to_device(gray).shape == (40, 50, 1) and io.to_pil(io.to_device(gray)).mode == "L"
    rgba = Image.fromarray(np.concatenate([a, a[..., :1]], 2), "RGBA")
    assert np.array_equal(io.to_device(rgba).cpu().numpy(), a)
    with pytest.raises(ValueError, match="'CMYK'"):
        io.to_device(Image.fromarray(a).convert("CMYK"))


def test_invalid_arguments_raise():
    x = torch.zeros(8, 8, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError, match="CUDA"):
        io.resize(x.cpu(), (4, 4))
    with pytest.raises(TypeError, match="uint8"):
        io.resize(x.float(), (4, 4))
    with pytest.raises(ValueError, match="1 or 3 channels"):
        io.resize(torch.zeros(8, 8, 4, dtype=torch.uint8, device=DEV), (4, 4))
    with pytest.raises(ValueError, match="zero size"):
        io.resize(torch.zeros(0, 8, 3, dtype=torch.uint8, device=DEV), (4, 4))
    with pytest.raises(ValueError, match="positive"):
        io.resize(x, (0, 4))
    for bad in (Image.Resampling.NEAREST, Image.Resampling.BOX, Image.Resampling.HAMMING, 17):
        with pytest.raises(ValueError, match="unsupported resample"):
            io.resize(x, (4, 4), bad)
    with pytest.raises(ValueError, match="contiguous"):
        io.gaussian_blur(x.transpose(0, 1), 2)
    with pytest.raises(ValueError, match="radius"):
        io.gaussian_blur(x, -1)
    with pytest.raises(ValueError, match="thresholds"):
        io.canny(x, float("inf"), 3)
    with pytest.raises(ValueError, match="differ in size"):
        io.red_overlay(x, torch.zeros(4, 8, 3, dtype=torch.uint8, device=DEV))
    with pytest.raises(ValueError, match="RGB"):
        io.luma(torch.zeros(8, 8, 1, dtype=torch.uint8, device=DEV))
    with pytest.raises(RuntimeError, match="does not fit"):
        io.outpaint_canvas(x, (4, 4), (0, 0), (0, 0, 0, 0))
    with pytest.raises(RuntimeError, match="2 channels"):
        N.check(N.lib().pp_app_blend_u8(N.PP_BLEND_HOLE_FILL, N.ptr(x), N.ptr(x), None, N.ptr(x), 8, 8, 2,
                                        N.current_stream()), "blend")
    with pytest.raises(RuntimeError, match="null"):
        N.check(N.lib().pp_resample_u8(N.ptr(x), None, None, 8, 8, 4, 4, 3, None, None, 0, None, None, 0,
                                       C.c_void_p(N.current_stream())), "resample")
