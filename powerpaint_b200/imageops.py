"""The app's image operations on the device, byte-exact to the libraries the app calls (DESIGN.md §6b).

Images are CUDA uint8 HWC tensors [h, w, c] with c = 1 (Pillow mode L) or 3 (RGB). Every op runs on torch's current
stream through the C ABI (`pp_resample_u8`, `pp_box_blur_u8`, `pp_canny_u8`, `pp_outpaint_canvas_u8`,
`pp_app_blend_u8`); there is no host fallback.

- `resize` = `PIL.Image.resize` (BILINEAR, BICUBIC or LANCZOS), `gaussian_blur` = `ImageFilter.GaussianBlur`,
  `canny` = `cv2.Canny` (aperture 3, L1 norm).
- `to_device` / `to_pil` move a PIL image across PCIe once each way.
- `outpaint_canvas`, `luma`, `hole_fill`, `red_overlay` and `paste_back` are the app's own per-pixel steps
  (ref:app.py:276-307,342-345,365-381,466-472).
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import numpy as np
import PIL.Image
import torch

from . import _native as N

_PRECISION_BITS = 22  # Pillow's fixed-point precision for 8-bit resampling

_RESAMPLE = {PIL.Image.Resampling.BILINEAR: ("bilinear", 1.0), PIL.Image.Resampling.BICUBIC: ("bicubic", 2.0),
             PIL.Image.Resampling.LANCZOS: ("lanczos", 3.0)}


def _filter(name: str, x: np.ndarray) -> np.ndarray:
    """Pillow's filter functions, elementwise in float64 with Pillow's operation order"""
    if name == "bilinear":
        x = np.abs(x)
        return np.where(x < 1.0, 1.0 - x, 0.0)
    if name == "bicubic":
        a = -0.5
        x = np.abs(x)
        return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                        np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))

    def sinc(v: float) -> float:  # math.sin: the C library's sin, as Pillow's
        if v == 0.0:
            return 1.0
        v = v * math.pi
        return math.sin(v) / v

    return np.array([sinc(v) * sinc(v / 3) if -3.0 <= v < 3.0 else 0.0 for v in x.ravel()]).reshape(x.shape)


def resample_tables(in_size: int, out_size: int, resample) -> Tuple[np.ndarray, np.ndarray]:
    """Pillow's `precompute_coeffs` + `normalize_coeffs_8bpc` for one axis: bounds int32 [out, 2] = (first source
    pixel, tap count) and k int32 [out, taps] in 22-bit fixed point (zero past a pixel's tap count)"""
    name, support0 = _RESAMPLE[resample]
    scale = float(in_size) / out_size
    fs = max(scale, 1.0)
    support = support0 * fs
    ss = 1.0 / fs
    center = (np.arange(out_size) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)
    n = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    taps = int(n.max())
    t = np.arange(taps)
    valid = t[None, :] < n[:, None]
    w = np.where(valid, _filter(name, ((t[None, :] + xmin[:, None]) - center[:, None] + 0.5) * ss), 0.0)
    total = np.zeros(out_size)
    for j in range(taps):  # Pillow's sequential sum
        total = total + w[:, j]
    w = np.where(total[:, None] != 0.0, w / np.where(total == 0.0, 1.0, total)[:, None], w)
    q = np.where(w < 0, -0.5 + w * (1 << _PRECISION_BITS), 0.5 + w * (1 << _PRECISION_BITS)).astype(np.int64)
    return np.stack([xmin, n], 1).astype(np.int32), q.astype(np.int32)


_TABLES: Dict[tuple, Tuple[torch.Tensor, torch.Tensor]] = {}


def _device_tables(in_size: int, out_size: int, resample, device) -> Tuple[torch.Tensor, torch.Tensor]:
    key = (in_size, out_size, resample, device)
    if key not in _TABLES:
        b, k = resample_tables(in_size, out_size, resample)
        _TABLES[key] = (torch.from_numpy(b).to(device), torch.from_numpy(k).to(device))
    return _TABLES[key]


def _check_image(u8: torch.Tensor, name: str = "image") -> Tuple[int, int, int]:
    if not torch.is_tensor(u8) or not u8.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if u8.dtype != torch.uint8:
        raise TypeError(f"{name} must be uint8, got {u8.dtype}")
    if u8.ndim != 3 or u8.shape[2] not in (1, 3):
        raise ValueError(f"{name} must be HWC with 1 or 3 channels, got shape {tuple(u8.shape)}")
    if not u8.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    h, w, c = u8.shape
    if h == 0 or w == 0:
        raise ValueError(f"{name} has a zero size: {tuple(u8.shape)}")
    return h, w, c


def resize(u8: torch.Tensor, size, resample=PIL.Image.Resampling.BICUBIC) -> torch.Tensor:
    """`Image.resize(size=(w, h), resample)`; a copy when the size is unchanged, as Pillow's"""
    h, w, c = _check_image(u8)
    ow, oh = (int(v) for v in size)
    if ow <= 0 or oh <= 0:
        raise ValueError(f"resize: target size {size} must be positive")
    try:
        resample = PIL.Image.Resampling(resample)
    except ValueError:
        raise ValueError(f"resize: unsupported resample filter {resample!r}") from None
    if resample not in _RESAMPLE:
        raise ValueError(f"resize: unsupported resample filter {resample.name} (BILINEAR, BICUBIC or LANCZOS)")
    out = torch.empty(oh, ow, c, dtype=torch.uint8, device=u8.device)
    bx = kx = by = ky = None
    if ow != w:
        bx, kx = _device_tables(w, ow, resample, u8.device)
    if oh != h:
        by, ky = _device_tables(h, oh, resample, u8.device)
    tmp = torch.empty(h, ow, c, dtype=torch.uint8, device=u8.device) if (ow != w and oh != h) else None
    N.check(N.lib().pp_resample_u8(N.ptr(u8), N.ptr(tmp), N.ptr(out), h, w, oh, ow, c, N.ptr(bx), N.ptr(kx),
                                   0 if kx is None else kx.shape[1], N.ptr(by), N.ptr(ky),
                                   0 if ky is None else ky.shape[1], N.current_stream(u8.device)), "pp_resample_u8")
    return out


def gaussian_blur(u8: torch.Tensor, radius: float) -> torch.Tensor:
    """`Image.filter(ImageFilter.GaussianBlur(radius))`: three box passes per axis; radius 0 is a copy"""
    h, w, c = _check_image(u8)
    radius = float(radius)
    if not radius >= 0 or math.isinf(radius):
        raise ValueError(f"gaussian_blur: radius {radius} must be finite and >= 0")
    if radius == 0:
        return u8.clone()
    box = N.lib().pp_gaussian_box_radius(radius, 3)
    out = torch.empty_like(u8)
    tmp = torch.empty_like(u8)
    N.check(N.lib().pp_box_blur_u8(N.ptr(u8), N.ptr(tmp), N.ptr(out), h, w, c, box, 3, N.current_stream(u8.device)),
            "pp_box_blur_u8")
    return out


def canny(u8: torch.Tensor, low: float, high: float) -> torch.Tensor:
    """`cv2.Canny(img, low, high)` (aperture 3, L1 gradient) -> uint8 [h, w, 1] in {0, 255}"""
    h, w, c = _check_image(u8)
    low, high = float(low), float(high)
    if not (math.isfinite(low) and math.isfinite(high)):
        raise ValueError(f"canny: thresholds ({low}, {high}) must be finite")
    nbytes = N.lib().pp_canny_workspace_bytes(h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=u8.device)
    out = torch.empty(h, w, 1, dtype=torch.uint8, device=u8.device)
    N.check(N.lib().pp_canny_u8(N.ptr(u8), N.ptr(out), N.ptr(ws), nbytes, h, w, c, low, high,
                                N.current_stream(u8.device)), "pp_canny_u8")
    return out


def to_device(pil: PIL.Image.Image, device=None) -> torch.Tensor:
    """One upload through pinned memory: mode RGB -> [h, w, 3], L -> [h, w, 1]; RGBA drops alpha, which is what
    `convert("RGB")` does"""
    if pil.mode not in ("RGB", "L", "RGBA"):
        raise ValueError(f"to_device: image mode {pil.mode!r} is not supported (RGB, RGBA or L)")
    a = np.asarray(pil)
    if a.ndim == 2:
        a = a[..., None]
    elif pil.mode == "RGBA":
        a = a[..., :3]
    host = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
    host.numpy()[...] = a
    return host.to(device or torch.device("cuda", torch.cuda.current_device()), non_blocking=True)


def to_pil(u8: torch.Tensor) -> PIL.Image.Image:
    """One download: [h, w, 3] -> RGB, [h, w, 1] -> L"""
    _check_image(u8)
    a = u8.cpu().numpy()
    return PIL.Image.fromarray(a[..., 0] if a.shape[2] == 1 else a)


def outpaint_canvas(u8: torch.Tensor, canvas_hw: Tuple[int, int], top_left: Tuple[int, int],
                    hole: Tuple[int, int, int, int]) -> Tuple[torch.Tensor, torch.Tensor]:
    """(image, mask), both RGB [c_h, c_w, 3]: the canvas filled with 127 and `u8` at top_left, the mask 255 with
    rows hole[0]:hole[1] x columns hole[2]:hole[3] set to 0"""
    h, w, c = _check_image(u8)
    if c != 3:
        raise ValueError("outpaint_canvas: the image must be RGB")
    ch, cw = canvas_hw
    img = torch.empty(ch, cw, 3, dtype=torch.uint8, device=u8.device)
    mask = torch.empty_like(img)
    N.check(N.lib().pp_outpaint_canvas_u8(N.ptr(u8), h, w, N.ptr(img), N.ptr(mask), ch, cw, top_left[0], top_left[1],
                                          *hole, N.current_stream(u8.device)), "pp_outpaint_canvas_u8")
    return img, mask


def _blend(op: int, a: torch.Tensor, b=None, c=None) -> torch.Tensor:
    h, w, ca = _check_image(a, "a")
    if ca != 3:
        raise ValueError("the image must be RGB")
    bc = 0
    for t in (b, c):
        if t is not None and tuple(_check_image(t)[:2]) != (h, w):
            raise ValueError(f"operands differ in size: {tuple(a.shape)} vs {tuple(t.shape)}")
    if b is not None:
        bc = b.shape[2]
    if c is not None and c.shape[2] != 3:
        raise ValueError("the image must be RGB")
    out = torch.empty(h, w, 1 if op == N.PP_BLEND_LUMA else 3, dtype=torch.uint8, device=a.device)
    N.check(N.lib().pp_app_blend_u8(op, N.ptr(a), N.ptr(b), N.ptr(c), N.ptr(out), h, w, bc,
                                    N.current_stream(a.device)), "pp_app_blend_u8")
    return out


def luma(rgb: torch.Tensor) -> torch.Tensor:
    """`convert("L")` of an RGB image -> [h, w, 1]"""
    return _blend(N.PP_BLEND_LUMA, rgb)


def hole_fill(img: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """`(img * (1 - mask / 255.0)).astype(np.uint8)` (the v2 app's masked input)"""
    return _blend(N.PP_BLEND_HOLE_FILL, img, mask)


def red_overlay(res: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """the app's mask preview: `res * (1 - mask / 512.0) + mask / 512.0 * red`, red = (180, 0, 0)"""
    return _blend(N.PP_BLEND_RED_OVERLAY, res, mask)


def paste_back(res: torch.Tensor, blurred_mask: torch.Tensor, img: torch.Tensor) -> torch.Tensor:
    """`np.uint8((res / 255.0 * mb + (1 - mb) * img / 255.0) * 255)` with mb = blurred_mask / 255.0"""
    return _blend(N.PP_BLEND_PASTE, res, blurred_mask, img)
