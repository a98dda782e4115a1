"""CPU tests of tiled VAE encode / decode (diffusers AutoencoderKL.enable_tiling): the host tile geometry against the
oracle's loops, the oracle's tiled path itself, the rounding rule the blend kernel reproduces, and the public API."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.vae_tiling import TiledAutoencoderKLOracle
from powerpaint_b200.models.autoencoder_kl import AutoencoderKL, vae_tile_geometry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(sample_size, f=0.25):
    om = TiledAutoencoderKLOracle(block_out_channels=(8, 8, 8, 8), norm_num_groups=4, layers_per_block=1,
                                   sample_size=sample_size)
    om.tile_overlap_factor = f
    return om.eval()


class _Recorder(nn.Module):
    """stand-in encoder / decoder: records (origin y, origin x, h, w) of each tile from the coordinate channels of
    its input and returns zeros of the output shape"""

    def __init__(self, calls, cout, size):
        super().__init__()
        self.calls, self.cout, self.size = calls, cout, size

    def forward(self, t):
        self.calls.append((int(t[0, 0, 0, 0]), int(t[0, 1, 0, 0]), t.shape[2], t.shape[3]))
        return torch.zeros(t.shape[0], self.cout, self.size(t.shape[2]), self.size(t.shape[3]))


def _trace(encode, h, w, sample_size, f=0.25):
    """tile origins / shapes, blend extents (in call order) and output shape of the oracle's tiled loop"""
    om = _oracle(sample_size, f)
    calls, blends = [], []
    if encode:
        om.encoder = _Recorder(calls, 8, lambda n: n // 8)
        om.quant_conv = nn.Identity()
    else:
        om.decoder = _Recorder(calls, 3, lambda n: n * 8)
        om.post_quant_conv = nn.Identity()
    bv, bh = om.blend_v, om.blend_h
    om.blend_v = lambda a, b, e: (blends.append(("v", min(a.shape[2], b.shape[2], e))), bv(a, b, e))[1]
    om.blend_h = lambda a, b, e: (blends.append(("h", min(a.shape[3], b.shape[3], e))), bh(a, b, e))[1]
    c = 3 if encode else 4
    x = torch.zeros(1, c, h, w)
    x[0, 0] = torch.arange(h, dtype=torch.float32)[:, None]
    x[0, 1] = torch.arange(w, dtype=torch.float32)[None, :]
    with torch.no_grad():
        if encode:
            out = om.tiled_encode(x).latent_dist.mean
        else:
            out = om.tiled_decode(x).sample
    return calls, blends, tuple(out.shape[2:])


def _check_geometry(encode, h, w, sample_size, f=0.25):
    lt = int(sample_size / 8)
    g = vae_tile_geometry(encode, h, w, sample_size, lt, f, 8)
    calls, blends, out_hw = _trace(encode, h, w, sample_size, f)
    assert [(t.y, t.x, t.h, t.w) for t in g.tiles] == calls, (encode, h, w)
    want = []
    for t in g.tiles:
        if t.row > 0:
            want.append(("v", t.blend_v))
        if t.col > 0:
            want.append(("h", t.blend_h))
    assert want == blends, (encode, h, w)
    assert (g.out_h, g.out_w) == out_hw, (encode, h, w)
    assert len(g.tiles) == g.rows * g.cols
    size = (lambda n: n // 8) if encode else (lambda n: n * 8)
    for t in g.tiles:
        assert (t.out_h, t.out_w) == (size(t.h), size(t.w))
    # the crops tile the output exactly once
    cover = np.zeros((g.out_h, g.out_w), dtype=np.int32)
    for t in g.tiles:
        cover[t.dst_y:t.dst_y + t.crop_h, t.dst_x:t.dst_x + t.crop_w] += 1
    assert (cover == 1).all()
    return g


LATENT_WIDTHS = (47, 48, 49, 63, 64, 65, 96, 100, 112, 341)


@pytest.mark.parametrize("w", LATENT_WIDTHS)
def test_decode_geometry_matches_oracle_loop(w):
    for h in (40, 64, 100, 170):
        _check_geometry(False, h, w, 512)


@pytest.mark.parametrize("w", LATENT_WIDTHS)
def test_encode_geometry_matches_oracle_loop(w):
    for h in (320, 512, 800, 1360):
        _check_geometry(True, h, 8 * w, 512)
    _check_geometry(True, 517, 8 * w + 3, 512)  # sides that are not multiples of 8


def test_geometry_custom_tile_size_and_overlap():
    for encode, h, w in ((False, 100, 70), (True, 800, 560), (False, 33, 129), (True, 264, 1032)):
        for ss, f in ((256, 0.25), (320, 0.25), (512, 0.5), (128, 0.125)):
            _check_geometry(encode, h, w, ss, f)


def test_geometry_of_the_app_canvases():
    """3:4 portrait expanded 2 x 2 and 4 x 4, and a 3:8 panorama (ref:app.py:258-307), SD-1.5 tiles (512 px, 64
    latent): output shapes equal the untiled ones, and at most 3 x 3 tile shapes"""
    for H, W in ((1360, 1024), (2728, 2048), (1704, 640)):
        ge = vae_tile_geometry(True, H, W, 512, 64, 0.25, 8)
        gd = vae_tile_geometry(False, H // 8, W // 8, 512, 64, 0.25, 8)
        assert (ge.out_h, ge.out_w) == (H // 8, W // 8) and (gd.out_h, gd.out_w) == (H, W)
        assert len(ge.groups()) <= 9 and len(gd.groups()) <= 9
    g = vae_tile_geometry(False, 100, 100, 512, 64, 0.25, 8)
    assert sorted({t.w for t in g.tiles}) == [4, 52, 64] and len(g.groups()) == 9


class _PointwiseDecoder(nn.Module):
    def __init__(self, g):
        super().__init__()
        self.mix = nn.Conv2d(4, 3, 1)
        with torch.no_grad():
            self.mix.weight.copy_(torch.randn(3, 4, 1, 1, generator=g))
            self.mix.bias.copy_(torch.randn(3, generator=g))

    def forward(self, z):
        return F.interpolate(self.mix(z), scale_factor=8.0, mode="nearest")


class _PointwiseEncoder(nn.Module):
    def __init__(self, g):
        super().__init__()
        self.mix = nn.Conv2d(3, 8, 1)
        with torch.no_grad():
            self.mix.weight.copy_(torch.randn(8, 3, 1, 1, generator=g))
            self.mix.bias.copy_(torch.randn(8, generator=g))

    def forward(self, x):
        return self.mix(F.avg_pool2d(x, 8))


@pytest.mark.parametrize("sample_size", [512, 256])
def test_oracle_tiled_equals_untiled_for_pointwise_nets(sample_size):
    """with an encoder / decoder that acts pixel by pixel every overlapping tile agrees, so blending changes nothing
    and the tiled result equals the untiled one: wrong origins, crops or extents would show"""
    g = torch.Generator().manual_seed(0)
    om = _oracle(sample_size)
    om.decoder, om.encoder = _PointwiseDecoder(g), _PointwiseEncoder(g)
    with torch.no_grad():
        for p in (om.quant_conv, om.post_quant_conv):
            p.weight.copy_(torch.randn(p.weight.shape, generator=g))
            p.bias.copy_(torch.randn(p.bias.shape, generator=g))
        for h, w in ((100, 70), (47, 113), (64, 65)):
            z = torch.randn(2, 4, h, w, generator=g)
            ref = om.decode(z).sample
            got = om.tiled_decode(z).sample
            assert got.shape == ref.shape
            assert torch.allclose(got, ref, rtol=1e-6, atol=1e-6), (got - ref).abs().max()
            x = torch.randn(2, 3, 8 * h, 8 * w, generator=g)
            ref = om.encode(x).latent_dist
            got = om.tiled_encode(x).latent_dist
            assert got.mean.shape == ref.mean.shape
            assert torch.allclose(got.mean, ref.mean, rtol=1e-6, atol=1e-6)
            assert torch.allclose(got.logvar, ref.logvar, rtol=1e-6, atol=1e-6)


def test_oracle_tiling_switch():
    """tiling on: at or below the tile size encode / decode return the untiled result exactly; above it they take
    the tiled loop"""
    om = TiledAutoencoderKLOracle.synthetic(tiny=True, sample_size=64)
    assert (om.tile_sample_min_size, om.tile_latent_min_size) == (64, 8)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for h, w in ((64, 64), (40, 64), (64, 24)):
            x = torch.rand(1, 3, h, w, generator=g) * 2 - 1
            z = torch.randn(1, 4, h // 8, w // 8, generator=g)
            om.disable_tiling()
            ref_m, ref_i = om.encode(x).latent_dist.mean, om.decode(z).sample
            om.enable_tiling()
            assert torch.equal(om.encode(x).latent_dist.mean, ref_m)
            assert torch.equal(om.decode(z).sample, ref_i)
        x = torch.rand(1, 3, 72, 64, generator=g) * 2 - 1
        z = torch.randn(1, 4, 9, 8, generator=g)
        assert torch.equal(om.encode(x).latent_dist.mean, om.tiled_encode(x).latent_dist.mean)
        assert torch.equal(om.decode(z).sample, om.tiled_decode(z).sample)
        om.disable_tiling()
        assert not torch.equal(om.decode(z).sample, om.tiled_decode(z).sample)


def test_blend_weights_are_fp32_roundings_of_the_double_expressions():
    """the rule pp_tile_blend implements: torch's `a * (1 - y/e) + b * (y/e)` with Python-float weights equals
    fp32(a * fp32(1 - y/e)) + fp32(b * fp32(y/e)), each step rounded to fp32 (no fused multiply-add)"""
    g = torch.Generator().manual_seed(2)
    om = _oracle(64)
    for e, ah, bh, w in ((128, 512, 512, 96), (16, 64, 40, 33), (7, 7, 9, 5), (3, 5, 3, 4)):
        a = torch.randn(2, 4, ah, w, generator=g) * 3
        b0 = torch.randn(2, 4, bh, w, generator=g) * 3
        got = om.blend_v(a, b0.clone(), e)
        ee = min(ah, bh, e)
        want = b0.numpy().copy()
        an = a.numpy()
        for y in range(ee):
            w0, w1 = np.float32(1 - y / ee), np.float32(y / ee)
            want[:, :, y, :] = (an[:, :, ah - ee + y, :] * w0).astype(np.float32) + (want[:, :, y, :] * w1).astype(np.float32)
        assert np.array_equal(got.numpy().view(np.int32), want.view(np.int32))
        got_h = om.blend_h(a.transpose(2, 3), b0.clone().transpose(2, 3), e)
        assert np.array_equal(got_h.transpose(2, 3).numpy().view(np.int32), want.view(np.int32))


def test_tiling_api_and_pipelines():
    from powerpaint_b200.pipelines import (StableDiffusionControlNetInpaintPipeline, StableDiffusionInpaintPipeline,
                                           StableDiffusionPowerPaintBrushNetPipeline)

    vae = AutoencoderKL.synthetic(tiny=True)
    assert (vae.use_tiling, vae.use_slicing) == (False, False)
    assert (vae.tile_sample_min_size, vae.tile_latent_min_size, vae.tile_overlap_factor) == (32, 4, 0.25)
    vae.enable_tiling()
    assert vae.use_tiling
    vae.disable_tiling()
    assert not vae.use_tiling
    vae.enable_tiling(False)
    assert not vae.use_tiling
    sd = AutoencoderKL(sample_size=512)
    assert (sd.tile_sample_min_size, sd.tile_latent_min_size) == (512, 64)
    assert AutoencoderKL(sample_size=[256, 256]).tile_latent_min_size == 32
    g = vae.tile_geometry(False, 10, 9)
    assert (g.out_h, g.out_w) == (80, 72) and g.rows == 4 and g.cols == 3
    pipes = (StableDiffusionInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=None, scheduler=None),
             StableDiffusionControlNetInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=None,
                                                      controlnet=None, scheduler=None),
             StableDiffusionPowerPaintBrushNetPipeline(vae=vae, text_encoder=None, text_encoder_brushnet=None,
                                                       tokenizer=None, unet=None, brushnet=None, scheduler=None))
    for p in pipes:
        p.enable_vae_tiling()
        assert vae.use_tiling
        p.disable_vae_tiling()
        assert not vae.use_tiling
    # the oracle VAE (what the CPU pipeline tests inject) answers the same calls
    om = TiledAutoencoderKLOracle.synthetic(tiny=True)
    StableDiffusionInpaintPipeline(vae=om, text_encoder=None, tokenizer=None, unet=None,
                                   scheduler=None).enable_vae_tiling()
    assert om.use_tiling


def test_sample_size_survives_save_and_load(tmp_path):
    pytest.importorskip("safetensors")
    vae = AutoencoderKL.synthetic(tiny=True, sample_size=96)
    vae.save_pretrained(str(tmp_path / "vae"))
    back = AutoencoderKL.from_pretrained(str(tmp_path), subfolder="vae")
    assert back.config.sample_size == 96
    assert (back.tile_sample_min_size, back.tile_latent_min_size) == (96, 12)
    assert AutoencoderKL.from_config({"block_out_channels": [16, 32, 32, 32], "norm_num_groups": 8}).config.sample_size == 32


def test_new_descriptor_structs_match_the_header(tmp_path):
    """sizeof / offsetof of pp_window and pp_tile_blend_desc in include/powerpaint_b200.h (plain C) equal the ctypes
    mirror"""
    import shutil
    import subprocess

    from powerpaint_b200 import _native as N

    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    structs = {"pp_window": N.Window, "pp_tile_blend_desc": N.TileBlendDesc}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "powerpaint_b200.h"', 'int main(void) {']
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append("  return 0; }")
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                        str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = dict(ln.split(" ", 1) for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                        check=True).stdout.splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == ctypes.sizeof(cls)
        for fname, _ in cls._fields_:
            assert int(out[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)
