"""GPU tests of tiled VAE encode / decode (AutoencoderKL.enable_tiling): the blend and window-copy kernels against
the oracle's loops bit for bit, the tiled programs against the oracle's fp32 tiled path (oracle/vae_tiling.py; rel-L2
<= 3e-2, the bound of the untiled VAE tests), canvases above one megapixel at SD-1.5 widths, and a pipeline call."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.fixture(scope="module", autouse=True)
def _fp32_exact():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _pair(tiny, sample_size):
    from oracle.vae_tiling import TiledAutoencoderKLOracle
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    pm = AutoencoderKL.synthetic(seed=4321, tiny=tiny, sample_size=sample_size)
    om = TiledAutoencoderKLOracle(block_out_channels=pm.config.block_out_channels, norm_num_groups=pm.config.norm_num_groups,
                                   layers_per_block=pm.config.layers_per_block, sample_size=sample_size)
    g = torch.Generator().manual_seed(7)
    sd = {k: (v + 0.05 * torch.randn(v.shape, generator=g) if v.dim() == 1 else v) for k, v in pm.state_dict().items()}
    pm.load_state_dict(sd)
    om.load_state_dict(sd)
    return om.to(DEV).eval(), pm.to(DEV)


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("encode,h,w,ss,C", [(False, 13, 13, 64, 4), (False, 20, 31, 64, 4), (True, 104, 152, 64, 8),
                                             (True, 200, 104, 96, 8)])
def test_tile_blend_is_bitwise_the_oracle_loop(encode, h, w, ss, C):
    """random fp32 tiles with ragged last rows / columns, blended in diffusers order by pp_tile_blend (in place in
    an NHWC store) and by the oracle's blend_v / blend_h (NCHW): torch.equal"""
    from oracle.vae_tiling import TiledAutoencoderKLOracle
    from powerpaint_b200 import ops
    from powerpaint_b200.models.autoencoder_kl import vae_tile_geometry

    geom = vae_tile_geometry(encode, h, w, ss, ss // 8, 0.25, 8)
    om = TiledAutoencoderKLOracle(block_out_channels=(8, 8, 8, 8), norm_num_groups=4, layers_per_block=1, sample_size=ss)
    e = int((ss // 8 if encode else ss) * 0.25)
    nb = 3
    g = torch.Generator(device=DEV).manual_seed(h * w)
    ref = [torch.randn(nb, C, t.out_h, t.out_w, device=DEV, generator=g) * 4 for t in geom.tiles]
    # product store: each tile its own slab, samples a padded stride apart
    stores = []
    for t, r in zip(geom.tiles, ref):
        slab = torch.full((nb, t.out_h * t.out_w * C + 64), float("nan"), device=DEV)
        v = slab[:, :t.out_h * t.out_w * C].view(nb, t.out_h, t.out_w, C)
        v.copy_(r.permute(0, 2, 3, 1))
        stores.append((slab, v))
    for k, t in enumerate(geom.tiles):
        if t.row > 0:
            ref[k] = om.blend_v(ref[k - geom.cols], ref[k], e)
        if t.col > 0:
            ref[k] = om.blend_h(ref[k - 1], ref[k], e)
        if t.blend_v or t.blend_h:
            ops.run(ops.tile_blend_desc(stores[k][1], stores[k - geom.cols][1] if t.blend_v else None,
                                        stores[k - 1][1] if t.blend_h else None, t.blend_v, t.blend_h))
    torch.cuda.synchronize()
    for (slab, v), r in zip(stores, ref):
        assert torch.equal(v, r.permute(0, 2, 3, 1))
        assert torch.isnan(slab[:, v[0].numel():]).all()  # the padding between samples is untouched


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_window_copy_is_exact(dtype):
    from powerpaint_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(3)
    nb, H, W, cs, cd, ch = 2, 37, 53, 8, 6, 5
    src = torch.randn(nb, H * W, cs, device=DEV, generator=g).to(dtype)
    dst = torch.full((nb, 40 * 30, cd), -7.75, device=DEV, dtype=dtype)
    wins = [((s * H * W + y * W + x) * cs, (s * 1200 + dy * 30 + dx) * cd, W * cs, 30 * cd, hh, ww)
            for s, (y, x, dy, dx, hh, ww) in [(0, (0, 0, 0, 0, 11, 7)), (1, (5, 40, 3, 9, 32, 13)),
                                              (0, (36, 52, 39, 29, 1, 1)), (1, (0, 0, 0, 0, 0, 4))]]
    ops.window_copy(ops.WindowList(src, dst, ch, wins))
    want = torch.full_like(dst, -7.75)
    sv, wv = src.view(nb, H, W, cs), want.view(nb, 40, 30, cd)
    for so, do, _, _, hh, ww in wins:
        s, p = divmod(so // cs, H * W)
        y, x = divmod(p, W)
        _, q = divmod(do // cd, 1200)
        dy, dx = divmod(q, 30)
        wv[s, dy:dy + hh, dx:dx + ww, :ch] = sv[s, y:y + hh, x:x + ww, :ch]
    torch.cuda.synchronize()
    assert torch.equal(dst, want)
    with pytest.raises(ValueError):
        ops.WindowList(src, dst, ch, [(0, 0, 0, 30 * cd, 81, 1)])  # runs past the end of dst


# ------------------------------------------------------------------ tiny VAE against the oracle's tiled path
@pytest.mark.parametrize("chunk", [None, 3 * 64 * 64])
def test_tiny_tiled_vae_matches_oracle(chunk, monkeypatch):
    """sample_size 64: 104 x 104 images and 13 x 13 latents give 3 x 3 tile shapes (the last two tiles of a row both
    partial); a small chunk size splits shape groups across several recorded passes"""
    from powerpaint_b200.models.autoencoder_kl import VaeEngine

    if chunk is not None:
        monkeypatch.setattr(VaeEngine, "TILE_CHUNK_PIXELS", chunk)
    om, pm = _pair(True, 64)
    om.enable_tiling()
    pm.enable_tiling()
    g = torch.Generator(device=DEV).manual_seed(11)
    for B, H, W in ((2, 104, 104), (1, 152, 200)):
        assert len(pm.tile_geometry(True, H, W).groups()) >= 4
        x = torch.rand(B, 3, H, W, device=DEV, generator=g) * 2 - 1
        with torch.no_grad():
            ref = om.encode(x).latent_dist
        d = pm.encode(x).latent_dist
        assert d.mean.shape == ref.mean.shape == (B, 4, H // 8, W // 8)
        assert _rel(d.mean, ref.mean) < 3e-2 and _rel(d.logvar, ref.logvar) < 3e-2, (_rel(d.mean, ref.mean), chunk)
        d2 = pm.tiled_encode(x).latent_dist
        assert torch.equal(d2.mean, d.mean) and torch.equal(d2.logvar, d.logvar)  # two runs: bit-identical
        z = torch.randn(B, 4, H // 8, W // 8, device=DEV, generator=g)
        with torch.no_grad():
            ref_img = om.decode(z).sample
        img = pm.decode(z).sample
        assert img.shape == ref_img.shape == (B, 3, H, W) and torch.isfinite(img).all()
        assert _rel(img, ref_img) < 3e-2, (_rel(img, ref_img), chunk)
        assert torch.equal(pm.tiled_decode(z).sample, img)
        u8 = pm.decode_postprocessed(z, uint8=True)
        want = ((img / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8).permute(0, 2, 3, 1)
        assert (u8.int() - want.int()).abs().max().item() <= 1
        pt = pm.decode_postprocessed(z, uint8=False)
        assert torch.allclose(pt, (img / 2 + 0.5).clamp(0, 1), atol=1e-6)
        # uint8 image + mask through the whole-canvas pre-processing, then the tile gather
        img8 = torch.randint(0, 256, (B, 3, H, W), device=DEV, generator=g, dtype=torch.uint8)
        mask = (torch.rand(B, 1, H, W, device=DEV, generator=g) > 0.5).to(torch.uint8) * 255
        a = pm.encode_uint8(img8, mask)
        imf = (img8.cpu().float() / 127.5 - 1.0).to(DEV)
        b = pm.encode(imf * ((mask.float() / 255.0) < 0.5)).latent_dist
        assert _rel(a.mean, b.mean) < 1e-6 and _rel(a.logvar, b.logvar) < 1e-6
    # small canvases: the tiling switch leaves them on the untiled programs, bit for bit
    x = torch.rand(1, 3, 64, 48, device=DEV, generator=g) * 2 - 1
    m_on = pm.encode(x).latent_dist.mean
    pm.disable_tiling()
    assert torch.equal(pm.encode(x).latent_dist.mean, m_on)


# ------------------------------------------------------------------ SD-1.5 widths
def test_sd15_tiled_1024x1360_matches_oracle():
    om, pm = _pair(False, 512)
    om.enable_tiling()
    pm.enable_tiling()
    g = torch.Generator(device=DEV).manual_seed(5)
    x = torch.rand(1, 3, 1360, 1024, device=DEV, generator=g) * 2 - 1
    with torch.no_grad():
        ref = om.encode(x).latent_dist
    d = pm.encode(x).latent_dist
    assert d.mean.shape == ref.mean.shape == (1, 4, 170, 128)
    assert _rel(d.mean, ref.mean) < 3e-2 and _rel(d.logvar, ref.logvar) < 3e-2, _rel(d.mean, ref.mean)
    del x, ref, d
    z = torch.randn(1, 4, 170, 128, device=DEV, generator=g)
    with torch.no_grad():
        ref_img = om.decode(z).sample
    img = pm.decode(z).sample
    assert img.shape == ref_img.shape == (1, 3, 1360, 1024)
    assert _rel(img, ref_img) < 3e-2, _rel(img, ref_img)
    print(f"[tiled SD-1.5 1024x1360] decode rel-L2 {_rel(img, ref_img):.3e}")


def _peak(eng, fn):
    eng._plans.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated(), out


def test_sd15_tiled_2048x2728_fits_and_peak_memory():
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    vae = AutoencoderKL.synthetic(seed=4321, sample_size=512).to(DEV)
    eng = vae.engine()
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.rand(1, 3, 2728, 2048, device=DEV, generator=g) * 2 - 1
    z = torch.randn(1, 4, 341, 256, device=DEV, generator=g)
    with pytest.raises(RuntimeError, match=r"16384.*enable_vae_tiling\(\)"):
        vae.decode(z)
    with pytest.raises(RuntimeError, match=r"16384.*enable_vae_tiling\(\)"):
        vae.encode(x)
    vae.decode(torch.randn(1, 4, 16, 16, device=DEV, generator=g))  # packs the weights outside the measurements
    z1024 = torch.randn(1, 4, 128, 128, device=DEV, generator=g)
    peak_untiled, _ = _peak(eng, lambda: vae.decode(z1024).sample)
    vae.enable_tiling()
    peak_tiled, img = _peak(eng, lambda: vae.decode(z).sample)
    assert img.shape == (1, 3, 2728, 2048) and torch.isfinite(img).all()
    print(f"[tiled SD-1.5] peak allocated: untiled 1024^2 decode {peak_untiled / 2**30:.2f} GiB, "
          f"tiled 2048x2728 decode {peak_tiled / 2**30:.2f} GiB")
    assert peak_tiled <= peak_untiled
    del img
    eng._plans.clear()
    d = vae.encode(x).latent_dist
    assert d.mean.shape == (1, 4, 341, 256) and torch.isfinite(d.mean).all() and torch.isfinite(d.logvar).all()


def test_tiled_programs_use_only_tested_kernel_variants(monkeypatch):
    """every GEMM / attention descriptor the tiled programs record at SD-1.5 widths resolves to a variant of the
    variant matrix of test_kernel_variants_gpu.py"""
    from test_kernel_variants_gpu import ATTN_CASES, GEMM_CASES, _Census

    from powerpaint_b200 import ops as o
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    census = _Census()
    source = ["?"]
    orig_add = o.Program.add

    def add(self, desc):
        census.record(source[0], desc)
        return orig_add(self, desc)
    monkeypatch.setattr(o.Program, "add", add)
    vae = AutoencoderKL.synthetic(seed=4321, sample_size=512).to(DEV)
    eng = vae.engine()
    for H, W in ((1360, 1024), (2728, 2048)):
        source[0] = f"tiled encode {H}x{W}"
        eng.tiled_plan(True, 1, H, W, vae.tile_geometry(True, H, W), vae._tiling_key())
        source[0] = f"tiled decode {H}x{W}"
        eng.tiled_plan(False, 1, H // 8, W // 8, vae.tile_geometry(False, H // 8, W // 8), vae._tiling_key())
        eng._plans.clear()
    monkeypatch.setattr(o.Program, "add", orig_add)
    used = {(kind, variant) for kind, _, variant, _, _ in census.sigs.values()}
    print(f"[tiled census] {len(census.sigs)} signatures, variants {sorted(used)}")
    assert {v for k, v in used if k == "gemm"} <= {v for _, v, _ in GEMM_CASES}
    assert {v for k, v in used if k == "attn"} <= {v for _, v, _ in ATTN_CASES}


# ------------------------------------------------------------------ pipeline
def test_pipeline_v1_1024x1360_needs_and_runs_with_vae_tiling():
    from powerpaint_b200.engine import NetConfig
    from powerpaint_b200.models import UNet2DConditionModel
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline
    from powerpaint_b200.schedulers import DDIMScheduler

    unet = UNet2DConditionModel.synthetic(NetConfig(in_channels=9, block_out_channels=(32, 64, 128, 128),
                                                    attention_head_dim=4, cross_attention_dim=64, norm_num_groups=8)).to(DEV)
    vae = AutoencoderKL.synthetic(tiny=True, sample_size=512).to(DEV)
    pipe = StableDiffusionInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=unet,
                                          scheduler=DDIMScheduler(), safety_checker=None)
    g = torch.Generator().manual_seed(0)
    B, H, W = 1, 1360, 1024
    img = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8).to(DEV)
    mask = torch.zeros(B, 1, H, W, dtype=torch.uint8)
    mask[:, :, 400:900, 300:700] = 255
    mask = mask.to(DEV)
    pe = torch.randn(B, 77, 64, generator=g) * 0.5
    ne = torch.randn(B, 77, 64, generator=g) * 0.5
    kw = dict(image=img, mask=mask, prompt_embeds=pe, negative_prompt_embeds=ne, height=H, width=W,
              num_inference_steps=3, guidance_scale=7.5)
    with pytest.raises(RuntimeError, match="enable_vae_tiling"):
        pipe(generator=torch.Generator().manual_seed(5), output_type="latent", **kw)
    pipe.enable_vae_tiling()
    lat = pipe(generator=torch.Generator().manual_seed(5), output_type="latent", **kw).images
    u8 = pipe(generator=torch.Generator().manual_seed(5), output_type="uint8", **kw).images
    assert lat.shape == (B, 4, H // 8, W // 8) and torch.isfinite(lat).all()
    assert u8.shape == (B, H, W, 3) and u8.dtype == torch.uint8
    want = vae.decode_postprocessed(lat / vae.config.scaling_factor, uint8=True)
    assert torch.equal(u8, want)
    pipe.disable_vae_tiling()
    assert not vae.use_tiling
