"""CPU tests: the C-ABI library loads and exports every symbol include/powerpaint_b200.h declares (no
compute calls without a GPU); host-side logic (weight packing, pre-processing, sharding, checks)."""
import ctypes
import os
import re

import numpy as np
import PIL.Image
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from powerpaint_b200 import _native, build

    path = build.build()
    lib = ctypes.CDLL(str(path))
    hdr = open(os.path.join(ROOT, "include", "powerpaint_b200.h")).read()
    declared = set(re.findall(r"\b(pp_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for sym in declared:
        assert hasattr(lib, sym), f"{sym} declared in the header but not exported"
    assert declared == set(_native.EXPORTED_SYMBOLS), declared ^ set(_native.EXPORTED_SYMBOLS)
    assert _native.lib().pp_abi_version() == _native.ABI_VERSION == 5
    assert _native.lib().pp_device_supported() in (0, 1)


def test_ctypes_struct_sizes_match_header_layout():
    from powerpaint_b200 import _native as N

    # pointer-heavy structs: sizes must be multiples of 8 and stable (guards accidental field drift)
    assert ctypes.sizeof(N.GemmDesc) % 8 == 0 and ctypes.sizeof(N.AttnDesc) % 8 == 0
    assert N.GemmDesc.rowvec_ld.offset > N.GemmDesc.rows_per_group.offset
    assert N.CfgDdimDesc.extra_per_copy.offset > N.CfgDdimDesc.guidance_from_coef.offset


def test_invalid_descriptors_fail_loudly_without_gpu():
    from powerpaint_b200 import _native as N

    L = N.lib()
    d = N.GemmDesc()  # all zeros
    assert L.pp_gemm_conv(ctypes.byref(d), None) != 0
    assert b"gemm" in L.pp_last_error()
    a = N.AttnDesc()
    assert L.pp_attention(ctypes.byref(a), None) != 0
    with pytest.raises(RuntimeError):
        N.check(1, "x")

    # the step kernels move latents, state, noise, blend inputs and fp32 eps (eps_ld 4) as float4: a view one float
    # off a 16-byte boundary must be refused when it is recorded. Integer addresses only: recording validates and
    # launches nothing.
    base = 1 << 20

    def refused(add, desc, what):
        prog = N.vp()
        N.check(L.pp_program_create(ctypes.byref(prog)), "pp_program_create")
        try:
            rc = add(prog, ctypes.byref(desc))
            return rc != 0 and what in L.pp_last_error()
        finally:
            L.pp_program_destroy(prog)

    def ddim(**kw):
        d = N.CfgDdimDesc()
        d.eps, d.eps_fp32, d.eps_ld = base, 1, 4
        d.latents, d.coef, d.batch, d.hw, d.do_cfg = base + 4096, base + 8192, 1, 64, 1
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def unipc(**kw):
        d = N.UniPCDesc()
        d.eps, d.eps_fp32, d.eps_ld = base, 1, 4
        d.latents, d.last_sample, d.m1, d.m2 = base + 4096, base + 8192, base + 12288, base + 16384
        d.coef, d.ucoef, d.batch, d.hw, d.do_cfg = base + 20480, base + 24576, 1, 64, 1
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    assert not refused(L.pp_program_add_cfg_ddim, ddim(), b"cfg_ddim"), L.pp_last_error()
    assert not refused(L.pp_program_add_cfg_ddim, ddim(eps=base + 4, eps_fp32=0), b"cfg_ddim")  # bf16 eps: scalar loads
    assert not refused(L.pp_program_add_cfg_ddim, ddim(eps=base + 4, eps_ld=8), b"cfg_ddim")    # strided eps: scalar
    blend = dict(blend_x0=base + 32768, blend_mask=base + 36868, blend_noise=base + 40960)    # the mask is read per float
    assert not refused(L.pp_program_add_cfg_ddim, ddim(**blend), b"cfg_ddim"), L.pp_last_error()
    for field in ("latents", "noise", "eps"):
        assert refused(L.pp_program_add_cfg_ddim, ddim(**{field: (getattr(ddim(), field) or base + 49152) + 4}),
                       b"cfg_ddim"), field
    for field in ("blend_x0", "blend_noise"):
        assert refused(L.pp_program_add_cfg_ddim, ddim(**blend | {field: blend[field] + 4}), b"cfg_ddim"), field
    assert not refused(L.pp_program_add_unipc, unipc(), b"unipc"), L.pp_last_error()
    assert not refused(L.pp_program_add_unipc, unipc(eps=base + 4, eps_fp32=0), b"unipc")
    assert not refused(L.pp_program_add_unipc, unipc(eps=base + 4, eps_ld=8), b"unipc")
    for field in ("latents", "last_sample", "m1", "m2", "eps"):
        assert refused(L.pp_program_add_unipc, unipc(**{field: getattr(unipc(), field) + 4}), b"unipc"), field


def test_group_norm_scratch_size_is_a_pure_host_query():
    from powerpaint_b200 import ops

    # stats [batch, groups, 2] + ticket counters + one partial per (sample, block): always larger than the
    # statistics alone, 16-byte granular offsets, bounded (~1200 blocks over the machine) for any shape
    for batch, hw, c, groups in [(16, 4096, 320, 32), (16, 64, 1280, 32), (2, 4, 64, 8), (1, 16384, 2560, 32)]:
        n = ops.gn_scratch_bytes(batch, hw, c, groups)
        assert n > batch * groups * 2 * 4 and n % 4 == 0
        assert n <= batch * groups * 8 + 64 + (148 * 8 + 2 * batch) * groups * 8
    with pytest.raises(ValueError):
        ops.gn_scratch_bytes(2, 64, 30, 5)  # channels not a multiple of 8


def test_weight_packing():
    from powerpaint_b200 import ops

    w = torch.arange(2 * 5 * 9, dtype=torch.float32).reshape(2, 5, 3, 3)
    p = ops.pack_conv3x3_weight(w)
    assert p.shape == (2, 9 * 64) and p.dtype == torch.bfloat16
    p3 = p.reshape(2, 9, 64).float()
    for tap in range(9):
        assert torch.equal(p3[:, tap, :5], w[:, :, tap // 3, tap % 3].to(torch.bfloat16).float())
    assert (p3[:, :, 5:] == 0).all()
    ps = ops.pack_conv3x3_weight(torch.randn(4, 72, 3, 3), split=64)  # 64 + 8 channels
    assert ps.shape == (4, 9 * 128)
    wl = torch.randn(6, 72)
    pl = ops.pack_concat_linear_weight(wl, 64)
    assert pl.shape == (6, 128) and torch.equal(pl[:, 64:72].float(), wl[:, 64:].to(torch.bfloat16).float())
    wg, bg = torch.arange(256 * 4, dtype=torch.float32).reshape(256, 4), torch.arange(256, dtype=torch.float32)
    wi, bi = ops.pack_geglu_weight(wg, bg, 128)
    assert torch.equal(bi[:64], bg[:64]) and torch.equal(bi[64:128], bg[128:192]) and torch.equal(bi[128:192], bg[64:128])
    assert torch.equal(wi[64:128].float(), wg[128:192].to(torch.bfloat16).float())


def test_prepare_mask_and_masked_image_like_reference():
    from powerpaint_b200.pipelines.common import postprocess_image, prepare_mask_and_masked_image, randn_tensor

    img = PIL.Image.fromarray((np.random.RandomState(0).rand(40, 48, 3) * 255).astype("uint8"))
    m = np.zeros((40, 48), "uint8")
    m[10:30, 10:30] = 255
    mask, masked = prepare_mask_and_masked_image(img, PIL.Image.fromarray(m), 32, 32)
    assert mask.shape == (1, 1, 32, 32) and masked.shape == (1, 3, 32, 32)
    assert set(mask.unique().tolist()) <= {0.0, 1.0}
    assert (masked[:, :, mask[0, 0] == 1] == 0).all() and masked.abs().max() <= 1
    t_img, t_mask = torch.rand(2, 3, 16, 16) * 2 - 1, torch.rand(2, 16, 16)
    mk, ms, im = prepare_mask_and_masked_image(t_img, t_mask, 16, 16, return_image=True)
    assert mk.shape == (2, 1, 16, 16) and torch.equal(im, t_img) and torch.equal(ms, t_img * (mk < 0.5))
    with pytest.raises(ValueError):
        prepare_mask_and_masked_image(t_img * 3, t_mask, 16, 16)
    with pytest.raises(TypeError):
        prepare_mask_and_masked_image(t_img, m, 16, 16)
    with pytest.raises(ValueError):
        prepare_mask_and_masked_image(None, t_mask, 16, 16)
    a = randn_tensor((2, 4, 8, 8), generator=torch.Generator().manual_seed(1), device="cpu", dtype=torch.float32)
    b = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(1))
    assert torch.equal(a, b)
    gl = [torch.Generator().manual_seed(i) for i in range(2)]
    c = randn_tensor((2, 4, 8, 8), generator=gl, device="cpu", dtype=torch.float32)
    assert torch.equal(c[1], torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(1))[0])
    pil = postprocess_image(torch.zeros(1, 3, 8, 8), "pil")
    assert pil[0].size == (8, 8) and np.array(pil[0]).max() == 128


def test_pipeline_check_inputs_errors_cpu():
    from powerpaint_b200.engine import NetConfig
    from powerpaint_b200.models import UNet2DConditionModel
    from oracle.vae import AutoencoderKLOracle as AutoencoderKL
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline
    from powerpaint_b200.schedulers import DDIMScheduler

    n = NetConfig(in_channels=9, block_out_channels=(32, 64, 128, 128), attention_head_dim=4, cross_attention_dim=64,
                  norm_num_groups=8)
    pipe = StableDiffusionInpaintPipeline(vae=AutoencoderKL.synthetic(tiny=True), text_encoder=None, tokenizer=None,
                                          unet=UNet2DConditionModel.synthetic(n), scheduler=DDIMScheduler())
    assert pipe.vae_scale_factor == 8
    with pytest.raises(ValueError):
        pipe.check_inputs("a", 100, 64, 1.0, 1)           # not divisible by 8
    with pytest.raises(ValueError):
        pipe.check_inputs("a", 64, 64, 1.5, 1)            # strength out of range
    with pytest.raises(ValueError):
        pipe.check_inputs("a", 64, 64, 1.0, 0)            # callback_steps
    with pytest.raises(ValueError):
        pipe.check_inputs(None, 64, 64, 1.0, 1)           # neither prompt nor embeds
    with pytest.raises(ValueError):
        pipe.check_inputs("a", 64, 64, 1.0, 1, prompt_embeds=torch.zeros(1, 77, 64))
    with pytest.warns(UserWarning, match="resident on the GPU"):  # the v2 app calls it (ref:app.py:199): accepted, no-op
        pipe.enable_model_cpu_offload()
    with pytest.raises(NotImplementedError):
        StableDiffusionInpaintPipeline(vae=pipe.vae, text_encoder=None, tokenizer=None, unet=pipe.unet,
                                       scheduler=DDIMScheduler(), safety_checker=object())


def test_shard_ranges():
    from powerpaint_b200.parallel import shard_ranges

    assert shard_ranges(32, 8) == [(4 * i, 4 * i + 4) for i in range(8)]
    assert shard_ranges(10, 4) == [(0, 3), (3, 6), (6, 8), (8, 10)]
    assert shard_ranges(2, 4) == [(0, 1), (1, 2), (2, 2), (2, 2)]
    with pytest.raises(ValueError):
        shard_ranges(4, 0)


def test_gemm_stats_geometry_is_a_pure_host_query():
    """which GEMMs / convs can emit GroupNorm partial sums from their epilogue, and in which layout"""
    from powerpaint_b200 import _native as nat
    from powerpaint_b200 import ops

    a = torch.zeros(8, dtype=torch.bfloat16)  # only non-null pointers are needed: nothing is launched

    def conv(nb, h, w, cin, cout, s2=False):
        return ops.gemm_desc(a0=a, w=a, out=a, N_=cout, a_mode=nat.PP_A_CONV3X3_S2 if s2 else nat.PP_A_CONV3X3, c0=cin,
                             nb=nb, h=h, w_=w)
    g = ops.gemm_stats_geometry(conv(16, 64, 64, 320, 320))
    assert g.supported and g.segs == 1 and g.seg_rows == 128 and g.tiles_per_group == 32 and g.wo * g.ho == 4096
    assert g.bytes == 16 * 32 * 320 * 4 * 4  # {sum, sum of squares, shift, pad} per (tile, channel)
    g = ops.gemm_stats_geometry(conv(16, 8, 8, 1280, 1280))
    assert g.supported and g.segs == 2 and g.seg_rows == 64 and g.tiles_per_group == 1
    g = ops.gemm_stats_geometry(conv(2, 107, 80, 320, 320, s2=True))
    assert g.supported and (g.wo, g.ho) == (40, 54)
    g = ops.gemm_stats_geometry(conv(4, 2, 2, 128, 128))
    assert g.supported and g.segs == 4 and g.seg_rows == 32 and (g.wo, g.ho) == (2, 2)  # a mostly-padding pixel box
    g = ops.gemm_stats_geometry(conv(64, 1, 1, 128, 128))
    assert not g.supported  # 2 tile rows per sample: the consumer runs its own statistics pass
    g = ops.gemm_stats_geometry(conv(2, 64, 64, 320, 4))
    assert not g.supported  # ragged N takes the generic epilogue
    lin = ops.gemm_desc(a0=a, w=a, out=a, N_=320, M=16 * 4096, c0=320, rows_per_group=4096)
    g = ops.gemm_stats_geometry(lin)
    assert g.supported and g.segs == 1 and g.tiles_per_group == 32
    lin = ops.gemm_desc(a0=a, w=a, out=a, N_=1280, M=6 * 64, c0=1280, rows_per_group=64)
    g = ops.gemm_stats_geometry(lin)
    assert g.supported and g.segs == 2 and g.seg_rows == 64
    lin = ops.gemm_desc(a0=a, w=a, out=a, N_=320, M=2 * 8560, c0=320, rows_per_group=8560)
    assert not ops.gemm_stats_geometry(lin).supported  # 80 x 107 latent: samples straddle the 128-row tiles


def test_layer_norm_record_and_split_k_queries_are_pure_host_queries():
    """host-only geometry answers that must describe the launch that actually runs: the per-row LayerNorm record count
    (a producer never runs split-K, whatever the plain launch of the same shape would pick) and the split-K
    workspace (only for long-K launches whose doubled tiles fit the SMs in one round)"""
    from powerpaint_b200 import _native as nat
    from powerpaint_b200 import ops

    a = torch.zeros(8, dtype=torch.bfloat16)  # only non-null pointers are needed: nothing is launched

    def lin(M, K, N, **kw):
        return ops.gemm_desc(a0=a, w=a, out=a, N_=N, M=M, c0=K, **kw)
    # SD-1.5 transformer widths: records = 2 per n-tile of the single-CTA tile width
    assert ops.gemm_row_stats_records(lin(65536, 320, 320)) == 4       # 2 x 160
    assert ops.gemm_row_stats_records(lin(16384, 640, 640)) == 8       # 4 x 160
    n1280 = ops.gemm_row_stats_records(lin(4096, 1280, 1280))          # K = 1280 would pair up without row_stats
    assert n1280 > 0 and n1280 % 2 == 0
    assert ops.gemm_row_stats_records(lin(4096, 1280, 1280, block_n=160)) == 16
    assert ops.gemm_row_stats_records(lin(1024, 320, 324)) == 0        # ragged N: generic epilogue, no records
    assert ops.gemm_row_stats_records(lin(1024, 320, 320, act=nat.PP_ACT_SILU)) == 0

    def conv(nb, h, w, cin, cout):
        return ops.gemm_desc(a0=a, w=a, out=a, N_=cout, a_mode=nat.PP_A_CONV3X3, c0=cin, nb=nb, h=h, w_=w)
    nbytes, tiles = ops.gemm_splitk_query(conv(16, 8, 8, 1280, 1280))  # 8 m-tiles: few tiles, K = 180 iterations
    assert nbytes > 0 and tiles > 0 and nbytes % (tiles * 128 * 4) == 0
    bn = nbytes // (tiles * 128 * 4)
    assert bn in (128, 160, 256) and tiles == 8 * ((1280 + bn - 1) // bn) and 2 * (tiles // 2) <= 74
    assert ops.gemm_splitk_query(conv(16, 64, 64, 320, 320)) == (0, 0)  # 512 m-tiles: nothing to gain
    assert ops.gemm_splitk_query(conv(16, 8, 8, 64, 1280)) == (0, 0)    # K = 9 iterations: too short to split
    assert ops.gemm_splitk_query(lin(65536, 320, 320)) == (0, 0)


def test_layer_norm_fold_algebra_cpu():
    """LayerNorm(x) W^T + b == rstd (x W'^T - mean u) + b' with the folded operands the engine hands to the GEMM
    (ops.fold_layer_norm_into_linear), also through the GEGLU row interleave; the only difference left is the bf16
    rounding of W' (the tensor core's operand)"""
    from powerpaint_b200 import ops

    g = torch.Generator().manual_seed(3)
    M, C, N = 64, 320, 256
    x = (torch.randn(M, C, generator=g) * 2 + 0.7).to(torch.bfloat16).float()
    w = torch.randn(N, C, generator=g) / C ** 0.5
    gamma = 1 + 0.3 * torch.randn(C, generator=g)
    beta = 0.3 * torch.randn(C, generator=g)
    bias = torch.randn(N, generator=g)
    wf, u, b = ops.fold_layer_norm_into_linear(w, gamma, beta, bias)
    assert wf.dtype == torch.bfloat16 and u.dtype == b.dtype == torch.float32
    assert torch.equal(u, wf.double().sum(1).float())  # row sums of exactly what the tensor core multiplies
    mean = x.mean(1, keepdim=True)
    rstd = (x.var(1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
    got = rstd * (x @ wf.float().t() - mean * u[None]) + b
    ref = torch.nn.functional.layer_norm(x, (C,), gamma, beta, 1e-5) @ w.t() + bias
    assert ((got - ref).norm() / ref.norm()).item() < 3e-3
    # with an un-rounded W' the identity is exact to fp32 round-off
    wx = w * gamma[None]
    exact = rstd * (x @ wx.t() - mean * wx.sum(1)[None]) + (w @ beta + bias)
    assert ((exact - ref).norm() / ref.norm()).item() < 1e-5
    # GEGLU: value / gate rows interleaved per tile, u and b' permuted with them
    for bn in (128, 256):
        wi, ui = ops.pack_geglu_weight(wf.float(), u, bn)
        _, bi = ops.pack_geglu_weight(wf.float(), b, bn)
        y = rstd * (x @ wi.float().t() - mean * ui[None]) + bi
        half = bn // 2
        yv = torch.cat([y[:, t * bn:t * bn + half] for t in range(N // bn)], 1)
        yg = torch.cat([y[:, t * bn + half:(t + 1) * bn] for t in range(N // bn)], 1)
        assert torch.allclose(yv, got[:, :N // 2], atol=1e-5) and torch.allclose(yg, got[:, N // 2:], atol=1e-5)


def test_header_is_plain_c_and_every_struct_field_offset_matches_the_ctypes_binding(tmp_path):
    """include/powerpaint_b200.h through a C compiler (`gcc -std=c99 -pedantic`, no C++): it links against the library,
    fails loudly without a GPU, and sizeof / offsetof of every descriptor field equal the ctypes mirror in
    powerpaint_b200/_native.py — the binding a maintainer would write (INTEGRATION.md) cannot drift from the header"""
    import shutil
    import subprocess

    from powerpaint_b200 import _native as N

    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    structs = {"pp_stats_geom": N.StatsGeom, "pp_gemm_desc": N.GemmDesc, "pp_attn_desc": N.AttnDesc,
               "pp_gn_desc": N.GnDesc, "pp_cfg_ddim_desc": N.CfgDdimDesc, "pp_unipc_desc": N.UniPCDesc}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include <string.h>', '#include "powerpaint_b200.h"',
             'int main(void) {']
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  pp_gemm_desc d; memset(&d, 0, sizeof d);',
              '  printf("abi %d\\n", pp_abi_version());',
              '  printf("status %d\\n", (int)pp_gemm_conv(&d, 0));',
              '  printf("error %s\\n", pp_last_error());', '  return 0; }']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    libdir = os.path.join(root, "powerpaint_b200")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"),
                        str(src), "-o", str(exe), "-L", libdir, "-lpowerpaint_b200", f"-Wl,-rpath,{libdir}"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = dict(ln.split(" ", 1) for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                        check=True).stdout.splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == ctypes.sizeof(cls), (cname, out[cname], ctypes.sizeof(cls))
        for fname, _ in cls._fields_:
            assert int(out[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)
    assert int(out["abi"]) == N.ABI_VERSION and int(out["status"]) != 0 and out["error"].strip()


def test_integration_md_stub_lists_the_descriptor_fields_of_the_binding():
    """the ctypes stub printed in INTEGRATION.md is the binding: same field names in the same order"""
    import re

    from powerpaint_b200 import _native as N

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    md = open(os.path.join(root, "INTEGRATION.md")).read()
    block = md[md.index("class pp_gemm_desc"):md.index("lib.pp_gemm_conv.argtypes")]
    assert re.findall(r'\("(\w+)", C\.', block) == [f for f, _ in N.GemmDesc._fields_]
    assert f"pp_abi_version() == {N.ABI_VERSION}" in block
