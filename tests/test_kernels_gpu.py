"""GPU parity tests of the individual CUDA kernels, called through the C ABI, against plain
PyTorch fp32 references of the same op (inputs rounded to bf16 first so only accumulation
order / output rounding differ)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _dev():
    return torch.device("cuda:0")


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def ops():
    from powerpaint_b200 import _native, ops as o

    assert _native.lib().pp_device_supported() == 1, "tests need an sm_90 (H100) device"
    return o


@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 0), (256, 320, 320, 0), (1000, 640, 768, 0),
                                      (4096, 1280, 320, 256), (77, 320, 768, 0), (300, 64, 1280, 64),
                                      (512, 320, 2560, 160), (16, 1280, 320, 0), (2048, 4, 320, 0)])
def test_gemm_plain(ops, M, N, K, bn):
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    a = torch.randn(M, K, device=_dev(), generator=g).to(BF16)
    w = (torch.randn(N, K, device=_dev(), generator=g) / math.sqrt(K)).to(BF16)
    bias = torch.randn(N, device=_dev(), generator=g)
    out = torch.full((M, N), float("nan"), device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=a, w=w, out=out, N_=N, M=M, bias=bias, block_n=bn))
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias
    assert torch.isfinite(out.float()).all()
    assert _rel(out, ref) < 6e-3, _rel(out, ref)
    assert (out.float() - ref).abs().max().item() < 0.05 * ref.abs().max().item() + 0.02


def test_gemm_epilogue_full(ops):
    from powerpaint_b200 import _native as nat

    M, N, K = 640, 320, 640
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn(M, K, device=_dev(), generator=g).to(BF16)
    w = (torch.randn(N, K, device=_dev(), generator=g) / math.sqrt(K)).to(BF16)
    bias = torch.randn(N, device=_dev(), generator=g)
    rowvec = torch.randn(5, N, device=_dev(), generator=g)
    r1 = torch.randn(M, N, device=_dev(), generator=g).to(BF16)
    r2 = torch.randn(M, N, device=_dev(), generator=g).to(BF16)
    for fp32 in (False, True):
        out = torch.zeros(M, N, device=_dev(), dtype=torch.float32 if fp32 else BF16)
        ops.run(ops.gemm_desc(a0=a, w=w, out=out, N_=N, M=M, bias=bias, rowvec=rowvec, rows_per_group=128,
                              res1=r1, res2=r2, alpha=0.5, act=nat.PP_ACT_SILU, out_fp32=fp32))
        torch.cuda.synchronize()
        v = a.float() @ w.float().t() + bias + rowvec.repeat_interleave(128, 0) + r1.float()
        v = v * 0.5 + r2.float()
        ref = F.silu(v)
        assert _rel(out, ref) < (2e-4 if fp32 else 6e-3), _rel(out, ref)


def test_gemm_two_sources_and_transposed(ops):
    from powerpaint_b200 import _native as nat

    M, N, c0, c1 = 512, 320, 320, 96
    g = torch.Generator(device="cuda").manual_seed(5)
    a0 = torch.randn(M, c0, device=_dev(), generator=g).to(BF16)
    a1 = torch.randn(M, c1, device=_dev(), generator=g).to(BF16)
    wfull = torch.randn(N, c0 + c1, device=_dev(), generator=g) / math.sqrt(c0 + c1)
    w = ops.pack_concat_linear_weight(wfull, c0)
    out = torch.zeros(M, N, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=a0, a1=a1, c1=c1, w=w, out=out, N_=N, M=M))
    ref = torch.cat([a0, a1], 1).float() @ wfull.to(BF16).float().t()
    assert _rel(out, ref) < 6e-3
    # transposed store: out_t[b, n, t]
    t_rows, t_ld = 128, 136
    out_t = torch.zeros(M // t_rows, N, t_ld, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=a0, a1=a1, c1=c1, w=w, out=out_t, N_=N, M=M, epilogue=nat.PP_EPI_TRANSPOSED,
                          t_rows=t_rows, t_ld=t_ld))
    torch.cuda.synchronize()
    ref_t = ref.reshape(M // t_rows, t_rows, N).permute(0, 2, 1)
    assert _rel(out_t[:, :, :t_rows], ref_t) < 6e-3
    assert (out_t[:, :, t_rows:] == 0).all()


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_geglu(ops, bn):
    from powerpaint_b200 import _native as nat

    M, C = 384, 320
    F_ = 4 * C
    g = torch.Generator(device="cuda").manual_seed(11)
    a = torch.randn(M, C, device=_dev(), generator=g).to(BF16)
    w = torch.randn(2 * F_, C, device=_dev(), generator=g) / math.sqrt(C)
    b = torch.randn(2 * F_, device=_dev(), generator=g)
    wi, bi = ops.pack_geglu_weight(w, b, bn)
    out = torch.zeros(M, F_, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=a, w=wi, out=out, N_=2 * F_, M=M, bias=bi, epilogue=nat.PP_EPI_GEGLU, block_n=bn))
    torch.cuda.synchronize()
    h = a.float() @ w.to(BF16).float().t() + b
    ref = h[:, :F_] * F.gelu(h[:, F_:])
    assert _rel(out, ref) < 6e-3, _rel(out, ref)


@pytest.mark.parametrize("nb,h,w,cin,cout", [(2, 64, 64, 320, 320), (3, 16, 16, 640, 1280), (5, 8, 8, 1280, 1280),
                                              (2, 32, 32, 16, 320), (2, 64, 64, 320, 4), (1, 24, 40, 32, 64),
                                              (3, 4, 4, 64, 64), (4, 2, 2, 128, 128), (9, 1, 1, 128, 64)])
def test_conv3x3(ops, nb, h, w, cin, cout):
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(nb * 100 + cin)
    x = torch.randn(nb, cin, h, w, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(cout, cin, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * cin)).to(BF16)
    bias = torch.randn(cout, device=_dev(), generator=g)
    temb = torch.randn(nb, cout, device=_dev(), generator=g)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    wp = ops.pack_conv3x3_weight(wt.float())
    out = torch.full((nb, h, w, cout), float("nan"), device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x_nhwc, w=wp, out=out, N_=cout, a_mode=nat.PP_A_CONV3X3, c0=cin, nb=nb, h=h, w_=w,
                          bias=bias, rowvec=temb))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), bias, padding=1) + temb[:, :, None, None]
    got = out.permute(0, 3, 1, 2).float()
    assert torch.isfinite(got).all()
    assert _rel(got, ref) < 6e-3, _rel(got, ref)


def test_conv3x3_two_sources(ops):
    from powerpaint_b200 import _native as nat

    nb, h, w, c0, c1, cout = 2, 16, 16, 640, 320, 640
    g = torch.Generator(device="cuda").manual_seed(21)
    x0 = torch.randn(nb, h, w, c0, device=_dev(), generator=g).to(BF16)
    x1 = torch.randn(nb, h, w, c1, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(cout, c0 + c1, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * (c0 + c1))).to(BF16)
    wp = ops.pack_conv3x3_weight(wt.float(), split=c0)
    res = torch.randn(nb, h, w, cout, device=_dev(), generator=g).to(BF16)
    out = torch.zeros(nb, h, w, cout, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x0, a1=x1, c0=c0, c1=c1, w=wp, out=out, N_=cout, a_mode=nat.PP_A_CONV3X3, nb=nb,
                          h=h, w_=w, res1=res))
    torch.cuda.synchronize()
    xin = torch.cat([x0, x1], -1).permute(0, 3, 1, 2).float()
    ref = F.conv2d(xin, wt.float(), None, padding=1) + res.permute(0, 3, 1, 2).float()
    assert _rel(out.permute(0, 3, 1, 2), ref) < 6e-3


@pytest.mark.parametrize("nb,h,w,c", [(2, 64, 64, 320), (3, 16, 16, 1280), (2, 8, 8, 64), (1, 2, 2, 128), (2, 12, 20, 32)])
def test_conv3x3_stride2(ops, nb, h, w, c):
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(31 + c)
    x = torch.randn(nb, c, h, w, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(c, c, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * c)).to(BF16)
    bias = torch.randn(c, device=_dev(), generator=g)
    wp = ops.pack_conv3x3_weight(wt.float())
    out = torch.zeros(nb, h // 2, w // 2, c, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x.permute(0, 2, 3, 1).contiguous(), w=wp, out=out, N_=c, a_mode=nat.PP_A_CONV3X3_S2,
                          c0=c, nb=nb, h=h, w_=w, bias=bias))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), bias, stride=2, padding=1)
    assert _rel(out.permute(0, 3, 1, 2), ref) < 6e-3


@pytest.mark.parametrize("B,H,d,nq,nk", [(2, 8, 40, 4096, 4096), (2, 8, 80, 1024, 1024), (3, 8, 160, 256, 256),
                                          (2, 8, 160, 64, 64), (2, 8, 40, 4096, 77), (2, 8, 80, 1024, 77),
                                          (2, 8, 160, 64, 77), (2, 4, 8, 64, 64), (2, 4, 16, 16, 77),
                                          (3, 4, 32, 4, 4), (2, 4, 32, 1, 77), (1, 2, 64, 300, 333),
                                          (1, 3, 96, 384, 200), (1, 2, 112, 300, 333)])
@pytest.mark.parametrize("vdt", [torch.bfloat16, torch.float16])
def test_attention(ops, B, H, d, nq, nk, vdt):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + d + nq)
    C_ = H * d
    q = (torch.randn(B, nq, C_, device=_dev(), generator=g)).to(BF16)
    k = (torch.randn(B, nk, C_, device=_dev(), generator=g)).to(BF16)
    v = (torch.randn(B, nk, C_, device=_dev(), generator=g)).to(BF16)
    vt_ld = (nk + 7) // 8 * 8
    vt = torch.full((B, C_, vt_ld), float("nan"), device=_dev(), dtype=vdt)
    vt[:, :, :nk] = v.permute(0, 2, 1).to(vdt)
    out = torch.full((B, nq, C_), float("nan"), device=_dev(), dtype=BF16)
    scale = 1.0 / math.sqrt(d)
    ops.run(ops.attn_desc(q=q, k=k, vt=vt, out=out, batch=B, heads=H, d=d, nq=nq, nk=nk, q_ld=C_, k_ld=C_,
                          vt_ld=vt_ld, o_ld=C_, q_batch_stride=nq * C_, k_batch_stride=nk * C_, scale=scale))
    torch.cuda.synchronize()
    qh = q.float().reshape(B, nq, H, d).transpose(1, 2)
    kh = k.float().reshape(B, nk, H, d).transpose(1, 2)
    vh = v.float().reshape(B, nk, H, d).transpose(1, 2)
    ref = F.scaled_dot_product_attention(qh, kh, vh).transpose(1, 2).reshape(B, nq, C_)
    assert torch.isfinite(out.float()).all()
    assert _rel(out, ref) < 1e-2, _rel(out, ref)


def test_attention_large_logits(ops):
    """rows whose running max jumps by far more than the lazy-rescale threshold"""
    B, H, d, nq, nk = 1, 2, 40, 256, 1024
    g = torch.Generator(device="cuda").manual_seed(77)
    C_ = H * d
    q = (torch.randn(B, nq, C_, device=_dev(), generator=g) * 4).to(BF16)
    k = torch.randn(B, nk, C_, device=_dev(), generator=g)
    k = (k * torch.linspace(0.2, 6.0, nk, device=_dev())[None, :, None]).to(BF16)  # later keys dominate
    v = torch.randn(B, nk, C_, device=_dev(), generator=g).to(BF16)
    vt = v.permute(0, 2, 1).contiguous().to(torch.float16)  # fp16 V^T -> dual-tile kernel
    out = torch.zeros(B, nq, C_, device=_dev(), dtype=BF16)
    ops.run(ops.attn_desc(q=q, k=k, vt=vt, out=out, batch=B, heads=H, d=d, nq=nq, nk=nk, q_ld=C_, k_ld=C_,
                          vt_ld=nk, o_ld=C_, q_batch_stride=nq * C_, k_batch_stride=nk * C_, scale=1 / math.sqrt(d)))
    torch.cuda.synchronize()
    qh = q.float().reshape(B, nq, H, d).transpose(1, 2)
    kh = k.float().reshape(B, nk, H, d).transpose(1, 2)
    vh = v.float().reshape(B, nk, H, d).transpose(1, 2)
    ref = F.scaled_dot_product_attention(qh, kh, vh).transpose(1, 2).reshape(B, nq, C_)
    assert _rel(out, ref) < 1.5e-2, _rel(out, ref)


@pytest.mark.parametrize("B,hw,c0,c1,groups,silu", [(2, 4096, 320, 0, 32, True), (3, 256, 1280, 1280, 32, True),
                                                    (2, 1024, 640, 320, 32, False), (2, 64, 32, 0, 32, True),
                                                    (2, 64, 1280, 640, 32, True), (1, 4, 64, 64, 8, True)])
def test_group_norm(ops, B, hw, c0, c1, groups, silu):
    g = torch.Generator(device="cuda").manual_seed(hw + c0)
    C_ = c0 + c1
    x0 = (torch.randn(B, hw, c0, device=_dev(), generator=g) * 2 + 0.5).to(BF16)
    x1 = (torch.randn(B, hw, c1, device=_dev(), generator=g) - 0.3).to(BF16) if c1 else None
    gamma = torch.randn(C_, device=_dev(), generator=g)
    beta = torch.randn(C_, device=_dev(), generator=g)
    # garbage-filled scratch + stats_prezeroed=False: the call has to clear its own ticket counters
    stats = torch.full(((ops.gn_scratch_bytes(B, hw, c0 + c1, groups) + 3) // 4,), float("nan"), device=_dev())
    y = torch.zeros(B, hw, C_, device=_dev(), dtype=BF16)
    ops.run(ops.gn_desc(x0=x0, x1=x1, c0=c0, c1=c1, batch=B, hw=hw, groups=groups, gamma=gamma, beta=beta,
                        eps=1e-5, silu=silu, stats=stats, y=y))
    torch.cuda.synchronize()
    x = torch.cat([x0, x1], -1) if c1 else x0
    ref = F.group_norm(x.float().permute(0, 2, 1), groups, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    assert _rel(y.permute(0, 2, 1), ref) < 5e-3, _rel(y.permute(0, 2, 1), ref)
    # second call on the same scratch without clearing it: the first call left the ticket counters at zero,
    # and the statistics are reduced in a fixed order, so the result is bit-identical
    y2 = torch.zeros_like(y)
    ops.run(ops.gn_desc(x0=x0, x1=x1, c0=c0, c1=c1, batch=B, hw=hw, groups=groups, gamma=gamma, beta=beta,
                        eps=1e-5, silu=silu, stats=stats, y=y2, stats_prezeroed=True))
    torch.cuda.synchronize()
    assert torch.equal(y, y2)


@pytest.mark.parametrize("rows,c", [(4096, 320), (1000, 640), (77, 1280), (5, 32), (64, 128)])
def test_layer_norm(ops, rows, c):
    g = torch.Generator(device="cuda").manual_seed(rows + c)
    x = (torch.randn(rows, c, device=_dev(), generator=g) * 3 + 1).to(BF16)
    gamma = torch.randn(c, device=_dev(), generator=g)
    beta = torch.randn(c, device=_dev(), generator=g)
    y = torch.zeros_like(x)
    ops.layer_norm(x, y, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (c,), gamma, beta, 1e-5)
    assert _rel(y, ref) < 4e-3


def test_small_ops(ops):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(2, 6, 10, 64, device=_dev(), generator=g).to(BF16)
    y = torch.zeros(2, 12, 20, 64, device=_dev(), dtype=BF16)
    ops.upsample2x(x, y)
    ref = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(y.float(), ref)
    a = torch.randn(4096, device=_dev(), generator=g).to(BF16)
    b = torch.randn(4096, device=_dev(), generator=g).to(BF16)
    c = torch.zeros_like(a)
    ops.add(a, b, c)
    assert torch.equal(c, (a.float() + b.float()).to(BF16))
    # layout conversion round trip
    z = torch.randn(3, 9, 7, 5, device=_dev(), generator=g)
    zn = ops.nchw_to_nhwc(z, 16)
    assert zn.shape == (3, 7, 5, 16)
    assert torch.equal(zn[..., :9].float(), z.to(BF16).float().permute(0, 2, 3, 1))
    assert (zn[..., 9:] == 0).all()
    back = ops.nhwc_to_nchw(zn, 9)
    assert torch.equal(back, z.to(BF16).float())
    # the timestep embedding is checked per element against fp64 in test_norm_and_small_kernels_gpu.py
    torch.cuda.synchronize()


U32 = 2.0 ** -24  # unit round-off of fp32


def _cfg_eps(eps, gscale, do_cfg, B):
    """(eps after CFG, |eps| magnitude of the terms) in fp64 from the stored eps rows (channels 0..3)"""
    e = eps.double()
    if not do_cfg:
        return e[:B], e[:B].abs()
    u, c = e[:B], e[B:2 * B]
    return u + gscale * (c - u), u.abs() + abs(gscale) * (c.abs() + u.abs())


def ref_cfg_ddim(eps, x, noise, cf, gscale, do_cfg, B, blend=None):
    """fp64 evaluation of the pp_cfg_ddim_desc row formula (include/powerpaint_b200.h) on the stored fp32 inputs:
    (x_prev, bound). The bound is a few fp32 round-offs of the sum of the magnitudes of every term, the most an fp32
    evaluation of the same expression (with or without FMA contraction) can be off."""
    cf = [float(v) for v in cf]
    e, ea = _cfg_eps(eps, gscale, do_cfg, B)
    xd = x.double()
    inv = 1.0 / cf[0]
    x0 = (xd - cf[1] * e) * inv
    x0a = (xd.abs() + abs(cf[1]) * ea) * abs(inv)
    nz = noise.double() if noise is not None else torch.zeros_like(xd)
    xp = cf[2] * x0 + cf[3] * e + cf[4] * nz
    xpa = abs(cf[2]) * x0a + abs(cf[3]) * ea + abs(cf[4]) * nz.abs()
    if blend is not None:
        o, m, nn = (t.double() for t in blend)
        m = m.reshape(1, -1, 1)
        a = cf[7]
        s1a = max(1 - a * a, 0.0) ** 0.5
        xp = (1 - m) * (a * o[None] + s1a * nn) + m * xp
        # sqrtf(1 - a*a) is off by about u / (1 - a^2) relative: a < 0.95 keeps that within the factor below
        xpa = (1 - m).abs() * (abs(a) * o[None].abs() + s1a * nn.abs()) * 16 + m.abs() * xpa
    return xp, 12 * U32 * xpa + 1e-30


def ref_unipc(eps, x, last, m1, m2, u, gscale, do_cfg, B):
    """fp64 evaluation of the pp_unipc_desc row formula: (x_next, x_c, m_t, bound of each)"""
    u = [float(v) for v in u]
    e, ea = _cfg_eps(eps, gscale, do_cfg, B)
    xd, ld, a1, a2 = x.double(), last.double(), m1.double(), m2.double()
    mt = u[0] * xd + u[1] * e
    mta = abs(u[0]) * xd.abs() + abs(u[1]) * ea
    if u[2] != 0:
        xc = u[3] * ld + u[4] * a1 + u[5] * a2 + u[6] * mt
        xca = abs(u[3]) * ld.abs() + abs(u[4]) * a1.abs() + abs(u[5]) * a2.abs() + abs(u[6]) * mta
    else:
        xc, xca = xd, xd.abs() * 0
    xn = u[7] * xc + u[8] * mt + u[9] * a1
    xna = abs(u[7]) * (xca + xc.abs()) + abs(u[8]) * mta + abs(u[9]) * a1.abs()
    b = lambda mag: 12 * U32 * mag + 1e-30  # noqa: E731
    return xn, xc, mt, b(xna), b(xca), b(mta)


def _eps_input(kind, nb, hw, g):
    """(tensor the kernel reads, eps_fp32, eps_ld, channels 0..3 as the kernel sees them)"""
    if kind == "fp32_vec":
        e = torch.randn(nb, hw, 4, device=_dev(), generator=g)
        return e, True, 4, e
    if kind == "fp32_strided":
        e = torch.randn(nb, hw, 8, device=_dev(), generator=g)
        return e, True, 8, e[..., :4]
    e = torch.randn(nb, hw, 8, device=_dev(), generator=g).to(BF16)
    return e, False, 8, e[..., :4].float()


def _within(got, ref, bound):
    return bool(((got.double() - ref).abs() <= bound).all())


def test_cfg_ddim(ops):
    """pp_cfg_ddim_step against the fp64 row formula to an fp32 round-off bound, per element; next_in equal to the bf16
    rounding of the stored latents bit for bit, the extra channels to bf16 of `extra` (one set per copy with
    extra_per_copy) followed by zeros, and channels 4 and up untouched without extra"""
    for case in ("cfg_extra", "no_cfg", "bf16_strided", "fp32_strided", "guidance_from_coef", "extra_per_copy", "blend",
                 "latents_only"):
        _cfg_ddim_case(ops, case)


def _cfg_ddim_case(ops, case):
    B, hw, C = 3, 37 * 13, 16
    g = torch.Generator(device="cuda").manual_seed(9)
    do_cfg = case != "no_cfg"
    nb = 2 * B if do_cfg else B
    eps, eps_fp32, eps_ld, eps_view = _eps_input({"bf16_strided": "bf16_strided", "fp32_strided": "fp32_strided"}
                                                 .get(case, "fp32_vec"), nb, hw, g)
    lat = torch.randn(B, hw, 4, device=_dev(), generator=g)
    n_copies = 2 if do_cfg else 1
    extra_c = 0 if case in ("blend", "latents_only") else 5
    extra = torch.randn((n_copies if case == "extra_per_copy" else 1) * B, hw, 5, device=_dev(), generator=g)
    noise = torch.randn(B, hw, 4, device=_dev(), generator=g) if case != "blend" else None
    a_t, a_p, sigma = 0.3, 0.45, 0.1
    row = [math.sqrt(a_t), math.sqrt(1 - a_t), math.sqrt(a_p), math.sqrt(1 - a_p - sigma ** 2), sigma, 3.25, 0, 0.7]
    coef = torch.tensor([[float("nan")] * 8, row], device=_dev(), dtype=torch.float32)
    gscale = 3.25 if case == "guidance_from_coef" else 7.5
    blend = None
    if case == "blend":
        blend = (torch.randn(hw, 4, device=_dev(), generator=g), torch.rand(hw, device=_dev(), generator=g),
                 torch.randn(B, hw, 4, device=_dev(), generator=g))
        blend[1][: hw // 2] = (blend[1][: hw // 2] > 0.5).float()  # the production mask is binary; the rest is not
    step = torch.tensor([1], device=_dev(), dtype=torch.int32)
    nxt = torch.full((n_copies * B, hw, C), float("nan"), device=_dev(), dtype=BF16)
    lat_in = lat.clone()
    ops.run(ops.cfg_ddim_desc(eps=eps, eps_fp32=eps_fp32, eps_ld=eps_ld, latents=lat, coef=coef, step_idx=step,
                              advance_step=True, noise=noise, guidance_scale=0.0 if case == "guidance_from_coef" else 7.5,
                              guidance_from_coef=case == "guidance_from_coef", do_cfg=do_cfg, batch=B, hw=hw,
                              next_in=nxt, next_c=C, n_copies=n_copies, extra=extra if extra_c else None,
                              extra_c=extra_c, extra_per_copy=case == "extra_per_copy",
                              blend_x0=blend[0] if blend else None, blend_mask=blend[1] if blend else None,
                              blend_noise=blend[2] if blend else None))
    torch.cuda.synchronize()
    ref, bound = ref_cfg_ddim(eps_view, lat_in, noise, row, gscale, do_cfg, B, blend)
    assert _within(lat, ref, bound), (case, ((lat.double() - ref).abs() / bound).max().item())
    assert step.item() == 2
    for cpy in range(n_copies):
        blk = nxt[cpy * B:(cpy + 1) * B]
        assert torch.equal(blk[..., :4], lat.to(BF16)), (case, cpy)
        if extra_c:
            ex = extra[cpy * B:(cpy + 1) * B] if case == "extra_per_copy" else extra
            assert torch.equal(blk[..., 4:9], ex.to(BF16)), cpy
            assert (blk[..., 9:] == 0).all()
        else:
            assert blk[..., 4:].isnan().all()  # only the 4 latent channels are refreshed


def test_unipc_step_kernel_matches_the_row_formula_and_replays_bit_identically(ops):
    """pp_unipc_step against the fp64 row formula to an fp32 round-off bound, per element, for the corrector on and off,
    CFG on and off, the three eps layouts and 1-3 copies of the net input; eager, program and graph runs
    bit-identical; m2 <- m1 exactly, and next_in the bf16 rounding of the stored latents"""
    g = torch.Generator(device="cuda").manual_seed(0)
    B, hw, C = 2, 37 * 13, 16
    ucoef = torch.randn(3, 12, device=_dev(), generator=g)
    coef = torch.full((3, 8), float("nan"), device=_dev())
    coef[:, 5] = torch.tensor([7.5, 3.0, 1.5])
    for use_c in (0.0, 1.0):
        ucoef[1, 2] = use_c
        for do_cfg in (False, True):
            for n_copies in (1, 2, 3):
                for eps_kind in ("fp32_vec", "fp32_strided", "bf16_strided"):
                    nb = 2 * B if do_cfg else B
                    eps, eps_fp32, eps_ld, eps_view = _eps_input(eps_kind, nb, hw, g)
                    state0 = [torch.randn(B, hw, 4, device=_dev(), generator=g) for _ in range(4)]
                    outs = []
                    for mode in ("eager", "program", "graph"):
                        lat, last, m1, m2 = (t.clone() for t in state0)
                        nxt = torch.full((n_copies * B, hw, C), float("nan"), dtype=BF16, device=_dev())
                        idx = torch.tensor([1], dtype=torch.int32, device=_dev())
                        d = ops.unipc_desc(eps=eps, eps_fp32=eps_fp32, eps_ld=eps_ld, latents=lat, last_sample=last,
                                           m1=m1, m2=m2, coef=coef, ucoef=ucoef, step_idx=idx,
                                           advance_step=mode != "eager", do_cfg=do_cfg, batch=B, hw=hw, next_in=nxt,
                                           next_c=C, n_copies=n_copies)
                        if mode == "eager":
                            ops.run(d)
                        else:
                            p = ops.Program()
                            p.add(d)
                            if mode == "graph":
                                p.build_graph()
                                p.launch()
                            else:
                                p.run()
                        torch.cuda.synchronize()
                        assert int(idx) == (1 if mode == "eager" else 2)
                        outs.append((lat, last, m1, m2, nxt))
                    tag = (use_c, do_cfg, n_copies, eps_kind)
                    xn, xc, mt, bxn, bxc, bmt = ref_unipc(eps_view, *state0, ucoef[1], float(coef[1, 5]), do_cfg, B)
                    lat, last, m1, m2, nxt = outs[0]
                    assert _within(lat, xn, bxn), tag
                    assert _within(last, xc, bxc), tag
                    assert _within(m1, mt, bmt), tag
                    assert torch.equal(m2, state0[2]), tag
                    if not use_c:
                        assert torch.equal(last, state0[0]), tag  # x_c = x: the stored sample is x itself
                    for c in range(n_copies):
                        assert torch.equal(nxt[c * B:(c + 1) * B, :, :4], lat.to(BF16)), tag
                    assert nxt[..., 4:].isnan().all(), tag
                    for o in outs[1:]:  # bit for bit (next_in keeps its NaN channels)
                        assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(o, outs[0])), tag


def test_program_and_graph(ops):
    """record GN -> conv -> LN in a program, replay as launches and as a CUDA graph"""
    from powerpaint_b200 import _native as nat

    nb, h, w, c = 2, 16, 16, 64
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(nb, h, w, c, device=_dev(), generator=g).to(BF16)
    gamma = torch.ones(c, device=_dev()); beta = torch.zeros(c, device=_dev())
    xn = torch.zeros_like(x)
    wt = (torch.randn(c, c, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * c)).to(BF16)
    wp = ops.pack_conv3x3_weight(wt.float())
    y = torch.zeros_like(x)
    z = torch.zeros_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        prog = ops.Program()
        prog.add(ops.gn_desc(x0=x, x1=None, c0=c, c1=0, batch=nb, hw=h * w, groups=32, gamma=gamma, beta=beta,
                             eps=1e-5, silu=True, y=xn))
        prog.add(ops.gemm_desc(a0=xn, w=wp, out=y, N_=c, a_mode=nat.PP_A_CONV3X3, c0=c, nb=nb, h=h, w_=w))
        prog.add_layer_norm(y, z, gamma, beta, nb * h * w, c, 1e-5)
        assert prog.num_ops == 3 and prog.num_launches == 4
        prog.run()
        s.synchronize()
        z1 = z.clone()
        z.zero_()
        prog.build_graph()
        prog.launch()
        s.synchronize()
    # replay == plain launches, bit for bit (the GroupNorm statistics are reduced in a fixed order)
    assert torch.equal(z, z1)
    ref = F.silu(F.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma, beta, 1e-5)).to(BF16).float()
    ref = F.conv2d(ref, wt.float(), None, padding=1).to(BF16).float().permute(0, 2, 3, 1)
    ref = F.layer_norm(ref, (c,), gamma, beta, 1e-5)
    assert _rel(z, ref) < 2e-2


# --------------------------------------------------------------------------- round-2 kernels
def _gn_from_producers(ops, prods, groups, silu=True, eps=1e-5):
    """prods: list of (out [B, hw, c] bf16, partials, geometry); GroupNorm over their channel concat
    driven by the producers' epilogue statistics, against torch on the stored bf16 values"""
    x0, p0, g0 = prods[0]
    x1, p1, g1 = prods[1] if len(prods) > 1 else (None, None, None)
    B, hw, c0 = x0.shape
    c1 = x1.shape[-1] if x1 is not None else 0
    gen = torch.Generator(device="cuda").manual_seed(c0 + c1)
    gamma = torch.randn(c0 + c1, device=_dev(), generator=gen)
    beta = torch.randn(c0 + c1, device=_dev(), generator=gen)
    y = torch.zeros(B, hw, c0 + c1, device=_dev(), dtype=BF16)
    stats = torch.full(((ops.gn_scratch_bytes(B, hw, c0 + c1, groups) + 3) // 4,), float("nan"), device=_dev())
    ops.run(ops.gn_desc(x0=x0, x1=x1, c0=c0, c1=c1, batch=B, hw=hw, groups=groups, gamma=gamma, beta=beta, eps=eps,
                        silu=silu, stats=stats, y=y, part0=p0, geom0=g0, part1=p1, geom1=g1))
    torch.cuda.synchronize()
    x = torch.cat([x0, x1], -1) if x1 is not None else x0
    ref = F.group_norm(x.float().permute(0, 2, 1), groups, gamma, beta, eps)
    if silu:
        ref = F.silu(ref)
    return _rel(y.permute(0, 2, 1), ref)


def _conv_with_stats(ops, nb, h, w, cin, cout, seed, stride2=False, block_n=0, mean_shift=0.0):
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(nb, h, w, cin, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(cout, cin, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * cin)).to(BF16)
    bias = torch.randn(cout, device=_dev(), generator=g) + mean_shift
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if stride2 else (h, w)
    out = torch.full((nb, ho * wo, cout), float("nan"), device=_dev(), dtype=BF16)
    d = ops.gemm_desc(a0=x, w=ops.pack_conv3x3_weight(wt.float()), out=out, N_=cout,
                      a_mode=nat.PP_A_CONV3X3_S2 if stride2 else nat.PP_A_CONV3X3, c0=cin, nb=nb, h=h, w_=w, bias=bias,
                      block_n=block_n)
    geo = ops.gemm_stats_geometry(d)
    assert geo.supported, "this shape should be able to emit statistics"
    part = torch.full((int(geo.bytes) // 4,), float("nan"), device=_dev())
    ops.attach_chan_stats(d, part)
    ops.run(d)
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), wt.float(), bias, stride=2 if stride2 else 1, padding=1)
    assert _rel(out.view(nb, ho, wo, cout).permute(0, 3, 1, 2), ref) < 6e-3
    return out, part, geo


@pytest.mark.parametrize("nb,h,w,cin,cout,bn,s2", [(2, 64, 64, 64, 320, 0, False), (5, 8, 8, 128, 1280, 0, False),
                                                   (3, 16, 16, 64, 640, 128, False), (2, 12, 20, 64, 64, 64, False),
                                                   (3, 32, 32, 64, 256, 256, False), (2, 32, 32, 64, 320, 0, True),
                                                   (3, 4, 4, 64, 320, 0, False), (2, 13, 27, 64, 320, 0, True)])
def test_group_norm_from_conv_epilogue_stats(ops, nb, h, w, cin, cout, bn, s2):
    out, part, geo = _conv_with_stats(ops, nb, h, w, cin, cout, seed=nb + h + cout, stride2=s2, block_n=bn)
    groups = 32 if cout % 32 == 0 else 8
    assert _gn_from_producers(ops, [(out, part, geo)], groups) < 5e-3


def test_group_norm_from_stats_concat_of_conv_and_linear(ops):
    """the up-path concat: hidden state from a 3x3 conv, skip from a transformer's proj_out (matrix mode,
    hw = 256 rows per sample and hw = 64: two samples per 128-row tile)"""
    for hw_side, nb in ((16, 3), (8, 5)):
        hw = hw_side * hw_side
        out0, p0, g0 = _conv_with_stats(ops, nb, hw_side, hw_side, 64, 640, seed=hw)
        g = torch.Generator(device="cuda").manual_seed(hw + 1)
        a = torch.randn(nb * hw, 320, device=_dev(), generator=g).to(BF16)
        wl = (torch.randn(320, 320, device=_dev(), generator=g) / math.sqrt(320)).to(BF16)
        res = torch.randn(nb * hw, 320, device=_dev(), generator=g).to(BF16)
        out1 = torch.zeros(nb, hw, 320, device=_dev(), dtype=BF16)
        d = ops.gemm_desc(a0=a, w=wl, out=out1, N_=320, M=nb * hw, res1=res, rows_per_group=hw)
        geo = ops.gemm_stats_geometry(d)
        assert geo.supported and geo.segs == max(1, 128 // hw)
        p1 = torch.full((int(geo.bytes) // 4,), float("nan"), device=_dev())
        ops.attach_chan_stats(d, p1)
        ops.run(d)
        torch.cuda.synchronize()
        assert _rel(out1.view(nb * hw, 320), a.float() @ wl.float().t() + res.float()) < 6e-3
        assert _gn_from_producers(ops, [(out0, p0, g0), (out1, p1, geo)], 32) < 5e-3


def test_group_norm_large_mean_small_spread(ops):
    """a group whose mean dwarfs its spread (late-UNet activations on real checkpoints): the statistics are
    combined as (count, mean, M2) in fp64, so the variance does not cancel — both statistics paths"""
    B, hw, c = 2, 4096, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.randn(B, hw, c, device=_dev(), generator=g) * 0.25 + 120.0).to(BF16)
    gamma = torch.ones(c, device=_dev())
    beta = torch.zeros(c, device=_dev())
    y = torch.zeros_like(x)
    ops.run(ops.gn_desc(x0=x, x1=None, c0=c, c1=0, batch=B, hw=hw, groups=8, gamma=gamma, beta=beta, eps=1e-5,
                        silu=False, y=y))
    torch.cuda.synchronize()
    ref = F.group_norm(x.double().permute(0, 2, 1), 8, None, None, 1e-5).float()
    assert _rel(y.permute(0, 2, 1), ref) < 1e-2, _rel(y.permute(0, 2, 1), ref)
    out, part, geo = _conv_with_stats(ops, 2, 32, 32, 64, 64, seed=77, mean_shift=200.0)
    assert _gn_from_producers(ops, [(out, part, geo)], 8, silu=False) < 1e-2


@pytest.mark.parametrize("nb,h,w,c", [(2, 13, 27, 64), (1, 3, 2, 32), (2, 15, 15, 128), (3, 7, 64, 32)])
def test_conv3x3_stride2_odd_sizes(ops, nb, h, w, c):
    """Downsample2D on an odd feature map (latents that are not multiples of 8): output ceil(h/2) x ceil(w/2)"""
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(h * w + c)
    x = torch.randn(nb, c, h, w, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(c, c, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * c)).to(BF16)
    bias = torch.randn(c, device=_dev(), generator=g)
    ho, wo = (h + 1) // 2, (w + 1) // 2
    out = torch.full((nb, ho, wo, c), float("nan"), device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x.permute(0, 2, 3, 1).contiguous(), w=ops.pack_conv3x3_weight(wt.float()), out=out, N_=c,
                          a_mode=nat.PP_A_CONV3X3_S2, c0=c, nb=nb, h=h, w_=w, bias=bias))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), bias, stride=2, padding=1)
    assert ref.shape[-2:] == (ho, wo)
    assert _rel(out.permute(0, 3, 1, 2), ref) < 6e-3


@pytest.mark.parametrize("nb,h,w,c", [(2, 64, 64, 128), (1, 16, 24, 32), (2, 9, 7, 64)])
def test_conv3x3_stride2_pad_bottom_right(ops, nb, h, w, c):
    """the VAE encoder's Downsample2D(padding=0): conv(F.pad(x, (0, 1, 0, 1)), stride 2)"""
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(h + w + c)
    x = torch.randn(nb, c, h, w, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(c, c, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * c)).to(BF16)
    bias = torch.randn(c, device=_dev(), generator=g)
    ref = F.conv2d(F.pad(x.float(), (0, 1, 0, 1)), wt.float(), bias, stride=2)
    ho, wo = ref.shape[-2:]
    assert (ho, wo) == (h // 2, w // 2)
    out = torch.full((nb, ho, wo, c), float("nan"), device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x.permute(0, 2, 3, 1).contiguous(), w=ops.pack_conv3x3_weight(wt.float()), out=out, N_=c,
                          a_mode=nat.PP_A_CONV3X3_S2P0, c0=c, nb=nb, h=h, w_=w, bias=bias))
    torch.cuda.synchronize()
    assert _rel(out.permute(0, 3, 1, 2), ref) < 6e-3


def test_upsample_nearest_to_size_and_device_alpha_and_quick_gelu(ops):
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(4)
    for (h, w, ho, wo) in ((54, 40, 107, 80), (6, 10, 12, 20), (5, 5, 9, 10), (27, 20, 54, 40)):
        x = torch.randn(2, h, w, 64, device=_dev(), generator=g).to(BF16)
        y = torch.zeros(2, ho, wo, 64, device=_dev(), dtype=BF16)
        ops.upsample_nearest(x, y)
        ref = F.interpolate(x.permute(0, 3, 1, 2).float(), size=(ho, wo), mode="nearest").permute(0, 2, 3, 1)
        assert torch.equal(y.float(), ref), (h, w, ho, wo)
    # alpha read from a device table through a device-side step index
    M, N, K = 256, 320, 320
    a = torch.randn(M, K, device=_dev(), generator=g).to(BF16)
    w_ = (torch.randn(N, K, device=_dev(), generator=g) / math.sqrt(K)).to(BF16)
    bias = torch.randn(N, device=_dev(), generator=g)
    table = torch.zeros(4, 8, device=_dev())
    table[:, 6] = torch.tensor([1.0, 0.5, 0.0, 2.0])
    step = torch.zeros(1, dtype=torch.int32, device=_dev())
    for mode_n in (N, 4):  # fast bf16 epilogue and the generic one (ragged N)
        out = torch.zeros(M, mode_n, device=_dev(), dtype=BF16)
        d = ops.gemm_desc(a0=a, w=w_[:mode_n].contiguous(), out=out, N_=mode_n, M=M, bias=bias[:mode_n].contiguous(),
                          alpha=0.5, alpha_dev=table[:, 6], alpha_step=step, alpha_stride=8)
        for i, s in enumerate([1.0, 0.5, 0.0, 2.0]):
            step.fill_(i)
            ops.run(d)
            torch.cuda.synchronize()
            ref = (a.float() @ w_[:mode_n].float().t() + bias[:mode_n]) * (0.5 * s)
            assert (out.float() - ref).abs().max().item() < 0.03 * max(ref.abs().max().item(), 1.0)
    out = torch.zeros(M, N, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=a, w=w_, out=out, N_=N, M=M, bias=bias, act=nat.PP_ACT_QUICK_GELU))
    torch.cuda.synchronize()
    pre = a.float() @ w_.float().t() + bias
    assert _rel(out, pre * torch.sigmoid(1.702 * pre)) < 6e-3


def test_attention_16384_tokens_d40(ops):
    """the C4 (1024^2 outpaint) self-attention shape: 128 x 128 latent tokens, d = 40"""
    B, H, d, n = 1, 2, 40, 16384
    g = torch.Generator(device="cuda").manual_seed(11)
    C_ = H * d
    q = torch.randn(B, n, C_, device=_dev(), generator=g).to(BF16)
    k = torch.randn(B, n, C_, device=_dev(), generator=g).to(BF16)
    v = torch.randn(B, n, C_, device=_dev(), generator=g).to(torch.float16)
    vt = v.transpose(1, 2).contiguous()
    out = torch.full((B, n, C_), float("nan"), device=_dev(), dtype=BF16)
    ops.run(ops.attn_desc(q=q, k=k, vt=vt, out=out, batch=B, heads=H, d=d, nq=n, nk=n, q_ld=C_, k_ld=C_, vt_ld=n,
                          o_ld=C_, q_batch_stride=n * C_, k_batch_stride=n * C_, scale=1.0 / math.sqrt(d)))
    torch.cuda.synchronize()
    qh, kh, vh = (t.float().view(B, n, H, d).transpose(1, 2) for t in (q, k, v))
    ref = F.scaled_dot_product_attention(qh, kh, vh).transpose(1, 2).reshape(B, n, C_)
    assert torch.isfinite(out.float()).all()
    assert _rel(out, ref) < 1.5e-2, _rel(out, ref)


def test_attention_16384_tokens_full_grid_is_reproducible(ops):
    """C4's launch (UNet batch 4 x 8 heads x 16384 tokens, 2048 CTAs, 128 key blocks each) repeated: every run must be
    finite and bit-identical to the first. Guards the hand-over of P between the four softmax warps of a group: with
    three score buffers a warp could run a block ahead and release PV(j) before a slower warp had written its rows
    (seen as NaN rows in the C4 loop; the outcome changed from run to run)."""
    B, H, d, n = 4, 8, 40, 16384
    g = torch.Generator(device="cuda").manual_seed(12)
    C_ = H * d
    q = torch.randn(B, n, C_, device=_dev(), generator=g).to(BF16)
    k = torch.randn(B, n, C_, device=_dev(), generator=g).to(BF16)
    vt = torch.randn(B, C_, n, device=_dev(), generator=g).to(torch.float16)
    outs = []
    for _ in range(4):
        out = torch.full((B, n, C_), float("nan"), device=_dev(), dtype=BF16)
        ops.run(ops.attn_desc(q=q, k=k, vt=vt, out=out, batch=B, heads=H, d=d, nq=n, nk=n, q_ld=C_, k_ld=C_, vt_ld=n,
                              o_ld=C_, q_batch_stride=n * C_, k_batch_stride=n * C_, scale=1.0 / math.sqrt(d)))
        torch.cuda.synchronize()
        assert torch.isfinite(out.float()).all()
        assert out.float().abs().max().item() <= vt.float().abs().max().item()  # a convex combination of V rows
        outs.append(out)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def _ln_fold_pack(w, gamma, beta, bias=None):
    """the host-side fold the engine performs (ops.fold_layer_norm_into_linear, checked on the CPU in
    tests/test_abi_and_host.py): W' = W * gamma (bf16), u = row sums of the bf16 W', b' = W beta (+ bias)"""
    from powerpaint_b200 import ops as o

    return o.fold_layer_norm_into_linear(w, gamma, beta, bias)


def _producer_with_row_stats(ops, M, C, K, seed, offset=0.0, bn=0):
    """x = a @ wp^T + bias + res (+ a common offset) with per-row LayerNorm records from the epilogue"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device=_dev(), generator=g).to(BF16)
    wp = (torch.randn(C, K, device=_dev(), generator=g) / math.sqrt(K)).to(BF16)
    bias = torch.randn(C, device=_dev(), generator=g) + offset
    res = torch.randn(M, C, device=_dev(), generator=g).to(BF16)
    x = torch.full((M, C), float("nan"), device=_dev(), dtype=BF16)
    d = ops.gemm_desc(a0=a, w=wp, out=x, N_=C, M=M, bias=bias, res1=res, block_n=bn)
    nrec = ops.gemm_row_stats_records(d)
    assert nrec > 0
    rec = torch.full((nrec, M + 3, 4), float("nan"), device=_dev(), dtype=torch.float32)  # ld > M on purpose
    final = torch.full((M, 2), float("nan"), device=_dev(), dtype=torch.float32)
    ticket = torch.zeros((M + 127) // 128, device=_dev(), dtype=torch.int32)
    ops.attach_row_stats(d, rec, final, ticket, 1e-5)
    for _ in range(2):  # twice: the tickets must be back at zero after a launch
        ops.run(d)
    torch.cuda.synchronize()
    assert (ticket == 0).all()
    ref = a.float() @ wp.float().t() + bias + res.float()
    assert _rel(x, ref) < 6e-3
    # {rstd, -rstd * mean} of the fp32 rows the epilogue computed
    mean, var = ref.double().mean(1), ref.double().var(1, unbiased=False)
    rstd = (var + 1e-5).rsqrt()
    assert torch.isfinite(final).all()
    assert ((final[:, 0].double() - rstd).abs() / rstd).max().item() < 2e-3
    assert (final[:, 1].double() + rstd * mean).abs().max().item() < 2e-3 * (1 + (rstd * mean).abs().max().item())
    return x, rec, ref, final


@pytest.mark.parametrize("M,C,bn,offset,K", [(256, 320, 0, 0.0, 192), (1000, 640, 0, 0.0, 192), (300, 1280, 64, 0.0, 192),
                                             (128, 32, 0, 0.0, 192), (512, 320, 256, 300.0, 192),
                                             # K = 1280: the record count must be the one of the launch that actually
                                             # runs (the one with row_stats attached)
                                             (1024, 1280, 0, 0.0, 1280)])
def test_gemm_row_stats_records(ops, M, C, bn, offset, K):
    """the records a producer emits combine to the mean / variance of the rows it computed — the fp32 values before
    the bf16 rounding of the store, which is what an fp32 LayerNorm of the exact activations would see (for a large
    common offset the stored bf16 values carry quantisation noise of their own: at 300 the bf16 step is 2) — also for
    a large common offset (shifted sums: no cancellation)"""
    x, rec, xf32, _ = _producer_with_row_stats(ops, M, C, K, M + C, offset, bn)
    r = rec[:, :M].double()
    cnt = r[..., 3]
    assert torch.isfinite(r).all() and (cnt.sum(0) == C).all()
    mean_i = r[..., 2] + r[..., 0] / cnt.clamp(min=1)
    mean = (mean_i * cnt).sum(0) / C
    m2 = (r[..., 1] - r[..., 0] ** 2 / cnt.clamp(min=1) + cnt * (mean_i - mean[None]) ** 2).sum(0)
    xf = xf32.double()
    assert (mean - xf.mean(1)).abs().max().item() < 1e-4 * (1 + abs(offset))
    var_ref = xf.var(1, unbiased=False)
    assert ((m2 / C - var_ref).abs() / var_ref).max().item() < 2e-3


@pytest.mark.parametrize("M,C,N,bn", [(256, 320, 640, 0), (1000, 640, 1280, 0), (300, 1280, 1280, 256), (128, 32, 64, 0)])
def test_gemm_layer_norm_fold_plain(ops, M, C, N, bn):
    """LayerNorm(x) @ W^T + b with the LayerNorm applied algebraically in the consumer's epilogue, against
    F.layer_norm on the same bf16 x in fp32"""
    x, _, _, rec = _producer_with_row_stats(ops, M, C, 192, M + C + N)
    g = torch.Generator(device="cuda").manual_seed(11)
    w = torch.randn(N, C, device=_dev(), generator=g) / math.sqrt(C)
    gamma = 1 + 0.3 * torch.randn(C, device=_dev(), generator=g)
    beta = 0.3 * torch.randn(C, device=_dev(), generator=g)
    bias = torch.randn(N, device=_dev(), generator=g)
    wf, u, b = _ln_fold_pack(w, gamma, beta, bias)
    out = torch.full((M, N), float("nan"), device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x, w=wf, out=out, N_=N, M=M, bias=b, block_n=bn, ln=(rec, u, 1e-5)))
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w.t() + bias
    assert torch.isfinite(out.float()).all()
    assert _rel(out, ref) < 8e-3, _rel(out, ref)


def test_gemm_layer_norm_fold_transposed_and_geglu(ops):
    from powerpaint_b200 import _native as nat

    M, C, hw = 512, 320, 256
    x, _, _, rec = _producer_with_row_stats(ops, M, C, 320, 77)
    g = torch.Generator(device="cuda").manual_seed(12)
    gamma = 1 + 0.3 * torch.randn(C, device=_dev(), generator=g)
    beta = 0.3 * torch.randn(C, device=_dev(), generator=g)
    lnx = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5)
    # V^T: fp16 transposed store
    wv = torch.randn(C, C, device=_dev(), generator=g) / math.sqrt(C)
    wf, u, b = _ln_fold_pack(wv, gamma, beta)
    vt = torch.zeros(M // hw, C, hw, device=_dev(), dtype=torch.float16)
    ops.run(ops.gemm_desc(a0=x, w=wf, out=vt, N_=C, M=M, bias=b, epilogue=nat.PP_EPI_TRANSPOSED, t_rows=hw, t_ld=hw,
                          t_fp16=True, ln=(rec, u, 1e-5)))
    torch.cuda.synchronize()
    ref = (lnx @ wv.t()).view(M // hw, hw, C).transpose(1, 2)
    assert _rel(vt, ref) < 8e-3, _rel(vt, ref)
    # GEGLU
    Fh = 1280
    wg = torch.randn(2 * Fh, C, device=_dev(), generator=g) / math.sqrt(C)
    bg = torch.randn(2 * Fh, device=_dev(), generator=g)
    wf, u, b = _ln_fold_pack(wg, gamma, beta, bg)
    wi, ui = ops.pack_geglu_weight(wf.float(), u, 128)
    _, bi = ops.pack_geglu_weight(wf.float(), b, 128)
    out = torch.zeros(M, Fh, device=_dev(), dtype=BF16)
    ops.run(ops.gemm_desc(a0=x, w=wi, out=out, N_=2 * Fh, M=M, bias=bi, epilogue=nat.PP_EPI_GEGLU, block_n=128,
                          ln=(rec, ui, 1e-5)))
    torch.cuda.synchronize()
    y = lnx @ wg.t() + bg
    ref = y[:, :Fh] * F.gelu(y[:, Fh:])
    assert _rel(out, ref) < 8e-3, _rel(out, ref)


@pytest.mark.parametrize("M,C,hw,bn,fold", [(1024, 320, 256, 160, False), (1024, 320, 256, 160, True), (512, 128, 128, 128, True),
                                            (2048, 640, 1024, 160, True)])
def test_gemm_rows_then_transposed_qkv(ops, M, C, hw, bn, fold):
    """to_q | to_k | to_v^T of one self-attention as ONE launch: columns [0, 2C) row-major bf16, columns [2C, 3C)
    transposed fp16 through the staging tile (optionally with the LayerNorm fold), against the three separate products"""
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(M + C)
    w = torch.randn(3 * C, C, device=_dev(), generator=g) / math.sqrt(C)
    qk = torch.full((M, 2 * C), float("nan"), device=_dev(), dtype=BF16)
    vt = torch.full((M // hw, C, hw), float("nan"), device=_dev(), dtype=torch.float16)
    if fold:
        x, _, _, rec = _producer_with_row_stats(ops, M, C, 192, 5 * M + C)
        gamma = 1 + 0.3 * torch.randn(C, device=_dev(), generator=g)
        beta = 0.3 * torch.randn(C, device=_dev(), generator=g)
        wf, u, b = _ln_fold_pack(w, gamma, beta)
        d = ops.gemm_desc(a0=x, w=wf, out=qk, N_=3 * C, M=M, bias=b, ln=(rec, u, 1e-5), block_n=bn,
                          epilogue=nat.PP_EPI_ROWS_THEN_TRANSPOSED, out_t=vt, trans_from_col=2 * C, t_rows=hw, t_ld=hw,
                          t_fp16=True)
        ref = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w.t()
    else:
        x = torch.randn(M, C, device=_dev(), generator=g).to(BF16)
        d = ops.gemm_desc(a0=x, w=w.to(BF16), out=qk, N_=3 * C, M=M, block_n=bn, epilogue=nat.PP_EPI_ROWS_THEN_TRANSPOSED,
                          out_t=vt, trans_from_col=2 * C, t_rows=hw, t_ld=hw, t_fp16=True)
        ref = x.float() @ w.to(BF16).float().t()
    ops.run(d)
    torch.cuda.synchronize()
    assert torch.isfinite(qk.float()).all() and torch.isfinite(vt.float()).all()
    assert _rel(qk, ref[:, :2 * C]) < 8e-3, _rel(qk, ref[:, :2 * C])
    vref = ref[:, 2 * C:].view(M // hw, hw, C).transpose(1, 2)
    assert _rel(vt, vref) < 8e-3, _rel(vt, vref)


@pytest.mark.parametrize("nb,h,w,cin,cout,two", [(16, 8, 8, 1280, 1280, False), (4, 16, 16, 1280, 1280, False),
                                                 (16, 8, 8, 1280, 1280, True), (4, 8, 8, 640, 1280, False)])
def test_conv3x3_split_k(ops, nb, h, w, cin, cout, two):
    """8x8-resolution convs (few tiles, long K) with split-K x2 across two CTAs per tile: the donor's fp32 partial tile
    goes through the workspace, the owner adds it (owner + donor, fixed order) — same result run after run, flags back at
    zero, residual / time-embedding / statistics epilogue unchanged"""
    from powerpaint_b200 import _native as nat

    g = torch.Generator(device="cuda").manual_seed(nb * 100 + cin + two)
    c1 = cin if two else 0
    x = torch.randn(nb, cin + c1, h, w, device=_dev(), generator=g).to(BF16)
    wt = (torch.randn(cout, cin + c1, 3, 3, device=_dev(), generator=g) / math.sqrt(9 * (cin + c1))).to(BF16)
    bias = torch.randn(cout, device=_dev(), generator=g)
    temb = torch.randn(nb, cout, device=_dev(), generator=g)
    res = torch.randn(nb, h, w, cout, device=_dev(), generator=g).to(BF16)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    x0 = x_nhwc[..., :cin].contiguous()
    x1 = x_nhwc[..., cin:].contiguous() if two else None
    wp = ops.pack_conv3x3_weight(wt.float(), cin if two else None)
    outs = []
    for split in (True, False):
        out = torch.full((nb, h, w, cout), float("nan"), device=_dev(), dtype=BF16)
        d = ops.gemm_desc(a0=x0, a1=x1, c1=c1, w=wp, out=out, N_=cout, a_mode=nat.PP_A_CONV3X3, c0=cin, nb=nb, h=h, w_=w,
                          bias=bias, rowvec=temb, res1=res)
        if split:
            nbytes, tiles = ops.gemm_splitk_query(d)
            assert nbytes > 0 and tiles > 0, "this shape is expected to split"
            ws = torch.full((nbytes // 4,), float("nan"), device=_dev(), dtype=torch.float32)
            flags = torch.zeros(tiles, device=_dev(), dtype=torch.int32)
            ops.attach_splitk(d, ws, flags)
        ops.run(d)
        torch.cuda.synchronize()
        first = out.clone()
        ops.run(d)  # again: flags must have been reset, result bit-identical
        torch.cuda.synchronize()
        assert torch.equal(out, first)
        if split:
            assert (flags == 0).all()
        outs.append(out)
    ref = F.conv2d(x.float(), wt.float(), bias, padding=1) + temb[:, :, None, None] + res.permute(0, 3, 1, 2).float()
    for out in outs:
        got = out.permute(0, 3, 1, 2).float()
        assert torch.isfinite(got).all()
        assert _rel(got, ref) < 6e-3, _rel(got, ref)
    assert _rel(outs[0], outs[1]) < 4e-3
