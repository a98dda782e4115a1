"""Every GEMM / conv and attention kernel variant, element by element, against an fp64 evaluation of the contract
include/powerpaint_b200.h states.

Each GPU case names the variant it means to run and asserts, through the host-only queries pp_gemm_variant /
pp_attention_variant, that the launch reaches it. Outputs live inside larger allocations: NaN where the kernel must
write, a finite sentinel around them (pitch columns, rows before and after, transposed-store pads) that must come
back bit-unchanged. Every output element must be finite and within a per-element bound derived from the operation's
own rounding (`gemm_bound`, `attn_bound`); the worst err / bound of each case is printed.

The CPU tests check the checker itself (it rejects a set of small, local corruptions and accepts the exact result
rounded to bf16), that the variant tables below equal the kernels the sources dispatch to, and that the queries
answer without a device.
"""
import ctypes as C
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F16 = torch.bfloat16, torch.float16
U16 = 2.0 ** -8     # relative rounding of a bf16 store (fp16 is finer)
U32 = 2.0 ** -24    # relative rounding of an fp32 store
C_ACC = 2.0 ** -16  # fp32 tensor-core accumulation, relative to the magnitude sum |A| |W|
U_TANH = 2.0 ** -11  # tanh.approx.f32 (PTX ISA): silu / quick-GELU / the GEGLU gate
GELU_REFIT = 3.1e-5  # absolute error of the tanh-form refit of erf-GELU with an exact tanh (DESIGN.md §3)
SMS = 132
SENTINEL = -7.75    # exact in bf16 / fp16 / fp32


@pytest.fixture(autouse=True)
def _fp32_exact():
    """fp32 matmuls in the references stay fp32 (no TF32) inside this file"""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


# =========================================================================== variant tables
GEMM_VARIANTS = sorted([(bn, m, 1) for bn in (64, 128, 160, 256) for m in (0, 1, 3, 4, 5)]
                       + [(128, 2, 1), (256, 2, 1)] + [(bn, 0, 2) for bn in (128, 160, 256)])
ATTN_DVS = (32, 48, 64, 80, 96, 128, 160, 192)
ATTN_VARIANTS = sorted((dv, f16) for dv in ATTN_DVS for f16 in (0, 1))
ATT_STAGES = {dv: (3 if dv <= 64 else 2 if dv <= 128 else 1) for dv in ATTN_DVS}


def _src(name):
    with open(os.path.join(ROOT, "powerpaint_b200", "csrc", name)) as f:
        return f.read()


def dispatched_gemm_variants():
    src = _src("gemm_conv.cu")
    plain = {(int(a), int(b), 1) for a, b in re.findall(r"case \d+ \* 8 \+ \d+: return FN<(\d+), (\d+)>", src)}
    for bn, m, _ in plain:  # the case label and the template arguments agree
        assert re.search(rf"case {bn} \* 8 \+ {m}: return FN<{bn}, {m}>", src)
    split = {(int(b), 0, 2) for b in re.findall(r"case \d+: return launch_splitk<(\d+)>", src)}
    return plain | split


def dispatched_attention_variants():
    src = _src("attention.cu")
    got = {}
    for idx, dv, f16 in re.findall(r"case (\d+): return FN<(\d+), (true|false)>", src):
        got[int(idx)] = (int(dv), int(f16 == "true"))
    assert sorted(got) == list(range(len(got)))
    return set(got.values())


# =========================================================================== fp64 references
def _gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _mat(t, rows, cols, ld):
    """[rows, cols] view of a flat / 2-D tensor with row pitch ld"""
    return t.reshape(-1)[: (rows - 1) * ld + cols].as_strided((rows, cols), (ld, 1))


def gemm_out_geometry(d):
    """(M, ho, wo) of a descriptor"""
    if d.a_mode == 0:
        return d.M, 0, 0
    if d.a_mode == 1:
        return d.nb * d.h * d.w, d.h, d.w
    ho, wo = ((d.h + 1) // 2, (d.w + 1) // 2) if d.a_mode == 2 else (d.h // 2, d.w // 2)
    return d.nb * ho * wo, ho, wo


def gemm_extents(d):
    """{pointer field: (rows, elements per row, row pitch in elements, dtype)} of every operand and output a descriptor
    reads or writes, as include/powerpaint_b200.h defines them (GEMM N columns before the GEGLU pairing)"""
    from powerpaint_b200 import _native as nat

    M, _, _ = gemm_out_geometry(d)
    N = d.N
    e = {}
    if d.a_mode:
        e["a0"] = (d.nb * d.h * d.w, d.c0, d.c0, BF16)
        if d.a1:
            e["a1"] = (d.nb * d.h * d.w, d.c1, d.c1, BF16)
    else:
        e["a0"] = (M, d.c0, d.lda0, BF16)
        if d.a1:
            e["a1"] = (M, d.c1, d.lda1, BF16)
    packed = d.a_mode != 0 or bool(d.a1)
    kw = (9 if d.a_mode else 1) * ((d.c0 + 63) // 64 * 64 + ((d.c1 + 63) // 64 * 64 if d.a1 else 0)) if packed \
        else d.c0
    e["b"] = (N, kw, kw if packed else d.ldb, BF16)
    e["bias"] = (1, N, N, torch.float32)
    if d.rowvec:
        e["rowvec"] = (d.nb if d.a_mode else (M + d.rows_per_group - 1) // d.rows_per_group, N, d.rowvec_ld or N,
                       torch.float32)
    e["res1"], e["res2"] = (M, N, d.ldr1, BF16), (M, N, d.ldr2, BF16)
    e["ln_stats"], e["ln_u"] = (M, 2, 2, torch.float32), (1, N, N, torch.float32)
    if d.epilogue == nat.PP_EPI_GEGLU:
        e["out"] = (M, N // 2, d.ldc, BF16)
    elif d.epilogue == nat.PP_EPI_TRANSPOSED:
        e["out"] = (M // d.t_rows * N, d.t_rows, d.t_ld, F16 if d.t_fp16 else BF16)
    elif d.epilogue == nat.PP_EPI_ROWS_THEN_TRANSPOSED:
        tfc = d.trans_from_col
        e["out"] = (M, tfc, d.ldc, BF16)
        e["out_t"] = (M // d.t_rows * (N - tfc), d.t_rows, d.t_ld, F16 if d.t_fp16 else BF16)
    else:
        e["out"] = (M, N, d.ldc, torch.float32 if d.out_fp32 else BF16)
    return {k: v for k, v in e.items() if getattr(d, k)}


def _acc_chunk(d, t, r0, r1):
    """fp64 A W^T and |A| |W|^T for output rows [r0, r1) (conv chunks: whole samples)"""
    pad = lambda c: (c + 63) // 64 * 64  # noqa: E731
    N = d.N
    p0, p1 = pad(d.c0), (pad(d.c1) if d.c1 else 0)
    taps = 1 if d.a_mode == 0 else 9
    packed = taps == 9 or d.c1 > 0
    kw = taps * (p0 + p1) if packed else d.c0
    ldb = kw if packed else d.ldb
    W = _mat(t["b"], N, kw, ldb).double()
    acc = mag = 0
    if d.a_mode == 0:
        srcs = [(_mat(t["a0"], d.M, d.c0, d.lda0)[r0:r1], 0)]
        if d.c1:
            srcs.append((_mat(t["a1"], d.M, d.c1, d.lda1)[r0:r1], p0))
        for a, off in srcs:
            a = a.double()
            w = W[:, off:off + a.shape[1]]
            acc = acc + a @ w.t()
            mag = mag + a.abs() @ w.abs().t()
        return acc, mag
    _, ho, wo = gemm_out_geometry(d)
    n0, n1 = r0 // (ho * wo), r1 // (ho * wo)
    xs = [t["a0"].reshape(d.nb, d.h, d.w, d.c0)[n0:n1].double()]
    if d.c1:
        xs.append(t["a1"].reshape(d.nb, d.h, d.w, d.c1)[n0:n1].double())
    s = 1 if d.a_mode == 1 else 2
    padding = (0, 0, 0, 1, 0, 1) if d.a_mode == 3 else (0, 0, 1, 1, 1, 1)
    for si, x in enumerate(xs):
        xp = F.pad(x, padding)
        for ky in range(3):
            for kx in range(3):
                tap = ky * 3 + kx
                off = tap * (p0 + p1) + (p0 if si else 0)
                w = W[:, off:off + x.shape[-1]]
                slab = xp[:, ky:ky + s * (ho - 1) + 1:s, kx:kx + s * (wo - 1) + 1:s].reshape(-1, x.shape[-1])
                acc = acc + slab @ w.t()
                mag = mag + slab.abs() @ w.abs().t()
    return acc, mag


def _row_chunks(d, rows_per_chunk=8192):
    M, ho, wo = gemm_out_geometry(d)
    unit = ho * wo if d.a_mode else d.t_rows if d.epilogue in (2, 3) else 1  # whole samples / transposed blocks
    step = max(1, rows_per_chunk // unit) * unit
    return [(r, min(M, r + step)) for r in range(0, M, step)]


def ref_gemm(d, t, block_n):
    """Yields (r0, r1, ref, bound, pre) per chunk of output rows: the fp64 value of every output column the contract
    defines (GEGLU: N / 2 of them), its per-element error bound, and the fp64 pre-activation rows (what a LayerNorm
    statistics producer summarises). `t` maps descriptor pointer fields to tensors; `block_n` is the launch's tile
    width (it defines the GEGLU interleave)."""
    M, ho, wo = gemm_out_geometry(d)
    N = d.N
    alpha = float(d.alpha)
    if d.alpha_dev:
        step = int(t["alpha_step"].reshape(-1)[0]) if d.alpha_step else 0
        alpha *= float(t["alpha_dev"].reshape(-1)[step * d.alpha_stride])
    for r0, r1 in _row_chunks(d):
        acc, mag = _acc_chunk(d, t, r0, r1)
        dev = acc.device
        rows = torch.arange(r0, r1, device=dev)
        if d.ln_stats:
            ln = t["ln_stats"].reshape(-1, 2)[r0:r1].double()
            u = t["ln_u"].reshape(-1)[:N].double()
            acc = ln[:, :1] * acc + ln[:, 1:] * u[None]
            mag = ln[:, :1].abs() * mag + ln[:, 1:].abs() * u.abs()[None]
        v = acc
        if d.bias:
            b = t["bias"].reshape(-1)[:N].double()
            v = v + b
            mag = mag + b.abs()
        if d.rowvec:
            grp = rows // d.rows_per_group if d.a_mode == 0 else rows // (ho * wo)
            rv = _mat(t["rowvec"], int(grp.max()) + 1, N, d.rowvec_ld or N).double()[grp]
            v = v + rv
            mag = mag + rv.abs()
        if d.res1:
            r = _mat(t["res1"], M, N, d.ldr1)[r0:r1].double()
            v, mag = v + r, mag + r.abs()
        v, mag = v * alpha, mag * abs(alpha)
        if d.res2:
            r = _mat(t["res2"], M, N, d.ldr2)[r0:r1].double()
            v, mag = v + r, mag + r.abs()
        pre = v
        u_out = U32 if d.out_fp32 else U16
        if d.epilogue == 1:  # GEGLU on the tile-interleaved halves
            half = block_n // 2
            col = torch.arange(N // 2, device=dev)
            ci = (col // half) * block_n + col % half
            a, g = v[:, ci], v[:, ci + half]
            ma, mg = mag[:, ci], mag[:, ci + half]
            gl = _gelu_erf(g)
            ref = a * gl
            gate_err = g.abs() * 0.5 * U_TANH + GELU_REFIT
            bound = U16 * ref.abs() + C_ACC * (ma * gl.abs() + a.abs() * 1.13 * mg) + a.abs() * gate_err
        else:
            if d.act == 1:
                ref = v * torch.sigmoid(v)
            elif d.act == 2:
                ref = v * torch.sigmoid(1.702 * v)
            else:
                ref = v
            act_err = v.abs() * U_TANH if d.act else 0.0
            bound = u_out * ref.abs() + C_ACC * mag * (1.13 if d.act else 1.0) + act_err
        yield r0, r1, ref, bound + 1e-30, pre


def gemm_got_chunk(d, outs, r0, r1):
    """the kernel's outputs for rows [r0, r1) in the row-major column order of ref_gemm"""
    N = d.N
    if d.epilogue in (0, 1):
        ncols = N // 2 if d.epilogue == 1 else N
        return outs["out"][r0:r1, :ncols]
    tfc = d.trans_from_col if d.epilogue == 3 else 0
    nt = N - tfc
    vt = outs["out_t" if d.epilogue == 3 else "out"]  # [(M / t_rows) * nt, t_rows]
    tr = d.t_rows
    blk = vt.reshape(-1, nt, tr)[r0 // tr:r1 // tr].permute(0, 2, 1).reshape(r1 - r0, nt)
    if tfc:
        return torch.cat([outs["out"][r0:r1, :tfc], blk], 1)
    return blk


class Canvas:
    """a [rows, cols] output with row pitch ld inside a larger allocation: NaN in the output region, SENTINEL in the
    pitch columns and in `pad_rows` rows before and after"""

    def __init__(self, rows, cols, ld, dtype, device, pad_rows=3):
        self.buf = torch.full(((rows + 2 * pad_rows) * ld,), SENTINEL, dtype=dtype, device=device)
        full = self.buf.view(rows + 2 * pad_rows, ld)
        self.view = full[pad_rows:pad_rows + rows, :cols]
        self.view.fill_(float("nan"))
        self.mask = torch.zeros(rows + 2 * pad_rows, ld, dtype=torch.bool, device=device)
        self.mask[pad_rows:pad_rows + rows, :cols] = True
        self.mask = self.mask.reshape(-1)
        self.ld = ld

    def sentinels_intact(self):
        outside = self.buf[~self.mask]
        want = torch.tensor(SENTINEL, dtype=self.buf.dtype, device=self.buf.device)
        itype = {2: torch.int16, 4: torch.int32}[self.buf.element_size()]
        bad = (outside.view(itype) != want.view(itype)).sum().item()
        return bad


def assert_within(name, got, ref, bound):
    """every element finite and |got - ref| <= bound; returns the worst err / bound"""
    got = got.double()
    fin = torch.isfinite(got)
    if not fin.all():
        idx = (~fin).nonzero()[0].tolist()
        raise AssertionError(f"{name}: {(~fin).sum().item()} non-finite outputs, first at {idx}")
    ratio = (got - ref).abs() / bound
    worst = ratio.max().item() if ratio.numel() else 0.0
    if not worst <= 1.0:
        idx = (ratio == ratio.max()).nonzero()[0].tolist()
        i = tuple(idx)
        raise AssertionError(f"{name}: err / bound = {worst:.3g} at {idx} (got {got[i].item():.6g}, "
                             f"ref {ref[i].item():.6g}, bound {bound[i].item():.3g}); "
                             f"{(ratio > 1).sum().item()} elements out of bound")
    return worst


def assert_canvases(name, canvases):
    for key, cv in canvases.items():
        bad = cv.sentinels_intact()
        if bad:
            raise AssertionError(f"{name}: {bad} sentinel elements around `{key}` were overwritten")


def check_gemm(name, d, t, outs, canvases, block_n):
    worst = 0.0
    for r0, r1, ref, bound, _ in ref_gemm(d, t, block_n):
        worst = max(worst, assert_within(f"{name} rows {r0}:{r1}", gemm_got_chunk(d, outs, r0, r1), ref, bound))
    assert_canvases(name, canvases)
    return worst


def ref_attention(d, t):
    """fp64 softmax(q k^T * scale) v on the 16-bit inputs as given, and its per-element bound. `t` holds flat
    buffers q, k, vt with element offsets q_off / k_off of the descriptor's q / k pointers."""
    B, H, dh, nq, nk = d.batch, d.heads, d.d, d.nq, d.nk
    qa = t["q"].reshape(-1)[t.get("q_off", 0):]
    ka = t["k"].reshape(-1)[t.get("k_off", 0):]
    va = t["vt"].reshape(-1)
    ref = torch.empty(B * nq, H * dh, dtype=torch.float64, device=qa.device)
    bound = torch.empty_like(ref)
    u_p = 2.0 ** -11 if d.vt_fp16 else 2.0 ** -8
    qc = max(1, (1 << 27) // max(1, H * nk))  # query rows per chunk: the fp64 score block stays ~1 GB
    for b in range(B):
        k = ka[b * d.k_batch_stride:].as_strided((H, nk, dh), (dh, d.k_ld, 1)).double()
        v = va[b * H * dh * d.vt_ld:].as_strided((H, nk, dh), (dh * d.vt_ld, 1, d.vt_ld)).double()
        vmax = v.abs().amax(dim=(-1, -2), keepdim=True)
        for i0 in range(0, nq, qc):
            i1 = min(nq, i0 + qc)
            q = qa[b * d.q_batch_stride + i0 * d.q_ld:].as_strided((H, i1 - i0, dh), (dh, d.q_ld, 1)).double()
            s = (q @ k.transpose(-1, -2)) * d.scale
            p = torch.exp(s - s.amax(-1, keepdim=True))
            sp = p.sum(-1, keepdim=True)
            r = (p @ v) / sp
            s_abs = (p @ v.abs()) / sp
            l_abs = ((q.abs() @ k.abs().transpose(-1, -2)) * d.scale).amax(-1, keepdim=True)
            bd = U16 * r.abs() + (2 * u_p + C_ACC * l_abs) * s_abs + nk * U32 * vmax / sp
            # [H, rows, d] -> [rows, H * d]
            ref[b * nq + i0:b * nq + i1] = r.permute(1, 0, 2).reshape(i1 - i0, H * dh)
            bound[b * nq + i0:b * nq + i1] = bd.permute(1, 0, 2).reshape(i1 - i0, H * dh)
    return ref, bound + 1e-30


def check_attention(name, d, t, out_view, canvases):
    ref, bound = ref_attention(d, t)
    worst = assert_within(name, out_view, ref, bound)
    assert_canvases(name, canvases)
    return worst


# =========================================================================== GEMM cases
def _gemm_cases():
    """(id, variant, spec): one case per variant and shape axis (mr = at least 3 tiles per CTA, tile count not a
    multiple of the SM count; rag = M % 128 in {1, 127} and ragged N; k1 = one k-iteration; kl = a ring that wraps
    many times; conv cases run the implicit-GEMM A operand)"""
    cases = []

    def add(variant, axis, **spec):
        cases.append((f"bn{variant[0]}-m{variant[1]}-k{variant[2]}-{axis}", variant, spec))

    for bn in (64, 128, 160, 256):
        # ---- mode 0: plain bf16 epilogue
        v = (bn, 0, 1)
        add(v, "mr", M=128 * 67 - 64, N=6 * bn - 8, K=128, bias=True, rowvec=True, rpg=1000, res1=True, res2=True,
            alpha=0.5, alpha_dev=True)
        add(v, "rag", M=128 * 3 + 1, N=2 * bn + 24, K=192, c1=40, act=1, res1=True)
        add(v, "rag127", M=128 * 5 + 127, N=bn + 8, K=64 * 3, lda_pad=24, bias=True, act=2)
        add(v, "k1", M=300, N=bn + 40, K=64, bias=True)
        add(v, "kl", M=640, N=2 * bn, K=64 * 40, bias=True, ldb_pad=16)
        add(v, "conv-mr", conv=1, nb=5, h=41, w=43, cin=64, N=6 * bn - 32, bias=True, rowvec=True, chan_stats=True)
        add(v, "conv-rag", conv=1, nb=3, h=13, w=11, cin=96, c1=40, N=bn + 24, bias=True, res1=True)
        if bn in (64, 128):
            add(v, "conv-s2", conv=2, nb=3, h=27, w=13, cin=64, N=bn, bias=True)
            add(v, "conv-s2p0", conv=3, nb=2, h=33, w=18, cin=128, N=bn + 16, bias=True)
        # ---- mode 1: generic epilogue (fp32 out, N % 8 != 0, non-staged transposed store)
        v = (bn, 1, 1)
        add(v, "mr-fp32", M=128 * 67 - 64, N=6 * bn - 8, K=128, out_fp32=True, alpha=1 / math.sqrt(512))
        add(v, "rag", M=128 * 3 + 1, N=2 * bn + 13, K=192, act=1, res1=True, rowvec=True, rpg=100, bias=True)
        add(v, "rag127-ln", M=128 * 2 + 127, N=bn + 5, K=128, ln=True, bias=True)
        add(v, "k1-trans", M=300, N=bn + 40, K=64, trans=True, t_rows=100, t_fp16=True, bias=True)
        add(v, "kl", M=640, N=bn + 3, K=64 * 40, act=2, bias=True, res2=True)
        add(v, "conv-rag", conv=1, nb=2, h=9, w=7, cin=64, N=bn - 4, bias=True, act=1)
        # ---- mode 3: LayerNorm-statistics producer; mode 4: LayerNorm-folded consumer
        for m in (3, 4):
            v = (bn, m, 1)
            extra = dict(row_stats=True, res1=True) if m == 3 else dict(ln=True)
            add(v, "mr", M=128 * 67 - 64, N=6 * bn - 8, K=128, bias=True, **extra)
            add(v, "rag", M=128 * 3 + 1, N=2 * bn + 24, K=192, bias=True, **extra)
            add(v, "rag127", M=128 * 2 + 127, N=bn + 8, K=128, **extra)
            add(v, "k1", M=300, N=bn + 40, K=64, bias=True, **extra)
            add(v, "kl", M=640, N=2 * bn, K=64 * 40, bias=True, **extra)
        # ---- mode 5: transposed columns through the staging tile (V^T; q | k | v^T in one launch)
        v = (bn, 5, 1)
        add(v, "mr-qkv", M=128 * 68, N=6 * bn - 8, K=128, trans=True, t_rows=256, t_fp16=True, tfc=2 * bn, bias=True)
        add(v, "rag-ln", M=512, N=2 * bn + 24, K=192, trans=True, t_rows=128, ln=True, bias=True)
        add(v, "k1", M=384, N=bn + 40, K=64, trans=True, t_rows=384, bias=True)
        add(v, "kl-qkv", M=512, N=3 * bn, K=64 * 40, trans=True, t_rows=256, t_fp16=True, tfc=bn, ln=True)
    for bn in (128, 256):
        v = (bn, 2, 1)
        add(v, "mr", M=128 * 67 - 64, N=6 * bn, K=128, geglu=True, bias=True)
        add(v, "rag-ln", M=128 * 3 + 1, N=2 * bn, K=192, geglu=True, ln=True, bias=True)
        add(v, "rag127", M=128 * 2 + 127, N=bn, K=128, geglu=True, bias=True)
        add(v, "k1", M=300, N=2 * bn, K=64, geglu=True, bias=True)
        add(v, "kl", M=640, N=bn, K=64 * 40, geglu=True, bias=True)
    for bn in (128, 160, 256):
        v = (bn, 0, 2)
        add(v, "rag", M=128 * 3 + 1, N=2 * bn - 8, K=64 * 40, splitk=True, bias=True, res1=True)
        add(v, "rag127", M=128 * 2 + 127, N=bn + 8, K=64 * 36, splitk=True, bias=True, rowvec=True, rpg=128)
        add(v, "kl", M=256, N=bn, K=64 * 80, splitk=True, bias=True)
        add(v, "conv", conv=1, nb=16, h=8, w=8, cin=256, N=2 * bn, splitk=True, bias=True, res1=True, rowvec=True)
        add(v, "conv-rag", conv=1, nb=5, h=7, w=9, cin=256, N=bn + 16, splitk=True, bias=True)
    return cases


GEMM_CASES = _gemm_cases()


def _ld(n, mult=8, extra=8):
    return (n + mult - 1) // mult * mult + extra


def gemm_layout(spec):
    """descriptor scalars and the extents of every tensor a case needs (no allocation)"""
    from powerpaint_b200 import _native as nat

    s = dict(spec)
    conv = s.get("conv", 0)
    N = s["N"]
    f = dict(a_mode=conv, epilogue=0, N=N, alpha=s.get("alpha", 1.0), act=s.get("act", 0),
             out_fp32=int(s.get("out_fp32", False)), t_fp16=int(s.get("t_fp16", False)))
    if conv:
        nb, h, w = s["nb"], s["h"], s["w"]
        f.update(nb=nb, h=h, w=w, c0=s["cin"], c1=s.get("c1", 0))
        ho, wo = (h, w) if conv == 1 else ((h + 1) // 2, (w + 1) // 2) if conv == 2 else (h // 2, w // 2)
        M = nb * ho * wo
    else:
        M = s["M"]
        c1 = s.get("c1", 0)
        f.update(M=M, c0=s["K"] - c1, c1=c1)
        f["lda0"] = f["c0"] + s.get("lda_pad", 0)
        f["lda1"] = c1 + (8 if c1 else 0)
    pad = lambda c: (c + 63) // 64 * 64  # noqa: E731
    taps = 9 if conv else 1
    packed = taps == 9 or f["c1"] > 0
    kw = taps * (pad(f["c0"]) + (pad(f["c1"]) if f["c1"] else 0)) if packed else f["c0"]
    f["ldb"] = kw if packed else kw + s.get("ldb_pad", 0)
    f["kw"] = kw
    f["M_out"] = M
    if s.get("geglu"):
        f["epilogue"] = nat.PP_EPI_GEGLU
        f["ldc"] = _ld(N // 2)
    elif s.get("trans"):
        f["epilogue"] = nat.PP_EPI_ROWS_THEN_TRANSPOSED if s.get("tfc") else nat.PP_EPI_TRANSPOSED
        f["t_rows"] = s["t_rows"]
        f["t_ld"] = s["t_rows"] + 16
        f["trans_from_col"] = s.get("tfc", 0)
        f["ldc"] = _ld(s["tfc"]) if s.get("tfc") else 0
    else:
        f["ldc"] = _ld(N, 4 if f["out_fp32"] else 8)
    if s.get("rowvec"):
        f["rows_per_group"] = s.get("rpg", 0) if not conv else 0
        f["rowvec_ld"] = _ld(N, 4, 4)
        f["groups"] = (M + f["rows_per_group"] - 1) // f["rows_per_group"] if not conv else s["nb"]
    f["ldr1"] = _ld(N)
    f["ldr2"] = _ld(N)
    if s.get("alpha_dev"):
        f["alpha_stride"] = 8
    f["block_n"] = spec.get("_bn", 0)
    return f


def fake_desc(spec, block_n):
    """the case's descriptor with placeholder (aligned, non-dereferenced) pointers: enough for the host queries"""
    from powerpaint_b200 import _native as nat

    f = gemm_layout(spec)
    d = nat.GemmDesc()
    for k in ("a_mode", "epilogue", "c0", "c1", "nb", "h", "w", "N", "ldb", "rows_per_group", "act", "out_fp32",
              "t_rows", "t_fp16", "alpha_stride", "trans_from_col"):
        if k in f:
            setattr(d, k, f[k])
    for k in ("lda0", "lda1", "rowvec_ld", "ldr1", "ldr2", "ldc", "t_ld"):
        if k in f:
            setattr(d, k, f[k])
    d.M = f.get("M", 0)
    d.alpha = f["alpha"]
    d.block_n = block_n
    addr = [1 << 20]

    def p():
        addr[0] += 1 << 16
        return addr[0]
    d.a0, d.b, d.out = p(), p(), p()
    if f["c1"]:
        d.a1 = p()
    for key, field in (("bias", "bias"), ("rowvec", "rowvec"), ("res1", "res1"), ("res2", "res2"),
                       ("alpha_dev", "alpha_dev"), ("chan_stats", "chan_stats")):
        if spec.get(key):
            setattr(d, field, p())
    if spec.get("alpha_dev"):
        d.alpha_step = p()
    if spec.get("ln"):
        d.ln_stats, d.ln_u, d.ln_eps = p(), p(), 1e-5
    if spec.get("row_stats"):
        d.row_stats, d.row_final, d.row_ticket, d.ln_eps = p(), p(), p(), 1e-5
        d.row_stats_ld = d.M + 8
    if spec.get("tfc"):
        d.out_t = p()
    if spec.get("splitk"):
        d.splitk_ws, d.splitk_flags = p(), p()
    return d


def query_gemm(d):
    """pp_gemm_variant of a bare C descriptor"""
    from powerpaint_b200 import ops as o

    return o.gemm_variant(o.Desc("gemm", d, None))


def query_attention(d):
    """pp_attention_variant of a bare C descriptor"""
    from powerpaint_b200 import ops as o

    return o.attention_variant(o.Desc("attn", d, None))


# =========================================================================== attention cases
ROUND_UP_D = {32: 24, 48: 40, 64: 56, 80: 72, 96: 88, 128: 120, 160: 152, 192: 176}


def _attn_cases():
    cases = []
    ragged_nk = (1, 17, 127, 128, 129)
    for i, (dv, f16) in enumerate(ATTN_VARIANTS):
        dd = ROUND_UP_D[dv]
        wrap_nk = (ATT_STAGES[dv] + 2) * 128 + 37  # the K / V ring wraps at least twice
        v = (dv, f16)
        cases.append((f"dv{dv}-f{f16}-wrap", v, dict(B=2, H=2, d=dv, nq=129, nk=wrap_nk, layout="plain")))
        cases.append((f"dv{dv}-f{f16}-round", v, dict(B=1, H=3, d=dd, nq=64, nk=ragged_nk[i % 5], layout="plain")))
        cases.append((f"dv{dv}-f{f16}-self", v, dict(B=2, H=2, d=dd if i % 2 else dv, nq=255, nk=255, layout="self")))
        cases.append((f"dv{dv}-f{f16}-cross", v, dict(B=2, H=2, d=dv, nq=193, nk=77, layout="cross")))
        cases.append((f"dv{dv}-f{f16}-nk", v, dict(B=1, H=2, d=dd, nq=65, nk=ragged_nk[(i + 2) % 5], layout="plain")))
    return cases


ATTN_CASES = _attn_cases()


def attn_layout(spec, f16):
    B, H, dh, nq, nk = spec["B"], spec["H"], spec["d"], spec["nq"], spec["nk"]
    C_ = H * dh
    lay = spec["layout"]
    f = dict(batch=B, heads=H, d=dh, nq=nq, nk=nk, o_ld=C_ + 16, vt_fp16=f16, scale=1.0 / math.sqrt(dh))
    if lay == "self":
        f.update(q_ld=2 * C_, k_ld=2 * C_, q_batch_stride=nq * 2 * C_, k_batch_stride=nk * 2 * C_, k_off=C_)
    else:
        f.update(q_ld=C_ + 8, k_ld=C_ + 16, q_batch_stride=nq * (C_ + 8), k_batch_stride=nk * (C_ + 16) + 8, k_off=0)
    f["vt_ld"] = 80 if lay == "cross" else (nk + 7) // 8 * 8 + 8
    return f


def fake_attn_desc(spec, f16):
    from powerpaint_b200 import _native as nat

    f = attn_layout(spec, f16)
    d = nat.AttnDesc()
    for k in ("batch", "heads", "d", "nq", "nk", "q_ld", "k_ld", "vt_ld", "o_ld", "q_batch_stride", "k_batch_stride",
              "scale", "vt_fp16"):
        setattr(d, k, f[k])
    d.q, d.k, d.vt, d.out = 1 << 20, 1 << 21, 1 << 22, 1 << 23
    return d


# =========================================================================== CPU tests
def test_dispatch_tables_equal_the_tested_variants():
    """a kernel variant added to (or dropped from) the dispatch switches without a case here fails on the CPU"""
    assert dispatched_gemm_variants() == set(GEMM_VARIANTS)
    assert dispatched_attention_variants() == set(ATTN_VARIANTS)
    assert {v for _, v, _ in GEMM_CASES} == set(GEMM_VARIANTS)
    assert {v for _, v, _ in ATTN_CASES} == set(ATTN_VARIANTS)
    for dv in ATTN_DVS:  # both the exact head dim and one rounded up into the width
        ds = {s["d"] for _, v, s in ATTN_CASES if v[0] == dv}
        assert dv in ds and any(x < dv for x in ds)


def test_variant_queries_answer_without_a_device_and_match_every_case():
    for cid, variant, spec in GEMM_CASES:
        assert query_gemm(fake_desc(spec, variant[0])) == variant, cid
    for cid, (dv, f16), spec in ATTN_CASES:
        assert query_attention(fake_attn_desc(spec, f16)) == (dv, f16), cid
    # automatic tile width, the rule's inputs one at a time
    from powerpaint_b200 import _native as nat

    d = fake_desc(dict(M=65536, N=320, K=320), 0)
    bn, mode, ks = query_gemm(d)
    assert mode == 0 and ks == 1 and bn in (64, 128, 160, 256)
    d.out_fp32 = 1
    assert query_gemm(d)[1] == 1
    d = fake_desc(dict(M=512, N=1280, K=320, geglu=True), 160)
    with pytest.raises(RuntimeError, match="GEGLU block_n"):
        query_gemm(d)  # 80 output columns are no TMA-store box: no GEGLU kernel at 160
    a = nat.AttnDesc()
    a.d = 200
    with pytest.raises(RuntimeError):
        query_attention(a)


def _cpu_gemm(spec, variant, seed=0):
    from powerpaint_b200 import _native as nat

    g = torch.Generator().manual_seed(seed)
    f = gemm_layout(spec)
    d = fake_desc(spec, variant[0])
    t = {}
    if spec.get("conv"):
        t["a0"] = torch.randn(f["nb"], f["h"], f["w"], f["c0"], generator=g).to(BF16)
    else:
        t["a0"] = torch.randn(f["M"], f["lda0"], generator=g).to(BF16)
    t["b"] = (torch.randn(d.N, f["ldb"], generator=g) / math.sqrt(f["kw"])).to(BF16)
    if spec.get("bias"):
        t["bias"] = torch.randn(d.N, generator=g)
    return d, t


def _cpu_exact_out(d, t, bn):
    chunks = list(ref_gemm(d, t, bn))
    ref = torch.cat([c[2] for c in chunks])
    bound = torch.cat([c[3] for c in chunks])
    return ref, bound


def test_ref_gemm_conv_path_matches_torch_conv():
    """the implicit-GEMM gather of ref_gemm (K ordered tap, source, channel; pad64 per source) against F.conv2d /
    F.pad in fp64, for the three conv modes and a two-source input"""
    g = torch.Generator().manual_seed(1)
    for a_mode, nb, h, w, c0, c1 in ((1, 2, 7, 5, 24, 16), (2, 2, 7, 9, 72, 0), (3, 1, 9, 6, 16, 0), (1, 1, 3, 3, 8, 0)):
        N = 24
        x0 = torch.randn(nb, h, w, c0, generator=g).to(BF16)
        x1 = torch.randn(nb, h, w, c1, generator=g).to(BF16) if c1 else None
        wt = torch.randn(N, c0 + c1, 3, 3, generator=g).to(BF16).double()
        p0, p1 = (c0 + 63) // 64 * 64, ((c1 + 63) // 64 * 64 if c1 else 0)
        packed = torch.randn(N, 9, p0 + p1, generator=g) * 100  # pads hold garbage the kernel multiplies by zero
        wr = wt.permute(0, 2, 3, 1).reshape(N, 9, c0 + c1)
        packed[:, :, :c0] = wr[:, :, :c0].float()
        if c1:
            packed[:, :, p0:p0 + c1] = wr[:, :, c0:].float()
        from powerpaint_b200 import _native as nat

        d = nat.GemmDesc()
        d.a_mode, d.nb, d.h, d.w, d.c0, d.c1, d.N, d.alpha = a_mode, nb, h, w, c0, c1, N, 1.0
        t = {"a0": x0, "b": packed.reshape(N, -1).to(BF16)}
        if c1:
            t["a1"] = x1
        ref, _ = _cpu_exact_out(d, t, 64)
        x = (torch.cat([x0, x1], -1) if c1 else x0).permute(0, 3, 1, 2).double()
        if a_mode == 1:
            want = F.conv2d(x, wt, padding=1)
        elif a_mode == 2:
            want = F.conv2d(x, wt, stride=2, padding=1)
        else:
            want = F.conv2d(F.pad(x, (0, 1, 0, 1)), wt, stride=2)
        want = want.permute(0, 2, 3, 1).reshape(-1, N)
        assert ref.shape == want.shape and torch.allclose(ref, want, rtol=1e-12, atol=1e-10), a_mode


def test_checker_accepts_the_rounded_result_and_rejects_local_corruptions():
    """the per-element bound passes the exact result rounded to bf16 and fails on each of: one element off by 4 bf16
    ulps, one 16-wide k-slice dropped from one element's sum, one row shifted by one, one tile left NaN, one sentinel
    overwritten; and for attention a row missing its last key block"""
    spec = dict(M=300, N=136, K=192, bias=True)
    d, t = _cpu_gemm(spec, (64, 0, 1), seed=3)
    ref, bound = _cpu_exact_out(d, t, 64)
    good = ref.to(BF16)
    assert assert_within("exact", good, ref, bound) <= 1.0

    def rejects(x, what):
        with pytest.raises(AssertionError):
            assert_within(what, x, ref, bound)
    x = good.clone()
    r, c = [int(i) for i in (ref.abs() == ref.abs().max()).nonzero()[0]]
    x[r, c] = (x[r, c].float() * (1 + 4 * 2.0 ** -7)).to(BF16)  # 4 ulps (the significand holds 7 bits)
    rejects(x, "4 ulps")
    a = _mat(t["a0"], d.M, d.c0, d.lda0).double()
    w = _mat(t["b"], d.N, d.c0, d.ldb).double()
    # the element with the largest 16-wide k-slice contribution loses that slice
    contrib = torch.stack([a[:, k:k + 16] @ w[:, k:k + 16].t() for k in range(0, d.c0, 16)])
    ks, r, c = [int(i) for i in (contrib.abs() == contrib.abs().max()).nonzero()[0]]
    x = good.clone()
    x[r, c] = (ref[r, c] - contrib[ks, r, c]).to(BF16)
    rejects(x, "k-slice dropped")
    x = good.clone()
    x[200, :] = good[201, :]
    rejects(x, "row shifted")
    x = good.clone()
    x[128:256, 64:128] = float("nan")
    rejects(x, "tile NaN")
    # sentinels
    cv = Canvas(4, 6, 16, BF16, "cpu")
    cv.view.copy_(torch.ones(4, 6))
    assert cv.sentinels_intact() == 0
    cv.buf[3 * 16 + 6] = 0.0  # first pitch column of the first output row
    assert cv.sentinels_intact() == 1
    with pytest.raises(AssertionError):
        assert_canvases("sentinel", {"out": cv})
    # attention: a row whose last key block (keys 128..) never entered the softmax
    from powerpaint_b200 import _native as nat

    B, H, dh, nq, nk = 1, 2, 32, 8, 200
    q = torch.randn(B * nq, H * dh, generator=torch.Generator().manual_seed(5)).to(BF16)
    k = torch.randn(B * nk, H * dh, generator=torch.Generator().manual_seed(6)).to(BF16)
    vt = torch.randn(B * H * dh, nk, generator=torch.Generator().manual_seed(7)).to(F16)
    ad = nat.AttnDesc()
    ad.batch, ad.heads, ad.d, ad.nq, ad.nk = B, H, dh, nq, nk
    ad.q_ld = ad.k_ld = H * dh
    ad.q_batch_stride, ad.k_batch_stride = nq * H * dh, nk * H * dh
    ad.vt_ld, ad.scale, ad.vt_fp16 = nk, 1 / math.sqrt(dh), 1
    aref, abound = ref_attention(ad, {"q": q, "k": k, "vt": vt})
    assert assert_within("attn exact", aref.to(BF16), aref, abound) <= 1.0
    ad2 = nat.AttnDesc.from_buffer_copy(ad)
    ad2.nk = 128
    ad2.k_batch_stride = nk * H * dh
    short, _ = ref_attention(ad2, {"q": q, "k": k, "vt": vt})
    x = aref.to(BF16).clone()
    x[3] = short[3].to(BF16)
    with pytest.raises(AssertionError):
        assert_within("attn missing block", x, aref, abound)


# =========================================================================== GPU: GEMM matrix
def _dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops():
    from powerpaint_b200 import _native, ops as o

    assert _native.lib().pp_device_supported() == 1, "tests need an sm_90 (H100) device"
    return o


def _nan_padded(rows, cols, ld, dtype, gen, scale=1.0):
    """an input [rows, ld] whose pitch columns are NaN (the kernel must never read them)"""
    x = torch.full((rows, ld), float("nan"), device=_dev(), dtype=dtype)
    x[:, :cols] = (torch.randn(rows, cols, device=_dev(), generator=gen) * scale).to(dtype)
    return x


def build_gemm(spec, variant, seed):
    """tensors, canvases and the filled descriptor of a case"""
    from powerpaint_b200 import _native as nat
    from powerpaint_b200 import ops as o

    bn = variant[0]
    f = gemm_layout(spec)
    d = fake_desc(spec, bn)
    g = torch.Generator(device="cuda").manual_seed(seed)
    M, N = f["M_out"], d.N
    t = {}
    if d.a_mode:
        t["a0"] = torch.randn(d.nb, d.h, d.w, d.c0, device=_dev(), generator=g).to(BF16)
        if d.c1:
            t["a1"] = torch.randn(d.nb, d.h, d.w, d.c1, device=_dev(), generator=g).to(BF16)
    else:
        t["a0"] = _nan_padded(M, d.c0, d.lda0, BF16, g)
        if d.c1:
            t["a1"] = _nan_padded(M, d.c1, d.lda1, BF16, g)
    taps = 9 if d.a_mode else 1
    if taps == 9 or d.c1:  # packed K: the pad64 segments hold finite garbage the kernel multiplies by zero A
        t["b"] = (torch.randn(N, f["kw"], device=_dev(), generator=g) * 100).to(BF16)
        p0 = (d.c0 + 63) // 64 * 64
        p1 = (d.c1 + 63) // 64 * 64 if d.c1 else 0
        wv = t["b"].view(N, taps, p0 + p1)
        wv[:, :, :d.c0] = (torch.randn(N, taps, d.c0, device=_dev(), generator=g) / math.sqrt(taps * (d.c0 + d.c1))).to(BF16)
        if d.c1:
            wv[:, :, p0:p0 + d.c1] = (torch.randn(N, taps, d.c1, device=_dev(), generator=g)
                                      / math.sqrt(taps * (d.c0 + d.c1))).to(BF16)
    else:
        t["b"] = _nan_padded(N, d.c0, d.ldb, BF16, g, 1 / math.sqrt(d.c0))
    if spec.get("bias"):
        t["bias"] = torch.randn(N, device=_dev(), generator=g)
    if spec.get("rowvec"):
        t["rowvec"] = _nan_padded(f["groups"], N, d.rowvec_ld, torch.float32, g)
    if spec.get("res1"):
        t["res1"] = _nan_padded(M, N, d.ldr1, BF16, g)
    if spec.get("res2"):
        t["res2"] = _nan_padded(M, N, d.ldr2, BF16, g)
    if spec.get("alpha_dev"):
        t["alpha_dev"] = torch.randn(4 * 8, device=_dev(), generator=g)
        t["alpha_step"] = torch.tensor([2], device=_dev(), dtype=torch.int32)
    if spec.get("ln"):
        # random, row-to-row different {rstd, -rstd * mean}: a stale or shifted next-tile prefetch is a per-row error
        rs = 0.5 + 1.5 * torch.rand(M, device=_dev(), generator=g)
        t["ln_stats"] = torch.stack([rs, -rs * torch.randn(M, device=_dev(), generator=g) * 2], 1).contiguous()
        t["ln_u"] = torch.randn(N, device=_dev(), generator=g) * 4
    outs, canv = {}, {}
    odt = torch.float32 if d.out_fp32 else BF16
    if d.epilogue == nat.PP_EPI_GEGLU:
        canv["out"] = Canvas(M, N // 2, d.ldc, BF16, _dev())
    elif d.epilogue in (nat.PP_EPI_TRANSPOSED, nat.PP_EPI_ROWS_THEN_TRANSPOSED):
        tfc = d.trans_from_col
        tdt = F16 if d.t_fp16 else BF16
        key = "out_t" if tfc else "out"
        canv[key] = Canvas(M // d.t_rows * (N - tfc), d.t_rows, d.t_ld, tdt, _dev())
        if tfc:
            canv["out"] = Canvas(M, tfc, d.ldc, BF16, _dev())
    else:
        canv["out"] = Canvas(M, N, d.ldc, odt, _dev())
    outs = {k: c.view for k, c in canv.items()}
    d.a0, d.a1, d.b = nat.ptr(t["a0"]), nat.ptr(t.get("a1")), nat.ptr(t["b"])
    for k in ("bias", "rowvec", "res1", "res2", "alpha_dev", "alpha_step", "ln_stats", "ln_u"):
        setattr(d, k, nat.ptr(t.get(k)))
    d.out = outs["out"].data_ptr()
    d.out_t = outs["out_t"].data_ptr() if "out_t" in outs else None
    extra = {}
    d.row_stats = d.row_final = d.row_ticket = d.splitk_ws = d.splitk_flags = d.chan_stats = None
    desc = o.Desc("gemm", d, [t, canv])
    if spec.get("row_stats"):
        nrec = o.gemm_row_stats_records(desc)
        assert nrec == 2 * ((N + bn - 1) // bn)
        extra["rec"] = torch.full((nrec, M + 5, 4), float("nan"), device=_dev())
        extra["final"] = torch.full((M, 2), float("nan"), device=_dev())
        extra["ticket"] = torch.zeros((M + 127) // 128, device=_dev(), dtype=torch.int32)
        o.attach_row_stats(desc, extra["rec"], extra["final"], extra["ticket"], 1e-5)
    if spec.get("splitk"):
        nbytes, tiles = o.gemm_splitk_query(desc)
        assert nbytes > 0
        extra["ws"] = torch.full((nbytes // 4,), float("nan"), device=_dev())
        extra["flags"] = torch.zeros(tiles, device=_dev(), dtype=torch.int32)
        o.attach_splitk(desc, extra["ws"], extra["flags"])
    if spec.get("chan_stats"):
        geo = o.gemm_stats_geometry(desc)
        assert geo.supported
        extra["geo"] = geo
        extra["part"] = torch.full((int(geo.bytes) // 4,), float("nan"), device=_dev())
        o.attach_chan_stats(desc, extra["part"])
    return desc, t, outs, canv, extra


def _m_tiles(d, bn, extra):
    if d.a_mode == 0:
        return (d.M + 127) // 128
    geo = extra.get("geo")
    return int(geo.bytes) // (geo.segs * d.N * 16) if geo is not None else None


def _check_row_stats(name, d, t, extra, bn):
    """mode 3: row_final against fp64 mean / rstd of the fp32 pre-rounding rows, the records combine to the same
    statistics, and the tickets are back at zero"""
    pre = torch.cat([c[4] for c in ref_gemm(d, t, bn)])
    mean, var = pre.mean(1), pre.var(1, unbiased=False)
    rstd = (var + 1e-5).rsqrt()
    fin = extra["final"].double()
    assert torch.isfinite(fin).all(), name
    e_rs = ((fin[:, 0] - rstd).abs() / rstd).max().item()
    e_nm = ((fin[:, 1] + rstd * mean).abs() / (1 + (rstd * mean).abs())).max().item()
    assert e_rs < 1e-4 and e_nm < 1e-4, (name, e_rs, e_nm)
    r = extra["rec"][:, :d.M].double()
    cnt = r[..., 3]
    assert torch.isfinite(r).all() and (cnt.sum(0) == d.N).all(), name
    mean_i = r[..., 2] + r[..., 0] / cnt.clamp(min=1)
    m = (mean_i * cnt).sum(0) / d.N
    m2 = (r[..., 1] - r[..., 0] ** 2 / cnt.clamp(min=1) + cnt * (mean_i - m[None]) ** 2).sum(0)
    assert ((m - mean).abs() / (var.sqrt() + mean.abs())).max().item() < 1e-5, name
    assert ((m2 / d.N - var).abs() / var).max().item() < 1e-4, name
    assert (extra["ticket"] == 0).all(), name
    return e_rs, e_nm


def _check_chan_stats(ops, name, d, outs, extra):
    """GroupNorm (32 groups, SiLU) driven by the epilogue's partial sums, against fp64 GroupNorm of the stored output"""
    M, ho, wo = gemm_out_geometry(d)
    nb, hw, c = d.nb, ho * wo, d.N
    x = outs["out"].contiguous().view(nb, hw, c)
    gen = torch.Generator(device="cuda").manual_seed(c)
    gamma = torch.randn(c, device=_dev(), generator=gen)
    beta = torch.randn(c, device=_dev(), generator=gen)
    y = torch.full((nb, hw, c), float("nan"), device=_dev(), dtype=BF16)
    stats = torch.full(((ops.gn_scratch_bytes(nb, hw, c, 32) + 3) // 4,), float("nan"), device=_dev())
    gd = ops.gn_desc(x0=x, x1=None, c0=c, c1=0, batch=nb, hw=hw, groups=32, gamma=gamma, beta=beta, eps=1e-5,
                     silu=True, stats=stats, y=y, part0=extra["part"], geom0=extra["geo"])
    ops.run(gd)
    torch.cuda.synchronize()
    first = y.clone()
    y.fill_(float("nan"))
    ops.run(gd)  # the fixed-order reduction: a second run is bit-identical
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), first.view(torch.int16)), f"{name}: group_norm differs between two runs"
    xg = x.double().view(nb, hw, 32, c // 32)
    mean = xg.mean((1, 3), keepdim=True)
    rstd = (xg.var((1, 3), unbiased=False, keepdim=True) + 1e-5).rsqrt()
    xn = ((xg - mean) * rstd).view(nb, hw, c)
    pre = xn * gamma.double() + beta.double()
    ref = pre * torch.sigmoid(pre)
    mag = (xn.abs() * gamma.double().abs() + beta.double().abs())
    bound = U16 * ref.abs() + 2.0 ** -16 * mag * 1.13 + U_TANH * pre.abs() + 1e-30
    return assert_within(f"{name} group_norm", y.view(nb * hw, c), ref.view(nb * hw, c), bound.view(nb * hw, c))


@pytest.mark.gpu
@pytest.mark.parametrize("cid,variant,spec", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_variant(ops, cid, variant, spec):
    desc, t, outs, canv, extra = build_gemm(spec, variant, seed=sum(map(ord, cid)))
    d = desc.c
    bn = variant[0]
    assert ops.gemm_variant(desc) == variant, (cid, ops.gemm_variant(desc))
    mt = _m_tiles(d, bn, extra)
    tiles = None if mt is None else mt * ((d.N + bn - 1) // bn)
    if "mr" in cid:
        assert tiles >= 3 * SMS and tiles % SMS != 0, (cid, tiles)
    ops.run(desc)
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in outs.items()}
    worst = check_gemm(cid, d, t, outs, canv, bn)
    msg = f"[gemm {cid}] variant (block_n, mode, ksplit) = {variant} tiles = {tiles} worst err/bound = {worst:.3f}"
    if spec.get("row_stats"):
        e_rs, e_nm = _check_row_stats(cid, d, t, extra, bn)
        msg += f" row_final rel err = {e_rs:.2e} / {e_nm:.2e}"
    if spec.get("chan_stats"):
        msg += f" group_norm worst err/bound = {_check_chan_stats(ops, cid, d, outs, extra):.3f}"
    assert_rerun_identical(ops, cid, desc, outs, first, canv, extra)
    print(msg)


def _bits(x):
    return x.view(torch.int16) if x.element_size() == 2 else x.view(torch.int32)


def assert_rerun_identical(ops, name, desc, outs, first, canv, extra):
    """the same inputs again give bit-identical outputs (and row_final), every split-K flag and row ticket is back at
    zero, and the sentinels are still intact"""
    final0 = extra["final"].clone() if "final" in extra else None
    for v in outs.values():
        v.fill_(float("nan"))
    if final0 is not None:
        extra["final"].fill_(float("nan"))
    ops.run(desc)
    torch.cuda.synchronize()
    for k, v in outs.items():
        assert torch.equal(_bits(v), _bits(first[k])), f"{name}: `{k}` differs between two runs on the same inputs"
    if final0 is not None:
        assert torch.equal(_bits(extra["final"]), _bits(final0)), f"{name}: row_final differs between two runs"
    if "flags" in extra:
        assert (extra["flags"] == 0).all(), name
    if "ticket" in extra:
        assert (extra["ticket"] == 0).all(), name
    assert_canvases(name, canv)


# =========================================================================== GPU: attention matrix
def build_attention(spec, f16, seed):
    from powerpaint_b200 import _native as nat
    from powerpaint_b200 import ops as o

    f = attn_layout(spec, f16)
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, H, dh, nq, nk = f["batch"], f["heads"], f["d"], f["nq"], f["nk"]
    C_ = H * dh
    t = {}
    if spec["layout"] == "self":
        qk = torch.randn(B * nq, 2 * C_, device=_dev(), generator=g).mul_(1.5).to(BF16)
        t.update(q=qk, k=qk, q_off=0, k_off=C_)
    else:
        # [batch, tokens, heads * d] at the descriptor's pitches; every element outside that view is NaN
        for name, n, ld, bs in (("q", nq, f["q_ld"], f["q_batch_stride"]), ("k", nk, f["k_ld"], f["k_batch_stride"])):
            buf = torch.full(((B - 1) * bs + n * ld,), float("nan"), device=_dev(), dtype=BF16)
            buf.as_strided((B, n, C_), (bs, ld, 1)).copy_(torch.randn(B, n, C_, device=_dev(), generator=g) * 1.5)
            t[name] = buf
        t.update(q_off=0, k_off=0)
    # V^T [batch, heads * d, vt_ld]: the key pad columns are NaN (TMA must stop at nk)
    t["vt"] = _nan_padded(B * C_, nk, f["vt_ld"], F16 if f16 else BF16, g)
    canv = {"out": Canvas(B * nq, C_, f["o_ld"], BF16, _dev())}
    d = nat.AttnDesc()
    for k in ("batch", "heads", "d", "nq", "nk", "q_ld", "k_ld", "vt_ld", "o_ld", "q_batch_stride", "k_batch_stride",
              "scale", "vt_fp16"):
        setattr(d, k, f[k])
    d.q = t["q"].data_ptr() + 2 * t["q_off"]
    d.k = t["k"].data_ptr() + 2 * t["k_off"]
    d.vt = t["vt"].data_ptr()
    d.out = canv["out"].view.data_ptr()
    return o.Desc("attn", d, [t, canv]), t, canv


@pytest.mark.gpu
@pytest.mark.parametrize("cid,variant,spec", ATTN_CASES, ids=[c[0] for c in ATTN_CASES])
def test_attention_variant(ops, cid, variant, spec):
    desc, t, canv = build_attention(spec, variant[1], seed=sum(map(ord, cid)))
    assert ops.attention_variant(desc) == variant, (cid, ops.attention_variant(desc))
    out = canv["out"].view
    ops.run(desc)
    torch.cuda.synchronize()
    first = out.clone()
    worst = check_attention(cid, desc.c, t, out, canv)
    out.fill_(float("nan"))
    ops.run(desc)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), first.view(torch.int16)), f"{cid}: two runs differ"
    assert_canvases(cid, canv)
    print(f"[attention {cid}] variant (dv, p_fp16) = {variant} stages = {ATT_STAGES[variant[0]]} "
          f"worst err/bound = {worst:.3f}")


# =========================================================================== GPU: census of the real programs
GEMM_PTRS = ("a0", "a1", "b", "bias", "rowvec", "res1", "res2", "out", "alpha_dev", "alpha_step", "chan_stats",
             "row_stats", "row_final", "row_ticket", "ln_stats", "ln_u", "out_t", "splitk_ws", "splitk_flags")
ATTN_PTRS = ("q", "k", "vt", "out")
# engine A/B switches (DESIGN.md §5): each must keep every launch it records inside the tested variants
ENGINE_SWITCHES = (("default", {}), ("SPLITK", {"SPLITK": True}), ("no LN_FOLD", {"LN_FOLD": False}),
                   ("no QKV_MERGED", {"QKV_MERGED": False}), ("no GN_FUSED", {"GN_FUSED": False}),
                   ("GEGLU_BLOCK_N=128", {"GEGLU_BLOCK_N": 128}))
# FusedDenoiser per-GPU shapes of bench.py (mode, images B, latent h, w) and the odd latent size of a 640 x 856 image
DENOISER_SHAPES = (("C2", "v1", 8, 64, 64), ("C3", "brushnet", 4, 64, 64), ("C4", "v1", 2, 128, 128),
                   ("C5", "controlnet", 2, 64, 64), ("odd 80x107", "v1", 1, 80, 107))


def _struct_copy(c):
    return type(c).from_buffer_copy(c)


def _signature(kind, c, variant):
    ptrs = GEMM_PTRS if kind == "gemm" else ATTN_PTRS
    scalars = tuple((f, getattr(c, f)) for f, _ in c._fields_ if f not in ptrs)
    nonnull = tuple(f for f in ptrs if getattr(c, f))
    extra = ()
    if kind == "attn":
        extra = (("k_minus_q", (c.k - c.q) // 2 if 0 <= c.k - c.q < 2 * (c.batch * c.q_batch_stride) else None),)
    elif c.rowvec:
        extra = (("rowvec_misalign", c.rowvec & 15),)
    return (kind, scalars, nonnull, extra, variant)


class _Census:
    def __init__(self):
        self.sigs = {}      # signature -> (kind, C struct copy, variant, first source)
        self.counts = {}    # source -> number of gemm / attention records

    def record(self, source, desc):
        from powerpaint_b200 import ops as o

        if desc.kind not in ("gemm", "attn"):
            return
        variant = o.gemm_variant(desc) if desc.kind == "gemm" else o.attention_variant(desc)
        sig = _signature(desc.kind, desc.c, variant)
        if sig not in self.sigs:
            self.sigs[sig] = (desc.kind, _struct_copy(desc.c), variant, source, dict(sig[3]))
        self.counts[source] = self.counts.get(source, 0) + 1


# the Program record methods besides `add` (which takes a descriptor): a census sees each call as a `ProgramCall`
PROGRAM_RECORD_METHODS = ("add_layer_norm", "add_upsample2x", "add_upsample_nearest", "add_softmax_rows",
                          "add_embed_gather", "add_causal_attention_small", "add_add", "add_time_embed",
                          "add_window_copy", "add_memset")


class ProgramCall:
    """one Program.add_<kind>(...) call: `kind` and the bound arguments by parameter name"""

    def __init__(self, kind, args):
        self.kind = kind
        self.args = args


def _capture_all(monkeypatch, census, tiled_vae=False):
    """record the production programs (the denoisers under every engine switch, VAE encode / decode at 512^2, the
    text encoder; `tiled_vae`: also a tiled VAE decode) and hand every recorded op to census.record(source, op): a
    Desc for Program.add, a ProgramCall for the other record methods"""
    import inspect

    from powerpaint_b200 import ops as o
    from powerpaint_b200.denoise import FusedDenoiser
    from powerpaint_b200.engine import NetConfig, Recorder
    from powerpaint_b200.models import BrushNetModel, CLIPTextModel, ControlNetModel, UNet2DConditionModel
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    source = ["?"]
    orig_add = o.Program.add

    def add(self, desc):
        census.record(source[0], desc)
        return orig_add(self, desc)
    monkeypatch.setattr(o.Program, "add", add)
    originals = {}
    for meth in PROGRAM_RECORD_METHODS:
        originals[meth] = orig = getattr(o.Program, meth)

        def hook(self, *args, _orig=orig, _kind=meth[len("add_"):], **kw):
            bound = inspect.signature(_orig).bind(self, *args, **kw).arguments
            census.record(source[0], ProgramCall(_kind, {k: v for k, v in bound.items() if k != "self"}))
            return _orig(self, *args, **kw)
        monkeypatch.setattr(o.Program, meth, hook)
    dev = _dev()
    u9 = UNet2DConditionModel.synthetic(NetConfig(in_channels=9), seed=1234).to(dev)
    u4 = UNet2DConditionModel.synthetic(NetConfig(in_channels=4), seed=1234).to(dev)
    bn = BrushNetModel.synthetic(NetConfig(in_channels=4), seed=99).to(dev)
    cn = ControlNetModel.synthetic(NetConfig(in_channels=4), seed=77).to(dev)
    for sw_name, sw in ENGINE_SWITCHES:
        with monkeypatch.context() as m:
            for attr, val in sw.items():
                m.setattr(Recorder, attr, val)
            for model in (u9, u4, bn, cn):
                model._engine = None  # repack under the switched options
            for name, mode, B, h, w in DENOISER_SHAPES:
                source[0] = f"{name} [{sw_name}]"
                if mode == "v1":
                    fd = FusedDenoiser(u9)
                elif mode == "brushnet":
                    fd = FusedDenoiser(u4, bn, "brushnet")
                else:
                    fd = FusedDenoiser(u9, cn, "controlnet")
                fd._get(B, h, w, True, 77, False, mode == "brushnet")
                del fd
                torch.cuda.empty_cache()
    for model in (u9, u4, bn, cn):
        model._engine = None
    del u9, u4, bn, cn
    torch.cuda.empty_cache()
    vae = AutoencoderKL.synthetic(seed=4321).to(dev)
    source[0] = "VAE encode 512x512"
    vae.engine().encode_plan(1, 512, 512)
    source[0] = "VAE decode 512x512"
    vae.engine().decode_plan(1, 64, 64)
    if tiled_vae:  # the SD checkpoint's tile sizes: an 80 x 80 latent decodes as 2 x 2 overlapping 64 x 64 tiles
        vae.tile_sample_min_size, vae.tile_latent_min_size = 512, 64
        source[0] = "VAE tiled decode 80x80"
        vae.engine().tiled_plan(False, 1, 80, 80, vae.tile_geometry(False, 80, 80), vae._tiling_key())
    del vae
    te = CLIPTextModel().to(dev)
    source[0] = "text encoder 2x77"
    te.engine().plan_for(2, 77, 0)
    del te
    torch.cuda.empty_cache()
    monkeypatch.setattr(o.Program, "add", orig_add)
    for meth, orig in originals.items():
        monkeypatch.setattr(o.Program, meth, orig)


def _fresh_gemm(c0, variant, seed):
    """the captured descriptor with every pointer moved to a fresh, seeded tensor of the extent the header implies
    (outputs inside sentinel canvases, input pitch columns NaN)"""
    from powerpaint_b200 import _native as nat
    from powerpaint_b200 import ops as o

    d = _struct_copy(c0)
    g = torch.Generator(device="cuda").manual_seed(seed)
    M, ho, wo = gemm_out_geometry(d)
    N = d.N
    t, canv, extra = {}, {}, {}
    if d.a_mode:
        t["a0"] = torch.randn(d.nb, d.h, d.w, d.c0, device=_dev(), generator=g).to(BF16)
        if d.a1:
            t["a1"] = torch.randn(d.nb, d.h, d.w, d.c1, device=_dev(), generator=g).to(BF16)
    else:
        t["a0"] = _nan_padded(M, d.c0, d.lda0, BF16, g)
        if d.a1:
            t["a1"] = _nan_padded(M, d.c1, d.lda1, BF16, g)
    taps = 9 if d.a_mode else 1
    ext = gemm_extents(d)
    if taps == 9 or d.a1:
        t["b"] = (torch.randn(N, ext["b"][1], device=_dev(), generator=g) / math.sqrt(taps * (d.c0 + d.c1))).to(BF16)
    else:
        t["b"] = _nan_padded(N, d.c0, d.ldb, BF16, g, 1 / math.sqrt(d.c0))
    if d.bias:
        t["bias"] = torch.randn(N, device=_dev(), generator=g)
    if d.rowvec:
        groups, _, ld, _ = ext["rowvec"]
        mis = (c0.rowvec & 15) // 4  # keep the production pointer's 16-byte misalignment (it selects the epilogue)
        buf = torch.full((groups * ld + 8,), float("nan"), device=_dev())
        t["rowvec"] = buf[mis:]
        t["rowvec"][:groups * ld].view(groups, ld)[:, :N] = torch.randn(groups, N, device=_dev(), generator=g)
    for r, ld in (("res1", d.ldr1), ("res2", d.ldr2)):
        if getattr(d, r):
            t[r] = _nan_padded(M, N, ld, BF16, g)
    if d.alpha_dev:
        t["alpha_dev"] = torch.randn(2 * max(1, d.alpha_stride) + 1, device=_dev(), generator=g)
        t["alpha_step"] = torch.tensor([1 if d.alpha_step else 0], device=_dev(), dtype=torch.int32)
    if d.ln_stats:
        rs = 0.5 + 1.5 * torch.rand(M, device=_dev(), generator=g)
        t["ln_stats"] = torch.stack([rs, -rs * torch.randn(M, device=_dev(), generator=g) * 2], 1).contiguous()
        t["ln_u"] = torch.randn(N, device=_dev(), generator=g) * 4
    if d.epilogue == nat.PP_EPI_GEGLU:
        canv["out"] = Canvas(M, N // 2, d.ldc, BF16, _dev(), pad_rows=8)
    elif d.epilogue in (nat.PP_EPI_TRANSPOSED, nat.PP_EPI_ROWS_THEN_TRANSPOSED):
        tfc = d.trans_from_col if d.epilogue == nat.PP_EPI_ROWS_THEN_TRANSPOSED else 0
        canv["out_t" if tfc else "out"] = Canvas(M // d.t_rows * (N - tfc), d.t_rows, d.t_ld, F16 if d.t_fp16 else BF16,
                                                 _dev(), pad_rows=8)
        if tfc:
            canv["out"] = Canvas(M, tfc, d.ldc, BF16, _dev(), pad_rows=8)
    else:
        canv["out"] = Canvas(M, N, d.ldc, torch.float32 if d.out_fp32 else BF16, _dev(), pad_rows=8)
    outs = {k: cv.view for k, cv in canv.items()}
    for f in GEMM_PTRS:
        setattr(d, f, None)
    for f in ("a0", "a1", "b", "bias", "rowvec", "res1", "res2", "alpha_dev", "alpha_step", "ln_stats", "ln_u"):
        if f in t:
            setattr(d, f, t[f].data_ptr())
    d.out = outs["out"].data_ptr()
    if "out_t" in outs:
        d.out_t = outs["out_t"].data_ptr()
    desc = o.Desc("gemm", d, [t, canv, extra])
    if c0.row_stats:
        nrec = o.gemm_row_stats_records(desc)
        extra["rec"] = torch.full((nrec, M + 5, 4), float("nan"), device=_dev())
        extra["final"] = torch.full((M, 2), float("nan"), device=_dev())
        extra["ticket"] = torch.zeros((M + 127) // 128, device=_dev(), dtype=torch.int32)
        o.attach_row_stats(desc, extra["rec"], extra["final"], extra["ticket"], c0.ln_eps)
    if c0.splitk_ws:
        nbytes, tiles = o.gemm_splitk_query(desc)
        extra["ws"] = torch.full((max(nbytes, 16) // 4,), float("nan"), device=_dev())
        extra["flags"] = torch.zeros(max(tiles, 1), device=_dev(), dtype=torch.int32)
        o.attach_splitk(desc, extra["ws"], extra["flags"])
    if c0.chan_stats:
        geo = o.gemm_stats_geometry(desc)
        extra["part"] = torch.full((int(geo.bytes) // 4,), float("nan"), device=_dev())
        o.attach_chan_stats(desc, extra["part"])
    return desc, t, outs, canv, extra


def _fresh_attention(c0, k_minus_q, seed):
    from powerpaint_b200 import ops as o

    d = _struct_copy(c0)
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, H, dh, nq, nk = d.batch, d.heads, d.d, d.nq, d.nk
    C_ = H * dh
    q_ext = (B - 1) * d.q_batch_stride + (nq - 1) * d.q_ld + C_
    k_ext = (B - 1) * d.k_batch_stride + (nk - 1) * d.k_ld + C_
    t = {}
    if k_minus_q is not None:  # K is a view into Q's buffer (the engine's merged q | k projection)
        buf = torch.full((max(q_ext, k_minus_q + k_ext),), float("nan"), device=_dev(), dtype=BF16)
        buf.as_strided((B, nq, C_), (d.q_batch_stride, d.q_ld, 1)).copy_(
            torch.randn(B, nq, C_, device=_dev(), generator=g) * 1.5)
        buf[k_minus_q:].as_strided((B, nk, C_), (d.k_batch_stride, d.k_ld, 1)).copy_(
            torch.randn(B, nk, C_, device=_dev(), generator=g) * 1.5)
        t.update(q=buf, k=buf, q_off=0, k_off=k_minus_q)
    else:
        for name, n, ld, bs, ext in (("q", nq, d.q_ld, d.q_batch_stride, q_ext), ("k", nk, d.k_ld, d.k_batch_stride,
                                                                                   k_ext)):
            buf = torch.full((ext,), float("nan"), device=_dev(), dtype=BF16)
            buf.as_strided((B, n, C_), (bs, ld, 1)).copy_(torch.randn(B, n, C_, device=_dev(), generator=g) * 1.5)
            t[name] = buf
        t.update(q_off=0, k_off=0)
    t["vt"] = _nan_padded(B * C_, nk, d.vt_ld, F16 if d.vt_fp16 else BF16, g)
    canv = {"out": Canvas(B * nq, C_, d.o_ld, BF16, _dev(), pad_rows=8)}
    d.q = t["q"].data_ptr() + 2 * t["q_off"]
    d.k = t["k"].data_ptr() + 2 * t["k_off"]
    d.vt = t["vt"].data_ptr()
    d.out = canv["out"].view.data_ptr()
    return o.Desc("attn", d, [t, canv]), t, canv


@pytest.mark.gpu
def test_descriptor_census_of_the_real_programs(ops, monkeypatch):
    """every distinct GEMM / attention descriptor the production programs record (the bench.py denoiser shapes C2-C5,
    the odd 80 x 107 latent, VAE encode / decode at 512^2, the text encoder; the denoisers also under each engine A/B
    switch), run on fresh seeded inputs against the fp64 bound, twice, bit-identical; and every variant they use is a
    case of the variant matrix above"""
    census = _Census()
    _capture_all(monkeypatch, census)
    per_variant = {}
    for kind, _, variant, _, _ in census.sigs.values():
        per_variant[(kind, variant)] = per_variant.get((kind, variant), 0) + 1
    print("\n[census] records per program:")
    for src, n in census.counts.items():
        print(f"[census]   {src}: {n} GEMM / attention launches")
    print(f"[census] {len(census.sigs)} distinct signatures; per variant:")
    for (kind, variant), n in sorted(per_variant.items()):
        print(f"[census]   {kind} {variant}: {n}")
    used_gemm = {v for (k, v) in per_variant if k == "gemm"}
    used_attn = {v for (k, v) in per_variant if k == "attn"}
    assert used_gemm <= set(GEMM_VARIANTS) and used_attn <= set(ATTN_VARIANTS)
    assert used_gemm <= {v for _, v, _ in GEMM_CASES} and used_attn <= {v for _, v, _ in ATTN_CASES}
    worst_all = 0.0
    for i, (kind, c0, variant, source, meta) in enumerate(census.sigs.values()):
        name = f"census #{i} {kind} {variant} from {source}"
        if kind == "gemm":
            desc, t, outs, canv, extra = _fresh_gemm(c0, variant, seed=1000 + i)
            assert ops.gemm_variant(desc) == variant, name
            ops.run(desc)
            torch.cuda.synchronize()
            first = {k: v.clone() for k, v in outs.items()}
            worst = check_gemm(name, desc.c, t, outs, canv, variant[0])
            if "final" in extra:
                _check_row_stats(name, desc.c, t, extra, variant[0])
        else:
            desc, t, canv = _fresh_attention(c0, meta.get("k_minus_q"), seed=1000 + i)
            assert ops.attention_variant(desc) == variant, name
            outs = {"out": canv["out"].view}
            extra = {}
            ops.run(desc)
            torch.cuda.synchronize()
            first = {"out": outs["out"].clone()}
            worst = check_attention(name, desc.c, t, outs["out"], canv)
        assert_rerun_identical(ops, name, desc, outs, first, canv, extra)
        worst_all = max(worst_all, worst)
        c = desc.c
        shape = (f"M={gemm_out_geometry(c)[0]} N={c.N} K={c.c0}+{c.c1} a_mode={c.a_mode} epi={c.epilogue}"
                 if kind == "gemm" else f"B={c.batch} H={c.heads} d={c.d} nq={c.nq} nk={c.nk}")
        print(f"[census] #{i} {kind} {variant} {shape} ({source}) worst err/bound = {worst:.3f}")
        del desc, t, outs, canv, extra, first
    print(f"[census] worst err/bound over all signatures = {worst_all:.3f}")
