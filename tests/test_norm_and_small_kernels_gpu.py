"""GroupNorm, LayerNorm and every other non-GEMM kernel a step launches, element by element against an fp64
reference of the contract include/powerpaint_b200.h states, at the descriptors the production programs record.

A census records the same programs as the GEMM / attention census of test_kernel_variants_gpu.py (plus a tiled VAE
decode) and keys every record of every op kind by its scalar arguments and which pointers are non-null. Each distinct
signature of a kind checked here runs again on fresh seeded inputs; every other kind must be named in
COVERED_ELSEWHERE, so a new op kind fails until someone covers it.

GroupNorm runs both statistics paths: the standalone two-pass kernel (NaN-filled scratch cleared by the call, then the
same scratch again with stats_prezeroed = 1: bit-identical, tickets back at zero) and the finalize kernel over per-tile
records, fed (a) by the captured producer GEMM(s) and (b) by records built in fp64 on the host with a different
shift per tile. The (mean, rstd) the kernels store are checked against fp64 statistics of the stored bf16 input to a
bound derived from the fp32 accumulation, and y against a per-element bound built from those stored statistics.

Kernels with an exact contract (upsample, add, embedding gather, layout conversions, image pre / post-processing) are
compared bit for bit; the timestep embedding, LayerNorm, the row softmax and the small causal attention to
per-element bounds. Outputs live in sentinel canvases (test_kernel_variants_gpu.Canvas). The CPU tests check the
checkers themselves and that every template instantiation the sources dispatch to is a case here.
"""
import math
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_kernel_variants_gpu import (
    BF16, DENOISER_SHAPES, ENGINE_SWITCHES, SENTINEL, U16, U32, U_TANH, Canvas, ProgramCall, _capture_all,
    _fresh_gemm, _src, _struct_copy, assert_canvases, assert_within, fake_desc, gemm_out_geometry)

EXP_APPROX = 2.0 ** -21  # relative error of __expf's ex2.approx, beyond the rounding of its argument
SMS = 132

# op kinds the census may record that are checked by other files (or are no kernel at all)
COVERED_ELSEWHERE = {
    "gemm": "test_kernel_variants_gpu.py (variant matrix and GEMM census)",
    "attn": "test_kernel_variants_gpu.py (variant matrix and attention census)",
    "pool_broadcast": "test_side_net_modes_gpu.py",
    "window_copy": "test_vae_tiling_gpu.py",
    "tile_blend": "test_vae_tiling_gpu.py",
    "memset": "not a kernel (cudaMemsetAsync of the GroupNorm scratch arenas)",
}
CHECKED_HERE = ("gn", "layer_norm", "upsample2x", "upsample_nearest", "softmax_rows", "embed_gather",
                "causal_attention_small", "add", "time_embed")


def _dev():
    return torch.device("cuda:0")


def _lib():
    from powerpaint_b200 import _native

    return _native.lib()


def _check(status, what):
    from powerpaint_b200 import _native

    _native.check(status, what)


def _stream():
    from powerpaint_b200 import _native

    return _native.current_stream()


def _padded(shape, dtype, fill=float("nan"), pad=64):
    """a contiguous tensor of `shape` inside a larger `fill`-filled allocation (a read past either end reads fill)"""
    n = math.prod(shape)
    buf = torch.full((n + 2 * pad,), fill, dtype=dtype, device=_dev())
    return buf[pad:pad + n].view(shape)


def _bits(x):
    return x.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[x.element_size()])


def assert_bits_equal(name, got, ref):
    got, ref = got.contiguous(), ref.contiguous().to(got.dtype)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    diff = _bits(got) != _bits(ref)
    if diff.any():
        i = diff.nonzero()[0].tolist()
        raise AssertionError(f"{name}: {diff.sum().item()} elements differ from the reference bit pattern, first at "
                             f"{i} (got {got[tuple(i)].item()}, want {ref[tuple(i)].item()})")


# =========================================================================== dispatch tables
def dispatched_instances(src_name, kernel, guard):
    """[(threshold, instantiation)] of an if / else-if chain `if (<guard> <= T) ... kernel<I>` (threshold None for
    the final else)"""
    src = _src(src_name)
    out = [(int(t), int(i)) for t, i in re.findall(rf"{guard} <= (\d+)\) PP_CUDA_CHECK\(launch\({kernel}<(\d+)>", src)]
    last = re.findall(rf"else PP_CUDA_CHECK\(launch\({kernel}<(\d+)>", src)
    return out + [(None, int(i)) for i in last]


def pick_instance(table, v):
    for t, i in table:
        if t is None or v <= t:
            return i
    raise AssertionError((table, v))


def layer_norm_instance(c):
    return pick_instance(dispatched_instances("norm.cu", "layer_norm_kernel", "CV"), c // 8)


def softmax_instance(cols):
    return pick_instance(dispatched_instances("image_ops.cu", "softmax_rows_kernel", "per"), (cols + 255) // 256)


def dispatched_causal_ds():
    src = _src("clip_ops.cu")
    return {int(d) for d in re.findall(r"causal_attention_small_kernel<(\d+)>", src)}


LN_CASES = [  # id, rows, c, input mean
    ("r1-c32", 1, 32, 0.0), ("c32-many", 3000, 32, 0.0), ("c320-2passes", 2 * SMS * 8 * 8 + 5, 320, 0.0),
    ("c520", 77, 520, 0.0), ("c768-mean", 154, 768, 40.0), ("c1000", 130, 1000, 0.0), ("r1-c1280", 1, 1280, 0.0),
    ("c1280-2passes-mean", SMS * 8 * 8 + 9, 1280, 25.0), ("c2048", 300, 2048, 0.0), ("c2048-mean", 2, 2048, 100.0)]
SOFTMAX_COLS = (1, 77, 1024, 1025, 4096, 4097, 16384)
CAUSAL_SEQS = (1, 77, 128)


# =========================================================================== GroupNorm: layout mirrors
def gn_geometry(batch, hw, C, groups):
    """the launch geometry and scratch layout of the standalone statistics path (norm.cu gn_geometry; the layout is the
    one include/powerpaint_b200.h documents for pp_gn_desc.stats)"""
    CV = C // 8
    lanes = max(1, 256 // CV)
    chunks = (SMS * 8 + batch - 1) // batch
    ppb = max((hw + chunks - 1) // chunks, lanes * 8)
    chunks = (hw + ppb - 1) // ppb
    stats_bytes = 4 * 2 * groups * batch
    ticket_offset = (stats_bytes + 15) & ~15
    partial_offset = ticket_offset + ((4 * batch + 15) & ~15)
    return dict(lanes=lanes, ppb=ppb, chunks=chunks, ticket_offset=ticket_offset,
                scratch_bytes=partial_offset + 4 * 2 * groups * chunks * batch)


def standalone_chain(batch, hw, C, groups):
    """longest run of sequential fp32 additions one term of a standalone (sample, group) sum goes through: the
    thread's pixels of its chunk, then the block's fold over lanes x channels of the group (+ the shifted difference)"""
    g = gn_geometry(batch, hw, C, groups)
    return (g["ppb"] + g["lanes"] - 1) // g["lanes"] + g["lanes"] * (C // groups) + 2


def producer_chain(geom):
    """the same for a producer epilogue record: >= 8 row lanes per segment, a 16-lane butterfly, the fp32 record"""
    return (geom.seg_rows + 7) // 8 + 6


HOST_RECORD_CHAIN = 2  # host-built records: fp64 sums rounded once to fp32


def tile_boxes(geom):
    """[(tile index, y0, y1, x0, x1)] of the valid pixels of every tile of one segment (matrix mode: a 1-row strip)"""
    out = []
    for t in range(geom.tiles_per_group):
        ty, tx = divmod(t, geom.tiles_x)
        y0, x0 = ty * geom.bh, tx * geom.bw
        out.append((t, y0, min(geom.ho, y0 + geom.bh), x0, min(geom.wo, x0 + geom.bw)))
    return out


def build_records(x, geom, batch, shift_offset=None):
    """the producer-record layout of the header, [m_tiles][segs][N][4] = {sum(x - shift), sum((x - shift)^2), shift, 0},
    built in fp64 from x [batch, hw, N] and rounded to fp32. shift = the segment's first valid pixel, plus
    shift_offset(t) (a per-tile constant) when given. Records of sample slots past `batch` stay NaN (never read)."""
    N = x.shape[-1]
    segs, T = geom.segs, geom.tiles_per_group
    m_tiles = (batch + segs - 1) // segs * T
    rec = torch.full((m_tiles, segs, N, 4), float("nan"), dtype=torch.float32, device=x.device)
    xi = x.double().view(batch, geom.ho, geom.wo, N)
    n = torch.arange(batch, device=x.device)
    for t, y0, y1, x0, x1 in tile_boxes(geom):
        slab = xi[:, y0:y1, x0:x1].reshape(batch, -1, N)
        shift = slab[:, 0].clone()
        if shift_offset is not None:
            shift = shift + shift_offset(t)
        shift = shift.float().double()  # the record stores it in fp32
        dlt = slab - shift[:, None]
        r = torch.stack([dlt.sum(1), (dlt * dlt).sum(1), shift, torch.zeros_like(shift)], -1)
        rec[(n // segs) * T + t, n % segs] = r.float()
    return rec


def finalize_emulation(recs, geoms, c_split, batch, groups, count_whole_box=False):
    """gn_finalize_kernel's arithmetic in fp64 on the host: (mean, var) per (sample, group) from the records of the
    sources; count_whole_box counts every tile as its full bw x bh box (the checker self-test's corruption)"""
    C = sum(c_split)
    cpg = C // groups
    S = torch.zeros(batch, groups, dtype=torch.float64)
    SS = torch.zeros_like(S)
    cnt = torch.zeros_like(S)
    R = None
    off = 0
    cols = []
    for rec, geom, cs in zip(recs, geoms, c_split):
        for t, y0, y1, x0, x1 in tile_boxes(geom):
            cb = geom.bw * geom.bh if count_whole_box else (y1 - y0) * (x1 - x0)
            for n in range(batch):
                r = rec[(n // geom.segs) * geom.tiles_per_group + t, n % geom.segs].double().cpu()
                cols.append((n, off, cs, cb, r))
        off += cs
    ch = torch.arange(C)
    first = {}
    for n, off, cs, cb, r in cols:  # R = the shift of the group's first channel in its first tile
        for g in range(groups):
            c = g * cpg
            if off <= c < off + cs and (n, g) not in first:
                first[(n, g)] = r[c - off, 2].item()
    R = torch.tensor([[first[(n, g)] for g in range(groups)] for n in range(batch)], dtype=torch.float64)
    for n, off, cs, cb, r in cols:
        grp = (ch[off:off + cs] // cpg)
        d = r[:, 2] - R[n, grp]
        S[n].index_add_(0, grp, r[:, 0] + cb * d)
        SS[n].index_add_(0, grp, r[:, 1] + d * (2 * r[:, 0] + cb * d))
        cnt[n].index_add_(0, grp, torch.full((cs,), float(cb), dtype=torch.float64))
    md = S / cnt
    return R + md, (SS - S * md).clamp(min=0) / cnt


def gn_truth(x, groups):
    """fp64 statistics of the stored input x [batch, hw, C] per (sample, group), and the magnitudes the bounds need:
    sum |x - mean| and max |x - mean| (every shift the kernels use is an element of the group)"""
    nb, hw, C = x.shape
    xg = x.double().view(nb, hw, groups, C // groups)
    mean = xg.mean((1, 3))
    var = xg.var((1, 3), unbiased=False)
    dev = (xg - mean[:, None, :, None]).abs()
    return mean, var, dev.sum((1, 3)), dev.amax((1, 3)), hw * (C // groups)


def gn_stats_bounds(truth, chain, eps, shift_extra=0.0):
    """bounds of the stored fp32 mean (absolute) and rstd (absolute) when every term of the shifted sums went through
    at most `chain` fp32 roundings; shifts lie within max|x - mean| + shift_extra of the mean"""
    mean, var, s1, mx, cnt = truth
    dsh = mx + shift_extra
    mag1 = s1 + cnt * dsh                 # >= sum |x - shift|
    mag2 = cnt * (var + dsh * dsh)        # >= sum (x - shift)^2
    d_md = chain * U32 * mag1 / cnt
    d_var = (chain + 1) * U32 * mag2 / cnt + 2 * dsh * d_md + d_md * d_md
    rstd = (var + eps).rsqrt()
    b_mean = d_md + 2 * U32 * mean.abs() + 1e-30
    b_rstd = rstd * (0.5 * d_var / (var + eps) * 1.01 + 3 * U32) + 1e-30
    return rstd, b_mean, b_rstd


def check_gn_stats(name, st, truth, chain, eps, shift_extra=0.0):
    """st: the kernel's [batch, groups, 2] (mean, rstd); returns the worst err / bound of each"""
    rstd, b_mean, b_rstd = gn_stats_bounds(truth, chain, eps, shift_extra)
    w_mean = assert_within(f"{name} stored mean", st[..., 0], truth[0], b_mean)
    w_rstd = assert_within(f"{name} stored rstd", st[..., 1], rstd, b_rstd)
    return w_mean, w_rstd


def gn_y_ref(x, st, gamma, beta, silu):
    """fp64 y = act(x a + b), a = rstd gamma, b = beta - mean a from the STORED statistics, and its per-element bound
    (fp32 a and b, the FMA, tanh.approx of SiLU, the bf16 store)"""
    nb, hw, C = x.shape
    groups = st.shape[1]
    grp = torch.arange(C, device=x.device) // (C // groups)
    m = st[..., 0].double()[:, grp][:, None]
    r = st[..., 1].double()[:, grp][:, None]
    g, b_ = gamma.double()[None, None], beta.double()[None, None]
    a = r * g
    b = b_ - m * a
    xd = x.double()
    pre = xd * a + b
    d_a = U32 * a.abs()
    d_b = 2 * U32 * (b_.abs() + (m * a).abs()) + m.abs() * d_a
    d_pre = xd.abs() * d_a + d_b + U32 * pre.abs()
    if silu:
        ref = pre * torch.sigmoid(pre)
        bound = U16 * ref.abs() + 1.13 * d_pre + U_TANH * pre.abs()
    else:
        ref = pre
        bound = U16 * ref.abs() + d_pre
    return ref, bound + 1e-30


def stats_geom_of_conv(nb, ho, wo, N):
    """the statistics geometry a 3x3 conv producing [nb, ho, wo, N] emits (host-only query)"""
    from powerpaint_b200 import ops as o

    d = fake_desc(dict(conv=1, nb=nb, h=ho, w=wo, cin=64, N=N, bias=True, chan_stats=True), 0)
    geo = o.gemm_stats_geometry(o.Desc("gemm", d, None))
    assert geo.supported, (nb, ho, wo, N)
    return geo


def _geom_tuple(g):
    return tuple(getattr(g, f) for f, _ in g._fields_)


# =========================================================================== small-op references and bounds
def ref_layer_norm(x, gamma, beta, eps):
    """fp64 LayerNorm of the bf16 rows x [rows, c] and the per-element bound of the kernel's fp32 two-pass arithmetic
    (a warp per row: 8 * MAX_VEC sequential additions per lane, a 5-step butterfly; rsqrtf; 4 rounded operations)"""
    rows, c = x.shape
    chain = 8 * layer_norm_instance(c) + 6
    xd = x.double()
    mean = xd.mean(1, keepdim=True)
    t = xd - mean
    var = (t * t).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    g, b = gamma.double()[None], beta.double()[None]
    ref = t * rstd * g + b
    d_mean = chain * U32 * xd.abs().sum(1, keepdim=True) / c + 2 * U32 * mean.abs()
    d_t = d_mean + U32 * t.abs()
    d_sq = chain * U32 * (t * t).sum(1, keepdim=True) + 2 * (t.abs() * d_t).sum(1, keepdim=True)
    rel_rstd = 0.5 * d_sq / (c * (var + eps)) * 1.01 + 4 * U32
    bound = g.abs() * rstd * (d_t + t.abs() * (rel_rstd + 3 * U32)) + U32 * (ref.abs() + b.abs()) + U16 * ref.abs()
    return ref, bound + 1e-30


def ref_softmax(s, per_thread):
    """fp64 softmax of the fp32 rows s and its per-element bound: __expf (its argument's rounding and ex2.approx), the
    fp32 row sum (PER_THREAD terms per thread, two 5-step butterflies and an 8-warp fold), the division and the
    product, the bf16 store; FTZ of exp results below 2^-126"""
    sd = s.double()
    mx = sd.amax(1, keepdim=True)
    x = sd - mx
    e = torch.exp(x)
    tot = e.sum(1, keepdim=True)
    p = e / tot
    rel_e = torch.where(e > 0, EXP_APPROX + 3 * U32 * x.abs(), torch.zeros_like(x))
    rel_sum = (rel_e * e).sum(1, keepdim=True) / tot + (per_thread + 16) * U32
    bound = p * (rel_e + rel_sum + 3 * U32) + U16 * p + 2.0 ** -125
    return p, bound


def ref_causal_attention(qkv, batch, seq, heads, d, scale):
    """fp64 causal softmax(q k^T * scale) v of the bf16 qkv [batch * seq, 3 * heads * d] (q | k | v) and its bound: the
    fp32 scores (d fused multiply-adds on the pre-scaled q) and __expf perturb every weight by a relative delta, the
    online rescaling multiplies the numerator and the denominator alike, the accumulations run over <= seq terms"""
    C = heads * d
    x = qkv.double().view(batch, seq, 3, heads, d).permute(2, 0, 3, 1, 4)  # [3, batch, heads, seq, d]
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * scale
    l_abs = ((q.abs() @ k.abs().transpose(-1, -2)) * scale).amax(-1, keepdim=True)
    causal = torch.ones(seq, seq, dtype=torch.bool, device=qkv.device).tril()
    s = s.masked_fill(~causal, float("-inf"))
    p = torch.exp(s - s.amax(-1, keepdim=True))
    sp = p.sum(-1, keepdim=True)
    r = (p @ v) / sp
    s_abs = (p @ v.abs()) / sp
    delta = EXP_APPROX + (d + 8) * U32 * l_abs
    bd = U16 * r.abs() + (2 * delta + 2 * (seq + 3) * U32) * s_abs
    to_rows = lambda t: t.permute(0, 2, 1, 3).reshape(batch * seq, C)  # noqa: E731
    return to_rows(r), to_rows(bd) + 1e-30


TIME_EMBED_C = 48  # relative error of the fp32 argument t * f in units of 2^-24: the rounded exponent, expf, t * f


def ref_time_embed(t, dim):
    """fp64 [cos(t f), sin(t f)] (f = 10000^(-k / half)) of the fp32 timesteps t [batch], and the bound
    U16 |e| + |t| c 2^-24 (+ the ulp-level error of cosf / sinf)"""
    half = dim // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
    a = t.double()[:, None] * f[None]
    e = torch.cat([torch.cos(a), torch.sin(a)], -1)
    bound = U16 * e.abs() + t.double().abs()[:, None] * TIME_EMBED_C * U32 + 2.0 ** -22
    return e, bound


def ref_postprocess_u8(x):
    """the reference's `(x / 2 + 0.5).clamp(0, 1)` in fp32, then numpy `(images * 255).round().astype("uint8")`"""
    v = (x.float().cpu() / 2 + 0.5).clamp(0, 1)
    return torch.from_numpy((v.numpy() * 255).round().astype("uint8")), v


def postprocess_tie_inputs():
    """fp32 inputs whose fp32 (x / 2 + 0.5) * 255 lands exactly on k + 0.5 for even k (round-half-even and
    round-half-away differ there), found around every (k + 0.5) / 255"""
    centre = ((np.arange(255) + 0.5) / 255).astype(np.float32).view(np.int32)
    v = (centre[:, None] + np.arange(-64, 65, dtype=np.int32)[None]).reshape(-1).view(np.float32)
    x = (v * np.float32(2) - np.float32(1)).astype(np.float32)
    y = ((x / np.float32(2) + np.float32(0.5)).clip(0, 1) * np.float32(255)).astype(np.float32)
    even_tie = (y - np.floor(y) == 0.5) & (np.floor(y) % 2 == 0)
    return torch.from_numpy(x[even_tie])


# =========================================================================== CPU tests
def test_dispatch_tables_are_cases_here():
    """every template instantiation norm.cu, image_ops.cu and clip_ops.cu dispatch to is reached by a case here"""
    ln = dispatched_instances("norm.cu", "layer_norm_kernel", "CV")
    sm = dispatched_instances("image_ops.cu", "softmax_rows_kernel", "per")
    assert [i for _, i in ln] == [1, 2, 3, 5, 8] and ln[-1][0] is None, ln
    assert [i for _, i in sm] == [4, 16, 64] and sm[-1][0] is None, sm
    assert {layer_norm_instance(c) for _, _, c, _ in LN_CASES} == {i for _, i in ln}
    assert {softmax_instance(c) for c in SOFTMAX_COLS} == {i for _, i in sm}
    assert dispatched_causal_ds() == {8, 16, 32, 64}
    # the UNet and text-encoder widths (768 runs <3>), one width not a multiple of 256, both
    # ends of the row range, and more rows than one grid pass (132 * 8 blocks of 8 warps)
    widths = {c for _, _, c, _ in LN_CASES}
    assert {32, 320, 768, 1280, 2048} <= widths and any(c % 256 for c in widths)
    rows = {r for _, r, _, _ in LN_CASES}
    assert 1 in rows and max(rows) > SMS * 8 * 8
    assert 16384 in SOFTMAX_COLS and 1 in SOFTMAX_COLS


def test_group_norm_scratch_layout_mirrors_the_library():
    """the Python mirror of the scratch layout (stats | tickets | partials) sizes the scratch like the library"""
    from powerpaint_b200 import ops as o

    for nb, hw, C, groups in ((2, 4096, 320, 32), (16, 64, 1280, 32), (4, 16384, 320, 32), (1, 140, 2560, 32),
                              (3, 64, 1920, 32), (1, 4, 64, 8), (2, 540, 960, 32)):
        assert gn_geometry(nb, hw, C, groups)["scratch_bytes"] == o.gn_scratch_bytes(nb, hw, C, groups)


def test_host_records_fold_to_the_fp64_statistics():
    """records built from the header's layout with a different shift per tile, folded as gn_finalize_kernel folds
    them, give the fp64 statistics: at a width-14 level with edge tiles, a concat whose groups straddle the sources,
    and two samples per tile with an odd batch"""
    g = torch.Generator().manual_seed(3)
    for nb, ho, wo, c0, c1 in ((2, 10, 14, 64, 32), (3, 8, 8, 48, 0)):
        geoms = [stats_geom_of_conv(nb, ho, wo, c) for c in (c0, c1) if c]
        xs = [(torch.randn(nb, ho * wo, c, generator=g) * 2 + 5).to(BF16) for c in (c0, c1) if c]
        recs = [build_records(x, gm, nb, lambda t: ((t % 5) - 2) * 0.75) for x, gm in zip(xs, geoms)]
        groups = 8 if c1 else 16
        mean, var = finalize_emulation(recs, geoms, [x.shape[-1] for x in xs], nb, groups)
        truth = gn_truth(torch.cat(xs, -1), groups)
        assert torch.allclose(mean, truth[0], rtol=0, atol=1e-5) and torch.allclose(var, truth[1], rtol=1e-5)
    assert stats_geom_of_conv(3, 8, 8, 48).segs == 2


def test_checkers_accept_the_rounded_result_and_reject_local_corruptions():
    """each new bound accepts the fp64 result rounded to the output type and rejects: one element off by 2 bf16 ulps;
    one group's stored mean from a finalize that counts an edge tile's whole 16 x 8 box instead of its 14 x 8 valid
    pixels; a stored rstd from the unbiased variance at the smallest production group (8 x 8 pixels x 40 channels);
    a softmax row missing its last column"""
    g = torch.Generator().manual_seed(11)

    def two_ulps(ref, bound, out_dtype=BF16):
        good = ref.to(out_dtype)
        assert assert_within("rounded", good, ref, bound) <= 1.0
        i = int(ref.abs().reshape(-1).argmax())
        bad = good.clone().reshape(-1)
        v = bad[i:i + 1]
        bad[i] = (v.view(torch.int16) + 2).view(BF16)[0]  # two ulps further from zero
        with pytest.raises(AssertionError):
            assert_within("2 ulps", bad.view(ref.shape), ref, bound)

    # GroupNorm y (SiLU and plain), from exact statistics stored in fp32
    nb, hw, C, groups = 2, 64, 1280, 32
    x = (torch.randn(nb, hw, C, generator=g) * 1.5 + 0.5).to(BF16)
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    truth = gn_truth(x, groups)
    st = torch.stack([truth[0], (truth[1] + 1e-5).rsqrt()], -1).float()
    for silu in (True, False):
        ref, bound = gn_y_ref(x, st, gamma, beta, silu)
        two_ulps(ref, bound)
    # stored statistics: exact rounded pass; the unbiased variance at 8 x 8 x 40 does not
    chain = standalone_chain(nb, hw, C, groups)
    check_gn_stats("exact", st, truth, chain, 1e-5)
    cnt = truth[4]
    assert cnt == 8 * 8 * 40
    bad = st.clone()
    bad[1, 7, 1] = float((truth[1][1, 7] * cnt / (cnt - 1) + 1e-5).rsqrt())
    with pytest.raises(AssertionError, match="stored rstd"):
        check_gn_stats("unbiased", bad, truth, chain, 1e-5)
    # the finalize's edge-tile count: width 14 with a 16 x 8 pixel box
    nb, ho, wo, C, groups = 1, 10, 14, 1280, 32
    geom = stats_geom_of_conv(nb, ho, wo, C)
    assert (geom.bw, geom.bh, geom.wo) == (16, 8, 14), _geom_tuple(geom)
    x = (torch.randn(nb, ho * wo, C, generator=g) * 1.5 + 0.5).to(BF16)
    rec = build_records(x, geom, nb, lambda t: ((t % 5) - 2) * 0.75)
    truth = gn_truth(x, groups)
    for whole_box in (False, True):
        mean, var = finalize_emulation([rec], [geom], [C], nb, groups, count_whole_box=whole_box)
        st = torch.stack([mean, (var + 1e-5).rsqrt()], -1).float()
        bad = torch.stack([truth[0], (truth[1] + 1e-5).rsqrt()], -1).float()
        bad[0, 5, 0] = st[0, 5, 0]  # only one group's mean comes from the finalize under test
        if whole_box:
            with pytest.raises(AssertionError, match="stored mean"):
                check_gn_stats("whole box", bad, truth, HOST_RECORD_CHAIN, 1e-5, 1.5)
        else:
            check_gn_stats("valid pixels", bad, truth, HOST_RECORD_CHAIN, 1e-5, 1.5)
    # LayerNorm
    for c in (320, 2048):
        xl = (torch.randn(9, c, generator=g) * 2 + 3).to(BF16)
        ref, bound = ref_layer_norm(xl, torch.randn(c, generator=g), torch.randn(c, generator=g), 1e-5)
        two_ulps(ref, bound)
    # softmax: the exact rows pass, 2 ulps fail, a row whose normaliser missed its last column fails
    s = torch.randn(6, 77, generator=g) * 3
    s[2, -1] = s[2].max() + 2.0  # the last column carries a visible share of the row
    p, bound = ref_softmax(s, 4)
    two_ulps(p, bound)
    short = torch.softmax(s[2, :-1].double(), 0)
    bad = p.to(BF16).clone()
    bad[2, :-1] = short.to(BF16)
    with pytest.raises(AssertionError):
        assert_within("softmax missing its last column", bad, p, bound)
    # causal attention
    qkv = torch.randn(2 * 77, 3 * 2 * 64, generator=g).to(BF16)
    r, bound = ref_causal_attention(qkv, 2, 77, 2, 64, 0.125)
    two_ulps(r, bound)
    # time embedding
    t = torch.tensor([999.0, 1.0, 500.5])
    e, bound = ref_time_embed(t, 320)
    two_ulps(e, bound)


def test_postprocess_references():
    """the fp32 tie inputs are exact ties to even (so a round-half-away kernel fails on them), and the bf16 sweep's
    reference is numpy's round-half-even"""
    x = postprocess_tie_inputs()
    assert x.numel() > 0
    u8, v = ref_postprocess_u8(x)
    y = v.numpy() * np.float32(255)
    assert (y - np.floor(y) == 0.5).all() and (u8.numpy() % 2 == 0).all()
    assert (u8.numpy().astype(np.int64) == np.floor(y).astype(np.int64)).all()  # half to even rounds these down


# =========================================================================== GPU fixtures
@pytest.fixture(scope="module")
def ops():
    from powerpaint_b200 import _native, ops as o

    assert _native.lib().pp_device_supported() == 1, "tests need an sm_90 (H100) device"
    return o


def _call_signature(call):
    sig = []
    for k, v in call.args.items():
        if isinstance(v, torch.Tensor) or v is None:
            sig.append((k, v is not None))
        elif isinstance(v, (int, float)):
            sig.append((k, v))
        else:  # a WindowList
            sig.append((k, (v.channels, v.count, v.max_pixels, v.src.element_size())))
    return tuple(sig)


def _struct_signature(c):
    import ctypes as C

    sig = []
    for f, typ in c._fields_:
        v = getattr(c, f)
        if typ is C.c_void_p:
            sig.append((f, bool(v)))
        elif isinstance(v, C.Structure):
            sig.append((f, _geom_tuple(v)))
        else:
            sig.append((f, v))
    return tuple(sig)


class OpCensus:
    """every op the production programs record, by kind: distinct signatures (scalar arguments and which pointers are
    non-null) with their first source; a GroupNorm over producer records keeps copies of its producer GEMMs"""

    def __init__(self):
        self.sigs = {}       # kind -> {signature: (C struct copy or argument dict, meta)}
        self.records = {}    # kind -> records
        self.producers = {}  # chan_stats pointer -> (GEMM struct copy, variant) of the latest GEMM that wrote it

    def record(self, source, op):
        from powerpaint_b200 import ops as o

        kind = op.kind
        self.records[kind] = self.records.get(kind, 0) + 1
        if isinstance(op, ProgramCall):
            sig, item = _call_signature(op), {k: v for k, v in op.args.items()
                                               if not isinstance(v, torch.Tensor) and v is not None}
            item["_nonnull"] = {k for k, v in op.args.items() if v is not None}
        else:
            if kind == "gemm" and op.c.chan_stats:
                self.producers[op.c.chan_stats] = (_struct_copy(op.c), o.gemm_variant(op))
            sig, item = _struct_signature(op.c), _struct_copy(op.c)
        per_kind = self.sigs.setdefault(kind, {})
        if sig in per_kind:
            return
        meta = {"source": source}
        if kind == "gn" and op.c.from_partials:
            meta["producers"] = [self.producers.get(op.c.part0)] + ([self.producers.get(op.c.part1)]
                                                                    if op.c.part1 else [])
        per_kind[sig] = (item, meta)


@pytest.fixture(scope="module")
def census(ops):
    c = OpCensus()
    with pytest.MonkeyPatch.context() as mp:
        _capture_all(mp, c, tiled_vae=True)
    torch.cuda.empty_cache()
    print(f"\n[op census] programs: denoisers {[s[0] for s in DENOISER_SHAPES]} under "
          f"{[s[0] for s in ENGINE_SWITCHES]}, VAE encode / decode 512x512, VAE tiled decode 80x80, text encoder")
    for kind in sorted(c.records):
        where = "checked here" if kind in CHECKED_HERE else \
            f"covered by {COVERED_ELSEWHERE.get(kind, 'test_program_replay_gpu.py')}"
        print(f"[op census]   {kind}: {c.records[kind]} records, {len(c.sigs.get(kind, {}))} signatures ({where})")
    return c


# =========================================================================== GPU: GroupNorm
def _scratch(floats):
    """a NaN-filled fp32 scratch of `floats` with a sentinel tail (the kernels must stay inside the scratch)"""
    buf = torch.full((floats + 64,), float("nan"), device=_dev())
    buf[floats:] = SENTINEL
    return buf


def _tail_intact(buf, floats):
    return bool((buf[floats:] == SENTINEL).all())


def run_group_norm(ops, name, x0, x1, groups, eps, silu, gamma, beta, parts=None):
    """one GroupNorm (standalone statistics unless `parts` = [(records, geom)] per source) into a sentinel canvas,
    twice; returns (y [batch, hw, C], stored (mean, rstd) [batch, groups, 2]). Standalone: NaN scratch cleared by the
    call, then the same scratch with stats_prezeroed = 1, tickets checked at zero after each run"""
    nb, hw, c0 = x0.shape
    c1 = x1.shape[-1] if x1 is not None else 0
    C = c0 + c1
    canv = Canvas(nb * hw, C, C, BF16, _dev(), pad_rows=8)
    y = canv.view.view(nb, hw, C)
    kw = dict(x0=x0, x1=x1, c0=c0, c1=c1, batch=nb, hw=hw, groups=groups, gamma=gamma, beta=beta, eps=eps,
              silu=silu, y=y)
    if parts is None:
        lay = gn_geometry(nb, hw, C, groups)
        floats = lay["scratch_bytes"] // 4
        scratch = _scratch(floats)
        tickets = scratch.view(torch.int32)[lay["ticket_offset"] // 4:lay["ticket_offset"] // 4 + nb]
        ops.run(ops.gn_desc(stats=scratch, stats_prezeroed=False, **kw))
    else:
        floats = nb * groups * 2
        scratch = _scratch(floats)
        tickets = None
        pk = dict(part0=parts[0][0], geom0=parts[0][1])
        if x1 is not None:
            pk.update(part1=parts[1][0], geom1=parts[1][1])
        ops.run(ops.gn_desc(stats=scratch, **kw, **pk))
    torch.cuda.synchronize()
    first, st = y.clone(), scratch[:nb * groups * 2].clone()
    assert tickets is None or (tickets == 0).all(), f"{name}: tickets not back at zero"
    y.fill_(float("nan"))
    scratch[:nb * groups * 2] = float("nan")
    if parts is None:
        ops.run(ops.gn_desc(stats=scratch, stats_prezeroed=True, **kw))
    else:
        ops.run(ops.gn_desc(stats=scratch, **kw, **pk))
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(first)), f"{name}: y differs between two runs"
    assert torch.equal(_bits(scratch[:nb * groups * 2]), _bits(st)), f"{name}: statistics differ between two runs"
    assert tickets is None or (tickets == 0).all(), f"{name}: tickets not back at zero after the prezeroed run"
    assert _tail_intact(scratch, floats), f"{name}: wrote past the end of its scratch"
    assert_canvases(name, {"y": canv})
    return first, st.view(nb, groups, 2)


def check_group_norm(ops, name, x0, x1, groups, eps, silu, gamma, beta, chain, parts=None, shift_extra=0.0):
    y, st = run_group_norm(ops, name, x0, x1, groups, eps, silu, gamma, beta, parts)
    x = torch.cat([x0, x1], -1) if x1 is not None else x0
    truth = gn_truth(x, groups)
    w_mean, w_rstd = check_gn_stats(name, st, truth, chain, eps, shift_extra)
    ref, bound = gn_y_ref(x, st, gamma, beta, silu)
    nb, hw, C = x.shape
    w_y = assert_within(f"{name} y", y.view(nb * hw, C), ref.view(nb * hw, C), bound.view(nb * hw, C))
    return max(w_mean, w_rstd, w_y), (w_mean, w_rstd, w_y)


def _gn_params(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return 1 + 0.5 * torch.randn(C, device=_dev(), generator=g), torch.randn(C, device=_dev(), generator=g)


def _randn_bf16(shape, seed, scale=1.5, mean=0.3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = _padded(shape, BF16)
    x.copy_(torch.randn(shape, device=_dev(), generator=g) * scale + mean)
    return x


def _tile_offset(t):
    return ((t % 5) - 2) * 0.75


def _host_parts(xs, geoms, nb):
    return [(build_records(x, gm, nb, _tile_offset), gm) for x, gm in zip(xs, geoms)]


GN_ADVERSARIAL = [  # id, batch, ho, wo, c0, c1, groups, input pattern
    ("large-mean-64x64-320", 2, 64, 64, 320, 0, 32, "large_mean"),
    ("outlier-first-element-32x32-640", 2, 32, 32, 640, 0, 32, "outlier_first"),
    ("outlier-edge-tile-20x27-1280+640", 2, 20, 27, 1280, 640, 32, "outlier_edge"),
    ("edge-tiles-10x14-1280+1280", 2, 10, 14, 1280, 1280, 32, "randn"),
    ("edge-tiles-20x27-640+320", 1, 20, 27, 640, 320, 32, "large_mean"),
    ("segs2-odd-batch-8x8-1280", 3, 8, 8, 1280, 0, 32, "randn"),
    ("straddle-16x16-1280+640", 2, 16, 16, 1280, 640, 32, "large_mean"),
    ("straddle-32x32-640+320", 2, 32, 32, 640, 320, 32, "outlier_first"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,nb,ho,wo,c0,c1,groups,pattern", GN_ADVERSARIAL, ids=[c[0] for c in GN_ADVERSARIAL])
def test_group_norm_adversarial(ops, cid, nb, ho, wo, c0, c1, groups, pattern):
    """both statistics paths (standalone; finalize over host-built records with a different shift per tile) at
    production shapes: a large mean over a small spread, an outlier at each group's first element (the standalone
    shift), an outlier in the first row of the edge tile (that tile's record shift), pixel counts that are not a
    multiple of the pixel box, two samples per tile with an odd batch, groups straddling the two sources"""
    hw = ho * wo
    seed = sum(map(ord, cid))
    xs = []
    for si, c in enumerate((c0, c1)):
        if not c:
            continue
        if pattern == "large_mean":
            x = _randn_bf16((nb, hw, c), seed + si, scale=2.0, mean=100.0 if si == 0 else -60.0)
        else:
            x = _randn_bf16((nb, hw, c), seed + si)
        if pattern == "outlier_first":  # pixel 0, first channel of every group that starts in this source
            cpg = (c0 + c1) // groups
            first = [g * cpg - (c0 if si else 0) for g in range(groups)]
            x[:, 0, [f for f in first if 0 <= f < c]] = 300.0
        xs.append(x)
    geoms = [stats_geom_of_conv(nb, ho, wo, c) for c in (c0, c1) if c]
    if pattern == "outlier_edge":  # the first (valid) pixel of the last tile: the shift of that tile's record
        t, y0, y1, x0_, x1_ = tile_boxes(geoms[0])[-1]
        assert y1 - y0 < geoms[0].bh or x1_ - x0_ < geoms[0].bw, "the last tile must be an edge tile"
        for x in xs:
            x.view(nb, ho, wo, -1)[:, y0, x0_] = 250.0
    x0, x1 = xs[0], (xs[1] if c1 else None)
    gamma, beta = _gn_params(c0 + c1, seed)
    if "straddle" in cid:
        assert c0 % ((c0 + c1) // groups) != 0, "a group must straddle the two sources"
    if "segs2" in cid:
        assert geoms[0].segs == 2 and nb % 2 == 1
    w_s, _ = check_group_norm(ops, f"{cid} standalone", x0, x1, groups, 1e-5, True, gamma, beta,
                              standalone_chain(nb, hw, c0 + c1, groups))
    w_p, parts = check_group_norm(ops, f"{cid} host records", x0, x1, groups, 1e-5, True, gamma, beta,
                                  HOST_RECORD_CHAIN, parts=_host_parts(xs, geoms, nb), shift_extra=1.5)
    print(f"[group_norm {cid}] boxes {[(g.bw, g.bh, g.segs) for g in geoms]} worst err/bound standalone {w_s:.3f}, "
          f"host records {w_p:.3f} (mean {parts[0]:.3f} rstd {parts[1]:.3f} y {parts[2]:.3f})")


@pytest.mark.gpu
def test_census_group_norm(ops, census):
    """every distinct GroupNorm the programs record, on fresh seeded inputs: the standalone path always; a signature
    recorded over producer records also through its captured producer GEMM(s) rebuilt fresh with chan_stats attached,
    and through host-built records with a different shift per tile"""
    sigs = census.sigs.get("gn", {})
    assert sigs, "the programs record GroupNorms"
    worst = {"standalone": 0.0, "producer": 0.0, "host records": 0.0}
    for i, (c, meta) in enumerate(sigs.values()):
        nb, hw, c0, c1, groups = c.batch, c.hw, c.c0, c.c1, c.groups
        C = c0 + c1
        name = f"census gn #{i} ({meta['source']}) batch={nb} hw={hw} C={c0}+{c1} silu={c.silu}"
        gamma, beta = _gn_params(C, 7000 + i)
        paths = []
        if c.from_partials:
            prods = meta["producers"]
            assert all(p is not None for p in prods), f"{name}: producer GEMM not captured"
            xs, parts = [], []
            for k, (gc, variant) in enumerate(prods):
                desc, _, outs, _, extra = _fresh_gemm(gc, variant, seed=8000 + 2 * i + k)
                assert desc.c.ldc == desc.c.N and gemm_out_geometry(desc.c)[0] == nb * hw, name
                geo = ops.gemm_stats_geometry(desc)
                assert _geom_tuple(geo) == _geom_tuple(c.geom0 if k == 0 else c.geom1), name
                ops.run(desc)
                xs.append(outs["out"].view(nb, hw, -1))
                parts.append((extra["part"], geo))
            torch.cuda.synchronize()
            x0, x1 = xs[0], (xs[1] if c1 else None)
            chain = max(producer_chain(g) for _, g in parts)
            w, _ = check_group_norm(ops, f"{name} producer", x0, x1, groups, c.eps, bool(c.silu), gamma, beta,
                                    chain, parts=parts)
            worst["producer"] = max(worst["producer"], w)
            paths.append(f"producer {w:.3f}")
            w, _ = check_group_norm(ops, f"{name} host records", x0, x1, groups, c.eps, bool(c.silu), gamma, beta,
                                    HOST_RECORD_CHAIN, parts=_host_parts(xs, [g for _, g in parts], nb),
                                    shift_extra=1.5)
            worst["host records"] = max(worst["host records"], w)
            paths.append(f"host records {w:.3f}")
        else:
            x0 = _randn_bf16((nb, hw, c0), 9000 + i)
            x1 = _randn_bf16((nb, hw, c1), 9500 + i, scale=1.0, mean=-0.4) if c1 else None
        w, _ = check_group_norm(ops, f"{name} standalone", x0, x1, groups, c.eps, bool(c.silu), gamma, beta,
                                standalone_chain(nb, hw, C, groups))
        worst["standalone"] = max(worst["standalone"], w)
        paths.append(f"standalone {w:.3f}")
        print(f"[census gn #{i}] batch={nb} hw={hw} C={c0}+{c1} groups={groups} silu={c.silu} "
              f"{'from_partials' if c.from_partials else 'standalone'} ({meta['source']}): worst err/bound "
              + ", ".join(paths))
        torch.cuda.empty_cache()
    print(f"[census gn] {len(sigs)} signatures; worst err/bound per path: "
          + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


# =========================================================================== GPU: LayerNorm
def check_layer_norm(name, rows, c, eps, mean, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = _padded((rows, c), BF16)
    x.copy_(torch.randn(rows, c, device=_dev(), generator=g) * 2 + mean)
    gamma = torch.randn(c, device=_dev(), generator=g)
    beta = torch.randn(c, device=_dev(), generator=g)
    canv = Canvas(rows, c, c, BF16, _dev(), pad_rows=8)

    def run():
        canv.view.fill_(float("nan"))
        _check(_lib().pp_layer_norm(x.data_ptr(), canv.view.data_ptr(), gamma.data_ptr(), beta.data_ptr(), rows, c,
                                    eps, _stream()), "pp_layer_norm")
        torch.cuda.synchronize()
        return canv.view.clone()
    first = run()
    ref, bound = ref_layer_norm(x, gamma, beta, eps)
    worst = assert_within(name, first, ref, bound)
    assert torch.equal(_bits(run()), _bits(first)), f"{name}: two runs differ"
    assert_canvases(name, {"y": canv})
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("cid,rows,c,mean", LN_CASES, ids=[c[0] for c in LN_CASES])
def test_layer_norm(ops, cid, rows, c, mean):
    worst = check_layer_norm(cid, rows, c, 1e-5, mean, sum(map(ord, cid)))
    print(f"[layer_norm {cid}] layer_norm_kernel<{layer_norm_instance(c)}> rows={rows} c={c} worst err/bound = "
          f"{worst:.3f}")


# =========================================================================== GPU: row softmax, causal attention
def _softmax_scores(rows, cols, ld_s, seed):
    """fp32 scores [rows, cols] at row pitch ld_s (pitch columns NaN) with rows of -inf entries, huge logits, the
    maximum in the last column"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.full((rows + 2, ld_s), float("nan"), device=_dev())
    s = buf[1:rows + 1, :cols]
    s.copy_(torch.randn(rows, cols, device=_dev(), generator=g) * 4)
    if rows > 6:
        s[0, ::3] = float("-inf")
        s[0, 0] = 1.0
        s[1] = s[1] * 1e3 + 1e4                       # very large logits, large spread
        s[2, -1] = s[2].max() + 2.0                   # the last column carries a visible share
        s[3] = float("-inf")
        s[3, cols // 2] = -5.0                        # one finite logit
        s[4] = torch.where(s[4] > 0, 3.0e38, -3.0e38)  # the largest finite floats
        s[5] = s[5] + 80.0                            # exp of every logit alone would overflow fp16
    return buf, s


def check_softmax(name, rows, cols, ld_s, ld_p, seed):
    buf, s = _softmax_scores(rows, cols, ld_s, seed)
    canv = Canvas(rows, cols, ld_p, BF16, _dev(), pad_rows=4)

    def run():
        canv.view.fill_(float("nan"))
        _check(_lib().pp_softmax_rows(s.data_ptr(), canv.view.data_ptr(), rows, cols, ld_s, ld_p, _stream()),
               "pp_softmax_rows")
        torch.cuda.synchronize()
        return canv.view.clone()
    first = run()
    p, bound = ref_softmax(s, softmax_instance(cols))
    worst = assert_within(name, first, p, bound)
    assert torch.equal(_bits(run()), _bits(first)), f"{name}: two runs differ"
    assert_canvases(name, {"p": canv})
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("cols", SOFTMAX_COLS)
def test_softmax_rows(ops, cols):
    rows = 37
    worst = check_softmax(f"softmax cols={cols}", rows, cols, cols + 5, cols + 13, cols)
    print(f"[softmax_rows cols={cols}] softmax_rows_kernel<{softmax_instance(cols)}> rows={rows} worst err/bound = "
          f"{worst:.3f}")


def check_causal(name, batch, seq, heads, d, scale, seed):
    C = heads * d
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = _padded((batch * seq, 3 * C), BF16)
    qkv.copy_(torch.randn(batch * seq, 3 * C, device=_dev(), generator=g) * 1.5)
    canv = Canvas(batch * seq, C, C, BF16, _dev(), pad_rows=8)

    def run():
        canv.view.fill_(float("nan"))
        _check(_lib().pp_causal_attention_small(qkv.data_ptr(), canv.view.data_ptr(), batch, seq, heads, d, scale,
                                                _stream()), "pp_causal_attention_small")
        torch.cuda.synchronize()
        return canv.view.clone()
    first = run()
    r, bound = ref_causal_attention(qkv, batch, seq, heads, d, scale)
    worst = assert_within(name, first, r, bound)
    assert torch.equal(_bits(run()), _bits(first)), f"{name}: two runs differ"
    assert_canvases(name, {"out": canv})
    return worst


CAUSAL_CASES = [(d, seq) for d in (8, 16, 32, 64) for seq in CAUSAL_SEQS]


@pytest.mark.gpu
@pytest.mark.parametrize("d,seq", CAUSAL_CASES, ids=[f"d{d}-seq{s}" for d, s in CAUSAL_CASES])
def test_causal_attention_small(ops, d, seq):
    heads = max(1, 256 // d)
    worst = check_causal(f"causal d={d} seq={seq}", 2, seq, heads, d, 1 / math.sqrt(d), 100 * d + seq)
    print(f"[causal_attention_small d={d} seq={seq}] heads={heads} worst err/bound = {worst:.3f}")


# =========================================================================== GPU: exact kernels
def check_upsample(name, nb, h, w, c, ho, wo, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = _padded((nb, h, w, c), BF16)
    x.copy_(torch.randn(nb, h, w, c, device=_dev(), generator=g))
    canv = Canvas(nb * ho * wo, c, c, BF16, _dev(), pad_rows=8)
    if (ho, wo) == (2 * h, 2 * w):
        _check(_lib().pp_upsample2x(x.data_ptr(), canv.view.data_ptr(), nb, h, w, c, _stream()), "pp_upsample2x")
    else:
        _check(_lib().pp_upsample_nearest(x.data_ptr(), canv.view.data_ptr(), nb, h, w, c, ho, wo, _stream()),
               "pp_upsample_nearest")
    torch.cuda.synchronize()
    ref = F.interpolate(x.permute(0, 3, 1, 2), size=(ho, wo), mode="nearest").permute(0, 2, 3, 1)
    assert_bits_equal(name, canv.view, ref.reshape(nb * ho * wo, c))
    assert_canvases(name, {"y": canv})


UPSAMPLE_CASES = [(2, 6, 10, 64, 12, 20), (2, 5, 7, 16, 13, 11), (1, 20, 27, 32, 10, 14), (2, 10, 14, 64, 20, 27),
                  (1, 7, 9, 8, 21, 18), (3, 40, 54, 8, 80, 107), (1, 9, 9, 24, 4, 30)]


@pytest.mark.gpu
def test_exact_small_ops(ops):
    """upsample (2x and explicit sizes up and down) against F.interpolate; add beyond one grid pass; the embedding
    gather at the table ends; both layout conversions (c, hw, c_ld not multiples of 32; bf16 and fp32 sources;
    c_pad > c zero-filled); image pre-processing with all three mask modes: bit for bit"""
    for i, case in enumerate(UPSAMPLE_CASES):
        check_upsample(f"upsample {case}", *case, seed=i)
    # add
    g = torch.Generator(device="cuda").manual_seed(5)
    for n in (8, 4104, 2 * SMS * 16 * 256 * 8 + 24):
        a = _padded((n,), BF16)
        b = _padded((n,), BF16)
        a.copy_(torch.randn(n, device=_dev(), generator=g) * 3)
        b.copy_(torch.randn(n, device=_dev(), generator=g) * 1e-3)
        canv = Canvas(n // 8, 8, 8, BF16, _dev(), pad_rows=4)
        _check(_lib().pp_add(a.data_ptr(), b.data_ptr(), canv.view.data_ptr(), n, _stream()), "pp_add")
        torch.cuda.synchronize()
        assert_bits_equal(f"add n={n}", canv.view.reshape(-1), (a.float() + b.float()).to(BF16))
        assert_canvases(f"add n={n}", {"y": canv})
    # embedding gather
    for rows, vocab, seq, dim, n_ext in ((2 * 77, 1000, 77, 768, 10), (3 * 5, 40, 5, 36, 12)):
        base = torch.randn(vocab, dim, device=_dev(), generator=g)
        ext = torch.randn(n_ext, dim, device=_dev(), generator=g) * 0.1
        pos = torch.randn(seq, dim, device=_dev(), generator=g)
        idx = torch.randint(0, vocab + n_ext, (rows,), device=_dev(), generator=g, dtype=torch.int32)
        idx[:4] = torch.tensor([0, vocab - 1, vocab, vocab + 9], dtype=torch.int32)
        canv = Canvas(rows, dim, dim, BF16, _dev(), pad_rows=4)
        _check(_lib().pp_embed_gather(idx.data_ptr(), base.data_ptr(), ext.data_ptr(), pos.data_ptr(),
                                      canv.view.data_ptr(), rows, vocab, seq, dim, _stream()), "pp_embed_gather")
        torch.cuda.synchronize()
        table = torch.cat([base, ext])
        ref = (table[idx.long()] + pos[torch.arange(rows, device=_dev()) % seq]).to(BF16)
        assert_bits_equal(f"embed_gather vocab={vocab}", canv.view, ref)
        assert_canvases("embed_gather", {"out": canv})
    # NCHW fp32 -> NHWC bf16 with zero-filled channel pad
    for nb, c, hw, c_pad in ((2, 3, 45, 8), (1, 37, 1000, 40), (3, 4, 33, 4), (2, 9, 35, 16)):
        x = _padded((nb, c, hw), torch.float32)
        x.copy_(torch.randn(nb, c, hw, device=_dev(), generator=g) * 5)
        canv = Canvas(nb * hw, c_pad, c_pad, BF16, _dev(), pad_rows=4)
        _check(_lib().pp_nchw_to_nhwc(x.data_ptr(), canv.view.data_ptr(), nb, c, hw, c_pad, _stream()),
               "pp_nchw_to_nhwc")
        torch.cuda.synchronize()
        ref = torch.zeros(nb, hw, c_pad, device=_dev(), dtype=BF16)
        ref[..., :c] = x.permute(0, 2, 1).to(BF16)
        assert_bits_equal(f"nchw_to_nhwc {(nb, c, hw, c_pad)}", canv.view, ref.view(nb * hw, c_pad))
        assert_canvases("nchw_to_nhwc", {"y": canv})
    # NHWC (bf16 / fp32, channel pitch c_ld) -> NCHW fp32
    for nb, c, hw, c_ld, dt in ((2, 3, 45, 8, BF16), (1, 37, 1000, 40, torch.float32), (2, 33, 67, 48, BF16),
                                (1, 4, 31, 4, torch.float32)):
        x = torch.full((nb, hw, c_ld), float("nan"), device=_dev(), dtype=dt)  # the pitch channels are never read
        x[..., :c] = (torch.randn(nb, hw, c, device=_dev(), generator=g) * 5).to(dt)
        canv = Canvas(nb * c, hw, hw, torch.float32, _dev(), pad_rows=4)
        _check(_lib().pp_nhwc_to_nchw(x.data_ptr(), int(dt == torch.float32), canv.view.data_ptr(), nb, c, hw, c_ld,
                                      _stream()), "pp_nhwc_to_nchw")
        torch.cuda.synchronize()
        assert_bits_equal(f"nhwc_to_nchw {(nb, c, hw, c_ld, dt)}", canv.view,
                          x[..., :c].float().permute(0, 2, 1).reshape(nb * c, hw))
        assert_canvases("nhwc_to_nchw", {"y": canv})
    # uint8 image (+ mask) -> bf16 NHWC
    nb, h, w, c_pad = 2, 37, 45, 8
    hw = h * w
    img = torch.randint(0, 256, (nb, 3, h, w), device=_dev(), generator=g, dtype=torch.uint8)
    img[0, :, 0, :4] = torch.tensor([0, 127, 128, 255], dtype=torch.uint8)
    m8 = torch.randint(0, 256, (nb, 1, h, w), device=_dev(), generator=g, dtype=torch.uint8)
    m8[0, 0, 0, :4] = torch.tensor([127, 128, 0, 255], dtype=torch.uint8)
    mf = torch.rand(nb, 1, h, w, device=_dev(), generator=g)
    mf[0, 0, 0, :4] = torch.tensor([0.5, float(np.nextafter(np.float32(0.5), np.float32(0))), 0.0, 1.0])
    for mode, mask in ((0, None), (1, m8), (2, mf)):
        for divisor, shift in ((127.5, -1.0), (255.0, 0.0)):
            canv = Canvas(nb * hw, c_pad, c_pad, BF16, _dev(), pad_rows=4)
            _check(_lib().pp_image_preprocess_u8(img.data_ptr(), mask.data_ptr() if mask is not None else None, mode,
                                                 canv.view.data_ptr(), nb, hw, c_pad, divisor, shift, _stream()),
                   "pp_image_preprocess_u8")
            torch.cuda.synchronize()
            px = img.cpu().numpy().reshape(nb, 3, hw).transpose(0, 2, 1).astype(np.float32)
            v = px / np.float32(divisor) + np.float32(shift)
            if mode:
                mk = mask.cpu().numpy().reshape(nb, hw, 1)
                mk = (mk.astype(np.float32) / np.float32(255)) if mode == 1 else mk
                v = v * (mk < np.float32(0.5)).astype(np.float32)
            ref = torch.zeros(nb, hw, c_pad, dtype=BF16)
            ref[..., :3] = torch.from_numpy(np.ascontiguousarray(v)).to(BF16)
            assert_bits_equal(f"image_preprocess mode={mode} /{divisor}{shift:+}", canv.view.cpu(),
                              ref.view(nb * hw, c_pad))
            assert_canvases("image_preprocess", {"out": canv})
    print("[exact small ops] upsample, add, embed_gather, nchw<->nhwc, image_preprocess: bit-exact")


def _u8_canvas(n, pad=64):
    buf = torch.full((n + 2 * pad,), 0xA5, dtype=torch.uint8, device=_dev())
    return buf, buf[pad:pad + n]


def _u8_tail_intact(buf, n, pad=64):
    return bool((buf[:pad] == 0xA5).all()) and bool((buf[pad + n:] == 0xA5).all())


def run_postprocess(x, x_fp32, c_ld, hw):
    """pp_image_postprocess of x [hw, c_ld] into a uint8 NHWC and an fp32 NCHW output (nb = 1)"""
    buf, u8 = _u8_canvas(hw * 3)
    u8.fill_(0)
    canv = Canvas(3, hw, hw, torch.float32, _dev(), pad_rows=2)
    _check(_lib().pp_image_postprocess(x.data_ptr(), x_fp32, c_ld, u8.data_ptr(), canv.view.data_ptr(), 1, hw,
                                       _stream()), "pp_image_postprocess")
    torch.cuda.synchronize()
    assert _u8_tail_intact(buf, hw * 3), "image_postprocess wrote outside its uint8 output"
    assert_canvases("image_postprocess f32", {"out": canv})
    return u8.view(hw, 3).cpu(), canv.view.cpu()


@pytest.mark.gpu
def test_image_postprocess_exhaustive(ops):
    """every finite bf16 value and +-inf, in each of the three channels (channel pitch 4, the pitch channel NaN), and
    fp32 inputs that are exact ties to even: uint8 against `(x / 2 + 0.5).clamp(0, 1)` then numpy round-half-even,
    fp32 NCHW against the clamp"""
    pat = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF16)
    vals = pat[~torch.isnan(pat.float())]
    hw = vals.numel()
    x = torch.full((hw, 4), float("nan"), dtype=BF16)
    for ch in range(3):
        x[:, ch] = vals.roll(ch * 7919)
    got_u8, got_f = run_postprocess(x.to(_dev()), 0, 4, hw)
    for ch in range(3):
        want_u8, want_f = ref_postprocess_u8(x[:, ch])
        assert_bits_equal(f"postprocess u8 bf16 channel {ch}", got_u8[:, ch], want_u8)
        assert_bits_equal(f"postprocess f32 bf16 channel {ch}", got_f[ch], want_f)
    ties = postprocess_tie_inputs()
    xf = torch.stack([ties, ties.flip(0), ties], 1).contiguous()
    got_u8, got_f = run_postprocess(xf.to(_dev()), 1, 3, ties.numel())
    for ch in range(3):
        want_u8, want_f = ref_postprocess_u8(xf[:, ch])
        assert_bits_equal(f"postprocess u8 fp32 ties channel {ch}", got_u8[:, ch], want_u8)
        assert_bits_equal(f"postprocess f32 fp32 ties channel {ch}", got_f[ch], want_f)
    print(f"[image_postprocess] {hw} bf16 values and {ties.numel()} fp32 ties to even: bit-exact")


def check_time_embed(name, table, step_idx, batch, dim):
    canv = Canvas(batch, dim, dim, BF16, _dev(), pad_rows=4)
    si = torch.tensor([step_idx], device=_dev(), dtype=torch.int32) if step_idx is not None else None
    _check(_lib().pp_time_embed(table.data_ptr(), si.data_ptr() if si is not None else None, canv.view.data_ptr(),
                                batch, dim, _stream()), "pp_time_embed")
    torch.cuda.synchronize()
    t = table[step_idx].expand(batch) if step_idx is not None else table[:batch]
    e, bound = ref_time_embed(t, dim)
    worst = assert_within(name, canv.view, e, bound)
    assert_canvases(name, {"out": canv})
    return worst


@pytest.mark.gpu
def test_time_embed(ops):
    """timesteps[0..batch) and the graph-replay form timesteps[*step_idx] for every row, against fp64 on the fp32
    arguments to U16 |e| + |t| c 2^-24"""
    table = torch.tensor([999.0, 981.0, 1.0, 500.0, 500.5, 0.0, 761.0, 21.0], device=_dev())
    worst = 0.0
    for dim in (320, 1280, 8):
        worst = max(worst, check_time_embed(f"time_embed dim={dim}", table, None, 8, dim))
        for s in (0, 3, 6):
            worst = max(worst, check_time_embed(f"time_embed step_idx={s} dim={dim}", table, s, 4, dim))
    print(f"[time_embed] worst err/bound = {worst:.3f}")


# =========================================================================== GPU: census of the small ops
@pytest.mark.gpu
def test_census_op_kinds_are_all_covered(census):
    """every op kind the programs record is checked here or names the file that checks it; a new kind fails"""
    from test_program_replay_gpu import REPLAY_EVALUATED  # the step kernels, on the programs' own activations

    recorded = set(census.records)
    unknown = recorded - set(CHECKED_HERE) - set(COVERED_ELSEWHERE) - set(REPLAY_EVALUATED)
    assert not unknown, f"op kinds recorded by the programs but checked nowhere: {sorted(unknown)}"
    assert {"gn", "layer_norm", "add", "time_embed", "softmax_rows", "embed_gather", "causal_attention_small",
            "window_copy", "tile_blend", "memset"} <= recorded, sorted(recorded)
    assert any(c.from_partials for c, _ in census.sigs["gn"].values())
    assert any(not c.from_partials for c, _ in census.sigs["gn"].values())


@pytest.mark.gpu
def test_census_small_ops(ops, census):
    """every distinct LayerNorm, upsample, softmax, embedding gather, causal attention, add and timestep embedding
    the programs record, on fresh seeded inputs"""
    worst = {}
    sig = census.sigs
    for i, (a, meta) in enumerate(sig.get("layer_norm", {}).values()):
        w = check_layer_norm(f"census layer_norm #{i} ({meta['source']})", a["rows"], a["c"], a["eps"], 3.0, 300 + i)
        worst["layer_norm"] = max(worst.get("layer_norm", 0.0), w)
        print(f"[census layer_norm #{i}] rows={a['rows']} c={a['c']} ({meta['source']}) worst err/bound = {w:.3f}")
    for kind in ("upsample2x", "upsample_nearest"):
        for i, (a, meta) in enumerate(sig.get(kind, {}).values()):
            ho, wo = (a["ho"], a["wo"]) if kind == "upsample_nearest" else (2 * a["h"], 2 * a["w"])
            check_upsample(f"census {kind} #{i}", a["nb"], a["h"], a["w"], a["c"], ho, wo, 400 + i)
            print(f"[census {kind} #{i}] {a['nb']}x{a['h']}x{a['w']}x{a['c']} -> {ho}x{wo} ({meta['source']}) exact")
    for i, (a, meta) in enumerate(sig.get("softmax_rows", {}).values()):
        w = check_softmax(f"census softmax #{i}", a["rows"], a["cols"], a["ld_s"], a["ld_p"], 500 + i)
        worst["softmax_rows"] = max(worst.get("softmax_rows", 0.0), w)
        print(f"[census softmax_rows #{i}] rows={a['rows']} cols={a['cols']} ld_p={a['ld_p']} ({meta['source']}) "
              f"worst err/bound = {w:.3f}")
    for i, (a, meta) in enumerate(sig.get("causal_attention_small", {}).values()):
        w = check_causal(f"census causal #{i}", a["batch"], a["seq"], a["heads"], a["d"], a["scale"], 600 + i)
        worst["causal_attention_small"] = max(worst.get("causal_attention_small", 0.0), w)
        print(f"[census causal_attention_small #{i}] batch={a['batch']} seq={a['seq']} heads={a['heads']} d={a['d']} "
              f"({meta['source']}) worst err/bound = {w:.3f}")
    g = torch.Generator(device="cuda").manual_seed(77)
    for i, (a, meta) in enumerate(sig.get("embed_gather", {}).values()):
        rows, vocab, seq, dim = a["rows"], a["vocab"], a["seq"], a["dim"]
        n_ext = 10
        base = torch.randn(vocab, dim, device=_dev(), generator=g)
        ext = torch.randn(n_ext, dim, device=_dev(), generator=g)
        pos = torch.randn(seq, dim, device=_dev(), generator=g)
        idx = torch.randint(0, vocab + n_ext, (rows,), device=_dev(), generator=g, dtype=torch.int32)
        idx[:4] = torch.tensor([0, vocab - 1, vocab, vocab + 9], dtype=torch.int32)
        canv = Canvas(rows, dim, dim, BF16, _dev(), pad_rows=4)
        _check(_lib().pp_embed_gather(idx.data_ptr(), base.data_ptr(), ext.data_ptr(), pos.data_ptr(),
                                      canv.view.data_ptr(), rows, vocab, seq, dim, _stream()), "pp_embed_gather")
        torch.cuda.synchronize()
        ref = (torch.cat([base, ext])[idx.long()] + pos[torch.arange(rows, device=_dev()) % seq]).to(BF16)
        assert_bits_equal(f"census embed_gather #{i}", canv.view, ref)
        assert_canvases("census embed_gather", {"out": canv})
        print(f"[census embed_gather #{i}] rows={rows} vocab={vocab} dim={dim} ({meta['source']}) exact")
        del base
    for i, (a, meta) in enumerate(sig.get("add", {}).values()):
        n = a["n"]
        x, y = _padded((n,), BF16), _padded((n,), BF16)
        x.copy_(torch.randn(n, device=_dev(), generator=g))
        y.copy_(torch.randn(n, device=_dev(), generator=g))
        canv = Canvas(n // 8, 8, 8, BF16, _dev(), pad_rows=4)
        _check(_lib().pp_add(x.data_ptr(), y.data_ptr(), canv.view.data_ptr(), n, _stream()), "pp_add")
        torch.cuda.synchronize()
        assert_bits_equal(f"census add #{i}", canv.view.reshape(-1), (x.float() + y.float()).to(BF16))
        assert_canvases("census add", {"y": canv})
        print(f"[census add #{i}] n={n} ({meta['source']}) exact")
    for i, (a, meta) in enumerate(sig.get("time_embed", {}).values()):
        table = torch.cat([torch.tensor([999.0, 1.0, 0.0, 500.5], device=_dev()),
                           torch.randint(0, 1000, (a["batch"] + 8,), device=_dev(), generator=g).float()])
        step = 5 if "step_idx" in a["_nonnull"] else None
        w = check_time_embed(f"census time_embed #{i}", table, step, a["batch"], a["dim"])
        worst["time_embed"] = max(worst.get("time_embed", 0.0), w)
        print(f"[census time_embed #{i}] batch={a['batch']} dim={a['dim']} step_idx={step is not None} "
              f"({meta['source']}) worst err/bound = {w:.3f}")
    print("[census small ops] worst err/bound per kind: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
