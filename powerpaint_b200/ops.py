"""Descriptor builders and immediate-mode wrappers over the C ABI (include/powerpaint_b200.h).

Every function takes torch CUDA tensors (device memory + stream plumbing only), fills the
C descriptor with raw pointers / pitches, and either launches on torch's current stream
(`gemm`, `attention`, ...) or returns the descriptor for recording into a `Program`.
There is no fallback: a failure raises `RuntimeError` carrying `pp_last_error()`.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _native as N

BF16 = torch.bfloat16


def _req(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


# --------------------------------------------------------------------------- weights
def pack_linear_weight(w: torch.Tensor) -> torch.Tensor:
    """nn.Linear / 1x1 conv weight [N, K(,1,1)] -> bf16 [N, K] K-major."""
    return w.reshape(w.shape[0], -1).to(BF16).contiguous()


def pad64(c: int) -> int:
    return (c + 63) // 64 * 64


def pack_conv3x3_weight(w: torch.Tensor, split: Optional[int] = None) -> torch.Tensor:
    """Conv2d weight [Cout, Cin, 3, 3] -> bf16 [Cout, 9 * (pad64(c0) + pad64(c1))], K ordered
    (tap = ky*3+kx, source, channel) with each (tap, source) segment zero-padded to 64.
    `split` = channels of source 0 when the input is a concat of two tensors."""
    cout, cin = w.shape[0], w.shape[1]
    c0 = cin if split is None else split
    c1 = cin - c0
    p0, p1 = pad64(c0), (pad64(c1) if c1 else 0)
    out = torch.zeros(cout, 9, p0 + p1, dtype=BF16, device=w.device)
    wt = w.permute(0, 2, 3, 1).reshape(cout, 9, cin).to(BF16)  # [cout, tap, cin]
    out[:, :, :c0] = wt[:, :, :c0]
    if c1:
        out[:, :, p0:p0 + c1] = wt[:, :, c0:]
    return out.reshape(cout, 9 * (p0 + p1)).contiguous()


def pack_concat_linear_weight(w: torch.Tensor, split: int) -> torch.Tensor:
    """1x1 conv weight over a two-source concat: [N, c0 + c1] -> [N, pad64(c0) + pad64(c1)]."""
    w = w.reshape(w.shape[0], -1)
    n, cin = w.shape
    c0, c1 = split, cin - split
    p0, p1 = pad64(c0), pad64(c1)
    out = torch.zeros(n, p0 + p1, dtype=BF16, device=w.device)
    out[:, :c0] = w[:, :c0].to(BF16)
    out[:, p0:p0 + c1] = w[:, c0:].to(BF16)
    return out.contiguous()


def pack_geglu_weight(w: torch.Tensor, b: torch.Tensor, block_n: int = 128):
    """GEGLU proj weight [2*F, K] (rows 0..F = value, F..2F = gate) -> tile-interleaved so every
    block_n-row tile holds block_n/2 value rows followed by their block_n/2 gate rows."""
    f2, k = w.shape
    f = f2 // 2
    half = block_n // 2
    assert f % half == 0, (f, half)
    wv, wg = w[:f].reshape(f // half, half, k), w[f:].reshape(f // half, half, k)
    wi = torch.cat([wv, wg], dim=1).reshape(f2, k)
    bv, bg = b[:f].reshape(f // half, half), b[f:].reshape(f // half, half)
    bi = torch.cat([bv, bg], dim=1).reshape(f2)
    return wi.to(BF16).contiguous(), bi.float().contiguous()


def fold_layer_norm_into_linear(w: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor,
                                bias: Optional[torch.Tensor] = None):
    """LayerNorm(x) W^T + b as a GEMM on the raw x:  rstd (x W'^T - mean u) + b'  with  W' = W * gamma (bf16, what the
    tensor core multiplies), u = row sums of that bf16 W', b' = W beta (+ b). Returns (W' bf16 [N, K], u fp32 [N],
    b' fp32 [N]); the statistics (mean, rstd) come from the producer of x at run time (pp_gemm_desc.ln_stats)."""
    w = w.reshape(w.shape[0], -1).float()
    b = w.double() @ beta.double()
    if bias is not None:
        b = b + bias.double()
    wf = (w * gamma.float()[None, :]).to(BF16)
    u = wf.double().sum(1)
    return wf.contiguous(), u.float().contiguous(), b.float().contiguous()


# --------------------------------------------------------------------------- descriptors
class Desc:
    """A filled C descriptor plus the tensors it points into (kept alive)."""

    def __init__(self, kind: str, c_struct, keep):
        self.kind = kind
        self.c = c_struct
        self.keep = keep


def gemm_desc(*, a0: torch.Tensor, w: torch.Tensor, out: torch.Tensor, N_: int,
              a_mode: int = N.PP_A_MATRIX, a1: Optional[torch.Tensor] = None,
              c0: Optional[int] = None, c1: int = 0, M: int = 0, lda0: int = 0, lda1: int = 0,
              nb: int = 0, h: int = 0, w_: int = 0, ldb: int = 0,
              bias: Optional[torch.Tensor] = None, rowvec: Optional[torch.Tensor] = None,
              rows_per_group: int = 0, rowvec_ld: int = 0, res1: Optional[torch.Tensor] = None, ldr1: int = 0,
              res2: Optional[torch.Tensor] = None, ldr2: int = 0, alpha: float = 1.0,
              act: int = N.PP_ACT_NONE, epilogue: int = N.PP_EPI_PLAIN, ldc: int = 0,
              out_fp32: bool = False, t_rows: int = 0, t_ld: int = 0, block_n: int = 0, t_fp16: bool = False,
              alpha_dev: Optional[torch.Tensor] = None, alpha_step: Optional[torch.Tensor] = None,
              alpha_stride: int = 0, chan_stats: Optional[torch.Tensor] = None,
              ln: Optional[tuple] = None, out_t: Optional[torch.Tensor] = None, trans_from_col: int = 0) -> Desc:
    """`ln` = (row stats [M, 2] fp32 = a producer's `row_final`, u [N] fp32, eps): LayerNorm of A folded into the
    epilogue — `w` must carry gamma (W * gamma) and `bias` the W @ beta term (include/powerpaint_b200.h)"""
    d = N.GemmDesc()
    d.a_mode, d.epilogue = a_mode, epilogue
    d.a0, d.a1 = N.ptr(a0), N.ptr(a1)
    d.c0 = c0 if c0 is not None else a0.shape[-1]
    d.c1 = c1
    d.lda0 = lda0 or d.c0
    d.lda1 = lda1 or c1
    d.nb, d.h, d.w = nb, h, w_
    d.M, d.N = M, N_
    d.b = N.ptr(w)
    d.ldb = ldb or w.shape[-1]
    d.bias, d.rowvec, d.rows_per_group = N.ptr(bias), N.ptr(rowvec), rows_per_group
    d.rowvec_ld = rowvec_ld
    d.res1, d.ldr1 = N.ptr(res1), (ldr1 or N_)
    d.res2, d.ldr2 = N.ptr(res2), (ldr2 or N_)
    d.alpha, d.act = alpha, act
    d.out = N.ptr(out)
    d.ldc = ldc or (N_ // 2 if epilogue == N.PP_EPI_GEGLU else trans_from_col if epilogue == N.PP_EPI_ROWS_THEN_TRANSPOSED
                    else N_)
    d.out_fp32 = 1 if out_fp32 else 0
    d.t_rows, d.t_ld = t_rows, t_ld
    d.block_n = block_n
    d.t_fp16 = 1 if t_fp16 else 0
    d.alpha_dev, d.alpha_step, d.alpha_stride = N.ptr(alpha_dev), N.ptr(alpha_step), alpha_stride
    d.chan_stats = N.ptr(chan_stats)
    d.out_t, d.trans_from_col = N.ptr(out_t), trans_from_col  # PP_EPI_ROWS_THEN_TRANSPOSED
    keep = [a0, a1, w, out, bias, rowvec, res1, res2, alpha_dev, alpha_step, chan_stats, out_t]
    if ln is not None:
        st, u, eps = ln
        if st.dtype != torch.float32 or st.dim() != 2 or st.shape[-1] != 2 or st.shape[0] < M or not st.is_contiguous():
            raise ValueError("ln row stats must be a contiguous fp32 [>= M, 2] tensor")
        if u.dtype != torch.float32 or u.numel() != N_ or not u.is_contiguous():
            raise ValueError("ln_u must be a contiguous fp32 [N] tensor")
        d.ln_stats, d.ln_u, d.ln_eps = N.ptr(st), N.ptr(u), eps
        keep += [st, u]
    return Desc("gemm", d, keep)


def gemm_splitk_query(desc: Desc):
    """host-only: (workspace bytes, tiles) if this launch could split K across two CTAs per tile, else (0, 0)"""
    t = N.i32(0)
    b = int(N.lib().pp_gemm_splitk_bytes(C.byref(desc.c), C.byref(t)))
    return b, int(t.value)


def attach_splitk(desc: Desc, ws: torch.Tensor, flags: torch.Tensor) -> None:
    """ws: fp32 workspace of at least the queried bytes; flags: zero-initialised int32, one per tile (left at zero)"""
    if ws.dtype != torch.float32 or flags.dtype != torch.int32:
        raise TypeError("split-K workspace must be fp32, flags int32")
    desc.c.splitk_ws, desc.c.splitk_flags = N.ptr(ws), N.ptr(flags)
    desc.keep += [ws, flags]


def gemm_row_stats_records(desc: Desc) -> int:
    """host-only: per-row LayerNorm records this GEMM can emit from its epilogue (0: it cannot)"""
    return int(N.lib().pp_gemm_row_stats_records(C.byref(desc.c)))


def gemm_variant(desc: Desc):
    """host-only: (block_n, mode, ksplit) of the kernel variant pp_gemm_conv would launch for this descriptor"""
    bn, mode, ks = N.i32(0), N.i32(0), N.i32(0)
    N.check(N.lib().pp_gemm_variant(C.byref(desc.c), C.byref(bn), C.byref(mode), C.byref(ks)), "pp_gemm_variant")
    return int(bn.value), int(mode.value), int(ks.value)


def gemm_staging(desc: Desc):
    """host-only: (res1 staged, row vector staged): the epilogue terms this launch stages in shared memory during the
    main loop"""
    r, v = N.i32(0), N.i32(0)
    N.check(N.lib().pp_gemm_staging(C.byref(desc.c), C.byref(r), C.byref(v)), "pp_gemm_staging")
    return bool(r.value), bool(v.value)


def attention_variant(desc: Desc):
    """host-only: (dv, p_fp16) of the kernel variant pp_attention would launch for this descriptor"""
    dv, f16 = N.i32(0), N.i32(0)
    N.check(N.lib().pp_attention_variant(C.byref(desc.c), C.byref(dv), C.byref(f16)), "pp_attention_variant")
    return int(dv.value), int(f16.value)


def attach_row_stats(desc: Desc, rec: torch.Tensor, final: torch.Tensor, ticket: torch.Tensor, eps: float) -> None:
    """rec: fp32 scratch [records, ld >= M, 4]; final: fp32 [>= M, 2] receives {rstd, -rstd * mean} per row; ticket: int32
    [>= ceil(M / 128)], zero-initialised (the kernel leaves it at zero)"""
    if final.dtype != torch.float32 or final.shape[-1] != 2 or not final.is_contiguous() or ticket.dtype != torch.int32:
        raise ValueError("row_final must be contiguous fp32 [M, 2], row_ticket int32")
    desc.c.row_stats, desc.c.row_stats_ld = N.ptr(rec), rec.shape[1]
    desc.c.row_final, desc.c.row_ticket, desc.c.ln_eps = N.ptr(final), N.ptr(ticket), eps
    desc.keep += [rec, final, ticket]


def gemm_stats_geometry(desc: Desc) -> "N.StatsGeom":
    """host-only: can this GEMM emit GroupNorm partial sums from its epilogue, and in which layout"""
    g = N.StatsGeom()
    N.check(N.lib().pp_gemm_stats_geometry(C.byref(desc.c), C.byref(g)), "pp_gemm_stats_geometry")
    return g


def attach_chan_stats(desc: Desc, buf: torch.Tensor) -> None:
    desc.c.chan_stats = N.ptr(buf)
    desc.keep.append(buf)


def attn_desc(*, q, k, vt, out, batch, heads, d, nq, nk, q_ld, k_ld, vt_ld, o_ld,
              q_batch_stride, k_batch_stride, scale) -> Desc:
    a = N.AttnDesc()
    a.q, a.k, a.vt, a.out = N.ptr(q), N.ptr(k), N.ptr(vt), N.ptr(out)
    a.batch, a.heads, a.d, a.nq, a.nk = batch, heads, d, nq, nk
    a.q_ld, a.k_ld, a.vt_ld, a.o_ld = q_ld, k_ld, vt_ld, o_ld
    a.q_batch_stride, a.k_batch_stride = q_batch_stride, k_batch_stride
    a.scale = scale
    a.vt_fp16 = 1 if vt.dtype == torch.float16 else 0
    return Desc("attn", a, (q, k, vt, out))


def gn_scratch_bytes(batch: int, hw: int, channels: int, groups: int) -> int:
    n = N.lib().pp_group_norm_scratch_bytes(batch, hw, channels, groups)
    if n <= 0:
        raise ValueError(f"invalid GroupNorm shape batch={batch} hw={hw} channels={channels} groups={groups}")
    return int(n)


def gn_desc(*, x0, x1, c0, c1, batch, hw, groups, gamma, beta, eps, silu, y, stats=None,
            stats_prezeroed=False, part0=None, geom0=None, part1=None, geom1=None) -> Desc:
    """`stats`: scratch of gn_scratch_bytes() bytes (fp32 tensor, 16-byte aligned); allocated (zeroed) here
    when omitted."""
    if stats is None:
        stats = torch.zeros((gn_scratch_bytes(batch, hw, c0 + c1, groups) + 3) // 4, dtype=torch.float32,
                            device=x0.device)
        stats_prezeroed = True
    g = N.GnDesc()
    g.x0, g.x1, g.c0, g.c1 = N.ptr(x0), N.ptr(x1), c0, c1
    g.batch, g.hw, g.groups = batch, hw, groups
    g.gamma, g.beta, g.eps, g.silu = N.ptr(gamma), N.ptr(beta), eps, 1 if silu else 0
    g.stats, g.y = N.ptr(stats), N.ptr(y)
    g.stats_prezeroed = 1 if stats_prezeroed else 0
    if part0 is not None:
        g.from_partials = 1
        g.part0, g.geom0 = N.ptr(part0), geom0
        if x1 is not None:
            g.part1, g.geom1 = N.ptr(part1), geom1
    return Desc("gn", g, (x0, x1, gamma, beta, stats, y, part0, part1))


RANDN_DRAW_BYTES = C.sizeof(N.RandnDraw)


def randn_draw_bytes(draws, n: int) -> torch.Tensor:
    """`n` pp_randn_draw entries as a uint8 host tensor: `draws` (tuples in the field order of `_native.RandnDraw`)
    first, then entries that match no row"""
    if len(draws) > n:
        raise ValueError(f"{len(draws)} draws for a table of {n}")
    arr = (N.RandnDraw * n)()
    for k, d in enumerate(draws):
        arr[k] = N.RandnDraw(*d)
    return torch.frombuffer(bytearray(arr), dtype=torch.uint8)


def _draws(table, noise):
    """(pointer, count) of a draw table (uint8 tensor of whole pp_randn_draw entries)"""
    if table is None:
        return None, 0
    if noise is not None:
        raise ValueError("noise and draws are exclusive")
    if table.dtype != torch.uint8 or table.numel() % RANDN_DRAW_BYTES or not table.is_contiguous():
        raise ValueError("draws: a contiguous uint8 table of whole pp_randn_draw entries")
    return N.ptr(table), table.numel() // RANDN_DRAW_BYTES


def cfg_ddim_desc(*, eps, eps_fp32, eps_ld, latents, coef, step_idx, advance_step, noise,
                  guidance_scale, do_cfg, batch, hw, next_in=None, next_c=0, n_copies=0,
                  extra=None, extra_c=0, guidance_from_coef=False, extra_per_copy=False, blend_x0=None,
                  blend_mask=None, blend_noise=None, draws=None) -> Desc:
    """pp_cfg_ddim_step (include/powerpaint_b200.h); `draws`: a device uint8 table of pp_randn_draw entries
    (`randn_draw_bytes`), the variance noise drawn in the kernel (exclusive with `noise`)"""
    d = N.CfgDdimDesc()
    d.eps, d.eps_fp32, d.eps_ld = N.ptr(eps), 1 if eps_fp32 else 0, eps_ld
    d.latents, d.coef, d.step_idx = N.ptr(latents), N.ptr(coef), N.ptr(step_idx)
    d.advance_step = 1 if advance_step else 0
    d.noise = N.ptr(noise)
    d.guidance_scale, d.do_cfg = guidance_scale, 1 if do_cfg else 0
    d.batch, d.hw = batch, hw
    d.next_in, d.next_c, d.n_copies = N.ptr(next_in), next_c, n_copies
    d.extra, d.extra_c = N.ptr(extra), extra_c
    d.guidance_from_coef = 1 if guidance_from_coef else 0
    d.extra_per_copy = 1 if extra_per_copy else 0
    d.blend_x0, d.blend_mask, d.blend_noise = N.ptr(blend_x0), N.ptr(blend_mask), N.ptr(blend_noise)
    d.draws, d.n_draws = _draws(draws, noise)
    return Desc("cfg_ddim", d, (eps, latents, coef, step_idx, noise, next_in, extra, blend_x0, blend_mask, blend_noise,
                                draws))


def unipc_desc(*, eps, eps_fp32, eps_ld, latents, last_sample, m1, m2, coef, ucoef, step_idx, advance_step, do_cfg,
               batch, hw, next_in=None, next_c=0, n_copies=0) -> Desc:
    d = N.UniPCDesc()
    d.eps, d.eps_fp32, d.eps_ld = N.ptr(eps), 1 if eps_fp32 else 0, eps_ld
    d.latents, d.last_sample, d.m1, d.m2 = N.ptr(latents), N.ptr(last_sample), N.ptr(m1), N.ptr(m2)
    d.coef, d.ucoef, d.step_idx = N.ptr(coef), N.ptr(ucoef), N.ptr(step_idx)
    d.advance_step, d.do_cfg = 1 if advance_step else 0, 1 if do_cfg else 0
    d.batch, d.hw = batch, hw
    d.next_in, d.next_c, d.n_copies = N.ptr(next_in), next_c, n_copies
    return Desc("unipc", d, (eps, latents, last_sample, m1, m2, coef, ucoef, step_idx, next_in))


def solver_desc(*, eps, eps_fp32, eps_ld, latents, m1, coef, scoef, step_idx, advance_step, do_cfg, batch, hw,
                noise=None, next_in=None, next_c=0, n_copies=0, draws=None) -> Desc:
    """pp_solver_step (include/powerpaint_b200.h): CFG + one folded DPM-Solver++ / Euler / Euler-ancestral step;
    `draws` as in `cfg_ddim_desc`"""
    d = N.SolverDesc()
    d.eps, d.eps_fp32, d.eps_ld = N.ptr(eps), 1 if eps_fp32 else 0, eps_ld
    d.latents, d.m1, d.noise = N.ptr(latents), N.ptr(m1), N.ptr(noise)
    d.coef, d.scoef, d.step_idx = N.ptr(coef), N.ptr(scoef), N.ptr(step_idx)
    d.advance_step, d.do_cfg = 1 if advance_step else 0, 1 if do_cfg else 0
    d.batch, d.hw = batch, hw
    d.next_in, d.next_c, d.n_copies = N.ptr(next_in), next_c, n_copies
    d.draws, d.n_draws = _draws(draws, noise)
    return Desc("solver", d, (eps, latents, m1, noise, coef, scoef, step_idx, next_in, draws))


def plms_desc(*, eps, eps_fp32, eps_ld, latents, cur_sample, ets, coef, pcoef, step_idx, advance_step, do_cfg,
              batch, hw, next_in=None, next_c=0, n_copies=0, blend_x0=None, blend_mask=None,
              blend_noise=None) -> Desc:
    """pp_plms_step (include/powerpaint_b200.h): CFG + one folded PNDM (PLMS) step + optional 4-channel blend;
    `ets` is the [3, batch, hw, 4] fp32 history ring"""
    d = N.PlmsDesc()
    d.eps, d.eps_fp32, d.eps_ld = N.ptr(eps), 1 if eps_fp32 else 0, eps_ld
    d.latents, d.cur_sample, d.ets = N.ptr(latents), N.ptr(cur_sample), N.ptr(ets)
    d.coef, d.pcoef, d.step_idx = N.ptr(coef), N.ptr(pcoef), N.ptr(step_idx)
    d.advance_step, d.do_cfg = 1 if advance_step else 0, 1 if do_cfg else 0
    d.batch, d.hw = batch, hw
    d.next_in, d.next_c, d.n_copies = N.ptr(next_in), next_c, n_copies
    d.blend_x0, d.blend_mask, d.blend_noise = N.ptr(blend_x0), N.ptr(blend_mask), N.ptr(blend_noise)
    return Desc("plms", d, (eps, latents, cur_sample, ets, coef, pcoef, step_idx, next_in, blend_x0, blend_mask,
                            blend_noise))


def _tile_view(t: torch.Tensor, name: str):
    """fp32 [batch, h, w, channels] with every sample contiguous (samples may sit any stride apart)"""
    if t.dtype != torch.float32 or t.dim() != 4 or not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA fp32 [batch, h, w, channels] tensor")
    _, h, w, c = t.shape
    if t.stride()[1:] != (w * c, c, 1):
        raise ValueError(f"{name}: each sample must be contiguous")
    return t.shape


def tile_blend_desc(b: torch.Tensor, av: Optional[torch.Tensor], ah: Optional[torch.Tensor], e_v: int,
                    e_h: int) -> Desc:
    """In-place blend_v (with av, the tile above, over e_v rows) then blend_h (with ah, the tile to the left, over
    e_h columns) of the fp32 tile b [batch, h, w, channels] (include/powerpaint_b200.h, pp_tile_blend_desc)"""
    nb, bh, bw, c = _tile_view(b, "b")
    d = N.TileBlendDesc()
    d.b, d.b_stride, d.batch, d.channels, d.b_h, d.b_w = N.ptr(b), b.stride(0), nb, c, bh, bw
    d.e_v, d.e_h = e_v, e_h
    if e_v:
        s = _tile_view(av, "av")
        if (s[0], s[2], s[3]) != (nb, bw, c):
            raise ValueError(f"av {tuple(s)} does not sit above b {tuple(b.shape)}")
        d.av, d.av_stride, d.av_h = N.ptr(av), av.stride(0), s[1]
    if e_h:
        s = _tile_view(ah, "ah")
        if (s[0], s[1], s[3]) != (nb, bh, c):
            raise ValueError(f"ah {tuple(s)} does not sit left of b {tuple(b.shape)}")
        d.ah, d.ah_stride, d.ah_w = N.ptr(ah), ah.stride(0), s[2]
    return Desc("tile_blend", d, (b, av, ah))


def pool_broadcast_desc(x: torch.Tensor, out: torch.Tensor, prev: Optional[torch.Tensor] = None) -> Desc:
    """out[s, p, c] = bf16(prev[s, p, c] + mean_p x[s, p, c]) over bf16 NHWC [batch, hw, channels] buffers
    (include/powerpaint_b200.h, pp_pool_broadcast_desc): the global pooling of a side net's residual"""
    for t, name in ((x, "x"), (out, "out"), (prev, "prev")):
        if t is None:
            continue
        if t.dtype != BF16 or t.dim() != 3 or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous CUDA bf16 [batch, hw, channels] tensor")
        if t.shape != x.shape:
            raise ValueError(f"{name} {tuple(t.shape)} does not match x {tuple(x.shape)}")
    d = N.PoolBroadcastDesc()
    d.x, d.prev, d.out = N.ptr(x), N.ptr(prev), N.ptr(out)
    d.batch, d.hw, d.channels = x.shape
    return Desc("pool_broadcast", d, (x, prev, out))


class WindowList:
    """Windows (src_off, dst_off, src_row, dst_row, rows, cols) in elements of src / dst, checked against both
    tensors on the host and uploaded once; `channels` elements are copied per pixel, pixels src_pix / dst_pix
    elements apart (pp_window_copy)."""

    def __init__(self, src: torch.Tensor, dst: torch.Tensor, channels: int, windows, src_pix: Optional[int] = None,
                 dst_pix: Optional[int] = None):
        if src.dtype != dst.dtype or src.dtype not in (BF16, torch.float32):
            raise TypeError("window copy: src and dst must both be bf16 or both fp32")
        if not (src.is_cuda and dst.is_cuda and src.is_contiguous() and dst.is_contiguous()):
            raise ValueError("window copy: src and dst must be contiguous CUDA tensors")
        self.src_pix = src_pix or src.shape[-1]
        self.dst_pix = dst_pix or dst.shape[-1]
        windows = [tuple(int(v) for v in w) for w in windows if w[4] > 0 and w[5] > 0]
        if not windows:
            raise ValueError("window copy: no non-empty window")
        for so, do, sr, dr, rows, cols in windows:
            for off, row, pix, n, what in ((so, sr, self.src_pix, src.numel(), "src"),
                                           (do, dr, self.dst_pix, dst.numel(), "dst")):
                if off < 0 or row < 0 or off + (rows - 1) * row + (cols - 1) * pix + channels > n:
                    raise ValueError(f"window copy: window {(so, do, sr, dr, rows, cols)} leaves {what}")
        arr = (N.Window * len(windows))(*[N.Window(*w) for w in windows])
        self.table = torch.frombuffer(bytearray(arr), dtype=torch.uint8).to(src.device)
        self.src, self.dst, self.channels = src, dst, channels
        self.count = len(windows)
        self.max_pixels = max(w[4] * w[5] for w in windows)

    def args(self):
        return (N.ptr(self.src), N.ptr(self.dst), self.src.element_size(), self.channels, self.src_pix, self.dst_pix,
                N.ptr(self.table), self.count, self.max_pixels)


# --------------------------------------------------------------------------- immediate mode
def window_copy(wl: WindowList) -> None:
    N.check(N.lib().pp_window_copy(*wl.args(), N.current_stream()), "pp_window_copy")


def run(desc: Desc) -> None:
    L = N.lib()
    s = N.current_stream()
    if desc.kind == "gemm":
        N.check(L.pp_gemm_conv(C.byref(desc.c), s), "pp_gemm_conv")
    elif desc.kind == "attn":
        N.check(L.pp_attention(C.byref(desc.c), s), "pp_attention")
    elif desc.kind == "gn":
        N.check(L.pp_group_norm(C.byref(desc.c), s), "pp_group_norm")
    elif desc.kind == "cfg_ddim":
        N.check(L.pp_cfg_ddim_step(C.byref(desc.c), s), "pp_cfg_ddim_step")
    elif desc.kind == "unipc":
        N.check(L.pp_unipc_step(C.byref(desc.c), s), "pp_unipc_step")
    elif desc.kind == "solver":
        N.check(L.pp_solver_step(C.byref(desc.c), s), "pp_solver_step")
    elif desc.kind == "plms":
        N.check(L.pp_plms_step(C.byref(desc.c), s), "pp_plms_step")
    elif desc.kind == "tile_blend":
        N.check(L.pp_tile_blend(C.byref(desc.c), s), "pp_tile_blend")
    elif desc.kind == "pool_broadcast":
        N.check(L.pp_pool_broadcast(C.byref(desc.c), s), "pp_pool_broadcast")
    else:
        raise ValueError(desc.kind)


def layer_norm(x, y, gamma, beta, eps):
    rows = x.numel() // x.shape[-1]
    N.check(N.lib().pp_layer_norm(N.ptr(x), N.ptr(y), N.ptr(gamma), N.ptr(beta), rows, x.shape[-1],
                                  eps, N.current_stream()), "pp_layer_norm")


def upsample2x(x, y):
    nb, h, w, c = x.shape
    N.check(N.lib().pp_upsample2x(N.ptr(x), N.ptr(y), nb, h, w, c, N.current_stream()), "pp_upsample2x")


def upsample_nearest(x, y):
    """F.interpolate(size=y.shape[1:3], mode="nearest") on NHWC bf16"""
    nb, h, w, c = x.shape
    N.check(N.lib().pp_upsample_nearest(N.ptr(x), N.ptr(y), nb, h, w, c, y.shape[1], y.shape[2],
                                        N.current_stream()), "pp_upsample_nearest")


def add(a, b, y):
    N.check(N.lib().pp_add(N.ptr(a), N.ptr(b), N.ptr(y), a.numel(), N.current_stream()), "pp_add")


def softmax_rows(s: torch.Tensor, p: torch.Tensor):
    """p = softmax(s, dim=-1): fp32 [rows, cols] -> bf16 [rows, cols]"""
    rows, cols = s.shape
    N.check(N.lib().pp_softmax_rows(N.ptr(s), N.ptr(p), rows, cols, s.stride(0), p.stride(0), N.current_stream()),
            "pp_softmax_rows")


def image_preprocess_u8(image: torch.Tensor, mask: Optional[torch.Tensor], c_pad: int = 8, divisor: float = 127.5,
                        shift: float = -1.0) -> torch.Tensor:
    """uint8 NCHW image (+ uint8 / fp32 [n,1,h,w] mask: the hole is zeroed) -> bf16 NHWC [n, h*w, c_pad]"""
    _req(image, torch.uint8, "image")
    nb, c, h, w = image.shape
    if c != 3:
        raise ValueError("image must have 3 channels")
    mode = 0
    if mask is not None:
        if tuple(mask.shape) != (nb, 1, h, w) or not mask.is_contiguous() or not mask.is_cuda:
            raise ValueError("mask must be a contiguous CUDA [n, 1, h, w] tensor")
        mode = 1 if mask.dtype == torch.uint8 else 2
        if mode == 2 and mask.dtype != torch.float32:
            raise TypeError("mask must be uint8 or float32")
    out = torch.empty(nb, h * w, c_pad, dtype=BF16, device=image.device)
    N.check(N.lib().pp_image_preprocess_u8(N.ptr(image), N.ptr(mask), mode, N.ptr(out), nb, h * w, c_pad, divisor, shift,
                                           N.current_stream()), "pp_image_preprocess_u8")
    return out


def image_postprocess(x: torch.Tensor, nb: int, h: int, w: int, *, uint8: bool):
    """decoded NHWC image [nb, h*w, c_ld] -> uint8 NHWC [nb,h,w,3] (uint8=True) or fp32 NCHW [nb,3,h,w] in [0,1]"""
    c_ld = x.shape[-1]
    if uint8:
        out = torch.empty(nb, h, w, 3, dtype=torch.uint8, device=x.device)
        a, b = N.ptr(out), None
    else:
        out = torch.empty(nb, 3, h, w, dtype=torch.float32, device=x.device)
        a, b = None, N.ptr(out)
    N.check(N.lib().pp_image_postprocess(N.ptr(x), 1 if x.dtype == torch.float32 else 0, c_ld, a, b, nb, h * w,
                                         N.current_stream()), "pp_image_postprocess")
    return out


def time_embed(timesteps, out, step_idx=None):
    batch, dim = out.shape
    N.check(N.lib().pp_time_embed(N.ptr(timesteps), N.ptr(step_idx), N.ptr(out), batch, dim,
                                  N.current_stream()), "pp_time_embed")


def nchw_to_nhwc(x: torch.Tensor, c_pad: Optional[int] = None) -> torch.Tensor:
    """fp32 NCHW -> bf16 NHWC (channels zero-padded to c_pad)."""
    _req(x, torch.float32, "x")
    nb, c, h, w = x.shape
    c_pad = c_pad or c
    y = torch.empty(nb, h, w, c_pad, dtype=BF16, device=x.device)
    N.check(N.lib().pp_nchw_to_nhwc(N.ptr(x), N.ptr(y), nb, c, h * w, c_pad, N.current_stream()),
            "pp_nchw_to_nhwc")
    return y


def nhwc_to_nchw(x: torch.Tensor, c: Optional[int] = None) -> torch.Tensor:
    """bf16/fp32 NHWC [nb, h, w, c_ld] -> fp32 NCHW [nb, c, h, w]."""
    nb, h, w, c_ld = x.shape
    c = c or c_ld
    y = torch.empty(nb, c, h, w, dtype=torch.float32, device=x.device)
    N.check(N.lib().pp_nhwc_to_nchw(N.ptr(x), 1 if x.dtype == torch.float32 else 0, N.ptr(y), nb, c,
                                    h * w, c_ld, N.current_stream()), "pp_nhwc_to_nchw")
    return y


def nhwc_fp32_from_nchw(x: torch.Tensor) -> torch.Tensor:
    """4-channel latents NCHW -> fp32 NHWC [nb, h*w, c] (boundary plumbing; 64 KB per image)"""
    nb, c, h, w = x.shape
    return x.float().permute(0, 2, 3, 1).contiguous().view(nb, h * w, c)


def nchw_from_nhwc_fp32(x: torch.Tensor, h: int, w: int) -> torch.Tensor:
    nb, hw, c = x.shape
    return x.view(nb, h, w, c).permute(0, 3, 1, 2).contiguous()


# --------------------------------------------------------------------------- programs
class Program:
    """A recorded op list (pp_program). Keeps every referenced tensor alive."""

    def __init__(self):
        self._h = N.vp()
        N.check(N.lib().pp_program_create(C.byref(self._h)), "pp_program_create")
        self._keep = []
        self.labels = []  # one short label per recorded op (diagnostics: `run_range`)
        self._graph = False

    def __del__(self):
        try:
            if self._h:
                N.lib().pp_program_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add(self, desc: Desc) -> None:
        L = N.lib()
        fn = {"gemm": L.pp_program_add_gemm, "attn": L.pp_program_add_attention,
              "gn": L.pp_program_add_group_norm, "cfg_ddim": L.pp_program_add_cfg_ddim,
              "unipc": L.pp_program_add_unipc, "tile_blend": L.pp_program_add_tile_blend,
              "solver": L.pp_program_add_solver_step, "pool_broadcast": L.pp_program_add_pool_broadcast,
              "plms": L.pp_program_add_plms_step}[desc.kind]
        N.check(fn(self._h, C.byref(desc.c)), f"pp_program_add_{desc.kind}")
        self._keep.append(desc.keep)
        self.labels.append(desc.kind)

    def add_layer_norm(self, x, y, gamma, beta, rows, c, eps):
        N.check(N.lib().pp_program_add_layer_norm(self._h, N.ptr(x), N.ptr(y), N.ptr(gamma), N.ptr(beta),
                                                  rows, c, eps), "pp_program_add_layer_norm")
        self._keep.append((x, y, gamma, beta))
        self.labels.append("layer_norm")

    def add_upsample2x(self, x, y, nb, h, w, c):
        N.check(N.lib().pp_program_add_upsample2x(self._h, N.ptr(x), N.ptr(y), nb, h, w, c),
                "pp_program_add_upsample2x")
        self._keep.append((x, y))
        self.labels.append("upsample2x")

    def add_upsample_nearest(self, x, y, nb, h, w, c, ho, wo):
        N.check(N.lib().pp_program_add_upsample_nearest(self._h, N.ptr(x), N.ptr(y), nb, h, w, c, ho, wo),
                "pp_program_add_upsample_nearest")
        self._keep.append((x, y))
        self.labels.append("upsample_nearest")

    def add_softmax_rows(self, s, p, rows, cols, ld_s, ld_p):
        N.check(N.lib().pp_program_add_softmax_rows(self._h, N.ptr(s), N.ptr(p), rows, cols, ld_s, ld_p),
                "pp_program_add_softmax_rows")
        self._keep.append((s, p))
        self.labels.append("softmax_rows")

    def add_window_copy(self, wl: WindowList):
        N.check(N.lib().pp_program_add_window_copy(self._h, *wl.args()), "pp_program_add_window_copy")
        self._keep.append(wl)
        self.labels.append("window_copy")

    def add_embed_gather(self, idx, base, ext, pos, out, rows, vocab, seq, dim):
        N.check(N.lib().pp_program_add_embed_gather(self._h, N.ptr(idx), N.ptr(base), N.ptr(ext), N.ptr(pos), N.ptr(out),
                                                    rows, vocab, seq, dim), "pp_program_add_embed_gather")
        self._keep.append((idx, base, ext, pos, out))
        self.labels.append("embed_gather")

    def add_causal_attention_small(self, qkv, out, batch, seq, heads, d, scale):
        N.check(N.lib().pp_program_add_causal_attention_small(self._h, N.ptr(qkv), N.ptr(out), batch, seq, heads, d,
                                                              scale), "pp_program_add_causal_attention_small")
        self._keep.append((qkv, out))
        self.labels.append("causal_attention_small")

    def add_add(self, a, b, y, n):
        N.check(N.lib().pp_program_add_add(self._h, N.ptr(a), N.ptr(b), N.ptr(y), n), "pp_program_add_add")
        self._keep.append((a, b, y))
        self.labels.append("add")

    def add_time_embed(self, timesteps, step_idx, out, batch, dim):
        N.check(N.lib().pp_program_add_time_embed(self._h, N.ptr(timesteps), N.ptr(step_idx), N.ptr(out),
                                                  batch, dim), "pp_program_add_time_embed")
        self._keep.append((timesteps, step_idx, out))
        self.labels.append("time_embed")

    def add_memset(self, t: torch.Tensor):
        N.check(N.lib().pp_program_add_memset(self._h, N.ptr(t), t.numel() * t.element_size()),
                "pp_program_add_memset")
        self._keep.append((t,))
        self.labels.append("memset")

    @property
    def num_ops(self) -> int:
        return N.lib().pp_program_num_ops(self._h)

    @property
    def num_launches(self) -> int:
        return N.lib().pp_program_num_launches(self._h)

    def run(self) -> None:
        N.check(N.lib().pp_program_run(self._h, N.current_stream()), "pp_program_run")

    def run_range(self, first: int, count: int) -> None:
        """diagnostic: replay ops [first, first + count) as plain launches"""
        N.check(N.lib().pp_program_run_range(self._h, first, count, N.current_stream()), "pp_program_run_range")

    def build_graph(self) -> None:
        """capture the recorded launches into a CUDA graph. Capture does not execute anything and cannot run on the
        legacy default stream, so it always happens on a private stream; the graph is later launched on whatever
        stream is current."""
        cur = torch.cuda.current_stream()
        cap = torch.cuda.Stream(device=cur.device)
        cap.wait_stream(cur)
        with torch.cuda.stream(cap):
            N.check(N.lib().pp_program_graph_build(self._h, cap.cuda_stream), "pp_program_graph_build")
        cur.wait_stream(cap)
        self._graph = True

    def launch(self) -> None:
        """Replay: CUDA graph if built, plain launches otherwise."""
        if self._graph:
            N.check(N.lib().pp_program_graph_launch(self._h, N.current_stream()), "pp_program_graph_launch")
        else:
            self.run()
