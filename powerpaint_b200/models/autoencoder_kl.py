"""AutoencoderKL (SD-1.5 VAE) on the repo's CUDA kernels — SURVEY.md §8f row 1.

Drop-in for the diffusers class the reference pipelines inject (`vae.encode(x).latent_dist.sample(generator)`,
`vae.decode(z, return_dict=False)[0]`, `vae.config.scaling_factor`; call sites `_encode_vae_image`
powerpaint/pipelines/pipeline_PowerPaint.py:657-669, decode :1051; pipeline_PowerPaint_Brushnet_CA.py:1338-1341,
:1476) with diffusers state-dict names, so `vae/diffusion_pytorch_model.safetensors` loads unchanged.

`encode` / `decode` replay a recorded `pp_program` (CUDA graph) of `VaeEngine`:

  reference (diffusers AutoencoderKL)                  here
  ---------------------------------------------------- ----------------------------------------------------
  ResnetBlock2D(temb=None): GN(eps 1e-6)+SiLU+conv x2   pp_group_norm (statistics from the producing conv's
                                                        epilogue) -> implicit-GEMM 3x3 conv, shortcut as res1
  Downsample2D(padding=0): F.pad(0,1,0,1) + conv s2     PP_A_CONV3X3_S2P0 (the pad is TMA's out-of-bounds zero)
  Upsample2D: nearest 2x + conv                         pp_upsample_nearest + conv
  mid-block Attention, 1 head x 512 channels            to_q|to_k GEMM + V^T GEMM, then per sample
                                                        S = QK^T (fp32) -> pp_softmax_rows -> O = PV, to_out(+res)
                                                        (O in chains of 2048-key GEMMs above 4096 keys)
  conv_out -> quant_conv (1x1)                          folded on the host into ONE 3x3 conv (exact: both linear)
  post_quant_conv (1x1) -> conv_in                      1x1 GEMM, then conv (not folded: the bias meets zero padding)

There is no CPU path: parameters must live on a CUDA device (the torch restatement used as the checker is
`oracle/vae.py`).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Optional, Tuple

import torch

from .. import _native as N
from .. import ops
from ..config import Config
from ..engine import BF16, Plan, Pool, Recorder, _ceil
from ..loading import rename_deprecated_vae_attention
from .base import DiffusersModel


# --------------------------------------------------------------------------- parameter layout
def vae_param_shapes(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512),
                     layers_per_block=2) -> "OrderedDict[str, Tuple[int, ...]]":
    d: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    boc = tuple(block_out_channels)

    def conv(name, cout, cin, k):
        d[name + ".weight"] = (cout, cin, k, k)
        d[name + ".bias"] = (cout,)

    def norm(name, c):
        d[name + ".weight"] = (c,)
        d[name + ".bias"] = (c,)

    def lin(name, cout, cin):
        d[name + ".weight"] = (cout, cin)
        d[name + ".bias"] = (cout,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    def mid(p, c):
        a = p + ".attentions.0"
        norm(a + ".group_norm", c)
        for n in ("to_q", "to_k", "to_v"):
            lin(f"{a}.{n}", c, c)
        lin(a + ".to_out.0", c, c)
        resnet(p + ".resnets.0", c, c)
        resnet(p + ".resnets.1", c, c)

    conv("encoder.conv_in", boc[0], in_channels, 3)
    c = boc[0]
    for i, co in enumerate(boc):
        for j in range(layers_per_block):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", c if j == 0 else co, co)
        if i != len(boc) - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", co, co, 3)
        c = co
    mid("encoder.mid_block", c)
    norm("encoder.conv_norm_out", c)
    conv("encoder.conv_out", 2 * latent_channels, c, 3)
    rev = list(reversed(boc))
    conv("decoder.conv_in", rev[0], latent_channels, 3)
    mid("decoder.mid_block", rev[0])
    c = rev[0]
    for i, co in enumerate(rev):
        for j in range(layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", c if j == 0 else co, co)
        if i != len(boc) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", co, co, 3)
        c = co
    norm("decoder.conv_norm_out", c)
    conv("decoder.conv_out", out_channels, c, 3)
    conv("quant_conv", 2 * latent_channels, 2 * latent_channels, 1)
    conv("post_quant_conv", latent_channels, latent_channels, 1)
    return d


# --------------------------------------------------------------------------- tile geometry
# Attention S = QK^T of one image is a [hw, hw] fp32 matrix and pp_softmax_rows takes at most 16384 columns
VAE_MAX_LATENT_PIXELS = 16384
# O = P V sums over all hw keys. The tensor cores' fp32 accumulation error grows with the number of k-steps, and on
# softmax weights (all non-negative) it does not cancel: above PV_K_SINGLE keys the product runs as a chain of GEMMs
# over PV_K_CHUNK keys each, every one adding the fp32 sum of the chunks before it through its row vector
PV_K_SINGLE = 4096
PV_K_CHUNK = 2048


def add_pv_product(prog, p: torch.Tensor, vt: torch.Tensor, out: torch.Tensor,
                   partial: Optional[Tuple[torch.Tensor, torch.Tensor]]) -> None:
    """record out = P V: p bf16 [hw, k_ld], vt bf16 [C, k_ld] (both with every one of the k_ld keys readable), out bf16
    [hw, C]. Above PV_K_SINGLE keys `partial` holds two fp32 [hw, C] buffers the chain's running sums alternate in."""
    hw, k_ld = p.shape
    C = vt.shape[0]
    if k_ld <= PV_K_SINGLE:
        prog.add(ops.gemm_desc(a0=p, c0=k_ld, lda0=k_ld, w=vt, ldb=k_ld, out=out, N_=C, M=hw))
        return
    prev = None
    for j, k0 in enumerate(range(0, k_ld, PV_K_CHUNK)):
        k1 = min(k_ld, k0 + PV_K_CHUNK)
        last = k1 == k_ld
        dst = out if last else partial[j % 2]
        prog.add(ops.gemm_desc(a0=p[:, k0:], c0=k1 - k0, lda0=k_ld, w=vt[:, k0:], ldb=k_ld, out=dst, N_=C, M=hw,
                               rowvec=prev, rows_per_group=1 if prev is not None else 0,
                               rowvec_ld=C if prev is not None else 0, out_fp32=not last))
        prev = dst


@dataclass(frozen=True)
class VaeTile:
    """One tile of diffusers' tiled_encode / tiled_decode loop (row-major order)."""
    row: int
    col: int
    y: int        # origin in the input (image for encode, latent for decode)
    x: int
    h: int        # input extent: the tile slice is clipped at the input's border
    w: int
    out_h: int    # extent of the encoded / decoded tile
    out_w: int
    crop_h: int   # the tile's top-left crop that lands in the output
    crop_w: int
    dst_y: int    # where the crop lands
    dst_x: int
    blend_v: int  # rows blended with the tile above (0: none)
    blend_h: int  # columns blended with the tile to the left (0: none)


@dataclass(frozen=True)
class VaeTileGeometry:
    rows: int
    cols: int
    out_h: int
    out_w: int
    tiles: Tuple[VaeTile, ...]

    def groups(self) -> "OrderedDict[Tuple[int, int], List[int]]":
        """tile indices per input shape (h, w), in row-major order of first appearance"""
        g: "OrderedDict[Tuple[int, int], List[int]]" = OrderedDict()
        for k, t in enumerate(self.tiles):
            g.setdefault((t.h, t.w), []).append(k)
        return g


def vae_tile_geometry(encode: bool, h: int, w: int, tile_sample_min_size: int, tile_latent_min_size: int,
                      tile_overlap_factor: float, scale: int) -> VaeTileGeometry:
    """The tiles of diffusers 0.27 `AutoencoderKL.tiled_encode` (image h x w) or `tiled_decode` (latent h x w):
    origins every int(tile * (1 - f)) input pixels, blend extent int(out_tile * f), crop to out_tile - extent.
    `scale` = 2 ** (len(block_out_channels) - 1): a decoded tile is `scale` times its latent, an encoded tile is
    its image floor-divided by 2 once per downsampler."""
    f = tile_overlap_factor
    if encode:
        tin, tout = tile_sample_min_size, tile_latent_min_size

        def out_size(n):
            return n // scale
    else:
        tin, tout = tile_latent_min_size, tile_sample_min_size

        def out_size(n):
            return n * scale
    overlap = int(tin * (1 - f))
    blend = int(tout * f)
    limit = tout - blend
    if overlap <= 0:
        raise ValueError(f"tile size {tin} with overlap factor {f} gives no tile stride")
    ys, xs = list(range(0, h, overlap)), list(range(0, w, overlap))
    tiles = []
    dst_y = 0
    for r, y in enumerate(ys):
        th = min(tin, h - y)
        oh = out_size(th)
        ch = len(range(oh)[:limit])  # tile[:limit] in Python slice semantics
        dst_x = 0
        for c, x in enumerate(xs):
            tw = min(tin, w - x)
            ow = out_size(tw)
            cw = len(range(ow)[:limit])
            ev = min(out_size(min(tin, h - ys[r - 1])), oh, blend) if r > 0 else 0
            eh = min(out_size(min(tin, w - xs[c - 1])), ow, blend) if c > 0 else 0
            tiles.append(VaeTile(r, c, y, x, th, tw, oh, ow, ch, cw, dst_y, dst_x, max(ev, 0), max(eh, 0)))
            dst_x += cw
        dst_y += ch
    return VaeTileGeometry(len(ys), len(xs), dst_y, dst_x, tuple(tiles))


# --------------------------------------------------------------------------- engine
class VaeEngine(Recorder):
    """Records VAE encode / decode as `pp_program`s over the conv / GroupNorm / GEMM kernels of the denoising
    step (buffer recycling, epilogue GroupNorm statistics, weight packing and the resnet are `Recorder`'s)."""

    GN_EPS = 1e-6

    # ---- blocks
    def _vae_attention(self, plan, prog, name, x, nb, h, w):
        """one head over all C channels: softmax(q k^T / sqrt(C)) v, then to_out + residual"""
        hw = h * w
        M = nb * hw
        C = x.shape[-1]
        hw_ld = _ceil(hw, 8)
        g = self._gn(plan, prog, x, None, nb, hw, name + ".group_norm", self.GN_EPS, False)
        wqk = self._cached("vqk:" + name, lambda: torch.cat(
            [self._raw(name + ".to_q.weight"), self._raw(name + ".to_k.weight")], 0).to(BF16).contiguous())
        bqk = self._cached("vqkb:" + name, lambda: torch.cat(
            [self._raw(name + ".to_q.bias"), self._raw(name + ".to_k.bias")], 0).contiguous())
        qk = self._linear(plan, prog, g, M, None, 2 * C, w=wqk, bias=bqk)
        # V^T [nb, C, hw_ld] and P [hw, hw_ld]: the kernels never write the pad columns, which the PV product reads,
        # so a recycled block is cleared first
        vt = plan.pool.buf(nb, C, hw_ld)
        pm = plan.pool.buf(hw, hw_ld)
        if hw_ld != hw:
            prog.add_memset(vt)
            prog.add_memset(pm)
        sm = plan.pool.buf(hw, hw, dtype=torch.float32)
        prog.add(ops.gemm_desc(a0=g, w=self.w_linear(name + ".to_v"), out=vt, N_=C, M=M, bias=self.vec(name + ".to_v.bias"),
                               epilogue=N.PP_EPI_TRANSPOSED, t_rows=hw, t_ld=hw_ld))
        plan.pool.free(g)
        o = plan.pool.buf(M, C)
        partial = None
        if hw_ld > PV_K_SINGLE:
            partial = (plan.pool.buf(hw, C, dtype=torch.float32), plan.pool.buf(hw, C, dtype=torch.float32))
        scale = 1.0 / math.sqrt(C)
        for b in range(nb):
            rows = qk[b * hw:(b + 1) * hw]
            prog.add(ops.gemm_desc(a0=rows, c0=C, lda0=2 * C, w=rows[:, C:], ldb=2 * C, out=sm, N_=hw, M=hw, alpha=scale,
                                   out_fp32=True))
            prog.add_softmax_rows(sm, pm, hw, hw, hw, hw_ld)
            add_pv_product(prog, pm, vt[b], o[b * hw:(b + 1) * hw], partial)
        plan.pool.free(qk, vt, pm, sm, *(partial or ()))
        out = self._linear(plan, prog, o, M, name + ".to_out.0", C, bias=self.vec(name + ".to_out.0.bias"), res1=x,
                           stats_hw=hw)
        plan.pool.free(o)
        return out

    def _vae_mid(self, plan, prog, name, x, nb, h, w):
        C = x.shape[-1]
        a = self._resnet(plan, prog, name + ".resnets.0", x, None, nb, h, w, C, eps=self.GN_EPS)
        plan.pool.free(x)
        b = self._vae_attention(plan, prog, name + ".attentions.0", a, nb, h, w)
        plan.pool.free(a)
        c = self._resnet(plan, prog, name + ".resnets.1", b, None, nb, h, w, C, eps=self.GN_EPS)
        plan.pool.free(b)
        return c

    def _check_latent(self, h: int, w: int, what: str):
        if h * w > VAE_MAX_LATENT_PIXELS:
            raise RuntimeError(
                f"VAE {what}: a {h}x{w} latent has {h * w} pixels, above the {VAE_MAX_LATENT_PIXELS} the VAE's "
                "mid-block attention supports per image (1048576 image pixels); call enable_vae_tiling() "
                "(AutoencoderKL.enable_tiling()) to encode / decode larger images tile by tile")

    def _latent_hw(self, H: int, W: int):
        for _ in range(len(self.cfg.block_out_channels) - 1):
            H, W = H // 2, W // 2
        return H, W

    # ---- encoder
    def encode_plan(self, nb: int, H: int, W: int) -> Plan:
        self._check_latent(*self._latent_hw(H, W), "encode")
        return self._plan(("enc", nb, H, W), lambda: self._build_encode(nb, H, W), graph=True)

    def _build_encode(self, nb, H, W, plan: Optional[Plan] = None, x_in: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None) -> Plan:
        """records the encoder into `plan` (a new one by default), reading bf16 NHWC x_in [nb, H*W, 8] and writing
        the fp32 moments [nb, h*w, 2 * latent_channels] to `out`"""
        cfg = self.cfg
        boc = cfg.block_out_channels
        self._check_latent(*self._latent_hw(H, W), "encode")
        plan = plan or Plan(Pool(self.device))
        prog = plan.program
        if x_in is None:
            x_in = torch.zeros(nb, H * W, 8, dtype=BF16, device=self.device)
            plan.inputs["x"] = x_in
        h, w = H, W
        cur = self._conv3(plan, prog, x_in, nb, h, w, "encoder.conv_in", boc[0], pad_in=8, stats=True)
        for i, co in enumerate(boc):
            for j in range(cfg.layers_per_block):
                nxt = self._resnet(plan, prog, f"encoder.down_blocks.{i}.resnets.{j}", cur, None, nb, h, w, co,
                                   eps=self.GN_EPS)
                plan.pool.free(cur)
                cur = nxt
            if i != len(boc) - 1:
                if h < 2 or w < 2:
                    raise ValueError(f"image {H}x{W} is too small for the VAE encoder")
                nxt = self._conv3(plan, prog, cur, nb, h, w, f"encoder.down_blocks.{i}.downsamplers.0.conv", co,
                                  a_mode=N.PP_A_CONV3X3_S2P0, stats=True)
                plan.pool.free(cur)
                cur = nxt
                h, w = h // 2, w // 2
        cur = self._vae_mid(plan, prog, "encoder.mid_block", cur, nb, h, w)
        gno = self._gn(plan, prog, cur, None, nb, h * w, "encoder.conv_norm_out", self.GN_EPS, True)
        plan.pool.free(cur)
        # conv_out followed by the 1x1 quant_conv: both linear, folded into one conv on the host (fp32)
        lc2 = 2 * cfg.latent_channels

        def folded():
            wq = self._raw("quant_conv.weight").reshape(lc2, lc2)
            wc = self._raw("encoder.conv_out.weight")
            wf = torch.einsum("oc,cikl->oikl", wq, wc)
            bf = wq @ self._raw("encoder.conv_out.bias") + self._raw("quant_conv.bias")
            return ops.pack_conv3x3_weight(wf), bf.contiguous()
        wf, bf = self._cached("enc_out_folded", folded)
        moments = out if out is not None else torch.empty(nb, h * w, lc2, dtype=torch.float32, device=self.device)
        prog.add(ops.gemm_desc(a0=gno, w=wf, out=moments, N_=lc2, a_mode=N.PP_A_CONV3X3, c0=gno.shape[-1], nb=nb, h=h,
                               w_=w, bias=bf, out_fp32=True))
        plan.pool.free(gno)
        if out is None:
            plan.outputs["moments"] = moments
            plan.outputs["hw"] = (h, w)
        return plan

    # ---- decoder
    def decode_plan(self, nb: int, h: int, w: int) -> Plan:
        self._check_latent(h, w, "decode")
        return self._plan(("dec", nb, h, w), lambda: self._build_decode(nb, h, w), graph=True)

    def _build_decode(self, nb, h, w, plan: Optional[Plan] = None, z_in: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None) -> Plan:
        """records the decoder into `plan` (a new one by default), reading bf16 NHWC z_in [nb, h*w, 8] and writing
        the fp32 image [nb, H*W, 4] (channels 0..2) to `out`"""
        cfg = self.cfg
        rev = list(reversed(cfg.block_out_channels))
        lc = cfg.latent_channels
        self._check_latent(h, w, "decode")
        plan = plan or Plan(Pool(self.device))
        prog = plan.program
        if z_in is None:
            z_in = torch.zeros(nb, h * w, 8, dtype=BF16, device=self.device)
            plan.inputs["z"] = z_in
        # post_quant_conv (1x1, latent -> latent): its own GEMM; channels >= lc of the output stay zero
        zq = torch.zeros(nb, h * w, 8, dtype=BF16, device=self.device)
        wpq = self._cached("pq:w", lambda: torch.nn.functional.pad(
            self._raw("post_quant_conv.weight").reshape(lc, lc), (0, 8 - lc)).to(BF16).contiguous())
        prog.add(ops.gemm_desc(a0=z_in, w=wpq, out=zq, N_=lc, M=nb * h * w, bias=self.vec("post_quant_conv.bias"), ldc=8))
        cur = self._conv3(plan, prog, zq, nb, h, w, "decoder.conv_in", rev[0], pad_in=8, stats=True)
        cur = self._vae_mid(plan, prog, "decoder.mid_block", cur, nb, h, w)
        for i, co in enumerate(rev):
            for j in range(cfg.layers_per_block + 1):
                nxt = self._resnet(plan, prog, f"decoder.up_blocks.{i}.resnets.{j}", cur, None, nb, h, w, co,
                                   eps=self.GN_EPS)
                plan.pool.free(cur)
                cur = nxt
            if i != len(rev) - 1:
                up = plan.pool.buf(nb, 4 * h * w, co)
                prog.add_upsample_nearest(cur, up, nb, h, w, co, 2 * h, 2 * w)
                plan.pool.free(cur)
                h, w = 2 * h, 2 * w
                cur = self._conv3(plan, prog, up, nb, h, w, f"decoder.up_blocks.{i}.upsamplers.0.conv", co, stats=True)
                plan.pool.free(up)
        gno = self._gn(plan, prog, cur, None, nb, h * w, "decoder.conv_norm_out", self.GN_EPS, True)
        plan.pool.free(cur)
        # fp32 image, 4 floats per pixel (3 used): the uint8 conversion must not see a bf16-rounded value
        image = out if out is not None else torch.zeros(nb, h * w, 4, dtype=torch.float32, device=self.device)
        prog.add(ops.gemm_desc(a0=gno, w=self.w_conv3("decoder.conv_out"), out=image, N_=cfg.out_channels,
                               a_mode=N.PP_A_CONV3X3, c0=gno.shape[-1], nb=nb, h=h, w_=w,
                               bias=self.vec("decoder.conv_out.bias"), out_fp32=True, ldc=4))
        plan.pool.free(gno)
        if out is None:
            plan.outputs["image"] = image
            plan.outputs["hw"] = (h, w)
        return plan

    # ---- tiled encode / decode
    # image pixels one recorded encoder / decoder pass covers (four 512^2 tiles, the pixels of one 1024^2 image):
    # the activation pool of a tiled plan is sized by one such pass, whatever the canvas
    TILE_CHUNK_PIXELS = 4 * 512 * 512

    def tiled_plan(self, encode: bool, nb: int, H: int, W: int, geom: VaeTileGeometry, key: tuple) -> Plan:
        return self._plan(("tenc" if encode else "tdec", nb, H, W) + key,
                          lambda: self._build_tiled(encode, nb, H, W, geom), graph=True)

    def _build_tiled(self, encode: bool, nb: int, H: int, W: int, geom: VaeTileGeometry) -> Plan:
        """ONE program over the whole canvas: per tile shape, gather the tiles of every sample out of the canvas and
        run the encoder / decoder on them in chunks of TILE_CHUNK_PIXELS, each writing its slab of an fp32 tile
        store; then blend every tile with its upper and left neighbours in diffusers' row-major order, in place;
        then copy each tile's crop into the output. Every chunk records into the plan's one activation pool."""
        cfg = self.cfg
        plan = Plan(Pool(self.device, best_fit=True))
        prog = plan.program
        C = 2 * cfg.latent_channels if encode else 4
        canvas = plan.pool.tensor(nb, H * W, 8, zero=True)
        out = plan.pool.tensor(nb, geom.out_h * geom.out_w, C, dtype=torch.float32, zero=True)
        plan.inputs["x" if encode else "z"] = canvas
        build = self._build_encode if encode else self._build_decode
        views: Dict[int, torch.Tensor] = {}  # tile -> fp32 [nb, out_h, out_w, C] in its group's store
        assembly = []
        # largest tiles first: with best-fit recycling the smaller passes that follow reuse their blocks
        for (th, tw), idx in sorted(geom.groups().items(), key=lambda g: -g[0][0] * g[0][1]):
            t0 = geom.tiles[idx[0]]
            ohw = t0.out_h * t0.out_w
            store = plan.pool.tensor(len(idx) * nb, ohw, C, dtype=torch.float32, zero=True)
            images = [(k, s) for k in idx for s in range(nb)]  # row r of the store holds images[r]
            per = max(1, self.TILE_CHUNK_PIXELS // (th * tw if encode else ohw))
            for r0 in range(0, len(images), per):
                chunk = images[r0:r0 + per]
                x_in = plan.pool.buf(len(chunk), th * tw, 8)
                gather = [((s * H * W + geom.tiles[k].y * W + geom.tiles[k].x) * 8, m * th * tw * 8, W * 8, tw * 8,
                           th, tw) for m, (k, s) in enumerate(chunk)]
                prog.add_window_copy(ops.WindowList(canvas, x_in, 8, gather))
                plan.pool.restart_gn_arena(prog)
                build(len(chunk), th, tw, plan, x_in, store[r0:r0 + len(chunk)])
                plan.pool.free(x_in)
            crops = []
            for j, k in enumerate(idx):
                t = geom.tiles[k]
                views[k] = store[j * nb:(j + 1) * nb].view(nb, t.out_h, t.out_w, C)
                crops += [((j * nb + s) * ohw * C, (s * geom.out_h * geom.out_w + t.dst_y * geom.out_w + t.dst_x) * C,
                           t.out_w * C, geom.out_w * C, t.crop_h, t.crop_w) for s in range(nb)]
            if any(c[4] and c[5] for c in crops):
                assembly.append(ops.WindowList(store, out, C, crops))
        for k, t in enumerate(geom.tiles):
            if t.blend_v or t.blend_h:
                prog.add(ops.tile_blend_desc(views[k], views[k - geom.cols] if t.blend_v else None,
                                             views[k - 1] if t.blend_h else None, t.blend_v, t.blend_h))
        for wl in assembly:
            prog.add_window_copy(wl)
        plan.outputs["moments" if encode else "image"] = out
        plan.outputs["hw"] = (geom.out_h, geom.out_w)
        return plan


# --------------------------------------------------------------------------- diffusers-facing module
class DiagonalGaussianDistribution:
    def __init__(self, parameters: torch.Tensor):
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        dev = generator.device if generator is not None else self.mean.device
        noise = torch.randn(self.mean.shape, generator=generator, device=dev, dtype=self.mean.dtype)
        return self.mean + self.std * noise.to(self.mean.device)

    def mode(self) -> torch.Tensor:
        return self.mean


class AutoencoderKL(DiffusersModel):
    def __init__(self, in_channels: int = 3, out_channels: int = 3, latent_channels: int = 4,
                 block_out_channels: Tuple[int, ...] = (128, 256, 512, 512), layers_per_block: int = 2,
                 norm_num_groups: int = 32, scaling_factor: float = 0.18215, sample_size: int = 32):
        super().__init__()
        if in_channels != 3 or out_channels != 3 or latent_channels > 4:
            raise NotImplementedError("the kernel path is built for RGB images and <= 4 latent channels (SD VAE)")
        if any(c % 8 for c in block_out_channels):
            raise ValueError("block_out_channels must be multiples of 8")
        self.config = Config(in_channels=in_channels, out_channels=out_channels, latent_channels=latent_channels,
                             block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                             scaling_factor=scaling_factor, norm_num_groups=norm_num_groups, sample_size=sample_size)
        # tiled encode / decode, off by default (diffusers AutoencoderKL.__init__); the tile_* attributes may be set
        self.use_tiling = False
        self.use_slicing = False
        self.tile_sample_min_size = sample_size
        ss = sample_size[0] if isinstance(sample_size, (list, tuple)) else sample_size
        self.tile_latent_min_size = int(ss / (2 ** (len(block_out_channels) - 1)))
        self.tile_overlap_factor = 0.25
        for name, shape in vae_param_shapes(in_channels, out_channels, latent_channels, block_out_channels,
                                            layers_per_block).items():
            self._register(name, torch.zeros(shape))

    def _make_engine(self, state_dict, device) -> VaeEngine:
        return VaeEngine(self.config, state_dict, device)

    # ---- tiling (diffusers AutoencoderKL.enable_tiling: opt-in, it blends tile seams and so changes the result)
    def enable_tiling(self, use_tiling: bool = True):
        """encode / decode images above tile_sample_min_size (latents above tile_latent_min_size) tile by tile"""
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    def tile_geometry(self, encode: bool, h: int, w: int) -> VaeTileGeometry:
        """the tiles tiled_encode (image h x w) / tiled_decode (latent h x w) runs with the current tile_* settings"""
        return vae_tile_geometry(encode, h, w, self.tile_sample_min_size, self.tile_latent_min_size,
                                 self.tile_overlap_factor, 2 ** (len(self.config.block_out_channels) - 1))

    def _tiling_key(self):
        return (self.tile_sample_min_size, self.tile_latent_min_size, self.tile_overlap_factor)

    # ---- encode
    @torch.no_grad()
    def _moments(self, x_nhwc: torch.Tensor, nb: int, H: int, W: int, tiled: bool = False) -> torch.Tensor:
        eng = self.engine()
        if tiled:
            plan = eng.tiled_plan(True, nb, H, W, self.tile_geometry(True, H, W), self._tiling_key())
        else:
            plan = eng.encode_plan(nb, H, W)
        plan.inputs["x"].copy_(x_nhwc.view_as(plan.inputs["x"]))
        plan.program.launch()
        h, w = plan.outputs["hw"]
        return ops.nhwc_to_nchw(plan.outputs["moments"].view(nb, h, w, -1)).to(self._out_dtype)

    def _tile_image(self, H: int, W: int) -> bool:
        return self.use_tiling and (W > self.tile_sample_min_size or H > self.tile_sample_min_size)

    def _tile_latent(self, h: int, w: int) -> bool:
        return self.use_tiling and (w > self.tile_latent_min_size or h > self.tile_latent_min_size)

    @torch.no_grad()
    def _encode(self, x: torch.Tensor, return_dict: bool, tiled: bool):
        nb, c, H, W = x.shape
        self.engine()  # raises on CPU parameters: there is no CPU path
        with torch.cuda.device(self.device):
            xn = ops.nchw_to_nhwc(x.to(self.device).float().contiguous(), 8)
            dist = DiagonalGaussianDistribution(self._moments(xn, nb, H, W, tiled))
        return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [B,3,H,W] in [-1,1] -> `.latent_dist` (DiagonalGaussianDistribution over [B,8,H/8,W/8] moments);
        tiled (`tiled_encode`) when tiling is on and a side exceeds tile_sample_min_size"""
        return self._encode(x, return_dict, self._tile_image(x.shape[-2], x.shape[-1]))

    def tiled_encode(self, x: torch.Tensor, return_dict: bool = True):
        """diffusers tiled_encode: overlapping tiles through the encoder, their moments blended at the seams"""
        return self._encode(x, return_dict, True)

    @torch.no_grad()
    def encode_uint8(self, image_u8: torch.Tensor, mask: Optional[torch.Tensor] = None) -> DiagonalGaussianDistribution:
        """uint8 NCHW image (hole zeroed where mask >= 0.5) straight into the encoder: `image / 127.5 - 1`,
        binarise, `image * (mask < 0.5)` (pipeline_PowerPaint.py:123-147) and the layout change are one kernel
        (over the whole canvas; a tiled encode gathers its tiles from its output)"""
        nb, c, H, W = image_u8.shape
        self.engine()
        with torch.cuda.device(self.device):
            xn = ops.image_preprocess_u8(image_u8.contiguous(), mask, c_pad=8)
            return DiagonalGaussianDistribution(self._moments(xn, nb, H, W, self._tile_image(H, W)))

    # ---- decode
    @torch.no_grad()
    def _decode_nhwc(self, z: torch.Tensor, tiled: bool):
        nb, c, h, w = z.shape
        eng = self.engine()
        if tiled:
            plan = eng.tiled_plan(False, nb, h, w, self.tile_geometry(False, h, w), self._tiling_key())
        else:
            plan = eng.decode_plan(nb, h, w)
        zi = plan.inputs["z"]
        zi.copy_(ops.nchw_to_nhwc(z.to(self.device).float().contiguous(), 8).view_as(zi))
        plan.program.launch()
        H, W = plan.outputs["hw"]
        return plan.outputs["image"], nb, H, W

    @torch.no_grad()
    def _decode(self, z: torch.Tensor, return_dict: bool, tiled: bool):
        self.engine()
        with torch.cuda.device(self.device):
            img, nb, H, W = self._decode_nhwc(z, tiled)
            out = ops.nhwc_to_nchw(img.view(nb, H, W, 4), 3).to(self._out_dtype)
        return SimpleNamespace(sample=out) if return_dict else (out,)

    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """tiled (`tiled_decode`) when tiling is on and a latent side exceeds tile_latent_min_size"""
        return self._decode(z, return_dict, self._tile_latent(z.shape[-2], z.shape[-1]))

    def tiled_decode(self, z: torch.Tensor, return_dict: bool = True):
        """diffusers tiled_decode: overlapping latent tiles through the decoder, blended at the seams"""
        return self._decode(z, return_dict, True)

    @torch.no_grad()
    def decode_postprocessed(self, z: torch.Tensor, uint8: bool) -> torch.Tensor:
        """decode + `VaeImageProcessor.postprocess` denormalisation in one pass over the image:
        uint8 NHWC [B,H,W,3] (what "pil" output is built from) or fp32 NCHW in [0,1] ("pt" / "np");
        tiled like `decode`"""
        self.engine()
        with torch.cuda.device(self.device):
            img, nb, H, W = self._decode_nhwc(z, self._tile_latent(z.shape[-2], z.shape[-1]))
            return ops.image_postprocess(img, nb, H, W, uint8=uint8)

    # ---- checkpoint directories in the diffusers layout (`<root>/vae`)
    @classmethod
    def from_config(cls, config: dict) -> "AutoencoderKL":
        if config.get("act_fn", "silu") != "silu":
            raise NotImplementedError(f"config.act_fn = {config['act_fn']!r}: the SD VAE uses silu")
        keys = ("in_channels", "out_channels", "latent_channels", "block_out_channels", "layers_per_block",
                "norm_num_groups", "scaling_factor", "sample_size")
        return cls(**{k: (tuple(config[k]) if isinstance(config[k], list) else config[k]) for k in keys if k in config})

    def _diffusers_config(self) -> dict:
        cfg = {"_class_name": "AutoencoderKL", "_diffusers_version": "0.27.0", "act_fn": "silu"}
        cfg.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in vars(self.config).items()})
        return cfg

    # older VAE checkpoints name the attention parameters query / key / value / proj_attn: renamed like diffusers does
    _checkpoint_state_dict = staticmethod(rename_deprecated_vae_attention)

    @classmethod
    def synthetic(cls, seed: int = 4321, tiny: bool = False, **kw) -> "AutoencoderKL":
        """deterministic random weights (no checkpoint reachable offline); `tiny` = small widths for tests"""
        if tiny:
            kw.setdefault("block_out_channels", (16, 32, 32, 32))
            kw.setdefault("norm_num_groups", 8)
            kw.setdefault("layers_per_block", 1)
        m = cls(**kw)
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p in m.named_parameters():
                if p.dim() >= 2:
                    p.copy_(torch.randn(p.shape, generator=g) / p[0].numel() ** 0.5)
                elif "norm" in name and name.endswith("weight"):
                    p.fill_(1.0)
                else:
                    p.zero_()
        return m.eval()
