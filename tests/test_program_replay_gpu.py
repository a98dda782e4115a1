"""The recorded programs on their own activations: which buffer each op reads, and whether every buffer survives
intact from its writer to its last reader.

Every op a Program records (a Desc through `add`, a ProgramCall through the other record methods) gets an exact read
and write footprint: a list of (pointer, rows, row bytes, pitch) regions, never a bounding interval, so two producers
writing disjoint columns of one concat buffer do not look like they alias. Side outputs count as writes: the GEMM's
GroupNorm partials, the LayerNorm row records, finals and tickets, split-K workspaces and flags, GroupNorm scratch, and
the step kernels' state, ring slots and step counter.

- Static dataflow (recording only): each plan is recorded twice, with the activation Pool and with a Pool that never
  recycles a freed block. For every byte every op reads, the op that last wrote it must be the same in both recordings
  (the per-step program runs twice in a row, so a block handed on too early inside one step or across the step
  boundary shows up), and a byte nothing wrote before it is read must sit in a plan input or persistent state, never in
  a recycled activation block.
- Replay: the real entry points run with `Program.run` replaced by one `run_range(i, 1)` per op. After every op, no
  byte of the pool, the plan state or the step state outside the op's write footprint may have changed, the split-K
  flags and the row / GroupNorm tickets are back at zero, and every op's outputs equal the fp64 evaluation of its
  contract on the inputs it actually read (snapshotted before the op: the step kernels, pool_broadcast and the GN
  scratch update in place), with the bounds of the census files; the exact ops are compared bit for bit. The weights
  are part of the tracked storage, so an op that writes into one fails at that op.
- A CUDA-graph step equals the op-by-op replay of the same step bit for bit, and two steps on a recycled pool equal
  two steps on a pool that never recycles, bit for bit.
"""
import ctypes
import inspect
import math

import numpy as np
import pytest
import torch

from test_kernel_variants_gpu import (DENOISER_SHAPES, ENGINE_SWITCHES, PROGRAM_RECORD_METHODS, U16, ProgramCall,
                                      _check_row_stats, assert_within, gemm_extents, gemm_got_chunk, gemm_out_geometry,
                                      ref_attention, ref_gemm)
from test_kernels_gpu import U32, _cfg_eps, ref_cfg_ddim, ref_unipc
from test_norm_and_small_kernels_gpu import (check_gn_stats, gn_geometry, gn_truth, gn_y_ref, producer_chain,
                                             ref_causal_attention, ref_layer_norm, ref_softmax, ref_time_embed,
                                             softmax_instance, standalone_chain)

DEV = "cuda"
BF16 = torch.bfloat16


# =========================================================================== footprints
def _p(v):
    """a pointer: ctypes field value, tensor or None"""
    if v is None:
        return 0
    return v.data_ptr() if isinstance(v, torch.Tensor) else int(v)


def _r(ptr, rows, row_bytes=None, pitch=None):
    """one region: `rows` rows of `row_bytes` bytes, `pitch` bytes apart (rows=1: a contiguous run of row_bytes)"""
    if row_bytes is None:
        rows, row_bytes = 1, rows
    ptr = _p(ptr)
    if not ptr or rows <= 0 or row_bytes <= 0:
        return []
    return [(ptr, int(rows), int(row_bytes), int(pitch if pitch is not None and rows > 1 else row_bytes))]


def _pad64(c):
    return (c + 63) // 64 * 64


def fp_gemm(op, step=0):
    """`step`: the value of *alpha_step when the op runs (the side-net scale row it reads)"""
    from powerpaint_b200 import ops as o

    d = op.c
    M = gemm_out_geometry(d)[0]
    R, W = [], []
    for f, (rows, cols, ld, dt) in gemm_extents(d).items():
        el = torch.empty(0, dtype=dt).element_size()
        (W if f in ("out", "out_t") else R).extend(_r(getattr(d, f), rows, cols * el, ld * el))
    R += _r(d.alpha_step, 4)
    if d.alpha_dev:
        R += _r(d.alpha_dev + 4 * (step if d.alpha_step else 0) * d.alpha_stride, 4)
    if d.chan_stats:
        W += _r(d.chan_stats, int(o.gemm_stats_geometry(op).bytes))
    if d.row_stats:
        W += _r(d.row_stats, o.gemm_row_stats_records(op), M * 16, d.row_stats_ld * 16)
        W += _r(d.row_final, M * 8) + _r(d.row_ticket, (M + 127) // 128 * 4)
    if d.splitk_ws:
        nbytes, tiles = o.gemm_splitk_query(op)
        W += _r(d.splitk_ws, nbytes) + _r(d.splitk_flags, tiles * 4)
    return R, W


def gemm_counters(op):
    d = op.c
    M = gemm_out_geometry(d)[0]
    out = []
    if d.row_ticket:
        out += _r(d.row_ticket, (M + 127) // 128 * 4)
    if d.splitk_flags:
        from powerpaint_b200 import ops as o

        out += _r(d.splitk_flags, o.gemm_splitk_query(op)[1] * 4)
    return out


def fp_attn(op):
    d = op.c
    C_ = d.heads * d.d
    R = []
    for b in range(d.batch):
        R += _r(d.q + 2 * b * d.q_batch_stride, d.nq, C_ * 2, d.q_ld * 2)
        R += _r(d.k + 2 * b * d.k_batch_stride, d.nk, C_ * 2, d.k_ld * 2)
    R += _r(d.vt, d.batch * C_, d.nk * 2, d.vt_ld * 2)
    return R, _r(d.out, d.batch * d.nq, C_ * 2, d.o_ld * 2)


def _gn_ticket_offset(batch, groups):
    """the ticket counters' offset in the standalone scratch: the layout mirror whose total size
    test_norm_and_small_kernels_gpu.py holds equal to pp_group_norm_scratch_bytes"""
    return gn_geometry(batch, 64, 8 * groups, groups)["ticket_offset"]


def fp_gn(op):
    from powerpaint_b200 import ops as o

    d = op.c
    rows = d.batch * d.hw
    R = _r(d.x0, rows * d.c0 * 2) + _r(d.x1, rows * d.c1 * 2)
    W = _r(d.y, rows * (d.c0 + d.c1) * 2)
    if d.from_partials:
        R += _r(d.part0, int(d.geom0.bytes)) + (_r(d.part1, int(d.geom1.bytes)) if d.x1 else [])
        W += _r(d.stats, d.batch * d.groups * 8)
    else:
        if d.stats_prezeroed:  # the tickets the arena memset (or the previous call) left at zero
            R += _r(d.stats + _gn_ticket_offset(d.batch, d.groups), d.batch * 4)
        W += _r(d.stats, o.gn_scratch_bytes(d.batch, d.hw, d.c0 + d.c1, d.groups))
    return R, W


def gn_counters(op):
    d = op.c
    return [] if d.from_partials else _r(d.stats + _gn_ticket_offset(d.batch, d.groups), d.batch * 4)


def _eps_region(d, nb):
    el = 4 if d.eps_fp32 else 2
    return _r(d.eps, nb * d.hw, 4 * el, d.eps_ld * el)


def _next_in(d, row_bytes):
    return _r(d.next_in, d.n_copies * d.batch * d.hw, row_bytes, d.next_c * 2) if d.next_in else []


def _step_common(d):
    nb = 2 * d.batch if d.do_cfg else d.batch
    st = d.batch * d.hw * 16
    R = _eps_region(d, nb) + _r(d.latents, st) + _r(d.step_idx, 4)
    W = _r(d.latents, st) + (_r(d.step_idx, 4) if d.advance_step else [])
    return R, W, st


def fp_cfg_ddim(op):
    d = op.c
    R, W, st = _step_common(d)
    R += _r(d.noise, st) + _r(d.blend_x0, d.hw * 16) + _r(d.blend_mask, d.hw * 4) + _r(d.blend_noise, st)
    if d.extra_c:
        R += _r(d.extra, (d.n_copies if d.extra_per_copy else 1) * d.batch * d.hw * d.extra_c * 4)
    W += _next_in(d, 8 if d.extra_c == 0 else d.next_c * 2)
    return R, W


def fp_unipc(op):
    d = op.c
    R, W, st = _step_common(d)
    for f in ("last_sample", "m1", "m2"):
        R += _r(getattr(d, f), st)
        W += _r(getattr(d, f), st)
    return R, W + _next_in(d, 8)


def fp_solver(op):
    d = op.c
    R, W, st = _step_common(d)
    R += _r(d.m1, st) + _r(d.noise, st)
    return R, W + _r(d.m1, st) + _next_in(d, 8)


def fp_plms(op, row=None):
    """`row`: the pcoef row the step reads (then the ring slot / cur_sample reads and writes are the row's); None:
    every slot, as the recording cannot know which step runs"""
    d = op.c
    R, W, st = _step_common(d)
    R += _r(d.blend_x0, d.hw * 16) + _r(d.blend_mask, d.hw * 4) + _r(d.blend_noise, st)
    if row is None:
        R += _r(d.cur_sample, st) + _r(d.ets, 3 * st)
        W += _r(d.cur_sample, st) + _r(d.ets, 3 * st)
    else:
        if row[1] != 0:
            R += _r(d.cur_sample, st)
        for k in range(3):
            if row[3 + k] != 0:
                R += _r(d.ets + k * st, st)
        if row[7] != 0:
            W += _r(d.cur_sample, st)
        if row[6] >= 0:
            W += _r(d.ets + int(row[6]) * st, st)
    return R, W + _next_in(d, 8)


def fp_tile_blend(op):
    d = op.c
    row = d.b_w * d.channels * 4
    R, W = [], []
    for s in range(d.batch):
        b = d.b + 4 * s * d.b_stride
        if d.e_v:
            R += _r(d.av + 4 * s * d.av_stride + (d.av_h - d.e_v) * row, d.e_v * row)
            R += _r(b, d.e_v * row)
            W += _r(b, d.e_v * row)
        if d.e_h:
            ah_row = d.ah_w * d.channels * 4
            R += _r(d.ah + 4 * s * d.ah_stride + (d.ah_w - d.e_h) * d.channels * 4, d.b_h, d.e_h * d.channels * 4, ah_row)
            R += _r(b, d.b_h, d.e_h * d.channels * 4, row)
            W += _r(b, d.b_h, d.e_h * d.channels * 4, row)
    return R, W


def fp_pool_broadcast(op):
    d = op.c
    n = d.batch * d.hw * d.channels * 2
    return _r(d.x, n) + _r(d.prev, n), _r(d.out, n)


def _windows(wl):
    from powerpaint_b200 import _native as N

    raw = bytes(wl.table.cpu().numpy().tobytes())
    return [N.Window.from_buffer_copy(raw, i * ctypes.sizeof(N.Window)) for i in range(wl.count)]


def fp_window_copy(a):
    wl = a["wl"]
    eb = wl.src.element_size()
    R, W = [], []
    for w in _windows(wl):
        for side, base, off, rowp, pix, out in (("src", wl.src, w.src_off, w.src_row, wl.src_pix, R),
                                                ("dst", wl.dst, w.dst_off, w.dst_row, wl.dst_pix, W)):
            start = base.data_ptr() + off * eb
            if pix == wl.channels:  # pixels back to back: one region of `rows` runs
                out += _r(start, w.rows, w.cols * pix * eb, rowp * eb)
            else:
                for y in range(w.rows):
                    out += _r(start + y * rowp * eb, w.cols, wl.channels * eb, pix * eb)
    return R, W


def _a(fn):
    return lambda op: fn(op.args)


FOOTPRINTS = {
    "gemm": fp_gemm, "attn": fp_attn, "gn": fp_gn, "cfg_ddim": fp_cfg_ddim, "unipc": fp_unipc, "solver": fp_solver,
    "plms": fp_plms, "tile_blend": fp_tile_blend, "pool_broadcast": fp_pool_broadcast,
    "window_copy": _a(fp_window_copy),
    "layer_norm": _a(lambda a: (_r(a["x"], a["rows"] * a["c"] * 2), _r(a["y"], a["rows"] * a["c"] * 2))),
    "upsample2x": _a(lambda a: (_r(a["x"], a["nb"] * a["h"] * a["w"] * a["c"] * 2),
                                _r(a["y"], a["nb"] * 4 * a["h"] * a["w"] * a["c"] * 2))),
    "upsample_nearest": _a(lambda a: (_r(a["x"], a["nb"] * a["h"] * a["w"] * a["c"] * 2),
                                      _r(a["y"], a["nb"] * a["ho"] * a["wo"] * a["c"] * 2))),
    "softmax_rows": _a(lambda a: (_r(a["s"], a["rows"], a["cols"] * 4, a["ld_s"] * 4),
                                  _r(a["p"], a["rows"], a["cols"] * 2, a["ld_p"] * 2))),
    "embed_gather": _a(lambda a: (_r(a["idx"], a["rows"] * 4), _r(a["out"], a["rows"] * a["dim"] * 2))),
    "causal_attention_small": _a(lambda a: (_r(a["qkv"], a["batch"] * a["seq"] * 3 * a["heads"] * a["d"] * 2),
                                            _r(a["out"], a["batch"] * a["seq"] * a["heads"] * a["d"] * 2))),
    "add": _a(lambda a: (_r(a["a"], a["n"] * 2) + _r(a["b"], a["n"] * 2), _r(a["y"], a["n"] * 2))),
    "time_embed": _a(lambda a: (_r(a["step_idx"], 4) + _r(a["timesteps"], a["timesteps"].numel() * 4),
                                _r(a["out"], a["batch"] * a["dim"] * 2))),
    "memset": _a(lambda a: ([], _r(a["t"], a["t"].numel() * a["t"].element_size()))),
}
COUNTERS = {"gemm": gemm_counters, "gn": gn_counters}


def footprint(op, step=0):
    return fp_gemm(op, step) if op.kind == "gemm" else FOOTPRINTS[op.kind](op)


# =========================================================================== capture
class Capture:
    """the ordered ops of every Program recorded while active, per Program instance"""

    def __init__(self, mp):
        from powerpaint_b200 import ops as o

        self.ops = {}  # id(program) -> [op]
        self.programs = {}  # id(program) -> program (kept alive: ids stay unique)
        orig_add = o.Program.add

        def add(prog, desc):
            orig_add(prog, desc)
            self._record(prog, desc)
        mp.setattr(o.Program, "add", add)
        for meth in PROGRAM_RECORD_METHODS:
            orig = getattr(o.Program, meth)

            def hook(prog, *args, _orig=orig, _kind=meth[len("add_"):], **kw):
                bound = inspect.signature(_orig).bind(prog, *args, **kw).arguments
                _orig(prog, *args, **kw)
                self._record(prog, ProgramCall(_kind, {k: v for k, v in bound.items() if k != "self"}))
            mp.setattr(o.Program, meth, hook)

    def _record(self, prog, op):
        self.programs[id(prog)] = prog
        self.ops.setdefault(id(prog), []).append(op)

    def of(self, prog):
        ops_ = self.ops.get(id(prog), [])
        assert len(ops_) == prog.num_ops == len(prog.labels), (len(ops_), prog.num_ops, len(prog.labels))
        assert [op.kind for op in ops_] == prog.labels
        return ops_


def _never_recycling_pool(mp, buf_blocks):
    """Pool.free keeps every block: each buffer of the plan gets storage of its own. `buf_blocks` collects the data
    pointers of the activation blocks (as opposed to inputs / persistent tensors)"""
    from powerpaint_b200.engine import Pool

    orig_buf = Pool.buf

    def buf(self, *shape, dtype=BF16):
        t = orig_buf(self, *shape, dtype=dtype)
        buf_blocks.add(self.raw_of[t.data_ptr()].data_ptr())
        return t
    mp.setattr(Pool, "free", lambda self, *tensors: None)
    mp.setattr(Pool, "buf", buf)


# =========================================================================== static dataflow
class Blocks:
    """the tracked storage of a plan: (start, nbytes, is activation block) sorted by address"""

    def __init__(self, tensors, buf_ptrs=()):
        seen = {}
        for t in tensors:
            if isinstance(t, torch.Tensor) and t.is_cuda and t.numel():
                st = t.untyped_storage()
                seen[st.data_ptr()] = st
        self.starts = sorted(seen)
        self.storages = [seen[p] for p in self.starts]
        self.sizes = [st.nbytes() for st in self.storages]
        self.is_buf = [p in buf_ptrs for p in self.starts]

    def locate(self, region):
        """(block index, offset) of a region that lies inside one tracked block, None for untracked memory (weights);
        a region that starts in a block and leaves it fails"""
        ptr, rows, rb, pitch = region
        i = int(np.searchsorted(self.starts, ptr, side="right")) - 1
        if i < 0 or ptr >= self.starts[i] + self.sizes[i]:
            return None
        off = ptr - self.starts[i]
        assert off + (rows - 1) * pitch + rb <= self.sizes[i], f"region {region} leaves its block"
        return i, off


def dataflow(seq, blocks, fresh):
    """seq: [(tag, op)] in execution order. For every read region: {writer tag: bytes}; `fresh`: also fail a read of an
    activation byte nothing wrote before"""
    fps = [footprint(op, tag[1] if tag[0] == "step" else 0) for tag, op in seq]
    gran = [0] * len(blocks.starts)
    located = []
    for R, W in fps:
        loc = ([(blocks.locate(r), r) for r in R], [(blocks.locate(w), w) for w in W])
        for lst in loc:
            for where, (_, rows, rb, pitch) in lst:
                if where is not None:
                    i, off = where
                    gran[i] = math.gcd(gran[i], off, rb, pitch if rows > 1 else 0)
        located.append(loc)
    last = [np.full((sz + (g or 1) - 1) // (g or 1), -1, np.int32) for sz, g in zip(blocks.sizes, gran)]

    def view(i, off, rows, rb, pitch):
        g = gran[i] or 1
        a = last[i][off // g:]
        return np.lib.stride_tricks.as_strided(a, shape=(rows, rb // g), strides=(pitch // g * 4, 4))
    sigs = []
    for k, (loc, (tag, op)) in enumerate(zip(located, seq)):
        for where, (_, rows, rb, pitch) in loc[0]:
            if where is None:
                sigs.append((tag, "untracked"))  # a weight or a table outside the plan's storage
                continue
            v = view(where[0], where[1], rows, rb, pitch)
            w, cnt = np.unique(v, return_counts=True)
            g = gran[where[0]] or 1
            sig = tuple(zip(w.tolist(), (cnt * g).tolist()))
            if fresh and blocks.is_buf[where[0]]:
                assert w[0] >= 0, f"{tag} {op.kind} reads activation bytes no op wrote before it"
            sigs.append((tag, sig))
        for where, (_, rows, rb, pitch) in loc[1]:
            if where is not None:
                view(where[0], where[1], rows, rb, pitch)[:] = k
    return sigs


def _compare(a, b, name):
    assert len(a) == len(b), name
    for (ta, sa), (tb, sb) in zip(a, b):
        assert ta == tb, name
        assert sa == sb, f"{name}: {ta} reads bytes last written by ops {sa} with the recycled pool, {sb} without"


def _denoiser_seq(cap, st, steps=2):
    seq = []
    for sp in st["side_plans"]:
        if sp.cond_program is not None:
            seq += [(("cond", i), op) for i, op in enumerate(cap.of(sp.cond_program))]
    seq += [(("ctx", i), op) for i, op in enumerate(cap.of(st["ctx_program"]))]
    body = cap.of(st["program"])
    for s in range(steps):
        seq += [(("step", s, i), op) for i, op in enumerate(body)]
    return seq


def _denoiser_tensors(st):
    pool = st["uplan"].pool
    return list(pool.buffers) + [v for v in st.values() if isinstance(v, torch.Tensor)] + list(st["residuals"])


def _record_denoiser(fd, args, fresh):
    with pytest.MonkeyPatch.context() as mp:
        bufs = set()
        if fresh:
            _never_recycling_pool(mp, bufs)
        cap = Capture(mp)
        st = fd._record(*args)
    return cap, st, bufs


def _static_denoiser(fd, args, name):
    if len(args[-1]) != len(fd.sides):  # pools: one flag per side net
        args = args[:-1] + ((False,) * len(fd.sides),)
    out = []
    for fresh in (False, True):
        cap, st, bufs = _record_denoiser(fd, args, fresh)
        out.append(dataflow(_denoiser_seq(cap, st), Blocks(_denoiser_tensors(st), bufs), fresh))
        del cap, st
        torch.cuda.empty_cache()
    _compare(out[0], out[1], name)
    return len(out[0])


# args of FusedDenoiser._record: B, h, w, do_cfg, ctx_len, with_noise, extra_per_copy, sched, blend, guess, pools
def _rec_args(B, h, w, sched="ddim", with_noise=False, blend=False, guess=False, pools=(), extra_per_copy=False):
    return (B, h, w, True, 77, with_noise, extra_per_copy, sched, blend, guess, pools)


@pytest.fixture(scope="module")
def ops():
    from powerpaint_b200 import _native, ops as o

    assert _native.lib().pp_device_supported() == 1, "tests need an sm_90 (H100) device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("switch", [s[0] for s in ENGINE_SWITCHES])
def test_static_dataflow_of_the_production_denoisers(ops, switch):
    """every bench / odd-size denoiser shape at SD-1.5 width under one engine switch: same last writer of every byte
    read with and without block recycling"""
    from powerpaint_b200.denoise import FusedDenoiser
    from powerpaint_b200.engine import NetConfig, Recorder
    from powerpaint_b200.models import BrushNetModel, ControlNetModel, UNet2DConditionModel

    sw = dict(ENGINE_SWITCHES)[switch]
    with pytest.MonkeyPatch.context() as mp:
        for attr, val in sw.items():
            mp.setattr(Recorder, attr, val)
        u9 = UNet2DConditionModel.synthetic(NetConfig(in_channels=9), seed=1234).to(DEV)
        u4 = UNet2DConditionModel.synthetic(NetConfig(in_channels=4), seed=1234).to(DEV)
        bn = BrushNetModel.synthetic(NetConfig(in_channels=4), seed=99).to(DEV)
        cn = ControlNetModel.synthetic(NetConfig(in_channels=4), seed=77).to(DEV)
        for name, mode, B, h, w in DENOISER_SHAPES:
            fd = {"v1": lambda: FusedDenoiser(u9), "brushnet": lambda: FusedDenoiser(u4, bn, "brushnet"),
                  "controlnet": lambda: FusedDenoiser(u9, cn, "controlnet")}[mode]()
            n = _static_denoiser(fd, _rec_args(B, h, w, extra_per_copy=mode == "brushnet"), f"{name} [{switch}]")
            print(f"[static] {name} [{switch}]: {n} reads, same writers")
            del fd
            torch.cuda.empty_cache()


def _tiny(mode, n_cn=1):
    from test_pipelines_gpu import _nets

    from powerpaint_b200.denoise import FusedDenoiser

    if mode == "v1":
        return FusedDenoiser(_nets(9, [("unet", 9, 1234)])["unet"][1])
    if mode == "brushnet":
        n = _nets(4, [("unet", 4, 1234), ("brushnet", 4, 99)])
        return FusedDenoiser(n["unet"][1], n["brushnet"][1], "brushnet")
    n = _nets(9, [("unet", 9, 1234), ("controlnet", 4, 77)])
    cns = [n["controlnet"][1]] + [_nets(4, [("controlnet", 4, 78 + k)])["controlnet"][1] for k in range(n_cn - 1)]
    return FusedDenoiser(n["unet"][1], cns if n_cn > 1 else cns[0], "controlnet")


STATIC_TINY = [
    ("v1 ddim eta", "v1", 1, dict(with_noise=True)), ("v1 unipc", "v1", 1, dict(sched="unipc")),
    ("v1 dpm++", "v1", 1, dict(sched="solver")), ("v1 dpm++ sde", "v1", 1, dict(sched="solver", with_noise=True)),
    ("v1 plms", "v1", 1, dict(sched="plms")), ("brushnet unipc", "brushnet", 1, dict(sched="unipc",
                                                                                     extra_per_copy=True)),
    ("multi-controlnet x2", "controlnet", 2, {}), ("controlnet guess pooled", "controlnet", 2,
                                                   dict(guess=True, pools=(True, False))),
    ("brushnet guess", "brushnet", 1, dict(guess=True, pools=(False,), extra_per_copy=True)),
]


@pytest.mark.gpu
def test_static_dataflow_of_schedulers_side_nets_and_blend(ops):
    """each scheduler kind, Multi-ControlNet, guess mode with a pooled side net, at the tiny width (odd latent 9x11),
    and the 4-channel blend at SD-1.5 width"""
    from powerpaint_b200.denoise import FusedDenoiser
    from powerpaint_b200.engine import NetConfig
    from powerpaint_b200.models import UNet2DConditionModel

    for name, mode, n_cn, kw in STATIC_TINY:
        fd = _tiny(mode, n_cn)
        kw = dict(kw)
        if "pools" in kw:
            kw["pools"] = kw["pools"][:len(fd.sides)]
        n = _static_denoiser(fd, _rec_args(2, 9, 11, **kw), name)
        print(f"[static] {name}: {n} reads, same writers")
    u4 = UNet2DConditionModel.synthetic(NetConfig(in_channels=4), seed=1234).to(DEV)
    for sched in ("ddim", "plms"):
        n = _static_denoiser(FusedDenoiser(u4), _rec_args(2, 32, 32, sched=sched, blend=True), f"blend {sched}")
        print(f"[static] 4-channel blend {sched} SD-1.5 32x32: {n} reads, same writers")


def _static_plan(make, name):
    out = []
    for fresh in (False, True):
        with pytest.MonkeyPatch.context() as mp:
            bufs = set()
            if fresh:
                _never_recycling_pool(mp, bufs)
            cap = Capture(mp)
            plan = make()
        progs = [cap.programs[k] for k in cap.ops]  # in the order they first recorded an op
        seq = [((j, i), op) for j, p in enumerate(progs) for i, op in enumerate(cap.of(p))]
        tens = list(plan.pool.buffers) + list(plan.inputs.values()) + [v for v in plan.outputs.values()
                                                                       if isinstance(v, torch.Tensor)]
        out.append(dataflow(seq, Blocks(tens, bufs), fresh))
        del plan, cap
        torch.cuda.empty_cache()
    _compare(out[0], out[1], name)
    return len(out[0])


@pytest.mark.gpu
def test_static_dataflow_of_vae_and_text_encoder(ops):
    from powerpaint_b200.models import CLIPTextModel
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    vae = AutoencoderKL.synthetic(seed=4321).to(DEV)
    e = vae.engine()
    vae.tile_sample_min_size, vae.tile_latent_min_size = 512, 64
    cases = [("VAE encode 512x512", lambda: e.encode_plan(1, 512, 512)),
             ("VAE decode 64x64", lambda: e.decode_plan(1, 64, 64)),
             ("VAE tiled decode 80x80",
              lambda: e.tiled_plan(False, 1, 80, 80, vae.tile_geometry(False, 80, 80), vae._tiling_key()))]
    for name, make in cases:
        n = _static_plan(lambda: (e._plans.clear(), make())[1], name)  # record anew each time, not from the cache
        print(f"[static] {name}: {n} reads, same writers")
    te = CLIPTextModel().to(DEV)
    n = _static_plan(lambda: (te.engine()._plans.clear(), te.engine().plan_for(2, 77, 0))[1], "text encoder")
    print(f"[static] text encoder 2x77: {n} reads, same writers")


# =========================================================================== replay
def ref_solver(eps, x, m1, noise, r, gscale, do_cfg, B):
    """fp64 pp_solver_desc row formula: (x_next, m_t, bound of each)"""
    r = [float(v) for v in r]
    e, ea = _cfg_eps(eps, gscale, do_cfg, B)
    xd, a1 = x.double(), m1.double()
    nz = noise.double() if noise is not None else torch.zeros_like(xd)
    mt = r[0] * xd + r[1] * e
    mta = abs(r[0]) * xd.abs() + abs(r[1]) * ea
    xn = r[2] * xd + r[3] * mt + r[4] * a1 + r[5] * nz
    xna = abs(r[2]) * xd.abs() + abs(r[3]) * mta + abs(r[4]) * a1.abs() + abs(r[5]) * nz.abs()
    return xn, mt, 12 * U32 * xna + 1e-30, 12 * U32 * mta + 1e-30


def ref_plms(eps, x, cur, ets, r, gscale, do_cfg, B, blend_args):
    """fp64 pp_plms_desc row formula: (x_next, bound, eps after CFG, bound); terms of weight 0 are not read"""
    r = [float(v) for v in r]
    e, ea = _cfg_eps(eps, gscale, do_cfg, B)
    xd = x.double()
    xn, xa = r[2] * e, abs(r[2]) * ea
    for wgt, t in ((r[0], xd), (r[1], cur), (r[3], ets[0]), (r[4], ets[1]), (r[5], ets[2])):
        if wgt != 0:
            xn, xa = xn + wgt * t.double(), xa + abs(wgt) * t.double().abs()
    if blend_args is not None:
        o, m, nn, a = blend_args
        o, m, nn = o.double(), m.double().reshape(1, -1, 1), nn.double()
        s1a = max(1 - a * a, 0.0) ** 0.5
        xn = (1 - m) * (a * o[None] + s1a * nn) + m * xn
        xa = (1 - m).abs() * (abs(a) * o[None].abs() + s1a * nn.abs()) * 16 + m.abs() * xa
    return xn, 12 * U32 * xa + 1e-30, e, 8 * U32 * ea + 1e-30


def _kept_tensors(progs):
    """every CUDA tensor the programs keep alive: each pointer an op was recorded with lies in one of them"""
    out, stack = [], [p._keep for p in progs]
    while stack:
        v = stack.pop()
        if isinstance(v, torch.Tensor):
            if v.is_cuda:
                out.append(v)
        elif isinstance(v, (list, tuple)):
            stack.extend(v)
        elif isinstance(v, dict):
            stack.extend(v.values())
        elif hasattr(v, "keep"):  # a Desc
            stack.append(v.keep)
        elif hasattr(v, "table"):  # a WindowList
            stack.extend([v.src, v.dst, v.table])
    return out


class Memory:
    """flat byte snapshots of the tracked storage (activations, state, weights), each block at a 256-byte aligned
    offset, and typed views of a snapshot by device pointer"""

    def __init__(self, tensors):
        self.blocks = Blocks(tensors)
        self.raw = [torch.empty(0, dtype=torch.uint8, device=DEV).set_(st, 0, (st.nbytes(),), (1,))
                    for st in self.blocks.storages]
        self.offs, n = [], 0
        for sz in self.blocks.sizes:
            self.offs.append(n)
            n += (sz + 255) // 256 * 256
        self.total = n

    def snapshot(self):
        snap = torch.zeros(self.total, dtype=torch.uint8, device=DEV)
        torch._foreach_copy_([snap[o:o + r.numel()] for o, r in zip(self.offs, self.raw)], self.raw)
        return snap

    def view(self, snap, ptr, n, dtype):
        i = int(np.searchsorted(self.blocks.starts, ptr, side="right")) - 1
        it = torch.empty(0, dtype=dtype).element_size()
        assert i >= 0, f"pointer {ptr:#x} outside the tracked storage"
        off = ptr - self.blocks.starts[i]
        assert off + n * it <= self.blocks.sizes[i], f"{n} elements at {ptr:#x} leave their block"
        return snap[self.offs[i] + off:self.offs[i] + off + n * it].view(dtype)

    def mat(self, snap, ptr, rows, cols, ld, dtype):
        return self.view(snap, ptr, (rows - 1) * ld + cols, dtype).as_strided((rows, cols), (ld, 1))

    def mask(self, regions):
        """a bool byte mask of `regions` over a snapshot"""
        m = torch.zeros(self.total, dtype=torch.bool, device=DEV)
        for reg in regions:
            where = self.blocks.locate(reg)
            assert where is not None, f"write region {reg} outside the tracked storage"
            i, off = where
            _, rows, rb, pitch = reg
            m.as_strided((rows, rb), (pitch, 1), self.offs[i] + off).fill_(True)
        return m


def _step_row(mem, snap, tab_ptr, step_ptr, width):
    step = int(mem.view(snap, step_ptr, 1, torch.int32)[0]) if step_ptr else 0
    return step, mem.view(snap, tab_ptr, (step + 1) * width, torch.float32)[step * width:].cpu()


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_bits(name, got, ref):
    assert torch.equal(_bits(got), _bits(ref.to(got.dtype))), f"{name}: not bit-identical"


def eval_gemm(name, op, mem, before, after):
    from powerpaint_b200 import ops as o

    d = op.c
    M = gemm_out_geometry(d)[0]
    ext = gemm_extents(d)
    # flat views over each operand's extent (ref_gemm re-strides them with the descriptor's pitches)
    t = {f: mem.view(before, getattr(d, f), (rows - 1) * ld + cols, dt)
         for f, (rows, cols, ld, dt) in ext.items() if f not in ("out", "out_t")}
    if d.alpha_dev:
        step = int(mem.view(before, d.alpha_step, 1, torch.int32)[0]) if d.alpha_step else 0
        t["alpha_dev"] = mem.view(before, d.alpha_dev, step * d.alpha_stride + 1, torch.float32)
        if d.alpha_step:
            t["alpha_step"] = mem.view(before, d.alpha_step, 1, torch.int32)
    outs = {f: mem.mat(after, getattr(d, f), *ext[f]) for f in ("out", "out_t") if f in ext}
    bn = o.gemm_variant(op)[0]
    for r0, r1, ref, bound, _ in ref_gemm(d, t, bn):
        assert_within(f"{name} rows {r0}:{r1}", gemm_got_chunk(d, outs, r0, r1), ref, bound)
    if d.row_stats:
        rec = o.gemm_row_stats_records(op)
        extra = {"final": mem.view(after, d.row_final, M * 2, torch.float32).view(M, 2),
                 "rec": mem.view(after, d.row_stats, rec * d.row_stats_ld * 4, torch.float32).view(
                     rec, d.row_stats_ld, 4),
                 "ticket": mem.view(after, d.row_ticket, (M + 127) // 128, torch.int32)}
        _check_row_stats(name, d, t, extra, bn)


def eval_attn(name, op, mem, before, after):
    d = op.c
    B, C_ = d.batch, d.heads * d.d
    vdt = torch.float16 if d.vt_fp16 else BF16
    t = {"q": mem.view(before, d.q, (B - 1) * d.q_batch_stride + (d.nq - 1) * d.q_ld + C_, BF16),
         "k": mem.view(before, d.k, (B - 1) * d.k_batch_stride + (d.nk - 1) * d.k_ld + C_, BF16),
         "vt": mem.view(before, d.vt, (B * C_ - 1) * d.vt_ld + d.nk, vdt)}
    ref, bound = ref_attention(d, t)
    assert_within(name, mem.mat(after, d.out, B * d.nq, C_, d.o_ld, BF16), ref, bound)


def eval_gn(name, op, mem, before, after):
    d = op.c
    nb, hw, C = d.batch, d.hw, d.c0 + d.c1
    xs = [mem.view(before, d.x0, nb * hw * d.c0, BF16).view(nb, hw, d.c0)]
    if d.x1:
        xs.append(mem.view(before, d.x1, nb * hw * d.c1, BF16).view(nb, hw, d.c1))
    x = torch.cat(xs, -1)
    gamma, beta = mem.view(before, d.gamma, C, torch.float32), mem.view(before, d.beta, C, torch.float32)
    st = mem.view(after, d.stats, nb * d.groups * 2, torch.float32).view(nb, d.groups, 2)
    if d.from_partials:
        chain = max(producer_chain(g) for g in ([d.geom0, d.geom1] if d.x1 else [d.geom0]))
    else:
        chain = standalone_chain(nb, hw, C, d.groups)
    check_gn_stats(name, st, gn_truth(x, d.groups), chain, d.eps)
    ref, bound = gn_y_ref(x, st, gamma, beta, bool(d.silu))
    y = mem.view(after, d.y, nb * hw * C, BF16).view(nb * hw, C)
    assert_within(f"{name} y", y, ref.view(nb * hw, C), bound.view(nb * hw, C))


def _upsample_ref(x, ho, wo):
    nb, h, w, c = x.shape
    if ho == 2 * h and wo == 2 * w:
        return x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    f32 = dict(dtype=torch.float32, device=x.device)
    iy = (torch.arange(ho, **f32) * (torch.tensor(float(h), **f32) / torch.tensor(float(ho), **f32))).floor().long()
    ix = (torch.arange(wo, **f32) * (torch.tensor(float(w), **f32) / torch.tensor(float(wo), **f32))).floor().long()
    return x[:, iy.clamp(max=h - 1)][:, :, ix.clamp(max=w - 1)]


def eval_call(name, op, mem, before, after):
    a = op.args
    V = mem.view
    k = op.kind
    if k == "memset":
        t = a["t"]
        assert not V(after, t.data_ptr(), t.numel() * t.element_size(), torch.uint8).any(), f"{name}: non-zero"
    elif k == "add":
        n = a["n"]
        x, y = (V(before, _p(a[f]), n, BF16).float() for f in ("a", "b"))
        assert_bits(name, V(after, _p(a["y"]), n, BF16), x + y)
    elif k in ("upsample2x", "upsample_nearest"):
        nb, h, w, c = a["nb"], a["h"], a["w"], a["c"]
        ho, wo = (2 * h, 2 * w) if k == "upsample2x" else (a["ho"], a["wo"])
        ref = _upsample_ref(V(before, _p(a["x"]), nb * h * w * c, BF16).view(nb, h, w, c), ho, wo)
        assert_bits(name, V(after, _p(a["y"]), ref.numel(), BF16).view_as(ref), ref)
    elif k == "layer_norm":
        rows, c = a["rows"], a["c"]
        ref, bound = ref_layer_norm(V(before, _p(a["x"]), rows * c, BF16).view(rows, c),
                                    V(before, _p(a["gamma"]), c, torch.float32),
                                    V(before, _p(a["beta"]), c, torch.float32), a["eps"])
        assert_within(name, V(after, _p(a["y"]), rows * c, BF16).view(rows, c), ref, bound)
    elif k == "softmax_rows":
        rows, cols = a["rows"], a["cols"]
        p, bound = ref_softmax(mem.mat(before, _p(a["s"]), rows, cols, a["ld_s"], torch.float32),
                               softmax_instance(cols))
        assert_within(name, mem.mat(after, _p(a["p"]), rows, cols, a["ld_p"], BF16), p, bound)
    elif k == "causal_attention_small":
        b, seq, h, dd = a["batch"], a["seq"], a["heads"], a["d"]
        qkv = V(before, _p(a["qkv"]), b * seq * 3 * h * dd, BF16).view(b * seq, 3 * h * dd)
        r, bound = ref_causal_attention(qkv, b, seq, h, dd, a["scale"])
        assert_within(name, V(after, _p(a["out"]), b * seq * h * dd, BF16).view(b * seq, h * dd), r, bound)
    elif k == "time_embed":
        b, dim, ts = a["batch"], a["dim"], a["timesteps"]
        table = V(before, ts.data_ptr(), ts.numel(), torch.float32)
        if a["step_idx"] is not None:
            t = table[int(V(before, _p(a["step_idx"]), 1, torch.int32)[0])].expand(b)
        else:
            t = table[:b]
        e, bound = ref_time_embed(t, dim)
        assert_within(name, V(after, _p(a["out"]), b * dim, BF16).view(b, dim), e, bound)
    elif k == "embed_gather":
        rows, vocab, seq, dim = a["rows"], a["vocab"], a["seq"], a["dim"]
        idx = V(before, _p(a["idx"]), rows, torch.int32).long()
        base = V(before, _p(a["base"]), vocab * dim, torch.float32).view(vocab, dim)
        n_ext = max(int(idx.max()) - vocab + 1, 0)
        tab = torch.cat([base, V(before, _p(a["ext"]), n_ext * dim, torch.float32).view(n_ext, dim)]) if n_ext \
            else base
        pos = V(before, _p(a["pos"]), seq * dim, torch.float32).view(seq, dim)
        ref = tab[idx] + pos[torch.arange(rows, device=DEV) % seq]
        assert_bits(name, V(after, _p(a["out"]), rows * dim, BF16).view(rows, dim), ref)
    elif k == "window_copy":
        wl = a["wl"]
        dt, ch = wl.src.dtype, wl.channels
        for w in _windows(wl):
            n_s = (w.rows - 1) * w.src_row + (w.cols - 1) * wl.src_pix + ch
            n_d = (w.rows - 1) * w.dst_row + (w.cols - 1) * wl.dst_pix + ch
            eb = wl.src.element_size()
            src = V(before, wl.src.data_ptr() + w.src_off * eb, n_s, dt).as_strided(
                (w.rows, w.cols, ch), (w.src_row, wl.src_pix, 1))
            dst = V(after, wl.dst.data_ptr() + w.dst_off * eb, n_d, dt).as_strided(
                (w.rows, w.cols, ch), (w.dst_row, wl.dst_pix, 1))
            assert_bits(name, dst, src)
    else:
        raise AssertionError(f"{name}: no evaluator for {k}")


def eval_tile_blend(name, op, mem, before, after):
    """the torch loop of diffusers blend_v then blend_h: fp32 weights from the double expression, each product and
    the sum rounded separately"""
    d = op.c
    C = d.channels
    f32 = dict(dtype=torch.float32, device=DEV)
    for s in range(d.batch):
        b = mem.view(before, d.b + 4 * s * d.b_stride, d.b_h * d.b_w * C, torch.float32).view(d.b_h, d.b_w, C).clone()
        if d.e_v:
            av = mem.view(before, d.av + 4 * s * d.av_stride, d.av_h * d.b_w * C, torch.float32).view(d.av_h, d.b_w, C)
            for y in range(d.e_v):
                w1, w2 = torch.tensor(1 - y / d.e_v, **f32), torch.tensor(y / d.e_v, **f32)
                b[y] = av[d.av_h - d.e_v + y] * w1 + b[y] * w2
        if d.e_h:
            ah = mem.view(before, d.ah + 4 * s * d.ah_stride, d.b_h * d.ah_w * C, torch.float32).view(d.b_h, d.ah_w, C)
            for x in range(d.e_h):
                w1, w2 = torch.tensor(1 - x / d.e_h, **f32), torch.tensor(x / d.e_h, **f32)
                b[:, x] = ah[:, d.ah_w - d.e_h + x] * w1 + b[:, x] * w2
        got = mem.view(after, d.b + 4 * s * d.b_stride, d.b_h * d.b_w * C, torch.float32).view(d.b_h, d.b_w, C)
        assert_bits(f"{name} sample {s}", got, b)


def eval_pool_broadcast(name, op, mem, before, after):
    """out = bf16(prev + mean_p x): fp64 against a bound of the fixed-order fp32 sum over hw terms"""
    d = op.c
    n = d.batch * d.hw * d.channels
    x = mem.view(before, d.x, n, BF16).view(d.batch, d.hw, d.channels).double()
    mean = x.mean(1, keepdim=True)
    prev = mem.view(before, d.prev, n, BF16).view(d.batch, d.hw, d.channels).double() if d.prev else 0.0
    ref = (prev + mean).expand(d.batch, d.hw, d.channels)
    d_sum = (d.hw + 2) * U32 * x.abs().mean(1, keepdim=True) + 2 * U32 * (mean.abs() + (prev.abs() if d.prev else 0))
    bound = U16 * ref.abs() + 1.01 * d_sum + 1e-30
    assert_within(name, mem.view(after, d.out, n, BF16).view(d.batch, d.hw, d.channels), ref, bound)


def check_step(name, op, mem, before, after):
    """the step kernel's outputs on the op's actual inputs against the fp64 row formula"""
    d = op.c
    B, hw = d.batch, d.hw
    nb = 2 * B if d.do_cfg else B
    n4 = B * hw * 4
    V = lambda s, p, n, dt=torch.float32: mem.view(s, p, n, dt)  # noqa: E731
    if d.eps_fp32:
        eps = V(before, d.eps, nb * hw * d.eps_ld).view(nb, hw, d.eps_ld)[..., :4]
    else:
        eps = V(before, d.eps, nb * hw * d.eps_ld, BF16).view(nb, hw, d.eps_ld)[..., :4].float()
    x = V(before, d.latents, n4).view(B, hw, 4)
    lat = V(after, d.latents, n4).view(B, hw, 4)
    step, cf = _step_row(mem, before, d.coef, d.step_idx, 8)
    gscale = float(cf[5]) if op.kind != "cfg_ddim" or d.guidance_from_coef else float(d.guidance_scale)
    stored = lat
    if op.kind == "cfg_ddim":
        blend = None
        if d.blend_x0:
            blend = (V(before, d.blend_x0, hw * 4).view(hw, 4), V(before, d.blend_mask, hw),
                     V(before, d.blend_noise, n4).view(B, hw, 4))
        noise = V(before, d.noise, n4).view(B, hw, 4) if d.noise else None
        ref, bound = ref_cfg_ddim(eps, x, noise, cf, gscale, d.do_cfg, B, blend)
        checks = [(lat, ref, bound)]
        assert not d.extra_c, "the fused loop refreshes the latent channels only"
    elif op.kind == "unipc":
        _, u = _step_row(mem, before, d.ucoef, d.step_idx, 12)
        st = [V(before, p, n4).view(B, hw, 4) for p in (d.last_sample, d.m1, d.m2)]
        xn, xc, mt, bxn, bxc, bmt = ref_unipc(eps, x, *st, u, gscale, d.do_cfg, B)
        checks = [(lat, xn, bxn), (V(after, d.last_sample, n4).view(B, hw, 4), xc, bxc),
                  (V(after, d.m1, n4).view(B, hw, 4), mt, bmt)]
        assert torch.equal(V(after, d.m2, n4), V(before, d.m1, n4)), "m2 <- m1"
    elif op.kind == "solver":
        _, r = _step_row(mem, before, d.scoef, d.step_idx, 8)
        noise = V(before, d.noise, n4).view(B, hw, 4) if d.noise else None
        xn, mt, bxn, bmt = ref_solver(eps, x, V(before, d.m1, n4).view(B, hw, 4), noise, r, gscale, d.do_cfg, B)
        checks = [(lat, xn, bxn), (V(after, d.m1, n4).view(B, hw, 4), mt, bmt)]
        stored = (r[6].to(DEV) * lat)  # fp32 r6 * x_next, what the kernel packs
    else:
        _, r = _step_row(mem, before, d.pcoef, d.step_idx, 8)
        cur = V(before, d.cur_sample, n4).view(B, hw, 4)
        ets = [V(before, d.ets + k * n4 * 4, n4).view(B, hw, 4) for k in range(3)]
        bl = None
        if d.blend_x0:
            bl = (V(before, d.blend_x0, hw * 4).view(hw, 4), V(before, d.blend_mask, hw),
                  V(before, d.blend_noise, n4).view(B, hw, 4), float(cf[7]))
        xn, bxn, e, be = ref_plms(eps, x, cur, ets, r, gscale, d.do_cfg, B, bl)
        checks = [(lat, xn, bxn)]
        if r[6] >= 0:  # the new eps replaces a ring slot, after the reads above
            checks.append((V(after, d.ets + int(r[6]) * n4 * 4, n4).view(B, hw, 4), e, be))
        if r[7] != 0:
            assert torch.equal(V(after, d.cur_sample, n4), V(before, d.latents, n4)), "cur_sample <- x"
    for k, (got, ref, bound) in enumerate(checks):
        bad = (got.double() - ref).abs() > bound
        assert not bad.any(), f"{op.kind} step {step} output {k}: {int(bad.sum())} elements off the fp64 row formula"
    if d.next_in:
        ni = V(after, d.next_in, d.n_copies * B * hw * d.next_c, BF16).view(d.n_copies * B, hw, d.next_c)
        for c in range(d.n_copies):
            assert torch.equal(ni[c * B:(c + 1) * B, :, :4], stored.to(BF16)), f"{op.kind} next_in copy {c}"
    if d.step_idx and d.advance_step:
        assert int(V(after, d.step_idx, 1, torch.int32)[0]) == step + 1
    return step


EVALUATORS = {"gemm": eval_gemm, "attn": eval_attn, "gn": eval_gn, "tile_blend": eval_tile_blend,
              "pool_broadcast": eval_pool_broadcast, "cfg_ddim": check_step, "unipc": check_step,
              "solver": check_step, "plms": check_step}
EVALUATORS.update({k: eval_call for k in ("memset", "add", "upsample2x", "upsample_nearest", "layer_norm",
                                          "softmax_rows", "causal_attention_small", "time_embed", "embed_gather",
                                          "window_copy")})
REPLAY_EVALUATED = tuple(EVALUATORS)  # op kinds whose outputs the replay evaluates


class Replay:
    """Program.run / launch replaced by one checked `run_range(i, 1)` per op: after each op nothing outside its write
    footprint moved (activations, state and weights alike), its counters are back at zero, and its outputs equal the
    fp64 (or exact) evaluation of its contract on the inputs it actually read"""

    def __init__(self, mp, extra_tensors=lambda: []):
        from powerpaint_b200 import ops as o

        self.cap = Capture(mp)
        self.extra = extra_tensors
        self.mem = None
        self.ops_run = 0
        self.kinds = {}
        self.step_checks = {}
        mp.setattr(o.Program, "run", lambda prog: self.run(prog))
        mp.setattr(o.Program, "launch", lambda prog: self.run(prog))

    def run(self, prog):
        if self.mem is None:  # every plan of this call is recorded by now
            self.mem = Memory(_kept_tensors(list(self.cap.programs.values())) + list(self.extra()))
        mem = self.mem
        after = mem.snapshot()  # the host may have written inputs since the previous run
        for i, op in enumerate(self.cap.of(prog)):
            name = f"op {i} ({op.kind})"
            before = after
            prog.run_range(i, 1)
            torch.cuda.synchronize()
            after = mem.snapshot()
            if op.kind == "plms":
                R, W = fp_plms(op, _step_row(mem, before, op.c.pcoef, op.c.step_idx, 8)[1].tolist())
            elif op.kind == "gemm":
                step = int(mem.view(before, op.c.alpha_step, 1, torch.int32)[0]) if op.c.alpha_step else 0
                R, W = fp_gemm(op, step)
            else:
                R, W = footprint(op)
            moved = (before != after) & ~mem.mask(W)
            if moved.any():
                at = int(moved.nonzero()[0])
                blk = int(np.searchsorted(mem.offs, at, side="right")) - 1
                raise AssertionError(f"{name} changed {int(moved.sum())} bytes outside its write footprint, first at "
                                     f"byte {at - mem.offs[blk]} of block {blk} ({mem.blocks.sizes[blk]} bytes)")
            for reg in COUNTERS.get(op.kind, lambda _: [])(op):
                assert not mem.view(after, reg[0], reg[2], torch.uint8).any(), f"{name} left a counter non-zero"
            res = EVALUATORS[op.kind](name, op, mem, before, after)
            if op.kind in ("cfg_ddim", "unipc", "solver", "plms"):
                self.step_checks[(op.kind, res)] = self.step_checks.get((op.kind, res), 0) + 1
            self.kinds[op.kind] = self.kinds.get(op.kind, 0) + 1
            self.ops_run += 1


def _inputs(fd, B, h, w, n_steps, sched, seed=0, blend=False, n_cn=1):
    """run() keyword arguments of a seeded n-step call"""
    from powerpaint_b200.schedulers import (DDIMScheduler, DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            PNDMScheduler, UniPCMultistepScheduler)

    g = torch.Generator().manual_seed(seed)
    cross = fd.unet.config.cross_attention_dim
    kw = dict(prompt_embeds=torch.randn(2 * B, 77, cross, generator=g) * 0.5, guidance_scale=7.5, use_graph=False)
    base = DDIMScheduler()
    if sched == "ddim":
        s = base
    elif sched == "unipc":
        s = UniPCMultistepScheduler.from_config(base.config)
    elif sched in ("dpm", "dpm_sde"):
        s = DPMSolverMultistepScheduler.from_config(base.config, algorithm_type="sde-dpmsolver++" if sched == "dpm_sde"
                                                    else "dpmsolver++")
    elif sched == "euler_a":
        s = EulerAncestralDiscreteScheduler.from_config(base.config)
    else:
        s = PNDMScheduler.from_config(base.config, skip_prk_steps=True)
    s.set_timesteps(10)
    kw["latents"] = torch.randn(B, 4, h, w, generator=g) * float(getattr(s, "init_noise_sigma", 1.0))
    kw["timesteps"] = s.timesteps[:n_steps]
    kw["coef"] = s.step_coefficients()[:n_steps]
    if sched == "unipc":
        kw["ucoef"] = s.unipc_coefficients()[:n_steps]
    elif sched in ("dpm", "dpm_sde", "euler_a"):
        kw["scoef"] = s.solver_coefficients()[:n_steps]
        if sched != "dpm":
            kw["noise_fn"] = lambda i: torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(100 + i))
    elif sched == "plms":
        kw["pcoef"] = s.plms_coefficients()[:n_steps]
    if fd.mode != "v1" or fd.unet.config.in_channels == 9:
        kw["extra"] = torch.randn((2 if fd.mode == "brushnet" else 1) * B, 5, h, w, generator=g)
    if fd.mode != "v1":
        kw["side_prompt_embeds"] = kw["prompt_embeds"]
    if fd.mode == "controlnet":
        imgs = [torch.rand(2 * B, 3, 8 * h, 8 * w, generator=g) for _ in range(n_cn)]
        kw["control_image"] = imgs if n_cn > 1 else imgs[0]
        if n_cn > 1:
            kw["side_scale"] = [1.0, 0.5][:n_cn]
    if blend:
        kw["blend"] = dict(x0=torch.randn(1, 4, h, w, generator=g), mask=(torch.rand(1, 1, h, w, generator=g) > 0.5)
                           .float(), noise=torch.randn(B, 4, h, w, generator=g),
                           sqrt_alpha=torch.rand(n_steps, generator=g) * 0.9)
    return kw


# (mode, scheduler, ControlNets, steps): v1 PLMS runs 6 steps, so steps 4 and 5 append to the ring slot that holds
# the oldest of the three entries they read
REPLAY_CASES = [("v1", "ddim", 1, 2), ("v1", "unipc", 1, 2), ("v1", "dpm", 1, 2), ("v1", "dpm_sde", 1, 2),
                ("v1", "euler_a", 1, 2), ("v1", "plms", 1, 6), ("brushnet", "ddim", 1, 2), ("brushnet", "unipc", 1, 2),
                ("controlnet", "ddim", 2, 2), ("controlnet", "plms", 1, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,sched,n_cn,steps", REPLAY_CASES)
def test_replay_tiny_loops_op_by_op(ops, mode, sched, n_cn, steps):
    """the tiny nets' fused loop (odd 9x11 latent) through FusedDenoiser.run, every op of the ControlNet
    conditioning, cross-attention and step programs checked as it runs"""
    fd = _tiny(mode, n_cn)
    with pytest.MonkeyPatch.context() as mp:
        rp = Replay(mp)
        fd.run(**_inputs(fd, 2, 9, 11, steps, sched, n_cn=n_cn))
    kind = {"ddim": "cfg_ddim", "unipc": "unipc", "plms": "plms"}.get(sched, "solver")
    assert rp.step_checks == {(kind, i): 1 for i in range(steps)}, rp.step_checks
    print(f"[replay] {mode} {sched} x{n_cn}: {rp.ops_run} ops checked, kinds {rp.kinds}")


@pytest.mark.gpu
def test_replay_v1_blend_and_sd15_width(ops):
    """the 4-channel blend (DDIM, and PLMS for 6 steps), and SD-1.5 width at 32x32 batch 2 and an odd 9x13 latent"""
    from powerpaint_b200.denoise import FusedDenoiser
    from test_pipelines_gpu import _nets

    u4 = _nets(4, [("unet", 4, 1234)])["unet"][1]
    for sched, steps in (("ddim", 2), ("plms", 6)):
        fd = FusedDenoiser(u4)
        with pytest.MonkeyPatch.context() as mp:
            rp = Replay(mp)
            fd.run(**_inputs(fd, 2, 9, 11, steps, sched, blend=True))
        print(f"[replay] v1 4-channel blend {sched}: {rp.ops_run} ops checked")
    u9 = _nets(9, [("unet", 9, 1234)], tiny=False)["unet"][1]
    for B, h, w in ((2, 32, 32), (1, 9, 13)):
        fd = FusedDenoiser(u9)
        with pytest.MonkeyPatch.context() as mp:
            rp = Replay(mp)
            fd.run(**_inputs(fd, B, h, w, 2, "ddim"))
        print(f"[replay] v1 SD-1.5 {B}x{h}x{w}: {rp.ops_run} ops checked, kinds {rp.kinds}")
        del fd, rp
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_replay_vae_and_text_encoder(ops):
    """the tiny VAE's encode, decode and tiled decode (3 x 3 overlapping latent tiles: window copies and seam blends),
    and the text encoder, through their public entry points, every op checked as it runs"""
    from powerpaint_b200.models import CLIPTextModel
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    g = torch.Generator(device=DEV).manual_seed(5)
    vae = AutoencoderKL.synthetic(tiny=True, seed=4321).to(DEV)
    seen = {}
    for name, call in (("encode", lambda: vae.encode(torch.rand(1, 3, 64, 72, device=DEV, generator=g) * 2 - 1)),
                       ("decode", lambda: vae.decode(torch.randn(1, 4, 8, 9, device=DEV, generator=g)))):
        with pytest.MonkeyPatch.context() as mp:
            rp = Replay(mp)
            call()
        print(f"[replay] VAE {name}: {rp.ops_run} ops checked, kinds {rp.kinds}")
        seen.update(rp.kinds)
    vae.enable_tiling()
    vae.tile_sample_min_size, vae.tile_latent_min_size = 64, 8
    assert len(vae.tile_geometry(False, 13, 13).groups()) >= 2
    with pytest.MonkeyPatch.context() as mp:
        rp = Replay(mp)
        vae.decode(torch.randn(1, 4, 13, 13, device=DEV, generator=g))
    print(f"[replay] VAE tiled decode 13x13: {rp.ops_run} ops checked, kinds {rp.kinds}")
    seen.update(rp.kinds)
    assert {"window_copy", "tile_blend", "softmax_rows"} <= set(seen), seen
    te = CLIPTextModel().to(DEV)
    ids = torch.randint(0, te.config.vocab_size, (2, 77), generator=torch.Generator().manual_seed(3))
    with pytest.MonkeyPatch.context() as mp:
        rp = Replay(mp)
        te(ids)
    print(f"[replay] text encoder 2x77: {rp.ops_run} ops checked, kinds {rp.kinds}")
    assert {"embed_gather", "causal_attention_small"} <= set(rp.kinds), rp.kinds


@pytest.mark.gpu
@pytest.mark.parametrize("mode,sched,n_cn,steps", [("v1", "ddim", 1, 2), ("v1", "unipc", 1, 2), ("v1", "dpm", 1, 2),
                                                   ("v1", "plms", 1, 6), ("brushnet", "unipc", 1, 2),
                                                   ("controlnet", "ddim", 2, 2)])
def test_graph_step_equals_replayed_step(ops, mode, sched, n_cn, steps):
    """the last step as a CUDA-graph launch (PDL edges between the kernels) and as one run_range(i, 1) per op with a
    synchronisation between ops, from the same saved state: latents, next_in and every state buffer bit-identical
    (PLMS: step 5, whose ring append replaces an entry the step reads). One launch each: evidence about the PDL
    ordering of this step, not a proof"""
    fd = _tiny(mode, n_cn)
    kw = _inputs(fd, 2, 9, 11, steps, sched, n_cn=n_cn)
    kw["use_graph"] = True
    fd.run(**kw)  # the graph is captured
    st = next(iter(fd._cache.values()))
    assert st["graph"]
    st["step_idx"].fill_(steps - 1)
    live = _denoiser_tensors(st)
    saved = [t.clone() for t in live]
    prog = st["program"]
    prog.launch()
    torch.cuda.synchronize()
    graph_out = [t.clone() for t in live]
    for t, s_ in zip(live, saved):
        t.copy_(s_)
    for i in range(prog.num_ops):
        prog.run_range(i, 1)
        torch.cuda.synchronize()
    assert int(st["step_idx"]) == steps
    for k, (a, b) in enumerate(zip(graph_out, live)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"buffer {k} differs between graph and replay"


@pytest.mark.gpu
@pytest.mark.parametrize("mode,sched,n_cn,steps", [("v1", "ddim", 1, 2), ("v1", "plms", 1, 6), ("brushnet", "unipc", 1, 2),
                                                   ("controlnet", "ddim", 2, 2), ("v1", "dpm", 1, 2)])
def test_recycled_pool_equals_fresh_pool(ops, mode, sched, n_cn, steps):
    """the loop recorded on the activation Pool and on a Pool that never recycles a block: bit-identical latents"""
    outs = []
    for fresh in (False, True):
        fd = _tiny(mode, n_cn)
        kw = _inputs(fd, 2, 9, 11, steps, sched, n_cn=n_cn)
        with pytest.MonkeyPatch.context() as mp:
            if fresh:
                _never_recycling_pool(mp, set())
            outs.append(fd.run(**kw).clone())
    assert torch.equal(outs[0], outs[1])


# =========================================================================== CPU
def _recordable_kinds():
    import re

    from powerpaint_b200 import ops as o

    src = inspect.getsource(o.Program.add)
    descs = set(re.findall(r'"(\w+)": L\.pp_program_add_', src))
    calls = {m[len("add_"):] for m in dir(o.Program) if m.startswith("add_")}
    return descs | calls


def test_every_recordable_op_kind_has_a_footprint_and_a_check():
    """a new op kind fails here until it has a footprint and an evaluator the replay runs on its actual inputs"""
    from test_norm_and_small_kernels_gpu import COVERED_ELSEWHERE

    kinds = _recordable_kinds()
    assert {"gemm", "attn", "gn", "cfg_ddim", "unipc", "solver", "plms", "memset", "window_copy"} <= kinds, kinds
    assert kinds <= set(FOOTPRINTS), sorted(kinds - set(FOOTPRINTS))
    assert kinds <= set(EVALUATORS), sorted(kinds - set(EVALUATORS))
    for k in ("cfg_ddim", "unipc", "solver", "plms"):
        assert k not in COVERED_ELSEWHERE


def test_step_footprints_follow_the_header():
    """the footprints of a step descriptor built from integer addresses: eps pitch, 8-byte next_in rows, state writes,
    and PLMS ring slots from the row"""
    from powerpaint_b200 import _native as N
    from powerpaint_b200 import ops as o

    d = N.PlmsDesc()
    d.eps, d.eps_fp32, d.eps_ld = 1 << 20, 0, 8
    d.latents, d.cur_sample, d.ets = 2 << 20, 3 << 20, 4 << 20
    d.step_idx, d.advance_step, d.do_cfg, d.batch, d.hw = 5 << 20, 1, 1, 2, 10
    d.next_in, d.next_c, d.n_copies = 6 << 20, 16, 2
    op = o.Desc("plms", d, ())
    st = 2 * 10 * 16
    R, W = fp_plms(op, [0.5, 0.0, 1.0, 0.0, 2.0, 0.0, 1.0, 0.0])
    assert (1 << 20, 40, 8, 16) in R                   # bf16 eps, CFG: 2B rows, 4 channels of a 8-wide row
    assert [r for r in R if r[0] >= 4 << 20 and r[0] < 5 << 20] == [((4 << 20) + st, 1, st, st)]
    assert ((4 << 20) + st, 1, st, st) in W and (3 << 20, 1, st, st) not in W
    assert (6 << 20, 40, 8, 32) in W and (5 << 20, 1, 4, 4) in W
    R, W = fp_plms(op, [0.5, 1.0, 1.0, 0.0, 0.0, 0.0, -1.0, 1.0])
    assert (3 << 20, 1, st, st) in R and (3 << 20, 1, st, st) in W
    assert not [r for r in W if (4 << 20) <= r[0] < (5 << 20)]


def test_dataflow_sees_a_block_handed_on_too_early():
    """the dataflow signature on a hand-made sequence: a writer that overwrites a block before its last reader changes
    the reader's last writer"""
    class Op:
        def __init__(self, kind, args):
            self.kind, self.args = kind, args

    class T:
        def __init__(self, p, n):
            self.p, self.n = p, n

        def data_ptr(self):
            return self.p

    def add(a, b, y):
        return ProgramCall("add", dict(a=a, b=b, y=y, n=8))
    blocks = Blocks([])
    blocks.starts, blocks.sizes, blocks.is_buf = [1000, 2000, 3000], [16, 16, 16], [True, True, True]
    a, b, c = 1000, 2000, 3000
    seq_ok = [("w", add(5000, 5000, a)), ("x", add(5000, 5000, b)), ("r", add(a, b, c))]
    seq_bad = [("w", add(5000, 5000, a)), ("x", add(5000, 5000, a)), ("r", add(a, a, c))]
    s_ok = dataflow(seq_ok, blocks, True)
    s_bad = dataflow(seq_bad, blocks, False)
    with pytest.raises(AssertionError):
        _compare(s_ok, s_bad, "hand-made")
    _compare(s_ok, dataflow(seq_ok, blocks, False), "same")
    with pytest.raises(AssertionError):
        dataflow([("r", add(a, b, c))], blocks, True)  # reads activation bytes nothing wrote
