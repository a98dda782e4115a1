"""The VAE programs at the batches and canvases bench.py and the app run, op by op against fp64.

The census and replay files record the VAE at batch 1 and small canvases only. bench.py's e2e leg encodes and decodes
at batch 8 / 4 / 2 x 512^2 and 2 x 1024^2; the app's 640-short-side canvases give odd latents (80 x 107, 81 x 107,
where the attention's pitch hw_ld != hw); canvases above one megapixel go through tiled encode / decode. At 1024^2
the mid-block attention sits at the library's limits: hw = 16384 softmax columns, a 16384^2 fp32 score GEMM, a PV
GEMM with K = 16384, GroupNorm over 2^20 pixels.

- Static dataflow of every plan of VAE_SHAPES: the same last writer of every byte read with the recycling pool and
  with a pool that never recycles (test_program_replay_gpu._static_plan).
- Census of every plan: each distinct GEMM runs on fresh seeded inputs against the fp64 bound of
  test_kernel_variants_gpu.py, twice, bit-identical; each distinct GroupNorm runs standalone and over its producer's
  epilogue records; softmax_rows, upsample, memset, window_copy, tile_blend and the image pre / post-processing at
  the recorded sizes. The census asserts that it reached the limit shapes, so it cannot silently shrink.
- Replay through the public vae.encode / vae.decode on synthetic SD-width weights: every op checked as it runs
  (test_program_replay_gpu.Replay).
- End to end at 2 x 1024^2 against the fp32 oracle (oracle/vae.py).

The fp64 references of the largest ops (16384^2 scores, GroupNorm over 2 x 2^20 x 256 values) are evaluated in row
blocks: the checkers are the census files', only their inputs are sliced.
"""
import time

import pytest
import torch

from test_kernel_variants_gpu import (BF16, C_ACC, SENTINEL, U16, Canvas, _Census, _fresh_attention, _fresh_gemm,
                                      assert_canvases, assert_rerun_identical, assert_within, check_attention,
                                      check_gemm, fake_desc, gemm_out_geometry)
from test_norm_and_small_kernels_gpu import (OpCensus, _geom_tuple, _gn_params, _randn_bf16, _softmax_scores,
                                             check_gn_stats, check_upsample, gn_truth, gn_y_ref, producer_chain,
                                             ref_postprocess_u8, ref_softmax, run_group_norm, softmax_instance,
                                             standalone_chain)
from test_program_replay_gpu import (EVALUATORS, Capture, Memory, ProgramCall, Replay, _bits, _static_plan,
                                     _windows, footprint)

from powerpaint_b200.models.autoencoder_kl import PV_K_CHUNK, PV_K_SINGLE

DEV = "cuda"
F32 = torch.float32
TILE_SAMPLE, TILE_LATENT, TILE_OVERLAP = 512, 64, 0.25  # the SD-1.5 checkpoint's tiling (sample_size 512)

# (what, nb, H, W, tiled): image H x W; a decode runs on the H / 8 x W / 8 latent
VAE_SHAPES = [
    ("encode", 8, 512, 512, False), ("decode", 8, 512, 512, False),      # bench C2
    ("encode", 4, 512, 512, False), ("decode", 4, 512, 512, False),      # bench C3
    ("encode", 2, 1024, 1024, False), ("decode", 2, 1024, 1024, False),  # bench C4: hw = 16384 per image
    ("encode", 2, 512, 512, False), ("decode", 2, 512, 512, False),      # bench C5
    ("encode", 1, 640, 856, False), ("decode", 1, 640, 856, False),      # app canvas: 80 x 107 latent
    ("encode", 2, 640, 856, False), ("decode", 2, 640, 856, False),      # hw = 8560, hw % 128 != 0, two images
    ("encode", 2, 648, 856, False), ("decode", 2, 648, 856, False),      # 81 x 107: hw_ld != hw
    ("encode", 1, 512, 2048, False), ("decode", 1, 512, 2048, False),    # hw = 16384, not square
    ("encode", 1, 1536, 1024, True), ("decode", 1, 1536, 1024, True),    # tiled: 4 x 3 tiles of 512^2 / 64^2
]
# the op kinds the VAE programs record; a new kind fails the census until it is checked here
VAE_KINDS = {"gemm", "gn", "softmax_rows", "upsample_nearest", "memset", "window_copy", "tile_blend"}


def _label(what, nb, H, W, tiled):
    return f"{'tiled ' if tiled else ''}{what} {nb}x{H}x{W}"


# =========================================================================== CPU
def test_shape_list_covers_the_bench_and_the_app():
    """every bench.py config's e2e encode and decode is in VAE_SHAPES (a new config fails here until it is added),
    and so are the app canvases, a non-square hw = 16384 and a tiled canvas at the checkpoint's tile sizes"""
    import bench

    for name, cfg in bench.CONFIGS.items():
        side = 8 * cfg["latent"]
        for what in ("encode", "decode"):
            assert (what, cfg["batch"], side, side, False) in VAE_SHAPES, (name, what)
    for what in ("encode", "decode"):
        for nb, H, W in ((1, 640, 856), (2, 640, 856), (2, 648, 856), (1, 512, 2048)):
            assert (what, nb, H, W, False) in VAE_SHAPES
        assert (what, 1, 1536, 1024, True) in VAE_SHAPES
    lat = {(nb, H // 8, W // 8) for _, nb, H, W, tiled in VAE_SHAPES if not tiled}
    assert (2, 128, 128) in lat and (1, 64, 256) in lat      # hw = 16384, square and not
    assert (2, 80, 107) in lat and 80 * 107 % 128 != 0        # GroupNorm images straddle 128-row m-tiles
    assert (2, 81, 107) in lat and 81 * 107 % 8 != 0          # the attention's pitch hw_ld != hw


def test_latent_limit_of_the_untiled_vae():
    """_check_latent takes 16384 latent pixels and refuses 16385 with its message; every untiled shape of the list is
    inside the limit and the tiled canvas is not"""
    from powerpaint_b200.models.autoencoder_kl import VAE_MAX_LATENT_PIXELS, VaeEngine

    assert VAE_MAX_LATENT_PIXELS == 16384
    eng = object.__new__(VaeEngine)  # the check reads no engine state: no device needed
    eng._check_latent(128, 128, "decode")
    eng._check_latent(64, 256, "encode")
    with pytest.raises(RuntimeError, match=r"a 5x3277 latent has 16385 pixels, above the 16384 .*enable_vae_tiling"):
        eng._check_latent(5, 3277, "decode")
    for what, nb, H, W, tiled in VAE_SHAPES:
        if tiled:
            with pytest.raises(RuntimeError, match="enable_vae_tiling"):
                eng._check_latent(H // 8, W // 8, what)
        else:
            eng._check_latent(H // 8, W // 8, what)


def test_tiled_canvas_needs_more_than_one_chunk():
    """the tiled 1536 x 1024 canvas: 4 x 3 tiles (six of them full 512^2 tiles) whose encoded / decoded images add up
    to more than TILE_CHUNK_PIXELS, so its plan runs the encoder / decoder in several passes (the passes the engine
    actually records are counted by the GPU census)"""
    from powerpaint_b200.models.autoencoder_kl import VaeEngine, vae_tile_geometry

    assert VaeEngine.TILE_CHUNK_PIXELS == 4 * 512 * 512
    for encode in (True, False):
        h, w = (1536, 1024) if encode else (192, 128)
        geom = vae_tile_geometry(encode, h, w, TILE_SAMPLE, TILE_LATENT, TILE_OVERLAP, 8)
        assert (geom.rows, geom.cols, geom.out_h, geom.out_w) == ((4, 3, 192, 128) if encode else (4, 3, 1536, 1024))
        full = (512, 512) if encode else (64, 64)
        assert len(geom.groups()[full]) == 6
        pixels = sum(t.h * t.w if encode else t.out_h * t.out_w for t in geom.tiles)
        assert pixels > VaeEngine.TILE_CHUNK_PIXELS, pixels


def test_attention_out_projection_emits_records_only_at_whole_m_tiles():
    """the attention's to_out GEMM asks for GroupNorm partial records with rows_per_group = hw. At hw % 128 != 0 a
    128-row m-tile straddles two images, so the library declines (the host-only geometry query) and the GroupNorm
    that reads the output computes standalone statistics; at the bench's hw it emits records"""
    from powerpaint_b200 import ops as o

    for hw, ok in ((4096, True), (16384, True), (80 * 107, False), (81 * 107, False), (80 * 64, True)):
        d = fake_desc(dict(M=2 * hw, N=512, K=512, bias=True, res1=True), 0)
        d.rows_per_group = hw
        assert bool(o.gemm_stats_geometry(o.Desc("gemm", d, None)).supported) == ok, hw


# =========================================================================== GPU fixtures and blocked checkers
@pytest.fixture(scope="module")
def ops():
    from powerpaint_b200 import _native, ops as o

    assert _native.lib().pp_device_supported() == 1, "tests need an sm_90 (H100) device"
    return o


@pytest.fixture(autouse=True)
def _fp64_references(monkeypatch):
    """fp32 references without TF32; the GEMM references in blocks of 2048 output rows (a 16384^2 fp64 score block
    and its bound would otherwise take 10 GB at a time)"""
    import test_kernel_variants_gpu as kv

    row_chunks = kv._row_chunks
    monkeypatch.setattr(kv, "_row_chunks", lambda d, rows_per_chunk=2048: row_chunks(d, rows_per_chunk))
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _vae():
    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    vae = AutoencoderKL.synthetic(seed=4321, sample_size=TILE_SAMPLE).to(DEV)
    assert (vae.tile_sample_min_size, vae.tile_latent_min_size, vae.tile_overlap_factor) == \
        (TILE_SAMPLE, TILE_LATENT, TILE_OVERLAP)
    return vae


def _plan_of(vae, what, nb, H, W, tiled):
    e = vae.engine()
    encode = what == "encode"
    h, w = (H, W) if encode else (H // 8, W // 8)
    if tiled:
        return e.tiled_plan(encode, nb, h, w, vae.tile_geometry(encode, h, w), vae._tiling_key())
    return e.encode_plan(nb, h, w) if encode else e.decode_plan(nb, h, w)


def check_gn_outputs(name, x, y, st, gamma, beta, silu, groups, chain, eps, pixels=1 << 18):
    """check_gn_stats and gn_y_ref of the norm census on x / y [nb, hw, C], the statistics per image and y in blocks
    of `pixels` pixels; returns the worst err / bound"""
    nb, hw, C = x.shape
    per = [gn_truth(x[b:b + 1], groups) for b in range(nb)]
    truth = tuple(torch.cat([p[k] for p in per]) for k in range(4)) + (per[0][4],)
    worst = max(check_gn_stats(name, st, truth, chain, eps))
    for b in range(nb):
        for p0 in range(0, hw, pixels):
            xb = x[b:b + 1, p0:p0 + pixels]
            ref, bound = gn_y_ref(xb, st[b:b + 1], gamma, beta, silu)
            got = y[b:b + 1, p0:p0 + pixels].reshape(-1, C)
            worst = max(worst, assert_within(f"{name} y image {b} pixels {p0}+", got, ref.view(-1, C),
                                             bound.view(-1, C)))
    return worst


def check_group_norm_blocked(ops, name, x0, groups, eps, silu, gamma, beta, chain, parts=None):
    y, st = run_group_norm(ops, name, x0, None, groups, eps, silu, gamma, beta, parts)
    return check_gn_outputs(name, x0, y, st, gamma, beta, silu, groups, chain, eps)


def check_softmax_rows_blocked(name, s, p, rows=2048):
    """ref_softmax of the norm census over blocks of `rows` rows of the fp32 scores s against the bf16 p"""
    per = softmax_instance(s.shape[1])
    worst = 0.0
    for r0 in range(0, s.shape[0], rows):
        ref, bound = ref_softmax(s[r0:r0 + rows], per)
        worst = max(worst, assert_within(f"{name} rows {r0}+", p[r0:r0 + rows], ref, bound))
    return worst


def _eval_gn_blocked(name, op, mem, before, after):
    """test_program_replay_gpu.eval_gn with the blocked fp64 evaluation (the VAE's GroupNorms read one source)"""
    d = op.c
    assert not d.x1, name
    nb, hw, C = d.batch, d.hw, d.c0
    x = mem.view(before, d.x0, nb * hw * C, BF16).view(nb, hw, C)
    y = mem.view(after, d.y, nb * hw * C, BF16).view(nb, hw, C)
    st = mem.view(after, d.stats, nb * d.groups * 2, F32).view(nb, d.groups, 2)
    gamma, beta = mem.view(before, d.gamma, C, F32), mem.view(before, d.beta, C, F32)
    chain = producer_chain(d.geom0) if d.from_partials else standalone_chain(nb, hw, C, d.groups)
    check_gn_outputs(name, x, y, st, gamma, beta, bool(d.silu), d.groups, chain, d.eps)


def _eval_softmax_blocked(name, op, mem, before, after):
    a = op.args
    rows, cols = a["rows"], a["cols"]
    s = mem.mat(before, a["s"].data_ptr(), rows, cols, a["ld_s"], F32)
    p = mem.mat(after, a["p"].data_ptr(), rows, cols, a["ld_p"], BF16)
    check_softmax_rows_blocked(name, s, p)


def _run_checked(prog, op, tensors, name):
    """run the one-op program `prog` once on fresh tensors and check it as the replay checks an op: nothing outside its
    write footprint moved, and its outputs equal the replay's evaluation of the op on its inputs"""
    mem = Memory(tensors)
    before = mem.snapshot()
    prog.run()
    torch.cuda.synchronize()
    after = mem.snapshot()
    _, W = footprint(op)
    moved = (before != after) & ~mem.mask(W)
    assert not moved.any(), f"{name}: {int(moved.sum())} bytes changed outside the write footprint"
    EVALUATORS[op.kind](name, op, mem, before, after)


# =========================================================================== GPU: static dataflow
@pytest.mark.gpu
def test_static_dataflow_of_the_vae_programs(ops):
    """every plan of VAE_SHAPES, recorded with the recycling pool and with one that never recycles: the same last
    writer of every byte every op reads (the per-image attention loop reuses one S and one P buffer)"""
    vae = _vae()
    e = vae.engine()
    for shape in VAE_SHAPES:
        t0 = time.perf_counter()
        torch.cuda.reset_peak_memory_stats()
        n = _static_plan(lambda: (e._plans.clear(), _plan_of(vae, *shape))[1], _label(*shape))
        e._plans.clear()
        torch.cuda.empty_cache()
        print(f"[vae static] {_label(*shape)}: {n} reads, same writers ({time.perf_counter() - t0:.1f} s, peak "
              f"allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB)")


# =========================================================================== GPU: census
class _VaeCensus:
    """the GEMM / attention census of test_kernel_variants_gpu.py, the op census of the norm file, the byte counts of
    the memsets (the op census keys a memset by its kind only) and, per plan, the batch of every conv_in launch (one per
    recorded encoder / decoder pass: its input has the 8 padded image / latent channels)"""

    def __init__(self):
        self.gemm, self.ops, self.memsets, self.passes = _Census(), OpCensus(), {}, {}

    def record(self, source, op):
        self.gemm.record(source, op)
        self.ops.record(source, op)
        if op.kind == "gemm" and op.c.a_mode == 1 and op.c.c0 == 8:
            self.passes.setdefault(source, []).append(op.c.nb)
        if op.kind == "memset":
            t = op.args["t"]
            self.memsets.setdefault(t.numel() * t.element_size(), source)


@pytest.fixture(scope="module")
def census(ops):
    c = _VaeCensus()
    vae = _vae()
    e = vae.engine()
    for shape in VAE_SHAPES:
        with pytest.MonkeyPatch.context() as mp:
            cap = Capture(mp)
            _plan_of(vae, *shape)
        for key in cap.ops:
            for op in cap.of(cap.programs[key]):
                c.record(_label(*shape), op)
        del cap
        e._plans.clear()
        torch.cuda.empty_cache()
    print(f"\n[vae census] {len(VAE_SHAPES)} plans: {len(c.gemm.sigs)} GEMM / attention signatures; "
          + ", ".join(f"{k} {n} records / {len(c.ops.sigs.get(k, {}))} signatures" for k, n in c.ops.records.items()))
    return c


def _gemm_limit(c, variant):
    """the limit shape a GEMM signature stands for, or None"""
    if c.a_mode == 0 and c.out_fp32 and c.M == 16384 and c.N == 16384:
        return "fp32 scores M = N = 16384"
    if c.a_mode == 0 and c.M == 16384 and c.N == 512 and c.c0 == PV_K_CHUNK and (c.rowvec or c.out_fp32):
        return f"PV chain over 16384 keys: {'fp32' if c.out_fp32 else 'bf16'} out, {'with' if c.rowvec else 'no'} " \
               "fp32 running sum"
    if variant[1] == 5 and c.M // c.t_rows > 1:
        return f"mode-5 store across {c.M // c.t_rows} images"
    if c.a_mode and c.chan_stats and gemm_out_geometry(c)[0] == 1 << 21:
        return "conv M = 2^21 with GroupNorm records"
    return None


@pytest.mark.gpu
def test_census_reaches_the_limits(census):
    """the recorded programs contain the limit shapes, so the checks below cannot silently fall back to small ones"""
    assert set(census.ops.records) <= VAE_KINDS, sorted(set(census.ops.records) - VAE_KINDS)
    gemms = [(c, v) for kind, c, v, _, _ in census.gemm.sigs.values() if kind == "gemm"]
    limits = {_gemm_limit(c, v) for c, v in gemms}
    for what in ("fp32 scores M = N = 16384", "conv M = 2^21 with GroupNorm records",
                 "PV chain over 16384 keys: fp32 out, no fp32 running sum",
                 "PV chain over 16384 keys: fp32 out, with fp32 running sum",
                 "PV chain over 16384 keys: bf16 out, with fp32 running sum"):
        assert what in limits, what
    # no single GEMM sums over more than PV_K_SINGLE keys
    assert not [c for c, _ in gemms if c.a_mode == 0 and c.c0 > PV_K_SINGLE and not c.out_fp32], "PV over > 4096 keys"
    assert any(x and x.startswith("mode-5 store across") for x in limits), limits
    assert any(a["cols"] == 16384 and a["rows"] == 16384 for a, _ in census.ops.sigs["softmax_rows"].values())
    gns = [c for c, _ in census.ops.sigs["gn"].values()]
    assert any(c.hw == 1 << 20 and c.batch == 2 for c in gns)
    assert any(c.hw == 1 << 20 and c.from_partials for c in gns)
    # hw % 128 != 0 at nb > 1: the attention's to_out GEMM requested records (rows_per_group = hw) and got none, so
    # the GroupNorm reading its output runs the standalone statistics pass
    odd = {c.rows_per_group for c, _ in gemms
           if c.a_mode == 0 and not c.rowvec and c.rows_per_group % 128 and c.M > c.rows_per_group}
    assert {80 * 107, 81 * 107} <= odd, odd
    assert not any(c.chan_stats for c, _ in gemms if c.a_mode == 0 and c.rows_per_group in odd)
    for hw in (80 * 107, 81 * 107):
        at = [c for c in gns if c.hw == hw and c.batch == 2]
        assert any(not c.from_partials for c in at) and any(c.from_partials for c in at), hw
    # the attention's V^T and P pads at hw_ld != hw are cleared before use
    assert 81 * 107 * 8672 * 2 in census.memsets and 2 * 512 * 8672 * 2 in census.memsets
    assert census.ops.sigs.get("window_copy") and census.ops.sigs.get("tile_blend")
    # the tiled canvas: its 12 tiles in several recorded passes, the full tiles four to a pass (TILE_CHUNK_PIXELS)
    for what in ("encode", "decode"):
        passes = census.passes[_label(what, 1, 1536, 1024, True)]
        print(f"[vae census] tiled {what} 1536x1024: encoder / decoder passes of {passes} tiles")
        assert len(passes) > 1 and max(passes) == 4 and sum(passes) == 12, passes


@pytest.mark.gpu
def test_census_gemm(ops, census):
    """every distinct GEMM (and attention) signature the VAE programs record, on fresh seeded inputs against the fp64
    bound, twice, bit-identical"""
    worst_all, n = 0.0, 0
    for i, (kind, c0, variant, source, meta) in enumerate(census.gemm.sigs.values()):
        name = f"vae census #{i} {kind} {variant} from {source}"
        if kind == "gemm":
            desc, t, outs, canv, extra = _fresh_gemm(c0, variant, seed=3000 + i)
            assert ops.gemm_variant(desc) == variant, name
            ops.run(desc)
            torch.cuda.synchronize()
            first = {k: v.clone() for k, v in outs.items()}
            worst = check_gemm(name, desc.c, t, outs, canv, variant[0])
        else:
            desc, t, canv = _fresh_attention(c0, meta.get("k_minus_q"), seed=3000 + i)
            assert ops.attention_variant(desc) == variant, name
            outs, extra = {"out": canv["out"].view}, {}
            ops.run(desc)
            torch.cuda.synchronize()
            first = {"out": outs["out"].clone()}
            worst = check_attention(name, desc.c, t, outs["out"], canv)
        assert_rerun_identical(ops, name, desc, outs, first, canv, extra)
        worst_all, n = max(worst_all, worst), n + 1
        c = desc.c
        if kind == "gemm":
            lim = _gemm_limit(c0, variant)
            shape = (f"M={gemm_out_geometry(c)[0]} N={c.N} K={c.c0}+{c.c1} a_mode={c.a_mode} epi={c.epilogue} "
                     f"fp32={c.out_fp32} stats={bool(c0.chan_stats)}")
        else:
            lim, shape = None, f"B={c.batch} H={c.heads} d={c.d} nq={c.nq} nk={c.nk}"
        print(f"[vae census{' limit: ' + lim if lim else ''}] #{i} {kind} {variant} {shape} ({source}) "
              f"worst err/bound = {worst:.3f}")
        del desc, t, outs, canv, extra, first
        torch.cuda.empty_cache()
    print(f"[vae census] {n} GEMM / attention signatures, worst err/bound = {worst_all:.3f}")


@pytest.mark.gpu
def test_census_group_norm(ops, census):
    """every distinct GroupNorm: the standalone statistics pass, and for one recorded over its producer's epilogue
    records also the finalize over the records of that producer GEMM rebuilt fresh"""
    sigs = census.ops.sigs["gn"]
    worst = {"standalone": 0.0, "producer": 0.0}
    for i, (c, meta) in enumerate(sigs.values()):
        nb, hw, C, groups = c.batch, c.hw, c.c0, c.groups
        assert not c.c1
        name = f"vae census gn #{i} ({meta['source']}) batch={nb} hw={hw} C={C} silu={c.silu}"
        gamma, beta = _gn_params(C, 7000 + i)
        paths = []
        if c.from_partials:
            assert len(meta["producers"]) == 1 and meta["producers"][0] is not None, f"{name}: producer not captured"
            (gc, variant), = meta["producers"]
            desc, _, outs, _, extra = _fresh_gemm(gc, variant, seed=8000 + i)
            assert desc.c.ldc == desc.c.N and gemm_out_geometry(desc.c)[0] == nb * hw, name
            geo = ops.gemm_stats_geometry(desc)
            assert _geom_tuple(geo) == _geom_tuple(c.geom0), name
            ops.run(desc)
            torch.cuda.synchronize()
            x0 = outs["out"].view(nb, hw, C)
            w = check_group_norm_blocked(ops, f"{name} producer", x0, groups, c.eps, bool(c.silu), gamma, beta,
                                         producer_chain(geo), parts=[(extra["part"], geo)])
            worst["producer"] = max(worst["producer"], w)
            paths.append(f"producer {w:.3f}")
        else:
            x0 = _randn_bf16((nb, hw, C), 9000 + i)
        w = check_group_norm_blocked(ops, f"{name} standalone", x0, groups, c.eps, bool(c.silu), gamma, beta,
                                     standalone_chain(nb, hw, C, groups))
        worst["standalone"] = max(worst["standalone"], w)
        paths.append(f"standalone {w:.3f}")
        lim = " limit: hw = 2^20" if hw == 1 << 20 else " limit: hw % 128 != 0, nb > 1" if hw % 128 and nb > 1 else ""
        print(f"[vae census gn{lim}] #{i} batch={nb} hw={hw} C={C} silu={c.silu} "
              f"{'from_partials' if c.from_partials else 'standalone'} ({meta['source']}): worst err/bound "
              + ", ".join(paths))
        x0 = None
        torch.cuda.empty_cache()
    print(f"[vae census gn] {len(sigs)} signatures; worst err/bound per path: "
          + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.gpu
def test_census_small_ops(ops, census):
    """every distinct softmax_rows, upsample, memset, window copy and tile blend the VAE programs record, on fresh
    inputs; the image pre- and post-processing kernels at every canvas of the list"""
    import numpy as np

    sig = census.ops.sigs
    for i, (a, meta) in enumerate(sig["softmax_rows"].values()):
        rows, cols, ld_s, ld_p = a["rows"], a["cols"], a["ld_s"], a["ld_p"]
        buf, s = _softmax_scores(rows, cols, ld_s, 500 + i)
        canv = Canvas(rows, cols, ld_p, BF16, DEV, pad_rows=4)
        runs = []
        for _ in range(2):
            canv.view.fill_(float("nan"))
            ops.softmax_rows(s, canv.view)
            torch.cuda.synchronize()
            runs.append(canv.view.clone())
        assert torch.equal(_bits(runs[0]), _bits(runs[1])), f"softmax #{i}: two runs differ"
        assert_canvases(f"softmax #{i}", {"p": canv})
        w = check_softmax_rows_blocked(f"vae census softmax #{i}", s, canv.view)
        lim = " limit: 16384 columns" if cols == 16384 else ""
        print(f"[vae census softmax_rows{lim}] #{i} rows={rows} cols={cols} ld_p={ld_p} ({meta['source']}) "
              f"worst err/bound = {w:.3f}")
        del buf, s, canv, runs
        torch.cuda.empty_cache()
    for i, (a, meta) in enumerate(sig["upsample_nearest"].values()):
        check_upsample(f"vae census upsample #{i}", a["nb"], a["h"], a["w"], a["c"], a["ho"], a["wo"], 400 + i)
        print(f"[vae census upsample_nearest #{i}] {a['nb']}x{a['h']}x{a['w']}x{a['c']} -> {a['ho']}x{a['wo']} "
              f"({meta['source']}) exact")
        torch.cuda.empty_cache()
    for nbytes, source in sorted(census.memsets.items()):
        pad = 256
        buf = torch.full((nbytes + 2 * pad,), 0xA5, dtype=torch.uint8, device=DEV)
        t = buf[pad:pad + nbytes]
        prog = ops.Program()
        prog.add_memset(t)
        _run_checked(prog, ProgramCall("memset", {"t": t}), [buf], f"memset {nbytes} bytes")
        assert (buf[:pad] == 0xA5).all() and (buf[pad + nbytes:] == 0xA5).all()
        print(f"[vae census memset] {nbytes} bytes ({source}) zero, nothing outside")
    g = torch.Generator(device=DEV).manual_seed(21)
    for i, (a, meta) in enumerate(sig["window_copy"].values()):
        wl = a["wl"]
        src = (torch.randn(wl.src.shape, device=DEV, generator=g) * 3).to(wl.src.dtype)
        dst = torch.full(wl.dst.shape, SENTINEL, dtype=wl.dst.dtype, device=DEV)
        wins = [(w.src_off, w.dst_off, w.src_row, w.dst_row, w.rows, w.cols) for w in _windows(wl)]
        fresh = ops.WindowList(src, dst, wl.channels, wins, wl.src_pix, wl.dst_pix)
        prog = ops.Program()
        prog.add_window_copy(fresh)
        _run_checked(prog, ProgramCall("window_copy", {"wl": fresh}), [src, dst], f"window_copy #{i}")
        print(f"[vae census window_copy #{i}] {wl.count} windows of {wl.channels} x {wl.src.dtype} channels, up to "
              f"{wl.max_pixels} pixels ({meta['source']}) exact")
    for i, (c, meta) in enumerate(sig["tile_blend"].values()):
        b = torch.randn(c.batch, c.b_h, c.b_w, c.channels, device=DEV, generator=g) * 4
        av = torch.randn(c.batch, c.av_h, c.b_w, c.channels, device=DEV, generator=g) * 4 if c.e_v else None
        ah = torch.randn(c.batch, c.b_h, c.ah_w, c.channels, device=DEV, generator=g) * 4 if c.e_h else None
        desc = ops.tile_blend_desc(b, av, ah, c.e_v, c.e_h)
        prog = ops.Program()
        prog.add(desc)
        _run_checked(prog, desc, [t for t in (b, av, ah) if t is not None], f"tile_blend #{i}")
        print(f"[vae census tile_blend #{i}] batch={c.batch} {c.b_h}x{c.b_w}x{c.channels} e_v={c.e_v} e_h={c.e_h} "
              f"({meta['source']}) exact")
    # image pre-processing (uint8 image + uint8 mask -> bf16 NHWC) over every encoded canvas, post-processing (fp32
    # NHWC -> uint8 NHWC / fp32 NCHW) over every decoded one: bit for bit
    for nb, H, W in sorted({(nb, H, W) for what, nb, H, W, _ in VAE_SHAPES if what == "encode"}):
        img = torch.randint(0, 256, (nb, 3, H, W), device=DEV, generator=g, dtype=torch.uint8)
        mask = torch.randint(0, 256, (nb, 1, H, W), device=DEV, generator=g, dtype=torch.uint8)
        got = ops.image_preprocess_u8(img, mask, c_pad=8)
        torch.cuda.synchronize()
        v = img.cpu().numpy().reshape(nb, 3, H * W).transpose(0, 2, 1).astype(np.float32) / np.float32(127.5) \
            + np.float32(-1.0)
        v = v * ((mask.cpu().numpy().reshape(nb, H * W, 1).astype(np.float32) / np.float32(255)) < np.float32(0.5))
        ref = torch.zeros(nb, H * W, 8, dtype=BF16)
        ref[..., :3] = torch.from_numpy(np.ascontiguousarray(v)).to(BF16)
        assert torch.equal(_bits(got.cpu()), _bits(ref)), f"image_preprocess {nb}x{H}x{W}"
        print(f"[vae census image_preprocess] {nb}x{H}x{W} exact")
    for nb, H, W in sorted({(nb, H, W) for what, nb, H, W, _ in VAE_SHAPES if what == "decode"}):
        x = torch.randn(nb, H * W, 4, device=DEV, generator=g) * 1.5
        u8 = ops.image_postprocess(x, nb, H, W, uint8=True)
        f = ops.image_postprocess(x, nb, H, W, uint8=False)
        torch.cuda.synchronize()
        want_u8, want_f = ref_postprocess_u8(x[..., :3])
        assert torch.equal(u8.cpu().view(nb, H * W, 3), want_u8), f"image_postprocess uint8 {nb}x{H}x{W}"
        assert torch.equal(_bits(f.cpu()), _bits(want_f.permute(0, 2, 1).reshape(nb, 3, H, W))), \
            f"image_postprocess fp32 {nb}x{H}x{W}"
        print(f"[vae census image_postprocess] {nb}x{H}x{W} exact")


# =========================================================================== GPU: replay
# (what, nb, H, W, tiled). C4 replays one 1024^2 image: the replay keeps two byte snapshots of all tracked storage and
# their byte masks on the device, about six times the plan's footprint; the census and static dataflow above run C4 at
# its bench batch of 2, and 8 x 512^2 replays the same activation volume as 2 x 1024^2 with batch > 1.
REPLAY_CASES = [("decode", 1, 1024, 1024, False), ("encode", 1, 1024, 1024, False), ("decode", 8, 512, 512, False),
                ("encode", 2, 648, 856, False), ("decode", 2, 648, 856, False), ("encode", 1, 1536, 1024, True),
                ("decode", 1, 1536, 1024, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("what,nb,H,W,tiled", REPLAY_CASES, ids=[_label(*c).replace(" ", "-") for c in REPLAY_CASES])
def test_replay_vae_op_by_op(ops, what, nb, H, W, tiled):
    """vae.encode / vae.decode on synthetic SD-width weights, every op checked as it runs: nothing outside its write
    footprint moves, its outputs equal the fp64 evaluation of its contract on the inputs it read"""
    vae = _vae()
    if tiled:
        vae.enable_tiling()
    g = torch.Generator(device=DEV).manual_seed(H + W + nb)
    if what == "encode":
        x = torch.rand(nb, 3, H, W, device=DEV, generator=g) * 2 - 1
        call = lambda: vae.encode(x).latent_dist.mean  # noqa: E731
    else:
        x = torch.randn(nb, 4, H // 8, W // 8, device=DEV, generator=g)
        call = lambda: vae.decode(x).sample  # noqa: E731
    vae.engine()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with pytest.MonkeyPatch.context() as mp:
        mp.setitem(EVALUATORS, "gn", _eval_gn_blocked)
        mp.setitem(EVALUATORS, "softmax_rows", _eval_softmax_blocked)
        rp = Replay(mp)
        out = call()
        torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated()
    assert torch.isfinite(out).all()
    want = {"gemm", "gn", "softmax_rows"} | ({"window_copy", "tile_blend"} if tiled else set()) \
        | ({"upsample_nearest"} if what == "decode" else set())
    assert want <= set(rp.kinds), rp.kinds
    print(f"[vae replay] {_label(what, nb, H, W, tiled)}: {rp.ops_run} ops checked, kinds {rp.kinds}; "
          f"tracked storage {rp.mem.total / 2**30:.2f} GiB, peak allocated {peak / 2**30:.2f} GiB, {dt:.1f} s")


# =========================================================================== GPU: P V over 16384 keys
def _pv_errors(p, vt, got, rows=2048):
    """worst err / bound of got = P V against fp64 under the single-GEMM census bound U16 |PV| + C_ACC P |V|, and the
    mean signed error relative to that magnitude (a one-sided accumulation drift shows here, rounding noise does not)"""
    v, va = vt.double().t(), vt.double().abs().t()
    worst, signed, n = 0.0, 0.0, 0
    for r0 in range(0, p.shape[0], rows):
        pd = p[r0:r0 + rows].double()
        ref, mag = pd @ v, pd @ va
        bound = U16 * ref.abs() + C_ACC * mag + 1e-30
        g = got[r0:r0 + rows].double()
        worst = max(worst, ((g - ref).abs() / bound).max().item())
        signed += ((g - ref) / mag).sum().item()
        n += g.numel()
    return worst, signed / n


@pytest.mark.gpu
def test_pv_product_over_16384_keys_on_softmax_weights(ops):
    """the attention's O = P V at hw = 16384 on what it multiplies in the VAE: rows of softmax weights (non-negative,
    each summing to one) against values with a non-zero mean. The chain add_pv_product records stays within the
    census bound of one GEMM (U16 |PV| + 2^-16 P |V|) on every element; one GEMM over all 16384 keys, on the same
    inputs, is measured alongside and printed"""
    from powerpaint_b200.models.autoencoder_kl import add_pv_product

    hw, C = 16384, 512
    g = torch.Generator(device=DEV).manual_seed(16384)
    s = torch.randn(hw, hw, device=DEV, generator=g) * 2
    p = torch.empty(hw, hw, device=DEV, dtype=BF16)
    ops.softmax_rows(s, p)
    del s
    vt = (torch.randn(C, hw, device=DEV, generator=g) * 0.5 + 1.0).to(BF16)
    part = (torch.empty(hw, C, device=DEV, dtype=F32), torch.empty(hw, C, device=DEV, dtype=F32))
    canv = Canvas(hw, C, C, BF16, DEV, pad_rows=8)
    prog = ops.Program()
    add_pv_product(prog, p, vt, canv.view, part)
    assert prog.num_ops == hw // PV_K_CHUNK
    prog.run()
    torch.cuda.synchronize()
    assert_canvases("PV chain", {"out": canv})
    v = vt.double().t()
    for r0 in range(0, hw, 2048):
        pd = p[r0:r0 + 2048].double()
        ref = pd @ v
        assert_within(f"PV chain rows {r0}+", canv.view[r0:r0 + 2048], ref,
                      U16 * ref.abs() + C_ACC * (pd @ v.abs()) + 1e-30)
    w_chain, d_chain = _pv_errors(p, vt, canv.view)
    one = torch.empty(hw, C, device=DEV, dtype=BF16)
    ops.run(ops.gemm_desc(a0=p, c0=hw, lda0=hw, w=vt, ldb=hw, out=one, N_=C, M=hw))
    torch.cuda.synchronize()
    w_one, d_one = _pv_errors(p, vt, one)
    print(f"[vae PV 16384 keys] chain of {prog.num_ops} GEMMs: worst err/bound = {w_chain:.3f}, mean signed error "
          f"{d_chain:+.2e} of P|V|; one GEMM: worst err/bound = {w_one:.3f}, mean signed error {d_one:+.2e} of P|V|")


# =========================================================================== GPU: end to end
@pytest.mark.gpu
def test_vae_2x1024_matches_the_fp32_oracle(ops):
    """bench C4's VAE work, 2 x 1024^2, against oracle/vae.py in fp32 (TF32 off): moments and the decoded image within
    test_vae_gpu.py's rel-L2 <= 3e-2, the uint8 output within one step of the float output rounded"""
    from test_vae_gpu import _pair, _rel

    om, pm = _pair(False)
    g = torch.Generator(device=DEV).manual_seed(1024)
    x = torch.rand(2, 3, 1024, 1024, device=DEV, generator=g) * 2 - 1
    with torch.no_grad():
        ref_mean, ref_logvar = om.quant_conv(om.encoder(x)).chunk(2, 1)
    d = pm.encode(x).latent_dist
    assert d.mean.shape == ref_mean.shape == (2, 4, 128, 128)
    e_mean, e_logvar = _rel(d.mean, ref_mean), _rel(d.logvar, ref_logvar.clamp(-30, 20))
    assert e_mean < 3e-2 and e_logvar < 3e-2, (e_mean, e_logvar)
    del x, d, ref_mean, ref_logvar
    pm.engine()._plans.clear()
    torch.cuda.empty_cache()
    z = torch.randn(2, 4, 128, 128, device=DEV, generator=g)
    with torch.no_grad():
        ref_img = om.decode(z, return_dict=False)[0]
    img = pm.decode(z, return_dict=False)[0]
    assert img.shape == ref_img.shape == (2, 3, 1024, 1024) and torch.isfinite(img).all()
    e_img = _rel(img, ref_img)
    assert e_img < 3e-2, e_img
    u8 = pm.decode_postprocessed(z, uint8=True)
    want = ((img / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8).permute(0, 2, 3, 1)
    assert u8.shape == (2, 1024, 1024, 3)
    assert (u8.int() - want.int()).abs().max().item() <= 1
    print(f"[vae e2e 2x1024^2] rel-L2 moments mean {e_mean:.2e} logvar {e_logvar:.2e}, image {e_img:.2e}")
