"""The GEMM / conv kernel at the edges of its schedule, where the hand-over protocol modelled in
test_gemm_protocol_model.py is exercised hardest:

  * one k-iteration per tile (K = 64) with a staged res1 (and a staged row vector) and several tiles per CTA: the
    producer runs whole tiles ahead on the ring, so its residual polls interleave most with its ring waits;
  * k-iterations per tile equal to STAGES and STAGES + 1: the ring phase flips exactly at a tile boundary;
  * tile counts of SMs + 1 and 2 x SMs + 1: CTAs walk different numbers of tiles;
  * mode 3 with one n-tile per row block, and with three, where a CTA's consecutive tiles lie in different row blocks
    (the verdict is collected a tile late), each then replayed twice from a CUDA graph;
  * split-K at the largest tile count the chooser still splits, then replayed.

Each case runs once. It asserts its variant through pp_gemm_variant and the tiles per CTA it means to reach (from the
device's SM count, the one the launch takes) and, through pp_gemm_staging, that res1 (and the row vector) take the
shared-memory path while the register route does not; it is checked element by element against fp64 (check_gemm of
test_kernel_variants_gpu), and where a register route exists (res1 moved to res2 at alpha 1; the row vector spread
over 64-row groups) bit for bit against it. The CPU test checks the split-K precondition: the owner spins on a flag
the donor CTA sets, so every split launch must fit the SMs in one wave.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gemm_residual_stage_gpu as rs  # noqa: E402
import test_kernel_variants_gpu as kv  # noqa: E402

ops = kv.ops  # the device check and the ops module, as a fixture

STAGES = {64: 8, 128: 5, 160: 5, 256: 3}  # stages_for() of gemm_conv.cu (pinned by test_gemm_protocol_model.py)


def _cdiv(a, b):
    return (a + b - 1) // b


def _cases(sms):
    """(id, variant, route, spec, tiles, replay) for a GPU with `sms` SMs"""
    cases = []

    def add(cid, variant, route, m_tiles, n_tiles, replay=False, **spec):
        bn = variant[0]
        spec = dict(spec, M=128 * m_tiles - spec.pop("m_short", 37), N=n_tiles * bn - spec.pop("n_short", 8), _bn=bn)
        cases.append((cid, variant, route, spec, m_tiles * n_tiles, replay))

    mt = _cdiv(3 * sms + 5, 2)  # two n-tiles: at least three tiles per CTA, the last wave partial
    for bn in (64, 128, 160, 256):
        for mode in (0, 3):
            st = dict(row_stats=True) if mode == 3 else {}
            add(f"k1-res-bn{bn}-m{mode}", (bn, mode, 1), "res2", mt, 2, K=64, bias=True, res1=True, **st)
            add(f"k1-res-rv-bn{bn}-m{mode}", (bn, mode, 1), "rpg64", mt, 2, K=64, bias=True, res1=True, rowvec=True,
                rpg=256, **st)
    for bn in (64, 160, 256):
        for kit in (STAGES[bn], STAGES[bn] + 1):  # the ring phase flips at the end of the first / inside the second tile
            add(f"ring-k{kit}-bn{bn}", (bn, 0, 1), "res2", 2 * sms + 1, 1, K=64 * kit, bias=True, res1=True)
    add("walk-sms+1-m0", (128, 0, 1), "res2", sms + 1, 1, K=128, bias=True, res1=True)
    add("walk-sms+1-m3", (128, 3, 1), "res2", sms + 1, 1, K=128, bias=True, res1=True, row_stats=True)
    add("walk-2sms+1-m3", (160, 3, 1), "res2", 2 * sms + 1, 1, K=192, bias=True, res1=True, row_stats=True)
    # mode 3: one n-tile per row block; three, the row blocks of a CTA's consecutive tiles (stride = grid) all differ
    add("m3-n1", (128, 3, 1), "res2", sms + 7, 1, replay=True, K=128, bias=True, res1=True, row_stats=True)
    add("m3-n3", (128, 3, 1), "res2", sms + 3, 3, replay=True, K=128, bias=True, res1=True, row_stats=True)
    # split-K: two n-tiles of 160 and sms // 4 m-tiles, 2 x tiles work items: one more m-tile would not fit the SMs
    add("splitk-max", (160, 0, 2), "res2", sms // 4, 2, replay=True, m_short=5, K=64 * 40, splitk=True, bias=True,
        res1=True)
    return cases


CASES = _cases(kv.SMS)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles_per_cta(tiles, split, sms):
    if split:
        return 1, 1
    grid = min(tiles, sms)
    return tiles // grid, _cdiv(tiles, grid)


def _replay_twice(ops, cid, desc, outs, extra, eager):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.run(desc)
    torch.cuda.synchronize()
    for k in ("flags", "ticket"):  # the capture did not run the kernel; the eager runs left these at zero
        if k in extra:
            assert (extra[k] == 0).all(), (cid, k)
    for rep in range(2):
        for v in outs.values():
            v.fill_(float("nan"))
        for k in ("final", "rec"):  # row_final and the mode-3 records must be written again by the replay
            if k in extra:
                extra[k].fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        rs._assert_bits(f"{cid} graph replay {rep + 1}", eager, rs._snapshot(outs, extra))
        for k in ("flags", "ticket"):
            if k in extra:
                assert (extra[k] == 0).all(), f"{cid}: `{k}` not back at zero after graph replay {rep + 1}"


@pytest.mark.gpu
@pytest.mark.parametrize("cid,variant,route,spec,tiles,replay", CASES, ids=[c[0] for c in CASES])
def test_schedule_edge(ops, cid, variant, route, spec, tiles, replay):
    sms = _sms()
    if sms != kv.SMS:  # the shapes are chosen for this SM count
        cases = {c[0]: c for c in _cases(sms)}
        _, variant, route, spec, tiles, replay = cases[cid]
    desc, t, outs, canv, extra, fill, keep = rs._prepare(spec, variant, seed=sum(map(ord, cid)))
    d = desc.c
    bn, mode, ks = variant
    if ks == 2:
        d.block_n = 0  # the chooser's own pick, not a forced tile width
    assert ops.gemm_variant(desc) == variant, (cid, ops.gemm_variant(desc))
    n_tiles = _cdiv(d.N, bn)
    assert _cdiv(d.M, 128) * n_tiles == tiles, cid
    lo, hi = _tiles_per_cta(tiles, ks == 2, sms)
    if cid.startswith(("k1", "m3")):
        assert hi >= 2, (cid, tiles, sms)
    if cid.startswith("ring") or "2sms+1" in cid:
        assert (lo, hi) == (2, 3), (cid, tiles, sms)
    if "sms+1" in cid and "2sms" not in cid:
        assert (lo, hi) == (1, 2), (cid, tiles, sms)
    if cid == "m3-n3":  # a CTA's consecutive tiles, grid apart, lie in different row blocks
        grid = min(tiles, sms)
        assert grid >= n_tiles and all((c // n_tiles) != ((c + grid) // n_tiles) for c in range(grid)), cid
    if ks == 2:
        assert 2 * tiles <= sms, (cid, tiles, sms)
        bigger = kv.fake_desc(dict(spec, M=d.M + 128), 0)
        assert kv.query_gemm(bigger)[2] == 1, f"{cid}: the chooser still splits at {tiles + n_tiles} tiles"
    # the staged path this case is about, and a register route that does not take it
    staged = ops.gemm_staging(desc)
    assert staged == (True, bool(spec.get("rowvec"))), (cid, staged)
    want = None
    if route:
        reg = rs._register_route(ops, desc, t, route, keep)
        assert ops.gemm_staging(reg) == ((False, False) if route == "res2" else (True, False)), (cid, route)
        want = rs._run(ops, reg, outs, extra, fill)
    got = rs._run(ops, desc, outs, extra, fill)
    worst = kv.check_gemm(cid, d, t, outs, canv, bn)
    msg = f"[edge {cid}] variant {variant} tiles = {tiles} on {sms} SMs, {lo}..{hi} per CTA, worst err/bound = {worst:.3f}"
    if spec.get("row_stats"):
        e_rs, e_nm = kv._check_row_stats(cid, d, t, extra, bn)
        msg += f", row_final rel err = {e_rs:.2e} / {e_nm:.2e}"
    if "flags" in extra:
        assert (extra["flags"] == 0).all(), cid
    if want is not None:
        rs._assert_bits(cid, got, want)
        msg += f", bit-identical to the {route} route"
    if replay:
        assert fill is None
        _replay_twice(ops, cid, desc, outs, extra, got)
        msg += ", two graph replays bit-identical"
    print(msg)


# --------------------------------------------------------------------------- CPU
def test_the_staging_query_follows_the_kernels_predicate():
    """pp_gemm_staging restates the kernel's stage_res / stage_rv for the host: the same expression in both places, and
    its answers on the launches it separates"""
    src = kv._src("gemm_conv.cu")
    kernel_rv = "kRes && p.rowvec != nullptr && (p.a_mode == PP_A_MATRIX ? p.rows_per_group % BLOCK_M == 0 : p.bn == 1);"
    assert "const bool stage_res = kRes && p.res1 != nullptr && !(kSplitK && khalf);" in src
    assert kernel_rv in src and "constexpr bool kRes = MODE == 0 || MODE == 3;" in src
    host = src[src.index("static int gemm_staging("):]
    host = host[:host.index("\n}\n")]
    assert "const bool kRes = mode == 0 || mode == 3;" in host and "*stage_res = kRes && d.res1 != nullptr;" in host
    assert "*stage_rv = " + kernel_rv.replace("p.rowvec", "d.rowvec").replace("p.a_mode", "d.a_mode").replace(
        "p.rows_per_group", "d.rows_per_group") in host
    from powerpaint_b200 import ops as o

    def staging(**spec):
        return o.gemm_staging(o.Desc("gemm", kv.fake_desc(dict(dict(M=1000, N=320, K=128, bias=True), **spec), 0), None))

    assert staging(res1=True) == (True, False)
    assert staging(res1=True, rowvec=True, rpg=256) == (True, True)
    assert staging(rowvec=True, rpg=192) == (False, False)  # tiles spanning two samples: the register look-ahead
    assert staging(res1=True, row_stats=True) == (True, False)  # mode 3
    assert staging(res1=True, out_fp32=True) == (False, False)  # mode 1
    assert staging(res1=True, act=1, rowvec=True, rpg=128) == (True, True)
    assert staging(conv=1, nb=16, h=8, w=8, cin=256, N=320, rowvec=True, res1=True) == (True, False)  # 2 samples a tile
    assert staging(conv=1, nb=2, h=64, w=64, cin=64, N=320, rowvec=True) == (False, True)  # one sample a tile


def test_every_split_launch_fits_the_sms_in_one_wave():
    """the split-K owner spins on a flag its donor CTA sets: both must be resident together, so a split launch has at
    most SMs work items (2 x tiles). The sweep crosses the chooser's thresholds: K iterations around
    SPLITK_MIN_K_ITERS (36), odd counts, tile counts around SMs / 2, forced and free tile widths, conv launches."""
    from powerpaint_b200 import ops as o

    sms = kv.SMS  # what the host queries assume without a device
    split = 0
    for k_iters in (34, 35, 36, 37, 38, 40, 72, 80):
        for n in (64, 120, 160, 256, 320, 512, 640, 1280):
            for m_tiles in (1, 2, 3, 8, 16, 21, 22, 26, 32, 33, 34, 43, 44, 66, 67, 130, 133):
                for bn in (0, 128, 160, 256):
                    d = kv.fake_desc(dict(M=128 * m_tiles - 3, N=n, K=64 * k_iters, splitk=True, bias=True, res1=True), bn)
                    try:
                        v = kv.query_gemm(d)
                    except RuntimeError:
                        continue
                    nbytes, tiles = o.gemm_splitk_query(o.Desc("gemm", d, None))
                    if v[2] == 2:
                        split += 1
                        assert 2 * tiles <= sms and tiles == m_tiles * _cdiv(n, v[0]), (k_iters, n, m_tiles, bn, v)
                        assert k_iters >= 36 and k_iters % 2 == 0, (k_iters, v)
                    else:
                        assert nbytes == 0, (k_iters, n, m_tiles, bn, v)
    for nb, hw, cin in ((2, 8, 256), (4, 8, 256), (8, 8, 256), (16, 8, 256), (17, 8, 256), (2, 16, 256), (4, 16, 320),
                        (1, 32, 512), (8, 16, 640)):
        for n in (256, 320, 640, 1280):
            d = kv.fake_desc(dict(conv=1, nb=nb, h=hw, w=hw, cin=cin, N=n, splitk=True, bias=True), 0)
            v = kv.query_gemm(d)
            nbytes, tiles = o.gemm_splitk_query(o.Desc("gemm", d, None))
            if v[2] == 2:
                split += 1
                assert 2 * tiles <= sms, (nb, hw, cin, n, v, tiles)
    assert split > 50, split  # the sweep reaches the split launches it means to bound
