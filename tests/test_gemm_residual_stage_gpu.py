"""The GEMM / conv epilogue's staged residual and row vector (modes 0 / 3).

res1 reaches the epilogue through the output staging tile (a TMA load during the tile's main loop), and the
time-embedding row vector through shared memory when every tile lies in one sample. Each GPU case runs once on that
path, is checked element by element against fp64 (`ref_gemm` of test_kernel_variants_gpu), and, where the same
arithmetic has a register route, bit for bit against it:
  * res1 -> res2 with alpha = 1: (x + r) * 1 + 0 and (x + 0) * 1 + r round the same sum once;
  * a row vector with rows_per_group = 128 k -> the same rows duplicated at rows_per_group = 64 (two samples per tile,
    the register look-ahead).
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_kernel_variants_gpu as kv  # noqa: E402

ops = kv.ops  # the device check and the ops module, as a fixture


def _cases():
    cases = []

    def add(name, variant, route, **spec):
        cases.append((f"bn{variant[0]}-m{variant[1]}-k{variant[2]}-{name}", variant, route, dict(spec, _bn=variant[0])))

    for bn in (64, 128, 160, 256):
        # several tiles per CTA (the staging barriers change phase), rows >= M, a last n-tile without its tail sub-tiles
        add("mr", (bn, 0, 1), "res2", M=128 * 140 - 91, N=4 * bn - 32, K=128, bias=True, res1=True)
        if bn != 64:
            add("mr", (bn, 3, 1), "res2", M=128 * 140 - 91, N=4 * bn - 32, K=128, bias=True, res1=True, row_stats=True)
    add("tail32", (160, 0, 1), "res2", M=1000, N=5 * 32, K=192, bias=True, res1=True)
    add("conv-odd", (160, 0, 1), "res2", conv=1, nb=2, h=80, w=107, cin=64, N=320, bias=True, res1=True,
        chan_stats=True)
    add("ldr1", (160, 0, 1), "res2", M=700, N=320, K=128, bias=True, res1=True, ldr1_pad=72)
    add("alias", (160, 0, 1), "res2", M=700, N=320, K=128, bias=True, res1=True, alias=True)
    add("conv-alias", (160, 0, 1), "res2", conv=1, nb=2, h=24, w=40, cin=64, N=320, bias=True, res1=True, alias=True)
    add("r1r2", (160, 0, 1), None, M=700, N=320, K=128, bias=True, res1=True, res2=True, alpha=0.5)
    add("rowvec1", (160, 0, 1), "rpg64", M=128 * 140, N=640, K=128, bias=True, rowvec=True, rpg=256, res1=True)
    add("conv-rowvec1", (160, 0, 1), None, conv=1, nb=2, h=80, w=107, cin=64, N=320, bias=True, rowvec=True,
        act=1)
    add("conv-rowvec2", (128, 0, 1), None, conv=1, nb=16, h=8, w=8, cin=256, N=1280, bias=True, rowvec=True)
    add("splitk", (160, 0, 2), "res2", M=128 * 3 + 1, N=2 * 160 - 8, K=64 * 40, splitk=True, bias=True, res1=True)
    return cases


CASES = _cases()


def _snapshot(outs, extra):
    got = {k: v.clone() for k, v in outs.items()}
    for k in ("rec", "final", "part"):
        if k in extra:
            got[k] = extra[k].clone()
    return got


def _run(ops, desc, outs, extra, before=None):
    for v in outs.values():
        v.fill_(float("nan"))
    if before:
        before()
    ops.run(desc)
    torch.cuda.synchronize()
    return _snapshot(outs, extra)


def _assert_bits(name, a, b):
    for k in a:
        assert torch.equal(kv._bits(a[k]), kv._bits(b[k])), f"{name}: `{k}` differs between the staged and register routes"


def _prepare(spec, variant, seed):
    from powerpaint_b200 import _native as nat

    desc, t, outs, canv, extra = kv.build_gemm(spec, variant, seed)
    d = desc.c
    keep = [desc]
    if spec.get("ldr1_pad"):
        r = torch.full((t["res1"].shape[0], d.ldr1 + spec["ldr1_pad"]), float("nan"), device="cuda", dtype=kv.BF16)
        r[:, :d.N] = t["res1"][:, :d.N]
        t["res1"], d.ldr1, d.res1 = r, r.shape[1], nat.ptr(r)
    fill = None
    if spec.get("alias"):
        # res1 is the output itself (an in-place residual add): the output is filled with the residual before each run
        res = t["res1"][:, :d.N].clone()
        full = torch.zeros(res.shape[0], d.ldc, device="cuda", dtype=kv.BF16)
        full[:, :d.N] = res
        t["res1"], d.ldr1, d.res1 = full, d.ldc, d.out

        def fill():
            outs["out"].copy_(res)
    return desc, t, outs, canv, extra, fill, keep


def _register_route(ops, desc, t, route, keep):
    """the same launch with res1 moved to res2 (alpha 1) or the row vector spread over 64-row groups"""
    from powerpaint_b200 import _native as nat

    d = desc.c
    c2 = type(d).from_buffer_copy(d)
    if route == "res2":
        assert d.alpha == 1.0 and not d.res2 and not d.alpha_dev
        c2.res2, c2.ldr2, c2.res1, c2.ldr1 = d.res1, d.ldr1, None, 0
    else:
        assert d.rows_per_group % 128 == 0
        rv = kv._mat(t["rowvec"], t["rowvec"].shape[0], d.N, d.rowvec_ld).repeat_interleave(d.rows_per_group // 64, 0)
        rv = rv.contiguous()
        keep.append(rv)
        c2.rowvec, c2.rowvec_ld, c2.rows_per_group = nat.ptr(rv), d.N, 64
    return ops.Desc("gemm", c2, [t, keep])


@pytest.mark.gpu
@pytest.mark.parametrize("cid,variant,route,spec", CASES, ids=[c[0] for c in CASES])
def test_staged_epilogue_terms(ops, cid, variant, route, spec):
    desc, t, outs, canv, extra, fill, keep = _prepare(spec, variant, seed=sum(map(ord, cid)))
    d = desc.c
    assert ops.gemm_variant(desc) == variant, (cid, ops.gemm_variant(desc))
    staged = ops.gemm_staging(desc)
    assert staged[0] == bool(spec.get("res1")), (cid, staged)  # res1 goes through the staging tile
    if route:
        reg = _register_route(ops, desc, t, route, keep)
        # the route under comparison takes the register path for the term this case stages
        if route == "res2":
            assert staged[0] and not ops.gemm_staging(reg)[0], cid
        else:
            assert staged[1] and not ops.gemm_staging(reg)[1], cid
        want = _run(ops, reg, outs, extra, fill)
    got = _run(ops, desc, outs, extra, fill)
    worst = kv.check_gemm(cid, d, t, outs, canv, variant[0])
    if spec.get("row_stats"):
        kv._check_row_stats(cid, d, t, extra, variant[0])
    if route:
        _assert_bits(cid, got, want)
    print(f"[staged {cid}] worst err/bound = {worst:.3f}" + (f", bit-identical to the {route} route" if route else ""))


@pytest.mark.gpu
def test_graph_replay_equals_eager(ops):
    cid, variant, _route, spec = next(c for c in CASES if c[0] == "bn160-m0-k1-mr")  # several tiles per CTA
    desc, t, outs, canv, extra, fill, keep = _prepare(spec, variant, seed=7)
    eager = _run(ops, desc, outs, extra)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.run(desc)
    for v in outs.values():
        v.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    _assert_bits("graph replay", eager, _snapshot(outs, extra))

