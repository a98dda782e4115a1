"""GPU tests of the DV <= 64 attention kernels (turn-taking warpgroups, look-ahead, row sums from the PV MMA).

SD-1.5's d = 40 runs at the PV width 48, so column 40 of O carries the softmax row sums (V^T row 40 is all ones in
shared memory). Every case is checked element by element against the fp64 reference and its bound from
test_kernel_variants_gpu.py, at the shapes where that trick could break: the C2 self-attention grid, 77 keys (one
ragged key block), one key, 129 keys (a block of one key), logits large enough that one key takes nearly all the weight,
and fp16 V^T near its largest values.
"""
import pytest
import torch

from test_kernel_variants_gpu import assert_canvases, assert_within, build_attention, ref_attention


@pytest.fixture(scope="module")
def ops():
    from powerpaint_b200 import _native, ops as o

    assert _native.lib().pp_device_supported() == 1, "tests need an sm_90 (H100) device"
    return o


def _run(ops, desc, out):
    out.fill_(float("nan"))
    ops.run(desc)
    torch.cuda.synchronize()
    return out.clone()


CASES = [
    # id, spec, P in fp16, logit scale (q and k multiplied by its square root), V^T amplitude
    ("c2-self-4096", dict(B=16, H=8, d=40, nq=4096, nk=4096, layout="self"), False, 1.0, 1.0),
    ("cross-77", dict(B=16, H=8, d=40, nq=4096, nk=77, layout="cross"), True, 1.0, 1.0),
    ("nk1", dict(B=2, H=3, d=40, nq=200, nk=1, layout="plain"), False, 1.0, 1.0),
    ("nk129", dict(B=2, H=3, d=40, nq=200, nk=129, layout="plain"), True, 1.0, 1.0),
    ("one-key-wins", dict(B=2, H=4, d=40, nq=300, nk=700, layout="plain"), False, 30.0, 1.0),
    ("fp16-vt-near-max", dict(B=2, H=4, d=40, nq=300, nk=700, layout="plain"), True, 1.0, 6.0e4),
]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,spec,f16,logit,vamp", CASES, ids=[c[0] for c in CASES])
def test_d40_within_the_fp64_bound(ops, cid, spec, f16, logit, vamp):
    desc, t, canv = build_attention(spec, f16, seed=sum(map(ord, cid)))
    assert ops.attention_variant(desc) == (48, f16)
    if logit != 1.0:
        t["q"].mul_(logit ** 0.5)
        if t["k"].data_ptr() != t["q"].data_ptr():
            t["k"].mul_(logit ** 0.5)
    if vamp != 1.0:
        v = t["vt"][:, :spec["nk"]]
        v.copy_((v.float() / v.float().abs().amax() * vamp).to(v.dtype))
    out = canv["out"].view
    first = _run(ops, desc, out)
    ref, bound = ref_attention(desc.c, t)
    worst = assert_within(cid, first, ref, bound)
    assert_canvases(cid, canv)
    if cid == "c2-self-4096":
        again = _run(ops, desc, out)
        assert torch.equal(again.view(torch.int16), first.view(torch.int16)), f"{cid}: two runs differ"
    print(f"[attention d=40 {cid}] worst err/bound = {worst:.3f}")
