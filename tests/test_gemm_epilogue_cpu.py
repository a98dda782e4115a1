"""CPU test: the GEMM / conv epilogue runs from the wgmma accumulator registers without pushing the kernel into spills.

The epilogue finishes each thread's accumulators in the fragment layout (two rows, two columns of every 8-column group)
and stores them with stmatrix, so no variant needs the fp32 shared-memory tile it used to go through. That only pays if
the register allocation holds: this test reads the `-Xptxas -v` log `build()` leaves for gemm_conv.cu and bounds the
spill stores of every `gemm_conv_kernel` variant by what the fp32-tile epilogue spilled.
"""
import re
from pathlib import Path

import pytest

from powerpaint_b200 import build as b

GEMM = re.compile(r"_ZN2pp16gemm_conv_kernelILi(\d+)ELi(\d+)ELb([01])EEEvNS_11GemmKParamsE")
# (BLOCK_N, MODE, split-K) -> spill-store bytes of the fp32-tile epilogue (ptxas, CUDA 12.9, sm_90a); 0 stays 0
SPILL_LIMIT = {
    **{(bn, mode, 0): 0 for bn, mode in [(64, 0), (64, 1), (64, 3), (64, 4), (64, 5), (128, 0), (128, 1), (128, 2),
                                         (128, 4), (128, 5), (160, 0), (160, 1), (160, 4), (160, 5), (256, 2), (256, 4)]},
    (128, 3, 0): 90, (160, 3, 0): 98, (256, 0, 0): 316, (256, 3, 0): 506, (256, 5, 0): 180, (256, 1, 0): 116,
    (256, 0, 1): 904, (160, 0, 1): 76, (128, 0, 1): 48,
}


@pytest.fixture(scope="module")
def spills():
    b.build()
    log = Path(str(b.BUILD_DIR / "gemm_conv") + ".ptxas.log").read_text()
    out, fn = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        g = GEMM.fullmatch(fn) if fn and m else None
        if g:
            key = (int(g.group(1)), int(g.group(2)), int(g.group(3)))
            out[key] = max(out.get(key, 0), int(m.group(1)))
    return out


def test_every_variant_is_in_the_log(spills):
    assert set(spills) == set(SPILL_LIMIT), sorted(set(spills) ^ set(SPILL_LIMIT))


def test_no_variant_spills_more_than_the_fp32_tile_epilogue(spills):
    over = {k: (spills[k], lim) for k, lim in SPILL_LIMIT.items() if spills[k] > lim}
    assert not over, f"(BLOCK_N, MODE, split-K): (spill bytes, limit): {over}"

