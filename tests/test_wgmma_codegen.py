"""CPU test: the compiled GEMM / conv and attention kernels keep their wgmma asynchronous.

ptxas serialises every `wgmma.mma_async` of a kernel (a `WARPGROUP.DEPBAR` wait for zero outstanding groups after each
HGMMA) when anything in the kernel forbids keeping MMAs in flight: a function call anywhere in it, `printf` included
(C7510), a wgmma issued under a runtime condition (C7519), or too few registers (C7512). The kernels still compute the
right results then, only slower, so no numerical test notices. This test reads what `build()` left behind: the
`-Xptxas -v` log of every source and the SASS of its object file.
"""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from powerpaint_b200 import build as b

SERIALISED = re.compile(r"\((C7510|C7512|C7519)\).*?function '(\w+)'")
GEMM = re.compile(r"^_ZN2pp16gemm_conv_kernelILi(\d+)ELi(\d+)ELb([01])EEEvNS_11GemmKParamsE$")
ATTN = re.compile(r"^_ZN2pp15attn_fwd_kernelILi(\d+)ELb([01])EEEvNS_11AttnKParamsE$")
# Head dims 160 / 192: O alone takes 80 / 96 of the 168 registers a thread may have (9 warps per CTA, one CTA per SM),
# so ptxas serialises their MMAs for lack of registers (C7512). SD-1.5 runs d = 40 / 80 / 160 at widths 48 / 80 / 160.
ATTN_REGISTER_BOUND_DV = {160, 192}


def _checked(fn: str) -> bool:
    m = ATTN.match(fn)
    return bool(GEMM.match(fn)) or bool(m and int(m.group(1)) not in ATTN_REGISTER_BOUND_DV)


def _cuobjdump() -> str:
    nvcc = shutil.which(b._nvcc()) or b._nvcc()
    return str(Path(nvcc).resolve().parent / "cuobjdump")


@pytest.fixture(scope="module")
def built():
    b.build()
    return {src: b.BUILD_DIR / src for src in ("gemm_conv", "attention")}


def test_ptxas_reports_no_serialised_wgmma(built):
    found = []
    for stem in built.values():
        log = Path(str(stem) + ".ptxas.log").read_text()
        found += [(code, fn) for code, fn in SERIALISED.findall(log) if _checked(fn)]
    assert not found, f"ptxas serialised the wgmma of: {sorted(set(found))}"


def test_every_mma_loop_keeps_a_group_in_flight(built):
    counts = {}
    for stem in built.values():
        sass = subprocess.run([_cuobjdump(), "-sass", str(stem) + ".o"], capture_output=True, text=True, check=True).stdout
        fn = None
        for line in sass.splitlines():
            m = re.search(r"Function : (\w+)", line)
            if m:
                fn = m.group(1)
                counts[fn] = [0, 0]
            elif fn and "HGMMA." in line:
                counts[fn][0] += 1
            elif fn and "WARPGROUP.DEPBAR" in line:
                counts[fn][1] += 1
    gemm = [fn for fn in counts if GEMM.match(fn)]
    attn = [fn for fn in counts if ATTN.match(fn) and _checked(fn)]
    assert len(gemm) == 25 and len(attn) == 12, (len(gemm), len(attn))
    serial = {fn: tuple(counts[fn]) for fn in gemm + attn if not 0 < counts[fn][1] < counts[fn][0]}
    assert not serial, f"one WARPGROUP.DEPBAR per HGMMA (or no HGMMA) in: {serial}"
