"""CPU tests of the device-drawn step noise: torch's CUDA randn launch policy, which generators take the device path,
the reservation of their Philox streams, the batcher's refusals, and the pp_randn_draw ABI."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from powerpaint_b200.pipelines import common

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES_N = [4 * 9 * 11, 4 * 64 * 64, 8 * 4 * 64 * 64, 8 * 4 * 128 * 128, 16 * 4 * 128 * 128]


def _torch_policy(numel, sms, max_threads_per_sm=2048):
    """`calc_execution_policy` of ATen/native/cuda/DistributionTemplates.h, transcribed with its uint32 grid
    arithmetic: (grid, counter_offset) for unroll 4 and 4 offsets per curand call"""
    block = 256
    grid = (numel + block - 1) // block
    blocks_per_sm = max_threads_per_sm // block
    grid = min((sms * blocks_per_sm) & 0xFFFFFFFF, grid & 0xFFFFFFFF)
    return grid, ((numel - 1) // (block * grid * 4) + 1) * 4


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("numel", SHAPES_N)
def test_policy_equals_torch_formula(numel, sms):
    grid, inc = _torch_policy(numel, sms)
    threads, per_step = common.randn_policy(numel, sms, 2048)
    assert threads == 256 * grid and per_step == inc
    cap = sms * 8
    assert (grid == cap) == (numel > 256 * cap)  # capped exactly when the draw outgrows one wave of the device


def test_policy_known_values():
    # uncapped: one element per thread
    assert common.randn_policy(4 * 9 * 11, 132, 2048) == (512, 4)
    assert common.randn_policy(4 * 64 * 64, 132, 2048) == (16384, 4)
    # capped at 132 SMs x 8 blocks: lane 1 from 270 336 elements on, lanes 2-3 from 540 672 on
    assert common.randn_policy(8 * 4 * 128 * 128, 132, 2048) == (270336, 4)
    assert common.randn_policy(16 * 4 * 128 * 128, 132, 2048) == (270336, 4)
    # 114 SMs: the batch-16 draw needs two curand_normal4 per thread
    assert common.randn_policy(16 * 4 * 128 * 128, 114, 2048) == (233472, 8)


@pytest.mark.parametrize("threads,numel", [(8, 5), (8, 31), (8, 32), (8, 33), (8, 100), (256, 1000)])
def test_element_to_thread_call_and_lane_mapping(threads, numel):
    """torch's grid-stride loop (`distribution_elementwise_grid_stride_kernel`, unroll 4) writes element li from
    thread li % threads, call (li / threads) / 4, lane (li / threads) % 4: the mapping the step kernels invert"""
    seen = {}
    rounded = ((numel - 1) // (threads * 4) + 1) * threads * 4
    for idx in range(threads):
        for k, linear in enumerate(range(idx, rounded, threads * 4)):
            for lane in range(4):
                li = linear + threads * lane
                if li < numel:
                    seen[li] = (idx, k, lane)
    assert sorted(seen) == list(range(numel))
    for li, (idx, k, lane) in seen.items():
        q = li // threads
        assert (li % threads, q // 4, q % 4) == (idx, k, lane)


class _FakeCudaGen:
    """the part of a CUDA torch.Generator the helper reads and advances"""

    def __init__(self, seed, offset=0, index=0):
        self.device = torch.device("cuda", index)
        self.seed, self.offset = seed, offset

    def initial_seed(self):
        return self.seed

    def get_offset(self):
        return self.offset

    def set_offset(self, v):
        assert v % 4 == 0
        self.offset = v


@pytest.fixture
def device_h100(monkeypatch):
    """a 132-SM device 0 whose default generator is a fake"""
    default = _FakeCudaGen(seed=67280421310721, offset=40)
    monkeypatch.setattr(common, "_device_policy", lambda index: (132, 2048))
    monkeypatch.setattr(common, "_default_generator", lambda index: default)
    return default


def test_generator_routing(device_h100):
    shape, dev = (2, 4, 9, 11), torch.device("cuda", 0)
    g = _FakeCudaGen(5)
    assert common.device_randn_draws(g, shape, dev, 3) is not None
    assert common.device_randn_draws([_FakeCudaGen(1), _FakeCudaGen(2)], shape, dev, 3) is not None
    assert common.device_randn_draws(None, shape, dev, 3) is not None
    assert common.device_randn_draws([_FakeCudaGen(1)], (1, 4, 9, 11), dev, 3) is not None
    # host path: CPU generators, a CPU loop, a generator on another device, one generator listed twice
    assert common.device_randn_draws(torch.Generator().manual_seed(1), shape, dev, 3) is None
    assert common.device_randn_draws([torch.Generator(), torch.Generator()], shape, dev, 3) is None
    assert common.device_randn_draws(None, shape, "cpu", 3) is None
    assert common.device_randn_draws(_FakeCudaGen(1, index=1), shape, dev, 3) is None
    twice = _FakeCudaGen(3)
    assert common.device_randn_draws([twice, twice], shape, dev, 3) is None and twice.offset == 0
    assert common.step_noise(torch.Generator(), shape, dev, 3).keys() == {"noise_fn"}
    assert common.step_noise(_FakeCudaGen(4), shape, dev, 3).keys() == {"randn_draws"}


def test_reservation_arithmetic(device_h100):
    dev = torch.device("cuda", 0)
    g = _FakeCudaGen(seed=2 ** 64 - 5, offset=12)
    rows = common.device_randn_draws(g, (16, 4, 128, 128), dev, 7)
    assert rows == [(2 ** 64 - 5, 12, 4, 270336, 0, 16)]
    assert g.offset == 12 + 7 * 4  # where seven torch.randn draws of that shape leave the generator
    gens = [_FakeCudaGen(seed=s, offset=8 * s) for s in (1, 2, 3)]
    rows = common.device_randn_draws(gens, (3, 4, 9, 11), dev, 5)
    assert rows == [(s, 8 * s, 4, 512, k, 1) for k, s in enumerate((1, 2, 3))]  # (1, 4, 9, 11) per generator
    assert [x.offset for x in gens] == [8 * s + 5 * 4 for s in (1, 2, 3)]
    rows = common.device_randn_draws(None, (1, 4, 64, 64), dev, 2)
    assert rows == [(67280421310721, 40, 4, 16384, 0, 1)] and device_h100.offset == 48


def test_solver_inputs_reserve_eulers_discarded_draws(device_h100):
    from powerpaint_b200 import schedulers as S

    dev = torch.device("cuda", 0)
    for sch, stochastic in ((S.EulerDiscreteScheduler(), False), (S.EulerAncestralDiscreteScheduler(), True)):
        sch.set_timesteps(6)
        g = _FakeCudaGen(9, offset=4)
        _, noise, finish = common.solver_loop_inputs(sch, sch.timesteps[2:], (1, 4, 8, 8), g, dev)
        assert finish is None and g.offset == 4 + 4 * 4
        assert noise.keys() == ({"randn_draws"} if stochastic else set())
        cpu = torch.Generator().manual_seed(1)
        _, noise, finish = common.solver_loop_inputs(sch, sch.timesteps, (1, 4, 8, 8), cpu, "cpu")
        assert (finish is None) == stochastic and noise.keys() == ({"noise_fn"} if stochastic else set())
        if finish is not None:
            want = torch.Generator().manual_seed(1)
            for _ in range(6):
                torch.randn(1, 4, 8, 8, generator=want)
            finish()
            assert torch.equal(cpu.get_state(), want.get_state())


@pytest.mark.parametrize("gen", [None, "cpu"])
@pytest.mark.parametrize("case", ["eta", "EulerAncestralDiscreteScheduler", "sde-dpmsolver++"])
def test_batcher_refuses_stochastic_requests_without_a_cuda_generator(case, gen):
    from types import SimpleNamespace

    from powerpaint_b200 import schedulers as S
    from powerpaint_b200.serving import RequestBatcher

    sch = {"eta": S.DDIMScheduler, "EulerAncestralDiscreteScheduler": S.EulerAncestralDiscreteScheduler,
           "sde-dpmsolver++": lambda: S.DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++")}[case]()
    pipe = SimpleNamespace(scheduler=sch, unet=SimpleNamespace(config=SimpleNamespace(in_channels=9)))
    b = RequestBatcher(pipe, 2, 64, 64)
    kw = dict(promptA="a", eta=0.5 if case == "eta" else 0.0)
    if gen == "cpu":
        kw["generator"] = torch.Generator().manual_seed(0)
    name = "`eta`" if case == "eta" else type(sch).__name__
    with pytest.raises(NotImplementedError, match="CUDA generator") as e:
        b.submit(**kw)
    assert name in str(e.value)
    assert b.plan is None and not b._sched.queue


def test_randn_draw_and_extended_descriptors_match_the_header(tmp_path):
    from powerpaint_b200 import _native as N
    from powerpaint_b200 import ops

    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    structs = [(N.RandnDraw, "pp_randn_draw"), (N.CfgDdimDesc, "pp_cfg_ddim_desc"), (N.SolverDesc, "pp_solver_desc")]
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "powerpaint_b200.h"', 'int main(void) {']
    for cls, cname in structs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        lines += [f'  printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in cls._fields_]
    lines.append("  return 0; }")
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                        str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = dict(ln.split(" ", 1) for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                         check=True).stdout.splitlines())
    for cls, cname in structs:
        assert int(out[cname]) == ctypes.sizeof(cls), cname
        for f, _ in cls._fields_:
            assert int(out[f"{cname}.{f}"]) == getattr(cls, f).offset, (cname, f)
    assert [f for f, _ in N.CfgDdimDesc._fields_][-2:] == ["draws", "n_draws"]
    assert [f for f, _ in N.SolverDesc._fields_][-2:] == ["draws", "n_draws"]
    # the host table: entries in field order, unused entries match no row
    t = ops.randn_draw_bytes([(2 ** 64 - 1, 8, 4, 512, 0, 2)], 3)
    assert t.dtype == torch.uint8 and t.numel() == 3 * ops.RANDN_DRAW_BYTES == 3 * 40
    e = N.RandnDraw.from_buffer_copy(bytes(t.numpy()[:40]))
    assert (e.seed, e.offset0, e.offset_per_step, e.threads, e.first_row, e.rows) == (2 ** 64 - 1, 8, 4, 512, 0, 2)
    assert N.RandnDraw.from_buffer_copy(bytes(t.numpy()[40:80])).rows == 0


def test_invalid_draw_tables_fail_loudly_without_gpu():
    """descriptors recorded from integer addresses (nothing is launched): noise with draws, a table without a count
    and a misaligned table are refused"""
    from powerpaint_b200 import _native as N
    from powerpaint_b200 import ops

    if not N.lib_path().exists():
        pytest.skip("library not built")

    class _P:  # an integer address standing in for a tensor
        def __init__(self, a):
            self.a = a

        def data_ptr(self):
            return self.a

    base = dict(eps=_P(1 << 20), eps_fp32=True, eps_ld=4, latents=_P(2 << 20), coef=_P(3 << 20), step_idx=_P(4 << 20),
                advance_step=True, do_cfg=True, batch=1, hw=64)
    prog = ops.Program()
    for label, noise, ptr, n in (("exclusive", _P(5 << 20), 6 << 20, 1), ("count", None, 6 << 20, 0),
                                 ("alignment", None, (6 << 20) + 4, 1)):
        d = ops.cfg_ddim_desc(**base, noise=noise, guidance_scale=7.5)
        d.c.draws, d.c.n_draws = ptr, n
        with pytest.raises(RuntimeError, match="draws"):
            prog.add(d)
        s = ops.solver_desc(**base, m1=_P(7 << 20), scoef=_P(8 << 20), noise=noise)
        s.c.draws, s.c.n_draws = ptr, n
        with pytest.raises(RuntimeError, match="draws"):
            prog.add(s)
