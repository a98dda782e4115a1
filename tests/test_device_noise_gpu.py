"""GPU tests of the device-drawn step noise: the step kernels reproduce torch's CUDA randn element for element, a
zero-weight draw table changes no bit, the fused loops with device-drawn noise equal the host-drawn loops bit for bit
on one CUDA graph, and the request batcher serves DDIM eta > 0, Euler ancestral and SDE-DPM-Solver++ requests as
their solo calls."""
import functools

import pytest
import torch

from powerpaint_b200 import ops
from powerpaint_b200.pipelines import common

pytestmark = pytest.mark.gpu

DEV = "cuda"
NOISE_ROW = {"ddim": [1.0, 0.0, 0.0, 0.0, 1.0, 1.0, 0.0, 0.0], "solver": [0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0, 1.0]}


def _clone(g):
    c = torch.Generator(device=g.device)
    c.set_state(g.get_state())
    return c


def _step_desc(kind, B, hw, table, step_idx, noise=None, seed=0):
    """a CFG step over B latent rows; with NOISE_ROW coefficients its output is the noise alone"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = dict(eps=torch.randn(2 * B, hw, 4, device=DEV, generator=g), latents=torch.randn(B, hw, 4, device=DEV, generator=g),
             coef=torch.tensor([NOISE_ROW["ddim"]] * 8, device=DEV), m1=torch.randn(B, hw, 4, device=DEV, generator=g),
             scoef=torch.tensor([NOISE_ROW["solver"]] * 8, device=DEV),
             next_in=torch.zeros(2 * B, hw, 16, dtype=torch.bfloat16, device=DEV))
    common_kw = dict(eps=t["eps"], eps_fp32=True, eps_ld=4, latents=t["latents"], coef=t["coef"], step_idx=step_idx,
                     advance_step=True, do_cfg=True, batch=B, hw=hw, next_in=t["next_in"], next_c=16, n_copies=2,
                     noise=noise, draws=table)
    if kind == "ddim":
        d = ops.cfg_ddim_desc(**common_kw, guidance_scale=0.0, guidance_from_coef=True)
    else:
        d = ops.solver_desc(**common_kw, m1=t["m1"], scoef=t["scoef"])
    return d, t


@pytest.mark.parametrize("kind", ["ddim", "solver"])
@pytest.mark.parametrize("case", ["1x64x64", "3x9x11", "8x64x64", "8x128x128 lane 1", "16x128x128 lanes 2-3",
                                  "list of 3", "advanced offset"])
def test_noise_only_step_outputs_torch_randn(kind, case):
    """x_next = noise: over several steps of one counter, the kernel's draw equals torch.randn from a clone of the
    generator, and afterwards the generator stands where those draws leave it"""
    B, h, w = {"1x64x64": (1, 64, 64), "3x9x11": (3, 9, 11), "8x64x64": (8, 64, 64), "8x128x128 lane 1": (8, 128, 128),
               "16x128x128 lanes 2-3": (16, 128, 128), "list of 3": (3, 9, 11), "advanced offset": (2, 64, 64)}[case]
    shape, steps = (B, 4, h, w), 3
    if case == "list of 3":
        gen = [torch.Generator(device=DEV).manual_seed(40 + k) for k in range(B)]
        torch.randn(7, generator=gen[1], device=DEV)  # the rows' streams stand at different offsets
    else:
        gen = torch.Generator(device=DEV).manual_seed(1234)
        if case == "advanced offset":
            torch.randn(1000, generator=gen, device=DEV)
            torch.randn(3, 5, generator=gen, device=DEV)
    ref = [_clone(g) for g in gen] if isinstance(gen, list) else _clone(gen)
    rows = common.device_randn_draws(gen, shape, DEV, steps)
    assert rows is not None
    table = ops.randn_draw_bytes(rows, B).to(DEV)
    step_idx = torch.zeros(1, dtype=torch.int32, device=DEV)
    d, t = _step_desc(kind, B, h * w, table, step_idx)
    for i in range(steps):
        ops.run(d)
        want = common.randn_tensor(shape, generator=ref, device=DEV, dtype=torch.float32)
        got = ops.nchw_from_nhwc_fp32(t["latents"], h, w)
        assert torch.equal(got, want), (case, kind, i, (got - want).abs().max().item())
        assert torch.equal(t["next_in"][:B, :, :4].float(), ops.nhwc_fp32_from_nchw(want).to(torch.bfloat16).float())
    gens, refs = (gen, ref) if isinstance(gen, list) else ([gen], [ref])
    for g, r in zip(gens, refs):
        assert g.get_offset() == r.get_offset()
        assert torch.equal(torch.randn(3, generator=g, device=DEV), torch.randn(3, generator=r, device=DEV))


@pytest.mark.parametrize("kind", ["ddim", "solver"])
def test_zero_weight_draw_table_is_bit_identical_to_no_noise(kind):
    """every row with sigma / r[5] = 0: the same bits as a descriptor without noise, on random coefficients"""
    B, h, w = 2, 9, 11
    g = torch.Generator(device=DEV).manual_seed(8)
    rows = common.device_randn_draws(g, (B, 4, h, w), DEV, 4)
    table = ops.randn_draw_bytes(rows, B).to(DEV)
    outs = []
    for tab in (None, table):
        step_idx = torch.zeros(1, dtype=torch.int32, device=DEV)
        d, t = _step_desc(kind, B, h * w, tab, step_idx, seed=3)
        r = torch.Generator(device=DEV).manual_seed(5)
        t["coef"].copy_(torch.rand(8, 8, device=DEV, generator=r) + 0.5)
        t["scoef"].copy_(torch.randn(8, 8, device=DEV, generator=r))
        t["coef"][:, 4] = 0.0
        t["scoef"][:, 5] = 0.0
        for _ in range(4):
            ops.run(d)
        torch.cuda.synchronize()
        outs.append({k: t[k].clone() for k in ("latents", "m1", "next_in")})
    for k in outs[0]:
        assert torch.equal(outs[0][k].view(torch.uint8), outs[1][k].view(torch.uint8)), k


# ------------------------------------------------------------------------------------------------ the fused loops
def _loop_case(case):
    from oracle.ddim import DDIMOracle
    from test_solver_schedulers_gpu import SCHEDS

    from powerpaint_b200.schedulers import DDIMScheduler

    if case == "v1 ddim eta 0.5":
        so, sp = DDIMOracle(), DDIMScheduler()
        so.step = functools.partial(DDIMOracle.step, so, eta=0.5)
        return "v1", sp, so
    mode, sched = {"brushnet euler_a": ("brushnet", "euler_a"), "controlnet sde": ("controlnet", "sde_dpmpp_2m")}[case]
    return mode, SCHEDS[sched][0](), SCHEDS[sched][1]()


@pytest.mark.parametrize("case", ["v1 ddim eta 0.5", "brushnet euler_a", "controlnet sde"])
def test_device_noise_loop_equals_host_noise_loop_on_one_graph(case):
    from test_pipelines_gpu import _cos, _nets, _rel
    from test_solver_schedulers_gpu import _oracle_loop

    from powerpaint_b200.denoise import FusedDenoiser

    mode, sp, so = _loop_case(case)
    kinds = {"v1": (9, [("unet", 9, 1234)]), "brushnet": (4, [("unet", 4, 1234), ("brushnet", 4, 99)]),
             "controlnet": (9, [("unet", 9, 1234), ("controlnet", 4, 77)])}[mode]
    nets = _nets(*kinds)
    om_u, pm_u, o = nets["unet"]
    side = nets.get("brushnet") or nets.get("controlnet")
    g = torch.Generator(device=DEV).manual_seed(4)
    B, h, steps = 2, 8, 8
    sp.set_timesteps(steps)
    so.set_timesteps(steps)
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g) * float(sp.init_noise_sigma)
    emb = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    extra = torch.randn(2 * B if mode == "brushnet" else B, 5, h, h, device=DEV, generator=g)
    ctrl = torch.cat([torch.rand(B, 3, 8 * h, 8 * h, device=DEV, generator=g)] * 2) if mode == "controlnet" else None
    host_gen, oracle_gen = _clone(g), _clone(g)
    if mode == "v1":
        kw = dict(coef=sp.step_coefficients(sp.timesteps, eta=0.5))
        noise = common.step_noise(g, lat.shape, DEV, steps)
    else:
        kw = dict(coef=sp.step_coefficients(), scoef=sp.solver_coefficients())
        _, noise, _ = common.solver_loop_inputs(sp, sp.timesteps, lat.shape, g, DEV)
    assert noise.keys() == {"randn_draws"}
    run = dict(latents=lat, prompt_embeds=emb, timesteps=sp.timesteps, guidance_scale=7.5, extra=extra,
               side_prompt_embeds=emb if side else None, control_image=ctrl, side_scale=0.8, **kw)
    den = FusedDenoiser(pm_u, side[1] if side else None, mode)
    launches = []
    orig = ops.Program.launch
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops.Program, "launch", lambda prog: (launches.append(prog._graph), orig(prog)))
        got = den.run(**run, **noise)
    assert len(launches) == steps and all(launches), "the device-noise loop replays one CUDA graph"
    host = den.run(**run, noise_fn=lambda i: torch.randn(lat.shape, generator=host_gen, device=DEV))
    assert torch.equal(got, host), (case, (got - host).abs().max().item())
    assert g.get_offset() == host_gen.get_offset()  # the reservation left the generator where the draws did
    again = den.run(**run, **common.step_noise(_clone(oracle_gen), lat.shape, DEV, steps))
    assert torch.equal(got, again)
    so_noise = [torch.randn(lat.shape, generator=oracle_gen, device=DEV) for _ in range(steps)]
    if hasattr(so, "sigmas"):
        so.sigmas = so.sigmas.float().to(DEV)
    so.timesteps = so.timesteps.to(DEV)
    ref = _oracle_loop(mode, om_u, side[0] if side else None, so, lat, emb, extra, ctrl, 7.5, 0.8, so_noise)
    # the tiny-config bound of test_solver_schedulers_gpu.py
    assert _rel(got, ref) < 5e-2 and _cos(got, ref) > 0.998, (case, _rel(got, ref), _cos(got, ref))


def test_pipeline_call_draws_the_host_paths_noise():
    """v1 pipeline, DDIM eta = 0.5, CUDA generator: the loop inputs `__call__` prepares carry device draws; the same
    loop with the host's per-step draws from the reserved stream gives the same latents"""
    from test_serving_gpu import _pipe, _request

    pipe = _pipe("v1")
    kw = _request("v1", 0, 6, 7.5, eta=0.5)
    g = torch.Generator(device=DEV).manual_seed(3)
    loop = pipe.prepare_loop(generator=g, **kw)
    run = dict(loop.run)
    draws = run.pop("randn_draws")
    assert run["noise_fn"] is None and len(draws) == 1
    host_gen = _clone(g)
    host_gen.set_offset(draws[0][1])
    shape = run["latents"].shape
    got = pipe.denoiser().run(**run, randn_draws=draws)
    run["noise_fn"] = lambda i: torch.randn(shape, generator=host_gen, device=DEV)
    host = pipe.denoiser().run(**run)
    assert torch.equal(got, host)
    assert host_gen.get_offset() == g.get_offset()
    # and `__call__` itself
    out = pipe(generator=torch.Generator(device=DEV).manual_seed(3), **kw).images
    assert torch.equal(out, got)


def test_sd15_size_euler_ancestral_batch_8():
    """an SD-1.5-size UNet at 512^2, batch 8 x CFG, Euler ancestral: device-drawn noise equals host-drawn noise"""
    from test_pipelines_gpu import _nets

    from powerpaint_b200.denoise import FusedDenoiser
    from powerpaint_b200.schedulers import DDIMScheduler, EulerAncestralDiscreteScheduler

    _, pm, o = _nets(9, [("unet", 9, 1234)], tiny=False)["unet"]
    sp = EulerAncestralDiscreteScheduler.from_config(DDIMScheduler().config)
    steps = 6
    sp.set_timesteps(steps)
    g = torch.Generator(device=DEV).manual_seed(21)
    B, h = 8, 64
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g) * float(sp.init_noise_sigma)
    emb = torch.randn(2 * B, 77, 768, device=DEV, generator=g) * 0.5
    extra = torch.cat([(torch.rand(B, 1, h, h, device=DEV, generator=g) > 0.5).float(),
                       torch.randn(B, 4, h, h, device=DEV, generator=g)], 1)
    host_gen = _clone(g)
    _, noise, _ = common.solver_loop_inputs(sp, sp.timesteps, lat.shape, g, DEV)
    run = dict(latents=lat, prompt_embeds=emb, timesteps=sp.timesteps, coef=sp.step_coefficients(),
               scoef=sp.solver_coefficients(), guidance_scale=7.5, extra=extra)
    den = FusedDenoiser(pm)
    got = den.run(**run, **noise)
    host = den.run(**run, noise_fn=lambda i: torch.randn(lat.shape, generator=host_gen, device=DEV))
    assert torch.isfinite(got).all()
    assert torch.equal(got, host), (got - host).abs().max().item()


# ------------------------------------------------------------------------------------------------------- serving
@pytest.mark.parametrize("case", ["v1 ddim eta", "brushnet euler_a", "controlnet sde"])
def test_batcher_serves_stochastic_requests_as_their_solo_calls(case):
    """4 slots. One stochastic request in every slot (same inputs, one generator each, seeded alike): each slot equals
    the same request replicated over FusedDenoiser's batch of 4 (the same 8 rows per launch, one draw entry per row)
    bit for bit, so every slot draws its own request's noise. Mixed requests (v1: stochastic and deterministic): v1
    slots equal their solo calls bit for bit and a stochastic slot is isolated from its cotenants. With a side net, 4
    slots differ from batch-1 solo calls by rounding (the tile shapes and the split of the GroupNorm / LayerNorm
    statistics depend on the launch's rows, as in test_serving_gpu's SD-1.5 cases; a ControlNet DDIM slot differs too),
    so those are held to a bound and reported."""
    from test_serving_gpu import COS, H, _batched, _check, _mixed, _pipe, _solo

    from powerpaint_b200 import schedulers as S
    from powerpaint_b200.serving import RequestBatcher

    mode = case.split()[0]
    base = S.DDIMScheduler().config
    sch = {"v1 ddim eta": None, "brushnet euler_a": S.EulerAncestralDiscreteScheduler.from_config(base),
           "controlnet sde": S.DPMSolverMultistepScheduler.from_config(
               base, algorithm_type="sde-dpmsolver++", final_sigmas_type="sigma_min")}[case]
    pipe = _pipe(mode, sch)
    reqs = _mixed(mode)
    if mode == "v1":  # stochastic and deterministic requests share the slots
        for r, eta in zip(reqs, (0.5, 0.0, 1.0, 0.0, 0.3)):
            r["eta"] = eta
    b = RequestBatcher(pipe, 4, H, H)
    admit = b._executor.admit
    # BrushNet's conditioning encode draws from the global RNG: reseeded per admission, the four slots hold one request
    b._executor.admit = lambda s, r: (torch.manual_seed(7), admit(s, r))[1]
    hs = [b.submit(generator=torch.Generator(device=DEV).manual_seed(0), **reqs[0]) for _ in range(4)]
    b.run()
    b._executor.admit = admit
    torch.manual_seed(7)
    run = dict(pipe.prepare_loop(generator=torch.Generator(device=DEV).manual_seed(0), **reqs[0]).run)
    d = run.pop("randn_draws")[0]
    rep = dict(latents=run["latents"].repeat(4, 1, 1, 1), prompt_embeds=run["prompt_embeds"].repeat_interleave(4, 0),
               randn_draws=[tuple(d[:4]) + (k, 1) for k in range(4)])
    if mode == "brushnet":
        rep.update(extra=run["extra"].repeat_interleave(4, 0),
                   side_prompt_embeds=run["side_prompt_embeds"].repeat_interleave(4, 0))
    else:
        rep["extra"] = run["extra"].repeat(4, 1, 1, 1)
    if mode == "controlnet":
        rep.update(control_image=run["control_image"].repeat_interleave(4, 0),
                   side_prompt_embeds=run["side_prompt_embeds"].repeat_interleave(4, 0))
    run.update(rep)
    fused = pipe.denoiser().run(**run)
    for s, h in enumerate(hs):
        assert torch.equal(h.result().images, fused[s:s + 1]), f"{case}: slot {s}"
    bound = dict(exact=True) if mode == "v1" else dict(rel_max=float("inf"), cos_min=-1.0)  # side nets: reported
    _check(f"{case} replicated vs solo", [h.result().images for h in hs], _solo(pipe, reqs[:1]) * 4, [], **bound)
    want = _solo(pipe, reqs)
    got = _batched(b, reqs)
    if mode == "v1":
        _check(case, got, want, [], exact=True)
        outs = []
        for others in ([reqs[1], reqs[2]], [reqs[3], reqs[4], reqs[2]]):
            torch.manual_seed(7)
            mine = b.submit(generator=torch.Generator(device=DEV).manual_seed(0), **reqs[0])
            for k, o in enumerate(others):
                b.submit(generator=torch.Generator(device=DEV).manual_seed(20 + k), **o)
            b.run()
            outs.append(mine.result().images)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], want[0])
    else:
        _check(case, got, want, [], rel_max=5e-2, cos_min=COS - 1e-3)
    assert b.plans_recorded == 1
