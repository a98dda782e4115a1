"""GPU tests of the side-net options on the kernel path: `pp_pool_broadcast` against an fp64 mean, and the fused
loops with several ControlNets, guess mode and globally pooled side nets against the fp32 oracle loops of
oracle/side_nets.py, held to the trajectory bounds of test_pipelines_gpu.py (cosine >= 0.998 for the tiny nets,
>= 0.999 at SD-1.5 width)."""
import pytest
import torch

from oracle import side_nets as osn
from test_pipelines_gpu import _cos, _nets, _rel, _scheds

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _fp32_exact():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


@pytest.mark.parametrize("C", [320, 640, 1280])
def test_pool_broadcast_matches_an_fp64_mean_and_replays_bit_identically(C):
    from powerpaint_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(C)
    for hw in (1, 7, 37 * 13, 4096):
        x = (torch.randn(3, hw, C, device=DEV, generator=g) + 0.5).to(BF16)
        for with_prev in (False, True):
            prev = torch.randn(3, hw, C, device=DEV, generator=g).to(BF16) if with_prev else None
            want = x.double().mean(1, keepdim=True) + (prev.double() if with_prev else 0)
            want = want.expand(3, hw, C)
            outs = []
            for mode in ("eager", "eager", "program"):
                out = torch.full((3, hw, C), float("nan"), device=DEV).to(BF16)
                d = ops.pool_broadcast_desc(x, out, prev)
                if mode == "eager":
                    ops.run(d)
                else:
                    p = ops.Program()
                    p.add(d)
                    p.run()
                torch.cuda.synchronize()
                outs.append(out)
            # the fp32 sum is within rounding of the fp64 mean; the bf16 store adds at most half an ulp (2^-9 rel)
            err = (outs[0].double() - want).abs()
            assert (err <= want.abs() * 2.0 ** -8 + 1e-4).all(), (hw, with_prev, float(err.max()))
            assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    # prev may be the output itself (the running Multi-ControlNet sum)
    x = torch.randn(2, 33, C, device=DEV, generator=g).to(BF16)
    acc = torch.randn(2, 33, C, device=DEV, generator=g).to(BF16)
    want = (acc.float() + x.float().mean(1, keepdim=True)).to(BF16)
    ops.run(ops.pool_broadcast_desc(x, acc, acc))
    assert torch.equal(acc, want) or (acc.float() - want.float()).abs().max() <= 2.0 ** -7 * want.float().abs().max()


def _cn_inputs(B, h, o, seed, K=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g)
    emb = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    mask = (torch.rand(B, 1, h, h, device=DEV, generator=g) > 0.5).float()
    ml = torch.randn(B, 4, h, h, device=DEV, generator=g)
    ctrls = [torch.rand(B, 3, 8 * h, 8 * h, device=DEV, generator=g) for _ in range(K)]
    return lat, emb, mask, ml, ctrls


def _controlnets(K, pools, tiny=True):
    from powerpaint_b200.models import ControlNetModel, synthetic_state_dict
    from oracle.unet import ControlNetOracle

    nets = _nets(9, [("unet", 9, 1234), ("controlnet", 4, 77)], tiny=tiny)
    om_u, pm_u, o = nets["unet"]
    oms, pms = [nets["controlnet"][0]], [nets["controlnet"][1]]
    n_cfg = pms[0]._cfg
    for k in range(1, K):
        sd = synthetic_state_dict(n_cfg, "controlnet", 77 + 13 * k)
        om = ControlNetOracle(nets["controlnet"][2])
        om.load_state_dict(sd)
        oms.append(om.to(DEV).eval())
        pms.append(ControlNetModel.from_state_dict(n_cfg, sd).to(DEV))
    for pm, pool in zip(pms, pools):
        pm.config.global_pool_conditions = pool
    return om_u, pm_u, o, oms, pms


CN_CASES = {  # name: (K, pools, guess, cfg, scales, windows)
    "two_nets": (2, (False, False), False, True, [0.5, 0.8], [(0.0, 1.0), (0.25, 0.75)]),
    "three_nets_guess": (3, (False, False, False), True, True, [0.5, 0.8, 1.0], None),
    "one_net_guess_cfg": (1, (False,), True, True, [0.7], None),
    "one_net_guess_no_cfg": (1, (False,), True, False, [0.7], None),
    "pooled": (1, (True,), True, True, [0.9], None),
    "pooled_then_plain": (2, (True, False), True, True, [0.9, 0.6], None),
    "plain_then_pooled_no_guess": (2, (False, True), False, True, [0.6, 0.9], None),
}


def _keeps(windows, n):
    if windows is None:
        return None
    return [[1.0 - float(i / n < s or (i + 1) / n > e) for i in range(n)] for s, e in windows]


@pytest.mark.parametrize("case", list(CN_CASES))
def test_controlnet_loops_tiny_against_the_oracle(case):
    from powerpaint_b200.denoise import FusedDenoiser

    K, pools, guess, cfg, scales, windows = CN_CASES[case]
    om_u, pm_u, o, oms, pms = _controlnets(K, pools)
    B, h, steps = 2, 8, 8
    lat, emb, mask, ml, ctrls = _cn_inputs(B, h, o, 3, K)
    gs = 7.5 if cfg else 1.0
    if not cfg:
        emb = emb[B:]
    so, sp, ts = _scheds(steps)
    keeps = _keeps(windows, steps)
    ref = osn.loop_controlnet(om_u, oms, pools, so, lat, emb, mask, ml, ctrls, gs, scales, keeps, guess)
    den = FusedDenoiser(pm_u, pms, "controlnet")
    n_ctrl = B if guess or not cfg else 2 * B
    ci = [c if n_ctrl == B else torch.cat([c] * 2) for c in ctrls]
    kw = dict(latents=lat, prompt_embeds=emb, side_prompt_embeds=emb, timesteps=ts, coef=sp.step_coefficients(ts),
              guidance_scale=gs, extra=torch.cat([mask, ml], 1), guess_mode=guess,
              control_image=ci if K > 1 else ci[0], side_scale=scales if K > 1 else scales[0],
              side_keep=keeps if K > 1 or keeps is None else keeps[0])
    got = den.run(**kw)
    assert torch.isfinite(got).all()
    assert _rel(got, ref) < 5e-2 and _cos(got, ref) > 0.998, (case, _rel(got, ref), _cos(got, ref))
    st = next(iter(den._cache.values()))
    assert st["graph"], "the loop replays one CUDA graph"
    if guess and cfg:
        # the side nets wrote only the conditional rows: the unconditional half is still zero after the run
        for r in st["residuals"]:
            assert not r[:B].any() and r[B:].any()
    again = den.run(**kw)
    assert torch.equal(got, again), "a seeded call is deterministic"


def test_controlnet_list_of_one_equals_the_single_net():
    from powerpaint_b200.denoise import FusedDenoiser

    om_u, pm_u, o, oms, pms = _controlnets(1, (False,))
    B, h = 2, 8
    lat, emb, mask, ml, ctrls = _cn_inputs(B, h, o, 5)
    so, sp, ts = _scheds(6)
    keep = [1.0, 1.0, 0.0, 1.0, 1.0, 1.0]
    kw = dict(latents=lat, prompt_embeds=emb, side_prompt_embeds=emb, timesteps=ts, coef=sp.step_coefficients(ts),
              guidance_scale=7.5, extra=torch.cat([mask, ml], 1))
    single = FusedDenoiser(pm_u, pms[0], "controlnet").run(control_image=torch.cat([ctrls[0]] * 2), side_scale=0.6,
                                                           side_keep=keep, **kw)
    listed = FusedDenoiser(pm_u, [pms[0]], "controlnet").run(control_image=[torch.cat([ctrls[0]] * 2)],
                                                             side_scale=[0.6], side_keep=[keep], **kw)
    assert torch.equal(single, listed)


def _conv_batches(den, B, h, guess):
    """batch of every implicit-GEMM conv the recorded step program launches (descriptor census)"""
    from powerpaint_b200 import _native as N
    from powerpaint_b200 import ops

    seen = []
    orig = ops.Program.add

    def add(self, desc):
        if desc.kind == "gemm" and desc.c.a_mode != N.PP_A_MATRIX:
            seen.append((desc.c.nb, desc.c.h, desc.c.w))
        elif desc.kind == "gemm":
            seen.append((None, desc.c.M, None))
        return orig(self, desc)
    ops.Program.add = add
    try:
        den._get(B, h, h, True, 77, False, False, guess=guess)
    finally:
        ops.Program.add = orig
    return seen


def test_guess_mode_census_side_net_runs_on_the_conditional_rows():
    from powerpaint_b200.denoise import FusedDenoiser

    _, pm_u, _, _, pms = _controlnets(1, (False,))
    B, h = 2, 8
    plain = _conv_batches(FusedDenoiser(pm_u, pms, "controlnet"), B, h, False)
    guess = _conv_batches(FusedDenoiser(pm_u, pms, "controlnet"), B, h, True)
    assert len(plain) == len(guess)
    conv_p = [s for s in plain if s[0] is not None]
    conv_g = [s for s in guess if s[0] is not None]
    assert all(s[0] == 2 * B for s in conv_p)
    side = [s for s in conv_g if s[0] == B]
    assert side and len(side) + sum(s[0] == 2 * B for s in conv_g) == len(conv_g)
    # the side net's matrix GEMMs (1x1 zero-convs, attention projections) have M = B * h * w rows at the top level
    mats_g = sorted(s[1] for s in guess if s[0] is None)
    assert B * h * h in mats_g and 2 * B * h * h in mats_g


BN_CASES = {"guess_cfg": (False, True, True), "guess_no_cfg": (False, True, False), "pooled": (True, True, True),
            "pooled_no_guess_flag": (True, False, True)}


@pytest.mark.parametrize("case", list(BN_CASES))
def test_brushnet_loops_tiny_against_the_oracle(case):
    from powerpaint_b200.denoise import FusedDenoiser

    pool, guess_flag, cfg = BN_CASES[case]
    guess = guess_flag or pool  # the pipelines force guess mode for a pooled net
    nets = _nets(4, [("unet", 4, 1234), ("brushnet", 4, 99)])
    (om_u, pm_u, o), (om_b, pm_b, _) = nets["unet"], nets["brushnet"]
    pm_b.config.global_pool_conditions = pool
    g = torch.Generator(device=DEV).manual_seed(7)
    B, h = 2, 8
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g)
    emb_t = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    emb_u = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    cond = torch.randn(B, 5, h, h, device=DEV, generator=g)  # guess mode: the images are not doubled
    gs = 7.5 if cfg else 1.0
    if not cfg:
        emb_t, emb_u = emb_t[B:], emb_u[B:]
    so, sp, ts = _scheds(8)
    ref = osn.loop_brushnet(om_u, om_b, pool, so, lat, emb_t, emb_u, cond, gs, 0.9, guess)
    den = FusedDenoiser(pm_u, pm_b, "brushnet")
    got = den.run(latents=lat, prompt_embeds=emb_u, side_prompt_embeds=emb_t, timesteps=ts,
                  coef=sp.step_coefficients(ts), guidance_scale=gs, extra=cond, side_scale=0.9, guess_mode=guess)
    assert _rel(got, ref) < 5e-2 and _cos(got, ref) > 0.998, (case, _rel(got, ref), _cos(got, ref))
    if cfg:
        for r in next(iter(den._cache.values()))["residuals"]:
            assert not r[:B].any() and r[B:].any()


def test_eager_side_nets_guess_mode_pooling_and_multi_sum():
    from powerpaint_b200.models import MultiControlNetModel

    om_u, pm_u, o, oms, pms = _controlnets(2, (False, True))
    g = torch.Generator(device=DEV).manual_seed(9)
    B, h = 2, 8
    x = torch.randn(B, 4, h, h, device=DEV, generator=g)
    emb = torch.randn(B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    ctrl = [torch.rand(B, 3, 8 * h, 8 * h, device=DEV, generator=g) for _ in range(2)]
    for guess in (False, True):
        d, m = pms[0](x, 500, emb, ctrl[0], 0.7, guess_mode=guess, return_dict=False)
        rd, rm = osn.controlnet(oms[0], x, 500, emb, ctrl[0], 0.7, guess, False)
        assert _cos(torch.cat([t.flatten() for t in d + [m]]), torch.cat([t.flatten() for t in rd + [rm]])) > 0.999
    d, m = pms[1](x, 500, emb, ctrl[1], 0.7, return_dict=False)
    rd, rm = osn.controlnet(oms[1], x, 500, emb, ctrl[1], 0.7, False, True)
    assert all(t.shape[2:] == (1, 1) for t in d + [m])
    assert _cos(torch.cat([t.flatten() for t in d + [m]]), torch.cat([t.flatten() for t in rd + [rm]])) > 0.999
    mc = MultiControlNetModel(pms)
    d, m = mc(x, 500, emb, ctrl, [0.5, 0.8], guess_mode=True)
    rd, rm = osn.multi_controlnet(oms, (False, True), x, 500, emb, ctrl, [0.5, 0.8], True)
    assert _cos(torch.cat([t.flatten() for t in d + [m]]), torch.cat([t.flatten() for t in rd + [rm]])) > 0.999
    # the UNet broadcast-adds pooled [B, C, 1, 1] residuals
    x9 = torch.cat([x, torch.randn(B, 5, h, h, device=DEV, generator=g)], 1)
    e = pm_u(x9, 500, emb, down_block_additional_residuals=rd, mid_block_additional_residual=rm).sample
    r = om_u(x9, 500, emb, down_block_additional_residuals=rd, mid_block_additional_residual=rm)
    assert _cos(e, r) > 0.999


def test_sd15_512_two_controlnets_and_brushnet_guess_mode():
    """SD-1.5 width, 512 x 512 (64 x 64 latents), one image x CFG: two ControlNets, and BrushNet in guess mode"""
    from powerpaint_b200.denoise import FusedDenoiser

    om_u, pm_u, o, oms, pms = _controlnets(2, (False, False), tiny=False)
    B, h, steps = 1, 64, 6
    lat, emb, mask, ml, ctrls = _cn_inputs(B, h, o, 11, 2)
    so, sp, ts = _scheds(steps)
    ref = osn.loop_controlnet(om_u, oms, (False, False), so, lat, emb, mask, ml, ctrls, 7.5, [0.5, 0.8])
    got = FusedDenoiser(pm_u, pms, "controlnet").run(
        latents=lat, prompt_embeds=emb, side_prompt_embeds=emb, timesteps=ts, coef=sp.step_coefficients(ts),
        guidance_scale=7.5, extra=torch.cat([mask, ml], 1), control_image=[torch.cat([c] * 2) for c in ctrls],
        side_scale=[0.5, 0.8])
    assert _cos(got, ref) > 0.999, ("two controlnets", _rel(got, ref), _cos(got, ref))
    del om_u, pm_u, oms, pms
    torch.cuda.empty_cache()
    nets = _nets(4, [("unet", 4, 1234), ("brushnet", 4, 99)], tiny=False)
    (om_u, pm_u, o), (om_b, pm_b, _) = nets["unet"], nets["brushnet"]
    g = torch.Generator(device=DEV).manual_seed(12)
    lat = torch.randn(B, 4, h, h, device=DEV, generator=g)
    emb_t = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    emb_u = torch.randn(2 * B, 77, o.cross_attention_dim, device=DEV, generator=g) * 0.5
    cond = torch.randn(B, 5, h, h, device=DEV, generator=g)
    ref = osn.loop_brushnet(om_u, om_b, False, so, lat, emb_t, emb_u, cond, 7.5, 1.0, True)
    got = FusedDenoiser(pm_u, pm_b, "brushnet").run(
        latents=lat, prompt_embeds=emb_u, side_prompt_embeds=emb_t, timesteps=ts, coef=sp.step_coefficients(ts),
        guidance_scale=7.5, extra=cond, side_scale=1.0, guess_mode=True)
    assert _cos(got, ref) > 0.999, ("brushnet guess", _rel(got, ref), _cos(got, ref))


# ---------------------------------------------------------------- the reference's `__call__` (pipeline_side_net_call.npz)
def _traj(out, key, what):
    from test_side_net_modes_cpu import _gold

    ref = _gold(key).to(out.device)
    assert out.shape == ref.shape and torch.isfinite(out).all(), what
    assert _rel(out, ref) < 5e-2 and _cos(out, ref) > 0.998, (what, _rel(out, ref), _cos(out, ref))


@pytest.mark.parametrize("name", ["cn_two_nets_windows", "cn_two_nets_default_window", "cn_three_nets_guess",
                                  "cn_guess_cfg", "cn_guess_no_cfg", "cn_pooled", "cn_pooled_then_plain"])
def test_controlnet_side_net_call_cuda_vs_reference_call(name):
    """the public ControlNet `__call__` on the GPU (host tensors in, latents out) against the final latents of the
    reference's own `__call__` with several nets, guess mode and pooled nets"""
    from test_side_net_modes_cpu import CONTROLNET_CASES, controlnet_golden_call, controlnet_golden_pipe

    pipe, _, _ = controlnet_golden_pipe(CONTROLNET_CASES[name][0], device=DEV)
    _traj(controlnet_golden_call(pipe, name), f"{name}_latents", f"controlnet __call__ {name}")


@pytest.mark.parametrize("name", ["bn_guess", "bn_guess_window", "bn_pooled"])
def test_brushnet_side_net_loop_cuda_vs_reference_call(name):
    """the fused BrushNet loop on the GPU, fed what the product's `__call__` prepares on the CPU (its conditioning
    latents come from the global CPU generator, as the reference's do), against the reference's own `__call__`"""
    from powerpaint_b200.denoise import FusedDenoiser
    from test_side_net_modes_cpu import BRUSHNET_CASES, _Recorder, brushnet_golden_call, brushnet_golden_pipe

    pool = BRUSHNET_CASES[name][0]
    pipe, _, _ = brushnet_golden_pipe(pool)
    rec = _Recorder()
    pipe.denoiser = lambda: rec
    brushnet_golden_call(pipe, name)
    kw = {k: (v.to(DEV) if torch.is_tensor(v) and k != "timesteps" else v) for k, v in rec.kw.items()}
    out = FusedDenoiser(pipe.unet.to(DEV), pipe.brushnet.to(DEV), "brushnet").run(**kw)
    _traj(out, f"{name}_latents", f"brushnet loop {name}")


def test_side_net_programs_use_only_tested_kernel_variants(monkeypatch):
    """every GEMM / attention variant the new step programs record (SD-1.5 width: C5 with two ControlNets, with a
    ControlNet in guess mode, with a pooled and a plain ControlNet; C3 BrushNet in guess mode and pooled) is a case of
    the variant matrix of test_kernel_variants_gpu.py"""
    from powerpaint_b200 import ops as o
    from powerpaint_b200.denoise import FusedDenoiser
    from test_kernel_variants_gpu import ATTN_CASES, ATTN_VARIANTS, GEMM_CASES, GEMM_VARIANTS, _Census

    census = _Census()
    source = ["?"]
    orig_add = o.Program.add

    def add(self, desc):
        census.record(source[0], desc)
        return orig_add(self, desc)
    monkeypatch.setattr(o.Program, "add", add)
    om_u, pm_u, _, _, pms = _controlnets(2, (False, False), tiny=False)
    del om_u
    for label, nets, pools, guess in (("C5 two ControlNets", pms, (False, False), False),
                                      ("C5 ControlNet guess mode", pms[:1], (False,), True),
                                      ("C5 pooled + plain ControlNet", pms, (True, False), True)):
        for pm, pool in zip(nets, pools):
            pm.config.global_pool_conditions = pool
        source[0] = label
        den = FusedDenoiser(pm_u, nets, "controlnet")
        den._get(2, 64, 64, True, 77, False, False, guess=guess)
        del den
    del pm_u, pms
    torch.cuda.empty_cache()
    nets = _nets(4, [("unet", 4, 1234), ("brushnet", 4, 99)], tiny=False)
    pm_u, pm_b = nets["unet"][1], nets["brushnet"][1]
    for label, pool in (("C3 BrushNet guess mode", False), ("C3 pooled BrushNet", True)):
        pm_b.config.global_pool_conditions = pool
        source[0] = label
        den = FusedDenoiser(pm_u, pm_b, "brushnet")
        den._get(4, 64, 64, True, 77, False, False, guess=True)
        del den
    monkeypatch.setattr(o.Program, "add", orig_add)
    used_gemm = {v for (k, _, v, _, _) in census.sigs.values() if k == "gemm"}
    used_attn = {v for (k, _, v, _, _) in census.sigs.values() if k == "attn"}
    assert census.counts and all(n > 0 for n in census.counts.values())
    assert used_gemm <= set(GEMM_VARIANTS) and used_attn <= set(ATTN_VARIANTS)
    assert used_gemm <= {v for _, v, _ in GEMM_CASES} and used_attn <= {v for _, v, _ in ATTN_CASES}
