"""CPU tests of the request batcher (`powerpaint_b200.serving`): the slot cycle over a fake executor, every refused
option, and that a request's loop inputs are exactly what the pipeline's `__call__` hands the fused denoiser."""
from types import SimpleNamespace

import pytest
import torch

from powerpaint_b200.serving import Request, RequestBatcher, SlotScheduler


class _FakeExecutor:
    """records the cycle; a request's step count is its `steps` keyword"""

    def __init__(self, slots):
        self.log = []
        self.counter = [0] * slots  # steps each slot has run since its last admission / reset
        self.on_replay = None

    def admit(self, s, req):
        if req.kwargs.get("fail"):
            raise ValueError("bad request")
        self.log.append(("admit", s, req.kwargs["name"]))
        self.counter[s] = 0
        return req.kwargs["steps"]

    def reset(self, s):
        self.log.append(("reset", s))
        self.counter[s] = 0

    def replay(self, k):
        self.log.append(("replay", k))
        self.counter = [c + k for c in self.counter]
        if self.on_replay is not None:
            self.on_replay()

    def retire(self, s, req):
        self.log.append(("retire", s, req.kwargs["name"]))
        return (req.kwargs["name"], self.counter[s])


def _req(name, steps, **kw):
    return Request(dict(name=name, steps=steps, **kw))


def test_fifo_admission_chunks_and_retirement():
    ex = _FakeExecutor(2)
    sch = SlotScheduler(2, ex)
    reqs = [sch.submit(_req(n, s)) for n, s in (("a", 5), ("b", 3), ("c", 4), ("d", 1))]
    sch.run()
    # every request ran exactly its own steps
    assert [r.result() for r in reqs] == [("a", 5), ("b", 3), ("c", 4), ("d", 1)]
    assert [r.steps for r in reqs] == [5, 3, 4, 1]
    admits = [e[1:] for e in ex.log if e[0] == "admit"]
    assert [n for _, n in admits] == ["a", "b", "c", "d"]  # FIFO
    # a(5) b(3) -> 3 steps, b retires; c(4) joins a(2 left) -> 2, a retires; d(1) joins c(2 left) -> 1; c alone -> 1
    assert [e[1] for e in ex.log if e[0] == "replay"] == [3, 2, 1, 1]
    assert ex.log[:3] == [("admit", 0, "a"), ("admit", 1, "b"), ("replay", 3)]
    assert ("admit", 1, "c") in ex.log and ("admit", 0, "d") in ex.log


def test_idle_slot_counters_are_reset_at_every_boundary():
    ex = _FakeExecutor(3)
    sch = SlotScheduler(3, ex)
    sch.submit(_req("a", 4))
    sch.submit(_req("b", 2))
    sch.run()
    # boundaries: before replay(2) slot 2 is idle; before replay(2) again slots 1 and 2 are idle
    chunks = []
    cur = []
    for e in ex.log:
        if e[0] == "reset":
            cur.append(e[1])
        if e[0] == "replay":
            chunks.append(sorted(cur))
            cur = []
    assert chunks == [[2], [1, 2]]
    assert max(ex.counter[1:]) <= 2  # an idle slot never runs more than one chunk past a reset


def test_requests_submitted_between_chunks_join_at_the_next_boundary():
    ex = _FakeExecutor(2)
    sch = SlotScheduler(2, ex)
    a = sch.submit(_req("a", 6))
    late = []

    def on_replay():
        if not late:
            late.append(sch.submit(_req("late", 2)))
    ex.on_replay = on_replay
    sch.run()
    i_first = ex.log.index(("replay", 6))
    i_late = next(i for i, e in enumerate(ex.log) if e[0] == "admit" and e[2] == "late")
    assert i_late > i_first  # admitted after the chunk it arrived in
    assert a.result() == ("a", 6) and late[0].result() == ("late", 2)


def test_a_driver_returns_once_its_own_request_is_done_under_sustained_load():
    """requests keep arriving between chunks; the caller driving with until=<its request> returns at the first
    boundary after its request is done, leaving the backlog to the next driver"""
    ex = _FakeExecutor(2)
    sch = SlotScheduler(2, ex)
    mine = sch.submit(_req("mine", 3))
    sch.submit(_req("other", 8))
    arrivals = iter(range(100))

    def on_replay():  # a new request after every chunk: the queue never empties
        i = next(arrivals)
        sch.submit(_req(f"late{i}", 5))
    ex.on_replay = on_replay
    sch.run(until=mine)
    assert mine.done() and mine.result() == ("mine", 3)
    assert [e for e in ex.log if e[0] == "replay"] == [("replay", 3)]  # no chunk past the one that finished it
    assert sch.queue and any(r is not None for r in sch.slots)  # the backlog is left for the next driver
    sch.run(until=sch.slots[1])
    assert ("retire", 1, "other") in ex.log


def test_failed_preparation_completes_only_that_request():
    ex = _FakeExecutor(1)
    sch = SlotScheduler(1, ex)
    bad = sch.submit(_req("bad", 3, fail=True))
    good = sch.submit(_req("good", 2))
    sch.run()
    with pytest.raises(ValueError, match="bad request"):
        bad.result()
    assert good.result() == ("good", 2)


# ---------------------------------------------------------------------------------------------------------- refusals
def _fake_pipe(kind="v1", in_channels=9, pool=False, multi=False, scheduler=None):
    from powerpaint_b200.schedulers import DDIMScheduler

    cfg = SimpleNamespace(global_pool_conditions=pool)
    pipe = SimpleNamespace(scheduler=scheduler or DDIMScheduler(),
                           unet=SimpleNamespace(config=SimpleNamespace(in_channels=in_channels)))
    if kind == "brushnet":
        pipe.brushnet = SimpleNamespace(config=cfg)
    if kind == "controlnet":
        pipe.controlnet = SimpleNamespace(nets=[SimpleNamespace(config=cfg)] * 2) if multi else \
            SimpleNamespace(config=cfg)
    return pipe


@pytest.mark.parametrize("pipe_kw,kw,match", [
    ({}, dict(eta=0.5), "eta"),
    ({}, dict(callback=lambda *a: None), "callback"),
    ({"kind": "brushnet"}, dict(callback_on_step_end=lambda *a: None), "callback_on_step_end"),
    ({"kind": "controlnet"}, dict(guess_mode=True), "guess_mode"),
    ({"kind": "controlnet", "pool": True}, {}, "global_pool_conditions"),
    ({"kind": "brushnet", "pool": True}, {}, "global_pool_conditions"),
    ({"kind": "controlnet", "multi": True}, {}, "several ControlNets"),
    ({"in_channels": 4}, {}, "4-channel UNet"),
    ({}, dict(num_images_per_prompt=2), "num_images_per_prompt"),
    ({}, dict(promptA=["a", "b"]), "promptA"),
    ({}, dict(prompt_embeds=torch.zeros(2, 77, 8)), "prompt_embeds"),
    ({}, dict(image=torch.zeros(2, 3, 64, 64)), "image"),
    ({}, dict(generator=[torch.Generator(), torch.Generator()]), "generator"),
    ({}, dict(height=128), "height"),
    ({}, dict(width=32), "width"),
    ({}, dict(guidance_scale=1.0), "guidance_scale"),
    ({}, dict(output_type="np"), "output_type"),
])
def test_refused_options_name_the_option(pipe_kw, kw, match):
    b = RequestBatcher(_fake_pipe(**pipe_kw), 2, 64, 64)
    with pytest.raises(NotImplementedError, match=match):
        b.submit(**{"promptA": "a", "guidance_scale": 7.5, **kw})
    assert b.plan is None and not b._sched.queue


@pytest.mark.parametrize("cls", ["EulerAncestralDiscreteScheduler", "sde-dpmsolver++"])
def test_stochastic_schedulers_are_refused(cls):
    from powerpaint_b200 import schedulers as S

    sch = S.DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++") if cls == "sde-dpmsolver++" \
        else getattr(S, cls)()
    b = RequestBatcher(_fake_pipe(scheduler=sch), 2, 64, 64)
    with pytest.raises(NotImplementedError, match=type(sch).__name__):
        b.submit(promptA="a")


def test_one_image_requests_are_accepted_and_construction_records_nothing():
    b = RequestBatcher(_fake_pipe("brushnet", in_channels=4), 2, 64, 64)
    r = b.submit(promptA="a", prompt_embeds=None, image=torch.zeros(1, 3, 64, 64), height=64, width=64,
                 output_type="latent", generator=torch.Generator())
    assert not r.done() and len(b._sched.queue) == 1 and b.plan is None and b.plans_recorded == 0


# ------------------------------------------------------------------- the loop inputs equal what __call__ hands over
def _tiny_cfg(cin):
    from oracle.unet import UNetConfig
    from powerpaint_b200.engine import NetConfig

    o = UNetConfig.tiny(cin)
    return o, NetConfig(in_channels=cin, block_out_channels=o.block_out_channels, attention_head_dim=o.attention_head_dim,
                        cross_attention_dim=o.cross_attention_dim, norm_num_groups=o.norm_num_groups)


class _Recorder:
    def __init__(self):
        self.kw = None

    def run(self, **kw):
        self.kw = kw
        return kw["latents"]


class _FakePlan:
    def __init__(self):
        self.kw = None

    def admit(self, s, **kw):
        self.kw = kw
        return len(kw["timesteps"])


def _scheduler(kind):
    from powerpaint_b200 import schedulers as S

    return {"ddim": S.DDIMScheduler, "unipc": S.UniPCMultistepScheduler, "plms": lambda: S.PNDMScheduler(skip_prk_steps=True),
            "dpm": lambda: S.DPMSolverMultistepScheduler(use_karras_sigmas=True),
            "euler": S.EulerDiscreteScheduler}[kind]()


def _pipe_and_call(mode, sched):
    from oracle.vae import AutoencoderKLOracle
    from powerpaint_b200.models import BrushNetModel, ControlNetModel, UNet2DConditionModel
    from powerpaint_b200.pipelines import (StableDiffusionControlNetInpaintPipeline, StableDiffusionInpaintPipeline,
                                           StableDiffusionPowerPaintBrushNetPipeline)

    vae = AutoencoderKLOracle.synthetic(tiny=True)
    o9, n9 = _tiny_cfg(9)
    _, n4 = _tiny_cfg(4)
    g = torch.Generator().manual_seed(11)
    H = 64
    img = torch.rand(1, 3, H, H, generator=g) * 2 - 1
    pe = torch.randn(1, 77, o9.cross_attention_dim, generator=g) * 0.5
    ne = torch.randn(1, 77, o9.cross_attention_dim, generator=g) * 0.5
    kw = dict(image=img, prompt_embeds=pe, negative_prompt_embeds=ne, num_inference_steps=5, guidance_scale=6.5,
              output_type="latent", height=H, width=H)
    if mode == "brushnet":
        pipe = StableDiffusionPowerPaintBrushNetPipeline(vae=vae, text_encoder=None, text_encoder_brushnet=None,
                                                         tokenizer=None, unet=UNet2DConditionModel(n4),
                                                         brushnet=BrushNetModel(n4), scheduler=_scheduler(sched))
        mask = torch.ones(1, 3, H, H)
        mask[:, :, 16:48, 16:48] = -1.0
        kw.update(mask=mask, prompt_embedsU=torch.randn(2, 77, o9.cross_attention_dim, generator=g),
                  brushnet_conditioning_scale=0.7, control_guidance_end=0.6)
    else:
        mask = torch.zeros(1, 1, H, H)
        mask[:, :, 8:40, 16:56] = 1
        kw.update(mask=mask)
        if mode == "controlnet":
            pipe = StableDiffusionControlNetInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None,
                                                            unet=UNet2DConditionModel(n9),
                                                            controlnet=ControlNetModel(n4), scheduler=_scheduler(sched))
            kw.update(control_image=torch.rand(1, 3, H, H, generator=g), controlnet_conditioning_scale=0.4,
                      control_guidance_start=0.2)
        else:
            pipe = StableDiffusionInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None,
                                                  unet=UNet2DConditionModel(n9), scheduler=_scheduler(sched),
                                                  safety_checker=None)
            kw.update(strength=0.6, num_inference_steps=8)
    return pipe, kw


def _same(a, b):
    if torch.is_tensor(a) or torch.is_tensor(b):
        return torch.is_tensor(a) and torch.is_tensor(b) and a.shape == b.shape and torch.equal(a, b)
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("mode,sched", [("v1", "ddim"), ("v1", "unipc"), ("v1", "plms"), ("v1", "dpm"),
                                        ("v1", "euler"), ("brushnet", "ddim"), ("brushnet", "unipc"),
                                        ("controlnet", "ddim"), ("controlnet", "plms")])
def test_slot_inputs_equal_what_call_hands_the_denoiser(mode, sched):
    pipe, kw = _pipe_and_call(mode, sched)
    rec = _Recorder()
    pipe.denoiser = lambda: rec
    torch.manual_seed(5)
    pipe(generator=torch.Generator().manual_seed(3), **kw)
    want = rec.kw
    b = RequestBatcher(pipe, 2, 64, 64)
    plan = _FakePlan()
    b._executor.plan_for = lambda run: plan
    req = b.submit(generator=torch.Generator().manual_seed(3), **kw)
    torch.manual_seed(5)
    n = b._executor.admit(1, req)
    got = plan.kw
    assert n == len(want["timesteps"])
    assert sorted(got) == sorted(want)
    for k in want:
        if k == "callback" or k == "noise_fn":
            assert got[k] is None and want[k] is None
            continue
        assert _same(got[k], want[k]), k


def test_batchers_of_one_pipeline_share_one_driver_lock():
    from powerpaint_b200.serving import pipeline_lock

    pipe, other = _fake_pipe(), _fake_pipe()
    a, b = RequestBatcher(pipe, 2, 64, 64), RequestBatcher(pipe, 4, 128, 128)
    assert a._drive is b._drive is pipeline_lock(pipe)
    assert RequestBatcher(other, 2, 64, 64)._drive is not a._drive


def test_unknown_keywords_fail_at_submit():
    from powerpaint_b200.pipelines import StableDiffusionInpaintPipeline
    from powerpaint_b200.schedulers import DDIMScheduler

    pipe = StableDiffusionInpaintPipeline(vae=None, text_encoder=None, tokenizer=None,
                                          unet=SimpleNamespace(config=SimpleNamespace(in_channels=9)),
                                          scheduler=DDIMScheduler(), safety_checker=None)
    with pytest.raises(TypeError):
        RequestBatcher(pipe, 2, 64, 64).submit(promptA="a", no_such_option=1)
