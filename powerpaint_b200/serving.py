"""Concurrent requests on one fused denoising loop.

`RequestBatcher(pipe, slots, height, width)` serves requests that differ in step count, guidance scale, inputs and
side-net scale from one slotted step program (`denoise.SlottedPlan`): slot s owns the UNet rows 2s / 2s + 1, and
every per-step scalar lives in the slot's own device tables, indexed by the slot's own step counter. Between graph
replays the host swaps requests in and out:

  1. admit queued requests FIFO into free slots: the pipeline's own `prepare_loop` (exactly what `__call__` runs
     before its loop), then the slot's rows of the net input, prompt and control image, its tables, state and counter;
  2. replay the graph k = min(remaining steps of the occupied slots) times;
  3. retire the slots that finished: decode their latents and complete their requests.

Idle slots sit on hold rows (their latents do not move) and their counters are reset at every boundary, so no slot
ever reads past its tables. DDIM with eta > 0 and the stochastic schedulers draw each slot's noise inside the step
kernels from the request's CUDA generator. Options that need the host inside the loop, or rows the slots do not have,
are refused when the request is submitted.
"""
from __future__ import annotations

import collections
import inspect
import threading
import time
from typing import Any, Deque, List, Optional

import torch

from .pipelines.common import LoopInputs, loop_output

OUTPUT_TYPES = ("latent", "uint8", "pil")

_PIPE_LOCKS: dict = {}  # id(pipeline) -> the lock its drivers hold
_PIPE_LOCKS_GUARD = threading.Lock()


def pipeline_lock(pipe) -> threading.Lock:
    """The lock every batcher of `pipe` holds while it drives: preparing a request mutates the pipeline (its
    scheduler's timesteps) and runs its VAE / text-encoder plans, so only one thread may use a pipeline at a time.
    Hold it around direct `pipe(...)` calls made while batchers of the same pipeline serve other threads."""
    with _PIPE_LOCKS_GUARD:
        return _PIPE_LOCKS.setdefault(id(pipe), threading.Lock())


class Request:
    """One submitted request; `result()` blocks until it is done and returns what `pipe(**kwargs)` returns for it (or
    raises what preparing it raised)."""

    def __init__(self, kwargs: dict):
        self.kwargs = kwargs
        self.steps: Optional[int] = None  # set on admission
        self._event = threading.Event()
        self._result: Any = None
        self._error: Optional[BaseException] = None
        self.finished_at: Optional[float] = None  # time.perf_counter() when the result was set

    def done(self) -> bool:
        return self._event.is_set()

    def result(self, timeout: Optional[float] = None):
        if not self._event.wait(timeout):
            raise TimeoutError("request not done")
        if self._error is not None:
            raise self._error
        return self._result

    def _finish(self, result=None, error: Optional[BaseException] = None) -> None:
        self._result, self._error = result, error
        self.finished_at = time.perf_counter()
        self._event.set()


class SlotScheduler:
    """The host side of the slot cycle, over an executor that does the device work:
        executor.admit(slot, request) -> steps   load a request into a free slot
        executor.reset(slot)                     zero an idle slot's step counter
        executor.replay(k)                       k steps of every slot
        executor.retire(slot, request) -> result decode a finished slot and park it
    """

    def __init__(self, slots: int, executor):
        if slots < 1:
            raise ValueError("at least one slot")
        self.executor = executor
        self.queue: Deque[Request] = collections.deque()
        self.slots: List[Optional[Request]] = [None] * slots
        self.remaining = [0] * slots
        self._lock = threading.Lock()  # guards `queue`: submitters append while the driver pops

    def submit(self, request: Request) -> Request:
        with self._lock:
            self.queue.append(request)
        return request

    def _next(self) -> Optional[Request]:
        with self._lock:
            return self.queue.popleft() if self.queue else None

    def _admit(self) -> None:
        for s in range(len(self.slots)):
            while self.slots[s] is None:
                req = self._next()
                if req is None:
                    return
                try:
                    n = self.executor.admit(s, req)
                except Exception as e:  # the request's own preparation failed: it alone is done
                    req._finish(error=e)
                    continue
                req.steps = n
                self.slots[s], self.remaining[s] = req, n

    def run(self, until: Optional[Request] = None) -> None:
        """drive the cycle until the queue is empty and every slot idle, or, with `until`, only until that request is
        done (checked at every chunk boundary): a caller that drives for others returns as soon as its own result is
        ready, and requests still in the slots wait for the next driver"""
        while True:
            if until is not None and until.done():
                return
            self._admit()
            live = [s for s, r in enumerate(self.slots) if r is not None]
            if not live:
                return
            for s, r in enumerate(self.slots):
                if r is None:
                    self.executor.reset(s)
            k = min(self.remaining[s] for s in live)
            self.executor.replay(k)
            for s in live:
                self.remaining[s] -= k
                if self.remaining[s] == 0:
                    req, self.slots[s] = self.slots[s], None
                    try:
                        req._finish(self.executor.retire(s, req))
                    except Exception as e:
                        req._finish(error=e)


def _batch_of(v, embeds: bool = False) -> int:
    """images (or prompts, generators, embeddings when `embeds`) in one keyword"""
    if isinstance(v, (list, tuple)):
        return len(v)
    if torch.is_tensor(v) and v.dim() == (3 if embeds else 4):
        return v.shape[0]
    return 1


class _PlanExecutor:
    """The device side of `SlotScheduler` for a pipeline: one `SlottedPlan`, recorded on the first admission."""

    def __init__(self, batcher: "RequestBatcher"):
        self.b = batcher
        self.plan = None
        self.key = None
        self.records = 0
        self.loops: dict = {}  # slot -> LoopInputs of the request in it

    def prepare(self, request: Request) -> LoopInputs:
        kw = dict(request.kwargs)
        out_type = kw.pop("output_type", "pil")
        loop = self.b.pipe.prepare_loop(**kw, output_type=out_type)
        lat = loop.run["latents"]
        if tuple(lat.shape[-2:]) != (self.b.height // 8, self.b.width // 8):
            raise ValueError(f"canvas {lat.shape[-2] * 8}x{lat.shape[-1] * 8} differs from the batcher's "
                             f"{self.b.height}x{self.b.width}: use one batcher per canvas size")
        return loop

    def admit(self, s: int, request: Request) -> int:
        loop = self.prepare(request)
        n = self.plan_for(loop.run).admit(s, **loop.run)
        self.loops[s] = loop
        return n

    def plan_for(self, run: dict):
        """the slotted plan for these loop inputs, recorded on first use and again when the scheduler kind or the
        weights changed while every slot is idle"""
        sched = "unipc" if run.get("ucoef") is not None else "solver" if run.get("scoef") is not None else \
            "plms" if run.get("pcoef") is not None else "ddim"
        den = self.b.pipe.denoiser()
        # the plan serves one scheduler kind and one set of weights (the parameter generation of each model)
        key = (sched, run["prompt_embeds"].shape[1], den.unet.generation, tuple(n.generation for n in den.sides))
        if self.plan is None or key != self.key:
            if self.loops:
                raise RuntimeError("the scheduler kind or the weights changed while requests are in the slots: "
                                   "submit this request again once they are done")
            self.plan = None  # release the old plan's storage before recording the new one
            self.plan = den.record_slots(self.b.slots, self.b.height // 8, self.b.width // 8, sched, key[1])
            self.key = key
            self.records += 1
        return self.plan

    def reset(self, s: int) -> None:
        self.plan.reset_counter(s)

    def replay(self, k: int) -> None:
        self.plan.replay(k)

    def retire(self, s: int, request: Request):
        latents = self.plan.slot_latents(s)
        self.plan.hold(s)
        return loop_output(self.b.pipe, self.loops.pop(s), latents)


class RequestBatcher:
    """Serve concurrent requests to `pipe` (a v1, BrushNet or ControlNet pipeline) from one slotted fused loop of
    `slots` requests at `height` x `width` pixels. Construction records nothing: the plan is recorded, and its graph
    captured, on the first run.

    `submit(**kwargs)` takes the pipeline's `__call__` keywords for one image and returns a `Request`; `run()` drives
    the loop until every submitted request is done; `batcher(**kwargs)` is a thread-safe blocking submit-and-wait, so
    concurrent callers (e.g. web-server handler threads) share the slots, one of them driving the loop at a time. All
    CUDA work happens in the driving thread, on one stream. Options the slots cannot serve are refused at submit; the
    pipeline's own argument checks run when the request is prepared, and what they raise is raised by
    `Request.result()`."""

    def __init__(self, pipe, slots: int, height: int, width: int):
        if slots < 1:
            raise ValueError("slots must be >= 1")
        if height % 8 or width % 8:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        self.pipe, self.slots, self.height, self.width = pipe, slots, height, width
        self._executor = _PlanExecutor(self)
        self._sched = SlotScheduler(slots, self._executor)
        self._drive = pipeline_lock(pipe)  # one driver at a time, across every batcher of this pipeline

    @property
    def plan(self):
        """the slotted plan (None until the first request is admitted)"""
        return self._executor.plan

    @property
    def plans_recorded(self) -> int:
        return self._executor.records

    # ------------------------------------------------------------------ refusals
    def _side_nets(self) -> list:
        side = getattr(self.pipe, "brushnet", None) or getattr(self.pipe, "controlnet", None)
        if side is None:
            return []
        return list(side.nets) if hasattr(side, "nets") else list(side) if isinstance(side, (list, tuple)) else [side]

    def _cuda_generator(self, g) -> bool:
        """`g` is one torch.Generator on the pipeline's CUDA device"""
        if not isinstance(g, torch.Generator) or g.device.type != "cuda":
            return False
        dev = getattr(self.pipe.unet, "device", None)
        if dev is None:
            return True
        dev = torch.device(dev)
        cur = torch.cuda.current_device
        return dev.type == "cuda" and (g.device.index if g.device.index is not None else cur()) == \
            (dev.index if dev.index is not None else cur())

    def check(self, kwargs: dict) -> None:
        """raise for a request the slots cannot serve"""
        def refuse(msg):
            raise NotImplementedError(f"RequestBatcher: {msg}")
        # the step kernels draw a slot's noise from its generator's Philox stream: that takes one CUDA generator on
        # the pipeline's device; any other generator's noise would be drawn on the host every step
        eta = float(kwargs.get("eta", 0.0) or 0.0) > 0
        sch = self.pipe.scheduler
        if (eta or getattr(sch, "stochastic", False)) and not self._cuda_generator(kwargs.get("generator")):
            what = "`eta` > 0" if eta else f"the stochastic scheduler {type(sch).__name__}"
            refuse(f"{what} draws noise on the host every step and needs a CUDA generator: pass one `torch.Generator` "
                   "on the pipeline's CUDA device")
        for k in ("callback", "callback_on_step_end"):
            if kwargs.get(k) is not None:
                refuse(f"`{k}` runs on the host inside the loop")
        if kwargs.get("guess_mode"):
            refuse("`guess_mode` runs the side net on the conditional rows only")
        nets = self._side_nets()
        if len(nets) > 1 or hasattr(getattr(self.pipe, "controlnet", None), "nets"):
            refuse("several ControlNets")
        if any(getattr(n.config, "global_pool_conditions", False) for n in nets):
            refuse("`global_pool_conditions`")
        if getattr(self.pipe, "brushnet", None) is None and self.pipe.unet.config.in_channels == 4:
            refuse("a 4-channel UNet (its known-region blend)")
        if kwargs.get("num_images_per_prompt", 1) != 1:
            refuse("`num_images_per_prompt` != 1: submit one image per request")
        for k in ("promptA", "promptB", "promptU", "prompt_embeds", "negative_prompt_embeds", "image", "mask",
                  "control_image", "latents", "generator"):
            if _batch_of(kwargs.get(k), k.endswith("embeds")) > 1:
                refuse(f"`{k}` holds more than one image: submit one image per request")
        for k, v in (("height", self.height), ("width", self.width)):
            if kwargs.get(k) is not None and kwargs[k] != v:
                refuse(f"`{k}` {kwargs[k]} differs from the batcher's {v}: use one batcher per canvas size")
        if float(kwargs.get("guidance_scale", 7.5)) <= 1.0:
            refuse("`guidance_scale` <= 1: every slot runs both classifier-free guidance rows")
        if kwargs.get("output_type", "pil") not in OUTPUT_TYPES:
            refuse(f"`output_type` {kwargs.get('output_type')!r}: one of {OUTPUT_TYPES}")

    # ------------------------------------------------------------------ API
    def submit(self, **kwargs) -> Request:
        self.check(kwargs)
        try:  # unknown keywords fail here, as they fail `pipe(...)`
            inspect.signature(self.pipe.prepare_loop).bind(**kwargs)
        except AttributeError:  # a pipeline without `prepare_loop` is refused at admission
            pass
        return self._sched.submit(Request(kwargs))

    def _drive_cycle(self, until: Optional[Request] = None) -> None:
        # the pipeline's device is current while the driver works, whatever thread drives
        with torch.no_grad(), torch.cuda.device(self.pipe.unet.device):
            self._sched.run(until)

    def run(self) -> None:
        """drive the loop until every submitted request is done"""
        with self._drive:
            self._drive_cycle()

    def __call__(self, **kwargs):
        req = self.submit(**kwargs)
        while not req.done():
            if self._drive.acquire(blocking=False):
                try:
                    self._drive_cycle(until=req)  # returns as soon as this caller's request is done
                finally:
                    self._drive.release()
            else:
                req._event.wait(0.005)  # another caller is driving; it returns once its own request is done
        return req.result()
