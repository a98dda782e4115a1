"""Canonical listing of every op the host planner records, to show that two versions of the planner record the same
programs.

    python tools/dump_programs.py --out DIR

Every `ops.Program.add*` call is logged: for `add`, every field of the C descriptor; for `add_window_copy`, its
arguments and the window table. A device pointer is written as (allocation token, byte offset): the allocator block
that contains it is looked up in `torch.cuda.memory_snapshot()` while the plans are alive, and tokens are numbered in
order of first appearance in the op stream, so neither addresses nor the order weights are packed in matter. Floats
are written bit for bit (hex). Per case the listing also has each program's op and launch count and the plan's bytes.

The cases use only the models' public calls and `FusedDenoiser._get`: the census shapes of the fused step under each
engine switch (each switch set in a child process, through its environment variable), the fused step's scheduler /
noise / blend / side-net options, the eager UNet / BrushNet / ControlNet forwards, VAE encode / decode at 512^2 and
tiled at 1024 x 1360, and the text encoder at 2 x 77 with and without added tokens. One file per case under DIR.
"""
from __future__ import annotations

import argparse
import bisect
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SWITCHES = {"default": {}, "splitk": {"PP_B200_SPLITK": "1"}, "no_ln_fold": {"PP_B200_LN_FOLD": "0"},
            "no_qkv_merged": {"PP_B200_QKV_MERGED": "0"}, "no_gn_fused": {"PP_B200_GN_FUSED": "0"},
            "geglu_bn128": {"PP_B200_GEGLU_BN": "128"}}
# (name, mode, images B, latent h, w) of the census (tests/test_kernel_variants_gpu.py DENOISER_SHAPES)
CENSUS = (("C2", "v1", 8, 64, 64), ("C3", "brushnet", 4, 64, 64), ("C4", "v1", 2, 128, 128),
          ("C5", "controlnet", 2, 64, 64), ("odd80x107", "v1", 1, 80, 107))


class Recorder:
    def __init__(self):
        import torch

        from powerpaint_b200 import ops

        self.torch, self.ops = torch, ops
        self.ops_log = []       # (program id, op name, [(field, kind, value)])
        self.programs = []      # in order of first op
        self._orig = {}

    def _val(self, name, v):
        torch = self.torch
        if isinstance(v, torch.Tensor):
            return (name, "p", v.data_ptr())
        if v is None:
            return (name, "p", 0)
        if isinstance(v, float):
            return (name, "f", v.hex())
        return (name, "i", int(v))

    def _struct(self, s, prefix=""):
        out = []
        for f, t in s._fields_:
            v = getattr(s, f)
            if t is ctypes.c_void_p:
                out.append((prefix + f, "p", v or 0))
            elif t is ctypes.c_float:
                out.append((prefix + f, "f", float(v).hex()))
            elif isinstance(v, ctypes.Structure):
                out += self._struct(v, prefix + f + ".")
            else:
                out.append((prefix + f, "i", int(v)))
        return out

    def _log(self, prog, op, fields):
        if not any(p is prog for p in self.programs):
            self.programs.append(prog)
        self.ops_log.append((prog, op, fields))

    def install(self):
        P = self.ops.Program
        rec = self
        for name in [n for n in vars(P) if n.startswith("add")]:
            orig = getattr(P, name)
            self._orig[name] = orig

            def hook(prog, *args, _orig=orig, _name=name):
                rec._record(prog, _name, args)
                return _orig(prog, *args)
            setattr(P, name, hook)

    def _record(self, prog, name, args):
        from powerpaint_b200 import _native as N

        if name == "add":
            desc = args[0]
            self._log(prog, "add:" + desc.kind, self._struct(desc.c))
        elif name == "add_window_copy":
            wl = args[0]
            fields = [self._val(f, getattr(wl, f)) for f in ("src", "dst", "table", "channels", "src_pix", "dst_pix",
                                                             "count", "max_pixels")]
            raw = bytes(wl.table.cpu().numpy().tobytes())
            table = (N.Window * wl.count).from_buffer_copy(raw)
            for k, w in enumerate(table):
                fields += [(f"w{k}.{f}", "i", int(getattr(w, f))) for f, _ in N.Window._fields_]
            self._log(prog, name, fields)
        else:
            self._log(prog, name, [self._val(f"a{k}", v) for k, v in enumerate(args)])

    def take(self, extra_lines):
        """the canonical listing of everything recorded since the last call"""
        blocks = []
        for seg in self.torch.cuda.memory_snapshot():
            addr = seg["address"]
            for b in seg["blocks"]:
                if b["state"] == "active_allocated":
                    blocks.append((addr, b["size"]))
                addr += b["size"]
        blocks.sort()
        starts = [b[0] for b in blocks]
        tokens = {}
        prog_no = {}
        lines = []

        def canon(p):
            if not p:
                return "null"
            i = bisect.bisect_right(starts, p) - 1
            if i < 0 or p >= blocks[i][0] + blocks[i][1]:
                return "unresolved"
            base = blocks[i][0]
            tok = tokens.setdefault(base, len(tokens))
            return f"T{tok}+{p - base}"
        for prog, op, fields in self.ops_log:
            pn = prog_no.setdefault(id(prog), len(prog_no))
            body = " ".join(f"{f}={canon(v) if k == 'p' else v}" for f, k, v in fields)
            lines.append(f"P{pn} {op} {body}")
        for prog in self.programs:
            lines.append(f"P{prog_no[id(prog)]} num_ops={prog.num_ops} num_launches={prog.num_launches}")
        lines += extra_lines
        self.ops_log, self.programs = [], []
        return lines


def _models(dev):
    from powerpaint_b200.engine import NetConfig
    from powerpaint_b200.models import BrushNetModel, ControlNetModel, UNet2DConditionModel

    # the listing does not depend on weight values: the models keep their zero initialisation
    return dict(u9=UNet2DConditionModel(NetConfig(in_channels=9)).to(dev),
                u4=UNet2DConditionModel(NetConfig(in_channels=4)).to(dev),
                bn=BrushNetModel(NetConfig(in_channels=4)).to(dev),
                cn=ControlNetModel(NetConfig(in_channels=4)).to(dev),
                cn2=ControlNetModel(NetConfig(in_channels=4)).to(dev))


def fused_cases(m, census_only):
    """(name, denoiser factory, _get arguments)"""
    from powerpaint_b200.denoise import FusedDenoiser

    def den(mode, sides=None, unet="u9"):
        return lambda: FusedDenoiser(m[unet], sides, mode) if sides is not None else FusedDenoiser(m[unet])
    mk = {"v1": den("v1"), "brushnet": den("brushnet", m["bn"], "u4"), "controlnet": den("controlnet", m["cn"])}
    cases = [(f"fused_{n}", mk[mode], (B, h, w, True, 77, False, mode == "brushnet")) for n, mode, B, h, w in CENSUS]
    if census_only:
        return cases
    cases += [
        ("fused_unipc", mk["v1"], (1, 64, 64, True, 77, False, False, "unipc")),
        ("fused_solver", mk["v1"], (1, 64, 64, True, 77, False, False, "solver")),
        ("fused_solver_noise", mk["v1"], (1, 64, 64, True, 77, True, False, "solver")),
        ("fused_ddim_eta_noise", mk["v1"], (1, 64, 64, True, 77, True, False)),
        ("fused_blend4", den("v1", None, "u4"), (1, 64, 64, True, 77, False, False, "ddim", True)),
        ("fused_extra_per_copy", mk["v1"], (1, 64, 64, True, 77, False, True)),
        ("fused_no_cfg", mk["v1"], (1, 64, 64, False, 77, False, False)),
        ("fused_brushnet_guess", mk["brushnet"], (2, 64, 64, True, 77, False, True, "ddim", False, True)),
        ("fused_controlnet_guess", mk["controlnet"], (2, 64, 64, True, 77, False, False, "ddim", False, True)),
        ("fused_2controlnets_one_pooled", den("controlnet", [m["cn"], m["cn2"]]), (2, 64, 64, True, 77, False, False)),
        ("fused_brushnet_pooled", mk["brushnet"], (2, 64, 64, True, 77, False, True)),
    ]
    return cases


def run_cases(out_dir, switch, census_only):
    import torch

    dev = torch.device("cuda:0")
    rec = Recorder()
    rec.install()
    m = _models(dev)
    written = []

    def emit(name, extra):
        lines = rec.take(extra)
        path = os.path.join(out_dir, f"{switch}__{name}.txt")
        with open(path, "w") as f:
            f.write("\n".join(lines) + "\n")
        written.append((name, sum(1 for ln in lines if " num_ops=" not in ln and not ln.startswith("bytes"))))

    for name, make, args in fused_cases(m, census_only):
        pooled = name.endswith("pooled")
        if pooled:  # the second ControlNet / the BrushNet pools its residuals globally
            (m["cn2"] if "2controlnets" in name else m["bn"]).config.global_pool_conditions = True
        d = make()
        st = d._get(*args)
        emit(name, [f"bytes={st['bytes']}"])
        if pooled:
            m["cn2"].config.global_pool_conditions = m["bn"].config.global_pool_conditions = False
        del d, st
        torch.cuda.empty_cache()
    if census_only:
        return written
    # slotted step programs (serving.RequestBatcher): 4 slots at 64 x 64 latents, one per mode and scheduler kind
    from powerpaint_b200.denoise import FusedDenoiser

    for name, d, sched in (("slotted_v1_ddim", FusedDenoiser(m["u9"]), "ddim"),
                           ("slotted_v1_plms", FusedDenoiser(m["u9"]), "plms"),
                           ("slotted_v1_solver", FusedDenoiser(m["u9"]), "solver"),
                           ("slotted_brushnet_unipc", FusedDenoiser(m["u4"], m["bn"], "brushnet"), "unipc"),
                           ("slotted_controlnet_ddim", FusedDenoiser(m["u9"], m["cn"], "controlnet"), "ddim")):
        sp = d.record_slots(4, 64, 64, sched)
        emit(name, [f"bytes={sp.bytes}"])
        del d, sp
        torch.cuda.empty_cache()
    g = torch.Generator(device=dev).manual_seed(0)
    B, h, w = 2, 64, 64
    t = torch.tensor(500.0)
    emb = torch.randn(B, 77, 768, device=dev, generator=g)

    def last_bytes(engine):  # the plan just used: the most recent entry of the engine's plan cache
        p = list(engine._plans.values())[-1]
        return [f"bytes={getattr(p, 'pool', p).bytes}"]  # the storage account of the plan (or of its pool)

    def plan_bytes(model):
        return last_bytes(model.engine())

    with torch.no_grad():
        m["u9"](torch.randn(B, 9, h, w, device=dev, generator=g), t, emb)
        emit("eager_unet", plan_bytes(m["u9"]))
        sd, sm, su = m["u4"].engine()._state_shapes(B, h, w)
        nchw = lambda s: torch.randn(B, s[0], s[1], s[2], device=dev, generator=g)  # noqa: E731
        m["u4"](torch.randn(B, 4, h, w, device=dev, generator=g), t, emb,
                down_block_add_samples=[nchw(s) for s in sd], mid_block_add_sample=nchw(sm),
                up_block_add_samples=[nchw(s) for s in su])
        emit("eager_unet_brushnet_adds", plan_bytes(m["u4"]))
        m["u9"](torch.randn(B, 9, h, w, device=dev, generator=g), t, emb,
                down_block_additional_residuals=[nchw(s) for s in sd], mid_block_additional_residual=nchw(sm))
        emit("eager_unet_controlnet_res", plan_bytes(m["u9"]))
        for net, kw in (("bn", dict(brushnet_cond=torch.randn(B, 5, h, w, device=dev, generator=g))),
                        ("cn", dict(controlnet_cond=torch.rand(B, 3, 8 * h, 8 * w, device=dev, generator=g)))):
            for opt in ("plain", "guess", "pooled"):
                m[net].config.global_pool_conditions = opt == "pooled"
                m[net](torch.randn(B, 4, h, w, device=dev, generator=g), t, emb, conditioning_scale=0.7,
                       guess_mode=opt == "guess", **kw)
                emit(f"eager_{net}_{opt}", plan_bytes(m[net]))
            m[net].config.global_pool_conditions = False
    for k in list(m):
        del m[k]
    torch.cuda.empty_cache()

    from powerpaint_b200.models.autoencoder_kl import AutoencoderKL

    vae = AutoencoderKL(sample_size=512).to(dev)
    vb = lambda: last_bytes(vae.engine())  # noqa: E731
    vae.encode(torch.rand(1, 3, 512, 512, device=dev, generator=g) * 2 - 1)
    emit("vae_encode_512", vb())
    vae.decode(torch.randn(1, 4, 64, 64, device=dev, generator=g))
    emit("vae_decode_512", vb())
    vae.enable_tiling()
    vae.encode(torch.rand(1, 3, 1360, 1024, device=dev, generator=g) * 2 - 1)
    emit("vae_encode_tiled_1024x1360", vb())
    vae.decode(torch.randn(1, 4, 170, 128, device=dev, generator=g))
    emit("vae_decode_tiled_1024x1360", vb())
    del vae
    torch.cuda.empty_cache()

    from powerpaint_b200.models import CLIPTextModel

    te = CLIPTextModel().to(dev)
    ids = torch.randint(0, 49405, (2, 77), generator=torch.Generator().manual_seed(1))
    te(ids)
    emit("clip_2x77", [])
    del te
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from synthetic_clip import make_text_encoder, make_tokenizer

    from powerpaint_b200.utils import TokenizerWrapper, add_tokens

    tok = TokenizerWrapper.from_tokenizer(make_tokenizer())
    te = CLIPTextModel.from_transformers(make_text_encoder(len(tok.wrapped), seed=0))
    add_tokens(tokenizer=tok, text_encoder=te, placeholder_tokens=["P_ctxt", "P_shape", "P_obj"],
               initialize_tokens=["a", "a", "a"], num_vectors_per_token=10)
    te = te.to(dev)
    ids = tok(["P_ctxt a cat", "P_obj the dog on P_shape"], padding="max_length", max_length=77, truncation=True,
              return_tensors="pt").input_ids
    te(ids)
    emit("clip_2x77_added_tokens", [])
    return written


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--switch", default=None, help="internal: run one switch set in this process")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.switch is not None:
        written = run_cases(args.out, args.switch, census_only=args.switch != "default")
        for name, n in written:
            print(f"{args.switch:14s} {name:34s} {n:6d} ops")
        return
    for sw, env in SWITCHES.items():  # the switches are read at import time: one process per set
        subprocess.run([sys.executable, os.path.abspath(__file__), "--out", args.out, "--switch", sw],
                       env=dict(os.environ, **env), check=True)


if __name__ == "__main__":
    main()
