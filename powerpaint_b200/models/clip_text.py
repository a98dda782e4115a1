"""CLIP text encoder on the repo's CUDA kernels — SURVEY.md §8f row 2.

Drop-in for the `transformers.CLIPTextModel` the reference pipelines inject as `text_encoder` /
`text_encoder_brushnet` (`self.text_encoder(text_input_ids)[0]`, powerpaint/pipelines/pipeline_PowerPaint.py:
317-518; the app builds it at app.py:84-112 and runs `add_tokens(...)` on it). Same module tree and state-dict
names (`text_model.embeddings.{token,position}_embedding`, `text_model.encoder.layers.{i}.{self_attn.{q,k,v,out}_proj,
layer_norm1, mlp.{fc1,fc2}, layer_norm2}`, `text_model.final_layer_norm`), so `add_tokens` can swap
`text_model.embeddings.token_embedding` for `EmbeddingLayerWithFixes` exactly as it does upstream and
`text_encoder/model.safetensors` loads unchanged.

`forward` replays one recorded `pp_program` (CUDA graph): embedding gather (the task-prompt splice of
`EmbeddingLayerWithFixes` — reference utils.py:387-445, a per-row Python loop with host syncs — is resolved on the
host into ONE gather index per position, including the reference's adjacent-run scan quirk), then per layer
LayerNorm -> q|k|v GEMM -> causal attention -> out_proj(+residual) -> LayerNorm -> fc1 + quick_gelu -> fc2(+residual),
and the final LayerNorm. No CPU path.
"""
from __future__ import annotations

from collections import OrderedDict
from types import SimpleNamespace

import torch
import torch.nn as nn

from .. import _native as N
from ..config import Config
from ..engine import BF16, Plan, Pool, Recorder
from .base import KernelModule


def clip_param_shapes(cfg) -> "OrderedDict[str, tuple]":
    d: "OrderedDict[str, tuple]" = OrderedDict()
    H, I = cfg.hidden_size, cfg.intermediate_size
    d["text_model.embeddings.token_embedding.weight"] = (cfg.vocab_size, H)
    d["text_model.embeddings.position_embedding.weight"] = (cfg.max_position_embeddings, H)
    for i in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}"
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            d[f"{p}.self_attn.{n}.weight"] = (H, H)
            d[f"{p}.self_attn.{n}.bias"] = (H,)
        for n in ("layer_norm1", "layer_norm2"):
            d[f"{p}.{n}.weight"] = (H,)
            d[f"{p}.{n}.bias"] = (H,)
        d[f"{p}.mlp.fc1.weight"] = (I, H)
        d[f"{p}.mlp.fc1.bias"] = (I,)
        d[f"{p}.mlp.fc2.weight"] = (H, I)
        d[f"{p}.mlp.fc2.bias"] = (H,)
    d["text_model.final_layer_norm.weight"] = (H,)
    d["text_model.final_layer_norm.bias"] = (H,)
    return d


class ClipEngine(Recorder):
    """records the text transformer for a fixed (batch, seq) as one program"""

    MAX_PLANS = 4

    def plan_for(self, nb: int, seq: int, n_ext: int) -> Plan:
        return self._plan((nb, seq, n_ext), lambda: self._build(nb, seq, n_ext), graph=True)

    def _build(self, nb, seq, n_ext) -> Plan:
        cfg = self.cfg
        H, heads = cfg.hidden_size, cfg.num_attention_heads
        d = H // heads
        M = nb * seq
        eps = cfg.layer_norm_eps
        act = {"quick_gelu": N.PP_ACT_QUICK_GELU}.get(cfg.hidden_act)
        if act is None:
            raise NotImplementedError(f"hidden_act {cfg.hidden_act!r}: the CLIP ViT-L/14 text tower of SD-1.5 uses quick_gelu")
        plan = Plan(Pool(self.device))
        prog = plan.program
        idx = torch.zeros(M, dtype=torch.int32, device=self.device)
        ext = torch.zeros(max(n_ext, 1), H, dtype=torch.float32, device=self.device)
        plan.inputs["idx"], plan.inputs["ext"] = idx, ext
        base = self.vec("text_model.embeddings.token_embedding.weight")
        pos = self.vec("text_model.embeddings.position_embedding.weight")
        x = plan.pool.buf(M, H)
        prog.add_embed_gather(idx, base, ext, pos, x, M, base.shape[0], seq, H)
        scale = d ** -0.5
        for i in range(cfg.num_hidden_layers):
            p = f"text_model.encoder.layers.{i}"
            l1 = plan.pool.buf(M, H)
            prog.add_layer_norm(x, l1, self.vec(p + ".layer_norm1.weight"), self.vec(p + ".layer_norm1.bias"), M, H, eps)
            wqkv = self._cached("qkv:" + p, lambda p=p: torch.cat(
                [self._raw(f"{p}.self_attn.{n}.weight") for n in ("q_proj", "k_proj", "v_proj")], 0).to(BF16).contiguous())
            bqkv = self._cached("qkvb:" + p, lambda p=p: torch.cat(
                [self._raw(f"{p}.self_attn.{n}.bias") for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous())
            qkv = self._linear(plan, prog, l1, M, None, 3 * H, w=wqkv, bias=bqkv)
            plan.pool.free(l1)
            a = plan.pool.buf(M, H)
            prog.add_causal_attention_small(qkv, a, nb, seq, heads, d, scale)
            plan.pool.free(qkv)
            x1 = self._linear(plan, prog, a, M, p + ".self_attn.out_proj", H, bias=self.vec(p + ".self_attn.out_proj.bias"),
                              res1=x)
            plan.pool.free(a, x)
            l2 = plan.pool.buf(M, H)
            prog.add_layer_norm(x1, l2, self.vec(p + ".layer_norm2.weight"), self.vec(p + ".layer_norm2.bias"), M, H, eps)
            f = self._linear(plan, prog, l2, M, p + ".mlp.fc1", cfg.intermediate_size, bias=self.vec(p + ".mlp.fc1.bias"),
                             act=act)
            plan.pool.free(l2)
            x = self._linear(plan, prog, f, M, p + ".mlp.fc2", H, bias=self.vec(p + ".mlp.fc2.bias"), res1=x1)
            plan.pool.free(f, x1)
        out = torch.empty(M, H, dtype=BF16, device=self.device)
        prog.add_layer_norm(x, out, self.vec("text_model.final_layer_norm.weight"),
                            self.vec("text_model.final_layer_norm.bias"), M, H, eps)
        plan.pool.free(x)
        plan.outputs["hidden"] = out
        return plan


class CLIPTextModel(KernelModule):
    def __init__(self, vocab_size: int = 49408, hidden_size: int = 768, intermediate_size: int = 3072,
                 num_hidden_layers: int = 12, num_attention_heads: int = 12, max_position_embeddings: int = 77,
                 layer_norm_eps: float = 1e-5, hidden_act: str = "quick_gelu", **unused):
        super().__init__()
        self.config = Config(vocab_size=vocab_size, hidden_size=hidden_size, intermediate_size=intermediate_size,
                             num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                             max_position_embeddings=max_position_embeddings, layer_norm_eps=layer_norm_eps,
                             hidden_act=hidden_act)
        if hidden_size % num_attention_heads or hidden_size // num_attention_heads not in (8, 16, 32, 64):
            raise NotImplementedError("head dim must be 8, 16, 32 or 64")
        if max_position_embeddings > 128:
            raise NotImplementedError("at most 128 positions (CLIP: 77)")
        self.text_model = nn.Module()
        emb = self.text_model.embeddings = nn.Module()
        emb.token_embedding = nn.Embedding(vocab_size, hidden_size)
        emb.position_embedding = nn.Embedding(max_position_embeddings, hidden_size)
        for name, shape in clip_param_shapes(self.config).items():
            if ".embeddings." in name:
                continue
            self._register(name, torch.zeros(shape))
        for p in self.parameters():
            p.requires_grad_(False)

    @property
    def device(self):
        return self.text_model.embeddings.position_embedding.weight.device

    @classmethod
    def from_transformers(cls, model) -> "CLIPTextModel":
        """copy config + weights of a `transformers.CLIPTextModel` (an `EmbeddingLayerWithFixes` already installed
        by `add_tokens` is carried over as is)"""
        c = model.config
        m = cls(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                max_position_embeddings=c.max_position_embeddings, layer_norm_eps=c.layer_norm_eps,
                hidden_act=c.hidden_act)
        tok = model.text_model.embeddings.token_embedding
        sd = {k: v for k, v in model.state_dict().items() if "position_ids" not in k}
        if hasattr(tok, "wrapped"):  # EmbeddingLayerWithFixes
            m.text_model.embeddings.token_embedding = tok
        m.load_state_dict(sd, strict=True)
        return m

    def get_input_embeddings(self):
        return self.text_model.embeddings.token_embedding

    def _make_engine(self, state_dict, device) -> ClipEngine:
        # EmbeddingLayerWithFixes keeps the base table under `.wrapped.weight`
        sd = {k.replace("token_embedding.wrapped.weight", "token_embedding.weight"): v for k, v in state_dict.items()}
        return ClipEngine(self.config, sd, device)

    # ---- the task-prompt splice, resolved to gather indices on the host
    def _gather_plan(self, input_ids: torch.Tensor):
        """(index [B, L] int32, ext [n, H] fp32): position p reads base row index[p] if < vocab, else row
        index[p] - vocab of `ext` — exactly what EmbeddingLayerWithFixes.forward produces (utils.py:447-483),
        including its asserts on malformed placeholder runs and the adjacent-run scan quirk (:438-439)."""
        tok = self.text_model.embeddings.token_embedding
        V = self.config.vocab_size
        ids = input_ids.detach().to("cpu", torch.int64)
        if ids.ndim == 1:
            ids = ids.unsqueeze(0)
        externals = list(getattr(tok, "external_embeddings", []))
        if not externals:
            if (ids >= V).any() or (ids < 0).any():
                raise IndexError("token id out of range")
            return ids.to(torch.int32), None
        num = tok.num_embeddings
        idx = torch.where(ids >= num, torch.zeros_like(ids), ids)  # replace_input_ids (:387-389)
        offs, tabs, o = {}, [], 0
        for e in externals:
            t = tok._embedding_of(e).detach().float()
            offs[e["name"]] = o
            o += t.shape[0]
            tabs.append(t)
        if (ids >= num).any():
            for r in range(ids.shape[0]):
                row = ids[r]
                for e in externals:
                    start, end, name = e["start"], e["end"], e["name"]
                    n = end - start
                    pos = (row == start).nonzero(as_tuple=False).flatten().tolist()
                    skip = -1
                    for p in pos:
                        if p == skip:
                            continue  # the reference's scan resumes one position after a replaced run
                        actual = [int(i) for i in row[p:p + n]]
                        target = list(range(start, end))
                        assert actual == target, (f"Invalid 'input_ids' in position: {p} to {p + n}. Expect '{target}' "
                                                  f"for embedding '{name}' but found '{actual}'.")
                        idx[r, p:p + n] = V + offs[name] + torch.arange(n)
                        skip = p + n
        return idx.to(torch.int32), torch.cat(tabs, 0)

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask=None, position_ids=None, output_attentions=None,
                output_hidden_states=None, return_dict=None):
        if attention_mask is not None or position_ids is not None or output_attentions or output_hidden_states:
            raise NotImplementedError("attention_mask / position_ids / extra outputs are outside the PowerPaint path "
                                      "(the pipelines pass input_ids only, pipeline_PowerPaint.py:402-410)")
        if input_ids.ndim == 1:
            input_ids = input_ids.unsqueeze(0)
        nb, seq = input_ids.shape
        if seq > self.config.max_position_embeddings:
            raise ValueError(f"sequence length {seq} exceeds max_position_embeddings")
        eng = self.engine()
        idx, ext = self._gather_plan(input_ids)
        tok = self.text_model.embeddings.token_embedding
        base = tok.wrapped.weight if hasattr(tok, "wrapped") else tok.weight
        if base.shape[0] != self.config.vocab_size:
            raise ValueError("token embedding table does not match config.vocab_size")
        with torch.cuda.device(self.device):
            plan = eng.plan_for(nb, seq, 0 if ext is None else ext.shape[0])
            plan.inputs["idx"].copy_(idx.reshape(-1).to(self.device))
            if ext is not None:
                plan.inputs["ext"].copy_(ext.to(self.device))
            plan.program.launch()
            hidden = plan.outputs["hidden"].view(nb, seq, -1).to(self._out_dtype)
        # pooled output like transformers (eos = highest id for the original CLIP vocabulary)
        eos = input_ids.to(hidden.device).to(torch.int64).argmax(dim=-1)
        pooled = hidden[torch.arange(nb, device=hidden.device), eos]
        if return_dict is False:
            return (hidden, pooled)
        out = _Output(last_hidden_state=hidden, pooler_output=pooled)
        return out


class _Output(SimpleNamespace):
    """attribute + index access like transformers' BaseModelOutputWithPooling (`text_encoder(ids)[0]`)"""

    def __getitem__(self, i):
        return (self.last_hidden_state, self.pooler_output)[i]
