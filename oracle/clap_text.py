"""Oracle: the CLAP text tower (``TextCLAPWrapper`` of the reference's ``query/pythorch.sh:95-127``) in plain PyTorch.

The deployed ``clap_text_model.onnx`` is ``TextCLAPWrapper`` exported with ``torch.onnx.export(opset 17,
do_constant_folding=True, dynamo=False)``: a transformers ``RobertaModel`` (``text_branch``), its pooler
``tanh(dense(h[:, 0]))``, ``text_projection = Linear -> ReLU -> Linear`` and ``F.normalize``.  transformers' masking
utilities do not trace, so this module restates the model with plain tensor operations, in float64 or float32:

* its state dict has the parameter names of ``RobertaModel`` (under ``text_branch.``) and of ``text_projection``, so
  weights load both ways (``tests/test_text_encoder_host.py`` pins it against ``RobertaModel(attn_implementation=
  "eager")`` in float64);
* ``attention`` selects the graph the TorchScript exporter writes: ``"eager"`` is transformers' eager attention
  (``MatMul(Q, K^T) -> Div(sqrt(d)) -> Add(mask) -> Softmax -> MatMul(V)``), ``"sdpa"`` is the opset-14 symbolic of
  ``scaled_dot_product_attention`` written out by hand (``Mul(Q, sqrt(s))``, ``Mul(K^T, sqrt(s))``, ``MatMul``,
  ``Add(mask)``, ``Softmax``, ``MatMul``);
* ``mask`` selects the additive mask's construction: ``"arith"`` is ``(1 - m) * finfo.min`` (``Cast/Sub/Mul``),
  ``"where"`` is transformers' ``masked_fill`` form (``Expand/Cast/Sub/Where``);
* ``layernorm_op=True`` and ``gelu="F"`` use ``nn.LayerNorm`` and ``F.gelu``, as ``RobertaModel`` does (the exporter
  writes one ``LayerNormalization`` op, and ``Div/Erf/Add/Mul/Mul``); the defaults write both out by hand;
* ``ln_affine=False`` drops every LayerNorm's scale and shift, so the decomposed form ends at its ``Div``;
* the position ids are RoBERTa's ``cumsum(ids != pad) * (ids != pad) + pad``; the token-type embedding is row 0 of
  its table, added as a constant (what constant folding leaves of it).

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class TextConfig:
    vocab: int = 50265
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    ffn: int = 3072
    max_pos: int = 514
    pad_id: int = 1
    eps: float = 1e-5
    type_vocab: int = 1
    proj: int = 512


ROBERTA_BASE = TextConfig()


def small_config(**kw) -> TextConfig:
    c = TextConfig(vocab=1000, hidden=128, layers=2, heads=4, ffn=512, max_pos=514, pad_id=1, proj=64)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


class _LN(nn.Module):
    def __init__(self, n, eps, affine=True):
        super().__init__()
        if affine:
            self.weight = nn.Parameter(torch.ones(n))
            self.bias = nn.Parameter(torch.zeros(n))
        self.eps, self.affine = eps, affine

    def forward(self, x):  # decomposed, as the exporter writes LayerNorm at opset 17 when it is not fused
        mu = x.mean(-1, keepdim=True)
        d = x - mu
        var = (d * d).mean(-1, keepdim=True)
        y = d / torch.sqrt(var + self.eps)
        return y * self.weight + self.bias if self.affine else y


class _Lin(nn.Module):
    def __init__(self, i, o):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(o, i))
        self.bias = nn.Parameter(torch.empty(o))

    def forward(self, x):
        return torch.matmul(x, self.weight.t()) + self.bias


def _ns(**kw):
    m = nn.Module()
    for k, v in kw.items():
        setattr(m, k, v)
    return m


class TextCLAP(nn.Module):
    def __init__(self, cfg: TextConfig, attention: str = "eager", mask: str = "arith", layernorm_op: bool = False,
                 gelu: str = "erf", ln_affine: bool = True):
        super().__init__()
        assert attention in ("eager", "sdpa") and mask in ("arith", "where") and gelu in ("erf", "F")
        assert ln_affine or not layernorm_op
        self.cfg, self.attention, self.mask_form, self.layernorm_op = cfg, attention, mask, layernorm_op
        self.gelu, self.ln_affine = gelu, ln_affine
        H = cfg.hidden
        ln = (lambda: nn.LayerNorm(H, eps=cfg.eps)) if layernorm_op else (lambda: _LN(H, cfg.eps, ln_affine))
        emb = _ns(word_embeddings=nn.Embedding(cfg.vocab, H, padding_idx=cfg.pad_id),
                  position_embeddings=nn.Embedding(cfg.max_pos, H, padding_idx=cfg.pad_id),
                  token_type_embeddings=nn.Embedding(cfg.type_vocab, H), LayerNorm=ln())
        layers = nn.ModuleList()
        for _ in range(cfg.layers):
            att = _ns(self=_ns(query=_Lin(H, H), key=_Lin(H, H), value=_Lin(H, H)),
                      output=_ns(dense=_Lin(H, H), LayerNorm=ln()))
            layers.append(_ns(attention=att, intermediate=_ns(dense=_Lin(H, cfg.ffn)),
                              output=_ns(dense=_Lin(cfg.ffn, H), LayerNorm=ln())))
        self.text_branch = _ns(embeddings=emb, encoder=_ns(layer=layers), pooler=_ns(dense=_Lin(H, H)))
        self.text_projection = nn.Sequential(nn.Linear(H, cfg.proj), nn.ReLU(), nn.Linear(cfg.proj, cfg.proj))

    def init_random(self, seed: int = 0, std: float = 0.02):
        """BERT-style N(0, std) weights with random LayerNorm affines and biases (so that none is the identity)."""
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p in self.named_parameters():
                if "LayerNorm.weight" in name:
                    p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g, dtype=torch.float64))
                elif name.endswith("bias"):
                    p.copy_(0.02 * torch.randn(p.shape, generator=g, dtype=torch.float64))
                else:
                    p.copy_(std * torch.randn(p.shape, generator=g, dtype=torch.float64))
        return self

    def forward(self, input_ids, attention_mask):
        cfg, dt = self.cfg, self.text_projection[0].weight.dtype
        tb = self.text_branch
        B, T = input_ids.shape
        nh, dh = cfg.heads, cfg.hidden // cfg.heads
        e = tb.embeddings
        m = input_ids.ne(cfg.pad_id).int()
        pos = (torch.cumsum(m, dim=1).type_as(m) * m).long() + cfg.pad_id
        x = e.word_embeddings(input_ids) + e.position_embeddings(pos) + e.token_type_embeddings.weight[0]
        h = e.LayerNorm(x)
        fmin = torch.finfo(dt).min
        if self.mask_form == "arith":
            add_mask = (1.0 - attention_mask[:, None, None, :].to(dt)) * fmin
        else:
            inv = 1.0 - attention_mask[:, None, None, :].expand(B, 1, T, T).to(dt)
            add_mask = inv.masked_fill(inv.to(torch.bool), fmin)
        for L in tb.encoder.layer:
            a = L.attention
            q = a.self.query(h).view(B, T, nh, dh).transpose(1, 2)
            k = a.self.key(h).view(B, T, nh, dh).transpose(1, 2)
            v = a.self.value(h).view(B, T, nh, dh).transpose(1, 2)
            if self.attention == "eager":
                s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(dh) + add_mask
            else:
                r = math.sqrt(1.0 / math.sqrt(dh))
                s = torch.matmul(q * r, k.transpose(-1, -2) * r) + add_mask
            ctx = torch.matmul(torch.softmax(s, dim=-1), v).transpose(1, 2).reshape(B, T, cfg.hidden)
            h = a.output.LayerNorm(a.output.dense(ctx) + h)
            f = L.intermediate.dense(h)
            if self.gelu == "F":  # what RobertaModel calls: x * 0.5 * (1 + erf(x / sqrt 2)) in the exporter's order
                f = F.gelu(f)
            else:
                f = f * 0.5 * (1.0 + torch.erf(f / math.sqrt(2.0)))
            h = L.output.LayerNorm(L.output.dense(f) + h)
        pooled = torch.tanh(tb.pooler.dense(h[:, 0]))
        return F.normalize(self.text_projection(pooled), dim=-1)


def transformers_state_dict(model: TextCLAP):
    """(RobertaModel state dict, text_projection state dict) of the oracle's weights."""
    sd = model.state_dict()
    rob = {k[len("text_branch."):]: v for k, v in sd.items() if k.startswith("text_branch.")}
    proj = {k[len("text_projection."):]: v for k, v in sd.items() if k.startswith("text_projection.")}
    return rob, proj


def export_onnx_bytes(model: TextCLAP, B: int = 1, T: int = 77) -> bytes:
    """ONNX bytes of `model` (in float32) with the reference's exporter arguments (opset 17, constant folding,
    input_ids and attention_mask int64 with dynamic batch and sequence axes, output text_embedding), through the two
    TorchScript exporter stages that need no ``onnx`` package (as tests/onnx_export.py does for the audio model).

    The export runs in a child process: it registers the exporter's opset 10-17 symbolics, which would otherwise stay
    registered and change what later exports at the exporter's default opset (the audio model's) produce."""
    import os
    import subprocess
    import sys
    import tempfile

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "model.pt"), os.path.join(d, "model.onnx")
        torch.save({"cfg": dict(model.cfg.__dict__), "attention": model.attention, "mask": model.mask_form,
                    "layernorm_op": model.layernorm_op, "gelu": model.gelu, "ln_affine": model.ln_affine,
                    "state": {k: v.float() for k, v in model.state_dict().items()}}, src)
        subprocess.run([sys.executable, "-m", "oracle.clap_text", src, dst, str(B), str(T)], cwd=root, check=True)
        with open(dst, "rb") as f:
            return f.read()


def _export_in_process(model: TextCLAP, B: int, T: int) -> bytes:
    import importlib
    import warnings

    from torch.onnx._internal.torchscript_exporter import utils as U
    from torch.onnx._internal.torchscript_exporter._globals import GLOBALS

    for v in range(10, 18):  # the symbolics of opsets 10-17 register on import
        importlib.import_module(f"torch.onnx._internal.torchscript_exporter.symbolic_opset{v}")
    model = model.float().eval()
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(3, model.cfg.vocab, (B, T), generator=g)
    mask = torch.ones(B, T, dtype=torch.long)
    dyn = {"input_ids": {0: "batch_size", 1: "sequence_length"},
           "attention_mask": {0: "batch_size", 1: "sequence_length"}, "text_embedding": {0: "batch_size"}}
    GLOBALS.export_onnx_opset_version = 17  # what torch.onnx.export(opset_version=17) sets around these stages
    with warnings.catch_warnings(), torch.no_grad():
        warnings.simplefilter("ignore")
        graph, params, _ = U._model_to_graph(model, (ids, mask), input_names=["input_ids", "attention_mask"],
                                             output_names=["text_embedding"], do_constant_folding=True,
                                             dynamic_axes=dyn)
        proto = graph._export_onnx(params, 17, dyn, False, torch.onnx.OperatorExportTypes.ONNX, True, True, {}, True,
                                   "", {})[0]
    return bytes(proto)


def run(model: TextCLAP, input_ids, attention_mask, dtype=torch.float64):
    """Embeddings f[B, proj] of int64 feeds (numpy or torch) by the oracle in `dtype`."""
    import numpy as np

    m = model.to(dtype).eval()
    with torch.no_grad():
        out = m(torch.as_tensor(np.asarray(input_ids), dtype=torch.long),
                torch.as_tensor(np.asarray(attention_mask), dtype=torch.long))
    return out.numpy()


if __name__ == "__main__":  # python -m oracle.clap_text <saved model> <out.onnx> B T  (export_onnx_bytes's child)
    import sys

    blob = torch.load(sys.argv[1])
    m = TextCLAP(TextConfig(**blob["cfg"]), blob["attention"], blob["mask"], blob["layernorm_op"], blob["gelu"],
                 blob["ln_affine"]).float()
    m.load_state_dict(blob["state"])
    with open(sys.argv[2], "wb") as f:
        f.write(_export_in_process(m, int(sys.argv[3]), int(sys.argv[4])))
