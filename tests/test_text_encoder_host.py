"""CPU tests of the CLAP text tower: the plain-torch oracle (oracle/clap_text.py) against transformers' RobertaModel,
the library's host-side lowering of exported text graphs (am_text_describe_file needs no GPU), the C ABI's new
symbols and the integration hook's wiring."""
import ctypes as C
import os
import re
import subprocess
import sys
import types

import numpy as np
import pytest

from audiomuse_ai_b200 import _lib, integration
from oracle import clap_text as ct
from tests import onnx_rewrite

VARIANTS = [("eager", "arith"), ("eager", "where"), ("sdpa", "arith"), ("sdpa", "where")]


def describe(path):
    lib = _lib.load()
    buf = C.create_string_buffer(1 << 16)
    r = lib.am_text_describe_file(os.fsencode(path), buf, 1 << 16)
    if r < 0:
        raise _lib.B200Error(r, _lib.last_error())
    return buf.value.decode()


def _feeds(cfg, B, T, seed):
    g = np.random.default_rng(seed)
    ids = g.integers(3, cfg.vocab, size=(B, T)).astype(np.int64)
    mask = np.ones((B, T), np.int64)
    ids[:, 0] = 0  # <s>
    if B > 1:
        n = max(2, T // 2)
        ids[1, n:] = cfg.pad_id
        mask[1, n:] = 0
    if B > 2:
        ids[2, 1:] = cfg.pad_id  # everything after <s> is padding
        mask[2, 1:] = 0
    return ids, mask


_PIN = """
import sys
import numpy as np
import torch
import transformers
from oracle import clap_text as ct
from tests.test_text_encoder_host import _feeds

attention, mask = sys.argv[1], sys.argv[2]
cfg = ct.small_config()
model = ct.TextCLAP(cfg, attention, mask).init_random(7).double().eval()
rc = transformers.RobertaConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
                                num_attention_heads=cfg.heads, intermediate_size=cfg.ffn,
                                max_position_embeddings=cfg.max_pos, pad_token_id=cfg.pad_id, layer_norm_eps=cfg.eps,
                                type_vocab_size=cfg.type_vocab, hidden_dropout_prob=0.0,
                                attention_probs_dropout_prob=0.0, attn_implementation="eager")
rob = transformers.RobertaModel(rc, add_pooling_layer=True).double().eval()
rob_sd, proj_sd = ct.transformers_state_dict(model)
missing, unexpected = rob.load_state_dict(rob_sd, strict=False)
assert not unexpected and all("position_ids" in k or "token_type_ids" in k for k in missing), (missing, unexpected)
proj = torch.nn.Sequential(torch.nn.Linear(cfg.hidden, cfg.proj), torch.nn.ReLU(),
                           torch.nn.Linear(cfg.proj, cfg.proj)).double()
proj.load_state_dict(proj_sd)
ids, m = _feeds(cfg, 3, 16, 1)
with torch.no_grad():
    out = rob(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(m)).pooler_output
    ref = torch.nn.functional.normalize(proj(out), dim=-1)
print(float(np.abs(ct.run(model, ids, m) - ref.numpy()).max()))
"""


@pytest.mark.parametrize("attention,mask", VARIANTS)
def test_oracle_matches_transformers_float64(attention, mask):
    """Padded rows and a row that is all padding after <s>.  transformers runs in a child process: building a
    RobertaModel imports the ONNX exporter's opset-11 symbolics, which would change later audio-model exports."""
    pytest.importorskip("transformers")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _PIN, attention, mask], cwd=root, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    assert float(r.stdout.strip().splitlines()[-1]) <= 1e-10


@pytest.fixture(scope="module")
def small_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("text_onnx")
    cfg = ct.small_config()
    out = {}
    for att, mk in VARIANTS:
        p = str(d / f"text_{att}_{mk}.onnx")
        with open(p, "wb") as f:
            f.write(ct.export_onnx_bytes(ct.TextCLAP(cfg, att, mk).init_random(3)))
        out[(att, mk)] = p
    return cfg, out


def _expect_program(text, cfg, attention, mask):
    head = (f"text model: {cfg.layers} layers; hidden {cfg.hidden}; heads {cfg.heads} x {cfg.hidden // cfg.heads}; "
            f"ffn {cfg.ffn}; vocab {cfg.vocab}; positions {cfg.max_pos}; pad id {cfg.pad_id}")
    assert text.startswith(head), text
    assert ("sdpa" if attention == "sdpa" else "eager") in text.splitlines()[1]
    assert ("Where" if mask == "where" else "Sub/Mul") in text.splitlines()[1]
    scale = float(re.search(r"score scale ([0-9.e-]+)", text).group(1))
    assert scale == pytest.approx(1.0 / np.sqrt(cfg.hidden // cfg.heads), rel=1e-6)
    H, F = cfg.hidden, cfg.ffn
    layer_lines = [ln for ln in text.splitlines() if re.match(r"L\d+ ", ln)]
    assert len(layer_lines) == cfg.layers
    for ln in layer_lines:
        assert f"qkv {H}->{3 * H}" in ln and f"out {H}->{H} +res" in ln and f"ffn {H}->{F} gelu  {F}->{H} +res" in ln
    assert (f"pooler token 0 {H}->{H} tanh; projection {H}->{cfg.proj} relu {cfg.proj}->{cfg.proj}; l2 normalise"
            in text)


@pytest.mark.parametrize("attention,mask", VARIANTS)
def test_describe_lowers_every_attention_and_mask_form(small_files, attention, mask):
    cfg, files = small_files
    _expect_program(describe(files[(attention, mask)]), cfg, attention, mask)


@pytest.mark.parametrize("attention,mask,ln_op", [
    pytest.param("eager", "arith", True, id="eager-arith"),
    pytest.param("sdpa", "where", True, id="sdpa-where"),
    pytest.param("eager", "where", False, id="eager-where-ln_without_affine")])
def test_describe_layernorm_op_and_functional_gelu(tmp_path, attention, mask, ln_op):
    """nn.LayerNorm and F.gelu, as RobertaModel writes them: one LayerNormalization op and Div/Erf/Add/Mul/Mul.  Without
    ln_op, decomposed LayerNorms without scale and shift (their Div is the hidden state) and F.gelu."""
    cfg = ct.small_config()
    model = ct.TextCLAP(cfg, attention, mask, layernorm_op=ln_op, gelu="F", ln_affine=ln_op).init_random(4)
    data = ct.export_onnx_bytes(model)
    assert (data.count(b"LayerNormalization") >= 2 * cfg.layers + 1) == ln_op
    p = str(tmp_path / "ln_op.onnx")
    with open(p, "wb") as f:
        f.write(data)
    _expect_program(describe(p), cfg, attention, mask)


def test_describe_with_external_data(small_files, tmp_path):
    cfg, files = small_files
    with open(files[("sdpa", "where")], "rb") as f:
        data = f.read()
    p = str(tmp_path / "ext.onnx")
    model, blob = onnx_rewrite.externalize(data, "ext.onnx.data")
    assert len(model) < len(data) // 10
    with open(p, "wb") as f:
        f.write(model)
    with open(p + ".data", "wb") as f:
        f.write(blob)
    _expect_program(describe(p), cfg, "sdpa", "where")
    os.remove(p + ".data")
    with pytest.raises(_lib.B200Error, match="external data"):
        describe(p)


def test_describe_roberta_base_size(tmp_path):
    cfg = ct.ROBERTA_BASE
    p = str(tmp_path / "roberta_base.onnx")
    with open(p, "wb") as f:
        f.write(ct.export_onnx_bytes(ct.TextCLAP(cfg, "sdpa", "where")))
    text = describe(p)
    _expect_program(text, cfg, "sdpa", "where")
    assert "text model: 12 layers; hidden 768; heads 12 x 64; ffn 3072; vocab 50265; positions 514; pad id 1" in text


def test_unsupported_node_fails_the_load_and_names_it(small_files, tmp_path):
    _, files = small_files
    with open(files[("eager", "arith")], "rb") as f:
        data = f.read()
    assert b"Tanh" in data
    p = str(tmp_path / "bad.onnx")
    with open(p, "wb") as f:
        f.write(data.replace(b"Tanh", b"Sinh"))  # the pooler's activation, renamed consistently
    with pytest.raises(_lib.B200Error, match=r"cannot lower node 'Sinh_\d+' \(Sinh\)"):
        describe(p)


def test_header_declares_the_text_entry_points():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "audiomuse_b200.h")) as f:
        hdr = f.read()
    names = ["am_text_load", "am_text_load_mem", "am_text_describe_file", "am_text_embedding_dim",
             "am_text_release_workspace", "am_text_free", "am_text_embed"]
    for n in names:
        assert re.search(r"AM_API [^;]*\b" + n + r"\(", hdr), n
        assert n in _lib.SIGNATURES
    assert "int am_text_embed(am_text_model* m, const int64_t* ids, const int64_t* mask, int B, int T, float* out)" in hdr


class _Session:
    def __init__(self):
        self.closed = False

    def close(self):
        self.closed = True


def test_apply_clap_text_replaces_the_loader_and_extends_unload(monkeypatch):
    from audiomuse_ai_b200 import clap_analyzer as b200_clap

    made = []

    class FakeTextSession:
        def __init__(self, path=None, blob=None):
            made.append(path)

    monkeypatch.setattr(b200_clap, "B200TextSession", FakeTextSession)
    ref = types.SimpleNamespace(config=types.SimpleNamespace(CLAP_TEXT_MODEL_PATH="/models/a.onnx"),
                                _text_session=None, _tokenizer=None, _load_text_model=None,
                                unload_clap_model=lambda: False, is_clap_model_loaded=lambda: False)
    integration._apply_clap_text(ref, None)
    ref.config.CLAP_TEXT_MODEL_PATH = "/models/b.onnx"  # read at call time
    assert isinstance(ref._load_text_model(), FakeTextSession) and made == ["/models/b.onnx"]
    assert ref.is_clap_model_loaded() is False  # without clap= nothing else changes

    audio = {"loaded": True}

    def unload_audio():
        was, audio["loaded"] = audio["loaded"], False
        return was

    ref.unload_clap_model, ref.is_clap_model_loaded = unload_audio, lambda: audio["loaded"]
    integration._apply_clap_text(ref, ref)
    s = _Session()
    ref._text_session, ref._tokenizer = s, object()
    assert ref.is_clap_model_loaded()
    assert ref.unload_clap_model() is True
    assert s.closed and ref._text_session is None and ref._tokenizer is None and not audio["loaded"]
    assert not ref.is_clap_model_loaded() and ref.unload_clap_model() is False
