"""CPU tests of the ONNX path: the oracle's graph interpreter (oracle/onnx_ref.py) against the PyTorch modules
that produced the files -- the reference's own export check (student_onnx_model.py:640-650, max diff < 1e-5) --
and the library's host-side loader / lowering (am_clap_describe_file needs no GPU)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from audiomuse_ai_b200 import _lib, weights
from oracle import mobilenet, onnx_ref, phinet
from tests import onnx_export, onnx_rewrite


def describe(path):
    lib = _lib.load()
    buf = C.create_string_buffer(1 << 16)
    r = lib.am_clap_describe_file(os.fsencode(path), buf, 1 << 16)
    if r < 0:
        raise _lib.B200Error(r, _lib.last_error())
    return buf.value.decode()


@pytest.fixture(scope="module")
def small_student():
    cfg = phinet.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256)
    return cfg, phinet.make_random_student(3, cfg)


@pytest.fixture(scope="module")
def small_mn():
    cfg = mobilenet.MNConfig(rows=mobilenet.SMALL_ROWS, head_dim=256)
    return cfg, mobilenet.make_random_mobilenet(5, cfg)


def test_interpreter_matches_torch_student(small_student):
    _, model = small_student
    g = onnx_ref.load(onnx_export.export_onnx_bytes(model))
    assert g.inputs == ["mel_spectrogram"] and g.outputs == ["embedding"] and g.opset == 17
    for T in (301, 1001):  # dynamic time axis
        x = phinet.synthetic_mel(1, 128, T, 7)
        with torch.no_grad():
            want = model(x).numpy()
        got = onnx_ref.run(g, {"mel_spectrogram": x.numpy()})[0]
        assert got.shape == (1, 512)
        assert np.abs(got - want).max() < 1e-5


def test_interpreter_matches_torch_mobilenet_and_rewrites(small_mn, tmp_path):
    _, model = small_mn
    raw = onnx_export.export_onnx_bytes(model)
    x = phinet.synthetic_mel(1, 128, 257, 9)
    with torch.no_grad():
        want = model(x).numpy()
    ext, blob = onnx_rewrite.externalize(raw, "m.onnx.data")
    (tmp_path / "m.onnx").write_bytes(ext)
    (tmp_path / "m.onnx.data").write_bytes(blob)
    assert len(ext) < len(raw) // 10
    for g in (onnx_ref.load(raw), onnx_ref.load(onnx_rewrite.attrs_to_inputs(raw)), onnx_ref.load(str(tmp_path / "m.onnx"))):
        got = onnx_ref.run(g, {"mel_spectrogram": x.numpy()})[0]
        assert np.abs(got - want).max() < 1e-5
    ops = {n.op for n in onnx_ref.load(raw).nodes}
    assert {"GlobalAveragePool", "HardSigmoid", "Gemm", "Relu"} <= ops  # a structurally different graph


class _FunctionalHeadStudent(phinet.StudentCLAPAudio):
    """The student with its projection head written out by hand, in the forms the exporter then writes: GELU as
    (x * 0.5) * (1 + erf(x * sqrt(1/2))), LayerNorm with Mul(d, d) for the square, and F.normalize's clamp as Max."""

    def forward(self, mel_spec):
        feats = self.phinet(mel_spec.squeeze(1).transpose(1, 2))
        h = self.projection_head
        e1 = h.linear1(feats)
        x = e1 + h.linear2(e1 * 0.5 * (1.0 + torch.erf(e1 * math.sqrt(0.5))))
        d = x - x.mean(-1, keepdim=True)
        ln = h.layer_norm
        x = d / torch.sqrt((d * d).mean(-1, keepdim=True) + ln.eps) * ln.weight + ln.bias
        return x / torch.maximum(x.norm(p=2, dim=1, keepdim=True), torch.tensor(1e-12))


def test_loader_lowers_student_onnx_like_the_blob(small_student, tmp_path):
    """The graph-driven lowering of the exported student must arrive at the same layer program as the
    hand-written state_dict exporter (weights.export_blob), whether the head's GELU, LayerNorm and L2 normalise
    come from modules or are written out by hand (_FunctionalHeadStudent)."""
    cfg, model = small_student
    functional = _FunctionalHeadStudent(cfg)
    functional.load_state_dict(model.state_dict())
    p_onnx = onnx_export.export_onnx(model, str(tmp_path / "s.onnx"))
    p_fn = onnx_export.export_onnx(functional, str(tmp_path / "fn.onnx"))
    with open(p_fn, "rb") as f:
        data = f.read()
    assert b"\x22\x03Max" in data and b"\x22\x03Pow" not in data and b"LayerNormalization" not in data
    wcfg = weights.StudentConfig(alpha=cfg.alpha, num_layers=cfg.num_layers, trunk_dim=cfg.trunk_dim)
    p_amw = tmp_path / "s.amw"
    p_amw.write_bytes(weights.export_blob(model.state_dict(), wcfg))
    d_onnx, d_amw = describe(p_onnx).splitlines(), describe(str(p_amw)).splitlines()
    assert d_onnx[0].startswith("source ONNX (ir") and d_amw[0].startswith("source AMW1")
    strip = lambda lines: [" ".join(l.split()) for l in lines[1:]]

    def norm(lines):  # register numbering differs (the ONNX walk allocates registers for fused intermediates)
        import re
        return [re.sub(r"r-?\d+", "r", l) for l in strip(lines)]

    assert norm(describe(p_fn).splitlines()) == norm(d_amw)
    assert norm(d_onnx) == norm(d_amw)
    assert "stem" in d_onnx[1] and "H=time" in d_onnx[1]
    assert sum("+residual" in l for l in d_onnx) == 3
    assert d_onnx[-1].split()[1] == "add_layernorm_l2"


def test_loader_lowers_mobilenet_and_all_encodings(small_mn, tmp_path):
    _, model = small_mn
    raw = onnx_export.export_onnx_bytes(model)
    (tmp_path / "a.onnx").write_bytes(raw)
    (tmp_path / "b.onnx").write_bytes(onnx_rewrite.attrs_to_inputs(raw))
    ext, blob = onnx_rewrite.externalize(raw, "c.onnx.data")
    (tmp_path / "c.onnx").write_bytes(ext)
    (tmp_path / "c.onnx.data").write_bytes(blob)
    d = [describe(str(tmp_path / f)) for f in ("a.onnx", "b.onnx", "c.onnx")]
    assert d[0] == d[1] == d[2]
    lines = d[0].splitlines()
    assert "conv_first" in lines[1] and "H=mel" in lines[1] and "hardswish" in lines[1]
    assert sum("squeeze_excite" in l for l in lines) == 4
    assert any("k 5x5" in l for l in lines)
    assert lines[-1].split()[1] == "l2norm"
    # external data without its side file: a clean error, not a crash
    os.remove(tmp_path / "c.onnx.data")
    with pytest.raises(_lib.B200Error) as e:
        describe(str(tmp_path / "c.onnx"))
    assert "external data" in str(e.value)


def test_loader_rejects_what_it_cannot_run(small_mn, tmp_path):
    _, model = small_mn
    raw = onnx_export.export_onnx_bytes(model)
    # same-length operator rename keeps the protobuf valid: Relu -> Selu (unsupported)
    bad = raw.replace(b"\x22\x04Relu", b"\x22\x04Selu", 1)
    assert bad != raw
    (tmp_path / "bad.onnx").write_bytes(bad)
    with pytest.raises(_lib.B200Error) as e:
        describe(str(tmp_path / "bad.onnx"))
    assert "Selu" in str(e.value) and "cannot lower node" in str(e.value)
    (tmp_path / "trunc.onnx").write_bytes(raw[: len(raw) // 2])
    with pytest.raises(_lib.B200Error):
        describe(str(tmp_path / "trunc.onnx"))
    (tmp_path / "junk.bin").write_bytes(b"\x00" * 64)
    with pytest.raises(_lib.B200Error):
        describe(str(tmp_path / "junk.bin"))
