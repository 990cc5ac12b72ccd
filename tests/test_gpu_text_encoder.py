"""The CLAP text tower on the device (am_text_embed through B200TextSession) against the float64 oracle
(oracle/clap_text.py), on files exported with the reference's exporter arguments in both attention forms (eager and
the SDPA symbolic) and both mask constructions.  Bar: max |delta| <= 1e-4 per component and cosine >= 0.99999 (the
reference's own PyTorch -> ONNX check is < 1e-5; the observed maximum is printed).  Also: a row of a batch of 64
against the same row alone, bit-identical repeats, and the load / unload / reload cycle through
integration.apply(clap_text=..., clap=...)."""
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from audiomuse_ai_b200 import integration
from audiomuse_ai_b200.clap_analyzer import B200TextSession
from oracle import clap_text as ct

MAX_ABS, MIN_COS = 1e-4, 0.99999
VARIANTS = [("eager", "arith"), ("eager", "where"), ("sdpa", "arith"), ("sdpa", "where")]
_observed = []


def _feeds(cfg, B, T, seed):
    g = np.random.default_rng(seed)
    ids = g.integers(3, cfg.vocab, size=(B, T)).astype(np.int64)
    mask = np.ones((B, T), np.int64)
    ids[:, 0] = 0
    for b in range(1, B):  # padded rows of every length; row 2 is all padding after <s>
        n = 1 if b == 2 else max(1, T - (b * 7) % T)
        ids[b, n:] = cfg.pad_id
        mask[b, n:] = 0
    return ids, mask


def _check(sess, model, B, T, seed):
    ids, mask = _feeds(model.cfg, B, T, seed)
    got = sess.run(None, {"input_ids": ids, "attention_mask": mask})[0]
    want = ct.run(model, ids, mask)
    err = float(np.abs(got.astype(np.float64) - want).max())
    cos = float((np.sum(got * want, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(want, axis=1))).min())
    _observed.append(err)
    print(f"B={B} T={T}: max |delta| {err:.3g}, min cosine {cos:.9f}")
    assert err <= MAX_ABS and cos >= MIN_COS, (B, T, err, cos)
    return got


@pytest.fixture(scope="module")
def small():
    cfg = ct.small_config(heads=2)  # dh = 64, as in roberta-base
    out = {}
    for att, mk in VARIANTS:
        model = ct.TextCLAP(cfg, att, mk).init_random(5)
        out[(att, mk)] = (model, B200TextSession(blob=ct.export_onnx_bytes(model)))
    yield out
    for _, s in out.values():
        s.close()


@pytest.mark.parametrize("attention,mask", VARIANTS)
@pytest.mark.parametrize("B,T", [(1, 1), (1, 16), (1, 77), (3, 16), (3, 77), (3, 512), (64, 77)])
def test_matches_float64_oracle(small, attention, mask, B, T):
    model, sess = small[(attention, mask)]
    _check(sess, model, B, T, seed=B * 1000 + T)


def test_narrow_heads_and_batch_64_at_512(small):
    cfg = ct.small_config()  # 4 heads of 32
    model = ct.TextCLAP(cfg, "eager", "arith").init_random(9)
    sess = B200TextSession(blob=ct.export_onnx_bytes(model))
    try:
        _check(sess, model, 64, 512, seed=3)
        _check(sess, model, 3, 16, seed=4)
    finally:
        sess.close()


@pytest.mark.parametrize("attention,mask", [("eager", "arith"), ("sdpa", "where")])
def test_layernorm_op_and_functional_gelu_match_float64_oracle(attention, mask):
    """nn.LayerNorm and F.gelu as RobertaModel has them: the LayerNormalization op and the Div/Erf/Add/Mul/Mul GELU."""
    cfg = ct.small_config(heads=2)
    model = ct.TextCLAP(cfg, attention, mask, layernorm_op=True, gelu="F").init_random(6)
    sess = B200TextSession(blob=ct.export_onnx_bytes(model))
    try:
        for B, T in [(1, 77), (3, 77), (64, 77), (3, 512)]:
            _check(sess, model, B, T, seed=7 * B + T)
    finally:
        sess.close()


def test_odd_hidden_and_projection_widths_match_float64_oracle():
    """H = 96 (3 heads of 32: the attention output's K tail [96, 128) is padding) and a 61-wide projection."""
    cfg = ct.small_config(hidden=96, heads=3, ffn=200, proj=61)
    model = ct.TextCLAP(cfg, "eager", "arith").init_random(8)
    sess = B200TextSession(blob=ct.export_onnx_bytes(model))
    try:
        for B, T in [(1, 77), (3, 16), (64, 77)]:
            _check(sess, model, B, T, seed=B + 3 * T)
    finally:
        sess.close()


@pytest.fixture(scope="module")
def base():
    model = ct.TextCLAP(ct.ROBERTA_BASE, "sdpa", "where").init_random(1)
    sess = B200TextSession(blob=ct.export_onnx_bytes(model))
    yield model, sess
    sess.close()


@pytest.mark.parametrize("B,T", [(1, 77), (3, 77), (64, 77), (3, 512)])
def test_roberta_base_size_matches_float64_oracle(base, B, T):
    model, sess = base
    _check(sess, model, B, T, seed=B + T)


def test_batch_rows_match_rows_run_alone_and_repeats_are_bit_identical(base):
    model, sess = base
    ids, mask = _feeds(model.cfg, 64, 77, 21)
    feed = {"input_ids": ids, "attention_mask": mask}
    full = sess.run(None, feed)[0]
    assert np.array_equal(full, sess.run(None, feed)[0])
    for b in (0, 1, 2, 37, 63):
        one = {"input_ids": ids[b:b + 1], "attention_mask": mask[b:b + 1]}
        alone = sess.run(None, one)[0]
        assert np.array_equal(alone, sess.run(None, one)[0])
        err = float(np.abs(alone[0] - full[b]).max())
        assert err <= MAX_ABS, (b, err)


def test_lifecycle_through_apply(small, tmp_path):
    model, _ = small[("eager", "arith")]
    path = tmp_path / "clap_text_model.onnx"
    path.write_bytes(ct.export_onnx_bytes(model))
    ref = types.SimpleNamespace(config=types.SimpleNamespace(CLAP_TEXT_MODEL_PATH=str(path)), _text_session=None,
                                _tokenizer=None, _load_text_model=None)
    integration.apply(clap=ref, clap_text=ref)
    ids, mask = _feeds(model.cfg, 1, 77, 5)
    want = ct.run(model, ids, mask)
    for _ in range(2):  # load, unload by the idle timer's call, reload
        ref._text_session = ref._load_text_model()
        assert ref.is_clap_model_loaded()
        got = ref._text_session.run(None, {"input_ids": ids, "attention_mask": mask})[0]
        assert np.abs(got - want).max() <= MAX_ABS
        s = ref._text_session
        assert ref.unload_clap_model() is True
        assert ref._text_session is None and s._h is None and not ref.is_clap_model_loaded()


def test_report_observed_maximum():
    if _observed:
        print(f"largest max |delta| over every comparison: {max(_observed):.3g} (bound {MAX_ABS})")
