"""oracle/encoder_steps.py against PyTorch run in float64 on the same weights: each step function of the encoder-step
oracle (tests/test_gpu_encoder_steps_exact.py) must agree with the module it restates to about 1e-12 relative, and
its fault variants must be the faults they name.  No GPU."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import encoder_steps as O

TORCH_ACT = {O.ACT_NONE: lambda x: x, O.ACT_RELU6: F.relu6, O.ACT_RELU: F.relu, O.ACT_HSWISH: F.hardswish,
             O.ACT_GELU: F.gelu, O.ACT_SIGMOID: torch.sigmoid, O.ACT_HSIGMOID: F.hardsigmoid, O.ACT_TANH: torch.tanh}


def _close(got, want, rel=1e-12):
    want = np.asarray(want)
    scale = max(np.abs(want).max(), 1e-300)
    assert np.abs(got - want).max() <= rel * scale, np.abs(got - want).max() / scale


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64))


def _layer(**kw):
    L = dict(pad_t=0, pad_b=0, pad_l=0, pad_r=0, kh=1, kw=1, stride=1, act=0, gate_act=0, h_is_time=1, residual=0)
    L.update(kw)
    return L


@pytest.mark.parametrize("kind", range(8))
def test_activations(kind):
    v = np.linspace(-9, 9, 2001)
    _close(O.act(kind, v), TORCH_ACT[kind](_t(v)).numpy())
    _close(O.act(O.ACT_GELU, v, gelu_tanh=True), F.gelu(_t(v), approximate="tanh").numpy())


@pytest.mark.parametrize("h_is_time,kh,kw,stride,pads", [(1, 5, 3, 2, (2, 1, 1, 2)), (0, 3, 3, 2, (1, 1, 1, 1)),
                                                         (1, 7, 7, 1, (0, 3, 3, 0))])
def test_conv_first(h_is_time, kh, kw, stride, pads):
    rng = np.random.default_rng(1)
    B, M, T, C = 2, 20, 37, 24
    mel = rng.standard_normal((B, M, T)) * 10 - 30
    sc, sh = rng.uniform(0.02, 0.1, M), rng.standard_normal(M)
    w, b = rng.standard_normal((C, kh * kw)), rng.standard_normal(C)
    L = _layer(kh=kh, kw=kw, stride=stride, pad_t=pads[0], pad_b=pads[1], pad_l=pads[2], pad_r=pads[3],
               act=O.ACT_HSWISH, h_is_time=h_is_time)
    x = _t(mel * sc[None, :, None] + sh[None, :, None])[:, None]          # (B, 1, mel, T)
    if h_is_time:
        x = x.transpose(2, 3)
    x = F.pad(x, (pads[2], pads[3], pads[0], pads[1]))
    want = F.hardswish(F.conv2d(x, _t(w).reshape(C, 1, kh, kw), _t(b), stride=stride)).permute(0, 2, 3, 1).numpy()
    y, e = O.conv_first(mel, dict(w=w, b=b, sc=sc, sh=sh), L, want.shape[1], want.shape[2])
    _close(y, want)
    assert np.all(e > 0)


def test_stem_and_its_padding_fault():
    rng = np.random.default_rng(2)
    B, M, T, C = 2, 16, 41, 24
    mel = rng.standard_normal((B, M, T)) * 10 - 30
    sc, sh = rng.uniform(0.02, 0.1, M), rng.standard_normal(M)
    dw, ps, pb = rng.standard_normal(9), rng.standard_normal(C), rng.standard_normal(C)
    L = _layer(kh=3, kw=3, stride=2, pad_t=1, pad_b=1, pad_l=0, pad_r=1, act=O.ACT_RELU6)
    x = _t(mel * sc[None, :, None] + sh[None, :, None])[:, None].transpose(2, 3)
    v = F.conv2d(F.pad(x, (0, 1, 1, 1)), _t(dw).reshape(1, 1, 3, 3), stride=2)
    want = F.relu6(F.conv2d(v, _t(ps).reshape(C, 1, 1, 1), _t(pb))).permute(0, 2, 3, 1).numpy()
    W = dict(sc=sc, sh=sh, dw=dw, pw_scale=ps, pw_shift=pb)
    y, _ = O.stem(mel, W, L, want.shape[1], want.shape[2])
    _close(y, want)
    # the fault: padded time rows carry bn0's shift
    xf = F.pad(x, (0, 1, 1, 1))
    xf[:, :, 0, :M] += _t(sh)
    xf[:, :, -1, :M] += _t(sh)
    vf = F.conv2d(xf, _t(dw).reshape(1, 1, 3, 3), stride=2)
    want_f = F.relu6(F.conv2d(vf, _t(ps).reshape(C, 1, 1, 1), _t(pb))).permute(0, 2, 3, 1).numpy()
    _close(O.stem(mel, W, L, want.shape[1], want.shape[2], bn_on_padding=True)[0], want_f)


@pytest.mark.parametrize("k,stride,pads,a", [(3, 2, (0, 1, 0, 1), O.ACT_RELU), (5, 1, (2, 2, 2, 2), O.ACT_HSWISH),
                                             (7, 2, (3, 3, 3, 3), O.ACT_RELU6)])
def test_depthwise(k, stride, pads, a):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((2, 13, 11, 24))
    w, b = rng.standard_normal((24, k * k)), rng.standard_normal(24)
    L = _layer(kh=k, kw=k, stride=stride, pad_t=pads[0], pad_b=pads[1], pad_l=pads[2], pad_r=pads[3], act=a)
    x = F.pad(_t(X).permute(0, 3, 1, 2), (pads[2], pads[3], pads[0], pads[1]))
    want = TORCH_ACT[a](F.conv2d(x, _t(w).reshape(24, 1, k, k), _t(b), stride=stride, groups=24)).permute(0, 2, 3, 1).numpy()
    _close(O.depthwise(X, dict(w=w, b=b), L, want.shape[1], want.shape[2])[0], want)


@pytest.mark.parametrize("a,residual", [(O.ACT_NONE, True), (O.ACT_RELU6, False), (O.ACT_RELU, False),
                                        (O.ACT_HSWISH, False)])
def test_pointwise(a, residual):
    rng = np.random.default_rng(4)
    X, R = rng.standard_normal((2, 5, 7, 40)), rng.standard_normal((2, 5, 7, 24))
    w, b = rng.standard_normal((24, 40)), rng.standard_normal(24)
    L = _layer(act=a, cin_p=48)
    want = TORCH_ACT[a](F.linear(_t(X), _t(w), _t(b))) + (_t(R) if residual else 0)
    _close(O.pointwise(X, dict(w=w, b=b), L, R if residual else None)[0], want.numpy())
    if a == O.ACT_HSWISH:  # the slope fault: ONNX HardSigmoid's default alpha 0.2 instead of 1/6
        v = F.linear(_t(X), _t(w), _t(b))
        _close(O.pointwise(X, dict(w=w, b=b), L, hsig_slope=0.2)[0], (v * torch.clamp(0.2 * v + 0.5, 0, 1)).numpy())


@pytest.mark.parametrize("inner,gate", [(O.ACT_RELU, O.ACT_HSIGMOID), (O.ACT_RELU, O.ACT_SIGMOID),
                                        (O.ACT_HSWISH, O.ACT_SIGMOID)])
def test_squeeze_excite(inner, gate):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((3, 6, 9, 40))
    W = dict(w1=rng.standard_normal((8, 40)), b1=rng.standard_normal(8), w2=rng.standard_normal((40, 8)),
             b2=rng.standard_normal(40))
    x = _t(X).permute(0, 3, 1, 2)
    s = TORCH_ACT[inner](F.conv2d(x.mean((2, 3), keepdim=True), _t(W["w1"])[:, :, None, None], _t(W["b1"])))
    g = TORCH_ACT[gate](F.conv2d(s, _t(W["w2"])[:, :, None, None], _t(W["b2"])))
    want = (x * g).permute(0, 2, 3, 1).numpy()
    _close(O.squeeze_excite(X, W, _layer(act=inner, gate_act=gate))[0], want)


@pytest.mark.parametrize("stride", [1, 2, 3])
def test_pool_over_the_stride_lattice(stride):
    rng = np.random.default_rng(6)
    X = rng.standard_normal((2, 9, 7, 48))
    # the mean over the positions a 1x1 stride-s convolution visits
    want = F.avg_pool2d(_t(X).permute(0, 3, 1, 2)[:, :40], 1, stride).mean((2, 3)).numpy()
    _close(O.pool(X, 40, stride)[0], want)


@pytest.mark.parametrize("a", [O.ACT_NONE, O.ACT_GELU, O.ACT_HSWISH])
def test_linear_and_its_faults(a):
    rng = np.random.default_rng(7)
    x, w, b = rng.standard_normal((3, 40)), rng.standard_normal((24, 40)), rng.standard_normal(24)
    _close(O.linear(x, w, b, a)[0], F.linear(TORCH_ACT[a](_t(x)), _t(w), _t(b)).numpy())
    _close(O.linear(x, w, None, a)[0], F.linear(TORCH_ACT[a](_t(x)), _t(w)).numpy())
    if a == O.ACT_GELU:
        want = F.linear(F.gelu(_t(x), approximate="tanh"), _t(w), _t(b)).numpy()
        _close(O.linear(x, w, b, a, gelu_tanh=True)[0], want)
    # without the lo terms: a plain bf16 GEMM
    xa = TORCH_ACT[a](_t(x)).numpy()
    _close(O.linear(x, w, b, a, drop_lo=True)[0], O.bf16r(xa) @ O.bf16r(w).T + b)


def test_row_ops():
    rng = np.random.default_rng(8)
    a, b = rng.standard_normal((3, 48)), rng.standard_normal((3, 48))
    g, bt, s, t = rng.standard_normal(48), rng.standard_normal(48), rng.standard_normal(48), rng.standard_normal(48)
    _close(O.add(a, b)[0], (_t(a) + _t(b)).numpy())
    _close(O.affine(a, s, t)[0], (_t(a) * _t(s) + _t(t)).numpy())
    _close(O.affine(a, None, t)[0], (_t(a) + _t(t)).numpy())
    _close(O.layernorm(a, g, bt, 1e-5)[0], F.layer_norm(_t(a), (48,), _t(g), _t(bt), 1e-5).numpy())
    _close(O.l2norm(a, 1e-12)[0], F.normalize(_t(a), dim=1, eps=1e-12).numpy())
    want = F.normalize(F.layer_norm(_t(a) + _t(b), (48,), _t(g), _t(bt), 1e-5), dim=1, eps=1e-12).numpy()
    _close(O.add_ln_l2(a, b, g, bt, 1e-5, 1e-12)[0], want)
    # eps outside the square root
    d = _t(a) - _t(a).mean(1, keepdim=True)
    want = (d / (d.pow(2).mean(1, keepdim=True).sqrt() + 1e-5) * _t(g) + _t(bt)).numpy()
    _close(O.layernorm(a, g, bt, 1e-5, eps_outside=True)[0], want)


def test_bf16_rounding_is_nearest_even():
    x = np.array([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -8 + 2.0 ** -20])
    np.testing.assert_array_equal(O.bf16r(x), [1.0, 1.0 + 4 * 2.0 ** -8, -1.0, 1.0 + 2 * 2.0 ** -8])
    assert math.isclose(O.gamma(1), 2.0 ** -23 + 2.0 ** -22)
