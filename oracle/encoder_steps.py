"""Oracle: the encoder's steps outside the inverted-residual block, in float64 with per-element error bounds.
TEST INFRASTRUCTURE ONLY (tests/test_gpu_encoder_steps_exact.py, tests/test_encoder_steps_oracle_host.py).

Each step function takes the device's own input to the step (the log-mel, or the previous step's bf16 output) and the
weights the kernel multiplies, and returns ``(y, e)``: the exact float64 result of the operation and a bound ``e`` on
the arithmetic error of the kernel's fp32 evaluation (before the output's own rounding).  ``output_bound`` adds the
rounding of the stored value.  The bounds are derived from the kernels' declared rounding points:

* an fp32 accumulation of n terms (serial FMA chains, warp / block trees, tensor-core MMAs): gamma(n) * sum |terms|,
  gamma(n) = n * 2^-23 + 2^-22 (one truncation per term, as tests/test_gpu_block_exact.py uses);
* one fp32 rounding: u = 2^-24 relative;
* an activation: its Lipschitz constant times the error of its argument, plus its fp32 evaluation error (``act_eval_error``;
  expf, erff and tanhf are within 2 ulp by the CUDA Math API's tables, rsqrtf within 2 ulp, sqrtf and division are
  correctly rounded without fast-math);
* the split-bf16 head linears: x = hi + lo + r with |x - hi| <= 2^-8 |x| and |r| <= 2^-16 |x|, likewise w; the GEMM
  forms hi.hi + hi.lo + lo.hi, so the dropped lo.lo, hi.r_w and r_x.hi terms are below 3.02 * 2^-16 |x| |w|;
* the reductions (channel mean, strided mean, LayerNorm mean and variance, the L2 norm) each with their own gamma;
* every stored bf16 value: half a bf16 ulp, <= 2^-8 |value|; every stored f32 value: u |value|.

Weights come from the ONNX file (``oracle.onnx_ref.load``), matched to the device's plan layer by layer
(``extract_weights``): 1x1 convolutions rounded to bf16 (round to nearest even) as build_model uploads them, any
BatchNormalization left in the trunk folded as the loader folds it (a double product stored as float), the head's
linears in fp32 (their split-bf16 representation error is in the bound).
"""
from __future__ import annotations

import math

import numpy as np
from scipy.special import erf

# csrc/model_spec.cuh
K_STEM, K_POINTWISE, K_DEPTHWISE, K_CONV_FIRST, K_SQUEEZE_EXCITE = 0, 1, 2, 4, 5
ACT_NONE, ACT_RELU6, ACT_RELU, ACT_HSWISH, ACT_GELU, ACT_SIGMOID, ACT_HSIGMOID, ACT_TANH = range(8)
V_POOL, V_LINEAR, V_UNARY, V_ADD, V_AFFINE, V_LAYERNORM, V_L2NORM, V_ADD_LN_L2 = range(8)
# encoder.cu StepKind
S_STEM, S_CONV_FIRST, S_FUSED, S_POINTWISE, S_DW3X3, S_DW_GENERIC, S_SQUEEZE_EXCITE = range(7)
STEP_NAMES = ["stem", "conv_first", "fused", "pointwise", "dw3x3", "dw_generic", "squeeze_excite"]
HEAD_NAMES = ["pool", "linear", "unary", "add", "affine", "layernorm", "l2norm", "add_layernorm_l2"]

U = 2.0 ** -24
TINY = 2.0 ** -126


def gamma(n):
    return n * 2.0 ** -23 + 2.0 ** -22


# ---------------------------------------------------------------- bf16
def bf16_bits(x):
    """round-to-nearest-even float32 -> bf16 on the uint32 view (x is rounded to float32 first)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_value(bits):
    return (np.asarray(bits).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def bf16r(x):
    return bf16_value(bf16_bits(x))


# ---------------------------------------------------------------- activations
def act(kind, v, hsig_slope=1.0 / 6.0, gelu_tanh=False):
    v = np.asarray(v, dtype=np.float64)
    if kind == ACT_RELU6:
        return np.clip(v, 0.0, 6.0)
    if kind == ACT_RELU:
        return np.maximum(v, 0.0)
    if kind == ACT_HSWISH:
        return v * np.clip(v * hsig_slope + 0.5, 0.0, 1.0)
    if kind == ACT_GELU:
        if gelu_tanh:
            return 0.5 * v * (1.0 + np.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))
        return 0.5 * v * (1.0 + erf(v / math.sqrt(2.0)))
    if kind == ACT_SIGMOID:
        return 1.0 / (1.0 + np.exp(-v))
    if kind == ACT_HSIGMOID:
        return np.clip(v * hsig_slope + 0.5, 0.0, 1.0)
    if kind == ACT_TANH:
        return np.tanh(v)
    return v


# Lipschitz constants (max |act'|; GELU's is 1.1289)
ACT_LIP = {ACT_NONE: 1.0, ACT_RELU6: 1.0, ACT_RELU: 1.0, ACT_HSWISH: 1.5, ACT_GELU: 1.13, ACT_SIGMOID: 0.25,
           ACT_HSIGMOID: 1.0 / 6.0, ACT_TANH: 1.0}


def act_eval_error(kind, v):
    """bound of |fp32 act(v) - act(v)| for an exact fp32 argument v (encoder_generic.cuh apply_act, gemm.cu epi_act)"""
    a = np.abs(np.asarray(v, dtype=np.float64))
    y = np.abs(act(kind, v))
    if kind == ACT_HSWISH:   # v * (1/6) (+ the constant's rounding), + 0.5, * v: four roundings of terms <= |v|(|v|/6 + 1/2)
        return 4 * U * a * (a / 6.0 + 0.5)
    if kind == ACT_HSIGMOID:
        return 3 * U * (a / 6.0 + 0.5)
    if kind == ACT_SIGMOID:  # expf 2 ulp, 1 + e, 1 / d: relative 2^-22 + 2u
        return (2.0 ** -22 + 3 * U) * y + TINY
    if kind == ACT_TANH:     # tanhf 2 ulp
        return 2.0 ** -22 * y + TINY
    if kind == ACT_GELU:     # v * c (c rounded), erff 2 ulp, 1 + erf, 0.5 v (exact), the product
        return 0.5 * a * (1.13 * 2 * U * a + 2.0 ** -22 + 2 * U) + U * y + TINY
    return np.zeros_like(a)


def output_bound(y, e, bf16=True):
    """bound of |stored - y| given the arithmetic bound e: + half a bf16 ulp (or the f32 rounding) of the value"""
    y = np.abs(y)
    return e + (2.0 ** -8 if bf16 else U) * (y + e) + TINY


# ---------------------------------------------------------------- trunk steps
def _mel_affine(mel, sc, sh):
    """x = mel * sc[mel bin] + sh[mel bin] and |mel sc| + |sh| (the magnitude its fp32 FMA rounds), [B, n_mels, T]"""
    if sc is None:
        return mel, np.abs(mel)
    s, t = np.asarray(sc, np.float64)[None, :, None], np.asarray(sh, np.float64)[None, :, None]
    return mel * s + t, np.abs(mel * s) + np.abs(t)


def _image(x, h_is_time, pads):
    """[B, n_mels, T] -> zero-padded image [B, H + pt + pb, W + pl + pr] with H = time (h_is_time) or mel"""
    img = np.transpose(x, (0, 2, 1)) if h_is_time else x
    pt, pb, pl, pr = pads
    return np.pad(img, ((0, 0), (pt, pb), (pl, pr)))


def _taps(img, kh, kw, s, Ho, Wo):
    for dy in range(kh):
        for dx in range(kw):
            yield dy * kw + dx, img[:, dy:dy + s * (Ho - 1) + 1:s, dx:dx + s * (Wo - 1) + 1:s]


def stem(mel, W, L, Ho, Wo, bn_on_padding=False):
    """stem_kernel: bn0 per mel bin, 3x3 stride-2 on the single channel (pad_t / pad_l, zeros outside the map), then
    relu6(v * pw_scale + pw_shift).  [B, Ho, Wo, cout]"""
    x, xa = _mel_affine(mel, W["sc"], W["sh"])
    pads = (L["pad_t"], L["pad_b"], L["pad_l"], L["pad_r"])
    img, imga = _image(x, True, pads), _image(xa, True, pads)
    if bn_on_padding:  # the fault: padded time rows carry bn0's shift of their mel bin
        pt, pb, pl, pr = pads
        sh = np.pad(np.asarray(W["sh"], np.float64), (pl, pr))[None, None, :]
        rows = np.zeros(img.shape[1], bool)
        rows[:pt] = True
        rows[img.shape[1] - pb:] = True
        img = img + rows[None, :, None] * sh
    v = np.zeros((mel.shape[0], Ho, Wo))
    va = np.zeros_like(v)
    for t, (win, wina) in zip(range(9), zip(_taps(img, 3, 3, 2, Ho, Wo), _taps(imga, 3, 3, 2, Ho, Wo))):
        v += W["dw"][t] * win[1]
        va += abs(W["dw"][t]) * wina[1]
    ev = gamma(11) * va                                   # the bn0 FMA per sample + 9 FMAs
    ps, pb_ = W["pw_scale"], W["pw_shift"]
    pre = v[..., None] * ps + pb_
    e_pre = np.abs(ps) * ev[..., None] + 2 * U * (np.abs(v[..., None] * ps) + np.abs(pb_))
    return act(ACT_RELU6, pre), e_pre


def conv_first(mel, W, L, Ho, Wo):
    """conv_first_kernel: optional per-mel affine on in-range samples, kh x kw stride-s convolution of the one-channel
    image (time, mel) or (mel, time), bias, activation.  [B, Ho, Wo, cout]"""
    x, xa = _mel_affine(mel, W.get("sc"), W.get("sh"))
    pads = (L["pad_t"], L["pad_b"], L["pad_l"], L["pad_r"])
    img, imga = _image(x, L["h_is_time"], pads), _image(xa, L["h_is_time"], pads)
    kh, kw, s = L["kh"], L["kw"], L["stride"]
    w, b = W["w"], W["b"]                                 # [cout, kh*kw], [cout]
    o = np.zeros((mel.shape[0], Ho, Wo, w.shape[0])) + b
    oa = np.zeros_like(o) + np.abs(b)
    for (t, win), (_, wina) in zip(_taps(img, kh, kw, s, Ho, Wo), _taps(imga, kh, kw, s, Ho, Wo)):
        o += win[..., None] * w[:, t]
        oa += wina[..., None] * np.abs(w[:, t])
    e = gamma(kh * kw + 2) * oa
    return act(L["act"], o), ACT_LIP[L["act"]] * e + act_eval_error(L["act"], o)


def depthwise(X, W, L, Ho, Wo):
    """depthwise_generic_kernel: K x K per channel, stride s, zero pads (pad_t, pad_b, pad_l, pad_r), bias, act"""
    k, s = L["kh"], L["stride"]
    Xp = np.pad(X, ((0, 0), (L["pad_t"], L["pad_b"]), (L["pad_l"], L["pad_r"]), (0, 0)))
    w, b = W["w"], W["b"]                                 # [c, k*k], [c]
    o = np.zeros((X.shape[0], Ho, Wo, X.shape[3])) + b
    oa = np.zeros_like(o) + np.abs(b)
    for dy in range(k):
        for dx in range(k):
            win = Xp[:, dy:dy + s * (Ho - 1) + 1:s, dx:dx + s * (Wo - 1) + 1:s]
            o += win * w[:, dy * k + dx]
            oa += np.abs(win) * np.abs(w[:, dy * k + dx])
    e = gamma(k * k + 1) * oa
    return act(L["act"], o), ACT_LIP[L["act"]] * e + act_eval_error(L["act"], o)


def pointwise(X, W, L, residual=None, hsig_slope=1.0 / 6.0):
    """the GEMM with its epilogue: act(X . Wb^T + bias) (+ residual), Wb the bf16 weights"""
    B, H, Wd, C = X.shape
    x = X.reshape(-1, C)
    pre = x @ W["w"].T + W["b"]
    e = gamma(L["cin_p"] + 2) * (np.abs(x) @ np.abs(W["w"]).T + np.abs(W["b"]))
    y = act(L["act"], pre, hsig_slope=hsig_slope)
    e = ACT_LIP[L["act"]] * e + act_eval_error(L["act"], pre)
    if residual is not None:
        r = residual.reshape(y.shape)
        e = e + U * (np.abs(y) + np.abs(r) + e)
        y = y + r
    return y.reshape(B, H, Wd, -1), e.reshape(B, H, Wd, -1)


def squeeze_excite(X, W, L):
    """channel_mean_kernel, se_gate_kernel, se_scale_kernel: x * gate(W2 . act(W1 . mean(x) + b1) + b2)"""
    B, H, Wd, C = X.shape
    HW = H * Wd
    m = X.reshape(B, HW, C).mean(1)
    em = gamma(HW + 1) * np.abs(X).reshape(B, HW, C).mean(1)
    hp = m @ W["w1"].T + W["b1"]
    e_hp = em @ np.abs(W["w1"]).T + gamma(C + 1) * (np.abs(m) @ np.abs(W["w1"]).T + np.abs(W["b1"]))
    h = act(L["act"], hp)
    e_h = ACT_LIP[L["act"]] * e_hp + act_eval_error(L["act"], hp)
    gp = h @ W["w2"].T + W["b2"]
    e_gp = e_h @ np.abs(W["w2"]).T + gamma(W["w2"].shape[1] + 1) * (np.abs(h) @ np.abs(W["w2"]).T + np.abs(W["b2"]))
    g = act(L["gate_act"], gp)
    e_g = ACT_LIP[L["gate_act"]] * e_gp + act_eval_error(L["gate_act"], gp)
    y = X * g[:, None, None, :]
    e = np.abs(X) * e_g[:, None, None, :] + U * np.abs(y)
    return y, e


# ---------------------------------------------------------------- head row program (f32 rows)
def pool(X, C, stride):
    """strided_mean_kernel: mean over the (h % s == 0, w % s == 0) positions of the first C channels"""
    lat = X[:, ::stride, ::stride, :C]
    n = lat.shape[1] * lat.shape[2]
    return lat.mean((1, 2)), gamma(n + 2) * np.abs(lat).mean((1, 2))


def linear(a, W, b, in_act, gelu_tanh=False, drop_lo=False):
    """split3_kernel + the split-bf16 GEMM with f32 output: in_act(a) . W^T + b"""
    x = act(in_act, a, gelu_tanh=gelu_tanh)
    ex = act_eval_error(in_act, a)
    bias = 0.0 if b is None else b
    if drop_lo:  # the fault: a plain bf16 GEMM
        return bf16r(x) @ bf16r(W).T + bias, np.zeros((a.shape[0], W.shape[0]))
    K = W.shape[1]
    Kp = (K + 7) // 8 * 8
    S = np.abs(x) @ np.abs(W).T
    e = 1.01 * ex @ np.abs(W).T + 3.02 * 2.0 ** -16 * S + gamma(3 * Kp + 1) * (1.02 * S + np.abs(bias))
    return x @ W.T + bias, e


def unary(a, kind, gelu_tanh=False):
    return act(kind, a, gelu_tanh=gelu_tanh), act_eval_error(kind, a)


def add(a, b):
    return a + b, np.zeros_like(a)


def affine(a, scale, shift):
    y = a * (1.0 if scale is None else scale) + (0.0 if shift is None else shift)
    e = U * np.abs(a * scale) if (scale is not None and shift is not None) else np.zeros_like(a)
    return y, e


def _layernorm(x, g, b, eps, dx=None, eps_outside=False):
    """(x - mean) / sqrt(var + eps) * g + b per row, and the bound of the kernel's error; dx: a bound of the error
    already in x (the fused kernel's a + b), carried through LayerNorm's first-order sensitivity"""
    E = x.shape[1]
    mu = x.mean(1, keepdims=True)
    d = x - mu
    var = (d * d).mean(1, keepdims=True)
    r = 1.0 / (np.sqrt(var) + eps) if eps_outside else 1.0 / np.sqrt(var + eps)
    y = d * r * g + b
    dmu = gamma(E + 1) * np.abs(x).mean(1, keepdims=True)
    ed = dmu + U * (np.abs(d) + dmu)
    evar = (ed * (2 * np.abs(d) + ed)).mean(1, keepdims=True) + gamma(E + 1) * ((np.abs(d) + ed) ** 2).mean(1, keepdims=True)
    rel_r = 1.01 * 0.5 * (evar + U * (var + eps)) / (var + eps) + 2.0 ** -22
    e = np.abs(g) * (ed * r * (1 + rel_r) + np.abs(d) * r * rel_r) + gamma(3) * (np.abs(d * r * g) + np.abs(b))
    if dx is not None:
        sens = dx + dx.mean(1, keepdims=True) + np.abs(d) * r * r * (np.abs(d) * dx).mean(1, keepdims=True)
        e = e + 1.01 * np.abs(g) * r * sens
    return y, e


def layernorm(a, g, b, eps, eps_outside=False):
    return _layernorm(a, g, b, eps, eps_outside=eps_outside)


def _l2(z, ez, eps2):
    E = z.shape[1]
    nz = np.sqrt((z * z).sum(1, keepdims=True))
    nrm = np.maximum(nz, eps2)
    y = z / nrm
    en = np.sqrt((ez * ez).sum(1, keepdims=True))
    rel = np.where(nz > eps2, 0.5 * gamma(E + 1) + U, 0.0)
    e = 1.01 * (ez + np.abs(y) * en) / nrm + np.abs(y) * rel
    return y, e


def l2norm(a, eps2):
    return _l2(a, np.zeros_like(a), eps2)


def add_ln_l2(a, b, g, bt, eps, eps2, eps_outside=False):
    """head_finalize_kernel: L2(LayerNorm(a + b)); a + b rounds once in fp32"""
    s = a + b
    z, ez = _layernorm(s, g, bt, eps, dx=U * np.abs(s), eps_outside=eps_outside)
    return _l2(z, ez, eps2)


# ---------------------------------------------------------------- weights from the ONNX file
def _fold_bn(w, b, bn, consts):
    """onnx_model.cu: a BatchNormalization after a convolution, folded into it: w * s and b * s + (beta - mu * s)
    with s = gamma / sqrt(var + eps) in double, each stored as float"""
    ga, be, mu, var = (np.asarray(consts[i], np.float64) for i in bn.inputs[1:5])
    eps = float(np.float32(bn.attrs.get("epsilon", 1e-5)))
    s = ga / np.sqrt(var + eps)
    w = (w.astype(np.float64) * s.reshape((-1,) + (1,) * (w.ndim - 1))).astype(np.float32)
    b = (b.astype(np.float64) * s + (be - mu * s)).astype(np.float32)
    return w, b


def extract_weights(g, layers, head, bf16_pointwise=True):
    """The weights the device multiplies for each plan layer and head op, read from the ONNX graph `g`
    (oracle.onnx_ref.Graph) in node order.  `layers` / `head`: the plan's records as dicts.  bf16_pointwise=False
    keeps the 1x1 convolutions in fp32 (to compare a chain of the step functions with the PyTorch module)."""
    consts = dict(g.initializers)
    for n in g.nodes:
        if n.op == "Constant" and "value" in n.attrs:
            consts[n.outputs[0]] = np.asarray(n.attrs["value"])
    consumers, producer = {}, {}
    for i, n in enumerate(g.nodes):
        for x in n.inputs:
            consumers.setdefault(x, []).append(i)
        for x in n.outputs:
            producer[x] = i
    f32 = lambda a: np.asarray(a, np.float32)

    # the per-mel normalisation of the input view
    sc = sh = None
    convs = []  # (node index, w, b)
    for i, n in enumerate(g.nodes):
        if n.op == "BatchNormalization" and not convs:
            ga, be, mu, var = (np.asarray(consts[x], np.float64) for x in n.inputs[1:5])
            eps = float(np.float32(n.attrs.get("epsilon", 1e-5)))
            s = ga / np.sqrt(var + eps)
            sc, sh = f32(s), f32(be - mu * s)
        elif n.op == "Conv":
            w = f32(consts[n.inputs[1]])
            b = f32(consts[n.inputs[2]]) if len(n.inputs) > 2 and n.inputs[2] else np.zeros(w.shape[0], np.float32)
            convs.append([i, w, b, n])
        elif n.op == "BatchNormalization":  # left in the trunk: folded into the producing convolution
            c = convs[-1]
            c[1], c[2] = _fold_bn(c[1], c[2], n, consts)
    out_layers = []
    ci = 0
    for L in layers:
        t = L["type"]
        if t == K_STEM:
            (_, k0, b0, _), (_, pw, pb, _) = convs[ci], convs[ci + 1]
            ci += 2
            pw = pw.reshape(-1)
            out_layers.append(dict(sc=sc if sc is not None else np.ones(128, np.float32),
                                   sh=sh if sh is not None else np.zeros(128, np.float32),
                                   dw=k0.reshape(-1).astype(np.float64), pw_scale=pw.astype(np.float64),
                                   pw_shift=(pw * np.float32(b0[0]) + pb).astype(np.float32).astype(np.float64)))
        elif t == K_CONV_FIRST:
            _, w, b, _ = convs[ci]
            ci += 1
            d = dict(w=w.reshape(w.shape[0], -1).astype(np.float64), b=b.astype(np.float64))
            if sc is not None:
                d.update(sc=sc, sh=sh)
            out_layers.append(d)
        elif t == K_POINTWISE:
            _, w, b, _ = convs[ci]
            ci += 1
            w = w.reshape(w.shape[0], -1)
            out_layers.append(dict(w=bf16r(w) if bf16_pointwise else w.astype(np.float64), b=b.astype(np.float64)))
        elif t == K_DEPTHWISE:
            _, w, b, _ = convs[ci]
            ci += 1
            out_layers.append(dict(w=w.reshape(w.shape[0], -1).astype(np.float64), b=b.astype(np.float64)))
        elif t == K_SQUEEZE_EXCITE:
            (_, w1, b1, _), (_, w2, b2, _) = convs[ci], convs[ci + 1]
            ci += 2
            out_layers.append(dict(w1=w1.reshape(w1.shape[0], -1).astype(np.float64), b1=b1.astype(np.float64),
                                   w2=w2.reshape(w2.shape[0], -1).astype(np.float64), b2=b2.astype(np.float64)))
        else:
            raise ValueError(f"layer type {t}")
    # ---- the head, in node order after the trunk
    first = convs[ci][0] if ci < len(convs) else (convs[ci - 1][0] + 1)
    events, skip = [], set()
    for i in range(first, len(g.nodes)):
        n = g.nodes[i]
        if i in skip:
            continue
        if n.op == "Conv":  # 1x1 stride-s convolution in front of the pooling: the first linear
            w, b = f32(consts[n.inputs[1]]), f32(consts[n.inputs[2]]) if len(n.inputs) > 2 else None
            events.append(("linear", w.reshape(w.shape[0], -1), b, n.outputs[0]))
        elif n.op in ("MatMul", "Gemm") and n.inputs[1] in consts:
            w = f32(consts[n.inputs[1]])
            w = w if (n.op == "Gemm" and n.attrs.get("transB", 0)) else w.T
            b = f32(consts[n.inputs[2]]) if n.op == "Gemm" and len(n.inputs) > 2 and n.inputs[2] else None
            events.append(("linear", w, b, n.outputs[0]))
        elif n.op == "LayerNormalization":
            events.append(("ln", f32(consts[n.inputs[1]]), f32(consts[n.inputs[2]]), n.outputs[0]))
        elif n.op == "Erf":  # exact GELU: Div(sqrt 2) -> Erf -> Add 1 -> Mul x -> Mul 0.5
            j = consumers[n.outputs[0]][0]
            m1 = consumers[g.nodes[j].outputs[0]][0]
            skip.update({j, m1, consumers[g.nodes[m1].outputs[0]][0]})
        elif n.op == "Sqrt":  # decomposed LayerNorm: ... Sqrt -> Div -> Mul g -> Add b
            dv = consumers[n.outputs[0]][0]
            mg = consumers[g.nodes[dv].outputs[0]][0]
            ab = consumers[g.nodes[mg].outputs[0]][0]
            cg = [x for x in g.nodes[mg].inputs if x in consts][0]
            cb = [x for x in g.nodes[ab].inputs if x in consts][0]
            skip.update({dv, mg, ab})
            events.append(("ln", f32(consts[cg]), f32(consts[cb]), g.nodes[ab].outputs[0]))
        elif n.op in ("Add", "Mul", "Sub", "Div") and any(x in consts for x in n.inputs):
            c = [x for x in n.inputs if x in consts][0]
            other = [x for x in n.inputs if x != c][0]
            v = f32(consts[c]).reshape(-1)
            if n.op == "Div" and abs(float(v[0]) - math.sqrt(2.0)) < 1e-4 and v.size == 1:
                continue  # GELU's division by sqrt(2)
            if n.op == "Add" and other in producer and g.nodes[producer[other]].op == "ReduceMean":
                continue  # the decomposed LayerNorm's var + eps
            events.append(("const", n.op, v, other, n.outputs[0]))
    out_head = []
    ei = 0
    for h in head:
        k = h["kind"]
        if k == V_LINEAR:
            while events[ei][0] != "linear":
                ei += 1
            _, w, b, out = events[ei]
            ei += 1
            if b is None and ei < len(events) and events[ei][0] == "const" and events[ei][1] == "Add" and events[ei][3] == out:
                b = events[ei][2]  # a bias add after a bias-free linear (merged by the loader)
                ei += 1
            out_head.append(dict(w=w.astype(np.float64), b=None if b is None else b.astype(np.float64)))
        elif k in (V_LAYERNORM, V_ADD_LN_L2):
            while events[ei][0] != "ln":
                ei += 1
            out_head.append(dict(g=events[ei][1].astype(np.float64), b=events[ei][2].astype(np.float64)))
            ei += 1
        elif k == V_AFFINE:
            while events[ei][0] != "const":
                ei += 1
            _, op, v, _, _ = events[ei]
            ei += 1
            v = np.broadcast_to(v, (h["N"],)).astype(np.float32)
            scale = shift = None
            if op == "Mul":
                scale = v
            elif op == "Div":
                scale = (np.float32(1.0) / v).astype(np.float32)
            elif op == "Add":
                shift = v
            else:
                shift = -v
            out_head.append(dict(scale=None if scale is None else scale.astype(np.float64),
                                 shift=None if shift is None else shift.astype(np.float64)))
        else:
            out_head.append({})
    return out_layers, out_head
