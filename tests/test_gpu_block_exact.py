"""One inverted-residual block, fused (fused_block.cu) and layer by layer (GEMM, depthwise dispatch, GEMM), against a
float64 oracle with the kernels' declared rounding points:

    E = bf16(relu6(X . W1^T + b1)), zero outside the image
    D = bf16(relu6(dw3x3(E, pad 1, stride) + bd))
    Y = bf16(D . W2^T + b2 (+ X))

Every sum is float64; bf16 rounding is round-to-nearest-even on the float32 bits.

(a) Operands on a dyadic grid, where every product and partial sum is exact in fp32, in the packed fp16 of the
    layer-by-layer depthwise and in the tensor cores' accumulation: Y (and E, D layer by layer) must equal the oracle
    bit for bit.
(b) Gaussian activations, folded weights like weights.random_state_dict and depthwise weights log-uniform in magnitude
    up to 30: every element within a bound derived per element below.  Two cases put a depthwise weight above the fp16
    maximum and a channel whose partial sums pass it before later taps cancel them; there the layer path must keep the
    fused path's (fp32) bound.

Each case runs am_debug_block (libaudiomuse_b200_debug.so) in a subprocess under a timeout and reports the ring depth
the fused plan chose and the depthwise kernel the layer path ran; test_every_branch_is_reached checks that the cases
reach all of them and the shapes listed there."""
import math
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DW_STRIP, DW_ROW, DW_GENERIC = 0, 1, 2  # include/audiomuse_b200_debug.h, am_debug_block path 1


def _pad16(c):
    return (c + 15) // 16 * 16


def _shipped_blocks(alpha=3.0):
    """(cin_p, cmid_p, cout_p, stride, has_expand, residual) of every block of a student, and the stem output shape
    at T = 1001 frames"""
    from audiomuse_ai_b200 import weights
    cfg = weights.StudentConfig(alpha=alpha)
    _, blocks = weights.block_plan(cfg)
    pl, pr, pt, pb = weights.correct_pad((1,) + tuple(cfg.input_hw))
    H, W = (1001 + pt + pb - 3) // 2 + 1, (cfg.n_mels + pl + pr - 3) // 2 + 1
    out = []
    for b in blocks:
        out.append(((_pad16(b.cin), _pad16(b.cmid), _pad16(b.cout), b.stride, int(b.block_id != 0), int(b.residual)),
                    (H, W)))
        H, W = (H - 1) // b.stride + 1, (W - 1) // b.stride + 1
    return out


SHIPPED = _shipped_blocks()
SHIPPED_DEPTHS = [4, 2, 4, 2, 3]  # fused plans of the shipped student's blocks 0-4 at T = 1001
ALPHA6_B1 = _shipped_blocks(6.0)[1][0]  # plans a one-stage ring


# name: (grid, B, H, W, (cin_p, cmid_p, cout_p, stride, has_expand, residual))
CASES = {
    # (a) dyadic grid: the shipped blocks 0-4 (block 0 at its full T = 1001 size), then the edges
    "exact_b0": ("exact", 1, 501, 64, SHIPPED[0][0]),
    "exact_b1": ("exact", 3, 37, 29, SHIPPED[1][0]),
    "exact_b2": ("exact", 1, 31, 21, SHIPPED[2][0]),
    "exact_b3": ("exact", 1, 63, 33, SHIPPED[3][0]),
    "exact_b4": ("exact", 3, 20, 16, SHIPPED[4][0]),
    "exact_alpha6_b1": ("exact", 1, 45, 19, ALPHA6_B1),
    "exact_1x1_k16": ("exact", 1, 1, 1, (16, 48, 16, 1, 1, 1)),
    "exact_1x1_s2_c192": ("exact", 3, 1, 1, (48, 96, 192, 2, 1, 0)),
    "exact_narrow_k48": ("exact", 3, 7, 5, (48, 112, 64, 2, 1, 0)),
    "exact_k208_c256": ("exact", 1, 9, 17, (208, 128, 256, 1, 1, 0)),
    "exact_noexp_s2": ("exact", 1, 15, 13, (64, 64, 80, 2, 0, 0)),
    "exact_noexp_res": ("exact", 3, 10, 9, (64, 64, 64, 1, 0, 1)),
    "exact_many_tiles_s2": ("exact", 3, 197, 101, (48, 176, 64, 2, 1, 0)),
    # narrow maps with enough work for the row depthwise (cout_p > 256: layer by layer only)
    "exact_row_s1": ("exact", 27, 32, 4, (576, 2592, 576, 1, 1, 1)),
    "exact_row_s2": ("exact", 27, 64, 2, (576, 2592, 576, 2, 1, 0)),
    # (b) realistic operands: blocks 0-4 at smaller maps, blocks 5-8 at their T = 1001 size (layer by layer only)
    "real_b0": ("real", 3, 40, 24, SHIPPED[0][0]),
    "real_b1": ("real", 1, 61, 64, SHIPPED[1][0]),
    "real_b2": ("real", 3, 25, 32, SHIPPED[2][0]),
    "real_b3": ("real", 1, 51, 31, SHIPPED[3][0]),
    "real_b4": ("real", 1, 126, 16, SHIPPED[4][0]),
    "real_alpha6_b1": ("real", 3, 13, 12, ALPHA6_B1),
    "real_b5": ("real", 1, *SHIPPED[5][1], SHIPPED[5][0]),
    "real_b6": ("real", 1, *SHIPPED[6][1], SHIPPED[6][0]),
    "real_b7": ("real", 1, *SHIPPED[7][1], SHIPPED[7][0]),
    "real_b8": ("real", 1, *SHIPPED[8][1], SHIPPED[8][0]),
    # (b) the fp16 range of the layer path's depthwise
    "fp16_weight_above_max": ("big_weight", 1, 17, 12, SHIPPED[2][0]),
    "fp16_partial_sum_overflow": ("overflow", 1, 19, 22, SHIPPED[3][0]),
}


# ---------------------------------------------------------------- bf16 and the oracle
def bf16_bits(x):
    """round-to-nearest-even float32 -> bf16 on the uint32 view (x is rounded to float32 first)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_value(bits):
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def bf16r(x):
    return bf16_value(bf16_bits(x))


def relu6(x):
    return np.clip(x, 0.0, 6.0)


def dw_sum(Ep, w, stride, Ho, Wo, bias=None, track_max=False):
    """bias + sum over the 9 taps (in the kernels' order dy, dx) of w[t] * Ep shifted, Ep padded by 1 on H and W;
    with track_max also the largest |partial sum| along that order"""
    acc = np.zeros(Ep.shape[:1] + (Ho, Wo, Ep.shape[3])) + (0.0 if bias is None else bias)
    mx = np.abs(acc) if track_max else None
    for dy in range(3):
        for dx in range(3):
            acc = acc + w[dy * 3 + dx] * Ep[:, dy:dy + stride * (Ho - 1) + 1:stride, dx:dx + stride * (Wo - 1) + 1:stride]
            if track_max:
                mx = np.maximum(mx, np.abs(acc))
    return (acc, mx) if track_max else acc


def pad_hw(a):
    return np.pad(a, ((0, 0), (1, 1), (1, 1), (0, 0)))


def gamma(n):
    """relative bound of an n-term fp32 accumulation on the tensor cores or the CUDA cores: one truncation per term"""
    return n * 2.0 ** -23 + 2.0 ** -22


def oracle(op, stride, has_expand, residual):
    X, W1, b1, wd, bd, W2, b2 = (op[k] for k in ("X", "W1", "b1", "wd", "bd", "W2", "b2"))
    X = bf16_value(X)
    B, H, W, cin = X.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    r = {}
    if has_expand:
        W1 = bf16_value(W1)
        e = X.reshape(-1, cin) @ W1.T + b1
        r["e"] = e.reshape(B, H, W, -1)
        r["eabs"] = (np.abs(X).reshape(-1, cin) @ np.abs(W1).T + np.abs(b1)).reshape(B, H, W, -1)
        r["E"] = bf16r(relu6(r["e"]))
    else:
        r["E"] = X
    d, dmax = dw_sum(pad_hw(r["E"]), wd, stride, Ho, Wo, bias=bd, track_max=True)
    r["d"], r["dmax"] = d, dmax
    r["dabs"] = dw_sum(pad_hw(r["E"]), np.abs(wd), stride, Ho, Wo, bias=np.abs(bd))
    r["D"] = bf16r(relu6(d))
    cmid = r["D"].shape[-1]
    W2 = bf16_value(W2)
    y = r["D"].reshape(-1, cmid) @ W2.T + b2
    yabs = np.abs(r["D"]).reshape(-1, cmid) @ np.abs(W2).T + np.abs(b2)
    if residual:
        y = y + X.reshape(y.shape)
        yabs = yabs + np.abs(X).reshape(y.shape)
    r["y"], r["yabs"] = y.reshape(B, Ho, Wo, -1), yabs.reshape(B, Ho, Wo, -1)
    r["W2abs"] = np.abs(W2)
    return r


def rounded_error(v, dv, ref, act=lambda x: x):
    """bound of |bf16(act(v')) - ref| over every v' within dv of v: bf16 rounding and act are monotone, so the two
    ends of the interval bound it.  Where dv cannot move v across a rounding boundary this is |bf16(act(v)) - ref|
    (0 for ref = that value); one bf16 ulp more where it can."""
    return np.maximum(np.abs(bf16r(act(v - dv)) - ref), np.abs(bf16r(act(v + dv)) - ref))


def bounds(r, op, stride, has_expand, fp16):
    """per-element bounds of |E_gpu - E|, |D_gpu - D| and |Y_gpu - y| (E, D the oracle's bf16 values, y unrounded):
    the arithmetic error of each stage (fp32 accumulation, the fp16 terms, the previous stage's error through the
    weights) widened by the stage's bf16 rounding"""
    wd = op["wd"]
    cin = op["X"].shape[-1]
    out = {}
    if has_expand:
        out["E"] = rounded_error(r["e"], gamma(cin + 1) * r["eabs"], r["E"], relu6)
        errE = out["E"]
    else:
        errE = np.zeros_like(r["E"])
    B, Ho, Wo, cmid = r["D"].shape
    if fp16:
        # packed fp16: the weights and the bias rounded to fp16 (2^-11 relative, 2^-25 absolute when subnormal), the
        # inputs too below 2^-14, and nine fused multiply-adds each rounding at 2^-11 of the largest partial sum
        u, tiny = 2.0 ** -11, 2.0 ** -25
        Eabs = dw_sum(pad_hw(np.abs(r["E"])), np.ones(9), stride, Ho, Wo)
        dd = (dw_sum(pad_hw(errE), np.abs(wd) * (1 + u), stride, Ho, Wo) + u * r["dabs"] +
              tiny * (Eabs + 1 + np.abs(wd).sum(0)) + 9 * (u * r["dmax"] * (1 + 2.0 ** -6) + tiny))
    else:
        dd = dw_sum(pad_hw(errE), np.abs(wd), stride, Ho, Wo) + gamma(10) * r["dabs"]
    out["D"] = rounded_error(r["d"], dd, r["D"], relu6)
    dy = (out["D"].reshape(-1, cmid) @ r["W2abs"].T).reshape(r["y"].shape) + gamma(cmid + 2) * r["yabs"]
    out["Y"] = rounded_error(r["y"], dy, r["y"])
    return out


# ---------------------------------------------------------------- operands
def make_operands(kind, B, H, W, cin, cmid, cout, has_expand, seed):
    rng = np.random.default_rng(seed)
    op = {}

    def sparse_signs(rows, cols, nnz):  # {0, +-1/2, +-1}, about nnz non-zeros per row
        m = np.zeros((rows, cols))
        for i in range(rows):
            j = rng.choice(cols, size=min(nnz, cols), replace=False)
            m[i, j] = rng.choice([-1.0, -0.5, 0.5, 1.0], size=j.size)
        return m

    if kind == "exact":
        X = rng.integers(-8, 9, size=(B, H, W, cin)) / 4.0                 # 2^-2 Z, |X| <= 2
        W1 = sparse_signs(cmid, cin, 8)
        b1 = rng.integers(-8, 25, size=cmid) / 8.0                         # 2^-3 Z
        wd = rng.integers(-4, 5, size=(9, cmid)) / 4.0                     # 2^-2 Z, |wd| <= 1
        bd = rng.integers(-64, 129, size=cmid) / 32.0 if has_expand else rng.integers(-32, 33, size=cmid) / 32.0
        W2 = sparse_signs(cout, cmid, 16)
        b2 = rng.integers(-64, 65, size=cout) / 64.0                       # 2^-6 Z
    else:
        X = rng.standard_normal((B, H, W, cin))
        bn = lambda c: rng.uniform(0.8, 1.2, c)                             # folded BatchNorm scale
        W1 = rng.standard_normal((cmid, cin)) * math.sqrt(2.0 / cin) * bn(cmid)[:, None]
        b1 = 0.1 * rng.standard_normal(cmid)
        mag = np.exp(rng.uniform(math.log(2.0 ** -6), math.log(30.0), size=(9, cmid)))
        wd = mag * rng.choice([-1.0, 1.0], size=(9, cmid))                 # a stand-in for trained BN folding
        bd = rng.standard_normal(cmid) * 2.0
        W2 = rng.standard_normal((cout, cmid)) * math.sqrt(1.0 / cmid) * bn(cout)[:, None]
        b2 = 0.1 * rng.standard_normal(cout)
        if kind in ("big_weight", "overflow"):
            # channels whose expansion is the constant 4 inside the image, with taps that cancel there exactly
            W1[:8] = 0.0
            b1[:8] = 4.0
            bd[:8] = 2.0
            big = 70000.0 if kind == "big_weight" else 20000.0
            for c in range(8):
                if kind == "big_weight":   # one weight above the fp16 maximum 65504, cancelled by the last tap
                    wd[:, c] = [big, 0, 0, 0, 0.25, 0, 0, 0, -big]
                else:                      # partial sums reach 4 * 4 * 20000 before the last four taps cancel them
                    wd[:, c] = [big, big, big, big, 0.25, -big, -big, -big, -big]
    op["X"] = bf16_bits(X)
    op["W1"] = bf16_bits(W1)
    op["b1"] = b1.astype(np.float32).astype(np.float64)
    op["wd"] = wd.astype(np.float32).astype(np.float64)
    op["bd"] = bd.astype(np.float32).astype(np.float64)
    op["W2"] = bf16_bits(W2)
    op["b2"] = b2.astype(np.float32).astype(np.float64)
    return op


# ---------------------------------------------------------------- running a case on the GPU
RUNNER = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(root)r)
from audiomuse_ai_b200 import _lib
lib = _lib.load_debug()
lib.am_launch_count.restype = C.c_uint64
a = np.load(%(inp)r)
B, H, W, cin, cmid, cout, S, ex, res = (int(v) for v in a["dims"])
Ho, Wo = (H - 1) // S + 1, (W - 1) // S + 1
p = lambda x: x.ctypes.data_as(C.c_void_p)
f32 = lambda k: np.ascontiguousarray(a[k], dtype=np.float32)
X, W1, W2 = (np.ascontiguousarray(a[k]) for k in ("X", "W1", "W2"))
b1, wd, bd, b2 = f32("b1"), f32("wd"), f32("bd"), f32("b2")
out = {}
for path in (0, 1):
    Y = np.zeros((B, Ho, Wo, cout), np.uint16)
    E = np.zeros((B, H, W, cmid), np.uint16)
    D = np.zeros((B, Ho, Wo, cmid), np.uint16)
    info = C.c_int(-1)
    n0 = lib.am_launch_count()
    st = lib.am_debug_block(path, B, H, W, cin, cmid, cout, S, ex, res, p(X), p(W1) if ex else None,
                            p(b1) if ex else None, p(wd), p(bd), p(W2), p(b2), p(Y), p(E), p(D), C.byref(info))
    out["st%%d" %% path] = st
    out["err%%d" %% path] = lib.am_last_error().decode() if st else ""
    out["launches%%d" %% path] = lib.am_launch_count() - n0
    out["info%%d" %% path] = info.value
    if st == 0:
        out["Y%%d" %% path] = Y
        if path == 1:
            out["E"], out["D"] = E, D
np.savez(%(outp)r, **out)
print("DONE")
"""

_REPORTS = {}  # case -> (fused ring depth or None when rejected, layer depthwise kernel)


def run_case(name, tmp_path):
    kind, B, H, W, (cin, cmid, cout, S, ex, res) = CASES[name]
    op = make_operands(kind, B, H, W, cin, cmid, cout, ex, seed=zlib.crc32(name.encode()))
    inp, outp = str(tmp_path / f"{name}_in.npz"), str(tmp_path / f"{name}_out.npz")
    np.savez(inp, dims=np.array([B, H, W, cin, cmid, cout, S, ex, res]), **op)
    r = subprocess.run([sys.executable, "-c", RUNNER % dict(root=ROOT, inp=inp, outp=outp)], capture_output=True,
                       text=True, timeout=300)
    assert "DONE" in r.stdout, f"{name}: rc={r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}"
    res_ = dict(np.load(outp))
    assert res_["st1"] == 0, f"{name}: layer path failed: {res_['err1']}"
    fused_ok = res_["st0"] == 0
    _REPORTS[name] = (int(res_["info0"]) if fused_ok else None, int(res_["info1"]))
    return op, res_


def _mismatch(name, what, got, want, bound=None):
    bad = np.argwhere(~(np.abs(got - want) <= (0 if bound is None else bound)))
    i = tuple(bad[0])
    extra = "" if bound is None else f" bound {bound[i]:.4g}"
    return (f"{name}: {what}: {len(bad)} of {got.size} elements differ; first at {i}: gpu {got[i]!r}, oracle "
            f"{want[i]!r}{extra}")


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c[0] == "exact"])
def test_block_bit_exact_on_dyadic_grid(name, tmp_path):
    kind, B, H, W, (cin, cmid, cout, S, ex, res) = CASES[name]
    op, out = run_case(name, tmp_path)
    r = oracle(op, S, ex, res)
    # not vacuous: a sizeable share of the expanded and depthwise values lies strictly inside the ReLU6 range
    if ex:
        assert np.mean((r["E"] > 0) & (r["E"] < 6)) >= 0.3, np.mean((r["E"] > 0) & (r["E"] < 6))
    assert np.mean((r["D"] > 0) & (r["D"] < 6)) >= 0.3, np.mean((r["D"] > 0) & (r["D"] < 6))
    # the grid keeps every value exact in fp32 (and fp16 for the depthwise), so the oracle's roundings are the GPU's
    assert np.all(np.abs(r["y"]) < 2.0 ** 17) and np.all(r["dmax"] < 64)
    Y = bf16_bits(r["y"])
    if cout <= 256:
        assert out["st0"] == 0, f"{name}: fused path failed: {out['err0']}"
        assert np.array_equal(out["Y0"], Y), _mismatch(name, "fused Y", bf16_value(out["Y0"]), bf16_value(Y))
    else:
        assert out["st0"] != 0 and out["launches0"] == 0, f"{name}: cout_p {cout} > 256 must be refused unlaunched"
    if ex:
        assert np.array_equal(out["E"], bf16_bits(r["E"])), _mismatch(name, "E", bf16_value(out["E"]), r["E"])
    assert np.array_equal(out["D"], bf16_bits(r["D"])), _mismatch(name, "D", bf16_value(out["D"]), r["D"])
    assert np.array_equal(out["Y1"], Y), _mismatch(name, "layer Y", bf16_value(out["Y1"]), bf16_value(Y))


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c[0] != "exact"])
def test_block_within_bound_on_realistic_operands(name, tmp_path):
    kind, B, H, W, (cin, cmid, cout, S, ex, res) = CASES[name]
    op, out = run_case(name, tmp_path)
    r = oracle(op, S, ex, res)
    b32 = bounds(r, op, S, ex, fp16=False)
    if cout <= 256:
        assert out["st0"] == 0, f"{name}: fused path failed: {out['err0']}"
        y0 = bf16_value(out["Y0"])
        assert np.all(np.abs(y0 - r["y"]) <= b32["Y"]), _mismatch(name, "fused Y", y0, r["y"], b32["Y"])
    else:
        assert out["st0"] != 0 and out["launches0"] == 0, f"{name}: cout_p {cout} > 256 must be refused unlaunched"
    # layer by layer: the fp16 terms only where the packed-fp16 depthwise ran; the fp16-range cases must keep the
    # fp32 bound whichever kernel ran
    fp16 = out["info1"] in (DW_STRIP, DW_ROW) and kind == "real"
    b = bounds(r, op, S, ex, fp16=True) if fp16 else b32
    if ex:
        e1 = bf16_value(out["E"])
        assert np.all(np.abs(e1 - r["E"]) <= b["E"]), _mismatch(name, "E", e1, r["E"], b["E"])
    d1, y1 = bf16_value(out["D"]), bf16_value(out["Y1"])
    assert np.all(np.abs(d1 - r["D"]) <= b["D"]), _mismatch(name, "D", d1, r["D"], b["D"])
    assert np.all(np.abs(y1 - r["y"]) <= b["Y"]), _mismatch(name, "layer Y", y1, r["y"], b["Y"])


def test_every_branch_is_reached(tmp_path):
    """the cases together reach every ring depth, depthwise kernel and edge shape listed in the module docstring"""
    for name in CASES:
        if name not in _REPORTS:
            run_case(name, tmp_path)
    fused = {n: CASES[n] for n in CASES if _REPORTS[n][0] is not None}
    depth = {n: _REPORTS[n][0] for n in fused}
    assert [depth[f"exact_b{i}"] for i in range(5)] == SHIPPED_DEPTHS
    assert [depth[f"real_b{i}"] for i in range(5)] == SHIPPED_DEPTHS
    assert depth["exact_alpha6_b1"] == 1 and depth["real_alpha6_b1"] == 1
    assert set(depth.values()) == {1, 2, 3, 4}

    def has(pred):
        return any(pred(B, H, W, *shape) for _, B, H, W, shape in fused.values())

    for s in (1, 2):
        for e in (0, 1):
            assert has(lambda B, H, W, ci, cm, co, S, ex, res: S == s and ex == e), (s, e)
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: res and ex) and has(lambda B, H, W, ci, cm, co, S, ex, res: res and not ex)
    for tail in (16, 32, 48):  # the last chunk of the expanded channels
        assert has(lambda B, H, W, ci, cm, co, S, ex, res: cm % 64 == tail), tail
    for chunks in (1, 2):
        assert has(lambda B, H, W, ci, cm, co, S, ex, res: (cm + 63) // 64 == chunks), chunks
    for ci_ in (16, 48, 80, 144, 208):  # K tails and 1-4 K blocks of the expansion
        assert has(lambda B, H, W, ci, cm, co, S, ex, res: ex and ci == ci_), ci_
    for co_ in (16, 64, 80, 144, 192, 256):  # 1-4 projection column blocks
        assert has(lambda B, H, W, ci, cm, co, S, ex, res: co == co_), co_
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: S == 2 and H % 2 and W % 2)
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: W < 8)
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: H == 1 and W == 1)
    out_hw = lambda H, W, S: ((H - 1) // S + 1, (W - 1) // S + 1)
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: all(v % 8 for v in out_hw(H, W, S)))
    tiles = lambda B, H, W, S: B * math.ceil(out_hw(H, W, S)[0] / 8) * math.ceil(out_hw(H, W, S)[1] / 8)
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: tiles(B, H, W, S) < 100)       # fewer tiles than SMs
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: tiles(B, H, W, S) >= 3 * 132)  # several tiles per CTA
    assert has(lambda B, H, W, ci, cm, co, S, ex, res: B == 1) and has(lambda B, H, W, ci, cm, co, S, ex, res: B == 3)
    # layer by layer
    kernels = {(CASES[n][4][3], _REPORTS[n][1]) for n in CASES}
    for k in ((1, DW_STRIP), (2, DW_STRIP), (1, DW_ROW), (2, DW_ROW)):
        assert k in kernels, k
    assert _REPORTS["fp16_weight_above_max"][1] == DW_GENERIC
    assert _REPORTS["fp16_partial_sum_overflow"][1] == DW_GENERIC
    assert all(_REPORTS[f"real_b{i}"][0] is None for i in range(5, 9))  # blocks 5-8: refused by the fused plan
