"""The encoder's steps outside the inverted-residual block, element by element against float64, through the encoder's
own dispatch (am_debug_encoder_trace in libaudiomuse_b200_debug.so: run_steps / forward_late / head_forward).

Every step and every head op is checked against oracle/encoder_steps.py, computed from the device's own input to it
(the log-mel, the previous step's traced bf16 output, the traced head registers), so errors do not compound.  The
bound per element is derived from the kernels' rounding points (see that module's docstring):

    stem          gamma(11) sum |dw| (|mel sc| + |sh|) through pw_scale, + the epilogue FMA, + half a bf16 ulp
    conv_first    gamma(kh kw + 2) (|b| + sum |w| |x|) through the activation (Lipschitz + fp32 evaluation)
    dw_generic    gamma(k^2 + 1) (|b| + sum |w| |x|) through the activation
    pointwise     gamma(cin_p + 2) (|b| + sum |x| |w_bf16|) through the epilogue's activation, + the residual add
    squeeze_excite channel mean gamma(HW + 1), both gate layers gamma(n + 1) with the activations, x * gate
    pool          gamma(n + 2) mean |x| over the stride lattice
    linear        3.02 * 2^-16 sum |x| |w| (split-bf16 representation) + gamma(3 Kp + 1) sum |terms|, input act error
    unary / add / affine   the fp32 evaluation (expf, erff, tanhf within 2 ulp) and one rounding
    layernorm     mean gamma(E + 1), variance gamma(E + 1), rsqrtf 2 ulp, the affine; l2norm gamma(E + 1) and sqrtf
    add_ln_l2     a + b rounded once, carried through LayerNorm's sensitivity, then the two above
    every stored value: half a bf16 ulp (trunk) or an fp32 rounding (head)

The fused block and the 3x3 depthwise steps (kStepFused, kStepDw3x3) are covered by tests/test_gpu_block_exact.py; here
their outputs only feed the next step's oracle (and their padded channels are checked).

Beyond the bounds: every trunk output's padded channels are exactly zero (the GEMM's K loop reads them), the trace's
embedding equals am_clap_embed's bit for bit, the cases together reach every step kind and head-op kind
(test_every_step_kind_is_reached), and each fault listed in test_bounds_catch_the_plausible_faults, evaluated as a
perturbed oracle on the traced data, falls outside its bound somewhere.

Each case runs in a subprocess under a timeout."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import encoder_steps as O  # noqa: E402


class Zoo(nn.Module):
    """What neither network reaches: a 5x3 stride-2 first convolution on the (time, mel) view after a per-mel
    BatchNorm and an asymmetric ZeroPad2d, a 7x7 stride-2 depthwise, squeeze-excite with a Sigmoid gate, and a head
    with a bias-free Linear, a standalone GELU, Tanh / Sigmoid, a constant scale and shift, a plain LayerNorm on a
    low-variance row and an Add skip, ending in F.normalize."""

    def __init__(self, n_mels=128, c0=24, c1=40, d=48, emb=32):
        super().__init__()
        self.bn0 = nn.BatchNorm2d(n_mels)
        self.pad = nn.ZeroPad2d((1, 2, 2, 1))               # mel left / right, time top / bottom
        self.conv0 = nn.Conv2d(1, c0, (5, 3), stride=2)
        self.dw7 = nn.Conv2d(c0, c0, 7, stride=2, padding=3, groups=c0)
        self.fc1, self.fc2 = nn.Conv2d(c0, 8, 1), nn.Conv2d(8, c0, 1)
        self.pw = nn.Conv2d(c0, c1, 1)
        self.lin1 = nn.Linear(c1, d)
        self.scale = nn.Parameter(0.01 * (1.0 + torch.rand(d)))
        self.shift = nn.Parameter(0.1 * torch.randn(d))
        self.ln = nn.LayerNorm(d)
        self.lin2 = nn.Linear(d, emb, bias=False)

    def forward(self, mel):
        x = mel.transpose(2, 3)                             # (B, 1, T, mel)
        x = self.bn0(x.permute(0, 3, 2, 1)).permute(0, 3, 2, 1)
        x = F.relu(self.conv0(self.pad(x)))
        x = F.hardswish(self.dw7(x))
        s = torch.sigmoid(self.fc2(F.relu(self.fc1(x.mean((2, 3), keepdim=True)))))
        x = F.relu6(self.pw(x * s))
        h = self.lin1(x.mean((2, 3)))
        g = F.gelu(h)
        t = torch.tanh(g) * self.scale + self.shift
        return F.normalize(self.lin2(torch.sigmoid(self.ln(t)) + g), p=2, dim=1)


def make_zoo(seed=7):
    from oracle.phinet import synthetic_mel
    torch.manual_seed(seed)
    m = Zoo()
    m.bn0.momentum = 1.0
    with torch.no_grad():
        m.ln.weight.copy_(0.5 + torch.rand(m.ln.weight.shape))
        m.ln.bias.copy_(0.1 * torch.randn(m.ln.bias.shape))
    m.train()
    with torch.no_grad():
        m(synthetic_mel(2, 128, 201, seed + 1))
    return m.eval()


def _model(kind):
    from oracle import mobilenet, phinet
    if kind == "phinet_small":
        return phinet.make_random_student(3, phinet.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256))
    if kind == "phinet_full":
        return phinet.make_random_student(0)
    if kind == "mobilenet_small":
        return mobilenet.make_random_mobilenet(5, mobilenet.MNConfig(rows=mobilenet.SMALL_ROWS, head_dim=256))
    return make_zoo()


# name: (model, B, T, AM_FUSED_BLOCKS)
CASES = {
    "phinet_small_T101_B3": ("phinet_small", 3, 101, 1),     # short: the late phase holds every block
    "phinet_small_T333_B1": ("phinet_small", 1, 333, 1),
    "phinet_small_T333_B3": ("phinet_small", 3, 333, 1),
    "phinet_small_unfused_T101_B3": ("phinet_small", 3, 101, 0),
    "phinet_full_T1001_B1": ("phinet_full", 1, 1001, 1),
    "mobilenet_small_T129_B3": ("mobilenet_small", 3, 129, 1),
    "mobilenet_small_T400_B1": ("mobilenet_small", 1, 400, 1),
    "zoo_T157_B3": ("zoo", 3, 157, 1),
    "zoo_T64_B1": ("zoo", 1, 64, 1),
}

RUNNER = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(root)r)
from audiomuse_ai_b200 import _lib
dbg = _lib.load_debug()
for name in ("am_clap_load", "am_clap_free", "am_clap_embedding_dim"):
    getattr(dbg, name).restype, getattr(dbg, name).argtypes = _lib.SIGNATURES[name]
p = lambda x: x.ctypes.data_as(C.c_void_p)
def chk(st):
    if st:
        raise SystemExit("error %%d: %%s" %% (st, dbg.am_last_error().decode()))
a = np.load(%(inp)r)
mel = np.ascontiguousarray(a["mel"], np.float32)
B, n_mels, T = mel.shape
m = C.c_void_p()
chk(dbg.am_clap_load(%(model)r.encode(), C.byref(m)))
counts = np.zeros(4, np.int32)
chk(dbg.am_debug_encoder_plan(m, T, p(counts), None, None, None, None))
ns, late, nl, nh = (int(v) for v in counts)
steps = np.zeros((ns, 9), np.int32); layers = np.zeros((nl, 18), np.int32)
head = np.zeros((nh, 8), np.int32); heps = np.zeros((nh, 2), np.float32)
chk(dbg.am_debug_encoder_plan(m, T, p(counts), p(steps), p(layers), p(head), p(heps)))
n_step = sum(B * int(s[5]) * int(s[6]) * int(s[7]) for s in steps)
n_head = sum(B * int(h[5]) for h in head)
E = dbg.am_clap_embedding_dim(m)
so = np.full(n_step, 0xFFFF, np.uint16); ho = np.full(n_head, np.nan, np.float32); emb = np.zeros((B, E), np.float32)
chk(dbg.am_debug_encoder_trace(m, p(mel), B, T, p(so), p(ho), p(emb)))
dbg.am_clap_free(m)
# the product library's entry point on the same input
lib = _lib.load()
m2 = C.c_void_p()
_lib.check(lib.am_clap_load(%(model)r.encode(), C.byref(m2)))
emb2 = np.zeros((B, E), np.float32)
_lib.check(lib.am_clap_embed(m2, p(mel), B, T, p(emb2)))
lib.am_clap_free(m2)
np.savez(%(outp)r, counts=counts, steps=steps, layers=layers, head=head, heps=heps, so=so, ho=ho, emb=emb, emb2=emb2)
print("DONE")
"""

LAYER_FIELDS = ["type", "cin", "cout", "kh", "kw", "stride", "pad_t", "pad_b", "pad_l", "pad_r", "act", "gate_act", "cmid",
                "h_is_time", "residual", "block_start", "cin_p", "cout_p"]
STEP_FIELDS = ["kind", "first", "last", "in_h", "in_w", "out_h", "out_w", "cout_p", "starts_block"]
HEAD_FIELDS = ["kind", "a", "b", "dst", "K", "N", "act", "stride"]

_MODELS = {}   # model kind -> onnx path
_TRACES = {}   # case -> traced and checked data
_WORST = {}    # step / head kind name -> worst error / bound


def _export(kind, tmp_path_factory):
    if kind not in _MODELS:
        from tests import onnx_export
        d = tmp_path_factory.mktemp("encoder_steps")
        _MODELS[kind] = (onnx_export.export_onnx(_model(kind), str(d / f"{kind}.onnx")), str(d))
    return _MODELS[kind]


def run_case(name, tmp_path_factory):
    if name in _TRACES:
        return _TRACES[name]
    from oracle import onnx_ref, phinet
    kind, B, T, fused = CASES[name]
    path, d = _export(kind, tmp_path_factory)
    mel = phinet.synthetic_mel(B, 128, T, 100 + T).numpy().reshape(B, 128, T)
    inp, outp = os.path.join(d, f"{name}_in.npz"), os.path.join(d, f"{name}_out.npz")
    np.savez(inp, mel=mel)
    env = dict(os.environ, AM_FUSED_BLOCKS=str(fused))
    r = subprocess.run([sys.executable, "-c", RUNNER % dict(root=ROOT, inp=inp, outp=outp, model=path)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert "DONE" in r.stdout, f"{name}: rc={r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}"
    a = dict(np.load(outp))
    steps = [dict(zip(STEP_FIELDS, map(int, s))) for s in a["steps"]]
    layers = [dict(zip(LAYER_FIELDS, map(int, s))) for s in a["layers"]]
    head = [dict(zip(HEAD_FIELDS, map(int, h)), eps=float(e[0]), eps2=float(e[1])) for h, e in zip(a["head"], a["heps"])]
    outs, off = [], 0
    for s in steps:
        n = B * s["out_h"] * s["out_w"] * s["cout_p"]
        outs.append(a["so"][off:off + n].reshape(B, s["out_h"], s["out_w"], s["cout_p"]))
        off += n
    houts, off = [], 0
    for h in head:
        houts.append(a["ho"][off:off + B * h["N"]].reshape(B, h["N"]).astype(np.float64))
        off += B * h["N"]
    W, HW = O.extract_weights(onnx_ref.load(path), layers, head)
    t = dict(name=name, B=B, T=T, mel=mel.astype(np.float64), steps=steps, layers=layers, head=head, outs=outs,
             houts=houts, W=W, HW=HW, late=int(a["counts"][1]), emb=a["emb"], emb2=a["emb2"])
    _TRACES[name] = t
    return t


def step_input(t, q):
    return t["mel"] if q == 0 else O.bf16_value(t["outs"][q - 1])


def block_in(t, q):
    """the residual source of step q: the input of the latest block-starting step at or before it"""
    for j in range(q, -1, -1):
        if t["steps"][j]["starts_block"]:
            return step_input(t, j)
    raise AssertionError("no block start")


def step_oracle(t, q, **fault):
    s = t["steps"][q]
    L, W = t["layers"][s["last"]], t["W"][s["last"]]
    x = step_input(t, q)
    k = s["kind"]
    if k == O.S_STEM:
        return O.stem(x, W, L, s["out_h"], s["out_w"], **fault)
    if k == O.S_CONV_FIRST:
        return O.conv_first(x, W, L, s["out_h"], s["out_w"])
    if k == O.S_DW_GENERIC:
        return O.depthwise(x[..., :L["cin"]], W, L, s["out_h"], s["out_w"])
    if k == O.S_SQUEEZE_EXCITE:
        return O.squeeze_excite(x[..., :L["cin"]], W, L)
    if k == O.S_POINTWISE:
        res = block_in(t, q)[..., :L["cout"]] if L["residual"] else None
        return O.pointwise(x[..., :L["cin"]], W, L, res, **fault)
    return None


def head_oracle(t, q, **fault):
    h, W = t["head"][q], t["HW"][q]
    regs = {}
    for j in range(q):
        regs[t["head"][j]["dst"]] = t["houts"][j]
    k = h["kind"]
    if k == O.V_POOL:
        X = O.bf16_value(t["outs"][-1])
        return O.pool(X, h["N"], 1 if fault.get("every_position") else h["stride"])
    a = regs.get(h["a"])
    if k == O.V_LINEAR:
        return O.linear(a, W["w"], W["b"], h["act"], gelu_tanh=fault.get("gelu_tanh", False),
                        drop_lo=fault.get("drop_lo", False))
    if k == O.V_UNARY:
        return O.unary(a, h["act"], gelu_tanh=fault.get("gelu_tanh", False))
    if k == O.V_ADD:
        return O.add(a, regs[h["b"]])
    if k == O.V_AFFINE:
        return O.affine(a, W["scale"], W["shift"])
    if k == O.V_LAYERNORM:
        return O.layernorm(a, W["g"], W["b"], h["eps"], eps_outside=fault.get("eps_outside", False))
    if k == O.V_L2NORM:
        return O.l2norm(a, h["eps2"])
    if k == O.V_ADD_LN_L2:
        return O.add_ln_l2(a, regs[h["b"]], W["g"], W["b"], h["eps"], h["eps2"], eps_outside=fault.get("eps_outside", False))
    raise AssertionError(k)


def _worst(key, ratio):
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)


@pytest.mark.parametrize("name", list(CASES))
def test_steps_and_head_within_bounds(name, tmp_path_factory):
    t = run_case(name, tmp_path_factory)
    np.testing.assert_array_equal(t["emb"], t["emb2"], err_msg=f"{name}: trace and am_clap_embed differ")
    for q, s in enumerate(t["steps"]):
        L = t["layers"][s["last"]]
        out = t["outs"][q]
        assert np.all(out[..., L["cout"]:] == 0), f"{name}: step {q} ({O.STEP_NAMES[s['kind']]}) padded channels"
        r = step_oracle(t, q)
        if r is None:
            continue
        y, e = r
        got = O.bf16_value(out[..., :L["cout"]])
        bound = O.output_bound(y, e)
        err = np.abs(got - y)
        bad = np.argwhere(~(err <= bound))
        assert bad.size == 0, (f"{name}: step {q} ({O.STEP_NAMES[s['kind']]}): {len(bad)} of {got.size} elements out of "
                               f"bound; first {tuple(bad[0])}: gpu {got[tuple(bad[0])]!r} oracle {y[tuple(bad[0])]!r} "
                               f"bound {bound[tuple(bad[0])]:.3g}")
        _worst(O.STEP_NAMES[s["kind"]], float((err / bound).max()))
    for q, h in enumerate(t["head"]):
        y, e = head_oracle(t, q)
        got = t["houts"][q]
        bound = O.output_bound(y, e, bf16=False)
        err = np.abs(got - y)
        bad = np.argwhere(~(err <= bound))
        assert bad.size == 0, (f"{name}: head op {q} ({O.HEAD_NAMES[h['kind']]}): {len(bad)} of {got.size} out of bound; "
                               f"first {tuple(bad[0])}: gpu {got[tuple(bad[0])]!r} oracle {y[tuple(bad[0])]!r} bound "
                               f"{bound[tuple(bad[0])]:.3g}")
        _worst(O.HEAD_NAMES[h["kind"]], float((err / bound).max()))
    np.testing.assert_array_equal(t["houts"][-1].astype(np.float32), t["emb"])
    print(f"[encoder steps] {name}: worst error / bound " +
          ", ".join(f"{k} {v:.3f}" for k, v in sorted(_WORST.items())))


def test_every_step_kind_is_reached(tmp_path_factory):
    """the cases together reach every step kind and head-op kind, and the plan shapes listed in the docstring"""
    for name in CASES:
        run_case(name, tmp_path_factory)
    kinds = {s["kind"] for t in _TRACES.values() for s in t["steps"]}
    hkinds = {h["kind"] for t in _TRACES.values() for h in t["head"]}
    assert kinds == set(range(7)), sorted(kinds)
    assert hkinds == set(range(8)), sorted(hkinds)
    assert _TRACES["phinet_small_T101_B3"]["late"] == 1            # the late phase holds every block
    assert _TRACES["phinet_small_T333_B3"]["late"] > 1
    layer_of = lambda t, k: [t["layers"][s["last"]] for s in t["steps"] if s["kind"] == k]
    mn = _TRACES["mobilenet_small_T129_B3"]
    assert layer_of(mn, O.S_CONV_FIRST)[0]["h_is_time"] == 0
    dws = {(L["kh"], L["stride"]) for t in _TRACES.values() for L in layer_of(t, O.S_DW_GENERIC)}
    assert {(3, 1), (3, 2), (5, 1), (5, 2), (7, 2)} <= dws, dws
    gates = {(L["act"], L["gate_act"]) for t in _TRACES.values() for L in layer_of(t, O.S_SQUEEZE_EXCITE)}
    assert (O.ACT_RELU, O.ACT_HSIGMOID) in gates and (O.ACT_RELU, O.ACT_SIGMOID) in gates, gates
    pw_acts = {L["act"] for t in _TRACES.values() for L in layer_of(t, O.S_POINTWISE)}
    assert {O.ACT_NONE, O.ACT_RELU6, O.ACT_RELU, O.ACT_HSWISH} <= pw_acts, pw_acts
    assert any(L["residual"] for t in _TRACES.values() for L in layer_of(t, O.S_POINTWISE))
    assert any(L["act"] == O.ACT_RELU6 for L in layer_of(_TRACES["phinet_small_unfused_T101_B3"], O.S_POINTWISE))
    pools = {h["stride"] for t in _TRACES.values() for h in t["head"] if h["kind"] == O.V_POOL}
    assert pools == {1, 2}, pools
    lin_acts = {h["act"] for t in _TRACES.values() for h in t["head"] if h["kind"] == O.V_LINEAR}
    assert {O.ACT_NONE, O.ACT_GELU, O.ACT_HSWISH} <= lin_acts, lin_acts
    unaries = {h["act"] for t in _TRACES.values() for h in t["head"] if h["kind"] == O.V_UNARY}
    assert {O.ACT_GELU, O.ACT_TANH, O.ACT_SIGMOID} <= unaries, unaries
    zoo = _TRACES["zoo_T157_B3"]
    c0 = layer_of(zoo, O.S_CONV_FIRST)[0]
    assert (c0["kh"], c0["kw"], c0["stride"], c0["h_is_time"]) == (5, 3, 2, 1)
    assert (c0["pad_t"], c0["pad_b"], c0["pad_l"], c0["pad_r"]) == (2, 1, 1, 2)
    assert any(h["kind"] == O.V_LINEAR and zoo["HW"][q]["b"] is None for q, h in enumerate(zoo["head"]))


def _outside(y, e, y_fault, bf16):
    return bool(np.any(np.abs(y_fault - y) > O.output_bound(y, e, bf16=bf16)))


def test_bounds_catch_the_plausible_faults(tmp_path_factory):
    """each fault, as a perturbed oracle on the traced inputs, leaves its bound somewhere (host-side, no GPU work)"""
    for name in CASES:
        run_case(name, tmp_path_factory)
    caught = {}

    def mark(fault, hit):
        caught[fault] = caught.get(fault, False) or hit

    for t in _TRACES.values():
        for q, s in enumerate(t["steps"]):
            L = t["layers"][s["last"]]
            if s["kind"] == O.S_STEM:
                y, e = step_oracle(t, q)
                mark("stem: bn0 applied to the padding", _outside(y, e, step_oracle(t, q, bn_on_padding=True)[0], True))
            if s["kind"] == O.S_POINTWISE and L["act"] == O.ACT_HSWISH:
                y, e = step_oracle(t, q)
                mark("GEMM epilogue: hardswish slope 0.2", _outside(y, e, step_oracle(t, q, hsig_slope=0.2)[0], True))
        for q, h in enumerate(t["head"]):
            y, e = head_oracle(t, q)
            if h["kind"] == O.V_POOL and h["stride"] > 1:
                mark("pool: every position", _outside(y, e, head_oracle(t, q, every_position=True)[0], False))
            if h["kind"] == O.V_LINEAR:
                mark("linear: split-bf16 without its lo terms", _outside(y, e, head_oracle(t, q, drop_lo=True)[0], False))
            if h["act"] == O.ACT_GELU and h["kind"] in (O.V_LINEAR, O.V_UNARY):
                mark("GELU in its tanh form", _outside(y, e, head_oracle(t, q, gelu_tanh=True)[0], False))
            if h["kind"] in (O.V_LAYERNORM, O.V_ADD_LN_L2):
                mark("LayerNorm: eps outside the square root",
                     _outside(y, e, head_oracle(t, q, eps_outside=True)[0], False))
    assert len(caught) == 6 and all(caught.values()), caught
