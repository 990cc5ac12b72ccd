"""The fused block kernel's tall tile (16 time rows x 8 mel columns, stride 1): which blocks take it, and bit-exact
outputs at its edges.

The plan gives the tall tile to a stride-1 block with cout_p <= 128 when its layout keeps the ring as deep as the 8 x 8
tile's; for the shipped student that is blocks 0 and 2 (block 4 has cout_p 144, and would fit 2 stages against 3).
am_debug_block's path 2 reports the plan's tile height on the host, without a device.

The GPU cases run the block on the dyadic grid of tests/test_gpu_block_exact.py, where every sum is exact, so the
fused Y must equal the float64 oracle bit for bit: a time extent that is not a multiple of 16, fewer tiles than SMs,
partial tiles along mel, cout_p 128 and 16, and the no-expansion and residual variants."""
import ctypes as C
import math
import subprocess
import sys
import zlib

import numpy as np
import pytest

from tests import test_gpu_block_exact as bx

PLAN_PATH = 2  # include/audiomuse_b200_debug.h, am_debug_block


def _tile_h(B, H, W, cin, cmid, cout, S, ex, res):
    from audiomuse_ai_b200 import _lib
    lib = _lib.load_debug()
    info = C.c_int(-1)
    st = lib.am_debug_block(PLAN_PATH, B, H, W, cin, cmid, cout, S, ex, res, *([None] * 10), C.byref(info))
    assert st == 0, lib.am_last_error().decode()
    return info.value


def test_plan_picks_the_tall_tile_for_shipped_blocks_0_and_2():
    heights = [_tile_h(1, H, W, *shape) for shape, (H, W) in bx.SHIPPED[:5]]
    assert heights == [16, 8, 16, 8, 8]


def test_plan_takes_the_tall_tile_at_stride_1_up_to_cout_128_only():
    assert _tile_h(1, 31, 21, 48, 96, 144, 1, 1, 0) == 8   # cout_p > 128
    assert _tile_h(1, 31, 21, 64, 128, 64, 2, 1, 0) == 8   # stride 2
    assert _tile_h(1, 31, 21, 16, 48, 16, 1, 1, 1) == 16


# name: (B, H, W, (cin_p, cmid_p, cout_p, stride, has_expand, residual)); every case takes the tall tile
CASES = {
    # no expansion (block 0's shape): 37 = 2 x 16 + 5 time rows, 21 = 2 x 8 + 5 mel columns, 9 tiles
    "tall_noexp_b0": (1, 37, 21, bx.SHIPPED[0][0]),
    # expansion + residual (block 2's shape), two windows of 43 = 2 x 16 + 11 rows
    "tall_res_b2": (2, 43, 19, bx.SHIPPED[2][0]),
    # cout_p = 128, the widest projection a warpgroup takes over all the columns; fewer rows than one tile
    "tall_c128": (1, 11, 13, (128, 192, 128, 1, 1, 1)),
    # cout_p = 16, cin_p = 16 (one K step of the expansion); narrower than one tile along mel
    "tall_c16": (3, 33, 5, (16, 48, 16, 1, 1, 1)),
    # no expansion + residual, with a partial last chunk (80 channels = 64 + 16)
    "tall_noexp_res": (1, 50, 11, (80, 80, 80, 1, 0, 1)),
    # several tiles per CTA: 8 windows x 16 x 4 = 512 tiles
    "tall_many_tiles": (8, 256, 32, (48, 96, 64, 1, 1, 0)),
}


def test_cases_take_the_tall_tile():
    for name, (B, H, W, shape) in CASES.items():
        assert _tile_h(B, H, W, *shape) == 16, name


def _tiles(B, H, W):
    return B * math.ceil(H / 16) * math.ceil(W / 8)


def test_cases_cover_the_edges():
    shapes = list(CASES.values())
    assert any(H % 16 for _, H, _, _ in shapes) and any(W % 8 for _, _, W, _ in shapes)
    assert any(_tiles(B, H, W) < 100 for B, H, W, _ in shapes)
    assert any(_tiles(B, H, W) >= 3 * 132 for B, H, W, _ in shapes)
    for want in ((0, 0), (0, 1), (1, 1)):
        assert any((s[4], s[5]) == want for _, _, _, s in shapes), want
    assert {s[2] for _, _, _, s in shapes} >= {16, 128}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_tall_tile_bit_exact_on_dyadic_grid(name, tmp_path):
    B, H, W, (cin, cmid, cout, S, ex, res) = CASES[name]
    op = bx.make_operands("exact", B, H, W, cin, cmid, cout, ex, seed=zlib.crc32(name.encode()))
    inp, outp = str(tmp_path / f"{name}_in.npz"), str(tmp_path / f"{name}_out.npz")
    np.savez(inp, dims=np.array([B, H, W, cin, cmid, cout, S, ex, res]), **op)
    r = subprocess.run([sys.executable, "-c", bx.RUNNER % dict(root=bx.ROOT, inp=inp, outp=outp)],
                       capture_output=True, text=True, timeout=300)
    assert "DONE" in r.stdout, f"{name}: rc={r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}"
    out = dict(np.load(outp))
    assert out["st0"] == 0, f"{name}: fused path failed: {out['err0']}"
    ref = bx.oracle(op, S, ex, res)
    assert np.mean((ref["D"] > 0) & (ref["D"] < 6)) >= 0.3  # not vacuous
    assert np.all(np.abs(ref["y"]) < 2.0 ** 17) and np.all(ref["dmax"] < 64)
    Y = bx.bf16_bits(ref["y"])
    assert np.array_equal(out["Y0"], Y), bx._mismatch(name, "fused Y", bx.bf16_value(out["Y0"]), bx.bf16_value(Y))
    assert np.array_equal(out["Y1"], Y), bx._mismatch(name, "layer Y", bx.bf16_value(out["Y1"]), bx.bf16_value(Y))
