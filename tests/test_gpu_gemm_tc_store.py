"""The TMA box stores of the element-wise gemm_tc epilogues (bias -> float32, LeakyReLU + BatchNorm -> hi/lo planes or
float32): with an output pitch wider than N and guard rows after M, only rows [0, M) x columns [0, N) change and they
hold the bytes of the same GEMM written at pitch N; an output base or pitch off 16-byte alignment is refused."""
import ctypes as C

import pytest

from diart_b200 import _lib

pytestmark = pytest.mark.gpu

SHAPES = [  # (M, Cin, N, epi); N <= 64 runs on 64-wide tiles for epi 0 (one partial 128-wide tile for epi 1 and 2)
    (1001, 64, 36, 0),       # 64-wide tiles: ragged M, one partial 32-column box
    (3001, 128, 200, 0),     # 128-wide tiles: ragged M, the second column tile ragged
    (777, 64, 52, 2),        # one partial column tile, LeakyReLU + BatchNorm -> float32
    (2049, 64, 300, 2),      # three column tiles, the last one ragged
    (999, 128, 32, 1),       # hi/lo planes: one partial 64-column box
    (1500, 64, 160, 1),      # two column tiles, the second one holds half a box
]


@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_tc_box_store_stays_inside_the_output(shape, cuda_device):
    M, Cin, N, epi = shape
    outside, equal, refused = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_bounds(M, Cin, N, epi, C.byref(outside), C.byref(equal), C.byref(refused)))
    assert outside.value == 1, f"shape {shape}: bytes outside rows [0, M) x columns [0, N) changed"
    assert equal.value == 1, f"shape {shape}: the output at pitch N + 40 differs from the output at pitch N"
    assert refused.value == 1, f"shape {shape}: a misaligned output base or pitch was accepted"
