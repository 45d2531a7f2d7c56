"""The weight-stationary MaxPool3 kernel of the wgmma GEMM (SincNet's conv1 and conv2): W stays in shared memory as the A
operand and the tile's halo rows are the B operand (D^T = W . X^T).  Checks that a B descriptor may start any whole number
of rows into a 64B-swizzled tile, that the kernel is taken for SincNet's shapes and writes the bytes of the tap-box kernel,
and that its pooled rows match the float32 SIMT GEMM pooled on the host."""
import ctypes as C

import pytest

from diart_b200 import _lib

pytestmark = pytest.mark.gpu


def test_wgmma_b_descriptor_row_shift(cuda_device):
    # base offset field 0, as for the A operand: a B start r rows into a tile is exact
    ok = C.c_uint()
    _lib.check(_lib.lib().dg_selftest_wgmma_b_row_shift(0, C.byref(ok)))
    assert ok.value == 0x1FF, f"shifts 0..8 exact: {ok.value:09b}"


SWAPPED_SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (888 * 6, 80, 5, 1, 60, 5),      # sinc_conv1, last halo past M
    (888 * 2, 64, 5, 1, 60, 5),      # sinc_conv2
    (888 * 3, 48, 3, 1, 64, 5),      # an odd number of k16 steps per tap
    (888 * 2, 64, 3, 2, 64, 5),      # dilation 2
    (888 * 40, 80, 5, 1, 60, 5),     # 320 tiles: more than one per SM on either consumer
]


@pytest.mark.parametrize("shape", SWAPPED_SHAPES)
def test_swapped_equals_tap_boxes(shape, cuda_device):
    # the same products in the same order per output element: pooled rows and InstanceNorm partials byte-equal
    equal, halo = C.c_int(), C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_halo(*shape, C.byref(equal), C.byref(halo)))
    assert halo.value == 1
    assert equal.value == 1


SIMT_SHAPES = [  # (M, Cin, KW, dil, N)
    (888 * 6, 80, 5, 1, 60),         # sinc_conv1
    (888 * 2, 64, 5, 1, 60),         # sinc_conv2
    (888 * 3, 48, 3, 2, 64),
]


@pytest.mark.parametrize("shape", SIMT_SHAPES)
def test_swapped_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N = shape
    diff, rms, ws = C.c_float(), C.c_float(), C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_pool3_simt(M, Cin, KW, dil, N, C.byref(diff), C.byref(rms), C.byref(ws)))
    assert ws.value == 1, "the shape should take the weight-stationary kernel"
    tol = 3e-5 * rms.value * (KW * Cin / 64) ** 0.5
    assert diff.value == diff.value, "NaN in the comparison"
    assert diff.value < tol, f"max abs diff {diff.value:.3e}, tol {tol:.3e}"
