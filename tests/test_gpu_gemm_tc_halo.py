"""The halo operand mode of the wgmma GEMM: a Conv1d tile loads its rows once and every tap's A descriptor starts a whole
number of rows into the 64B-swizzled halo.  Checks that the descriptor row shift is exact, that the halo mode writes the
same bytes as the tap-box mode (for SincNet's 80-channel conv1: the folded overlapping-row form it replaces), and that it
matches the float32 SIMT GEMM within test_gpu_gemm_tc.py's tolerance."""
import ctypes as C

import pytest

from diart_b200 import _lib

pytestmark = pytest.mark.gpu


def test_wgmma_descriptor_row_shift(cuda_device):
    # base offset field 0: the swizzle follows the absolute shared-memory address, so a start r rows into a tile is exact
    ok = C.c_uint()
    _lib.check(_lib.lib().dg_selftest_wgmma_row_shift(0, C.byref(ok)))
    assert ok.value == 0x1FF, f"shifts 0..8 exact: {ok.value:09b}"


HALO_SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (888 * 6, 80, 5, 1, 60, 5),      # sinc_conv1: MaxPool1d(3) epilogue, 111-row tiles, 6 items, last halo past M
    (888 * 2, 64, 5, 1, 60, 5),      # sinc_conv2
    (2368, 64, 5, 1, 512, 1),        # tdnn1: split epilogue, 4 column tiles
    (1000, 80, 5, 1, 64, 0),         # sinc_conv1 without the pooling epilogue, ragged M
    (777, 64, 3, 2, 128, 2),         # dilation 2, ragged M
    (40000, 64, 5, 1, 64, 0),        # 313 tiles: more than one per SM
]


@pytest.mark.parametrize("shape", HALO_SHAPES)
def test_halo_equals_tap_boxes(shape, cuda_device):
    equal, halo = C.c_int(), C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_halo(*shape, C.byref(equal), C.byref(halo)))
    assert halo.value == 1, "the shape should take the halo mode"
    assert equal.value == 1


SIMT_SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (5328, 80, 5, 1, 64, 0),         # sinc_conv1
    (1776, 64, 5, 1, 64, 0),         # sinc_conv2
    (2368, 64, 5, 1, 512, 1),        # tdnn1
]


@pytest.mark.parametrize("shape", SIMT_SHAPES)
def test_halo_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N, epi = shape
    diff, rms = C.c_float(), C.c_float()
    _lib.check(_lib.lib().dg_selftest_gemm_tc(M, Cin, KW, dil, N, epi, C.byref(diff), C.byref(rms)))
    tol = 3e-5 * rms.value * (KW * Cin / 64) ** 0.5
    assert diff.value == diff.value, "NaN in the comparison"
    assert diff.value < tol, f"max abs diff {diff.value:.3e}, tol {tol:.3e}"
