"""The ping-pong gemm_tc kernel (two consumer warpgroups, one shared staging tile for the element-wise epilogues) at the
tile counts where its hand-offs matter, against the float32 SIMT GEMM (same bar as test_gpu_gemm_tc.py), and the
independence of every epilogue's output from the grid it runs on."""
import ctypes as C

import pytest

from diart_b200 import _lib

pytestmark = pytest.mark.gpu

SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (33900, 64, 1, 1, 128, 0),       # 265 m-tiles: more than the grid, an odd number of tiles on some CTAs
    (128, 64, 1, 1, 128, 1),         # one tile: the second consumer never gets one
    (32768, 64, 1, 1, 1024, 0),      # K = 64 and many tiles: the epilogue is longer than the mainloop
    (1001, 64, 1, 1, 200, 0),        # ragged M and N, bias -> float32
    (777, 128, 3, 2, 352, 1),        # ragged M and N, hi/lo planes
    (999, 64, 1, 1, 72, 2),          # ragged M and N, LeakyReLU + BatchNorm -> float32
]


@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_tc_pingpong_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N, epi = shape
    diff, rms = C.c_float(), C.c_float()
    _lib.check(_lib.lib().dg_selftest_gemm_tc(M, Cin, KW, dil, N, epi, C.byref(diff), C.byref(rms)))
    tol = 3e-5 * rms.value * (KW * Cin / 64) ** 0.5
    print(f"shape {shape}: max abs diff {diff.value:.3e}, output rms {rms.value:.3e}, tol {tol:.3e}")
    assert diff.value == diff.value, "NaN in the comparison"
    assert diff.value < tol


def test_gemm_tc_planes_reject_partial_column_groups(cuda_device):
    # hi/lo planes are stored 32 columns at a time: N = 328 would overwrite the first columns of the next row
    diff, rms = C.c_float(), C.c_float()
    with pytest.raises(ValueError, match="multiple of 32"):
        _lib.check(_lib.lib().dg_selftest_gemm_tc(777, 128, 3, 2, 328, 1, C.byref(diff), C.byref(rms)))


GRID_SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (3000, 64, 1, 1, 200, 0),        # bias -> float32, 128-wide tiles
    (3000, 128, 1, 1, 64, 0),        # bias -> float32, 64-wide tiles
    (2000, 128, 3, 2, 512, 1),       # LeakyReLU + BatchNorm -> hi/lo planes
    (1500, 64, 2, 3, 1500, 2),       # LeakyReLU + BatchNorm -> float32
    (2880, 64, 9, 12, 128, 3),       # Conv2d on 12 x 12 padded maps, residual, ReLU; 128-wide tiles
    (2880, 64, 9, 12, 64, 3),        # 64-wide tiles
    (2880, 64, 9, 12, 32, 3),        # 32-wide tiles
    (1776, 64, 1, 1, 256, 4),        # statistics pooling
    (2664, 64, 5, 1, 64, 5),         # MaxPool1d(3) + InstanceNorm partial sums
]


@pytest.mark.parametrize("shape", GRID_SHAPES)
def test_gemm_tc_output_does_not_depend_on_grid(shape, cuda_device):
    equal = C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_grid(*shape, C.byref(equal)))
    assert equal.value == 1, f"shape {shape}: outputs differ between SM caps 0, 1, 3 and 7"
