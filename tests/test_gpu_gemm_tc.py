"""The wgmma/TMA shifted-window GEMM (gemm_tc) through its self-test entry points.

- Against the float32 SIMT GEMM on the same seeded random operands, layer shapes of the path.  Bar: max |diff| < 3e-5 x
  output RMS x sqrt(K/64) (three bf16 products carry 16 significand bits per operand).
- The ping-pong kernel (two consumer warpgroups, one shared staging tile for the element-wise epilogues) at the tile counts
  where its hand-offs matter, against the SIMT GEMM, and the independence of every epilogue's output from the grid it runs on.
- The halo operand mode: a Conv1d tile loads its rows once and every tap's A descriptor starts a whole number of rows into
  the 64B-swizzled halo.  Checks that the descriptor row shift is exact, that the halo mode writes the same bytes as the
  tap-box mode (for SincNet's 80-channel conv1: the folded overlapping-row form it replaces), and that it matches the SIMT
  GEMM.
- The weight-stationary MaxPool3 kernel (SincNet's conv1 and conv2): W stays in shared memory as the A operand and the
  tile's halo rows are the B operand (D^T = W . X^T).  Checks that a B descriptor may start any whole number of rows into a
  64B-swizzled tile, that the kernel is taken for SincNet's shapes and writes the bytes of the tap-box kernel, and that its
  pooled rows match the SIMT GEMM pooled on the host.
- The TMA box stores of the element-wise epilogues (bias -> float32, LeakyReLU + BatchNorm -> hi/lo planes or float32):
  with an output pitch wider than N and guard rows after M, only rows [0, M) x columns [0, N) change and they hold the
  bytes of the same GEMM written at pitch N; an output base or pitch off 16-byte alignment is refused."""
import ctypes as C

import pytest

from diart_b200 import _lib

pytestmark = pytest.mark.gpu


def simt_tol(rms, KW, Cin):
    """the bar against the float32 SIMT GEMM: 3e-5 x output RMS x sqrt(K/64)"""
    return 3e-5 * rms * (KW * Cin / 64) ** 0.5


# ---------------------------------------------------------------------------------------------- against the SIMT GEMM
SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (1000, 64, 1, 1, 256, 0),        # one k-block, ragged M
    (2368, 64, 5, 1, 512, 1),        # tdnn1-like, split epilogue
    (1184, 512, 3, 2, 512, 1),       # tdnn2 (dilation 2)
    (1184, 512, 3, 3, 512, 2),       # tdnn3 (dilation 3), f32 epilogue
    (1184, 512, 1, 1, 1500, 2),      # tdnn5: N not a multiple of the tile
    (4096, 256, 1, 1, 1024, 0),      # LSTM input projection
    (300, 128, 2, 7, 128, 0),        # BN=128 variant, odd dilation
    (5328, 128, 5, 1, 64, 0),        # SincNet conv1 (80 -> 128 padded channels, N = 64 of a 128 tile)
    (768, 3008, 1, 1, 512, 0),       # Linear(3000, 512) with K padded to 47 k-blocks
]


@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_tc_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N, epi = shape
    diff, rms = C.c_float(), C.c_float()
    _lib.check(_lib.lib().dg_selftest_gemm_tc(M, Cin, KW, dil, N, epi, C.byref(diff), C.byref(rms)))
    tol = simt_tol(rms.value, KW, Cin)
    print(f"shape {shape}: max abs diff {diff.value:.3e}, output rms {rms.value:.3e}, tol {tol:.3e}")
    assert diff.value == diff.value, "NaN in the comparison"
    assert diff.value < tol


# ---------------------------------------------------------------------------------------------- ping-pong consumers
PINGPONG_SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (33900, 64, 1, 1, 128, 0),       # 265 m-tiles: more than the grid, an odd number of tiles on some CTAs
    (128, 64, 1, 1, 128, 1),         # one tile: the second consumer never gets one
    (32768, 64, 1, 1, 1024, 0),      # K = 64 and many tiles: the epilogue is longer than the mainloop
    (1001, 64, 1, 1, 200, 0),        # ragged M and N, bias -> float32
    (777, 128, 3, 2, 352, 1),        # ragged M and N, hi/lo planes
    (999, 64, 1, 1, 72, 2),          # ragged M and N, LeakyReLU + BatchNorm -> float32
]


@pytest.mark.parametrize("shape", PINGPONG_SHAPES)
def test_gemm_tc_pingpong_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N, epi = shape
    diff, rms = C.c_float(), C.c_float()
    _lib.check(_lib.lib().dg_selftest_gemm_tc(M, Cin, KW, dil, N, epi, C.byref(diff), C.byref(rms)))
    tol = simt_tol(rms.value, KW, Cin)
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


# ---------------------------------------------------------------------------------------------- halo operand mode
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


HALO_SIMT_SHAPES = [  # (M, Cin, KW, dil, N, epi)
    (5328, 80, 5, 1, 64, 0),         # sinc_conv1
    (1776, 64, 5, 1, 64, 0),         # sinc_conv2
    (2368, 64, 5, 1, 512, 1),        # tdnn1
]


@pytest.mark.parametrize("shape", HALO_SIMT_SHAPES)
def test_halo_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N, epi = shape
    diff, rms = C.c_float(), C.c_float()
    _lib.check(_lib.lib().dg_selftest_gemm_tc(M, Cin, KW, dil, N, epi, C.byref(diff), C.byref(rms)))
    tol = simt_tol(rms.value, KW, Cin)
    assert diff.value == diff.value, "NaN in the comparison"
    assert diff.value < tol, f"max abs diff {diff.value:.3e}, tol {tol:.3e}"


# ---------------------------------------------------------------------------------------------- weight-stationary MaxPool3
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


SWAPPED_SIMT_SHAPES = [  # (M, Cin, KW, dil, N)
    (888 * 6, 80, 5, 1, 60),         # sinc_conv1
    (888 * 2, 64, 5, 1, 60),         # sinc_conv2
    (888 * 3, 48, 3, 2, 64),
]


@pytest.mark.parametrize("shape", SWAPPED_SIMT_SHAPES)
def test_swapped_matches_simt(shape, cuda_device):
    M, Cin, KW, dil, N = shape
    diff, rms, ws = C.c_float(), C.c_float(), C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_pool3_simt(M, Cin, KW, dil, N, C.byref(diff), C.byref(rms), C.byref(ws)))
    assert ws.value == 1, "the shape should take the weight-stationary kernel"
    tol = simt_tol(rms.value, KW, Cin)
    assert diff.value == diff.value, "NaN in the comparison"
    assert diff.value < tol, f"max abs diff {diff.value:.3e}, tol {tol:.3e}"


# ---------------------------------------------------------------------------------------------- TMA box stores
BOUNDS_SHAPES = [  # (M, Cin, N, epi); N <= 64 runs on 64-wide tiles for epi 0 (one partial 128-wide tile for epi 1 and 2)
    (1001, 64, 36, 0),       # 64-wide tiles: ragged M, one partial 32-column box
    (3001, 128, 200, 0),     # 128-wide tiles: ragged M, the second column tile ragged
    (777, 64, 52, 2),        # one partial column tile, LeakyReLU + BatchNorm -> float32
    (2049, 64, 300, 2),      # three column tiles, the last one ragged
    (999, 128, 32, 1),       # hi/lo planes: one partial 64-column box
    (1500, 64, 160, 1),      # two column tiles, the second one holds half a box
]


@pytest.mark.parametrize("shape", BOUNDS_SHAPES)
def test_gemm_tc_box_store_stays_inside_the_output(shape, cuda_device):
    M, Cin, N, epi = shape
    outside, equal, refused = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib().dg_selftest_gemm_tc_bounds(M, Cin, N, epi, C.byref(outside), C.byref(equal), C.byref(refused)))
    assert outside.value == 1, f"shape {shape}: bytes outside rows [0, M) x columns [0, N) changed"
    assert equal.value == 1, f"shape {shape}: the output at pitch N + 40 differs from the output at pitch N"
    assert refused.value == 1, f"shape {shape}: a misaligned output base or pitch was accepted"
