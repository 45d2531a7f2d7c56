"""The C-ABI library builds, loads without a GPU, and exports every symbol include/diart_b200.h declares
(no compute calls here)."""
import ctypes
import os
import re

from diart_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    text = open(os.path.join(ROOT, "include", "diart_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dg_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = _lib.lib()
    names = header_functions()
    assert len(names) >= 25
    for name in names:
        assert hasattr(lib, name), f"{name} is declared in the header but not exported"
    assert set(names) == set(_lib.SIGNATURES), "ctypes signature table and header disagree"
    assert lib.dg_version() >= 100
    assert isinstance(lib.dg_last_error(), bytes)


def test_argument_errors_without_gpu():
    lib = _lib.lib()
    assert lib.dg_seg_create(None, 0, 0, None) == -1
    assert b"null" in lib.dg_last_error()
    assert lib.dg_emb_create(None, 0, 77, 0, None) == -1
    assert lib.dg_osp(None, 1, 1, 1, 3.0, 10.0, 0, None, None) == -1
    out = ctypes.c_void_p()
    assert lib.dg_cluster_create(64, 512, 0.6, 0.3, 1.0, 0, ctypes.byref(out)) == -1   # > 32 global speakers


def test_host_fp16_split_matches_ieee():
    """The host-side hi/lo split of weights into fp16 planes is IEEE round-to-nearest-even: checked against numpy
    float16, including subnormals, ties and saturation."""
    import numpy as np

    lib = _lib.lib()
    rng = np.random.default_rng(7)
    x = np.concatenate([
        rng.standard_normal(20000).astype(np.float32) * np.float32(10.0) ** rng.integers(-9, 5, 20000).astype(np.float32),
        np.array([0.0, -0.0, 1.0, -1.0, 65504.0, 65519.9, 65520.0, 1e6, -1e6, 6.1035e-5, 6.0e-8, 2.98e-8, 2.9802322e-8,
                  3.0e-8, 8.9e-8, 1.0009766, 1.0004883, 1.0014648, np.inf, -np.inf], np.float32)])
    hi = np.empty(x.size, np.uint16)
    lo = np.empty(x.size, np.uint16)
    assert lib.dg_selftest_split_f16_host(x.ctypes.data, x.size, hi.ctypes.data, lo.ctypes.data) == 0
    with np.errstate(over="ignore"):
        ref_hi = np.clip(x, -65504, 65504).astype(np.float16)
        ref_hi = np.where(np.abs(x) >= 65520, np.sign(x) * np.float16(65504), x.astype(np.float16)).astype(np.float16)
        res = x - ref_hi.astype(np.float32)
        ref_lo = np.where(np.abs(res) >= 65520, np.sign(res) * np.float16(65504), res.astype(np.float16)).astype(np.float16)
    assert np.array_equal(hi, ref_hi.view(np.uint16))
    fin = np.isfinite(x)
    assert np.array_equal(lo[fin], ref_lo.view(np.uint16)[fin])
    back = hi.view(np.float16).astype(np.float64) + lo.view(np.float16).astype(np.float64)
    ok = fin & (np.abs(x) < 6e4)
    # 22 significand bits for the pair, with the absolute floor of the fp16 subnormal step (2^-25 after rounding)
    assert np.all(np.abs(back[ok] - x[ok]) <= np.maximum(np.abs(x[ok]) * 2.0 ** -21, 2.0 ** -25 * 1.0001))
